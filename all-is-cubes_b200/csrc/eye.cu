// eye.cu — characters' eyes on the device: step_eye_position (all-is-cubes/src/character/eye.rs:90-121) and
// compute_view_transform (eye.rs:187-203) with the world camera StandardCameras::update builds from it (stdcam.rs:237-256:
// set_view_transform, compute_matrices, set_measured_exposure), for a batch of eyes on one context, or on a device
// group's device 0, where its camera table and exposure outputs live.  One thread per eye, uncontracted f64
// (-fmad=false), as the reference's.  The camera matrices are camera_math.cuh's, the host's own code, and the look
// ray is the frames' project_ndc.  Neither call reads or changes the scene: it fixes the device and the stream.
#include <cmath>

#include "camera_math.cuh"
#include "internal.h"

using namespace aicb;

static_assert(sizeof(aicb_eye) == 72, "aicb_eye is 72 bytes");
static_assert(sizeof(aicb_eye_view_params) == 48, "aicb_eye_view_params is 48 bytes");

namespace {

constexpr unsigned EYES_PER_BLOCK = 128;

struct EyeStepParams {
    aicb_eye *eyes;
    const aicb_body *bodies;
    uint64_t n;
    double dt;
    double k21;   // 1e21^dt
    double k9;    // 1e-9^dt
};

// set_measured_exposure's rule for the batch (camera_struct.rs:169-181)
enum : uint32_t { EXPOSURE_FIXED = 0, EXPOSURE_AUTOMATIC_ONE = 1, EXPOSURE_AUTOMATIC = 2 };

struct EyeViewParams {
    const aicb_eye *eyes;
    const aicb_body *bodies;
    const double *rotations;   // [n][4] i, j, k, r
    const float *exposures;    // [n] or nullptr
    double *eye_to_world;      // [n][16] or nullptr
    aicb_camera *cameras;      // [n] or nullptr
    double *look_rays;         // [n][6] or nullptr
    uint32_t *status;          // [n] or nullptr
    uint64_t n;
    double fov_cot, aspect, far;   // camera_math::projection_terms of the batch's options and viewport
    uint32_t fb_width, fb_height;
    float fixed_exposure;
    uint32_t exposure_rule;
};

// step_eye_position (eye.rs:107-116) for one eye: euclid's vector operators component by component.
__global__ void __launch_bounds__(EYES_PER_BLOCK) eye_step_kernel(const __grid_constant__ EyeStepParams P) {
    const uint64_t i = (uint64_t)blockIdx.x * EYES_PER_BLOCK + threadIdx.x;
    if (i >= P.n) return;
    aicb_eye &e = P.eyes[i];
    const aicb_body &b = P.bodies[i];
    double p[3], vel[3], v[3];
    for (int a = 0; a < 3; a++) {
        p[a] = e.displacement_pos[a];
        vel[a] = e.displacement_vel[a];
        v[a] = b.velocity[a];
    }
    for (int a = 0; a < 3; a++) vel[a] = vel[a] - (v[a] - e.previous_body_velocity[a]) * 0.04;
    const double len = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);   // Vector3D::length
    for (int a = 0; a < 3; a++) vel[a] = vel[a] - (p[a] * (len + 1.0)) * P.k21;
    for (int a = 0; a < 3; a++) vel[a] = vel[a] * P.k9;
    for (int a = 0; a < 3; a++) p[a] = p[a] + vel[a] * P.dt;
    for (int a = 0; a < 3; a++) {
        e.displacement_pos[a] = p[a];
        e.displacement_vel[a] = vel[a];
        e.previous_body_velocity[a] = v[a];   // the next tick's record_previous_velocity
    }
}

__global__ void __launch_bounds__(EYES_PER_BLOCK) eye_views_kernel(const __grid_constant__ EyeViewParams P) {
    const uint64_t i = (uint64_t)blockIdx.x * EYES_PER_BLOCK + threadIdx.x;
    if (i >= P.n) return;
    const aicb_eye &e = P.eyes[i];
    const aicb_body &b = P.bodies[i];
    const double *q = P.rotations + 4 * i;
    const camera_math::Quat rot{q[0], q[1], q[2], q[3]};
    // compute_view_transform: the body's position plus the displacement
    const double t[3] = {b.position[0] + e.displacement_pos[0], b.position[1] + e.displacement_pos[1],
                         b.position[2] + e.displacement_pos[2]};
    double m[16];
    if (!camera_math::projection_view_inverse(rot, t, P.fov_cot, P.aspect, P.far, m)) {
        if (P.status) P.status[i] = AICB_EYE_NOT_INVERTIBLE;
        return;
    }
    if (P.eye_to_world) camera_math::view_transform_matrix(rot, t, P.eye_to_world + 16 * i);
    if (P.cameras) {
        aicb_camera &c = P.cameras[i];
        float exposure;
        if (P.exposure_rule == EXPOSURE_FIXED) {
            exposure = P.fixed_exposure;
        } else {
            exposure = c.exposure;
            if (P.exposures) {
                const float v = P.exposures[i];
                // PositiveSign::try_from: not NaN, not negative; -0 is +0
                if (!(v != v) && !(v < 0.0f)) exposure = P.exposure_rule == EXPOSURE_AUTOMATIC_ONE ? 1.0f
                                                         : (v == 0.0f ? 0.0f : v);
            }
        }
        for (int k = 0; k < 16; k++) c.inverse_projection_view[k] = m[k];
        c.fb_width = P.fb_width;
        c.fb_height = P.fb_height;
        c.exposure = exposure;
        c._pad = 0;
    }
    if (P.look_rays) {
        // Camera::project_ndc_into_world((0, 0)): the near and far points of the screen centre
        double o[3], f[3];
        project_ndc(m, 0.0, 0.0, 0.0, o);
        project_ndc(m, 0.0, 0.0, 1.0, f);
        double *r = P.look_rays + 6 * i;
        for (int a = 0; a < 3; a++) {
            r[a] = o[a];
            r[3 + a] = f[a] - o[a];
        }
    }
    if (P.status) P.status[i] = 0;
}

unsigned blocks_for(size_t n) { return (unsigned)((n + EYES_PER_BLOCK - 1) / EYES_PER_BLOCK); }

// Both calls run on c0 alone, a context or a group's device 0, ordered after the caller's stream and before its next
// work (join_caller / release_caller).
aicb_status step_eyes(aicb_ctx *c0, aicb_eye *eyes, const aicb_body *bodies, size_t n, double dt,
                      cudaStream_t caller) {
    CU(cudaSetDevice(c0->device));
    if (!(dt > 0.0 && dt <= 1.0)) return aicb_fail(AICB_ERR_INVALID, "dt must be finite and in (0, 1]");
    if (n == 0) return AICB_OK;
    if (!eyes || !bodies) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_device_pointer(eyes, c0->device, false, 8, "eyes"));
    TRY(check_device_pointer(bodies, c0->device, false, 8, "bodies"));
    if (n > (size_t)UINT32_MAX * EYES_PER_BLOCK) return aicb_fail(AICB_ERR_INVALID, "too many eyes");
    EyeStepParams P;
    memset(&P, 0, sizeof P);
    P.eyes = eyes;
    P.bodies = bodies;
    P.n = n;
    P.dt = dt;
    P.k21 = std::pow(1e21, dt);   // f64::powf
    P.k9 = std::pow(1e-9, dt);
    TRY(join_caller(&c0, 1, caller));
    eye_step_kernel<<<blocks_for(n), EYES_PER_BLOCK, 0, c0->stream.get()>>>(P);
    CU(cudaGetLastError());
    return release_caller(c0, caller);
}

aicb_status eye_views(aicb_ctx *c0, const aicb_eye *eyes, const aicb_body *bodies, const double (*rotations)[4],
                      const float *exposures, size_t n, const aicb_eye_view_params *params, double (*eye_to_world)[16],
                      aicb_camera *cameras, double (*look_rays)[6], uint32_t *status, cudaStream_t caller) {
    CU(cudaSetDevice(c0->device));
    if (!params) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n == 0) return AICB_OK;
    if (!eyes || !bodies || !rotations) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_device_pointer(eyes, c0->device, false, 8, "eyes"));
    TRY(check_device_pointer(bodies, c0->device, false, 8, "bodies"));
    TRY(check_device_pointer(rotations, c0->device, false, 8, "rotations"));
    if (exposures) TRY(check_device_pointer(exposures, c0->device, false, 4, "exposures"));
    if (eye_to_world) TRY(check_device_pointer(eye_to_world, c0->device, false, 8, "eye_to_world"));
    if (cameras) TRY(check_device_pointer(cameras, c0->device, false, 8, "cameras"));
    if (look_rays) TRY(check_device_pointer(look_rays, c0->device, false, 8, "look_rays"));
    if (status) TRY(check_device_pointer(status, c0->device, false, 4, "status"));
    if (n > (size_t)UINT32_MAX * EYES_PER_BLOCK) return aicb_fail(AICB_ERR_INVALID, "too many eyes");
    EyeViewParams P;
    memset(&P, 0, sizeof P);
    P.eyes = eyes;
    P.bodies = bodies;
    P.rotations = &rotations[0][0];
    P.exposures = exposures;
    P.eye_to_world = eye_to_world ? &eye_to_world[0][0] : nullptr;
    P.cameras = cameras;
    P.look_rays = look_rays ? &look_rays[0][0] : nullptr;
    P.status = status;
    P.n = n;
    camera_math::projection_terms(params->fov_y_degrees, params->view_distance, params->nominal_width,
                                  params->nominal_height, &P.fov_cot, &P.aspect, &P.far);
    P.fb_width = params->fb_width;
    P.fb_height = params->fb_height;
    P.fixed_exposure = params->fixed_exposure;
    P.exposure_rule = !params->automatic_exposure                      ? EXPOSURE_FIXED
                      : params->lighting_display == AICB_LIGHT_NONE ? EXPOSURE_AUTOMATIC_ONE
                                                                       : EXPOSURE_AUTOMATIC;
    TRY(join_caller(&c0, 1, caller));
    eye_views_kernel<<<blocks_for(n), EYES_PER_BLOCK, 0, c0->stream.get()>>>(P);
    CU(cudaGetLastError());
    return release_caller(c0, caller);
}

}  // namespace

extern "C" {

aicb_status aicb_step_eyes_device(aicb_scene *s, aicb_eye *eyes, const aicb_body *bodies, size_t n, double dt,
                                  void *stream) {
    return on_scene(s, [&](Replicas r) { return step_eyes(r.ctx[0], eyes, bodies, n, dt, (cudaStream_t)stream); });
}

aicb_status aicb_eye_views_device(aicb_scene *s, const aicb_eye *eyes, const aicb_body *bodies,
                                  const double (*rotations)[4], const float *exposures, size_t n,
                                  const aicb_eye_view_params *params, double (*eye_to_world)[16], aicb_camera *cameras,
                                  double (*look_rays)[6], uint32_t *status, void *stream) {
    return on_scene(s, [&](Replicas r) {
        return eye_views(r.ctx[0], eyes, bodies, rotations, exposures, n, params, eye_to_world, cameras, look_rays,
                         status, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_step_eyes_device(aicb_group_scene *gs, aicb_eye *eyes, const aicb_body *bodies, size_t n,
                                        double dt, void *stream) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return step_eyes(gs->group->ctx[0], eyes, bodies, n, dt, (cudaStream_t)stream);
}

aicb_status aicb_group_eye_views_device(aicb_group_scene *gs, const aicb_eye *eyes, const aicb_body *bodies,
                                        const double (*rotations)[4], const float *exposures, size_t n,
                                        const aicb_eye_view_params *params, double (*eye_to_world)[16],
                                        aicb_camera *cameras, double (*look_rays)[6], uint32_t *status, void *stream) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return eye_views(gs->group->ctx[0], eyes, bodies, rotations, exposures, n, params, eye_to_world, cameras,
                     look_rays, status, (cudaStream_t)stream);
}

}  // extern "C"
