// exposure.cu — automatic exposure over a scene's cells and light on the device: character::exposure::State::step
// (all-is-cubes/src/character/exposure.rs:67-136) for a batch of eyes, on one context and on a device group.  One warp
// per eye: lanes 0-9 each cast one of the tick's 10 rays with the frames' Raycaster arithmetic (caster_begin /
// caster_step), the warp's copy of the 100 samples lives in shared memory, and lane 0 folds them in array order.  A
// block's Derived::visible is BLOCK_VISIBLE in its record, derived when it is placed.  A call reads the scene and writes
// only the states and exposures: the host mirror of the block ids, the light state and a frame in flight are left
// alone.  All f32 arithmetic is uncontracted (-fmad=false), as the reference's.
#include <cmath>
#include <vector>

#include "exact_math.cuh"
#include "internal.h"

using namespace aicb;

namespace {

constexpr int N_SAMPLES = 100;   // State::luminance_samples
constexpr int N_RAYS = 10;       // rays per tick
constexpr unsigned EYES_PER_BLOCK = 4;

struct ExposureParams {
    DeviceScene scene;
    uint64_t max_steps;            // 0 under LightPhysics::None, else 2 * maximum_distance
    float dt;                      // dt as f32
    uint32_t step;                 // dt != 0: the reference returns early at dt == 0
    aicb_exposure_state *states;   // [n], in place
    const double *m;               // [n][16] eye-to-world, m11..m44
    float *out;                    // [n] State::exposure(), or nullptr
    uint64_t n;
};

// A cube's block id from its cell word.
__device__ __forceinline__ uint32_t cell_id(const DeviceScene &S, uint32_t idx) {
    return S.wide_cells ? (__ldg((const uint32_t *)S.cells + idx) & 0xffffu)
                        : ((uint32_t)__ldg((const uint16_t *)S.cells + idx) & 0x3fffu);
}

// Rgb::luminance (color.rs:288-297)
__device__ __forceinline__ float luminance(float r, float g, float b) { return g * 0.7152f + (r * 0.2126f + b * 0.0722f); }

// Sky::sample(direction).luminance() (sky.rs:32-41): the octant of the direction as given, -0.0 counting as >= 0.
__device__ float sky_luminance(const DeviceScene &S, const double d[3]) {
    const int k = S.sky_kind ? ((d[0] >= 0.0) << 2) + ((d[1] >= 0.0) << 1) + (d[2] >= 0.0) : 0;
    return luminance(S.sky_colors[k][0], S.sky_colors[k][1], S.sky_colors[k][2]);
}

// One ray's sample: `for step in ray.cast().within(bounds, false).take(max_steps)` (exposure.rs:100-119).  Every step
// of the cast is in the bounds (the exit step is not one), so cube_ahead is always a cube of the Space.
__device__ float ray_sample(const DeviceScene &S, uint64_t max_steps, const double o[3], const double d_in[3]) {
    double d[3] = {d_in[0], d_in[1], d_in[2]};
    // Parameters::new (raycast.rs:749-771)
    if (!((fabs(d[0]) < 1e100) & (fabs(d[1]) < 1e100) & (fabs(d[2]) < 1e100))) d[0] = d[1] = d[2] = 0.0;
    Ray r;
    r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
    r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    r.sx = signum_101(d[0]); r.sy = signum_101(d[1]); r.sz = signum_101(d[2]);
    r.tdx = 1.0 / fabs(d[0]); r.tdy = 1.0 / fabs(d[1]); r.tdz = 1.0 / fabs(d[2]);
    r.half_over_len = 0.5 / sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    Level lv;
    lv.lox = S.lo[0]; lv.loy = S.lo[1]; lv.loz = S.lo[2];
    lv.nx = S.size[0]; lv.ny = S.size[1]; lv.nz = S.size[2];
    lv.base = 0;
    Caster cs;
    bool valid;
    if (max_steps == 0 || !caster_begin(cs, r, o[0], o[1], o[2], lv, &valid)) return sky_luminance(S, d_in);
    for (uint64_t steps = 1;; steps++) {
        const uint32_t id = cell_id(S, cs.idx);
        if (__ldg(&S.blocks[id].flags) & BLOCK_VISIBLE) {
            // get_light(cube_behind): the cube itself when the ray starts inside it (Face7::Within)
            uint32_t t;
            if (cs.face == AICB_FACE_WITHIN) {
                t = S.light ? __ldg(S.light + cs.idx) : TEXEL_ONE;
            } else {
                int c[3] = {cs.rx + S.lo[0], cs.ry + S.lo[1], cs.rz + S.lo[2]};
                c[(cs.face - 1) % 3] += cs.face >= AICB_FACE_PX ? 1 : -1;
                const uint32_t dx = (uint32_t)(c[0] - S.lo[0]), dy = (uint32_t)(c[1] - S.lo[1]),
                               dz = (uint32_t)(c[2] - S.lo[2]);
                if ((dx < (uint32_t)S.size[0]) & (dy < (uint32_t)S.size[1]) & (dz < (uint32_t)S.size[2]))
                    t = S.light ? __ldg(S.light + (dx * (uint32_t)S.size[1] + dy) * (uint32_t)S.size[2] + dz) : TEXEL_ONE;
                else
                    t = S.light ? light_outside(S, c[0], c[1], c[2]) : TEXEL_ONE;
            }
            if ((t >> 24) == 255u)   // PackedLight::valid: LightStatus::Visible alone (data.rs:127-135)
                return luminance(__ldg(S.tables + (t & 255u)), __ldg(S.tables + ((t >> 8) & 255u)),
                                 __ldg(S.tables + ((t >> 16) & 255u)));
        }
        if (steps >= max_steps || !valid || caster_step(cs, r, lv.nx, lv.ny, lv.nz)) return sky_luminance(S, d_in);
    }
}

__global__ void __launch_bounds__(32 * EYES_PER_BLOCK) exposure_kernel(const __grid_constant__ ExposureParams P) {
    __shared__ float samples[EYES_PER_BLOCK][N_SAMPLES];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint64_t i = (uint64_t)blockIdx.x * EYES_PER_BLOCK + w;
    if (i >= P.n) return;   // the whole warp
    aicb_exposure_state &st = P.states[i];
    float exposure_log = st.exposure_log;
    const double *m = P.m + 16 * i;
    // vt.transform_point3d(Point3D::origin()): euclid's sums with the zero coordinates kept (0 * inf is NaN), and
    // None unless w > 0
    const double hw = 0.0 * m[3] + 0.0 * m[7] + 0.0 * m[11] + m[15];
    if (P.step && hw > 0.0) {
        float *s = samples[w];
        for (int k = (int)lane; k < N_SAMPLES; k += 32) s[k] = st.luminance_samples[k];
        // the index advances before each ray, as a usize: (index + 1) % 100, then + 1 per ray
        const uint32_t first = (uint32_t)(((uint64_t)st.luminance_sample_index + 1u) % N_SAMPLES);
        __syncwarp();
        if (lane < N_RAYS) {
            const uint32_t index = (first + lane) % N_SAMPLES;
            const double o[3] = {(0.0 * m[0] + 0.0 * m[4] + 0.0 * m[8] + m[12]) / hw,
                                 (0.0 * m[1] + 0.0 * m[5] + 0.0 * m[9] + m[13]) / hw,
                                 (0.0 * m[2] + 0.0 * m[6] + 0.0 * m[10] + m[14]) / hw};
            // vec3(index.rem_euclid(10) / 10 * 2 - 1, index.div_euclid(10) / 10 * 2 - 1, -1), not normalised
            const double vx = (double)(index % 10u) / 10.0 * 2.0 - 1.0, vy = (double)(index / 10u) / 10.0 * 2.0 - 1.0,
                         vz = -1.0;
            const double d[3] = {vx * m[0] + vy * m[4] + vz * m[8], vx * m[1] + vy * m[5] + vz * m[9],
                                 vx * m[2] + vy * m[6] + vz * m[10]};
            s[index] = ray_sample(P.scene, P.max_steps, o, d);
        }
        __syncwarp();
        if (lane == 0) {
            // luminance_average: Sum for f32 folds from -0.0 in array order, times 100f32.recip()
            float sum = -0.0f;
            for (int k = 0; k < N_SAMPLES; k++) sum = sum + s[k];
            const float avg = sum * (1.0f / 100.0f);
            // compute_target_exposure (exposure.rs:168-174); f32::clamp lets NaN through
            float derived = 0.9f / avg;
            if (derived < 0.1f) derived = 0.1f;
            if (derived > 4.0f) derived = 4.0f;
            const float target = derived * 0.375f + 1.0f * (1.0f - 0.375f);
            if (isfinite(target)) exposure_log = exposure_log + (logf_exact(target) - exposure_log) * P.dt * 2.0f;
            st.luminance_sample_index = (first + N_RAYS - 1) % N_SAMPLES;
            st.exposure_log = exposure_log;
        }
        for (int k = (int)lane; k < N_SAMPLES; k += 32) st.luminance_samples[k] = s[k];
    }
    if (lane == 0 && P.out) P.out[i] = expf_libm(exposure_log);
}

// The eyes (in device 0's memory) in ranges, one per listed context; context i walks its own replica and stores into
// device 0's buffers.  Device 0's stream ends after every part (fan_in), and device 0 is current.
aicb_status issue_exposure(Replicas r, double dt, aicb_exposure_state *states, const double *m, float *out, size_t n) {
    const std::vector<WarpRange> ranges = warp_ranges(n, r.n);
    TRY(fan_out(r.ctx, ranges.size()));
    for (size_t i = 0; i < ranges.size(); i++) {
        const size_t begin = ranges[i].begin, count = ranges[i].count;
        if (count == 0) continue;
        ExposureParams P;
        memset(&P, 0, sizeof P);
        P.scene = r.scene[i]->ds;
        P.max_steps = 2 * (uint64_t)r.scene[i]->host->light_max_distance;
        P.dt = (float)dt;
        P.step = dt != 0.0 ? 1u : 0u;
        P.states = states + begin;
        P.m = m + 16 * begin;
        P.out = out ? out + begin : nullptr;
        P.n = count;
        CU(cudaSetDevice(r.ctx[i]->device));
        exposure_kernel<<<(unsigned)((count + EYES_PER_BLOCK - 1) / EYES_PER_BLOCK), 32 * EYES_PER_BLOCK, 0,
                          r.ctx[i]->stream.get()>>>(P);
        CU(cudaGetLastError());
    }
    return fan_in(r.ctx, ranges.size());
}

aicb_status check_dt(double dt) {
    if (!(dt >= 0.0 && dt <= 1.7976931348623157e308)) return aicb_fail(AICB_ERR_INVALID, "dt must be finite and >= 0");
    return AICB_OK;
}

// The host form: states and matrices staged in device 0's d_exposure, the results copied back once every part is done.
aicb_status exposure_host(Replicas r, aicb_exposure_state *states, const double (*m)[16], size_t n, double dt,
                          float *out) {
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n && (!states || !m)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_dt(dt));
    if (n == 0) return AICB_OK;
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t st_at = 0, m_at = up(n * sizeof(aicb_exposure_state)), out_at = m_at + up(n * 16 * sizeof(double));
    TRY(c0->d_exposure.ensure(out_at + (out ? n * sizeof(float) : 0)));
    char *base = c0->d_exposure.get<char>();
    cudaStream_t s = c0->stream.get();
    CU(cudaMemcpyAsync(base + st_at, states, n * sizeof(aicb_exposure_state), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(base + m_at, m, n * 16 * sizeof(double), cudaMemcpyHostToDevice, s));
    TRY(issue_exposure(r, dt, reinterpret_cast<aicb_exposure_state *>(base + st_at),
                       reinterpret_cast<const double *>(base + m_at), out ? reinterpret_cast<float *>(base + out_at) : nullptr,
                       n));
    CU(cudaMemcpyAsync(states, base + st_at, n * sizeof(aicb_exposure_state), cudaMemcpyDeviceToHost, s));
    if (out) CU(cudaMemcpyAsync(out, base + out_at, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return AICB_OK;
}

aicb_status exposure_device(Replicas r, aicb_exposure_state *states, const double (*m)[16], size_t n, double dt,
                            float *out, cudaStream_t caller) {
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    TRY(check_dt(dt));
    if (n == 0) return AICB_OK;
    if (!states || !m) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_device_pointer(states, c0->device, false, 4, "states"));
    TRY(check_device_pointer(m, c0->device, false, 8, "eye_to_world"));
    if (out) TRY(check_device_pointer(out, c0->device, false, 4, "exposure_out"));
    TRY(join_caller(r.ctx, r.n, caller));
    TRY(issue_exposure(r, dt, states, &m[0][0], out, n));
    if (r.n > 1) CU(cudaStreamSynchronize(c0->stream.get()));   // a group call returns with its output final
    return release_caller(c0, caller);
}

}  // namespace

extern "C" {

aicb_status aicb_step_exposure(aicb_scene *s, aicb_exposure_state *states, const double (*m)[16], size_t n, double dt,
                               float *out) {
    return on_scene(s, [&](Replicas r) { return exposure_host(r, states, m, n, dt, out); });
}

aicb_status aicb_step_exposure_device(aicb_scene *s, aicb_exposure_state *states, const double (*m)[16], size_t n,
                                      double dt, float *out, void *stream) {
    return on_scene(s, [&](Replicas r) { return exposure_device(r, states, m, n, dt, out, (cudaStream_t)stream); });
}

aicb_status aicb_group_step_exposure(aicb_group_scene *gs, aicb_exposure_state *states, const double (*m)[16],
                                     size_t n, double dt, float *out) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return exposure_host(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, states, m, n, dt, out);
}

aicb_status aicb_group_step_exposure_device(aicb_group_scene *gs, aicb_exposure_state *states, const double (*m)[16],
                                            size_t n, double dt, float *out, void *stream) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return exposure_device(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, states, m, n, dt, out,
                           (cudaStream_t)stream);
}

}  // extern "C"
