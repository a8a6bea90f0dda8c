// Host-side mirror of all_is_cubes_render::camera::Camera as far as the raytracer needs it:
// view transform -> world_to_eye, projection, inverse_projection_view; and the NDC -> world
// ray unprojection.  No GPU code here; exported through the C ABI (include/aicb200.h).
//
// Reference: all-is-cubes-render/src/camera/camera_struct.rs:387-416 (compute_matrices),
// :459-471 (look_at_y_up), :238-257 (project_ndc_into_world); all-is-cubes/src/camera.rs:34-40
// (eye_for_look_at); graphics_options.rs:194-198 (repair).
//
// The matrix/quaternion algebra is euclid 0.22.14 (Transform3D / Rotation3D /
// RigidTransform3D), restated once for the host and the device in ../csrc/camera_math.cuh.
//
// Compiled with -ffp-contract=off / -fmad=false semantics (host code; nvcc passes it to g++).
#include <cmath>
#include <cstring>
#include <limits>

#include "../../include/aicb200.h"
#include "../csrc/camera_math.cuh"

namespace {

using namespace aicb::camera_math;

Quat around_x(double radians) {
    double h = radians / 2.0;
    return Quat{std::sin(h), 0.0, 0.0, std::cos(h)};
}
Quat around_y(double radians) {
    double h = radians / 2.0;
    return Quat{0.0, std::sin(h), 0.0, std::cos(h)};
}

// Camera::compute_matrices (camera_struct.rs:387-416)
bool compute(const Quat &rotation, const double trans[3], double fov_y_degrees, double view_distance,
             double nominal_w, double nominal_h, aicb_camera *out) {
    double fov_cot, aspect, far;
    projection_terms(fov_y_degrees, view_distance, nominal_w, nominal_h, &fov_cot, &aspect, &far);
    return projection_view_inverse(rotation, trans, fov_cot, aspect, far, out->inverse_projection_view);
}

}  // namespace

extern "C" {

aicb_status aicb_camera_from_view(const double q[4], const double translation_[3], double fov_y_degrees,
                                  double view_distance, double nominal_width, double nominal_height,
                                  uint32_t fb_width, uint32_t fb_height, float exposure, aicb_camera *out) {
    if (!q || !translation_ || !out) return AICB_ERR_INVALID;
    std::memset(out, 0, sizeof *out);
    Quat rot{q[0], q[1], q[2], q[3]};
    if (!compute(rot, translation_, fov_y_degrees, view_distance, nominal_width, nominal_height, out))
        return AICB_ERR_INVALID;
    out->fb_width = fb_width;
    out->fb_height = fb_height;
    out->exposure = exposure;
    return AICB_OK;
}

// look_at_y_up (camera_struct.rs:459-471)
aicb_status aicb_camera_look_at(const double eye[3], const double target[3], double fov_y_degrees,
                                double view_distance, double nominal_width, double nominal_height,
                                uint32_t fb_width, uint32_t fb_height, float exposure, aicb_camera *out) {
    if (!eye || !target || !out) return AICB_ERR_INVALID;
    double look[3] = {target[0] - eye[0], target[1] - eye[1], target[2] - eye[2]};
    double yaw = std::atan2(look[0], -look[2]);
    double pitch = std::atan2(-look[1], std::sqrt(look[0] * look[0] + look[2] * look[2]));
    Quat rot = q_then(around_x(-pitch), around_y(-yaw));
    double q[4] = {rot.i, rot.j, rot.k, rot.r};
    return aicb_camera_from_view(q, eye, fov_y_degrees, view_distance, nominal_width, nominal_height, fb_width,
                                 fb_height, exposure, out);
}

// ViewTransform::to_transform (RigidTransform3D::to_transform): rotation.to_transform().then(translation.to_transform())
void aicb_view_transform_matrix(const double q[4], const double translation_[3], double out[16]) {
    view_transform_matrix(Quat{q[0], q[1], q[2], q[3]}, translation_, out);
}

// Body::look_rotation (physics/body.rs:285-292): around_x(-pitch.to_radians()).then(around_y(-yaw.to_radians())),
// f64::to_radians being x * (PI / 180)
void aicb_look_rotation(double yaw_degrees, double pitch_degrees, double out[4]) {
    const Quat q = q_then(around_x(-(pitch_degrees * (M_PI / 180.0))), around_y(-(yaw_degrees * (M_PI / 180.0))));
    out[0] = q.i;
    out[1] = q.j;
    out[2] = q.k;
    out[3] = q.r;
}

// eye_for_look_at (all-is-cubes/src/camera.rs:34-40)
void aicb_eye_for_look_at(const aicb_aab *bounds, const double direction[3], double out_eye[3]) {
    double radius = 0.0;
    for (int a = 0; a < 3; a++) radius = std::fmax(radius, (double)bounds->size[a]);
    double len = std::sqrt(direction[0] * direction[0] + direction[1] * direction[1] + direction[2] * direction[2]);
    for (int a = 0; a < 3; a++) {
        // GridAab::center (grid_aab.rs:391-395): (lower + upper) / 2 in f64
        double upper = (double)((int64_t)bounds->lower[a] + (int64_t)bounds->size[a]);
        double center = ((double)bounds->lower[a] + upper) / 2.0;
        out_eye[a] = center + (direction[a] / len) * radius;
    }
}

// Camera::project_ndc_into_world (camera_struct.rs:238-257)
void aicb_camera_project_ndc(const aicb_camera *cam, double x, double y, double out[6]) {
    const double *m = cam->inverse_projection_view;
    double p[2][3];
    for (int k = 0; k < 2; k++) {
        double z = (double)k;
        double hx = x * m[0] + y * m[4] + z * m[8] + m[12];
        double hy = x * m[1] + y * m[5] + z * m[9] + m[13];
        double hz = x * m[2] + y * m[6] + z * m[10] + m[14];
        double hw = x * m[3] + y * m[7] + z * m[11] + m[15];
        if (hw > 0.0) {
            p[k][0] = hx / hw;
            p[k][1] = hy / hw;
            p[k][2] = hz / hw;
        } else {
            p[k][0] = p[k][1] = p[k][2] = std::numeric_limits<double>::quiet_NaN();
        }
    }
    for (int a = 0; a < 3; a++) {
        out[a] = p[0][a];
        out[3 + a] = p[1][a] - p[0][a];
    }
}
}
