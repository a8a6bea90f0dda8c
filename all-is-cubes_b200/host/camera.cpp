// Host-side mirror of all_is_cubes_render::camera::Camera as far as the raytracer needs it:
// view transform -> world_to_eye, projection, inverse_projection_view; and the NDC -> world
// ray unprojection.  No GPU code here; exported through the C ABI (include/aicb200.h).
//
// Reference: all-is-cubes-render/src/camera/camera_struct.rs:387-416 (compute_matrices),
// :459-471 (look_at_y_up), :238-257 (project_ndc_into_world); all-is-cubes/src/camera.rs:34-40
// (eye_for_look_at); graphics_options.rs:194-198 (repair).
//
// The matrix/quaternion algebra is euclid 0.22.14 (Transform3D / Rotation3D /
// RigidTransform3D), which is a crates.io dependency NOT vendored in the reference tree; it is
// restated here from its published definitions (row-vector convention, m11..m44) and pinned by
// the reference's own camera tests (camera/tests.rs:78-109 exact frustum corners, :198-222) and
// the text.rs ASCII golden images — see tests/test_camera.py.
//
// Compiled with -ffp-contract=off / -fmad=false semantics (host code; nvcc passes it to g++).
#include <cmath>
#include <cstring>
#include <limits>

#include "../../include/aicb200.h"

namespace {

struct Mat4 {
    // m[r][c] = m{r+1}{c+1}
    double m[4][4];
};

// Transform3D::then: row-vector convention, result = self * other
Mat4 then(const Mat4 &a, const Mat4 &b) {
    Mat4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j] + a.m[i][3] * b.m[3][j];
    return r;
}

// Transform3D::determinant
double determinant(const Mat4 &t) {
    const double m11 = t.m[0][0], m12 = t.m[0][1], m13 = t.m[0][2], m14 = t.m[0][3];
    const double m21 = t.m[1][0], m22 = t.m[1][1], m23 = t.m[1][2], m24 = t.m[1][3];
    const double m31 = t.m[2][0], m32 = t.m[2][1], m33 = t.m[2][2], m34 = t.m[2][3];
    const double m41 = t.m[3][0], m42 = t.m[3][1], m43 = t.m[3][2], m44 = t.m[3][3];
    return m14 * m23 * m32 * m41 - m13 * m24 * m32 * m41 - m14 * m22 * m33 * m41 + m12 * m24 * m33 * m41 +
           m13 * m22 * m34 * m41 - m12 * m23 * m34 * m41 - m14 * m23 * m31 * m42 + m13 * m24 * m31 * m42 +
           m14 * m21 * m33 * m42 - m11 * m24 * m33 * m42 - m13 * m21 * m34 * m42 + m11 * m23 * m34 * m42 +
           m14 * m22 * m31 * m43 - m12 * m24 * m31 * m43 - m14 * m21 * m32 * m43 + m11 * m24 * m32 * m43 +
           m12 * m21 * m34 * m43 - m11 * m22 * m34 * m43 - m13 * m22 * m31 * m44 + m12 * m23 * m31 * m44 +
           m13 * m21 * m32 * m44 - m11 * m23 * m32 * m44 - m12 * m21 * m33 * m44 + m11 * m22 * m33 * m44;
}

// Transform3D::inverse: adjugate scaled by 1/det
bool inverse(const Mat4 &t, Mat4 *out) {
    const double det = determinant(t);
    if (det == 0.0) return false;
    const double m11 = t.m[0][0], m12 = t.m[0][1], m13 = t.m[0][2], m14 = t.m[0][3];
    const double m21 = t.m[1][0], m22 = t.m[1][1], m23 = t.m[1][2], m24 = t.m[1][3];
    const double m31 = t.m[2][0], m32 = t.m[2][1], m33 = t.m[2][2], m34 = t.m[2][3];
    const double m41 = t.m[3][0], m42 = t.m[3][1], m43 = t.m[3][2], m44 = t.m[3][3];
    Mat4 a;
    a.m[0][0] = m23 * m34 * m42 - m24 * m33 * m42 + m24 * m32 * m43 - m22 * m34 * m43 - m23 * m32 * m44 + m22 * m33 * m44;
    a.m[0][1] = m14 * m33 * m42 - m13 * m34 * m42 - m14 * m32 * m43 + m12 * m34 * m43 + m13 * m32 * m44 - m12 * m33 * m44;
    a.m[0][2] = m13 * m24 * m42 - m14 * m23 * m42 + m14 * m22 * m43 - m12 * m24 * m43 - m13 * m22 * m44 + m12 * m23 * m44;
    a.m[0][3] = m14 * m23 * m32 - m13 * m24 * m32 - m14 * m22 * m33 + m12 * m24 * m33 + m13 * m22 * m34 - m12 * m23 * m34;
    a.m[1][0] = m24 * m33 * m41 - m23 * m34 * m41 - m24 * m31 * m43 + m21 * m34 * m43 + m23 * m31 * m44 - m21 * m33 * m44;
    a.m[1][1] = m13 * m34 * m41 - m14 * m33 * m41 + m14 * m31 * m43 - m11 * m34 * m43 - m13 * m31 * m44 + m11 * m33 * m44;
    a.m[1][2] = m14 * m23 * m41 - m13 * m24 * m41 - m14 * m21 * m43 + m11 * m24 * m43 + m13 * m21 * m44 - m11 * m23 * m44;
    a.m[1][3] = m13 * m24 * m31 - m14 * m23 * m31 + m14 * m21 * m33 - m11 * m24 * m33 - m13 * m21 * m34 + m11 * m23 * m34;
    a.m[2][0] = m22 * m34 * m41 - m24 * m32 * m41 + m24 * m31 * m42 - m21 * m34 * m42 - m22 * m31 * m44 + m21 * m32 * m44;
    a.m[2][1] = m14 * m32 * m41 - m12 * m34 * m41 - m14 * m31 * m42 + m11 * m34 * m42 + m12 * m31 * m44 - m11 * m32 * m44;
    a.m[2][2] = m12 * m24 * m41 - m14 * m22 * m41 + m14 * m21 * m42 - m11 * m24 * m42 - m12 * m21 * m44 + m11 * m22 * m44;
    a.m[2][3] = m14 * m22 * m31 - m12 * m24 * m31 - m14 * m21 * m32 + m11 * m24 * m32 + m12 * m21 * m34 - m11 * m22 * m34;
    a.m[3][0] = m23 * m32 * m41 - m22 * m33 * m41 - m23 * m31 * m42 + m21 * m33 * m42 + m22 * m31 * m43 - m21 * m32 * m43;
    a.m[3][1] = m12 * m33 * m41 - m13 * m32 * m41 + m13 * m31 * m42 - m11 * m33 * m42 - m12 * m31 * m43 + m11 * m32 * m43;
    a.m[3][2] = m13 * m22 * m41 - m12 * m23 * m41 - m13 * m21 * m42 + m11 * m23 * m42 + m12 * m21 * m43 - m11 * m22 * m43;
    a.m[3][3] = m12 * m23 * m31 - m13 * m22 * m31 + m13 * m21 * m32 - m11 * m23 * m32 - m12 * m21 * m33 + m11 * m22 * m33;
    const double s = 1.0 / det;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) out->m[i][j] = a.m[i][j] * s;
    return true;
}

struct Quat {
    double i, j, k, r;
};

// Rotation3D::then (Hamilton product, other applied after self)
Quat q_then(const Quat &s, const Quat &o) {
    return Quat{
        o.i * s.r + o.r * s.i + o.j * s.k - o.k * s.j,
        o.j * s.r + o.r * s.j + o.k * s.i - o.i * s.k,
        o.k * s.r + o.r * s.k + o.i * s.j - o.j * s.i,
        o.r * s.r - o.i * s.i - o.j * s.j - o.k * s.k,
    };
}
Quat q_inverse(const Quat &q) { return Quat{-q.i, -q.j, -q.k, q.r}; }
Quat around_x(double radians) {
    double h = radians / 2.0;
    return Quat{std::sin(h), 0.0, 0.0, std::cos(h)};
}
Quat around_y(double radians) {
    double h = radians / 2.0;
    return Quat{0.0, std::sin(h), 0.0, std::cos(h)};
}
// Rotation3D::transform_vector3d
void q_transform(const Quat &q, const double v[3], double out[3]) {
    // cross = vector_part x v * 2
    double cx = (q.j * v[2] - q.k * v[1]) * 2.0;
    double cy = (q.k * v[0] - q.i * v[2]) * 2.0;
    double cz = (q.i * v[1] - q.j * v[0]) * 2.0;
    out[0] = v[0] + q.r * cx + q.j * cz - q.k * cy;
    out[1] = v[1] + q.r * cy + q.k * cx - q.i * cz;
    out[2] = v[2] + q.r * cz + q.i * cy - q.j * cx;
}
// Rotation3D::to_transform
Mat4 q_to_transform(const Quat &q) {
    double i2 = q.i + q.i, j2 = q.j + q.j, k2 = q.k + q.k;
    double ii = q.i * i2, ij = q.i * j2, ik = q.i * k2;
    double jj = q.j * j2, jk = q.j * k2, kk = q.k * k2;
    double ri = q.r * i2, rj = q.r * j2, rk = q.r * k2;
    Mat4 t;
    std::memset(&t, 0, sizeof t);
    t.m[0][0] = 1.0 - (jj + kk);
    t.m[0][1] = ij + rk;
    t.m[0][2] = ik - rj;
    t.m[1][0] = ij - rk;
    t.m[1][1] = 1.0 - (ii + kk);
    t.m[1][2] = jk + ri;
    t.m[2][0] = ik + rj;
    t.m[2][1] = jk - ri;
    t.m[2][2] = 1.0 - (ii + jj);
    t.m[3][3] = 1.0;
    return t;
}
Mat4 translation(const double v[3]) {
    Mat4 t;
    std::memset(&t, 0, sizeof t);
    t.m[0][0] = t.m[1][1] = t.m[2][2] = t.m[3][3] = 1.0;
    t.m[3][0] = v[0];
    t.m[3][1] = v[1];
    t.m[3][2] = v[2];
    return t;
}

double repair(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Camera::compute_matrices (camera_struct.rs:387-416)
bool compute(const Quat &rotation, const double trans[3], double fov_y_degrees, double view_distance,
             double nominal_w, double nominal_h, aicb_camera *out) {
    double fov_y = repair(fov_y_degrees, 1.0, 189.0);       // graphics_options.rs:195
    double far = repair(view_distance, 1.0, 10000.0);       // graphics_options.rs:196
    double fov_cot = 1.0 / std::tan((fov_y / 2.0) * (M_PI / 180.0));  // f64::to_radians = x * (PI/180)
    double aspect = nominal_w / nominal_h;                  // viewport.rs:80-83
    if (!std::isfinite(aspect)) aspect = 1.0;
    double near = 1.0 / 32.0;                               // camera_struct.rs:202-205

    Mat4 proj;
    std::memset(&proj, 0, sizeof proj);
    proj.m[0][0] = fov_cot / aspect;
    proj.m[1][1] = fov_cot;
    proj.m[2][2] = far / (near - far);
    proj.m[2][3] = -1.0;
    proj.m[3][2] = (far * near) / (near - far);

    // RigidTransform3D::inverse: rotation^-1, translation = rotation^-1 * (-translation);
    // to_transform: rotation.to_transform().then(translation.to_transform())
    Quat rinv = q_inverse(rotation);
    double neg[3] = {-trans[0], -trans[1], -trans[2]};
    double tinv[3];
    q_transform(rinv, neg, tinv);
    Mat4 world_to_eye = then(q_to_transform(rinv), translation(tinv));

    Mat4 inv;
    if (!inverse(then(world_to_eye, proj), &inv)) return false;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) out->inverse_projection_view[i * 4 + j] = inv.m[i][j];
    return true;
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
    const Mat4 t = then(q_to_transform(Quat{q[0], q[1], q[2], q[3]}), translation(translation_));
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) out[i * 4 + j] = t.m[i][j];
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
