// camera_math.cuh — the camera algebra of all_is_cubes_render::camera::Camera, for the host (host/camera.cpp, and the
// oracle's copy of it) and the device (eye.cu) alike: euclid 0.22.14's Transform3D, Rotation3D and RigidTransform3D
// as the camera uses them, and the body of Camera::compute_matrices (camera_struct.rs:387-416) once the host has
// computed the field of view's cotangent and the aspect ratio.
//
// euclid is a crates.io dependency that the reference tree does not vendor; it is restated here from its published
// definitions (row-vector convention, m11..m44) and pinned by the reference's own camera tests (camera/tests.rs:78-109
// exact frustum corners, :198-222) and the text.rs ASCII golden images — see tests/test_camera.py.
//
// Every function is a fixed sequence of correctly rounded +, -, * and one division, so the host (-ffp-contract=off)
// and the device (-fmad=false) give the same bits.  Trigonometry (tan, sin, cos) stays with the host: it is not
// correctly rounded in glibc, and the reference calls glibc's.
#pragma once
#include <cmath>

#ifdef __CUDACC__
#define AICB_CAM_FN __host__ __device__ __forceinline__
#else   // a plain C++ compiler (host/camera.cpp as the library's host code, and in the oracle)
#define AICB_CAM_FN inline
#endif

namespace aicb {
namespace camera_math {

struct Mat4 {
    // m[r][c] = m{r+1}{c+1}
    double m[4][4];
};

struct Quat {
    double i, j, k, r;
};

AICB_CAM_FN Mat4 zero4() {
    Mat4 t;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) t.m[i][j] = 0.0;
    return t;
}

// Transform3D::then: row-vector convention, result = self * other
AICB_CAM_FN Mat4 then(const Mat4 &a, const Mat4 &b) {
    Mat4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j] + a.m[i][3] * b.m[3][j];
    return r;
}

// Transform3D::determinant
AICB_CAM_FN double determinant(const Mat4 &t) {
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

// Transform3D::inverse: adjugate scaled by 1/det; false (None) when det == 0
AICB_CAM_FN bool inverse(const Mat4 &t, Mat4 *out) {
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

// Rotation3D::then (Hamilton product, other applied after self)
AICB_CAM_FN Quat q_then(const Quat &s, const Quat &o) {
    return Quat{
        o.i * s.r + o.r * s.i + o.j * s.k - o.k * s.j,
        o.j * s.r + o.r * s.j + o.k * s.i - o.i * s.k,
        o.k * s.r + o.r * s.k + o.i * s.j - o.j * s.i,
        o.r * s.r - o.i * s.i - o.j * s.j - o.k * s.k,
    };
}

AICB_CAM_FN Quat q_inverse(const Quat &q) { return Quat{-q.i, -q.j, -q.k, q.r}; }

// Rotation3D::transform_vector3d
AICB_CAM_FN void q_transform(const Quat &q, const double v[3], double out[3]) {
    // cross = vector_part x v * 2
    const double cx = (q.j * v[2] - q.k * v[1]) * 2.0;
    const double cy = (q.k * v[0] - q.i * v[2]) * 2.0;
    const double cz = (q.i * v[1] - q.j * v[0]) * 2.0;
    out[0] = v[0] + q.r * cx + q.j * cz - q.k * cy;
    out[1] = v[1] + q.r * cy + q.k * cx - q.i * cz;
    out[2] = v[2] + q.r * cz + q.i * cy - q.j * cx;
}

// Rotation3D::to_transform
AICB_CAM_FN Mat4 q_to_transform(const Quat &q) {
    const double i2 = q.i + q.i, j2 = q.j + q.j, k2 = q.k + q.k;
    const double ii = q.i * i2, ij = q.i * j2, ik = q.i * k2;
    const double jj = q.j * j2, jk = q.j * k2, kk = q.k * k2;
    const double ri = q.r * i2, rj = q.r * j2, rk = q.r * k2;
    Mat4 t = zero4();
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

// Translation3D::to_transform
AICB_CAM_FN Mat4 translation(const double v[3]) {
    Mat4 t = zero4();
    t.m[0][0] = t.m[1][1] = t.m[2][2] = t.m[3][3] = 1.0;
    t.m[3][0] = v[0];
    t.m[3][1] = v[1];
    t.m[3][2] = v[2];
    return t;
}

// ViewTransform::to_transform (RigidTransform3D::to_transform): rotation.to_transform().then(translation.to_transform())
AICB_CAM_FN void view_transform_matrix(const Quat &rotation, const double trans[3], double out[16]) {
    const Mat4 t = then(q_to_transform(rotation), translation(trans));
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) out[i * 4 + j] = t.m[i][j];
}

// The host's part of Camera::compute_matrices (camera_struct.rs:387-416), once per camera or batch: the repaired field
// of view's cotangent (graphics_options.rs:194-198, f64::to_radians being x * (PI / 180)), the aspect ratio of the
// nominal viewport size (viewport.rs:80-83, 1 when not finite) and far, the repaired view distance.  Host only: tan is
// glibc's, as the reference's.
inline void projection_terms(double fov_y_degrees, double view_distance, double nominal_w, double nominal_h,
                             double *fov_cot, double *aspect, double *far) {
    const double fov_y = fov_y_degrees < 1.0 ? 1.0 : (fov_y_degrees > 189.0 ? 189.0 : fov_y_degrees);
    *far = view_distance < 1.0 ? 1.0 : (view_distance > 10000.0 ? 10000.0 : view_distance);
    *fov_cot = 1.0 / std::tan((fov_y / 2.0) * (M_PI / 180.0));
    const double a = nominal_w / nominal_h;
    *aspect = std::isfinite(a) ? a : 1.0;
}

// Camera::compute_matrices (camera_struct.rs:387-416) after the host's part (projection_terms).  out: inverse_projection_view, m11..m44; false where the projection-view matrix has no inverse (the reference panics).
AICB_CAM_FN bool projection_view_inverse(const Quat &rotation, const double trans[3], double fov_cot, double aspect,
                                         double far, double out[16]) {
    const double near = 1.0 / 32.0;   // camera_struct.rs:202-205
    Mat4 proj = zero4();
    proj.m[0][0] = fov_cot / aspect;
    proj.m[1][1] = fov_cot;
    proj.m[2][2] = far / (near - far);
    proj.m[2][3] = -1.0;
    proj.m[3][2] = (far * near) / (near - far);

    // RigidTransform3D::inverse: rotation^-1, translation = rotation^-1 * (-translation);
    // to_transform: rotation.to_transform().then(translation.to_transform())
    const Quat rinv = q_inverse(rotation);
    const double neg[3] = {-trans[0], -trans[1], -trans[2]};
    double tinv[3];
    q_transform(rinv, neg, tinv);
    const Mat4 world_to_eye = then(q_to_transform(rinv), translation(tinv));

    Mat4 inv;
    if (!inverse(then(world_to_eye, proj), &inv)) return false;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) out[i * 4 + j] = inv.m[i][j];
    return true;
}

}  // namespace camera_math
}  // namespace aicb
