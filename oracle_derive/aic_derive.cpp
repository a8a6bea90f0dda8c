// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// compute_derived (block/eval/derived.rs:80-216) for the fields of EvaluatedBlock that light propagation reads: the
// face colours, colour, emission, opaque faces and visible.  A restatement in the reference's own order: for each face
// in Face::ALL, its face_transform, the data bounds transformed by its inverse, one trace_for_eval per (v, u) of
// iproduct!(y_range, x_range), the VoxSum of the face and the all-faces sum.  apply_transmittance and Rgba::from(ColorBuf)
// are the raytracer oracle's (../oracle/aic_oracle.cpp, compiled into this library a second time), so orc_set_libm
// selects the powf here too.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_derive {
using namespace orc;

// Face::rotation_from_nz (face.rs:395-405): the images of +X, +Y, +Z, for NX NY NZ PX PY PZ
static const int BASIS[6][3][3] = {
    {{0, 1, 0}, {0, 0, 1}, {1, 0, 0}},    // RYZX
    {{0, 0, 1}, {1, 0, 0}, {0, 1, 0}},    // RZXY
    {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}},    // RXYZ
    {{0, -1, 0}, {0, 0, 1}, {-1, 0, 0}},  // RyZx
    {{0, 0, 1}, {-1, 0, 0}, {0, -1, 0}},  // RZxy
    {{1, 0, 0}, {0, -1, 0}, {0, 0, -1}},  // RXyz
};

// Gridgid: p -> R p + t
struct Gridgid {
    int r[3][3];   // r[k]: the image of axis k
    int t[3];
};

// Face::face_transform = rotation_from_nz().to_positive_octant_transform(scale) (rotation.rs:325-354): every basis
// vector that points negative adds scale on its axis.
static Gridgid face_transform(int face, int scale) {
    Gridgid g;
    std::memcpy(g.r, BASIS[face], sizeof g.r);
    for (int i = 0; i < 3; i++) g.t[i] = 0;
    for (int k = 0; k < 3; k++)
        for (int i = 0; i < 3; i++)
            if (g.r[k][i] < 0) g.t[i] += scale;
    return g;
}
static void apply(const Gridgid &g, const int p[3], int out[3]) {
    for (int i = 0; i < 3; i++) out[i] = g.r[0][i] * p[0] + g.r[1][i] * p[1] + g.r[2][i] * p[2] + g.t[i];
}
static void apply_inverse(const Gridgid &g, const int q[3], int out[3]) {   // R is orthonormal: R^-1 = R^T
    for (int k = 0; k < 3; k++)
        out[k] = g.r[k][0] * (q[0] - g.t[0]) + g.r[k][1] * (q[1] - g.t[1]) + g.r[k][2] * (q[2] - g.t[2]);
}
// Gridgid::transform_cube (matrix.rs:171-176): the lesser corner of the images of the cube's corners
static void transform_cube(const Gridgid &g, const int c[3], int out[3]) {
    const int hi[3] = {c[0] + 1, c[1] + 1, c[2] + 1};
    int a[3], b[3];
    apply(g, c, a);
    apply(g, hi, b);
    for (int i = 0; i < 3; i++) out[i] = std::min(a[i], b[i]);
}

struct Voxels {
    int res;
    int lo[3], hi[3];
    const uint16_t *indices;
    const aicb_voxel *palette;
    bool contains(const int c[3]) const {
        for (int i = 0; i < 3; i++)
            if (c[i] < lo[i] || c[i] >= hi[i]) return false;
        return true;
    }
    const aicb_voxel &at(const int c[3]) const {   // Z-major (vol.rs:1013-1018)
        const size_t sy = hi[1] - lo[1], sz = hi[2] - lo[2];
        return palette[indices[((size_t)(c[0] - lo[0]) * sy + (c[1] - lo[1])) * sz + (c[2] - lo[2])]];
    }
};

struct VoxSum {
    float color_sum[3] = {0.0f, 0.0f, 0.0f};
    float alpha_sum = 0.0f;
    float emission_sum[3] = {0.0f, 0.0f, 0.0f};
    size_t count = 0;

    void add(const VoxSum &o) {   // derive_more::AddAssign: componentwise
        for (int i = 0; i < 3; i++) color_sum[i] = color_sum[i] + o.color_sum[i];
        alpha_sum = alpha_sum + o.alpha_sum;
        for (int i = 0; i < 3; i++) emission_sum[i] = emission_sum[i] + o.emission_sum[i];
        count = count + o.count;
    }
    // VoxSum += EvalTrace (derived.rs:267-276)
    void add_trace(const float color[4], const float emission[3]) {
        const float alpha = color[3];
        for (int i = 0; i < 3; i++) color_sum[i] = color_sum[i] + color[i] * alpha;
        alpha_sum = alpha_sum + alpha;
        for (int i = 0; i < 3; i++) emission_sum[i] = emission_sum[i] + emission[i];
        count += 1;
    }
};

// Rgb::try_from(Vector3D) (color.rs:849-858) -> PositiveSign::try_from: false (the reference's expect() panics) for a
// negative or NaN component; -0 becomes +0.
static bool rgb_try_from(float v[3]) {
    for (int i = 0; i < 3; i++) {
        if (v[i] > 0.0f) continue;
        if (v[i] == 0.0f) { v[i] = 0.0f; continue; }
        return false;
    }
    return true;
}

// VoxSum::color (derived.rs:235-254)
static bool voxsum_color(const VoxSum &s, float surface_area, float out[4]) {
    if (!(s.alpha_sum > 0.0f)) {
        out[0] = out[1] = out[2] = out[3] = 0.0f;
        return true;
    }
    float c[3] = {s.color_sum[0] / s.alpha_sum, s.color_sum[1] / s.alpha_sum, s.color_sum[2] / s.alpha_sum};
    if (!rgb_try_from(c)) return false;
    out[0] = c[0];
    out[1] = c[1];
    out[2] = c[2];
    out[3] = zo_clamped(s.alpha_sum / surface_area);
    return true;
}
// VoxSum::emission (derived.rs:256-265)
static bool voxsum_emission(const VoxSum &s, float surface_area, float out[3]) {
    if (s.count == 0) {
        out[0] = out[1] = out[2] = 0.0f;
        return true;
    }
    for (int i = 0; i < 3; i++) out[i] = s.emission_sum[i] / surface_area;
    return rgb_try_from(out);
}

// trace_for_eval (raytracer_components.rs:174-200): color = Rgba::from(ColorBuf), emission
static void trace_for_eval(const Voxels &v, const int origin[3], int axis, int dir, float color[4], float emission[3]) {
    const float thickness = 1.0f / (float)v.res;   // Resolution::recip_f32
    int cube[3] = {origin[0], origin[1], origin[2]};
    ColorBuf buf;
    buf.light[0] = buf.light[1] = buf.light[2] = 0.0f;
    buf.transmittance = 1.0f;
    emission[0] = emission[1] = emission[2] = 0.0f;
    while (v.contains(cube)) {
        const aicb_voxel &vox = v.at(cube);
        float adj[4], coeff;
        apply_transmittance(vox.rgba, thickness, adj, &coeff);
        const float k = ps_clamped(coeff);   // Rgb * f32 (color.rs:912-924)
        for (int i = 0; i < 3; i++) emission[i] = emission[i] + ps_mul(vox.emission[i], k) * buf.transmittance;
        // ColorBuf::from(Rgba) (:150-163), then add_color_internal (:87-92)
        const float surface_t = 1.0f - adj[3];
        for (int i = 0; i < 3; i++) buf.light[i] = buf.light[i] + (adj[i] * adj[3]) * buf.transmittance;
        buf.transmittance = buf.transmittance * surface_t;
        if (buf.transmittance < 1.0f / 256.0f) break;   // ColorBuf::opaque
        cube[axis] += dir;
    }
    colorbuf_to_rgba(buf, color);
}

static void single(const aicb_voxel &v, aicb_block_light &o) {   // derived.rs:84-104
    for (int f = 0; f < 6; f++) std::memcpy(o.face_colors[f], v.rgba, 16);
    std::memcpy(o.color, v.rgba, 16);
    std::memcpy(o.emission, v.emission, 12);
    o.opaque_faces = v.rgba[3] == 1.0f ? 0x3f : 0;   // fully_opaque
    const bool emits = v.emission[0] != 0.0f || v.emission[1] != 0.0f || v.emission[2] != 0.0f;
    o.visible = (v.rgba[3] != 0.0f || emits) ? 1 : 0;
}

// false where the reference panics
static bool compute_derived(const aicb_block_desc &b, aicb_block_light &o) {
    std::memset(&o, 0, sizeof o);
    static const aicb_voxel AIR = {{0, 0, 0, 0}, {0, 0, 0}, 0};
    // Evoxels::single_voxel (voxel_storage.rs:364-383)
    if (!b.indices) {
        single(b.n_palette ? b.palette[0] : AIR, o);
        return true;
    }
    Voxels v;
    v.res = b.resolution;
    for (int i = 0; i < 3; i++) {
        v.lo[i] = b.voxel_bounds.lower[i];
        v.hi[i] = b.voxel_bounds.lower[i] + (int)b.voxel_bounds.size[i];
    }
    v.indices = b.indices;
    v.palette = b.palette;
    if (v.res == 1) {
        const int origin[3] = {0, 0, 0};
        single(v.contains(origin) ? v.at(origin) : AIR, o);
        return true;
    }
    const int res = v.res;
    VoxSum all;
    bool ok = true;
    for (int face = 0; face < 6; face++) {
        const Gridgid g = face_transform(face, res);
        // data_bounds.transform(transform.inverse())
        int a[3], c[3];
        apply_inverse(g, v.lo, a);
        apply_inverse(g, v.hi, c);
        int rl[3], ru[3];
        for (int i = 0; i < 3; i++) {
            rl[i] = std::min(a[i], c[i]);
            ru[i] = std::max(a[i], c[i]);
        }
        const int axis = face % 3, dir = face < 3 ? 1 : -1;   // face.opposite()
        VoxSum face_sum;
        for (int vv = rl[1]; vv < ru[1]; vv++)
            for (int u = rl[0]; u < ru[0]; u++) {
                const int p[3] = {u, vv, rl[2]};
                int cube[3];
                transform_cube(g, p, cube);
                float color[4], emission[3];
                trace_for_eval(v, cube, axis, dir, color, emission);
                face_sum.add_trace(color, emission);
            }
        all.add(face_sum);
        ok &= voxsum_color(face_sum, (float)(res * res), o.face_colors[face]);
    }
    const float surface_area = (float)(6.0 * res * res);
    ok &= voxsum_color(all, surface_area, o.color);
    ok &= voxsum_emission(all, surface_area, o.emission);
    // opaque[face]: full_block_bounds.abut(face, -1) inside the data bounds, and every voxel of it fully opaque
    for (int face = 0; face < 6; face++) {
        const int axis = face % 3;
        int slo[3] = {0, 0, 0}, shi[3] = {res, res, res};
        if (face < 3) shi[axis] = 1; else slo[axis] = res - 1;
        bool inside = true;
        for (int i = 0; i < 3; i++) inside &= v.lo[i] <= slo[i] && shi[i] <= v.hi[i];
        bool opaque = inside;
        for (int x = slo[0]; opaque && x < shi[0]; x++)
            for (int y = slo[1]; opaque && y < shi[1]; y++)
                for (int z = slo[2]; opaque && z < shi[2]; z++) {
                    const int q[3] = {x, y, z};
                    opaque = v.at(q).rgba[3] == 1.0f;
                }
        if (opaque) o.opaque_faces |= (uint8_t)(1u << face);
    }
    // VoxelOpacityMask::visible: some data voxel's opacity_category() is not Invisible
    bool visible = false;
    for (size_t k = 0; k < b.n_indices && !visible; k++) {
        const aicb_voxel &x = b.palette[b.indices[k]];
        visible = x.rgba[3] != 0.0f || x.emission[0] != 0.0f || x.emission[1] != 0.0f || x.emission[2] != 0.0f;
    }
    o.visible = visible ? 1 : 0;
    return ok;
}

}  // namespace orc_derive

extern "C" {
// compute_derived's light fields of n valid blocks.  Returns 0, or 1 where the reference panics, with *bad = the
// block's position (out is then undefined).
int orc_derive_block_light(const aicb_block_desc *descs, size_t n, aicb_block_light *out, size_t *bad) {
    for (size_t i = 0; i < n; i++)
        if (!orc_derive::compute_derived(descs[i], out[i])) {
            if (bad) *bad = i;
            return 1;
        }
    return 0;
}
}
