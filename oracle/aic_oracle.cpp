// ORACLE — TEST INFRASTRUCTURE ONLY.  See aic_oracle.hpp for the rules.
//
// CPU restatement of all-is-cubes' raytracer hot path.  Citations are file:line in the
// reference checkout (commit 7ab02ee1).  Arithmetic follows the Rust source operation by
// operation: f64 for ray geometry, f32 for colour, no FMA contraction, Rust semantics for
// min/max/clamp/round/saturating casts (SURVEY.md Appendix B).
#include "aic_oracle.hpp"
#include "../all-is-cubes_b200/csrc/exact_math.cuh"   // LIBM_CR: the correctly rounded powf / expf

#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

namespace orc {

static const double INF = std::numeric_limits<double>::infinity();

// ---------------------------------------------------------------------------------------------
// Rust float helpers
// ---------------------------------------------------------------------------------------------
static inline double rmax(double a, double b) { return std::fmax(a, b); }  // f64::max ignores NaN
static inline float rmaxf(float a, float b) { return std::fmaxf(a, b); }
static inline double rclamp(double v, double lo, double hi) {  // f64::clamp: NaN passes through
    if (v < lo) return lo;
    if (v > hi) return hi;
    return v;
}
static inline float rclampf(float v, float lo, float hi) {
    if (v < lo) return lo;
    if (v > hi) return hi;
    return v;
}
// f64::rem_euclid(1.0): r = x % 1.0; if r < 0 { r + 1.0 }
static inline double rem_euclid1(double x) {
    double r = std::fmod(x, 1.0);
    return (r < 0.0) ? r + 1.0 : r;
}
// PositiveSign::<f32>::new_clamped (restricted_number.rs:240-248); NaN is unreachable in the
// reference (it panics) — we map it to 0.
static inline float ps_clamped(float v) { return (v > 0.0f) ? v : 0.0f; }
// ZeroOne::<f32>::new_clamped (restricted_number.rs:315-326)
static inline float zo_clamped(float v) {
    if (v > 0.0f && v <= 1.0f) return v;
    if (v <= 0.0f) return 0.0f;
    return 1.0f;  // v >= 1 (NaN unreachable)
}
// PositiveSign * PositiveSign (restricted_number.rs:753-768): 0 * inf = 0
static inline float ps_mul(float a, float b) {
    float v = a * b;
    return (v != v) ? 0.0f : v;
}
// `x as u8` from f32: saturating, NaN -> 0
static inline uint8_t sat_u8(float v) {
    if (!(v > 0.0f)) return 0;
    if (v >= 255.0f) return 255;
    return (uint8_t)v;
}

// ---------------------------------------------------------------------------------------------
// raycast.rs
// ---------------------------------------------------------------------------------------------

// raycast.rs:782-788
int32_t signum_101(double x) {
    if (x == 0.0 || std::isnan(x)) return 0;  // NaN.signum() = NaN, `as i32` = 0
    return std::signbit(x) ? -1 : 1;          // f64::signum is +-1 even for +-0
}

// raycast.rs:797-819
double scale_to_integer_step(double s, double ds) {
    if (ds == 0.0 && !std::isnan(s)) {
        return INF;
    } else if (ds < 0.0) {
        s = -s;
        ds = -ds;
    }
    s = rem_euclid1(s);
    return (1.0 - s) / ds;
}

// math/cube.rs:97-119
bool cube_containing(const double p[3], int32_t out[3]) {
    const double MIN_INCLUSIVE = (double)I32_MIN;
    const double MAX_EXCLUSIVE = (double)I32_MAX + 1.0;
    if ((MIN_INCLUSIVE <= p[0]) & (MIN_INCLUSIVE <= p[1]) & (MIN_INCLUSIVE <= p[2]) &
        (p[0] < MAX_EXCLUSIVE) & (p[1] < MAX_EXCLUSIVE) & (p[2] < MAX_EXCLUSIVE)) {
        out[0] = (int32_t)std::floor(p[0]);
        out[1] = (int32_t)std::floor(p[1]);
        out[2] = (int32_t)std::floor(p[2]);
        return true;
    }
    return false;
}

static inline bool aab_contains_cube(const Aab &b, const int32_t c[3]) {
    for (int a = 0; a < 3; a++)
        if (c[a] < b.lo[a] || c[a] >= b.hi[a]) return false;
    return true;
}

// GridAab::intersection_cubes (grid_aab.rs:506-515) .unwrap_or(ORIGIN_EMPTY)
static Aab intersect_or_empty(const Aab &a, const Aab &b) {
    Aab r;
    for (int i = 0; i < 3; i++) {
        r.lo[i] = a.lo[i] > b.lo[i] ? a.lo[i] : b.lo[i];
        r.hi[i] = a.hi[i] < b.hi[i] ? a.hi[i] : b.hi[i];
    }
    for (int i = 0; i < 3; i++)
        if (r.hi[i] <= r.lo[i]) return Aab{{0, 0, 0}, {0, 0, 0}};
    return r;
}

// State::EMPTY with Parameters::ZERO (raycast.rs:502-509, 735-746)
void Raycaster::set_empty() {
    for (int a = 0; a < 3; a++) {
        origin[a] = 0.0;
        dir[a] = 0.0;
        step[a] = 0;
        t_delta[a] = INF;
        cube[a] = 0;
        t_max[a] = 0.0;
    }
    last_face = AICB_FACE_WITHIN;
    last_t_distance = 0.0;
    bounds = Aab{{0, 0, 0}, {0, 0, 0}};
}

// Raycaster::new -> Parameters::new (raycast.rs:749-771) -> State::from_parameters (513-545)
void Raycaster::init(const double o[3], const double d_in[3]) {
    double d[3] = {d_in[0], d_in[1], d_in[2]};
    // raycast.rs:760-764: every |d| must compare Less than 1e100, else direction := 0
    bool all_small = true;
    for (int a = 0; a < 3; a++)
        if (!(std::fabs(d[a]) < 1e100)) all_small = false;
    if (!all_small) d[0] = d[1] = d[2] = 0.0;

    for (int a = 0; a < 3; a++) {
        origin[a] = o[a];
        dir[a] = d[a];
        step[a] = signum_101(d[a]);
        t_delta[a] = 1.0 / std::fabs(d[a]);
    }
    first_last = FL_BEGINNING;
    include_exit = true;

    int32_t c[3];
    Aab mb = maximum_bounds();
    if (!cube_containing(origin, c) || !aab_contains_cube(mb, c)) {
        set_empty();
        return;
    }
    for (int a = 0; a < 3; a++) {
        cube[a] = c[a];
        t_max[a] = scale_to_integer_step(origin[a], dir[a]);
    }
    last_face = AICB_FACE_WITHIN;
    last_t_distance = 0.0;
    bounds = mb;
}

// raycast.rs:223-230
void Raycaster::within(const Aab &b, bool inc_exit) {
    bounds = intersect_or_empty(bounds, b);
    first_last = FL_BEGINNING;
    include_exit = inc_exit;
    fast_forward();
}

// raycast.rs:548-557
void Raycaster::current(RaycastStep *out) const {
    for (int a = 0; a < 3; a++) {
        out->cube[a] = cube[a];
        out->t_max[a] = t_max[a];
    }
    out->face = last_face;
    out->t_distance = last_t_distance;
}

// raycast.rs:563-570
bool Raycaster::valid_for_stepping() const {
    bool nonzero = step[0] != 0 || step[1] != 0 || step[2] != 0;
    bool any_nan = std::isnan(t_max[0]) || std::isnan(t_max[1]) || std::isnan(t_max[2]);
    bool any_finite = std::isfinite(t_max[0]) || std::isfinite(t_max[1]) || std::isfinite(t_max[2]);
    return nonzero && !any_nan && any_finite;
}

// raycast.rs:577-626
bool Raycaster::do_step() {
    int axis;
    if (t_max[0] < t_max[1]) {
        axis = (t_max[0] < t_max[2]) ? 0 : 2;
    } else {
        axis = (t_max[1] < t_max[2]) ? 1 : 2;
    }
    last_t_distance = t_max[axis];
    // checked_add
    int64_t nc = (int64_t)cube[axis] + (int64_t)step[axis];
    if (nc < (int64_t)I32_MIN || nc > (int64_t)I32_MAX) return false;
    cube[axis] = (int32_t)nc;
    t_max[axis] += t_delta[axis];
    // FACE_TABLE[axis][step > 0]: {PX,NX},{PY,NY},{PZ,NZ}
    last_face = (step[axis] > 0) ? (AICB_FACE_NX + axis) : (AICB_FACE_PX + axis);
    return true;
}

// ray_plane_intersection (raycast.rs:821-832), euclid dot = x*x' + y*y' + z*z'
static double ray_plane_intersection(const double o[3], const double d[3], const int32_t plane_origin[3],
                                     const int32_t plane_normal[3]) {
    double po[3], pn[3], rel[3];
    for (int a = 0; a < 3; a++) {
        po[a] = (double)plane_origin[a];
        pn[a] = (double)plane_normal[a];
        rel[a] = po[a] - o[a];
    }
    double num = rel[0] * pn[0] + rel[1] * pn[1] + rel[2] * pn[2];
    double den = d[0] * pn[0] + d[1] * pn[1] + d[2] * pn[2];
    return num / den;
}

// raycast.rs:632-704
void Raycaster::fast_forward() {
    int32_t plane_origin[3];
    for (int a = 0; a < 3; a++) plane_origin[a] = (step[a] < 0) ? bounds.hi[a] : bounds.lo[a];

    double max_t = 0.0;
    for (int a = 0; a < 3; a++) {
        int32_t direction = step[a];
        if (direction == 0) continue;
        int32_t normal[3] = {0, 0, 0};
        normal[a] = direction;
        double it = ray_plane_intersection(origin, dir, plane_origin, normal);
        max_t = rmax(max_t, it);
    }

    if (max_t > last_t_distance) {
        double len = std::sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        double t_start = max_t - 0.5 / len;
        if (!std::isfinite(t_start)) t_start = max_t;
        double ff[3];
        for (int a = 0; a < 3; a++) ff[a] = origin[a] + dir[a] * t_start;  // Ray::advance, ray.rs:107-112
        int32_t c[3];
        if (!cube_containing(ff, c)) {
            set_empty();
            return;
        }
        for (int a = 0; a < 3; a++) {
            origin[a] = ff[a];
            cube[a] = c[a];
            t_max[a] = scale_to_integer_step(ff[a], dir[a]) + t_start;
        }
        last_t_distance = t_start;
        // last_face, bounds, step, t_delta preserved
    }
}

// raycast.rs:711-728
void Raycaster::oob(bool *enter, bool *exit_) const {
    bool e = false, x = false;
    for (int a = 0; a < 3; a++) {
        bool low = cube[a] < bounds.lo[a];
        bool high = cube[a] >= bounds.hi[a];
        bool en, ex;
        if (step[a] == 0) {
            en = low | high;
            ex = low | high;
        } else if (step[a] < 0) {
            en = high;
            ex = low;
        } else {
            en = low;
            ex = high;
        }
        e |= en;
        x |= ex;
    }
    *enter = e;
    *exit_ = x;
}

// raycast.rs:239-284
bool Raycaster::next(RaycastStep *out) {
    for (;;) {
        bool enter, exit_;
        oob(&enter, &exit_);
        if ((first_last == FL_IN_BOUNDS || first_last == FL_BEGINNING) && !enter && !exit_) {
            current(out);
            if (!valid_for_stepping()) {
                first_last = FL_ENDED;
                return last_face == AICB_FACE_WITHIN;
            }
            (void)do_step();
            first_last = FL_IN_BOUNDS;
            return true;
        } else if (first_last == FL_BEGINNING && enter && !exit_) {
            if (!valid_for_stepping()) {
                first_last = FL_ENDED;
                return false;
            }
            if (!do_step()) return false;
        } else if (first_last == FL_IN_BOUNDS && !enter && exit_) {
            first_last = FL_ENDED;
            if (include_exit) {
                current(out);
                return true;
            }
            return false;
        } else {
            // (Ended, _, _) | (_, _, true); (InBounds, true, false) is unreachable
            return false;
        }
    }
}

// raycast.rs:409-439
void intersection_point(const RaycastStep &s, const double o[3], const double d[3], double out[3]) {
    if (s.face == AICB_FACE_WITHIN) {
        out[0] = o[0];
        out[1] = o[1];
        out[2] = o[2];
        return;
    }
    int face_axis = (s.face - 1) % 3;
    for (int a = 0; a < 3; a++) {
        double p = (double)s.cube[a];
        int32_t sd = signum_101(d[a]);
        if (a == face_axis) {
            if (sd < 0) p += 1.0;
        } else if (sd == 0) {
            p = o[a];
        } else {
            double off = (s.t_max[a] - s.t_distance) * d[a];
            p += (sd > 0) ? (1.0 - rclamp(off, 0.0, 1.0)) : rclamp(-off, 0.0, 1.0);
        }
        out[a] = p;
    }
}

// ---------------------------------------------------------------------------------------------
// PackedLight (space/light/data.rs)
// ---------------------------------------------------------------------------------------------
struct Lut {
    float v[256];
    Lut() {
        // Defined by scalar_out_arithmetic (data.rs:232-243): exp2f((v - 144) / 10), 0 -> 0.
        // tests/test_oracle_color.py checks all 256 entries against the reference's table
        // (data.rs:301-354) via tests/golden/packed_light_lut.json.
        v[0] = 0.0f;
        for (int i = 1; i < 256; i++) {
            float e = ((float)i - 144.0f) / 10.0f;
            v[i] = (float)std::exp2((double)e);
        }
    }
};
static const Lut LUT;

enum { ST_UNINIT = 0, ST_NO_RAYS = 1, ST_OPAQUE = 128, ST_VISIBLE = 255 };
struct PackedLight {
    uint8_t r, g, b, status;
};
static const PackedLight PL_ONE = {144, 144, 144, ST_VISIBLE};
static const PackedLight PL_NO_RAYS = {0, 0, 0, ST_NO_RAYS};
static const PackedLight PL_UNINIT = {0, 0, 0, ST_UNINIT};

// data.rs:213-217
static uint8_t scalar_in(float value) {
    float x = std::round(std::log2(value) * 10.0f + 144.0f);
    return sat_u8(x);
}
static PackedLight pl_some(const float rgb[3]) {
    return PackedLight{scalar_in(rgb[0]), scalar_in(rgb[1]), scalar_in(rgb[2]), ST_VISIBLE};
}
static inline bool pl_valid(PackedLight p) { return p.status == ST_VISIBLE; }  // data.rs:127-135
// data.rs:145-158
static inline void pl_value_ao(PackedLight p, float out[4]) {
    out[0] = LUT.v[p.r];
    out[1] = LUT.v[p.g];
    out[2] = LUT.v[p.b];
    out[3] = (p.status == ST_VISIBLE) ? 1.0f : (p.status == ST_OPAQUE) ? 0.25f : 0.0f;
}

// ---------------------------------------------------------------------------------------------
// Scene snapshot == SpaceRaytracer fields (sr.rs:51-60)
// ---------------------------------------------------------------------------------------------
struct Block {
    bool invisible;  // AIR (always_invisible) — checked on the cube, sr.rs:547
    bool single;     // Evoxels::single_voxel() is Some
    aicb_voxel voxel;  // the single voxel
    int resolution;
    Aab vb;
    int32_t vsize[3];
    std::vector<uint16_t> indices;
    std::vector<aicb_voxel> palette;
};

}  // namespace orc

struct orc_scene {
    orc::Aab bounds;
    int32_t size[3];
    std::vector<uint16_t> ids;
    std::vector<orc::PackedLight> light;
    bool has_light;
    std::vector<orc::Block> blocks;
    aicb_sky sky;
    orc::PackedLight sky_faces[6];  // BlockSky.faces NX..PZ (sky.rs:54-82)
    orc::PackedLight sky_mean;
};

namespace orc {

static const aicb_voxel VOXEL_AIR = {{0, 0, 0, 0}, {0, 0, 0}, 0};

// Sky::sample (sky.rs:32-41)
static void sky_sample(const aicb_sky &sky, const double d[3], float out[3]) {
    int idx = 0;
    if (sky.kind != 0) idx = ((d[0] >= 0.0) << 2) + ((d[1] >= 0.0) << 1) + (d[2] >= 0.0);
    out[0] = sky.colors[idx][0];
    out[1] = sky.colors[idx][1];
    out[2] = sky.colors[idx][2];
}

// GridRotation basis for Face::rotation_from_nz (face.rs:395-405): returns the images of
// (1,0,0) and (0,1,0) and (0,0,1).
static void rotation_from_nz(int face, int fx[3], int fy[3], int fz[3]) {
    static const int tbl[7][3][3] = {
        /* Within: IDENTITY */ {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}},
        /* NX: RYZX */ {{0, 1, 0}, {0, 0, 1}, {1, 0, 0}},
        /* NY: RZXY */ {{0, 0, 1}, {1, 0, 0}, {0, 1, 0}},
        /* NZ: RXYZ */ {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}},
        /* PX: RyZx */ {{0, -1, 0}, {0, 0, 1}, {-1, 0, 0}},
        /* PY: RZxy */ {{0, 0, 1}, {-1, 0, 0}, {0, -1, 0}},
        /* PZ: RXyz */ {{1, 0, 0}, {0, -1, 0}, {0, 0, -1}},
    };
    for (int i = 0; i < 3; i++) {
        fx[i] = tbl[face][0][i];
        fy[i] = tbl[face][1][i];
        fz[i] = tbl[face][2][i];
    }
}

// Sky::for_blocks (sky.rs:54-82), Sky::mean (sky.rs:45-50)
static void build_block_sky(orc_scene *s) {
    const aicb_sky &sky = s->sky;
    if (sky.kind == 0) {
        PackedLight p = pl_some(sky.colors[0]);
        for (int f = 0; f < 6; f++) s->sky_faces[f] = p;
        s->sky_mean = p;
        return;
    }
    static const int pts[4][3] = {{-1, -1, -1}, {-1, 1, -1}, {1, -1, -1}, {1, 1, -1}};
    for (int f = 0; f < 6; f++) {
        int fx[3], fy[3], fz[3];
        rotation_from_nz(f + 1, fx, fy, fz);
        float sum[3] = {0, 0, 0};  // Rgb::sum folds from zero (color.rs:937-945)
        for (int k = 0; k < 4; k++) {
            double d[3];
            for (int i = 0; i < 3; i++) d[i] = (double)(pts[k][0] * fx[i] + pts[k][1] * fy[i] + pts[k][2] * fz[i]);
            float c[3];
            sky_sample(sky, d, c);
            for (int i = 0; i < 3; i++) sum[i] = sum[i] + c[i];
        }
        float q[3];
        for (int i = 0; i < 3; i++) q[i] = ps_mul(sum[i], ps_clamped(0.25f));
        s->sky_faces[f] = pl_some(q);
    }
    float sum[3] = {0, 0, 0};
    for (int k = 0; k < 8; k++)
        for (int i = 0; i < 3; i++) sum[i] = sum[i] + sky.colors[k][i];
    float q[3];
    for (int i = 0; i < 3; i++) q[i] = ps_mul(sum[i], ps_clamped(1.0f / 8.0f));
    s->sky_mean = pl_some(q);
}

// BlockSky::light_outside (sky.rs:113-147)
static PackedLight light_outside(const orc_scene &s, const int32_t c[3]) {
    // lower[a]: cmp(bounds.lo-1, c); upper[a]: cmp(c, bounds.hi). -1 Less, 0 Equal, 1 Greater
    int lower[3], upper[3];
    for (int a = 0; a < 3; a++) {
        if (s.bounds.lo[a] == I32_MIN) {
            lower[a] = -1;
        } else {
            int32_t beyond = s.bounds.lo[a] - 1;
            lower[a] = (beyond < c[a]) ? -1 : (beyond == c[a]) ? 0 : 1;
        }
        upper[a] = (c[a] < s.bounds.hi[a]) ? -1 : (c[a] == s.bounds.hi[a]) ? 0 : 1;
    }
    int n_equal = 0, n_less = 0, which = -1;
    for (int a = 0; a < 3; a++) {
        if (lower[a] == 0) { n_equal++; which = a; } else if (lower[a] < 0) n_less++;
        if (upper[a] == 0) { n_equal++; which = 3 + a; } else if (upper[a] < 0) n_less++;
    }
    if (n_less == 6) return PL_UNINIT;
    if (n_equal == 1 && n_less == 5) return s.sky_faces[which];  // nx,ny,nz,px,py,pz
    return PL_NO_RAYS;
}

// Vol::get via index_into_aab_zmaj (vol.rs:988-1019)
static inline bool vol_index(const Aab &b, const int32_t size[3], const int32_t c[3], size_t *idx) {
    uint32_t dx = (uint32_t)c[0] - (uint32_t)b.lo[0];
    uint32_t dy = (uint32_t)c[1] - (uint32_t)b.lo[1];
    uint32_t dz = (uint32_t)c[2] - (uint32_t)b.lo[2];
    if ((dx >= (uint32_t)size[0]) | (dy >= (uint32_t)size[1]) | (dz >= (uint32_t)size[2])) return false;
    *idx = ((size_t)dx * (size_t)size[1] + (size_t)dy) * (size_t)size[2] + (size_t)dz;
    return true;
}

// SpaceRaytracer::get_packed_light (sr.rs:241-246)
static PackedLight get_packed_light(const orc_scene &s, const int32_t c[3]) {
    size_t idx;
    if (vol_index(s.bounds, s.size, c, &idx)) return s.has_light ? s.light[idx] : PL_ONE;
    return light_outside(s, c);
}

// ---------------------------------------------------------------------------------------------
// Surface / TraceStep / SurfaceIter / DepthIter (surface.rs)
// ---------------------------------------------------------------------------------------------
struct Surface {
    int block_index;
    float color[4];
    float emission[3];
    int32_t cube[3];
    int resolution;
    int32_t voxel[3];
    double t_distance;
    double ip[3];
    int normal;
};
enum { TS_ENTER_SURFACE = 0, TS_INVISIBLE = 1, TS_ENTER_BLOCK = 2 };
struct TraceStep {
    int kind;
    double t_distance;
    int block_index;
    Surface surface;
};

static inline bool voxel_invisible(const aicb_voxel &v) {
    // color.fully_transparent() && emission == Rgb::ZERO (surface.rs:315, 395)
    return v.rgba[3] == 0.0f && v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f;
}

struct SurfaceIter {
    const orc_scene *sc;
    double origin[3], dir[3];
    Raycaster block_rc;
    // VoxelSurfaceIter (surface.rs:361-372)
    bool have_inner;
    Raycaster voxel_rc;
    double sub_origin[3];
    const Block *inner_block;
    int inner_block_index;
    int32_t block_cube[3];

    // SurfaceIter::new (surface.rs:265-273)
    void init(const orc_scene *scene, const double o[3], const double d[3]) {
        sc = scene;
        for (int a = 0; a < 3; a++) {
            origin[a] = o[a];
            dir[a] = d[a];
        }
        block_rc.init(o, d);
        block_rc.within(scene->bounds, true);
        have_inner = false;
    }

    // VoxelSurfaceIter::next (surface.rs:379-410)
    bool inner_next(TraceStep *out) {
        RaycastStep rc;
        if (!voxel_rc.next(&rc)) return false;
        const Block &b = *inner_block;
        double antiscale = 1.0 / (double)b.resolution;  // Resolution::recip_f64
        double t = rc.t_distance * antiscale;
        size_t idx;
        if (!vol_index(b.vb, b.vsize, rc.cube, &idx)) {
            out->kind = TS_INVISIBLE;
            out->t_distance = t;
            return true;
        }
        const aicb_voxel &v = b.palette[b.indices[idx]];
        if (voxel_invisible(v)) {
            out->kind = TS_INVISIBLE;
            out->t_distance = t;
            return true;
        }
        out->kind = TS_ENTER_SURFACE;
        out->t_distance = t;
        Surface &s = out->surface;
        s.block_index = inner_block_index;
        std::memcpy(s.color, v.rgba, sizeof s.color);
        std::memcpy(s.emission, v.emission, sizeof s.emission);
        double ip[3];
        intersection_point(rc, sub_origin, dir, ip);
        for (int a = 0; a < 3; a++) {
            s.cube[a] = block_cube[a];
            s.voxel[a] = rc.cube[a];
            s.ip[a] = ip[a] * antiscale + (double)block_cube[a];
        }
        s.resolution = b.resolution;
        s.t_distance = t;
        s.normal = rc.face;
        return true;
    }

    // SurfaceIter::next (surface.rs:283-354)
    bool next(TraceStep *out) {
        if (have_inner && inner_next(out)) return true;
        have_inner = false;

        RaycastStep rc;
        if (!block_rc.next(&rc)) return false;

        size_t idx;
        if (!vol_index(sc->bounds, sc->size, rc.cube, &idx)) {
            out->kind = TS_INVISIBLE;
            out->t_distance = rc.t_distance;
            return true;
        }
        int bi = sc->ids[idx];
        const Block &b = sc->blocks[bi];
        if (b.invisible) {
            out->kind = TS_INVISIBLE;
            out->t_distance = rc.t_distance;
            return true;
        }
        if (b.single) {
            if (voxel_invisible(b.voxel)) {
                out->kind = TS_INVISIBLE;
                out->t_distance = rc.t_distance;
                return true;
            }
            out->kind = TS_ENTER_SURFACE;
            out->t_distance = rc.t_distance;
            Surface &s = out->surface;
            s.block_index = bi;
            std::memcpy(s.color, b.voxel.rgba, sizeof s.color);
            std::memcpy(s.emission, b.voxel.emission, sizeof s.emission);
            for (int a = 0; a < 3; a++) {
                s.cube[a] = rc.cube[a];
                s.voxel[a] = 0;
            }
            s.resolution = 1;
            s.t_distance = rc.t_distance;
            intersection_point(rc, origin, dir, s.ip);
            s.normal = rc.face;
            return true;
        }
        // recursive_raycast (raycast.rs:458-476)
        for (int a = 0; a < 3; a++) {
            block_cube[a] = rc.cube[a];
            sub_origin[a] = (origin[a] - (double)rc.cube[a]) * (double)b.resolution;
        }
        voxel_rc.init(sub_origin, dir);
        voxel_rc.within(b.vb, true);
        inner_block = &b;
        inner_block_index = bi;
        have_inner = true;
        out->kind = TS_ENTER_BLOCK;
        out->t_distance = rc.t_distance;
        out->block_index = bi;
        return true;
    }
};

enum { DS_SPAN = 0, DS_INVISIBLE = 1, DS_ENTER_BLOCK = 2 };
struct DepthStep {
    int kind;
    Surface surface;
    double exit_t_distance;
    double t_distance;
    int block_index;
};

// DepthIter (surface.rs:414-491)
struct DepthIter {
    SurfaceIter *it;
    bool have_last;
    Surface last_surface;
    bool have_buffered;
    DepthStep buffered;

    void init(SurfaceIter *s) {
        it = s;
        have_last = false;
        have_buffered = false;
    }
    void flush(double t, DepthStep *out) {
        if (have_last) {
            have_last = false;
            out->kind = DS_SPAN;
            out->surface = last_surface;
            out->exit_t_distance = t;
        } else {
            out->kind = DS_INVISIBLE;
        }
    }
    bool next(DepthStep *out) {
        if (have_buffered) {
            have_buffered = false;
            *out = buffered;
            return true;
        }
        TraceStep ts{};
        if (!it->next(&ts)) return false;
        switch (ts.kind) {
            case TS_ENTER_SURFACE: {
                double exit_t = ts.surface.t_distance;
                if (have_last) {
                    out->kind = DS_SPAN;
                    out->surface = last_surface;
                    out->exit_t_distance = exit_t;
                } else {
                    out->kind = DS_INVISIBLE;
                }
                last_surface = ts.surface;
                have_last = true;
                break;
            }
            case TS_INVISIBLE:
                flush(ts.t_distance, out);
                break;
            default:  // EnterBlock
                flush(ts.t_distance, out);
                buffered.kind = DS_ENTER_BLOCK;
                buffered.t_distance = ts.t_distance;
                buffered.block_index = ts.block_index;
                have_buffered = true;
                break;
        }
        return true;
    }
};

// ---------------------------------------------------------------------------------------------
// Colour arithmetic (raytracer_components.rs, color.rs)
// ---------------------------------------------------------------------------------------------
struct ColorBuf {
    float light[3];
    float transmittance;
};

// The two f32 transcendentals of the per-ray path: f32::powf (raytracer_components.rs:233) and f32::exp (sr.rs:751).
// Rust's std calls the platform libm; mode 0 does the same (glibc powf / expf).  Mode 1 ("cr") is the correctly
// rounded f32, computed by the CUDA path's own header (exact_math.cuh) compiled as host code, so that the oracle and
// the device do not depend on two f64 libms agreeing (libdevice's and glibc's f64 pow, rounded to f32, do not always).
// The parity tests compare the GPU with mode 1 exactly (0 ULP) and bound mode 0 against mode 1 per call (<= 1 ULP),
// so that a libm difference cannot hide a kernel difference.  Selected by orc_set_libm() / ORC_LIBM=cr.
static std::atomic<int> g_libm_mode{-1};
static int libm_mode() {
    int m = g_libm_mode.load(std::memory_order_relaxed);
    if (m < 0) {
        const char *e = std::getenv("ORC_LIBM");
        m = (e && std::strcmp(e, "cr") == 0) ? 1 : 0;
        g_libm_mode.store(m, std::memory_order_relaxed);
    }
    return m;
}
static inline float orc_powf_mode(float x, float y) { return libm_mode() ? aicb::powf_exact(x, y) : std::pow(x, y); }
static inline float orc_expf_mode(float x) { return libm_mode() ? aicb::expf_exact(x) : std::exp(x); }

// apply_transmittance (raytracer_components.rs:215-258)
static void apply_transmittance(const float color[4], float thickness_in, float out_color[4], float *coeff) {
    float thickness = rmaxf(thickness_in, 0.0f);
    if (thickness == 0.0f) {
        if (color[3] == 1.0f) {  // fully_opaque
            std::memcpy(out_color, color, 4 * sizeof(float));
            *coeff = 1.0f;
        } else {
            out_color[0] = out_color[1] = out_color[2] = out_color[3] = 0.0f;
            *coeff = 0.0f;
        }
        return;
    }
    float unit_t = 1.0f - color[3];
    float depth_t = orc_powf_mode(unit_t, thickness);  // f32::powf -> libm powf (or the round-once mode)
    float alpha = zo_clamped(1.0f - depth_t);
    out_color[0] = color[0];
    out_color[1] = color[1];
    out_color[2] = color[2];
    out_color[3] = alpha;
    float c = (unit_t == 1.0f) ? thickness : (depth_t - 1.0f) / (unit_t - 1.0f);
    *coeff = rmaxf(c, 0.0f);
}

// Rgb::luminance (color.rs:288-297)
static inline float luminance(const float c[3]) { return c[1] * 0.7152f + (c[0] * 0.2126f + c[2] * 0.0722f); }

// Rgba::from(ColorBuf) (raytracer_components.rs:122-146)
static void colorbuf_to_rgba(const ColorBuf &b, float out[4]) {
    if (b.transmittance >= 1.0f) {
        out[0] = out[1] = out[2] = out[3] = 0.0f;
        return;
    }
    float alpha = 1.0f - b.transmittance;
    float c[3] = {b.light[0] / alpha, b.light[1] / alpha, b.light[2] / alpha};
    bool ok = true;
    for (int i = 0; i < 3; i++) {
        if (c[i] > 0.0f) {
        } else if (c[i] == 0.0f) {
            c[i] = 0.0f;
        } else {
            ok = false;  // negative or NaN
        }
    }
    if (!ok) {
        c[0] = 1.0f;
        c[1] = 0.0f;
        c[2] = 0.0f;
    }
    out[0] = c[0];
    out[1] = c[1];
    out[2] = c[2];
    // ZeroOne::try_from(alpha).unwrap_or(1)
    if (alpha > 0.0f && alpha <= 1.0f) out[3] = alpha;
    else if (alpha == 0.0f) out[3] = 0.0f;
    else out[3] = 1.0f;
}

// component_to_srgb / component_to_srgb8 (color.rs:1038-1054)
static inline float component_to_srgb(float c) {
    if (c <= 0.0031308f) return c * (323.0f / 25.0f);
    return (211.0f * std::pow(c, 5.0f / 12.0f) - 11.0f) / 200.0f;
}
static inline uint8_t component_to_srgb8(float c) { return sat_u8(std::round(component_to_srgb(c) * 255.0f)); }

// Camera::post_process_color (camera_struct.rs:376-382) + ToneMappingOperator::apply
// (graphics_options.rs:352-368) + Rgba::to_srgb8 (color.rs:669-676)
static void encode_srgb8(const ColorBuf &b, float exposure, int tone_mapping, float maximum_intensity,
                         uint8_t out[4]) {
    float rgba[4];
    colorbuf_to_rgba(b, rgba);
    float c[3];
    for (int i = 0; i < 3; i++) c[i] = ps_mul(rgba[i], exposure);
    if (std::isfinite(maximum_intensity)) {
        if (tone_mapping == AICB_TONE_CLAMP) {
            for (int i = 0; i < 3; i++) c[i] = (c[i] > maximum_intensity) ? maximum_intensity : c[i];
        } else {
            float scale = 1.0f / (1.0f + luminance(c) / maximum_intensity);
            float s = ps_clamped(scale);
            for (int i = 0; i < 3; i++) c[i] = ps_mul(c[i], s);
        }
    }
    out[0] = component_to_srgb8(c[0]);
    out[1] = component_to_srgb8(c[1]);
    out[2] = component_to_srgb8(c[2]);
    out[3] = sat_u8(std::round(rgba[3] * 255.0f));
}

// ---------------------------------------------------------------------------------------------
// Accumulators (accum.rs, text.rs)
// ---------------------------------------------------------------------------------------------
enum { EX_NONE = -1, EX_ENTER_SPACE = 0, EX_SKY = 1, EX_BACKDROP = 2, EX_INCOMPLETE = 3, EX_PAINT = 4, EX_DEBUG_RG = 5 };
struct Hit {
    int exception;
    ColorBuf surface;
    bool has_t;
    double t_distance;
    int block_index;  // -1 for exceptions
    bool has_position;
    int32_t cube[3];
    int resolution;
    int32_t voxel[3];
    int face;
};

struct Accum {
    int mode;  // 0 ColorBuf, 1 CharacterBuf, 2 DepthBuf
    ColorBuf color;
    // passive observers (mode 0) / DepthBuf state (mode 2)
    double depth;
    bool have_hit;
    aicb_hit first_hit;
    // CharacterBuf (text.rs:52-123): -2 Empty '.', -1 EnteredSpace ' ', -3 Hit("X"), -4 Hit(" "), >=0 Hit(block)
    int32_t text;

    void init(int m) {
        mode = m;
        color.light[0] = color.light[1] = color.light[2] = 0.0f;
        color.transmittance = 1.0f;
        depth = INF;
        have_hit = false;
        for (int a = 0; a < 3; a++) first_hit.cube[a] = first_hit.voxel[a] = -1;
        first_hit.resolution = -1;
        first_hit.face = -1;
        text = -2;
    }
    bool opaque() const {
        switch (mode) {
            case 0: return color.transmittance < 1.0f / 256.0f;  // raytracer_components.rs:105-109
            case 1: return text >= 0 || text <= -3;
            default: return depth < INF;  // accum.rs:269-273
        }
    }
    void add(const Hit &h) {
        // observers
        if (h.has_t) depth = std::fmin(depth, h.t_distance);  // accum.rs:275-282 (f64::min ignores NaN)
        if (h.has_position && !have_hit) {
            have_hit = true;
            for (int a = 0; a < 3; a++) {
                first_hit.cube[a] = h.cube[a];
                first_hit.voxel[a] = h.voxel[a];
            }
            first_hit.resolution = h.resolution;
            first_hit.face = h.face;
        }
        if (mode == 1) {
            // text.rs:90-98
            bool is_hit = text >= 0 || text <= -3;
            if (h.exception == EX_ENTER_SPACE && !is_hit) {
                text = -1;
            } else if (h.exception == EX_SKY) {
            } else if (!is_hit) {
                if (h.exception == EX_INCOMPLETE) text = -3;
                else if (h.exception != EX_NONE) text = -4;
                else text = h.block_index;
            }
            return;
        }
        // ColorBuf::add (accum.rs:227-238)
        if (h.exception == EX_DEBUG_RG) {
            float red = ps_clamped(h.surface.light[0]);
            float green = ps_clamped(h.surface.light[1]);
            float rgba[4];
            colorbuf_to_rgba(color, rgba);
            float blue = ps_clamped(luminance(rgba) * 0.2f);
            color.light[0] = red;
            color.light[1] = green;
            color.light[2] = blue;
            color.transmittance = 0.0f;
        } else {
            // add_color_internal (raytracer_components.rs:87-92)
            for (int i = 0; i < 3; i++) color.light[i] = color.light[i] + h.surface.light[i] * color.transmittance;
            color.transmittance = color.transmittance * h.surface.transmittance;
        }
    }
};

// ---------------------------------------------------------------------------------------------
// The bounce RNG (raytracer/mod.rs:56: `type BounceRng = rand::rngs::SmallRng`) and the direction distribution
// (surface.rs:135-136: rand_distr::UnitSphere).  Both crates are dependencies that are NOT under /root/reference
// (Cargo.lock: rand 0.10.1, rand_distr 0.6.0): restated from their published algorithms, parity UNPINNED — the
// reference itself excludes LightingOption::Bounce from its image tests (test-renderers/cases/src/lib.rs:45-50).
//   SmallRng on 64-bit targets = xoshiro256++ (Blackman & Vigna); seed_from_u64 fills the 256-bit state with
//   SplitMix64 outputs; an all-zero state is replaced by seed_from_u64(0).
//   Uniform<f64>::new(-1, 1): value1_2 = f64 from (next_u64 >> 12) with exponent 0; (value1_2 - 1) * 2 + (-1).
//   UnitSphere (Marsaglia 1972): draw (x1, x2) until x1^2 + x2^2 < 1; (2 x1 sqrt(1-s), 2 x2 sqrt(1-s), 1 - 2 s).
// The known-answer vectors of the xoshiro256++ reference implementation pin the generator itself
// (tests/test_oracle_bounce.py).
// ---------------------------------------------------------------------------------------------
struct BounceRng {
    uint64_t s[4];
};
static inline uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static void bounce_rng_seed(BounceRng *r, uint64_t state) {
    for (int i = 0; i < 4; i++) {
        state += 0x9e3779b97f4a7c15ull;
        uint64_t z = state;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        r->s[i] = z ^ (z >> 31);
    }
    if ((r->s[0] | r->s[1] | r->s[2] | r->s[3]) == 0) bounce_rng_seed(r, 0);
}
static uint64_t bounce_rng_next(BounceRng *r) {
    uint64_t *s = r->s;
    const uint64_t result = rotl64(s[0] + s[3], 23) + s[0];
    const uint64_t t = s[1] << 17;
    s[2] ^= s[0];
    s[3] ^= s[1];
    s[1] ^= s[2];
    s[0] ^= s[3];
    s[2] ^= t;
    s[3] = rotl64(s[3], 45);
    return result;
}
static inline double bounce_uniform_m1_1(BounceRng *r) {
    const uint64_t bits = (bounce_rng_next(r) >> 12) | 0x3ff0000000000000ull;
    double value1_2;
    std::memcpy(&value1_2, &bits, 8);
    const double value0_1 = value1_2 - 1.0;
    return value0_1 * 2.0 + (-1.0);
}
static void bounce_unit_sphere(BounceRng *r, double out[3]) {
    for (;;) {
        const double x1 = bounce_uniform_m1_1(r), x2 = bounce_uniform_m1_1(r);
        const double sum = x1 * x1 + x2 * x2;
        if (sum >= 1.0) continue;
        const double factor = 2.0 * std::sqrt(1.0 - sum);
        out[0] = x1 * factor;
        out[1] = x2 * factor;
        out[2] = 1.0 - 2.0 * sum;
        return;
    }
}

// ---------------------------------------------------------------------------------------------
// TracingState + trace_ray_impl (sr.rs:135-238, 595-769)
// ---------------------------------------------------------------------------------------------
struct Tracer {
    const orc_scene *sc;
    const aicb_options *opt;
    Accum *acc;
    double t_to_absolute_distance;
    float t_to_view_distance;
    bool have_fog;
    float fog_light[3];
    float fog_blend;
    size_t cubes_traced;
    size_t secondary_cubes = 0;   // TracingState::secondary_info (sr.rs:615-616)
    bool allow_bounce = true;     // trace_ray_impl's allow_ray_bounce (sr.rs:139)
    bool force_sky = false;       // secondary rays are traced with include_sky = true (surface.rs:159)
    BounceRng rng{};

    // count_step_should_stop (sr.rs:625-656)
    bool count_step_should_stop() {
        if (cubes_traced == 0) {
            Hit h{};
            h.exception = EX_ENTER_SPACE;
            h.surface = ColorBuf{{0, 0, 0}, 1.0f};  // ColorBuf::from(Rgba::TRANSPARENT)
            h.block_index = -1;
            acc->add(h);
        }
        cubes_traced += 1;
        if (cubes_traced > 1000) {
            Hit h{};
            h.exception = EX_INCOMPLETE;
            h.surface = ColorBuf{{0, 0, 0}, 1.0f};
            h.block_index = -1;
            acc->add(h);
            return true;
        }
        return acc->opaque();
    }

    // distance_fog (sr.rs:745-768)
    bool distance_fog(double t_distance, float *amount) const {
        if (!have_fog) return false;
        float rel = rclampf((float)t_distance * t_to_view_distance, 0.0f, 1.0f);
        float fog_exponential = 1.0f - orc_expf_mode(-1.6f * rel);
        float fog_exp_fudged = fog_exponential / 0.79810348f;
        float p4 = (rel * rel) * (rel * rel);  // powi(4)
        *amount = zo_clamped(fog_exp_fudged * (1.0f - fog_blend) + p4 * fog_blend);
        return true;
    }

    // get_interpolated_light (sr.rs:248-359)
    void interpolated_light(const Surface &s, int mode, float out[3]) const {
        const double eps = 0.5 / 256.0;
        int fx[3], fy[3], fz[3];
        rotation_from_nz(s.normal, fx, fy, fz);
        double rfx[3], rfy[3];
        for (int i = 0; i < 3; i++) {
            rfx[i] = (double)fx[i];
            rfy[i] = (double)fy[i];
        }
        const double *sp = s.ip;
        double mix_1 = rem_euclid1((sp[0] * rfx[0] + sp[1] * rfx[1] + sp[2] * rfx[2]) - 0.5);
        double mix_2 = rem_euclid1((sp[0] * rfy[0] + sp[1] * rfy[1] + sp[2] * rfy[2]) - 0.5);
        double dir_1[3], dir_2[3];
        if (mix_1 > 0.5) {
            mix_1 = 1.0 - mix_1;
            for (int i = 0; i < 3; i++) dir_1[i] = -rfx[i];
        } else {
            for (int i = 0; i < 3; i++) dir_1[i] = rfx[i];
        }
        if (mix_2 > 0.5) {
            mix_2 = 1.0 - mix_2;
            for (int i = 0; i < 3; i++) dir_2[i] = -rfy[i];
        } else {
            for (int i = 0; i < 3; i++) dir_2[i] = rfy[i];
        }
        auto modifier = [mode](double x) -> double {
            if (mode == AICB_LIGHT_COARSE) {  // coarsestep (surface.rs:510-514)
                return (rclamp(std::floor(x * 4.0), 0.0, 3.0) + 0.5) / 4.0;
            } else if (mode == AICB_LIGHT_SMOOTHSTEP) {  // smoothstep (surface.rs:517-520)
                double c = rclamp(x, 0.0, 1.0);
                return 3.0 * (c * c) - 2.0 * ((c * c) * c);
            }
            return x;
        };
        mix_1 = modifier(mix_1);
        mix_2 = modifier(mix_2);

        const double lin_lo = -0.5, lin_hi = 0.5;
        double off_near12[3], off_near1far2[3], off_near2far1[3], off_far12[3];
        for (int i = 0; i < 3; i++) {
            off_near12[i] = dir_1[i] * lin_lo + dir_2[i] * lin_lo;
            off_near1far2[i] = dir_1[i] * lin_lo + dir_2[i] * lin_hi;
            off_near2far1[i] = dir_1[i] * lin_hi + dir_2[i] * lin_lo;
            off_far12[i] = dir_1[i] * lin_hi + dir_2[i] * lin_hi;
        }

        // face.dot(v) (face.rs:733-746); cube.center() = cube + 0.5
        auto face_dot = [&](const double v[3]) -> double {
            switch (s.normal) {
                case AICB_FACE_NX: return -v[0];
                case AICB_FACE_NY: return -v[1];
                case AICB_FACE_NZ: return -v[2];
                case AICB_FACE_PX: return v[0];
                case AICB_FACE_PY: return v[1];
                case AICB_FACE_PZ: return v[2];
                default: return 0.0;
            }
        };
        double center[3] = {(double)s.cube[0] + 0.5, (double)s.cube[1] + 0.5, (double)s.cube[2] + 0.5};
        double height_in_cube = face_dot(sp) - face_dot(center) + 0.5;

        double normal[3] = {0, 0, 0};
        if (s.normal != AICB_FACE_WITHIN) {
            int ax = (s.normal - 1) % 3;
            normal[ax] = (s.normal >= AICB_FACE_PX) ? 1.0 : -1.0;
        }

        auto get_light = [&](const double p[3]) -> PackedLight {
            int32_t c[3];
            if (cube_containing(p, c)) return get_packed_light(*sc, c);
            return sc->sky_mean;
        };
        auto mix4 = [](const float a[4], const float b[4], float amount, float out4[4]) {
            for (int i = 0; i < 4; i++) out4[i] = a[i] + (b[i] - a[i]) * amount;
        };
        auto fetch_2d = [&](const double origin_2d[3], float out4[4]) {
            double p[3];
            for (int i = 0; i < 3; i++) p[i] = origin_2d[i] + off_near12[i];
            PackedLight near12 = get_light(p);
            for (int i = 0; i < 3; i++) p[i] = origin_2d[i] + off_near1far2[i];
            PackedLight near1far2 = get_light(p);
            for (int i = 0; i < 3; i++) p[i] = origin_2d[i] + off_near2far1[i];
            PackedLight near2far1 = get_light(p);
            for (int i = 0; i < 3; i++) p[i] = origin_2d[i] + off_far12[i];
            PackedLight far12 = get_light(p);
            if (!pl_valid(near1far2) && !pl_valid(near2far1)) far12 = near12;
            float a[4], b[4], c[4], d[4], ab[4], cd[4];
            pl_value_ao(near12, a);
            pl_value_ao(near1far2, b);
            pl_value_ao(near2far1, c);
            pl_value_ao(far12, d);
            mix4(a, b, (float)mix_2, ab);
            mix4(c, d, (float)mix_2, cd);
            mix4(ab, cd, (float)mix_1, out4);
        };

        double o2d[3];
        for (int i = 0; i < 3; i++) o2d[i] = sp[i] + normal[i] * (1.0 - eps);
        float front[4];
        fetch_2d(o2d, front);
        float final_mix[4];
        if (height_in_cube > (1.0 - eps)) {
            std::memcpy(final_mix, front, sizeof front);
        } else {
            for (int i = 0; i < 3; i++) o2d[i] = sp[i] + normal[i] * eps;
            float same[4];
            fetch_2d(o2d, same);
            mix4(same, front, (float)height_in_cube, final_mix);
        }
        float w = rmaxf(final_mix[3], 0.1f);
        for (int i = 0; i < 3; i++) {
            float v = final_mix[i] / w;
            out[i] = (v == 0.0f) ? 0.0f : v;  // Rgb::try_from normalises -0
        }
    }

    // compute_illumination (surface.rs:113-206)
    void illumination(const Surface &s, bool bounce, float out[3]) {
        if (opt->lighting_display == AICB_LIGHT_BOUNCE && bounce) {   // surface.rs:119-166
            const int samples = opt->bounce_samples;
            float accum[3] = {0.0f, 0.0f, 0.0f};
            double normal[3] = {0, 0, 0};
            if (s.normal != AICB_FACE_WITHIN) normal[(s.normal - 1) % 3] = (s.normal >= AICB_FACE_PX) ? 1.0 : -1.0;
            for (int k = 0; k < samples; k++) {
                double sphere[3], dir[3], origin[3];
                bounce_unit_sphere(&rng, sphere);
                for (int a = 0; a < 3; a++) {
                    dir[a] = normal[a] + sphere[a];
                    origin[a] = s.ip[a] + normal[a] * 0.0001;
                }
                Accum light_accum;
                light_accum.init(0);
                Tracer child;
                child.sc = sc;
                child.opt = opt;
                child.acc = &light_accum;
                child.allow_bounce = false;
                child.force_sky = true;
                secondary_cubes += child.trace(origin, dir);
                float rgba[4];
                colorbuf_to_rgba(light_accum.color, rgba);
                for (int a = 0; a < 3; a++) accum[a] = accum[a] + rgba[a];
            }
            const float recip = ps_clamped(1.0f / (float)samples);   // Rgb * f32 (color.rs:912-927)
            for (int a = 0; a < 3; a++) out[a] = ps_mul(accum[a], recip);
            return;
        }
        switch (opt->lighting_display) {
            case AICB_LIGHT_NONE:
                out[0] = out[1] = out[2] = 1.0f;
                return;
            case AICB_LIGHT_FLAT:
            case AICB_LIGHT_BOUNCE: {  // no bounce at this surface (budget spent, or not fully opaque) -> Flat (surface.rs:171-176)
                int32_t c[3] = {s.cube[0], s.cube[1], s.cube[2]};
                if (s.normal != AICB_FACE_WITHIN) {
                    int ax = (s.normal - 1) % 3;
                    c[ax] += (s.normal >= AICB_FACE_PX) ? 1 : -1;
                }
                PackedLight p = get_packed_light(*sc, c);
                out[0] = LUT.v[p.r];
                out[1] = LUT.v[p.g];
                out[2] = LUT.v[p.b];
                return;
            }
            default:
                interpolated_light(s, opt->lighting_display, out);
                return;
        }
    }

    // Surface::to_light (surface.rs:73-106) + trace_through_surface (sr.rs:697-717)
    void trace_through_surface(const Surface &s) {
        float diffuse[4];
        std::memcpy(diffuse, s.color, sizeof diffuse);
        if (opt->transparency == AICB_TRANSPARENCY_THRESHOLD) {  // limit_alpha (graphics_options.rs:496-507)
            if (diffuse[3] > opt->transparency_threshold) {
                diffuse[3] = 1.0f;
            } else {
                diffuse[0] = diffuse[1] = diffuse[2] = diffuse[3] = 0.0f;
            }
        }
        if (diffuse[3] == 0.0f && s.emission[0] == 0.0f && s.emission[1] == 0.0f && s.emission[2] == 0.0f) return;

        float illum[3];
        illumination(s, allow_bounce && diffuse[3] == 1.0f, illum);   // surface.rs:85-88: the RNG only where fully opaque

        // diffuse.reflect(illum) + emission (color.rs:708-710)
        float outgoing[3];
        for (int i = 0; i < 3; i++) outgoing[i] = ps_mul(ps_mul(diffuse[i], illum[i]), diffuse[3]) + s.emission[i];
        float transmittance = 1.0f - diffuse[3];

        float fog_amount;
        if (distance_fog(s.t_distance, &fog_amount)) {
            float comp = 1.0f - fog_amount;
            for (int i = 0; i < 3; i++) outgoing[i] = ps_mul(outgoing[i], comp) + ps_mul(fog_light[i], fog_amount);
            transmittance = transmittance * comp;
        }

        Hit h{};
        h.exception = EX_NONE;
        h.surface.light[0] = outgoing[0];
        h.surface.light[1] = outgoing[1];
        h.surface.light[2] = outgoing[2];
        h.surface.transmittance = transmittance;
        h.has_t = true;
        h.t_distance = s.t_distance;
        h.block_index = s.block_index;
        h.has_position = true;
        for (int a = 0; a < 3; a++) {
            h.cube[a] = s.cube[a];
            h.voxel[a] = s.voxel[a];
        }
        h.resolution = s.resolution;
        h.face = s.normal;
        acc->add(h);
    }

    // trace_through_span (sr.rs:720-740)
    void trace_through_span(const Surface &s_in, double exit_t) {
        Surface s = s_in;
        float thickness = (float)((exit_t - s.t_distance) * t_to_absolute_distance);
        float adj[4], coeff;
        apply_transmittance(s.color, thickness, adj, &coeff);
        std::memcpy(s.color, adj, sizeof adj);
        float k = ps_clamped(coeff);  // Rgb * f32 (color.rs:912-927)
        for (int i = 0; i < 3; i++) s.emission[i] = ps_mul(s.emission[i], k);
        trace_through_surface(s);
    }

    // trace_ray_impl (sr.rs:135-238) + finish (sr.rs:658-693)
    size_t trace(const double origin[3], const double dir[3]) {
        bool include_sky = force_sky || opt->include_sky != 0;
        if (allow_bounce) {   // sr.rs:165-178: seeded from the direction's bits
            uint64_t b[3];
            std::memcpy(b, dir, 24);
            bounce_rng_seed(&rng, b[0] + b[1] + b[2]);
        }
        secondary_cubes = 0;
        float sky_light[3] = {0, 0, 0};
        if (include_sky) sky_sample(sc->sky, dir, sky_light);
        t_to_absolute_distance = std::sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        t_to_view_distance = (float)(t_to_absolute_distance / opt->view_distance);
        have_fog = (opt->fog != AICB_FOG_NONE) && include_sky;
        std::memcpy(fog_light, sky_light, sizeof sky_light);
        fog_blend = (opt->fog == AICB_FOG_ABRUPT) ? 1.0f : (opt->fog == AICB_FOG_COMPROMISE) ? 0.5f : 0.0f;
        cubes_traced = 0;

        SurfaceIter it;
        it.init(sc, origin, dir);
        if (opt->transparency == AICB_TRANSPARENCY_VOLUMETRIC) {
            DepthIter di;
            di.init(&it);
            DepthStep ds{};
            while (di.next(&ds)) {
                if (count_step_should_stop()) break;
                if (ds.kind == DS_SPAN) trace_through_span(ds.surface, ds.exit_t_distance);
            }
        } else {
            TraceStep ts{};
            while (it.next(&ts)) {
                if (count_step_should_stop()) break;
                if (ts.kind == TS_ENTER_SURFACE) trace_through_surface(ts.surface);
            }
        }
        // finish
        Hit h{};
        h.exception = EX_SKY;
        if (include_sky) {
            h.surface = ColorBuf{{sky_light[0] * 1.0f, sky_light[1] * 1.0f, sky_light[2] * 1.0f}, 1.0f - 1.0f};
        } else {
            h.surface = ColorBuf{{0, 0, 0}, 1.0f};
        }
        h.has_t = true;
        h.t_distance = INF;
        h.block_index = -1;
        acc->add(h);
        if (opt->debug_pixel_cost) {
            Hit d{};
            d.exception = EX_DEBUG_RG;
            float k = ps_clamped((float)cubes_traced);
            // (rgb_const!(0.02, 0.002, 0.0) * n).with_alpha_one().into()
            d.surface = ColorBuf{{ps_mul(0.02f, k) * 1.0f, ps_mul(0.002f, k) * 1.0f, ps_mul(0.0f, k) * 1.0f}, 0.0f};
            d.block_index = -1;
            acc->add(d);
        }
        return cubes_traced + secondary_cubes;   // RaytraceInfo + secondary_info (sr.rs:689-692)
    }
};

// ---------------------------------------------------------------------------------------------
// Pixel -> ray (viewport.rs:104-113, renderer.rs:424-451, camera_struct.rs:238-257)
// ---------------------------------------------------------------------------------------------
static void project_ndc3(const aicb_camera &cam, double x, double y, double z, double out[3]) {
    const double *m = cam.inverse_projection_view;  // m11 m12 m13 m14 / m21 ... row-major
    // euclid Transform3D::transform_point3d_homogeneous
    double hx = x * m[0] + y * m[4] + z * m[8] + m[12];
    double hy = x * m[1] + y * m[5] + z * m[9] + m[13];
    double hz = x * m[2] + y * m[6] + z * m[10] + m[14];
    double hw = x * m[3] + y * m[7] + z * m[11] + m[15];
    if (hw > 0.0) {
        out[0] = hx / hw;
        out[1] = hy / hw;
        out[2] = hz / hw;
    } else {
        out[0] = out[1] = out[2] = std::numeric_limits<double>::quiet_NaN();
    }
}

static void pixel_ray(const aicb_camera &cam, uint32_t xch, uint32_t ych, int sample, double origin[3], double dir[3]) {
    double W = (double)cam.fb_width, H = (double)cam.fb_height;
    double x0 = (double)xch / W * 2.0 - 1.0;
    double x1 = (double)(xch + 1) / W * 2.0 - 1.0;
    double y0 = -((double)ych / H * 2.0 - 1.0);
    double y1 = -((double)(ych + 1) / H * 2.0 - 1.0);
    double px, py;
    if (sample < 0) {
        // Box2D::center = (min + max) / 2
        px = (x0 + x1) / 2.0;
        py = (y0 + y1) / 2.0;
    } else {
        static const double SP[4][2] = {{1. / 8., 5. / 8.}, {3. / 8., 1. / 8.}, {5. / 8., 7. / 8.}, {7. / 8., 3. / 8.}};
        px = x0 + (x1 - x0) * SP[sample][0];
        py = y0 + (y1 - y0) * SP[sample][1];
    }
    double nearp[3], farp[3];
    project_ndc3(cam, px, py, 0.0, nearp);
    project_ndc3(cam, px, py, 1.0, farp);
    for (int a = 0; a < 3; a++) {
        origin[a] = nearp[a];
        dir[a] = farp[a] - nearp[a];
    }
}

struct PixelOut {
    ColorBuf color;
    double depth;
    aicb_hit hit;
    uint32_t steps;
    int32_t text;
};

// RtScene::trace_patch (renderer.rs:424-451) with only the world layer.
static size_t trace_pixel(const orc_scene *sc, const aicb_camera &cam, const aicb_options &opt, int accum_mode,
                          uint32_t x, uint32_t y, PixelOut *po) {
    size_t total = 0;
    Tracer tr;
    tr.sc = sc;
    tr.opt = &opt;
    if (opt.antialiasing_always) {
        Accum acc[4];
        for (int i = 0; i < 4; i++) {
            acc[i].init(accum_mode);
            tr.acc = &acc[i];
            double o[3], d[3];
            pixel_ray(cam, x, y, i, o, d);
            total += tr.trace(o, d);
        }
        // ColorBuf::mean (raytracer_components.rs:97-102): sums fold from zero
        float l[3] = {0, 0, 0}, t = 0.0f;
        for (int i = 0; i < 4; i++) {
            for (int c = 0; c < 3; c++) l[c] = l[c] + acc[i].color.light[c];
            t = t + acc[i].color.transmittance;
        }
        for (int c = 0; c < 3; c++) po->color.light[c] = l[c] / 4.0f;
        po->color.transmittance = t / 4.0f;
        // DepthBuf::mean = min (accum.rs:284-297); hit/text: first sample with a hit (text.rs:100-113)
        po->depth = INF;
        for (int i = 0; i < 4; i++) po->depth = std::fmin(po->depth, acc[i].depth);
        po->hit = acc[0].first_hit;
        po->text = acc[0].text;
        for (int i = 0; i < 4; i++)
            if (acc[i].have_hit) {
                po->hit = acc[i].first_hit;
                break;
            }
        {
            // reduce: (Hit, _) | (_, Hit) => Hit(first); (Entered, Entered) => Entered; else Empty
            int32_t cur = acc[0].text;
            for (int i = 1; i < 4; i++) {
                int32_t b = acc[i].text;
                bool ah = cur >= 0 || cur <= -3, bh = b >= 0 || b <= -3;
                if (ah) {
                } else if (bh) cur = b;
                else if (cur == -1 && b == -1) cur = -1;
                else cur = -2;
            }
            po->text = cur;
        }
    } else {
        Accum acc;
        acc.init(accum_mode);
        tr.acc = &acc;
        double o[3], d[3];
        pixel_ray(cam, x, y, -1, o, d);
        total += tr.trace(o, d);
        po->color = acc.color;
        po->depth = acc.depth;
        po->hit = acc.first_hit;
        po->text = acc.text;
    }
    po->steps = (uint32_t)total;
    return total;
}

// RtScene::trace_patch + trace_ray_through_layers (renderer.rs:424-478): UI layer (no sky), backdrop, world layer
// (sky), NO_WORLD_TO_SHOW if the accumulator is not opaque in the end.  ColorBuf accumulators only.
static size_t trace_pixel_layers(const orc_scene *world, const aicb_camera *wcam, const aicb_options *wopt,
                                 const orc_scene *ui, const aicb_camera *ucam, const aicb_options *uopt,
                                 const float *backdrop_rgba, const float *no_world_rgba, uint32_t x, uint32_t y, ColorBuf *out) {
    size_t total = 0;
    const aicb_options *lead = world ? wopt : uopt;
    const int n = lead->antialiasing_always ? 4 : 1;
    ColorBuf acc_color[4];
    for (int i = 0; i < n; i++) {
        Accum acc;
        acc.init(0);
        if (ui) {
            aicb_options o = *uopt;
            o.include_sky = 0;
            Tracer tr;
            tr.sc = ui;
            tr.opt = &o;
            tr.acc = &acc;
            double ro[3], rd[3];
            pixel_ray(*ucam, x, y, n == 4 ? i : -1, ro, rd);
            total += tr.trace(ro, rd);
        }
        if (backdrop_rgba && !(backdrop_rgba[0] == 0.0f && backdrop_rgba[1] == 0.0f && backdrop_rgba[2] == 0.0f && backdrop_rgba[3] == 0.0f)) {
            Hit h{};
            h.exception = EX_BACKDROP;
            // ColorBuf::from(Rgba) (raytracer_components.rs:111-120)
            h.surface = ColorBuf{{backdrop_rgba[0] * backdrop_rgba[3], backdrop_rgba[1] * backdrop_rgba[3], backdrop_rgba[2] * backdrop_rgba[3]},
                                 1.0f - backdrop_rgba[3]};
            h.block_index = -1;
            acc.add(h);
        }
        if (world) {
            aicb_options o = *wopt;
            o.include_sky = 1;
            Tracer tr;
            tr.sc = world;
            tr.opt = &o;
            tr.acc = &acc;
            double ro[3], rd[3];
            pixel_ray(*wcam, x, y, n == 4 ? i : -1, ro, rd);
            total += tr.trace(ro, rd);
        }
        if (!acc.opaque() && no_world_rgba) {   // *accum = P::paint(NO_WORLD_TO_SHOW): a fresh accumulator with that one hit
            acc.init(0);
            Hit h{};
            h.exception = EX_PAINT;
            h.surface = ColorBuf{{no_world_rgba[0] * no_world_rgba[3], no_world_rgba[1] * no_world_rgba[3], no_world_rgba[2] * no_world_rgba[3]},
                                 1.0f - no_world_rgba[3]};
            h.block_index = -1;
            acc.add(h);
        }
        acc_color[i] = acc.color;
    }
    if (n == 4) {
        float l[3] = {0, 0, 0}, t = 0.0f;
        for (int i = 0; i < 4; i++) {
            for (int c = 0; c < 3; c++) l[c] = l[c] + acc_color[i].light[c];
            t = t + acc_color[i].transmittance;
        }
        for (int c = 0; c < 3; c++) out->light[c] = l[c] / 4.0f;
        out->transmittance = t / 4.0f;
    } else {
        *out = acc_color[0];
    }
    return total;
}

}  // namespace orc

// ---------------------------------------------------------------------------------------------
// C API
// ---------------------------------------------------------------------------------------------
using namespace orc;

extern "C" {

double orc_scale_to_integer_step(double s, double ds) { return scale_to_integer_step(s, ds); }

int orc_raycast(const double origin[3], const double dir[3], const int32_t *b, int include_exit, int max_steps,
                int32_t *out_cube_face, double *out_t, double *out_point) {
    Raycaster rc;
    rc.init(origin, dir);
    double ray_o[3] = {origin[0], origin[1], origin[2]};
    if (b) {
        Aab bb{{b[0], b[1], b[2]}, {b[3], b[4], b[5]}};
        rc.within(bb, include_exit != 0);
    }
    int n = 0;
    RaycastStep s;
    while (n < max_steps && rc.next(&s)) {
        out_cube_face[4 * n + 0] = s.cube[0];
        out_cube_face[4 * n + 1] = s.cube[1];
        out_cube_face[4 * n + 2] = s.cube[2];
        out_cube_face[4 * n + 3] = s.face;
        out_t[n] = s.t_distance;
        if (out_point) intersection_point(s, ray_o, dir, out_point + 3 * n);
        n++;
    }
    return n;
}

int orc_recursive_raycast(const double origin[3], const double dir[3], int nth, int resolution,
                          const int32_t b[6], int max_steps, double out_sub_ray[6], int32_t *out_cube_face,
                          double *out_t) {
    Raycaster rc;
    rc.init(origin, dir);
    RaycastStep s;
    for (int i = 0; i <= nth; i++)
        if (!rc.next(&s)) return -1;
    double sub_o[3];
    for (int a = 0; a < 3; a++) {
        sub_o[a] = (origin[a] - (double)s.cube[a]) * (double)resolution;
        out_sub_ray[a] = sub_o[a];
        out_sub_ray[3 + a] = dir[a];
    }
    Raycaster in;
    in.init(sub_o, dir);
    Aab bb{{b[0], b[1], b[2]}, {b[3], b[4], b[5]}};
    in.within(bb, true);
    int n = 0;
    while (n < max_steps && in.next(&s)) {
        out_cube_face[4 * n + 0] = s.cube[0];
        out_cube_face[4 * n + 1] = s.cube[1];
        out_cube_face[4 * n + 2] = s.cube[2];
        out_cube_face[4 * n + 3] = s.face;
        out_t[n] = s.t_distance;
        n++;
    }
    return n;
}

// The bounce RNG for tests/test_oracle_bounce.py: state from seed_from_u64(seed) or, if state_or_null is given, from
// those four words; writes n next_u64() outputs, then n_dirs UnitSphere samples drawn after them.
void orc_bounce_rng(uint64_t seed, const uint64_t *state_or_null, size_t n, uint64_t *out, size_t n_dirs, double (*dirs)[3]) {
    BounceRng r;
    if (state_or_null) std::memcpy(r.s, state_or_null, 32);
    else bounce_rng_seed(&r, seed);
    for (size_t i = 0; i < n; i++) out[i] = bounce_rng_next(&r);
    for (size_t i = 0; i < n_dirs; i++) bounce_unit_sphere(&r, dirs[i]);
}

void orc_apply_transmittance(const float rgba[4], float thickness, float out[5]) {
    apply_transmittance(rgba, thickness, out, out + 4);
}
float orc_packed_light_lut(int v) { return LUT.v[v & 255]; }
int orc_packed_light_scalar_in(float v) { return scalar_in(v); }
void orc_to_srgb8(const float cb[4], float exposure, int tone_mapping, float maximum_intensity, uint8_t out[4]) {
    ColorBuf b{{cb[0], cb[1], cb[2]}, cb[3]};
    encode_srgb8(b, exposure, tone_mapping, maximum_intensity, out);
}

orc_scene *orc_scene_create(const aicb_scene_desc *d) {
    orc_scene *s = new orc_scene();
    for (int a = 0; a < 3; a++) {
        s->bounds.lo[a] = d->bounds.lower[a];
        s->bounds.hi[a] = d->bounds.lower[a] + (int32_t)d->bounds.size[a];
        s->size[a] = (int32_t)d->bounds.size[a];
    }
    size_t vol = (size_t)s->size[0] * s->size[1] * s->size[2];
    s->ids.assign(d->block_ids, d->block_ids + vol);
    s->has_light = d->light != nullptr;
    if (s->has_light) {
        s->light.resize(vol);
        std::memcpy(s->light.data(), d->light, vol * 4);
    }
    s->blocks.resize(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) {
        const aicb_block_desc &bd = d->blocks[i];
        Block &b = s->blocks[i];
        b.invisible = bd.is_air != 0;
        b.resolution = bd.resolution;
        for (int a = 0; a < 3; a++) {
            b.vb.lo[a] = bd.voxel_bounds.lower[a];
            b.vb.hi[a] = bd.voxel_bounds.lower[a] + (int32_t)bd.voxel_bounds.size[a];
            b.vsize[a] = (int32_t)bd.voxel_bounds.size[a];
        }
        if (bd.indices == nullptr) {
            b.single = true;
            b.voxel = bd.n_palette ? bd.palette[0] : VOXEL_AIR;
        } else if (bd.resolution == 1) {
            // single_voxel_or_palette (voxel_storage.rs:371-383): indices.get([0,0,0]) or AIR
            b.single = true;
            int32_t z[3] = {0, 0, 0};
            size_t idx;
            b.voxel = vol_index(b.vb, b.vsize, z, &idx) ? bd.palette[bd.indices[idx]] : VOXEL_AIR;
        } else {
            b.single = false;
            b.indices.assign(bd.indices, bd.indices + bd.n_indices);
            b.palette.assign(bd.palette, bd.palette + bd.n_palette);
        }
    }
    s->sky = d->sky;
    build_block_sky(s);
    return s;
}
void orc_scene_destroy(orc_scene *s) { delete s; }

int orc_surface_steps(const orc_scene *sc, const double od[6], int depth_iter, int max_steps, double *rec) {
    SurfaceIter it;
    it.init(sc, od, od + 3);
    int n = 0;
    auto put_surface = [&](double *r, const Surface &s) {
        r[3] = s.ip[0]; r[4] = s.ip[1]; r[5] = s.ip[2];
        r[6] = s.cube[0]; r[7] = s.cube[1]; r[8] = s.cube[2];
        r[9] = s.voxel[0]; r[10] = s.voxel[1]; r[11] = s.voxel[2];
        r[12] = s.resolution; r[13] = s.normal;
        r[14] = s.color[0]; r[15] = s.color[1]; r[16] = s.color[2]; r[17] = s.color[3];
    };
    const double nan = std::numeric_limits<double>::quiet_NaN();
    if (!depth_iter) {
        TraceStep ts{};
        while (n < max_steps && it.next(&ts)) {
            double *r = rec + 18 * n;
            for (int i = 0; i < 18; i++) r[i] = nan;
            r[0] = ts.kind;
            r[1] = ts.t_distance;
            if (ts.kind == TS_ENTER_SURFACE) put_surface(r, ts.surface);
            n++;
        }
    } else {
        DepthIter di;
        di.init(&it);
        DepthStep ds{};
        while (n < max_steps && di.next(&ds)) {
            double *r = rec + 18 * n;
            for (int i = 0; i < 18; i++) r[i] = nan;
            r[0] = ds.kind;
            if (ds.kind == DS_SPAN) {
                r[1] = ds.surface.t_distance;
                r[2] = ds.exit_t_distance;
                put_surface(r, ds.surface);
            } else if (ds.kind == DS_ENTER_BLOCK) {
                r[1] = ds.t_distance;
            }
            n++;
        }
    }
    return n;
}

int orc_trace_rays(const orc_scene *sc, const double (*od)[6], size_t n, const aicb_options *opt, int accum_mode,
                   float (*out_cb)[4], double *depth, aicb_hit *hit, uint32_t *steps, int32_t *text) {
    for (size_t i = 0; i < n; i++) {
        Accum acc;
        acc.init(accum_mode);
        Tracer tr;
        tr.sc = sc;
        tr.opt = opt;
        tr.acc = &acc;
        size_t c = tr.trace(od[i], od[i] + 3);
        if (out_cb) {
            out_cb[i][0] = acc.color.light[0];
            out_cb[i][1] = acc.color.light[1];
            out_cb[i][2] = acc.color.light[2];
            out_cb[i][3] = acc.color.transmittance;
        }
        if (depth) depth[i] = acc.depth;
        if (hit) hit[i] = acc.first_hit;
        if (steps) steps[i] = (uint32_t)c;
        if (text) text[i] = acc.text;
    }
    return 0;
}

static uint64_t render_rows_impl(const orc_scene *sc, const aicb_camera *cam, const aicb_options *opt,
                                 const std::vector<uint32_t> &rows, int accum_mode, int n_threads,
                                 uint8_t (*out_srgb8)[4], float (*out_cb)[4], double *depth, aicb_hit *hit,
                                 uint32_t *steps, int32_t *text) {
    if (n_threads <= 0) n_threads = orc_hardware_threads();
    // Work items are 64-pixel chunks of a row, handed out dynamically (the reference nests a
    // per-pixel parallel iterator inside a per-row one, renderer.rs:537-555).
    const uint32_t W = cam->fb_width;
    const uint32_t CH = 64;
    const size_t chunks_per_row = (W + CH - 1) / CH;
    const size_t n_items = rows.size() * chunks_per_row;
    std::atomic<size_t> next_item{0};
    std::atomic<uint64_t> total{0};
    auto worker = [&]() {
        uint64_t local = 0;
        for (;;) {
            size_t item = next_item.fetch_add(1);
            if (item >= n_items) break;
            size_t ri = item / chunks_per_row;
            uint32_t xb = (uint32_t)(item % chunks_per_row) * CH;
            uint32_t xe = xb + CH < W ? xb + CH : W;
            uint32_t y = rows[ri];
            for (uint32_t x = xb; x < xe; x++) {
                PixelOut po;
                local += trace_pixel(sc, *cam, *opt, accum_mode, x, y, &po);
                size_t o = ri * (size_t)W + x;
                if (out_srgb8) encode_srgb8(po.color, cam->exposure, opt->tone_mapping, opt->maximum_intensity, out_srgb8[o]);
                if (out_cb) {
                    out_cb[o][0] = po.color.light[0];
                    out_cb[o][1] = po.color.light[1];
                    out_cb[o][2] = po.color.light[2];
                    out_cb[o][3] = po.color.transmittance;
                }
                if (depth) depth[o] = po.depth;
                if (hit) hit[o] = po.hit;
                if (steps) steps[o] = po.steps;
                if (text) text[o] = po.text;
            }
        }
        total.fetch_add(local);
    };
    std::vector<std::thread> th;
    for (int i = 1; i < n_threads; i++) th.emplace_back(worker);
    worker();
    for (auto &t : th) t.join();
    return total.load();
}

uint64_t orc_render(const orc_scene *sc, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                    int accum_mode, int n_threads, uint8_t (*out_srgb8)[4], float (*out_cb)[4], double *depth,
                    aicb_hit *hit, uint32_t *steps, int32_t *text) {
    std::vector<uint32_t> rows;
    for (uint32_t y = 0; y < cam->fb_height; y++) {
        if (shard && shard->count > 1) {
            uint32_t sr = shard->strip_rows ? shard->strip_rows : 1;
            if ((y / sr) % shard->count != shard->index) continue;
        }
        rows.push_back(y);
    }
    return render_rows_impl(sc, cam, opt, rows, accum_mode, n_threads, out_srgb8, out_cb, depth, hit, steps, text);
}

uint64_t orc_render_rows(const orc_scene *sc, const aicb_camera *cam, const aicb_options *opt, uint32_t row_begin,
                         uint32_t row_end, int n_threads, uint8_t (*out_srgb8)[4], float (*out_cb)[4]) {
    std::vector<uint32_t> rows;
    for (uint32_t y = row_begin; y < row_end && y < cam->fb_height; y++) rows.push_back(y);
    return render_rows_impl(sc, cam, opt, rows, 0, n_threads, out_srgb8, out_cb, nullptr, nullptr, nullptr, nullptr);
}

uint64_t orc_render_rowlist(const orc_scene *sc, const aicb_camera *cam, const aicb_options *opt, const uint32_t *row_list,
                            size_t n_rows, int n_threads, uint8_t (*out_srgb8)[4], float (*out_cb)[4]) {
    std::vector<uint32_t> rows(row_list, row_list + n_rows);
    return render_rows_impl(sc, cam, opt, rows, 0, n_threads, out_srgb8, out_cb, nullptr, nullptr, nullptr, nullptr);
}

// draw_rgba through every layer (renderer.rs:282-308, 454-478); single-threaded (tests).
uint64_t orc_render_layers(const orc_scene *world, const aicb_camera *wcam, const aicb_options *wopt, const orc_scene *ui,
                           const aicb_camera *ucam, const aicb_options *uopt, const float *backdrop_rgba,
                           const float *no_world_rgba, uint8_t (*out_srgb8)[4], float (*out_cb)[4]) {
    const aicb_camera *lead_cam = world ? wcam : ucam;
    const aicb_options *lead_opt = world ? wopt : uopt;
    uint64_t total = 0;
    for (uint32_t y = 0; y < lead_cam->fb_height; y++)
        for (uint32_t x = 0; x < lead_cam->fb_width; x++) {
            ColorBuf c;
            total += trace_pixel_layers(world, wcam, wopt, ui, ucam, uopt, backdrop_rgba, no_world_rgba, x, y, &c);
            const size_t o = (size_t)y * lead_cam->fb_width + x;
            if (out_srgb8) encode_srgb8(c, lead_cam->exposure, lead_opt->tone_mapping, lead_opt->maximum_intensity, out_srgb8[o]);
            if (out_cb) { out_cb[o][0] = c.light[0]; out_cb[o][1] = c.light[1]; out_cb[o][2] = c.light[2]; out_cb[o][3] = c.transmittance; }
        }
    return total;
}

// Rgba::from(ColorBuf).to_srgb8() (ortho.rs:130) for a batch of accumulators: no exposure, no tone mapping.
void orc_colorbuf_to_srgb8(const float (*cb)[4], size_t n, uint8_t (*out)[4]) {
    for (size_t i = 0; i < n; i++) {
        ColorBuf c{{cb[i][0], cb[i][1], cb[i][2]}, cb[i][3]};
        encode_srgb8(c, 1.0f, AICB_TONE_CLAMP, std::numeric_limits<float>::infinity(), out[i]);
    }
}

void orc_pixel_ray(const aicb_camera *cam, uint32_t x, uint32_t y, int sample, double out[6]) {
    pixel_ray(*cam, x, y, sample, out, out + 3);
}

void orc_scene_block_sky(const orc_scene *s, uint8_t out[7][4]) {
    for (int f = 0; f < 6; f++) {
        out[f][0] = s->sky_faces[f].r; out[f][1] = s->sky_faces[f].g; out[f][2] = s->sky_faces[f].b; out[f][3] = s->sky_faces[f].status;
    }
    out[6][0] = s->sky_mean.r; out[6][1] = s->sky_mean.g; out[6][2] = s->sky_mean.b; out[6][3] = s->sky_mean.status;
}

// libm mode of the two per-ray transcendentals: 0 = platform powf/expf (what Rust's std calls), 1 = correctly rounded.
void orc_set_libm(int mode) { g_libm_mode.store(mode ? 1 : 0, std::memory_order_relaxed); }
int orc_get_libm(void) { return libm_mode(); }
float orc_powf(float x, float y, int mode) { return mode ? aicb::powf_exact(x, y) : std::pow(x, y); }
float orc_expf(float x, int mode) { return mode ? aicb::expf_exact(x) : std::exp(x); }

int orc_hardware_threads(void) {
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int)n : 1;
}
}
