// body.cu — bodies against a scene's cells on the device: step_one_body (all-is-cubes/src/physics/step.rs:316-976)
// with collide_along_ray, find_colliding_cubes, aab_raycast and nudge_on_ray (physics/collision.rs:100-249, 374-536),
// for a batch of bodies, on one context and on a device group.  One thread per body (body_step_kernel).  The Space
// level and the voxel level are two instantiations of one collide_along_ray template; the voxel level never recurses.
// A block's collision (Hard, None, mixed) is derived when it is placed and kept in BlockRec::flags; a voxel's is the
// AICB_VOXEL_NO_COLLISION bit of its palette entry's .w lane (block_words.cuh: voxel_flags).  A call reads the scene
// and writes only its results.
//
// Two sets of the reference are not stored:
//   - collide_along_ray's already_colliding set.  Its members are inserted only at the cast's first step (the Within
//     step at t = 0: no later step can report a Within contact on the Space level, and the voxel level at a later step
//     is a NotAlreadyColliding cast of its own).  So a contact is a member iff its cube lies in the first step's cubes
//     and, for a voxel contact, the first step's recursion into that cube (StopAt::Anything, the same ray) ended on the
//     same voxel at its own Within step: both are re-derived from the first step's box, exactly, for any box size.
//   - the ContactSet.  The caller's contact buffer holds its first max_contacts members; a contact past them is a
//     member iff an earlier move segment's cast reported it (one cast never reports a contact twice: it reports at its
//     first step and at the step it stops at, with different faces), which is re-derived by casting that segment again.
#include <cmath>
#include <vector>

#include "internal.h"

using namespace aicb;

namespace {

constexpr double POSITION_EPSILON = 1e-6 * 1e-6;            // physics/mod.rs:28
constexpr double VELOCITY_EPSILON_SQUARED = 1e-12;          // step.rs:301
constexpr double VELOCITY_MAGNITUDE_LIMIT = 1e4;            // step.rs:307
constexpr double VELOCITY_MAGNITUDE_LIMIT_SQUARED = VELOCITY_MAGNITUDE_LIMIT * VELOCITY_MAGNITUDE_LIMIT;
constexpr int32_t I32_MIN_ = INT32_MIN, I32_MAX_ = INT32_MAX;

struct BodyParams {
    DeviceScene scene;
    uint32_t wide_bricks;
    uint32_t max_contacts;
    double dt;
    double gravity[3];
    aicb_body *bodies;
    const double *edv;            // [n][3] or nullptr
    aicb_body_step_info *info;    // or nullptr
    aicb_contact *contacts;       // [n][max_contacts] or nullptr
    uint64_t n;
};

struct GAab {   // GridAab, exclusive upper
    int32_t lo[3], hi[3];
};
struct FAab {
    double lo[3], hi[3];
};
struct FRay {
    double o[3], d[3];
};
struct RayEnd {
    double t;
    aicb_contact c;
};

__device__ __forceinline__ int opposite(int f) { return f == AICB_FACE_WITHIN ? f : (f <= AICB_FACE_NZ ? f + 3 : f - 3); }
__device__ __forceinline__ int face_axis(int f) { return (f - 1) % 3; }
__device__ __forceinline__ double fco(const FAab &b, int f) {   // Aab::face_coordinate_outward
    return f >= AICB_FACE_PX ? b.hi[f - AICB_FACE_PX] : -b.lo[f - AICB_FACE_NX];
}
__device__ __forceinline__ bool finite3(const double *v) { return isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }

__device__ FAab translate(const FAab &b, const double v[3]) {
    FAab r;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        r.lo[a] = b.lo[a] + v[a];
        r.hi[a] = b.hi[a] + v[a];
    }
    return r;
}

// `f as i32`: saturating, NaN -> 0
__device__ __forceinline__ int32_t sat_i32(double v) {
    if (v != v) return 0;
    if (v <= -2147483648.0) return I32_MIN_;
    if (v >= 2147483647.0) return I32_MAX_;
    return (int32_t)v;
}
__device__ GAab round_up_to_grid(const FAab &b) {
    GAab g;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        g.lo[a] = sat_i32(floor(b.lo[a]));
        g.hi[a] = sat_i32(ceil(b.hi[a]));
    }
    return g;
}
__device__ __forceinline__ bool in_grid(const GAab &g, const int32_t c[3]) {
    return c[0] >= g.lo[0] && c[0] < g.hi[0] && c[1] >= g.lo[1] && c[1] < g.hi[1] && c[2] >= g.lo[2] && c[2] < g.hi[2];
}

// nudge_on_ray (collision.rs:498-536), in place on the segment.
__device__ void nudge_on_ray(const FAab &aab, FRay &seg, int face, double subdivision, bool backward) {
    if (seg.d[0] == 0.0 && seg.d[1] == 0.0 && seg.d[2] == 0.0) return;
    if (face == AICB_FACE_WITHIN) return;
    const int a = face_axis(face);
    const bool pos = face >= AICB_FACE_PX;
    const double e = seg.o[a] + seg.d[a];
    const double fc_scaled = (pos ? aab.hi[a] + e : -(aab.lo[a] + e)) * subdivision;
    const double penetration_depth = (fc_scaled - round(fc_scaled)) / subdivision;
    const double direction_projection = pos ? seg.d[a] : -seg.d[a];
    const double translation = (backward ? -POSITION_EPSILON : POSITION_EPSILON) - penetration_depth;
    const double k = 1.0 + translation / direction_projection;
#pragma unroll
    for (int i = 0; i < 3; i++) seg.d[i] = seg.d[i] * k;
}

// Raycaster::new(origin, direction) with no .within (raycast.rs:196-284, 497-819): an unbounded cast, whose bounds are
// Raycaster's maximum bounds.
struct Caster {
    double o[3], d[3], t_delta[3], t_max[3];
    int32_t step[3], cube[3];
    int face, state;   // state: 0 beginning, 1 in bounds, 2 ended
    double last_t;
    bool empty;        // State::EMPTY (bounds 0..0)
};

__device__ __forceinline__ int32_t signum_101(double x) { return (x == 0.0 || x != x) ? 0 : (signbit(x) ? -1 : 1); }

__device__ double scale_to_integer_step(double s, double ds) {
    if (ds == 0.0 && !(s != s)) return HUGE_VAL;
    if (ds < 0.0) {
        s = -s;
        ds = -ds;
    }
    double r = fmod(s, 1.0);
    if (r < 0.0) r = r + 1.0;
    return (1.0 - r) / ds;
}

__device__ void caster_init(Caster &c, const double o[3], const double d_in[3]) {
    double d[3] = {d_in[0], d_in[1], d_in[2]};
    if (!((fabs(d[0]) < 1e100) & (fabs(d[1]) < 1e100) & (fabs(d[2]) < 1e100))) d[0] = d[1] = d[2] = 0.0;
    c.state = 0;
    c.face = AICB_FACE_WITHIN;
    c.last_t = 0.0;
    bool ok = true;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        c.o[a] = o[a];
        c.d[a] = d[a];
        c.step[a] = signum_101(d[a]);
        c.t_delta[a] = 1.0 / fabs(d[a]);
        // Cube::containing, within the maximum bounds [I32_MIN + 1, I32_MAX - 1)
        ok &= (-2147483648.0 <= o[a]) & (o[a] < 2147483648.0);
    }
    if (ok) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            c.cube[a] = (int32_t)floor(o[a]);
            ok &= (c.cube[a] >= I32_MIN_ + 1) & (c.cube[a] < I32_MAX_ - 1);
        }
    }
    c.empty = !ok;
    if (!ok) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            c.o[a] = c.d[a] = 0.0;
            c.step[a] = 0;
            c.t_delta[a] = HUGE_VAL;
            c.cube[a] = 0;
            c.t_max[a] = 0.0;
        }
        return;
    }
#pragma unroll
    for (int a = 0; a < 3; a++) c.t_max[a] = scale_to_integer_step(o[a], d[a]);
}

// Raycaster::next: false when the cast has ended; else its step in `s`.
struct Step {
    int32_t cube[3];
    int face;
    double t;
};
__device__ bool caster_next(Caster &c, Step &s) {
    for (;;) {
        bool enter = false, exit_ = false;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const int32_t lo = c.empty ? 0 : I32_MIN_ + 1, hi = c.empty ? 0 : I32_MAX_ - 1;
            const bool low = c.cube[a] < lo, high = c.cube[a] >= hi;
            if (c.step[a] == 0) {
                enter |= low | high;
                exit_ |= low | high;
            } else if (c.step[a] < 0) {
                enter |= high;
                exit_ |= low;
            } else {
                enter |= low;
                exit_ |= high;
            }
        }
        const bool valid = (c.step[0] != 0 || c.step[1] != 0 || c.step[2] != 0) &&
                           !(c.t_max[0] != c.t_max[0] || c.t_max[1] != c.t_max[1] || c.t_max[2] != c.t_max[2]) &&
                           (isfinite(c.t_max[0]) || isfinite(c.t_max[1]) || isfinite(c.t_max[2]));
        if (c.state <= 1 && !enter && !exit_) {
#pragma unroll
            for (int a = 0; a < 3; a++) s.cube[a] = c.cube[a];
            s.face = c.face;
            s.t = c.last_t;
            if (!valid) {
                c.state = 2;
                return c.face == AICB_FACE_WITHIN;
            }
            int axis;
            if (c.t_max[0] < c.t_max[1]) axis = c.t_max[0] < c.t_max[2] ? 0 : 2;
            else axis = c.t_max[1] < c.t_max[2] ? 1 : 2;
            c.last_t = c.t_max[axis];
            const int64_t nc = (int64_t)c.cube[axis] + c.step[axis];
            if (nc >= (int64_t)I32_MIN_ && nc <= (int64_t)I32_MAX_) {
                c.cube[axis] = (int32_t)nc;
                c.t_max[axis] = c.t_max[axis] + c.t_delta[axis];
                c.face = c.step[axis] > 0 ? AICB_FACE_NX + axis : AICB_FACE_PX + axis;
            }
            c.state = 1;
            return true;
        } else if (c.state == 0 && enter && !exit_) {
            if (!valid) {
                c.state = 2;
                return false;
            }
            int axis;
            if (c.t_max[0] < c.t_max[1]) axis = c.t_max[0] < c.t_max[2] ? 0 : 2;
            else axis = c.t_max[1] < c.t_max[2] ? 1 : 2;
            c.last_t = c.t_max[axis];
            const int64_t nc = (int64_t)c.cube[axis] + c.step[axis];
            if (nc < (int64_t)I32_MIN_ || nc > (int64_t)I32_MAX_) return false;
            c.cube[axis] = (int32_t)nc;
            c.t_max[axis] = c.t_max[axis] + c.t_delta[axis];
            c.face = c.step[axis] > 0 ? AICB_FACE_NX + axis : AICB_FACE_PX + axis;
        } else if (c.state == 1 && !enter && exit_) {
            c.state = 2;
#pragma unroll
            for (int a = 0; a < 3; a++) s.cube[a] = c.cube[a];
            s.face = c.face;
            s.t = c.last_t;
            return true;   // include_exit
        } else {
            return false;
        }
    }
}

// aab_raycast (collision.rs:374-382)
__device__ void aab_raycast(Caster &c, const FAab &aab, const FRay &ray, bool reversed) {
    double o[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double v = reversed ? -ray.d[a] : ray.d[a];
        o[a] = ray.o[a] + (v >= 0.0 ? aab.hi[a] : aab.lo[a]);
    }
    caster_init(c, o, ray.d);
}

// ---- the scene --------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool in_scene(const DeviceScene &S, const int32_t c[3], uint32_t *idx) {
    const uint32_t dx = (uint32_t)c[0] - (uint32_t)S.lo[0], dy = (uint32_t)c[1] - (uint32_t)S.lo[1],
                   dz = (uint32_t)c[2] - (uint32_t)S.lo[2];
    if ((dx >= (uint32_t)S.size[0]) | (dy >= (uint32_t)S.size[1]) | (dz >= (uint32_t)S.size[2])) return false;
    *idx = (dx * (uint32_t)S.size[1] + dy) * (uint32_t)S.size[2] + dz;
    return true;
}
__device__ __forceinline__ uint32_t cell_id(const DeviceScene &S, uint32_t idx) {
    return S.wide_cells ? (__ldg((const uint32_t *)S.cells + idx) & 0xffffu)
                        : ((uint32_t)__ldg((const uint16_t *)S.cells + idx) & 0x3fffu);
}
// BLOCK_COLLISION_* of a block id (0: Hard)
__device__ __forceinline__ uint32_t block_collision(const DeviceScene &S, uint32_t id) {
    return __ldg(&S.blocks[id].flags) & (BLOCK_COLLISION_NONE | BLOCK_COLLISION_MIXED);
}

// The voxels of one mixed block (EvoxelsRef), and where its cube is.
struct Voxels {
    GAab vb;
    uint32_t base, pal_off, res;
    int32_t cube[3];
};

struct Body {
    double position[3], velocity[3];
    FAab box, occupying;
};

// ---- collide_along_ray ------------------------------------------------------------------------------------------
struct NoCallback {
    __device__ void operator()(const aicb_contact &) const {}
};

__device__ aicb_contact make_contact(int kind, const int32_t cube[3], int face) {
    aicb_contact c;
    memset(&c, 0, sizeof c);
    c.cube[0] = cube[0];
    c.cube[1] = cube[1];
    c.cube[2] = cube[2];
    c.kind = (uint8_t)kind;
    c.face = (uint8_t)face;
    return c;
}
__device__ __forceinline__ bool contact_eq(const aicb_contact &x, const aicb_contact &y) {
    return x.kind == y.kind && x.face == y.face && x.resolution == y.resolution && x.cube[0] == y.cube[0] &&
           x.cube[1] == y.cube[1] && x.cube[2] == y.cube[2] && x.voxel[0] == y.voxel[0] && x.voxel[1] == y.voxel[1] &&
           x.voxel[2] == y.voxel[2];
}

// collide_along_ray (collision.rs:100-226) on level L: the Space (`V` unused) or the voxels `V` of one mixed block,
// which report nothing.  Returns true with *out for a collision.
template <bool VOXEL, class CB>
__device__ bool collide(const BodyParams &P, const Voxels &V, const FRay &ray, const FAab &aab, CB &callback,
                        bool not_already, RayEnd *out);

// CollisionSpace::recurse (collision.rs:302-324) for cube `c` of block record `rec`
__device__ bool recurse(const BodyParams &P, const int32_t c[3], const BlockRec &rec, const FRay &ray, const FAab &aab,
                        bool not_already, RayEnd *out) {
    Voxels V;
    V.res = rec.kind_res >> 8;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        V.vb.lo[a] = rec.vlo[a];
        V.vb.hi[a] = rec.vlo[a] + (int32_t)rec.vsize[a];
        V.cube[a] = c[a];
    }
    V.base = rec.brick_off;
    V.pal_off = rec.pal_off;
    const double res = (double)V.res;
    FRay vray;
    FAab vaab;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        vray.o[a] = (ray.o[a] + -(double)c[a]) * res;
        vray.d[a] = ray.d[a] * res;
        vaab.lo[a] = aab.lo[a] * res;
        vaab.hi[a] = aab.hi[a] * res;
    }
    NoCallback none;
    if (!collide<true>(P, V, vray, vaab, none, not_already, out)) return false;
    // wrap_as_voxel (collision.rs:48-76)
#pragma unroll
    for (int a = 0; a < 3; a++) {
        out->c.voxel[a] = out->c.cube[a];
        out->c.cube[a] = c[a];
    }
    out->c.kind = AICB_CONTACT_VOXEL;
    out->c.resolution = (uint8_t)V.res;
    return true;
}

__device__ __forceinline__ BlockRec load_rec(const DeviceScene &S, uint32_t id) {
    BlockRec r;
    const uint4 *bp = reinterpret_cast<const uint4 *>(S.blocks + id);
    const uint4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
    memcpy(&r, &b0, 16);
    memcpy(reinterpret_cast<char *>(&r) + 16, &b1, 16);
    return r;
}

template <bool VOXEL, class CB>
__device__ bool collide(const BodyParams &P, const Voxels &V, const FRay &ray, const FAab &aab, CB &callback,
                        bool not_already, RayEnd *out) {
    const DeviceScene &S = P.scene;
    GAab bounds;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        bounds.lo[a] = VOXEL ? V.vb.lo[a] : S.lo[a];
        bounds.hi[a] = VOXEL ? V.vb.hi[a] : S.lo[a] + S.size[a];
    }
    GAab first;                  // the first step's cubes: already_colliding's members lie in them
    bool have_first = false;
    bool first_step = true;
    Caster cs;
    aab_raycast(cs, aab, ray, false);
    Step st;
    while (caster_next(cs, st)) {
        const bool is_first = first_step;
        first_step = false;
        FRay seg = ray;
#pragma unroll
        for (int a = 0; a < 3; a++) seg.d[a] = ray.d[a] * st.t;
        nudge_on_ray(aab, seg, opposite(st.face), 1.0, false);
        double e[3];
#pragma unroll
        for (int a = 0; a < 3; a++) e[a] = seg.o[a] + seg.d[a];
        if (st.t >= 1.0) break;
        const GAab g = round_up_to_grid(translate(aab, e));
        GAab pib;
        bool nonempty = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            pib.lo[a] = max(g.lo[a], bounds.lo[a]);
            pib.hi[a] = min(g.hi[a], bounds.hi[a]);
            nonempty &= pib.hi[a] > pib.lo[a];
        }
        if (!nonempty) continue;
        if (is_first) {
            first = pib;
            have_first = true;
        }
        bool have = false;
        RayEnd hit;
        hit.t = 0.0;
        int32_t c[3];
        for (c[0] = pib.lo[0]; c[0] < pib.hi[0]; c[0]++)
            for (c[1] = pib.lo[1]; c[1] < pib.hi[1]; c[1]++)
                for (c[2] = pib.lo[2]; c[2] < pib.hi[2]; c[2]++) {
                    RayEnd found;
                    if constexpr (VOXEL) {
                        const uint32_t vi = ((uint32_t)(c[0] - V.vb.lo[0]) * (uint32_t)(V.vb.hi[1] - V.vb.lo[1]) +
                                             (uint32_t)(c[1] - V.vb.lo[1])) *
                                                (uint32_t)(V.vb.hi[2] - V.vb.lo[2]) +
                                            (uint32_t)(c[2] - V.vb.lo[2]);
                        const uint32_t w = P.wide_bricks ? __ldg((const uint32_t *)S.bricks + V.base + vi) >> 16
                                                         : (uint32_t)(__ldg(S.bricks + V.base + vi) & 0x7fffu);
                        const uint32_t fl = __float_as_uint(__ldg(&S.palette[2 * (size_t)(V.pal_off + w) + 1].w));
                        if (fl & AICB_VOXEL_NO_COLLISION) continue;
                        found.t = st.t;
                        found.c = make_contact(AICB_CONTACT_BLOCK, c, st.face);
                    } else {
                        uint32_t idx = 0;
                        in_scene(S, c, &idx);
                        const uint32_t id = cell_id(S, idx);
                        const uint32_t k = block_collision(S, id);
                        if (k == BLOCK_COLLISION_NONE) continue;
                        if (k == 0) {
                            found.t = st.t;
                            found.c = make_contact(AICB_CONTACT_BLOCK, c, st.face);
                        } else {
                            const BlockRec rec = load_rec(S, id);
                            if (!recurse(P, c, rec, ray, aab, not_already && st.face != AICB_FACE_WITHIN, &found))
                                continue;
                        }
                    }
                    if (not_already) {
                        if (found.c.face == AICB_FACE_WITHIN) {
                            callback(found.c);
                            continue;
                        }
                        // already_colliding.contains(contact.without_normal()), re-derived from the first step
                        if (have_first && !is_first && in_grid(first, c)) {
                            bool member = true;
                            if constexpr (!VOXEL) {
                                if (found.c.kind == AICB_CONTACT_VOXEL) {
                                    uint32_t idx = 0;
                                    in_scene(S, c, &idx);
                                    RayEnd w;
                                    member = recurse(P, c, load_rec(S, cell_id(S, idx)), ray, aab, false, &w) &&
                                             w.c.face == AICB_FACE_WITHIN && w.c.voxel[0] == found.c.voxel[0] &&
                                             w.c.voxel[1] == found.c.voxel[1] && w.c.voxel[2] == found.c.voxel[2];
                                }
                            }
                            if (member) continue;
                        }
                    }
                    callback(found.c);
                    if (!have || found.t < hit.t) {
                        hit = found;
                        have = true;
                    }
                }
        if (have) {
            *out = hit;
            return true;
        }
    }
    return false;
}

__device__ FRay zero_ray() {
    FRay r;
    for (int a = 0; a < 3; a++) r.o[a] = r.d[a] = 0.0;
    return r;
}

// Contact::aab (contact.rs:59-76)
__device__ FAab contact_aab(const aicb_contact &c) {
    FAab b;
    if (c.kind == AICB_CONTACT_BLOCK) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            b.lo[a] = (double)c.cube[a];
            b.hi[a] = (double)c.cube[a] + 1.0;
        }
        return b;
    }
    const double r = 1.0 / (double)c.resolution;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        b.lo[a] = (double)c.voxel[a] * r + (double)c.cube[a];
        b.hi[a] = ((double)c.voxel[a] + 1.0) * r + (double)c.cube[a];
    }
    return b;
}

__device__ __forceinline__ double volume(const FAab &b) {
    const double v = (b.hi[0] - b.lo[0]) * (b.hi[1] - b.lo[1]) * (b.hi[2] - b.lo[2]);
    return v == 0.0 ? 0.0 : v;
}

__device__ void set_position(Body &b, const double p[3]) {   // Body::set_position (body.rs:197-207)
    if (!finite3(p)) return;
#pragma unroll
    for (int a = 0; a < 3; a++) b.position[a] = p[a];
    b.occupying = translate(b.box, b.position);
}

// attempt_push_out (step.rs:697-741)
__device__ bool attempt_push_out(const BodyParams &P, const Body &body, const double dir[3], double np[3], double *dist) {
    const DeviceScene &S = P.scene;
    FRay ray;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        ray.o[a] = body.position[a];
        ray.d[a] = dir[a];
    }
    Caster cs;
    aab_raycast(cs, body.box, ray, true);
    Step st;
    while (caster_next(cs, st)) {
        FRay seg = ray;
#pragma unroll
        for (int a = 0; a < 3; a++) seg.d[a] = ray.d[a] * st.t;
        nudge_on_ray(body.box, seg, st.face, 1.0, true);
        double e[3];
#pragma unroll
        for (int a = 0; a < 3; a++) e[a] = seg.o[a] + seg.d[a];
        const GAab g = round_up_to_grid(translate(body.box, e));
        bool clear = true;
        int32_t c[3];
        for (c[0] = g.lo[0]; clear && c[0] < g.hi[0]; c[0]++)
            for (c[1] = g.lo[1]; clear && c[1] < g.hi[1]; c[1]++)
                for (c[2] = g.lo[2]; clear && c[2] < g.hi[2]; c[2]++) {
                    uint32_t idx;
                    if (in_scene(S, c, &idx) && block_collision(S, cell_id(S, idx)) == 0) clear = false;
                }
        if (!clear) continue;
#pragma unroll
        for (int a = 0; a < 3; a++) np[a] = e[a];
        const double len = sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        const double d = st.t * len;
        if (d != d) return false;
        *dist = d;
        return true;
    }
    return false;
}

struct AnyContact {
    bool any = false;
    __device__ void operator()(const aicb_contact &) { any = true; }
};
struct LastContact {
    bool any = false;
    aicb_contact last;
    __device__ void operator()(const aicb_contact &c) {
        any = true;
        last = c;
    }
};

// push_out (step.rs:662-693)
__device__ bool push_out(const BodyParams &P, Body &body, double out[3]) {
    AnyContact any;
    RayEnd unused;
    Voxels none;
    collide<false>(P, none, zero_ray(), body.occupying, any, false, &unused);
    if (!any.any) return false;
    bool have = false;
    double best_pos[3] = {0, 0, 0}, best = 0.0;
    for (int k = 0; k < 27; k++) {
        double dir[3] = {(double)(k / 9 - 1), (double)(k / 3 % 3 - 1), (double)(k % 3 - 1)};
        if (k == 13)
            for (int a = 0; a < 3; a++) dir[a] = -body.velocity[a];
        double p[3], d;
        if (!attempt_push_out(P, body, dir, p, &d)) continue;
        if (!have || d < best) {
            have = true;
            best = d;
            for (int a = 0; a < 3; a++) best_pos[a] = p[a];
        }
    }
    if (!have) return false;
    double old[3];
    for (int a = 0; a < 3; a++) old[a] = body.position[a];
    set_position(body, best_pos);
    for (int a = 0; a < 3; a++) out[a] = best_pos[a] - old[a];
    return true;
}

// How many shrinks crush_if_colliding may take for a box {lo, hi} before it counts as not finishing
// (AICB_BODY_CRUSH_UNFINISHED).  Each shrink that changes the box moves one face inward onto a face of a cube or voxel
// (up to one rounding), and every voxel face lies on a plane k / 128, so a crush that finishes crosses at most the
// planes of resolution 128 inside the box on each of its six faces; four times that, plus 64, leaves room for
// rounding.  A shrink that changes nothing is the reference's endless loop and is caught at once.
__device__ double crush_limit(const double lo[3], const double hi[3]) {
    double planes = 0.0;
    for (int a = 0; a < 3; a++) planes = planes + 2.0 * (ceil((hi[a] - lo[a]) * 128.0) + 1.0);
    const double limit = 4.0 * planes + 64.0;
    return limit < 1e9 ? limit : 1e9;
}

// crush_if_colliding (step.rs:747-798); a panic status or 0
__device__ uint32_t crush_if_colliding(const BodyParams &P, Body &body, double info[6]) {
    const FAab original = body.occupying;
    const double limit = crush_limit(original.lo, original.hi);
    for (double iter = 0.0;; iter = iter + 1.0) {
        if (iter >= limit) return AICB_BODY_CRUSH_UNFINISHED;
        LastContact lc;
        RayEnd unused;
        Voxels none;
        collide<false>(P, none, zero_ray(), body.occupying, lc, false, &unused);
        if (!lc.any) break;
        const FAab ca = contact_aab(lc.last);
        int least_face = -1;
        double least = 0.0;
        for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) {
            const double d = fco(body.occupying, f) + fco(ca, opposite(f));
            if (d >= 0.0 && (least_face < 0 || d < least)) {
                least_face = f;
                least = d;
            }
        }
        if (least_face < 0) return AICB_BODY_NO_PENETRATION;
        FAab shrunk;
        bool ok = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            shrunk.lo[a] = body.occupying.lo[a] - (least_face == AICB_FACE_NX + a ? -least : 0.0);
            shrunk.hi[a] = body.occupying.hi[a] + (least_face == AICB_FACE_PX + a ? -least : 0.0);
            ok &= shrunk.lo[a] <= shrunk.hi[a];
        }
        if (!ok) break;
        bool same = true;
#pragma unroll
        for (int a = 0; a < 3; a++) same &= shrunk.lo[a] == body.occupying.lo[a] && shrunk.hi[a] == body.occupying.hi[a];
        if (same) return AICB_BODY_CRUSH_UNFINISHED;   // the same box finds the same contact: the reference loops forever
        body.occupying = shrunk;
    }
    for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) info[f - 1] = fco(original, f) - fco(body.occupying, f);
    return 0;
}

// uncrush's per-contact reduction (step.rs:848-898)
struct UncrushContacts {
    const Body *body;
    const FAab *single;
    double *clear;   // [7], by Face7
    bool collided = false;
    __device__ void operator()(const aicb_contact &contact) {
        collided = true;
        const FAab ca = contact_aab(contact);
        for (int a = 0; a < 3; a++) {
            const FAab &s = single[a];
            bool inter = true;
            for (int i = 0; i < 3; i++) inter &= fmax(s.lo[i], ca.lo[i]) <= fmin(s.hi[i], ca.hi[i]);
            if (!inter) continue;
            const double lb = ca.lo[a], ub = ca.hi[a], p = body->position[a];
            int face;
            if (ub <= p) face = AICB_FACE_NX + a;
            else if (lb >= p) face = AICB_FACE_PX + a;
            else {
                clear[AICB_FACE_NX + a] = fco(body->occupying, AICB_FACE_NX + a);
                clear[AICB_FACE_PX + a] = fco(body->occupying, AICB_FACE_PX + a);
                continue;
            }
            clear[face] = fmin(clear[face], -fco(ca, opposite(face)));
        }
    }
};

// uncrush (step.rs:806-976)
__device__ uint8_t uncrush(const BodyParams &P, Body &body, uint8_t axes[3]) {
    const FAab full = translate(body.box, body.position);
    bool eq = true;
    for (int a = 0; a < 3; a++) eq &= full.lo[a] == body.occupying.lo[a] && full.hi[a] == body.occupying.hi[a];
    if (eq) return AICB_UNCRUSH_NOT_NEEDED;
    int n_axes = 0;
    for (int attempt = 0; attempt < 3; attempt++) {
        const double current_volume = volume(body.occupying);
        FAab single[3];
        for (int a = 0; a < 3; a++) {
            single[a] = body.occupying;
            single[a].lo[a] = full.lo[a];
            single[a].hi[a] = full.hi[a];
        }
        double clear[7];
        clear[0] = 0.0;
        for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) clear[f] = fco(full, f);
        UncrushContacts u{&body, single, clear};
        RayEnd unused;
        Voxels none;
        collide<false>(P, none, zero_ray(), full, u, false, &unused);
        if (!u.collided) {
            body.occupying = full;
            return AICB_UNCRUSH_COMPLETE;
        }
        int best_axis = -1;
        double best_volume = 0.0;
        FAab best_aab = body.occupying;
        for (int a = 0; a < 3; a++) {
            const double lo = -clear[AICB_FACE_NX + a], hi = clear[AICB_FACE_PX + a];
            if (!(lo <= hi)) continue;
            FAab e = body.occupying;
            e.lo[a] = lo;
            e.hi[a] = hi;
            bool inside = true;
            for (int i = 0; i < 3; i++) inside &= e.lo[i] <= body.position[i] && body.position[i] <= e.hi[i];
            if (!inside) continue;
            double v = volume(e) - current_volume;
            v = v > 0.0 ? v : 0.0;
            if (!(v > 0.0)) continue;
            if (best_axis < 0 || v >= best_volume) {
                best_axis = a;
                best_volume = v;
                best_aab = e;
            }
        }
        if (best_axis < 0) break;
        body.occupying = best_aab;
        axes[n_axes++] = (uint8_t)best_axis;
    }
    return n_axes ? AICB_UNCRUSH_PARTIAL : AICB_UNCRUSH_NOT_POSSIBLE;
}

// The ContactSet of one body: the caller's buffer holds its first members; membership past them is re-derived from
// the earlier segments' casts (see the top of this file).
struct MatchContact {
    aicb_contact want;
    bool found = false;
    __device__ void operator()(const aicb_contact &c) { found |= contact_eq(c, want); }
};

struct Segments {
    FRay ray[3];
    int n = 0;   // segments cast before the current one
};

struct StepContacts {
    const BodyParams *P;
    const Body *body;
    const Segments *segs;
    aicb_contact *buf;   // or nullptr
    uint32_t cap;
    uint32_t n = 0;      // the set's size
    aicb_contact already;
    __device__ void operator()(const aicb_contact &c) {
        if (c.face == AICB_FACE_WITHIN) already = c;
        const uint32_t stored = n < cap ? n : cap;
        for (uint32_t k = 0; k < stored; k++)
            if (contact_eq(buf[k], c)) return;
        if (n >= cap) {
            for (int i = 0; i < segs->n; i++) {
                MatchContact m;
                m.want = c;
                RayEnd unused;
                Voxels none;
                collide<false>(*P, none, segs->ray[i], body->box, m, true, &unused);
                if (m.found) return;
            }
        }
        if (n < cap) buf[n] = c;
        n++;
    }
};

__global__ void __launch_bounds__(128) body_step_kernel(const __grid_constant__ BodyParams P) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    aicb_body ab = P.bodies[i];
    aicb_body_step_info info;
    memset(&info, 0, sizeof info);
    info.uncrush_axes[0] = info.uncrush_axes[1] = info.uncrush_axes[2] = AICB_AXIS_NONE;
    double edv[3] = {0.0, 0.0, 0.0};
    if (P.edv)
        for (int a = 0; a < 3; a++) edv[a] = P.edv[3 * i + a];
    // a body the reference could not hold
    bool valid = finite3(ab.position) && finite3(ab.velocity) && finite3(edv);
    for (int k = 0; k < 6; k++) valid &= isfinite(ab.collision_box[k]) && isfinite(ab.occupying[k]);
    for (int a = 0; a < 3; a++)
        valid &= ab.collision_box[a] < ab.collision_box[3 + a] && ab.occupying[a] <= ab.occupying[3 + a];
    if (!valid) {
        info.status = AICB_BODY_INVALID;
        if (P.info) P.info[i] = info;
        return;
    }
    Body body;
    for (int a = 0; a < 3; a++) {
        body.position[a] = ab.position[a];
        body.velocity[a] = ab.velocity[a];
        body.box.lo[a] = ab.collision_box[a];
        body.box.hi[a] = ab.collision_box[3 + a];
        body.occupying.lo[a] = ab.occupying[a];
        body.occupying.hi[a] = ab.occupying[3 + a];
    }
    const bool space = !ab.noclip;
    Segments segs;
    StepContacts set{&P, &body, &segs, P.contacts ? P.contacts + i * P.max_contacts : nullptr,
                     P.contacts ? P.max_contacts : 0u};
    set.already.kind = AICB_CONTACT_NONE;
    uint32_t panic = 0;
    double v0[3];
    for (int a = 0; a < 3; a++) {
        v0[a] = body.velocity[a];
        body.velocity[a] = body.velocity[a] + edv[a];
    }
    const double p2 = body.position[0] * body.position[0] + body.position[1] * body.position[1] +
                      body.position[2] * body.position[2];
    if (isfinite(p2)) {
        if (!ab.flying && space)
            for (int a = 0; a < 3; a++) body.velocity[a] = body.velocity[a] + P.gravity[a] * P.dt;
        if (space) {
            info.uncrush = uncrush(P, body, info.uncrush_axes);
            info.has_push_out = push_out(P, body, info.push_out);
            panic = crush_if_colliding(P, body, info.initial_crush);
        }
        const double v2 = body.velocity[0] * body.velocity[0] + body.velocity[1] * body.velocity[1] +
                          body.velocity[2] * body.velocity[2];
        bool move = true;
        if (!isfinite(v2)) {
            body.velocity[0] = body.velocity[1] = body.velocity[2] = 0.0;
        } else if (v2 <= VELOCITY_EPSILON_SQUARED) {
            info.quiescent = 1;
            move = false;
        } else if (v2 > VELOCITY_MAGNITUDE_LIMIT_SQUARED) {
            const double k = VELOCITY_MAGNITUDE_LIMIT / sqrt(v2);
            for (int a = 0; a < 3; a++) body.velocity[a] = body.velocity[a] * k;
        }
        if (move && !panic) {
            double delta[3];
            for (int a = 0; a < 3; a++) delta[a] = body.velocity[a] * P.dt;
            if (space) {
                while (!(delta[0] == 0.0 && delta[1] == 0.0 && delta[2] == 0.0)) {
                    if (segs.n >= 3) {
                        panic = AICB_BODY_SLIDING_UNFINISHED;
                        break;
                    }
                    // collide_and_advance (step.rs:594-659)
                    FRay movement;
                    for (int a = 0; a < 3; a++) {
                        movement.o[a] = body.position[a];
                        movement.d[a] = delta[a];
                    }
                    RayEnd hit;
                    Voxels none;
                    aicb_move_segment &ms = info.move_segments[segs.n];
                    const bool stopped = collide<false>(P, none, movement, body.box, set, true, &hit);
                    segs.ray[segs.n++] = movement;
                    if (stopped) {
                        const int face = hit.c.face, axis = face_axis(face);
                        FRay motion = movement;
                        for (int a = 0; a < 3; a++) motion.d[a] = movement.d[a] * hit.t;
                        nudge_on_ray(body.box, motion, opposite(face),
                                     hit.c.kind == AICB_CONTACT_VOXEL ? (double)hit.c.resolution : 1.0, true);
                        double np[3];
                        for (int a = 0; a < 3; a++) np[a] = body.position[a] + motion.d[a];
                        set_position(body, np);
                        for (int a = 0; a < 3; a++) {
                            delta[a] = delta[a] - motion.d[a];
                            ms.delta_position[a] = motion.d[a];
                        }
                        delta[axis] = 0.0;
                        body.velocity[axis] = 0.0;
                        ms.stopped_by = hit.c;
                    } else {
                        double np[3];
                        for (int a = 0; a < 3; a++) np[a] = body.position[a] + delta[a];
                        set_position(body, np);
                        for (int a = 0; a < 3; a++) {
                            ms.delta_position[a] = delta[a];
                            delta[a] = 0.0;
                        }
                    }
                }
            } else {
                double np[3];
                for (int a = 0; a < 3; a++) np[a] = body.position[a] + delta[a];
                set_position(body, np);
                for (int a = 0; a < 3; a++) info.move_segments[0].delta_position[a] = delta[a];
            }
        }
        for (int a = 0; a < 3; a++) info.delta_v[a] = body.velocity[a] - v0[a];
    }
    if (panic) {
        memset(&info, 0, sizeof info);
        info.status = panic;
        if (P.info) P.info[i] = info;
        return;
    }
    info.already_colliding = set.already;
    info.n_contacts = set.n;
    if (set.n > P.max_contacts) info.status |= AICB_BODY_CONTACTS_TRUNCATED;
    for (int a = 0; a < 3; a++) {
        ab.position[a] = body.position[a];
        ab.velocity[a] = body.velocity[a];
        ab.occupying[a] = body.occupying.lo[a];
        ab.occupying[3 + a] = body.occupying.hi[a];
    }
    P.bodies[i] = ab;
    if (P.info) P.info[i] = info;
}

struct StepArgs {
    double dt;
    const double *gravity;
    uint32_t max_contacts;
};

aicb_status check_scalars(const StepArgs &a) {
    if (!(a.dt > 0.0 && a.dt <= 1.0)) return aicb_fail(AICB_ERR_INVALID, "dt must be finite and in (0, 1]");
    if (!a.gravity || !std::isfinite(a.gravity[0]) || !std::isfinite(a.gravity[1]) || !std::isfinite(a.gravity[2]))
        return aicb_fail(AICB_ERR_INVALID, "gravity must be finite");
    return AICB_OK;
}

// The batch (in device 0's memory) in ranges of whole warps, one per listed context, as cursor.cu issues its queries.
aicb_status issue_step(Replicas r, const StepArgs &a, aicb_body *bodies, const double *edv, aicb_body_step_info *info,
                       aicb_contact *contacts, size_t n) {
    const std::vector<WarpRange> ranges = warp_ranges(n, r.n);
    TRY(fan_out(r.ctx, ranges.size()));
    for (size_t i = 0; i < ranges.size(); i++) {
        const size_t begin = ranges[i].begin, count = ranges[i].count;
        if (count == 0) continue;
        BodyParams P;
        memset(&P, 0, sizeof P);
        P.scene = r.scene[i]->ds;
        P.wide_bricks = r.scene[i]->host->wide_bricks ? 1u : 0u;
        P.max_contacts = a.max_contacts;
        P.dt = a.dt;
        for (int k = 0; k < 3; k++) P.gravity[k] = a.gravity[k];
        P.bodies = bodies + begin;
        P.edv = edv ? edv + 3 * begin : nullptr;
        P.info = info ? info + begin : nullptr;
        P.contacts = contacts ? contacts + begin * a.max_contacts : nullptr;
        P.n = count;
        CU(cudaSetDevice(r.ctx[i]->device));
        body_step_kernel<<<(unsigned)((count + 127) / 128), 128, 0, r.ctx[i]->stream.get()>>>(P);
        CU(cudaGetLastError());
    }
    return fan_in(r.ctx, ranges.size());
}

bool host_body_valid(const aicb_body &b, const double *edv) {
    auto fin = [](const double *v, int k) {
        for (int i = 0; i < k; i++)
            if (!std::isfinite(v[i])) return false;
        return true;
    };
    if (!fin(b.position, 3) || !fin(b.velocity, 3) || (edv && !fin(edv, 3)) || !fin(b.collision_box, 6) ||
        !fin(b.occupying, 6))
        return false;
    for (int a = 0; a < 3; a++)
        if (!(b.collision_box[a] < b.collision_box[3 + a]) || !(b.occupying[a] <= b.occupying[3 + a])) return false;
    return true;
}

// The host form: the bodies staged in device 0's d_bodies, the results copied back once every part is done.
aicb_status step_host(Replicas r, aicb_body *bodies, const double (*edv)[3], size_t n, const StepArgs &a,
                      aicb_body_step_info *info, aicb_contact *contacts) {
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n && !bodies) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_scalars(a));
    for (size_t i = 0; i < n; i++)
        if (!host_body_valid(bodies[i], edv ? edv[i] : nullptr))
            return aicb_fail(AICB_ERR_INVALID, "a body is not finite, or its collision box is empty or inverted, or "
                                               "its occupying box inverted");
    if (n == 0) return AICB_OK;
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t n_contacts = contacts ? n * (size_t)a.max_contacts : 0;
    const size_t body_at = 0, edv_at = up(n * sizeof(aicb_body)), info_at = edv_at + (edv ? up(n * 24) : 0),
                 con_at = info_at + (info ? up(n * sizeof(aicb_body_step_info)) : 0);
    TRY(c0->d_bodies.ensure(con_at + n_contacts * sizeof(aicb_contact)));
    char *base = c0->d_bodies.get<char>();
    cudaStream_t s = c0->stream.get();
    CU(cudaMemcpyAsync(base + body_at, bodies, n * sizeof(aicb_body), cudaMemcpyHostToDevice, s));
    if (edv) CU(cudaMemcpyAsync(base + edv_at, edv, n * 24, cudaMemcpyHostToDevice, s));
    TRY(issue_step(r, a, reinterpret_cast<aicb_body *>(base + body_at),
                   edv ? reinterpret_cast<const double *>(base + edv_at) : nullptr,
                   info ? reinterpret_cast<aicb_body_step_info *>(base + info_at) : nullptr,
                   contacts ? reinterpret_cast<aicb_contact *>(base + con_at) : nullptr, n));
    CU(cudaMemcpyAsync(bodies, base + body_at, n * sizeof(aicb_body), cudaMemcpyDeviceToHost, s));
    if (info) CU(cudaMemcpyAsync(info, base + info_at, n * sizeof(aicb_body_step_info), cudaMemcpyDeviceToHost, s));
    if (n_contacts)
        CU(cudaMemcpyAsync(contacts, base + con_at, n_contacts * sizeof(aicb_contact), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return AICB_OK;
}

aicb_status step_device(Replicas r, aicb_body *bodies, const double (*edv)[3], size_t n, const StepArgs &a,
                        aicb_body_step_info *info, aicb_contact *contacts, cudaStream_t caller) {
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    TRY(check_scalars(a));
    if (n == 0) return AICB_OK;
    if (!bodies) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_device_pointer(bodies, c0->device, false, 8, "bodies"));
    if (edv) TRY(check_device_pointer(edv, c0->device, false, 8, "external_delta_v"));
    if (info) TRY(check_device_pointer(info, c0->device, false, 8, "info"));
    if (contacts && a.max_contacts) TRY(check_device_pointer(contacts, c0->device, false, 4, "contacts"));
    TRY(join_caller(r.ctx, r.n, caller));
    TRY(issue_step(r, a, bodies, edv ? &edv[0][0] : nullptr, info, a.max_contacts ? contacts : nullptr, n));
    if (r.n > 1) CU(cudaStreamSynchronize(c0->stream.get()));   // a group call returns with its output final
    return release_caller(c0, caller);
}

}  // namespace

extern "C" {

aicb_status aicb_step_bodies(aicb_scene *s, aicb_body *bodies, const double (*edv)[3], size_t n, double dt,
                             const double gravity[3], aicb_body_step_info *info, aicb_contact *contacts,
                             uint32_t max_contacts) {
    const StepArgs a{dt, gravity, max_contacts};
    return on_scene(s, [&](Replicas r) { return step_host(r, bodies, edv, n, a, info, contacts); });
}

aicb_status aicb_step_bodies_device(aicb_scene *s, aicb_body *bodies, const double (*edv)[3], size_t n, double dt,
                                    const double gravity[3], aicb_body_step_info *info, aicb_contact *contacts,
                                    uint32_t max_contacts, void *stream) {
    const StepArgs a{dt, gravity, max_contacts};
    return on_scene(s, [&](Replicas r) {
        return step_device(r, bodies, edv, n, a, info, contacts, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_step_bodies(aicb_group_scene *gs, aicb_body *bodies, const double (*edv)[3], size_t n,
                                   double dt, const double gravity[3], aicb_body_step_info *info,
                                   aicb_contact *contacts, uint32_t max_contacts) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    const StepArgs a{dt, gravity, max_contacts};
    return step_host(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, bodies, edv, n, a, info,
                     contacts);
}

aicb_status aicb_group_step_bodies_device(aicb_group_scene *gs, aicb_body *bodies, const double (*edv)[3], size_t n,
                                          double dt, const double gravity[3], aicb_body_step_info *info,
                                          aicb_contact *contacts, uint32_t max_contacts, void *stream) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    const StepArgs a{dt, gravity, max_contacts};
    return step_device(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, bodies, edv, n, a, info,
                       contacts, (cudaStream_t)stream);
}

}  // extern "C"
