// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// CPU restatement of step_one_body (all-is-cubes/src/physics/step.rs:316-976) and the collision functions it calls
// (physics/collision.rs:100-249, 374-536), built on the raytracer oracle's Raycaster (Raycaster::new without .within:
// Ray::cast, raycast.rs:196-202) and its scene (../oracle/aic_oracle.cpp, compiled into this library a second time and
// changed in nothing).  The raytracer oracle's scene does not keep collision, so each scene here keeps beside it every
// block's uniform_collision (derived as compute_derived derives it, block/eval/derived.rs:85-104, 159-190) and reads its
// voxels' AICB_VOXEL_NO_COLLISION flags from the palettes the scene keeps.
//
// The ContactSet (a hash set in the reference) is kept in first-insertion order; the per-call already_colliding set
// of collide_along_ray is an exact set.
//
// Parity pinning: tests/test_oracle_body_step.py runs the known answers of physics/tests.rs, step.rs:986-1087 and
// collision.rs:554-723.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_body {
using namespace orc;

enum Collision : uint8_t { HARD = 0, NONE = 1, MIXED = 2 };   // Some(Hard), Some(None), None (recurse)

static const double POSITION_EPSILON = 1e-6 * 1e-6;           // physics/mod.rs:28
static const double VELOCITY_EPSILON_SQUARED = 1e-12;         // step.rs:301
static const double VELOCITY_MAGNITUDE_LIMIT = 1e4;           // step.rs:307
static const double VELOCITY_MAGNITUDE_LIMIT_SQUARED = VELOCITY_MAGNITUDE_LIMIT * VELOCITY_MAGNITUDE_LIMIT;

struct Scene {
    orc_scene *s = nullptr;
    std::vector<uint8_t> collision;   // per block id: uniform_collision
};

static Collision voxel_collision(const aicb_voxel &v) { return (v.flags & AICB_VOXEL_NO_COLLISION) ? NONE : HARD; }

// uniform_collision of a block definition (derived.rs:85-104, 159-190; AIR_EVALUATED for is_air).
static Collision uniform_collision(const aicb_block_desc &bd) {
    if (bd.is_air) return NONE;
    if (bd.indices == nullptr) return bd.n_palette ? voxel_collision(bd.palette[0]) : NONE;   // Evoxel::AIR
    if (bd.resolution == 1) {
        const bool at_origin = bd.n_indices == 1 && bd.voxel_bounds.lower[0] == 0 && bd.voxel_bounds.lower[1] == 0 &&
                               bd.voxel_bounds.lower[2] == 0;
        return at_origin ? voxel_collision(bd.palette[bd.indices[0]]) : NONE;
    }
    bool less_than_full = false;
    for (int a = 0; a < 3; a++)
        if (bd.voxel_bounds.lower[a] != 0 || bd.voxel_bounds.size[a] != bd.resolution) less_than_full = true;
    // iter::chain(outside, ...).all_equal_value().ok(): None for an empty or unequal sequence
    auto all_equal = [&](auto &&each, Collision *out) {
        int have = less_than_full ? (int)NONE : -1;
        bool equal = true;
        each([&](Collision c) {
            if (have < 0) have = c;
            else if (have != (int)c) equal = false;
        });
        if (have < 0 || !equal) return false;
        *out = (Collision)have;
        return true;
    };
    Collision c;
    if (all_equal([&](auto f) { for (size_t k = 0; k < bd.n_palette; k++) f(voxel_collision(bd.palette[k])); }, &c))
        return c;
    if (all_equal([&](auto f) { for (size_t k = 0; k < bd.n_indices; k++) f(voxel_collision(bd.palette[bd.indices[k]])); },
                  &c))
        return c;
    return MIXED;
}

// ---- geometry -----------------------------------------------------------------------------------------------------
struct FAab {   // Aab: lower, upper
    double lo[3], hi[3];
};
struct FRay {
    double o[3], d[3];
};

static int opposite(int f) { return f == AICB_FACE_WITHIN ? f : (f <= AICB_FACE_NZ ? f + 3 : f - 3); }
static int face_axis(int f) { return (f - 1) % 3; }
static bool face_positive(int f) { return f >= AICB_FACE_PX; }

// Aab::face_coordinate_outward (aab.rs:170-179)
static double fco(const FAab &b, int f) { return face_positive(f) ? b.hi[face_axis(f)] : -b.lo[face_axis(f)]; }
static FAab translate(const FAab &b, const double v[3]) {
    FAab r;
    for (int a = 0; a < 3; a++) {
        r.lo[a] = b.lo[a] + v[a];
        r.hi[a] = b.hi[a] + v[a];
    }
    return r;
}
static FAab scale(const FAab &b, double s) {
    FAab r;
    for (int a = 0; a < 3; a++) {
        r.lo[a] = b.lo[a] * s;
        r.hi[a] = b.hi[a] * s;
    }
    return r;
}
static bool aab_eq(const FAab &x, const FAab &y) {
    for (int a = 0; a < 3; a++)
        if (!(x.lo[a] == y.lo[a]) || !(x.hi[a] == y.hi[a])) return false;
    return true;
}
// Aab::contains, intersects (aab.rs:302-327)
static bool contains(const FAab &b, const double p[3]) {
    for (int a = 0; a < 3; a++)
        if (!(b.lo[a] <= p[a] && p[a] <= b.hi[a])) return false;
    return true;
}
static bool intersects(const FAab &x, const FAab &y) {
    for (int a = 0; a < 3; a++) {
        const double lo = std::fmax(x.lo[a], y.lo[a]), hi = std::fmin(x.hi[a], y.hi[a]);
        if (!(lo <= hi)) return false;
    }
    return true;
}
// PositiveSign::new_strict(size.volume()) (aab.rs:232-234)
static double volume(const FAab &b) {
    const double v = (b.hi[0] - b.lo[0]) * (b.hi[1] - b.lo[1]) * (b.hi[2] - b.lo[2]);
    return v == 0.0 ? 0.0 : v;
}
// `f as i32`: saturating, NaN -> 0
static int32_t sat_i32(double v) {
    if (v != v) return 0;
    if (v <= -2147483648.0) return I32_MIN;
    if (v >= 2147483647.0) return I32_MAX;
    return (int32_t)v;
}
// Aab::round_up_to_grid (aab.rs:532-537)
static Aab round_up_to_grid(const FAab &b) {
    Aab g;
    for (int a = 0; a < 3; a++) {
        g.lo[a] = sat_i32(std::floor(b.lo[a]));
        g.hi[a] = sat_i32(std::ceil(b.hi[a]));
    }
    return g;
}
// GridAab::intersection_cubes (grid_aab.rs:506-515)
static bool intersection_cubes(const Aab &x, const Aab &y, Aab *out) {
    for (int a = 0; a < 3; a++) {
        out->lo[a] = std::max(x.lo[a], y.lo[a]);
        out->hi[a] = std::min(x.hi[a], y.hi[a]);
        if (out->hi[a] <= out->lo[a]) return false;
    }
    return true;
}
static FRay scale_direction(const FRay &r, double t) {
    FRay o = r;
    for (int a = 0; a < 3; a++) o.d[a] = r.d[a] * t;
    return o;
}
static void unit_endpoint(const FRay &r, double out[3]) {
    for (int a = 0; a < 3; a++) out[a] = r.o[a] + r.d[a];
}

// nudge_on_ray (collision.rs:498-536)
static FRay nudge_on_ray(const FAab &aab, const FRay &segment, int face, double subdivision, bool backward) {
    if (segment.d[0] == 0.0 && segment.d[1] == 0.0 && segment.d[2] == 0.0) return segment;
    if (face == AICB_FACE_WITHIN) return segment;
    double e[3];
    unit_endpoint(segment, e);
    const double fc_scaled = fco(translate(aab, e), face) * subdivision;
    const double penetration_depth = (fc_scaled - std::round(fc_scaled)) / subdivision;
    const int a = face_axis(face);
    const double direction_projection = face_positive(face) ? segment.d[a] : -segment.d[a];   // Face7::dot
    const double epsilon_nudge = backward ? -POSITION_EPSILON : POSITION_EPSILON;
    const double translation = epsilon_nudge - penetration_depth;
    return scale_direction(segment, 1.0 + translation / direction_projection);
}

// aab_raycast (collision.rs:374-382): the leading corner's unbounded Raycaster
static Raycaster aab_raycast(const FAab &aab, const FRay &ray, bool reversed) {
    double o[3];
    for (int a = 0; a < 3; a++) {
        const double v = reversed ? -ray.d[a] : ray.d[a];
        o[a] = ray.o[a] + (v >= 0.0 ? aab.hi[a] : aab.lo[a]);   // Octant::from_vector, corner_point
    }
    Raycaster rc;
    rc.init(o, ray.d);
    return rc;
}

// ---- contacts -----------------------------------------------------------------------------------------------------
static aicb_contact block_contact(const int32_t cube[3], int face) {
    aicb_contact c;
    std::memset(&c, 0, sizeof c);
    for (int a = 0; a < 3; a++) c.cube[a] = cube[a];
    c.kind = AICB_CONTACT_BLOCK;
    c.face = (uint8_t)face;
    return c;
}
static bool contact_eq(const aicb_contact &x, const aicb_contact &y) {
    return x.kind == y.kind && x.face == y.face && x.resolution == y.resolution && x.cube[0] == y.cube[0] &&
           x.cube[1] == y.cube[1] && x.cube[2] == y.cube[2] && x.voxel[0] == y.voxel[0] && x.voxel[1] == y.voxel[1] &&
           x.voxel[2] == y.voxel[2];
}
static aicb_contact without_normal(aicb_contact c) {
    c.face = AICB_FACE_WITHIN;
    return c;
}
// Contact::aab (contact.rs:59-76)
static FAab contact_aab(const aicb_contact &c) {
    FAab b;
    if (c.kind == AICB_CONTACT_BLOCK) {
        for (int a = 0; a < 3; a++) {
            b.lo[a] = (double)c.cube[a];
            b.hi[a] = (double)c.cube[a] + 1.0;
        }
        return b;
    }
    const double r = 1.0 / (double)c.resolution;
    for (int a = 0; a < 3; a++) {
        b.lo[a] = (double)c.voxel[a] * r + (double)c.cube[a];
        b.hi[a] = ((double)c.voxel[a] + 1.0) * r + (double)c.cube[a];
    }
    return b;
}

struct RayEnd {
    double t;
    aicb_contact contact;
};

struct Drop {   // the voxel level's callback: `drop`
    void operator()(const aicb_contact &) const {}
};

// collide_along_ray (collision.rs:100-226) on one level.  VOXEL: the voxels of block `blk` (EvoxelsRef), which never
// recurses and reports nothing; otherwise the Space, whose mixed cubes recurse with `drop` as their callback.
struct Level {
    const Scene *sc;
    const Block *blk;   // voxel level: the block
};

template <class CB>
static bool collide_along_ray(const Level &L, const FRay &ray, const FAab &aab, CB &&callback, bool not_already,
                              RayEnd *out) {
    std::vector<aicb_contact> already_colliding;
    const orc_scene &s = *L.sc->s;
    const Aab bounds = L.blk ? L.blk->vb : s.bounds;
    Raycaster rc = aab_raycast(aab, ray, false);
    RaycastStep st;
    while (rc.next(&st)) {
        const FRay offset_segment = nudge_on_ray(aab, scale_direction(ray, st.t_distance), opposite(st.face), 1.0, false);
        double e[3];
        unit_endpoint(offset_segment, e);
        const FAab step_aab = translate(aab, e);
        if (st.t_distance >= 1.0) break;
        Aab pib;
        if (!intersection_cubes(round_up_to_grid(step_aab), bounds, &pib)) continue;
        bool have = false;
        RayEnd hit{};
        int32_t c[3];
        for (c[0] = pib.lo[0]; c[0] < pib.hi[0]; c[0]++)
            for (c[1] = pib.lo[1]; c[1] < pib.hi[1]; c[1]++)
                for (c[2] = pib.lo[2]; c[2] < pib.hi[2]; c[2]++) {
                    RayEnd found;
                    size_t idx;
                    vol_index(bounds, L.blk ? L.blk->vsize : s.size, c, &idx);
                    if (L.blk) {
                        if (voxel_collision(L.blk->palette[L.blk->indices[idx]]) == NONE) continue;
                        found = {st.t_distance, block_contact(c, st.face)};
                    } else {
                        const uint16_t id = s.ids[idx];
                        const Collision k = (Collision)L.sc->collision[id];
                        if (k == NONE) continue;
                        if (k == HARD) {
                            found = {st.t_distance, block_contact(c, st.face)};
                        } else {
                            // CollisionSpace::recurse (collision.rs:302-324)
                            const Block &b = s.blocks[id];
                            const double res = (double)b.resolution;
                            FRay vray;
                            for (int a = 0; a < 3; a++) {
                                vray.o[a] = (ray.o[a] + -(double)c[a]) * res;
                                vray.d[a] = ray.d[a] * res;
                            }
                            const Level V{L.sc, &b};
                            RayEnd v;
                            const bool sub_not_already = not_already && st.face != AICB_FACE_WITHIN;
                            if (!collide_along_ray(V, vray, scale(aab, res), Drop{},
                                                   sub_not_already, &v))
                                continue;
                            // wrap_as_voxel (collision.rs:48-76)
                            found.t = v.t;
                            found.contact = v.contact;
                            for (int a = 0; a < 3; a++) {
                                found.contact.voxel[a] = v.contact.cube[a];
                                found.contact.cube[a] = c[a];
                            }
                            found.contact.kind = AICB_CONTACT_VOXEL;
                            found.contact.resolution = (uint8_t)b.resolution;
                        }
                    }
                    if (not_already) {
                        if (found.contact.face == AICB_FACE_WITHIN) {
                            already_colliding.push_back(found.contact);
                            callback(found.contact);
                            continue;
                        }
                        const aicb_contact wn = without_normal(found.contact);
                        bool member = false;
                        for (const auto &x : already_colliding) member |= contact_eq(x, wn);
                        if (member) continue;
                    }
                    callback(found.contact);
                    const double nearest = have ? hit.t : INF;
                    if (found.t < nearest) {
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

// ---- the step -----------------------------------------------------------------------------------------------------
struct Body {
    double position[3], velocity[3];
    FAab collision_box, occupying;
    bool flying, noclip;
};

static bool finite3(const double v[3]) { return std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]); }

static FAab uncrushed(const Body &b) { return translate(b.collision_box, b.position); }

// Body::set_position (body.rs:197-207)
static void set_position(Body &b, const double p[3]) {
    if (!finite3(p)) return;
    for (int a = 0; a < 3; a++) b.position[a] = p[a];
    b.occupying = uncrushed(b);
}

struct Panic {
    uint32_t status;
};

static const FRay ZERO_RAY = {{0, 0, 0}, {0, 0, 0}};

// push_out and attempt_push_out (step.rs:662-741)
static bool attempt_push_out(const Scene &sc, const Body &body, const double direction[3], double new_pos[3],
                             double *distance) {
    FRay ray;
    for (int a = 0; a < 3; a++) {
        ray.o[a] = body.position[a];
        ray.d[a] = direction[a];
    }
    const orc_scene &s = *sc.s;
    Raycaster rc = aab_raycast(body.collision_box, ray, true);
    RaycastStep st;
    while (rc.next(&st)) {
        const FRay adjusted = nudge_on_ray(body.collision_box, scale_direction(ray, st.t_distance), st.face, 1.0, true);
        double e[3];
        unit_endpoint(adjusted, e);
        const Aab g = round_up_to_grid(translate(body.collision_box, e));
        bool clear = true;
        int32_t c[3];
        for (c[0] = g.lo[0]; clear && c[0] < g.hi[0]; c[0]++)
            for (c[1] = g.lo[1]; clear && c[1] < g.hi[1]; c[1]++)
                for (c[2] = g.lo[2]; clear && c[2] < g.hi[2]; c[2]++) {
                    size_t idx;
                    if (vol_index(s.bounds, s.size, c, &idx) && sc.collision[s.ids[idx]] == HARD) clear = false;
                }
        if (!clear) continue;
        for (int a = 0; a < 3; a++) new_pos[a] = e[a];
        const double len = std::sqrt(direction[0] * direction[0] + direction[1] * direction[1] +
                                     direction[2] * direction[2]);
        const double d = st.t_distance * len;
        if (d != d) return false;   // NotNan::new(..).ok()?
        *distance = d;
        return true;
    }
    return false;
}

static bool push_out(const Scene &sc, Body &body, double out[3]) {
    bool colliding = false;
    RayEnd unused;
    collide_along_ray(Level{&sc, nullptr}, ZERO_RAY, body.occupying, [&](const aicb_contact &) { colliding = true; },
                      false, &unused);
    if (!colliding) return false;
    bool have = false;
    double best_pos[3] = {0, 0, 0}, best = 0.0;
    for (int dx = -1; dx <= 1; dx++)
        for (int dy = -1; dy <= 1; dy++)
            for (int dz = -1; dz <= 1; dz++) {
                double dir[3] = {(double)dx, (double)dy, (double)dz};
                if (dx == 0 && dy == 0 && dz == 0)
                    for (int a = 0; a < 3; a++) dir[a] = -body.velocity[a];
                double p[3], d;
                if (!attempt_push_out(sc, body, dir, p, &d)) continue;
                if (!have || d < best) {   // min_by_key: the first minimum
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

// How many shrinks crush_if_colliding may take (the product's rule, restated) for a box {lo, hi} before it counts as not finishing
// (AICB_BODY_CRUSH_UNFINISHED).  Each shrink that changes the box moves one face inward onto a face of a cube or voxel
// (up to one rounding), and every voxel face lies on a plane k / 128, so a crush that finishes crosses at most the
// planes of resolution 128 inside the box on each of its six faces; four times that, plus 64, leaves room for
// rounding.  A shrink that changes nothing is the reference's endless loop and is caught at once.
static double crush_limit(const double lo[3], const double hi[3]) {
    double planes = 0.0;
    for (int a = 0; a < 3; a++) planes = planes + 2.0 * (std::ceil((hi[a] - lo[a]) * 128.0) + 1.0);
    const double limit = 4.0 * planes + 64.0;
    return limit < 1e9 ? limit : 1e9;
}

// crush_if_colliding (step.rs:747-798)
static void crush_if_colliding(const Scene &sc, Body &body, double info[6]) {
    const FAab original = body.occupying;
    const double limit = crush_limit(original.lo, original.hi);
    for (double iter = 0.0;; iter = iter + 1.0) {
        if (iter >= limit) throw Panic{AICB_BODY_CRUSH_UNFINISHED};
        bool have = false;
        aicb_contact a_contact{};
        RayEnd unused;
        collide_along_ray(Level{&sc, nullptr}, ZERO_RAY, body.occupying,
                          [&](const aicb_contact &c) {
                              a_contact = c;
                              have = true;
                          },
                          false, &unused);
        if (!have) break;
        const FAab ca = contact_aab(a_contact);
        int least_face = -1;
        double least = 0.0;
        for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) {
            const double d = fco(body.occupying, f) + fco(ca, opposite(f));
            if (d >= 0.0 && (least_face < 0 || d < least)) {
                least_face = f;
                least = d;
            }
        }
        if (least_face < 0) throw Panic{AICB_BODY_NO_PENETRATION};
        // expand_or_shrink(FaceMap::splat(0.0).with(face, -depth)) (aab.rs:423-428)
        double dist[7] = {0, 0, 0, 0, 0, 0, 0};
        dist[least_face] = -least;
        FAab shrunk;
        bool ok = true;
        for (int a = 0; a < 3; a++) {
            shrunk.lo[a] = body.occupying.lo[a] - dist[AICB_FACE_NX + a];
            shrunk.hi[a] = body.occupying.hi[a] + dist[AICB_FACE_PX + a];
        }
        for (int a = 0; a < 3; a++) ok &= shrunk.lo[a] <= shrunk.hi[a];
        if (!ok) break;   // "cannot resolve by crushing"
        if (aab_eq(shrunk, body.occupying)) throw Panic{AICB_BODY_CRUSH_UNFINISHED};   // the reference loops forever
        body.occupying = shrunk;
    }
    for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) info[f - 1] = fco(original, f) - fco(body.occupying, f);
}

// uncrush (step.rs:806-976)
static uint8_t uncrush(const Scene &sc, Body &body, uint8_t axes[3]) {
    axes[0] = axes[1] = axes[2] = AICB_AXIS_NONE;
    const FAab full = uncrushed(body);
    if (aab_eq(full, body.occupying)) return AICB_UNCRUSH_NOT_NEEDED;
    int n_axes = 0;
    for (int attempt = 0; attempt < 3; attempt++) {
        const double current_volume = volume(body.occupying);
        bool collided = false;
        FAab single[3];
        for (int a = 0; a < 3; a++) {
            single[a] = body.occupying;
            single[a].lo[a] = full.lo[a];
            single[a].hi[a] = full.hi[a];
        }
        double clear[7];
        for (int f = AICB_FACE_NX; f <= AICB_FACE_PZ; f++) clear[f] = fco(full, f);
        RayEnd unused;
        collide_along_ray(Level{&sc, nullptr}, ZERO_RAY, full,
                          [&](const aicb_contact &contact) {
                              collided = true;
                              const FAab ca = contact_aab(contact);
                              for (int a = 0; a < 3; a++) {
                                  if (!intersects(single[a], ca)) continue;
                                  const double lb = ca.lo[a], ub = ca.hi[a], p = body.position[a];
                                  int face;
                                  if (ub <= p) face = AICB_FACE_NX + a;
                                  else if (lb >= p) face = AICB_FACE_PX + a;
                                  else {
                                      clear[AICB_FACE_NX + a] = fco(body.occupying, AICB_FACE_NX + a);
                                      clear[AICB_FACE_PX + a] = fco(body.occupying, AICB_FACE_PX + a);
                                      continue;
                                  }
                                  clear[face] = std::fmin(clear[face], -fco(ca, opposite(face)));
                              }
                          },
                          false, &unused);
        if (!collided) {
            body.occupying = full;
            return AICB_UNCRUSH_COMPLETE;
        }
        int best_axis = -1;
        double best_volume = 0.0;
        FAab best_aab{};
        for (int a = 0; a < 3; a++) {
            const double lo = -clear[AICB_FACE_NX + a], hi = clear[AICB_FACE_PX + a];
            if (!(lo <= hi)) continue;   // with_axis_range: None
            FAab e = body.occupying;
            e.lo[a] = lo;
            e.hi[a] = hi;
            if (!contains(e, body.position)) continue;
            double v = volume(e) - current_volume;   // saturating_sub: PositiveSign::new_clamped
            v = v > 0.0 ? v : 0.0;
            if (!(v > 0.0)) continue;
            if (best_axis < 0 || v >= best_volume) {   // max_by_key: the last maximum
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

struct ContactSet {
    std::vector<aicb_contact> v;
    void insert(const aicb_contact &c) {
        for (const auto &x : v)
            if (contact_eq(x, c)) return;
        v.push_back(c);
    }
};

// step_one_body (step.rs:316-590) with Some(space), a tick that is not paused.
static void step_one_body(const Scene &sc, Body &body, double dt, const double gravity[3], const double edv[3],
                          aicb_body_step_info &info, ContactSet &set) {
    double v0[3];
    for (int a = 0; a < 3; a++) v0[a] = body.velocity[a];
    for (int a = 0; a < 3; a++) body.velocity[a] = body.velocity[a] + edv[a];
    const bool space = !body.noclip;
    auto collision_callback = [&](const aicb_contact &c) {
        if (c.face == AICB_FACE_WITHIN) info.already_colliding = c;
        set.insert(c);
    };
    const double p2 = body.position[0] * body.position[0] + body.position[1] * body.position[1] +
                      body.position[2] * body.position[2];
    if (!std::isfinite(p2)) return;   // quiescent false, NotNeeded, delta_v zero
    if (!body.flying && space)
        for (int a = 0; a < 3; a++) body.velocity[a] = body.velocity[a] + gravity[a] * dt;
    info.uncrush = AICB_UNCRUSH_NOT_NEEDED;
    info.uncrush_axes[0] = info.uncrush_axes[1] = info.uncrush_axes[2] = AICB_AXIS_NONE;
    if (space) {
        info.uncrush = uncrush(sc, body, info.uncrush_axes);
        info.has_push_out = push_out(sc, body, info.push_out);
        crush_if_colliding(sc, body, info.initial_crush);
    }
    const double v2 = body.velocity[0] * body.velocity[0] + body.velocity[1] * body.velocity[1] +
                      body.velocity[2] * body.velocity[2];
    if (!std::isfinite(v2)) {
        body.velocity[0] = body.velocity[1] = body.velocity[2] = 0.0;
    } else if (v2 <= VELOCITY_EPSILON_SQUARED) {
        info.quiescent = 1;
        for (int a = 0; a < 3; a++) info.delta_v[a] = body.velocity[a] - v0[a];
        return;
    } else if (v2 > VELOCITY_MAGNITUDE_LIMIT_SQUARED) {
        const double k = VELOCITY_MAGNITUDE_LIMIT / std::sqrt(v2);
        for (int a = 0; a < 3; a++) body.velocity[a] = body.velocity[a] * k;
    }
    double delta[3];
    for (int a = 0; a < 3; a++) delta[a] = body.velocity[a] * dt;
    if (space) {
        int seg = 0;
        while (!(delta[0] == 0.0 && delta[1] == 0.0 && delta[2] == 0.0)) {
            if (seg >= 3) throw Panic{AICB_BODY_SLIDING_UNFINISHED};
            // collide_and_advance (step.rs:594-659)
            FRay movement;
            for (int a = 0; a < 3; a++) {
                movement.o[a] = body.position[a];
                movement.d[a] = delta[a];
            }
            RayEnd hit;
            aicb_move_segment &ms = info.move_segments[seg];
            if (collide_along_ray(Level{&sc, nullptr}, movement, body.collision_box, collision_callback, true, &hit)) {
                const int face = hit.contact.face;
                const int axis = face_axis(face);
                const FRay motion = nudge_on_ray(body.collision_box, scale_direction(movement, hit.t), opposite(face),
                                                 hit.contact.kind == AICB_CONTACT_VOXEL ? (double)hit.contact.resolution
                                                                                        : 1.0,
                                                 true);
                double np[3];
                for (int a = 0; a < 3; a++) np[a] = body.position[a] + motion.d[a];
                set_position(body, np);
                for (int a = 0; a < 3; a++) {
                    delta[a] = delta[a] - motion.d[a];
                    ms.delta_position[a] = motion.d[a];
                }
                delta[axis] = 0.0;
                body.velocity[axis] = 0.0;
                ms.stopped_by = hit.contact;
            } else {
                double np[3];
                for (int a = 0; a < 3; a++) np[a] = body.position[a] + delta[a];
                set_position(body, np);
                for (int a = 0; a < 3; a++) {
                    ms.delta_position[a] = delta[a];
                    delta[a] = 0.0;
                }
            }
            seg++;
        }
    } else {
        double np[3];
        for (int a = 0; a < 3; a++) np[a] = body.position[a] + delta[a];
        set_position(body, np);
        for (int a = 0; a < 3; a++) info.move_segments[0].delta_position[a] = delta[a];
    }
    for (int a = 0; a < 3; a++) info.delta_v[a] = body.velocity[a] - v0[a];
}

static bool body_valid(const aicb_body &b, const double *edv) {
    if (!finite3(b.position) || !finite3(b.velocity) || (edv && !finite3(edv))) return false;
    for (int k = 0; k < 6; k++)
        if (!std::isfinite(b.collision_box[k]) || !std::isfinite(b.occupying[k])) return false;
    for (int a = 0; a < 3; a++) {
        if (!(b.collision_box[a] < b.collision_box[3 + a])) return false;
        if (!(b.occupying[a] <= b.occupying[3 + a])) return false;
    }
    return true;
}

}  // namespace orc_body

extern "C" {

typedef struct orc_body_scene orc_body_scene;

orc_body_scene *orc_body_scene_create(const aicb_scene_desc *d) {
    auto *bs = new orc_body::Scene();
    bs->s = orc_scene_create(d);
    bs->collision.resize(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) bs->collision[i] = orc_body::uniform_collision(d->blocks[i]);
    return reinterpret_cast<orc_body_scene *>(bs);
}

void orc_body_scene_destroy(orc_body_scene *p) {
    auto *bs = reinterpret_cast<orc_body::Scene *>(p);
    if (!bs) return;
    orc_scene_destroy(bs->s);
    delete bs;
}

// uniform_collision of one block definition: 0 Hard, 1 None, 2 mixed.
int orc_block_uniform_collision(const aicb_block_desc *b) { return orc_body::uniform_collision(*b); }

// step_one_body for bodies [0, n) (aicb_step_bodies' semantics); n_threads threads share the batch.  Returns 0, or 1
// if a body is invalid (nothing written then).
int orc_step_bodies(const orc_body_scene *p, aicb_body *bodies, const double (*edv)[3], size_t n, double dt,
                    const double gravity[3], aicb_body_step_info *info_out, aicb_contact *contacts,
                    uint32_t max_contacts, int n_threads) {
    using namespace orc_body;
    const Scene &sc = *reinterpret_cast<const Scene *>(p);
    for (size_t i = 0; i < n; i++)
        if (!body_valid(bodies[i], edv ? edv[i] : nullptr)) return 1;
    auto one = [&](size_t i) {
        aicb_body &ab = bodies[i];
        Body b;
        for (int a = 0; a < 3; a++) {
            b.position[a] = ab.position[a];
            b.velocity[a] = ab.velocity[a];
            b.collision_box.lo[a] = ab.collision_box[a];
            b.collision_box.hi[a] = ab.collision_box[3 + a];
            b.occupying.lo[a] = ab.occupying[a];
            b.occupying.hi[a] = ab.occupying[3 + a];
        }
        b.flying = ab.flying != 0;
        b.noclip = ab.noclip != 0;
        aicb_body_step_info info;
        std::memset(&info, 0, sizeof info);
        info.uncrush_axes[0] = info.uncrush_axes[1] = info.uncrush_axes[2] = AICB_AXIS_NONE;
        ContactSet set;
        const double zero[3] = {0, 0, 0};
        try {
            step_one_body(sc, b, dt, gravity, edv ? edv[i] : zero, info, set);
        } catch (const Panic &e) {
            std::memset(&info, 0, sizeof info);
            info.status = e.status;
            if (info_out) info_out[i] = info;
            return;
        }
        info.n_contacts = (uint32_t)set.v.size();
        if (set.v.size() > max_contacts) info.status |= AICB_BODY_CONTACTS_TRUNCATED;
        if (contacts)
            for (size_t k = 0; k < set.v.size() && k < max_contacts; k++) contacts[i * max_contacts + k] = set.v[k];
        for (int a = 0; a < 3; a++) {
            ab.position[a] = b.position[a];
            ab.velocity[a] = b.velocity[a];
            ab.occupying[a] = b.occupying.lo[a];
            ab.occupying[3 + a] = b.occupying.hi[a];
        }
        if (info_out) info_out[i] = info;
    };
    const int nt = std::max(1, n_threads);
    std::atomic<size_t> next{0};
    std::vector<std::thread> threads;
    for (int t = 0; t < nt; t++)
        threads.emplace_back([&] {
            for (size_t i; (i = next.fetch_add(1)) < n;) one(i);
        });
    for (auto &t : threads) t.join();
    return 0;
}

static orc_body::Body to_body(const aicb_body &ab) {
    orc_body::Body b;
    for (int a = 0; a < 3; a++) {
        b.position[a] = ab.position[a];
        b.velocity[a] = ab.velocity[a];
        b.collision_box.lo[a] = ab.collision_box[a];
        b.collision_box.hi[a] = ab.collision_box[3 + a];
        b.occupying.lo[a] = ab.occupying[a];
        b.occupying.hi[a] = ab.occupying[3 + a];
    }
    b.flying = ab.flying != 0;
    b.noclip = ab.noclip != 0;
    return b;
}

// crush_if_colliding and uncrush alone (the step.rs:986-1087 tests): the body's occupying updated in place.
int orc_crush_if_colliding(const orc_body_scene *p, aicb_body *ab, double info[6]) {
    orc_body::Body b = to_body(*ab);
    try {
        orc_body::crush_if_colliding(*reinterpret_cast<const orc_body::Scene *>(p), b, info);
    } catch (const orc_body::Panic &e) {
        return (int)e.status;
    }
    for (int a = 0; a < 3; a++) {
        ab->occupying[a] = b.occupying.lo[a];
        ab->occupying[3 + a] = b.occupying.hi[a];
    }
    return 0;
}

int orc_uncrush(const orc_body_scene *p, aicb_body *ab, uint8_t axes[3]) {
    orc_body::Body b = to_body(*ab);
    const int r = orc_body::uncrush(*reinterpret_cast<const orc_body::Scene *>(p), b, axes);
    for (int a = 0; a < 3; a++) {
        ab->occupying[a] = b.occupying.lo[a];
        ab->occupying[3 + a] = b.occupying.hi[a];
    }
    return r;
}

// collide_along_ray on the Space level for one ray (the collision.rs tests): returns 1 with *t and *contact for a
// collision; every reported contact in reported[0 .. *n_reported) (up to max_reported).
int orc_collide_along_ray(const orc_body_scene *p, const double origin_dir[6], const double aab[6], int not_already,
                          double *t, aicb_contact *contact, aicb_contact *reported, uint32_t max_reported,
                          uint32_t *n_reported) {
    using namespace orc_body;
    const Scene &sc = *reinterpret_cast<const Scene *>(p);
    FRay ray;
    FAab box;
    for (int a = 0; a < 3; a++) {
        ray.o[a] = origin_dir[a];
        ray.d[a] = origin_dir[3 + a];
        box.lo[a] = aab[a];
        box.hi[a] = aab[3 + a];
    }
    uint32_t k = 0;
    RayEnd end;
    const bool hit = collide_along_ray(Level{&sc, nullptr}, ray, box,
                                       [&](const aicb_contact &c) {
                                           if (k < max_reported) reported[k] = c;
                                           k++;
                                       },
                                       not_already != 0, &end);
    *n_reported = k;
    if (hit) {
        *t = end.t;
        *contact = end.contact;
    }
    return hit ? 1 : 0;
}

}  // extern "C"
