// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// The light oracle (../oracle/aic_light.cpp, compiled into this library a second time, with the raytracer oracle it
// builds its sky from) with a live block table: definitions replaced or appended after creation, and the light side of
// a redefinition.  It changes nothing there.
//
// The reference leaves the light side of SpaceChange::BlockEvaluation as a TODO (space/palette.rs:862-863).  What it
// defines is what placing a block in a cube does to light: Mutation::set -> side_effects_of_set ->
// modified_cube_needs_update (space.rs:499-531, space/light/updater.rs:135-173).  orc_light_relight_blocks applies that
// rule, without Mutation::set's same-block skip, to every cube that holds a redefined block, in increasing linear index
// order.
//
// orc_light_compute_debug is Space::compute_light::<LightUpdateCubeInfo>: compute_light with the rays that ended on a
// face opaque for light, recorded where the reference records them (space/light/debug.rs, updater.rs:838-853).
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"
#include "../oracle/aic_light.cpp"

namespace orc_blocks {
using namespace orc;

// the EvaluatedBlock members light reads, from a block descriptor (as orc_light_create converts them)
static LBlock light_block_of(const aicb_block_desc &bd) {
    LBlock b;
    std::memset(&b, 0, sizeof b);
    b.all_opaque = true;
    for (int f = 0; f < 6; f++) {
        b.opaque[f] = (bd.light_opaque_faces >> f) & 1;
        b.all_opaque = b.all_opaque && b.opaque[f];
        std::memcpy(b.face_color[f + 1], bd.light_face_colors[f], 16);
    }
    std::memcpy(b.face_color[0], bd.light_color, 16);
    std::memcpy(b.emission, bd.light_emission, 12);
    b.has_emission = !(b.emission[0] == 0.0f && b.emission[1] == 0.0f && b.emission[2] == 0.0f);
    b.visible = bd.light_visible != 0;
    return b;
}

// modified_cube_needs_update (updater.rs:135-173) for the cube at linear index `idx`, with the block it holds now
static void modified_cube_needs_update(orc_light &L, size_t idx) {
    int32_t c[3];
    l_cube_of(L, idx, c);
    if (opaque_for_light(L.blocks[L.ids[idx]])) {
        L.light[idx] = L_OPAQUE;
        q_remove(L, idx);
    } else {
        light_needs_update(L, c, PRIO_NEWLY_VISIBLE);
    }
    for (int f = 0; f < 6; f++) {
        int32_t nc[3] = {c[0], c[1], c[2]};
        nc[f % 3] += (f < 3) ? -1 : 1;
        const int opp = (f < 3) ? f + 3 : f - 3;
        if (!get_evaluated(L, nc).opaque[opp]) light_needs_update(L, nc, PRIO_NEWLY_VISIBLE);
    }
}

// ---- Space::compute_light::<LightUpdateCubeInfo> (space.rs:810, space/light/debug.rs) ------------------------------
// The preorder index of every node of the chart: walk_ray_tree's depth-first order, children NX..PZ (updater.rs:500).
static const std::vector<uint32_t> &preorder_of() {
    static const std::vector<uint32_t> pre = [] {
        const std::vector<FlatNode> &ch = chart();
        std::vector<uint32_t> p(ch.size(), 0);
        std::vector<uint32_t> stack{0};
        uint32_t next = 0;
        while (!stack.empty()) {
            const uint32_t i = stack.back();
            stack.pop_back();
            p[i] = next++;
            for (int f = 5; f >= 0; f--)
                if (ch[i].children[f]) stack.push_back(ch[i].children[f]);
        }
        return p;
    }();
    return pre;
}

struct RayRecord {
    uint32_t node;   // preorder index of the node whose cube was struck
    aicb_light_ray ray;
};

// walk_ray_tree (updater.rs:427-529), as walk() in ../oracle/aic_light.cpp, with D = LightUpdateCubeInfo: after
// LightBuffer::traverse, a ray that ended on a face opaque for light is pushed as traverse pushes it (updater.rs:816-853:
// a face other than Within, opaque, with alpha > 0).
static float walk_debug(orc_light &L, LightBuffer &b, std::vector<RayRecord> &rays, const int32_t origin[3],
                        const int32_t cube[3], int face7, uint32_t node_index, bool have_prev, PL prev, RayState rs) {
    const FlatNode &node = chart()[node_index];
    b.visits++;
    float prod[6];
    for (int f = 0; f < 6; f++) prod[f] = node.weight[f] * rs.dw[f];
    const float bundle = fm_sum(prod);
    if (bundle <= 0.0f) return bundle;
    const double dx = ((double)cube[0] + 0.5) - ((double)origin[0] + 0.5),
                 dy = ((double)cube[1] + 0.5) - ((double)origin[1] + 0.5),
                 dz = ((double)cube[2] + 0.5) - ((double)origin[2] + 0.5);
    size_t idx;
    if (dx * dx + dy * dy + dz * dz > b.max_dist_sq || !l_index(L, cube, &idx)) {
        end_of_ray(L, b, rs, bundle, node.weight);
        return bundle;
    }
    const LBlock &ev = L.blocks[L.ids[idx]];
    bool have_ahead = false;
    PL ahead = L_UNINIT;
    traverse(L, b, rs, cube, face7, ev, &have_ahead, &ahead, have_prev, prev, node.weight);
    const float hit_alpha = face7 ? ev.face_color[face7][3] : 0.0f;
    if (ev.visible && face7 != 0 && ev.opaque[face7 - 1] && hit_alpha > 0.0f) {
        RayRecord r;
        std::memset(&r, 0, sizeof r);
        r.node = preorder_of()[node_index];
        int32_t lc[3] = {cube[0], cube[1], cube[2]};   // hit.adjacent()
        lc[(face7 - 1) % 3] += (face7 >= 4) ? 1 : -1;
        const PL stored = have_prev ? prev : light_get(L, lc);
        const float sv[3] = {lut(stored.r), lut(stored.g), lut(stored.b)};
        for (int i = 0; i < 3; i++) {
            r.ray.trigger_cube[i] = cube[i];
            r.ray.value_cube[i] = lc[i];
            const float col = ev.face_color[face7][i] > 1.0f ? 1.0f : ev.face_color[face7][i];   // Rgba::clamp
            r.ray.light_from_struck_face[i] = ev.emission[i] + ps_mul_l(ps_mul_l(col, sv[i]), hit_alpha);
        }
        r.ray.value[0] = stored.r; r.ray.value[1] = stored.g; r.ray.value[2] = stored.b; r.ray.value[3] = stored.s;
        rays.push_back(r);
    }
    if (!(rs.alpha > 0.0f)) {
        end_of_ray(L, b, rs, bundle, node.weight);
        return bundle;
    }
    float child_sum = 0.0f;
    for (int f = 0; f < 6; f++) {
        if (node.children[f]) {
            int32_t nc[3] = {cube[0], cube[1], cube[2]};
            nc[f % 3] += (f < 3) ? -1 : 1;
            const int opp = (f < 3) ? f + 3 : f - 3;
            child_sum += walk_debug(L, b, rays, origin, nc, opp + 1, node.children[f], have_ahead, ahead, rs);
        }
    }
    end_of_ray(L, b, rs, std::fmax(bundle - child_sum, 0.0f), node.weight);
    return bundle;
}

// compute_light (updater.rs:368-418) + finish (:932-944), as compute_light() in ../oracle/aic_light.cpp, with its rays
static PL compute_light_debug(orc_light &L, const int32_t cube[3], std::vector<RayRecord> &rays) {
    LightBuffer b;
    b.max_dist_sq = (double)L.max_distance * (double)L.max_distance;
    const LBlock &ev = get_evaluated(L, cube);
    const bool origin_opaque = ev.all_opaque;
    if (origin_opaque) {
        if (!opaque_for_light(ev)) add_weighted_light(b, ev.emission, 1.0f);
    } else {
        RayState rs;
        rs.alpha = 1.0f;
        for (int f = 0; f < 6; f++) {   // directions_to_seek_light (updater.rs:669-690)
            const int opp = (f < 3) ? f + 3 : f - 3;
            int32_t nf[3] = {cube[0], cube[1], cube[2]}, no[3] = {cube[0], cube[1], cube[2]};
            nf[f % 3] += (f < 3) ? -1 : 1;
            no[opp % 3] += (opp < 3) ? -1 : 1;
            rs.dw[f] = (ev.visible || get_evaluated(L, no).visible || get_evaluated(L, nf).has_emission) ? 1.0f : 0.0f;
        }
        walk_debug(L, b, rays, cube, cube, 0, 0, false, L_UNINIT, rs);
    }
    L.node_visits.fetch_add(b.visits, std::memory_order_relaxed);
    const float scale = ps_clamped_l(1.0f / std::fmax(b.total_weight, 1.0f));
    if (b.total_weight > 0.0f)
        return PL{scalar_in_l(ps_mul_l(b.incoming[0], scale)), scalar_in_l(ps_mul_l(b.incoming[1], scale)),
                  scalar_in_l(ps_mul_l(b.incoming[2], scale)), 255};
    return origin_opaque ? L_OPAQUE : L_NO_RAYS;
}

}  // namespace orc_blocks

using namespace orc_blocks;

extern "C" {

// SpaceChange::BlockEvaluation: new definitions for existing indices (light is not touched)
void orc_light_update_blocks(orc_light *L, const uint16_t *indices, const aicb_block_desc *descs, size_t n) {
    for (size_t i = 0; i < n; i++) L->blocks.at(indices[i]) = light_block_of(descs[i]);
}

// SpaceChange::BlockIndex past the table: the blocks become the next indices
void orc_light_append_blocks(orc_light *L, const aicb_block_desc *descs, size_t n) {
    for (size_t i = 0; i < n; i++) L->blocks.push_back(light_block_of(descs[i]));
}

// The light side of a redefinition: modified_cube_needs_update for every cube holding one of the indices, in increasing
// linear index order (no relaxation: orc_light_evaluate follows)
void orc_light_relight_blocks(orc_light *L, const uint16_t *indices, size_t n) {
    if (L->max_distance == 0 || n == 0) return;
    std::vector<char> redefined(L->blocks.size(), 0);
    for (size_t i = 0; i < n; i++) redefined.at(indices[i]) = 1;
    for (size_t idx = 0; idx < L->ids.size(); idx++)
        if (redefined[L->ids[idx]]) modified_cube_needs_update(*L, idx);
}

// SpaceChange::Physics on the light side: LightStorage::maybe_reinitialize_for_physics_change (updater.rs:80-113).  The
// BlockSky is replaced (Sky::for_blocks through the raytracer oracle's construction; light reads nothing else of the
// sky, so Space::set_physics's early return for an unchanged physics, space.rs:609-612, changes nothing here).  A
// different LightPhysics reinitialises the light: an empty volume and queue under None, else fast_evaluate_light over
// the whole volume (initialize_light's uniform fill is overwritten there, texel by texel).
void orc_light_set_physics(orc_light *L, const aicb_sky *sky, uint8_t light_max_distance) {
    orc_scene s;
    s.sky = *sky;
    build_block_sky(&s);
    for (int f = 0; f < 6; f++) L->sky_faces[f] = PL{s.sky_faces[f].r, s.sky_faces[f].g, s.sky_faces[f].b, s.sky_faces[f].status};
    if (light_max_distance == L->max_distance) return;   // "TODO: if only sky color is different, trigger light updates"
    L->max_distance = light_max_distance;
    L->by_priority.clear();
    L->by_cube.clear();
    if (light_max_distance == 0) {
        L->light.clear();
        return;
    }
    L->light.assign(L->ids.size(), L_UNINIT);
    orc_light_fast_evaluate(L);
}

// The load rule of Space::new_from_builder (space.rs:290-313): every cube whose light is LightStatus::Uninitialized is
// inserted in the queue at Priority::UNINIT, in increasing linear index order.  Returns the number of such cubes (0
// under LightPhysics::None, which has no light storage).
size_t orc_light_queue_uninitialized(orc_light *L) {
    if (L->max_distance == 0) return 0;
    size_t n = 0;
    for (size_t idx = 0; idx < L->light.size(); idx++)
        if (L->light[idx].s == 0) {
            q_insert(*L, idx, PRIO_UNINIT);
            n++;
        }
    return n;
}

// LightStorage::light_needs_update_in_region (updater.rs:122-133): every cube of region ∩ bounds is inserted at
// `priority`.  The sweep branch (more than 400 cubes) queues the same set at the same priority.  Priority::MIN (0)
// never enters the queue: -1 and nothing changes.
int orc_light_queue_region(orc_light *L, const aicb_aab *region, uint8_t priority) {
    if (priority == 0) return -1;
    if (L->max_distance == 0) return 0;
    int64_t lo[3], hi[3];
    for (int a = 0; a < 3; a++) {
        lo[a] = std::max<int64_t>(region->lower[a], L->bounds.lo[a]);
        hi[a] = std::min<int64_t>((int64_t)region->lower[a] + region->size[a], L->bounds.hi[a]);
        if (hi[a] <= lo[a]) return 0;
    }
    for (int64_t x = lo[0]; x < hi[0]; x++)
        for (int64_t y = lo[1]; y < hi[1]; y++)
            for (int64_t z = lo[2]; z < hi[2]; z++) {
                const int32_t c[3] = {(int32_t)x, (int32_t)y, (int32_t)z};
                light_needs_update(*L, c, priority);
            }
    return 0;
}

// Each cube's queued priority, Z-major, 0 where it is not queued
void orc_light_get_queue(const orc_light *L, uint8_t *out) {
    std::memset(out, 0, L->ids.size());
    for (const auto &kv : L->by_cube) out[kv.first] = (uint8_t)kv.second;
}

// Space::compute_light::<LightUpdateCubeInfo> for explicit cubes, against the current field: each cube's texel (what
// orc_light_compute gives), its number of rays, and the rays packed cube after cube in the order the walk pushes them,
// with the preorder index of the node each was struck at.  Returns the total; the rays and nodes are written only if
// `capacity` holds them all.
size_t orc_light_compute_debug(orc_light *L, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4],
                               aicb_light_ray *rays_or_null, uint32_t *nodes_or_null, size_t capacity,
                               uint32_t *ray_counts) {
    std::vector<RayRecord> all;
    for (size_t i = 0; i < n; i++) {
        const size_t before = all.size();
        const PL p = compute_light_debug(*L, cubes[i], all);
        out[i][0] = p.r; out[i][1] = p.g; out[i][2] = p.b; out[i][3] = p.s;
        ray_counts[i] = (uint32_t)(all.size() - before);
    }
    if (all.size() <= capacity)
        for (size_t k = 0; k < all.size(); k++) {
            if (rays_or_null) rays_or_null[k] = all[k].ray;
            if (nodes_or_null) nodes_or_null[k] = all[k].node;
        }
    return all.size();
}

}
