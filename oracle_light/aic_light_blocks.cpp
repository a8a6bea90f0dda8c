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

}
