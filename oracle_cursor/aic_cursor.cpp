// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// CPU restatement of cursor_raycast (all-is-cubes/src/character/cursor.rs:26-107) and StandardCameras::project_cursor
// (all-is-cubes-render/src/camera/stdcam.rs:357-389), built on the raytracer oracle's Raycaster (Raycaster::new +
// within, raycast.rs:196-230) and its scene (../oracle/aic_oracle.cpp, compiled into this library a second time, and
// changed in nothing).  The raytracer oracle's scene does not keep what only the cursor reads, so each scene here
// keeps its blocks' AICB_BLOCK_* flags and its single voxels' AICB_VOXEL_* flags beside it.
//
// Parity pinning: tests/test_oracle_cursor.py runs the seven known answers of cursor.rs:310-436.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_cur {
using namespace orc;

struct Scene {
    orc_scene *s = nullptr;
    std::vector<bool> block_selectable;    // BlockAttributes::selectable; AIR's is false (evaluated.rs:419-421)
    std::vector<bool> single_selectable;   // a single-voxel block's Evoxel::selectable (Evoxel::AIR's is false)
};

static bool voxel_selectable(const aicb_voxel &v) { return (v.flags & AICB_VOXEL_NOT_SELECTABLE) == 0; }

// Face7::normal_vector (face.rs)
static void face_normal(int face, int32_t n[3]) {
    n[0] = n[1] = n[2] = 0;
    if (face != AICB_FACE_WITHIN) n[(face - 1) % 3] = face >= AICB_FACE_PX ? 1 : -1;
}

static uint32_t texel(PackedLight p) {
    return (uint32_t)p.r | ((uint32_t)p.g << 8) | ((uint32_t)p.b << 16) | ((uint32_t)p.status << 24);
}

// Space::get_light -> LightStorage::get (updater.rs:585-594): PackedLight::ONE under LightPhysics::None, the stored
// texel inside the bounds, BlockSky::light_outside beyond them.
static uint32_t get_light(const orc_scene &s, const int32_t c[3]) {
    if (!s.has_light) return texel(PL_ONE);
    return texel(get_packed_light(s, c));
}

static void miss(aicb_cursor *out) {
    std::memset(out, 0, sizeof *out);
    out->block_id = out->preceding_block_id = AICB_CURSOR_NONE;
}

// cursor_raycast (cursor.rs:26-107) for one ray; true with *out written if a cube was selected.
static bool cursor_raycast(const Scene &cs, const double origin[3], const double dir[3], double maximum_distance,
                           aicb_cursor *out) {
    const orc_scene &s = *cs.s;
    // ray.direction = ray.direction.normalize()  (euclid: self / self.length(), length = sqrt(x*x + y*y + z*z))
    const double len = std::sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    const double d[3] = {dir[0] / len, dir[1] / len, dir[2] / len};
    Raycaster rc;
    rc.init(origin, d);
    rc.within(s.bounds, false);
    RaycastStep step;
    while (rc.next(&step)) {
        if (step.t_distance > maximum_distance) break;
        size_t idx;
        if (!vol_index(s.bounds, s.size, step.cube, &idx)) continue;   // never: the cast stays within the bounds
        const uint16_t id = s.ids[idx];
        const Block &b = s.blocks[id];
        int face_selected = -1;
        if (!cs.block_selectable[id]) continue;
        if (b.single) {
            if (!cs.single_selectable[id]) continue;
            face_selected = step.face;
        } else {
            // step.recursive_raycast(ray, resolution, voxels.bounds()) (raycast.rs:458-476)
            double sub[3];
            for (int a = 0; a < 3; a++) sub[a] = (origin[a] - (double)step.cube[a]) * (double)b.resolution;
            Raycaster vr;
            vr.init(sub, d);
            vr.within(b.vb, true);
            RaycastStep vs;
            bool hit = false;
            while (vr.next(&vs)) {
                if (face_selected < 0) face_selected = vs.face;   // the first face hit: a face of the voxel bounds
                size_t vi;
                if (!vol_index(b.vb, b.vsize, vs.cube, &vi)) continue;   // get_opt_evoxel: None
                if (voxel_selectable(b.palette[b.indices[vi]])) {
                    hit = true;
                    break;
                }
            }
            if (!hit) continue;
        }
        std::memset(out, 0, sizeof *out);
        intersection_point(step, origin, d, out->point_entered);
        out->distance = step.t_distance > 0.0 ? step.t_distance : 0.0;   // PositiveSign::new_clamped
        int32_t n[3];
        face_normal(step.face, n);
        for (int a = 0; a < 3; a++) {
            out->cube[a] = step.cube[a];
            out->preceding_cube[a] = step.cube[a] + n[a];
        }
        out->block_id = id;
        const uint32_t lt = get_light(s, step.cube);
        std::memcpy(out->light, &lt, 4);
        if (step.face == AICB_FACE_WITHIN) {
            out->preceding_block_id = AICB_CURSOR_NONE;
        } else {
            size_t pidx;
            out->preceding_block_id = vol_index(s.bounds, s.size, out->preceding_cube, &pidx) ? s.ids[pidx]
                                                                                              : AICB_CURSOR_OUTSIDE;
            const uint32_t pl = get_light(s, out->preceding_cube);
            std::memcpy(out->preceding_light, &pl, 4);
        }
        out->face_entered = (uint8_t)step.face;
        out->face_selected = (uint8_t)face_selected;
        return true;
    }
    return false;
}

// Camera::project_ndc_into_world (camera_struct.rs:238-257)
static void ndc_ray(const aicb_camera &cam, double x, double y, double o[3], double d[3]) {
    double nearp[3], farp[3];
    project_ndc3(cam, x, y, 0.0, nearp);
    project_ndc3(cam, x, y, 1.0, farp);
    for (int a = 0; a < 3; a++) {
        o[a] = nearp[a];
        d[a] = farp[a] - nearp[a];
    }
}

}  // namespace orc_cur

extern "C" {

typedef struct orc_cursor_scene orc_cursor_scene;

orc_cursor_scene *orc_cursor_scene_create(const aicb_scene_desc *d) {
    auto *cs = new orc_cur::Scene();
    cs->s = orc_scene_create(d);
    cs->block_selectable.resize(d->n_blocks);
    cs->single_selectable.resize(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) {
        const aicb_block_desc &bd = d->blocks[i];
        cs->block_selectable[i] = !bd.is_air && !(bd.flags & AICB_BLOCK_NOT_SELECTABLE);
        // Evoxels::single_voxel (voxel_storage.rs:364-383): One(v), or a resolution-1 block's voxel at the origin,
        // Evoxel::AIR (not selectable) where its bounds hold none; a block without a palette is AIR
        bool sel = false;
        if (bd.indices == nullptr) {
            sel = bd.n_palette && orc_cur::voxel_selectable(bd.palette[0]);
        } else if (bd.resolution == 1) {
            const orc::Block &b = cs->s->blocks[i];
            const int32_t z[3] = {0, 0, 0};
            size_t idx;
            sel = orc::vol_index(b.vb, b.vsize, z, &idx) && orc_cur::voxel_selectable(bd.palette[bd.indices[idx]]);
        }
        cs->single_selectable[i] = sel;
    }
    return reinterpret_cast<orc_cursor_scene *>(cs);
}

void orc_cursor_scene_destroy(orc_cursor_scene *p) {
    auto *cs = reinterpret_cast<orc_cur::Scene *>(p);
    if (!cs) return;
    orc_scene_destroy(cs->s);
    delete cs;
}

// cursor_raycast for n rays {origin, direction}; max_distance_or_null: f64::INFINITY for every ray.
void orc_cursor_raycast(const orc_cursor_scene *p, const double (*origin_dir)[6], const double *max_distance_or_null,
                        size_t n, aicb_cursor *out) {
    const auto &cs = *reinterpret_cast<const orc_cur::Scene *>(p);
    for (size_t i = 0; i < n; i++) {
        const double maxd = max_distance_or_null ? max_distance_or_null[i] : orc::INF;
        if (!orc_cur::cursor_raycast(cs, origin_dir[i], origin_dir[i] + 3, maxd, out + i)) orc_cur::miss(out + i);
    }
}

// project_cursor for n NDC points: the UI layer with f64::INFINITY, then the world layer with world_max_distance.
void orc_project_cursor(const orc_cursor_scene *world, const aicb_camera *world_cam, const orc_cursor_scene *ui,
                        const aicb_camera *ui_cam, const double (*ndc)[2], size_t n, double world_max_distance,
                        aicb_cursor *out) {
    for (size_t i = 0; i < n; i++) {
        double o[3], d[3];
        if (ui) {
            orc_cur::ndc_ray(*ui_cam, ndc[i][0], ndc[i][1], o, d);
            if (orc_cur::cursor_raycast(*reinterpret_cast<const orc_cur::Scene *>(ui), o, d, orc::INF, out + i)) {
                out[i].layer = 1;
                continue;
            }
        }
        if (world) {
            orc_cur::ndc_ray(*world_cam, ndc[i][0], ndc[i][1], o, d);
            if (orc_cur::cursor_raycast(*reinterpret_cast<const orc_cur::Scene *>(world), o, d, world_max_distance,
                                        out + i)) {
                out[i].layer = 2;
                continue;
            }
        }
        orc_cur::miss(out + i);
    }
}

}  // extern "C"
