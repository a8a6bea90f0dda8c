// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// CPU restatement of character::exposure::State::step (all-is-cubes/src/character/exposure.rs:67-136) and its
// helpers luminance_average and compute_target_exposure (exposure.rs:139-174), built on the raytracer oracle's
// Raycaster (Raycaster::new + within, raycast.rs:196-230), its scene, light and sky (../oracle/aic_oracle.cpp, compiled
// into this library a second time, and changed in nothing).  Each scene here keeps beside it what only the exposure
// reads: every block's Derived::visible (derived.rs:214, 393-399), derived from the block descriptors (a voxel the block
// uses inside its voxel bounds is visible; an is_air block is not), and the LightPhysics' maximum_distance.
//
// f32::ln and f32::exp follow the raytracer oracle's libm switch (orc_set_libm / ORC_LIBM): glibc's logf / expf, or the
// correctly rounded logf_exact / expf_exact of exact_math.cuh, which the device evaluates.
//
// Parity pinning: tests/test_oracle_exposure.py runs the known answers of exposure.rs:168-241.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_exp {
using namespace orc;

constexpr size_t N_SAMPLES = 100;

struct Scene {
    orc_scene *s = nullptr;
    std::vector<bool> visible;   // per block id: Derived::visible
    uint8_t maximum_distance;    // LightPhysics::Rays { maximum_distance }; 0 = None
};

static bool voxel_visible(const aicb_voxel &v) {
    return !(v.rgba[3] == 0.0f && v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f);
}

// Derived::visible of one descriptor: Evoxels::single_voxel (voxel_storage.rs:364-383) or every voxel in the bounds
static bool block_visible(const aicb_block_desc &b) {
    if (b.is_air) return false;
    if (b.indices == nullptr) return b.n_palette && voxel_visible(b.palette[0]);
    if (b.resolution == 1) {
        const bool at_origin = b.n_indices == 1 && b.voxel_bounds.lower[0] == 0 && b.voxel_bounds.lower[1] == 0 &&
                               b.voxel_bounds.lower[2] == 0;
        return at_origin && voxel_visible(b.palette[b.indices[0]]);
    }
    for (size_t k = 0; k < b.n_indices; k++)
        if (voxel_visible(b.palette[b.indices[k]])) return true;
    return false;
}

static float lum(const float c[3]) { return c[1] * 0.7152f + (c[0] * 0.2126f + c[2] * 0.0722f); }   // color.rs:288-297

static float ln_f32(float x) { return libm_mode() ? aicb::logf_exact(x) : std::log(x); }
static float exp_f32(float x) { return libm_mode() ? aicb::expf_exact(x) : std::exp(x); }

// compute_target_exposure (exposure.rs:168-174); f32::clamp lets NaN through
static float target_exposure(float luminance) {
    float d = 0.9f / luminance;
    if (d < 0.1f) d = 0.1f;
    if (d > 4.0f) d = 4.0f;
    return d * 0.375f + 1.0f * (1.0f - 0.375f);
}

// luminance_average (exposure.rs:139-143): Sum for f32 folds from -0.0, times 100f32.recip()
static float luminance_average(const aicb_exposure_state &st) {
    float sum = -0.0f;
    for (size_t k = 0; k < N_SAMPLES; k++) sum = sum + st.luminance_samples[k];
    return sum * (1.0f / 100.0f);
}

// Sky::sample(direction).luminance()
static float sky_lum(const orc_scene &s, const double d[3]) {
    float c[3];
    sky_sample(s.sky, d, c);
    return lum(c);
}

// Space::get_light (updater.rs:585-594): PackedLight::ONE under LightPhysics::None, the stored texel inside the
// bounds, BlockSky::light_outside beyond them.
static PackedLight get_light(const orc_scene &s, const int32_t c[3]) { return s.has_light ? get_packed_light(s, c) : PL_ONE; }

// State::step (exposure.rs:67-136), usize index arithmetic in size_t
static void step(const Scene &sc, aicb_exposure_state &st, const double m[16], double dt) {
    if (dt == 0.0) return;
    const orc_scene &s = *sc.s;
    const size_t max_steps = (size_t)sc.maximum_distance * 2;
    // Transform3D::transform_point3d(origin): None unless w > 0
    const double x = 0.0 * m[0] + 0.0 * m[4] + 0.0 * m[8] + m[12];
    const double y = 0.0 * m[1] + 0.0 * m[5] + 0.0 * m[9] + m[13];
    const double z = 0.0 * m[2] + 0.0 * m[6] + 0.0 * m[10] + m[14];
    const double w = 0.0 * m[3] + 0.0 * m[7] + 0.0 * m[11] + m[15];
    if (!(w > 0.0)) return;
    const double origin[3] = {x / w, y / w, z / w};
    const double sqrtedge = std::sqrt((double)N_SAMPLES);
    size_t index = st.luminance_sample_index;
    for (int ray = 0; ray < 10; ray++) {
        index = (index + 1) % N_SAMPLES;
        st.luminance_sample_index = (uint32_t)index;
        const double indexf = (double)index;
        // f64::rem_euclid / div_euclid of a non-negative integer by 10
        double r = std::fmod(indexf, sqrtedge);
        if (r < 0.0) r = r + std::fabs(sqrtedge);
        double q = std::trunc(indexf / sqrtedge);
        if (std::fmod(indexf, sqrtedge) < 0.0) q = sqrtedge > 0.0 ? q - 1.0 : q + 1.0;
        const double v[3] = {r / sqrtedge * 2.0 - 1.0, q / sqrtedge * 2.0 - 1.0, -1.0};
        // Transform3D::transform_vector3d
        const double d[3] = {v[0] * m[0] + v[1] * m[4] + v[2] * m[8], v[0] * m[1] + v[1] * m[5] + v[2] * m[9],
                             v[0] * m[2] + v[1] * m[6] + v[2] * m[10]};
        float sample = 0.0f;
        bool found = false;
        Raycaster rc;
        rc.init(origin, d);
        rc.within(s.bounds, false);
        RaycastStep rs;
        for (size_t taken = 0; !found && taken < max_steps && rc.next(&rs); taken++) {
            size_t idx;
            if (!vol_index(s.bounds, s.size, rs.cube, &idx)) {   // never: the cast stays within the bounds
                sample = sky_lum(s, d);
                found = true;
            } else if (sc.visible[s.ids[idx]]) {
                int32_t behind[3] = {rs.cube[0], rs.cube[1], rs.cube[2]};
                if (rs.face != AICB_FACE_WITHIN) behind[(rs.face - 1) % 3] += rs.face >= AICB_FACE_PX ? 1 : -1;
                const PackedLight p = get_light(s, behind);
                if (pl_valid(p)) {
                    const float c[3] = {LUT.v[p.r], LUT.v[p.g], LUT.v[p.b]};
                    sample = lum(c);
                    found = true;
                }
            }
        }
        if (!found) sample = sky_lum(s, d);   // nothing was hit
        st.luminance_samples[index] = sample;
    }
    const float target = target_exposure(luminance_average(st));
    if (std::isfinite(target)) {
        const float delta_log = ln_f32(target) - st.exposure_log;
        st.exposure_log = st.exposure_log + delta_log * (float)dt * 2.0f;
    }
}

}  // namespace orc_exp

extern "C" {

typedef struct orc_exposure_scene orc_exposure_scene;

orc_exposure_scene *orc_exposure_scene_create(const aicb_scene_desc *d) {
    auto *sc = new orc_exp::Scene();
    sc->s = orc_scene_create(d);
    sc->maximum_distance = d->light_max_distance;
    sc->visible.resize(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) sc->visible[i] = orc_exp::block_visible(d->blocks[i]);
    return reinterpret_cast<orc_exposure_scene *>(sc);
}

void orc_exposure_scene_destroy(orc_exposure_scene *p) {
    auto *sc = reinterpret_cast<orc_exp::Scene *>(p);
    if (!sc) return;
    orc_scene_destroy(sc->s);
    delete sc;
}

// State::step for n eyes in place (eye_to_world: m11..m44 each); exposure_out_or_null[i] = State::exposure().
void orc_exposure_step(const orc_exposure_scene *p, aicb_exposure_state *states, const double (*eye_to_world)[16],
                       size_t n, double dt, float *exposure_out_or_null) {
    const auto &sc = *reinterpret_cast<const orc_exp::Scene *>(p);
    for (size_t i = 0; i < n; i++) {
        orc_exp::step(sc, states[i], eye_to_world[i], dt);
        if (exposure_out_or_null) exposure_out_or_null[i] = orc_exp::exp_f32(states[i].exposure_log);
    }
}

float orc_exposure_target(float luminance) { return orc_exp::target_exposure(luminance); }
float orc_exposure_average(const aicb_exposure_state *st) { return orc_exp::luminance_average(*st); }
int orc_exposure_block_visible(const orc_exposure_scene *p, uint32_t id) {
    return reinterpret_cast<const orc_exp::Scene *>(p)->visible[id] ? 1 : 0;
}

}  // extern "C"
