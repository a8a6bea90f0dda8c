// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// CPU restatement of RaytraceToTexture's per-pixel work (all-is-cubes-gpu/src/raytrace_to_texture.rs:591-683): the
// Split accumulator (:922-977) traced through the layers, Split::mean, P::paint, the per-layer exposure,
// half::f16::from_f32 and the depth transform.  It is built on the raytracer oracle (the Tracer and the ColorBuf +
// DepthBuf accumulator of ../oracle/aic_oracle.cpp, compiled into this library a second time) and changes nothing
// there.
//
// Parity pinning: the reference has no test for this caller ("TODO: Test PixelPicker", :998), so Split and trace_one
// are pinned only by this restatement of their source; the layer tracing under them is the oracle's
// trace_pixel_layers, which the reference's layer images pin.
//
// Split::add (:962-968) sets the layer of the first hit after which the ColorBuf is not Invisible (transmittance
// != 1).  The Tracer composites a layer's hits into the accumulator itself, so the rule is applied after each add
// made here (backdrop, paint) and after each layer's trace.  That equals the per-hit rule as long as no hit raises the
// transmittance; every trace that did is counted (orc_texture_monotonic_violations), and the tests require none.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_tex {
using namespace orc;

// enum InLayer (:946-950), Option<InLayer> as 0 = None
enum { LAYER_NONE = 0, LAYER_WORLD = 1, LAYER_UI = -1 };

static std::atomic<uint64_t> g_violations{0};

// struct Split (:922-930): ColorBuf + DepthBuf live in the oracle's Accum (mode 0 keeps both, accum.rs:227-238 and
// 275-282), plus the layer.
struct Split {
    Accum acc;
    int layer;
    void init() {
        acc.init(0);
        layer = LAYER_NONE;
    }
    // the tail of Split::add (:965-967): self.layer = self.layer.or(Some(*hit.block)) unless Invisible
    void settle(int block_layer) {
        if (acc.color.transmittance != 1.0f && layer == LAYER_NONE) layer = block_layer;
    }
    // Split::add for a hit the oracle makes itself
    void add(const Hit &h, int block_layer) {
        acc.add(h);
        settle(block_layer);
    }
};

// One layer's SpaceRaytracer::trace_ray into the Split; the rule is applied once the layer's hits are in.
static size_t trace_layer(Split &sp, const orc_scene *sc, const aicb_options &opt, const double o[3], const double d[3],
                          int block_layer) {
    const float before = sp.acc.color.transmittance;
    Tracer tr;
    tr.sc = sc;
    tr.opt = &opt;
    tr.acc = &sp.acc;
    const size_t n = tr.trace(o, d);
    if (sp.acc.color.transmittance > before) g_violations.fetch_add(1, std::memory_order_relaxed);
    sp.settle(block_layer);
    return n;
}

// Rgba -> ColorBuf (raytracer_components.rs:111-120)
static ColorBuf colorbuf_from_rgba(const float c[4]) {
    return ColorBuf{{c[0] * c[3], c[1] * c[3], c[2] * c[3]}, 1.0f - c[3]};
}

// trace_ray_through_layers (renderer.rs:454-478) for one sample, into a fresh Split.  A NULL ray skips its layer.
static size_t trace_sample(const orc_scene *world, const aicb_options *wopt, const orc_scene *ui, const aicb_options *uopt,
                           const float *backdrop_rgba, const float *no_world_rgba, const double *world_ray,
                           const double *ui_ray, Split *out) {
    size_t total = 0;
    Split sp;
    sp.init();
    if (ui && ui_ray) {
        aicb_options o = *uopt;
        o.include_sky = 0;   // ui.trace_ray(.., false)
        total += trace_layer(sp, ui, o, ui_ray, ui_ray + 3, LAYER_UI);
    }
    if (backdrop_rgba && !(backdrop_rgba[0] == 0.0f && backdrop_rgba[1] == 0.0f && backdrop_rgba[2] == 0.0f &&
                           backdrop_rgba[3] == 0.0f)) {
        // Exception::Backdrop with the UI layer's block data (renderer.rs:242-252, 458-466)
        Hit h{};
        h.exception = EX_BACKDROP;
        h.surface = colorbuf_from_rgba(backdrop_rgba);
        h.block_index = -1;
        sp.add(h, LAYER_UI);
    }
    if (world && world_ray) {
        aicb_options o = *wopt;
        o.include_sky = 1;   // world.trace_ray(.., true)
        total += trace_layer(sp, world, o, world_ray, world_ray + 3, LAYER_WORLD);
    }
    if (!sp.acc.opaque() && no_world_rgba) {
        // *accum = P::paint(NO_WORLD_TO_SHOW, world options) (accum.rs:135-151): Self::default() + one add
        sp.init();
        Hit h{};
        h.exception = EX_PAINT;
        h.surface = colorbuf_from_rgba(no_world_rgba);
        h.block_index = -1;
        sp.add(h, LAYER_WORLD);
    }
    *out = sp;
    return total;
}

// Split::mean (:970-976): ColorBuf::mean (raytracer_components.rs:97-102), DepthBuf::mean (accum.rs:284-297: reduce by
// f64::min), the first sample's layer that has one.
static void split_mean(const Split *s, int n, ColorBuf *color, double *depth, int *layer) {
    if (n == 1) {
        *color = s[0].acc.color;
        *depth = s[0].acc.depth;
        *layer = s[0].layer;
        return;
    }
    float l[3] = {0, 0, 0}, t = 0.0f;
    for (int i = 0; i < n; i++) {
        for (int c = 0; c < 3; c++) l[c] = l[c] + s[i].acc.color.light[c];
        t = t + s[i].acc.color.transmittance;
    }
    for (int c = 0; c < 3; c++) color->light[c] = l[c] / (float)n;
    color->transmittance = t / (float)n;
    double d = s[0].acc.depth;
    for (int i = 1; i < n; i++) d = std::fmin(d, s[i].acc.depth);
    *depth = d;
    *layer = LAYER_NONE;
    for (int i = 0; i < n; i++)
        if (s[i].layer != LAYER_NONE) {
            *layer = s[i].layer;
            break;
        }
}

// half::f16::from_f32 (half 2.x, f32_to_f16_fallback): round to nearest even, overflow to infinity, NaN kept quiet
static uint16_t f16_from_f32(float value) {
    uint32_t x;
    std::memcpy(&x, &value, 4);
    const uint32_t sign = x & 0x80000000u, exp = x & 0x7F800000u, man = x & 0x007FFFFFu;
    if (exp == 0x7F800000u) {
        const uint32_t nan_bit = man == 0 ? 0u : 0x0200u;
        return (uint16_t)((sign >> 16) | 0x7C00u | nan_bit | (man >> 13));
    }
    const uint32_t half_sign = sign >> 16;
    const int32_t half_exp = ((int32_t)(exp >> 23) - 127) + 15;
    if (half_exp >= 0x1F) return (uint16_t)(half_sign | 0x7C00u);
    if (half_exp <= 0) {
        if (14 - half_exp > 24) return (uint16_t)half_sign;
        const uint32_t m = man | 0x00800000u;
        uint32_t half_man = m >> (14 - half_exp);
        const uint32_t round_bit = 1u << (13 - half_exp);
        if ((m & round_bit) != 0 && (m & (3 * round_bit - 1)) != 0) half_man += 1;
        return (uint16_t)(half_sign | half_man);
    }
    const uint32_t he = (uint32_t)half_exp << 10, half_man = man >> 13, round_bit = 0x00001000u;
    if ((man & round_bit) != 0 && (man & (3 * round_bit - 1)) != 0) return (uint16_t)((half_sign | he | half_man) + 1);
    return (uint16_t)(half_sign | he | half_man);
}

// trace_one's stores (:643-674) from the pixel's Split
static void store_texels(const ColorBuf &c, double depth, int layer, float exposure_world, float exposure_ui,
                         const double m[16], uint16_t out_rgba[4], float *out_depth) {
    // ColorBuf::into_premultiplied_rgba (raytracer_components.rs:70-77)
    float a = 1.0f - c.transmittance;
    a = a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a);   // f32::clamp: NaN passes
    const float e = layer == LAYER_UI ? exposure_ui : (layer == LAYER_WORLD ? exposure_world : 1.0f);
    out_rgba[0] = f16_from_f32(c.light[0] * e);
    out_rgba[1] = f16_from_f32(c.light[1] * e);
    out_rgba[2] = f16_from_f32(c.light[2] * e);
    out_rgba[3] = f16_from_f32(a);
    // DepthBuf::depth().clamp(0, 1) (f64::clamp: NaN passes)
    double d = depth;
    if (d < 0.0) d = 0.0;
    if (d > 1.0) d = 1.0;
    // euclid 0.22 Transform3D::transform_point3d_homogeneous(point3(0, 0, d)): x*m13 + y*m23 + z*m33 + m43, ...
    const double px = 0.0, py = 0.0, pz = d;
    const double z = px * m[2] + py * m[6] + pz * m[10] + m[14];
    const double w = px * m[3] + py * m[7] + pz * m[11] + m[15];
    const double projected = z / w;
    // f32::from(layer.unwrap_or(InLayer::Ui) as i8)
    const float factor = (float)(int8_t)(layer == LAYER_WORLD ? 1 : -1);
    *out_depth = (float)projected * factor;
}

}  // namespace orc_tex

using namespace orc_tex;

extern "C" {

// RaytraceToTexture::do_some_tracing's trace_one for each listed pixel (raytrace_to_texture.rs:591-683).  Either layer
// may be NULL; the lead layer (the world's, else the UI's) chooses the sample points.  pixels NULL = every pixel in
// row-major order.  Returns cubes_traced summed.
uint64_t orc_render_layers_texture(const orc_scene *world, const aicb_camera *wcam, const aicb_options *wopt,
                                   const orc_scene *ui, const aicb_camera *ucam, const aicb_options *uopt,
                                   const float *backdrop_rgba, const float *no_world_rgba,
                                   const double depth_transform[16], const uint32_t *pixels, size_t n_pixels,
                                   uint16_t (*out_rgba16f)[4], float *out_depth) {
    const aicb_camera *lead_cam = world ? wcam : ucam;
    const aicb_options *lead = world ? wopt : uopt;
    const int n = lead->antialiasing_always ? 4 : 1;
    const float ew = world ? wcam->exposure : 1.0f, eu = ui ? ucam->exposure : 1.0f;
    uint64_t total = 0;
    for (size_t p = 0; p < n_pixels; p++) {
        const uint32_t idx = pixels ? pixels[p] : (uint32_t)p;
        const uint32_t x = idx % lead_cam->fb_width, y = idx / lead_cam->fb_width;
        Split s[4];
        for (int i = 0; i < n; i++) {
            double wr[6], ur[6];
            if (world) pixel_ray(*wcam, x, y, n == 4 ? i : -1, wr, wr + 3);
            if (ui) pixel_ray(*ucam, x, y, n == 4 ? i : -1, ur, ur + 3);
            total += trace_sample(world, wopt, ui, uopt, backdrop_rgba, no_world_rgba, world ? wr : nullptr,
                                  ui ? ur : nullptr, &s[i]);
        }
        ColorBuf c;
        double d;
        int layer;
        split_mean(s, n, &c, &d, &layer);
        store_texels(c, d, layer, ew, eu, depth_transform, out_rgba16f[p], &out_depth[p]);
    }
    return total;
}

// One sample per ray pair: trace_ray_through_layers into a Split (hand-built rays; a NULL ray array skips its layer).
// Per sample: ColorBuf (light, transmittance), DepthBuf, layer (0 none, 1 World, -1 Ui).
uint64_t orc_texture_trace_samples(const orc_scene *world, const aicb_options *wopt, const orc_scene *ui,
                                   const aicb_options *uopt, const float *backdrop_rgba, const float *no_world_rgba,
                                   const double (*world_rays)[6], const double (*ui_rays)[6], size_t n,
                                   float (*out_colorbuf)[4], double *out_depth, int32_t *out_layer) {
    uint64_t total = 0;
    for (size_t i = 0; i < n; i++) {
        Split s;
        total += trace_sample(world, wopt, ui, uopt, backdrop_rgba, no_world_rgba, world_rays ? world_rays[i] : nullptr,
                              ui_rays ? ui_rays[i] : nullptr, &s);
        for (int c = 0; c < 3; c++) out_colorbuf[i][c] = s.acc.color.light[c];
        out_colorbuf[i][3] = s.acc.color.transmittance;
        out_depth[i] = s.acc.depth;
        out_layer[i] = s.layer;
    }
    return total;
}

// Split::mean of n (1 or 4) given samples and trace_one's stores.
void orc_texture_mean_and_store(const float (*colorbuf)[4], const double *depth, const int32_t *layer, int n,
                                float exposure_world, float exposure_ui, const double depth_transform[16],
                                uint16_t out_rgba16f[4], float *out_depth, int32_t *out_layer) {
    Split s[4];
    for (int i = 0; i < n && i < 4; i++) {
        s[i].init();
        for (int c = 0; c < 3; c++) s[i].acc.color.light[c] = colorbuf[i][c];
        s[i].acc.color.transmittance = colorbuf[i][3];
        s[i].acc.depth = depth[i];
        s[i].layer = layer[i];
    }
    ColorBuf c;
    double d;
    int l;
    split_mean(s, n, &c, &d, &l);
    store_texels(c, d, l, exposure_world, exposure_ui, depth_transform, out_rgba16f, out_depth);
    *out_layer = l;
}

uint16_t orc_f16_from_f32(float v) { return f16_from_f32(v); }

uint64_t orc_texture_monotonic_violations(void) { return g_violations.load(); }

}  // extern "C"
