// ORACLE — TEST INFRASTRUCTURE ONLY (see ../oracle/aic_oracle.hpp).
//
// CPU restatement of the desktop app's terminal frame (all-is-cubes-desktop/src/terminal.rs:114-142): RtRenderer::draw
// into ColorCharacterBuf (:341-394) through every layer (trace_ray_through_layers, renderer.rs:454-478), ColorBuf::mean +
// CharacterBuf::mean over the antialiasing samples, and ColorCharacterBuf::output (:355-366): the text and
// Camera::post_process_color(Rgba::from(ColorBuf)).  It is built on the raytracer oracle (the Tracer and the ColorBuf
// accumulator of ../oracle/aic_oracle.cpp, compiled into this library a second time) and changes nothing there.
//
// ColorCharacterBuf is the oracle's ColorBuf accumulator (mode 0: its opacity is the stop rule, terminal.rs:371-374)
// plus a CharacterBuf (text.rs:52-123) that every hit is also added to.  The Tracer composites a layer's hits into the
// ColorBuf itself, so the hits of a layer's trace reach the CharacterBuf after the trace, in the order the trace made
// them: EnterSpace (the first counted step, sr.rs:629-637), the surfaces, Incomplete (sr.rs:643-651), the sky and
// debug_pixel_cost's DebugOverrideRg (finish, sr.rs:669-688).  Of the surfaces only the first can change a CharacterBuf
// (a Hit is kept; text.rs:64-71), and the ColorBuf's first-hit observer records exactly that one: the first hit with a
// position the accumulator was given, i.e. the first visible surface under the ColorBuf's stop rule.
//
// Parity pinning: the reference has no test for this caller; CharacterBuf is pinned by the reference's print_space
// images (text.rs:196-341, tests/golden/text_images.json), which a world-only frame reproduces, and the colour by the
// layers oracle that aicb_render_layers_srgb8 is checked against.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fno-fast-math (Rust never contracts to FMA).
#include "../oracle/aic_oracle.cpp"

namespace orc_term {
using namespace orc;

// CharacterBuf states as include/aicb200.h numbers them; the layer of a block index as aicb_terminal_pixel::layer
enum { TEXT_ENTERED = -1, TEXT_EMPTY = -2, TEXT_X = -3, TEXT_BLANK = -4 };
enum { LAYER_NONE = 0, LAYER_WORLD = 1, LAYER_UI = 2 };

// CharacterBuf (text.rs:52-123) with the layer whose Space named the block
struct CharacterBuf {
    int32_t text = TEXT_EMPTY;
    int32_t layer = LAYER_NONE;
    bool is_hit() const { return text >= 0 || text <= TEXT_X; }   // State::Hit
    // CharacterBuf::add (text.rs:86-94) with CharacterRtData (:27-47): a surface's block data is its block's
    // (from_block), an exception's is exception(): "X" for Incomplete, " " otherwise
    void add(int exception, int32_t block, int32_t block_layer) {
        if (exception == EX_ENTER_SPACE) {
            if (!is_hit()) text = TEXT_ENTERED;
        } else if (exception == EX_SKY) {
        } else if (!is_hit()) {   // add_character_hit (:64-71)
            if (exception == EX_NONE) {
                text = block;
                layer = block_layer;
            } else {
                text = exception == EX_INCOMPLETE ? TEXT_X : TEXT_BLANK;
            }
        }
    }
};

// CharacterBuf::mean (text.rs:96-108): reduce; (Hit, _) | (_, Hit) => the first Hit; (Entered, Entered) => Entered
static CharacterBuf character_mean(const CharacterBuf *s, int n) {
    CharacterBuf cur = s[0];
    for (int i = 1; i < n; i++) {
        if (cur.is_hit()) continue;
        if (s[i].is_hit()) cur = s[i];
        else cur.text = (cur.text == TEXT_ENTERED && s[i].text == TEXT_ENTERED) ? TEXT_ENTERED : TEXT_EMPTY;
    }
    return cur;
}

// ColorCharacterBuf (terminal.rs:344-394) without override_color (never set by the reference)
struct ColorCharacterBuf {
    Accum color;
    CharacterBuf text;
    void init() {
        color.init(0);
        text = CharacterBuf();
    }
    bool opaque() const { return color.opaque(); }
    // ColorCharacterBuf::add for a hit made here (backdrop, paint)
    void add(const Hit &h, int block_layer) {
        color.add(h);
        text.add(h.exception, h.block_index, block_layer);
    }
};

// Space block index of a cube (Vol::get)
static int32_t block_at(const orc_scene *sc, const int32_t cube[3]) {
    size_t idx;
    if (!vol_index(sc->bounds, sc->size, cube, &idx)) return -1;
    return sc->ids[idx];
}

// One layer's SpaceRaytracer::trace_ray into the ColorCharacterBuf.  Returns RaytraceInfo::cubes_traced.
static size_t trace_layer(ColorCharacterBuf &a, const orc_scene *sc, const aicb_options &opt, const double o[3],
                          const double d[3], int block_layer) {
    a.color.have_hit = false;   // the first-surface observer, for this layer's trace
    Tracer tr;
    tr.sc = sc;
    tr.opt = &opt;
    tr.acc = &a.color;
    const size_t n = tr.trace(o, d);
    if (tr.cubes_traced > 0) a.text.add(EX_ENTER_SPACE, -1, LAYER_NONE);
    if (a.color.have_hit) a.text.add(EX_NONE, block_at(sc, a.color.first_hit.cube), block_layer);
    if (tr.cubes_traced > 1000) a.text.add(EX_INCOMPLETE, -1, LAYER_NONE);
    a.text.add(EX_SKY, -1, LAYER_NONE);
    if (opt.debug_pixel_cost) a.text.add(EX_DEBUG_RG, -1, LAYER_NONE);
    return n;
}

// Rgba -> ColorBuf (raytracer_components.rs:111-120)
static ColorBuf colorbuf_from_rgba(const float c[4]) {
    return ColorBuf{{c[0] * c[3], c[1] * c[3], c[2] * c[3]}, 1.0f - c[3]};
}

// trace_ray_through_layers (renderer.rs:454-478) for one sample, into a fresh ColorCharacterBuf.  A NULL ray skips
// its layer.
static size_t trace_sample(const orc_scene *world, const aicb_options *wopt, const orc_scene *ui, const aicb_options *uopt,
                           const float *backdrop_rgba, const float *no_world_rgba, const double *world_ray,
                           const double *ui_ray, ColorCharacterBuf *out) {
    size_t total = 0;
    ColorCharacterBuf a;
    a.init();
    if (ui && ui_ray) {
        aicb_options o = *uopt;
        o.include_sky = 0;   // ui.trace_ray(.., false)
        total += trace_layer(a, ui, o, ui_ray, ui_ray + 3, LAYER_UI);
    }
    if (backdrop_rgba && !(backdrop_rgba[0] == 0.0f && backdrop_rgba[1] == 0.0f && backdrop_rgba[2] == 0.0f &&
                           backdrop_rgba[3] == 0.0f)) {
        Hit h{};   // Exception::Backdrop (renderer.rs:458-466): CharacterRtData " "
        h.exception = EX_BACKDROP;
        h.surface = colorbuf_from_rgba(backdrop_rgba);
        h.block_index = -1;
        a.add(h, LAYER_NONE);
    }
    if (world && world_ray) {
        aicb_options o = *wopt;
        o.include_sky = 1;   // world.trace_ray(.., true)
        total += trace_layer(a, world, o, world_ray, world_ray + 3, LAYER_WORLD);
    }
    if (!a.opaque() && no_world_rgba) {
        // *accum = P::paint(NO_WORLD_TO_SHOW, ..) (accum.rs:135-151): Self::default() + one Exception::Paint add
        a.init();
        Hit h{};
        h.exception = EX_PAINT;
        h.surface = colorbuf_from_rgba(no_world_rgba);
        h.block_index = -1;
        a.add(h, LAYER_NONE);
    }
    *out = a;
    return total;
}

// ColorCharacterBuf::mean (terminal.rs:386-393) and ColorCharacterBuf::output (:355-366) with the camera's exposure and
// the options' tone mapping: Camera::post_process_color (camera_struct.rs:376-382, graphics_options.rs:352-368).
static void mean_and_output(const ColorCharacterBuf *s, int n, float exposure, int tone_mapping, float maximum_intensity,
                            float out_rgba[4], int32_t *out_text, int32_t *out_layer) {
    ColorBuf c = s[0].color.color;
    if (n > 1) {   // ColorBuf::mean (raytracer_components.rs:97-102): sums fold from zero
        float l[3] = {0, 0, 0}, t = 0.0f;
        for (int i = 0; i < n; i++) {
            for (int k = 0; k < 3; k++) l[k] = l[k] + s[i].color.color.light[k];
            t = t + s[i].color.color.transmittance;
        }
        for (int k = 0; k < 3; k++) c.light[k] = l[k] / (float)n;
        c.transmittance = t / (float)n;
    }
    CharacterBuf cb[4];
    for (int i = 0; i < n; i++) cb[i] = s[i].text;
    const CharacterBuf text = character_mean(cb, n);
    float rgba[4];
    colorbuf_to_rgba(c, rgba);
    float v[3];
    for (int i = 0; i < 3; i++) v[i] = ps_mul(rgba[i], exposure);
    if (std::isfinite(maximum_intensity)) {
        if (tone_mapping == AICB_TONE_CLAMP) {
            for (int i = 0; i < 3; i++) v[i] = (v[i] > maximum_intensity) ? maximum_intensity : v[i];
        } else {
            const float s_ = ps_clamped(1.0f / (1.0f + luminance(v) / maximum_intensity));
            for (int i = 0; i < 3; i++) v[i] = ps_mul(v[i], s_);
        }
    }
    out_rgba[0] = v[0];
    out_rgba[1] = v[1];
    out_rgba[2] = v[2];
    out_rgba[3] = rgba[3];
    *out_text = text.text;
    *out_layer = text.layer;
}

}  // namespace orc_term

using namespace orc_term;

extern "C" {

// The terminal's frame, every pixel in row-major order.  Either layer may be NULL; the lead layer (the world's, else
// the UI's) chooses the sample points and the post-processing.  Returns cubes_traced summed.
uint64_t orc_render_layers_terminal(const orc_scene *world, const aicb_camera *wcam, const aicb_options *wopt,
                                    const orc_scene *ui, const aicb_camera *ucam, const aicb_options *uopt,
                                    const float *backdrop_rgba, const float *no_world_rgba, float (*out_rgba)[4],
                                    int32_t *out_text, int32_t *out_layer) {
    const aicb_camera *lead_cam = world ? wcam : ucam;
    const aicb_options *lead = world ? wopt : uopt;
    const int n = lead->antialiasing_always ? 4 : 1;
    uint64_t total = 0;
    for (uint32_t y = 0; y < lead_cam->fb_height; y++)
        for (uint32_t x = 0; x < lead_cam->fb_width; x++) {
            ColorCharacterBuf s[4];
            for (int i = 0; i < n; i++) {
                double wr[6], ur[6];
                if (world) pixel_ray(*wcam, x, y, n == 4 ? i : -1, wr, wr + 3);
                if (ui) pixel_ray(*ucam, x, y, n == 4 ? i : -1, ur, ur + 3);
                total += trace_sample(world, wopt, ui, uopt, backdrop_rgba, no_world_rgba, world ? wr : nullptr,
                                      ui ? ur : nullptr, &s[i]);
            }
            const size_t o = (size_t)y * lead_cam->fb_width + x;
            mean_and_output(s, n, lead_cam->exposure, lead->tone_mapping, lead->maximum_intensity, out_rgba[o],
                            &out_text[o], &out_layer[o]);
        }
    return total;
}

// One sample per ray pair: trace_ray_through_layers into a ColorCharacterBuf (hand-built rays; a NULL ray array skips
// its layer).  Per sample: ColorBuf (light, transmittance), text, layer.
uint64_t orc_terminal_trace_samples(const orc_scene *world, const aicb_options *wopt, const orc_scene *ui,
                                    const aicb_options *uopt, const float *backdrop_rgba, const float *no_world_rgba,
                                    const double (*world_rays)[6], const double (*ui_rays)[6], size_t n,
                                    float (*out_colorbuf)[4], int32_t *out_text, int32_t *out_layer) {
    uint64_t total = 0;
    for (size_t i = 0; i < n; i++) {
        ColorCharacterBuf s;
        total += trace_sample(world, wopt, ui, uopt, backdrop_rgba, no_world_rgba, world_rays ? world_rays[i] : nullptr,
                              ui_rays ? ui_rays[i] : nullptr, &s);
        for (int c = 0; c < 3; c++) out_colorbuf[i][c] = s.color.color.light[c];
        out_colorbuf[i][3] = s.color.color.transmittance;
        out_text[i] = s.text.text;
        out_layer[i] = s.text.layer;
    }
    return total;
}

// Rgba::to_srgb8 (color.rs:669-676, 1038-1054) of post-processed RGBA: the encoder draw_rgba applies after
// post_process_color (renderer.rs:287-291).
void orc_terminal_to_srgb8(const float (*rgba)[4], size_t n, uint8_t (*out)[4]) {
    for (size_t i = 0; i < n; i++) {
        for (int k = 0; k < 3; k++) out[i][k] = component_to_srgb8(rgba[i][k]);
        out[i][3] = sat_u8(std::round(rgba[i][3] * 255.0f));
    }
}

// CharacterBuf::add of hand-built hits, in order, to state (text, layer): exception (-1 = a surface of `block` in
// `block_layer`; else the oracle's EX_* numbering).
void orc_character_add(int32_t state[2], const int32_t *exceptions, const int32_t *blocks, const int32_t *block_layers,
                       size_t n) {
    CharacterBuf c;
    c.text = state[0];
    c.layer = state[1];
    for (size_t i = 0; i < n; i++) c.add(exceptions[i], blocks[i], block_layers[i]);
    state[0] = c.text;
    state[1] = c.layer;
}

// CharacterBuf::mean of n (1..4) states (text, layer).
void orc_character_mean(const int32_t (*states)[2], int n, int32_t out[2]) {
    CharacterBuf c[4];
    for (int i = 0; i < n && i < 4; i++) {
        c[i].text = states[i][0];
        c[i].layer = states[i][1];
    }
    const CharacterBuf m = character_mean(c, n < 4 ? n : 4);
    out[0] = m.text;
    out[1] = m.layer;
}

}  // extern "C"
