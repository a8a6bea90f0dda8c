// texture_target.cu — RaytraceToTexture's state on the device (all-is-cubes-gpu/src/raytrace_to_texture.rs): the update
// strategy and its pick position, dirty_pixels, and the colour and depth render targets of RaytraceToTexture::Inner,
// on one context or a device group (include/aicb200.h: aicb_texture_target_*, aicb_group_texture_target_*).
//
// A batch is a layered texture call whose pixel tasks are picks: the kernel that lists the batch's rays computes each
// pick's pixel (pick_pixel, trace_kernel.cuh) and the texture epilogue stores its texels at the pixel's framebuffer
// position, in the target's buffers.  PixelPicker's order is built here: the key of every pixel (:861-876), then a
// stable radix sort of the pixel indices by key (CUB's DeviceRadixSort::SortPairs, which is stable, as Rust's
// sort_by_key is).  On a group the order and the targets are device 0's; every device reads the order and stores its
// texels over peer access.
#include <algorithm>
#include <cstring>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "internal.h"

struct aicb_texture_target {
    std::vector<aicb_ctx *> ctx;   // one context, or a group's (device 0's first); every buffer is device 0's
    uint32_t w = 0, h = 0;
    uint32_t strategy = 0;         // AICB_TEXTURE_INCREMENTAL (= aicb::PICK_INCREMENTAL) or _CONSISTENT
    uint32_t central = 0;          // PixelPicker's central_pixel_count (Incremental)
    uint64_t dirty = 0, next = 0;  // dirty_pixels; the pick position
    DeviceBuffer order;            // Incremental: sorted_pixels, one u32 pixel index per pixel
    DeviceBuffer rgba, depth;      // the render targets: w * h texels, 4 x f16 bits and f32
    DeviceBuffer picks;            // aicb_texture_target_picks' staging

    uint64_t cycle_length() const {
        const uint64_t n = (uint64_t)w * h;
        return strategy == AICB_TEXTURE_INCREMENTAL ? 2 * std::max<uint64_t>(central, n - central) : n;
    }
};
struct aicb_group_texture_target : aicb_texture_target {};

static_assert(AICB_TEXTURE_INCREMENTAL == aicb::PICK_INCREMENTAL && AICB_TEXTURE_CONSISTENT == aicb::PICK_CONSISTENT,
              "a target's strategy is its batches' pick kind");

static const uint32_t CENTRAL_PIXEL_LIMIT = 60000;   // raytrace_to_texture.rs:877
static const uint64_t MAX_PIXELS = 0xffffffffull / 4;   // aicb_render_layers_texture's limit on a batch

// PixelPicker::new's sort key (raytrace_to_texture.rs:861-876) of every pixel, in f64 as the reference computes it:
// the Chebyshev distance from image_center = size / 2 - 0.5 plus blend = ((x ^ y) rem 4) * 2, truncated `as i64`
// (never negative); and the pixel indices to sort along.
static __global__ void k_picker_keys(uint32_t w, uint32_t h, uint32_t n, uint32_t *keys, uint32_t *index) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t x = i % w, y = i / w;
    const double cx = (double)w / 2.0 - 0.5, cy = (double)h / 2.0 - 0.5;
    const double blend = (double)(((x ^ y) % 4) * 2);
    const double square_radius = fmax(fabs((double)x - cx), fabs((double)y - cy));
    keys[i] = (uint32_t)(int64_t)(square_radius + blend);
    index[i] = i;
}

// Picks start .. start + n - 1 of a target, by the function the batches' kernels use.
static __global__ void k_target_picks(uint32_t picks, const uint32_t *order, uint32_t central, uint32_t w, uint32_t h,
                                      uint64_t start, uint32_t n, uint32_t *out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = aicb::pick_pixel(picks, order, central, w, h, start + i);
}

// A w x h viewport's state, made on device 0 before anything of the target changes: both targets of zero bits
// (DrawableTexture::resize makes new textures, frame_texture.rs:43-69) and, for Incremental, PixelPicker::new's order.
static aicb_status new_viewport(aicb_texture_target *t, uint32_t w, uint32_t h) {
    if (w == 0 || h == 0 || (uint64_t)w * h > MAX_PIXELS)
        return aicb_fail(AICB_ERR_INVALID, "a texture target's size must be at least 1 x 1 and at most 2^30 - 1 pixels");
    const uint32_t n = w * h;
    aicb_ctx *ctx = t->ctx[0];
    CU(cudaSetDevice(ctx->device));
    const cudaStream_t stream = ctx->stream.get();
    DeviceBuffer rgba, depth, order;
    TRY(rgba.ensure((size_t)n * 8));
    TRY(depth.ensure((size_t)n * 4));
    CU(cudaMemsetAsync(rgba.get(), 0, (size_t)n * 8, stream));
    CU(cudaMemsetAsync(depth.get(), 0, (size_t)n * 4, stream));
    if (t->strategy == AICB_TEXTURE_INCREMENTAL) {
        TRY(order.ensure((size_t)n * 4));
        DeviceBuffer keys, sorted_keys, index, scratch;
        TRY(keys.ensure((size_t)n * 4));
        TRY(sorted_keys.ensure((size_t)n * 4));
        TRY(index.ensure((size_t)n * 4));
        k_picker_keys<<<(n + 255) / 256, 256, 0, stream>>>(w, h, n, keys.get<uint32_t>(), index.get<uint32_t>());
        CU(cudaGetLastError());
        // keys <= max(w, h) / 2 + 6: only their low bits are sorted
        const uint32_t max_key = std::max(w, h) / 2 + 7;
        const int end_bit = 32 - __builtin_clz(max_key);
        size_t scratch_bytes = 0;
        CU(cub::DeviceRadixSort::SortPairs(nullptr, scratch_bytes, keys.get<uint32_t>(), sorted_keys.get<uint32_t>(),
                                           index.get<uint32_t>(), order.get<uint32_t>(), (int)n, 0, end_bit, stream));
        TRY(scratch.ensure(scratch_bytes + 16));
        CU(cub::DeviceRadixSort::SortPairs(scratch.get(), scratch_bytes, keys.get<uint32_t>(),
                                           sorted_keys.get<uint32_t>(), index.get<uint32_t>(), order.get<uint32_t>(),
                                           (int)n, 0, end_bit, stream));
        CU(cudaStreamSynchronize(stream));   // before the sort's scratch is freed
    } else {
        CU(cudaStreamSynchronize(stream));
    }
    t->w = w;
    t->h = h;
    t->rgba = std::move(rgba);
    t->depth = std::move(depth);
    t->order = std::move(order);
    t->central = std::min(CENTRAL_PIXEL_LIMIT, n / 4);
    return AICB_OK;
}

static aicb_status target_create(aicb_ctx *const *ctx, size_t n_ctx, uint32_t w, uint32_t h, int strategy,
                                 aicb_texture_target *t) {
    if (strategy != AICB_TEXTURE_INCREMENTAL && strategy != AICB_TEXTURE_CONSISTENT)
        return aicb_fail(AICB_ERR_INVALID, "strategy must be AICB_TEXTURE_INCREMENTAL or AICB_TEXTURE_CONSISTENT");
    t->ctx.assign(ctx, ctx + n_ctx);
    t->strategy = (uint32_t)strategy;
    ContextLocks lock(t->ctx);
    TRY(new_viewport(t, w, h));
    t->next = 0;
    t->dirty = t->cycle_length();   // :188
    return AICB_OK;
}

static void target_destroy(aicb_texture_target *t) {
    if (!t) return;
    if (!t->ctx.empty()) cudaSetDevice(t->ctx[0]->device);   // (the buffers are device 0's)
    delete t;
}

// UpdateStrategy::resize (:311-324, 810-821): nothing for the same size; otherwise new targets and, for Incremental, a
// new PixelPicker whose position is 0 (Consistent keeps `next`).  dirty_pixels is left alone.
static aicb_status target_resize(aicb_texture_target *t, uint32_t w, uint32_t h) {
    if (!t) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    if (w == t->w && h == t->h) return AICB_OK;
    TRY(new_viewport(t, w, h));
    if (t->strategy == AICB_TEXTURE_INCREMENTAL) t->next = 0;
    return AICB_OK;
}

static aicb_status target_mark_dirty(aicb_texture_target *t) {
    if (!t) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    t->dirty = t->cycle_length();   // RaytraceToTexture::dirty (:587-589)
    return AICB_OK;
}

// do_some_tracing (:591-745) without its budget rule: n picks from the pick position, traced through the layers as
// aicb_render_layers_texture traces a pixel list (cut into whole-warp ranges on a group), stored at their framebuffer
// positions (store_one, :685-690).
static aicb_status target_trace(aicb_texture_target *t, const LayeredCall &c, const double *depth_transform, size_t n,
                                size_t *n_traced, aicb_render_info *info) {
    if (!t) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    const aicb_layer *lead = nullptr;
    TRY(aicb_check_layers_texture(c.world, c.ui, c.no_world_rgba, depth_transform, nullptr, false,
                                  (size_t)t->w * t->h, t->rgba.get(), t->depth.get<float>(), &lead));
    if (lead->camera->fb_width != t->w || lead->camera->fb_height != t->h)
        return aicb_fail(AICB_ERR_INVALID, "the cameras' framebuffer size must be the texture target's");
    if (contexts(c, lead) != t->ctx)
        return aicb_fail(AICB_ERR_INVALID, "the layers' scenes must be on the texture target's context or group");
    if (n > MAX_PIXELS) return aicb_fail(AICB_ERR_INVALID, "too many picks");
    if (n_traced) *n_traced = 0;
    if (info) std::memset(info, 0, sizeof *info);
    if (t->dirty == 0 || n == 0) return AICB_OK;   // :596-600
    Outputs target;
    target.target.out_rgba16f = t->rgba.get<uint2>();
    target.target.out_tex_depth = t->depth.get<float>();
    aicb_texture_outputs(c.world, c.ui, depth_transform, &target);
    target.target.picks = t->strategy;
    target.target.pixel_list = t->order.get<const uint32_t>();   // (nullptr for Consistent)
    target.target.pick_central = t->central;
    std::vector<LayerPart> parts;
    for (const WarpRange &r : warp_ranges(n, c.n)) {
        LayerPart p;
        const size_t i = parts.size();
        p.world = c.world_scenes ? c.world_scenes[i] : nullptr;
        p.ui = c.ui_scenes ? c.ui_scenes[i] : nullptr;
        p.out = target;
        p.out.target.n_list = (uint32_t)r.count;
        p.out.target.pick_base = t->next + r.begin;
        parts.push_back(p);
    }
    aicb_render_info total;
    TRY(aicb_trace_layers(c.world, c.ui, c.backdrop_rgba, c.no_world_rgba, parts.data(), parts.size(), {}, &total,
                          nullptr));
    t->next += n;
    t->dirty -= std::min<uint64_t>(n, t->dirty);   // :731
    if (n_traced) *n_traced = n;
    if (info) *info = total;
    return AICB_OK;
}

static aicb_status target_state(const aicb_texture_target *t, aicb_texture_target_info *out) {
    if (!t || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    std::memset(out, 0, sizeof *out);
    out->width = t->w;
    out->height = t->h;
    out->strategy = t->strategy;
    out->dirty_pixels = t->dirty;
    out->next_pick = t->next;
    out->cycle_length = t->cycle_length();
    return AICB_OK;
}

static aicb_status target_picks(aicb_texture_target *t, uint64_t start, size_t n, uint32_t *out) {
    if (!t || (n && !out)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > MAX_PIXELS) return aicb_fail(AICB_ERR_INVALID, "too many picks");
    ContextLocks lock(t->ctx);
    if (n == 0) return AICB_OK;
    aicb_ctx *ctx = t->ctx[0];
    CU(cudaSetDevice(ctx->device));
    TRY(t->picks.ensure(n * 4));
    k_target_picks<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream.get()>>>(
        t->strategy, t->order.get<const uint32_t>(), t->central, t->w, t->h, start, (uint32_t)n,
        t->picks.get<uint32_t>());
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, t->picks.get(), n * 4, cudaMemcpyDeviceToHost, ctx->stream.get()));
    CU(cudaStreamSynchronize(ctx->stream.get()));
    return AICB_OK;
}

static aicb_status target_buffers(aicb_texture_target *t, void **d_rgba16f, void **d_depth) {
    if (!t || !d_rgba16f || !d_depth) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    *d_rgba16f = t->rgba.get();
    *d_depth = t->depth.get();
    return AICB_OK;
}

static aicb_status target_read(aicb_texture_target *t, uint16_t (*rgba16f)[4], float *depth, size_t n) {
    if (!t) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(t->ctx);
    if (n != (size_t)t->w * t->h) return aicb_fail(AICB_ERR_INVALID, "n must be the texture target's width * height");
    aicb_ctx *ctx = t->ctx[0];
    CU(cudaSetDevice(ctx->device));
    if (rgba16f) CU(cudaMemcpyAsync(rgba16f, t->rgba.get(), n * 8, cudaMemcpyDeviceToHost, ctx->stream.get()));
    if (depth) CU(cudaMemcpyAsync(depth, t->depth.get(), n * 4, cudaMemcpyDeviceToHost, ctx->stream.get()));
    CU(cudaStreamSynchronize(ctx->stream.get()));
    return AICB_OK;
}

// The layers of a one-context call (as aicb200.cu's one_context gives them).
static LayeredCall one_context(const aicb_layer *world, const aicb_layer *ui, const float *backdrop_rgba,
                               const float *no_world_rgba) {
    return {world, ui, world ? &world->scene : nullptr, ui ? &ui->scene : nullptr, 1, backdrop_rgba, no_world_rgba};
}

extern "C" {

aicb_status aicb_texture_target_create(aicb_ctx *ctx, uint32_t width, uint32_t height, int strategy,
                                       aicb_texture_target **out) {
    if (!ctx || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    aicb_texture_target *t = new aicb_texture_target();
    const aicb_status st = target_create(&ctx, 1, width, height, strategy, t);
    if (st != AICB_OK) {
        target_destroy(t);
        return st;
    }
    *out = t;
    return AICB_OK;
}

void aicb_texture_target_destroy(aicb_texture_target *t) { target_destroy(t); }

aicb_status aicb_texture_target_resize(aicb_texture_target *t, uint32_t width, uint32_t height) {
    return target_resize(t, width, height);
}

aicb_status aicb_texture_target_mark_dirty(aicb_texture_target *t) { return target_mark_dirty(t); }

aicb_status aicb_texture_target_trace(aicb_texture_target *t, const aicb_layer *world, const aicb_layer *ui,
                                      const float backdrop_rgba[4], const float no_world_rgba[4],
                                      const double depth_transform[16], size_t n, size_t *n_traced,
                                      aicb_render_info *info) {
    return target_trace(t, one_context(world, ui, backdrop_rgba, no_world_rgba), depth_transform, n, n_traced, info);
}

aicb_status aicb_texture_target_state(const aicb_texture_target *t, aicb_texture_target_info *out) {
    return target_state(t, out);
}

aicb_status aicb_texture_target_picks(aicb_texture_target *t, uint64_t start, size_t n, uint32_t *out) {
    return target_picks(t, start, n, out);
}

aicb_status aicb_texture_target_buffers(aicb_texture_target *t, void **d_rgba16f, void **d_depth) {
    return target_buffers(t, d_rgba16f, d_depth);
}

aicb_status aicb_texture_target_read(aicb_texture_target *t, uint16_t (*rgba16f)[4], float *depth, size_t n) {
    return target_read(t, rgba16f, depth, n);
}

aicb_status aicb_group_texture_target_create(aicb_group *g, uint32_t width, uint32_t height, int strategy,
                                             aicb_group_texture_target **out) {
    if (!g || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    aicb_group_texture_target *t = new aicb_group_texture_target();
    const aicb_status st = target_create(g->ctx.data(), g->ctx.size(), width, height, strategy, t);
    if (st != AICB_OK) {
        target_destroy(t);
        return st;
    }
    *out = t;
    return AICB_OK;
}

void aicb_group_texture_target_destroy(aicb_group_texture_target *t) { target_destroy(t); }

aicb_status aicb_group_texture_target_resize(aicb_group_texture_target *t, uint32_t width, uint32_t height) {
    return target_resize(t, width, height);
}

aicb_status aicb_group_texture_target_mark_dirty(aicb_group_texture_target *t) { return target_mark_dirty(t); }

aicb_status aicb_group_texture_target_trace(aicb_group_texture_target *t, const aicb_group_layer *world,
                                            const aicb_group_layer *ui, const float backdrop_rgba[4],
                                            const float no_world_rgba[4], const double depth_transform[16], size_t n,
                                            size_t *n_traced, aicb_render_info *info) {
    aicb_layer views[2];
    LayeredCall c;
    TRY(group_call(world, ui, backdrop_rgba, no_world_rgba, views, &c));
    return target_trace(t, c, depth_transform, n, n_traced, info);
}

aicb_status aicb_group_texture_target_state(const aicb_group_texture_target *t, aicb_texture_target_info *out) {
    return target_state(t, out);
}

aicb_status aicb_group_texture_target_picks(aicb_group_texture_target *t, uint64_t start, size_t n, uint32_t *out) {
    return target_picks(t, start, n, out);
}

aicb_status aicb_group_texture_target_buffers(aicb_group_texture_target *t, void **d_rgba16f, void **d_depth) {
    return target_buffers(t, d_rgba16f, d_depth);
}

aicb_status aicb_group_texture_target_read(aicb_group_texture_target *t, uint16_t (*rgba16f)[4], float *depth,
                                           size_t n) {
    return target_read(t, rgba16f, depth, n);
}

}  // extern "C"
