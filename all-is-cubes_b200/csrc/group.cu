// group.cu — one process, several GPUs, behind the C ABI: the row-strip sharding of SURVEY §8(e) for hosts that are
// not Python (the reference's Rust process owns all its threads; a Rust `impl HeadlessRenderer` cannot call
// torch.distributed).  An aicb_group is one aicb_ctx per device; an aicb_group_scene is the scene replicated on each of
// them.  aicb_group_render_srgb8 cuts the frame into interleaved 16-row strips (strip s -> device s mod n), every
// device's last kernel stores its pixels straight into device 0's frame over NVLink (peer access), device 0's stream
// waits for the others' completion events and copies the frame to the caller: compute and delivery are one kernel
// chain per device, there is no collective and no host thread per GPU.
// Replaces the Rayon rows x pixels dispatch of trace_scene_to_image_impl (renderer.rs:516-556) across devices.
// Layered frames, terminal frames and texture targets (layers_srgb8 / _terminal / _texture, which serve
// aicb_render_layers_* on one context and aicb_group_render_layers_* on a group) cut the work the same way, or a pixel
// list into ranges of whole warps, and hand the parts to aicb_trace_layers (aicb200.cu).  Every call issues a pass on
// every device before it waits for any, and re-issues it on a device whose hit stream overflowed (aicb_trace_pass).
// A host call draws as its blocking device-output twin does, into regions of device 0's staging buffer that stand for
// the caller's pointers (stage_outputs); the last pass copies them to the caller (deliver).
// Light propagation (aicb_group_light_*) hands the replicas to light.cu, which runs one context's rounds over them.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "internal.h"

static const uint32_t GROUP_STRIP_ROWS = 16;

aicb_status fan_out(aicb_ctx *const *ctx, size_t n) {
    CU(cudaSetDevice(ctx[0]->device));
    CU(cudaEventRecord(ctx[0]->ev_join.get(), ctx[0]->stream.get()));
    for (size_t i = 1; i < n; i++) {
        CU(cudaSetDevice(ctx[i]->device));
        CU(cudaStreamWaitEvent(ctx[i]->stream.get(), ctx[0]->ev_join.get(), 0));
    }
    return AICB_OK;
}

aicb_status fan_in(aicb_ctx *const *ctx, size_t n) {
    for (size_t i = 1; i < n; i++) {
        CU(cudaSetDevice(ctx[i]->device));
        CU(cudaEventRecord(ctx[i]->ev_join.get(), ctx[i]->stream.get()));
    }
    CU(cudaSetDevice(ctx[0]->device));
    for (size_t i = 1; i < n; i++) CU(cudaStreamWaitEvent(ctx[0]->stream.get(), ctx[i]->ev_join.get(), 0));
    return AICB_OK;
}

// ---- layered frames and texture targets -------------------------------------------------------------------------------
// Every context's part of a layered call.  A whole frame or texture: interleaved 16-row strips, outputs at their
// framebuffer positions in device 0's buffers (`target`).  A pixel list: contiguous ranges of whole warps (a warp
// takes 32 consecutive list entries), as even as whole warps allow; context i traces its range from its own copy of
// it (its d_aux), or of a list in device 0's memory (pixels_on_device) in place, and stores at the range's offset, so
// list order is kept.  One context: one part, every row or the whole list.
static aicb_status layer_parts(const LayeredCall &c, aicb_ctx *const *ctx, const Outputs &target,
                               const uint32_t *pixels, bool pixels_on_device, size_t n_pixels,
                               std::vector<LayerPart> *parts) {
    auto part = [&](size_t i) {
        LayerPart p;
        p.world = c.world_scenes ? c.world_scenes[i] : nullptr;
        p.ui = c.ui_scenes ? c.ui_scenes[i] : nullptr;
        p.out = target;
        return p;
    };
    if (!pixels) {
        for (size_t i = 0; i < c.n; i++) {
            parts->push_back(part(i));
            parts->back().shard = {GROUP_STRIP_ROWS, (uint32_t)i, (uint32_t)c.n};
        }
        return AICB_OK;
    }
    const std::vector<WarpRange> ranges = warp_ranges(n_pixels, c.n);
    for (size_t i = 0; i < ranges.size(); i++) {
        const size_t begin = ranges[i].begin, count = ranges[i].count;
        LayerPart p = part(i);
        if (pixels_on_device) {
            p.out.target.pixel_list = pixels + begin;
        } else {
            CU(cudaSetDevice(ctx[i]->device));
            TRY(ctx[i]->d_aux.ensure(count * 4 + 16));
            CU(cudaMemcpy(ctx[i]->d_aux.get(), pixels + begin, count * 4, cudaMemcpyHostToDevice));
            p.out.target.pixel_list = ctx[i]->d_aux.get<const uint32_t>();
        }
        p.out.target.n_list = (uint32_t)count;
        p.out.target.out_rgba16f = target.target.out_rgba16f + begin;
        p.out.target.out_tex_depth = target.target.out_tex_depth + begin;
        parts->push_back(p);
    }
    return AICB_OK;
}

std::vector<WarpRange> warp_ranges(size_t n_items, size_t n_ctx) {
    const size_t warps = (n_items + 31) / 32;
    const size_t used = std::max<size_t>(1, std::min(n_ctx, warps));
    std::vector<WarpRange> ranges;
    size_t begin = 0;
    for (size_t i = 0; i < used; i++) {
        const size_t count = std::min(32 * (warps / used + (i < warps % used ? 1 : 0)), n_items - begin);
        ranges.push_back({begin, count});
        begin += count;
    }
    return ranges;
}

aicb_status deliver(aicb_ctx *const *ctx, size_t n, const std::vector<Delivery> &copies) {
    TRY(fan_in(ctx, n));
    cudaStream_t stream = ctx[0]->stream.get();
    for (const Delivery &d : copies)
        if (d.bytes) CU(cudaMemcpyAsync(d.to, d.from, d.bytes, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    for (const Delivery &d : copies)
        if (d.then && d.bytes) std::memcpy(d.then, d.to, d.bytes);
    return AICB_OK;
}

// Every listed context's stream waits for the work queued on the caller's stream (device 0's; none if NULL) so far,
// which may be writing the call's inputs or still using its output buffers' memory.
static aicb_status after_caller(aicb_ctx *const *ctx, size_t n, cudaStream_t caller) {
    if (!caller) return AICB_OK;
    CU(cudaSetDevice(ctx[0]->device));
    CU(cudaEventRecord(ctx[0]->ev_join.get(), caller));
    for (size_t i = 0; i < n; i++) {
        CU(cudaSetDevice(ctx[i]->device));
        CU(cudaStreamWaitEvent(ctx[i]->stream.get(), ctx[0]->ev_join.get(), 0));
    }
    return AICB_OK;
}

// The caller's stream (device 0's; none if NULL) waits for the call's work on the first n listed contexts.
static aicb_status before_caller(aicb_ctx *const *ctx, size_t n, cudaStream_t caller) {
    if (!caller) return AICB_OK;
    TRY(fan_in(ctx, n));
    CU(cudaEventRecord(ctx[0]->ev_join.get(), ctx[0]->stream.get()));
    CU(cudaStreamWaitEvent(caller, ctx[0]->ev_join.get(), 0));
    return AICB_OK;
}

// A host call's outputs (`how`) each in a region of device 0's d_out at a 256-byte aligned offset, mapped to a frame's
// target as a device call's are (output_target); `copies` takes the regions to the caller's non-NULL pointers.
static aicb_status stage_outputs(aicb_ctx *root, const aicb_device_outputs &host, Staging how, DeviceCall call,
                                 Outputs *target, std::vector<Delivery> *copies) {
    const size_t n = host.len;
    aicb_device_outputs staged{};
    staged.len = n;
    size_t bytes = 0;
    char *base = nullptr;
    // one output's region: counted on the first walk over the outputs, placed and listed on the second (base set)
    auto take = [&](auto *given, auto *&region, size_t size, bool stored = false) {
        if (!given && !stored) return;
        if (base) {
            region = (std::remove_reference_t<decltype(region)>)(base + bytes);
            if (given) copies->push_back({given, region, n * size});
        }
        bytes += (n * size + 255) & ~(size_t)255;
    };
    auto walk = [&] {
        take(host.srgb8, staged.srgb8, 4);
        take(host.rgba16f, staged.rgba16f, 8);
        take(host.colorbuf, staged.colorbuf, 16, how == STAGE_COLORBUF);
        take(host.depth, staged.depth, 8);
        take(host.hit, staged.hit, sizeof(aicb_hit));
        take(host.steps, staged.steps, 4);
        take(host.text, staged.text, 4);
        take(host.texel_rgba16f, staged.texel_rgba16f, 8);
        take(host.texel_depth, staged.texel_depth, 4);
        take(host.terminal, staged.terminal, sizeof(aicb_terminal_pixel));
    };
    walk();
    CU(cudaSetDevice(root->device));
    TRY(root->d_out.ensure(bytes + 16));
    base = root->d_out.get<char>();
    bytes = 0;
    walk();
    // A pageable destination (a Rust Vec<[u8; 4]>, a numpy array) cannot take an asynchronous DMA: the frame goes to a
    // pinned staging buffer of the library's and is copied out by the host.  Pinned / registered memory is written
    // directly.
    if (how == STAGE_PINNED && n) {
        cudaPointerAttributes attr;
        const cudaError_t pe = cudaPointerGetAttributes(&attr, host.srgb8);
        if (pe != cudaSuccess) cudaGetLastError();
        if (pe != cudaSuccess || attr.type == cudaMemoryTypeUnregistered) {
            TRY(root->h_stage.ensure(n * 4));
            Delivery &d = copies->front();
            d.then = d.to;
            d.to = root->h_stage.get();
        }
    }
    return output_target(&staged, call, false, target);
}

// The contexts of a validated layered call: those of its lead layer's replicas.
std::vector<aicb_ctx *> contexts(const LayeredCall &c, const aicb_layer *lead) {
    aicb_scene *const *scenes = lead == c.world ? c.world_scenes : c.ui_scenes;
    std::vector<aicb_ctx *> ctx;
    for (size_t i = 0; i < c.n; i++) ctx.push_back(scenes[i]->ctx);
    return ctx;
}

// The rest of a layered call once device 0's outputs are in `target`: the parts, the layers and the delivery of
// `copies`, then the caller's stream.
static aicb_status draw_layers(const LayeredCall &c, const std::vector<aicb_ctx *> &ctx, const Outputs &target,
                               const uint32_t *pixels, bool pixels_on_device, size_t n_pixels,
                               const std::vector<Delivery> &copies, cudaStream_t caller, aicb_render_info *info) {
    std::vector<LayerPart> parts;
    TRY(layer_parts(c, ctx.data(), target, pixels, pixels_on_device, n_pixels, &parts));
    aicb_render_info total;
    TRY(aicb_trace_layers(c.world, c.ui, c.backdrop_rgba, c.no_world_rgba, parts.data(), parts.size(), copies, &total,
                          nullptr));
    TRY(before_caller(ctx.data(), parts.size(), caller));
    if (info) *info = total;
    return AICB_OK;
}

// A validated layered host call: its outputs staged in device 0's d_out.
static aicb_status layers_host(const LayeredCall &c, const aicb_layer *lead, const double *depth_transform,
                               const uint32_t *pixels, const aicb_device_outputs &host, aicb_render_info *info) {
    const std::vector<aicb_ctx *> ctx = contexts(c, lead);
    ContextLocks lock(ctx);
    Outputs target;
    std::vector<Delivery> copies;
    TRY(stage_outputs(ctx[0], host, STAGE_GIVEN, DEV_LAYERS, &target, &copies));
    if (target.kind == aicb::TGT_TEX) aicb_texture_outputs(c.world, c.ui, depth_transform, &target);
    target.full_frame = true;
    return draw_layers(c, ctx, target, pixels, false, host.len, copies, nullptr, info);
}

aicb_status layers_srgb8(const LayeredCall &c, uint8_t (*out)[4], size_t out_len, aicb_render_info *info) {
    const aicb_layer *lead = nullptr;
    TRY(aicb_check_layers(c.world, c.ui, c.no_world_rgba, out_len, &lead));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::srgb8, out, out_len);
    return layers_host(c, lead, nullptr, nullptr, o, info);
}

aicb_status layers_terminal(const LayeredCall &c, aicb_terminal_pixel *out, size_t out_len, aicb_render_info *info) {
    const aicb_layer *lead = nullptr;
    TRY(aicb_check_layers(c.world, c.ui, c.no_world_rgba, out_len, &lead));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::terminal, out, out_len);
    return layers_host(c, lead, nullptr, nullptr, o, info);
}

aicb_status layers_texture(const LayeredCall &c, const double *depth_transform, const uint32_t *pixels, size_t n_pixels,
                           uint16_t (*out_rgba16f)[4], float *out_depth, aicb_render_info *info) {
    const aicb_layer *lead = nullptr;
    TRY(aicb_check_layers_texture(c.world, c.ui, c.no_world_rgba, depth_transform, pixels, false, n_pixels, out_rgba16f,
                                  out_depth, &lead));
    if (info) std::memset(info, 0, sizeof *info);
    if (n_pixels == 0) return AICB_OK;
    aicb_device_outputs o{};
    o.texel_rgba16f = out_rgba16f;
    o.texel_depth = out_depth;
    o.len = n_pixels;
    return layers_host(c, lead, depth_transform, pixels, o, info);
}

aicb_status layers_device(const LayeredCall &c, const double *depth_transform, const uint32_t *d_pixels, size_t n_pixels,
                          const aicb_device_outputs *outs, cudaStream_t stream, bool async, aicb_render_info *info) {
    if (!outs) return aicb_fail(AICB_ERR_INVALID, "outs is NULL");
    if (outs->full_frame) return aicb_fail(AICB_ERR_INVALID, "full_frame is for aicb_render_device");
    const aicb_layer *lead = nullptr;
    const bool texels = outs->texel_rgba16f || outs->texel_depth;
    if (texels) {
        TRY(aicb_check_layers_texture(c.world, c.ui, c.no_world_rgba, depth_transform, d_pixels, true, n_pixels,
                                      outs->texel_rgba16f, outs->texel_depth, &lead));
        if (outs->len != n_pixels) return aicb_fail(AICB_ERR_INVALID, "outs->len must equal n_pixels");
    } else {
        TRY(aicb_check_layers(c.world, c.ui, c.no_world_rgba, outs->len, &lead));
        if (d_pixels || n_pixels) return aicb_fail(AICB_ERR_INVALID, "a pixel list is for the texture's texels");
    }
    const std::vector<aicb_ctx *> ctx = contexts(c, lead);
    ContextLocks lock(ctx);
    CU(cudaSetDevice(ctx[0]->device));
    Outputs target;
    TRY(device_target(outs, ctx[0]->device, DEV_LAYERS, false, false, &target));
    if (d_pixels && n_pixels) TRY(check_device_pointer(d_pixels, ctx[0]->device, false, 4, "the pixel list"));
    if (target.kind == aicb::TGT_TEX) aicb_texture_outputs(c.world, c.ui, depth_transform, &target);
    target.full_frame = true;
    if (info) std::memset(info, 0, sizeof *info);
    if (async) {
        if (!stream) stream = ctx[0]->stream.get();
        if (texels && n_pixels == 0) return issue_empty_frame(lead->scene, lead->options, stream);
        std::vector<LayerPart> parts;
        TRY(layer_parts(c, ctx.data(), target, d_pixels, true, n_pixels, &parts));
        return aicb_trace_layers(c.world, c.ui, c.backdrop_rgba, c.no_world_rgba, parts.data(), parts.size(), {},
                                 nullptr, stream);
    }
    if (texels && n_pixels == 0) return AICB_OK;
    TRY(after_caller(ctx.data(), c.n, stream));
    return draw_layers(c, ctx, target, d_pixels, true, n_pixels, {}, stream, info);
}

// ---- world-only frames and ray batches of one scene -------------------------------------------------------------------
// The parts' info summed: counters add up, times are the slowest part's.
static void sum_info(const std::vector<FramePart> &parts, aicb_render_info *info) {
    if (!info) return;
    std::memset(info, 0, sizeof *info);
    for (const FramePart &p : parts) aicb_merge_info(info, &p.info, false);
}

// A frame of the replicas' scene with the caller's options as given: interleaved 16-row strips as
// aicb_group_render_srgb8 cuts them, each part storing at framebuffer positions in device 0's outputs (`target`); with
// `shard` (one context), that shard's rows, packed.  A caller's stream (`caller`, or NULL) goes first, the delivery of
// `copies` follows the frame, and then the caller's stream waits for it.
static aicb_status draw_frame(Replicas r, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                              Outputs target, const std::vector<Delivery> &copies, cudaStream_t caller,
                              aicb_render_info *info) {
    std::vector<LayerPart> strips;   // (the parts' shards)
    std::vector<FramePart> parts;
    if (shard) {
        parts.push_back({r.scene[0], shard, target});
    } else {
        target.full_frame = true;
        const aicb_layer w0 = {r.scene[0], cam, opt};
        const LayeredCall world = {&w0, nullptr, r.scene, nullptr, r.n, nullptr, nullptr};
        TRY(layer_parts(world, r.ctx, target, nullptr, false, 0, &strips));
        for (const LayerPart &p : strips) parts.push_back({p.world, &p.shard, p.out});
    }
    TRY(after_caller(r.ctx, parts.size(), caller));
    TRY(aicb_trace_pass(parts.data(), parts.size(), cam, opt, info != nullptr, copies));
    TRY(before_caller(r.ctx, parts.size(), caller));
    sum_info(parts, info);
    return AICB_OK;
}

aicb_status frame_host(Replicas r, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                       const aicb_device_outputs &host, Staging how, aicb_render_info *info) {
    Outputs target;
    std::vector<Delivery> copies;
    TRY(stage_outputs(r.ctx[0], host, how, DEV_FRAME, &target, &copies));
    return draw_frame(r, cam, opt, shard, target, copies, nullptr, info);
}

// Context i uploads its range of the batch to its own d_aux (or with rays_on_device reads it in place from device 0's
// memory) and stores at the range's offset in device 0's outputs.
static aicb_status draw_rays(Replicas r, const double (*origin_dir)[6], bool rays_on_device, size_t n,
                             const aicb_options *opt, const Outputs &target, const std::vector<Delivery> &copies,
                             cudaStream_t caller, aicb_render_info *info) {
    const std::vector<WarpRange> ranges = warp_ranges(n, r.n);
    std::vector<FramePart> parts;
    TRY(after_caller(r.ctx, ranges.size(), caller));
    for (size_t i = 0; i < ranges.size(); i++) {
        const size_t begin = ranges[i].begin, count = ranges[i].count;
        aicb_ctx *ctx = r.ctx[i];
        CU(cudaSetDevice(ctx->device));
        const double *rays = (const double *)(origin_dir + begin);
        if (!rays_on_device) {
            TRY(ctx->d_aux.ensure(count * 48 + 16));
            if (count) CU(cudaMemcpy(ctx->d_aux.get(), origin_dir + begin, count * 48, cudaMemcpyHostToDevice));
            rays = ctx->d_aux.get<double>();
        }
        FramePart p{r.scene[i]};
        p.out = target;
        aicb::TargetParams &t = p.out.target;
        t.out_colorbuf += begin;
        if (t.out_depth) t.out_depth += begin;
        if (t.out_hit) t.out_hit += begin;
        if (t.out_steps) t.out_steps += begin;
        p.out.rays = rays;
        p.out.n_rays = count;
        parts.push_back(p);
    }
    TRY(aicb_trace_pass(parts.data(), parts.size(), nullptr, opt, info != nullptr, copies));
    TRY(before_caller(r.ctx, parts.size(), caller));
    sum_info(parts, info);
    return AICB_OK;
}

aicb_status rays_host(Replicas r, const double (*origin_dir)[6], const aicb_options *opt,
                      const aicb_device_outputs &host, aicb_render_info *info) {
    if (host.len > 0xffffffffull) return aicb_fail(AICB_ERR_INVALID, "too many rays");
    Outputs target;
    std::vector<Delivery> copies;
    TRY(stage_outputs(r.ctx[0], host, STAGE_COLORBUF, DEV_RAYS, &target, &copies));
    return draw_rays(r, origin_dir, false, host.len, opt, target, copies, nullptr, info);
}

// ---- batches of views of one scene -------------------------------------------------------------------------------
// View v is drawn by replica v mod n, interleaved as row strips are, since views differ in cost.  Every replica traces
// its views as one frame (TGT_VIEWS) and stores them at their view-major positions in device 0's outputs (`target`);
// with `d_cameras` every replica reads device 0's camera table, otherwise each takes its own copy of the caller's
// (through its pinned h_views, on its stream).  A caller's stream, the delivery of `copies` and the info are
// draw_frame's.
static aicb_status draw_views(Replicas r, const aicb_camera *cameras, bool on_device, size_t n_views, uint32_t width,
                              uint32_t height, const aicb_options *opt, const Outputs &target,
                              const std::vector<Delivery> &copies, cudaStream_t caller, aicb_render_info *info) {
    if (info) std::memset(info, 0, sizeof *info);
    if (n_views == 0 || (uint64_t)width * height == 0) return AICB_OK;
    const size_t used = std::min(r.n, n_views);
    std::vector<FramePart> parts;
    TRY(after_caller(r.ctx, used, caller));
    for (size_t i = 0; i < used; i++) {
        const aicb_camera *table = cameras;
        if (!on_device) {
            aicb_ctx *ctx = r.ctx[i];
            const size_t bytes = n_views * sizeof(aicb_camera);
            CU(cudaSetDevice(ctx->device));
            TRY(ctx->h_views.ensure(bytes));
            TRY(ctx->d_views.ensure(bytes));
            std::memcpy(ctx->h_views.get(), cameras, bytes);
            CU(cudaMemcpyAsync(ctx->d_views.get(), ctx->h_views.get(), bytes, cudaMemcpyHostToDevice, ctx->stream.get()));
            table = ctx->d_views.get<const aicb_camera>();
        }
        FramePart p{r.scene[i]};
        p.out = target;
        views_part(&p.out, table, n_views, i, r.n);
        parts.push_back(p);
    }
    const aicb_camera size = views_frame_camera(width, height);
    TRY(aicb_trace_pass(parts.data(), parts.size(), &size, opt, info != nullptr, copies));
    TRY(before_caller(r.ctx, parts.size(), caller));
    sum_info(parts, info);
    return AICB_OK;
}

aicb_status views_host(Replicas r, const aicb_camera *cameras, size_t n_views, const aicb_options *opt,
                       const aicb_device_outputs &host, Staging how, aicb_render_info *info) {
    Outputs target;
    std::vector<Delivery> copies;
    TRY(stage_outputs(r.ctx[0], host, how, DEV_FRAME, &target, &copies));
    const uint32_t width = n_views ? cameras[0].fb_width : 0, height = n_views ? cameras[0].fb_height : 0;
    return draw_views(r, cameras, false, n_views, width, height, opt, target, copies, nullptr, info);
}

aicb_status views_device(Replicas r, const aicb_camera *d_cameras, size_t n_views, uint32_t width, uint32_t height,
                         const aicb_options *opt, const aicb_device_outputs *outs, cudaStream_t caller,
                         aicb_render_info *info) {
    CU(cudaSetDevice(r.ctx[0]->device));
    Outputs target;
    TRY(device_target(outs, r.ctx[0]->device, DEV_FRAME, true, false, &target));
    if (n_views) TRY(check_device_pointer(d_cameras, r.ctx[0]->device, false, 8, "the camera table"));
    return draw_views(r, d_cameras, true, n_views, width, height, opt, target, {}, caller, info);
}

// The layers of a group call as device 0 sees them (its replicas, the cameras and options), and every replica of each.
static aicb_layer on_device0(const aicb_group_layer *l) {
    aicb_layer r;
    r.scene = (l && l->scene) ? l->scene->scene[0] : nullptr;
    r.camera = l ? l->camera : nullptr;
    r.options = l ? l->options : nullptr;
    return r;
}

aicb_status group_call(const aicb_group_layer *world, const aicb_group_layer *ui, const float *backdrop_rgba,
                              const float *no_world_rgba, aicb_layer views[2], LayeredCall *c) {
    const bool have_world = world && world->scene, have_ui = ui && ui->scene;
    if (have_world && have_ui && world->scene->group != ui->scene->group)
        return aicb_fail(AICB_ERR_INVALID, "the layers must be scenes of the same group");
    // (no scene at all: validation rejects the call)
    const aicb_group *g = have_world ? world->scene->group : (have_ui ? ui->scene->group : nullptr);
    views[0] = on_device0(world);
    views[1] = on_device0(ui);
    *c = {world ? &views[0] : nullptr, ui ? &views[1] : nullptr,
          have_world ? world->scene->scene.data() : nullptr, have_ui ? ui->scene->scene.data() : nullptr,
          g ? g->ctx.size() : 0, backdrop_rgba, no_world_rgba};
    return AICB_OK;
}

// ---- light propagation ------------------------------------------------------------------------------------------------
// Light needs more than frames: device 0 stores into every device's light volume (the push of a round), and every
// device's walks raise priorities in device 0's queue with atomics.  Checked and enabled at the first light call.
static aicb_status ensure_light_peers(aicb_group *g) {
    if (g->light_peers) return AICB_OK;
    const int root = g->ctx[0]->device;
    for (size_t i = 1; i < g->ctx.size(); i++) {
        const int dev = g->ctx[i]->device;
        if (dev == root) continue;
        int can = 0, atomics = 0;
        CU(cudaDeviceCanAccessPeer(&can, root, dev));
        if (!can) return aicb_fail(AICB_ERR_UNSUPPORTED, "the root device cannot access a device's memory (no P2P / NVLink path)");
        CU(cudaDeviceGetP2PAttribute(&atomics, cudaDevP2PAttrNativeAtomicSupported, dev, root));
        if (!atomics) return aicb_fail(AICB_ERR_UNSUPPORTED, "a device has no native atomics on the root device's memory");
        CU(cudaSetDevice(root));
        cudaError_t e = cudaDeviceEnablePeerAccess(dev, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
        if (e != cudaSuccess) return aicb_cuda_fail(e, "cudaDeviceEnablePeerAccess");
    }
    g->light_peers = true;
    return AICB_OK;
}

// The body of a group entry point: the handle checked, every context's lock held, with `peers` the light calls' peer
// access ready, `call` run on the group scene's replicas.
template <typename Call>
static aicb_status on_group(const aicb_group_scene *gs, bool peers, Call call) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    if (peers) TRY(ensure_light_peers(gs->group));
    return call(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()});
}

extern "C" {

void aicb_group_destroy(aicb_group *g) { delete g; }

aicb_status aicb_group_create(const int *device_ids, int n_devices, aicb_group **out) {
    if (!device_ids || n_devices < 1 || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument or no devices");
    *out = nullptr;
    aicb_group *g = new aicb_group();
    for (int i = 0; i < n_devices; i++) {
        aicb_ctx *c = nullptr;
        aicb_status st = aicb_ctx_create(device_ids[i], &c);
        if (st != AICB_OK) {
            aicb_group_destroy(g);
            return st;
        }
        g->ctx.push_back(c);
    }
    // every device stores into device 0's frame
    const int root = g->ctx[0]->device;
    for (int i = 1; i < n_devices; i++) {
        const int dev = g->ctx[i]->device;
        if (dev == root) continue;
        int can = 0;
        cudaDeviceCanAccessPeer(&can, dev, root);
        if (!can) {
            aicb_group_destroy(g);
            return aicb_fail(AICB_ERR_UNSUPPORTED, "device cannot access the root device's memory (no P2P / NVLink path)");
        }
        cudaSetDevice(dev);
        cudaError_t e = cudaDeviceEnablePeerAccess(root, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
        if (e != cudaSuccess) {
            aicb_group_destroy(g);
            return aicb_cuda_fail(e, "cudaDeviceEnablePeerAccess");
        }
    }
    *out = g;
    return AICB_OK;
}

int aicb_group_size(const aicb_group *g) { return g ? (int)g->ctx.size() : 0; }

void aicb_group_scene_destroy(aicb_group_scene *gs) {
    if (!gs) return;
    for (size_t i = gs->scene.size(); i-- > 0;) aicb_scene_destroy(gs->scene[i]);   // replica 0, the owner, last
    delete gs;
}

aicb_status aicb_group_scene_create(aicb_group *g, const aicb_scene_desc *d, aicb_group_scene **out) {
    if (!g || !d || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    std::vector<aicb_scene *> scene(g->ctx.size());   // the scene is replicated (<= ~0.3 GB at 256^3), SURVEY §8(e)
    ContextLocks lock(g->ctx);
    TRY(scenes_create(g->ctx.data(), scene.size(), d, scene.data()));
    *out = new aicb_group_scene{g, std::move(scene)};
    return AICB_OK;
}

aicb_status aicb_group_scene_create_device(aicb_group *g, const aicb_scene_desc *d, uint32_t flags, void *stream,
                                           aicb_group_scene **out) {
    if (!g || !d || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    std::vector<aicb_scene *> scene(g->ctx.size());
    ContextLocks lock(g->ctx);
    TRY(scenes_create_device(g->ctx.data(), scene.size(), d, flags, (cudaStream_t)stream, scene.data()));
    *out = new aicb_group_scene{g, std::move(scene)};
    return AICB_OK;
}

aicb_status aicb_group_scene_update_cubes(aicb_group_scene *gs, const int32_t (*cubes)[3], const uint16_t *ids,
                                          const uint8_t (*light)[4], size_t n) {
    return on_group(gs, false, [&](Replicas r) { return scenes_update_cubes(r, cubes, ids, light, n); });
}

aicb_status aicb_group_scene_update_region(aicb_group_scene *gs, const aicb_aab *region, const uint16_t *ids,
                                           uint16_t uniform_id, const uint8_t (*light)[4]) {
    return on_group(gs, false, [&](Replicas r) { return scenes_update_region(r, region, ids, uniform_id, light); });
}

aicb_status aicb_group_render_srgb8(aicb_group_scene *gs, const aicb_camera *cam, const aicb_options *opt,
                                    uint8_t (*out)[4], size_t out_len, aicb_render_info *info) {
    if (!gs || !cam || !opt) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    const size_t pixels = (size_t)cam->fb_width * cam->fb_height;
    if (out_len != pixels) return aicb_fail(AICB_ERR_INVALID, "Viewport size does not match output buffer length");
    if (pixels && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    aicb_status st = aicb_check_render_args(gs->scene[0], cam, opt, nullptr, out_len);
    if (st != AICB_OK) return st;
    const aicb_device_outputs o = one_output(&aicb_device_outputs::srgb8, out, out_len);
    // the caller's options as given (a world-only frame of aicb_trace_layers would force include_sky)
    return on_group(gs, false, [&](Replicas r) { return frame_host(r, cam, opt, nullptr, o, STAGE_GIVEN, info); });
}

// The world-only outputs of one context on the group, with the single-context calls' validation against replica 0.
aicb_status aicb_group_render_colorbuf(aicb_group_scene *gs, const aicb_camera *cam, const aicb_options *opt,
                                       float (*out_colorbuf)[4], double *depth, aicb_hit *hit, uint32_t *steps,
                                       size_t out_len, aicb_render_info *info) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(aicb_check_render_args(gs->scene[0], cam, opt, nullptr, out_len));
    if (out_len && !out_colorbuf) return aicb_fail(AICB_ERR_INVALID, "out_colorbuf is NULL");
    const aicb_device_outputs o = colorbuf_outputs(out_colorbuf, depth, hit, steps, out_len);
    return on_group(gs, false, [&](Replicas r) { return frame_host(r, cam, opt, nullptr, o, STAGE_COLORBUF, info); });
}

aicb_status aicb_group_render_rgba16f(aicb_group_scene *gs, const aicb_camera *cam, const aicb_options *opt,
                                      uint16_t (*out)[4], size_t out_len, aicb_render_info *info) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(aicb_check_render_args(gs->scene[0], cam, opt, nullptr, out_len));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::rgba16f, out, out_len);
    return on_group(gs, false, [&](Replicas r) { return frame_host(r, cam, opt, nullptr, o, STAGE_GIVEN, info); });
}

aicb_status aicb_group_trace_rays(aicb_group_scene *gs, const double (*origin_dir)[6], size_t n, const aicb_options *opt,
                                  float (*out_colorbuf)[4], double *depth, aicb_hit *hit, uint32_t *steps,
                                  aicb_render_info *info) {
    if (!gs || (n && !origin_dir)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(validate_options(opt));
    if (n && !out_colorbuf) return aicb_fail(AICB_ERR_INVALID, "out_colorbuf is NULL");
    const aicb_device_outputs o = colorbuf_outputs(out_colorbuf, depth, hit, steps, n);
    return on_group(gs, false, [&](Replicas r) { return rays_host(r, origin_dir, opt, o, info); });
}

aicb_status aicb_group_render_text(aicb_group_scene *gs, const aicb_camera *cam, const aicb_options *opt, int32_t *out,
                                   size_t out_len, aicb_render_info *info) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(aicb_check_render_args(gs->scene[0], cam, opt, nullptr, out_len));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::text, out, out_len);
    return on_group(gs, false, [&](Replicas r) { return frame_host(r, cam, opt, nullptr, o, STAGE_GIVEN, info); });
}

aicb_status aicb_group_ortho_image_size(const aicb_group_scene *gs, uint32_t resolution, uint32_t *width,
                                        uint32_t *height) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    return aicb_ortho_image_size(gs->scene[0], resolution, width, height);
}

aicb_status aicb_group_render_orthographic(aicb_group_scene *gs, uint32_t resolution, uint8_t (*out)[4], size_t out_len,
                                           aicb_render_info *info) {
    return on_group(gs, false, [&](Replicas r) { return ortho_srgb8(r, resolution, out, out_len, info); });
}

aicb_status aicb_group_scene_update_blocks(aicb_group_scene *gs, const uint16_t *indices, const aicb_block_desc *descs,
                                           size_t n) {
    return on_group(gs, false, [&](Replicas r) { return scenes_update_blocks(r, indices, descs, n); });
}

aicb_status aicb_group_scene_append_blocks(aicb_group_scene *gs, const aicb_block_desc *descs, size_t n) {
    return on_group(gs, false, [&](Replicas r) { return scenes_append_blocks(r, descs, n); });
}

aicb_status aicb_group_scene_update_blocks_device(aicb_group_scene *gs, const uint16_t *indices,
                                                  const aicb_block_desc *descs, size_t n, uint32_t flags, void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_blocks_device(r, false, indices, descs, n, flags, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_append_blocks_device(aicb_group_scene *gs, const aicb_block_desc *descs, size_t n,
                                                  uint32_t flags, void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_blocks_device(r, true, nullptr, descs, n, flags, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_fill_uniform(aicb_group_scene *gs, const aicb_block_desc *block) {
    return on_group(gs, false, [&](Replicas r) { return scenes_fill_uniform(r, block); });
}

aicb_status aicb_group_scene_fill_uniform_device(aicb_group_scene *gs, const aicb_block_desc *block, uint32_t flags,
                                                 void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_fill_uniform_device(r, block, flags, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_set_physics(aicb_group_scene *gs, const aicb_sky *sky, uint8_t light_max_distance) {
    return on_group(gs, false, [&](Replicas r) {
        // a reinitialisation runs as aicb_group_light_fast_evaluate does, over the light calls' peers
        if (light_max_distance && light_max_distance != r.scene[0]->host->light_max_distance)
            TRY(ensure_light_peers(gs->group));
        return scenes_set_physics(r, sky, light_max_distance);
    });
}

aicb_status aicb_group_scene_upload_light(aicb_group_scene *gs, const uint8_t (*light)[4], size_t n_texels) {
    return on_group(gs, false, [&](Replicas r) { return scenes_upload_light(r, light, n_texels); });
}

aicb_status aicb_group_render_layers_srgb8(const aicb_group_layer *world, const aicb_group_layer *ui,
                                           const float backdrop_rgba[4], const float no_world_rgba[4], uint8_t (*out)[4],
                                           size_t out_len, aicb_render_info *info) {
    aicb_layer views[2];
    LayeredCall c;
    TRY(group_call(world, ui, backdrop_rgba, no_world_rgba, views, &c));
    return layers_srgb8(c, out, out_len, info);
}

// A batch of views on the group, validated as one context's (check_views) before any device is touched.
aicb_status aicb_group_render_views_srgb8(aicb_group_scene *gs, const aicb_camera *cameras, size_t n_views,
                                          const aicb_options *opt, uint8_t (*out)[4], size_t out_len,
                                          aicb_render_info *info) {
    uint32_t w, h;
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::srgb8, out, out_len);
    return on_group(gs, false, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_PINNED, info); });
}

aicb_status aicb_group_render_views_rgba16f(aicb_group_scene *gs, const aicb_camera *cameras, size_t n_views,
                                            const aicb_options *opt, uint16_t (*out)[4], size_t out_len,
                                            aicb_render_info *info) {
    uint32_t w, h;
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::rgba16f, out, out_len);
    return on_group(gs, false, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_GIVEN, info); });
}

aicb_status aicb_group_render_views_colorbuf(aicb_group_scene *gs, const aicb_camera *cameras, size_t n_views,
                                             const aicb_options *opt, float (*out_colorbuf)[4], double *depth,
                                             aicb_hit *hit, uint32_t *steps, size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out_colorbuf) return aicb_fail(AICB_ERR_INVALID, "out_colorbuf is NULL");
    const aicb_device_outputs o = colorbuf_outputs(out_colorbuf, depth, hit, steps, out_len);
    return on_group(gs, false, [&](Replicas r) {
        return views_host(r, cameras, n_views, opt, o, STAGE_COLORBUF, info);
    });
}

aicb_status aicb_group_render_views_text(aicb_group_scene *gs, const aicb_camera *cameras, size_t n_views,
                                         const aicb_options *opt, int32_t *out, size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return aicb_fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::text, out, out_len);
    return on_group(gs, false, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_GIVEN, info); });
}

aicb_status aicb_group_render_views_device(aicb_group_scene *gs, const aicb_camera *d_cameras, size_t n_views,
                                           uint32_t fb_width, uint32_t fb_height, const aicb_options *opt,
                                           const aicb_device_outputs *outs, void *stream, aicb_render_info *info) {
    if (!gs || !outs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (outs->full_frame) return aicb_fail(AICB_ERR_INVALID, "full_frame is for aicb_render_device");
    TRY(check_views(d_cameras, false, n_views, &fb_width, &fb_height, opt, outs->len));
    return on_group(gs, false, [&](Replicas r) {
        return views_device(r, d_cameras, n_views, fb_width, fb_height, opt, outs, (cudaStream_t)stream, info);
    });
}

// The device-output calls on the group: every device stores into the caller's device-0 buffers; blocking.
aicb_status aicb_group_render_device(aicb_group_scene *gs, const aicb_camera *cam, const aicb_options *opt,
                                     const aicb_device_outputs *outs, void *stream, aicb_render_info *info) {
    if (!gs || !outs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (outs->full_frame) return aicb_fail(AICB_ERR_INVALID, "full_frame is for aicb_render_device");
    TRY(aicb_check_render_args(gs->scene[0], cam, opt, nullptr, outs->len));
    return on_group(gs, false, [&](Replicas r) {
        CU(cudaSetDevice(r.ctx[0]->device));
        Outputs target;
        TRY(device_target(outs, r.ctx[0]->device, DEV_FRAME, true, false, &target));
        return draw_frame(r, cam, opt, nullptr, target, {}, (cudaStream_t)stream, info);
    });
}

aicb_status aicb_group_trace_rays_device(aicb_group_scene *gs, const double (*d_origin_dir)[6], size_t n,
                                         const aicb_options *opt, const aicb_device_outputs *outs, void *stream,
                                         aicb_render_info *info) {
    if (!gs || !outs || (n && !d_origin_dir)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(validate_options(opt));
    if (outs->full_frame) return aicb_fail(AICB_ERR_INVALID, "full_frame is for aicb_render_device");
    if (outs->len != n) return aicb_fail(AICB_ERR_INVALID, "outs->len must equal the number of rays");
    if (n > 0xffffffffull) return aicb_fail(AICB_ERR_INVALID, "too many rays");
    return on_group(gs, false, [&](Replicas r) {
        CU(cudaSetDevice(r.ctx[0]->device));
        Outputs target;
        TRY(device_target(outs, r.ctx[0]->device, DEV_RAYS, true, false, &target));
        if (n) TRY(check_device_pointer(d_origin_dir, r.ctx[0]->device, false, 8, "the ray batch"));
        return draw_rays(r, d_origin_dir, true, n, opt, target, {}, (cudaStream_t)stream, info);
    });
}

aicb_status aicb_group_render_layers_device(const aicb_group_layer *world, const aicb_group_layer *ui,
                                            const float backdrop_rgba[4], const float no_world_rgba[4],
                                            const double depth_transform[16], const uint32_t *d_pixels,
                                            size_t n_pixels, const aicb_device_outputs *outs, void *stream,
                                            aicb_render_info *info) {
    aicb_layer views[2];
    LayeredCall c;
    TRY(group_call(world, ui, backdrop_rgba, no_world_rgba, views, &c));
    return layers_device(c, depth_transform, d_pixels, n_pixels, outs, (cudaStream_t)stream, false, info);
}

aicb_status aicb_group_render_layers_terminal(const aicb_group_layer *world, const aicb_group_layer *ui,
                                              const float backdrop_rgba[4], const float no_world_rgba[4],
                                              aicb_terminal_pixel *out, size_t out_len, aicb_render_info *info) {
    aicb_layer views[2];
    LayeredCall c;
    TRY(group_call(world, ui, backdrop_rgba, no_world_rgba, views, &c));
    return layers_terminal(c, out, out_len, info);
}

aicb_status aicb_group_render_layers_texture(const aicb_group_layer *world, const aicb_group_layer *ui,
                                             const float backdrop_rgba[4], const float no_world_rgba[4],
                                             const double depth_transform[16], const uint32_t *pixels, size_t n_pixels,
                                             uint16_t (*out_rgba16f)[4], float *out_depth, aicb_render_info *info) {
    aicb_layer views[2];
    LayeredCall c;
    TRY(group_call(world, ui, backdrop_rgba, no_world_rgba, views, &c));
    return layers_texture(c, depth_transform, pixels, n_pixels, out_rgba16f, out_depth, info);
}

// ---- light propagation: the single-context calls' arguments, validation and results (light.cu) --------------------
aicb_status aicb_group_light_fast_evaluate(aicb_group_scene *gs) {
    return on_group(gs, true, [&](Replicas r) { return light_fast_evaluate(r); });
}

aicb_status aicb_group_light_compute(aicb_group_scene *gs, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]) {
    return on_group(gs, true, [&](Replicas r) { return light_compute(r, cubes, n, out); });
}

aicb_status aicb_group_light_compute_debug(aicb_group_scene *gs, const int32_t (*cubes)[3], size_t n,
                                           uint8_t (*out_texels)[4], aicb_light_ray *rays, size_t ray_capacity,
                                           uint32_t *ray_counts, size_t *n_rays_total) {
    return on_group(gs, true, [&](Replicas r) {
        return light_compute_debug(r, cubes, n, out_texels, rays, ray_capacity, ray_counts, n_rays_total);
    });
}

aicb_status aicb_group_light_evaluate(aicb_group_scene *gs, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                                      uint64_t *node_visits) {
    return on_group(gs, true, [&](Replicas r) {
        return light_evaluate(r, epsilon, updates_done, max_diff, node_visits);
    });
}

aicb_status aicb_group_light_update_from_queue(aicb_group_scene *gs, uint64_t max_updates, aicb_light_updates_info *info) {
    return on_group(gs, true, [&](Replicas r) { return light_update_from_queue(r, max_updates, info); });
}

aicb_status aicb_group_light_edit_and_propagate(aicb_group_scene *gs, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                                size_t n_edits, uint8_t epsilon, uint64_t *updates_done,
                                                uint8_t *max_diff) {
    return on_group(gs, true, [&](Replicas r) {
        return light_edit_and_propagate(r, cubes, new_ids, n_edits, epsilon, updates_done, max_diff);
    });
}

aicb_status aicb_group_light_edit_cubes(aicb_group_scene *gs, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                        size_t n, size_t *n_changed) {
    return on_group(gs, true, [&](Replicas r) { return light_edit_cubes(r, cubes, new_ids, n, n_changed); });
}

aicb_status aicb_group_light_relight_blocks(aicb_group_scene *gs, const uint16_t *indices, size_t n, uint8_t epsilon,
                                            uint64_t *updates_done, uint8_t *max_diff) {
    return on_group(gs, true, [&](Replicas r) {
        return light_relight_blocks(r, indices, n, epsilon, updates_done, max_diff);
    });
}

aicb_status aicb_group_light_edit_region(aicb_group_scene *gs, const aicb_aab *region, const uint16_t *ids,
                                         uint16_t uniform_id, size_t *n_changed) {
    return on_group(gs, true, [&](Replicas r) { return light_edit_region(r, region, ids, uniform_id, n_changed); });
}

// The queue is device 0's and the scan reads replica 0's volume (the replicas' are identical).
aicb_status aicb_group_light_queue_uninitialized(aicb_group_scene *gs, size_t *n_queued) {
    return on_group(gs, true, [&](Replicas r) { return light_queue_uninitialized(r, n_queued); });
}

aicb_status aicb_group_light_queue_region(aicb_group_scene *gs, const aicb_aab *region, uint8_t priority) {
    return on_group(gs, true, [&](Replicas r) { return light_queue_region(r, region, priority); });
}

aicb_status aicb_group_light_download_queue(aicb_group_scene *gs, uint8_t *priorities, size_t n_texels, size_t *n_queued) {
    return on_group(gs, false, [&](Replicas r) {
        return light_download_queue(r.scene[0], priorities, n_texels, n_queued);
    });
}

// The calls with inputs or outputs in device memory: device 0's, which every replica reads over peer access (a group
// enables it at creation); each returns once every replica's writes are done.
aicb_status aicb_group_scene_update_cubes_device(aicb_group_scene *gs, const int32_t (*cubes)[3], const uint16_t *ids,
                                                 const uint8_t (*light)[4], size_t n, void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_update_cubes_device(r, cubes, ids, light, n, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_update_region_device(aicb_group_scene *gs, const aicb_aab *region, const uint16_t *ids,
                                                  uint16_t uniform_id, const uint8_t (*light)[4], void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_update_region_device(r, region, ids, uniform_id, light, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_upload_light_device(aicb_group_scene *gs, const uint8_t (*light)[4], size_t n_texels,
                                                 void *stream) {
    return on_group(gs, false, [&](Replicas r) {
        return scenes_upload_light_device(r, light, n_texels, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_scene_download_ids_device(aicb_group_scene *gs, uint16_t *out, size_t n, void *stream) {
    return on_group(gs, false, [&](Replicas r) { return scene_download_ids_device(r, out, n, (cudaStream_t)stream); });
}

aicb_status aicb_group_light_edit_cubes_device(aicb_group_scene *gs, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                               size_t n, size_t *n_changed, void *stream) {
    return on_group(gs, true, [&](Replicas r) {
        return light_edit_cubes_device(r, cubes, new_ids, n, n_changed, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_light_edit_region_device(aicb_group_scene *gs, const aicb_aab *region, const uint16_t *ids,
                                                uint16_t uniform_id, size_t *n_changed, void *stream) {
    return on_group(gs, true, [&](Replicas r) {
        return light_edit_region_device(r, region, ids, uniform_id, n_changed, (cudaStream_t)stream);
    });
}

aicb_status aicb_group_light_download_device(aicb_group_scene *gs, uint8_t (*out)[4], size_t n_texels, void *stream) {
    return on_group(gs, false, [&](Replicas r) { return light_download_device(r, out, n_texels, (cudaStream_t)stream); });
}

aicb_status aicb_group_light_download(aicb_group_scene *gs, int replica, uint8_t (*out)[4], size_t n_texels) {
    return on_group(gs, false, [&](Replicas r) {
        if (replica < 0 || (size_t)replica >= r.n) return aicb_fail(AICB_ERR_INVALID, "no such replica");
        return light_download(r.scene[replica], out, n_texels);
    });
}

// The set of changed cubes is device 0's: device 0 applies every round and the push keeps the replicas identical, so its
// indices and texels are every replica's.
aicb_status aicb_group_light_changes_count(const aicb_group_scene *gs, size_t *n_changed) {
    return on_group(gs, false, [&](Replicas r) { return light_changes_count(r.scene[0], n_changed); });
}

aicb_status aicb_group_light_take_changes(aicb_group_scene *gs, uint32_t *indices, uint8_t (*texels)[4], size_t capacity,
                                          size_t *n_taken) {
    return on_group(gs, false, [&](Replicas r) {
        return light_take_changes(r.scene[0], indices, texels, capacity, n_taken);
    });
}

aicb_status aicb_group_light_stats(const aicb_group_scene *gs, uint64_t out[4]) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    return light_stats(gs->scene[0], out);   // device 0's counters are the group's (light.cu)
}

}  // extern "C"
