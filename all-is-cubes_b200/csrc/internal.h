// internal.h — objects behind the opaque handles of include/aicb200.h (shared by aicb200.cu and light.cu).
#pragma once
#include <mutex>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "trace_kernel.cuh"

aicb_status aicb_fail(aicb_status st, const std::string &msg);
aicb_status aicb_cuda_fail(cudaError_t e, const char *what);
#define CU(call)                                                   \
    do {                                                           \
        cudaError_t e__ = (call);                                  \
        if (e__ != cudaSuccess) return aicb_cuda_fail(e__, #call); \
    } while (0)

struct LightNodePre;    // light_kernel.cuh
struct LightChain;      // light_kernel.cuh
struct LightBlockDev;   // light_kernel.cuh

struct aicb_ctx {
    int device = 0;
    int num_sms = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_k[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // AICB_PROFILE_KERNELS
    bool profile_kernels = false;
    bool stage_timing = true;    // record the per-kernel events of a frame (aicb_render_info::stage_ms)
    void *h_delta = nullptr, *d_delta = nullptr;  // staging of aicb_scene_update_cubes batches (pinned / device)
    size_t h_delta_bytes = 0;
    cudaEvent_t ev_delta = nullptr;
    void *d_debug = nullptr;
    uint32_t debug_warps = 0;
    unsigned int *d_tile_counter = nullptr;
    unsigned long long *d_counters = nullptr;
    float *d_lut = nullptr;
    // staging output buffers (grown on demand)
    void *d_out = nullptr;
    size_t d_out_bytes = 0;
    void *d_aux = nullptr;
    size_t d_aux_bytes = 0;
    // per-task streams between gen -> trace -> resolve, or -> shade -> encode (trace_kernel.cuh)
    void *d_rays = nullptr;
    size_t d_rays_bytes = 0;
    void *d_task_cb = nullptr;   // TaskOut per task
    size_t d_task_cb_bytes = 0;
    void *d_hits = nullptr;      // HitRecord stream (march -> resolve, or march -> shade -> encode)
    size_t d_hits_bytes = 0;
    void *d_contrib = nullptr;   // ShadedHit per hit (shade -> encode): not used by frames that run resolve_kernel
    size_t d_contrib_bytes = 0;
    void *d_bin_list = nullptr;  // task ids of the rays that enter the space, per chord-length bin
    size_t d_bin_list_bytes = 0;
    // LightingOption::Bounce: the same streams for the secondary rays of a chunk, and the per-task bounce state
    void *d_rays2 = nullptr, *d_task_cb2 = nullptr, *d_hits2 = nullptr, *d_contrib2 = nullptr, *d_bin_list2 = nullptr;
    size_t d_rays2_bytes = 0, d_task_cb2_bytes = 0, d_hits2_bytes = 0, d_contrib2_bytes = 0, d_bin_list2_bytes = 0;
    void *d_bounce = nullptr;    // per task: secondary ray (48 B), RNG state (32 B), Rgb sum + steps (16 B), request (4 B)
    size_t d_bounce_bytes = 0;
    uint32_t hits_per_task = 8;  // capacity of the hit stream per ray; raised x4 when a frame overflows it,
    uint32_t shallow_frames = 0; //   lowered again after 16 frames in a row that needed a small fraction of it
    bool deep_frames = false;    // the last frame met >= 3/4 visible surfaces per ray: no resolve_kernel (launch_trace)
    void *h_stage = nullptr;     // pinned staging of frames whose destination is pageable host memory
    size_t h_stage_bytes = 0;
    // the frame whose per-frame scratch (streams, counters, events) is in use
    bool frame_in_flight = false;
    cudaStream_t last_stream = nullptr;
    struct aicb_scene *last_scene = nullptr;
    void *d_task_aux = nullptr;
    size_t d_task_aux_bytes = 0;
    void *d_task_depth = nullptr;   // per task: the UI pass's DepthBuf for the world pass (aicb_render_layers_texture)
    size_t d_task_depth_bytes = 0;
    void *d_task_text = nullptr;    // per task: the UI pass's CharacterBuf for the world pass (aicb_render_layers_terminal)
    size_t d_task_text_bytes = 0;
    // light propagation: the static ray chart (space/light/chart), built and uploaded on first use
    LightNodePre *d_chart_pre = nullptr;   // the chart in depth-first preorder (the lockstep walk)
    uint32_t chart_nodes = 0;
    LightChain *d_chains = nullptr;         // the chart as chains, the per-node cube offsets, the Euler tour of the chain tree
    uchar4 *d_node_rel = nullptr;
    uint16_t *d_euler = nullptr;
    uint32_t n_chains = 0, n_euler = 0;
    float4 *d_term_scratch = nullptr;       // term slots of the chain walk, one set per resident warp
    uint32_t chain_walk_blocks = 0;
    std::mutex mu;
};

struct aicb_scene {
    aicb_ctx *ctx = nullptr;
    aicb::DeviceScene ds{};
    std::vector<uint8_t> block_kind;   // host copy, for update_cubes
    size_t volume = 0;
    uint64_t device_bytes = 0;
    void *d_cells = nullptr;
    uint32_t *d_light = nullptr;
    aicb::BlockRec *d_blocks = nullptr;
    uint16_t *d_bricks = nullptr;
    float4 *d_palette = nullptr;
    float2 *d_pal_tab = nullptr;   // per palette entry: {alpha, log2(1 - alpha) bound} (marching kernel)
    float4 *d_blk_tab = nullptr;   // per block id: that pair and the palette entry of single-voxel blocks
    size_t n_bricks = 0, n_palette = 0;   // elements in d_bricks / d_palette (aicb_scene_update_blocks appends)
    // state of the last asynchronous render
    bool pending = false;
    uint64_t pending_rays = 0;
    uint64_t pending_pixels = 0;
    uint32_t pending_out_bytes_per_pixel = 0;
    bool pending_fused = false;    // shading and encode ran as one kernel (resolve_kernel)
    // ---- light propagation state (light.cu) ----
    std::vector<uint16_t> h_ids;            // host mirror of Space::contents (edits are applied in order on the host)
    std::vector<uint32_t> h_block_light;    // per block: bits 0-5 opaque faces, 6 all-opaque, 7 visible, 8 has emission
    LightBlockDev *d_light_blocks = nullptr;
    uint8_t *d_pending = nullptr;           // per cube: queued priority (0 = not queued) — LightUpdateQueue
    uint32_t *d_list = nullptr;             // work list of one round (cube indices)
    uint32_t *d_new_light = nullptr;        // computed texels of one round
    uint8_t *d_diff = nullptr;              // difference_priority of one round
    uint32_t *d_scalars = nullptr;          // [0] list length, [1] max priority, [2] max diff, [3] updates
    float4 *d_sky_term = nullptr;           // per chart node: the sky light its bundle collects (end_of_ray), for this scene's sky
    uint32_t *d_changed = nullptr;          // list positions whose cube changed by more than one unit this round
    uint32_t *d_tile_max = nullptr;         // per LIGHT_TILE cubes: upper bound of the queued priorities
    uint32_t light_max_distance = 0;
    uint64_t light_stats[4] = {0, 0, 0, 0};  // last propagation: cube updates, chart node visits, rounds queued, device microseconds
};

// Where a frame's kernels store their outputs, and what the layers hand on between passes (launch_trace).
struct Outputs {
    bool full_frame = false;
    uchar4 *srgb8 = nullptr;
    float4 *colorbuf = nullptr;
    uint2 *rgba16f = nullptr;
    double *depth = nullptr;
    aicb_hit *hit = nullptr;
    uint32_t *steps = nullptr;
    int32_t *text = nullptr;
    // layers (renderer.rs:454-478)
    const float4 *in_accum = nullptr;
    float4 *out_accum = nullptr;
    const float *backdrop = nullptr;    // premultiplied light rgb + transmittance
    const float *no_world = nullptr;    // ColorBuf (light rgb, transmittance)
    int force_antialias = -1;           // the world layer's antialiasing option governs every layer's sample points
    // RaytraceToTexture's targets (aicb_render_layers_texture): the TEX kernels; rgba16f takes the colour texels
    bool texture = false;
    const uint32_t *pixel_list = nullptr;   // device: the pixel tasks (y * fb_width + x), or nullptr for every pixel
    uint32_t n_list = 0;
    const double *rays = nullptr;           // device: the tasks of a frame without a camera (origin, direction per ray)
    uint64_t n_rays = 0;
    bool aux = false;                       // the marching kernel that also counts steps and blocks (render_aux)
    float *tex_depth = nullptr;
    const double *in_depth = nullptr;
    double *out_task_depth = nullptr;
    uint32_t tex_layer = aicb::TEX_WORLD;
    float tex_exposure[2] = {1.0f, 1.0f};
    double depth_m[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // the terminal's ColorCharacterBuf (aicb_render_layers_terminal): the TERM kernels; tex_layer names the pass's layer
    bool terminal = false;
    aicb_terminal_pixel *term = nullptr;
    const int2 *in_text = nullptr;
    int2 *out_task_text = nullptr;
    int32_t text_start = AICB_TEXT_EMPTY;
};

// One device's share of a layered frame or texture (aicb_trace_layers): that device's scenes of the layers (nullptr for
// an absent layer; both on one context), its row strips of a whole frame or its range of a pixel list
// (target.pixel_list), and where it stores its outputs.  A single context draws with one part and no strips.
struct LayerPart {
    aicb_scene *world = nullptr, *ui = nullptr;
    aicb_shard shard = {1, 0, 1};
    Outputs target;
};

// One context's share of one pass of a frame (aicb_trace_pass): the scene it traces, its row strips, where it stores,
// a device-to-host copy queued behind every issue (if copy_bytes), and its finished passes' info, summed.
struct FramePart {
    aicb_scene *scene = nullptr;
    const aicb_shard *shard = nullptr;   // nullptr: every row
    Outputs out;
    void *copy_to = nullptr;
    const void *copy_from = nullptr;
    size_t copy_bytes = 0;
    aicb_render_info info{};
};

// aicb200.cu: the layer rules shared by aicb_render_layers_* and aicb_group_render_layers_*.  The layers give the
// cameras and options (their scenes only say which layers exist).  Validation of the arguments of the single-context
// calls; the texture target's exposures and depth transform; the passes of a frame over every part, and the one loop
// that re-issues a pass whose hit stream overflowed (aicb_trace_pass); the one merge of aicb_render_info.  The passes
// need the locks of the parts' contexts.  (C linkage: aicb200.cu defines them among the entry points of the C ABI.)
extern "C" {
aicb_status aicb_check_render_args(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                   const aicb_shard *shard, size_t out_len);
aicb_status aicb_check_layers(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba, size_t out_len,
                              const aicb_layer **lead_out);
aicb_status aicb_check_layers_texture(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba,
                                      const double *depth_transform, const uint32_t *pixels, size_t n_pixels,
                                      const void *out_rgba16f, const float *out_depth, const aicb_layer **lead_out);
void aicb_texture_target(const aicb_layer *world, const aicb_layer *ui, const double *depth_transform, Outputs *target);
aicb_status aicb_trace_layers(const aicb_layer *world, const aicb_layer *ui, const float *backdrop_rgba,
                              const float *no_world_rgba, LayerPart *parts, size_t n_parts, aicb_render_info *total);
aicb_status aicb_trace_pass(FramePart *parts, size_t n_parts, const aicb_camera *cam, const aicb_options *opt,
                            bool want_info);
void aicb_merge_info(aicb_render_info *sum, const aicb_render_info *one, bool same_part);
aicb_status aicb_ensure_device(void **p, size_t *cur, size_t want);
// aicb_scene_update_blocks' validation alone: AICB_OK if that call would accept the update (changes nothing)
aicb_status aicb_scene_check_blocks(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs, size_t n);
}
