// internal.h — objects behind the opaque handles of include/aicb200.h (shared by aicb200.cu, group.cu and light.cu).
#pragma once
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
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
#define TRY(call)                                  \
    do {                                           \
        aicb_status st__ = (call);                 \
        if (st__ != AICB_OK) return st__;          \
    } while (0)

// ---- owners of the library's CUDA resources -----------------------------------------------------------------------
// Each frees what it holds when it is destroyed or replaced, on the current device: whoever destroys an object that
// holds them sets its device first.
struct DeviceMemory {
    static cudaError_t alloc(void **p, size_t bytes) { return cudaMalloc(p, bytes); }
    static void release(void *p) { cudaFree(p); }
};
struct PinnedMemory {
    static cudaError_t alloc(void **p, size_t bytes) { return cudaMallocHost(p, bytes); }
    static void release(void *p) { cudaFreeHost(p); }
};

template <typename Memory>
class Buffer {
public:
    Buffer() = default;
    Buffer(Buffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
    Buffer &operator=(Buffer &&o) noexcept {
        if (this != &o) {
            reset();
            p_ = std::exchange(o.p_, nullptr);
            bytes_ = std::exchange(o.bytes_, 0);
        }
        return *this;
    }
    ~Buffer() { reset(); }

    // At least `bytes`, contents not kept: a smaller buffer is freed first, and stays empty if the allocation fails.
    aicb_status ensure(size_t bytes) {
        if (bytes_ >= bytes) return AICB_OK;
        reset();
        void *p = nullptr;
        CU(Memory::alloc(&p, bytes));
        p_ = p;
        bytes_ = bytes;
        return AICB_OK;
    }
    // Exactly `bytes + pad` bytes, the first `bytes` copied from the host; the buffer changes only if both steps succeed.
    aicb_status upload(const void *src, size_t bytes, size_t pad = 0) {
        Buffer b;
        TRY(b.ensure(bytes + pad));
        CU(cudaMemcpy(b.p_, src, bytes, cudaMemcpyHostToDevice));
        *this = std::move(b);
        return AICB_OK;
    }
    template <typename T>
    aicb_status upload(const std::vector<T> &v) { return upload(v.data(), v.size() * sizeof(T)); }
    void reset() {
        if (p_) Memory::release(p_);
        p_ = nullptr;
        bytes_ = 0;
    }

    template <typename T = void>
    T *get() const { return static_cast<T *>(p_); }
    size_t bytes() const { return bytes_; }
    explicit operator bool() const { return p_ != nullptr; }

private:
    void *p_ = nullptr;
    size_t bytes_ = 0;
};
using DeviceBuffer = Buffer<DeviceMemory>;
using PinnedBuffer = Buffer<PinnedMemory>;

struct EventDestroy {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct StreamDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
using Event = std::unique_ptr<CUevent_st, EventDestroy>;
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;

inline aicb_status create_event(Event &e, unsigned int flags) {
    cudaEvent_t raw = nullptr;
    CU(cudaEventCreateWithFlags(&raw, flags));
    e.reset(raw);
    return AICB_OK;
}

// A cube's cell word: its block id with the block's kind in the top bits (16-bit cells up to 16384 block ids).
inline uint32_t cell_word(uint32_t id, uint8_t kind, bool wide) { return id | ((uint32_t)kind << (wide ? 16 : 14)); }

// One chunk's streams between the kernels of a frame (trace_kernel.cuh): the listed rays' records (array A, then
// array B), a TaskOut per task, the HitRecord stream (march -> resolve, or march -> shade -> encode), a ShadedHit per
// hit (shade -> encode: not used by frames that run resolve_kernel) and the task ids of the rays that enter the space,
// per cost bin (longest first).
struct ChunkStreams {
    DeviceBuffer rays, task_out, hits, shaded, bin_list;

    aicb_status size(uint64_t chunk_cap, uint32_t hit_capacity, bool shade) {
        TRY(rays.ensure(chunk_cap * (sizeof(aicb::RayRecordA) + sizeof(aicb::RayRecordB)) + 16));
        TRY(task_out.ensure(chunk_cap * sizeof(aicb::TaskOut) + 16));
        TRY(hits.ensure((size_t)hit_capacity * sizeof(aicb::HitRecord) + 64));
        if (shade) TRY(shaded.ensure((size_t)hit_capacity * sizeof(aicb::ShadedHit) + 64));
        return bin_list.ensure((size_t)aicb::N_BINS * chunk_cap * 4 + 64);
    }
    void bind(aicb::TraceParams &P, uint64_t chunk_cap, bool shade) const {
        P.rays_a = rays.get<aicb::RayRecordA>();   // 64-byte aligned: cudaMalloc aligns to 256 bytes
        P.rays_b = (aicb::RayRecordB *)(rays.get<char>() + chunk_cap * sizeof(aicb::RayRecordA));
        P.task_out = task_out.get<aicb::TaskOut>();
        P.hits = hits.get<aicb::HitRecord>();
        P.shaded = shade ? shaded.get<aicb::ShadedHit>() : nullptr;
        P.bin_list = bin_list.get<uint32_t>();
    }
    void release_hits() {
        hits.reset();
        shaded.reset();
    }
};

// The view and task layout of a frame whose TaskOut stream primary.task_out holds: a frame with the same key finds each
// task's steps of that frame at its own index, and lists its rays by them (launch_trace).  The zero key holds nothing.
struct RayOrderKey {
    const aicb_scene *scene = nullptr;
    double view[16] = {};   // the camera's inverse_projection_view
    uint32_t fb_width = 0, fb_height = 0, n_samples = 0;
    uint32_t strip_rows = 0, shard_index = 0, shard_count = 0;
    bool operator==(const RayOrderKey &o) const {
        return scene == o.scene && std::memcmp(view, o.view, sizeof view) == 0 && fb_width == o.fb_width &&
               fb_height == o.fb_height && n_samples == o.n_samples && strip_rows == o.strip_rows &&
               shard_index == o.shard_index && shard_count == o.shard_count;
    }
};

// Light propagation's static ray chart (space/light/chart) on a context's device, uploaded on first use (ensure_chart):
// in depth-first preorder (LightNodePre, the lockstep walk); as chains, the per-node cube offsets and the Euler tour of
// the chain tree; and the chain walk's term slots, one set per resident warp of its `walk_blocks`.
struct LightChart {
    DeviceBuffer pre, chains, node_rel, euler, term_scratch;
    uint32_t nodes = 0, n_chains = 0, n_euler = 0, walk_blocks = 0;
};

// A scene's light propagation state (light.cu), in two parts: what every replica's own walks need, and what replica 0
// alone holds and the other replicas' kernels reach through peer pointers.  Between light calls only the queue and the
// set of changed cubes hold anything, so round buffers serve other jobs too (the accessors below).
struct LightState {
    struct Own {
        DeviceBuffer sky_term;         // per chart node: the sky light its bundle collects (end_of_ray) from this sky
        DeviceBuffer overflow;         // list positions whose chain walk overflowed (k_compute_overflow's work)
        DeviceBuffer overflow_count;   // replicas 1..n-1: its length (replica 0's is its LightCounters::overflow)
    } own;
    struct Shared {
        DeviceBuffer pending;          // per cube: queued priority (0 = not queued) — LightUpdateQueue
        DeviceBuffer tile_max;         // per LIGHT_TILE cubes: upper bound of the queued priorities
        DeviceBuffer step;             // a budgeted round's cut (light.cu: LightStepCut), then per tile: its rank base
        DeviceBuffer list, new_light, diff;   // one round's cubes, their computed texels, their difference_priority
        DeviceBuffer counters;         // LightCounters
        DeviceBuffer changes;          // one bit per cube: the set of changed cubes (SpaceChange::CubeLight)
        DeviceBuffer dirty, push_targets;     // a group's: the segments written this round, the other replicas' fields
    } shared;

    // Replica `replica` of `n_replicas`'s part(s) and the scene's light volume, where `s` (this state's scene) has none
    // yet; the scene changes only if every step succeeds.  A new own part takes `terms` as its sky_term (nullptr: the
    // scene's sky, tabulated here).
    aicb_status ensure(aicb_scene *s, size_t replica, size_t n_replicas, const std::vector<float4> *terms);

    // replica 0's overflow list is also the round's `changed` list: its overflow is computed before k_compact_changed
    uint32_t *changed() const { return own.overflow.get<uint32_t>(); }
    // taking the set of changed cubes: the chunks' output positions, then the indices and texels
    uint32_t *chunk_sums() const { return shared.diff.get<uint32_t>(); }
    uint32_t *taken_indices() const { return shared.list.get<uint32_t>(); }
    uint32_t *taken_texels() const { return shared.new_light.get<uint32_t>(); }
};

// Members are destroyed in reverse order of declaration: the stream and events go after the buffers.
struct aicb_ctx {
    int device = 0;
    int num_sms = 0;
    Stream stream;
    Event ev0, ev1;              // the start and end of the context's last frame, and nothing else (wait_context)
    Event ev_light[2];           // the start and end of the last light propagation (light_stats[3])
    Event ev_join;              // this context's stream reached a point another context's stream waits for (fan_in)
    Event ev_k[5];               // AICB_PROFILE_KERNELS
    bool profile_kernels = false;
    bool stage_timing = true;    // record the per-kernel events of a frame (aicb_render_info::stage_ms)
    PinnedBuffer h_delta;        // staging of cube and box updates and edit lists (pinned / device)
    DeviceBuffer d_delta;
    Event ev_delta;
    DeviceBuffer d_debug;
    uint32_t debug_warps = 0;
    // the frame counters (8 x u64), then the per-chunk counters (4 + N_BINS x u32) of the primary and the secondary
    // (Bounce) pass: one memset per frame
    DeviceBuffer d_counters;
    unsigned int *d_tile_counter = nullptr;   // the per-chunk counters in d_counters
    DeviceBuffer d_lut;
    // staging output buffers (grown on demand)
    DeviceBuffer d_out, d_aux;
    // the per-chunk streams of a frame, and with LightingOption::Bounce the same for the secondary rays of a chunk
    // and the per-task bounce state: secondary ray (48 B), RNG state (32 B), Rgb sum + steps (16 B), request (4 B)
    ChunkStreams primary, secondary;
    DeviceBuffer d_bounce;
    uint32_t hits_per_task = 8;  // capacity of the hit stream per ray; raised x4 when a frame overflows it,
    uint32_t shallow_frames = 0; //   lowered again after 16 frames in a row that needed a small fraction of it
    bool deep_frames = false;    // the last frame met >= 3/4 visible surfaces per ray: no resolve_kernel (launch_trace)
    RayOrderKey order_key;       // the frame whose steps primary.task_out holds
    bool ray_ordered = false;    // the frame in flight listed its rays by the previous frame's steps (ray_order)
    PinnedBuffer h_stage;        // pinned staging of frames whose destination is pageable host memory
    // the frame whose per-frame scratch (streams, counters, events) is in use
    bool frame_in_flight = false;
    cudaStream_t last_stream = nullptr;
    struct aicb_scene *last_scene = nullptr;
    DeviceBuffer d_task_aux;
    DeviceBuffer d_task_depth;   // per task: the UI pass's DepthBuf for the world pass (aicb_render_layers_texture)
    DeviceBuffer d_task_text;    // per task: the UI pass's CharacterBuf for the world pass (aicb_render_layers_terminal)
    LightChart light_chart;
    DeviceBuffer d_derive;       // aicb_derive_block_light's per-palette-entry and per-ray terms and its results
    DeviceBuffer d_inputs;       // the device-input calls' scratch: verdict, sorted cube lists, staged entries
    DeviceBuffer d_cursor;       // the host cursor calls' queries and results (cursor.cu), apart from a frame's buffers
    DeviceBuffer d_bodies;       // the host body steps' bodies and results (body.cu)
    DeviceBuffer d_exposure;     // the host exposure steps' states, matrices and exposures (exposure.cu)
    PinnedBuffer h_views;        // the host view batches' camera table, staged (pinned) and on the device
    DeviceBuffer d_views;
    std::mutex mu;
};

// A scene's block table: everything indexed by block id or by pool offset, on the device.  It is written in one way
// (aicb200.cu): definitions are flattened against the table's bookkeeping (SpaceHost), then placed in it, appended at
// the next ids or written over existing ones, with their voxel data appended to the pools.  Elements in use: per block
// id, SpaceHost::block_count(); in the pools, SpaceHost::n_bricks and n_palette.  The buffers may be larger: they grow
// geometrically (grow_buffer), to multiples of 16 bytes.
//
// Each id's extent in both pools is recorded.  A definition written over an id makes its old extents dead; once a
// pool's dead part exceeds its live part, the pool is compacted (compact_pools): its live extents are gathered on the
// device into a buffer of the live size, and every id's records follow them.  A pool thus holds at most twice its live
// data after every call, and each dead element is copied O(1) times, amortised.  A frame's hit records hold absolute
// pool positions, so a compaction runs only once nothing on the context can read the pools (wait_context), as
// aicb_scene_update_blocks waits anyway.
//
// The brick pool holds one word per voxel in one of two forms (trace_kernel.cuh, BRICK_WIDE): u16 words while every
// block's palette has at most 32768 entries, u32 words once a block with more is placed (SpaceHost::wide_bricks).  A
// pool widens in place (widen_bricks_kernel) and stays wide until fill_uniform replaces the table.  Positions and
// lengths in the pool are counted in words of either form.
struct BlockTable {
    struct Extent {
        uint32_t brick_off, n_bricks;   // words of the brick pool
        uint32_t pal_off, n_pal;        // palette entries (two float4 each, and one pal_tab pair)
    };

    DeviceBuffer blocks;    // per block id: BlockRec
    DeviceBuffer blk_tab;   // per block id: the pal_tab pair and the palette entry of single-voxel blocks
    DeviceBuffer light;     // per block id: LightBlockDev (light propagation)
    DeviceBuffer bricks;    // voxel words of the recursive blocks: u16, or u32 if wide
    DeviceBuffer palette;   // two float4 per palette entry
    DeviceBuffer pal_tab;   // per palette entry: {alpha, log2(1 - alpha) bound} (marching kernel)

    // the scene's pointers into the current buffers (LightParams::blocks is read from `light` by light_params)
    void bind(aicb::DeviceScene &ds) const {
        ds.blocks = blocks.get<aicb::BlockRec>();
        ds.blk_tab = blk_tab.get<float4>();
        ds.bricks = bricks.get<uint16_t>();
        ds.palette = palette.get<float4>();
        ds.pal_tab = pal_tab.get<float2>();
    }
};

// What a scene keeps on the host: the Space's size and block ids, the block table's bookkeeping and the light
// settings.  It is the same for every replica of a group scene, so it exists once: a one-context scene owns its own,
// and a group's replica 0 owns the group's, which the other replicas point to (aicb_group_scene_destroy destroys
// replica 0 last).  A call changes it once, after every replica's allocations for the call have succeeded, so a failed
// call never leaves it describing data that a replica's arrays lack.
struct SpaceHost {
    size_t volume = 0;
    std::vector<uint16_t> h_ids;           // mirror of Space::contents (edits are applied in order on the host)
    bool ids_stale = false;                // a device-input call changed the cells since h_ids was last written;
                                           // the first host reader rebuilds it from replica 0's cells (refresh_mirror)
    std::vector<uint8_t> kind;             // per block id: its kind, which its cubes' cell words carry
    std::vector<BlockTable::Extent> extent;   // per block id: its voxel data in the pools
    size_t n_bricks = 0, n_palette = 0;    // brick words, float4s
    size_t dead_bricks = 0, dead_pal = 0;  // of those, brick words and palette entries no id's extent holds
    bool wide_bricks = false;
    uint32_t light_max_distance = 0;
    uint64_t light_stats[4] = {0, 0, 0, 0};  // last propagation: cube updates, chart node visits, rounds queued, device microseconds

    size_t block_count() const { return kind.size(); }
    size_t brick_word_bytes() const { return wide_bricks ? 4 : 2; }
    // what aicb_scene_device_bytes counts of a replica's table: the per-id records and the pools' elements in use,
    // live or dead
    size_t table_bytes() const {
        return block_count() * (sizeof(aicb::BlockRec) + sizeof(float4) + sizeof(LightBlockDev)) +
               n_bricks * brick_word_bytes() + n_palette * sizeof(float4) + n_palette / 2 * sizeof(float2);
    }
};

struct aicb_scene {
    aicb_ctx *ctx = nullptr;
    aicb::DeviceScene ds{};
    std::unique_ptr<SpaceHost> own_host;   // a one-context scene's and a group's replica 0's; nullptr on the others
    SpaceHost *host = nullptr;             // own_host, or replica 0's
    uint64_t device_bytes = 0;   // every array but the block table's (aicb_scene_device_bytes adds table_bytes)
    DeviceBuffer d_cells;
    DeviceBuffer d_light;
    BlockTable blocks;
    // state of the last asynchronous render
    bool pending = false;
    uint64_t pending_rays = 0;
    uint64_t pending_pixels = 0;
    uint64_t pending_out_bytes = 0;   // the frame's output bytes (aicb_render_info::algorithmic_bytes)
    bool pending_fused = false;    // shading and encode ran as one kernel (resolve_kernel)
    LightState light;              // light propagation state (light.cu)
};

// A frame's outputs (launch_trace): `target` is TraceParams::target as the kernels see it, where they store and what
// the layers hand on between passes; the other fields are the host's choices the kernels do not see in it.
struct Outputs {
    aicb::TargetParams target{};
    int kind = aicb::TGT_FRAME;         // the compositing kernels' target: TGT_FRAME, TGT_TEX, TGT_TERM or TGT_VIEWS
    bool full_frame = false;            // outputs at framebuffer positions (TraceParams::out_full_frame)
    bool aux = false;                   // the marching kernel that also counts steps and blocks (a ColorBuf set)
    const double *rays = nullptr;       // device: the tasks of a frame without a camera (origin, direction per ray)
    uint64_t n_rays = 0;
    int force_antialias = -1;           // the world layer's antialiasing option governs every layer's sample points
    uint32_t n_views = 0;               // TGT_VIEWS: the views this frame traces (target.cameras, view_first, view_step)
};

// A frame whose pixel tasks are listed: a pixel list, or a texture target's picks (one task per entry, 32 per warp).
// task_pixel recognises one by its n_list, which is never 0 for these (a call with no pixel or pick returns first).
inline bool listed(const aicb::TargetParams &t) { return t.pixel_list || t.picks != aicb::PICK_LIST; }

// One context's share of a layered frame or texture (aicb_trace_layers): that context's scenes of the layers (nullptr
// for an absent layer; both on one context), its row strips of a whole frame or its range of a pixel list
// (out.target.pixel_list), and where it stores its outputs.
struct LayerPart {
    aicb_scene *world = nullptr, *ui = nullptr;
    aicb_shard shard = {1, 0, 1};
    Outputs out;
};

// One context's share of one pass of a frame (aicb_trace_pass): the scene it traces, its row strips, where it stores,
// and its finished passes' info, summed.
struct FramePart {
    aicb_scene *scene = nullptr;
    const aicb_shard *shard = nullptr;   // nullptr: every row
    Outputs out;
    aicb_render_info info{};
};

// A copy of device 0's outputs to the caller (none if bytes == 0).  With `then`, `to` is the context's pinned staging
// (aicb_ctx::h_stage) and the host copies it on to `then` once the device's copy is done.
struct Delivery {
    void *to;
    const void *from;
    size_t bytes;
    void *then = nullptr;
};

// aicb200.cu: the layer rules of the layered calls.  The layers give the cameras and options (their scenes only say
// which layers exist).  Validation of their arguments; the texture target's exposures and depth transform; the passes
// of a frame over every part, and the one loop that re-issues a pass whose hit stream overflowed and delivers its
// outputs (aicb_trace_pass); the one merge of aicb_render_info.  The passes need the locks of the parts' contexts.
// (C linkage: aicb200.cu defines them among the entry points of the C ABI.)
extern "C" {
aicb_status aicb_check_render_args(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                   const aicb_shard *shard, size_t out_len);
aicb_status aicb_check_layers(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba, size_t out_len,
                              const aicb_layer **lead_out);
aicb_status aicb_check_layers_texture(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba,
                                      const double *depth_transform, const uint32_t *pixels, bool pixels_on_device,
                                      size_t n_pixels, const void *out_rgba16f, const float *out_depth,
                                      const aicb_layer **lead_out);
void aicb_texture_outputs(const aicb_layer *world, const aicb_layer *ui, const double *depth_transform, Outputs *out);
aicb_status aicb_trace_layers(const aicb_layer *world, const aicb_layer *ui, const float *backdrop_rgba,
                              const float *no_world_rgba, LayerPart *parts, size_t n_parts,
                              const std::vector<Delivery> &copies, aicb_render_info *total, cudaStream_t async);
aicb_status aicb_trace_pass(FramePart *parts, size_t n_parts, const aicb_camera *cam, const aicb_options *opt,
                            bool want_info, const std::vector<Delivery> &copies);
void aicb_merge_info(aicb_render_info *sum, const aicb_render_info *one, bool same_part);
}

// aicb200.cu: a block definition as scene creation accepts it (AICB_ERR_INVALID, or AICB_ERR_UNSUPPORTED for a palette
// the brick pool cannot index); and, for a valid one, whether its voxels are Evoxels::single_voxel (voxel_storage.rs:364)
// and that voxel.
aicb_status check_block_desc(const aicb_block_desc &b);
inline bool is_single_voxel(const aicb_block_desc &b) { return b.indices == nullptr || b.resolution == 1; }
aicb_voxel single_voxel_of(const aicb_block_desc &b);

// The check_block_desc checks that read no voxel, in its order: those before its index scan (resolution, n_indices
// against voxel_bounds, the bounds, NULL palettes) and the one after it (a palette over 65536 entries).
aicb_status check_block_scalars(const aicb_block_desc &b);
aicb_status check_block_palette(const aicb_block_desc &b);

// blocks.cu: the light-side record of a block definition.
__host__ __device__ LightBlockDev light_block(const aicb_block_desc &b);

// ---- calls over several contexts ----------------------------------------------------------------------------------
// A device group (group.cu): one context per listed device, device 0's first; every other device reaches device 0's
// memory as a peer.  A group scene: a scene's replica on each of them.
struct aicb_group {
    std::vector<aicb_ctx *> ctx;
    bool light_peers = false;  // device 0 reaches every device too, and the devices have native peer atomics
    ~aicb_group() {
        for (aicb_ctx *c : ctx) aicb_ctx_destroy(c);
    }
};

struct aicb_group_scene {
    aicb_group *group = nullptr;
    std::vector<aicb_scene *> scene;
};

// A call that runs on several contexts lists them device 0's first, with a scene's replica on each (a group scene's
// replicas, in the group's order); a single context is the one-context case and runs as it would alone.  The call
// holds every listed context's lock throughout, and device 0 is where its results are collected.

// Every listed context's lock, for the whole of a call.
struct ContextLocks {
    std::vector<std::unique_lock<std::mutex>> locks;
    explicit ContextLocks(const std::vector<aicb_ctx *> &ctx) {
        for (aicb_ctx *c : ctx) locks.emplace_back(c->mu);
    }
};

// A scene's replicas, one per listed context (ctx[i] is scene[i]'s context), device 0's first.  Every call that acts on
// a scene runs once over them: the one-context entry points (on_scene) and the group's (group.cu) only check the handle,
// take the locks and build the list.  The shared function validates its other arguments against the scene's host part
// (SpaceHost) before anything changes, so a rejected call changes no replica; it changes the host part once, and its
// loops over the replicas do device work only.
struct Replicas {
    aicb_scene *const *scene;
    aicb_ctx *const *ctx;
    size_t n;
};

// The body of a one-context entry point: the handle checked, the context's lock held, `call` run on the scene as a
// list of one.
template <typename Call>
aicb_status on_scene(aicb_scene *s, Call call) {
    if (!s) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    return call(Replicas{&s, &s->ctx, 1});
}

// aicb200.cu: creating a scene and changing it, on each of n contexts (a group scene's replicas hold identical tables,
// cells and light).  The block definitions are validated and flattened once, against the table's bookkeeping, a new
// scene's cells are encoded once and a batch of cubes is deduplicated once; only then does each replica place them on
// its own device.
aicb_status scenes_create(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, aicb_scene **out);
aicb_status scenes_update_cubes(Replicas r, const int32_t (*cubes)[3], const uint16_t *ids, const uint8_t (*light)[4],
                                size_t n);
// The context's pinned staging (h_delta) and its device side (d_delta) with room for a batch of `bytes`, once the
// previous batch (the copy ordered before aicb_ctx::ev_delta) has left it.
aicb_status delta_room(aicb_ctx *ctx, size_t bytes);
// A box of cubes inside a scene's bounds: its lower corner as offsets from the scene's, and its size.
struct RegionBox {
    uint32_t lo[3], size[3];
    size_t volume() const { return (size_t)size[0] * size[1] * size[2]; }
};
// The arguments of the box calls (aicb_scene_update_region, aicb_light_edit_region) against a scene: AICB_ERR_INVALID
// for a NULL region, a region not inside the bounds, or an id (every entry of `ids`, or with ids == nullptr
// `uniform_id`) past the table.
aicb_status check_region(const aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                         RegionBox *box);
// check_region's first part: the region alone, as a box (AICB_ERR_INVALID: NULL, not inside the bounds, too large).
aicb_status check_box(const aicb_scene *s, const aicb_aab *region, RegionBox *box);
// One replica's share of a box call, on its context's device and stream: the ids (2 bytes per cube; none if uniform)
// and `light` (if given and the scene has a light volume) go through the context's staging, or with on_device are
// read where they are (device memory the replica's device reaches), and k_region_cells / k_region_texels write them.  With d_mask (ceil(volume / 32) words) the cubes whose block id changes are marked there
// and counted into *d_n_changed (if given).  The caller records aicb_ctx::ev_delta behind its last kernel, and writes
// the host mirror once (mirror_region).
aicb_status region_cells(aicb_scene *s, const RegionBox &box, const uint16_t *ids, uint16_t uniform_id,
                         const uint8_t (*light)[4], bool on_device, uint32_t *d_mask, uint32_t *d_n_changed);
// The host mirror takes a box call's ids row by row.
void mirror_region(SpaceHost &h, const aicb::DeviceScene &ds, const RegionBox &box, const uint16_t *ids,
                   uint16_t uniform_id);
// SpaceChange::CubeBlock / CubeLight for every cube of a box.
aicb_status scenes_update_region(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                 const uint8_t (*light)[4]);

// ---- scene inputs in device memory (aicb200.cu: the scene calls; light.cu: the light edits) -----------------------
// Inputs are device memory of replica 0's device.  Each call makes replica 0's stream wait for the caller's (`caller`,
// NULL: none) before reading them, and the caller's stream wait for replica 0's before returning, so the caller may
// reuse the buffers for work it queues afterwards.  Validation runs on the device and reduces the inputs to an
// InputVerdict, the only bytes read back before the call decides; on a group the call returns once every replica's
// writes are done.
struct InputVerdict {
    unsigned long long first_bad;   // 2 * i + 0: entry i's cube out of bounds; + 1: its id past the table; ~0: none
                                    // (block definitions, k_block_verdict: i, the first with a bad voxel index)
    uint32_t count;                 // the entries the call applies: distinct cubes, or changing entries
    uint32_t _pad;
};
// The first n listed contexts' streams wait for the caller's (join_caller); the caller's waits for replica 0's
// (release_caller).
aicb_status join_caller(aicb_ctx *const *ctx, size_t n, cudaStream_t caller);
aicb_status release_caller(aicb_ctx *ctx, cudaStream_t caller);
// A cube list (int32[n][3] cubes, u16[n] ids) checked and sorted on replica 0's stream, in its context's d_inputs:
// verdict (first_bad over the list; count 0), each entry's Z-major index in list order (idx), and (keys, vals) the
// indices sorted stably with each entry's list position; `extra` bytes follow for the caller.  The scratch is 256-byte
// aligned piece by piece.  Nothing is read back.
struct CubeList {
    InputVerdict *verdict;
    uint32_t *idx, *keys, *vals;
    void *extra;
    void *temp;              // CUB's scratch, temp_bytes
    size_t temp_bytes;
};
aicb_status stage_cube_list(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *ids, uint32_t n,
                            size_t extra_bytes, size_t temp_bytes, CubeList *l);
// The verdict read back (replica 0's stream synchronised): AICB_ERR_INVALID with the host twin's message for a bad
// entry, else *count.
aicb_status read_verdict(aicb_ctx *ctx, const InputVerdict *d_verdict, uint32_t *count);
// A box call's region (check_box), its arrays' pointers, and its ids (every id < the table's size, checked on the
// device; or uniform_id) against replica 0.  For a non-empty box every replica's stream then waits for the caller's.
aicb_status check_region_device(Replicas r, const aicb_aab *region, const uint16_t *d_ids, uint16_t uniform_id,
                                const uint8_t (*d_light)[4], cudaStream_t caller, RegionBox *box);
// `bytes` of replica 0's d_inputs scratch at `from` copied to replica k's (k > 0), which grows to hold them; the copy
// is queued on replica k's stream.  Returns the copy's address.
aicb_status copy_to_replica(Replicas r, size_t k, const void *from, size_t bytes, void **to);
// Rebuilds the host mirror from replica 0's cells if a device-input call left it stale (one device-to-host copy of
// 2 bytes per cube).
aicb_status refresh_mirror(aicb_scene *s0);
aicb_status scenes_update_cubes_device(Replicas r, const int32_t (*cubes)[3], const uint16_t *ids,
                                       const uint8_t (*light)[4], size_t n, cudaStream_t caller);
aicb_status scenes_update_region_device(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                        const uint8_t (*light)[4], cudaStream_t caller);
aicb_status scenes_upload_light_device(Replicas r, const uint8_t (*light)[4], size_t n_texels, cudaStream_t caller);
aicb_status scene_download_ids_device(Replicas r, uint16_t *out, size_t n, cudaStream_t caller);
aicb_status scenes_update_blocks(Replicas r, const uint16_t *indices, const aicb_block_desc *descs, size_t n_blocks);
aicb_status scenes_append_blocks(Replicas r, const aicb_block_desc *descs, size_t n_blocks);
// The same with each definition's indices and palette in device 0's memory (aicb_scene_update_blocks_device and
// aicb_scene_append_blocks_device).  `flags`: AICB_BLOCKS_*.
aicb_status scenes_blocks_device(Replicas r, bool append, const uint16_t *indices, const aicb_block_desc *descs, size_t n_blocks,
                                 uint32_t flags, cudaStream_t caller);
// scenes_create and scenes_fill_uniform with the block ids, the light and each definition's voxels in device 0's
// memory (aicb_scene_create_device, aicb_scene_fill_uniform_device).  Both return once every replica is complete.
aicb_status scenes_create_device(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, uint32_t flags,
                                 cudaStream_t caller, aicb_scene **out);
aicb_status scenes_fill_uniform_device(Replicas r, const aicb_block_desc *block, uint32_t flags, cudaStream_t caller);

// blocks.cu: one definition whose voxel data is in device memory, as its kernels read it.  aicb200.cu fills it from the
// descriptor and the table's bookkeeping; the kernels take the caller's pointers as they are.
enum : uint32_t { SINGLE_NONE = 0, SINGLE_AIR = 1, SINGLE_FIRST = 2, SINGLE_INDEXED = 3 };   // single_voxel_of
constexpr uint32_t NO_ID = ~0u, NO_WORD = ~0u;
constexpr int32_t LIGHT_GIVEN = -1, LIGHT_SINGLE = -2;
struct DeviceBlockJob {
    const uint16_t *indices;     // the caller's, Z-major (nullptr: none)
    const aicb_voxel *palette;   // the caller's
    uint64_t n_indices;
    uint32_t n_palette;
    uint32_t single;             // SINGLE_*: a single-voxel block's voxel (SINGLE_NONE: not a single voxel)
    uint32_t kind;               // KIND_*
    uint32_t brick_off;          // its brick words' first pool position (recursive)
    uint32_t pal_off;            // its palette entries' first pool position
    uint32_t n_entries;          // palette entries it adds: 0 (air), 1 (single voxel) or n_palette
    uint32_t id;                 // the id whose records it writes; NO_ID: a later definition of the call writes them
    int32_t derived;             // its light record: LIGHT_GIVEN (`light`), LIGHT_SINGLE (its voxel's) or derive's record
    uint32_t light_visible;      // ORed into Derived::visible
    uint32_t masks;              // collision masks (block_words.cuh) of a recursive job's palette (bits 0-1) and of the
                                 // entries its voxels use (bits 2-3), and bit 4 if one of those entries is visible,
                                 // ORed in by k_block_palette and k_block_bricks
    aicb::BlockRec rec;
    LightBlockDev light;
};
// k_block_verdict over jobs [0, n) on `stream`: v->first_bad = the first job with a voxel index past its palette
// (v reset by the caller), kinds[i] = the kind of job i's single voxel.
aicb_status issue_block_verdict(cudaStream_t stream, const DeviceBlockJob *jobs, uint32_t n, uint64_t most_indices,
                                InputVerdict *v, uint8_t *kinds);
// The jobs' brick words, palette entries and per-id records into table `t` (room made, positions in the jobs);
// `derived`: derive's records (device 0's memory), or nullptr.
aicb_status issue_block_data(cudaStream_t stream, DeviceBlockJob *jobs, uint32_t n, uint64_t most_words,
                             uint64_t most_entries, bool wide_bricks, const BlockTable &t,
                             const aicb_block_light *derived);
// Every cell whose id has word[id] != NO_WORD takes that word, on the context's stream.
aicb_status issue_rekind_cells(const aicb_ctx *ctx, void *cells, bool wide, size_t n, const uint32_t *word);
// derive.cu: aicb_derive_block_light's kernels on definitions whose voxel data is in the context's device memory,
// the per-block error words read back.  For each block, rec[i] is its record in *out (device memory, valid until the
// context's next derive), or LIGHT_SINGLE for a single voxel, which is its own derived data.
aicb_status derive_on_device(aicb_ctx *ctx, const aicb_block_desc *descs, size_t n, std::vector<int32_t> *rec,
                             const aicb_block_light **out);
aicb_status scenes_fill_uniform(Replicas r, const aicb_block_desc *block);
aicb_status scenes_upload_light(Replicas r, const uint8_t (*light)[4], size_t n_texels);
// Space::set_physics over the replicas.
aicb_status scenes_set_physics(Replicas r, const aicb_sky *sky, uint8_t light_max_distance);

// group.cu: the order between the listed contexts' streams: every other context's stream waits until device 0's has
// reached this point (fan_out), or device 0's until every other one's has (fan_in, which leaves device 0 current).
aicb_status fan_out(aicb_ctx *const *ctx, size_t n);
aicb_status fan_in(aicb_ctx *const *ctx, size_t n);

// group.cu: the layered calls (aicb_render_layers_* and aicb_group_render_layers_*), which validate, lock, trace the
// layers over one part per context (aicb_trace_layers), collect the parts' outputs on device 0 (a host call's in its
// staging buffer, as the world-only host calls below do), copy them to the caller and fill info.  `world` and `ui`
// are the layers as device 0 sees them; world_scenes / ui_scenes each layer's replica on every one of the n contexts
// (nullptr for an absent layer).
struct LayeredCall {
    const aicb_layer *world, *ui;
    aicb_scene *const *world_scenes, *const *ui_scenes;
    size_t n;
    const float *backdrop_rgba, *no_world_rgba;
};
// A group call's layers as device 0 sees them (`views`, filled here) and each layer's replicas; AICB_ERR_INVALID for
// scenes of two groups.
aicb_status group_call(const aicb_group_layer *world, const aicb_group_layer *ui, const float *backdrop_rgba,
                       const float *no_world_rgba, aicb_layer views[2], LayeredCall *c);
// The contexts of a validated layered call: those of its lead layer's replicas, device 0's first.
std::vector<aicb_ctx *> contexts(const LayeredCall &c, const aicb_layer *lead);
aicb_status layers_srgb8(const LayeredCall &c, uint8_t (*out)[4], size_t out_len, aicb_render_info *info);
aicb_status layers_terminal(const LayeredCall &c, aicb_terminal_pixel *out, size_t out_len, aicb_render_info *info);
aicb_status layers_texture(const LayeredCall &c, const double *depth_transform, const uint32_t *pixels, size_t n_pixels,
                           uint16_t (*out_rgba16f)[4], float *out_depth, aicb_render_info *info);
// The layered calls into the caller's device memory (aicb_render_layers_device, aicb_group_render_layers_device): the
// output set chooses the call (sRGB8, terminal or texture).  With `async` (one context) both passes are issued on
// `stream` (NULL: the context's) and aicb_render_finish finishes them; otherwise the call blocks as the host calls do,
// behind the work queued on `stream` before it, and `stream` waits for the outputs.
aicb_status layers_device(const LayeredCall &c, const double *depth_transform, const uint32_t *d_pixels, size_t n_pixels,
                          const aicb_device_outputs *outs, cudaStream_t stream, bool async, aicb_render_info *info);

// group.cu: one scene's world-only outputs over its replicas (aicb_render_* on one context, aicb_group_render_* and
// aicb_group_trace_rays on a group).  The caller has validated the arguments and holds every context's lock.  A frame
// is cut into interleaved 16-row strips (with `shard`, one context only: that shard's rows, packed); a ray batch into
// contiguous ranges of whole warps (warp_ranges).  Every part stores into device 0's buffers.
//
// A host call draws as a blocking device call does, its outputs (aicb_device_outputs of the caller's host pointers)
// staged in device 0's d_out and copied to the caller (stage_outputs).  `how`: the outputs given; a ColorBuf set, whose
// colorbuf is stored whether or not the caller wants it; an sRGB8 frame that takes a pageable destination through
// the context's pinned staging (the one-context aicb_render_srgb8 only).
enum Staging { STAGE_GIVEN, STAGE_COLORBUF, STAGE_PINNED };
aicb_status frame_host(Replicas r, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                       const aicb_device_outputs &host, Staging how, aicb_render_info *info);
aicb_status rays_host(Replicas r, const double (*origin_dir)[6], const aicb_options *opt,
                      const aicb_device_outputs &host, aicb_render_info *info);
// The outputs of a host call of one output (`field`, at `p`) or of the ColorBuf set, n elements each.
template <typename T>
aicb_device_outputs one_output(T aicb_device_outputs::*field, T p, size_t n) {
    aicb_device_outputs o{};
    o.*field = p;
    o.len = n;
    return o;
}
inline aicb_device_outputs colorbuf_outputs(float (*colorbuf)[4], double *depth, aicb_hit *hit, uint32_t *steps,
                                            size_t n) {
    aicb_device_outputs o{};
    o.colorbuf = colorbuf;
    o.depth = depth;
    o.hit = hit;
    o.steps = steps;
    o.len = n;
    return o;
}
// A batch of views (aicb_render_views_* and aicb_group_render_views_*): n_views cameras of one framebuffer size and
// one set of options, their outputs view-major (view v's pixel (x, y) at v * W * H + y * W + x).
// aicb200.cu: the batch's arguments, before anything is issued (AICB_ERR_INVALID): the options, a camera table for
// n_views > 0, out_len == n_views * W * H, and fewer than 2^32 tasks (task_base is 32-bit).  With `host_cameras`
// the size is the first camera's and every camera must have it (*width / *height are set); otherwise the call gives it.
aicb_status check_views(const aicb_camera *cameras, bool host_cameras, size_t n_views, uint32_t *width,
                        uint32_t *height, const aicb_options *opt, size_t out_len);
// group.cu: a validated batch over the replicas: view v is drawn by replica v mod n, which traces its views' tiles end
// to end as one frame and stores them in device 0's outputs.  The host form stages the caller's outputs (as frame_host
// does) and each replica's copy of the camera table (through its context's pinned h_views into d_views); the device
// form reads a camera table in device 0's memory, and its outputs there, as aicb_group_render_device does.
aicb_status views_host(Replicas r, const aicb_camera *cameras, size_t n_views, const aicb_options *opt,
                       const aicb_device_outputs &host, Staging how, aicb_render_info *info);
aicb_status views_device(Replicas r, const aicb_camera *d_cameras, size_t n_views, uint32_t width, uint32_t height,
                         const aicb_options *opt, const aicb_device_outputs *outs, cudaStream_t caller,
                         aicb_render_info *info);
// The camera a batch's frames are launched with (launch_trace): the framebuffer size alone.
inline aicb_camera views_frame_camera(uint32_t width, uint32_t height) {
    aicb_camera c{};
    c.fb_width = width;
    c.fb_height = height;
    c.exposure = 1.0f;
    return c;
}
// One replica's views of a batch as a frame's outputs: the views r, r + n, ... of the camera table.
inline void views_part(Outputs *o, const aicb_camera *cameras, size_t n_views, size_t replica, size_t n_replicas) {
    o->kind = aicb::TGT_VIEWS;
    o->full_frame = false;
    o->n_views = (uint32_t)((n_views - replica + n_replicas - 1) / n_replicas);
    o->target.cameras = cameras;
    o->target.view_first = (uint32_t)replica;
    o->target.view_step = (uint32_t)n_replicas;
}

// aicb200.cu: render_orthographic over the replicas, validated against replica 0 (the caller holds the locks).
aicb_status ortho_srgb8(Replicas r, uint32_t resolution, uint8_t (*out)[4], size_t out_len, aicb_render_info *info);

// group.cu: n items cut into contiguous ranges of whole 32-item warps, one per context, as even as whole warps allow:
// min(n_ctx, warps) ranges, device 0's first (one empty range for n_items == 0).
struct WarpRange {
    size_t begin, count;
};
std::vector<WarpRange> warp_ranges(size_t n_items, size_t n_ctx);
// aicb200.cu: the outputs of a device-output call (aicb_device_outputs) as a frame's target, validated before anything
// is issued: the set of one host call of `call`'s kind (with need_colorbuf, a ColorBuf set must hold colorbuf, as on a
// group; output_target), and for a caller's pointers (device_target) every pointer memory of `device` and aligned to
// its stores' width (check_device_pointer).
enum DeviceCall { DEV_FRAME, DEV_RAYS, DEV_LAYERS };
aicb_status output_target(const aicb_device_outputs *d, DeviceCall call, bool need_colorbuf, Outputs *o);
aicb_status device_target(const aicb_device_outputs *d, int device, DeviceCall call, bool need_colorbuf, bool peer_ok,
                          Outputs *o);
// aicb200.cu: a frame of no rays on `stream`, for aicb_render_finish to finish (an asynchronous call with nothing to
// trace).
aicb_status issue_empty_frame(aicb_scene *s, const aicb_options *opt, cudaStream_t stream);
// A caller's device buffer: memory of `device`, or with peer_ok of a device it reaches as a peer, aligned to `align`
// bytes (AICB_ERR_INVALID).
aicb_status check_device_pointer(const void *p, int device, bool peer_ok, size_t align, const char *what);
// Device 0's stream waits for the streams of the n listed contexts, then copies the outputs to the caller, and the host
// waits for the copies.
aicb_status deliver(aicb_ctx *const *ctx, size_t n, const std::vector<Delivery> &copies);
// aicb200.cu: GraphicsOptions as every frame call accepts them (AICB_ERR_INVALID otherwise).
aicb_status validate_options(const aicb_options *o);

// light.cu: the light calls over a scene's replicas.  On a group, device 0 has peer access to every other device and
// they to device 0, with native atomics.  After every call the replicas' light volumes are identical.
aicb_status light_fast_evaluate(Replicas r);
aicb_status light_compute(Replicas r, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]);
// compute_light::<LightUpdateCubeInfo>: light_compute's texels on replica 0 alone, with each cube's rays.
aicb_status light_compute_debug(Replicas r, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4], aicb_light_ray *rays,
                                size_t capacity, uint32_t *ray_counts, size_t *n_rays_total);
aicb_status light_evaluate(Replicas r, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                           uint64_t *node_visits);
// update_light_from_queue: relaxation rounds until max_updates cube updates are made or the queue is empty.
aicb_status light_update_from_queue(Replicas r, uint64_t max_updates, aicb_light_updates_info *info);
// Mutation::set x n in list order, without propagation; *n_changed (if given): the entries whose id differs from the
// block their cube holds at that point of the list.
aicb_status light_edit_cubes(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n, size_t *n_changed);
// light_edit_cubes, then evaluate_light(epsilon).
aicb_status light_edit_and_propagate(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n_edits,
                                     uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff);
aicb_status light_relight_blocks(Replicas r, const uint16_t *indices, size_t n, uint8_t epsilon,
                                 uint64_t *updates_done, uint8_t *max_diff);
// Mutation::fill / fill_uniform(region): Mutation::set for every cube of a box, without propagation.
aicb_status light_edit_region(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                              size_t *n_changed);
// The light edits with their lists in device memory (see the device-input calls above).
aicb_status light_edit_cubes_device(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                                    size_t *n_changed, cudaStream_t caller);
aicb_status light_edit_region_device(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                     size_t *n_changed, cudaStream_t caller);
aicb_status light_download_device(Replicas r, uint8_t (*out)[4], size_t n_texels, cudaStream_t caller);
// Space::set_physics on the replicas' light side, once nothing on their contexts reads their arrays: `sky` holds the
// new sky in a DeviceScene's sky fields, which every replica takes; `max_distance` is the new LightPhysics (0 = None).
aicb_status light_set_physics(Replicas r, const aicb::DeviceScene &sky, uint32_t max_distance);
// The light update queue: the load rule of Space::new_from_builder and light_needs_update_in_region over replica 0's
// volume and device 0's queue, and a copy of the queue's bytes.
aicb_status light_queue_uninitialized(Replicas r, size_t *n_queued);
aicb_status light_queue_region(Replicas r, const aicb_aab *region, uint8_t priority);
aicb_status light_download_queue(aicb_scene *s, uint8_t *priorities, size_t n_texels, size_t *n_queued);
aicb_status light_download(aicb_scene *s, uint8_t (*out)[4], size_t n_texels);
// The set of changed cubes of replica 0 (the other replicas' texels are identical); the caller holds the locks.
aicb_status light_changes_count(const aicb_scene *s, size_t *n_changed);
aicb_status light_take_changes(aicb_scene *s, uint32_t *indices, uint8_t (*texels)[4], size_t capacity, size_t *n_taken);
// The counters of replica 0's last light call, which are the group's.
aicb_status light_stats(const aicb_scene *s, uint64_t out[4]);
