// aicb200.cu — host side of libaicb200.so: the C ABI of include/aicb200.h, scene flattening
// (SpaceRaytracer::new, sr.rs:64-88, 543-549) into the two-level brick index, and kernel launch.
//
// No CPU fallback lives here: every compute entry point needs a CUDA device and fails with
// AICB_ERR_CUDA otherwise.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>

#include "internal.h"

using namespace aicb;

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_last_error = "";

aicb_status aicb_fail(aicb_status st, const std::string &msg) {
    g_last_error = msg;
    return st;
}
aicb_status aicb_cuda_fail(cudaError_t e, const char *what) {
    aicb_status st = (e == cudaErrorMemoryAllocation) ? AICB_ERR_OOM : AICB_ERR_CUDA;
    return aicb_fail(st, std::string(what) + ": " + cudaGetErrorString(e));
}
static aicb_status fail(aicb_status st, const std::string &msg) { return aicb_fail(st, msg); }
static aicb_status cuda_fail(cudaError_t e, const char *what) { return aicb_cuda_fail(e, what); }

void aicb_light_scene_init(aicb_scene *s, const aicb_scene_desc *d);   // light.cu
aicb_status aicb_light_scene_upload(aicb_scene *s, const aicb_scene_desc *d);
aicb_status aicb_light_blocks_update(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs, size_t n);
void aicb_light_scene_free(aicb_scene *s);
void aicb_light_ctx_free(aicb_ctx *c);

// PackedLight::some -> scalar_in (light/data.rs:213-217)
static uint8_t scalar_in(float v) {
    float x = std::round(std::log2(v) * 10.0f + 144.0f);
    if (!(x > 0.0f)) return 0;
    if (x >= 255.0f) return 255;
    return (uint8_t)x;
}
static uint32_t texel_some(const float rgb[3]) {
    return (uint32_t)scalar_in(rgb[0]) | ((uint32_t)scalar_in(rgb[1]) << 8) | ((uint32_t)scalar_in(rgb[2]) << 16) |
           (255u << 24);
}
static float ps_mul_h(float a, float b) {
    float v = a * b;
    return (v != v) ? 0.0f : v;
}

// Sky::for_blocks + Sky::mean (sky.rs:45-82)
static void build_block_sky(const aicb_sky &sky, DeviceScene *ds) {
    ds->sky_kind = sky.kind ? 1 : 0;
    std::memcpy(ds->sky_colors, sky.colors, sizeof ds->sky_colors);
    if (!sky.kind) {
        uint32_t t = texel_some(sky.colors[0]);
        for (int f = 0; f < 6; f++) ds->sky_faces[f] = t;
        ds->sky_mean = t;
        return;
    }
    // Face::rotation_from_nz basis (face.rs:395-405): images of +X, +Y, +Z
    static const int basis[6][3][3] = {
        {{0, 1, 0}, {0, 0, 1}, {1, 0, 0}},    // NX RYZX
        {{0, 0, 1}, {1, 0, 0}, {0, 1, 0}},    // NY RZXY
        {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}},    // NZ RXYZ
        {{0, -1, 0}, {0, 0, 1}, {-1, 0, 0}},  // PX RyZx
        {{0, 0, 1}, {-1, 0, 0}, {0, -1, 0}},  // PY RZxy
        {{1, 0, 0}, {0, -1, 0}, {0, 0, -1}},  // PZ RXyz
    };
    static const int pts[4][3] = {{-1, -1, -1}, {-1, 1, -1}, {1, -1, -1}, {1, 1, -1}};
    for (int f = 0; f < 6; f++) {
        float sum[3] = {0, 0, 0};
        for (int k = 0; k < 4; k++) {
            int d[3];
            for (int i = 0; i < 3; i++)
                d[i] = pts[k][0] * basis[f][0][i] + pts[k][1] * basis[f][1][i] + pts[k][2] * basis[f][2][i];
            int idx = ((d[0] >= 0) << 2) + ((d[1] >= 0) << 1) + (d[2] >= 0);
            for (int i = 0; i < 3; i++) sum[i] = sum[i] + sky.colors[idx][i];
        }
        float q[3];
        for (int i = 0; i < 3; i++) q[i] = ps_mul_h(sum[i], 0.25f);
        ds->sky_faces[f] = texel_some(q);
    }
    float sum[3] = {0, 0, 0};
    for (int k = 0; k < 8; k++)
        for (int i = 0; i < 3; i++) sum[i] = sum[i] + sky.colors[k][i];
    float q[3];
    for (int i = 0; i < 3; i++) q[i] = ps_mul_h(sum[i], 1.0f / 8.0f);
    ds->sky_mean = texel_some(q);
}

// component_to_srgb8 (math/color.rs:1038-1054) evaluated with the platform powf — exactly what the
// reference computes on this host — and inverted into thresholds: thr[k] = the smallest non-negative
// f32 whose encoding is >= k.  The device encodes by searching this table.
static uint8_t srgb8_host(float c) {
    float s = (c <= 0.0031308f) ? c * (323.0f / 25.0f) : (211.0f * std::pow(c, 5.0f / 12.0f) - 11.0f) / 200.0f;
    float v = std::round(s * 255.0f);
    if (!(v > 0.0f)) return 0;
    if (v >= 255.0f) return 255;
    return (uint8_t)v;
}
static void build_srgb_thresholds(float *thr) {
    thr[0] = 0.0f;
    for (int k = 1; k < 256; k++) {
        // bisection over the bit patterns of non-negative floats (monotone in value)
        uint32_t lo = 0, hi = 0x7f800000u;  // +0 .. +inf
        while (lo < hi) {
            uint32_t mid = lo + (hi - lo) / 2;
            float f;
            std::memcpy(&f, &mid, 4);
            if (srgb8_host(f) >= k) hi = mid; else lo = mid + 1;
        }
        std::memcpy(&thr[k], &lo, 4);
    }
}

// PackedLight::scalar_in (light/data.rs:213-217) inverted into thresholds with the platform log2f
// (see light_kernel.cuh scalar_in_t): thr[k] = the smallest non-negative f32 whose quantised value is >= k.
static void build_light_thresholds(float *thr) {
    thr[0] = 0.0f;
    for (int k = 1; k < 256; k++) {
        uint32_t lo = 0, hi = 0x7f800000u;
        while (lo < hi) {
            uint32_t mid = lo + (hi - lo) / 2;
            float f;
            std::memcpy(&f, &mid, 4);
            if (scalar_in(f) >= k) hi = mid; else lo = mid + 1;
        }
        std::memcpy(&thr[k], &lo, 4);
    }
}

static bool voxel_invisible(const aicb_voxel &v) {
    return v.rgba[3] == 0.0f && v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f;
}

// TracingBlock::from_block (sr.rs:579-587) for one block definition: its 32-byte record, classification, brick words
// and palette entries (appended to `bricks` / `palette`; the record's offsets are relative to those vectors), plus
// what the marching kernel needs of each surface: {alpha, an upper bound of log2(1 - alpha)} per palette entry.
// Shared by aicb_scene_create and aicb_scene_update_blocks.
static const aicb_voxel AIR_VOXEL = {{0, 0, 0, 0}, {0, 0, 0}, 0};

static float2 surface_entry(float alpha) {
    float l2a;
    if (alpha >= 1.0f) l2a = -INFINITY;
    else if (!(alpha > 0.0f)) l2a = 0.0f;
    else {
        const float unit_t = 1.0f - alpha;   // the f32 value apply_transmittance raises to the span's thickness
        l2a = std::nextafterf((float)std::log2((double)unit_t), INFINITY);
        if (l2a > 0.0f) l2a = 0.0f;
    }
    return make_float2(alpha, l2a);
}

// blk_tab entry of a block: what the marching kernel needs of a single-voxel surface on the Space level.
// `pal_off` indexes `pal_tab`; `pal_base` is added to it for the device-wide palette index.
static float4 block_entry(uint8_t kind, uint32_t pal_off, const std::vector<float2> &pal_tab, uint32_t pal_base) {
    if (kind != KIND_SINGLE) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const float2 e = pal_tab[pal_off];
    const uint32_t pal = pal_off + pal_base;
    float palf;
    std::memcpy(&palf, &pal, 4);
    return make_float4(e.x, e.y, palf, 0.0f);
}

static aicb_status flatten_block(const aicb_block_desc &b, BlockRec &r, uint8_t &kind, std::vector<uint16_t> &bricks,
                                 std::vector<float4> &palette, std::vector<float2> &pal_tab) {
    std::memset(&r, 0, sizeof r);
    const uint32_t res = b.resolution;
    if (res == 0 || (res & (res - 1)) || res > 128) return fail(AICB_ERR_INVALID, "block resolution must be 1..128, power of 2");
    auto push_voxel = [&](const aicb_voxel &v) {
        palette.push_back(make_float4(v.rgba[0], v.rgba[1], v.rgba[2], v.rgba[3]));
        palette.push_back(make_float4(v.emission[0], v.emission[1], v.emission[2], 0.0f));
        pal_tab.push_back(surface_entry(v.rgba[3]));
    };
    bool single = false;
    aicb_voxel sv = AIR_VOXEL;
    if (b.indices == nullptr) {
        single = true;
        if (b.n_palette) {
            if (!b.palette) return fail(AICB_ERR_INVALID, "palette is NULL");
            sv = b.palette[0];
        }
    } else {
        const uint64_t nvox = (uint64_t)b.voxel_bounds.size[0] * b.voxel_bounds.size[1] * b.voxel_bounds.size[2];
        if (nvox != b.n_indices) return fail(AICB_ERR_INVALID, "n_indices does not match voxel_bounds");
        for (int a = 0; a < 3; a++) {
            int64_t lo = b.voxel_bounds.lower[a], hi = lo + (int64_t)b.voxel_bounds.size[a];
            if (lo < 0 || hi > (int64_t)res) return fail(AICB_ERR_INVALID, "voxel_bounds must lie within [0, resolution)^3");
        }
        if (!b.palette && b.n_palette) return fail(AICB_ERR_INVALID, "palette is NULL");
        for (size_t k = 0; k < b.n_indices; k++)
            if (b.indices[k] >= b.n_palette) return fail(AICB_ERR_INVALID, "voxel index out of palette range");
        if (res == 1) {
            // single_voxel_or_palette (voxel_storage.rs:371-383)
            single = true;
            sv = (nvox == 1 && b.voxel_bounds.lower[0] == 0 && b.voxel_bounds.lower[1] == 0 && b.voxel_bounds.lower[2] == 0)
                     ? b.palette[b.indices[0]]
                     : AIR_VOXEL;
        }
    }
    if (b.is_air) {
        kind = KIND_INVISIBLE;
        r.kind_res = KIND_INVISIBLE | (1u << 8);
    } else if (single) {
        kind = voxel_invisible(sv) ? KIND_INVISIBLE : KIND_SINGLE;
        r.kind_res = kind | (1u << 8);
        r.pal_off = (uint32_t)(palette.size() / 2);
        r.vsize[0] = r.vsize[1] = r.vsize[2] = 1;
        push_voxel(sv);
    } else {
        if (b.n_palette > 32768) return fail(AICB_ERR_UNSUPPORTED, "block palettes above 32768 entries are not supported");
        kind = KIND_RECURSIVE;
        r.kind_res = KIND_RECURSIVE | (res << 8);
        for (int a = 0; a < 3; a++) {
            r.vlo[a] = (int16_t)b.voxel_bounds.lower[a];
            r.vsize[a] = (uint16_t)b.voxel_bounds.size[a];
        }
        if (bricks.size() + b.n_indices > 0xffffffffull) return fail(AICB_ERR_INVALID, "brick pool exceeds 2^32 voxels");
        r.brick_off = (uint32_t)bricks.size();
        r.pal_off = (uint32_t)(palette.size() / 2);
        for (size_t k = 0; k < b.n_indices; k++) {
            uint16_t v = b.indices[k];
            bricks.push_back((uint16_t)(v | (voxel_invisible(b.palette[v]) ? 0x8000u : 0u)));
        }
        for (size_t k = 0; k < b.n_palette; k++) push_voxel(b.palette[k]);
    }
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// kernel dispatch
// ---------------------------------------------------------------------------------------------
typedef void (*kernel_fn)(const TraceParams, uint32_t);

template <bool V, bool W, bool AUX>
static kernel_fn kernel_of() {
    return trace_kernel<V, W, AUX>;
}

static kernel_fn select_kernel(bool volumetric, bool wide, bool aux) {
#define PICK(V, W, A) if (volumetric == V && wide == W && aux == A) return kernel_of<V, W, A>();
    PICK(false, false, false) PICK(false, false, true) PICK(false, true, false) PICK(false, true, true)
    PICK(true, false, false) PICK(true, false, true) PICK(true, true, false) PICK(true, true, true)
#undef PICK
    return nullptr;
}

// Launch with (or without) programmatic stream serialization: see grid_dependency_sync() in trace_kernel.cuh.
template <typename... KArgs, typename... Args>
static cudaError_t launch_after(bool overlap, void (*kern)(KArgs...), unsigned grid, unsigned block, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg;
    std::memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3(grid, 1, 1);
    cfg.blockDim = dim3(block, 1, 1);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = overlap ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

// One edited cube of aicb_scene_update_cubes: linear index, encoded cell, optional light texel.
struct CubeDelta {
    uint32_t idx, cell, light, has_light;
};

static __global__ void scatter_cubes_kernel(const CubeDelta *ops, uint32_t n, uint32_t wide, void *cells, uint32_t *light) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CubeDelta op = ops[i];
    if (wide) ((uint32_t *)cells)[op.idx] = op.cell; else ((uint16_t *)cells)[op.idx] = (uint16_t)op.cell;
    if (op.has_light) light[op.idx] = op.light;
}

static aicb_status validate_options(const aicb_options *o) {
    if (!o) return fail(AICB_ERR_INVALID, "options is NULL");
    if (o->fog > AICB_FOG_PHYSICAL) return fail(AICB_ERR_INVALID, "bad fog option");
    if (o->lighting_display > AICB_LIGHT_BOUNCE) return fail(AICB_ERR_INVALID, "bad lighting option");
    if (o->lighting_display == AICB_LIGHT_BOUNCE && o->bounce_samples < 1)
        return fail(AICB_ERR_INVALID, "LightingOption::Bounce needs bounce_samples >= 1");
    if (o->transparency > AICB_TRANSPARENCY_THRESHOLD) return fail(AICB_ERR_INVALID, "bad transparency option");
    if (o->tone_mapping > AICB_TONE_REINHARD) return fail(AICB_ERR_INVALID, "bad tone mapping option");
    if (!(o->view_distance >= 1.0 && o->view_distance <= 10000.0))
        return fail(AICB_ERR_INVALID, "view_distance must be repaired to [1, 10000]");
    return AICB_OK;
}

static uint32_t shard_rows(uint32_t fb_height, const aicb_shard *sh) {
    if (!sh || sh->count <= 1) return fb_height;
    uint32_t sr = sh->strip_rows ? sh->strip_rows : 1;
    uint32_t rows = 0;
    uint32_t n_strips = (fb_height + sr - 1) / sr;
    for (uint32_t s = sh->index; s < n_strips; s += sh->count) {
        uint32_t begin = s * sr;
        uint32_t end = begin + sr < fb_height ? begin + sr : fb_height;
        rows += end - begin;
    }
    return rows;
}

static aicb_status ensure(void **p, size_t *cur, size_t want) {
    if (*cur >= want) return AICB_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cur = 0;
    CU(cudaMalloc(p, want));
    *cur = want;
    return AICB_OK;
}

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
};

// Launches the trace kernel on `stream`. Camera rays when cam != NULL, explicit rays otherwise.
static aicb_status launch_trace(aicb_scene *sc, const aicb_camera *cam, const aicb_options *opt,
                                const aicb_shard *shard, const double *d_rays, uint64_t n_rays, const Outputs &out,
                                bool aux, cudaStream_t stream) {
    aicb_ctx *ctx = sc->ctx;
    TraceParams P;
    std::memset(&P, 0, sizeof P);
    P.scene = sc->ds;
    uint64_t pixels;
    if (cam) {
        std::memcpy(P.m, cam->inverse_projection_view, sizeof P.m);
        P.fb_width = cam->fb_width;
        P.fb_height = cam->fb_height;
        P.exposure = cam->exposure;
        P.local_rows = shard_rows(cam->fb_height, shard);
        if (shard && shard->count > 1) {
            P.strip_rows = shard->strip_rows ? shard->strip_rows : 1;
            P.shard_index = shard->index;
            P.shard_count = shard->count;
        } else {
            P.strip_rows = 1;
            P.shard_index = 0;
            P.shard_count = 1;
        }
        P.tiles_x = (P.fb_width + TILE_W - 1) / TILE_W;
        P.tiles_y = (P.local_rows + TILE_H - 1) / TILE_H;
        if ((uint64_t)P.tiles_x * P.tiles_y * 32 > 0xffffffffull) return fail(AICB_ERR_INVALID, "frame too large");
        P.n_tasks = P.tiles_x * P.tiles_y * 32;
        pixels = (uint64_t)P.fb_width * P.local_rows;
    } else {
        P.exposure = 1.0f;
        P.rays = d_rays;
        P.n_rays = n_rays;
        if (n_rays > 0xffffffffull) return fail(AICB_ERR_INVALID, "too many rays");
        P.tiles_x = (uint32_t)((n_rays + 31) / 32);
        P.tiles_y = 1;
        P.n_tasks = (uint32_t)n_rays;
        P.shard_count = 1;
        P.strip_rows = 1;
        pixels = n_rays;
    }
    P.fog = opt->fog;
    P.lighting = opt->lighting_display;
    P.transparency = opt->transparency;
    P.threshold = opt->transparency_threshold;
    P.antialias = (cam && opt->antialiasing_always) ? 1 : 0;
    if (cam && out.force_antialias >= 0) P.antialias = (uint32_t)out.force_antialias;
    P.tone_mapping = opt->tone_mapping;
    P.maximum_intensity = opt->maximum_intensity;
    P.view_distance = opt->view_distance;
    P.debug_pixel_cost = opt->debug_pixel_cost;
    P.include_sky = opt->include_sky;
    P.out_full_frame = out.full_frame ? 1 : 0;
    P.out_srgb8 = out.srgb8;
    P.out_colorbuf = out.colorbuf;
    P.out_rgba16f = out.rgba16f;
    P.out_depth = out.depth;
    P.out_hit = out.hit;
    P.out_steps = out.steps;
    P.out_text = out.text;
    P.in_accum = out.in_accum;
    P.out_accum = out.out_accum;
    if (out.backdrop) { std::memcpy(P.backdrop, out.backdrop, 16); P.has_backdrop = 1; }
    if (out.no_world) { std::memcpy(P.no_world, out.no_world, 16); P.has_no_world = 1; }
    P.counters = ctx->d_counters;
    P.task_counter = ctx->d_tile_counter;
    {
        const char *e = getenv("AICB_REFILL_THRESHOLD");
        int v = e ? atoi(e) : 4;
        P.refill_threshold = (uint32_t)(v < 1 ? 1 : (v > 32 ? 32 : v));
        const char *e3 = getenv("AICB_TAIL_DIVISOR");
        int v3 = e3 ? atoi(e3) : 2;
        P.tail_divisor = (uint32_t)(v3 < 1 ? 1 : (v3 > 32 ? 32 : v3));
        const char *e2 = getenv("AICB_EVENT_THRESHOLD");
        int v2 = e2 ? atoi(e2) : 24;
        P.event_threshold = (uint32_t)(v2 < 1 ? 1 : (v2 > 32 ? 32 : v2));
    }

    sc->pending = true;
    sc->pending_pixels = pixels;
    sc->pending_rays = pixels * (P.antialias ? 4 : 1);
    sc->pending_out_bytes_per_pixel = out.srgb8 ? 4 : (out.rgba16f ? 8 : 16);

    // ---- the four kernels of a frame, chunked so the per-frame streams stay bounded ---------------------------
    P.n_samples = P.antialias ? 4 : 1;
    const uint64_t total_tasks = (uint64_t)P.n_tasks * P.n_samples;
    // Tasks per chunk (a multiple of 32 * n_samples): at most 4 M (0.6 GB of ray records); fewer when the hit stream
    // has been enlarged after an overflow, so that the per-frame streams stay within ~8 GB however deep the scene is.
    uint64_t CHUNK = (uint64_t)4 << 20;
    {
        const uint64_t per_task = sizeof(RayRecord) + sizeof(TaskOut) + 4 * N_BINS +
                                  (uint64_t)ctx->hits_per_task * (sizeof(HitRecord) + sizeof(ShadedHit));
        uint64_t fit = ((uint64_t)8 << 30) / per_task;
        if (fit < (1u << 17)) fit = 1u << 17;
        if (fit < CHUNK) CHUNK = fit & ~(uint64_t)127;
    }
    const uint64_t chunk_cap = total_tasks < CHUNK ? total_tasks : CHUNK;
    {
        aicb_status st = ensure(&ctx->d_rays, &ctx->d_rays_bytes, chunk_cap * sizeof(RayRecord) + 16);
        if (st != AICB_OK) return st;
        st = ensure(&ctx->d_task_cb, &ctx->d_task_cb_bytes, chunk_cap * sizeof(TaskOut) + 16);
        if (st != AICB_OK) return st;
        uint64_t cap = chunk_cap * ctx->hits_per_task;
        if (cap < (1u << 16)) cap = 1u << 16;
        if (cap > 0xfffffff0ull) cap = 0xfffffff0ull;
        cap &= ~(uint64_t)(HIT_CHUNK - 1);  // lanes take whole chunks of the stream
        P.hit_capacity = (uint32_t)cap;
        st = ensure(&ctx->d_hits, &ctx->d_hits_bytes, cap * sizeof(HitRecord) + 64);
        if (st != AICB_OK) return st;
        st = ensure(&ctx->d_contrib, &ctx->d_contrib_bytes, cap * sizeof(ShadedHit) + 64);
        if (st != AICB_OK) return st;
        st = ensure(&ctx->d_bin_list, &ctx->d_bin_list_bytes, (size_t)N_BINS * chunk_cap * 4 + 64);
        if (st != AICB_OK) return st;
    }
    P.ray_records = (RayRecord *)ctx->d_rays;
    P.task_out = (TaskOut *)ctx->d_task_cb;
    P.hits = (HitRecord *)ctx->d_hits;
    P.shaded = (ShadedHit *)ctx->d_contrib;
    P.hit_counter = ctx->d_tile_counter + 1;
    P.bin_count = ctx->d_tile_counter + 4;
    P.bin_list = (uint32_t *)ctx->d_bin_list;
    P.bin_stride = (uint32_t)chunk_cap;
    P.overflow_flag = (unsigned int *)(ctx->d_counters + 7);
    if (stream != ctx->stream) CU(cudaStreamWaitEvent(stream, ctx->ev_delta, 0));  // pending cube edits
    // The per-frame streams, counters and events belong to the context: a frame issued on another stream than the
    // previous one must not start before that one is through with them.
    if (ctx->frame_in_flight && ctx->last_stream != stream) CU(cudaStreamWaitEvent(stream, ctx->ev1, 0));
    ctx->frame_in_flight = true;
    ctx->last_stream = stream;
    ctx->last_scene = sc;
    CU(cudaMemsetAsync(ctx->d_counters, 0, 8 * sizeof(unsigned long long) + 2 * (4 + N_BINS) * sizeof(unsigned int), stream));
    CU(cudaEventRecord(ctx->ev0, stream));
    if (total_tasks > 0) {
        const bool volumetric = opt->transparency == AICB_TRANSPARENCY_VOLUMETRIC;
        const int lc = opt->lighting_display == AICB_LIGHT_NONE ? LC_NONE
                       : (opt->lighting_display == AICB_LIGHT_FLAT ? LC_FLAT
                          : (opt->lighting_display == AICB_LIGHT_BOUNCE ? LC_BOUNCE : LC_INTERP));
        // LightingOption::Bounce: the secondary rays of a chunk run through the same kernels on a second set of streams
        TraceParams Q;
        const bool bounce = lc == LC_BOUNCE;
        if (bounce) {
            aicb_status st = ensure(&ctx->d_rays2, &ctx->d_rays2_bytes, chunk_cap * sizeof(RayRecord) + 16);
            if (st == AICB_OK) st = ensure(&ctx->d_task_cb2, &ctx->d_task_cb2_bytes, chunk_cap * sizeof(TaskOut) + 16);
            if (st == AICB_OK) st = ensure(&ctx->d_hits2, &ctx->d_hits2_bytes, (size_t)P.hit_capacity * sizeof(HitRecord) + 64);
            if (st == AICB_OK) st = ensure(&ctx->d_contrib2, &ctx->d_contrib2_bytes, (size_t)P.hit_capacity * sizeof(ShadedHit) + 64);
            if (st == AICB_OK) st = ensure(&ctx->d_bin_list2, &ctx->d_bin_list2_bytes, (size_t)N_BINS * chunk_cap * 4 + 64);
            // per task: request (4) + RNG state (32) + Rgb sum and steps (16) + the secondary ray (48)
            if (st == AICB_OK) st = ensure(&ctx->d_bounce, &ctx->d_bounce_bytes, chunk_cap * 100 + 256);
            if (st != AICB_OK) return st;
            char *b = (char *)ctx->d_bounce;
            P.bounce_mode = BOUNCE_PRIMARY;
            P.bounce_samples = opt->bounce_samples;
            P.bounce_rays = (double *)b;                                   // 48 B per task, 16-aligned
            P.bounce_rng = (unsigned long long *)(b + chunk_cap * 48);     // 32 B
            P.bounce_sum = (float4 *)(b + chunk_cap * 80);                 // 16 B
            P.bounce_req = (uint32_t *)(b + chunk_cap * 96);               // 4 B
            Q = P;
            Q.bounce_mode = BOUNCE_SECONDARY;
            Q.rays = P.bounce_rays;
            Q.tiles_y = 1;
            Q.shard_count = 1; Q.shard_index = 0; Q.strip_rows = 1;
            Q.antialias = 0;
            Q.n_samples = 1;
            Q.task_base = 0;
            Q.lighting = AICB_LIGHT_FLAT;      // no bounce budget left (surface.rs:171-176)
            Q.include_sky = 1;                 // surface.rs:159
            Q.exposure = 1.0f;
            Q.out_full_frame = 0;
            Q.out_srgb8 = nullptr; Q.out_colorbuf = nullptr; Q.out_rgba16f = nullptr; Q.out_depth = nullptr;
            Q.out_hit = nullptr; Q.out_steps = nullptr; Q.out_text = nullptr;
            Q.in_accum = nullptr; Q.out_accum = nullptr; Q.has_backdrop = 0; Q.has_no_world = 0;
            Q.ray_records = (RayRecord *)ctx->d_rays2;
            Q.task_out = (TaskOut *)ctx->d_task_cb2;
            Q.hits = (HitRecord *)ctx->d_hits2;
            Q.shaded = (ShadedHit *)ctx->d_contrib2;
            Q.bin_list = (uint32_t *)ctx->d_bin_list2;
            Q.task_counter = ctx->d_tile_counter + (4 + N_BINS);
            Q.hit_counter = Q.task_counter + 1;
            Q.bin_count = Q.task_counter + 4;
            Q.debug_warp_times = nullptr;
        }
        kernel_fn k = select_kernel(volumetric, sc->ds.wide_cells != 0, aux);
        int blocks_per_sm = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k, WARPS_PER_BLOCK * 32, 0));
        if (blocks_per_sm < 1) blocks_per_sm = 1;
        if (const char *e = getenv("AICB_BLOCKS_PER_SM")) {  // experiments: cap the resident marching blocks
            int v = atoi(e);
            if (v >= 1 && v < blocks_per_sm) blocks_per_sm = v;
        }
        for (uint64_t base = 0; base < total_tasks; base += CHUNK) {
            const uint32_t n = (uint32_t)(total_tasks - base < CHUNK ? total_tasks - base : CHUNK);
            P.task_base = (uint32_t)base;
            const bool first = base == 0;  // stage times are reported for the first chunk
            if (!first) CU(cudaMemsetAsync(ctx->d_tile_counter, 0, (4 + N_BINS) * sizeof(unsigned int), stream));
            const bool prof = ctx->profile_kernels && first;
            const bool stage = first && ctx->stage_timing;
            if (stage) cudaEventRecord(ctx->ev_k[0], stream);
            gen_kernel<<<(n + 127) / 128, 128, 0, stream>>>(P, n);
            if (stage) cudaEventRecord(ctx->ev_k[1], stream);
            uint64_t want = ((uint64_t)n + WARPS_PER_BLOCK * 32 - 1) / (WARPS_PER_BLOCK * 32);
            uint64_t grid = (uint64_t)ctx->num_sms * blocks_per_sm;  // persistent: a multiple of the SM count
            if (grid > want) grid = want;
            if (prof) {
                if (!ctx->d_debug) cudaMalloc(&ctx->d_debug, 4 * 8 * (size_t)ctx->num_sms * 64 * WARPS_PER_BLOCK);
                P.debug_warp_times = (unsigned long long *)ctx->d_debug;
                ctx->debug_warps = (uint32_t)grid * WARPS_PER_BLOCK;
            }
            // the frame's kernels follow each other with programmatic dependent launch (no events between them)
            const bool overlap = ctx->dependent_launch && !stage && !prof && !bounce;
            CU(launch_after(overlap, k, (unsigned)grid, WARPS_PER_BLOCK * 32, stream, P, n));
            P.debug_warp_times = nullptr;
            if (stage) cudaEventRecord(ctx->ev_k[2], stream);
            switch (lc) {
                case LC_NONE: CU(launch_after(overlap, shade_kernel<LC_NONE>, ctx->num_sms * 8, 128, stream, P)); break;
                case LC_FLAT: CU(launch_after(overlap, shade_kernel<LC_FLAT>, ctx->num_sms * 8, 128, stream, P)); break;
                case LC_BOUNCE: CU(launch_after(overlap, shade_kernel<LC_BOUNCE>, ctx->num_sms * 8, 128, stream, P)); break;
                default: CU(launch_after(overlap, shade_kernel<LC_INTERP>, ctx->num_sms * 8, 128, stream, P)); break;
            }
            if (bounce) {
                const unsigned tb = (n + 127) / 128;
                bounce_select_kernel<<<tb, 128, 0, stream>>>(P, n);
                Q.n_rays = n;
                Q.n_tasks = n;
                Q.tiles_x = (n + 31) / 32;
                for (uint32_t pass = 0; pass < P.bounce_samples; pass++) {
                    Q.bounce_pass = pass;
                    CU(cudaMemsetAsync(Q.task_counter, 0, (4 + N_BINS) * sizeof(unsigned int), stream));
                    bounce_gen_kernel<<<tb, 128, 0, stream>>>(P, n);
                    gen_kernel<<<tb, 128, 0, stream>>>(Q, n);
                    k<<<(unsigned)grid, WARPS_PER_BLOCK * 32, 0, stream>>>(Q, n);
                    shade_kernel<LC_FLAT><<<ctx->num_sms * 8, 128, 0, stream>>>(Q);
                    encode_kernel<<<tb, 128, 0, stream>>>(Q, n);
                }
                bounce_resolve_kernel<<<tb, 128, 0, stream>>>(P, n);
            }
            if (stage) cudaEventRecord(ctx->ev_k[3], stream);
            const uint32_t n_pixels = n / P.n_samples;
            CU(launch_after(overlap, encode_kernel, (n_pixels + 127) / 128, 128, stream, P, n));
            if (stage) cudaEventRecord(ctx->ev_k[4], stream);
        }
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(ctx->ev1, stream));
    return AICB_OK;
}

static aicb_status finish(aicb_scene *sc, aicb_render_info *info) {
    aicb_ctx *ctx = sc->ctx;
    if (ctx->last_scene != sc)
        return fail(AICB_ERR_BUSY, "the context's last frame belongs to another scene (one frame per context is tracked)");
    CU(cudaEventSynchronize(ctx->ev1));
    ctx->frame_in_flight = false;
    unsigned long long c[8];
    CU(cudaMemcpy(c, ctx->d_counters, sizeof c, cudaMemcpyDeviceToHost));
    sc->pending = false;
    if (ctx->profile_kernels && sc->pending_rays) {  // AICB_PROFILE_KERNELS=1: per-kernel times of the first chunk
        float t[4] = {0, 0, 0, 0};
        for (int i = 0; i < 4; i++) cudaEventElapsedTime(&t[i], ctx->ev_k[i], ctx->ev_k[i + 1]);
        if (ctx->d_debug && ctx->debug_warps) {
            std::vector<unsigned long long> w(4 * (size_t)ctx->debug_warps);
            cudaMemcpy(w.data(), ctx->d_debug, w.size() * 8, cudaMemcpyDeviceToHost);
            unsigned long long t0 = ~0ull, t1 = 0, passes = 0, rays = 0;
            for (uint32_t i = 0; i < ctx->debug_warps; i++) { t0 = std::min(t0, w[4 * i]); t1 = std::max(t1, w[4 * i + 1]); passes += w[4 * i + 2]; rays += w[4 * i + 3]; }
            std::vector<double> ends;
            for (uint32_t i = 0; i < ctx->debug_warps; i++) ends.push_back((double)(w[4 * i + 1] - t0) * 1e-6);
            std::sort(ends.begin(), ends.end());
            auto q = [&](double f) { return ends[(size_t)(f * (ends.size() - 1))]; };
            fprintf(stderr, "[aicb200] march warps %u: end times ms min %.3f p10 %.3f p50 %.3f p90 %.3f p99 %.3f max %.3f; passes/warp %.0f rays %llu\n",
                    ctx->debug_warps, q(0), q(0.1), q(0.5), q(0.9), q(0.99), q(1.0), (double)passes / ctx->debug_warps, rays);
        }
        fprintf(stderr, "[aicb200] gen %.3f ms  march %.3f ms  shade %.3f ms  encode %.3f ms  (hits %llu)\n", t[0], t[1], t[2],
                t[3], c[3]);
    }
    if (c[7]) {  // the hit stream of some chunk overflowed: the frame is incomplete
        if (ctx->hits_per_task >= 2048)
            return fail(AICB_ERR_OOM, "hit stream overflowed at its largest capacity (2048 hit records per ray)");
        ctx->hits_per_task *= 4;
        ctx->shallow_frames = 0;
        return fail(AICB_ERR_RETRY, "hit stream overflowed; its capacity has been raised - re-issue the render");
    }
    // a deep frame must not inflate the scratch buffers for the life of the context: after 16 frames in a row that
    // would have fitted a quarter of the capacity, give the large buffers back
    if (ctx->hits_per_task > 8 && c[3] * 16 < (unsigned long long)sc->pending_rays * ctx->hits_per_task) {
        if (++ctx->shallow_frames >= 16) {
            ctx->hits_per_task /= 4;
            ctx->shallow_frames = 0;
            if (ctx->d_hits) { cudaFree(ctx->d_hits); ctx->d_hits = nullptr; ctx->d_hits_bytes = 0; }
            if (ctx->d_contrib) { cudaFree(ctx->d_contrib); ctx->d_contrib = nullptr; ctx->d_contrib_bytes = 0; }
            if (ctx->d_hits2) { cudaFree(ctx->d_hits2); ctx->d_hits2 = nullptr; ctx->d_hits2_bytes = 0; }
            if (ctx->d_contrib2) { cudaFree(ctx->d_contrib2); ctx->d_contrib2 = nullptr; ctx->d_contrib2_bytes = 0; }
        }
    } else {
        ctx->shallow_frames = 0;
    }
    if (info) {
        std::memset(info, 0, sizeof *info);
        float ms = 0.0f;
        CU(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        info->kernel_ms = ms;
        if (sc->pending_rays && ctx->stage_timing)
            for (int i = 0; i < 4; i++) cudaEventElapsedTime(&info->stage_ms[i], ctx->ev_k[i], ctx->ev_k[i + 1]);
        info->cubes_traced = c[0];
        info->rays = sc->pending_rays;
        for (int i = 0; i < 5; i++) info->counters[i] = c[1 + i];
        info->counters[5] = sc->pending_pixels;
        // SURVEY 8(d): 2 B per outer/inner step, 32 B per surface hit, 4 B per light texel,
        // 32 B per recursive block entered (our BlockRec), + output bytes per pixel
        info->algorithmic_bytes = 2 * c[1] + 2 * c[2] + 32 * c[3] + 4 * c[4] + 32 * c[5] +
                                  (uint64_t)sc->pending_out_bytes_per_pixel * sc->pending_pixels;
        info->flaws = 0;
    }
    sc->pending = false;
    return AICB_OK;
}


// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

uint32_t aicb_abi_version(void) { return AICB_ABI_VERSION; }
const char *aicb_last_error(void) { return g_last_error.c_str(); }

aicb_status aicb_ctx_create(int device_id, aicb_ctx **out) {
    if (!out) return fail(AICB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(AICB_ERR_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") +
                                       (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    if (device_id < 0) CU(cudaGetDevice(&device_id));
    if (device_id >= n) return fail(AICB_ERR_INVALID, "device_id out of range");
    CU(cudaSetDevice(device_id));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device_id));
    if (prop.major != 9 || prop.minor != 0)   // sm_90a code loads on compute capability 9.0 only
        return fail(AICB_ERR_CUDA, "device is not compute capability 9.0; this library is built for sm_90a only");
    aicb_ctx *c = new aicb_ctx();
    c->device = device_id;
    c->num_sms = prop.multiProcessorCount;
    CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CU(cudaEventCreate(&c->ev0));
    CU(cudaEventCreate(&c->ev1));
    c->profile_kernels = getenv("AICB_PROFILE_KERNELS") != nullptr;
    if (const char *e = getenv("AICB_PDL")) c->dependent_launch = atoi(e) != 0;
    for (int i = 0; i < 5; i++) CU(cudaEventCreate(&c->ev_k[i]));
    CU(cudaEventCreateWithFlags(&c->ev_delta, cudaEventDisableTiming));
    // the frame counters (8 x u64) and the per-chunk counters (4 + N_BINS x u32) share one allocation: one memset per frame
    CU(cudaMalloc(&c->d_counters, 8 * sizeof(unsigned long long) + 2 * (4 + N_BINS) * sizeof(unsigned int)));  // + the secondary (Bounce) pass's block
    c->d_tile_counter = (unsigned int *)(c->d_counters + 8);
    // PackedLight decode table (light/data.rs:232-243 scalar_out_arithmetic; table :301-354)
    float lut[768];
    lut[0] = 0.0f;
    for (int i = 1; i < 256; i++) lut[i] = (float)std::exp2((double)(((float)i - 144.0f) / 10.0f));
    build_srgb_thresholds(lut + 256);
    build_light_thresholds(lut + 512);
    CU(cudaMalloc(&c->d_lut, sizeof lut));
    CU(cudaMemcpy(c->d_lut, lut, sizeof lut, cudaMemcpyHostToDevice));
    *out = c;
    return AICB_OK;
}

// Per-kernel event records of a frame (aicb_render_info::stage_ms) are on by default; a caller that only wants frames
// turns them off (five stream operations per frame less).
aicb_status aicb_ctx_stage_timing(aicb_ctx *c, int enable) {
    if (!c) return fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(c->mu);
    c->stage_timing = enable != 0;
    return AICB_OK;
}

void aicb_ctx_destroy(aicb_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->d_out) cudaFree(c->d_out);
    if (c->d_aux) cudaFree(c->d_aux);
    if (c->d_rays) cudaFree(c->d_rays);
    if (c->d_task_cb) cudaFree(c->d_task_cb);
    if (c->d_hits) cudaFree(c->d_hits);
    if (c->d_contrib) cudaFree(c->d_contrib);
    if (c->d_bin_list) cudaFree(c->d_bin_list);
    for (void *q : {c->d_rays2, c->d_task_cb2, c->d_hits2, c->d_contrib2, c->d_bin_list2, c->d_bounce})
        if (q) cudaFree(q);
    if (c->d_debug) cudaFree(c->d_debug);
    if (c->h_delta) cudaFreeHost(c->h_delta);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (c->d_delta) cudaFree(c->d_delta);
    if (c->ev_delta) cudaEventDestroy(c->ev_delta);
    if (c->d_task_aux) cudaFree(c->d_task_aux);
    aicb_light_ctx_free(c);
    if (c->d_lut) cudaFree(c->d_lut);
    if (c->d_counters) cudaFree(c->d_counters);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    for (int i = 0; i < 5; i++) if (c->ev_k[i]) cudaEventDestroy(c->ev_k[i]);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

aicb_status aicb_scene_create(aicb_ctx *ctx, const aicb_scene_desc *d, aicb_scene **out) {
    if (!ctx || !d || !out) return fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    const int64_t LIM = 1 << 30;
    uint64_t volume = 1;
    for (int a = 0; a < 3; a++) {
        int64_t lo = d->bounds.lower[a], hi = lo + (int64_t)d->bounds.size[a];
        if (lo < -LIM || hi > LIM) return fail(AICB_ERR_INVALID, "space bounds must lie within +-2^30");
        volume *= d->bounds.size[a];
        if (volume > (1ull << 31)) return fail(AICB_ERR_INVALID, "space volume exceeds 2^31 cubes");
    }
    if (volume && !d->block_ids) return fail(AICB_ERR_INVALID, "block_ids is NULL");
    if (d->n_blocks > 65536) return fail(AICB_ERR_INVALID, "more than 65536 blocks");
    if (volume && d->n_blocks == 0) return fail(AICB_ERR_INVALID, "non-empty space with an empty block table");

    // ---- flatten the block table --------------------------------------------------------------
    if (d->n_blocks && !d->blocks) return fail(AICB_ERR_INVALID, "blocks is NULL");
    std::vector<BlockRec> recs(d->n_blocks);
    std::vector<uint8_t> kinds(d->n_blocks);
    std::vector<uint16_t> bricks;
    std::vector<float4> palette;
    std::vector<float2> pal_tab;
    std::vector<float4> blk_tab(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) {
        aicb_status fst = flatten_block(d->blocks[i], recs[i], kinds[i], bricks, palette, pal_tab);
        if (fst != AICB_OK) return fst;
        blk_tab[i] = block_entry(kinds[i], recs[i].pal_off, pal_tab, 0);
    }

    aicb_scene *s = new aicb_scene();
    s->ctx = ctx;
    s->volume = (size_t)volume;
    s->block_kind = kinds;
    DeviceScene &ds = s->ds;
    for (int a = 0; a < 3; a++) {
        ds.lo[a] = d->bounds.lower[a];
        ds.size[a] = (int32_t)d->bounds.size[a];
    }
    ds.wide_cells = d->n_blocks > 16384 ? 1 : 0;

    auto cleanup = [&](aicb_status st) {
        aicb_scene_destroy(s);
        return st;
    };
#define CUS(call)                                                        \
    do {                                                                 \
        cudaError_t e__ = (call);                                        \
        if (e__ != cudaSuccess) return cleanup(cuda_fail(e__, #call));   \
    } while (0)

    // ---- cells: block id with its kind in the top bits ------------------------------------------
    if (volume) {
        for (size_t i = 0; i < volume; i++)
            if (d->block_ids[i] >= d->n_blocks) return cleanup(fail(AICB_ERR_INVALID, "block id out of range"));
        if (ds.wide_cells) {
            std::vector<uint32_t> cells(volume);
            for (size_t i = 0; i < volume; i++) cells[i] = d->block_ids[i] | ((uint32_t)kinds[d->block_ids[i]] << 16);
            CUS(cudaMalloc(&s->d_cells, volume * 4));
            CUS(cudaMemcpy(s->d_cells, cells.data(), volume * 4, cudaMemcpyHostToDevice));
            s->device_bytes += volume * 4;
        } else {
            std::vector<uint16_t> cells(volume);
            for (size_t i = 0; i < volume; i++)
                cells[i] = (uint16_t)(d->block_ids[i] | ((uint32_t)kinds[d->block_ids[i]] << 14));
            CUS(cudaMalloc(&s->d_cells, volume * 2));
            CUS(cudaMemcpy(s->d_cells, cells.data(), volume * 2, cudaMemcpyHostToDevice));
            s->device_bytes += volume * 2;
        }
        if (d->light) {
            CUS(cudaMalloc(&s->d_light, volume * 4));
            CUS(cudaMemcpy(s->d_light, d->light, volume * 4, cudaMemcpyHostToDevice));
            s->device_bytes += volume * 4;
        }
    }
    if (!recs.empty()) {
        CUS(cudaMalloc(&s->d_blocks, recs.size() * sizeof(BlockRec)));
        CUS(cudaMemcpy(s->d_blocks, recs.data(), recs.size() * sizeof(BlockRec), cudaMemcpyHostToDevice));
        s->device_bytes += recs.size() * sizeof(BlockRec);
    }
    s->n_bricks = bricks.size();
    s->n_palette = palette.size();
    if (!bricks.empty()) {
        CUS(cudaMalloc(&s->d_bricks, bricks.size() * 2));
        CUS(cudaMemcpy(s->d_bricks, bricks.data(), bricks.size() * 2, cudaMemcpyHostToDevice));
        s->device_bytes += bricks.size() * 2;
    }
    if (!palette.empty()) {
        CUS(cudaMalloc(&s->d_palette, palette.size() * sizeof(float4)));
        CUS(cudaMemcpy(s->d_palette, palette.data(), palette.size() * sizeof(float4), cudaMemcpyHostToDevice));
        s->device_bytes += palette.size() * sizeof(float4);
        CUS(cudaMalloc(&s->d_pal_tab, pal_tab.size() * sizeof(float2)));
        CUS(cudaMemcpy(s->d_pal_tab, pal_tab.data(), pal_tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
        s->device_bytes += pal_tab.size() * sizeof(float2);
    }
    if (!blk_tab.empty()) {
        CUS(cudaMalloc(&s->d_blk_tab, blk_tab.size() * sizeof(float4)));
        CUS(cudaMemcpy(s->d_blk_tab, blk_tab.data(), blk_tab.size() * sizeof(float4), cudaMemcpyHostToDevice));
        s->device_bytes += blk_tab.size() * sizeof(float4);
    }
#undef CUS
    ds.cells = s->d_cells;
    ds.light = s->d_light;
    ds.blocks = s->d_blocks;
    ds.bricks = s->d_bricks;
    ds.palette = s->d_palette;
    ds.blk_tab = s->d_blk_tab;
    ds.pal_tab = s->d_pal_tab;
    ds.tables = ctx->d_lut;
    build_block_sky(d->sky, &ds);
    {
        aicb_status lst = aicb_light_scene_upload(s, d);
        if (lst != AICB_OK) return cleanup(lst);
    }
    *out = s;
    return AICB_OK;
}

void aicb_scene_destroy(aicb_scene *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    if (s->ctx->last_scene == s) {   // its frame (if any) must be through with the scene's arrays
        if (s->ctx->frame_in_flight) cudaEventSynchronize(s->ctx->ev1);
        s->ctx->last_scene = nullptr;
        s->ctx->frame_in_flight = false;
    }
    if (s->d_cells) cudaFree(s->d_cells);
    if (s->d_light) cudaFree(s->d_light);
    if (s->d_blocks) cudaFree(s->d_blocks);
    if (s->d_bricks) cudaFree(s->d_bricks);
    if (s->d_palette) cudaFree(s->d_palette);
    if (s->d_pal_tab) cudaFree(s->d_pal_tab);
    if (s->d_blk_tab) cudaFree(s->d_blk_tab);
    aicb_light_scene_free(s);
    delete s;
}

uint64_t aicb_scene_device_bytes(const aicb_scene *s) { return s ? s->device_bytes : 0; }

aicb_status aicb_scene_update_cubes(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *ids,
                                    const uint8_t (*light)[4], size_t n) {
    if (!s || (n && (!cubes || !ids))) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    if (n == 0) return AICB_OK;
    const DeviceScene &ds = s->ds;
    // validate everything before touching any state
    for (size_t i = 0; i < n; i++) {
        uint32_t dx = (uint32_t)(cubes[i][0] - ds.lo[0]), dy = (uint32_t)(cubes[i][1] - ds.lo[1]),
                 dz = (uint32_t)(cubes[i][2] - ds.lo[2]);
        if (dx >= (uint32_t)ds.size[0] || dy >= (uint32_t)ds.size[1] || dz >= (uint32_t)ds.size[2])
            return fail(AICB_ERR_INVALID, "cube out of bounds");
        if (ids[i] >= s->block_kind.size()) return fail(AICB_ERR_INVALID, "block id out of range");
    }
    // one pinned staging buffer, one H2D copy, one scatter kernel per batch; a cube named twice keeps its
    // last value (the scatter is parallel, so duplicates are resolved here)
    const size_t need = n * sizeof(CubeDelta);
    if (ctx->h_delta_bytes < need) {
        if (ctx->h_delta) { cudaEventSynchronize(ctx->ev_delta); cudaFreeHost(ctx->h_delta); cudaFree(ctx->d_delta); }
        ctx->h_delta = nullptr; ctx->d_delta = nullptr; ctx->h_delta_bytes = 0;
        size_t cap = need < 65536 ? 65536 : need * 2;
        CU(cudaMallocHost(&ctx->h_delta, cap));
        CU(cudaMalloc(&ctx->d_delta, cap));
        ctx->h_delta_bytes = cap;
    }
    CU(cudaEventSynchronize(ctx->ev_delta));  // the previous batch has left the staging buffer
    CubeDelta *ops = (CubeDelta *)ctx->h_delta;
    std::unordered_map<uint32_t, uint32_t> seen;
    seen.reserve(n * 2);
    uint32_t m = 0;
    for (size_t i = 0; i < n; i++) {
        const uint32_t dx = (uint32_t)(cubes[i][0] - ds.lo[0]), dy = (uint32_t)(cubes[i][1] - ds.lo[1]),
                       dz = (uint32_t)(cubes[i][2] - ds.lo[2]);
        const size_t idx = ((size_t)dx * ds.size[1] + dy) * ds.size[2] + dz;
        if (!s->h_ids.empty()) s->h_ids[idx] = ids[i];
        CubeDelta op;
        op.idx = (uint32_t)idx;
        op.cell = ds.wide_cells ? (ids[i] | ((uint32_t)s->block_kind[ids[i]] << 16))
                                : (ids[i] | ((uint32_t)s->block_kind[ids[i]] << 14));
        op.has_light = (light && s->d_light) ? 1u : 0u;
        op.light = 0;
        if (op.has_light) std::memcpy(&op.light, light[i], 4);
        auto it = seen.find(op.idx);
        if (it == seen.end()) { seen.emplace(op.idx, m); ops[m++] = op; } else { ops[it->second] = op; }
    }
    CU(cudaMemcpyAsync(ctx->d_delta, ops, (size_t)m * sizeof(CubeDelta), cudaMemcpyHostToDevice, ctx->stream));
    scatter_cubes_kernel<<<(m + 127) / 128, 128, 0, ctx->stream>>>((const CubeDelta *)ctx->d_delta, m, ds.wide_cells, s->d_cells,
                                                                   s->d_light);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev_delta, ctx->stream));  // renders on other streams wait for it (launch_trace)
    return AICB_OK;  // stream-ordered before any later render of this context
}

// == SpaceChange::BlockEvaluation / BlockIndex (space.rs:1062-1100; UpdatingSpaceRaytracer::update handles them in
// updating.rs:128-150 by re-running TracingBlock::from_block for the changed indices): replace the definition of
// existing block indices.  New voxel data is appended to the brick pool and the palette (the replaced ranges are
// reclaimed by the next aicb_scene_create); cubes that hold a block whose classification changed are re-encoded.
// Does not queue light updates: call aicb_light_evaluate afterwards if the change affects light.
aicb_status aicb_scene_update_blocks(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs, size_t n) {
    if (!s || (n && (!indices || !descs))) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    if (n == 0) return AICB_OK;
    const size_t n_blocks = s->block_kind.size();
    std::vector<BlockRec> recs(n);
    std::vector<uint8_t> kinds(n);
    std::vector<uint16_t> bricks;
    std::vector<float4> palette;
    std::vector<float2> pal_tab;
    // validate and flatten everything before touching any state
    for (size_t i = 0; i < n; i++) {
        if (indices[i] >= n_blocks) return fail(AICB_ERR_INVALID, "block index out of range (new indices need a new scene)");
        aicb_status fst = flatten_block(descs[i], recs[i], kinds[i], bricks, palette, pal_tab);
        if (fst != AICB_OK) return fst;
    }
    if (s->n_bricks + bricks.size() > 0xffffffffull) return fail(AICB_ERR_INVALID, "brick pool exceeds 2^32 voxels");
    bool any_kind_changed = false;
    for (size_t i = 0; i < n; i++) any_kind_changed |= s->block_kind[indices[i]] != kinds[i];
    if (any_kind_changed && s->h_ids.size() != s->volume)
        return fail(AICB_ERR_INVALID, "scene has no host mirror of its block ids");
    CU(cudaDeviceSynchronize());   // nothing (on any stream) may still be reading the arrays that are replaced

    // ---- grow the pools: the new arrays are complete before any pointer of the scene changes ----------------
    const size_t n_pal_old = s->n_palette / 2;   // palette entries (2 x float4 each)
    uint16_t *nb = nullptr;
    float4 *np = nullptr;
    float2 *nt = nullptr;
    auto grow = [&]() -> cudaError_t {
        cudaError_t e;
        if (!bricks.empty()) {
            if ((e = cudaMalloc(&nb, (s->n_bricks + bricks.size()) * 2)) != cudaSuccess) return e;
            if (s->n_bricks && (e = cudaMemcpy(nb, s->d_bricks, s->n_bricks * 2, cudaMemcpyDeviceToDevice)) != cudaSuccess) return e;
            if ((e = cudaMemcpy(nb + s->n_bricks, bricks.data(), bricks.size() * 2, cudaMemcpyHostToDevice)) != cudaSuccess) return e;
        }
        if (!palette.empty()) {
            if ((e = cudaMalloc(&np, (s->n_palette + palette.size()) * sizeof(float4))) != cudaSuccess) return e;
            if (s->n_palette && (e = cudaMemcpy(np, s->d_palette, s->n_palette * sizeof(float4), cudaMemcpyDeviceToDevice)) != cudaSuccess) return e;
            if ((e = cudaMemcpy(np + s->n_palette, palette.data(), palette.size() * sizeof(float4), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
            if ((e = cudaMalloc(&nt, (n_pal_old + pal_tab.size()) * sizeof(float2))) != cudaSuccess) return e;
            if (n_pal_old && (e = cudaMemcpy(nt, s->d_pal_tab, n_pal_old * sizeof(float2), cudaMemcpyDeviceToDevice)) != cudaSuccess) return e;
            if ((e = cudaMemcpy(nt + n_pal_old, pal_tab.data(), pal_tab.size() * sizeof(float2), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
        }
        return cudaSuccess;
    };
    {
        const cudaError_t e = grow();
        if (e != cudaSuccess) {
            if (nb) cudaFree(nb);
            if (np) cudaFree(np);
            if (nt) cudaFree(nt);
            return cuda_fail(e, "growing the brick pool / palette");
        }
    }
    if (nb) {
        if (s->d_bricks) cudaFree(s->d_bricks);
        s->d_bricks = nb;
        s->ds.bricks = nb;
        s->device_bytes += bricks.size() * 2;
    }
    if (np) {
        if (s->d_palette) cudaFree(s->d_palette);
        if (s->d_pal_tab) cudaFree(s->d_pal_tab);
        s->d_palette = np;
        s->ds.palette = np;
        s->d_pal_tab = nt;
        s->ds.pal_tab = nt;
        s->device_bytes += palette.size() * sizeof(float4) + pal_tab.size() * sizeof(float2);
    }
    // ---- patch the block table ------------------------------------------------------------------------------
    std::vector<uint8_t> kind_changed(n_blocks, 0);
    for (size_t i = 0; i < n; i++) {
        BlockRec &r = recs[i];
        const float4 bt = block_entry(kinds[i], r.pal_off, pal_tab, (uint32_t)n_pal_old);
        if (kinds[i] == KIND_RECURSIVE) r.brick_off += (uint32_t)s->n_bricks;
        if (kinds[i] != KIND_INVISIBLE || !descs[i].is_air) r.pal_off += (uint32_t)n_pal_old;
        CU(cudaMemcpy(s->d_blocks + indices[i], &r, sizeof r, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(s->d_blk_tab + indices[i], &bt, sizeof bt, cudaMemcpyHostToDevice));
        if (s->block_kind[indices[i]] != kinds[i]) {
            kind_changed[indices[i]] = 1;
            s->block_kind[indices[i]] = kinds[i];
        }
    }
    s->n_bricks += bricks.size();
    s->n_palette += palette.size();
    // ---- cubes whose block changed its classification carry the kind in their cell word -------------------
    if (any_kind_changed) {
        std::vector<CubeDelta> ops;
        for (size_t idx = 0; idx < s->volume; idx++) {
            const uint16_t id = s->h_ids[idx];
            if (!kind_changed[id]) continue;
            CubeDelta op;
            op.idx = (uint32_t)idx;
            op.cell = s->ds.wide_cells ? (id | ((uint32_t)s->block_kind[id] << 16)) : (id | ((uint32_t)s->block_kind[id] << 14));
            op.light = 0;
            op.has_light = 0;
            ops.push_back(op);
        }
        if (!ops.empty()) {
            CubeDelta *d_ops = nullptr;
            CU(cudaMalloc(&d_ops, ops.size() * sizeof(CubeDelta)));
            cudaError_t e = cudaMemcpy(d_ops, ops.data(), ops.size() * sizeof(CubeDelta), cudaMemcpyHostToDevice);
            if (e == cudaSuccess) {
                scatter_cubes_kernel<<<(unsigned)((ops.size() + 127) / 128), 128, 0, ctx->stream>>>(d_ops, (uint32_t)ops.size(),
                                                                                              s->ds.wide_cells, s->d_cells, s->d_light);
                e = cudaStreamSynchronize(ctx->stream);
            }
            cudaFree(d_ops);
            if (e != cudaSuccess) return cuda_fail(e, "re-encoding cells");
        }
    }
    return aicb_light_blocks_update(s, indices, descs, n);
}

aicb_status aicb_scene_upload_light(aicb_scene *s, const uint8_t (*light)[4], size_t n_texels) {
    if (!s || !light) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n_texels != s->volume) return fail(AICB_ERR_INVALID, "light volume size mismatch");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    if (!s->d_light && s->volume) {
        CU(cudaMalloc(&s->d_light, s->volume * 4));
        s->device_bytes += s->volume * 4;
        s->ds.light = s->d_light;
    }
    if (s->volume) {   // ordered behind queued cube deltas; renders on other streams wait for ev_delta (launch_trace)
        CU(cudaMemcpyAsync(s->d_light, light, s->volume * 4, cudaMemcpyHostToDevice, s->ctx->stream));
        CU(cudaEventRecord(s->ctx->ev_delta, s->ctx->stream));
        CU(cudaStreamSynchronize(s->ctx->stream));
    }
    return AICB_OK;
}

size_t aicb_shard_pixel_count(const aicb_camera *cam, const aicb_shard *shard) {
    if (!cam) return 0;
    return (size_t)cam->fb_width * shard_rows(cam->fb_height, shard);
}

static aicb_status check_render_args(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                     const aicb_shard *shard, size_t out_len) {
    if (!s || !cam) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_status st = validate_options(opt);
    if (st != AICB_OK) return st;
    if (shard && shard->count > 1 && shard->index >= shard->count) return fail(AICB_ERR_INVALID, "shard index >= count");
    if (out_len != aicb_shard_pixel_count(cam, shard))
        return fail(AICB_ERR_INVALID, "Viewport size does not match output buffer length");
    return AICB_OK;
}

aicb_status aicb_render_srgb8(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                              uint8_t (*out)[4], size_t out_len, aicb_render_info *info) {
    aicb_status st = check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    st = ensure(&ctx->d_out, &ctx->d_out_bytes, out_len * 4 + 16);
    if (st != AICB_OK) return st;
    Outputs o;
    o.srgb8 = (uchar4 *)ctx->d_out;
    // A pageable destination (a Rust Vec<[u8; 4]>, a numpy array) cannot take an asynchronous DMA: the frame goes to a
    // pinned staging buffer of the library's and is copied out by the host.  Pinned / registered memory is written directly.
    bool staged = false;
    if (out_len) {
        cudaPointerAttributes attr;
        const cudaError_t pe = cudaPointerGetAttributes(&attr, out);
        if (pe != cudaSuccess) cudaGetLastError();
        staged = pe != cudaSuccess || attr.type == cudaMemoryTypeUnregistered;
        if (staged && ctx->h_stage_bytes < out_len * 4) {
            if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
            ctx->h_stage = nullptr;
            ctx->h_stage_bytes = 0;
            CU(cudaMallocHost(&ctx->h_stage, out_len * 4));
            ctx->h_stage_bytes = out_len * 4;
        }
    }
    void *dst = staged ? ctx->h_stage : (void *)out;
    for (int attempt = 0;; attempt++) {
        st = launch_trace(s, cam, opt, shard, nullptr, 0, o, false, ctx->stream);
        if (st != AICB_OK) return st;
        // the copy is queued behind the frame: one host synchronisation per call
        if (out_len) CU(cudaMemcpyAsync(dst, ctx->d_out, out_len * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        st = finish(s, info);
        if (st != AICB_ERR_RETRY) break;   // (the capacity grows x4 per retry and ends in AICB_ERR_OOM at its cap)
    }
    if (st == AICB_OK && staged && out_len) std::memcpy(out, ctx->h_stage, out_len * 4);
    return st;
}

aicb_status aicb_render_rgba16f(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                                uint16_t (*out)[4], size_t out_len, aicb_render_info *info) {
    aicb_status st = check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    st = ensure(&ctx->d_out, &ctx->d_out_bytes, out_len * 8 + 16);
    if (st != AICB_OK) return st;
    Outputs o;
    o.rgba16f = (uint2 *)ctx->d_out;
    for (int attempt = 0;; attempt++) {
        st = launch_trace(s, cam, opt, shard, nullptr, 0, o, false, ctx->stream);
        if (st != AICB_OK) return st;
        if (out_len) CU(cudaMemcpyAsync(out, ctx->d_out, out_len * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        st = finish(s, info);
        if (st != AICB_ERR_RETRY) break;
    }
    return st;
}

static aicb_status render_aux(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                              const double *d_rays, uint64_t n_rays, float (*out_cb)[4], double *depth, aicb_hit *hit,
                              uint32_t *steps, size_t n, aicb_render_info *info) {
    aicb_ctx *ctx = s->ctx;
    // layout of the aux staging buffer: colorbuf | depth | hit | steps
    size_t off_cb = 0, off_depth = off_cb + n * 16, off_hit = off_depth + n * 8, off_steps = off_hit + n * sizeof(aicb_hit);
    size_t total = off_steps + n * 4 + 16;
    aicb_status st = ensure(&ctx->d_aux, &ctx->d_aux_bytes, total);
    if (st != AICB_OK) return st;
    char *base = (char *)ctx->d_aux;
    Outputs o;
    o.colorbuf = (float4 *)(base + off_cb);
    o.depth = (double *)(base + off_depth);
    o.hit = (aicb_hit *)(base + off_hit);
    o.steps = (uint32_t *)(base + off_steps);
    for (int attempt = 0;; attempt++) {
        st = launch_trace(s, cam, opt, shard, d_rays, n_rays, o, true, ctx->stream);
        if (st != AICB_OK) return st;
        CU(cudaStreamSynchronize(ctx->stream));
        st = finish(s, info);
        if (st != AICB_ERR_RETRY) break;
    }
    if (st != AICB_OK) return st;
    if (n) {
        if (out_cb) CU(cudaMemcpyAsync(out_cb, o.colorbuf, n * 16, cudaMemcpyDeviceToHost, ctx->stream));
        if (depth) CU(cudaMemcpyAsync(depth, o.depth, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (hit) CU(cudaMemcpyAsync(hit, o.hit, n * sizeof(aicb_hit), cudaMemcpyDeviceToHost, ctx->stream));
        if (steps) CU(cudaMemcpyAsync(steps, o.steps, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return AICB_OK;
}

aicb_status aicb_render_colorbuf(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                 const aicb_shard *shard, float (*out_cb)[4], double *depth, aicb_hit *hit,
                                 uint32_t *steps, size_t out_len, aicb_render_info *info) {
    aicb_status st = check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    return render_aux(s, cam, opt, shard, nullptr, 0, out_cb, depth, hit, steps, out_len, info);
}

aicb_status aicb_render_srgb8_device(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                     const aicb_shard *shard, void *d_out, size_t out_len, void *stream) {
    aicb_status st = check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !d_out) return fail(AICB_ERR_INVALID, "d_out is NULL");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    Outputs o;
    o.srgb8 = (uchar4 *)d_out;
    return launch_trace(s, cam, opt, shard, nullptr, 0, o, false, stream ? (cudaStream_t)stream : s->ctx->stream);
}

aicb_status aicb_render_srgb8_device_frame(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                           const aicb_shard *shard, void *d_frame, size_t frame_len, void *stream) {
    if (!s || !cam) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_status st = check_render_args(s, cam, opt, shard, aicb_shard_pixel_count(cam, shard));
    if (st != AICB_OK) return st;
    if (frame_len != (size_t)cam->fb_width * cam->fb_height)
        return fail(AICB_ERR_INVALID, "Viewport size does not match frame buffer length");
    if (frame_len && !d_frame) return fail(AICB_ERR_INVALID, "d_frame is NULL");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    Outputs o;
    o.full_frame = true;
    o.srgb8 = (uchar4 *)d_frame;
    return launch_trace(s, cam, opt, shard, nullptr, 0, o, false, stream ? (cudaStream_t)stream : s->ctx->stream);
}

// ---- full-frame buffers shared between ranks (CUDA IPC) ------------------------------------------
// Behind the pixels of a shared frame sits a small control block in the same allocation (so it travels with the IPC
// handle): two monotonic counters that replace the collective of the delivery step.
//   arrived   += 1 by every rank once its strips of a frame are stored (aicb_frame_signal, after the rank's encode_kernel
//                in stream order; system-scope fence + atomic, so the pixels are visible before the count);
//   consumed  := k by the owner once it is through with frame k (aicb_frame_release);
// aicb_frame_wait_arrived / aicb_frame_wait_consumed are one-thread kernels that spin on them in stream order.  A wait
// gives up after ~2 s (it must never wedge a GPU) and leaves AICB_FRAME_TIMEOUT in the block's third word.
struct FrameControl {
    unsigned int arrived;
    unsigned int consumed;
    unsigned int timed_out;
    unsigned int _pad;
};
static size_t frame_control_offset(size_t n_pixels) { return (n_pixels * 4 + 255) & ~(size_t)255; }

static __global__ void frame_signal_kernel(FrameControl *c) {
    __threadfence_system();
    atomicAdd_system(&c->arrived, 1u);
}
static __global__ void frame_release_kernel(FrameControl *c, unsigned int frame_id) {
    __threadfence_system();
    *(volatile unsigned int *)&c->consumed = frame_id;
    __threadfence_system();
}
static __global__ void frame_wait_kernel(FrameControl *c, int which, unsigned int target) {
    volatile unsigned int *p = which ? &c->consumed : &c->arrived;
    const long long t0 = clock64();
    while ((int)(*p - target) < 0) {
        __nanosleep(200);
        if (clock64() - t0 > 4000000000ll) {   // ~2 s at 2 GHz
            c->timed_out = 1u;
            break;
        }
    }
    __threadfence_system();
}

aicb_status aicb_frame_create(aicb_ctx *ctx, size_t n_pixels, void **d_frame, uint8_t handle_out[64]) {
    if (!ctx || !d_frame || !handle_out) return fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    void *p = nullptr;
    const size_t off = frame_control_offset(n_pixels);
    CU(cudaMalloc(&p, off + 256));
    cudaError_t e = cudaMemset((char *)p + off, 0, 256);
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return cuda_fail(e, "cudaIpcGetMemHandle");
    }
    std::memcpy(handle_out, &h, 64);
    *d_frame = p;
    return AICB_OK;
}

static aicb_status frame_ctl(aicb_ctx *ctx, void *d_frame, size_t n_pixels, void *stream, cudaStream_t *st, FrameControl **c) {
    if (!ctx || !d_frame) return fail(AICB_ERR_INVALID, "NULL argument");
    CU(cudaSetDevice(ctx->device));
    *st = stream ? (cudaStream_t)stream : ctx->stream;
    *c = (FrameControl *)((char *)d_frame + frame_control_offset(n_pixels));
    return AICB_OK;
}
aicb_status aicb_frame_signal(aicb_ctx *ctx, void *d_frame, size_t n_pixels, void *stream) {
    cudaStream_t st;
    FrameControl *c;
    aicb_status r = frame_ctl(ctx, d_frame, n_pixels, stream, &st, &c);
    if (r != AICB_OK) return r;
    frame_signal_kernel<<<1, 1, 0, st>>>(c);
    CU(cudaGetLastError());
    return AICB_OK;
}
aicb_status aicb_frame_release(aicb_ctx *ctx, void *d_frame, size_t n_pixels, uint32_t frame_id, void *stream) {
    cudaStream_t st;
    FrameControl *c;
    aicb_status r = frame_ctl(ctx, d_frame, n_pixels, stream, &st, &c);
    if (r != AICB_OK) return r;
    frame_release_kernel<<<1, 1, 0, st>>>(c, frame_id);
    CU(cudaGetLastError());
    return AICB_OK;
}
aicb_status aicb_frame_wait_arrived(aicb_ctx *ctx, void *d_frame, size_t n_pixels, uint32_t count, void *stream) {
    cudaStream_t st;
    FrameControl *c;
    aicb_status r = frame_ctl(ctx, d_frame, n_pixels, stream, &st, &c);
    if (r != AICB_OK) return r;
    frame_wait_kernel<<<1, 1, 0, st>>>(c, 0, count);
    CU(cudaGetLastError());
    return AICB_OK;
}
aicb_status aicb_frame_wait_consumed(aicb_ctx *ctx, void *d_frame, size_t n_pixels, uint32_t frame_id, void *stream) {
    cudaStream_t st;
    FrameControl *c;
    aicb_status r = frame_ctl(ctx, d_frame, n_pixels, stream, &st, &c);
    if (r != AICB_OK) return r;
    frame_wait_kernel<<<1, 1, 0, st>>>(c, 1, frame_id);
    CU(cudaGetLastError());
    return AICB_OK;
}
// 1 if a wait on this frame ever gave up (a rank died or never rendered its strips).
aicb_status aicb_frame_timed_out(aicb_ctx *ctx, void *d_frame, size_t n_pixels, uint32_t *out) {
    if (!ctx || !d_frame || !out) return fail(AICB_ERR_INVALID, "NULL argument");
    CU(cudaSetDevice(ctx->device));
    FrameControl h;
    CU(cudaMemcpy(&h, (char *)d_frame + frame_control_offset(n_pixels), sizeof h, cudaMemcpyDeviceToHost));
    *out = h.timed_out;
    return AICB_OK;
}

aicb_status aicb_frame_open(aicb_ctx *ctx, const uint8_t handle[64], void **d_frame) {
    if (!ctx || !handle || !d_frame) return fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, 64);
    // opened on THIS rank's device: lazily enables peer access to the exporting GPU (NVLink P2P)
    CU(cudaIpcOpenMemHandle(d_frame, h, cudaIpcMemLazyEnablePeerAccess));
    return AICB_OK;
}

aicb_status aicb_frame_close(aicb_ctx *ctx, void *d_frame, int opened) {
    if (!ctx || !d_frame) return fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    if (opened) CU(cudaIpcCloseMemHandle(d_frame)); else CU(cudaFree(d_frame));
    return AICB_OK;
}

aicb_status aicb_frame_read(aicb_ctx *ctx, const void *d_frame, uint8_t (*out)[4], size_t n_pixels, void *stream) {
    if (!ctx || !d_frame || !out) return fail(AICB_ERR_INVALID, "NULL argument");
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    CU(cudaMemcpyAsync(out, d_frame, n_pixels * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return AICB_OK;
}

// == print_space's per-pixel CharacterBuf (raytracer/text.rs:52-123, 139-180): which block each pixel shows.
aicb_status aicb_render_text(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, int32_t *out, size_t out_len,
                             aicb_render_info *info) {
    aicb_status st = check_render_args(s, cam, opt, nullptr, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    st = ensure(&ctx->d_aux, &ctx->d_aux_bytes, out_len * 4 + 16);
    if (st != AICB_OK) return st;
    Outputs o;
    o.text = (int32_t *)ctx->d_aux;
    for (;;) {
        st = launch_trace(s, cam, opt, nullptr, nullptr, 0, o, false, ctx->stream);
        if (st != AICB_OK) return st;
        CU(cudaStreamSynchronize(ctx->stream));
        st = finish(s, info);
        if (st != AICB_ERR_RETRY) break;
    }
    if (st != AICB_OK) return st;
    if (out_len) CU(cudaMemcpy(out, ctx->d_aux, out_len * 4, cudaMemcpyDeviceToHost));
    return AICB_OK;
}

// == RtScene::trace_ray_through_layers for every pixel + the encoder of draw_rgba (renderer.rs:454-478, 287-291):
// the UI layer's Space is traced first (its own camera, no sky), the backdrop colour is added, the world layer
// continues in the same accumulator (its rays start opaque where the UI covered the pixel), and a pixel that is not
// opaque in the end — there is no world — is painted NO_WORLD_TO_SHOW.  The world layer's options choose the sample
// points (antialiasing) and the post-processing.
aicb_status aicb_render_layers_srgb8(const aicb_layer *world, const aicb_layer *ui, const float backdrop_rgba[4],
                                     const float no_world_rgba[4], uint8_t (*out)[4], size_t out_len,
                                     aicb_render_info *info) {
    const bool have_world = world && world->scene, have_ui = ui && ui->scene;
    if (!have_world && !have_ui && !no_world_rgba) return fail(AICB_ERR_INVALID, "no layer to draw");
    const aicb_layer *lead = have_world ? world : ui;
    if (!lead || !lead->camera || !lead->options) return fail(AICB_ERR_INVALID, "a layer needs its camera and options");
    if (have_ui && (!ui->camera || !ui->options)) return fail(AICB_ERR_INVALID, "a layer needs its camera and options");
    if (have_world && have_ui) {
        if (world->scene->ctx != ui->scene->ctx) return fail(AICB_ERR_INVALID, "the layers must live on one context");
        if (world->camera->fb_width != ui->camera->fb_width || world->camera->fb_height != ui->camera->fb_height)
            return fail(AICB_ERR_INVALID, "the layers' cameras must share the framebuffer size");
    }
    aicb_status st = check_render_args(lead->scene, lead->camera, lead->options, nullptr, out_len);
    if (st != AICB_OK) return st;
    if (have_ui && have_world) {
        st = validate_options(ui->options);
        if (st != AICB_OK) return st;
    }
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    aicb_ctx *ctx = lead->scene->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    st = ensure(&ctx->d_out, &ctx->d_out_bytes, out_len * 4 + 16);
    if (st != AICB_OK) return st;
    const int aa = lead->options->antialiasing_always ? 1 : 0;
    // Rgba -> ColorBuf (raytracer_components.rs:111-120): premultiplied light, transmittance = 1 - alpha
    float backdrop[4] = {0, 0, 0, 1}, no_world[4] = {0, 0, 0, 0};
    const bool have_backdrop = backdrop_rgba && !(backdrop_rgba[0] == 0.0f && backdrop_rgba[1] == 0.0f &&
                                                   backdrop_rgba[2] == 0.0f && backdrop_rgba[3] == 0.0f);
    if (have_backdrop) {
        for (int i = 0; i < 3; i++) backdrop[i] = backdrop_rgba[i] * backdrop_rgba[3];
        backdrop[3] = 1.0f - backdrop_rgba[3];
    }
    if (no_world_rgba) {
        for (int i = 0; i < 3; i++) no_world[i] = no_world_rgba[i] * no_world_rgba[3];
        no_world[3] = 1.0f - no_world_rgba[3];
    }
    aicb_render_info total;
    std::memset(&total, 0, sizeof total);
    auto add_info = [&](const aicb_render_info &one) {
        total.cubes_traced += one.cubes_traced;
        total.rays += one.rays;
        total.algorithmic_bytes += one.algorithmic_bytes;
        for (int k = 0; k < 6; k++) total.counters[k] += one.counters[k];
        total.kernel_ms += one.kernel_ms;
        for (int k = 0; k < 4; k++) total.stage_ms[k] += one.stage_ms[k];
        total.flaws |= one.flaws;
    };
    auto run = [&](aicb_scene *sc, const aicb_camera *cam, const aicb_options *opt, const Outputs &o) -> aicb_status {
        for (;;) {
            aicb_status r = launch_trace(sc, cam, opt, nullptr, nullptr, 0, o, false, ctx->stream);
            if (r != AICB_OK) return r;
            CU(cudaStreamSynchronize(ctx->stream));
            aicb_render_info one;
            r = finish(sc, &one);
            if (r == AICB_ERR_RETRY) continue;
            if (r == AICB_OK) add_info(one);
            return r;
        }
    };
    if (have_ui && have_world) {
        const size_t n_tasks = (((size_t)ui->camera->fb_width + TILE_W - 1) / TILE_W) * (((size_t)ui->camera->fb_height + TILE_H - 1) / TILE_H) * 32 * (aa ? 4 : 1);
        st = ensure(&ctx->d_task_aux, &ctx->d_task_aux_bytes, n_tasks * sizeof(float4) + 16);
        if (st != AICB_OK) return st;
        aicb_options ui_opt = *ui->options;
        ui_opt.include_sky = 0;   // ui.trace_ray(.., false)
        Outputs o1;
        o1.out_accum = (float4 *)ctx->d_task_aux;
        o1.backdrop = have_backdrop ? backdrop : nullptr;
        o1.force_antialias = aa;
        st = run(ui->scene, ui->camera, &ui_opt, o1);
        if (st != AICB_OK) return st;
        aicb_options w_opt = *world->options;
        w_opt.include_sky = 1;    // world.trace_ray(.., true)
        Outputs o2;
        o2.srgb8 = (uchar4 *)ctx->d_out;
        o2.in_accum = (const float4 *)ctx->d_task_aux;
        o2.no_world = no_world_rgba ? no_world : nullptr;
        st = run(world->scene, world->camera, &w_opt, o2);
    } else if (have_world) {
        aicb_options w_opt = *world->options;
        w_opt.include_sky = 1;
        Outputs o;
        o.srgb8 = (uchar4 *)ctx->d_out;
        // without a UI Space the backdrop is still added in front of the world: as the accumulator's starting value
        if (have_backdrop) {
            const size_t n_tasks = (((size_t)world->camera->fb_width + TILE_W - 1) / TILE_W) * (((size_t)world->camera->fb_height + TILE_H - 1) / TILE_H) * 32 * (aa ? 4 : 1);
            st = ensure(&ctx->d_task_aux, &ctx->d_task_aux_bytes, n_tasks * sizeof(float4) + 16);
            if (st != AICB_OK) return st;
            std::vector<float4> init(n_tasks, make_float4(backdrop[0] * 1.0f, backdrop[1] * 1.0f, backdrop[2] * 1.0f, 1.0f * backdrop[3]));
            CU(cudaMemcpy(ctx->d_task_aux, init.data(), n_tasks * sizeof(float4), cudaMemcpyHostToDevice));
            o.in_accum = (const float4 *)ctx->d_task_aux;
        }
        o.no_world = no_world_rgba ? no_world : nullptr;
        st = run(world->scene, world->camera, &w_opt, o);
    } else {
        aicb_options ui_opt = *ui->options;
        ui_opt.include_sky = 0;
        Outputs o;
        o.srgb8 = (uchar4 *)ctx->d_out;
        o.backdrop = have_backdrop ? backdrop : nullptr;
        o.no_world = no_world_rgba ? no_world : nullptr;
        st = run(ui->scene, ui->camera, &ui_opt, o);
    }
    if (st != AICB_OK) return st;
    if (out_len) CU(cudaMemcpy(out, ctx->d_out, out_len * 4, cudaMemcpyDeviceToHost));
    if (info) *info = total;
    return AICB_OK;
}

// == render_orthographic (raytracer/ortho.rs:30-84) with MultiOrthoCamera (:143-199) / OrthoCamera (:209-297): five
// pixel-perfect axis-aligned views (top, left, front, right, bottom) of the whole Space in one image, `resolution`
// pixels per cube, GraphicsOptions::UNALTERED_COLORS, one ray per pixel, Rgba::from(ColorBuf).to_srgb8() (no
// post-processing); pixels between the views are transparent.  The reference traces AaRays; its AxisAlignedRaycaster
// "produces exactly the same RaycastSteps" as the Raycaster on Ray::from(aa_ray) (raycast/axis_aligned.rs:8-9 and its
// tests), so the rays go through the general marching kernel.
static void ortho_views(const DeviceScene &ds, uint32_t res, uint32_t vw[5], uint32_t vh[5], uint32_t ox[5], uint32_t oy[5],
                        uint32_t *W, uint32_t *H) {
    const uint32_t sx = (uint32_t)ds.size[0] * res, sy = (uint32_t)ds.size[1] * res, sz = (uint32_t)ds.size[2] * res;
    // order: top (PY), left (NX), front (PZ), right (PX), bottom (NY)
    vw[0] = sx; vh[0] = sz;
    vw[1] = sz; vh[1] = sy;
    vw[2] = sx; vh[2] = sy;
    vw[3] = sz; vh[3] = sy;
    vw[4] = sx; vh[4] = sz;
    ox[0] = vw[1] + 1; oy[0] = 0;
    ox[1] = 0; oy[1] = vh[0] + 1;
    ox[2] = vw[1] + 1; oy[2] = vh[0] + 1;
    ox[3] = vw[1] + vw[2] + 2; oy[3] = vh[0] + 1;
    ox[4] = vw[1] + 1; oy[4] = vh[0] + vh[2] + 2;
    uint32_t w = 0, h = 0;
    for (int i = 0; i < 5; i++) {
        w = std::max(w, ox[i] + vw[i]);
        h = std::max(h, oy[i] + vh[i]);
    }
    *W = w;
    *H = h;
}

aicb_status aicb_ortho_image_size(const aicb_scene *s, uint32_t resolution, uint32_t *width, uint32_t *height) {
    if (!s || !width || !height) return fail(AICB_ERR_INVALID, "NULL argument");
    if (resolution == 0 || (resolution & (resolution - 1)) || resolution > 128)
        return fail(AICB_ERR_INVALID, "resolution must be a power of two up to 128");
    uint32_t vw[5], vh[5], ox[5], oy[5];
    ortho_views(s->ds, resolution, vw, vh, ox, oy, width, height);
    return AICB_OK;
}

aicb_status aicb_render_orthographic(aicb_scene *s, uint32_t resolution, uint8_t (*out)[4], size_t out_len,
                                     aicb_render_info *info) {
    uint32_t W = 0, H = 0;
    aicb_status st = aicb_ortho_image_size(s, resolution, &W, &H);
    if (st != AICB_OK) return st;
    if (out_len != (size_t)W * H) return fail(AICB_ERR_INVALID, "Viewport size does not match output buffer length");
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    const DeviceScene &ds = s->ds;
    uint32_t vw[5], vh[5], ox[5], oy[5];
    ortho_views(ds, resolution, vw, vh, ox, oy, &W, &H);
    const double inv = 1.0 / (double)resolution;   // (a power of two: exact)
    const double lb[3] = {(double)ds.lo[0], (double)ds.lo[1], (double)ds.lo[2]};
    const double ub[3] = {(double)ds.lo[0] + ds.size[0], (double)ds.lo[1] + ds.size[1], (double)ds.lo[2] + ds.size[2]};
    std::vector<double> rays;
    std::vector<uint32_t> where;
    for (int v = 0; v < 5; v++) {
        for (uint32_t py = 0; py < vh[v]; py++)
            for (uint32_t px = 0; px < vw[v]; px++) {
                // pixel centre, y flipped, scaled to cubes (ortho.rs:278-283); then the view's rotation and corner
                const double u = ((double)px + 0.5) * inv, w = -(((double)py + 0.5) * inv);
                double o[3], d[3] = {0, 0, 0};
                switch (v) {
                    case 0: o[0] = lb[0] + u; o[1] = ub[1]; o[2] = lb[2] - w; d[1] = -1.0; break;   // top: Face::PY
                    case 1: o[0] = lb[0]; o[1] = ub[1] + w; o[2] = lb[2] + u; d[0] = 1.0; break;    // left: Face::NX
                    case 2: o[0] = lb[0] + u; o[1] = ub[1] + w; o[2] = ub[2]; d[2] = -1.0; break;   // front: Face::PZ
                    case 3: o[0] = ub[0]; o[1] = ub[1] + w; o[2] = ub[2] - u; d[0] = -1.0; break;   // right: Face::PX
                    default: o[0] = lb[0] + u; o[1] = lb[1]; o[2] = ub[2] + w; d[1] = 1.0; break;   // bottom: Face::NY
                }
                for (int a = 0; a < 3; a++) rays.push_back(o[a]);
                for (int a = 0; a < 3; a++) rays.push_back(d[a]);
                where.push_back((oy[v] + py) * W + (ox[v] + px));
            }
    }
    const size_t n = where.size();
    std::vector<uchar4> px(n);
    if (n) {
        double *d_rays = nullptr;
        CU(cudaMalloc(&d_rays, n * 48 + 16));
        cudaError_t e = cudaMemcpy(d_rays, rays.data(), n * 48, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            st = ensure(&ctx->d_out, &ctx->d_out_bytes, n * 4 + 16);
            if (st == AICB_OK) {
                aicb_options opt;   // GraphicsOptions::UNALTERED_COLORS (graphics_options.rs:168)
                std::memset(&opt, 0, sizeof opt);
                opt.fog = AICB_FOG_NONE;
                opt.lighting_display = AICB_LIGHT_NONE;
                opt.transparency = AICB_TRANSPARENCY_VOLUMETRIC;
                opt.tone_mapping = AICB_TONE_CLAMP;
                opt.maximum_intensity = INFINITY;
                opt.view_distance = 200.0;
                opt.include_sky = 1;
                Outputs o;
                o.srgb8 = (uchar4 *)ctx->d_out;
                for (;;) {
                    st = launch_trace(s, nullptr, &opt, nullptr, d_rays, n, o, false, ctx->stream);
                    if (st != AICB_OK) break;
                    e = cudaStreamSynchronize(ctx->stream);
                    if (e != cudaSuccess) break;
                    st = finish(s, info);
                    if (st != AICB_ERR_RETRY) break;
                }
                if (st == AICB_OK && e == cudaSuccess) e = cudaMemcpy(px.data(), ctx->d_out, n * 4, cudaMemcpyDeviceToHost);
            }
        }
        cudaFree(d_rays);
        if (e != cudaSuccess) return cuda_fail(e, "orthographic render");
        if (st != AICB_OK) return st;
    }
    std::memset(out, 0, out_len * 4);   // Rgba::TRANSPARENT between the views
    for (size_t i = 0; i < n; i++) std::memcpy(out[where[i]], &px[i], 4);
    return AICB_OK;
}

aicb_status aicb_render_finish(aicb_scene *s, aicb_render_info *info) {
    if (!s) return fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    return finish(s, info);
}

aicb_status aicb_trace_rays(aicb_scene *s, const double (*origin_dir)[6], size_t n, const aicb_options *opt,
                            float (*out_cb)[4], double *depth, aicb_hit *hit, uint32_t *steps,
                            aicb_render_info *info) {
    if (!s || (n && !origin_dir)) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_status st = validate_options(opt);
    if (st != AICB_OK) return st;
    aicb_ctx *ctx = s->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    double *d_rays = nullptr;
    CU(cudaMalloc(&d_rays, n * 48 + 16));
    cudaError_t e = cudaMemcpy(d_rays, origin_dir, n * 48, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(d_rays);
        return cuda_fail(e, "cudaMemcpy rays");
    }
    st = render_aux(s, nullptr, opt, nullptr, d_rays, n, out_cb, depth, hit, steps, n, info);
    cudaFree(d_rays);
    return st;
}

}
