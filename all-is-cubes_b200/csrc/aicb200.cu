// aicb200.cu — host side of libaicb200.so: the C ABI of include/aicb200.h, scene flattening
// (SpaceRaytracer::new, sr.rs:64-88, 543-549) into the two-level brick index, and kernel launch.
//
// No CPU fallback lives here: every compute entry point needs a CUDA device and fails with
// AICB_ERR_CUDA otherwise.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>

#include "block_words.cuh"
#include "brick_room.h"
#include "host_tables.h"
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

// TracingBlock::from_block (sr.rs:579-587) for one block definition: its 32-byte record, classification, brick words
// in the wide form (trace_kernel.cuh) and palette entries (appended to `bricks` / `palette`; the record's offsets are
// relative to those vectors), plus what the marching kernel needs of each surface: {alpha, an upper bound of
// log2(1 - alpha)} per palette entry.
// Called by flatten_blocks alone.
static const char *const BRICKS_PAST_2_32 = "brick pool exceeds 2^32 voxels";
static const aicb_voxel AIR_VOXEL = {{0, 0, 0, 0}, {0, 0, 0}, AICB_VOXEL_NOT_SELECTABLE | AICB_VOXEL_NO_COLLISION};   // Evoxel::AIR

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

aicb_status check_block_scalars(const aicb_block_desc &b) {
    const uint32_t res = b.resolution;
    if (res == 0 || (res & (res - 1)) || res > 128) return fail(AICB_ERR_INVALID, "block resolution must be 1..128, power of 2");
    if (b.indices == nullptr) {
        if (b.n_palette && !b.palette) return fail(AICB_ERR_INVALID, "palette is NULL");
        return AICB_OK;
    }
    const uint64_t nvox = (uint64_t)b.voxel_bounds.size[0] * b.voxel_bounds.size[1] * b.voxel_bounds.size[2];
    if (nvox != b.n_indices) return fail(AICB_ERR_INVALID, "n_indices does not match voxel_bounds");
    for (int a = 0; a < 3; a++) {
        int64_t lo = b.voxel_bounds.lower[a], hi = lo + (int64_t)b.voxel_bounds.size[a];
        if (lo < 0 || hi > (int64_t)res) return fail(AICB_ERR_INVALID, "voxel_bounds must lie within [0, resolution)^3");
    }
    if (!b.palette && b.n_palette) return fail(AICB_ERR_INVALID, "palette is NULL");
    return AICB_OK;
}

aicb_status check_block_palette(const aicb_block_desc &b) {
    if (b.indices && !b.is_air && b.resolution != 1 && b.n_palette > 65536)
        return fail(AICB_ERR_UNSUPPORTED, "block palettes above 65536 entries are not supported: a voxel's palette "
                                          "index (VoxelIndex) is 16 bits");
    return AICB_OK;
}

static const char *const BAD_VOXEL_INDEX = "voxel index out of palette range";

aicb_status check_block_desc(const aicb_block_desc &b) {
    TRY(check_block_scalars(b));
    for (size_t k = 0; b.indices && k < b.n_indices; k++)
        if (b.indices[k] >= b.n_palette) return fail(AICB_ERR_INVALID, BAD_VOXEL_INDEX);
    return check_block_palette(b);
}

aicb_voxel single_voxel_of(const aicb_block_desc &b) {
    if (b.indices == nullptr) return b.n_palette ? b.palette[0] : AIR_VOXEL;
    // single_voxel_or_palette (voxel_storage.rs:371-383)
    const bool at_origin = b.n_indices == 1 && b.voxel_bounds.lower[0] == 0 && b.voxel_bounds.lower[1] == 0 &&
                           b.voxel_bounds.lower[2] == 0;
    return at_origin ? b.palette[b.indices[0]] : AIR_VOXEL;
}

// The record of a definition of kind `kind` (an air block's is KIND_INVISIBLE) whose voxel data starts at brick word
// `brick_off` and palette entry `pal_off`.  Of its collision bits only an air block's are here: the others come from
// the voxels, which flatten_block reads on the host and k_block_records on the device.  So is a recursive block's
// BLOCK_VISIBLE; a single voxel's is its kind's.
static BlockRec block_rec(const aicb_block_desc &b, uint8_t kind, uint32_t brick_off, uint32_t pal_off) {
    BlockRec r;
    std::memset(&r, 0, sizeof r);
    r.flags = (b.is_air || (b.flags & AICB_BLOCK_NOT_SELECTABLE)) ? AICB_BLOCK_NOT_SELECTABLE : 0u;
    if (b.is_air) r.flags |= BLOCK_COLLISION_NONE;   // AIR_EVALUATED
    if (!b.is_air && kind == KIND_SINGLE) r.flags |= BLOCK_VISIBLE;
    if (b.is_air) {
        r.kind_res = KIND_INVISIBLE | (1u << 8);
    } else if (kind != KIND_RECURSIVE) {
        r.kind_res = kind | (1u << 8);
        r.pal_off = pal_off;
        r.vsize[0] = r.vsize[1] = r.vsize[2] = 1;
    } else {
        r.kind_res = KIND_RECURSIVE | ((uint32_t)b.resolution << 8);
        for (int a = 0; a < 3; a++) {
            r.vlo[a] = (int16_t)b.voxel_bounds.lower[a];
            r.vsize[a] = (uint16_t)b.voxel_bounds.size[a];
        }
        r.brick_off = brick_off;
        r.pal_off = pal_off;
    }
    return r;
}

static aicb_status flatten_block(const aicb_block_desc &b, BlockRec &r, uint8_t &kind, std::vector<uint32_t> &bricks,
                                 std::vector<float4> &palette, std::vector<float2> &pal_tab) {
    std::memset(&r, 0, sizeof r);
    TRY(check_block_desc(b));
    auto push_voxel = [&](const aicb_voxel &v) {
        palette.push_back(make_float4(v.rgba[0], v.rgba[1], v.rgba[2], v.rgba[3]));
        palette.push_back(make_float4(v.emission[0], v.emission[1], v.emission[2], voxel_flags(v)));
        pal_tab.push_back(surface_entry(v.rgba[3]));
    };
    const bool single = is_single_voxel(b);
    const aicb_voxel sv = single ? single_voxel_of(b) : AIR_VOXEL;
    if (b.is_air) {
        kind = KIND_INVISIBLE;
        r = block_rec(b, kind, 0, 0);
    } else if (single) {
        kind = voxel_invisible(sv) ? KIND_INVISIBLE : KIND_SINGLE;
        r = block_rec(b, kind, 0, (uint32_t)(palette.size() / 2));
        if (sv.flags & AICB_VOXEL_NO_COLLISION) r.flags |= BLOCK_COLLISION_NONE;
        push_voxel(sv);
    } else {
        kind = KIND_RECURSIVE;
        if (bricks.size() + b.n_indices > 0xffffffffull) return fail(AICB_ERR_INVALID, BRICKS_PAST_2_32);
        r = block_rec(b, kind, (uint32_t)bricks.size(), (uint32_t)(palette.size() / 2));
        bool visible = false;
        for (size_t k = 0; k < b.n_indices; k++) {
            const uint32_t v = b.indices[k];
            const bool inv = voxel_invisible(b.palette[v]);
            visible |= !inv;
            bricks.push_back(v << 16 | (inv ? 0x8000u : 0u));
        }
        if (visible) r.flags |= BLOCK_VISIBLE;
        for (size_t k = 0; k < b.n_palette; k++) push_voxel(b.palette[k]);
        const bool less = less_than_full(r);
        uint32_t pal_mask = 0, used_mask = 0;
        for (size_t k = 0; k < b.n_palette; k++) pal_mask |= collision_mask(b.palette[k].flags);
        if ((pal_mask | (less ? 2u : 0u)) == 3u)   // the palette disagrees: the entries in use decide
            for (size_t k = 0; k < b.n_indices && used_mask != 3u; k++) used_mask |= collision_mask(b.palette[b.indices[k]].flags);
        r.flags |= block_collision(pal_mask, used_mask, less);
    }
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// kernel dispatch
// ---------------------------------------------------------------------------------------------
typedef void (*kernel_fn)(const TraceParams, uint32_t);

template <bool V, bool W, bool AUX, bool B>
static kernel_fn kernel_of() {
    return trace_kernel<V, W, AUX, B>;
}

// The marching kernel of a frame: Volumetric transparency, u32 cells, the step counters (ColorBuf), u32 brick words.
static kernel_fn select_kernel(bool volumetric, bool wide, bool aux, bool wide_bricks) {
#define PICK(V, W, A, B) if (volumetric == V && wide == W && aux == A && wide_bricks == B) return kernel_of<V, W, A, B>();
    PICK(false, false, false, false) PICK(false, false, true, false) PICK(false, true, false, false)
    PICK(false, true, true, false) PICK(true, false, false, false) PICK(true, false, true, false)
    PICK(true, true, false, false) PICK(true, true, true, false)
    PICK(false, false, false, true) PICK(false, false, true, true) PICK(false, true, false, true)
    PICK(false, true, true, true) PICK(true, false, false, true) PICK(true, false, true, true)
    PICK(true, true, false, true) PICK(true, true, true, true)
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

// A u16 cell word (id | kind << 14) as the u32 cell word of the same cube: cell_word(id, kind, true).
static __device__ __forceinline__ uint32_t widened_cell(uint32_t w) { return (w & 0x3fffu) | ((w >> 14) << 16); }

// A scene's cells from u16 to u32 words (a block table grown past 16384 ids): one streaming pass, eight cells per
// thread and step (one 16-byte load, two 16-byte stores, evict-first), the last n % 8 cells one at a time.
static __global__ void __launch_bounds__(256) widen_cells_kernel(const uint16_t *__restrict__ in, uint32_t *__restrict__ out,
                                                                 size_t n) {
    const size_t stride = (size_t)gridDim.x * blockDim.x, first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n8 = n / 8;
    for (size_t i = first; i < n8; i += stride) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4 *>(in) + i);
        __stcs(reinterpret_cast<uint4 *>(out) + 2 * i,
               make_uint4(widened_cell(v.x & 0xffffu), widened_cell(v.x >> 16), widened_cell(v.y & 0xffffu),
                          widened_cell(v.y >> 16)));
        __stcs(reinterpret_cast<uint4 *>(out) + 2 * i + 1,
               make_uint4(widened_cell(v.z & 0xffffu), widened_cell(v.z >> 16), widened_cell(v.w & 0xffffu),
                          widened_cell(v.w >> 16)));
    }
    for (size_t i = n8 * 8 + first; i < n; i += stride) out[i] = widened_cell(in[i]);
}

// A narrow brick word (index | invisible << 15) in the wide form (index << 16 | invisible << 15).
static __device__ __forceinline__ uint32_t widened_brick(uint32_t w) { return (w & 0x7fffu) << 16 | (w & 0x8000u); }

// A scene's brick pool from u16 to u32 words (a block with more than 32768 palette entries placed): one streaming
// pass, as widen_cells_kernel.
static __global__ void __launch_bounds__(256) widen_bricks_kernel(const uint16_t *__restrict__ in,
                                                                  uint32_t *__restrict__ out, size_t n) {
    const size_t stride = (size_t)gridDim.x * blockDim.x, first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n8 = n / 8;
    for (size_t i = first; i < n8; i += stride) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4 *>(in) + i);
        __stcs(reinterpret_cast<uint4 *>(out) + 2 * i,
               make_uint4(widened_brick(v.x & 0xffffu), widened_brick(v.x >> 16), widened_brick(v.y & 0xffffu),
                          widened_brick(v.y >> 16)));
        __stcs(reinterpret_cast<uint4 *>(out) + 2 * i + 1,
               make_uint4(widened_brick(v.z & 0xffffu), widened_brick(v.z >> 16), widened_brick(v.w & 0xffffu),
                          widened_brick(v.w >> 16)));
    }
    for (size_t i = n8 * 8 + first; i < n; i += stride) out[i] = widened_brick(in[i]);
}

// Every u16 cell of a scene set to one word (Mutation::fill_uniform over the whole Space): one 16-byte streaming store
// per eight cells, the last n % 8 cells one at a time.
static __global__ void __launch_bounds__(256) fill_cells_kernel(uint16_t *__restrict__ cells, size_t n, uint32_t word) {
    const size_t stride = (size_t)gridDim.x * blockDim.x, first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t pair = word | word << 16;
    const size_t n8 = n / 8;
    for (size_t i = first; i < n8; i += stride) __stcs(reinterpret_cast<uint4 *>(cells) + i, make_uint4(pair, pair, pair, pair));
    for (size_t i = n8 * 8 + first; i < n; i += stride) cells[i] = (uint16_t)word;
}

// One work item of a box update: a 16-byte-aligned chunk of PER elements of the scene's array, or the part of it that
// one row of the box covers.  A box is size[0] x size[1] rows of size[2] consecutive elements (the arrays are Z-major);
// a row touches at most `chunks_per_row` chunks, so item = row * chunks_per_row + k.  False: chunk k lies past the row.
struct RowChunk {
    uint32_t at;    // the first element's linear index in the scene
    uint32_t pos;   // ... and its position in the box, Z-major (the index into the caller's dense arrays)
    uint32_t n;     // elements: PER for a whole chunk, fewer at a row's unaligned head and tail
};
template <uint32_t PER>
static __device__ __forceinline__ bool row_chunk(const DeviceScene &S, const RegionBox &box, uint32_t item,
                                                 uint32_t chunks_per_row, RowChunk *c) {
    const uint32_t row = item / chunks_per_row, k = item - row * chunks_per_row;
    const uint32_t rx = row / box.size[1], ry = row - rx * box.size[1];
    const uint32_t first = ((box.lo[0] + rx) * (uint32_t)S.size[1] + box.lo[1] + ry) * (uint32_t)S.size[2] + box.lo[2];
    const uint32_t end = first + box.size[2], chunk = (first / PER + k) * PER;
    if (chunk >= end) return false;
    c->at = max(chunk, first);
    c->n = min(chunk + PER, end) - c->at;
    c->pos = row * box.size[2] + (c->at - first);
    return true;
}

// The cells of a box (aicb_scene_update_region, aicb_light_edit_region): each gets cell_word(id, kind of id), the kind
// from the block table's records on the device.  The ids are the caller's dense array (Z-major within the box), or with
// UNIFORM one id.  A whole chunk is one 16-byte store (and one 16-byte load of the ids where their address allows it);
// a row's head and tail are written one cell at a time.  MASK: the old cells are read first (one 16-byte load per whole
// chunk), bit `pos` of `mask` (zeroed by the caller) is set for every cube whose block id changes, and the changed
// cubes are counted into *n_changed if it is given.
template <bool WIDE, bool UNIFORM, bool MASK>
static __global__ void __launch_bounds__(256) k_region_cells(const DeviceScene S, const RegionBox box,
                                                             const uint16_t *__restrict__ ids, uint32_t uniform_id,
                                                             uint32_t chunks_per_row, uint32_t n_items,
                                                             uint32_t *__restrict__ mask, uint32_t *n_changed) {
    using Cell = typename std::conditional<WIDE, uint32_t, uint16_t>::type;
    constexpr uint32_t PER = 16 / sizeof(Cell), KIND_SHIFT = WIDE ? 16 : 14, ID_MASK = WIDE ? 0xffffu : 0x3fffu;
    Cell *cells = (Cell *)S.cells;
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t changed = 0;
    RowChunk c;
    if (item < n_items && row_chunk<PER>(S, box, item, chunks_per_row, &c)) {
        const bool whole = c.n == PER;
        uint32_t id[PER], word[PER];
        if (UNIFORM) {
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) id[k] = uniform_id;
        } else if (whole && ((uintptr_t)(ids + c.pos) & (2 * PER - 1)) == 0) {
            __align__(16) uint32_t w[PER / 2];
            if constexpr (WIDE) *(uint2 *)w = __ldg((const uint2 *)(ids + c.pos));
            else *(uint4 *)w = __ldg((const uint4 *)(ids + c.pos));
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) id[k] = (w[k / 2] >> (16 * (k & 1))) & 0xffffu;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) id[k] = k < c.n ? (uint32_t)__ldg(ids + c.pos + k) : 0u;
        }
        if (MASK) {
            __align__(16) Cell old[PER];
            if (whole) {
                *(uint4 *)old = *(const uint4 *)(cells + c.at);
            } else {
#pragma unroll
                for (uint32_t k = 0; k < PER; k++) old[k] = k < c.n ? cells[c.at + k] : (Cell)0;
            }
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) changed |= (k < c.n && ((uint32_t)old[k] & ID_MASK) != id[k] ? 1u : 0u) << k;
        }
        if (UNIFORM) {
            const uint32_t w = uniform_id | (__ldg(&S.blocks[uniform_id].kind_res) & 0xffu) << KIND_SHIFT;
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) word[k] = w;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < PER; k++) word[k] = id[k] | (__ldg(&S.blocks[id[k]].kind_res) & 0xffu) << KIND_SHIFT;
        }
        if (whole) {
            uint4 v;
            if constexpr (WIDE) v = make_uint4(word[0], word[1], word[2], word[3]);
            else v = make_uint4(word[0] | word[1] << 16, word[2] | word[3] << 16, word[4] | word[5] << 16, word[6] | word[7] << 16);
            *(uint4 *)(cells + c.at) = v;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < PER; k++)
                if (k < c.n) cells[c.at + k] = (Cell)word[k];
        }
        if (MASK && changed) {
            const uint32_t shift = c.pos & 31u;
            atomicOr(mask + (c.pos >> 5), changed << shift);
            if (shift + c.n > 32u) atomicOr(mask + (c.pos >> 5) + 1, changed >> (32u - shift));
        }
    }
    if (MASK) {
        const uint32_t total = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(changed));
        if ((threadIdx.x & 31u) == 0 && total && n_changed) atomicAdd(n_changed, total);
    }
}

// The texels of a box (aicb_scene_update_region's dense light): 4 texels per chunk, one 16-byte store per whole chunk
// (and one 16-byte load where the caller's array allows it), a row's head and tail one texel at a time.
static __global__ void __launch_bounds__(256) k_region_texels(const DeviceScene S, const RegionBox box,
                                                              const uint32_t *__restrict__ texels, uint32_t chunks_per_row,
                                                              uint32_t n_items, uint32_t *__restrict__ light) {
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    RowChunk c;
    if (item >= n_items || !row_chunk<4>(S, box, item, chunks_per_row, &c)) return;
    if (c.n == 4 && ((uintptr_t)(texels + c.pos) & 15u) == 0) {
        *(uint4 *)(light + c.at) = __ldg((const uint4 *)(texels + c.pos));
    } else {
        for (uint32_t k = 0; k < c.n; k++) light[c.at + k] = __ldg(texels + c.pos + k);
    }
}

// One run of a pool compaction (compact_pools): `bytes` bytes from byte `src` of the old pool to byte `dst` of the new
// one.  Offsets and lengths are even (a u16 brick word is a pool's smallest element; u32 brick words, float2 and
// float4 are multiples of it).
struct PoolSegment {
    uint64_t src, dst, bytes;
};

// Gathers a pool's live runs into a new buffer: blocks take segments in a grid-stride loop.  Within a segment, every
// 16-byte chunk of the destination that it covers whole is one coalesced 16-byte store, assembled from the one or two
// aligned 16-byte source chunks that hold its bytes (a funnel shift when the run moves by other than a multiple of 16
// bytes).  The at most seven u16 halves of words at either end, whose chunk a neighbouring segment shares, are stored
// one at a time, whatever the pool's element size.  Both buffers are multiples of 16 bytes (grow_buffer, compact_pools), so an aligned source chunk that holds one
// byte of a run lies inside the old buffer.
static __global__ void __launch_bounds__(256) compact_pool_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst,
                                                                  const PoolSegment *__restrict__ segs, uint32_t n_segs) {
    for (uint32_t k = blockIdx.x; k < n_segs; k += gridDim.x) {
        const PoolSegment g = segs[k];
        const uint64_t shift = g.src - g.dst;   // modulo 2^64: dst + shift is the source of a destination byte
        const uint64_t c0 = (g.dst + 15) / 16, c1 = (g.dst + g.bytes) / 16;   // the chunks the segment covers whole
        const uint32_t s = (uint32_t)(shift & 15), b = (s & 3) * 8;
        for (uint64_t c = c0 + threadIdx.x; c < c1; c += blockDim.x) {
            const uint4 *p = reinterpret_cast<const uint4 *>(src + ((c * 16 + shift) & ~15ull));
            const uint4 lo = p[0];
            uint4 out = lo;
            if (s) {
                const uint4 hi = p[1];
                const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#define FS(i) __funnelshift_r(w[i], w[(i) + 1], b)
                switch (s >> 2) {
                    case 0: out = make_uint4(FS(0), FS(1), FS(2), FS(3)); break;
                    case 1: out = make_uint4(FS(1), FS(2), FS(3), FS(4)); break;
                    case 2: out = make_uint4(FS(2), FS(3), FS(4), FS(5)); break;
                    default: out = make_uint4(FS(3), FS(4), FS(5), FS(6)); break;
                }
#undef FS
            }
            reinterpret_cast<uint4 *>(dst)[c] = out;
        }
        // the words before the first whole chunk (threads 0-7) and after the last (threads 8-15)
        const uint64_t end = g.dst + g.bytes, head_end = min(c0 * 16, end), tail = max(c1 * 16, head_end);
        if (threadIdx.x < 16) {
            const uint64_t x = threadIdx.x < 8 ? g.dst + 2 * threadIdx.x : tail + 2 * (threadIdx.x - 8);
            if (x < (threadIdx.x < 8 ? head_end : end))
                reinterpret_cast<uint16_t *>(dst)[x / 2] = reinterpret_cast<const uint16_t *>(src)[(x + shift) / 2];
        }
    }
}

// After a compaction, each id's record takes its extents' new offsets ({brick word, palette entry} per id); a single
// voxel's blk_tab entry carries its absolute palette entry (block_entry).
static __global__ void rebase_blocks_kernel(BlockRec *blocks, float4 *blk_tab, const uint2 *__restrict__ off, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    BlockRec r = blocks[i];
    r.brick_off = off[i].x;
    r.pal_off = off[i].y;
    blocks[i] = r;
    if ((r.kind_res & 0xffu) == KIND_SINGLE) blk_tab[i].z = __uint_as_float(off[i].y);
}

aicb_status validate_options(const aicb_options *o) {
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

// A layered frame's accumulators before its world pass, where a backdrop but no UI layer lies in front of the world.
static __global__ void __launch_bounds__(256) fill_accum_kernel(float4 *__restrict__ accum, size_t n, float4 v) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) accum[i] = v;
}

// The compositing kernels of a frame's target (TGT_*): resolve_kernel with None / Flat lighting, encode_kernel after
// shade_kernel.
static kernel_fn resolve_for(int lc, int tgt) {
    switch (tgt) {
        case TGT_TEX: return lc == LC_NONE ? resolve_kernel<LC_NONE, TGT_TEX> : resolve_kernel<LC_FLAT, TGT_TEX>;
        case TGT_TERM: return lc == LC_NONE ? resolve_kernel<LC_NONE, TGT_TERM> : resolve_kernel<LC_FLAT, TGT_TERM>;
        case TGT_VIEWS: return lc == LC_NONE ? resolve_kernel<LC_NONE, TGT_VIEWS> : resolve_kernel<LC_FLAT, TGT_VIEWS>;
        default: return lc == LC_NONE ? resolve_kernel<LC_NONE, TGT_FRAME> : resolve_kernel<LC_FLAT, TGT_FRAME>;
    }
}
static kernel_fn encode_for(int tgt) {
    switch (tgt) {
        case TGT_TEX: return encode_kernel<TGT_TEX>;
        case TGT_TERM: return encode_kernel<TGT_TERM>;
        case TGT_VIEWS: return encode_kernel<TGT_VIEWS>;
        default: return encode_kernel<TGT_FRAME>;
    }
}

// Launches the trace kernel on `stream`. Camera rays when cam != NULL, the explicit rays of `out` otherwise; with a
// TGT_VIEWS target, cam gives only the framebuffer size and the rays of out.n_views views come from the target's
// camera table (the caller has checked that the batch's tasks fit in 32 bits).  With
// `continues`, the pass continues the context's frame in flight on the same stream (the world pass of a layered frame
// behind its UI pass, aicb_render_layers_device): the frame counters, the overflow flag and the start event carry on,
// so finish reports both passes, and the frame is finished on `sc`.
static aicb_status launch_trace(aicb_scene *sc, const aicb_camera *cam, const aicb_options *opt,
                                const aicb_shard *shard, const Outputs &out, cudaStream_t stream,
                                bool continues = false) {
    aicb_ctx *ctx = sc->ctx;
    TraceParams P;
    std::memset(&P, 0, sizeof P);
    P.scene = sc->ds;
    uint64_t pixels;
    if (cam) {
        std::memcpy(P.m, cam->inverse_projection_view, sizeof P.m);
        P.fb_width = cam->fb_width;
        P.fb_height = cam->fb_height;
        P.inv_width = 1.0 / (double)cam->fb_width;
        P.inv_height = 1.0 / (double)cam->fb_height;
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
        if (listed(out.target)) {   // one pixel task per listed pixel, 32 consecutive entries per warp
            P.tiles_x = (out.target.n_list + 31) / 32;
            P.tiles_y = 1;
            P.n_tasks = out.target.n_list;
            pixels = out.target.n_list;
        }
        if (out.kind == TGT_VIEWS) {   // the views' tile-ordered tasks end to end
            P.n_tasks = P.tiles_x * P.tiles_y * 32 * out.n_views;
            pixels *= out.n_views;
        }
    } else {
        P.exposure = 1.0f;
        P.rays = out.rays;
        P.n_rays = out.n_rays;
        if (out.n_rays > 0xffffffffull) return fail(AICB_ERR_INVALID, "too many rays");
        P.tiles_x = (uint32_t)((out.n_rays + 31) / 32);
        P.tiles_y = 1;
        P.n_tasks = (uint32_t)out.n_rays;
        P.shard_count = 1;
        P.strip_rows = 1;
        pixels = out.n_rays;
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
    P.target = out.target;
    const int tgt = out.kind;
    if (tgt == TGT_VIEWS) P.target.view_tiles = P.tiles_x * P.tiles_y;
    P.counters = ctx->d_counters.get<unsigned long long>();
    P.task_counter = ctx->d_tile_counter;
    P.refill_threshold = REFILL_THRESHOLD;
    P.tail_divisor = TAIL_DIVISOR;
    P.event_threshold = EVENT_THRESHOLD;

    uint64_t frame_pixels = pixels, frame_rays = pixels * (P.antialias ? 4 : 1);
    uint64_t out_bytes =
        (P.target.out_srgb8 ? 4 : (tgt == TGT_TEX ? 12 : (tgt == TGT_TERM ? 24 : (P.target.out_rgba16f ? 8 : 16)))) * pixels;
    if (continues && ctx->last_scene) {
        aicb_scene *prev = ctx->last_scene;
        frame_pixels += prev->pending_pixels;
        frame_rays += prev->pending_rays;
        out_bytes += prev->pending_out_bytes;
        prev->pending = false;
    }
    sc->pending = true;
    sc->pending_pixels = frame_pixels;
    sc->pending_rays = frame_rays;
    sc->pending_out_bytes = out_bytes;

    // ---- the kernels of a frame, chunked so the per-frame streams stay bounded ----------------------------------
    P.n_samples = P.antialias ? 4 : 1;
    // gen -> march -> resolve (shading and encode in one kernel) with None / Flat lighting, unless the context's last
    // frame met 3/4 of a visible surface per ray or more; otherwise gen -> march -> shade -> encode.  resolve_kernel
    // saves the ShadedHit round trip, the scan of the dead slots and a kernel drain, but its warps also list and
    // composite, so fewer of them shade at once: where a warp has several 32-slot shading rounds the separate
    // shade_kernel is faster.  Measured on one H100 SXM at 700 W: the opaque bench frames (C0, C1, C3: 0.3-0.5 visible
    // surfaces per ray) 7-17 % faster fused; the C2 frame (1.0 per ray) 7 % slower with None and 11 % with Flat
    // lighting, and 1.8x slower in shade + encode with interpolated lighting, which therefore never takes this path.
    const bool fused = (opt->lighting_display == AICB_LIGHT_NONE || opt->lighting_display == AICB_LIGHT_FLAT) &&
                       !ctx->deep_frames;
    const uint64_t total_tasks = (uint64_t)P.n_tasks * P.n_samples;
    // Tasks per chunk (a multiple of 32 * n_samples): at most 4 M (0.6 GB of ray records); fewer when the hit stream
    // has been enlarged after an overflow, so that the per-frame streams stay within ~8 GB however deep the scene is.
    uint64_t CHUNK = (uint64_t)4 << 20;
    {
        const uint64_t per_task = sizeof(RayRecordA) + sizeof(RayRecordB) + sizeof(TaskOut) + 4 * N_BINS +
                                  (uint64_t)ctx->hits_per_task * (sizeof(HitRecord) + (fused ? 0 : sizeof(ShadedHit)));
        uint64_t fit = ((uint64_t)8 << 30) / per_task;
        if (fit < (1u << 17)) fit = 1u << 17;
        if (fit < CHUNK) CHUNK = fit & ~(uint64_t)127;
    }
    const uint64_t chunk_cap = total_tasks < CHUNK ? total_tasks : CHUNK;
    uint64_t cap = chunk_cap * ctx->hits_per_task;
    if (cap < (1u << 16)) cap = 1u << 16;
    if (cap > 0xfffffff0ull) cap = 0xfffffff0ull;
    cap &= ~(uint64_t)(HIT_CHUNK - 1);  // lanes take whole chunks of the stream
    P.hit_capacity = (uint32_t)cap;
    // Ray order: a frame of one chunk of camera rays that repeats the context's previous frame's view and layout (an
    // interactive caller redraws a view that rests, its scene edited or not) lists its rays by the steps its tiles'
    // rays took then, costliest first, so that the marching kernel does not end on long rays it took late (gen_rays).
    // A moved camera takes the chord bins: with the camera turning 0.5 degrees a frame, the previous frame's order
    // measured 1 % slower than the chord order on C2 (tools/orbit_bench.py, H100 SXM, 700 W).  So do pixel lists and
    // texture picks, explicit rays, batches of views, Bounce, chunked frames and the passes of a layered frame, whose
    // scenes alternate.  The order never changes a result, so a key that matches a frame of a freed scene does no harm.
    RayOrderKey key;
    if (cam && tgt != TGT_VIEWS && !listed(out.target) && opt->lighting_display != AICB_LIGHT_BOUNCE &&
        total_tasks > 0 && total_tasks <= CHUNK) {
        key.scene = sc;
        std::memcpy(key.view, cam->inverse_projection_view, sizeof key.view);
        key.fb_width = P.fb_width;
        key.fb_height = P.fb_height;
        key.n_samples = P.n_samples;
        key.strip_rows = P.strip_rows;
        key.shard_index = P.shard_index;
        key.shard_count = P.shard_count;
    }
    const bool order_by_steps = key.scene && key == ctx->order_key;
    ctx->order_key = RayOrderKey{};   // until this frame's streams are in place
    TRY(ctx->primary.size(chunk_cap, P.hit_capacity, !fused));
    ctx->primary.bind(P, chunk_cap, !fused);
    P.order_by_steps = order_by_steps ? 1 : 0;
    ctx->order_key = key;
    ctx->ray_ordered = (continues && ctx->ray_ordered) || order_by_steps;
    P.ray_counter = ctx->d_tile_counter + 2;
    sc->pending_fused = fused;
    P.hit_counter = ctx->d_tile_counter + 1;
    P.bin_count = ctx->d_tile_counter + 4;
    P.bin_stride = (uint32_t)chunk_cap;
    P.overflow_flag = (unsigned int *)(P.counters + 7);
    if (stream != ctx->stream.get()) CU(cudaStreamWaitEvent(stream, ctx->ev_delta.get(), 0));  // pending cube edits
    // The per-frame streams, counters and events belong to the context: a frame issued on another stream than the
    // previous one must not start before that one is through with them.
    if (ctx->frame_in_flight && ctx->last_stream != stream) CU(cudaStreamWaitEvent(stream, ctx->ev1.get(), 0));
    ctx->frame_in_flight = true;
    ctx->last_stream = stream;
    ctx->last_scene = sc;
    if (continues) {
        CU(cudaMemsetAsync(ctx->d_tile_counter, 0, 2 * (4 + N_BINS) * sizeof(unsigned int), stream));
    } else {
        CU(cudaMemsetAsync(P.counters, 0, 8 * sizeof(unsigned long long) + 2 * (4 + N_BINS) * sizeof(unsigned int), stream));
        CU(cudaEventRecord(ctx->ev0.get(), stream));
    }
    if (total_tasks > 0) {
        const bool volumetric = opt->transparency == AICB_TRANSPARENCY_VOLUMETRIC;
        const int lc = opt->lighting_display == AICB_LIGHT_NONE ? LC_NONE
                       : (opt->lighting_display == AICB_LIGHT_FLAT ? LC_FLAT
                          : (opt->lighting_display == AICB_LIGHT_BOUNCE ? LC_BOUNCE : LC_INTERP));
        // LightingOption::Bounce: the secondary rays of a chunk run through the same kernels on a second set of streams
        TraceParams Q;
        const bool bounce = lc == LC_BOUNCE;
        if (bounce) {
            TRY(ctx->secondary.size(chunk_cap, P.hit_capacity, true));
            // per task: request (4) + RNG state (32) + Rgb sum and steps (16) + the secondary ray (48) + record index (4)
            TRY(ctx->d_bounce.ensure(chunk_cap * 104 + 256));
            char *b = ctx->d_bounce.get<char>();
            P.bounce_mode = BOUNCE_PRIMARY;
            P.bounce_samples = opt->bounce_samples;
            P.bounce_rays = (double *)b;                                   // 48 B per task, 16-aligned
            P.bounce_rng = (unsigned long long *)(b + chunk_cap * 48);     // 32 B
            P.bounce_sum = (float4 *)(b + chunk_cap * 80);                 // 16 B
            P.bounce_req = (uint32_t *)(b + chunk_cap * 96);               // 4 B
            P.ray_index = (uint32_t *)(b + chunk_cap * 100);               // 4 B
            Q = P;
            Q.ray_index = nullptr;
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
            Q.target = {};   // the secondary rays store nothing of the frame's
            ctx->secondary.bind(Q, chunk_cap, true);
            Q.task_counter = ctx->d_tile_counter + (4 + N_BINS);
            Q.hit_counter = Q.task_counter + 1;
            Q.ray_counter = Q.task_counter + 2;
            Q.bin_count = Q.task_counter + 4;
            Q.debug_warp_times = nullptr;
        }
        kernel_fn k = select_kernel(volumetric, sc->ds.wide_cells != 0, out.aux, sc->host->wide_bricks);
        int blocks_per_sm = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k, WARPS_PER_BLOCK * 32, 0));
        if (blocks_per_sm < 1) blocks_per_sm = 1;
        for (uint64_t base = 0; base < total_tasks; base += CHUNK) {
            const uint32_t n = (uint32_t)(total_tasks - base < CHUNK ? total_tasks - base : CHUNK);
            P.task_base = (uint32_t)base;
            const bool first = base == 0;  // stage times are reported for the first chunk
            if (!first) CU(cudaMemsetAsync(ctx->d_tile_counter, 0, (4 + N_BINS) * sizeof(unsigned int), stream));
            const bool prof = ctx->profile_kernels && first;
            const bool stage = first && ctx->stage_timing;
            if (stage) cudaEventRecord(ctx->ev_k[0].get(), stream);
            if (tgt == TGT_VIEWS) gen_views_kernel<<<(n + 127) / 128, 128, 0, stream>>>(P, n);
            else gen_kernel<<<(n + 127) / 128, 128, 0, stream>>>(P, n);
            if (stage) cudaEventRecord(ctx->ev_k[1].get(), stream);
            uint64_t want = ((uint64_t)n + WARPS_PER_BLOCK * 32 - 1) / (WARPS_PER_BLOCK * 32);
            uint64_t grid = (uint64_t)ctx->num_sms * blocks_per_sm;  // persistent: a multiple of the SM count
            if (grid > want) grid = want;
            if (prof) {
                TRY(ctx->d_debug.ensure(4 * 8 * (size_t)ctx->num_sms * 64 * WARPS_PER_BLOCK));
                P.debug_warp_times = ctx->d_debug.get<unsigned long long>();
                ctx->debug_warps = (uint32_t)grid * WARPS_PER_BLOCK;
            }
            // the frame's kernels follow each other with programmatic dependent launch (no events between them)
            const bool overlap = !stage && !prof && !bounce;
            CU(launch_after(overlap, k, (unsigned)grid, WARPS_PER_BLOCK * 32, stream, P, n));
            P.debug_warp_times = nullptr;
            if (stage) cudaEventRecord(ctx->ev_k[2].get(), stream);
            if (fused) {
                const unsigned rb = (n + 127) / 128;   // one warp per 32 tasks
                CU(launch_after(overlap, resolve_for(lc, tgt), rb, 128, stream, P, n));
                if (stage) cudaEventRecord(ctx->ev_k[3].get(), stream);
            } else if (!bounce) {
                switch (lc) {
                    case LC_NONE: CU(launch_after(overlap, shade_kernel<LC_NONE>, ctx->num_sms * SHADE_BLOCKS_PER_SM, 128, stream, P)); break;
                    case LC_FLAT: CU(launch_after(overlap, shade_kernel<LC_FLAT>, ctx->num_sms * SHADE_BLOCKS_PER_SM, 128, stream, P)); break;
                    default: CU(launch_after(overlap, shade_kernel<LC_INTERP>, ctx->num_sms * SHADE_BLOCKS_PER_SM_INTERP, 128, stream, P)); break;
                }
                if (stage) cudaEventRecord(ctx->ev_k[3].get(), stream);
                const uint32_t n_pixels = n / P.n_samples;
                CU(launch_after(overlap, encode_for(tgt), (n_pixels + 127) / 128, 128, stream, P, n));
                if (stage) cudaEventRecord(ctx->ev_k[4].get(), stream);
            } else {
                shade_kernel<LC_BOUNCE><<<ctx->num_sms * SHADE_BLOCKS_PER_SM, 128, 0, stream>>>(P);
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
                    shade_kernel<LC_FLAT><<<ctx->num_sms * SHADE_BLOCKS_PER_SM, 128, 0, stream>>>(Q);
                    encode_kernel<TGT_FRAME><<<tb, 128, 0, stream>>>(Q, n);
                }
                bounce_resolve_kernel<<<tb, 128, 0, stream>>>(P, n);
                if (stage) cudaEventRecord(ctx->ev_k[3].get(), stream);
                const uint32_t n_pixels = n / P.n_samples;
                encode_for(tgt)<<<(n_pixels + 127) / 128, 128, 0, stream>>>(P, n);
                if (stage) cudaEventRecord(ctx->ev_k[4].get(), stream);
            }
        }
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(ctx->ev1.get(), stream));
    return AICB_OK;
}

static aicb_status finish(aicb_scene *sc, aicb_render_info *info) {
    aicb_ctx *ctx = sc->ctx;
    if (ctx->last_scene != sc)
        return fail(AICB_ERR_BUSY, "the context's last frame belongs to another scene (one frame per context is tracked)");
    CU(cudaEventSynchronize(ctx->ev1.get()));
    ctx->frame_in_flight = false;
    unsigned long long c[8];
    CU(cudaMemcpy(c, ctx->d_counters.get(), sizeof c, cudaMemcpyDeviceToHost));
    sc->pending = false;
    if (ctx->profile_kernels && sc->pending_rays) {  // AICB_PROFILE_KERNELS=1: per-kernel times of the first chunk
        float t[4] = {0, 0, 0, 0};
        for (int i = 0; i < (sc->pending_fused ? 3 : 4); i++) cudaEventElapsedTime(&t[i], ctx->ev_k[i].get(), ctx->ev_k[i + 1].get());
        if (ctx->d_debug && ctx->debug_warps) {
            std::vector<unsigned long long> w(4 * (size_t)ctx->debug_warps);
            cudaMemcpy(w.data(), ctx->d_debug.get(), w.size() * 8, cudaMemcpyDeviceToHost);
            unsigned long long t0 = ~0ull, t1 = 0, passes = 0, rays = 0;
            for (uint32_t i = 0; i < ctx->debug_warps; i++) { t0 = std::min(t0, w[4 * i]); t1 = std::max(t1, w[4 * i + 1]); passes += w[4 * i + 2]; rays += w[4 * i + 3]; }
            std::vector<double> ends;
            for (uint32_t i = 0; i < ctx->debug_warps; i++) ends.push_back((double)(w[4 * i + 1] - t0) * 1e-6);
            std::sort(ends.begin(), ends.end());
            auto q = [&](double f) { return ends[(size_t)(f * (ends.size() - 1))]; };
            fprintf(stderr, "[aicb200] march warps %u: end times ms min %.3f p10 %.3f p50 %.3f p90 %.3f p99 %.3f max %.3f; passes/warp %.0f rays %llu\n",
                    ctx->debug_warps, q(0), q(0.1), q(0.5), q(0.9), q(0.99), q(1.0), (double)passes / ctx->debug_warps, rays);
        }
        if (sc->pending_fused)
            fprintf(stderr, "[aicb200] gen %.3f ms  march %.3f ms  resolve (shade + encode) %.3f ms  (hits %llu)\n", t[0], t[1],
                    t[2], c[3]);
        else
            fprintf(stderr, "[aicb200] gen %.3f ms  march %.3f ms  shade %.3f ms  encode %.3f ms  (hits %llu)\n", t[0], t[1], t[2],
                    t[3], c[3]);
    }
    if (sc->pending_rays) ctx->deep_frames = c[3] * 4 >= sc->pending_rays * 3;   // visible surfaces per ray >= 3/4
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
            ctx->primary.release_hits();
            ctx->secondary.release_hits();
        }
    } else {
        ctx->shallow_frames = 0;
    }
    if (info) {
        std::memset(info, 0, sizeof *info);
        float ms = 0.0f;
        CU(cudaEventElapsedTime(&ms, ctx->ev0.get(), ctx->ev1.get()));
        info->kernel_ms = ms;
        if (sc->pending_rays && ctx->stage_timing)   // a fused frame: [2] is resolve_kernel, [3] stays 0
            for (int i = 0; i < (sc->pending_fused ? 3 : 4); i++)
                cudaEventElapsedTime(&info->stage_ms[i], ctx->ev_k[i].get(), ctx->ev_k[i + 1].get());
        info->cubes_traced = c[0];
        info->rays = sc->pending_rays;
        for (int i = 0; i < 5; i++) info->counters[i] = c[1 + i];
        info->counters[5] = sc->pending_pixels;
        // SURVEY 8(d): 2 B per outer/inner step, 32 B per surface hit, 4 B per light texel,
        // 32 B per recursive block entered (our BlockRec), + output bytes per pixel
        info->algorithmic_bytes = 2 * c[1] + 2 * c[2] + 32 * c[3] + 4 * c[4] + 32 * c[5] + sc->pending_out_bytes;
        info->flaws = 0;
        info->ray_order = ctx->ray_ordered ? 1 : 0;
    }
    sc->pending = false;
    return AICB_OK;
}

// ---- outputs in the caller's device memory (aicb_device_outputs) --------------------------------------------------
aicb_status issue_empty_frame(aicb_scene *s, const aicb_options *opt, cudaStream_t stream) {
    return launch_trace(s, nullptr, opt, nullptr, Outputs{}, stream);
}

// A caller's device buffer: memory of `device`, or with peer_ok of a device it reaches as a peer (a frame of another
// rank mapped into this process, aicb_render_srgb8_device_frame), aligned to `align` bytes, the width of the kernels'
// stores to it or loads from it (a misaligned vector access would fault the context).
aicb_status check_device_pointer(const void *p, int device, bool peer_ok, size_t align, const char *what) {
    if ((uintptr_t)p % align)
        return fail(AICB_ERR_INVALID, std::string(what) + " is not aligned to " + std::to_string(align) + " bytes");
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) cudaGetLastError();
    if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged))
        return fail(AICB_ERR_INVALID, std::string(what) + " is not device memory");
    if (a.device == device) return AICB_OK;
    int can = 0;
    if (peer_ok && cudaDeviceCanAccessPeer(&can, device, a.device) == cudaSuccess && can) return AICB_OK;
    return fail(AICB_ERR_INVALID, std::string(what) + " is memory of another device");
}

aicb_status output_target(const aicb_device_outputs *d, DeviceCall call, bool need_colorbuf, Outputs *o) {
    if (!d) return fail(AICB_ERR_INVALID, "outs is NULL");
    const void *const ptr[10] = {d->srgb8, d->rgba16f, d->colorbuf, d->depth, d->hit,
                                 d->steps, d->text,    d->texel_rgba16f, d->texel_depth, d->terminal};
    unsigned set = 0;
    for (int i = 0; i < 10; i++)
        if (ptr[i]) set |= 1u << i;
    // the sets of outputs one host call gives: sRGB8, rgba16f, ColorBuf and its companions, text; layered: sRGB8,
    // the terminal's pixels, the texture's two texels
    const unsigned SRGB8 = 1, RGBA16F = 2, AUX = 4 | 8 | 16 | 32, TEXT = 64, TEXELS = 128 | 256, TERMINAL = 512;
    const bool aux = set && !(set & ~AUX);
    bool ok = false;
    switch (call) {
        case DEV_FRAME: ok = set == SRGB8 || set == RGBA16F || aux || set == TEXT; break;
        case DEV_RAYS: ok = aux; break;
        case DEV_LAYERS: ok = set == SRGB8 || set == TERMINAL || set == TEXELS; break;
    }
    if (set == 0 && d->len == 0) ok = true;
    if (!ok) return fail(AICB_ERR_INVALID, "the outputs are not a set that this call gives (aicb_device_outputs)");
    if (aux && need_colorbuf && d->len && !d->colorbuf) return fail(AICB_ERR_INVALID, "colorbuf is NULL");
    TargetParams &t = o->target;
    t.out_srgb8 = (uchar4 *)d->srgb8;
    t.out_text = d->text;
    o->aux = aux;
    if (aux) {
        t.out_colorbuf = (float4 *)d->colorbuf;
        t.out_depth = d->depth;
        t.out_hit = d->hit;
        t.out_steps = d->steps;
    }
    if (set == RGBA16F) t.out_rgba16f = (uint2 *)d->rgba16f;
    if (set == TEXELS) {
        o->kind = TGT_TEX;
        t.out_rgba16f = (uint2 *)d->texel_rgba16f;
        t.out_tex_depth = d->texel_depth;
    }
    if (set == TERMINAL) {
        o->kind = TGT_TERM;
        t.out_term = d->terminal;
        t.text_start = AICB_TEXT_EMPTY;
    }
    return AICB_OK;
}

aicb_status device_target(const aicb_device_outputs *d, int device, DeviceCall call, bool need_colorbuf, bool peer_ok,
                          Outputs *o) {
    TRY(output_target(d, call, need_colorbuf, o));
    const void *const ptr[10] = {d->srgb8, d->rgba16f, d->colorbuf, d->depth, d->hit,
                                 d->steps, d->text,    d->texel_rgba16f, d->texel_depth, d->terminal};
    static const char *const name[10] = {"srgb8", "rgba16f", "colorbuf", "depth", "hit",
                                         "steps", "text",    "texel_rgba16f", "texel_depth", "terminal"};
    // the width of each output's stores (uchar4, uint2, float4, double, aicb_hit, u32, i32, uint2, float, 2 x float2)
    static const size_t align[10] = {4, 8, 16, 8, 4, 4, 4, 8, 4, 8};
    for (int i = 0; i < 10; i++)
        if (ptr[i]) TRY(check_device_pointer(ptr[i], device, peer_ok, align[i], name[i]));
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// a scene's block table (internal.h): flattened once, placed on each replica
// ---------------------------------------------------------------------------------------------
static size_t round16(size_t bytes) { return (bytes + 15) & ~(size_t)15; }

// Room for `bytes` in `buf`, of which the first `used` are kept.  A buffer that is too small is replaced by one of at
// least twice its size (`bytes` rounded up to 16 if it was empty), its `used` bytes copied on `stream`; the replaced
// buffer goes to `retired`.  Appending k elements one call at a time thus reallocates O(log k) times.
static aicb_status grow_buffer(DeviceBuffer &buf, size_t used, size_t bytes, cudaStream_t stream,
                               std::vector<DeviceBuffer> *retired) {
    if (buf.bytes() >= bytes) return AICB_OK;
    DeviceBuffer b;
    TRY(b.ensure(std::max(round16(bytes), 2 * buf.bytes())));
    if (used) CU(cudaMemcpyAsync(b.get(), buf.get(), used, cudaMemcpyDeviceToDevice, stream));
    if (buf) retired->push_back(std::move(buf));
    buf = std::move(b);
    return AICB_OK;
}

// Returns once nothing on the context can read a scene's arrays: its frame in flight, whichever scene drew it (the
// context's frames run one after another, launch_trace, so it is behind every earlier one), and the context's stream.
static aicb_status wait_context(aicb_ctx *ctx) {
    if (ctx->frame_in_flight) CU(cudaEventSynchronize(ctx->ev1.get()));
    CU(cudaStreamSynchronize(ctx->stream.get()));
    return AICB_OK;
}

// The arrays a scene replaced, freed when the call ends, once nothing can read them (wait_context).
struct Retired {
    aicb_ctx *ctx;
    std::vector<DeviceBuffer> bufs;
    ~Retired() {
        if (!bufs.empty()) wait_context(ctx);
    }
};

// What a call allocated for each replica before changing any, freed on each replica's device once an allocation fails.
template <typename T>
static aicb_status free_each(Replicas r, std::vector<T> &per_replica, aicb_status st) {
    for (size_t i = 0; i < per_replica.size(); i++) {
        cudaSetDevice(r.ctx[i]->device);
        per_replica[i] = T();
    }
    return st;
}

// Block definitions flattened against a table's bookkeeping: per definition its record (brick_off / pal_off already
// offsets into the table's pools) and extents, blk_tab entry, kind and light record; and the voxel data they append to
// the pools.  The brick words are in the form the table's pool has once they are placed: wide if it is wide already or
// if a palette has more than 32768 entries.
struct FlatBlocks {
    std::vector<BlockRec> recs;
    std::vector<BlockTable::Extent> extents;
    std::vector<float4> blk_tab;
    std::vector<uint8_t> kinds;
    std::vector<LightBlockDev> light;
    bool wide_bricks = false;
    std::vector<uint32_t> bricks;      // the words in the wide form (flatten_block); their count in either form
    std::vector<uint16_t> narrow;      // the words in the narrow form, unless wide_bricks
    size_t brick_word_bytes() const { return wide_bricks ? 4 : 2; }
    const void *brick_words() const { return wide_bricks ? (const void *)bricks.data() : narrow.data(); }
    std::vector<float4> palette;
    std::vector<float2> pal_tab;
    size_t words = 0, entries = 0;   // brick words and palette entries added (the vectors' sizes, if on the host)
};

// Validates and flattens n definitions against `h`, for the next ids (indices == nullptr) or for existing `indices`.
// Changes nothing.
static aicb_status flatten_blocks(const SpaceHost &h, const aicb_block_desc *descs, size_t n, const uint16_t *indices,
                                  FlatBlocks *f) {
    if (!indices && h.block_count() + n > 65536) return fail(AICB_ERR_INVALID, "more than 65536 blocks");
    const uint32_t pal_base = (uint32_t)(h.n_palette / 2);   // palette entries (2 x float4 each)
    f->recs.resize(n);
    f->extents.resize(n);
    f->blk_tab.resize(n);
    f->kinds.resize(n);
    f->light.resize(n);
    for (size_t i = 0; i < n; i++) {
        if (indices && indices[i] >= h.block_count())
            return fail(AICB_ERR_INVALID, "block index out of range (new indices need a new scene)");
        BlockRec &r = f->recs[i];
        const size_t bricks_before = f->bricks.size(), pal_before = f->pal_tab.size();
        TRY(flatten_block(descs[i], r, f->kinds[i], f->bricks, f->palette, f->pal_tab));
        f->blk_tab[i] = block_entry(f->kinds[i], r.pal_off, f->pal_tab, pal_base);
        if (f->kinds[i] == KIND_RECURSIVE) r.brick_off += (uint32_t)h.n_bricks;
        if (!descs[i].is_air) r.pal_off += pal_base;
        f->extents[i] = {r.brick_off, (uint32_t)(f->bricks.size() - bricks_before), r.pal_off,
                         (uint32_t)(f->pal_tab.size() - pal_before)};
        f->light[i] = light_block(descs[i]);
        if (f->kinds[i] == KIND_RECURSIVE && descs[i].n_palette > 32768) f->wide_bricks = true;
    }
    if (h.wide_bricks) f->wide_bricks = true;
    if (!f->wide_bricks) {
        f->narrow.resize(f->bricks.size());
        for (size_t k = 0; k < f->bricks.size(); k++) f->narrow[k] = (uint16_t)(f->bricks[k] >> 16 | (f->bricks[k] & 0x8000u));
    }
    f->words = f->bricks.size();
    f->entries = f->pal_tab.size();
    // live data only: the dead part of the pool is compacted away before it could push positions past 2^32
    // (flatten_placeable)
    if (brick_room(h.n_bricks, h.dead_bricks, f->words) == BrickRoom::too_big) return fail(AICB_ERR_INVALID, BRICKS_PAST_2_32);
    return AICB_OK;
}

// single_voxel_of's source (DeviceBlockJob::single) for a definition whose voxels the host does not read.
static uint32_t single_source(const aicb_block_desc &b) {
    if (!is_single_voxel(b)) return SINGLE_NONE;
    if (b.indices == nullptr) return b.n_palette ? SINGLE_FIRST : SINGLE_AIR;
    const bool at_origin = b.n_indices == 1 && b.voxel_bounds.lower[0] == 0 && b.voxel_bounds.lower[1] == 0 &&
                           b.voxel_bounds.lower[2] == 0;
    return at_origin ? SINGLE_INDEXED : SINGLE_AIR;
}

// flatten_blocks for n validated definitions whose voxels are in device memory: the kind of each single voxel is
// `kinds`' (read back from the device), everything else comes from the descriptors' sizes.  The voxel data, the
// blk_tab entries and, with `derive`, the light records are left to the device (DeviceDefs).
static void flatten_device(const SpaceHost &h, const aicb_block_desc *descs, size_t n, const std::vector<uint8_t> &kinds,
                           bool derive, FlatBlocks *f) {
    const size_t pal_base = h.n_palette / 2;
    f->recs.resize(n);
    f->extents.resize(n);
    f->blk_tab.assign(n, make_float4(0.0f, 0.0f, 0.0f, 0.0f));
    f->kinds.resize(n);
    f->light.assign(n, LightBlockDev{});
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        const bool single = is_single_voxel(b);
        const uint8_t kind = b.is_air ? KIND_INVISIBLE : single ? kinds[i] : KIND_RECURSIVE;
        const size_t words = kind == KIND_RECURSIVE ? b.n_indices : 0, entries = b.is_air ? 0 : single ? 1 : b.n_palette;
        const BlockRec r = block_rec(b, kind, (uint32_t)(h.n_bricks + f->words), (uint32_t)(pal_base + f->entries));
        f->recs[i] = r;
        f->extents[i] = {r.brick_off, (uint32_t)words, r.pal_off, (uint32_t)entries};
        f->kinds[i] = kind;
        if (!derive) f->light[i] = light_block(b);
        if (kind == KIND_RECURSIVE && b.n_palette > 32768) f->wide_bricks = true;
        f->words += words;
        f->entries += entries;
    }
    if (h.wide_bricks) f->wide_bricks = true;
}

// Every replica's narrow brick pool as a wide one, with room for `add` more words: once every replica's new buffer is
// allocated (grow_buffer's size rule, in words), each replica's words are re-encoded into it on the device, queued on
// its context's stream, and the old buffer is retired.
static aicb_status widen_bricks(Replicas r, size_t add) {
    SpaceHost &h = *r.scene[0]->host;
    std::vector<DeviceBuffer> wide(r.n);
    for (size_t i = 0; i < r.n; i++) {
        CU(cudaSetDevice(r.ctx[i]->device));
        const size_t bytes = std::max(round16((h.n_bricks + add) * 4), 2 * r.scene[i]->blocks.bricks.bytes());
        const aicb_status st = wide[i].ensure(bytes);
        if (st != AICB_OK) return free_each(r, wide, st);
    }
    for (size_t i = 0; i < r.n; i++) {
        aicb_ctx *ctx = r.ctx[i];
        BlockTable &t = r.scene[i]->blocks;
        const size_t want = (std::max<size_t>(h.n_bricks / 8, 1) + 255) / 256, cap = (size_t)ctx->num_sms * 16;
        CU(cudaSetDevice(ctx->device));
        if (h.n_bricks)
            widen_bricks_kernel<<<(unsigned)std::min(want, cap), 256, 0, ctx->stream.get()>>>(
                t.bricks.get<const uint16_t>(), wide[i].get<uint32_t>(), h.n_bricks);
        CU(cudaGetLastError());
        Retired retired{ctx, {}};
        if (t.bricks) retired.bufs.push_back(std::move(t.bricks));
        t.bricks = std::move(wide[i]);
        t.bind(r.scene[i]->ds);
    }
    h.wide_bricks = true;
    return AICB_OK;
}

// Placing `f` (flattened against `h`, with the pool in f's form) takes three steps.  room: on each replica, every
// buffer of table `t` grown to hold h's elements in use and f's (grow_buffer; the caller binds t, whatever fails).
// copy: on each replica, f queued on `stream` at the positions h gives: the voxel data after the pools' elements in
// use, the per-id records appended (indices == nullptr) or written at `indices`, in order, so a repeated index keeps
// its last definition.  book: f in the bookkeeping, once.
static aicb_status room(BlockTable &t, const SpaceHost &h, const FlatBlocks &f, const uint16_t *indices,
                        cudaStream_t stream, Retired &retired) {
    const size_t count = h.block_count(), added = indices ? 0 : f.kinds.size(), wb = f.brick_word_bytes();
    auto grow = [&](DeviceBuffer &b, size_t used, size_t add) {
        return add ? grow_buffer(b, used, used + add, stream, &retired.bufs) : AICB_OK;
    };
    TRY(grow(t.blocks, count * sizeof(BlockRec), added * sizeof(BlockRec)));
    TRY(grow(t.bricks, h.n_bricks * wb, f.words * wb));
    TRY(grow(t.palette, h.n_palette * sizeof(float4), 2 * f.entries * sizeof(float4)));
    TRY(grow(t.pal_tab, h.n_palette / 2 * sizeof(float2), f.entries * sizeof(float2)));
    TRY(grow(t.blk_tab, count * sizeof(float4), added * sizeof(float4)));
    return grow(t.light, count * sizeof(LightBlockDev), added * sizeof(LightBlockDev));
}

static aicb_status copy(const BlockTable &t, const SpaceHost &h, const FlatBlocks &f, const uint16_t *indices,
                        cudaStream_t stream) {
    auto put = [&](void *dst, const void *src, size_t bytes) {
        if (bytes) CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
        return AICB_OK;
    };
    const size_t wb = f.brick_word_bytes();
    TRY(put(t.bricks.get<char>() + h.n_bricks * wb, f.brick_words(), f.bricks.size() * wb));
    TRY(put(t.palette.get<float4>() + h.n_palette, f.palette.data(), f.palette.size() * sizeof(float4)));
    TRY(put(t.pal_tab.get<float2>() + h.n_palette / 2, f.pal_tab.data(), f.pal_tab.size() * sizeof(float2)));
    // the per-id records: one run of n at the end of the table, or one record at each index
    const size_t n = f.kinds.size(), runs = indices ? n : 1, len = indices ? 1 : n;
    for (size_t i = 0; i < runs; i++) {
        const size_t id = indices ? indices[i] : h.block_count();
        TRY(put(t.blocks.get<BlockRec>() + id, f.recs.data() + i, len * sizeof(BlockRec)));
        TRY(put(t.blk_tab.get<float4>() + id, f.blk_tab.data() + i, len * sizeof(float4)));
        TRY(put(t.light.get<LightBlockDev>() + id, f.light.data() + i, len * sizeof(LightBlockDev)));
    }
    return AICB_OK;
}

static void book(SpaceHost &h, const FlatBlocks &f, const uint16_t *indices) {
    const size_t n = f.kinds.size(), count = h.block_count(), added = indices ? 0 : n;
    h.kind.resize(count + added);
    h.extent.resize(count + added);
    for (size_t i = 0; i < n; i++) {
        const size_t id = indices ? indices[i] : count + i;
        if (indices) {   // the extents written over, an earlier definition of this call included, are dead
            h.dead_bricks += h.extent[id].n_bricks;
            h.dead_pal += h.extent[id].n_pal;
        }
        h.kind[id] = f.kinds[i];
        h.extent[id] = f.extents[i];
    }
    h.n_bricks += f.words;
    h.n_palette += 2 * f.entries;
    h.wide_bricks = f.wide_bricks;
}

// f (flatten_placeable) placed in every replica's table: room in each, then the copies, recorded in ev_delta (renders
// on other streams wait for it, launch_trace), and the bookkeeping.  Records are written over in place (`indices`)
// only once every replica has room and its context has been waited for (wait_context).
// Definitions in device memory (scenes_blocks_device): what the device read back (each single voxel's kind), the light
// records derive made on device 0, and per replica the jobs its kernels place (built by flatten_device).
struct DeviceDefs {
    std::vector<uint8_t> kinds;
    bool derive = false;
    std::vector<int32_t> derived;            // per definition: derive's record, or LIGHT_SINGLE
    const aicb_block_light *d_derived = nullptr;
    std::vector<DeviceBlockJob> jobs;
    uint64_t most_words = 0, most_entries = 0;
};

// The jobs of `f` (flattened against h) for `dev`: the caller's pointers and each definition's pool positions, and the
// per-id records of each id's last definition.
static void device_jobs(const SpaceHost &h, const aicb_block_desc *descs, const FlatBlocks &f, const uint16_t *indices,
                        DeviceDefs &dev) {
    const size_t n = f.kinds.size();
    dev.jobs.assign(n, DeviceBlockJob{});
    dev.most_words = dev.most_entries = 0;
    std::unordered_map<uint32_t, size_t> last;
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        DeviceBlockJob &J = dev.jobs[i];
        J.indices = b.indices;
        J.palette = b.palette;
        J.n_indices = b.n_indices;
        J.n_palette = (uint32_t)b.n_palette;
        J.single = single_source(b);
        J.kind = f.kinds[i];
        J.brick_off = f.extents[i].brick_off;
        J.pal_off = f.extents[i].pal_off;
        J.n_entries = f.extents[i].n_pal;
        J.id = (uint32_t)(indices ? indices[i] : h.block_count() + i);
        J.derived = dev.derive ? dev.derived[i] : LIGHT_GIVEN;
        J.light_visible = b.light_visible;
        J.rec = f.recs[i];
        J.light = f.light[i];
        dev.most_words = std::max<uint64_t>(dev.most_words, f.extents[i].n_bricks);
        dev.most_entries = std::max<uint64_t>(dev.most_entries, J.n_entries);
        if (indices) {
            const auto [at, first] = last.emplace(J.id, i);
            if (!first) {
                dev.jobs[at->second].id = NO_ID;
                at->second = i;
            }
        }
    }
}

// copy's device form: the jobs go up through the context's staging and blocks.cu's kernels write table `t` on the
// context's stream, reading the caller's buffers on device 0 (as a peer on the other devices).
static aicb_status copy_device(aicb_ctx *ctx, const BlockTable &t, const FlatBlocks &f, const DeviceDefs &dev) {
    cudaStream_t stream = ctx->stream.get();
    const size_t bytes = dev.jobs.size() * sizeof(DeviceBlockJob);
    TRY(delta_room(ctx, bytes));
    std::memcpy(ctx->h_delta.get(), dev.jobs.data(), bytes);
    CU(cudaMemcpyAsync(ctx->d_delta.get(), ctx->h_delta.get(), bytes, cudaMemcpyHostToDevice, stream));
    return issue_block_data(stream, ctx->d_delta.get<DeviceBlockJob>(), (uint32_t)dev.jobs.size(),
                            dev.most_words, dev.most_entries, f.wide_bricks, t, dev.d_derived);
}

static aicb_status place(Replicas r, const FlatBlocks &f, const uint16_t *indices, const DeviceDefs *dev) {
    SpaceHost &h = *r.scene[0]->host;
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *s = r.scene[i];
        CU(cudaSetDevice(r.ctx[i]->device));
        if (indices) TRY(wait_context(r.ctx[i]));
        Retired retired{r.ctx[i], {}};
        const aicb_status st = room(s->blocks, h, f, indices, r.ctx[i]->stream.get(), retired);
        s->blocks.bind(s->ds);
        TRY(st);
    }
    for (size_t i = 0; i < r.n; i++) {
        aicb_ctx *ctx = r.ctx[i];
        cudaStream_t stream = ctx->stream.get();
        CU(cudaSetDevice(ctx->device));
        if (!dev) TRY(copy(r.scene[i]->blocks, h, f, indices, stream));
        else TRY(copy_device(ctx, r.scene[i]->blocks, f, *dev));
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));
    }
    book(h, f, indices);
    return AICB_OK;
}

// Compacts every replica's brick pool and/or palette pool (palette and pal_tab), planned once from the bookkeeping:
// each pool's live extents, in pool order, go to the front of a new buffer of the live size, and each id's extent
// follows them.  Once every replica's new buffers are allocated, compact_pool_kernel gathers each replica's pools and
// rebase_blocks_kernel moves its records and blk_tab entries, queued on its context's stream, and the old buffers are
// retired.  The caller has waited for every context (wait_context), since a frame's hit records hold absolute pool
// positions.
static aicb_status compact_pools(Replicas r, bool bricks, bool palette) {
    SpaceHost &h = *r.scene[0]->host;
    const size_t count = h.block_count();
    std::vector<BlockTable::Extent> ext = h.extent;
    // one pool's plan: its live extents in pool order, gathered to the front; the ids' new offsets go to `ext`.  Each
    // run (neighbouring extents merged) of `elem`-byte elements becomes segments of at most 16 KiB of `segs`.
    std::vector<PoolSegment> segs;
    auto plan = [&](uint32_t BlockTable::Extent::*off, uint32_t BlockTable::Extent::*len, std::initializer_list<size_t> elems,
                    std::vector<std::pair<size_t, size_t>> *seg_ranges) {
        std::vector<uint32_t> order;
        for (uint32_t id = 0; id < count; id++)
            if (ext[id].*len) order.push_back(id);
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ext[a].*off < ext[b].*off; });
        std::vector<std::array<size_t, 3>> runs;   // src, dst, elements
        size_t live = 0;
        for (const uint32_t id : order) {
            BlockTable::Extent &e = ext[id];
            if (!runs.empty() && runs.back()[0] + runs.back()[2] == e.*off) runs.back()[2] += e.*len;
            else runs.push_back({e.*off, live, e.*len});
            e.*off = (uint32_t)live;
            live += e.*len;
        }
        const size_t SEG = 16384;
        for (const size_t elem : elems) {
            const size_t first = segs.size();
            for (const auto &r : runs)
                for (size_t k = 0; k < r[2] * elem; k += SEG)
                    segs.push_back({r[0] * elem + k, r[1] * elem + k, std::min(SEG, r[2] * elem - k)});
            seg_ranges->push_back({first, segs.size() - first});
        }
        return live;
    };
    std::vector<std::pair<size_t, size_t>> ranges;   // per buffer gathered: its segments in `segs`
    const size_t wb = h.brick_word_bytes();
    const size_t live_bricks = bricks ? plan(&BlockTable::Extent::brick_off, &BlockTable::Extent::n_bricks, {wb}, &ranges) : 0;
    const size_t live_pal = palette ? plan(&BlockTable::Extent::pal_off, &BlockTable::Extent::n_pal,
                                           {2 * sizeof(float4), sizeof(float2)}, &ranges) : 0;
    std::vector<uint2> off(count);
    for (size_t id = 0; id < count; id++) off[id] = make_uint2(ext[id].brick_off, ext[id].pal_off);
    struct NewPools {
        DeviceBuffer bricks, palette, pal_tab, segs, off;
    };
    std::vector<NewPools> to(r.n);
    for (size_t i = 0; i < r.n; i++) {
        NewPools &p = to[i];
        CU(cudaSetDevice(r.ctx[i]->device));
        aicb_status st = p.segs.ensure(segs.size() * sizeof(PoolSegment));
        if (st == AICB_OK) st = p.off.ensure(count * sizeof(uint2));
        if (st == AICB_OK && bricks) st = p.bricks.ensure(round16(live_bricks * wb));
        if (st == AICB_OK && palette) st = p.palette.ensure(live_pal * 2 * sizeof(float4));
        if (st == AICB_OK && palette) st = p.pal_tab.ensure(round16(live_pal * sizeof(float2)));
        if (st != AICB_OK) return free_each(r, to, st);
    }
    for (size_t i = 0; i < r.n; i++) {
        aicb_ctx *ctx = r.ctx[i];
        cudaStream_t stream = ctx->stream.get();
        BlockTable &t = r.scene[i]->blocks;
        NewPools &p = to[i];
        CU(cudaSetDevice(ctx->device));
        if (!segs.empty())
            CU(cudaMemcpyAsync(p.segs.get(), segs.data(), segs.size() * sizeof(PoolSegment), cudaMemcpyHostToDevice,
                               stream));
        if (count) CU(cudaMemcpyAsync(p.off.get(), off.data(), count * sizeof(uint2), cudaMemcpyHostToDevice, stream));
        Retired retired{ctx, {}};
        size_t next = 0;
        auto gather = [&](DeviceBuffer &buf, DeviceBuffer &into) {
            const auto [first, n] = ranges[next++];
            if (n) {
                const unsigned grid = (unsigned)std::min(n, (size_t)ctx->num_sms * 8);
                compact_pool_kernel<<<grid, 256, 0, stream>>>(buf.get<const uint8_t>(), into.get<uint8_t>(),
                                                              p.segs.get<const PoolSegment>() + first, (uint32_t)n);
            }
            if (buf) retired.bufs.push_back(std::move(buf));
            buf = std::move(into);
        };
        if (bricks) gather(t.bricks, p.bricks);
        if (palette) {
            gather(t.palette, p.palette);
            gather(t.pal_tab, p.pal_tab);
        }
        t.bind(r.scene[i]->ds);
        if (count)
            rebase_blocks_kernel<<<(unsigned)((count + 127) / 128), 128, 0, stream>>>(
                t.blocks.get<BlockRec>(), t.blk_tab.get<float4>(), p.off.get<const uint2>(), (uint32_t)count);
        retired.bufs.push_back(std::move(p.segs));
        retired.bufs.push_back(std::move(p.off));
        CU(cudaGetLastError());
    }
    if (bricks) {
        h.n_bricks = live_bricks;
        h.dead_bricks = 0;
    }
    if (palette) {
        h.n_palette = live_pal * 2;
        h.dead_pal = 0;
    }
    h.extent = std::move(ext);
    return AICB_OK;
}

// Scene creation's checks before it reads a block, in order: the bounds, then the NULLs.  *volume: the bounds' cubes.
static aicb_status check_scene_desc(const aicb_scene_desc *d, uint64_t *volume) {
    const int64_t LIM = 1 << 30;
    *volume = 1;
    for (int a = 0; a < 3; a++) {
        int64_t lo = d->bounds.lower[a], hi = lo + (int64_t)d->bounds.size[a];
        if (lo < -LIM || hi > LIM) return fail(AICB_ERR_INVALID, "space bounds must lie within +-2^30");
        *volume *= d->bounds.size[a];
        if (*volume > (1ull << 31)) return fail(AICB_ERR_INVALID, "space volume exceeds 2^31 cubes");
    }
    if (*volume && !d->block_ids) return fail(AICB_ERR_INVALID, "block_ids is NULL");
    if (*volume && d->n_blocks == 0) return fail(AICB_ERR_INVALID, "non-empty space with an empty block table");
    if (d->n_blocks && !d->blocks) return fail(AICB_ERR_INVALID, "blocks is NULL");
    return AICB_OK;
}

// A new scene's cells from the caller's ids (Z-major over the bounds, device memory the scene's device reaches):
// region_cells over boxes of whole x layers, or of one layer's whole rows, small enough that their work items (at
// most 2^30) are counted in 32 bits.  Each box's ids are one contiguous run of the caller's array.
static aicb_status device_cells(aicb_scene *s, const uint16_t *ids) {
    const uint32_t sx = (uint32_t)s->ds.size[0], sy = (uint32_t)s->ds.size[1], sz = (uint32_t)s->ds.size[2];
    const uint64_t LIMIT = 1ull << 30, row_items = (sz + (s->ds.wide_cells ? 3 : 7)) / (s->ds.wide_cells ? 4 : 8) + 1;
    const uint32_t ny = (uint32_t)std::min<uint64_t>(sy, std::max<uint64_t>(1, LIMIT / row_items));
    const uint32_t nx = ny < sy ? 1 : (uint32_t)std::min<uint64_t>(sx, std::max<uint64_t>(1, LIMIT / (row_items * sy)));
    for (uint32_t x = 0; x < sx; x += nx)
        for (uint32_t y = 0; y < sy; y += ny) {
            const RegionBox box = {{x, y, 0}, {std::min(nx, sx - x), std::min(ny, sy - y), sz}};
            TRY(region_cells(s, box, ids + ((size_t)x * sy + y) * sz, 0, nullptr, true, nullptr, nullptr));
        }
    return AICB_OK;
}

// The body of scene creation, host and device form, once the definitions are flattened (f, against an empty table):
// one scene per context, complete when it is returned (until then a failure frees every scene made), and then the
// host part, once.  The host form (dev == nullptr) uploads `cells`, encoded on the host, and the light.  The device
// form writes each replica's table with blocks.cu's kernels, encodes its cells from the caller's ids with
// k_region_cells (the kinds from the records just written) and copies the light, each replica reading device 0's
// buffers (as a peer on the other devices); its host mirror of the ids starts stale (refresh_mirror).
static aicb_status create_scenes(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, uint64_t volume,
                                 const FlatBlocks &f, const void *cells, const DeviceDefs *dev, aicb_scene **out) {
    auto host = std::make_unique<SpaceHost>();   // empty until every replica holds the table
    const bool wide = d->n_blocks > 16384;
    const size_t cell_bytes = volume * (wide ? 4 : 2);
    auto create = [&](aicb_ctx *c, aicb_scene **o) {
        CU(cudaSetDevice(c->device));
        std::unique_ptr<aicb_scene> s(new aicb_scene());
        s->ctx = c;
        s->host = host.get();
        DeviceScene &ds = s->ds;
        for (int a = 0; a < 3; a++) {
            ds.lo[a] = d->bounds.lower[a];
            ds.size[a] = (int32_t)d->bounds.size[a];
        }
        ds.wide_cells = wide ? 1 : 0;
        if (volume) {
            if (dev) TRY(s->d_cells.ensure(cell_bytes));
            else TRY(s->d_cells.upload(cells, cell_bytes));
            s->device_bytes += cell_bytes;
            if (d->light) {
                if (dev) {
                    TRY(s->d_light.ensure(volume * 4));
                    CU(cudaMemcpyPeerAsync(s->d_light.get(), c->device, d->light, ctx[0]->device, volume * 4,
                                           c->stream.get()));
                } else {
                    TRY(s->d_light.upload(d->light, volume * 4));
                }
                s->device_bytes += volume * 4;
            }
        }
        ds.cells = s->d_cells.get();
        ds.light = s->d_light.get<uint32_t>();
        ds.tables = c->d_lut.get<float>();
        build_block_sky(d->sky, &ds);
        Retired retired{c, {}};   // (a new table replaces no array)
        TRY(room(s->blocks, *host, f, nullptr, c->stream.get(), retired));
        s->blocks.bind(ds);
        if (dev) {
            TRY(copy_device(c, s->blocks, f, *dev));
            if (volume) TRY(device_cells(s.get(), d->block_ids));
            CU(cudaEventRecord(c->ev_delta.get(), c->stream.get()));
        } else {
            TRY(copy(s->blocks, *host, f, nullptr, c->stream.get()));
        }
        CU(cudaStreamSynchronize(c->stream.get()));
        *o = s.release();
        return AICB_OK;
    };
    for (size_t i = 0; i < n; i++) {
        const aicb_status st = create(ctx[i], &out[i]);
        if (st != AICB_OK) {
            for (size_t k = i; k-- > 0;) aicb_scene_destroy(out[k]);
            return st;
        }
    }
    host->volume = (size_t)volume;
    if (dev) host->ids_stale = true;
    else host->h_ids.assign(d->block_ids, d->block_ids + volume);
    host->light_max_distance = d->light_max_distance;
    book(*host, f, nullptr);
    out[0]->own_host = std::move(host);
    return AICB_OK;
}

aicb_status scenes_create(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, aicb_scene **out) {
    uint64_t volume;
    TRY(check_scene_desc(d, &volume));
    const SpaceHost empty;
    FlatBlocks f;
    TRY(flatten_blocks(empty, d->blocks, d->n_blocks, nullptr, &f));

    // ---- cells: block id with its kind in the top bits --------------------------------------------------------------
    const bool wide = d->n_blocks > 16384;
    std::vector<uint16_t> cells16(wide ? 0 : volume);
    std::vector<uint32_t> cells32(wide ? volume : 0);
    for (size_t i = 0; i < volume; i++) {
        const uint16_t id = d->block_ids[i];
        if (id >= d->n_blocks) return fail(AICB_ERR_INVALID, "block id out of range");
        if (wide) cells32[i] = cell_word(id, f.kinds[id], true);
        else cells16[i] = (uint16_t)cell_word(id, f.kinds[id], false);
    }
    return create_scenes(ctx, n, d, volume, f, wide ? (const void *)cells32.data() : cells16.data(), nullptr, out);
}

// flatten_blocks against the scene's table, for an update (`indices`) or an append (nullptr) of the scene's replicas,
// such that the result can be placed: brick positions are u32, so when the live data fits but the pool's words in use
// plus the new ones would not (brick_room), every replica's brick pool is compacted first and the definitions are
// flattened again against the compacted table.  A compaction moves the pools, so each replica's context is waited
// for first (wait_context).  Wide definitions for a narrow pool widen every replica's pool first.
static aicb_status flatten_placeable(Replicas r, const aicb_block_desc *descs, size_t n_blocks, const uint16_t *indices,
                                     DeviceDefs *dev, FlatBlocks *f) {
    const SpaceHost &h = *r.scene[0]->host;
    auto flatten = [&]() {
        if (!dev) return flatten_blocks(h, descs, n_blocks, indices, f);
        flatten_device(h, descs, n_blocks, dev->kinds, dev->derive, f);
        return AICB_OK;
    };
    TRY(flatten());
    if (brick_room(h.n_bricks, h.dead_bricks, f->words) == BrickRoom::compact_first) {
        for (size_t i = 0; i < r.n; i++) {
            CU(cudaSetDevice(r.ctx[i]->device));
            TRY(wait_context(r.ctx[i]));
        }
        TRY(compact_pools(r, true, false));
        *f = FlatBlocks();
        TRY(flatten());
    }
    if (dev) device_jobs(h, descs, *f, indices, *dev);
    return f->wide_bricks && !h.wide_bricks ? widen_bricks(r, f->words) : AICB_OK;
}

// The context's staging (h_delta / d_delta) with room for a batch of `bytes`, once the previous batch has left it.
aicb_status delta_room(aicb_ctx *ctx, size_t bytes) {
    if (std::min(ctx->h_delta.bytes(), ctx->d_delta.bytes()) < bytes) {
        if (ctx->h_delta) cudaEventSynchronize(ctx->ev_delta.get());   // the previous batch's copy may still read it
        ctx->h_delta.reset();
        ctx->d_delta.reset();
        const size_t cap = bytes < 65536 ? 65536 : bytes * 2;
        TRY(ctx->h_delta.ensure(cap));
        TRY(ctx->d_delta.ensure(cap));
    }
    CU(cudaEventSynchronize(ctx->ev_delta.get()));  // the previous batch has left the staging buffer
    return AICB_OK;
}

// One pinned staging buffer, one H2D copy and one scatter kernel per batch and replica, stream-ordered before any later
// render of the context.  The batch is validated and built once: a cube named twice keeps its last value (the scatter
// is parallel, so duplicates are resolved here).
aicb_status scenes_update_cubes(Replicas r, const int32_t (*cubes)[3], const uint16_t *ids, const uint8_t (*light)[4],
                                size_t n) {
    if (n && (!cubes || !ids)) return fail(AICB_ERR_INVALID, "NULL argument");
    CU(cudaSetDevice(r.ctx[0]->device));
    if (n == 0) return AICB_OK;
    SpaceHost &h = *r.scene[0]->host;
    const DeviceScene &ds = r.scene[0]->ds;
    // validate and build the whole batch before touching any state
    std::vector<uint32_t> idx(n);
    std::vector<CubeDelta> ops;
    ops.reserve(n);
    std::unordered_map<uint32_t, uint32_t> seen;
    seen.reserve(n * 2);
    for (size_t i = 0; i < n; i++) {
        const uint32_t dx = (uint32_t)(cubes[i][0] - ds.lo[0]), dy = (uint32_t)(cubes[i][1] - ds.lo[1]),
                       dz = (uint32_t)(cubes[i][2] - ds.lo[2]);
        if (dx >= (uint32_t)ds.size[0] || dy >= (uint32_t)ds.size[1] || dz >= (uint32_t)ds.size[2])
            return fail(AICB_ERR_INVALID, "cube out of bounds");
        if (ids[i] >= h.block_count()) return fail(AICB_ERR_INVALID, "block id out of range");
        idx[i] = (uint32_t)(((size_t)dx * ds.size[1] + dy) * ds.size[2] + dz);
        CubeDelta op;
        op.idx = idx[i];
        op.cell = cell_word(ids[i], h.kind[ids[i]], ds.wide_cells);
        op.has_light = (light && r.scene[0]->d_light) ? 1u : 0u;
        op.light = 0;
        if (op.has_light) std::memcpy(&op.light, light[i], 4);
        const auto [at, first] = seen.emplace(op.idx, (uint32_t)ops.size());
        if (first) ops.push_back(op); else ops[at->second] = op;
    }
    TRY(refresh_mirror(r.scene[0]));   // (the mirror is written below)
    const uint32_t m = (uint32_t)ops.size();
    const size_t bytes = (size_t)m * sizeof(CubeDelta);
    for (size_t k = 0; k < r.n; k++) {
        aicb_scene *s = r.scene[k];
        aicb_ctx *ctx = r.ctx[k];
        cudaStream_t stream = ctx->stream.get();
        CU(cudaSetDevice(ctx->device));
        TRY(delta_room(ctx, bytes));
        std::memcpy(ctx->h_delta.get(), ops.data(), bytes);
        CU(cudaMemcpyAsync(ctx->d_delta.get(), ctx->h_delta.get(), bytes, cudaMemcpyHostToDevice, stream));
        scatter_cubes_kernel<<<(m + 127) / 128, 128, 0, stream>>>(ctx->d_delta.get<const CubeDelta>(), m, s->ds.wide_cells,
                                                                  s->d_cells.get(), s->d_light.get<uint32_t>());
        CU(cudaGetLastError());
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));  // renders on other streams wait for it (launch_trace)
    }
    if (!h.h_ids.empty())
        for (size_t i = 0; i < n; i++) h.h_ids[idx[i]] = ids[i];
    return AICB_OK;
}

aicb_status check_box(const aicb_scene *s, const aicb_aab *region, RegionBox *box) {
    if (!region) return fail(AICB_ERR_INVALID, "NULL argument");
    for (int a = 0; a < 3; a++) {
        const int64_t lo = (int64_t)region->lower[a] - s->ds.lo[a];
        if (lo < 0 || lo + (int64_t)region->size[a] > (int64_t)s->ds.size[a])
            return fail(AICB_ERR_INVALID, "region is not inside the bounds");
        box->lo[a] = (uint32_t)lo;
        box->size[a] = region->size[a];
    }
    // the kernels' work items, at most size[2] / 4 + 2 per row, are counted in 32 bits
    if ((uint64_t)box->size[0] * box->size[1] * (box->size[2] / 4 + 2) > 0xffffffffull)
        return fail(AICB_ERR_INVALID, "region too large");
    return AICB_OK;
}

aicb_status check_region(const aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                         RegionBox *box) {
    TRY(check_box(s, region, box));
    const size_t count = s->host->block_count();
    if (!ids) {
        if (uniform_id >= count) return fail(AICB_ERR_INVALID, "block id out of range");
        return AICB_OK;
    }
    uint16_t highest = 0;
    for (size_t i = 0, n = box->volume(); i < n; i++) highest = std::max(highest, ids[i]);
    if (box->volume() && highest >= count) return fail(AICB_ERR_INVALID, "block id out of range");
    return AICB_OK;
}

void mirror_region(SpaceHost &h, const DeviceScene &ds, const RegionBox &box, const uint16_t *ids,
                   uint16_t uniform_id) {
    if (h.h_ids.empty()) return;
    const size_t rows = (size_t)box.size[0] * box.size[1], sz = box.size[2];
    for (size_t row = 0; row < rows; row++) {
        uint16_t *dst = h.h_ids.data() + ((size_t)(box.lo[0] + row / box.size[1]) * ds.size[1] + box.lo[1] +
                                          row % box.size[1]) * ds.size[2] + box.lo[2];
        if (ids) std::memcpy(dst, ids + row * sz, sz * 2);
        else std::fill(dst, dst + sz, uniform_id);
    }
}

aicb_status region_cells(aicb_scene *s, const RegionBox &box, const uint16_t *ids, uint16_t uniform_id,
                         const uint8_t (*light)[4], bool on_device, uint32_t *d_mask, uint32_t *d_n_changed) {
    aicb_ctx *ctx = s->ctx;
    cudaStream_t stream = ctx->stream.get();
    const size_t vol = box.volume(), rows = (size_t)box.size[0] * box.size[1], sz = box.size[2];
    if (!s->d_light) light = nullptr;
    // the ids, then (16-byte aligned) the texels
    const size_t id_bytes = ids ? (vol * 2 + 15) / 16 * 16 : 0, bytes = id_bytes + (light ? vol * 4 : 0);
    if (bytes && !on_device) {
        TRY(delta_room(ctx, bytes));
        if (ids) std::memcpy(ctx->h_delta.get(), ids, vol * 2);
        if (light) std::memcpy(ctx->h_delta.get<char>() + id_bytes, light, vol * 4);
        CU(cudaMemcpyAsync(ctx->d_delta.get(), ctx->h_delta.get(), bytes, cudaMemcpyHostToDevice, stream));
    }
    if (d_mask) CU(cudaMemsetAsync(d_mask, 0, (vol + 31) / 32 * 4, stream));
    const bool wide = s->ds.wide_cells;
    const uint32_t per = wide ? 4u : 8u, chunks_per_row = (uint32_t)((sz + per - 1) / per + 1);
    const uint32_t n_items = (uint32_t)(rows * chunks_per_row);
    const uint16_t *d_ids = on_device ? ids : ids ? ctx->d_delta.get<const uint16_t>() : nullptr;
    auto launch = [&](auto kernel) {
        kernel<<<(n_items + 255) / 256, 256, 0, stream>>>(s->ds, box, d_ids, uniform_id, chunks_per_row, n_items, d_mask,
                                                          d_n_changed);
    };
    switch ((wide ? 4 : 0) | (ids ? 0 : 2) | (d_mask ? 1 : 0)) {
    case 0: launch(k_region_cells<false, false, false>); break;
    case 1: launch(k_region_cells<false, false, true>); break;
    case 2: launch(k_region_cells<false, true, false>); break;
    case 3: launch(k_region_cells<false, true, true>); break;
    case 4: launch(k_region_cells<true, false, false>); break;
    case 5: launch(k_region_cells<true, false, true>); break;
    case 6: launch(k_region_cells<true, true, false>); break;
    default: launch(k_region_cells<true, true, true>); break;
    }
    if (light) {
        const uint32_t cpr = (uint32_t)((sz + 3) / 4 + 1), n = (uint32_t)(rows * cpr);
        const uint32_t *texels = on_device ? (const uint32_t *)light
                                           : (const uint32_t *)(ctx->d_delta.get<const char>() + id_bytes);
        k_region_texels<<<(n + 255) / 256, 256, 0, stream>>>(s->ds, box, texels, cpr, n, s->d_light.get<uint32_t>());
    }
    CU(cudaGetLastError());
    return AICB_OK;
}

// The box form of scenes_update_cubes: nothing is built per cube on the host.  Every replica stages the caller's dense
// arrays in its own context and writes its own cells and texels, stream-ordered like a cube update.
aicb_status scenes_update_region(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                 const uint8_t (*light)[4]) {
    RegionBox box;
    TRY(check_region(r.scene[0], region, ids, uniform_id, &box));
    if (box.volume() == 0) return AICB_OK;
    TRY(refresh_mirror(r.scene[0]));
    for (size_t k = 0; k < r.n; k++) {
        CU(cudaSetDevice(r.ctx[k]->device));
        TRY(region_cells(r.scene[k], box, ids, uniform_id, light, false, nullptr, nullptr));
        CU(cudaEventRecord(r.ctx[k]->ev_delta.get(), r.ctx[k]->stream.get()));  // renders on other streams wait for it
    }
    mirror_region(*r.scene[0]->host, r.scene[0]->ds, box, ids, uniform_id);
    return AICB_OK;
}

// The body of aicb_scene_update_blocks and its device form (dev: the definitions' voxels are in device memory).  The
// host form finds the cubes whose block changes kind in the host mirror and scatters their new words; the device form
// re-encodes them in one pass over every replica's cells against a per-id table of new words, so it needs no mirror.
static aicb_status update_blocks(Replicas r, const uint16_t *indices, const aicb_block_desc *descs, size_t n_blocks,
                                 DeviceDefs *dev) {
    const SpaceHost &h = *r.scene[0]->host;
    FlatBlocks f;
    TRY(flatten_placeable(r, descs, n_blocks, indices, dev, &f));
    // cubes that hold a block whose kind changes carry the new kind in their cell words
    std::vector<uint8_t> kind(h.kind);
    for (size_t i = 0; i < n_blocks; i++) kind[indices[i]] = f.kinds[i];
    const bool wide = r.scene[0]->ds.wide_cells;
    std::vector<CubeDelta> ops;
    std::vector<uint32_t> word;   // the device form's table: per id its new cell word, or NO_WORD
    if (kind != h.kind && dev) {
        word.assign(kind.size(), NO_WORD);
        for (size_t id = 0; id < kind.size(); id++)
            if (kind[id] != h.kind[id]) word[id] = cell_word((uint32_t)id, kind[id], wide);
    } else if (kind != h.kind) {
        TRY(refresh_mirror(r.scene[0]));
        if (h.h_ids.size() != h.volume) return fail(AICB_ERR_INVALID, "scene has no host mirror of its block ids");
        uint32_t idx = 0;
        for (const uint16_t id : h.h_ids) {
            if (kind[id] != h.kind[id]) ops.push_back({idx, cell_word(id, kind[id], wide), 0, 0});
            idx++;
        }
    }
    TRY(place(r, f, indices, dev));   // (which waits for every context: compaction moves the pools)
    const bool compact_bricks = h.dead_bricks > h.n_bricks - h.dead_bricks;
    const bool compact_palette = h.dead_pal > h.n_palette / 2 - h.dead_pal;
    if (compact_bricks || compact_palette) TRY(compact_pools(r, compact_bricks, compact_palette));
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *sc = r.scene[i];
        aicb_ctx *ctx = r.ctx[i];
        cudaStream_t stream = ctx->stream.get();
        CU(cudaSetDevice(ctx->device));
        Retired retired{ctx, {}};
        if (!ops.empty()) {
            DeviceBuffer d_ops;
            TRY(d_ops.ensure(ops.size() * sizeof(CubeDelta)));
            CU(cudaMemcpyAsync(d_ops.get(), ops.data(), ops.size() * sizeof(CubeDelta), cudaMemcpyHostToDevice, stream));
            scatter_cubes_kernel<<<(unsigned)((ops.size() + 127) / 128), 128, 0, stream>>>(
                d_ops.get<const CubeDelta>(), (uint32_t)ops.size(), sc->ds.wide_cells, sc->d_cells.get(),
                sc->d_light.get<uint32_t>());
            retired.bufs.push_back(std::move(d_ops));
            CU(cudaGetLastError());
        }
        if (!word.empty() && h.volume) {
            DeviceBuffer d_word;
            TRY(d_word.upload(word.data(), word.size() * 4));
            TRY(issue_rekind_cells(ctx, sc->d_cells.get(), wide, h.volume, d_word.get<const uint32_t>()));
            retired.bufs.push_back(std::move(d_word));
        }
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));
        TRY(wait_context(ctx));   // the call returns once its writes are done
    }
    return AICB_OK;
}

aicb_status scenes_update_blocks(Replicas r, const uint16_t *indices, const aicb_block_desc *descs, size_t n_blocks) {
    if (n_blocks && (!indices || !descs)) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n_blocks == 0) return AICB_OK;
    return update_blocks(r, indices, descs, n_blocks, nullptr);
}

// The copies are queued on the context's stream and ev_delta is recorded behind them, as aicb_scene_update_cubes does:
// a frame issued later on another stream waits for them (launch_trace).  The new entries go to spare capacity that no
// cell refers to until a later, stream-ordered cube update, so a frame in flight is not disturbed; an array that has to
// move is freed only after it (Retired).
static aicb_status append_blocks(Replicas r, const aicb_block_desc *descs, size_t n_blocks, DeviceDefs *dev) {
    const SpaceHost &h = *r.scene[0]->host;
    FlatBlocks f;
    TRY(flatten_placeable(r, descs, n_blocks, nullptr, dev, &f));
    // u16 cells hold ids below 16384 (scenes_create): a table that grows past that takes u32 cells, re-encoded behind
    // every queued cube update of each context
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *sc = r.scene[i];
        aicb_ctx *ctx = r.ctx[i];
        if (sc->ds.wide_cells || h.block_count() + n_blocks <= 16384) continue;
        CU(cudaSetDevice(ctx->device));
        if (h.volume) {
            Retired retired{ctx, {}};
            DeviceBuffer wide;
            TRY(wide.ensure(h.volume * 4));
            const size_t want = (std::max<size_t>(h.volume / 8, 1) + 255) / 256, cap = (size_t)ctx->num_sms * 16;
            widen_cells_kernel<<<(unsigned)std::min(want, cap), 256, 0, ctx->stream.get()>>>(
                sc->d_cells.get<const uint16_t>(), wide.get<uint32_t>(), h.volume);
            CU(cudaGetLastError());
            retired.bufs.push_back(std::move(sc->d_cells));
            sc->d_cells = std::move(wide);
            sc->ds.cells = sc->d_cells.get();
            sc->device_bytes += h.volume * 2;
        }
        sc->ds.wide_cells = 1;
    }
    return place(r, f, nullptr, dev);
}

aicb_status scenes_append_blocks(Replicas r, const aicb_block_desc *descs, size_t n_blocks) {
    if (n_blocks && !descs) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n_blocks == 0) return AICB_OK;
    return append_blocks(r, descs, n_blocks, nullptr);
}

// Mutation::fill_uniform over the whole Space (space.rs:1461-1474), the source of SpaceChange::EveryBlock: the table
// becomes [block] in exact-size buffers, as a new scene's, and every cell id 0 with its kind, written on the device
// (u32 cells go back to u16: a one-block table fits them).  Light is not touched.  Each replica's context is waited for
// first, since the table and the cells are replaced, and the call returns once its writes are done.  Every replica's
// new arrays are allocated before any replica changes, so a failure leaves the scene as it was.  `f` is the block
// flattened against `empty`, an empty table's bookkeeping; with `dev` its voxels are in device memory (copy_device).
static aicb_status fill_uniform(Replicas r, const SpaceHost &empty, const FlatBlocks &f, const DeviceDefs *dev) {
    const uint32_t word = cell_word(0, f.kinds[0], false);
    SpaceHost &h = *r.scene[0]->host;
    struct Fresh {
        BlockTable table;
        DeviceBuffer narrow;   // the u16 cells of a replica that has u32 cells
    };
    std::vector<Fresh> fresh(r.n);
    for (size_t i = 0; i < r.n; i++) {
        CU(cudaSetDevice(r.ctx[i]->device));
        TRY(wait_context(r.ctx[i]));
        Retired retired{r.ctx[i], {}};   // (a new table replaces no array)
        aicb_status st = AICB_OK;
        if (r.scene[i]->ds.wide_cells && h.volume) st = fresh[i].narrow.ensure(h.volume * 2);
        if (st == AICB_OK) st = room(fresh[i].table, empty, f, nullptr, r.ctx[i]->stream.get(), retired);
        if (st != AICB_OK) return free_each(r, fresh, st);
    }
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *sc = r.scene[i];
        aicb_ctx *ctx = r.ctx[i];
        cudaStream_t stream = ctx->stream.get();
        CU(cudaSetDevice(ctx->device));
        Retired retired{ctx, {}};
        BlockTable &old = sc->blocks;
        for (DeviceBuffer *b : {&old.blocks, &old.blk_tab, &old.light, &old.bricks, &old.palette, &old.pal_tab})
            if (*b) retired.bufs.push_back(std::move(*b));
        sc->blocks = std::move(fresh[i].table);
        sc->blocks.bind(sc->ds);
        if (dev) TRY(copy_device(ctx, sc->blocks, f, *dev));
        else TRY(copy(sc->blocks, empty, f, nullptr, stream));
        if (fresh[i].narrow) {
            retired.bufs.push_back(std::move(sc->d_cells));
            sc->d_cells = std::move(fresh[i].narrow);
            sc->ds.cells = sc->d_cells.get();
            sc->device_bytes -= h.volume * 2;
        }
        sc->ds.wide_cells = 0;
        if (h.volume) {
            const size_t want = (std::max<size_t>(h.volume / 8, 1) + 255) / 256, cap = (size_t)ctx->num_sms * 16;
            fill_cells_kernel<<<(unsigned)std::min(want, cap), 256, 0, stream>>>(sc->d_cells.get<uint16_t>(), h.volume,
                                                                                  word);
            CU(cudaGetLastError());
        }
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));
        TRY(wait_context(ctx));   // the call returns once its writes are done
    }
    h.kind.clear();
    h.extent.clear();
    h.n_bricks = h.n_palette = h.dead_bricks = h.dead_pal = 0;
    book(h, f, nullptr);
    h.h_ids.assign(h.volume, 0);
    h.ids_stale = false;
    return AICB_OK;
}

aicb_status scenes_fill_uniform(Replicas r, const aicb_block_desc *block) {
    if (!block) return fail(AICB_ERR_INVALID, "NULL argument");
    const SpaceHost empty;
    FlatBlocks f;
    TRY(flatten_blocks(empty, block, 1, nullptr, &f));
    return fill_uniform(r, empty, f, nullptr);
}

// Space::set_physics (space.rs:609-630) on a scene's replicas: the sky tables once (Sky::for_blocks, Sky::mean), then, if
// the sky or the LightPhysics differs, each replica's context is waited for (an issued frame may still read the light
// volume a change to None frees) and light.cu applies the change.  The sky is read as aicb_scene_create reads it.
aicb_status scenes_set_physics(Replicas r, const aicb_sky *sky, uint8_t light_max_distance) {
    if (!sky) return fail(AICB_ERR_INVALID, "NULL argument");
    const DeviceScene &cur = r.scene[0]->ds;
    DeviceScene next = cur;
    build_block_sky(*sky, &next);
    bool same_sky = next.sky_kind == cur.sky_kind;
    for (int k = 0; k < (next.sky_kind ? 8 : 1); k++)   // Uniform's colour, or the eight octants'
        for (int i = 0; i < 3; i++) same_sky = same_sky && next.sky_colors[k][i] == cur.sky_colors[k][i];
    if (same_sky && light_max_distance == r.scene[0]->host->light_max_distance)
        return AICB_OK;   // no SpaceChange::Physics
    for (size_t i = 0; i < r.n; i++) {
        CU(cudaSetDevice(r.ctx[i]->device));
        TRY(wait_context(r.ctx[i]));
    }
    const aicb_status st = light_set_physics(r, next, light_max_distance);
    cudaSetDevice(r.ctx[0]->device);
    return st;
}

// Every replica takes the texels, ordered behind its queued cube updates; renders on other streams wait for ev_delta
// (launch_trace).  A replica with no light volume gets one.
aicb_status scenes_upload_light(Replicas r, const uint8_t (*light)[4], size_t n_texels) {
    if (!light) return fail(AICB_ERR_INVALID, "NULL argument");
    const size_t volume = r.scene[0]->host->volume;
    if (n_texels != volume) return fail(AICB_ERR_INVALID, "light volume size mismatch");
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *s = r.scene[i];
        cudaStream_t stream = r.ctx[i]->stream.get();
        CU(cudaSetDevice(r.ctx[i]->device));
        if (!s->d_light && volume) {
            TRY(s->d_light.ensure(volume * 4));
            s->device_bytes += volume * 4;
            s->ds.light = s->d_light.get<uint32_t>();
        }
        if (volume) {
            CU(cudaMemcpyAsync(s->d_light.get(), light, volume * 4, cudaMemcpyHostToDevice, stream));
            CU(cudaEventRecord(r.ctx[i]->ev_delta.get(), stream));
            CU(cudaStreamSynchronize(stream));
        }
    }
    return AICB_OK;
}


// ---------------------------------------------------------------------------------------------
// scene inputs in device memory (internal.h): validated on the device, one verdict read back
// ---------------------------------------------------------------------------------------------
aicb_status join_caller(aicb_ctx *const *ctx, size_t n, cudaStream_t caller) {
    if (!caller) return AICB_OK;
    CU(cudaSetDevice(ctx[0]->device));
    CU(cudaEventRecord(ctx[0]->ev_join.get(), caller));
    for (size_t i = 0; i < n; i++) {
        if (ctx[i]->stream.get() == caller) continue;
        CU(cudaSetDevice(ctx[i]->device));
        CU(cudaStreamWaitEvent(ctx[i]->stream.get(), ctx[0]->ev_join.get(), 0));
    }
    CU(cudaSetDevice(ctx[0]->device));
    return AICB_OK;
}

aicb_status release_caller(aicb_ctx *ctx, cudaStream_t caller) {
    if (!caller || caller == ctx->stream.get()) return AICB_OK;
    CU(cudaSetDevice(ctx->device));
    CU(cudaEventRecord(ctx->ev_join.get(), ctx->stream.get()));
    CU(cudaStreamWaitEvent(caller, ctx->ev_join.get(), 0));
    return AICB_OK;
}

// Every replica's stream has finished the call's work (the group calls return once their writes are done).
static aicb_status settle_replicas(Replicas r) {
    if (r.n == 1) return AICB_OK;
    for (size_t i = 0; i < r.n; i++) {
        CU(cudaSetDevice(r.ctx[i]->device));
        CU(cudaStreamSynchronize(r.ctx[i]->stream.get()));
    }
    CU(cudaSetDevice(r.ctx[0]->device));
    return AICB_OK;
}

// At least `bytes` of the context's d_inputs, once its stream no longer uses the smaller buffer.
static aicb_status inputs_room(aicb_ctx *ctx, size_t bytes) {
    if (ctx->d_inputs.bytes() >= bytes) return AICB_OK;
    CU(cudaStreamSynchronize(ctx->stream.get()));
    return ctx->d_inputs.ensure(bytes);
}

static size_t align256(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// One entry of a cube list per thread: its Z-major index (0 for a cube out of bounds) and its list position, and the
// list's first bad entry (the host loop's first failing check) by atomicMin.
static __global__ void __launch_bounds__(256) k_check_cubes(const int32_t *__restrict__ cubes, const uint16_t *__restrict__ ids,
                                                            uint32_t n, int3 lo, int3 size, uint32_t n_blocks,
                                                            uint32_t *__restrict__ idx, uint32_t *__restrict__ pos,
                                                            InputVerdict *v) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t dx = (uint32_t)(cubes[3 * i] - lo.x), dy = (uint32_t)(cubes[3 * i + 1] - lo.y),
                   dz = (uint32_t)(cubes[3 * i + 2] - lo.z);
    const bool inside = dx < (uint32_t)size.x && dy < (uint32_t)size.y && dz < (uint32_t)size.z;
    idx[i] = inside ? (dx * (uint32_t)size.y + dy) * (uint32_t)size.z + dz : 0u;
    pos[i] = i;
    if (!inside) atomicMin(&v->first_bad, 2ull * i);
    else if (ids[i] >= n_blocks) atomicMin(&v->first_bad, 2ull * i + 1);
}

// Whether any id of a dense array is past the table (first_bad = 1); grid-stride.
static __global__ void __launch_bounds__(256) k_check_ids(const uint16_t *__restrict__ ids, size_t n, uint32_t n_blocks,
                                                          InputVerdict *v) {
    bool bad = false;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        bad |= ids[i] >= n_blocks;
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31u) == 0) atomicMin(&v->first_bad, 1ull);
}

// aicb_scene_update_cubes' batch from a sorted cube list: the last entry for each cube (the last of its run, the sort
// being stable) gives its CubeDelta, the kind from the block table's records; the deltas go to `ops` in any order
// (their cubes are distinct) and are counted in v->count.  An entry with an id past the table is skipped: its call is
// rejected.
static __global__ void __launch_bounds__(256) k_cube_deltas(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                            uint32_t n, const uint16_t *__restrict__ ids,
                                                            const uint32_t *__restrict__ light, const BlockRec *blocks,
                                                            uint32_t n_blocks, uint32_t wide, CubeDelta *ops, InputVerdict *v) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n || (p + 1 < n && keys[p + 1] == keys[p])) return;
    const uint32_t i = vals[p], id = ids[i];
    if (id >= n_blocks) return;
    CubeDelta op;
    op.idx = keys[p];
    op.cell = id | (__ldg(&blocks[id].kind_res) & 0xffu) << (wide ? 16 : 14);
    op.light = light ? light[i] : 0u;
    op.has_light = light ? 1u : 0u;
    ops[atomicAdd(&v->count, 1u)] = op;
}

// Each cube's block id from its cell word (16-bit cells: id | kind << 14; 32-bit: id | kind << 16); grid-stride.
static __global__ void __launch_bounds__(256) k_decode_ids(const void *__restrict__ cells, uint32_t wide, size_t n,
                                                           uint16_t *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = wide ? (uint16_t)(((const uint32_t *)cells)[i] & 0xffffu) : (uint16_t)(((const uint16_t *)cells)[i] & 0x3fffu);
}

static unsigned stride_grid(const aicb_ctx *ctx, size_t n) {
    return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)ctx->num_sms * 16));
}

static aicb_status reset_verdict(InputVerdict *v, cudaStream_t stream) {
    CU(cudaMemsetAsync(&v->first_bad, 0xff, sizeof v->first_bad, stream));
    CU(cudaMemsetAsync(&v->count, 0, sizeof v->count, stream));
    return AICB_OK;
}

aicb_status stage_cube_list(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *ids, uint32_t n,
                            size_t extra_bytes, size_t temp_bytes, CubeList *l) {
    aicb_ctx *ctx = s->ctx;
    cudaStream_t stream = ctx->stream.get();
    int end_bit = 1;
    while (end_bit < 32 && ((uint64_t)1 << end_bit) < s->host->volume) end_bit++;
    size_t sort_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                       (const uint32_t *)nullptr, (uint32_t *)nullptr, n, 0, end_bit, stream));
    l->temp_bytes = std::max(sort_bytes, temp_bytes);
    const size_t a = align256((size_t)n * 4);
    TRY(inputs_room(ctx, 256 + 4 * a + align256(extra_bytes) + l->temp_bytes));
    char *p = ctx->d_inputs.get<char>();
    l->verdict = (InputVerdict *)p;
    l->idx = (uint32_t *)(p + 256);
    uint32_t *pos = (uint32_t *)(p + 256 + a);
    l->keys = (uint32_t *)(p + 256 + 2 * a);
    l->vals = (uint32_t *)(p + 256 + 3 * a);
    l->extra = p + 256 + 4 * a;
    l->temp = p + 256 + 4 * a + align256(extra_bytes);
    const DeviceScene &ds = s->ds;
    TRY(reset_verdict(l->verdict, stream));
    k_check_cubes<<<(n + 255) / 256, 256, 0, stream>>>(&cubes[0][0], ids, n, make_int3(ds.lo[0], ds.lo[1], ds.lo[2]),
                                                       make_int3(ds.size[0], ds.size[1], ds.size[2]),
                                                       (uint32_t)s->host->block_count(), l->idx, pos, l->verdict);
    CU(cudaGetLastError());
    size_t tb = l->temp_bytes;
    CU(cub::DeviceRadixSort::SortPairs(l->temp, tb, l->idx, l->keys, pos, l->vals, n, 0, end_bit, stream));
    return AICB_OK;
}

aicb_status read_verdict(aicb_ctx *ctx, const InputVerdict *d_verdict, uint32_t *count) {
    InputVerdict v;
    CU(cudaMemcpyAsync(&v, d_verdict, sizeof v, cudaMemcpyDeviceToHost, ctx->stream.get()));
    CU(cudaStreamSynchronize(ctx->stream.get()));
    if (v.first_bad != ~0ull) return fail(AICB_ERR_INVALID, v.first_bad & 1 ? "block id out of range" : "cube out of bounds");
    *count = v.count;
    return AICB_OK;
}

aicb_status check_region_device(Replicas r, const aicb_aab *region, const uint16_t *d_ids, uint16_t uniform_id,
                                const uint8_t (*d_light)[4], cudaStream_t caller, RegionBox *box) {
    aicb_scene *s = r.scene[0];
    aicb_ctx *ctx = r.ctx[0];
    TRY(check_box(s, region, box));
    CU(cudaSetDevice(ctx->device));
    const size_t count = s->host->block_count(), vol = box->volume();
    if (!d_ids && uniform_id >= count) return fail(AICB_ERR_INVALID, "block id out of range");
    if (vol == 0) return AICB_OK;
    if (d_ids) TRY(check_device_pointer(d_ids, ctx->device, false, 2, "block_ids"));
    if (d_light) TRY(check_device_pointer(d_light, ctx->device, false, 4, "light"));
    TRY(join_caller(r.ctx, r.n, caller));
    if (!d_ids) return AICB_OK;
    TRY(inputs_room(ctx, 256));
    InputVerdict *v = ctx->d_inputs.get<InputVerdict>();
    TRY(reset_verdict(v, ctx->stream.get()));
    k_check_ids<<<stride_grid(ctx, vol), 256, 0, ctx->stream.get()>>>(d_ids, vol, (uint32_t)count, v);
    CU(cudaGetLastError());
    uint32_t unused;
    return read_verdict(ctx, v, &unused);
}

aicb_status copy_to_replica(Replicas r, size_t k, const void *from, size_t bytes, void **to) {
    aicb_ctx *c = r.ctx[k];
    CU(cudaSetDevice(c->device));
    TRY(inputs_room(c, bytes));
    CU(cudaMemcpyPeerAsync(c->d_inputs.get(), c->device, from, r.ctx[0]->device, bytes, c->stream.get()));
    *to = c->d_inputs.get();
    return AICB_OK;
}

aicb_status refresh_mirror(aicb_scene *s0) {
    SpaceHost &h = *s0->host;
    if (!h.ids_stale) return AICB_OK;
    if (h.volume) {
        aicb_ctx *ctx = s0->ctx;
        cudaStream_t stream = ctx->stream.get();
        CU(cudaSetDevice(ctx->device));
        DeviceBuffer ids;
        TRY(ids.ensure(h.volume * 2));
        k_decode_ids<<<stride_grid(ctx, h.volume), 256, 0, stream>>>(s0->d_cells.get(), s0->ds.wide_cells, h.volume,
                                                                      ids.get<uint16_t>());
        CU(cudaGetLastError());
        h.h_ids.resize(h.volume);
        CU(cudaMemcpyAsync(h.h_ids.data(), ids.get(), h.volume * 2, cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
    }
    h.ids_stale = false;
    return AICB_OK;
}

// The batch is checked and de-duplicated on replica 0's device (k_check_cubes, a stable radix sort by cube, the last
// entry of each run: k_cube_deltas), and only the verdict and the number of distinct cubes come back.  Every replica
// then scatters the same deltas (scatter_cubes_kernel), the others from a peer copy of replica 0's.
aicb_status scenes_update_cubes_device(Replicas r, const int32_t (*cubes)[3], const uint16_t *ids,
                                       const uint8_t (*light)[4], size_t n, cudaStream_t caller) {
    if (n && (!cubes || !ids)) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_scene *s0 = r.scene[0];
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n == 0) return AICB_OK;
    if (n > 0xffffffffull) return fail(AICB_ERR_INVALID, "more than 2^32 - 1 cubes");
    TRY(check_device_pointer(cubes, c0->device, false, 4, "cubes"));
    TRY(check_device_pointer(ids, c0->device, false, 2, "block_ids"));
    if (light) TRY(check_device_pointer(light, c0->device, false, 4, "light"));
    TRY(join_caller(r.ctx, 1, caller));
    const uint32_t nn = (uint32_t)n;
    CubeList l;
    TRY(stage_cube_list(s0, cubes, ids, nn, n * sizeof(CubeDelta), 0, &l));
    CubeDelta *ops = (CubeDelta *)l.extra;
    const bool lit = light && s0->d_light;
    k_cube_deltas<<<(nn + 255) / 256, 256, 0, c0->stream.get()>>>(l.keys, l.vals, nn, ids,
                                                                  lit ? (const uint32_t *)light : nullptr, s0->ds.blocks,
                                                                  (uint32_t)s0->host->block_count(), s0->ds.wide_cells,
                                                                  ops, l.verdict);
    CU(cudaGetLastError());
    uint32_t m = 0;
    TRY(read_verdict(c0, l.verdict, &m));
    for (size_t k = 0; k < r.n; k++) {
        aicb_scene *s = r.scene[k];
        aicb_ctx *ctx = r.ctx[k];
        CU(cudaSetDevice(ctx->device));
        void *from = ops;
        if (k > 0) TRY(copy_to_replica(r, k, ops, (size_t)m * sizeof(CubeDelta), &from));
        scatter_cubes_kernel<<<(m + 127) / 128, 128, 0, ctx->stream.get()>>>((const CubeDelta *)from, m, s->ds.wide_cells,
                                                                            s->d_cells.get(), s->d_light.get<uint32_t>());
        CU(cudaGetLastError());
        CU(cudaEventRecord(ctx->ev_delta.get(), ctx->stream.get()));   // renders on other streams wait for it
    }
    s0->host->ids_stale = true;
    TRY(settle_replicas(r));
    return release_caller(c0, caller);
}

// The box form: the ids are checked on the device (check_region_device), then every replica's k_region_cells and
// k_region_texels read the caller's arrays where they are (peer memory for the other replicas).
aicb_status scenes_update_region_device(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                        const uint8_t (*light)[4], cudaStream_t caller) {
    RegionBox box;
    TRY(check_region_device(r, region, ids, uniform_id, light, caller, &box));
    if (box.volume() == 0) return AICB_OK;
    for (size_t k = 0; k < r.n; k++) {
        CU(cudaSetDevice(r.ctx[k]->device));
        TRY(region_cells(r.scene[k], box, ids, uniform_id, light, true, nullptr, nullptr));
        CU(cudaEventRecord(r.ctx[k]->ev_delta.get(), r.ctx[k]->stream.get()));   // renders on other streams wait for it
    }
    r.scene[0]->host->ids_stale = true;
    TRY(settle_replicas(r));
    return release_caller(r.ctx[0], caller);
}

aicb_status scenes_upload_light_device(Replicas r, const uint8_t (*light)[4], size_t n_texels, cudaStream_t caller) {
    if (!light) return fail(AICB_ERR_INVALID, "NULL argument");
    const size_t volume = r.scene[0]->host->volume;
    if (n_texels != volume) return fail(AICB_ERR_INVALID, "light volume size mismatch");
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (volume == 0) return AICB_OK;
    TRY(check_device_pointer(light, c0->device, false, 4, "light"));
    TRY(join_caller(r.ctx, r.n, caller));
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *s = r.scene[i];
        cudaStream_t stream = r.ctx[i]->stream.get();
        CU(cudaSetDevice(r.ctx[i]->device));
        if (!s->d_light) {
            TRY(s->d_light.ensure(volume * 4));
            s->device_bytes += volume * 4;
            s->ds.light = s->d_light.get<uint32_t>();
        }
        CU(cudaMemcpyPeerAsync(s->d_light.get(), r.ctx[i]->device, light, c0->device, volume * 4, stream));
        CU(cudaEventRecord(r.ctx[i]->ev_delta.get(), stream));
    }
    TRY(settle_replicas(r));
    return release_caller(c0, caller);
}

aicb_status scene_download_ids_device(Replicas r, uint16_t *out, size_t n, cudaStream_t caller) {
    aicb_scene *s = r.scene[0];
    aicb_ctx *ctx = r.ctx[0];
    if (!out) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n != s->host->volume) return fail(AICB_ERR_INVALID, "block id volume size mismatch");
    CU(cudaSetDevice(ctx->device));
    if (n == 0) return AICB_OK;
    TRY(check_device_pointer(out, ctx->device, false, 2, "out"));
    TRY(join_caller(r.ctx, 1, caller));
    k_decode_ids<<<stride_grid(ctx, n), 256, 0, ctx->stream.get()>>>(s->d_cells.get(), s->ds.wide_cells, n, out);
    CU(cudaGetLastError());
    if (r.n > 1) CU(cudaStreamSynchronize(ctx->stream.get()));   // a group call returns with its output final
    return release_caller(ctx, caller);
}

// The first failure of the host twin that the descriptors' scalars decide (flatten_blocks' checks without the index
// scan): at definition `at` before its scan, or after it (`after_scan`); at == n for the brick pool's room, which is
// checked after every definition.  at == SIZE_MAX: none.
struct HostVerdict {
    size_t at = SIZE_MAX;
    bool after_scan = false;
    aicb_status st = AICB_OK;
    std::string msg;
};

static HostVerdict host_checks(const SpaceHost &h, const uint16_t *indices, const aicb_block_desc *descs, size_t n) {
    HostVerdict v;
    auto failed = [&](size_t at, bool after, aicb_status st) {
        v.at = at;
        v.after_scan = after;
        v.st = st;
        v.msg = aicb_last_error();
        return v;
    };
    if (!indices && h.block_count() + n > 65536) return failed(0, false, fail(AICB_ERR_INVALID, "more than 65536 blocks"));
    size_t words = 0;
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        if (indices && indices[i] >= h.block_count())
            return failed(i, false, fail(AICB_ERR_INVALID, "block index out of range (new indices need a new scene)"));
        aicb_status st = check_block_scalars(b);
        if (st != AICB_OK) return failed(i, false, st);
        if ((st = check_block_palette(b)) != AICB_OK) return failed(i, true, st);
        if (b.is_air || is_single_voxel(b)) continue;
        if (words + b.n_indices > 0xffffffffull) return failed(i, true, fail(AICB_ERR_INVALID, BRICKS_PAST_2_32));
        words += b.n_indices;
    }
    if (brick_room(h.n_bricks, h.dead_bricks, words) == BrickRoom::too_big)
        return failed(n, false, fail(AICB_ERR_INVALID, BRICKS_PAST_2_32));
    return v;
}

// Each definition's voxel pointers: device memory of device 0, aligned to their elements.
static aicb_status check_def_pointers(const aicb_ctx *c0, const aicb_block_desc *descs, size_t n) {
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        const std::string name = "block " + std::to_string(i) + "'s ";
        if (b.indices && b.n_indices) TRY(check_device_pointer(b.indices, c0->device, false, 2, (name + "indices").c_str()));
        if (b.palette && b.n_palette) TRY(check_device_pointer(b.palette, c0->device, false, 4, (name + "palette").c_str()));
    }
    return AICB_OK;
}

// n definitions whose voxels are in device 0's memory, checked against `h` (for `indices`, or appended) once the first
// n_ctx contexts' streams wait for the caller's.  The host checks what the scalars decide; one pass on device 0 scans
// the voxel indices of the definitions before the first host-side failure and reads the kind of each single voxel,
// and with `ids` checks those `volume` block ids against the n definitions (k_check_ids; the host twin checks them
// after every definition, scene creation's "block id out of range").  Those bytes are all that comes back before the
// call decides, and the status and message are the host twin's first failure.  With AICB_BLOCKS_DERIVE_LIGHT,
// derive's kernels then run on device 0 on the caller's voxels and their error words come back too.
static aicb_status check_device_defs(aicb_ctx *const *ctx, size_t n_ctx, const SpaceHost &h, const uint16_t *indices,
                                     const aicb_block_desc *descs, size_t n, uint32_t flags, cudaStream_t caller,
                                     const uint16_t *ids, size_t volume, DeviceDefs *dev) {
    aicb_ctx *c0 = ctx[0];
    const HostVerdict hv = host_checks(h, indices, descs, n);
    const size_t n_scan = std::min(n, hv.at == SIZE_MAX ? n : hv.at + (hv.after_scan ? 1 : 0));
    TRY(join_caller(ctx, n_ctx, caller));
    dev->kinds.assign(n, KIND_INVISIBLE);
    unsigned long long bad = ~0ull;
    bool bad_id = false;
    if (n_scan) {   // the verdicts (16 bytes each: the definitions', the ids') and the kinds, read back together
        std::vector<DeviceBlockJob> jobs(n_scan, DeviceBlockJob{});
        uint64_t most = 0;
        for (size_t i = 0; i < n_scan; i++) {
            jobs[i].indices = descs[i].indices;
            jobs[i].palette = descs[i].palette;
            jobs[i].n_indices = descs[i].indices ? descs[i].n_indices : 0;
            jobs[i].n_palette = (uint32_t)std::min<size_t>(descs[i].n_palette, 0xffffffffu);
            jobs[i].single = single_source(descs[i]);
            most = std::max(most, jobs[i].n_indices);
        }
        const size_t verdicts = 2 * sizeof(InputVerdict);
        const size_t head = align256(verdicts + n_scan), job_bytes = n_scan * sizeof(DeviceBlockJob);
        cudaStream_t stream = c0->stream.get();
        TRY(inputs_room(c0, head + job_bytes));
        char *p = c0->d_inputs.get<char>();
        InputVerdict *v = (InputVerdict *)p;
        DeviceBlockJob *d_jobs = (DeviceBlockJob *)(p + head);
        CU(cudaMemcpyAsync(d_jobs, jobs.data(), job_bytes, cudaMemcpyHostToDevice, stream));
        TRY(reset_verdict(v, stream));
        TRY(reset_verdict(v + 1, stream));
        TRY(issue_block_verdict(stream, d_jobs, (uint32_t)n_scan, most, v, (uint8_t *)p + verdicts));
        if (ids && volume) {
            k_check_ids<<<stride_grid(c0, volume), 256, 0, stream>>>(ids, volume, (uint32_t)n, v + 1);
            CU(cudaGetLastError());
        }
        std::vector<char> back(verdicts + n_scan);
        CU(cudaMemcpyAsync(back.data(), p, back.size(), cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        bad = ((const InputVerdict *)back.data())[0].first_bad;
        bad_id = ((const InputVerdict *)back.data())[1].first_bad != ~0ull;
        std::memcpy(dev->kinds.data(), back.data() + verdicts, n_scan);
    }
    // the host twin's first failure: block order, and within a block the scalars, the scan, the palette's size; then
    // the ids
    if (bad != ~0ull && (bad < hv.at || (bad == hv.at && hv.after_scan))) return fail(AICB_ERR_INVALID, BAD_VOXEL_INDEX);
    if (hv.at != SIZE_MAX) return fail(hv.st, hv.msg);
    if (bad_id) return fail(AICB_ERR_INVALID, "block id out of range");
    if (flags & AICB_BLOCKS_DERIVE_LIGHT) {
        dev->derive = true;
        TRY(derive_on_device(c0, descs, n, &dev->derived, &dev->d_derived));
    }
    return AICB_OK;
}

// aicb_scene_update_blocks_device / append_blocks_device over the replicas: the definitions checked on device 0
// (check_device_defs), then the host twin's body (update_blocks, append_blocks) with the voxel data placed by
// blocks.cu's kernels on every replica, which read device 0's buffers (as a peer on other devices).
aicb_status scenes_blocks_device(Replicas r, bool append, const uint16_t *indices, const aicb_block_desc *descs, size_t n,
                                 uint32_t flags, cudaStream_t caller) {
    if (n && (!descs || (!append && !indices))) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n == 0) return AICB_OK;
    if (append) indices = nullptr;
    if (flags & ~AICB_BLOCKS_DERIVE_LIGHT) return fail(AICB_ERR_INVALID, "unknown flags");
    TRY(check_def_pointers(c0, descs, n));
    DeviceDefs dev;
    TRY(check_device_defs(r.ctx, r.n, *r.scene[0]->host, indices, descs, n, flags, caller, nullptr, 0, &dev));
    TRY(indices ? update_blocks(r, indices, descs, n, &dev) : append_blocks(r, descs, n, &dev));
    TRY(settle_replicas(r));
    return release_caller(c0, caller);
}

// The jobs of n checked definitions whose voxels are in device memory, flattened against `empty` (a new table).
static void flatten_new_table(const SpaceHost &empty, const aicb_block_desc *descs, size_t n, DeviceDefs &dev,
                              FlatBlocks *f) {
    flatten_device(empty, descs, n, dev.kinds, dev.derive, f);
    device_jobs(empty, descs, *f, nullptr, dev);
}

// aicb_scene_create_device over n contexts: the pointers, then scene creation's checks in the host form's order, the
// definitions' and the ids' verdicts read back once (check_device_defs), and the body both forms share.  The light is
// a device-to-device copy per replica.
aicb_status scenes_create_device(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, uint32_t flags,
                                 cudaStream_t caller, aicb_scene **out) {
    aicb_ctx *c0 = ctx[0];
    CU(cudaSetDevice(c0->device));
    if (flags & ~AICB_BLOCKS_DERIVE_LIGHT) return fail(AICB_ERR_INVALID, "unknown flags");
    const bool cubes = d->bounds.size[0] && d->bounds.size[1] && d->bounds.size[2];
    if (cubes && d->block_ids) TRY(check_device_pointer(d->block_ids, c0->device, false, 2, "block_ids"));
    if (cubes && d->light) TRY(check_device_pointer(d->light, c0->device, false, 4, "light"));
    if (d->blocks) TRY(check_def_pointers(c0, d->blocks, d->n_blocks));
    uint64_t volume;
    TRY(check_scene_desc(d, &volume));
    const SpaceHost empty;
    DeviceDefs dev;
    TRY(check_device_defs(ctx, n, empty, nullptr, d->blocks, d->n_blocks, flags, caller, d->block_ids, volume, &dev));
    FlatBlocks f;
    flatten_new_table(empty, d->blocks, d->n_blocks, dev, &f);
    TRY(create_scenes(ctx, n, d, volume, f, nullptr, &dev, out));
    return release_caller(c0, caller);
}

// aicb_scene_fill_uniform_device over the replicas: the block checked on device 0 (check_device_defs), then
// fill_uniform with its voxel data placed by blocks.cu's kernels.
aicb_status scenes_fill_uniform_device(Replicas r, const aicb_block_desc *block, uint32_t flags, cudaStream_t caller) {
    if (!block) return fail(AICB_ERR_INVALID, "NULL argument");
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (flags & ~AICB_BLOCKS_DERIVE_LIGHT) return fail(AICB_ERR_INVALID, "unknown flags");
    TRY(check_def_pointers(c0, block, 1));
    const SpaceHost empty;
    DeviceDefs dev;
    TRY(check_device_defs(r.ctx, r.n, empty, nullptr, block, 1, flags, caller, nullptr, 0, &dev));
    FlatBlocks f;
    flatten_new_table(empty, block, 1, dev, &f);
    TRY(fill_uniform(r, empty, f, &dev));   // (which returns once every replica's writes are done)
    cudaSetDevice(c0->device);
    return release_caller(c0, caller);
}


// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
aicb_status check_views(const aicb_camera *cameras, bool host_cameras, size_t n_views, uint32_t *width,
                        uint32_t *height, const aicb_options *opt, size_t out_len) {
    TRY(validate_options(opt));
    if (n_views && !cameras) return fail(AICB_ERR_INVALID, "cameras is NULL");
    if (host_cameras) {
        *width = n_views ? cameras[0].fb_width : 0;
        *height = n_views ? cameras[0].fb_height : 0;
        for (size_t v = 1; v < n_views; v++)
            if (cameras[v].fb_width != *width || cameras[v].fb_height != *height)
                return fail(AICB_ERR_INVALID, "the views' cameras must share the framebuffer size");
    }
    const uint64_t per_view = (uint64_t)*width * *height;
    if (per_view && n_views > SIZE_MAX / per_view) return fail(AICB_ERR_INVALID, "batch too large");
    if (out_len != n_views * per_view)
        return fail(AICB_ERR_INVALID, "output length must be n_views * fb_width * fb_height");
    if (per_view && n_views) {   // n_views * tiles * 32 * samples < 2^32
        const uint64_t tasks = ((uint64_t)*width + TILE_W - 1) / TILE_W * (((uint64_t)*height + TILE_H - 1) / TILE_H) *
                               32 * (opt->antialiasing_always ? 4 : 1);   // (< 2^63: width, height < 2^32)
        if (tasks > 0xffffffffull || n_views > 0xffffffffull / tasks)
            return fail(AICB_ERR_INVALID, "batch too large: its tasks reach 2^32");
    }
    return AICB_OK;
}

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
    // the context is the caller's once every step has succeeded; until then a failure frees what was created
    std::unique_ptr<aicb_ctx> c(new aicb_ctx());
    c->device = device_id;
    c->num_sms = prop.multiProcessorCount;
    cudaStream_t stream = nullptr;
    CU(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    c->stream.reset(stream);
    TRY(create_event(c->ev0, cudaEventDefault));
    TRY(create_event(c->ev1, cudaEventDefault));
    for (Event &e : c->ev_light) TRY(create_event(e, cudaEventDefault));
    c->profile_kernels = getenv("AICB_PROFILE_KERNELS") != nullptr;
    for (int i = 0; i < 5; i++) TRY(create_event(c->ev_k[i], cudaEventDefault));
    TRY(create_event(c->ev_delta, cudaEventDisableTiming));
    TRY(create_event(c->ev_join, cudaEventDisableTiming));
    TRY(c->d_counters.ensure(8 * sizeof(unsigned long long) + 2 * (4 + N_BINS) * sizeof(unsigned int)));
    c->d_tile_counter = (unsigned int *)(c->d_counters.get<unsigned long long>() + 8);
    // PackedLight decode table (light/data.rs:232-243 scalar_out_arithmetic; table :301-354)
    float lut[768];
    lut[0] = 0.0f;
    for (int i = 1; i < 256; i++) lut[i] = (float)std::exp2((double)(((float)i - 144.0f) / 10.0f));
    build_srgb_thresholds(lut + 256);
    build_light_thresholds(lut + 512);
    TRY(c->d_lut.upload(lut, sizeof lut));
    *out = c.release();
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

#ifdef AICB_SHADE_PHASES
// tools/shade_phases.py only (not in the header): copy the phase cycle sums of shade_hit<LC_INTERP> on the current
// device to out[10], then zero them.
int aicb_debug_shade_phases(unsigned long long *out) {
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemcpyFromSymbol(out, aicb::g_shade_phase, sizeof(aicb::g_shade_phase)) != cudaSuccess) return -1;
    const unsigned long long zero[10] = {};
    return cudaMemcpyToSymbol(aicb::g_shade_phase, zero, sizeof zero) == cudaSuccess ? 0 : -1;
}
#endif

int aicb_ctx_device(const aicb_ctx *c) { return c ? c->device : -1; }

void aicb_ctx_destroy(aicb_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    delete c;
}

aicb_status aicb_scene_create(aicb_ctx *ctx, const aicb_scene_desc *d, aicb_scene **out) {
    if (!ctx || !d || !out) return fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    std::lock_guard<std::mutex> lock(ctx->mu);
    return scenes_create(&ctx, 1, d, out);
}

aicb_status aicb_scene_create_device(aicb_ctx *ctx, const aicb_scene_desc *d, uint32_t flags, void *stream,
                                     aicb_scene **out) {
    if (!ctx || !d || !out) return fail(AICB_ERR_INVALID, "NULL argument");
    *out = nullptr;
    std::lock_guard<std::mutex> lock(ctx->mu);
    return scenes_create_device(&ctx, 1, d, flags, (cudaStream_t)stream, out);
}

void aicb_scene_destroy(aicb_scene *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    wait_context(s->ctx);
    if (s->ctx->last_scene == s) {
        s->ctx->last_scene = nullptr;
        s->ctx->frame_in_flight = false;
    }
    delete s;
}

uint64_t aicb_scene_device_bytes(const aicb_scene *s) { return s ? s->device_bytes + s->host->table_bytes() : 0; }

aicb_status aicb_scene_set_physics(aicb_scene *s, const aicb_sky *sky, uint8_t light_max_distance) {
    return on_scene(s, [&](Replicas r) { return scenes_set_physics(r, sky, light_max_distance); });
}

aicb_status aicb_scene_update_cubes(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *ids,
                                    const uint8_t (*light)[4], size_t n) {
    return on_scene(s, [&](Replicas r) { return scenes_update_cubes(r, cubes, ids, light, n); });
}

aicb_status aicb_scene_update_region(aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                     const uint8_t (*light)[4]) {
    return on_scene(s, [&](Replicas r) { return scenes_update_region(r, region, ids, uniform_id, light); });
}

// == SpaceChange::BlockEvaluation / BlockIndex (space.rs:1062-1100; UpdatingSpaceRaytracer::update handles them in
// updating.rs:128-150 by re-running TracingBlock::from_block for the changed indices): replace the definition of
// existing block indices.  New voxel data is appended to the brick pool and the palette, and the replaced ranges are
// reclaimed by compaction (BlockTable); cubes that hold a block whose classification changed are re-encoded.
// Does not touch light: aicb_light_relight_blocks with the same indices applies the light side of the change.
aicb_status aicb_scene_update_blocks(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs, size_t n) {
    return on_scene(s, [&](Replicas r) { return scenes_update_blocks(r, indices, descs, n); });
}

// == SpaceChange::BlockIndex for indices past the table (palette.rs:207-210; UpdatingSpaceRaytracer::update appends
// TracingBlock::from_block of each, updating.rs:145-151): the blocks become the table's next indices.
aicb_status aicb_scene_append_blocks(aicb_scene *s, const aicb_block_desc *descs, size_t n) {
    return on_scene(s, [&](Replicas r) { return scenes_append_blocks(r, descs, n); });
}

aicb_status aicb_scene_update_blocks_device(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs,
                                            size_t n, uint32_t flags, void *stream) {
    return on_scene(s, [&](Replicas r) { return scenes_blocks_device(r, false, indices, descs, n, flags, (cudaStream_t)stream); });
}

aicb_status aicb_scene_append_blocks_device(aicb_scene *s, const aicb_block_desc *descs, size_t n, uint32_t flags,
                                            void *stream) {
    return on_scene(s, [&](Replicas r) { return scenes_blocks_device(r, true, nullptr, descs, n, flags, (cudaStream_t)stream); });
}

// == SpaceChange::EveryBlock (Mutation::fill_uniform over the whole bounds, space.rs:1461-1474).
aicb_status aicb_scene_fill_uniform(aicb_scene *s, const aicb_block_desc *block) {
    return on_scene(s, [&](Replicas r) { return scenes_fill_uniform(r, block); });
}

aicb_status aicb_scene_fill_uniform_device(aicb_scene *s, const aicb_block_desc *block, uint32_t flags, void *stream) {
    return on_scene(s, [&](Replicas r) { return scenes_fill_uniform_device(r, block, flags, (cudaStream_t)stream); });
}

aicb_status aicb_scene_upload_light(aicb_scene *s, const uint8_t (*light)[4], size_t n_texels) {
    return on_scene(s, [&](Replicas r) { return scenes_upload_light(r, light, n_texels); });
}

aicb_status aicb_scene_update_cubes_device(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *ids,
                                           const uint8_t (*light)[4], size_t n, void *stream) {
    return on_scene(s, [&](Replicas r) { return scenes_update_cubes_device(r, cubes, ids, light, n, (cudaStream_t)stream); });
}

aicb_status aicb_scene_update_region_device(aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                            const uint8_t (*light)[4], void *stream) {
    return on_scene(s, [&](Replicas r) {
        return scenes_update_region_device(r, region, ids, uniform_id, light, (cudaStream_t)stream);
    });
}

aicb_status aicb_scene_upload_light_device(aicb_scene *s, const uint8_t (*light)[4], size_t n_texels, void *stream) {
    return on_scene(s, [&](Replicas r) { return scenes_upload_light_device(r, light, n_texels, (cudaStream_t)stream); });
}

aicb_status aicb_scene_download_ids_device(aicb_scene *s, uint16_t *out, size_t n, void *stream) {
    return on_scene(s, [&](Replicas r) { return scene_download_ids_device(r, out, n, (cudaStream_t)stream); });
}

size_t aicb_shard_pixel_count(const aicb_camera *cam, const aicb_shard *shard) {
    if (!cam) return 0;
    return (size_t)cam->fb_width * shard_rows(cam->fb_height, shard);
}

aicb_status aicb_check_render_args(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
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
    aicb_status st = aicb_check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::srgb8, out, out_len);
    return on_scene(s, [&](Replicas r) { return frame_host(r, cam, opt, shard, o, STAGE_PINNED, info); });
}

aicb_status aicb_render_rgba16f(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                                uint16_t (*out)[4], size_t out_len, aicb_render_info *info) {
    aicb_status st = aicb_check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::rgba16f, out, out_len);
    return on_scene(s, [&](Replicas r) { return frame_host(r, cam, opt, shard, o, STAGE_GIVEN, info); });
}

aicb_status aicb_render_colorbuf(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                 const aicb_shard *shard, float (*out_cb)[4], double *depth, aicb_hit *hit,
                                 uint32_t *steps, size_t out_len, aicb_render_info *info) {
    aicb_status st = aicb_check_render_args(s, cam, opt, shard, out_len);
    if (st != AICB_OK) return st;
    const aicb_device_outputs o = colorbuf_outputs(out_cb, depth, hit, steps, out_len);
    return on_scene(s, [&](Replicas r) { return frame_host(r, cam, opt, shard, o, STAGE_COLORBUF, info); });
}

aicb_status aicb_render_device(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, const aicb_shard *shard,
                               const aicb_device_outputs *outs, void *stream) {
    if (!s || !cam || !outs) return fail(AICB_ERR_INVALID, "NULL argument");
    const bool full = outs->full_frame != 0;
    TRY(aicb_check_render_args(s, cam, opt, shard, full ? aicb_shard_pixel_count(cam, shard) : outs->len));
    if (full && outs->len != (size_t)cam->fb_width * cam->fb_height)
        return fail(AICB_ERR_INVALID, "Viewport size does not match frame buffer length");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    Outputs o;
    TRY(device_target(outs, s->ctx->device, DEV_FRAME, false, full, &o));
    o.full_frame = full;
    return launch_trace(s, cam, opt, shard, o, stream ? (cudaStream_t)stream : s->ctx->stream.get());
}

aicb_status aicb_render_srgb8_device(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                     const aicb_shard *shard, void *d_out, size_t out_len, void *stream) {
    aicb_device_outputs o{};
    o.srgb8 = (uint8_t(*)[4])d_out;
    o.len = out_len;
    return aicb_render_device(s, cam, opt, shard, &o, stream);
}

aicb_status aicb_render_srgb8_device_frame(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt,
                                           const aicb_shard *shard, void *d_frame, size_t frame_len, void *stream) {
    aicb_device_outputs o{};
    o.srgb8 = (uint8_t(*)[4])d_frame;
    o.len = frame_len;
    o.full_frame = 1;
    return aicb_render_device(s, cam, opt, shard, &o, stream);
}

aicb_status aicb_trace_rays_device(aicb_scene *s, const double (*d_origin_dir)[6], size_t n, const aicb_options *opt,
                                   const aicb_device_outputs *outs, void *stream) {
    if (!s || !outs || (n && !d_origin_dir)) return fail(AICB_ERR_INVALID, "NULL argument");
    TRY(validate_options(opt));
    if (outs->full_frame) return fail(AICB_ERR_INVALID, "full_frame is for camera frames");
    if (outs->len != n) return fail(AICB_ERR_INVALID, "outs->len must equal the number of rays");
    if (n > 0xffffffffull) return fail(AICB_ERR_INVALID, "too many rays");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    Outputs o;
    TRY(device_target(outs, s->ctx->device, DEV_RAYS, false, false, &o));
    if (n) TRY(check_device_pointer(d_origin_dir, s->ctx->device, false, 8, "the ray batch"));
    o.rays = (const double *)d_origin_dir;   // gen_kernel reads the caller's batch in place
    o.n_rays = n;
    return launch_trace(s, nullptr, opt, nullptr, o, stream ? (cudaStream_t)stream : s->ctx->stream.get());
}

// ---- full-frame buffers shared between ranks (CUDA IPC) ------------------------------------------
// Behind the pixels of a shared frame sits a small control block in the same allocation (so it travels with the IPC
// handle): two monotonic counters that replace the collective of the delivery step.
//   arrived   += 1 by every rank once its strips of a frame are stored (aicb_frame_signal, after the rank's last kernel
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
    *st = stream ? (cudaStream_t)stream : ctx->stream.get();
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
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream.get();
    CU(cudaMemcpyAsync(out, d_frame, n_pixels * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return AICB_OK;
}

// == print_space's per-pixel CharacterBuf (raytracer/text.rs:52-123, 139-180): which block each pixel shows.
aicb_status aicb_render_text(aicb_scene *s, const aicb_camera *cam, const aicb_options *opt, int32_t *out, size_t out_len,
                             aicb_render_info *info) {
    aicb_status st = aicb_check_render_args(s, cam, opt, nullptr, out_len);
    if (st != AICB_OK) return st;
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::text, out, out_len);
    return on_scene(s, [&](Replicas r) { return frame_host(r, cam, opt, nullptr, o, STAGE_GIVEN, info); });
}

// A batch of views of one scene (internal.h: check_views, views_host): the single-camera calls' outputs, view-major.
aicb_status aicb_render_views_srgb8(aicb_scene *s, const aicb_camera *cameras, size_t n_views, const aicb_options *opt,
                                    uint8_t (*out)[4], size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!s) return fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::srgb8, out, out_len);
    return on_scene(s, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_PINNED, info); });
}

aicb_status aicb_render_views_rgba16f(aicb_scene *s, const aicb_camera *cameras, size_t n_views, const aicb_options *opt,
                                      uint16_t (*out)[4], size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!s) return fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::rgba16f, out, out_len);
    return on_scene(s, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_GIVEN, info); });
}

aicb_status aicb_render_views_colorbuf(aicb_scene *s, const aicb_camera *cameras, size_t n_views,
                                       const aicb_options *opt, float (*out_cb)[4], double *depth, aicb_hit *hit,
                                       uint32_t *steps, size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!s) return fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    const aicb_device_outputs o = colorbuf_outputs(out_cb, depth, hit, steps, out_len);
    return on_scene(s, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_COLORBUF, info); });
}

aicb_status aicb_render_views_text(aicb_scene *s, const aicb_camera *cameras, size_t n_views, const aicb_options *opt,
                                   int32_t *out, size_t out_len, aicb_render_info *info) {
    uint32_t w, h;
    if (!s) return fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_views(cameras, true, n_views, &w, &h, opt, out_len));
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const aicb_device_outputs o = one_output(&aicb_device_outputs::text, out, out_len);
    return on_scene(s, [&](Replicas r) { return views_host(r, cameras, n_views, opt, o, STAGE_GIVEN, info); });
}

// The batch as one frame on `stream`, reading the caller's camera table where it is; aicb_render_finish finishes it.
aicb_status aicb_render_views_device(aicb_scene *s, const aicb_camera *d_cameras, size_t n_views, uint32_t fb_width,
                                     uint32_t fb_height, const aicb_options *opt, const aicb_device_outputs *outs,
                                     void *stream) {
    if (!s || !outs) return fail(AICB_ERR_INVALID, "NULL argument");
    if (outs->full_frame) return fail(AICB_ERR_INVALID, "full_frame is for aicb_render_device");
    TRY(check_views(d_cameras, false, n_views, &fb_width, &fb_height, opt, outs->len));
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    Outputs o;
    TRY(device_target(outs, s->ctx->device, DEV_FRAME, false, false, &o));
    if (n_views) TRY(check_device_pointer(d_cameras, s->ctx->device, false, 8, "the camera table"));
    cudaStream_t st = stream ? (cudaStream_t)stream : s->ctx->stream.get();
    if (outs->len == 0) return issue_empty_frame(s, opt, st);
    views_part(&o, d_cameras, n_views, 0, 1);
    const aicb_camera size = views_frame_camera(fb_width, fb_height);
    return launch_trace(s, &size, opt, nullptr, o, st);
}

// Arguments shared by the layered entry points: at least one layer (or the paint colour), complete layers, one context
// and one framebuffer size.  `lead` is the layer whose options choose the sample points.
aicb_status aicb_check_layers(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba, size_t out_len,
                              const aicb_layer **lead_out) {
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
    aicb_status st = aicb_check_render_args(lead->scene, lead->camera, lead->options, nullptr, out_len);
    if (st != AICB_OK) return st;
    if (have_ui && have_world) {
        st = validate_options(ui->options);
        if (st != AICB_OK) return st;
    }
    *lead_out = lead;
    return AICB_OK;
}

// RaytraceInfo of several passes (renderer.rs:555): counters add up.  Times add up over the passes of one part, which
// run one after another; over the parts of a frame, which run side by side, the frame took as long as its slowest part.
void aicb_merge_info(aicb_render_info *sum, const aicb_render_info *one, bool same_part) {
    auto time = [same_part](float t, float u) { return same_part ? t + u : std::max(t, u); };
    sum->cubes_traced += one->cubes_traced;
    sum->rays += one->rays;
    sum->algorithmic_bytes += one->algorithmic_bytes;
    for (int k = 0; k < 6; k++) sum->counters[k] += one->counters[k];
    sum->kernel_ms = time(sum->kernel_ms, one->kernel_ms);
    for (int k = 0; k < 4; k++) sum->stage_ms[k] = time(sum->stage_ms[k], one->stage_ms[k]);
    sum->flaws |= one->flaws;
    sum->ray_order |= one->ray_order;
}

// A pass is issued on every part before any part's pass is finished, so that the devices of a group overlap; a context
// tracks one frame (finish), so its next pass waits until this one is finished.  finish decides whether a part's hit
// stream overflowed and raises that context's capacity (x4 per retry, AICB_ERR_OOM at the cap); such a part is
// re-issued alone.  With want_info, each finished pass is added to its part's info; without, finish skips its event
// queries, as a caller that passes no aicb_render_info expects.  Every round delivers `copies` (deliver): device 0
// (parts[0]'s context) copies behind that round's parts, before the host waits for them, so a frame and its copy
// cost one host synchronisation.  The caller holds the parts' contexts' locks.
aicb_status aicb_trace_pass(FramePart *parts, size_t n_parts, const aicb_camera *cam, const aicb_options *opt,
                            bool want_info, const std::vector<Delivery> &copies) {
    std::vector<size_t> todo(n_parts), again;
    for (size_t i = 0; i < n_parts; i++) todo[i] = i;
    while (!todo.empty()) {
        std::vector<aicb_ctx *> round = {parts[0].scene->ctx};   // device 0, then the other contexts of the round
        for (size_t i : todo) {
            const FramePart &p = parts[i];
            aicb_ctx *ctx = p.scene->ctx;
            CU(cudaSetDevice(ctx->device));
            aicb_status r = launch_trace(p.scene, cam, opt, p.shard, p.out, ctx->stream.get());
            if (r != AICB_OK) return r;
            if (i) round.push_back(ctx);
        }
        if (!copies.empty()) TRY(deliver(round.data(), round.size(), copies));
        again.clear();
        for (size_t i : todo) {
            aicb_scene *sc = parts[i].scene;
            CU(cudaSetDevice(sc->ctx->device));
            CU(cudaStreamSynchronize(sc->ctx->stream.get()));
            aicb_render_info one{};
            aicb_status r = finish(sc, want_info ? &one : nullptr);
            if (r == AICB_ERR_RETRY) { again.push_back(i); continue; }
            if (r != AICB_OK) return r;
            aicb_merge_info(&parts[i].info, &one, true);
        }
        todo.swap(again);
    }
    return AICB_OK;
}

// RtScene::trace_ray_through_layers for every pixel task of every part (renderer.rs:454-478): the UI layer's Space is
// traced first (its own camera, no sky), the backdrop colour is added, the world layer continues in the same
// accumulator (its rays start opaque where the UI covered the pixel), and a pixel that is not opaque in the end — there
// is no world — is painted NO_WORLD_TO_SHOW.  The last pass writes each part's target; with texture targets the UI pass
// hands its DepthBuf on next to its ColorBuf, with terminal targets its CharacterBuf.  Each pass runs on every part
// through aicb_trace_pass (a re-issued world pass starts from the same accumulator), and the last pass delivers
// `copies`.  With `async` (one part), the passes are issued back to back on that stream instead, the world pass
// continuing the UI pass's frame, and aicb_render_finish on the last pass's scene finishes them (total is not filled).
// The caller holds the parts' contexts' locks.
aicb_status aicb_trace_layers(const aicb_layer *world, const aicb_layer *ui, const float *backdrop_rgba,
                              const float *no_world_rgba, LayerPart *parts, size_t n_parts,
                              const std::vector<Delivery> &copies, aicb_render_info *total, cudaStream_t async) {
    const bool have_world = world && world->scene, have_ui = ui && ui->scene;
    const aicb_layer *lead = have_world ? world : ui;
    aicb_status st = AICB_OK;
    const int aa = lead->options->antialiasing_always ? 1 : 0;
    // per-task buffers between the passes: one entry per ray of the part's task layout (launch_trace)
    auto n_tasks = [&](const LayerPart &p) -> size_t {
        return (listed(p.out.target) ? (size_t)p.out.target.n_list
                                        : (((size_t)lead->camera->fb_width + TILE_W - 1) / TILE_W) *
                                              ((shard_rows(lead->camera->fb_height, &p.shard) + TILE_H - 1) / TILE_H) * 32) *
               (aa ? 4 : 1);
    };
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
    auto add_backdrop = [&](Outputs &o) {
        if (!have_backdrop) return;
        std::memcpy(o.target.backdrop, backdrop, 16);
        o.target.has_backdrop = 1;
    };
    auto add_no_world = [&](Outputs &o) {
        if (!no_world_rgba) return;
        std::memcpy(o.target.no_world, no_world, 16);
        o.target.has_no_world = 1;
    };
    // one pass of the frame on every part: `layer` picks the part's scene, `outputs(part, ctx)` its Outputs, and the
    // pass delivers `pass_copies`; each part's info sums its passes
    std::vector<FramePart> pass_parts(n_parts);
    bool first_pass = true;
    auto pass = [&](aicb_scene *LayerPart::*layer, const aicb_camera *cam, const aicb_options *opt,
                    const std::vector<Delivery> &pass_copies, auto outputs) -> aicb_status {
        for (size_t i = 0; i < n_parts; i++) {
            pass_parts[i].scene = parts[i].*layer;
            pass_parts[i].shard = &parts[i].shard;
            pass_parts[i].out = outputs(parts[i], pass_parts[i].scene->ctx);
        }
        if (!async) return aicb_trace_pass(pass_parts.data(), n_parts, cam, opt, true, pass_copies);
        const FramePart &p = pass_parts[0];
        const bool continues = !first_pass;
        first_pass = false;
        return launch_trace(p.scene, cam, opt, p.shard, p.out, async, continues);
    };
    if (have_ui && have_world) {
        for (size_t i = 0; i < n_parts; i++) {
            aicb_ctx *ctx = parts[i].world->ctx;
            CU(cudaSetDevice(ctx->device));
            TRY(ctx->d_task_aux.ensure(n_tasks(parts[i]) * sizeof(float4) + 16));
            if (parts[i].out.kind == TGT_TEX) {   // the UI pass's DepthBuf, only when there is a UI layer
                TRY(ctx->d_task_depth.ensure(n_tasks(parts[i]) * sizeof(double) + 16));
            }
            if (parts[i].out.kind == TGT_TERM) {   // the UI pass's CharacterBuf, only when there is a UI layer
                TRY(ctx->d_task_text.ensure(n_tasks(parts[i]) * sizeof(int2) + 16));
            }
        }
        aicb_options ui_opt = *ui->options;
        ui_opt.include_sky = 0;   // ui.trace_ray(.., false)
        st = pass(&LayerPart::ui, ui->camera, &ui_opt, {}, [&](const LayerPart &p, aicb_ctx *ctx) {
            // the pass that writes no pixel keeps the task layout and the target kind only
            Outputs o;
            o.kind = p.out.kind;
            o.target.pixel_list = p.out.target.pixel_list;
            o.target.n_list = p.out.target.n_list;
            o.target.picks = p.out.target.picks;
            o.target.pick_central = p.out.target.pick_central;
            o.target.pick_base = p.out.target.pick_base;
            o.target.tex_layer = TEX_UI;
            if (o.kind == TGT_TEX) o.target.out_task_depth = ctx->d_task_depth.get<double>();
            if (o.kind == TGT_TERM) {
                o.target.out_task_text = ctx->d_task_text.get<int2>();
                o.target.text_start = AICB_TEXT_EMPTY;
            }
            o.target.out_accum = ctx->d_task_aux.get<float4>();
            add_backdrop(o);
            o.force_antialias = aa;
            return o;
        });
        if (st != AICB_OK) return st;
        aicb_options w_opt = *world->options;
        w_opt.include_sky = 1;    // world.trace_ray(.., true)
        st = pass(&LayerPart::world, world->camera, &w_opt, copies, [&](const LayerPart &p, aicb_ctx *ctx) {
            Outputs o = p.out;
            // a re-issued world pass starts from the same accumulator
            o.target.in_accum = ctx->d_task_aux.get<const float4>();
            if (o.kind == TGT_TEX) o.target.in_depth = ctx->d_task_depth.get<const double>();
            if (o.kind == TGT_TERM) o.target.in_text = ctx->d_task_text.get<const int2>();
            o.target.tex_layer = TEX_WORLD;
            add_no_world(o);
            return o;
        });
    } else if (have_world) {
        aicb_options w_opt = *world->options;
        w_opt.include_sky = 1;
        // without a UI Space the backdrop is still added in front of the world: as the accumulator's starting value
        if (have_backdrop) {
            for (size_t i = 0; i < n_parts; i++) {
                aicb_ctx *ctx = parts[i].world->ctx;
                const size_t n = n_tasks(parts[i]);
                CU(cudaSetDevice(ctx->device));
                TRY(ctx->d_task_aux.ensure(n * sizeof(float4) + 16));
                // stream-ordered: behind the context's last frame, which may still read the accumulators
                const cudaStream_t stream = async ? async : ctx->stream.get();
                if (ctx->frame_in_flight && ctx->last_stream != stream) CU(cudaStreamWaitEvent(stream, ctx->ev1.get(), 0));
                fill_accum_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
                    ctx->d_task_aux.get<float4>(), n, make_float4(backdrop[0], backdrop[1], backdrop[2], backdrop[3]));
                CU(cudaGetLastError());
            }
        }
        st = pass(&LayerPart::world, world->camera, &w_opt, copies, [&](const LayerPart &p, aicb_ctx *ctx) {
            Outputs o = p.out;
            o.target.tex_layer = TEX_WORLD;
            if (have_backdrop) {
                o.target.in_accum = ctx->d_task_aux.get<const float4>();
                if (o.kind == TGT_TERM) o.target.text_start = AICB_TEXT_BLANK;   // the backdrop's hit names no block
            }
            add_no_world(o);
            return o;
        });
    } else {
        aicb_options ui_opt = *ui->options;
        ui_opt.include_sky = 0;
        st = pass(&LayerPart::ui, ui->camera, &ui_opt, copies, [&](const LayerPart &p, aicb_ctx *) {
            Outputs o = p.out;
            o.target.tex_layer = TEX_UI;
            add_backdrop(o);
            add_no_world(o);
            return o;
        });
    }
    if (st != AICB_OK || async) return st;
    std::memset(total, 0, sizeof *total);
    for (const FramePart &p : pass_parts) aicb_merge_info(total, &p.info, false);
    return AICB_OK;
}

aicb_status aicb_check_layers_texture(const aicb_layer *world, const aicb_layer *ui, const float *no_world_rgba,
                                      const double *depth_transform, const uint32_t *pixels, bool pixels_on_device,
                                      size_t n_pixels, const void *out_rgba16f, const float *out_depth,
                                      const aicb_layer **lead_out) {
    const bool have_world = world && world->scene;
    const aicb_layer *lead0 = have_world ? world : ui;
    if (!lead0 || !lead0->camera) return fail(AICB_ERR_INVALID, "a layer needs its camera and options");
    const size_t fb_pixels = (size_t)lead0->camera->fb_width * lead0->camera->fb_height;
    aicb_status st = aicb_check_layers(world, ui, no_world_rgba, fb_pixels, lead_out);
    if (st != AICB_OK) return st;
    if (!depth_transform) return fail(AICB_ERR_INVALID, "depth_transform is NULL");
    if (!pixels && n_pixels != fb_pixels && n_pixels != 0)
        return fail(AICB_ERR_INVALID, "without a pixel list n_pixels must be fb_width * fb_height");
    if (n_pixels > 0xffffffffull / 4) return fail(AICB_ERR_INVALID, "too many pixels");
    if (n_pixels && (!out_rgba16f || !out_depth)) return fail(AICB_ERR_INVALID, "an output is NULL");
    if (pixels && !pixels_on_device)   // (a device list is read as it is)
        for (size_t i = 0; i < n_pixels; i++)
            if (pixels[i] >= fb_pixels) return fail(AICB_ERR_INVALID, "pixel index >= fb_width * fb_height");
    return AICB_OK;
}

void aicb_texture_outputs(const aicb_layer *world, const aicb_layer *ui, const double *depth_transform, Outputs *out) {
    out->full_frame = true;
    out->kind = TGT_TEX;
    // the exposure of each layer's camera (:603-605); a missing layer's is never used
    out->target.tex_exposure[0] = (world && world->scene) ? world->camera->exposure : 1.0f;
    out->target.tex_exposure[1] = (ui && ui->scene) ? ui->camera->exposure : 1.0f;
    const int cols[8] = {2, 6, 10, 14, 3, 7, 11, 15};   // m13 m23 m33 m43, m14 m24 m34 m44 (row-major m11..m44)
    for (int k = 0; k < 8; k++) out->target.depth_m[k] = depth_transform[cols[k]];
}

// The layered calls on one context: its scenes of the layers (group.cu draws them).
static LayeredCall one_context(const aicb_layer *world, const aicb_layer *ui, const float *backdrop_rgba,
                               const float *no_world_rgba) {
    return {world, ui, world ? &world->scene : nullptr, ui ? &ui->scene : nullptr, 1, backdrop_rgba, no_world_rgba};
}

// == RtScene::trace_ray_through_layers for every pixel + the encoder of draw_rgba (renderer.rs:454-478, 287-291).
// The world layer's options choose the sample points (antialiasing) and the post-processing.
aicb_status aicb_render_layers_srgb8(const aicb_layer *world, const aicb_layer *ui, const float backdrop_rgba[4],
                                     const float no_world_rgba[4], uint8_t (*out)[4], size_t out_len,
                                     aicb_render_info *info) {
    return layers_srgb8(one_context(world, ui, backdrop_rgba, no_world_rgba), out, out_len, info);
}

// == the desktop terminal's frame (terminal.rs:114-142): RtScene::trace_ray_through_layers into ColorCharacterBuf
// (:341-394) for every pixel and ColorCharacterBuf::output: post-processed linear RGBA, text and the text's layer.
aicb_status aicb_render_layers_terminal(const aicb_layer *world, const aicb_layer *ui, const float backdrop_rgba[4],
                                        const float no_world_rgba[4], aicb_terminal_pixel *out, size_t out_len,
                                        aicb_render_info *info) {
    return layers_terminal(one_context(world, ui, backdrop_rgba, no_world_rgba), out, out_len, info);
}

// == RaytraceToTexture::do_some_tracing's trace_one over a batch of pixels (raytrace_to_texture.rs:591-683): the
// layers as aicb_render_layers_srgb8 traces them, accumulated in a Split (:922-977), stored as the colour and depth
// texels.  Outputs are packed in list order; without a list they are the whole texture, row-major.
aicb_status aicb_render_layers_texture(const aicb_layer *world, const aicb_layer *ui, const float backdrop_rgba[4],
                                       const float no_world_rgba[4], const double depth_transform[16],
                                       const uint32_t *pixels, size_t n_pixels, uint16_t (*out_rgba16f)[4],
                                       float *out_depth, aicb_render_info *info) {
    return layers_texture(one_context(world, ui, backdrop_rgba, no_world_rgba), depth_transform, pixels, n_pixels,
                          out_rgba16f, out_depth, info);
}

// The three layered calls into the caller's device memory, issued on its stream and finished by aicb_render_finish.
aicb_status aicb_render_layers_device(const aicb_layer *world, const aicb_layer *ui, const float backdrop_rgba[4],
                                      const float no_world_rgba[4], const double depth_transform[16],
                                      const uint32_t *d_pixels, size_t n_pixels, const aicb_device_outputs *outs,
                                      void *stream) {
    return layers_device(one_context(world, ui, backdrop_rgba, no_world_rgba), depth_transform, d_pixels, n_pixels,
                         outs, (cudaStream_t)stream, true, nullptr);
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

}  // extern "C"

// The five views of an orthographic image for its kernels: view v's pixel (px, py) is number first[v] + py * vw[v] + px
// of the views' pixels, and lands at (oy[v] + py) * W + ox[v] + px of the image.
struct OrthoViews {
    uint32_t vw[5], vh[5], ox[5], oy[5];
    uint64_t first[6];
    uint32_t W;
    double inv, lb[3], ub[3];
};

static __device__ __forceinline__ uint32_t ortho_view_of(const OrthoViews &V, uint64_t k) {
    uint32_t v = 0;
    while (k >= V.first[v + 1]) v++;
    return v;
}

// Ray k of the views' pixels, for k in [begin, begin + n): the pixel centre, y flipped, scaled to cubes
// (ortho.rs:278-283), then the view's rotation and corner.  Every sum and product is rounded on its own, as the
// reference rounds them: contracted into an FMA, lb + (px + 0.5) * inv could round differently.  (The library is
// built with -fmad=false; the explicit roundings keep this kernel exact without it.)
static __global__ void __launch_bounds__(256) ortho_rays_kernel(const OrthoViews V, uint64_t begin, uint32_t n,
                                                                double *__restrict__ rays) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = begin + i;
    const uint32_t v = ortho_view_of(V, k);
    const uint64_t local = k - V.first[v];
    const uint32_t px = (uint32_t)(local % V.vw[v]), py = (uint32_t)(local / V.vw[v]);
    const double u = __dmul_rn(__dadd_rn((double)px, 0.5), V.inv), w = -__dmul_rn(__dadd_rn((double)py, 0.5), V.inv);
    auto add = [](double a, double b) { return __dadd_rn(a, b); };
    auto sub = [](double a, double b) { return __dsub_rn(a, b); };
    const double *lb = V.lb, *ub = V.ub;
    double o[3], d[3] = {0.0, 0.0, 0.0};
    switch (v) {
        case 0: o[0] = add(lb[0], u); o[1] = ub[1]; o[2] = sub(lb[2], w); d[1] = -1.0; break;   // top: Face::PY
        case 1: o[0] = lb[0]; o[1] = add(ub[1], w); o[2] = add(lb[2], u); d[0] = 1.0; break;    // left: Face::NX
        case 2: o[0] = add(lb[0], u); o[1] = add(ub[1], w); o[2] = ub[2]; d[2] = -1.0; break;   // front: Face::PZ
        case 3: o[0] = ub[0]; o[1] = add(ub[1], w); o[2] = sub(ub[2], u); d[0] = -1.0; break;   // right: Face::PX
        default: o[0] = add(lb[0], u); o[1] = lb[1]; o[2] = add(ub[2], w); d[1] = 1.0; break;   // bottom: Face::NY
    }
    double *r = rays + 6 * (size_t)i;
    for (int a = 0; a < 3; a++) {
        r[a] = o[a];
        r[3 + a] = d[a];
    }
}

// The traced pixels, in the rays' order, to their places in the image.
static __global__ void __launch_bounds__(256) ortho_place_kernel(const OrthoViews V, const uchar4 *__restrict__ traced,
                                                                 uint64_t n, uchar4 *__restrict__ image) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t v = ortho_view_of(V, k);
    const uint64_t local = k - V.first[v];
    const uint32_t px = (uint32_t)(local % V.vw[v]), py = (uint32_t)(local / V.vw[v]);
    image[(size_t)(V.oy[v] + py) * V.W + V.ox[v] + px] = traced[k];
}

// The views' rays are built on the device, each context building its range of whole warps of them into its d_aux, and
// go through the explicit-ray path; every context stores its pixels in ray order at its range's offset in device 0's
// d_out.  Device 0 clears the image to Rgba::TRANSPARENT first and places the pixels once every context is done.
aicb_status ortho_srgb8(Replicas r, uint32_t resolution, uint8_t (*out)[4], size_t out_len, aicb_render_info *info) {
    aicb_scene *s = r.scene[0];
    uint32_t W = 0, H = 0;
    aicb_status st = aicb_ortho_image_size(s, resolution, &W, &H);
    if (st != AICB_OK) return st;
    if (out_len != (size_t)W * H) return fail(AICB_ERR_INVALID, "Viewport size does not match output buffer length");
    if (out_len && !out) return fail(AICB_ERR_INVALID, "out is NULL");
    const DeviceScene &ds = s->ds;
    OrthoViews V;
    ortho_views(ds, resolution, V.vw, V.vh, V.ox, V.oy, &V.W, &H);
    V.inv = 1.0 / (double)resolution;   // (a power of two: exact)
    for (int a = 0; a < 3; a++) {
        V.lb[a] = (double)ds.lo[a];
        V.ub[a] = (double)ds.lo[a] + ds.size[a];
    }
    V.first[0] = 0;
    for (int v = 0; v < 5; v++) V.first[v + 1] = V.first[v] + (uint64_t)V.vw[v] * V.vh[v];
    const uint64_t n = V.first[5];
    if (info) std::memset(info, 0, sizeof *info);
    aicb_ctx *root = r.ctx[0];
    CU(cudaSetDevice(root->device));
    const size_t off_traced = (out_len * 4 + 255) & ~(size_t)255;   // d_out: the image, then the traced pixels
    TRY(root->d_out.ensure(off_traced + n * 4 + 16));
    uchar4 *image = root->d_out.get<uchar4>(), *traced = (uchar4 *)(root->d_out.get<char>() + off_traced);
    CU(cudaMemsetAsync(image, 0, out_len * 4, root->stream.get()));
    std::vector<FramePart> parts;
    if (n) {
        const std::vector<WarpRange> ranges = warp_ranges(n, r.n);
        for (size_t i = 0; i < ranges.size(); i++) {
            if (ranges[i].count > 0xffffffffull) return fail(AICB_ERR_INVALID, "too many rays");
            aicb_ctx *ctx = r.ctx[i];
            const uint32_t count = (uint32_t)ranges[i].count;
            CU(cudaSetDevice(ctx->device));
            TRY(ctx->d_aux.ensure((size_t)count * 48 + 16));
            ortho_rays_kernel<<<(count + 255) / 256, 256, 0, ctx->stream.get()>>>(V, ranges[i].begin, count,
                                                                                  ctx->d_aux.get<double>());
            CU(cudaGetLastError());
            FramePart p{r.scene[i]};
            p.out.target.out_srgb8 = traced + ranges[i].begin;
            p.out.rays = ctx->d_aux.get<double>();
            p.out.n_rays = count;
            parts.push_back(p);
        }
        aicb_options opt;   // GraphicsOptions::UNALTERED_COLORS (graphics_options.rs:168)
        std::memset(&opt, 0, sizeof opt);
        opt.fog = AICB_FOG_NONE;
        opt.lighting_display = AICB_LIGHT_NONE;
        opt.transparency = AICB_TRANSPARENCY_VOLUMETRIC;
        opt.tone_mapping = AICB_TONE_CLAMP;
        opt.maximum_intensity = INFINITY;
        opt.view_distance = 200.0;
        opt.include_sky = 1;
        TRY(aicb_trace_pass(parts.data(), parts.size(), nullptr, &opt, info != nullptr, {}));
        TRY(fan_in(r.ctx, parts.size()));
        ortho_place_kernel<<<(unsigned)((n + 255) / 256), 256, 0, root->stream.get()>>>(V, traced, n, image);
        CU(cudaGetLastError());
        if (info)
            for (const FramePart &p : parts) aicb_merge_info(info, &p.info, false);
    }
    return deliver(r.ctx, 1, {{out, image, out_len * 4}});   // (the other contexts are waited for above)
}

extern "C" {

aicb_status aicb_render_orthographic(aicb_scene *s, uint32_t resolution, uint8_t (*out)[4], size_t out_len,
                                     aicb_render_info *info) {
    return on_scene(s, [&](Replicas r) { return ortho_srgb8(r, resolution, out, out_len, info); });
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
    const aicb_device_outputs o = colorbuf_outputs(out_cb, depth, hit, steps, n);
    return on_scene(s, [&](Replicas r) { return rays_host(r, origin_dir, opt, o, info); });
}

}
