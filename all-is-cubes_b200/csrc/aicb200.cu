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

static bool voxel_invisible(const aicb_voxel &v) {
    return v.rgba[3] == 0.0f && v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f;
}

// TracingBlock::from_block (sr.rs:579-587) for one block definition: its 32-byte record, classification, brick words
// in the wide form (trace_kernel.cuh) and palette entries (appended to `bricks` / `palette`; the record's offsets are
// relative to those vectors), plus what the marching kernel needs of each surface: {alpha, an upper bound of
// log2(1 - alpha)} per palette entry.
// Called by flatten_blocks alone.
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

static aicb_status flatten_block(const aicb_block_desc &b, BlockRec &r, uint8_t &kind, std::vector<uint32_t> &bricks,
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
        if (b.n_palette > 65536)
            return fail(AICB_ERR_UNSUPPORTED, "block palettes above 65536 entries are not supported: a voxel's palette "
                                              "index (VoxelIndex) is 16 bits");
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
            const uint32_t v = b.indices[k];
            bricks.push_back(v << 16 | (voxel_invisible(b.palette[v]) ? 0x8000u : 0u));
        }
        for (size_t k = 0; k < b.n_palette; k++) push_voxel(b.palette[k]);
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
        default: return lc == LC_NONE ? resolve_kernel<LC_NONE, TGT_FRAME> : resolve_kernel<LC_FLAT, TGT_FRAME>;
    }
}
static kernel_fn encode_for(int tgt) {
    return tgt == TGT_TEX ? encode_kernel<TGT_TEX> : (tgt == TGT_TERM ? encode_kernel<TGT_TERM> : encode_kernel<TGT_FRAME>);
}

// Launches the trace kernel on `stream`. Camera rays when cam != NULL, the explicit rays of `out` otherwise.  With
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
        if (out.target.pixel_list) {   // one pixel task per listed pixel, 32 consecutive entries per warp
            P.tiles_x = (out.target.n_list + 31) / 32;
            P.tiles_y = 1;
            P.n_tasks = out.target.n_list;
            pixels = out.target.n_list;
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
    TRY(ctx->primary.size(chunk_cap, P.hit_capacity, !fused));
    ctx->primary.bind(P, chunk_cap, !fused);
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
            gen_kernel<<<(n + 127) / 128, 128, 0, stream>>>(P, n);
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
    // live data only: the dead part of the pool is compacted away before it could push positions past 2^32
    // (flatten_placeable)
    if (brick_room(h.n_bricks, h.dead_bricks, f->bricks.size()) == BrickRoom::too_big)
        return fail(AICB_ERR_INVALID, "brick pool exceeds 2^32 voxels");
    return AICB_OK;
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
    TRY(grow(t.bricks, h.n_bricks * wb, f.bricks.size() * wb));
    TRY(grow(t.palette, h.n_palette * sizeof(float4), f.palette.size() * sizeof(float4)));
    TRY(grow(t.pal_tab, h.n_palette / 2 * sizeof(float2), f.pal_tab.size() * sizeof(float2)));
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
    h.n_bricks += f.bricks.size();
    h.n_palette += f.palette.size();
    h.wide_bricks = f.wide_bricks;
}

// f (flatten_placeable) placed in every replica's table: room in each, then the copies, recorded in ev_delta (renders
// on other streams wait for it, launch_trace), and the bookkeeping.  Records are written over in place (`indices`)
// only once every replica has room and its context has been waited for (wait_context).
static aicb_status place(Replicas r, const FlatBlocks &f, const uint16_t *indices) {
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
        CU(cudaSetDevice(r.ctx[i]->device));
        TRY(copy(r.scene[i]->blocks, h, f, indices, r.ctx[i]->stream.get()));
        CU(cudaEventRecord(r.ctx[i]->ev_delta.get(), r.ctx[i]->stream.get()));
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

aicb_status scenes_create(aicb_ctx *const *ctx, size_t n, const aicb_scene_desc *d, aicb_scene **out) {
    const int64_t LIM = 1 << 30;
    uint64_t volume = 1;
    for (int a = 0; a < 3; a++) {
        int64_t lo = d->bounds.lower[a], hi = lo + (int64_t)d->bounds.size[a];
        if (lo < -LIM || hi > LIM) return fail(AICB_ERR_INVALID, "space bounds must lie within +-2^30");
        volume *= d->bounds.size[a];
        if (volume > (1ull << 31)) return fail(AICB_ERR_INVALID, "space volume exceeds 2^31 cubes");
    }
    if (volume && !d->block_ids) return fail(AICB_ERR_INVALID, "block_ids is NULL");
    if (volume && d->n_blocks == 0) return fail(AICB_ERR_INVALID, "non-empty space with an empty block table");
    if (d->n_blocks && !d->blocks) return fail(AICB_ERR_INVALID, "blocks is NULL");
    auto host = std::make_unique<SpaceHost>();   // empty until every replica holds the table
    FlatBlocks f;
    TRY(flatten_blocks(*host, d->blocks, d->n_blocks, nullptr, &f));

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
    const void *cells = wide ? (const void *)cells32.data() : cells16.data();
    const size_t cell_bytes = volume * (wide ? 4 : 2);

    // ---- one scene per context, complete when it is returned; until then a failure frees it ------------------------
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
            TRY(s->d_cells.upload(cells, cell_bytes));
            s->device_bytes += cell_bytes;
            if (d->light) {
                TRY(s->d_light.upload(d->light, volume * 4));
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
        TRY(copy(s->blocks, *host, f, nullptr, c->stream.get()));
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
    host->h_ids.assign(d->block_ids, d->block_ids + volume);
    host->light_max_distance = d->light_max_distance;
    book(*host, f, nullptr);
    out[0]->own_host = std::move(host);
    return AICB_OK;
}

// flatten_blocks against the scene's table, for an update (`indices`) or an append (nullptr) of the scene's replicas,
// such that the result can be placed: brick positions are u32, so when the live data fits but the pool's words in use
// plus the new ones would not (brick_room), every replica's brick pool is compacted first and the definitions are
// flattened again against the compacted table.  A compaction moves the pools, so each replica's context is waited
// for first (wait_context).  Wide definitions for a narrow pool widen every replica's pool first.
static aicb_status flatten_placeable(Replicas r, const aicb_block_desc *descs, size_t n_blocks, const uint16_t *indices,
                                     FlatBlocks *f) {
    const SpaceHost &h = *r.scene[0]->host;
    TRY(flatten_blocks(h, descs, n_blocks, indices, f));
    if (brick_room(h.n_bricks, h.dead_bricks, f->bricks.size()) == BrickRoom::compact_first) {
        for (size_t i = 0; i < r.n; i++) {
            CU(cudaSetDevice(r.ctx[i]->device));
            TRY(wait_context(r.ctx[i]));
        }
        TRY(compact_pools(r, true, false));
        *f = FlatBlocks();
        TRY(flatten_blocks(h, descs, n_blocks, indices, f));
    }
    return f->wide_bricks && !h.wide_bricks ? widen_bricks(r, f->bricks.size()) : AICB_OK;
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

aicb_status check_region(const aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                         RegionBox *box) {
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
                         const uint8_t (*light)[4], uint32_t *d_mask, uint32_t *d_n_changed) {
    aicb_ctx *ctx = s->ctx;
    cudaStream_t stream = ctx->stream.get();
    const size_t vol = box.volume(), rows = (size_t)box.size[0] * box.size[1], sz = box.size[2];
    if (!s->d_light) light = nullptr;
    // the ids, then (16-byte aligned) the texels
    const size_t id_bytes = ids ? (vol * 2 + 15) / 16 * 16 : 0, bytes = id_bytes + (light ? vol * 4 : 0);
    if (bytes) {
        TRY(delta_room(ctx, bytes));
        if (ids) std::memcpy(ctx->h_delta.get(), ids, vol * 2);
        if (light) std::memcpy(ctx->h_delta.get<char>() + id_bytes, light, vol * 4);
        CU(cudaMemcpyAsync(ctx->d_delta.get(), ctx->h_delta.get(), bytes, cudaMemcpyHostToDevice, stream));
    }
    if (d_mask) CU(cudaMemsetAsync(d_mask, 0, (vol + 31) / 32 * 4, stream));
    const bool wide = s->ds.wide_cells;
    const uint32_t per = wide ? 4u : 8u, chunks_per_row = (uint32_t)((sz + per - 1) / per + 1);
    const uint32_t n_items = (uint32_t)(rows * chunks_per_row);
    const uint16_t *d_ids = ids ? ctx->d_delta.get<const uint16_t>() : nullptr;
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
        k_region_texels<<<(n + 255) / 256, 256, 0, stream>>>(
            s->ds, box, (const uint32_t *)(ctx->d_delta.get<const char>() + id_bytes), cpr, n, s->d_light.get<uint32_t>());
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
    for (size_t k = 0; k < r.n; k++) {
        CU(cudaSetDevice(r.ctx[k]->device));
        TRY(region_cells(r.scene[k], box, ids, uniform_id, light, nullptr, nullptr));
        CU(cudaEventRecord(r.ctx[k]->ev_delta.get(), r.ctx[k]->stream.get()));  // renders on other streams wait for it
    }
    mirror_region(*r.scene[0]->host, r.scene[0]->ds, box, ids, uniform_id);
    return AICB_OK;
}

aicb_status scenes_update_blocks(Replicas r, const uint16_t *indices, const aicb_block_desc *descs, size_t n_blocks) {
    if (n_blocks && (!indices || !descs)) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n_blocks == 0) return AICB_OK;
    const SpaceHost &h = *r.scene[0]->host;
    FlatBlocks f;
    TRY(flatten_placeable(r, descs, n_blocks, indices, &f));
    // cubes that hold a block whose kind changes carry the new kind in their cell words
    std::vector<uint8_t> kind(h.kind);
    for (size_t i = 0; i < n_blocks; i++) kind[indices[i]] = f.kinds[i];
    std::vector<CubeDelta> ops;
    if (kind != h.kind) {
        if (h.h_ids.size() != h.volume) return fail(AICB_ERR_INVALID, "scene has no host mirror of its block ids");
        const bool wide = r.scene[0]->ds.wide_cells;
        uint32_t idx = 0;
        for (const uint16_t id : h.h_ids) {
            if (kind[id] != h.kind[id]) ops.push_back({idx, cell_word(id, kind[id], wide), 0, 0});
            idx++;
        }
    }
    TRY(place(r, f, indices));   // (which waits for every context: compaction moves the pools)
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
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));
        TRY(wait_context(ctx));   // the call returns once its writes are done
    }
    return AICB_OK;
}

// The copies are queued on the context's stream and ev_delta is recorded behind them, as aicb_scene_update_cubes does:
// a frame issued later on another stream waits for them (launch_trace).  The new entries go to spare capacity that no
// cell refers to until a later, stream-ordered cube update, so a frame in flight is not disturbed; an array that has to
// move is freed only after it (Retired).
aicb_status scenes_append_blocks(Replicas r, const aicb_block_desc *descs, size_t n_blocks) {
    if (n_blocks && !descs) return fail(AICB_ERR_INVALID, "NULL argument");
    if (n_blocks == 0) return AICB_OK;
    const SpaceHost &h = *r.scene[0]->host;
    FlatBlocks f;
    TRY(flatten_placeable(r, descs, n_blocks, nullptr, &f));
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
    return place(r, f, nullptr);
}

// Mutation::fill_uniform over the whole Space (space.rs:1461-1474), the source of SpaceChange::EveryBlock: the table
// becomes [block] in exact-size buffers, as a new scene's, and every cell id 0 with its kind, written on the device
// (u32 cells go back to u16: a one-block table fits them).  Light is not touched.  Each replica's context is waited for
// first, since the table and the cells are replaced, and the call returns once its writes are done.  Every replica's
// new arrays are allocated before any replica changes, so a failure leaves the scene as it was.
aicb_status scenes_fill_uniform(Replicas r, const aicb_block_desc *block) {
    if (!block) return fail(AICB_ERR_INVALID, "NULL argument");
    const SpaceHost empty;   // an empty table's bookkeeping, which the new tables are placed against
    FlatBlocks f;
    TRY(flatten_blocks(empty, block, 1, nullptr, &f));
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
        TRY(copy(sc->blocks, empty, f, nullptr, stream));
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
    return AICB_OK;
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

// == SpaceChange::EveryBlock (Mutation::fill_uniform over the whole bounds, space.rs:1461-1474).
aicb_status aicb_scene_fill_uniform(aicb_scene *s, const aicb_block_desc *block) {
    return on_scene(s, [&](Replicas r) { return scenes_fill_uniform(r, block); });
}

aicb_status aicb_scene_upload_light(aicb_scene *s, const uint8_t (*light)[4], size_t n_texels) {
    return on_scene(s, [&](Replicas r) { return scenes_upload_light(r, light, n_texels); });
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
        return (p.out.target.pixel_list ? (size_t)p.out.target.n_list
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

void aicb_texture_target(const aicb_layer *world, const aicb_layer *ui, const double *depth_transform, Outputs *out) {
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
