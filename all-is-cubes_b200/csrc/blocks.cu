// blocks.cu — block definitions whose voxel data is in device memory (aicb_scene_update_blocks_device,
// aicb_scene_append_blocks_device): the kernels that check them and write them into a scene's block table, and the
// light-side record of a definition.  aicb200.cu decides where everything goes, from sizes the host has; these
// kernels only move the caller's voxels into place, in the form flatten_block gives them on the host.
//   k_block_verdict  the first block with a voxel index >= its palette's size (atomicMin), and the kind of each
//                    single-voxel block, whose voxel decides it: the only bytes read back before the call places;
//   k_block_bricks   each recursive block's brick words, straight into the pool after the words in use, 16 bytes per
//                    store where the pool's alignment allows;
//   k_block_palette  each palette entry as the pool's two float4 and its pal_tab pair (surface_entry);
//   k_block_records  each written id's BlockRec, blk_tab entry and light record;
//   k_rekind_cells   the cells of the ids whose kind changed, in one streaming pass against a per-id table.
#include <algorithm>
#include <cstring>

#include "block_words.cuh"
#include "internal.h"
#include "light_kernel.cuh"

using namespace aicb;

// The light-side record of a block definition (internal.h): its face colours, emission and flags.
__host__ __device__ LightBlockDev light_block(const aicb_block_desc &b) {
    LightBlockDev o;
    memset(&o, 0, sizeof o);
    memcpy(o.face_color[0], b.light_color, 16);
    for (int f = 0; f < 6; f++) memcpy(o.face_color[f + 1], b.light_face_colors[f], 16);
    memcpy(o.emission, b.light_emission, 12);
    uint32_t fl = b.light_opaque_faces & 0x3f;
    if (fl == 0x3f) fl |= LB_ALL_OPAQUE;
    if (b.light_visible) fl |= LB_VISIBLE;
    if (!(b.light_emission[0] == 0.0f && b.light_emission[1] == 0.0f && b.light_emission[2] == 0.0f)) fl |= LB_EMISSIVE;
    o.flags = fl;
    return o;
}

namespace {

const unsigned THREADS = 256;

// single_voxel_of on the device: AIR, palette[0] or palette[indices[0]] (an index past the palette is the call's
// rejection, and reads AIR here).
__device__ aicb_voxel single_voxel(const DeviceBlockJob &J) {
    aicb_voxel v;
    memset(&v, 0, sizeof v);
    v.flags = AICB_VOXEL_NOT_SELECTABLE | AICB_VOXEL_NO_COLLISION;   // Evoxel::AIR
    if (J.single == SINGLE_FIRST) v = J.palette[0];
    else if (J.single == SINGLE_INDEXED) {
        const uint32_t k = J.indices[0];
        if (k < J.n_palette) v = J.palette[k];
    }
    return v;
}

__device__ __forceinline__ bool invisible_at(const aicb_voxel *palette, uint32_t k) {
    const float *p = reinterpret_cast<const float *>(palette + k);
    return __ldg(p + 3) == 0.0f && __ldg(p + 4) == 0.0f && __ldg(p + 5) == 0.0f && __ldg(p + 6) == 0.0f;
}

// grid (jobs, chunks): job blockIdx.x's indices, gridDim.y CTAs each
__global__ void __launch_bounds__(THREADS) k_block_verdict(const DeviceBlockJob *jobs, InputVerdict *v, uint8_t *kinds) {
    const DeviceBlockJob &J = jobs[blockIdx.x];
    bool bad = false;
    if (J.indices)
        for (uint64_t k = (uint64_t)blockIdx.y * THREADS + threadIdx.x; k < J.n_indices; k += (uint64_t)gridDim.y * THREADS)
            bad |= __ldg(J.indices + k) >= J.n_palette;
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicMin(&v->first_bad, (unsigned long long)blockIdx.x);
    if (blockIdx.y == 0 && threadIdx.x == 0 && J.single != SINGLE_NONE)
        kinds[blockIdx.x] = (uint8_t)(voxel_invisible(single_voxel(J)) ? KIND_INVISIBLE : KIND_SINGLE);
}

// A warp's OR of `mask` into a job's mask word.
__device__ __forceinline__ void or_masks(DeviceBlockJob &J, uint32_t mask) {
    mask = __reduce_or_sync(0xffffffffu, mask);
    if ((threadIdx.x & 31) == 0 && mask) atomicOr(&J.masks, mask);
}

// Brick words of the recursive jobs at pool positions [brick_off, brick_off + n_indices), in groups of 16 bytes of
// the pool: a whole group is one store, a group cut by the range's ends is stored word by word.  The collision masks of
// the entries the voxels use go into the job's mask word (bits 2-3), and bit 4 if one of them is visible.
template <bool WIDE>
__global__ void __launch_bounds__(THREADS) k_block_bricks(DeviceBlockJob *jobs, void *pool) {
    using Word = typename std::conditional<WIDE, uint32_t, uint16_t>::type;
    constexpr uint32_t G = 16 / sizeof(Word);
    DeviceBlockJob &J = jobs[blockIdx.x];
    if (J.kind != KIND_RECURSIVE) return;
    uint32_t used = 0;
    const uint64_t lo = J.brick_off, hi = lo + J.n_indices;
    Word *out = static_cast<Word *>(pool);
    for (uint64_t g = lo / G + (uint64_t)blockIdx.y * THREADS + threadIdx.x; g * G < hi; g += (uint64_t)gridDim.y * THREADS) {
        union {
            uint4 v;
            Word w[G];
        } u;
#pragma unroll
        for (uint32_t j = 0; j < G; j++) {
            const uint64_t p = g * G + j;
            if (p < lo || p >= hi) continue;
            const uint32_t k = __ldg(J.indices + (p - lo));
            const uint32_t inv = invisible_at(J.palette, k) ? 0x8000u : 0u;
            used |= collision_mask(__ldg(&J.palette[k].flags)) | (inv ? 0u : 4u);
            u.w[j] = (Word)(WIDE ? k << 16 | inv : k | inv);
        }
        if (g * G >= lo && g * G + G <= hi) reinterpret_cast<uint4 *>(out)[g] = u.v;
        else
            for (uint32_t j = 0; j < G; j++)
                if (g * G + j >= lo && g * G + j < hi) out[g * G + j] = u.w[j];
    }
    or_masks(J, used << 2);
}

// Palette entries: a recursive job's palette, a single voxel's one entry; air has none.  A recursive job's palette's
// collision mask goes into its mask word (bits 0-1).
__global__ void __launch_bounds__(THREADS) k_block_palette(DeviceBlockJob *jobs, float4 *palette, float2 *pal_tab) {
    DeviceBlockJob &J = jobs[blockIdx.x];
    uint32_t mask = 0;
    for (uint32_t e = blockIdx.y * THREADS + threadIdx.x; e < J.n_entries; e += gridDim.y * THREADS) {
        const aicb_voxel v = J.kind == KIND_RECURSIVE ? J.palette[e] : single_voxel(J);
        const size_t at = (size_t)J.pal_off + e;
        palette[2 * at] = make_float4(v.rgba[0], v.rgba[1], v.rgba[2], v.rgba[3]);
        palette[2 * at + 1] = make_float4(v.emission[0], v.emission[1], v.emission[2], voxel_flags(v));
        pal_tab[at] = surface_entry(v.rgba[3]);
        mask |= collision_mask(v.flags);
    }
    if (J.kind == KIND_RECURSIVE) or_masks(J, mask);
}

// compute_derived of a single voxel (derived.rs:84-104), as derive.cu's single_light.
__device__ aicb_block_light single_light(const aicb_voxel &v) {
    aicb_block_light o;
    memset(&o, 0, sizeof o);
    for (int f = 0; f < 6; f++) memcpy(o.face_colors[f], v.rgba, sizeof v.rgba);
    memcpy(o.color, v.rgba, sizeof v.rgba);
    memcpy(o.emission, v.emission, sizeof v.emission);
    o.opaque_faces = v.rgba[3] == 1.0f ? 0x3f : 0;
    const bool emits = !(v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f);
    o.visible = (!(v.rgba[3] == 0.0f) || emits) ? 1 : 0;
    return o;
}

// One thread per job that writes its id's records (a repeated id: its last definition of the call).
// A recursive job's collision and visible bits come from the masks k_block_palette and k_block_bricks left in its mask
// word.
__global__ void __launch_bounds__(THREADS) k_block_records(const DeviceBlockJob *jobs, uint32_t n, BlockRec *blocks,
                                                           float4 *blk_tab, LightBlockDev *light,
                                                           const aicb_block_light *derived) {
    const uint32_t i = blockIdx.x * THREADS + threadIdx.x;
    if (i >= n) return;
    const DeviceBlockJob &J = jobs[i];
    if (J.id == NO_ID) return;
    BlockRec rec = J.rec;   // an air block's collision bits and a single voxel's visible bit are in it already (block_rec)
    if (J.kind == KIND_RECURSIVE && (J.masks & 16u)) rec.flags |= BLOCK_VISIBLE;
    if (!(rec.flags & BLOCK_COLLISION_NONE)) {
        if (J.kind == KIND_RECURSIVE)
            rec.flags |= block_collision(J.masks & 3u, (J.masks >> 2) & 3u, less_than_full(rec));
        else if (single_voxel(J).flags & AICB_VOXEL_NO_COLLISION)
            rec.flags |= BLOCK_COLLISION_NONE;
    }
    blocks[J.id] = rec;
    float4 e = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (J.kind == KIND_SINGLE) {
        const float2 s = surface_entry(single_voxel(J).rgba[3]);
        e = make_float4(s.x, s.y, __uint_as_float(J.rec.pal_off), 0.0f);
    }
    blk_tab[J.id] = e;
    if (J.derived == LIGHT_GIVEN) {
        light[J.id] = J.light;
        return;
    }
    // the descriptor's light fields from compute_derived; light_visible ORs in the caller's animation hint
    const aicb_block_light d = J.derived == LIGHT_SINGLE ? single_light(single_voxel(J)) : derived[J.derived];
    aicb_block_desc b;
    memset(&b, 0, sizeof b);
    memcpy(b.light_face_colors, d.face_colors, sizeof d.face_colors);
    memcpy(b.light_color, d.color, sizeof d.color);
    memcpy(b.light_emission, d.emission, sizeof d.emission);
    b.light_opaque_faces = d.opaque_faces;
    b.light_visible = (uint8_t)(d.visible | J.light_visible);
    light[J.id] = light_block(b);
}

// Cells whose id has a word in `word` (~0u: the id keeps its kind) take it: 16 bytes per load, a store only where a
// cell changed; the last n % per cells one at a time.
template <bool WIDE>
__global__ void __launch_bounds__(THREADS) k_rekind_cells(void *cells, size_t n, const uint32_t *__restrict__ word) {
    using Cell = typename std::conditional<WIDE, uint32_t, uint16_t>::type;
    constexpr uint32_t PER = 16 / sizeof(Cell), ID_MASK = WIDE ? 0xffffu : 0x3fffu;
    Cell *c = static_cast<Cell *>(cells);
    const size_t stride = (size_t)gridDim.x * THREADS, first = (size_t)blockIdx.x * THREADS + threadIdx.x;
    const size_t groups = n / PER;
    for (size_t g = first; g < groups; g += stride) {
        union {
            uint4 v;
            Cell w[PER];
        } u;
        u.v = __ldcs(reinterpret_cast<const uint4 *>(c) + g);
        bool changed = false;
#pragma unroll
        for (uint32_t j = 0; j < PER; j++) {
            const uint32_t t = __ldg(word + (u.w[j] & ID_MASK));
            if (t != NO_WORD) {
                u.w[j] = (Cell)t;
                changed = true;
            }
        }
        if (changed) reinterpret_cast<uint4 *>(c)[g] = u.v;
    }
    for (size_t i = groups * PER + first; i < n; i += stride) {
        const uint32_t t = word[c[i] & ID_MASK];
        if (t != NO_WORD) c[i] = (Cell)t;
    }
}

unsigned chunks_for(uint64_t most, uint64_t per_cta, unsigned cap) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((most + per_cta - 1) / per_cta, cap));
}

}  // namespace

aicb_status issue_block_verdict(cudaStream_t stream, const DeviceBlockJob *jobs, uint32_t n, uint64_t most_indices,
                                InputVerdict *v, uint8_t *kinds) {
    if (n == 0) return AICB_OK;
    k_block_verdict<<<dim3(n, chunks_for(most_indices, THREADS * 8, 1024)), THREADS, 0, stream>>>(jobs, v, kinds);
    CU(cudaGetLastError());
    return AICB_OK;
}

aicb_status issue_block_data(cudaStream_t stream, DeviceBlockJob *jobs, uint32_t n, uint64_t most_words,
                             uint64_t most_entries, bool wide_bricks, const BlockTable &t,
                             const aicb_block_light *derived) {
    if (n == 0) return AICB_OK;
    if (most_words) {
        const dim3 grid(n, chunks_for(most_words, THREADS * (wide_bricks ? 4 : 8) * 4, 1024));
        if (wide_bricks) k_block_bricks<true><<<grid, THREADS, 0, stream>>>(jobs, t.bricks.get());
        else k_block_bricks<false><<<grid, THREADS, 0, stream>>>(jobs, t.bricks.get());
    }
    if (most_entries)
        k_block_palette<<<dim3(n, chunks_for(most_entries, THREADS * 4, 256)), THREADS, 0, stream>>>(
            jobs, t.palette.get<float4>(), t.pal_tab.get<float2>());
    k_block_records<<<(n + THREADS - 1) / THREADS, THREADS, 0, stream>>>(jobs, n, t.blocks.get<BlockRec>(),
                                                                         t.blk_tab.get<float4>(),
                                                                         t.light.get<LightBlockDev>(), derived);
    CU(cudaGetLastError());
    return AICB_OK;
}

aicb_status issue_rekind_cells(const aicb_ctx *ctx, void *cells, bool wide, size_t n, const uint32_t *word) {
    if (n == 0) return AICB_OK;
    const unsigned grid = chunks_for(n, (uint64_t)THREADS * (wide ? 4 : 8), (unsigned)ctx->num_sms * 16);
    if (wide) k_rekind_cells<true><<<grid, THREADS, 0, ctx->stream.get()>>>(cells, n, word);
    else k_rekind_cells<false><<<grid, THREADS, 0, ctx->stream.get()>>>(cells, n, word);
    CU(cudaGetLastError());
    return AICB_OK;
}
