// block_words.cuh — what one palette entry of a block definition becomes in a scene's block table: its invisible flag
// (the brick words' bit 15) and what the marching kernel needs of its surface, {alpha, an upper bound of
// log2(1 - alpha)} (pal_tab).  __host__ __device__, so that the host flattening (aicb200.cu: flatten_block) and the
// kernels that flatten definitions held in device memory (blocks.cu) evaluate one expression each, and their tables
// are the same bytes.  tests/test_gpu_block_words.py checks surface_entry on the device against the host on every f32
// bit pattern of alpha.
#pragma once
#include <cmath>
#include <cstring>

#include <cuda_runtime.h>

#include "../../include/aicb200.h"

namespace aicb {

// A voxel the marching kernel steps over (bit 15 of its brick word): fully transparent and not emissive.
__host__ __device__ inline bool voxel_invisible(const aicb_voxel &v) {
    return v.rgba[3] == 0.0f && v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f;
}

// The .w lane of a palette entry's second float4 (its emission): the voxel's AICB_VOXEL_NOT_SELECTABLE bit, which only
// the cursor reads, and its AICB_VOXEL_NO_COLLISION bit, which only the body step reads.  The other bits of
// aicb_voxel::flags are not kept.
__host__ __device__ inline float voxel_flags(const aicb_voxel &v) {
    const uint32_t f = v.flags & (AICB_VOXEL_NOT_SELECTABLE | AICB_VOXEL_NO_COLLISION);
    float w;
    memcpy(&w, &f, 4);
    return w;
}

// A voxel's collision as a bit of a collision mask: 1 some voxel is Hard, 2 some voxel is None.
__host__ __device__ inline uint32_t collision_mask(uint32_t voxel_flags_word) {
    return (voxel_flags_word & AICB_VOXEL_NO_COLLISION) ? 2u : 1u;
}

// A recursive block's BlockRec collision bits (trace_kernel.cuh: BLOCK_COLLISION_*) from the collision masks of its
// palette and of the palette entries its voxels use, as compute_derived's uniform_collision (derived.rs:159-190): the
// implicit air outside voxel bounds smaller than the block counts as None; then the palette, if all its entries agree;
// then the entries in use; else mixed.  An empty sequence agrees on nothing.
__host__ __device__ inline uint32_t block_collision(uint32_t palette_mask, uint32_t used_mask, bool less_than_full) {
    const uint32_t outside = less_than_full ? 2u : 0u, p = palette_mask | outside, u = used_mask | outside;
    if (p == 1u || u == 1u) return 0u;
    if (p == 2u || u == 2u) return 2u;   // BLOCK_COLLISION_NONE
    return 4u;                           // BLOCK_COLLISION_MIXED
}

// {alpha, l2a}: l2a >= log2(1 - alpha) (the f32 value apply_transmittance raises to a span's thickness), so the
// marching kernel's log-domain transmittance stays an upper bound.  log2 is evaluated in f64 (glibc's on the host,
// libdevice's on the device), rounded to f32 and stepped up by one ulp.
__host__ __device__ inline float2 surface_entry(float alpha) {
    float l2a;
    if (alpha >= 1.0f) l2a = -INFINITY;
    else if (!(alpha > 0.0f)) l2a = 0.0f;
    else {
        const float unit_t = 1.0f - alpha;
        l2a = nextafterf((float)log2((double)unit_t), INFINITY);
        if (l2a > 0.0f) l2a = 0.0f;
    }
    return make_float2(alpha, l2a);
}

}  // namespace aicb
