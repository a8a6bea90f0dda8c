// derive.cu — compute_derived (block/eval/derived.rs:80-216) for the light fields of EvaluatedBlock, on the device
// (include/aicb200.h: aicb_derive_block_light).
//
// A single voxel is its own derived data, copied on the host.  Every other block is traced: one ray per voxel face of
// each of the six sides of its data bounds (trace_for_eval, raytracer_components.rs:174-200), whose four VoxSum terms
// are summed per face in the reference's order.  Four kernels, in stream order:
//   k_derive_palette  apply_transmittance(color, 1 / resolution) of every palette entry, once: what a voxel adds to a
//                     ray (ColorBuf::from(adjusted color), emission * coefficient) and its opacity category;
//   k_derive_scan     one thread per voxel: Derived::visible (any voxel not Invisible) and, on each surface layer that
//                     lies inside the data bounds, any voxel not fully opaque (an AND / OR, order-free);
//   k_derive_trace    one thread per ray: the ray's EvalTrace as VoxSum terms, stored at the pixel's iproduct! position;
//   k_derive_reduce   one thread per (block, face) sums that face's terms one after another, in iproduct! order (f32
//                     addition is not associative: a tree would round differently); then one thread per block adds
//                     the six face sums in Face::ALL order and forms the colours, emission, opaque bits and visible.
//
// The library is compiled without contraction (-fmad=false): every a * b + c below is a rounded multiply and a rounded
// add, as Rust computes them.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "internal.h"

using namespace aicb;

namespace {

// A block that is not a single voxel, as the kernels see it.  Its rays are numbered face by face in Face::ALL order;
// within a face by the pixel's position in iproduct!(v, u).
struct DeriveRec {
    uint64_t vox_off;       // its first index in the index pool
    uint64_t ray_off;       // its first ray
    uint32_t pal_off;       // its first palette entry
    uint32_t res;
    uint32_t lo[3], sz[3];  // the data bounds (inside [0, res)^3)
    uint32_t opaque_cand;   // bit f: the surface layer of face f lies inside the data bounds (full_block_bounds.abut)
    uint32_t _pad;
};

// What one palette entry adds to a ray that reaches it with transmittance T: light += light * T, emission += emission
// * T, T *= transmittance; and its opacity category.
const uint32_t PAL_VISIBLE = 1, PAL_OPAQUE = 2;

const float OPAQUE_BELOW = 1.0f / 256.0f;   // ColorBuf::opaque (raytracer_components.rs:104-109)

const unsigned THREADS = 256;
const unsigned REDUCE_BLOCKS = 32;           // derived blocks per k_derive_reduce thread block, six threads each

// The last record whose `field` offset is <= i: the record holding element i (records with no elements share the next
// one's offset and are skipped).
template <uint64_t DeriveRec::*field>
__device__ __forceinline__ uint32_t rec_of(const DeriveRec *recs, uint32_t n, uint64_t i) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (recs[mid].*field <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// apply_transmittance (raytracer_components.rs:215-258) at thickness 1 / res, then ColorBuf::from (:150-163) and
// Rgb * f32 (color.rs:912-924).
__global__ void __launch_bounds__(THREADS) k_derive_palette(const DeriveRec *recs, uint32_t n_recs, const uint32_t *pal_rec,
                                                            const aicb_voxel *palette, uint32_t n_pal, float4 *terms) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_pal; p += gridDim.x * blockDim.x) {
        const aicb_voxel v = palette[p];
        const float thickness = 1.0f / (float)recs[pal_rec[p]].res;   // a power of two: exact
        const float unit_t = 1.0f - v.rgba[3];
        const float depth_t = powf_exact(unit_t, thickness);
        const float alpha = zo_clamped(1.0f - depth_t);
        const float c = (unit_t == 1.0f) ? thickness : (depth_t - 1.0f) / (unit_t - 1.0f);
        const float k = ps_clamped(fmaxf(c, 0.0f));
        const bool visible = !(v.rgba[3] == 0.0f) ||
                             !(v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f);
        const uint32_t flags = (visible ? PAL_VISIBLE : 0u) | (v.rgba[3] == 1.0f ? PAL_OPAQUE : 0u);
        terms[2 * p] = make_float4(v.rgba[0] * alpha, v.rgba[1] * alpha, v.rgba[2] * alpha, 1.0f - alpha);
        terms[2 * p + 1] = make_float4(ps_mul(v.emission[0], k), ps_mul(v.emission[1], k), ps_mul(v.emission[2], k),
                                       __uint_as_float(flags));
    }
}

// Per block: bit 0 = visible, bit 1 + f = a voxel of face f's surface layer is not fully opaque.
__global__ void __launch_bounds__(THREADS) k_derive_scan(const DeriveRec *recs, uint32_t n_recs, const uint16_t *indices,
                                                         uint64_t n_vox, const float4 *pal_terms, uint32_t *flags) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vox; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = rec_of<&DeriveRec::vox_off>(recs, n_recs, i);
        const DeriveRec &R = recs[r];
        const uint32_t pal = __float_as_uint(pal_terms[2 * (R.pal_off + indices[i]) + 1].w);
        uint32_t bits = (pal & PAL_VISIBLE) ? 1u : 0u;
        if (R.opaque_cand && !(pal & PAL_OPAQUE)) {
            const uint64_t k = i - R.vox_off;   // Z-major: ((x * sy) + y) * sz + z
            const uint32_t z = (uint32_t)(k % R.sz[2]), y = (uint32_t)(k / R.sz[2] % R.sz[1]),
                           x = (uint32_t)(k / R.sz[2] / R.sz[1]);
            const uint32_t c[3] = {R.lo[0] + x, R.lo[1] + y, R.lo[2] + z};
            for (int f = 0; f < 6; f++)
                if (c[f % 3] == (f < 3 ? 0u : R.res - 1)) bits |= 2u << f;
            bits &= 1u | (R.opaque_cand << 1);
        }
        // most voxels find their bits set already: read before the atomic
        if (bits & ~*(volatile uint32_t *)&flags[r]) atomicOr(&flags[r], bits);
    }
}

// The ray of face f and lane j: its first voxel (an index relative to the block's first), the index step, its length,
// and its pixel's position in iproduct!(v, u).  face.face_transform(res) maps (u, v, depth) to the block as
// Face::rotation_from_nz (face.rs:395-405) and a translation to the positive octant; in the block's axes:
//   NX: u = +y, v = +z     NY: u = +z, v = +x     NZ: u = +x, v = +y
//   PX: u = -y, v = +z     PY: u = +z, v = -x     PZ: u = +x, v = -y
// and each ray starts at the data layer nearest the face and runs inwards (face.opposite()).  Lanes run along z on the
// X and Y faces (the brick is Z-major, so neighbouring lanes read neighbouring voxels) and along y on the Z faces.
struct FaceRay {
    uint64_t first;
    int64_t step;
    uint32_t len;
    uint64_t pos;
};
__device__ __forceinline__ FaceRay face_ray(const DeriveRec &R, int f, uint64_t j) {
    const uint64_t sx = R.sz[0], sy = R.sz[1], sz = R.sz[2];
    const bool pos_face = f >= 3;
    FaceRay o;
    uint64_t x = 0, y = 0, z = 0;
    switch (f % 3) {
    case 0:   // X faces: j = y * sz + z
        y = j / sz; z = j % sz;
        x = pos_face ? sx - 1 : 0;
        o.step = pos_face ? -(int64_t)(sy * sz) : (int64_t)(sy * sz);
        o.len = (uint32_t)sx;
        o.pos = z * sy + (pos_face ? sy - 1 - y : y);
        break;
    case 1:   // Y faces: j = x * sz + z
        x = j / sz; z = j % sz;
        y = pos_face ? sy - 1 : 0;
        o.step = pos_face ? -(int64_t)sz : (int64_t)sz;
        o.len = (uint32_t)sy;
        o.pos = (pos_face ? sx - 1 - x : x) * sz + z;
        break;
    default:  // Z faces: j = x * sy + y
        x = j / sy; y = j % sy;
        z = pos_face ? sz - 1 : 0;
        o.step = pos_face ? -1 : 1;
        o.len = (uint32_t)sz;
        o.pos = (pos_face ? sy - 1 - y : y) * sx + x;
        break;
    }
    o.first = (x * sy + y) * sz + z;
    return o;
}

__device__ __forceinline__ uint64_t face_rays(const DeriveRec &R, int f) {
    const uint32_t a = (f % 3 + 1) % 3, b = (f % 3 + 2) % 3;
    return (uint64_t)R.sz[a] * R.sz[b];
}

// trace_for_eval, then Rgba::from(ColorBuf) (raytracer_components.rs:122-146) and the terms VoxSum += EvalTrace adds
// (derived.rs:267-276): rgb * alpha, alpha, emission.
__global__ void __launch_bounds__(THREADS) k_derive_trace(const DeriveRec *recs, uint32_t n_recs, const uint16_t *indices,
                                                          const float4 *pal_terms, uint64_t n_rays, float4 *terms) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rays; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = rec_of<&DeriveRec::ray_off>(recs, n_recs, i);
        const DeriveRec &R = recs[r];
        uint64_t j = i - R.ray_off, face_off = 0;
        int f = 0;
        for (; f < 5; f++) {
            const uint64_t n = face_rays(R, f);
            if (j < n) break;
            j -= n;
            face_off += n;
        }
        const FaceRay ray = face_ray(R, f, j);
        const uint16_t *idx = indices + R.vox_off;
        const float4 *pal = pal_terms + 2 * (size_t)R.pal_off;
        float T = 1.0f, l0 = 0.0f, l1 = 0.0f, l2 = 0.0f, e0 = 0.0f, e1 = 0.0f, e2 = 0.0f;
        int64_t v = (int64_t)ray.first;
        for (uint32_t k = 0; k < ray.len; k++, v += ray.step) {
            const uint32_t p = idx[v];
            const float4 a = pal[2 * p], b = pal[2 * p + 1];
            e0 = e0 + b.x * T;
            e1 = e1 + b.y * T;
            e2 = e2 + b.z * T;
            l0 = l0 + a.x * T;
            l1 = l1 + a.y * T;
            l2 = l2 + a.z * T;
            T = T * a.w;
            if (T < OPAQUE_BELOW) break;
        }
        float c0 = 0.0f, c1 = 0.0f, c2 = 0.0f, alpha = 0.0f;
        if (!(T >= 1.0f)) {
            const float ca = 1.0f - T;
            c0 = l0 / ca;
            c1 = l1 / ca;
            c2 = l2 / ca;
            // Rgb::try_from: a component that is negative or NaN makes the colour red; -0 becomes +0
            if (!((c0 > 0.0f || c0 == 0.0f) && (c1 > 0.0f || c1 == 0.0f) && (c2 > 0.0f || c2 == 0.0f))) {
                c0 = 1.0f; c1 = 0.0f; c2 = 0.0f;
            } else {
                c0 = c0 == 0.0f ? 0.0f : c0;
                c1 = c1 == 0.0f ? 0.0f : c1;
                c2 = c2 == 0.0f ? 0.0f : c2;
            }
            alpha = (ca > 0.0f && ca <= 1.0f) ? ca : (ca == 0.0f ? 0.0f : 1.0f);   // ZeroOne::try_from(..).unwrap_or(1)
        }
        float4 *out = terms + 2 * (R.ray_off + face_off + ray.pos);
        out[0] = make_float4(c0 * alpha, c1 * alpha, c2 * alpha, alpha);
        out[1] = make_float4(e0, e1, e2, 0.0f);
    }
}

// Rgb::try_from(v) (color.rs:849-858): false for a negative or NaN component, whose expect() panics; -0 becomes +0.
__device__ __forceinline__ bool rgb_try_from(float &v) {
    if (v > 0.0f) return true;
    if (v == 0.0f) {
        v = 0.0f;
        return true;
    }
    return false;
}

// VoxSum::color (derived.rs:235-254) into out[4]; false where it panics.
__device__ __forceinline__ bool voxsum_color(const float s[7], float area, float out[4]) {
    if (!(s[3] > 0.0f)) {
        out[0] = out[1] = out[2] = out[3] = 0.0f;
        return true;
    }
    bool ok = true;
    for (int c = 0; c < 3; c++) {
        out[c] = s[c] / s[3];
        ok &= rgb_try_from(out[c]);
    }
    out[3] = zo_clamped(s[3] / area);
    return ok;
}

__global__ void __launch_bounds__(REDUCE_BLOCKS * 6) k_derive_reduce(const DeriveRec *recs, uint32_t n_recs,
                                                                     const float4 *terms, const uint32_t *flags,
                                                                     aicb_block_light *out, uint32_t *err) {
    __shared__ float face_sum[REDUCE_BLOCKS][6][7];
    __shared__ uint32_t face_err[REDUCE_BLOCKS];
    const uint32_t lb = threadIdx.x / 6, f = threadIdx.x % 6;
    const uint32_t r = blockIdx.x * REDUCE_BLOCKS + lb;
    if (f == 0) face_err[lb] = 0;
    __syncthreads();
    float s[7] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    const DeriveRec *R = r < n_recs ? &recs[r] : nullptr;
    if (R) {
        uint64_t off = R->ray_off;
        for (uint32_t g = 0; g < f; g++) off += face_rays(*R, g);
        const uint64_t n = face_rays(*R, f);
        const float4 *t = terms + 2 * off;
#pragma unroll 8
        for (uint64_t k = 0; k < n; k++) {
            const float4 a = t[2 * k], b = t[2 * k + 1];
            s[0] = s[0] + a.x;
            s[1] = s[1] + a.y;
            s[2] = s[2] + a.z;
            s[3] = s[3] + a.w;
            s[4] = s[4] + b.x;
            s[5] = s[5] + b.y;
            s[6] = s[6] + b.z;
        }
        float col[4];
        if (!voxsum_color(s, (float)(R->res * R->res), col)) atomicOr(&face_err[lb], 1u);
        for (int c = 0; c < 4; c++) out[r].face_colors[f][c] = col[c];
        for (int c = 0; c < 7; c++) face_sum[lb][f][c] = s[c];
    }
    __syncthreads();
    if (!R || f != 0) return;
    // all_faces_sum += face_sum in Face::ALL order (derived.rs:136), then color / emission of the whole surface
    float all[7] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    uint64_t count = 0;
    for (int g = 0; g < 6; g++) {
        for (int c = 0; c < 7; c++) all[c] = all[c] + face_sum[lb][g][c];
        count += face_rays(*R, g);
    }
    const float area = (float)(6 * R->res * R->res);   // surface_area_f64() as f32: exact
    bool ok = face_err[lb] == 0;
    float col[4];
    ok &= voxsum_color(all, area, col);
    aicb_block_light &o = out[r];
    for (int c = 0; c < 4; c++) o.color[c] = col[c];
    for (int c = 0; c < 3; c++) {   // VoxSum::emission (derived.rs:256-265)
        float e = count == 0 ? 0.0f : all[4 + c] / area;
        ok &= rgb_try_from(e);
        o.emission[c] = e;
    }
    o.opaque_faces = (uint8_t)(R->opaque_cand & ~(flags[r] >> 1) & 0x3f);
    o.visible = (uint8_t)(flags[r] & 1);
    o._pad[0] = o._pad[1] = 0;
    err[r] = ok ? 0u : 1u;
}

unsigned grid_for(uint64_t n, int num_sms) {
    const uint64_t want = (n + THREADS - 1) / THREADS;
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, (uint64_t)num_sms * 32));
}

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// compute_derived of a single voxel (derived.rs:84-104)
aicb_block_light single_light(const aicb_voxel &v) {
    aicb_block_light o;
    std::memset(&o, 0, sizeof o);
    for (int f = 0; f < 6; f++) std::memcpy(o.face_colors[f], v.rgba, sizeof v.rgba);
    std::memcpy(o.color, v.rgba, sizeof v.rgba);
    std::memcpy(o.emission, v.emission, sizeof v.emission);
    o.opaque_faces = v.rgba[3] == 1.0f ? 0x3f : 0;
    const bool emits = !(v.emission[0] == 0.0f && v.emission[1] == 0.0f && v.emission[2] == 0.0f);
    o.visible = (!(v.rgba[3] == 0.0f) || emits) ? 1 : 0;
    return o;
}

// compute_derived of n validated blocks: into `out` (host memory), or with on_device (the blocks' voxels in the
// context's device memory, copied device to device into the kernels' inputs) left in d_derive, each block's record
// in *rec (LIGHT_SINGLE: a single voxel, which the caller derives from its voxel) and the records at *d_out.
aicb_status derive(aicb_ctx *ctx, const aicb_block_desc *descs, size_t n, aicb_block_light *out, bool on_device = false,
                   std::vector<int32_t> *rec = nullptr, const aicb_block_light **d_out_ptr = nullptr) {
    std::vector<aicb_block_light> result(on_device ? 0 : n);
    if (on_device) rec->assign(n, LIGHT_SINGLE);
    std::vector<DeriveRec> recs;
    std::vector<size_t> rec_block;   // per record: its position in descs
    uint64_t n_vox = 0, n_rays = 0;
    uint32_t n_pal = 0;
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        if (is_single_voxel(b)) {
            if (!on_device) result[i] = single_light(single_voxel_of(b));
            continue;
        }
        if (on_device) (*rec)[i] = (int32_t)recs.size();
        DeriveRec R;
        std::memset(&R, 0, sizeof R);
        R.vox_off = n_vox;
        R.ray_off = n_rays;
        R.pal_off = n_pal;
        R.res = b.resolution;
        for (int a = 0; a < 3; a++) {
            R.lo[a] = (uint32_t)b.voxel_bounds.lower[a];
            R.sz[a] = b.voxel_bounds.size[a];
        }
        // full_block_bounds.abut(face, -1) inside the data bounds (derived.rs:199-205)
        const bool spans[3] = {R.lo[0] == 0 && R.sz[0] == R.res, R.lo[1] == 0 && R.sz[1] == R.res,
                               R.lo[2] == 0 && R.sz[2] == R.res};
        for (int f = 0; f < 6; f++) {
            const int a = f % 3;
            const bool touches = R.sz[a] > 0 && (f < 3 ? R.lo[a] == 0 : R.lo[a] + R.sz[a] == R.res);
            if (touches && spans[(a + 1) % 3] && spans[(a + 2) % 3]) R.opaque_cand |= 1u << f;
        }
        n_vox += b.n_indices;
        n_rays += 2 * ((uint64_t)R.sz[0] * R.sz[1] + (uint64_t)R.sz[1] * R.sz[2] + (uint64_t)R.sz[0] * R.sz[2]);
        if ((uint64_t)n_pal + b.n_palette > 0xffffffffull) return aicb_fail(AICB_ERR_INVALID, "palettes exceed 2^32 entries");
        n_pal += (uint32_t)b.n_palette;
        recs.push_back(R);
        rec_block.push_back(i);
    }
    if (!recs.empty()) {
        const uint32_t n_recs = (uint32_t)recs.size();
        const cudaStream_t stream = ctx->stream.get();
        // upload: records, each palette entry's record, palettes, indices
        const size_t up_recs = 0, up_pal_rec = align16(n_recs * sizeof(DeriveRec));
        const size_t up_pal = up_pal_rec + align16((size_t)n_pal * 4), up_idx = up_pal + (size_t)n_pal * sizeof(aicb_voxel);
        const size_t up_bytes = up_idx + align16(n_vox * 2);
        TRY(delta_room(ctx, up_bytes));
        char *h = ctx->h_delta.get<char>();
        std::memcpy(h + up_recs, recs.data(), n_recs * sizeof(DeriveRec));
        uint32_t *h_pal_rec = (uint32_t *)(h + up_pal_rec);
        for (uint32_t r = 0; r < n_recs; r++) {
            const aicb_block_desc &b = descs[rec_block[r]];
            std::fill(h_pal_rec + recs[r].pal_off, h_pal_rec + recs[r].pal_off + b.n_palette, r);
            if (on_device) continue;
            if (b.n_palette) std::memcpy(h + up_pal + recs[r].pal_off * sizeof(aicb_voxel), b.palette, b.n_palette * sizeof(aicb_voxel));
            if (b.n_indices) std::memcpy(h + up_idx + recs[r].vox_off * 2, b.indices, b.n_indices * 2);
        }
        char *d = ctx->d_delta.get<char>();
        CU(cudaMemcpyAsync(d, h, on_device ? up_pal : up_bytes, cudaMemcpyHostToDevice, stream));
        for (uint32_t r = 0; on_device && r < n_recs; r++) {
            const aicb_block_desc &b = descs[rec_block[r]];
            if (b.n_palette)
                CU(cudaMemcpyAsync(d + up_pal + recs[r].pal_off * sizeof(aicb_voxel), b.palette,
                                   b.n_palette * sizeof(aicb_voxel), cudaMemcpyDeviceToDevice, stream));
            if (b.n_indices)
                CU(cudaMemcpyAsync(d + up_idx + recs[r].vox_off * 2, b.indices, b.n_indices * 2,
                                   cudaMemcpyDeviceToDevice, stream));
        }
        CU(cudaEventRecord(ctx->ev_delta.get(), stream));
        // scratch: palette terms, ray terms, per-record flags and errors, results
        const size_t s_pal = 0, s_rays = align16((size_t)n_pal * 32), s_flags = s_rays + n_rays * 32;
        const size_t s_err = s_flags + align16(n_recs * 4), s_out = s_err + align16(n_recs * 4);
        const size_t s_bytes = s_out + (size_t)n_recs * sizeof(aicb_block_light);
        TRY(ctx->d_derive.ensure(s_bytes));
        char *s = ctx->d_derive.get<char>();
        CU(cudaMemsetAsync(s + s_flags, 0, n_recs * 4, stream));
        const DeriveRec *d_recs = (const DeriveRec *)(d + up_recs);
        const uint16_t *d_idx = (const uint16_t *)(d + up_idx);
        float4 *pal_terms = (float4 *)(s + s_pal), *ray_terms = (float4 *)(s + s_rays);
        uint32_t *flags = (uint32_t *)(s + s_flags), *err = (uint32_t *)(s + s_err);
        aicb_block_light *d_out = (aicb_block_light *)(s + s_out);
        if (n_pal) {
            k_derive_palette<<<grid_for(n_pal, ctx->num_sms), THREADS, 0, stream>>>(
                d_recs, n_recs, (const uint32_t *)(d + up_pal_rec), (const aicb_voxel *)(d + up_pal), n_pal, pal_terms);
            CU(cudaGetLastError());
        }
        if (n_vox) {
            k_derive_scan<<<grid_for(n_vox, ctx->num_sms), THREADS, 0, stream>>>(d_recs, n_recs, d_idx, n_vox, pal_terms, flags);
            CU(cudaGetLastError());
        }
        if (n_rays) {
            k_derive_trace<<<grid_for(n_rays, ctx->num_sms), THREADS, 0, stream>>>(d_recs, n_recs, d_idx, pal_terms, n_rays,
                                                                                  ray_terms);
            CU(cudaGetLastError());
        }
        k_derive_reduce<<<(n_recs + REDUCE_BLOCKS - 1) / REDUCE_BLOCKS, REDUCE_BLOCKS * 6, 0, stream>>>(
            d_recs, n_recs, ray_terms, flags, d_out, err);
        CU(cudaGetLastError());
        std::vector<aicb_block_light> lights(on_device ? 0 : n_recs);
        std::vector<uint32_t> errs(n_recs);
        if (on_device) *d_out_ptr = d_out;
        else CU(cudaMemcpyAsync(lights.data(), d_out, n_recs * sizeof(aicb_block_light), cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpyAsync(errs.data(), err, n_recs * 4, cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        for (uint32_t r = 0; r < n_recs; r++) {
            if (errs[r])
                return aicb_fail(AICB_ERR_INVALID, "block " + std::to_string(rec_block[r]) +
                                                       ": its colour or emission sum is NaN or negative, where "
                                                       "compute_derived's Rgb::try_from(..).expect(..) panics");
            if (!on_device) result[rec_block[r]] = lights[r];
        }
    }
    if (!on_device) std::memcpy(out, result.data(), n * sizeof(aicb_block_light));
    return AICB_OK;
}

}  // namespace

aicb_status derive_on_device(aicb_ctx *ctx, const aicb_block_desc *descs, size_t n, std::vector<int32_t> *rec,
                             const aicb_block_light **out) {
    *out = nullptr;
    return derive(ctx, descs, n, nullptr, true, rec, out);
}

extern "C" aicb_status aicb_derive_block_light(aicb_ctx *ctx, const aicb_block_desc *descs, size_t n,
                                               aicb_block_light *out) {
    if (!ctx) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n == 0) return AICB_OK;
    if (!descs || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    for (size_t i = 0; i < n; i++) {
        const aicb_status st = check_block_desc(descs[i]);
        if (st != AICB_OK) return aicb_fail(st, "block " + std::to_string(i) + ": " + aicb_last_error());
    }
    std::lock_guard<std::mutex> lock(ctx->mu);
    CU(cudaSetDevice(ctx->device));
    return derive(ctx, descs, n, out);
}
