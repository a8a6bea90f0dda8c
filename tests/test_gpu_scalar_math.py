"""The device's scalar leaf functions against the oracle over whole input domains.

The frame tests only ever feed these functions the few million values their images produce; each of the functions
below replaces the reference's formula with something faster that is argued, not shown, to be exact:
- component_to_srgb8 and scalar_in_t search the host-built threshold tables (host_tables.h) instead of calling powf
  / log2f: every f32 bit pattern, against the direct formulas;
- f16x2_texel, __floats2half2_rn for the rgba16f and texture texels: every f32 bit pattern, against half::f16::from_f32;
- powf_exact / expf_exact and their double-double fallbacks powf_libm / expf_libm: dense sweeps, against the oracle's
  LIBM_CR mode (the same header on the host), and wherever that differs from glibc's f64 pow / exp rounded to f32, a
  60-digit evaluation says which is nearer;
- div_known_recip (ray generation, project_ndc, caster_begin, scale_to_integer_step): the pixel quotients, random
  pairs over its exponent window and beyond, project_ndc's three quotients by one w, against IEEE division;
- scale_to_integer_step, rem_euclid1 and the ColorBuf -> sRGB8 encoding on their edge cases.

A CUDA driver is compiled with the library's own flags (__graft_entry__.NVCC_FLAGS, -fmad=false included) and
includes the library's headers, so it runs the library's code.  It evaluates each check on the device in chunks and
compares on every host thread; each check prints one JSON line (count, mismatches, first mismatching input).

test_host_threshold_search is the host half of the threshold premise and needs no GPU: the tables the library
builds, searched as the device searches them, equal the direct formulas on all 2^32 f32 bit patterns on the host
that builds them."""
import json
import os
import struct
import subprocess
from decimal import Context, Decimal

import pytest

import __graft_entry__ as g

ROOT = g.ROOT
CSRC = os.path.join(g.PKG, "csrc")
ORACLE_LIB = g.ORACLE_LIB
TEXTURE_LIB = os.path.join(ROOT, "oracle_texture", "libtexorc.so")

COMMON = r"""
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

static uint32_t fbits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static float ffrom(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

// Runs f(i, part) for i in [0, n) on every host thread; part is the thread's own accumulator.
template <class P, class F> static P parallel(uint64_t n, F f) {
    const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
    std::vector<P> part(nt);
    std::vector<std::thread> th;
    for (unsigned w = 0; w < nt; w++)
        th.emplace_back([&, w] {
            const uint64_t lo = n * w / nt, hi = n * (w + 1) / nt;
            for (uint64_t i = lo; i < hi; i++) f(i, part[w]);
        });
    for (auto &t : th) t.join();
    P all;
    for (auto &p : part) all.add(p);
    return all;
}

struct Tally {
    uint64_t n = 0, mismatch[2] = {0, 0}, first[2] = {UINT64_MAX, UINT64_MAX};
    void bad(int v, uint64_t i) { mismatch[v]++; first[v] = std::min(first[v], i); }
    void add(const Tally &o) {
        n += o.n;
        for (int v = 0; v < 2; v++) { mismatch[v] += o.mismatch[v]; first[v] = std::min(first[v], o.first[v]); }
    }
};
"""

HOST_DRIVER = COMMON + r"""
#include "host_tables.h"
using namespace aicb;

// The device's 8-step search (trace_kernel.cuh component_to_srgb8, light_kernel.cuh scalar_in_t) over thr[1..255]
static unsigned search(const float *thr, float c) {
    int lo = 0, hi = 255;
    for (int i = 0; i < 8; i++) {
        const int mid = (lo + hi + 1) >> 1;
        if (c >= thr[mid]) lo = mid; else hi = mid - 1;
    }
    return (unsigned)lo;
}

int main() {
    float srgb[256], light[256];
    build_srgb_thresholds(srgb);
    build_light_thresholds(light);
    const Tally t = parallel<Tally>(1ull << 32, [&](uint64_t i, Tally &p) {
        const float c = ffrom((uint32_t)i);
        p.n++;
        if (search(srgb, c) != srgb8_host(c)) p.bad(0, i);
        if (search(light, c) != scalar_in(c)) p.bad(1, i);
    });
    std::printf("{\"n\": %llu, \"mismatch\": [%llu, %llu], \"first\": [\"0x%08llx\", \"0x%08llx\"]}\n",
                (unsigned long long)t.n, (unsigned long long)t.mismatch[0], (unsigned long long)t.mismatch[1],
                (unsigned long long)(t.first[0] & 0xffffffffu), (unsigned long long)(t.first[1] & 0xffffffffu));
    return 0;
}
"""

GPU_DRIVER = COMMON + r"""
#include <dlfcn.h>
#include <mutex>
#include <cuda_fp16.h>
#include "host_tables.h"
#include "light_kernel.cuh"   // trace_kernel.cuh and exact_math.cuh with it
using namespace aicb;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    std::fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); std::exit(3); } } while (0)

// ---- the oracle, loaded by name so that each reference says which library it comes from
static void *sym(const char *lib, const char *name) {
    void *h = dlopen(lib, RTLD_NOW | RTLD_LOCAL);
    void *s = h ? dlsym(h, name) : nullptr;
    if (!s) { std::fprintf(stderr, "%s: %s\n", name, dlerror()); std::exit(4); }
    return s;
}
static int (*orc_packed_light_scalar_in)(float);
static void (*orc_to_srgb8)(const float *, float, int, float, uint8_t *);
static float (*orc_powf)(float, float, int);
static float (*orc_expf)(float, int);
static double (*orc_scale_to_integer_step)(double, double);
static uint16_t (*orc_f16_from_f32)(float);
static const int LIBM_CR = 1;

// ---- inputs: every generator is __host__ __device__, so the device evaluates case i and the host recomputes the
// same inputs for its reference
#define HD __host__ __device__ __forceinline__
HD uint64_t mix64(uint64_t x) {   // splitmix64's finaliser
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
HD float f_of(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    return ffrom(u);
#endif
}
HD double d_of(uint64_t u) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)u);
#else
    double d; std::memcpy(&d, &u, 8); return d;
#endif
}
HD uint64_t d_bits(double d) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u; std::memcpy(&u, &d, 8); return u;
#endif
}
// sign * (1 + mant 2^-52) * 2^e for -1022 <= e <= 1023; below, the subnormal with the leading bits of that
// significand (truncated): built from bits, so host and device agree
HD double make_double(bool neg, int e, uint64_t mant) {
    mant &= 0xfffffffffffffull;
    uint64_t b;
    if (e >= -1022) b = ((uint64_t)(e + 1023) << 52) | mant;
    else b = e < -1074 ? 0 : (mant | (1ull << 52)) >> (-1022 - e);
    return d_of(b | (neg ? 1ull << 63 : 0));
}

// Arguments where the correctly rounded result (the oracle's LIBM_CR) and glibc's f64 pow / exp rounded to f32 differ:
// reported with both results, and checked in Python against a 60-digit evaluation
static std::mutex g_mu;
static uint64_t g_glibc_differs;
static std::string g_disputed;
static void dispute(float x, float y, float cr, float glibc) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (g_glibc_differs++ >= 1000) return;
    char s[96];
    std::snprintf(s, sizeof s, "%s[%u, %u, %u, %u]", g_disputed.empty() ? "" : ", ", fbits(x), fbits(y), fbits(cr),
                  fbits(glibc));
    g_disputed += s;
}

template <class C> __global__ void k_map(C c, uint64_t base, uint32_t m, typename C::Out *out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < m) out[t] = c.dev(c.gen(base + t));
}

// Case i of check c on the device, then c.check on every host thread: bit v of its result marks variant v wrong
template <class C> static void sweep(const char *name, const C &c, uint64_t n) {
    using Out = typename C::Out;
    const uint64_t CHUNK = (1ull << 28) / sizeof(Out);
    Out *d_out, *h_out;
    CK(cudaMalloc(&d_out, CHUNK * sizeof(Out)));
    CK(cudaMallocHost(&h_out, CHUNK * sizeof(Out)));
    Tally t;
    g_glibc_differs = 0;
    g_disputed.clear();
    for (uint64_t base = 0; base < n; base += CHUNK) {
        const uint32_t m = (uint32_t)std::min(CHUNK, n - base);
        k_map<<<(m + 255) / 256, 256>>>(c, base, m, d_out);
        CK(cudaGetLastError());
        CK(cudaMemcpy(h_out, d_out, m * sizeof(Out), cudaMemcpyDeviceToHost));
        t.add(parallel<Tally>(m, [&](uint64_t j, Tally &p) {
            p.n++;
            const int bad = c.check(c.gen(base + j), h_out[j]);
            for (int v = 0; v < 2; v++) if (bad >> v & 1) p.bad(v, base + j);
        }));
    }
    CK(cudaFree(d_out));
    CK(cudaFreeHost(h_out));
    std::string first[2];
    for (int v = 0; v < 2; v++) first[v] = t.mismatch[v] ? "\"" + c.show(c.gen(t.first[v])) + "\"" : "null";
    std::printf("{\"check\": \"%s\", \"n\": %llu, \"mismatch\": [%llu, %llu], \"first\": [%s, %s], "
                "\"glibc_differs\": %llu, \"disputed\": [%s]}\n", name, (unsigned long long)t.n,
                (unsigned long long)t.mismatch[0], (unsigned long long)t.mismatch[1], first[0].c_str(), first[1].c_str(),
                (unsigned long long)g_glibc_differs, g_disputed.c_str());
    std::fflush(stdout);
}

static std::string fmt(const char *f, double a, double b = 0, double c = 0, double d = 0) {
    char s[256];
    std::snprintf(s, sizeof s, f, a, b, c, d);
    return s;
}
static std::string fs(float x) {   // value and bit pattern
    char s[64];
    std::snprintf(s, sizeof s, "%.9g (0x%08x)", (double)x, fbits(x));
    return s;
}


// ---- the threshold encoders and the f16 conversion: every f32 bit pattern
struct SrgbCheck {
    const float *thr;   // device copy of the library's tables
    using Out = uint8_t;
    HD float gen(uint64_t i) const { return f_of((uint32_t)i); }
    __device__ Out dev(float c) const { return component_to_srgb8(thr + 256, c); }
    int check(float c, Out got) const {
        // the oracle's encoding of a ColorBuf {c, 0, 0, T = 0} with exposure 1 and no tone mapping is
        // component_to_srgb8(c) for every c >= 0 and +inf; below zero (and for NaN) Rgba::from(ColorBuf) takes over,
        // so those components are compared with the direct formula, which encodes them as 0
        uint8_t want;
        if (c >= 0.0f) {
            const float cb[4] = {c, 0.0f, 0.0f, 0.0f};
            uint8_t o[4];
            orc_to_srgb8(cb, 1.0f, AICB_TONE_CLAMP, INFINITY, o);
            want = o[0];
        } else {
            want = srgb8_host(c);
        }
        return got != want;
    }
    std::string show(float c) const { return "c = " + fs(c); }
};

struct LightCheck {
    const float *tables;
    using Out = uint8_t;
    HD float gen(uint64_t i) const { return f_of((uint32_t)i); }
    __device__ Out dev(float v) const { return (Out)aicb_light::scalar_in_t(tables, v); }
    int check(float v, Out got) const { return got != (Out)orc_packed_light_scalar_in(v); }
    std::string show(float v) const { return "v = " + fs(v); }
};

// finish_pixel's texel store f16x2_texel(x, y) (__floats2half2_rn), here (x, -x), both halves against
// half::f16::from_f32.  NaN inputs
// are compared by NaN-ness only: the payload and sign of a NaN differ between x86 and the GPU, and neither the
// reference nor any consumer of a texel gives them meaning.
struct F16Check {
    struct Out { uint16_t lo, hi; };
    HD float gen(uint64_t i) const { return f_of((uint32_t)i); }
    __device__ Out dev(float x) const {
        const uint32_t h = f16x2_texel(x, -x);
        return Out{(uint16_t)h, (uint16_t)(h >> 16)};
    }
    static bool same(float x, uint16_t got) {
        const uint16_t want = orc_f16_from_f32(x);
        if (x != x) return (got & 0x7c00u) == 0x7c00u && (got & 0x3ffu) != 0;
        return got == want;
    }
    int check(float x, Out got) const { return !(same(x, got.lo) && same(-x, got.hi)); }
    std::string show(float x) const { return "x = " + fs(x); }
};

// ---- pow and exp, against the oracle's LIBM_CR (the same header, compiled for the host): variant 0 is the short path
// with its fallback, variant 1 the fallback alone
struct PowOut { float exact, libm; };
template <class G> struct PowCheck {
    G g;
    using Out = PowOut;
    HD float2 gen(uint64_t i) const { return g(i); }
    __device__ Out dev(float2 a) const { return Out{powf_exact(a.x, a.y), powf_libm(a.x, a.y)}; }
    int check(float2 a, Out got) const {
        const float want = orc_powf(a.x, a.y, LIBM_CR), glibc = (float)std::pow((double)a.x, (double)a.y);
        if (fbits(want) != fbits(glibc)) dispute(a.x, a.y, want, glibc);
        return (fbits(got.exact) != fbits(want)) | (fbits(got.libm) != fbits(want)) << 1;
    }
    std::string show(float2 a) const { return "u = " + fs(a.x) + ", th = " + fs(a.y); }
};
template <class G> static PowCheck<G> pow_check(G g) { return PowCheck<G>{g}; }

struct PowAllU {   // every f32 u in (0, 1) at one thickness
    float th;
    HD float2 operator()(uint64_t i) const { return make_float2(f_of((uint32_t)i + 1u), th); }
};
struct PowGrid {   // thickness k / 16 for k = 1..256, u in (0, 1) every `stride` bit patterns, at a phase set by k
    uint32_t stride, per;
    HD float2 operator()(uint64_t i) const {
        const uint32_t k = (uint32_t)(i / per) + 1u, j = (uint32_t)(i % per);
        return make_float2(f_of(1u + j * stride + (k * 2654435761u) % stride), (float)k / 16.0f);
    }
};
struct PowRandom {   // u in (0, 1); th half log-uniform over [2^-20, 2^10), half any positive finite f32
    HD float2 operator()(uint64_t i) const {
        const uint64_t h = mix64(i), h2 = mix64(i ^ 0x5bd1e995u);
        const float u = f_of(1u + (uint32_t)((h >> 32) % 0x3f7fffffu));
        const uint32_t tb = (i & 1) ? ((uint32_t)(107 + (h2 >> 32) % 30) << 23) | ((uint32_t)h2 & 0x7fffffu)
                                    : 1u + (uint32_t)((h2 >> 32) % 0x7f7fffffu);
        return make_float2(u, f_of(tb));
    }
};

struct ExpOut { float exact, libm; };
template <class G> struct ExpCheck {
    G g;
    using Out = ExpOut;
    HD float gen(uint64_t i) const { return g(i); }
    __device__ Out dev(float x) const { return Out{expf_exact(x), expf_libm(x)}; }
    int check(float x, Out got) const {
        const float want = orc_expf(x, LIBM_CR), glibc = (float)std::exp((double)x);
        if (fbits(want) != fbits(glibc) && want == want) dispute(x, 0.0f, want, glibc);
        return (fbits(got.exact) != fbits(want)) | (fbits(got.libm) != fbits(want)) << 1;
    }
    std::string show(float x) const { return "x = " + fs(x); }
};
template <class G> static ExpCheck<G> exp_check(G g) { return ExpCheck<G>{g}; }

struct ExpFog {    // every f32 in [-1.6, 0]: -0 .. -1.6f by bit pattern, then +0
    uint32_t count;
    HD float operator()(uint64_t i) const { return i + 1 == count ? 0.0f : f_of(0x80000000u + (uint32_t)i); }
};
struct ExpWide {   // every `stride`-th f32 of [-104, 89]: +0 .. 89 by bit pattern, then -0 .. -104
    uint32_t stride, npos;
    HD float operator()(uint64_t i) const {
        return i < npos ? f_of((uint32_t)(i * stride)) : f_of(0x80000000u + (uint32_t)((i - npos) * stride));
    }
};

// ---- div_known_recip(a, b, RN(1 / b)) against a / b, both on the device
struct DivOut { double got, want; };
template <class G> struct DivCheck {
    G g;
    using Out = DivOut;
    HD double2 gen(uint64_t i) const { return g(i); }
    __device__ Out dev(double2 ab) const { return Out{div_known_recip(ab.x, ab.y, 1.0 / ab.y), ab.x / ab.y}; }
    int check(double2, Out o) const { return d_bits(o.got) != d_bits(o.want); }
    std::string show(double2 ab) const { return fmt("a = %a, b = %a", ab.x, ab.y); }
};
template <class G> static DivCheck<G> div_check(G g) { return DivCheck<G>{g}; }

HD uint64_t tri(uint64_t w) { return (w - 1) * (w + 2) / 2; }   // pixel quotients before width w
struct DivPixels {   // x / W for every W in 1..16384 and every x in 0..W
    HD double2 operator()(uint64_t i) const {
        uint64_t w = (uint64_t)((sqrt(8.0 * (double)i + 9.0) - 1.0) / 2.0);
        while (tri(w + 1) <= i) w++;
        while (tri(w) > i) w--;
        return make_double2((double)(i - tri(w)), (double)w);
    }
};
struct DivRandom {
    // b's exponent over [-420, 420] and a's over [-1074, 210] (subnormal a included), random signs and significands;
    // a quarter of the cases sit on either side of the window's bounds on |b| (2^+-400) and |a| (2^200, 2^-600), and a
    // quarter have quotients from 2^-1080 to 2^-1000, across the bottom of the normal range
    HD double2 operator()(uint64_t i) const {
        const uint64_t h0 = mix64(i), h1 = mix64(h0), h2 = mix64(h1);
        int eb = -420 + (int)(h2 % 841), ea = -1074 + (int)((h2 >> 16) % 1285);
        switch ((h2 >> 40) & 7) {
        case 4: eb = ((h2 >> 48) & 1 ? 400 : -401) + (int)((h2 >> 50) % 2); break;
        case 5: ea = 199 + (int)((h2 >> 48) % 3); break;
        case 6: ea = -601 + (int)((h2 >> 48) % 3); break;
        case 7: ea = eb - 1080 + (int)((h2 >> 48) % 81); break;
        default: break;
        }
        ea = ea < -1074 ? -1074 : (ea > 210 ? 210 : ea);
        // one case in 16 has an exact power of two for b
        const uint64_t mb = ((h2 >> 56) & 15) == 0 ? 0 : h1;
        return make_double2(make_double(h0 >> 63, ea, h0), make_double(h1 >> 63, eb, mb));
    }
};

// project_ndc's shape: three numerators over one w > 0 and one RN(1 / w)
struct NdcOut { double got[3], want[3]; };
struct NdcCheck {
    using Out = NdcOut;
    struct In { double h[4]; };
    HD In gen(uint64_t i) const {
        const uint64_t hw = mix64(i), hx = mix64(hw);
        In in;
        // w: mostly a homogeneous coordinate of a camera (2^-30 .. 2^30), one case in 8 anywhere in the window
        const int ew = ((hw >> 60) == 0) ? -420 + (int)(hw % 841) : -30 + (int)(hw % 61);
        in.h[3] = make_double(false, ew, hw >> 4);
        for (int k = 0; k < 3; k++) {
            const uint64_t h = mix64(hx + k);
            const int kind = (int)(h >> 60);
            if (kind == 0) in.h[k] = (h & 1) ? -0.0 : 0.0;                                   // a zero, either sign
            else if (kind == 1) in.h[k] = make_double(h & 1, -1074 + (int)(h % 500), h >> 8);  // tiny
            else in.h[k] = make_double(h & 1, ew - 8 + (int)((h >> 8) % 12), h >> 12);      // ~ w * [2^-8, 2^3]
        }
        return in;
    }
    __device__ Out dev(In in) const {
        const double rw = 1.0 / in.h[3];
        Out o;
        for (int k = 0; k < 3; k++) { o.got[k] = div_known_recip(in.h[k], in.h[3], rw); o.want[k] = in.h[k] / in.h[3]; }
        return o;
    }
    int check(In, Out o) const {
        int bad = 0;
        for (int k = 0; k < 3; k++) bad |= d_bits(o.got[k]) != d_bits(o.want[k]);
        return bad;
    }
    std::string show(In in) const { return fmt("(%a, %a, %a) / %a", in.h[0], in.h[1], in.h[2], in.h[3]); }
};

// ---- list checks: the inputs are a host vector with a device copy
template <class T> struct List {
    const T *h = nullptr, *d = nullptr;
    HD T operator[](uint64_t i) const {
#ifdef __CUDA_ARCH__
        return d[i];
#else
        return h[i];
#endif
    }
};
template <class T> static List<T> upload(const std::vector<T> &v) {
    T *d;
    CK(cudaMalloc(&d, v.size() * sizeof(T)));
    CK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return List<T>{v.data(), d};
}

// Equal bits, or both NaN: a NaN's sign and payload differ between x86 and the GPU and mean nothing here
static bool same_f64(double got, double want) { return want != want ? got != got : d_bits(got) == d_bits(want); }

// values of s around the integers: integers, +-0, integer +- k ulp, 2^52 .. 2^53, huge, NaN, inf; both signs
static std::vector<double> integer_edges() {
    std::vector<double> v;
    const double ints[] = {0.0, 1.0, 2.0, 3.0, 7.0, 100.0, 4095.0, 65536.0, 1e6, 0x1p31, 0x1p40, 0x1p51,
                           0x1p52 - 1, 0x1p52, 0x1p52 + 1, 0x1p53 - 1, 0x1p53, 0x1p53 + 2, 0x1p60, 1e300};
    for (double x : ints)
        for (int k = -3; k <= 3; k++) {
            double y = x;
            for (int s = 0; s < (k < 0 ? -k : k); s++) y = std::nextafter(y, k < 0 ? -INFINITY : INFINITY);
            v.push_back(y);
            v.push_back(-y);
        }
    const double more[] = {0.5, 0.25, 1.5, 0x1p-30, 0x1p-1074, 0x1p-1022, 0.1, 0.9, 12.375, 1e-300, DBL_MAX,
                           INFINITY, NAN};
    for (double x : more) { v.push_back(x); v.push_back(-x); }
    return v;
}

struct StepCheck {   // scale_to_integer_step(s, ds) for every (s, ds) of the two lists
    List<double> s, ds;
    uint64_t nds;
    using Out = double;
    HD double2 gen(uint64_t i) const { return make_double2(s[i / nds], ds[i % nds]); }
    __device__ Out dev(double2 a) const { return scale_to_integer_step(a.x, a.y, 1.0 / fabs(a.y)); }
    int check(double2 a, Out got) const { return !same_f64(got, orc_scale_to_integer_step(a.x, a.y)); }
    std::string show(double2 a) const { return fmt("s = %a, ds = %a", a.x, a.y); }
};

struct RemCheck {    // rem_euclid1 against f64::rem_euclid(1.0) = fmod(x, 1), + 1 if negative
    List<double> x;
    using Out = double;
    HD double gen(uint64_t i) const { return x[i]; }
    __device__ Out dev(double v) const { return rem_euclid1(v); }
    int check(double v, Out got) const {
        const double r = std::fmod(v, 1.0);
        return !same_f64(got, r < 0.0 ? r + 1.0 : r);
    }
    std::string show(double v) const { return fmt("x = %a", v); }
};

// Camera::post_process_color + to_srgb8 of ColorBuf cb under one camera's settings
struct EncodeCase { float cb[4]; float exposure, max_intensity; int tone; };
struct EncodeCheck {
    List<EncodeCase> c;
    const float *thr;        // device tables + 256
    TraceParams *params;     // one per case on the device: exposure, tone mapping, maximum intensity
    using Out = uchar4;
    HD uint64_t gen(uint64_t i) const { return i; }
    __device__ Out dev(uint64_t i) const {
        const EncodeCase e = c[i];
        return encode_srgb8(params[i], thr, e.cb[0], e.cb[1], e.cb[2], e.cb[3]);
    }
    int check(uint64_t i, Out got) const {
        const EncodeCase e = c[i];
        uint8_t want[4];
        orc_to_srgb8(e.cb, e.exposure, e.tone, e.max_intensity, want);
        return got.x != want[0] || got.y != want[1] || got.z != want[2] || got.w != want[3];
    }
    std::string show(uint64_t i) const {
        const EncodeCase e = c[i];
        return fmt("cb = (%a, %a, %a, %a)", e.cb[0], e.cb[1], e.cb[2], e.cb[3]) +
               fmt(", exposure %a, maximum %a, tone %g", e.exposure, e.max_intensity, e.tone);
    }
};

static std::vector<EncodeCase> encode_cases() {
    const float light_edges[] = {0.0f, -0.0f, 1e-30f, 1e-7f, 0.001f, 0.0031308f, 0.04f, 0.5f, 0.99f, 1.0f, 1.5f,
                                 10.0f, 1e6f, 3.4e38f, INFINITY, -1e-30f, -0.5f, -INFINITY, NAN};
    const float t_edges[] = {0.0f, 0.25f, 0.5f, 0.999f, std::nextafter(1.0f, 0.0f), 1.0f, 1.5f, -0.5f, 1e-7f, NAN};
    const float exposures[] = {1.0f, 0.5f, 2.0f, 0.0f, 1e-3f, 37.0f};
    const float maxima[] = {INFINITY, 1.0f, 0.5f, 4.0f, 1e-6f};
    std::vector<EncodeCase> v;
    uint64_t h = 12345;
    const int nl = sizeof light_edges / sizeof *light_edges, nt = sizeof t_edges / sizeof *t_edges;
    for (float ex : exposures)
        for (float mx : maxima)
            for (int tone = 0; tone < 2; tone++) {
                // the edges: each light value in each channel with a random other two, at every transmittance
                for (int li = 0; li < nl; li++)
                    for (int ti = 0; ti < nt; ti++)
                        for (int ch = 0; ch < 3; ch++) {
                            EncodeCase e{{0, 0, 0, t_edges[ti]}, ex, mx, tone};
                            for (int k = 0; k < 3; k++) {
                                h = mix64(h);
                                e.cb[k] = k == ch ? light_edges[li] : (float)(h >> 40) * 0x1p-22f;
                            }
                            v.push_back(e);
                        }
                // random ColorBufs: light in [0, 4) (a few in [0, 2^20)), T in [0, 1]
                for (int r = 0; r < 20000; r++) {
                    EncodeCase e{{0, 0, 0, 0}, ex, mx, tone};
                    for (int k = 0; k < 3; k++) {
                        h = mix64(h);
                        e.cb[k] = (float)(h >> 40) * ((r & 15) ? 0x1p-22f : 0x1p-4f);
                    }
                    h = mix64(h);
                    e.cb[3] = (float)(h >> 40) * 0x1p-24f;
                    v.push_back(e);
                }
            }
    return v;
}

int main(int argc, char **argv) {
    const char *tex = argv[2];
    orc_packed_light_scalar_in = (int (*)(float))sym(argv[1], "orc_packed_light_scalar_in");
    orc_to_srgb8 = (void (*)(const float *, float, int, float, uint8_t *))sym(argv[1], "orc_to_srgb8");
    orc_powf = (float (*)(float, float, int))sym(argv[1], "orc_powf");
    orc_expf = (float (*)(float, int))sym(argv[1], "orc_expf");
    orc_scale_to_integer_step = (double (*)(double, double))sym(argv[1], "orc_scale_to_integer_step");
    orc_f16_from_f32 = (uint16_t (*)(float))sym(tex, "orc_f16_from_f32");

    // the library's tables (DeviceScene::tables): [256, 512) sRGB8 thresholds, [512, 768) light thresholds
    float tables[768] = {};
    build_srgb_thresholds(tables + 256);
    build_light_thresholds(tables + 512);
    float *d_tables;
    CK(cudaMalloc(&d_tables, sizeof tables));
    CK(cudaMemcpy(d_tables, tables, sizeof tables, cudaMemcpyHostToDevice));

    const uint64_t ALL = 1ull << 32;
    for (int a = 3; a < argc; a++) {
        const std::string m = argv[a];
        if (m == "srgb8") sweep("srgb8", SrgbCheck{d_tables}, ALL);
        else if (m == "light") sweep("light", LightCheck{d_tables}, ALL);
        else if (m == "f16") sweep("f16", F16Check{}, ALL);
        else if (m == "pow_all_u") {
            for (float th : {0.5f, 1.5f, 16.0f})
                sweep(("pow_all_u " + fmt("%g", th)).c_str(), pow_check(PowAllU{th}), 0x3f7fffffu);
        } else if (m == "pow_grid") {
            const uint32_t stride = 509, per = 0x3f7fffffu / stride;
            sweep("pow_grid", pow_check(PowGrid{stride, per}), (uint64_t)per * 256);
        } else if (m == "pow_random") sweep("pow_random", pow_check(PowRandom{}), 200000000ull);
        else if (m == "exp_fog") sweep("exp_fog", exp_check(ExpFog{0x3fccccceu}), 0x3fccccceu);
        else if (m == "exp_wide") {
            const uint32_t stride = 7, npos = fbits(89.0f) / stride + 1, nneg = fbits(104.0f) / stride + 1;
            sweep("exp_wide", exp_check(ExpWide{stride, npos}), (uint64_t)npos + nneg);
        } else if (m == "div_pixels") sweep("div_pixels", div_check(DivPixels{}), tri(16385));
        else if (m == "div_random") sweep("div_random", div_check(DivRandom{}), 100000000ull);
        else if (m == "div_ndc") sweep("div_ndc", NdcCheck{}, 10000000ull);
        else if (m == "step") {
            const std::vector<double> s = integer_edges();
            std::vector<double> ds = {0.0, 0x1p-1074, 0x1p-1030, 0x1p-1022, 0x1p-401, 0x1p-400, 0x1p-399, 1e-10, 0.1,
                                      0.5, 1.0, 3.0, 0x1p399, 0x1p400, 0x1p401, 1e100, INFINITY, NAN};
            for (size_t k = 0, n = ds.size(); k < n; k++) ds.push_back(-ds[k]);
            for (size_t k = 0, n = ds.size(); k < n; k++) ds.push_back(std::nextafter(ds[k], 1.0));
            sweep("step", StepCheck{upload(s), upload(ds), ds.size()}, (uint64_t)s.size() * ds.size());
        } else if (m == "rem") {
            const std::vector<double> x = integer_edges();
            sweep("rem", RemCheck{upload(x)}, x.size());
        } else if (m == "encode") {
            const std::vector<EncodeCase> v = encode_cases();
            std::vector<TraceParams> params(v.size());
            for (size_t i = 0; i < v.size(); i++) {
                std::memset(&params[i], 0, sizeof(TraceParams));
                params[i].exposure = v[i].exposure;
                params[i].maximum_intensity = v[i].max_intensity;
                params[i].tone_mapping = (uint32_t)v[i].tone;
            }
            sweep("encode", EncodeCheck{upload(v), d_tables + 256, (TraceParams *)upload(params).d}, v.size());
        } else {
            std::fprintf(stderr, "unknown check %s\n", m.c_str());
            return 2;
        }
    }
    return 0;
}
"""


def _compile(tmp, name, source, extra):
    src, exe = tmp / f"{name}.cu", tmp / name
    src.write_text(source)
    flags = [f for f in g.NVCC_FLAGS if f != "-shared"]
    cmd = [g.NVCC] + flags + ["-Xcompiler", "-pthread", "-I", CSRC, "-o", str(exe), str(src)] + extra
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return str(exe)


def _lines(out):
    return {t["check"]: t for t in map(json.loads, out.splitlines())}


def test_host_threshold_search(tmp_path):
    # The threshold tables as the library builds them, searched in 8 steps as the device searches them, equal
    # srgb8_host (platform powf) and scalar_in (platform log2f) on every f32 bit pattern: NaNs, +-0, subnormals, +-inf.
    # This is the premise the device encoders rest on, that both formulas are monotone in c on this host's libm.
    exe = _compile(tmp_path, "host_tables", HOST_DRIVER, [])
    t = json.loads(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    assert t["n"] == 2 ** 32
    assert t["mismatch"] == [0, 0], t


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    g.build_texture_oracle()
    return _compile(tmp_path_factory.mktemp("scalar_math"), "scalar_math", GPU_DRIVER, ["-ldl"])


def run(driver, *checks):
    out = subprocess.run([driver, ORACLE_LIB, TEXTURE_LIB, *checks], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return _lines(out.stdout)


def check(t, n, variants=1):
    assert t["n"] == n, t
    for v, name in enumerate(["", " (the fallback alone)"][:variants]):
        assert t["mismatch"][v] == 0, f"{t['check']}{name}: {t['mismatch'][v]} of {n} differ, first at {t['first'][v]}"


def _f32(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def check_cr(t, n, op):
    """The device equals the oracle's LIBM_CR on all n arguments, and wherever LIBM_CR differs from glibc's f64 pow /
    exp rounded to f32, LIBM_CR is the nearer to the exact value (60 significant digits)."""
    check(t, n, variants=2)
    assert t["glibc_differs"] == len(t["disputed"]) <= 1000, t["glibc_differs"]
    ctx = Context(prec=60)
    for xb, yb, crb, libb in t["disputed"]:
        x, y, cr, lib = (_f32(b) for b in (xb, yb, crb, libb))
        exact = ctx.exp(Decimal(x)) if op == "exp" else ctx.exp(ctx.multiply(ctx.ln(Decimal(x)), Decimal(y)))
        assert abs(exact - Decimal(cr)) < abs(exact - Decimal(lib)), (t["check"], x, y, cr, lib)
    print(f"{t['check']}: {n} arguments, glibc's f64 {op} rounded to f32 is not the nearest f32 at {len(t['disputed'])}")


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["srgb8", "light", "f16"])
def test_every_f32_pattern(driver, which):
    # component_to_srgb8 and scalar_in_t with the library's thresholds, and f16x2_texel (__floats2half2_rn), as
    # finish_pixel stores rgba16f and texture texels, on all 2^32 inputs
    check(run(driver, which)[which], 2 ** 32)


@pytest.mark.gpu
def test_powf(driver):
    # powf_exact and, on its own, its double-double fallback powf_libm: every f32 u in (0, 1) at thickness 0.5, 1.5 and
    # 16; thickness k / 16 up to 16 at 1/509 of them; 2 * 10^8 random (u, thickness) pairs
    r = run(driver, "pow_all_u", "pow_grid", "pow_random")
    for th in ("0.5", "1.5", "16"):
        check_cr(r["pow_all_u " + th], 0x3F7FFFFF, "pow")
    check_cr(r["pow_grid"], (0x3F7FFFFF // 509) * 256, "pow")
    check_cr(r["pow_random"], 200_000_000, "pow")


@pytest.mark.gpu
def test_expf(driver):
    # expf_exact and, on its own, expf_libm: every f32 in [-1.6, 0] (distance_fog's exponents), and every 7th f32 of [-104, 89],
    # from results that underflow to 0 to ones that overflow to inf
    r = run(driver, "exp_fog", "exp_wide")
    check_cr(r["exp_fog"], 0x3FCCCCCE, "exp")
    check_cr(r["exp_wide"], 0x42B20000 // 7 + 1 + 0x42D00000 // 7 + 1, "exp")


@pytest.mark.gpu
def test_div_known_recip(driver):
    # x / W for every framebuffer size W up to 16384 and every x in 0..W; 10^8 random pairs over and around the
    # exponent window; 10^7 of project_ndc's three quotients by one w
    r = run(driver, "div_pixels", "div_random", "div_ndc")
    check(r["div_pixels"], 16384 * 16387 // 2)
    check(r["div_random"], 100_000_000)
    check(r["div_ndc"], 10_000_000)


@pytest.mark.gpu
def test_step_rem_encode(driver):
    # scale_to_integer_step and rem_euclid1 around the integers, and the ColorBuf -> sRGB8 encoding (Rgba::from,
    # post_process_color with Clamp and Reinhard, the threshold search, alpha's sat_u8) on random and edge ColorBufs
    r = run(driver, "step", "rem", "encode")
    for name in ("step", "rem", "encode"):
        assert r[name]["n"] > 0
        check(r[name], r[name]["n"])
