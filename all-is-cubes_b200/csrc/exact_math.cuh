// exact_math.cuh — the f32 transcendentals of the shading path, (float)pow((double)x, (double)y) and
// (float)exp((double)x), evaluated by a short f64 polynomial and rounded once, bit-identical to the libm call.
//
// Why it is exact: the short paths use only correctly rounded operations (+, *, fma, rint, conversions), so they give
// the same f64 value y on the device and on the host.  That value is within a relative EXACT_MATH_BOUND of the true
// result, and so is the libm call's f64 value (libdevice pow and exp and glibc's are within 2 ULP of f64).  When
// y * (1 - bound) and y * (1 + bound) round to the same f32 (Ziv's rounding test), no f32 rounding boundary lies
// between y and the libm value, and the f32 results are equal.  Otherwise, and for the arguments outside the short
// paths' domains, the libm call itself is made.  tests/test_exact_math.py compiles this header as host code with the
// project's -fmad=false contract and checks every f32 exp argument in [-1.6, 0] and a dense grid of pow arguments
// against glibc.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace aicb {

#define AICB_HD_INLINE __host__ __device__ __forceinline__

// Bound on the relative error of the short paths' f64 values plus that of the libm call, with ample margin: the
// analysis below gives < 2^-43 for pow and < 2^-48 for exp.  A wider bound only sends more arguments to libm (about
// one in 2^15 here).
constexpr double EXACT_MATH_BOUND = 0x1p-40;

namespace exact_math {

AICB_HD_INLINE double pow2i(int k) {  // 2^k for -1022 <= k <= 1023, exactly
    const uint64_t bits = (uint64_t)(k + 1023) << 52;
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)bits);
#else
    double d;
    std::memcpy(&d, &bits, sizeof d);
    return d;
#endif
}

AICB_HD_INLINE uint32_t f32_bits(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u;
    std::memcpy(&u, &f, sizeof u);
    return u;
#endif
}

AICB_HD_INLINE float f32_from_bits(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    std::memcpy(&f, &u, sizeof f);
    return f;
#endif
}

// e^p for -746 < p <= 1 (2^k stays a normal f64).  p = k ln2 + r with |r| <= ln2 / 2 + 2^-40 (ln2 in two parts; the
// fmas are exact in their products, so r carries 2 roundings, <= 2^-52 |r|), then Taylor to degree 12: the truncation
// is < 0.347^13 / 13! < 2^-52 relative, and the 13 Horner fmas add < 2^-50.  Total < 2^-49 relative.
AICB_HD_INLINE double exp_core(double p) {
    constexpr double LOG2E = 1.4426950408889634, LN2_HI = 0x1.62e42fefa39efp-1, LN2_LO = 0x1.abc9e3b39803fp-56;
    const double k = rint(p * LOG2E);
    double r = fma(-k, LN2_HI, p);
    r = fma(-k, LN2_LO, r);
    double q = 1.0 / 479001600.0;          // 1/12!
    q = fma(q, r, 1.0 / 39916800.0);
    q = fma(q, r, 1.0 / 3628800.0);
    q = fma(q, r, 1.0 / 362880.0);
    q = fma(q, r, 1.0 / 40320.0);
    q = fma(q, r, 1.0 / 5040.0);
    q = fma(q, r, 1.0 / 720.0);
    q = fma(q, r, 1.0 / 120.0);
    q = fma(q, r, 1.0 / 24.0);
    q = fma(q, r, 1.0 / 6.0);
    q = fma(q, r, 0.5);
    q = fma(q, r, 1.0);
    q = fma(q, r, 1.0);
    return q * pow2i((int)k);
}

// ln x for a normal f32 x > 0.  x = 2^e m with m in [sqrt(1/2), sqrt(2)); ln m = 2 atanh(s), s = (m - 1) / (m + 1),
// |s| <= 0.1716, summed to s^19: the truncation is < s^20 / 21 < 2^-55 relative.  m - 1 and m + 1 are exact; 1 / (m + 1)
// is a linear seed (2^-6) and three Newton steps (2^-48), and s is corrected once from the exact remainder, to
// < 2^-52.  With the series' roundings and the e ln2 term, ln x is within 2^-50 relative.
AICB_HD_INLINE double log_core(float x) {
    constexpr double LN2_HI = 0x1.62e42fefa39efp-1, LN2_LO = 0x1.abc9e3b39803fp-56;
    const uint32_t b = f32_bits(x);
    int e = (int)(b >> 23) - 127;
    uint32_t mb = b & 0x7fffffu;
    if (mb > 0x3504f3u) e += 1;                       // m >= sqrt(2): take m / 2
    const double m = (double)f32_from_bits(mb | (mb > 0x3504f3u ? 0x3f000000u : 0x3f800000u));
    const double f = m - 1.0, d = m + 1.0;
    double r = fma(-0.23901599922648398, d, 0.9850615000483445);   // 1 / d on [1.707, 2.415] to 2^-6
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    const double q = f * r;
    const double s = fma(fma(-d, q, f), r, q);
    const double s2 = s * s;
    double t = 1.0 / 19.0;
    t = fma(t, s2, 1.0 / 17.0);
    t = fma(t, s2, 1.0 / 15.0);
    t = fma(t, s2, 1.0 / 13.0);
    t = fma(t, s2, 1.0 / 11.0);
    t = fma(t, s2, 1.0 / 9.0);
    t = fma(t, s2, 1.0 / 7.0);
    t = fma(t, s2, 1.0 / 5.0);
    t = fma(t, s2, 1.0 / 3.0);
    const double lnm = fma(2.0 * s * s2, t, 2.0 * s);
    return fma((double)e, LN2_HI, fma((double)e, LN2_LO, lnm));
}

// The f32 nearest to a value known only to within EXACT_MATH_BOUND of y, if every value there rounds to it.
AICB_HD_INLINE bool round_certain(double y, float &out) {
    const float lo = (float)(y * (1.0 - EXACT_MATH_BOUND)), hi = (float)(y * (1.0 + EXACT_MATH_BOUND));
    out = lo;
    return lo == hi;
}

}  // namespace exact_math

// Out of line: one copy of the libm code in a kernel, off the short paths' register budget.
static __host__ __device__ __noinline__ float powf_libm(float x, float y) { return (float)pow((double)x, (double)y); }
static __host__ __device__ __noinline__ float expf_libm(float x) { return (float)exp((double)x); }

// (float)pow((double)x, (double)y), bit for bit.  Short path: x a normal f32 in (0, 1), y > 0 finite (apply_transmittance's
// unit transmittance and thickness).  p = y ln x is within 2^-50 |p| (one more rounding), and it matters only while
// p >= -120: below, the result is under 2^-173 and every value within the bound rounds to +0.  There
// |p| 2^-50 < 2^-43, so e^p is within 2^-43 relative.
AICB_HD_INLINE float powf_exact(float x, float y) {
    if ((x >= 0x1p-126f) & (x < 1.0f) & (y > 0.0f) & (y <= 3.4028235e38f)) {
        const double p = (double)y * exact_math::log_core(x);
        if (p < -120.0) return 0.0f;
        float out;
        if (exact_math::round_certain(exact_math::exp_core(p), out)) return out;
    }
    return powf_libm(x, y);
}

// (float)exp((double)x), bit for bit.  Short path: x in [-1.6, 0] (distance_fog's exponent), where it is exhaustively
// checked.
AICB_HD_INLINE float expf_exact(float x) {
    if ((x >= -1.6f) & (x <= 0.0f)) {
        float out;
        if (exact_math::round_certain(exact_math::exp_core((double)x), out)) return out;
    }
    return expf_libm(x);
}

}  // namespace aicb
