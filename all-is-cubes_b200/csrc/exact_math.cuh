// exact_math.cuh — the f32 transcendentals of the shading path, x^y and e^x for f32 arguments, correctly rounded to
// f32: a short f64 polynomial and Ziv's rounding test, with a double-double evaluation as the fallback.
//
// Why it is exact: the short paths and the double-double evaluation use only correctly rounded operations (+, *, fma,
// rint, reciprocal, conversions), so they give the same values on the device and on the host.  The short paths' f64
// value y is within a relative EXACT_MATH_BOUND of the true result; when y * (1 - bound) and y * (1 + bound) round to
// the same f32 (Ziv's rounding test), that f32 is the correctly rounded result.  Otherwise (about one call in 2^15)
// the double-double evaluation is made, to within CR_BOUND, and tested again; what is still undecided lies within
// 2^-90 of an f32 rounding midpoint and is taken to be that midpoint (an exact case such as (m^2)^1.5 = m^3), rounded
// to even.  Outside the short paths' domains, powf_libm / expf_libm make Ziv's test on the f64 libm value at
// LIBM_BOUND first, which decides all but about one call in 2^24, and evaluate the rest in double-double.
//
// The f64 libm value, rounded once, is not enough by itself: libdevice's f64 pow and glibc's round to different f32s
// on 48 of the 2^30 unit transmittances at thickness 1.5 (glibc's is the nearest f32 there), each of them an argument
// the short path hands to the fallback.  The oracle's LIBM_CR mode includes this header as host code, so the device
// and the oracle compute the same correctly rounded f32.  tests/test_exact_math.py compiles the header as host
// code with the project's -fmad=false contract and checks it against glibc; tests/test_gpu_scalar_math.py checks the
// device's results against the host's on every f32 exp argument in [-1.6, 0], a stride of [-104, 89], every unit
// transmittance at three thicknesses, a thickness grid and random pairs, and checks every disagreement with glibc
// against a 60-digit evaluation.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace aicb {

#ifdef __CUDACC__
#define AICB_HD_INLINE __host__ __device__ __forceinline__
#define AICB_HD_NOINLINE __host__ __device__ __noinline__
#else   // a plain C++ compiler (the oracle)
#define AICB_HD_INLINE inline __attribute__((always_inline))
#define AICB_HD_NOINLINE __attribute__((noinline))
#endif

// Bound on the relative error of the short paths' f64 values, with ample margin: the analysis below gives < 2^-43 for
// pow and < 2^-48 for exp.  A wider bound only sends more arguments to the fallback (about one in 2^15 here).
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

// ---- double-double: a value hi + lo with |lo| <= ulp(hi) / 2, about 106 bits
struct DD {
    double hi, lo;
};
AICB_HD_INLINE DD fast_two_sum(double a, double b) {  // |a| >= |b| or a == 0
    const double s = a + b;
    return DD{s, b - (s - a)};
}
AICB_HD_INLINE DD two_sum(double a, double b) {
    const double s = a + b, bb = s - a;
    return DD{s, (a - (s - bb)) + (b - bb)};
}
AICB_HD_INLINE DD two_prod(double a, double b) {
    const double p = a * b;
    return DD{p, fma(a, b, -p)};
}
AICB_HD_INLINE DD dd_add(DD a, DD b) {  // accurate under cancellation too
    DD s = two_sum(a.hi, b.hi);
    const DD t = two_sum(a.lo, b.lo);
    s = fast_two_sum(s.hi, s.lo + t.hi);
    return fast_two_sum(s.hi, s.lo + t.lo);
}
AICB_HD_INLINE DD dd_add_same_sign(DD a, DD b) {  // a and b of one sign: no cancellation, error <= 2^-104 |a + b|
    const DD s = two_sum(a.hi, b.hi);
    return fast_two_sum(s.hi, s.lo + (a.lo + b.lo));
}
AICB_HD_INLINE DD dd_mul(DD a, DD b) {
    const DD p = two_prod(a.hi, b.hi);
    return fast_two_sum(p.hi, p.lo + (a.hi * b.lo + a.lo * b.hi));
}
AICB_HD_INLINE DD dd_mul_d(DD a, double b) {
    const DD p = two_prod(a.hi, b);
    return fast_two_sum(p.hi, p.lo + a.lo * b);
}
// 1 / b for b > 0 to about 2^-105: RN(1 / b) (the device's reciprocal instruction, not a division routine, whose
// registers would count against every kernel that calls the fallback) and its remainder, which fma gives exactly.
AICB_HD_INLINE DD dd_recip(double b) {
#ifdef __CUDA_ARCH__
    const double r = __drcp_rn(b);
#else
    const double r = 1.0 / b;
#endif
    return DD{r, fma(-b, r, 1.0) * r};
}

// ln 2 in three parts
constexpr double LN2_HI = 0x1.62e42fefa39efp-1, LN2_MID = 0x1.abc9e3b39803fp-56, LN2_LO = 0x1.7b57a079a1934p-111;

// ln x for a finite f32 x > 0, to about 2^-102 relative.  x = 2^e m with m in [sqrt(1/2), sqrt(2)) (the f64 of x is
// normal, subnormal f32s included); ln m = 2 atanh(s), s = (m - 1) / (m + 1) (m - 1 and m + 1 exact), |s| <= 0.1716,
// summed to s^43: the truncation is < s^44 < 2^-110 relative.  |e ln2| >= 0.69 > |ln m| when e != 0, so the final sum
// does not cancel.
AICB_HD_INLINE DD log_dd(float x) {
    const double xd = (double)x;
    uint64_t b;
#ifdef __CUDA_ARCH__
    b = (uint64_t)__double_as_longlong(xd);
#else
    std::memcpy(&b, &xd, sizeof b);
#endif
    int e = (int)(b >> 52) - 1023;
    uint64_t mb = b & 0xfffffffffffffull;
    const bool half = mb > 0x6a09e667f3bcdull;   // m >= sqrt(2): take m / 2
    if (half) e += 1;
    mb |= (uint64_t)(half ? 1022 : 1023) << 52;
    double m;
#ifdef __CUDA_ARCH__
    m = __longlong_as_double((long long)mb);
#else
    std::memcpy(&m, &mb, sizeof m);
#endif
    const DD s = dd_mul_d(dd_recip(m + 1.0), m - 1.0);
    const DD s2 = dd_mul(s, s);
    DD term = s, sum = s;
#pragma unroll 1   // rolled: the fallback's registers count against every kernel that calls it
    for (int k = 1; k <= 21; k++) {
        term = dd_mul(term, s2);
        sum = dd_add_same_sign(sum, dd_mul(term, dd_recip((double)(2 * k + 1))));
    }
    const double ed = (double)e;
    DD eln2 = two_prod(ed, LN2_HI);
    eln2 = dd_add(eln2, two_prod(ed, LN2_MID));
    eln2 = dd_add(eln2, DD{ed * LN2_LO, 0.0});
    return dd_add(eln2, DD{2.0 * sum.hi, 2.0 * sum.lo});
}

// e^p for -104 <= p.hi <= 89, to about 2^-103 relative.  p = k ln2 + r, |r| <= 0.35: k ln2_hi is subtracted exactly
// (the difference is a multiple of 2^-54 below 0.36), the rest in double-double; e^r by Horner to r^27 / 27!, whose
// truncation is < 0.35^28 / 28! < 2^-130.  2^k is a normal f64 here, so the scaling is exact.
AICB_HD_INLINE DD exp_dd(DD p) {
    const double k = rint(p.hi * 1.4426950408889634);
    DD r{fma(-k, LN2_HI, p.hi), 0.0};
    r = dd_add(r, DD{p.lo, 0.0});
    r = dd_add(r, two_prod(-k, LN2_MID));
    r = dd_add(r, DD{-k * LN2_LO, 0.0});
    DD t{1.0, 0.0};
#pragma unroll 1
    for (int n = 27; n >= 1; n--) t = dd_add(DD{1.0, 0.0}, dd_mul(dd_mul(t, r), dd_recip((double)n)));
    const double s = pow2i((int)k);
    return DD{t.hi * s, t.lo * s};
}

// RN_f32(hi + lo) for a normalised double-double: (float)hi, unless hi is exactly the midpoint between two f32s, where
// the sign of lo decides.  (No other midpoint can lie between hi and hi + lo: hi is the f64 nearest to it, and every
// f32 midpoint is an f64.)
AICB_HD_INLINE float round_dd_f32(DD v) {
    const float f = (float)v.hi;
    if ((double)f == v.hi || v.lo == 0.0) return f;
    const float g = nextafterf(f, v.hi > (double)f ? INFINITY : -INFINITY);
    if (v.hi != 0.5 * ((double)f + (double)g)) return f;
    return (v.lo > 0.0) == (g > f) ? g : f;
}

// Bound on the relative error of exp_dd(y log_dd(x)) for |y ln x| <= 104 (ln x's 2^-102 becomes 104 2^-102 < 2^-95
// absolute in p, and so relative in e^p), with ample margin.
constexpr double CR_BOUND = 0x1p-90;

// The f32 nearest to v, known to within CR_BOUND: Ziv's test at that bound; what it leaves undecided is within 2^-90 of
// a rounding midpoint and is taken to be that midpoint, rounded to even.
AICB_HD_INLINE float round_cr(DD v) {
    const double e = fabs(v.hi) * CR_BOUND;
    const float lo = round_dd_f32(fast_two_sum(v.hi, v.lo - e)), hi = round_dd_f32(fast_two_sum(v.hi, v.lo + e));
    if (lo == hi) return lo;
    return (float)(0.5 * (double)lo + 0.5 * (double)hi);
}

// The f32 nearest to the f64 libm value v, if every value within LIBM_BOUND of v rounds to it: libdevice's f64 pow
// and exp are within 2 ULP (2^-51 relative), glibc's within 1.
constexpr double LIBM_BOUND = 0x1p-49;
AICB_HD_INLINE bool libm_certain(double v, float &out) {
    const float lo = (float)(v * (1.0 - LIBM_BOUND)), hi = (float)(v * (1.0 + LIBM_BOUND));
    out = lo;
    return lo == hi;
}

}  // namespace exact_math

// The double-double evaluation, out of line in two calls (y ln x, then e^p rounded), because a kernel's register count
// covers the functions it calls: each is no larger than the libm call, and what passes between them is one DD.
static AICB_HD_NOINLINE exact_math::DD pow_exponent_dd(float x, float y) {   // y ln x for finite x > 0
    return exact_math::dd_mul_d(exact_math::log_dd(x), (double)y);
}
static AICB_HD_NOINLINE float exp_dd_f32(exact_math::DD p) {   // e^p correctly rounded to f32
    if (p.hi < -104.0) return 0.0f;       // e^p < 2^-150.04: rounds to +0
    if (p.hi > 89.0) return INFINITY;     // e^p > FLT_MAX (1 + 2^-24): rounds to +inf
    return exact_math::round_cr(exact_math::exp_dd(p));
}

// The f64 libm calls, out of line: one copy in a kernel, off the short paths' register budget.
static AICB_HD_NOINLINE double pow_f64(float x, float y) { return pow((double)x, (double)y); }
static AICB_HD_NOINLINE double exp_f64(float x) { return exp((double)x); }

// x^y and e^x correctly rounded to f32, for every f32 argument.  The f64 libm call decides almost every argument
// (Ziv's test at LIBM_BOUND); the rest, within 2^-49 of an f32 rounding midpoint, take the double-double evaluation.
// The special cases (a zero, infinite or NaN argument, x = +-1, y = 0, x < 0 with y not an integer) have exact
// results, 0, +-1, inf or NaN, which the libm call gives.  Inline: in the kernels that call them directly (None, Flat
// and Bounce lighting), every call is then one level deep and no larger than the libm call, and their registers are
// the same as with the libm call alone.
AICB_HD_INLINE float powf_libm(float x, float y) {
    const double v = pow_f64(x, y);
    const float ax = fabsf(x);
    if (!((ax > 0.0f) & (ax <= 3.4028235e38f) & (fabsf(y) <= 3.4028235e38f) & (ax != 1.0f) & (y != 0.0f) &
          ((x > 0.0f) | (y == truncf(y)))))
        return (float)v;
    float r;
    if (!exact_math::libm_certain(v, r)) {
        r = exp_dd_f32(pow_exponent_dd(ax, y));
        if ((x < 0.0f) && (fabsf(y) < 0x1p24f) && ((long long)y & 1)) r = -r;   // a negative base: y is an integer
    }
    return r;
}
AICB_HD_INLINE float expf_libm(float x) {
    const double v = exp_f64(x);
    if (!((x >= -104.0f) & (x <= 89.0f))) return x < -104.0f ? 0.0f : (float)v;   // rounds to +0; inf; NaN
    float r;
    if (exact_math::libm_certain(v, r)) return r;
    return exp_dd_f32(exact_math::DD{(double)x, 0.0});
}

// powf_libm and expf_libm in one out-of-line call, for the short paths' callers (shade_kernel<LC_INTERP>, at 64
// registers), where the arguments outside their domains are rare.
static AICB_HD_NOINLINE float powf_libm_call(float x, float y) { return powf_libm(x, y); }
static AICB_HD_NOINLINE float expf_libm_call(float x) { return expf_libm(x); }

// x^y correctly rounded.  Short path: x a normal f32 in (0, 1), y > 0 finite (apply_transmittance's
// unit transmittance and thickness).  p = y ln x is within 2^-50 |p| (one more rounding), and it matters only while
// p >= -120: below, the result is under 2^-173 and every value within the bound rounds to +0.  There
// |p| 2^-50 < 2^-43, so e^p is within 2^-43 relative.
AICB_HD_INLINE float powf_exact(float x, float y) {
    if ((x >= 0x1p-126f) & (x < 1.0f) & (y > 0.0f) & (y <= 3.4028235e38f)) {
        const double p = (double)y * exact_math::log_core(x);
        if (p < -120.0) return 0.0f;
        float out;
        if (exact_math::round_certain(exact_math::exp_core(p), out)) return out;
        return exp_dd_f32(pow_exponent_dd(x, y));
    }
    return powf_libm_call(x, y);
}

// e^x correctly rounded.  Short path: x in [-1.6, 0] (distance_fog's exponent), where it is exhaustively
// checked.
AICB_HD_INLINE float expf_exact(float x) {
    if ((x >= -1.6f) & (x <= 0.0f)) {
        float out;
        if (exact_math::round_certain(exact_math::exp_core((double)x), out)) return out;
        return exp_dd_f32(exact_math::DD{(double)x, 0.0});
    }
    return expf_libm_call(x);
}

}  // namespace aicb
