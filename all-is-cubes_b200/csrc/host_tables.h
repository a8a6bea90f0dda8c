// host_tables.h — the two f32 -> u8 quantisers that the device evaluates as threshold searches, in their direct form
// with the platform libm, and the threshold tables built from them (DeviceScene::tables [256, 768)).
//
// component_to_srgb8 (trace_kernel.cuh) and scalar_in_t (light_kernel.cuh) search thr[1..255] in 8 steps instead of
// calling powf / log2f.  The search equals the direct formula for every f32 only if the formula, evaluated with this
// host's libm, is monotone in c over all f32; tests/test_gpu_scalar_math.py checks both searches against the direct
// forms on all 2^32 bit patterns, on the host and on the device.  Host code only; included by aicb200.cu and by that
// test's driver.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace aicb {

// PackedLight::some -> scalar_in (light/data.rs:213-217)
static inline uint8_t scalar_in(float v) {
    float x = std::round(std::log2(v) * 10.0f + 144.0f);
    if (!(x > 0.0f)) return 0;
    if (x >= 255.0f) return 255;
    return (uint8_t)x;
}

// component_to_srgb8 (math/color.rs:1038-1054) evaluated with the platform powf — exactly what the
// reference computes on this host — and inverted into thresholds: thr[k] = the smallest non-negative
// f32 whose encoding is >= k.  The device encodes by searching this table.
static inline uint8_t srgb8_host(float c) {
    float s = (c <= 0.0031308f) ? c * (323.0f / 25.0f) : (211.0f * std::pow(c, 5.0f / 12.0f) - 11.0f) / 200.0f;
    float v = std::round(s * 255.0f);
    if (!(v > 0.0f)) return 0;
    if (v >= 255.0f) return 255;
    return (uint8_t)v;
}
static inline void build_srgb_thresholds(float *thr) {
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
static inline void build_light_thresholds(float *thr) {
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

}  // namespace aicb
