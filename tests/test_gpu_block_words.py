"""surface_entry (block_words.cuh), the pal_tab pair of a palette entry, is one __host__ __device__ function: the host
flattening of aicb_scene_update_blocks and the device kernels of aicb_scene_update_blocks_device both call it, so their
tables are the same bytes only if the device's f64 log2 (libdevice), rounded to f32 and stepped up one ulp, equals the
host's (glibc) on every input.  A driver compiled with the library's flags and headers (as tests/test_gpu_scalar_math.py
compiles its own) evaluates it on the device for all 2^32 bit patterns of alpha and compares both halves of the pair
with the host's, bit for bit."""
import json
import subprocess

import pytest

from test_gpu_scalar_math import _compile

DRIVER = r"""
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>
#include "block_words.cuh"
using namespace aicb;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    std::fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 3; } } while (0)

__global__ void k_surface(uint64_t base, uint32_t n, uint2 *out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float2 e = surface_entry(__uint_as_float((uint32_t)(base + i)));
        out[i] = make_uint2(__float_as_uint(e.x), __float_as_uint(e.y));
    }
}

int main() {
    const uint32_t CHUNK = 1u << 27;
    uint2 *d = nullptr;
    CK(cudaMalloc(&d, (size_t)CHUNK * sizeof(uint2)));
    std::vector<uint2> h(CHUNK);
    const unsigned T = std::max(1u, std::thread::hardware_concurrency());
    uint64_t mismatch = 0, first = ~0ull;
    for (uint64_t base = 0; base < (1ull << 32); base += CHUNK) {
        k_surface<<<1024, 256>>>(base, CHUNK, d);
        CK(cudaGetLastError());
        CK(cudaMemcpy(h.data(), d, (size_t)CHUNK * sizeof(uint2), cudaMemcpyDeviceToHost));
        std::vector<uint64_t> bad(T, 0), at(T, ~0ull);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; t++)
            th.emplace_back([&, t] {
                for (uint64_t i = t; i < CHUNK; i += T) {
                    const uint32_t bits = (uint32_t)(base + i);
                    float a;
                    std::memcpy(&a, &bits, 4);
                    const float2 e = surface_entry(a);
                    uint32_t x, y;
                    std::memcpy(&x, &e.x, 4);
                    std::memcpy(&y, &e.y, 4);
                    if (x != h[i].x || y != h[i].y) {
                        bad[t]++;
                        if (at[t] == ~0ull) at[t] = base + i;
                    }
                }
            });
        for (auto &x : th) x.join();
        for (unsigned t = 0; t < T; t++) {
            mismatch += bad[t];
            first = std::min(first, at[t]);
        }
    }
    std::printf("{\"n\": %llu, \"mismatch\": %llu, \"first\": \"0x%08llx\"}\n", 1ull << 32,
                (unsigned long long)mismatch, (unsigned long long)(first & 0xffffffffu));
    return 0;
}
"""


@pytest.mark.gpu
def test_surface_entry_device_equals_host_on_every_alpha(tmp_path):
    exe = _compile(tmp_path, "block_words", DRIVER, [])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    t = json.loads(out.stdout)
    assert t["n"] == 2 ** 32
    assert t["mismatch"] == 0, t
