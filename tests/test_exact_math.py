"""The shading path's f32 transcendentals (csrc/exact_math.cuh): powf_exact and expf_exact are a short f64 polynomial
and Ziv's rounding test, with the libm call as the fallback, and must give (float)pow((double)x, (double)y) and
(float)exp((double)x) bit for bit.  The header is compiled here as host code with the project's -fmad=false and
-ffp-contract=off contract; its short paths use only correctly rounded operations, so they compute on the host the
f64 values the device computes.  Each check also measures the short path's f64 error against x87 long double powl /
expl, which must stay well inside the bound the rounding test assumes (EXACT_MATH_BOUND = 2^-40)."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER_DIR = os.path.join(ROOT, "all-is-cubes_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

DRIVER = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <thread>
#include <vector>
#include "exact_math.cuh"
using namespace aicb;

static uint32_t bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static float from_bits(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

struct Tally {
    unsigned long long n = 0, mismatch = 0, fallback = 0;
    double max_rel = 0.0;
    float bad_x = 0.0f, bad_y = 0.0f;
    void add(const Tally &o) {
        n += o.n; fallback += o.fallback; max_rel = std::fmax(max_rel, o.max_rel);
        if (o.mismatch && !mismatch) { bad_x = o.bad_x; bad_y = o.bad_y; }
        mismatch += o.mismatch;
    }
};

// one pow argument pair: the result against glibc, the short path's f64 value against powl
static void check_pow(float u, float th, bool measure, Tally &t) {
    t.n++;
    const float got = powf_exact(u, th), want = (float)pow((double)u, (double)th);
    if (bits(got) != bits(want) && t.mismatch++ == 0) { t.bad_x = u; t.bad_y = th; }
    if ((u >= 0x1p-126f) & (u < 1.0f) & (th > 0.0f)) {
        const double p = (double)th * exact_math::log_core(u);
        if (p < -120.0) return;
        const double y = exact_math::exp_core(p);
        float o;
        if (!exact_math::round_certain(y, o)) t.fallback++;
        if (measure) {
            const long double ref = powl((long double)u, (long double)th);
            if (ref > 0x1p-1000L) t.max_rel = std::fmax(t.max_rel, (double)fabsl(((long double)y - ref) / ref));
        }
    }
}

static void check_exp(float x, Tally &t) {
    t.n++;
    const float got = expf_exact(x), want = (float)exp((double)x);
    if (bits(got) != bits(want) && t.mismatch++ == 0) t.bad_x = x;
    const double y = exact_math::exp_core((double)x);
    float o;
    if (!exact_math::round_certain(y, o)) t.fallback++;
    const long double ref = expl((long double)x);
    t.max_rel = std::fmax(t.max_rel, (double)fabsl(((long double)y - ref) / ref));
}

template <class F> static Tally parallel(uint64_t n, F f) {
    const unsigned nt = std::thread::hardware_concurrency() ? std::thread::hardware_concurrency() : 4;
    std::vector<Tally> part(nt);
    std::vector<std::thread> th;
    for (unsigned w = 0; w < nt; w++)
        th.emplace_back([&, w] { for (uint64_t i = w; i < n; i += nt) f(i, part[w]); });
    for (auto &x : th) x.join();
    Tally t;
    for (auto &p : part) t.add(p);
    return t;
}

int main(int argc, char **argv) {
    const char *mode = argv[1];
    Tally t;
    if (!std::strcmp(mode, "exp")) {
        // every f32 in [-1.6, 0]: -0 .. -1.6f by bit pattern, and +0
        const uint32_t lo = 0x80000000u, hi = bits(-1.6f);
        t = parallel((uint64_t)(hi - lo) + 2, [&](uint64_t i, Tally &p) {
            check_exp(i == (uint64_t)(hi - lo) + 1 ? 0.0f : from_bits(lo + (uint32_t)i), p);
        });
    } else if (!std::strcmp(mode, "pow_all_u")) {
        // every f32 u in (0, 1) at one thickness
        const float th = std::strtof(argv[2], nullptr);
        t = parallel(bits(1.0f) - 1u, [&](uint64_t i, Tally &p) {
            check_pow(from_bits((uint32_t)i + 1u), th, (i & 255u) == 0, p);
        });
    } else if (!std::strcmp(mode, "pow_grid")) {
        // thickness k / 16 for k = 1..256, u in (0, 1) every `stride` bit patterns, at a phase
        // that depends on k
        const uint32_t stride = (uint32_t)std::strtoul(argv[2], nullptr, 0);
        const uint32_t per = (bits(1.0f) - 1u) / stride;
        t = parallel((uint64_t)per * 256u, [&](uint64_t i, Tally &p) {
            const uint32_t k = (uint32_t)(i / per) + 1u, j = (uint32_t)(i % per);
            const uint32_t ub = 1u + j * stride + (k * 2654435761u) % stride;
            check_pow(from_bits(ub), (float)k / 16.0f, (j & 63u) == 0, p);
        });
    } else if (!std::strcmp(mode, "pow_random")) {
        // random f32 u in (0, 1) and random positive finite f32 thickness: half log-uniform in [2^-20, 2^10], half any
        const uint64_t n = std::strtoull(argv[2], nullptr, 0);
        t = parallel(n, [&](uint64_t i, Tally &p) {
            std::mt19937_64 g(i * 0x9e3779b97f4a7c15ull + 17u);
            const float u = from_bits(1u + (uint32_t)(g() % (bits(1.0f) - 1u)));
            float th;
            if (i & 1) th = (float)std::exp2(-20.0 + 30.0 * (double)(g() >> 11) * 0x1p-53);
            else th = from_bits(1u + (uint32_t)(g() % (bits(3.4028235e38f))));
            check_pow(u, th, true, p);
        });
    } else {
        return 2;
    }
    std::printf("{\"n\": %llu, \"mismatch\": %llu, \"fallback\": %llu, \"max_rel\": %.6e, \"bad_x\": %.9g, \"bad_y\": %.9g}\n",
                t.n, t.mismatch, t.fallback, t.max_rel, (double)t.bad_x, (double)t.bad_y);
    return 0;
}
"""

BOUND = 2.0 ** -40
EXP_ERR, POW_ERR = 2.0 ** -48, 2.0 ** -43   # the error analyses of exp_core and of powf_exact's short path


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("exact_math")
    src, exe = d / "driver.cu", d / "driver"
    src.write_text(DRIVER)
    cmd = [NVCC, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false",
           "-Xcompiler", "-ffp-contract=off,-fno-fast-math,-O2,-pthread", "-I", HEADER_DIR, "-o", str(exe), str(src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return str(exe)


def run(driver, *args):
    out = subprocess.run([driver] + [str(a) for a in args], capture_output=True, text=True, check=True).stdout
    return json.loads(out)


def check(t, err_bound, expect_n=None):
    assert t["mismatch"] == 0, f"{t['mismatch']} results differ from libm, first at ({t['bad_x']!r}, {t['bad_y']!r})"
    # the short path's own error stays within its analysed bound, far inside the rounding test's: the margin, not
    # luck, is what makes it exact
    assert t["max_rel"] < err_bound <= BOUND / 8, t
    # and the libm fallback stays rare
    assert t["fallback"] <= t["n"] * 2.0 ** -12, t
    if expect_n is not None:
        assert t["n"] == expect_n


def test_expf_exact_every_fog_exponent(driver):
    # all f32 in [-1.6, 0], both zeros included
    check(run(driver, "exp"), EXP_ERR, expect_n=0x3FCCCCCD + 2)


@pytest.mark.parametrize("th", ["0.5", "1.5", "16"])
def test_powf_exact_every_unit_transmittance(driver, th):
    # all f32 u in (0, 1) at three thicknesses of the grid below: a fraction, a mixed number and its largest value
    check(run(driver, "pow_all_u", th), POW_ERR, expect_n=0x3F7FFFFF)


def test_powf_exact_thickness_grid(driver):
    # every thickness k / 16 up to 16, each against 1/509 of the f32s in (0, 1) (a different phase per thickness)
    check(run(driver, "pow_grid", 509), POW_ERR)


def test_powf_exact_random_arguments(driver):
    check(run(driver, "pow_random", 20_000_000), POW_ERR)
