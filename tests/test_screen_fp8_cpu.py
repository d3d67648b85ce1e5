"""CPU checks of the e4m3 screen's arithmetic: the row scale and the bound screen_rel_err_fp8 (similari_b200/csrc/
sb_engine.cuh, compiled for the host by nvcc), against an independent numpy model of e4m3 round-to-nearest-even."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "similari_b200", "csrc")

PROBE = r"""
#include <cstdio>
#include "sb_engine.cuh"
int main() {
  float x;
  int d;
  char op;
  while (scanf(" %c", &op) == 1) {
    if (op == 's' && scanf("%a", &x) == 1) printf("%a\n", sb::fp8_row_scale(x));
    if (op == 'e' && scanf("%d", &d) == 1) printf("%a\n", sb::screen_rel_err_fp8(d));
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def probe():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tempfile.mkdtemp()
    src, exe = os.path.join(d, "probe.cu"), os.path.join(d, "probe")
    with open(src, "w") as f:
        f.write(PROBE)
    subprocess.check_call([nvcc, "-std=c++17", "-I", CSRC, src, "-o", exe])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return [float.fromhex(v) for v in out.split()]

    return run


def e4m3_rne(x):
    """numpy model of cvt.rn.satfinite.e4m3 for |x| <= 448: the decoded value.  Normal binades 2^-6 .. 2^8 keep 3
    fraction bits; below 2^-6 the spacing is 2^-9."""
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.maximum(e, -6.0)
    q = np.exp2(e - 3.0)                       # spacing of the binade
    r = np.round(a / q) * q                    # numpy rounds halves to even
    return np.sign(x) * np.minimum(r, 448.0)


def test_e4m3_model_decodes_known_codes():
    # every e4m3 code below the maximum is its own rounding; halves go to the even neighbour
    codes = [0.0, 2.0 ** -9, 3 * 2.0 ** -9, 2.0 ** -6, 1.0, 1.125, 240.0, 256.0, 288.0, 448.0]
    assert np.array_equal(e4m3_rne(codes), codes)
    assert e4m3_rne(1.0625) == 1.0 and e4m3_rne(1.1875) == 1.25 and e4m3_rne(432.0) == 448.0
    assert e4m3_rne(2.0 ** -10) == 0.0 and e4m3_rne(3 * 2.0 ** -10) == 2.0 ** -8


def test_row_scale_is_the_power_of_two_that_fits(probe):
    rng = np.random.default_rng(3)
    amax = np.concatenate([np.float32(2.0) ** np.arange(-90, 91, dtype=np.float32),
                           (np.float32(2.0) ** rng.integers(-90, 90, 400)).astype(np.float32)
                           * rng.uniform(1.0, 2.0, 400).astype(np.float32),
                           np.float32([224.0, 223.99998, 447.99997, 448.0, 0.875, 0.87499994])])
    got = np.float32(probe([f"s {float(a).hex()}" for a in amax]))
    k = np.log2(got)
    assert np.array_equal(k, np.round(k))                      # a power of two
    y = amax.astype(np.float64) * got
    assert np.all(y >= 224.0) and np.all(y < 448.0)          # the scaled maximum lands in [224, 448): no saturation
    # rows without a usable maximum get 1 (they keep every pair through fp8_norm_ok)
    assert probe([f"s {v}" for v in ("0x0p+0", "inf", "nan", "0x1p-120")]) == [1.0, 1.0, 1.0, 1.0]


def test_e4m3_rounding_within_the_bound_terms():
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.uniform(-448.0, 448.0, 20000), rng.uniform(-2.0 ** -5, 2.0 ** -5, 20000)])
    err = np.abs(e4m3_rne(x) - x)
    normal = np.abs(x) >= 2.0 ** -6
    assert np.all(err[normal] <= 2.0 ** -4 * np.abs(x[normal]))     # u = 2^-4
    assert np.all(err[~normal] <= 2.0 ** -10)                       # the subnormal floor


@pytest.mark.parametrize("d", [8, 64, 128, 136, 256, 512])
def test_fp8_bound_covers_its_terms(probe, d):
    e = probe([f"e {d}"])[0]
    u = 2.0 ** -4
    rnd = 2 * u + u * u
    sub = 2 * (1 + u) * np.sqrt(d) * 2.0 ** -10 / 224.0
    acc = -(-d // 32) * 34 * 2.0 ** -12 * (1 + u) ** 2
    assert e >= rnd + sub + acc
    assert e < 0.3   # d <= 512: still a filter on unit-norm features at selective thresholds


def test_fp8_bound_on_random_rows_with_exact_accumulation():
    """The operand part of the bound holds on scaled rows rounded by the model (exact f64 accumulation)."""
    rng = np.random.default_rng(8)
    d = 512
    u = 2.0 ** -4
    for _ in range(200):
        a = rng.standard_normal(d) * np.exp2(rng.integers(-6, 6, d))
        b = a + rng.standard_normal(d) * 0.3
        sa = np.exp2(np.floor(np.log2(447.99 / np.max(np.abs(a)))))
        sb = np.exp2(np.floor(np.log2(447.99 / np.max(np.abs(b)))))
        dot = np.dot(a * sa, b * sb)
        dot8 = np.dot(e4m3_rne(a * sa), e4m3_rne(b * sb))
        lim = (2 * u + u * u + 2 * (1 + u) * np.sqrt(d) * 2.0 ** -10 / 224.0) * np.linalg.norm(a * sa) * np.linalg.norm(b * sb)
        assert abs(dot8 - dot) <= lim
