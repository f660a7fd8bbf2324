"""The fixed-point helpers of the deterministic backward (pf3plat_b200/csrc/gs_det.cuh), compiled for the host with nvcc:
no GPU needed.  Terms spanning the documented range (2^-80 resolution, |term| < 2^45), both signs, are summed in many
random orders; the limbs must come out identical, and the decoded value must be the exact sum of the rounded terms
(fractions.Fraction) rounded once to float.  NaN, Inf and out-of-range terms must poison."""
import os
import shutil
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pf3plat_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

E, RANGE_LOG2, MAX_TERMS = 80, 45, 2 ** 21

# stdin: "N K", N lines "bits count" (the term as float bits in hex, repeated count times), K lines of N indices (an
# order of the N entries).  stdout, per order: the three limbs, the poison flag and the decoded float's bits.
_PROGRAM = r"""
#include <cstdio>
#include <vector>
#include "gs_det.cuh"
int main() {
    int n, k;
    if (scanf("%d %d", &n, &k) != 2) return 1;
    std::vector<unsigned> bits(n);
    std::vector<long long> count(n);
    for (int i = 0; i < n; i++) if (scanf("%x %lld", &bits[i], &count[i]) != 2) return 1;
    for (int o = 0; o < k; o++) {
        long long acc[GS_DET_LIMBS] = {0, 0, 0};
        bool poison = false;
        for (int j = 0; j < n; j++) {
            int i;
            if (scanf("%d", &i) != 1) return 1;
            long long limb[GS_DET_LIMBS];
            if (!gs_det_encode(gs_det_u2f(bits[i]), limb)) { poison = true; continue; }
            for (long long r = 0; r < count[i]; r++)   // the 64-bit adds the device does with RED.ADD.64 (wrapping)
                for (int l = 0; l < GS_DET_LIMBS; l++)
                    acc[l] = (long long)((unsigned long long)acc[l] + (unsigned long long)limb[l]);
        }
        printf("%lld %lld %lld %d %08x\n", acc[0], acc[1], acc[2], (int)poison, gs_det_f2u(gs_det_decode(acc, poison)));
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def det_prog(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("det")
    src = d / "det_host.cu"
    src.write_text(_PROGRAM)
    exe = d / "det_host"
    subprocess.run([NVCC, "-std=c++17", "-O2", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


def _bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _float(b: int) -> float:
    return struct.unpack("<f", struct.pack("<I", b))[0]


def _run(exe, terms, orders, counts=None):
    counts = counts or [1] * len(terms)
    lines = [f"{len(terms)} {len(orders)}"] + [f"{_bits(t):08x} {c}" for t, c in zip(terms, counts)]
    lines += [" ".join(map(str, o)) for o in orders]
    out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    rows = [r.split() for r in out.strip().splitlines()]
    return [(tuple(int(x) for x in r[:3]), bool(int(r[3])), _float(int(r[4], 16))) for r in rows]


def _rounded(t: float) -> Fraction:
    """The term as the encoder holds it: round(t * 2^80) (ties to even) * 2^-80."""
    return Fraction(round(Fraction(t) * 2 ** E), 2 ** E)


def _terms(rng, n):
    """float32 terms with exponents across the whole range (and below the resolution), both signs."""
    exps = rng.integers(-90, RANGE_LOG2, n)
    mant = rng.uniform(1.0, 2.0, n)
    sign = rng.choice([-1.0, 1.0], n)
    t = (sign * mant * np.exp2(exps.astype(np.float64))).astype(np.float32)
    t = t[np.abs(t.astype(np.float64)) < 2.0 ** RANGE_LOG2]
    return [float(x) for x in t] + [0.0, -0.0, 2.0 ** -80, -(2.0 ** -81), 2.0 ** -81 * 3, 1e-45, -1e-45]


def test_sums_are_order_independent_and_exactly_rounded(det_prog):
    rng = np.random.default_rng(0)
    for trial in range(4):
        terms = _terms(rng, 3000)
        n = len(terms)
        orders = [list(range(n)), list(range(n))[::-1]] + [list(rng.permutation(n)) for _ in range(14)]
        res = _run(det_prog, terms, orders)
        assert all(r == res[0] for r in res), f"trial {trial}: limbs differ between orders"
        limbs, poison, got = res[0]
        assert not poison
        exact = sum((_rounded(t) for t in terms), Fraction(0))
        assert (limbs[0] + limbs[1] * 2 ** 42 + limbs[2] * 2 ** 84) == exact * 2 ** E
        # the reference is the single rounding of the exact fraction (np.float32(float(x)) would round twice)
        assert got == _round_once(exact), (trial, got, float(exact))


def _round_once(x: Fraction) -> float:
    """x rounded to the nearest float32, ties to even, in exact arithmetic."""
    if x == 0:
        return 0.0
    sign = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (e - 23)                 # every sum here is a normal float32 (>= 2^-80)
    return sign * float(round(a / ulp) * ulp)


def test_cancellation_and_single_terms(det_prog):
    # large terms that cancel leave the small ones exact; a single term decodes to itself (it is already a float)
    f32 = lambda x: float(np.float32(x))
    terms = [2.0 ** 44 * 1.5, f32(3.0e-7), -(2.0 ** 44) * 1.5, 2.0 ** -70, -1.0]
    (limbs, poison, got), = _run(det_prog, terms, [list(range(5))])
    assert got == _round_once(sum((_rounded(t) for t in terms), Fraction(0)))
    for t in [1.0, -1.0, f32(3.0e-7), f32(1e13), -(2.0 ** -80), float(np.nextafter(np.float32(2.0 ** 45), 0))]:
        (_, _, got), = _run(det_prog, [t], [[0]])
        assert got == t, t
    # below half the resolution a term contributes nothing; exactly half rounds to even (0)
    (limbs, _, got), = _run(det_prog, [2.0 ** -82, 2.0 ** -81], [[0, 1]])
    assert limbs == (0, 0, 0) and got == 0.0


def test_headroom_of_the_documented_term_count(det_prog):
    # 2^21 - 1 terms of the largest magnitude in range, of either sign: no limb overflows
    big = float(np.nextafter(np.float32(2.0 ** RANGE_LOG2), 0))
    for s in (1.0, -1.0):
        (limbs, poison, got), = _run(det_prog, [s * big], [[0]], counts=[MAX_TERMS - 1])
        exact = Fraction(s * big) * (MAX_TERMS - 1)
        assert not poison and got == _round_once(exact)
    # mixed magnitudes and signs at the term limit, two orders
    terms = [big, -big / 3, 2.0 ** -60, -(2.0 ** 20) - 0.5]
    counts = [MAX_TERMS // 4] * 4
    res = _run(det_prog, terms, [[0, 1, 2, 3], [3, 2, 1, 0]], counts=counts)
    assert res[0] == res[1]
    exact = sum((_rounded(np.float32(t).item()) * c for t, c in zip(terms, counts)), Fraction(0))
    assert res[0][2] == _round_once(exact)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf"), 2.0 ** 45, -(2.0 ** 45), 1e30])
def test_non_finite_and_out_of_range_terms_poison(det_prog, bad):
    terms = [1.0, bad, -3.5]
    res = _run(det_prog, terms, [[0, 1, 2], [2, 1, 0]])
    for limbs, poison, got in res:
        assert poison and np.isnan(got)
        assert limbs == res[0][0]
        # the poisoned term added nothing: the limbs hold the finite terms alone
        assert limbs[0] + limbs[1] * 2 ** 42 + limbs[2] * 2 ** 84 == Fraction(-2.5) * 2 ** E
