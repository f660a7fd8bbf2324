"""Which copy path each CTA of the Gaussian head takes, restated on the CPU, and a check that the shape list of
tests/test_gpu_gaussian_head_regimes.py reaches every path at every d_sh; ABI refusals at the batch and frame limits.

In csrc/gs_gaussian_head.cu, CTA x of camera y = 2 scene + slot holds pixels px0 = 128 x .. px0 + n - 1, n = min(128,
hw - px0), and Gaussians first = y hw + px0 onwards.  `store_block` writes a block of `count` floats (3 n means, 9 n
covariances, 3 d_sh n harmonics) by one bulk TMA store when the destination and the byte count are both 16-byte
aligned, by a coalesced loop otherwise; `bulk_in` loads the 3 d_sh n floats of dL/dharmonics the same way.  The
outputs come from the caching allocator (aligned); the cotangent's base may be anywhere a caller's tensor starts."""
import ctypes

import pytest

from tests.test_gpu_gaussian_head_regimes import SHAPES

TMA, LOOP = "tma", "loop"
D_SH = (1, 4, 9, 16, 25)


def _aligned(byte_offset, count):
    return byte_offset % 16 == 0 and (count * 4) % 16 == 0


def cta_paths(b, h, w, d_sh, cot_offset_bytes=0):
    """one dict per CTA: n, whether the CTA is full, and TMA or LOOP for the means, covariance and harmonics stores and
    the dL/dharmonics load (whose base lies cot_offset_bytes past a 16-byte boundary)"""
    hw, HS = h * w, 3 * d_sh
    out = []
    for cam in range(2 * b):
        for x in range((hw + 127) // 128):
            px0 = 128 * x
            n = min(128, hw - px0)
            first = cam * hw + px0
            out.append({
                "n": n, "full": n == 128,
                "means": TMA if _aligned(first * 3 * 4, n * 3) else LOOP,
                "cov": TMA if _aligned(first * 9 * 4, n * 9) else LOOP,
                "harm": TMA if _aligned(first * HS * 4, n * HS) else LOOP,
                "load": TMA if _aligned(cot_offset_bytes + first * HS * 4, n * HS) else LOOP,
                # the load's two conditions apart: the byte count alone, and the address alone
                "size_ok": (n * HS * 4) % 16 == 0, "ptr_ok": (cot_offset_bytes + first * HS * 4) % 16 == 0,
            })
    return out


def test_the_predicate_on_hand_worked_cases():
    # 1 x 1, d_sh 1: a single Gaussian per camera; 3, 9 and 3 floats never make 16 bytes: every path loops
    for p in cta_paths(2, 1, 1, 1):
        assert (p["means"], p["cov"], p["harm"], p["load"]) == (LOOP,) * 4
    # 8 x 16 = one full CTA per camera, every block a multiple of 16 bytes: all TMA, misaligned cotangent loops
    assert all(p["means"] == p["cov"] == p["harm"] == p["load"] == TMA for p in cta_paths(3, 8, 16, 25))
    assert all(p["load"] == LOOP and p["size_ok"] for p in cta_paths(3, 8, 16, 25, cot_offset_bytes=4))
    # hw = 129, d_sh 9: camera 0's full CTA is aligned, camera 1's full CTA starts at Gaussian 129: loops
    ps = cta_paths(1, 1, 129, 9)
    assert [(p["n"], p["means"], p["load"]) for p in ps] == [(128, TMA, TMA), (1, LOOP, LOOP), (128, LOOP, LOOP),
                                                             (1, LOOP, LOOP)]
    # d_sh 4 and 16: 3 d_sh is a multiple of 4, so the harmonics store is always TMA on an aligned output
    for d in (4, 16):
        assert all(p["harm"] == TMA for p in cta_paths(2, 3, 7, d))


def reached(d_sh):
    got = set()
    for b, V, h, w, deg, off in SHAPES:
        if (deg + 1) ** 2 != d_sh:
            continue
        for p in cta_paths(b, h, w, d_sh, 4 * off):
            for k in ("means", "cov", "harm"):
                got.add((k, p[k]))
            got.add(("load", p["load"], "full" if p["full"] else "partial"))
            if p["load"] == LOOP and p["size_ok"] and not p["ptr_ok"]:
                got.add(("load loop on the address alone",))
    return got


@pytest.mark.parametrize("d_sh", D_SH)
def test_the_gpu_shape_list_reaches_every_path(d_sh):
    got = reached(d_sh)
    want = {("means", TMA), ("means", LOOP), ("cov", TMA), ("cov", LOOP), ("harm", TMA),
            ("load", LOOP, "full"), ("load", LOOP, "partial"), ("load", TMA, "partial"),
            ("load loop on the address alone",)}
    if d_sh % 2:  # for d_sh 4 and 16 the aligned output never takes the harmonics loop (see above)
        want.add(("harm", LOOP))
    assert want <= got, sorted(want - got)


def test_the_gpu_shape_list_holds_the_issue_shapes():
    hws = {h * w for b, V, h, w, deg, off in SHAPES}
    assert {127, 128, 129, 257} <= hws
    assert any(h == w == 1 for _, _, h, w, _, _ in SHAPES)
    assert any(h == 1 and w > 1 for _, _, h, w, _, _ in SHAPES) and any(w == 1 and h > 1 for _, _, h, w, _, _ in SHAPES)
    for deg in range(5):
        assert {h * w % 4 for _, _, h, w, dg, _ in SHAPES if dg == deg} >= {1, 2, 3}, deg
    assert {6, 16} <= {V for _, V, *_ in SHAPES} and max(b for b, *_ in SHAPES) >= 64


def test_abi_refuses_the_batch_and_frame_limits_without_a_device():
    from pf3plat_b200 import _capi
    L = _capi.lib()

    def cfg(**kw):
        a = dict(batch=1, views=2, height=4, width=4, d_sh=1, scale_min=0.5, scale_max=15.0, eps=1e-8)
        a.update(kw)
        return _capi.GsGaussianHeadConfig(**a)

    def scratch(**kw):
        return L.gs_gaussian_head_scratch_bytes(ctypes.byref(cfg(**kw)))

    # the largest accepted batch (grid.y = 2 b <= 65535) and frame, then one past each
    assert scratch(batch=32767, height=1, width=1) == 32767 * 2 * 1 * 12 * 4
    assert scratch(batch=32768, height=1, width=1) == -1
    assert scratch(height=1 << 14, width=1 << 14) == 2 * ((1 << 28) // 128) * 12 * 4
    assert scratch(height=(1 << 14) + 1, width=1 << 14) == -1
    assert scratch(height=1, width=(1 << 28) + 1) == -1
    ins, out = _capi.GsGaussianHeadInputs(), _capi.GsGaussianHeadOutputs()
    gout, gin = _capi.GsGaussianHeadOutGrads(), _capi.GsGaussianHeadInGrads()
    for bad in (cfg(batch=32768), cfg(height=(1 << 14) + 1, width=1 << 14)):
        assert L.gs_gaussian_head_forward(ctypes.byref(bad), ctypes.byref(ins), ctypes.byref(out), None) == -1
        assert b"batch in [1, 32767]" in L.gs_last_error()
        assert L.gs_gaussian_head_backward(ctypes.byref(bad), ctypes.byref(ins), ctypes.byref(gout),
                                           ctypes.byref(gin), None) == -1
        assert b"batch in [1, 32767]" in L.gs_last_error()
