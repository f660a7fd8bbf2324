"""GPU tests of the plane-sweep cost volume (csrc/gs_costvolume.cu) in the regimes tests/test_gpu_costvolume.py does not
reach, against the fp64 oracle (tests/costvolume_oracle.py) run on the device:

  * feature widths past the kernels' first 256-channel pass, ragged ones included (the forward's read-modify-write of
    the cost, the backward's per-pass G1 rows and its re-walk of the source scatter);
  * five to eight views (the source rotation (vi + s) mod v and the 1 / (v - 1) mean);
  * NaN and +-Inf at channels beyond the first 32-bit poison word and beyond the first pass, in the target role and in
    the sampled source role, and under a cotangent that is zero on whole rows;
  * a scatter that puts 2 088 960 terms on each of four elements, just under the fixed-point limbs' headroom of 2^21;
  * the deterministic term limit seen from Python, and terms beyond the limbs' range of 2^45;
  * scenes computed alone against their rows of a batched call, bit for bit.

Tolerances are those of tests/test_gpu_costvolume.py: 1e-4 on values and 1e-3 on gradients, element-wise, with the same
non-finite elements."""
import itertools
import math

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from pf3plat_b200.costvolume import plane_sweep_cost_volume
from tests import costvolume_oracle as O
from tests.test_gpu_costvolume import (DEV, GRAD_RTOL, VALUE_RTOL, oracle_per_scene, reference_ops, run, seeded_case,
                                       worst_ratio)

pytestmark = pytest.mark.gpu
U = 2.0 ** -24  # unit roundoff of float32


def oracle_ratios(cost, grad, ov, og, deterministic):
    """worst ratios (value, gradient) against the oracle.  In deterministic mode an infinite gradient term decodes to
    NaN (DESIGN.md 5.11), so there the gradient must match the oracle's finiteness rather than its NaN / Inf pattern."""
    if deterministic:
        fin = torch.isfinite(og)
        assert torch.equal(torch.isfinite(grad), fin), "deterministic gradient: finiteness differs from the oracle"
        og = torch.where(fin, og, grad.double())
    return worst_ratio(cost, ov, VALUE_RTOL, "value vs oracle"), worst_ratio(grad, og, GRAD_RTOL, "grad vs oracle")


def split_ratio(got, want, rtol, what, big):
    """worst_ratio over the elements in `big` and over the rest separately, so that a few huge elements do not set the
    floor for all the others"""
    return max(worst_ratio(got[m], want[m], rtol, what) for m in (big, ~big) if bool(m.any()))


def coordinates(f, K, E, near, far, D):
    """the oracle's sample coordinates for each source slot: (ix, iy), each [(v b), D, h*w], fp64 on the CPU"""
    h, w = f.shape[-2:]
    Kd = O.unnormalised_intrinsics(K.double().cpu(), h, w)
    depth = O.depth_candidates(near.double().cpu(), far.double().cpu(), D)
    return [O.sample_coordinates(Kd, p, depth, h, w) for p in O.relative_poses(E.double().cpu())]


def taps(ix, iy, h, w):
    """the four bilinear taps of every sample: [(row, pixel index, weight, in bounds)], each [(v b), D, h*w]"""
    x0, y0 = torch.floor(ix), torch.floor(iy)
    out = []
    for tx, ty, wt in ((x0, y0, (x0 + 1 - ix) * (y0 + 1 - iy)), (x0 + 1, y0, (ix - x0) * (y0 + 1 - iy)),
                       (x0, y0 + 1, (x0 + 1 - ix) * (iy - y0)), (x0 + 1, y0 + 1, (ix - x0) * (iy - y0))):
        inb = (tx >= 0) & (tx <= w - 1) & (ty >= 0) & (ty <= h - 1)
        out.append((torch.where(inb, ty * w + tx, torch.zeros_like(tx)).long(), wt, inb))
    return out


def with_4x4(K):
    K4 = torch.eye(4, device=K.device).repeat(*K.shape[:2], 1, 1)
    K4[..., :3, :3] = K
    return K4


# ---- 1. channel widths: later passes, ragged float4 padding ----

WIDTHS = [(2, C) for C in (5, 130, 256, 257, 300, 512, 771)] + [(3, 257), (3, 512)]


@pytest.mark.parametrize("v,C", WIDTHS, ids=[f"v{v}_c{C}" for v, C in WIDTHS])
def test_channel_widths(v, C):
    f, K, E, near, far, D, cot = seeded_case(2, v, C, 24, 32, 16, seed=1000 * v + C)
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    c0, g0 = run(f, K, E, near, far, D, cot)
    c1, g1 = run(f, K, E, near, far, D, cot, deterministic=True)
    c2, g2 = run(f, K, E, near, far, D, cot, deterministic=True)
    assert torch.equal(c0, c1) and torch.equal(c1, c2), "the forward differs between modes"
    assert torch.equal(g1, g2), "the deterministic gradient differs between two runs"
    r = [*oracle_ratios(c0, g0, ov, og, False), *oracle_ratios(c1, g1, ov, og, True)]
    print(f"v={v} C={C} (Cp4={(C + 3) // 4}): worst ratios default value {r[0]:.3f} grad {r[1]:.3f}, "
          f"deterministic value {r[2]:.3f} grad {r[3]:.3f}")
    assert max(r) <= 1.0, r


# ---- 2. five to eight views ----

VIEWS = [(5, 1, 7, 3), (5, 3, 64, 4), (6, 1, 64, 3), (6, 3, 7, 4), (8, 1, 64, 4), (8, 3, 7, 3)]  # v, b, C, K rows


@pytest.mark.parametrize("v,b,C,rows", VIEWS, ids=[f"v{v}_b{b}_c{C}_k{r}" for v, b, C, r in VIEWS])
def test_many_views(v, b, C, rows):
    f, K, E, near, far, D, cot = seeded_case(b, v, C, 20, 24, 8, seed=100 * v + 10 * b + C)
    assert len(torch.unique(near)) == b * v and len(torch.unique(far)) == b * v
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    Kin = with_4x4(K) if rows == 4 else K
    r = []
    for det in (False, True):
        r += oracle_ratios(*run(f, Kin, E, near, far, D, cot, deterministic=det), ov, og, det)
    print(f"v={v} b={b} C={C} K {rows}x{rows}: worst ratios default value {r[0]:.3f} grad {r[1]:.3f}, "
          f"deterministic value {r[2]:.3f} grad {r[3]:.3f}")
    assert max(r) <= 1.0, r


# ---- 3. non-finite features past the first poison word and the first pass ----

def zoom_case(C, h, w, D, seed):
    """v = 2, b = 1.  View 1 sits one unit behind view 0 on the optical axis and the depth range [0.2, 0.45] lies in
    front of view 0.  View 0's samples land in the middle of view 1; every sample of view 1 lies behind view 0's camera,
    is divided by 1e-3 and falls far outside the image.  So view 1's gradient is the source role alone (the scatter)
    and view 0's is the feat01 role alone (the G1 rows)."""
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(1, 2, C, h, w, generator=g)
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]]).repeat(1, 2, 1, 1)
    E = torch.eye(4).repeat(1, 2, 1, 1)
    E[0, 1, 2, 3] = -1.0
    near, far = torch.full((1, 2), 0.2), torch.full((1, 2), 0.45)
    cot = torch.randn(2, D, h, w, generator=g)
    return [t.to(DEV) for t in (f, K, E, near, far)] + [D, cot.to(DEV)]


NONFINITE = list(itertools.product((math.nan, math.inf, -math.inf), (33, 255, 256, 299)))


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("role", ["target", "source", "target_zero_cotangent"])
def test_nonfinite_past_the_first_word_and_pass(role, deterministic):
    C, h, w, D = 300, 24, 32, 8
    f, K, E, near, far, D, cot = zoom_case(C, h, w, D, seed=41)
    (ix, iy), = coordinates(f, K, E, near, far, D)
    inb = [t[2] for t in taps(ix, iy, h, w)]
    assert not any(bool(m[1].any()) for m in inb), "a sample of view 1 is in bounds"
    assert all(bool(m[0].all()) for m in inb), "a tap of view 0's samples is out of bounds"
    g = torch.Generator().manual_seed(7)
    if role == "source":  # pixels of view 1 that view 0's samples read
        tapped = torch.zeros(h * w, dtype=torch.bool)
        for idx, _, m in taps(ix, iy, h, w):
            tapped[idx[0][m[0]]] = True
        pool = torch.nonzero(tapped).flatten()
        view = 1
    else:  # pixels of view 0, whose own samples all land in view 1
        pool, view = torch.arange(h * w), 0
    assert len(pool) >= len(NONFINITE)
    pix = pool[torch.randperm(len(pool), generator=g)[:len(NONFINITE)]].tolist()
    for p, (val, ch) in zip(pix, NONFINITE):
        f[0, view, ch, p // w, p % w] = val
    if role == "target_zero_cotangent":
        cot[0] = 0.0  # view 0's rows: every source-role term is 0 x feat01, NaN where feat01 is not finite
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    # the regime: non-finite gradients at every one of the channels, in the view the role sends them to
    reached = 0 if role == "source" else 1  # through view 0's G1 rows, or through the scatter into view 1
    bad = {int(c) for c in torch.nonzero(~torch.isfinite(og[0, reached]))[:, 0]}
    assert bad == {33, 255, 256, 299}, bad
    assert not torch.isfinite(ov).all()
    cost, grad = run(f, K, E, near, far, D, cot, deterministic=deterministic)
    r = oracle_ratios(cost, grad, ov, og, deterministic)
    print(f"{role} det={deterministic}: {int((~torch.isfinite(og)).sum())} non-finite gradients, "
          f"{int((~torch.isfinite(ov)).sum())} non-finite values; worst ratios value {r[0]:.3f} grad {r[1]:.3f}")
    assert max(r) <= 1.0, r


# ---- 4. a scatter concentrated at the limbs' headroom ----

def concentrated_case(C, sign, seed):
    """b = 1, v = 2, 256 x 255, D = 32.  View 1 sits one unit behind view 0; focal length 1 px, principal point
    (100.45, 80.45) px, depths in [1e-4, 2e-4].  Every sample of view 0 lands in the cell [100, 101) x [80, 81) of
    view 1, so each of that cell's four pixels is a tap of all D h w = 2 088 960 samples; every sample of view 1 is
    behind view 0's camera and lands near x = -1e5.  Features in [12, 16], cotangent sign x [16, 64]."""
    b, v, h, w, D = 1, 2, 256, 255, 32
    g = torch.Generator().manual_seed(seed)
    K = torch.zeros(b, v, 3, 3)
    K[..., 0, 0], K[..., 0, 2] = 1.0 / w, 100.45 / w
    K[..., 1, 1], K[..., 1, 2] = 1.0 / h, 80.45 / h
    K[..., 2, 2] = 1.0
    E = torch.eye(4).repeat(b, v, 1, 1)
    E[0, 1, 2, 3] = -1.0
    near, far = torch.full((b, v), 1e-4), torch.full((b, v), 2e-4)
    f = 12.0 + 4.0 * torch.rand(b, v, C, h, w, generator=g)
    cot = sign * (16.0 + 48.0 * torch.rand(v * b, D, h, w, generator=g))
    return [t.to(DEV) for t in (f, K, E, near, far)] + [D, cot.to(DEV)]


@pytest.mark.parametrize("sign", [1.0, -1.0], ids=["positive", "negative"])
def test_concentrated_scatter_at_the_limbs_headroom(sign):
    """Each of the four cell pixels of view 1 receives one source-role term per sample of view 0, and nothing else:
    view 1's own samples are all out of bounds, so its feat01 role there is exactly 0.

    Bound of the deterministic path.  A term is t = fl(w fl(gd fl(f01 ...))) with gd = fl(fl(dL/dcost) scale) and
    scale = fl(1 / sqrt(C) / (v - 1)): at most five float32 roundings (scale, gd, gd f01, the weight w rounded from
    fp64, w gs), so |t - t*| <= ((1 + u)^5 - 1) |t*| against the exact term t*, with u = 2^-24.  At C = 4 and v = 2
    the scale is 1/2 and gd is exact, which leaves three.  The fixed-point encoding of a term in [2^4, 2^10] is exact
    (resolution 2^-80, range 2^45), the integer sum is exact (2 088 960 < 2^21 terms: no limb overflows), and decoding
    rounds once.  All terms have the same sign, so sum |t - t*| <= ((1 + u)^5 - 1) |sum t*|, and the decoded sum is
    within (1 + u)^6 - 1 < 8 u of the exact one.  The fp64 oracle's own error (2^21 fp64 additions, about 2^-32
    relative) and the fp64 projection's (about 1e-13 on a weight of at least 0.18) are far below that."""
    C = 4
    f, K, E, near, far, D, cot = concentrated_case(C, sign, seed=11)
    h, w = f.shape[-2:]
    (ix, iy), = coordinates(f, K, E, near, far, D)
    assert bool((torch.floor(ix[0]) == 100).all()) and bool((torch.floor(iy[0]) == 80).all())
    assert float(ix[1].max()) < -1e4
    terms = D * h * w
    assert terms == 2088960 and terms < 2 ** 21
    # terms between 2^4 and 2^10: w in [wmin, wmax], |gd| = |cot| / 2 in [8, 32], f01 in [12, 16]
    ax, ay = ix[0] - 100.0, iy[0] - 80.0
    wmin = float((torch.minimum(ax, 1 - ax) * torch.minimum(ay, 1 - ay)).min())
    wmax = float((torch.maximum(ax, 1 - ax) * torch.maximum(ay, 1 - ay)).max())
    assert wmin * 8 * 12 >= 2 ** 4 and wmax * 32 * 16 <= 2 ** 10, (wmin, wmax)
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    cell = torch.tensor([80 * w + 100, 80 * w + 101, 81 * w + 100, 81 * w + 101], device=DEV)
    want = og[0, 1].reshape(C, -1)[:, cell]
    assert bool(((want * sign) > 0).all())
    dets = [run(f, K, E, near, far, D, cot, deterministic=True) for _ in range(3)]
    assert all(torch.equal(dets[0][0], c) and torch.equal(dets[0][1], g) for c, g in dets[1:]), \
        "deterministic runs differ"
    c0, g0 = run(f, K, E, near, far, D, cot)
    fr = f.detach().clone().requires_grad_(True)
    (gref,) = torch.autograd.grad(reference_ops(fr, K, E, near, far, D), fr, cot)
    rel = lambda g: float(((g[0, 1].reshape(C, -1)[:, cell].double() - want).abs() / want.abs()).max())
    r_det, r_def, r_ref = rel(dets[0][1]), rel(g0), rel(gref)
    rest = torch.ones(C, h * w, dtype=torch.bool, device=DEV)
    rest[:, cell] = False
    r = [worst_ratio(dets[0][0], ov, VALUE_RTOL, "value"), worst_ratio(c0, ov, VALUE_RTOL, "value")]
    for g in (dets[0][1], g0):
        r.append(worst_ratio(g[:, 0], og[:, 0], GRAD_RTOL, "view 0 (feat01 role)"))
        assert bool((g[0, 1].reshape(C, -1)[rest] == 0).all()) and bool((og[0, 1].reshape(C, -1)[rest] == 0).all())
    print(f"concentrated scatter ({terms} terms per element, sign {sign:+.0f}): relative error at the cell, "
          f"deterministic {r_det:.3e} ({r_det / U:.2f} u), default {r_def:.3e}, PyTorch's float32 ops {r_ref:.3e}; "
          f"worst ratios values {r[0]:.3f} / {r[1]:.3f}, view 0 grad {r[2]:.3f} / {r[3]:.3f}")
    assert r_det <= 8 * U, r_det
    assert r_def <= GRAD_RTOL, (r_def, r_ref)
    assert max(r) <= 1.0, r


# ---- 5. the deterministic term limit from Python ----

def launched(fn):
    """names of the device kernels `fn` launches, and the exception it raised (or None)"""
    err = None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        try:
            fn()
        except Exception as e:  # returned to the caller, which checks its type
            err = e
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages()}, err


def test_deterministic_limit_from_python():
    """(v - 1) D h w = 2^21 terms can reach one element: one more than the limbs hold.  The forward does not use them,
    the deterministic backward refuses the call before any launch, and the default backward is unaffected."""
    f, K, E, near, far, D, cot = seeded_case(1, 2, 4, 256, 256, 32, seed=21)
    assert (2 - 1) * D * 256 * 256 == 2 ** 21
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    costs = []
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            costs.append(plane_sweep_cost_volume(f, K, E, near, far, D))
        finally:
            torch.use_deterministic_algorithms(False)
    assert torch.equal(costs[0], costs[1])
    fr = f.detach().clone().requires_grad_(True)
    cost = plane_sweep_cost_volume(fr, K, E, near, far, D)
    torch.cuda.synchronize()

    def det_backward():
        torch.use_deterministic_algorithms(True)
        try:
            torch.autograd.grad(cost, fr, cot, retain_graph=True)
        finally:
            torch.use_deterministic_algorithms(False)

    names, err = launched(det_backward)
    assert isinstance(err, ValueError), err
    assert not any("k_cv" in n for n in names), names
    out = {}
    names, err = launched(lambda: out.setdefault("g", torch.autograd.grad(cost, fr, cot)[0]))
    assert err is None and any("k_cv_backward" in n for n in names), names  # the profiler does see the kernels
    r = [worst_ratio(costs[0], ov, VALUE_RTOL, "value"), worst_ratio(out["g"], og, GRAD_RTOL, "grad")]
    print(f"(v - 1) D h w = 2^21: deterministic backward refused; worst ratios value {r[0]:.3f}, default grad {r[1]:.3f}")
    assert max(r) <= 1.0, r


# ---- 6. terms beyond the limbs' range ----

@pytest.mark.parametrize("deterministic", [False, True])
def test_terms_beyond_the_fixed_point_range(deterministic):
    """The identity pose of the golden case v2_identity, made exact: identical cameras, intrinsics with power-of-two
    entries (K = [[8, 0, 8], [0, 4, 4], [0, 0, 1]] px) and depths 1 and 4, so that every sample lands exactly on its
    own pixel in the kernel's fp64 and the oracle's alike, and every tap weight is exactly 1 or 0.  (With a weight of
    1e-16 rather than 0, the round-off that sets it, which the two compute differently, would be multiplied by 2^46.)
    One target pixel of view 0 gets 2^44 in channel 2 and a cotangent of 8 on all its rows, so (scale 1/2) its
    source-role term on the weight-1 tap is 2^46, beyond the limbs' range of 2^45.  The default path adds it in float;
    the deterministic one poisons exactly the elements that receive such a term."""
    b, v, C, h, w, D = 1, 2, 4, 8, 16, 2
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=31)
    K[:] = torch.tensor([[0.5, 0.0, 0.5], [0.0, 0.5, 0.5], [0.0, 0.0, 1.0]], device=DEV)
    E[:] = torch.eye(4, device=DEV)
    near[:], far[:] = 1.0, 4.0
    py, px, ch = 5, 7, 2
    f[0, 0, ch, py, px] = 2.0 ** 44
    cot[0, :, py, px] = 8.0
    (ix, iy), = coordinates(f, K, E, near, far, D)
    xs = torch.arange(w, dtype=torch.float64).repeat(h)
    ys = torch.arange(h, dtype=torch.float64).repeat_interleave(w)
    assert torch.equal(ix, xs.expand_as(ix)) and torch.equal(iy, ys.expand_as(iy))
    p = py * w + px
    poisoned = torch.zeros(b, v, C, h * w, dtype=torch.bool)
    for idx, wt, m in taps(ix, iy, h, w):
        sel = m[0, :, p]
        assert bool(((wt[0, :, p][sel] == 1) | (wt[0, :, p][sel] == 0)).all())
        poisoned[0, 1, ch, idx[0, :, p][sel & (wt[0, :, p] > 0.5)]] = True
    poisoned = poisoned.reshape(b, v, C, h, w).to(DEV)
    assert int(poisoned.sum()) == 1
    ov, og = oracle_per_scene(f, K, E, near, far, D, cot)
    assert bool(torch.isfinite(og).all()) and float(og[poisoned].abs().min()) >= 2 ** 45
    cost, grad = run(f, K, E, near, far, D, cot, deterministic=deterministic)
    big_v, big_g = ov.abs() > 1e6, og.abs() > 1e6
    rv = split_ratio(cost, ov, VALUE_RTOL, "value", big_v)
    if deterministic:
        assert torch.equal(torch.isnan(grad), poisoned) and bool(torch.isfinite(grad[~poisoned]).all())
        rg = split_ratio(grad[~poisoned], og[~poisoned], GRAD_RTOL, "grad", big_g[~poisoned])
    else:
        assert bool(torch.isfinite(grad).all())
        rg = split_ratio(grad, og, GRAD_RTOL, "grad", big_g)
    print(f"terms beyond 2^45 det={deterministic}: {int(poisoned.sum())} poisoned element(s); worst ratios value "
          f"{rv:.3f}, grad {rg:.3f}")
    assert max(rv, rg) <= 1.0, (rv, rg)


# ---- 7. scene independence ----

def test_scenes_alone_match_their_rows_of_the_batch():
    b, v, C, h, w, D = 5, 3, 40, 20, 24, 8
    f, K, E, near, far, D, cot = seeded_case(b, v, C, h, w, D, seed=51)
    batched = {det: run(f, K, E, near, far, D, cot, deterministic=det) for det in (False, True)}
    for i in range(b):
        rows = [vi * b + i for vi in range(v)]
        one = lambda t: t[i:i + 1]
        for det in (False, True):
            c1, g1 = run(one(f), one(K), one(E), one(near), one(far), D, cot[rows], deterministic=det)
            assert torch.equal(c1, batched[det][0][rows]), (i, det)
            if det:
                assert torch.equal(g1, batched[det][1][i:i + 1]), i
    assert not torch.equal(batched[True][0][0], batched[True][0][1])
    print(f"b={b} v={v} C={C}: every scene alone equals its rows of the batch, bit for bit")
