"""The Gaussian head's kernels (csrc/gs_gaussian_head.cu) past the shapes and cotangents of test_gpu_gaussian_head.py,
with every torch.empty poisoned (tests/poison.py) so that an output or gradient element a kernel leaves unwritten reads
as NaN: the training shape, every subset of the four cotangents with the input gradients that skip the finalize's
c2w or depth work, cotangents that arrive as a DC-only slice, expanded or 4 bytes off 16-byte alignment, ragged and
degenerate frames, long view lists, large batches, non-finite inputs confined to their Gaussian, and zero or
underflowing raw quaternions in the head and in the fused adapter.  Bounds as in test_gpu_gaussian_head.py: values
within 1e-5 (|ref| + 1), gradients within 1e-3 (|ref| + rms ref), the same non-finite elements.

SHAPES is the shape list whose copy paths (bulk TMA or coalesced loop for each store and for the dL/dharmonics load)
tests/test_gaussian_head_regimes_cpu.py checks, per d_sh, against a restatement of the kernels' alignment tests."""
import itertools

import numpy as np
import pytest
import torch

from pf3plat_b200.adapter import GaussianAdapterCfg
from tests import gaussian_head_oracle as O
from tests.gaussian_head_route import existing_route
from tests.poison import poisoned  # noqa: F401  (fixture)
from tests.test_gaussian_head_cpu import case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ("means", "covariances", "harmonics", "opacities")

# (b, V, h, w, sh_degree, harmonics cotangent offset in floats): 1 x 1, 1 x w and h x 1 frames; hw = 127, 128, 129, 257;
# hw % 4 in {1, 2, 3} at every d_sh; 6 and 16 views; 64 scenes; and at every d_sh a cotangent 4 bytes off alignment on
# a frame with a full and a partial CTA per camera
SHAPES = [
    (1, 2, 1, 1, 0, 0), (2, 3, 1, 13, 1, 0), (2, 2, 11, 1, 2, 0), (1, 2, 1, 127, 3, 0), (2, 2, 8, 16, 4, 0),
    (1, 3, 3, 43, 0, 0), (1, 2, 257, 1, 2, 0), (2, 6, 5, 6, 3, 0), (1, 16, 3, 3, 1, 0), (64, 2, 2, 3, 4, 0),
    (2, 2, 3, 3, 0, 0), (1, 2, 2, 5, 0, 0), (1, 2, 2, 7, 1, 0), (1, 2, 3, 2, 1, 0), (1, 2, 5, 1, 2, 0),
    (2, 2, 3, 2, 2, 0), (2, 2, 1, 5, 3, 0), (1, 3, 7, 1, 3, 0), (1, 2, 3, 3, 4, 0), (2, 2, 7, 1, 4, 0),
    (1, 2, 1, 6, 4, 0), (1, 2, 2, 6, 3, 0), (1, 2, 1, 131, 4, 0), (1, 2, 2, 66, 0, 0), (2, 2, 1, 8, 1, 0),
    (1, 2, 2, 4, 2, 0), (1, 2, 1, 7, 0, 0), (2, 2, 2, 2, 4, 0), (1, 2, 3, 5, 1, 0),
    (1, 2, 10, 13, 0, 1), (1, 2, 10, 13, 1, 1), (1, 2, 10, 13, 2, 1), (1, 2, 10, 13, 3, 1), (1, 2, 10, 13, 4, 1),
]


def cfg_for(deg):
    return GaussianAdapterCfg(gaussian_scale_min=O.SCALE_MIN, gaussian_scale_max=O.SCALE_MAX, sh_degree=int(deg))


def _prep(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return got, ref


def value_ratio(got, ref):
    got, ref = _prep(got, ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isfinite(got), np.isfinite(ref))
    f = np.isfinite(ref)
    return float((np.abs(got[f] - ref[f]) / (1e-5 * (np.abs(ref[f]) + 1.0))).max(initial=0.0))


def grad_ratio(got, ref):
    got, ref = _prep(got, ref)
    assert np.array_equal(np.isfinite(got), np.isfinite(ref)), (np.argwhere(np.isfinite(got) != np.isfinite(ref))[:5])
    f = np.isfinite(ref)
    rms = float(np.sqrt((ref[f] ** 2).mean())) if f.any() else 0.0
    return float((np.abs(got[f] - ref[f]) / (1e-3 * (np.abs(ref[f]) + rms) + 1e-30)).max(initial=0.0))


def fragile_mask(c):
    """[b, G]: Gaussians with a sigmoid argument beyond float32 saturation, whose cotangents are zeroed (as
    test_gpu_gaussian_head.py does)"""
    raw = np.asarray(c["raw"], np.float64)
    b = c["c2w"].shape[0]
    h, w = raw.shape[-2:]
    big = (np.abs(raw[:, :5]) > 15).any(1) | (np.abs(np.asarray(c["logits"], np.float64)[:, 1]) > 15)
    return big.reshape(2, b, h * w).transpose(1, 0, 2).reshape(b, 2 * h * w)


def masked_cotangents(c, keys=KEYS):
    keep = ~fragile_mask(c)
    out = {}
    for k in keys:
        a = np.asarray(c["cot_" + k], np.float64)
        out[k] = a * keep.reshape(keep.shape + (1,) * (a.ndim - 2))
    return out


def seeded(b, V, h, w, deg, seed=0):
    from tests.golden.make_gaussian_head_golden import make_case
    return make_case(seed, b, V, h, w, deg)


def scenes_of(c, idx):
    """the case restricted to scenes idx (a list), in that order"""
    b, V = c["c2w"].shape[:2]
    idx = list(idx)
    out = {"sh_degree": c["sh_degree"], "c2w": c["c2w"][idx], "K": c["K"][idx],
           "depths": c["depths"].reshape(b, V, *c["depths"].shape[1:])[idx].reshape(-1, *c["depths"].shape[1:]),
           "raw": c["raw"][idx + [b + i for i in idx]], "logits": c["logits"][idx + [b + i for i in idx]]}
    for k in KEYS:
        if "cot_" + k in c:
            out["cot_" + k] = c["cot_" + k][idx]
    return out


class _Misaligned(torch.autograd.Function):
    """Identity on the harmonics; its backward hands the cotangent on as a contiguous [b, G, d_sh, 3] buffer that
    starts 4 bytes past a 16-byte boundary, seen through the harmonics' transpose, so that the op receives it at that
    address"""

    @staticmethod
    def forward(ctx, x):
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        b, G, _, d_sh = g.shape
        buf = torch.empty(g.numel() + 4, device=g.device)
        view = buf[1:1 + g.numel()].view(b, G, d_sh, 3)
        assert view.data_ptr() % 16 == 4
        view.copy_(g.transpose(-1, -2))
        return view.transpose(-1, -2)


def run_head(c, cot=None, need=O.INPUTS, harm_offset=0, layout=None):
    """values and the gradients (None where an input does not require grad) of sum_k <cot_k, out_k> over the keys of
    `cot`; layout "sum" takes out.sum() for every cotangent of ones, "dc" reads harmonics[..., 0] only"""
    from pf3plat_b200.gaussian_head import gaussian_head
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(cot is not None and k in need)
         for k in O.INPUTS}
    K = torch.tensor(np.asarray(c["K"]), dtype=torch.float32, device=DEV)
    h, w = c["raw"].shape[-2:]
    g = gaussian_head(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(c["sh_degree"]), (h, w))
    vals = {k: getattr(g, k) for k in KEYS}
    if cot is None:
        return vals, None
    outs = dict(vals)
    if harm_offset:
        outs["harmonics"] = _Misaligned.apply(outs["harmonics"])
    if layout == "sum":
        loss = sum(outs[k].sum() for k in cot)
    elif layout == "dc":
        loss = (torch.tensor(cot["harmonics"][..., 0], dtype=torch.float32, device=DEV) * outs["harmonics"][..., 0]).sum()
    else:
        loss = sum((torch.tensor(np.asarray(cot[k]), dtype=torch.float32, device=DEV) * outs[k]).sum() for k in cot)
    loss.backward()
    return vals, {k: (t[k].grad if k in need else None) for k in O.INPUTS}


def oracle(c, cot):
    """fp64 values and gradients; zeros for an input no cotangent reaches"""
    vals, grads = O.run(c, {k: cot.get(k, np.zeros_like(np.asarray(c["cot_" + k], np.float64))) for k in KEYS})
    return vals, grads


def np_(d):
    return {k: v.detach().cpu().numpy() for k, v in d.items() if v is not None}


def compare(c, cot, need=O.INPUTS, **kw):
    vals, grads = run_head(c, cot, need, **kw)
    ov, og = oracle(c, cot)
    vr = max(value_ratio(v, ov[k]) for k, v in np_(vals).items())
    gr = max((grad_ratio(g, og[k]) for k, g in np_(grads).items()), default=0.0)
    return vr, gr, vals, grads


# ---- the training shape ----

@pytest.fixture(scope="module")
def training_case():
    return seeded(14, 3, 256, 256, 4, seed=14256)


def test_training_shape(poisoned, training_case):
    c = training_case
    b, V, hw = 14, 3, 256 * 256
    cot = masked_cotangents(c)
    vals, grads = run_head(c, cot)
    torch.cuda.synchronize()
    assert poisoned.off_thread_calls() > 0  # the backward's gradients were allocated on autograd's thread, poisoned
    v, g = np_(vals), np_(grads)
    # two scenes against the oracle
    sub = scenes_of(c, [0, 13])
    ov, og = oracle(sub, masked_cotangents(sub))
    rows = [0, 13]
    item_rows = rows + [b + i for i in rows]
    vr = max(value_ratio(v[k][rows], ov[k]) for k in KEYS)
    gsub = {"raw": g["raw"][item_rows], "logits": g["logits"][item_rows],
            "depths": g["depths"].reshape(b, V, -1)[rows].reshape(-1, 1, 256, 256), "c2w": g["c2w"][rows]}
    gr = {k: grad_ratio(gsub[k], og[k]) for k in O.INPUTS}
    print(f"training shape vs oracle: values {vr:.3f}, gradients " + ", ".join(f"{k} {r:.3f}" for k, r in gr.items()))
    if gr["c2w"] > 1.0:  # the existing route's own float32 distance from fp64 at the same inputs
        t = {k: torch.tensor(np.asarray(sub[k]), dtype=torch.float32, device=DEV).requires_grad_(True) for k in O.INPUTS}
        K = torch.tensor(sub["K"], dtype=torch.float32, device=DEV)
        outs = existing_route(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(4), 256, 256)
        cs = masked_cotangents(sub)
        sum((torch.tensor(cs[k], dtype=torch.float32, device=DEV) * o).sum() for k, o in zip(KEYS, outs)).backward()
        print(f"existing route's dL/dc2w vs oracle: {grad_ratio(t['c2w'].grad.cpu().numpy(), og['c2w']):.3f}")
    assert vr <= 1.0 and max(gr.values()) <= 1.0
    # all 14 scenes against the existing route on the device
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(True) for k in O.INPUTS}
    K = torch.tensor(c["K"], dtype=torch.float32, device=DEV)
    outs = existing_route(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(4), 256, 256)
    sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * o).sum() for k, o in zip(KEYS, outs)).backward()
    rv = max(value_ratio(v[k], o.detach().cpu().numpy()) for k, o in zip(KEYS, outs))
    rg = {k: grad_ratio(g[k], t[k].grad.cpu().numpy()) for k in O.INPUTS}
    print(f"training shape vs the existing route: values {rv:.3f}, gradients "
          + ", ".join(f"{k} {r:.3f}" for k, r in rg.items()))
    assert rv <= 1.0 and max(rg.values()) <= 1.0
    del outs, t
    # scenes 0 and 13 alone: bit-identical to their rows
    for bi in (0, 13):
        one = scenes_of(c, [bi])
        vo, go = run_head(one, {k: cot[k][bi:bi + 1] for k in KEYS})
        for k in KEYS:
            assert torch.equal(vo[k], vals[k][bi:bi + 1]), k
        assert torch.equal(go["c2w"], grads["c2w"][bi:bi + 1])
        assert torch.equal(go["depths"], grads["depths"][bi * V:(bi + 1) * V])
        assert torch.equal(go["raw"], grads["raw"][[bi, b + bi]])
        assert torch.equal(go["logits"], grads["logits"][[bi, b + bi]])
    assert hw // 128 == 512


# ---- cotangent subsets ----

NEED_SUBSETS = [s for r in range(1, 5) for s in itertools.combinations(O.INPUTS, r)
                if not ("c2w" in s and "depths" in s)]
COT_SUBSETS = [s for r in range(1, 5) for s in itertools.combinations(KEYS, r)]


@pytest.mark.parametrize("cots", COT_SUBSETS, ids=["+".join(k[:4] for k in s) for s in COT_SUBSETS])
def test_every_cotangent_subset_and_input_grad_subset(poisoned, cots):
    c = seeded(2, 4, 9, 15, 2, seed=91)  # two CTAs per camera, two middle views
    cot = masked_cotangents(c, cots)
    worst = [0.0, 0.0]
    for need in NEED_SUBSETS:
        vr, gr, _, grads = compare(c, cot, need)
        worst = [max(worst[0], vr), max(worst[1], gr)]
        assert vr <= 1.0 and gr <= 1.0, need
        for k in O.INPUTS:
            assert (grads[k] is None) == (k not in need)
    assert poisoned.off_thread_calls() > 0
    print(f"cotangents {cots}: worst value ratio {worst[0]:.3f}, gradient ratio {worst[1]:.3f}")


# ---- cotangent layouts ----

@pytest.mark.parametrize("layout", ["dc", "sum"])
def test_cotangent_layouts(poisoned, layout):
    c = seeded(2, 3, 10, 13, 3, seed=92)
    if layout == "dc":
        cot = {"harmonics": masked_cotangents(c, ("harmonics",))["harmonics"]}
        ref = dict(cot)
        ref["harmonics"] = np.zeros_like(cot["harmonics"])
        ref["harmonics"][..., 0] = cot["harmonics"][..., 0]
    else:
        cot = {k: np.ones_like(np.asarray(c["cot_" + k], np.float64)) for k in KEYS}
        ref = cot
    vals, grads = run_head(c, cot, layout=layout)
    ov, og = oracle(c, ref)
    vr = max(value_ratio(v, ov[k]) for k, v in np_(vals).items())
    gr = max(grad_ratio(g, og[k]) for k, g in np_(grads).items())
    print(f"layout {layout}: value ratio {vr:.3f}, gradient ratio {gr:.3f}")
    assert vr <= 1.0 and gr <= 1.0


# ---- shapes, and the copy paths they reach ----

@pytest.mark.parametrize("b,V,h,w,deg,off", SHAPES)
def test_shapes_and_copy_paths(poisoned, b, V, h, w, deg, off):
    c = seeded(b, V, h, w, deg, seed=1000 * b + 100 * V + h * w + deg)
    cot = masked_cotangents(c)
    vals, grads = run_head(c, cot, harm_offset=off)
    ov, og = oracle(c, cot)
    vr = {k: value_ratio(v, ov[k]) for k, v in np_(vals).items()}
    gr = max(grad_ratio(g, og[k]) for k, g in np_(grads).items())
    print(f"b={b} V={V} {h}x{w} d_sh={(deg + 1) ** 2} offset={off}: value ratio {max(vr.values()):.3f}, gradient ratio "
          f"{gr:.3f}")
    assert gr <= 1.0
    over = {k: r for k, r in vr.items() if r > 1.0}
    if over:
        # On frames one pixel high or wide the pixel size 1 / h or 1 / w is 1, the Gaussians are large (covariance
        # entries ~ 200) and off-diagonal entries cancel: float32 alone lands past the bound.  Ours is then held to the
        # bound plus twice the distance of the reference's own statements run in float32.
        v32 = O.values32(c)
        for k, r in over.items():
            r32 = value_ratio(v32[k], ov[k])
            print(f"  {k}: ours {r:.3f}, the reference's float32 statements {r32:.3f} of the bound")
            assert r <= 1.0 + 2.0 * r32, k


def test_the_largest_batch(poisoned):
    b = 32767
    c = seeded(b, 2, 1, 1, 0, seed=32767)
    cot = masked_cotangents(c)
    vals, grads = run_head(c, cot)
    v, g = np_(vals), np_(grads)
    for k, a in list(v.items()) + list(g.items()):
        assert not np.isnan(a).any(), k  # clean inputs: nothing left unwritten in any scene
    rows = [0, 1, 9999, 16383, 32766]
    sub = scenes_of(c, rows)
    ov, og = oracle(sub, masked_cotangents(sub))
    item_rows = rows + [b + i for i in rows]
    vr = max(value_ratio(v[k][rows], ov[k]) for k in KEYS)
    gsub = {"raw": g["raw"][item_rows], "logits": g["logits"][item_rows],
            "depths": g["depths"].reshape(b, 2, -1)[rows].reshape(-1, 1, 1, 1), "c2w": g["c2w"][rows]}
    gr = max(grad_ratio(gsub[k], og[k]) for k in O.INPUTS)
    print(f"b = 32767: value ratio {vr:.3f}, gradient ratio {gr:.3f}")
    assert vr <= 1.0 and gr <= 1.0


# ---- non-finite confinement ----

def _gaussian_nonfinite(a, b):
    """[b, G] bool: any non-finite element of each Gaussian"""
    return ~np.isfinite(a.reshape(b, a.shape[1], -1)).all(-1)


@pytest.mark.parametrize("kind", ["nan_offset", "nan_scale", "inf_quat", "nan_sh", "inf_depth"])
def test_non_finite_is_confined(poisoned, kind):
    b, V, h, w = 3, 3, 12, 12
    c = seeded(b, V, h, w, 2, seed=93)
    cot = masked_cotangents(c)
    clean_v, clean_g = (np_(d) for d in run_head(c, cot))
    bi, s, py, px = 1, 0, 5, 7  # scene 1, slot 0 (conv item 1), pixel (5, 7)
    p = py * w + px
    c = dict(c)
    c["raw"], c["depths"] = c["raw"].copy(), c["depths"].copy()
    item = s * b + bi
    if kind == "nan_offset":
        c["raw"][item, 0, py, px] = np.nan
    elif kind == "nan_scale":
        c["raw"][item, 3, py, px] = np.nan
    elif kind == "inf_quat":
        c["raw"][item, 7, py, px] = np.inf
    elif kind == "nan_sh":
        c["raw"][item, 9 + 4, py, px] = np.nan
    else:
        c["depths"][bi * V + 0, 0, py, px] = np.inf
    vals, grads = run_head(c, cot)
    v, g = np_(vals), np_(grads)
    ov, og = oracle(c, cot)
    others = [i for i in range(b) if i != bi]
    oi = others + [b + i for i in others]
    for k in KEYS:
        assert np.array_equal(v[k][others], clean_v[k][others], equal_nan=True), k
    assert np.array_equal(g["raw"][oi], clean_g["raw"][oi]) and np.array_equal(g["logits"][oi], clean_g["logits"][oi])
    assert np.array_equal(g["c2w"][others], clean_g["c2w"][others])
    dd, cd = g["depths"].reshape(b, V, -1), clean_g["depths"].reshape(b, V, -1)
    assert np.array_equal(dd[others], cd[others])
    # within the scene: only the Gaussian at (slot s, p) and its own camera's dL/dc2w may differ from the clean run
    gauss = s * h * w + p
    keep = np.ones(2 * h * w, bool)
    keep[gauss] = False
    for k in KEYS:
        assert np.array_equal(v[k][bi, keep], clean_v[k][bi, keep]), k
    assert np.isfinite(g["c2w"][bi, V - 1]).all() and np.isfinite(g["c2w"][bi, 1:V - 1]).all()
    # Row 3 of c2w: the reference multiplies the homogeneous direction by the whole 4 x 4 and drops the fourth
    # component, so a NaN direction gives 0 * NaN = NaN in its gradient there; the head does not read row 3 and gives 0.
    assert (g["c2w"][:, :, 3] == 0).all()
    g["c2w"], og["c2w"] = g["c2w"][:, :, :3], og["c2w"][:, :, :3]
    if kind.startswith("nan"):
        for k in KEYS:
            value_ratio(v[k], ov[k])  # the same non-finite elements as the oracle
        for k in O.INPUTS:
            grad_ratio(g[k], og[k])
    else:  # which Gaussians, not which elements: an infinity's NaNs depend on the order of the covariance products
        for k in KEYS:
            assert np.array_equal(_gaussian_nonfinite(v[k], b), _gaussian_nonfinite(ov[k], b)), k
        assert np.array_equal(~np.isfinite(g["raw"]).all(1), ~np.isfinite(og["raw"]).all(1))
        assert np.array_equal(~np.isfinite(g["depths"]), ~np.isfinite(og["depths"]))
        assert np.array_equal(~np.isfinite(g["c2w"]).all((2, 3)), ~np.isfinite(og["c2w"]).all((2, 3)))
    bad = _gaussian_nonfinite(v["means"], b) | _gaussian_nonfinite(v["covariances"], b) | \
        _gaussian_nonfinite(v["harmonics"], b)
    assert set(map(tuple, np.argwhere(bad))) <= {(bi, gauss)}


# ---- zero and underflowing raw quaternions ----

DEGENERATE = ["b2_v5_6x7_d16_degenerate", "b3_v6_3x5_d25_degenerate"]


def zero_quaternion_pixels(c):
    """(item, pixel) of raw quaternions that are exactly 0, and of those whose float32 squares underflow"""
    q = np.asarray(c["raw"])[:, 5:9].reshape(c["raw"].shape[0], 4, -1)
    exact = np.argwhere((q == 0).all(1))
    tiny = np.argwhere(~(q == 0).all(1) & ((q.astype(np.float32) ** 2).sum(1, dtype=np.float32) == 0))
    return exact, tiny


@pytest.mark.parametrize("name", DEGENERATE)
def test_zero_and_underflowing_quaternions_in_the_head(poisoned, name):
    c = case(name)
    exact, tiny = zero_quaternion_pixels(c)
    assert len(exact) and len(tiny)
    vr, gr, _, grads = compare(c, masked_cotangents(c))
    d = grads["raw"].detach().cpu().numpy().reshape(c["raw"].shape[0], c["raw"].shape[1], -1)
    assert np.isfinite(d).all()
    for item, p in exact:
        assert (d[item, 5:9, p] == 0).all()
    print(f"{name}: head value ratio {vr:.3f}, gradient ratio {gr:.3f}")
    assert vr <= 1.0 and gr <= 1.0


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("name", DEGENERATE)
def test_zero_and_underflowing_quaternions_in_the_fused_adapter(poisoned, name, deterministic):
    c = case(name)
    exact, _ = zero_quaternion_pixels(c)
    cot = masked_cotangents(c)
    h, w = c["raw"].shape[-2:]
    t = {k: torch.tensor(np.asarray(c[k]), dtype=torch.float32, device=DEV).requires_grad_(True) for k in O.INPUTS}
    K = torch.tensor(c["K"], dtype=torch.float32, device=DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        outs = existing_route(t["raw"], t["logits"], t["depths"], t["c2w"], K, cfg_for(c["sh_degree"]), h, w)
        sum((torch.tensor(cot[k], dtype=torch.float32, device=DEV) * o).sum() for k, o in zip(KEYS, outs)).backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    ov, og = oracle(c, cot)
    vr = max(value_ratio(o.detach().cpu().numpy(), ov[k]) for k, o in zip(KEYS, outs))
    gr = max(grad_ratio(t[k].grad.cpu().numpy(), og[k]) for k in O.INPUTS)
    d = t["raw"].grad.cpu().numpy().reshape(c["raw"].shape[0], c["raw"].shape[1], -1)
    assert np.isfinite(d).all()
    for item, p in exact:
        assert (d[item, 5:9, p] == 0).all()
    print(f"{name} (deterministic={deterministic}): adapter value ratio {vr:.3f}, gradient ratio {gr:.3f}")
    assert vr <= 1.0 and gr <= 1.0
