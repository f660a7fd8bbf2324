"""CPU tests of the layer-by-layer LPIPS checkers (tests/lpips_layerwise.py):
  * the restated workspace plan agrees with gs_lpips_workspace_bytes, and the two storage roundings are pinned bit for bit;
  * with nothing rounded, the conditioned backward is autograd of the fp64 oracle (oracle/lpips_oracle.py);
  * a mutation table: errors a kernel could make, built into the rounding-faithful model, each shown with the verdict of
    the end-to-end rule of tests/test_gpu_lpips.py (the model's own fp64 error standing in for PyTorch's) and of the
    layer-wise rule.  The layer-wise rule rejects every one; the end-to-end rule accepts most of them."""
import ctypes

import pytest
import torch

from oracle import lpips_oracle as lo
from tests import lpips_layerwise as lw

SD = lo.random_state_dict(11)


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


# ---------------------------------------------------------------------------------------------------------------------
# plan and roundings
# ---------------------------------------------------------------------------------------------------------------------
def test_the_restated_plan_has_the_library_s_size_and_disjoint_regions(capi):
    L = capi.lib()
    for prec in ("tf32", "bf16"):
        for grads in range(4):
            for h, w in ((16, 16), (37, 53), (17, 130), (64, 48)):
                for n in (1, 2, 5):
                    cfg = capi.GsLpipsConfig(batch=n, height=h, width=w, normalize=1, in0_stride=3 * h * w,
                                             in1_stride=3 * h * w, grads=grads, precision=capi.LPIPS_PRECISIONS[prec])
                    p = lw.Plan(n, h, w, grads, prec)
                    assert p.total == L.gs_lpips_workspace_bytes(ctypes.byref(cfg)), (prec, grads, h, w, n)
                    if not grads:
                        continue
                    regions = [(p.act[l], p.nimg * p.h[lw.LEVEL[l]] * p.w[lw.LEVEL[l]] * lw.COUT[l]) for l in range(13)]
                    regions += [(p.pool[k], p.nimg * p.h[lw.LEVEL[l]] * p.w[lw.LEVEL[l]] * lw.CIN[l])
                                for k, l in enumerate(lw.POOLED)]
                    regions += [(g, p.nb * h * w * 64) for g in p.grad] + [(p.partial, 5 * n * 32 * 2 // p.esize)]
                    regions.sort()
                    for (o, e), (o2, _) in zip(regions, regions[1:]):
                        assert o % 256 == 0 and o + e * p.esize <= o2
                    assert regions[-1][0] + regions[-1][1] * p.esize <= p.total


def _bits(*words):
    return torch.tensor([w - (1 << 32) if w >= 1 << 31 else w for w in words], dtype=torch.int32).view(torch.float32)


def _words(x):
    return [v & 0xFFFFFFFF for v in x.view(torch.int32).tolist()]


def test_tf32_rna_on_hand_built_bit_patterns():
    cases = {  # input -> cvt.rna.tf32.f32
        0x3F801000: 0x3F802000,  # 1 + half a TF32 unit, kept bits even: a tie, away from zero (RNE would keep 1.0)
        0xBF801000: 0xBF802000,  # the same tie, negative
        0x3F803000: 0x3F804000,  # a tie with odd kept bits
        0x3F800FFF: 0x3F800000,  # just below the tie
        0x3F801001: 0x3F802000,  # just above
        0x3FFFF000: 0x40000000,  # a tie carried into the exponent: 1.99976 -> 2
        0xBFFFFFFF: 0xC0000000,
        0x00001000: 0x00002000,  # subnormal tie
        0x00000FFF: 0x00000000,  # subnormal below the tie
        0x807FF000: 0x80800000,  # largest subnormals carry into the smallest normal
        0x7F7FEFFF: 0x7F7FE000,  # large, below the tie
        0x7F7FFFFF: 0x7F800000,  # the largest finite value rounds to Inf
        0xFF7FFFFF: 0xFF800000,
        0x7F800000: 0x7F800000,  # Inf
        0xFF800000: 0xFF800000,
        0x7FC00001: 0x7FC00001,  # NaN payloads pass through
        0x7F800001: 0x7F800001,
        0x00000000: 0x00000000,
        0x80000000: 0x80000000,
    }
    got = _words(lw.tf32_rna(_bits(*cases)))
    assert got == list(cases.values()), [hex(v) for v in got]
    # random finite values: 13 low bits clear, within half a unit, ties away from zero
    x = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * torch.exp2(torch.randint(-60, 60, (100000,)).float())
    r = lw.tf32_rna(x)
    assert all(v & 0x1FFF == 0 for v in _words(r))
    assert bool(((r.double() - x.double()).abs() <= lw.unit(x.double(), "tf32") / 2).all())


def test_bf16_rne_is_torch_s_bfloat16():
    g = torch.Generator().manual_seed(1)
    words = torch.randint(-(1 << 31), (1 << 31) - 1, (200000,), generator=g, dtype=torch.int64).to(torch.int32)
    x = torch.cat([words.view(torch.float32),
                   _bits(0x3F808000, 0x3F818000, 0xBF808000, 0x7F7FFFFF, 0x7F7F8000, 0x00008000, 0x00018000,
                         0x7F800000, 0xFF800000, 0x7FC00001, 0x00000000, 0x80000000)])
    ours, ref = lw.bf16_rne(x), x.to(torch.bfloat16).to(torch.float32)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(ours), nan)
    assert torch.equal(ours[~nan].view(torch.int32), ref[~nan].view(torch.int32))


def _inputs(n, h, w, seed):
    """Noise images with a flat patch: the patch gives equal activations in a pool window (ties) on both sides."""
    g = torch.Generator().manual_seed(seed)
    x0, x1 = torch.rand(n, 3, h, w, generator=g), torch.rand(n, 3, h, w, generator=g)
    x0[:, :, h // 4:h // 2 + 4, w // 4:w // 2 + 4] = 0.25
    x1[:, :, h // 4:h // 2 + 4, w // 4:w // 2 + 4] = 0.75
    dout = 0.5 + torch.rand(n, generator=g, dtype=torch.float64)
    return x0, x1, dout


@pytest.mark.parametrize("grads", [1, 2, 3])
@pytest.mark.parametrize("normalize", [False, True])
def test_unrounded_conditioned_backward_is_autograd_of_the_fp64_oracle(grads, normalize):
    n, h, w = 2, 37, 21
    x0, x1, dout = _inputs(n, h, w, seed=grads)
    W = lw.Weights(SD, None)
    acts, _, v = lw.forward(x0, x1, W, normalize)
    v64, g0, g1 = lo.with_grads(x0, x1, SD, normalize, dout)
    i0, nb = (0 if grads & 1 else n), (2 * n if grads == 3 else n)
    _, din = lw.backward(acts, W, dout, n, i0, nb, normalize)
    ref = torch.cat([g0, g1])[i0:i0 + nb]
    err_v, err_g = float((v - v64).abs().max() / v64.abs().max()), float((din - ref).abs().max() / ref.abs().max())
    print(f"[layerwise] fp64 model vs autograd, grads={grads} normalize={normalize}: value {err_v:.1e}, grad {err_g:.1e}")
    assert err_v <= 1e-12 and err_g <= 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# the mutation table
# ---------------------------------------------------------------------------------------------------------------------
NOISE = 2.0 ** -20  # relative perturbation of every sum of the model: fp32 accumulation order's share, roughly


def _drop_k_step(tap, c0):
    def f(w):
        w = w.clone()
        w[:, c0:c0 + 32, tap // 3, tap % 3] = 0
        return w
    return f


def _zero_bias_tile(j):
    def f(b):
        b = b.clone()
        b[64 * j:64 * j + 64] = 0
        return b
    return f


def _permute_8(tap, c0):
    def f(w):
        w = w.clone()
        idx = torch.arange(c0, c0 + 8)
        w[:, idx, tap // 3, tap % 3] = w[:, idx.roll(1), tap // 3, tap % 3]
        return w
    return f


SCALE1 = float(SD["scaling_layer.scale"].reshape(-1)[1])

# name -> (precision, mutant, the end-to-end rule's measured verdict (True: accepts it), why the layer-wise rule sees it)
MUTANTS = {
    "conv5_2 backward-data x1.01": (
        "tf32", lw.Mutant(bwd_scale={11: 1.01}), True,
        "the relu5_3-only backward carries the whole gradient through conv5_2"),
    "conv2_1 backward (dL/dz of conv2_1) x1.05": (
        "tf32", lw.Mutant(bwd_scale={3: 1.05}), True, "every dL/dz0 element moves by up to 5 %"),
    "conv5_2 forward: tap 4's last 32-channel K step missing": (
        "tf32", lw.Mutant(fwd_weight={11: _drop_k_step(4, 480)}), True, "the per-layer forward check of conv5_2"),
    "conv5_3 forward: bias missing on N tile 1 (channels 64..127)": (
        "tf32", lw.Mutant(fwd_bias={12: _zero_bias_tile(1)}), True, "the per-layer forward check of conv5_3"),
    "unpool routes to the last maximum on ties": (
        "tf32", lw.Mutant(route_last_max=True), False, "the flat patch makes equal maxima in pool windows"),
    "BF16 conv3_2 forward: 8 channels permuted inside tap 0's second K step": (
        "bf16", lw.Mutant(fwd_weight={5: _permute_8(0, 72)}), True, "the per-layer forward check of conv3_2"),
    "head backward of relu5_3 without its projection term": (
        "tf32", lw.Mutant(head_no_proj=(4,)), True, "the relu5_3-only backward"),
    "conv1_1 backward missing / scale on channel 1": (
        "tf32", lw.Mutant(conv0_bwd_factor={1: SCALE1}), False, "conv1_1's backward checked alone"),
}


def _old_rule(prec, v, din, v_model, din_model, v64, g64):
    """tests/test_gpu_lpips.py (TF32) / test_gpu_lpips_bf16.py (BF16), the model standing in for PyTorch."""
    floor_v, floor_g = ((1e-4, 1e-6), 1e-3) if prec == "tf32" else ((1e-3, 1e-5), 1e-2)
    err, err_t = (v - v64).abs(), float((v_model - v64).abs().max())
    bound = torch.clamp(floor_v[0] * v64.abs() + floor_v[1], min=2 * err_t)
    rel, rel_t = lw.rel_l2(din, g64), lw.rel_l2(din_model, g64)
    return bool((err <= bound).all()) and rel <= max(2 * rel_t, floor_g), rel, rel_t


def _new_rule(prec, x0, x1, normalize, dout, W, mut, noise_seed):
    """The layer-wise rule of tests/test_gpu_lpips_layerwise.py on the model with `mut`: -> (worst ratio per check)."""
    n = x0.shape[0]
    gen = torch.Generator().manual_seed(noise_seed)
    acts, pools, v = lw.forward(x0, x1, W, normalize, mut=mut, noise=(NOISE, gen))
    worst = {}
    cur = lw.scaled_input(torch.cat([x0, x1]), W, normalize)
    pi = 0
    for l in range(lw.LAYERS):
        if l in lw.POOLED:
            assert torch.equal(pools[pi], torch.nn.functional.max_pool2d(acts[l - 1], 2, 2))
            cur, pi = pools[pi], pi + 1
        _, ref, sabs = lw.layer_forward(l, cur, W, with_abs=True)
        rep = lw.forward_report(acts[l], ref, sabs, prec)
        worst["forward"] = max(worst.get("forward", 0.0), rep["worst_ratio"], rep["flip_frac"] / lw.FLIP_MAX[prec])
        cur = acts[l]
    worst["head"] = float(((v - lw.head_value(acts, W, n)).abs() / v.abs()).max()) / lw.HEAD_REL
    din_all = None
    for keep in (None, 0, 1, 2, 3, 4):
        Wk = W.with_lin(keep)
        dz0, din = lw.backward(acts, Wk, dout, n, 0, n, normalize, mut=mut, noise=(NOISE, gen))
        din_all = din if keep is None else din_all
        dz0_ref, din_ref = lw.backward(acts, Wk, dout, n, 0, n, normalize)
        for name, a, b in (("dz0", dz0, dz0_ref), ("din", din, din_ref)):
            rep = lw.grad_report(a, b, prec)
            worst["backward"] = max(worst.get("backward", 0.0), rep["rel_ratio"], rep["elem_ratio"])
        worst["conv1_1 backward"] = max(worst.get("conv1_1 backward", 0.0), lw.conv0_report(din, dz0, Wk, normalize))
    return worst, v, din_all


@pytest.fixture(scope="module")
def table():
    n, h, w, normalize = 2, 32, 32, True
    x0, x1, dout = _inputs(n, h, w, seed=7)
    v64, g64, _ = lo.with_grads(x0, x1, SD, normalize, dout)
    rows, models = {}, {}
    for prec in ("tf32", "bf16"):
        W = lw.Weights(SD, prec)
        models[prec] = (W,) + _new_rule(prec, x0, x1, normalize, dout, W, None, noise_seed=3)
    for name, (prec, mut, _, _) in MUTANTS.items():
        W, _, v_model, din_model = models[prec]
        worst, v, din = _new_rule(prec, x0, x1, normalize, dout, W, mut, noise_seed=3)
        old, rel, rel_t = _old_rule(prec, v, din, v_model, din_model, v64, g64)
        rows[name] = (old, worst, rel, rel_t)
        print(f"[layerwise] mutant {name} ({prec}): end-to-end rule {'accepts' if old else 'rejects'} (grad rel-L2 "
              f"{rel:.2e}, model {rel_t:.2e}); layer-wise worst ratios " + ", ".join(f"{k} {r:.2g}" for k, r in worst.items()))
    return models, rows


def test_the_unmutated_model_passes_the_layerwise_rule_with_headroom(table):
    models, _ = table
    for prec, (_, worst, _, _) in models.items():
        print(f"[layerwise] unmutated {prec} model: worst ratios " + ", ".join(f"{k} {r:.2g}" for k, r in worst.items()))
        assert max(worst.values()) <= 0.6, (prec, worst)


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant(table, name):
    _, rows = table
    prec, _, old_expected, why = MUTANTS[name]
    old, worst, rel, rel_t = rows[name]
    assert old == old_expected, (name, rel, rel_t)
    assert max(worst.values()) > 1.0, (name, worst, why)
