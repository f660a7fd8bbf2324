"""GPU tests of LPIPS-VGG layer by layer (csrc/gs_lpips.cu against tests/lpips_layerwise.py), in TF32 and BF16.

gs_lpips_forward / gs_lpips_backward run through the C ABI on a workspace the test owns, so every activation, pooled map
and the final dL/dz0 can be read back (tests/lpips_layerwise.py's Plan restates the layout).  Then:
  forward   each of the 13 activations against fp64 of its layer on the kernel's own input, per element
            |ours - ref| <= u(ref) + GAMMA sum |a w|, and the fraction of stored values that differ from the rounded
            reference; every pooled map bit-exact against the max of the kernel's own activation; the distance within
            1e-6 relative of the fp64 head on the kernel's taps;
  backward  dL/dz0 (the gradient buffer k_conv0_bwd reads) and dL/din against the fp64 backward conditioned on the
            kernel's forward (its ReLU masks, its pool routes, rounding where the kernels round), once with the real
            lin weights and once per tap with the other four zeroed, so the deep layers' backward is seen on its own;
            and conv1_1's backward alone: dL/din against fp64 of the kernel's own dL/dz0, per element.
The bounds are in tests/lpips_layerwise.py; every check prints its worst ratio (bound = 1)."""
import ctypes

import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200 import lpips as pl
from tests import lpips_layerwise as lw
from tests import test_gpu_lpips as tl

pytestmark = pytest.mark.gpu
DEV = tl.DEV
SD = tl.SD

# tests/test_gpu_lpips.py's shapes (M tails, floor-pool drops, a 1x1 level-4 map) with grads 1, 2 and 3 in turn, and
# two 1xN level-4 maps
CASES = [(kind, n, h, w, normalize, (1, 2, 3)[i % 3]) for i, (kind, n, h, w, normalize, _) in enumerate(tl.CASES)]
CASES += [("noise", 2, 16, 48, True, 3), ("out_of_range", 1, 20, 150, False, 1)]

_packs = {}


def _pack(prec, keep):
    """Packed weights with every lin weight but tap `keep`'s zeroed (None: the real ones); the conv weights are the same,
    so a backward with any of them reads the forward's workspace."""
    if (prec, keep) not in _packs:
        sd = dict(SD)
        for t, k in enumerate(pl.LIN_KEYS):
            if keep is not None and t != keep:
                sd[k] = torch.zeros_like(SD[k])
        m = pl.LPIPS(weights=sd).to(DEV)
        _packs[(prec, keep)] = (m, m._pack(DEV, prec))
    return _packs[(prec, keep)][1].handle


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _forward(prec, x0, x1, normalize, grads):
    n, _, h, w = x0.shape
    cfg = _capi.GsLpipsConfig(batch=n, height=h, width=w, normalize=int(normalize), in0_stride=3 * h * w,
                              in1_stride=3 * h * w, grads=grads, precision=_capi.LPIPS_PRECISIONS[prec])
    plan = lw.Plan(n, h, w, grads, prec)
    L = _capi.lib()
    assert L.gs_lpips_workspace_bytes(ctypes.byref(cfg)) == plan.total
    ws = torch.empty(plan.total, dtype=torch.uint8, device=DEV)
    assert ws.data_ptr() % 256 == 0
    out = torch.empty(n, dtype=torch.float32, device=DEV)
    _capi.check(L.gs_lpips_forward(_pack(prec, None), ctypes.byref(cfg), x0.data_ptr(), x1.data_ptr(), ws.data_ptr(),
                                   out.data_ptr(), _stream()))
    return cfg, plan, ws, out


def _backward(prec, keep, cfg, plan, ws, dout):
    n, h, w = cfg.batch, cfg.height, cfg.width
    g = [torch.empty(n, 3, h, w, dtype=torch.float32, device=DEV) if cfg.grads & (1 << k) else None for k in range(2)]
    ptr = lambda t: t.data_ptr() if t is not None else None
    _capi.check(_capi.lib().gs_lpips_backward(_pack(prec, keep), ctypes.byref(cfg), dout.data_ptr(), ws.data_ptr(),
                                              ptr(g[0]), ptr(g[1]), _stream()))
    torch.cuda.synchronize()
    return lw.nchw64(plan.dz0_nhwc(ws)), torch.cat([t for t in g if t is not None]).double()


@pytest.mark.parametrize("prec", ["tf32", "bf16"])
@pytest.mark.parametrize("kind,n,h,w,normalize,grads", CASES)
def test_every_layer_on_its_own_inputs(prec, kind, n, h, w, normalize, grads):
    x0, x1 = (t.contiguous() for t in tl._pair(kind, n, h, w, seed=h * 1000 + w + n))
    dout = (0.5 + torch.rand(n, generator=torch.Generator().manual_seed(grads))).to(DEV)
    label = f"[layerwise {prec}] {kind} {n}x3x{h}x{w} normalize={normalize} grads={grads}"
    cfg, plan, ws, out = _forward(prec, x0, x1, normalize, grads)
    torch.cuda.synchronize()
    W = lw.Weights(SD, prec, device=DEV)
    fails = []

    def verdict(what, ratio):
        print(f"{label} {what}: worst ratio {ratio:.3g}")
        if not ratio <= 1.0:
            fails.append((what, ratio))

    # forward: every layer on its own input, every pool, the head
    acts = [lw.nchw64(plan.act_nhwc(ws, l)) for l in range(lw.LAYERS)]
    cur = lw.scaled_input(torch.cat([x0, x1]), W, normalize)
    for l in range(lw.LAYERS):
        if l in lw.POOLED:
            k = lw.POOLED.index(l)
            pooled = lw.nchw64(plan.pool_nhwc(ws, k))
            same = torch.equal(pooled, torch.nn.functional.max_pool2d(acts[l - 1], 2, 2))
            print(f"{label} pool {k}: bit-exact {same}")
            if not same:
                fails.append((f"pool {k}", None))
            cur = pooled
        _, ref, sabs = lw.layer_forward(l, cur, W, with_abs=True)
        rep = lw.forward_report(acts[l], ref, sabs, prec)
        print(f"{label} layer {l} forward: worst ratio {rep['worst_ratio']:.3g}, flipped {rep['flip_frac']:.2e}")
        if not (rep["worst_ratio"] <= 1.0 and rep["flip_frac"] <= lw.FLIP_MAX[prec]):
            fails.append((f"layer {l} forward", rep))
        cur = acts[l]
    head = lw.head_value(acts, W, n)
    verdict("head value", float(((out.double() - head).abs() / head.abs()).max()) / lw.HEAD_REL)

    # backward: the real lin weights, then each tap alone
    i0, nb = (0 if grads & 1 else n), plan.nb
    for keep in (None, 0, 1, 2, 3, 4):
        Wk = W.with_lin(keep)
        dz0, din = _backward(prec, keep, cfg, plan, ws, dout)
        dz0_ref, din_ref = lw.backward(acts, Wk, dout.double(), n, i0, nb, normalize)
        tag = "lin" if keep is None else f"tap {keep} alone"
        for name, a, b in (("dL/dz0", dz0, dz0_ref), ("dL/din", din, din_ref)):
            rep = lw.grad_report(a, b, prec)
            print(f"{label} {tag} {name}: rel-L2 {rep['rel']:.2e} (ratio {rep['rel_ratio']:.3g}), element-wise ratio "
                  f"{rep['elem_ratio']:.3g}")
            if not (rep["rel_ratio"] <= 1.0 and rep["elem_ratio"] <= 1.0):
                fails.append((f"{tag} {name}", rep))
        verdict(f"{tag} conv1_1 backward alone", lw.conv0_report(din, dz0, Wk, normalize))
    assert not fails, fails
