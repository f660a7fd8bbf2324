"""GPU checks of the device optimizer step (pf3plat_b200.optimizer.Adam over csrc/gs_optimizer.cu, DESIGN.md 5.19)
against the reference sequence of tests/optimizer_oracle.py (PF3plat's NaN loop, Lightning's clip, torch.optim.Adam's
default foreach route on CUDA, zero_grad), every test under poisoned allocations:
  1. parity over 50 steps of fresh gradients and a schedule of lr values, with and without the clip, on PF3plat-like
     shapes (0-d, one element, odd lengths, biases and norms, 3x3x256x256 convolutions, a tensor of many chunks and a
     4-byte-misaligned view);
  2. a single NaN (first tensor, a middle tensor, the last element of an odd-length last tensor) skips the step;
  3. Inf without NaN, with and without the clip: the same NaN pattern as the reference;
  4. gradients that are None on some steps, and gradients that come back at new addresses;
  5. bit-reproducibility;
  6. state dicts to and from torch.optim.Adam;
  7. no host wait: an eager step under set_sync_debug_mode("error"), and decoder + loss + backward + step captured in
     one CUDA graph, with a workspace large enough (bit-equal to the eager sequence) and too small (the step skips);
  8. refusals that need a device.

Parity bound.  Before each step the oracle is given the device optimizer's state, so every comparison is of one step
from equal inputs.  The arithmetic is torch's, op for op; the step size is formed from the float32 device lr (torch uses
the Python double), so an update may differ in its last bit.  The bound is a few ulps of each result's terms: 4 ulps
for the moments, 2 ulps of the parameter plus 8 ulps of its update.
The clip is the one larger source.  The device sums the squares in fp64 and rounds the root once; torch's
_foreach_norm + vector_norm accumulate in fp32 and land up to ~1e-6 away (measured on the H100: tens of ulps of the
norm, hence of coef and of every clipped gradient, and more where a moment nearly cancels).  So with the clip the
oracle is given the fp64 total (clip_grads_with_norm_, the same formula), and the test asserts separately that torch's
own total lies within 2^-16 of it: the whole difference from the reference is the reference's fp32 norm."""
import contextlib
import copy
import functools

import pytest
import torch

from pf3plat_b200.optimizer import Adam
from tests.optimizer_oracle import exact_total_norm, reference_step
from tests.poison import poisoned  # noqa: F401

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


@contextlib.contextmanager
def _deterministic(on=True):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


SHAPES = [(), (1,), (7,), (33,), (256,), (512,), (64, 3, 3, 3), (256, 256, 3, 3), (256,), (256, 256, 3, 3),
          (1_000_003,), (129, 65), "misaligned", (4099,)]


def _make_params(dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for s in SHAPES:
        if s == "misaligned":  # a Parameter made from buf[1:]: 4 bytes past a 16-byte boundary
            buf = torch.randn(2050, generator=g, device=dev)
            p = torch.nn.Parameter(buf[1:])
            assert p.data_ptr() % 16 == 4
        else:
            p = torch.nn.Parameter(torch.randn(s, generator=g, device=dev))
        out.append(p)
    return out


def _clones(params):
    return [torch.nn.Parameter(p.detach().clone()) for p in params]


def _grads(params, g, scale, misaligned=True):
    """Fresh random gradients; the misaligned parameter's gradient is a misaligned view too."""
    out = []
    for k, p in enumerate(params):
        if misaligned and SHAPES[k] == "misaligned":
            buf = torch.randn(p.numel() + 1, generator=g, device=p.device) * scale
            out.append(buf[1:])
        else:
            out.append(torch.randn(p.shape, generator=g, device=p.device) * scale)
    return out


def _set_grads(params, grads, in_place=True):
    for p, gr in zip(params, grads):
        if gr is None:
            p.grad = None
        elif in_place and p.grad is not None:
            p.grad.copy_(gr)
        else:
            p.grad = gr.clone() if gr.is_contiguous() and gr.data_ptr() % 16 == 0 else gr
    return params


def _ulp(x):
    x = x.abs().float()
    return torch.nextafter(x, torch.full_like(x, float("inf"))) - x


def _sync_oracle(ours, opt, theirs, ref):
    """The oracle takes the device optimizer's parameters and state, so that the next step starts from equal inputs."""
    for p, q in zip(ours, theirs):
        q.data.copy_(p.detach())
        if p in opt.state and opt.state[p]:
            st, rt = opt.state[p], ref.state[q]
            if not rt:
                rt["step"] = torch.tensor(0.0)
                rt["exp_avg"], rt["exp_avg_sq"] = torch.zeros_like(q), torch.zeros_like(q)
            rt["step"].fill_(float(st["step"]))
            rt["exp_avg"].copy_(st["exp_avg"])
            rt["exp_avg_sq"].copy_(st["exp_avg_sq"])


def _total(grads, max_norm):
    """The fp64 total the oracle clips with, after checking torch's own fp32 total against it."""
    if max_norm is None:
        return None
    gs = [g for g in grads if g is not None]
    exact, torch_total = exact_total_norm(gs), torch.nn.utils.get_total_norm(gs)
    if torch.isfinite(exact):
        assert abs(float(torch_total) - float(exact)) <= 2.0 ** -16 * float(exact), (float(torch_total), float(exact))
    else:
        assert not torch.isfinite(torch_total)
    return exact


def _coef(total, max_norm):
    return 1.0 if max_norm is None else torch.clamp(max_norm / (total + 1e-6), max=1.0)


def _compare(ours, opt, theirs, ref, before, grads, coef, tag):
    for k, (p, q) in enumerate(zip(ours, theirs)):
        st, rt = opt.state.get(p, {}), ref.state.get(q, {})
        assert bool(st) == bool(rt), (tag, k)
        assert p.grad is None or not p.grad.any(), (tag, k, "gradient not zeroed")
        if not st:
            assert torch.equal(p.detach(), q.detach()), (tag, k)
            continue
        assert float(st["step"]) == float(rt["step"]), (tag, k, float(st["step"]), float(rt["step"]))
        p0, m0, v0 = before[k]
        g = grads[k] * coef if grads[k] is not None else torch.zeros_like(p)
        gc = g.reshape(p.shape)
        # a few ulps of the largest term each result sums: m = b1 m0 + (1 - b1) g, v = b2 v0 + (1 - b2) g^2
        big = lambda *ts: functools.reduce(torch.maximum, [t.abs() for t in ts])
        pairs = (("exp_avg", st["exp_avg"], rt["exp_avg"], 4 * _ulp(big(rt["exp_avg"], m0, 0.1 * gc))),
                 ("exp_avg_sq", st["exp_avg_sq"], rt["exp_avg_sq"], 4 * _ulp(big(rt["exp_avg_sq"], v0, 1e-3 * gc * gc))),
                 ("param", p.detach(), q.detach(), 2 * _ulp(q.detach()) + 8 * _ulp(q.detach() - p0)))
        for name, a, b, tol in pairs:
            na, nb = torch.isnan(a), torch.isnan(b)
            assert torch.equal(na, nb), (tag, k, name, "NaN pattern")
            fin = ~nb
            err = (a - b).abs()[fin]
            bad = err > tol[fin]
            assert not bad.any(), (tag, k, name, float(err.max()), int(bad.sum()))


def _snapshot(ours, opt):
    out = []
    for p in ours:
        st = opt.state.get(p)
        if st:
            out.append((p.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()))
        else:
            out.append((p.detach().clone(), None, None))
    return out


def _step_both(ours, opt, theirs, ref, grads, max_norm, lr, tag):
    _sync_oracle(ours, opt, theirs, ref)
    for group in ref.param_groups:
        group["lr"] = lr
    opt.param_groups[0]["lr"] = lr
    before = [(p.detach().clone(), *(opt.state[p][k].clone() if opt.state.get(p) else torch.zeros_like(p)
                                     for k in ("exp_avg", "exp_avg_sq"))) for p in ours]
    _set_grads(ours, grads)
    _set_grads(theirs, [None if g is None else g.clone() for g in grads], in_place=False)
    kept = [None if q.grad is None else q.grad.clone() for q in theirs]  # step() zeroes ours, which may be `grads`
    total = _total(kept, max_norm)
    coef = _coef(total, max_norm)
    skipped = reference_step(ref, max_norm, total)
    opt.step()
    torch.cuda.synchronize()
    _compare(ours, opt, theirs, ref, before, kept, coef, tag)
    return skipped


def _pair(dev, max_norm, seed=0):
    ours = _make_params(dev, seed)
    theirs = _clones(ours)
    return ours, Adam(ours, lr=2e-4, max_norm=max_norm), theirs, torch.optim.Adam(theirs, lr=2e-4)


def _scale(params, k, max_norm):
    """Gradient scale that puts the total norm on alternating sides of max_norm (0.5 when there is none)."""
    n = sum(p.numel() for p in params)
    return (max_norm or 0.5) / n ** 0.5 * (0.5 if k % 2 else 2.0)


@pytest.mark.parametrize("max_norm", [0.5, None])
def test_parity_over_fifty_steps(poisoned, max_norm):
    dev = _dev()
    ours, opt, theirs, ref = _pair(dev, max_norm)
    g = torch.Generator(device=dev).manual_seed(1)
    sched = torch.optim.lr_scheduler.OneCycleLR(torch.optim.SGD([torch.zeros(1, requires_grad=True)], lr=2e-4),
                                                2e-4, 60, pct_start=0.1, cycle_momentum=False, anneal_strategy="cos")
    for k in range(50):
        lr = sched.get_last_lr()[0]
        assert not _step_both(ours, opt, theirs, ref, _grads(ours, g, _scale(ours, k, max_norm)), max_norm, lr,
                              f"step {k}")
        sched.optimizer.step()
        sched.step()
    assert int(opt.skipped) == 0


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_a_single_nan_skips_the_step(poisoned, where):
    dev = _dev()
    ours, opt, theirs, ref = _pair(dev, 0.5)
    g = torch.Generator(device=dev).manual_seed(2)
    for k in range(2):
        _step_both(ours, opt, theirs, ref, _grads(ours, g, _scale(ours, k, 0.5)), 0.5, 2e-4, f"warm-up {k}")
    grads = _grads(ours, g, _scale(ours, 0, 0.5))
    t = {"first": 0, "middle": len(ours) // 2, "last": len(ours) - 1}[where]
    assert where != "last" or ours[t].numel() % 2 == 1
    flat = grads[t].view(-1)
    flat[0 if where != "last" else -1] = float("nan")
    before = [(p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(),
               float(opt.state[p]["step"])) for p in ours]
    _set_grads(ours, grads)
    opt.step()
    torch.cuda.synchronize()
    assert int(opt.skipped) == 1
    for k, p in enumerate(ours):
        p0, m0, v0, s0 = before[k]
        assert torch.equal(p.detach(), p0) and torch.equal(opt.state[p]["exp_avg"], m0), k
        assert torch.equal(opt.state[p]["exp_avg_sq"], v0) and float(opt.state[p]["step"]) == s0, k
        assert not p.grad.any(), k
    # the oracle skips the same step; the next clean step matches it
    _set_grads(theirs, [x.clone() for x in grads], in_place=False)
    assert reference_step(ref, 0.5)
    assert not _step_both(ours, opt, theirs, ref, _grads(ours, g, _scale(ours, 1, 0.5)), 0.5, 2e-4, "after")


@pytest.mark.parametrize("max_norm", [0.5, None])
def test_inf_without_nan_gives_the_reference_nan_pattern(poisoned, max_norm):
    dev = _dev()
    ours, opt, theirs, ref = _pair(dev, max_norm)
    g = torch.Generator(device=dev).manual_seed(3)
    _step_both(ours, opt, theirs, ref, _grads(ours, g, _scale(ours, 0, max_norm)), max_norm, 2e-4, "warm-up")
    grads = _grads(ours, g, _scale(ours, 1, max_norm))
    grads[3].view(-1)[5] = float("inf")
    grads[10].view(-1)[123_456] = float("-inf")
    _sync_oracle(ours, opt, theirs, ref)
    before = _snapshot(ours, opt)
    _set_grads(ours, grads)
    _set_grads(theirs, [x.clone() for x in grads], in_place=False)
    grads = [q.grad.clone() for q in theirs]
    total = _total(grads, max_norm)
    coef = _coef(total, max_norm)
    assert not reference_step(ref, max_norm, total)
    opt.step()
    torch.cuda.synchronize()
    assert int(opt.skipped) == 0
    for k, (p, q) in enumerate(zip(ours, theirs)):
        assert torch.equal(torch.isnan(p.detach()), torch.isnan(q.detach())), k
    assert torch.isnan(ours[3].detach()).any() and torch.isnan(ours[10].detach()).any()
    _compare(ours, opt, theirs, ref, [(b[0], b[1], b[2]) for b in before],
             [x.masked_fill(~torch.isfinite(x), 0.0) for x in grads], coef, "inf")


def test_none_gradients_leave_their_parameters_alone(poisoned):
    dev = _dev()
    ours, opt, theirs, ref = _pair(dev, 0.5)
    g = torch.Generator(device=dev).manual_seed(4)
    tables = []
    for k in range(8):
        grads = _grads(ours, g, _scale(ours, k, 0.5))
        for t in range(len(grads)):
            if (t + k) % 3 == 0:
                grads[t] = None
        if k == 5:  # every gradient comes back at a new address
            for p in ours:
                p.grad = None
        _step_both(ours, opt, theirs, ref, grads, 0.5, 2e-4, f"step {k}")
        tables.append(opt._table.data_ptr())
    steps = [float(opt.state[p]["step"]) if opt.state.get(p) else 0.0 for p in ours]
    assert steps == [float(sum((t + k) % 3 != 0 for k in range(8))) for t in range(len(ours))]
    assert len(set(tables)) > 1


def test_the_same_inputs_give_bit_equal_results(poisoned):
    dev = _dev()
    runs = []
    for det in (False, True, False):
        with _deterministic(det):
            ours = _make_params(dev, seed=5)
            opt = Adam(ours, lr=2e-4, max_norm=0.5)
            g = torch.Generator(device=dev).manual_seed(6)
            for k in range(4):
                _set_grads(ours, _grads(ours, g, _scale(ours, k, 0.5)))
                opt.step()
            torch.cuda.synchronize()
            runs.append([p.detach().clone() for p in ours] + [opt.state[p][n].clone() for p in ours
                                                              for n in ("exp_avg", "exp_avg_sq")])
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


@pytest.mark.parametrize("direction", ["torch_to_ours", "ours_to_torch"])
def test_state_dicts_move_between_torch_adam_and_this_one(poisoned, direction):
    dev = _dev()
    src_params = _make_params(dev, seed=7)
    g = torch.Generator(device=dev).manual_seed(8)
    src = (torch.optim.Adam(src_params, lr=2e-4) if direction == "torch_to_ours"
           else Adam(src_params, lr=2e-4, max_norm=0.5))
    for k in range(3):
        _set_grads(src_params, _grads(src_params, g, _scale(src_params, k, 0.5)), in_place=False)
        if direction == "torch_to_ours":
            reference_step(src, 0.5)
        else:
            src.step()
    sd = src.state_dict()
    for st in sd["state"].values():
        assert st["step"].device.type == "cpu" and st["step"].dtype == torch.float32 and st["step"].dim() == 0
        assert float(st["step"]) == 3.0
    ours_p, theirs_p = _clones(src_params), _clones(src_params)
    opt, ref = Adam(ours_p, lr=1.0, max_norm=0.5), torch.optim.Adam(theirs_p, lr=1.0)
    # deep copies, as from a checkpoint file: a live state dict holds the source's own moment tensors, and loading it
    # into both optimizers would make them update the same tensors
    (opt if direction == "torch_to_ours" else ref).load_state_dict(copy.deepcopy(sd))
    (ref if direction == "torch_to_ours" else opt).load_state_dict(copy.deepcopy(src.state_dict()))
    assert opt.param_groups[0]["lr"] == 2e-4 and opt.param_groups[0]["max_norm"] == 0.5
    for p, q in zip(ours_p, theirs_p):
        assert torch.equal(opt.state[p]["exp_avg"], ref.state[q]["exp_avg"].to(dev))
        assert float(opt.state[p]["step"]) == float(ref.state[q]["step"]) == 3.0
    for k in range(10):
        _step_both(ours_p, opt, theirs_p, ref, _grads(ours_p, g, _scale(ours_p, k, 0.5)), 0.5, 2e-4, f"step {k}")


def test_an_eager_step_never_waits_for_the_device(poisoned):
    dev = _dev()
    ours = _make_params(dev, seed=9)
    opt = Adam(ours, lr=2e-4, max_norm=0.5)
    g = torch.Generator(device=dev).manual_seed(10)
    _set_grads(ours, _grads(ours, g, 1e-3))
    opt.step()
    grads = _grads(ours, g, 1e-3)
    _set_grads(ours, grads)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step()
        opt.param_groups[0]["lr"] = 1e-4
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def _decoder_case(dev):
    from pf3plat_b200.synthetic import make_scene
    scenes = [make_scene(20_000, 2, 64, 64, seed=40 + k) for k in range(2)]
    st = lambda f: torch.stack([f(s) for s in scenes]).to(dev)
    c = lambda s: s.covariances
    leaves = {"means": st(lambda s: s.means),
              "cov": st(lambda s: torch.stack([c(s)[:, 0, 0], c(s)[:, 0, 1], c(s)[:, 0, 2], c(s)[:, 1, 1],
                                               c(s)[:, 1, 2], c(s)[:, 2, 2]], -1)),
              "harm": st(lambda s: s.harmonics), "opac": st(lambda s: s.opacities)}
    cams = {"ext": st(lambda s: s.extrinsics), "intr": st(lambda s: s.intrinsics), "near": st(lambda s: s.near),
            "far": st(lambda s: s.far)}
    target = torch.rand(2, 2, 3, 64, 64, generator=torch.Generator().manual_seed(11)).to(dev)
    return leaves, cams, target


def _train_step(params, opt, cams, target, ws):
    from pf3plat_b200.losses import photometric_loss
    from pf3plat_b200.render import decoder_forward
    color, _ = decoder_forward(*params, cams["ext"], cams["intr"], cams["near"], cams["far"], (64, 64),
                               torch.zeros(3, device=target.device), depth_mode=None, sh_eval_max_degree=4,
                               workspace=ws)
    mse, ssim = photometric_loss(color.flatten(0, 1), target.flatten(0, 1))
    (mse + ssim).backward()
    opt.step()


@pytest.mark.parametrize("capacity", ["enough", "too_small"])
def test_decoder_loss_backward_and_step_in_one_cuda_graph(poisoned, capacity):
    from pf3plat_b200.rasterizer import SyncFreeWorkspace, last_stats
    dev = _dev()
    leaves, cams, target = _decoder_case(dev)
    params = [torch.nn.Parameter(t.clone()) for t in leaves.values()]
    eager = [torch.nn.Parameter(t.clone()) for t in leaves.values()]
    opt = Adam(params, lr=torch.tensor(1e-3, device=dev), max_norm=0.5)
    ref = Adam(eager, lr=torch.tensor(1e-3, device=dev), max_norm=0.5)
    with _deterministic():
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            from pf3plat_b200.render import decoder_forward
            with torch.no_grad():
                decoder_forward(*leaves.values(), cams["ext"], cams["intr"], cams["near"], cams["far"], (64, 64),
                                torch.zeros(3, device=dev))
            D = last_stats(dev)["num_rendered"]
            cap = int(D * 2) if capacity == "enough" else max(D // 4, 1)
            ws = SyncFreeWorkspace(dev, 2, 4, 20_000, (64, 64), cap, deterministic=True)
            ws_eager = SyncFreeWorkspace(dev, 2, 4, 20_000, (64, 64), cap, deterministic=True)
            for _ in range(2):  # state, chunk table and gradients exist before capture
                _train_step(params, opt, cams, target, ws)
                _train_step(eager, ref, cams, target, ws_eager)
            torch.cuda.synchronize()
        before = [p.detach().clone() for p in params] + [opt.state[p][k].clone() for p in params
                                                          for k in ("exp_avg", "exp_avg_sq")]
        skipped0 = int(opt.skipped)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            _train_step(params, opt, cams, target, ws)
        for k in range(5):
            with torch.cuda.stream(s):
                graph.replay()
                _train_step(eager, ref, cams, target, ws_eager)
            torch.cuda.synchronize()
            if capacity == "enough":
                for a, b in zip(params, eager):
                    assert torch.equal(a.detach(), b.detach()), k
                    for n in ("exp_avg", "exp_avg_sq", "step"):
                        assert torch.equal(opt.state[a][n], ref.state[b][n]), (k, n)
            else:
                after = [p.detach() for p in params] + [opt.state[p][n] for p in params
                                                        for n in ("exp_avg", "exp_avg_sq")]
                for a, b in zip(after, before):
                    assert torch.equal(a, b), k
                assert int(opt.skipped) == skipped0 + k + 1
        if capacity == "enough":
            assert int(opt.skipped) == 0 and not ws.status()[1]
        else:
            assert skipped0 == 2 and ws.status()[1]


def test_refusals_that_need_a_device(poisoned):
    dev = _dev()
    p = torch.nn.Parameter(torch.zeros(4, device=dev))
    with pytest.raises(TypeError, match="float32"):
        Adam([torch.nn.Parameter(torch.zeros(4, device=dev, dtype=torch.float64))])
    with pytest.raises(TypeError, match="float32"):
        Adam([torch.nn.Parameter(torch.zeros(4, device=dev, dtype=torch.bfloat16))])
    with pytest.raises(TypeError, match="CUDA"):
        Adam([p, torch.nn.Parameter(torch.zeros(4))])
    with pytest.raises(ValueError, match="one param group"):
        Adam([{"params": [p]}, {"params": [torch.nn.Parameter(torch.zeros(4, device=dev))]}])
    with pytest.raises(ValueError, match="weight_decay"):
        Adam([{"params": [p], "weight_decay": 0.1}])
    with pytest.raises(ValueError, match="not contiguous"):
        Adam([torch.nn.Parameter(torch.zeros(4, 4, device=dev).t())])
    opt = Adam([p], lr=1e-3)
    p.grad = torch.zeros(4, 2, device=dev)[:, 0]
    with pytest.raises(ValueError, match="not contiguous"):
        opt.step()
    p.grad = torch.zeros(4, device=dev).to_sparse()
    with pytest.raises(ValueError, match="sparse"):
        opt.step()
    p.grad = torch.zeros(4, device=dev)
    opt.step()
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="float lr"):
        with torch.cuda.graph(graph, stream=s):
            opt.step()
    torch.cuda.synchronize()
