"""The encoder depth glue's kernels (pf3plat_b200.encoder_depth, csrc/gs_encoder_depth.cu) against the fp64 oracle
(tests/encoder_depth_oracle.py) and the reference's own fp64 record (tests/golden/encoder_depth.npz): values
element-wise within 1e-5 (|ref| + 1), gradients within 1e-3 (|ref| + rms ref), with the same non-finite elements.
Where a pre-clamp value lies within rounding of a clamp bound, its pixel's cotangent is zeroed (as
tests/strict_parity.py does) and every other pixel is held to the bound.  The mono cue equals the reference's lines run
on the same device, bit for bit.  Also: bit-identical reruns, side streams, scenes computed alone, the backward under
deterministic algorithms, the training shape, and the stretch from a UniDepth stand-in to the adapter and the pose loss
under sync debug mode "error"."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from einops import rearrange

from tests import encoder_depth_oracle as O
from tests.test_encoder_depth_cpu import CASES, CUES, DEPTH, PDF, at_pixels, du_args, du_cotangents, reference_mono_cue

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
VAL_TOL, GRAD_TOL = 1e-5, 1e-3


def value_ratio(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isfinite(got), np.isfinite(ref))
    f = np.isfinite(ref)
    return float((np.abs(got[f] - ref[f]) / (VAL_TOL * (np.abs(ref[f]) + 1.0))).max(initial=0.0))


def grad_ratio(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape and np.array_equal(np.isfinite(got), np.isfinite(ref))
    f = np.isfinite(ref)
    rms = math.sqrt(float((ref[f] ** 2).mean())) if f.any() else 0.0
    return float((np.abs(got[f] - ref[f]) / (GRAD_TOL * (np.abs(ref[f]) + rms) + 1e-30)).max(initial=0.0))


def cuda(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def fragile(depth, ss, K, near, far, grid):
    """pixels whose pre-clamp shift or shifted depth lies within float32 rounding of a clamp bound: [b v, h, w]"""
    _, _, (sraw, pre, lo, hi) = O.depth_update_forward(depth, ss, K, near, far, grid)
    tol = 1e-5
    with np.errstate(invalid="ignore"):
        f = (np.abs(np.abs(sraw) - 5.0) <= tol * 6.0) | (np.abs(pre - lo) <= tol * (np.abs(lo) + 1.0)) | \
            (np.abs(pre - hi) <= tol * (np.abs(hi) + 1.0))
    return f


def run_du(depth, ss, K, near, far, grid, gd, gx):
    from pf3plat_b200.encoder_depth import depth_update
    s = cuda(ss).requires_grad_(True)
    depths, xyz = depth_update(cuda(depth), s, cuda(K), cuda(near), cuda(far), grid)
    terms = []
    if gd is not None:
        terms.append((depths * cuda(gd)).sum())
    if gx is not None:
        terms.append((xyz * cuda(gx)).sum())
    sum(terms).backward()
    return depths.detach().cpu().numpy(), xyz.detach().cpu().numpy(), s.grad.cpu().numpy()


def check_du(depth, ss, K, near, far, grid, gd, gx, record=None):
    frag = fragile(depth, ss, K, near, far, grid)
    b, v = np.shape(near)
    h, w = np.shape(depth)[-2:]
    keep = ~frag.reshape(b * v, 1, h, w)
    gd = None if gd is None else np.where(keep, gd, 0.0)
    gx = None if gx is None else np.where(keep.reshape(b, v, 1, h, w), gx, 0.0)
    got_d, got_x, got_g = run_du(depth, ss, K, near, far, grid, gd, gx)
    od, ox, _ = O.depth_update_forward(depth, ss, K, near, far, grid)
    og = O.depth_update_backward(depth, ss, K, near, far, grid, gd, gx)
    r = (value_ratio(got_d, od), value_ratio(got_x, ox), grad_ratio(got_g, og))
    if record is not None:
        r += (value_ratio(at_pixels(got_d, record), record["depths64"]),
              value_ratio(at_pixels(got_x, record), record["xyz64"]))
    assert max(r) <= 1.0, r
    assert (got_g[..., 0] == 0).all()
    return r, int(frag.sum())


@pytest.mark.parametrize("name", DEPTH)
def test_depth_update_matches_the_oracle_and_the_reference_record(name):
    c = CASES[name]
    gd, gx = du_cotangents(c)
    r, nfrag = check_du(*du_args(c), gd, gx, record=c)
    print(f"{name}: ratios {['%.3f' % x for x in r]}, {nfrag} fragile pixels zeroed")


@pytest.mark.parametrize("b,v,h,w,grid", [(1, 2, 64, 64, (28, 28)), (2, 3, 256, 256, (42, 42)),
                                          (3, 2, 48, 80, (37, 29)), (1, 3, 100, 60, (7, 7))])
def test_depth_update_seeded_shapes_and_either_cotangent(b, v, h, w, grid):
    rng = np.random.default_rng(b * 1000 + h)
    near = rng.uniform(0.5, 1.5, (b, v)).astype(np.float32)
    far = (near + rng.uniform(5.0, 50.0, (b, v))).astype(np.float32)
    depth = (rng.uniform(0.2, 1.1, (b * v, 1, h, w)) * far.reshape(-1, 1, 1, 1)).astype(np.float32)
    ss = rng.normal(0.0, 3.0, (b, v, grid[0] * grid[1], 2)).astype(np.float32)
    K = np.tile(np.array([[1.1, 0.0, 0.5], [0.0, 0.9, 0.5], [0.0, 0.0, 1.0]], np.float32), (b, v, 1, 1))
    gd = rng.normal(size=(b * v, 1, h, w)).astype(np.float32)
    gx = rng.normal(size=(b, v, 3, h, w)).astype(np.float32)
    for a, bb in ((gd, gx), (gd, None), (None, gx)):
        check_du(depth, ss, K, near, far, grid, a, bb)


@pytest.mark.parametrize("name", sorted(set(DEPTH) | set(CUES)))
def test_mono_cue_equals_the_reference_route_on_the_device(name):
    """on the recorded depths where the case has them, else on depth_update's own output for the case"""
    from pf3plat_b200.encoder_depth import depth_update, mono_cue
    c = CASES[name]
    b, v = c["near"].shape
    near, far = cuda(c["near"]), cuda(c["far"])
    if "depths32" in c or "depths" in c:
        d = cuda(c["depths32"] if "depths32" in c else c["depths"])
    else:
        depth, ss, K, _, _, grid = du_args(c)
        d = depth_update(cuda(depth), cuda(ss), cuda(K), near, far, grid)[0]
    got = mono_cue(d, near, far, b, v)
    assert torch.equal(got, reference_mono_cue(d, near, far, b, v))
    if "mono_bin32" in c:
        assert np.array_equal(got.argmax(1).cpu().numpy(), c["mono_bin32"].astype(np.int64))


@pytest.mark.parametrize("b,v,h,w,lo,hi", [(1, 2, 64, 64, 1.0, 100.0), (14, 3, 256, 256, 0.5, 100.0),
                                           (3, 3, 48, 80, 0.1, 2.0)])
def test_mono_cue_seeded_shapes_equal_the_reference_route(b, v, h, w, lo, hi):
    from pf3plat_b200.encoder_depth import mono_cue
    g = torch.Generator(device=DEV).manual_seed(h + b)
    near = torch.full((b, v), lo, device=DEV)
    far = torch.full((b, v), hi, device=DEV)
    # depths both in the disparity range the hypotheses span and in the depth range, as the reference compares them
    d = torch.rand((b * v, 1, h, w), generator=g, device=DEV) * (1.0 / lo) * 1.2
    d[: b * v // 2] = d[: b * v // 2] * hi
    assert torch.equal(mono_cue(d, near, far, b, v), reference_mono_cue(d, near, far, b, v))


def run_pdf(logits, s, g):
    from pf3plat_b200.encoder_depth import pdf_peak
    x = cuda(logits).requires_grad_(True)
    out = pdf_peak(x, s)
    (out * cuda(g)).sum().backward()
    return out.detach().cpu().numpy(), x.grad.cpu().numpy()


@pytest.mark.parametrize("name", PDF)
def test_pdf_peak_matches_the_oracle_and_the_reference_record(name):
    c = CASES[name]
    s = int(c["upscale"])
    out, g = run_pdf(c["logits"], s, c["g_pdf"])
    r = (value_ratio(out, O.pdf_peak_forward(c["logits"], s)), grad_ratio(g, O.pdf_peak_backward(c["logits"], s,
                                                                                                  c["g_pdf"])),
         value_ratio(out, c["pdf_max64"]), grad_ratio(g, c["d_logits64"]))
    print(f"{name}: ratios {['%.3f' % x for x in r]}")
    assert max(r) <= 1.0, r


@pytest.mark.parametrize("n,D,h,w,s", [(28, 128, 64, 64, 4), (4, 32, 13, 22, 4), (3, 128, 9, 7, 1), (2, 5, 4, 4, 3)])
def test_pdf_peak_seeded_shapes(n, D, h, w, s):
    rng = np.random.default_rng(n * D + h)
    x = rng.normal(0.0, 3.0, (n, D, h, w)).astype(np.float32)
    g = rng.normal(size=(n, 1, h * s, w * s)).astype(np.float32)
    out, gr = run_pdf(x, s, g)
    if s in (1, 2, 4):
        assert value_ratio(out, O.pdf_peak_forward(x, s)) <= 1.0
        assert grad_ratio(gr, O.pdf_peak_backward(x, s, g)) <= 1.0
    ref = F.interpolate(torch.max(F.softmax(cuda(x), dim=1), dim=1, keepdim=True)[0], scale_factor=s)
    assert value_ratio(out, ref.cpu().numpy()) <= 1.0  # the nearest upsampling's index map, any integer s


def seeded_stretch(b, v, h, w, grid, D=128, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    near = 0.5 + torch.rand((b, v), generator=g, device=DEV)
    far = near + 50.0 + 50.0 * torch.rand((b, v), generator=g, device=DEV)
    depth = (0.2 + torch.rand((b * v, 1, h, w), generator=g, device=DEV)) * 40.0
    ss = torch.randn((b, v, grid[0] * grid[1], 2), generator=g, device=DEV) * 3.0
    K = torch.tensor([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]], device=DEV).expand(b, v, 3, 3).contiguous()
    logits = torch.randn((v * b, D, h // 4, w // 4), generator=g, device=DEV) * 2.0
    cot = [torch.randn(shape, generator=g, device=DEV) for shape in
           ((b * v, 1, h, w), (b, v, 3, h, w), (v * b, 1, h, w))]
    return near, far, depth, ss, K, logits, cot


def stretch(inp, b, v, grid):
    from pf3plat_b200.encoder_depth import depth_update, mono_cue, pdf_peak
    near, far, depth, ss0, K, logits0, (gd, gx, gp) = inp
    ss = ss0.detach().clone().requires_grad_(True)
    logits = logits0.detach().clone().requires_grad_(True)
    depths, xyz = depth_update(depth, ss, K, near, far, grid)
    cue = mono_cue(depths, near, far, b, v)
    peak = pdf_peak(logits, 4)
    ((depths * gd).sum() + (xyz * gx).sum() + (peak * gp).sum()).backward()
    return depths, xyz, cue, peak, ss.grad, logits.grad


def test_bit_identical_reruns_side_streams_and_scenes_alone():
    b, v, h, w, grid = 4, 3, 64, 96, (28, 28)
    inp = seeded_stretch(b, v, h, w, grid, seed=1)
    inp[0].fill_(0.7)  # every scene shares near[0, 0] and far[0, 0], so that a scene alone builds the same hypotheses
    inp[1].fill_(80.0)
    first = stretch(inp, b, v, grid)
    again = stretch(inp, b, v, grid)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        on_side = stretch(inp, b, v, grid)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for x, y, z in zip(first, again, on_side):
        assert torch.equal(x, y) and torch.equal(x, z)
    near, far, depth, ss, K, logits, (gd, gx, gp) = inp
    for s in (0, 2):
        rows, vb = slice(s * v, (s + 1) * v), [vi * b + s for vi in range(v)]
        one = (near[s:s + 1], far[s:s + 1], depth[rows], ss[s:s + 1], K[s:s + 1], logits[vb],
               (gd[rows], gx[s:s + 1], gp[vb]))
        alone = stretch(one, 1, v, grid)
        assert torch.equal(alone[0], first[0][rows]) and torch.equal(alone[1], first[1][s:s + 1])
        assert torch.equal(alone[2], first[2][vb]) and torch.equal(alone[3], first[3][vb])
        assert torch.equal(alone[4], first[4][s:s + 1]) and torch.equal(alone[5], first[5][vb])


def test_backward_under_deterministic_algorithms_and_the_reference_bilinear_backward():
    b, v, h, w, grid = 2, 3, 64, 64, (28, 28)
    inp = seeded_stretch(b, v, h, w, grid, seed=2)
    default = stretch(inp, b, v, grid)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a, bb = stretch(inp, b, v, grid), stretch(inp, b, v, grid)
        x = torch.randn(b * v, 2, 28, 28, device=DEV, requires_grad=True)
        try:  # the reference's :285 under the same flag
            F.interpolate(x, (h, w), mode="bilinear").sum().backward()
            verdict = "runs"
        except RuntimeError as e:
            verdict = f"raises: {str(e).splitlines()[0]}"
    finally:
        torch.use_deterministic_algorithms(prev)
    for x1, x2, x3 in zip(a, bb, default):
        assert torch.equal(x1, x2) and torch.equal(x1, x3)
    print(f"reference bilinear backward under use_deterministic_algorithms(True) on {torch.__version__}: {verdict}")


def test_training_shape():
    b, v, h, w, grid = 14, 3, 256, 256, (28, 28)
    inp = seeded_stretch(b, v, h, w, grid, seed=3)
    depths, xyz, cue, peak, dss, dlog = stretch(inp, b, v, grid)
    near, far, depth, ss, K, logits, (gd, gx, gp) = inp
    assert depths.numel() == 14 * 3 * 256 * 256 and cue.shape == (v * b, 128, 64, 64) and peak.shape == (v * b, 1, 256, 256)
    assert torch.equal(cue, reference_mono_cue(depths.detach(), near, far, b, v))
    for s in (0, 13):  # one scene of each output against the oracle
        rows = slice(s * v, (s + 1) * v)
        args = (depth[rows].cpu().numpy(), ss[s:s + 1].cpu().numpy(), K[s:s + 1].cpu().numpy(),
                near[s:s + 1].cpu().numpy(), far[s:s + 1].cpu().numpy(), grid)
        frag = fragile(*args).reshape(v, 1, h, w)
        assert value_ratio(depths[rows].detach().cpu().numpy(), O.depth_update_forward(*args)[0]) <= 1.0
        assert value_ratio(xyz[s:s + 1].detach().cpu().numpy(), O.depth_update_forward(*args)[1]) <= 1.0
        if not frag.any():
            og = O.depth_update_backward(*args, gd[rows].cpu().numpy(), gx[s:s + 1].cpu().numpy())
            assert grad_ratio(dss[s:s + 1].cpu().numpy(), og) <= 1.0
        vb = [vi * b + s for vi in range(v)]
        lg = logits[vb].cpu().numpy()
        assert value_ratio(peak[vb].detach().cpu().numpy(), O.pdf_peak_forward(lg, 4)) <= 1.0
        assert grad_ratio(dlog[vb].cpu().numpy(), O.pdf_peak_backward(lg, 4, gp[vb].cpu().numpy())) <= 1.0


def test_the_depth_stretch_runs_without_a_host_synchronisation():
    """UniDepth stand-in -> depth_update -> mono_cue and pdf_peak -> the adapter (:529-533) and the pose loss's terms,
    forward and backward, with the drop-in lines of INTEGRATION.md 4"""
    from pf3plat_b200 import losses
    from pf3plat_b200.adapter import GaussianAdapter, GaussianAdapterCfg
    from pf3plat_b200.encoder_depth import depth_update, mono_cue, pdf_peak
    from tests.pose_loss_cases import seeded_case
    b, v, h, w, grid = 2, 3, 64, 64, (28, 28)
    near, far, depth, ss0, K, logits0, _ = seeded_stretch(b, v, h, w, grid, seed=4)
    case = seeded_case(b, v, h, w, 50, 200, seed=5).to(DEV)
    corre, conf = case.matches()
    adapter = GaussianAdapter(GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=2)).cuda()
    c2w = torch.eye(4, device=DEV).repeat(b, v, 1, 1)
    raw = torch.randn(b, 2, h * w, 1, 1, 7 + 3 * 9, device=DEV, requires_grad=True)
    xy = torch.rand(b, 2, h * w, 1, 1, 2, device=DEV)
    opac = torch.rand(b, 2, h * w, 1, 1, device=DEV)

    def run(check):
        ss = ss0.clone().requires_grad_(True)
        logits = logits0.clone().requires_grad_(True)
        if check:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            depths, xyz = depth_update(depth, ss, K, near, far, grid)
            cue = mono_cue(depths, near, far, b, v)
            peak = pdf_peak(logits, 4)
            L3, L2 = losses.pose_terms(case.abspose, depths, xyz, K, corre, conf, h, w)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        # the adapter inverts K with torch's synchronising .inverse() (outside this stretch)
        g = adapter.forward(rearrange(c2w, "b v i j -> b v () () () i j")[:, (0, -1)],
                            rearrange(K, "b v i j -> b v () () () i j")[:, (0, -1)], xy,
                            rearrange(depths, "(b v) 1 h w -> b v (h w) 1 1", b=b, v=v)[:, (0, -1)], opac, raw, (h, w))
        loss = L3.sum() + L2.sum() + g.means.square().mean() + (peak * cue[:, :1].repeat_interleave(4, -1)
                                                                 .repeat_interleave(4, -2)).sum()
        if check:
            torch.cuda.set_sync_debug_mode("error")
        try:
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        return ss.grad, logits.grad

    run(False)  # warm up: library load, the linspace table, the pose loss's pinned pool
    dss, dlog = run(True)
    assert torch.isfinite(dss).all() and torch.isfinite(dlog).all()
    assert dss[..., 1].abs().sum() > 0 and (dss[..., 0] == 0).all()


def test_inputs_are_refused():
    from pf3plat_b200.encoder_depth import depth_update, mono_cue, pdf_peak
    b, v, h, w, grid = 1, 2, 16, 16, (4, 4)
    near, far, depth, ss, K, logits, _ = seeded_stretch(b, v, h, w, grid, D=8)
    with pytest.raises(ValueError, match="must not require grad"):
        depth_update(depth.clone().requires_grad_(True), ss, K, near, far, grid)
    with pytest.raises(TypeError, match="float32"):
        depth_update(depth.double(), ss, K, near, far, grid)
    with pytest.raises(ValueError, match="scale_shift"):
        depth_update(depth, ss, K, near, far, (4, 5))
    with pytest.raises(ValueError, match="multiples of 4"):
        mono_cue(depth[..., :14], near, far, b, v)
    with pytest.raises(TypeError, match="float32"):
        pdf_peak(logits.half())
    with pytest.raises(ValueError, match="integer"):
        pdf_peak(logits, 2.5)
