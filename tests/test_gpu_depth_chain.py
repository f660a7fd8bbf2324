"""GPU parity of the fused depth channel's backward and of the adapter -> decoder gradient chain.

Depth gradients here are signed, seeded normal fields that differ per pixel and per view, so that reading dL/ddepth at
the wrong pixel or view, or losing part of its sum, changes the result; and the depth term is either the whole loss or at
least 30 % of dL/dmeans3D, not a 1e-3 afterthought next to an MSE.  The cameras are turned (their view matrices are not
symmetric), so that a row / column mix-up of the view matrix shows.  References: the batched CPU oracle in fp64
(tests/batch_oracle.py), the adapter -> decoder chain oracle (tests/chain_oracle.py), the reference's two-pass depth route
(tests/ref_callsite.py) and the adapter oracle (oracle/adapter_oracle.py).

Criteria are tests/util.py's (element-wise 1e-3 gradient rule, 1e-2 for Gaussians at a fragile decision); per-camera
gradients -- sums over Gaussians -- use that rule carried through the sum (tests/chain_oracle.camera_grad_check).  Every
test asserts, on the oracle's intermediates, that its regime was reached, and prints "[regime]" lines."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import Scene, make_scene, make_target
from tests import test_gpu_adapter as gpu_adapter
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.chain_oracle import ChainOracle, DecoderOracle, camera_grad_check, default_sh_rotation, make_chain_inputs
from tests.regimes import opaque_stack_scene
from tests.test_gpu_regimes import _check_grads, _check_images, _settings, _termination
from tests.util import check_grad, check_image_strict

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _turned(sc: Scene, seed: int, angle: float = 0.12) -> Scene:
    """sc with every camera turned by `angle` radians about a random axis perpendicular to its optical axis, through the
    point 6 units ahead of it (a turn about the optical axis alone would keep the view matrix's third row and column
    equal)."""
    g = torch.Generator().manual_seed(seed)
    V = sc.extrinsics.shape[0]
    ext = sc.extrinsics.double()
    ahead = ext @ torch.tensor([0.0, 0.0, 6.0, 1.0], dtype=torch.float64)
    phi = 2 * torch.pi * torch.rand(V, generator=g, dtype=torch.float64)
    K = torch.zeros(V, 3, 3, dtype=torch.float64)
    K[:, 0, 2], K[:, 1, 2] = angle * torch.sin(phi), -angle * torch.cos(phi)      # axis (cos phi, sin phi, 0)
    turn = torch.eye(4, dtype=torch.float64).repeat(V, 1, 1)
    turn[:, :3, :3] = torch.linalg.matrix_exp(K - K.transpose(-1, -2))
    shift = lambda p: torch.cat([torch.cat([torch.eye(3, dtype=torch.float64).expand(V, 3, 3), p[:, :3, None]], -1),
                                 torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64).expand(V, 1, 4)], 1)
    kw = dict(sc.__dict__)
    kw["extrinsics"] = (shift(ahead) @ turn @ shift(-ahead) @ ext).float()
    return Scene(**kw)


def _asymmetry(cams) -> float:
    """Smallest, over the views, |third row - third column| of the world->camera rotation."""
    vm = cams["viewmatrix"].double().cpu()                 # transposed: vm[:3, 2] is the third ROW of w2c
    return float((vm[:, :3, 2] - vm[:, 2, :3]).norm(dim=-1).min())


def _depth_field(V, hw, seed):
    """Seeded signed normal weights, different at every pixel of every view."""
    rng = np.random.default_rng(seed)
    return rng.standard_normal((V, *hw)) / (hw[0] * hw[1])


def _leaves(ins, dev, means2D_views=None):
    leaves = {k: v.to(dev).clone().requires_grad_(True) for k, v in ins.items()}
    if means2D_views is not None:
        P = ins["means3D"].shape[1]
        leaves["means2D"] = torch.zeros(means2D_views, P, 3, device=dev, requires_grad=True)
    return leaves


def _run(bs, ins, dL=None, dLd=None):
    """rasterize_batch with means2D; backward of <dL, colour> + <dLd, depth> (either may be None: that output is left out
    of the loss).  Returns (outputs, {name: grad})."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = bs.viewmatrix.device
    leaves = _leaves(ins, dev, bs.viewmatrix.shape[0])
    out = rasterize_batch(bs, **leaves)
    outs, grads = [], []
    if dL is not None:
        outs.append(out[0]); grads.append(torch.as_tensor(dL, dtype=torch.float32, device=dev))
    if dLd is not None:
        outs.append(out[2]); grads.append(torch.as_tensor(dLd, dtype=torch.float32, device=dev))
    torch.autograd.backward(outs, grads)
    return [o.detach() for o in out], {k: t.grad for k, t in leaves.items()}


def _check_depth(depth, ob, label):
    for v, r in enumerate(ob.views):
        derr = np.abs(depth[v].cpu().numpy() - r.depth)[~r.px_fragile].max()
        assert derr <= 1e-3, (label, v, derr)


# ---------------------------------------------------------------------------------------------------------------------
# 1.-3. the fused depth channel of rasterize_batch
# ---------------------------------------------------------------------------------------------------------------------
_VPS = 9
_NEAR = 1.0 / np.tile(np.linspace(0.8, 1.25, _VPS), 2)


def _depth_batch(geometry, P=1500, hw=(32, 48)):
    """S = 2 scenes x 9 views (camera chunks 8 + 1), per-view view_scale 0.8 .. 1.25, turned cameras.
    geometry "cov3D": shs + cov3D_precomp; "scalerot": per-view colors_precomp + scales + rotations (norms 0.6 .. 1.5)."""
    scenes = [_turned(make_scene(P, _VPS, *hw, seed=300 + k), seed=310 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=_NEAR)
    out = {"means3D": ins["means3D"], "opacities": ins["opacities"]}
    if geometry == "cov3D":
        out["shs"], out["cov3D_precomp"] = ins["shs"], ins["cov3D_precomp"]
    else:
        g = torch.Generator().manual_seed(8)
        out["colors_precomp"] = torch.rand(2 * _VPS, P, 3, generator=g)
        out["scales"] = ins["scales"]
        out["rotations"] = (ins["rotations"] * torch.linspace(0.6, 1.5, 2 * P).reshape(2, P, 1)).contiguous()
    return cams, out, hw


def _assert_depth_regime(label, cams, ob, w):
    asym = _asymmetry(cams)
    corr = float(np.corrcoef(w[0].ravel(), w[1].ravel())[0, 1])
    print(f"[regime] {label}: S={ob.S} VPS={ob.VPS} view_scale {ob.s.min():.3f}..{ob.s.max():.3f}; visible per view "
          f"{(ob.radii > 0).sum(axis=1).min()}..{(ob.radii > 0).sum(axis=1).max()}; view-matrix row/column gap "
          f">= {asym:.3f}; depth weights: mean {w.mean():.2e}, std {w.std():.2e}, corr(view 0, view 1) {corr:.3f}")
    assert ob.VPS > 8 and len(set(np.round(ob.s, 6).tolist())) == _VPS and (np.abs(ob.s - 1) > 0.02).all()
    assert asym > 0.05
    assert abs(corr) < 0.1 and np.abs(w.mean()) < 0.1 * w.std()
    assert (ob.radii > 0).mean() > 0.3


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_depth_only_backward_matches_fp64_oracle_under_every_compositor(geometry):
    from pf3plat_b200._capi import GS_TUNE_BWD_OCC4, GS_TUNE_BWD_V1, GS_TUNE_PBWD_2PHASE
    dev = _dev()
    cams, ins, hw = _depth_batch(geometry)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    w = _depth_field(ob.V, hw, seed=41)
    _assert_depth_regime(f"depth only, {geometry}", cams, ob, w)
    gref = ob.backward(np.zeros((ob.V, 3, *hw)), w)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    for tuning, label in ((0, "default"), (GS_TUNE_BWD_V1, "bwd v1"), (GS_TUNE_BWD_OCC4, "bwd occ4"),
                          (GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd")):
        (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True, tuning=tuning), ins, dLd=w)
        _check_depth(depth, ob, label)
        zero = "shs" if "shs" in grads else "colors_precomp"
        assert int(torch.count_nonzero(grads.pop(zero))) == 0, (label, zero)
        assert set(grads) == {k for k in gref if gref[k] is not None} - {zero}
        _check_grads(f"depth only {geometry} {label}", grads, gref, aff, ob.VPS)


def test_depth_and_colour_at_comparable_weight():
    dev = _dev()
    cams, ins, hw = _depth_batch("cov3D")
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    target = make_target(ob.V, *hw, seed=3).numpy()
    dL = 2 * (ob.color - target) / target.size
    w = _depth_field(ob.V, hw, seed=42)
    gc = ob.backward(dL)["means3D"]
    gd = ob.backward(np.zeros_like(dL), w)["means3D"]
    lam = float(np.linalg.norm(gc) / np.linalg.norm(gd))
    dLd = lam * w
    share = np.linalg.norm(lam * gd) / (np.linalg.norm(gc) + np.linalg.norm(lam * gd))
    print(f"[regime] colour MSE + depth: depth weight {lam:.3e}, depth share of |dL/dmeans3D| {share:.1%}, "
          f"|colour + depth| / |colour| {np.linalg.norm(gc + lam * gd) / np.linalg.norm(gc):.3f}")
    assert share >= 0.3
    gref = ob.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dL=dL, dLd=dLd)
    _check_images(color, ob, "colour + depth", depth=depth)
    _check_grads("colour + depth", grads, gref, ob.affected(), ob.VPS)


def test_depth_flag_with_null_depth_gradient_matches_the_colour_only_kernels():
    """with_depth=True and a colour-only loss: the backward is handed a NULL dL_ddepth (the autograd engine would
    materialise a zero tensor, so the backward node is applied directly) -- the DEPTH=true kernels must give the
    with_depth=False gradients (2e-5 relative: the same sums in another association) and the oracle's."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = _dev()
    cams, ins, hw = _depth_batch("cov3D")
    ob = oracle_batch(_settings(cams, hw), dtype=np.float64, **ins)
    target = make_target(ob.V, *hw, seed=4).numpy()
    dL = 2 * (ob.color - target) / target.size
    dcams = {k: v.to(dev) for k, v in cams.items()}
    _, plain = _run(_settings(dcams, hw), ins, dL=dL)
    leaves = _leaves(ins, dev, ob.V)
    out = rasterize_batch(_settings(dcams, hw, with_depth=True), **leaves)
    assert len(out) == 3
    g = out[0].grad_fn.apply(torch.as_tensor(dL, dtype=torch.float32, device=dev), None, None)
    names = ("means3D", "means2D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")
    nulled = {k: t for k, t in zip(names, g) if t is not None}
    print(f"[regime] NULL dL_ddepth under GS_FLAG_DEPTH: gradients returned {sorted(nulled)}")
    assert set(nulled) == set(plain)
    for k, a in nulled.items():
        b = plain[k]
        err = float((a - b).abs().max())
        assert err <= 2e-5 * float(b.abs().max()) + 1e-12, (k, err, float(b.abs().max()))
    _check_grads("NULL dL_ddepth", nulled, ob.backward(dL), ob.affected(), ob.VPS)


# ---------------------------------------------------------------------------------------------------------------------
# 4. depth-only loss in the hard regimes
# ---------------------------------------------------------------------------------------------------------------------
def test_depth_only_on_opaque_stacks_matches_fp64_oracle():
    dev = _dev()
    hw = (48, 64)
    sc = _turned(opaque_stack_scene(6, 10, 2, *hw, seed=110), seed=111, angle=0.05)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    for v, r in enumerate(ob.views):
        early, t_next, raw_alpha = _termination(r)
        print(f"[regime] opaque stacks, depth only, view {v}: early-terminated pixels {early.mean():.1%}, Gaussians at "
              f"the 0.99 clamp {int((raw_alpha >= 0.99).sum())}, fragile pixels {r.px_fragile.mean():.2%}")
        assert early.mean() >= 0.3 and np.nanmax(t_next) < 1e-4 and (raw_alpha >= 0.99).any()
    w = _depth_field(ob.V, hw, seed=43)
    gref = ob.backward(np.zeros((ob.V, 3, *hw)), w)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dLd=w)
    _check_depth(depth, ob, "opaque stacks")
    assert int(torch.count_nonzero(grads.pop("shs"))) == 0
    # every Gaussian held to the strict rule, as the opaque-stack colour test does
    _check_grads("opaque stacks depth only vs fp64", grads, gref, np.zeros((ob.S, ob.P), bool), ob.VPS)


def test_depth_only_with_huge_footprints_matches_fp64_oracle():
    """x400 footprints: every Gaussian covers most of the image, and the compositor's per-block moment sums are shifted
    by hundreds of pixels to its own offset -- for the depth term's sum as for the others."""
    dev = _dev()
    views, P, hw = 2, 24, (48, 80)
    sc = make_scene(P, views, *hw, seed=17)
    sc.covariances.mul_(400.0)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    ntiles = ((hw[0] + 15) // 16) * ((hw[1] + 15) // 16)
    for v, r in enumerate(ob.views):
        print(f"[regime] huge footprints, depth only, view {v}: max radius {int(r.radii.max())} px, Gaussians touching "
              f"every tile {int((r.tiles_touched == ntiles).sum())} of {P}")
        assert r.radii.max() >= max(hw) and (r.tiles_touched == ntiles).sum() >= P // 3
    w = _depth_field(ob.V, hw, seed=44)
    gref = ob.backward(np.zeros((ob.V, 3, *hw)), w)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    (color, radii, depth), grads = _run(_settings(dcams, hw, with_depth=True), ins, dLd=w)
    assert int(torch.count_nonzero(grads.pop("shs"))) == 0
    _check_grads("huge footprints depth only", grads, gref, np.zeros((ob.S, ob.P), bool), ob.VPS)


# ---------------------------------------------------------------------------------------------------------------------
# 5. decoder_forward(depth_mode="depth"), fused route
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("near", [0.5, 2.0])
def test_decoder_fused_depth_gradient_matches_chain_oracle_and_two_pass_route(near):
    from pf3plat_b200.render import decoder_forward
    from tests.ref_callsite import render_depth_like_reference
    dev = _dev()
    b, v, P, hw = 2, 3, 1500, (48, 64)
    scs = [_turned(make_scene(P, v, *hw, seed=320 + k), seed=330 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs])
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), near), torch.full((b, v), 100.0 * near)
    bg = torch.tensor([0.3, 0.2, 0.1])
    names = ("means", "covariances", "harmonics", "opacities")
    w = _depth_field(b * v, hw, seed=45)
    # the GPU, fused route (extrinsics without grad)
    lg = [st(n).to(dev).requires_grad_(True) for n in names]
    color, depth = decoder_forward(*lg, ext.to(dev), intr.to(dev), nr.to(dev), fr.to(dev), hw, bg.to(dev),
                                   depth_mode="depth")
    (depth * torch.as_tensor(w, dtype=torch.float32, device=dev).reshape(b, v, *hw)).sum().backward()
    # the chain oracle
    lo = [st(n).double().requires_grad_(True) for n in names]
    dec = DecoderOracle(*lo, ext, intr, nr, fr, hw, bg)
    dec.backward(np.zeros((b * v, 3, *hw)), w)
    aff = dec.affected().reshape(-1)
    # the reference's two-pass route: camera-space z rendered as a colour, per view, Gaussians repeated
    lr = [st(n).to(dev).requires_grad_(True) for n in names]
    flat = lambda t: t.reshape(b * v, *t.shape[2:]).to(dev)
    rep = lambda t: t.repeat_interleave(v, dim=0)
    rd = render_depth_like_reference(flat(ext), flat(intr), flat(nr), flat(fr), hw, rep(lr[0]), rep(lr[1]), rep(lr[3]))
    (rd * torch.as_tensor(w, dtype=torch.float32, device=dev)).sum().backward()
    print(f"[regime] decoder depth, near {near}: view_scale {1 / near:g}, view-matrix row/column gap "
          f"{_asymmetry({'viewmatrix': torch.linalg.inv(flat(ext).cpu()).transpose(-1, -2)}):.3f}, visible per view "
          f"{(dec.ob.radii > 0).sum(axis=1).tolist()}, affected {int(aff.sum())}")
    assert (dec.ob.radii > 0).mean() > 0.3 and abs(float(dec.ob.s[0]) - 1 / near) < 1e-6
    for v_, r in enumerate(dec.ob.views):
        check_image_strict(color.reshape(b * v, 3, *hw)[v_], r, 0.03, label=f"decoder near {near} view {v_}")
    dd = np.abs(depth.detach().reshape(b * v, *hw).cpu().numpy() - dec.depth)
    frag = np.stack([r.px_fragile for r in dec.ob.views])
    assert dd[~frag].max() <= 1e-4 * np.abs(dec.depth).max(), dd[~frag].max()
    assert int(torch.count_nonzero(lg[2].grad)) == 0 and lr[2].grad is None
    for k, (a, o, r) in enumerate(zip(lg, lo, lr)):
        if k == 2:
            continue
        n = names[k]
        check_grad(f"decoder near {near} dL/d{n} vs chain oracle", a.grad.reshape(b * P, -1), o.grad.reshape(b * P, -1),
                   aff)
        check_grad(f"decoder near {near} dL/d{n} vs two-pass route", a.grad.reshape(b * P, -1),
                   r.grad.reshape(b * P, -1).cpu().numpy(), aff)
    assert not lg[1].grad.reshape(-1, 9)[:, [3, 6, 7]].any()          # the index_select backward: upper triangle only


# ---------------------------------------------------------------------------------------------------------------------
# 6. adapter -> decoder, as PF3plat trains through it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pose_grad", [False, True])
def test_adapter_to_decoder_chain_matches_chain_oracle(pose_grad):
    """b = 2 scenes, 2 context views of 24 x 32 each, sh_degree 4 with the SH rotation derived from the (proper)
    extrinsics, 3 target views per scene at 48 x 64, near 0.5, background (0.3, 0.2, 0.1), loss = MSE + <w, depth>.
    pose_grad: the target extrinsics require grad, so decoder_forward takes the two-pass route."""
    from pf3plat_b200.adapter import GaussianAdapter, GaussianAdapterCfg
    from pf3plat_b200.render import decoder_forward
    dev = _dev()
    b, vc, vt, chw, hw, deg = 2, 2, 3, (24, 32), (48, 64), 4
    inp = make_chain_inputs(61, b, vc, chw, vt, deg, 0.5)
    bg = torch.tensor([0.3, 0.2, 0.1])
    R = chw[0] * chw[1]
    G = vc * R
    ch = ChainOracle(inp["extrinsics"], inp["intrinsics"], inp["coordinates"], inp["depths"], inp["opacities"],
                     inp["raw_gaussians"], chw, deg, inp["target_extrinsics"], inp["target_intrinsics"], inp["near"],
                     inp["far"], hw, bg, two_pass=pose_grad)
    V = b * vt
    target = make_target(V, *hw, seed=6).numpy()
    dL = 2 * (ch.color - target) / target.size
    dLd = 0.1 * _depth_field(V, hw, seed=46) * (hw[0] * hw[1]) / target.size
    ch.backward(dL, dLd)
    ref = ch.grads()
    aff = ch.affected()
    D = ch.decoder
    rot = default_sh_rotation(inp["extrinsics"], (deg + 1) ** 2)
    print(f"[regime] adapter -> decoder ({'two-pass' if pose_grad else 'fused'} route): G per scene {G}, visible per "
          f"view {(D.ob.radii > 0).sum(axis=1).tolist()}, affected {int(aff.sum())}, SH rotation derived from the "
          f"extrinsics: {rot is not None}")
    assert (D.ob.radii > 0).mean() > 0.5 and (D.ob_depth is not None) == pose_grad and rot is not None
    # the GPU
    L = {k: inp[k].to(dev).requires_grad_(True) for k in ("extrinsics", "intrinsics", "coordinates", "depths",
                                                          "opacities", "raw_gaussians")}
    adapter = GaussianAdapter(GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=deg)).to(dev)
    g = adapter.forward(L["extrinsics"][:, :, None], L["intrinsics"][:, :, None], L["coordinates"], L["depths"],
                        L["opacities"], L["raw_gaussians"], chw)
    text = inp["target_extrinsics"].to(dev).requires_grad_(pose_grad)
    color, depth = decoder_forward(g.means.reshape(b, G, 3), g.covariances.reshape(b, G, 3, 3),
                                   g.harmonics.reshape(b, G, 3, -1), g.opacities.reshape(b, G), text,
                                   inp["target_intrinsics"].to(dev), inp["near"].to(dev), inp["far"].to(dev), hw,
                                   bg.to(dev), depth_mode="depth")
    f32 = lambda a: torch.as_tensor(a, dtype=torch.float32, device=dev)
    torch.autograd.backward([color, depth], [f32(dL).reshape(color.shape), f32(dLd).reshape(depth.shape)])
    for v_, r in enumerate(D.ob.views):
        check_image_strict(color.reshape(V, 3, *hw)[v_], r, 0.03, label=f"chain view {v_}")
    frag = np.stack([r.px_fragile for r in D.ob.views])
    dd = np.abs(depth.detach().reshape(V, *hw).cpu().numpy() - ch.depth)
    assert dd[~frag].max() <= 1e-4 * np.abs(ch.depth).max(), dd[~frag].max()
    label = "two-pass" if pose_grad else "fused"
    a = aff.reshape(-1)
    raw, rraw = L["raw_gaussians"].grad.reshape(b * G, -1), ref["raw_gaussians"].reshape(b * G, -1)
    for part, sl in (("scales", slice(0, 3)), ("rotations", slice(3, 7)), ("sh", slice(7, None))):
        check_grad(f"chain {label} dL/draw[{part}]", raw[:, sl], rraw[:, sl], a)
    for k in ("depths", "coordinates", "opacities"):
        check_grad(f"chain {label} dL/d{k}", L[k].grad.reshape(b * G, -1), ref[k].reshape(b * G, -1), a)
    for k in ("extrinsics", "intrinsics"):
        camera_grad_check(f"chain {label} dL/dcontext {k}", L[k].grad, ref[k], ch.contributions(k), aff)
    if pose_grad:
        aff_t = np.repeat(ch.decoder.affected()[:, None], vt, axis=1)          # (b, vt, G)
        camera_grad_check(f"chain {label} dL/dtarget extrinsics", text.grad, ref["target_extrinsics"],
                          ch.contributions("target_extrinsics"), aff_t)
    else:
        assert text.grad is None


# ---------------------------------------------------------------------------------------------------------------------
# 7. adapter kernels: NULL incoming gradients, SH degrees 1 and 2
# ---------------------------------------------------------------------------------------------------------------------
def test_adapter_backward_null_incoming_gradients_are_zeros():
    """gs_adapter_backward with NULL dL/dscales and dL/drotations, then also NULL dL/dharmonics ("NULL = zero" in
    GsAdapterOutGrads): the per-Gaussian gradients bit for bit those of the call with zero-filled buffers, the per-camera
    sums equal up to their atomic accumulation order, and an exactly zero raw SH gradient.  A call with
    non-zero incoming gradients runs right before each NULL call, so that what it leaves in shared memory would show."""
    import os
    import sys
    from oracle import adapter_oracle
    from pf3plat_b200 import _capi
    from pf3plat_b200.sh_rotation import sh_rotation_blocks
    dev = _dev()
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    import make_adapter_golden as mk
    V, R, deg = 2, 1001, 4
    d = (deg + 1) ** 2
    inp = mk.make_inputs(23, 1, V, 1, R, deg)
    f = lambda t, *s: t.reshape(*s).float().contiguous().to(dev)
    ext, intr = f(inp["extrinsics"], V, 4, 4), f(inp["intrinsics"], V, 3, 3)
    kinv = torch.linalg.inv(intr).contiguous()
    pixel = 1 / torch.tensor((R, 1), dtype=torch.float32, device=dev)
    mult = (0.1 * torch.einsum("vij,j->vi", torch.linalg.inv(intr[:, :2, :2]), pixel)).sum(-1).contiguous()
    D = sh_rotation_blocks(ext[:, :3, :3].cpu(), d).float().contiguous().to(dev)
    mask = adapter_oracle.sh_mask(deg).to(dev)
    coords, depths, raw = f(inp["coordinates"], V, R, 2), f(inp["depths"], V, R), f(inp["raw_gaussians"], V, R, -1)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    cfg = _capi.GsAdapterConfig(V=V, R=R, d_sh=d, scale_min=0.5, scale_max=15.0, eps=1e-8, c2w=p(ext), kinv=p(kinv),
                                multiplier=p(mult), sh_rotation=p(D), sh_mask=p(mask))
    ain = _capi.GsAdapterInputs(coordinates=p(coords), depths=p(depths), raw_gaussians=p(raw))
    g = torch.Generator().manual_seed(9)
    rn = lambda *s: torch.randn(*s, generator=g).to(dev)
    gm, gc, gh, gs, gr = rn(V, R, 3), rn(V, R, 3, 3), rn(V, R, d, 3), rn(V, R, 3), rn(V, R, 4)

    def call(harm, scales, rot):
        out = {"coordinates": torch.full((V, R, 2), float("nan"), device=dev),
               "depths": torch.full((V, R), float("nan"), device=dev),
               "raw_gaussians": torch.full((V, R, 7 + 3 * d), float("nan"), device=dev),
               "c2w": torch.full((V, 4, 4), float("nan"), device=dev), "kinv": torch.full((V, 3, 3), float("nan"), device=dev),
               "multiplier": torch.full((V,), float("nan"), device=dev)}
        gout = _capi.GsAdapterOutGrads(means=p(gm), covariances=p(gc), harmonics=p(harm), scales=p(scales), rotations=p(rot))
        gin = _capi.GsAdapterInGrads(**{k: p(t) for k, t in out.items()})
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(_capi.lib().gs_adapter_backward(ctypes.byref(cfg), ctypes.byref(ain), ctypes.byref(gout),
                                                    ctypes.byref(gin), stream))
        torch.cuda.synchronize(dev)
        return out

    z3, z4, zh = torch.zeros_like(gs), torch.zeros_like(gr), torch.zeros_like(gh)
    full = call(gh, gs, gr)
    zero_sr = call(gh, z3, z4)
    call(gh, gs, gr)
    null_sr = call(gh, None, None)
    zero_all = call(zh, z3, z4)
    call(gh, gs, gr)
    null_all = call(None, None, None)
    sh_full = full["raw_gaussians"][..., 7:]
    print(f"[regime] adapter NULL gradients: V={V} R={R} d_sh={d} (tail block {R % 128} Gaussians); max |raw SH grad| "
          f"with harmonics {float(sh_full.abs().max()):.3e}; scales/rotations change dL/draw: "
          f"{not torch.equal(full['raw_gaussians'], zero_sr['raw_gaussians'])}")
    assert float(sh_full.abs().max()) > 0 and not torch.equal(full["raw_gaussians"], zero_sr["raw_gaussians"])
    for k in full:
        assert torch.isfinite(null_sr[k]).all() and torch.isfinite(null_all[k]).all(), k
        if k in ("c2w", "kinv", "multiplier"):
            # per-camera sums, accumulated by one atomic add per CTA in whatever order the CTAs finish: the same terms,
            # so equal up to the rounding of that order
            for a, z in ((null_sr[k], zero_sr[k]), (null_all[k], zero_all[k])):
                assert float((a - z).abs().max()) <= 1e-5 * float(z.abs().max()), k
        else:
            assert torch.equal(null_sr[k], zero_sr[k]), k
            assert torch.equal(null_all[k], zero_all[k]), k
    assert int(torch.count_nonzero(null_all["raw_gaussians"][..., 7:])) == 0


@pytest.mark.parametrize("b,v,r,deg", [(2, 3, 131, 1), (1, 2, 1001, 1), (2, 3, 131, 2), (1, 2, 1001, 2)])
def test_adapter_kernels_match_oracle_at_sh_degrees_1_and_2(b, v, r, deg):
    """d_sh 4 and 9: raw rows of 76 B and 136 B, harmonics rows of 48 B and 108 B -- sizes no other test stages -- with
    ragged Gaussian counts, against the fp64 adapter oracle at the adapter tests' tolerances."""
    print(f"[regime] adapter sh_degree {deg}: raw row {4 * (7 + 3 * (deg + 1) ** 2)} B, R={r} (tail block {r % 128})")
    gpu_adapter.test_kernels_match_oracle_on_larger_and_ragged_inputs(b, v, r, deg)
