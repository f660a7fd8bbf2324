"""GPU parity of the fused depth channel's camera gradient: dL/ddepth -> camera-space z -> the z column of each view
matrix (flat entries 2, 6, 10, 14 of the transposed matrix) -> the extrinsics, the one camera gradient the reference's
depth pass has (render_depth_cuda builds its fake colour z = (extrinsics^-1 @ mean).z in torch, cuda_splatting.py:239-242).

The oracle is that construction in fp64: the batched CPU oracle renders colors_precomp = z on a black background, its
colour gradient per (view, Gaussian) is dL/dz, and dL/dviewmatrix_z is its sum against (view_scale * mean, 1).  Per-view
sums over Gaussians are held to tests/chain_oracle.camera_grad_check (the element-wise 1e-3 rule carried through the sum,
with 1e-2 slack for the Gaussians at a fragile decision).  The other 12 entries of the view-matrix gradient must be
exactly 0.  Depth weights are seeded signed fields that differ per pixel and view; cameras are turned, so that the view
matrix's third row and third column differ.  Every test prints "[regime]" lines and asserts its regime was reached.
The adapter -> decoder chain with a pose gradient, against ChainOracle(two_pass=True), is
tests/test_gpu_depth_chain.py::test_adapter_to_decoder_chain_matches_chain_oracle."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.chain_oracle import DecoderOracle, camera_grad_check
from tests.regimes import edge_straddle_scene, opaque_stack_scene
from tests.test_gpu_backward_paths import PATH_RTOL, _agree, _stream_ctx
from tests.test_gpu_depth_chain import _asymmetry, _depth_batch, _depth_field, _leaves, _turned
from tests.test_gpu_regimes import _settings
from tests.util import check_grad

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def view_z_oracle(cams, hw, ins, w):
    """The reference's construction in fp64 for the batch (cams, ins) under the depth weights w [V,H,W].
    Returns (ref [V,4], per-Gaussian contributions [V,P,4], affected [V,P], the oracle)."""
    bs = _settings(cams, hw)
    V = bs.viewmatrix.shape[0]
    geo = {k: v for k, v in ins.items() if k not in ("shs", "colors_precomp")}
    means = ins["means3D"].double().cpu().numpy()
    S, P = means.shape[:2]
    VPS = V // S
    s = bs.view_scale.cpu().numpy().astype(np.float32).astype(np.float64)        # held in fp32, as the kernels do
    vm = bs.viewmatrix.double().cpu().numpy()                                     # transposed: [:, :, 2] is the z column
    hom = np.concatenate([means[np.arange(V) // VPS] * s[:, None, None], np.ones((V, P, 1))], -1)   # (s m, 1)
    z = np.einsum("vpj,vj->vp", hom, vm[:, :, 2])
    ob = oracle_batch(bs._replace(bg=torch.zeros(V, 3)), colors_precomp=np.repeat(z[..., None], 3, -1),
                      dtype=np.float64, **geo)
    gz = ob.backward(np.repeat(np.asarray(w, np.float64)[:, None] / 3.0, 3, axis=1))["colors_precomp"].sum(-1)
    contrib = gz[..., None] * hom
    return contrib.sum(axis=1), contrib, np.repeat(ob.affected(), VPS, axis=0), ob


def _gpu(cams_dev, hw, ins, w, tuning=0, view_grad=True):
    """rasterize_batch with depth, Gaussians requiring grad and (view_grad) a view matrix requiring grad; backward of
    <w, depth>.  Returns (view-matrix gradient or None, {Gaussian input: grad}, outputs)."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = cams_dev["viewmatrix"].device
    vm = cams_dev["viewmatrix"].clone().requires_grad_(view_grad)
    bs = _settings({**cams_dev, "viewmatrix": vm}, hw, with_depth=True, tuning=tuning)
    leaves = _leaves(ins, dev)
    out = rasterize_batch(bs, **leaves)
    out[2].backward(torch.as_tensor(w, dtype=torch.float32, device=dev))
    return vm.grad, {k: t.grad for k, t in leaves.items()}, [o.detach() for o in out]


def _check_view_grad(label, got, ref, contrib, aff):
    V = ref.shape[0]
    assert got is not None and got.shape == (V, 4, 4) and got.dtype == torch.float32, label
    rest = got.clone()
    rest[:, :, 2] = 0
    assert int(torch.count_nonzero(rest)) == 0, f"{label}: gradient outside the z column"
    return camera_grad_check(label, got[:, :, 2], ref, contrib, aff)


def _assert_regime(label, cams, ob, ref, turned=True):
    asym = _asymmetry(cams)
    vis = (ob.radii > 0).sum(axis=1)
    print(f"[regime] {label}: S={ob.S} VPS={ob.VPS} P={ob.P}, view_scale {ob.s.min():.3f}..{ob.s.max():.3f}, visible "
          f"per view {vis.min()}..{vis.max()}, view-matrix row/column gap >= {asym:.3f}, |dL/dviewmatrix_z| per view "
          f"{np.abs(ref).max(axis=1).min():.2e}..{np.abs(ref).max(axis=1).max():.2e}")
    assert vis.min() > 0 and (np.abs(ref).max(axis=1) > 0).all()
    if turned:
        assert asym > 0.02


def _case(label, cams, ins, hw, seed, tunings=((0, "default"),), turned=True):
    dev = _dev()
    w = _depth_field(cams["viewmatrix"].shape[0], hw, seed)
    ref, contrib, aff, ob = view_z_oracle(cams, hw, ins, w)
    _assert_regime(label, cams, ob, ref, turned)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    for tuning, name in tunings:
        gv, _, _ = _gpu(dcams, hw, ins, w, tuning=tuning)
        _check_view_grad(f"{label} {name}", gv, ref, contrib, aff)


# ---------------------------------------------------------------------------------------------------------------------
# 1. every backward kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_view_z_gradient_under_every_backward_variant(geometry):
    """S = 2 scenes x 9 views (camera chunks 8 + 1), per-view view_scale 0.8 .. 1.25, turned cameras; the default
    kernels, the round-1 compositor, the 4-CTA compositor and the two-phase preprocess backward.  The Gaussians'
    gradients of the kernels that also write the view-matrix gradient agree with those of the kernels that do not."""
    from pf3plat_b200._capi import GS_TUNE_BWD_OCC4, GS_TUNE_BWD_V1, GS_TUNE_PBWD_2PHASE
    dev = _dev()
    cams, ins, hw = _depth_batch(geometry)
    tunings = ((0, "default"), (GS_TUNE_BWD_V1, "bwd v1"), (GS_TUNE_BWD_OCC4, "bwd occ4"),
               (GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd"))
    _case(f"every backward, {geometry}", cams, ins, hw, seed=51, tunings=tunings)
    w = _depth_field(cams["viewmatrix"].shape[0], hw, 51)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    for tuning, name in ((0, "default"), (GS_TUNE_PBWD_2PHASE, "2-phase")):
        _, with_view, out_a = _gpu(dcams, hw, ins, w, tuning=tuning)
        gv, without, out_b = _gpu(dcams, hw, ins, w, tuning=tuning, view_grad=False)
        assert gv is None
        for a, b in zip(out_a, out_b):
            assert torch.equal(a, b)
        # the compositor's per-Gaussian atomics add in a different order on every run: agreement, not identity
        worst = _agree(f"{geometry} {name}: Gaussian gradients with / without the view-matrix gradient", with_view,
                       without)
        print(f"[regime] {geometry} {name}: Gaussian gradients with / without the view-matrix gradient differ by "
              f"{worst:.2e} of max-abs (bound {PATH_RTOL:g})")


# ---------------------------------------------------------------------------------------------------------------------
# 2. every binning path
# ---------------------------------------------------------------------------------------------------------------------
def test_view_z_gradient_on_every_binning_path():
    """2 scenes x 3 views on a context of its own, walked through the exact path, the per-view strata trial, the
    stratified path and the radix fallback."""
    from pf3plat_b200._capi import GS_TUNE_FORCE_RADIX_BINNING, GS_TUNE_NO_SPECULATION
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = (32, 48)
    # test_gpu_backward_paths' cloud, whose binning states on a fresh context are known (cameras not turned)
    scenes = [make_scene(2500, 3, *hw, seed=70 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    w = _depth_field(6, hw, seed=52)
    ref, contrib, aff, ob = view_z_oracle(cams, hw, ins, w)
    _assert_regime("binning paths", cams, ob, ref, turned=False)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    sequence = [("exact", GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("radix fallback", GS_TUNE_FORCE_RADIX_BINNING, 0)]
    states = []
    stream = _stream_ctx(dev)
    with torch.cuda.stream(stream):
        for label, tuning, want in sequence:
            gv, _, _ = _gpu(dcams, hw, ins, w, tuning=tuning)
            st = last_stats(dev)
            states.append(st["speculative"])
            assert st["speculative"] == want and st["overflow_redos"] == 0, (label, st)
            _check_view_grad(f"binning {label}", gv, ref, contrib, aff)
        stream.synchronize()
    print(f"[regime] binning paths: speculative per call {states}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. views per scene, near planes, ragged frames, opaque stacks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vps", [1, 3, 9, 19])
def test_view_z_gradient_views_per_scene(vps):
    hw = (32, 48)
    scenes = [_turned(make_scene(1200, vps, *hw, seed=400 + 10 * vps + k), seed=450 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, vps), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    _case(f"{vps} views per scene", cams, ins, hw, seed=53 + vps)


@pytest.mark.parametrize("near", [0.5, 1.0, 2.0])
def test_view_z_gradient_near_planes(near):
    hw = (32, 48)
    scenes = [_turned(make_scene(1500, 3, *hw, seed=500 + k), seed=510 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=np.full(6, near))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    _case(f"near {near}", cams, ins, hw, seed=54)


def test_view_z_gradient_ragged_frame():
    """33 x 250: partial warp rows and columns of the backward compositor, a partial last tile row, Gaussians straddling
    the last row and column."""
    hw = (33, 250)
    sc = _turned(edge_straddle_scene(600, 120, 2, *hw, seed=77), seed=78)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    _case("33 x 250 frame", cams, ins, hw, seed=55)


def test_view_z_gradient_opaque_stacks():
    """Six nearly opaque sheets: most pixels terminate early, alpha clamps at 0.99 near the centres."""
    hw = (48, 64)
    sc = _turned(opaque_stack_scene(6, 10, 2, *hw, seed=110), seed=111, angle=0.05)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    _case("opaque stacks", cams, ins, hw, seed=56)


# ---------------------------------------------------------------------------------------------------------------------
# 4. no gradient the reference lacks
# ---------------------------------------------------------------------------------------------------------------------
def test_colour_only_loss_gives_the_extrinsics_no_gradient():
    """A loss that does not read the depth: extrinsics.grad stays None, as on the two-pass route; the Gaussians' gradients
    equal those of the two-pass route's colour render."""
    from pf3plat_b200.render import decoder_forward, render_depth, render_views
    dev = _dev()
    b, v, hw = 2, 3, (32, 48)
    scs = [_turned(make_scene(1500, v, *hw, seed=600 + k), seed=610 + k).to(dev) for k in range(b)]
    st = lambda n: torch.stack([getattr(s, n) for s in scs])
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), 0.5, device=dev), torch.full((b, v), 50.0, device=dev)
    bg = torch.tensor([0.3, 0.2, 0.1], device=dev)
    target = make_target(b * v, *hw, seed=7).to(dev).reshape(b, v, 3, *hw)
    names = ("means", "covariances", "harmonics", "opacities")
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    grads = []
    for route in ("fused", "two-pass"):
        e = ext.clone().requires_grad_(True)
        L = [st(n).clone().requires_grad_(True) for n in names]
        if route == "fused":
            color, depth = decoder_forward(*L, e, intr, nr, fr, hw, bg, depth_mode="depth")
        else:
            color = render_views(flat(e), flat(intr), flat(nr), flat(fr), hw, bg.reshape(1, 3).expand(b * v, 3),
                                 *L).reshape(b, v, 3, *hw)
            depth = render_depth(L[0], L[1], L[3], e, intr, nr, fr, hw)
        assert depth.requires_grad
        ((color - target) ** 2).mean().backward()
        print(f"[regime] colour-only loss, {route} route: extrinsics.grad is {None if e.grad is None else 'set'}")
        assert e.grad is None, route
        grads.append([t.grad for t in L])
    for n, a, r in zip(names, *grads):
        err = float((a - r).abs().max())
        assert err <= PATH_RTOL * float(r.abs().max()), (n, err)
    # the operator alone, with a view matrix requiring grad
    from pf3plat_b200.rasterizer import rasterize_batch
    cams, ins = scene_batch_args([s.to("cpu") for s in scs])
    vm = cams["viewmatrix"].to(dev).requires_grad_(True)
    bs = _settings({**{k: t.to(dev) for k, t in cams.items()}, "viewmatrix": vm}, hw, with_depth=True)
    leaves = _leaves({k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}, dev)
    out = rasterize_batch(bs, **leaves)
    out[0].sum().backward()
    assert vm.grad is None and leaves["means3D"].grad is not None


@pytest.mark.parametrize("scale_invariant", [True, False])
def test_view_batch_values_do_not_depend_on_the_pose_gradient(scale_invariant):
    """make_view_batch with extrinsics requiring grad: the kernel's matrices, bit for bit; only viewmatrix carries a
    gradient."""
    from pf3plat_b200.cameras import make_view_batch
    dev = _dev()
    sc = _turned(make_scene(10, 5, 32, 48, seed=640), seed=641).to(dev)
    near = torch.linspace(0.5, 2.0, 5, device=dev)
    plain = make_view_batch(sc.extrinsics, sc.intrinsics, near, 100 * near, scale_invariant)
    e = sc.extrinsics.clone().requires_grad_(True)
    vb = make_view_batch(e, sc.intrinsics, near, 100 * near, scale_invariant)
    for k in ("viewmatrix", "projmatrix", "campos", "tanfov", "scale"):
        assert torch.equal(getattr(vb, k), getattr(plain, k)), k
        assert getattr(vb, k).requires_grad == (k == "viewmatrix"), k


def test_drop_in_rasterizer_gives_viewmatrix_no_gradient():
    """The reference op hands viewmatrix no gradient, with or without return_depth."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    dev = _dev()
    hw = (32, 48)
    sc = _turned(make_scene(800, 1, *hw, seed=620), seed=621)
    cams, ins = scene_batch_args([sc])
    vm = cams["viewmatrix"][0].to(dev).requires_grad_(True)
    rs = GaussianRasterizationSettings(image_height=hw[0], image_width=hw[1], tanfovx=float(cams["tanfov"][0, 0]),
                                       tanfovy=float(cams["tanfov"][0, 1]), bg=cams["bg"][0].to(dev), scale_modifier=1.0,
                                       viewmatrix=vm, projmatrix=cams["projmatrix"][0].to(dev), sh_degree=4,
                                       campos=cams["campos"][0].to(dev), prefiltered=False, debug=False)
    means = ins["means3D"][0].to(dev).requires_grad_(True)
    color, radii, depth = GaussianRasterizer(rs)(means3D=means, means2D=None, opacities=ins["opacities"][0].to(dev),
                                                 shs=ins["shs"][0].to(dev), cov3D_precomp=ins["cov3D_precomp"][0].to(dev),
                                                 return_depth=True)
    (color.sum() + depth.sum()).backward()
    assert vm.grad is None and means.grad is not None and float(means.grad.abs().max()) > 0


def test_view_z_gradient_needs_the_depth_flag():
    """gs_backward refuses dL_dviewmatrix_z for a forward without GS_FLAG_DEPTH."""
    from pf3plat_b200 import _capi
    from pf3plat_b200.rasterizer import _context, _make_config, rasterize_batch
    dev = _dev()
    hw = (16, 16)
    cams, ins = scene_batch_args([make_scene(200, 1, *hw, seed=630)])
    dcams = {k: v.to(dev) for k, v in cams.items()}
    leaves = _leaves({k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}, dev)
    bs = _settings(dcams, hw)
    color, _ = rasterize_batch(bs, **leaves)
    node = color.grad_fn
    keep = []
    S, P, V, M, H, W = node.dims
    cfg = _make_config(bs, S, P, M, keep)
    gin = _capi.GsInputs(**{k: None if t is None else t.data_ptr() for k, t in node.ins.items()})
    dcol = torch.zeros(V, 3, H, W, device=dev)
    out = {k: torch.empty(n, device=dev) for k, n in (("m", S * P * 3), ("o", S * P), ("sh", S * P * M * 3),
                                                      ("c", S * P * 6), ("vz", V * 4))}
    ig = _capi.GsInGrads(dL_dmeans3D=out["m"].data_ptr(), dL_dopacities=out["o"].data_ptr(),
                         dL_dshs=out["sh"].data_ptr(), dL_dcov3D=out["c"].data_ptr(), dL_dviewmatrix_z=out["vz"].data_ptr())
    og = _capi.GsOutGrads(dcol.data_ptr(), None)
    stream = torch.cuda.current_stream(dev).cuda_stream
    rc = _capi.lib().gs_backward(_context(dev, stream), ctypes.byref(cfg), ctypes.byref(gin), node.handle.ptr,
                                 ctypes.byref(og), ctypes.byref(ig), stream)
    assert rc == -1 and b"GS_FLAG_DEPTH" in _capi.lib().gs_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# 5. decoder_forward(depth_mode="depth") with predicted poses: one render
# ---------------------------------------------------------------------------------------------------------------------
def _two_pass_route(L, ext, intr, nr, fr, hw, bg):
    """The route decoder_forward took for "depth" while the extrinsics required grad: a colour render, then
    render_depth's second render with the camera-space z as its colour."""
    from pf3plat_b200.render import render_depth, render_views
    b, v = ext.shape[:2]
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    color = render_views(flat(ext), flat(intr), flat(nr), flat(fr), hw, bg.reshape(1, 3).expand(b * v, 3), *L)
    return color.reshape(b, v, *color.shape[1:]), render_depth(L[0], L[1], L[3], ext, intr, nr, fr, hw)


def _counting(monkeypatch):
    from pf3plat_b200 import render
    calls = []
    inner = render.rasterize_batch

    def wrapped(bs, *a, **k):
        calls.append(bs.viewmatrix.shape[0])
        return inner(bs, *a, **k)

    monkeypatch.setattr(render, "rasterize_batch", wrapped)
    return calls


@pytest.mark.parametrize("near", [0.5, 2.0])
def test_decoder_depth_on_predicted_poses_is_one_render_and_matches_the_two_pass_route(near, monkeypatch):
    from pf3plat_b200.render import decoder_forward
    dev = _dev()
    b, v, P, hw = 2, 3, 1500, (48, 64)
    scs = [_turned(make_scene(P, v, *hw, seed=700 + k), seed=710 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs])
    ext, intr = st("extrinsics"), st("intrinsics")
    nr, fr = torch.full((b, v), near), torch.full((b, v), 100.0 * near)
    bg = torch.tensor([0.3, 0.2, 0.1])
    names = ("means", "covariances", "harmonics", "opacities")
    V = b * v
    # the fp64 oracle of the two-pass route, with per-Gaussian contributions to the extrinsics' gradient; loss = MSE
    # against a target + <w, depth>, whose incoming gradients the GPU routes are handed as they are
    lo = [st(n).double().requires_grad_(True) for n in names]
    z_ext = ext.double()[:, :, None].expand(b, v, P, 4, 4).clone().requires_grad_(True)
    dec = DecoderOracle(*lo, ext, intr, nr, fr, hw, bg, two_pass=True, z_extrinsics=z_ext)
    target = make_target(V, *hw, seed=8).numpy()
    dL = 2 * (dec.color - target) / target.size
    w = _depth_field(V, hw, seed=57)
    dec.backward(dL, w)
    ref = z_ext.grad.sum(dim=2)
    f32 = lambda a: torch.as_tensor(a, dtype=torch.float32, device=dev)

    def run(route):
        e = ext.to(dev).requires_grad_(True)
        L = [st(n).to(dev).requires_grad_(True) for n in names]
        args = (e, intr.to(dev), nr.to(dev), fr.to(dev), hw, bg.to(dev))
        if route == "fused":
            calls = _counting(monkeypatch)
            color, depth = decoder_forward(*L, *args, depth_mode="depth")
            monkeypatch.undo()
            assert calls == [V], calls
        else:
            color, depth = _two_pass_route(L, *args)
        torch.autograd.backward([color, depth], [f32(dL).reshape(color.shape), f32(w).reshape(depth.shape)])
        return color.detach(), depth.detach(), e.grad, [t.grad for t in L]

    c_new, d_new, e_new, g_new = run("fused")
    c_old, d_old, e_old, g_old = run("two-pass")
    aff = dec.affected()                                                       # (b, G)
    aff_t = np.repeat(aff[:, None], v, axis=1)                                 # (b, v, G)
    print(f"[regime] decoder depth on predicted poses, near {near}: one operator call of {V} views; visible per view "
          f"{(dec.ob.radii > 0).sum(axis=1).tolist()}, affected {int(aff.sum())}; colour bit-identical to the two-pass "
          f"route: {torch.equal(c_new, c_old)}")
    assert (dec.ob.radii > 0).mean() > 0.3
    # same preprocess, binning and colour arithmetic: the depth channel is a separate accumulator
    assert torch.equal(c_new, c_old)
    frag = np.stack([r.px_fragile | q.px_fragile for r, q in zip(dec.ob.views, dec.ob_depth.views)])
    for got in (d_new, d_old):
        dd = np.abs(got.reshape(V, *hw).cpu().numpy() - dec.depth)
        assert dd[~frag].max() <= 1e-4 * np.abs(dec.depth).max(), dd[~frag].max()
    a = aff.reshape(-1)
    for k, n in enumerate(names):
        if k == 2:          # SH: the colour render's gradient on both routes
            continue
        new, old = g_new[k].reshape(b * P, -1), g_old[k].reshape(b * P, -1)
        check_grad(f"near {near} dL/d{n} fused vs two-pass route", new, old.cpu().numpy(), a)
        check_grad(f"near {near} dL/d{n} fused vs fp64 oracle", new, lo[k].grad.reshape(b * P, -1), a)
    contrib = z_ext.grad
    camera_grad_check(f"near {near} dL/dextrinsics fused vs fp64 oracle", e_new, ref, contrib, aff_t)
    camera_grad_check(f"near {near} dL/dextrinsics fused vs two-pass route", e_new, e_old.cpu().numpy(), contrib, aff_t)


# ---------------------------------------------------------------------------------------------------------------------
# 6. the training shape
# ---------------------------------------------------------------------------------------------------------------------
def test_training_shape_fused_route_matches_the_two_pass_route():
    """b = 14 scenes x 3 target views, 131072 pixel-aligned Gaussians per scene, 256 x 256, predicted (turned) poses;
    loss = MSE on the colour + a signed depth term.  Colour bit-identical; the extrinsics' gradient within 1e-3
    element-wise (relative to |two-pass| + its rms), the Gaussians' within 1e-3 of their max-abs."""
    dev = _dev()
    b, v, hw = 14, 3, (256, 256)
    scs = [_turned(make_pixel_aligned_scene(*hw, v, seed=800 + k), seed=820 + k, angle=0.05) for k in range(b)]
    st = lambda name: torch.stack([getattr(s, name) for s in scs]).to(dev)
    means, cov, sh, opac, ext, intr = (st(n) for n in ("means", "covariances", "harmonics", "opacities", "extrinsics",
                                                       "intrinsics"))
    nr, fr = torch.full((b, v), 1.0, device=dev), torch.full((b, v), 100.0, device=dev)
    bg = torch.zeros(3, device=dev)
    target = make_target(b * v, *hw, seed=9).to(dev).reshape(b, v, 3, *hw)
    w = torch.as_tensor(_depth_field(b * v, hw, seed=58), dtype=torch.float32, device=dev).reshape(b, v, *hw)

    def run(route):
        from pf3plat_b200.render import decoder_forward
        e = ext.clone().requires_grad_(True)
        L = [t.clone().requires_grad_(True) for t in (means, cov, sh, opac)]
        if route == "fused":
            color, depth = decoder_forward(*L, e, intr, nr, fr, hw, bg, depth_mode="depth")
        else:
            color, depth = _two_pass_route(L, e, intr, nr, fr, hw, bg)
        (((color - target) ** 2).mean() + 1e-3 * (depth * w).sum()).backward()
        return color.detach(), depth.detach(), e.grad, [t.grad for t in L]

    new, old = run("fused"), run("two-pass")
    torch.cuda.synchronize()
    dmax = float(old[1].abs().max())
    derr = float((new[1] - old[1]).abs().max())
    print(f"[regime] training shape: {b} x {v} views, {means.shape[1]} Gaussians per scene, 256 x 256; colour "
          f"bit-identical {torch.equal(new[0], old[0])}; max |depth difference| {derr:.2e} of max depth {dmax:.2f}")
    assert means.shape[1] == 131072
    assert torch.equal(new[0], old[0])
    assert derr <= 1e-4 * dmax

    a, r = new[2].double(), old[2].double()
    rms = float(r.pow(2).mean().sqrt())
    ratio = float(((a - r).abs() / (r.abs() + rms)).max())
    print(f"[regime] training shape dL/dextrinsics: rms {rms:.3e}, worst |fused - two-pass| / (|two-pass| + rms) "
          f"{ratio:.2e}")
    assert rms > 0 and ratio <= 1e-3, ratio
    for k, n in ((0, "means"), (1, "covariances"), (3, "opacities")):
        err = float((new[3][k] - old[3][k]).abs().max() / old[3][k].abs().max())
        print(f"[regime] training shape dL/d{n}: max |fused - two-pass| / max |two-pass| {err:.2e}")
        assert err <= 1e-3, (n, err)
