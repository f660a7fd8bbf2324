"""GPU tests of the camera gradient (gs_backward_cam, BatchSettings.camera_gradients, set_camera_gradients): dL/dviewmatrix,
dL/dprojmatrix and dL/dcampos of every output, against the fp64 autograd oracle of tests/camera_oracle.py with the rule
of tests.chain_oracle.camera_grad_check.  Every test prints "[parity]" lines."""
import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_scene, make_target
from tests.camera_oracle import camera_oracle
from tests.chain_oracle import camera_grad_check
from tests.test_gpu_depth_chain import _depth_batch, _depth_field
from tests.test_gpu_regimes import _settings

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts, set_camera_gradients
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    set_camera_gradients(False)
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()


def _gpu(bs, ins, dL, w=None, dA=None):
    """rasterize_batch with camera gradients on and the three camera inputs as leaves; returns their gradients and the
    outputs."""
    from pf3plat_b200.rasterizer import rasterize_batch
    cams = [bs.viewmatrix.to(DEV).clone().requires_grad_(True), bs.projmatrix.to(DEV).clone().requires_grad_(True),
            bs.campos.to(DEV).clone().requires_grad_(True)]
    d = lambda t: None if t is None else t.to(DEV)
    bs = bs._replace(viewmatrix=cams[0], projmatrix=cams[1], campos=cams[2], bg=d(bs.bg), tanfov=d(bs.tanfov),
                     view_scale=d(bs.view_scale), depth_near_far=d(bs.depth_near_far), camera_gradients=True)
    leaves = {k: v.to(DEV).clone().requires_grad_(True) for k, v in ins.items()}
    out = rasterize_batch(bs, **leaves)
    names = ["color", "radii"] + (["depth"] if bs.with_depth else []) + (["alpha"] if bs.with_alpha else [])
    o = dict(zip(names, out))
    f = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32, device=DEV)
    ts, gs = [o["color"]], [f(dL)]
    if w is not None:
        ts.append(o["depth"]); gs.append(f(w))
    if dA is not None:
        ts.append(o["alpha"]); gs.append(f(dA))
    torch.autograd.backward(ts, gs)
    return [c.grad.reshape(c.shape[0], -1) for c in cams], {k: v.detach() for k, v in o.items()}


def _check(label, got, ref, rtol=1e-3):
    for name, g, r in zip(("viewmatrix", "projmatrix", "campos"), got, ref):
        V = r.shape[0]
        camera_grad_check(f"{label} dL/d{name}", g, r, np.zeros((V, 1) + r.shape[1:]), np.zeros((V, 1), bool), rtol=rtol)


def _loss(V, hw, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((V, 3, *hw)) / (hw[0] * hw[1])


TUNINGS = ((0, "default"), (_capi.GS_TUNE_BWD_V1, "bwd v1"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"),
           (_capi.GS_TUNE_FWD_WS, "warp-specialised fwd"))


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_camera_grad_against_oracle_under_every_compositor(geometry):
    """2 scenes x 9 views, view_scale 0.8 .. 1.25, turned cameras; SH (cov3D) or colors_precomp + scales/rotations with
    scale_modifier 1.3; colour + depth loss."""
    cams, ins, hw = _depth_batch(geometry)
    V = cams["viewmatrix"].shape[0]
    bs = _settings(cams, hw, sh_degree=3, with_depth=True, scale_modifier=1.0 if geometry == "cov3D" else 1.3)
    dL, w = _loss(V, hw, 5), _depth_field(V, hw, 6)
    ref = camera_oracle(bs, ins, dL, w)
    for tuning, name in TUNINGS:
        got, _ = _gpu(bs._replace(tuning=tuning), ins, dL, w)
        _check(f"{geometry} {name}", got, ref)


@pytest.mark.parametrize("mode", ["disparity", "relative_disparity", "log"])
def test_camera_grad_depth_modes_alpha_and_antialiasing(mode):
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
    bs = _settings(cams, hw, sh_degree=3, with_depth=True)._replace(depth_mode=mode, depth_near_far=nf, with_alpha=True,
                                                                      antialiasing=True)
    dL, w, dA = _loss(V, hw, 7), _depth_field(V, hw, 8), _depth_field(V, hw, 9)
    ref = camera_oracle(bs, ins, dL, w, dA, antialiasing=True, depth_mode=mode, near_far=nf)
    got, _ = _gpu(bs, ins, dL, w, dA)
    # relative disparity divides by 1/near - 1/far: on an H100 its fp32 chain was measured at 1.26e-3 (|ref| + rms)
    _check(f"{mode} + alpha + aa", got, ref, rtol=2e-3 if mode == "relative_disparity" else 1e-3)


@pytest.mark.parametrize("aa", [False, True])
def test_camera_grad_degree4(aa):
    """SH degree 4 (25 coefficients, band 4 non-zero): the B4 camera kernels, band 4's share of dL/dd reaching dL/dcampos;
    colour + disparity loss, with and without anti-aliasing."""
    from tests.sh4_oracle import with_band4
    from tests.test_gpu_depth_chain import _turned
    from tests.batch_oracle import scene_batch_args
    hw = (32, 48)
    scenes = [with_band4(_turned(make_scene(1200, 5, *hw, seed=60 + k), seed=70 + k), seed=80 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=np.linspace(0.6, 1.6, 10).astype(np.float32))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    assert ins["shs"].shape[2] == 25 and float(ins["shs"][:, :, 16:].abs().max()) > 0
    V = 10
    nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
    bs = _settings(cams, hw, sh_degree=4, with_depth=True)._replace(sh_eval_max_degree=4, antialiasing=aa,
                                                                      depth_mode="disparity", depth_near_far=nf)
    dL, w = _loss(V, hw, 21), _depth_field(V, hw, 22)
    ref = camera_oracle(bs, ins, dL, w, antialiasing=aa, depth_mode="disparity", near_far=nf)
    got, _ = _gpu(bs, ins, dL, w)
    _check(f"degree 4{' + aa' if aa else ''}", got, ref)


@pytest.mark.parametrize("vps", [1, 19])
def test_camera_grad_views_per_scene_and_ragged_frame(vps):
    """1 or 19 views per scene, 3 scenes, a 33 x 250 frame, near 0.5 .. 2 (view_scale 2 .. 0.5)."""
    from tests.batch_oracle import scene_batch_args
    hw = (33, 250)
    scenes = [make_scene(600, vps, *hw, seed=40 + k) for k in range(3)]
    near = np.linspace(0.5, 2.0, 3 * vps).astype(np.float32)
    cams, ins = scene_batch_args(scenes, near=near)
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    V = 3 * vps
    bs = _settings(cams, hw, sh_degree=3)
    dL = _loss(V, hw, 11)
    ref = camera_oracle(bs, ins, dL)
    got, _ = _gpu(bs, ins, dL)
    _check(f"vps {vps}", got, ref)


BINNING = ((0, "default"), (_capi.GS_TUNE_FORCE_RADIX_BINNING, "radix"), (_capi.GS_TUNE_NO_SPECULATION, "exact"),
           (_capi.GS_TUNE_NO_STRATA, "no strata"))


@pytest.mark.parametrize("variant", ["plain", "aa_log_alpha"])
def test_camera_grad_deterministic_on_every_binning_path(variant):
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    bs = _settings(cams, hw, sh_degree=3, with_depth=True)
    dL, w = _loss(V, hw, 12), _depth_field(V, hw, 13)
    if variant == "plain":
        ref = camera_oracle(bs, ins, dL, w)
        dA = None
    else:   # anti-aliasing, an f(z) depth mode and alpha under the deterministic camera kernels
        nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
        bs = bs._replace(antialiasing=True, depth_mode="log", depth_near_far=nf, with_alpha=True)
        dA = _depth_field(V, hw, 23)
        ref = camera_oracle(bs, ins, dL, w, dA, antialiasing=True, depth_mode="log", near_far=nf)
    torch.use_deterministic_algorithms(True)
    try:
        first = None
        for tuning, name in BINNING:
            for _ in range(2):
                got, _ = _gpu(bs._replace(tuning=tuning), ins, dL, w, dA)
                if first is None:
                    first = got
                    _check("deterministic", got, ref)
                for a, b in zip(got, first):
                    assert torch.equal(a, b), name
            print(f"[parity] {variant}: deterministic camera grads bit-identical on {name}")
    finally:
        torch.use_deterministic_algorithms(False)


def test_setting_off_is_bit_identical_and_refusals():
    """With the setting off, a call whose projmatrix and campos require grad (so that they are live autograd inputs of the
    operator) returns the outputs and gradients, bit for bit, of a call with plain camera tensors, and gives them no
    gradient.  Refused: the two-phase preprocess backward with the camera gradient, and the z column requested together
    with it in one C call."""
    import ctypes
    from pf3plat_b200.rasterizer import _make_config, rasterize_batch
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    dcams = {k: v.to(DEV) for k, v in cams.items()}
    dL = torch.as_tensor(_loss(V, hw, 14), dtype=torch.float32, device=DEV)
    runs, live = [], None
    torch.use_deterministic_algorithms(True)   # (float atomics would differ run to run whatever the setting)
    try:
        for with_leaves in (False, True):
            bs = _settings(dcams, hw, sh_degree=3, with_depth=True)
            vm = bs.viewmatrix.clone().requires_grad_(True)
            pm, cp = bs.projmatrix.clone().requires_grad_(with_leaves), bs.campos.clone().requires_grad_(with_leaves)
            leaves = {k: v.to(DEV).clone().requires_grad_(True) for k, v in ins.items()}
            out = rasterize_batch(bs._replace(viewmatrix=vm, projmatrix=pm, campos=cp), **leaves)
            torch.autograd.backward([out[0], out[2]], [dL, torch.ones_like(out[2]) * 1e-3])
            runs.append([out[0], out[2], vm.grad] + [leaves[k].grad for k in sorted(leaves)])
            live = (pm.grad, cp.grad)
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    assert live == (None, None)
    bs = _settings(cams, hw, sh_degree=3)._replace(tuning=_capi.GS_TUNE_PBWD_2PHASE)
    with pytest.raises(ValueError, match="GS_TUNE_PBWD_2PHASE"):
        _gpu(bs, ins, _loss(V, hw, 15))
    # the C entry with both the z column and GsCameraGrads
    from pf3plat_b200 import rasterizer as R
    bs = _settings(dcams, hw, sh_degree=3, with_depth=True)
    S, P, M = ins["means3D"].shape[0], ins["means3D"].shape[1], ins["shs"].shape[2]
    keep: list = []
    cfg = _make_config(R._resolve_degree(bs), S, P, M, keep)
    t = {k: v.to(DEV).contiguous() for k, v in ins.items()}
    gin = _capi.GsInputs(means3D=t["means3D"].data_ptr(), opacities=t["opacities"].data_ptr(), shs=t["shs"].data_ptr(),
                         cov3D_precomp=t["cov3D_precomp"].data_ptr())
    color = torch.empty(V, 3, *hw, device=DEV)
    radii = torch.empty(V, P, dtype=torch.int32, device=DEV)
    depth = torch.empty(V, *hw, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    ctx = R.current_context()
    saved = ctypes.c_void_p()
    L = _capi.lib()
    _capi.check(L.gs_forward(ctx, ctypes.byref(cfg), ctypes.byref(gin),
                             ctypes.byref(_capi.GsOutputs(color.data_ptr(), radii.data_ptr(), depth.data_ptr())),
                             ctypes.byref(saved), stream))
    try:
        gz, gv = torch.empty(V, 4, device=DEV), torch.empty(V, 16, device=DEV)
        gdep = torch.ones(V, *hw, device=DEV)
        rc = L.gs_backward_cam(ctx, ctypes.byref(cfg), ctypes.byref(gin), saved,
                               ctypes.byref(_capi.GsOutGrads(dL.data_ptr(), gdep.data_ptr())), None,
                               ctypes.byref(_capi.GsInGrads(dL_dviewmatrix_z=gz.data_ptr())),
                               ctypes.byref(_capi.GsCameraGrads(gv.data_ptr(), None, None)), stream)
        assert rc == -1 and b"dL_dviewmatrix_z" in L.gs_last_error()
    finally:
        L.gs_saved_free(ctx, saved, stream)
        torch.cuda.synchronize()


def test_make_view_batch_straight_through_matches_the_reference_glue():
    """make_view_batch(camera_gradients=True) on CUDA: the kernel's values, and the gradients of render_cuda's glue --
    the 1/near rescale of the extrinsics' translation, inverse(), view @ P, the rescaled translation as campos -- with
    near 0.5 .. 2 and turned cameras, in all 16 entries of the extrinsics."""
    from pf3plat_b200.cameras import get_fov, get_projection_matrix, make_view_batch
    from tests.test_gpu_depth_chain import _turned
    sc = _turned(make_scene(10, 6, 32, 48, seed=5), seed=6)
    ext = sc.extrinsics.double()
    near = torch.linspace(0.5, 2.0, 6, dtype=torch.float64)
    far = 100 * near
    g = torch.Generator().manual_seed(9)
    wv, wp, wc = (torch.randn(6, *shape, generator=g, dtype=torch.float64) for shape in ((4, 4), (4, 4), (3,)))
    # the glue in fp64, differentiated by autograd (tests/ref_callsite.py, render_cuda's lines)
    e64 = ext.clone().requires_grad_(True)
    e = e64.clone()
    e[..., :3, 3] = e[..., :3, 3] * (1 / near)[:, None]
    fov_x, fov_y = get_fov(sc.intrinsics.double()).unbind(-1)
    pt = get_projection_matrix(near / near, far / near, fov_x, fov_y).transpose(-1, -2)
    view = e.inverse().transpose(-1, -2)
    ((view * wv).sum() + ((view @ pt) * wp).sum() + (e[:, :3, 3] * wc).sum()).backward()
    # ours
    e32 = ext.float().to(DEV).requires_grad_(True)
    vb = make_view_batch(e32, sc.intrinsics.to(DEV), near.float().to(DEV), far.float().to(DEV), True, camera_gradients=True)
    f = lambda x: x.float().to(DEV)
    ((vb.viewmatrix * f(wv)).sum() + (vb.projmatrix * f(wp)).sum() + (vb.campos * f(wc)).sum()).backward()
    got, ref = e32.grad.double().cpu(), e64.grad
    err = float(((got - ref).abs() / (ref.abs() + ref.abs().max() * 1e-3)).max())
    print(f"[parity] make_view_batch straight-through vs glue autograd: worst rel err {err:.2e}")
    assert err < 1e-3
    plain = make_view_batch(ext.float().to(DEV), sc.intrinsics.to(DEV), near.float().to(DEV), far.float().to(DEV), True)
    for a, b in ((vb.viewmatrix, plain.viewmatrix), (vb.projmatrix, plain.projmatrix), (vb.campos, plain.campos)):
        assert torch.equal(a.detach(), b)


def _decoder_inputs(b, v, P, hw, seed):
    scs = [make_scene(P, v, *hw, seed=seed + k) for k in range(b)]
    st = lambda f: torch.stack([f(sc) for sc in scs]).to(DEV)
    return dict(means=st(lambda s: s.means), covariances=st(lambda s: s.covariances),
                harmonics=st(lambda s: s.harmonics), opacities=st(lambda s: s.opacities),
                extrinsics=st(lambda s: s.extrinsics), intrinsics=st(lambda s: s.intrinsics),
                near=st(lambda s: s.near), far=st(lambda s: s.far))


def test_decoder_forward_matches_the_reference_glue_route():
    """decoder_forward(camera_gradients=True) at PF3plat's training shape (14 scenes x 3 views x 131072 Gaussians,
    256 x 256): dL/dextrinsics in all 16 entries against render_cuda's glue run view by view through the drop-in."""
    from pf3plat_b200.rasterizer import set_camera_gradients
    from pf3plat_b200.render import decoder_forward
    from tests.ref_callsite import render_like_reference
    b, v, hw = 14, 3, (256, 256)
    d = _decoder_inputs(b, v, 131072, hw, 70)
    bg = torch.zeros(3, device=DEV)
    target = make_target(b * v, *hw, seed=2).to(DEV).reshape(b, v, 3, *hw)
    e1 = d["extrinsics"].clone().requires_grad_(True)
    color, _ = decoder_forward(d["means"], d["covariances"], d["harmonics"], d["opacities"], e1, d["intrinsics"],
                               d["near"], d["far"], hw, bg, camera_gradients=True)
    ((color - target) ** 2).mean().backward()
    set_camera_gradients(True)
    try:
        e2 = d["extrinsics"].clone().requires_grad_(True)
        rep = lambda t: t.repeat_interleave(v, dim=0)
        flat = lambda t: t.reshape(b * v, *t.shape[2:])
        img = render_like_reference(flat(e2), flat(d["intrinsics"]), flat(d["near"]), flat(d["far"]), hw,
                                    bg.expand(b * v, 3), rep(d["means"]), rep(d["covariances"]), rep(d["harmonics"]),
                                    rep(d["opacities"]))
        ((img.reshape(b, v, 3, *hw) - target) ** 2).mean().backward()
    finally:
        set_camera_gradients(False)
    g1, g2 = e1.grad.reshape(b * v, 16).double(), e2.grad.reshape(b * v, 16).double()
    err = (g1 - g2).abs().max(dim=1).values / g2.abs().max(dim=1).values
    print(f"[parity] decoder_forward vs reference glue: worst per-view max rel err {float(err.max()):.2e}, "
          f"bottom-row entries {float(g1[:, 12:].abs().max()):.2e} / {float(g2[:, 12:].abs().max()):.2e}")
    assert float(err.max()) < 1e-4


def test_pose_recovery_by_adam_through_decoder_forward():
    """A target pose perturbed by 2 degrees about a random axis and by 3 % of the baseline in a random direction, near
    0.7 (so the 1/near rescale is in the chain), a scene with depths from 1.5 to 20: Adam on the MSE through
    decoder_forward, 300 steps, learning rate 5e-3 on a cosine schedule, in deterministic mode, must cut the rotation and
    the translation errors at least tenfold."""
    hw = (128, 128)
    d = _decoder_inputs(1, 1, 40000, hw, 90)
    d["near"], d["far"] = d["near"] * 0.7, d["far"] * 0.7
    bg = torch.zeros(3, device=DEV)
    args = (d["means"], d["covariances"], d["harmonics"], d["opacities"])
    true = d["extrinsics"]
    with torch.no_grad():
        target, _ = decoder_forward_(args, true, d, hw, bg)
    g = torch.Generator().manual_seed(3)
    axis = torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0)
    K = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
    dR = torch.linalg.matrix_exp(np.deg2rad(2.0) * K).to(DEV, torch.float32)
    base = float(true[0, 0, :3, 3].norm().clamp_min(1.0))
    dt = (0.03 * base * torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)).to(DEV)
    start = true.clone()
    start[0, 0, :3, :3] = dR @ true[0, 0, :3, :3]
    start[0, 0, :3, 3] = true[0, 0, :3, 3] + dt
    # parameters: a rotation vector and a translation offset applied to the perturbed pose
    w = torch.zeros(3, device=DEV, requires_grad=True)
    t = torch.zeros(3, device=DEV, requires_grad=True)
    steps = 300
    opt = torch.optim.Adam([w, t], lr=5e-3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps)

    def pose():
        Kw = torch.zeros(3, 3, device=DEV).index_put(
            (torch.tensor([0, 0, 1, 1, 2, 2]), torch.tensor([1, 2, 0, 2, 0, 1])),
            torch.stack([-w[2], w[1], w[2], -w[0], -w[1], w[0]]))
        e = torch.zeros_like(start)
        e[0, 0, :3, :3] = torch.linalg.matrix_exp(Kw) @ start[0, 0, :3, :3]
        e[0, 0, :3, 3] = start[0, 0, :3, 3] + t
        e[0, 0, 3, 3] = 1.0
        return e

    def errors(e):
        # the angle from the skew part, in fp64 (arccos of the trace loses small angles to rounding)
        R = e[0, 0, :3, :3].double() @ true[0, 0, :3, :3].double().T
        A = 0.5 * (R - R.T)
        rot = float(torch.asin(torch.stack([A[2, 1], A[0, 2], A[1, 0]]).norm().clamp(max=1.0)))
        return rot, float((e[0, 0, :3, 3] - true[0, 0, :3, 3]).double().norm())

    r0, t0 = errors(pose().detach())
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(steps):
            opt.zero_grad()
            img, _ = decoder_forward_(args, pose(), d, hw, bg)
            ((img - target) ** 2).mean().backward()
            opt.step()
            sched.step()
    finally:
        torch.use_deterministic_algorithms(False)
    r1, t1 = errors(pose().detach())
    print(f"[parity] pose recovery: rotation {np.rad2deg(r0):.3f} -> {np.rad2deg(r1):.5f} deg, "
          f"translation {t0:.4f} -> {t1:.6f}")
    assert r1 < r0 / 10 and t1 < t0 / 10


def decoder_forward_(args, ext, d, hw, bg):
    from pf3plat_b200.render import decoder_forward
    return decoder_forward(*args, ext, d["intrinsics"], d["near"], d["far"], hw, bg, camera_gradients=True)
