"""GPU tests of the intrinsics gradient (gs_backward_cam_tanfov, BatchSettings.tanfov with camera gradients on,
render_views / decoder_forward's intrinsics.grad): dL/dtanfov of every output against the fp64 autograd oracle of
tests/intrinsics_oracle.py with the rule of tests.chain_oracle.camera_grad_check, next to the three camera gradients.
Every test prints "[parity]" lines."""
from math import isqrt

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.synthetic import make_scene, make_target
from tests.chain_oracle import camera_grad_check
from tests.intrinsics_oracle import clamped_pairs, intrinsics_oracle
from tests.test_gpu_depth_chain import _depth_batch, _depth_field
from tests.test_gpu_regimes import _settings

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAMES = ("viewmatrix", "projmatrix", "campos", "tanfov")


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


def _gpu(bs, ins, dL, w=None, dA=None, want=(True, True, True, True)):
    """rasterize_batch with camera gradients on and the four camera inputs as leaves (want: which require grad); returns
    their gradients (None where not wanted) and the outputs."""
    from pf3plat_b200.rasterizer import rasterize_batch
    cams = [t.to(DEV).float().reshape(t.shape[0], *s).clone().requires_grad_(r)
            for t, s, r in zip((bs.viewmatrix, bs.projmatrix, bs.campos, bs.tanfov), ((4, 4), (4, 4), (3,), (2,)), want)]
    d = lambda t: None if t is None else t.to(DEV)
    bs = bs._replace(viewmatrix=cams[0], projmatrix=cams[1], campos=cams[2], tanfov=cams[3], bg=d(bs.bg),
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
    grads = [None if c.grad is None else c.grad.reshape(c.shape[0], -1) for c in cams]
    return grads, {k: v.detach() for k, v in o.items()}, {k: v.grad for k, v in leaves.items()}


def _check(label, got, ref, rtol=1e-3):
    for name, g, r in zip(NAMES, got, ref):
        V = r.shape[0]
        camera_grad_check(f"{label} dL/d{name}", g, r, np.zeros((V, 1) + r.shape[1:]), np.zeros((V, 1), bool), rtol=rtol)


def _loss(V, hw, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((V, 3, *hw)) / (hw[0] * hw[1])


TUNINGS = ((0, "default"), (_capi.GS_TUNE_BWD_V1, "bwd v1"), (_capi.GS_TUNE_BWD_OCC4, "bwd occ4"),
           (_capi.GS_TUNE_FWD_WS, "warp-specialised fwd"))
BINNING = ((0, "default"), (_capi.GS_TUNE_FORCE_RADIX_BINNING, "radix"), (_capi.GS_TUNE_NO_SPECULATION, "exact"),
           (_capi.GS_TUNE_NO_STRATA, "no strata"))


@pytest.mark.parametrize("geometry", ["cov3D", "scalerot"])
def test_tanfov_grad_against_oracle_under_every_compositor(geometry):
    """2 scenes x 9 views, view_scale 0.8 .. 1.25, turned cameras; SH degree 3 + cov3D, or colors_precomp + scales /
    rotations with scale_modifier 1.3; colour + depth loss."""
    cams, ins, hw = _depth_batch(geometry)
    V = cams["viewmatrix"].shape[0]
    bs = _settings(cams, hw, sh_degree=3, with_depth=True, scale_modifier=1.0 if geometry == "cov3D" else 1.3)
    dL, w = _loss(V, hw, 5), _depth_field(V, hw, 6)
    ref = intrinsics_oracle(bs, ins, dL, w)
    for tuning, name in TUNINGS:
        got, _, _ = _gpu(bs._replace(tuning=tuning), ins, dL, w)
        _check(f"{geometry} {name}", got, ref)


@pytest.mark.parametrize("mode", ["disparity", "relative_disparity", "log"])
def test_tanfov_grad_depth_modes_alpha_and_antialiasing(mode):
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
    bs = _settings(cams, hw, sh_degree=3, with_depth=True)._replace(depth_mode=mode, depth_near_far=nf, with_alpha=True,
                                                                      antialiasing=True)
    dL, w, dA = _loss(V, hw, 7), _depth_field(V, hw, 8), _depth_field(V, hw, 9)
    ref = intrinsics_oracle(bs, ins, dL, w, dA, antialiasing=True, depth_mode=mode, near_far=nf)
    got, _, _ = _gpu(bs, ins, dL, w, dA)
    # relative disparity divides by 1/near - 1/far: its fp32 chain has the camera gradient's looser bound
    _check(f"{mode} + alpha + aa", got, ref, rtol=2e-3 if mode == "relative_disparity" else 1e-3)


@pytest.mark.parametrize("aa", [False, True])
def test_tanfov_grad_degree4(aa):
    """SH degree 4 (band 4 non-zero), the B4 camera kernels; colour + disparity loss, with and without anti-aliasing."""
    from tests.batch_oracle import scene_batch_args
    from tests.sh4_oracle import with_band4
    from tests.test_gpu_depth_chain import _turned
    hw = (32, 48)
    scenes = [with_band4(_turned(make_scene(1200, 5, *hw, seed=60 + k), seed=70 + k), seed=80 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=np.linspace(0.6, 1.6, 10).astype(np.float32))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    V = 10
    nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
    bs = _settings(cams, hw, sh_degree=4, with_depth=True)._replace(sh_eval_max_degree=4, antialiasing=aa,
                                                                      depth_mode="disparity", depth_near_far=nf)
    dL, w = _loss(V, hw, 21), _depth_field(V, hw, 22)
    ref = intrinsics_oracle(bs, ins, dL, w, antialiasing=aa, depth_mode="disparity", near_far=nf)
    got, _, _ = _gpu(bs, ins, dL, w)
    _check(f"degree 4{' + aa' if aa else ''}", got, ref)


@pytest.mark.parametrize("vps", [1, 19])
def test_tanfov_grad_views_per_scene_and_ragged_frame(vps):
    """1 or 19 views per scene, 3 scenes, a 33 x 250 frame, near 0.5 .. 2 (view_scale 2 .. 0.5)."""
    from tests.batch_oracle import scene_batch_args
    hw = (33, 250)
    scenes = [make_scene(600, vps, *hw, seed=40 + k) for k in range(3)]
    cams, ins = scene_batch_args(scenes, near=np.linspace(0.5, 2.0, 3 * vps).astype(np.float32))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    V = 3 * vps
    bs = _settings(cams, hw, sh_degree=3)
    dL = _loss(V, hw, 11)
    ref = intrinsics_oracle(bs, ins, dL)
    got, _, _ = _gpu(bs, ins, dL)
    _check(f"vps {vps}", got, ref)


@pytest.mark.parametrize("aa", [False, True])
def test_tanfov_grad_cloud_straddling_the_guard_band(aa):
    """Large Gaussians beyond the guard band whose footprints reach into the frame (the clamp term), unequal tanfov per
    axis and per view, alpha and an f(z) depth mode."""
    from tests.test_intrinsics_grad_cpu import scene
    bs, ins = scene(P=400, hw=(48, 64), n_edge=40)
    assert all(clamped_pairs(bs, ins, v) >= 40 for v in range(2))
    nf = np.array([[0.5, 50.0], [0.6, 40.0]])
    bs = bs._replace(with_alpha=True, depth_mode="log", depth_near_far=torch.tensor(nf), antialiasing=aa)
    V, hw = 2, (48, 64)
    dL, w, dA = _loss(V, hw, 31), _depth_field(V, hw, 32), _depth_field(V, hw, 33)
    ins32 = {k: v.float() for k, v in ins.items()}
    ref = intrinsics_oracle(bs, ins32, dL, w, dA, antialiasing=aa, depth_mode="log", near_far=nf)
    got, _, _ = _gpu(bs, ins32, dL, w, dA)
    _check(f"guard band{' + aa' if aa else ''}", got, ref)


@pytest.mark.parametrize("variant", ["plain", "aa_log_alpha"])
def test_tanfov_grad_deterministic_on_every_binning_path(variant):
    """Deterministic mode: dL/dtanfov (and the other three) bit for bit the same on every binning path and run to run,
    and the three camera outputs bit for bit the same with and without dL/dtanfov requested."""
    cams, ins, hw = _depth_batch("cov3D")
    V = cams["viewmatrix"].shape[0]
    bs = _settings(cams, hw, sh_degree=3, with_depth=True)
    dL, w, dA = _loss(V, hw, 12), _depth_field(V, hw, 13), None
    kw = {}
    if variant == "aa_log_alpha":
        nf = torch.stack([1.0 / cams["view_scale"], 40.0 / cams["view_scale"]], -1)
        bs = bs._replace(antialiasing=True, depth_mode="log", depth_near_far=nf, with_alpha=True)
        dA = _depth_field(V, hw, 23)
        kw = dict(antialiasing=True, depth_mode="log", near_far=nf)
    ref = intrinsics_oracle(bs, ins, dL, w, dA, **kw)
    torch.use_deterministic_algorithms(True)
    try:
        first = None
        for tuning, name in BINNING:
            for _ in range(2):
                got, _, _ = _gpu(bs._replace(tuning=tuning), ins, dL, w, dA)
                if first is None:
                    first = got
                    _check("deterministic", got, ref)
                for a, b in zip(got, first):
                    assert torch.equal(a, b), name
            without, _, _ = _gpu(bs._replace(tuning=tuning), ins, dL, w, dA, want=(True, True, True, False))
            assert without[3] is None
            for a, b in zip(without[:3], first[:3]):
                assert torch.equal(a, b), name
            print(f"[parity] {variant}: deterministic camera + tanfov grads bit-identical on {name}, "
                  f"camera grads the same without tanfov")
    finally:
        torch.use_deterministic_algorithms(False)


def _decoder_inputs(b, v, P, hw, seed):
    scs = [make_scene(P, v, *hw, seed=seed + k) for k in range(b)]
    st = lambda f: torch.stack([f(sc) for sc in scs]).to(DEV)
    return dict(means=st(lambda s: s.means), covariances=st(lambda s: s.covariances),
                harmonics=st(lambda s: s.harmonics), opacities=st(lambda s: s.opacities),
                extrinsics=st(lambda s: s.extrinsics), intrinsics=st(lambda s: s.intrinsics),
                near=st(lambda s: s.near), far=st(lambda s: s.far))


def _skewed(K, seed):
    """The intrinsics with off-centre principal points, unequal focal lengths and a small skew."""
    g = torch.Generator().manual_seed(seed)
    K = K.clone()
    n = K.shape[:-2]
    K[..., 0, 0] *= (1 + 0.1 * torch.randn(n, generator=g)).to(K.device)
    K[..., 0, 2] += (0.05 * torch.randn(n, generator=g)).to(K.device)
    K[..., 1, 2] += (0.05 * torch.randn(n, generator=g)).to(K.device)
    K[..., 0, 1] += (0.01 * torch.randn(n, generator=g)).to(K.device)
    return K


def test_settings_off_or_intrinsics_without_grad_are_bit_identical():
    """Camera gradients off: intrinsics that require grad get none, and every output and gradient is the bytes of a call
    whose intrinsics do not.  On, with intrinsics that do not require grad: the same bytes as with intrinsics that do
    (the extrinsics' gradient included), in deterministic mode."""
    from pf3plat_b200.render import decoder_forward
    hw = (64, 64)
    d = _decoder_inputs(2, 2, 3000, hw, 50)
    K0 = _skewed(d["intrinsics"], 1)
    bg = torch.zeros(3, device=DEV)
    target = make_target(4, *hw, seed=4).to(DEV).reshape(2, 2, 3, *hw)
    torch.use_deterministic_algorithms(True)
    try:
        for cam in (False, True):
            runs = []
            for kreq in (False, True):
                e = d["extrinsics"].clone().requires_grad_(True)
                K = K0.clone().requires_grad_(kreq)
                m = d["means"].clone().requires_grad_(True)
                color, depth = decoder_forward(m, d["covariances"], d["harmonics"], d["opacities"], e, K, d["near"],
                                               d["far"], hw, bg, depth_mode="depth", camera_gradients=cam)
                (((color - target) ** 2).mean() + 1e-3 * depth.mean()).backward()
                runs.append((color, depth, e.grad, m.grad, K.grad))
            for a, b in zip(runs[0][:4], runs[1][:4]):
                assert torch.equal(a, b), cam
            assert runs[0][4] is None
            if cam:
                assert runs[1][4] is not None and float(runs[1][4].abs().max()) > 0
            else:
                assert runs[1][4] is None
    finally:
        torch.use_deterministic_algorithms(False)
    print("[parity] camera gradients off / intrinsics without grad: bit-identical outputs and gradients")


def test_decoder_forward_intrinsics_grad_matches_the_reference_glue():
    """decoder_forward(camera_gradients=True) at PF3plat's training shape (14 scenes x 3 views x 131072 Gaussians,
    256 x 256), skewed off-centre intrinsics: intrinsics.grad in all nine entries, view by view, against the operator's
    dL/dtanfov and dL/dprojmatrix carried through render_cuda's glue (get_fov, get_projection_matrix, view @ P) by fp64
    autograd -- the glue tests/test_intrinsics_grad_cpu.py pins to the reference's own at 1e-10."""
    from pf3plat_b200.cameras import get_fov, get_projection_matrix, make_view_batch
    from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch
    from pf3plat_b200.render import decoder_forward
    b, v, hw = 14, 3, (256, 256)
    d = _decoder_inputs(b, v, 131072, hw, 70)
    K0 = _skewed(d["intrinsics"], 2)
    bg = torch.zeros(3, device=DEV)
    target = make_target(b * v, *hw, seed=2).to(DEV).reshape(b, v, 3, *hw)
    K = K0.clone().requires_grad_(True)
    color, _ = decoder_forward(d["means"], d["covariances"], d["harmonics"], d["opacities"], d["extrinsics"], K,
                               d["near"], d["far"], hw, bg, camera_gradients=True)
    ((color - target) ** 2).mean().backward()
    got = K.grad.reshape(b * v, 9).double().cpu()
    # the operator's own camera gradients on the same views, then the glue in fp64
    flat = lambda t: t.reshape(b * v, *t.shape[2:])
    ext, nr, fr = flat(d["extrinsics"]), flat(d["near"]), flat(d["far"])
    vb = make_view_batch(ext, flat(K0), nr, fr, True)
    pm, tf = vb.projmatrix.clone().requires_grad_(True), vb.tanfov.clone().requires_grad_(True)
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=vb.viewmatrix, projmatrix=pm,
                       campos=vb.campos, bg=bg.expand(b * v, 3), sh_degree=isqrt(d["harmonics"].shape[-1]) - 1,
                       tanfov=tf, view_scale=vb.scale,
                       camera_gradients=True)
    shs = d["harmonics"].transpose(-1, -2)
    from pf3plat_b200.render import _cov6
    img = rasterize_batch(bs, d["means"], d["opacities"], shs=shs, cov3D_precomp=_cov6(d["covariances"]))[0]
    ((img.reshape(b, v, 3, *hw) - target) ** 2).mean().backward()
    K64 = flat(K0).double().cpu().requires_grad_(True)
    n64, f64 = nr.double().cpu(), fr.double().cpu()
    fov_x, fov_y = get_fov(K64).unbind(-1)
    tan = torch.stack(((0.5 * fov_x).tan(), (0.5 * fov_y).tan()), -1)
    pt = get_projection_matrix(n64 * (1 / n64), f64 * (1 / n64), fov_x, fov_y).transpose(-1, -2)
    full = vb.viewmatrix.double().cpu() @ pt
    ((tan * tf.grad.double().cpu()).sum() + (full * pm.grad.double().cpu()).sum()).backward()
    ref = K64.grad.reshape(b * v, 9)
    err = (got - ref).abs().max(dim=1).values / ref.abs().max(dim=1).values
    print(f"[parity] decoder_forward intrinsics grad vs glue composition: worst per-view max rel err {float(err.max()):.2e}")
    assert float(err.max()) < 1e-3
    assert (ref[:, [0, 1, 2, 4, 5]].abs() > 0).all()


def _refine(with_pose):
    """Adam on the MSE through decoder_forward(camera_gradients=True): fx and fy of a target view perturbed by +4 % and
    -3 % (and, with_pose, its pose by 1 degree and 2 % of the baseline); returns the focal and pose errors before and
    after 300 steps, in deterministic mode."""
    from pf3plat_b200.render import decoder_forward
    hw = (128, 128)
    d = _decoder_inputs(1, 1, 40000, hw, 90)
    d["near"], d["far"] = d["near"] * 0.7, d["far"] * 0.7
    bg = torch.zeros(3, device=DEV)
    args = (d["means"], d["covariances"], d["harmonics"], d["opacities"])
    true_e, true_k = d["extrinsics"], d["intrinsics"]
    with torch.no_grad():
        target, _ = decoder_forward(*args, true_e, true_k, d["near"], d["far"], hw, bg)
    start_e = true_e.clone()
    if with_pose:
        g = torch.Generator().manual_seed(3)
        axis = torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0)
        A = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
        start_e[0, 0, :3, :3] = torch.linalg.matrix_exp(np.deg2rad(1.0) * A).to(DEV, torch.float32) @ true_e[0, 0, :3, :3]
        base = float(true_e[0, 0, :3, 3].norm().clamp_min(1.0))
        start_e[0, 0, :3, 3] += (0.02 * base * torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)).to(DEV)
    log_f0 = torch.tensor([np.log(1.04), np.log(0.97)], device=DEV)
    lf = log_f0.clone().requires_grad_(True)        # log of the focal factors applied to the true fx, fy
    w = torch.zeros(3, device=DEV, requires_grad=True)
    t = torch.zeros(3, device=DEV, requires_grad=True)

    def cams():
        # fx and fy scaled, the principal point and the skew left alone
        S = torch.ones(3, 3, device=DEV) + torch.diag(torch.stack([lf[0].exp() - 1, lf[1].exp() - 1,
                                                                   torch.zeros((), device=DEV)]))
        K = true_k * S
        if not with_pose:
            return start_e, K
        Kw = torch.zeros(3, 3, device=DEV).index_put(
            (torch.tensor([0, 0, 1, 1, 2, 2]), torch.tensor([1, 2, 0, 2, 0, 1])),
            torch.stack([-w[2], w[1], w[2], -w[0], -w[1], w[0]]))
        e = torch.zeros_like(start_e)
        e[0, 0, :3, :3] = torch.linalg.matrix_exp(Kw) @ start_e[0, 0, :3, :3]
        e[0, 0, :3, 3] = start_e[0, 0, :3, 3] + t
        e[0, 0, 3, 3] = 1.0
        return e, K

    def errors():
        e, _ = cams()
        R = e[0, 0, :3, :3].double() @ true_e[0, 0, :3, :3].double().T
        A = 0.5 * (R - R.T)
        rot = float(torch.asin(torch.stack([A[2, 1], A[0, 2], A[1, 0]]).norm().clamp(max=1.0)))
        return float(lf.detach().abs().max()), rot, float((e[0, 0, :3, 3] - true_e[0, 0, :3, 3]).double().norm())

    before = errors()
    steps = 300
    params = [lf, w, t] if with_pose else [lf]
    opt = torch.optim.Adam(params, lr=5e-3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps)
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(steps):
            opt.zero_grad()
            e, K = cams()
            img, _ = decoder_forward(*args, e, K, d["near"], d["far"], hw, bg, camera_gradients=True)
            ((img - target) ** 2).mean().backward()
            opt.step()
            sched.step()
    finally:
        torch.use_deterministic_algorithms(False)
    return before, errors()


@pytest.mark.parametrize("with_pose", [False, True])
def test_focal_recovery_by_adam_through_decoder_forward(with_pose):
    (f0, r0, t0), (f1, r1, t1) = _refine(with_pose)
    print(f"[parity] focal recovery{' with pose' if with_pose else ''}: focal log-error {f0:.4f} -> {f1:.6f}, "
          f"rotation {np.rad2deg(r0):.3f} -> {np.rad2deg(r1):.5f} deg, translation {t0:.4f} -> {t1:.6f}")
    assert f1 < f0 / 10
    if with_pose:
        assert r1 < r0 / 10 and t1 < t0 / 10
