"""GPU checks of the sync-free rasterizer path (SyncFreeWorkspace, gs_forward_sync_free / gs_backward_sync_free,
DESIGN.md 5.18), every test under poisoned allocations:
  1. the same results as the default path: images, depth, alpha and radii bit for bit, gradients bit for bit under
     deterministic algorithms (within a tight bound with float atomics) -- C2, the training shape, ragged frames, P = 0,
     an off-screen cloud, tile lists above 8192 and above 65536, every depth mode, alpha, anti-aliasing, SH degrees 0-4,
     camera and intrinsics gradients;
  2. no host wait: decoder + photometric loss + backward captured in a CUDA graph and replayed on a moving cloud, and an
     eager call under torch.cuda.set_sync_debug_mode("error");
  3. capacity: exactly enough, one short, 1 and 0, inside guard regions;
  4. no interference with default calls on the same context;
  5. scenes computed alone give their rows of the batch."""
import contextlib

import pytest
import torch

from pf3plat_b200.cameras import make_view_batch
from pf3plat_b200.rasterizer import BatchSettings, SyncFreeWorkspace, last_stats, rasterize_batch
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene
from tests.poison import poisoned  # noqa: F401
from tests.regimes import long_list_scene, offscreen_scene

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


def _batch(scenes, dev):
    """Scenes of equal P and views -> view batch and operator inputs (S, P, ...)."""
    cat = lambda f: torch.cat([f(s) for s in scenes]).to(dev)
    ext, intr = cat(lambda s: s.extrinsics), cat(lambda s: s.intrinsics)
    near, far, bg = cat(lambda s: s.near), cat(lambda s: s.far), cat(lambda s: s.background)
    vb = make_view_batch(ext, intr, near, far)
    st = lambda f: torch.stack([f(s) for s in scenes]).to(dev)
    c = lambda s: s.covariances
    ins = {"means3D": st(lambda s: s.means), "opacities": st(lambda s: s.opacities),
           "shs": st(lambda s: s.harmonics.transpose(-1, -2)),
           "cov3D_precomp": st(lambda s: torch.stack([c(s)[:, 0, 0], c(s)[:, 0, 1], c(s)[:, 0, 2], c(s)[:, 1, 1],
                                                      c(s)[:, 1, 2], c(s)[:, 2, 2]], -1))}
    return vb, bg, torch.stack([near, far], -1), ins, scenes[0].image_shape


def _run(batch, ws=None, *, depth_mode=None, alpha=False, aa=False, degree=4, cam=False, seed=3, square=False):
    """One forward + backward of a fixed random linear loss (square: half the sum of squares, whose incoming gradient
    of a row does not depend on the batch around it); {name: tensor} of outputs and gradients."""
    vb, bg, nf, ins, (h, w) = batch
    dev = bg.device
    leaf = lambda t: t.detach().clone().requires_grad_(True)
    cams = {"viewmatrix": vb.viewmatrix, "projmatrix": vb.projmatrix, "campos": vb.campos, "tanfov": vb.tanfov}
    cams = {k: leaf(v) if cam else v.detach() for k, v in cams.items()}
    bs = BatchSettings(image_height=h, image_width=w, bg=bg, sh_degree=degree, view_scale=vb.scale,
                       with_depth=depth_mode is not None, depth_mode=depth_mode or "depth",
                       depth_near_far=nf if depth_mode in ("relative_disparity", "log") else None, with_alpha=alpha,
                       antialiasing=aa, camera_gradients=cam, sh_eval_max_degree=4, **cams)
    leaves = {k: leaf(v) for k, v in ins.items()}
    out = rasterize_batch(bs, **leaves, workspace=ws)
    g = torch.Generator(device=dev).manual_seed(seed)
    named = {"color": out[0], "radii": out[1]}
    if depth_mode is not None:
        named["depth"] = out[2]
    if alpha:
        named["alpha"] = out[-1]
    weight = (lambda t: 0.5 * t) if square else (lambda t: torch.rand(t.shape, generator=g, device=dev))
    loss = sum((t * weight(t)).sum() for k, t in named.items() if k != "radii")
    wrt = {**leaves, **({k: v for k, v in cams.items()} if cam else {})}
    if ins["means3D"].shape[1] > 0:
        grads = torch.autograd.grad(loss, list(wrt.values()))
        named.update({"d_" + k: gr for k, gr in zip(wrt, grads)})
    return {k: v.detach() for k, v in named.items()}


def _workspace(batch, capacity, **kw):
    vb, bg, nf, ins, hw = batch
    S, P = ins["means3D"].shape[:2]
    return SyncFreeWorkspace(bg.device, S, vb.viewmatrix.shape[0], P, hw, capacity, **kw)


def _required(batch, **kw):
    """D of a default forward of the batch, from its stats"""
    _run(batch, **kw)
    return last_stats(_dev())["num_rendered"]


def _compare(a, b, exact_grads, label):
    assert a.keys() == b.keys(), label
    for k in a:
        if not k.startswith("d_") or exact_grads:
            assert torch.equal(a[k], b[k]), (label, k)
        else:   # float atomics: a different summation order
            scale = a[k].abs().max().clamp_min(1e-30)
            assert float((a[k] - b[k]).abs().max() / scale) < 1e-4, (label, k)


def _parity(batch, margin=1.0, det=True, **kw):
    with _deterministic(det):
        ref = _run(batch, **kw)
        D = last_stats(_dev())["num_rendered"]
        ws = _workspace(batch, max(int(D * margin), 0), depth=True, alpha=True, deterministic=True, camera_grad=True)
        got = _run(batch, ws, **kw)
    assert ws.status() == (D, False)
    _compare(ref, got, det, str(kw))
    return D


def test_c2_cloud(poisoned):
    batch = _batch([make_scene(500_000, 8, 256, 256, seed=0)], _dev())
    _parity(batch, depth_mode="depth", alpha=True)


def test_c2_cloud_float_atomics(poisoned):
    batch = _batch([make_scene(500_000, 8, 256, 256, seed=0)], _dev())
    _parity(batch, margin=1.3, det=False, depth_mode="depth")


def _training_scenes(b=14, v=3):
    return [make_pixel_aligned_scene(256, 256, v, seed=s) for s in range(b)]


def test_training_shape(poisoned):
    _parity(_batch(_training_scenes(), _dev()), depth_mode="depth", cam=True)


@pytest.mark.parametrize("case", ["ragged", "empty", "offscreen"])
def test_small_and_degenerate_shapes(poisoned, case):
    dev = _dev()
    if case == "ragged":
        batch = _batch([make_scene(3000, 3, 37, 53, seed=s) for s in range(2)], dev)
    elif case == "empty":
        batch = _batch([make_scene(0, 2, 40, 24, seed=1)], dev)
    else:
        batch = _batch([offscreen_scene(500, 500, 2, 40, 56, seed=2)], dev)
        sc = batch[3]["means3D"]
        batch[3]["means3D"] = sc + torch.tensor([0.0, 0.0, -1e3], device=dev)   # every Gaussian behind the cameras
    D = _parity(batch, depth_mode="disparity", alpha=True)
    assert (D == 0) == (case != "ragged")


@pytest.mark.parametrize("n,views,hw", [(10_000, 2, (40, 52)), (70_000, 1, (16, 16))], ids=["above8192", "above65536"])
def test_long_tile_lists(poisoned, n, views, hw):
    sc = long_list_scene(n, views, *hw, box=(2.0, 2.0, 13.0, 13.0), seed=11)
    _parity(_batch([sc], _dev()), depth_mode="depth", alpha=True)
    assert last_stats(_dev())["max_tile_list"] == -1


FEATURES = [dict(depth_mode="depth", degree=4, aa=False), dict(depth_mode="disparity", degree=3, aa=True),
            dict(depth_mode="relative_disparity", degree=2, alpha=True), dict(depth_mode="log", degree=1, aa=True),
            dict(degree=0, alpha=True, aa=True)]


@pytest.mark.parametrize("feat", FEATURES, ids=lambda f: "-".join(f"{k}={v}" for k, v in f.items()))
@pytest.mark.parametrize("cam", [False, True])
def test_features(poisoned, feat, cam):
    _parity(_batch([make_scene(20_000, 3, 72, 88, seed=5 + k) for k in range(2)], _dev()), cam=cam, **feat)


def test_capacity_limits_inside_guard_regions(poisoned):
    dev = _dev()
    batch = _batch([make_scene(20_000, 3, 64, 80, seed=21)], dev)
    kw = dict(depth_mode="depth", alpha=True, cam=True)
    with _deterministic():
        ref = _run(batch, **kw)
        D = last_stats(dev)["num_rendered"]
        assert D > 2
        vb, bg, nf, ins, hw = batch
        from pf3plat_b200.rasterizer import sync_free_workspace_bytes
        need = sync_free_workspace_bytes(1, 3, 20_000, *hw, 2 * D, deterministic=True, camera_grad=True)
        guard = 1 << 16
        big = torch.empty(2 * guard + need, dtype=torch.uint8, device=dev)
        pattern = (torch.arange(guard, device=dev) * 7 % 251).to(torch.uint8)
        big[:guard], big[-guard:] = pattern, pattern
        inner = big[guard:guard + need]
        flags = dict(depth=True, alpha=True, deterministic=True, camera_grad=True)
        for cap in (D, D - 1, 1, 0):
            ws = _workspace(batch, cap, buffer=inner, **flags)
            got = _run(batch, ws, **kw)
            assert torch.equal(big[:guard], pattern) and torch.equal(big[-guard:], pattern), cap
            assert torch.equal(got["radii"], ref["radii"]), cap
            if cap == D:
                _compare(ref, got, True, "capacity = D")
                assert ws.status() == (D, False)
                continue
            assert ws.status() == (D, True), cap
            for k, t in got.items():
                if k != "radii":
                    assert torch.isnan(t).all(), (cap, k)
        # the status stays set through a later call that fits (an off-screen cloud: D = 0), until it is cleared
        off = (vb, bg, nf, {**ins, "means3D": ins["means3D"] + torch.tensor([0.0, 0.0, -1e3], device=dev)}, hw)
        ref_off = _run(off, **kw)
        got_off = _run(off, ws, **kw)
        _compare(ref_off, got_off, True, "off-screen after an exceeded call")
        assert ws.status() == (D, True)
        ws.clear_status()
        assert ws.status() == (0, False)
        ws = _workspace(batch, 2 * D, buffer=inner, **flags)
        _compare(ref, _run(batch, ws, **kw), True, "capacity 2D after exhaustion")
        assert ws.status() == (D, False)
        assert torch.equal(big[:guard], pattern) and torch.equal(big[-guard:], pattern)


def test_eager_call_never_synchronises(poisoned):
    dev = _dev()
    batch = _batch([make_scene(50_000, 4, 128, 128, seed=31)], dev)
    D = _required(batch, depth_mode="depth")
    ws = _workspace(batch, 2 * D, depth=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(batch, ws, depth_mode="depth")
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_reused_workspace_and_flag_refusals(poisoned):
    dev = _dev()
    batch = _batch([make_scene(5_000, 2, 48, 48, seed=41)], dev)
    vb, bg, nf, ins, (h, w) = batch
    ws = _workspace(batch, 10**6)
    bs = BatchSettings(image_height=h, image_width=w, viewmatrix=vb.viewmatrix, projmatrix=vb.projmatrix,
                       campos=vb.campos, bg=bg, sh_degree=3, tanfov=vb.tanfov, view_scale=vb.scale)
    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    first = rasterize_batch(bs, **leaves, workspace=ws)[0]
    rasterize_batch(bs, **{k: v.detach() for k, v in ins.items()}, workspace=ws)
    with pytest.raises(RuntimeError, match="reused"):
        first.sum().backward()
    with pytest.raises(ValueError, match="depth=True"):
        rasterize_batch(bs._replace(with_depth=True), **ins, workspace=ws)
    with pytest.raises(ValueError, match="sized for"):
        rasterize_batch(bs, ins["means3D"][:, :100], ins["opacities"][:, :100], shs=ins["shs"][:, :100],
                        cov3D_precomp=ins["cov3D_precomp"][:, :100], workspace=ws)
    out = rasterize_batch(bs, **{k: v.clone().requires_grad_(True) for k, v in ins.items()}, workspace=ws)[0]
    with _deterministic(), pytest.raises(ValueError, match="deterministic=True"):
        out.sum().backward()


def test_no_interference_with_default_calls(poisoned):
    dev = _dev()
    a = _batch([make_scene(40_000, 4, 96, 128, seed=51)], dev)
    b = _batch([make_scene(10_000, 2, 64, 64, seed=52) for _ in range(2)], dev)
    kw = dict(depth_mode="depth", alpha=True)
    flags = dict(depth=True, alpha=True, deterministic=True)
    wa, wb = _workspace(a, 10**6, **flags), _workspace(b, 10**6, **flags)

    def sequence(with_sync_free):
        s = torch.cuda.Stream(dev)   # a fresh stream: a fresh context with nothing learned yet
        outs = []
        with torch.cuda.stream(s):
            for step in range(8):
                if with_sync_free:
                    _run(a, wa, **kw)
                    _run(b, wb, **kw)
                x = a if step % 3 != 2 else b
                outs.append((_run(x, **kw), last_stats(dev)))
                if with_sync_free:
                    _run(x, wa if x is a else wb, **kw)
        torch.cuda.synchronize()
        return outs

    with _deterministic():
        plain, mixed = sequence(False), sequence(True)
    for k, ((o1, s1), (o2, s2)) in enumerate(zip(plain, mixed)):
        _compare(o1, o2, True, f"step {k}")
        assert s1 == s2, (k, s1, s2)


def test_scenes_are_independent(poisoned):
    dev = _dev()
    scenes = [make_scene(8_000, 2, 64, 96, seed=60 + k) for k in range(5)]
    kw = dict(depth_mode="depth", alpha=True, cam=True, square=True)
    flags = dict(depth=True, alpha=True, deterministic=True, camera_grad=True)
    with _deterministic():
        whole = _batch(scenes, dev)
        got = _run(whole, _workspace(whole, 10**6, **flags), **kw)
        for k, sc in enumerate(scenes):
            one = _batch([sc], dev)
            alone = _run(one, _workspace(one, 10**6, **flags), **kw)
            for name, t in alone.items():
                rows = got[name][k:k + 1] if name in ("d_means3D", "d_opacities", "d_shs", "d_cov3D_precomp") \
                    else got[name][2 * k:2 * k + 2]
                assert torch.equal(rows, t), (k, name)


def _moving(means, g, px):
    m = means + torch.randn(means.shape, generator=g, device=means.device) * (means[..., 2:3] * px) * \
        torch.tensor([1.0, 1.0, 0.0], device=means.device)
    redraw = torch.rand(means.shape[:2], generator=g, device=means.device) < 0.05
    perm = torch.randperm(means.shape[1], generator=g, device=means.device)
    return torch.where(redraw[..., None], means[:, perm], m)


def test_training_step_in_a_cuda_graph(poisoned):
    """decoder_forward + photometric_loss + backward at b = 14, v = 3, 131072 Gaussians per scene, 256 x 256."""
    from pf3plat_b200.losses import photometric_loss
    from pf3plat_b200.render import decoder_forward
    dev = _dev()
    b, v = 14, 3
    scenes = _training_scenes(b, v)
    st = lambda f: torch.stack([f(s) for s in scenes]).to(dev)
    c = lambda s: s.covariances
    means0 = st(lambda s: s.means)
    cov6 = st(lambda s: torch.stack([c(s)[:, 0, 0], c(s)[:, 0, 1], c(s)[:, 0, 2], c(s)[:, 1, 1], c(s)[:, 1, 2],
                                     c(s)[:, 2, 2]], -1))
    harm, opac = st(lambda s: s.harmonics), st(lambda s: s.opacities)
    ext, intr = st(lambda s: s.extrinsics), st(lambda s: s.intrinsics)
    near, far = st(lambda s: s.near), st(lambda s: s.far)
    bg = torch.zeros(3, device=dev)
    target = torch.rand(b, v, 3, 256, 256, generator=torch.Generator().manual_seed(9)).to(dev)
    static = {"means": means0.clone(), "cov": cov6.clone(), "harm": harm.clone(), "opac": opac.clone()}

    def step(inputs, ws):
        leaves = [t.detach().requires_grad_(True) for t in inputs.values()]
        color, _ = decoder_forward(leaves[0], leaves[1], leaves[2], leaves[3], ext, intr, near, far, (256, 256), bg,
                                   depth_mode=None, sh_eval_max_degree=4, workspace=ws)
        loss = photometric_loss(color.flatten(0, 1), target.flatten(0, 1))
        return (color.detach(),) + torch.autograd.grad(loss, leaves)

    with _deterministic():
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            step(static, None)
            D = last_stats(dev)["num_rendered"]
            ws = SyncFreeWorkspace(dev, b, b * v, means0.shape[1], (256, 256), int(D * 1.5), deterministic=True)
            for _ in range(2):
                step(static, ws)
            torch.cuda.synchronize()
            pool = {k: last_stats(dev)[k] for k in ("pool_reserved_bytes", "pool_used_bytes")}
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            outs = step(static, ws)
        with torch.cuda.stream(s):
            assert {k: last_stats(dev)[k] for k in pool} == pool
        g = torch.Generator(device=dev).manual_seed(17)
        px = 2.0 * (0.5 / 0.86) / 256
        for k in range(5):
            moved = _moving(means0, g, px)
            static["means"].copy_(moved)
            graph.replay()
            ref = step({**static, "means": moved}, None)
            torch.cuda.synchronize()
            for name, a, r in zip(("color", "means", "cov", "harm", "opac"), outs, ref):
                assert torch.equal(a, r), (k, name)
        with torch.cuda.stream(s):
            assert {k: last_stats(dev)[k] for k in pool} == pool
        required, exceeded = ws.status()
        assert not exceeded and required <= int(D * 1.5)
