"""Lazy strata (DESIGN.md 5.2): with per-view depth strata the stratum sort sorts only the strata each tile's previous
forward read, and k_composite_fwd sorts any further stratum it reaches.  Every output and every gradient of
the deterministic backward must be bit-identical to GS_TUNE_ALL_STRATA (every stratum sorted up front) on the same
inputs: colour, radii, depth, the accumulated opacity 1 - final_T, and dL/d(means3D, opacities, shs, cov3D_precomp).

The two settings run the same call sequence, each on a stream of its own (hence a rasterizer context, and a learned
"strata needed" table, of its own).  Each test's shape (Gaussians per scene) is one no other test renders, and the module
starts and ends with no context cached."""
import pytest
import torch

from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.batch_oracle import scene_batch_args
from tests.test_gpu_forward_variants import _with_culled
from tests.test_gpu_regimes import _settings

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _fresh_contexts():
    """Contexts are cached per (device, stream) and torch reuses streams: start and end with none cached."""
    import gc
    from pf3plat_b200.rasterizer import destroy_contexts
    torch.cuda.synchronize()
    destroy_contexts()
    yield
    gc.collect()
    torch.cuda.synchronize()
    destroy_contexts()

KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _inputs(scenes, dev):
    cams, ins = scene_batch_args(scenes, device=dev)
    hw = scenes[0].image_shape
    return cams, hw, {k: v for k, v in ins.items() if k in KEEP}


def _call(bs, ins, backward):
    from pf3plat_b200.rasterizer import last_stats, rasterize_batch
    dev = bs.viewmatrix.device
    leaves = {k: v.clone().requires_grad_(backward) for k, v in ins.items()}
    out = rasterize_batch(bs, **leaves)
    st = last_stats(dev)
    if not backward:
        return [o.detach().clone() for o in out], None, st
    V, _, H, W = out[0].shape
    target = make_target(V, H, W).to(dev)
    loss = ((out[0] - target) ** 2).mean() + 1e-3 * out[2].mean() + 1e-2 * out[3].mean()
    loss.backward()
    return [o.detach().clone() for o in out], {k: t.grad.clone() for k, t in leaves.items()}, st


def _both(dev, calls):
    """calls: [(bs, ins, backward)].  Returns {tuning: [(outputs, grads, stats)]} for the default and GS_TUNE_ALL_STRATA."""
    from pf3plat_b200 import _capi
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    res = {}
    try:
        for extra in (0, _capi.GS_TUNE_ALL_STRATA):
            stream = torch.cuda.Stream(dev)
            with torch.cuda.stream(stream):
                res[extra] = [_call(bs._replace(tuning=bs.tuning | extra), ins, bw) for bs, ins, bw in calls]
                stream.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return res


def _identical(label, res):
    from pf3plat_b200 import _capi
    lazy, ref = res[0], res[_capi.GS_TUNE_ALL_STRATA]
    for i, ((out, grads, st), (out0, grads0, st0)) in enumerate(zip(lazy, ref)):
        for name, a, b in zip(("color", "radii", "depth", "alpha"), out, out0):
            assert torch.equal(a, b), f"{label} call {i}: {name} differs (max |diff| {float((a.double() - b.double()).abs().max()):.3e})"
        assert (grads is None) == (grads0 is None)
        for k in grads0 or {}:
            assert torch.equal(grads[k], grads0[k]), f"{label} call {i}: dL/d{k} differs"
        assert st["num_rendered"] == st0["num_rendered"] and st["max_tile_list"] == st0["max_tile_list"], (label, i, st, st0)
        print(f"[lazy strata] {label} call {i}: speculative={st['speculative']} D={st['num_rendered']} "
              f"redos={st['overflow_redos']}")
    return lazy


def _bs(cams, hw):
    return _settings(cams, hw, with_depth=True)._replace(with_alpha=True)


def test_c2_static_steady_state():
    dev = _dev()
    cams, hw, ins = _inputs([_with_culled(make_scene(500_000, 8, 256, 256, seed=0), 11)], dev)
    bs = _bs(cams, hw)
    lazy = _identical("C2", _both(dev, [(bs, ins, False)] * 4 + [(bs, ins, True)]))
    assert [st["speculative"] for _, _, st in lazy] == [0, 2, 2, 2, 2]   # exact, trial, then lazy strata in steady state
    assert lazy[-1][2]["overflow_redos"] == 0


def test_stale_table_runs_the_compositor_sort():
    """The table is learned on C2, where every tile saturates within its first few strata; then the same shape renders
    with weaker opacities.  Divided by 20 everywhere, about 1.5 units of optical depth are left per pixel: no pixel
    saturates, every tile reads its whole list, so every stratum the stratum sort skipped must be sorted by the
    compositor -- a wrong lazy sort cannot match the reference.  The nearer half divided by 20 moves saturation deeper
    tile by tile.  A last C2 call then learns the dense table back."""
    dev = _dev()
    sc = _with_culled(make_scene(500_000, 8, 256, 256, seed=0), 13)
    cams, hw, ins = _inputs([sc], dev)
    near = sc.means[:, 2] < sc.means[:, 2].median()
    faint_near = dict(ins, opacities=torch.where(near.to(dev)[None], ins["opacities"] / 20, ins["opacities"]))
    faint_all = dict(ins, opacities=ins["opacities"] / 20)
    bs = _bs(cams, hw)
    calls = [(bs, ins, False)] * 4 + [(bs, faint_near, True), (bs, ins, False), (bs, faint_all, True), (bs, ins, True)]
    lazy = _identical("stale table", _both(dev, calls))
    assert all(st["speculative"] == 2 for _, _, st in lazy[1:]), [st["speculative"] for _, _, st in lazy]
    # the faint cloud really is unsaturated: the accumulated opacity stays well below 1 - 1e-4 almost everywhere
    assert float((lazy[6][0][3] < 0.999).float().mean()) > 0.9


def test_moving_cloud():
    dev = _dev()
    sc = _with_culled(make_scene(500_000, 8, 256, 256, seed=0), 17)
    cams, hw, ins = _inputs([sc], dev)
    g = torch.Generator().manual_seed(77)
    base = sc.means
    px_at_depth = 2.0 * (0.5 / 0.86) / 256
    calls = []
    for k in range(6):
        m = base + torch.randn(base.shape, generator=g) * (base[:, 2:3] * px_at_depth) * torch.tensor([1.0, 1.0, 0.0])
        redraw = torch.rand(base.shape[0], generator=g) < 0.05
        z = base[redraw, 2:3]
        m[redraw] = torch.cat([(torch.rand(int(redraw.sum()), 2, generator=g) * 2.1 - 1.05) * (0.5 / 0.86) * z, z], 1)
        calls.append((_bs(cams, hw), dict(ins, means3D=m[None].contiguous().to(dev)), k == 5))
    _identical("moving cloud", _both(dev, calls))


def test_pixel_aligned_c5_keeps_per_tile_strata():
    dev = _dev()
    cams, hw, ins = _inputs([_with_culled(make_pixel_aligned_scene(128, 128, 4, seed=3), 19)], dev)
    bs = _bs(cams, hw)
    lazy = _identical("C5", _both(dev, [(bs, ins, False)] * 5 + [(bs, ins, True)]))
    assert lazy[-1][2]["speculative"] == 2


def test_multi_scene():
    dev = _dev()
    scenes = [_with_culled(make_scene(150_000, 3, 192, 160, seed=s), 23) for s in (5, 6)]
    cams, hw, ins = _inputs(scenes, dev)
    bs = _bs(cams, hw)
    lazy = _identical("two scenes", _both(dev, [(bs, ins, False)] * 4 + [(bs, ins, True)]))
    assert lazy[-1][2]["speculative"] == 2
