"""GPU parity of the backward on every layout the forward can leave its tile lists in, on tile lists longer than the
shared-memory sort (8192 entries), on frames whose sides are not multiples of the tile or of the backward compositor's
8 x 4 warp block, and for saved states whose backward runs after later forwards on the same context.

The backward compositor walks each pixel's list from `ranges[tile].x` up to `n_contrib`, in whatever layout the forward
left: dense (exact path, radix fallback) or sparse (speculative paths: tile t of view v starts at t * BIN_SUB * sub_cap).
Every test states which path ran (`last_stats()`) or which regime the oracle saw, and prints it in "[regime]" lines.

References: the batched CPU oracle in fp64 (tests/batch_oracle.py).  Incoming gradients are seeded normal fields,
different at every pixel of every view, for colour and for depth.  Criteria are tests/util.py's; paths that build
identical lists must also agree with each other within 2e-5 of each gradient's max-abs (only the order of the atomic
additions differs)."""
import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.regimes import edge_straddle_scene, long_list_scene
from tests.test_gpu_depth_chain import _leaves
from tests.test_gpu_regimes import _check_grads, _check_images, _check_radii, _settings
from tests.test_oracle_ragged_cpu import edge_contributors

pytestmark = pytest.mark.gpu

PATH_RTOL = 2e-5


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _incoming(V, hw, seed):
    """Seeded dL/dcolor [V,3,H,W] and dL/ddepth [V,H,W]: signed, different at every pixel and view."""
    rng = np.random.default_rng(seed)
    n = hw[0] * hw[1]
    return ((rng.standard_normal((V, 3, *hw)) / n).astype(np.float32),
            (rng.standard_normal((V, *hw)) / n).astype(np.float32))


def _forward(bs, ins, grad=True):
    """rasterize_batch on device copies of `ins` (and a means2D sink).  Returns (outputs, leaves)."""
    from pf3plat_b200.rasterizer import rasterize_batch
    dev = bs.viewmatrix.device
    if not grad:
        with torch.no_grad():
            return rasterize_batch(bs, **{k: v.to(dev) for k, v in ins.items()}), None
    leaves = _leaves(ins, dev, bs.viewmatrix.shape[0])
    return rasterize_batch(bs, **leaves), leaves


def _backward(out, leaves, dL, dLd):
    dev = out[0].device
    torch.autograd.backward([out[0], out[2]], [torch.as_tensor(dL, device=dev), torch.as_tensor(dLd, device=dev)])
    return {k: t.grad.detach().clone() for k, t in leaves.items()}


def _run(bs, ins, dL, dLd):
    out, leaves = _forward(bs, ins)
    grads = _backward(out, leaves, dL, dLd)
    return [o.detach() for o in out], grads


def _check_all(label, out, grads, ob, gref, max_fragile_frac=0.03):
    color, radii, depth = out
    _check_images(color, ob, label, max_fragile_frac=max_fragile_frac, depth=depth)
    _check_radii(radii, ob, label)
    assert set(grads) == {k for k in gref if gref[k] is not None}
    _check_grads(label, grads, gref, ob.affected(), ob.VPS)


def _agree(label, grads, ref):
    """grads within PATH_RTOL of ref's max-abs, tensor by tensor; returns the worst ratio."""
    worst = 0.0
    for k, t in ref.items():
        scale = float(t.abs().max())
        err = float((grads[k] - t).abs().max())
        assert err <= PATH_RTOL * scale, (label, k, err, scale)
        worst = max(worst, err / max(scale, 1e-30))
    return worst


def _stream_ctx(dev):
    """A stream of its own, hence a rasterizer context of its own: the shapes used there have no history."""
    return torch.cuda.Stream(dev)


# ---------------------------------------------------------------------------------------------------------------------
# 1. every binning state of one shape
# ---------------------------------------------------------------------------------------------------------------------
def test_every_binning_state_backward_matches_oracle():
    """2 scenes x 3 views on a context of its own, walked through every binning state in turn; each call's backward
    against the oracle and against the exact path's."""
    from pf3plat_b200._capi import (GS_TUNE_FORCE_RADIX_BINNING, GS_TUNE_NO_SPECULATION, GS_TUNE_NO_STRATA,
                                    GS_TUNE_SEPARATE_EMIT)
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = (32, 48)
    scenes = [make_scene(2500, 3, *hw, seed=70 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=71)
    gref = ob.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    sequence = [("exact", GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", GS_TUNE_NO_STRATA | GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", GS_TUNE_NO_STRATA, 1), ("radix fallback", GS_TUNE_FORCE_RADIX_BINNING, 0)]
    stream = _stream_ctx(dev)
    states, first, worst = [], None, 0.0
    with torch.cuda.stream(stream):
        for label, tuning, want in sequence:
            out, grads = _run(_settings(dcams, hw, with_depth=True, tuning=tuning), ins, dL, dLd)
            st = last_stats(dev)
            states.append(st["speculative"])
            assert st["speculative"] == want, (label, st)
            assert st["overflow_redos"] == 0, (label, st)
            _check_all(label, out, grads, ob, gref)
            if first is None:
                first = (out, grads)
            else:
                for a, b in zip(out, first[0]):
                    assert torch.equal(a, b), label
                worst = max(worst, _agree(label, grads, first[1]))
        stream.synchronize()
    print(f"[regime] binning paths: S={ob.S} VPS={ob.VPS} P={ob.P}; speculative per call {states}; worst gradient "
          f"difference from the exact path {worst:.2e} of max-abs")


# ---------------------------------------------------------------------------------------------------------------------
# 2. per-tile depth strata
# ---------------------------------------------------------------------------------------------------------------------
def test_per_tile_strata_backward_matches_oracle():
    """The pixel-aligned cloud crowds each tile into one or two per-view strata: the per-view strata trial (call 2)
    overflows, is redone exactly, and from then on the shape is stratified on per-(view, tile) boundaries."""
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    sc = make_pixel_aligned_scene(128, 128, 3, seed=2)
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    stream = _stream_ctx(dev)
    states, redos = [], []
    with torch.cuda.stream(stream):
        for _ in range(5):
            _forward(bs, ins, grad=False)
            st = last_stats(dev)
            states.append(st["speculative"])
            redos.append(st["overflow_redos"])
        ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
        dL, dLd = _incoming(ob.V, hw, seed=72)
        gref = ob.backward(dL, dLd)
        out, grads = _run(bs, ins, dL, dLd)
        st = last_stats(dev)
        stream.synchronize()
    print(f"[regime] per-tile strata: P={ob.P}, speculative per call {states + [st['speculative']]}, overflow redos "
          f"after each call {redos + [st['overflow_redos']]}")
    # call 1 exact; call 2 the per-view trial, overflowed and redone; later calls stratified on per-tile boundaries
    assert states[0] == 0 and redos[0] == 0
    assert states[1] == 0 and redos[1] == 1
    assert states[2:] == [2, 2, 2] and redos[2:] == [1, 1, 1]
    assert st["speculative"] == 2 and st["overflow_redos"] == 1
    _check_all("per-tile strata", [o.detach() for o in out], grads, ob, gref)


# ---------------------------------------------------------------------------------------------------------------------
# 3. overflow and exact redo
# ---------------------------------------------------------------------------------------------------------------------
def _squeezed(sc, f):
    """The same cloud (same P, so the same shape to the library) with its centres pulled towards the optical axis by f:
    about 1/f^2 times as many tile entries in the central tiles."""
    kw = dict(sc.__dict__)
    kw["means"] = sc.means * torch.tensor([f, f, 1.0])
    return type(sc)(**kw)


def test_overflow_redo_backward_matches_oracle():
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = (48, 64)
    sparse = make_scene(3000, 2, *hw, seed=73)
    dense = _squeezed(sparse, 0.63)                  # 2.5x the entries per central tile
    cams, ins_s = scene_batch_args([sparse])
    _, ins_d = scene_batch_args([dense])
    keep = ("means3D", "opacities", "shs", "cov3D_precomp")
    ins_s, ins_d = ({k: i[k] for k in keep} for i in (ins_s, ins_d))
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins_d)
    dL, dLd = _incoming(ob.V, hw, seed=74)
    gref = ob.backward(dL, dLd)
    stream = _stream_ctx(dev)
    with torch.cuda.stream(stream):
        states = []
        for _ in range(3):                           # exact, strata trial, stratified: capacities learned
            _forward(bs, ins_s, grad=False)
            states.append(last_stats(dev)["speculative"])
        before = last_stats(dev)
        out, grads = _run(bs, ins_d, dL, dLd)
        after = last_stats(dev)
        stream.synchronize()
    print(f"[regime] overflow: sparse calls speculative {states}, max tile list {before['max_tile_list']}; dense call "
          f"speculative {after['speculative']}, max tile list {after['max_tile_list']}, overflow redos "
          f"{before['overflow_redos']} -> {after['overflow_redos']}")
    assert states[-1] >= 1 and before["overflow_redos"] == 0
    assert after["overflow_redos"] == before["overflow_redos"] + 1 and after["speculative"] == 0
    assert after["max_tile_list"] >= 1.5 * before["max_tile_list"]
    _check_all("overflow redo", out, grads, ob, gref)


# ---------------------------------------------------------------------------------------------------------------------
# 4. tile lists longer than the shared-memory sort
# ---------------------------------------------------------------------------------------------------------------------
def _long_list_check(label, sc, seed, max_fragile_frac):
    from pf3plat_b200._capi import GS_TUNE_BWD_OCC4, GS_TUNE_BWD_V1
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs", "cov3D_precomp")}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    lists = [r.ranges[:, 1] - r.ranges[:, 0] for r in ob.views]
    for v, r in enumerate(ob.views):
        print(f"[regime] {label} view {v}: tile lists {lists[v].tolist()}, max n_contrib {r.n_contrib.max()}, "
              f"final_T >= {r.final_T.min():.3f}")
        assert r.n_contrib.max() > 8192 and lists[v].max() > 8192 and r.final_T.min() > 1e-3
    dL, dLd = _incoming(ob.V, hw, seed=seed)
    gref = ob.backward(dL, dLd)
    dcams = {k: v.to(dev) for k, v in cams.items()}
    grads0 = None
    for tuning, name in ((0, "default"), (GS_TUNE_BWD_OCC4, "bwd occ4"), (GS_TUNE_BWD_V1, "bwd v1")):
        out, grads = _run(_settings(dcams, hw, with_depth=True, tuning=tuning), ins, dL, dLd)
        st = last_stats(dev)
        assert st["max_tile_list"] > 8192 and st["speculative"] == 0, st     # the radix fallback
        _check_all(f"{label} {name}", out, grads, ob, gref, max_fragile_frac=max_fragile_frac)
        if grads0 is None:
            grads0 = grads
        else:
            _agree(f"{label} {name}", grads, grads0)
    return lists


def test_long_tile_list_backward_matches_fp64_oracle():
    """One 16 x 16 tile, 10 000 faint splats: every pixel's last contributor lies beyond list position 8192, so the
    backward walks about 40 batches of 256 entries per tile."""
    _long_list_check("long list 16x16", long_list_scene(10000, 1, 16, 16, seed=1), seed=75, max_fragile_frac=0.06)


def test_long_tile_list_multi_view_ragged_with_empty_tiles():
    """3 views of a 40 x 52 frame: 9000 faint splats packed into the first tile, 150 ordinary ones in the lower left;
    the right-hand tile columns are empty in every view."""
    sc = long_list_scene(9000, 3, 40, 52, box=(2.0, 2.0, 13.0, 13.0), n_sparse=150, sparse_box=(0.0, 18.0, 24.0, 39.0),
                         seed=2)
    lists = _long_list_check("long list 3 x 40x52", sc, seed=76, max_fragile_frac=0.03)
    assert all((n == 0).sum() >= 4 for n in lists)


# ---------------------------------------------------------------------------------------------------------------------
# 5. ragged frames
# ---------------------------------------------------------------------------------------------------------------------
RAGGED = [(37, 53), (17, 130), (100, 9), (5, 7), (1, 40), (33, 250)]


@pytest.mark.parametrize("hw", RAGGED, ids=[f"{h}x{w}" for h, w in RAGGED])
def test_ragged_frame_backward_matches_oracle_under_every_kernel(hw):
    from pf3plat_b200._capi import GS_TUNE_BWD_OCC4, GS_TUNE_BWD_V1, GS_TUNE_PBWD_2PHASE
    dev = _dev()
    H, W = hw
    sc = edge_straddle_scene(600, 120, 2, H, W, seed=77)
    cams, ins = scene_batch_args([sc])
    geometry = ("scales", "rotations") if H in (17, 1) else ("cov3D_precomp",)
    ins = {k: ins[k] for k in ("means3D", "opacities", "shs") + geometry}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=78)
    gref = ob.backward(dL, dLd)
    for v, r in enumerate(ob.views):
        counts = []
        for mask in (np.s_[:, W - 1], np.s_[H - 1, :]):
            m = np.zeros(hw, bool)
            m[mask] = True
            edge = edge_contributors(r, m)
            counts.append(int(edge.sum()))
            # the oracle gives every one of them gradient (from the edge pixels, at least)
            assert edge.sum() >= 5 and (np.abs(gref["opacities"][0, edge]) > 0).all()
        print(f"[regime] ragged {H}x{W} view {v}: partial warp column {W % 8} px, partial warp row {H % 4} px, partial "
              f"tile {W % 16}x{H % 16}; Gaussians composited into the last column {counts[0]}, into the last row "
              f"{counts[1]}")
    dcams = {k: v.to(dev) for k, v in cams.items()}
    for tuning, name in ((0, "default"), (GS_TUNE_BWD_OCC4, "bwd occ4"), (GS_TUNE_BWD_V1, "bwd v1"),
                         (GS_TUNE_PBWD_2PHASE, "2-phase preprocess bwd")):
        out, grads = _run(_settings(dcams, hw, with_depth=True, tuning=tuning), ins, dL, dLd)
        _check_all(f"ragged {H}x{W} {name}", out, grads, ob, gref)


# ---------------------------------------------------------------------------------------------------------------------
# 6. saved state across later calls on the same context
# ---------------------------------------------------------------------------------------------------------------------
def test_saved_state_survives_later_calls_on_the_context():
    """Forward A with grad; then, on the same context, a speculative forward + backward of the same shape on another
    cloud (B), an overflow redo of that shape, and forwards of five other shapes (more than the context's four shape
    slots: A's is evicted).  A's backward, run last, must match an isolated run of A and the oracle.  The backwards of A
    and B run in the opposite order from their forwards; a second pair (C, D) runs its backwards in forward order."""
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    hw = (40, 56)
    keep = ("means3D", "opacities", "shs", "cov3D_precomp")

    def batch(sc):
        cams, ins = scene_batch_args([sc])
        return {k: v.to(dev) for k, v in cams.items()}, cams, {k: ins[k] for k in keep}

    sc_a = make_scene(2000, 2, *hw, seed=80)
    dcams, cams, ins_a = batch(sc_a)
    _, _, ins_b = batch(make_scene(2000, 2, *hw, seed=81))
    _, _, ins_dense = batch(_squeezed(sc_a, 0.6))
    bs = _settings(dcams, hw, with_depth=True)
    ob_a = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins_a)
    ob_b = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins_b)
    dL_a, dLd_a = _incoming(2, hw, seed=82)
    dL_b, dLd_b = _incoming(2, hw, seed=83)

    iso_stream = _stream_ctx(dev)
    with torch.cuda.stream(iso_stream):
        iso_out, iso = _run(bs, ins_a, dL_a, dLd_a)
        iso_stream.synchronize()

    others = [(24, 24), (16, 80), (56, 40), (33, 17), (8, 8)]
    stream = _stream_ctx(dev)
    log = []
    with torch.cuda.stream(stream):
        _forward(bs, ins_a, grad=False)                                      # the shape's history: exact
        out_a, leaves_a = _forward(bs, ins_a)                                # A: the strata trial
        log.append(("A", last_stats(dev)["speculative"]))
        out_b, leaves_b = _forward(bs, ins_b)                                # B: stratified
        st_b = last_stats(dev)
        log.append(("B", st_b["speculative"]))
        grads_b = _backward(out_b, leaves_b, dL_b, dLd_b)
        _forward(bs, ins_dense, grad=False)                                  # overflow, exact redo
        st_dense = last_stats(dev)
        log.append(("dense", st_dense["speculative"]))
        for ohw in others:                                                   # evict A's shape slot
            oc, _, oi = batch(make_scene(300, 1, *ohw, seed=84))
            _forward(_settings(oc, ohw, with_depth=True), oi, grad=False)
            _forward(_settings(oc, ohw, with_depth=True), oi, grad=False)
        _forward(bs, ins_a, grad=False)                                      # A's shape again: a fresh slot
        log.append(("A again", last_stats(dev)["speculative"]))
        grads_a = _backward(out_a, leaves_a, dL_a, dLd_a)
        # C and D: two shapes, backwards in the order of their forwards
        sc_c, sc_d = make_scene(1500, 2, 24, 40, seed=85), make_scene(1500, 3, 36, 20, seed=86)
        cc, cc_cpu, ins_c = batch(sc_c)
        cd, cd_cpu, ins_d = batch(sc_d)
        out_c, leaves_c = _forward(_settings(cc, (24, 40), with_depth=True), ins_c)
        out_d, leaves_d = _forward(_settings(cd, (36, 20), with_depth=True), ins_d)
        dL_c, dLd_c = _incoming(2, (24, 40), seed=87)
        dL_d, dLd_d = _incoming(3, (36, 20), seed=88)
        grads_c = _backward(out_c, leaves_c, dL_c, dLd_c)
        grads_d = _backward(out_d, leaves_d, dL_d, dLd_d)
        stream.synchronize()
    print(f"[regime] saved state: speculative per call {log}; overflow redos {st_dense['overflow_redos']}; "
          f"{len(others)} other shapes in between")
    assert log[0][1] == 2 and log[1][1] == 2                 # A and B on the speculative (stratified) path
    assert st_dense["overflow_redos"] == 1 and st_dense["speculative"] == 0
    assert log[3][1] == 0                                   # A's slot was evicted: the shape starts over
    worst = _agree("A after later calls vs isolated A", grads_a, iso)
    print(f"[regime] saved state: A's gradients differ from an isolated run by {worst:.2e} of max-abs")
    for a, b in zip(out_a, iso_out):
        assert torch.equal(a.detach(), b)
    _check_all("saved A", [o.detach() for o in out_a], grads_a, ob_a, ob_a.backward(dL_a, dLd_a))
    _check_all("saved B", [o.detach() for o in out_b], grads_b, ob_b, ob_b.backward(dL_b, dLd_b))
    for name, out, grads, c, ins, hw_, dL, dLd in (("C", out_c, grads_c, cc_cpu, ins_c, (24, 40), dL_c, dLd_c),
                                                  ("D", out_d, grads_d, cd_cpu, ins_d, (36, 20), dL_d, dLd_d)):
        ob = oracle_batch(_settings(c, hw_, with_depth=True), dtype=np.float64, **ins)
        _check_all(f"saved {name}", [o.detach() for o in out], grads, ob, ob.backward(dL, dLd))
