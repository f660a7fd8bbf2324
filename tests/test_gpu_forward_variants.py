"""GPU parity of the forward's kernel variants (include/gsplat_b200.h, GS_TUNE_*) against the default build and the fp64
oracle: the persistent warp-specialised compositor (GS_TUNE_FWD_WS) with many tiles per CTA, early stops and partial
tiles in one launch, on every tile-list layout and through gs_render_host; the 16-byte SH staging of k_preprocess on
device-resident SH (GS_TUNE_PRE_SH_RAW16) where a block ends inside a 16-byte piece, and for several scenes; per-tile
strata switched off (GS_TUNE_NO_TILE_STRATA); the merge-sort stratum sort (GS_TUNE_STRATA_MERGE_SORT) and the
register-bounded preprocess (GS_TUNE_PRE_OCC6).

Method: the default build and each variant run the same call sequence, each on a stream of its own (hence a rasterizer
context of its own), under torch.use_deterministic_algorithms(True).  Every output (color, radii, depth) and every
gradient of the variant must be torch.equal to the default's -- the deterministic backward reads the final_T and
n_contrib the forward saved, so this pins them bit for bit -- and the variant's own outputs and gradients must pass the
fp64 batched oracle (tests/batch_oracle.py) at tests/util.py's criteria.  Every test asserts which binning path ran
(`last_stats()`) and prints its counts in "[regime]" lines.

Every shape here (views, tiles, Gaussians per scene, scenes) is one no other test uses: the stream pool hands out the
same few streams again, and a context keyed to a reused stream must not already know the shape's speculation state."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200.synthetic import Scene, make_pixel_aligned_scene, make_scene
from tests.batch_oracle import oracle_batch, scene_batch_args
from tests.regimes import TANFOV, edge_straddle_scene, long_list_scene, opaque_stack_scene
from tests.test_gpu_backward_paths import _incoming, _squeezed
from tests.test_gpu_depth_chain import _leaves
from tests.test_gpu_regimes import _check_grads, _check_images, _check_radii, _settings

pytestmark = pytest.mark.gpu

# k_composite_fwd_ws (gs_composite_fwd.cu): 8 consumer warps + 1 producer warp, a ring of CP_STAGES stages of CP_BATCH
CP_THREADS, CP_STAGES, CP_BATCH = 288, 4, 128
MAX_CTAS_PER_SM = 2048 // CP_THREADS          # 7: the thread limit of an SM, whatever the registers allow
KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")
FIELDS = ("means", "covariances", "harmonics", "opacities", "scales", "rotations")


def _dev():
    assert torch.cuda.is_available(), "GPU test needs CUDA"
    return torch.device("cuda:0")


def _tunings():
    from pf3plat_b200 import _capi
    return _capi


# ---------------------------------------------------------------------------------------------------------------------
# running one call sequence per variant, each on a context of its own
# ---------------------------------------------------------------------------------------------------------------------
def _call(bs, ins, incoming):
    """One rasterize_batch call; with `incoming` = (dL/dcolor, dL/ddepth) also the backward (means2D included).
    Returns (outputs, {name: grad} or None, last_stats() of the forward)."""
    from pf3plat_b200.rasterizer import last_stats, rasterize_batch
    dev = bs.viewmatrix.device
    if incoming is None:
        with torch.no_grad():
            out = rasterize_batch(bs, **{k: v.to(dev) for k, v in ins.items()})
        return [o.clone() for o in out], None, last_stats(dev)
    leaves = _leaves(ins, dev, bs.viewmatrix.shape[0])
    out = rasterize_batch(bs, **leaves)
    st = last_stats(dev)
    dL, dLd = incoming
    outs, grads = [out[0]], [torch.as_tensor(dL, device=dev)]
    if bs.with_depth:
        outs.append(out[2])
        grads.append(torch.as_tensor(dLd, device=dev))
    torch.autograd.backward(outs, grads)
    return [o.detach() for o in out], {k: t.grad.detach().clone() for k, t in leaves.items()}, st


def _on_own_streams(dev, calls, tunings):
    """For each extra tuning in `tunings` (0: the default build), the call sequence `calls` -- (bs, ins, incoming or
    None) -- with bs.tuning | extra, on a stream of its own, under deterministic algorithms.
    Returns {extra: [(outputs, grads, stats) per call]}."""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    res = {}
    try:
        for extra in tunings:
            stream = torch.cuda.Stream(dev)
            with torch.cuda.stream(stream):
                res[extra] = [_call(bs._replace(tuning=bs.tuning | extra), ins, inc) for bs, ins, inc in calls]
                stream.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    return res


def _first_difference(a, b):
    idx = (a != b).nonzero()
    return tuple(int(i) for i in idx[0]) if len(idx) else None


def _identical(label, run, ref):
    """Outputs and gradients of `run` bit-identical to those of `ref`."""
    (out, grads, _), (out0, grads0, _) = run, ref
    assert len(out) == len(out0)
    for name, a, b in zip(("color", "radii", "depth"), out, out0):
        assert torch.equal(a, b), (f"{label}: {name} differs, first at {_first_difference(a, b)} "
                                   f"(max |diff| {float((a.double() - b.double()).abs().max()):.3e})")
    assert (grads is None) == (grads0 is None)
    if grads0 is not None:
        assert set(grads) == set(grads0)
        for k in grads0:
            assert torch.equal(grads[k], grads0[k]), (f"{label}: dL/d{k} differs, first at "
                                                      f"{_first_difference(grads[k], grads0[k])}")


def _oracle_check(label, run, ob, gref, aff, max_fragile_frac=0.03):
    out, grads, _ = run
    _check_images(out[0], ob, label, max_fragile_frac=max_fragile_frac, depth=out[2] if len(out) > 2 else None)
    _check_radii(out[1], ob, label)
    if grads is not None:
        assert set(grads) == {k for k in gref if gref[k] is not None}
        _check_grads(label, grads, gref, aff, ob.VPS)


def _name(extra):
    c = _tunings()
    names = {0: "default", c.GS_TUNE_FWD_WS: "fwd ws", c.GS_TUNE_STRATA_MERGE_SORT: "strata merge sort",
             c.GS_TUNE_PRE_OCC6: "pre occ6", c.GS_TUNE_NO_TILE_STRATA: "no tile strata",
             c.GS_TUNE_PRE_SH_RAW16: "pre sh raw16", c.GS_TUNE_NO_SPECULATION: "exact"}
    return names[extra]


def _with_culled(sc: Scene, k: int) -> Scene:
    """sc plus k Gaussians behind every camera (culled in every view: no pixel, radius or gradient changes), so that the
    shape -- Gaussians per scene -- is one no other test renders."""
    means = torch.zeros(k, 3)
    means[:, 2] = -1.0
    cov = torch.eye(3).repeat(k, 1, 1) * 1e-4
    add = {"means": means, "covariances": cov, "harmonics": torch.zeros(k, *sc.harmonics.shape[1:]),
           "opacities": torch.full((k,), 0.5), "scales": torch.full((k, 3), 1e-2),
           "rotations": torch.tensor([[1.0, 0, 0, 0]]).repeat(k, 1)}
    kw = dict(sc.__dict__)
    for n in FIELDS:
        kw[n] = torch.cat([kw[n], add[n]]).contiguous()
    return Scene(**kw)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the persistent loop: several tiles per CTA, early stops, empty and partial tiles in one launch
# ---------------------------------------------------------------------------------------------------------------------
WS_HW, WS_VPS = (72, 100), 19        # 5 x 7 tiles per view, the last row (8 px) and column (4 px) partial


def _opaque_and_edge_scene(seed, n_keep=None):
    """26 opaque sheets (opaque_stack_scene, 24 x 24 Gaussians each) kept left of pixel column 30 in view 0 -- tile
    columns 0-1 hold lists of 700-1800 entries whose pixels all stop within the first few hundred --, tile columns 3-4
    empty, and 200 edge_straddle_scene splats on the last row and column.  The scene's last n_keep Gaussians (the
    deepest sheets' first ones are dropped) so that several scenes share P."""
    h, w = WS_HW
    st = opaque_stack_scene(26, 24, WS_VPS, h, w, seed=seed)
    u = (st.means[:, 0] / st.means[:, 2] / TANFOV + 1) * (w / 2) - 0.5
    keep = u < 30.0
    ed = edge_straddle_scene(0, 200, WS_VPS, h, w, seed=seed + 1)
    kw = dict(st.__dict__)
    for n in FIELDS:
        kw[n] = torch.cat([getattr(st, n)[keep], getattr(ed, n)]).contiguous()
    sc = Scene(**kw)
    if n_keep is not None:
        kw = dict(sc.__dict__)
        for n in FIELDS:
            kw[n] = kw[n][-n_keep:].contiguous()
        sc = Scene(**kw)
    return sc


def _many_tiles_batch():
    """2 scenes x 19 views of 72 x 100: 1330 work items.  P is a multiple of 4, so that gs_render_host's zero-copy SH feed
    takes two scenes (P * M * 12 % 16 == 0)."""
    n = min(_opaque_and_edge_scene(s).means.shape[0] for s in (200, 210)) // 4 * 4
    scenes = [_opaque_and_edge_scene(s, n) for s in (200, 210)]
    cams, ins = scene_batch_args(scenes)
    return cams, {k: ins[k] for k in KEEP}, WS_HW


def _early_stop_tiles(orc):
    """bool[tiles]: tiles on which k_composite_fwd_ws's producer is certain to stop before the end of the list.  Every
    pixel of such a tile stops its walk at a Gaussian (the first one after its last contributor that reaches it: it would
    take T below 1e-4); the consumer warp whose pixels stop last reports in the batch k of that Gaussian; the producer
    waits for every consumer's release of batch b - CP_STAGES before it fills batch b, so it sees the report by batch
    k + CP_STAGES at the latest -- and stops there if the list has more batches than that."""
    H, W = orc.H, orc.W
    gx = (W + 15) // 16
    xy, co, pl, rg = orc.xy.astype(np.float64), orc.conic_opacity.astype(np.float64), orc.point_list, orc.ranges
    out = np.zeros(rg.shape[0], bool)
    for t in range(rg.shape[0]):
        s, e = int(rg[t, 0]), int(rg[t, 1])
        nb = -(-(e - s) // CP_BATCH)
        if nb <= CP_STAGES:
            continue
        ids = pl[s:s + (nb - CP_STAGES) * CP_BATCH]     # the stopping Gaussians must lie in these batches
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        dx, dy = xy[ids, 0:1] - xs[None], xy[ids, 1:2] - ys[None]
        power = -0.5 * (co[ids, 0:1] * dx * dx + co[ids, 2:3] * dy * dy) - co[ids, 1:2] * dx * dy
        a = co[ids, 3:4] * np.exp(np.minimum(power, 0.0))
        reach = (power <= 0) & (a >= 1 / 255)
        later = np.arange(len(ids))[:, None] >= orc.n_contrib[ys, xs][None]
        out[t] = (reach & later).any(axis=0).all()
    return out


@pytest.mark.parametrize("with_depth", [True, False], ids=["depth", "no_depth"])
def test_ws_persistent_loop_many_tiles_per_cta(with_depth):
    c = _tunings()
    dev = _dev()
    cams, ins, hw = _many_tiles_batch()
    H, W = hw
    V = cams["viewmatrix"].shape[0]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    items = V * gx * gy
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    # at most MAX_CTAS_PER_SM CTAs of 288 threads are resident per SM: the persistent grid is smaller than the work
    assert items >= 8 * sms and items > MAX_CTAS_PER_SM * sms, (items, sms)
    ob = oracle_batch(_settings(cams, hw, with_depth=with_depth), dtype=np.float64, **ins)
    early = np.stack([_early_stop_tiles(r) for r in ob.views])
    lens = np.stack([r.ranges[:, 1] - r.ranges[:, 0] for r in ob.views])
    empty = lens == 0
    partial = np.zeros((gy, gx), bool)
    if W % 16:
        partial[:, -1] = True
    if H % 16:
        partial[-1, :] = True
    partial = np.broadcast_to(partial.reshape(-1), lens.shape)
    ordinary = ~early & ~empty
    print(f"[regime] ws persistent loop ({'depth' if with_depth else 'no depth'}): S={ob.S} VPS={ob.VPS} P={ob.P} "
          f"{H}x{W}; work items {items} on {sms} SMs (<= {MAX_CTAS_PER_SM * sms} resident CTAs: >= "
          f"{items / (MAX_CTAS_PER_SM * sms):.2f} items per CTA); early-stop tiles {int(early.sum())} (partial "
          f"{int((early & partial).sum())}), empty {int(empty.sum())}, ordinary {int(ordinary.sum())}, partial "
          f"{int(partial.sum())}; longest list {int(lens.max())}")
    assert early.sum() >= 0.2 * items and (early & partial).sum() >= V
    assert empty.sum() >= 0.1 * items and ordinary.sum() >= 0.2 * items
    assert (lens[early] > CP_STAGES * CP_BATCH).all()
    # interleaved: every view has tiles of all three kinds
    assert early.any(axis=1).all() and empty.any(axis=1).all() and ordinary.any(axis=1).all()
    dL, dLd = _incoming(V, hw, seed=140)
    gref = ob.backward(dL, dLd if with_depth else None)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    runs = _on_own_streams(dev, [(_settings(dcams, hw, with_depth=with_depth), ins, (dL, dLd))],
                           (0, c.GS_TUNE_FWD_WS))
    for extra, (run,) in runs.items():
        st = run[2]
        assert st["speculative"] == 0 and st["overflow_redos"] == 0, st        # exact capacities, shared-memory sort
        assert CP_STAGES * CP_BATCH < st["max_tile_list"] <= 8192, st
    ws = runs[c.GS_TUNE_FWD_WS][0]
    _identical("ws persistent loop", ws, runs[0][0])
    _oracle_check("ws persistent loop", ws, ob, gref, aff)


# ---------------------------------------------------------------------------------------------------------------------
# 2. every tile-list layout, under the forward compositor, stratum-sort and preprocess variants
# ---------------------------------------------------------------------------------------------------------------------
def _layout_variants():
    c = _tunings()
    return (c.GS_TUNE_FWD_WS, c.GS_TUNE_STRATA_MERGE_SORT, c.GS_TUNE_PRE_OCC6)


def _check_sequence(label, runs, ob, gref, aff, variants, max_fragile_frac=0.03):
    """Every call of every variant bit-identical to the default's, and against the oracle where it has gradients."""
    for extra in variants:
        for k, (run, ref) in enumerate(zip(runs[extra], runs[0])):
            name = f"{label} call {k} {_name(extra)}"
            _identical(name, run, ref)
            if run[1] is not None:
                _oracle_check(name, run, ob, gref, aff, max_fragile_frac)


def test_every_binning_state_under_forward_variants():
    """2 scenes x 3 views walked through every binning state in turn (the sequence of
    test_every_binning_state_backward_matches_oracle): exact, per-view strata trial, stratified, stratified with
    k_emit_buckets, exact re-learning unstratified, whole-tile speculative, radix fallback."""
    c = _tunings()
    dev = _dev()
    hw = (32, 48)
    scenes = [make_scene(2613, 3, *hw, seed=150 + k) for k in range(2)]
    cams, ins = scene_batch_args(scenes, near=1.0 / np.tile(np.linspace(0.8, 1.25, 3), 2))
    ins = {k: ins[k] for k in KEEP}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=151)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    sequence = [("exact", c.GS_TUNE_NO_SPECULATION, 0), ("per-view strata trial", 0, 2), ("stratified", 0, 2),
                ("stratified, k_emit_buckets", c.GS_TUNE_SEPARATE_EMIT, 2),
                ("exact, re-learn unstratified", c.GS_TUNE_NO_STRATA | c.GS_TUNE_NO_SPECULATION, 0),
                ("whole-tile", c.GS_TUNE_NO_STRATA, 1), ("radix fallback", c.GS_TUNE_FORCE_RADIX_BINNING, 0)]
    calls = [(_settings(dcams, hw, with_depth=True, tuning=t), ins, (dL, dLd)) for _, t, _ in sequence]
    variants = _layout_variants()
    runs = _on_own_streams(dev, calls, (0,) + variants)
    for extra, rs in runs.items():
        states = [r[2]["speculative"] for r in rs]
        print(f"[regime] binning states, {_name(extra)}: speculative per call {states}; overflow redos "
              f"{[r[2]['overflow_redos'] for r in rs]}")
        assert states == [want for _, _, want in sequence], (extra, states)
        assert all(r[2]["overflow_redos"] == 0 for r in rs), extra
    _check_sequence("binning states", runs, ob, gref, aff, variants)


def test_overflow_redo_under_forward_variants():
    """Three calls of a sparse cloud teach the shape its capacities (the last one stratified); the same shape with its
    centres squeezed to the middle overflows them.  The compositor runs on the overflowed list before the verdict is
    read, then the call is redone exactly."""
    dev = _dev()
    hw = (48, 64)
    sparse = make_scene(3011, 2, *hw, seed=152)
    dense = _squeezed(sparse, 0.63)
    cams, ins_s = scene_batch_args([sparse])
    _, ins_d = scene_batch_args([dense])
    ins_s, ins_d = ({k: i[k] for k in KEEP} for i in (ins_s, ins_d))
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins_d)
    dL, dLd = _incoming(ob.V, hw, seed=153)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    calls = [(bs, ins_s, None)] * 3 + [(bs, ins_d, (dL, dLd))]
    variants = _layout_variants()
    runs = _on_own_streams(dev, calls, (0,) + variants)
    for extra, rs in runs.items():
        st = [r[2] for r in rs]
        print(f"[regime] overflow, {_name(extra)}: speculative per call {[s['speculative'] for s in st]}, overflow "
              f"redos {[s['overflow_redos'] for s in st]}, max tile list {[s['max_tile_list'] for s in st]}")
        assert [s["speculative"] for s in st] == [0, 2, 2, 0], extra
        assert [s["overflow_redos"] for s in st] == [0, 0, 0, 1], extra
        assert st[3]["max_tile_list"] >= 1.5 * st[2]["max_tile_list"]
    _check_sequence("overflow redo", runs, ob, gref, aff, variants)


def test_long_tile_list_under_forward_variants():
    """3 views of 40 x 52: 9300 faint splats in the first tile (most of its pixels' last contributors beyond list
    position 8192), 170 ordinary ones in the lower left, the right-hand tile columns empty.  Lists this long take the radix
    fallback."""
    c = _tunings()
    dev = _dev()
    hw = (40, 52)
    sc = long_list_scene(9300, 3, *hw, box=(2.0, 2.0, 13.0, 13.0), n_sparse=170, sparse_box=(0.0, 18.0, 24.0, 39.0),
                         seed=154)
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    for v, r in enumerate(ob.views):
        lens = r.ranges[:, 1] - r.ranges[:, 0]
        t0 = r.n_contrib[:16, :16]
        print(f"[regime] long list view {v}: tile lists {lens.tolist()}, first tile's pixels with n_contrib > 8192 "
              f"{(t0 > 8192).mean():.1%} (max {t0.max()})")
        assert lens.max() > 8192 and (t0 > 8192).mean() >= 0.5 and (lens == 0).sum() >= 4
    dL, dLd = _incoming(ob.V, hw, seed=155)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    variants = (c.GS_TUNE_FWD_WS, c.GS_TUNE_PRE_OCC6)
    runs = _on_own_streams(dev, [(_settings(dcams, hw, with_depth=True), ins, (dL, dLd))], (0,) + variants)
    for extra, (run,) in runs.items():
        st = run[2]
        assert st["speculative"] == 0 and st["max_tile_list"] > 8192, (extra, st)     # the radix fallback
    _check_sequence("long list", runs, ob, gref, aff, variants, max_fragile_frac=0.03)


def test_pixel_aligned_strata_under_forward_variants():
    """The pixel-aligned cloud: the per-view strata trial (call 2) overflows and is redone exactly; by default the shape
    then moves to per-(view, tile) strata.  With GS_TUNE_NO_TILE_STRATA the trial's overflow sends it to whole-tile sorts
    for good.  Every call of every variant gives the exact path's bytes; the last call's gradients are bit-identical."""
    c = _tunings()
    dev = _dev()
    sc = _with_culled(make_pixel_aligned_scene(128, 128, 3, seed=2), 5)
    hw = sc.image_shape
    cams, ins = scene_batch_args([sc])
    ins = {k: ins[k] for k in KEEP}
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=156)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    calls = [(bs, ins, None)] * 5 + [(bs, ins, (dL, dLd))]
    variants = _layout_variants() + (c.GS_TUNE_NO_TILE_STRATA,)
    runs = _on_own_streams(dev, calls, (0,) + variants)
    exact = _on_own_streams(dev, [(bs, ins, None), (bs, ins, (dL, dLd))], (c.GS_TUNE_NO_SPECULATION,))
    exact = exact[c.GS_TUNE_NO_SPECULATION]
    for extra, rs in runs.items():
        states = [r[2]["speculative"] for r in rs]
        redos = [r[2]["overflow_redos"] for r in rs]
        print(f"[regime] pixel-aligned, {_name(extra)}: P={ob.P}, speculative per call {states}, overflow redos {redos}")
        # call 1 exact; call 2 the per-view trial, overflowed and redone exactly; then per-tile strata -- or, with the
        # knob, whole-tile sorts from then on
        want = 1 if extra == c.GS_TUNE_NO_TILE_STRATA else 2
        assert states == [0, 0] + [want] * 4 and redos == [0] + [1] * 5, (extra, states, redos)
        for k, run in enumerate(rs):
            _identical(f"pixel-aligned call {k} {_name(extra)} vs exact", run, exact[0 if run[1] is None else 1])
    _check_sequence("pixel-aligned", runs, ob, gref, aff, variants)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the warp-specialised compositor through gs_render_host
# ---------------------------------------------------------------------------------------------------------------------
def test_ws_through_host_entry():
    """Case 1's batch through gs_render_host with GS_TUNE_FWD_WS: a pinned feed (the SH block pulled zero-copy by
    k_sh_colour on a second stream), a pageable one (copied) and a pinned one whose images the compositor writes straight
    into the caller's buffers (GS_TUNE_DIRECT_OUTPUT).  Each feed twice, on one context: the shape's first call is exact,
    the later ones are stratified.  Every byte equals the device entry's default output."""
    from pf3plat_b200 import _capi, rasterizer
    from pf3plat_b200.rasterizer import last_stats
    dev = _dev()
    cams, ins, hw = _many_tiles_batch()
    S, P, M = ins["means3D"].shape[0], ins["means3D"].shape[1], ins["shs"].shape[2]
    V = cams["viewmatrix"].shape[0]
    assert M == 25 and S == 2 and (P * M * 12) % 16 == 0           # the zero-copy feed takes both scenes
    dcams = {k: v.to(dev) for k, v in cams.items()}
    ref = _on_own_streams(dev, [(_settings(dcams, hw, with_depth=True), ins, None)], (0,))[0][0][0]
    ref = [t.cpu() for t in ref]

    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree = P, S, V, M, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    cfg.flags = _capi.GS_FLAG_DEPTH
    stream = torch.cuda.Stream(dev)
    states = {}
    with torch.cuda.stream(stream):
        ctx = rasterizer.current_context(dev)
        for label, pinned, tuning in (("pinned", True, _capi.GS_TUNE_FWD_WS), ("pageable", False, _capi.GS_TUNE_FWD_WS),
                                      ("pinned, direct output", True, _capi.GS_TUNE_FWD_WS | _capi.GS_TUNE_DIRECT_OUTPUT)):
            mem = (lambda t: t.pin_memory()) if pinned else (lambda t: t.clone())
            host = {k: mem(v.contiguous().float()) for k, v in {**ins, **cams}.items()}
            for k in ("viewmatrix", "projmatrix", "campos", "bg", "tanfov", "view_scale"):
                setattr(cfg, k, host[k].data_ptr())
            gin = _capi.GsInputs(means3D=host["means3D"].data_ptr(), opacities=host["opacities"].data_ptr(),
                                 shs=host["shs"].data_ptr(), cov3D_precomp=host["cov3D_precomp"].data_ptr())
            color, radii, depth = mem(torch.empty(V, 3, *hw)), mem(torch.empty(V, P, dtype=torch.int32)), mem(
                torch.empty(V, *hw))
            gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr(), depth=depth.data_ptr())
            cfg.tuning = tuning
            states[label] = []
            for _ in range(2):
                for t in (color, radii, depth):
                    t.zero_()
                _capi.check(_capi.lib().gs_render_host(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                       stream.cuda_stream))
                states[label].append(last_stats(dev)["speculative"])
                for name, a, b in zip(("color", "radii", "depth"), (color, radii, depth), ref):
                    assert torch.equal(a, b), f"host entry {label}: {name} differs, first at {_first_difference(a, b)}"
        stream.synchronize()
    print(f"[regime] ws through gs_render_host: S={S} P={P} M={M} (P*M*12 % 16 == 0: zero-copy feed), speculative per "
          f"call {states}")
    assert sum(states.values(), []) == [0, 2, 2, 2, 2, 2], states


# ---------------------------------------------------------------------------------------------------------------------
# 4. 16-byte SH staging on device-resident SH
# ---------------------------------------------------------------------------------------------------------------------
PRE_THREADS = 128                     # Gaussians per k_preprocess CTA


def _raw16_engages(S, P, M):
    """launch_preprocess's rule (gs_preprocess.cu): with GS_TUNE_PRE_SH_RAW16 and M > 16, the 16-byte pieces are staged
    if every CTA's block starts 16-byte aligned -- the first one's does (torch's allocator hands out 512-byte aligned
    blocks), and the first of scene s sits s * P * M * 12 bytes further; else the compacting 4-byte gather runs."""
    return M > 16 and (S == 1 or (P * M * 12) % 16 == 0)


RAW16_CASES = [(1, 3021), (2, 1500), (2, 1501)]


@pytest.mark.parametrize("S,P", RAW16_CASES, ids=[f"S{s}_P{p}" for s, p in RAW16_CASES])
def test_raw16_sh_staging_on_device_sh(S, P):
    c = _tunings()
    dev = _dev()
    hw = (40, 56)
    scenes = [make_scene(P, 2, *hw, seed=160 + k) for k in range(S)]
    cams, ins = scene_batch_args(scenes)
    ins = {k: ins[k] for k in KEEP}
    M = ins["shs"].shape[2]
    row_f, want_f = 3 * M, 3 * 16       # floats per row; the evaluated coefficients (bands 0-3) come first
    n = P % PRE_THREADS or PRE_THREADS  # the tail CTA's Gaussians
    nfl = n * row_f
    ragged = np.arange(nfl // 4 * 4, nfl)  # floats after the last whole 16-byte piece of its block
    engaged = _raw16_engages(S, P, M)
    print(f"[regime] raw16: S={S} P={P} M={M}; RAW16 {'engages' if engaged else 'falls back to the compacting gather'}; "
          f"tail CTA {n} Gaussians, n*3M % 4 = {nfl % 4}, columns of its ragged end {(ragged % row_f).tolist()}")
    assert M == 25 and engaged == {(1, 3021): True, (2, 1500): True, (2, 1501): False}[(S, P)]
    if S == 1:
        # the tail block ends inside a 16-byte piece; every wanted coefficient of its last row still sits in whole
        # pieces -- the 4-byte loop of the ragged end only sees columns beyond the evaluated ones
        assert nfl % 4 != 0 and (ragged % row_f >= want_f).all()
    ob = oracle_batch(_settings(cams, hw, with_depth=True), dtype=np.float64, **ins)
    dL, dLd = _incoming(ob.V, hw, seed=161)
    gref = ob.backward(dL, dLd)
    aff = ob.affected()
    dcams = {k: v.to(dev) for k, v in cams.items()}
    bs = _settings(dcams, hw, with_depth=True)
    # an exact call (counting preprocess), then the strata trial (preprocess appending to the buckets)
    runs = _on_own_streams(dev, [(bs, ins, (dL, dLd))] * 2, (0, c.GS_TUNE_PRE_SH_RAW16))
    for extra, rs in runs.items():
        assert [r[2]["speculative"] for r in rs] == [0, 2], extra
    _check_sequence(f"raw16 S={S} P={P}", runs, ob, gref, aff, (c.GS_TUNE_PRE_SH_RAW16,))
