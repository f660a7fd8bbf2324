"""GPU checks of the sync-free rasterizer path (DESIGN.md 5.18) past its first shapes, every test under poisoned
allocations.  The tile lists themselves are read back from the workspace and checked against a plain sort
(tests/sync_free_layout.py: check_lists), on scenes whose lists are designed (tests/regimes.py: designed_tiles):
  1. every size-class edge of the tile merge sort in one call -- 1, 1023/1024/1025, 2047/2048/2049, 4095/4096/4097,
     8191/8192 -- with and without an 8193-list; several long lists (k_tile_sort_long) of different lengths and depth
     patterns in one call; each depth pattern (random, equal, ulp, binades, reversed) on 8193-, 20000- and 3000-lists;
     indices on both sides of 2^24; lists that shift across the edges call by call on one workspace; a scene batch with
     an empty scene.  Each is bit-equal to the default path and to its radix binning, gradients included;
  2. every input form (scales + rotations, colours, a means2D sink, (S, P, 1) opacities, the depth's view-matrix
     gradient at each depth mode, a colour-only loss of a forward with depth and alpha) bit-equal to the default path,
     and all-NaN gradients one instance short of the capacity, inside guard bands;
  3. the tuning knobs the sync-free entries honour give the default path's result with the same knob; those they do
     not read change no bit; the status words over fitting and exceeded calls."""
import contextlib

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi
from pf3plat_b200.cameras import make_view_batch
from pf3plat_b200.rasterizer import BatchSettings, SyncFreeWorkspace, last_stats, rasterize_batch, \
    sync_free_workspace_bytes
from pf3plat_b200.synthetic import make_scene
from tests.poison import poisoned  # noqa: F401
from tests.regimes import DEPTH_PATTERNS, PARKED, SHIFT_CALLS, SHIFT_POOL, designed_cameras, designed_case, \
    designed_tiles
from tests.sync_free_layout import check_lists, read_lists

pytestmark = pytest.mark.gpu

RADIX = _capi.GS_TUNE_FORCE_RADIX_BINNING
ALL_FLAGS = dict(depth=True, alpha=True, deterministic=True, camera_grad=True)


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


class Batch:
    """cameras (ViewBatch), background, (near, far), operator inputs {name: (S, P, ...)}, image shape, and the designed
    per-tile lengths {(view, tile): n} of the batch's views when it was built from designed cells"""

    def __init__(self, vb, bg, nf, ins, hw, lengths=None):
        self.vb, self.bg, self.nf, self.ins, self.hw, self.lengths = vb, bg, nf, ins, hw, lengths

    def with_inputs(self, **kw):
        ins = {k: v for k, v in {**self.ins, **kw}.items() if v is not None}
        return Batch(self.vb, self.bg, self.nf, ins, self.hw, self.lengths)

    @property
    def D(self):
        return sum(self.lengths.values())


def _cameras(ext, intr, near, far, dev):
    vb = make_view_batch(ext.to(dev), intr.to(dev), near.to(dev), far.to(dev))
    return vb, torch.zeros(ext.shape[0], 3, device=dev), torch.stack([near, far], -1).to(dev)


def _designed_batch(scene_cells, h, w, views, dev, P=None, seed=0):
    """One scene per entry of scene_cells (a list of designed cells, or None: an empty scene), each with the views of
    designed_cameras(views); every scene padded to P Gaussians with splats parked in front of no camera."""
    parts = [designed_tiles(h, w, cells, seed=seed + k) if cells else None for k, cells in enumerate(scene_cells)]
    P = P or max([d.means.shape[0] for d in parts if d is not None] + [1])
    S = len(scene_cells)
    means = torch.tensor(PARKED).repeat(S, P, 1)
    scales = torch.full((S, P, 3), 1e-3)
    rot = torch.tensor([1.0, 0.0, 0.0, 0.0]).repeat(S, P, 1)
    cov6 = torch.tensor([1e-6, 0.0, 0.0, 1e-6, 0.0, 1e-6]).repeat(S, P, 1)
    opac = torch.full((S, P), 0.02)
    sh = torch.zeros(S, P, 1, 3)
    lengths = {}
    for k, d in enumerate(parts):
        if d is None:
            continue
        n = d.means.shape[0]
        means[k, :n], scales[k, :n], rot[k, :n], cov6[k, :n] = d.means, d.scales, d.rotations, d.cov6
        opac[k, :n], sh[k, :n] = d.opacities, d.sh
        lengths.update({(k * views + v, t): m for (v, t), m in d.lengths.items()})
    ext, intr, near, far, _ = designed_cameras(views)
    rep = lambda t: t.repeat(S, *([1] * (t.dim() - 1)))
    vb, bg, nf = _cameras(rep(ext), rep(intr), rep(near), rep(far), dev)
    ins = {"means3D": means.to(dev), "opacities": opac.to(dev), "shs": sh.to(dev), "cov3D_precomp": cov6.to(dev)}
    extra = {"scales": scales.to(dev), "rotations": rot.to(dev)}
    b = Batch(vb, bg, nf, ins, (h, w), lengths)
    b.extra = extra
    return b


def _case_batch(name, dev, **kw):
    h, w, views, cells = designed_case(name)
    return _designed_batch([cells], h, w, views, dev, **kw)


def _run(b: Batch, ws=None, *, depth_mode=None, alpha=False, degree=0, max_degree=4, cam=False, vz=False, tuning=0,
         loss_on=None, square=False, aa=False, seed=3):
    """One forward + backward of a fixed random linear loss (square: half the sum of squares) over the outputs named
    in loss_on (all of them by default); {name: tensor} of outputs and gradients.  cam: the full camera gradient;
    vz: a view matrix that requires grad without it (the depth channel's z column)."""
    (h, w), dev = b.hw, b.bg.device
    leaf = lambda t: t.detach().clone().requires_grad_(True)
    cams = {"viewmatrix": b.vb.viewmatrix, "projmatrix": b.vb.projmatrix, "campos": b.vb.campos, "tanfov": b.vb.tanfov}
    cams = {k: leaf(v) if (cam or (vz and k == "viewmatrix")) else v.detach() for k, v in cams.items()}
    bs = BatchSettings(image_height=h, image_width=w, bg=b.bg, sh_degree=degree, view_scale=b.vb.scale,
                       with_depth=depth_mode is not None, depth_mode=depth_mode or "depth",
                       depth_near_far=b.nf if depth_mode in ("relative_disparity", "log") else None, with_alpha=alpha,
                       antialiasing=aa, camera_gradients=cam, sh_eval_max_degree=max_degree, tuning=tuning, **cams)
    leaves = {k: leaf(v) for k, v in b.ins.items()}
    out = rasterize_batch(bs, **leaves, workspace=ws)
    g = torch.Generator(device=dev).manual_seed(seed)
    named = {"color": out[0], "radii": out[1]}
    if depth_mode is not None:
        named["depth"] = out[2]
    if alpha:
        named["alpha"] = out[-1]
    weight = (lambda t: 0.5 * t) if square else (lambda t: torch.rand(t.shape, generator=g, device=dev))
    loss = sum((t * weight(t)).sum() for k, t in named.items() if k != "radii" and (loss_on is None or k in loss_on))
    wrt = {**leaves, **{k: v for k, v in cams.items() if v.requires_grad}}
    if b.ins["means3D"].shape[1] > 0:
        grads = torch.autograd.grad(loss, list(wrt.values()))
        named.update({"d_" + k: gr for k, gr in zip(wrt, grads)})
    return {k: v.detach() for k, v in named.items()}


def _compare(a, b, exact_grads, label):
    assert a.keys() == b.keys(), (label, sorted(a), sorted(b))
    for k in a:
        if not k.startswith("d_") or exact_grads:
            assert torch.equal(a[k], b[k]), (label, k)
        else:   # float atomics: a different summation order
            scale = a[k].abs().max().clamp_min(1e-30)
            assert float((a[k] - b[k]).abs().max() / scale) < 1e-4, (label, k)


def _workspace(b: Batch, capacity, **kw):
    S, P = b.ins["means3D"].shape[:2]
    return SyncFreeWorkspace(b.bg.device, S, b.vb.viewmatrix.shape[0], P, b.hw, capacity, **kw)


def _designed_parity(b: Batch, ws=None, radix=True, **kw):
    """b on the default path (and on its radix binning) and on the sync-free path: bit-equal outputs and deterministic
    gradients; the workspace's lists pass check_lists with the designed lengths and D.  Returns the lists."""
    dev = b.bg.device
    kw = {"depth_mode": "depth", "alpha": True, **kw}
    with _deterministic():
        ref = _run(b, **kw)
        assert last_stats(dev)["num_rendered"] == b.D
        refs = [("default", ref)] + ([("radix", _run(b, tuning=RADIX, **kw))] if radix else [])
        ws = ws or _workspace(b, b.D + 17, **ALL_FLAGS)
        got = _run(b, ws, **kw)
    lists = check_lists(ws, got["radii"], b.lengths, b.D)   # first: a wrong order is named as such
    for label, r in refs:
        _compare(r, got, True, label)
    return lists


def _distinct(bits):
    return np.unique(bits).size


def _assert_regime(pattern, bits):
    """the device's depth words of one tile are in the regime the pattern claims"""
    if pattern == "equal":
        assert _distinct(bits) == 1
    elif pattern == "ulp":
        assert _distinct(bits) >= 256 and _distinct(bits >> 16) == 1, (_distinct(bits), _distinct(bits >> 16))
    elif pattern == "binades":
        assert all(_distinct((bits >> (8 * k)) & 255) > 1 for k in range(4))


# ---------------------------------------------------------------------------------------------------------------------
# 1. designed tile lists
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["class_edges", "class_edges_8193"])
def test_every_class_edge_in_one_call(poisoned, name):
    b = _case_batch(name, _dev())
    lists = _designed_parity(b)
    assert lists.status["max_list"] == (8193 if name.endswith("8193") else 8192)


def test_several_long_lists_in_one_call(poisoned):
    b = _case_batch("long_lists", _dev())
    lists = _designed_parity(b)
    h, w, views, cells = designed_case("long_lists")
    gx = -(-w // 16)
    for v, tx, ty, n, pattern in cells:
        idx, bits = lists.tile_entries(v, ty * gx + tx)
        assert idx.shape[0] == n
        _assert_regime(pattern, bits)


@pytest.mark.parametrize("pattern", DEPTH_PATTERNS)
def test_each_depth_pattern(poisoned, pattern):
    b = _case_batch("pattern_" + pattern, _dev())
    lists = _designed_parity(b)
    for (v, t), n in b.lengths.items():
        idx, bits = lists.tile_entries(v, t)
        assert idx.shape[0] == n
        _assert_regime(pattern, bits)
        if pattern == "reversed":   # depth falls as the index rises: the sorted list is the indices backwards
            assert (np.diff(idx.astype(np.int64)) < 0).all()


def test_indices_on_both_sides_of_2_to_the_24(poisoned):
    """P = 2^24 + 8192 Gaussians in one view at degree 0, all but 10096 parked behind the camera; those 10096 form one
    list (k_tile_sort_long), at indices 2^24 - 4096 .. 2^24 + 5999, so the index's top digit varies.  Default path,
    radix binning and sync-free path with deterministic gradients together stay below 20 GB of device memory
    (asserted)."""
    dev = _dev()
    h, w, views, cells = designed_case("index_digit3")
    d = designed_tiles(h, w, cells)
    n, P = d.means.shape[0], (1 << 24) + 8192
    idx = torch.arange((1 << 24) - 4096, (1 << 24) - 4096 + n, device=dev)
    means = torch.tensor(PARKED, device=dev).repeat(1, P, 1)
    cov6 = torch.tensor([1e-6, 0.0, 0.0, 1e-6, 0.0, 1e-6], device=dev).repeat(1, P, 1)
    opac = torch.full((1, P), 0.02, device=dev)
    sh = torch.zeros(1, P, 1, 3, device=dev)
    means[0, idx], cov6[0, idx], opac[0, idx], sh[0, idx] = (d.means.to(dev), d.cov6.to(dev), d.opacities.to(dev),
                                                              d.sh.to(dev))
    ext, intr, near, far, _ = designed_cameras(1)
    vb, bg, nf = _cameras(ext, intr, near, far, dev)
    b = Batch(vb, bg, nf, {"means3D": means, "opacities": opac, "shs": sh, "cov3D_precomp": cov6}, (h, w),
              {(0, cells[0][2] * (w // 16) + cells[0][1]): n})
    torch.cuda.reset_peak_memory_stats(dev)
    lists = _designed_parity(b, cam=False)
    peak = torch.cuda.max_memory_allocated(dev)
    assert peak < 20 << 30, peak
    top = lists.index >> 24
    assert (top == 0).sum() == 4096 and (top == 1).sum() == n - 4096


def test_lists_shifting_across_the_edges_on_one_workspace(poisoned):
    """12 eager calls on one workspace whose designed lists move across 1024, 2048, 4096 and 8192 and back; the
    third needs 25000 instances of a capacity of 24800.  Every call matches a default call of the same cloud."""
    dev = _dev()
    h, w, views, _ = designed_case("shifting")
    full = _designed_batch([list(SHIFT_POOL)], h, w, views, dev)
    P = full.ins["means3D"].shape[1]
    cap = 24800
    ws = _workspace(full, cap, **ALL_FLAGS)
    gx = -(-w // 16)
    starts = np.cumsum([0] + [c[3] for c in SHIFT_POOL])
    most = 0
    kw = dict(depth_mode="depth", alpha=True)
    for call, ks in enumerate(SHIFT_CALLS):
        assert all(k <= c[3] for k, c in zip(ks, SHIFT_POOL)), call
        keep = torch.zeros(P, dtype=torch.bool)
        for s, k in zip(starts, ks):
            keep[s:s + k] = True
        means = torch.where(keep.to(dev)[None, :, None], full.ins["means3D"], torch.tensor(PARKED, device=dev))
        b = full.with_inputs(means3D=means)
        b.lengths = {(c[0], c[2] * gx + c[1]): k for c, k in zip(SHIFT_POOL, ks) if k}
        with _deterministic():
            ref = _run(b, **kw)
            got = _run(b, ws, **kw)
        most = max(most, b.D)
        lists = check_lists(ws, got["radii"], b.lengths, b.D)
        assert torch.equal(ref["radii"], got["radii"]), call
        if b.D > cap:
            assert lists.status["verdict"] == 1
            for k, t in got.items():
                if k != "radii":
                    assert torch.isnan(t).all(), (call, k)
        else:
            _compare(ref, got, True, f"call {call}")
        assert (lists.status["required"], bool(lists.status["exceeded"])) == (most, most > cap), call
    assert ws.status() == (25000, True)


def test_scene_batch_with_an_empty_scene(poisoned):
    """S = 3: an empty scene, one with lists above 8192, an ordinary one; each computed alone gives its rows."""
    dev = _dev()
    h, w, views, long_cells = designed_case("scene_long")
    ordinary = designed_case("scene_ordinary")[3]
    kw = dict(depth_mode="depth", alpha=True, cam=True, square=True)
    whole = _designed_batch([None, long_cells, ordinary], h, w, views, dev)
    P = whole.ins["means3D"].shape[1]
    _designed_parity(whole, **kw)
    with _deterministic():
        got = _run(whole, _workspace(whole, whole.D, **ALL_FLAGS), **kw)
        for k, cells in enumerate([None, long_cells, ordinary]):
            one = _designed_batch([cells], h, w, views, dev, P=P, seed=k)
            ws = _workspace(one, max(one.D, 1), **ALL_FLAGS)
            alone = _run(one, ws, **kw)
            check_lists(ws, alone["radii"], one.lengths, one.D)
            for name, t in alone.items():
                per_scene = name in ("d_means3D", "d_opacities", "d_shs", "d_cov3D_precomp")
                rows = got[name][k:k + 1] if per_scene else got[name][views * k:views * (k + 1)]
                assert torch.equal(rows, t), (k, name)


# ---------------------------------------------------------------------------------------------------------------------
# 2. input forms and the overflow NaN contract
# ---------------------------------------------------------------------------------------------------------------------
def _cloud(dev, scenes=1, views=2, P=12_000, hw=(56, 72), seed=70):
    """an ordinary make_scene cloud, with the extra forms' inputs: scales, rotations, colours, a means2D sink"""
    sc = [make_scene(P, views, *hw, seed=seed + k) for k in range(scenes)]
    cat = lambda f: torch.cat([f(s) for s in sc]).to(dev)
    st = lambda f: torch.stack([f(s) for s in sc]).to(dev)
    vb, bg, nf = _cameras(cat(lambda s: s.extrinsics), cat(lambda s: s.intrinsics), cat(lambda s: s.near),
                          cat(lambda s: s.far), dev)
    c = lambda s: s.covariances
    ins = {"means3D": st(lambda s: s.means), "opacities": st(lambda s: s.opacities),
           "shs": st(lambda s: s.harmonics.transpose(-1, -2)),
           "cov3D_precomp": st(lambda s: torch.stack([c(s)[:, 0, 0], c(s)[:, 0, 1], c(s)[:, 0, 2], c(s)[:, 1, 1],
                                                      c(s)[:, 1, 2], c(s)[:, 2, 2]], -1))}
    b = Batch(vb, bg, nf, ins, hw)
    g = torch.Generator().manual_seed(seed)
    V = vb.viewmatrix.shape[0]
    b.extra = {"scales": st(lambda s: s.scales), "rotations": st(lambda s: s.rotations),
               "colors_precomp": torch.rand(V, P, 3, generator=g).to(dev), "means2D": torch.zeros(V, P, 3, device=dev)}
    return b


FORMS = ["scales_rotations", "colors_precomp", "means2D", "opacities_p1", "camera_grad", "color_only_loss"] + \
        [f"view_z_{m}" for m in ("depth", "disparity", "relative_disparity", "log")]


def _form(b: Batch, form):
    """(batch, run keywords) of one input form"""
    kw = dict(degree=3, depth_mode="depth", alpha=True)
    if form == "scales_rotations":
        return b.with_inputs(cov3D_precomp=None, scales=b.extra["scales"], rotations=b.extra["rotations"]), kw
    if form == "colors_precomp":
        return b.with_inputs(shs=None, colors_precomp=b.extra["colors_precomp"]), kw
    if form == "means2D":
        return b.with_inputs(means2D=b.extra["means2D"]), kw
    if form == "opacities_p1":
        return b.with_inputs(opacities=b.ins["opacities"][..., None]), kw
    if form == "camera_grad":
        return b, {**kw, "cam": True}
    if form == "color_only_loss":
        return b, {**kw, "loss_on": ("color",)}
    return b, {**kw, "vz": True, "depth_mode": form[len("view_z_"):]}


@pytest.mark.parametrize("form", FORMS)
def test_input_forms_and_their_overflow(poisoned, form):
    dev = _dev()
    b, kw = _form(_cloud(dev), form)
    with _deterministic():
        ref = _run(b, **kw)
        D = last_stats(dev)["num_rendered"]
        assert D > 2
        S, P = b.ins["means3D"].shape[:2]
        V = b.vb.viewmatrix.shape[0]
        need = sync_free_workspace_bytes(S, V, P, *b.hw, D, deterministic=True, camera_grad=True)
        guard = 1 << 16
        big = torch.empty(2 * guard + need, dtype=torch.uint8, device=dev)
        pattern = (torch.arange(guard, device=dev) * 7 % 251).to(torch.uint8)
        big[:guard], big[-guard:] = pattern, pattern
        for cap in (D, D - 1):
            ws = _workspace(b, cap, buffer=big[guard:guard + need], **ALL_FLAGS)
            got = _run(b, ws, **kw)
            assert torch.equal(big[:guard], pattern) and torch.equal(big[-guard:], pattern), cap
            assert torch.equal(got["radii"], ref["radii"]), cap
            if cap == D:
                _compare(ref, got, True, form)
                check_lists(ws, got["radii"], D=D)
                continue
            assert ws.status() == (D, True)
            check_lists(ws, got["radii"], D=D)
            assert got.keys() == ref.keys()
            for k, t in got.items():
                if k == "radii":
                    continue
                if k == "d_viewmatrix" and kw.get("vz"):   # the depth's gradient reaches the z column alone
                    assert torch.isnan(t[..., 2]).all() and not t[..., :2].any() and not t[..., 3].any(), k
                else:
                    assert torch.isnan(t).all(), (cap, k)
    expected = {"scales_rotations": ("d_scales", "d_rotations"), "colors_precomp": ("d_colors_precomp",),
                "means2D": ("d_means2D",), "camera_grad": ("d_viewmatrix", "d_projmatrix", "d_campos", "d_tanfov")}
    for k in expected.get(form, ("d_viewmatrix",) if kw.get("vz") else ()):
        assert k in got, k
    if form == "color_only_loss":
        assert "d_viewmatrix" not in got


# ---------------------------------------------------------------------------------------------------------------------
# 3. tuning knobs and status words
# ---------------------------------------------------------------------------------------------------------------------
HONOURED = [("FWD_WS", dict(max_degree=4, degree=4), True), ("PRE_OCC6", dict(max_degree=3, degree=3), True),
            ("PRE_SH_RAW16", dict(max_degree=4, degree=4), True), ("BWD_OCC4", dict(max_degree=4, degree=4), True),
            ("PBWD_2PHASE", dict(max_degree=3, degree=3), True), ("BWD_V1", dict(max_degree=4, degree=4), False)]


@pytest.mark.parametrize("knob,kw,det", HONOURED, ids=[k for k, _, _ in HONOURED])
def test_honoured_knobs_match_the_default_path_with_the_same_knob(poisoned, knob, kw, det):
    dev = _dev()
    b = _cloud(dev, scenes=2, views=2, P=15_000, hw=(64, 80), seed=80)
    kw = dict(kw, depth_mode="depth", tuning=getattr(_capi, "GS_TUNE_" + knob))
    with _deterministic(det):
        ref = _run(b, **kw)
        D = last_stats(dev)["num_rendered"]
        ws = _workspace(b, D, depth=True, deterministic=det)
        got = _run(b, ws, **kw)
    _compare(ref, got, det, knob)
    check_lists(ws, got["radii"], D=D)
    assert ws.status() == (D, False)


IGNORED = ["FORCE_RADIX_BINNING", "NO_SPECULATION", "NO_STRATA", "ALL_STRATA", "STRATA_MERGE_SORT"]


def test_knobs_of_the_default_binning_change_no_sync_free_bit(poisoned):
    dev = _dev()
    b = _case_batch("long_lists", dev)
    kw = dict(depth_mode="depth", alpha=True)
    ws = _workspace(b, b.D, **ALL_FLAGS)
    with _deterministic():
        base = _run(b, ws, **kw)
        lists = read_lists(ws)
        for knob in IGNORED:
            got = _run(b, ws, tuning=getattr(_capi, "GS_TUNE_" + knob), **kw)
            _compare(base, got, True, knob)
            again = read_lists(ws)
            assert np.array_equal(lists.ranges, again.ranges) and np.array_equal(lists.index, again.index), knob


def test_status_words_over_a_sequence(poisoned):
    """D1 < D2 > D3, all fitting: (D2, False); an exceeded call in the middle: exceeded until clear_status(); SF_D and
    SF_MAX_LIST describe the last call."""
    dev = _dev()
    h, w, views, _ = designed_case("shifting")
    full = _designed_batch([list(SHIFT_POOL)], h, w, views, dev)
    P = full.ins["means3D"].shape[1]
    starts = np.cumsum([0] + [c[3] for c in SHIFT_POOL])

    def subset(ks):
        keep = torch.zeros(P, dtype=torch.bool)
        for s, k in zip(starts, ks):
            keep[s:s + k] = True
        means = torch.where(keep.to(dev)[None, :, None], full.ins["means3D"], torch.tensor(PARKED, device=dev))
        return full.with_inputs(means3D=means), sum(ks), max(ks)

    small, mid, big = (1000, 10, 10, 10, 10), (9000, 4000, 2000, 8000, 1000), (3000, 3000, 100, 0, 5)
    ws = _workspace(full, 24000, depth=True)
    for seq, want in (((small, mid, big), (sum(mid), False)), ((small, SHIFT_CALLS[2], big), (25000, True))):
        ws.clear_status()
        for ks in seq:
            b, D, longest = subset(ks)
            out = _run(b, ws, depth_mode="depth")
            words = read_lists(ws).status
            assert (words["D"], words["max_list"]) == (D, longest)
        assert ws.status() == want, seq
        check_lists(ws, out["radii"], D=sum(big))
    ws.clear_status()
    assert ws.status() == (0, False)
