"""GPU tests of the pose loss (csrc/gs_pose_loss.cu) past the shapes of tests/test_gpu_pose_loss.py, every one with each
torch.empty poisoned (tests/poison.py), against the fp64 oracle (oracle/pose_loss_oracle.py) on the device:
per-segment and one-sided cotangents through `pose_terms`, 2 to 16 views with a non-finite depth under every source
view, key counts b v h w at and around powers of two (the sort's bit width), long runs on one pixel, 2^20 matches in
one segment and millions in one call, degenerate frames, the later golden cases against both reference records,
confinement of non-finite inputs to their scene, and determinism.  Element-wise bound as in the rest of the suite:
|ours - ref| <= 1e-3 (|ref| + rms(ref)), with the same non-finite elements; each test prints its worst ratio to it."""
import numpy as np
import pytest
import torch

from oracle import pose_loss_oracle as po
from pf3plat_b200 import losses
from tests.poison import poisoned  # noqa: F401  (fixture)
from tests.pose_loss_cases import GRADS, NEW_GOLDEN_CASES, Case, golden_case, load_golden, pairs_of, seeded_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RTOL = 1e-3
OUTS = ("L3", "L2") + GRADS


def _ratio(label, ours, ref):
    """Same non-finite pattern, then the worst |ours - ref| / (|ref| + rms(ref)) over the finite elements."""
    a = ours.detach().double().reshape(-1)
    b = (ref if torch.is_tensor(ref) else torch.from_numpy(np.asarray(ref, np.float64))).detach().double()
    b = b.to(a.device).reshape(-1)
    assert a.shape == b.shape, label
    fa, fb = torch.isfinite(a), torch.isfinite(b)
    bad = torch.nonzero(fa != fb).reshape(-1)[:8].tolist()
    assert not bad, f"{label}: finite mismatch at {bad} (ours {a[bad].tolist()}, ref {b[bad].tolist()})"
    assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{label}: NaN mismatch"
    if not fa.any():
        return 0.0
    rms = float(torch.sqrt(torch.mean(b[fb] ** 2)))
    r = (a[fa] - b[fa]).abs() / (b[fa].abs() + rms + 1e-300)
    worst = float(r.max())
    assert worst <= RTOL, f"{label}: worst ratio {worst:.3e} at {int(torch.argmax(r))}"
    return worst / RTOL


def _compare(label, ours, ref, keys=OUTS):
    worst = max(_ratio(f"{label} {k}", ours[k], ref[k]) for k in keys)
    print(f"[pose-loss regimes] {label}: worst {worst:.3g} of the bound")
    return worst


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _mean_cot(case):
    S = case.b * len(pairs_of(case.v))
    return torch.full((S,), 0.025 / S, dtype=torch.float64), torch.full((S,), 0.005 / S, dtype=torch.float64)


def _ours(case, g3, g2, need=GRADS):
    """pose_terms on the device; gradients of sum(g3 L3) + sum(g2 L2), a None cotangent leaving its term out."""
    c = case.to(DEV)
    leaves = {k: getattr(c, k).clone().requires_grad_(k in need) for k in ("abspose", "depth", "xyz", "w", "conf")}
    corre, conf = c.matches(w=leaves["w"], conf=leaves["conf"])
    L3, L2 = losses.pose_terms(leaves["abspose"], leaves["depth"], leaves["xyz"], c.K, corre, conf, c.h, c.width)
    outs, cots = zip(*[(L, g.to(device=DEV, dtype=torch.float32)) for L, g in ((L3, g3), (L2, g2)) if g is not None])
    grads = torch.autograd.grad(outs, [leaves[k] for k in need], cots)
    torch.cuda.synchronize()
    out = {"L3": L3.detach(), "L2": L2.detach()}
    out.update(dict(zip(need, grads)))
    return out


def _oracle(case, g3, g2):
    c = case.to(DEV)
    corre, conf = c.matches()
    f32 = lambda g: None if g is None else g.to(torch.float32).double()  # noqa: E731  (the cotangents the kernel sees)
    return po.terms_and_grads(c.abspose, c.depth, c.xyz, c.K, corre, conf, c.h, c.width, f32(g3), f32(g2))


def _both(label, case, g3=None, g2=None, mean=True):
    if mean:
        g3, g2 = _mean_cot(case)
    ours = _ours(case, g3, g2)
    return ours, _compare(label, ours, _oracle(case, g3, g2))


def _with_matches(base, seg_matches, seed=0):
    """base's poses, depth, xyz, K and conf with the matches {segment: (id_a, id_c)} (others empty), random weights."""
    S = base.b * len(pairs_of(base.v))
    g = torch.Generator().manual_seed(seed)
    ia, ic, counts = [], [], np.zeros(S, np.int64)
    for s in range(S):
        a, c = seg_matches.get(s, (torch.zeros(0, dtype=torch.int64),) * 2)
        ia.append(torch.as_tensor(a, dtype=torch.int64))
        ic.append(torch.as_tensor(c, dtype=torch.int64))
        counts[s] = len(ia[-1])
    M = int(counts.sum())
    w = 0.05 + 0.95 * torch.rand(M, generator=g)
    return Case(base.abspose, base.depth, base.xyz, base.K, torch.cat(ia), torch.cat(ic), w, counts, base.conf, base.h,
                base.width)


def _random_matches(base, n_min, n_max, seed, empty=()):
    g = torch.Generator().manual_seed(seed)
    hw = base.h * base.width
    out = {}
    for s in range(base.b * len(pairs_of(base.v))):
        n = 0 if s in empty else int(torch.randint(n_min, n_max + 1, (1,), generator=g))
        out[s] = (torch.randint(0, hw, (n,), generator=g), torch.randint(0, hw, (n,), generator=g))
    return out


def _offsets(case):
    return np.concatenate([[0], np.cumsum(case.counts)]).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# per-segment cotangents through pose_terms


@pytest.mark.parametrize("kind", ["random", "zeros", "nan"])
def test_per_segment_cotangents(kind, poisoned):  # noqa: F811
    case = seeded_case(3, 4, 40, 24, 1, 300, seed=701)
    S = case.b * 6
    g = torch.Generator().manual_seed(702)
    g3 = torch.randn(S, generator=g, dtype=torch.float64) * torch.rand(S, generator=g, dtype=torch.float64) * 10
    g2 = torch.randn(S, generator=g, dtype=torch.float64) * 0.1
    if kind == "zeros":
        g3[::3] = 0.0
        g2[1::4] = 0.0
        g3[5] = g2[5] = 0.0
    s3, s2 = 7, 11  # a NaN L3 cotangent in one segment, a NaN L2 cotangent in another
    if kind == "nan":
        g3[s3] = float("nan")
        g2[s2] = float("nan")
    ours, _ = _both(f"cotangents {kind}", case, g3, g2, mean=False)
    assert poisoned.off_thread_calls() > 0
    if kind == "zeros":  # a segment with both cotangents 0 contributes nothing: its dconf and dw are exactly 0
        o = _offsets(case)
        assert float(ours["conf"].reshape(-1)[5]) == 0.0 and (ours["w"][o[5]:o[6]] == 0).all()
    if kind == "nan":
        o = _offsets(case)
        nan_w = torch.nonzero(~torch.isfinite(ours["w"])).reshape(-1).cpu()
        assert torch.equal(nan_w, torch.arange(o[s3], o[s3 + 1]))  # the L2 cotangent does not reach dw
        assert torch.nonzero(~torch.isfinite(ours["conf"].reshape(-1))).reshape(-1).tolist() == [s3]
        # pixels: only those the two segments' matches name, in their scenes and views
        allowed_d, allowed_x = set(), set()
        hw = case.h * case.width
        for s in (s3, s2):
            i, (a, c) = divmod(s, 6)[0], pairs_of(4)[s % 6]
            for p, q in zip(case.id_a[o[s]:o[s + 1]].tolist(), case.id_c[o[s]:o[s + 1]].tolist()):
                allowed_x.update({((i * 4 + a) * hw + p), ((i * 4 + c) * hw + q)})
                if s == s2:
                    allowed_d.add((i * 4 + a) * hw + p)
        bad_d = set(torch.nonzero(~torch.isfinite(ours["depth"].reshape(-1))).reshape(-1).tolist())
        xyz = ours["xyz"].reshape(case.b * 4, 3, hw).permute(0, 2, 1).reshape(-1, 3)
        bad_x = set(torch.nonzero(~torch.isfinite(xyz).all(-1)).reshape(-1).tolist())
        assert bad_d and bad_d <= allowed_d and bad_x and bad_x <= allowed_x
        assert torch.isfinite(ours["abspose"][torch.arange(3, device=DEV) != 1]).all()  # segments 7 and 11 are scene 1's


@pytest.mark.parametrize("which", ["seeded", "v3_b2_nonfinite_weights_conf", "v3_b1_nan_depth_unmatched",
                                   "v3_b2_nonfinite_K"])
def test_one_sided_cotangents_are_a_zero_cotangent_through_the_chain(which, poisoned):  # noqa: F811
    case = seeded_case(2, 3, 32, 32, 0, 50, seed=703) if which == "seeded" else golden_case(load_golden(), which)
    S = case.b * len(pairs_of(case.v))
    g = torch.Generator().manual_seed(704)
    g3 = torch.randn(S, generator=g, dtype=torch.float64)
    g2 = torch.randn(S, generator=g, dtype=torch.float64)
    worst = 0.0
    for a, b in ((g3, None), (None, g2)):
        ours = _ours(case, a, b)
        worst = max(worst, _compare(f"one-sided {which} L{'3' if b is None else '2'} only", ours, _oracle(case, a, b)))
        zero = _ours(case, a if a is not None else torch.zeros(S), b if b is not None else torch.zeros(S))
        for k in GRADS:  # a None cotangent is bit for bit a zero one
            assert torch.equal(_bits(ours[k]), _bits(zero[k])), k
    assert poisoned.off_thread_calls() > 0
    print(f"[pose-loss regimes] one-sided {which}: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# views: the dense pass's segment index for every source view


@pytest.mark.parametrize("b,v", [(1, 2), (2, 3), (3, 4), (4, 5), (2, 6), (1, 7), (3, 8), (1, 16)])
def test_views_with_a_nonfinite_depth_under_every_source_view(b, v, poisoned):  # noqa: F811
    base = seeded_case(b, v, 16, 20, 0, 0, seed=710 + v)
    P = len(pairs_of(v))
    # two or more matches per nonempty segment: one match has dL/dw = 0 up to the rounding of two cancelling terms
    case = _with_matches(base, _random_matches(base, 2, 10, seed=711 + v, empty=(1, b * P - 2)), seed=712)
    worst = _both(f"views b={b} v={v} clean", case)[1]
    assert 0 in case.counts or b * P == 1
    o = _offsets(case)
    for a in range(v - 1):  # one run per source view, the NaN in scene a mod b
        i = a % b
        used = set()
        for k, (sa, _) in enumerate(pairs_of(v)):
            s = i * P + k
            if sa == a:
                used.update(case.id_a[o[s]:o[s + 1]].tolist())
        p = next(x for x in range(16 * 20) if x not in used)
        bad = Case(case.abspose, case.depth.clone(), case.xyz, case.K, case.id_a, case.id_c, case.w, case.counts,
                   case.conf, case.h, case.width)
        bad.depth.view(b, v, -1)[i, a, p] = float("nan")
        ours, r = _both(f"views b={b} v={v} NaN depth under view {a}", bad)
        worst = max(worst, r)
        ga = ours["abspose"][i]
        # the pairs (a, c > a) are poisoned: views c > a, and view a itself when it goes through the inverse
        assert (~torch.isfinite(ga)).any(-1).any(-1).tolist() == [x > a or (x == a and a > 0) for x in range(v)]
    assert poisoned.off_thread_calls() > 0
    print(f"[pose-loss regimes] views b={b} v={v}: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# the sort's key width: b v h w at 2^k - 1, 2^k, 2^k + 1


def _end_bit(pix):  # the kernel's end_bit_of(key_end = pix)
    return max(1, int(pix).bit_length())


def _entry(key, v, hw, P):
    """-> (segment, side, pixel) of a match entry with this key: the source side of pair (view, v-1) for a source view,
    the target side of pair (0, view) for the last view"""
    i, r = divmod(key, v * hw)
    view, p = divmod(r, hw)
    pr = (view, v - 1) if view < v - 1 else (0, view)
    return i * P + pairs_of(v).index(pr), 0 if view < v - 1 else 1, p


@pytest.mark.parametrize("v,h,w", [(3, 11, 31), (4, 16, 16), (5, 5, 41), (7, 889, 337), (2, 1024, 1024),
                                   (3, 129, 5419)])
def test_key_width_edges_on_the_first_last_and_top_bit_keys(v, h, w, poisoned):  # noqa: F811
    """b = 1 and v h w = 2^k - 1, 2^k, 2^k + 1 for k = 10 and 21.  Matches on key 0, the last key and, where one fits,
    keys k0 and k0 + 2^(bits-1) (bits = the sort's end bit) as the two sides of one pair, so that their entries
    alternate in entry order: with a bit too few they would sort together and break each other's runs."""
    hw, pix, P = h * w, v * h * w, len(pairs_of(v))
    assert min(abs(pix - 2 ** k) for k in (10, 21)) <= 1
    base = seeded_case(1, v, h, w, 0, 0, seed=720 + v)
    m = {s: [a.tolist(), c.tolist()] for s, (a, c) in _random_matches(base, 1, 40, seed=721 + v).items()}
    g = torch.Generator().manual_seed(722)
    rnd = lambda: int(torch.randint(0, hw, (1,), generator=g))  # noqa: E731
    for key in (0, pix - 1):
        s, side, p = _entry(key, v, hw, P)
        for _ in range(3):
            m[s][side].append(p)
            m[s][1 - side].append(rnd())
    half = 2 ** (_end_bit(pix) - 1)
    if half < pix:  # keys k0 = (view 0, pixel 0) and k0 + half = (view c, q) in pair (0, c)
        c, q = divmod(half, hw)
        assert 0 < c < v
        s = pairs_of(v).index((0, c))
        for p0 in range(4):
            m[s][0].append(p0 if p0 < 2 else 0)
            m[s][1].append(q)
    case = _with_matches(base, {s: (torch.tensor(a), torch.tensor(c)) for s, (a, c) in m.items()}, seed=723)
    _both(f"key width v={v} {h}x{w} (v h w = {pix}, {_end_bit(pix)} bits)", case)
    assert poisoned.off_thread_calls() > 0


@pytest.mark.parametrize("b,v,h,w", [(3, 11, 1, 31), (2, 2, 16, 16), (5, 5, 41, 1), (7, 7, 127, 337),
                                     (2, 4, 512, 512), (3, 3, 43, 5419)])
def test_key_width_edges_with_sentinels_in_another_scene(b, v, h, w, poisoned):  # noqa: F811
    """b v h w at 2^k - 1, 2^k, 2^k + 1 (k = 10, 21) with b >= 2, matches on key 0 and the last key, then a bad index in
    the first or last scene: every other scene keeps its bits, and the bad segment is NaN in L3, L2, dT, dconf, dw and
    at exactly the pixels its in-range indices name."""
    hw, pix, P = h * w, b * v * h * w, len(pairs_of(v))
    base = seeded_case(b, v, h, w, 0, 0, seed=730 + b)
    m = {s: [a.tolist(), c.tolist()] for s, (a, c) in _random_matches(base, 2, 30, seed=731).items()}
    for key in (0, pix - 1):
        s, side, p = _entry(key, v, hw, P)
        m[s][side] += [p, p]
        m[s][1 - side] += [1 % hw, 0]
    clean = _with_matches(base, {s: (torch.tensor(a), torch.tensor(c)) for s, (a, c) in m.items()}, seed=732)
    ref, worst = _both(f"sentinels b={b} v={v} {h}x{w} clean", clean)
    for i in (0, b - 1):
        s = i * P + P - 1  # the scene's last pair (v-2, v-1)
        a, c = pairs_of(v)[P - 1]
        at = int(_offsets(clean)[s])  # two matches first in the segment: (0, -1) and (hw, 0), one past the last pixel
        ins = lambda t, x: torch.cat([t[:at], torch.tensor(x, dtype=t.dtype), t[at:]])  # noqa: E731
        counts = clean.counts.copy()
        counts[s] += 2
        bad = Case(clean.abspose, clean.depth, clean.xyz, clean.K, ins(clean.id_a, [0, hw]), ins(clean.id_c, [-1, 0]),
                   ins(clean.w, [0.5, 0.7]), counts, clean.conf, h, w)
        ours = _ours(bad, *_mean_cot(bad))
        assert torch.isnan(ours["L3"][s]) and torch.isnan(ours["L2"][s]) and torch.isnan(ours["conf"].reshape(-1)[s])
        keep = torch.arange(b * P, device=DEV) != s
        for k in ("L3", "L2"):
            assert torch.equal(_bits(ours[k][keep]), _bits(ref[k][keep])), k
        assert torch.equal(_bits(ours["conf"].reshape(-1)[keep]), _bits(ref["conf"].reshape(-1)[keep]))
        o, oc = _offsets(bad), _offsets(clean)
        assert torch.isnan(ours["w"][o[s]:o[s + 1]]).all()
        assert torch.equal(_bits(ours["w"][:o[s]]), _bits(ref["w"][:oc[s]]))
        assert torch.equal(_bits(ours["w"][o[s + 1]:]), _bits(ref["w"][oc[s + 1]:]))
        other = torch.arange(b, device=DEV) != i
        for k in ("abspose", "xyz"):
            assert torch.equal(_bits(ours[k][other]), _bits(ref[k][other])), k
        dd, dr = ours["depth"].reshape(b, v, hw), ref["depth"].reshape(b, v, hw)
        assert torch.equal(_bits(dd[other]), _bits(dr[other]))
        # the bad scene: NaN exactly where the segment's in-range indices point, the clean bits elsewhere
        ia = bad.id_a[o[s]:o[s + 1]]
        ic = bad.id_c[o[s]:o[s + 1]]
        ok = (ia >= 0) & (ia < hw) & (ic >= 0) & (ic < hw)
        want_d = torch.zeros(v, hw, dtype=torch.bool)
        want_d[a, ia[ok]] = True
        want_x = want_d.clone()
        want_x[c, ic[ok]] = True
        assert torch.equal(torch.isnan(dd[i]).cpu(), want_d)
        xi = ours["xyz"][i].reshape(v, 3, hw)
        assert torch.equal(torch.isnan(xi).any(1).cpu(), want_x) and torch.equal(torch.isnan(xi).all(1).cpu(), want_x)
        assert torch.equal(_bits(dd[i][~want_d.to(DEV)]), _bits(dr[i][~want_d.to(DEV)]))
        xr = ref["xyz"][i].reshape(v, 3, hw)
        assert torch.equal(_bits(xi.permute(0, 2, 1)[~want_x.to(DEV)]), _bits(xr.permute(0, 2, 1)[~want_x.to(DEV)]))
    assert poisoned.off_thread_calls() > 0
    print(f"[pose-loss regimes] sentinels b={b} v={v} {h}x{w}: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# runs


def test_long_runs_identical_pairs_and_scene_slices(poisoned):  # noqa: F811
    b, v, h, w = 3, 2, 64, 64
    hw = h * w
    base = seeded_case(b, v, h, w, 0, 0, seed=740)
    g = torch.Generator().manual_seed(741)
    n = 120_000
    m = {0: (torch.full((n,), 1234), torch.randint(0, hw, (n,), generator=g)),   # every match on one source pixel
         1: (torch.arange(0, hw, 3), torch.arange(0, hw, 3))}                    # p == q across the pair
    pq = torch.randint(0, hw, (2, 40), generator=g)
    m[2] = (pq[0].repeat(50), pq[1].repeat(50))                                  # 40 (p, q) pairs, each 50 times
    case = _with_matches(base, m, seed=742)
    ours, worst = _both("runs", case)
    # each scene alone has the bits of its slice of the batch (the stable sort keeps entry order within a pixel)
    o = _offsets(case)
    for i in range(b):
        sl = slice(int(o[i]), int(o[i + 1]))
        one = Case(case.abspose[i:i + 1], case.depth[i * v:(i + 1) * v], case.xyz[i:i + 1], case.K[i:i + 1],
                   case.id_a[sl], case.id_c[sl], case.w[sl], case.counts[i:i + 1], case.conf[i:i + 1], h, w)
        g3, g2 = _mean_cot(case)
        alone = _ours(one, g3[i:i + 1], g2[i:i + 1])
        for k in ("L3", "L2", "conf"):
            assert torch.equal(_bits(alone[k].reshape(-1)), _bits(ours[k].reshape(-1)[i:i + 1])), (i, k)
        for k in ("abspose", "xyz"):
            assert torch.equal(_bits(alone[k][0]), _bits(ours[k][i])), (i, k)
        assert torch.equal(_bits(alone["depth"]), _bits(ours["depth"][i * v:(i + 1) * v])), i
        assert torch.equal(_bits(alone["w"]), _bits(ours["w"][sl])), i
    assert poisoned.off_thread_calls() > 0
    print(f"[pose-loss regimes] runs: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# scale


@pytest.mark.parametrize("what", ["one segment of 2^20", "several million", "training shape, 2048 per segment"])
def test_scale(what, poisoned):  # noqa: F811
    if what == "one segment of 2^20":
        base = seeded_case(1, 2, 256, 256, 0, 0, seed=750)
        case = _with_matches(base, _random_matches(base, 2 ** 20, 2 ** 20, seed=751), seed=752)
    elif what == "several million":
        base = seeded_case(4, 3, 256, 256, 0, 0, seed=753)
        case = _with_matches(base, _random_matches(base, 250_000, 400_000, seed=754), seed=755)
        assert case.counts.sum() > 3_000_000
    else:
        base = seeded_case(14, 3, 256, 256, 0, 0, seed=756)
        case = _with_matches(base, _random_matches(base, 2048, 2048, seed=757), seed=758)
    _both(f"scale: {what} ({int(case.counts.sum())} matches)", case)
    assert poisoned.off_thread_calls() > 0


# ---------------------------------------------------------------------------------------------------------------------
# frames


@pytest.mark.parametrize("b,v,h,w", [(2, 3, 1, 300), (2, 3, 300, 1), (3, 4, 1, 1), (2, 3, 257, 263)])
def test_frames(b, v, h, w, poisoned):  # noqa: F811
    base = seeded_case(b, v, h, w, 0, 0, seed=760 + h)
    case = _with_matches(base, _random_matches(base, 0, 700, seed=761 + w), seed=762)
    if h * w > 1:
        _both(f"frame b={b} v={v} {h}x{w}", case)
    else:  # every match of a segment reads the same two pixels: e3 is constant and dL/dw is 0 up to rounding
        g3, g2 = _mean_cot(case)
        ours = _ours(case, g3, g2)
        _compare(f"frame b={b} v={v} {h}x{w}", ours, _oracle(case, g3, g2), keys=("L3", "L2", "abspose", "depth",
                                                                                 "xyz", "conf"))
        assert ours["w"].abs().max() <= 1e-6 * ours["conf"].abs().max()
    assert poisoned.off_thread_calls() > 0


# ---------------------------------------------------------------------------------------------------------------------
# the golden cases recorded later, against both reference records


@pytest.mark.parametrize("name", NEW_GOLDEN_CASES)
def test_new_golden_cases_match_both_records(name, poisoned):  # noqa: F811
    z = load_golden()
    case = golden_case(z, name)
    ours, worst = _both(f"golden {name} vs oracle", case)
    # the records hold the loss, not its terms: form it from ours as the reference does
    loss = ours["L3"].double().mean() * 0.025 + ours["L2"].double().mean() * 0.005
    for tag in ("f32", "f64"):
        worst = max(worst, _ratio(f"{name} loss vs {tag}", loss, z[f"{name}/{tag}/loss"]))
        for k in GRADS:
            ref = z[f"{name}/{tag}/grad_{k}"]
            got = ours[k]
            if name == "v3_b2_clamp" and k == "w" and tag == "f64":
                # a single weight of exactly +-float32(1e-12) passes the float32 clamp and is clamped in float64: the
                # float32 record is the truth there (PF3plat trains in float32)
                o = _offsets(case)
                keep = np.ones(len(ref), bool)
                keep[[o[0], o[5]]] = False
                ref, got = ref[keep], got[torch.from_numpy(keep).to(DEV)]
            worst = max(worst, _ratio(f"{name} dL/d{k} vs {tag}", got, ref))
    assert poisoned.off_thread_calls() > 0
    print(f"[pose-loss regimes] golden {name}: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# confinement


@pytest.mark.parametrize("what", ["NaN weight", "Inf weight", "NaN conf", "Inf conf", "Inf K_c", "NaN pose view 1",
                                  "Inf pose view 2"])
def test_nonfinite_input_stays_in_its_scene(what, poisoned):  # noqa: F811
    b, v, h, w = 3, 3, 24, 20
    clean = seeded_case(b, v, h, w, 1, 60, seed=770)
    bad = seeded_case(b, v, h, w, 1, 60, seed=770)
    i = 1
    o = _offsets(clean)
    if what.endswith("weight"):
        bad.w[o[3 * i + 1]] = float("nan" if what.startswith("NaN") else "inf")
    elif what.endswith("conf"):
        bad.conf[i, 2] = float("nan" if what.startswith("NaN") else "inf")
    elif what == "Inf K_c":
        bad.K[i, 2, 0, 0] = float("inf")
    else:
        bad.abspose[i, 1 if "1" in what else 2, 0, 3] = float("nan" if what.startswith("NaN") else "inf")
    g3, g2 = _mean_cot(clean)
    rc, rb = _ours(clean, g3, g2), _ours(bad, g3, g2)
    _compare(f"confinement {what}", rb, _oracle(bad, g3, g2))
    other = torch.arange(b, device=DEV) != i
    segs = torch.arange(b * 3, device=DEV) // 3 != i
    for k in ("L3", "L2"):
        assert torch.equal(_bits(rb[k][segs]), _bits(rc[k][segs])), k
    assert torch.equal(_bits(rb["conf"][other]), _bits(rc["conf"][other]))
    for k in ("abspose", "xyz"):
        assert torch.equal(_bits(rb[k][other]), _bits(rc[k][other])), k
    assert torch.equal(_bits(rb["depth"].reshape(b, -1)[other]), _bits(rc["depth"].reshape(b, -1)[other]))
    mine = torch.zeros(len(clean.w), dtype=torch.bool, device=DEV)
    mine[o[3 * i]:o[3 * i + 3]] = True
    assert torch.equal(_bits(rb["w"][~mine]), _bits(rc["w"][~mine]))
    assert not all(torch.isfinite(rb[k]).all() for k in ("L3", "L2") + GRADS)  # the bad scene is not clean
    assert poisoned.off_thread_calls() > 0


# ---------------------------------------------------------------------------------------------------------------------
# determinism


def test_deterministic_algorithms_give_the_same_bits(monkeypatch, poisoned):  # noqa: F811
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # the glue's 4x4 matmuls under the deterministic setting
    cases = []
    base = seeded_case(3, 8, 16, 20, 0, 0, seed=780)
    cases.append(_with_matches(base, _random_matches(base, 0, 30, seed=781, empty=(2,)), seed=782))
    cases[-1].depth.view(3, 8, -1)[1, 2, 5] = float("nan")
    base = seeded_case(2, 2, 64, 64, 0, 0, seed=783)
    cases.append(_with_matches(base, {0: (torch.full((50_000,), 77), torch.arange(50_000) % 4096),
                                      1: (torch.arange(4096), torch.arange(4096))}, seed=784))
    cases.append(golden_case(load_golden(), "v3_b2_nonfinite_weights_conf"))
    cases.append(seeded_case(1, 3, 11, 31, 1, 300, seed=785))
    for n, case in enumerate(cases):
        g = torch.Generator().manual_seed(786 + n)
        S = case.b * len(pairs_of(case.v))
        g3, g2 = torch.randn(S, generator=g), torch.randn(S, generator=g)
        free = _ours(case, g3, g2)
        torch.use_deterministic_algorithms(True)
        try:
            det = _ours(case, g3, g2)
        finally:
            torch.use_deterministic_algorithms(False)
        for k in OUTS:
            assert torch.equal(_bits(free[k]), _bits(det[k])), (n, k)
    assert poisoned.off_thread_calls() > 0
