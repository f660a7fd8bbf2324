"""GPU tests of the pose (correspondence) loss (pf3plat_b200.losses.pose_loss -> csrc/gs_pose_loss.cu) against the fp64
oracle (oracle/pose_loss_oracle.py) and the reference's own Losspose (tests/golden/pose_loss.npz)."""
import numpy as np
import pytest
import torch

from oracle import pose_loss_oracle as po
from pf3plat_b200 import losses
from tests.pose_loss_cases import GOLDEN_CASES, GRADS, golden_case, load_golden, pairs_of, seeded_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RTOL = 1e-3   # BASELINE.json's gradient tolerance, element-wise: |ours - ref| <= 1e-3 (|ref| + rms(ref))


def _ours(case, need=GRADS, stream=None):
    """pose_loss on the objects Losspose receives; -> dict of the loss and the gradients of the `need` leaves."""
    c = case.to(DEV)
    leaves = {k: getattr(c, k if k != "depth" else "depth").clone() for k in ("abspose", "depth", "xyz", "w", "conf")}
    for k in need:
        leaves[k].requires_grad_(True)
    corre, conf = c.matches(w=leaves["w"], conf=leaves["conf"])
    img = torch.zeros(c.b, c.v, 3, c.h, c.width, device=DEV)
    batch = {"context": {"image": img}, "target": {"image": img, "intrinsics": c.K}}
    relpose = torch.eye(4, device=DEV).repeat(c.b, len(pairs_of(c.v)), 1, 1)
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        loss = losses.pose_loss(batch, (relpose, leaves["abspose"]), (leaves["depth"],), (corre, None, conf),
                                leaves["xyz"])
        grads = torch.autograd.grad(loss, [leaves[k] for k in need]) if need else ()
    torch.cuda.synchronize()
    out = {"loss": loss.detach()}
    out.update(dict(zip(need, grads)))
    return out


def _oracle(case, device="cpu"):
    c = case.to(device)
    corre, conf = c.matches()
    return po.loss_and_grads(c.abspose, c.depth, c.xyz, c.K, corre, conf, c.h, c.width)


def _check(label, ours, ref, rtol=RTOL):
    """Same non-finite pattern (NaN where NaN), then the element-wise relative criterion on the finite elements."""
    a = ours.detach().double().cpu().numpy().reshape(-1)
    b = np.asarray(ref.detach().cpu().numpy() if torch.is_tensor(ref) else ref, np.float64).reshape(-1)
    assert a.shape == b.shape, label
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert (fa == fb).all(), f"{label}: finite mismatch at {np.argwhere(fa != fb)[:8].reshape(-1).tolist()}"
    assert (np.isnan(a) == np.isnan(b)).all(), f"{label}: NaN mismatch"
    if fa.any():
        rms = float(np.sqrt(np.mean(b[fb] ** 2)))
        ratio = np.abs(a[fa] - b[fa]) / (np.abs(b[fa]) + rms + 1e-300)
        print(f"[pose-loss] {label}: worst ratio {ratio.max():.2e} over {fa.sum()} elements")
        assert ratio.max() <= rtol, f"{label}: worst ratio {ratio.max():.3e} at {int(np.argmax(ratio))}"


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases_match_the_oracle_and_the_reference_float32_record(name):
    z = load_golden()
    case = golden_case(z, name)
    ours, orc = _ours(case), _oracle(case)
    _check(f"{name} loss vs oracle", ours["loss"], orc["loss"])
    _check(f"{name} loss vs f32 record", ours["loss"], z[f"{name}/f32/loss"])
    for k in GRADS:
        _check(f"{name} dL/d{k} vs oracle", ours[k], orc[k])
        _check(f"{name} dL/d{k} vs f32 record", ours[k], z[f"{name}/f32/grad_{k}"])


SEEDED = [  # (b, v, h, w, min matches, max matches)
    (1, 2, 7, 9, 0, 3), (2, 3, 32, 32, 0, 50), (3, 4, 40, 24, 1, 300), (4, 4, 64, 64, 100, 400),
    (14, 3, 256, 256, 500, 2047),
]


@pytest.mark.parametrize("b,v,h,w,nmin,nmax", SEEDED)
def test_seeded_cases_match_the_oracle(b, v, h, w, nmin, nmax):
    case = seeded_case(b, v, h, w, nmin, nmax, seed=b * 100 + v * 10 + h)
    ours, orc = _ours(case), _oracle(case, DEV)
    _check(f"seeded {b}x{v}x{h}x{w} loss", ours["loss"], orc["loss"])
    for k in GRADS:
        _check(f"seeded {b}x{v}x{h}x{w} dL/d{k}", ours[k], orc[k])


def test_unmatched_nan_poisons_only_what_the_reference_poisons_and_keeps_other_bits():
    z = load_golden()
    name = "v3_b1_nan_depth_unmatched"
    bad = golden_case(z, name)
    clean = golden_case(z, name)
    k = int(np.flatnonzero(np.isnan(bad.depth.numpy().reshape(-1)))[0])
    clean.depth.view(-1)[k] = 2.0
    ob, oc = _ours(bad), _ours(clean)
    assert torch.equal(_bits(ob["loss"]), _bits(oc["loss"]))            # no match reads the pixel
    for g in ("xyz", "w", "conf"):
        assert torch.equal(_bits(ob[g]), _bits(oc[g])), g
    gd_b, gd_c = ob["depth"].reshape(-1), oc["depth"].reshape(-1)
    assert torch.isnan(gd_b[k]) and torch.isnan(gd_b).sum() == 1
    keep = torch.arange(gd_b.numel(), device=DEV) != k
    assert torch.equal(_bits(gd_b[keep]), _bits(gd_c[keep]))
    ga = ob["abspose"][0]
    assert torch.isfinite(ga[0]).all() and torch.isnan(ga[1]).all() and torch.isnan(ga[2]).all()


def test_out_of_range_index_is_never_read_and_poisons_only_its_segment():
    case = seeded_case(2, 3, 16, 16, 3, 20, seed=5)
    bad = seeded_case(2, 3, 16, 16, 3, 20, seed=5)
    s = 4  # scene 1, pair (0, 2)
    o = int(np.sum(case.counts[:s]))
    bad.id_a[o + 1] = 16 * 16
    bad.id_c[o] = -3
    c, b = case.to(DEV), bad.to(DEV)

    def terms(x):
        corre, conf = x.matches()
        return losses.pose_terms(x.abspose, x.depth, x.xyz, x.K, corre, conf, x.h, x.width)

    L3c, L2c = terms(c)
    L3b, L2b = terms(b)
    assert torch.isnan(L3b[s]) and torch.isnan(L2b[s])
    keep = torch.arange(L3c.numel(), device=DEV) != s
    assert torch.equal(L3b[keep], L3c[keep]) and torch.equal(L2b[keep], L2c[keep])
    # gradients: scene 0 is untouched
    og = _ours(bad)
    assert torch.isfinite(og["abspose"][0]).all() and torch.isfinite(og["xyz"][0]).all()
    assert torch.isnan(og["conf"][1, 1])


def test_bit_identical_across_runs_and_streams():
    case = seeded_case(14, 3, 256, 256, 500, 2047, seed=11)
    r1, r2 = _ours(case), _ours(case)
    side = torch.cuda.Stream()
    r3 = _ours(case, stream=side)
    for k in ("loss",) + GRADS:
        assert torch.equal(_bits(r1[k]), _bits(r2[k])), k
        assert torch.equal(_bits(r1[k]), _bits(r3[k])), k


def test_forward_and_backward_do_not_synchronise_with_the_host():
    case = seeded_case(4, 4, 64, 64, 100, 400, seed=3).to(DEV)
    leaves = [case.abspose.clone().requires_grad_(True), case.depth.clone().requires_grad_(True),
              case.xyz.clone().requires_grad_(True)]
    corre, conf = case.matches()
    img = torch.zeros(case.b, case.v, 3, case.h, case.width, device=DEV)
    batch = {"context": {"image": img}, "target": {"image": img, "intrinsics": case.K}}
    relpose = torch.eye(4, device=DEV).repeat(case.b, 6, 1, 1)
    _ours(case)  # warm up: library load, allocator, pinned pool
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = losses.pose_loss(batch, (relpose, leaves[0]), (leaves[1],), (corre, None, conf), leaves[2])
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(torch.isfinite(t.grad).all() for t in leaves)


def test_only_requested_gradients_are_computed_and_they_keep_their_bits():
    case = seeded_case(3, 4, 40, 24, 1, 300, seed=9)
    full = _ours(case)
    for need in (("depth",), ("xyz",), ("abspose",), ("w", "conf"), ("abspose", "depth")):
        part = _ours(case, need=need)
        for k in need:
            assert torch.equal(_bits(part[k]), _bits(full[k])), (need, k)


def test_intrinsics_that_require_grad_are_refused():
    case = seeded_case(1, 3, 8, 8, 1, 4, seed=2).to(DEV)
    corre, conf = case.matches()
    img = torch.zeros(1, 3, 3, 8, 8, device=DEV)
    batch = {"context": {"image": img}, "target": {"image": img, "intrinsics": case.K.clone().requires_grad_(True)}}
    with pytest.raises(ValueError, match="intrinsics"):
        losses.pose_loss(batch, (None, case.abspose), (case.depth,), (corre, None, conf), case.xyz)


def test_no_matches_at_all():
    case = seeded_case(2, 3, 8, 8, 0, 0, seed=4)
    ours, orc = _ours(case), _oracle(case)
    assert float(ours["loss"]) == 0.0 == float(orc["loss"])
    for k in ("abspose", "depth", "xyz", "conf"):
        assert (ours[k] == 0).all(), k
