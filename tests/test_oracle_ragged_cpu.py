"""Pins the C oracle (oracle/gs_oracle.c, through OracleRender) against the autograd restatement (oracle/torch_oracle.py)
in fp64 on the frames and lists the GPU backward tests of tests/test_gpu_backward_paths.py use it for: frames whose sides
are not multiples of the 16-pixel tile (nor of the backward compositor's 8 x 4 warp block) -- down to one smaller than a
tile and ones a single pixel high -- with Gaussians straddling the last row and column; and one tile list longer than
8192 entries (the shared-memory sort's capacity) whose pixels' last contributors sit near its end.

Same criteria as tests/test_oracle_gradients.py: images within 1e-9, radii equal, every gradient (means2D included) within
1e-5 of its tensor's max-abs."""
import numpy as np
import pytest
import torch

from oracle import torch_oracle
from oracle.gs_oracle import OracleRender
from tests.regimes import edge_straddle_scene, long_list_scene
from tests.util import view_args


def _relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def edge_contributors(orc, mask) -> np.ndarray:
    """bool[P]: Gaussians that the oracle composites into some pixel of `mask` -- alpha >= 1/255 there, at a list
    position before that pixel's n_contrib (so not behind an early termination)."""
    hit = np.zeros(orc.P, bool)
    xy, co, pl, rg = orc.xy.astype(np.float64), orc.conic_opacity.astype(np.float64), orc.point_list, orc.ranges
    gx = (orc.W + 15) // 16
    for y, x in zip(*np.nonzero(mask)):
        s, e = rg[(y // 16) * gx + x // 16]
        ids = pl[s:s + min(e - s, int(orc.n_contrib[y, x]))]
        dx, dy = xy[ids, 0] - x, xy[ids, 1] - y
        power = -0.5 * (co[ids, 0] * dx * dx + co[ids, 2] * dy * dy) - co[ids, 1] * dx * dy
        alpha = np.minimum(0.99, co[ids, 3] * np.exp(np.minimum(power, 0.0)))
        hit[ids[(power <= 0) & (alpha >= 1 / 255)]] = True
    return hit


def _pin(sc, v, geometry, seed):
    """C oracle vs autograd on view v with seeded incoming colour and depth gradients.  Returns the C oracle's render and
    its gradients."""
    st, kw = view_args(sc, v, use_sh=geometry != "rgb_cov")
    if geometry == "sh_scalerot":
        kw.pop("cov3D_precomp")
        kw["scales"] = sc.scales.numpy()
        kw["rotations"] = sc.rotations.numpy()
    kw = {k: np.asarray(a, np.float64) for k, a in kw.items()}
    r = OracleRender(st, dtype=np.float64, with_depth=True, **kw)
    H, W = sc.image_shape
    rng = np.random.default_rng(seed)
    dL = rng.standard_normal((3, H, W)) / (H * W)
    dLd = rng.standard_normal((H, W)) / (H * W)
    g = r.backward(dL, dLd)

    tk = {k: torch.tensor(a, requires_grad=True) for k, a in kw.items()}
    m2d = torch.zeros(kw["means3D"].shape[0], 3, dtype=torch.float64, requires_grad=True)
    color, radii, depth = torch_oracle.render(st, means2D=m2d, with_depth=True, **tk)
    assert np.abs(color.detach().numpy() - r.color).max() < 1e-9
    assert (radii.numpy() == r.radii).all()
    assert np.abs(depth.detach().numpy() - r.depth).max() < 1e-8
    ((color * torch.tensor(dL)).sum() + (depth * torch.tensor(dLd)).sum()).backward()
    for name, t in tk.items():
        err = _relerr(g[name], t.grad.numpy().reshape(np.asarray(g[name]).shape))
        assert err < 1e-5, (name, err)
    err = _relerr(g["means2D"], m2d.grad.numpy())
    assert err < 1e-5, ("means2D", err)
    return r, g


# (H, W): 37 x 53 and 17 x 130 leave partial tiles, warp columns and warp rows; 100 x 9 a 9-wide frame (one full warp
# column and one of a single pixel); 5 x 7 is smaller than one tile and than one warp block; 1 x 40 is one pixel high
# (make_scene's camera stays well defined: tanfov does not depend on the frame, and the footprints are merely tall).
RAGGED = [((37, 53), "sh_cov"), ((17, 130), "sh_scalerot"), ((100, 9), "rgb_cov"), ((5, 7), "sh_cov"),
          ((1, 40), "sh_scalerot"), ((33, 250), "sh_cov")]


@pytest.mark.parametrize("hw,geometry", RAGGED, ids=[f"{h}x{w}-{g}" for (h, w), g in RAGGED])
def test_c_oracle_matches_autograd_on_ragged_frames(hw, geometry):
    H, W = hw
    sc = edge_straddle_scene(200, 60, 2, H, W, seed=11)
    for v in range(2):
        r, g = _pin(sc, v, geometry, seed=20 + v)
        # Gaussians reaching the last column / the last row get gradient from there
        for label, mask in (("column", np.s_[:, W - 1]), ("row", np.s_[H - 1, :])):
            m = np.zeros(hw, bool)
            m[mask] = True
            edge = edge_contributors(r, m)
            assert edge.sum() >= 5, (label, int(edge.sum()))
            assert (np.abs(g["opacities"][edge, 0]) > 0).all(), label
        assert r.num_rendered > 100


def test_c_oracle_matches_autograd_beyond_the_shared_memory_sort():
    """One 16 x 16 tile, 10 000 faint splats: the tile list is longer than 8192 entries and every pixel's last
    contributor lies beyond position 8192, while its transmittance stays above 0.1."""
    sc = long_list_scene(10000, 1, 16, 16, seed=1)
    r, g = _pin(sc, 0, "sh_cov", seed=5)
    n = r.ranges[0, 1] - r.ranges[0, 0]
    print(f"[regime] long list: tile list {n}, n_contrib {r.n_contrib.min()}..{r.n_contrib.max()}, "
          f"final_T >= {r.final_T.min():.3f}")
    assert n > 8192 and r.n_contrib.max() > 8192 and np.median(r.n_contrib) > 8192
    assert r.final_T.min() > 0.05
