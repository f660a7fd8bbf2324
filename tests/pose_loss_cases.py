"""Inputs of the pose-loss tests: the golden cases of tests/golden/pose_loss.npz and seeded cases up to PF3plat's
training shape, as the objects Losspose.forward receives."""
import math
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pose_loss.npz")
GOLDEN_CASES = ("v2_b1_16x20", "v3_b2_ragged", "v4_b3_24x24", "v4_b1_zero_weights", "v2_b2_edges",
                "v3_b1_nan_depth_unmatched", "v3_b1_inf_depth_unmatched", "v3_b2_nonfinite_depth_matched",
                "v3_b1_nan_xyz_unmatched")
# cases added later (tests/test_gpu_pose_loss_regimes.py): more views, signed and clamped weights, non-finite weights,
# confidences, intrinsics and poses, one-pixel-high and one-pixel-wide frames
NEW_GOLDEN_CASES = ("v5_b2_ragged", "v6_b1_ragged", "v3_b1_signed_weights", "v3_b2_clamp",
                    "v3_b2_nonfinite_weights_conf", "v3_b2_nonfinite_K", "v3_b2_nonfinite_pose0",
                    "v3_b2_nonfinite_pose1", "v3_b1_1x37", "v3_b1_37x1")
GRADS = ("abspose", "depth", "xyz", "w", "conf")


def pairs_of(v):
    return [(a, c) for a in range(v) for c in range(a + 1, v)]


class Case:
    """abspose [b,v,4,4], depth [b*v,1,h,w], xyz [b,v,3,h,w], K [b,v,3,3], w [M], conf [b,P]; the matches as packed
    int64 index arrays with per-segment counts (scene-major, then pair)."""

    def __init__(self, abspose, depth, xyz, K, id_a, id_c, w, counts, conf, h, width):
        self.abspose, self.depth, self.xyz, self.K = abspose, depth, xyz, K
        self.id_a, self.id_c, self.w, self.counts, self.conf = id_a, id_c, w, counts, conf
        self.b, self.v = abspose.shape[:2]
        self.h, self.width = h, width

    def to(self, device, dtype=None):
        f = lambda t: t.to(device=device, dtype=dtype or t.dtype)
        return Case(f(self.abspose), f(self.depth), f(self.xyz), f(self.K), self.id_a.to(device), self.id_c.to(device),
                    f(self.w), self.counts, f(self.conf), self.h, self.width)

    def matches(self, w=None, conf=None):
        """-> (corr[0], corr[2]) of Losspose: {(a, c): [(id_a, id_c, w)] * b}, {(a, c): [b]}; w / conf override the
        case's (e.g. leaves that require grad; slices of them keep the graph)."""
        w = self.w if w is None else w
        conf = self.conf if conf is None else conf
        pairs = pairs_of(self.v)
        off = np.concatenate([[0], np.cumsum(self.counts)])
        corre = {pr: [] for pr in pairs}
        s = 0
        for _ in range(self.b):
            for pr in pairs:
                o0, o1 = int(off[s]), int(off[s + 1])
                corre[pr].append((self.id_a[o0:o1], self.id_c[o0:o1], w[o0:o1]))
                s += 1
        return corre, {pr: conf[:, k] for k, pr in enumerate(pairs)}


def golden_case(z, name) -> Case:
    t = lambda k: torch.from_numpy(z[f"{name}/{k}"])
    b, v, h, w = (int(z[f"{name}/{k}"]) for k in ("b", "v", "height", "width"))
    return Case(t("abspose"), t("depth").reshape(b * v, 1, h, w), t("xyz"), t("K"), t("id_a"), t("id_c"), t("w"),
                z[f"{name}/counts"], t("conf"), h, w)


def load_golden():
    return np.load(GOLDEN)


def _rotation(g, angle):
    k = torch.randn(3, generator=g, dtype=torch.float64)
    k = k / k.norm()
    K = torch.tensor([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def seeded_case(b, v, h, w, n_min, n_max, seed) -> Case:
    """Random small-rotation poses, normalised intrinsics, depth in [1.5, 4], xyz ~ N(0, 1); per segment a random
    number of matches in [n_min, n_max], half of them consistent with the projection (both Huber regimes)."""
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    abspose = torch.eye(4, dtype=torch.float64).repeat(b, v, 1, 1)
    for i in range(b):
        for j in range(v):
            abspose[i, j, :3, :3] = _rotation(g, 0.15 * float(u(1)))
            abspose[i, j, :3, 3] = 0.2 * (u(3) - 0.5)
    K = torch.zeros(b, v, 3, 3, dtype=torch.float64)
    K[..., 0, 0], K[..., 1, 1] = 0.9 + 0.2 * u(b, v), 0.9 + 0.2 * u(b, v)
    K[..., 0, 2], K[..., 1, 2] = 0.45 + 0.1 * u(b, v), 0.45 + 0.1 * u(b, v)
    K[..., 2, 2] = 1.0
    depth = 1.5 + 2.5 * u(b * v, 1, h, w)
    xyz = torch.randn(b, v, 3, h, w, generator=g, dtype=torch.float64)
    P = len(pairs_of(v))
    counts = torch.randint(n_min, n_max + 1, (b * P,), generator=g).numpy()
    M = int(counts.sum())
    id_a = torch.randint(0, h * w, (M,), generator=g)
    id_c = torch.randint(0, h * w, (M,), generator=g)
    # half the matches: q = a pixel next to p (the small-motion regime of real correspondences)
    near = torch.rand(M, generator=g) < 0.5
    id_c = torch.where(near, (id_a + torch.randint(-1, 2, (M,), generator=g)).clamp(0, h * w - 1), id_c)
    wts = torch.rand(M, generator=g, dtype=torch.float64)
    conf = 0.2 + 0.8 * u(b, P)
    return Case(abspose.float(), depth.float(), xyz.float(), K.float(), id_a, id_c, wts.float(), counts, conf.float(),
                h, w)
