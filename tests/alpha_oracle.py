"""The accumulated opacity alpha = 1 - T_final of a batched call, and its gradients, from the fp64 oracle by composition.

The rasterizer's oracles (oracle/gs_oracle.c, oracle/torch_oracle.py) return colour and depth only.  A render whose colours
are all 1 on a black background has 1 - T_final in every channel: C = sum_i alpha_i T_i = 1 - prod_i (1 - alpha_i), with the
same skip decisions, clamp and early stop as any other render of the same geometry.  So:
  * forward: alpha is channel 0 of `tests.batch_oracle.oracle_batch` with colors_precomp = 1 and bg = 0;
  * backward: the gradients are linear in the incoming gradients, so those of <dL_dcolor, colour> + <dL_dalpha, alpha> are
    the colour render's backward plus that render's backward with dL/dC = (dL_dalpha, 0, 0).  Its dL/dcolors (the
    constant colours') are discarded: alpha gives colours and SH nothing.
tests/test_alpha_cpu.py pins the composition to an autograd restatement and to finite differences."""
from __future__ import annotations

import numpy as np
import torch

from tests.batch_oracle import _np, oracle_batch

GEOMETRY = ("means3D", "means2D", "opacities", "scales", "rotations", "cov3D_precomp")


class AlphaOracle:
    """bs: BatchSettings with CPU tensors; ins: the Gaussian inputs of rasterize_batch.  `base` is the oracle of the colour
    (and depth) images -- `oracle_batch` in fp64 by default, or any object with `.color`, `.affected()` and `.backward(...)`
    returning per-input gradients (tests.sh4_oracle.ShOracleBatch, tests.depth_modes_oracle.DepthModeOracle).
    `alpha` [V,H,W], `frag` [V,H,W] (fragile alpha pixels); `backward(dL_dalpha, *base_args)` returns base.backward(*base_args)
    with the alpha terms added to the geometry gradients."""

    def __init__(self, bs, ins, base=None):
        V = int(bs.viewmatrix.shape[0])
        P = ins["means3D"].shape[1]
        self.V = V
        geo = {k: v for k, v in ins.items() if k not in ("shs", "colors_precomp")}
        self.ob_alpha = oracle_batch(bs._replace(bg=torch.zeros(V, 3, dtype=torch.float64), with_depth=False),
                                     colors_precomp=np.ones((V, P, 3)), dtype=np.float64, **geo)
        self.base = oracle_batch(bs, dtype=np.float64, **ins) if base is None else base
        self.alpha = self.ob_alpha.color[:, 0]
        self.frag = np.stack([r.px_fragile for r in self.ob_alpha.views])
        self.final_T = np.stack([r.final_T for r in self.ob_alpha.views])

    @property
    def color(self):
        return self.base.color

    def affected(self) -> np.ndarray:
        return self.base.affected() | self.ob_alpha.affected()

    def alpha_grads(self, dL_dalpha) -> dict:
        """The gradients of <dL_dalpha, alpha> alone (colors_precomp: None)."""
        dA = _np(dL_dalpha, np.float64)
        dC = np.zeros((self.V, 3) + dA.shape[1:])
        dC[:, 0] = dA
        g = self.ob_alpha.backward(dC)
        g["colors_precomp"] = None
        return g

    def backward(self, dL_dalpha, *base_args) -> dict:
        ga = self.alpha_grads(dL_dalpha)
        if not base_args:
            return ga
        g = self.base.backward(*base_args)
        for k in GEOMETRY:
            if g.get(k) is not None and ga.get(k) is not None:
                g[k] = g[k] + ga[k]
        return g
