"""fp64 restatement of the Gaussian head (pf3plat_b200.gaussian_head): depth_predictor_multiview.py:397-415,
encoder_costvolume.py:509-540 (with map_pdf_to_opacity, :174-187) and :556-573, for gaussians_per_pixel =
num_surfaces = 1.  NumPy inputs, float64 torch tensors inside so that the gradients come from autograd; the per-Gaussian
arithmetic is gaussian_adapter.py:60-92 restated with oracle/adapter_oracle.py's helpers, the Wigner-D blocks
as data.

Rounding the reference fixes in float32 even in a float64 run is kept: pixel_size = 1 / tensor((w, h), float32)
(encoder_costvolume.py:517 and gaussian_adapter.py:67).
"""
import numpy as np
import torch

from oracle import adapter_oracle
from pf3plat_b200.sh_rotation import sh_rotation_blocks

SCALE_MIN, SCALE_MAX = 0.5, 15.0


def sh_rotation(c2w, d_sh):
    """[b, 2, d_sh, d_sh]: the Wigner-D blocks of c2w[:, (0, -1), :3, :3] after the reference's guard (every determinant
    allclose to 1, else every camera uses the identity; NaN fails), in fp64"""
    rot = torch.as_tensor(np.asarray(c2w, np.float64))[:, (0, -1), :3, :3]
    ok = bool(torch.allclose(torch.det(rot), rot.new_tensor(1.0)))
    if not ok:
        rot = torch.eye(3, dtype=torch.float64).expand(rot.shape)
    return sh_rotation_blocks(rot, d_sh)


def head(raw, logits, depths, c2w, K, sh_degree, sh_rot=None, smin=SCALE_MIN, smax=SCALE_MAX, eps=1e-8):
    """float64 torch tensors (leaves may require grad) -> dict of means [b, G, 3], covariances [b, G, 3, 3], harmonics
    [b, G, 3, d_sh], opacities [b, G], G = 2 h w.  float32 tensors give the same statements in float32."""
    b, V = c2w.shape[:2]
    C, h, w = raw.shape[1:]
    hw, dt = h * w, raw.dtype
    r = raw.reshape(2, b, C, hw).permute(1, 0, 3, 2)                    # b v (h w) c
    u = (torch.arange(w, dtype=dt) + 0.5) / w
    v = (torch.arange(h, dtype=dt) + 0.5) / h
    grid = torch.stack(torch.meshgrid(u, v, indexing="xy"), -1).reshape(hw, 2)
    ps = torch.tensor(1.0 / np.array([w, h], np.float32), dtype=dt)
    xy = grid + (r[..., :2].sigmoid() - 0.5) * ps                          # [b, 2, hw, 2]
    sel = (0, V - 1)
    ext = c2w[:, sel][:, :, None]
    intr = K[:, sel][:, :, None]
    dep = depths.reshape(b, V, hw)[:, sel]
    q = logits.reshape(2, b, 2, hw)[:, :, 1].transpose(0, 1).sigmoid()     # [b, 2, hw]
    opac = 0.5 * ((1 - (1 - q)) + q)
    # gaussian_adapter.py:60-92 with oracle/adapter_oracle.py's helpers, pixel_size float32 as above
    d_sh = (sh_degree + 1) ** 2
    scales, rotations, sh = r[..., 2:].split((3, 4, 3 * d_sh), dim=-1)
    scales = smin + (smax - smin) * scales.sigmoid()
    multiplier = adapter_oracle.get_scale_multiplier(intr, ps)
    scales = scales * dep[..., None] * multiplier[..., None]
    rotations = rotations / (rotations.norm(dim=-1, keepdim=True) + eps)
    sh = sh.reshape(*sh.shape[:-1], 3, d_sh) * adapter_oracle.sh_mask(sh_degree).to(dt)
    rot = ext[..., :3, :3].detach()
    cov = rot @ adapter_oracle.build_covariance(scales, rotations) @ rot.transpose(-1, -2)
    origins, directions = adapter_oracle.get_world_rays(xy, ext, intr)
    means = origins + directions * dep[..., None]
    if sh_rot is not None:
        parts = []
        for degree in range(int(round(d_sh ** 0.5))):
            lo, hi = degree ** 2, (degree + 1) ** 2
            parts.append(torch.einsum("...ij,...j->...i", sh_rot[:, :, None, None, lo:hi, lo:hi], sh[..., lo:hi]))
        sh = torch.cat(parts, dim=-1)
    out = {"means": means, "covariances": cov, "harmonics": sh}
    d_sh = (sh_degree + 1) ** 2
    return {"means": out["means"].reshape(b, 2 * hw, 3), "covariances": out["covariances"].reshape(b, 2 * hw, 3, 3),
            "harmonics": out["harmonics"].reshape(b, 2 * hw, 3, d_sh), "opacities": opac.reshape(b, 2 * hw)}


INPUTS = ("raw", "logits", "depths", "c2w")
OUTPUTS = ("means", "covariances", "harmonics", "opacities")


def run(case, cot=None):
    """fp64 values, and the gradients into raw, logits, depths, c2w of sum_k <cot_k, out_k> when cot is given"""
    deg = int(case["sh_degree"])
    t = {k: torch.tensor(np.asarray(case[k], np.float64), requires_grad=cot is not None) for k in INPUTS}
    K = torch.tensor(np.asarray(case["K"], np.float64))
    sh = sh_rotation(case["c2w"], (deg + 1) ** 2) if deg > 0 else None
    out = head(t["raw"], t["logits"], t["depths"], t["c2w"], K, deg, sh)
    vals = {k: out[k].detach().numpy() for k in OUTPUTS}
    if cot is None:
        return vals, None
    loss = sum((torch.tensor(np.asarray(cot[k], np.float64)) * out[k]).sum() for k in OUTPUTS)
    loss.backward()
    return vals, {k: t[k].grad.numpy() for k in INPUTS}


def values32(case):
    """the same statements in float32, as the reference runs them: the yardstick for how far float32 alone lands from
    fp64 where a quantity is ill-conditioned (covariance entries that cancel between large scales)"""
    deg = int(case["sh_degree"])
    t = {k: torch.tensor(np.asarray(case[k]), dtype=torch.float32) for k in INPUTS}
    K = torch.tensor(np.asarray(case["K"]), dtype=torch.float32)
    sh = sh_rotation(case["c2w"], (deg + 1) ** 2).float() if deg > 0 else None
    out = head(t["raw"], t["logits"], t["depths"], t["c2w"], K, deg, sh)
    return {k: out[k].numpy() for k in OUTPUTS}
