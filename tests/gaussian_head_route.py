"""The route an INTEGRATION.md section 4 user runs today for the stretch pf3plat_b200.gaussian_head replaces: the
reference's glue statements (depth_predictor_multiview.py:398-415, encoder_costvolume.py:509-540 and :556-573,
restated in torch on the device) around the repository's fused pf3plat_b200.adapter.GaussianAdapter, plus the input
handling of decoder_forward (the harmonics made contiguous in the rasterizer's layout, the 6-entry covariance gather).
Used by tests/test_gpu_gaussian_head.py and scripts/bench_gaussian_head.py."""
import torch
from einops import rearrange, repeat

from pf3plat_b200.adapter import GaussianAdapter
from pf3plat_b200.render import _cov6

_ADAPTERS = {}


def adapter_for(cfg, dev):
    key = (cfg.gaussian_scale_min, cfg.gaussian_scale_max, cfg.sh_degree, dev)
    if key not in _ADAPTERS:
        _ADAPTERS[key] = GaussianAdapter(cfg).to(dev)
    return _ADAPTERS[key]


def existing_route(raw, logits, depths, c2w, K, cfg, h, w):
    """-> (means, covariances, harmonics, opacities) as the encoder returns them"""
    b, V = c2w.shape[:2]
    v, dev = 2, raw.device
    raw_gaussians = rearrange(raw, "(v b) c h w -> b v (h w) c", v=v, b=b)                    # :398-400
    _, raw_densities = logits.split(1, dim=1)                                                  # :403-406
    densities = repeat(torch.sigmoid(raw_densities), "(v b) dpt h w -> b v (h w) srf dpt", b=b, v=v, srf=1)
    ys, xs = torch.meshgrid((torch.arange(h, device=dev) + 0.5) / h, (torch.arange(w, device=dev) + 0.5) / w,
                            indexing="ij")
    xy_ray = rearrange(torch.stack([xs, ys], -1), "h w xy -> (h w) () xy")                     # :509-510
    gaussians = rearrange(raw_gaussians, "... (srf c) -> ... srf c", srf=1)
    offset_xy = gaussians[..., :2].sigmoid()
    pixel_size = 1 / torch.tensor((w, h), dtype=torch.float32, device=dev)
    xy_ray = xy_ray + (offset_xy - 0.5) * pixel_size                                           # :518
    densities = densities[:, (0, -1)]
    opac = 0.5 * (1 - (1 - densities) ** 1 + densities ** (1 / 1))                            # :174-187, gpp = 1
    g = adapter_for(cfg, dev).forward(
        rearrange(c2w, "b v i j -> b v () () () i j")[:, (0, -1)],
        rearrange(K, "b v i j -> b v () () () i j")[:, (0, -1)],
        rearrange(xy_ray, "b v r srf xy -> b v r srf () xy")[:, (0, -1)],
        rearrange(depths, "(b v) 1 h w -> b v (h w) 1 1", b=b, v=V)[:, (0, -1)],
        opac,
        rearrange(gaussians[..., 2:], "b v r srf c -> b v r srf () c"),
        (h, w))
    return (rearrange(g.means[:, (0, -1)], "b v r srf spp xyz -> b (v r srf spp) xyz"),             # :556-573
            rearrange(g.covariances[:, (0, -1)], "b v r srf spp i j -> b (v r srf spp) i j"),
            rearrange(g.harmonics[:, (0, -1)], "b v r srf spp c d_sh -> b (v r srf spp) c d_sh"),
            rearrange(1 * g.opacities[:, (0, -1)], "b v r srf spp -> b (v r srf spp)"))


def decoder_inputs(means, covariances, harmonics, opacities):
    """what decoder_forward / render_views hand the rasterizer: (S, G, d_sh, 3) harmonics (contiguous: a copy unless
    they are the transposed view of such a buffer) and the 6-entry covariances"""
    return means.contiguous(), _cov6(covariances), harmonics.transpose(-1, -2).contiguous(), opacities.contiguous()
