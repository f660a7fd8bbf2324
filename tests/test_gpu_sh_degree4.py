"""GPU tests of the opt-in degree-4 SH evaluation (GsConfig.sh_eval_max_degree = 4): parity with the fp64 degree-4 oracle
(tests/sh4_oracle.py), every binning path and backward compositor, deterministic mode, the SH staging cases, the host
entry, the drop-in's process-wide setting and the adapter -> decoder chain."""
import ctypes

import numpy as np
import pytest
import torch

from pf3plat_b200 import _capi, rasterizer
from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene, make_target
from tests.batch_oracle import scene_batch_args
from tests.sh4_oracle import SH_BANDS4, ShOracleBatch, with_band4
from tests.util import check_grad, check_image_strict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _call(scenes, deg=4, tuning=0, use_scales=False, with_depth=False, views=None):
    cams, ins = scene_batch_args(scenes, device=DEV)
    h, w = scenes[0].image_shape
    bs = BatchSettings(image_height=h, image_width=w, sh_degree=4, with_depth=with_depth, tuning=tuning,
                       sh_eval_max_degree=deg, **cams)
    if use_scales:
        ins.pop("cov3D_precomp")
    else:
        ins.pop("scales"), ins.pop("rotations")
    return bs, ins


def _run(bs, ins, W=None, means2D=False, grads=True):
    leaves = {k: v.detach().requires_grad_(grads) for k, v in ins.items()}   # (views keep their addresses)
    m2d = None
    if means2D:
        m2d = torch.zeros(bs.viewmatrix.shape[0], ins["means3D"].shape[1], 3, device=DEV, requires_grad=True)
    out = rasterize_batch(bs, leaves["means3D"], leaves["opacities"], shs=leaves["shs"],
                          cov3D_precomp=leaves.get("cov3D_precomp"), scales=leaves.get("scales"),
                          rotations=leaves.get("rotations"), means2D=m2d)
    color = out[0]
    if grads:
        (color * W).sum().backward()
    g = {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in leaves.items()}
    if m2d is not None:
        g["means2D"] = m2d.grad.detach().clone()
    return color.detach(), out[1], g


@pytest.mark.parametrize("use_scales", [False, True])
def test_degree4_against_fp64_oracle(use_scales):
    sc = with_band4(make_scene(4000, 3, 64, 96, seed=11))
    bs, ins = _call([sc], use_scales=use_scales)
    W = torch.as_tensor(make_target(3, 64, 96).numpy() - 0.5, device=DEV)
    color, radii, g = _run(bs, ins, W, means2D=True)
    c3, _, _ = _run(bs._replace(sh_eval_max_degree=3), ins, grads=False)
    assert (color - c3).abs().max() > 1e-2      # band 4 really changes the image
    orc = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins.get("cov3D_precomp"),
                        scales=ins.get("scales"), rotations=ins.get("rotations"))
    for v in range(3):
        check_image_strict(color[v], orc.batch.views[v], 0.02, f"deg4 view {v}")
    assert np.array_equal(radii.cpu().numpy(), orc.radii)
    go = orc.backward(W.cpu().numpy())
    aff = orc.affected()[0]
    check_grad("shs", g["shs"][0], go["shs"][0], aff, bands=SH_BANDS4)
    assert go["shs"][0, :, 16:25].std() > 1e-4
    check_grad("means3D", g["means3D"][0], go["means3D"][0], aff)
    check_grad("opacities", g["opacities"][0], go["opacities"][0], aff)
    for v in range(3):
        check_grad(f"means2D view {v}", g["means2D"][v], go["means2D"][v], aff)
    if use_scales:
        check_grad("scales", g["scales"][0], go["scales"][0], aff)
        check_grad("rotations", g["rotations"][0], go["rotations"][0], aff)
    else:
        check_grad("cov3D", g["cov3D_precomp"][0], go["cov3D_precomp"][0], aff)


def test_degree4_pixel_aligned_cloud_sampled_views():
    """C5's shape (one Gaussian per pixel of two context views) at 256^2, two of its target views against the oracle."""
    sc = with_band4(make_pixel_aligned_scene(256, 256, 4, seed=2))
    bs, ins = _call([sc])
    W = torch.as_tensor(make_target(4, 256, 256).numpy() - 0.5, device=DEV)
    color, _, g = _run(bs, ins, W)
    keep = [0, 3]
    sub = lambda t: t[keep]
    bs2 = bs._replace(viewmatrix=sub(bs.viewmatrix), projmatrix=sub(bs.projmatrix), campos=sub(bs.campos),
                      bg=sub(bs.bg), tanfov=sub(bs.tanfov), view_scale=sub(bs.view_scale))
    orc = ShOracleBatch(bs2, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins["cov3D_precomp"])
    for j, v in enumerate(keep):
        check_image_strict(color[v], orc.batch.views[j], 0.05, f"C5 deg4 view {v}")


_PATHS = [0, _capi.GS_TUNE_NO_SPECULATION, _capi.GS_TUNE_NO_STRATA, _capi.GS_TUNE_SEPARATE_EMIT,
          _capi.GS_TUNE_NO_SPECULATION | _capi.GS_TUNE_FORCE_RADIX_BINNING, _capi.GS_TUNE_FWD_WS]


def test_degree4_every_binning_path_gives_the_same_image():
    sc = with_band4(make_scene(20000, 4, 96, 128, seed=4))
    ref = None
    for tuning in _PATHS:
        bs, ins = _call([sc], tuning=tuning)
        for _ in range(3):   # exact, trial and stratified calls of the speculative policy
            color, radii, _ = _run(bs, ins, grads=False)
            if ref is None:
                ref = (color, radii)
            assert torch.equal(color, ref[0]) and torch.equal(radii, ref[1]), tuning


def test_degree4_backward_compositors_and_determinism():
    sc = with_band4(make_scene(8000, 3, 64, 96, seed=6))
    W = torch.as_tensor(make_target(3, 64, 96).numpy() - 0.5, device=DEV)
    bs, ins = _call([sc])
    _, _, g0 = _run(bs, ins, W)
    for tuning in (_capi.GS_TUNE_BWD_V1, _capi.GS_TUNE_BWD_OCC4):
        _, _, g1 = _run(bs._replace(tuning=tuning), ins, W)
        for k in ("shs", "means3D", "opacities", "cov3D_precomp"):
            err = (g1[k] - g0[k]).abs().max() / g0[k].abs().max()
            assert err < 1e-4, (tuning, k, float(err))
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_run(bs, ins, W)[2] for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(False)
    for k in ("shs", "means3D", "opacities", "cov3D_precomp"):
        assert torch.equal(runs[0][k], runs[1][k]), k
        assert (runs[0][k] - g0[k]).abs().max() <= 1e-4 * g0[k].abs().max(), k
    assert runs[0]["shs"][..., 16:25, :].abs().max() > 0


@pytest.mark.parametrize("S,P", [(1, 4096), (1, 1001), (2, 4096), (2, 1001)])
def test_degree4_staging_cases(S, P):
    """Aligned (P % 4 == 0) and unaligned (P % 4 != 0: the second scene's block is not 16-byte aligned, and the ragged last
    CTA's block is not a multiple of 16 bytes) SH blocks; against the oracle."""
    scs = [with_band4(make_scene(P, 2, 48, 64, seed=30 + k), seed=40 + k) for k in range(S)]
    bs, ins = _call(scs)
    W = torch.as_tensor(np.concatenate([make_target(2, 48, 64, seed=k).numpy() for k in range(S)]) - 0.5, device=DEV)
    color, _, g = _run(bs, ins, W)
    orc = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins["cov3D_precomp"])
    for v in range(2 * S):
        check_image_strict(color[v], orc.batch.views[v], 0.03, f"S={S} P={P} view {v}")
    go = orc.backward(W.cpu().numpy())
    aff = orc.affected()
    for k in range(S):
        check_grad(f"shs scene {k}", g["shs"][k], go["shs"][k], aff[k], bands=SH_BANDS4)
        check_grad(f"means3D scene {k}", g["means3D"][k], go["means3D"][k], aff[k])
    # a block whose base address is only 4-byte aligned: the cp.async fallback of both kernels, same bits
    buf = torch.empty(ins["shs"].numel() + 1, device=DEV)
    shifted = buf[1:].view_as(ins["shs"])
    shifted.copy_(ins["shs"])
    assert shifted.data_ptr() % 16 != 0
    c2, _, g2 = _run(bs, dict(ins, shs=shifted), W)
    assert torch.equal(c2, color)
    # (the compositor's float atomics make the colour gradients differ in the last bits between two runs)
    assert (g2["shs"] - g["shs"]).abs().max() <= 1e-5 * g["shs"].abs().max()


def test_degree4_requests_that_evaluate_lower_degrees():
    sc = with_band4(make_scene(3000, 2, 48, 64, seed=8))
    bs, ins = _call([sc])
    default = bs._replace(sh_eval_max_degree=None)
    # sh_degree = 3 with the request for 4 is the default evaluation
    c_a, _, _ = _run(bs._replace(sh_degree=3), ins, grads=False)
    c_b, _, _ = _run(default._replace(sh_degree=3), ins, grads=False)
    assert torch.equal(c_a, c_b)
    # M = 16 with the request for 4 evaluates degree 3
    ins16 = dict(ins, shs=ins["shs"][:, :, :16].contiguous())
    c_c, _, _ = _run(bs, ins16, grads=False)
    c_d, _, _ = _run(default, ins16, grads=False)
    assert torch.equal(c_c, c_d)
    # values above 4 evaluate 4
    c_4, _, _ = _run(bs, ins, grads=False)
    c_9, _, _ = _run(bs._replace(sh_eval_max_degree=9), ins, grads=False)
    assert torch.equal(c_4, c_9)


def test_degree4_tuning_knobs():
    sc = with_band4(make_scene(3000, 2, 48, 64, seed=9))
    bs, ins = _call([sc])
    W = torch.ones(2, 3, 48, 64, device=DEV)
    color, _, _ = _run(bs, ins, grads=False)
    # the 16-byte staging (what gs_render_host's zero-copy feed uses) is supported: same bits
    c_raw, _, _ = _run(bs._replace(tuning=_capi.GS_TUNE_PRE_SH_RAW16), ins, grads=False)
    assert torch.equal(c_raw, color)
    with pytest.raises(ValueError, match="GS_TUNE_PRE_OCC6"):
        _run(bs._replace(tuning=_capi.GS_TUNE_PRE_OCC6), ins, grads=False)
    with pytest.raises(ValueError, match="GS_TUNE_PBWD_2PHASE"):
        _run(bs._replace(tuning=_capi.GS_TUNE_PBWD_2PHASE), ins, W)


def test_degree4_host_entry_matches_device_entry():
    P, V, hw = 20000, 3, (64, 80)
    sc = with_band4(make_scene(P, V, *hw, seed=12))
    bs, ins = _call([sc])
    c_dev, r_dev, _ = _run(bs, ins, grads=False)
    host = {k: v[0].cpu().contiguous() for k, v in ins.items()}
    cams = {"viewmatrix": bs.viewmatrix, "projmatrix": bs.projmatrix, "campos": bs.campos, "bg": bs.bg,
            "tanfov": bs.tanfov, "view_scale": bs.view_scale}
    cams = {k: v.cpu().contiguous() for k, v in cams.items()}
    cfg = _capi.GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M, cfg.sh_degree, cfg.sh_eval_max_degree = P, 1, V, 25, 4, 4
    cfg.image_height, cfg.image_width, cfg.scale_modifier = hw[0], hw[1], 1.0
    for k, t in cams.items():
        setattr(cfg, k, t.data_ptr())
    ctx = rasterizer.current_context(DEV)
    color = torch.empty(V, 3, *hw).pin_memory()
    radii = torch.empty(V, P, dtype=torch.int32).pin_memory()
    gout = _capi.GsOutputs(color=color.data_ptr(), radii=radii.data_ptr())
    pin = {k: v.pin_memory() for k, v in host.items()}
    for src in (host, pin):   # pageable: the copy engine's pieced upload; pinned: the zero-copy feeds
        gin = _capi.GsInputs(means3D=src["means3D"].data_ptr(), opacities=src["opacities"].data_ptr(),
                             shs=src["shs"].data_ptr(), cov3D_precomp=src["cov3D_precomp"].data_ptr())
        for tuning in ((0,) if src is host else (0, _capi.GS_TUNE_NO_SPLIT_COLOUR, _capi.GS_TUNE_NO_ZERO_COPY)):
            cfg.tuning = tuning
            for _ in range(2):
                color.zero_(); radii.zero_()
                _capi.check(_capi.lib().gs_render_host(ctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                       torch.cuda.current_stream(DEV).cuda_stream))
                assert torch.equal(color, c_dev.cpu()) and torch.equal(radii, r_dev.cpu()), tuning


def test_dropin_process_wide_setting():
    """GaussianRasterizer (the reference's per-view module) under set_sh_eval_max_degree(4) equals rasterize_batch at
    degree 4; a backward taken after the setting went back to 3 still differentiates degree 4."""
    from pf3plat_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    sc = with_band4(make_scene(3000, 1, 48, 64, seed=13))
    bs, ins = _call([sc])
    W = torch.as_tensor(make_target(1, 48, 64).numpy()[0] - 0.5, device=DEV)
    c_ref, r_ref, g_ref = _run(bs, ins, W[None])
    rs = GaussianRasterizationSettings(
        image_height=48, image_width=64, tanfovx=float(bs.tanfov[0, 0]), tanfovy=float(bs.tanfov[0, 1]), bg=bs.bg[0],
        scale_modifier=1.0, viewmatrix=bs.viewmatrix[0], projmatrix=bs.projmatrix[0], sh_degree=4, campos=bs.campos[0],
        prefiltered=False, debug=False)
    s = float(bs.view_scale[0])
    means = ins["means3D"][0].clone().requires_grad_(True)
    shs = ins["shs"][0].clone().requires_grad_(True)
    opac = ins["opacities"][0].clone().requires_grad_(True)
    assert rasterizer.get_sh_eval_max_degree() == 3
    rasterizer.set_sh_eval_max_degree(4)
    try:
        color, radii = GaussianRasterizer(rs)(means3D=means * s, means2D=None, opacities=opac, shs=shs,
                                              cov3D_precomp=ins["cov3D_precomp"][0] * (s * s))
    finally:
        rasterizer.set_sh_eval_max_degree(3)
    # (view scale applied in torch here, in the kernel there: equal to rounding)
    assert (color - c_ref[0]).abs().max() < 1e-5 and torch.equal(radii, r_ref[0])
    (color * W).sum().backward()
    assert shs.grad[:, 16:25].abs().max() > 0
    err = (shs.grad - g_ref["shs"][0]).abs().max() / g_ref["shs"][0].abs().max()
    assert err < 1e-4, float(err)
    with torch.no_grad():
        c3, _ = GaussianRasterizer(rs)(means3D=means * s, means2D=None, opacities=opac, shs=shs,
                                       cov3D_precomp=ins["cov3D_precomp"][0] * (s * s))
    assert (c3 - color).abs().max() > 1e-2   # the setting is back at 3


def test_decoder_forward_keyword_and_chain_gradient_reaches_band4():
    """decoder_forward(depth_mode="depth", sh_eval_max_degree=4) on poses that require grad: the band-4 columns of the
    harmonics receive a gradient that matches the oracle's, and the default keyword leaves them without one."""
    from pf3plat_b200.render import decoder_forward
    b, v, hw = 1, 2, (48, 64)
    sc = with_band4(make_scene(3000, v, *hw, seed=14))
    d = sc.to(DEV)
    ext = d.extrinsics[None].clone().requires_grad_(True)
    harm = d.harmonics[None].clone().requires_grad_(True)
    nr, fr = d.near[None], d.far[None]
    bg = torch.zeros(3, device=DEV)
    W = torch.as_tensor(make_target(v, *hw).numpy() - 0.5, device=DEV)
    color, depth = decoder_forward(d.means[None], d.covariances[None], harm, d.opacities[None], ext, d.intrinsics[None],
                                   nr, fr, hw, bg, depth_mode="depth", sh_eval_max_degree=4)
    ((color[0] * W).sum() + 1e-3 * depth.sum()).backward()
    g4 = harm.grad[0, :, :, 16:25].clone()
    assert ext.grad is not None and g4.abs().max() > 0
    bs, ins = _call([sc])
    orc = ShOracleBatch(bs, ins["means3D"], ins["opacities"], ins["shs"], deg=4, cov3D_precomp=ins["cov3D_precomp"])
    for k in range(v):
        check_image_strict(color[0, k], orc.batch.views[k], 0.03, f"decoder deg4 view {k}")
    go = orc.backward(W.cpu().numpy())
    check_grad("harmonics band 4", g4.permute(0, 2, 1), go["shs"][0, :, 16:25], orc.affected()[0])
    harm.grad = None
    color, _ = decoder_forward(d.means[None], d.covariances[None], harm, d.opacities[None], ext, d.intrinsics[None],
                               nr, fr, hw, bg, depth_mode="depth")
    (color[0] * W).sum().backward()
    assert not harm.grad[0, :, :, 16:25].any()
