"""PF3plat's photometric training loss on the device (csrc/gs_losses.cu).

Every PF3plat training config trains with `loss: [lpips, mse, multissim, pose]`.  This module covers the two
photometric terms:
  * `ssim`  -- drop-in for `ssim` of PF3plat's src/loss/loss_multissim.py:57-65 (one scale of SSIM despite the module's
               name: zero-padded 11x11 Gaussian window, sigma 1.5, population covariance, no clipping);
  * `photometric_loss` -- `LossMse` (loss_mse.py:35) + `LossMultiSSIM` (loss_multissim.py:41-43) in one forward and one
               backward kernel, each term already weighted as the reference logs it (`loss/mse`, `loss/MultiSSIM`).
Both are differentiable with respect to both images.  LPIPS is `pf3plat_b200.lpips.LPIPS`.  The fourth term:
  * `pose_loss` -- `Losspose` (src/loss/loss_pose.py:29-129), the correspondence loss, in one forward and one backward
               pass over the matches (csrc/gs_pose_loss.cu), taking the objects `Losspose.forward` receives.
Inputs must be float32 CUDA tensors; there is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import _capi

_WINDOW = 11


def _layout(t: torch.Tensor):
    """-> (tensor to read, n images, (c, h, w), floats between images).  (n,c,h,w) or (b,v,c,h,w) inputs whose (c,h,w)
    blocks are contiguous and whose batch dimensions collapse to one stride (e.g. color[:, 1:-1] with b == 1, or any
    contiguous tensor) are read in place; anything else is copied to a contiguous tensor first."""
    if t.dim() not in (4, 5):
        raise ValueError(f"expected a (n, c, h, w) or (b, v, c, h, w) tensor, got shape {tuple(t.shape)}")
    lead, chw = t.shape[:-3], t.shape[-3:]
    n = 1
    for s in lead:
        n *= s
    if n == 0:
        return t, 0, tuple(chw), 0
    numel = chw[0] * chw[1] * chw[2]
    block_ok = t[(0,) * len(lead)].is_contiguous()
    dims = [(s, st) for s, st in zip(lead, t.stride()[:-3]) if s != 1]
    stride = dims[-1][1] if dims else numel
    collapses = all(dims[i][1] == dims[i + 1][0] * dims[i + 1][1] for i in range(len(dims) - 1))
    if not (block_ok and collapses and stride >= numel):
        t = t.contiguous()
        stride = numel
    return t, n, tuple(chw), stride


def _check(a: torch.Tensor, b: torch.Tensor):
    if not (torch.is_tensor(a) and torch.is_tensor(b)) or a.shape != b.shape or a.dim() not in (4, 5):
        raise ValueError("expected two tensors of the same (n, c, h, w) or (b, v, c, h, w) shape")
    if a.device.type != "cuda" or b.device != a.device:
        raise RuntimeError("pf3plat_b200.losses needs both images on the same CUDA device (there is no CPU fallback)")
    if a.dtype != torch.float32 or b.dtype != torch.float32:
        raise TypeError(f"pf3plat_b200.losses needs float32 images, got {a.dtype} and {b.dtype}")


def _config(n, chw, sp, sg):
    c, h, w = chw
    return _capi.GsLossConfig(batch=n, channels=c, height=h, width=w, pred_stride=sp, gt_stride=sg, with_mse=1)


class _Photometric(torch.autograd.Function):
    """(pred, gt) -> per-image (ssim, mse), each (n,); one forward and one backward kernel for both."""

    @staticmethod
    def forward(ctx, pred, gt):
        p, n, chw, sp = _layout(pred)
        g, _, _, sg = _layout(gt)
        cfg = _config(n, chw, sp, sg)
        L = _capi.lib()
        dev = pred.device
        ssim = torch.empty((n,), dtype=torch.float32, device=dev)
        mse = torch.empty((n,), dtype=torch.float32, device=dev)
        if n:
            with torch.cuda.device(dev):
                nbytes = int(L.gs_photometric_scratch_bytes(cfg))
                scratch = torch.empty((max(1, nbytes // 8),), dtype=torch.float64, device=dev)
                _capi.check(L.gs_photometric_forward(cfg, p.data_ptr(), g.data_ptr(), scratch.data_ptr(), ssim.data_ptr(),
                                                     mse.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(pred, gt)
        ctx.set_materialize_grads(False)
        return ssim, mse

    @staticmethod
    def backward(ctx, d_ssim, d_mse):
        pred, gt = ctx.saved_tensors
        need_p, need_g = ctx.needs_input_grad[:2]
        if not (need_p or need_g) or (d_ssim is None and d_mse is None):
            return None, None
        p, n, chw, sp = _layout(pred)
        g, _, _, sg = _layout(gt)
        cfg = _config(n, chw, sp, sg)
        dev = pred.device
        # incoming gradients go to the kernel as device arrays (an expanded grad of .mean() has stride 0)
        ds = d_ssim.to(torch.float32).contiguous() if d_ssim is not None else None
        dm = d_mse.to(torch.float32).contiguous() if d_mse is not None else None
        gp = torch.empty(pred.shape, dtype=torch.float32, device=dev) if need_p else None
        gg = torch.empty(gt.shape, dtype=torch.float32, device=dev) if need_g else None
        if n:
            ptr = lambda t: t.data_ptr() if t is not None else None
            with torch.cuda.device(dev):
                _capi.check(_capi.lib().gs_photometric_backward(cfg, p.data_ptr(), g.data_ptr(), ptr(ds), ptr(dm), ptr(gp),
                                                                ptr(gg), None, torch.cuda.current_stream(dev).cuda_stream))
        return gp, gg


def _per_image(img1, img2):
    _check(img1, img2)
    s, m = _Photometric.apply(img1, img2)
    lead = img1.shape[:-3]
    return s.reshape(lead), m.reshape(lead)


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    """`ssim` of loss_multissim.py:57-65: the mean SSIM over (n, c, h, w) if size_average, else the mean per image,
    shape (n,) (or (b, v) for (b, v, c, h, w) inputs).  Differentiable with respect to both images."""
    if window_size != _WINDOW:
        raise ValueError(f"only window_size=11 is implemented (the reference's default), got {window_size}")
    s, _ = _per_image(img1, img2)
    return s.mean() if size_average else s


def photometric_loss(prediction: torch.Tensor, target: torch.Tensor, mse_weight: float = 1.0, ssim_weight: float = 0.1):
    """-> (mse_term, ssim_term) = (mse_weight * mean((prediction - target)^2), ssim_weight * (1 - ssim(prediction, target))),
    i.e. LossMse and LossMultiSSIM of PF3plat with its default weights (config/loss/mse.yaml, multissim.yaml).  Pass
    `color[:, 1:-1]` and `image[:, 1:-1]` as the reference's losses do."""
    s, m = _per_image(prediction, target)
    return mse_weight * m.mean(), ssim_weight * (1.0 - s.mean())


def pose_pairs(v: int):
    """The view pairs of Losspose, in its order (loss_pose.py:47)."""
    return [(a, c) for a in range(v) for c in range(a + 1, v)]


def _f32(t: torch.Tensor, what: str) -> torch.Tensor:
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise RuntimeError(f"pose_loss needs {what} as a CUDA tensor (there is no CPU fallback)")
    if t.dtype != torch.float32:
        raise TypeError(f"pose_loss needs float32 {what}, got {t.dtype}")
    return t.contiguous()


def _pinned_upload(values, dtype, dev):
    host = torch.tensor(values, dtype=dtype).pin_memory()
    return host.to(dev, non_blocking=True)


class _PoseLoss(torch.autograd.Function):
    """(T [S,16], depth [b*v,h,w], xyz [b,v,3,h,w], w [M], conf [S]; constants) -> per-segment (L3 [S], L2 [S])."""

    @staticmethod
    def forward(ctx, T, depth, xyz, w, conf, kinv_a, k_c, seg, offsets, id_a, id_c, dims):
        b, v, h, wd, S, M = dims
        cfg = _capi.GsPoseLossConfig(batch=b, views=v, height=h, width=wd, segments=S, matches=M)
        ins = _capi.GsPoseLossInputs(T=T.data_ptr(), kinv_a=kinv_a.data_ptr(), k_c=k_c.data_ptr(), conf=conf.data_ptr(),
                                     seg=seg.data_ptr(), offsets=offsets.data_ptr(), id_a=id_a.data_ptr(),
                                     id_c=id_c.data_ptr(), w=w.data_ptr(), depth=depth.data_ptr(), xyz=xyz.data_ptr())
        dev = T.device
        L3 = torch.empty((S,), dtype=torch.float32, device=dev)
        L2 = torch.empty((S,), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_pose_loss_forward(cfg, ins, L3.data_ptr(), L2.data_ptr(),
                                                         torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(T, depth, xyz, w, conf, kinv_a, k_c, seg, offsets, id_a, id_c)
        ctx.dims = dims
        ctx.set_materialize_grads(False)
        return L3, L2

    @staticmethod
    def backward(ctx, d3, d2):
        T, depth, xyz, w, conf, kinv_a, k_c, seg, offsets, id_a, id_c = ctx.saved_tensors
        need = ctx.needs_input_grad[:5]
        if not any(need) or (d3 is None and d2 is None):
            return (None,) * 12
        b, v, h, wd, S, M = ctx.dims
        dev = T.device
        cfg = _capi.GsPoseLossConfig(batch=b, views=v, height=h, width=wd, segments=S, matches=M)
        ins = _capi.GsPoseLossInputs(T=T.data_ptr(), kinv_a=kinv_a.data_ptr(), k_c=k_c.data_ptr(), conf=conf.data_ptr(),
                                     seg=seg.data_ptr(), offsets=offsets.data_ptr(), id_a=id_a.data_ptr(),
                                     id_c=id_c.data_ptr(), w=w.data_ptr(), depth=depth.data_ptr(), xyz=xyz.data_ptr())
        # incoming gradients go to the kernel as device arrays (an expanded grad of .mean() has stride 0)
        g3 = d3.to(torch.float32).contiguous() if d3 is not None else None
        g2 = d2.to(torch.float32).contiguous() if d2 is not None else None
        outs = [torch.empty(t.shape, dtype=torch.float32, device=dev) if n else None
                for t, n in zip((T, depth, xyz, w, conf), need)]
        ptr = lambda t: t.data_ptr() if t is not None else None
        grads = _capi.GsPoseLossGrads(dL_dT=ptr(outs[0]), dL_ddepth=ptr(outs[1]), dL_dxyz=ptr(outs[2]),
                                      dL_dw=ptr(outs[3]), dL_dconf=ptr(outs[4]))
        L = _capi.lib()
        with torch.cuda.device(dev):
            scratch = None
            if need[1] or need[2]:
                nbytes = int(L.gs_pose_loss_scratch_bytes(cfg))
                if nbytes < 0:
                    _capi.check(-1)
                scratch = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dev)
            _capi.check(L.gs_pose_loss_backward(cfg, ins, ptr(g3), ptr(g2), grads, ptr(scratch),
                                                torch.cuda.current_stream(dev).cuda_stream))
        return tuple(outs) + (None,) * 7


def pose_terms(abspose, depth, xyz_h, intrinsics, matches, conf, h: int, w: int):
    """-> per-segment (L3, L2), each (b * pairs,), scene-major then pair in `pose_pairs(v)` order.

    abspose [b, v, 4, 4] (c2w[1]); depth [b*v, 1, h, w] or [b*v, h, w]; xyz_h [b, v, 3, h, w]; intrinsics [b, v, 3, 3]
    (data, not differentiated); matches {(a, c): [(id_a, id_c, w)] * b} with int64 flat pixel indices; conf
    {(a, c): [b]}.  Differentiable with respect to abspose, depth, xyz_h, the match weights and conf."""
    b, v = abspose.shape[:2]
    pairs = pose_pairs(v)
    P = len(pairs)
    if intrinsics.requires_grad:
        raise ValueError("pose_loss treats the intrinsics as data: it has no gradient for them (detach them first)")
    dev = abspose.device
    abspose = _f32(abspose, "c2w[1]")
    depth = _f32(depth, "depth[0]")
    xyz = _f32(xyz_h, "xyz_h")
    K = _f32(intrinsics, "intrinsics")
    if depth.numel() != b * v * h * w or tuple(xyz.shape) != (b, v, 3, h, w) or tuple(K.shape) != (b, v, 3, 3):
        raise ValueError(f"pose_loss: shapes disagree with b={b}, v={v}, h={h}, w={w}: depth {tuple(depth.shape)}, "
                         f"xyz_h {tuple(xyz.shape)}, intrinsics {tuple(K.shape)}")
    # T_s (get_relative_Rt, loss_pose.py:60-63): c2w[c] for a == 0, else c2w[c] @ inverse(c2w[a]).  inv_ex does not
    # wait for the device as inverse's error check does; integer-list indexing would upload an index, so none is used.
    inv = torch.linalg.inv_ex(abspose[:, 1:v - 1]).inverse if v > 2 else None  # the sources a > 0
    T = torch.stack([abspose[:, c] if a == 0 else abspose[:, c] @ inv[:, a - 1] for a, c in pairs], dim=1)
    Kinv = torch.linalg.inv_ex(K).inverse
    kinv_a = torch.stack([Kinv[:, a] for a, _ in pairs], dim=1).reshape(b * P, 9)
    k_c = torch.stack([K[:, c] for _, c in pairs], dim=1).reshape(b * P, 9)
    cf = _f32(torch.stack([conf[pr] for pr in pairs], dim=1), "conf").reshape(b * P)
    # the matches, scene-major then pair, one torch.cat per field
    trip = [matches[pr][i] for i in range(b) for pr in pairs]
    counts = [int(t[0].shape[0]) for t in trip]
    offsets = [0]
    for n in counts:
        offsets.append(offsets[-1] + n)
    M = offsets[-1]
    id_a = torch.cat([t[0].reshape(-1) for t in trip]).to(device=dev, dtype=torch.int64)
    id_c = torch.cat([t[1].reshape(-1) for t in trip]).to(device=dev, dtype=torch.int64)
    wts = _f32(torch.cat([t[2].reshape(-1) for t in trip]), "match weights")
    seg = _pinned_upload([[i, a, c] for i in range(b) for a, c in pairs], torch.int32, dev)
    off = _pinned_upload(offsets, torch.int64, dev)
    dims = (b, v, h, w, b * P, M)
    return _PoseLoss.apply(T.reshape(b * P, 16).contiguous(), depth, xyz, wts, cf, kinv_a, k_c, seg, off, id_a.contiguous(),
                           id_c.contiguous(), dims)


def pose_loss(batch, c2w, depth, corr, xyz_h, weight_2d: float = 0.005, weight_3d: float = 0.025) -> torch.Tensor:
    """`Losspose.forward(prediction, batch, gaussians, global_step, c2w, depth, corr, xyz_h)` of PF3plat
    (loss_pose.py:29-129) with its config's weights (config/loss/pose.yaml): weight_3d * mean(L3) + weight_2d * mean(L2)
    over every (scene, pair) segment, empty ones included.  `c2w[1]` is the absolute pose, `depth[0]` the
    [(b v), 1, h, w] depth, `corr[0][(a, c)]` the b (id_a, id_c, w) match lists and `corr[2][(a, c)]` the per-scene
    confidences; the relative-pose terms the reference computes and discards are not computed."""
    _, _, _, h, w = batch["context"]["image"].shape
    L3, L2 = pose_terms(c2w[1], depth[0], xyz_h, batch["target"]["intrinsics"], corr[0], corr[2], h, w)
    return L3.mean() * weight_3d + L2.mean() * weight_2d
