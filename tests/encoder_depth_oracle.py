"""fp64 NumPy restatement of the encoder's depth glue (pf3plat_b200.encoder_depth), and an exact float32 restatement of
the mono cue's bin choice.

- depth_update_forward / _backward: encoder_costvolume.py:265, :285-287 (get_scaleshift) and the unprojections
  :304-307 / :506-528, with PyTorch's bilinear source index (align_corners=False) and clamp's backward mask.
- mono_bins_f32: :292-298 in float32 as the reference rounds it (hypotheses, the ÷4 downsample, |d - h_k|, the first
  minimum; a NaN counts as smallest).
- pdf_peak_forward / _backward: depth_predictor_multiview.py:379-384, the argmax tied to the lowest index.
"""
import numpy as np
import torch

SHIFT_LIMIT = 5.0


def bilinear_taps(out, inp, scale=None):
    """per destination index: (i0, i1, l0, l1) of PyTorch's bilinear source index, in fp64"""
    scale = inp / out if scale is None else scale
    src = np.maximum(scale * (np.arange(out) + 0.5) - 0.5, 0.0)
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < inp - 1)
    l1 = src - i0
    return i0, i1, 1.0 - l1, l1


def clamp(x, lo, hi):
    """torch.clamp with tensor bounds: NaN propagates"""
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(x), x, np.minimum(np.maximum(x, lo), hi))


def upsample_shift(ss, grid, h, w):
    """channel 1 of scale_shift [b, v, gh gw, 2], bilinearly upsampled to [b v, h, w] (unclamped)"""
    gh, gw = grid
    b, v = ss.shape[:2]
    s = np.asarray(ss, np.float64)[..., 1].reshape(b * v, gh, gw)
    y0, y1, hy0, hy1 = bilinear_taps(h, gh)
    x0, x1, wx0, wx1 = bilinear_taps(w, gw)
    top = wx0[None, None] * s[:, y0][:, :, x0] + wx1[None, None] * s[:, y0][:, :, x1]
    bot = wx0[None, None] * s[:, y1][:, :, x0] + wx1[None, None] * s[:, y1][:, :, x1]
    return hy0[None, :, None] * top + hy1[None, :, None] * bot


def directions(K, h, w):
    """K^-1 [(x + 1/2) / w, (y + 1/2) / h, 1] per item: [b v, 3, h, w]"""
    K = np.asarray(K, np.float64).reshape(-1, 3, 3)
    u, v = (np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h
    uv1 = np.stack([np.broadcast_to(u[None], (h, w)), np.broadcast_to(v[:, None], (h, w)), np.ones((h, w))])
    return np.einsum("nij,jhw->nihw", np.linalg.inv(K), uv1)


def depth_update_forward(depth, ss, K, near, far, grid):
    b, v = np.shape(near)
    h, w = np.shape(depth)[-2:]
    lo = np.asarray(near, np.float64).reshape(-1, 1, 1)
    hi = np.asarray(far, np.float64).reshape(-1, 1, 1)
    d0 = clamp(np.asarray(depth, np.float64)[:, 0], lo, hi)
    sraw = upsample_shift(ss, grid, h, w)
    pre = d0 + clamp(sraw, -SHIFT_LIMIT, SHIFT_LIMIT)
    depths = clamp(pre, lo, hi)
    xyz = directions(K, h, w) * depths[:, None]
    return depths[:, None], xyz.reshape(b, v, 3, h, w), (sraw, pre, lo, hi)


def depth_update_backward(depth, ss, K, near, far, grid, g_depths, g_xyz):
    b, v = np.shape(near)
    h, w = np.shape(depth)[-2:]
    gh, gw = grid
    _, _, (sraw, pre, lo, hi) = depth_update_forward(depth, ss, K, near, far, grid)
    g = np.zeros((b * v, h, w)) if g_depths is None else np.asarray(g_depths, np.float64).reshape(b * v, h, w).copy()
    if g_xyz is not None:
        g += (np.asarray(g_xyz, np.float64).reshape(b * v, 3, h, w) * directions(K, h, w)).sum(1)
    with np.errstate(invalid="ignore"):
        mask = (pre >= lo) & (pre <= hi) & (sraw >= -SHIFT_LIMIT) & (sraw <= SHIFT_LIMIT)
    g = np.where(mask, g, 0.0)
    y0, y1, hy0, hy1 = bilinear_taps(h, gh)
    x0, x1, wx0, wx1 = bilinear_taps(w, gw)
    out = np.zeros((b * v, gh, gw))
    for ys, hy in ((y0, hy0), (y1, hy1)):
        for xs, wx in ((x0, wx0), (x1, wx1)):
            contrib = g * hy[None, :, None] * wx[None, None, :]
            np.add.at(out, (slice(None), ys[:, None], xs[None, :]), contrib)
    d = np.zeros((b, v, gh * gw, 2))
    d[..., 1] = out.reshape(b, v, gh * gw)
    return d


def linspace_table():
    """torch.linspace(0, 1, 128) as the CPU computes it, the table the reference copies to the device"""
    return torch.linspace(0.0, 1.0, 128).numpy()


def hypotheses_f32(near00, far00):
    """h_k = fl32(a + fl32(lin_k fl32(B))), a = fl32(1 / far), B = (double)fl32(1 / near) - (double)a"""
    f32 = np.float32
    a = f32(1.0) / f32(far00)
    B = f32(float(f32(1.0) / f32(near00)) - float(a))
    return (a + linspace_table() * B).astype(np.float32)


def downsample4_f32(depths):
    """F.interpolate(bilinear, align_corners=False) by exactly ÷4 in float32: taps 4i+1, 4i+2 at weight 1/2"""
    d = np.asarray(depths, np.float32)[:, 0]
    a, b = d[:, 1::4, 1::4], d[:, 1::4, 2::4]
    c, e = d[:, 2::4, 1::4], d[:, 2::4, 2::4]
    h = np.float32(0.5)
    return h * (h * a + h * b) + h * (h * c + h * e)


def mono_bins_f32(depths, near, far, b, v):
    """the index of the one in the mono cue, [(v b), h/4, w/4] int64"""
    hyp = hypotheses_f32(np.asarray(near)[0, 0], np.asarray(far)[0, 0])
    dn = downsample4_f32(depths)
    with np.errstate(invalid="ignore"):
        diff = np.abs(dn[:, None] - hyp[None, :, None, None]).astype(np.float32)
    bins = np.argmin(diff, axis=1)  # the first minimum; NumPy, as torch.argmin, takes the first NaN as the minimum
    h4, w4 = bins.shape[-2:]
    return bins.reshape(b, v, h4, w4).transpose(1, 0, 2, 3).reshape(v * b, h4, w4)


def mono_cue_f32(depths, near, far, b, v):
    bins = mono_bins_f32(depths, near, far, b, v)
    return (np.arange(128)[None, :, None, None] == bins[:, None]).astype(np.float32)


def _peak(logits):
    x = np.asarray(logits, np.float64)
    with np.errstate(invalid="ignore"):
        kmax = np.argmax(np.where(np.isnan(x), np.inf, x), axis=1)  # a NaN wins (its pixel is NaN anyway)
        m = np.take_along_axis(x, kmax[:, None], 1)
        e = np.exp(x - m)
    p = 1.0 / e.sum(1)
    return p, kmax, e


def nearest_up(a, s):
    return np.repeat(np.repeat(a, s, axis=-2), s, axis=-1)


def pdf_peak_forward(logits, s):
    p, _, _ = _peak(logits)
    return nearest_up(p, s)[:, None]


def pdf_peak_backward(logits, s, g_out):
    p, kmax, e = _peak(logits)
    n, D, h, w = np.shape(logits)
    G = np.asarray(g_out, np.float64)[:, 0].reshape(n, h, s, w, s).sum((2, 4))
    pk = e * p[:, None]
    delta = (np.arange(D)[None, :, None, None] == kmax[:, None]).astype(np.float64)
    return (G * p)[:, None] * (delta - pk)
