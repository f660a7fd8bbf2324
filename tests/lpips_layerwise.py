"""Layer-by-layer checkers of csrc/gs_lpips.cu: each kernel against fp64 on the kernel's own inputs.

The end-to-end tests (tests/test_gpu_lpips.py, tests/test_gpu_lpips_bf16.py) compare the whole network with fp64 under a
bound taken from PyTorch's own error.  That bound cannot be tight: rounding activations to TF32 or BF16 flips ReLU signs
and max-pool argmaxes, and those decisions, not accumulation noise, set the end-to-end error.  So a kernel a few per cent
wrong in one layer passes there.  Here every kernel is checked where it acts:

  * `Plan` restates `make_plan`: where the forward leaves every activation and pooled map (NHWC, fp32 holding TF32
    values or bf16) in the caller's workspace, and which gradient buffer holds dL/dz0 after the backward;
  * `tf32_rna` / `bf16_rne` are the kernels' two storage roundings (`cvt.rna.tf32.f32`, `__float2bfloat16_rn`);
  * `layer_forward` is one layer in fp64 on the kernel's input activation and the weights as packed (TF32- or
    BF16-rounded; conv1_1's stay fp32, with the scaling layer in fp32 as the kernel does it);
  * `head_value` is the distance in fp64 on the kernel's taps;
  * `backward` reproduces `lpips_backward` step by step in fp64, conditioned on the kernel's forward: ReLU masks from its
    activations, pool routes from its pre-pool activations (first maximum, or last NaN), the head's closed form, and the
    storage rounding exactly where the kernels store a gradient.

`forward` chains `layer_forward`, so with `noise` (a relative perturbation of every sum before rounding, standing in for
fp32 accumulation order) and a `Mutant` it is a rounding-faithful model of the kernels, which is how
tests/test_lpips_layerwise_cpu.py shows what these checks see and what the end-to-end rule misses.  With `prec=None`
nothing is rounded and the whole thing is the fp64 network.

Criteria (the bounds are chosen from H100 measurements; DESIGN.md 5.10 records them):
  forward, per element   |ours - ref| <= u(ref) + GAMMA * sum_k |a_k w_k|      (u: one unit of the storage format)
                         plus the fraction of elements whose stored value differs from the rounded reference
  gradients              rel-L2 <= GRAD_REL[prec], and per element |a - b| <= GRAD_TAU[prec] (|b| + rms(b))
"""
from __future__ import annotations

import dataclasses

import torch
import torch.nn.functional as F

from oracle import lpips_oracle as lo

LAYERS, NTAPS = 13, 5
CIN = (3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512)
COUT = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
LEVEL = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)
TAP_OF = (-1, 0, -1, 1, -1, -1, 2, -1, -1, 3, -1, -1, 4)
TAP_LAYER = (1, 3, 6, 9, 12)
POOLED = (2, 4, 7, 10)  # layers whose input is a max-pool
EPS = 1e-10
HEAD_BLOCKS = 32
MANT_BITS = {"tf32": 10, "bf16": 7, "fp32": 23, None: 52}

# the bounds (DESIGN.md 5.10: measured worst values on an H100 and the headroom over them)
GAMMA = 2.0 ** -16          # forward: accumulation error per unit of sum |a w| (fp32 sums of up to 4608 products)
FLIP_MAX = {"tf32": 0.05, "bf16": 5e-3}       # fraction of stored activations that differ from the rounded reference
GRAD_REL = {"tf32": 2e-3, "bf16": 2e-2}       # rel-L2 of dL/dz0 and dL/din against the conditioned backward
GRAD_TAU = {"tf32": 2e-2, "bf16": 1.5e-1}       # element-wise |a - b| <= tau (|b| + rms(b)) for the same
HEAD_REL = 1e-6                                # distance against fp64 on the kernel's taps
CONV0_GAMMA = 2.0 ** -18                       # conv1_1 backward: |a - b| <= CONV0_GAMMA sum |w g| mul/scale + u32(b)


# ---------------------------------------------------------------------------------------------------------------------
# workspace layout (make_plan in csrc/gs_lpips.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _align256(n):
    return (n + 255) & ~255


@dataclasses.dataclass
class Plan:
    """Byte offsets of the workspace regions of GsLpipsConfig(batch=N, height=H, width=W, grads, precision)."""
    N: int
    H: int
    W: int
    grads: int
    prec: str

    def __post_init__(self):
        N, esize = self.N, self.esize
        self.nimg = 2 * N
        self.nb = (N if self.grads & 1 else 0) + (N if self.grads & 2 else 0)
        self.h = [self.H >> v for v in range(5)]
        self.w = [self.W >> v for v in range(5)]
        off = 0

        def take(elems):
            nonlocal off
            o = off
            off += _align256(elems * esize)
            return o

        self.act, self.pool, self.grad, self.ping = [None] * LAYERS, [], [None, None], [None, None]
        if self.grads:
            for l in range(LAYERS):
                v = LEVEL[l]
                if l in POOLED:
                    self.pool.append(take(self.nimg * self.h[v] * self.w[v] * CIN[l]))
                self.act[l] = take(self.nimg * self.h[v] * self.w[v] * COUT[l])
            self.grad = [take(self.nb * self.h[0] * self.w[0] * 64) for _ in range(2)]
        else:
            self.ping = [take(self.nimg * self.h[0] * self.w[0] * 64) for _ in range(2)]
        self.partial = off
        self.total = off + _align256(8 * NTAPS * N * HEAD_BLOCKS)

    @property
    def esize(self):
        return 2 if self.prec == "bf16" else 4

    @property
    def dtype(self):
        return torch.bfloat16 if self.prec == "bf16" else torch.float32

    def dz0_buffer(self):
        """Index of the gradient buffer holding dL/dz0 when k_conv0_bwd runs: lpips_backward's swaps replayed."""
        cur = 0
        for l in range(LAYERS - 1, 0, -1):
            if l not in POOLED:
                cur ^= 1
        return cur

    def _region(self, ws, off, shape):
        n = 1
        for s in shape:
            n *= s
        return ws[off:off + n * self.esize].view(self.dtype).reshape(shape)

    def act_nhwc(self, ws, l):
        v = LEVEL[l]
        return self._region(ws, self.act[l], (self.nimg, self.h[v], self.w[v], COUT[l]))

    def pool_nhwc(self, ws, k):
        v = LEVEL[POOLED[k]]
        return self._region(ws, self.pool[k], (self.nimg, self.h[v], self.w[v], CIN[POOLED[k]]))

    def dz0_nhwc(self, ws):
        return self._region(ws, self.grad[self.dz0_buffer()], (self.nb, self.h[0], self.w[0], 64))


def nchw64(t):
    """(n, h, w, c) NHWC of any float type -> (n, c, h, w) float64."""
    return t.permute(0, 3, 1, 2).to(torch.float64).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# storage roundings
# ---------------------------------------------------------------------------------------------------------------------
def tf32_rna(x: torch.Tensor) -> torch.Tensor:
    """float32 -> float32 holding a TF32 value: 10 explicit mantissa bits, ties away from zero (cvt.rna.tf32.f32).  NaN
    and Inf pass through; a carry runs into the exponent, so the largest finite values round to Inf."""
    assert x.dtype == torch.float32
    b = x.contiguous().view(torch.int32)
    finite = (b & 0x7F800000) != 0x7F800000
    r = torch.where(finite, (b + 0x1000) & ~0x1FFF, b)
    return r.view(torch.float32)


def bf16_rne(x: torch.Tensor) -> torch.Tensor:
    """float32 -> float32 holding a BF16 value: round to nearest, ties to even (__float2bfloat16_rn); NaN stays NaN."""
    assert x.dtype == torch.float32
    b = x.contiguous().view(torch.int32)
    nan = torch.isnan(x)
    r = (b + 0x7FFF + ((b >> 16) & 1)) & ~0xFFFF
    return torch.where(nan, b | 0x00400000, r).view(torch.float32)


def store(x: torch.Tensor, prec) -> torch.Tensor:
    """An fp64 value as a kernel stores it: fp32, then the storage rounding (prec None: unrounded fp64)."""
    if prec is None:
        return x
    f = x.to(torch.float32)
    return (tf32_rna(f) if prec == "tf32" else bf16_rne(f)).to(torch.float64)


def unit(x: torch.Tensor, prec) -> torch.Tensor:
    """One unit in the last place of the storage format at |x| (0 at 0)."""
    _, e = torch.frexp(x.abs())
    u = torch.ldexp(torch.ones_like(x), (e - 1 - MANT_BITS[prec]).to(torch.int32))
    return torch.where(x == 0, torch.zeros_like(x), u)


# ---------------------------------------------------------------------------------------------------------------------
# weights as the kernels read them
# ---------------------------------------------------------------------------------------------------------------------
class Weights:
    """The state dict as packed for `prec`: layers 1..12 rounded (TF32 rna or BF16 rne), conv1_1 fp32; fp64 tensors."""

    def __init__(self, sd, prec, device="cpu"):
        self.prec = prec
        convs = lo.conv_keys()
        self.w, self.b = [], []
        for l, (wk, bk) in enumerate(convs):
            w = sd[wk].to(device, torch.float32)
            self.w.append((w if l == 0 else store(w.double(), prec).float()).double())
            self.b.append(sd[bk].to(device, torch.float64))
        self.lin = [sd[k].to(device, torch.float32).reshape(-1).double() for k in lo.lin_keys()]
        self.shift = sd["scaling_layer.shift"].to(device, torch.float32).reshape(1, 3, 1, 1)
        self.scale = sd["scaling_layer.scale"].to(device, torch.float32).reshape(1, 3, 1, 1)

    def with_lin(self, keep):
        """A copy whose lin weights are zero except tap `keep`'s (None: all kept)."""
        c = object.__new__(Weights)
        c.__dict__.update(self.__dict__)
        c.lin = [v if keep is None or t == keep else torch.zeros_like(v) for t, v in enumerate(self.lin)]
        return c


@dataclasses.dataclass
class Mutant:
    """A deliberate error in the rounding-faithful model, in the place a kernel slip would put it."""
    fwd_weight: dict = dataclasses.field(default_factory=dict)   # layer -> fn(w (Cout, Cin, 3, 3)) for its forward
    fwd_bias: dict = dataclasses.field(default_factory=dict)     # layer -> fn(b) for its forward
    bwd_scale: dict = dataclasses.field(default_factory=dict)    # layer -> factor on its backward-data sums
    route_last_max: bool = False                                 # unpool to the last maximum of a window on ties
    head_no_proj: tuple = ()                                     # taps whose head backward loses the projection term
    conv0_bwd_factor: dict = dataclasses.field(default_factory=dict)  # input channel -> factor on dL/din


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
def scaled_input(x: torch.Tensor, W: Weights, normalize: bool) -> torch.Tensor:
    """k_conv0_fwd's input transform in IEEE fp32 (2x - 1, then (x - shift) / scale); x (n, 3, h, w) float32.  In fp64
    when nothing is rounded (W.prec None), as the fp64 network does it."""
    dt = torch.float64 if W.prec is None else torch.float32
    x = x.to(dt)
    if normalize:
        x = 2 * x - 1
    return (x - W.shift.to(dt)) / W.scale.to(dt)


def _perturb(z, noise):
    """z (1 + e), e uniform in [-noise, noise] from `noise`'s generator: (scale, torch.Generator) or None."""
    if noise is None:
        return z
    scale, gen = noise
    e = torch.rand(z.shape, generator=gen, dtype=torch.float64).to(z.device)
    return z * (1 + scale * (2 * e - 1))


def layer_forward(l, x, W: Weights, with_abs=False, mut: Mutant | None = None, noise=None):
    """Layer l in fp64 on its input x (NCHW; for l = 0 the scaled fp32 image): (stored activation, unrounded fp64
    activation, sum |a w| + |b| or None)."""
    w, b = W.w[l], W.b[l]
    if mut is not None:
        w = mut.fwd_weight.get(l, lambda t: t)(w)
        b = mut.fwd_bias.get(l, lambda t: t)(b)
    x = x.to(torch.float64)
    r = torch.relu(_perturb(F.conv2d(x, w, b, padding=1), noise))
    s = F.conv2d(x.abs(), W.w[l].abs(), W.b[l].abs(), padding=1) if with_abs else None
    return store(r, W.prec), r, s


def forward(x0, x1, W: Weights, normalize, mut: Mutant | None = None, noise=None):
    """The network on both images (2N, NCHW, fp64 values of what each kernel stores): (acts[13], pools[4], value (N,))."""
    x = scaled_input(torch.cat([x0, x1]), W, normalize)
    acts, pools = [], []
    cur = x
    for l in range(LAYERS):
        if l in POOLED:
            cur = F.max_pool2d(cur, 2, 2)
            pools.append(cur)
        cur = layer_forward(l, cur, W, mut=mut, noise=noise)[0]
        acts.append(cur)
    return acts, pools, head_value(acts, W, x0.shape[0])


def head_value(acts, W: Weights, N: int) -> torch.Tensor:
    """The distance (N,) in fp64 from the five taps (NCHW, 2N images)."""
    total = 0
    for t, l in enumerate(TAP_LAYER):
        f = acts[l].to(torch.float64)
        n = f / (f.pow(2).sum(1, keepdim=True).sqrt() + EPS)
        d = ((n[:N] - n[N:]) ** 2 * W.lin[t].reshape(1, -1, 1, 1)).sum(1)
        total = total + d.mean(dim=(1, 2))
    return total


# ---------------------------------------------------------------------------------------------------------------------
# conditioned backward
# ---------------------------------------------------------------------------------------------------------------------
def _mask(a):
    return ~(a <= 0)  # ReLU's backward: the gradient passes where act > 0 or act is NaN


def route(a: torch.Tensor, last_max=False) -> torch.Tensor:
    """Boolean (n, c, h, w): the element of each 2x2 window max_pool2d's backward routes to, PyTorch's scan
    `val > maxval || isnan(val)` (first maximum, or last NaN); the rows and columns a floor pool drops are False."""
    n, c, h, w = a.shape
    ho, wo = h // 2, w // 2
    q = [a[:, :, dy:2 * ho:2, dx:2 * wo:2] for dy in (0, 1) for dx in (0, 1)]
    m, k = q[0], torch.zeros_like(q[0], dtype=torch.int64)
    for j in (1, 2, 3):
        up = (q[j] >= m if last_max else q[j] > m) | torch.isnan(q[j])
        m, k = torch.where(up, q[j], m), torch.where(up, torch.full_like(k, j), k)
    r = torch.zeros(a.shape, dtype=torch.bool, device=a.device)
    for j, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        r[:, :, dy:2 * ho:2, dx:2 * wo:2] = k == j
    return r


def _upsample(gp, shape):
    u = torch.zeros(shape, dtype=gp.dtype, device=gp.device)
    ho, wo = gp.shape[2], gp.shape[3]
    u[:, :, :2 * ho, :2 * wo] = gp.repeat_interleave(2, 2).repeat_interleave(2, 3)
    return u


def head_backward(f, t, W: Weights, dout, N, i0, nb, prec, no_proj=False):
    """k_head_bwd: dL/df of images [i0, i0 + nb) of tap t (activation f, 2N images, NCHW) under its ReLU mask, stored."""
    HW = f.shape[2] * f.shape[3]
    idx = torch.arange(i0, i0 + nb, device=f.device)
    other = torch.where(idx < N, idx + N, idx - N)
    a, b = f[idx], f[other]
    s = a.pow(2).sum(1, keepdim=True).sqrt()
    na, nbn = s + EPS, b.pow(2).sum(1, keepdim=True).sqrt() + EPS
    sc = (2 * dout.to(f)[idx % N] / HW).reshape(-1, 1, 1, 1)
    n = a / na
    gn = sc * W.lin[t].reshape(1, -1, 1, 1) * (n - b / nbn)
    dot = (n * gn).sum(1, keepdim=True)
    proj = torch.where(s == 0, torch.zeros_like(s), dot * na / s)  # the limit at s = 0 (csrc/gs_lpips.cu, top)
    if no_proj:
        proj = torch.zeros_like(proj)
    df = (gn - n * proj) / na
    return store(torch.where(_mask(a), df, torch.zeros_like(df)), prec)


def conv0_backward(dz0, W: Weights, normalize, with_abs=False, mut: Mutant | None = None):
    """k_conv0_bwd in fp64: dL/dx = conv1_1's transposed convolution (fp32 weights) x mul / scale; and, with_abs, the
    same on |w| |g| (the scale of its rounding error)."""
    mul = 2.0 if normalize else 1.0
    sc = W.scale.to(torch.float64)
    d = F.conv_transpose2d(dz0, W.w[0], padding=1) * mul / sc
    if mut is not None and mut.conv0_bwd_factor:
        f = torch.ones(1, 3, 1, 1, dtype=d.dtype, device=d.device)
        for c, v in mut.conv0_bwd_factor.items():
            f[0, c] = v
        d = d * f
    s = F.conv_transpose2d(dz0.abs(), W.w[0].abs(), padding=1) * mul / sc if with_abs else None
    return d, s


def backward(acts, W: Weights, dout, N, i0, nb, normalize, mut: Mutant | None = None, noise=None):
    """lpips_backward on the kernel's activations (2N images, NCHW): (dL/dz0 of images [i0, i0 + nb), dL/dx of the same).
    Every stored gradient is rounded as the kernels round it (W.prec); `noise` perturbs each backward-data sum."""
    prec = W.prec
    mut = mut or Mutant()
    sel = slice(i0, i0 + nb)
    g = head_backward(acts[12], 4, W, dout, N, i0, nb, prec, 4 in mut.head_no_proj)
    for l in range(LAYERS - 1, 0, -1):
        d = _perturb(F.conv_transpose2d(g, W.w[l], padding=1), noise) * mut.bwd_scale.get(l, 1.0)
        below = acts[l - 1][sel]
        if l not in POOLED:
            g = store(torch.where(_mask(below), d, torch.zeros_like(d)), prec)
            continue
        gp = store(d, prec)
        t = TAP_OF[l - 1]
        h = head_backward(acts[l - 1], t, W, dout, N, i0, nb, prec, t in mut.head_no_proj)
        routed = route(below, mut.route_last_max) & _mask(below)
        g = torch.where(routed, store(h + _upsample(gp, h.shape), prec), h)
    return g, conv0_backward(g, W, normalize, mut=mut)[0]


# ---------------------------------------------------------------------------------------------------------------------
# criteria
# ---------------------------------------------------------------------------------------------------------------------
def forward_report(ours, ref, sabs, prec, gamma=GAMMA):
    """ours: stored activation; ref: unrounded fp64 activation on the same input; sabs: sum |a w| + |b|.
    -> worst |ours - ref| / (u(ref) + gamma sabs), and the fraction of elements that differ from store(ref)."""
    ours, ref = ours.to(torch.float64), ref.to(torch.float64)
    tol = unit(ref, prec) + gamma * sabs
    err = (ours - ref).abs()
    worst = float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0
    flips = float((ours != store(ref, prec)).double().mean()) if err.numel() else 0.0
    return {"worst_ratio": worst, "flip_frac": flips}


def conv0_report(din, dz0, W: Weights, normalize):
    """k_conv0_bwd alone: its dL/dx against fp64 of the kernel's own dL/dz0, per element
    |ours - ref| <= CONV0_GAMMA sum |w g| mul/scale + one fp32 unit -> worst ratio."""
    ref, s = conv0_backward(dz0.to(torch.float64), W, normalize, with_abs=True)
    tol = CONV0_GAMMA * s + unit(ref, "fp32")
    return float(((din.to(torch.float64) - ref).abs() / tol.clamp_min(1e-300)).max())


def rel_l2(a, b):
    nb = float(b.norm())
    return float((a - b).norm()) / nb if nb > 0 else float((a - b).norm())


def grad_report(ours, ref, prec):
    """rel-L2 over its bound and the worst element-wise |a - b| / (tau (|b| + rms(b))): both pass at <= 1."""
    ours, ref = ours.to(torch.float64), ref.to(torch.float64)
    rms = float(ref.pow(2).mean().sqrt())
    tau = GRAD_TAU[prec]
    elem = float(((ours - ref).abs() / (tau * (ref.abs() + rms))).max()) if rms > 0 else float((ours - ref).abs().max())
    rel = rel_l2(ours, ref)
    return {"rel": rel, "rel_ratio": rel / GRAD_REL[prec], "elem_ratio": elem}
