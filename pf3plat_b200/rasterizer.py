"""Host-side mirror of the reference's rasterizer operator, backed by the C ABI (include/gsplat_b200.h).

Surface replaced: the `diff_gaussian_rasterization` module PF3plat imports
(PF3plat's src/model/decoder/cuda_splatting.py:5-8) -- `GaussianRasterizationSettings` (12-field
NamedTuple, constructed at :99-112 and :192-205) and `GaussianRasterizer` (nn.Module called with keywords at
:117-124 and :210-217, returning the 2-tuple `(color, radii)`).  Same names, argument meaning and error
behaviour; PyTorch is used for device memory, streams and autograd plumbing only.

`rasterize_batch` is the batched form of the same operator (V views of S scenes per call) used by
`pf3plat_b200.render`; the per-view reference call is its S = V = 1 case.
"""
from __future__ import annotations

import atexit
import ctypes
import math
import threading
from typing import NamedTuple, Optional

import torch
from torch import nn

from . import _capi
from ._capi import GsConfig, GsInGrads, GsInputs, GsOutGrads, GsOutputs, GsStats, GsSyncFreeWorkspace


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


# ---------------------------------------------------------------------------------------------------------
# contexts: one GsContext per (device, stream)
# ---------------------------------------------------------------------------------------------------------
_contexts: dict[tuple[int, int], ctypes.c_void_p] = {}
_locks: dict[tuple[int, int], threading.RLock] = {}
_registry_lock = threading.Lock()


def _key(device: torch.device, stream_ptr: int) -> tuple[int, int]:
    return (device.index if device.index is not None else torch.cuda.current_device(), stream_ptr)


def _context(device: torch.device, stream_ptr: int) -> ctypes.c_void_p:
    key = _key(device, stream_ptr)
    with _registry_lock:
        ctx = _contexts.get(key)
        if ctx is None:
            ctx = ctypes.c_void_p()
            _capi.check(_capi.lib().gs_context_create(ctypes.byref(ctx)))
            _contexts[key] = ctx
            _locks[key] = threading.RLock()
    return ctx


def _context_lock(device: torch.device, stream_ptr: int) -> threading.RLock:
    """A GsContext serves one call at a time (include/gsplat_b200.h): the forward of one thread and the backward the
    autograd engine runs on another take this lock around their gs_* calls."""
    _context(device, stream_ptr)
    return _locks[_key(device, stream_ptr)]


def trim_memory(device=None) -> None:
    """Hands the cached blocks of every context's private memory pool on `device` (all devices if None) back to the
    driver -- the counterpart of torch.cuda.empty_cache() for the memory this library holds outside torch's allocator."""
    with _registry_lock:
        items = list(_contexts.items())
    for (dev_index, _), ctx in items:
        if device is None or torch.device(device).index in (None, dev_index):
            with torch.cuda.device(dev_index):
                _capi.check(_capi.lib().gs_context_trim(ctx))


def destroy_contexts() -> None:
    """Destroys every cached GsContext (registered with atexit; also usable from tests)."""
    with _registry_lock:
        items = list(_contexts.items())
        _contexts.clear()
        _locks.clear()
    for (dev_index, _), ctx in items:
        try:
            with torch.cuda.device(dev_index):
                _capi.lib().gs_context_destroy(ctx)
        except Exception:
            pass


atexit.register(destroy_contexts)


def current_context(device=None) -> ctypes.c_void_p:
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        return _context(device, torch.cuda.current_stream(device).cuda_stream)


def last_stats(device=None) -> dict:
    st = GsStats()
    _capi.check(_capi.lib().gs_get_stats(current_context(device), ctypes.byref(st)))
    return {k: getattr(st, k) for k, _ in GsStats._fields_ if not k.endswith("_")}


def set_profiling(enabled: bool, device=None) -> None:
    _capi.check(_capi.lib().gs_set_profiling(current_context(device), int(enabled)))


def stage_ms(device=None) -> dict:
    arr = (ctypes.c_float * _capi.GS_NUM_STAGES)()
    _capi.check(_capi.lib().gs_get_stage_ms(current_context(device), arr))
    return dict(zip(_capi.STAGE_NAMES, [float(x) for x in arr]))


class SyncFreeWorkspace:
    """Caller-owned memory of the sync-free rasterizer path (gs_forward_sync_free / gs_backward_sync_free, DESIGN.md
    5.18): one torch-allocated byte buffer that holds the saved state, the tile lists of at most `instance_capacity`
    tile instances and all scratch of one forward and its backward.  Passing it as `workspace=` to `rasterize_batch` or
    `render.decoder_forward` selects that path: the host never waits for the device, the library allocates nothing and
    reads nothing back, so the call can be captured in a CUDA graph.  While a call needs no more instances than the
    capacity, its outputs are the default path's; past it, colour, depth and alpha are NaN and the backward's gradients
    too (a NaN-skipping optimizer step then skips the step), and status() reports it.

    The shape (scenes, views, Gaussians per scene, image) is fixed.  `depth`, `alpha` and `camera_grad` say which
    outputs and gradients calls may ask for, `deterministic` whether their backward may run under
    torch.use_deterministic_algorithms(True); `buffer` (optional) is a uint8 CUDA tensor, 256-byte aligned, of at least
    `nbytes` to use instead of a new allocation.  The workspace belongs to one forward at a time: the backward of a
    forward whose workspace a later forward has reused raises RuntimeError when run eagerly (a CUDA graph replay does
    not run that check)."""

    def __init__(self, device, scenes: int, views: int, gaussians_per_scene: int, image_shape, instance_capacity: int, *,
                 depth: bool = False, alpha: bool = False, deterministic: bool = False, camera_grad: bool = False,
                 buffer: Optional[torch.Tensor] = None):
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError(f"SyncFreeWorkspace needs a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        h, w = (int(x) for x in image_shape)
        self.dims = (int(scenes), int(views), int(gaussians_per_scene), h, w)
        self.instance_capacity = int(instance_capacity)
        self.depth, self.alpha = bool(depth), bool(alpha)
        self.deterministic, self.camera_grad = bool(deterministic), bool(camera_grad)
        self.nbytes = sync_free_workspace_bytes(*self.dims, self.instance_capacity, deterministic=self.deterministic,
                                                camera_grad=self.camera_grad)
        if buffer is None:
            buffer = torch.empty(self.nbytes, dtype=torch.uint8, device=device)
        elif buffer.device != device or buffer.dtype != torch.uint8 or not buffer.is_contiguous():
            raise ValueError(f"buffer must be a contiguous uint8 tensor on {device}")
        elif buffer.numel() < self.nbytes or buffer.data_ptr() % 256:
            raise ValueError(f"buffer must hold {self.nbytes} bytes at a 256-byte aligned address")
        self.buffer = buffer
        self.device = device
        self.generation = 0   # forwards run on it (the eager reuse check of the backward)
        self._ws = GsSyncFreeWorkspace(buffer.data_ptr(), buffer.numel(), self.instance_capacity)
        self.clear_status()

    def status(self) -> tuple:
        """(required_instances, exceeded): the most tile instances any forward since the last clear_status() needed, and
        whether any of them exceeded the capacity.  Synchronises with the device."""
        words = self.buffer[:32].view(torch.int32).cpu().tolist()
        return words[5] & 0xffffffff, bool(words[4])

    def clear_status(self) -> None:
        """Resets the status words (stream-ordered; graph-capturable)."""
        self.buffer[:32].zero_()

    def _check(self, dev, S, V, P, H, W, with_depth, with_alpha, camera) -> None:
        if dev != self.device:
            raise ValueError(f"the workspace is on {self.device}, the inputs on {dev}")
        if (S, V, P, H, W) != self.dims:
            raise ValueError(f"the workspace was sized for (scenes, views, gaussians, height, width) = {self.dims}, "
                             f"the call has {(S, V, P, H, W)}")
        for wanted, have, name in ((with_depth, self.depth, "depth"), (with_alpha, self.alpha, "alpha"),
                                   (camera, self.camera_grad, "camera_grad")):
            if wanted and not have:
                raise ValueError(f"the call needs a workspace created with {name}=True")


def sync_free_workspace_bytes(scenes: int, views: int, gaussians_per_scene: int, height: int, width: int,
                              instance_capacity: int, *, deterministic: bool = False, camera_grad: bool = False) -> int:
    """Bytes of a SyncFreeWorkspace (gs_sync_free_workspace_bytes); ValueError for a bad shape or capacity."""
    cfg = GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.image_height, cfg.image_width = (int(gaussians_per_scene), int(scenes), int(views),
                                                              int(height), int(width))
    needs = ((_capi.GS_SYNC_FREE_DETERMINISTIC if deterministic else 0) |
             (_capi.GS_SYNC_FREE_CAMERA_GRAD if camera_grad else 0))
    out = ctypes.c_int64()
    _capi.check(_capi.lib().gs_sync_free_workspace_bytes(ctypes.byref(cfg), int(instance_capacity), needs,
                                                         ctypes.byref(out)))
    return out.value


def sync_free_capacity(margin: float = 1.5, device=None) -> int:
    """An instance capacity for a SyncFreeWorkspace: the tile instances of the last default forward on this device and
    stream (last_stats()["num_rendered"]) times `margin`."""
    n = last_stats(device)["num_rendered"]
    if n < 0:
        raise RuntimeError("the last forward on this context did not report its tile instances (a sync-free call)")
    return int(math.ceil(n * float(margin)))


class _SavedHandle:
    """Owns a GsSaved*; released on the stream of the forward when the autograd graph lets go of it."""

    def __init__(self, ctx, ptr, stream_ptr, device):
        self.ctx, self.ptr, self.stream_ptr, self.device = ctx, ptr, stream_ptr, device

    def __del__(self):
        try:
            if self.ptr:
                with torch.cuda.device(self.device):
                    _capi.lib().gs_saved_free(self.ctx, self.ptr, self.stream_ptr)
                self.ptr = None
        except Exception:
            pass


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _f32c(t: Optional[torch.Tensor], device=None) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if device is not None and t.device != device:
        t = t.to(device)
    return t.detach().to(torch.float32).contiguous()


class BatchSettings(NamedTuple):
    """GaussianRasterizationSettings for V views at once (see include/gsplat_b200.h: GsConfig)."""
    image_height: int
    image_width: int
    viewmatrix: torch.Tensor                 # (V,4,4) transposed
    projmatrix: torch.Tensor                 # (V,4,4) transposed
    campos: torch.Tensor                     # (V,3)
    bg: torch.Tensor                         # (V,3)
    sh_degree: int
    tanfov: Optional[torch.Tensor] = None    # (V,2) device tensor, or
    tanfovx: float = 0.0                     # one host pair for all views
    tanfovy: float = 0.0
    view_scale: Optional[torch.Tensor] = None  # (V,)
    scale_modifier: float = 1.0
    prefiltered: bool = False
    with_depth: bool = False
    debug: bool = False
    tuning: int = 0                          # GS_TUNE_* knobs (testing)
    # highest SH degree evaluated (GsConfig.sh_eval_max_degree): 3, or 4 to evaluate and train band 4 of a 25-coefficient
    # block; None = the process-wide setting (set_sh_eval_max_degree)
    sh_eval_max_degree: Optional[int] = None
    # also differentiate the cameras: a viewmatrix, projmatrix, campos or tanfov that requires grad gets the full gradient
    # of every output (gs_backward_cam_tanfov) instead of the depth channel's z column alone; None = the process-wide
    # setting (set_camera_gradients, default off)
    camera_gradients: Optional[bool] = None
    # what the depth channel (with_depth) composites: PF3plat's DepthRenderingMode -- "depth" (camera-space z of the
    # view-scaled scene), "disparity", "relative_disparity" or "log" (f(z) of render_depth_cuda at the unscaled z)
    depth_mode: str = "depth"
    depth_near_far: Optional[torch.Tensor] = None  # (V,2) unscaled near, far: needed by "relative_disparity" and "log"
    # anti-aliasing (GS_FLAG_ANTIALIAS): the screen-space filter with opacity compensation -- each splat drawn at opacity
    # o * rho, rho = sqrt(det Sigma2 / det(Sigma2 + dilation I)) per (view, Gaussian); None = the process-wide setting
    # (set_antialiasing, default off)
    antialiasing: Optional[bool] = None
    # also return the accumulated opacity alpha = 1 - T_final (V,H,W) of the colour pass (GsAlpha); its gradient reaches
    # the geometry and the opacities, never SH, colours or cameras
    with_alpha: bool = False


# ---------------------------------------------------------------------------------------------------------
# highest SH degree evaluated, for callers that cannot pass BatchSettings (the drop-in GaussianRasterizer)
# ---------------------------------------------------------------------------------------------------------
_sh_eval_max_degree = 3


def set_sh_eval_max_degree(degree: int) -> None:
    """Process-wide highest SH degree the rasterizer evaluates when BatchSettings.sh_eval_max_degree is None: 3 (the
    default: bands 0..3, as upstream) or 4 (band 4 too, for 25-coefficient blocks such as PF3plat's adapter output).
    The degree evaluated is min(sh_degree, this, the largest degree the coefficients cover).  A forward's backward uses
    the degree that forward used, whatever the setting is by then."""
    global _sh_eval_max_degree
    _sh_eval_max_degree = _check_degree(degree)


def get_sh_eval_max_degree() -> int:
    return _sh_eval_max_degree


def _check_degree(degree) -> int:
    # (GsConfig.sh_eval_max_degree <= 0 selects the library default 3, so 0 cannot be expressed; sh_degree = 0 can)
    degree = int(degree)
    if degree < 1:
        raise ValueError(f"sh_eval_max_degree must be >= 1, got {degree}")
    return degree


def _resolve_degree(bs: BatchSettings) -> BatchSettings:
    """bs with sh_eval_max_degree and antialiasing made explicit (the process-wide settings in place of None)."""
    if bs.sh_eval_max_degree is None:
        bs = bs._replace(sh_eval_max_degree=_sh_eval_max_degree)
    if bs.antialiasing is None:
        bs = bs._replace(antialiasing=_antialiasing)
    if bs.camera_gradients is None:
        bs = bs._replace(camera_gradients=_camera_gradients)
    return bs


# ---------------------------------------------------------------------------------------------------------
# anti-aliasing, for callers that cannot pass BatchSettings (the drop-in GaussianRasterizer, an unmodified render_cuda)
# ---------------------------------------------------------------------------------------------------------
_antialiasing = False


def set_antialiasing(enabled: bool) -> None:
    """Process-wide anti-aliasing setting used when BatchSettings.antialiasing (or the `antialiasing` argument of the
    drop-in, render_views, decoder_forward) is None: False (the default, upstream's default behaviour) or True (the
    screen-space filter with opacity compensation, upstream's `antialiasing=True`).  A forward's backward differentiates
    what that forward rendered, whatever the setting is by then."""
    global _antialiasing
    enabled = bool(enabled)
    if enabled:
        _check_antialias_supported()
    _antialiasing = enabled


def get_antialiasing() -> bool:
    return _antialiasing


def _check_antialias_supported() -> None:
    # a library that predates the flag ignores the bit instead of refusing it: ask it what it honours
    if not _capi.lib().gs_supported_flags() & _capi.GS_FLAG_ANTIALIAS:
        raise RuntimeError(f"{_capi.LIB_PATH} does not support anti-aliasing (GS_FLAG_ANTIALIAS): rebuild it")


# ---------------------------------------------------------------------------------------------------------
# camera gradients, for callers that cannot pass BatchSettings (the drop-in GaussianRasterizer, an unmodified render_cuda)
# ---------------------------------------------------------------------------------------------------------
_camera_gradients = False


def set_camera_gradients(enabled: bool) -> None:
    """Process-wide camera-gradient setting used when BatchSettings.camera_gradients (or the `camera_gradients` argument of
    the drop-in, render_views, decoder_forward) is None: False (the default: as in the reference op, only the depth
    channel reaches the view matrix's z column) or True (viewmatrix, projmatrix, campos and a tanfov tensor get the
    gradient of colour, depth, alpha and the anti-aliasing factor; make_view_batch carries it on to the extrinsics and
    the intrinsics).  A forward's backward uses the setting of that forward."""
    global _camera_gradients
    _camera_gradients = bool(enabled)


def get_camera_gradients() -> bool:
    return _camera_gradients


def _make_config(bs: BatchSettings, S: int, P: int, M: int, keep: list) -> GsConfig:
    V = bs.viewmatrix.shape[0]
    dev = bs.viewmatrix.device
    cfg = GsConfig()
    cfg.P, cfg.S, cfg.V, cfg.M = P, S, V, M
    cfg.sh_degree = int(bs.sh_degree)
    cfg.image_height, cfg.image_width = int(bs.image_height), int(bs.image_width)
    cfg.flags = (_capi.GS_FLAG_DEPTH if bs.with_depth else 0) | (_capi.GS_FLAG_PREFILTERED if bs.prefiltered else 0)
    if _antialiasing if bs.antialiasing is None else bs.antialiasing:
        _check_antialias_supported()
        cfg.flags |= _capi.GS_FLAG_ANTIALIAS
    cfg.tanfovx, cfg.tanfovy = float(bs.tanfovx), float(bs.tanfovy)
    cfg.scale_modifier = float(bs.scale_modifier)
    cfg.tuning = int(bs.tuning)
    cfg.sh_eval_max_degree = _check_degree(_sh_eval_max_degree if bs.sh_eval_max_degree is None else bs.sh_eval_max_degree)
    if bs.depth_mode not in _capi.DEPTH_MODES:
        raise ValueError(f"depth_mode must be one of {sorted(_capi.DEPTH_MODES)}, got {bs.depth_mode!r}")
    cfg.depth_mode = _capi.DEPTH_MODES[bs.depth_mode]
    tensors = {
        "viewmatrix": _f32c(bs.viewmatrix).reshape(V, 16), "projmatrix": _f32c(bs.projmatrix, dev).reshape(V, 16),
        "campos": _f32c(bs.campos, dev).reshape(V, 3), "bg": _f32c(bs.bg, dev).reshape(V, 3),
        "tanfov": None if bs.tanfov is None else _f32c(bs.tanfov, dev).reshape(V, 2),
        "view_scale": None if bs.view_scale is None else _f32c(bs.view_scale, dev).reshape(V),
        "depth_near_far": None if bs.depth_near_far is None else _f32c(bs.depth_near_far, dev).reshape(V, 2),
    }
    for k, t in tensors.items():
        setattr(cfg, k, _ptr(t))
        keep.append(t)
    return cfg


class _RasterizeBatch(torch.autograd.Function):
    """The reference's _RasterizeGaussians (SURVEY.md section 3.4), batched over views.

    `viewmatrix`, `projmatrix`, `campos` and `tanfov` are bs.viewmatrix, bs.projmatrix, bs.campos and bs.tanfov, handed
    in as tensor inputs so that autograd can route gradients to them.  By default the view matrix gets one only through the fused depth channel
    (bs.with_depth), as the reference's depth pass gives its cameras one through its fake colour z
    (cuda_splatting.py:239-242): dL/dviewmatrix is zero outside the z column, and None when the depth is not part of the
    loss; projmatrix, campos and tanfov get None.  Colour, projection and culling give the cameras no gradient, as in the
    reference op.  With bs.camera_gradients, the four get the full gradient of every output the loss reads
    (gs_backward_cam_tanfov), the depth channel's included; tanfov's is the partial derivative with projmatrix held
    fixed.  bs.with_alpha appends the accumulated opacity (gs_forward_ex /
    gs_backward_ex).  Under torch.use_deterministic_algorithms(True) the backward is bit-reproducible."""

    @staticmethod
    def forward(ctx, means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, viewmatrix,
                projmatrix, campos, tanfov, bs: BatchSettings, workspace: Optional[SyncFreeWorkspace] = None):
        # an output the loss does not use arrives in backward as None instead of a zero tensor: a colour-only loss
        # then gives the view matrices no gradient at all (and the kernels read no depth gradient: the same sums)
        ctx.set_materialize_grads(False)
        # the SH degree this forward evaluates is fixed here: ctx.bs carries it to the backward
        bs = _resolve_degree(bs)
        dev = means3D.device
        if dev.type != "cuda":
            raise RuntimeError("pf3plat_b200 rasterizer needs CUDA tensors (there is no CPU fallback)")
        S, P = means3D.shape[0], means3D.shape[1]
        V = bs.viewmatrix.shape[0]
        M = 0 if shs is None else shs.shape[2]
        H, W = int(bs.image_height), int(bs.image_width)
        keep: list = []
        with torch.cuda.device(dev):
            stream_ptr = torch.cuda.current_stream(dev).cuda_stream
            gctx = _context(dev, stream_ptr)
            cfg = _make_config(bs, S, P, M, keep)
            ins = {
                "means3D": _f32c(means3D), "opacities": _f32c(opacities), "shs": _f32c(shs),
                "colors_precomp": _f32c(colors_precomp), "scales": _f32c(scales), "rotations": _f32c(rotations),
                "cov3D_precomp": _f32c(cov3D_precomp),
            }
            gin = GsInputs(**{k: _ptr(t) for k, t in ins.items()})
            color = torch.empty((V, 3, H, W), dtype=torch.float32, device=dev)
            radii = torch.empty((V, P), dtype=torch.int32, device=dev)
            depth = torch.empty((V, H, W), dtype=torch.float32, device=dev) if bs.with_depth else None
            gout = GsOutputs(_ptr(color), _ptr(radii), _ptr(depth))
            alpha = torch.empty((V, H, W), dtype=torch.float32, device=dev) if bs.with_alpha else None
            cam_leaves = (viewmatrix, projmatrix, campos, tanfov)
            want_cam = bool(bs.camera_gradients) and any(t is not None and t.requires_grad for t in cam_leaves)
            want_view_z = bs.with_depth and viewmatrix.requires_grad and not want_cam
            needs_grad = want_cam or want_view_z or any(t is not None and t.requires_grad for t in
                                            (means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                             cov3D_precomp))
            saved = ctypes.c_void_p()
            if workspace is not None:
                workspace._check(dev, S, V, P, H, W, bs.with_depth, bs.with_alpha, want_cam)
            with _context_lock(dev, stream_ptr):
                if workspace is not None:
                    workspace.generation += 1
                    rc = _capi.lib().gs_forward_sync_free(
                        gctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                        ctypes.byref(_capi.GsAlpha(_ptr(alpha), None)) if alpha is not None else None,
                        ctypes.byref(workspace._ws), ctypes.byref(saved) if needs_grad else None, stream_ptr)
                elif alpha is not None:
                    rc = _capi.lib().gs_forward_ex(gctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                   ctypes.byref(_capi.GsAlpha(_ptr(alpha), None)),
                                                   ctypes.byref(saved) if needs_grad else None, stream_ptr)
                else:
                    rc = _capi.lib().gs_forward(gctx, ctypes.byref(cfg), ctypes.byref(gin), ctypes.byref(gout),
                                                ctypes.byref(saved) if needs_grad else None, stream_ptr)
                _capi.check(rc)
        if needs_grad:
            ctx.handle = _SavedHandle(gctx, saved, stream_ptr, dev)
            ctx.bs = bs
            ctx.workspace = workspace
            ctx.ws_generation = None if workspace is None else workspace.generation
            ctx.ins = ins            # contiguous fp32 inputs the backward kernels re-read
            # `ins` aliases the caller's tensors when they already are fp32-contiguous; autograd's own version check is
            # bypassed for them, so do it by hand: an in-place update between forward and backward must raise, as it
            # does with the reference op (which hands its inputs to save_for_backward)
            srcs = {"means3D": means3D, "opacities": opacities, "shs": shs, "colors_precomp": colors_precomp,
                    "scales": scales, "rotations": rotations, "cov3D_precomp": cov3D_precomp}
            ctx.versions = [(k, t, t._version) for k, t in srcs.items() if t is not None]
            ctx.cfg_keep = keep
            ctx.dims = (S, P, V, M, H, W)
            ctx.want_means2D = means2D is not None and means2D.requires_grad
            ctx.view_z = (viewmatrix.shape, viewmatrix.dtype) if want_view_z else None
            ctx.cam = [(None, None, None, False) if t is None else (t.shape, t.dtype, t.device, t.requires_grad)
                       for t in cam_leaves] if want_cam else None
        ctx.mark_non_differentiable(radii)
        return (color, radii) + ((depth,) if bs.with_depth else ()) + ((alpha,) if bs.with_alpha else ())

    @staticmethod
    def backward(ctx, grad_color, grad_radii=None, *grad_extra):
        S, P, V, M, H, W = ctx.dims
        ins = ctx.ins
        for name, t, version in ctx.versions:
            if t._version != version:
                raise RuntimeError(f"one of the variables needed for gradient computation has been modified by an inplace "
                                   f"operation: {name} is at version {t._version}; expected version {version} instead")
        dev = ins["means3D"].device
        bs = ctx.bs
        ws = ctx.workspace
        if ws is not None and ws.generation != ctx.ws_generation:
            raise RuntimeError("the sync-free workspace of this forward has been reused by a later forward: its saved "
                               "state is gone (run the backward before the next forward on the workspace)")
        grad_depth = grad_extra[0] if bs.with_depth else None
        # an alpha the loss does not read arrives as None: the call is then gs_backward's, kernels included
        grad_alpha = grad_extra[-1] if bs.with_alpha else None
        keep: list = []
        with torch.cuda.device(dev):
            stream_ptr = torch.cuda.current_stream(dev).cuda_stream
            gctx = _context(dev, stream_ptr)
            cfg = _make_config(bs, S, P, M, keep)
            if torch.are_deterministic_algorithms_enabled():
                # bit-reproducible gradients: fixed-point accumulation instead of float atomics (DESIGN.md 5.11)
                cfg.flags |= _capi.GS_FLAG_DETERMINISTIC
            gin = GsInputs(**{k: _ptr(t) for k, t in ins.items()})
            gcol = _f32c(grad_color) if grad_color is not None else torch.zeros((V, 3, H, W), device=dev)
            gdep = _f32c(grad_depth) if (bs.with_depth and grad_depth is not None) else None
            og = GsOutGrads(_ptr(gcol), _ptr(gdep))
            e = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
            g = {
                "dL_dmeans3D": e(S, P, 3), "dL_dmeans2D": e(V, P, 3) if ctx.want_means2D else None,
                "dL_dshs": e(S, P, M, 3) if ins["shs"] is not None else None,
                "dL_dcolors": e(V, P, 3) if ins["colors_precomp"] is not None else None,
                "dL_dopacities": e(*ins["opacities"].shape),
                "dL_dscales": e(S, P, 3) if ins["scales"] is not None else None,
                "dL_drotations": e(S, P, 4) if ins["scales"] is not None else None,
                "dL_dcov3D": e(S, P, 6) if ins["cov3D_precomp"] is not None else None,
                "dL_dviewmatrix_z": e(V, 4) if ctx.view_z is not None and gdep is not None else None,
            }
            ig = GsInGrads(**{k: _ptr(t) for k, t in g.items()})
            # (dL/dtanfov only when tanfov requires grad: the other three are the same bytes with or without it)
            gcam = [e(V, 16), e(V, 16), e(V, 3), e(V, 2) if ctx.cam[3][3] else None] if ctx.cam is not None else None
            if ws is not None and cfg.flags & _capi.GS_FLAG_DETERMINISTIC and not ws.deterministic:
                raise ValueError("a deterministic backward needs a workspace created with deterministic=True")
            with _context_lock(dev, stream_ptr):
                if ws is not None:
                    galpha = _f32c(grad_alpha)
                    rc = _capi.lib().gs_backward_sync_free(
                        gctx, ctypes.byref(cfg), ctypes.byref(gin), ctx.handle.ptr, ctypes.byref(og),
                        ctypes.byref(_capi.GsAlpha(None, _ptr(galpha))), ctypes.byref(ig),
                        ctypes.byref(_capi.GsCameraGrads(*[_ptr(t) for t in gcam[:3]])) if gcam is not None else None,
                        _ptr(gcam[3]) if gcam is not None else None, ctypes.byref(ws._ws), stream_ptr)
                elif gcam is not None:
                    galpha = _f32c(grad_alpha)
                    rc = _capi.lib().gs_backward_cam_tanfov(
                        gctx, ctypes.byref(cfg), ctypes.byref(gin), ctx.handle.ptr, ctypes.byref(og),
                        ctypes.byref(_capi.GsAlpha(None, _ptr(galpha))), ctypes.byref(ig),
                        ctypes.byref(_capi.GsCameraGrads(*[_ptr(t) for t in gcam[:3]])), _ptr(gcam[3]), stream_ptr)
                elif grad_alpha is not None:
                    galpha = _f32c(grad_alpha)
                    rc = _capi.lib().gs_backward_ex(gctx, ctypes.byref(cfg), ctypes.byref(gin), ctx.handle.ptr,
                                                    ctypes.byref(og), ctypes.byref(_capi.GsAlpha(None, _ptr(galpha))),
                                                    ctypes.byref(ig), stream_ptr)
                else:
                    rc = _capi.lib().gs_backward(gctx, ctypes.byref(cfg), ctypes.byref(gin), ctx.handle.ptr,
                                                 ctypes.byref(og), ctypes.byref(ig), stream_ptr)
                _capi.check(rc)
            gview = gproj = gcampos = gtan = None
            if gcam is not None:
                gview, gproj, gcampos, gtan = (gt.reshape(shape).to(device, dtype) if req else None
                                               for gt, (shape, dtype, device, req) in zip(gcam, ctx.cam))
            if g["dL_dviewmatrix_z"] is not None:
                # flat entries 2, 6, 10, 14 of the transposed matrix: its z column
                gview = torch.zeros((V, 4, 4), dtype=torch.float32, device=dev)
                gview[:, :, 2] = g["dL_dviewmatrix_z"]
                shape, dtype = ctx.view_z
                gview = gview.reshape(shape).to(dtype)
        return (g["dL_dmeans3D"], g["dL_dmeans2D"], g["dL_dshs"], g["dL_dcolors"], g["dL_dopacities"],
                g["dL_dscales"], g["dL_drotations"], g["dL_dcov3D"], gview, gproj, gcampos, gtan, None, None)


def rasterize_batch(bs: BatchSettings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
                    rotations=None, cov3D_precomp=None, means2D=None, *, workspace: Optional[SyncFreeWorkspace] = None):
    """Batched operator.  Shapes: means3D (S,P,3); opacities (S,P) or (S,P,1); shs (S,P,M,3); colors_precomp
    (V,P,3); scales (S,P,3); rotations (S,P,4); cov3D_precomp (S,P,6); means2D (V,P,3) (gradient sink only).
    Returns (color (V,3,H,W), radii (V,P)[, depth (V,H,W)][, alpha (V,H,W)]).  With bs.with_depth, a bs.viewmatrix that
    requires grad gets dL/ddepth's gradient in its z column (see _RasterizeBatch); bs.with_alpha appends the accumulated
    opacity 1 - T_final.  With bs.camera_gradients, bs.viewmatrix, bs.projmatrix, bs.campos and bs.tanfov that require
    grad get the full camera gradient instead.  `workspace` (a SyncFreeWorkspace of this call's shape) selects the
    sync-free path: no host wait, no allocation by the library, graph-capturable; None = the default path."""
    _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp)
    # means2D exists in the reference op only as a sink for the screen-space gradient (cuda_splatting.py:93-97); the
    # batched entry neither allocates nor fills it unless the caller passes one
    return _RasterizeBatch.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                 bs.viewmatrix, bs.projmatrix, bs.campos, bs.tanfov, bs, workspace)


def _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp):
    # same checks and messages as the reference op's GaussianRasterizer.forward (SURVEY.md section 8(b))
    if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or (
            (scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")


class GaussianRasterizer(nn.Module):
    """Drop-in for diff_gaussian_rasterization.GaussianRasterizer (cuda_splatting.py:113-124, :206-217)."""

    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def _batch_settings(self, device, with_depth=False, camera_gradients=False) -> BatchSettings:
        rs = self.raster_settings
        f = lambda x: float(x)  # accepts python floats and 0-dim tensors (cuda_splatting.py:102-103 vs :195-196)
        # detached unless camera gradients are on: the reference op gives the cameras no gradient, with or without
        # return_depth
        d = (lambda t: t) if camera_gradients else (lambda t: t.detach())
        return BatchSettings(
            image_height=int(rs.image_height), image_width=int(rs.image_width),
            viewmatrix=d(rs.viewmatrix).reshape(1, 4, 4).to(device), projmatrix=d(rs.projmatrix).reshape(1, 4, 4),
            campos=d(rs.campos).reshape(1, 3), bg=rs.bg.reshape(1, 3), sh_degree=int(rs.sh_degree),
            tanfovx=f(rs.tanfovx), tanfovy=f(rs.tanfovy), scale_modifier=float(rs.scale_modifier),
            prefiltered=bool(rs.prefiltered), with_depth=with_depth, debug=bool(rs.debug))

    def markVisible(self, positions: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            dev = positions.device
            P = positions.shape[0]
            keep: list = []
            with torch.cuda.device(dev):
                stream_ptr = torch.cuda.current_stream(dev).cuda_stream
                gctx = _context(dev, stream_ptr)
                cfg = _make_config(self._batch_settings(dev), 1, P, 0, keep)
                pos = _f32c(positions)
                present = torch.empty((P,), dtype=torch.uint8, device=dev)
                with _context_lock(dev, stream_ptr):
                    _capi.check(_capi.lib().gs_mark_visible(gctx, ctypes.byref(cfg), pos.data_ptr(), present.data_ptr(),
                                                            stream_ptr))
            return present.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, return_depth: bool = False, return_alpha: bool = False,
                antialiasing: Optional[bool] = None, camera_gradients: Optional[bool] = None):
        """Returns (color (3,H,W), radii (P,)) like the reference op; `return_depth=True` (opt-in, not used by
        PF3plat) appends the composited camera-space depth (H,W), `return_alpha=True` then the accumulated opacity
        1 - T_final (H,W).  `antialiasing`: the screen-space filter with opacity compensation (upstream's
        GaussianRasterizationSettings.antialiasing, which this 12-field settings tuple does not carry); None = the
        process-wide setting (set_antialiasing).  `camera_gradients`: viewmatrix, projmatrix and campos of the settings
        get the full gradient of the outputs (None = the process-wide setting, set_camera_gradients); off, the reference
        op's behaviour, they get none.  tanfovx and tanfovy get none either way: the settings carry them as Python
        floats (an unmodified render_cuda hands over `.item()`s), so no gradient could reach the intrinsics through them;
        render_views / decoder_forward give the intrinsics theirs."""
        _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp)
        u = lambda t: None if t is None else t.unsqueeze(0)
        cam = _camera_gradients if camera_gradients is None else bool(camera_gradients)
        bs = self._batch_settings(means3D.device, with_depth=return_depth, camera_gradients=cam)._replace(
            with_alpha=bool(return_alpha), antialiasing=None if antialiasing is None else bool(antialiasing),
            camera_gradients=cam)
        out = _RasterizeBatch.apply(u(means3D), u(means2D), u(shs), u(colors_precomp), u(opacities), u(scales),
                                    u(rotations), u(cov3D_precomp), bs.viewmatrix, bs.projmatrix, bs.campos, None, bs)
        return tuple(o[0] for o in out)
