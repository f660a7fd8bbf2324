"""PF3plat's pose path between PnP and the networks that read the poses, on the device (csrc/gs_poses.cu).

- `camera_synchronization(Ps, confidence, N)` is a drop-in for src/flow_util.py's function of that name (forward only).
- `refine_poses(pred_pose_enc, delta_pose, gamma)` is encoder_costvolume.py:465-473 and the `.inverse()` of its result,
  forward and backward.
- `plucker_rays(abspose, intrinsics, h, w)` is the Plücker embedding of encoder_costvolume.py:387-392 (forward only).

None of them synchronises the device with the host.  Inputs must be float32 CUDA tensors; there is no CPU fallback.

Divergences from the reference, none of which PF3plat's training or evaluation reaches:
- camera_synchronization on non-finite input: on the CPU the reference raises from `torch.svd`.  Raising would need a
  host read, so here every output of a scene whose L (as built, or its column block after the squarings) is non-finite
  is NaN, the other scenes keep their values, and that scene's NaN mass turns the batch-wide chaining fallback off,
  as a NaN mass does in the reference.
- camera_synchronization needs the chain pairs (k, k+1) for every N, because the device decides the fallback.
- refine_poses on a singular pose returns a non-finite inverse instead of raising.
- camera_synchronization on a rotation block of rank 1 (reachable only through degenerate pairwise transforms): the
  reference's answer depends on LAPACK's arbitrary basis of the block's null plane; here it is a proper rotation that
  agrees with the block on its one singular direction.  The zero block gives I, as in the reference.
"""
from __future__ import annotations

import torch

from . import _capi

_SYNC_DEFAULTS = dict(squares=10, so3_projection=True, normalize_confidences=True, double=True,
                      center_first_camera=True)


def _check_cuda_float(name: str, t, device=None) -> None:
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise RuntimeError(f"{name} must be a CUDA tensor (there is no CPU fallback)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if device is not None and t.device != device:
        raise ValueError(f"{name} is on {t.device}, expected {device}")


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def camera_synchronization(Ps, confidence, N, **kw):
    """src/flow_util.py camera_synchronization at the arguments PF3plat calls it with: Ps[(i, j)] [b, 4, 4] the pairwise
    transform i -> j, confidence[(i, j)] [b]; returns [b, N, 4, 4] float32.  Needs 2 <= N <= 16, inputs that do not
    require grad, and the pair (k, k+1) for every k < N - 1."""
    for k, v in kw.items():
        if k not in _SYNC_DEFAULTS or v != _SYNC_DEFAULTS[k]:
            raise ValueError(f"camera_synchronization supports only {_SYNC_DEFAULTS}, got {k}={v!r}")
    N = int(N)
    if not 2 <= N <= _capi.GS_POSES_MAX_VIEWS:
        raise ValueError(f"camera_synchronization needs 2 <= N <= {_capi.GS_POSES_MAX_VIEWS}, got N={N}")
    keys = list(Ps)
    # the reference's sanity checks (camera_chaining's for N = 2), then what the device path needs
    for k in range(N - 1):
        if (k, k + 1) not in Ps:
            raise AssertionError(f"camera_synchronization: pair {(k, k + 1)} is missing")
    if N > 2:
        views = set()
        for i, j in keys:
            if (i, j) not in confidence or i == j or (j, i) in Ps:
                raise AssertionError(f"camera_synchronization: bad pair {(i, j)}")
            views.update((i, j))
        for vi in range(N):
            if vi not in views:
                raise AssertionError(f"View {vi} is not in any pairwise views")
    if N == 2:
        keys = [(0, 1)]
    for i, j in keys:
        if not (0 <= i < N and 0 <= j < N):
            raise ValueError(f"camera_synchronization: pair {(i, j)} is outside 0 <= i, j < N={N}")
    dev = Ps[keys[0]].device if torch.is_tensor(Ps[keys[0]]) else None
    mats = [Ps[k] for k in keys]
    confs = [confidence[k] for k in keys] if N > 2 else []
    for k, t in zip(keys, mats):
        _check_cuda_float(f"camera_synchronization: Ps[{k}]", t, dev)
    for k, t in zip(keys, confs):
        _check_cuda_float(f"camera_synchronization: confidence[{k}]", t, dev)
    b = mats[0].shape[0] if mats[0].dim() == 3 else -1
    if b < 1 or any(tuple(t.shape) != (b, 4, 4) for t in mats) or any(tuple(t.shape) != (b,) for t in confs):
        raise ValueError("camera_synchronization needs every Ps[(i, j)] as [b, 4, 4] and every confidence[(i, j)] as "
                         "[b] with one b >= 1")
    if any(t.requires_grad for t in mats + confs):
        raise ValueError("camera_synchronization is forward only: its inputs must not require grad")
    cfg = _capi.GsPoseSyncConfig(batch=b, views=N, pairs=len(keys))
    for q, (i, j) in enumerate(keys):
        cfg.pair_i[q], cfg.pair_j[q] = i, j
    L = _capi.lib()
    with torch.cuda.device(dev):
        P = torch.stack(mats).contiguous()
        C = torch.stack(confs).contiguous() if confs else None
        out = torch.empty((b, N, 4, 4), dtype=torch.float32, device=dev)
        nbytes = int(L.gs_pose_sync_scratch_bytes(cfg))
        if nbytes < 0:
            _capi.check(-1)
        scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        _capi.check(L.gs_pose_sync(cfg, P.data_ptr(), C.data_ptr() if C is not None else None, out.data_ptr(),
                                   scratch.data_ptr(), _stream(dev)))
    return out


def _refine_structs(pose_enc, delta, gamma):
    b, v, _ = pose_enc.shape
    return (_capi.GsRefinePosesConfig(batch=b, views=v),
            _capi.GsRefinePosesInputs(pose_enc=pose_enc.data_ptr(), delta=delta.data_ptr(), gamma=gamma.data_ptr()))


class _RefinePoses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pose_enc, delta, gamma):
        b, v, _ = pose_enc.shape
        dev = pose_enc.device
        cfg, ins = _refine_structs(pose_enc, delta, gamma)
        A = torch.empty((b, v, 4, 4), dtype=torch.float32, device=dev)
        Ai = torch.empty_like(A)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_refine_poses_forward(cfg, ins, A.data_ptr(), Ai.data_ptr(), _stream(dev)))
        ctx.save_for_backward(pose_enc, delta, gamma)
        ctx.set_materialize_grads(False)
        return A, Ai

    @staticmethod
    def backward(ctx, dA, dAi):
        if dA is None and dAi is None:
            return None, None, None
        pose_enc, delta, gamma = ctx.saved_tensors
        dev = pose_enc.device
        cfg, ins = _refine_structs(pose_enc, delta, gamma)
        gA = dA.to(torch.float32).contiguous() if dA is not None else None
        gAi = dAi.to(torch.float32).contiguous() if dAi is not None else None
        d_pose = torch.empty_like(pose_enc)
        d_delta = torch.empty_like(delta)
        d_gamma = torch.empty((1,), dtype=torch.float32, device=dev)
        grads = _capi.GsRefinePosesGrads(dL_dabspose=gA.data_ptr() if gA is not None else None,
                                         dL_dabspose_inv=gAi.data_ptr() if gAi is not None else None,
                                         dL_dpose_enc=d_pose.data_ptr(), dL_ddelta=d_delta.data_ptr(),
                                         dL_dgamma=d_gamma.data_ptr())
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gs_refine_poses_backward(cfg, ins, grads, _stream(dev)))
        return d_pose, d_delta, d_gamma


def refine_poses(pred_pose_enc: torch.Tensor, delta_pose: torch.Tensor, gamma: torch.Tensor):
    """encoder_costvolume.py:465-473 and the `.inverse()` of its result: pred_pose_enc, delta_pose [b, v, 9] (rotation
    6-d, translation), gamma one element (the encoder's `self.gamma`).  Returns (abspose, abspose_inv), both
    [b, v, 4, 4]; gradients reach all three inputs from either output.  View 0 is pred_pose_enc[:, 0] (its delta gets a
    zero gradient); abspose_inv is the general 4 x 4 inverse, non-finite where abspose is singular."""
    _check_cuda_float("refine_poses: pred_pose_enc", pred_pose_enc)
    dev = pred_pose_enc.device
    _check_cuda_float("refine_poses: delta_pose", delta_pose, dev)
    _check_cuda_float("refine_poses: gamma", gamma, dev)
    if pred_pose_enc.dim() != 3 or pred_pose_enc.shape[-1] != 9 or pred_pose_enc.shape[0] < 1 or \
            pred_pose_enc.shape[1] < 1 or tuple(delta_pose.shape) != tuple(pred_pose_enc.shape) or gamma.numel() != 1:
        raise ValueError(f"refine_poses needs pred_pose_enc and delta_pose [b, v, 9] and a one-element gamma, got "
                         f"{tuple(pred_pose_enc.shape)}, {tuple(delta_pose.shape)}, {tuple(gamma.shape)}")
    return _RefinePoses.apply(pred_pose_enc.contiguous(), delta_pose.contiguous(), gamma.reshape(1).contiguous())


def plucker_rays(abspose: torch.Tensor, intrinsics: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """plucker_embedding(h, w, *get_world_rays(grid, abspose.inverse(), intrinsics)) of encoder_costvolume.py:387-392 on
    the (h, w) pixel-centre grid: abspose [b, v, 4, 4] world-to-camera, intrinsics [b, v, 3, 3] normalised.  Returns a
    contiguous [(b v), 6, h, w] (ray direction, origin x direction), b-major.  Forward only."""
    _check_cuda_float("plucker_rays: abspose", abspose)
    _check_cuda_float("plucker_rays: intrinsics", intrinsics, abspose.device)
    h, w = int(h), int(w)
    if abspose.dim() != 4 or tuple(abspose.shape[2:]) != (4, 4) or tuple(intrinsics.shape) != (*abspose.shape[:2], 3, 3):
        raise ValueError(f"plucker_rays needs abspose [b, v, 4, 4] and intrinsics [b, v, 3, 3], got "
                         f"{tuple(abspose.shape)}, {tuple(intrinsics.shape)}")
    b, v = abspose.shape[:2]
    if b < 1 or v < 1 or h < 1 or w < 1:
        raise ValueError(f"plucker_rays needs b, v, h, w >= 1, got {b}, {v}, {h}, {w}")
    if abspose.requires_grad or intrinsics.requires_grad:
        raise ValueError("plucker_rays is forward only: abspose and intrinsics must not require grad")
    dev = abspose.device
    out = torch.empty((b * v, 6, h, w), dtype=torch.float32, device=dev)
    cfg = _capi.GsPluckerConfig(batch=b, views=v, height=h, width=w)
    A, K = abspose.contiguous(), intrinsics.contiguous()
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().gs_plucker_rays(cfg, A.data_ptr(), K.data_ptr(), out.data_ptr(), _stream(dev)))
    return out
