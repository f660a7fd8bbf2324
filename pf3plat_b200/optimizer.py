"""PF3plat's optimizer step on the device (csrc/gs_optimizer.cu, DESIGN.md 5.19).

PF3plat's ModelWrapper.optimizer_step (src/model/model_wrapper.py:210-241) runs its closure, then asks every gradient
`torch.any(torch.isnan(param.grad))` in a Python `if` -- one host synchronisation per trainable tensor -- and skips the
step on the first NaN; otherwise Lightning clips (clip_grad_norm_ with the Trainer's gradient_clip_val) and steps
torch.optim.Adam; then it zeroes the gradients.  `Adam` here does all of that in one `step()`: three kernel launches
for any number of tensors, no host wait, so the step can sit in the same CUDA graph as the forward and backward.

    step = skip if any gradient holds a NaN (not Inf) -- params, moments and step counts then stay bit for bit;
           else g *= min(max_norm / (||g||_2 + 1e-6), 1) (max_norm=None: no clip), then torch.optim.Adam's update;
           gradients zeroed in place either way (zero_grad(set_to_none=False)).

It is a torch.optim.Optimizer, so Lightning's configure_optimizers and OneCycleLR drive it unchanged, and its
state_dict is torch.optim.Adam's (per parameter `step`, `exp_avg`, `exp_avg_sq`): checkpoints move between the two.
Only what PF3plat uses is accepted: one param group of float32 CUDA parameters on one device, no weight decay, no
amsgrad, no maximize."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _capi

_CHUNK_DTYPE = np.dtype([("param", "<u8"), ("grad", "<u8"), ("exp_avg", "<u8"), ("exp_avg_sq", "<u8"),
                         ("begin", "<i8"), ("count", "<i4"), ("tensor", "<i4")])
assert _CHUNK_DTYPE.itemsize == ctypes.sizeof(_capi.GsAdamChunk)


def chunk_table(numels, chunk: int = _capi.GS_ADAM_CHUNK) -> np.ndarray:
    """(tensor, begin, count) of every chunk of tensors with `numels` elements, in order; an empty tensor gets one
    chunk of count 0 so that its step still advances."""
    tensor, begin, count = [], [], []
    for t, n in enumerate(numels):
        starts = np.arange(0, max(n, 1), chunk, dtype=np.int64)
        tensor.append(np.full(len(starts), t, dtype=np.int32))
        begin.append(starts)
        count.append(np.minimum(n - starts, chunk).astype(np.int32))
    return np.concatenate(tensor), np.concatenate(begin), np.concatenate(count)


def scratch_bytes(tensors: int, chunks: int) -> int:
    """gs_adam_scratch_bytes for a valid config."""
    cfg = _capi.GsAdamConfig(tensors=tensors, chunks=chunks, beta1=0.9, beta2=0.999, eps=1e-8, max_norm=-1.0,
                             zero_grads=1)
    return int(_capi.lib().gs_adam_scratch_bytes(ctypes.byref(cfg)))


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam with PF3plat's NaN-gradient skip and Lightning's gradient-norm clip in front of it and
    zero_grad(set_to_none=False) behind it, on the device in three launches with no host synchronisation.

    lr: a float (eager steps only: its value is written to the device at each step) or a 0-d float32 CUDA tensor on the
    parameters' device (read by the kernel, so a captured graph follows later changes to it).  max_norm: Lightning's
    gradient_clip_val (None: no clip).  `skipped` counts the skipped steps on the device (int32)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, *, max_norm=None, weight_decay=0.0,
                 amsgrad=False, maximize=False):
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                        maximize=maximize, foreach=None, capturable=False, differentiable=False, fused=None,
                        decoupled_weight_decay=False, max_norm=max_norm)
        super().__init__(params, defaults)
        group = self.param_groups[0]
        self._device = group["params"][0].device
        self._steps = torch.zeros(len(group["params"]), dtype=torch.float32, device=self._device)
        self._lr = torch.zeros((), dtype=torch.float32, device=self._device)
        self.skipped = torch.zeros((), dtype=torch.int32, device=self._device)
        self._key = None       # the pointers the uploaded chunk table was built for
        self._table = None     # device copy of the chunk table
        self._host_table = None
        self._cfg = None
        self._scratch = None

    # -- validation ------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_group(group):
        if group["weight_decay"] != 0:
            raise ValueError(f"Adam: weight_decay={group['weight_decay']!r} is not supported (PF3plat uses none)")
        if group["amsgrad"]:
            raise ValueError("Adam: amsgrad=True is not supported (PF3plat uses plain Adam)")
        if group["maximize"]:
            raise ValueError("Adam: maximize=True is not supported")
        if group.get("decoupled_weight_decay"):
            raise ValueError("Adam: decoupled_weight_decay=True is not supported")
        b1, b2 = group["betas"]
        if not (0.0 <= float(b1) < 1.0 and 0.0 <= float(b2) < 1.0):
            raise ValueError(f"Adam: betas must lie in [0, 1), got {group['betas']!r}")
        if not (0.0 <= float(group["eps"]) < math.inf):
            raise ValueError(f"Adam: eps must be finite and >= 0, got {group['eps']!r}")
        mn = group["max_norm"]
        if mn is not None and not (0.0 <= float(mn) < math.inf):
            raise ValueError(f"Adam: max_norm must be None or finite and >= 0, got {mn!r}")
        lr = group["lr"]
        if torch.is_tensor(lr):
            if lr.dim() != 0 or lr.dtype != torch.float32 or lr.device.type != "cuda":
                raise TypeError(f"Adam: a tensor lr must be a 0-d float32 CUDA tensor, got {lr.dtype} {tuple(lr.shape)} "
                                f"on {lr.device}")
        elif not (0.0 <= float(lr) < math.inf):
            raise ValueError(f"Adam: lr must be finite and >= 0, got {lr!r}")
        device = None
        for i, p in enumerate(group["params"]):
            if p.device.type != "cuda":
                raise TypeError(f"Adam: params[{i}] is on {p.device}; every parameter must be a CUDA tensor")
            if p.dtype != torch.float32:
                raise TypeError(f"Adam: params[{i}] is {p.dtype}; every parameter must be float32")
            if device is not None and p.device != device:
                raise ValueError(f"Adam: params[{i}] is on {p.device}, params[0] on {device}; mixed-device parameters "
                                 f"are not supported")
            if not p.is_contiguous():
                raise ValueError(f"Adam: params[{i}] is not contiguous")
            device = p.device
        if torch.is_tensor(lr) and lr.device != device:
            raise ValueError(f"Adam: lr is on {lr.device}, the parameters on {device}")

    def add_param_group(self, param_group):
        if self.param_groups:
            raise ValueError("Adam: one param group only (PF3plat's configure_optimizers passes self.parameters())")
        super().add_param_group(param_group)
        self._check_group(self.param_groups[0])

    # -- torch.optim.Adam's state format ---------------------------------------------------------------------------
    def state_dict(self):
        """torch.optim.Adam's format: `step` a 0-d float32 CPU tensor (so this call reads the device)."""
        sd = super().state_dict()
        sd["state"] = {k: {**v, "step": v["step"].detach().to(device="cpu", dtype=torch.float32, copy=True)}
                       for k, v in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        max_norm = self.param_groups[0]["max_norm"]
        super().load_state_dict(state_dict)
        group = self.param_groups[0]
        group.setdefault("max_norm", max_norm)  # a torch.optim.Adam state dict has none: keep ours
        for k, v in self.defaults.items():
            group.setdefault(k, v)
        self._check_group(group)
        for i, p in enumerate(group["params"]):
            st = self.state.get(p)
            if not st:
                continue
            self._steps[i].fill_(float(st["step"]))
            st["step"] = self._steps[i]
            for k in ("exp_avg", "exp_avg_sq"):
                st[k] = st[k].to(device=p.device, dtype=torch.float32).contiguous()
        self._key = None

    def zero_grad(self, set_to_none: bool = False):
        """Zeroes the gradients in place by default, so that their addresses (and a captured graph's) stay put.  step()
        has zeroed them already; this is one multi-tensor launch, without the per-tensor Python of the base class."""
        if set_to_none:
            return super().zero_grad(set_to_none=True)
        grads = [p.grad for p in self.param_groups[0]["params"] if p.grad is not None]
        if grads:
            torch._foreach_zero_(grads)

    # -- the step --------------------------------------------------------------------------------------------------
    def _build_table(self, entries, key):
        for i, p, g in entries:
            if g.dtype != torch.float32 or g.device != p.device or g.shape != p.shape:
                raise TypeError(f"Adam: the gradient of params[{i}] is {g.dtype} {tuple(g.shape)} on {g.device}; "
                                f"expected float32 {tuple(p.shape)} on {p.device}")
            if not g.is_contiguous():
                raise ValueError(f"Adam: the gradient of params[{i}] is not contiguous")
        tensor, begin, count = chunk_table([p.numel() for _, p, _ in entries])
        table = np.zeros(len(tensor), dtype=_CHUNK_DTYPE)
        state = [self.state[p] for _, p, _ in entries]
        ptr = lambda f: np.array(f, dtype=np.uint64)[tensor]
        table["param"] = ptr([p.data_ptr() for _, p, _ in entries])
        table["grad"] = ptr([g.data_ptr() for _, _, g in entries])
        table["exp_avg"] = ptr([s["exp_avg"].data_ptr() for s in state])
        table["exp_avg_sq"] = ptr([s["exp_avg_sq"].data_ptr() for s in state])
        table["begin"], table["count"] = begin, count
        table["tensor"] = np.array([i for i, _, _ in entries], dtype=np.int32)[tensor]
        cfg = _capi.GsAdamConfig(tensors=len(self.param_groups[0]["params"]), chunks=len(table), zero_grads=1)
        self._set_hyperparameters(cfg)
        need = _capi.lib().gs_adam_scratch_bytes(ctypes.byref(cfg))
        if need < 0:
            _capi.check(-1)
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self._device)
        # a new pinned buffer each time: the previous one may still feed a copy in flight
        self._host_table = torch.from_numpy(table.view(np.uint8)).pin_memory()
        self._table = torch.empty(self._host_table.numel(), dtype=torch.uint8, device=self._device)
        self._table.copy_(self._host_table, non_blocking=True)
        self._cfg, self._key = cfg, key

    def _set_hyperparameters(self, cfg):
        group = self.param_groups[0]
        b1, b2 = group["betas"]
        mn = group["max_norm"]
        cfg.beta1, cfg.beta2, cfg.eps = float(b1), float(b2), float(group["eps"])
        cfg.max_norm = -1.0 if mn is None else float(mn)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        group = self.param_groups[0]
        capturing = torch.cuda.is_current_stream_capturing()
        lr = group["lr"]
        if torch.is_tensor(lr):
            lr_ptr = lr.data_ptr()
        else:
            if capturing:
                raise RuntimeError("Adam.step: a float lr cannot be captured in a CUDA graph (the graph would keep "
                                   "this step's value); set the param group's lr to a 0-d float32 CUDA tensor")
            self._lr.fill_(float(lr))
            lr_ptr = self._lr.data_ptr()
        entries = [(i, p, p.grad) for i, p in enumerate(group["params"]) if p.grad is not None]
        if not entries:
            return loss
        for i, p, _ in entries:
            st = self.state[p]
            if not st:
                if capturing:
                    raise RuntimeError("Adam.step: parameters without optimizer state under CUDA graph capture; run "
                                       "one eager step first")
                self._steps[i].zero_()
                st["step"] = self._steps[i]
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        for i, _, g in entries:
            if g.layout != torch.strided:
                raise ValueError(f"Adam: the gradient of params[{i}] is sparse")
        key = tuple((i, p.data_ptr(), g.data_ptr()) for i, p, g in entries)
        if key != self._key or self._cfg is None:
            if capturing:
                raise RuntimeError("Adam.step: the gradients moved since the last eager step; under CUDA graph capture "
                                   "the chunk table cannot be rebuilt (run one eager step with these gradients first)")
            self._build_table(entries, key)
        else:
            self._set_hyperparameters(self._cfg)  # a scheduler or the caller may change them between steps
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _capi.check(_capi.lib().gs_adam_step(ctypes.byref(self._cfg), self._table.data_ptr(),
                                                 self._steps.data_ptr(), lr_ptr, self.skipped.data_ptr(),
                                                 self._scratch.data_ptr(), ctypes.c_void_p(stream)))
        return loss
