"""Generates tests/golden/ssim_loss.npz by running the REFERENCE's own photometric losses (PF3plat's
src/loss/loss_multissim.py and src/loss/loss_mse.py, imported unmodified from a PF3plat checkout) on small seeded
inputs, in float32 and in float64, and recording their values and autograd gradients.

Needs a PF3plat checkout, named by $PF3PLAT_ROOT.  The loss modules import types from the rest of the tree only for
annotations; those modules (src.dataset.types, src.model.decoder.decoder, src.model.types) and the abstract base
src.loss.loss are stubbed, and the packages are bare modules, so that nothing but torch, einops and jaxtyping is
needed.  `ssim` itself is the reference's function, window construction included.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_ssim_loss_golden.py
"""
import importlib.util
import os
import sys
import types
from dataclasses import fields
from typing import Generic, TypeVar

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("PF3PLAT_ROOT", "")


def require_reference():
    if not REF_ROOT or not os.path.isfile(os.path.join(REF_ROOT, "src/loss/loss_multissim.py")):
        raise SystemExit(f"set PF3PLAT_ROOT to a PF3plat checkout (got {REF_ROOT!r})")


def _stub_loss_base():
    A, B = TypeVar("A"), TypeVar("B")

    class Loss(torch.nn.Module, Generic[A, B]):
        def __init__(self, cfg):  # the reference's base takes the wrapper's single field as its cfg
            super().__init__()
            (f,) = fields(type(cfg))
            self.cfg = getattr(cfg, f.name)
            self.name = f.name
    return Loss


def load_reference_losses():
    """-> (loss_multissim module, loss_mse module) of the reference, unmodified."""
    require_reference()
    for name in ("src", "src.loss", "src.dataset", "src.model", "src.model.decoder"):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF_ROOT, *name.split("."))]
        sys.modules[name] = m
    stubs = {"src.dataset.types": {"BatchedExample": dict}, "src.model.decoder.decoder": {"DecoderOutput": object},
             "src.model.types": {"Gaussians": object}, "src.loss.loss": {"Loss": _stub_loss_base()}}
    for name, attrs in stubs.items():
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    mods = []
    for name in ("loss_multissim", "loss_mse"):
        spec = importlib.util.spec_from_file_location(f"src.loss.{name}",
                                                      os.path.join(REF_ROOT, "src", "loss", f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
        mods.append(mod)
    return tuple(mods)


def _render_like(g, n, c, h, w):
    """Coloured discs on a black background: large flat regions where every moment is zero."""
    img = torch.zeros(n, c, h, w, dtype=torch.float64)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    for i in range(n):
        for _ in range(4):
            cy, cx = torch.rand(2, generator=g, dtype=torch.float64) * torch.tensor([h, w], dtype=torch.float64)
            r = 2.0 + 6.0 * float(torch.rand(1, generator=g, dtype=torch.float64))
            col = torch.rand(c, generator=g, dtype=torch.float64)
            a = torch.clamp(r - torch.sqrt((ys - cy) ** 2 + (xs - cx) ** 2), 0, 1)
            img[i] = img[i] * (1 - a) + col[:, None, None] * a
    return img


def make_case(name, g):
    """-> (x, y) float64, (n, c, h, w): x plays the prediction, y the ground truth."""
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    if name == "random":
        return u(2, 3, 24, 20), u(2, 3, 24, 20)
    if name == "render":
        y = _render_like(g, 2, 3, 32, 32)
        x = (y + 0.05 * torch.randn(y.shape, generator=g, dtype=torch.float64) * (y > 0)).clamp(0, 1)
        return x, y
    if name == "identical":
        x = u(2, 3, 16, 16)
        return x, x.clone()
    if name == "out_of_range":
        return -0.1 + 1.3 * u(2, 3, 20, 18), -0.1 + 1.3 * u(2, 3, 20, 18)
    if name == "tiny_5x7":
        return u(2, 3, 5, 7), u(2, 3, 5, 7)
    if name == "tiny_1x1":
        return u(3, 3, 1, 1), u(3, 3, 1, 1)
    if name == "batch_37x45":
        return u(2, 3, 37, 45), u(2, 3, 37, 45)
    raise KeyError(name)


CASES = ("random", "render", "identical", "out_of_range", "tiny_5x7", "tiny_1x1", "batch_37x45")


def run_reference(ms, mse_mod, x, y, w_img, dtype):
    """The reference's ssim (both size_average settings), its gradients, and the two loss modules' forward."""
    xa = x.to(dtype).clone().requires_grad_(True)
    ya = y.to(dtype).clone().requires_grad_(True)
    per = ms.ssim(xa, ya, size_average=False)
    mean = ms.ssim(xa, ya)
    gx, gy = torch.autograd.grad((per * w_img.to(dtype)).sum(), (xa, ya))
    # the loss modules read color[:, 1:-1] of (b, v, c, h, w): embed the n images as the inner views of one scene
    pad = lambda t: torch.cat([torch.zeros_like(t[:1]), t, torch.zeros_like(t[:1])])[None]
    pred = types.SimpleNamespace(color=pad(xa))
    batch = {"context": {"image": pad(ya)}, "target": {"image": pad(ya)}}
    l_ssim = ms.LossMultiSSIM(ms.LossMultiSSIMCfgWrapper(ms.LossMultiSSIMCfg(weight=1.0)))
    l_mse = mse_mod.LossMse(mse_mod.LossMseCfgWrapper(mse_mod.LossMseCfg(weight=1.0)))
    lm = l_mse.forward(pred, batch, None, 0, None, None, None, None)
    ls = l_ssim.forward(pred, batch, None, 0, None, None, None, None)
    return dict(ssim_mean=mean.detach(), ssim_img=per.detach(), grad_x=gx, grad_y=gy, loss_mse=lm.detach(),
                loss_multissim=ls.detach())


def main():
    ms, mse_mod = load_reference_losses()
    arrays = {}
    for i, name in enumerate(CASES):
        g = torch.Generator().manual_seed(1000 + i)
        x, y = make_case(name, g)
        x32, y32 = x.float(), y.float()             # every dtype sees the same float32-representable inputs
        w_img = torch.randn(x.shape[0], generator=g, dtype=torch.float64)
        arrays[f"{name}/x"] = x32.numpy()
        arrays[f"{name}/y"] = y32.numpy()
        arrays[f"{name}/w_img"] = w_img.numpy()
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            out = run_reference(ms, mse_mod, x32.double(), y32.double(), w_img, dt)
            for k, v in out.items():
                arrays[f"{name}/{tag}/{k}"] = v.numpy()
        print(name, tuple(x.shape), "ssim f64", arrays[f"{name}/f64/ssim_img"])
    path = os.path.join(HERE, "ssim_loss.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
