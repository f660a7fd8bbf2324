"""PF3plat's optimizer step restated in plain torch: the reference sequence pf3plat_b200.optimizer.Adam is checked against.

ModelWrapper.optimizer_step (src/model/model_wrapper.py:210-241), after its closure:
  1. for every parameter whose .grad is not None, `torch.any(torch.isnan(param.grad))` in a Python `if`; the first NaN
     skips the step (:226-235);
  2. otherwise `optimizer.step()`, Lightning's optimizer wrapper, which first clips: Lightning's
     Precision.clip_grad_by_norm is `torch.nn.utils.clip_grad_norm_(<every parameter of the optimizer>, clip_val)` with
     the Trainer's gradient_clip_val (0.5 in PF3plat's config/main.yaml; None = no clip, Lightning's default).  Lightning
     is not installed here, so that call is restated below rather than imported;
  3. then torch.optim.Adam (model_wrapper.py:780: one param group, default betas and eps, foreach on CUDA);
  4. `optimizer.zero_grad()` (:241).  The reference's default sets the gradients to None; the device op zeroes them in
     place, so the oracle zeroes in place too (the next backward gives the same gradients either way)."""
import torch


def exact_total_norm(grads) -> torch.Tensor:
    """The 2-norm of all gradients summed in fp64 and rounded to fp32 once (inf where torch's fp32 squares overflow)."""
    s = sum(float(g.double().square().sum()) for g in grads)
    return torch.tensor(float("inf") if s > torch.finfo(torch.float32).max else s ** 0.5, dtype=torch.float32,
                        device=grads[0].device)


def reference_step(optimizer: torch.optim.Optimizer, max_norm=None, total_norm=None) -> bool:
    """One optimizer_step after the closure; True when it skipped the update.  total_norm: clip with this total instead
    of clip_grad_norm_'s own fp32 one (torch.nn.utils.clip_grads_with_norm_, the second half of clip_grad_norm_)."""
    skip_step = False
    for group in optimizer.param_groups:
        for param in group["params"]:
            if param.grad is not None and torch.any(torch.isnan(param.grad)):
                skip_step = True
                break
        if skip_step:
            break
    if not skip_step:
        if max_norm is not None:  # Lightning: clip_gradients before the wrapped optimizer's step
            params = [p for group in optimizer.param_groups for p in group["params"]]
            if total_norm is None:
                torch.nn.utils.clip_grad_norm_(params, max_norm)
            else:
                torch.nn.utils.clip_grads_with_norm_(params, max_norm, total_norm)
        optimizer.step()
    optimizer.zero_grad(set_to_none=False)
    return skip_step
