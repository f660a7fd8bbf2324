"""Times the SH rotation blocks on one GPU: the device op pf3plat_b200.sh_rotation.guarded_sh_rotation_blocks (two
launches, csrc/gs_sh_rotation.cu) against the tensor route it replaces in the Gaussian head (torch.det, isclose().all(),
torch.where, then sh_rotation_blocks' least-squares fit), and pf3plat_b200.gaussian_head with each of them building its
sh_rotation input (the tensor version of sh_rotation_for_slots is kept here as `tensor_slots`), each followed by
decoder_forward's input handling as in scripts/bench_gaussian_head.py.

  blocks  N in {2, 28, 256, 65534} rotations, d_sh in {9, 25}
  head    forward, and forward + backward of a loss on all four outputs, at PF3plat's training shape: b = 14,
          256 x 256, d_sh = 25, V in {2, 3}

The two variants alternate within one run; a round is --steps calls between two device synchronisations, timed with CUDA
events, and the median over --rounds rounds is reported with the spread ((max - min) / median).  Also per variant: the
kernel launches of one call (torch.profiler) and its synchronising calls (torch.cuda.set_sync_debug_mode("warn")), and
the largest difference between the variants' outputs.  Also reported: the card, its power limit and its maximum SM
clock, read in the same run.

Usage:  python scripts/bench_sh_rotation.py [--steps 20] [--warmup 3] [--rounds 9] [--out DIR]
Writes DIR/bench_sh_rotation.json (default: a temporary directory) and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import pf3plat_b200.gaussian_head as head_mod  # noqa: E402
from bench_gaussian_head import seeded_inputs, step  # noqa: E402
from pf3plat_b200.sh_rotation import guarded_sh_rotation_blocks, sh_rotation_blocks  # noqa: E402

DEVICE_SLOTS = head_mod.sh_rotation_for_slots


def tensor_blocks(rot, d_sh):
    """the head's former tensor route on [..., 3, 3] rotations: the guard as torch ops, then the fit"""
    det = torch.det(rot)
    ok = torch.isclose(det, torch.ones_like(det)).all()
    rot = torch.where(ok, rot, torch.eye(3, dtype=rot.dtype, device=rot.device))
    return sh_rotation_blocks(rot, d_sh).contiguous()


def tensor_slots(c2w, d_sh):
    """sh_rotation_for_slots before the device op"""
    if d_sh == 1:
        return None
    c = c2w.detach()
    return tensor_blocks(torch.stack([c[:, 0, :3, :3], c[:, -1, :3, :3]], 1), d_sh)


def timed(fn, steps, rounds_out):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    rounds_out.append(a.elapsed_time(e) / steps)


def count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(x.message) for x in caught)


def count_launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
               and "memset" not in e.name.lower())


def compare(variants, args):
    """variants: name -> zero-argument callable; alternating timed rounds, launches and syncs per variant"""
    for fn in variants.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            timed(fn, args.steps, times[k])
    res = {}
    for k, ts in times.items():
        med = statistics.median(ts)
        res[f"{k}_ms"] = round(med, 4)
        res[f"{k}_spread"] = round((max(ts) - min(ts)) / med, 3)
        res[f"{k}_launches"] = count_launches(variants[k])
        res[f"{k}_sync_calls"] = count_syncs(variants[k])
    names = list(variants)
    res["speedup"] = round(res[f"{names[0]}_ms"] / res[f"{names[1]}_ms"], 2)
    return res


def rotations(n, dev):
    q, r = torch.linalg.qr(torch.randn(n, 3, 3, generator=torch.Generator().manual_seed(n), dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r, dim1=-2, dim2=-1))[:, None, :]
    q[torch.det(q) < 0, :, 0] *= -1
    return q.float().to(dev)


def with_slots(slots, fn):
    def run():
        head_mod.sh_rotation_for_slots = slots
        try:
            return fn()
        finally:
            head_mod.sh_rotation_for_slots = DEVICE_SLOTS
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sh_rotation.py needs a CUDA device")
    dev = torch.device("cuda:0")
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        info["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"

    blocks = {}
    for n in (2, 28, 256, 65534):
        rot = rotations(n, dev)
        for d_sh in (9, 25):
            res = compare({"tensor_route": lambda: tensor_blocks(rot, d_sh),
                           "device_op": lambda: guarded_sh_rotation_blocks(rot, d_sh)}, args)
            res["max_abs_diff"] = float((tensor_blocks(rot, d_sh) - guarded_sh_rotation_blocks(rot, d_sh)).abs().max())
            blocks[f"n{n}_dsh{d_sh}"] = res

    head = {}
    for V in (2, 3):
        b, h, w = 14, 256, 256
        inp = seeded_inputs(b, V, h, w, 4, dev)
        res = {}
        with torch.no_grad():
            old = with_slots(tensor_slots, lambda: step("ours", inp, False))()
            new = step("ours", inp, False)
            res["max_abs_diff"] = {k: float((a - c).abs().max()) for k, a, c in
                                   zip(("means", "covariances6", "harmonics", "opacities"), old, new)}
            del old, new
        for label, backward in (("forward", False), ("forward_backward", True)):
            r = compare({"tensor_slots": with_slots(tensor_slots, lambda: step("ours", inp, backward)),
                         "device_slots": lambda: step("ours", inp, backward)}, args)
            res.update({f"{label}_{k}": v for k, v in r.items()})
        head[f"b{b}_v{V}_{h}_dsh25"] = res
        del inp
        torch.cuda.empty_cache()
    out = {"bench": "sh_rotation", **info, "torch": torch.__version__, "steps": args.steps, "rounds": args.rounds,
           "blocks": blocks, "gaussian_head": head}
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_sh_rotation_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bench_sh_rotation.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
