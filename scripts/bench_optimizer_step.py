"""Times PF3plat's optimizer step three ways, alternating in one process (DESIGN.md 5.19):

  (a) reference: the host NaN loop of ModelWrapper.optimizer_step (one `torch.any(torch.isnan(g))` host read per tensor)
      + clip_grad_norm_(0.5) + torch.optim.Adam (foreach) + zero_grad;
  (b) stock capturable: a device NaN flag from torch ops (isnan of _foreach_max, which propagates NaN but not Inf)
      + clip_grad_norm_(0.5, foreach=True) + torch.optim.Adam(fused=True) skipping on that flag through its found_inf
      + zero_grad;
  (c) pf3plat_b200.optimizer.Adam(max_norm=0.5).step(), which zeroes the gradients itself; (c+z) adds the zero_grad()
      call of INTEGRATION.md's recipe.

on three parameter sets: a PF3plat-like set (~400 tensors, ~28 M elements), one 100 M-element tensor (bandwidth) and
2000 tiny tensors (launches).  zero_grad keeps the gradients (set_to_none=False) in every route, so each step streams
the same bytes.  GPU time per step from CUDA events, host time per step from the host clock around the calls (route (a)
waits for the device inside them).  Bytes per element are the count of the design, not a measurement: (c) reads
g once in pass 1, then g, p, m, v and writes p, m, v, g in pass 2 (36 B); (a) and (b) as estimated in DESIGN.md.
Prints the results as one JSON line as well; --out PATH also writes them to PATH."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pf3plat_b200.optimizer import Adam  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet
BYTES_PER_ELEMENT = {"a": 90, "b": 45, "c": 36, "c+z": 40}  # estimates (DESIGN.md 5.19)


def pf3plat_like():
    shapes = []
    for i in range(100):
        c = (64, 128, 192, 256)[i % 4]
        shapes += [(c, c, 3, 3), (c,), (c,), (1 + (37 * i) % 1000,)]
    return shapes + [(), (), (1,), (3, 3)]


SETS = {"pf3plat_like": pf3plat_like, "one_100M": lambda: [(100_000_000,)],
        "tiny_2000": lambda: [(1 + (13 * i) % 256,) for i in range(2000)]}


def make(shapes, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    ps = [torch.nn.Parameter(torch.randn(s, generator=g, device=dev) * 0.1) for s in shapes]
    for p in ps:
        p.grad = torch.randn(p.shape, generator=g, device=dev) * 1e-4
    return ps


def route_a(params, opt):
    skip = False
    for p in params:
        if p.grad is not None and torch.any(torch.isnan(p.grad)):
            skip = True
            break
    if not skip:
        torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step()
    opt.zero_grad(set_to_none=False)


def route_b(params, opt):
    grads = [p.grad for p in params]
    opt.found_inf = torch.isnan(torch.stack(torch._foreach_max(grads))).any().float()
    torch.nn.utils.clip_grad_norm_(params, 0.5, foreach=True)
    opt.step()
    opt.zero_grad(set_to_none=False)


def route_c(params, opt):
    opt.step()


def route_cz(params, opt):
    opt.step()
    opt.zero_grad()


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        out = f"unavailable ({e})"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="steps per timed window")
    ap.add_argument("--reps", type=int, default=5, help="alternating windows per route")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sets", default=",".join(SETS))
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optimizer_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    results = {"card": name, "power_limit_and_max_sm_clock": power, "sets": {}}
    for set_name in args.sets.split(","):
        shapes = SETS[set_name]()
        n = sum(int(torch.Size(s).numel()) for s in shapes)
        routes = {}
        pa = make(shapes, dev, 0)
        routes["a"] = (route_a, pa, torch.optim.Adam(pa, lr=2e-4))
        pb = make(shapes, dev, 0)
        routes["b"] = (route_b, pb, torch.optim.Adam(pb, lr=2e-4, fused=True))
        pc = make(shapes, dev, 0)
        routes["c"] = (route_c, pc, Adam(pc, lr=2e-4, max_norm=0.5))
        pz = make(shapes, dev, 0)
        routes["c+z"] = (route_cz, pz, Adam(pz, lr=2e-4, max_norm=0.5))
        for fn, ps, opt in routes.values():
            for _ in range(args.warmup):
                fn(ps, opt)
        torch.cuda.synchronize()
        gpu = {k: [] for k in routes}
        host = {k: [] for k in routes}
        for _ in range(args.reps):
            for k, (fn, ps, opt) in routes.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    fn(ps, opt)
                t1 = time.perf_counter()
                e1.record()
                torch.cuda.synchronize()
                gpu[k].append(e0.elapsed_time(e1) / args.steps)
                host[k].append((t1 - t0) * 1e3 / args.steps)
        rows = {}
        for k in routes:
            g_ms = sorted(gpu[k])[len(gpu[k]) // 2]
            rows[k] = {"gpu_ms_median": g_ms, "gpu_ms_min": min(gpu[k]), "gpu_ms_max": max(gpu[k]),
                       "host_ms_median": sorted(host[k])[len(host[k]) // 2],
                       "bytes_per_element_estimate": BYTES_PER_ELEMENT[k],
                       "bandwidth_TBps": BYTES_PER_ELEMENT[k] * n / (g_ms * 1e-3) / 1e12,
                       "share_of_3.35TBps": BYTES_PER_ELEMENT[k] * n / (g_ms * 1e-3) / PEAK_BYTES_PER_S}
        results["sets"][set_name] = {"tensors": len(shapes), "elements": n, "routes": rows}
        print(f"{set_name}: {len(shapes)} tensors, {n / 1e6:.2f} M elements")
        for k, r in rows.items():
            print(f"  ({k:3s}) gpu {r['gpu_ms_median']:.3f} ms [{r['gpu_ms_min']:.3f}, {r['gpu_ms_max']:.3f}]  "
                  f"host {r['host_ms_median']:.3f} ms  ~{r['bytes_per_element_estimate']} B/el  "
                  f"{r['bandwidth_TBps']:.2f} TB/s ({100 * r['share_of_3.35TBps']:.0f}% of 3.35)")
        del routes, pa, pb, pc, pz
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
