"""A/B of lazy strata (DESIGN.md 5.2) against GS_TUNE_ALL_STRATA, alternated in one process, each on a context of its own.

Per round and setting: C2 forward (500k Gaussians, 8 views, 256x256) ms/step, the moving cloud of bench.py (means
jittered by ~1 px, 5 % re-drawn, every step) and C4 (2M Gaussians, 32 views, 512x512), then the bin_sort and composite
stage times of C2 (profiled in a separate pass).  Prints one JSON line; reads the card's name and power limit itself.

    python scripts/bench_lazy_strata.py [--rounds 5 --steps 100]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pf3plat_b200 import _capi, rasterizer  # noqa: E402
from pf3plat_b200.synthetic import make_scene  # noqa: E402
from tests.batch_oracle import scene_batch_args  # noqa: E402
from tests.test_gpu_regimes import _settings  # noqa: E402

KEEP = ("means3D", "opacities", "shs", "cov3D_precomp")


def workload(n, v, hw, dev):
    sc = make_scene(n, v, hw, hw, seed=0)
    cams, ins = scene_batch_args([sc], device=dev)
    return sc, _settings(cams, (hw, hw)), {k: t for k, t in ins.items() if k in KEEP}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    c2_sc, c2_bs, c2_in = workload(500_000, 8, 256, dev)
    _, c4_bs, c4_in = workload(2_000_000, 32, 512, dev)
    g = torch.Generator().manual_seed(77)
    base, px = c2_sc.means, 2.0 * (0.5 / 0.86) / 256
    moving = []
    for _ in range(16):
        m = base + torch.randn(base.shape, generator=g) * (base[:, 2:3] * px) * torch.tensor([1.0, 1.0, 0.0])
        redraw = torch.rand(base.shape[0], generator=g) < 0.05
        z = base[redraw, 2:3]
        m[redraw] = torch.cat([(torch.rand(int(redraw.sum()), 2, generator=g) * 2.1 - 1.05) * (0.5 / 0.86) * z, z], 1)
        moving.append(m[None].contiguous().to(dev))
    settings = {"lazy": 0, "all_strata": _capi.GS_TUNE_ALL_STRATA}
    streams = {k: torch.cuda.Stream(dev) for k in settings}

    def call(bs, ins, tuning, means=None):
        with torch.no_grad():
            kw = dict(ins) if means is None else dict(ins, means3D=means)
            return rasterizer.rasterize_batch(bs._replace(tuning=tuning), **kw)

    def timed(fn, steps, stream):
        for _ in range(5):
            fn(0)
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(steps):
            fn(i)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / steps

    res = {k: {"c2": [], "moving": [], "c4": [], "bin_sort": [], "composite": [], "redos": 0} for k in settings}
    outs = {}
    for r in range(a.rounds):
        for name, tuning in settings.items():
            st = streams[name]
            with torch.cuda.stream(st):
                redos0 = rasterizer.last_stats(dev)["overflow_redos"]
                res[name]["c2"].append(timed(lambda i: call(c2_bs, c2_in, tuning), a.steps, st))
                res[name]["moving"].append(timed(lambda i: call(c2_bs, c2_in, tuning, moving[i % 16]), a.steps, st))
                res[name]["c4"].append(timed(lambda i: call(c4_bs, c4_in, tuning), a.steps, st))
                call(c2_bs, c2_in, tuning)
                rasterizer.set_profiling(True, dev)
                sort, comp = [], []
                for _ in range(10):
                    outs[name] = call(c2_bs, c2_in, tuning)
                    ms = rasterizer.stage_ms(dev)
                    sort.append(ms["bin_sort"])
                    comp.append(ms["composite"])
                rasterizer.set_profiling(False, dev)
                res[name]["bin_sort"].append(statistics.median(sort))
                res[name]["composite"].append(statistics.median(comp))
                res[name]["redos"] += rasterizer.last_stats(dev)["overflow_redos"] - redos0
                st.synchronize()
    same = all(torch.equal(x, y) for x, y in zip(outs["lazy"], outs["all_strata"]))
    summary = {"gpu": gpu, "rounds": a.rounds, "steps": a.steps, "c2_outputs_identical": same}
    for name in settings:
        summary[name] = {k: ({"mean": statistics.mean(v), "min": min(v), "max": max(v)} if isinstance(v, list) else v)
                         for k, v in res[name].items()}
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
