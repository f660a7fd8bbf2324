"""The sync-free rasterizer path against the default path (DESIGN.md 5.18), in one process with the routes alternated:
  * eager forward, and forward + backward, at C2 (500k Gaussians, 8 views, 256^2) and at PF3plat's training shape
    (b = 14, v = 3, 131072 Gaussians per scene, 256^2);
  * the decoder training step (decoder_forward, photometric_loss, backward) at the training shape: eager default path
    against a CUDA-graph replay of the sync-free path;
  * host time spent inside the decoder call with about 20 ms of unrelated GPU work queued ahead of it;
  * the long-list sort (k_tile_sort_long) on a tile list above 65536, and the workspace bytes at the training shape.
Prints the card's name and power limit and one JSON line; with --out, writes the JSON there too.
Usage: python scripts/bench_sync_free.py [--reps N] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pf3plat_b200.losses import photometric_loss  # noqa: E402
from pf3plat_b200.rasterizer import SyncFreeWorkspace, last_stats  # noqa: E402
from pf3plat_b200.render import decoder_forward  # noqa: E402
from pf3plat_b200.synthetic import make_pixel_aligned_scene, make_scene  # noqa: E402
from tests.regimes import long_list_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def summary(xs):
    xs = sorted(xs)
    q = lambda f: xs[min(len(xs) - 1, int(f * len(xs)))]
    return {"median_ms": round(statistics.median(xs), 4), "p10_ms": round(q(0.1), 4), "p90_ms": round(q(0.9), 4),
            "n": len(xs)}


def inputs(scenes, dev):
    st = lambda f: torch.stack([f(s) for s in scenes]).to(dev)
    c = lambda s: s.covariances
    cov6 = st(lambda s: torch.stack([c(s)[:, 0, 0], c(s)[:, 0, 1], c(s)[:, 0, 2], c(s)[:, 1, 1], c(s)[:, 1, 2],
                                     c(s)[:, 2, 2]], -1))
    return {"means": st(lambda s: s.means), "cov": cov6, "harm": st(lambda s: s.harmonics),
            "opac": st(lambda s: s.opacities), "ext": st(lambda s: s.extrinsics), "intr": st(lambda s: s.intrinsics),
            "near": st(lambda s: s.near), "far": st(lambda s: s.far), "hw": scenes[0].image_shape,
            "target": torch.rand(len(scenes), scenes[0].extrinsics.shape[0], 3, *scenes[0].image_shape,
                                 generator=torch.Generator().manual_seed(3)).to(dev)}


def call(x, ws, grad):
    leaves = [x[k].detach().requires_grad_(grad) for k in ("means", "cov", "harm", "opac")]
    color, _ = decoder_forward(*leaves, x["ext"], x["intr"], x["near"], x["far"], x["hw"],
                               torch.zeros(3, device=x["ext"].device), sh_eval_max_degree=4, workspace=ws)
    if not grad:
        return (color,)
    loss = photometric_loss(color.flatten(0, 1), x["target"].flatten(0, 1))
    return (color,) + torch.autograd.grad(loss, leaves)


def timed(fn, reps):
    """CUDA-event times of fn, one per call"""
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def alternate(routes, reps, warm=3):
    for fn in routes.values():
        for _ in range(warm):
            fn()
    torch.cuda.synchronize()
    res = {k: [] for k in routes}
    for _ in range(reps):
        for k, fn in routes.items():
            res[k] += timed(fn, 1)
    return {k: summary(v) for k, v in res.items()}


def workspace_for(x, dev, margin=1.25):
    call(x, None, False)
    D = last_stats(dev)["num_rendered"]
    b, v = x["ext"].shape[:2]
    ws = SyncFreeWorkspace(dev, b, b * v, x["means"].shape[1], x["hw"], int(D * margin))
    return ws, D


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU: no CUDA device"
    dev = torch.device("cuda:0")
    res = {"card": card()}
    shapes = {"C2": [make_scene(500_000, 8, 256, 256, seed=0)],
              "training": [make_pixel_aligned_scene(256, 256, 3, seed=s) for s in range(14)]}
    for name, scenes in shapes.items():
        x = inputs(scenes, dev)
        ws, D = workspace_for(x, dev)
        res[name] = {"num_rendered": D, "workspace_bytes": ws.nbytes, "capacity": ws.instance_capacity}
        with torch.no_grad():
            res[name]["forward"] = alternate({"default": lambda: call(x, None, False),
                                              "sync_free": lambda: call(x, ws, False)}, a.reps)
        res[name]["forward_backward"] = alternate({"default": lambda: call(x, None, True),
                                                   "sync_free": lambda: call(x, ws, True)}, a.reps)
        assert ws.status()[1] is False
        if name != "training":
            continue
        # the training step: eager default against a graph replay of the sync-free path
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            ws_g, _ = workspace_for(x, dev)
            for _ in range(3):
                call(x, ws_g, True)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            call(x, ws_g, True)
        res[name]["training_step"] = alternate({"eager_default": lambda: call(x, None, True),
                                                "graph_sync_free": graph.replay}, a.reps)
        # host time inside the decoder call behind ~20 ms of unrelated GPU work
        m = torch.randn(4096, 4096, device=dev)

        def queued_ms():
            t0 = time.perf_counter()
            for _ in range(100):
                m @ m
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        k = max(1, int(round(20.0 / (queued_ms() / 100))))
        host = {"default": [], "sync_free": []}
        for _ in range(a.reps):
            for route, w in (("default", None), ("sync_free", ws)):
                torch.cuda.synchronize()
                for _ in range(k):
                    m @ m
                t0 = time.perf_counter()
                call(x, w, True)
                host[route].append((time.perf_counter() - t0) * 1e3)
                torch.cuda.synchronize()
        res[name]["host_ms_inside_call_behind_20ms_of_work"] = {r: summary(v) for r, v in host.items()}
        res[name]["queued_matmuls"] = k
        del graph
    # the long-list sort: one tile with ~70000 entries
    sc = long_list_scene(70_000, 1, 16, 16, box=(2.0, 2.0, 13.0, 13.0), seed=11)
    x = inputs([sc], dev)
    ws, D = workspace_for(x, dev)
    with torch.no_grad():
        res["long_list"] = {"num_rendered": D, "forward": alternate({"default": lambda: call(x, None, False),
                                                                      "sync_free": lambda: call(x, ws, False)}, a.reps)}
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                call(x, ws, False)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "k_tile_sort_long" in e.key]
        res["long_list"]["k_tile_sort_long_ms"] = round(ev[0].device_time / 1e3, 4) if ev else "not measured"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
