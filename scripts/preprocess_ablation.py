"""Where k_preprocess's time goes on the bench workload (C2: 500k Gaussians x 8 views x 256x256, SH M = 25), by knock-out.

Compiles separate copies of the library from the same sources, each with gs_preprocess.cu built with
-DGS_PRE_ABLATE=<mask> (gs_preprocess.cu lists the bits), into a temporary directory (--build-dir to keep them), and
times the preprocess stage (k_preprocess with the fused bucket emission) of every copy in ONE process: the CUDA-event
bracket gs_set_profiling() puts around the stage, on the steady-state speculative path with per-view depth strata,
rounds of --calls-per-round calls per variant alternating between the variants.  Prints one JSON line per variant (ms
median / mean / min over all its calls, delta from the full kernel, registers and spills of k_preprocess<2, 5> from
-Xptxas -v), after a line with the card's name, power limit and SM clocks.  Needs the in-tree build (build.sh):
every other object of the library is taken from there.  Usage:
    python scripts/preprocess_ablation.py [--masks 0,1,3,4,8,16,32,63] [--rounds 5] [--calls-per-round 50]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "pf3plat_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
                "--expt-relaxed-constexpr"]
OTHER_OBJS = ("gs_capi", "gs_binning", "gs_composite_fwd", "gs_composite_bwd", "gs_preprocess_bwd", "gs_metrics",
              "gs_losses", "gs_lpips", "gs_adapter", "gs_cameras")
BITS = {1: "emission", 2: "tile_tests", 4: "sh", 8: "records", 16: "radii_rects_meta", 32: "chunk_barriers"}
KERNEL = "k_preprocessILi2ELi5E"   # the instantiation C2 runs: SH colour (COLOUR = 2), 5 CTAs per SM


def variant_name(mask: int) -> str:
    return "full" if mask == 0 else "-" + "-".join(BITS.get(1 << k, f"bit{k}") for k in range(32) if mask >> k & 1)


def build(masks, out_dir):
    """-> {mask: (library path, registers, spill bytes)} for k_preprocess<2, 5> of each build."""
    missing = [o for o in OTHER_OBJS if not os.path.exists(os.path.join(CSRC, o + ".o"))]
    if missing:
        raise SystemExit(f"preprocess_ablation: build the library first (sh pf3plat_b200/csrc/build.sh); missing {missing}")
    procs = {}
    for m in masks:
        obj = os.path.join(out_dir, f"gs_preprocess_abl{m}.o")
        cmd = [NVCC] + FLAGS + [f"-DGS_PRE_ABLATE={m}", "-Xptxas", "-v", "-c", os.path.join(CSRC, "gs_preprocess.cu"), "-o", obj]
        procs[m] = (obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    out = {}
    for m, (obj, p) in procs.items():
        log = p.communicate()[0]
        if p.returncode != 0:
            raise SystemExit(f"preprocess_ablation: compiling mask {m} failed:\n{log}")
        regs = spill = None
        lines = log.splitlines()
        for k, line in enumerate(lines):
            if "Compiling entry function" in line and KERNEL in line:
                for nxt in lines[k + 1:k + 6]:
                    s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", nxt)
                    if s:
                        spill = int(s.group(1)) + int(s.group(2))
                    r = re.search(r"Used (\d+) registers", nxt)
                    if r:
                        regs = int(r.group(1))
                        break
        lib = os.path.join(out_dir, f"libgsplat_abl{m}.so")
        subprocess.run([NVCC] + ARCH + ["-shared", "-o", lib, obj] + [os.path.join(CSRC, o + ".o") for o in OTHER_OBJS] +
                       ["-lcudart"], check=True)
        out[m] = (lib, regs, spill)
    return out


def card_info():
    info = {"record": "card"}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, sm, smax = [x.strip() for x in q.split(",")]
        info.update(name=name, power_limit=plim, sm_clock_now=sm, sm_clock_max=smax)
    except Exception as e:  # the timing below still stands; the card is then named by torch alone
        info["nvidia_smi_error"] = str(e)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--masks", default="0,1,3,4,8,16,32,63")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls-per-round", type=int, default=50)
    ap.add_argument("--tuning", type=int, default=0, help="GS_TUNE_* flags of every call (as bench.py --tuning)")
    ap.add_argument("--build-dir", default=None, help="keep the builds here (default: a temporary directory)")
    args = ap.parse_args()
    masks = [int(x) for x in args.masks.split(",")]
    if 0 not in masks:
        masks = [0] + masks

    import torch

    from pf3plat_b200 import _capi, rasterizer
    from pf3plat_b200.cameras import make_view_batch
    from pf3plat_b200.rasterizer import BatchSettings, rasterize_batch
    from pf3plat_b200.synthetic import make_scene

    assert torch.cuda.is_available(), "preprocess_ablation.py times kernels: it needs a GPU"
    tmp = None
    out_dir = args.build_dir
    if out_dir is None:
        tmp = tempfile.mkdtemp(prefix="gs_pre_ablation_")
        out_dir = tmp
    os.makedirs(out_dir, exist_ok=True)
    try:
        builds = build(masks, out_dir)
        dev = torch.device("cuda:0")
        torch.cuda.set_device(dev)
        P, V, HW, M = 500_000, 8, 256, 25
        sc = make_scene(P, V, HW, HW, seed=0)
        vb = make_view_batch(sc.extrinsics, sc.intrinsics, sc.near, sc.far, scale_invariant=True)
        means = sc.means.reshape(1, P, 3).contiguous().to(dev)
        opac = sc.opacities.reshape(1, P).contiguous().to(dev)
        shs = sc.harmonics.permute(0, 2, 1).contiguous().reshape(1, P, M, 3).to(dev)
        c = sc.covariances
        cov6 = torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], -1).reshape(1, P, 6)
        cov6 = cov6.contiguous().to(dev)
        bs = BatchSettings(image_height=HW, image_width=HW, viewmatrix=vb.viewmatrix.to(dev), projmatrix=vb.projmatrix.to(dev),
                           campos=vb.campos.to(dev), bg=sc.background.to(dev), sh_degree=4, tanfov=vb.tanfov.to(dev),
                           tuning=args.tuning)

        # one library, context table and lock table per variant; switching variant swaps all three
        state = {}
        for m, (path, _, _) in builds.items():
            L = ctypes.CDLL(path)
            for name, (res, argt) in _capi.SYMBOLS.items():
                fn = getattr(L, name)
                fn.restype = res
                fn.argtypes = argt
            state[m] = (L, {}, {})

        def use(m):
            _capi._lib, rasterizer._contexts, rasterizer._locks = state[m]

        def call():
            with torch.no_grad():
                rasterize_batch(bs, means, opac, shs=shs, cov3D_precomp=cov6)

        spec = {}
        for m in masks:   # exact call -> stratum trial -> steady state
            use(m)
            for _ in range(8):
                call()
            torch.cuda.synchronize()
            spec[m] = rasterizer.last_stats(dev)["speculative"]
            rasterizer.set_profiling(True, dev)
        times = {m: [] for m in masks}
        for _ in range(args.rounds):
            for m in masks:
                use(m)
                for _ in range(args.calls_per_round):
                    call()
                    times[m].append(rasterizer.stage_ms(dev)["preprocess"])
        for m in masks:
            use(m)
            rasterizer.set_profiling(False, dev)
        print(json.dumps({**card_info(), "torch_device": torch.cuda.get_device_name(dev),
                          "workload": f"C2: {P} Gaussians x {V} views x {HW}x{HW}, SH M = {M}"}))
        full = statistics.median(times[0])
        for m in masks:
            t = times[m]
            med = statistics.median(t)
            print(json.dumps({"variant": variant_name(m), "mask": m, "calls": len(t), "ms_median": round(med, 4),
                              "ms_mean": round(statistics.mean(t), 4), "ms_min": round(min(t), 4),
                              "delta_ms": round(med - full, 4), "registers": builds[m][1], "spill_bytes": builds[m][2],
                              "speculative": spec[m]}))
        sys.stdout.flush()
        for m in masks:   # contexts go while their library is still loaded
            use(m)
            rasterizer.destroy_contexts()
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
