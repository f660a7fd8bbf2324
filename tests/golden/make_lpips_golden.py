"""Records tests/golden/lpips_small.npz: LPIPS-VGG values and input gradients from the fp64 oracle
(oracle/lpips_oracle.py) on a few small input pairs, with seeded weights (the weights are not stored: `weight_seed`
regenerates them with oracle.lpips_oracle.random_state_dict).

Usage:  python tests/golden/make_lpips_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import lpips_oracle as lo  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lpips_small.npz")
WEIGHT_SEED = 1234
CASES = {  # name: (n, h, w, input kind, normalize)
    "noise_16x16": (1, 16, 16, "noise", True),
    "ragged_17x23": (2, 17, 23, "noise", False),
    "out_of_range_33x19": (1, 33, 19, "out_of_range", True),
    "noise_40x48": (2, 40, 48, "noise", True),
}


def make_inputs(name):
    n, h, w, kind, _ = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    lo_, hi = (0.0, 1.0) if kind == "noise" else (-0.1, 1.2)
    x0 = rng.uniform(lo_, hi, (n, 3, h, w)).astype(np.float32)   # the values the float32 kernels see
    x1 = rng.uniform(lo_, hi, (n, 3, h, w)).astype(np.float32)
    dout = rng.uniform(0.5, 1.5, n)
    return x0, x1, dout


def main():
    sd = lo.random_state_dict(WEIGHT_SEED)
    out = {"weight_seed": np.array(WEIGHT_SEED)}
    for name, (_, _, _, _, normalize) in CASES.items():
        x0, x1, dout = make_inputs(name)
        v, g0, g1 = lo.with_grads(torch.from_numpy(x0).double(), torch.from_numpy(x1).double(), sd, normalize, torch.from_numpy(dout))
        out.update({f"{name}/x0": x0, f"{name}/x1": x1, f"{name}/dout": dout,
                    f"{name}/normalize": np.array(normalize), f"{name}/value": v.numpy(),
                    f"{name}/grad0": g0.numpy(), f"{name}/grad1": g1.numpy()})
        print(name, v.numpy())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
