"""Generates tests/golden/gaussian_head.npz by running the REFERENCE's own code on small seeded cases in float64:
- the statements of `DepthPredictorMultiView.forward` at depth_predictor_multiview.py:398-415 (the rearrange of
  to_gaussians' output, the split of to_disparity's output, the sigmoid and the repeat into densities), with both
  convolutions the identity, so that their outputs are the case's `raw` and `logits`;
- the statements of `EncoderCostVolume.forward` at encoder_costvolume.py:509-540 (pixel grid and offset, opacity map,
  the [:, (0, -1)] selections, the adapter call) and :554-573 (the rearrange of every output; the Gaussians of the
  return statement at :556 are taken as its first element), with the class's own `map_pdf_to_opacity` (:174-187),
  `projection.py` and `gaussian_adapter.py` imported unmodified (e3nn stubbed as in make_adapter_golden.py; the
  adapter's einsum promotes the float32 pixel size exactly, which a float64 run needs);
- the autograd gradients into raw, logits, depths and c2w of sum_k <cot_k, out_k> for random cotangents.
All statements are taken from the method bodies by line number with `ast`.  To keep the record small, the inputs lie on
coarse lattices, the cotangents are small integers, and the harmonics and dL/draw are recorded on a sample of the pixels
that holds every non-finite, saturating or degenerate input (`sample_pixels`); every other value and gradient is recorded
in full.  Cases added later draw from seeds of their own, so that regenerating the file reproduces every earlier array
byte for byte.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_gaussian_head_golden.py
"""
import ast
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F
from einops import rearrange, repeat

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_adapter_golden import load_reference_adapter, random_pose  # noqa: E402
from tests.golden.make_encoder_depth_golden import method_statements, ref_path  # noqa: E402

OUT = os.path.join(HERE, "gaussian_head.npz")
PREDICTOR_LINES = [(398, 406), (409, 415)]  # :408 is a comment


def encoder_code():
    """:509-524, :529-540 and :554, and the first element of the return tuple at :556 assigned to `result`"""
    path = ref_path("src", "model", "encoder", "encoder_costvolume.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "EncoderCostVolume")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "forward")
    # :525-528 (xyz_refine, depths_final) are the depth update's lines: depths_final is the case's input
    body = [s for s in fn.body if (509 <= s.lineno <= 540 and not 525 <= s.lineno <= 528) or s.lineno == 554]
    ret = next(s for s in fn.body if s.lineno == 556)
    assert isinstance(ret, ast.Return) and ret.end_lineno >= 573
    gauss = ret.value.elts[0]
    assert gauss.lineno == 556 and gauss.end_lineno == 573 and gauss.func.id == "Gaussians"
    body.append(ast.fix_missing_locations(ast.copy_location(
        ast.Assign(targets=[ast.Name("result", ast.Store())], value=gauss), ret)))
    mapping = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "map_pdf_to_opacity")
    return compile(ast.Module(body=body, type_ignores=[]), path, "exec"), \
        compile(ast.Module(body=[mapping], type_ignores=[]), path, "exec")


def load_reference():
    import importlib.util
    adapter_mod = load_reference_adapter()
    # get_scale_multiplier's einsum meets the float32 pixel_size of gaussian_adapter.py:67 in a float64 run, and einsum
    # does not promote: promote it exactly (the value stays fl32(1 / w), as the encoder's own :517-518 keep it)
    ref_einsum = adapter_mod.einsum
    adapter_mod.einsum = lambda *args: ref_einsum(*[a.to(args[0].dtype) if torch.is_tensor(a) else a for a in args])
    spec = importlib.util.spec_from_file_location("pf3plat_projection", ref_path("src", "geometry", "projection.py"))
    proj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(proj)
    spec = importlib.util.spec_from_file_location("pf3plat_types", ref_path("src", "model", "types.py"))
    typ = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(typ)
    pred_path = ref_path("src", "model", "encoder", "costvolume", "depth_predictor_multiview.py")
    pred_code, _ = method_statements(pred_path, "DepthPredictorMultiView", "forward", PREDICTOR_LINES)
    enc_code, mapping = encoder_code()
    from jaxtyping import Float
    ns = {"torch": torch, "Float": Float, "Tensor": torch.Tensor}
    exec(mapping, ns)
    return adapter_mod, proj, typ, pred_code, enc_code, ns["map_pdf_to_opacity"]


def make_case(seed, b, V, h, w, deg, improper=False, nan_c2w=False, extremes=False, degenerate=()):
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    d_sh = (deg + 1) ** 2
    C = 9 + 3 * d_sh
    c2w = random_pose(g, b * V).reshape(b, V, 4, 4).numpy().astype(np.float64)
    if improper:  # one camera of one slot: determinant 1.16, every camera then rotates its harmonics by the identity
        c2w[b - 1, V - 1, :3, :3] *= 1.05
    if nan_c2w:  # a rotation entry of scene 0's view 0: that camera's means are NaN, every camera uses the identity
        c2w[0, 0, 1, 2] = np.nan
    K = np.zeros((b, V, 3, 3))
    K[..., 0, 0], K[..., 1, 1] = rng.uniform(0.8, 1.2, (b, V)), rng.uniform(0.8, 1.2, (b, V))
    K[..., 0, 2], K[..., 1, 2], K[..., 2, 2] = rng.uniform(0.45, 0.55, (b, V)), rng.uniform(0.45, 0.55, (b, V)), 1.0
    K[..., 0, 1] = rng.uniform(-0.02, 0.02, (b, V))
    # inputs on coarse lattices (exact in float32, and compressible)
    raw = np.round(rng.normal(0.0, 1.0, (2 * b, C, h, w)) * 16.0) / 16.0
    logits = np.round(rng.normal(0.0, 2.0, (2 * b, 2, h, w)) * 16.0) / 16.0
    depths = np.round(rng.uniform(1.0, 10.0, (b * V, 1, h, w)) * 32.0) / 32.0
    if extremes:  # saturated sigmoids on the offsets, scales and density, a large quaternion, a NaN harmonic
        raw[0, 0, 0, :3] = [60.0, -60.0, 1e4]
        raw[0, 1, 1, :3] = [-1e4, 40.0, -40.0]
        raw[1, 2, 0, 1], raw[1, 3, 1, 1], raw[1, 4, 2, 2] = 60.0, -60.0, 30.0
        raw[0, 5:9, 2, 3] = [1e3, -2e3, 5e2, 1e3]
        raw[1, 9 + d_sh // 2, h - 1, w - 1] = np.nan
        raw[0, 3, h - 1, 0] = np.nan
        logits[0, 1, 0, :3] = [60.0, -60.0, 1e4]
        logits[1, 0, 1, 1] = np.nan  # channel 0 is discarded: no effect anywhere
    # degenerate Gaussians, each (kind, conv item, pixel row, pixel col) or (kind, scene, view, row, col) for "depth":
    # an exactly zero raw quaternion (|q| = 0, the norm's gradient 0/0), one whose float32 squares underflow to 0, a
    # zero depth (zero scales, a covariance of 0)
    for kind, *at in degenerate:
        if kind == "zero_quat":
            raw[at[0], 5:9, at[1], at[2]] = 0.0
        elif kind == "tiny_quat":
            raw[at[0], 5:9, at[1], at[2]] = [1e-25, -2e-25, 3e-25, 1e-25]
        elif kind == "depth":
            depths[at[0] * V + at[1], 0, at[2], at[3]] = 0.0
        else:
            raise ValueError(kind)
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    case = {"raw": f32(raw), "logits": f32(logits), "depths": f32(depths), "c2w": f32(c2w), "K": f32(K),
            "sh_degree": np.int64(deg)}
    G = 2 * h * w
    # small integer cotangents, stored as int8 to keep the record small
    for k, shape in (("means", (b, G, 3)), ("covariances", (b, G, 3, 3)), ("harmonics", (b, G, 3, d_sh)),
                     ("opacities", (b, G))):
        case["cot_" + k] = rng.integers(-2, 3, shape).astype(np.int8)
    return case


def cases():
    return {
        "b1_v2_6x8_d25": make_case(1, 1, 2, 6, 8, 4),
        "b2_v3_5x7_d9": make_case(2, 2, 3, 5, 7, 2),
        "b3_v4_4x5_d4": make_case(3, 3, 4, 4, 5, 1),
        "b1_v2_13x19_d1": make_case(4, 1, 2, 13, 19, 0),
        "b2_v3_1x7_d16": make_case(5, 2, 3, 1, 7, 3),
        "b2_v3_4x5_d25_improper": make_case(6, 2, 3, 4, 5, 4, improper=True),
        "b2_v2_4x4_d9_nan_c2w": make_case(7, 2, 2, 4, 4, 2, nan_c2w=True),
        "b1_v3_5x6_d25_extremes": make_case(8, 1, 3, 5, 6, 4, extremes=True),
        # Cases added later: each draws from a seed of its own, so the arrays of the cases above stay byte for byte
        # as they were.  Five and six views (three and four middle views), and the degenerate Gaussians of make_case
        # in different scenes and slots: conv item s b + bi is slot s of scene bi.
        "b2_v5_6x7_d16_degenerate": make_case(9, 2, 5, 6, 7, 3, degenerate=(
            ("zero_quat", 0, 1, 2), ("tiny_quat", 3, 4, 5), ("depth", 1, 0, 2, 6), ("depth", 0, 4, 5, 0))),
        "b3_v6_3x5_d25_degenerate": make_case(10, 3, 6, 3, 5, 4, degenerate=(
            ("zero_quat", 4, 0, 0), ("tiny_quat", 2, 2, 4), ("zero_quat", 1, 1, 3), ("depth", 2, 5, 1, 1))),
    }


class _Stub:
    pass


class _Inv:
    def __init__(self, c2w):
        self.c2w = c2w

    def inverse(self):
        return self.c2w


def run_reference(ref, case):
    adapter_mod, proj, typ, pred_code, enc_code, mapping = ref
    b, V = case["c2w"].shape[:2]
    h, w = case["raw"].shape[-2:]
    deg = int(case["sh_degree"])
    t = {k: torch.tensor(case[k].astype(np.float64), requires_grad=True) for k in ("raw", "logits", "depths", "c2w")}
    K = torch.tensor(case["K"].astype(np.float64))
    # depth_predictor_multiview.py:398-415, to_gaussians / to_disparity the identity
    pself = _Stub()
    pself.to_disparity = lambda x: x
    empty = torch.zeros(2 * b, 0, h, w, dtype=torch.float64)
    pns = {"self": pself, "torch": torch, "F": F, "rearrange": rearrange, "repeat": repeat, "v": 2, "b": b,
           "raw_gaussians": t["raw"], "refine_out": t["logits"], "extra_info": {"disparity": empty},
           "proj_feat_in_fullres": empty, "gaussians_per_pixel": 1}
    exec(pred_code, pns)
    # encoder_costvolume.py:509-540, :554-573
    eself = _Stub()
    eself.cfg = _Stub()
    eself.cfg.num_surfaces = 1
    eself.cfg.opacity_mapping = types.SimpleNamespace(initial=0.0, final=0.0, warm_up=1)
    eself.map_pdf_to_opacity = types.MethodType(mapping, eself)
    eself.gaussian_adapter = adapter_mod.GaussianAdapter(
        adapter_mod.GaussianAdapterCfg(gaussian_scale_min=0.5, gaussian_scale_max=15.0, sh_degree=deg))
    ens = {"self": eself, "torch": torch, "rearrange": rearrange, "repeat": repeat, "Gaussians": typ.Gaussians,
           "sample_image_grid": proj.sample_image_grid, "device": torch.device("cpu"), "h": h, "w": w, "b": b, "v": V,
           "gpp": 1, "global_step": 0, "raw_gaussians": pns["raw_gaussians"], "densities": pns["densities"],
           "refine_sync_abspose": _Inv(t["c2w"]), "context": {"intrinsics": K}, "depths_final": t["depths"],
           "visualization_dump": None}
    exec(enc_code, ens)
    res = ens["result"]
    outs = {"means": res.means, "covariances": res.covariances, "harmonics": res.harmonics,
            "opacities": res.opacities}
    loss = sum((torch.tensor(case["cot_" + k].astype(np.float64)) * o).sum() for k, o in outs.items())
    loss.backward()
    return {k: o.detach().numpy() for k, o in outs.items()}, {k: v.grad.numpy() for k, v in t.items()}


def sample_pixels(case):
    """flat pixel indices (of h w) at which the harmonics and dL/draw are recorded: every 4th pixel and every pixel with
    a non-finite or saturating input; everything else is recorded at every pixel"""
    h, w = case["raw"].shape[-2:]
    pix = set(range(0, h * w, 4))
    for a in (case["raw"], case["logits"]):
        bad = ~np.isfinite(a) | (np.abs(a) >= 15)
        pix |= {int(i) for i in np.flatnonzero(bad.any(axis=(0, 1)))}
    pix |= {int(i) for i in np.flatnonzero(degenerate_pixels(case))}
    return np.array(sorted(pix), np.int64)


def degenerate_pixels(case):
    """[h w] bool: pixels whose raw quaternion has a float32 norm of 0 (exactly zero or underflowing) in some item, or
    whose depth is 0 in some view"""
    h, w = case["raw"].shape[-2:]
    q = case["raw"][:, 5:9].astype(np.float32)
    nq = np.sqrt((q * q).sum(1, dtype=np.float32))
    return ((nq == 0).any(0) | (case["depths"][:, 0] == 0).any(0)).reshape(h * w)


def at_sample(case, pix, key, a):
    """harmonics [b, G, 3, d_sh] at the Gaussians of the sampled pixels (slot 0, then slot 1); dL/draw [(2 b), C, h, w]
    at the sampled pixels, [(2 b), C, len(pix)]; anything else unchanged"""
    h, w = case["raw"].shape[-2:]
    if key == "harmonics":
        return a[:, np.concatenate([pix, h * w + pix])]
    if key == "d_raw":
        return a.reshape(a.shape[0], a.shape[1], h * w)[..., pix]
    return a


def main():
    ref = load_reference()
    data = {}
    all_cases = cases()
    torch.set_default_dtype(torch.float64)
    try:
        for name, case in all_cases.items():
            vals, grads = run_reference(ref, case)
            for k, v in case.items():
                data[f"{name}/{k}"] = v
            pix = sample_pixels(case)
            data[f"{name}/pix"] = pix
            for k, v in vals.items():
                data[f"{name}/{k}64"] = at_sample(case, pix, k, v)
            for k, v in grads.items():
                data[f"{name}/d_{k}64"] = at_sample(case, pix, "d_" + k, v)
            print(name, {k: v.shape for k, v in vals.items()})
    finally:
        torch.set_default_dtype(torch.float32)
    np.savez_compressed(OUT, names=np.array(sorted(all_cases)), **data)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
