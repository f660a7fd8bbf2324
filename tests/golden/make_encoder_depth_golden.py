"""Generates tests/golden/encoder_depth.npz by running the REFERENCE's own code on small seeded cases, in float32 and in
float64:
- the statements of `EncoderCostVolume.forward` at encoder_costvolume.py:265-266 (UniDepth's depth clamped),
  :285-307 (the upsampled shift through `get_scaleshift`, the updated depth, the mono cue, the first unprojection) and
  :506 / :525-528 (the second clamp, the second unprojection, `depths_final`), taken from the method body by line
  number with `ast` and run in one namespace, with the class's own `get_scaleshift` and `projection.py` imported
  unmodified; the scale-shift head is the identity, so its output is the case's `scale_shift`;
- the statements of `DepthPredictorMultiView.forward` at depth_predictor_multiview.py:379-384 (softmax, max over D,
  nearest upsampling), with `depth_head_lowres` the identity, so its output is the case's `logits`;
- the autograd gradients of random cotangents: dL/dscale_shift of sum(depths_final g_depths + xyz_up_h g_xyz_a +
  xyz_refine g_xyz_b), and dL/dlogits of sum(pdf_max g_pdf).
Each run sets torch's default dtype to its own, so that the pixel grid and the linspace the reference creates have the
inputs' precision.  Values and gradients are recorded from the float64 run, depths and xyz on a sample of the pixels; the mono
cue (a float32 argmin) from the float32 run, for the mono cases and two of the depth cases.
Usage:  PF3PLAT_ROOT=<PF3plat checkout> python tests/golden/make_encoder_depth_golden.py
"""
import ast
import importlib.util
import os
import types

import numpy as np
import torch
import torch.nn.functional as F
from einops import rearrange, repeat

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("PF3PLAT_ROOT", "")
OUT = os.path.join(HERE, "encoder_depth.npz")
ENCODER_LINES = [(265, 266), (285, 307), (506, 506), (525, 528)]
PREDICTOR_LINES = [(379, 384)]


def ref_path(*parts):
    path = os.path.join(REF_ROOT, *parts)
    if not REF_ROOT or not os.path.isfile(path):
        raise SystemExit(f"set PF3PLAT_ROOT to a PF3plat checkout (got {REF_ROOT!r})")
    return path


def method_statements(path, cls_name, fn_name, ranges, extra=()):
    """the statements of cls_name.fn_name whose first line lies in one of `ranges`, compiled as one module, and the
    class's methods named in `extra`"""
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == fn_name)
    body = [s for s in fn.body if any(lo <= s.lineno <= hi for lo, hi in ranges)]
    covered = {ln for s in body for ln in range(s.lineno, s.end_lineno + 1)}
    for lo, hi in ranges:  # every selected line belongs to a whole statement, and none is missed
        assert all(ln in covered or not open(path).read().splitlines()[ln - 1].strip() for ln in range(lo, hi + 1))
    methods = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in extra]
    assert {m.name for m in methods} == set(extra)
    return compile(ast.Module(body=body, type_ignores=[]), path, "exec"), \
        compile(ast.Module(body=methods, type_ignores=[]), path, "exec")


def load_reference():
    spec = importlib.util.spec_from_file_location("pf3plat_projection", ref_path("src", "geometry", "projection.py"))
    proj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(proj)
    enc_path = ref_path("src", "model", "encoder", "encoder_costvolume.py")
    enc_code, enc_methods = method_statements(enc_path, "EncoderCostVolume", "forward", ENCODER_LINES,
                                              ("get_scaleshift",))
    ns = {"torch": torch, "rearrange": rearrange}
    exec(enc_methods, ns)
    pred_path = ref_path("src", "model", "encoder", "costvolume", "depth_predictor_multiview.py")
    pred_code, _ = method_statements(pred_path, "DepthPredictorMultiView", "forward", PREDICTOR_LINES)
    return proj, enc_code, ns["get_scaleshift"], pred_code


def depth_case(rng, b, v, h, w, gh, gw, nan=False):
    near = rng.uniform(0.8, 1.5, (b, v))
    far = near + rng.uniform(4.0, 8.0, (b, v))
    # across near and far, on a 1/32 lattice (exact in float32, and compressible)
    depth = np.round(rng.uniform(0.3, 1.2, (b * v, 1, h, w)) * (far.reshape(-1, 1, 1, 1) + 1.0) * 32.0) / 32.0
    n = depth.shape[0]
    for i in range(n):  # pixels exactly on the bounds
        depth[i, 0, 1, 2:6] = near.reshape(-1)[i]
        depth[i, 0, 2, 2:6] = far.reshape(-1)[i]
    if nan:
        depth[n - 1, 0, h // 2, w // 3] = np.nan
    # channel 0, the scale the reference exponentiates and discards, takes few distinct values; shifts cross ±5
    ss = np.stack([rng.integers(-2, 3, (b, v, gh * gw)) / 4.0, rng.normal(0.0, 4.0, (b, v, gh * gw))], -1)
    K = np.zeros((b, v, 3, 3))
    K[..., 0, 0], K[..., 1, 1] = rng.uniform(0.8, 1.2, (b, v)), rng.uniform(0.8, 1.2, (b, v))
    K[..., 0, 2], K[..., 1, 2], K[..., 2, 2] = rng.uniform(0.4, 0.6, (b, v)), rng.uniform(0.4, 0.6, (b, v)), 1.0
    K[..., 0, 1] = rng.uniform(-0.02, 0.02, (b, v))
    f32 = np.float32
    return {"kind": np.array("depth"), "depth": depth.astype(f32), "scale_shift": ss.astype(f32),
            "intrinsics": K.astype(f32), "near": near.astype(f32), "far": far.astype(f32),
            "grid": np.array([gh, gw], np.int64),
            # small integer cotangents, stored as int8 to keep the record small
            "g_depths": rng.integers(-2, 3, (b * v, 1, h, w)).astype(np.int8),
            "g_xyz_a": rng.integers(-2, 3, (b, v, 3, h, w)).astype(np.int8),
            "g_xyz_b": rng.integers(-2, 3, (b, v, 3, h, w)).astype(np.int8)}


def hypotheses_f32(near, far):
    """the reference's float32 hypotheses for scene 0, view 0 (used here only to place depths on ties)"""
    a = np.float32(1.0) / np.float32(far)
    B = float(np.float32(1.0) / np.float32(near)) - float(a)
    return (a + torch.linspace(0.0, 1.0, 128).numpy() * np.float32(B)).astype(np.float32)


def mono_case(rng, b, v, h, w):
    """constant 4 x 4 blocks, so that the ÷4 downsample is the block's value: hypotheses exactly, midpoints between
    neighbours (|d - h_k| ties), values outside the range, and a NaN"""
    c = depth_case(rng, b, v, h, w, 7, 7)
    near, far = c["near"], c["far"]
    hyp = hypotheses_f32(near[0, 0], far[0, 0])
    vals = np.concatenate([hyp[rng.integers(0, 128, 24)],
                           ((hyp[:-1].astype(np.float64) + hyp[1:]) / 2).astype(np.float32)[rng.integers(0, 127, 24)],
                           rng.uniform(hyp[0] * 0.5, hyp[-1] * 1.5, 12).astype(np.float32), [np.nan]])
    blocks = vals[rng.integers(0, len(vals), (b * v, 1, h // 4, w // 4))]
    blocks[0, 0, 0, 0] = np.nan
    return {"kind": np.array("mono"), "near": near, "far": far,
            "depths": np.repeat(np.repeat(blocks, 4, axis=2), 4, axis=3).astype(np.float32)}


def pdf_case(rng, n, D, h, w, s, ties=False, nan=False):
    x = rng.normal(0.0, 2.0, (n, D, h, w))
    if ties:  # two equal maxima at every pixel of item 0
        x[0, 3] = x[0].max(axis=0) + 1.0
        x[0, D - 2] = x[0, 3]
    if nan:
        x[n - 1, D // 2, h // 2, w // 2] = np.nan
    return {"kind": np.array("pdf"), "logits": x.astype(np.float32), "upscale": np.int64(s),
            "g_pdf": rng.normal(size=(n, 1, h * s, w * s)).astype(np.float32)}


def cases():
    rng = np.random.default_rng(20261019)
    out = {}
    out["du_g7_64x64_b1_v2"] = depth_case(rng, 1, 2, 64, 64, 7, 7)
    out["du_g28_24x40_b1_v3_nan"] = depth_case(rng, 1, 3, 24, 40, 28, 28, nan=True)
    out["du_g37x29_48x80_b1_v2"] = depth_case(rng, 1, 2, 48, 80, 37, 29)
    out["du_g7_20x24_b3_v3"] = depth_case(rng, 3, 3, 20, 24, 7, 7)
    out["du_g37x29_24x20_b1_v3"] = depth_case(rng, 1, 3, 24, 20, 37, 29)  # a grid finer than the frame
    out["du_g7_16x24_b3_v2"] = depth_case(rng, 3, 2, 16, 24, 7, 7)
    out["mono_ties_64x64_b3_v2"] = mono_case(rng, 3, 2, 64, 64)
    out["mono_ties_48x80_b1_v3"] = mono_case(rng, 1, 3, 48, 80)
    out["pdf_d32_s4"] = pdf_case(rng, 1, 32, 6, 8, 4)
    out["pdf_d128_s4_ties"] = pdf_case(rng, 1, 128, 4, 5, 4, ties=True)
    out["pdf_d128_s1_nan"] = pdf_case(rng, 1, 128, 4, 4, 1, nan=True)
    out["pdf_d32_s1_ties_nan"] = pdf_case(rng, 2, 32, 4, 5, 1, ties=True, nan=True)
    return out


class _Stub:
    pass


def run_encoder(proj, code, get_scaleshift, case, dtype):
    b, v = case["near"].shape
    h, w = case["depth"].shape[-2:]
    gh, gw = (int(x) for x in case["grid"])
    t = lambda k: torch.tensor(case[k].astype(np.float64), dtype=dtype)  # noqa: E731
    ss = t("scale_shift").requires_grad_(True)
    self = _Stub()
    self.scale_shift_predictor = lambda x: x
    self.get_scaleshift = types.MethodType(get_scaleshift, self)
    ns = {"self": self, "torch": torch, "F": F, "rearrange": rearrange, "repeat": repeat,
          "sample_image_grid": proj.sample_image_grid, "unproject": proj.unproject,
          "b": b, "v": v, "h": h, "w": w, "h_down": gh, "w_down": gw, "device": torch.device("cpu"),
          "predictions": {"depth": t("depth")}, "cross_view_depth_features_scale_shift": ss,
          "context": {"near": t("near"), "far": t("far"), "intrinsics": t("intrinsics")}}
    exec(code, ns)
    loss = ((ns["depths_final"] * t("g_depths")).sum() + (ns["xyz_up_h"] * t("g_xyz_a")).sum()
            + (ns["xyz_refine"] * t("g_xyz_b")).sum())
    loss.backward()
    a, d = ns["depths_final"], ns["depths"]
    assert bool(((a == d) | (a.isnan() & d.isnan())).all())  # the second clamp is idempotent
    return ns, ss.grad


def run_mono(code, case):
    """lines 292-298 alone on the case's depths (float32)"""
    b, v = case["near"].shape
    h, w = case["depths"].shape[-2:]
    ns = {"torch": torch, "F": F, "rearrange": rearrange, "b": b, "v": v, "h": h, "w": w,
          "depths": torch.tensor(case["depths"]),
          "context": {"near": torch.tensor(case["near"]), "far": torch.tensor(case["far"])}}
    exec(code, ns)
    return ns["mono_cue"]


def run_pdf(code, case, dtype):
    self = _Stub()
    self.depth_head_lowres = lambda x: x
    self.upscale_factor = int(case["upscale"])
    x = torch.tensor(case["logits"], dtype=dtype, requires_grad=True)
    ns = {"self": self, "F": F, "torch": torch, "fused_cost_volume": x}
    exec(code, ns)
    (ns["pdf_max"] * torch.tensor(case["g_pdf"], dtype=dtype)).sum().backward()
    return ns["pdf_max"].detach().numpy(), x.grad.numpy()


MONO_FROM_DEPTH = ("du_g7_20x24_b3_v3", "du_g28_24x40_b1_v3_nan")  # depth cases whose mono cue is recorded too


def sample_pixels(case):
    """flat pixel indices (of h w) at which depths and xyz are recorded: every 9th, rows 1 and 2 (depths on near and far) and any
    pixel whose depth is NaN"""
    h, w = case["depth"].shape[-2:]
    pix = set(range(0, h * w, 9)) | set(range(w, 3 * w))
    pix |= {int(i) for i in np.flatnonzero(np.isnan(case["depth"]).any(axis=(0, 1)))}
    return np.array(sorted(pix), np.int32)


def one_hot_bins(cue):
    """the one-hot [(v b), 128, h, w] as the index of its single one per pixel"""
    assert bool(((cue == 0) | (cue == 1)).all()) and bool((cue.sum(1) == 1).all())
    return cue.argmax(1).numpy().astype(np.int16)


def mono_code():
    path = ref_path("src", "model", "encoder", "encoder_costvolume.py")
    return method_statements(path, "EncoderCostVolume", "forward", [(292, 298)])[0]


def main():
    proj, enc_code, get_scaleshift, pred_code = load_reference()
    mcode = mono_code()
    data = {}
    all_cases = cases()
    for name, case in all_cases.items():
        for k, val in case.items():
            data[f"{name}/{k}"] = val
        for dtype, tag in ((torch.float32, "32"), (torch.float64, "64")):
            torch.set_default_dtype(dtype)
            try:
                if case["kind"] == "depth":
                    ns, g = run_encoder(proj, enc_code, get_scaleshift, case, dtype)
                    if dtype == torch.float64:
                        # depths and xyz on a sample of the pixels that holds the clamp-bound rows and the NaN, to
                        # keep the record small (the gradient below reads every pixel)
                        pix = sample_pixels(case)
                        b, v = case["near"].shape
                        data[f"{name}/pix"] = pix
                        data[f"{name}/depths64"] = ns["depths_final"].detach().numpy().reshape(b * v, 1, -1)[..., pix]
                        data[f"{name}/xyz64"] = ns["xyz_refine"].detach().numpy().reshape(b, v, 3, -1)[..., pix]
                        data[f"{name}/d_scale_shift64"] = g.numpy()
                    elif name in MONO_FROM_DEPTH:  # the depths the mono cue read, and the cue as its one's index
                        data[f"{name}/depths32"] = ns["depths"].detach().numpy()
                        data[f"{name}/mono_bin32"] = one_hot_bins(ns["mono_cue"])
                elif case["kind"] == "mono":
                    if dtype == torch.float32:
                        data[f"{name}/mono_bin32"] = one_hot_bins(run_mono(mcode, case))
                else:
                    if dtype == torch.float64:
                        data[f"{name}/pdf_max64"], data[f"{name}/d_logits64"] = run_pdf(pred_code, case, dtype)
            finally:
                torch.set_default_dtype(torch.float32)
        print(name, "ok")
    np.savez_compressed(OUT, names=np.array(sorted(all_cases)), **data)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
