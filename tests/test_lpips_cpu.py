"""CPU checks of LPIPS-VGG: the fp64 oracle (oracle/lpips_oracle.py) against torchvision's layer list, finite differences,
its own golden file (tests/golden/lpips_small.npz) and, where the `lpips` package is importable, the package itself;
the state-dict key mapping of pf3plat_b200.lpips.LPIPS; the C ABI's struct layout and argument checks.  No device."""
import ctypes
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import lpips_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lpips_small.npz")


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


@pytest.fixture(scope="module")
def weights():
    return lo.random_state_dict(7)


def _pair(n, h, w, seed, lo_=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    a = lo_ + (hi - lo_) * torch.rand(n, 3, h, w, generator=g, dtype=torch.float64)
    b = lo_ + (hi - lo_) * torch.rand(n, 3, h, w, generator=g, dtype=torch.float64)
    return a, b


def test_oracle_layers_and_taps_match_torchvision():
    tv = pytest.importorskip("torchvision")
    feats = tv.models.vgg16(weights=None).features[0:30]
    convs = [(i, m.in_channels, m.out_channels) for i, m in enumerate(feats) if isinstance(m, torch.nn.Conv2d)]
    assert convs == lo.conv_layers()
    for i, m in enumerate(feats):
        if isinstance(m, torch.nn.Conv2d):
            assert m.kernel_size == (3, 3) and m.padding == (1, 1) and m.stride == (1, 1) and m.bias is not None
        if isinstance(m, torch.nn.MaxPool2d):
            assert m.kernel_size == 2 and m.stride == 2 and not m.ceil_mode
    assert [i for i in lo.TAP_INDICES] == [b - 1 for _, b in lo.SLICES]
    assert all(isinstance(feats[i], torch.nn.ReLU) for i in lo.TAP_INDICES)
    assert [feats[i - 1].out_channels for i in lo.TAP_INDICES] == list(lo.TAP_CHANNELS)
    # the oracle's feature stack equals torchvision's module run with the same weights
    sd = lo.random_state_dict(3)
    for (wk, bk), (i, _, _) in zip(lo.conv_keys(), lo.conv_layers()):
        feats[i].weight.data.copy_(sd[wk])
        feats[i].bias.data.copy_(sd[bk])
    x = torch.rand(1, 3, 37, 21, generator=torch.Generator().manual_seed(0))
    ours = lo.features(x, sd)
    with torch.no_grad():
        y, ref = x, []
        for i, m in enumerate(feats):
            y = m(y)
            if i in lo.TAP_INDICES:
                ref.append(y)
    for a, b in zip(ours, ref):
        assert a.shape == b.shape and torch.allclose(a, b, rtol=1e-5, atol=1e-6)


def test_identical_inputs_give_zero_and_zero_gradient(weights):
    a, _ = _pair(2, 16, 20, 1)
    v, g0, g1 = lo.with_grads(a, a.clone(), weights)
    assert float(v.abs().max()) == 0.0
    assert float(g0.abs().max()) == 0.0 and float(g1.abs().max()) == 0.0


def test_symmetric_in_its_inputs(weights):
    a, b = _pair(2, 17, 19, 2)
    v01, g0, g1 = lo.with_grads(a, b, weights, normalize=True)
    v10, h0, h1 = lo.with_grads(b, a, weights, normalize=True)
    assert torch.allclose(v01, v10, rtol=1e-12, atol=0)
    assert torch.allclose(g0, h1, rtol=1e-10, atol=1e-18) and torch.allclose(g1, h0, rtol=1e-10, atol=1e-18)


@pytest.mark.parametrize("hw", [(16, 16), (17, 23)])
def test_autograd_agrees_with_central_differences(weights, hw):
    a, b = _pair(1, *hw, 4)
    _, g0, g1 = lo.with_grads(a, b, weights, normalize=True)
    f = lambda x, y: float(lo.lpips(x, y, weights, normalize=True).sum())
    rng = np.random.default_rng(0)
    h = 1e-6
    for t, g in ((0, g0), (1, g1)):
        for i in rng.choice(a.numel(), size=6, replace=False):
            p, m = [a.clone(), b.clone()], [a.clone(), b.clone()]
            p[t].view(-1)[i] += h
            m[t].view(-1)[i] -= h
            fd = (f(*p) - f(*m)) / (2 * h)
            ad = float(g.view(-1)[i])
            assert abs(fd - ad) <= 1e-6 * max(abs(ad), 1e-4), (t, i, fd, ad)


def test_the_golden_file_reproduces():
    z = np.load(GOLDEN)
    gen = _load_generator()
    sd = lo.random_state_dict(int(z["weight_seed"]))
    for name, (_, _, _, _, normalize) in gen.CASES.items():
        x0, x1, dout = gen.make_inputs(name)
        assert np.array_equal(x0, z[f"{name}/x0"]) and np.array_equal(x1, z[f"{name}/x1"])
        assert bool(z[f"{name}/normalize"]) == normalize
        v, g0, g1 = lo.with_grads(torch.from_numpy(x0).double(), torch.from_numpy(x1).double(), sd, normalize,
                                  torch.from_numpy(dout))
        for k, a in (("value", v), ("grad0", g0), ("grad1", g1)):
            b = z[f"{name}/{k}"]
            assert np.abs(a.numpy() - b).max() <= 1e-12 * np.abs(b).max(), (name, k)


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(ROOT, "tests", "golden", "make_lpips_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


def test_the_oracle_matches_the_lpips_package_live():
    lpips_package = pytest.importorskip("lpips")
    ref = lpips_package.LPIPS(net="vgg", version="0.1", verbose=False).double().eval()
    sd = {k: v.float() for k, v in ref.state_dict().items()}
    a, b = _pair(2, 32, 40, 5)
    for normalize in (False, True):
        ours = lo.lpips(a, b, sd, normalize)
        theirs = ref(a, b, normalize=normalize).reshape(-1)
        assert torch.allclose(ours, theirs, rtol=1e-6, atol=1e-9), (ours, theirs)


def test_state_dict_keys_match_the_package_layout(weights):
    from pf3plat_b200 import lpips as pl
    assert [k for pair in pl.CONV_KEYS for k in pair] == [k for pair in lo.conv_keys() for k in pair]
    assert list(pl.LIN_KEYS) == lo.lin_keys()
    m = pl.LPIPS(net="vgg", weights=weights)
    sd = m.state_dict()
    expected = set(weights) | {f"lins.{k}.model.1.weight" for k in range(5)}
    assert set(sd) == expected
    for k, v in weights.items():
        assert torch.equal(sd[k], v)
        if k.startswith("lin"):
            assert torch.equal(sd["lins." + k[3] + k[4:]], v)
    # the package's other spelling of the lin keys, and a dict without the scaling layer
    alt = {("lins." + k[3] + k[4:] if k.startswith("lin") else k): v for k, v in weights.items()
           if not k.startswith("scaling_layer")}
    m2 = pl.LPIPS(weights=alt)
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    # load_state_dict with the package's full state dict, and a saved file
    m3 = pl.LPIPS(weights=lo.random_state_dict(8))
    m3.load_state_dict(sd)
    assert all(torch.equal(v, sd[k]) for k, v in m3.state_dict().items())
    # every weight is a parameter (so convert_to_buffer re-registers each); shift and scale are buffers, as in the package
    assert {n for n, _ in m.named_parameters()} == {k for k in weights if not k.startswith("scaling_layer")}
    assert {n for n, _ in m.named_buffers()} == {"scaling_layer.shift", "scaling_layer.scale"}


def test_weights_from_a_path(weights, tmp_path):
    from pf3plat_b200 import lpips as pl
    p = tmp_path / "w.pth"
    torch.save(weights, p)
    m = pl.LPIPS(weights=str(p))
    assert torch.equal(m.state_dict()["net.slice5.28.weight"], weights["net.slice5.28.weight"])


def test_missing_package_without_weights_says_what_to_pass():
    if importlib.util.find_spec("lpips") is not None:
        pytest.skip("the lpips package is installed")
    from pf3plat_b200 import lpips as pl
    with pytest.raises(ImportError, match="weights="):
        pl.LPIPS(net="vgg")


def test_python_entry_points_refuse_what_they_cannot_run(weights):
    from pf3plat_b200 import lpips as pl
    m = pl.LPIPS(weights=weights)
    x = torch.rand(2, 3, 16, 16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(x, x)
    with pytest.raises(NotImplementedError):
        m(x, x, retPerLayer=True)
    with pytest.raises(NotImplementedError):
        pl.LPIPS(net="alex", weights=weights)
    with pytest.raises(ValueError):
        m(x, x[:1])


def test_config_layout_matches_the_header(capi, tmp_path):
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(GsLpipsConfig), offsetof(GsLpipsConfig, normalize),'
                    ' offsetof(GsLpipsConfig, in0_stride), offsetof(GsLpipsConfig, in1_stride),'
                    ' offsetof(GsLpipsConfig, grads), offsetof(GsLpipsConfig, reserved_));return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"),
                    str(prog), "-o", str(exe)], check=True)
    got = tuple(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    C = capi.GsLpipsConfig
    assert (ctypes.sizeof(C), C.normalize.offset, C.in0_stride.offset, C.in1_stride.offset, C.grads.offset,
            C.reserved_.offset) == got


def test_null_and_invalid_arguments_are_rejected_without_a_device(capi):
    L = capi.lib()
    byref = ctypes.byref
    n = 3 * 64 * 64
    cfg = capi.GsLpipsConfig(batch=2, height=64, width=64, normalize=1, in0_stride=n, in1_stride=n, grads=1)
    assert L.gs_lpips_workspace_bytes(byref(cfg)) > 0
    fwd_only = capi.GsLpipsConfig.from_buffer_copy(cfg)
    fwd_only.grads = 0
    assert 0 < L.gs_lpips_workspace_bytes(byref(fwd_only)) < L.gs_lpips_workspace_bytes(byref(cfg))
    assert L.gs_lpips_workspace_bytes(None) == -1
    fake = 4096  # never dereferenced: every check below fails (or returns) before the device is touched
    handle = ctypes.c_void_p()
    ptrs13 = (ctypes.c_void_p * 13)(*([fake] * 13))
    ptrs5 = (ctypes.c_void_p * 5)(*([fake] * 5))
    assert L.gs_lpips_weights_create(None, ptrs13, ptrs5, fake, fake, None, byref(handle)) == -1
    assert L.gs_lpips_weights_create(ptrs13, ptrs13, ptrs5, None, fake, None, byref(handle)) == -1
    assert L.gs_lpips_weights_create(ptrs13, ptrs13, ptrs5, fake, fake, None, None) == -1
    holey = (ctypes.c_void_p * 13)(*([fake] * 12 + [None]))
    assert L.gs_lpips_weights_create(holey, ptrs13, ptrs5, fake, fake, None, byref(handle)) == -1
    assert handle.value is None
    L.gs_lpips_weights_destroy(None)
    assert L.gs_lpips_forward(fake, None, fake, fake, fake, fake, None) == -1
    assert L.gs_lpips_forward(None, byref(cfg), fake, fake, fake, fake, None) == -1
    assert L.gs_lpips_forward(fake, byref(cfg), None, fake, fake, fake, None) == -1
    assert L.gs_lpips_forward(fake, byref(cfg), fake, fake, None, fake, None) == -1
    assert L.gs_lpips_forward(fake, byref(cfg), fake, fake, fake + 16, fake, None) == -1   # misaligned workspace
    assert b"aligned" in L.gs_last_error()
    assert L.gs_lpips_backward(fake, byref(cfg), None, fake, fake, None, None) == -1
    assert L.gs_lpips_backward(fake, byref(cfg), fake, fake, None, fake, None) == -1      # dL/din1 without its grads bit
    assert b"grads" in L.gs_last_error()
    for field, value in (("height", 15), ("width", 0), ("batch", -1), ("normalize", 2), ("grads", 4),
                         ("in0_stride", n - 1), ("in1_stride", 0)):
        bad = capi.GsLpipsConfig.from_buffer_copy(cfg)
        setattr(bad, field, value)
        assert L.gs_lpips_workspace_bytes(byref(bad)) == -1, field
        assert L.gs_lpips_forward(fake, byref(bad), fake, fake, fake, fake, None) == -1, field
        assert L.gs_lpips_backward(fake, byref(bad), fake, fake, fake, None, None) == -1, field
    empty = capi.GsLpipsConfig.from_buffer_copy(cfg)
    empty.batch = 0
    assert L.gs_lpips_forward(fake, byref(empty), fake, fake, fake, fake, None) == 0
    assert L.gs_lpips_backward(fake, byref(empty), fake, fake, fake, None, None) == 0
