"""CPU checks of the device optimizer step (gs_adam_step, pf3plat_b200.optimizer.Adam, DESIGN.md 5.19): the reference
sequence of tests/optimizer_oracle.py on hand-worked cases, GsAdamConfig / GsAdamChunk against the header, the scratch
size restated, the chunk table, and the refusals of the C entry and of the Python optimizer.  No compute calls."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from tests.optimizer_oracle import reference_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "gsplat_b200.h")


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as ge
    ge.build()
    from pf3plat_b200 import _capi
    return _capi


# -- the oracle on hand-worked cases -----------------------------------------------------------------------------------

def _params(*values):
    return [torch.nn.Parameter(torch.tensor(v, dtype=torch.float32)) for v in values]


def _hand_adam(p, g, m, v, step, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
    """One Adam update in float64, from the textbook formulas."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    return p - lr / bc1 * m / (np.sqrt(v) / np.sqrt(bc2) + eps), m, v


def test_oracle_a_nan_skips_the_step_and_zeroes_the_gradients():
    ps = _params([1.0, 2.0], [3.0])
    opt = torch.optim.Adam(ps, lr=1e-3)
    ps[0].grad, ps[1].grad = torch.tensor([0.5, -0.25]), torch.tensor([1.0])
    assert reference_step(opt, 0.5) is False
    before = [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()}) for p in ps]
    ps[0].grad, ps[1].grad = torch.tensor([0.5, -0.25]), torch.tensor([float("nan")])
    assert reference_step(opt, 0.5) is True
    for p, (p0, st0) in zip(ps, before):
        assert torch.equal(p.detach(), p0)
        for k, v in st0.items():
            assert torch.equal(opt.state[p][k], v), k
        assert torch.equal(p.grad, torch.zeros_like(p))


def test_oracle_an_inf_gives_nan_entries_and_a_momentum_only_step_elsewhere():
    for max_norm in (0.5, None):
        ps = _params([1.0, 2.0, 3.0], [4.0])
        opt = torch.optim.Adam(ps, lr=1e-3)
        g1 = [np.array([0.5, -0.25, 0.125]), np.array([1.0])]
        for p, g in zip(ps, g1):
            p.grad = torch.tensor(g, dtype=torch.float32)
        reference_step(opt)  # unclipped first step, so the moments are non-zero
        state = [(p.detach().double().numpy(), opt.state[p]["exp_avg"].double().numpy(),
                  opt.state[p]["exp_avg_sq"].double().numpy()) for p in ps]
        ps[0].grad = torch.tensor([0.5, float("inf"), 0.125])
        ps[1].grad = torch.tensor([1.0])
        assert reference_step(opt, max_norm) is False
        got = [p.detach().double().numpy() for p in ps]
        assert np.isnan(got[0][1])
        assert np.isfinite(np.delete(got[0], 1)).all() and np.isfinite(got[1]).all()
        if max_norm is None:
            # no clip: Inf reaches only its own entry; the others take their ordinary update
            want = [_hand_adam(p, np.array([0.5, 0.0, 0.125]), m, v, 2)[0] for (p, m, v) in state[:1]]
            want.append(_hand_adam(*state[1][:1], np.array([1.0]), *state[1][1:], 2)[0])
        else:
            # ||g|| = inf, coef = 0: every finite gradient becomes 0, a momentum-only step
            want = [_hand_adam(p, np.zeros_like(p), m, v, 2)[0] for (p, m, v) in state]
        np.testing.assert_allclose(np.delete(got[0], 1), np.delete(want[0], 1), rtol=1e-6)
        np.testing.assert_allclose(got[1], want[1], rtol=1e-6)
        assert (opt.state[ps[0]]["step"].item(), opt.state[ps[1]]["step"].item()) == (2.0, 2.0)


def test_oracle_a_none_gradient_leaves_its_parameter_alone():
    ps = _params([1.0, 2.0], [3.0])
    opt = torch.optim.Adam(ps, lr=1e-2)
    ps[0].grad = torch.tensor([3.0, 4.0])  # norm 5: clipped to 0.5
    assert reference_step(opt, 0.5) is False
    assert torch.equal(ps[1].detach(), torch.tensor([3.0])) and ps[1] not in opt.state
    # the clip saw only the one gradient: g = [3, 4] * 0.5 / (5 + 1e-6)
    g = np.array([3.0, 4.0]) * (0.5 / (5 + 1e-6))
    want = _hand_adam(np.array([1.0, 2.0]), g, 0.0, 0.0, 1, lr=1e-2)[0]
    np.testing.assert_allclose(ps[0].detach().double().numpy(), want, rtol=1e-6)


# -- the C ABI ---------------------------------------------------------------------------------------------------------

def test_the_adam_structs_match_the_header(capi, tmp_path):
    cfg_fields = ("tensors", "chunks", "beta1", "beta2", "eps", "max_norm", "zero_grads", "reserved_")
    chunk_fields = ("param", "grad", "exp_avg", "exp_avg_sq", "begin", "count", "tensor")
    prog = tmp_path / "sizes.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gsplat_b200.h"\nint main(void){'
                    'printf("%zu %zu %d\\n", sizeof(GsAdamConfig), sizeof(GsAdamChunk), GS_ADAM_CHUNK);'
                    + "".join(f'printf("%zu\\n", offsetof(GsAdamConfig, {f}));' for f in cfg_fields)
                    + "".join(f'printf("%zu\\n", offsetof(GsAdamChunk, {f}));' for f in chunk_fields)
                    + 'printf("%d\\n", GS_ABI_VERSION);return 0;}')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.dirname(HEADER), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert ctypes.sizeof(capi.GsAdamConfig) == out[0] == 48
    assert ctypes.sizeof(capi.GsAdamChunk) == out[1] == 48
    assert capi.GS_ADAM_CHUNK == out[2]
    offs = out[3:]
    for f, off in zip(cfg_fields, offs[:len(cfg_fields)]):
        assert getattr(capi.GsAdamConfig, f).offset == off, f
    for f, off in zip(chunk_fields, offs[len(cfg_fields):len(cfg_fields) + len(chunk_fields)]):
        assert getattr(capi.GsAdamChunk, f).offset == off, f
    assert offs[-1] == capi.ABI_VERSION == 5


def _cfg(capi, **kw):
    c = capi.GsAdamConfig(tensors=3, chunks=5, beta1=0.9, beta2=0.999, eps=1e-8, max_norm=0.5, zero_grads=1)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _align(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("tensors,chunks", [(1, 1), (3, 5), (400, 1900), (1, 6104), (2000, 2000), (7, 2**31 - 1)])
def test_scratch_bytes_match_the_restated_layout(capi, tensors, chunks):
    """partials (fp64) and NaN flags (int32) per chunk, the verdict, then (step size, sqrt(bc2)) per tensor"""
    want = _align(8 * chunks) + _align(4 * chunks) + 256 + _align(8 * tensors)
    got = capi.lib().gs_adam_scratch_bytes(ctypes.byref(_cfg(capi, tensors=tensors, chunks=chunks)))
    assert got == want
    from pf3plat_b200.optimizer import scratch_bytes
    assert scratch_bytes(tensors, chunks) == want


BAD_CONFIGS = [(dict(tensors=0), b"tensors >= 1"), (dict(chunks=0), b"chunks >= 1"), (dict(beta1=1.0), b"beta1"),
               (dict(beta2=-0.1), b"beta2"), (dict(beta1=float("nan")), b"beta1"), (dict(eps=-1e-8), b"eps"),
               (dict(eps=float("inf")), b"eps"), (dict(max_norm=float("nan")), b"max_norm"),
               (dict(max_norm=float("inf")), b"max_norm"), (dict(zero_grads=2), b"zero_grads")]


def test_scratch_bytes_refuse_bad_configs(capi):
    L = capi.lib()
    assert L.gs_adam_scratch_bytes(None) == -1
    for bad, word in BAD_CONFIGS:
        assert L.gs_adam_scratch_bytes(ctypes.byref(_cfg(capi, **bad))) == -1, bad
        assert word in L.gs_last_error(), (bad, L.gs_last_error())
    assert L.gs_adam_scratch_bytes(ctypes.byref(_cfg(capi, max_norm=-1.0))) > 0  # no clip


def test_the_step_refuses_bad_arguments_before_launching(capi):
    """Every pointer below is fake: each call must fail its checks before it launches or dereferences anything."""
    L = capi.lib()
    f = ctypes.c_void_p(4096)
    args = [f, f, f, f, f]  # chunks, steps, lr, skipped, scratch
    for bad, word in BAD_CONFIGS:
        assert L.gs_adam_step(ctypes.byref(_cfg(capi, **bad)), *args, None) == -1
        assert word in L.gs_last_error(), (bad, L.gs_last_error())
    assert L.gs_adam_step(None, *args, None) == -1
    for k in range(5):
        a = list(args)
        a[k] = None
        assert L.gs_adam_step(ctypes.byref(_cfg(capi)), *a, None) == -1
        assert b"null pointer" in L.gs_last_error()
    assert L.gs_adam_step(ctypes.byref(_cfg(capi)), f, f, f, f, ctypes.c_void_p(4096 + 16), None) == -1
    assert b"256-byte aligned" in L.gs_last_error()


def test_the_chunk_table_covers_every_element_once(capi):
    from pf3plat_b200.optimizer import chunk_table
    C = capi.GS_ADAM_CHUNK
    numels = [1, 0, C - 1, C, C + 1, 3 * C + 5, 7]
    tensor, begin, count = chunk_table(numels)
    assert list(np.bincount(tensor, minlength=len(numels))) == [1, 1, 1, 1, 2, 4, 1]
    assert (np.diff(tensor) >= 0).all() and (count <= C).all() and (count >= 0).all()
    for t, n in enumerate(numels):
        sel = tensor == t
        assert count[sel].sum() == n
        assert list(begin[sel]) == list(range(0, max(n, 1), C))
    big = chunk_table([2**33 + 3])  # 64-bit element offsets
    assert big[1][-1] == (2**33 + 3) // C * C and big[2][-1] == (2**33 + 3) % C


# -- the Python optimizer's refusals -----------------------------------------------------------------------------------

def test_the_optimizer_refuses_what_pf3plat_does_not_use(capi):
    from pf3plat_b200.optimizer import Adam
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(TypeError, match=r"params\[0\].*CUDA"):
        Adam(p)
    for kw, word in ((dict(weight_decay=0.01), "weight_decay"), (dict(amsgrad=True), "amsgrad"),
                     (dict(maximize=True), "maximize"), (dict(betas=(1.0, 0.999)), "betas"),
                     (dict(eps=-1.0), "eps"), (dict(max_norm=float("nan")), "max_norm"),
                     (dict(max_norm=-0.5), "max_norm"), (dict(lr=float("inf")), "lr"),
                     (dict(lr=torch.tensor(1e-3)), "lr")):
        with pytest.raises((ValueError, TypeError), match=word):
            Adam(p, **kw)
    with pytest.raises(TypeError, match="lr"):
        Adam(p, lr=torch.tensor([1e-3]))
