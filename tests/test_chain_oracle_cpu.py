"""The adapter -> decoder chain oracle (tests/chain_oracle.py), without a GPU: with the adapter bypassed it is the batched
oracle plus its backward bit for bit; through the adapter its gradients agree with fp64 central finite differences of
the chain itself, on both depth routes."""
import numpy as np
import pytest
import torch

from pf3plat_b200.cameras import make_view_batch
from pf3plat_b200.rasterizer import BatchSettings
from pf3plat_b200.synthetic import make_scene
from tests.batch_oracle import oracle_batch
from tests.chain_oracle import ChainOracle, DecoderOracle, make_chain_inputs


def test_decoder_oracle_is_the_batched_oracle_with_the_decoder_layout():
    """S = 2 scenes x 2 target views, near 0.5 / 2.0, non-zero background: images, depth * near and every gradient at the
    decoder's inputs equal oracle_batch + OracleBatch.backward on the rasterizer's layout (6-vector covariance, (d_sh, 3)
    harmonics), with the covariance gradient landing on the upper triangle of the (3, 3) matrix only."""
    b, v, hw = 2, 2, (24, 32)
    scenes = [make_scene(300, v, *hw, seed=200 + k) for k in range(b)]
    st = lambda name: torch.stack([getattr(sc, name) for sc in scenes]).double()
    means, cov, harm, opac = (st(n).requires_grad_(True) for n in ("means", "covariances", "harmonics", "opacities"))
    ext, intr = st("extrinsics"), st("intrinsics")
    near = torch.tensor([[0.5, 2.0], [2.0, 0.5]], dtype=torch.float64)
    far = 100.0 * near
    bg = torch.tensor([0.2, 0.5, 0.1], dtype=torch.float64)
    dec = DecoderOracle(means, cov, harm, opac, ext, intr, near, far, hw, bg)

    vb = make_view_batch(ext.reshape(4, 4, 4), intr.reshape(4, 3, 3), near.reshape(4), far.reshape(4))
    bs = BatchSettings(image_height=hw[0], image_width=hw[1], viewmatrix=vb.viewmatrix, projmatrix=vb.projmatrix,
                       campos=vb.campos, bg=bg.expand(4, 3), sh_degree=4, tanfov=vb.tanfov, view_scale=vb.scale,
                       with_depth=True)
    c = cov.detach()
    cov6 = torch.stack([c[..., 0, 0], c[..., 0, 1], c[..., 0, 2], c[..., 1, 1], c[..., 1, 2], c[..., 2, 2]], -1)
    ob = oracle_batch(bs, means.detach(), opac.detach(), shs=harm.detach().permute(0, 1, 3, 2).contiguous(),
                      cov3D_precomp=cov6, dtype=np.float64)
    assert (ob.radii > 0).mean() > 0.5 and sorted(set(ob.s.tolist())) == [0.5, 2.0]
    assert np.array_equal(dec.color, ob.color)
    nr = near.reshape(4, 1, 1).numpy()
    assert np.array_equal(dec.depth, ob.depth * nr)

    rng = np.random.default_rng(3)
    dLc = rng.standard_normal((4, 3, *hw))
    dLd = rng.standard_normal((4, *hw))
    dec.backward(dLc, dLd)
    g = ob.backward(dLc, dLd * nr)
    assert np.array_equal(means.grad.numpy(), g["means3D"])
    assert np.array_equal(opac.grad.numpy(), g["opacities"])
    assert np.array_equal(harm.grad.transpose(-1, -2).numpy(), g["shs"])
    G = cov.grad.reshape(b, -1, 9).numpy()
    assert np.array_equal(G[..., [0, 1, 2, 4, 5, 8]], g["cov3D_precomp"])
    assert not G[..., [3, 6, 7]].any()


def _tiny(two_pass):
    inp = make_chain_inputs(11, 1, 1, (4, 4), 2, 4, 0.5)
    bg = torch.tensor([0.3, 0.1, 0.2])
    return inp, bg


def _chain(inp, bg, two_pass, frag_rel=0.0, **over):
    a = {**inp, **over}
    return ChainOracle(a["extrinsics"], a["intrinsics"], a["coordinates"], a["depths"], a["opacities"],
                       a["raw_gaussians"], (4, 4), 4, a["target_extrinsics"], a["target_intrinsics"], a["near"], a["far"],
                       (16, 16), bg, two_pass=two_pass, frag_rel=frag_rel)


def _fd(loss, base, idx, eps):
    p, m = base.clone(), base.clone()
    p[idx] += eps
    m[idx] -= eps
    return (loss(p) - loss(m)) / (2 * eps)


@pytest.mark.parametrize("two_pass", [False, True])
def test_chain_gradients_match_finite_differences(two_pass):
    """1 scene, 1 context view of 4 x 4, 2 target views of 16 x 16, near 0.5, loss <wc, colour> + <wd, depth>.  Central
    differences (eps 1e-6, agreeing with eps 4e-6, i.e. the loss is smooth there) at entries of the raw Gaussians (scale,
    quaternion, SH of degrees 0, 1, 3), depths, coordinates, the context camera's translation -- its rotation also enters
    the covariance and the SH rotation, where the reference detaches it -- and, on the two-pass route, every entry of the
    target extrinsics' top three rows (the fake colour's z; the rasterized camera is detached)."""
    inp, bg = _tiny(two_pass)
    ch = _chain(inp, bg, two_pass, frag_rel=1e-4)      # the fragility bands of the GPU tests
    rng = np.random.default_rng(5)
    wc = rng.standard_normal(ch.color.shape)
    wd = rng.standard_normal(ch.depth.shape)
    ch.backward(wc, wd)
    g = ch.grads()
    aff = ch.affected()[0, 0]
    vis = (ch.decoder.ob.radii > 0).any(axis=0)
    print(f"[regime] tiny chain ({'two-pass' if two_pass else 'fused'}): visible Gaussians {int(vis.sum())} of 16, "
          f"affected {int(aff.sum())}")
    assert vis.sum() >= 8
    assert not aff.any()          # no fragile decision anywhere: every entry below is away from one

    def loss_of(name):
        def f(x):
            c = _chain(inp, bg, two_pass, **{name: x})
            return float((c.color * wc).sum() + (c.depth * wd).sum())
        return f

    def check(name, base, gref, idx):
        base = base.double()
        f = loss_of(name)
        fd1, fd4 = _fd(f, base, idx, 1e-6), _fd(f, base, idx, 4e-6)
        scale = float(gref.abs().max())
        gi = float(gref[idx])
        print(f"[fd] {name}{list(idx)}: autograd {gi:.6e} fd {fd1:.6e}")
        assert abs(fd1 - fd4) <= 1e-6 * scale, (name, idx, fd1, fd4)
        assert abs(fd1 - gi) <= 1e-5 * scale, (name, idx, fd1, gi)

    gaussians = [int(i) for i in np.nonzero(vis)[0][:3]]
    for i in gaussians:
        for k in (0, 2, 3, 6, 7, 8, 7 + 25 + 10, 7 + 50 + 15):
            check("raw_gaussians", inp["raw_gaussians"], g["raw_gaussians"], (0, 0, i, k))
        check("depths", inp["depths"], g["depths"], (0, 0, i))
        check("coordinates", inp["coordinates"], g["coordinates"], (0, 0, i, 0))
        check("coordinates", inp["coordinates"], g["coordinates"], (0, 0, i, 1))
    for r in range(3):
        check("extrinsics", inp["extrinsics"], g["extrinsics"], (0, 0, r, 3))
    if two_pass:
        ad = ch.adapter_out
        dec_in = [ad["means"].detach().reshape(1, 16, 3), ad["covariances"].detach().reshape(1, 16, 3, 3),
                  ad["harmonics"].detach().reshape(1, 16, 3, 25), ad["opacities"].detach().reshape(1, 16)]
        tgt = inp["target_extrinsics"].double()

        def f(x):
            d = DecoderOracle(*dec_in, tgt, inp["target_intrinsics"].double(), inp["near"].double(),
                              inp["far"].double(), (16, 16), bg.double(), two_pass=True, z_extrinsics=x, frag_rel=0)
            return float((d.color * wc).sum() + (d.depth * wd).sum())

        gt = g["target_extrinsics"]
        assert float(gt.abs().max()) > 0
        for v in range(2):
            for r in range(3):
                for c in range(4):
                    idx = (0, v, r, c)
                    fd1, fd4 = _fd(f, tgt, idx, 1e-6), _fd(f, tgt, idx, 4e-6)
                    scale = float(gt.abs().max())
                    print(f"[fd] target_extrinsics{list(idx)}: autograd {float(gt[idx]):.6e} fd {fd1:.6e}")
                    assert abs(fd1 - fd4) <= 1e-6 * scale
                    assert abs(fd1 - float(gt[idx])) <= 1e-5 * scale, (idx, fd1, float(gt[idx]))
