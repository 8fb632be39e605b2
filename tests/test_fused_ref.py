"""CPU checks of tests/fused_ref.py: its layouts and references against the oracle's own composition, and the lattice certificate of
every case tests/test_gpu_fused_epilogue.py runs."""
import numpy as np
import pytest
import torch

import fused_ref as F
from oracle import cyclegan_oracle as O


def test_shuffle_rows_is_the_pixel_shuffle():
    """conv row r, column s * C + c of a shuffled layer is output row 2r + s, channel c: the oracle's raw reshape"""
    p = torch.arange(2 * 3 * 8, dtype=torch.float64).reshape(2, 3, 8)
    assert torch.equal(F.shuffle_rows(p), O.pixel_shuffle_reshape(p))
    q = F.shuffle_rows(p)
    for r in range(3):
        for s in range(2):
            for c in range(4):
                assert q[1, 2 * r + s, c] == p[1, r, s * 4 + c]


@pytest.mark.parametrize("layer", list(F.LAYERS))
def test_forward_matches_the_oracle_composition(layer):
    """conv -> IN -> GLU (-> pixel shuffle) of the oracle, layer by layer, against conv_p + forward: P's column layout, the shuffled
    view and the statistics"""
    Cin, kw, Cout, sw, gated, sh, _ = F.LAYERS[layer]
    B, R = 2, 8
    x, wa, wg, ba, bg, par, resid = F.dense_forward_case(layer, B, R, seed=1)
    P = F.conv_p(x, wa, wg, ba, bg, sw)
    assert P.shape == (B, R, Cout * (2 if gated else 1))
    y, st = F.forward(P, par, gated, sh, resid=resid)
    xt = torch.from_numpy(x).double()
    t = lambda a: torch.from_numpy(a).double()
    a = O.conv1d_same(xt, t(wa), t(ba), sw)
    if gated:
        g = O.conv1d_same(xt, t(wg), t(bg), sw)
        if sh == 2:
            a, g = O.pixel_shuffle_reshape(a), O.pixel_shuffle_reshape(g)
        ref = O.glu(O.instance_norm(a, t(par[0]), t(par[1])), O.instance_norm(g, t(par[2]), t(par[3])))
    else:
        ref = O.instance_norm(a, t(par[0]), t(par[1])) + t(resid)
    assert y.shape == (B, R * sh, Cout // sh)
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(F.forward_oracle(P, par, gated, sh, resid=resid), ref, rtol=1e-12, atol=1e-12)
    # the statistics: over the shuffled view; given back, they reproduce y
    assert torch.allclose(st[:, 0], a.mean(dim=1))
    y2, _ = F.forward(P, par, gated, sh, resid=resid, stats=st)
    torch.testing.assert_close(y2, y, rtol=0, atol=0)


@pytest.mark.parametrize("gated", [True, False])
def test_backward_matches_autograd(gated):
    """the closed-form IN (+ GLU) backward, with exact statistics and with the same statistics passed in, against autograd"""
    rng = np.random.default_rng(3)
    B, R, C = 3, 16, 8
    bp = (rng.standard_normal((B, R, C * (2 if gated else 1))) * 1.5 + 0.2).astype(np.float32)
    par = tuple((rng.standard_normal(C) * 0.3 + k).astype(np.float32) for k in (0.0, 1.0, 0.0, 1.0))
    if not gated:
        par = par[:2] + (None, None)
    dy = rng.standard_normal((B, R, C)).astype(np.float32)
    dp, grads = F.backward(bp, par, dy, gated)
    dp_ag, grads_ag = F.backward_autograd(bp, par, dy, gated)
    torch.testing.assert_close(dp, dp_ag, rtol=1e-10, atol=1e-12)
    for g, r in zip(grads, grads_ag):
        if r is not None:
            torch.testing.assert_close(g, r, rtol=1e-10, atol=1e-12)
    _, st = F.forward(bp, par, gated, 1, resid=None if gated else np.zeros((B, R, C), np.float32))
    dp2, _ = F.backward(bp, par, dy, gated, stats=st)
    torch.testing.assert_close(dp2, dp, rtol=1e-12, atol=1e-13)
    # statistics off by 1e-3 move the result: they are used, not recomputed
    dp3, _ = F.backward(bp, par, dy, gated, stats=st * (1 + 1e-3))
    assert (dp3 - dp).abs().max() > 1e-6


def test_lattice_values():
    rng = np.random.default_rng(0)
    x = F.lattice_x(rng, 5, 64, 32)
    assert set(np.unique(x)) <= {-2, -1, 0, 1, 2}
    assert not x[0].any() and np.count_nonzero(x[1]) == 1
    w = F.lattice_weights(rng, 3, 4, 5)
    assert set(np.unique(w)) <= {-2, -1, 1, 2}
    beta, gamma = F.lattice_affine(rng, 64)
    assert np.all(beta == np.round(beta)) and np.all(np.log2(np.abs(gamma)) == np.round(np.log2(np.abs(gamma))))


def test_lattice_conv_is_integer_and_dgrad_wired():
    """the float64 conv of a lattice case is integer-valued; dgrad is the adjoint of the convolution"""
    x, wa, wg, ba, bg, _, _ = F.lattice_forward_case("res_h1", 2, 32, seed=5)
    P = F.conv_p(x, wa, wg, ba, bg, 1)
    assert torch.equal(P, P.round())
    dP, wa2, wg2, _ = F.dense_dgrad_case("res_h1", 2, 16, seed=6, accumulate=0)
    xx = np.random.default_rng(7).standard_normal((2, 16, 512))
    lhs = (F.conv_p(xx, wa2, wg2, np.zeros(1024), np.zeros(1024), 1) * torch.from_numpy(dP).double()).sum()
    rhs = (F.dgrad(dP, wa2, wg2) * torch.from_numpy(xx)).sum()
    assert abs(float(lhs - rhs)) < 1e-9 * abs(float(lhs))


def test_certificate_of_every_lattice_case():
    """every forward lattice case of the GPU test stays below 2^24: P and its per-sample column sums are exact in fp32"""
    import test_gpu_fused_epilogue as T
    for layer, B, R, seed in T.lattice_cases():
        x, wa, wg, ba, bg, _, resid = F.lattice_forward_case(layer, B, R, seed)
        largest, colsum = F.certificate(x, wa, wg, ba, bg, F.LAYERS[layer][3])
        assert largest < 2 ** 24 and colsum < 2 ** 24, (layer, B, R, largest, colsum)
    for pair, B, R, seed, acc in T.lattice_bwd_cases():
        down = F.BWD_PAIRS[pair][0]
        dP, wa, wg, dx0 = F.lattice_dgrad_case(down, B, R, seed, acc)
        bound = F.dgrad(np.abs(dP), np.abs(wa), None if wg is None else np.abs(wg))
        if dx0 is not None:
            bound = bound + torch.from_numpy(np.abs(dx0)).double()
        assert float(bound.max()) < 2 ** 24, (pair, B, R)
