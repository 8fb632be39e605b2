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


@pytest.mark.parametrize("gated,shuffle", [(True, 1), (True, 2), (False, 1), (False, 2)])
def test_shuffle_backward_and_conv_bias_match_autograd(gated, shuffle):
    """the closed form in the shuffled view and the conv-bias gradients (per conv column, so per phase) against autograd of the oracle"""
    rng = np.random.default_rng(5)
    B, Rw, C = 3, 8, 4
    nt = C * shuffle * (2 if gated else 1)
    bp = (rng.standard_normal((B, Rw, nt)) * 1.5 + 0.2).astype(np.float32)
    par = tuple((rng.standard_normal(C) * 0.3 + k).astype(np.float32) for k in (0.0, 1.0, 0.0, 1.0))
    if not gated:
        par = par[:2] + (None, None)
    dy = rng.standard_normal((B, Rw * shuffle, C)).astype(np.float32)
    dp, grads, bias = F.backward(bp, par, dy, gated, shuffle=shuffle, bias=True)
    dp_ag, grads_ag, bias_ag = F.backward_autograd(bp, par, dy, gated, shuffle=shuffle, bias=True)
    torch.testing.assert_close(dp, dp_ag, rtol=1e-10, atol=1e-10)
    for g, ga in zip(grads, grads_ag):
        if ga is not None:
            torch.testing.assert_close(g, ga, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(torch.cat([b for b in bias if b is not None]), bias_ag, rtol=1e-10, atol=1e-10)
    if shuffle == 2:                      # not analytically zero: the norm removes the mean over both phases, not per phase
        assert bias[0].abs().max() > 1e-3
    else:
        assert bias[0].abs().max() < 1e-9


def test_norm_bounds_hold_for_a_float32_replay():
    """the statistics and dP bounds of fused_ref hold for float32 evaluations of the kernels' formulas (a CPU replay, sequential sums)"""
    rng = np.random.default_rng(9)
    B, R, C = 4, 96, 8
    v = (rng.standard_normal((B, R, C)) * np.array([1e-4, 1.0, 30.0, 1e-2])[:, None, None] + rng.standard_normal((B, 1, C)) * 50)
    v[3, 0] += 2000 * 1e-2                                      # a far outlier at position 0
    v = v.astype(np.float32)
    v64 = torch.from_numpy(v).double()
    for form in ("stream", "shifted"):
        x = v
        if form == "stream":
            m = (x.sum(axis=1, dtype=np.float32) * np.float32(1 / R)).astype(np.float32)
            d = (x - m[:, None]).astype(np.float32)
            var = ((d * d).sum(axis=1, dtype=np.float32) * np.float32(1 / R)).astype(np.float32)
        else:
            k = x[:, 0]
            d = (x - k[:, None]).astype(np.float32)
            m1 = d.sum(axis=1, dtype=np.float32) * np.float32(1 / R)
            var = np.maximum((d * d).sum(axis=1, dtype=np.float32) * np.float32(1 / R) - m1 * m1, 0).astype(np.float32)
            m = (k + m1).astype(np.float32)
        rs = np.float32(1) / np.sqrt(var + np.float32(F.EPS))
        m64, r64 = F.stats_of(v64)
        em, er = F.stats_bound(v64, form, R + 13)
        assert (torch.from_numpy(m).double() - m64).abs().le(em).all(), form
        assert (torch.from_numpy(rs).double() / r64 - 1).abs().le(er).all(), form


def test_dispatch_mirror_matches_the_launch_code():
    """fused_ref's dispatch mirror against the configuration macros and rules parsed from simt_kernels.cu"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voice-converter-cyclegan_b200", "csrc",
                            "simt_kernels.cu")).read()
    fwd = [tuple(int(n) for n in t) for t in re.findall(r"X\((\d+), (\d+)\)", re.search(r"#define STREAM_FWD_CONFIGS\(X\)(.*)", src).group(1))]
    bwd = [(int(a), int(b), c == "true") for a, b, c in
           re.findall(r"X\((\d+), (\d+), (true|false)\)", re.search(r"#define STREAM_CONFIGS\(X\)(.*)", src).group(1))]
    assert sorted(fwd) == sorted(F.STREAM_FWD) and sorted(bwd) == sorted(F.STREAM_BWD)
    # each dispatch line: R == 256 / NQL * NRT, C % (4 NQL)
    for R, cm, nql, nrt in re.findall(r"if \(R == (\d+) && C % (\d+) == 0\) \{ \*err = launch_post_fwd_stream<(\d+), (\d+)>", src):
        assert int(R) == 256 // int(nql) * int(nrt) and int(cm) == 4 * int(nql)
        assert F.post_fwd_kernels(2, int(R), int(cm), 1, True) == ["post_fwd_stream_kernel<%s, %s>" % (nql, nrt)]
    for R, cm, nql, nrt, g in re.findall(r"if \(R == (\d+) && C % (\d+) == 0(?: && pp.sh == 1)?\) \{ \*err = launch_post_bwd_stream<(\d+), (\d+), (\w+)>", src):
        assert int(R) == 256 // int(nql) * int(nrt) and int(cm) == 4 * int(nql)
        assert F.post_bwd_kernels(2, int(R), int(cm), 1, g == "true") == ["post_bwd_stream_kernel<%s, %s, %s>" % (nql, nrt, g)]
    assert "if (pp.R <= 32) ONEPASS(4); else if (pp.R <= 48) ONEPASS(6); else ONEPASS(8);" in src
    assert "pp.has_in && pp.R <= 64 && forms.onepass" in src
    assert F.post_bwd_kernels(2, 40, 128, 1, True) == ["post_bwd_onepass_kernel<true, 6>"]
    assert F.post_bwd_kernels(2, 64, 128, 2, False) == ["post_bwd_onepass_kernel<false, 8>"]
    assert F.post_bwd_kernels(2, 384, 16, 1, True, det=True, bias=True) == ["post_bwd_sums_kernel<true>", "reduce_parts_kernel",
                                                                 "post_apply_bwd_kernel<true, true>", "reduce_parts_kernel"]
    assert F.post_fwd_kernels(2, 384, 16, 1, True, resid=True) == ["post_stats_kernel<true, false>", "post_apply_fwd_kernel<true, true, false>"]
    assert len(F.post_instantiations(src)) == 6 + 7 + 6 + 12
