"""The float64 emulation of tests/gemm_ref.py on the CPU: its wiring, how far its mutants lie, the lattice certificate, and the
launch mirror's coverage of the GPU case list.  No GPU needed."""
import numpy as np
import pytest
import torch

import gemm_ref as G
from oracle.cyclegan_oracle import conv2d_same
from parity_util import rel_l2
from test_gpu_kernels import CONV_CASES

SMALL = CONV_CASES + G.ODD_CASES
PRECS = (G.FP32, G.BF16X3, G.BF16, G.F16F8)
DENSE_TOL = 2e-5                     # tests/test_gpu_gemm_exact.py: F16F8 kernels vs emulation, randn operands
ids = [c[0] for c in SMALL]


def _exact_conv(case, x, w, b, dy):
    """float64 forward, dx, dw of the fp32 values through the oracle's conv2d_same and its autograd"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    xr = torch.as_tensor(x, dtype=torch.float64).requires_grad_(True)
    wr = torch.as_tensor(w, dtype=torch.float64).requires_grad_(True)
    y = conv2d_same(xr, wr, torch.as_tensor(b, dtype=torch.float64), (sh, sw))
    y.backward(torch.as_tensor(dy, dtype=torch.float64))
    return y.detach(), xr.grad, wr.grad


@pytest.mark.parametrize("case", SMALL, ids=ids)
def test_formula_wiring(case):
    """operands whose lo planes are all zero: every precision's emulation is the float64 convolution exactly -- the roles, the
    data-gradient flips, the strides and the 2-D taps of the plane products are wired as conv2d_same's (each case's geometry, with
    at most 40 / 36 channels)"""
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    Cin, Cout = min(Cin, 40), min(Cout, 36)
    case = (name, B, H, W, Cin, kh, kw, Cout, sh, sw)
    rng = np.random.default_rng(7)
    Ho, Wo = -(-H // sh), -(-W // sw)
    x, w, b, dy = (G._lat_values(s, "int", "act", rng, 0.9) for s in ((B, H, W, Cin), (kh, kw, Cin, Cout), (Cout,), (B, Ho, Wo, Cout)))
    y0, dx0, dw0 = _exact_conv(case, x, w, b, dy)
    for prec in PRECS:
        if not G.supports(case, prec):
            continue
        P = G.case_planes(prec, x, w, dy)
        for role in ("x", "w", "dy"):
            for k, v in P[role].items():
                if k in ("lo", "8lo"):
                    assert not v.any(), (case[0], prec, role, k)
        e = G.emulate(case, prec, x, w, b, dy, w16=1, P=P)
        assert torch.equal(e["y"], y0) and torch.equal(e["dx"], dx0) and torch.equal(e["dw"], dw0), (case[0], prec)
        assert torch.equal(e["db"], torch.as_tensor(dy, dtype=torch.float64).reshape(-1, Cout).sum(0))
        if prec == G.F16F8:                  # the 2-unit weight gradient: its cross products of all-zero lo planes add nothing
            e = G.emulate(case, prec, x, w, b, dy, w16=0, P=P, forms=("wgrad",))
            assert torch.equal(e["dw"], dw0), case[0]


@pytest.mark.parametrize("case", SMALL, ids=ids)
def test_coarse_mutants_far_from_emulation(case):
    """on the dense tier's inputs, every coarse F16F8 mutant (cross terms lost, one cross product lost, rescale off by 2) lies at
    least 5x the dense tolerance from the emulation, so the dense tier rejects it"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    x, w, b, dy = G.dense_case(case)
    for prec in (G.F16F8,):
        names = G.COARSE_MUTANTS[prec]
        if not G.supports(case, prec):
            continue
        P = G.case_planes(prec, x, w, dy)
        spec = {"fwd": (P["x"], P["w"], None), "dgrad": (P["dy"], P["w"], (B, H, W, Cin)), "wgrad": (P["x"], P["dy"], (kh, kw, Cin, Cout))}
        for form, (Pa, Pb, shape) in spec.items():
            prods = {(ka, kb): G.combine(form, Pa, Pb, [(1.0, ka, kb)], (sh, sw), shape) for _, ka, kb in G.pairs(prec, form, 0)}
            ref = sum(c * prods[(ka, kb)] for c, ka, kb in G.pairs(prec, form, 0))
            for name in names:
                mut = sum(c * prods[(ka, kb)] for c, ka, kb in G.mutant_pairs(prec, form, name, 0))
                d = rel_l2(mut, ref)
                assert d >= 5 * DENSE_TOL, (case[0], prec, form, name, d)


@pytest.mark.parametrize("case", SMALL, ids=ids)
def test_lattice_certificate_and_blocks(case):
    """every lattice case satisfies its certificate in every precision, and losing any single (tap, stage) block of the forward or
    data-gradient cross terms changes the exact result"""
    for prec in PRECS:
        if not G.supports(case, prec):
            continue
        x, w, b, dy = G.lattice_case(case, prec)
        P = G.case_planes(prec, x, w, dy)
        cert = G.certificate(case, prec, x, w, b, dy, w16=0, P=P)
        if prec == G.F16F8:                  # (wgrad_f16 changes the weight gradient alone)
            cert += G.certificate(case, prec, x, w, b, dy, w16=1, P=P, forms=("wgrad",))
        for form, phase, largest, bound in cert:
            assert largest < bound, (case[0], prec, form, phase, largest, bound)
        for form in ("fwd", "dgrad"):
            nz = G.block_nonzero(case, prec, form, P)
            assert all(nz.values()), (case[0], prec, form, [k for k, v in nz.items() if not v])


@pytest.mark.parametrize("case", G.BIG_CASES, ids=[c[0] for c in G.BIG_CASES])
def test_lattice_blocks_big(case):
    """in the big cases' F16F8 lattices, 8 random (tap, stage) blocks per data form are each visible in the exact result (their
    certificates are checked on the GPU, in float64 there, before each comparison of tests/test_gpu_gemm_exact.py)"""
    x, w, b, dy = G.lattice_case(case, G.F16F8)
    P = G.case_planes(G.F16F8, x, w, dy)
    rng = np.random.default_rng(3)
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    for form, K in (("fwd", Cin), ("dgrad", Cout)):
        blocks = [(int(rng.integers(kh * kw)), int(rng.integers(-(-K // 64)))) for _ in range(8)]
        nz = G.block_nonzero(case, G.F16F8, form, P, blocks)
        assert all(nz.values()), (case[0], form, [k for k, v in nz.items() if not v])


@pytest.mark.parametrize("case", SMALL, ids=ids)
def test_lattice_sum_order_independent(case):
    """under the certificate the F16F8 forward (the lattice closest to its bound) summed term by term in float32 gives the float64
    result in forward and in reverse order"""
    for prec in (G.F16F8,):
        if not G.supports(case, prec):
            continue
        x, w, b, dy = G.lattice_case(case, prec)
        fwd, rev, exact = G.fp32_sum_orders(case, prec, x, w, b)
        assert torch.equal(fwd.double(), exact) and torch.equal(rev.double(), exact), (case[0], prec)


def test_launch_mirror_coverage_at_132_sms():
    """the GPU case list reaches every NT and TN instantiation and the tile-walk, split-K, tail and padding paths on an H100 SXM
    (132 SMs); tests/test_gpu_gemm_exact.py asserts the same with the device's SM count"""
    cov = G.coverage(CONV_CASES + G.ODD_CASES + G.BIG_CASES, 132)
    assert all(cov.values()), [k for k, v in cov.items() if not v]


def test_launch_mirror_split_k():
    """the split-K mirror on hand-checked shapes: big.split walks 30 items of 1152 rows, the 29th has 513 rows and the last none"""
    t = G.tn_launch(32769, 64, 64, 1, G.BF16X3, 0, 132)
    assert (t["ksplit"], t["chunk"], t["uneven"], t["empty"]) == (30, 1152, True, True)
    assert t["num_kb"][28] == 9 and t["num_kb"][29] == 0 and sum(t["num_kb"][:28]) == 28 * 18
    assert G.tn_launch(2 * 128, 128, 24, 15, G.BF16X3, 0, 132)["ksplit"] == 1          # fewer than 1024 rows never split
