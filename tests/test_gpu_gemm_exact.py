"""The tensor-core convolutions against the float64 emulation of their operand planes (tests/gemm_ref.py).

A. Lattice tier: operands on a dyadic lattice whose certificate proves every partial sum exact in the kernels' accumulators, whatever
   the order.  y, dx, dw and db must equal the emulation bit for bit in every precision (fp32 SIMT, bf16x3, bf16, F16F8 with
   `wgrad_f16` 0 and 1), split-K partials included.  A lost (tap, stage) block, a wrong rescale or a misplaced plane changes bits.
B. Dense tier: unit randn operands, relative L2 to the emulation <= 2e-5 (10x below the coarse F16F8 mutants of gemm_ref; 5e-5 for
   bf16x3); the forward and data gradient are bitwise deterministic over two calls.
C. Launches and coverage: each call makes exactly the tensor-core launches the launch mirror expects, and the case list reaches every
   NT / TN instantiation, multi-tile persistent walks, uneven and empty split-K items, tails and padding.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_ref as G
from parity_util import rel_l2
from test_gpu_kernels import CONV_CASES

pytestmark = pytest.mark.gpu

CASES = CONV_CASES + G.ODD_CASES + G.BIG_CASES
BIG = {c[0] for c in G.BIG_CASES}
# the dense tier's ceiling: 10x below the coarse F16F8 mutants of gemm_ref (2e-4 .. 3e-4).  bf16x3 updates its accumulator three
# times per product pair, and its gap grows accordingly: 2.84e-5 at D.d3 (K = 9216), 3.1x bf16's 9.2e-6 on the same case (H100 80GB
# HBM3, 700 W); its own coarse mutants lie at 1.7e-3 to 2.4e-3
DENSE_TOL = {G.BF16X3: 5e-5, G.BF16: 2e-5, G.F16F8: 2e-5}
PNAME = {G.FP32: "fp32", G.BF16X3: "bf16x3", G.BF16: "bf16", G.F16F8: "f16f8"}


@pytest.fixture(scope="module")
def eng():
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    yield lib, h, N
    lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(lib):
    cap = 64
    ms = (C.c_double * cap)(); fl = (C.c_double * cap)(); meta = (C.c_longlong * (4 * cap))(); n = C.c_int(0)
    assert lib.cgvc_profile_launches(ms, fl, meta, cap, C.byref(n)) == 0
    return [tuple(meta[4 * i: 4 * i + 4]) for i in range(min(n.value, cap))]


def _check_launches(got, case, prec, form):
    """exactly the tensor-core launches of the mirror: (class, M, N, K)"""
    if prec == G.FP32:
        assert got == [], (case[0], form, got)
        return
    L = G.case_launches(case, prec, 0, _nsm())
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    if form == "fwd":
        f = L["fwd"]
        want = [(0, f["M"], f["N"], f["K"])]
    else:
        want = [(0, d["M"], d["N"], d["K"]) for d in L["dgrad"]]
        assert sum(d["M"] for d in L["dgrad"]) == B * H * W
        want.append((1, B * -(-H // sh) * -(-W // sw), Cout, kh * kw * Cin))
    assert got == want, (case[0], prec, form, got, want)


def _call(eng, case, prec, x, w, b, dy, w16, launches=False):
    """cgvc_conv_forward + cgvc_conv_backward on device copies of the fp32 inputs: {'y', 'dx', 'dw', 'db'} (fp32 cuda)"""
    lib, h, N = eng
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    xd, wd, bd, dyd = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in (x, w, b, dy))
    assert lib.cgvc_set_option(h, b"wgrad_f16", int(w16)) == 0
    try:
        if launches:
            lib.cgvc_profile_enable(1)
        y = torch.full(dyd.shape, float("nan"), device="cuda")
        N.check(h, lib.cgvc_conv_forward(h, prec, _p(xd), _p(wd), _p(bd), _p(y), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
        if launches:
            _check_launches(_launches(lib), case, prec, "fwd")
            lib.cgvc_profile_enable(1)                        # (re-enabling clears the records)
        dx = torch.full_like(xd, float("nan")); dw = torch.zeros_like(wd); db = torch.zeros_like(bd)
        N.check(h, lib.cgvc_conv_backward(h, prec, _p(xd), _p(wd), _p(dyd), _p(dx), _p(dw), _p(db), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
        if launches:
            _check_launches(_launches(lib), case, prec, "bwd")
        torch.cuda.synchronize()
    finally:
        lib.cgvc_profile_enable(0)
        assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0
    return {"y": y, "dx": dx, "dw": dw, "db": db}


def _where(case, key, flat):
    """a readable position of output element `flat`: (m, n), its 128-row tile, and the tap of a weight-gradient element"""
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    if key == "dw":
        t, rem = divmod(flat, Cin * Cout)
        c, n = divmod(rem, Cout)
        return "tap %d (ky %d, kx %d), c %d, n %d" % (t, t // kw, t % kw, c, n)
    if key == "db":
        return "n %d" % flat
    ncol = Cout if key == "y" else Cin
    m, n = divmod(flat, ncol)
    if key == "y":
        return "m %d, n %d, tile %d" % (m, n, m // 128)
    # dx rows are walked per output parity class: the row within its class
    Wd = W
    b_, rem = divmod(m, H * Wd); yy, xx = divmod(rem, Wd)
    cls = (yy % sh, xx % sw)
    hy, wx = -(-(H - cls[0]) // sh), -(-(W - cls[1]) // sw)
    mc = (b_ * hy + yy // sh) * wx + xx // sw
    return "input (b %d, y %d, x %d), n %d; parity class %s row %d, tile %d" % (b_, yy, xx, n, cls, mc, mc // 128)


def _assert_exact(case, prec, key, got, ref):
    g = got.double().reshape(-1); r = ref.reshape(-1)
    bad = torch.nonzero(g != r).reshape(-1)
    if bad.numel():
        lines = ["  %s: got %r, emulation %r" % (_where(case, key, int(i)), float(g[i]), float(r[i])) for i in bad[:8].tolist()]
        raise AssertionError("%s prec %d %s: %d of %d values differ from the exact emulation; first:\n%s"
                             % (case[0], prec, key, bad.numel(), g.numel(), "\n".join(lines)))


LATTICE_PARAMS = [(c, p) for c in CASES for p in (G.FP32, G.BF16X3, G.BF16, G.F16F8)
                  if G.supports(c, p) and not (p == G.FP32 and c[0] in BIG)]


@pytest.mark.parametrize("case,prec", LATTICE_PARAMS, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in LATTICE_PARAMS])
def test_lattice_bit_exact(eng, case, prec):
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    for w16 in ((0, 1) if prec == G.F16F8 else (0,)):
        cert = G.certificate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P)
        for form, phase, largest, bound in cert:
            assert largest < bound, (case[0], prec, w16, form, phase, largest, bound)
        ref = G.emulate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P)
        got = _call(eng, case, prec, x, w, b, dy, w16, launches=w16 == 0)
        print("lattice %-10s prec=%d w16=%d certificate used %s" % (case[0], prec, w16, " ".join(
            "%s/%s %.2f" % (f, ph, l / bd) for f, ph, l, bd in cert)))
        for key in ("y", "dx", "dw", "db"):
            _assert_exact(case, prec, key, got[key], ref[key])


DENSE_PARAMS = [(c, p) for c in CASES for p in (G.BF16X3, G.BF16, G.F16F8) if G.supports(c, p)]


@pytest.mark.parametrize("case,prec", DENSE_PARAMS, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in DENSE_PARAMS])
def test_dense_close_and_deterministic(eng, case, prec):
    x, w, b, dy = G.dense_case(case)
    P = G.case_planes(prec, x, w, dy)
    first = None
    for w16 in ((0, 1) if prec == G.F16F8 else (0,)):
        ref = G.emulate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P)
        got = _call(eng, case, prec, x, w, b, dy, w16)
        errs = {k: rel_l2(got[k].cpu(), ref[k].cpu()) for k in ("y", "dx", "dw")}
        print("dense %-10s prec=%d w16=%d gap to the emulation: %s" % (case[0], prec, w16, " ".join("%s=%.2e" % kv for kv in errs.items())))
        for k, v in errs.items():
            assert v <= DENSE_TOL[prec], (case[0], prec, w16, k, v)
        if first is None:
            first = got
        else:                                                  # the second call: forward and data gradient bitwise equal
            for k in ("y", "dx"):
                assert torch.equal(first[k], got[k]), (case[0], prec, k, "not deterministic")
    if prec != G.F16F8:
        again = _call(eng, case, prec, x, w, b, dy, 0)
        for k in ("y", "dx"):
            assert torch.equal(first[k], again[k]), (case[0], prec, k, "not deterministic")


def test_case_list_coverage():
    nsm = _nsm()
    cov = G.coverage(CASES, nsm)
    print("coverage of the case list at %d SMs:" % nsm)
    for k, v in cov.items():
        print("  %-72s %s" % (k, ", ".join(v[:3]) + (" ..." if len(v) > 3 else "") if v else "MISSING"))
    assert all(cov.values()), [k for k, v in cov.items() if not v]
