"""GPU parity of the per-kernel C-ABI entry points against the CPU oracle's primitives (float64).

Tolerances: the fp32 SIMT path must agree to 2e-5 relative (it is the reference arithmetic, fp32);
the tensor-core bf16x3 path to 2e-4 relative per kernel (north_star: 1e-3 on activations end to end).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from parity_util import rel_l2, rel_max

pytestmark = pytest.mark.gpu

# every conv geometry on the hot path (module.py:161-211), at small batch:
#   (name, B, H, W, Cin, kh, kw, Cout, sh, sw)
CONV_CASES = [
    ("G.h1", 2, 1, 128, 24, 1, 15, 128, 1, 1),
    ("G.d1", 2, 1, 128, 128, 1, 5, 256, 1, 2),
    ("G.d2", 2, 1, 64, 256, 1, 5, 512, 1, 2),
    ("G.res_h1", 3, 1, 32, 512, 1, 3, 1024, 1, 1),
    ("G.res_h2", 3, 1, 32, 1024, 1, 3, 512, 1, 1),
    ("G.u1", 2, 1, 32, 512, 1, 5, 1024, 1, 1),
    ("G.u2", 2, 1, 64, 512, 1, 5, 512, 1, 1),
    ("G.o1", 2, 1, 128, 256, 1, 15, 24, 1, 1),
    ("G.odd_T", 1, 1, 33, 512, 1, 3, 64, 1, 1),       # ragged: width not a multiple of any tile
    ("G.d_oddT", 1, 1, 66, 128, 1, 5, 64, 1, 2),
    ("D.h1", 2, 24, 128, 1, 3, 3, 128, 1, 2),
    ("D.d1", 2, 24, 64, 128, 3, 3, 256, 2, 2),
    ("D.d2", 2, 12, 32, 256, 3, 3, 512, 2, 2),
    ("D.d3", 2, 6, 16, 512, 6, 3, 1024, 1, 2),
]


@pytest.fixture(scope="module")
def eng():
    import cgvc
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    code = lib.cgvc_create(C.byref(cfg), C.byref(h))
    assert code == 0, lib.cgvc_last_error(None)
    yield lib, h, N
    lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _rand(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64)


def _oracle_conv(x, w, b, sh, sw):
    from oracle import cyclegan_oracle as O
    return O.conv2d_same(x, w, b, (sh, sw))


def _run_conv_case(eng, case, prec, tol, tol_dw=None):
    lib, h, N = eng
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    x = _rand((B, H, W, Cin), 1); w = _rand((kh, kw, Cin, Cout), 2) / np.sqrt(kh * kw * Cin); b = _rand((Cout,), 3)
    x32, w32, b32 = (t.float() for t in (x, w, b))
    x, w, b = x32.double(), w32.double(), b32.double()
    xr = x.clone().requires_grad_(True); wr = w.clone().requires_grad_(True); br = b.clone().requires_grad_(True)
    y_ref = _oracle_conv(xr, wr, br, sh, sw)
    dy = _rand(tuple(y_ref.shape), 4).float()
    y_ref.backward(dy.double())
    xd, wd, bd, dyd = x32.cuda(), w32.cuda(), b32.cuda(), dy.cuda()
    y = torch.empty(tuple(y_ref.shape), dtype=torch.float32, device="cuda")
    code = lib.cgvc_conv_forward(h, prec, _p(xd), _p(wd), _p(bd), _p(y), B, H, W, Cin, kh, kw, Cout, sh, sw, None)
    if code == N.ERR_UNSUPPORTED:
        pytest.skip("%s: not a tensor-core shape" % name)
    N.check(h, code)
    dx = torch.full_like(xd, float("nan")); dw = torch.zeros_like(wd); db = torch.zeros_like(bd)
    N.check(h, lib.cgvc_conv_backward(h, prec, _p(xd), _p(wd), _p(dyd), _p(dx), _p(dw), _p(db), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
    torch.cuda.synchronize()
    errs = {"y": rel_l2(y.cpu(), y_ref.detach()), "dx": rel_l2(dx.cpu(), xr.grad), "dw": rel_l2(dw.cpu(), wr.grad),
            "db": rel_l2(db.cpu(), br.grad), "y_max": rel_max(y.cpu(), y_ref.detach())}
    print("conv %-10s prec=%d " % (name, prec) + " ".join("%s=%.2e" % kv for kv in errs.items()))
    for k, v in errs.items():
        assert v < (tol_dw if (k == "dw" and tol_dw) else tol), (name, k, v)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_fp32(eng, case):
    _run_conv_case(eng, case, 0, 2e-5)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_bf16x3(eng, case):
    _run_conv_case(eng, case, 1, 2e-4)


@pytest.mark.parametrize("case", [c for c in CONV_CASES if c[4] % 4 == 0], ids=[c[0] for c in CONV_CASES if c[4] % 4 == 0])
def test_conv_f16f8(eng, case):
    """CGVC_PREC_F16F8, the 2-MMA-unit precision: fp16 hi*hi MMA + two e4m3 cross-term MMAs rescaled by scale-input-d -- forward, data
    gradient (gradient planes with the activation-role scales against the weight planes) and weight gradient (activation x gradient
    planes, MN-major e4m3 tiles, rescale 2^-12), all three against float64.  The arithmetic itself is 1.04e-5 from float64 (a CPU
    emulation of the planes, K = 1536 .. 9216); 5e-5 rejects an fp16-only kernel (2.9e-4), a lost cross product (2.1e-4) and a rescale
    off by 2 (2.9e-4)."""
    lib, h, N = eng
    assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0
    _run_conv_case(eng, case, 3, 5e-5)


@pytest.mark.parametrize("case", [c for c in CONV_CASES if c[4] % 4 == 0], ids=[c[0] for c in CONV_CASES if c[4] % 4 == 0])
def test_conv_f16f8_weight_gradient_from_fp16_planes(eng, case):
    """Option `wgrad_f16` (the default of an F16F8 engine): the weight gradient (a leaf of the graph: its rounding error is not propagated into other layers) from the
    fp16 planes alone, one MMA unit per product.  Per-product error 2^-11 / sqrt(3) per operand -> <= 4e-4 relative L2 on random
    data (measured 2.4e-4..3.5e-4); forward and data gradient are unchanged."""
    lib, h, N = eng
    assert lib.cgvc_set_option(h, b"wgrad_f16", 1) == 0
    try:
        _run_conv_case(eng, case, 3, 5e-5, tol_dw=6e-4)
    finally:
        assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0


def test_conv_backward_accumulates(eng):
    """dw / dbias are accumulated into (GRAD-arena semantics); dx is overwritten."""
    lib, h, N = eng
    B, H, W, Cin, kh, kw, Cout = 1, 1, 32, 64, 1, 3, 64
    x = torch.randn(B, H, W, Cin, device="cuda"); w = torch.randn(kh, kw, Cin, Cout, device="cuda"); dy = torch.randn(B, H, W, Cout, device="cuda")
    dw1 = torch.zeros_like(w); db1 = torch.zeros(Cout, device="cuda"); dx = torch.empty_like(x)
    N.check(h, lib.cgvc_conv_backward(h, 0, _p(x), _p(w), _p(dy), _p(dx), _p(dw1), _p(db1), B, H, W, Cin, kh, kw, Cout, 1, 1, None))
    dw2 = dw1.clone(); db2 = db1.clone()
    N.check(h, lib.cgvc_conv_backward(h, 0, _p(x), _p(w), _p(dy), _p(dx), _p(dw2), _p(db2), B, H, W, Cin, kh, kw, Cout, 1, 1, None))
    torch.cuda.synchronize()
    assert rel_l2(dw2.cpu(), 2 * dw1.cpu()) < 1e-6 and rel_l2(db2.cpu(), 2 * db1.cpu()) < 1e-6


# (B, R (positions after shuffle), C (channels after shuffle), shuffle)
POST_CASES = [(3, 32, 1024, 1), (2, 64, 512, 2), (2, 128, 256, 2), (2, 384, 256, 1), (2, 48, 1024, 1), (1, 33, 64, 1), (5, 64, 256, 1), (700, 32, 128, 1), (3, 96, 512, 1)]


@pytest.mark.parametrize("case", POST_CASES, ids=["B%d_R%d_C%d_s%d" % c for c in POST_CASES])
def test_in_glu_fwd_bwd(eng, case):
    from oracle import cyclegan_oracle as O
    lib, h, N = eng
    B, R, C_, sh = case
    Cc = C_ * sh
    p = (_rand((B, R // sh, 2 * Cc), 10) * 1.7 + 0.3).float()
    ba, ga, bg, gg = (_rand((C_,), 11 + i).float() * 0.3 + (1.0 if i % 2 else 0.0) for i in range(4))
    dy = _rand((B, R, C_), 20).float()
    pr = p.double().requires_grad_(True)
    par = [t.double().requires_grad_(True) for t in (ba, ga, bg, gg)]
    a = pr[..., :Cc].reshape(B, R, C_); g = pr[..., Cc:].reshape(B, R, C_)      # raw reshape == pixel_shuffler (module.py:135-146)
    y_ref = O.glu(O.instance_norm(a, par[0], par[1]), O.instance_norm(g, par[2], par[3]))
    y_ref.backward(dy.double())
    pd, dyd = p.cuda(), dy.cuda()
    dev = [t.cuda() for t in (ba, ga, bg, gg)]
    y = torch.empty(B, R, C_, device="cuda"); stats = torch.empty(B, 4, C_, device="cuda")
    N.check(h, lib.cgvc_in_glu_forward(h, _p(pd), _p(dev[0]), _p(dev[1]), _p(dev[2]), _p(dev[3]), _p(y), _p(stats), B, R, C_, sh, None))
    dp = torch.empty_like(pd); grads = [torch.zeros(C_, device="cuda") for _ in range(4)]
    N.check(h, lib.cgvc_in_glu_backward(h, _p(dyd), _p(pd), _p(stats), _p(dev[0]), _p(dev[1]), _p(dev[2]), _p(dev[3]), _p(dp),
                                        _p(grads[0]), _p(grads[1]), _p(grads[2]), _p(grads[3]), B, R, C_, sh, None))
    torch.cuda.synchronize()
    errs = {"y": rel_l2(y.cpu(), y_ref.detach()), "dp": rel_l2(dp.cpu(), pr.grad)}
    for i, n in enumerate(("dbeta_a", "dgamma_a", "dbeta_g", "dgamma_g")):
        errs[n] = rel_l2(grads[i].cpu(), par[i].grad)
    print("in_glu", case, " ".join("%s=%.2e" % kv for kv in errs.items()))
    for k, v in errs.items():
        assert v < 2e-5, (case, k, v)
