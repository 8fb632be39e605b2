"""The operand planes of the tensor-core path against the numpy reference of tests/f16f8_ref.py, and the F16F8 window measured.

a. Every counted plane writer (the pad-split, the tap im2col, the instance-norm / GLU kernels forward and backward in every dispatch
   form): each plane value equals the reference, and the saturation counter equals the reference count of cgvc_sat4 groups exactly --
   the count dynamic loss scaling trusts when it accepts a step.  A second call doubles the count; a NULL counter gives the same planes.
   The two writers of the layers without an instance norm -- the GLU-only form's y and dP planes (generator h1) and the discriminator
   input layer's y planes (conv_c1_glu_fwd) -- are checked by the same protocol in test_gpu_glu_layers.py.
b. The F16F8 GEMMs against float64 with each operand scaled by powers of two: the window in which the planes are parity-grade.
c. The train step's gradients at every loss scale the dynamic scaler can reach, against the float64 oracle.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import f16f8_ref as R
from parity_util import rel_l2

pytestmark = pytest.mark.gpu

BF16, F16F8 = 1, 3
SENTINEL = 0x55                      # plane bytes before a call: 85.3 as fp16, 0.0195 as e4m3, 3.7e12 as bf16 -- never what a writer writes here


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


def _ru(x, m):
    return (x + m - 1) // m * m


def _planes(prec, n):
    """device plane buffers for n values, filled with SENTINEL bytes: (hi, lo)"""
    if prec == F16F8:
        hi = torch.empty(n, dtype=torch.float16, device="cuda"); lo = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    else:
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda"); lo = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    hi.view(torch.uint8).fill_(SENTINEL); lo.view(torch.uint8).fill_(SENTINEL)
    return hi, lo


def _bf16_values(t):
    return R.bf16_decode(t.view(torch.int16).cpu().numpy().view(np.uint16))


def check_planes(prec, hi, lo, x, what):
    """the planes (hi, lo) hold exactly the planes of fp32 x (flattened in plane order)"""
    x = np.ascontiguousarray(x, np.float32).reshape(-1)
    n = x.size
    if prec == F16F8:
        q16, q8hi, q8lo = R.quant_planes(x)
        l8 = lo.cpu().numpy()
        R.assert_same_values(hi.cpu().numpy(), q16, what + ": q16")
        R.assert_same_values(R.e4m3_decode(l8[:n]), R.e4m3_decode(q8hi), what + ": q8hi")
        R.assert_same_values(R.e4m3_decode(l8[n:]), R.e4m3_decode(q8lo), what + ": q8lo")
    else:
        bh, bl = R.split_bf16(x)
        R.assert_same_values(_bf16_values(hi), R.bf16_decode(bh), what + ": bf16 hi")
        R.assert_same_values(_bf16_values(lo), R.bf16_decode(bl), what + ": bf16 lo")


def _edge_filled(n, rng):
    """n fp32 values: the edge table (as much of it as fits, shuffled) among log-uniform magnitudes 2^-30 .. 2^18 of random sign"""
    x = R.log_uniform(n, rng)
    e = R.edge_values()
    e = e[rng.permutation(e.size)][:n]
    pos = rng.choice(n, e.size, replace=False)
    x[pos] = e
    return x


def _counted_calls(prec, call, n, ref_fn, what):
    """call(hi, lo, sat) three times: with a counter, again with the same counter (the count doubles), with NULL (same planes)"""
    sat = torch.zeros(1, dtype=torch.int64, device="cuda")
    expect = None
    for k, ctr in enumerate((sat, sat, None)):
        hi, lo = _planes(prec, n)
        call(hi, lo, ctr)
        torch.cuda.synchronize()
        x, expect = ref_fn()
        check_planes(prec, hi, lo, x, "%s (call %d)" % (what, k))
        if ctr is not None:
            want = (k + 1) * expect if prec == F16F8 else 0               # bf16 planes are not counted
            assert int(sat.item()) == want, (what, k, int(sat.item()), want)
    return expect


# ---- a. the writers ---------------------------------------------------------------------------------------------------------------
SPLIT_SHAPES = [(r, c) for c in (24, 128, 360, 1000) for r in (1, 7, 129)] + [(2200, 1000)]   # the last one wraps the grid-stride loop


@pytest.mark.parametrize("prec", [F16F8, BF16], ids=["f16f8", "bf16"])
@pytest.mark.parametrize("shape", SPLIT_SHAPES, ids=["%dx%d" % s for s in SPLIT_SHAPES])
def test_split_planes_exact(eng, prec, shape):
    """The pad-split (tc_split_planes: the generator's input and output-gradient splits): planes [rows, Cpad], zero columns past C.
    2200 x 1024 elements lie above the launchers' grid cap (132 * 16 blocks of 256 threads, 4 values per thread for F16F8), so their
    grid-stride loops take a second lap."""
    lib, h, N = eng
    rows, Cn = shape
    cpad = _ru(Cn, 128 if prec == F16F8 else 64)
    rng = np.random.default_rng(rows * 1000 + Cn)
    x = _edge_filled(rows * Cn, rng).reshape(rows, Cn)
    xd = torch.from_numpy(x).cuda()
    xp = np.zeros((rows, cpad), np.float32); xp[:, :Cn] = x

    def call(hi, lo, sat):
        N.check(h, lib.cgvc_split_planes(h, prec, _p(xd), rows, Cn, _p(hi), _p(lo), _p(sat), None))
    n = _counted_calls(prec, call, rows * cpad, lambda: (xp, R.sat_count(xp)), "split %dx%d" % shape)
    print("split %dx%d prec %d: %d saturated groups" % (rows, Cn, prec, n))
    if prec == F16F8 and rows * Cn >= 1000:
        assert n > 0                                   # the inputs reach past the window


def _im2col_ref(x, T, kw, d):
    M, Cn = x.shape
    pl = (kw - 1) // 2
    cpad = _ru(kw * Cn, 128)
    out = np.zeros((M, cpad), np.float32)
    for m in range(M):
        w = m % T
        for t in range(kw):
            ws = w + d * (t - pl)
            if 0 <= ws < T:
                out[m, t * Cn:(t + 1) * Cn] = x[m - w + ws]
    return out


@pytest.mark.parametrize("prec", [F16F8, BF16], ids=["f16f8", "bf16"])
@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("T,samples", [(32, 5), (128, 3)])
def test_im2col_planes_exact(eng, prec, d, T, samples):
    """The tap lowering of the generator's 15-tap edge layers (option edge_lower): dir = +1 is h1's input, dir = -1 the o1 output
    gradient -- the lambda-scaled L1 gradient, the main saturation site of a train step.  Zero rows outside each sample."""
    lib, h, N = eng
    kw, Cn = 15, 24
    M = T * samples
    rng = np.random.default_rng(7 + T + d)
    x = _edge_filled(M * Cn, rng).reshape(M, Cn)
    xd = torch.from_numpy(x).cuda()
    ref = _im2col_ref(x, T, kw, d)

    def call(hi, lo, sat):
        N.check(h, lib.cgvc_im2col_planes(h, prec, _p(xd), M, T, Cn, kw, d, _p(hi), _p(lo), _p(sat), None))
    n = _counted_calls(prec, call, ref.size, lambda: (ref, R.sat_count(ref)), "im2col T=%d dir=%d" % (T, d))
    print("im2col T=%d dir=%+d prec %d: %d saturated groups" % (T, d, prec, n))
    if prec == F16F8:
        assert n > 0


# (B, R, C, shuffle, gate, post_stream, post_onepass): the forward / backward kernel form each one takes (simt_kernels.cu dispatch)
POST_PLANE_CASES = [
    (6, 32, 128, 1, 1, 1, 1),      # streaming / streaming
    (6, 48, 128, 1, 1, 1, 1),      # streaming / streaming
    (6, 64, 128, 1, 1, 1, 1),      # streaming / streaming
    (6, 96, 96, 1, 1, 1, 1),       # streaming / streaming
    (6, 128, 64, 2, 1, 1, 1),      # streaming / streaming, pixel shuffle
    (6, 384, 32, 1, 1, 1, 1),      # streaming / streaming
    (6, 32, 96, 1, 1, 0, 1),       # stats + apply / one-pass; C = 96: the lanes of channels 96..127 have cvalid == false
    (6, 48, 128, 1, 1, 0, 1),      # stats + apply / one-pass
    (6, 64, 256, 2, 1, 0, 1),      # stats + apply / one-pass, pixel shuffle
    (6, 516, 96, 1, 1, 1, 1),      # stats + apply / sums + apply, cvalid == false
    (6, 64, 128, 2, 1, 1, 0),      # streaming / sums + apply (post_onepass = 0), pixel shuffle
    (6, 32, 128, 1, 0, 1, 1),      # residual h2 form: stats + apply with resid / streaming
    (6, 32, 96, 1, 0, 1, 1),       # residual: stats + apply / one-pass, cvalid == false
    (6, 64, 128, 2, 0, 1, 1),      # residual: stats + apply / one-pass, pixel shuffle
    (6, 516, 128, 1, 0, 1, 1),     # residual: stats + apply / sums + apply
    (6, 48, 96, 1, 0, 1, 0),       # residual: stats + apply / sums + apply (post_onepass = 0), cvalid == false
]


def _post_oracle(p, par, resid, dy, B, R_, Cn, sh, gate):
    from oracle import cyclegan_oracle as O
    Cc = Cn * sh
    pr = torch.from_numpy(p).double().requires_grad_(True)
    pars = [torch.from_numpy(t).double().requires_grad_(True) for t in par]
    a = pr[..., :Cc].reshape(B, R_, Cn)
    if gate:
        g = pr[..., Cc:].reshape(B, R_, Cn)
        y = O.glu(O.instance_norm(a, pars[0], pars[1]), O.instance_norm(g, pars[2], pars[3]))
    else:
        y = O.instance_norm(a, pars[0], pars[1]) + torch.from_numpy(resid).double()
    y.backward(torch.from_numpy(dy).double())
    return y.detach().numpy(), pr.grad.numpy(), [None if t.grad is None else t.grad.numpy() for t in pars]


@pytest.mark.parametrize("prec", [F16F8, BF16], ids=["f16f8", "bf16"])
@pytest.mark.parametrize("case", POST_PLANE_CASES, ids=["B%d_R%d_C%d_s%d_g%d_st%d_op%d" % c for c in POST_PLANE_CASES])
def test_in_glu_planes_exact(eng, prec, case):
    """Instance norm (+ GLU | + residual) forward and backward with planes: the planes are the quantisation of the kernel's own fp32
    y / dp of the same call (so exact whatever the kernel's summation order), and y, dp and the parameter gradients are within the
    2e-5 of test_in_glu_fwd_bwd of float64.  Magnitudes reach both window edges: forward beta_a per channel from the edge table with a
    small gamma_a; backward dy scaled by 2^k per sample, k from -40 to +20, and a second call with a NaN in one sample and an inf in
    another."""
    lib, h, N = eng
    B, R_, Cn, sh, gate, stream, onepass = case
    Cc = Cn * sh
    ldp = (2 if gate else 1) * Cc
    rng = np.random.default_rng(list(case))
    p = (rng.standard_normal((B, R_ // sh, ldp)) * 1.7 + 0.3).astype(np.float32)
    edge = R.edge_values(); edge = edge[np.isfinite(edge)]
    beta_a = np.resize(edge[rng.permutation(edge.size)], Cn).astype(np.float32)
    gamma_a = np.exp2(-rng.integers(4, 30, Cn)).astype(np.float32)
    beta_g = (rng.standard_normal(Cn) * 0.3).astype(np.float32); gamma_g = (rng.standard_normal(Cn) * 0.3 + 1.0).astype(np.float32)
    resid = None if gate else rng.standard_normal((B, R_, Cn)).astype(np.float32)
    ks = np.linspace(-40, 20, B).round().astype(int)
    dy = (rng.standard_normal((B, R_, Cn)) * np.exp2(ks)[:, None, None]).astype(np.float32)
    y_ref, dp_ref, par_ref = _post_oracle(p, (beta_a, gamma_a, beta_g, gamma_g), resid, dy, B, R_, Cn, sh, gate)

    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pd, dyd, rd = dev(p), dev(dy), dev(resid)
    pars = [dev(t) for t in (beta_a, gamma_a, beta_g, gamma_g)]
    y = torch.empty(B, R_, Cn, device="cuda"); stats = torch.empty(B, 4, Cn, device="cuda")
    dp = torch.empty_like(pd)
    assert lib.cgvc_set_option(h, b"post_stream", stream) == 0 and lib.cgvc_set_option(h, b"post_onepass", onepass) == 0
    try:
        def fwd(hi, lo, sat):
            N.check(h, lib.cgvc_in_glu_forward_planes(h, _p(pd), _p(pars[0]), _p(pars[1]), _p(pars[2]), _p(pars[3]), _p(y), _p(stats),
                                                      B, R_, Cn, sh, prec, gate, _p(rd), _p(hi), _p(lo), _p(sat), None))

        def y_now():
            yy = y.cpu().numpy()
            return yy, R.sat_count(yy)
        nf = _counted_calls(prec, fwd, B * R_ * Cn, y_now, "forward %s" % (case,))
        errs = {"y": rel_l2(y.cpu().numpy(), y_ref)}

        grads = []

        def bwd_with(dyt):
            def bwd(hi, lo, sat):
                grads[:] = [torch.zeros(Cn, device="cuda") for _ in range(4)]
                N.check(h, lib.cgvc_in_glu_backward_planes(h, _p(dyt), _p(pd), _p(stats), _p(pars[0]), _p(pars[1]), _p(pars[2]),
                                                           _p(pars[3]), _p(dp), _p(grads[0]), _p(grads[1]), _p(grads[2]), _p(grads[3]),
                                                           B, R_, Cn, sh, prec, gate, _p(hi), _p(lo), _p(sat), None))
            return bwd

        def dp_now():
            d = dp.cpu().numpy()
            return d, R.sat_count(d)
        nb = _counted_calls(prec, bwd_with(dyd), pd.numel(), dp_now, "backward %s" % (case,))
        dpn = dp.cpu().numpy()
        errs["dp"] = max(rel_l2(dpn[b], dp_ref[b]) for b in range(B))          # per sample: their scales are 2^60 apart
        names = ("dbeta_a", "dgamma_a", "dbeta_g", "dgamma_g")[:4 if gate else 2]
        for i, n in enumerate(names):
            errs[n] = rel_l2(grads[i].cpu().numpy(), par_ref[i])

        bad = dy.copy(); bad[1, R_ // 3, 5] = np.nan; bad[2, 0, Cn - 1] = np.inf
        nbad = _counted_calls(prec, bwd_with(dev(bad)), pd.numel(), dp_now, "backward NaN / inf %s" % (case,))
    finally:
        assert lib.cgvc_set_option(h, b"post_stream", 1) == 0 and lib.cgvc_set_option(h, b"post_onepass", 1) == 0
    print("in_glu planes %s prec %d: saturated groups fwd %d bwd %d bwd(NaN/inf) %d; " % (case, prec, nf, nb, nbad)
          + " ".join("%s=%.2e" % kv for kv in errs.items()))
    for k, v in errs.items():
        assert v < 2e-5, (case, k, v)
    if prec == F16F8:
        assert nb > 0 and nbad > nb                    # dy * 2^20 leaves the window; NaN and inf are counted


# ---- b. the GEMM window -----------------------------------------------------------------------------------------------------------
WINDOW_CASES = [
    ("G.res_h1", 3, 1, 32, 512, 1, 3, 1024, 1, 1),
    ("G.d1", 2, 1, 128, 128, 1, 5, 256, 1, 2),
    ("D.d1", 2, 24, 64, 128, 3, 3, 256, 2, 2),
    ("G.o1", 2, 1, 128, 256, 1, 15, 24, 1, 1),           # the 32-wide output tile
]
ACT_WINDOW = (2.0 ** -7, 256.0)       # activations and gradients (S_hi = 1, S_lo = 2^12): full precision for |v| in [lo, hi)
WGT_WINDOW = (2.0 ** -10, 32.0)       # weights (S_hi = 8, S_lo = 2^15)


def _window_reference(case):
    from oracle import cyclegan_oracle as O
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    g = torch.Generator().manual_seed(5)
    x = torch.randn((B, H, W, Cin), generator=g, dtype=torch.float64).float()
    w = (torch.randn((kh, kw, Cin, Cout), generator=g, dtype=torch.float64) / np.sqrt(kh * kw * Cin)).float()
    b = torch.randn((Cout,), generator=g, dtype=torch.float64).float()
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    y = O.conv2d_same(xr, wr, br, (sh, sw))
    dy = torch.randn(tuple(y.shape), generator=g, dtype=torch.float64).float()
    y.backward(dy.double())
    return (x, w, b, dy), (y.detach().numpy(), xr.grad.numpy(), wr.grad.numpy(), br.grad.numpy())


def _err(got, ref):
    got = np.asarray(got, np.float64)
    return rel_l2(got, ref) if np.isfinite(got).all() else float("inf")


def _sweep(eng, case, prec, octaves):
    """errors of y, dx, dw, db against float64 with one operand (x, w or dy) scaled by 2^k: {(operand, k): (errs, max|v|, rms v)}"""
    lib, h, N = eng
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    (x, w, b, dy), (y0, dx0, dw0, db0) = _window_reference(case)
    xd, wd, bd, dyd = (t.cuda() for t in (x, w, b, dy))
    out = {}
    for op in ("x", "w", "dy"):
        base = {"x": x, "w": w, "dy": dy}[op]
        vmax, vrms = float(base.abs().max()), float(base.double().pow(2).mean().sqrt())
        for k in octaves:
            s = 2.0 ** k
            sx, sw_, sdy = (s if op == "x" else 1.0), (s if op == "w" else 1.0), (s if op == "dy" else 1.0)
            xs, ws, dys, bs = xd * sx, wd * sw_, dyd * sdy, bd * (sx * sw_)
            yv = torch.empty(tuple(y0.shape), device="cuda")
            N.check(h, lib.cgvc_conv_forward(h, prec, _p(xs), _p(ws), _p(bs), _p(yv), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
            dx = torch.empty_like(xs); dw = torch.zeros_like(ws); db = torch.zeros_like(bs)
            N.check(h, lib.cgvc_conv_backward(h, prec, _p(xs), _p(ws), _p(dys), _p(dx), _p(dw), _p(db), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
            torch.cuda.synchronize()
            errs = (_err(yv.cpu(), y0 * sx * sw_), _err(dx.cpu(), dx0 * sw_ * sdy), _err(dw.cpu(), dw0 * sx * sdy), _err(db.cpu(), db0 * sdy))
            out[(op, k)] = (errs, vmax * s, vrms * s)
    return out


def _print_curve(name, prec, res, octaves, inside):
    for op in ("x", "w", "dy"):
        print("%s prec %d, %s * 2^k:  k  max|v|     rms v      y        dx       dw       db" % (name, prec, op))
        for k in octaves:
            (e, vmax, vrms) = res[(op, k)]
            print("   %+4d %9.2e %9.2e  %s%s" % (k, vmax, vrms, " ".join("%8.1e" % v for v in e), "" if inside(op, vmax, vrms) else "   (outside)"))


@pytest.mark.parametrize("case", WINDOW_CASES, ids=[c[0] for c in WINDOW_CASES])
def test_f16f8_gemm_window(eng, case):
    """F16F8 forward, data gradient and weight gradient (wgrad_f16 = 1, the default of an F16F8 engine) with x, w and dy scaled by 2^k
    one at a time, against float64.

    The window the formats predict, per element v of an operand (tests/f16f8_ref.py has the planes):
    - activations and gradients (S_hi = 1, S_lo = 2^12): q16 = fp16(v) carries 11 bits, the lo plane e4m3((v - q16) * 2^12) the next 4.
      The lo plane is normal (full precision) while |v - q16| * 2^12 >= 2^-6, with |v - q16| ~ 2^-12 |v|: |v| >= ~2^-7.  It flushes to
      zero once |v - q16| * 2^12 <= 2^-10, i.e. below |v| ~ 2^-10, where only fp16's 11 bits remain (2^-12 relative; a GEMM of such
      operands still sits near 3e-4); below 2^-14 fp16 itself is subnormal and loses a bit per octave.  The hi cross term
      e4m3(q16) flushes for |q16| <= 2^-10.  Upwards the lo plane may clamp from |v| >= 256 (the residual reaches 2^-3 there, * 2^12 >
      448), the hi plane from 448 on, and fp16 overflows at 65504.  Full precision: 2^-7 <= |v| < 256.
    - weights (S_hi = 8, S_lo = 2^15): the hi plane clamps above |v| = 56 and the lo plane from |v| >= 32 (residual 2^-6 * 2^15 = 512), so
      the planes are exact below 32; the lo plane stays normal down to |v| ~ 2^-9 and flushes below ~2^-13: full precision down to about
      2^-10.
    Asserted (4e-4, dw 6e-4 as test_conv_f16f8_weight_gradient_from_fp16_planes) for the octaves whose largest element lies below the
    upper edge and whose RMS lies at or above the lower edge; the rest of the curve is printed."""
    lib, h, N = eng
    octaves = list(range(-30, 19, 2))
    assert lib.cgvc_set_option(h, b"wgrad_f16", 1) == 0
    try:
        res = _sweep(eng, case, F16F8, octaves)
    finally:
        assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0

    def inside(op, vmax, vrms):
        lo, hi = WGT_WINDOW if op == "w" else ACT_WINDOW
        return vmax < hi and vrms >= lo
    _print_curve(case[0], F16F8, res, octaves, inside)
    bad, n_in = [], 0
    for (op, k), (e, vmax, vrms) in res.items():
        if not inside(op, vmax, vrms):
            continue
        n_in += 1
        for out_name, v in zip(("y", "dx", "dw", "db"), e):
            if v >= (6e-4 if out_name == "dw" else 4e-4):
                bad.append((op, k, out_name, v))
    assert n_in >= 12 and not bad, bad


@pytest.mark.parametrize("case", WINDOW_CASES, ids=[c[0] for c in WINDOW_CASES])
def test_bf16x3_gemm_has_no_window(eng, case):
    """bf16x3 over +-40 octaves of each operand: bf16 has fp32's exponent range, so the planes never clamp or flush here and every
    octave stays within the 2e-4 of test_conv_bf16x3."""
    octaves = list(range(-40, 41, 4))
    res = _sweep(eng, case, BF16, octaves)
    _print_curve(case[0], BF16, res, octaves, lambda op, vmax, vrms: True)
    bad = [(op, k, n, v) for (op, k), (e, _, _) in res.items() for n, v in zip(("y", "dx", "dw", "db"), e) if not v < 2e-4]
    assert not bad, bad


# ---- c. the loss scales the scaler can reach ---------------------------------------------------------------------------------------
# The lowest loss scale at which the batch-2 train step's gradients are parity-grade (measured, see test_gradients_at_every_loss_scale)
PARITY_LOWER_EDGE = 2.0 ** 4


def _scale_sweep(P, A, B, lam_c, lam_i, scales):
    """worst relative L2 of the gradient tensors against float64 and sat_grad, per loss scale, from a dynamic-mode F16F8 engine"""
    import cgvc
    from cgvc import native as N
    from oracle import cyclegan_oracle as O
    _, G, _, _ = O.gradients(A, B, P, lam_c, lam_i)
    batch = A.shape[0]
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision="f16f8", log_dir='/tmp/cgvc_log',
                      loss_scale="dynamic")
    m.set_params({k: v.numpy() for k, v in P.items()})
    ref = {k: v.to("cuda") for k, v in G.items()}
    out = {}
    for s in scales:
        m._chk(m._lib.cgvc_set_loss_scale_state(m._handle, float(s), 0, 0, m._stream()))
        m.compute_gradients(A.numpy(), B.numpy(), lam_c, lam_i)
        st = m.loss_scale_state()
        assert st["scale"] == s, st
        worst, name, zero_max = 0.0, "", 0.0
        for k, g_ref in ref.items():
            g = m._view(N.ARENA_GRAD, k).double()
            n = float(g_ref.norm())
            if n < 1e-9:                               # conv biases feeding an instance norm: analytically zero
                zero_max = max(zero_max, float(g.abs().max()))
                continue
            e = float((g - g_ref).norm()) / n
            if not np.isfinite(e):
                e = float("inf")
            if e >= worst:
                worst, name = e, k
        out[s] = (worst, name, int(st["sat_grad"]), zero_max)
        print("loss scale 2^%-3d  sat_grad %6d  worst gradient rel_l2 %.3e (%s)  zero-gradient biases max %.1e"
              % (int(np.log2(s)), st["sat_grad"], worst, name, zero_max))
    del m
    torch.cuda.empty_cache()
    return out


def test_gradients_at_every_loss_scale(oracle_params64):
    """compute_gradients of a dynamic-mode F16F8 engine at batch 2 (the weights and inputs of test_losses_and_gradients, lambdas
    10 / 5) at every scale the dynamic scaler can reach, 2^0 ... 2^24 in steps of 4: the gradients are formed with the scale, quantised
    into the planes, and the scale removed again.  Too small a scale pushes the gradient planes below the window (fp16 subnormals, the
    e4m3 planes flushed to zero) without any count; too large a scale saturates them, which sat_grad reports.

    Asserted: every scale at or above PARITY_LOWER_EDGE (the measured lowest parity-grade scale) whose planes did not saturate is within
    1e-3 of float64 -- what dynamic mode relies on when it accepts a step -- and the static scale of batch 2 (2^10) and 2^16, where a
    batch-256 run settled (DESIGN.md section 10), lie at least 2^4 above that edge."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=9, batch=2, frames=128, dtype=torch.float64)
    scales = [2.0 ** k for k in range(0, 25, 2)]
    res = _scale_sweep(oracle_params64, A, B, 10.0, 5.0, scales)
    parity = [s for s in scales if res[s][0] < 1e-3 and res[s][2] == 0]
    print("parity-grade (rel_l2 < 1e-3, no saturation) at scales 2^%s; lowest 2^%d; the test's edge 2^%d"
          % ([int(np.log2(s)) for s in parity], int(np.log2(min(parity))) if parity else -1, int(np.log2(PARITY_LOWER_EDGE))))
    bad = [(s, res[s]) for s in scales if s >= PARITY_LOWER_EDGE and res[s][2] == 0 and not res[s][0] < 1e-3]
    assert not bad, bad
    assert any(res[s][2] == 0 for s in scales if s >= PARITY_LOWER_EDGE)
    assert 2.0 ** 10 >= 16 * PARITY_LOWER_EDGE and 2.0 ** 16 >= 16 * PARITY_LOWER_EDGE


def test_gradients_at_the_scale_lambda_1e4_settles_on(oracle_params64):
    """The corner of test_saturation_is_counted_and_the_dynamic_scale_recovers: batch 1, lambda_cycle = 1e4.  The scaled L1 gradient
    saturates the planes down to a scale of 4, so dynamic mode settles on 2.  Whether the gradients are parity-grade there is reported,
    not asserted (DESIGN.md section 10 has the verdict); the planes must not saturate at 2."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=60, batch=1, frames=128, dtype=torch.float64)
    res = _scale_sweep(oracle_params64, A, B, 1e4, 5.0, [2.0, 4.0, 2.0 ** 8])
    worst, name, sat, _ = res[2.0]
    print("lambda_cycle 1e4, batch 1, loss scale 2: worst gradient rel_l2 %.3e (%s), sat_grad %d: %s"
          % (worst, name, sat, "parity-grade" if worst < 1e-3 else "NOT parity-grade (1e-3)"))
    assert sat == 0 and res[4.0][2] > 0
