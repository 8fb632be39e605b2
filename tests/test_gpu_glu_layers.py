"""The layers without an instance norm and the loss heads against float64 (tests/glu_ref.py), through the entry points that run the
train step's own launches.

a. GLU-only form (post_apply_fwd / post_apply_bwd <false, true>): the generator's h1 at R = 128, conversion lengths R = 36 and 516 (a row
   tail of the 32-position blocks), the discriminator's h1 at R = 1536, and the bench's batch.  y and dP against float64; their planes
   and saturation counts by the counted-call protocol of test_gpu_planes.py, also with dy scaled per sample across 2^-40 .. 2^20 and a
   NaN / inf sample; the conv-bias gradients with atomic adds and with the deterministic partial rows.
b. The discriminator's input layer, fused (conv_c1_glu_fwd, glu_bwd_wgrad_c1, glu_bwd_proj_c1 + gather_taps) and unfused (conv_c1_fwd +
   the GLU-only form, wgrad_c1, proj_taps + gather_taps), deterministic off and on, and at the bench's D-loss shape (512 samples,
   T = 128, M = 786 432 rows).
c. The head (head_fwd, head_loss_bwd) in the step's three roles and with saturated logits; the L1 loss (l1_loss_grad).

Tiers.  Lattice (glu_ref's dyadic cases, g = 0 so that sigmoid = 1/2 exactly): every output bitwise.  Dense (randn): y and dP within
glu_ref.y_bound / dp_bound of float64 at the kernel's own P; every reduction within gamma_L * sum |terms| (+ the propagated dP error),
L the longest fp32 addition chain of its launch (glu_ref.*_chain); the head's gradients at the kernel's own prob.
A failure names the sample, position and channel, and the CTA or row block, of the first wrong values.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import f16f8_ref as Q
import glu_ref as G

pytestmark = pytest.mark.gpu

FP32, BF16X3, F16F8 = 0, 1, 3
PNAME = {FP32: "fp32", BF16X3: "bf16x3", F16F8: "f16f8"}
SENTINEL = 0x55
U = G.U

# worst measured values (fraction of the bound) are printed as MEAS lines and recorded in DESIGN.md section 10


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _make_engine(det):
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 16, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    work = None
    if det:
        N.check(h, lib.cgvc_set_option(h, b"deterministic", 1))
        nb = C.c_size_t(0)
        N.check(h, lib.cgvc_arena_bytes(h, N.ARENA_WORK, C.byref(nb)))
        work = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
        N.check(h, lib.cgvc_bind_arena(h, N.ARENA_WORK, C.c_void_p(work.data_ptr()), nb.value))
    return lib, h, N, work


@pytest.fixture(scope="module")
def engines():
    e = {det: _make_engine(det) for det in (0, 1)}
    yield e
    for lib, h, N, _ in e.values():
        lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _planes(prec, n):
    if prec == FP32:
        return None, None
    if prec == F16F8:
        hi = torch.empty(n, dtype=torch.float16, device="cuda"); lo = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    else:
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda"); lo = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    hi.view(torch.uint8).fill_(SENTINEL); lo.view(torch.uint8).fill_(SENTINEL)
    return hi, lo


def check_planes(prec, hi, lo, x, where, what):
    """the planes hold exactly the planes of the kernel's own fp32 output x"""
    if prec == FP32:
        return
    x = np.ascontiguousarray(x, np.float32).reshape(-1)
    n = x.size
    if prec == F16F8:
        q16, q8hi, q8lo = Q.quant_planes(x)
        l8 = lo.cpu().numpy()
        pairs = ((hi.cpu().numpy().astype(np.float64), q16.astype(np.float64)), (Q.e4m3_decode(l8[:n]), Q.e4m3_decode(q8hi)),
                 (Q.e4m3_decode(l8[n:]), Q.e4m3_decode(q8lo)))
    else:
        bh, bl = Q.split_bf16(x)
        d = lambda t: Q.bf16_decode(t.view(torch.int16).cpu().numpy().view(np.uint16)).astype(np.float64)
        pairs = ((d(hi), Q.bf16_decode(bh).astype(np.float64)), (d(lo), Q.bf16_decode(bl).astype(np.float64)))
    for k, (g, r) in enumerate(pairs):
        report(~Q.same_values(g, r), g, r, where, "%s: plane %d not the quantisation of the kernel's output" % (what, k))


def report(bad, got, ref, where, what):
    bad = np.asarray(bad).reshape(-1)
    idx = np.flatnonzero(bad)
    if idx.size:
        g = np.asarray(got, np.float64).reshape(-1); r = np.asarray(ref, np.float64).reshape(-1)
        lines = ["  %s: got %r, reference %r" % (where(int(i)), g[i], r[i]) for i in idx[:8]]
        raise AssertionError("%s: %d of %d values wrong; first:\n%s" % (what, idx.size, bad.size, "\n".join(lines)))


def bits(got, ref, where, what):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    report(~Q.same_values(got, ref), got, ref, where, what)


def within(got, ref, bound, where, what):
    """|got - ref| <= bound elementwise (torch float64 tensors); returns the worst ratio"""
    err = (got - ref).abs()
    report((~(err <= bound)).cpu().numpy(), got.cpu().numpy(), ref.cpu().numpy(), where, what)
    return float((err / bound).max())


def _np(t):
    return t.double().cpu().numpy()


# ---- a. the GLU-only form -------------------------------------------------------------------------------------------------------
GLU_C = 128
GLU_SHAPES = [(4, 128), (3, 36), (2, 516), (2, 1536), (512, 128)]


def _where_glu(R, ld):
    def w(i):
        m, col = divmod(i, ld)
        b, r = divmod(m, R)
        br, c = divmod(col, GLU_C) if ld == 2 * GLU_C else (0, col)
        return "sample %d, position %d, %s channel %d (32-position block %d)" % (b, r, "gate" if br else "a", c, r // G.POST_ROWS)
    return w


def _glu_fwd(eng, prec, P, B, R, sat=None, with_y=True):
    lib, h, N, _ = eng
    y = torch.full((B, R, GLU_C), float("nan"), device="cuda") if with_y else None
    hi, lo = _planes(prec, B * R * GLU_C)
    N.check(h, lib.cgvc_glu_forward_planes(h, _p(P), _p(y), B, R, GLU_C, prec, _p(hi), _p(lo), _p(sat), None))
    torch.cuda.synchronize()
    return y, hi, lo


def _glu_bwd(eng, prec, dy, P, B, R, sat=None, bias=True):
    lib, h, N, _ = eng
    dp = torch.full((B, R, 2 * GLU_C), float("nan"), device="cuda")
    hi, lo = _planes(prec, B * R * 2 * GLU_C)
    db = [torch.zeros(GLU_C, device="cuda") + 0.25 for _ in range(2)] if bias else [None, None]
    N.check(h, lib.cgvc_glu_backward_planes(h, _p(dy), _p(P), _p(dp), _p(db[0]), _p(db[1]), B, R, GLU_C, prec, _p(hi), _p(lo), _p(sat), None))
    torch.cuda.synchronize()
    return dp, hi, lo, db


def _counted(prec, run, out_of):
    """run(sat) three times -- with a counter, again with it (the count doubles), with NULL: the same planes each time.  out_of(result)
    gives the kernel's fp32 output; returns the first result and the count"""
    sat = torch.zeros(1, dtype=torch.int64, device="cuda")
    first = None
    for k, ctr in enumerate((sat, sat, None)):
        r = run(ctr)
        x = out_of(r).cpu().numpy()
        if first is None:
            first, expect = r, Q.sat_count(x)
        else:
            for a, b in zip(r[1:3], first[1:3]):
                if a is not None:
                    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), ("planes differ on call", k)
        if ctr is not None:
            want = (k + 1) * expect if prec == F16F8 else 0
            assert int(sat.item()) == want, ("saturation count", k, int(sat.item()), want)
    return first, expect


GLU_PARAMS = [(s, p, t) for s in GLU_SHAPES for p in (FP32, BF16X3, F16F8) for t in ("lattice", "dense")]


@pytest.mark.parametrize("shape,prec,tier", GLU_PARAMS, ids=["B%dR%d-%s-%s" % (s + (PNAME[p], t)) for s, p, t in GLU_PARAMS])
def test_glu_only_form(engines, shape, prec, tier):
    B, R = shape
    what = "GLU B%d R%d %s %s" % (B, R, PNAME[prec], tier)
    rng = np.random.default_rng(_seed("glu", B, R, tier))
    M = B * R
    if tier == "lattice":
        P, dy = G.lattice_glu_case(rng, M, GLU_C)
    else:
        P = rng.standard_normal((M, 2 * GLU_C)).astype(np.float32) * 2
        dy = rng.standard_normal((M, GLU_C)).astype(np.float32)
    Pd, dyd = _dev(P).reshape(B, R, 2 * GLU_C), _dev(dy).reshape(B, R, GLU_C)
    eng = engines[0]
    (y, hi, lo), _ = _counted(prec, lambda s: _glu_fwd(eng, prec, Pd, B, R, s), lambda r: r[0])
    wy = _where_glu(R, GLU_C)
    check_planes(prec, hi, lo, y.cpu().numpy(), wy, what + " y")
    if prec != FP32:                                  # planes only: the same bits
        _, hi2, lo2 = _glu_fwd(eng, prec, Pd, B, R, with_y=False)
        assert torch.equal(hi2.view(torch.uint8), hi.view(torch.uint8)) and torch.equal(lo2.view(torch.uint8), lo.view(torch.uint8)), what
    ref = G.glu_forward(Pd.reshape(M, -1))
    if tier == "lattice":
        bits(_np(y), (Pd[..., :GLU_C] / 2).double().cpu().numpy(), wy, what + ": y != a / 2 (the device's sigmoid(0) is not exactly 1/2?)")
    ry = within(y.reshape(M, -1).double(), ref, G.y_bound(Pd.reshape(M, -1)), wy, what + ": y beyond y_bound")
    (dp, dhi, dlo, db), _ = _counted(prec, lambda s: _glu_bwd(eng, prec, dyd, Pd, B, R, s, bias=False), lambda r: r[0])
    wp = _where_glu(R, 2 * GLU_C)
    check_planes(prec, dhi, dlo, dp.cpu().numpy(), wp, what + " dP")
    dref, ba, bg = G.glu_backward(Pd.reshape(M, -1), dyd.reshape(M, -1))
    if tier == "lattice":
        bits(_np(dp.reshape(M, -1)), dref.cpu().numpy(), wp, what + ": dP not exact")
    rp = within(dp.reshape(M, -1).double(), dref, G.dp_bound(Pd.reshape(M, -1), dyd.reshape(M, -1)), wp, what + ": dP beyond dp_bound")
    # conv-bias gradients, atomic and deterministic: 0.25 + column sums of dP
    L = G.post_bias_chain(B, R)
    eb = G.dp_bound(Pd.reshape(M, -1), dyd.reshape(M, -1)).sum(dim=0)
    bound = G.gamma(L) * (dref.abs().sum(dim=0) + 0.25) + eb + 1e-45
    worst = 0.0
    for det in (0, 1):
        outs = [_glu_bwd(engines[det], prec, dyd, Pd, B, R)[3] for _ in range(2 if det else 1)]
        got = torch.cat(outs[0]).double()
        want = torch.cat([ba, bg]) + 0.25
        wb = lambda i: "%s bias channel %d" % ("gate" if i >= GLU_C else "a", i % GLU_C)
        if tier == "lattice":
            bits(_np(got), want.cpu().numpy(), wb, what + " det=%d: dbias not exact" % det)
        worst = max(worst, within(got, want, bound, wb, what + " det=%d: dbias beyond gamma_%d" % (det, L)))
        if det:
            assert torch.equal(torch.cat(outs[0]), torch.cat(outs[1])), what + ": deterministic dbias differs between calls"
    print("MEAS glu %s y=%.3g dp=%.3g dbias=%.3g" % (what.replace(" ", "|"), ry, rp, worst))


@pytest.mark.parametrize("R", [128, 36])
def test_glu_only_planes_across_scales(engines, R):
    """F16F8 dP planes with dy scaled per sample by 2^-40 .. 2^20 (the window's edges and beyond), then a NaN / inf sample: the planes
    equal the quantisation of the kernel's own dP and the count equals the reference count (test_in_glu_planes_exact's protocol)"""
    B = 13
    rng = np.random.default_rng(_seed("scales", R))
    P = _dev(rng.standard_normal((B, R, 2 * GLU_C)).astype(np.float32) * 3)
    dy = rng.standard_normal((B, R, GLU_C)).astype(np.float32) * np.exp2(np.linspace(-40, 20, B)).astype(np.float32)[:, None, None]
    for name, d in (("scaled", dy), ("nan-inf", np.where(rng.random(dy.shape) < 0.01, np.float32(np.inf), dy).astype(np.float32))):
        if name == "nan-inf":
            d[3, 0, :4] = np.nan
        dd = _dev(d)
        (dp, hi, lo, _), n = _counted(F16F8, lambda s: _glu_bwd(engines[0], F16F8, dd, P, B, R, s, bias=False), lambda r: r[0])
        check_planes(F16F8, hi, lo, dp.cpu().numpy(), _where_glu(R, 2 * GLU_C), "GLU planes %s R%d" % (name, R))
        y, yhi, ylo = _glu_fwd(engines[0], F16F8, P * torch.from_numpy(np.exp2(np.linspace(-30, 12, B)).astype(np.float32)).cuda()[:, None, None], B, R)
        check_planes(F16F8, yhi, ylo, y.cpu().numpy(), _where_glu(R, GLU_C), "GLU y planes R%d" % R)
        print("MEAS glu planes %s R%d saturated groups %d" % (name, R, n))
        assert name != "scaled" or n > 0, "the scale sweep should saturate some groups"


# ---- b. the discriminator's input layer ------------------------------------------------------------------------------------------
H0 = 24
DISC_CASES = [(B, T) for B in (1, 3, 12) for T in (16, 48, 128, 144)]


def _where_disc(Ho, Wo, ld):
    def w(i):
        m, col = divmod(i, ld)
        b, r = divmod(m, Ho * Wo)
        y, x = divmod(r, Wo)
        return "sample %d, position (%d, %d), column %d (row %d, 64-row tile %d)" % (b, y, x, col, m, m // G.C1_ROWS)
    return w


def _disc_fwd(eng, prec, dops, B, T, fuse, sat=None):
    lib, h, N, _ = eng
    x, wa, wg, ba, bg = dops
    Ho, Wo = G.out_rows(H0, T)
    M = B * Ho * Wo
    p = torch.full((M, 2 * G.C1), float("nan"), device="cuda")
    y = torch.full((M, G.C1), float("nan"), device="cuda")
    hi, lo = _planes(prec, M * G.C1)
    fused = C.c_int(-1)
    N.check(h, lib.cgvc_disc_input_forward(h, prec, _p(x), _p(wa), _p(wg), _p(ba), _p(bg), _p(p), _p(y), _p(hi), _p(lo), _p(sat),
                                           B, H0, T, G.KH, G.KW, G.C1, G.SH, G.SW, fuse, C.byref(fused), None))
    torch.cuda.synchronize()
    assert fused.value == fuse
    return y, hi, lo, p


def _disc_bwd(eng, dy, p, dops, B, T, fuse, wgrad=True, dx=True):
    lib, h, N, _ = eng
    x, wa, wg, _, _ = dops
    g = [torch.zeros(G.KH * G.KW * G.C1, device="cuda") - 0.5 for _ in range(2)] + [torch.zeros(G.C1, device="cuda") + 0.5 for _ in range(2)]
    if not wgrad:
        g = [None] * 4
    d = torch.full((B, H0, T), float("nan"), device="cuda") if dx else None
    fused = C.c_int(-1)
    N.check(h, lib.cgvc_disc_input_backward(h, _p(dy), _p(p), _p(x), _p(wa), _p(wg), _p(g[0]), _p(g[1]), _p(g[2]), _p(g[3]), _p(d),
                                            B, H0, T, G.KH, G.KW, G.C1, G.SH, G.SW, fuse, C.byref(fused), None))
    torch.cuda.synchronize()
    assert fused.value == fuse
    return g, d


def _disc_case(B, T, tier):
    rng = np.random.default_rng(_seed("disc", B, T, tier))
    Ho, Wo = G.out_rows(H0, T)
    M = B * Ho * Wo
    if tier == "lattice":
        x, wa, wg, ba, bg = G.lattice_disc_case(rng, B, H0, T)
        dy = G.lattice_disc_dy(rng, M)
    else:
        x = rng.standard_normal((B, H0, T)).astype(np.float32)
        s = 1 / 3
        wa, wg = ((rng.standard_normal((G.KH, G.KW, 1, G.C1)) * s).astype(np.float32) for _ in range(2))
        ba, bg = ((rng.standard_normal(G.C1) * 0.1).astype(np.float32) for _ in range(2))
        dy = rng.standard_normal((M, G.C1)).astype(np.float32)
    return (x, wa, wg, ba, bg), dy


def _check_disc(engines, B, T, tier, prec, dev_ref):
    what = "D.h1 B%d T%d %s %s" % (B, T, PNAME[prec], tier)
    ops, dy = _disc_case(B, T, tier)
    dops = tuple(_dev(a) for a in ops)
    dyd = _dev(dy)
    x, wa, wg, ba, bg = ops
    Ho, Wo = G.out_rows(H0, T)
    M = B * Ho * Wo
    meas = {}
    outs = {}
    for fuse in (1, 0):
        (y, hi, lo, p), _ = _counted(prec, lambda s: _disc_fwd(engines[0], prec, dops, B, T, fuse, s), lambda r: r[0])
        outs[fuse] = (y, hi, lo, p)
    y, hi, lo, p = outs[1]
    wP, wy = _where_disc(Ho, Wo, 2 * G.C1), _where_disc(Ho, Wo, G.C1)
    # the two paths evaluate the same fmaf chain from the bias in tap order and the same a * sigmoid(g): bitwise equal
    bits(_np(outs[0][3]), _np(p), wP, what + ": unfused P differs from fused")
    bits(_np(outs[0][0]), _np(y), wy, what + ": unfused y differs from fused")
    for k in (1, 2):
        if outs[1][k] is not None:
            assert torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8)), what + ": unfused planes differ from fused"
    check_planes(prec, hi, lo, y.cpu().numpy(), wy, what + " y")
    Pref = G.disc_input_p(x, wa, wg, ba, bg, device=dev_ref)
    if tier == "lattice":
        bits(_np(p), Pref.cpu().numpy(), wP, what + ": P not the exact convolution")
        bits(_np(y), (p[:, :G.C1] / 2).double().cpu().numpy(), wy, what + ": y != a / 2")
    absP = G.disc_input_p(np.abs(x), np.abs(wa), np.abs(wg), np.abs(ba), np.abs(bg), device=dev_ref)
    meas["P"] = within(p.double().to(dev_ref), Pref, 10 * U * absP + 1e-45, wP, what + ": P beyond gamma_10")
    meas["y"] = within(y.double().to(dev_ref), G.glu_forward(p.to(dev_ref)), G.y_bound(p.to(dev_ref)), wy, what + ": y beyond y_bound")
    del outs, hi, lo
    # backward at the kernel's own P
    if tier == "lattice":
        assert G.disc_certificate(x, wa, p.to(dev_ref), dyd.to(dev_ref), device=dev_ref) < 2 ** 24, what + ": lattice certificate"
    ref = G.disc_input_backward(x, wa, wg, p.to(dev_ref), dyd.to(dev_ref), device=dev_ref)
    edp = G.dp_bound(p.to(dev_ref), dyd.to(dev_ref))
    adp = torch.cat([dyd.abs().double().to(dev_ref), dyd.abs().double().to(dev_ref) * p[:, :G.C1].abs().double().to(dev_ref)], dim=-1) + edp

    def terms(v):
        """(dw, dx, db) sums of |terms| for a nonnegative dP-like v: |x| gathered against v, v against |w|"""
        xt = torch.from_numpy(np.abs(x)).double().to(dev_ref)[..., None].requires_grad_(True)
        wt = torch.from_numpy(np.concatenate([np.abs(wa), np.abs(wg)], -1)).double().to(dev_ref).requires_grad_(True)
        G.O.conv2d_same(xt, wt, None, (G.SH, G.SW)).backward(v.reshape(B, Ho, Wo, -1))
        return wt.grad.reshape(-1, 2 * G.C1), xt.grad[..., 0], v.sum(dim=0)
    (tw, tx, tb), (ew_, ex_, eb_) = terms(adp), terms(edp)
    del adp
    Lw, Lx = G.c1_wgrad_chain(M), G.c1_dgrad_chain()
    ew = tw * G.gamma(Lw + 1) + ew_
    got = {}
    for det in (0, 1):
        for fuse in (1, 0):
            g, dx = _disc_bwd(engines[det], dyd, p, dops, B, T, fuse)
            got[(det, fuse)] = (g, dx)
            tag = "%s fuse=%d det=%d" % (what, fuse, det)
            wdw = lambda i: "tap %d channel %d" % divmod(i, G.C1)
            wdb = lambda i: "channel %d" % i
            wdx = lambda i: "sample %d, position (%d, %d)" % (i // (H0 * T), (i // T) % H0, i % T)
            rdw = [ref[0].reshape(-1, G.C1) - 0.5, ref[1].reshape(-1, G.C1) - 0.5]
            rdb = [ref[2] + 0.5, ref[3] + 0.5]
            if tier == "lattice":
                for k in range(2):
                    bits(_np(g[k]), rdw[k].reshape(-1).cpu().numpy(), wdw, tag + ": dw_%s not exact" % "ag"[k])
                    bits(_np(g[2 + k]), rdb[k].cpu().numpy(), wdb, tag + ": db_%s not exact" % "ag"[k])
                bits(_np(dx), ref[4].cpu().numpy(), wdx, tag + ": dx not exact")
            for k in range(2):
                meas["dw"] = max(meas.get("dw", 0), within(g[k].double().to(dev_ref).reshape(-1, G.C1), rdw[k], ew[:, k * G.C1:(k + 1) * G.C1] + 0.5 * U + 1e-45,
                                                           wdw, tag + ": dw_%s beyond gamma_%d" % ("ag"[k], Lw)))
                Lb = Lw if fuse else G.post_bias_chain(B, Ho * Wo)
                meas["db"] = max(meas.get("db", 0), within(g[2 + k].double().to(dev_ref), rdb[k], G.gamma(Lb + 1) * (tb[k * G.C1:(k + 1) * G.C1] + 0.5) + eb_[k * G.C1:(k + 1) * G.C1] + 1e-45,
                                                           wdb, tag + ": db_%s beyond gamma_%d" % ("ag"[k], Lb)))
            meas["dx"] = max(meas.get("dx", 0), within(dx.double().to(dev_ref), ref[4], G.gamma(Lx) * tx + ex_ + 1e-45, wdx, tag + ": dx beyond gamma_%d" % Lx))
    # deterministic mode: the same bits on a second call; the fused / unfused gap of the backward (summation order only)
    g2, dx2 = _disc_bwd(engines[1], dyd, p, dops, B, T, 1)
    for a, b in zip(g2 + [dx2], got[(1, 1)][0] + [got[(1, 1)][1]]):
        assert torch.equal(a, b), what + ": deterministic backward differs between calls"
    gap = max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) for a, b in zip(got[(0, 1)][0] + [got[(0, 1)][1]], got[(0, 0)][0] + [got[(0, 0)][1]]))
    if tier == "lattice":
        assert gap == 0, (what, "fused and unfused backward differ on the lattice", gap)
    print("MEAS disc %s P=%.3g y=%.3g dw=%.3g db=%.3g dx=%.3g fused_vs_unfused_bwd=%.3g" % (
        what.replace(" ", "|"), meas["P"], meas["y"], meas["dw"], meas["db"], meas["dx"], gap))


DISC_PARAMS = [(c, t) for c in DISC_CASES for t in ("lattice", "dense")]


@pytest.mark.parametrize("case,tier", DISC_PARAMS, ids=["B%dT%d-%s" % (c + (t,)) for c, t in DISC_PARAMS])
def test_disc_input_layer(engines, case, tier):
    B, T = case
    _check_disc(engines, B, T, tier, F16F8 if (B + T) % 2 == 0 else BF16X3, "cpu")


def test_disc_input_layer_fp32_writes_no_planes(engines):
    _check_disc(engines, 3, 48, "dense", FP32, "cpu")


def test_disc_input_layer_at_the_bench_shape(engines):
    """the D-loss pass of a batch-256 step: 512 samples, T = 128, M = 786 432 rows; float64 reference on the GPU"""
    _check_disc(engines, 512, 128, "dense", F16F8, "cuda")
    torch.cuda.empty_cache()


# ---- c. head and losses ----------------------------------------------------------------------------------------------------------
HEAD_ROWS = [6 * 8 * n for n in (1, 2, 128, 512)] + [4096]     # the step's shapes at T = 128; 4096: a power of two
ROLES = [("real", 1.0, 0.5, True), ("fake", 0.0, 0.5, True), ("g_adv", 1.0, 1.0, False)]


def _head(eng, y, w, b, rows, target, coef, gm, wgrad):
    lib, h, N, _ = eng
    prob = torch.full((rows,), float("nan"), device="cuda")
    N.check(h, lib.cgvc_head_forward(h, _p(y), rows, _p(w), _p(b), _p(prob), None))
    loss = torch.zeros(1, device="cuda") + 0.125
    dy = torch.full((rows, 1024), float("nan"), device="cuda")
    dw = torch.zeros(1024, device="cuda") + 0.5 if wgrad else None
    db = torch.zeros(1, device="cuda") + 0.5 if wgrad else None
    gmd = None if gm is None else torch.tensor([gm], dtype=torch.float32, device="cuda")
    N.check(h, lib.cgvc_head_loss_backward(h, _p(prob), _p(y), rows, _p(w), target, coef, _p(gmd), _p(loss), _p(dy), _p(dw), _p(db), None))
    torch.cuda.synchronize()
    return prob, loss, dy, dw, db


HEAD_PARAMS = [(r, role, gm, t) for r in HEAD_ROWS for role in ROLES for gm in (None, 2.0 ** 10) for t in ("lattice", "dense", "saturated")]


@pytest.mark.parametrize("rows,role,gm,tier", HEAD_PARAMS,
                         ids=["r%d-%s-gm%s-%s" % (r, role[0], "1" if gm is None else "2^10", t) for r, role, gm, t in HEAD_PARAMS])
def test_head_and_lsgan_loss(engines, rows, role, gm, tier):
    name, target, coef, wgrad = role
    what = "head rows %d %s gm %s %s" % (rows, name, gm, tier)
    rng = np.random.default_rng(_seed("head", rows, tier))
    if tier == "lattice":
        y, w, b = G.lattice_head_case(rng, rows)
    else:
        y = rng.standard_normal((rows, 1024)).astype(np.float32)
        w = (rng.standard_normal(1024) / 32).astype(np.float32)
        b = np.array([0.1], np.float32)
        if tier == "saturated":                       # logits near +-20: prob rounds to 1 or to 2e-9
            z = y @ w
            y = (y * (20 / np.abs(z).clip(1e-3))[:, None]).astype(np.float32)
    gmv = 1.0 if gm is None else gm
    wr = lambda i: "row %d (CTA %d of the grid-stride loop)" % (i, (i // 8) % min(-(-rows // 8), 296))
    for det in (0, 1):
        prob, loss, dy, dw, db = _head(engines[det], _dev(y), _dev(w), _dev(b), rows, target, coef, gm, wgrad)
        tag = what + " det=%d" % det
        pref = G.head_forward(y, w, b)
        if tier == "lattice":
            assert bool((prob == 0.5).all()), tag + ": prob != 1/2 on the lattice"
        # prob: one rounding of the dot product chain (8 per lane + 5 shuffles over 1024 terms), then the fast sigmoid
        z_err = G.gamma(8 * 4 + 5 + 1) * (np.abs(y) @ np.abs(w) + abs(b[0]))
        pb = torch.from_numpy(z_err) * pref * (1 - pref) + G.sigmoid_err(torch.from_numpy(y.astype(np.float64) @ w + b[0])) + U * pref + 1e-45
        meas_p = within(prob.double().cpu(), pref, pb, wr, tag + ": prob beyond its bound")
        lref, dyref, dwref, dbref = G.head_loss_backward(prob.cpu(), y, w, target, coef, gmv)
        L = G.head_chain(rows)
        dz = dyref[:, 0] / torch.from_numpy(w.astype(np.float64))[0]
        ldz = (prob.cpu().double() - target) ** 2 * coef / rows
        if tier == "lattice" and rows & (rows - 1) == 0:      # 1 / rows dyadic: loss, dz, dw, db exact
            assert float(loss) == 0.125 + lref, tag
            if wgrad:
                assert float(db) == 0.5 + float(dbref), tag
                bits(_np(dw), (dwref + 0.5).numpy(), lambda i: "column %d" % i, tag + ": dw not exact")
        if tier != "lattice":
            assert abs(float(loss) - 0.125 - lref) <= G.gamma(L + 4) * (float(ldz.sum()) + 0.125), (tag, "loss", float(loss) - 0.125, lref)
        dzb = 8 * U * dz.abs() + 1e-45
        within(dy.double().cpu(), dyref, dzb[:, None] * abs(torch.from_numpy(w.astype(np.float64)))[None, :] + U * dyref.abs() + 1e-45, wr,
               tag + ": dy beyond its bound")
        if wgrad:
            ab = (dz.abs()[:, None] * torch.from_numpy(np.abs(y).astype(np.float64))).sum(dim=0)
            within(dw.double().cpu(), dwref + 0.5, G.gamma(L + 8) * (ab + 0.5) + 1e-45, lambda i: "column %d" % i, tag + ": dw beyond gamma")
            assert abs(float(db) - 0.5 - float(dbref)) <= G.gamma(L + 8) * (float(dz.abs().sum()) + 0.5), (tag, "db", float(db) - 0.5, float(dbref))
        else:
            assert dw is None


L1_N = [100, 256 * 37 + 5, 592 * 256 * 3 + 77]


@pytest.mark.parametrize("n", L1_N)
@pytest.mark.parametrize("acc", [0, 1])
@pytest.mark.parametrize("scaled", [False, True], ids=["plain", "gscale-gm"])
def test_l1_loss_grad(engines, n, acc, scaled):
    what = "L1 n %d acc %d %s" % (n, acc, scaled)
    rng = np.random.default_rng(_seed("l1", n))
    yh = rng.standard_normal(n).astype(np.float32)
    y = rng.standard_normal(n).astype(np.float32)
    y[rng.random(n) < 0.1] = 0; yh[y == 0] = 0                  # exactly-zero differences
    d0 = rng.standard_normal(n).astype(np.float32)
    gs, gm = (10.0, 2.0 ** 12) if scaled else (None, None)
    want_d = G.l1_grad_bits(yh, y, gs, gm, d0 if acc else None)
    lref = G.l1_loss(yh, y)
    for det in (0, 1):
        lib, h, N, _ = engines[det]
        d = _dev(d0)
        loss = torch.zeros(1, device="cuda") + 0.25
        gsd = None if gs is None else torch.tensor([gs], dtype=torch.float32, device="cuda")
        gmd = None if gm is None else torch.tensor([gm], dtype=torch.float32, device="cuda")
        yhd, yd = _dev(yh), _dev(y)
        N.check(h, lib.cgvc_l1_loss_grad(h, _p(yhd), _p(yd), n, _p(gsd), _p(gmd), _p(loss), _p(d), acc, None))
        torch.cuda.synchronize()
        bits(d.cpu().numpy(), want_d, lambda i: "element %d (CTA %d)" % (i, (i // 256) % min(-(-n // 256), 592)), what + " det=%d: d" % det)
        L = G.l1_chain(n)
        assert abs(float(loss) - 0.25 - lref) <= G.gamma(L) * (lref + 0.25) + U * lref, (what, det, float(loss) - 0.25, lref)
