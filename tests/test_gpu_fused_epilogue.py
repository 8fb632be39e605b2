"""The gather-GEMM's fused instance-norm epilogues (csrc/tc_gemm.cu nt_tile_epilogue) against float64, element by element.

Forward (EPI 1 gated, EPI 2 residual h2, EPI 5 gated + pixel shuffle): every generator layer whose norm the epilogue fuses, at R = 32,
64 and 128 positions per sample, with tail tiles (a last 128-row tile that is only part samples) and one multi-wave persistent walk, in
bf16x3, bf16 and f16f8, in the training form (P and stats kept), without the fp32 y, and in the inference form (P = stats = NULL).
Backward (EPI 3 gated, EPI 4 residual; opt-in `fuse_bwd`): the three data-gradient launches of a residual block whose epilogue runs the
upstream layer's IN backward, with and without accumulation, in bf16x3 and bf16.

Tiers (fused_ref.py has the references and the lattice):
  P        lattice: bitwise the exact convolution + bias.   dense: bitwise the fallback's plain-epilogue P.
  mean     lattice: bitwise float64 (sums of integers, R a power of two).   dense: within MEAN_ULPS u * mean|P| of float64 of the
           kernel's own P.
  rstd     within RSTD_ULPS u (relative) of float64 of the kernel's own P.
  y        per element within y_bound() of float64 evaluated with the kernel's own P and statistics: the rounding of the scale / offset
           products and of the fma (EPI 2: IEEE operations only), plus the __expf / __fdividef error of fast_sigmoid (EPI 1 / 5).
           The fallback's y lies within FALLBACK_Y_L2 (per-sample relative L2) of the fused y.
  planes   bitwise f16f8_ref.quant_planes / split_bf16 of the kernel's own y; the y = NULL and inference forms give the training
           form's bits.
  dY       (EPI 4 dx) lattice: bitwise the exact data gradient (+ dx0).   dense: bitwise the fallback's plain data gradient.
  dP       the planes' value (hi + lo) per sample within DP_L2 relative L2 and, per (sample, channel), within DP_MAX of the column's
           largest term, of float64 from the kernel's dY, bp and stats; the affine gradients within AFFINE_L2.
A failure names the sample, position, channel, 128-row tile and column tile of the first wrong values.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import f16f8_ref as Q
import fused_ref as F

pytestmark = pytest.mark.gpu

BF16X3, BF16, F16F8 = 1, 2, 3
NPL = {BF16: 1, BF16X3: 2, F16F8: 3}
PNAME = {BF16X3: "bf16x3", BF16: "bf16", F16F8: "f16f8"}
U = 2.0 ** -24
SENTINEL = 0x55

# bounds (see the module docstring).  Measured worst values on one H100 80GB HBM3 at 700 W (also in DESIGN.md section 10): mean 3.0 u,
# rstd 3.0 u (fallback about 19 u), y 0.29 / 0.97 / 0.28 of y_bound for EPI 1 / 2 / 5, fused vs fallback y 2.2e-5, dP 2.5e-6 relative
# L2 and 7.8e-6 of the column, affine gradients 1.7e-7
MEAN_ULPS = 16           # dense mean: |mean - float64| <= MEAN_ULPS * u * mean|P| (tree depth of the column sums + the 1/R product)
RSTD_ULPS = 16           # |rstd / float64 - 1| <= RSTD_ULPS * u
RSTD_ULPS_FALLBACK = 64  # the same for the separate statistics kernel of the fallback, which rounds its variance differently
FALLBACK_Y_L2 = 1e-4     # per-sample relative L2 between the fused and the fallback y: their means round differently, and in a
                         # sample whose spread is near epsilon that rounding (u |mean|) is a sizeable fraction of the spread
DP_L2 = 2e-5             # per-sample relative L2 of the dP planes' value
DP_MAX = 1e-4            # per (sample, channel): max |dP - float64| / max of the column's |terms|
AFFINE_L2 = 2e-5         # dbeta / dgamma relative L2

# (B, R): 128-row tiles of whole samples at R = 32, 64, 128, and tails (M % 128 != 0) at R = 32 and 64
SHAPES = [(8, 32), (4, 64), (3, 128), (5, 32), (3, 64)]
WALK = ("res_h1", 270, 32)      # 68 row tiles x 8 column tiles = 544 tiles: four waves of a 132-SM persistent grid
FWD_CASES = [(layer, B, R) for layer in F.LAYERS for B, R in SHAPES] + [WALK]
BWD_CASES = [(pair, B, R, acc) for pair in F.BWD_PAIRS for B, R in SHAPES for acc in (0, 1)]


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def lattice_cases():
    """(layer, B, R, seed) of every forward lattice case"""
    return [(layer, B, R, _seed("fwd", layer, B, R)) for layer, B, R in FWD_CASES]


def lattice_bwd_cases():
    return [(pair, B, R, _seed("bwd", pair, B, R, acc), acc) for pair, B, R, acc in BWD_CASES]


def tail(B, R):
    return (B * R) % 128 != 0


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


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _planes(prec, n):
    if prec == F16F8:
        hi = torch.empty(n, dtype=torch.float16, device="cuda"); lo = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    else:
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda"); lo = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    hi.view(torch.uint8).fill_(SENTINEL); lo.view(torch.uint8).fill_(SENTINEL)
    return hi, lo


def _plane_values(prec, hi, lo):
    """decoded planes in float64: F16F8 (q16, q8hi, q8lo), bf16 (hi, lo)"""
    if prec == F16F8:
        n = hi.numel(); b = lo.cpu().numpy()
        return hi.cpu().numpy().astype(np.float64), Q.e4m3_decode(b[:n]), Q.e4m3_decode(b[n:])
    d = lambda t: Q.bf16_decode(t.view(torch.int16).cpu().numpy().view(np.uint16)).astype(np.float64)
    return d(hi), d(lo)


def _ref_planes(prec, y):
    y = np.ascontiguousarray(y, np.float32).reshape(-1)
    if prec == F16F8:
        q16, h8, l8 = Q.quant_planes(y)
        return q16.astype(np.float64), Q.e4m3_decode(h8), Q.e4m3_decode(l8)
    bh, bl = Q.split_bf16(y)
    return Q.bf16_decode(bh).astype(np.float64), Q.bf16_decode(bl).astype(np.float64)


# ---- where a wrong value sits ----------------------------------------------------------------------------------------------------
def _col_tile(epi, ch):
    """the 256-wide column tile holding normalised channel ch: 128 a + 128 g channels (EPI 1), 256 channels (EPI 2, 3, 4),
    64 post-shuffle channels x (a, a + C, g, g + C) (EPI 5)"""
    return ch // {1: 128, 2: 256, 3: 256, 4: 256, 5: 64}[epi]


def _where_fwd(layer, R, kind, flat):
    Cin, kw, Cout, sw, gated, sh, epi = F.LAYERS[layer]
    Cn = Cout // sh
    if kind == "p":
        nt = Cout * (2 if gated else 1)
        m, col = divmod(flat, nt)
        b, r = divmod(m, R)
        br, ch = divmod(col, Cout)
        s, c = divmod(ch, Cn)
        pos = r * sh + s
        return "sample %d, position %d, %s channel %d (P row %d, column %d): 128-row tile %d, column tile %d" % (
            b, pos, "gate" if br else "a", c, m, col, m // 128, _col_tile(epi, c))
    if kind == "stats":
        b, rem = divmod(flat, 4 * Cn)
        k, c = divmod(rem, Cn)
        return "sample %d, %s, channel %d: 128-row tiles %d..%d, column tile %d" % (
            b, ("mean_a", "rstd_a", "mean_g", "rstd_g")[k], c, b * R // 128, (b * R + R - 1) // 128, _col_tile(epi, c))
    b, rem = divmod(flat, R * sh * Cn)
    pos, c = divmod(rem, Cn)
    m = b * R + pos // sh
    return "sample %d, position %d, channel %d (conv row %d): 128-row tile %d, column tile %d" % (b, pos, c, m, m // 128, _col_tile(epi, c))


def _where_bwd(R, Cn, ld, epi, flat):
    m, col = divmod(flat, ld)
    b, r = divmod(m, R)
    br, c = divmod(col, Cn)
    return "sample %d, position %d, %s channel %d: 128-row tile %d, column tile %d" % (b, r, "gate" if br else "a", c, m // 128, _col_tile(epi, c))


def _report(bad, got, ref, where, what):
    idx = np.flatnonzero(bad.reshape(-1))
    if idx.size:
        g = np.asarray(got, np.float64).reshape(-1); r = np.asarray(ref, np.float64).reshape(-1)
        lines = ["  %s: got %r, reference %r" % (where(int(i)), g[i], r[i]) for i in idx[:8]]
        raise AssertionError("%s: %d of %d values wrong; first:\n%s" % (what, idx.size, bad.size, "\n".join(lines)))


def _assert_bits(got, ref, where, what):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    _report(~Q.same_values(got, ref), got, ref, where, what)


def _t64(t):
    return t.double().cpu().numpy()


# ---- forward ---------------------------------------------------------------------------------------------------------------------
def _fwd(eng, prec, layer, B, R, ops, form="train", fuse=1):
    """cgvc_conv_in_forward; form: train (p, stats, y), noy (y NULL), infer (p = stats = NULL)"""
    lib, h, N = eng
    Cin, kw, Cout, sw, gated, sh, _ = F.LAYERS[layer]
    x, wa, wg, ba, bg, par, resid = ops
    Cn = Cout // sh
    p = None if form == "infer" else _nan(B, R, Cout * (2 if gated else 1))
    stats = None if form == "infer" else _nan(B, 4, Cn)
    y = None if form == "noy" else _nan(B, R * sh, Cn)
    hi, lo = _planes(prec, B * R * sh * Cn)
    fused = C.c_int(-1)
    N.check(h, lib.cgvc_conv_in_forward(h, prec, _p(x), _p(wa), _p(wg), _p(ba), _p(bg), _p(par[0]), _p(par[1]), _p(par[2]), _p(par[3]),
                                        _p(resid), _p(p), _p(stats), _p(y), _p(hi), _p(lo), B, R * sw, Cin, kw, Cout, sw, sh, fuse,
                                        C.byref(fused), None))
    torch.cuda.synchronize()
    return {"p": p, "stats": stats, "y": y, "hi": hi, "lo": lo, "fused": fused.value}


def _check_stats(layer, R, prec, got, P, exact_mean, what, rstd_ulps=RSTD_ULPS):
    """the kernel's statistics against float64 of its own P; returns (worst mean error in u * mean|P|, worst rstd error in u)"""
    _, _, Cout, _, gated, sh, epi = F.LAYERS[layer]
    a, g = F.branches(P, gated, sh)
    st = got.double()
    where = lambda i: _where_fwd(layer, R, "stats", i)
    worst_m, worst_r = 0.0, 0.0
    for k, v in ((0, a), (2, g)):
        if v is None:
            continue
        m64, r64 = F.stats_of(v)
        mk, rk = st[:, k], st[:, k + 1]
        full = lambda t, kk: torch.zeros_like(st).index_copy_(1, torch.tensor([kk], device=st.device), t[:, None]).cpu().numpy()
        if exact_mean:
            bad = np.zeros(st.shape, bool); bad[:, k] = (mk != m64).cpu().numpy()
            _report(bad, _t64(st), full(m64, k), where, what + ": mean not bitwise float64")
        scale = v.abs().mean(dim=1) + 1e-300
        em = ((mk - m64).abs() / (U * scale))
        bad = np.zeros(st.shape, bool); bad[:, k] = (em > MEAN_ULPS).cpu().numpy()
        _report(bad, _t64(st), full(m64, k), where, what + ": mean beyond %d u mean|P|" % MEAN_ULPS)
        er = ((rk / r64 - 1).abs() / U)
        bad = np.zeros(st.shape, bool); bad[:, k + 1] = (er > rstd_ulps).cpu().numpy()
        _report(bad, _t64(st), full(r64, k + 1), where, what + ": rstd beyond %d u" % rstd_ulps)
        worst_m, worst_r = max(worst_m, float(em.max())), max(worst_r, float(er.max()))
    return worst_m, worst_r


def _check_y(layer, R, prec, out, P, par, resid, what):
    """y per element against float64 from the kernel's own P and statistics, and the planes bitwise against the quantisation of y;
    returns the worst error / bound"""
    _, _, Cout, _, gated, sh, _ = F.LAYERS[layer]
    st = out["stats"].double()
    ref, _ = F.forward(P, par, gated, sh, resid=resid, stats=st)
    bound = F.y_bound(P, st, par, gated, sh, resid)
    y = out["y"].double()
    err = (y - ref).abs()
    where = lambda i: _where_fwd(layer, R, "y", i)
    _report((~(err <= bound)).cpu().numpy(), _t64(y), _t64(ref), where, what + ": y beyond its rounding bound")
    yn = out["y"].cpu().numpy()
    for k, (g, r) in enumerate(zip(_plane_values(prec, out["hi"], out["lo"]), _ref_planes(prec, yn))):
        _assert_bits(g, r, where, "%s: plane %d not the quantisation of y" % (what, k))
    return float((err / bound).max())


def _fwd_ops(layer, B, R, tier):
    seed = _seed("fwd", layer, B, R)
    ops = (F.lattice_forward_case if tier == "lattice" else F.dense_forward_case)(layer, B, R, seed)
    x, wa, wg, ba, bg, par, resid = ops
    return ops, (_dev(x), _dev(wa), _dev(wg), _dev(ba), _dev(bg), tuple(_dev(t) for t in par), _dev(resid))


FWD_PARAMS = [(c, p, t) for c in FWD_CASES for p in (BF16X3, BF16, F16F8) for t in ("lattice", "dense")]


@pytest.mark.parametrize("case,prec,tier", FWD_PARAMS,
                         ids=["%s-B%dR%d-%s-%s" % (c + (PNAME[p], t)) for c, p, t in FWD_PARAMS])
def test_forward(eng, case, prec, tier):
    layer, B, R = case
    Cin, kw, Cout, sw, gated, sh, epi = F.LAYERS[layer]
    ops, dops = _fwd_ops(layer, B, R, tier)
    x, wa, wg, ba, bg, par, resid = ops
    what = "%s B%d R%d %s %s" % (layer, B, R, PNAME[prec], tier)
    tr = _fwd(eng, prec, layer, B, R, dops)
    assert tr["fused"] == 1, what + ": the fused epilogue did not run"
    P = tr["p"].double()
    fb = _fwd(eng, prec, layer, B, R, dops, fuse=0)
    assert fb["fused"] == 0
    wp = lambda i: _where_fwd(layer, R, "p", i)
    if tier == "lattice":
        largest, colsum = F.certificate(x, wa, wg, ba, bg, sw, device="cuda")
        assert largest < 2 ** 24 and colsum < 2 ** 24, (what, largest, colsum)
        exact = F.conv_p(x, wa, wg, ba, bg, sw, device="cuda")
        _assert_bits(_t64(P), _t64(exact), wp, what + ": P not the exact convolution")
    _assert_bits(_t64(fb["p"]), _t64(P), wp, what + ": P differs from the fallback's plain-epilogue P")
    wm, wr = _check_stats(layer, R, prec, tr["stats"], P, tier == "lattice", what)
    wy = _check_y(layer, R, prec, tr, P, par, resid, what)
    # the fallback against float64 of its own P and statistics, and its y against the fused y
    _check_stats(layer, R, prec, fb["stats"], fb["p"].double(), tier == "lattice", what + " (fallback)", RSTD_ULPS_FALLBACK)
    wyf = _check_y(layer, R, prec, fb, fb["p"].double(), par, resid, what + " (fallback)")
    yd = (fb["y"] - tr["y"]).double().reshape(B, -1)
    gap = float((yd.norm(dim=1) / tr["y"].double().reshape(B, -1).norm(dim=1).clamp_min(1e-300)).max())
    assert gap <= FALLBACK_Y_L2, (what, "fused y vs the fallback's", gap)
    # the y = NULL and inference forms write the training form's bits; a second call repeats them
    noy = _fwd(eng, prec, layer, B, R, dops, form="noy")
    inf = _fwd(eng, prec, layer, B, R, dops, form="infer")
    again = _fwd(eng, prec, layer, B, R, dops)
    assert noy["fused"] == 1 and inf["fused"] == 1
    wy_ = lambda i: _where_fwd(layer, R, "y", i)
    for name, o in (("y = NULL", noy), ("inference", inf), ("repeat", again)):
        for k, (g, r) in enumerate(zip(_plane_values(prec, o["hi"], o["lo"]), _plane_values(prec, tr["hi"], tr["lo"]))):
            _assert_bits(g, r, wy_, "%s %s: plane %d" % (what, name, k))
        if o["y"] is not None:
            _assert_bits(_t64(o["y"]), _t64(tr["y"]), wy_, "%s %s: y" % (what, name))
        if o["p"] is not None:
            _assert_bits(_t64(o["p"]), _t64(tr["p"]), wp, "%s %s: P" % (what, name))
            _assert_bits(_t64(o["stats"]), _t64(tr["stats"]), lambda i: _where_fwd(layer, R, "stats", i), "%s %s: stats" % (what, name))
    print("MEAS fwd %s EPI%d NPL%d mean_u=%.3g rstd_u=%.3g y_ratio=%.3g y_ratio_fallback=%.3g fallback_y_l2=%.3g"
          % (what.replace(" ", "|"), epi, NPL[prec], wm, wr, wy, wyf, gap))


REFUSED = [("res_h1", 8, 16), ("res_h2", 8, 16), ("u1", 8, 16), ("res_h1", 2, 256), ("res_h2", 2, 256), ("u2", 2, 256), ("d1", 2, 256)]


@pytest.mark.parametrize("prec", [BF16X3, F16F8], ids=["bf16x3", "f16f8"])
@pytest.mark.parametrize("case", REFUSED, ids=["%s-B%dR%d" % c for c in REFUSED])
def test_forward_refusals_match_the_fallback(eng, case, prec):
    """R = 16 (half a warp per sample) and R = 256 (more than a tile) are refused: fused = 0, and every output equals the fallback's,
    in the training and the inference form (which then needs a temporary P)"""
    layer, B, R = case
    _, dops = _fwd_ops(layer, B, R, "dense")
    fb = _fwd(eng, prec, layer, B, R, dops, fuse=0)
    for form in ("train", "infer"):
        o = _fwd(eng, prec, layer, B, R, dops, form=form)
        assert o["fused"] == 0, (case, form)
        for k in ("p", "stats", "y"):
            if o[k] is not None:
                assert torch.equal(torch.nan_to_num(o[k], 7.0), torch.nan_to_num(fb[k], 7.0)), (case, form, k)
        assert torch.equal(o["hi"].view(torch.uint8), fb["hi"].view(torch.uint8)) and torch.equal(o["lo"].view(torch.uint8), fb["lo"].view(torch.uint8))


WINDOW = [("res_h1", 4, 64), ("res_h2", 4, 64), ("u1", 4, 64)]


@pytest.mark.parametrize("case", WINDOW, ids=["%s-B%dR%d" % c for c in WINDOW])
def test_f16f8_planes_at_the_window_edges(eng, case):
    """f16f8 with beta_a per channel from the edge table and a small gamma_a (as test_in_glu_planes_exact): y sits at the planes'
    window edges, and the fused planes clamp exactly as the reference.  The fused epilogues do not count saturation; the reference count
    of saturated groups is printed as a measurement only."""
    layer, B, R = case
    _, _, Cout, _, gated, sh, _ = F.LAYERS[layer]
    ops, _ = _fwd_ops(layer, B, R, "dense")
    x, wa, wg, ba, bg, par, resid = ops
    rng = np.random.default_rng(_seed("window", layer))
    Cn = Cout // sh
    edge = Q.edge_values(); edge = edge[np.isfinite(edge)]
    beta_a = np.resize(edge[rng.permutation(edge.size)], Cn).astype(np.float32)
    gamma_a = np.exp2(-rng.integers(4, 30, Cn)).astype(np.float32)
    par = (beta_a, gamma_a) + par[2:]
    ops = (x, wa, wg, ba, bg, par, resid)
    dops = (_dev(x), _dev(wa), _dev(wg), _dev(ba), _dev(bg), tuple(_dev(t) for t in par), _dev(resid))
    for fuse in (1, 0):
        o = _fwd(eng, F16F8, layer, B, R, dops, fuse=fuse)
        assert o["fused"] == fuse
        _check_y(layer, R, F16F8, o, o["p"].double(), par, resid, "%s window fuse=%d" % (layer, fuse))
        print("MEAS window %s fuse=%d reference saturated groups %d of %d" % (layer, fuse, Q.sat_count(o["y"].cpu().numpy()), o["y"].numel() // 4))


# ---- backward --------------------------------------------------------------------------------------------------------------------
def _bwd(eng, prec, pair, B, R, dd, acc, fuse=1, gate=None, up=None):
    """cgvc_conv_in_backward; dd = device (dP, wa, wg, dx0); up = device (bp, stats, par) of the upstream layer"""
    lib, h, N = eng
    down, upl, epi = F.BWD_PAIRS[pair]
    Cin, kw, Cout, _, _, _, _ = F.LAYERS[down]
    gate = (epi == 3) if gate is None else gate
    dP, wa, wg, dx0 = dd
    bp, stats, par = up
    ld = Cin * (2 if gate else 1)
    if gate:
        dx = None if dx0 is None else dx0.clone()
    else:
        dx = dx0.clone() if acc else _nan(B, R, Cin)
    hi, lo = _planes(prec, B * R * ld)
    grads = [torch.zeros(Cin, device="cuda") for _ in range(4 if gate else 2)] + ([] if gate else [None, None])
    fused = C.c_int(-1)
    N.check(h, lib.cgvc_conv_in_backward(h, prec, _p(dP), _p(wa), _p(wg), _p(bp), _p(stats), _p(par[0]), _p(par[1]), _p(par[2]), _p(par[3]),
                                         _p(dx), _p(hi), _p(lo), _p(grads[0]), _p(grads[1]), _p(grads[2]), _p(grads[3]),
                                         B, R, Cin, kw, Cout, int(gate), acc, fuse, C.byref(fused), None))
    torch.cuda.synchronize()
    if gate and dx0 is not None:
        assert torch.equal(dx, dx0), (pair, "the gated form wrote dx")
    return {"dx": dx, "hi": hi, "lo": lo, "grads": grads, "fused": fused.value}


def _bwd_ops(pair, B, R, acc, tier):
    down, upl, epi = F.BWD_PAIRS[pair]
    seed = _seed("bwd", pair, B, R, acc)
    dP, wa, wg, dx0 = (F.lattice_dgrad_case if tier == "lattice" else F.dense_dgrad_case)(down, B, R, seed, acc)
    bp, stats, par = F.upstream_case(upl, B, R, seed + 1)
    return (dP, wa, wg, dx0), (bp, stats, par), (_dev(dP), _dev(wa), _dev(wg), _dev(dx0)), (_dev(bp), _dev(stats), tuple(_dev(t) for t in par))


def _dp_value(prec, o):
    hi, lo = _plane_values(prec, o["hi"], o["lo"])
    return hi + lo


def _check_dp(pair, B, R, prec, o, dY, bp, stats, par, what):
    """dP planes and affine gradients against float64 from dY, bp and stats; returns (worst per-sample L2, worst per-column max ratio,
    worst affine L2)"""
    down, upl, epi = F.BWD_PAIRS[pair]
    Cn = F.LAYERS[down][0]
    gated = epi == 3
    ref, gref = F.backward(bp, par, dY.cpu(), gated, stats=stats)
    ref = ref.numpy()
    ld = ref.shape[-1]
    got = _dp_value(prec, o).reshape(B, R, ld)
    where = lambda i: _where_bwd(R, Cn, ld, epi, i)
    l2 = np.array([np.linalg.norm(got[b] - ref[b]) / max(np.linalg.norm(ref[b]), 1e-300) for b in range(B)])
    if (l2 > DP_L2).any():
        b = int(np.argmax(l2))
        _report(np.abs(got - ref) > DP_L2 * np.abs(ref).max(), got, ref, where, "%s: dP sample %d relative L2 %.3g" % (what, b, l2[b]))
    # per (sample, channel): relative to the largest term of the column, gamma rstd |dn| (+ the mean terms)
    scale = np.abs(ref).max(axis=1, keepdims=True) + 1e-300
    ratio = np.abs(got - ref) / scale
    _report(ratio > DP_MAX, got, ref, where, "%s: dP beyond %g of its column" % (what, DP_MAX))
    worst_aff = 0.0
    for k, (g, r) in enumerate(zip(o["grads"], gref)):
        if r is None:
            continue
        e = float(np.linalg.norm(g.double().cpu().numpy() - r.numpy()) / np.linalg.norm(r.numpy()))
        assert e <= AFFINE_L2, (what, ("dbeta_a", "dgamma_a", "dbeta_g", "dgamma_g")[k], e)
        worst_aff = max(worst_aff, e)
    return float(l2.max()), float(ratio.max()), worst_aff


BWD_PARAMS = [(c, p, t) for c in BWD_CASES for p in (BF16X3, BF16) for t in ("lattice", "dense")]


@pytest.mark.parametrize("case,prec,tier", BWD_PARAMS,
                         ids=["%s-B%dR%d-acc%d-%s-%s" % (c + (PNAME[p], t)) for c, p, t in BWD_PARAMS])
def test_backward(eng, case, prec, tier):
    pair, B, R, acc = case
    down, upl, epi = F.BWD_PAIRS[pair]
    Cin = F.LAYERS[down][0]
    (dP, wa, wg, dx0), (bp, stats, par), dd, up = _bwd_ops(pair, B, R, acc, tier)
    what = "%s B%d R%d acc%d %s %s" % (pair, B, R, acc, PNAME[prec], tier)
    o = _bwd(eng, prec, pair, B, R, dd, acc, up=up)
    assert o["fused"] == 1, what + ": the fused epilogue did not run"
    fb = _bwd(eng, prec, pair, B, R, dd, acc, fuse=0, up=up)
    assert fb["fused"] == 0
    wdx = lambda i: _where_bwd(R, Cin, Cin, epi, i)
    # dY: the kernel's own (the residual form writes it to dx); the gated form's is the plain data gradient, read through a residual call
    if epi == 4:
        dY = o["dx"]
        _assert_bits(_t64(dY), _t64(fb["dx"]), wdx, what + ": dY differs from the fallback's plain data gradient")
    else:
        zb = torch.zeros(B, R, Cin, device="cuda"); zs = torch.zeros(B, 4, Cin, device="cuda"); zc = torch.zeros(Cin, device="cuda")
        dY = _bwd(eng, prec, pair, B, R, dd, acc, fuse=0, gate=False, up=(zb, zs, (zc, zc + 1, None, None)))["dx"]
    if tier == "lattice":
        exact = F.dgrad(dP, wa, wg, device="cuda")
        if dx0 is not None:
            exact = exact + torch.from_numpy(dx0).double().cuda()
        _assert_bits(_t64(dY), _t64(exact), wdx, what + ": dY not the exact data gradient")
    l2, mx, aff = _check_dp(pair, B, R, prec, o, dY, bp, stats, par, what)
    l2f, mxf, afff = _check_dp(pair, B, R, prec, fb, dY, bp, stats, par, what + " (fallback)")
    a, b = _dp_value(prec, o).reshape(B, -1), _dp_value(prec, fb).reshape(B, -1)
    gap = float(max(np.linalg.norm(a[i] - b[i]) / np.linalg.norm(b[i]) for i in range(B)))
    assert gap <= 2 * DP_L2, (what, "fused dP vs the fallback's", gap)
    print("MEAS bwd %s EPI%d NPL%d dp_l2=%.3g dp_max=%.3g affine_l2=%.3g fallback_dp_l2=%.3g fallback_affine_l2=%.3g fused_vs_fallback=%.3g"
          % (what.replace(" ", "|"), epi, NPL[prec], l2, mx, aff, l2f, afff, gap))


@pytest.mark.parametrize("pair", list(F.BWD_PAIRS))
def test_f16f8_backward_is_not_fused(eng, pair):
    """there is no F16F8 fused backward: fuse = 1 reports fused = 0 and writes the fallback's planes"""
    B, R, acc = 4, 64, 1
    _, (bp, stats, par), dd, up = _bwd_ops(pair, B, R, acc, "dense")
    o = _bwd(eng, F16F8, pair, B, R, dd, acc, up=up)
    fb = _bwd(eng, F16F8, pair, B, R, dd, acc, fuse=0, up=up)
    assert o["fused"] == 0 and fb["fused"] == 0
    assert torch.equal(o["hi"].view(torch.uint8), fb["hi"].view(torch.uint8)) and torch.equal(o["lo"].view(torch.uint8), fb["lo"].view(torch.uint8))
    if o["dx"] is not None and F.BWD_PAIRS[pair][2] == 4:
        assert torch.equal(o["dx"], fb["dx"])


# ---- coverage --------------------------------------------------------------------------------------------------------------------
def test_case_tables_reach_every_fused_instantiation():
    """every fused branch of launch_nt -- EPI 1 / 2 / 5 x NPL 1 / 2 / 3 and EPI 3 / 4 x NPL 1 / 2 -- at R = 32, 64 and 128, and with
    a tail tile at R = 32 and 64 (R = 128 fills whole tiles); plus a multi-wave persistent walk"""
    reached = {}
    for (layer, B, R), prec, tier in FWD_PARAMS:
        reached.setdefault((F.LAYERS[layer][6], NPL[prec]), set()).add((R, tail(B, R)))
    for (pair, B, R, acc), prec, tier in BWD_PARAMS:
        reached.setdefault((F.BWD_PAIRS[pair][2], NPL[prec]), set()).add((R, tail(B, R)))
    want = {(32, False), (64, False), (128, False), (32, True), (64, True)}
    inst = [(e, n) for e in (1, 2, 5) for n in (1, 2, 3)] + [(e, n) for e in (3, 4) for n in (1, 2)]
    print("coverage (EPI, NPL): (R, tail) reached")
    for k in inst:
        print("  EPI %d NPL %d: %s" % (k + (sorted(reached.get(k, ())),)))
        assert want <= reached.get(k, set()), (k, sorted(want - reached.get(k, set())))
    Cin, kw, Cout, sw, gated, sh, epi = F.LAYERS[WALK[0]]
    tiles = -(-WALK[1] * WALK[2] // 128) * (2 * Cout // 256)
    assert tiles >= 4 * 132, tiles
