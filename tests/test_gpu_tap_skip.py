"""Per-tile tap ranges of the forward / data-gradient gather-GEMM (tc_gemm.cu nt_tile_taps): a 128-row tile contracts only over the
taps that some of its output rows read inside the tensor; a tap that lies in the padding for the whole tile is skipped.

A. The rule, mirrored here on the CPU: rows are walked output row y outermost (m = (y * B + b) * Wx + x), and tap t is kept for a
   tile whose rows cover output rows y_lo .. y_hi if some y in that range has 0 <= y * sy + oy[t] < Hs.  At batch 256 it keeps the
   fractions of the discriminator's launches that DESIGN.md section 5 lists.
B. Lattice inputs (tests/gemm_ref.py) on the discriminator's 2-D layers at batches whose tiles hold one output row and at batches whose
   tiles straddle output rows (with an M tail and odd extents): forward and data gradient equal the emulation bit for bit.
C. What each tile actually skips: one kernel row of weights set to NaN reaches exactly the tiles whose kept taps include that row;
   every other output is finite and equal to the emulation with that row zeroed.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

import gemm_ref as G
from oracle.cyclegan_oracle import same_pad
from test_gpu_kernels import CONV_CASES

# ------------------------------------------------------------------------------------------------ the rule (CPU mirror)
MODEL = {c[0]: c for c in CONV_CASES}


def with_batch(name, B, H=None, W=None):
    c = MODEL[name]
    return ("%s.b%d%s" % (name, B, "" if H is None else ".%dx%d" % (H, W)), B, H or c[2], W or c[3]) + c[4:]


def nt_geoms(case, form):
    """geom.h fwd_geom / dgrad_geoms: the NT launches of one form, each with its rows (B, Hy, Wx), source height Hs, row stride sy,
    and per tap its row offset oy and kernel row ky; data-gradient classes also carry their parity (py, px)"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    ph, _ = same_pad(H, kh, sh)
    pw, _ = same_pad(W, kw, sw)
    Ho, Wo = -(-H // sh), -(-W // sw)
    if form == "fwd":
        taps = [(i, j) for i in range(kh) for j in range(kw)]
        return [{"B": B, "Hy": Ho, "Wx": Wo, "Hs": H, "sy": sh, "oy": [i - ph for i, _ in taps], "ky": [i for i, _ in taps]}]
    out = []
    for py in range(sh):
        for px in range(sw):
            hy, wx = -(-(H - py) // sh), -(-(W - px) // sw)
            if hy <= 0 or wx <= 0:
                continue
            taps = [(i, j) for i in range(kh) for j in range(kw) if (py + ph - i) % sh == 0 and (px + pw - j) % sw == 0]
            out.append({"B": B, "Hy": hy, "Wx": wx, "Hs": Ho, "sy": 1, "oy": [(py + ph - i) // sh for i, _ in taps],
                        "ky": [i for i, _ in taps], "py": py, "px": px})
    return out


def kept(g, y_lo, y_hi):
    """per tap: whether rows of output rows y_lo .. y_hi read it inside the source (its valid y interval meets the range)"""
    res = []
    for oy in g["oy"]:
        lo = -(oy // g["sy"])                         # ceil(-oy / sy): the first y whose source row is >= 0
        hi = (g["Hs"] - 1 - oy) // g["sy"]            # the last y whose source row is < Hs
        res.append(max(lo, y_lo) <= min(hi, y_hi))
    return res


def tile_taps(g):
    """kept taps of every 128-row tile, rows in the order m = (y * B + b) * Wx + x"""
    bw = g["B"] * g["Wx"]
    M = bw * g["Hy"]
    return [kept(g, m0 // bw, min(m0 + 127, M - 1) // bw) for m0 in range(0, M, 128)]


def kept_fraction(g):
    tt = tile_taps(g)
    return Fraction(sum(sum(k) for k in tt), len(tt) * len(g["oy"]))


def test_kept_fractions_at_batch_256():
    frac = {}
    for name in ("D.d1", "D.d2", "D.d3"):
        case = with_batch(name, 256)
        frac[name + " fwd"] = kept_fraction(nt_geoms(case, "fwd")[0])
        for g in nt_geoms(case, "dgrad"):
            frac["%s dgrad (%d, %d)" % (name, g["py"], g["px"])] = kept_fraction(g)
    print({k: str(v) for k, v in frac.items()})
    want = {"D.d3 fwd": Fraction(27, 36), "D.d3 dgrad (0, 0)": Fraction(27, 36), "D.d3 dgrad (0, 1)": Fraction(27, 36),
            "D.d2 fwd": Fraction(17, 18), "D.d1 fwd": Fraction(35, 36)}
    for px in (0, 1):
        want["D.d2 dgrad (0, %d)" % px] = Fraction(11, 12)
        want["D.d2 dgrad (1, %d)" % px] = Fraction(1)
        want["D.d1 dgrad (0, %d)" % px] = Fraction(23, 24)
        want["D.d1 dgrad (1, %d)" % px] = Fraction(1)
    assert frac == want


def test_every_tile_keeps_a_tap():
    """TF-SAME: every output row reads its source somewhere, so no tile has an empty contraction"""
    for name in ("D.d1", "D.d2", "D.d3"):
        for B in (1, 3, 37, 256):
            for form in ("fwd", "dgrad"):
                for g in nt_geoms(with_batch(name, B), form):
                    assert all(any(k) for k in tile_taps(g)), (name, B, form, g)


def test_one_dimensional_layers_keep_every_tap():
    """Hy == 1 (the generator): nothing is skipped"""
    for c in CONV_CASES:
        if c[2] == 1:
            for form in ("fwd", "dgrad"):
                for g in nt_geoms(c, form):
                    assert all(all(k) for k in tile_taps(g)), (c[0], form)


# ------------------------------------------------------------------------------------------------ the kernels (GPU)
# tiles of one output row: B * Wx a multiple of 128; straddling tiles: B * Wx not a multiple of 128, with an M tail; odd extents give
# stride-2 data-gradient classes of unequal rows and taps
ONE_ROW = [with_batch("D.d1", 8), with_batch("D.d2", 8), with_batch("D.d3", 64)]
STRADDLE = [with_batch("D.d1", 3, 25, 65), with_batch("D.d2", 3), with_batch("D.d2", 6, 13, 33), with_batch("D.d3", 37),
            with_batch("D.d3", 5, 7, 17)]
PRECS = (G.BF16X3, G.BF16, G.F16F8)
PNAME = {G.BF16X3: "bf16x3", G.BF16: "bf16", G.F16F8: "f16f8"}


def test_case_list_reaches_skipping_tiles():
    for cases, straddle in ((ONE_ROW, False), (STRADDLE, True)):
        for c in cases:
            bw = [g["B"] * g["Wx"] for g in nt_geoms(c, "fwd") + nt_geoms(c, "dgrad")]
            assert all((v % 128 != 0) == straddle for v in bw), (c[0], bw)
            assert min(kept_fraction(g) for g in nt_geoms(c, "fwd") + nt_geoms(c, "dgrad")) < 1, c[0]
    tails = [c[0] for c in STRADDLE if any(g["B"] * g["Wx"] * g["Hy"] % 128 for g in nt_geoms(c, "fwd") + nt_geoms(c, "dgrad"))]
    odd = [c[0] for c in STRADDLE if c[2] % 2 or c[3] % 2]
    assert tails and odd


def _gpu():
    from test_gpu_gemm_exact import _call, _assert_exact
    return _call, _assert_exact


@pytest.fixture(scope="module")
def eng():
    import ctypes as C
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    yield lib, h, N
    lib.cgvc_destroy(h)


LATTICE = [(c, p) for c in ONE_ROW + STRADDLE for p in PRECS]


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec", LATTICE, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in LATTICE])
def test_lattice_bit_exact(eng, case, prec):
    _call, _assert_exact = _gpu()
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    for form, phase, largest, bound in G.certificate(case, prec, x, w, b, dy, device="cuda", P=P, forms=("fwd", "dgrad")):
        assert largest < bound, (case[0], prec, form, phase, largest, bound)
    ref = G.emulate(case, prec, x, w, b, dy, device="cuda", P=P, forms=("fwd", "dgrad"))
    got = _call(eng, case, prec, x, w, b, dy, 0, launches=True)
    for key in ("y", "dx"):
        _assert_exact(case, prec, key, got[key], ref[key])


def nan_rows(case, form, ky):
    """boolean [B, Ho, Wo] (fwd) or [B, H, W] (dgrad): the outputs whose tile keeps a tap of kernel row ky"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    if form == "fwd":
        out = np.zeros((B, -(-H // sh), -(-W // sw)), bool)
    else:
        out = np.zeros((B, H, W), bool)
    for g in nt_geoms(case, form):
        hot = np.array([any(k and r == ky for k, r in zip(kt, g["ky"])) for kt in tile_taps(g)])
        y, b, x = np.meshgrid(np.arange(g["Hy"]), np.arange(B), np.arange(g["Wx"]), indexing="ij")
        tile = ((y * B + b) * g["Wx"] + x) // 128
        if form == "fwd":
            out[b, y, x] = hot[tile]
        else:
            out[b, y * sh + g["py"], x * sw + g["px"]] = hot[tile]
    return out


PROBE = [(with_batch("D.d3", 37), p, r) for p in PRECS for r in (0, 5)] + \
        [(with_batch("D.d3", 5, 7, 17), G.F16F8, 5), (with_batch("D.d1", 3, 25, 65), G.F16F8, 2), (with_batch("D.d2", 8), G.BF16X3, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec,ky", PROBE, ids=["%s-%s-ky%d" % (c[0], PNAME[p], r) for c, p, r in PROBE])
def test_nan_kernel_row_reaches_only_tiles_that_keep_it(eng, case, prec, ky):
    _call, _assert_exact = _gpu()
    x, w, b, dy = G.lattice_case(case, prec)
    w0 = w.copy(); w0[ky] = 0.0
    wn = w.copy(); wn[ky] = np.nan
    ref = G.emulate(case, prec, x, w0, b, dy, device="cuda", forms=("fwd", "dgrad"))
    got = _call(eng, case, prec, x, wn, b, dy, 0)
    for key, form in (("y", "fwd"), ("dx", "dgrad")):
        hot = torch.as_tensor(nan_rows(case, form, ky), device="cuda")
        g, r = got[key].double(), ref[key]
        assert 0 < int(hot.sum()) < hot.numel(), (case[0], key, "the probe must split the outputs")
        nan_out = torch.isnan(g).all(-1)
        bad = torch.nonzero(nan_out != hot)
        assert bad.numel() == 0, (case[0], PNAME[prec], key, "NaN rows differ from the kept taps at", bad[:8].tolist())
        assert torch.equal(g[~hot], r[~hot]), (case[0], PNAME[prec], key, "finite rows differ from the emulation")
