"""CPU known-answer tests of tests/weight_planes_ref.py: the row orders, the folded and gated columns and the padding worked out by hand
from the layout comments, and the element values at the edges of the weight window with their codes worked out by hand (not through
f16f8_ref's encoder)."""
import numpy as np

import weight_planes_ref as W


def _params_for(L, fill):
    """a PARAM vector holding L's kernels and biases at the offsets the Layer names"""
    taps_cin_cout = L.taps * L.cin * L.cout
    n = max(L.ka, L.kg, L.ba, L.bg) + taps_cin_cout + L.cout
    p = np.zeros(n, np.float32)
    for b, (k, bb) in enumerate(((L.ka, L.ba), (L.kg, L.bg))[:2 if L.gated else 1]):
        p[k:k + taps_cin_cout] = fill(b, taps_cin_cout)
        p[bb:bb + L.cout] = 1000 * (b + 1) + np.arange(L.cout)
    return p


def _coded(L):
    """kernel element (tap, ci, co) of branch b = b * 2^13 + tap * 2^10 + ci * 2^5 + co: unique for taps < 8, cin, cout < 32, and exact
    as hi + lo"""
    def fill(b, n):
        t, ci, co = np.unravel_index(np.arange(n), (L.taps, L.cin, L.cout))
        return (b * 8192 + t * 1024 + ci * 32 + co).astype(np.float32)
    return fill


def test_perm2_tile_by_hand():
    """gated + pixel shuffle, cout = 256 (Ch = 128 post-shuffle channels): 256-row tiles [64 a(c) | 64 a(c + Ch) | 64 g(c) | 64 g(c + Ch)]"""
    L = W.Layer(kh=1, kw=1, cin=2, cout=256, gated=1, shuffle=2, ka=0, kg=600, ba=1200, bg=1500)
    assert L.perm() == 2 and L.dims()[0] == 512
    # rows worked out from the comment: (branch, co) -> row
    hand = {(0, 0): 0, (0, 63): 63, (0, 64): 256, (0, 127): 319, (0, 128): 64, (0, 191): 127, (0, 192): 320, (0, 255): 383,
            (1, 0): 128, (1, 63): 191, (1, 128): 192, (1, 200): 256 + 192 + 8, (1, 64): 256 + 128, (1, 255): 511}
    for (b, co), row in hand.items():
        assert W.perm_rows(2, 256, b)[co] == row, (b, co)
    rows = np.concatenate([W.perm_rows(2, 256, b) for b in (0, 1)])
    assert sorted(rows.tolist()) == list(range(512))             # a permutation of the 512 rows
    # the first tile element by element, from an explicit loop over its four 64-row quarters
    p = np.zeros(1800, np.float32)
    p[0:512] = np.arange(512) % 256 + 1                           # a: w[ci][co] = co + 1 (both ci)
    p[600:1112] = -(np.arange(512) % 256 + 1)                     # g: -(co + 1)
    p[1200:1456] = np.arange(256) + 0.5                           # bias_a
    p[1500:1756] = -(np.arange(256) + 0.5)                        # bias_g
    pl = W.bf16_planes(L, p)
    wf = W.Q.bf16_decode(pl["wf_hi"])
    bias = pl["bias"].view(np.float32)
    for quarter, (sign, s) in enumerate(((1, 0), (1, 1), (-1, 0), (-1, 1))):
        for c in range(64):
            co = s * 128 + c
            row = quarter * 64 + c
            assert wf[0, row, 0] == sign * (co + 1) and wf[0, row, 1] == sign * (co + 1), (row, co)
            assert bias[row] == sign * (co + 0.5)
    assert (wf[0, :, 2:] == 0).all()                              # cin_k = 64: columns 2 .. 63 are padding


def test_perm1_and_perm0_rows():
    assert W.perm_rows(1, 256, 0)[[0, 127, 128, 255]].tolist() == [0, 127, 256, 383]
    assert W.perm_rows(1, 256, 1)[[0, 127, 128, 255]].tolist() == [128, 255, 384, 511]
    assert W.perm_rows(0, 12, 1).tolist() == list(range(12, 24))
    assert W.Layer(kh=1, kw=3, cin=8, cout=12, gated=1).perm() == 0           # gated but cout % 128 != 0
    assert W.Layer(kh=1, kw=3, cin=8, cout=128, gated=1, shuffle=1).perm() == 1
    assert W.Layer(kh=1, kw=3, cin=8, cout=64, gated=1, shuffle=2).perm() == 0


def test_folded_column_by_hand():
    """o1's tap-folded form: a 1 x 1 layer with cout = fold * n columns, column co = t * n + n' of the TF kernel [1, fold, cin, n]"""
    fold, cin, n = 3, 4, 8
    L = W.Layer(kh=1, kw=1, cin=cin, cout=fold * n, gated=0, shuffle=1, fold=fold, ka=0, ba=200)
    assert L.ok() and L.q_ok() and L.perm() == 0
    p = np.zeros(300, np.float32)
    K = np.arange(fold * cin * n, dtype=np.float32).reshape(fold, cin, n) + 1         # TF kernel [fold][cin][n] at ka (h = 1 dropped)
    p[:K.size] = K.reshape(-1)
    p[200:200 + fold * n] = 7.0                                                        # a bias a folded layer must not pick up
    pl = W.bf16_planes(L, p)
    wd, wf = W.Q.bf16_decode(pl["wd_hi"]), W.Q.bf16_decode(pl["wf_hi"])
    co = 13                                                                            # t = 1, n' = 5
    for ci in range(cin):
        assert wd[0, ci, co] == K[1, ci, 5] and wf[0, co, ci] == K[1, ci, 5]
    assert wd[0, 2, 0] == K[0, 2, 0] and wd[0, 2, 23] == K[2, 2, 7]
    assert (pl["bias"] == 0).all()
    assert (wd[0, cin:, :] == 0).all() and (wd[0, :, fold * n:] == 0).all()           # cin_n = 128, nt_k = 64
    assert W.Layer(kh=1, kw=1, cin=4, cout=18, fold=3).ok() is False                   # n = 6 is not a multiple of 4


def test_gated_data_gradient_column_by_hand():
    """the gate branch of a gated layer sits at data-gradient column cout + co; its forward rows follow perm 0 (cout = 12)"""
    L = W.Layer(kh=1, kw=3, cin=5, cout=12, gated=1, shuffle=1, ka=0, kg=400, ba=800, bg=900)
    p = _params_for(L, _coded(L))
    pl = W.bf16_planes(L, p)
    wd = W.decode("wd_hi", pl["wd_hi"]) + W.decode("wd_lo", pl["wd_lo"])
    nt_n, cin_k, cin_n, nt_k, cin_q, nt_q = L.dims()
    assert (nt_n, cin_k, cin_n, nt_k, cin_q, nt_q) == (128, 64, 128, 64, 128, 128)
    for t in range(3):
        for ci in range(5):
            assert wd[t, ci, 12 + 5] == 8192 + t * 1024 + ci * 32 + 5           # gate, co = 5
            assert wd[t, ci, 5] == t * 1024 + ci * 32 + 5                       # a, co = 5
    assert (wd[:, 5:, :] == 0).all() and (wd[:, :, 24:] == 0).all()
    bias = pl["bias"].view(np.float32)
    assert bias[17] == 2000 + 5 and bias[5] == 1000 + 5 and (bias[24:] == 0).all()
    # cin = 5: no F16F8 planes (quads of input channels)
    assert not L.q_ok()


def test_f16f8_layouts_follow_the_bf16_ones():
    """the F16F8 planes are the same scatter of other element values: with values exact in both formats they decode equal"""
    L = W.Layer(kh=1, kw=5, cin=8, cout=128, gated=1, shuffle=2, ka=0, kg=6000, ba=12000, bg=12200)
    p = _params_for(L, lambda b, n: ((np.arange(n) % 61) - 30 + 64 * b).astype(np.float32) / 4)
    b16, q = W.bf16_planes(L, p), W.f16f8_planes(L, p)
    assert np.array_equal(W.decode("wf_hi", b16["wf_hi"])[:, :, :8], W.decode("wq16", q["wq16"])[:, :, :8])
    assert np.array_equal(W.decode("wd_hi", b16["wd_hi"])[:, :, :256], W.decode("wdq16", q["wdq16"])[:, :, :256])
    assert (q["wq16"][:, :, 8:] == 0).all() and (q["wdq16"][:, 8:, :] == 0).all() and (q["wq8lo"] == 0).all()
    assert set(W.f16f8_planes(L, p, train=False)) == {"wq16", "wq8hi", "wq8lo", "bias"}


def _q(w):
    q16, hi, lo = W.Q.quant_planes(np.array([w], np.float32), W.Q.WGT)
    return int(q16.view(np.uint16)[0]), int(hi[0]), int(lo[0])


def test_weight_window_codes_by_hand():
    """fp16 bits, e4m3 hi = e4m3(fp16(w) * 8), e4m3 lo = e4m3((w - fp16(w)) * 2^15): round to nearest even at ties, saturation to +-448
    (0x7E / 0xFE) where the scaled value exceeds 448, 0x7F never produced.  e4m3 code = sign | exponent + 7 << 3 | mantissa."""
    cases = [
        (1 + 2.0 ** -11, (0x3C00, 0x50, 0x58)),           # fp16 tie -> 1 (even); hi 8; lo 2^-11 * 2^15 = 16
        (1 + 3 * 2.0 ** -11, (0x3C02, 0x50, 0xD8)),       # fp16 tie -> 1 + 2^-9; hi 8 (8.0156 rounds to 8); lo -16
        (1.0625 / 8, (0x3040, 0x38, 0x00)),               # hi = e4m3(1.0625): tie between 1 (m 0) and 1.125 (m 1) -> 1 = 0x38
        (1.1875 / 8, (0x30C0, 0x3A, 0x00)),               # 1.1875: tie between 1.125 (m 1) and 1.25 (m 2) -> 1.25 = 0x3A
        (50.0, (0x5240, 0x7C, 0x00)),                     # hi = e4m3(400): tie between 384 (m 4) and 416 (m 5) -> 384
        (54.0, (0x52C0, 0x7E, 0x00)),                     # hi = e4m3(432): tie between 416 and 448 (m 6) -> 448
        (56.0, (0x5300, 0x7E, 0x00)),                     # the hi plane's edge: 448 exactly
        (58.0, (0x5340, 0x7E, 0x00)),                     # 464, beyond the edge: saturates to 448 (not 480 / NaN)
        (-60.0, (0xD380, 0xFE, 0x00)),
        (28.0 + 2.0 ** -7, (0x4F00, 0x76, 0x78)),         # fp16 tie at 28 -> 28 (even); hi 224; residual 2^-7 -> lo 256, no clamp
        (32.0 + 448 * 2.0 ** -15, (0x5000, 0x78, 0x7E)),  # residual 448 / 2^15: lo = 448 exactly, the last unclamped residual
        (32.015, (0x5000, 0x78, 0x7E)),                   # residual 0.015 * 2^15 = 491.5: clamps to 448 (RNE alone would give 480)
        (-32.015, (0xD000, 0xF8, 0xFE)),
        (65504.0, (0x7BFF, 0x7E, 0x00)),                  # fp16 max: hi clamps
        (65519.0, (0x7BFF, 0x7E, 0x7E)),                  # still fp16 65504; residual 15 * 2^15 clamps
        (65520.0, (0x7C00, 0x7E, 0xFE)),                  # fp16 overflows to inf: hi saturates to 448, lo = (w - inf) * 2^15 to -448
        (-65520.0, (0xFC00, 0xFE, 0x7E)),
        (2.0 ** -25, (0x0000, 0x00, 0x00)),               # fp16 tie between 0 and 2^-24 -> 0; lo = e4m3(2^-10): tie -> 0
        (3 * 2.0 ** -26, (0x0001, 0x00, 0x80)),           # fp16 2^-24 (subnormal); lo = -2^-26 * 2^15 = -2^-11 -> -0
        (2.0 ** -14, (0x0400, 0x00, 0x00)),               # fp16's lower edge; hi = e4m3(2^-11) -> 0
        (0.0, (0x0000, 0x00, 0x00)),
        (-0.0, (0x8000, 0x80, 0x00)),                     # -0: fp16 -0, hi -0, lo (-0) - (-0) = +0
    ]
    for w, want in cases:
        assert _q(w) == want, (w, [hex(v) for v in _q(w)], [hex(v) for v in want])


def test_bf16_split_codes_by_hand():
    for w, (hi, lo) in ((1 + 2.0 ** -8, (0x3F80, 0x3B80)),          # tie -> 1 (even); lo = 2^-8
                        (1 + 3 * 2.0 ** -8, (0x3F82, 0xBB80)),      # tie -> 1 + 2^-6 (even); lo = -2^-8
                        (1 + 2.0 ** -8 + 2.0 ** -23, (0x3F81, 0xBB80)),  # just above the tie: rounds up; lo = bf16(-(2^-8 - 2^-23)) = -2^-8
                        (-0.0, (0x8000, 0x0000))):
        h, l = W.Q.split_bf16(np.array([w], np.float32))
        assert (int(h[0]), int(l[0])) == (hi, lo), (w, hex(int(h[0])), hex(int(l[0])))


def test_stress_set_reaches_every_edge():
    s = W.stress_values()
    assert s.dtype == np.float32 and np.isfinite(s).all()
    q16, hi, lo = W.Q.quant_planes(s, W.Q.WGT)
    f = q16.astype(np.float64)
    assert (hi == 0x7E).any() and (hi == 0xFE).any() and (lo == 0x7E).any() and (lo == 0xFE).any()     # both clamps, both signs
    assert np.isinf(f).any() and ((np.abs(f) > 0) & (np.abs(f) < 2.0 ** -14)).any()                    # fp16 overflow and subnormals
    assert (np.signbit(s) & (s == 0)).any() and ((s == 0) & ~np.signbit(s)).any()
    assert (hi != 0x7F).all() and (lo != 0x7F).all() and (hi != 0xFF).all() and (lo != 0xFF).all()    # never NaN
    x = W.stress_fill((2, 3, 10, 12), np.random.default_rng(0))
    assert x.shape == (2, 3, 10, 12) and set(np.unique(x).tolist()) <= set(np.unique(s).tolist())
    assert np.abs(x[..., -1, :]).max() > 60000 and np.abs(x[..., -1]).max() > 60000                  # the tails carry the edges too


def test_padding_is_zero_and_extents_are_rounded():
    L = W.Layer(kh=3, kw=3, cin=36, cout=44, gated=1, shuffle=1, ka=0, kg=20000, ba=40000, bg=40100)
    p = _params_for(L, lambda b, n: np.full(n, 1.5 + b, np.float32))
    nt_n, cin_k, cin_n, nt_k, cin_q, nt_q = L.dims()
    assert (nt_n, cin_k, cin_n, nt_k, cin_q, nt_q) == (128, 64, 128, 128, 128, 128)
    b16, q = W.bf16_planes(L, p), W.f16f8_planes(L, p)
    wf = W.decode("wf_hi", b16["wf_hi"])
    assert wf.shape == (9, 128, 64) and (wf[:, :88, :36] > 0).all() and (wf[:, 88:, :] == 0).all() and (wf[:, :, 36:] == 0).all()
    wdq = W.decode("wdq16", q["wdq16"])
    assert wdq.shape == (9, 128, 128) and (wdq[:, :36, :88] > 0).all() and (wdq[:, 36:, :] == 0).all() and (wdq[:, :, 88:] == 0).all()
    assert (b16["wf_lo"] == 0).all()                                                                    # 1.5, 2.5: exact in bf16
    assert W.kept_planes(L, "f16f8", False) == ("wq16", "wq8hi", "wq8lo", "bias")
    assert W.kept_planes(L, "bf16x3", True) == ("wf_hi", "wf_lo", "wd_hi", "wd_lo", "bias")


def test_whole_model_encoder_equals_f16f8_ref():
    """quant_w (the encoder the whole-model comparisons use) against f16f8_ref.quant_planes with the weight scales, value by value and
    bit by bit, for the finite weights PARAM holds: log-uniform magnitudes over the whole fp32 range the planes see, the stress set, f16f8_ref's edge values, every fp16
    value and the midpoints of every pair of neighbouring e4m3 values (both scaled back to weight magnitudes)"""
    rng = np.random.default_rng(7)
    f16 = np.arange(65536, dtype=np.uint16).view(np.float16).astype(np.float32)
    e = W.Q.E4M3_VALUES[:0x7F]
    mids = ((e[:-1] + e[1:]) / 2).astype(np.float32)
    edges = W.Q.edge_values()
    parts = [W.Q.log_uniform(2_000_000, rng, -40, 18), W.stress_values(), edges[np.isfinite(edges)], f16[np.isfinite(f16)],
             mids / 8, 1 + mids / 32768, 32 + mids / 32768, -(1 + mids / 32768)]
    for k, x in enumerate(parts):
        x = np.asarray(x, np.float32)
        got = W.quant_w(x)
        q16, hi, lo = W.Q.quant_planes(x, W.Q.WGT)
        for name, g, r in zip(("q16", "q8hi", "q8lo"), got, (q16.view(np.uint16), hi, lo)):
            bad = np.flatnonzero(g != r)
            assert bad.size == 0, (k, name, x[bad[:4]].tolist(), g[bad[:4]].tolist(), r[bad[:4]].tolist())


def test_differences_name_the_element():
    L = W.Layer(kh=1, kw=2, cin=4, cout=8, gated=1, ka=0, kg=100, ba=200, bg=300)
    p = _params_for(L, lambda b, n: np.full(n, 1.0 + b, np.float32))
    ref = W.f16f8_planes(L, p)
    assert all(W.differences(n, ref[n], ref[n]) == "" for n in ref)
    got = ref["wdq8hi"].copy()
    got[1, 3, 9] = 0x7E
    assert W.differences("wdq8hi", got, ref["wdq8hi"]) == \
        "1 of %d elements differ: element [1, 3, 9] got 0x7e (448.0) reference 0x58 (16.0)" % got.size
    got = ref["bias"].copy()
    got[0] = np.float32(2.5).view(np.uint32)
    assert "element [0] got 0x40200000 (2.5) reference 0x447a0000 (1000.0)" in W.differences("bias", got, ref["bias"])
    h = ref["wq16"].copy()
    h[0, 8, 0] = 0x3C00                                           # row 8: the gate branch (2.0)
    assert "got 0x3c00 (1.0) reference 0x4000 (2.0)" in W.differences("wq16", h, ref["wq16"])
