"""Float64 emulation of the tensor-core convolutions' arithmetic, built on the operand planes of tests/f16f8_ref.py.

With conv(a, b) the TF-SAME cross-correlation of the oracle (conv2d_same) and its autograd for the two gradients, a kernel of precision
p computes, in exact arithmetic, the sum of its plane products:

    fp32 (0):    conv(x, w)
    bf16 (2):    conv(xh, wh)                                          xh, xl = split_bf16(x)
    bf16x3 (1):  conv(xh, wh) + conv(xh, wl) + conv(xl, wh)            (no lo x lo term)
    F16F8 (3):   conv(q16x, q16w) + 2^-15 (conv(x8hi, w8lo) + conv(x8lo, w8hi))      x: activation scales, w: weight scales

plus the bias.  The data gradient pairs dy (activation role) with w the same way; the weight gradient pairs x with dy, and in F16F8
reads the fp16 planes alone (`wgrad_f16` = 1) or adds 2^-12 (x8hi (x) dy8lo + x8lo (x) dy8hi), both operands in the activation role.
db is the column sum of the fp32 dy.

Also here:
- mutants: the same sums with one piece of the arithmetic wrong (fp16 only, one cross product lost, the rescale off by 2, the cross
  terms of one (tap, 64-channel stage) block lost);
- the lattice generator and its certificate: operands whose planes are few-bit dyadic values, sparse enough that every partial sum
  of every kernel is exact in its accumulator whatever the order, so the kernel must equal the emulation bit for bit;
- the launch mirror: tc_gemm.cu's choice of tile width, stage count and split-K, used to assert which paths a case list reaches.

Every function takes torch or numpy fp32 inputs on the CPU and computes in float64 on `device` (the CPU or a GPU).
"""
import math

import numpy as np
import torch

import f16f8_ref as R
from oracle.cyclegan_oracle import conv2d_same, same_pad

FP32, BF16X3, BF16, F16F8 = 0, 1, 2, 3

# (name, B, H, W, Cin, kh, kw, Cout, sh, sw), beside tests/test_gpu_kernels.py CONV_CASES: what the model-sized small cases do not
# reach (launch mirror, 132 SMs): persistent CTAs that walk several tiles, several 128-wide column tiles, uneven and empty split-K
# items, and stride-2 data gradients on odd extents
BIG_CASES = [
    ("big.o1", 270, 1, 128, 256, 1, 15, 24, 1, 1),        # fwd BN 32 x 270 tiles; dgrad BN 256 x 270; split-K 13, uneven
    ("big.h1", 270, 1, 128, 24, 1, 15, 128, 1, 1),        # dgrad BN 32 x 270; fwd BN 128 x 270
    ("big.res_h1", 67, 1, 128, 512, 1, 3, 1024, 1, 1),    # fwd BN 256 x 268 tiles; split-K 8, uneven
    ("big.n384", 89, 1, 128, 100, 1, 5, 384, 1, 1),       # BN 128 x 3 column tiles; Cin padding; N tail in dgrad
    ("big.split", 1, 1, 32769, 64, 1, 1, 64, 1, 1),       # M % 128 = 1; split-K 30 with an empty last item
]
ODD_CASES = [
    ("odd.d1", 1, 1, 65, 128, 1, 5, 64, 1, 2),            # 1-D stride 2 on an odd width: parity classes of 33 and 32 rows
    ("odd.D", 1, 13, 33, 64, 3, 3, 128, 2, 2),            # 2-D stride 2 on odd extents: four classes, unequal tap sets
]


def dense_case(case, seed=0):
    """unit randn x and dy, weights randn / sqrt(K), randn bias (fp32 numpy): the inputs of the dense tier"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = -(-H // sh), -(-W // sw)
    x = torch.randn((B, H, W, Cin), generator=g)
    w = torch.randn((kh, kw, Cin, Cout), generator=g) / math.sqrt(kh * kw * Cin)
    b = torch.randn((Cout,), generator=g)
    dy = torch.randn((B, Ho, Wo, Cout), generator=g)
    return tuple(t.numpy() for t in (x, w, b, dy))


Q_ACC = 2.0 ** -15          # kernels.cuh CGVC_Q_ACC_SHIFT: the forward / data-gradient cross terms
Q_WGRAD = 2.0 ** -12        # tc_gemm.cu CGVC_Q_WGRAD_SHIFT: the weight-gradient cross terms
ACC_BITS = 24               # fp32 accumulators (FFMA, fp16 / bf16 MMAs)
E4M3_ACC_BITS = 13          # the e4m3 cross phase of the forward / data-gradient kernel (Hopper's FP8 MMA is reported to keep ~14 bits)


# ------------------------------------------------------------------------------------------------ planes
def planes(x, prec, role):
    """decoded operand planes (float64 numpy) of fp32 x: {'x'} (fp32), {'hi', 'lo'} (bf16), {'hi', '8hi', '8lo'} (F16F8; role 'act'
    or 'wgt' picks the scales)"""
    x = np.ascontiguousarray(np.asarray(x, np.float32))
    if prec == FP32:
        return {"x": x.astype(np.float64)}
    if prec in (BF16X3, BF16):
        hi, lo = R.split_bf16(x)
        return {"hi": R.bf16_decode(hi).astype(np.float64), "lo": R.bf16_decode(lo).astype(np.float64)}
    q16, h8, l8 = R.quant_planes(x, R.ACT if role == "act" else R.WGT)
    return {"hi": q16.astype(np.float64), "8hi": R.e4m3_decode(h8), "8lo": R.e4m3_decode(l8)}


def pairs(prec, form, w16=1):
    """(coefficient, activation plane, weight plane) of each product; form 'fwd' / 'dgrad' (a = x or dy, b = w) or 'wgrad' (a = x,
    b = dy).  The first pair is the main product; the rest are the cross terms."""
    if prec == FP32:
        return [(1.0, "x", "x")]
    if prec == BF16:
        return [(1.0, "hi", "hi")]
    if prec == BF16X3:
        return [(1.0, "hi", "hi"), (1.0, "hi", "lo"), (1.0, "lo", "hi")]
    if form == "wgrad":
        return [(1.0, "hi", "hi")] if w16 else [(1.0, "hi", "hi"), (Q_WGRAD, "8hi", "8lo"), (Q_WGRAD, "8lo", "8hi")]
    return [(1.0, "hi", "hi"), (Q_ACC, "8hi", "8lo"), (Q_ACC, "8lo", "8hi")]


# ------------------------------------------------------------------------------------------------ the three products
def _t(a, device):
    return torch.as_tensor(np.asarray(a, np.float64), device=device)


def conv_fwd(a, b, s):
    return conv2d_same(a, b, None, s)


def conv_dx(dy, b, xshape, s):
    xz = torch.zeros(xshape, dtype=torch.float64, device=dy.device, requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(conv2d_same(xz, b, None, s), xz, dy)[0]


def conv_dw(a, dy, wshape, s):
    wz = torch.zeros(wshape, dtype=torch.float64, device=dy.device, requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(conv2d_same(a, wz, None, s), wz, dy)[0]


def combine(form, P_a, P_b, prs, s, out_shape, absolute=False, device="cpu"):
    """sum of coefficient * product over the pairs prs, planes P_a / P_b (dicts of numpy planes)"""
    acc = None
    for c, ka, kb in prs:
        a, b = _t(P_a[ka], device), _t(P_b[kb], device)
        if absolute:
            a, b = a.abs(), b.abs()
        if form == "fwd":
            r = conv_fwd(a, b, s)
        elif form == "dgrad":
            r = conv_dx(a, b, out_shape, s)
        else:
            r = conv_dw(a, b, out_shape, s)
        r = r * c
        acc = r if acc is None else acc + r
    return acc


def emulate(case, prec, x, w, b, dy, w16=1, device="cpu", forms=("fwd", "dgrad", "wgrad"), P=None):
    """what the kernels of precision prec compute (float64 torch on device): {'y', 'dx', 'dw', 'db'} for the requested forms.
    P: planes already computed by case_planes (reused across calls)"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    s = (sh, sw)
    P = P or case_planes(prec, x, w, dy)
    out = {}
    if "fwd" in forms:
        y = combine("fwd", P["x"], P["w"], pairs(prec, "fwd"), s, None, device=device)
        out["y"] = y + _t(b, device) if b is not None else y
    if "dgrad" in forms:
        out["dx"] = combine("dgrad", P["dy"], P["w"], pairs(prec, "dgrad"), s, (B, H, W, Cin), device=device)
    if "wgrad" in forms:
        out["dw"] = combine("wgrad", P["x"], P["dy"], pairs(prec, "wgrad", w16), s, (kh, kw, Cin, Cout), device=device)
        out["db"] = _t(dy, device).reshape(-1, Cout).sum(0)
    return out


def case_planes(prec, x, w, dy):
    return {"x": planes(x, prec, "act"), "w": planes(w, prec, "wgt"), "dy": planes(dy, prec, "act") if dy is not None else None}


# ------------------------------------------------------------------------------------------------ mutants
def _tap_operands(case, form, Pa, Pw, ka, kb):
    """per tap t: (A_t [M, K], B_t [K, N]) whose product is tap t's share of the forward (K = Cin) or data-gradient (K = Cout) GEMM,
    rows M of the forward output grid (a data-gradient row whose source for tap t lies in the padding is zero)"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    pt, pb = same_pad(H, kh, sh); pl, pr = same_pad(W, kw, sw)
    T = kh * kw
    w = torch.as_tensor(Pw[kb]).reshape(T, Cin, Cout)
    if form == "fwd":
        a = torch.nn.functional.pad(torch.as_tensor(Pa[ka]).permute(0, 3, 1, 2), (pl, pr, pt, pb))
        u = torch.nn.functional.unfold(a, (kh, kw), stride=(sh, sw))              # [B, Cin * T, L]
        u = u.permute(0, 2, 1).reshape(-1, Cin, T)
        return [(u[:, :, t], w[t]) for t in range(T)]
    ones = torch.nn.functional.pad(torch.ones(1, 1, H, W, dtype=torch.float64), (pl, pr, pt, pb))
    valid = torch.nn.functional.unfold(ones, (kh, kw), stride=(sh, sw))[0].T         # [L, T]: tap t of row m reads the input
    dy = torch.as_tensor(Pa[ka]).reshape(B, -1, Cout)
    return [((dy * valid[None, :, t:t + 1]).reshape(-1, Cout), w[t].T) for t in range(T)]


def block_nonzero(case, prec, form, P, blocks=None):
    """for each (tap, 64-channel stage) block of the forward (stages over Cin) or data-gradient (stages over Cout) contraction:
    whether its cross terms (every product of a single-product precision) are nonzero in some output, i.e. whether losing the block
    changes the exact result.  blocks: list of (tap, stage) to check (default all); returns {(tap, stage): bool}"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    prs = pairs(prec, form)
    prs = prs[1:] if len(prs) > 1 else prs
    Pa = P["x"] if form == "fwd" else P["dy"]
    K = Cin if form == "fwd" else Cout
    if blocks is None:
        blocks = [(t, s) for t in range(kh * kw) for s in range(-(-K // 64))]
    ops = [(c, _tap_operands(case, form, Pa, P["w"], ka, kb)) for c, ka, kb in prs]
    out = {}
    for t, s in blocks:
        sl = slice(64 * s, 64 * s + 64)
        r = sum(c * (o[t][0][:, sl] @ o[t][1][sl]) for c, o in ops)
        out[(t, s)] = bool((r != 0).any())
    return out


def mutant_pairs(prec, form, name, w16=1):
    """the pairs of a coarse mutant: 'main_only' (every cross term lost), 'drop_cross' (the first cross product lost), 'rescale_x2'
    (the cross terms rescaled by twice the right power of two)"""
    prs = pairs(prec, form, w16)
    if name == "main_only":
        return prs[:1]
    if name == "drop_cross":
        return prs[:1] + prs[2:]
    if name == "rescale_x2":
        return prs[:1] + [(2 * c, a, b) for c, a, b in prs[1:]]
    raise ValueError(name)


COARSE_MUTANTS = {BF16X3: ("main_only", "drop_cross"), F16F8: ("main_only", "drop_cross", "rescale_x2")}


# ------------------------------------------------------------------------------------------------ lattice operands and certificate
def lsb_exp(v):
    """the exponent of the finest power of two among the nonzero values of v (None if all are zero)"""
    v = np.abs(np.asarray(v, np.float64)).ravel()
    v = v[v != 0]
    if v.size == 0:
        return None
    m, e = np.frexp(v)
    ints = (m * 2.0 ** 53).astype(np.int64)
    tz = np.log2((ints & -ints).astype(np.float64)).astype(np.int64)
    return int((e - 53 + tz).min())


def _lat_values(shape, kind, role, rng, density):
    """fp32 lattice operand: h + l with h = +-2^a (a in {0, 1}) and l a few-bit offset of independent sign that sets every lo plane,
    on a random sparsity mask of the given density.
      kind 'int':   h only (the fp32 kernels need nothing finer)
      kind 'bf16':  l = +-2^(a-10): bf16 hi = h, lo = l
      kind 'f16f8': l = +-2^(a-13): q16 = h, e4m3 hi = h * S_hi, lo = l * S_lo (both exact, normal e4m3)"""
    a = rng.integers(0, 2, shape)
    h = np.ldexp(1.0, a) * rng.choice([-1.0, 1.0], shape)
    if kind == "int":
        v = h
    else:
        sh = {"bf16": -10, "f16f8": -13}[kind]
        v = h + np.ldexp(1.0, a + sh) * rng.choice([-1.0, 1.0], shape)
    v = v * (rng.random(shape) < density)
    return v.astype(np.float32)


LATTICE_KIND = {FP32: "int", BF16X3: "bf16", BF16: "bf16", F16F8: "f16f8"}
CERT_MARGIN = 3.0           # the lattice aims at an expected largest sum this far below the certificate's bound


def _contraction_lengths(case):
    """forward K, largest data-gradient K (over the parity classes), weight-gradient K (output rows), in scalar products per output"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    Ho, Wo = -(-H // sh), -(-W // sw)
    kd = max(len(g["taps"]) for g in dgrad_classes(case))
    return kh * kw * Cin, kd * Cout, B * Ho * Wo


def lattice_case(case, prec, seed=0):
    """lattice operands (x, w, b, dy) of a case for precision prec: fp32 numpy.  The densities of x and dy are chosen from the
    contraction lengths so that the expected sums lie CERT_MARGIN below the certificate; `certificate` decides."""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    Ho, Wo = -(-H // sh), -(-W // sw)
    kind = LATTICE_KIND[prec]
    rng = np.random.default_rng([seed, prec, B, H, W, Cin, kh, kw, Cout, sh, sw])
    # scalar products of one output that a 2^24 (or 2^13) accumulator holds exactly, in units of the finest term: the plane
    # magnitudes are 2^a, a in {0, 1}, so a main product costs 2.25 units on average in units of its own lsb, and the lo offsets put
    # the finest term 2^10 (bf16) or 2^13 (F16F8) below the main product's lsb
    # (the column sums of db add fp32 dy values of mean magnitude 1.5 whose finest bit lies 2^10 / 2^13 below their leading one)
    shift = {"int": 0, "bf16": 10, "f16f8": 13}[kind]
    n_max = 2.0 ** (ACC_BITS - shift) / 2.25 / CERT_MARGIN
    n_db = 2.0 ** (ACC_BITS - shift) / 1.5 / CERT_MARGIN
    kf, kd, kwg = _contraction_lengths(case)
    dx_ = min(1.0, n_max / kf)
    ddy = min(1.0, n_max / kd, n_max / (kwg * dx_), n_db / kwg)
    x = _lat_values((B, H, W, Cin), kind, "act", rng, dx_)
    w = _lat_values((kh, kw, Cin, Cout), kind, "wgt", rng, 1.0)
    dy = _lat_values((B, Ho, Wo, Cout), kind, "act", rng, ddy)
    b = _lat_values((Cout,), "int", "act", rng, 1.0)
    return x, w, b, dy


def certificate(case, prec, x, w, b, dy, w16=1, device="cpu", P=None, forms=("fwd", "dgrad", "wgrad", "db")):
    """per form, the largest sum of |terms| over the outputs against the bound under which every partial sum is exact:
    {form: (phase, largest, bound)} with form in fwd / dgrad / wgrad / db and phase 'total' or 'e4m3' (the F16F8 forward and
    data-gradient cross phase, before the rescale).  Holds when largest < bound for every entry."""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    s = (sh, sw)
    P = P or case_planes(prec, x, w, dy)
    res = []
    memo = {}

    def lsb(Pd, k):
        if (id(Pd), k) not in memo:
            memo[(id(Pd), k)] = lsb_exp(Pd[k])
        return memo[(id(Pd), k)]

    spec = [("fwd", P["x"], P["w"], None, b), ("dgrad", P["dy"], P["w"], (B, H, W, Cin), None),
            ("wgrad", P["x"], P["dy"], (kh, kw, Cin, Cout), None)]
    for form, Pa, Pb, shape, bias in spec:
        if form not in forms:
            continue
        prs = pairs(prec, form, w16)
        # finest power of two among the terms (coefficients are powers of two; a plane that is all zero has no terms)
        ex = [lsb(Pa, ka) + lsb(Pb, kb) + int(math.log2(c)) for c, ka, kb in prs if lsb(Pa, ka) is not None and lsb(Pb, kb) is not None]
        if bias is not None and lsb_exp(bias) is not None:
            ex.append(lsb_exp(bias))
        g = 2.0 ** min(ex)
        prods = [combine(form, Pa, Pb, [(1.0, ka, kb)], s, shape, absolute=True, device=device) for _, ka, kb in prs]
        tot = sum(c * p for (c, _, _), p in zip(prs, prods))
        if bias is not None:
            tot = tot + _t(np.abs(bias), device)
        res.append((form, "total", float(tot.max()), 2.0 ** ACC_BITS * g))
        if prec == F16F8 and form != "wgrad":
            # (an operand whose fp16 plane holds it exactly has all-zero e4m3 lo planes: those cross products have no terms)
            ec = [lsb(Pa, ka) + lsb(Pb, kb) for _, ka, kb in prs[1:] if lsb(Pa, ka) is not None and lsb(Pb, kb) is not None]
            if ec:
                res.append((form, "e4m3", float(sum(prods[1:]).max()), 2.0 ** E4M3_ACC_BITS * 2.0 ** min(ec)))
    if "db" in forms:
        dyc = np.abs(np.asarray(dy, np.float64)).reshape(-1, Cout).sum(0)
        res.append(("db", "total", float(dyc.max()), 2.0 ** ACC_BITS * 2.0 ** lsb_exp(dy)))
    return res


def fp32_sum_orders(case, prec, x, w, b, P=None):
    """the forward of a case summed term by term in float32, in forward and in reverse order of (pair, tap, channel), with the
    bias last: (forward, reverse, float64), torch [B, Ho, Wo, Cout] on the CPU"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    P = P or case_planes(prec, x, w, None)
    Ho, Wo = -(-H // sh), -(-W // sw)
    pt, pb = same_pad(H, kh, sh); pl, pr = same_pad(W, kw, sw)
    cols, rows = [], []
    for c, ka, kb in pairs(prec, "fwd"):
        a = torch.nn.functional.pad(_t(P["x"][ka], "cpu").permute(0, 3, 1, 2), (pl, pr, pt, pb))
        u = torch.nn.functional.unfold(a, (kh, kw), stride=(sh, sw))          # [B, Cin * kh * kw, L], index c * kh * kw + tap
        cols.append(u.permute(0, 2, 1).reshape(B * Ho * Wo, -1) * c)
        rows.append(_t(P["w"][kb], "cpu").permute(2, 0, 1, 3).reshape(-1, Cout))
    A = torch.cat(cols, 1); Bm = torch.cat(rows, 0)
    exact = A @ Bm + _t(b, "cpu")
    A32, B32 = A.float(), Bm.float()
    out = []
    for order in (range(A.shape[1]), reversed(range(A.shape[1]))):
        acc = torch.zeros(A.shape[0], Cout, dtype=torch.float32)
        for k in order:
            acc += A32[:, k:k + 1] * B32[k:k + 1]
        acc += torch.as_tensor(np.asarray(b, np.float32))
        out.append(acc.reshape(B, Ho, Wo, Cout))
    return out[0], out[1], exact.reshape(B, Ho, Wo, Cout)


# ------------------------------------------------------------------------------------------------ launch mirror (tc_gemm.cu)
def _ru(v, m):
    return (v + m - 1) // m * m


def tile_rows(n_real, n_padded):
    return 256 if n_padded % 256 == 0 else (32 if n_real <= 32 else 128)


def nt_stages(bn, npl):
    """NTCfg<BN, NPL>::STAGES"""
    return (192 * 1024) // ((2 if npl == 2 else 1) * (128 * 128 + bn * 128))


def tn_stages(npl, w16):
    """TNCfg<NPL, W16>::STAGES"""
    return (192 * 1024) // ((1 if (npl == 1 or w16) else 2) * (64 * 256 + 64 * 512))


NPL = {BF16X3: 2, BF16: 1, F16F8: 3}


def dgrad_classes(case):
    """geom.h dgrad_geoms: per non-empty output parity class, its rows and taps (widx)"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    ph, _ = same_pad(H, kh, sh); pw, _ = same_pad(W, kw, sw)
    out = []
    for py in range(sh):
        for px in range(sw):
            hy, wx = -(-(H - py) // sh), -(-(W - px) // sw)
            if hy <= 0 or wx <= 0:
                continue
            taps = [i * kw + j for i in range(kh) for j in range(kw) if (py + ph - i) % sh == 0 and (px + pw - j) % sw == 0]
            out.append({"rows": B * hy * wx, "taps": taps})
    return out


def nt_launch(M, N, C, ntaps, prec, nsm):
    """launch_nt: one plain-epilogue NT launch of M rows, N real columns, C padded contraction channels per tap"""
    npl = NPL[prec]
    Nw = _ru(N, 128)
    bn = tile_rows(N, Nw)
    n_tiles = 1 if bn == 32 else Nw // bn
    tiles = -(-M // 128) * n_tiles
    num_kb = ntaps * (C // 64) * (2 if npl == 3 else 1)
    S = nt_stages(bn, npl)
    return {"bn": bn, "npl": npl, "n_tiles": n_tiles, "tiles": tiles, "grid": min(tiles, nsm), "num_kb": num_kb, "stages": S,
            "M": M, "N": N, "K": ntaps * C}


def tn_launch(M, N, Cin, ntaps, prec, w16, nsm):
    """launch_tn: the weight-gradient launch (M output rows, N = Cout, Cin input channels), its split-K and chunks"""
    npl = NPL[prec]
    w16 = 1 if (prec == F16F8 and w16) else 0
    g_ld = _ru(N, 128) if prec == F16F8 else _ru(N, 64)
    x_ld = _ru(Cin, 128) if prec == F16F8 else _ru(Cin, 64)
    tiles = -(-g_ld // 256) * -(-x_ld // 128) * ntaps
    maxsplit = max(1, min(32, M // 1024))
    ks, best = 1, 0.0
    for k in range(1, maxsplit + 1):
        items = tiles * k
        eff = items / (-(-items // nsm) * nsm)
        if items < nsm:
            eff *= 0.5
        if eff > best + 0.02:
            best, ks = eff, k
    chunk = _ru(-(-M // ks), 64)
    num_kb = [max(0, -(-(min(M, (i + 1) * chunk) - i * chunk) // 64)) for i in range(ks)]
    return {"npl": npl, "w16": w16, "ksplit": ks, "chunk": chunk, "items": tiles * ks, "grid": min(tiles * ks, nsm),
            "stages": tn_stages(npl, w16), "uneven": ks > 1 and M % chunk != 0, "empty": ks > 1 and (ks - 1) * chunk >= M,
            "num_kb": num_kb}


def case_launches(case, prec, w16, nsm):
    """the tensor-core launches one cgvc_conv_forward + cgvc_conv_backward call of precision prec makes:
    {'fwd': nt, 'dgrad': [nt per parity class], 'wgrad': tn}"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    Ho, Wo = -(-H // sh), -(-W // sw)
    q = prec == F16F8
    cin_p = _ru(Cin, 128) if q else _ru(Cin, 64)
    cout_p = _ru(Cout, 128) if q else _ru(Cout, 64)
    return {"fwd": nt_launch(B * Ho * Wo, Cout, cin_p, kh * kw, prec, nsm),
            "dgrad": [nt_launch(c["rows"], Cin, cout_p, len(c["taps"]), prec, nsm) for c in dgrad_classes(case)],
            "wgrad": tn_launch(B * Ho * Wo, Cout, Cin, kh * kw, prec, w16, nsm)}


def supports(case, prec):
    """the tensor-core path takes the case (F16F8 packs quads of input channels)"""
    return prec != F16F8 or case[4] % 4 == 0


PREC_NAMES = {BF16X3: "bf16x3", BF16: "bf16", F16F8: "f16f8"}


def coverage(cases, nsm):
    """requirement -> names of the cases (with their precision) that reach it; every list must be non-empty"""
    req = {}

    def hit(key, name):
        req.setdefault(key, [])
        if name is not None:
            req[key].append(name)

    for prec in (BF16X3, BF16, F16F8):
        pn = PREC_NAMES[prec]
        for bn in (32, 128, 256):
            for role in ("fwd", "dgrad"):
                hit("NT %s BN %d %s" % (pn, bn, role), None)
            hit("NT %s BN %d: > 2 x SMs tiles, num_kb %% STAGES != 0" % (pn, bn), None)
        for key in ("M % 128 tail", "BN 128 with several column tiles", "Cin padded in the contraction",
                    "stride-2 dgrad, odd extent, 1-D", "stride-2 dgrad, odd extent, 2-D"):
            hit("NT %s %s" % (pn, key), None)
        for w16 in ((0, 1) if prec == F16F8 else (0,)):
            tn = "TN %s%s" % (pn, " w16" if w16 else "")
            hit(tn + ": split-K >= 2 with an uneven last chunk", None)
            hit(tn + ": an empty split item", None)
        for case in cases:
            if not supports(case, prec):
                continue
            name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
            for w16 in ((0, 1) if prec == F16F8 else (0,)):
                L = case_launches(case, prec, w16, nsm)
                tn = "TN %s%s" % (pn, " w16" if w16 else "")
                if L["wgrad"]["uneven"]:
                    hit(tn + ": split-K >= 2 with an uneven last chunk", name)
                if L["wgrad"]["empty"]:
                    hit(tn + ": an empty split item", name)
            for role, nts in (("fwd", [L["fwd"]]), ("dgrad", L["dgrad"])):
                for nt in nts:
                    hit("NT %s BN %d %s" % (pn, nt["bn"], role), name)
                    # (F16F8 at BN 256 runs 4 stages over 4 * taps * Cpad / 128 K blocks: its ring always ends a tile where it began)
                    ring_odd = nt["num_kb"] % nt["stages"] != 0 or (prec == F16F8 and nt["bn"] == 256)
                    if nt["tiles"] > 2 * nsm and ring_odd:
                        hit("NT %s BN %d: > 2 x SMs tiles, num_kb %% STAGES != 0" % (pn, nt["bn"]), "%s %s" % (name, role))
                    if nt["M"] % 128:
                        hit("NT %s M %% 128 tail" % pn, "%s %s" % (name, role))
                    if nt["bn"] == 128 and nt["n_tiles"] > 1:
                        hit("NT %s BN 128 with several column tiles" % pn, "%s %s" % (name, role))
            if Cin % (128 if prec == F16F8 else 64):
                hit("NT %s Cin padded in the contraction" % pn, name)
            odd = (sh == 2 and H % 2 == 1) or (sw == 2 and W % 2 == 1)
            if odd:
                hit("NT %s stride-2 dgrad, odd extent, %s" % (pn, "1-D" if H == 1 else "2-D"), name)
    return req
