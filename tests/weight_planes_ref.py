"""numpy construction of the tensor-core weight planes (csrc/tc_gemm.cu, "weight planes") of one registered layer from PARAM, bit for bit.

Written from the layout comments of csrc/tc_gemm.cuh (TcLayer) and csrc/tc_gemm.cu (perm_row, w_src, the padded extents), not by
calling the engine.  A layer is registered with its TF shape (kh, kw, cin, cout per branch, gated, shuffle, fold) and the PARAM offsets
of its kernels and biases; Ntot = cout * (gated ? 2 : 1), taps = kh * kw, and its planes are

    wf_hi / wf_lo     bf16   [taps][nt_n][cin_k]   forward: row perm_row(co, branch), column ci
    wd_hi / wd_lo     bf16   [taps][cin_n][nt_k]   data gradient: row ci, column branch * cout + co
    wq16 / wq8hi / wq8lo     [taps][nt_n][cin_q]   F16F8 forward (fp16, e4m3, e4m3; weight-role scales 8 and 2^15)
    wdq16 / wdq8hi / wdq8lo  [taps][cin_n][nt_q]   F16F8 data gradient, columns as wd
    bias              fp32   [nt_n]                bias[perm_row(co, branch)] = bias_branch[co]; none (all zero) for tap-folded layers

with *_k = rounded up to 64, *_n and *_q = rounded up to 128, and every element outside the layer's (ci < cin, co < cout) zero.  The
element at (tap, ci, co) of a branch is w_src: the TF kernel [taps][cin][cout], or for a tap-folded layer (fold > 0: a 1 x 1 layer whose
cout columns are (t, n) pairs, co = t * (cout / fold) + n) the kernel [fold][cin][cout / fold] element (t, ci, n).

Forward row order (perm_row), for the channel co of branch b (0: a, 1: gate):
    perm 0 (not gated, or cout not a multiple of 128):  b * cout + co
    perm 1 (gated, cout % 128 == 0):  256-row tiles [128 a | 128 g]:  (co // 128) * 256 + b * 128 + co % 128
    perm 2 (gated, pixel shuffle, cout % 128 == 0; Ch = cout / 2 post-shuffle channels, co = s * Ch + c):
           256-row tiles [64 a(c) | 64 a(c + Ch) | 64 g(c) | 64 g(c + Ch)]:  (c // 64) * 256 + b * 128 + s * 64 + c % 64

Element values: bf16 hi = bf16_rn(w), lo = bf16_rn(w - hi); F16F8 as tests/f16f8_ref.py quant_planes with the weight scales.
"""
import numpy as np

import f16f8_ref as Q

MAX_TAPS = 18                      # CGVC_MAX_TAPS
BF16_PLANES = ("wf_hi", "wf_lo", "wd_hi", "wd_lo")
Q_PLANES = ("wq16", "wq8hi", "wq8lo")
QD_PLANES = ("wdq16", "wdq8hi", "wdq8lo")
PLANE_DTYPE = dict([(n, np.uint16) for n in BF16_PLANES + ("wq16", "wdq16")] + [(n, np.uint8) for n in ("wq8hi", "wq8lo", "wdq8hi", "wdq8lo")]
                   + [("bias", np.uint32)])


def ru(v, m):
    return (v + m - 1) // m * m


class Layer(object):
    """One registered layer: the fields of include/cgvc.h cgvc_weight_layer_info that describe the registration."""
    FIELDS = ("kh", "kw", "cin", "cout", "gated", "shuffle", "fold", "ka", "kg", "ba", "bg")

    def __init__(self, **kw):
        for f in self.FIELDS:
            setattr(self, f, int(kw.get(f, 0)))
        if self.shuffle == 0:
            self.shuffle = 1

    @property
    def taps(self):
        return self.kh * self.kw

    @property
    def ntot(self):
        return self.cout * (2 if self.gated else 1)

    def dims(self):
        """padded extents (nt_n, cin_k, cin_n, nt_k, cin_q, nt_q)"""
        return (ru(self.ntot, 128), ru(self.cin, 64), ru(self.cin, 128), ru(self.ntot, 64), ru(self.cin, 128), ru(self.ntot, 128))

    def ok(self):
        """the shape has tensor-core planes at all"""
        if self.fold and (self.gated or self.taps != 1 or self.cout % self.fold or (self.cout // self.fold) % 4):
            return False
        return self.taps <= MAX_TAPS and self.ntot % 4 == 0

    def q_ok(self):
        """... and F16F8 planes (quads of input channels)"""
        return self.ok() and self.cin % 4 == 0

    def perm(self):
        if self.gated and self.shuffle == 2 and self.cout % 128 == 0:
            return 2
        return 1 if self.gated and self.cout % 128 == 0 else 0

    def branches(self):
        return (0, 1) if self.gated else (0,)

    def __repr__(self):
        return "Layer(%s)" % ", ".join("%s=%d" % (f, getattr(self, f)) for f in self.FIELDS)


def perm_rows(perm, cout, branch):
    """forward-plane row of every output channel co = 0 .. cout-1 of a branch"""
    co = np.arange(cout)
    if perm == 1:
        return (co // 128) * 256 + branch * 128 + co % 128
    if perm == 2:
        ch = cout // 2
        s = (co >= ch).astype(np.int64)
        c = co - s * ch
        return (c // 64) * 256 + branch * 128 + s * 64 + c % 64
    return branch * cout + co


def kernel(L, params, branch):
    """the branch's weights as float32 [taps][cin][cout] in the layer's (tap, ci, co) indexing (w_src)"""
    off = L.kg if branch else L.ka
    if L.fold:
        fn = L.cout // L.fold
        k = np.asarray(params[off:off + L.fold * L.cin * fn], np.float32).reshape(L.fold, L.cin, fn)
        return np.ascontiguousarray(k.transpose(1, 0, 2).reshape(1, L.cin, L.cout))
    return np.asarray(params[off:off + L.taps * L.cin * L.cout], np.float32).reshape(L.taps, L.cin, L.cout)


def _place(L, parts, fwd_cols, dg_cols, names):
    """scatter the per-branch element planes parts[branch][k] ([taps][cin][cout] each) into the forward and data-gradient layouts"""
    nt_n = L.dims()[0]
    out = {}
    for k, (nf, nd) in enumerate(names):
        dt = parts[0][k].dtype
        f = np.zeros((L.taps, nt_n, fwd_cols), dt)
        d = np.zeros((L.taps, dg_cols[0], dg_cols[1]), dt)
        for b in L.branches():
            v = parts[b][k]
            f[:, perm_rows(L.perm(), L.cout, b), :L.cin] = v.transpose(0, 2, 1)
            d[:, :L.cin, b * L.cout:(b + 1) * L.cout] = v
        out[nf], out[nd] = f, d
    return out


def bias_plane(L, params):
    out = np.zeros(L.dims()[0], np.float32)
    if not L.fold:
        for b in L.branches():
            off = L.bg if b else L.ba
            out[perm_rows(L.perm(), L.cout, b)] = np.asarray(params[off:off + L.cout], np.float32)
    return out.view(np.uint32)


def bf16_planes(L, params):
    """{wf_hi, wf_lo, wd_hi, wd_lo, bias} as bit patterns (uint16, bias uint32)"""
    nt_n, cin_k, cin_n, nt_k, _, _ = L.dims()
    parts = {b: Q.split_bf16(kernel(L, params, b)) for b in L.branches()}
    out = _place(L, parts, cin_k, (cin_n, nt_k), (("wf_hi", "wd_hi"), ("wf_lo", "wd_lo")))
    out["bias"] = bias_plane(L, params)
    return out


def e4m3_sat(v):
    """f16f8_ref.e4m3_encode for fp32 v that is not NaN, at the speed a whole model needs: torch's float8_e4m3fn cast (round to nearest
    even) after clamping to +-448, which is the saturation.  Equal to e4m3_encode on the test's sample (test_weight_planes_ref.py)"""
    import torch
    t = torch.from_numpy(np.array(v, np.float32, copy=True))
    return t.clamp_(-Q.E4M3_MAX, Q.E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


_HI_BY_FP16 = None


def quant_w(x):
    """f16f8_ref.quant_planes(x, WGT) as bit patterns (q16 uint16, q8hi, q8lo): the hi plane looked up per fp16 value, whose 65536
    codes come from f16f8_ref's encoder itself"""
    global _HI_BY_FP16
    if _HI_BY_FP16 is None:
        f = np.arange(65536, dtype=np.uint16).view(np.float16).astype(np.float32)
        with np.errstate(invalid="ignore", over="ignore"):
            _HI_BY_FP16 = Q.e4m3_encode(f * np.float32(Q.WGT[0]))
    x = np.asarray(x, np.float32)
    q16 = Q.fp16_rn(x)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = e4m3_sat((x - q16.astype(np.float32)) * np.float32(Q.WGT[1]))
    bits = q16.view(np.uint16)
    return bits, _HI_BY_FP16[bits], lo


def f16f8_planes(L, params, train=True):
    """{wq16, wq8hi, wq8lo, bias} and with train also {wdq16, wdq8hi, wdq8lo} as bit patterns"""
    _, _, cin_n, _, cin_q, nt_q = L.dims()
    parts = {b: quant_w(kernel(L, params, b)) for b in L.branches()}
    out = _place(L, parts, cin_q, (cin_n, nt_q), (("wq16", "wdq16"), ("wq8hi", "wdq8hi"), ("wq8lo", "wdq8lo")))
    if not train:
        for n in QD_PLANES:
            del out[n]
    out["bias"] = bias_plane(L, params)
    return out


def plane_shape(L, name):
    nt_n, cin_k, cin_n, nt_k, cin_q, nt_q = L.dims()
    return {"wf_hi": (L.taps, nt_n, cin_k), "wf_lo": (L.taps, nt_n, cin_k), "wd_hi": (L.taps, cin_n, nt_k), "wd_lo": (L.taps, cin_n, nt_k),
            "wq16": (L.taps, nt_n, cin_q), "wq8hi": (L.taps, nt_n, cin_q), "wq8lo": (L.taps, nt_n, cin_q),
            "wdq16": (L.taps, cin_n, nt_q), "wdq8hi": (L.taps, cin_n, nt_q), "wdq8lo": (L.taps, cin_n, nt_q), "bias": (nt_n,)}[name]


def kept_planes(L, precision, train):
    """the planes an engine of `precision` ('bf16x3', 'bf16' or 'f16f8') keeps current for L"""
    if precision == "f16f8" and L.q_ok():
        return Q_PLANES + (QD_PLANES if train else ()) + ("bias",)
    return BF16_PLANES + ("bias",)


def planes(L, params, precision, train=True):
    if precision == "f16f8" and L.q_ok():
        return f16f8_planes(L, params, train)
    return bf16_planes(L, params)


def decode(name, bits):
    """bit patterns -> float64 values, for messages"""
    bits = np.asarray(bits)
    if name in ("wq16", "wdq16"):
        return bits.astype(np.uint16).view(np.float16).astype(np.float64)
    if name in BF16_PLANES:
        return Q.bf16_decode(bits.astype(np.uint16)).astype(np.float64)
    if name == "bias":
        return bits.astype(np.uint32).view(np.float32).astype(np.float64)
    return Q.e4m3_decode(bits.astype(np.uint8))


def differences(name, got, ref, limit=4):
    """'' if got == ref, else how many elements differ and the first ones: index ([tap, row, column]), bits and values"""
    bad = np.flatnonzero(got.reshape(-1) != ref.reshape(-1))
    if bad.size == 0:
        return ""
    out = []
    for i in bad[:limit]:
        g, r = got.reshape(-1)[i], ref.reshape(-1)[i]
        out.append("element %s got %#x (%r) reference %#x (%r)" % (list(int(v) for v in np.unravel_index(i, ref.shape)), int(g),
                                                                    float(decode(name, g)), int(r), float(decode(name, r))))
    return "%d of %d elements differ: %s" % (bad.size, ref.size, "; ".join(out))


# ---- the stress tier: the edges of the weight window --------------------------------------------------------------------------------
def stress_values():
    """fp32 values at the edges of the weight planes, both signs: +-0; fp16 and bf16 ties; e4m3 ties of the hi plane (fp16(w) * 8)
    and of the lo plane ((w - fp16(w)) * 2^15); the lo plane's clamp edge (|w - fp16(w)| * 2^15 > 448, reached from |w| >= 32 + 448 /
    2^15) and values near 28, where the fp16 residual is at most 2^-7 and the lo plane does not clamp; the hi plane's edge (fp16(w) * 8
    beyond 448 from |w| > 56; values then round to 448 until 464, clamp above); the fp16 edge 65504 / 65520 (fp16 overflow); fp16
    subnormal magnitudes down to the last tie at 2^-25"""
    v = [0.0, 1.0,
         1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 2048 + 1, 2048 + 3,                   # fp16 ties (to even: 1, 1 + 2^-9, 2048, 2052)
         1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, 1 + 2.0 ** -8 + 2.0 ** -23,              # bf16 ties and one just above
         1.0625 / 8, 1.1875 / 8, 50.0, 54.0,                                        # e4m3 ties of fp16(w) * 8 (-> 1, 1.25, 384, 448)
         1 + 1.0625 * 2.0 ** -15, 1 + 1.1875 * 2.0 ** -15,                          # e4m3 ties of the residual * 2^15
         28.0, 28.0 + 2.0 ** -7, 28.0 + 3 * 2.0 ** -7, 31.99, 32.0,
         32.0 + 448 * 2.0 ** -15, 32.0 + 449 * 2.0 ** -15, 32.015, 32.0 + 2.0 ** -6 - 2.0 ** -18, 33.3,
         55.99, 56.0, 56.01, 56.03125, 57.9, 58.0, 60.0, 63.99,
         1000.1, 65504.0, 65519.0, 65519.99, 65520.0, 70000.0,
         2.0 ** -14, 2.0 ** -14 - 2.0 ** -24, 2.0 ** -15, 2.0 ** -20, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -26, 1e-30,
         0.0123, -0.0456]
    a = np.array(v, np.float32)
    a = np.concatenate([a, np.nextafter(a, np.float32(np.inf)), np.nextafter(a, np.float32(0))])
    a = np.concatenate([a, -a, np.array([-0.0], np.float32)])
    return a


def stress_fill(shape, rng):
    """a tensor of `shape` (TF layout, [.., cin, cout] for kernels) whose elements cycle through stress_values() in a shuffled order,
    with the last input channel and the last output channel -- the elements next to the planes' padding -- also taking them"""
    s = stress_values()
    n = int(np.prod(shape))
    out = s[rng.permutation(np.resize(np.arange(s.size), n))].reshape(shape)
    if len(shape) >= 2:
        m = out[..., -1, :].size
        out[..., -1, :] = np.resize(s[::-1], m).reshape(out[..., -1, :].shape)
        m = out[..., -1].size
        out[..., -1] = np.resize(s[::3], m).reshape(out[..., -1].shape)
    return out.astype(np.float32)
