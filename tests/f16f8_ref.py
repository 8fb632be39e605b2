"""numpy reference of the operand planes the CUDA kernels write (csrc/kernels.cuh, csrc/simt_kernels.cu), bit for bit.

F16F8 planes of an fp32 tensor x (cgvc_quant4), element by element:
    q16  = fp16_rn(x)
    q8hi = e4m3(float(q16) * S_hi)
    q8lo = e4m3((x - float(q16)) * S_lo)          the subtraction and both products in fp32
with the activation-role scales (S_hi, S_lo) = (1, 2^12) or the weight-role scales (8, 2^15).  e4m3 is the conversion
__nv_cvt_float2_to_fp8x2(..., __NV_SATFINITE, __NV_E4M3): round to nearest even on the 256 codes of float8 e4m3fn, finite magnitudes
above 448 and +-inf to +-448, NaN to 0x7F; magnitudes <= 2^-10 (half the smallest subnormal, 2^-9) round to zero.  The encoder is
built from the 256 codes themselves, not from any library cast.

cgvc_sat4 counts a group of 4 consecutive values as saturated when for one of them
    !(|fp16(x) * S_hi| <= 448) || !(|(x - fp16(x)) * S_lo| <= 448)            (NaN and inf compare false)

bf16 planes (split_bf16, st4_split): hi = bf16_rn(x), lo = bf16_rn(x - float(hi)).

Planes are compared by decoded value (float64), NaN equal to NaN and -0 equal to +0: the sign of a flushed zero and the payload of a
NaN are not part of the contract.
"""
import numpy as np

ACT = (1.0, 4096.0)          # CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO
WGT = (8.0, 32768.0)         # CGVC_Q_W_SHI, CGVC_Q_W_SLO
E4M3_MAX = 448.0


def _e4m3_decode_table():
    v = np.empty(256, np.float64)
    for code in range(256):
        s, e, m = code >> 7, (code >> 3) & 15, code & 7
        if e == 15 and m == 7:
            mag = np.nan                              # e4m3fn has no inf; S.1111.111 is NaN
        elif e == 0:
            mag = m * 2.0 ** -9                       # subnormals: m/8 * 2^(1-7)
        else:
            mag = (1 + m / 8) * 2.0 ** (e - 7)
        v[code] = -mag if s else mag
    return v


E4M3_VALUES = _e4m3_decode_table()
_POS = E4M3_VALUES[:0x7F]                             # codes 0x00 .. 0x7E: 0 .. 448, increasing with the code
assert np.all(np.diff(_POS) > 0) and _POS[-1] == E4M3_MAX


def e4m3_encode(v):
    """float array -> uint8 e4m3fn codes, round to nearest even, saturating to +-448, NaN -> 0x7F"""
    v = np.asarray(v, np.float64)
    a = np.abs(v)
    fin = np.isfinite(a)
    ac = np.where(fin, np.minimum(a, E4M3_MAX), E4M3_MAX)
    hi = np.clip(np.searchsorted(_POS, ac, side="left"), 0, len(_POS) - 1)     # first code >= |v|
    lo = np.maximum(hi - 1, 0)
    dlo, dhi = ac - _POS[lo], _POS[hi] - ac
    pick_hi = (dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0))                      # tie: the even code (even mantissa)
    code = np.where(pick_hi, hi, lo).astype(np.uint8)
    code = np.where(np.signbit(v), code | 0x80, code).astype(np.uint8)
    return np.where(np.isnan(v), np.uint8(0x7F), code).astype(np.uint8)


def e4m3_decode(codes):
    return E4M3_VALUES[np.asarray(codes, np.uint8)]


def fp16_rn(x):
    """fp32 -> fp16 round to nearest even (overflow to inf), as __float2half_rn"""
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float32).astype(np.float16)


def bf16_rn(x):
    """fp32 -> bf16 bits (uint16), round to nearest even, as __float2bfloat16_rn (NaN stays NaN)"""
    x = np.ascontiguousarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FC0), r).astype(np.uint16)


def bf16_decode(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def split_bf16(x):
    """bf16 hi / lo planes (uint16 bits) of fp32 x"""
    x = np.asarray(x, np.float32)
    hi = bf16_rn(x)
    with np.errstate(invalid="ignore"):
        lo = bf16_rn(x - bf16_decode(hi))
    return hi, lo


def quant_planes(x, scales=ACT):
    """F16F8 planes of fp32 x: (q16 as float16, q8hi codes, q8lo codes), element by element"""
    x = np.asarray(x, np.float32)
    s_hi, s_lo = np.float32(scales[0]), np.float32(scales[1])
    q16 = fp16_rn(x)
    f = q16.astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = e4m3_encode(f * s_hi)
        lo = e4m3_encode((x - f) * s_lo)
    return q16, hi, lo


def sat_elements(x, scales=ACT):
    """per element: its planes clamped or its fp16 value is not finite (the term of cgvc_sat4)"""
    x = np.asarray(x, np.float32)
    s_hi, s_lo = np.float32(scales[0]), np.float32(scales[1])
    f = fp16_rn(x).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = (np.abs(f * s_hi) <= np.float32(E4M3_MAX)) & (np.abs((x - f) * s_lo) <= np.float32(E4M3_MAX))
    return ~ok


def sat_count(x, scales=ACT):
    """cgvc_sat4 summed over the groups of 4 consecutive elements of x (flattened; size a multiple of 4)"""
    bad = sat_elements(np.asarray(x, np.float32).reshape(-1), scales)
    assert bad.size % 4 == 0
    return int(bad.reshape(-1, 4).any(axis=1).sum())


def same_values(a, b):
    """element-wise equality of decoded values: NaN == NaN, -0 == +0"""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return (a == b) | (np.isnan(a) & np.isnan(b))


def assert_same_values(got, ref, what):
    eq = same_values(got, ref)
    if not eq.all():
        i = np.flatnonzero(~eq.reshape(-1))
        g = np.asarray(got, np.float64).reshape(-1); r = np.asarray(ref, np.float64).reshape(-1)
        raise AssertionError("%s: %d of %d values differ, first at flat index %s: got %s, reference %s"
                             % (what, i.size, eq.size, i[:8].tolist(), g[i[:8]].tolist(), r[i[:8]].tolist()))


def edge_values():
    """the window edges of the planes as fp32 values: the literals of the tests, their +-1-ulp neighbours, +-0, NaN, +-inf and fp16
    subnormals, both signs"""
    core = [448.0, 448.0001, 448.25, 384.12, 384.1, 256.0, 224.0, 65504.0, 65520.0, 65519.0, 2.0 ** -6, 2.0 ** -7, 2.0 ** -9, 2.0 ** -10,
            3 * 2.0 ** -10, 2.0 ** -11, 2.0 ** -14, 2.0 ** -15, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 1e-30, 1.0, 1e6]
    c = np.array(core, np.float32)
    nb = np.concatenate([c, np.nextafter(c, np.float32(np.inf)), np.nextafter(c, np.float32(0))])
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], np.float32)
    return np.concatenate([nb, -nb, special]).astype(np.float32)


def log_uniform(n, rng, lo=-30, hi=18):
    """n fp32 values with log2-uniform magnitudes in [2^lo, 2^hi) and random signs"""
    mag = np.exp2(rng.uniform(lo, hi, n))
    return (mag * rng.choice([-1.0, 1.0], n)).astype(np.float32)
