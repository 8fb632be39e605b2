"""The numpy reference of the operand planes (tests/f16f8_ref.py), pinned by hand literals and cross-checked against torch's
float8_e4m3fn cast.  No GPU: test_gpu_planes.py compares the kernels' planes with this reference."""
import numpy as np
import torch

import f16f8_ref as R


def _code(v):
    return int(R.e4m3_encode(np.array([v], np.float32))[0])


def test_e4m3_decode_table_is_float8_e4m3fn():
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float64).numpy()
    assert np.array_equal(np.isnan(codes), np.isnan(R.E4M3_VALUES))
    fin = ~np.isnan(codes)
    assert np.array_equal(codes[fin], R.E4M3_VALUES[fin])
    assert np.flatnonzero(np.isnan(R.E4M3_VALUES)).tolist() == [0x7F, 0xFF]


def test_e4m3_encoder_literals():
    assert _code(448.0) == 0x7E
    assert _code(2.0 ** -6) == 0x08                   # smallest normal
    assert _code(2.0 ** -9) == 0x01                   # smallest subnormal
    assert _code(2.0 ** -10) == 0x00                  # half of it: a tie, to the even code 0
    assert _code(np.nextafter(np.float32(2.0 ** -10), np.float32(1))) == 0x01
    assert _code(3 * 2.0 ** -10) == 0x02              # 1.5 * 2^-9: a tie, to the even code 2
    assert _code(-448.0) == 0xFE and _code(-(2.0 ** -9)) == 0x81
    for v in (449.0, 1e6, np.inf, 3.4e38):
        assert _code(v) == 0x7E, v                    # __NV_SATFINITE: clamp, never NaN
    assert _code(-np.inf) == 0xFE
    assert _code(np.nan) == 0x7F
    assert _code(464.0) == 0x7E and _code(1.0) == 0x38 and _code(1.0625) == 0x38 and _code(1.1875) == 0x3A   # 1 + 1.5/8: tie to even


def test_e4m3_encoder_matches_torch_on_clamped_finite_values():
    rng = np.random.default_rng(0)
    v = np.concatenate([R.log_uniform(200000, rng, -14, 10), R.edge_values(), R.E4M3_VALUES[np.isfinite(R.E4M3_VALUES)],
                        (R._POS[1:] + R._POS[:-1]) / 2]).astype(np.float32)          # the midpoints: every tie
    v = v[np.isfinite(v)]
    v = np.concatenate([v, -v])
    clamped = np.clip(v, -448.0, 448.0).astype(np.float32)
    ref = torch.from_numpy(clamped).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    got = R.e4m3_encode(clamped)
    assert R.same_values(R.e4m3_decode(got), R.e4m3_decode(ref)).all()
    assert np.array_equal(R.e4m3_encode(v), got)      # clamping first changes nothing: the encoder saturates


def test_fp16_literals():
    f = lambda v: float(R.fp16_rn(np.array([v], np.float32))[0])
    assert f(65504.0) == 65504.0
    assert f(65519.0) == 65504.0
    assert np.isinf(f(65520.0)) and f(-65520.0) < 0
    assert f(2.0 ** -24) == 2.0 ** -24
    assert f(2.0 ** -25) == 0.0                       # a tie, to even (zero)
    assert f(3 * 2.0 ** -25) == 2.0 ** -23


def test_bf16_split_matches_torch():
    rng = np.random.default_rng(1)
    x = np.concatenate([R.log_uniform(100000, rng, -120, 120), R.edge_values()]).astype(np.float32)
    hi, lo = R.split_bf16(x)
    t = torch.from_numpy(x)
    th = t.to(torch.bfloat16)
    tl = (t - th.float()).to(torch.bfloat16)
    assert R.same_values(R.bf16_decode(hi), th.float().numpy()).all()
    assert R.same_values(R.bf16_decode(lo), tl.float().numpy()).all()
    fin = np.isfinite(x) & (np.abs(x) < 1e38) & (np.abs(x) > 2.0 ** -100)   # lo stays a normal number
    err = np.abs(x[fin].astype(np.float64) - R.bf16_decode(hi[fin]) - R.bf16_decode(lo[fin]))
    assert np.all(err <= 2.0 ** -17 * np.abs(x[fin]) + 1e-45)


def test_quant_planes_definition():
    x = np.array([1.0 + 2.0 ** -13, 3.0, -1000.0, 2.0 ** -20], np.float32)
    q16, hi, lo = R.quant_planes(x)
    assert q16.tolist() == [1.0, 3.0, -1000.0, 2.0 ** -20]
    assert R.e4m3_decode(hi).tolist() == [1.0, 3.0, -448.0, 0.0]          # hi plane: clamped, flushed
    assert R.e4m3_decode(lo).tolist()[:2] == [0.5, 0.0]                   # residual 2^-13 * 2^12
    q16w, hiw, low = R.quant_planes(x, R.WGT)
    assert R.e4m3_decode(hiw).tolist()[:2] == [8.0, 24.0]
    assert R.e4m3_decode(low).tolist()[0] == 4.0


def test_sat_literals():
    """The sat table: value, fp16(x), the residual scaled by 2^12, counted -- each column checked in fp32 arithmetic."""
    rows = [(448.0, 448.0, 0.0, False), (448.0001, 448.0, 0.375, False), (448.25, 448.25, 0.0, True),
            (384.12, 384.0, 491.5, True), (384.1, 384.0, 409.6, False), (65520.0, np.inf, None, True)]
    for v, f16, res, counted in rows:
        x = np.array([v], np.float32)
        f = R.fp16_rn(x).astype(np.float32)
        assert f[0] == f16, v
        if res is not None:
            r = float(((x - f) * np.float32(4096.0))[0])
            assert abs(r - res) < 0.01 * max(res, 1.0), (v, r)
        assert bool(R.sat_elements(x)[0]) == counted, v
        assert R.sat_count(np.array([v, 0, 0, 0], np.float32)) == int(counted)
    # a group counts once, whichever and however many of its values clamp; NaN and inf count
    assert R.sat_count(np.array([448.25, 448.25, 1, 1, 0, 0, 0, 0, np.nan, 0, 0, 0, 0, 0, 0, -np.inf], np.float32)) == 3
    # 448 is the largest value that does not count: the threshold is inclusive
    assert R.sat_count(np.array([448.0, -448.0, 255.9, 2.0 ** -30], np.float32)) == 0


def test_weight_role_window_edges():
    """Weight-role scales (8, 2^15): no clamp below 32 (hi plane up to 56, lo plane residual <= 2^-7 * 2^15 = 256 below 32), clamps
    from 32 on (residual up to 2^-6)."""
    rng = np.random.default_rng(2)
    w = R.log_uniform(200000, rng, -30, 5)           # |w| < 32
    assert not R.sat_elements(w, R.WGT).any()
    w = np.float32(32.0 + 2.0 ** -6)                 # fp16 ulp 2^-5 at 32: residual 2^-6 * 2^15 = 512 > 448
    assert R.sat_elements(np.array([w]), R.WGT)[0]
    assert R.sat_elements(np.array([56.25], np.float32), R.WGT)[0] and not R.sat_elements(np.array([56.0], np.float32), R.WGT)[0]
