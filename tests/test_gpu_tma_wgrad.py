"""The weight-gradient gather-GEMM's TMA form: the activation operand as boxes of whole output rows of the source planes.

A dense geometry whose 64-row stages are boxes of the source planes (64 / Wx whole output rows, or 64 positions of one output row,
with Wx >= 8) loads its X tiles by TMA, the padding, the samples past the batch and the channels past the plane's width zero-filled by
the hardware; every other launch keeps the cp.async gather: geometries outside the rule, the packed forms, and F16F8 with
`wgrad_f16 = 0` (whose producers widen the e4m3 planes to fp16).  Both fill the stages with the same bytes, so dW and db are those of
tests/gemm_ref.py's emulation bit for bit in the lattice tier, split-K partials and deterministic mode included, and within the dense
tier's tolerance otherwise.  torch.profiler's kernel names show which form each launch took (the last template argument of
tc_gg_tn_kernel is 1 for the TMA form); `tn_tma_rule` mirrors the host's choice (tc_gemm.cu tn_tma_maps).
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import gemm_ref as G
from parity_util import rel_l2
from test_gpu_gemm_exact import DENSE_TOL, PNAME, _assert_exact, _call, _p, eng  # noqa: F401  (eng: the module's engine fixture)


def tn_tma_rule(Wx, sx):
    """tc_gemm.cu tn_tma_maps for a dense launch of output width Wx and stride sx: None (gather), else the stage's boxes as
    (K-rows per box, boxes per stage, samples per box)"""
    wx = min(Wx, 64)
    if Wx < 8 or 64 % wx or Wx % wx or wx * sx > 256 or sx > 8:
        return None
    return wx, 64 // wx, 64 // wx


def tn_stage_boxes(Hy, Wx, sx):
    """the boxes of one stage as the kernel issues them: (K-rows per box, boxes per stage, samples per box), or None (gather)"""
    r = tn_tma_rule(Wx, sx)
    if r is None:
        return None
    wx = r[0]
    return (64, 1, 64 // wx) if Hy == 1 or Wx >= 64 else (wx, 64 // wx, 1)


# the weight-gradient launches of one bench.py step (batch 256 x [24, 128], f16f8, wgrad_f16 = 1): (layer, Hy, Wx, sx) and the stage
# as DESIGN.md section 5 describes it: (K-rows per box, boxes per stage, samples per box)
BENCH_TN = [
    ("G.h1 (im2col)", 1, 128, 1, (64, 1, 1)),     # 64 positions of one sample
    ("G.d1", 1, 64, 2, (64, 1, 1)),               # one sample
    ("G.d2", 1, 32, 2, (64, 1, 2)),               # two samples
    ("G.res h1 / h2", 1, 32, 1, (64, 1, 2)),
    ("G.u1", 1, 32, 1, (64, 1, 2)),
    ("G.u2", 1, 64, 1, (64, 1, 1)),
    ("G.o1 (folded)", 1, 128, 1, (64, 1, 1)),
    ("D.d1", 12, 32, 2, (32, 2, 1)),              # 2 output rows of one sample
    ("D.d2", 6, 16, 2, (16, 4, 1)),               # 4 output rows; 96 rows per sample, so stages straddle samples
    ("D.d3", 6, 8, 2, (8, 8, 1)),                 # 8 output rows; 48 rows per sample
]


def test_rule_mirror_matches_the_step_table():
    for name, Hy, Wx, sx, stage in BENCH_TN:
        assert tn_stage_boxes(Hy, Wx, sx) == stage, name
        rows, nbox, _ = stage
        assert rows * nbox == 64 and (rows * 128) % 1024 == 0, name     # every box on a 1024-byte boundary of the stage
    # just outside: too narrow for a 1024-byte-aligned box, a width that 64 neither divides nor is divided by
    for Wx in (4, 33, 96, 65):
        assert tn_tma_rule(Wx, 1) is None, Wx
    assert tn_tma_rule(8, 2) is not None and tn_tma_rule(128, 2) is not None


# (name, B, H, W, Cin, kh, kw, Cout, sh, sw)
CASES = [
    ("G.h1.im2col", 2, 1, 128, 360, 1, 1, 256, 1, 1),        # Wx 128: 64 positions of one sample per stage; 3 channel tiles
    ("G.h1", 2, 1, 128, 24, 1, 15, 128, 1, 1),               # Cin 24: (bf16) the second channel atom lies past x_ld; 7 + 7 pad taps
    ("G.d1", 2, 1, 128, 128, 1, 5, 256, 1, 2),               # Wx 64, stride 2: a box strides over 128 source positions
    ("G.d2", 2, 1, 64, 256, 1, 5, 512, 1, 2),                # Wx 32, stride 2: two samples per box
    ("G.res.tail", 3, 1, 32, 512, 1, 3, 1024, 1, 1),         # M 96: the last stage's second sample is past the batch
    ("G.u2", 2, 1, 64, 512, 1, 5, 512, 1, 1),                # one sample per stage, padding on both sides
    ("G.o1.ntail", 2, 1, 128, 256, 1, 1, 360, 1, 1),         # N 360: the second column tile is partly past the real columns
    ("D.d1", 2, 24, 64, 128, 3, 3, 256, 2, 2),               # Hy 12, Wx 32, stride 2: two output-row boxes per stage
    ("D.d2", 2, 12, 32, 256, 3, 3, 512, 2, 2),               # Hy 6, Wx 16: stages straddle samples
    ("D.d3.tail", 5, 6, 16, 512, 6, 3, 1024, 1, 2),          # Hy 6, Wx 8: 8 boxes per stage, straddling; M 240: last stage past B
    ("split.empty", 385, 1, 64, 64, 1, 1, 64, 1, 1),         # split-K 24 at 132 SMs: an uneven item and an empty one
    ("out.Wx4", 8, 1, 4, 64, 1, 3, 64, 1, 1),                # Wx 4 -> gather
    ("out.Wx33", 2, 1, 33, 128, 1, 3, 128, 1, 1),            # Wx 33 -> gather
    ("out.Wx96", 2, 1, 96, 128, 1, 3, 128, 1, 1),            # Wx 96 -> gather
]


def _geom(case):
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    return B, -(-H // sh), -(-W // sw), sw


def expected_tma(case, prec, w16):
    """TMA (True) or gather (False) for the case's weight-gradient launch"""
    _, Hy, Wx, sx = _geom(case)
    return tn_tma_rule(Wx, sx) is not None and (prec != G.F16F8 or bool(w16))


def test_cases_cover_both_forms_and_split_k():
    forms = [expected_tma(c, G.BF16X3, 0) for c in CASES]
    assert any(forms) and not all(forms)
    L = G.case_launches([c for c in CASES if c[0] == "split.empty"][0], G.BF16, 0, 132)["wgrad"]
    assert L["ksplit"] > 1 and L["uneven"] and L["empty"], L
    # the second channel atom out of bounds (bf16 x_ld 64), and rows past M in the last stage
    assert any(-(-c[4] // 64) * 64 % 128 for c in CASES if expected_tma(c, G.BF16, 0))
    assert any((c[1] * _geom(c)[1] * _geom(c)[2]) % 64 for c in CASES if expected_tma(c, G.BF16, 0))


def _tn_forms(prof):
    """TMA flag of every tc_gg_tn_kernel launch in the trace, in launch order"""
    evs = [e for e in prof.events() if "tc_gg_tn_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    out = []
    for e in evs:
        m = re.search(r"tc_gg_tn_kernel<(\d+), (\d+), (\d+), (\d+), (\d+)>", e.name)
        assert m, e.name
        out.append((int(m.group(4)), m.group(5) == "1"))
    return out


def _check_form(eng, case, prec, x, w, b, dy, w16):
    from torch.profiler import ProfilerActivity, profile
    # the profiler may drop the first kernel records of a session: the last of two calls must show the launch's form
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            _call(eng, case, prec, x, w, b, dy, w16)
    seen = _tn_forms(prof)
    assert seen and seen[-1] == (0, expected_tma(case, prec, w16)), (case[0], prec, w16, seen)


LATTICE = [(c, p) for c in CASES for p in (G.BF16X3, G.BF16, G.F16F8) if G.supports(c, p)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec", LATTICE, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in LATTICE])
def test_lattice_bit_exact_and_form(eng, case, prec):  # noqa: F811
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    for w16 in ((1, 0) if prec == G.F16F8 else (0,)):
        cert = G.certificate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P, forms=("wgrad", "db"))
        for form, phase, largest, bound in cert:
            assert largest < bound, (case[0], prec, w16, form, phase, largest, bound)
        ref = G.emulate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P, forms=("wgrad",))
        got = _call(eng, case, prec, x, w, b, dy, w16, launches=True)
        for key in ("dw", "db"):
            _assert_exact(case, prec, key, got[key], ref[key])
        _check_form(eng, case, prec, x, w, b, dy, w16)


DENSE = [(c, p) for c in CASES for p in (G.BF16X3, G.F16F8) if G.supports(c, p) and expected_tma(c, p, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec", DENSE, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in DENSE])
def test_dense_close(eng, case, prec):  # noqa: F811
    x, w, b, dy = G.dense_case(case)
    P = G.case_planes(prec, x, w, dy)
    ref = G.emulate(case, prec, x, w, b, dy, w16=1, device="cuda", P=P, forms=("wgrad",))
    got = _call(eng, case, prec, x, w, b, dy, 1)
    err = rel_l2(got["dw"].cpu(), ref["dw"].cpu())
    assert err <= DENSE_TOL[prec], (case[0], prec, err)


@pytest.fixture(scope="module")
def det_eng():
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    assert lib.cgvc_set_option(h, b"deterministic", 1) == 0
    keep = {}
    for kind in (N.ARENA_PARAM, N.ARENA_WORK):
        nb = C.c_size_t(0)
        assert lib.cgvc_arena_bytes(h, kind, C.byref(nb)) == 0
        keep[kind] = torch.empty((nb.value + 3) // 4, dtype=torch.float32, device="cuda")
        assert lib.cgvc_bind_arena(h, kind, C.c_void_p(keep[kind].data_ptr()), nb.value) == 0
    yield lib, h, N
    lib.cgvc_destroy(h)


DET = [(c, p) for c in CASES if c[0] in ("split.empty", "G.res.tail", "D.d3.tail", "out.Wx33") for p in (G.BF16X3, G.F16F8)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,prec", DET, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in DET])
def test_deterministic_bit_exact_and_form(det_eng, case, prec):
    lib, h, N = det_eng
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    xd, wd, dyd = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in (x, w, dy))
    from torch.profiler import ProfilerActivity, profile
    for w16 in ((1, 0) if prec == G.F16F8 else (0,)):
        ref = G.emulate(case, prec, x, w, b, dy, w16=w16, device="cuda", P=P, forms=("wgrad",))
        assert lib.cgvc_set_option(h, b"wgrad_f16", w16) == 0
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(2):
                    dw = torch.zeros_like(wd); db = torch.zeros(Cout, device="cuda")
                    N.check(h, lib.cgvc_conv_backward(h, prec, _p(xd), _p(wd), _p(dyd), None, _p(dw), _p(db), B, H, W, Cin, kh, kw, Cout,
                                                      sh, sw, None))
                    torch.cuda.synchronize()
                    assert torch.equal(dw.double().cpu().reshape(-1), torch.as_tensor(ref["dw"]).cpu().reshape(-1)), (name, w16)
                    assert torch.equal(db.double().cpu().reshape(-1), torch.as_tensor(ref["db"]).cpu().reshape(-1)), (name, w16)
        finally:
            assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0
        seen = _tn_forms(prof)
        assert seen and seen[-1] == (0, expected_tma(case, prec, w16)), (name, prec, w16, seen)


@pytest.mark.gpu
def test_packed_weight_gradients_gather():
    """the packed generator's convolutions take the packed weight gradient, which gathers (its tap-lowered edge layers contract
    over im2col rows that are already packed: those are dense launches and follow the rule)"""
    import cgvc
    from torch.profiler import ProfilerActivity, profile
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision="bf16x3", log_dir='/tmp/cgvc_log')
    g = torch.Generator(device="cuda").manual_seed(5)
    xs = [torch.randn(24, T, device="cuda", generator=g).requires_grad_(True) for T in (64, 128)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            sum(y.sum() for y in m.generator_packed(xs, "A2B")).backward()
            torch.cuda.synchronize()
    packed = [ta for pk, ta in _tn_forms(prof) if pk > 0]
    assert packed and not any(packed), packed
