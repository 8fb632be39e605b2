"""The forward / data-gradient gather-GEMM's TMA form: the activation operand as tiled boxes of the source planes.

A dense geometry whose 128-row tiles are boxes of the source planes (128 / Wx whole samples, or 128 positions of one sample, at one
output row) loads its activation tiles by TMA, with the padding and the samples past the batch zero-filled by the hardware; every other
geometry keeps the cp.async gather.  Both fill the stages with the same bytes, so the results are those of tests/gemm_ref.py's emulation
bit for bit in the lattice tier, and within the dense tier's tolerance otherwise.  torch.profiler's kernel names show which form each
launch took (the last template argument of tc_gg_nt_kernel is 1 for the TMA form).
"""
import re

import pytest
import torch

import gemm_ref as G
from parity_util import rel_l2
from test_gpu_gemm_exact import DENSE_TOL, PNAME, _assert_exact, _call, eng  # noqa: F401  (eng: the module's engine fixture)

pytestmark = pytest.mark.gpu

# (name, B, H, W, Cin, kh, kw, Cout, sh, sw): the step's layer shapes at batches that put them on either side of the rule
CASES = [
    ("G.h1", 2, 1, 128, 24, 1, 15, 128, 1, 1),             # one sample per tile, 7 + 7 padding taps
    ("G.d1", 2, 1, 128, 128, 1, 5, 256, 1, 2),             # stride 2: a box strides over 128 source positions for 64 outputs
    ("G.res_h1.tail", 3, 1, 32, 512, 1, 3, 1024, 1, 1),    # 4 samples per box; the last tile's 4th sample is past the batch
    ("G.u2", 2, 1, 64, 512, 1, 5, 512, 1, 1),               # 2 samples per box, left and right padding
    ("G.wide", 1, 1, 256, 128, 1, 5, 128, 1, 1),            # Wx = 256: a box is half a sample
    ("D.d1", 4, 24, 64, 128, 3, 3, 256, 2, 2),              # 2-D, stride 2: a tile is one output row y of 4 samples
    ("D.d2", 8, 12, 32, 256, 3, 3, 512, 2, 2),              # 2-D: 8 samples per box
    ("D.d3", 16, 6, 16, 512, 6, 3, 1024, 1, 2),             # 2-D, 6 x 3 taps, 16 samples of 8 positions per box
    ("D.d1.outside", 2, 24, 64, 128, 3, 3, 256, 2, 2),      # B * Wx = 64: tiles span two output rows -> gather
    ("G.odd_T", 1, 1, 33, 512, 1, 3, 64, 1, 1),             # Wx = 33 divides no tile -> gather
    ("odd.d1", 1, 1, 65, 128, 1, 5, 64, 1, 2),              # forward Wx = 33 -> gather; data-gradient classes 33 (gather), 32 (TMA)
]


def _tma_rule(B, Hy, Wx, sx):
    """the host's choice (tc_gemm.cu nt_tma_maps) for a launch of this geometry"""
    wx = min(Wx, 128)
    return 128 % wx == 0 and Wx % wx == 0 and (Hy == 1 or (B * Wx) % 128 == 0) and wx * sx <= 256


def expected_forms(case):
    """TMA (True) or gather (False) for the forward launch, then each data-gradient parity class in launch order"""
    _, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    out = [_tma_rule(B, -(-H // sh), -(-W // sw), sw)]
    for py in range(sh):
        for px in range(sw):
            Hy, Wx = -(-(H - py) // sh), -(-(W - px) // sw)
            if Hy > 0 and Wx > 0:
                out.append(_tma_rule(B, Hy, Wx, 1))
    return out


def test_rule_covers_both_forms():
    forms = [f for c in CASES for f in expected_forms(c)]
    assert any(forms) and not all(forms)
    assert expected_forms(("odd.d1", 1, 1, 65, 128, 1, 5, 64, 1, 2)) == [False, False, True]


def _nt_forms(prof):
    """TMA flag of every tc_gg_nt_kernel launch in the trace, in launch order"""
    evs = [e for e in prof.events() if "tc_gg_nt_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    out = []
    for e in evs:
        m = re.search(r"tc_gg_nt_kernel<(\d+), (\d+), (\d+), (\d+), (\d+)>", e.name)
        assert m, e.name
        out.append(m.group(5) == "1")
    return out


PARAMS = [(c, p) for c in CASES for p in (G.BF16X3, G.F16F8) if G.supports(c, p)]


@pytest.mark.parametrize("case,prec", PARAMS, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in PARAMS])
def test_lattice_bit_exact_and_form(eng, case, prec):  # noqa: F811
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    ref = G.emulate(case, prec, x, w, b, dy, w16=0, device="cuda", P=P)
    got = _call(eng, case, prec, x, w, b, dy, 0, launches=True)
    for key in ("y", "dx", "dw", "db"):
        _assert_exact(case, prec, key, got[key], ref[key])
    # the profiler may drop the first kernel records of a session: the second of two calls must show every launch's form
    from torch.profiler import ProfilerActivity, profile
    want = expected_forms(case)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            _call(eng, case, prec, x, w, b, dy, 0)
    seen = _nt_forms(prof)
    assert len(seen) >= len(want) and seen[-len(want):] == want, (case[0], seen, want)


DENSE = [(c, G.F16F8) for c in CASES if G.supports(c, G.F16F8)]


@pytest.mark.parametrize("case,prec", DENSE, ids=["%s-%s" % (c[0], PNAME[p]) for c, p in DENSE])
def test_dense_close_and_deterministic(eng, case, prec):  # noqa: F811
    x, w, b, dy = G.dense_case(case)
    P = G.case_planes(prec, x, w, dy)
    ref = G.emulate(case, prec, x, w, b, dy, w16=1, device="cuda", P=P)
    first = _call(eng, case, prec, x, w, b, dy, 1)
    for k in ("y", "dx", "dw"):
        assert rel_l2(first[k].cpu(), ref[k].cpu()) <= DENSE_TOL[prec], (case[0], k)
    again = _call(eng, case, prec, x, w, b, dy, 1)
    for k in ("y", "dx"):
        assert torch.equal(first[k], again[k]), (case[0], k, "not deterministic")
