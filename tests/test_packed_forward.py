"""Packed variable-length generator forward (cgvc_generator_forward_packed / CycleGAN.test_packed): utterances of different
lengths in one call give each utterance what the float64 oracle and test() give for it alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from parity_util import rel_l2

pytestmark = pytest.mark.gpu

# boundaries fall mid-tile at every level (T, T/2, T/4)
LENGTHS = [36, 516, 128, 784, 132, 1400, 64]
ERR_ARG = -1                                           # CGVC_ERR_ARG (include/cgvc.h)
TAPS = {"h1_glu": 1, "d1": 2, "d2": 4, "r1": 4, "r2": 4, "r3": 4, "r4": 4, "r5": 4, "r6": 4, "u1": 2, "u2": 1}


def _utterances(seed, lengths):
    from oracle import cyclegan_oracle as O
    return [O.synthetic_batch(seed=seed + i, batch=1, frames=T, dtype=torch.float64)[0][0].numpy() for i, T in enumerate(lengths)]


def _model(oracle_params64, prec, max_batch=8, max_frames=512):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='test', max_batch=max_batch, max_frames=max_frames, precision=prec)
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    return m


def _split_tap(flat, lengths, div):
    rows = np.cumsum([0] + [T // div for T in lengths])
    v = flat.reshape(rows[-1], -1)
    return [v[rows[u]:rows[u + 1]] for u in range(len(lengths))]


@pytest.fixture(scope="module")
def oracle_refs(oracle_params64):
    from oracle import cyclegan_oracle as O
    xs = _utterances(100, LENGTHS)
    refs = {}
    for scope, d in (("generator_A2B", "A2B"), ("generator_B2A", "B2A")):
        out = []
        for x in xs:
            taps = {}
            y = O.generator_forward(torch.from_numpy(x[None]), oracle_params64, scope, taps)
            out.append((y[0].numpy(), {k: taps[k].numpy().reshape(-1) for k in TAPS}))
        refs[d] = out
    return xs, refs


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "f16f8"])
def test_packed_matches_oracle(oracle_params64, oracle_refs, prec):
    xs, refs = oracle_refs
    m = _model(oracle_params64, prec)
    m.set_debug_taps(True)
    for edge in (1, 0):
        m.set_option("edge_lower", edge)
        for d in ("A2B", "B2A"):
            ys = m.test_packed(xs, d)
            got_taps = {k: _split_tap(m.debug_activation(k), LENGTHS, div) for k, div in TAPS.items()}
            worst = 0.0
            for u, (y, (y_ref, taps_ref)) in enumerate(zip(ys, refs[d])):
                assert y.shape == (24, LENGTHS[u]) and y.dtype == np.float32
                e = rel_l2(y, y_ref); worst = max(worst, e)
                assert e < 1e-3, (prec, edge, d, u, "out", e)
                for k in TAPS:
                    e = rel_l2(got_taps[k][u].reshape(-1), taps_ref[k]); worst = max(worst, e)
                    assert e < 1e-3, (prec, edge, d, u, k, e)
            print("packed[%s, edge_lower=%d, %s] worst rel_l2 vs oracle %.2e" % (prec, edge, d, worst))


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16", "f16f8"])
def test_packed_matches_test(oracle_params64, prec):
    """Each utterance == test() on it alone; includes 4, 8 and 12 frames (shorter than the 15-tap halo, 1-3 rows at T/4).  Lengths for
    which test() takes a specialised instance-norm kernel (convert._special_norm_length: 64, 128, 512, ...) sum in another order and
    are covered by the oracle test instead."""
    lengths = [4, 516, 8, 132, 12, 68, 1400, 200]
    xs = _utterances(200, lengths)
    m = _model(oracle_params64, prec)
    for edge in (1, 0):
        m.set_option("edge_lower", edge)
        for d in ("A2B", "B2A"):
            ys = m.test_packed(xs, d)
            for u, (x, y) in enumerate(zip(xs, ys)):
                e = rel_l2(y, m.test(x[None], d)[0])
                assert e < 1e-5, (prec, edge, d, lengths[u], e)


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_packed_invariance(oracle_params64, prec):
    m = _model(oracle_params64, prec)
    xs = _utterances(300, LENGTHS)
    ys = m.test_packed(xs, "A2B")
    perm = [5, 0, 3, 6, 1, 4, 2]
    yp = m.test_packed([xs[i] for i in perm], "A2B")
    for j, i in enumerate(perm):
        assert rel_l2(yp[j], ys[i]) < 1e-6, (i, rel_l2(yp[j], ys[i]))
    again = m.test_packed(xs, "A2B")
    assert all(np.array_equal(a, b) for a, b in zip(ys, again))            # deterministic
    # n equal-length utterances == the [n, 24, T] batch through test()
    xb = np.stack(_utterances(400, [132] * 5))
    yb = m.test(xb, "B2A")
    for u, y in enumerate(m.test_packed(list(xb), "B2A")):
        assert rel_l2(y, yb[u]) < 1e-5
    # CUDA tensors in, CUDA tensors out
    yd = m.test_packed([torch.from_numpy(x).cuda() for x in xs[:3]], "A2B")
    assert all(t.is_cuda and t.dtype == torch.float32 for t in yd)
    for u in range(3):
        assert rel_l2(yd[u].cpu().numpy(), ys[u]) < 1e-6


def test_packed_errors_and_growth(oracle_params64):
    import cgvc
    from cgvc import _native as N
    m = _model(oracle_params64, "bf16x3", max_batch=4, max_frames=128)
    lib, h = m._lib, m._handle
    x = torch.zeros(24 * 512, device="cuda"); y = torch.empty_like(x)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(offs, n=None, direction=0):
        o = np.asarray(offs, dtype=np.int64)
        return lib.cgvc_generator_forward_packed(h, direction, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()),
                                                 o.ctypes.data_as(C.POINTER(C.c_longlong)), len(o) - 1 if n is None else n, st)

    def msg():
        return lib.cgvc_last_error(h).decode()

    assert call([0, 64, 130]) == ERR_ARG and "utterance 1" in msg()       # 66 frames: not a multiple of 4
    assert call([0, 64, 64, 128]) == ERR_ARG and "utterance 1" in msg()   # zero length
    assert call([0, 128, 64]) == ERR_ARG and "utterance 1" in msg()       # decreasing offsets
    assert call([0, 4, 8, 12, 16, 20]) == ERR_ARG                          # n = 5 > max_batch = 4
    assert call([0, 256, 516]) == ERR_ARG                                  # 516 frames > 4 x 128
    assert call([0, 64], direction=2) == N.ERR_DIRECTION
    assert call([0, 64, 192]) == 0                                         # the engine is still usable
    torch.cuda.synchronize()
    xs = _utterances(600, [68, 132, 36])
    for x, yy in zip(xs, m.test_packed(xs, "B2A")):
        assert rel_l2(yy, m.test(x[None], "B2A")[0]) < 1e-5
    with pytest.raises(Exception, match="Conversion direction must be specified."):
        m.test_packed([np.zeros((24, 8))], "A2A")
    with pytest.raises(cgvc._native.CgvcError):
        m.test_packed([np.zeros((24, 6))], "A2B")
    # test_packed grows the engine for a call over its capacity
    xs = _utterances(500, [1400, 516, 132, 12, 784])
    ys = m.test_packed(xs, "A2B")
    for x, yy in zip(xs, ys):
        assert rel_l2(yy, m.test(x[None], "A2B")[0]) < 1e-5
