"""Engine options belong to their handle: setting one on an engine changes what that engine launches and nothing another engine in the
process does, and a captured step is never replayed with the options it was captured under once they have changed."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# options that select other kernels, with a value that is not their default
CHANGED = {"prep_batched": 0, "post_onepass": 0, "post_stream": 0, "tc_debug": 1}


def _model(params, det=True, **opts):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision="f16f8", seed=11,
                      log_dir='/tmp/cgvc_log', deterministic=det)
    m.set_params({k: v.numpy() for k, v in params.items()})
    for k, v in opts.items():
        m.set_option(k, v)
    return m


def _inputs():
    rs = np.random.RandomState(17)
    return rs.randn(2, 24, 128), rs.randn(2, 24, 128)


def _step_launches(m, A, B):
    """Kernels launched by one cgvc_train_step of m (the counter is process-wide: nothing else runs meanwhile)."""
    before, after = C.c_ulonglong(0), C.c_ulonglong(0)
    m._lib.cgvc_kernel_launches(C.byref(before))
    m.train(A, B, 10.0, 5.0, 2e-4, 1e-4)
    m._lib.cgvc_kernel_launches(C.byref(after))
    return after.value - before.value


def _record(m, params, A, B):
    """(launches of one eager train step, losses, GRAD) of m: the gradients of a deterministic cgvc_compute_gradients call on `params`."""
    from cgvc import native as N
    m.set_params({k: v.numpy() for k, v in params.items()})
    losses, _, _ = m.compute_gradients(A, B, 10.0, 5.0)
    end = max(o + int(np.prod(s)) for o, s in m._table.values())
    grad = m._arenas[N.ARENA_GRAD][:end].cpu()
    return _step_launches(m, A, B), losses, grad


def test_options_belong_to_their_handle(oracle_params64):
    A, B = _inputs()
    ea = _model(oracle_params64, det=False)
    eb = _model(oracle_params64, cuda_graph=0)
    a_before = _step_launches(ea, A, B)
    ref = _record(eb, oracle_params64, A, B)
    for k, v in CHANGED.items():
        ea.set_option(k, v)
    a_after = _step_launches(ea, A, B)
    ec = _model(oracle_params64, cuda_graph=0)
    for name, m in (("B", eb), ("C", ec)):
        got = _record(m, oracle_params64, A, B)
        assert got[0] == ref[0], (name, got[0], ref[0])
        assert got[1] == ref[1], (name, got[1], ref[1])
        assert torch.equal(got[2], ref[2]), (name, int((got[2] != ref[2]).sum()))
    assert a_after != a_before, (a_before, a_after)
    print("launches per step: A %d -> %d with %s; B and C %d" % (a_before, a_after, CHANGED, ref[0]))


def test_changed_options_are_never_replayed_stale(oracle_params64):
    A, B = _inputs()
    m = _model(oracle_params64, det=False)

    def eager_launches():
        m.set_option("cuda_graph", 0)
        n = _step_launches(m, A, B)
        m.set_option("cuda_graph", 1)
        return n

    default = eager_launches()
    assert _step_launches(m, A, B) == default               # captures the step
    assert _step_launches(m, A, B) == default               # replays it
    for name, value, back in (("two_streams", 0, 1), ("fuse_in", 0, 1), ("edge_lower", 0, 1), ("post_onepass", 0, 1),
                              ("prep_batched", 0, 1), ("tc_debug", 1, 0)):
        m.set_option(name, value)
        got = _step_launches(m, A, B)
        want = eager_launches()
        assert got == want, (name, value, got, want)
        m.set_option(name, back)
        got = _step_launches(m, A, B)
        assert got == default, (name, back, got, default)
        print("%s = %d: %d launches per step (default options %d)" % (name, value, want, default))
