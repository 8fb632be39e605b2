"""convert.py host logic with a model that has test_packed (CPU): chunking of utterances of any lengths, crop, (de)normalisation."""
import importlib

import numpy as np
import pytest


def _convert():
    import cgvc  # noqa: F401
    return importlib.import_module("cgvc.convert")


class _PackedAffineModel:
    """stand-in for CycleGAN.test_packed: y = 2x + 1 per utterance, records the calls and the capacity requests"""

    def __init__(self):
        self.calls, self.capacity = [], []

    def test_packed(self, inputs, direction):
        if direction not in ("A2B", "B2A"):
            raise Exception('Conversion direction must be specified.')
        assert all(x.ndim == 2 and x.shape[0] == 24 and x.shape[1] % 4 == 0 for x in inputs)
        self.calls.append(([x.shape[1] for x in inputs], direction))
        return [(2.0 * x + 1.0).astype(np.float32) for x in inputs]

    def test(self, inputs, direction):
        raise AssertionError("a model with test_packed is not called through test()")

    def _ensure_capacity(self, batch, frames):
        self.capacity.append((batch, frames))


def _stats(rs):
    return {"mean_A": rs.randn(24, 1), "std_A": rs.rand(24, 1) + 0.5, "mean_B": rs.randn(24, 1), "std_B": rs.rand(24, 1) + 0.5}


def test_plan_chunks_bounds():
    Cv = _convert()
    assert Cv.plan_chunks([400] * 7, max_group=3, frame_budget=10000) == [[0, 1, 2], [3, 4, 5], [6]]
    assert Cv.plan_chunks([600, 500, 700, 300], max_group=8, frame_budget=1200) == [[0, 1], [2, 3]]
    # an utterance over the budget gets a chunk of its own
    assert Cv.plan_chunks([200, 5000, 200, 200], max_group=8, frame_budget=1000) == [[0], [1], [2, 3]]
    assert Cv.plan_chunks([], max_group=8, frame_budget=1000) == []
    assert [T for T in range(4, 2000, 4) if Cv._special_norm_length(T)] == [32, 48, 64, 96, 128, 192, 256, 384, 512, 768, 1536]


def test_convert_features_keeps_fused_lengths_on_test():
    """padded lengths whose single-utterance forward takes a specialised instance-norm kernel go through test(), the rest packed"""
    Cv = _convert()
    rs = np.random.RandomState(6)
    st = _stats(rs)

    class Both(_PackedAffineModel):
        def test(self, inputs, direction):
            self.calls.append((("test",) + inputs.shape, direction))
            return (2.0 * inputs + 1.0).astype(np.float32)

    m = Both()
    utts = [rs.randn(n, 24) for n in (128, 400, 510, 127)]                 # padded 128, 400, 512, 128
    out = Cv.convert_features(m, utts, "A2B", st)
    assert m.calls == [([400], "A2B"), (("test", 1, 24, 512), "A2B"), (("test", 2, 24, 128), "A2B")]
    x = np.pad(utts[2].T, ((0, 0), (1, 1)), mode="edge")
    want = ((2.0 * ((x - st["mean_A"]) / st["std_A"]) + 1.0).astype(np.float32).astype(np.float64) * st["std_B"] + st["mean_B"]).T
    assert np.allclose(out[2], want[1:511], rtol=1e-6, atol=1e-6)


def test_convert_features_packed_chunks_crop_and_denormalise():
    Cv = _convert()
    rs = np.random.RandomState(5)
    st = _stats(rs)
    lens = [130, 401, 57, 1398, 260, 9]                                    # padded 132, 404, 60, 1400, 260, 12
    utts = [rs.randn(n, 24) for n in lens]
    m = _PackedAffineModel()
    out = Cv.convert_features(m, utts, "A2B", st, max_group=3, frame_budget=1000)
    assert [c[0] for c in m.calls] == [[132, 404, 60], [1400], [260, 12]]
    assert all(c[1] == "A2B" for c in m.calls)
    assert m.capacity == [(3, 468)]                                        # sized once: 3 utterances, 1400 frames in one chunk
    for u, o in zip(utts, out):
        T = u.shape[0]; Tp = -(-T // 4) * 4; left = (Tp - T) // 2
        assert o.shape == (T, 24) and o.flags["C_CONTIGUOUS"]
        x = np.pad(u.T, ((0, 0), (left, Tp - T - left)), mode="edge")
        want = ((2.0 * ((x - st["mean_A"]) / st["std_A"]) + 1.0).astype(np.float32).astype(np.float64) * st["std_B"] + st["mean_B"]).T
        assert np.allclose(o, want[left:left + T], rtol=1e-6, atol=1e-6)
    out2 = Cv.convert_features(_PackedAffineModel(), utts[:1], "B2A", st)
    x = np.pad(utts[0].T, ((0, 0), (1, 1)), mode="edge")
    want = ((2.0 * ((x - st["mean_B"]) / st["std_B"]) + 1.0).astype(np.float32).astype(np.float64) * st["std_A"] + st["mean_A"]).T
    assert np.allclose(out2[0], want[1:131], rtol=1e-6, atol=1e-6)
    with pytest.raises(Exception, match="Conversion direction must be specified."):
        Cv.convert_features(m, utts, "A2A", st)
