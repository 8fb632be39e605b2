"""train.py --deterministic: argument parsing and the flag reaching both models the driver builds, on the CPU with a stand-in engine."""
import importlib
import sys

import numpy as np


def _drv():
    import cgvc  # noqa: F401
    return importlib.import_module("cgvc.train")


def test_deterministic_is_parsed(monkeypatch):
    T = _drv()
    seen = {}
    monkeypatch.setattr(T, "train", lambda *a, **kw: seen.update(kw))
    for argv, want in (([], False), (["--deterministic"], True)):
        monkeypatch.setattr(sys, "argv", ["train.py", "--synthetic", "4"] + argv)
        T.main()
        assert seen["deterministic"] is want


def test_deterministic_reaches_the_training_and_validation_models(monkeypatch, tmp_path):
    T = _drv()
    M = importlib.import_module("cgvc.model")
    made = []

    class Stub:
        def __init__(self, num_features, mode='train', **kw):
            self.mode = mode; self.kw = kw; self.train_step = 0; self.last_loss_scale = None
            made.append(self)

        def train(self, input_A, input_B, lambda_cycle, lambda_identity, generator_learning_rate, discriminator_learning_rate):
            self.train_step += 1
            return np.float32(1.0), np.float32(0.5)

        def save(self, directory, filename):
            return filename

    monkeypatch.setattr(M, "CycleGAN", Stub)
    monkeypatch.setattr(T, "validation_conversions", lambda *a, **kw: None)
    for det in (True, False):
        made.clear()
        T.train(None, None, str(tmp_path / "m"), "x.ckpt", 0, num_epochs=1, mini_batch_size=2, synthetic=5, log_every=1,
                device_data=False, validation_A_dir=str(tmp_path), deterministic=det)
        assert [m.mode for m in made] == ["train", "test"]
        assert all(m.kw["deterministic"] is det for m in made)
