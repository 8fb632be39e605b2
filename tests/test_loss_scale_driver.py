"""train.py --loss_scale: argument parsing and the loss-scaler part of the periodic log line, on the CPU with a stand-in engine."""
import importlib
import sys

import numpy as np
import pytest


def _drv():
    import cgvc  # noqa: F401
    return importlib.import_module("cgvc.train")


def test_loss_scale_is_parsed_and_passed_to_the_model(monkeypatch):
    T = _drv()
    seen = {}
    monkeypatch.setattr(T, "train", lambda *a, **kw: seen.update(kw))
    for argv, want in (([], "static"), (["--loss_scale", "dynamic"], "dynamic"), (["--loss_scale", "monitor"], "monitor")):
        monkeypatch.setattr(sys, "argv", ["train.py", "--synthetic", "4"] + argv)
        T.main()
        assert seen["loss_scale"] == want
    monkeypatch.setattr(sys, "argv", ["train.py", "--loss_scale", "sometimes"])
    with pytest.raises(SystemExit):
        T.main()


def test_log_line_reports_the_scaler(monkeypatch, capsys, tmp_path):
    T = _drv()
    M = importlib.import_module("cgvc.model")
    made = []

    class Stub:
        def __init__(self, num_features, mode='train', **kw):
            self.kw = kw; self.train_step = 0; self.last_loss_scale = None
            made.append(self)

        def train(self, input_A, input_B, lambda_cycle, lambda_identity, generator_learning_rate, discriminator_learning_rate):
            self.train_step += 1
            if self.kw["loss_scale"] != "static":
                self.last_loss_scale = {"scale": 512.0 / self.train_step, "good_steps": 0, "skipped": self.train_step - 1, "last_skipped": True,
                                        "nonfinite": 1 if self.train_step == 2 else 0, "sat_grad": 7, "sat_act": 0}
            return np.float32(1.0), np.float32(0.5)

        def save(self, directory, filename):
            return filename

    monkeypatch.setattr(M, "CycleGAN", Stub)
    T.train(None, None, str(tmp_path / "m"), "x.ckpt", 0, num_epochs=1, mini_batch_size=2, synthetic=5, log_every=1, device_data=False,
            loss_scale="dynamic")
    out = capsys.readouterr().out.splitlines()
    assert made[0].kw["loss_scale"] == "dynamic"
    it = [l for l in out if l.startswith("Iteration")]
    assert len(it) == 2
    assert it[0].endswith("Loss Scale: 512, Skipped Steps: 0, Saturated Groups (gradient / activation): 7 / 0")
    assert it[1].endswith("Loss Scale: 256, Skipped Steps: 1, Saturated Groups (gradient / activation): 7 / 0, Non-finite Gradients")
    T.train(None, None, str(tmp_path / "m"), "x.ckpt", 0, num_epochs=1, mini_batch_size=2, synthetic=5, log_every=1, device_data=False)
    out = capsys.readouterr().out
    assert made[1].kw["loss_scale"] == "static" and "Loss Scale" not in out
