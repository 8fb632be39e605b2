"""train.py --loss_scale_per_network: argument parsing and the per-network part of the periodic log line, on the CPU with a stand-in
engine."""
import importlib
import sys

import numpy as np


def _drv():
    import cgvc  # noqa: F401
    return importlib.import_module("cgvc.train")


def test_flag_is_parsed_and_passed_to_the_model(monkeypatch):
    T = _drv()
    seen = {}
    monkeypatch.setattr(T, "train", lambda *a, **kw: seen.update(kw))
    for argv, want in (([], False), (["--loss_scale", "dynamic", "--loss_scale_per_network"], True)):
        monkeypatch.setattr(sys, "argv", ["train.py", "--synthetic", "4"] + argv)
        T.main()
        assert seen["loss_scale_per_network"] is want


def test_log_line_reports_both_networks(monkeypatch, capsys, tmp_path):
    T = _drv()
    M = importlib.import_module("cgvc.model")
    made = []

    class Stub:
        def __init__(self, num_features, mode='train', **kw):
            self.kw = kw; self.train_step = 0; self.last_loss_scale = None
            made.append(self)

        def train(self, input_A, input_B, lambda_cycle, lambda_identity, generator_learning_rate, discriminator_learning_rate):
            self.train_step += 1
            self.last_loss_scale = {"scale": 512.0 / self.train_step, "good_steps": 0, "skipped": self.train_step - 1,
                                    "last_skipped": True, "nonfinite": 0, "sat_grad": 7, "sat_act": 0}
            if self.kw["loss_scale_per_network"]:
                self.last_loss_scale.update({"scale_G": 512.0 / self.train_step, "scale_D": 512.0, "sat_grad_G": 7, "sat_grad_D": 0,
                                             "ufl_grad_G": 3, "ufl_grad_D": 250, "groups_G": 1000, "groups_D": 1000,
                                             "good_steps_G": 0, "good_steps_D": self.train_step})
            return np.float32(1.0), np.float32(0.5)

        def save(self, directory, filename):
            return filename

    monkeypatch.setattr(M, "CycleGAN", Stub)
    T.train(None, None, str(tmp_path / "m"), "x.ckpt", 0, num_epochs=1, mini_batch_size=2, synthetic=5, log_every=1, device_data=False,
            loss_scale="dynamic", loss_scale_per_network=True)
    out = capsys.readouterr().out.splitlines()
    assert made[0].kw["loss_scale_per_network"] is True
    it = [l for l in out if l.startswith("Iteration")]
    assert it[0].endswith("Loss Scale (G / D): 512 / 512, Skipped Steps: 0, Saturated Groups (gradient G / D, activation): 7 / 0, 0, "
                          "Underflow Fraction (G / D): 3.00e-03 / 2.50e-01")
    assert it[1].startswith("Iteration") and "Loss Scale (G / D): 256 / 512, Skipped Steps: 1" in it[1]
    T.train(None, None, str(tmp_path / "m"), "x.ckpt", 0, num_epochs=1, mini_batch_size=2, synthetic=5, log_every=1, device_data=False,
            loss_scale="dynamic")
    out = capsys.readouterr().out
    assert made[1].kw["loss_scale_per_network"] is False and "Loss Scale: 512, Skipped Steps: 0" in out and "(G / D)" not in out
