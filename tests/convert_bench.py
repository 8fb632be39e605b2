"""Conversion throughput: the length-grouped path (one `model.test` call per group of equal padded length) against the packed
path (`model.test_packed`, utterances of any lengths per call) through `convert.convert_features`.  Prints one JSON line.

Corpus: 200 seeded synthetic utterances, lengths uniform over the multiples of 4 in [400, 1400] (the spread of real utterances),
24 x N(0, 1) features, identity MCEP statistics; glorot weights from seed 0.  Per precision the two paths alternate after a warm-up
of each; wall time includes the host-to-device and device-to-host copies and ends in a device synchronise.  Device time is CUDA
events around the generator-forward engine calls alone.

    python tests/convert_bench.py [--precisions f16f8,bf16x3] [--repeats 3] [--utterances 200]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


class _TimedLib:
    """The model's library handle with CUDA events around every generator-forward call (counts them too)."""

    def __init__(self, lib):
        self._lib, self.calls, self.events = lib, 0, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in ("cgvc_generator_forward", "cgvc_generator_forward_packed"):
            return fn
        import torch

        def timed(*args):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r = fn(*args)
            b.record()
            self.calls += 1
            self.events.append((a, b))
            return r
        return timed

    def take(self):
        ms = sum(a.elapsed_time(b) for a, b in self.events)
        n = self.calls
        self.calls, self.events = 0, []
        return n, ms


class _Grouped:
    """the model without test_packed: convert_features takes its length-grouped path"""

    def __init__(self, m):
        self._m = m

    def test(self, inputs, direction):
        return self._m.test(inputs, direction)

    def _ensure_capacity(self, batch, frames):
        self._m._ensure_capacity(batch, frames)


def _gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="f16f8,bf16x3")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--utterances", type=int, default=200)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("convert_bench.py needs a CUDA device")
    import cgvc
    from cgvc import convert as Cv

    rs = np.random.RandomState(0)
    lengths = 4 * rs.randint(100, 351, size=a.utterances)                  # multiples of 4 in [400, 1400]
    corpus = [rs.randn(int(T), 24) for T in lengths]                        # time-major, like pyworld's coded_sp
    stats = {"mean_A": np.zeros((24, 1)), "std_A": np.ones((24, 1)), "mean_B": np.zeros((24, 1)), "std_B": np.ones((24, 1))}
    frames = int(lengths.sum())
    launches = C.c_ulonglong(0)
    result = {"utterances": a.utterances, "frames": frames, "gpu": None, "power_limit": None, "precisions": {}}
    for prec in a.precisions.split(","):
        m = cgvc.CycleGAN(num_features=24, mode="test", precision=prec, seed=0)
        lib = _TimedLib(m._lib)
        m._lib = lib
        paths = {"grouped": _Grouped(m), "packed": m}
        outs, rec = {}, {k: {"wall_s": [], "device_ms": [], "calls": None, "kernel_launches": None} for k in paths}
        for name, model in paths.items():                                  # warm-up: sizes the engine, loads the modules
            outs[name] = Cv.convert_features(model, corpus, "A2B", stats)
            torch.cuda.synchronize()
            lib.take()
        for _ in range(a.repeats):
            for name, model in paths.items():
                lib._lib.cgvc_kernel_launches(C.byref(launches)); l0 = launches.value
                t0 = time.perf_counter()
                outs[name] = Cv.convert_features(model, corpus, "A2B", stats)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                lib._lib.cgvc_kernel_launches(C.byref(launches))
                calls, ms = lib.take()
                r = rec[name]
                r["wall_s"].append(dt); r["device_ms"].append(ms); r["calls"] = calls; r["kernel_launches"] = launches.value - l0
        agree = max(float(np.linalg.norm(p - g) / np.linalg.norm(g)) for p, g in zip(outs["packed"], outs["grouped"]))
        res = {}
        for name, r in rec.items():
            fps = [frames / t for t in r["wall_s"]]
            res[name] = {"frames_per_s_median": float(np.median(fps)), "frames_per_s_spread": float(max(fps) - min(fps)),
                         "wall_s": [round(t, 4) for t in r["wall_s"]], "device_ms_median": float(np.median(r["device_ms"])),
                         "engine_calls": r["calls"], "kernel_launches": r["kernel_launches"]}
        res["speedup_wall"] = res["packed"]["frames_per_s_median"] / res["grouped"]["frames_per_s_median"]
        res["speedup_device"] = res["grouped"]["device_ms_median"] / res["packed"]["device_ms_median"]
        res["max_rel_l2_packed_vs_grouped"] = agree
        result["precisions"][prec] = res
        del m, lib
        torch.cuda.empty_cache()
    result["gpu"], result["power_limit"] = _gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
