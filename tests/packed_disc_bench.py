"""Discriminator forward throughput over utterances of different lengths: packed calls (`CycleGAN.discriminate_packed` on CUDA
tensors, --chunk utterances per call) against one `cgvc_discriminator_forward` call per length group (the [b, 24, T] stack of the
utterances of each length).  Prints one JSON line with the card's name and power limit.

Corpus: 200 seeded synthetic utterances, lengths uniform over the multiples of 16 in [400, 1392], 24 x N(0, 1) features; glorot
weights from seed 0.  The engine is sized for both paths up front (no growth in the timed window).  Per precision the two paths
alternate after a warm-up of each; device time is CUDA events around each path's whole sequence (input staging included), wall time
ends in a device synchronise.  The probabilities of both paths are compared (largest absolute difference).

    python tests/packed_disc_bench.py [--precisions f16f8,bf16x3] [--repeats 3] [--utterances 200] [--chunk 50]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from packed_autograd_bench import _gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="f16f8,bf16x3")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--utterances", type=int, default=200)
    ap.add_argument("--chunk", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("packed_disc_bench.py needs a CUDA device")
    import cgvc

    rs = np.random.RandomState(0)
    lengths = [int(T) for T in 16 * rs.randint(25, 88, size=a.utterances)]      # multiples of 16 in [400, 1392]
    frames = sum(lengths)
    xs = [torch.from_numpy(rs.randn(24, T).astype(np.float32)).cuda() for T in lengths]
    groups = {}
    for u, T in enumerate(lengths):
        groups.setdefault(T, []).append(u)
    chunks = [list(range(i, min(i + a.chunk, a.utterances))) for i in range(0, a.utterances, a.chunk)]
    max_rows = max(sum(lengths[u] for u in c) for c in chunks)
    max_batch = max(a.chunk, max(len(v) for v in groups.values()))
    max_frames = max(max(lengths), -(-max_rows // (16 * max_batch)) * 16)

    def packed(m, out):
        for c in chunks:
            for u, p in zip(c, m.discriminate_packed([xs[u] for u in c], "B")):
                out[u] = p

    def grouped(m, out):
        for T, us in groups.items():
            x = torch.stack([xs[u] for u in us])
            p = torch.empty(len(us), 6, T // 16, 1, device="cuda")
            m._chk(m._lib.cgvc_discriminator_forward(m._handle, 1, C.c_void_p(x.data_ptr()), C.c_void_p(p.data_ptr()), len(us), T,
                                                     m._stream()))
            for i, u in enumerate(us):
                out[u] = p[i]

    result = {"utterances": a.utterances, "frames": frames, "length_groups": len(groups), "packed_calls": len(chunks),
              "gpu": None, "power_limit": None, "precisions": {}}
    for prec in a.precisions.split(","):
        m = cgvc.CycleGAN(num_features=24, mode="test", precision=prec, seed=0, max_batch=max_batch, max_frames=max_frames,
                          log_dir="/tmp/cgvc_log")
        paths = {"grouped": grouped, "packed": packed}
        rec = {k: {"wall_s": [], "device_ms": []} for k in paths}
        outs = {k: [None] * a.utterances for k in paths}
        for name, fn in paths.items():                                      # warm-up, and the results of each path
            fn(m, outs[name])
        torch.cuda.synchronize()
        diff = max(float((p - q).abs().max()) for p, q in zip(outs["packed"], outs["grouped"]))
        for _ in range(a.repeats):
            for name, fn in paths.items():
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                fn(m, [None] * a.utterances)
                e1.record()
                torch.cuda.synchronize()
                rec[name]["wall_s"].append(time.perf_counter() - t0)
                rec[name]["device_ms"].append(e0.elapsed_time(e1))
        res = {}
        for name, r in rec.items():
            fps = [frames / t for t in r["wall_s"]]
            res[name] = {"frames_per_s_median": float(np.median(fps)), "frames_per_s_spread": float(max(fps) - min(fps)),
                         "wall_s": [round(t, 4) for t in r["wall_s"]], "device_ms_median": float(np.median(r["device_ms"]))}
        res["speedup_wall"] = res["packed"]["frames_per_s_median"] / res["grouped"]["frames_per_s_median"]
        res["speedup_device"] = res["grouped"]["device_ms_median"] / res["packed"]["device_ms_median"]
        res["prob_max_abs_diff_packed_vs_grouped"] = diff
        result["precisions"][prec] = res
        del m
        torch.cuda.empty_cache()
    result["gpu"], result["power_limit"] = _gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
