"""Differentiable generator throughput over utterances of different lengths: forward + backward of one generator through packed tapes
(`CycleGAN.generator_packed`, utterances of any lengths per call) against one tape call per length group (`CycleGAN.generator` on
the [b, 24, T] stack of the utterances of each length).  Prints one JSON line.

Corpus: 200 seeded synthetic utterances, lengths uniform over the multiples of 4 in [400, 1400] (the spread of real utterances, as in
tests/convert_bench.py), 24 x N(0, 1) features; glorot weights from seed 0; the upstream gradient of the mean of the outputs times a
seeded N(0, 1) tensor.  The packed path takes --chunk utterances per call.  The engine is sized for both paths up front (no growth in
the timed window).  Per precision the two paths alternate after a warm-up of each; device time is CUDA events around each path's whole
forward + backward sequence (input and gradient staging included), wall time ends in a device synchronise.  Both paths' gradients are
compared (relative L2 over the generator's variables) where both leave one loss scale in the gradient arena (not F16F8, whose
length groups have batches of different scales).

    python tests/packed_autograd_bench.py [--precisions f16f8,bf16x3] [--repeats 3] [--utterances 200] [--chunk 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


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
    ap.add_argument("--chunk", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("packed_autograd_bench.py needs a CUDA device")
    import cgvc

    rs = np.random.RandomState(0)
    lengths = [int(T) for T in 4 * rs.randint(100, 351, size=a.utterances)]      # multiples of 4 in [400, 1400]
    frames = sum(lengths)
    xs = [torch.from_numpy(rs.randn(24, T).astype(np.float32)).cuda() for T in lengths]
    gs = [torch.from_numpy(rs.randn(24, T).astype(np.float32)).cuda() / (24 * frames) for T in lengths]
    groups = {}
    for u, T in enumerate(lengths):
        groups.setdefault(T, []).append(u)
    chunks = [list(range(i, min(i + a.chunk, a.utterances))) for i in range(0, a.utterances, a.chunk)]
    max_rows = max(sum(lengths[u] for u in c) for c in chunks)
    max_batch = max(a.chunk, max(len(v) for v in groups.values()))
    max_frames = max(max(lengths), -(-max_rows // (4 * max_batch)) * 4)

    def packed(m):
        for c in chunks:
            ys = m.generator_packed([xs[u] for u in c], "A2B")
            torch.autograd.backward(ys, [gs[u] for u in c])

    def grouped(m):
        for T, us in groups.items():
            y = m.generator(torch.stack([xs[u] for u in us]), "A2B")
            y.backward(torch.stack([gs[u] for u in us]))

    result = {"utterances": a.utterances, "frames": frames, "length_groups": len(groups), "packed_calls": len(chunks),
              "gpu": None, "power_limit": None, "precisions": {}}
    for prec in a.precisions.split(","):
        m = cgvc.CycleGAN(num_features=24, mode="train", precision=prec, seed=0, max_batch=max_batch, max_frames=max_frames,
                          log_dir="/tmp/cgvc_log")
        paths = {"grouped": grouped, "packed": packed}
        rec = {k: {"wall_s": [], "device_ms": []} for k in paths}
        grads = {}
        for name, fn in paths.items():                                      # warm-up; the gradients of one pass of each path
            m.zero_grad()
            fn(m)
            torch.cuda.synchronize()
            try:
                grads[name] = {k: v.double().clone() for k, v in m.grads("generator_A2B").items()}
            except RuntimeError:                                            # F16F8: length groups of different loss scales
                grads[name] = None
        comparable = all(g is not None for g in grads.values())
        for _ in range(a.repeats):
            for name, fn in paths.items():
                m.zero_grad()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                fn(m)
                e1.record()
                torch.cuda.synchronize()
                rec[name]["wall_s"].append(time.perf_counter() - t0)
                rec[name]["device_ms"].append(e0.elapsed_time(e1))
        if comparable:
            num = sum(float(((grads["packed"][k] - grads["grouped"][k]) ** 2).sum()) for k in grads["packed"])
            den = sum(float((grads["grouped"][k] ** 2).sum()) for k in grads["grouped"])
        res = {}
        for name, r in rec.items():
            fps = [frames / t for t in r["wall_s"]]
            res[name] = {"frames_per_s_median": float(np.median(fps)), "frames_per_s_spread": float(max(fps) - min(fps)),
                         "wall_s": [round(t, 4) for t in r["wall_s"]], "device_ms_median": float(np.median(r["device_ms"]))}
        res["speedup_wall"] = res["packed"]["frames_per_s_median"] / res["grouped"]["frames_per_s_median"]
        res["speedup_device"] = res["grouped"]["device_ms_median"] / res["packed"]["device_ms_median"]
        res["grad_rel_l2_packed_vs_grouped"] = float(np.sqrt(num / den)) if comparable else None
        result["precisions"][prec] = res
        del m
        torch.cuda.empty_cache()
    result["gpu"], result["power_limit"] = _gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
