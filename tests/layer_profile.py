#!/usr/bin/env python
"""Per-layer timing of the tensor-core kernels inside the real train step (CUDA events around every launch, steady state).

    python tests/layer_profile.py [--batch 256] [--steps 2] [--debug-sweep] > gpurun_out/layer_profile.json

Not a pytest file.  Prints one JSON object: rows = one entry per distinct (kernel class, M, N, K) with launch count,
mean ms, algorithmic TFLOP/s and the fraction of the measured bf16 peak; with --debug-sweep the same table is taken with
the forward/data-gradient kernel's diagnostic knobs (no epilogue stores / no accumulator reads / no activation gather) to see
what bounds a tile.  Timings are serialised on one stream (two_streams = 0), like bench.py's roofline pass.
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cgvc  # noqa: E402
from cgvc import native  # noqa: E402

CLS = {0: "nt (fwd/dgrad, plain epilogue)", 1: "tn (wgrad)", 2: "nt (fwd, fused IN epilogue)"}


def collect(lib, cap=8192):
    ms = (C.c_double * cap)(); fl = (C.c_double * cap)(); meta = (C.c_longlong * (4 * cap))(); n = C.c_int(0)
    assert lib.cgvc_profile_launches(ms, fl, meta, cap, C.byref(n)) == 0
    return [(int(meta[4 * i]), int(meta[4 * i + 1]), int(meta[4 * i + 2]), int(meta[4 * i + 3]), ms[i], fl[i]) for i in range(min(n.value, cap))]


def table(recs, steps, peak):
    agg = {}
    for cls, M, N, K, ms, fl in recs:
        a = agg.setdefault((cls, M, N, K), [0, 0.0, 0.0]); a[0] += 1; a[1] += ms; a[2] += fl
    rows = []
    for (cls, M, N, K), (cnt, ms, fl) in agg.items():
        tf = fl / (ms * 1e-3) / 1e12 if ms > 0 else 0.0
        rows.append({"kernel": CLS[cls], "M": M, "N": N, "K": K, "launches_per_step": cnt / steps, "ms_per_launch": ms / cnt,
                     "ms_per_step": ms / steps, "tflops": tf, "frac_of_bf16_peak": tf / peak, "mma_rate_frac": 3 * tf / peak})
    rows.sort(key=lambda r: -r["ms_per_step"])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--debug-sweep", action="store_true")
    ap.add_argument("--debug", default="", help="comma-separated tc_debug values to run (overrides --debug-sweep)")
    ap.add_argument("--fuse-bwd", type=int, default=0)
    ap.add_argument("--infer", action="store_true", help="profile the generator-only forward (convert.py path, BASELINE config 5) instead of the train step")
    ap.add_argument("--precision", default="f16f8")
    a = ap.parse_args()
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"bf16_tflops_sustained": 1400.0}
    peak = peaks["bf16_tflops_sustained"]
    dev = torch.device("cuda", 0)
    m = cgvc.CycleGAN(num_features=24, mode="test" if a.infer else "train", max_batch=a.batch, max_frames=128, precision=a.precision, seed=0, log_dir="/tmp/cgvc_lp")
    lib = native.load()
    A = torch.randn(a.batch, 24, 128, device=dev); B = torch.randn(a.batch, 24, 128, device=dev)
    step = (lambda: m.test(A, "A2B")) if a.infer else (lambda: m.train_async(A, B, 10.0, 5.0, 2e-4, 1e-4))
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    lib.cgvc_set_option(m._handle, b"two_streams", 0)
    out = {"batch": a.batch, "steps": a.steps, "peak_bf16_tflops_sustained": peak, "workload": "infer" if a.infer else "train", "precision": a.precision, "runs": {}}
    lib.cgvc_set_option(m._handle, b"fuse_bwd", a.fuse_bwd)
    dbgs = [int(x) for x in a.debug.split(",")] if a.debug else ([0, 1, 2, 4, 6] if a.debug_sweep else [0])
    for dbg in dbgs:
        lib.cgvc_set_option(m._handle, b"tc_debug", dbg)
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        lib.cgvc_profile_enable(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            step()
        e1.record()
        recs = collect(lib)
        lib.cgvc_profile_enable(0)
        rows = table(recs, a.steps, peak)
        tot = {c: sum(r["ms_per_step"] for r in rows if r["kernel"] == CLS[c]) for c in CLS}
        out["runs"]["tc_debug=%d" % dbg] = {"ms_per_step_single_stream": e0.elapsed_time(e1) / a.steps,
                                            "ms_per_step_by_class": {CLS[c]: tot[c] for c in CLS}, "rows": rows}
    lib.cgvc_set_option(m._handle, b"tc_debug", 0)
    print(json.dumps(out))
    # human-readable copy on stderr
    for name, run in out["runs"].items():
        print("== %s: %.2f ms/step single stream; by class %s" % (name, run["ms_per_step_single_stream"],
              {k: round(v, 2) for k, v in run["ms_per_step_by_class"].items()}), file=sys.stderr)
        for r in run["rows"][:40]:
            print("  %-32s M=%-7d N=%-5d K=%-5d x%-4.1f %.3f ms  %6.1f TF/s  mma-rate %.2f" %
                  (r["kernel"], r["M"], r["N"], r["K"], r["launches_per_step"], r["ms_per_launch"], r["tflops"], r["mma_rate_frac"]), file=sys.stderr)


if __name__ == "__main__":
    main()
