"""Times the reference's step rebuilt in Python from the differentiable networks (tests/test_gpu_autograd.py python_step + adam_step)
against the fused train step (CycleGAN.train_async) at batch 1 and 16, T = 128, in the default precision, on one GPU; prints the card
and its power limit beside the numbers.  CUDA events around `--steps` steps after `--warmup`.

    python tests/autograd_bench.py [--steps 20] [--warmup 3] [--precision bf16x3]
"""
import argparse
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name() + ", power limit unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "autograd_bench needs a GPU"
    import cgvc
    from oracle import cyclegan_oracle as O
    from test_gpu_autograd import python_step
    print("card: %s" % card())
    for batch in (1, 16):
        m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision=args.precision, log_dir='/tmp/cgvc_log')
        A, B = (t.cuda() for t in O.synthetic_batch(seed=1, batch=batch, frames=128))

        def py():
            python_step(m, A, B, 10.0, 5.0)
            m.adam_step(2e-4, 1e-4)
        ms_py = timed(py, args.steps, args.warmup)
        ms_fused = timed(lambda: m.train_async(A, B, 10.0, 5.0, 2e-4, 1e-4), args.steps, args.warmup)
        print("batch %2d T 128 %s: python step %.2f ms, fused train step %.2f ms, ratio %.2f" % (batch, args.precision, ms_py, ms_fused, ms_py / ms_fused))
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
