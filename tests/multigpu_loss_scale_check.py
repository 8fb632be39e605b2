"""Run under torchrun with >= 2 GPUs: with loss_scale='dynamic' every rank takes the same skip decision and keeps the same scale.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 tests/multigpu_loss_scale_check.py

  1. a NaN in rank 1's input only: both ranks skip the step (non-finite after the gradient all-reduce);
  2. saturated gradient planes on rank 0 only (its lambda_cycle = 1e4): the summed count halves the scale on both ranks;
  3. after each step the scaler states and the parameters are identical across ranks.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cgvc  # noqa: E402


def _same_everywhere(m, world, what):
    st = m.loss_scale_state()
    key = torch.tensor([st["scale"], st["good_steps"], st["skipped"], st["last_skipped"]], dtype=torch.float64, device="cuda")
    keys = [torch.empty_like(key) for _ in range(world)]
    dist.all_gather(keys, key)
    p = m._arenas[0]
    ref = p.clone()
    dist.broadcast(ref, src=0)
    assert all(torch.equal(k, keys[0]) for k in keys), (what, keys)
    assert torch.equal(p, ref), what
    return st


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    per = 1
    rs = np.random.RandomState(0)
    A = rs.randn(per * world, 24, 128).astype(np.float32); B = rs.randn(per * world, 24, 128).astype(np.float32)
    a, b = A[rank * per:(rank + 1) * per], B[rank * per:(rank + 1) * per]
    for pipelined in (1, 0):
        m = cgvc.CycleGAN(24, mode='train', max_batch=per, max_frames=128, precision="f16f8", device=lr, seed=123, data_parallel=True,
                          log_dir='/tmp/cgvc_log', loss_scale='dynamic')
        m.set_option("pipelined_comm", pipelined)
        m.train(a, b, 10.0, 5.0, 2e-4, 1e-4)
        st = _same_everywhere(m, world, "clean step")
        assert not st["last_skipped"] and st["scale"] == 512.0
        bad = a.copy()
        if rank == 1:
            bad[0, 5, 9] = np.nan
        m.train(bad, b, 10.0, 5.0, 2e-4, 1e-4)
        st = _same_everywhere(m, world, "NaN on rank 1")
        assert st["last_skipped"] and st["skipped"] == 1 and st["scale"] == 256.0 and st["nonfinite"], st
        m.train(a, b, 1e4 if rank == 0 else 10.0, 5.0, 2e-4, 1e-4)
        st = _same_everywhere(m, world, "saturation on rank 0")
        assert st["last_skipped"] and st["skipped"] == 2 and st["scale"] == 128.0 and st["sat_grad"] > 0 and not st["nonfinite"], st
        m.train(a, b, 10.0, 5.0, 2e-4, 1e-4)
        st = _same_everywhere(m, world, "clean step after the skips")
        assert not st["last_skipped"]
        if rank == 0:
            print("MULTIGPU LOSS SCALE world=%d pipelined_comm=%d: %s" % (world, pipelined, st), flush=True)
        del m
        torch.cuda.empty_cache()
    if rank == 0:
        print("MULTIGPU LOSS SCALE OK", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
