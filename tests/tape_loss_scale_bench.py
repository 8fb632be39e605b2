"""Loss scaling of the differentiable networks at f16f8, batch B x 128, with the reference's losses composed in Python from the tapes
(model.py:44-108, as tests/test_gpu_tape_loss_scale.py python_step), for DESIGN.md section 12:

  1. static tapes in monitor mode + adam_step: the fraction of N steps in which a gradient plane saturated;
  2. tape_loss_scale='dynamic' + apply_gradients (one scale, and per network): the skipped steps and the scales they settle at;
  3. the step time of static tapes + adam_step against dynamic tapes + apply_gradients: CUDA events over K steps, the median of 3
     runs of each, alternated.

The card's name and power limit are read in the same run.  Prints one JSON line.

    python tests/tape_loss_scale_bench.py --batch 256 --steps 200 --time-steps 10
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def l1_loss(y, y_hat):
    return torch.mean(torch.abs(y - y_hat))


def l2_loss(y, y_hat):
    return torch.mean(torch.square(y - y_hat))


def python_step(m, A, B, lambda_cycle, lambda_identity):
    gen_B = m.generator(A, 'A2B'); cycle_A = m.generator(gen_B, 'B2A')
    gen_A = m.generator(B, 'B2A'); cycle_B = m.generator(gen_A, 'A2B')
    id_A = m.generator(A, 'B2A'); id_B = m.generator(B, 'A2B')
    dA_fake = m.discriminator(gen_A, 'A'); dB_fake = m.discriminator(gen_B, 'B')
    g_loss = (l2_loss(torch.ones_like(dB_fake), dB_fake) + l2_loss(torch.ones_like(dA_fake), dA_fake)
              + lambda_cycle * (l1_loss(A, cycle_A) + l1_loss(B, cycle_B)) + lambda_identity * (l1_loss(A, id_A) + l1_loss(B, id_B)))
    dA_real = m.discriminator(A, 'A'); dB_real = m.discriminator(B, 'B')
    dA_f = m.discriminator(gen_A.detach(), 'A'); dB_f = m.discriminator(gen_B.detach(), 'B')
    d_loss = ((l2_loss(torch.ones_like(dA_real), dA_real) + l2_loss(torch.zeros_like(dA_f), dA_f)) / 2
              + (l2_loss(torch.ones_like(dB_real), dB_real) + l2_loss(torch.zeros_like(dB_f), dB_f)) / 2)
    m.zero_grad()
    g_loss.backward()
    m.zero_grad("discriminator_A"); m.zero_grad("discriminator_B")
    d_loss.backward()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as ex:             # the numbers are still reported, marked as of an unknown card
        return "unknown (%s)" % ex, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--time-steps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tape_loss_scale_bench.py measures on the GPU; there is none")
    import cgvc
    from oracle import cyclegan_oracle as O
    pool = [tuple(t.cuda() for t in O.synthetic_batch(seed=a.seed + i, batch=a.batch, frames=a.frames)) for i in range(4)]
    lr = (2e-4, 1e-4)

    def model(tape, ls, nets=False):
        return cgvc.CycleGAN(num_features=24, mode='train', max_batch=a.batch, max_frames=a.frames, precision='f16f8', seed=a.seed,
                             log_dir='/tmp/cgvc_log', loss_scale=ls, tape_loss_scale=tape, loss_scale_per_network=nets)

    res = {"batch": a.batch, "frames": a.frames, "steps": a.steps}
    # 1. static tapes, monitor mode: a step saturated when the counters grew during it
    m = model('static', 'monitor')
    sat_steps, prev = 0, m.loss_scale_state()["sat_grad"]
    for i in range(a.steps):
        python_step(m, *pool[i % len(pool)], 10.0, 5.0)
        m.adam_step(*lr)
        cur = m.loss_scale_state()["sat_grad"]
        sat_steps += cur > prev
        prev = cur
        if i % 50 == 0:
            print("static step %d: %d saturated so far" % (i, sat_steps), file=sys.stderr, flush=True)
    res["static_saturated_steps"] = int(sat_steps)
    res["static_saturated_fraction"] = sat_steps / a.steps
    res["static_scale"] = m.tape_loss_scale(a.batch)
    del m
    torch.cuda.empty_cache()
    # 2. dynamic tapes
    for nets in (False, True):
        m = model('dynamic', 'dynamic', nets)
        for i in range(a.steps):
            python_step(m, *pool[i % len(pool)], 10.0, 5.0)
            m.apply_gradients(*lr)
        st = m.loss_scale_state()
        print("dynamic (per network %s): %s" % (nets, st), file=sys.stderr, flush=True)
        tag = "dynamic_nets" if nets else "dynamic"
        res[tag] = {"skipped": st["skipped"], "scale": st["scale"]}
        if nets:
            res[tag].update(scale_G=st["scale_G"], scale_D=st["scale_D"])
        del m
        torch.cuda.empty_cache()
    # 3. step time, alternated
    ms = {"static": [], "dynamic": []}
    models = {"static": model('static', 'static'), "dynamic": model('dynamic', 'dynamic')}
    for kind, mm in models.items():                     # warm-up (graph capture of the optimizer tail, allocator)
        for i in range(2):
            python_step(mm, *pool[i], 10.0, 5.0)
            mm.adam_step(*lr) if kind == "static" else mm.apply_gradients(*lr)
    for _ in range(3):
        for kind, mm in models.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.time_steps):
                python_step(mm, *pool[i % len(pool)], 10.0, 5.0)
                mm.adam_step(*lr) if kind == "static" else mm.apply_gradients(*lr)
            e1.record()
            torch.cuda.synchronize()
            ms[kind].append(e0.elapsed_time(e1) / a.time_steps)
    for kind in ms:
        res[kind + "_step_ms"] = sorted(ms[kind])[1]
        res[kind + "_step_ms_runs"] = ms[kind]
    res["dynamic_over_static"] = res["dynamic_step_ms"] / res["static_step_ms"] - 1
    res["card"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
