"""Loss scaling of the F16F8 gradient planes (engine options "loss_scale" / "loss_scale_growth_interval", include/cgvc.h): the
saturation counters, the non-finite check of GRAD, step skipping and the adaptive scale, against the static scale and the float64
oracle.

A train step is not bit-reproducible from run to run (its gradient atomics reorder sums, DESIGN.md section 7), so "the same result
as the static scale" is checked as: no further from a static run than a second static run is."""
import numpy as np
import pytest
import torch

from parity_util import rel_l2

pytestmark = pytest.mark.gpu

ARENAS = (0, 2, 3)          # PARAM, ADAM_M, ADAM_V


def _model(prec, batch, mode="static", P=None, **kw):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision=prec, log_dir='/tmp/cgvc_log',
                      loss_scale=mode, **kw)
    if P is not None:
        m.set_params({k: v.numpy() for k, v in P.items()})
    return m


def _snap(m):
    torch.cuda.synchronize(m.device)
    return [m._arenas[a].clone() for a in ARENAS]


def _step_count(m):
    import ctypes as C
    t = C.c_longlong(0)
    m._chk(m._lib.cgvc_get_adam_step(m._handle, C.byref(t)))
    return t.value


def _update_err(before, after, ref_after):
    """worst relative error of the weight update per tensor, as test_train_steps_match_oracle measures it"""
    worst = 0.0
    for name in after:
        du = ref_after[name] - before[name]
        if np.abs(du).max() == 0 or ("bias" in name and "block" in name):
            continue
        e = np.linalg.norm((after[name].astype(np.float64) - before[name] - du).ravel()) / np.linalg.norm(du.ravel())
        assert e < (0.1 if after[name].size >= 4096 else 0.3), (name, e)
        worst = max(worst, e)
    return worst


@pytest.mark.parametrize("graph", [1, 0])
@pytest.mark.parametrize("prec", ["f16f8", "bf16x3"])
def test_monitor_and_dynamic_follow_static(oracle_params64, prec, graph):
    """Three train() steps at batch 2 from the same weights: monitor and dynamic (growth interval above the step count) land where
    static does, take no skip, keep the static scale, and count no saturation on these inputs.  "Where static does" is measured on
    the weight update and the moments as a whole (relative L2): Adam's first steps are sign descent, so a gradient element within
    rounding of zero moves its weight 2 lr the other way in any two runs, and a maximum over 120M elements only sees those.  The
    cycle and identity weights are 0: an L1 element within rounding of a sign change flips its whole gradient (see
    test_batch64_losses_and_gradients_match_oracle), which makes two static runs differ by ~7e-3 now and then; the adversarial
    gradients still pass through the loss scale."""
    from oracle import cyclegan_oracle as O
    batches = [O.synthetic_batch(seed=40 + s, batch=2, frames=128, dtype=torch.float32) for s in range(3)]
    runs = {}
    for mode in ("static", "static2", "monitor", "dynamic"):
        m = _model(prec, 2, mode.rstrip("2"), oracle_params64)
        m.set_option("cuda_graph", graph)
        if mode == "dynamic":
            m.set_option("loss_scale_growth_interval", 100)
        init = _snap(m)
        for A, B in batches:
            m.train(A.numpy(), B.numpy(), 0.0, 0.0, 2e-4, 1e-4)
            if mode in ("monitor", "dynamic"):
                st = m.last_loss_scale
                print("[%s graph=%d %s] %s" % (prec, graph, mode, st))
                assert st["sat_grad"] == 0 and st["sat_act"] == 0 and st["nonfinite"] == 0, st
                assert st["scale"] == (1024.0 if prec == "f16f8" else 1.0) and not m.last_step_skipped
        assert _step_count(m) == 3
        runs[mode] = [(b - a).double() for a, b in zip(init, _snap(m))]          # the update; the moments start at zero
        del m
        torch.cuda.empty_cache()

    def rel(x, y):
        return float((x - y).norm() / y.norm())
    spread = [rel(b, a) for a, b in zip(runs["static"], runs["static2"])]
    bad = []
    for mode in ("monitor", "dynamic"):
        for i, (a, b) in enumerate(zip(runs["static"], runs[mode])):
            e = rel(b, a)
            print("[%s graph=%d] %s arena %d: relative L2 difference vs static %.3e (static vs static %.3e)" % (prec, graph, mode, ARENAS[i], e, spread[i]))
            if e > 2 * spread[i] + 1e-3:
                bad.append((mode, ARENAS[i], e, spread[i]))
    assert not bad, bad


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16", "f16f8"])
def test_nonfinite_input_skips_the_step(oracle_params64, prec):
    """A NaN in input_A: the step is skipped -- PARAM, ADAM_M, ADAM_V and the Adam step count bit-unchanged -- and the next clean
    step goes through (F16F8: at half the scale).  The two steps that went through match two float64 oracle steps on the same
    inputs, as in test_train_steps_match_oracle (bf16 is not parity-grade: its error is only printed)."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=50, batch=1, frames=128, dtype=torch.float64)
    ref = O.OracleCycleGAN(dtype=torch.float64, params={k: v.clone() for k, v in oracle_params64.items()})
    for _ in range(2):
        ref.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    m = _model(prec, 1, "dynamic", oracle_params64)
    start = m.get_params()
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    s0 = m.last_loss_scale["scale"]
    before, t0 = _snap(m), _step_count(m)
    bad = A.numpy().copy(); bad[0, 3, 17] = np.nan
    m.train(bad, B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    st = m.loss_scale_state()
    print("[%s] NaN step: %s" % (prec, st))
    assert m.last_step_skipped and st["skipped"] == 1 and st["good_steps"] == 0 and st["nonfinite"] & 1
    after = _snap(m)
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert _step_count(m) == t0 == 1
    assert st["scale"] == (s0 / 2 if prec == "f16f8" else 1.0)
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    assert not m.last_step_skipped and _step_count(m) == 2 and m.last_loss_scale["skipped"] == 1
    p = m._arenas[0]
    assert torch.isfinite(p).all() and not torch.equal(p, before[0])
    ref_after = {k: v.numpy() for k, v in ref.P.items()}
    if prec == "bf16":
        try:
            print("[bf16] 2-step update vs oracle: worst %.3e" % _update_err(start, m.get_params(), ref_after))
        except AssertionError as e:
            print("[bf16] 2-step update outside the parity tolerance: %s" % (e,))
    else:
        print("[%s] 2-step update around the skip vs oracle: worst %.3e" % (prec, _update_err(start, m.get_params(), ref_after)))


@pytest.mark.parametrize("t0", [0, 999])
def test_adam_step_in_dynamic_mode_equals_static(t0):
    """cgvc_adam_step is the same call in every loss-scale mode: with the step count on the device (dynamic mode) it gives the
    bit-identical update of static mode (test_gpu_adam_step_matches_tf_formula checks that one against the TF formula) and
    advances the device step count."""
    import ctypes as C
    import cgvc
    from cgvc import native as N
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=1, max_frames=128, precision="f16f8", log_dir='/tmp/cgvc_log')
    gen = torch.Generator(device="cuda").manual_seed(11)
    state = [torch.randn(m._arenas[a].numel(), device="cuda", generator=gen) * s for a, s in ((0, 1e-1), (1, 1e-3), (2, 1e-4), (3, 1e-8))]
    state[3].abs_()
    out = {}
    for mode in (0, 2):
        m.set_option("loss_scale", mode)
        for a, x in zip((0, 1, 2, 3), state):
            m._arenas[a].copy_(x)
        m._chk(m._lib.cgvc_set_adam_step(m._handle, t0))
        m._chk(m._lib.cgvc_adam_step(m._handle, C.c_float(2e-4), C.c_float(1e-4), C.c_float(0.5), m._stream()))
        assert _step_count(m) == t0 + 1
        out[mode] = _snap(m)
    for i, (a, b) in enumerate(zip(out[0], out[2])):
        assert torch.equal(a, b), ARENAS[i]
    assert not torch.equal(out[0][0], state[0])
    m.set_option("loss_scale", 0)
    assert _step_count(m) == t0 + 1                  # the count moves back to the host with the mode


def test_saturation_is_counted_and_the_dynamic_scale_recovers(oracle_params64):
    """F16F8 at batch 1 with lambda_cycle = 1e4: the scaled L1 gradient is ~1.7e3, above the e4m3 range of the planes and below fp16
    overflow.  Monitor mode counts it; dynamic mode skips and halves until the planes fit, then takes a step that matches the oracle."""
    from oracle import cyclegan_oracle as O
    P = {k: v.clone() for k, v in oracle_params64.items()}
    A, B = O.synthetic_batch(seed=60, batch=1, frames=128, dtype=torch.float64)
    ref = O.OracleCycleGAN(dtype=torch.float64, params=P)
    ref.train(A.numpy(), B.numpy(), 1e4, 5.0, 2e-4, 1e-4)
    ref_after = {k: v.numpy() for k, v in ref.P.items()}

    mon = _model("f16f8", 1, "monitor", oracle_params64)
    before = mon.get_params()
    mon.train(A.numpy(), B.numpy(), 1e4, 5.0, 2e-4, 1e-4)
    st = mon.last_loss_scale
    print("monitor: %s" % st)
    assert st["sat_grad"] > 0 and not mon.last_step_skipped and st["scale"] == 512.0
    try:
        print("monitor (static scale 512): worst update error vs oracle %.3e" % _update_err(before, mon.get_params(), ref_after))
    except AssertionError as e:                       # a finding to report, not a failure of this test
        print("monitor (static scale 512): update outside the oracle tolerance: %s" % (e,))
    del mon

    dyn = _model("f16f8", 1, "dynamic", oracle_params64)
    scales = []
    for _ in range(12):
        dyn.train(A.numpy(), B.numpy(), 1e4, 5.0, 2e-4, 1e-4)
        st = dyn.last_loss_scale
        scales.append((st["scale"], st["sat_grad"], st["last_skipped"]))
        if not st["last_skipped"]:
            break
    print("dynamic: (scale after the step, saturated groups, skipped) per step: %s" % scales)
    assert scales[0][2] and not scales[-1][2]
    assert [s for s, _, _ in scales[:-1]] == [512.0 / 2 ** (i + 1) for i in range(len(scales) - 1)]
    assert _step_count(dyn) == 1 and dyn.last_loss_scale["skipped"] == len(scales) - 1
    after = dyn.get_params()
    assert all(np.isfinite(v).all() for v in after.values())
    print("dynamic: worst update error vs oracle %.3e" % _update_err(before, after, ref_after))


def test_growth_doubles_the_scale(oracle_params64):
    """growth_interval = 2: the scale doubles after two clean steps, and the two updates track the oracle."""
    from oracle import cyclegan_oracle as O
    P = {k: v.clone() for k, v in oracle_params64.items()}
    ref = O.OracleCycleGAN(dtype=torch.float64, params=P)
    m = _model("f16f8", 1, "dynamic", oracle_params64)
    m.set_option("loss_scale_growth_interval", 2)
    before = m.get_params()
    seen = []
    for step in range(2):
        A, B = O.synthetic_batch(seed=20 + step, batch=1, frames=128, dtype=torch.float64)
        ref.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        seen.append((m.last_loss_scale["scale"], m.last_loss_scale["good_steps"]))
    assert seen == [(512.0, 1), (1024.0, 0)], seen
    err = _update_err(before, m.get_params(), {k: v.numpy() for k, v in ref.P.items()})
    print("growth: worst 2-step update error vs oracle %.3e" % err)


def test_state_survives_save_load_and_unscaled_gradients(oracle_params64, tmp_path):
    """save / load round-trip the scaler state; compute_gradients in dynamic mode hands out unscaled gradients like static mode."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=70, batch=1, frames=128, dtype=torch.float32)
    m = _model("f16f8", 1, "dynamic", oracle_params64)
    m.set_option("loss_scale_growth_interval", 3)
    bad = A.numpy().copy(); bad[0, 0, 0] = np.inf
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    m.train(bad, B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    st = m.loss_scale_state()
    assert (st["scale"], st["good_steps"], st["skipped"]) == (256.0, 1, 1)
    path = m.save(str(tmp_path), "ls.ckpt")
    z = np.load(path + ".npz")
    assert float(z["loss_scale"]) == 256.0 and int(z["loss_scale_good_steps"]) == 1 and int(z["loss_scale_skipped"]) == 1
    m2 = _model("f16f8", 1, "dynamic")
    m2.load(path)
    st2 = m2.loss_scale_state()
    assert (st2["scale"], st2["good_steps"], st2["skipped"]) == (256.0, 1, 1) and _step_count(m2) == 2
    m3 = _model("f16f8", 1, "static")
    m3.load(path)                                     # a static engine loads such a checkpoint as before
    # unscaled gradients: dynamic (scale 256 here) and static (512) hand out the same d loss / d w
    m2.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    m3.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    m2.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
    m3.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
    g2, g3 = m2.get_grads(), m3.get_grads()
    # conv biases feeding an instance norm have a zero gradient (rounding noise here), as in test_train_steps_match_oracle
    worst = max((rel_l2(g2[k], g3[k]), k) for k in g3 if not ("bias" in k and "block" in k))
    print("compute_gradients dynamic vs static: worst rel_l2 %.2e (%s)" % worst)
    assert worst[0] < 1e-3
