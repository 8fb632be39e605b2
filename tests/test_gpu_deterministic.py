"""Deterministic mode (engine option "deterministic"): train steps and gradients bitwise reproducible whatever the stream schedule or
graph replay, still within the oracle tolerance, with exact fixed-order reductions (DESIGN.md section 11)."""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_ref as G
from parity_util import rel_l2
from test_gpu_kernels import CONV_CASES

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "bf16x3", "bf16", "f16f8"]
SCHED = [(10, 5, 2e-4, 1e-4), (7, 5, 1e-4, 5e-5), (10, 0, 3e-4, 1e-4), (10, 5, 2e-4, 2e-4)]     # (lambda_c, lambda_id, lr_g, lr_d)
DET_SLAB_FLOATS = 8 << 20           # CGVC_DET_SLAB_FLOATS of kernels.cuh: the partials slab of one lane / entry point


def _model(prec, batch=8, det=True, **kw):
    import cgvc
    return cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision=prec, seed=11,
                         log_dir='/tmp/cgvc_log', deterministic=det, **kw)


def _inject(m, params):
    m.set_params({k: v.numpy() for k, v in params.items()})


def _inputs(seed, batch, frames=128):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=seed, batch=batch, frames=frames, dtype=torch.float32)
    return A.numpy(), B.numpy()


def _grads_run(m, A, B):
    L, gA, gB = m.compute_gradients(A, B, 10.0, 5.0)
    end = max(o + int(np.prod(s)) for o, s in m._table.values())
    from cgvc import native as N
    return L, gA, gB, m._arenas[N.ARENA_GRAD][:end].cpu()


def _assert_same(a, b, what):
    La, gAa, gBa, Ga = a
    Lb, gAb, gBb, Gb = b
    assert La == Lb, (what, La, Lb)
    assert np.array_equal(gAa, gAb) and np.array_equal(gBa, gBb), what
    nd = int((Ga != Gb).sum())
    assert nd == 0, "%s: %d GRAD elements differ" % (what, nd)


@pytest.mark.parametrize("prec,batch", [(p, 8) for p in PRECISIONS] + [("f16f8", 64)])
def test_gradients_do_not_depend_on_the_schedule(oracle_params64, prec, batch):
    m = _model(prec, batch)
    _inject(m, oracle_params64)
    A, B = _inputs(31, batch)
    runs = {}
    for name, opts in (("two_streams", {"two_streams": 1}), ("again", {"two_streams": 1}), ("one_stream", {"two_streams": 0}),
                       ("fuse_bwd+side_wgrad", {"two_streams": 1, "fuse_bwd": 1, "side_wgrad": 1})):
        for k, v in opts.items():
            m.set_option(k, v)
        runs[name] = _grads_run(m, A, B)
        for k in ("fuse_bwd", "side_wgrad"):
            m.set_option(k, 0)
    for name in ("again", "one_stream", "fuse_bwd+side_wgrad"):
        _assert_same(runs["two_streams"], runs[name], "%s %s" % (prec, name))
    # for the record: what default mode does between the two schedules (not asserted)
    m.set_option("deterministic", 0)
    d = []
    for ts in (1, 0):
        m.set_option("two_streams", ts)
        d.append(_grads_run(m, A, B)[3])
    m.set_option("two_streams", 1)
    print("%s batch %d: default mode, two_streams 1 vs 0: %d of %d GRAD elements differ" % (prec, batch, int((d[0] != d[1]).sum()), d[0].numel()))


def _trajectory(prec, params, schedule, loss_scale="static", **opts):
    from cgvc import native as N
    m = _model(prec, 2, loss_scale=loss_scale)
    _inject(m, params)
    for k, v in opts.items():
        m.set_option(k, v)
    rs = np.random.RandomState(5)
    losses = []
    for lc, li, lg, ld in schedule:
        A, B = rs.randn(2, 24, 128), rs.randn(2, 24, 128)
        m.train(A, B, lc, li, lg, ld)
        losses.append(dict(m.last_losses))
    end = max(o + int(np.prod(s)) for o, s in m._table.values())
    state = [m._arenas[k][:end].cpu() for k in (N.ARENA_PARAM, N.ARENA_ADAM_M, N.ARENA_ADAM_V)]
    ls = m.loss_scale_state() if loss_scale != "static" else None
    step = C.c_longlong(0)
    m._lib.cgvc_get_adam_step(m._handle, C.byref(step))
    del m
    torch.cuda.empty_cache()
    return losses, state, ls, step.value


@pytest.mark.parametrize("prec,loss_scale", [(p, "static") for p in PRECISIONS] + [("f16f8", "dynamic")])
def test_train_steps_are_bitwise_equal_across_schedules(oracle_params64, prec, loss_scale):
    runs = {name: _trajectory(prec, oracle_params64, SCHED, loss_scale, **opts)
            for name, opts in (("graph", {"cuda_graph": 1}), ("eager", {"cuda_graph": 0}), ("one_stream", {"two_streams": 0}))}
    ref = runs["graph"]
    for name in ("eager", "one_stream"):
        got = runs[name]
        assert got[0] == ref[0], (prec, name, "losses")
        for what, a, b in zip(("PARAM", "ADAM_M", "ADAM_V"), got[1], ref[1]):
            assert torch.equal(a, b), (prec, name, what, int((a != b).sum()))
        assert got[2] == ref[2] and got[3] == ref[3], (prec, name, got[2], ref[2])


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_deterministic_gradients_stay_parity_grade(oracle_params64, prec):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=9, batch=2, frames=128, dtype=torch.float64)
    L, Gref, gA, gB = O.gradients(A, B, oracle_params64, 10.0, 5.0)
    m = _model(prec, 2)
    _inject(m, oracle_params64)
    losses, genA, genB = m.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
    det = m.get_grads()
    m.set_option("deterministic", 0)
    losses0, _, _ = m.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
    dflt = m.get_grads()
    for k, v in L.items():
        assert abs(losses[k] - float(v)) < 1e-3 * abs(float(v)), k
        assert abs(losses[k] - losses0[k]) <= 2e-6 * abs(losses0[k]), k
    assert rel_l2(genA, gA.numpy()) < 1e-3 and rel_l2(genB, gB.numpy()) < 1e-3
    reorder = 3e-4 if prec == "f16f8" else 1e-4
    worst = (0.0, "")
    assert len(Gref) == 280
    for name, g_ref in Gref.items():
        g_ref = g_ref.numpy()
        n = np.linalg.norm(g_ref.ravel())
        if n < 1e-9:                                           # conv biases feeding an instance norm: analytically zero
            assert np.abs(det[name]).max() < 1e-5, name
            continue
        e = np.linalg.norm((det[name].astype(np.float64) - g_ref).ravel()) / n
        assert e < 1e-3, (name, e)
        n0 = np.linalg.norm(dflt[name].astype(np.float64).ravel())
        if n0 > 1e-6:
            e0 = np.linalg.norm((det[name].astype(np.float64) - dflt[name]).ravel()) / n0
            worst = max(worst, (e0, name))
            assert e0 < reorder, (name, e0)
    print("%s: deterministic vs default mode, worst gradient rel. diff %.2e (%s)" % (prec, worst[0], worst[1]))


# ---- the per-kernel entry points ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def det_eng():
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    assert lib.cgvc_set_option(h, b"deterministic", 1) == 0
    keep = {}
    for kind in (N.ARENA_PARAM, N.ARENA_WORK):
        nb = C.c_size_t(0)
        assert lib.cgvc_arena_bytes(h, kind, C.byref(nb)) == 0
        keep[kind] = torch.empty((nb.value + 3) // 4, dtype=torch.float32, device="cuda")
        assert lib.cgvc_bind_arena(h, kind, C.c_void_p(keep[kind].data_ptr()), nb.value) == 0
    yield lib, h, N
    lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# model-sized cases (ksplit 1), split-K cases (big.o1: 13 uneven splits, big.split: 30 with an empty last split, which deterministic
# mode drops) and big.res_h1, whose 8 planned splits of a 1.57 M-element gradient exceed the slab, so the launcher lowers them to 5
EXACT_CASES = [c for c in G.BIG_CASES if c[0] in ("big.o1", "big.res_h1", "big.split")] + \
    [c for c in CONV_CASES if c[0] in ("G.res_h1", "D.d2", "G.o1")]


@pytest.mark.parametrize("case", EXACT_CASES, ids=[c[0] for c in EXACT_CASES])
@pytest.mark.parametrize("prec", [G.BF16X3, G.F16F8, G.FP32])
def test_conv_backward_reductions_are_exact(det_eng, case, prec):
    lib, h, N = det_eng
    name, B, H, W, Cin, kh, kw, Cout, sh, sw = case
    if not G.supports(case, prec) or (prec == G.FP32 and name.startswith("big")):
        pytest.skip("no such path")
    if name == "big.res_h1":
        L = G.case_launches(case, prec, 0, torch.cuda.get_device_properties(0).multi_processor_count)["wgrad"]
        assert L["ksplit"] * kh * kw * Cin * Cout > DET_SLAB_FLOATS, L["ksplit"]
    x, w, b, dy = G.lattice_case(case, prec)
    P = G.case_planes(prec, x, w, dy)
    ref = G.emulate(case, prec, x, w, b, dy, w16=0, device="cuda", P=P)
    assert lib.cgvc_set_option(h, b"wgrad_f16", 0) == 0
    xd, wd, dyd = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in (x, w, dy))
    for _ in range(2):
        dw = torch.zeros_like(wd); db = torch.zeros(Cout, device="cuda")
        N.check(h, lib.cgvc_conv_backward(h, prec, _p(xd), _p(wd), _p(dyd), None, _p(dw), _p(db), B, H, W, Cin, kh, kw, Cout, sh, sw, None))
        torch.cuda.synchronize()
        assert torch.equal(dw.double().cpu().reshape(-1), torch.as_tensor(ref["dw"]).cpu().reshape(-1)), name
        assert torch.equal(db.double().cpu().reshape(-1), torch.as_tensor(ref["db"]).cpu().reshape(-1)), name


@pytest.mark.parametrize("form", ["gated", "residual", "shuffle"])
def test_in_glu_backward_parameter_gradients_are_repeatable(det_eng, form):
    lib, h, N = det_eng
    Bn, R, Cn = 16, 64, 256
    gate, sh = {"gated": (1, 1), "residual": (0, 1), "shuffle": (1, 2)}[form]
    g = torch.Generator(device="cuda").manual_seed(3)
    ldp = (2 if gate else 1) * Cn * sh
    p = torch.randn(Bn * R // sh, ldp, device="cuda", generator=g)
    pars = [torch.randn(Cn, device="cuda", generator=g) * 0.1 + (1.0 if i % 2 else 0.0) for i in range(4)]
    y = torch.empty(Bn * R * Cn, device="cuda"); stats = torch.empty(Bn * 4 * Cn, device="cuda")
    N.check(h, lib.cgvc_in_glu_forward_planes(h, _p(p), _p(pars[0]), _p(pars[1]), _p(pars[2]), _p(pars[3]), _p(y), _p(stats),
                                              Bn, R, Cn, sh, N.PREC_FP32_SIMT, gate, None, None, None, None, None))
    dy = torch.randn(Bn * R * Cn, device="cuda", generator=g)
    outs = []
    for onepass in (1, 1, 0):
        assert lib.cgvc_set_option(h, b"post_onepass", onepass) == 0
        dp = torch.empty_like(p); grads = [torch.zeros(Cn, device="cuda") for _ in range(4)]
        N.check(h, lib.cgvc_in_glu_backward_planes(h, _p(dy), _p(p), _p(stats), _p(pars[0]), _p(pars[1]), _p(pars[2]), _p(pars[3]),
                                                   _p(dp), _p(grads[0]), _p(grads[1]), _p(grads[2]), _p(grads[3]),
                                                   Bn, R, Cn, sh, N.PREC_FP32_SIMT, gate, None, None, None, None))
        torch.cuda.synchronize()
        outs.append([t.cpu() for t in [dp] + grads])
    assert lib.cgvc_set_option(h, b"post_onepass", 1) == 0
    for o in outs[1:]:
        for a, b in zip(o, outs[0]):
            assert torch.equal(a, b), form
    assert outs[0][2].abs().sum() > 0


# ---- resume, driver, plumbing ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss_scale", ["static", "dynamic"])
def test_resume_from_checkpoint_is_bitwise(oracle_params64, tmp_path, loss_scale):
    from cgvc import native as N
    rs = np.random.RandomState(8)
    batches = [(rs.randn(2, 24, 128), rs.randn(2, 24, 128)) for _ in range(4)]

    def state(m):
        end = max(o + int(np.prod(s)) for o, s in m._table.values())
        step = C.c_longlong(0)
        m._lib.cgvc_get_adam_step(m._handle, C.byref(step))
        return [m._arenas[k][:end].cpu() for k in (N.ARENA_PARAM, N.ARENA_ADAM_M, N.ARENA_ADAM_V)], step.value

    straight = _model("f16f8", 2, loss_scale=loss_scale)
    _inject(straight, oracle_params64)
    for (A, B), (lc, li, lg, ld) in zip(batches, SCHED):
        straight.train(A, B, lc, li, lg, ld)
    ref = state(straight)
    del straight
    first = _model("f16f8", 2, loss_scale=loss_scale)
    _inject(first, oracle_params64)
    for (A, B), (lc, li, lg, ld) in zip(batches[:2], SCHED[:2]):
        first.train(A, B, lc, li, lg, ld)
    path = first.save(str(tmp_path), "half")
    del first
    resumed = _model("f16f8", 2, loss_scale=loss_scale)
    resumed.load(path)
    for (A, B), (lc, li, lg, ld) in zip(batches[2:], SCHED[2:]):
        resumed.train(A, B, lc, li, lg, ld)
    got = state(resumed)
    assert got[1] == ref[1] == 4
    for what, a, b in zip(("PARAM", "ADAM_M", "ADAM_V"), got[0], ref[0]):
        assert torch.equal(a, b), (loss_scale, what, int((a != b).sum()))


def test_training_driver_runs_repeat(tmp_path):
    from cgvc.train import train
    for d in ("a", "b"):
        train(None, None, str(tmp_path / d), "m.ckpt", 0, 2, 4, synthetic=16, precision="f16f8", deterministic=True)
    za, zb = np.load(str(tmp_path / "a" / "m.ckpt.npz")), np.load(str(tmp_path / "b" / "m.ckpt.npz"))
    assert sorted(za.files) == sorted(zb.files)
    for k in za.files:
        assert np.array_equal(za[k], zb[k]), k


def test_option_on_a_live_model_and_short_work(oracle_params64):
    from cgvc import native as N
    m = _model("bf16x3", 2, det=False)
    _inject(m, oracle_params64)
    A, B = _inputs(4, 2)
    lib, h = m._lib, m._handle
    work0 = m._arenas[N.ARENA_WORK].numel() * 4
    # switched on behind the model's back: the bound WORK is now short, and the call is refused before anything is enqueued
    assert lib.cgvc_set_option(h, b"deterministic", 1) == 0
    before, after = C.c_ulonglong(0), C.c_ulonglong(0)
    lib.cgvc_kernel_launches(C.byref(before))
    gA = torch.empty(2, 24, 128, device="cuda"); gB = torch.empty_like(gA)
    Ad, Bd = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    for call in (lambda: lib.cgvc_compute_gradients(h, _p(Ad), _p(Bd), 2, 128, C.c_float(10.0), C.c_float(5.0), _p(gA), _p(gB), _p(m._losses), None),
                 lambda: lib.cgvc_train_step(h, _p(Ad), _p(Bd), 2, 128, C.c_float(10.0), C.c_float(5.0), C.c_float(2e-4), C.c_float(1e-4),
                                             None, None, _p(m._losses), None)):
        assert call() == -3                                    # CGVC_ERR_UNBOUND
    lib.cgvc_kernel_launches(C.byref(after))
    assert after.value == before.value
    # through the model: WORK grows and the steps run, the same bits as a model created deterministic; back to 0 trains again
    m.set_option("deterministic", 1)
    assert m._arenas[N.ARENA_WORK].numel() * 4 > work0
    got = _grads_run(m, A, B)
    ref_m = _model("bf16x3", 2)
    _inject(ref_m, oracle_params64)
    _assert_same(got, _grads_run(ref_m, A, B), "live switch")
    del ref_m
    m.train(A, B, 10.0, 5.0, 2e-4, 1e-4)
    m.set_option("deterministic", 0)
    g0, d0 = m.train(A, B, 10.0, 5.0, 2e-4, 1e-4)
    assert np.isfinite(g0) and np.isfinite(d0)
