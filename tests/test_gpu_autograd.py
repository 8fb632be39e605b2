"""The networks as differentiable torch operators (CycleGAN.generator / .discriminator over the activation-tape ABI of include/cgvc.h).

1. The tape forward gives cgvc_generator_forward / cgvc_discriminator_forward's outputs bit for bit, in every precision.
2. Per network, d input and every variable gradient against float64 autograd of the oracle, from a random upstream gradient of the
   magnitude a mean-reduced loss gives (1 / elements: the static F16F8 loss scale is sized for those), GRAD outside the network untouched.
3. The reference's graph (model.py:44-108) rebuilt in Python from the operators and torch losses, against cgvc_compute_gradients and,
   after one adam_step, against cgvc_train_step.
4. Deterministic mode: the same GRAD bits on repeated Python steps and in a fresh engine.
5. The contract's errors launch nothing; a second backward of one tape adds exactly the same gradients; monitor-mode counting.
6. The head backward from an upstream dprob (head_loss_bwd_kernel's dprob path) against float64: bitwise on glu_ref's lattice, within
   the dense bound of test_gpu_glu_layers.py otherwise.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import glu_ref as GR
from parity_util import rel_l2

pytestmark = pytest.mark.gpu

PRECS = ["fp32", "bf16x3", "f16f8"]
TOL = {"fp32": 1e-5, "bf16x3": 1e-3, "f16f8": 1e-3}
NETS = ("generator_A2B", "generator_B2A", "discriminator_A", "discriminator_B")


def _model(prec, max_batch=3, max_frames=516, params=None, **kw):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=max_batch, max_frames=max_frames, precision=prec, log_dir='/tmp/cgvc_log', **kw)
    if params is not None:
        m.set_params({k: v.numpy() for k, v in params.items()})
    return m


@pytest.fixture(scope="module")
def models(oracle_params64):
    out = {p: _model(p, params=oracle_params64) for p in PRECS}
    yield out
    out.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def params_cuda(oracle_params64):
    return {k: v.cuda() for k, v in oracle_params64.items()}


def _batch(seed, batch, frames):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=seed, batch=batch, frames=frames)
    return A.cuda(), B.cuda()


def _launches(m):
    n = C.c_ulonglong(0)
    m._lib.cgvc_kernel_launches(C.byref(n))
    return n.value


# ---- 1. forward ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16", "f16f8"])
def test_tape_forward_is_bitwise_the_forward(models, oracle_params64, prec):
    m = models[prec] if prec in models else _model(prec, params=oracle_params64)
    for batch, frames in ((3, 516), (1, 36), (2, 128)):
        x, _ = _batch(7 + frames, batch, frames)
        for d in ("A2B", "B2A"):
            with torch.no_grad():
                y = m.generator(x, d)
            assert torch.equal(y, m.test(x, d)), (prec, d, batch, frames)
        if frames % 16 == 0:
            for w in ("A", "B"):
                with torch.no_grad():
                    p = m.discriminator(x, w)
                assert np.array_equal(p.cpu().numpy(), m.discriminate(x, w)), (prec, w, batch, frames)


# ---- 2. per-network gradients against float64 ----------------------------------------------------------------------------------------
def _oracle(params_cuda, kind, scope, x, g):
    from oracle import cyclegan_oracle as O
    P = {k: v.clone().requires_grad_(True) for k, v in params_cuda.items() if k.startswith(scope + "/")}
    xx = x.double().clone().requires_grad_(True)
    y = (O.generator_forward if kind == "gen" else O.discriminator_forward)(xx, P, scope)
    (y * g.double()).sum().backward()
    return y.detach(), xx.grad, {k: v.grad for k, v in P.items()}


def _check_grads(tag, got, ref, tol):
    total = float(torch.sqrt(sum((r.double() ** 2).sum() for r in ref.values())))
    worst = (0.0, None)
    for name, r in ref.items():
        gn = got[name].double()
        rn = float(r.norm())
        if rn < 1e-9 * total:          # conv biases feeding an instance norm: analytically zero, compared against the network's gradient
            e = float(gn.norm()) / total
        else:
            e = float((gn - r).norm()) / rn
        worst = max(worst, (e, name))
        assert e < tol, (tag, name, e)
    print("%s worst gradient %s %.2e" % (tag, worst[1], worst[0]))


GEN_CASES = [(d, b, t) for d in ("A2B", "B2A") for b in (1, 3) for t in (128, 36, 516)]


@pytest.mark.parametrize("direction,batch,frames", GEN_CASES)
def test_generator_gradients_match_float64(models, params_cuda, direction, batch, frames):
    scope = "generator_" + direction
    x, _ = _batch(100 + batch + frames, batch, frames)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(batch * 1000 + frames), dtype=torch.float64).cuda() / x.numel()
    y_ref, dx_ref, G_ref = _oracle(params_cuda, "gen", scope, x, g)
    for prec in PRECS:
        m = models[prec]
        m.zero_grad()
        xg = x.clone().requires_grad_(True)
        y = m.generator(xg, direction)
        (y * g.float()).sum().backward()
        tag = "gen[%s %s B=%d T=%d]" % (prec, direction, batch, frames)
        e = rel_l2(xg.grad.cpu().numpy(), dx_ref.cpu().numpy())
        print("%s d in rel_l2 %.2e" % (tag, e))
        assert e < TOL[prec], (tag, "d in", e)
        _check_grads(tag, m.grads(scope), G_ref, TOL[prec])
        for other in NETS:
            if other != scope:
                assert all(bool((v == 0).all()) for v in m.grads(other).values()), (tag, "GRAD touched outside", other)


DISC_CASES = [(w, b, t) for w in ("A", "B") for b in (1, 3) for t in (128, 144)]


@pytest.mark.parametrize("which,batch,frames", DISC_CASES)
def test_discriminator_gradients_match_float64(models, params_cuda, which, batch, frames):
    scope = "discriminator_" + which
    x, _ = _batch(200 + batch + frames, batch, frames)
    shape = (batch, 6, frames // 16, 1)
    g = torch.randn(shape, generator=torch.Generator().manual_seed(batch * 77 + frames), dtype=torch.float64).cuda() / (batch * 6 * frames // 16)
    y_ref, dx_ref, G_ref = _oracle(params_cuda, "disc", scope, x, g)
    for prec in PRECS:
        m = models[prec]
        m.zero_grad()
        xg = x.clone().requires_grad_(True)
        p = m.discriminator(xg, which)
        (p * g.float()).sum().backward()
        tag = "disc[%s %s B=%d T=%d]" % (prec, which, batch, frames)
        e = rel_l2(xg.grad.cpu().numpy(), dx_ref.cpu().numpy())
        print("%s d in rel_l2 %.2e" % (tag, e))
        assert e < TOL[prec], (tag, "d in", e)
        _check_grads(tag, m.grads(scope), G_ref, TOL[prec])
        for other in NETS:
            if other != scope:
                assert all(bool((v == 0).all()) for v in m.grads(other).values()), (tag, "GRAD touched outside", other)


# ---- 3. the reference graph in Python ------------------------------------------------------------------------------------------------
def l1_loss(y, y_hat):          # utils.py:6-8
    return torch.mean(torch.abs(y - y_hat))


def l2_loss(y, y_hat):          # utils.py:10-12
    return torch.mean(torch.square(y - y_hat))


def python_step(m, A, B, lambda_cycle, lambda_identity):
    """model.py:44-108 on the differentiable operators: GRAD ends up as cgvc_compute_gradients leaves it (loss-scaled)"""
    gen_B = m.generator(A, 'A2B'); cycle_A = m.generator(gen_B, 'B2A')
    gen_A = m.generator(B, 'B2A'); cycle_B = m.generator(gen_A, 'A2B')
    id_A = m.generator(A, 'B2A'); id_B = m.generator(B, 'A2B')
    dA_fake = m.discriminator(gen_A, 'A'); dB_fake = m.discriminator(gen_B, 'B')
    L = {}
    L["cycle_loss"] = l1_loss(A, cycle_A) + l1_loss(B, cycle_B)
    L["identity_loss"] = l1_loss(A, id_A) + l1_loss(B, id_B)
    L["generator_loss_A2B"] = l2_loss(torch.ones_like(dB_fake), dB_fake)
    L["generator_loss_B2A"] = l2_loss(torch.ones_like(dA_fake), dA_fake)
    L["generator_loss"] = (L["generator_loss_A2B"] + L["generator_loss_B2A"] + lambda_cycle * L["cycle_loss"]
                           + lambda_identity * L["identity_loss"])
    dA_real = m.discriminator(A, 'A'); dB_real = m.discriminator(B, 'B')
    dA_f = m.discriminator(gen_A.detach(), 'A'); dB_f = m.discriminator(gen_B.detach(), 'B')
    L["discriminator_loss_A"] = (l2_loss(torch.ones_like(dA_real), dA_real) + l2_loss(torch.zeros_like(dA_f), dA_f)) / 2
    L["discriminator_loss_B"] = (l2_loss(torch.ones_like(dB_real), dB_real) + l2_loss(torch.zeros_like(dB_f), dB_f)) / 2
    L["discriminator_loss"] = L["discriminator_loss_A"] + L["discriminator_loss_B"]
    m.zero_grad()
    L["generator_loss"].backward()
    m.zero_grad("discriminator_A"); m.zero_grad("discriminator_B")     # the D optimizer follows the D loss alone (model.py:107-108)
    L["discriminator_loss"].backward()
    return {k: float(v.detach()) for k, v in L.items()}


def _reset_adam(m, params):
    from cgvc import native as N
    m.set_params({k: v.numpy() for k, v in params.items()})
    m._arenas[N.ARENA_ADAM_M].zero_(); m._arenas[N.ARENA_ADAM_V].zero_()
    m._chk(m._lib.cgvc_set_adam_step(m._handle, 0))


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_python_step_matches_fused_step(models, oracle_params64, prec):
    m = models[prec]
    A, B = _batch(9, 2, 128)
    ref_losses, _, _ = m.compute_gradients(A, B, 10.0, 5.0)
    ref = {k: torch.from_numpy(v.copy()) for k, v in m.get_grads().items()}
    losses = python_step(m, A, B, 10.0, 5.0)
    worst_l = max(abs(losses[k] - ref_losses[k]) / abs(ref_losses[k]) for k in ref_losses)
    assert worst_l < 1e-3, (prec, losses, ref_losses)
    got = m.grads()
    assert len(got) == 280
    total = {net: float(torch.sqrt(sum((v.double() ** 2).sum() for k, v in ref.items() if k.startswith(net)))) for net in NETS}
    worst = (0.0, None)
    for name, r in ref.items():
        g = got[name].double().cpu(); rn = float(r.double().norm())
        net = name.split("/")[0]
        e = float((g - r.double()).norm()) / rn if rn > 1e-9 * total[net] else float((g - r.double()).norm()) / total[net]
        worst = max(worst, (e, name))
        assert e < 1e-3, (prec, name, e)
    print("python step [%s] vs compute_gradients: worst loss %.2e, worst gradient %s %.2e" % (prec, worst_l, worst[1], worst[0]))
    # one Adam step after each, from the same state
    lr_g, lr_d = 2e-4, 1e-4
    _reset_adam(m, oracle_params64)
    python_step(m, A, B, 10.0, 5.0)
    m.adam_step(lr_g, lr_d)
    p_py = m.get_params()
    _reset_adam(m, oracle_params64)
    m.train(A, B, 10.0, 5.0, lr_g, lr_d)
    p_fused = m.get_params()
    e = max(rel_l2(p_py[k], p_fused[k]) for k in p_py)
    moved = max(rel_l2(p_fused[k], oracle_params64[k].numpy()) for k in p_py)
    print("adam step [%s]: parameters python vs train_step %.2e (the step moved them by up to %.2e)" % (prec, e, moved))
    assert e < 1e-3
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})


# ---- 4. deterministic mode -----------------------------------------------------------------------------------------------------------
def test_deterministic_python_step(oracle_params64):
    from cgvc import native as N
    A, B = _batch(11, 2, 128)
    bits = []
    for fresh in (0, 0, 1):
        if fresh or not bits:
            m = _model("bf16x3", 2, 128, params=oracle_params64, deterministic=True)
        python_step(m, A, B, 10.0, 5.0)
        torch.cuda.synchronize()
        bits.append(m._arenas[N.ARENA_GRAD].clone())
    assert torch.equal(bits[0], bits[1]) and torch.equal(bits[0], bits[2])


# ---- 5. contract ---------------------------------------------------------------------------------------------------------------------
def test_tape_errors_launch_nothing(models, oracle_params64):
    from cgvc import native as N
    m, m2 = models["bf16x3"], models["f16f8"]
    h, lib = m._handle, m._lib
    x, _ = _batch(5, 1, 128)
    dy = torch.zeros_like(x)
    dprob = torch.zeros(1, 6, 8, 1, device="cuda")

    def ptr(t):
        return C.c_void_p(t.data_ptr())
    _, gtape = m._tape_forward(0, 0, x)
    _, dtape = m._tape_forward(1, 0, x)
    _, otape = m2._tape_forward(0, 0, x)
    torch.cuda.synchronize()
    zeros = torch.zeros_like(gtape)
    cases = [("not a tape", lambda: lib.cgvc_generator_backward_tape(h, ptr(zeros), ptr(dy), None, None), N.ERR_ARG),
             ("other engine", lambda: lib.cgvc_generator_backward_tape(h, ptr(otape), ptr(dy), None, None), N.ERR_ARG),
             ("wrong kind", lambda: lib.cgvc_discriminator_backward_tape(h, ptr(gtape), ptr(dprob), None, None), N.ERR_ARG),
             ("wrong kind", lambda: lib.cgvc_generator_backward_tape(h, ptr(dtape), ptr(dy), None, None), N.ERR_ARG),
             ("undersized", lambda: lib.cgvc_generator_forward_tape(h, 0, ptr(x), ptr(dy), 1, 128, ptr(gtape), gtape.numel() - 1, None),
              N.ERR_UNBOUND),
             ("stale", None, N.ERR_ARG)]
    for what, call, code in cases:
        if call is None:                                       # the parameters change after the forward
            m._params_updated()
            torch.cuda.synchronize()
            call = lambda: lib.cgvc_generator_backward_tape(h, ptr(gtape), ptr(dy), None, None)    # noqa: E731
        before = _launches(m)
        assert call() == code, what
        assert _launches(m) == before, (what, "launched")
    # a forward-only engine has no GRAD
    t = __import__("cgvc").CycleGAN(num_features=24, mode='test', max_batch=1, max_frames=128, precision="bf16x3")
    _, ttape = t._tape_forward(0, 0, x)
    before = _launches(t)
    assert t._lib.cgvc_generator_backward_tape(t._handle, ptr(ttape), ptr(dy), None, None) == N.ERR_UNBOUND
    assert _launches(t) == before
    # through autograd the refusal is an exception
    y = m.generator(x.clone().requires_grad_(True), 'A2B')
    m._params_updated()
    with pytest.raises(RuntimeError, match="stale"):
        y.sum().backward()


def test_second_backward_doubles_grad_exactly(oracle_params64):
    from cgvc import native as N
    m = _model("bf16x3", 1, 128, params=oracle_params64, deterministic=True)
    x, _ = _batch(6, 1, 128)
    for kind in ("gen", "disc"):
        m.zero_grad()
        xg = x.clone().requires_grad_(True)
        y = m.generator(xg, 'B2A') if kind == "gen" else m.discriminator(xg, 'B')
        loss = (y * torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda() / y.numel()).sum()
        loss.backward(retain_graph=True)
        torch.cuda.synchronize()
        once, dx1 = m._arenas[N.ARENA_GRAD].clone(), xg.grad.clone()
        assert bool((once != 0).any())
        loss.backward()
        torch.cuda.synchronize()
        assert torch.equal(m._arenas[N.ARENA_GRAD], 2 * once), kind
        assert torch.equal(xg.grad, 2 * dx1), kind


def test_monitor_mode_counts_saturated_tape_gradients(oracle_params64):
    m = _model("f16f8", 1, 128, params=oracle_params64, loss_scale='monitor')
    x, _ = _batch(8, 1, 128)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(4)).cuda() / x.numel()
    counts = []
    for mult in (1.0, 2.0 ** 20):
        before = m.loss_scale_state()["sat_grad"]
        m.zero_grad()
        (m.generator(x, 'A2B') * (g * mult)).sum().backward()
        counts.append(m.loss_scale_state()["sat_grad"] - before)
    print("monitor: saturated gradient-plane groups %d (mean-loss magnitude), %d (x 2^20)" % tuple(counts))
    assert counts[0] == 0 and counts[1] > 0


# ---- 6. the head backward from dprob -------------------------------------------------------------------------------------------------
U = GR.U


@pytest.mark.parametrize("rows", [48, 96, 6 * 8 * 128, 4096])
@pytest.mark.parametrize("tier", ["lattice", "dense"])
@pytest.mark.parametrize("gm", [None, 2.0 ** 10])
@pytest.mark.parametrize("det", [0, 1])
def test_head_backward_from_dprob(rows, tier, gm, det):
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 16, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0
    work = None
    if det:
        N.check(h, lib.cgvc_set_option(h, b"deterministic", 1))
        nb = C.c_size_t(0)
        N.check(h, lib.cgvc_arena_bytes(h, N.ARENA_WORK, C.byref(nb)))
        work = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
        N.check(h, lib.cgvc_bind_arena(h, N.ARENA_WORK, C.c_void_p(work.data_ptr()), nb.value))
    rng = np.random.default_rng(rows * 7 + (tier == "dense"))
    if tier == "lattice":
        y, w, b = GR.lattice_head_case(rng, rows)
        dprob = rng.integers(-4, 5, rows).astype(np.float32)
    else:
        y = rng.standard_normal((rows, 1024)).astype(np.float32)
        w = (rng.standard_normal(1024) / 32).astype(np.float32)
        b = np.array([0.1], np.float32)
        dprob = rng.standard_normal(rows).astype(np.float32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()    # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)    # noqa: E731
    yd, wd, bd, dpd = dev(y), dev(w), dev(b), dev(dprob)
    prob = torch.empty(rows, device="cuda")
    N.check(h, lib.cgvc_head_forward(h, p(yd), rows, p(wd), p(bd), p(prob), None))
    dy = torch.full((rows, 1024), float("nan"), device="cuda")
    dw = torch.zeros(1024, device="cuda") + 0.5
    db = torch.zeros(1, device="cuda") + 0.5
    gmd = None if gm is None else torch.tensor([gm], device="cuda")
    N.check(h, lib.cgvc_head_backward(h, p(prob), p(yd), rows, p(wd), p(dpd), p(gmd), p(dy), p(dw), p(db), None))
    torch.cuda.synchronize()
    lib.cgvc_destroy(h)
    gmv = 1.0 if gm is None else gm
    pr = prob.double().cpu()
    dz = gmv * torch.from_numpy(dprob).double() * pr * (1 - pr)
    w64 = torch.from_numpy(w).double(); y64 = torch.from_numpy(y).double()
    dyref, dwref, dbref = dz[:, None] * w64[None, :], (dz[:, None] * y64).sum(dim=0), dz.sum()
    tag = "head dprob rows %d %s gm %s det %d" % (rows, tier, gm, det)
    if tier == "lattice":                          # prob = 1/2, dprob integers: every output exact
        assert bool((prob == 0.5).all()), tag
        assert torch.equal(dy.double().cpu(), dyref), tag
        assert torch.equal(dw.double().cpu(), dwref + 0.5) and float(db) == 0.5 + float(dbref), tag
        return
    L = GR.head_chain(rows)
    dzb = 8 * U * dz.abs() + 1e-45
    assert bool(((dy.double().cpu() - dyref).abs() <= dzb[:, None] * w64.abs()[None, :] + U * dyref.abs() + 1e-45).all()), tag
    ab = (dz.abs()[:, None] * y64.abs()).sum(dim=0)
    assert bool(((dw.double().cpu() - dwref - 0.5).abs() <= GR.gamma(L + 8) * (ab + 0.5) + 8 * U * ab + 1e-45).all()), tag
    assert abs(float(db) - 0.5 - float(dbref)) <= GR.gamma(L + 8) * (float(dz.abs().sum()) + 0.5) + 8 * U * float(dz.abs().sum()), tag
