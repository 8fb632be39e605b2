"""The packed generator as a differentiable torch operator (CycleGAN.generator_packed over the kind 2 activation tapes of include/cgvc.h):
utterances of different lengths, forward and backward, in one call each.

1. The outputs are test_packed()'s bit for bit, in every precision and with edge_lower 1 and 0.
2. d x_i and every variable gradient against float64 autograd of the oracle, per utterance and summed, from a random upstream gradient at
   the mean-loss magnitude; GRAD outside the network untouched.
3. One packed call == one generator() call per utterance: the gradients they add and the d x they return.
4. A whole-utterance objective in PyTorch: the cycle loss through two chained packed calls against float64, then one adam_step against a
   float64 TF-Adam update from the unscaled grads() (the packed call's loss scale is removed exactly once).
5. Deterministic mode: the same GRAD bits on a repeat and in a fresh engine.
6. The contract's errors launch nothing; a second backward of one tape adds exactly the same gradients; monitor-mode counting.

Lengths: tile boundaries mid-utterance at T, T/2 and T/4; utterances shorter than the 15-tap halo (4, 8, 12 frames); a length test()
sends through a specialised instance-norm kernel (128; left out of the separate-call comparison, whose norms sum in another order);
long ones (784, 1400).  The comparisons with float64 (2, 4) and the saturation count at the mean-loss magnitude (6) take 40, 44 and 48
frames instead of 4, 8 and 12: at T/4 those are instance norms over 1, 2 and 3 rows, whose gradient is analytically (near) zero -- only
the 1e-6 in the variance keeps it from vanishing -- and amplified by the inverse spread of one to three values, so float32 and float64
disagree there by orders of magnitude above the bounds whatever the engine does, in one tape call per utterance as in one packed call
(and the F16F8 planes saturate); the separate-call comparison (3), the forward and the deterministic and contract tests keep them."""
import ctypes as C

import numpy as np
import pytest
import torch

from parity_util import rel_l2

pytestmark = pytest.mark.gpu

LENGTHS = [36, 516, 4, 128, 784, 12, 1400, 8, 132]
PLAIN = [36, 516, 4, 784, 12, 1400, 8, 132]          # without the lengths of test()'s specialised instance-norm kernels
WELL = [36, 516, 40, 128, 784, 44, 1400, 48, 132]    # every instance norm over >= 9 rows: well-conditioned against float64
PRECS = ["fp32", "bf16x3", "f16f8"]
TOL = {"fp32": 1e-5, "bf16x3": 1e-3, "f16f8": 1e-3}
NETS = ("generator_A2B", "generator_B2A", "discriminator_A", "discriminator_B")
MAX_BATCH, MAX_FRAMES = 9, 344                       # 9 x 344 >= the 3020 frames of LENGTHS: no growth inside a test


def _model(prec, params=None, **kw):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=MAX_BATCH, max_frames=MAX_FRAMES, precision=prec, log_dir='/tmp/cgvc_log',
                      **kw)
    if params is not None:
        m.set_params({k: v.numpy() for k, v in params.items()})
    return m


@pytest.fixture(scope="module")
def models(oracle_params64):
    out = {p: _model(p, oracle_params64) for p in PRECS}
    yield out
    out.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def params_cuda(oracle_params64):
    return {k: v.cuda() for k, v in oracle_params64.items()}


def _utterances(seed, lengths):
    from oracle import cyclegan_oracle as O
    return [O.synthetic_batch(seed=seed + i, batch=1, frames=T)[0][0].cuda() for i, T in enumerate(lengths)]


def _upstream(seed, lengths):
    total = 24 * sum(lengths)
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(24, T, generator=g, dtype=torch.float64) / total).cuda() for T in lengths]


def _launches(m):
    n = C.c_ulonglong(0)
    m._lib.cgvc_kernel_launches(C.byref(n))
    return n.value


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


def _untouched(m, scope, tag):
    for other in NETS:
        if other != scope:
            assert all(bool((v == 0).all()) for v in m.grads(other).values()), (tag, "GRAD touched outside", other)


# ---- 1. forward ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16", "f16f8"])
def test_packed_tape_forward_is_bitwise_test_packed(models, oracle_params64, prec):
    m = models[prec] if prec in models else _model(prec, oracle_params64)
    xs = _utterances(10, LENGTHS)
    for edge in (1, 0):
        m.set_option("edge_lower", edge)
        for d in ("A2B", "B2A"):
            with torch.no_grad():
                ys = m.generator_packed(xs, d)
            ref = m.test_packed(xs, d)
            assert len(ys) == len(xs)
            for u, (y, r) in enumerate(zip(ys, ref)):
                assert y.shape == (24, LENGTHS[u]) and torch.equal(y, r), (prec, edge, d, u)
    m.set_option("edge_lower", 1)


# ---- 2. gradients against float64 ----------------------------------------------------------------------------------------------------
def _oracle(params_cuda, scope, xs, gs):
    """sum over utterances of the oracle's autograd: d x_i and the variable gradients of sum_i <G(x_i), g_i>"""
    from oracle import cyclegan_oracle as O
    P = {k: v.clone().requires_grad_(True) for k, v in params_cuda.items() if k.startswith(scope + "/")}
    xx = [x.double().clone().requires_grad_(True) for x in xs]
    loss = sum((O.generator_forward(x[None], P, scope)[0] * g).sum() for x, g in zip(xx, gs))
    loss.backward()
    return [x.grad for x in xx], {k: v.grad for k, v in P.items()}


@pytest.mark.parametrize("direction", ["A2B", "B2A"])
@pytest.mark.parametrize("edge", [1, 0])
def test_packed_gradients_match_float64(models, params_cuda, direction, edge):
    scope = "generator_" + direction
    xs = _utterances(20 + edge, WELL)
    gs = _upstream(30 + edge, WELL)
    dx_ref, G_ref = _oracle(params_cuda, scope, xs, gs)
    for prec in PRECS:
        m = models[prec]
        m.set_option("edge_lower", edge)
        m.zero_grad()
        xg = [x.clone().requires_grad_(True) for x in xs]
        ys = m.generator_packed(xg, direction)
        sum((y * g.float()).sum() for y, g in zip(ys, gs)).backward()
        tag = "packed[%s %s edge_lower=%d]" % (prec, direction, edge)
        worst = 0.0
        for u, (x, r) in enumerate(zip(xg, dx_ref)):
            e = rel_l2(x.grad.cpu().numpy(), r.cpu().numpy()); worst = max(worst, e)
            assert e < TOL[prec], (tag, "d x", u, WELL[u], e)
        print("%s d x worst rel_l2 %.2e" % (tag, worst))
        _check_grads(tag, m.grads(scope), G_ref, TOL[prec])
        _untouched(m, scope, tag)
        m.set_option("edge_lower", 1)


# ---- 3. one packed call == one call per utterance ------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_packed_equals_separate_calls(models, prec):
    m = models[prec]
    xs = _utterances(40, PLAIN)
    gs = _upstream(41, PLAIN)
    for d in ("A2B", "B2A"):
        scope = "generator_" + d
        m.zero_grad()
        sep_dx = []
        for x, g in zip(xs, gs):
            xg = x[None].clone().requires_grad_(True)
            (m.generator(xg, d) * g.float()[None]).sum().backward()
            sep_dx.append(xg.grad[0])
        sep = {k: v.clone() for k, v in m.grads(scope).items()}
        m.zero_grad()
        xg = [x.clone().requires_grad_(True) for x in xs]
        sum((y * g.float()).sum() for y, g in zip(m.generator_packed(xg, d), gs)).backward()
        got = m.grads(scope)
        total = float(torch.sqrt(sum((r.double() ** 2).sum() for r in sep.values())))
        worst = 0.0
        for name, r in sep.items():
            rn = float(r.double().norm())
            # biases feeding an instance norm (analytically zero): their rounding noise compared against the network's gradient
            e = float((got[name].double() - r.double()).norm()) / (rn if rn >= 1e-9 * total else total)
            worst = max(worst, e)
            assert e < 1e-5, (prec, d, name, e)
        for u, (x, r) in enumerate(zip(xg, sep_dx)):
            e = rel_l2(x.grad.cpu().numpy(), r.cpu().numpy())
            assert e < 1e-5, (prec, d, "d x", PLAIN[u], e)
        print("packed vs separate [%s %s]: worst gradient rel_l2 %.2e" % (prec, d, worst))


# ---- 4. a whole-utterance objective --------------------------------------------------------------------------------------------------
def _cycle_loss(ys, xs, total, signs=None):
    """the L1 cycle loss over all utterances; with signs (the engine's sign(y - x)), the same loss at the float64 point, where the
    subgradient takes the engine's signs: an element whose y - x is within rounding of 0 would otherwise flip the sign of its gradient"""
    if signs is None:
        return sum((y - x).abs().sum() for y, x in zip(ys, xs)) / total
    return sum((s * (y - x)).sum() for y, x, s in zip(ys, xs, signs)) / total


def _reset_adam(m, params):
    from cgvc import native as N
    m.set_params({k: v.numpy() for k, v in params.items()})
    m._arenas[N.ARENA_ADAM_M].zero_(); m._arenas[N.ARENA_ADAM_V].zero_()
    m._chk(m._lib.cgvc_set_adam_step(m._handle, 0))


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_cycle_objective_and_adam(models, oracle_params64, params_cuda, prec):
    from oracle import cyclegan_oracle as O
    m = models[prec]
    xs = _utterances(50, WELL)
    total = 24 * sum(WELL)
    _reset_adam(m, oracle_params64)
    m.zero_grad()
    ys = m.generator_packed(m.generator_packed(xs, "A2B"), "B2A")
    signs = [torch.sign(y.detach() - x).double() for y, x in zip(ys, xs)]
    _cycle_loss(ys, xs, total).backward()
    # float64 reference of both generators' gradients
    P = {k: v.clone().requires_grad_(True) for k, v in params_cuda.items() if k.startswith("generator_")}
    y64 = [O.generator_forward(O.generator_forward(x.double()[None], P, "generator_A2B"), P, "generator_B2A")[0] for x in xs]
    _cycle_loss(y64, [x.double() for x in xs], total, signs).backward()
    ref = {k: v.grad for k, v in P.items()}
    for scope in ("generator_A2B", "generator_B2A"):
        _check_grads("cycle[%s %s]" % (prec, scope), m.grads(scope), {k: v for k, v in ref.items() if k.startswith(scope + "/")}, 1e-3)
    g = {k: v.double().cpu() for k, v in m.grads().items()}
    lr_g, lr_d = 2e-4, 1e-4
    m.adam_step(lr_g, lr_d)
    got = m.get_params()
    b1, b2, eps = 0.5, 0.999, 1e-8
    lr_t = lr_g * np.sqrt(1 - b2) / (1 - b1)
    worst = 0.0
    for name in g:
        if not name.startswith("generator_"):
            continue
        p0 = oracle_params64[name].float().double()
        mm, vv = (1 - b1) * g[name], (1 - b2) * g[name] ** 2
        p_ref = p0 - lr_t * mm / (vv.sqrt() + eps)
        e = rel_l2(got[name], p_ref.numpy()); worst = max(worst, e)
        assert e < 1e-6, (prec, name, e)
    print("adam after the packed cycle loss [%s]: worst parameter rel_l2 vs float64 TF-Adam %.2e" % (prec, worst))
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})


# ---- 5. deterministic mode -----------------------------------------------------------------------------------------------------------
def test_deterministic_packed_backward(oracle_params64):
    from cgvc import native as N
    xs = _utterances(60, LENGTHS)
    gs = [g.float() for g in _upstream(61, LENGTHS)]
    bits = []
    for fresh in (0, 0, 1):
        if fresh or not bits:
            m = _model("bf16x3", oracle_params64, deterministic=True)
        m.zero_grad()
        for d in ("A2B", "B2A"):
            xg = [x.clone().requires_grad_(True) for x in xs]
            sum((y * g).sum() for y, g in zip(m.generator_packed(xg, d), gs)).backward()
        torch.cuda.synchronize()
        bits.append(m._arenas[N.ARENA_GRAD].clone())
    assert bool((bits[0] != 0).any())
    assert torch.equal(bits[0], bits[1]) and torch.equal(bits[0], bits[2])


# ---- 6. contract ---------------------------------------------------------------------------------------------------------------------
def test_packed_tape_errors_launch_nothing(models):
    from cgvc import native as N
    m = models["bf16x3"]
    h, lib = m._handle, m._lib
    xs = _utterances(70, [36, 132])
    _, gtape, offsets = m._packed_tape_forward(0, xs)
    x = torch.zeros(24 * 4096, device="cuda"); y = torch.empty_like(x)
    dprob = torch.zeros(1, 6, 8, 1, device="cuda")
    torch.cuda.synchronize()

    def ptr(t):
        return C.c_void_p(t.data_ptr())

    def fwd(offs, n=None, direction=0, nbytes=None):
        o = np.asarray(offs, dtype=np.int64)
        return lib.cgvc_generator_forward_packed_tape(h, direction, ptr(x), ptr(y), o.ctypes.data_as(C.POINTER(C.c_longlong)),
                                                      len(o) - 1 if n is None else n, ptr(gtape),
                                                      gtape.numel() if nbytes is None else nbytes, None)
    cap = m._max_batch * m._max_frames                   # (an earlier test may have grown the engine)
    cases = [("bad offsets", lambda: fwd([0, 36, 134]), N.ERR_ARG),
             ("too many utterances", lambda: fwd(list(range(0, 4 * (m._max_batch + 2), 4))), N.ERR_ARG),
             ("too many frames", lambda: fwd([0, cap + 4]), N.ERR_ARG),
             ("bad direction", lambda: fwd([0, 36], direction=2), N.ERR_DIRECTION),
             ("short tape", lambda: fwd([0, 36, 168], nbytes=gtape.numel() - 1), N.ERR_UNBOUND),
             ("kind 2 to the discriminator", lambda: lib.cgvc_discriminator_backward_tape(h, ptr(gtape), ptr(dprob), None, None), N.ERR_ARG),
             ("stale", None, N.ERR_ARG)]
    for what, call, code in cases:
        if call is None:                                       # the parameters change after the forward
            m._params_updated()
            torch.cuda.synchronize()
            call = lambda: lib.cgvc_generator_backward_tape(h, ptr(gtape), ptr(y), None, None)    # noqa: E731
        before = _launches(m)
        assert call() == code, (what, lib.cgvc_last_error(h))
        assert _launches(m) == before, (what, "launched")
    # the same errors through the Python operator
    with pytest.raises(Exception, match="Conversion direction must be specified."):
        m.generator_packed(xs, "A2A")
    with pytest.raises(ValueError):
        m.generator_packed([torch.zeros(23, 8, device="cuda")], "A2B")
    with pytest.raises(TypeError):
        m.generator_packed([torch.zeros(24, 8)], "A2B")
    from cgvc import _native
    with pytest.raises(_native.CgvcError):
        m.generator_packed([torch.zeros(24, 6, device="cuda")], "A2B")


def test_packed_second_backward_doubles_grad_exactly(oracle_params64):
    from cgvc import native as N
    m = _model("bf16x3", oracle_params64, deterministic=True)
    xs = _utterances(80, LENGTHS)
    gs = [g.float() for g in _upstream(81, LENGTHS)]
    m.zero_grad()
    xg = [x.clone().requires_grad_(True) for x in xs]
    loss = sum((y * g).sum() for y, g in zip(m.generator_packed(xg, 'B2A'), gs))
    loss.backward(retain_graph=True)
    torch.cuda.synchronize()
    once, dx1 = m._arenas[N.ARENA_GRAD].clone(), [x.grad.clone() for x in xg]
    assert bool((once != 0).any())
    loss.backward()
    torch.cuda.synchronize()
    assert torch.equal(m._arenas[N.ARENA_GRAD], 2 * once)
    assert all(torch.equal(x.grad, 2 * d) for x, d in zip(xg, dx1))


def test_monitor_mode_counts_packed_gradients_into_network_0(oracle_params64):
    m = _model("f16f8", oracle_params64, loss_scale='monitor', loss_scale_per_network=True)
    xs = _utterances(90, WELL)
    gs = [g.float() for g in _upstream(91, WELL)]
    counts = []
    for mult in (1.0, 2.0 ** 20):
        before = m.loss_scale_state()
        m.zero_grad()
        sum((y * (g * mult)).sum() for y, g in zip(m.generator_packed(xs, 'A2B'), gs)).backward()
        after = m.loss_scale_state()
        counts.append((after["sat_grad_G"] - before["sat_grad_G"], after["sat_grad_D"] - before["sat_grad_D"]))
    print("monitor: saturated packed gradient-plane groups (G, D) %s (mean-loss magnitude), %s (x 2^20)" % tuple(counts))
    assert counts[0] == (0, 0) and counts[1][0] > 0 and counts[1][1] == 0
