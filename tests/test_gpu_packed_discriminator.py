"""The packed discriminator forward (CycleGAN.discriminate_packed over cgvc_discriminator_forward_packed): utterances of different
lengths, every length a multiple of 16, scored in one call.

1. Probabilities against float64 of the oracle's discriminator, per utterance, for both discriminators in every precision and with
   fuse_c1 1 and 0.
2. One packed call == one discriminate() call per utterance (fp32, bf16x3), short utterances included.
3. Host and CUDA inputs give the same bits; the result does not depend on the other utterances of the call.
4. Every argument error launches nothing.
5. The differentiable form (CycleGAN.discriminator_packed, kind 3 tapes): its forward is discriminate_packed() bit for bit; d x_i and all
   30 variable gradients against float64 autograd of the oracle, per utterance and summed; packed against one tape call per utterance;
   the whole-utterance adversarial objective through generator_packed(); deterministic mode; the tape contract and monitor counting.

Lengths: 128-row tile boundaries mid-utterance at every level, utterances of 16 and 32 frames (levels of one or two columns), long
ones (784, 1392).  The comparisons with float64 leave out the 16-frame utterances: d3's instance norms there cover 6 positions, a
statistic float32 and float64 disagree on at the bounds below whatever the engine does, in a separate call as in a packed one."""
import ctypes as C

import numpy as np
import pytest
import torch

from parity_util import rel_l2

pytestmark = pytest.mark.gpu

LENGTHS = [32, 784, 16, 400, 48, 1392, 16, 128, 208]
WELL = [32, 784, 400, 48, 1392, 128, 208]              # every instance norm over >= 12 positions
PRECS = ["fp32", "bf16x3", "bf16", "f16f8"]
TOL = {"fp32": 1e-5, "bf16x3": 1e-3, "bf16": 5e-3, "f16f8": 1e-3}
MAX_BATCH, MAX_FRAMES = 9, 384                         # 9 x 384 >= the 3024 frames of LENGTHS: no growth inside a test


def _model(prec, params, **kw):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='test', max_batch=MAX_BATCH, max_frames=MAX_FRAMES, precision=prec, log_dir='/tmp/cgvc_log',
                      **kw)
    m.set_params({k: v.numpy() for k, v in params.items()})
    return m


@pytest.fixture(scope="module")
def models(oracle_params64):
    out = {p: _model(p, oracle_params64) for p in PRECS}
    yield out
    out.clear()
    torch.cuda.empty_cache()


def _utterances(seed, lengths):
    from oracle import cyclegan_oracle as O
    return [O.synthetic_batch(seed=seed + i, batch=1, frames=T)[0][0].cuda() for i, T in enumerate(lengths)]


def _launches(m):
    n = C.c_ulonglong(0)
    m._lib.cgvc_kernel_launches(C.byref(n))
    return n.value


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("fuse_c1", [1, 0])
def test_packed_probabilities_match_float64(models, oracle_params64, prec, fuse_c1):
    from oracle import cyclegan_oracle as O
    m = models[prec]
    m.set_option("fuse_c1", fuse_c1)
    try:
        xs = _utterances(10, WELL)
        for which in ("A", "B"):
            got = m.discriminate_packed(xs, which)
            with torch.no_grad():
                ref = [O.discriminator_forward(x.double().cpu()[None], oracle_params64, "discriminator_" + which)[0] for x in xs]
            for u, (g, r) in enumerate(zip(got, ref)):
                assert tuple(g.shape) == (6, WELL[u] // 16, 1), (u, tuple(g.shape))
                e = rel_l2(g.double().cpu(), r)
                assert e < TOL[prec], (prec, fuse_c1, which, u, WELL[u], e)
            e = rel_l2(torch.cat([g.reshape(-1) for g in got]).double().cpu(), torch.cat([r.reshape(-1) for r in ref]))
            print("packed discriminator %s %s fuse_c1 %d: rel_l2 %.2e" % (prec, which, fuse_c1, e))
    finally:
        m.set_option("fuse_c1", 1)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_packed_equals_separate_calls(models, prec):
    m = models[prec]
    xs = _utterances(30, LENGTHS)
    for which in ("A", "B"):
        got = m.discriminate_packed(xs, which)
        for u, x in enumerate(xs):
            one = torch.as_tensor(m.discriminate(x[None].cpu().numpy(), which))[0]
            e = rel_l2(got[u].cpu(), one)
            assert e < 1e-5, (prec, which, u, LENGTHS[u], e)


def test_host_input_and_neighbours_do_not_matter(models):
    m = models["bf16x3"]
    xs = _utterances(50, LENGTHS)
    dev = m.discriminate_packed(xs, "B")
    host = m.discriminate_packed([x.cpu().numpy().astype(np.float64) for x in xs], "B")
    for d, h in zip(dev, host):
        assert isinstance(h, np.ndarray) and np.array_equal(d.cpu().numpy(), h)
    # the same utterance among other neighbours, at another offset: the same bits (every tile that reads it sees only its rows)
    perm = list(reversed(range(len(xs))))
    rev = m.discriminate_packed([xs[i] for i in perm], "B")
    for j, i in enumerate(perm):
        assert torch.equal(rev[j], dev[i]), (i, LENGTHS[i])


def test_packed_errors_launch_nothing(models):
    from cgvc import native as N
    m = models["bf16x3"]
    h, lib = m._handle, m._lib
    x = torch.zeros(24 * 4096, device="cuda"); p = torch.empty(6 * 4096 // 16, device="cuda")
    torch.cuda.synchronize()

    def fwd(offs, which=0, n=None):
        o = np.asarray(offs, dtype=np.int64)
        return lib.cgvc_discriminator_forward_packed(h, which, C.c_void_p(x.data_ptr()), C.c_void_p(p.data_ptr()),
                                                     o.ctypes.data_as(C.POINTER(C.c_longlong)), len(o) - 1 if n is None else n, None)
    cap = m._max_batch * m._max_frames
    cases = [("length not a multiple of 16", lambda: fwd([0, 32, 68]), N.ERR_ARG, b"utterance 1"),
             ("empty utterance", lambda: fwd([0, 16, 16]), N.ERR_ARG, b"utterance 1"),
             ("offsets[0] != 0", lambda: fwd([16, 32]), N.ERR_ARG, None),
             ("too many utterances", lambda: fwd(list(range(0, 16 * (m._max_batch + 2), 16))), N.ERR_ARG, None),
             ("no utterances", lambda: fwd([0], n=0), N.ERR_ARG, None),
             ("too many frames", lambda: fwd([0, cap + 16]), N.ERR_ARG, None),
             ("bad which", lambda: fwd([0, 32], which=2), N.ERR_ARG, None)]
    for what, call, code, msg in cases:
        before = _launches(m)
        assert call() == code, (what, lib.cgvc_last_error(h))
        assert _launches(m) == before, (what, "launched")
        if msg:
            assert msg in lib.cgvc_last_error(h), (what, lib.cgvc_last_error(h))
    with pytest.raises(ValueError):
        m.discriminate_packed([torch.zeros(23, 16, device="cuda")], "A")
    from cgvc import _native
    with pytest.raises(_native.CgvcError):
        m.discriminate_packed([torch.zeros(24, 24, device="cuda")], "A")


# ---- the differentiable packed discriminator (CycleGAN.discriminator_packed, kind 3 tapes) -------------------------------------------
GPRECS = ["fp32", "bf16x3", "f16f8"]
NETS = ("generator_A2B", "generator_B2A", "discriminator_A", "discriminator_B")


def _train_model(prec, params, **kw):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=MAX_BATCH, max_frames=MAX_FRAMES, precision=prec, log_dir='/tmp/cgvc_log',
                      **kw)
    m.set_params({k: v.numpy() for k, v in params.items()})
    return m


@pytest.fixture(scope="module")
def gmodels(oracle_params64):
    out = {p: _train_model(p, oracle_params64) for p in GPRECS}
    yield out
    out.clear()
    torch.cuda.empty_cache()


def _upstream(seed, lengths):
    """a random d prob per utterance at the magnitude of the mean of all outputs"""
    total = 6 * sum(T // 16 for T in lengths)
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(6, T // 16, 1, generator=g, dtype=torch.float64) / total).cuda() for T in lengths]


def _check_grads(tag, got, ref, tol):
    total = float(torch.sqrt(sum((r.double() ** 2).sum() for r in ref.values())))
    worst = (0.0, None)
    for name, r in ref.items():
        gn = got[name].double().cpu()
        r = r.double().cpu()
        rn = float(r.norm())
        e = float(gn.norm()) / total if rn < 1e-9 * total else float((gn - r).norm()) / rn
        worst = max(worst, (e, name))
        assert e < tol, (tag, name, e)
    print("%s worst gradient %s %.2e" % (tag, worst[1], worst[0]))
    return worst[0]


def _untouched(m, scope, tag):
    for other in NETS:
        if other != scope:
            assert all(bool((v == 0).all()) for v in m.grads(other).values()), (tag, "GRAD touched outside", other)


@pytest.mark.parametrize("fuse_c1", [1, 0])
def test_tape_forward_is_bitwise_discriminate_packed(gmodels, fuse_c1):
    xs = _utterances(5, LENGTHS)
    for prec, m in gmodels.items():
        m.set_option("fuse_c1", fuse_c1)
        for which in ("A", "B"):
            ref = m.discriminate_packed(xs, which)
            got = m.discriminator_packed(xs, which)
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), (prec, which, fuse_c1)
        m.set_option("fuse_c1", 1)


@pytest.mark.parametrize("which", ["A", "B"])
@pytest.mark.parametrize("fuse_c1", [1, 0])
def test_packed_gradients_match_float64(gmodels, oracle_params64, which, fuse_c1):
    from oracle import cyclegan_oracle as O
    scope = "discriminator_" + which
    xs = _utterances(20 + fuse_c1, WELL)
    gs = _upstream(30 + fuse_c1, WELL)
    P = {k: v.clone().cuda().requires_grad_(True) for k, v in oracle_params64.items() if k.startswith(scope + "/")}
    x64 = [x.double().requires_grad_(True) for x in xs]
    ys = [O.discriminator_forward(x[None], P, scope)[0] for x in x64]
    sum((y * g).sum() for y, g in zip(ys, gs)).backward()
    G_ref = {k: v.grad for k, v in P.items()}
    assert len(G_ref) == 30
    for prec, m in gmodels.items():
        m.set_option("fuse_c1", fuse_c1)
        m.zero_grad()
        xg = [x.clone().requires_grad_(True) for x in xs]
        sum((y * g.float()).sum() for y, g in zip(m.discriminator_packed(xg, which), gs)).backward()
        tag = "packed D[%s %s fuse_c1=%d]" % (prec, which, fuse_c1)
        worst = 0.0
        for u, (x, r) in enumerate(zip(xg, x64)):
            e = rel_l2(x.grad.cpu(), r.grad.cpu()); worst = max(worst, e)
            assert e < TOL[prec], (tag, "d x", u, WELL[u], e)
        print("%s d x worst rel_l2 %.2e" % (tag, worst))
        _check_grads(tag, m.grads(scope), G_ref, TOL[prec])
        _untouched(m, scope, tag)
        m.set_option("fuse_c1", 1)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_packed_gradients_equal_separate_calls(gmodels, prec):
    m = gmodels[prec]
    xs = _utterances(40, LENGTHS)
    gs = [g.float() for g in _upstream(41, LENGTHS)]
    m.zero_grad()
    xg = [x.clone().requires_grad_(True) for x in xs]
    sum((y * g).sum() for y, g in zip(m.discriminator_packed(xg, "A"), gs)).backward()
    packed, dx_p = {k: v.clone() for k, v in m.grads("discriminator_A").items()}, [x.grad for x in xg]
    m.zero_grad()
    dx_s = []
    for x, g in zip(xs, gs):
        xu = x[None].clone().requires_grad_(True)
        (m.discriminator(xu, "A")[0] * g).sum().backward()
        dx_s.append(xu.grad[0])
    sep = m.grads("discriminator_A")
    # the biases of d1 .. d3 feed an instance norm: their gradient is analytically zero, both sides hold float32 rounding of it, so they
    # are measured against the network's gradient (as _check_grads does against float64, where that zero is exact)
    total = float(torch.sqrt(sum((v.double() ** 2).sum() for v in sep.values())))
    worst = 0.0
    for name, r in sep.items():
        d = float((packed[name].double() - r.double()).norm())
        e = d / total if ("downsample2d" in name and name.endswith("/bias")) else d / float(r.double().norm())
        worst = max(worst, e)
        assert e < 1e-5, (prec, name, e)
    print("packed vs separate[%s]: worst gradient rel_l2 %.2e" % (prec, worst))
    for u, (a, b) in enumerate(zip(dx_p, dx_s)):
        assert rel_l2(a.cpu(), b.cpu()) < 1e-5, (prec, u, LENGTHS[u])


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_adversarial_objective_over_whole_utterances(gmodels, oracle_params64, prec):
    """discriminator_packed(generator_packed(xs, 'A2B'), 'B') with the LSGAN generator term mean((p - 1)^2) over all outputs"""
    from oracle import cyclegan_oracle as O
    m = gmodels[prec]
    xs = _utterances(60, WELL)
    m.zero_grad()
    ps = m.discriminator_packed(m.generator_packed(xs, "A2B"), "B")
    nout = sum(p.numel() for p in ps)
    (sum(((p - 1) ** 2).sum() for p in ps) / nout).backward()
    P = {k: v.clone().cuda().requires_grad_(True) for k, v in oracle_params64.items()
         if k.startswith("generator_A2B/") or k.startswith("discriminator_B/")}
    p64 = [O.discriminator_forward(O.generator_forward(x.double()[None], P, "generator_A2B"), P, "discriminator_B")[0] for x in xs]
    (sum(((p - 1) ** 2).sum() for p in p64) / nout).backward()
    for scope in ("generator_A2B", "discriminator_B"):
        _check_grads("adversarial[%s %s]" % (prec, scope), m.grads(scope),
                     {k: v.grad for k, v in P.items() if k.startswith(scope + "/")}, 1e-3)


def test_deterministic_packed_backward(oracle_params64):
    from cgvc import native as N
    xs = _utterances(70, LENGTHS)
    gs = [g.float() for g in _upstream(71, LENGTHS)]
    bits = []
    for fresh in (0, 0, 1):
        if fresh or not bits:
            m = _train_model("bf16x3", oracle_params64, deterministic=True)
        m.zero_grad()
        for which in ("A", "B"):
            xg = [x.clone().requires_grad_(True) for x in xs]
            sum((y * g).sum() for y, g in zip(m.discriminator_packed(xg, which), gs)).backward()
        torch.cuda.synchronize()
        bits.append(m._arenas[N.ARENA_GRAD].clone())
    assert bool((bits[0] != 0).any())
    assert torch.equal(bits[0], bits[1]) and torch.equal(bits[0], bits[2])


def test_packed_tape_contract(oracle_params64):
    from cgvc import native as N
    m = _train_model("bf16x3", oracle_params64, deterministic=True)
    h, lib = m._handle, m._lib
    xs = _utterances(80, LENGTHS)
    gs = [g.float() for g in _upstream(81, LENGTHS)]
    # a second backward of one tape adds exactly the same gradients
    m.zero_grad()
    xg = [x.clone().requires_grad_(True) for x in xs]
    loss = sum((y * g).sum() for y, g in zip(m.discriminator_packed(xg, "B"), gs))
    loss.backward(retain_graph=True)
    torch.cuda.synchronize()
    once, dx1 = m._arenas[N.ARENA_GRAD].clone(), [x.grad.clone() for x in xg]
    assert bool((once != 0).any())
    loss.backward()
    torch.cuda.synchronize()
    assert torch.equal(m._arenas[N.ARENA_GRAD], 2 * once)
    assert all(torch.equal(x.grad, 2 * d) for x, d in zip(xg, dx1))
    # errors launch nothing: a kind 3 tape given to the generator backward, bad arguments of the tape forward
    _, dtape, offsets = m._packed_tape_forward(0, [xs[0], xs[1]], 3)
    x = torch.zeros(24 * 4096, device="cuda"); y = torch.empty_like(x)
    torch.cuda.synchronize()

    def ptr(t):
        return C.c_void_p(t.data_ptr())

    def fwd(offs, which=0, nbytes=None):
        o = np.asarray(offs, dtype=np.int64)
        return lib.cgvc_discriminator_forward_packed_tape(h, which, ptr(x), ptr(y), o.ctypes.data_as(C.POINTER(C.c_longlong)), len(o) - 1,
                                                          ptr(dtape), dtape.numel() if nbytes is None else nbytes, None)
    nb = C.c_size_t(0)
    assert lib.cgvc_tape_bytes(h, 3, 2, int(offsets[-1]), C.byref(nb)) == 0 and nb.value <= dtape.numel()
    cases = [("kind 3 to the generator", lambda: lib.cgvc_generator_backward_tape(h, ptr(dtape), ptr(y), None, None), N.ERR_ARG),
             ("length not a multiple of 16", lambda: fwd([0, 32, 40]), N.ERR_ARG),
             ("bad which", lambda: fwd([0, 32], which=2), N.ERR_ARG),
             ("short tape", lambda: fwd([0, 32, 816], nbytes=dtape.numel() - 1), N.ERR_UNBOUND),
             ("tape bytes of a bad geometry", lambda: lib.cgvc_tape_bytes(h, 3, 2, 40, C.byref(nb)), N.ERR_ARG)]
    for what, call, code in cases:
        before = _launches(m)
        assert call() == code, (what, lib.cgvc_last_error(h))
        assert _launches(m) == before, (what, "launched")


def test_monitor_mode_counts_packed_gradients_into_network_1(oracle_params64):
    m = _train_model("f16f8", oracle_params64, loss_scale='monitor', loss_scale_per_network=True)
    xs = _utterances(90, WELL)
    gs = [g.float() for g in _upstream(91, WELL)]
    counts = []
    for mult in (1.0, 2.0 ** 20):
        before = m.loss_scale_state()
        m.zero_grad()
        sum((y * (g * mult)).sum() for y, g in zip(m.discriminator_packed(xs, 'A'), gs)).backward()
        after = m.loss_scale_state()
        counts.append((after["sat_grad_G"] - before["sat_grad_G"], after["sat_grad_D"] - before["sat_grad_D"]))
    print("monitor: saturated packed D gradient-plane groups (G, D) %s (mean-loss magnitude), %s (x 2^20)" % tuple(counts))
    assert counts[0] == (0, 0) and counts[1][0] == 0 and counts[1][1] > 0
