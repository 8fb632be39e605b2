"""Dynamic loss scaling of the differentiable networks (tape_loss_scale='dynamic', include/cgvc.h cgvc_apply_gradients).

1. Without an overflow, dynamic tapes + apply_gradients() give what static tapes + adam_step() give, bit for bit, at the same scale.
2. An upstream gradient that saturates the gradient planes skips the step and halves the saturating network's scale; at the settled
   scale the gradients match float64.  Static tapes in monitor mode count the same saturation.
3. The corner of DESIGN.md section 10 (batch 1, lambda_cycle = 1e4, per-network scales) through tapes.
4. A non-finite upstream gradient skips the step and sets its network's nonfinite bit.  5. Growth.  6. Packed tapes.
7. A one-rank communicator, and two identical runs, give the same bits.  8. Refusals launch nothing; tapes go stale.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NETS = ("generator_A2B", "generator_B2A", "discriminator_A", "discriminator_B")
LR = (2e-4, 1e-4)


def _model(prec, batch, params, frames=128, tape='dynamic', ls='dynamic', nets=False, det=False, data_parallel=False, **opts):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=frames, precision=prec, log_dir='/tmp/cgvc_log',
                      loss_scale=ls, tape_loss_scale=tape, loss_scale_per_network=nets, deterministic=det, data_parallel=data_parallel)
    for k, v in opts.items():
        m.set_option(k, v)
    m.set_params({k: v.numpy() for k, v in params.items()})
    return m


def _batch(seed, batch, frames):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=seed, batch=batch, frames=frames)
    return A.cuda(), B.cuda()


def _launches(m):
    n = C.c_ulonglong(0)
    m._lib.cgvc_kernel_launches(C.byref(n))
    return n.value


def _set_scales(m, s_G, s_D=None, good=0, skipped=0):
    m._chk(m._lib.cgvc_set_loss_scale_state(m._handle, float(s_G), good, skipped, m._stream()))
    if m.loss_scale_per_network and s_D is not None:
        m._chk(m._lib.cgvc_set_loss_scale_net_state(m._handle, 1, float(s_D), good, m._stream()))


def _snap(m):
    """PARAM, ADAM_M, ADAM_V, GRAD and the Adam step count"""
    from cgvc import native as N
    torch.cuda.synchronize()
    t = C.c_longlong(0)
    m._chk(m._lib.cgvc_get_adam_step(m._handle, C.byref(t)))
    return [m._arenas[a].clone() for a in (N.ARENA_PARAM, N.ARENA_ADAM_M, N.ARENA_ADAM_V, N.ARENA_GRAD)] + [t.value]


def _same(a, b, n=3):
    return all(torch.equal(x, y) for x, y in zip(a[:n], b[:n])) and a[4] == b[4]


def l1_loss(y, y_hat):          # utils.py:6-8
    return torch.mean(torch.abs(y - y_hat))


def l2_loss(y, y_hat):          # utils.py:10-12
    return torch.mean(torch.square(y - y_hat))


def python_step(m, A, B, lambda_cycle, lambda_identity):
    """model.py:44-108 on the differentiable operators (test_gpu_autograd.py): GRAD ends up loss-scaled as the tapes formed it"""
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


def _worst(got, ref, floor=1e-9):
    """the worst relative L2 error of the gradient tensors against a reference; those under floor x their network's norm (conv biases
    feeding an instance norm: analytically zero) against that norm"""
    total = {net: float(torch.sqrt(sum((r.double() ** 2).sum() for k, r in ref.items() if k.startswith(net))))
             for net in {k.split("/")[0] for k in ref}}
    worst = (0.0, None)
    for name, r in ref.items():
        g, r = got[name].double().reshape(r.shape), r.double().to(got[name].device)
        net = name.split("/")[0]
        rn = float(r.norm())
        e = float((g - r).norm()) / (rn if rn > floor * total[net] else total[net])
        worst = max(worst, (e if np.isfinite(e) else float("inf"), name))
    return worst


# ---- 1. equal to static tapes + adam_step where nothing overflows ------------------------------------------------------------------
@pytest.mark.parametrize("graph", [0, 1])
@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_equal_to_adam_step_without_overflow(oracle_params64, prec, graph):
    A, B = _batch(9, 2, 128)
    s = _model(prec, 2, oracle_params64, tape='static', ls='static', det=True, cuda_graph=graph)
    d = _model(prec, 2, oracle_params64, det=True, cuda_graph=graph)
    _set_scales(d, s.tape_loss_scale(2))
    g = torch.randn(A.shape, generator=torch.Generator().manual_seed(5)).cuda() / A.numel()
    gp = torch.randn(2, 6, 8, 1, generator=torch.Generator().manual_seed(6)).cuda() / 96
    dins = []
    for m in (s, d):                       # each tape backward's d in
        m.zero_grad()
        xs = [A.clone().requires_grad_(True) for _ in range(2)]
        (m.generator(xs[0], 'A2B') * g).sum().backward()
        (m.discriminator(xs[1], 'B') * gp).sum().backward()
        dins.append([x.grad for x in xs])
    assert all(torch.equal(a, b) for a, b in zip(*dins))
    for m in (s, d):
        python_step(m, A, B, 10.0, 5.0)
    before = _snap(s)
    assert torch.equal(before[3], _snap(d)[3])                  # GRAD
    s.adam_step(*LR)
    d.apply_gradients(*LR)
    st = d.loss_scale_state()
    a, b = _snap(s), _snap(d)
    assert _same(a, b) and a[4] == 1 and not torch.equal(a[0], before[0])
    assert not st["last_skipped"] and st["skipped"] == 0 and st["scale"] == s.tape_loss_scale(2)


# ---- 2. overflow skips ---------------------------------------------------------------------------------------------------------------
def _gen_oracle(params, scope, x, g):
    from oracle import cyclegan_oracle as O
    P = {k: v.cuda().clone().requires_grad_(True) for k, v in params.items() if k.startswith(scope + "/")}
    y = O.generator_forward(x.double(), P, scope)
    (y * g.double()).sum().backward()
    return {k: v.grad for k, v in P.items()}


@pytest.mark.parametrize("nets", [False, True])
def test_overflow_skips_and_settles(oracle_params64, nets):
    """a sum-reduced L1 loss: its upstream gradient is 3072 times (the elements) the mean-loss size the static scale is made for, so the
    generator's planes saturate until its scale has fallen"""
    x, tgt = _batch(31, 1, 128)
    m = _model("f16f8", 1, oracle_params64, nets=nets, det=True)
    seen = []
    for i in range(14):
        m.zero_grad()
        y = m.generator(x, 'A2B')
        (y - tgt).abs().sum().backward()
        got = {k: v.clone() for k, v in m.grads("generator_A2B").items()}
        g_up = torch.sign(y.detach() - tgt)
        before = _snap(m)
        m.apply_gradients(*LR)
        st = m.loss_scale_state()
        seen.append((st["scale"], st.get("scale_D"), st["sat_grad"], st["last_skipped"], st["skipped"]))
        if not st["last_skipped"]:
            break
        assert _same(before, _snap(m)) and st["skipped"] == i + 1
    print("tape dynamic (per network %s): (scale, s_D, sat_grad, skipped, skips) per step: %s" % (nets, seen))
    assert seen[0][3] and not seen[-1][3]
    assert [s[0] for s in seen[:-1]] == [512.0 / 2 ** (i + 1) for i in range(len(seen) - 1)]
    if nets:
        assert all(s[1] == 512.0 for s in seen)                    # only the saturating network's scale halves
    worst = _worst(got, _gen_oracle(oracle_params64, "generator_A2B", x, g_up))
    print("settled at %g: worst generator gradient vs float64 %.3e (%s)" % (seen[-1][0], worst[0], worst[1]))
    assert worst[0] < 1e-3
    # the same loss on static tapes: monitor mode sees the saturation the static scale causes
    mon = _model("f16f8", 1, oracle_params64, tape='static', ls='monitor')
    c0 = mon.loss_scale_state()["sat_grad"]
    (mon.generator(x, 'A2B') - tgt).abs().sum().backward()
    sat = mon.loss_scale_state()["sat_grad"] - c0
    print("static tapes, monitor mode: %d saturated gradient-plane groups" % sat)
    assert sat > 0


# ---- 3. the corner --------------------------------------------------------------------------------------------------------------------
def test_the_corner_through_tapes(oracle_params64):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=60, batch=1, frames=128, dtype=torch.float64)
    A32, B32 = A.float().cuda(), B.float().cuda()
    m = _model("f16f8", 1, oracle_params64, nets=True, det=True)
    seen = []
    for _ in range(14):
        python_step(m, A32, B32, 1e4, 5.0)
        got = {k: v.clone() for k, v in m.grads().items()}
        m.apply_gradients(*LR)
        st = m.loss_scale_state()
        seen.append((st["scale_G"], st["scale_D"], st["sat_grad_G"], st["sat_grad_D"], st["last_skipped"]))
        if not st["last_skipped"]:
            break
    print("tapes, per-network dynamic, lambda_cycle 1e4: (s_G, s_D, sat G, sat D, skipped) per step: %s" % seen)
    assert seen[0][4] and not seen[-1][4]
    _, Gref, _, _ = O.gradients(A, B, oracle_params64, 1e4, 5.0)
    assert len(Gref) == len(got) == 280
    worst = _worst(got, Gref)
    print("settled at s_G %g, s_D %g: worst of 280 gradients vs float64 %.3e (%s)" % (seen[-1][0], seen[-1][1], worst[0], worst[1]))
    assert worst[0] < 1e-3


# ---- 4. non-finite, 5. growth -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_nonfinite_upstream_skips(oracle_params64, prec):
    x, _ = _batch(33, 1, 128)
    m = _model(prec, 1, oracle_params64)
    for kind, bit in (("gen", 1), ("disc", 2)):
        m.zero_grad()
        y = m.generator(x, 'B2A') if kind == "gen" else m.discriminator(x, 'A')
        g = torch.full_like(y, 1.0 / y.numel())
        g.view(-1)[7] = float("inf")
        y.backward(g)
        before = _snap(m)
        scale = m.loss_scale_state()["scale"]
        m.apply_gradients(*LR)
        st = m.loss_scale_state()
        print("[%s] inf in d %s: %s" % (prec, "out" if kind == "gen" else "prob", st))
        assert st["last_skipped"] and st["nonfinite"] == bit and _same(before, _snap(m))
        assert st["scale"] == (1.0 if prec == "bf16x3" else scale / 2)


def test_growth(oracle_params64):
    x, _ = _batch(34, 1, 128)
    m = _model("f16f8", 1, oracle_params64, loss_scale_growth_interval=2)
    _set_scales(m, 256.0)
    g = torch.randn(1, 24, 128, generator=torch.Generator().manual_seed(8)).cuda() / 3072
    scales = []
    for _ in range(2):
        m.zero_grad()
        (m.generator(x, 'A2B') * g).sum().backward()
        m.apply_gradients(*LR)
        scales.append(m.loss_scale_state()["scale"])
    assert scales == [256.0, 512.0]


# ---- 6. packed tapes ------------------------------------------------------------------------------------------------------------------
def test_packed_tapes_follow_the_scaler(oracle_params64):
    lens = (64, 128, 96)
    xs = [torch.randn(24, t, generator=torch.Generator().manual_seed(40 + t)).cuda() for t in lens]
    m = _model("f16f8", 3, oracle_params64, nets=True, det=True)

    def lsgan(ps):
        return sum(l2_loss(torch.ones_like(p), p) for p in ps)
    _set_scales(m, 512.0, 512.0)
    m.zero_grad()
    lsgan(m.discriminator_packed(m.generator_packed(xs, 'A2B'), 'B')).backward()
    packed = {k: v.clone() for k, v in m.grads().items()}
    m.zero_grad()
    lsgan([m.discriminator(m.generator(x[None], 'A2B'), 'B') for x in xs]).backward()
    single = m.grads()
    worst = _worst(packed, {k: v for k, v in single.items() if k.startswith(("generator_A2B", "discriminator_B"))}, floor=1e-4)
    print("packed vs per-utterance tapes at s_G = s_D = 512: worst gradient %.3e (%s)" % worst)
    assert worst[0] < 3e-3
    # a generator scale that saturates: the packed step is skipped, and only s_G halves
    _set_scales(m, 2.0 ** 24, 512.0)
    m.zero_grad()
    lsgan(m.discriminator_packed(m.generator_packed(xs, 'A2B'), 'B')).backward()
    m.apply_gradients(*LR)
    st = m.loss_scale_state()
    assert st["last_skipped"] and st["scale_G"] == 2.0 ** 23 and st["scale_D"] == 512.0
    assert st["sat_grad_G"] > 0 or st["nonfinite"] & 1


# ---- 7. data parallel and determinism -------------------------------------------------------------------------------------------------
def test_single_rank_communicator_and_determinism(oracle_params64):
    import torch.distributed as dist
    if not dist.is_initialized():
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29579", rank=0, world_size=1)
    A, B = _batch(35, 1, 128)
    runs = []
    for dp, pipelined in ((False, 1), (False, 1), (True, 1), (True, 0)):
        m = _model("f16f8", 1, oracle_params64, nets=True, det=True, data_parallel=dp, pipelined_comm=pipelined)
        _set_scales(m, 2.0 ** 24, 2.0 ** 24)
        python_step(m, A, B, 10.0, 5.0)
        m.apply_gradients(*LR)                                     # skipped
        st0 = m.loss_scale_state()
        _set_scales(m, 1024.0, 1024.0, skipped=1)
        python_step(m, A, B, 10.0, 5.0)
        m.apply_gradients(*LR)
        st1 = m.loss_scale_state()
        torch.cuda.synchronize()
        runs.append((_snap(m), st0, st1, m._ls_dev.clone(), m._lsn_dev.clone()))
        print("[communicator %s, pipelined %d] %s | %s" % (dp, pipelined, st0, st1))
        del m
        torch.cuda.empty_cache()
    ref = runs[0]
    assert ref[1]["last_skipped"] and not ref[2]["last_skipped"] and ref[0][4] == 1
    for r in runs[1:]:
        assert _same(ref[0], r[0], 4) and r[1] == ref[1] and r[2] == ref[2]
        assert torch.equal(r[3], ref[3]) and torch.equal(r[4], ref[4])


# ---- 8. contract ----------------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing_and_tapes_go_stale(oracle_params64):
    import cgvc
    from cgvc import native as N
    m = _model("f16f8", 1, oracle_params64, tape='static', ls='static')
    h, lib = m._handle, m._lib
    for what, call, code in (("option off", lambda: lib.cgvc_apply_gradients(h, 1e-4, 1e-4, None), N.ERR_ARG),
                             ("not in dynamic mode", lambda: lib.cgvc_set_option(h, b"tape_loss_scale", 1), N.ERR_ARG)):
        before = _launches(m)
        assert call() == code, what
        assert _launches(m) == before, what
    m.set_option("loss_scale", 2)
    m.set_option("tape_loss_scale", 1)
    assert lib.cgvc_set_option(h, b"loss_scale", 0) == N.ERR_ARG
    before = _launches(m)
    assert lib.cgvc_apply_gradients(h, 1e-4, 1e-4, None) == N.ERR_ARG          # no scale yet
    assert _launches(m) == before
    t = cgvc.CycleGAN(num_features=24, mode='test', max_batch=1, max_frames=128, precision="f16f8", loss_scale='dynamic',
                      tape_loss_scale='dynamic')
    before = _launches(t)
    assert t._lib.cgvc_apply_gradients(t._handle, 1e-4, 1e-4, None) == N.ERR_UNBOUND
    assert _launches(t) == before
    # a tape written before apply_gradients is stale afterwards, whether the step went through or was skipped
    x, _ = _batch(36, 1, 128)
    for s in (512.0, 2.0 ** 24):
        _set_scales(m, s)
        y = m.generator(x.clone().requires_grad_(True), 'A2B')
        y.mean().backward(retain_graph=True)
        m.apply_gradients(*LR)
        assert m.loss_scale_state()["last_skipped"] == (s > 512.0)
        with pytest.raises(RuntimeError, match="stale"):
            y.mean().backward()
        m.zero_grad()
