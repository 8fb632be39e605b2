"""Per-network loss scales (engine option "loss_scale_per_network", include/cgvc.h) and the underflow counters of the F16F8 gradient
planes.

a. Every counted plane writer adds, besides its saturation count, the groups whose fp16 plane lies below the lower edge (ufl) and the
   groups it counted into the handle's plane counters: both equal the numpy reference below, built on f16f8_ref.fp16_rn, for operands
   spread over 2^-40 .. 2^20 with the edge values (NaN, inf, +-0, fp16 subnormals) among them.
b. The train step: with both scales equal, the per-network step is the single-scale step bit for bit (deterministic mode) and the
   per-network saturation counts sum to the single-scale count; s_D = s_G 2^+-4 moves the update by no more than rounding.
c. Attribution and the corner DESIGN.md section 10 leaves open: batch 1, lambda_cycle = 1e4.  The generators' planes saturate, the
   discriminators' do not; in dynamic mode only s_G falls, and the gradients at the settled scales are compared with float64.
d. Mechanics: per-network halving (saturation, non-finite values in one range), per-network growth, skipped steps, save / load,
   CUDA graphs, determinism and the one-rank communicator paths.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import f16f8_ref as R
import glu_ref as G

pytestmark = pytest.mark.gpu

F16F8 = 3
FP16_MIN_NORMAL = 2.0 ** -14


# ---- the reference -----------------------------------------------------------------------------------------------------------------
def ufl_elements(x):
    """per element: finite, non-zero and its fp16 value below the smallest normal fp16 (subnormal or flushed to zero)"""
    x = np.asarray(x, np.float32).reshape(-1)
    with np.errstate(invalid="ignore"):
        return np.isfinite(x) & (x != 0) & (np.abs(R.fp16_rn(x).astype(np.float64)) < FP16_MIN_NORMAL)


def ufl_counts(x):
    """(ufl, groups) of the 4-value groups of x (flattened, size a multiple of 4), as cgvc_count_planes adds them"""
    u = ufl_elements(x)
    assert u.size % 4 == 0
    return int(u.reshape(-1, 4).any(axis=1).sum()), u.size // 4


def test_reference_on_the_edges():
    x = np.array([2.0 ** -14, 2.0 ** -15, 0.0, -0.0, np.nan, np.inf, 1023.5 * 2.0 ** -24, 1023.4 * 2.0 ** -24, 1e-30, -1e-30, 1.0, 2.0 ** -24],
                 np.float32)
    assert ufl_elements(x).tolist() == [False, True, False, False, False, False, False, True, True, True, False, True]


# ---- a. the writers -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    ctr = torch.zeros(2, dtype=torch.int64, device="cuda")
    N.check(h, lib.cgvc_set_plane_counters(h, C.c_void_p(ctr.data_ptr())))
    yield lib, h, N, ctr
    N.check(h, lib.cgvc_set_plane_counters(h, None))
    lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _planes(n):
    return torch.empty(n, dtype=torch.float16, device="cuda"), torch.empty(2 * n, dtype=torch.uint8, device="cuda")


def _wide(n, rng):
    """n fp32 values: log-uniform magnitudes 2^-40 .. 2^20 of random sign, with the edge table of f16f8_ref among them"""
    x = R.log_uniform(n, rng, lo=-40, hi=20)
    e = R.edge_values()
    e = e[rng.permutation(e.size)][:n]
    x[rng.choice(n, e.size, replace=False)] = e
    return x


def _check_counted(eng, call, ref_fn, what):
    """call(hi, lo, sat) twice: the plane counters and sat grow by the reference's counts each time"""
    lib, h, N, ctr = eng
    sat = torch.zeros(1, dtype=torch.int64, device="cuda")
    ctr.zero_()
    for k in (1, 2):
        call(sat)
        torch.cuda.synchronize()
        x = ref_fn()
        ufl, groups = ufl_counts(x)
        got = ctr.cpu().tolist()
        assert got == [k * ufl, k * groups], (what, k, got, ufl, groups)
        assert int(sat.item()) == k * R.sat_count(x), what
    print("%s: ufl %d of %d groups" % (what, ufl, groups))
    return ufl, groups


@pytest.mark.parametrize("shape", [(7, 24), (129, 360), (2200, 1000)], ids=lambda s: "%dx%d" % s)
def test_split_planes_underflow(eng, shape):
    lib, h, N, _ = eng
    rows, Cn = shape
    cpad = (Cn + 127) // 128 * 128
    x = _wide(rows * Cn, np.random.default_rng(rows + Cn)).reshape(rows, Cn)
    xd = torch.from_numpy(x).cuda()
    xp = np.zeros((rows, cpad), np.float32); xp[:, :Cn] = x
    hi, lo = _planes(rows * cpad)
    ufl, _ = _check_counted(eng, lambda sat: N.check(h, lib.cgvc_split_planes(h, F16F8, _p(xd), rows, Cn, _p(hi), _p(lo), _p(sat), None)),
                            lambda: xp, "split %dx%d" % shape)
    assert ufl > 0


@pytest.mark.parametrize("d", [1, -1])
def test_im2col_planes_underflow(eng, d):
    lib, h, N, _ = eng
    T, samples, kw, Cn = 32, 5, 15, 24
    M = T * samples
    x = _wide(M * Cn, np.random.default_rng(3 + d)).reshape(M, Cn)
    xd = torch.from_numpy(x).cuda()
    pl, cpad = (kw - 1) // 2, 384
    ref = np.zeros((M, cpad), np.float32)
    for m in range(M):
        w = m % T
        for t in range(kw):
            ws = w + d * (t - pl)
            if 0 <= ws < T:
                ref[m, t * Cn:(t + 1) * Cn] = x[m - w + ws]
    hi, lo = _planes(M * cpad)
    _check_counted(eng, lambda sat: N.check(h, lib.cgvc_im2col_planes(h, F16F8, _p(xd), M, T, Cn, kw, d, _p(hi), _p(lo), _p(sat), None)),
                   lambda: ref, "im2col dir %+d" % d)


# (B, R, C, shuffle, gate, post_stream, post_onepass): streaming, stats + apply / one-pass, sums + apply, residual
POST_CASES = [(6, 64, 128, 1, 1, 1, 1), (6, 32, 96, 1, 1, 0, 1), (6, 516, 96, 1, 1, 1, 1), (6, 64, 128, 2, 0, 1, 1), (6, 48, 96, 1, 0, 1, 0)]


@pytest.mark.parametrize("case", POST_CASES, ids=["B%d_R%d_C%d_s%d_g%d_st%d_op%d" % c for c in POST_CASES])
def test_in_glu_planes_underflow(eng, case):
    """forward: y's planes, beta_a per channel from the edge table with a small gamma_a; backward: dP's planes, dy scaled by 2^k per
    sample, k from -40 to +20, then with a NaN and an inf in it"""
    lib, h, N, _ = eng
    B, R_, Cn, sh, gate, stream, onepass = case
    Cc = Cn * sh
    ldp = (2 if gate else 1) * Cc
    rng = np.random.default_rng(list(case))
    p = (rng.standard_normal((B, R_ // sh, ldp)) * 1.7 + 0.3).astype(np.float32)
    edge = R.edge_values(); edge = edge[np.isfinite(edge)]
    beta_a = np.resize(edge[rng.permutation(edge.size)], Cn).astype(np.float32)
    gamma_a = np.exp2(-rng.integers(4, 30, Cn)).astype(np.float32)
    beta_g = (rng.standard_normal(Cn) * 0.3).astype(np.float32); gamma_g = (rng.standard_normal(Cn) * 0.3 + 1.0).astype(np.float32)
    resid = None if gate else rng.standard_normal((B, R_, Cn)).astype(np.float32)
    ks = np.linspace(-40, 20, B).round().astype(int)
    dy = (rng.standard_normal((B, R_, Cn)) * np.exp2(ks)[:, None, None]).astype(np.float32)
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pd, rd = dev(p), dev(resid)
    pars = [dev(t) for t in (beta_a, gamma_a, beta_g, gamma_g)]
    y = torch.empty(B, R_, Cn, device="cuda"); stats = torch.empty(B, 4, Cn, device="cuda"); dp = torch.empty_like(pd)
    grads = [torch.zeros(Cn, device="cuda") for _ in range(4)]
    hi, lo = _planes(max(B * R_ * Cn, pd.numel()))
    assert lib.cgvc_set_option(h, b"post_stream", stream) == 0 and lib.cgvc_set_option(h, b"post_onepass", onepass) == 0
    try:
        _check_counted(eng, lambda sat: N.check(h, lib.cgvc_in_glu_forward_planes(
            h, _p(pd), _p(pars[0]), _p(pars[1]), _p(pars[2]), _p(pars[3]), _p(y), _p(stats), B, R_, Cn, sh, F16F8, gate, _p(rd), _p(hi),
            _p(lo), _p(sat), None)), lambda: y.cpu().numpy(), "forward %s" % (case,))
        bad = dy.copy(); bad[1, R_ // 3, 5] = np.nan; bad[2, 0, Cn - 1] = np.inf
        for name, d in (("backward", dy), ("backward NaN / inf", bad)):
            dyd = dev(d)
            ufl, _ = _check_counted(eng, lambda sat: N.check(h, lib.cgvc_in_glu_backward_planes(
                h, _p(dyd), _p(pd), _p(stats), _p(pars[0]), _p(pars[1]), _p(pars[2]), _p(pars[3]), _p(dp), _p(grads[0]), _p(grads[1]),
                _p(grads[2]), _p(grads[3]), B, R_, Cn, sh, F16F8, gate, _p(hi), _p(lo), _p(sat), None)), lambda: dp.cpu().numpy(),
                "%s %s" % (name, case))
            assert ufl > 0                                 # dy * 2^-40 lies below the edge
    finally:
        assert lib.cgvc_set_option(h, b"post_stream", 1) == 0 and lib.cgvc_set_option(h, b"post_onepass", 1) == 0


@pytest.mark.parametrize("B,R_", [(2, 128), (3, 48)])
def test_glu_planes_underflow(eng, B, R_):
    """the GLU-only form (generator h1): y's planes forward, dP's planes backward"""
    lib, h, N, _ = eng
    Cn = 128
    rng = np.random.default_rng(B * R_)
    P = np.concatenate([_wide(B * R_ * Cn, rng).reshape(B, R_, Cn), rng.standard_normal((B, R_, Cn)).astype(np.float32) * 3],
                       axis=2).astype(np.float32)
    P[np.isnan(P)] = 0.0
    Pd = torch.from_numpy(P).cuda()
    y = torch.empty(B, R_, Cn, device="cuda")
    hi, lo = _planes(B * R_ * 2 * Cn)
    _check_counted(eng, lambda sat: N.check(h, lib.cgvc_glu_forward_planes(h, _p(Pd), _p(y), B, R_, Cn, F16F8, _p(hi), _p(lo), _p(sat), None)),
                   lambda: y.cpu().numpy(), "glu forward B%d R%d" % (B, R_))
    dy = torch.from_numpy(_wide(B * R_ * Cn, rng).reshape(B, R_, Cn)).cuda()
    dp = torch.empty(B, R_, 2 * Cn, device="cuda")
    db = [torch.zeros(Cn, device="cuda") for _ in range(2)]
    _check_counted(eng, lambda sat: N.check(h, lib.cgvc_glu_backward_planes(h, _p(dy), _p(Pd), _p(dp), _p(db[0]), _p(db[1]), B, R_, Cn,
                                                                             F16F8, _p(hi), _p(lo), _p(sat), None)),
                   lambda: dp.cpu().numpy(), "glu backward B%d R%d" % (B, R_))


@pytest.mark.parametrize("fuse", [1, 0])
def test_disc_input_planes_underflow(eng, fuse):
    """the discriminator's input layer: y's planes from the one-pass kernel (fuse 1) and from the convolution + GLU kernels (fuse 0);
    the input spans 2^-40 .. 2^20"""
    lib, h, N, _ = eng
    B, T = 3, 48
    rng = np.random.default_rng(90 + fuse)
    x = R.log_uniform(B * 24 * T, rng, lo=-40, hi=20).reshape(B, 24, T)
    w = [(rng.standard_normal((G.KH, G.KW, 1, G.C1)) * 0.3).astype(np.float32) for _ in range(2)]
    b = [(rng.standard_normal(G.C1) * 1e-6).astype(np.float32) for _ in range(2)]
    x_d, wa, wg, ba, bg = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in (x, w[0], w[1], b[0], b[1]))
    Ho, Wo = G.out_rows(24, T)
    M = B * Ho * Wo
    p = torch.empty(M, 2 * G.C1, device="cuda"); y = torch.empty(M, G.C1, device="cuda")
    hi, lo = _planes(M * G.C1)
    fused = C.c_int(-1)
    _check_counted(eng, lambda sat: N.check(h, lib.cgvc_disc_input_forward(
        h, F16F8, _p(x_d), _p(wa), _p(wg), _p(ba), _p(bg), _p(p), _p(y), _p(hi), _p(lo), _p(sat), B, 24, T, G.KH, G.KW, G.C1, G.SH, G.SW,
        fuse, C.byref(fused), None)), lambda: y.cpu().numpy(), "disc input fuse %d" % fuse)
    assert fused.value == fuse


def test_counters_are_off_without_a_target(eng):
    lib, h, N, ctr = eng
    x = torch.full((4, 128), 1e-30, device="cuda")
    hi, lo = _planes(4 * 128)
    ctr.zero_()
    N.check(h, lib.cgvc_set_plane_counters(h, None))
    try:
        N.check(h, lib.cgvc_split_planes(h, F16F8, _p(x), 4, 128, _p(hi), _p(lo), None, None))
        torch.cuda.synchronize()
        assert ctr.cpu().tolist() == [0, 0]
    finally:
        N.check(h, lib.cgvc_set_plane_counters(h, _p(ctr)))


# ---- the train step -----------------------------------------------------------------------------------------------------------------
ARENAS = (0, 1, 2, 3)          # PARAM, GRAD, ADAM_M, ADAM_V


def _model(batch, mode, P, nets, **opts):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision="f16f8", log_dir='/tmp/cgvc_log',
                      loss_scale=mode, loss_scale_per_network=nets)
    for k, v in opts.items():
        m.set_option(k, v)
    m.set_params({k: v.numpy() for k, v in P.items()})
    return m


def _snap(m):
    torch.cuda.synchronize(m.device)
    return [m._arenas[a].clone() for a in ARENAS]


def _step_count(m):
    t = C.c_longlong(0)
    m._chk(m._lib.cgvc_get_adam_step(m._handle, C.byref(t)))
    return t.value


def _set_scales(m, s_G, s_D, good=(0, 0)):
    m._chk(m._lib.cgvc_set_loss_scale_state(m._handle, float(s_G), good[0], 0, m._stream()))
    if m.loss_scale_per_network:
        m._chk(m._lib.cgvc_set_loss_scale_net_state(m._handle, 0, float(s_G), good[0], m._stream()))
        m._chk(m._lib.cgvc_set_loss_scale_net_state(m._handle, 1, float(s_D), good[1], m._stream()))


def _launches():
    import cgvc  # noqa: F401
    from cgvc import native as N
    n = C.c_ulonglong(0)
    N.load().cgvc_kernel_launches(C.byref(n))
    return n.value


def test_equal_scales_give_the_single_scale_step(oracle_params64):
    """Deterministic mode, batch 2, lambdas 10 / 5, dynamic mode: with s_G = s_D = 1024 (the static scale of batch 2) the per-network
    step gives the single-scale step's PARAM, GRAD, ADAM_M, ADAM_V and losses bit for bit, and the networks' saturation counts sum to
    its sat_grad.  s_D = s_G 2^+-4: the generator range is unchanged bit for bit.  At 2^+4 the discriminators' update moves from the
    equal-scale one by no more than two non-deterministic single-scale runs differ (2 x that spread + 1e-3, the bound of
    test_monitor_and_dynamic_follow_static).  At 2^-4 (s_D = 2^6) it moved 1.24e-3 on an H100 (DESIGN.md section 10): the
    discriminators' planes cross the fp16 lower edge there, which their underflow fraction shows -- asserted to rise tenfold."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=41, batch=2, frames=128, dtype=torch.float32)
    out, gend = {}, None
    for key, nets, s_D in (("single", False, 1024.0), ("nets", True, 1024.0), ("up", True, 2.0 ** 14), ("down", True, 2.0 ** 6)):
        m = _model(2, "dynamic", oracle_params64, nets, deterministic=1)
        _set_scales(m, 1024.0, s_D)
        init = _snap(m)
        l0 = _launches()
        losses = m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        st = m.loss_scale_state()
        out[key] = (init, _snap(m), losses, st, _launches() - l0)
        gend = m._generator_end
        print("[%s] %s, %d launches" % (key, st, out[key][4]))
        assert not st["last_skipped"]
        del m
        torch.cuda.empty_cache()
    runs = []
    for _ in range(2):
        m = _model(2, "dynamic", oracle_params64, False)
        _set_scales(m, 1024.0, 1024.0)
        init = _snap(m)
        m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        runs.append((_snap(m)[0] - init[0]).double())
        del m
        torch.cuda.empty_cache()
    spread = float((runs[1][gend:] - runs[0][gend:]).norm() / runs[0][gend:].norm())
    single, nets = out["single"], out["nets"]
    for i, (a, b) in enumerate(zip(single[1], nets[1])):
        assert torch.equal(a, b), ARENAS[i]
    assert single[2] == nets[2]
    assert nets[3]["sat_grad_G"] + nets[3]["sat_grad_D"] == single[3]["sat_grad"] == nets[3]["sat_grad"]
    assert nets[3]["groups_G"] > 0 and nets[3]["groups_D"] > 0
    assert nets[4] == single[4]                         # the per-network scaler replaces the single one
    for key in ("up", "down"):
        init, after, _, st, _ = out[key]
        g_same = torch.equal(after[0][:gend], single[1][0][:gend])
        upd = [(b - a).double() for a, b in zip(init, after)]
        ref = [(b - a).double() for a, b in zip(single[0], single[1])]
        e = float((upd[0][gend:] - ref[0][gend:]).norm() / ref[0][gend:].norm())
        print("s_D = s_G 2^%+d: generator PARAM identical %s, discriminator update vs equal scales: relative L2 %.3e (single scale vs "
              "single scale, non-deterministic: %.3e)" % (4 if key == "up" else -4, g_same, e, spread))
        assert g_same
        if key == "up":
            assert e <= 2 * spread + 1e-3, (key, e, spread)
    frac = lambda key: out[key][3]["ufl_grad_D"] / out[key][3]["groups_D"]
    print("discriminator underflow fraction at s_D 2^6 / 2^10 / 2^14: %.3e / %.3e / %.3e" % (frac("down"), frac("nets"), frac("up")))
    assert frac("down") > 10 * frac("nets") > 10 * frac("up")


def test_attribution_in_monitor_mode(oracle_params64):
    """batch 1, lambda_cycle = 1e4 at the static scale 512: the generators' planes saturate, the discriminators' do not"""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=60, batch=1, frames=128, dtype=torch.float64)
    m = _model(1, "monitor", oracle_params64, True)
    m.train(A.numpy(), B.numpy(), 1e4, 5.0, 2e-4, 1e-4)
    st = m.last_loss_scale
    print("monitor, lambda_cycle 1e4: %s" % st)
    assert st["sat_grad_G"] > 0 and st["sat_grad_D"] == 0 and st["sat_grad"] == st["sat_grad_G"]
    assert st["scale"] == st["scale_G"] == st["scale_D"] == 512.0 and not m.last_step_skipped


def _grad_errors(m, ref):
    from cgvc import native as N
    errs = {}
    for k, g_ref in ref.items():
        n = float(g_ref.norm())
        if n < 1e-9:                                   # conv biases feeding an instance norm: analytically zero
            continue
        g = m._view(N.ARENA_GRAD, k).double()
        e = float((g - g_ref).norm()) / n
        errs[k] = e if np.isfinite(e) else float("inf")
    return errs


def test_the_corner_settles_with_two_scales(oracle_params64):
    """Dynamic mode, batch 1, lambda_cycle = 1e4: the first steps are skipped, s_G halves each time and s_D stays at 512.  At the
    settled scales (deterministic mode, compute_gradients) the discriminator gradients are those of the static scale and the generator
    gradients those of single-scale mode at s_G, bit for bit; every tensor's error against float64 is printed, the worst reported."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=60, batch=1, frames=128, dtype=torch.float64)
    m = _model(1, "dynamic", oracle_params64, True, deterministic=1)
    seen = []
    for _ in range(12):
        m.train(A.numpy(), B.numpy(), 1e4, 5.0, 2e-4, 1e-4)
        st = m.last_loss_scale
        seen.append((st["scale_G"], st["scale_D"], st["sat_grad_G"], st["sat_grad_D"], st["last_skipped"]))
        if not st["last_skipped"]:
            break
    print("per-network dynamic, lambda_cycle 1e4: (s_G, s_D, sat G, sat D, skipped) per step: %s" % seen)
    assert seen[0][4] and not seen[-1][4]
    assert [s[0] for s in seen[:-1]] == [512.0 / 2 ** (i + 1) for i in range(len(seen) - 1)]
    assert all(s[1] == 512.0 and s[3] == 0 for s in seen)
    s_G = seen[-1][0]
    ufl = m.last_loss_scale
    print("settled: s_G %g, s_D %g; underflow fraction G %.3e, D %.3e" % (s_G, ufl["scale_D"], ufl["ufl_grad_G"] / ufl["groups_G"],
                                                                         ufl["ufl_grad_D"] / ufl["groups_D"]))
    _, Gref, _, _ = O.gradients(A, B, oracle_params64, 1e4, 5.0)
    ref = {k: v.to("cuda") for k, v in Gref.items()}
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    m.compute_gradients(A.numpy(), B.numpy(), 1e4, 5.0)
    torch.cuda.synchronize()
    g_nets = m._arenas[1].clone()
    e_nets = _grad_errors(m, ref)
    gend = m._generator_end
    del m
    s = _model(1, "dynamic", oracle_params64, False, deterministic=1)
    res = {}
    for scale in (512.0, s_G):
        _set_scales(s, scale, scale)
        s.compute_gradients(A.numpy(), B.numpy(), 1e4, 5.0)
        torch.cuda.synchronize()
        res[scale] = (s._arenas[1].clone(), _grad_errors(s, ref))
    assert torch.equal(g_nets[gend:], res[512.0][0][gend:])          # the discriminators: their gradients at the static scale
    assert torch.equal(g_nets[:gend], res[s_G][0][:gend])            # the generators: single-scale mode at s_G
    worst = max(e_nets.items(), key=lambda kv: kv[1])
    worst_D = max(((k, v) for k, v in e_nets.items() if k.startswith("discriminator")), key=lambda kv: kv[1])
    worst_single = max(res[s_G][1].items(), key=lambda kv: kv[1])
    print("settled at s_G %g, s_D 512: worst of %d gradient tensors vs float64 %.3e (%s); worst discriminator tensor %.3e (%s); "
          "single scale %g: worst %.3e (%s)" % (s_G, len(ref), worst[1], worst[0], worst_D[1], worst_D[0], s_G, worst_single[1],
                                               worst_single[0]))
    assert worst_D[1] < 1e-3


@pytest.mark.parametrize("graph", [1, 0])
def test_halving_per_network_and_skipped_steps(oracle_params64, graph):
    """A non-finite lambda_cycle makes only the generator range non-finite (the D-loss pass does not read it): s_G halves, s_D
    stays.  s_D = 2^24 saturates only the discriminators' planes: s_D halves, s_G keeps counting good steps and, with growth interval
    2, doubles although both steps were skipped.  Every skipped step leaves PARAM, ADAM_M, ADAM_V and t bit-unchanged."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=70, batch=1, frames=128, dtype=torch.float32)
    m = _model(1, "dynamic", oracle_params64, True, cuda_graph=graph, loss_scale_growth_interval=2)
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    st = m.last_loss_scale
    assert not st["last_skipped"] and (st["scale_G"], st["scale_D"], st["good_steps_G"], st["good_steps_D"]) == (512.0, 512.0, 1, 1)
    before, t0 = _snap(m), _step_count(m)
    m.train(A.numpy(), B.numpy(), float("nan"), 5.0, 2e-4, 1e-4)
    st = m.loss_scale_state()
    print("[graph %d] NaN lambda_cycle: %s" % (graph, st))
    assert st["last_skipped"] and st["nonfinite"] == 1
    assert (st["scale_G"], st["scale_D"], st["good_steps_G"], st["good_steps_D"]) == (256.0, 1024.0, 0, 0)   # D: its second good step
    after = _snap(m)
    for i in (0, 2, 3):
        assert torch.equal(before[i], after[i]), ARENAS[i]
    assert _step_count(m) == t0
    _set_scales(m, 512.0, 2.0 ** 24)
    seen = []
    for _ in range(2):
        m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        st = m.last_loss_scale
        seen.append((st["scale_G"], st["scale_D"], st["good_steps_G"], st["sat_grad_G"], st["sat_grad_D"], st["last_skipped"]))
    print("[graph %d] s_D = 2^24: (s_G, s_D, good G, sat G, sat D, skipped) %s" % (graph, seen))
    assert seen[0][5] and seen[0][4] > 0 and seen[0][3] == 0 and seen[0][:3] == (512.0, 2.0 ** 23, 1)
    assert seen[1][0] == 1024.0 and seen[1][2] == 0 and seen[1][1] <= 2.0 ** 23
    assert st["scale"] == st["scale_G"]


def test_deterministic_twice(oracle_params64):
    """two fresh deterministic engines, three per-network dynamic steps each (the second with s_D = 2^24, skipped): the same bits"""
    from oracle import cyclegan_oracle as O
    batches = [O.synthetic_batch(seed=80 + s, batch=2, frames=128, dtype=torch.float32) for s in range(3)]
    runs = []
    for _ in range(2):
        m = _model(2, "dynamic", oracle_params64, True, deterministic=1)
        states = []
        for i, (A, B) in enumerate(batches):
            if i == 1:
                _set_scales(m, 1024.0, 2.0 ** 24)
            losses = m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
            states.append((losses, m.loss_scale_state()))
        runs.append((_snap(m), states))
        del m
        torch.cuda.empty_cache()
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a, b)
    assert runs[0][1] == runs[1][1]
    assert runs[0][1][1][1]["last_skipped"]


def test_save_load_both_scales(oracle_params64, tmp_path):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=71, batch=1, frames=128, dtype=torch.float32)
    m = _model(1, "dynamic", oracle_params64, True, loss_scale_growth_interval=5)
    _set_scales(m, 64.0, 2048.0, good=(2, 3))
    m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
    st = m.loss_scale_state()
    assert (st["scale_G"], st["good_steps_G"], st["scale_D"], st["good_steps_D"]) == (64.0, 3, 2048.0, 4)
    path = m.save(str(tmp_path), "nets.ckpt")
    m2 = _model(1, "dynamic", oracle_params64, True)
    m2.load(path)
    st2 = m2.loss_scale_state()
    assert (st2["scale_G"], st2["good_steps_G"], st2["scale_D"], st2["good_steps_D"], st2["scale"]) == (64.0, 3, 2048.0, 4, 64.0)
    # a single-scale checkpoint loads into both networks
    s = _model(1, "dynamic", oracle_params64, False)
    _set_scales(s, 128.0, 128.0, good=(1, 1))
    p1 = s.save(str(tmp_path), "single.ckpt")
    m3 = _model(1, "dynamic", oracle_params64, True)
    m3.load(p1)
    st3 = m3.loss_scale_state()
    assert (st3["scale_G"], st3["good_steps_G"], st3["scale_D"], st3["good_steps_D"]) == (128.0, 1, 128.0, 1)


@pytest.mark.parametrize("pipelined", [1, 0])
def test_single_rank_communicator(oracle_params64, pipelined):
    """a one-rank NCCL communicator (its all-reduce is an identity): the per-network step with the counter all-reduce gives the plain
    per-network step's scales and counts, and takes the same per-network decision on a saturating s_D"""
    import torch.distributed as dist
    import cgvc
    from oracle import cyclegan_oracle as O
    if not dist.is_initialized():
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29578", rank=0, world_size=1)
    A, B = O.synthetic_batch(seed=72, batch=2, frames=128, dtype=torch.float32)
    seen = []
    for dp in (False, True):
        m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision="f16f8", seed=17, data_parallel=dp,
                          log_dir='/tmp/cgvc_log', loss_scale="dynamic", loss_scale_per_network=True)
        m.set_option("pipelined_comm", pipelined)
        m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        st0 = m.loss_scale_state()
        _set_scales(m, 1024.0, 2.0 ** 24)
        before = _snap(m)
        m.train(A.numpy(), B.numpy(), 10.0, 5.0, 2e-4, 1e-4)
        st1 = m.loss_scale_state()
        after = _snap(m)
        assert all(torch.equal(before[i], after[i]) for i in (0, 2, 3))
        key = lambda st: (st["scale_G"], st["scale_D"], st["last_skipped"], st["sat_grad_G"] == 0, st["sat_grad_D"] > 0, st["groups_G"],
                          st["groups_D"])
        seen.append((key(st0), key(st1)))
        print("[pipelined %d, communicator %s] %s | %s" % (pipelined, dp, st0, st1))
        del m
        torch.cuda.empty_cache()
    assert seen[0] == seen[1]
    assert seen[1][1][:3] == (1024.0, 2.0 ** 23, True)
