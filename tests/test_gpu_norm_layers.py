"""The separate instance-norm (+ GLU | + residual, + pixel-shuffle view) kernels of csrc/simt_kernels.cu (launch_post_fwd /
launch_post_bwd) against float64, element by element, in every form the engine dispatches: the streaming forward and backward, the
one-pass backward, stats + apply (also packed), sums + apply and the deterministic form with reduce_parts.  They run every instance
norm the GEMM epilogue does not fuse: every default backward, the discriminator's whole forward and the conversions.

Lattice tier (bitwise; tests/fused_ref.py has the argument for each form):
  forward   P in {-1, 0, 1}, gate branch 0 and beta_g = 0 (the fast sigmoid of 0 is exactly 1/2), gamma powers of two, integer beta,
            R a power of two: every sum and 1 / R product is exact, sqrtf and the division are IEEE, so mean and rstd equal a float32
            replay of the exact variance, and in zero-mean columns y = fl(fma(x, fl(rstd gamma), beta)) / 2 (+ resid: one more
            rounding).  Sample 0 is all zero (rstd = fl(1 / sqrt(eps))), sample 1 has one nonzero value (eps dominates).
  backward  statistics given with integer means and power-of-two rstd, the gate branch equal to its mean: dP, the affine and the
            conv-bias gradients are dyadic and every sum is exact while the certificate holds (sum of |terms| under 2^24 units).
  zero-sum  R = 48, 96, 384, 33, 516: dy cancels in pairs of positions with equal x, so sum dna = sum dna xhat = 0, c2 = c3 = 0
            whatever 1 / R rounds to, and dP = fl(gamma rstd) dna exactly.
Dense tier (randn, variances from 1e-9 to 1e4 around eps, |mean| / std up to 1e3, samples whose position 0 is a far outlier): the
  statistics within fused_ref.stats_bound of their form, y within y_bound at the kernel's own statistics, dP within norm_bwd_bound, and
  the affine and conv-bias gradients within gamma_L of their |terms| plus the propagated error.
Every case asserts the kernels that ran (torch.profiler) against fused_ref's dispatch mirror, and test_every_instantiation_is_reached
checks that the case tables reach every instantiation in simt_kernels.cu.
"""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest
import torch

import fused_ref as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = F.U
EPS32 = np.float32(1e-6)
FP32 = 0
# the worst measured fraction of each bound is printed by the dense cases (and recorded in DESIGN.md section 10)
WORST = {}
SEEN = set()             # the instance-norm kernels torch.profiler saw over the module

# (name, B, R, C, sh, gated, resid): the step's own shapes, then conversion lengths, cvalid tails, B = 1 and the B limit
STEP = [("D.d1", 512, 384, 256, 1, True, False), ("D.d2", 512, 96, 512, 1, True, False), ("D.d3", 512, 48, 1024, 1, True, False),
        ("G.d1", 256, 64, 256, 1, True, False), ("G.d2", 256, 32, 512, 1, True, False), ("G.res_h1", 256, 32, 1024, 1, True, False),
        ("G.res_h2", 256, 32, 512, 1, False, True), ("G.u1", 256, 64, 512, 2, True, False), ("G.u2", 256, 128, 256, 2, True, False)]
OTHER = [("conv129", 3, 129, 256, 1, True, False), ("conv258", 2, 258, 256, 2, True, False), ("conv350", 2, 350, 512, 1, True, False),
         ("conv700", 2, 700, 256, 2, True, False), ("conv700h2", 2, 700, 512, 1, False, True),
         ("c96", 3, 40, 96, 1, True, False), ("c160", 2, 20, 160, 2, True, False), ("c96h2", 3, 56, 96, 1, False, True),
         ("b1", 1, 64, 128, 1, True, False), ("h2r64", 4, 64, 256, 1, False, True), ("h2r20", 4, 20, 128, 1, False, True),
         ("h2r40", 4, 40, 128, 1, False, True), ("r40", 4, 40, 128, 1, True, False), ("r56", 3, 56, 128, 2, True, False),
         ("r33", 4, 33, 64, 1, True, False), ("bmax", 65535, 4, 32, 1, True, False)]
DENSE = STEP + OTHER
# (forms): options for each run; "det" adds deterministic mode
FORMS = {"default": dict(post_onepass=1, post_stream=1, deterministic=0), "nostream": dict(post_onepass=1, post_stream=0, deterministic=0),
         "noonepass": dict(post_onepass=0, post_stream=1, deterministic=0), "det": dict(post_onepass=1, post_stream=1, deterministic=1)}
# packed: utterance lengths in frames (multiples of 4), at P's level divisors 1, 2 and 4 (shuffle 2 at 2 and 4, as u1 / u2)
UTTS = [4, 8, 12, 132, 516, 1400, 4, 12]
PACKED = [(div, sh, gated) for div, sh in ((1, 1), (2, 1), (2, 2), (4, 1), (4, 2)) for gated in (True, False) if gated or sh == 1]


def _seed(*key):
    return zlib.crc32(repr(key).encode())


@pytest.fixture(scope="module")
def eng():
    import cgvc  # noqa: F401
    from cgvc import native as N
    lib = N.load()
    cfg = N.Config(24, 1, 128, N.PREC_FP32_SIMT, 0, 0)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == 0, lib.cgvc_last_error(None)
    assert lib.cgvc_set_option(h, b"deterministic", 1) == 0
    nb = C.c_size_t(0)
    assert lib.cgvc_arena_bytes(h, N.ARENA_WORK, C.byref(nb)) == 0
    work = torch.empty((nb.value + 3) // 4, dtype=torch.float32, device="cuda")
    assert lib.cgvc_bind_arena(h, N.ARENA_WORK, C.c_void_p(work.data_ptr()), nb.value) == 0
    assert lib.cgvc_set_option(h, b"deterministic", 0) == 0
    yield lib, h, N
    lib.cgvc_destroy(h)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _launches(lib):
    n = C.c_ulonglong(0)
    assert lib.cgvc_kernel_launches(C.byref(n)) == 0
    return n.value


def _run(eng, form, fn, expect):
    """fn() under the options of `form`, asserting that it launched the kernels `expect` (fused_ref's dispatch mirror): their names
    with template arguments from torch.profiler, and their number from cgvc_kernel_launches.  Returns the names."""
    lib, h, N = eng
    for k, v in FORMS[form].items():
        assert lib.cgvc_set_option(h, k.encode(), v) == 0
    try:
        torch.cuda.synchronize()
        n0 = _launches(lib)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        n1 = _launches(lib)
    finally:
        for k, v in FORMS["default"].items():
            lib.cgvc_set_option(h, k.encode(), v)
    names = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m = re.search(r"(post_\w+|reduce_parts_kernel)(<[^>(]*>)?", _demangle(e.name))
        if m:
            names.append(m.group(1) + (m.group(2) or ""))
    assert n1 - n0 == len(expect), (form, n1 - n0, expect)
    # the profiler may drop kernel records of a short session, so a case checks that what it saw is an ordered part of the
    # expected launches (and the launch count above); test_zz_profiler_saw_every_instantiation checks that every kernel was seen
    it = iter(expect)
    assert all(n in it for n in names), (form, names, expect)
    SEEN.update(names)
    return expect


def _demangle(name):
    if not name.startswith("_Z"):
        return name
    import subprocess
    return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip() or name


def _fwd(eng, P, par, B, R, C_, sh, gated, resid=None, packed=None):
    """cgvc_in_glu_forward_planes (cgvc_in_glu_forward_packed) in fp32; packed = (offsets [n + 1] frames, div, max_len): B = 1, R = all view rows"""
    lib, h, N = eng
    nst = len(packed[0]) - 1 if packed else B
    y = _nan(B * R * C_); st = _nan(nst, 4, C_)
    off = _dev(np.asarray(packed[0], np.int64)) if packed else None
    n, div, mx = (nst, packed[1], packed[2]) if packed else (0, 0, 0)
    if packed:
        assert B == 1
        return y, st, lambda: N.check(h, lib.cgvc_in_glu_forward_packed(h, _p(P), *(_p(t) for t in par), _p(y), _p(st), R, C_, sh, FP32,
                                                                          int(gated), _p(resid), _p(off), n, div, mx, None, None, None, None))
    return y, st, lambda: N.check(h, lib.cgvc_in_glu_forward_planes(h, _p(P), *(_p(t) for t in par), _p(y), _p(st), B, R, C_, sh, FP32,
                                                                      int(gated), _p(resid), None, None, None, None))


def _bwd(eng, dy, P, st, par, B, R, C_, sh, gated, g0=None, affine=True, bias=True):
    """cgvc_in_glu_backward_bias; g0: initial gradients (dbeta_a, dgamma_a, dbeta_g, dgamma_g, dbias_a, dbias_g) to accumulate into"""
    lib, h, N = eng
    dp = _nan(*P.shape)
    Cc = C_ * sh
    g = [torch.zeros(C_, device="cuda") for _ in range(4)] + [torch.zeros(Cc, device="cuda") for _ in range(2)]
    if g0 is not None:
        for t, v in zip(g, g0):
            t.copy_(torch.as_tensor(v))
    gp = [t if (affine if i < 4 else bias) else None for i, t in enumerate(g)]
    call = lambda: N.check(h, lib.cgvc_in_glu_backward_bias(h, _p(dy), _p(P), _p(st), *(_p(t) for t in par), _p(dp), *(_p(t) for t in gp),
                                                             B, R, C_, sh, FP32, int(gated), None, None, None, None))
    return dp, g, call


def _where(shape_names, flat, shape):
    idx = np.unravel_index(flat, shape)
    return ", ".join("%s %d" % (n, int(i)) for n, i in zip(shape_names, idx))


def _report(bad, got, ref, names, what):
    bad = np.asarray(bad)
    idx = np.flatnonzero(bad.reshape(-1))
    if idx.size:
        g = np.asarray(got, np.float64).reshape(-1); r = np.asarray(ref, np.float64).reshape(-1)
        lines = ["  %s: got %r, reference %r" % (_where(names, int(i), bad.shape), g[i], r[i]) for i in idx[:8]]
        raise AssertionError("%s: %d of %d values wrong; first:\n%s" % (what, idx.size, bad.size, "\n".join(lines)))


def _np(t):
    return t.double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


def _t64(t):
    return (t if isinstance(t, torch.Tensor) else torch.from_numpy(np.asarray(t, np.float64))).double().cuda()


def _assert_equal(got, ref, names, what):
    got, ref = _np(got), _np(ref)
    _report(~((got == ref) | (np.isnan(got) & np.isnan(ref))), got, ref, names, what)


def _assert_within(got, ref, bound, names, what, key):
    """|got - ref| <= bound per element (on the device; moved to the host only to name the failures); returns the worst fraction"""
    got, ref, bound = _t64(got), _t64(ref), _t64(bound)
    got, ref, bound = torch.broadcast_tensors(got, ref, bound)
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        _report(bad.cpu().numpy(), _np(got), _np(ref), names, what)
    frac = float((err / bound).max()) if err.numel() else 0.0
    WORST[key] = max(WORST.get(key, 0.0), frac)
    return frac


# ---- lattice: forward --------------------------------------------------------------------------------------------------------------
def _lattice_fwd_case(B, R, C_, sh, gated, seed):
    """P [B * R / sh, ldp] in {-1, 0, 1} with the even channels zero-mean per sample, gate branch 0; sample 0 zero, sample 1 one value"""
    rng = np.random.default_rng(seed)
    v = np.zeros((B, R, C_), np.float32)          # the normalised view of the a branch
    for b in range(2, B):
        v[b] = rng.integers(-1, 2, (R, C_))
        for c in range(0, C_, 2):                 # zero-mean: the second half of the positions negates a permutation of the first
            perm = rng.permutation(R)
            half = R // 2
            v[b, perm[half:2 * half], c] = -v[b, perm[:half], c]
            if R % 2:
                v[b, perm[-1], c] = 0
    if B > 1:
        v[1, rng.integers(R), rng.integers(1, C_, 1)[0] | 1] = rng.choice([-1.0, 1.0])
    a = torch.from_numpy(v)
    if sh == 2:
        a = F.unshuffle_rows(a)
    Cc = C_ * sh
    P = torch.cat([a, torch.zeros_like(a)], dim=-1) if gated else a
    beta_a = rng.integers(-2, 3, C_).astype(np.float32)
    gamma_a = (rng.choice([-1.0, 1.0], C_) * np.exp2(rng.integers(-1, 2, C_))).astype(np.float32)
    gamma_g = np.exp2(rng.integers(-1, 2, C_)).astype(np.float32)
    par = (beta_a, gamma_a, np.zeros(C_, np.float32), gamma_g) if gated else (beta_a, gamma_a, None, None)
    resid = None if gated else rng.integers(-4, 5, (B, R, C_)).astype(np.float32)
    assert P.shape == (B, R // sh, Cc * (2 if gated else 1))
    return P.reshape(B * R // sh, -1).numpy(), v, par, resid


def _replay_stats(v):
    """mean (exact) and rstd = fl(1 / fl(sqrt(fl(var + eps)))) in float32 of the exact variance"""
    x = v.astype(np.float64)
    m = x.mean(axis=1)
    var = ((x - m[:, None]) ** 2).mean(axis=1)
    assert np.array_equal(var.astype(np.float32).astype(np.float64), var), "variance not exact in fp32: the lattice case is too large"
    rs = np.float32(1) / np.sqrt(var.astype(np.float32) + EPS32)
    return m, rs.astype(np.float32)


LATTICE_FWD = [(R, sh, gated, form) for R in (32, 64, 128) for sh in (1, 2) for gated in (True, False) for form in ("default", "nostream")
               if gated or sh == 1]


@pytest.mark.parametrize("R0,sh,gated,form", LATTICE_FWD)
def test_lattice_forward_is_bitwise(eng, R0, sh, gated, form):
    R = R0 * sh
    B, C_ = 5, 128
    P, v, par, resid = _lattice_fwd_case(B, R, C_, sh, gated, _seed("lf", R, sh, gated))
    Pd, pard, rd = _dev(P), tuple(_dev(t) for t in par), _dev(resid)
    y, st, call = _fwd(eng, Pd, pard, B, R, C_, sh, gated, rd)
    names = _run(eng, form, call, F.post_fwd_kernels(B, R, C_, sh, gated, resid is not None, form != "nostream"))
    what = "lattice forward R %d sh %d %s (%s)" % (R, sh, "gated" if gated else "residual", names)
    m, rs = _replay_stats(v)
    got = st.cpu().numpy()
    _assert_equal(got[:, 0], m, ("sample", "channel"), what + ": mean_a")
    _assert_equal(got[:, 1], rs, ("sample", "channel"), what + ": rstd_a")
    assert got[0, 1, 0] == np.float32(1) / np.sqrt(EPS32)
    if gated:
        _assert_equal(got[:, 2], 0 * m, ("sample", "channel"), what + ": mean_g")
        _assert_equal(got[:, 3], np.full_like(rs, np.float32(1) / np.sqrt(EPS32)), ("sample", "channel"), what + ": rstd_g")
    # y in the zero-mean columns (and all of samples 0 and 1's zero columns): fl(fma(x, fl(rstd gamma), beta)) / 2, or + resid
    sca = (rs * par[1][None, :]).astype(np.float64)
    na = (v.astype(np.float64) * sca[:, None, :] + par[0][None, None, :].astype(np.float64)).astype(np.float32)
    ref = na * np.float32(0.5) if gated else (na + resid).astype(np.float32)
    zero_mean = (m == 0)[:, None, :] & np.ones((1, R, 1), bool)
    yk = y.cpu().numpy().reshape(B, R, C_)
    _assert_equal(np.where(zero_mean, yk, 0), np.where(zero_mean, ref, 0), ("sample", "position", "channel"), what + ": y")
    # and everywhere within the dense bound at the kernel's statistics
    yr, _ = F.forward(torch.from_numpy(P).reshape(B, R // sh, -1), par, gated, sh, resid=resid, stats=torch.from_numpy(got).double())
    bound = F.y_bound(torch.from_numpy(P).reshape(B, R // sh, -1).double(), torch.from_numpy(got).double(), par, gated, sh, resid)
    _assert_within(yk, yr, bound, ("sample", "position", "channel"), what + ": y beyond its bound", "lattice y")


# ---- lattice: backward -------------------------------------------------------------------------------------------------------------
def _lsb_ok(terms_abs_sum, values):
    """sum |terms| in units of the finest nonzero value below 2^24"""
    v = np.abs(np.asarray(values, np.float64).reshape(-1))
    v = v[v > 0]
    if v.size == 0:
        return True
    m, e = np.frexp(v)
    mi = (m * 2.0 ** 53).astype(np.int64)
    tz = np.array([(int(x) & -int(x)).bit_length() - 1 for x in mi])
    unit = 2.0 ** (e - 53 + tz).min()
    return float(np.max(terms_abs_sum)) / unit < 2 ** 24


def _lattice_bwd_case(B, R, C_, sh, gated, seed, zero_sum):
    """P, stats [B, 4, C], par, dy [B, R, C]; zero_sum: dy cancels in pairs of positions with equal x"""
    rng = np.random.default_rng(seed)
    ma = rng.integers(-2, 3, (B, C_)).astype(np.float32)
    ra = np.exp2(rng.integers(0, 2, (B, C_))).astype(np.float32)
    mg = rng.integers(-2, 3, (B, C_)).astype(np.float32)
    rg = np.exp2(rng.integers(0, 2, (B, C_))).astype(np.float32)
    dv = rng.integers(-1, 2, (B, R, C_)).astype(np.float32)
    dy = rng.integers(-1, 2, (B, R, C_)).astype(np.float32)
    if zero_sum:
        for b in range(B):
            for c in range(C_):
                perm = rng.permutation(R)
                half = R // 2
                dv[b, perm[half:2 * half], c] = dv[b, perm[:half], c]
                dy[b, perm[half:2 * half], c] = -dy[b, perm[:half], c]
                if R % 2:
                    dy[b, perm[-1], c] = 0
    a = torch.from_numpy(ma[:, None, :] + dv)
    g = torch.from_numpy(np.broadcast_to(mg[:, None, :], (B, R, C_)).copy())
    if sh == 2:
        a, g = F.unshuffle_rows(a), F.unshuffle_rows(g)
    P = torch.cat([a, g], dim=-1) if gated else a
    stats = np.stack([ma, ra, mg, rg], axis=1).astype(np.float32)
    beta_a = rng.integers(-2, 3, C_).astype(np.float32)
    gamma_a = (rng.choice([-1.0, 1.0], C_) * np.exp2(rng.integers(-1, 1, C_))).astype(np.float32)
    gamma_g = (rng.choice([-1.0, 1.0], C_) * np.exp2(rng.integers(-1, 1, C_))).astype(np.float32)
    par = (beta_a, gamma_a, np.zeros(C_, np.float32), gamma_g) if gated else (beta_a, gamma_a, None, None)
    return P.reshape(B * R // sh, -1).numpy(), stats, par, dy


def _bwd_reference(P, stats, par, dy, B, R, C_, sh, gated):
    dP, grads, bias = F.backward(torch.from_numpy(P).reshape(B, R // sh, -1), par, dy, gated, stats=torch.from_numpy(stats), shuffle=sh,
                                 bias=True)
    return dP.reshape(B * R // sh, -1), list(grads) + list(bias)


GRAD_NAMES = ("dbeta_a", "dgamma_a", "dbeta_g", "dgamma_g", "dbias_a", "dbias_g")


def _check_bwd_exact(dp, g, g0, ref_dp, ref_g, gated, what):
    _assert_equal(dp.cpu().numpy(), ref_dp.numpy(), ("conv row", "column"), what + ": dP")
    for i, (t, r) in enumerate(zip(g, ref_g)):
        if r is None or (not gated and i in (2, 3, 5)):
            continue
        r = r.numpy() + (g0[i] if g0 is not None else 0)
        _assert_equal(t.cpu().numpy(), r, ("column",), what + ": " + GRAD_NAMES[i])


LATTICE_BWD = [(R, sh, gated, form, acc) for R in (32, 64, 128) for sh in (1, 2) for gated in (True, False)
               for form in ("default", "noonepass", "det") for acc in (0, 1) if gated or sh == 1]


@pytest.mark.parametrize("R0,sh,gated,form,acc", LATTICE_BWD)
def test_lattice_backward_is_bitwise(eng, R0, sh, gated, form, acc):
    R = R0 * sh
    B, C_ = 4, 128
    P, stats, par, dy = _lattice_bwd_case(B, R, C_, sh, gated, _seed("lb", R, sh, gated), False)
    ref_dp, ref_g = _bwd_reference(P, stats, par, dy, B, R, C_, sh, gated)
    absdp = np.abs(ref_dp.numpy()).reshape(B, R // sh, -1).sum(axis=(0, 1))
    assert _lsb_ok(absdp, ref_dp.numpy()), "lattice certificate fails: the case is too large"
    rng = np.random.default_rng(_seed("g0", R, sh))
    g0 = [rng.integers(-8, 9, n).astype(np.float32) for n in (C_, C_, C_, C_, C_ * sh, C_ * sh)] if acc else None
    dp, g, call = _bwd(eng, _dev(dy), _dev(P), _dev(stats), tuple(_dev(t) for t in par), B, R, C_, sh, gated, g0=g0)
    names = _run(eng, form, call, F.post_bwd_kernels(B, R, C_, sh, gated, form != "noonepass", True, form == "det", True, True))
    _check_bwd_exact(dp, g, g0, ref_dp, ref_g, gated, "lattice backward R %d sh %d %s acc %d (%s)" % (
        R, sh, "gated" if gated else "residual", acc, names))


ZERO_SUM = [(R, sh, gated, C_, form) for R, sh, gated, C_ in ((48, 1, True, 64), (96, 1, True, 32), (384, 1, True, 32), (384, 2, True, 64),
                                                                (33, 1, True, 64), (516, 1, True, 32), (516, 2, True, 32), (48, 1, False, 64),
                                                                (96, 2, True, 32))
            for form in ("default", "det")]


@pytest.mark.parametrize("R,sh,gated,C_,form", ZERO_SUM)
def test_zero_sum_lattice_backward_is_bitwise(eng, R, sh, gated, C_, form):
    """c2 = c3 = 0 whatever fl(1 / R) is: row, phase and channel placement of every streaming configuration, exactly"""
    B = 3
    P, stats, par, dy = _lattice_bwd_case(B, R, C_, sh, gated, _seed("zs", R, sh, gated), True)
    ref_dp, ref_g = _bwd_reference(P, stats, par, dy, B, R, C_, sh, gated)
    dp, g, call = _bwd(eng, _dev(dy), _dev(P), _dev(stats), tuple(_dev(t) for t in par), B, R, C_, sh, gated)
    names = _run(eng, form, call, F.post_bwd_kernels(B, R, C_, sh, gated, True, True, form == "det", True, True))
    _check_bwd_exact(dp, g, None, ref_dp, ref_g, gated, "zero-sum backward R %d sh %d C %d (%s)" % (R, sh, C_, names))


# ---- dense tier --------------------------------------------------------------------------------------------------------------------
def _dense_case(B, R, C_, sh, gated, seed, device="cuda"):
    """P with per-sample scales 10^-4.5 ... 10^2 (variance 1e-9 ... 1e4), column offsets up to 1e3 std, and every third sample's position
    0 a far outlier; affine parameters near (0, 1); dy randn"""
    g = torch.Generator(device=device).manual_seed(seed)
    Cc = C_ * sh
    nt = Cc * (2 if gated else 1)
    P = torch.randn(B, R // sh, nt, device=device, generator=g, dtype=torch.float64)
    scale = 10.0 ** (torch.linspace(-4.5, 2.0, B, device=device, dtype=torch.float64)[torch.randperm(B, device=device, generator=g)])
    off = torch.randn(B, 1, nt, device=device, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(0, 4, (B, 1, nt), device=device,
                                                                                                           generator=g)
    P = (P + off) * scale[:, None, None]
    out = torch.arange(B, device=device) % 3 == 2
    P[out, 0, :] += 60.0 * scale[out, None] * torch.sign(torch.randn(int(out.sum()), nt, device=device, generator=g, dtype=torch.float64))
    P = P.float()
    par = [(torch.randn(C_, device=device, generator=g) * 0.3 + k) for k in (0.0, 1.0, 0.0, 1.0)]
    if not gated:
        par[2] = par[3] = None
    resid = None if gated else torch.randn(B * R * C_, device=device, generator=g)
    dy = torch.randn(B * R * C_, device=device, generator=g)
    return P.reshape(B * R // sh, nt).contiguous(), par, resid, dy


def _check_stats_dense(st, P3, gated, sh, form, L, what):
    a, g = F.branches(P3.double(), gated, sh)
    for k, v in ((0, a), (2, g)):
        if v is None:
            continue
        m64, r64 = F.stats_of(v)
        em, er = F.stats_bound(v, form, L)
        _assert_within(st[:, k], m64, em, ("sample", "channel"), what + ": mean", "mean " + form)
        _assert_within(st[:, k + 1] / r64 - 1, 0 * r64, er, ("sample", "channel"), what + ": rstd (relative)", "rstd " + form)


@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
@pytest.mark.parametrize("form", ["default", "nostream", "noonepass", "det"])
def test_dense_forward_and_backward(eng, case, form):
    name, B, R, C_, sh, gated, resid_ = case
    if form != "default" and B > 512 or (form in ("noonepass", "det") and name.startswith("D.")):
        pytest.skip("the form is covered at the smaller shapes")
    P, par, resid, dy = _dense_case(B, R, C_, sh, gated, _seed("dense", name))
    P3 = P.reshape(B, R // sh, -1)
    what = "%s (%s)" % (name, form)
    # forward
    y, st, call = _fwd(eng, P, par, B, R, C_, sh, gated, resid)
    names = _run(eng, form, call, F.post_fwd_kernels(B, R, C_, sh, gated, resid is not None, form != "nostream"))
    fform = "stream" if names[0].startswith("post_fwd_stream") else "shifted"
    L1 = F.post_chain(1, R)
    _check_stats_dense(st, P3, gated, sh, fform, L1, what + " forward " + str(names))
    par64 = [None if t is None else t.double() for t in par]
    r3 = None if resid is None else resid.reshape(B, R, C_)
    yr, _ = F.forward(P3.double(), par64, gated, sh, resid=None if r3 is None else r3.double(), stats=st.double())
    bound = F.y_bound(P3.double(), st.double(), par64, gated, sh, None if r3 is None else r3.double())
    _assert_within(y.reshape(B, R, C_), yr, bound, ("sample", "position", "channel"), what + ": y", "y " + fform)
    # backward at the kernel's statistics; the affine and conv-bias gradients accumulate into nonzero values
    g0 = [torch.randn(n, device="cuda").cpu().numpy() for n in (C_, C_, C_, C_, C_ * sh, C_ * sh)]
    data_only = name.startswith("D.") and form == "default"
    dp, g, call = _bwd(eng, dy, P, st, par, B, R, C_, sh, gated, g0=g0)
    names = _run(eng, form, call, F.post_bwd_kernels(B, R, C_, sh, gated, form != "noonepass", form != "nostream", form == "det", True, True))
    bform = names[0].split("<")[0]
    dpr, grads, bias = F.backward(P3.double(), par64, dy.reshape(B, R, C_).double(), gated, stats=st.double(), shuffle=sh, bias=True)
    Lg = F.post_chain(B, R)
    edp, eg = F.norm_bwd_bound(P3.double(), par64, dy.reshape(B, R, C_).double(), gated, st.double(), sh, L1, Lg)
    f = _assert_within(dp.reshape(B, R // sh, -1), dpr, edp, ("sample", "conv row", "column"), what + ": dP " + str(names), "dP " + bform)
    for i, (t, r) in enumerate(zip(g, list(grads) + list(bias))):
        if r is None:
            continue
        if i < 4:
            eb = eg[i // 2][i % 2] + F.gamma(Lg) * torch.from_numpy(np.abs(g0[i])).cuda()
        else:
            ed = edp.reshape(B * R // sh, -1).sum(dim=0)
            Cc = C_ * sh
            ed = ed[:Cc] if i == 4 else ed[Cc:]
            tabs = dpr.abs().reshape(B * R // sh, -1).sum(dim=0)
            tabs = tabs[:Cc] if i == 4 else tabs[Cc:]
            eb = ed + F.gamma(Lg) * (tabs + torch.from_numpy(np.abs(g0[i])).cuda())
        _assert_within(t, r + torch.from_numpy(g0[i]).cuda().double(), eb, ("column",), what + ": " + GRAD_NAMES[i] + " " + str(names),
                       GRAD_NAMES[i][:-2] + " " + bform)
    if data_only:
        # the discriminator's data-gradient pass of a generator step: no parameter gradient, the same dP bits
        dp2, _, call = _bwd(eng, dy, P, st, par, B, R, C_, sh, gated, affine=False, bias=False)
        _run(eng, form, call, F.post_bwd_kernels(B, R, C_, sh, gated, True, True, False, False, False))
        assert torch.equal(dp2, dp), what + ": the data-gradient-only pass changes dP"
    print("%s: worst dP fraction %.3g" % (what, f))


# ---- packed ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("div,sh,gated", PACKED)
def test_packed_forward_is_the_unpacked_per_utterance(eng, div, sh, gated):
    """each utterance's statistics and y equal the unpacked stats + apply call on it alone bitwise, and lie within the dense bounds"""
    C_ = 64
    lens = [n // div for n in UTTS]                                    # conv rows per utterance at P's level
    off = np.concatenate([[0], np.cumsum(UTTS)]).astype(np.int64)
    rows = sum(lens)
    g = torch.Generator(device="cuda").manual_seed(_seed("pk", div, sh, gated))
    nt = C_ * sh * (2 if gated else 1)
    P = torch.randn(rows, nt, device="cuda", generator=g) * 3 + 1
    P[0] += 40                                                         # the first utterance's position 0 far out
    par = [(torch.randn(C_, device="cuda", generator=g) * 0.3 + k) for k in (0.0, 1.0, 0.0, 1.0)]
    if not gated:
        par[2] = par[3] = None
    R = rows * sh
    resid = None if gated else torch.randn(R * C_, device="cuda", generator=g)
    y, st, call = _fwd(eng, P, par, 1, R, C_, sh, gated, resid, packed=(off, div, max(UTTS)))
    names = _run(eng, "default", call, F.post_fwd_kernels(len(UTTS), max(UTTS) * sh // div, C_, sh, gated, resid is not None, packed=True))
    r0 = 0
    for u, n in enumerate(lens):
        Pu = P[r0:r0 + n].contiguous()
        ru = None if resid is None else resid[r0 * sh * C_:(r0 + n) * sh * C_].contiguous()
        yu, stu, cu = _fwd(eng, Pu, par, 1, n * sh, C_, sh, gated, ru)
        _run(eng, "nostream", cu, F.post_fwd_kernels(1, n * sh, C_, sh, gated, ru is not None, stream=False))
        what = "packed div %d sh %d utterance %d (%d conv rows from row %d)" % (div, sh, u, n, r0)
        _assert_equal(st[u].cpu().numpy(), stu[0].cpu().numpy(), ("stat", "channel"), what + ": statistics")
        _assert_equal(y[r0 * sh * C_:(r0 + n) * sh * C_].cpu().numpy(), yu.cpu().numpy(), ("element",), what + ": y")
        P3 = Pu.reshape(1, n, nt)
        _check_stats_dense(st[u:u + 1], P3, gated, sh, "shifted", F.post_chain(1, n * sh), what)
        r0 += n


# ---- coverage ------------------------------------------------------------------------------------------------------------------------
def _all_reached():
    got = set()
    for R0, sh, gated, form in LATTICE_FWD:
        got.update(F.post_fwd_kernels(5, R0 * sh, 128, sh, gated, not gated, form != "nostream"))
    for R0, sh, gated, form, _ in LATTICE_BWD:
        got.update(F.post_bwd_kernels(4, R0 * sh, 128, sh, gated, form != "noonepass", True, form == "det", True, True))
    for R, sh, gated, C_, form in ZERO_SUM:
        got.update(F.post_bwd_kernels(3, R, C_, sh, gated, True, True, form == "det", True, True))
    for name, B, R, C_, sh, gated, resid in DENSE:
        for form in FORMS:
            if form != "default" and B > 512 or (form in ("noonepass", "det") and name.startswith("D.")):
                continue
            got.update(F.post_fwd_kernels(B, R, C_, sh, gated, resid, form != "nostream"))
            got.update(F.post_bwd_kernels(B, R, C_, sh, gated, form != "noonepass", form != "nostream", form == "det", True, True))
    for div, sh, gated in PACKED:
        got.update(F.post_fwd_kernels(1, 4, 64, sh, gated, not gated, packed=True))
    return got


def test_every_instantiation_is_reached():
    src = open(os.path.join(ROOT, "voice-converter-cyclegan_b200", "csrc", "simt_kernels.cu")).read()
    want = set(F.post_instantiations(src)) | {"reduce_parts_kernel"}
    got = _all_reached()
    missing = sorted(want - got)
    assert not missing, "instantiations no case reaches: %s" % missing
    print("reached: %s" % ", ".join(sorted(got)))


def test_zz_profiler_saw_every_instantiation():
    """over the module's cases (run before this one), torch.profiler recorded every instantiation; prints the worst measured fraction
    of each bound"""
    for k in sorted(WORST):
        print("worst %-36s %.3g" % (k, WORST[k]))
    if not WORST:
        pytest.skip("run with the rest of the module")
    src = open(os.path.join(ROOT, "voice-converter-cyclegan_b200", "csrc", "simt_kernels.cu")).read()
    missing = sorted((set(F.post_instantiations(src)) | {"reduce_parts_kernel"}) - SEEN)
    assert not missing, "instantiations the profiler never saw run: %s" % missing
