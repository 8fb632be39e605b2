"""float64 references of the generator's instance-normed layers, as the fused gather-GEMM epilogues compute them
(csrc/tc_gemm.cu nt_tile_epilogue), and an integer lattice on which their convolutions are exact.

Layer forms (module.py:66-146), P = conv(x) + bias [B, R, Ntot] with the a branch in columns [0, Cout) and the gate branch after:
    gated (EPI 1):        y = IN(a) * sigmoid(IN(g))
    residual h2 (EPI 2):  y = resid + IN(a)
    gated + shuffle (EPI 5): conv row r, column s * C + c (C = Cout / 2) is output row 2r + s, channel c of the shuffled view, and
                          IN runs over its 2R positions
The backward forms (EPI 3 / 4) take dY, the gradient of y, and give dP and the affine-parameter gradients.

Everything here is built on the oracle's instance_norm, glu, pixel_shuffle_reshape and conv1d_same; tests/test_fused_ref.py pins it.

The lattice: x in {0, +-1, +-2} on a sparsity mask, w in {+-1, +-2}, integer biases and residuals, gamma powers of two and integer
beta.  Then every product and every partial sum of P is an integer, and when the certificate holds (every sum of |terms| below 2^24)
P is exact in fp32 whatever the summation order -- in every precision, as the bf16 and e4m3 lo planes of such values are zero.  The
per-sample column sums of P are exact too, and R and 2R are powers of two, so the kernels' means are exact.
"""
import re

import numpy as np
import torch

from oracle import cyclegan_oracle as O

EPS = O.IN_EPS
# the generator layers whose instance norm the forward epilogues fuse: (Cin, kw, Cout, stride, gated, shuffle, EPI)
LAYERS = {
    "d1": (128, 5, 256, 2, True, 1, 1),
    "d2": (256, 5, 512, 2, True, 1, 1),
    "res_h1": (512, 3, 1024, 1, True, 1, 1),
    "res_h2": (1024, 3, 512, 1, False, 1, 2),
    "u1": (512, 5, 1024, 1, True, 2, 5),
    "u2": (512, 5, 512, 1, True, 2, 5),
}
# the data-gradient launches whose epilogue runs the upstream layer's IN backward: (downstream layer, upstream layer, EPI)
BWD_PAIRS = {
    "res_h2>res_h1": ("res_h2", "res_h1", 3),
    "res_h1>res_h2": ("res_h1", "res_h2", 4),
    "res_h1>d2": ("res_h1", "d2", 3),
}


def _t(a, device="cpu"):
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).to(device)


def conv_p(x, wa, wg, ba, bg, stride, device="cpu"):
    """P [B, R, Ntot] in float64: the a branch, then the gate branch (wg None: not gated)"""
    x = _t(x, device).double()
    a = O.conv1d_same(x, _t(wa, device).double(), _t(ba, device).double(), stride)
    if wg is None:
        return a
    return torch.cat([a, O.conv1d_same(x, _t(wg, device).double(), _t(bg, device).double(), stride)], dim=-1)


def shuffle_rows(pb):
    """the kernels' reading of one branch [B, R, Cc] of a shuffled layer: output row 2r + s, channel c = conv row r, column s * Cc/2 + c"""
    B, R, Cc = pb.shape
    C = Cc // 2
    out = pb.new_empty(B, 2 * R, C)
    out[:, 0::2, :] = pb[:, :, :C]
    out[:, 1::2, :] = pb[:, :, C:]
    return out


def branches(P, gated, shuffle):
    """(a, g) in the normalised view [B, R * shuffle, C]; g None when not gated"""
    P = _t(P)
    Cc = P.shape[-1] // (2 if gated else 1)
    a, g = P[..., :Cc], (P[..., Cc:] if gated else None)
    if shuffle == 2:
        a, g = shuffle_rows(a), (None if g is None else shuffle_rows(g))
    return a, g


def stats_of(v):
    """exact (mean, rstd) per (sample, channel) of v [B, R, C] in float64"""
    m = v.mean(dim=1)
    var = ((v - m[:, None, :]) ** 2).mean(dim=1)
    return m, torch.rsqrt(var + EPS)


def forward(P, par, gated, shuffle, resid=None, stats=None):
    """y [B, R * shuffle, C] from P in float64, with the exact statistics of P (stats None) or the given ones: a [B, 4, C] array of
    (mean_a, rstd_a, mean_g, rstd_g).  par = (beta_a, gamma_a, beta_g, gamma_g).  Returns y and the statistics used."""
    a, g = branches(_t(P).double(), gated, shuffle)
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t, a.device).double() for t in par)
    if stats is None:
        ma, ra = stats_of(a)
        mg, rg = stats_of(g) if gated else (torch.zeros_like(ma), torch.ones_like(ra))
    else:
        s = _t(stats, a.device).double()
        ma, ra, mg, rg = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    na = (a - ma[:, None]) * ra[:, None] * gamma_a + beta_a
    if gated:
        y = na * torch.sigmoid((g - mg[:, None]) * rg[:, None] * gamma_g + beta_g)
    else:
        y = na + _t(resid, a.device).double()
    return y, torch.stack([ma, ra, mg, rg], dim=1)


def forward_oracle(P, par, gated, shuffle, resid=None):
    """the same forward composed from the oracle's instance_norm / glu / pixel_shuffle_reshape (exact statistics)"""
    P = _t(P).double()
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t).double() for t in par)
    Cc = P.shape[-1] // (2 if gated else 1)
    a = P[..., :Cc]
    if shuffle == 2:
        a = O.pixel_shuffle_reshape(a)
    na = O.instance_norm(a, beta_a, gamma_a)
    if not gated:
        return na + _t(resid).double()
    g = P[..., Cc:]
    if shuffle == 2:
        g = O.pixel_shuffle_reshape(g)
    return O.glu(na, O.instance_norm(g, beta_g, gamma_g))


def _in_bwd(v, m, r, gamma, dn):
    """IN backward per (sample, channel), statistics given: dx = gamma r (dn - mean(dn) - xhat mean(dn xhat)); (dx, dbeta, dgamma)"""
    xh = (v - m[:, None]) * r[:, None]
    dx = gamma * r[:, None] * (dn - dn.mean(dim=1, keepdim=True) - xh * (dn * xh).mean(dim=1, keepdim=True))
    return dx, dn.sum(dim=(0, 1)), (dn * xh).sum(dim=(0, 1))


def unshuffle_rows(v):
    """the inverse of shuffle_rows: the view [B, 2R, C] back in conv layout [B, R, 2C]"""
    return torch.cat([v[:, 0::2, :], v[:, 1::2, :]], dim=-1)


def backward(bp, par, dy, gated, stats=None, shuffle=1, bias=False):
    """closed form of the IN (+ GLU) backward in float64: dP [B, R, Ntot] in the layout of bp (conv rows; with shuffle 2 the norm runs
    over the 2R positions of the shuffled view) and the parameter gradients (dbeta_a, dgamma_a, dbeta_g, dgamma_g; the last two None
    when not gated), with the exact statistics of bp or the given ones.  bias: also the conv-bias gradients, the column sums of dP
    (dbias_a, dbias_g [Cout]; conv column s * C + c feeds only the phase-s positions of the view)."""
    bp = _t(bp).double()
    dy = _t(dy, bp.device).double()
    a, g = branches(bp, gated, shuffle)
    unview = unshuffle_rows if shuffle == 2 else (lambda v: v)
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t, bp.device).double() for t in par)
    if stats is None:
        ma, ra = stats_of(a)
        mg, rg = stats_of(g) if gated else (None, None)
    else:
        s = _t(stats, bp.device).double()
        ma, ra, mg, rg = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    if not gated:
        dx, db, dgm = _in_bwd(a, ma, ra, gamma_a, dy)
        dP, grads = unview(dx), (db, dgm, None, None)
    else:
        na = (a - ma[:, None]) * ra[:, None] * gamma_a + beta_a
        sg = torch.sigmoid((g - mg[:, None]) * rg[:, None] * gamma_g + beta_g)
        dna = dy * sg
        dng = dna * na * (1 - sg)
        dxa, dba, dga = _in_bwd(a, ma, ra, gamma_a, dna)
        dxg, dbg, dgg = _in_bwd(g, mg, rg, gamma_g, dng)
        dP, grads = torch.cat([unview(dxa), unview(dxg)], dim=-1), (dba, dga, dbg, dgg)
    if not bias:
        return dP, grads
    cs = dP.sum(dim=(0, 1))
    Cc = dP.shape[-1] // (2 if gated else 1)
    return dP, grads, (cs[:Cc], cs[Cc:] if gated else None)


def backward_autograd(bp, par, dy, gated, resid=None, shuffle=1, bias=False):
    """the same by autograd of forward_oracle (exact statistics); bias: also the conv-bias gradients, those of a bias added to bp"""
    bp = _t(bp).double().clone().requires_grad_(True)
    ps = [None if t is None else _t(t).double().clone().requires_grad_(True) for t in par]
    dy = _t(dy).double()
    b = torch.zeros(bp.shape[-1], dtype=torch.float64, requires_grad=True)
    y = forward_oracle(bp + b, ps, gated, shuffle, resid=None if gated else torch.zeros_like(dy))
    y.backward(dy)
    grads = tuple(None if t is None else t.grad for t in ps)
    return (bp.grad, grads, b.grad) if bias else (bp.grad, grads)


# ---- the integer lattice ---------------------------------------------------------------------------------------------------------
# per-sample densities of x: an all-zero sample (variance 0: rstd = eps^-1/2), a sample with one nonzero input (small variance: the
# epsilon matters), then sparse and dense ones
DENSITIES = (0.0, -1.0, 0.3, 0.05, 0.6)


def lattice_x(rng, B, W, Cin):
    x = np.zeros((B, W, Cin), np.float32)
    for b in range(B):
        d = DENSITIES[b % len(DENSITIES)]
        if d < 0:
            x[b, rng.integers(W), rng.integers(Cin)] = rng.choice([-2, -1, 1, 2])
        elif d > 0:
            mask = rng.random((W, Cin)) < d
            x[b][mask] = rng.choice([-2, -1, 1, 2], int(mask.sum()))
    return x


def lattice_weights(rng, kw, Cin, Cout):
    return rng.choice(np.array([-2, -1, 1, 2], np.float32), (kw, Cin, Cout))


def lattice_affine(rng, C):
    """gamma powers of two, beta small integers"""
    return (rng.integers(-2, 3, C).astype(np.float32), (rng.choice([-1.0, 1.0], C) * np.exp2(rng.integers(-2, 2, C))).astype(np.float32))


def lattice_forward_case(layer, B, R, seed):
    """x, wa, wg, ba, bg, par (beta_a, gamma_a, beta_g, gamma_g), resid for `layer` with R output positions per sample"""
    Cin, kw, Cout, sw, gated, sh, _ = LAYERS[layer]
    rng = np.random.default_rng(seed)
    x = lattice_x(rng, B, R * sw, Cin)
    wa = lattice_weights(rng, kw, Cin, Cout); ba = rng.integers(-3, 4, Cout).astype(np.float32)
    wg = bg = None
    if gated:
        wg = lattice_weights(rng, kw, Cin, Cout); bg = rng.integers(-3, 4, Cout).astype(np.float32)
    C = Cout // sh
    beta_a, gamma_a = lattice_affine(rng, C)
    beta_g, gamma_g = lattice_affine(rng, C) if gated else (None, None)
    resid = None if gated else rng.integers(-4, 5, (B, R, Cout)).astype(np.float32)
    return x, wa, wg, ba, bg, (beta_a, gamma_a, beta_g, gamma_g), resid


def dense_forward_case(layer, B, R, seed):
    """unit-scale randn operands; sample b's input is scaled by 2^-(4 (b % 4)), so that some samples' variance lies near epsilon"""
    Cin, kw, Cout, sw, gated, sh, _ = LAYERS[layer]
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, R * sw, Cin)).astype(np.float32)
    x *= np.exp2(-4.0 * (np.arange(B) % 4)).astype(np.float32)[:, None, None]
    s = 1.0 / np.sqrt(kw * Cin)
    wa = (rng.standard_normal((kw, Cin, Cout)) * s).astype(np.float32); ba = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    wg = bg = None
    if gated:
        wg = (rng.standard_normal((kw, Cin, Cout)) * s).astype(np.float32); bg = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    C = Cout // sh
    aff = lambda: ((rng.standard_normal(C) * 0.3).astype(np.float32), (rng.standard_normal(C) * 0.3 + 1.0).astype(np.float32))
    beta_a, gamma_a = aff()
    beta_g, gamma_g = aff() if gated else (None, None)
    resid = None if gated else rng.standard_normal((B, R, Cout)).astype(np.float32)
    return x, wa, wg, ba, bg, (beta_a, gamma_a, beta_g, gamma_g), resid


def certificate(x, wa, wg, ba, bg, stride, resid=None, device="cpu"):
    """(largest sum of |terms| of any P element, largest per-(sample, column) sum of those over the sample's positions); both must lie
    below 2^24 for P and its column sums to be exact in fp32 in any order.  The residual adds one exact integer per y element."""
    ax = np.abs(x)
    A = conv_p(ax, np.abs(wa), None if wg is None else np.abs(wg), np.abs(ba), None if bg is None else np.abs(bg), stride, device)
    return float(A.max()), float(A.sum(dim=1).max())


def lattice_dgrad_case(layer_down, B, R, seed, accumulate):
    """dP [B, R, Ntot] of the downstream layer, its weights, and dx0 (accumulate) on the lattice: dY = dgrad(dP) + dx0 is exact"""
    Cin, kw, Cout, _, gated, _, _ = LAYERS[layer_down]
    rng = np.random.default_rng(seed)
    nt = Cout * (2 if gated else 1)
    dP = np.zeros((B, R, nt), np.float32)
    mask = rng.random((B, R, nt)) < 0.1
    dP[mask] = rng.choice([-2, -1, 1, 2], int(mask.sum()))
    wa = lattice_weights(rng, kw, Cin, Cout); wg = lattice_weights(rng, kw, Cin, Cout) if gated else None
    dx0 = rng.integers(-8, 9, (B, R, Cin)).astype(np.float32) if accumulate else None
    return dP, wa, wg, dx0


def dense_dgrad_case(layer_down, B, R, seed, accumulate):
    Cin, kw, Cout, _, gated, _, _ = LAYERS[layer_down]
    rng = np.random.default_rng(seed)
    nt = Cout * (2 if gated else 1)
    dP = rng.standard_normal((B, R, nt)).astype(np.float32)
    s = 1.0 / np.sqrt(kw * Cout)
    wa = (rng.standard_normal((kw, Cin, Cout)) * s).astype(np.float32)
    wg = (rng.standard_normal((kw, Cin, Cout)) * s).astype(np.float32) if gated else None
    dx0 = rng.standard_normal((B, R, Cin)).astype(np.float32) if accumulate else None
    return dP, wa, wg, dx0


def dgrad(dP, wa, wg, device="cpu"):
    """the data gradient of a stride-1 TF-'SAME' 1-D layer in float64: dx [B, R, Cin] from dP [B, R, Ntot] (autograd of the oracle)"""
    dP = _t(dP, device).double()
    B, R, _ = dP.shape
    Cin = wa.shape[1]
    x = torch.zeros(B, R, Cin, dtype=torch.float64, device=device, requires_grad=True)
    Cout = wa.shape[2]
    y = O.conv1d_same(x, _t(wa, device).double(), None)
    if wg is not None:
        y = torch.cat([y, O.conv1d_same(x, _t(wg, device).double(), None)], dim=-1)
    y.backward(dP)
    return x.grad


def upstream_case(layer_up, B, R, seed):
    """bp (the upstream layer's pre-norm output), its fp32 statistics and affine parameters for the backward cases"""
    _, _, Cout, _, gated, _, _ = LAYERS[layer_up]
    rng = np.random.default_rng(seed)
    nt = Cout * (2 if gated else 1)
    bp = (rng.standard_normal((B, R, nt)) * 1.5 + 0.2).astype(np.float32)
    _, st = forward(bp, _unit_par(Cout, gated), gated, 1, resid=None if gated else np.zeros((B, R, Cout), np.float32))
    stats = st.float().numpy()
    aff = lambda: ((rng.standard_normal(Cout) * 0.3).astype(np.float32), (rng.standard_normal(Cout) * 0.3 + 1.0).astype(np.float32))
    beta_a, gamma_a = aff()
    beta_g, gamma_g = aff() if gated else (None, None)
    return bp, stats, (beta_a, gamma_a, beta_g, gamma_g)


def _unit_par(C, gated):
    z, o = np.zeros(C, np.float32), np.ones(C, np.float32)
    return (z, o, z, o) if gated else (z, o, None, None)


# ---- rounding bounds of the instance-norm arithmetic (the fused epilogues and the separate kernels of csrc/simt_kernels.cu) -------
U = 2.0 ** -24
NORM_ULPS = 8            # y_bound: the normalised value's rounding


def y_bound(P, st, par, gated, shuffle, resid):
    """per-element bound of |y - float64(y from the kernel's P and statistics)|, u = 2^-24:
    normalised value n = fma(v, sc, of), sc = fl(rstd gamma), of = fl(beta - fl(mean sc)): four roundings, |dn| <= NORM_ULPS u (|v sc| +
    |mean sc| + |beta|) with a factor 2 over them;
    EPI 2: y = n + resid, one more rounding of |y|;  EPI 1 / 5: y = n_a * s(n_g), s = __fdividef(1, 1 + __expf(-n_g)) with __expf
    within 2 + 1.173 |n_g| ulp and __fdividef within 2 ulp: |ds| <= s (1 - s) |dn_g| + s (6 + 1.2 |n_g|) u, then one rounding of |y|"""
    a, g = branches(P, gated, shuffle)
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t).double().to(a.device) for t in par)
    ma, ra, mg, rg = st[:, 0, None], st[:, 1, None], st[:, 2, None], st[:, 3, None]

    def norm_err(v, m, r, gam, bet):
        sc = (r * gam).abs()
        return (v * (r * gam) + bet - m * (r * gam)), NORM_ULPS * U * ((v * sc).abs() + (m * sc).abs() + bet.abs())
    na, ea = norm_err(a, ma, ra, gamma_a, beta_a)
    if not gated:
        y = na + _t(resid).double().to(a.device)
        return ea + U * y.abs() + 1e-45
    ng, eg = norm_err(g, mg, rg, gamma_g, beta_g)
    s = torch.sigmoid(ng)
    y = na * s
    return s * ea + na.abs() * (s * (1 - s) * eg + s * (6 + 1.2 * ng.abs()) * U) + U * y.abs() + 1e-45


def gamma(L):
    """a sum along a chain of at most L fp32 additions lies within gamma_L * sum |terms| of the exact sum"""
    return L * U / (1 - L * U)


def stats_bound(v, form, L):
    """per (sample, channel) bounds (|mean - float64|, |rstd / float64 - 1|) of the statistics of v [B, R, C] (float64, the kernel's own
    P in the normalised view), for the forward form that computed them; L: the longest fp32 addition chain of its column sums.
      "stream" (post_fwd_stream): two-pass, m = fl(fl(sum x) fl(1/R)), var = fl(fl(sum fma(d, d)) fl(1/R)), d = fl(x - m).  The sum of
        the squares is over x - m of the rounded m, which adds R (m - mean)^2.
      "shifted" (post_stats + post_apply_fwd, and its packed form): one pass about k = x_0, the sample's position 0: S1 = sum fl(x - k),
        S2 = sum fl(d^2), m' = fl(S1 / R), var = max(fl(fl(S2 / R) - m'^2), 0), mean = fl(k + m').  S2 / R = var + (mean - x_0)^2, so the
        cancellation costs u ((x_0 - mean)^2 + var): the relative error grows with (x_0 - mean)^2 / var.
    Both: rstd = 1 / sqrtf(var + eps) with IEEE sqrtf and division: half the relative error of var + eps, plus 2 u."""
    R = v.shape[1]
    mean = v.mean(dim=1)
    var = ((v - mean[:, None]) ** 2).mean(dim=1)
    gl = gamma(L)
    if form == "stream":
        em = gl * v.abs().sum(dim=1) / R + 3 * U * mean.abs()
        ev = (gl + 3 * U) * var + em ** 2 + 2 * em * ((v - mean[:, None]).abs().mean(dim=1))
    else:
        k = v[:, 0]
        d = v - k[:, None]
        m1 = d.mean(dim=1)
        em1 = (gl + 3 * U) * d.abs().mean(dim=1) + 2 * U * d.abs().max(dim=1).values
        em = em1 + U * (k + m1).abs()
        s2 = (d * d).mean(dim=1)
        ev = (gl + 4 * U) * s2 + (2 * m1.abs() + em1) * em1 + 3 * U * m1 * m1 + 2 * U * d.abs().max(dim=1).values * d.abs().mean(dim=1)
    ve = var + EPS
    er = 0.5 * (ev + 2 * U * ve) / ve + 3 * U
    return 2 * em + 1e-45, 2 * er


def in_bwd_bound(v, m, r, gamma_, dn, edn, L):
    """per-element bound of |dx - float64| of one branch of the IN backward as the kernels form it: ah = fma(x, r, fl(-m r)),
    sc = fl(r gamma), S1 = sum dn, S2 = sum fma(dn, ah), c2 = fl(fl(sc S1) fl(1/R)), c3 likewise, dx = fma(sc, dn, -fma(ah, c3, c2));
    dn carries the error edn (from the GLU); the sums lie within gamma_L of exact over their |terms|.  v, dn [B, R, C]; m, r [B, C]."""
    R = v.shape[1]
    m, r = m[:, None], r[:, None]
    ah = (v - m) * r
    eah = 2 * U * ((v * r).abs() + (m * r).abs())
    sc = r * gamma_
    S1 = dn.sum(dim=1, keepdim=True); S2 = (dn * ah).sum(dim=1, keepdim=True)
    gl = gamma(L)
    eS1 = gl * dn.abs().sum(dim=1, keepdim=True) + edn.sum(dim=1, keepdim=True)
    eS2 = (gl + U) * (dn * ah).abs().sum(dim=1, keepdim=True) + (edn * ah.abs() + dn.abs() * eah).sum(dim=1, keepdim=True)
    c2, c3 = sc * S1 / R, sc * S2 / R
    ec2 = sc.abs() * eS1 / R + 4 * U * c2.abs()
    ec3 = sc.abs() * eS2 / R + 4 * U * c3.abs()
    dx = sc * dn - ah * c3 - c2
    e = sc.abs() * edn + U * (sc * dn).abs() + eah * c3.abs() + ah.abs() * ec3 + ec2 + 2 * U * ((ah * c3).abs() + c2.abs() + dx.abs())
    return 2 * e + 1e-45, 2 * eS1[:, 0], 2 * eS2[:, 0]


def norm_bwd_bound(bp, par, dy, gated, stats, shuffle, L, Lg):
    """bounds of the separate backward kernels at the given statistics: (dP [conv layout of bp] per element, [(dbeta_a, dgamma_a),
    (dbeta_g, dgamma_g)] per channel); L: the chain of the per-sample sums, Lg: that of the gradients over all samples"""
    bp = _t(bp).double(); dy = _t(dy, bp.device).double()
    a, g = branches(bp, gated, shuffle)
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t, bp.device).double() for t in par)
    s = _t(stats, bp.device).double()
    ma, ra, mg, rg = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    unview = unshuffle_rows if shuffle == 2 else (lambda v: v)
    if not gated:
        e, _, _ = in_bwd_bound(a, ma, ra, gamma_a, dy, torch.zeros_like(dy), L)
        _, gb, gg = in_bwd_bound(a, ma, ra, gamma_a, dy, torch.zeros_like(dy), Lg)
        return unview(e), [(gb.sum(dim=0), gg.sum(dim=0))]
    sca, scg = ra[:, None] * gamma_a, rg[:, None] * gamma_g
    na = (a - ma[:, None]) * sca + beta_a
    ng = (g - mg[:, None]) * scg + beta_g
    ena = NORM_ULPS * U * ((a * sca).abs() + (ma[:, None] * sca).abs() + beta_a.abs())
    eng = NORM_ULPS * U * ((g * scg).abs() + (mg[:, None] * scg).abs() + beta_g.abs())
    sg = torch.sigmoid(ng)
    es = sg * (1 - sg) * eng + sg * (6 + 1.2 * ng.abs()) * U
    dna = dy * sg
    edna = dy.abs() * es + U * dna.abs()
    dng = dna * na * (1 - sg)
    edng = (edna * na.abs() + dna.abs() * ena) * (1 - sg) + (dna * na).abs() * es + 3 * U * dng.abs()
    ea, _, _ = in_bwd_bound(a, ma, ra, gamma_a, dna, edna, L)
    eg, _, _ = in_bwd_bound(g, mg, rg, gamma_g, dng, edng, L)
    _, ba, ga = in_bwd_bound(a, ma, ra, gamma_a, dna, edna, Lg)
    _, bg, gg = in_bwd_bound(g, mg, rg, gamma_g, dng, edng, Lg)
    return torch.cat([unview(ea), unview(eg)], dim=-1), [(ba.sum(dim=0), ga.sum(dim=0)), (bg.sum(dim=0), gg.sum(dim=0))]


def post_chain(B, R):
    """an upper bound of the longest fp32 addition chain of every reduction the separate kernels make for B samples of R positions:
    rows per thread (at most R / 8 in sums + apply, NRT or NR in the streaming and one-pass forms), 5 shuffle levels, 8 warps or
    position lanes, then one atomic or one reduce_parts row per (sample, 32-position block), and the accumulated gradient itself"""
    return -(-R // 8) + 5 + 8 + B * -(-R // 32) + 1


# ---- which kernels a launch of the separate instance-norm kernels runs (launch_post_fwd / launch_post_bwd) -----------------------
POST_ROWS = 32
STREAM_FWD = ((32, 4), (16, 3), (16, 4), (8, 3), (8, 4), (4, 6))                  # (NQL, NRT): R = 256 / NQL * NRT, C % (4 NQL) == 0
STREAM_BWD = ((32, 4, True), (32, 4, False), (16, 3, True), (16, 4, True), (8, 3, True), (8, 4, True), (4, 6, True))


def _b(v):
    return "true" if v else "false"


def post_fwd_stream_dispatch(B, R, C, sh, gated, resid, stream):
    """the streaming forward's configuration (NQL, NRT) for a shape, or None"""
    if not (gated and not resid and stream and sh in (1, 2) and B * (C // 16) < 2 ** 30):
        return None
    for nql, nrt in STREAM_FWD:
        if R == 256 // nql * nrt and C % (4 * nql) == 0:
            return nql, nrt
    return None


def post_bwd_stream_dispatch(B, R, C, sh, gated, onepass, stream):
    if not (onepass and stream and sh in (1, 2) and B * (C // 16) < 2 ** 30):
        return None
    for nql, nrt, g in STREAM_BWD:
        if g == gated and R == 256 // nql * nrt and C % (4 * nql) == 0 and (gated or sh == 1):
            return nql, nrt, g
    return None


def post_fwd_kernels(B, R, C, sh, gated, resid=False, stream=True, packed=False):
    """the kernels (demangled names with their template arguments) one launch_post_fwd of an instance-normed layer runs, in order"""
    if packed:
        return ["post_stats_kernel<%s, true>" % _b(gated), "post_apply_fwd_kernel<true, %s, true>" % _b(gated)]
    cfg = post_fwd_stream_dispatch(B, R, C, sh, gated, resid, stream)
    if cfg:
        return ["post_fwd_stream_kernel<%d, %d>" % cfg]
    return ["post_stats_kernel<%s, false>" % _b(gated), "post_apply_fwd_kernel<true, %s, false>" % _b(gated)]


def post_bwd_kernels(B, R, C, sh, gated, onepass=True, stream=True, det=False, affine=True, bias=False):
    """the same for launch_post_bwd: deterministic mode takes sums + apply and reduces the per-sample sums (affine gradients given)
    and the bias partials (bias given) with reduce_parts"""
    if not det:
        cfg = post_bwd_stream_dispatch(B, R, C, sh, gated, onepass, stream)
        if cfg:
            return ["post_bwd_stream_kernel<%d, %d, %s>" % (cfg[0], cfg[1], _b(cfg[2]))]
        if R <= 64 and onepass:
            return ["post_bwd_onepass_kernel<%s, %d>" % (_b(gated), 4 if R <= 32 else 6 if R <= 48 else 8)]
    k = ["post_bwd_sums_kernel<%s>" % _b(gated)]
    if det and affine:
        k.append("reduce_parts_kernel")
    k.append("post_apply_bwd_kernel<true, %s>" % _b(gated))
    if det and bias:
        k.append("reduce_parts_kernel")
    return k


def post_instantiations(src):
    """every instantiation of the separate instance-norm kernels with has_in (demangled), from simt_kernels.cu's launch code"""
    fwd = re.search(r"#define STREAM_FWD_CONFIGS\(X\)(.*)", src).group(1)
    bwd = re.search(r"#define STREAM_CONFIGS\(X\)(.*)", src).group(1)
    onepass = sorted(set(int(n) for n in re.findall(r"ONEPASS\((\d+)\)", src)))
    out = ["post_fwd_stream_kernel<%s, %s>" % t for t in re.findall(r"X\((\d+), (\d+)\)", fwd)]
    out += ["post_bwd_stream_kernel<%s, %s, %s>" % t for t in re.findall(r"X\((\d+), (\d+), (true|false)\)", bwd)]
    out += ["post_bwd_onepass_kernel<%s, %d>" % (g, n) for g in ("true", "false") for n in onepass]
    for g in ("true", "false"):
        out += ["post_stats_kernel<%s, %s>" % (g, pk) for pk in ("true", "false")]
        out += ["post_apply_fwd_kernel<true, %s, %s>" % (g, pk) for pk in ("true", "false")]
        out += ["post_bwd_sums_kernel<%s>" % g, "post_apply_bwd_kernel<true, %s>" % g]
    return sorted(set(out))
