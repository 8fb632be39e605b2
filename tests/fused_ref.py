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
        a, g = shuffle_rows(a), shuffle_rows(g)
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


def backward(bp, par, dy, gated, stats=None):
    """closed form of the IN (+ GLU) backward of a layer without shuffle in float64: dP [B, R, Ntot] and the parameter gradients
    (dbeta_a, dgamma_a, dbeta_g, dgamma_g; the last two None when not gated), with the exact statistics of bp or the given ones"""
    bp = _t(bp).double()
    dy = _t(dy, bp.device).double()
    a, g = branches(bp, gated, 1)
    beta_a, gamma_a, beta_g, gamma_g = (None if t is None else _t(t, bp.device).double() for t in par)
    if stats is None:
        ma, ra = stats_of(a)
        mg, rg = stats_of(g) if gated else (None, None)
    else:
        s = _t(stats, bp.device).double()
        ma, ra, mg, rg = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    if not gated:
        dx, db, dgm = _in_bwd(a, ma, ra, gamma_a, dy)
        return dx, (db, dgm, None, None)
    na = (a - ma[:, None]) * ra[:, None] * gamma_a + beta_a
    sg = torch.sigmoid((g - mg[:, None]) * rg[:, None] * gamma_g + beta_g)
    dna = dy * sg
    dng = dna * na * (1 - sg)
    dxa, dba, dga = _in_bwd(a, ma, ra, gamma_a, dna)
    dxg, dbg, dgg = _in_bwd(g, mg, rg, gamma_g, dng)
    return torch.cat([dxa, dxg], dim=-1), (dba, dga, dbg, dgg)


def backward_autograd(bp, par, dy, gated, resid=None):
    """the same by autograd of forward_oracle (exact statistics)"""
    bp = _t(bp).double().clone().requires_grad_(True)
    ps = [None if t is None else _t(t).double().clone().requires_grad_(True) for t in par]
    y = forward_oracle(bp, ps, gated, 1, resid=torch.zeros(bp.shape[0], bp.shape[1], bp.shape[2], dtype=torch.float64) if not gated else None)
    y.backward(_t(dy).double())
    return bp.grad, tuple(None if t is None else t.grad for t in ps)


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
