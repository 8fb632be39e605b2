"""float64 references of the layers without an instance norm and of the loss heads, as the kernels of csrc/simt_kernels.cu compute
them, with a dyadic lattice on which their results are exact and the fp32 addition-chain lengths of their launches.

    GLU-only form (generator h1, discriminator h1): P [M, 2C] = [a | g], y = a * sigmoid(g); backward dP = (dy s, dy a s (1 - s)),
        conv-bias gradients = column sums of dP (post_apply_fwd / post_apply_bwd <false, true>).
    discriminator input layer: P = conv2d_same(x [B, H, W, 1], [w_a | w_g]) + [b_a | b_g], strides (1, 2), then the GLU above
        (conv_c1_glu_fwd, or conv_c1_fwd + the GLU-only form); backward: dW, db, dx (glu_bwd_wgrad_c1, glu_bwd_proj_c1 + gather_taps,
        or the GLU-only backward + wgrad_c1 + proj_taps + gather_taps).
    head: prob = sigmoid(y . w + b) (head_fwd); LSGAN loss coef * mean((prob - target)^2) and its gradients (head_loss_bwd).
    L1: mean |yhat - y| and d = s sign(yhat - y) (l1_loss_grad).

Everything is built on the oracle's conv2d_same, glu, l1_loss and l2_loss plus autograd; tests/test_glu_ref.py pins it.

The lattice: dyadic integers, gate weights and gate bias zero.  Then g = 0, and the kernels' fast sigmoid __fdividef(1, 1 + __expf(-0))
is exactly 1/2 (ex2.approx(0) = 1, rcp.approx(2) = 1/2), so y = a / 2 and dP = (dy / 2, dy a / 4) are exact, and so is every sum of them
in any order while the certificate holds: the sum of |terms| of every output, in units of its finest term, stays below 2^24.
"""
import numpy as np
import torch

from oracle import cyclegan_oracle as O

U = 2.0 ** -24
C1 = 128                 # channels per branch of the discriminator's input layer
KH, KW, SH, SW = 3, 3, 1, 2
NUM_SMS = 132
C1_ROWS = 64             # kC1Rows: rows staged per tile by the c1 weight-gradient kernels
POST_ROWS = 32           # kPostRows


def _t(a, device="cpu"):
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)).to(device)


# ---- references ------------------------------------------------------------------------------------------------------------------
def glu_forward(P):
    """y [.., C] of P [.., 2C] in float64"""
    P = _t(P).double()
    C = P.shape[-1] // 2
    return O.glu(P[..., :C], P[..., C:])


def glu_backward(P, dy):
    """(dP, dbias_a, dbias_g) in float64 by autograd of the oracle's glu; dbias = column sums of dP over every leading axis"""
    P = _t(P).double().clone().requires_grad_(True)
    glu_forward(P).backward(_t(dy, P.device).double())
    dP = P.grad
    C = dP.shape[-1] // 2
    s = dP.reshape(-1, 2 * C).sum(dim=0)
    return dP, s[:C], s[C:]


def out_rows(H, W, sh=SH, sw=SW):
    return -(-H // sh), -(-W // sw)


def disc_input_p(x, wa, wg, ba, bg, sh=SH, sw=SW, device="cpu"):
    """P [B * Ho * Wo, 2C] in float64: x [B, H, W], w [kh, kw, 1, C] (TF layout)"""
    x = _t(x, device).double()[..., None]
    a = O.conv2d_same(x, _t(wa, device).double(), _t(ba, device).double(), (sh, sw))
    g = O.conv2d_same(x, _t(wg, device).double(), _t(bg, device).double(), (sh, sw))
    return torch.cat([a, g], dim=-1).reshape(-1, 2 * a.shape[-1])


def disc_input_backward(x, wa, wg, P, dy, sh=SH, sw=SW, device="cpu"):
    """(dw_a, dw_g, db_a, db_g, dx) in float64: autograd of conv2d_same + glu, with the GLU's backward evaluated at the given P (the
    kernel's own) -- the convolution's output is replaced by P through a straight-through term, so that its rounding is not counted
    against the backward"""
    x = _t(x, device).double().clone().requires_grad_(True)
    ws = [_t(w, device).double().clone().requires_grad_(True) for w in (wa, wg)]
    bs = [torch.zeros(ws[0].shape[-1], dtype=torch.float64, device=device, requires_grad=True) for _ in range(2)]
    B, H, W = x.shape
    Ho, Wo = out_rows(H, W, sh, sw)
    a = O.conv2d_same(x[..., None], ws[0], bs[0], (sh, sw))
    g = O.conv2d_same(x[..., None], ws[1], bs[1], (sh, sw))
    Pk = _t(P, device).double().reshape(B, Ho, Wo, -1)
    C = a.shape[-1]
    a = a + (Pk[..., :C] - a).detach()
    g = g + (Pk[..., C:] - g).detach()
    O.glu(a, g).backward(_t(dy, device).double().reshape(B, Ho, Wo, C))
    return ws[0].grad, ws[1].grad, bs[0].grad, bs[1].grad, x.grad


def head_forward(y, w, b):
    """prob [rows] = sigmoid(y [rows, 1024] . w + b) in float64"""
    y = _t(y).double()
    return torch.sigmoid(y @ _t(w, y.device).double().reshape(-1) + _t(b, y.device).double().reshape(()))


def head_loss_backward(prob, y, w, target, coef, grad_mult=1.0):
    """(loss, dy, dw, db) in float64 from the kernel's own prob: loss = coef * l2_loss (the oracle's), gradients by autograd through the
    sigmoid's output (d prob / d z = prob (1 - prob)), times grad_mult"""
    prob = _t(prob).double()
    y = _t(y, prob.device).double()
    w = _t(w, prob.device).double().reshape(-1)
    z = torch.zeros_like(prob, requires_grad=True)
    p = prob + z * prob * (1 - prob)                      # value prob, derivative prob (1 - prob)
    loss = coef * O.l2_loss(torch.full_like(prob, float(target)), p)
    loss.backward()
    dz = z.grad * grad_mult
    return float(loss.detach()), dz[:, None] * w[None, :], (dz[:, None] * y).sum(dim=0), dz.sum()


def l1_loss(yhat, y):
    return float(O.l1_loss(_t(y).double(), _t(yhat).double()))


def l1_grad_bits(yhat, y, gscale=None, grad_mult=None, d0=None):
    """d as the kernel forms it, bit for bit: s = fl(fl(gscale * fl(1 / n)) * grad_mult) (or fl(1 / n) alone), d = s sign(yhat - y) (the
    sign of an fp32 difference is exact), then fl(d0 + d) when accumulating"""
    yhat = np.asarray(yhat, np.float32).reshape(-1); y = np.asarray(y, np.float32).reshape(-1)
    inv = np.float32(1) / np.float32(yhat.size)
    s = np.float32(gscale) * inv if gscale is not None else inv
    if grad_mult is not None:
        s = np.float32(s * np.float32(grad_mult))
    e = yhat - y
    d = np.where(e > 0, s, np.where(e < 0, -s, np.float32(0))).astype(np.float32)
    return d if d0 is None else (np.asarray(d0, np.float32).reshape(-1) + d).astype(np.float32)


# ---- the kernels' fp32 addition chains -------------------------------------------------------------------------------------------
# A sum of n fp32 terms added in any order along a chain of at most L additions lies within gamma_L * sum |terms| of the exact sum,
# gamma_L = L u / (1 - L u).  L below: the longest chain of one launch, from its own grid arithmetic.
def gamma(L):
    return L * U / (1 - L * U)


def c1_wgrad_chain(M):
    """glu_bwd_wgrad_c1 / wgrad_c1 (C = 128 per branch: 32 column quads, 8 position lanes): rows per thread, then the 8 lanes, then
    one atomic (or one slab row) per CTA"""
    rpb = -(-M // (NUM_SMS * 8)); rpb = -(-rpb // C1_ROWS) * C1_ROWS
    nb = -(-M // rpb)
    return -(-rpb // 8) + 8 + nb + 1


def post_bias_chain(B, R):
    """post_apply_bwd: 4 rows per thread, 8 position lanes, one atomic (or slab row) per (sample, 32-position block)"""
    return 4 + 8 + B * (-(-R // POST_ROWS)) + 1


def c1_dgrad_chain(kh=KH, kw=KW):
    """proj (8 products per lane, 5 butterfly / shuffle levels) then gather_taps (at most kh * kw terms)"""
    return 8 + 5 + kh * kw


def head_chain(rows):
    """head_loss_bwd: rows per warp (grid-stride over nb <= 296 CTAs of 8 warps), 8 warps, nb CTAs"""
    nb = min(-(-rows // 8), 296)
    return -(-rows // (nb * 8)) + 8 + nb + 1


def l1_chain(n):
    """l1_loss_grad: elements per thread (grid-stride over nb <= 592 CTAs), 5 shuffle levels, 8 warps, nb CTAs, and the 1 / n product"""
    nb = min(-(-n // 256), 592)
    return -(-n // (nb * 256)) + 5 + 8 + nb + 2


# ---- error of the kernels' own elementwise GLU arithmetic ------------------------------------------------------------------------
def sigmoid_err(g):
    """|fast sigmoid - sigmoid| <= s (6 + 1.2 |g|) u (__expf within 2 + 1.173 |g| ulp, __fdividef within 2 ulp)"""
    s = torch.sigmoid(g)
    return s * (6 + 1.2 * g.abs()) * U


def y_bound(P):
    """|y - float64(y of the kernel's P)|: the sigmoid's error times |a|, then one rounding"""
    P = _t(P).double()
    C = P.shape[-1] // 2
    a, g = P[..., :C], P[..., C:]
    return a.abs() * sigmoid_err(g) + U * (a * torch.sigmoid(g)).abs() + 1e-45


def dp_bound(P, dy):
    """|dP - float64| per element: da = fl(dy s) carries the sigmoid's error and one rounding; dg = fl(fl(da a) (1 - s)) adds two
    roundings, and 1 - s carries the sigmoid's absolute error"""
    P = _t(P).double(); dy = _t(dy, P.device).double()
    C = P.shape[-1] // 2
    a, g = P[..., :C], P[..., C:]
    s = torch.sigmoid(g); es = sigmoid_err(g)
    ea = dy.abs() * (es + U * s)
    eg = (dy * a).abs() * (es * (1 - s) + s * es + 4 * U * s * (1 - s)) + ea * a.abs()
    return torch.cat([ea, eg], dim=-1) + 1e-45


# ---- the lattice -----------------------------------------------------------------------------------------------------------------
def lattice_glu_case(rng, M, C):
    """P [M, 2C]: a integers in [-8, 8], g = 0; dy integers in [-4, 4]"""
    P = np.zeros((M, 2 * C), np.float32)
    P[:, :C] = rng.integers(-8, 9, (M, C))
    dy = rng.integers(-4, 5, (M, C)).astype(np.float32)
    return P, dy


def lattice_disc_case(rng, B, H, W):
    """x [B, H, W] sparse integers in {+-1, +-2}, w_a in {+-1, +-2}, integer b_a, w_g = b_g = 0"""
    x = np.zeros((B, H, W), np.float32)
    m = rng.random((B, H, W)) < 0.5
    x[m] = rng.choice([-2, -1, 1, 2], int(m.sum()))
    wa = rng.choice(np.array([-2, -1, 1, 2], np.float32), (KH, KW, 1, C1))
    ba = rng.integers(-3, 4, C1).astype(np.float32)
    z = np.zeros_like(wa)
    return x, wa, z, ba, np.zeros(C1, np.float32)


def lattice_disc_dy(rng, M):
    return rng.integers(-2, 3, (M, C1)).astype(np.float32)


def disc_certificate(x, wa, P, dy, sh=SH, sw=SW, device="cpu"):
    """the largest sum of |terms| of any backward output of the lattice case, in units of 1/4 (dP's finest unit; x and w are integers):
    dw and db over all rows, dx over its taps and channels.  Below 2^24, every such sum is exact in any order."""
    ax = np.abs(x); P = _t(P, device).double(); dy = _t(dy, device).double()
    C = P.shape[-1] // 2
    adp = torch.cat([dy.abs() / 2, (dy * P[:, :C]).abs() / 4], dim=-1)
    B, H, W = x.shape
    Ho, Wo = out_rows(H, W, sh, sw)
    # the convolution's backward with |x|, |w| and |dP| as its output gradient
    xt = _t(ax, device).double()[..., None]
    wt = _t(np.concatenate([np.abs(wa), np.abs(wa)], axis=-1), device).double().clone().requires_grad_(True)
    xg = xt.clone().requires_grad_(True)
    out = O.conv2d_same(xg, wt, None, (sh, sw))
    out.backward(adp.reshape(B, Ho, Wo, 2 * C))
    return 4 * max(float(wt.grad.max()), float(adp.sum(dim=0).max()), float(xg.grad.max()))


def lattice_head_case(rng, rows):
    """y [rows, 1024] integers in [-3, 3], w in {+-1}, b = 0, and every row's y . w = 0 (its second half is minus the first times
    w[:512] w[512:]), so that prob = 1/2 exactly and loss, dy, dw and db are dyadic"""
    w = rng.choice(np.array([-1.0, 1.0], np.float32), 1024)
    v = rng.integers(-3, 4, (rows, 512)).astype(np.float32)
    y = np.concatenate([v, -v * (w[:512] * w[512:])], axis=1)
    return y, w, np.zeros(1, np.float32)
