"""CPU checks of the row rules behind the packed generator tapes (cgvc_generator_forward_packed_tape / cgvc_generator_backward_tape of
kind 2): utterances of different lengths, every length a multiple of 4, concatenated along time.  The kernels' index rules are restated
here in numpy and held against the oracle's per-utterance TF-'SAME' convolution and instance norm and their autograd gradients, for
every layer shape of the generator, so that a row that strays into a neighbouring utterance shows without a GPU:

- the weight-gradient rows (tc_gemm.cu tc_gg_tn_kernel<.., PK>, simt_kernels.cu wgrad_simt_kernel<true, PackGeom>): K-row m of the
  output level finds its utterance at frame m * dout, reads local position (m - off[u] / dout) * stride + tap offset of the source
  level, and a zero row outside [0, len_u / div);
- the data-gradient parity classes (geom.h dgrad_geoms; tc_conv_dgrad and conv_dgrad_simt give the class kernels pk.div = div * stride):
  class px of a stride-s layer holds the input rows s * m + px, row m reads d P at the output level exactly as a stride-1 forward row;
- the instance-norm backward segments (post_bwd_sums_kernel / post_apply_bwd_kernel with PK): sample b owns the view rows
  [off[b] / div, off[b+1] / div), view row r of it is conv row (s0 + r) / sh, column ((s0 + r) % sh) * C of the pixel-shuffle view."""
import numpy as np
import pytest
import torch

from oracle import cyclegan_oracle as O

LENGTHS = [36, 516, 4, 128, 784, 12, 1400, 8, 132]
OFF = np.concatenate([[0], np.cumsum(LENGTHS)]).astype(np.int64)
N = len(LENGTHS)

# (name, taps, stride, divisor of the input level, pixel shuffle): every convolution of the generator, in the packed walk's geometry
LAYERS = [("h1", 15, 1, 1, 1), ("d1", 5, 2, 1, 1), ("d2", 5, 2, 2, 1), ("r.h1", 3, 1, 4, 1), ("r.h2", 3, 1, 4, 1),
          ("u1", 5, 1, 4, 2), ("u2", 5, 1, 2, 2), ("o1", 15, 1, 1, 1)]


def pack_find(off, f):
    """kernels.cuh pack_find: the utterance u with off[u] <= f < off[u+1]"""
    return np.searchsorted(off, f, side="right") - 1


def same_taps(k, s):
    """geom.h fwd_geom of a 1-D layer whose input length is a multiple of s: tap offsets j - pad_left (pad_left is the same for every
    utterance, as every length is a multiple of 4)"""
    pl, _ = O.same_pad(4 * s * 16, k, s)
    for L in (4 * s, 8 * s, 12 * s, 400 * s):
        assert O.same_pad(L, k, s)[0] == pl
    return [j - pl for j in range(k)]


def tn_source_rows(off, k, s, div):
    """[taps, M] source row of every (tap, output row) of the packed weight gradient, -1 for a zero row"""
    dout = div * s
    M = int(off[-1]) // dout
    m = np.arange(M)
    u = pack_find(off, m * dout)
    o0, o1 = off[u], off[u + 1]
    out = []
    for ox in same_taps(k, s):
        xx = (m - o0 // dout) * s + ox
        ok = (xx >= 0) & (xx < (o1 - o0) // div)
        out.append(np.where(ok, o0 // div + xx, -1))
    return np.stack(out)


def dgrad_classes(off, k, s, div):
    """the packed data gradient as the class kernels run it: [(dst rows, [(weight tap, source rows or -1)])] per parity class.  d P is
    read at the output level, of divisor div * s; class px's row m is input row s * m + px"""
    pl, _ = O.same_pad(4 * s * 16, k, s)
    dsrc = div * s
    classes = []
    for px in range(s):
        M = int(off[-1]) // div // s                       # (input rows - px + s - 1) / s: every level's row count is a multiple of s
        m = np.arange(M)
        u = pack_find(off, m * dsrc)
        o0, o1 = off[u], off[u + 1]
        rx = m - o0 // dsrc
        taps = []
        for j in range(k):
            if (px + pl - j) % s:
                continue
            xx = rx + (px + pl - j) // s
            ok = (xx >= 0) & (xx < (o1 - o0) // dsrc)
            taps.append((j, np.where(ok, o0 // dsrc + xx, -1)))
        classes.append((m * s + px, taps))
    return classes


def gather(x, rows):
    return np.where(rows[:, None] >= 0, x[np.maximum(rows, 0)], 0.0)


def per_utterance_conv(x, w, s, div):
    """the oracle over each utterance alone: outputs, and (given dY) d x and d w by autograd"""
    b = torch.zeros(w.shape[2], dtype=torch.float64)
    wt = torch.tensor(w, requires_grad=True)
    xs, ys = [], []
    for u in range(N):
        xu = torch.tensor(x[OFF[u] // div:OFF[u + 1] // div][None], requires_grad=True)
        xs.append(xu)
        ys.append(O.conv1d_same(xu, wt, b, stride=s)[0])
    return xs, wt, ys


@pytest.mark.parametrize("name,k,s,div,sh", LAYERS)
def test_packed_rows_match_per_utterance_convolution(name, k, s, div, sh):
    rs = np.random.RandomState(k * 10 + s + div)
    cin, cout = 3, 2
    rows_in = int(OFF[-1]) // div
    x = rs.randn(rows_in, cin)
    w = rs.randn(k, cin, cout)
    xs, wt, ys = per_utterance_conv(x, w, s, div)
    y = torch.cat(ys).detach().numpy()
    assert y.shape[0] == rows_in // s
    dy = rs.randn(*y.shape)
    torch.autograd.backward(ys, [torch.tensor(d) for d in np.split(dy, np.cumsum([len(t) for t in ys])[:-1])])
    dx_ref = np.concatenate([t.grad[0].numpy() for t in xs])
    src = tn_source_rows(OFF, k, s, div)
    # forward: the packed gather of the forward kernels (the same rows the weight gradient contracts over)
    fwd = sum(gather(x, src[t]) @ w[t] for t in range(k))
    assert np.allclose(fwd, y, rtol=0, atol=1e-10), name
    # weight gradient: dW[t] = X[src(., t)]^T dY
    dw = np.stack([gather(x, src[t]).T @ dy for t in range(k)])
    assert np.allclose(dw, wt.grad.numpy(), rtol=0, atol=1e-9), name
    # data gradient: every parity class, rows s * m + px written once
    dx = np.full((rows_in, cin), np.nan)
    for dst, taps in dgrad_classes(OFF, k, s, div):
        acc = np.zeros((len(dst), cin))
        for j, rows in taps:
            acc += gather(dy, rows) @ w[j].T
        assert np.all(np.isnan(dx[dst])), (name, "a row written twice")
        dx[dst] = acc
    assert not np.isnan(dx).any(), (name, "a row never written")
    assert np.allclose(dx, dx_ref, rtol=0, atol=1e-10), name


def test_rows_never_leave_their_utterance():
    for name, k, s, div, sh in LAYERS:
        for t, rows in enumerate(tn_source_rows(OFF, k, s, div)):
            m = np.arange(len(rows))
            ok = rows >= 0
            assert (pack_find(OFF, m[ok] * div * s) == pack_find(OFF, rows[ok] * div)).all(), (name, t)
            assert rows.max() < int(OFF[-1]) // div
        for dst, taps in dgrad_classes(OFF, k, s, div):
            for j, rows in taps:
                ok = rows >= 0
                assert (pack_find(OFF, dst[ok] * div) == pack_find(OFF, rows[ok] * div * s)).all(), (name, j)
                assert rows.max() < int(OFF[-1]) // (div * s)


def segment_view(off, vdiv, sh, b):
    """post_sample + the kernels' addressing: sample b's (conv row, column offset in units of C) for each of its view rows"""
    s0, R = off[b] // vdiv, (off[b + 1] - off[b]) // vdiv
    assert s0 % sh == 0 and 4 % (vdiv * sh) == 0
    r = np.arange(R)
    return s0 // sh + (r >> (sh - 1)), r & (sh - 1)


# (view-level divisor, shuffle, gated): the instance-normed layers' outputs -- d1, d2, r.h1, r.h2, u1, u2
NORMS = [(2, 1, True), (4, 1, True), (4, 1, False), (2, 2, True), (1, 2, True)]


@pytest.mark.parametrize("vdiv,sh,gated", NORMS)
def test_instance_norm_backward_segments(vdiv, sh, gated):
    rs = np.random.RandomState(vdiv * 10 + sh + gated)
    C = 4                                                # channels after the shuffle view; conv columns per branch Cc = C * sh
    Cc = C * sh
    conv_rows = int(OFF[-1]) // vdiv // sh
    P = rs.randn(conv_rows, 2 * Cc if gated else Cc) * 2 + 0.5
    ga, ba, gg, bg = (rs.randn(C) for _ in range(4))
    dy = rs.randn(int(OFF[-1]) // vdiv, C)
    # the oracle, per utterance: the conv output viewed through the pixel shuffle, instance norm (+ GLU)
    Pt = torch.tensor(P, requires_grad=True)
    prm = [torch.tensor(v, requires_grad=True) for v in (ga, ba, gg, bg)]
    outs = []
    for u in range(N):
        pu = Pt[OFF[u] // vdiv // sh:OFF[u + 1] // vdiv // sh][None]
        a = O.pixel_shuffle_reshape(pu[..., :Cc], sh) if sh > 1 else pu[..., :Cc]
        y = O.instance_norm(a, prm[1], prm[0])
        if gated:
            g = O.pixel_shuffle_reshape(pu[..., Cc:], sh) if sh > 1 else pu[..., Cc:]
            y = O.glu(y, O.instance_norm(g, prm[3], prm[2]))
        outs.append(y[0])
    torch.autograd.backward(outs, [torch.tensor(d) for d in np.split(dy, OFF[1:-1] // vdiv)])
    # the kernels' rule: per sample b, its view rows and statistics; dP written at (conv row, column offset)
    dP = np.full_like(P, np.nan)
    dga, dba, dgg, dbg = (np.zeros(C) for _ in range(4))
    for b in range(N):
        crow, phase = segment_view(OFF, vdiv, sh, b)
        cols = phase[:, None] * C + np.arange(C)[None, :]
        xa = P[crow[:, None], cols]
        xg = P[crow[:, None], Cc + cols] if gated else None
        d = dy[OFF[b] // vdiv:OFF[b + 1] // vdiv]
        R = len(crow)

        def stats(x):
            m = x.mean(0)
            return m, 1 / np.sqrt(((x - m) ** 2).mean(0) + O.IN_EPS)
        ma, ra = stats(xa)
        ahat = (xa - ma) * ra
        na = ahat * ga + ba
        dna = d
        if gated:
            mg, rg = stats(xg)
            ghat = (xg - mg) * rg
            sg = 1 / (1 + np.exp(-(ghat * gg + bg)))
            dna = d * sg
            dng = dna * na * (1 - sg)
            S1g, S2g = dng.sum(0), (dng * ghat).sum(0)
            dP[crow[:, None], Cc + cols] = rg * gg * dng - rg * gg * S1g / R - ghat * rg * gg * S2g / R
            dbg += S1g; dgg += S2g
        S1a, S2a = dna.sum(0), (dna * ahat).sum(0)
        dP[crow[:, None], cols] = ra * ga * dna - ra * ga * S1a / R - ahat * ra * ga * S2a / R
        dba += S1a; dga += S2a
    assert not np.isnan(dP).any()
    assert np.allclose(dP, Pt.grad.numpy(), rtol=0, atol=1e-9)
    assert np.allclose(dga, prm[0].grad.numpy(), atol=1e-9) and np.allclose(dba, prm[1].grad.numpy(), atol=1e-9)
    if gated:
        assert np.allclose(dgg, prm[2].grad.numpy(), atol=1e-9) and np.allclose(dbg, prm[3].grad.numpy(), atol=1e-9)
