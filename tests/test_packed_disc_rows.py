"""CPU checks of the row rules behind the packed discriminator (cgvc_discriminator_forward_packed): utterances of different lengths,
every length a multiple of 16, concatenated along time, with every level of the network a packed 2-D grid (kernels.cuh PackGeom2).
A grid of H rows at time divisor d holds utterance u as [H][len_u / d] at rows H * off[u] / d.  The kernels' index rules are restated
here in numpy and held against the oracle's per-utterance TF-'SAME' 2-D convolution and instance norm, for every convolution of the
discriminator, so that a row that strays into a neighbouring utterance shows without a GPU:

- the forward gather (tc_gg_nt_kernel<.., 2>, gg_simt_kernel<.., PackGeom2>, the c1 kernels with PackGeom2): row m of the output
  grid finds its utterance by pack2_pos (pack_find at frame floor(m * dout / Hy)), splits its local row into (y, x) with the
  utterance's width, and reads (y * sy + oy, x * sx + ox) of its own utterance in the source grid, zero outside [0, Hs) x [0, W_u);
- the instance-norm segments: d_i's output grid is described by the row prefix sums H * off[u] / d (div 1), one sample per utterance."""
import numpy as np
import pytest
import torch

from oracle import cyclegan_oracle as O

LENGTHS = [32, 784, 16, 400, 48, 1392, 16, 128, 208]
OFF = np.concatenate([[0], np.cumsum(LENGTHS)]).astype(np.int64)
N = len(LENGTHS)
H0 = 24

# (name, kh, kw, sh, sw, rows of the input grid, time divisor of the input grid): every convolution of the discriminator
LAYERS = [("h1", 3, 3, 1, 2, 24, 1), ("d1", 3, 3, 2, 2, 24, 2), ("d2", 3, 3, 2, 2, 12, 4), ("d3", 6, 3, 1, 2, 6, 8)]


def pack_find(off, f):
    """kernels.cuh pack_find: the utterance u with off[u] <= f < off[u+1]"""
    return np.searchsorted(off, f, side="right") - 1


def pack2_pos(off, H, div, m):
    """kernels.cuh pack2_pos: utterance, (y, x) of rows m of a grid of H rows at divisor div"""
    u = pack_find(off, m * div // H)
    w = (off[u + 1] - off[u]) // div
    loc = m - H * off[u] // div
    return u, loc // w, loc % w


def pack2_row(off, u, H, div, y, x):
    """kernels.cuh pack2_row: the row of (y, x) of utterance u, -1 outside its [0, H) x [0, len_u / div)"""
    w = (off[u + 1] - off[u]) // div
    ok = (y >= 0) & (y < H) & (x >= 0) & (x < w)
    return np.where(ok, H * off[u] // div + y * w + x, -1)


def same_taps(kh, kw, sh, sw, H):
    """geom.h fwd_geom over (1, H, all frames / div): the tap offsets, the same for every utterance (every width is even)"""
    pt, _ = O.same_pad(H, kh, sh)
    pl, _ = O.same_pad(64, kw, sw)
    for W in (2, 4, 50, 174):
        assert O.same_pad(W, kw, sw)[0] == pl
    return [(i - pt, j - pl) for i in range(kh) for j in range(kw)]


def fwd_source_rows(off, kh, kw, sh, sw, H, div):
    """[taps, M] source row of every (tap, output row) of the packed 2-D forward gather, -1 for a zero row"""
    Ho, dout = -(-H // sh), div * sw
    M = Ho * int(off[-1]) // dout
    u, y, x = pack2_pos(off, Ho, dout, np.arange(M))
    return np.stack([pack2_row(off, u, H, div, y * sh + oy, x * sw + ox) for oy, ox in same_taps(kh, kw, sh, sw, H)])


def gather(x, rows):
    return np.where(rows[:, None] >= 0, x[np.maximum(rows, 0)], 0.0)


@pytest.mark.parametrize("name,kh,kw,sh,sw,H,div", LAYERS)
def test_packed_2d_gather_matches_per_utterance_convolution(name, kh, kw, sh, sw, H, div):
    rs = np.random.RandomState(kh * 100 + H + div)
    cin, cout = 3, 2
    x = rs.randn(H * int(OFF[-1]) // div, cin)
    w = rs.randn(kh, kw, cin, cout)
    b = torch.zeros(cout, dtype=torch.float64)
    ys = []
    for u in range(N):
        xu = x[H * OFF[u] // div:H * OFF[u + 1] // div].reshape(1, H, -1, cin)
        ys.append(O.conv2d_same(torch.tensor(xu), torch.tensor(w), b, (sh, sw))[0].reshape(-1, cout).numpy())
    y_ref = np.concatenate(ys)
    src = fwd_source_rows(OFF, kh, kw, sh, sw, H, div)
    assert src.shape[1] == len(y_ref)
    y = sum(gather(x, src[t]) @ w.reshape(kh * kw, cin, cout)[t] for t in range(kh * kw))
    assert np.allclose(y, y_ref, rtol=0, atol=1e-10), name


def test_rows_never_leave_their_utterance():
    for name, kh, kw, sh, sw, H, div in LAYERS:
        Ho, dout = -(-H // sh), div * sw
        src = fwd_source_rows(OFF, kh, kw, sh, sw, H, div)
        m = np.arange(src.shape[1])
        u_out = pack_find(OFF, m * dout // Ho)
        for t, rows in enumerate(src):
            ok = rows >= 0
            assert (pack_find(OFF, rows[ok] * div // H) == u_out[ok]).all(), (name, t)
            lo, hi = H * OFF[u_out] // div, H * OFF[u_out + 1] // div
            assert ((rows[ok] >= lo[ok]) & (rows[ok] < hi[ok])).all(), (name, t)


# (H, divisor) of the instance-normed outputs: d1, d2, d3
NORMS = [(12, 4), (6, 8), (6, 16)]


@pytest.mark.parametrize("H,div", NORMS)
def test_instance_norm_segments(H, div):
    """the row prefix sums the engine copies beside the offsets describe each utterance's rows at that level, and the kernels'
    per-segment statistics are the oracle's instance norm over the utterance's H x len_u / div positions"""
    rs = np.random.RandomState(H + div)
    C = 4
    seg = H * OFF // div
    assert (np.diff(seg) == H * np.array(LENGTHS) // div).all()
    P = rs.randn(int(seg[-1]), C) * 2 + 0.5
    beta, gamma = rs.randn(C), rs.randn(C)
    for u in range(N):
        r = P[seg[u]:seg[u + 1]]
        ref = O.instance_norm(torch.tensor(r.reshape(1, H, -1, C)), torch.tensor(beta), torch.tensor(gamma))
        m = r.mean(0)
        y = (r - m) / np.sqrt(((r - m) ** 2).mean(0) + O.IN_EPS) * gamma + beta
        assert np.allclose(y, ref.reshape(-1, C).numpy(), rtol=0, atol=1e-10)


def test_head_rows_are_the_callers_blocks():
    """the head is row-local: d3's output rows of utterance u are its [6][len_u / 16] probability block at 6 * off[u] / 16"""
    H, div = H0 // 4, 16
    for u in range(N):
        rows = pack2_row(OFF, np.full(H * LENGTHS[u] // div, u), H, div, np.repeat(np.arange(H), LENGTHS[u] // div),
                         np.tile(np.arange(LENGTHS[u] // div), H))
        assert (rows == H * OFF[u] // div + np.arange(H * LENGTHS[u] // div)).all()


def dgrad_classes(off, kh, kw, sh, sw, H, div):
    """the packed 2-D data gradient as the class kernels run it (geom.h dgrad_geoms over (1, H, all frames / div); tc_conv_dgrad and
    conv_dgrad_simt give them pk.div = div * sw): [(destination rows, [(weight tap, source rows or -1)])] per parity class.  Class (py,
    px) has Hy = (H - py + sh - 1) / sh rows at divisor div * sw; its row (y, x) reads d P at the output level (Ho rows, divisor
    div * sw) and is stored to (y * sh + py, x * sw + px) of its own utterance in the input grid"""
    pt, _ = O.same_pad(H, kh, sh)
    pl, _ = O.same_pad(64, kw, sw)
    Ho, dsrc = -(-H // sh), div * sw
    classes = []
    for py in range(sh):
        for px in range(sw):
            Hy = (H - py + sh - 1) // sh
            M = Hy * int(off[-1]) // dsrc
            u, y, x = pack2_pos(off, Hy, dsrc, np.arange(M))
            dst = pack2_row(off, u, H, div, y * sh + py, x * sw + px)
            taps = []
            for i in range(kh):
                for j in range(kw):
                    if (py + pt - i) % sh or (px + pl - j) % sw:
                        continue
                    taps.append((i * kw + j, pack2_row(off, u, Ho, dsrc, y + (py + pt - i) // sh, x + (px + pl - j) // sw)))
            classes.append((dst, taps))
    return classes


@pytest.mark.parametrize("name,kh,kw,sh,sw,H,div", LAYERS)
def test_packed_2d_backward_rows_match_per_utterance_autograd(name, kh, kw, sh, sw, H, div):
    """the weight-gradient rows (tc_gg_tn_kernel<.., 2>, wgrad_simt_kernel<true, PackGeom2>, the c1 weight gradients: the forward
    gather, a zero row outside the utterance) and every data-gradient parity class, against autograd per utterance"""
    rs = np.random.RandomState(kh * 1000 + H + div)
    cin, cout = 3, 2
    rows_in = H * int(OFF[-1]) // div
    x = rs.randn(rows_in, cin)
    w = rs.randn(kh, kw, cin, cout)
    wt = torch.tensor(w, requires_grad=True)
    b = torch.zeros(cout, dtype=torch.float64)
    xs, ys = [], []
    for u in range(N):
        xu = torch.tensor(x[H * OFF[u] // div:H * OFF[u + 1] // div].reshape(1, H, -1, cin), requires_grad=True)
        xs.append(xu)
        ys.append(O.conv2d_same(xu, wt, b, (sh, sw))[0].reshape(-1, cout))
    dy = rs.randn(sum(len(t) for t in ys), cout)
    torch.autograd.backward(ys, [torch.tensor(d) for d in np.split(dy, np.cumsum([len(t) for t in ys])[:-1])])
    dx_ref = np.concatenate([t.grad[0].reshape(-1, cin).numpy() for t in xs])
    src = fwd_source_rows(OFF, kh, kw, sh, sw, H, div)
    wf = w.reshape(kh * kw, cin, cout)
    dw = np.stack([gather(x, src[t]).T @ dy for t in range(kh * kw)])
    assert np.allclose(dw, wt.grad.numpy().reshape(kh * kw, cin, cout), rtol=0, atol=1e-9), name
    dx = np.full((rows_in, cin), np.nan)
    for dst, taps in dgrad_classes(OFF, kh, kw, sh, sw, H, div):
        assert (dst >= 0).all(), (name, "a class row outside its utterance")
        acc = np.zeros((len(dst), cin))
        for t, rows in taps:
            acc += gather(dy, rows) @ wf[t].T
        assert np.all(np.isnan(dx[dst])), (name, "a row written twice")
        dx[dst] = acc
    assert not np.isnan(dx).any(), (name, "a row never written")
    assert np.allclose(dx, dx_ref, rtol=0, atol=1e-10), name
