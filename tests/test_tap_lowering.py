"""CPU checks of the algebra behind `edge_lower` (engine.cu edge_on, simt_kernels.cu im2col_taps_kernel / col2im_taps_kernel,
tc_gemm.cu w_src / tn_dst): the generator's two 15-tap layers with 24 channels on one side (module.py:85-86 h1, module.py:148 o1)
are computed on the GPU as dense 1 x 1 GEMMs over an im2col of the 24-channel tensor.  The index conventions the kernels implement
(dir = +1 / -1, pad_left = 7, zero outside the sample, TF kernel [15,24,128] read as a [360,128] matrix, o1's taps folded into
output columns t * 24 + n) are restated here in numpy and held against the oracle's TF-'SAME' convolution and its autograd
gradients, so a sign or offset error in the lowering would show without a GPU.  (The CUDA kernels themselves are compared with the
oracle and with the 15-tap gather-GEMMs in tests/test_gpu_model.py, and layer by layer against the float64 emulation of
their operand planes in tests/test_gpu_edge_layers.py; the restatements live in tests/edge_ref.py.)"""
import numpy as np
import torch

from oracle import cyclegan_oracle as O

from edge_ref import F_, KW, PL, col2im_replay, col2im_taps, fold_columns, im2col_taps, o1_z_weights


def test_pad_left_matches_tf_same():
    for T in (36, 128, 516):
        assert O.same_pad(T, KW, 1) == (PL, KW - 1 - PL)


def test_h1_is_a_dense_gemm_over_the_im2col_of_the_input():
    rs = np.random.RandomState(0)
    n, T, Cout = 3, 36, 16
    x = rs.randn(n, T, F_); w = rs.randn(KW, F_, Cout); b = rs.randn(Cout); dy = rs.randn(n, T, Cout)
    xt = torch.tensor(x, requires_grad=True); wt = torch.tensor(w, requires_grad=True)
    y_ref = O.conv1d_same(xt, wt, torch.tensor(b))
    y_ref.backward(torch.tensor(dy))
    xcol = im2col_taps(x, +1)
    w2 = w.reshape(KW * F_, Cout)                       # TF's [15,24,Cout] kernel as it lies in memory
    # forward
    assert np.allclose(xcol @ w2 + b, y_ref.detach().numpy(), atol=1e-10)
    # weight gradient lands in the same [15,24,Cout] memory
    dw = np.einsum('ntk,ntc->kc', xcol, dy).reshape(KW, F_, Cout)
    assert np.allclose(dw, wt.grad.numpy(), atol=1e-10)
    # data gradient: dense dP . W^T, then the tap-shifted sum with the opposite direction
    dx = col2im_taps(dy @ w2.T, F_, -1)
    assert np.allclose(dx, xt.grad.numpy(), atol=1e-10)


def test_o1_is_a_dense_gemm_with_folded_taps_plus_a_tap_shifted_sum():
    rs = np.random.RandomState(1)
    n, T, Cin = 2, 64, 20
    u = rs.randn(n, T, Cin); w = rs.randn(KW, Cin, F_); b = rs.randn(F_); dout = rs.randn(n, T, F_)
    ut = torch.tensor(u, requires_grad=True); wt = torch.tensor(w, requires_grad=True)
    y_ref = O.conv1d_same(ut, wt, torch.tensor(b))
    y_ref.backward(torch.tensor(dout))
    wf = fold_columns(w)                                # [Cin, 15 * 24]
    # forward: Z = U . W', out[m, c] = b[c] + sum_t Z[m + t - 7, (t, c)]
    z = u @ wf
    assert np.allclose(col2im_taps(z, F_, +1, b), y_ref.detach().numpy(), atol=1e-10)
    # backward: dZ = im2col(d_out) with the opposite direction; dense data and weight gradients
    dz = im2col_taps(dout, -1)
    assert np.allclose(dz @ wf.T, ut.grad.numpy(), atol=1e-10)
    dwf = np.einsum('ntc,ntk->ck', u, dz)               # [Cin, (t, n)]; tn_dst scatters column t * 24 + n to kernel element [t][c][n]
    dw = np.stack([dwf[:, t * F_:(t + 1) * F_] for t in range(KW)], axis=0)
    assert np.allclose(dw, wt.grad.numpy(), atol=1e-10)


def test_fold_index_functions():
    """w_src / tn_dst of tc_gemm.cu restated: column co of the folded layer <-> element (t, ci, n) of the [KW, Cin, 24] kernel."""
    Cin, fold_n = 8, F_
    w = np.arange(KW * Cin * fold_n, dtype=np.int64).reshape(KW, Cin, fold_n)
    flat = w.ravel()
    for co in (0, 5, 23, 24, 100, KW * fold_n - 1):
        for ci in (0, 3, Cin - 1):
            t = co // fold_n
            assert flat[(t * Cin + ci) * fold_n + (co - t * fold_n)] == w[t, ci, co % fold_n]


def test_fold_of_a_tf_kernel():
    """edge_ref.o1_z_weights: column t * 24 + n of the folded [256, 360] matrix is element [t][c][n] of o1's TF kernel, and the 1 x 1
    layer over it followed by the tap-shifted sum is the 15-tap convolution"""
    rs = np.random.RandomState(2)
    w = rs.randn(KW, 256, F_)
    wf = o1_z_weights(w)
    assert wf.shape == (1, 1, 256, KW * F_)
    for t, c, n in ((0, 0, 0), (7, 100, 5), (14, 255, 23), (3, 17, 12)):
        assert wf[0, 0, c, t * F_ + n] == w[t, c, n]
    u = rs.randn(2, 20, 256); b = rs.randn(F_)
    y_ref = O.conv1d_same(torch.tensor(u), torch.tensor(w), torch.tensor(b)).numpy()
    assert np.allclose(col2im_taps(u @ wf[0, 0], F_, +1, b), y_ref, atol=1e-10)


def test_col2im_replay_is_the_kernels_fp32_order():
    """edge_ref.col2im_replay: bias first, then taps 0..14 in order in float32, skipping rows outside the sample, per sample or per
    packed utterance; it agrees with the float64 col2im to fp32 rounding, and an element whose partial sums all round shows the order"""
    rs = np.random.RandomState(3)
    for direction in (+1, -1):
        for T, offsets in ((4, None), (36, None), (None, np.array([0, 4, 40, 48, 176]))):
            rows = 3 * T if T else int(offsets[-1])
            z = rs.randn(rows, KW * F_).astype(np.float32)
            b = rs.randn(F_).astype(np.float32) if direction == +1 else None
            got = col2im_replay(z, F_, direction, T=T, offsets=offsets, bias=b)
            bounds = [(s, T) for s in range(0, rows, T)] if T else list(zip(offsets[:-1], np.diff(offsets)))
            ref = np.concatenate([col2im_taps(z[s:s + L].astype(np.float64)[None], F_, direction, b)[0] for s, L in bounds])
            assert np.allclose(got, ref, rtol=0, atol=1e-5)
            # the same in a plain float32 loop, element by element
            s0, L = bounds[-1]
            for m in (0, L - 1, L // 2):
                for c in (0, 23):
                    acc = np.float32(b[c]) if b is not None else np.float32(0)
                    for t in range(KW):
                        ws = m + direction * (t - PL)
                        if 0 <= ws < L:
                            acc = np.float32(acc + z[s0 + ws, t * F_ + c])
                    assert acc == got[s0 + m, c], (direction, T, m, c)
    # order matters: 1 + 2^-24 + ... rounds differently from the reverse order; the replay takes the kernel's
    z = np.zeros((1, KW * F_), np.float32)
    z[0, PL * F_] = 2.0 ** -24
    got = col2im_replay(z, F_, +1, T=1, bias=np.ones(F_, np.float32))
    assert got[0, 0] == np.float32(1.0)
