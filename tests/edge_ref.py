"""Host references of the generator's tap-lowered edge layers (`edge_lower`: engine.cu edge_on, simt_kernels.cu im2col_taps_kernel /
col2im_taps_kernel, tc_gemm.cu w_src / tn_dst): h1 (module.py:85-86) and o1 (module.py:148), 15 taps with 24 channels on one side,
computed as dense 1 x 1 GEMMs over an im2col of the 24-channel tensor.

- im2col_taps / col2im_taps / fold_columns: the index conventions the kernels implement, in float64 numpy (tests/test_tap_lowering.py
  holds them against the oracle's convolution);
- col2im_replay: col2im_taps_kernel's own fp32 arithmetic (bias first, then taps 0..14 in order, out-of-sample rows skipped), so that the
  kernel's out / dx can be required to equal it bit for bit on the device's own z / dz;
- the gemm_ref cases whose emulation gives the lowered GEMMs' exact results: the 15-tap convolutions (P, out, du, dx, the kernel
  gradients) and the 1 x 1 layers over the folded weights (z, dz).
"""
import numpy as np

KW, F_, PL = 15, 24, 7          # taps, narrow channel count, TF SAME pad_left at stride 1 = (kw - 1) // 2
H1_OUT, O1_IN = 128, 256        # h1's output channels per branch (a, g); o1's input channels


def sample_bounds(rows, T=None, offsets=None):
    """(start, length) of every sample: rows / T samples of T rows, or the packed utterances of offsets"""
    if offsets is not None:
        return [(int(offsets[u]), int(offsets[u + 1] - offsets[u])) for u in range(len(offsets) - 1)]
    return [(s, T) for s in range(0, rows, T)]


def im2col_taps(x, direction):
    """x [n, T, C] -> [n, T, KW * C]: out[m, t*C + c] = x[m + direction * (t - PL), c], zero outside the sample (im2col_taps_kernel)."""
    n, T, C = x.shape
    out = np.zeros((n, T, KW * C), dtype=x.dtype)
    for t in range(KW):
        s = direction * (t - PL)
        lo = max(0, -s); hi = max(lo, min(T, T - s))           # (a sample shorter than the shift: no rows)
        out[:, lo:hi, t * C:(t + 1) * C] = x[:, lo + s:hi + s, :]
    return out


def col2im_taps(z, C, direction, bias=None):
    """z [n, T, KW * C] -> [n, T, C]: y[m, c] = bias[c] + sum_t z[m + direction * (t - PL), t*C + c] over rows of the sample (col2im_taps_kernel)."""
    n, T, _ = z.shape
    y = np.zeros((n, T, C), dtype=z.dtype)
    for t in range(KW):
        s = direction * (t - PL)
        lo = max(0, -s); hi = max(lo, min(T, T - s))
        y[:, lo:hi, :] += z[:, lo + s:hi + s, t * C:(t + 1) * C]
    return y if bias is None else y + bias


def fold_columns(w):
    """TF kernel [KW, Cin, Cout] -> [Cin, KW * Cout] with column t * Cout + n (TcLayer::fold / w_src)."""
    return np.concatenate([w[t] for t in range(KW)], axis=1)


def col2im_replay(z, C, direction, T=None, offsets=None, bias=None):
    """col2im_taps_kernel in float32, in its order: y[m] = bias (or 0), then += z[m + direction * (t - PL), t*C:(t+1)*C] for t = 0..KW-1,
    skipping the taps whose row lies outside m's sample.  z [rows, >= KW * C] fp32 (rows of B samples of T, or packed utterances)."""
    z = np.asarray(z, np.float32)
    rows = z.shape[0]
    y = np.zeros((rows, C), np.float32)
    if bias is not None:
        y += np.asarray(bias, np.float32)
    for s0, L in sample_bounds(rows, T, offsets):
        ys = y[s0:s0 + L]
        zs = z[s0:s0 + L]
        for t in range(KW):
            s = direction * (t - PL)
            lo, hi = max(0, -s), min(L, L - s)
            if lo < hi:
                ys[lo:hi] += zs[lo + s:hi + s, t * C:(t + 1) * C]
    return y


def h1_case(B, T):
    """gemm_ref case of h1 with its two branches as one convolution of 2 x 128 output columns (P = [a | g])"""
    return ("edge.h1", B, 1, T, F_, 1, KW, 2 * H1_OUT, 1, 1)


def o1_case(B, T):
    return ("edge.o1", B, 1, T, O1_IN, 1, KW, F_, 1, 1)


def h1_dz_case(B, T):
    """dz = dP . W^T as a 1 x 1 layer of 2 x 128 input and KW * F output columns (weights [256, 360] = W^T)"""
    return ("edge.h1.dz", B, 1, T, 2 * H1_OUT, 1, 1, KW * F_, 1, 1)


def o1_z_case(B, T):
    """z = u . W' as a 1 x 1 layer over the folded weights [256, KW * F]"""
    return ("edge.o1.z", B, 1, T, O1_IN, 1, 1, KW * F_, 1, 1)


def h1_weights(wa, wg):
    """[KW, F, 128] a and g kernels -> the [1, KW, F, 256] weights of h1_case"""
    return np.concatenate([wa, wg], axis=-1)[None]


def h1_dz_weights(wa, wg):
    """the [1, 1, 256, KW * F] weights of h1_dz_case: W^T of the [KW * F, 256] matrix"""
    return np.ascontiguousarray(np.concatenate([wa, wg], axis=-1).reshape(KW * F_, 2 * H1_OUT).T)[None, None]


def o1_z_weights(w):
    """the [1, 1, 256, KW * F] weights of o1_z_case"""
    return np.ascontiguousarray(fold_columns(w))[None, None]
