"""CPU checks of tests/glu_ref.py (the float64 references of the layers without an instance norm and of the loss heads), and the map from
every kernel of csrc/simt_kernels.cu and csrc/tc_gemm.cu to the unit test that reaches it."""
import os
import re

import numpy as np
import torch

import glu_ref as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_glu_backward_is_the_closed_form():
    rng = np.random.default_rng(1)
    P = rng.standard_normal((7, 2 * 12)); dy = rng.standard_normal((7, 12))
    dP, ba, bg = G.glu_backward(P, dy)
    a, g = P[:, :12], P[:, 12:]
    s = 1 / (1 + np.exp(-g))
    want = np.concatenate([dy * s, dy * a * s * (1 - s)], axis=1)
    assert np.allclose(dP.numpy(), want, rtol=1e-13, atol=0)
    assert np.allclose(ba.numpy(), want[:, :12].sum(0)) and np.allclose(bg.numpy(), want[:, 12:].sum(0))


def test_disc_input_p_is_the_tf_same_convolution():
    """a direct loop over TF-'SAME' taps (pad top 1, pad left 0 at an even width with stride 2 and 3 taps)"""
    rng = np.random.default_rng(2)
    B, H, W = 2, 5, 8
    x = rng.standard_normal((B, H, W)); wa = rng.standard_normal((3, 3, 1, 4)); wg = rng.standard_normal((3, 3, 1, 4))
    ba, bg = rng.standard_normal(4), rng.standard_normal(4)
    P = G.disc_input_p(x, wa, wg, ba, bg).numpy().reshape(B, H, W // 2, 8)
    Ho, Wo = G.out_rows(H, W)
    pt, pl = 1, 0
    for b in range(B):
        for yo in range(Ho):
            for xo in range(Wo):
                acc_a, acc_g = ba.copy(), bg.copy()
                for i in range(3):
                    for j in range(3):
                        yy, xx = yo + i - pt, 2 * xo + j - pl
                        if 0 <= yy < H and 0 <= xx < W:
                            acc_a += x[b, yy, xx] * wa[i, j, 0]; acc_g += x[b, yy, xx] * wg[i, j, 0]
                assert np.allclose(P[b, yo, xo], np.concatenate([acc_a, acc_g]), rtol=1e-12, atol=1e-12)


def test_disc_input_backward_matches_finite_differences_and_uses_the_given_p():
    rng = np.random.default_rng(3)
    B, H, W = 1, 4, 6
    x = rng.standard_normal((B, H, W)); wa = rng.standard_normal((3, 3, 1, 2)); wg = rng.standard_normal((3, 3, 1, 2))
    z = np.zeros(2)
    P = G.disc_input_p(x, wa, wg, z, z)
    dy = rng.standard_normal((P.shape[0], 2))
    dwa, dwg, dba, dbg, dx = G.disc_input_backward(x, wa, wg, P, dy)

    def loss(x_, wa_):
        return float((G.glu_forward(G.disc_input_p(x_, wa_, wg, z, z)) * torch.from_numpy(dy)).sum())
    e = 1e-6
    wp = wa.copy(); wp[1, 2, 0, 1] += e; wm = wa.copy(); wm[1, 2, 0, 1] -= e
    assert abs((loss(x, wp) - loss(x, wm)) / (2 * e) - float(dwa[1, 2, 0, 1])) < 1e-7
    xp = x.copy(); xp[0, 2, 3] += e; xm = x.copy(); xm[0, 2, 3] -= e
    assert abs((loss(xp, wa) - loss(xm, wa)) / (2 * e) - float(dx[0, 2, 3])) < 1e-7
    # with another P the GLU's backward follows it, the convolution's stays
    dP2, _, _ = G.glu_backward(P + 1, dy)
    assert np.allclose(G.disc_input_backward(x, wa, wg, P + 1, dy)[2].numpy(), dP2[:, :2].sum(0).numpy())


def test_lattice_cases_are_exact():
    rng = np.random.default_rng(4)
    x, wa, wg, ba, bg = G.lattice_disc_case(rng, 2, 24, 16)
    P = G.disc_input_p(x, wa, wg, ba, bg)
    assert bool((P[:, G.C1:] == 0).all()) and bool((P == P.round()).all())
    dy = G.lattice_disc_dy(rng, P.shape[0])
    assert G.disc_certificate(x, wa, P, dy) < 2 ** 24
    dP, _, _ = G.glu_backward(P, dy)
    assert bool((dP * 4 == (dP * 4).round()).all())
    y, w, b = G.lattice_head_case(rng, 64)
    assert bool((G.head_forward(y, w, b) == 0.5).all())
    Pg, dyg = G.lattice_glu_case(rng, 32, 8)
    assert bool((G.glu_forward(Pg) == torch.from_numpy(Pg[:, :8]).double() / 2).all())


def test_head_loss_backward_is_the_lsgan_gradient():
    rng = np.random.default_rng(5)
    rows = 48
    y = rng.standard_normal((rows, 1024)); w = rng.standard_normal(1024) / 32; b = np.array([0.1])
    prob = G.head_forward(y, w, b)
    for target, coef, gm in ((1.0, 0.5, 1.0), (0.0, 0.5, 8.0), (1.0, 1.0, 1.0)):
        loss, dy, dw, db = G.head_loss_backward(prob, y, w, target, coef, gm)
        p = prob.numpy()
        assert np.isclose(loss, coef * np.mean((p - target) ** 2))
        dz = gm * coef * 2 * (p - target) / rows * p * (1 - p)
        assert np.allclose(dy.numpy(), dz[:, None] * w[None, :]) and np.allclose(dw.numpy(), dz @ y) and np.isclose(float(db), dz.sum())


def test_l1_references():
    yh = np.array([1, -2, 3, 0.5, 7], np.float32); y = np.array([1, 2, -3, 0.25, 7.5], np.float32)
    d = G.l1_grad_bits(yh, y, 10.0, 4.0, np.ones(5, np.float32))
    s = np.float32(np.float32(10.0) * (np.float32(1) / np.float32(5))) * np.float32(4.0)
    assert d.tolist() == [1.0, 1 - s, 1 + s, 1 + s, 1 - s]
    assert np.isclose(G.l1_loss(yh, y), np.mean(np.abs(yh - y)))


def test_chain_lengths_follow_the_launch_grids():
    # bench D-loss shape: M = 786 432 rows -> 768 rows per CTA of 1024 CTAs
    assert G.c1_wgrad_chain(786432) == 768 // 8 + 8 + 1024 + 1
    assert G.c1_wgrad_chain(64) == 8 + 8 + 1 + 1
    assert G.head_chain(48) == 1 + 8 + 6 + 1 and G.head_chain(48 * 512) == 11 + 8 + 296 + 1
    assert G.l1_chain(100) == 1 + 5 + 8 + 1 + 2 and G.l1_chain(592 * 256 * 3 + 77) == 4 + 5 + 8 + 592 + 2
    assert G.post_bias_chain(2, 516) == 4 + 8 + 2 * 17 + 1


# ---- which unit test reaches each kernel -----------------------------------------------------------------------------------------
REACHED = {
    "gg_simt_kernel": "test_gpu_kernels.py", "wgrad_simt_kernel": "test_gpu_kernels.py",
    "colsum_kernel": "test_gpu_kernels.py", "reduce_parts_kernel": "test_gpu_deterministic.py",
    "post_stats_kernel": "test_gpu_norm_layers.py",
    "post_apply_fwd_kernel": "test_gpu_norm_layers.py / test_gpu_glu_layers.py (GLU-only form)",
    "post_bwd_sums_kernel": "test_gpu_norm_layers.py",
    "post_apply_bwd_kernel": "test_gpu_norm_layers.py / test_gpu_glu_layers.py (GLU-only form)",
    "post_bwd_onepass_kernel": "test_gpu_norm_layers.py", "post_fwd_stream_kernel": "test_gpu_norm_layers.py",
    "post_bwd_stream_kernel": "test_gpu_norm_layers.py",
    "head_fwd_kernel": "test_gpu_glu_layers.py", "head_loss_bwd_kernel": "test_gpu_glu_layers.py", "l1_loss_grad_kernel": "test_gpu_glu_layers.py",
    "wgrad_c1_kernel": "test_gpu_glu_layers.py", "gather_taps_kernel": "test_gpu_glu_layers.py", "glu_bwd_wgrad_c1_kernel": "test_gpu_glu_layers.py",
    "glu_bwd_proj_c1_kernel": "test_gpu_glu_layers.py", "proj_taps_kernel": "test_gpu_glu_layers.py", "conv_c1_fwd_kernel": "test_gpu_glu_layers.py",
    "conv_c1_glu_fwd_kernel": "test_gpu_glu_layers.py", "pad_split_q_kernel": "test_gpu_planes.py", "pad_split_kernel": "test_gpu_planes.py",
    "im2col_taps_kernel": "test_gpu_planes.py", "col2im_taps_kernel": "test_gpu_edge_layers.py",
    "check_finite_kernel": "test_gpu_loss_scale.py", "loss_scale_update_kernel": "test_gpu_loss_scale.py",
}
# kernels checked only through whole-model tests against the oracle, with the reason no unit tier is needed
EXEMPT = {
    "transpose_ft_kernel": "a pure permutation: every generator forward against the oracle would show a wrong element",
    "transpose_packed_kernel": "a pure permutation: the packed conversions equal the per-utterance ones bitwise (test_packed_forward.py)",
    "add_kernel": "one fp32 add per element, in every train step against the oracle",
    "adam_kernel": "elementwise TF Adam, checked against the oracle's Adam by the trajectory tests",
    "finalize_losses_kernel": "scalar algebra of 8 losses, compared with the oracle's losses every step",
    "split_bf16_kernel": "the bf16 split of the weight planes, exercised by every bf16x3 GEMM test",
    "set_scalars_kernel": "copies up to 6 kernel arguments into device scalars",
    "sample_plan_kernel": "integer index arithmetic, mirrored on the host by cgvc.preprocess.counter_sample_plan (test_train_driver.py)",
    "gather_minibatch_kernel": "a copy of the crops the plan names (test_train_driver.py)",
    "scale_kernel": "one product per element (Adam's grad_scale path), in every train step against the oracle",
}


# the same for csrc/tc_gemm.cu
REACHED_TC = {
    "tc_gg_nt_kernel": "test_gpu_gemm_exact.py", "tc_gg_tn_kernel": "test_gpu_gemm_exact.py",
    "prep_weights_kernel": "test_gpu_weight_planes.py", "copy_bias_kernel": "test_gpu_weight_planes.py",
    "prep_weights_q_kernel": "test_gpu_weight_planes.py (prep_batched 0)", "prep_weights_qd_kernel": "test_gpu_weight_planes.py (prep_batched 0)",
    "prep_weights_q_all_kernel": "test_gpu_weight_planes.py",
}


def _kernels(source):
    src = open(os.path.join(ROOT, "voice-converter-cyclegan_b200", "csrc", source)).read()
    return set(re.findall(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\([^)]*\)\s*)?(?:void\s+)?(\w+)\s*\(", src))


def _audit(names, reached, exempt):
    missing = sorted(n for n in names if n not in reached and n not in exempt)
    assert not missing, "kernels with neither a unit test nor an exemption: %s" % missing
    stale = sorted(n for n in list(reached) + list(exempt) if n not in names)
    assert not stale, "entries for kernels that no longer exist: %s" % stale
    for n, where in reached.items():
        f = where.split(" ")[0]
        assert os.path.exists(os.path.join(ROOT, "tests", f)), (n, f)


def test_every_kernel_has_a_unit_test_or_an_exemption():
    names = _kernels("simt_kernels.cu")
    assert len(names) > 20, sorted(names)
    _audit(names, REACHED, EXEMPT)


def test_every_tensor_core_kernel_has_a_unit_test():
    names = _kernels("tc_gemm.cu")
    assert len(names) >= 7, sorted(names)
    _audit(names, REACHED_TC, {})
