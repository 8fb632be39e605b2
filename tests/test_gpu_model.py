"""GPU parity of the hot path through the reference-facing API (cgvc.CycleGAN -> C ABI -> CUDA) against the CPU
oracle in float64, on identical injected weights and inputs.

Tolerance (BASELINE.json north_star): 1e-3 relative on generator activations and losses.  Gradients and
post-Adam weights are held to the same bound (relative L2 per tensor).
"""
import math

import numpy as np
import pytest
import torch

from parity_util import rel_l2, rel_max

pytestmark = pytest.mark.gpu

TOL = 1e-3
PRECISIONS = ["fp32", "bf16x3", "f16f8"]


@pytest.fixture(scope="module")
def models(oracle_params64):
    import cgvc
    out = {}
    for prec in PRECISIONS:
        m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision=prec, log_dir='/tmp/cgvc_log')
        m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
        m.set_debug_taps(True)
        out[prec] = m
    return out


def test_param_table_matches_oracle(models):
    from oracle import cyclegan_oracle as O
    m = models["fp32"]
    specs = O.param_specs()
    assert m.param_names() == [n for n, _, _ in specs]
    off = total = 0
    for n, shp, _ in specs:
        off = (off + 3) // 4 * 4          # the engine starts every tensor on a 16-byte boundary
        assert m._table[n] == (off, tuple(shp)), n
        off += int(np.prod(shp)); total += int(np.prod(shp))
    assert total == m.n_params == 119787058


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("frames", [128, 64, 36, 516, 784, 1400])
def test_generator_forward_activations(models, oracle_params64, prec, frames):
    from oracle import cyclegan_oracle as O
    m = models[prec]
    A, _ = O.synthetic_batch(seed=7, batch=2, frames=frames, dtype=torch.float64)
    taps = {}
    y_ref = O.generator_forward(A, oracle_params64, "generator_A2B", taps)
    y = m.test(A.numpy(), 'A2B')
    assert y.shape == (2, 24, frames) and y.dtype == np.float32
    worst = 0.0
    for name in ["h1_glu", "d1", "d2", "r1", "r2", "r3", "r4", "r5", "r6", "u1", "u2"]:
        got = m.debug_activation(name)
        ref = taps[name].numpy().reshape(-1)
        e = rel_l2(got, ref); worst = max(worst, e)
        print("gen[%s,T=%d] %-6s rel_l2=%.2e rel_max=%.2e" % (prec, frames, name, e, rel_max(got, ref)))
        assert e < TOL, (name, e)
    e = rel_l2(y, y_ref.numpy())
    print("gen[%s,T=%d] out    rel_l2=%.2e" % (prec, frames, e))
    assert e < TOL
    # B2A uses the other generator's weights
    y2 = m.test(A.numpy(), 'B2A')
    assert rel_l2(y2, O.generator_forward(A, oracle_params64, "generator_B2A").numpy()) < TOL


@pytest.mark.parametrize("prec", PRECISIONS)
def test_generator_forward_T516_golden(models, prec):
    """The committed float64 golden vector of a 516-frame utterance (tests/golden/make_golden.py): real utterances are 400-1400
    frames, where samples do not tile the 128-row GEMM tiles (statistics through the two-phase kernels, im2col loads that cross
    sample boundaries mid-tile)."""
    import os
    from oracle import cyclegan_oracle as O
    Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cyclegan_golden.npz"))
    A516, _ = O.synthetic_batch(seed=int(Z["seed_x"]) + 1, batch=1, frames=516, dtype=torch.float64)
    y = models[prec].test(A516.numpy(), 'B2A')
    e = rel_l2(y, Z["gen_B2A_out_T516"])
    print("gen[%s,T=516] vs golden rel_l2=%.2e" % (prec, e))
    assert y.shape == (1, 24, 516) and e < TOL


@pytest.mark.parametrize("prec", PRECISIONS)
def test_discriminator_forward(models, oracle_params64, prec):
    from oracle import cyclegan_oracle as O
    m = models[prec]
    A, B = O.synthetic_batch(seed=8, batch=2, frames=128, dtype=torch.float64)
    for which, x in (("A", A), ("B", B)):
        taps = {}
        ref = O.discriminator_forward(x, oracle_params64, "discriminator_" + which, taps)
        got = m.discriminate(x.numpy(), which)
        assert got.shape == (2, 6, 8, 1)
        for name in ["h1_glu", "d1", "d2", "d3"]:
            e = rel_l2(m.debug_activation(name), taps[name].numpy().reshape(-1))
            print("disc[%s] %-6s rel_l2=%.2e" % (prec, name, e))
            assert e < TOL, (name, e)
        assert rel_l2(got, ref.numpy()) < TOL


@pytest.mark.parametrize("frames", [128, 64, 36])
def test_generator_forward_f16f8(oracle_params64, frames):
    """The 2-MMA-unit precision (CGVC_PREC_F16F8) on an inference engine (nothing kept for backward): every generator layer boundary
    and the output within the north-star tolerance of the float64 oracle, also after a 58-convolution cycle."""
    import cgvc
    from oracle import cyclegan_oracle as O
    m = cgvc.CycleGAN(num_features=24, mode='test', max_batch=2, max_frames=128, precision="f16f8")
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    m.set_debug_taps(True)
    A, _ = O.synthetic_batch(seed=7, batch=2, frames=frames, dtype=torch.float64)
    taps = {}
    y_ref = O.generator_forward(A, oracle_params64, "generator_A2B", taps)
    y = m.test(A.numpy(), 'A2B')
    for name in ["h1_glu", "d1", "d2", "r1", "r2", "r3", "r4", "r5", "r6", "u1", "u2"]:
        e = rel_l2(m.debug_activation(name), taps[name].numpy().reshape(-1))
        print("gen[f16f8,T=%d] %-6s rel_l2=%.2e" % (frames, name, e))
        assert e < TOL, (name, e)
    e = rel_l2(y, y_ref.numpy())
    print("gen[f16f8,T=%d] out    rel_l2=%.2e" % (frames, e))
    assert e < TOL
    # a cycle (A2B then B2A: 58 convolutions deep) stays inside the tolerance too
    y2 = m.test(y, 'B2A')
    e2 = rel_l2(y2, O.generator_forward(y_ref, oracle_params64, "generator_B2A").numpy())
    print("gen[f16f8,T=%d] cycle  rel_l2=%.2e" % (frames, e2))
    assert e2 < TOL
    d = m.discriminate(A.numpy()[:, :, :frames // 16 * 16], 'A') if frames % 16 == 0 else None
    if d is not None:
        assert rel_l2(d, O.discriminator_forward(A[:, :, :frames // 16 * 16], oracle_params64, "discriminator_A").numpy()) < TOL



def test_network_operators_are_callable_with_variable_scopes(oracle_params64):
    """module.py:148-213 as eager operators: `generator_gatedcnn(x, reuse, scope_name)` / `discriminator(...)` run the native
    networks with per-scope variables (created on first use, reused with reuse=True, TF's errors otherwise), and CycleGAN takes
    any descriptor with the engine's architecture and refuses others."""
    import copy
    import cgvc
    from cgvc import module as M
    from oracle import cyclegan_oracle as O
    M.reset_default_graph()
    A, _ = O.synthetic_batch(seed=12, batch=2, frames=64, dtype=torch.float64)
    y0 = M.generator_gatedcnn(A.numpy(), reuse=False, scope_name="gen_x")
    assert y0.shape == (2, 24, 64) and np.isfinite(y0).all()
    with pytest.raises(ValueError, match="already exists"):
        M.generator_gatedcnn(A.numpy(), reuse=False, scope_name="gen_x")
    with pytest.raises(ValueError, match="does not exist"):
        M.generator_gatedcnn(A.numpy(), reuse=True, scope_name="gen_never_made")
    assert np.array_equal(M.generator_gatedcnn(A.numpy(), reuse=True, scope_name="gen_x"), y0)
    # a second and a third scope get their own variables (the third one lives in a second engine)
    y1 = M.generator_gatedcnn(A.numpy(), scope_name="gen_y"); y2 = M.generator_gatedcnn(A.numpy(), scope_name="gen_z")
    assert not np.array_equal(y0, y1) and not np.array_equal(y1, y2)
    # injected variables: the operator reproduces the oracle network
    names = [n for n, _ in M.generator_gatedcnn.variables(24)]
    assert list(M.scope_variables("gen_y").keys()) == ["gen_y/" + n for n in names]
    M.assign_scope_variables("gen_y", {n: oracle_params64["generator_B2A/" + n].numpy() for n in names})
    ref = O.generator_forward(A, oracle_params64, "generator_B2A").numpy()
    assert rel_l2(M.generator_gatedcnn(A.numpy(), reuse=True, scope_name="gen_y"), ref) < TOL
    assert np.array_equal(M.generator_gatedcnn(A.numpy(), reuse=True, scope_name="gen_x"), y0)      # other scopes untouched
    dn = [n for n, _ in M.discriminator.variables()]
    d0 = M.discriminator(A.numpy(), scope_name="disc_x")
    assert d0.shape == (2, 6, 4, 1)
    M.assign_scope_variables("disc_x", {n: oracle_params64["discriminator_A/" + n].numpy() for n in dn})
    assert rel_l2(M.discriminator(A.numpy(), reuse=True, scope_name="disc_x"), O.discriminator_forward(A, oracle_params64, "discriminator_A").numpy()) < TOL
    with pytest.raises(ValueError, match="holds a generator"):
        M.discriminator(A.numpy(), reuse=True, scope_name="gen_x")
    M.reset_default_graph()
    # the model class: an equal descriptor is accepted, a different architecture or a non-descriptor refused
    m = cgvc.CycleGAN(num_features=24, mode='test', generator=copy.deepcopy(M.generator_gatedcnn), discriminator=copy.deepcopy(M.discriminator))
    assert m.test(A.numpy(), 'A2B').shape == (2, 24, 64)
    other = copy.deepcopy(M.generator_gatedcnn)
    other.layers = other.layers[:-1] + [("conv", "o1_conv", 5, 1, None)]
    with pytest.raises(ValueError, match="o1_conv/kernel"):
        cgvc.CycleGAN(num_features=24, mode='test', generator=other)
    with pytest.raises(TypeError):
        cgvc.CycleGAN(num_features=24, mode='test', generator=lambda x: x)


def test_direction_error(models):
    with pytest.raises(Exception, match="Conversion direction must be specified."):
        models["fp32"].test(np.zeros((1, 24, 128)), 'A2C')


@pytest.fixture(scope="module")
def oracle_grads(oracle_params64):
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=9, batch=2, frames=128, dtype=torch.float64)
    L, G, gA, gB = O.gradients(A, B, oracle_params64, 10.0, 5.0)
    return A, B, L, G, gA, gB


@pytest.mark.parametrize("prec", PRECISIONS)
def test_losses_and_gradients(models, oracle_grads, prec):
    m = models[prec]
    A, B, L, G, gA, gB = oracle_grads
    losses, genA, genB = m.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
    for k, v in L.items():
        e = abs(losses[k] - float(v)) / abs(float(v))
        print("loss[%s] %-22s got=%.6f ref=%.6f rel=%.2e" % (prec, k, losses[k], float(v), e))
        assert e < TOL, (k, e)
    assert rel_l2(genA, gA.numpy()) < TOL and rel_l2(genB, gB.numpy()) < TOL
    grads = m.get_grads()
    worst = []
    for name, g_ref in G.items():
        g_ref = g_ref.numpy()
        ref_norm = np.linalg.norm(g_ref.ravel())
        e = np.linalg.norm((grads[name].astype(np.float64) - g_ref).ravel()) / (ref_norm + 1e-30)
        # conv biases feeding an instance norm have an analytically zero gradient: compare those absolutely
        if ref_norm < 1e-9:
            e = np.abs(grads[name]).max()
            assert e < 1e-5, (name, e)
            continue
        worst.append((e, name))
        assert e < TOL, (name, e)
    worst.sort(reverse=True)
    print("grads[%s] worst:" % prec, ["%s %.2e" % (n, e) for e, n in worst[:6]])


def test_weight_gradient_precisions_of_f16f8_match_oracle(models, oracle_grads):
    """F16F8 weight-gradient GEMMs read the fp16 planes alone by default (option `wgrad_f16` = 1: 1 MMA unit per product instead of 2).
    A weight gradient is a leaf of the graph -- its rounding error (<= 4e-4 relative L2 per tensor for random-sign sums) is not
    propagated anywhere -- so all 280 tensors stay inside the same 1e-3 of the float64 oracle (test_losses_and_gradients checks the
    default); here both forms side by side: the 2-unit form (`wgrad_f16` = 0) is tighter, and losses, generated batches and data
    gradients do not depend on the option at all."""
    m = models["f16f8"]
    lib, h = m._lib, m._handle
    A, B, L, G, gA, gB = oracle_grads
    res = {}
    try:
        for w16 in (1, 0):
            assert lib.cgvc_set_option(h, b"wgrad_f16", w16) == 0
            l, a, b = m.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
            res[w16] = (l, a, b, m.get_grads())
    finally:
        assert lib.cgvc_set_option(h, b"wgrad_f16", 1) == 0
    (l1, a1, b1, g1), (l0, a0, b0, g0) = res[1], res[0]
    assert all(abs(l1[k] - l0[k]) <= 1e-6 * abs(l0[k]) for k in l0) and np.array_equal(a0, a1) and np.array_equal(b0, b1)
    rows = []
    for name, g_ref in G.items():
        g_ref = g_ref.numpy(); n = np.linalg.norm(g_ref.ravel())
        if n < 1e-9:
            continue
        e1 = np.linalg.norm((g1[name].astype(np.float64) - g_ref).ravel()) / n
        e0 = np.linalg.norm((g0[name].astype(np.float64) - g_ref).ravel()) / n
        rows.append((e1, e0, name))
        assert e1 < TOL and e0 < TOL, (name, e1, e0)
    rows.sort(reverse=True)
    med = lambda i: sorted(r[i] for r in rows)[len(rows) // 2]
    print("f16f8 gradients vs oracle, wgrad_f16=1 / 0: worst %.2e (%s; %.2e with the 2-unit form), worst of the 2-unit form %.2e, medians %.2e / %.2e"
          % (rows[0][0], rows[0][2], rows[0][1], max(r[1] for r in rows), med(0), med(1)))
    assert max(r[1] for r in rows) < 2.5e-4 and rows[0][0] < 6e-4


def _b64_picks():
    picks = []
    for net in ("generator_A2B", "generator_B2A"):
        picks += [net + "/" + n for n in ("h1_conv/kernel", "h1_conv_gates/bias", "downsample1d_block2_h1_gates/kernel", "InstanceNorm_3/gamma",
                                          "residual1d_block1_h1_conv/kernel", "residual1d_block6_h2_conv/kernel", "InstanceNorm_20/beta",
                                          "upsample1d_block1_h1_conv/kernel", "upsample1d_block2_h1_gates/kernel", "o1_conv/kernel", "o1_conv/bias")]
    for net in ("discriminator_A", "discriminator_B"):
        picks += [net + "/" + n for n in ("h1_conv/kernel", "downsample2d_block1_h1_conv/kernel", "downsample2d_block3_h1_gates/kernel", "InstanceNorm_4/gamma",
                                          "dense/kernel", "dense/bias")]
    return picks


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
@pytest.mark.parametrize("lambdas", [(0.0, 0.0), (10.0, 5.0)])
def test_batch64_losses_and_gradients_match_oracle(lambdas, prec):
    """BASELINE.json configs[1]: the full step at batch 64 -- the 8 losses, both generated batches and 34 gradient tensors spread
    over all four networks against the CPU oracle (float64 autograd) on the same 64 samples.

    The L1 cycle / identity terms have the gradient sign(x_hat - x) / N, which is discontinuous in the forward pass: an element whose
    |x_hat - x| is below the forward error (~1e-5) may get the other sign in ANY implementation that is not bit-identical to the
    oracle, and flipping k of the N signs changes the upstream gradient by 2 sqrt(k / N) relative -- 7e-3 for the ~9 such elements
    expected among the 786 432 of a batch-64 step, however exact the kernels are (at batch 2 the expectation is 0.3 elements, which
    is why test_losses_and_gradients can ask for 1e-3).  So the generator gradients are checked twice: with lambda_cycle =
    lambda_identity = 0 (only the smooth adversarial term; also the identity-off code path of train.py:98-99) to 1e-3, and with the
    reference's lambdas to 1e-3 plus the bound for the elements the oracle itself finds within 2e-4 of a sign change."""
    import cgvc
    from oracle import cyclegan_oracle as O
    lam_c, lam_i = lambdas
    P = O.init_params(seed=4321, dtype=torch.float64, perturb_affine=True)
    A, B = O.synthetic_batch(seed=64, batch=64, frames=128, dtype=torch.float64)
    Pg = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    taps = {}
    L, gA, gB = O.losses(A, B, Pg, lam_c, lam_i, taps)
    gnames = [k for k in Pg if "generator" in k]; dnames = [k for k in Pg if "discriminator" in k]
    gg = torch.autograd.grad(L["generator_loss"], [Pg[k] for k in gnames], retain_graph=True)
    dg = torch.autograd.grad(L["discriminator_loss"], [Pg[k] for k in dnames])
    G = dict(zip(gnames + dnames, list(gg) + list(dg)))
    near = sum(int(((taps[k].detach() - x).abs() < 2e-4).sum()) for k, x in (("cycle_A", A), ("cycle_B", B), ("id_A", A), ("id_B", B)))
    n_l1 = 4 * A.numel()
    flip_bound = 2.0 * math.sqrt(near / n_l1) if (lam_c or lam_i) else 0.0
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=64, max_frames=128, precision=prec, log_dir='/tmp/cgvc_log')
    m.set_params({k: v.numpy() for k, v in P.items()})
    losses, genA, genB = m.compute_gradients(A.numpy(), B.numpy(), lam_c, lam_i)
    for k, v in L.items():
        e = abs(losses[k] - float(v)) / abs(float(v))
        print("loss[B=64,%s,lam=%g/%g] %-22s got=%.6f ref=%.6f rel=%.2e" % (prec, lam_c, lam_i, k, losses[k], float(v), e))
        assert e < TOL, (k, e)
    assert rel_l2(genA, gA.detach().numpy()) < TOL and rel_l2(genB, gB.detach().numpy()) < TOL
    grads = m.get_grads()
    errs = []
    for name in _b64_picks():
        g_ref = G[name].detach().numpy().astype(np.float64)
        e = np.linalg.norm((grads[name].astype(np.float64) - g_ref).ravel()) / (np.linalg.norm(g_ref.ravel()) + 1e-30)
        errs.append((e, name))
    worst_g = max(x for x in errs if "generator" in x[1]); worst_d = max(x for x in errs if "discriminator" in x[1])
    print("grads[B=64," + prec + ",lam=%g/%g]: generators worst %.2e (%s), discriminators worst %.2e (%s); %d of %d L1 elements within 2e-4 of a sign "
          "change -> bound 1e-3 + %.2e" % (lam_c, lam_i, worst_g[0], worst_g[1], worst_d[0], worst_d[1], near, n_l1, flip_bound))
    for e, name in errs:
        assert e < TOL + (flip_bound if "generator" in name else 0.0), (name, e)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_train_steps_match_oracle(oracle_params64, prec):
    """Two full train() calls (G step + D step + 2x Adam) track the oracle: returned losses and updated weights."""
    import cgvc
    from oracle import cyclegan_oracle as O
    P = {k: v.clone() for k, v in oracle_params64.items()}
    ref = O.OracleCycleGAN(dtype=torch.float64, params=P)
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=1, max_frames=128, precision=prec, log_dir='/tmp/cgvc_log')
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    before = m.get_params()
    for step in range(2):
        A, B = O.synthetic_batch(seed=20 + step, batch=1, frames=128, dtype=torch.float64)
        lam_id = 5.0 if step == 0 else 0.0            # train.py:98-99 switches identity off later: exercise both
        g_ref, d_ref = ref.train(A.numpy(), B.numpy(), 10.0, lam_id, 2e-4, 1e-4)
        g, d = m.train(A.numpy(), B.numpy(), 10.0, lam_id, 2e-4, 1e-4)
        assert g.dtype == np.float32 and d.dtype == np.float32
        print("step %d [%s] G %.5f/%.5f D %.5f/%.5f" % (step, prec, g, g_ref, d, d_ref))
        assert abs(g - g_ref) / abs(g_ref) < TOL and abs(d - d_ref) / abs(d_ref) < TOL
        # identity loss is still reported when its weight is 0 (model.py:157)
        assert m.last_losses["identity_loss"] > 0
    after = m.get_params()
    assert m.train_step == 2
    worst = 0.0
    for name in after:
        delta_ref = ref.P[name].numpy() - before[name]
        delta = after[name].astype(np.float64) - before[name]
        if np.abs(delta_ref).max() == 0:
            continue
        # Adam's first steps move every weight by ~lr regardless of gradient scale; compare the update itself
        e = np.linalg.norm((delta - delta_ref).ravel()) / np.linalg.norm(delta_ref.ravel())
        worst = max(worst, e)
        if "bias" in name and "block" in name:
            continue   # conv biases feeding an instance norm: zero gradient, Adam moves them by sign(noise) * lr
        # Adam's first two steps are sign descent: an element whose gradient sign differs from the oracle's (|g| within the gradient
        # error of zero) moves the opposite way, 2 * lr off.  One such element in a 128-element bias vector is already
        # 2 / sqrt(128) = 0.18 of that tensor's update; the large tensors average it out (measured 0.02 ... 0.06)
        assert e < (0.1 if after[name].size >= 4096 else 0.3), (name, e)
    print("train[%s]: worst relative error of the 2-step weight update: %.3e" % (prec, worst))


def test_save_load_roundtrip(models, tmp_path):
    import cgvc
    m = models["fp32"]
    path = m.save(str(tmp_path / "ckpt"), "model.ckpt")
    assert path == str(tmp_path / "ckpt" / "model.ckpt")
    m2 = cgvc.CycleGAN(num_features=24, mode='test', max_batch=1, max_frames=128, precision="fp32")
    m2.load(path)
    x = np.random.RandomState(0).randn(1, 24, 128)
    assert np.array_equal(m.test(x, 'A2B'), m2.test(x, 'A2B'))


# ---------------------------------------------------------------------------------------------------------------
# BASELINE.json's full sizes (batch 256 x [24,128]; inference batch 1024), through size-independent properties
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["bf16x3", "f16f8"])
def big_model(request, oracle_params64):
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=256, max_frames=128, precision=request.param, log_dir='/tmp/cgvc_log')
    m.set_params({k: v.numpy() for k, v in oracle_params64.items()})
    return m


def test_full_size_forward_is_per_sample(big_model, oracle_params64):
    """Instance norm is per sample (module.py:9-20): row i of a 512-sample generator forward equals the oracle run on
    that sample alone (convert.py path).  512 samples: a forward of this size on the batch-256 training engine grows its work
    arena to ~44 GB, which fits an 80 GB H100 next to the training arenas (1024 would need ~88 GB)."""
    from oracle import cyclegan_oracle as O
    A, _ = O.synthetic_batch(seed=31, batch=512, frames=128, dtype=torch.float32)
    y = big_model.test(A.numpy(), 'A2B')
    assert y.shape == (512, 24, 128)
    for i in (0, 317, 511):
        with torch.no_grad():
            ref = O.generator_forward(A[i:i + 1].double(), oracle_params64, "generator_A2B").numpy()
        assert rel_l2(y[i:i + 1], ref) < TOL, i
    assert np.isfinite(y).all()


def test_full_size_gradients_are_batch_means(big_model):
    """Every loss is a batch mean and no op mixes samples (SURVEY.md 8e): the batch-256 gradients equal the average of the
    two half-batch gradients, and the losses likewise.  Checks the full-size step without needing the CPU oracle."""
    from oracle import cyclegan_oracle as O
    A, B = O.synthetic_batch(seed=32, batch=256, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    L, _, _ = big_model.compute_gradients(A, B, 10.0, 5.0)
    g_full = big_model.get_grads()
    L1, _, _ = big_model.compute_gradients(A[:128], B[:128], 10.0, 5.0)
    g1 = big_model.get_grads()
    L2, _, _ = big_model.compute_gradients(A[128:], B[128:], 10.0, 5.0)
    g2 = big_model.get_grads()
    for k in L:
        assert abs(L[k] - 0.5 * (L1[k] + L2[k])) / abs(L[k]) < 1e-5, k
    worst = 0.0
    for name in g_full:
        if "bias" in name and "block" in name and "upsample" not in name:
            continue          # conv bias in front of an instance norm: analytically zero gradient, only rounding noise
        ref = 0.5 * (g1[name].astype(np.float64) + g2[name])
        n = np.linalg.norm(ref.ravel())
        if n < 1e-9:
            continue
        e = np.linalg.norm((g_full[name] - ref).ravel()) / n
        worst = max(worst, e)
        assert e < 2e-4, (name, e)
    print("full-size gradient linearity: worst rel. diff %.2e" % worst)


def test_forward_is_deterministic(big_model):
    x = np.random.RandomState(5).randn(64, 24, 128)
    assert np.array_equal(big_model.test(x, 'B2A'), big_model.test(x, 'B2A'))


def test_fused_epilogue_matches_unfused(big_model):
    """The instance-norm epilogue fused into the forward conv kernel (generator layers with whole samples per tile) and the
    separate streaming kernels are two implementations of module.py:9-20,85-98: same activations, same gradients."""
    from oracle import cyclegan_oracle as O
    big_model.set_debug_taps(True)
    lib, h = big_model._lib, big_model._handle
    A, B = O.synthetic_batch(seed=41, batch=8, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    out = {}
    for flag in (1, 0):
        assert lib.cgvc_set_option(h, b"fuse_in", flag) == 0
        y = big_model.test(A, 'A2B')
        taps = {k: big_model.debug_activation(k) for k in ("d1", "d2", "r1", "r6", "u2")}
        # (f16f8: the two paths differ by ~2e-5 in the forward pass, enough to flip the sign of an L1 gradient element or two, which
        #  moves every generator gradient by ~7e-3 -- see test_batch64_losses_and_gradients_match_oracle; compare on the smooth loss)
        lam = (0.0, 0.0) if big_model.precision == "f16f8" else (10.0, 5.0)
        L, _, _ = big_model.compute_gradients(A, B, *lam)
        out[flag] = (y, taps, L, big_model.get_grads())
    lib.cgvc_set_option(h, b"fuse_in", 1)
    big_model.set_debug_taps(False)
    # two fp32 evaluation orders of the same layer; in f16f8 the results are re-quantised into fp16 + e4m3 planes layer by layer, so
    # last-bit differences propagate at the plane resolution (both paths stay within 5e-5 of the oracle)
    tol = 1e-4 if big_model.precision == "f16f8" else 2e-5
    assert rel_l2(out[1][0], out[0][0]) < tol
    for k in out[1][1]:
        assert rel_l2(out[1][1][k], out[0][1][k]) < tol, k
    for k in out[1][2]:
        assert abs(out[1][2][k] - out[0][2][k]) / abs(out[0][2][k]) < tol, k
    for k in ("generator_A2B/residual1d_block3_h1_conv/kernel", "generator_B2A/downsample1d_block1_h1_gates/kernel", "generator_A2B/InstanceNorm_6/gamma"):
        assert rel_l2(out[1][3][k], out[0][3][k]) < 2e-4, k


def test_edge_layer_tap_lowering_matches_tap_gemm(big_model):
    """The generator's 15-tap, 24-channel edge layers (module.py:85-86 h1, module.py:148 o1) as dense 1 x 1 GEMMs over an im2col of the
    24-channel side (`edge_lower` = 1, default: h1 with K = 15 * 24, o1 with its taps folded into 15 * 24 output columns + the tap-shifted
    sum) against the 15-tap gather-GEMMs (`edge_lower` = 0): same activations, same losses, same gradients -- forward, data gradient
    (through the cycle passes) and weight gradient of both layers."""
    from oracle import cyclegan_oracle as O
    big_model.set_debug_taps(True)
    lib, h = big_model._lib, big_model._handle
    A, B = O.synthetic_batch(seed=45, batch=6, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    tol = 1e-4 if big_model.precision == "f16f8" else 2e-5
    out = {}
    for flag in (1, 0):
        assert lib.cgvc_set_option(h, b"edge_lower", flag) == 0
        y = big_model.test(A, 'B2A')
        taps = {k: big_model.debug_activation(k) for k in ("h1_glu", "d1", "u2", "out_cl")}
        # the smooth losses only (lambda = 0): adversarial gradients through both generators' first passes ...
        L0, gA, gB = big_model.compute_gradients(A, B, 0.0, 0.0)
        g0 = big_model.get_grads()
        # ... and the full objective, whose cycle terms also drive the data gradient of h1 (cycle passes).  The L1 terms' sign(x^ - x)
        # flips for an element whose difference is within the forward tolerance of zero, and ONE flip among the N elements of a term
        # moves every upstream gradient by 2 / sqrt(N) (1.5e-2 here; see test_batch64_losses_and_gradients_match_oracle): count the flips
        L1, gA1, gB1 = big_model.compute_gradients(A, B, 10.0, 5.0)
        g1 = big_model.get_grads()
        pairs = ((big_model.test(gB1, 'B2A'), A), (big_model.test(gA1, 'A2B'), B), (big_model.test(A, 'B2A'), A), (big_model.test(B, 'A2B'), B))
        signs = [np.sign(p - q) for p, q in pairs]
        out[flag] = (y, taps, L0, g0, gA, gB, L1, g1, signs)
    lib.cgvc_set_option(h, b"edge_lower", 1)
    big_model.set_debug_taps(False)
    assert rel_l2(out[1][0], out[0][0]) < tol
    for k in out[1][1]:
        assert rel_l2(out[1][1][k], out[0][1][k]) < tol, k
    for idx in (2, 6):
        for k in out[1][idx]:
            assert abs(out[1][idx][k] - out[0][idx][k]) / abs(out[0][idx][k]) < tol, (idx, k)
    assert rel_l2(out[1][4], out[0][4]) < tol and rel_l2(out[1][5], out[0][5]) < tol
    near = sum(int((s1 != s0).sum()) for s1, s0 in zip(out[1][8], out[0][8]))      # L1 elements whose sign differs between the two runs
    flip_bound = 3.0 * np.sqrt(near / float(A.size))
    keys = ("generator_A2B/h1_conv/kernel", "generator_A2B/h1_conv_gates/kernel", "generator_B2A/h1_conv/kernel", "generator_B2A/h1_conv_gates/bias",
            "generator_A2B/o1_conv/kernel", "generator_B2A/o1_conv/kernel", "generator_A2B/o1_conv/bias",
            "generator_A2B/residual1d_block3_h1_conv/kernel", "generator_B2A/upsample1d_block2_h1_gates/kernel", "generator_A2B/InstanceNorm_6/gamma")
    worst = [(0.0, ""), (0.0, "")]
    # (f16f8: the two paths round different intermediate sums into the fp16 + e4m3 planes; each stays within 3.6e-4 of the oracle)
    gtol = 6e-4 if big_model.precision == "f16f8" else 2e-4
    for i, (idx, bound) in enumerate(((3, gtol), (7, gtol + flip_bound))):
        for k in keys:
            e = rel_l2(out[1][idx][k], out[0][idx][k])
            worst[i] = max(worst[i], (e, k))
            assert e < bound, (idx, k, e, near)
    print("edge_lower 1 vs 0 (%s): worst gradient rel. diff, smooth loss %.2e (%s); full objective %.2e (%s), %d L1 sign flips between the runs"
          % (big_model.precision, worst[0][0], worst[0][1], worst[1][0], worst[1][1], near))


def test_batched_weight_planes_match_per_layer_kernels(oracle_params64):
    """F16F8 weight planes (fp16 + two e4m3 planes, forward and data-gradient layouts, gate-interleaved / pixel-shuffle / tap-folded row
    orders, biases) built by the one-launch job-table kernel (`prep_batched` = 1, default) against the per-layer kernels: the planes are
    meant to be bit-identical, so the (deterministic) forward passes must be bit-identical and the gradients equal up to the order of
    their atomics."""
    import cgvc
    from oracle import cyclegan_oracle as O
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=4, max_frames=128, precision="f16f8", seed=3, log_dir='/tmp/cgvc_log')
    P = {k: v.numpy() for k, v in oracle_params64.items()}
    A, B = O.synthetic_batch(seed=61, batch=4, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    out = {}
    for flag in (0, 1):
        m.set_option("prep_batched", flag)
        m.set_params(P)                                   # rebuilds every plane with the selected kernels
        yA, yB = m.test(A, 'A2B'), m.test(B, 'B2A')
        dA = m.discriminate(A, 'A')
        L, gA, gB = m.compute_gradients(A, B, 10.0, 5.0)
        out[flag] = (yA, yB, dA, L, gA, gB, m.get_grads())
    m.set_option("prep_batched", 1)
    for i in (0, 1, 2, 4, 5):
        assert np.array_equal(out[1][i], out[0][i]), i
    for k in out[1][3]:
        assert abs(out[1][3][k] - out[0][3][k]) <= 2e-6 * abs(out[0][3][k]), k
    for k, g0 in out[0][6].items():
        n0 = np.linalg.norm(g0.astype(np.float64).ravel())
        if n0 > 1e-6:
            assert np.linalg.norm((out[1][6][k].astype(np.float64) - g0).ravel()) / n0 < 2e-5, k


def test_side_stream_weight_gradients_and_kernel_variants_match_default_path(big_model):
    """Scheduling / kernel-variant switches must not change results: weight-gradient GEMMs on side streams (`side_wgrad`) vs inline, the
    one-pass GLU / instance-norm backward kernel (`post_onepass`) vs sums + apply and its streaming (cp.async double-buffered) form vs the register-resident one (`post_stream`),
    the discriminator input layer's fused forward / backward (`fuse_c1`) vs conv + GLU kernels and a dP round trip
    -- same losses, same gradients up to the summation order of the gradient atomics."""
    from oracle import cyclegan_oracle as O
    lib, h = big_model._lib, big_model._handle
    A, B = O.synthetic_batch(seed=51, batch=12, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    defaults = {b"side_wgrad": 0, b"post_onepass": 1, b"fuse_c1": 1, b"post_stream": 1}
    cases = (("default", {}), ("side_wgrad", {b"side_wgrad": 1}), ("two_kernel_post", {b"post_onepass": 0}),
             ("unfused_c1", {b"fuse_c1": 0}), ("register_onepass", {b"post_stream": 0}))
    out = {}
    for name, opts in cases:
        for k, v in opts.items():
            assert lib.cgvc_set_option(h, k, v) == 0
        L, gA, gB = big_model.compute_gradients(A, B, 10.0, 5.0)
        out[name] = (L, gA, big_model.get_grads())
        for k in opts:
            assert lib.cgvc_set_option(h, k, defaults[k]) == 0
    for name, _ in cases[1:]:
        # the unfused discriminator input layer writes its dP in fp32 (D.h1 has no tensor-core slot, so no planes) and sums its weight,
        # bias and projection terms in another order than the fused kernels -- the only difference (test_gpu_glu_layers.py);
        # the three instance-norm backward forms add their per-sample sums in different orders, and in f16f8 a last-bit difference of a
        # dP element can land on the other side of a rounding boundary of its fp16 + e4m3 planes: the difference then travels down
        # the backward chain at the plane resolution (8e-5 measured at the generator's first layer; each form is within 3.6e-4 of the oracle)
        # (bf16x3: the same through the 2^-17 resolution of the bf16 hi / lo planes, 2.2e-5 measured)
        reorder = name in ("unfused_c1", "two_kernel_post", "register_onepass")
        tol = (3e-4 if big_model.precision == "f16f8" else 1e-4) if reorder else 2e-5      # (a wrong sum in any of these kernels shows at >= 1e-2)
        for k in out["default"][0]:
            assert abs(out[name][0][k] - out["default"][0][k]) <= 2e-6 * abs(out["default"][0][k]), (name, k)
        assert rel_l2(out[name][1], out["default"][1]) < 1e-6
        worst = (0.0, "")
        for k, g0 in out["default"][2].items():
            n0 = np.linalg.norm(g0.astype(np.float64).ravel())
            if n0 < 1e-6:
                continue
            e = np.linalg.norm((out[name][2][k].astype(np.float64) - g0).ravel()) / n0
            worst = max(worst, (e, k))
            assert e < tol, (name, k, e)
        print("%s vs default: worst gradient rel. diff %.2e (%s)" % (name, worst[0], worst[1]))


@pytest.mark.parametrize("frames,batch", [(128, 6), (256, 3), (512, 2), (64, 3)])
def test_fused_backward_matches_streaming_kernels(frames, batch):
    """The GLU / instance-norm backward fused into the data-gradient kernel's epilogue (residual blocks + second down-sampling
    layer of the generator; 32, 64 or 128 positions per sample) against the separate streaming kernels: every gradient tensor of
    the step.  frames = 64 gives 16 positions per sample, which the fused path must refuse (falls back, trivially equal)."""
    import cgvc
    from oracle import cyclegan_oracle as O
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=frames, precision="bf16x3", seed=5, log_dir='/tmp/cgvc_log')
    P = O.init_params(seed=77, dtype=torch.float32, perturb_affine=True)
    m.set_params({k: v.numpy() for k, v in P.items()})
    A, B = O.synthetic_batch(seed=43, batch=batch, frames=frames, dtype=torch.float32)
    out = {}
    for flag in (1, 0):
        assert m._lib.cgvc_set_option(m._handle, b"fuse_bwd", flag) == 0
        L, gA, gB = m.compute_gradients(A.numpy(), B.numpy(), 10.0, 5.0)
        out[flag] = (L, m.get_grads())
    m._lib.cgvc_set_option(m._handle, b"fuse_bwd", 0)
    for k in out[1][0]:
        assert abs(out[1][0][k] - out[0][0][k]) <= 1e-6 * abs(out[0][0][k]), k           # the forward pass is the same code
    worst = (0.0, "")
    for name, g0 in out[0][1].items():
        g1 = out[1][1][name]
        n0 = np.linalg.norm(g0.astype(np.float64).ravel())
        if n0 < 1e-6:
            # conv biases in front of an instance norm: analytically zero gradient; the streaming kernels accumulate their
            # rounding noise, the fused epilogue leaves them at exactly zero
            assert "/bias" in name and np.abs(g1).max() < 1e-5, name
            continue
        e = np.linalg.norm((g1.astype(np.float64) - g0).ravel()) / n0
        worst = max(worst, (e, name))
        assert e < 5e-5, (name, e)
    print("fused vs streaming backward, T=%d: worst gradient rel. diff %.2e (%s)" % (frames, worst[0], worst[1]))


def test_graph_replay_matches_eager_steps():
    """cgvc_train_step replays captured CUDA graphs (one per lane/shape configuration); scalars (lambdas, learning rates,
    Adam step) are fed through device memory, so changing them between replays must behave exactly like eager launches."""
    import cgvc
    rs = np.random.RandomState(3)
    ms = []
    for flag in (1, 0):
        m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision="bf16x3", seed=11)
        assert m._lib.cgvc_set_option(m._handle, b"cuda_graph", flag) == 0
        ms.append(m)
    sched = [(10, 5, 2e-4, 1e-4), (10, 5, 1e-4, 5e-5), (10, 0, 2e-4, 1e-4), (7, 5, 2e-4, 1e-4), (10, 0, 3e-4, 1e-4), (10, 5, 2e-4, 1e-4)]
    for lam_c, lam_i, lg, ld in sched:
        A = rs.randn(2, 24, 128); B = rs.randn(2, 24, 128)
        r = [m.train(A, B, lam_c, lam_i, lg, ld) for m in ms]
        # two runs of the same step differ in the order of their gradient atomics (~1e-6); Adam's early sign-descent steps turn that
        # into ~sqrt(1e-6) of an update (DESIGN.md section 7), so the trajectories agree to ~1e-4 ... 1e-3 after a few steps, not to rounding
        assert abs(r[0][0] - r[1][0]) <= 2e-3 * abs(r[1][0]) and abs(r[0][1] - r[1][1]) <= 2e-3 * abs(r[1][1]), (r, lam_c, lam_i)
    p1, p0 = ms[0].get_params(), ms[1].get_params()
    for k in ("generator_A2B/residual1d_block3_h1_conv/kernel", "generator_B2A/upsample1d_block1_h1_conv/kernel",
              "discriminator_A/downsample2d_block2_h1_gates/kernel", "discriminator_B/dense/kernel", "generator_A2B/InstanceNorm_6/gamma"):
        # (measured run to run after these six steps: 1e-4 ... 5.4e-4; a wrong learning rate / lambda / step count would show at >= 1e-2)
        print("graph vs eager after 6 steps: %s rel. diff %.2e" % (k, rel_l2(p1[k], p0[k])))
        assert rel_l2(p1[k], p0[k]) < 2e-3, k


def test_single_rank_communicator_paths_match_plain_step():
    """The data-parallel code paths on a one-rank NCCL communicator (the all-reduce is then an identity, so a plain model is the
    reference): per-network all-reduces on the communication stream pipelined with Adam + plane refresh (`pipelined_comm` = 1, default)
    and the single all-reduce followed by Adam (`pipelined_comm` = 0) give the plain step's losses and weights."""
    import torch.distributed as dist
    import cgvc
    if not dist.is_initialized():
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29577", rank=0, world_size=1)
    rs = np.random.RandomState(21)
    ms = [cgvc.CycleGAN(num_features=24, mode='train', max_batch=2, max_frames=128, precision="f16f8", seed=17, data_parallel=dp, log_dir='/tmp/cgvc_log')
          for dp in (False, True, True)]
    ms[2].set_option("pipelined_comm", 0)
    assert ms[1]._nranks == 1 and ms[2]._nranks == 1
    names = ("generator_A2B/residual1d_block2_h1_conv/kernel", "generator_B2A/o1_conv/kernel", "discriminator_A/downsample2d_block3_h1_conv/kernel",
             "discriminator_B/dense/kernel", "generator_B2A/InstanceNorm_9/gamma")
    # Two runs of the same step differ in the order of their gradient atomics (~1e-6 relative); Adam's early steps are sign descent
    # (update = lr * g / (|g| + eps')), which turns that into ~1e-3 of an update and lets the trajectories drift apart step by step
    # (DESIGN.md section 7).  So: the first step is compared tightly -- one update moves a weight by lr / |w| ~ 1e-2 relative, a network
    # whose Adam range or plane refresh the pipelined schedule missed would show at that size -- and the state after four steps at 3e-3
    # (measured run to run: 0.2e-3 ... 1.2e-3; a wrong range would be >= 1e-2).
    for step in range(4):
        A = rs.randn(2, 24, 128); B = rs.randn(2, 24, 128)
        r = [m.train(A, B, 10, 5 if step < 3 else 0, 2e-4, 1e-4) for m in ms]
        for k in (1, 2):
            tol = 2e-4 if step == 0 else 3e-3
            assert abs(r[k][0] - r[0][0]) <= tol * abs(r[0][0]) and abs(r[k][1] - r[0][1]) <= tol * abs(r[0][1]), (step, k, r)
        if step == 0:
            p0 = ms[0].get_params()
            for k in (1, 2):
                pk = ms[k].get_params()
                for name in names:
                    assert rel_l2(pk[name], p0[name]) < 2e-4, (k, name)
    p0 = ms[0].get_params()
    for k in (1, 2):
        pk = ms[k].get_params()
        for name in names:
            print("one-rank communicator path %d vs plain step after 4 steps: %s rel. diff %.2e" % (k, name, rel_l2(pk[name], p0[name])))
            assert rel_l2(pk[name], p0[name]) < 3e-3, (k, name)


def test_tensorboard_summaries(tmp_path):
    """model.py:153-169: the 8 scalar tags under generator_summaries/ and discriminator_summaries/."""
    import glob
    import cgvc
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=1, max_frames=128, precision="bf16x3", log_dir=str(tmp_path), summary_interval=1)
    x = np.random.RandomState(0).randn(1, 24, 128)
    m.train(x, x[:, ::-1].copy(), 10, 5, 2e-4, 1e-4)
    assert m.generator_summaries == ['generator_summaries/' + n for n in ('cycle_loss', 'identity_loss', 'generator_loss_A2B', 'generator_loss_B2A', 'generator_loss')]
    assert m.discriminator_summaries == ['discriminator_summaries/' + n for n in ('discriminator_loss_A', 'discriminator_loss_B', 'discriminator_loss')]
    if m.writer is not None:
        m.writer.flush()
        assert glob.glob(str(tmp_path / "*" / "events.out.tfevents.*"))


@pytest.mark.parametrize("prec", ["bf16x3", "f16f8"])
def test_loss_curve_tracks_oracle(prec):
    """40 consecutive train() steps (fresh minibatch per step, identity term switched off for the last 10, like
    train.py:98-99) replayed on the engine against the committed oracle trajectories (tests/golden/loss_curve.npz, made by
    tests/golden/make_loss_curve.py: the same run in float64 and in float32).

    A trajectory cannot be matched to 1e-3 beyond the first update, by ANY implementation that is not bit-identical:
    the first Adam steps are sign descent (update = lr * g / (|g| + eps')), so a gradient perturbation of relative size eta
    flips the sign of a fraction ~eta of the 1.2e8 elements and perturbs the update vector by ~sqrt(eta).  The oracle's own
    float32 run (eta ~ 1e-7) follows its float64 run to ~1e-6 for 9 steps, is knocked onto a neighbouring trajectory by a
    sign flip in an L1 gradient (1e-4 at step 9) and sits a few percent away on the adversarial terms from step ~18 on;
    the engine (gradients exact to ~1e-4) is at 2e-4 after one update and in the same few-percent envelope later.  So "loss curves match" is tested as
      (a) steps 0 and 1 (pre-update forward, and the loss after one Adam update): every logged loss within 1e-3 of float64;
      (b) the whole run stays inside the float32 oracle's envelope: per loss, the engine's worst deviation from the float64
          run is at most 5x the float32 run's worst deviation (+5e-3) -- measured 1.0x .. 2.1x over four runs (the engine's
          gradient atomics make runs differ from each other at this level too);
      (c) the levels agree: mean of every loss over the last 10 steps within 8 % of the float64 run's (measured 0.8-3.4 %)."""
    import os
    import cgvc
    from oracle import cyclegan_oracle as O
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_curve.npz"))
    steps, batch, seed_w, seed_x = int(z["steps"]), int(z["batch"]), int(z["seed_w"]), int(z["seed_x"])
    ref64, ref32 = z["f64"], z["f32"]
    P = O.init_params(seed=seed_w, dtype=torch.float32, perturb_affine=True)
    m = cgvc.CycleGAN(num_features=24, mode='train', max_batch=batch, max_frames=128, precision=prec, log_dir='/tmp/cgvc_log')
    m.set_params({k: v.numpy() for k, v in P.items()})
    got = []
    for t in range(steps):
        A, B = O.synthetic_batch(seed=seed_x + t, batch=batch, frames=128, dtype=torch.float32)
        lam_id = 5.0 if t < (3 * steps) // 4 else 0.0
        m.train(A.numpy(), B.numpy(), 10.0, lam_id, 2e-4, 1e-4)
        got.append([m.last_losses[k] for k in O.LOSS_NAMES])
    got = np.array(got)
    dev = np.abs(got - ref64) / np.abs(ref64)
    floor = np.abs(ref32 - ref64) / np.abs(ref64)
    out = os.environ.get("CGVC_LOSS_CURVE_CSV")
    if out:
        with open(out, "w") as f:
            f.write("step," + ",".join("%s_engine,%s_oracle64,%s_oracle32" % (n, n, n) for n in O.LOSS_NAMES) + "\n")
            for t in range(steps):
                f.write(str(t) + "," + ",".join("%.9g,%.9g,%.9g" % (got[t, i], ref64[t, i], ref32[t, i]) for i in range(8)) + "\n")
    m10 = np.abs(got[-10:].mean(axis=0) - ref64[-10:].mean(axis=0)) / np.abs(ref64[-10:].mean(axis=0))
    print("loss curve: steps 0-1 worst engine-vs-f64 %.2e (f32 oracle %.2e); whole run worst %.2e at step %d (f32 oracle %.2e); "
          "last-10-step means within %.2e; last step G %.5f (oracle %.5f) D %.5f (oracle %.5f)"
          % (dev[:2].max(), floor[:2].max(), dev.max(), int(dev.max(axis=1).argmax()), floor.max(), m10.max(), got[-1, 4], ref64[-1, 4], got[-1, 7], ref64[-1, 7]))
    assert dev[:2].max() < TOL, dev[:2].max(axis=1)
    assert (dev.max(axis=0) <= 5.0 * floor.max(axis=0) + 5e-3).all(), (dev.max(axis=0), floor.max(axis=0))
    assert m10.max() < 0.08, m10
