"""The tensor-core weight planes (every GEMM's B operand) against tests/weight_planes_ref.py, byte for byte, padding included.

Every registered layer of the four networks and every plane the engine keeps (cgvc_weight_planes), in bf16x3, bf16 and F16F8, on
training and forward-only engines and with `prep_batched` 0 (three kernels per layer branch) and 1 (the job-table kernel):

A. Layouts and values: the oracle's init weights, and a stress set at the edges of the weight window (weight_planes_ref.stress_values:
   ties of fp16, bf16 and e4m3, both clamp edges of the e4m3 planes, fp16 overflow and subnormals) in every kernel and bias, with the
   planes' tails -- the last input and output channel, next to the padding -- holding them too.
B. Refresh: after every way PARAM changes (set_params, train() replayed as a graph and eager, the one-rank communicator step whose
   pipelined schedule refreshes network by network, adam_step after a tape backward, load(), a step skipped by the dynamic loss scale)
   the planes equal the reference built from the PARAM of that moment.  One Adam step (lr 2e-4) moves every weight's planes, so a layer
   left one step behind shows in most of its elements.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import weight_planes_ref as W

pytestmark = pytest.mark.gpu

ALL_PLANES = W.BF16_PLANES + W.Q_PLANES + W.QD_PLANES + ("bias",)
NETWORKS = ("generator_A2B", "generator_B2A", "discriminator_A", "discriminator_B")


def _N():
    from cgvc import native
    return native


def _model(precision, mode="train", **kw):
    import cgvc
    return cgvc.CycleGAN(num_features=24, mode=mode, max_batch=1, max_frames=128, precision=precision, seed=5, log_dir="/tmp/cgvc_log", **kw)


def _layers(m):
    N = _N()
    info = N.WeightLayerInfo()
    m._chk(m._lib.cgvc_weight_planes(m._handle, 0, C.byref(info), None, None, 0, None, None))
    out = []
    for i in range(info.n_layers):
        m._chk(m._lib.cgvc_weight_planes(m._handle, i, C.byref(info), None, None, 0, None, None))
        L = W.Layer(**{f: getattr(info, f) for f in W.Layer.FIELDS})
        got = (info.nt_n, info.cin_k, info.cin_n, info.nt_k, info.cin_q, info.nt_q)
        assert got == L.dims(), (i, L, got)
        assert bool(info.q_ok) == L.q_ok(), (i, L)
        out.append(L)
    return out


def _label(m, i, L):
    name = next(n for n, (off, _) in m._table.items() if off == L.ka)
    shape = m._table[name][1]
    lowered = L.taps == 1 and int(np.prod(shape[:-2])) > 1
    return "layer %d (%s%s)" % (i, name, ", tap-lowered 1 x 1 form" + (" with folded taps" if L.fold else "") if lowered else "")


def _plane(m, i, name, L):
    """the engine's plane as bit patterns shaped like the reference's; None if the engine refuses it (and only as CGVC_ERR_ARG)"""
    lib, h = m._lib, m._handle
    n = C.c_size_t(0)
    rc = lib.cgvc_weight_planes(h, i, None, name.encode(), None, 0, C.byref(n), None)
    if rc != 0:
        assert rc == _N().ERR_ARG, (i, name, rc)
        return None
    buf = torch.empty(n.value, dtype=torch.uint8, device=m.device)
    m._chk(lib.cgvc_weight_planes(h, i, None, name.encode(), C.c_void_p(buf.data_ptr()), n.value, C.byref(n), m._stream()))
    return buf.cpu().numpy().view(W.PLANE_DTYPE[name]).reshape(W.plane_shape(L, name))


def _param_arena(m):
    torch.cuda.synchronize(m.device)
    return m._arenas[_N().ARENA_PARAM].cpu().numpy()


def _check(engines, what):
    """engines: [(label, model, precision, train)], all holding the same PARAM.  Every layer's reference is built once per precision
    family and compared with every engine's planes; the planes an engine does not keep must be refused."""
    params = _param_arena(engines[0][1])
    for _, m, _, _ in engines[1:]:
        assert np.array_equal(_param_arena(m).view(np.uint32), params.view(np.uint32))
    layers = _layers(engines[0][1])
    bad, compared = [], 0
    for i, L in enumerate(layers):
        refs = {}
        for tag, m, prec, train in engines:
            key = ("f16f8" if prec == "f16f8" and L.q_ok() else "bf16", train)
            if key not in refs:
                refs[key] = W.planes(L, params, prec, train)
            ref = refs[key]
            kept = W.kept_planes(L, prec, train)
            for name in ALL_PLANES:
                got = _plane(m, i, name, L)
                if name not in kept:
                    if got is not None:
                        bad.append("%s %s: plane %s should not be kept" % (tag, _label(m, i, L), name))
                    continue
                if got is None:
                    bad.append("%s %s: plane %s refused" % (tag, _label(m, i, L), name))
                    continue
                compared += got.size
                diff = W.differences(name, got, ref[name])
                if diff:
                    bad.append("%s %s: plane %s %s: %s" % (tag, _label(m, i, L), name, W.plane_shape(L, name), diff))
    print("%s: %d layers, %d plane elements compared over %d engines" % (what, len(layers), compared, len(engines)))
    assert not bad, "%s: %d planes differ from the reference:\n%s" % (what, len(bad), "\n".join(bad[:12]))


@pytest.fixture(scope="module")
def init_params():
    from oracle import cyclegan_oracle as O
    return {k: v.numpy() for k, v in O.init_params(seed=3, dtype=torch.float32, perturb_affine=True).items()}


def _stress_params(m):
    rng = np.random.default_rng(11)
    return {n: W.stress_fill(shape, rng) for n, (_, shape) in m._table.items() if n.endswith("/kernel") or n.endswith("/bias")}


def test_every_layer_of_the_four_networks_is_registered():
    """the store's registration against the parameter table: every convolution of the four networks except the discriminator's
    single-channel input layer (its own fused kernels), plus the generators' tap-lowered edge layers; the entry point's refusals"""
    N = _N()
    m = _model("bf16x3", mode="test")
    layers = _layers(m)
    assert len(layers) == 46
    want = set()
    for net in NETWORKS:
        for n, (off, shape) in m._table.items():
            if n.startswith(net + "/") and n.endswith("/kernel") and len(shape) >= 3 and not ("discriminator" in net and shape[-2] == 1):
                if "gates" not in n:
                    want.add(off)
    assert {L.ka for L in layers} == want
    for i, L in enumerate(layers):
        name = next(n for n, (off, _) in m._table.items() if off == L.ka)
        shape = m._table[name][1]
        taps = int(np.prod(shape[:-2]))
        if L.fold:                                   # o1: [1, 15, 256, 24] as 256 -> 15 * 24 columns
            assert (L.taps, L.cin, L.cout, L.fold, L.gated) == (1, shape[-2], taps * shape[-1], taps, 0)
        elif L.taps == 1 and taps > 1:               # h1: [1, 15, 24, 128] as K = 15 * 24
            assert (L.cin, L.cout, L.gated) == (taps * shape[-2], shape[-1], 1)
        else:
            assert (L.kh * L.kw, L.cin, L.cout) == (taps, shape[-2], shape[-1]), name
        if L.gated:
            gname = next(n for n, (off, _) in m._table.items() if off == L.kg)
            assert gname.endswith("gates/kernel") and m._table[gname][1] == shape, name
            assert m._table[gname.replace("/kernel", "/bias")][0] == L.bg, name
        if not L.fold:
            assert m._table[name.replace("/kernel", "/bias")][0] == L.ba, name
    for net in NETWORKS:
        assert sum(1 for L in layers if next(n for n, (o, _) in m._table.items() if o == L.ka).startswith(net)) == (20 if "gen" in net else 3)
    lib, h = m._lib, m._handle
    n = C.c_size_t(0)
    assert lib.cgvc_weight_planes(h, 46, None, None, None, 0, None, None) == N.ERR_ARG
    assert lib.cgvc_weight_planes(h, -1, None, None, None, 0, None, None) == N.ERR_ARG
    assert lib.cgvc_weight_planes(h, 0, None, b"wf_mid", None, 0, C.byref(n), None) == N.ERR_ARG
    assert lib.cgvc_weight_planes(h, 0, None, b"bias", None, 0, C.byref(n), None) == 0 and n.value == layers[0].dims()[0] * 4
    small = torch.empty(n.value - 4, dtype=torch.uint8, device=m.device)
    assert lib.cgvc_weight_planes(h, 0, None, b"bias", C.c_void_p(small.data_ptr()), n.value - 4, C.byref(n), None) == N.ERR_ARG


@pytest.mark.parametrize("values", ["init", "stress"])
@pytest.mark.parametrize("family", ["bf16", "f16f8"])
def test_planes_match_reference(family, values, init_params):
    """bf16: bf16x3 and bf16 engines, training and forward-only.  f16f8: training and forward-only engines, each with prep_batched 0
    and 1"""
    if family == "bf16":
        specs = [("bf16x3/train", "bf16x3", "train", None), ("bf16x3/test", "bf16x3", "test", None),
                 ("bf16/train", "bf16", "train", None), ("bf16/test", "bf16", "test", None)]
    else:
        specs = [("f16f8/%s/prep_batched=%d" % (mode, pb), "f16f8", mode, pb) for mode in ("train", "test") for pb in (0, 1)]
    engines = []
    for tag, prec, mode, pb in specs:
        m = _model(prec, mode=mode)
        if pb is not None:
            m.set_option("prep_batched", pb)
        engines.append((tag, m, prec, mode == "train"))
    params = init_params if values == "init" else _stress_params(engines[0][1])
    for _, m, _, _ in engines:
        m.set_params(params)
    _check(engines, "%s %s" % (family, values))


def _tape_step(m, rs):
    x = torch.tensor(rs.randn(1, 24, 128), dtype=torch.float32, device=m.device)
    m.zero_grad()
    y = m.generator(x, "A2B")
    p = m.discriminator(y, "B")
    (y.square().mean() + p.mean()).backward()
    m.adam_step(2e-4, 1e-4)


@pytest.mark.parametrize("precision", ["bf16x3", "f16f8"])
def test_planes_follow_every_parameter_change(precision, init_params, tmp_path):
    import torch.distributed as dist
    from oracle import cyclegan_oracle as O
    rs = np.random.RandomState(7)
    A, B = O.synthetic_batch(seed=71, batch=1, frames=128, dtype=torch.float32)
    A, B = A.numpy(), B.numpy()
    m = _model(precision)
    eng = [(precision, m, precision, True)]

    def step(what, change, moves=True):
        before = _param_arena(m).copy()
        change()
        after = _param_arena(m)
        assert np.array_equal(before.view(np.uint32), after.view(np.uint32)) != moves, what
        _check(eng, "%s after %s" % (precision, what))

    step("set_params", lambda: m.set_params(init_params))
    step("train() replayed as a CUDA graph (second step)", lambda: [m.train(A, B, 10.0, 5.0, 2e-4, 1e-4) for _ in range(2)])
    m.set_option("cuda_graph", 0)
    step("train() with cuda_graph 0", lambda: m.train(A, B, 10.0, 5.0, 2e-4, 1e-4))
    m.set_option("cuda_graph", 1)
    step("adam_step after a tape backward", lambda: _tape_step(m, rs))
    path = m.save(str(tmp_path), "ckpt")
    m.train(A, B, 10.0, 5.0, 2e-4, 1e-4)
    step("load()", lambda: m.load(path))
    m.set_option("loss_scale", 2)
    bad = A.copy()
    bad[0, 3, 17] = np.nan

    def skipped():
        m.train(bad, B, 10.0, 5.0, 2e-4, 1e-4)
        assert m.last_step_skipped
    step("a step skipped by the dynamic loss scale", skipped, moves=False)
    eng.clear()

    # the one-rank communicator step: Adam and the plane refresh network by network (tc_refresh_weights_range)
    if not dist.is_initialized():
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29577", rank=0, world_size=1)
    m = _model(precision, data_parallel=True)
    assert m._nranks == 1 and m._options.get("pipelined_comm", 1) == 1
    eng.append(("%s/one-rank communicator" % precision, m, precision, True))
    m.set_params(init_params)
    step("the pipelined one-rank communicator step", lambda: m.train(A, B, 10.0, 5.0, 2e-4, 1e-4))
