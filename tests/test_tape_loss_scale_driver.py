"""tape_loss_scale='dynamic' on the host side, on a stub library: the constructor's checks, the argument order and refusals of
apply_gradients(), grads() dividing the gradient arena by the scaler's device scale(s), adam_step() and tape_loss_scale() refusing, and
the option applied again when the engine is re-created for a larger batch."""
import ctypes as C
import importlib

import pytest
import torch

import cgvc  # noqa: F401

M = importlib.import_module("cgvc.model")
N = importlib.import_module("cgvc._native")

TABLE = ["generator_A2B/w", "generator_B2A/w", "discriminator_A/w", "discriminator_B/w"]


class StubLib:
    """The calls the tape loss-scale path makes, recorded; the scaler state is s (one scale) or s_G / s_D (per network)."""

    def __init__(self, s=1024.0, s_G=2.0, s_D=512.0):
        self.calls = []
        self.s, self.s_G, self.s_D = s, s_G, s_D

    def cgvc_loss_scale_state(self, h, out, stream):
        self.calls.append(("state",))
        info = N.LossScaleInfo(scale=self.s, good_steps=3, skipped=1)
        C.memmove(out.value, C.byref(info), C.sizeof(info))
        return 0

    def cgvc_loss_scale_net_state(self, h, out, stream):
        self.calls.append(("net_state",))
        nets = (N.LossScaleNetInfo * 2)(N.LossScaleNetInfo(scale=self.s_G), N.LossScaleNetInfo(scale=self.s_D))
        C.memmove(out.value, nets, C.sizeof(nets))
        return 0

    def cgvc_apply_gradients(self, h, lr_g, lr_d, stream):
        self.calls.append(("apply", lr_g, lr_d))
        return 0

    def cgvc_adam_step(self, h, lr_g, lr_d, grad_scale, stream):
        self.calls.append(("adam", lr_g, lr_d, grad_scale))
        return 0

    # engine re-creation (_ensure_capacity -> _create_engine)
    def cgvc_get_adam_step(self, h, t):
        t._obj.value = 7
        return 0

    def cgvc_destroy(self, h):
        self.calls.append(("destroy",))
        return 0

    def cgvc_create(self, cfg, h):
        self.calls.append(("create", cfg._obj.max_batch, cfg._obj.max_frames))
        h._obj.value = 2
        return 0

    def cgvc_param_count(self, h, nt, ne):
        nt._obj.value, ne._obj.value = len(TABLE), len(TABLE)
        return 0

    def cgvc_param_info(self, h, i, name, off, nd, shp):
        name._obj.value, off._obj.value, nd._obj.value = TABLE[i].encode(), i, 1
        shp._obj[0] = 1
        return 0

    def cgvc_arena_bytes(self, h, kind, nbytes):
        nbytes._obj.value = 64
        return 0

    def cgvc_bind_arena(self, h, kind, p, n):
        return 0

    def cgvc_set_option(self, h, name, value):
        self.calls.append(("option", name, value))
        return 0

    def cgvc_set_adam_step(self, h, t):
        self.calls.append(("set_t", t.value))
        return 0

    def cgvc_set_loss_scale_state(self, h, scale, good, skipped, stream):
        self.calls.append(("set_state", scale, good, skipped))
        return 0

    def cgvc_set_loss_scale_net_state(self, h, net, scale, good, stream):
        self.calls.append(("set_net", net, scale, good))
        return 0

    def cgvc_params_updated(self, h, stream):
        return 0


def _model(prec="f16f8", per_network=False, dynamic=True, **stub):
    m = object.__new__(M.CycleGAN)
    m.num_features, m.precision, m.device, m.mode = 24, prec, torch.device("cpu"), "train"
    m._max_batch, m._max_frames, m._handle = 2, 64, C.c_void_p(1)
    m._tape_scales, m._grad_token, m.train_step, m._data_parallel = set(), None, 0, False
    m._options = {"loss_scale": 2}
    if per_network:
        m._options["loss_scale_per_network"] = 1
    if dynamic:
        m._options["tape_loss_scale"] = 1
    m._tape_dynamic = dynamic
    m._table = {n: (i, (1,)) for i, n in enumerate(TABLE)}
    m._arenas = {N.ARENA_GRAD: torch.tensor([1024.0, 2048.0, 512.0, 1536.0])}
    m._ls_dev = torch.zeros(C.sizeof(N.LossScaleInfo), dtype=torch.uint8)
    m._lsn_dev = torch.zeros(2 * C.sizeof(N.LossScaleNetInfo), dtype=torch.uint8)
    m._lib = StubLib(**stub)
    m._stream = lambda: C.c_void_p(0)
    return m


def test_constructor_checks_tape_loss_scale():
    with pytest.raises(ValueError, match="needs loss_scale='dynamic'"):
        M.CycleGAN(24, loss_scale='monitor', tape_loss_scale='dynamic')
    with pytest.raises(ValueError, match="needs loss_scale='dynamic'"):
        M.CycleGAN(24, tape_loss_scale='dynamic')
    with pytest.raises(ValueError, match="'static' or 'dynamic'"):
        M.CycleGAN(24, loss_scale='dynamic', tape_loss_scale='monitor')


def test_apply_gradients_argument_order_and_refusals():
    m = _model()
    m.apply_gradients(2e-4, 1e-4)
    assert m._lib.calls == [("apply", 2e-4, 1e-4)]
    assert m.train_step == 1
    with pytest.raises(RuntimeError, match="apply_gradients"):
        m.adam_step(2e-4, 1e-4)
    with pytest.raises(RuntimeError, match="scaler"):
        m.tape_loss_scale(4)
    # static tapes keep adam_step and refuse apply_gradients, before the library is called
    s = _model(dynamic=False)
    with pytest.raises(RuntimeError, match="tape_loss_scale='dynamic'"):
        s.apply_gradients(2e-4, 1e-4)
    s.adam_step(2e-4, 1e-4)
    assert s._lib.calls == [("adam", 2e-4, 1e-4, 1.0)]
    assert s.tape_loss_scale(4) == 2048.0


def test_grads_divide_by_the_device_scale():
    m = _model(s=512.0)
    g = m.grads()
    assert [float(v) for v in g.values()] == [2.0, 4.0, 1.0, 3.0]
    assert ("net_state",) not in m._lib.calls
    assert list(m.grads("discriminator_A")) == ["discriminator_A/w"]
    # after apply_gradients the scale may have changed: refused until zero_grad
    m.apply_gradients(1e-3, 1e-3)
    with pytest.raises(RuntimeError, match="after apply_gradients"):
        m.grads()
    m.zero_grad()
    assert [float(v) for v in m.grads().values()] == [0.0] * 4


def test_grads_divide_per_network():
    m = _model(per_network=True, s=2.0, s_G=2.0, s_D=512.0)
    g = m.grads()
    assert [float(v) for v in g.values()] == [512.0, 1024.0, 1.0, 3.0]
    assert ("net_state",) in m._lib.calls
    # outside F16F8 the engine keeps one scale whatever the option says
    b = _model(prec="bf16x3", per_network=True, s=1.0, s_G=0.0, s_D=0.0)
    assert [float(v) for v in b.grads().values()] == [1024.0, 2048.0, 512.0, 1536.0]


def test_unset_scale_reads_as_one():
    m = _model(s=0.0)                     # the scaler before the first tape backward
    assert [float(v) for v in m.grads().values()] == [1024.0, 2048.0, 512.0, 1536.0]


def test_options_follow_engine_re_creation(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    m = _model(per_network=True)
    m.device = torch.device("cpu", 0)     # cgvc_config takes the device index
    m._options = {"loss_scale": 2, "loss_scale_per_network": 1, "tape_loss_scale": 1}
    m._arenas = {}
    state = {"scale": 256.0, "good_steps": 5, "skipped": 2, "scale_G": 8.0, "good_steps_G": 1, "scale_D": 256.0, "good_steps_D": 5}
    monkeypatch.setattr(m, "loss_scale_state", lambda: dict(state))
    m._ensure_capacity(4, 64)
    calls = m._lib.calls
    assert ("create", 4, 64) in calls
    opts = [c[1:] for c in calls if c[0] == "option"]
    assert opts == [(b"loss_scale", 2), (b"loss_scale_per_network", 1), (b"tape_loss_scale", 1)]   # tape_loss_scale after loss_scale
    assert calls.index(("set_state", 256.0, 5, 2)) > calls.index(("option", b"tape_loss_scale", 1))
    assert ("set_net", 0, 8.0, 1) in calls and ("set_net", 1, 256.0, 5) in calls
    assert ("set_t", 7) in calls
