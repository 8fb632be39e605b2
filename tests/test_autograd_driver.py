"""The differentiable networks' host side (CycleGAN.generator / .discriminator, zero_grad, grads, adam_step) on a stub library: the
argument order of the tape calls, the tape sizing, which gradients autograd asks for, and the loss-scale arithmetic of grads() and
adam_step().  The stub's 'networks' are y = 2 x (generator) and p[b, h, t] = sum of x's 16-frame block (discriminator), their
backward adds a marker into GRAD."""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch


class StubLib:
    def __init__(self, grad):
        self.grad = grad
        self.calls = []

    @staticmethod
    def _t(ptr, n):
        return torch.from_numpy(np.ctypeslib.as_array((C.c_float * n).from_address(ptr.value)))

    def cgvc_tape_bytes(self, h, kind, batch, frames, out):
        self.calls.append(("bytes", kind, batch, frames))
        out._obj.value = 4096 + 4 * batch * 24 * frames
        return 0

    def cgvc_generator_forward_tape(self, h, d, x, y, batch, frames, tape, nbytes, stream):
        self.calls.append(("gfwd", d, batch, frames, nbytes))
        n = batch * 24 * frames
        self._t(y, n).copy_(2 * self._t(x, n))
        self._t(tape, 1)[0] = 100 + d
        return 0

    def cgvc_discriminator_forward_tape(self, h, w, x, p, batch, frames, tape, nbytes, stream):
        self.calls.append(("dfwd", w, batch, frames, nbytes))
        xs = self._t(x, batch * 24 * frames).view(batch, 6, 4, frames // 16, 16)
        self._t(p, batch * 6 * (frames // 16)).copy_(xs.sum(dim=(2, 4)).reshape(-1))
        self._t(tape, 1)[0] = 200 + w
        return 0

    def cgvc_generator_backward_tape(self, h, tape, dy, dx, stream):
        d = int(self._t(tape, 1)[0]) - 100
        self.calls.append(("gbwd", d, dx.value is not None))
        self.grad[d] += 1024.0                       # a loss-scaled contribution
        if dx.value:
            n = self._nx
            self._t(dx, n).copy_(2 * self._t(dy, n))
        return 0

    def cgvc_discriminator_backward_tape(self, h, tape, dp, dx, stream):
        w = int(self._t(tape, 1)[0]) - 200
        self.calls.append(("dbwd", w, dx.value is not None))
        self.grad[2 + w] += 1024.0
        if dx.value:
            b, t = self._shape
            g = self._t(dp, b * 6 * (t // 16)).view(b, 6, 1, t // 16, 1)
            self._t(dx, b * 24 * t).copy_(g.expand(b, 6, 4, t // 16, 16).reshape(-1))
        return 0

    def cgvc_adam_step(self, h, lr_g, lr_d, grad_scale, stream):
        self.calls.append(("adam", lr_g, lr_d, grad_scale))
        return 0


def _model(prec, batch, frames):
    import cgvc  # noqa: F401
    M = importlib.import_module("cgvc.model")
    N = importlib.import_module("cgvc._native")
    m = object.__new__(M.CycleGAN)
    m.num_features, m.precision, m.device = 24, prec, torch.device("cpu")
    m._max_batch, m._max_frames, m._handle = batch, frames, C.c_void_p(1)
    m._tape_scales, m._grad_token, m.train_step = set(), None, 0
    m._table = {"generator_A2B/w": (0, (1,)), "generator_B2A/w": (1, (1,)), "discriminator_A/w": (2, (1,)), "discriminator_B/w": (3, (1,))}
    m._arenas = {N.ARENA_GRAD: torch.zeros(4)}
    m._lib = StubLib(m._arenas[N.ARENA_GRAD])
    m._stream = lambda: C.c_void_p(0)
    return m


@pytest.mark.parametrize("prec,scale", [("f16f8", 1024.0), ("bf16x3", 1.0)])
def test_autograd_wiring_on_a_stub_library(prec, scale):
    b, t = 2, 32
    m = _model(prec, b, t)
    m._lib._nx, m._lib._shape = b * 24 * t, (b, t)
    if scale != 1.0:          # 2^(9 + min(floor(log2 batch), 9))
        assert (m.tape_loss_scale(1), m.tape_loss_scale(2), m.tape_loss_scale(3), m.tape_loss_scale(4096)) == (512, 1024, 1024, 2 ** 18)
    else:
        assert m.tape_loss_scale(7) == 1.0
    x = torch.randn(b, 24, t, requires_grad=True)
    real = torch.randn(b, 24, t)
    y = m.generator(x, 'B2A')
    assert torch.equal(y, 2 * x.detach())
    p = m.discriminator(y, 'A')
    q = m.discriminator(real, 'B')                      # an input without grad: the weight gradients still run
    assert p.shape == (b, 6, t // 16, 1)
    assert m._lib.calls[:2] == [("bytes", 0, b, t), ("gfwd", 1, b, t, 4096 + 4 * b * 24 * t)]
    assert m._lib.calls[3][:4] == ("dfwd", 0, b, t)
    m.zero_grad()
    (p.sum() + q.sum()).backward()
    # d in is asked for only where autograd needs it: not for the real sample
    assert sorted(c for c in m._lib.calls if c[0].endswith("bwd")) == [("dbwd", 0, True), ("dbwd", 1, False), ("gbwd", 1, True)]
    assert torch.equal(x.grad, torch.full_like(x, 2.0))           # d sum(D(2x)) / dx through both stub backward passes
    g = m.grads()
    assert [float(v) for v in g.values()] == [0.0, 1024.0 / scale, 1024.0 / scale, 1024.0 / scale]
    assert list(m.grads("discriminator_B")) == ["discriminator_B/w"]
    m.adam_step(2e-4, 1e-4)
    assert m._lib.calls[-1] == ("adam", 2e-4, 1e-4, 1.0 / scale)
    m.zero_grad("generator_B2A")
    assert float(m._arenas[importlib.import_module("cgvc._native").ARENA_GRAD][1]) == 0.0
    # tapes of a batch with another loss scale must not share one gradient arena
    if scale != 1.0:
        m.discriminator(torch.randn(1, 24, t), 'A').sum().backward()
        with pytest.raises(RuntimeError, match="different loss scales"):
            m.adam_step(2e-4, 1e-4)
        m.zero_grad()
        assert m._grad_scale() == 1.0
    with pytest.raises(Exception, match="direction"):
        m.generator(x, 'A2A')
