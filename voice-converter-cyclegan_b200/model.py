"""`CycleGAN`: the reference's model class (model.py:7-169 of /root/reference) on the native H100 engine.

Same constructor and method signatures as the reference; the TensorFlow-1 session is replaced by libcgvc.so
(hand-written sm_90a CUDA behind the C ABI in include/cgvc.h).  PyTorch is used for device storage
(arenas, staging) only -- no torch op runs on the hot path.

Differences a user of the reference should know:
  * weights are glorot-uniform like TF's default (SURVEY.md Appendix A.3), drawn from `seed`
  * minibatches larger than 1 are first-class (the reference hard-codes 1, train.py:16)
  * `train`/`test` accept host numpy arrays (as in the reference) or CUDA torch tensors (zero-copy)
  * checkpoints are .npz files keyed by the TF variable names (plus `<var>/Adam`, `<var>/Adam_1`, `adam_step`)
  * with `torch.distributed` initialised and `data_parallel=True`, one process per GPU trains data-parallel:
    a single NCCL all-reduce of the flat gradient arena per step
  * `loss_scale='monitor'` counts saturated F16F8 gradient / activation planes and non-finite gradients every step;
    `loss_scale='dynamic'` also skips such steps and adapts the loss scale (include/cgvc.h, DESIGN.md section 10);
    `loss_scale_per_network=True` gives the generators and the discriminators a scale each and counts their planes apart, with the
    groups below the fp16 lower edge beside the saturated ones (F16F8 only)
  * `deterministic=True` makes every train step bit-reproducible on one GPU: the same weights, Adam and loss-scale state and inputs give
    the same bits whatever the stream schedule or CUDA-graph replay, so a rerun of a seed or a resumed checkpoint follows the
    same trajectory (include/cgvc.h option "deterministic", DESIGN.md section 11; the NCCL sum of a data-parallel step is not covered)
  * `generator(x, direction)` / `discriminator(x, which)` are the four networks as differentiable torch operators on CUDA tensors, for
    objectives other than the fused step's: `loss.backward()` adds their weight gradients into the gradient arena, `zero_grad()`,
    `grads()` and `adam_step()` complete a step (include/cgvc.h "activation tapes", DESIGN.md section 12).  The network descriptors
    given to the constructor are `generator_descriptor` / `discriminator_descriptor`; `generator_packed(inputs, direction)` and
    `discriminator_packed(inputs, which)` are the networks over a list of utterances of different lengths in one call, for
    utterance-level objectives
  * `tape_loss_scale='dynamic'` (with `loss_scale='dynamic'`) puts those networks' backward passes on the engine's loss scaler:
    `apply_gradients()` then all-reduces (data parallel), checks and updates the scale, and skips an overflowing step on the device,
    as train() does (include/cgvc.h cgvc_apply_gradients, DESIGN.md section 12)
"""
from __future__ import annotations

import ctypes as C
import math
import os
from collections import OrderedDict
from datetime import datetime

import numpy as np
import torch

from . import _native as N
from .module import discriminator as _discriminator, generator_gatedcnn as _generator_gatedcnn


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _direction(direction):
    """'A2B' -> 0, 'B2A' -> 1 (model.py:128-137)"""
    d = {'A2B': 0, 'B2A': 1}.get(direction)
    if d is None:
        raise Exception('Conversion direction must be specified.')
    return d


class CycleGAN(object):
    _tape_dynamic = False            # tape_loss_scale='dynamic'
    _grads_applied = False           # apply_gradients() ran since the last zero_grad()

    def __init__(self, num_features, discriminator=_discriminator, generator=_generator_gatedcnn, mode='train',
                 log_dir='./log', *, max_batch=1, max_frames=None, precision='bf16x3', device=None, seed=0,
                 data_parallel=False, summary_interval=0, loss_scale='static', deterministic=False, loss_scale_per_network=False,
                 tape_loss_scale='static'):
        for net in (discriminator, generator):
            if not hasattr(net, "check_engine_table"):
                raise TypeError("CycleGAN(discriminator=..., generator=...) takes network descriptors (cgvc.module.generator_gatedcnn / "
                                "cgvc.module.discriminator or equivalents), not %r: the native engine runs its own kernel graph" % (net,))
        if tape_loss_scale not in ('static', 'dynamic'):
            raise ValueError("tape_loss_scale must be 'static' or 'dynamic', got %r" % (tape_loss_scale,))
        if tape_loss_scale == 'dynamic' and loss_scale != 'dynamic':
            raise ValueError("tape_loss_scale='dynamic' needs loss_scale='dynamic'")
        if not torch.cuda.is_available():
            raise RuntimeError("CycleGAN needs a CUDA device (sm_90a); there is no CPU fallback")
        self.num_features = num_features
        self.input_shape = [None, num_features, None]
        self.discriminator_descriptor = discriminator
        self.generator_descriptor = generator
        self.mode = mode
        self.precision = precision
        self._lib = N.load()
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device if isinstance(device, int) else torch.device(device).index or 0)
        self._handle = C.c_void_p(0)
        self._max_batch = int(max_batch)
        self._max_frames = int(max_frames) if max_frames else 128
        self._arenas = {}
        self._options = {}
        if loss_scale not in N.LOSS_SCALE_MODES:
            raise ValueError("loss_scale must be one of %s, got %r" % (sorted(N.LOSS_SCALE_MODES), loss_scale))
        if loss_scale != 'static':
            self._options["loss_scale"] = N.LOSS_SCALE_MODES[loss_scale]     # applied by _create_engine, like any remembered option
        if loss_scale_per_network:
            self._options["loss_scale_per_network"] = 1
        if tape_loss_scale == 'dynamic':
            self._options["tape_loss_scale"] = 1                 # after "loss_scale": the engine accepts it in dynamic mode only
        self._tape_dynamic = tape_loss_scale == 'dynamic'
        if deterministic:
            self._options["deterministic"] = 1
        self.last_step_skipped = False
        self.last_loss_scale = None
        self._tape_scales = set()        # loss scales of the tape backward calls since zero_grad (adam_step divides by it)
        self._grad_token = None
        self._create_engine()
        # the descriptors state the architecture the caller expects (model.py:14-15); the engine must implement exactly that
        for scope in ("generator_A2B", "generator_B2A"):
            generator.check_engine_table(self._table, scope, num_features)
        for scope in ("discriminator_A", "discriminator_B"):
            discriminator.check_engine_table(self._table, scope, num_features)
        self._init_params(seed)
        self._rank, self._nranks = 0, 1
        self._data_parallel = bool(data_parallel)
        if data_parallel:
            self._attach_communicator()
        self.train_step = 0
        self.last_losses = None
        self.writer = None
        self.summary_interval = summary_interval
        if self.mode == 'train':
            now = datetime.now()
            self.log_dir = os.path.join(log_dir, now.strftime('%Y%m%d-%H%M%S'))
            if summary_interval:
                self.generator_summaries, self.discriminator_summaries = self.summary()

    # ------------------------------------------------------------------ engine plumbing
    def _chk(self, code):
        N.check(self._handle, code)

    def _create_engine(self):
        cfg = N.Config(self.num_features, self._max_batch, self._max_frames, N.PRECISIONS[self.precision],
                       self.device.index, 1 if self.mode == 'train' else 0)
        h = C.c_void_p(0)
        code = self._lib.cgvc_create(C.byref(cfg), C.byref(h))
        if code != 0:
            raise N.CgvcError(code, (self._lib.cgvc_last_error(None) or b"?").decode())
        self._handle = h
        nt, ne = C.c_int(0), C.c_size_t(0)
        self._chk(self._lib.cgvc_param_count(h, C.byref(nt), C.byref(ne)))
        self.n_params = ne.value
        self._table = OrderedDict()
        for i in range(nt.value):
            name, off, nd, shp = C.c_char_p(), C.c_size_t(), C.c_int(), (C.c_int * 4)()
            self._chk(self._lib.cgvc_param_info(h, i, C.byref(name), C.byref(off), C.byref(nd), C.byref(shp)))
            self._table[name.value.decode()] = (off.value, tuple(shp[k] for k in range(nd.value)))
        self._generator_end = max(o + int(np.prod(s)) for n, (o, s) in self._table.items() if 'generator' in n)
        if "deterministic" in self._options:                  # sizes WORK (its partials slab): set before the arenas are bound
            self._chk(self._lib.cgvc_set_option(h, b"deterministic", self._options["deterministic"]))
        kinds = [N.ARENA_PARAM, N.ARENA_WORK]
        if self.mode == 'train':
            kinds += [N.ARENA_GRAD, N.ARENA_ADAM_M, N.ARENA_ADAM_V]
        for kind in kinds:
            nbytes = C.c_size_t(0)
            self._chk(self._lib.cgvc_arena_bytes(h, kind, C.byref(nbytes)))
            old = self._arenas.get(kind)
            if kind == N.ARENA_WORK or old is None:
                t = torch.empty((nbytes.value + 3) // 4, dtype=torch.float32, device=self.device)
                if kind != N.ARENA_WORK:
                    t.zero_()
                self._arenas[kind] = t
            t = self._arenas[kind]
            self._chk(self._lib.cgvc_bind_arena(h, kind, _ptr(t), t.numel() * 4))
        self._losses = torch.zeros(8, dtype=torch.float32, device=self.device)
        self._losses_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self._ls_dev = torch.zeros(C.sizeof(N.LossScaleInfo), dtype=torch.uint8, device=self.device)
        self._ls_host = torch.zeros(C.sizeof(N.LossScaleInfo), dtype=torch.uint8).pin_memory()
        self._lsn_dev = torch.zeros(2 * C.sizeof(N.LossScaleNetInfo), dtype=torch.uint8, device=self.device)
        self._lsn_host = torch.zeros(2 * C.sizeof(N.LossScaleNetInfo), dtype=torch.uint8).pin_memory()
        self._staging = {}
        for name, value in self._options.items():            # the engine is re-created when batch / frames outgrow it
            self._chk(self._lib.cgvc_set_option(self._handle, name.encode(), int(value)))

    def set_option(self, name, value):
        """Engine options of include/cgvc.h (`two_streams`, `cuda_graph`, `fuse_in`, `fuse_bwd`, `debug_taps`, `loss_scale`, ...);
        remembered across engine re-creations."""
        self._chk(self._lib.cgvc_set_option(self._handle, name.encode(), int(value)))
        self._options[name] = int(value)
        if name == "tape_loss_scale":
            self._tape_dynamic = bool(value)
        if name == "deterministic":
            # the option changes the WORK plan: a larger arena is allocated and bound before the next call needs it
            nbytes = C.c_size_t(0)
            self._chk(self._lib.cgvc_arena_bytes(self._handle, N.ARENA_WORK, C.byref(nbytes)))
            work = self._arenas[N.ARENA_WORK]
            if nbytes.value > work.numel() * 4:
                torch.cuda.synchronize(self.device)                      # the old arena may still be read by enqueued work
                del work
                self._arenas.pop(N.ARENA_WORK)
                work = torch.empty((nbytes.value + 3) // 4, dtype=torch.float32, device=self.device)
                self._arenas[N.ARENA_WORK] = work
                self._chk(self._lib.cgvc_bind_arena(self._handle, N.ARENA_WORK, _ptr(work), work.numel() * 4))

    @property
    def loss_scale(self):
        """'static', 'monitor' or 'dynamic' (engine option "loss_scale")."""
        mode = self._options.get("loss_scale", 0)
        return next(k for k, v in N.LOSS_SCALE_MODES.items() if v == mode)

    @property
    def loss_scale_per_network(self):
        """engine option "loss_scale_per_network": a loss scale each for the generators and the discriminators"""
        return bool(self._options.get("loss_scale_per_network", 0))

    def _enqueue_loss_scale_state(self):
        self._chk(self._lib.cgvc_loss_scale_state(self._handle, _ptr(self._ls_dev), self._stream()))
        self._ls_host.copy_(self._ls_dev, non_blocking=True)
        if self.loss_scale_per_network:
            self._chk(self._lib.cgvc_loss_scale_net_state(self._handle, _ptr(self._lsn_dev), self._stream()))
            self._lsn_host.copy_(self._lsn_dev, non_blocking=True)

    def _read_loss_scale_state(self):
        """after the stream synchronisation that follows _enqueue_loss_scale_state"""
        info = N.LossScaleInfo.from_buffer_copy(self._ls_host.numpy().tobytes())
        self.last_loss_scale = {f: getattr(info, f) for f, _ in N.LossScaleInfo._fields_}
        self.last_loss_scale["last_skipped"] = bool(info.last_skipped)
        if self.loss_scale_per_network:
            nets = (N.LossScaleNetInfo * 2).from_buffer_copy(self._lsn_host.numpy().tobytes())
            for net, tag in zip(nets, ("G", "D")):
                self.last_loss_scale.update({"scale_" + tag: net.scale, "good_steps_" + tag: net.good_steps,
                                             "sat_grad_" + tag: net.sat_grad, "ufl_grad_" + tag: net.ufl_grad,
                                             "groups_" + tag: net.groups})
        self.last_step_skipped = self.last_loss_scale["last_skipped"]
        return dict(self.last_loss_scale)

    def loss_scale_state(self):
        """The loss scaler's state after the most recent step (synchronises): scale, good_steps, skipped, last_skipped and the last
        step's sat_grad / sat_act (saturated 4-value groups of the F16F8 gradient / activation planes) and nonfinite (bit 0: a
        generator gradient, bit 1: a discriminator gradient).  The counters are collected in 'monitor' and 'dynamic' mode only.
        With loss_scale_per_network also, per network (suffix _G the generators, _D the discriminators): scale, good_steps and the
        last step's sat_grad, ufl_grad (groups whose fp16 plane is subnormal or flushed) and groups (all counted)."""
        self._enqueue_loss_scale_state()
        torch.cuda.current_stream(self.device).synchronize()
        return self._read_loss_scale_state()

    def _ensure_capacity(self, batch, frames):
        if batch <= self._max_batch and frames <= self._max_frames:
            return
        step = C.c_longlong(0)
        self._lib.cgvc_get_adam_step(self._handle, C.byref(step))
        ls = self.loss_scale_state() if self.loss_scale == 'dynamic' else None
        self._lib.cgvc_destroy(self._handle)
        self._max_batch = max(batch, self._max_batch)
        self._max_frames = max(frames, self._max_frames)
        self._arenas.pop(N.ARENA_WORK, None)
        torch.cuda.empty_cache()
        self._create_engine()
        self._lib.cgvc_set_adam_step(self._handle, step)
        if ls is not None and ls["scale"] >= 1:
            self._chk(self._lib.cgvc_set_loss_scale_state(self._handle, ls["scale"], ls["good_steps"], ls["skipped"], self._stream()))
            if self.loss_scale_per_network:
                self._set_net_scales(ls)
        if self._data_parallel:
            # cgvc_destroy freed the NCCL communicator with the old engine: a data-parallel model must get a new one, or it would
            # silently train without the all-reduce.  Collective: every rank has to grow in the same call (same batch / frames).
            self._attach_communicator()
        else:
            self._params_updated()

    def _set_net_scales(self, ls):
        for k, tag in enumerate(("G", "D")):
            if ls.get("scale_" + tag, 0) >= 1:
                self._chk(self._lib.cgvc_set_loss_scale_net_state(self._handle, k, float(ls["scale_" + tag]),
                                                                  int(ls["good_steps_" + tag]), self._stream()))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _params_updated(self):
        self._chk(self._lib.cgvc_params_updated(self._handle, self._stream()))

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.cgvc_destroy(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    # ------------------------------------------------------------------ parameters
    def param_names(self):
        return list(self._table.keys())

    def _view(self, arena, name):
        off, shape = self._table[name]
        n = int(np.prod(shape))
        return self._arenas[arena][off:off + n].view(shape)

    def _init_params(self, seed):
        """glorot-uniform kernels, zero biases / beta, unit gamma (tf.get_variable defaults, Appendix A.3)."""
        gen = torch.Generator(device=self.device)
        gen.manual_seed(int(seed))
        for name, (off, shape) in self._table.items():
            v = self._view(N.ARENA_PARAM, name)
            if name.endswith("/kernel"):
                rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
                fan_in, fan_out = rf * shape[-2], rf * shape[-1]
                lim = math.sqrt(6.0 / (fan_in + fan_out))
                v.copy_((torch.rand(shape, generator=gen, device=self.device) * 2 - 1) * lim)
            elif name.endswith("/gamma"):
                v.fill_(1.0)
            else:
                v.zero_()
        self._params_updated()

    def get_params(self):
        """name -> numpy array (TF layouts)."""
        torch.cuda.synchronize(self.device)
        return OrderedDict((n, self._view(N.ARENA_PARAM, n).cpu().numpy()) for n in self._table)

    def set_params(self, params):
        """Inject weights (name -> array-like in TF layout); missing names keep their value."""
        for n, a in params.items():
            if n not in self._table:
                raise KeyError("unknown variable %r" % n)
            t = torch.as_tensor(np.asarray(a, dtype=np.float32))
            self._view(N.ARENA_PARAM, n).copy_(t.reshape(self._table[n][1]))
        self._params_updated()

    def get_grads(self):
        torch.cuda.synchronize(self.device)
        return OrderedDict((n, self._view(N.ARENA_GRAD, n).cpu().numpy()) for n in self._table)

    # ------------------------------------------------------------------ differentiable networks (activation tapes)
    def generator(self, x, direction):
        """Differentiable generator forward: x a CUDA tensor [batch, 24, frames] (frames a multiple of 4) -> [batch, 24, frames], bit
        for bit what test() gives.  Its backward adds d loss / d (the generator's variables) into the gradient arena (grads()) and
        returns d loss / d x.  direction 'A2B' or 'B2A'."""
        return _NetFn.apply(x, self._token(), self, 0, _direction(direction))

    def discriminator(self, x, which):
        """Differentiable discriminator forward: x a CUDA tensor [batch, 24, frames] (frames a multiple of 16) -> probabilities
        [batch, 6, frames / 16, 1] as discriminate() gives them.  Backward as generator().  which 'A' or 'B'."""
        w = {'A': 0, 'B': 1}.get(which)
        if w is None:
            raise ValueError("which must be 'A' or 'B', got %r" % (which,))
        return _NetFn.apply(x, self._token(), self, 1, w)

    def generator_packed(self, inputs, direction):
        """Differentiable packed generator: inputs a list of CUDA tensors [24, T_i] (every T_i a positive multiple of 4) -> the list of
        converted [24, T_i] tensors, bit for bit what test_packed() gives on them.  One engine call runs the forward of all utterances and
        one their backward, which adds d loss / d (the generator's variables) into the gradient arena -- with the loss scale of a batch
        of len(inputs), tape_loss_scale(len(inputs)) -- and returns d loss / d x_i for the inputs that require it.  Every convolution
        tap, instance norm and edge-layer sum stays inside its own utterance, forward and backward.  direction 'A2B' or 'B2A'."""
        d = _direction(direction)
        inputs = list(inputs)
        if not inputs:
            return []
        return list(_PackedFn.apply(self._token(), self, 2, d, *inputs))

    def discriminator_packed(self, inputs, which):
        """Differentiable packed discriminator: inputs a list of CUDA tensors [24, T_i] (every T_i a positive multiple of 16) -> the
        list of [6, T_i / 16, 1] probabilities, bit for bit what discriminate_packed() gives on them.  One engine call runs the forward
        of all utterances and one their backward, which adds d loss / d (the discriminator's variables) into the gradient arena -- with
        the loss scale of a batch of len(inputs) -- and returns d loss / d x_i for the inputs that require it.  Every convolution tap and
        instance norm stays inside its own utterance, forward and backward, so the output of generator_packed() chains straight in.
        which 'A' or 'B'."""
        w = {'A': 0, 'B': 1}.get(which)
        if w is None:
            raise ValueError("which must be 'A' or 'B', got %r" % (which,))
        inputs = list(inputs)
        if not inputs:
            return []
        return list(_PackedFn.apply(self._token(), self, 3, w, *inputs))

    def _token(self):
        # a leaf that requires grad, so that autograd runs a network's backward -- and with it the weight gradients -- even when its
        # input does not require grad (a real sample)
        if self._grad_token is None:
            self._grad_token = torch.zeros(0, device=self.device, requires_grad=True)
        return self._grad_token

    def tape_loss_scale(self, batch):
        """The factor the tape backward calls of a `batch`-sample application leave in the gradient arena: the static loss scale of the
        F16F8 gradient planes, 2^(9 + min(floor(log2 batch), 9)), and 1 in the other precisions (include/cgvc.h cgvc_adam_step).
        With tape_loss_scale='dynamic' the tapes use the scaler's current scale instead, which only the device knows: grads() and
        apply_gradients() remove it there."""
        if self._tape_dynamic:
            raise RuntimeError("tape_loss_scale='dynamic': the tapes use the loss scaler's scale, not a static one; grads() and "
                               "apply_gradients() remove it on the device")
        if N.PRECISIONS[self.precision] != N.PREC_F16F8:
            return 1.0
        return float(2 ** (9 + min(int(batch).bit_length() - 1, 9)))

    def _tape_forward(self, kind, which, x):
        """x [batch, 24, frames] through the generator (kind 0) or the discriminator (kind 1), with its activation tape: (y, tape)."""
        if not (isinstance(x, torch.Tensor) and x.device.type == self.device.type):
            raise TypeError("the differentiable networks take a tensor on the engine's device (%s)" % self.device)
        x = x.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if x.dim() != 3 or x.shape[1] != self.num_features:
            raise ValueError("expected [batch, %d, frames], got %r" % (self.num_features, tuple(x.shape)))
        batch, _, frames = x.shape
        self._ensure_capacity(batch, frames)
        if kind == 1:
            y = torch.empty((batch, self.num_features // 4, frames // 16, 1), dtype=torch.float32, device=self.device)
        else:
            y = torch.empty_like(x)
        return y, self._tape_call(kind, which, x, y, batch, frames, (batch, frames))

    def _packed_tape_forward(self, which, xs, kind=2):
        """The [24, T_i] utterances xs through the generator (kind 2) or the discriminator (kind 3) in one call, with its activation
        tape: (ys, tape, offsets)."""
        for x in xs:
            if not (isinstance(x, torch.Tensor) and x.device.type == self.device.type):
                raise TypeError("the differentiable networks take a tensor on the engine's device (%s)" % self.device)
        offsets = self._packed_offsets(xs)
        x = self._pack(xs)
        y = torch.empty_like(x) if kind == 2 else torch.empty(self.num_features // 4 * int(offsets[-1]) // 16, device=self.device)
        n = len(offsets) - 1
        tape = self._tape_call(kind, which, x, y, n, int(offsets[-1]), (offsets.ctypes.data_as(C.POINTER(C.c_longlong)), n))
        return (self._unpack(y, offsets) if kind == 2 else self._unpack_prob(y, offsets)), tape, offsets

    def _unpack_prob(self, p, offsets):
        """The [6, T_i / 16, 1] probabilities of packed utterances in p, as views"""
        H = self.num_features // 4
        return [p[H * offsets[u] // 16:H * offsets[u + 1] // 16].reshape(H, -1, 1) for u in range(len(offsets) - 1)]

    def _tape_call(self, kind, which, x, y, batch, frames, geom):
        """A tape of `kind` sized by cgvc_tape_bytes(batch, frames) (kind 2: n utterances of offsets[n] frames in all), written by that
        kind's forward from x to y; geom: the forward's geometry arguments.  The caching allocator aligns the tape to 512 bytes."""
        nbytes = C.c_size_t(0)
        self._chk(self._lib.cgvc_tape_bytes(self._handle, kind, batch, frames, C.byref(nbytes)))
        tape = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
        fn = getattr(self._lib, ("cgvc_generator_forward_tape", "cgvc_discriminator_forward_tape",
                                 "cgvc_generator_forward_packed_tape", "cgvc_discriminator_forward_packed_tape")[kind])
        self._chk(fn(self._handle, which, _ptr(x), _ptr(y), *geom, _ptr(tape), nbytes.value, self._stream()))
        return tape

    def _tape_backward(self, kind, tape, geom, dy, want_dx):
        """d loss / d x of a tape's application from d loss / d y, or None without want_dx; adds the network's variable gradients into
        the gradient arena.  geom: x's shape, or for a packed tape (kinds 2, 3) the utterances' offsets, with dy and d x lists of their
        blocks."""
        if kind in (2, 3):
            dy = self._pack(dy)
            x_shape, batch = (self.num_features * int(geom[-1]),), len(geom) - 1
        else:
            dy = dy.to(device=self.device, dtype=torch.float32).contiguous()
            x_shape, batch = geom, geom[0]
        dx = torch.empty(x_shape, dtype=torch.float32, device=self.device) if want_dx else None
        fn = self._lib.cgvc_discriminator_backward_tape if kind in (1, 3) else self._lib.cgvc_generator_backward_tape
        self._chk(fn(self._handle, _ptr(tape), _ptr(dy), _ptr(dx), self._stream()))
        if not self._tape_dynamic:
            self._tape_scales.add(self.tape_loss_scale(batch))
        if kind not in (2, 3):
            return dx
        return self._unpack(dx, geom) if want_dx else [None] * batch

    def zero_grad(self, network=None):
        """Zero the gradient arena before the backward passes of a new step; with network ('generator_A2B', ..., 'discriminator_B')
        only that network's variables -- e.g. a discriminator's after the generator loss was back-propagated through it, since its
        optimizer follows the discriminator loss alone (model.py:107-108)."""
        if network is None:
            self._arenas[N.ARENA_GRAD].zero_()
            self._tape_scales.clear()
            self._grads_applied = False
            return
        names = [n for n in self._table if n.startswith(network + "/")]
        if not names:
            raise KeyError("no network %r" % (network,))
        for n in names:
            self._view(N.ARENA_GRAD, n).zero_()

    def grads(self, network=None):
        """name -> d loss / d variable (TF layout) as the tape backward calls since zero_grad() accumulated it, on the device, with
        their loss scale removed: views of the gradient arena when that scale is 1, else scaled copies -- read them, do not write
        them.  network: 'generator_A2B', 'generator_B2A', 'discriminator_A' or 'discriminator_B' (None: all four).
        With tape_loss_scale='dynamic': copies divided by the scaler's current scale -- per network with loss_scale_per_network --
        on the device, without a host synchronisation; refused after apply_gradients() until zero_grad(), since a skipped step has
        already halved the scale the arena was formed with."""
        if self._tape_dynamic:
            if self._grads_applied:
                raise RuntimeError("grads() after apply_gradients(): the loss scale may have changed since the gradient arena was formed; "
                                   "read grads() before apply_gradients(), and zero_grad() starts the next step")
            s_gen, s_disc = self._device_scales()
        else:
            s = self._grad_scale()
        out = OrderedDict()
        for n in self._table:
            if network is None or n.startswith(network + "/"):
                v = self._view(N.ARENA_GRAD, n).detach()
                if self._tape_dynamic:
                    out[n] = v / (s_gen if n.startswith("generator") else s_disc)
                else:
                    out[n] = v if s == 1.0 else v * s
        if not out:
            raise KeyError("no network %r" % (network,))
        return out

    def _device_scales(self):
        """The scaler's current scales of the generators' and the discriminators' gradients as device tensors, enqueued on the
        current stream (no synchronisation).  Before the first tape backward sets the scaler they read 0, taken as 1."""
        self._chk(self._lib.cgvc_loss_scale_state(self._handle, _ptr(self._ls_dev), self._stream()))
        s = self._ls_dev[:4].view(torch.float32).clamp_min(1.0)
        if not (self.loss_scale_per_network and N.PRECISIONS[self.precision] == N.PREC_F16F8):
            return s, s
        self._chk(self._lib.cgvc_loss_scale_net_state(self._handle, _ptr(self._lsn_dev), self._stream()))
        k = C.sizeof(N.LossScaleNetInfo)
        return self._lsn_dev[:4].view(torch.float32).clamp_min(1.0), self._lsn_dev[k:k + 4].view(torch.float32).clamp_min(1.0)

    def _grad_scale(self):
        if len(self._tape_scales) > 1:
            raise RuntimeError("the gradient arena mixes tape backward calls of different loss scales (batches %s): zero_grad() between "
                               "batches whose scales differ" % sorted(self._tape_scales))
        return 1.0 / next(iter(self._tape_scales)) if self._tape_scales else 1.0

    def adam_step(self, generator_learning_rate, discriminator_learning_rate):
        """One Adam update of all four networks (model.py:107-108) from the gradient arena that the tape backward calls filled, with
        their loss scale removed; advances the Adam step count like train().  It never skips a step, and with data_parallel=True it
        does not all-reduce the gradient arena: replicas that call it drift apart.  tape_loss_scale='dynamic' takes
        apply_gradients() instead, which does both."""
        if self._tape_dynamic:
            raise RuntimeError("tape_loss_scale='dynamic': use apply_gradients(), which removes the device loss scale and skips "
                               "overflowing steps")
        self._chk(self._lib.cgvc_adam_step(self._handle, float(generator_learning_rate), float(discriminator_learning_rate),
                                           self._grad_scale(), self._stream()))
        self.train_step += 1

    def apply_gradients(self, generator_learning_rate, discriminator_learning_rate):
        """The train step's optimizer tail over the gradient arena that the tape backward calls filled (tape_loss_scale='dynamic';
        include/cgvc.h cgvc_apply_gradients): with data_parallel=True the all-reduce, then the non-finite check and the loss-scale
        update, then Adam with the scale removed -- or, on overflow, a skipped step and a halved scale.  Enqueued without a host
        synchronisation; loss_scale_state() reports skipped and the scales as after train().  Advances train_step like train()."""
        if not self._tape_dynamic:
            raise RuntimeError("apply_gradients() needs tape_loss_scale='dynamic'; static tapes take adam_step()")
        self._chk(self._lib.cgvc_apply_gradients(self._handle, float(generator_learning_rate), float(discriminator_learning_rate),
                                                 self._stream()))
        self._grads_applied = True
        self.train_step += 1

    # ------------------------------------------------------------------ data parallel
    def _attach_communicator(self):
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("data_parallel=True needs torch.distributed to be initialised (one process per GPU)")
        rank, world = dist.get_rank(), dist.get_world_size()
        idbuf = (C.c_char * 128)()
        if rank == 0:
            self._chk(self._lib.cgvc_comm_unique_id(self._handle, idbuf))
        obj = [bytes(idbuf)]
        dist.broadcast_object_list(obj, src=0)
        idbuf = (C.c_char * 128).from_buffer_copy(obj[0])
        self._chk(self._lib.cgvc_comm_init(self._handle, idbuf, rank, world))
        self._rank, self._nranks = rank, world
        # every replica must start from identical weights: broadcast rank 0's parameter arena
        dist.broadcast(self._arenas[N.ARENA_PARAM], src=0)
        self._params_updated()

    # ------------------------------------------------------------------ staging
    def _to_device(self, x, key):
        """Host array (any float dtype, model.py feeds float64) or CUDA tensor -> fp32 CUDA tensor [B,F,T]."""
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.to(dtype=torch.float32).contiguous()
        a = np.asarray(x)
        if a.ndim != 3 or a.shape[1] != self.num_features:
            raise ValueError("expected [batch, %d, frames], got %r" % (self.num_features, a.shape))
        return self._stage([a], key).view(a.shape)

    def _stage(self, arrays, key):
        """Host arrays (any float dtype) -> one fp32 CUDA tensor holding them back to back, through the pinned buffer kept for `key`."""
        n = sum(a.size for a in arrays)
        st = self._staging.get(key)
        if st is None or st[0].numel() != n:
            st = (torch.empty(n, dtype=torch.float32).pin_memory(), torch.empty(n, dtype=torch.float32, device=self.device))
            self._staging[key] = st
        hv, o = st[0].numpy(), 0
        for a in arrays:                  # cast to fp32 at the boundary, like the placeholder feed (model.py:35-42)
            hv[o:o + a.size] = a.reshape(-1)
            o += a.size
        st[1].copy_(st[0], non_blocking=True)
        return st[1]

    def _pack(self, tensors):
        """Tensors on the engine's device -> one fp32 tensor holding them back to back (the packed utterance layout)."""
        return torch.cat([t.detach().to(device=self.device, dtype=torch.float32).reshape(-1) for t in tensors])

    def _unpack(self, y, offsets):
        """The [24, T_i] utterances of a packed tensor or array y, as views."""
        F = self.num_features
        return [y[F * offsets[u]:F * offsets[u + 1]].reshape(F, -1) for u in range(len(offsets) - 1)]

    def _result(self, y, on_device):
        """A result on the device as it is, or for host inputs as a float32 numpy array (synchronises)."""
        if on_device:
            return y
        out = torch.empty(y.shape, dtype=torch.float32).pin_memory()
        out.copy_(y, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return out.numpy().copy()

    # ------------------------------------------------------------------ the reference API
    def train(self, input_A, input_B, lambda_cycle, lambda_identity, generator_learning_rate, discriminator_learning_rate):
        """One G step + one D step from the same pre-update weights (model.py:110-125).
        Returns (generator_loss, discriminator_loss) as fp32 scalars (pre-update values)."""
        A = self._to_device(input_A, "A")
        B = self._to_device(input_B, "B")
        if A.shape != B.shape:
            raise ValueError("input_A and input_B must have the same shape")
        batch, _, frames = A.shape
        self._ensure_capacity(batch, frames)
        self._chk(self._lib.cgvc_train_step(self._handle, _ptr(A), _ptr(B), batch, frames,
                                            float(lambda_cycle), float(lambda_identity),
                                            float(generator_learning_rate), float(discriminator_learning_rate),
                                            None, None, _ptr(self._losses), self._stream()))
        self._losses_host.copy_(self._losses, non_blocking=True)
        monitored = self.loss_scale != 'static'
        if monitored:
            self._enqueue_loss_scale_state()
        torch.cuda.current_stream(self.device).synchronize()
        if monitored:
            self._read_loss_scale_state()
        l = self._losses_host.numpy()
        self.last_losses = {k: float(v) for k, v in zip(N.LOSS_NAMES, l)}
        if self.writer is not None and self.summary_interval and self.train_step % self.summary_interval == 0:
            self._write_summaries()
        self.train_step += 1
        return np.float32(l[4]), np.float32(l[7])

    def train_async(self, A_dev, B_dev, lambda_cycle, lambda_identity, generator_learning_rate, discriminator_learning_rate):
        """Device-resident variant: enqueue one step, no host synchronisation.  Losses land in self._losses."""
        batch, _, frames = A_dev.shape
        self._chk(self._lib.cgvc_train_step(self._handle, _ptr(A_dev), _ptr(B_dev), batch, frames,
                                            float(lambda_cycle), float(lambda_identity),
                                            float(generator_learning_rate), float(discriminator_learning_rate),
                                            None, None, _ptr(self._losses), self._stream()))
        self.train_step += 1

    def fetch_losses(self):
        """(generator_loss, discriminator_loss) of the most recent train_async step: the one device -> host read (32 bytes) and stream
        synchronisation a device-resident training loop needs, at the steps it logs."""
        self._losses_host.copy_(self._losses, non_blocking=True)
        monitored = self.loss_scale != 'static'
        if monitored:
            self._enqueue_loss_scale_state()
        torch.cuda.current_stream(self.device).synchronize()
        if monitored:
            self._read_loss_scale_state()
        l = self._losses_host.numpy()
        self.last_losses = {k: float(v) for k, v in zip(N.LOSS_NAMES, l)}
        if self.writer is not None and self.summary_interval:
            self._write_summaries()
        return np.float32(l[4]), np.float32(l[7])

    def compute_gradients(self, input_A, input_B, lambda_cycle, lambda_identity):
        """Forward + backward only (what the two `minimize` calls differentiate, model.py:107-108).
        Returns (losses dict, generation_A, generation_B); gradients via get_grads()."""
        A = self._to_device(input_A, "A"); B = self._to_device(input_B, "B")
        batch, _, frames = A.shape
        self._ensure_capacity(batch, frames)
        gA = torch.empty_like(A); gB = torch.empty_like(B)
        self._chk(self._lib.cgvc_compute_gradients(self._handle, _ptr(A), _ptr(B), batch, frames, float(lambda_cycle),
                                                   float(lambda_identity), _ptr(gA), _ptr(gB), _ptr(self._losses), self._stream()))
        torch.cuda.synchronize(self.device)
        l = self._losses.cpu().numpy()
        return {k: float(v) for k, v in zip(N.LOSS_NAMES, l)}, gA.cpu().numpy(), gB.cpu().numpy()

    def test(self, inputs, direction):
        """Generator forward (model.py:128-137).  inputs [B, 24, T] with T a multiple of 4."""
        d = _direction(direction)
        x = self._to_device(inputs, "test")
        batch, _, frames = x.shape
        self._ensure_capacity(batch, frames)
        y = torch.empty_like(x)
        self._chk(self._lib.cgvc_generator_forward(self._handle, d, _ptr(x), _ptr(y), batch, frames, self._stream()))
        return self._result(y, isinstance(inputs, torch.Tensor) and inputs.is_cuda)

    def test_packed(self, inputs, direction):
        """Generator forward of utterances of different lengths in one engine call.  inputs: a list of [24, T_i] arrays, every
        T_i a positive multiple of 4: host arrays of any float dtype (returns a list of float32 numpy arrays) or CUDA tensors
        (returns a list of CUDA tensors).  Each result is what test() gives for that utterance alone, up to the summation order
        of its instance-norm statistics."""
        d = _direction(direction)
        if len(inputs) == 0:
            return []
        on_device = all(isinstance(x, torch.Tensor) and x.is_cuda for x in inputs)
        offsets = self._packed_offsets(inputs)
        x = self._pack(inputs) if on_device else self._stage([np.asarray(a) for a in inputs], "test_packed")
        y = torch.empty_like(x)
        off = offsets.ctypes.data_as(C.POINTER(C.c_longlong))
        self._chk(self._lib.cgvc_generator_forward_packed(self._handle, d, _ptr(x), _ptr(y), off, len(offsets) - 1, self._stream()))
        return self._unpack(self._result(y, on_device), offsets)

    def _packed_offsets(self, inputs):
        """the n + 1 frame offsets of packed [24, T_i] utterances; grows the engine to hold them"""
        for x in inputs:
            if len(x.shape) != 2 or x.shape[0] != self.num_features:
                raise ValueError("expected [%d, frames] utterances, got %r" % (self.num_features, tuple(x.shape)))
        offsets = np.cumsum([0] + [int(x.shape[1]) for x in inputs], dtype=np.int64)
        n, total = len(inputs), int(offsets[-1])
        if n > self._max_batch or total > self._max_batch * self._max_frames:
            batch = max(n, self._max_batch)
            self._ensure_capacity(batch, max(self._max_frames, -(-total // (4 * batch)) * 4))
        return offsets

    def discriminate(self, inputs, which):
        """Discriminator forward (module.py:188-213): which in {'A','B'}; returns [B, 6, T/16, 1]."""
        x = self._to_device(inputs, "disc")
        batch, _, frames = x.shape
        self._ensure_capacity(batch, frames)
        y = torch.empty((batch, self.num_features // 4, frames // 16, 1), dtype=torch.float32, device=self.device)
        self._chk(self._lib.cgvc_discriminator_forward(self._handle, {'A': 0, 'B': 1}[which], _ptr(x), _ptr(y), batch, frames, self._stream()))
        torch.cuda.synchronize(self.device)
        return y.cpu().numpy()

    def discriminate_packed(self, inputs, which):
        """Discriminator forward of utterances of different lengths in one engine call.  inputs: a list of [24, T_i] arrays, every
        T_i a positive multiple of 16: host arrays of any float dtype (returns a list of float32 numpy arrays) or CUDA tensors
        (returns a list of CUDA tensors).  Result i is [6, T_i / 16, 1], what discriminate() gives for that utterance alone, up to
        the summation order of its instance-norm statistics."""
        w = {'A': 0, 'B': 1}[which]
        if len(inputs) == 0:
            return []
        on_device = all(isinstance(x, torch.Tensor) and x.is_cuda for x in inputs)
        offsets = self._packed_offsets(inputs)
        x = self._pack(inputs) if on_device else self._stage([np.asarray(a) for a in inputs], "disc_packed")
        H = self.num_features // 4
        p = torch.empty(H * int(offsets[-1]) // 16, dtype=torch.float32, device=self.device)
        off = offsets.ctypes.data_as(C.POINTER(C.c_longlong))
        self._chk(self._lib.cgvc_discriminator_forward_packed(self._handle, w, _ptr(x), _ptr(p), off, len(offsets) - 1, self._stream()))
        return self._unpack_prob(self._result(p, on_device), offsets)

    def set_debug_taps(self, on=True):
        """Keep the fp32 copy of every generator layer output of the next test() calls for debug_activation() (parity tests).
        Off by default: the conversion path then writes only what the next layer reads."""
        self.set_option("debug_taps", 1 if on else 0)

    def debug_activation(self, name):
        n = C.c_size_t(0)
        self._chk(self._lib.cgvc_debug_activation(self._handle, name.encode(), None, 0, C.byref(n), self._stream()))
        out = torch.empty(n.value, dtype=torch.float32, device=self.device)
        self._chk(self._lib.cgvc_debug_activation(self._handle, name.encode(), _ptr(out), n.value, C.byref(n), self._stream()))
        torch.cuda.synchronize(self.device)
        return out.cpu().numpy()

    def save(self, directory, filename):
        """model.py:140-146.  Writes <directory>/<filename>.npz keyed by TF variable names; returns the joined path."""
        if not os.path.exists(directory):
            os.makedirs(directory)
        path = os.path.join(directory, filename)
        torch.cuda.synchronize(self.device)
        blob = {}
        for n in self._table:
            blob[n] = self._view(N.ARENA_PARAM, n).cpu().numpy()
            if self.mode == 'train':
                blob[n + "/Adam"] = self._view(N.ARENA_ADAM_M, n).cpu().numpy()
                blob[n + "/Adam_1"] = self._view(N.ARENA_ADAM_V, n).cpu().numpy()
        step = C.c_longlong(0)
        self._lib.cgvc_get_adam_step(self._handle, C.byref(step))
        blob["adam_step"] = np.int64(step.value)
        if self.loss_scale != 'static':
            ls = self.loss_scale_state()
            blob["loss_scale"] = np.float32(ls["scale"])
            blob["loss_scale_good_steps"] = np.int64(ls["good_steps"])
            blob["loss_scale_skipped"] = np.int64(ls["skipped"])
            for tag in ("G", "D") if self.loss_scale_per_network else ():
                blob["loss_scale_" + tag] = np.float32(ls["scale_" + tag])
                blob["loss_scale_good_steps_" + tag] = np.int64(ls["good_steps_" + tag])
        blob["train_step"] = np.int64(self.train_step)
        with open(path + ".npz" if not path.endswith(".npz") else path, "wb") as f:
            np.savez(f, **blob)
        return path

    def load(self, filepath):
        """model.py:148-150.  Accepts this engine's `.npz` checkpoints and TensorFlow V2 bundles written by the reference's
        `tf.train.Saver` (`<filepath>.index` + `<filepath>.data-*`, e.g. the SF1-TM1 model the reference's README publishes):
        the variable names are the same in both."""
        from . import tf_checkpoint as tfc
        if tfc.is_bundle(filepath):
            return self._load_tf_bundle(filepath)
        p = filepath if filepath.endswith(".npz") else filepath + ".npz"
        z = np.load(p)
        for n in self._table:
            self._view(N.ARENA_PARAM, n).copy_(torch.from_numpy(z[n]))
            if self.mode == 'train' and (n + "/Adam") in z:
                self._view(N.ARENA_ADAM_M, n).copy_(torch.from_numpy(z[n + "/Adam"]))
                self._view(N.ARENA_ADAM_V, n).copy_(torch.from_numpy(z[n + "/Adam_1"]))
        if "adam_step" in z:
            self._lib.cgvc_set_adam_step(self._handle, int(z["adam_step"]))
        if "train_step" in z:
            self.train_step = int(z["train_step"])
        if self.loss_scale == 'dynamic' and "loss_scale" in z and float(z["loss_scale"]) >= 1:
            # a single-scale checkpoint sets both networks' scales; a per-network one then sets each
            self._chk(self._lib.cgvc_set_loss_scale_state(self._handle, float(z["loss_scale"]), int(z["loss_scale_good_steps"]),
                                                          int(z["loss_scale_skipped"]), self._stream()))
            if self.loss_scale_per_network:
                ls = {}
                for tag in ("G", "D"):
                    if "loss_scale_" + tag in z:
                        ls["scale_" + tag] = float(z["loss_scale_" + tag])
                        ls["good_steps_" + tag] = int(z["loss_scale_good_steps_" + tag])
                self._set_net_scales(ls)
        self._params_updated()

    def _load_tf_bundle(self, prefix):
        from . import tf_checkpoint as tfc
        want = set(self._table)
        if self.mode == 'train':
            want |= {n + s for n in self._table for s in ("/Adam", "/Adam_1")} | {"beta2_power", "beta2_power_1"}
        t = tfc.read_checkpoint(prefix, names=want)
        missing = [n for n in self._table if n not in t]
        if missing:
            raise KeyError("TensorFlow checkpoint %s lacks %d variables, e.g. %s" % (prefix, len(missing), missing[0]))
        for n, (off, shape) in self._table.items():
            a = np.asarray(t[n], dtype=np.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError("%s: checkpoint shape %r, expected %r" % (n, a.shape, shape))
            self._view(N.ARENA_PARAM, n).copy_(torch.from_numpy(a))
            if self.mode == 'train' and (n + "/Adam") in t and (n + "/Adam_1") in t:
                self._view(N.ARENA_ADAM_M, n).copy_(torch.from_numpy(np.asarray(t[n + "/Adam"], dtype=np.float32)))
                self._view(N.ARENA_ADAM_V, n).copy_(torch.from_numpy(np.asarray(t[n + "/Adam_1"], dtype=np.float32)))
        if self.mode == 'train' and "beta2_power" in t:
            # tf.train.AdamOptimizer keeps beta2^t (Appendix A.6): recover the step count both optimizers share
            b2p = float(np.asarray(t["beta2_power"]).reshape(-1)[0])
            if 0.0 < b2p < 1.0:
                self._lib.cgvc_set_adam_step(self._handle, int(round(math.log(b2p) / math.log(0.999))))
            elif b2p <= 0.0:
                # beta2^t underflows fp32 after ~87k steps: any large t gives the same (unit) bias correction
                self._lib.cgvc_set_adam_step(self._handle, 1000000)
        self._params_updated()

    def summary(self):
        """model.py:153-169: the same 8 scalar tags, written every `summary_interval` steps."""
        try:
            from torch.utils.tensorboard import SummaryWriter
            self.writer = SummaryWriter(self.log_dir)
        except Exception:
            self.writer = None
        g = ['generator_summaries/' + n for n in N.LOSS_NAMES[:5]]
        d = ['discriminator_summaries/' + n for n in N.LOSS_NAMES[5:]]
        return g, d

    def _write_summaries(self):
        for n, v in self.last_losses.items():
            scope = 'generator_summaries/' if not n.startswith('discriminator') else 'discriminator_summaries/'
            self.writer.add_scalar(scope + n, v, self.train_step)


class _NetFn(torch.autograd.Function):
    """One network application (kind 0 generator, 1 discriminator) with its activation tape: forward writes it, backward consumes it
    (the tape is not modified, so retain_graph backward passes each add their gradients again)."""

    @staticmethod
    def forward(ctx, x, token, model, kind, which):
        y, tape = model._tape_forward(kind, which, x)
        ctx.model, ctx.kind, ctx.x_shape = model, kind, tuple(x.shape)
        ctx.save_for_backward(tape)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        tape, = ctx.saved_tensors
        dx = ctx.model._tape_backward(ctx.kind, tape, ctx.x_shape, dy, ctx.needs_input_grad[0])
        return dx, None, None, None, None


class _PackedFn(torch.autograd.Function):
    """One packed application over utterances of different lengths -- the generator (kind 2, CycleGAN.generator_packed) or the
    discriminator (kind 3, CycleGAN.discriminator_packed) -- with its activation tape: forward writes it, backward consumes it
    (unmodified, as _NetFn's)"""

    @staticmethod
    def forward(ctx, token, model, kind, which, *xs):
        ys, tape, offsets = model._packed_tape_forward(which, xs, kind)
        ctx.model, ctx.kind, ctx.offsets = model, kind, offsets
        ctx.save_for_backward(tape)
        return tuple(ys)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *dys):
        tape, = ctx.saved_tensors
        want = ctx.needs_input_grad[4:]
        dxs = ctx.model._tape_backward(ctx.kind, tape, ctx.offsets, dys, any(want))
        return (None, None, None, None) + tuple(dx if w else None for dx, w in zip(dxs, want))
