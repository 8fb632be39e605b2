"""Network descriptors and eager network operators: the host-side mirror of the reference's `module.py`.

In the reference, `generator_gatedcnn` (module.py:148-185) and `discriminator` (module.py:188-213) are graph-building
callables that (a) are injected into `CycleGAN(...)` (model.py:9,14-15) and (b) create their variables under a TF variable
scope on the first call and reuse them on later calls (`reuse=True`).  Here each of them is a `_NetDescriptor`:

  * `layers` is the architecture table (one row per block of module.py).  `variables(num_features)` expands it into the TF
    variable names / shapes in creation order (SURVEY.md Appendix A.4/A.5).  `CycleGAN.__init__` checks that expansion
    against the parameter table of the native engine (cgvc_param_info) and refuses a descriptor that describes anything
    else -- the engine implements exactly these two architectures (csrc/engine.cu build_generator / build_discriminator),
    and the descriptor is how the host states which one it expects.
  * calling it, `generator_gatedcnn(inputs, reuse=False, scope_name=...)`, is the eager operator: it runs the native
    network on `inputs` ([batch, 24, frames], numpy or CUDA tensor) with the variables of `scope_name`, created
    (glorot-uniform, like tf.get_variable's default) on the first call and reused with `reuse=True`, with TF's error
    behaviour for the two misuse cases.  `scope_variables` / `assign_scope_variables` read and inject those variables.
    Given a numpy array it returns one; given a CUDA tensor it returns a CUDA tensor that autograd differentiates through the native
    network (CycleGAN.generator / CycleGAN.discriminator): its backward returns d inputs and adds the scope's variable gradients up,
    which `scope_gradients` reads and `zero_scope_gradients` clears.
"""
from __future__ import annotations

from collections import OrderedDict


def _inorm(idx):
    return "InstanceNorm" if idx == 0 else "InstanceNorm_%d" % idx


class _NetDescriptor:
    def __init__(self, name, kind, layers):
        self.__name__ = name
        self.kind = kind              # 'generator' | 'discriminator'
        self.layers = layers          # rows: (block type, name / name prefix, kernel, strides, filters[, shuffle])

    # ------------------------------------------------------------------ the table the engine is checked against
    def variables(self, num_features=24):
        """[(TF variable name relative to the network scope, shape)] in creation order."""
        out, idx = [], 0
        cin = num_features if self.kind == "generator" else 1
        for row in self.layers:
            typ, name, k, filters = row[0], row[1], row[2], row[4]
            kshape = (list(k) if isinstance(k, (tuple, list)) else [k]) if k is not None else None
            if typ == "gated":                   # conv || conv_gates -> GLU (no norm): module.py:159-161, 199-201
                for suffix in ("", "_gates"):
                    out.append((name + suffix + "/kernel", tuple(kshape + [cin, filters])))
                    out.append((name + suffix + "/bias", (filters,)))
                cin = filters
            elif typ in ("gated_in", "gated_in_shuffle"):     # conv -> IN || gates -> IN -> GLU: module.py:85-133
                cn = filters // 2 if typ == "gated_in_shuffle" else filters       # IN runs after the pixel shuffle (module.py:124-125)
                for conv in ("h1_conv", "h1_gates"):
                    out.append((name + conv + "/kernel", tuple(kshape + [cin, filters])))
                    out.append((name + conv + "/bias", (filters,)))
                    out.append((_inorm(idx) + "/beta", (cn,))); out.append((_inorm(idx) + "/gamma", (cn,))); idx += 1
                cin = cn
            elif typ == "residual":              # module.py:66-83: gated_in (filters) then h2_conv (filters // 2) + IN, added to the input
                for conv in ("h1_conv", "h1_gates"):
                    out.append((name + conv + "/kernel", tuple(kshape + [cin, filters])))
                    out.append((name + conv + "/bias", (filters,)))
                    out.append((_inorm(idx) + "/beta", (filters,))); out.append((_inorm(idx) + "/gamma", (filters,))); idx += 1
                out.append((name + "h2_conv/kernel", tuple(kshape + [filters, filters // 2])))
                out.append((name + "h2_conv/bias", (filters // 2,)))
                out.append((_inorm(idx) + "/beta", (filters // 2,))); out.append((_inorm(idx) + "/gamma", (filters // 2,))); idx += 1
                cin = filters // 2
            elif typ == "conv":                  # plain convolution (o1_conv, module.py:182); filters None = num_features
                f = num_features if filters is None else filters
                out.append((name + "/kernel", tuple(kshape + [cin, f]))); out.append((name + "/bias", (f,)))
                cin = f
            elif typ == "dense":                 # tf.layers.dense (module.py:211)
                out.append((name + "/kernel", (cin, filters))); out.append((name + "/bias", (filters,)))
                cin = filters
            else:
                raise ValueError("unknown block type %r" % (typ,))
        return out

    def check_engine_table(self, table, scope, num_features=24):
        """Raise if the native engine's parameter table for `scope` is not this descriptor's architecture."""
        want = [(scope + "/" + n, tuple(s)) for n, s in self.variables(num_features)]
        got = [(n, tuple(s)) for n, (_, s) in table.items() if n.startswith(scope + "/")]
        if want != got:
            bad = next((w, g) for w, g in zip(want + [None] * len(got), got + [None] * len(want)) if w != g)
            raise ValueError("%s does not describe the network the native engine implements for scope %r: first difference %r vs %r"
                             % (self.__name__, scope, bad[0], bad[1]))

    # ------------------------------------------------------------------ the eager operator
    def __call__(self, inputs, reuse=False, scope_name=None):
        return _apply(self, inputs, reuse, scope_name or self.__name__)

    def __repr__(self):
        return "<native %s descriptor: %s, %d blocks>" % (self.kind, self.__name__, len(self.layers))


# module.py:159-183  (type, name / prefix, kernel, stride, filters)
generator_gatedcnn = _NetDescriptor(
    "generator_gatedcnn", "generator",
    [("gated", "h1_conv", 15, 1, 128),
     ("gated_in", "downsample1d_block1_", 5, 2, 256), ("gated_in", "downsample1d_block2_", 5, 2, 512)]
    + [("residual", "residual1d_block%d_" % i, 3, 1, 1024) for i in range(1, 7)]
    + [("gated_in_shuffle", "upsample1d_block1_", 5, 1, 1024), ("gated_in_shuffle", "upsample1d_block2_", 5, 1, 512),
       ("conv", "o1_conv", 15, 1, None)])

# module.py:199-211
discriminator = _NetDescriptor(
    "discriminator", "discriminator",
    [("gated", "h1_conv", (3, 3), (1, 2), 128),
     ("gated_in", "downsample2d_block1_", (3, 3), (2, 2), 256), ("gated_in", "downsample2d_block2_", (3, 3), (2, 2), 512),
     ("gated_in", "downsample2d_block3_", (6, 3), (1, 2), 1024), ("dense", "dense", None, None, 1)])


# ---------------------------------------------------------------------------------------------------------------------
# Variable scopes of the eager operators.  One native engine (mode='test': parameters + forward workspace) holds two
# generator and two discriminator networks; scopes are assigned to its slots in creation order, further engines are made
# when a third scope of a kind appears.
# ---------------------------------------------------------------------------------------------------------------------
_ENGINES = []          # [{'model': CycleGAN, 'generator': [scope or None, scope or None], 'discriminator': [...]}]
_SCOPES = OrderedDict()   # scope_name -> (kind, engine index, slot)
_SLOT_SCOPE = {"generator": ("generator_A2B", "generator_B2A"), "discriminator": ("discriminator_A", "discriminator_B")}


def _new_engine():
    from .model import CycleGAN
    m = CycleGAN(num_features=24, mode='test', max_batch=1, max_frames=128, seed=len(_ENGINES))
    _ENGINES.append({"model": m, "generator": [None, None], "discriminator": [None, None]})
    return len(_ENGINES) - 1


def _scope(desc, scope_name, reuse):
    if scope_name in _SCOPES:
        kind, ei, slot = _SCOPES[scope_name]
        if kind != desc.kind:
            raise ValueError("Variable scope %s holds a %s, not a %s" % (scope_name, kind, desc.kind))
        if not reuse:
            # tf.get_variable in a non-reusing scope that already has the variable (module.py:155-158 `assert scope.reuse is False`)
            raise ValueError("Variable %s/h1_conv/kernel already exists, disallowed. Did you mean to set reuse=True?" % scope_name)
        return ei, slot
    if reuse:
        raise ValueError("Variable %s/h1_conv/kernel does not exist, or was not created with tf.get_variable(). "
                         "Did you mean to set reuse=None?" % scope_name)
    for ei, e in enumerate(_ENGINES):
        for slot in (0, 1):
            if e[desc.kind][slot] is None:
                e[desc.kind][slot] = scope_name
                _SCOPES[scope_name] = (desc.kind, ei, slot)
                return ei, slot
    ei = _new_engine()
    _ENGINES[ei][desc.kind][0] = scope_name
    _SCOPES[scope_name] = (desc.kind, ei, 0)
    return ei, 0


def _train_model(ei):
    """the engine of slot group ei as a training engine (gradient arena and backward workspace), made on the first differentiable call"""
    m = _ENGINES[ei]["model"]
    if m.mode != 'train':
        from .model import CycleGAN
        t = CycleGAN(num_features=24, mode='train', max_batch=m._max_batch, max_frames=m._max_frames, log_dir='/tmp/cgvc_log')
        t.set_params(m.get_params())
        t.zero_grad()
        _ENGINES[ei]["model"] = m = t
    return m


def _apply(desc, inputs, reuse, scope_name):
    ei, slot = _scope(desc, scope_name, reuse)
    m = _ENGINES[ei]["model"]
    if hasattr(inputs, "is_cuda") and inputs.is_cuda:
        m = _train_model(ei)
        if desc.kind == "generator":
            return m.generator(inputs, 'A2B' if slot == 0 else 'B2A')
        return m.discriminator(inputs, 'A' if slot == 0 else 'B')
    if desc.kind == "generator":
        return m.test(inputs, 'A2B' if slot == 0 else 'B2A')
    return m.discriminate(inputs, 'A' if slot == 0 else 'B')


def scope_variables(scope_name):
    """OrderedDict TF variable name ('<scope_name>/h1_conv/kernel', ...) -> numpy array (TF layout) of an operator scope."""
    kind, ei, slot = _SCOPES[scope_name]
    pre = _SLOT_SCOPE[kind][slot] + "/"
    P = _ENGINES[ei]["model"].get_params()
    return OrderedDict((scope_name + "/" + n[len(pre):], v) for n, v in P.items() if n.startswith(pre))


def assign_scope_variables(scope_name, values):
    """Inject variables (names relative to the scope or prefixed with it) into an operator scope (tf.assign)."""
    kind, ei, slot = _SCOPES[scope_name]
    pre = _SLOT_SCOPE[kind][slot] + "/"
    upd = {}
    for n, v in values.items():
        rel = n[len(scope_name) + 1:] if n.startswith(scope_name + "/") else n
        upd[pre + rel] = v
    _ENGINES[ei]["model"].set_params(upd)


def scope_gradients(scope_name):
    """OrderedDict TF variable name -> d loss / d variable (CUDA tensors) that the backward passes of the scope's differentiable calls
    added up since zero_scope_gradients (loss scale removed)."""
    kind, ei, slot = _SCOPES[scope_name]
    pre = _SLOT_SCOPE[kind][slot]
    G = _train_model(ei).grads(pre)
    return OrderedDict((scope_name + n[len(pre):], v) for n, v in G.items())


def zero_scope_gradients():
    """Clear the variable gradients of every scope."""
    for e in _ENGINES:
        if e["model"].mode == 'train':
            e["model"].zero_grad()


def reset_default_graph():
    """Forget every operator scope and free their engines (tf.reset_default_graph)."""
    _SCOPES.clear()
    del _ENGINES[:]
