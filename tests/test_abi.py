"""Host-side checks that need no GPU: libcgvc.so builds/loads, exports every symbol include/cgvc.h declares,
and the product fails loudly (no CPU fallback) when no CUDA device is present."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "cgvc.h")).read()
    return sorted(set(re.findall(r"^\s*(?:int|const char\*)\s+(cgvc_\w+)\s*\(", src, flags=re.M)))


def test_library_exports_every_declared_symbol():
    from cgvc import native
    lib = native.load()
    decl = _declared_symbols()
    assert len(decl) >= 25
    for name in decl:
        assert hasattr(lib, name), "libcgvc.so does not export %s" % name
    assert sorted(native.EXPORTED_SYMBOLS) == decl, "ctypes prototypes and include/cgvc.h disagree"
    assert lib.cgvc_abi_version() == 1


def test_weight_layer_info_matches_the_header():
    """cgvc_weight_layer_info (include/cgvc.h) and its ctypes mirror: the same fields in the same order, of the same C types"""
    from cgvc import native
    src = open(os.path.join(ROOT, "include", "cgvc.h")).read()
    body = re.search(r"typedef struct cgvc_weight_layer_info \{(.*?)\} cgvc_weight_layer_info;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    decl = []
    for ctype, names in re.findall(r"(long long|int)\s+([\w\s,]+);", body):
        decl += [(n.strip(), ctype) for n in names.split(",")]
    mirror = [(n, {C.c_int: "int", C.c_longlong: "long long"}[t]) for n, t in native.WeightLayerInfo._fields_]
    assert mirror == decl
    assert native.load().cgvc_weight_planes.argtypes[2] == C.POINTER(native.WeightLayerInfo)


def test_library_is_sm90a_with_wgmma():
    import subprocess
    from cgvc import native
    out = subprocess.run(["cuobjdump", "-lelf", native.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run(["cuobjdump", "-sass", native.lib_path()], capture_output=True, text=True).stdout
    assert "HGMMA.64x256x16.F32.BF16" in sass, "bf16 wgmma kernels missing from the build"
    assert "QGMMA.64x256x32.F32.E4M3.E4M3" in sass, "the e4m3 wgmma of the F16F8 precision are missing from the build"
    assert "UTMALDG" in sass, "TMA tile loads missing from the build"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure path")
def test_fails_loudly_without_gpu():
    import cgvc
    from cgvc import native
    lib = native.load()
    cfg = native.Config(24, 1, 128, 1, 0, 1)
    h = C.c_void_p(0)
    assert lib.cgvc_create(C.byref(cfg), C.byref(h)) != 0
    assert b"no CPU fallback" in lib.cgvc_last_error(None)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        cgvc.CycleGAN(num_features=24)


def test_bad_config_is_rejected_before_touching_the_device():
    from cgvc import native
    lib = native.load()
    h = C.c_void_p(0)
    for cfg in (native.Config(25, 1, 128, 1, 0, 1), native.Config(24, 0, 128, 1, 0, 1), native.Config(24, 1, 130, 1, 0, 1), native.Config(24, 1, 128, 7, 0, 1)):
        assert lib.cgvc_create(C.byref(cfg), C.byref(h)) == -1
    assert lib.cgvc_create(None, C.byref(h)) == -1


def test_descriptors_mirror_reference_module():
    """The descriptors' layer tables expand to the TF variable names / shapes of module.py:148-213 (the oracle's table, which is
    pinned by the parameter counts of the reference text) -- that expansion is what CycleGAN checks the native engine against."""
    import copy
    from collections import OrderedDict
    import cgvc
    from oracle import cyclegan_oracle as O
    assert cgvc.generator_gatedcnn.kind == "generator" and cgvc.discriminator.kind == "discriminator"
    assert len(cgvc.generator_gatedcnn.layers) == 12 and len(cgvc.discriminator.layers) == 5
    assert cgvc.generator_gatedcnn.variables(24) == [(n, tuple(s)) for n, s, _ in O.generator_param_specs()]
    assert cgvc.discriminator.variables(24) == [(n, tuple(s)) for n, s, _ in O.discriminator_param_specs()]
    # a table standing in for the engine's: the matching descriptor passes, a different architecture is refused
    table = OrderedDict(("generator_A2B/" + n, (0, tuple(s))) for n, s, _ in O.generator_param_specs())
    cgvc.generator_gatedcnn.check_engine_table(table, "generator_A2B", 24)
    other = copy.deepcopy(cgvc.generator_gatedcnn)
    other.layers = [r if r[1] != "residual1d_block3_" else ("residual", "residual1d_block3_", 5, 1, 1024) for r in other.layers]
    with pytest.raises(ValueError, match="residual1d_block3_h1_conv/kernel"):
        other.check_engine_table(table, "generator_A2B", 24)
    with pytest.raises(ValueError):
        cgvc.discriminator.check_engine_table(table, "generator_A2B", 24)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "voice-converter-cyclegan_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in txt.replace("# oracle", ""), "%s mentions the oracle" % f
