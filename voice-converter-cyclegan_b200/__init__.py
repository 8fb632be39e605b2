"""voice-converter-cyclegan_b200: the CycleGAN-VC training/inference hot path of leimao/Voice-Converter-CycleGAN
re-built for H100 (sm_90a).  `CycleGAN` mirrors the reference class (model.py:7-169); `generator_gatedcnn` and
`discriminator` mirror the network callables of module.py as native-engine descriptors.

The directory name is not a Python identifier; import it through the root shim:  `import cgvc`.
"""
from .module import discriminator, generator_gatedcnn          # noqa: F401


def __getattr__(name):
    # CycleGAN pulls in torch + the native library; keep `import cgvc` cheap for tools that only need descriptors
    if name == "CycleGAN":
        from .model import CycleGAN
        return CycleGAN
    if name == "native":
        from . import _native
        return _native
    raise AttributeError(name)
