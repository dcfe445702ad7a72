"""diff_pruning_b200 — H100-native (sm_90a) Taylor-importance / finetune hot path of VainF/Diff-Pruning.

See DESIGN.md. Public surface mirrors the reference's (SURVEY.md §8(b1)).
"""
from .models import (  # noqa: F401
    CIFAR10_DDPM_CONFIG, LSUN256_DDPM_CONFIG, TINY_TEST_CONFIG, DDPMScheduler, UNet2DModel, UNet2DOutput,
    trace_mode,
)

__version__ = "0.1.0"


def __getattr__(name):   # lazy: sampling pulls in the engine / the shared library
    if name in ("DDIMScheduler", "DDIMPipeline", "DDPMPipeline", "DiffusionPipeline"):
        from . import sampling
        return getattr(sampling, name)
    raise AttributeError(name)
