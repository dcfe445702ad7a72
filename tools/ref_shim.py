"""Import shim that makes the READ-ONLY reference checkout importable in the build container.

Only used by tools/gen_golden.py (fixture generation) — never by the product, tests, smoke() or bench.
The four shims are documented in SURVEY.md §8(c)/Appendix A; no reference file is modified or copied.
"""
import importlib.util
import os
import sys
import types

import torch  # noqa: F401  (must precede the matplotlib stub)

REF = os.environ["DPB200_REFERENCE"]   # path of the reference checkout


def install():
    import huggingface_hub
    import huggingface_hub.constants as hc

    if not hasattr(hc, "hf_cache_home"):
        hc.hf_cache_home = os.path.expanduser("~/.cache/huggingface")
    for name in ("HfFolder", "cached_download"):
        if not hasattr(huggingface_hub, name):
            setattr(huggingface_hub, name, type(name, (), {}))

    class _Plt(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith("__"):
                raise AttributeError(k)
            return lambda *a, **kw: None

    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = _Plt("matplotlib.pyplot")
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = mpl.pyplot

    orig = importlib.util.find_spec
    importlib.util.find_spec = lambda n, *a, **k: None if n == "transformers" else orig(n, *a, **k)
    sys.path[:0] = [os.path.join(REF, "ddpm_exp"), REF]
    import diffusers  # noqa: F401

    importlib.util.find_spec = orig
    import torch_pruning  # noqa: F401

    return diffusers, torch_pruning


def install_ldm():
    """Makes ldm_exp's `ldm` package importable on CPUs: omegaconf (openaimodel.py:476) and the text-encoder dependencies that
    ldm/modules/encoders/modules.py imports at the top (clip, kornia) are stubbed; the classes used from these modules need none of them."""
    sys.path.insert(0, os.path.join(REF, "ldm_exp"))
    oc, lc = types.ModuleType("omegaconf"), types.ModuleType("omegaconf.listconfig")
    lc.ListConfig = type("ListConfig", (list,), {})
    oc.listconfig = lc
    sys.modules.setdefault("omegaconf", oc)
    sys.modules.setdefault("omegaconf.listconfig", lc)
    for name in ("clip", "kornia"):
        sys.modules.setdefault(name, types.ModuleType(name))


def install_vq_model():
    """Makes ldm/models/autoencoder.py importable: pytorch_lightning and taming-transformers are not in the build container.
    LightningModule is stood in by nn.Module, and taming's VectorQuantizer2 by a module that builds what its constructor builds as
    recalled (taming is not in the reference tree): `embedding` = nn.Embedding(n_e, e_dim) re-drawn U(-1/n_e, 1/n_e), so a seeded
    VQModelInterface draws its parameters in the reference's order.  encode() does not use the quantizer."""
    import torch.nn as nn
    install_ldm()
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningModule = nn.Module

    class VectorQuantizer2(nn.Module):
        def __init__(self, n_e, e_dim, beta, remap=None, unknown_index="random", sane_index_shape=False, legacy=True):
            super().__init__()
            self.n_e, self.e_dim, self.beta, self.legacy = n_e, e_dim, beta, legacy
            self.embedding = nn.Embedding(self.n_e, self.e_dim)
            self.embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)
    mods = {n: types.ModuleType(n) for n in ("taming", "taming.modules", "taming.modules.vqvae", "taming.modules.vqvae.quantize")}
    mods["taming.modules.vqvae.quantize"].VectorQuantizer2 = VectorQuantizer2
    sys.modules.setdefault("pytorch_lightning", pl)
    for n, m in mods.items():
        sys.modules.setdefault(n, m)


def cpu_ddim_sampler():
    """The reference's DDIMSampler (ldm/models/diffusion/ddim.py) with a register_buffer that leaves tensors on their device: the
    original moves every tensor buffer to CUDA (ddim.py:18-22).  Everything else, the schedule and the sampling loop, is the unmodified
    reference code."""
    from ldm.models.diffusion.ddim import DDIMSampler

    class CpuDDIMSampler(DDIMSampler):
        def register_buffer(self, name, attr):
            setattr(self, name, attr)
    return CpuDDIMSampler


def cpu_generalized_steps(record=None):
    """ddpm_exp's generalized_steps (functions/denoising.py:10-33) on the CPU: the unmodified function, run with `Tensor.to('cuda')`
    (denoising.py:20 hard-codes it) redirected to the CPU.  record: a list that receives every torch.randn_like draw (the step noise)."""
    from functions.denoising import generalized_steps

    def run(*a, **kw):
        to, randn_like = torch.Tensor.to, torch.randn_like

        def to_cpu(self, *args, **kwargs):
            if args and args[0] == "cuda":
                args = ("cpu",) + args[1:]
            return to(self, *args, **kwargs)

        def draw(*args, **kwargs):
            n = randn_like(*args, **kwargs)
            if record is not None:
                record.append(n.clone())
            return n
        torch.Tensor.to, torch.randn_like = to_cpu, draw
        try:
            return generalized_steps(*a, **kw)
        finally:
            torch.Tensor.to, torch.randn_like = to, randn_like
    return run
