"""Checkpoint I/O in the `diffusers` directory layout the reference scripts read and write (host-side, no CUDA):

    <dir>/model_index.json                        pipeline: which classes sit in which sub-folder
    <dir>/unet/config.json                        UNet2DModel constructor kwargs (+ _class_name, _diffusers_version)
    <dir>/unet/diffusion_pytorch_model.bin        torch.save(state_dict)   (or .safetensors)
    <dir>/scheduler/scheduler_config.json         scheduler constructor kwargs

Replaces, for the DDPM family on the hot path: `ModelMixin.save_pretrained / from_pretrained`
(diffusers/models/modeling_utils.py:250-330, 333-680), `ConfigMixin.save_config / load_config`
(diffusers/configuration_utils.py:138-170, 273-420), `DiffusionPipeline.save_pretrained / from_pretrained`
(diffusers/pipelines/pipeline_utils.py:485-560, 563-1000) — as called at ddpm_prune.py:50,132,140, ddpm_train.py:292-306,498 and
ddpm_sample.py:27-41.  Only local directories (there is no hub access here); unknown config keys are kept and written back so
a checkpoint written by the reference round-trips.  Pruned networks are saved the reference's way — `torch.save(model)` of the
whole module (ddpm_prune.py:135) — which works because UNet2DModel pickles without its launch plans.
"""
from __future__ import annotations

import inspect
import json
import os
from types import SimpleNamespace
from typing import Optional

import torch

DIFFUSERS_VERSION = "0.17.0.dev0"          # the reference's vendored diffusers (diffusers/__init__.py)
CONFIG_NAME = "config.json"
SCHEDULER_CONFIG_NAME = "scheduler_config.json"
MODEL_INDEX_NAME = "model_index.json"
WEIGHTS_NAME = "diffusion_pytorch_model.bin"
SAFETENSORS_WEIGHTS_NAME = "diffusion_pytorch_model.safetensors"


def _jsonable(v):
    if isinstance(v, tuple):
        return [_jsonable(x) for x in v]
    if isinstance(v, list):
        return [_jsonable(x) for x in v]
    return v


def config_dict(obj) -> dict:
    """Constructor kwargs of a model / scheduler as the reference writes them: sorted keys, tuples as lists, plus the keys a
    reference-written file carried that this implementation does not interpret (`_extra_config`)."""
    cfg = dict(vars(obj.config))
    cfg.update(getattr(obj, "_extra_config", {}))
    out = {"_class_name": type(obj).__name__, "_diffusers_version": DIFFUSERS_VERSION}
    out.update({k: _jsonable(v) for k, v in sorted(cfg.items())})
    return out


def save_config(obj, save_directory: str, name: str):
    os.makedirs(save_directory, exist_ok=True)
    with open(os.path.join(save_directory, name), "w", encoding="utf-8") as f:
        f.write(json.dumps(config_dict(obj), indent=2, sort_keys=True) + "\n")


def _resolve(path: str, subfolder: Optional[str]) -> str:
    d = os.path.join(path, subfolder) if subfolder else path
    if not os.path.isdir(d):
        raise OSError(f"diff_pruning_b200: {d} is not a local directory (hub downloads are not supported)")
    return d


def load_config(path: str, name: str, subfolder: Optional[str] = None) -> dict:
    d = _resolve(path, subfolder)
    fn = os.path.join(d, name)
    if not os.path.isfile(fn) and name == SCHEDULER_CONFIG_NAME and os.path.isfile(os.path.join(d, CONFIG_NAME)):
        fn = os.path.join(d, CONFIG_NAME)          # old checkpoints keep the scheduler config in config.json
    with open(fn, "r", encoding="utf-8") as f:
        return json.load(f)


def build_from_config(cls, cfg: dict, **overrides):
    """cls(**kwargs) from a config dict: private keys dropped, keys the constructor does not name are remembered on the
    instance (`_extra_config`) and written back by save_config."""
    kw = {k: v for k, v in cfg.items() if not k.startswith("_")}
    kw.update(overrides)
    names = set(inspect.signature(cls.__init__).parameters) - {"self"}
    known = {k: v for k, v in kw.items() if k in names}
    extra = {k: v for k, v in kw.items() if k not in names}
    obj = cls(**known)
    cfg_ns = getattr(obj, "config", None)
    if isinstance(cfg_ns, SimpleNamespace):
        extra = {k: v for k, v in extra.items() if not hasattr(cfg_ns, k)}
        for k, v in extra.items():       # visible through `.config` too, so `OtherScheduler.from_config(this.config)` sees them
            setattr(cfg_ns, k, v)        # (e.g. a DDPM scheduler's clip_sample / prediction_type re-read as DDIM, ddpm_prune.py:140)
    obj._extra_config = extra
    return obj


# ------------------------------------------------------------------------------------------------ model weights
def save_model(model, save_directory: str, safe_serialization: bool = False):
    """ModelMixin.save_pretrained: config.json + weights (torch.save of the state dict, or safetensors)."""
    save_config(model, save_directory, CONFIG_NAME)
    sd = {k: v.detach().to("cpu").contiguous() for k, v in model.state_dict().items()}
    if safe_serialization:
        from safetensors.torch import save_file
        save_file(sd, os.path.join(save_directory, SAFETENSORS_WEIGHTS_NAME), metadata={"format": "pt"})
    else:
        torch.save(sd, os.path.join(save_directory, WEIGHTS_NAME))


def load_model(cls, path: str, subfolder: Optional[str] = None, **overrides):
    """ModelMixin.from_pretrained for a local directory: build from config.json, then strict load of the weights."""
    d = _resolve(path, subfolder)
    model = build_from_config(cls, load_config(path, CONFIG_NAME, subfolder), **overrides)
    st, bn = os.path.join(d, SAFETENSORS_WEIGHTS_NAME), os.path.join(d, WEIGHTS_NAME)
    if os.path.isfile(st):
        from safetensors.torch import load_file
        sd = load_file(st, device="cpu")
    elif os.path.isfile(bn):
        sd = torch.load(bn, map_location="cpu", weights_only=True)
    else:
        raise OSError(f"diff_pruning_b200: no {SAFETENSORS_WEIGHTS_NAME} or {WEIGHTS_NAME} in {d}")
    sd = convert_deprecated_attention_keys(sd)
    hint = ("pruned networks are stored as whole modules (torch.save(model) / torch.load, ddpm_prune.py:135, "
            "ddpm_train.py:292), not as a state dict next to the unpruned config.json")
    try:
        missing, unexpected = model.load_state_dict(sd, strict=False)
    except RuntimeError as e:                                   # shape mismatch
        raise RuntimeError(f"diff_pruning_b200: weights in {d} do not fit the architecture of its config.json: {hint}.  {e}") from None
    if missing or unexpected:
        raise RuntimeError(f"diff_pruning_b200: weights in {d} do not match the architecture of its config.json "
                           f"(missing {list(missing)[:4]}, unexpected {list(unexpected)[:4]}): {hint}")
    return model.eval()                                   # modeling_utils.py:640 puts loaded models in eval mode


_DEPRECATED_ATTN = (("query", "to_q"), ("key", "to_k"), ("value", "to_v"), ("proj_attn", "to_out.0"))


def convert_deprecated_attention_keys(sd: dict) -> dict:
    """Hub DDPM checkpoints (google/ddpm-cifar10-32, ddpm-ema-bedroom-256, ...) predate the Attention refactor and store the
    attention projections as `<block>.query / key / value / proj_attn`; the reference renames them at load time
    (modeling_utils.py:809-851, for blocks built with `_from_deprecated_attn_block=True`: unet_2d_blocks.py:441,730,1805).
    Every attention block of UNet2DModel is such a block, so the rename is purely by key suffix; already-converted files pass through."""
    out = {}
    for k, v in sd.items():
        parts = k.rsplit(".", 2)
        if len(parts) == 3 and parts[2] in ("weight", "bias") and ".attentions." in k:
            for old, new in _DEPRECATED_ATTN:
                if parts[1] == old:
                    k = f"{parts[0]}.{new}.{parts[2]}"
                    break
        out[k] = v
    return out


def allow_module_pickles():
    """torch >= 2.6 defaults torch.load to weights_only=True; the reference stores and reloads WHOLE modules (`torch.save(model)`
    ddpm_prune.py:135 / `torch.load(path)` ddpm_train.py:292, ddpm_sample.py:27).  Allow-list the classes such a pickle contains
    (this package's module classes + the torch.nn leaves + the config containers) so the unchanged `torch.load` call works."""
    import argparse
    import collections
    import sys
    import torch.nn as nn
    from types import SimpleNamespace as _NS
    from . import models
    cls = [getattr(models, n) for n in ("UNet2DModel", "UNet2DOutput", "Timesteps", "TimestepEmbedding", "Upsample2D", "Downsample2D",
                                        "ResnetBlock2D", "Attention", "DownBlock2D", "AttnDownBlock2D", "UNetMidBlock2D", "UpBlock2D",
                                        "AttnUpBlock2D")]
    cls += [nn.Conv2d, nn.Linear, nn.GroupNorm, nn.SiLU, nn.Dropout, nn.ModuleList, nn.Identity, nn.Parameter, _NS,
            collections.OrderedDict, set]
    # the module paths a REFERENCE-written pickle names (the weights-only unpickler matches globals by that string)
    ref_paths = {"diffusers.models.unet_2d": ("UNet2DModel",), "diffusers.models.embeddings": ("Timesteps", "TimestepEmbedding"),
                 "diffusers.models.resnet": ("Upsample2D", "Downsample2D", "ResnetBlock2D"),
                 "diffusers.models.attention_processor": ("Attention",),
                 "diffusers.models.unet_2d_blocks": ("DownBlock2D", "AttnDownBlock2D", "UNetMidBlock2D", "UpBlock2D", "AttnUpBlock2D")}
    cls += [(getattr(models, n), f"{path}.{n}") for path, names in ref_paths.items() for n in names]
    # the weights-only unpickler only fills plain dict / OrderedDict instances (SETITEMS), so the config container of a reference
    # pickle (FrozenDict, an OrderedDict subclass) is materialised as the OrderedDict it is
    cls.append((collections.OrderedDict, "diffusers.configuration_utils.FrozenDict"))
    # ddpm_exp's pickles (prune.py:281, runners/diffusion_simple.py:270-283) name models.diffusion.*; their `config` is an
    # argparse.Namespace, and the level / mid / temb containers are plain nn.Module instances
    from . import ddpm_exp
    cls += [(getattr(ddpm_exp, n), f"models.diffusion.{n}") for n in ("Model", "ResnetBlock", "AttnBlock", "Downsample", "Upsample")]
    cls += [ddpm_exp.Model, ddpm_exp.ResnetBlock, ddpm_exp.AttnBlock, ddpm_exp.Downsample, ddpm_exp.Upsample, nn.Module,
            argparse.Namespace]
    mod = sys.modules.get("diffusers.models.attention_processor")
    if mod is not None and "compat" in (getattr(mod, "__file__", "") or ""):
        cls += [getattr(mod, n) for n in ("AttnProcessor", "AttnProcessor2_0")]
    torch.serialization.add_safe_globals(cls)


# ------------------------------------------------------------------------------------------------ pipelines
def save_pipeline(pipe, save_directory: str, safe_serialization: bool = False):
    """DiffusionPipeline.save_pretrained: model_index.json + one sub-folder per component."""
    os.makedirs(save_directory, exist_ok=True)
    index = {"_class_name": type(pipe).__name__, "_diffusers_version": DIFFUSERS_VERSION,
             "scheduler": ["diffusers", type(pipe.scheduler).__name__], "unet": ["diffusers", type(pipe.unet).__name__]}
    with open(os.path.join(save_directory, MODEL_INDEX_NAME), "w", encoding="utf-8") as f:
        f.write(json.dumps(index, indent=2, sort_keys=True) + "\n")
    pipe.unet.save_pretrained(os.path.join(save_directory, "unet"), safe_serialization=safe_serialization)
    pipe.scheduler.save_pretrained(os.path.join(save_directory, "scheduler"))


def load_pipeline(cls, path: str, unet=None, scheduler=None, **unused):
    """DiffusionPipeline.from_pretrained(local dir[, unet=..., scheduler=...]): components passed in replace the stored ones
    (ddpm_train.py:304-308 passes the pruned unet)."""
    from . import models, sampling
    _resolve(path, None)
    classes = {"UNet2DModel": models.UNet2DModel, "DDPMScheduler": models.DDPMScheduler, "DDIMScheduler": sampling.DDIMScheduler}
    idx_fn = os.path.join(path, MODEL_INDEX_NAME)
    index = json.load(open(idx_fn, encoding="utf-8")) if os.path.isfile(idx_fn) else {}
    if unet is None:
        name = (index.get("unet") or [None, "UNet2DModel"])[1]
        if name not in classes:
            raise NotImplementedError(f"diff_pruning_b200: pipeline component class {name}")
        unet = classes[name].from_pretrained(path, subfolder="unet")
    if scheduler is None:
        # the stored scheduler config is re-interpreted by the scheduler class this pipeline runs (what
        # `DDIMScheduler.from_pretrained(save_path, subfolder="scheduler")` does at ddpm_prune.py:140)
        sched_cls = sampling.DDIMScheduler if cls.__name__ == "DDIMPipeline" else models.DDPMScheduler
        scheduler = sched_cls.from_pretrained(path, subfolder="scheduler")
    return cls(unet=unet, scheduler=scheduler)
