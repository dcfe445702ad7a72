"""ddpm_exp's FID sampling loop and prune.py's Taylor loop (the DDIM codebase that produced the paper's CIFAR-10 results) on the engine.

Model          — ddpm_exp/models/diffusion.py:192-300: module tree, names and construction order of the reference, so
                 `torch.manual_seed(s); Model(cfg)` draws the reference's parameters and the state dicts match key for key.  The leaves are
                 nn.Conv2d / nn.Linear / nn.GroupNorm; AttnBlock, Downsample and Upsample are the VQ first stage's (autoencoder.py), which
                 the reference copied from the same source.  Model.forward(x, t) runs the planned sm_90a engine (Plan._build_ddim_model)
                 on CUDA; with grad enabled it is one autograd node whose backward fills Parameter.grad.  On the CPU it raises outside
                 models.trace_mode(), under which the modules run their torch forward (models/diffusion.py:113-136, 268-300).
noise_estimation_loss, taylor_loop, OursStopRule
               — functions/losses.py:4-15 and prune.py:236-258: the Taylor-importance loop over 1000 timesteps as graph replays
                 (TaylorScorer.forward_loss / backward), with the `--pruner ours` stop rule.
EMAHelper      — models/ema.py: register / state_dict / load_state_dict / ema, the shadow a list.
load_model     — runners/diffusion.py:100-195: a pickled pruned Model, a pickled [Model, ..., ema_shadow] list, a ckpt.pth list
                 [Module | state_dict, optimizer, epoch, step, (ema)], or a plain state dict from a local path.
sample_image   — runners/diffusion.py:492-537 with sample_type "generalized": the uniform / quad timestep sequences and
                 functions/denoising.py:10-33 generalized_steps.  Per step: the forward as one CUDA graph replay, torch.randn_like for
                 the step noise (drawn at every step, eta 0 included, as the reference does, so the generator advances alike), and
                 the update on dp_ddim_cfg_step (generalized_update), which writes x' to the NCHW state and to the plan's NHWC input.
sample_fid     — runners/diffusion.py:390-427: seeded rounds of sample_image, inverse_data_transform + tvu.save_image bytes on the device
                 (dp_decode_images), `{img_id}.png` files, and optionally the FID moments of those bytes (fid.Moments).

Under torch.distributed (torchrun) every rank seeds with its rank + seed and samples into the folder it is given, as finetune.py:204-206
gives each accelerate process its own; the only collectives are the optional moments' shift broadcast and all-reduce.
"""
from __future__ import annotations

import argparse
import glob
import os
import random
from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .autoencoder import AttnBlock, Downsample, Normalize, Upsample
from .engine import _stream, capture_graphs, frozen_weights, get_plan, unet_apply
from .models import ddpm_exp_frequencies
from .models import tracing as trace_mode_active


CIFAR10_CONFIG = {   # ddpm_exp/configs/cifar10.yml
    "data": {"dataset": "CIFAR10", "image_size": 32, "channels": 3, "logit_transform": False, "uniform_dequantization": False,
             "gaussian_dequantization": False, "random_flip": True, "rescaled": True, "num_workers": 4},
    "model": {"type": "simple", "in_channels": 3, "out_ch": 3, "ch": 128, "ch_mult": [1, 2, 2, 2], "num_res_blocks": 2,
              "attn_resolutions": [16], "dropout": 0.1, "var_type": "fixedlarge", "ema_rate": 0.9999, "ema": True, "resamp_with_conv": True},
    "diffusion": {"beta_schedule": "linear", "beta_start": 0.0001, "beta_end": 0.02, "num_diffusion_timesteps": 1000},
    "training": {"batch_size": 128, "n_epochs": 10000, "n_iters": 5000000, "snapshot_freq": 5000, "validation_freq": 2000},
    "sampling": {"batch_size": 64, "last_only": True},
    "optim": {"weight_decay": 0.0, "optimizer": "Adam", "lr": 0.0002, "beta1": 0.9, "amsgrad": False, "eps": 0.00000001, "grad_clip": 1.0},
}


def dict2namespace(config) -> argparse.Namespace:
    """The reference's yml dict as the nested argparse.Namespace its runners read (main.py / finetune.py dict2namespace); namespaces pass
    through."""
    if not isinstance(config, dict):
        return config
    ns = argparse.Namespace()
    for k, v in config.items():
        setattr(ns, k, dict2namespace(v) if isinstance(v, dict) else v)
    return ns


class ResnetBlock(nn.Module):
    """models/diffusion.py:76-136: GroupNorm + SiLU + 3x3 conv, + temb_proj(SiLU(temb)) per image, GroupNorm + SiLU + dropout + 3x3 conv,
    and a 1x1 nin_shortcut when the width changes."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        if conv_shortcut:
            raise NotImplementedError("ResnetBlock with a 3x3 conv_shortcut (Model never builds one)")
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.temb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = Normalize(out_channels)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, x, temb):
        """models/diffusion.py:113-136 in torch: the module-by-module forward of models.trace_mode() (the pruning tracer and the op
        counter walk it); Model.forward runs the engine plan otherwise."""
        h = self.conv1(_silu(self.norm1(x)))
        h = h + self.temb_proj(_silu(temb))[:, :, None, None]
        h = self.conv2(self.dropout(_silu(self.norm2(h))))
        if self.in_channels != self.out_channels:
            x = self.nin_shortcut(x)
        return x + h


def _silu(x):
    return x * torch.sigmoid(x)


def _timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """get_timestep_embedding (models/diffusion.py:6-24): sin | cos of t * ddpm_exp's frequencies."""
    emb = t.float()[:, None] * ddpm_exp_frequencies(dim).to(t.device)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1)
    return F.pad(emb, (0, 1, 0, 0)) if dim % 2 == 1 else emb


class Model(nn.Module):
    """models/diffusion.py:192-300 (config.model.type 'simple' or 'bayesian')."""

    def __init__(self, config):
        super().__init__()
        config = dict2namespace(config)
        self.config = config
        ch, out_ch, ch_mult = config.model.ch, config.model.out_ch, tuple(config.model.ch_mult)
        num_res_blocks = config.model.num_res_blocks
        attn_resolutions = config.model.attn_resolutions
        dropout = config.model.dropout
        in_channels = config.model.in_channels
        resolution = config.data.image_size
        resamp_with_conv = config.model.resamp_with_conv
        if config.model.type == "bayesian":
            self.logvar = nn.Parameter(torch.zeros(config.diffusion.num_diffusion_timesteps))
        self.ch = ch
        self.temb_ch = self.ch * 4
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels

        self.temb = nn.Module()
        self.temb.dense = nn.ModuleList([nn.Linear(self.ch, self.temb_ch), nn.Linear(self.temb_ch, self.temb_ch)])
        self.conv_in = nn.Conv2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)

        curr_res = resolution
        in_ch_mult = (1,) + ch_mult
        self.down = nn.ModuleList()
        block_in = None
        for i_level in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in, block_out = ch * in_ch_mult[i_level], ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            down = nn.Module()
            down.block, down.attn = block, attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)

        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)

        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = skip_in = ch * ch_mult[i_level]
            for i_block in range(self.num_res_blocks + 1):
                if i_block == self.num_res_blocks:
                    skip_in = ch * in_ch_mult[i_level]
                block.append(ResnetBlock(in_channels=block_in + skip_in, out_channels=block_out, temb_channels=self.temb_ch,
                                         dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block, up.attn = block, attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)

        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def __getstate__(self):
        # engine plans and captured graphs hold device buffers: never pickled with the module (torch.save(model), prune.py:281)
        return {k: v for k, v in self.__dict__.items() if not k.startswith("_dpb200")}

    def forward(self, x, t):
        """models/diffusion.py:268-300 on the engine.  t: (B,) timesteps, integer-valued (generalized_steps passes them as float).  With
        grad enabled the plan records its backward and `loss.backward()` accumulates into Parameter.grad (prune.py:236-258); x gets no
        gradient.  Under models.trace_mode() the modules run in torch, on any device."""
        if trace_mode_active():
            return self._torch_forward(x, t)
        if x.device.type != "cuda":
            raise RuntimeError("diff_pruning_b200: the ddpm_exp Model runs on a CUDA device (no CPU fallback outside models.trace_mode())")
        if self.training and any(m.p > 0 for m in self.modules() if isinstance(m, nn.Dropout)):
            raise RuntimeError("diff_pruning_b200: the ddpm_exp Model plan is an evaluation plan (dropout off): call model.eval()")
        assert x.shape[2] == x.shape[3] == self.resolution
        t = torch.as_tensor(t, device=x.device)
        if t.is_floating_point() and not torch.equal(t, t.trunc()):
            raise ValueError("diff_pruning_b200: the ddpm_exp Model plan takes integer-valued timesteps")
        return unet_apply(self, x, t)

    def _torch_forward(self, x, t):
        assert x.shape[2] == x.shape[3] == self.resolution
        temb = self.temb.dense[1](_silu(self.temb.dense[0](_timestep_embedding(torch.as_tensor(t, device=x.device), self.ch))))
        hs = [self.conv_in(x)]
        for i_level in range(self.num_resolutions):
            for i_block in range(self.num_res_blocks):
                h = self.down[i_level].block[i_block](hs[-1], temb)
                if len(self.down[i_level].attn) > 0:
                    h = self.down[i_level].attn[i_block](h)
                hs.append(h)
            if i_level != self.num_resolutions - 1:
                hs.append(self.down[i_level].downsample(hs[-1]))
        h = self.mid.block_2(self.mid.attn_1(self.mid.block_1(hs[-1], temb)), temb)
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                h = self.up[i_level].block[i_block](torch.cat([h, hs.pop()], dim=1), temb)
                if len(self.up[i_level].attn) > 0:
                    h = self.up[i_level].attn[i_block](h)
            if i_level != 0:
                h = self.up[i_level].upsample(h)
        return self.conv_out(_silu(self.norm_out(h)))


def noise_estimation_loss(model, x0: torch.Tensor, t: torch.Tensor, e: torch.Tensor, b: torch.Tensor, keepdim: bool = False):
    """functions/losses.py:4-15 for autograd callers: a = (1 - b).cumprod(0)[t], x = x0 sqrt(a) + e sqrt(1 - a), then
    ||e - model(x, t)||^2 summed over C, H, W per image, and averaged over the batch unless keepdim."""
    a = (1 - b).cumprod(dim=0).index_select(0, t).view(-1, 1, 1, 1)
    x = x0 * a.sqrt() + e * (1.0 - a).sqrt()
    output = model(x, t.float())
    if keepdim:
        return (e - output).square().sum(dim=(1, 2, 3))
    return (e - output).square().sum(dim=(1, 2, 3)).mean(dim=0)


class EMAHelper:
    """models/ema.py: the shadow is a list of parameter copies in Model.parameters() order."""

    def __init__(self, mu=0.999):
        self.mu = mu
        self.shadow = []

    def register(self, module):
        for p in module.parameters():
            if p.requires_grad:
                self.shadow.append(p.data.clone())

    def ema(self, module):
        for s, p in zip(self.shadow, module.parameters()):
            if p.requires_grad:
                p.data.copy_(s.data)

    def state_dict(self):
        return self.shadow

    def load_state_dict(self, state_dict):
        self.shadow = state_dict if isinstance(state_dict, list) else state_dict.values()


def _torch_load(path):
    from .checkpoint import allow_module_pickles
    allow_module_pickles()
    return torch.load(path, map_location="cpu")


def _apply_ema(model, config, shadow, use_ema):
    if use_ema and config.model.ema:
        h = EMAHelper(mu=config.model.ema_rate)
        h.register(model)
        h.load_state_dict(shadow)
        h.ema(model)
    return model


def load_model(config, path: Optional[str] = None, pruned: Optional[str] = None, use_ema: bool = False) -> Model:
    """Diffusion.build_model (runners/diffusion.py:100-195) from local files, the model on the CPU in eval mode:
      pruned: torch.save(model) of a pruned Model (prune.py:281), or a list [Model, ..., ema_shadow] (the EMA copy with use_ema);
      path:   a ckpt.pth list [Module | state_dict, optimizer_state, epoch, step, (ema_shadow)] (runners/diffusion_simple.py:270-283;
              the EMA copy with use_ema), or a plain state dict (the pretrained `ema_cifar10` file, which is never downloaded).
    Pickles that name models.diffusion.* load onto this module's classes (checkpoint.allow_module_pickles), pruned widths as saved."""
    config = dict2namespace(config)
    if pruned is not None:
        states = _torch_load(pruned)
        if isinstance(states, nn.Module):
            model = states
        elif isinstance(states, list):
            model = _apply_ema(states[0], config, states[-1], use_ema)
        else:
            raise NotImplementedError(f"pruned checkpoint of type {type(states).__name__}")
    elif path is not None:
        if not os.path.isfile(path):
            raise OSError(f"diff_pruning_b200: {path} is not a local file (checkpoints are never downloaded)")
        states = _torch_load(path)
        if isinstance(states, (list, tuple)):
            if isinstance(states[0], nn.Module):
                model = states[0]
            else:
                model = Model(config)
                model.load_state_dict(states[0], strict=True)
            model = _apply_ema(model, config, states[-1], use_ema)
        else:
            model = Model(config)
            model.load_state_dict(states)
    else:
        raise ValueError("load_model needs a checkpoint path or a pruned model file")
    return model.eval()


# ------------------------------------------------------------------------------------------------------------------- Taylor loop
class OursStopRule:
    """prune.py:248-253 (`--pruner ours`): max_loss starts at 0 and takes the loss when the loss exceeds it; the loop breaks when
    loss < max_loss * thr, an fp32 product as on the reference's 0-dim fp32 tensors, BEFORE loss.backward(): the stopping step's gradient
    is not accumulated.  A NaN loss neither raises max_loss nor stops."""

    def __init__(self, thr: float):
        self.thr = np.float32(thr)
        self.max_loss = np.float32(0.0)

    def stop(self, loss: float) -> bool:
        l32 = np.float32(loss)
        if l32 > self.max_loss:
            self.max_loss = l32
        return bool(l32 < self.max_loss * self.thr)


STOPPING_PRUNERS = ("ours",)
TAYLOR_LOOP_PRUNERS = ("taylor", "first_order_taylor", "second_order_taylor", "abs_taylor", "fisher", "ours")   # prune.py:236


def taylor_loop(model: Model, x: torch.Tensor, e: torch.Tensor, betas: torch.Tensor, pruner: str = "taylor", thr: float = 0.01,
                n_steps: int = 1000, use_graph: bool = True):
    """The loop of prune.py:236-258 on the engine: for step_k = 0 .. n_steps - 1, noise_estimation_loss(model, x, t = step_k for every
    image, e, betas) and its backward, the gradients accumulating into Parameter.grad from zero (model.zero_grad() first).  x (the data
    batch after data_transform) and e are (B, C, H, W) fp32 on a CUDA device, fixed for every step; betas the fp32 schedule, whose alphas
    table is (1 - b).cumprod(0) on the betas' device, as the loss computes it.

    Every step is one forward + loss graph replay and one backward graph replay (TaylorScorer.forward_loss / backward).  With
    pruner "ours" the host reads every step's loss and OursStopRule decides before the backward; the other pruners never stop and the
    losses stay on the device until the end.  Returns (losses of the steps that ran, the stopping one last, as a CPU fp32 tensor;
    the index of the stopping step or None)."""
    from .scoring import TaylorScorer
    if pruner not in TAYLOR_LOOP_PRUNERS:
        raise ValueError(f"prune.py runs its Taylor loop for {TAYLOR_LOOP_PRUNERS}, not {pruner!r}")
    if n_steps > betas.shape[0]:      # the reference's index_select fails past the table; the device gather would read past it
        raise ValueError(f"n_steps {n_steps} exceeds the {betas.shape[0]} timesteps of the schedule")
    if x.device.type != "cuda":
        raise RuntimeError("diff_pruning_b200: the ddpm_exp Taylor loop runs on a CUDA device (no CPU fallback)")
    acp = (1 - betas).cumprod(dim=0).to(x.device)
    model.zero_grad()
    ts = TaylorScorer(model, x, e, alphas_cumprod=acp, use_graph=use_graph, reduction="sum_mean")
    rule = OursStopRule(thr) if pruner in STOPPING_PRUNERS else None
    losses = torch.zeros(n_steps, device=x.device, dtype=torch.float32)
    stopped_at = None
    for k in range(n_steps):
        loss = ts.forward_loss(k)
        losses[k:k + 1].copy_(loss)
        if rule is not None and rule.stop(float(loss.item())):
            stopped_at = k
            break
        ts.backward()
    n = n_steps if stopped_at is None else stopped_at + 1
    return losses[:n].cpu(), stopped_at


PRUNERS = ("taylor", "random", "magnitude", "reinit", "first_order_taylor", "second_order_taylor", "abs_taylor", "fisher", "ours")


def _importance(pruner: str):
    """prune.py:191-208: the vendored torch_pruning importance of each `--pruner`, on the engine's device reductions."""
    from .compat import torch_pruning as tp
    if pruner in ("taylor", "ours"):
        return tp.importance.TaylorImportance(variant="vendored")         # the vendored sum_k (w dw)^2
    if pruner in ("first_order_taylor", "second_order_taylor"):
        return tp.importance.FullTaylorImportance(order=1 if pruner == "first_order_taylor" else 2)
    if pruner == "abs_taylor":
        return tp.importance.AbsTaylorImportance()
    if pruner == "fisher":
        return tp.importance.FisherImportance()
    if pruner == "magnitude":
        return tp.importance.MagnitudeImportance()
    return tp.importance.RandomImportance()                                # random, reinit


def prune(model: Model, config, x: torch.Tensor, pruner: str, pruning_ratio: float, thr: float = 0.01, timesteps: int = 1000,
          skip_type: str = "uniform", eta: float = 0.0, n_steps: int = 1000, use_graph: bool = True, preview: bool = True):
    """prune.py:179-291 for a Model on a CUDA device (in place), x the loaded batch in [0, 1] (B, C, S, S).  In the reference's order:
    the example input (torch.randn on the CPU generator, then moved, as prune.py:190 draws it), MagnitudePruner over the Model's groups
    (conv_out ignored), the MACs / parameters before, the preview noise (sampling.batch_size images on the device generator), then for the
    Taylor criteria data_transform(x) (`rescaled`: 2 x - 1), e = randn_like(x) and taylor_loop; the interactive pruner step, the
    `reinit` re-initialisation, the MACs / parameters after and the preview sample (sample_image from the preview noise; preview=False
    skips it).  Returns a SimpleNamespace: model, macs (before, after), params (before, after), losses, stopped_at, groups (root,
    channels, ch_groups, n_pruned, imp, idxs of every pruned group, in order) and samples.  torch.save(model) writes what prune.py:281
    writes; load_model(config, pruned=...) reads it back."""
    from .compat import torch_pruning as tp
    config = dict2namespace(config)
    if pruner not in PRUNERS:
        raise ValueError(f"pruner must be one of {PRUNERS}, got {pruner!r}")
    if getattr(config.data, "logit_transform", False) or not getattr(config.data, "rescaled", True) or hasattr(config, "image_mean") or \
            getattr(config.data, "uniform_dequantization", False) or getattr(config.data, "gaussian_dequantization", False):
        raise NotImplementedError("data_transform other than `rescaled` (2 x - 1)")
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("diff_pruning_b200: ddpm_exp.prune runs on a CUDA device (no CPU fallback)")
    model.eval()
    S = config.data.image_size
    example = {"x": torch.randn(1, 3, S, S).to(dev), "t": torch.ones(1).to(dev)}
    imp = _importance(pruner)
    mp = tp.pruner.MagnitudePruner(model, example, importance=imp, iterative_steps=1, channel_groups={}, ch_sparsity=pruning_ratio,
                                   ignored_layers=[model.conv_out], root_module_types=[nn.Conv2d, nn.Linear])
    base_macs, base_params = tp.utils.count_ops_and_params(model, example)
    noise = torch.randn(config.sampling.batch_size, config.data.channels, S, S, device=dev)
    betas = beta_schedule(config).to(dev)
    losses, stopped_at = torch.zeros(0), None
    if pruner in TAYLOR_LOOP_PRUNERS:
        x = 2 * x.to(dev, torch.float32) - 1.0
        e = torch.randn_like(x)
        losses, stopped_at = taylor_loop(model, x, e, betas, pruner, thr, n_steps, use_graph)
    groups = []
    for g in mp.step(interactive=True):
        groups.append({"root": g.root, "channels": g.channels, "ch_groups": g.ch_groups, "n_pruned": g.n_pruned, "imp": g.imp,
                       "idxs": list(g.idxs)})
        g.prune()
    if pruner == "reinit":
        def reset_parameters(_):          # prune.py:270-274: the function resets every module of the model on each call of apply
            for m in model.modules():
                if hasattr(m, "reset_parameters"):
                    m.reset_parameters()
        model.apply(reset_parameters)
    macs, params = tp.utils.count_ops_and_params(model, example)
    samples = sample_image(noise, model, betas, timesteps, skip_type, eta) if preview else None
    return SimpleNamespace(model=model, macs=(base_macs, macs), params=(base_params, params), losses=losses, stopped_at=stopped_at,
                           groups=groups, samples=samples)



# ------------------------------------------------------------------------------------------------------------------- sampling
def beta_schedule(config) -> torch.Tensor:
    """get_beta_schedule (runners/diffusion.py:28-56) as the fp32 tensor Diffusion.__init__ keeps (float64 numpy, then .float())."""
    d = config.diffusion
    T = d.num_diffusion_timesteps
    if d.beta_schedule == "quad":
        betas = np.linspace(d.beta_start ** 0.5, d.beta_end ** 0.5, T, dtype=np.float64) ** 2
    elif d.beta_schedule == "linear":
        betas = np.linspace(d.beta_start, d.beta_end, T, dtype=np.float64)
    elif d.beta_schedule == "const":
        betas = d.beta_end * np.ones(T, dtype=np.float64)
    elif d.beta_schedule == "jsd":
        betas = 1.0 / np.linspace(T, 1, T, dtype=np.float64)
    elif d.beta_schedule == "sigmoid":
        betas = 1 / (np.exp(-np.linspace(-6, 6, T)) + 1) * (d.beta_end - d.beta_start) + d.beta_start
    else:
        raise NotImplementedError(d.beta_schedule)
    return torch.from_numpy(betas).float()


def timestep_sequence(num_timesteps: int, timesteps: int, skip_type: str):
    """(seq, seq_next) of Diffusion.sample_image (runners/diffusion.py:499-511) and generalized_steps (denoising.py:13)."""
    if skip_type == "uniform":
        seq = list(range(0, num_timesteps, num_timesteps // timesteps))
    elif skip_type == "quad":
        seq = [int(s) for s in list(np.linspace(0, np.sqrt(num_timesteps * 0.8), timesteps) ** 2)]
    else:
        raise NotImplementedError(skip_type)
    return seq, [-1] + list(seq[:-1])


def step_scalars(betas: torch.Tensor, seq, seq_next, eta: float):
    """Per step, in sampling order, (i, sqrt(1 - a_t), sqrt(a_t), sqrt(a_next), c1, c2) as Python floats holding the fp32 values
    generalized_steps computes (denoising.py:4-7, 21-26): compute_alpha's cat([0], betas) and (1 - beta).cumprod(0) on the betas' device
    (a device scan need not round like the CPU loop), then the reference's expressions in its operation order, on one-element tensors."""
    ac = (1 - torch.cat([torch.zeros(1).to(betas.device), betas], dim=0)).cumprod(dim=0)
    rows = []
    for i, j in zip(reversed(seq), reversed(seq_next)):
        at, at_next = ac[i + 1:i + 2], ac[j + 1:j + 2]
        c1 = eta * ((1 - at / at_next) * (1 - at_next) / (1 - at)).sqrt()
        c2 = ((1 - at_next) - c1 ** 2).sqrt()
        rows.append(torch.cat([(1 - at).sqrt(), at.sqrt(), at_next.sqrt(), c1, c2]))
    vals = torch.stack(rows).cpu().tolist()
    return [(int(i),) + tuple(v) for i, v in zip(reversed(seq), vals)]


def _sampling_run(model, plan, use_graph: bool) -> SimpleNamespace:
    """The forward of `plan` as one captured graph (or the eager launch list), cached on the model per plan."""
    cache = model.__dict__.setdefault("_dpb200_ddim_runs", {})
    key = (id(plan), use_graph)
    run = cache.get(key)
    if run is not None and run.plan is plan:
        return run
    run = SimpleNamespace(plan=plan, graph=None)
    if use_graph:
        run.graph, = capture_graphs(plan.dev, plan.run_forward)
    cache[key] = run
    return run


@torch.no_grad()
def sample_image(x: torch.Tensor, model: Model, betas: torch.Tensor, timesteps: int = 100, skip_type: str = "quad", eta: float = 0.0,
                 use_graph: bool = True, x0_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Diffusion.sample_image(x, model, last=True) with sample_type "generalized" (runners/diffusion.py:492-537): x is x_T (B, C, H, W)
    on a CUDA device, betas the fp32 schedule of beta_schedule(config); returns the last sample.  The step noise is
    torch.randn_like(x) at every step, on the default generator of x's device, drawn after the step's forward as the reference draws it.
    x0_out (optional, (S, B, C, H, W)): every step's x0 prediction, in sampling order.  use_graph=False runs the launch list eagerly."""
    dev = x.device
    if dev.type != "cuda":
        raise RuntimeError("diff_pruning_b200: sample_image samples on a CUDA device (no CPU fallback)")
    if x.dtype != torch.float32:
        raise TypeError(f"x_T must be float32, got {x.dtype}")
    lib = L.load()
    B, C_, H, W = x.shape
    seq, seq_next = timestep_sequence(betas.shape[0], timesteps, skip_type)
    steps = step_scalars(betas.to(dev), seq, seq_next, float(eta))
    was_training = model.training
    model.eval()
    try:
        frozen = model.__dict__.get("_dpb200_frozen", False)
        with (_NullCtx() if frozen else frozen_weights(model)):
            plan = get_plan(model, B, H, W, dev, need_grad=False)
            plan.ensure_packed()
            run = _sampling_run(model, plan, use_graph)
            x_in, y_out = plan.x_in, plan.y_out
            x = x.contiguous()
            bufs = [torch.empty_like(x), torch.empty_like(x)]
            tmp = torch.empty_like(x) if eta != 0 else None
            L.check(lib.dp_nchw_to_nhwc(x.data_ptr(), x_in.ptr, x_in.ld, B, C_, H, W, _stream()), "x_T nchw->nhwc")
            for k, (i, sb, sa, sap, c1, c2) in enumerate(steps):
                plan.t_dev.fill_(i)
                if run.graph is not None:
                    run.graph.replay()
                else:
                    plan.run_forward()
                noise = torch.randn_like(x)
                cur, nxt = (x if k == 0 else bufs[(k - 1) % 2]), bufs[k % 2]
                x0 = x0_out[k].data_ptr() if x0_out is not None else None
                generalized_update(lib, y_out.ptr, y_out.ld, cur, noise, nxt, tmp, x_in.ptr, x_in.ld, x0, sb, sa, sap, c1, c2)
    finally:
        model.train(was_training)
    return bufs[(len(steps) - 1) % 2]


def generalized_update(lib, eps: int, ld_eps: int, x: torch.Tensor, noise: torch.Tensor, x_out: torch.Tensor, tmp: Optional[torch.Tensor],
                       x_in: int, ld_in: int, x0: Optional[int], sb: float, sa: float, sap: float, c1: float, c2: float):
    """generalized_steps' update (denoising.py:21-27) on dp_ddim_cfg_step, unguided: x0 = (x - e sqrt(1 - a_t)) / sqrt(a_t) and
    x' = (sqrt(a_next) x0 + c1 n) + c2 e, every operation rounded on its own in that order, so x' and x0 equal the reference's fp32 values
    for the same eps_hat (the NHWC plan output at `eps`, pixel stride ld_eps) and noise.  x' goes to x_out (NCHW) and to the plan's NHWC
    input x_in; x0 (NCHW) to the address x0 unless None.
      c1 == 0 (eta 0): c1 n is a zero, which leaves sqrt(a_next) x0 as it is; the kernel's sqrt(a_next) x0 + c2 e is the update.  One launch.
      c1 != 0: the kernel adds its noise term after its direction term, the reference the other way round.  Launch 1 forms
        v = (sqrt(a_next) x0 + 0 e) + c1 n into tmp (and x0); launch 2 reads v as its state with sqrt(1 - a_t) = 0, sqrt(a_t) = 1 and
        sqrt(a_next) = 1, which leave v unchanged, and adds c2 e."""
    B, C_, H, W = x.shape
    s = _stream()
    if c1 == 0.0:
        L.check(lib.dp_ddim_cfg_step(eps, ld_eps, x.data_ptr(), None, x_out.data_ptr(), x_in, ld_in, x0, B, C_, H, W, 0, 0.0, sb, sa, sap,
                                     c2, 0.0, s), "ddim generalized step")
        return
    L.check(lib.dp_ddim_cfg_step(eps, ld_eps, x.data_ptr(), noise.data_ptr(), tmp.data_ptr(), x_in, ld_in, x0, B, C_, H, W, 0, 0.0, sb, sa,
                                 sap, 0.0, c1, s), "ddim generalized step (noise term)")
    L.check(lib.dp_ddim_cfg_step(eps, ld_eps, tmp.data_ptr(), None, x_out.data_ptr(), x_in, ld_in, None, B, C_, H, W, 0, 0.0, 0.0, 1.0, 1.0,
                                 c2, 0.0, s), "ddim generalized step (direction term)")


class _NullCtx:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


def _rank_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


@torch.no_grad()
def sample_fid(model: Model, config, image_folder: str, total: int = 50000, batch_size: Optional[int] = None, timesteps: int = 100,
               skip_type: str = "quad", eta: float = 0.0, seed: int = 2333, write_images: bool = True, inception=None,
               fid_dims: int = 2048):
    """Diffusion.sample_fid (runners/diffusion.py:390-427) for a model on a CUDA device: seeds torch / random / numpy with
    rank + seed, continues img_id from the files already in image_folder, and runs (total - img_id) // batch_size rounds of
    x_T = torch.randn(...) -> sample_image -> the bytes tvu.save_image(inverse_data_transform(x)) writes (dp_decode_images) ->
    `{img_id}.png` (write_images).  With an Inception model (fid.InceptionV3) the FID moments of the same bytes accumulate on the device,
    and under torch.distributed over several ranks they are summed over the ranks at the end.  image_folder is this process's folder
    (finetune.py:204-206 gives every process its own).  Returns (mu, sigma, n_images): mu / sigma None without an Inception model."""
    config = dict2namespace(config)
    if getattr(config.data, "logit_transform", False) or not getattr(config.data, "rescaled", True) or hasattr(config, "image_mean"):
        raise NotImplementedError("inverse_data_transform other than `rescaled` ((x + 1) / 2, clamped)")
    if config.data.channels != 3:
        raise NotImplementedError("sample_fid writes RGB images (data.channels 3)")
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("diff_pruning_b200: sample_fid samples on a CUDA device (no CPU fallback)")
    rank, world = _rank_world()
    torch.manual_seed(rank + seed)
    random.seed(rank + seed)
    np.random.seed(rank + seed)
    n = config.sampling.batch_size if batch_size is None else batch_size
    C_, S = config.data.channels, config.data.image_size
    os.makedirs(image_folder, exist_ok=True)
    img_id = len(glob.glob(f"{image_folder}/*"))
    n_rounds = (total - img_id) // n
    betas = beta_schedule(config).to(dev)
    lib = L.load()
    mom = block = None
    if inception is not None:
        from . import fid
        block = fid._block_of(inception, fid_dims)
        mom = fid.Moments(fid_dims, device=dev)
    u8 = torch.empty((n, S, S, C_), dtype=torch.uint8, device=dev)
    n_images = 0
    with frozen_weights(model):
        for r in range(n_rounds):
            x = torch.randn(n, C_, S, S, device=dev)
            sample_image(x, model, betas, timesteps, skip_type, eta)
            x_in = get_plan(model, n, S, S, dev, need_grad=False).x_in       # the last step wrote the final sample there too
            L.check(lib.dp_decode_images(x_in.ptr, x_in.ld, n, C_, S, S, u8.data_ptr(), None, _stream()), "decode_images")
            if mom is not None:
                plan = inception.plan(n, "u8", (S, S))
                plan.load(u8)
                plan.run()
                if world > 1 and r == 0:    # rank 0's first batch is the shift of every rank's moments
                    if rank == 0:
                        mom.add(plan.feat[block])
                    mom.share_shift(0)
                    if rank > 0:
                        mom.add(plan.feat[block])
                else:
                    mom.add(plan.feat[block])
            if write_images:
                from PIL import Image
                for img in u8.cpu().numpy():
                    Image.fromarray(img).save(os.path.join(image_folder, f"{img_id}.png"))
                    img_id += 1
            n_images += n
    if mom is None:
        return None, None, n_images
    if world > 1:
        mom.all_reduce()
    mu, sigma = mom.finalize()
    return mu, sigma, n_images
