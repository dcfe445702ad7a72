"""Module tree of the reference's UNet2DModel — the drop-in boundary (SURVEY.md §8(b1)).

The classes below keep the *names, construction order, parameter shapes and attribute names* of
  diffusers/models/unet_2d.py:83-217        (UNet2DModel)
  diffusers/models/unet_2d_blocks.py:391-472, 681-762, 911-994, 1754-1831, 1982-2060 (5 block classes)
  diffusers/models/resnet.py:101-220, 456-639 (Upsample2D, Downsample2D, ResnetBlock2D)
  diffusers/models/attention_processor.py:36-157 (Attention)
  diffusers/models/embeddings.py:155-229    (TimestepEmbedding, Timesteps)
so that (i) ``torch.manual_seed(s); UNet2DModel(**cfg)`` yields bit-identical parameters to the
reference, (ii) state dicts are interchangeable, (iii) torch_pruning-style tools can walk real
nn.Conv2d / nn.Linear / nn.GroupNorm leaves and mutate them in place.

Execution:
  * CUDA tensors  -> the planned sm_90a engine (engine.py) behind one autograd node; the C-ABI
    library must be present, otherwise a RuntimeError is raised (no silent fallback).
  * ``with trace_mode():`` -> leaf-module-by-leaf-module execution with torch ops. This exists only
    for structure discovery (dependency tracing with forward hooks at batch 1, MAC counting,
    CPU host-logic tests). It is never used for the hot loop.
"""
from __future__ import annotations

import contextlib
import inspect
import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

_TRACE = [False]


@contextlib.contextmanager
def trace_mode(enabled: bool = True):
    """Run modules leaf by leaf with torch ops (structure discovery only)."""
    old = _TRACE[0]
    _TRACE[0] = enabled
    try:
        yield
    finally:
        _TRACE[0] = old


def tracing() -> bool:
    return _TRACE[0]


def sinusoidal_frequencies(embedding_dim: int, downscale_freq_shift: float = 1.0, max_period: int = 10000):
    """exp(-ln(max_period) * i / (half - shift)) as float32 — embeddings.py:38-43 (same op order)."""
    half = embedding_dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32)
    exponent = exponent / (half - downscale_freq_shift)
    return torch.exp(exponent)


class Timesteps(nn.Module):
    """embeddings.py:215-229."""

    def __init__(self, num_channels: int, flip_sin_to_cos: bool, downscale_freq_shift: float):
        super().__init__()
        self.num_channels = num_channels
        self.flip_sin_to_cos = flip_sin_to_cos
        self.downscale_freq_shift = downscale_freq_shift

    def forward(self, timesteps):
        freqs = sinusoidal_frequencies(self.num_channels, self.downscale_freq_shift).to(timesteps.device)
        arg = timesteps[:, None].float() * freqs[None, :]
        emb = torch.cat([torch.sin(arg), torch.cos(arg)], dim=-1)
        if self.flip_sin_to_cos:
            half = self.num_channels // 2
            emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
        if self.num_channels % 2 == 1:
            emb = F.pad(emb, (0, 1, 0, 0))
        return emb


class TimestepEmbedding(nn.Module):
    """embeddings.py:155-212 (no cond_proj / post_act in the DDPM configs)."""

    def __init__(self, in_channels: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, sample):
        return self.linear_2(self.act(self.linear_1(sample)))


class Upsample2D(nn.Module):
    """resnet.py:101-170 (use_conv=True, nearest x2)."""

    def __init__(self, channels, use_conv=False, out_channels=None, name="conv"):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.name = name
        self.conv = nn.Conv2d(self.channels, self.out_channels, 3, padding=1) if use_conv else None

    def forward(self, hidden_states):
        assert hidden_states.shape[1] == self.channels
        hidden_states = F.interpolate(hidden_states, scale_factor=2.0, mode="nearest")
        if self.use_conv:
            hidden_states = self.conv(hidden_states)
        return hidden_states


class Downsample2D(nn.Module):
    """resnet.py:173-220 (use_conv=True, stride 2, asymmetric pad when padding == 0)."""

    def __init__(self, channels, use_conv=False, out_channels=None, padding=1, name="conv"):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.padding = padding
        self.name = name
        if not use_conv:
            raise NotImplementedError("only the conv downsampler is on the DDPM hot path")
        self.conv = nn.Conv2d(self.channels, self.out_channels, 3, stride=2, padding=padding)

    def forward(self, hidden_states):
        assert hidden_states.shape[1] == self.channels
        if self.padding == 0:
            hidden_states = F.pad(hidden_states, (0, 1, 0, 1), mode="constant", value=0)
        return self.conv(hidden_states)


class ResnetBlock2D(nn.Module):
    """resnet.py:456-639, time_embedding_norm == 'default', no up/down."""

    def __init__(self, *, in_channels, out_channels=None, dropout=0.0, temb_channels=512, groups=32,
                 eps=1e-6, output_scale_factor=1.0):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.output_scale_factor = output_scale_factor
        self.norm1 = nn.GroupNorm(num_groups=groups, num_channels=in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(num_groups=groups, num_channels=out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.conv_shortcut = None
        if in_channels != out_channels:
            self.conv_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, input_tensor, temb):
        h = F.silu(self.norm1(input_tensor))
        h = self.conv1(h)
        h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.dropout(F.silu(self.norm2(h)))
        h = self.conv2(h)
        if self.conv_shortcut is not None:
            input_tensor = self.conv_shortcut(input_tensor)
        return (input_tensor + h) / self.output_scale_factor


class Attention(nn.Module):
    """attention_processor.py:36-157 + legacy AttnProcessor :415-470 (self-attention, spatial input).

    ``scale`` is fixed at construction (attention_processor.py:87) and ``inner`` follows
    ``to_q.out_features`` so the block keeps working after channel pruning (SURVEY.md §7).
    """

    def __init__(self, query_dim, heads=1, dim_head=None, eps=1e-5, norm_num_groups=32,
                 rescale_output_factor=1.0, residual_connection=True, dropout=0.0):
        super().__init__()
        dim_head = query_dim if dim_head is None else dim_head
        inner_dim = dim_head * heads
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.rescale_output_factor = rescale_output_factor
        self.residual_connection = residual_connection
        self.group_norm = nn.GroupNorm(num_channels=query_dim, num_groups=norm_num_groups, eps=eps, affine=True)
        self.to_q = nn.Linear(query_dim, inner_dim, bias=True)
        self.to_k = nn.Linear(query_dim, inner_dim, bias=True)
        self.to_v = nn.Linear(query_dim, inner_dim, bias=True)
        self.to_out = nn.ModuleList([nn.Linear(inner_dim, query_dim, bias=True), nn.Dropout(dropout)])

    def forward(self, hidden_states):
        residual = hidden_states
        b, c, hh, ww = hidden_states.shape
        x = self.group_norm(hidden_states.view(b, c, hh * ww)).transpose(1, 2)
        q, k, v = self.to_q(x), self.to_k(x), self.to_v(x)
        hd = self.heads

        def split(t):  # (b, n, inner) -> (b*heads, n, inner/heads)
            return t.reshape(b, -1, hd, t.shape[-1] // hd).permute(0, 2, 1, 3).reshape(b * hd, -1, t.shape[-1] // hd)

        q, k, v = split(q), split(k), split(v)
        probs = torch.softmax(torch.bmm(q, k.transpose(1, 2)) * self.scale, dim=-1)
        o = torch.bmm(probs, v)
        o = o.reshape(b, hd, -1, o.shape[-1]).permute(0, 2, 1, 3).reshape(b, -1, hd * o.shape[-1])
        o = self.to_out[1](self.to_out[0](o))
        o = o.transpose(-1, -2).reshape(b, c, hh, ww)
        if self.residual_connection:
            o = o + residual
        return o / self.rescale_output_factor


def _attn(channels, head_dim, eps, groups, scale):
    return Attention(channels, heads=channels // head_dim if head_dim is not None else 1,
                     dim_head=head_dim if head_dim is not None else channels, eps=eps,
                     norm_num_groups=groups, rescale_output_factor=scale, residual_connection=True)


class DownBlock2D(nn.Module):
    """unet_2d_blocks.py:911-994."""
    has_attention = False

    def __init__(self, in_channels, out_channels, temb_channels, num_layers, resnet_eps, resnet_groups,
                 attn_num_head_channels, downsample_padding, add_downsample, dropout=0.0):
        super().__init__()
        resnets, attentions = [], []
        for i in range(num_layers):
            cin = in_channels if i == 0 else out_channels
            resnets.append(ResnetBlock2D(in_channels=cin, out_channels=out_channels, temb_channels=temb_channels,
                                         eps=resnet_eps, groups=resnet_groups, dropout=dropout))
            if self.has_attention:  # interleaved construction order matters for seeded init
                attentions.append(_attn(out_channels, attn_num_head_channels, resnet_eps, resnet_groups, 1.0))
        if self.has_attention:
            self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        if add_downsample:
            self.downsamplers = nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                            padding=downsample_padding, name="op")])
        else:
            self.downsamplers = None

    def forward(self, hidden_states, temb=None):
        output_states = ()
        for i, resnet in enumerate(self.resnets):
            hidden_states = resnet(hidden_states, temb)
            if self.has_attention:
                hidden_states = self.attentions[i](hidden_states)
            output_states += (hidden_states,)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                hidden_states = d(hidden_states)
            output_states += (hidden_states,)
        return hidden_states, output_states


class AttnDownBlock2D(DownBlock2D):
    """unet_2d_blocks.py:681-762."""
    has_attention = True


class UNetMidBlock2D(nn.Module):
    """unet_2d_blocks.py:391-472 (num_layers = 1)."""

    def __init__(self, in_channels, temb_channels, resnet_eps, resnet_groups, attn_num_head_channels,
                 output_scale_factor=1.0, add_attention=True, dropout=0.0):
        super().__init__()
        self.add_attention = add_attention
        mk = lambda: ResnetBlock2D(in_channels=in_channels, out_channels=in_channels, temb_channels=temb_channels,
                                   eps=resnet_eps, groups=resnet_groups, dropout=dropout,
                                   output_scale_factor=output_scale_factor)
        resnets = [mk()]
        attentions = [_attn(in_channels, attn_num_head_channels, resnet_eps, resnet_groups, output_scale_factor)
                      if add_attention else None]
        resnets.append(mk())
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)

    def forward(self, hidden_states, temb=None):
        hidden_states = self.resnets[0](hidden_states, temb)
        for attn, resnet in zip(self.attentions, self.resnets[1:]):
            if attn is not None:
                hidden_states = attn(hidden_states)
            hidden_states = resnet(hidden_states, temb)
        return hidden_states


class UpBlock2D(nn.Module):
    """unet_2d_blocks.py:1982-2060."""
    has_attention = False

    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, num_layers, resnet_eps,
                 resnet_groups, attn_num_head_channels, add_upsample, dropout=0.0):
        super().__init__()
        resnets, attentions = [], []
        for i in range(num_layers):
            res_skip = in_channels if i == num_layers - 1 else out_channels
            res_in = prev_output_channel if i == 0 else out_channels
            resnets.append(ResnetBlock2D(in_channels=res_in + res_skip, out_channels=out_channels,
                                         temb_channels=temb_channels, eps=resnet_eps, groups=resnet_groups,
                                         dropout=dropout))
            if self.has_attention:
                attentions.append(_attn(out_channels, attn_num_head_channels, resnet_eps, resnet_groups, 1.0))
        if self.has_attention:
            self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)
        if add_upsample:
            self.upsamplers = nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
        else:
            self.upsamplers = None

    def forward(self, hidden_states, res_hidden_states_tuple, temb=None):
        for i, resnet in enumerate(self.resnets):
            res = res_hidden_states_tuple[-1]
            res_hidden_states_tuple = res_hidden_states_tuple[:-1]
            hidden_states = torch.cat([hidden_states, res], dim=1)
            hidden_states = resnet(hidden_states, temb)
            if self.has_attention:
                hidden_states = self.attentions[i](hidden_states)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                hidden_states = u(hidden_states)
        return hidden_states


class AttnUpBlock2D(UpBlock2D):
    """unet_2d_blocks.py:1754-1831."""
    has_attention = True


_DOWN = {"DownBlock2D": DownBlock2D, "AttnDownBlock2D": AttnDownBlock2D}
_UP = {"UpBlock2D": UpBlock2D, "AttnUpBlock2D": AttnUpBlock2D}


@dataclass
class UNet2DOutput:
    sample: torch.Tensor


class UNet2DModel(nn.Module):
    """unet_2d.py:83-316 — positional time embedding, no class conditioning (the DDPM configs)."""

    def __init__(self, sample_size=None, in_channels=3, out_channels=3, center_input_sample=False,
                 time_embedding_type="positional", freq_shift=0, flip_sin_to_cos=True,
                 down_block_types=("DownBlock2D", "AttnDownBlock2D", "AttnDownBlock2D", "AttnDownBlock2D"),
                 up_block_types=("AttnUpBlock2D", "AttnUpBlock2D", "AttnUpBlock2D", "UpBlock2D"),
                 block_out_channels=(224, 448, 672, 896), layers_per_block=2, mid_block_scale_factor=1,
                 downsample_padding=1, act_fn="silu", attention_head_dim=8, norm_num_groups=32, norm_eps=1e-5,
                 resnet_time_scale_shift="default", add_attention=True, class_embed_type=None,
                 num_class_embeds=None, dropout=0.0, **unused):
        super().__init__()
        if len(down_block_types) != len(up_block_types):
            raise ValueError("Must provide the same number of `down_block_types` as `up_block_types`.")
        if len(block_out_channels) != len(down_block_types):
            raise ValueError("Must provide the same number of `block_out_channels` as `down_block_types`.")
        if time_embedding_type != "positional" or resnet_time_scale_shift != "default" \
                or class_embed_type is not None or num_class_embeds is not None or act_fn not in ("silu", "swish"):
            raise NotImplementedError("only the DDPM UNet2DModel configuration family is supported")
        self.config = SimpleNamespace(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
            center_input_sample=center_input_sample, time_embedding_type=time_embedding_type,
            freq_shift=freq_shift, flip_sin_to_cos=flip_sin_to_cos, down_block_types=tuple(down_block_types),
            up_block_types=tuple(up_block_types), block_out_channels=tuple(block_out_channels),
            layers_per_block=layers_per_block, mid_block_scale_factor=mid_block_scale_factor,
            downsample_padding=downsample_padding, act_fn=act_fn, attention_head_dim=attention_head_dim,
            norm_num_groups=norm_num_groups, norm_eps=norm_eps, resnet_time_scale_shift=resnet_time_scale_shift,
            add_attention=add_attention, class_embed_type=None, num_class_embeds=None)
        self.sample_size = sample_size
        time_embed_dim = block_out_channels[0] * 4

        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], kernel_size=3, padding=(1, 1))
        self.time_proj = Timesteps(block_out_channels[0], flip_sin_to_cos, freq_shift)
        self.time_embedding = TimestepEmbedding(block_out_channels[0], time_embed_dim)
        self.class_embedding = None

        # registration order down_blocks -> up_blocks -> mid_block mirrors unet_2d.py:147-149 (state-dict key order)
        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])
        out_ch = block_out_channels[0]
        for i, typ in enumerate(down_block_types):
            in_ch, out_ch = out_ch, block_out_channels[i]
            final = i == len(block_out_channels) - 1
            self.down_blocks.append(_DOWN[typ](in_ch, out_ch, time_embed_dim, layers_per_block, norm_eps,
                                               norm_num_groups, attention_head_dim, downsample_padding,
                                               not final, dropout=dropout))
        self.mid_block = UNetMidBlock2D(block_out_channels[-1], time_embed_dim, norm_eps, norm_num_groups,
                                        attention_head_dim, mid_block_scale_factor, add_attention, dropout=dropout)
        rev = list(reversed(block_out_channels))
        out_ch = rev[0]
        for i, typ in enumerate(up_block_types):
            prev, out_ch = out_ch, rev[i]
            in_ch = rev[min(i + 1, len(block_out_channels) - 1)]
            final = i == len(block_out_channels) - 1
            self.up_blocks.append(_UP[typ](in_ch, prev, out_ch, time_embed_dim, layers_per_block + 1, norm_eps,
                                           norm_num_groups, attention_head_dim, not final, dropout=dropout))
        groups_out = norm_num_groups if norm_num_groups is not None else min(block_out_channels[0] // 4, 32)
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=groups_out, eps=norm_eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, kernel_size=3, padding=1)

    def __getstate__(self):
        # engine plans hold device buffers + ctypes structs: never pickled / deep-copied with the module
        # (torch.save(model) at ddpm_prune.py:135 and copy.deepcopy in op counters must keep working)
        d = self.__dict__.copy()
        d.pop("_dpb200_plans", None)
        d.pop("_dpb200_frozen", None)
        d.pop("_dpb200_weights_epoch", None)
        return d

    def __setstate__(self, state):
        super().__setstate__(state)
        if "config" not in self.__dict__ and "_internal_dict" in self.__dict__:
            self._adopt_reference_layout()

    def _adopt_reference_layout(self):
        """This instance was unpickled from a whole-module pickle written by the REFERENCE (`torch.save(model)`, ddpm_prune.py:135 /
        ddpm_train.py:487-493): its attribute soup is diffusers' (config in `_internal_dict`, processors, ...), its leaves carry
        the (possibly pruned) weights.  Rebuild this package's module tree from the stored config and transplant every leaf's
        tensors and widths; `Attention.scale` keeps the pickled (stale after pruning, attention_processor.py:87) value."""
        names = set(inspect.signature(UNet2DModel.__init__).parameters) - {"self", "unused"}
        cfg = {k: v for k, v in dict(self.__dict__["_internal_dict"]).items() if k in names and not k.startswith("_")}
        new = UNet2DModel(**cfg)
        for name, leaf in new.named_modules():
            if isinstance(leaf, (nn.Conv2d, nn.Linear, nn.GroupNorm)):
                src = self.get_submodule(name)
                leaf.weight = nn.Parameter(src.weight.detach().clone(), requires_grad=src.weight.requires_grad)
                if src.bias is not None:
                    leaf.bias = nn.Parameter(src.bias.detach().clone(), requires_grad=src.bias.requires_grad)
                if isinstance(leaf, nn.Conv2d):
                    leaf.out_channels, leaf.in_channels = leaf.weight.shape[0], leaf.weight.shape[1]
                elif isinstance(leaf, nn.Linear):
                    leaf.out_features, leaf.in_features = leaf.weight.shape
                else:
                    leaf.num_channels = leaf.weight.shape[0]
            elif isinstance(leaf, Attention):
                leaf.scale = float(self.get_submodule(name).scale)
            elif isinstance(leaf, nn.Dropout):
                leaf.p = float(self.get_submodule(name).p)
            elif isinstance(leaf, (Upsample2D, Downsample2D)):
                leaf.channels, leaf.out_channels = leaf.conv.in_channels, leaf.conv.out_channels
        for m in new.modules():      # widths of the containers' convs were set above; refresh the static attributes (ddpm_prune.py:112-116)
            if isinstance(m, (Upsample2D, Downsample2D)):
                m.channels, m.out_channels = m.conv.in_channels, m.conv.out_channels
        new.train(bool(self.__dict__.get("training", False)))
        self.__dict__.clear()
        self.__dict__.update(new.__dict__)

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _timesteps(self, sample, timestep):
        t = timestep
        if not torch.is_tensor(t):
            t = torch.tensor([t], dtype=torch.long, device=sample.device)
        elif t.dim() == 0:
            t = t[None].to(sample.device)
        return t * torch.ones(sample.shape[0], dtype=t.dtype, device=t.device)

    # ---- checkpoint I/O in the diffusers directory layout (checkpoint.py; modeling_utils.py:250-330, 333-680)
    def save_pretrained(self, save_directory, safe_serialization=False, **unused):
        from . import checkpoint
        checkpoint.save_model(self, save_directory, safe_serialization=safe_serialization)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **overrides):
        from . import checkpoint
        overrides = {k: v for k, v in overrides.items() if k in inspect.signature(cls.__init__).parameters}
        return checkpoint.load_model(cls, pretrained_model_name_or_path, subfolder=subfolder, **overrides)

    @classmethod
    def from_config(cls, config, **kw):
        from . import checkpoint
        cfg = dict(vars(config)) if not isinstance(config, dict) else dict(config)
        return checkpoint.build_from_config(cls, cfg, **kw)

    def forward(self, sample, timestep, class_labels=None, return_dict=True):
        if self.config.center_input_sample:
            sample = 2 * sample - 1.0
        timesteps = self._timesteps(sample, timestep)
        if tracing():
            out = self._forward_traced(sample, timesteps)
        else:
            if not sample.is_cuda:
                raise RuntimeError(
                    "diff_pruning_b200: UNet2DModel runs on the sm_90a CUDA engine only; move the model and "
                    "inputs to a CUDA device (CPU execution exists only under models.trace_mode() for "
                    "dependency tracing). No CPU fallback is provided.")
            from .engine import unet_apply
            out = unet_apply(self, sample, timesteps)
        if not return_dict:
            return (out,)
        return UNet2DOutput(sample=out)

    def _forward_traced(self, sample, timesteps):
        t_emb = self.time_proj(timesteps).to(dtype=self.dtype)
        emb = self.time_embedding(t_emb)
        sample = self.conv_in(sample)
        skips = (sample,)
        for blk in self.down_blocks:
            sample, res = blk(hidden_states=sample, temb=emb)
            skips += res
        sample = self.mid_block(sample, emb)
        for blk in self.up_blocks:
            n = len(blk.resnets)
            res, skips = skips[-n:], skips[:-n]
            sample = blk(sample, res, emb)
        return self.conv_out(self.conv_act(self.conv_norm_out(sample)))


def ddpm_alphas_cumprod(num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02):
    """scheduling_ddpm.py:141,157-158 (linear schedule), float32."""
    betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    return torch.cumprod(1.0 - betas, dim=0)


class DDPMScheduler:
    """Subset of scheduling_ddpm.py used on the hot path: tables (:123-169) and add_noise (:408-429)."""

    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, beta_schedule="linear", **unused):
        if beta_schedule != "linear":
            raise NotImplementedError(beta_schedule)
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                                      beta_end=beta_end, beta_schedule=beta_schedule)
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self._dev_tables = {}

    # ---- scheduler_config.json I/O (checkpoint.py; configuration_utils.py:138-170, scheduling_utils.py:83-160)
    def save_pretrained(self, save_directory, **unused):
        from . import checkpoint
        checkpoint.save_config(self, save_directory, checkpoint.SCHEDULER_CONFIG_NAME)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kw):
        from . import checkpoint
        cfg = checkpoint.load_config(pretrained_model_name_or_path, checkpoint.SCHEDULER_CONFIG_NAME, subfolder)
        return checkpoint.build_from_config(cls, cfg, **kw)

    @classmethod
    def from_config(cls, config, **kw):
        from . import checkpoint
        cfg = dict(vars(config)) if not isinstance(config, dict) else dict(config)
        return checkpoint.build_from_config(cls, cfg, **kw)

    def add_noise(self, original_samples, noise, timesteps):
        if original_samples.is_cuda and not tracing():
            from .engine import add_noise_cuda
            return add_noise_cuda(self, original_samples, noise, timesteps)
        if not tracing():
            raise RuntimeError("diff_pruning_b200: DDPMScheduler.add_noise is a CUDA op (no CPU fallback); "
                               "use models.trace_mode() for host-side structure tests")
        ac = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        a = (ac[timesteps] ** 0.5).flatten()
        s = ((1 - ac[timesteps]) ** 0.5).flatten()
        while a.dim() < original_samples.dim():
            a, s = a.unsqueeze(-1), s.unsqueeze(-1)
        return a * original_samples + s * noise


CIFAR10_DDPM_CONFIG = dict(  # tools/ddpm_cifar10_config.json (values only)
    sample_size=32, in_channels=3, out_channels=3, center_input_sample=False, time_embedding_type="positional",
    freq_shift=1, flip_sin_to_cos=False,
    down_block_types=("DownBlock2D", "AttnDownBlock2D", "DownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "UpBlock2D", "AttnUpBlock2D", "UpBlock2D"),
    block_out_channels=(128, 256, 256, 256), layers_per_block=2, mid_block_scale_factor=1, downsample_padding=0,
    act_fn="silu", attention_head_dim=None, norm_num_groups=32, norm_eps=1e-6)

LSUN256_DDPM_CONFIG = dict(  # google/ddpm-ema-{bedroom,church}-256 architecture (SURVEY.md §8 "C3")
    sample_size=256, in_channels=3, out_channels=3, center_input_sample=False, time_embedding_type="positional",
    freq_shift=1, flip_sin_to_cos=False,
    down_block_types=("DownBlock2D", "DownBlock2D", "DownBlock2D", "DownBlock2D", "AttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"),
    block_out_channels=(128, 128, 256, 256, 512, 512), layers_per_block=2, mid_block_scale_factor=1,
    downsample_padding=0, act_fn="silu", attention_head_dim=None, norm_num_groups=32, norm_eps=1e-6)

TINY_TEST_CONFIG = dict(  # small member of the same family for fast parity tests
    sample_size=16, in_channels=3, out_channels=3, center_input_sample=False, time_embedding_type="positional",
    freq_shift=1, flip_sin_to_cos=False, down_block_types=("DownBlock2D", "AttnDownBlock2D"),
    up_block_types=("AttnUpBlock2D", "UpBlock2D"), block_out_channels=(32, 64), layers_per_block=1,
    mid_block_scale_factor=1, downsample_padding=0, act_fn="silu", attention_head_dim=None, norm_num_groups=8,
    norm_eps=1e-6)
