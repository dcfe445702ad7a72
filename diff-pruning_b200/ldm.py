"""Latent-diffusion `UNetModel` (BASELINE configs[4]: ldm_exp/prune_ldm.py Taylor scoring on the class-conditional ImageNet LDM).

Module tree, construction order and parameter names of the reference's OpenAI-style UNet in its spatial-transformer configuration
(`ldm_exp/ldm/modules/diffusionmodules/openaimodel.py:413-742`, `ldm_exp/ldm/modules/attention.py:152-257`; cin256-v2.yaml:
model_channels 192, channel_mult (1,2,3,5), 2 res blocks, attention at ds {2,4,8}, num_heads 1, transformer_depth 1, context_dim 512),
so `torch.manual_seed(s); UNetModel(**cfg)` reproduces the reference's parameters (incl. its zero-initialised output convolutions) and
state-dict keys, and `torch_pruning`-style tools find real nn.Conv2d / nn.Linear / nn.GroupNorm / nn.LayerNorm leaves.

On CUDA the forward (and, through autograd, the backward) is the planned sm_90a engine (engine.Plan._build_ldm); under
models.trace_mode() the leaves run as torch ops (dependency tracing, host-side structure tests).  No CPU fallback otherwise.

Not rebuilt: the AttentionBlock (non-transformer) variant, resblock_updown, scale-shift norm, num_classes label embedding, 1-D / 3-D.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from .models import UNet2DOutput, tracing


def ldm_timestep_embedding(timesteps, dim, max_period=10000):
    """util.py:151-170: cos | sin, frequencies exp(-ln(max_period) * i / half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half).to(timesteps.device)
    args = timesteps[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def _zero(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


class Upsample(nn.Module):
    def __init__(self, channels, use_conv=True, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        if not use_conv:
            raise NotImplementedError("conv_resample=False")
        self.conv = nn.Conv2d(channels, self.out_channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2, mode="nearest"))


class Downsample(nn.Module):
    def __init__(self, channels, use_conv=True, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        if not use_conv:
            raise NotImplementedError("conv_resample=False")
        self.op = nn.Conv2d(channels, self.out_channels, 3, stride=2, padding=1)

    def forward(self, x):
        return self.op(x)


class ResBlock(nn.Module):
    """openaimodel.py:163-275 (use_scale_shift_norm False, no up/down)."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None):
        super().__init__()
        self.channels, self.emb_channels, self.dropout = channels, emb_channels, dropout
        self.out_channels = out_channels or channels
        self.in_layers = nn.Sequential(nn.GroupNorm(32, channels), nn.SiLU(), nn.Conv2d(channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(nn.GroupNorm(32, self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        _zero(nn.Conv2d(self.out_channels, self.out_channels, 3, padding=1)))
        self.skip_connection = nn.Identity() if self.out_channels == channels else nn.Conv2d(channels, self.out_channels, 1)

    def forward(self, x, emb):
        h = self.in_layers(x)
        h = h + self.emb_layers(emb)[:, :, None, None]
        return self.skip_connection(x) + self.out_layers(h)


class CrossAttention(nn.Module):
    """attention.py:152-193."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = query_dim if context_dim is None else context_dim
        self.scale, self.heads = dim_head ** -0.5, heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))

    def forward(self, x, context=None):
        h = self.heads
        context = x if context is None else context
        q, k, v = self.to_q(x), self.to_k(context), self.to_v(context)
        b = q.shape[0]

        def split(t):
            return t.reshape(b, t.shape[1], h, -1).permute(0, 2, 1, 3).reshape(b * h, t.shape[1], -1)
        q, k, v = split(q), split(k), split(v)
        attn = (torch.bmm(q, k.transpose(1, 2)) * self.scale).softmax(dim=-1)
        o = torch.bmm(attn, v)
        o = o.reshape(b, h, o.shape[1], -1).permute(0, 2, 1, 3).reshape(b, o.shape[1], -1)
        return self.to_out(o)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        x, gate = self.proj(x).chunk(2, dim=-1)
        return x * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4, dropout=0.0):
        super().__init__()
        inner = int(dim * mult)
        self.net = nn.Sequential(GEGLU(dim, inner), nn.Dropout(dropout), nn.Linear(inner, dim))

    def forward(self, x):
        return self.net(x)


class BasicTransformerBlock(nn.Module):
    """attention.py:196-212."""

    def __init__(self, dim, n_heads, d_head, dropout=0.0, context_dim=None):
        super().__init__()
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.ff = FeedForward(dim, dropout=dropout)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)

    def forward(self, x, context=None):
        x = self.attn1(self.norm1(x)) + x
        x = self.attn2(self.norm2(x), context=context) + x
        return self.ff(self.norm3(x)) + x


class SpatialTransformer(nn.Module):
    """attention.py:215-257."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None):
        super().__init__()
        self.in_channels = in_channels
        inner = n_heads * d_head
        self.norm = nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Conv2d(in_channels, inner, kernel_size=1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, n_heads, d_head, dropout=dropout, context_dim=context_dim)
                                                 for _ in range(depth)])
        self.proj_out = _zero(nn.Conv2d(inner, in_channels, kernel_size=1))

    def forward(self, x, context=None):
        b, c, h, w = x.shape
        x_in = x
        x = self.proj_in(self.norm(x))
        x = x.reshape(b, x.shape[1], h * w).transpose(1, 2)
        for blk in self.transformer_blocks:
            x = blk(x, context=context)
        x = x.transpose(1, 2).reshape(b, -1, h, w)
        return self.proj_out(x) + x_in


class TimestepEmbedSequential(nn.Sequential):
    def forward(self, x, emb, context=None):
        for layer in self:
            if isinstance(layer, ResBlock):
                x = layer(x, emb)
            elif isinstance(layer, SpatialTransformer):
                x = layer(x, context)
            else:
                x = layer(x)
        return x


class UNetModel(nn.Module):
    """openaimodel.py:413-742 (use_spatial_transformer=True family)."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions, dropout=0,
                 channel_mult=(1, 2, 4, 8), conv_resample=True, num_heads=-1, num_head_channels=-1, use_spatial_transformer=True,
                 transformer_depth=1, context_dim=None, legacy=True, **unused):
        super().__init__()
        if not use_spatial_transformer or context_dim is None:
            raise NotImplementedError("only the spatial-transformer (cross-attention conditioned) LDM UNet is on the path")
        if num_heads == -1 and num_head_channels == -1:
            raise ValueError("Either num_heads or num_head_channels has to be set")
        bad = {k: v for k, v in unused.items() if k in ("resblock_updown", "use_scale_shift_norm", "num_classes", "n_embed") and v}
        if bad:
            raise NotImplementedError(f"UNetModel options outside the cin256 family: {bad}")
        self.config = SimpleNamespace(image_size=image_size, in_channels=in_channels, model_channels=model_channels,
                                      out_channels=out_channels, num_res_blocks=num_res_blocks,
                                      attention_resolutions=tuple(attention_resolutions), dropout=dropout, channel_mult=tuple(channel_mult),
                                      num_heads=num_heads, num_head_channels=num_head_channels, transformer_depth=transformer_depth,
                                      context_dim=context_dim, sample_size=image_size)
        self.image_size, self.in_channels, self.model_channels, self.out_channels = image_size, in_channels, model_channels, out_channels
        ted = model_channels * 4
        self.time_embed = nn.Sequential(nn.Linear(model_channels, ted), nn.SiLU(), nn.Linear(ted, ted))

        def transformer(ch):
            if num_head_channels == -1:
                heads, dim_head = num_heads, ch // num_heads
            else:
                heads, dim_head = ch // num_head_channels, num_head_channels
            if legacy:
                dim_head = ch // heads
            return SpatialTransformer(ch, heads, dim_head, depth=transformer_depth, context_dim=context_dim)

        self.input_blocks = nn.ModuleList([TimestepEmbedSequential(nn.Conv2d(in_channels, model_channels, 3, padding=1))])
        chans, ch, ds = [model_channels], model_channels, 1
        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [ResBlock(ch, ted, dropout, out_channels=mult * model_channels)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    layers.append(transformer(ch))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, conv_resample, out_channels=ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(ResBlock(ch, ted, dropout), transformer(ch), ResBlock(ch, ted, dropout))
        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = chans.pop()
                layers = [ResBlock(ch + ich, ted, dropout, out_channels=model_channels * mult)]
                ch = model_channels * mult
                if ds in attention_resolutions:
                    layers.append(transformer(ch))
                if level and i == num_res_blocks:
                    layers.append(Upsample(ch, conv_resample, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(nn.GroupNorm(32, ch), nn.SiLU(), _zero(nn.Conv2d(model_channels, out_channels, 3, padding=1)))

    def __getstate__(self):
        d = self.__dict__.copy()
        for k in ("_dpb200_plans", "_dpb200_frozen", "_dpb200_weights_epoch"):
            d.pop(k, None)
        return d

    @property
    def device(self):
        return next(self.parameters()).device

    def forward(self, x, timesteps=None, context=None, y=None, return_dict=False, **kwargs):
        if y is not None:
            raise NotImplementedError("num_classes label embedding")
        if not torch.is_tensor(timesteps):
            timesteps = torch.tensor([timesteps], dtype=torch.long, device=x.device)
        if timesteps.dim() == 0:
            timesteps = timesteps[None]
        timesteps = timesteps.to(x.device) * torch.ones(x.shape[0], dtype=timesteps.dtype, device=x.device)
        if tracing():
            out = self._forward_traced(x, timesteps, context)
        else:
            if not x.is_cuda:
                raise RuntimeError("diff_pruning_b200: the LDM UNetModel runs on the sm_90a CUDA engine only (CPU execution exists only under "
                                   "models.trace_mode()). No CPU fallback is provided.")
            from .engine import unet_apply
            out = unet_apply(self, x, timesteps, context=context)
        return UNet2DOutput(sample=out) if return_dict else out

    def _forward_traced(self, x, timesteps, context):
        emb = self.time_embed(ldm_timestep_embedding(timesteps, self.model_channels))
        hs, h = [], x
        for module in self.input_blocks:
            h = module(h, emb, context)
            hs.append(h)
        h = self.middle_block(h, emb, context)
        for module in self.output_blocks:
            h = module(torch.cat([h, hs.pop()], dim=1), emb, context)
        return self.out(h)


def ldm_alphas_cumprod(num_timesteps=1000, linear_start=0.0015, linear_end=0.0195):
    """ldm/modules/diffusionmodules/util.py:21-27 `make_beta_schedule("linear")`: betas = linspace(sqrt(start), sqrt(end))^2 in float64,
    alphas_cumprod in float64 -> float32 (ldm/models/diffusion/ddpm.py:117-131)."""
    betas = torch.linspace(linear_start ** 0.5, linear_end ** 0.5, num_timesteps, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0).to(torch.float32)


CIN256_V2_CONFIG = dict(  # ldm_exp/configs/latent-diffusion/cin256-v2.yaml unet_config.params
    image_size=64, in_channels=3, out_channels=3, model_channels=192, attention_resolutions=(8, 4, 2), num_res_blocks=2,
    channel_mult=(1, 2, 3, 5), num_heads=1, use_spatial_transformer=True, transformer_depth=1, context_dim=512)

LDM_TINY_CONFIG = dict(  # small member of the same family for parity tests
    image_size=16, in_channels=3, out_channels=3, model_channels=32, attention_resolutions=(2, 1), num_res_blocks=1,
    channel_mult=(1, 2), num_heads=1, use_spatial_transformer=True, transformer_depth=1, context_dim=16)
