"""ORACLE — test infrastructure only (same rules as unet_oracle.py: tests and scripts, never the product).

A torch functional restatement of ddpm_exp's Model forward (ddpm_exp/models/diffusion.py) and of generalized_steps
(functions/denoising.py:10-33), evaluated from a flat state dict in float32 or float64 (the dtype of the weights and inputs it is given).
Widths come from the weights, so pruned networks evaluate as they are; the block structure (levels, blocks per level, where attention
and the nin_shortcut sit) from the keys.

Parity pin: tests/test_ddpm_exp_host.py checks it against tests/golden/ddpm_exp_tiny.pt, written by tools/gen_golden.py from the
UNMODIFIED reference modules.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def timestep_embedding(t: Tensor, dim: int, dtype) -> Tensor:
    """diffusion.py:6-24: sin | cos of t * exp(arange(half) * -(ln(1e4) / (half - 1))), the frequencies rounded in float32 as the
    reference rounds them, the product and sin / cos in `dtype`."""
    half = dim // 2
    freqs = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1))).to(device=t.device, dtype=dtype)
    e = t.to(dtype)[:, None] * freqs[None]
    e = torch.cat([torch.sin(e), torch.cos(e)], 1)
    return F.pad(e, (0, 1, 0, 0)) if dim % 2 else e


def _silu(x):
    return x * torch.sigmoid(x)


def _norm(sd, name, x):
    """diffusion.py:31-32: GroupNorm(32, eps 1e-6)."""
    return F.group_norm(x, 32, sd[name + ".weight"], sd[name + ".bias"], eps=1e-6)


def _conv(sd, name, x, pad=1, stride=1):
    return F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"], stride=stride, padding=pad)


def resnet(sd, name, x, temb, shortcut: bool):
    """diffusion.py:113-136 (dropout off)."""
    h = _conv(sd, name + ".conv1", _silu(_norm(sd, name + ".norm1", x)))
    h = h + F.linear(_silu(temb), sd[name + ".temb_proj.weight"], sd[name + ".temb_proj.bias"])[:, :, None, None]
    h = _conv(sd, name + ".conv2", _silu(_norm(sd, name + ".norm2", h)))
    if shortcut:
        x = _conv(sd, name + ".nin_shortcut", x, pad=0)
    return x + h


def attn(sd, name, x):
    """diffusion.py:166-189: the scale is int(c) ** -0.5 with c = q's width."""
    h_ = _norm(sd, name + ".norm", x)
    q, k, v = (_conv(sd, f"{name}.{n}", h_, pad=0) for n in "qkv")
    b, c, h, w = q.shape
    w_ = torch.bmm(q.reshape(b, c, h * w).permute(0, 2, 1), k.reshape(b, c, h * w)) * (int(c) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    h_ = torch.bmm(v.reshape(b, v.shape[1], h * w), w_.permute(0, 2, 1)).reshape(b, v.shape[1], h, w)
    return x + _conv(sd, name + ".proj_out", h_, pad=0)


def _count(sd, prefix) -> int:
    n = 0
    while any(k.startswith(f"{prefix}.{n}.") for k in sd):
        n += 1
    return n


def forward(sd: Dict[str, Tensor], x: Tensor, t: Tensor, shortcuts: Dict[str, bool] = None) -> Tensor:
    """Model.forward (diffusion.py:268-300).  shortcuts: block name -> whether it applies its nin_shortcut (the reference decides by
    its construction-time in_channels != out_channels); by default, whether the block has one."""
    dt = x.dtype
    sc = (lambda n: shortcuts[n]) if shortcuts is not None else (lambda n: f"{n}.nin_shortcut.weight" in sd)
    ch = sd["temb.dense.0.weight"].shape[1]
    temb = timestep_embedding(t, ch, dt)
    temb = F.linear(_silu(F.linear(temb, sd["temb.dense.0.weight"], sd["temb.dense.0.bias"])), sd["temb.dense.1.weight"],
                    sd["temb.dense.1.bias"])
    L = _count(sd, "down")
    hs: List[Tensor] = [_conv(sd, "conv_in", x)]
    for i in range(L):
        nb = _count(sd, f"down.{i}.block")
        for j in range(nb):
            n = f"down.{i}.block.{j}"
            h = resnet(sd, n, hs[-1], temb, sc(n))
            if f"down.{i}.attn.0.q.weight" in sd:
                h = attn(sd, f"down.{i}.attn.{j}", h)
            hs.append(h)
        if f"down.{i}.downsample.conv.weight" in sd:
            hs.append(_conv(sd, f"down.{i}.downsample.conv", F.pad(hs[-1], (0, 1, 0, 1)), pad=0, stride=2))
    h = resnet(sd, "mid.block_1", hs[-1], temb, sc("mid.block_1"))
    h = attn(sd, "mid.attn_1", h)
    h = resnet(sd, "mid.block_2", h, temb, sc("mid.block_2"))
    for i in reversed(range(L)):
        for j in range(_count(sd, f"up.{i}.block")):
            n = f"up.{i}.block.{j}"
            h = resnet(sd, n, torch.cat([h, hs.pop()], dim=1), temb, sc(n))
            if f"up.{i}.attn.0.q.weight" in sd:
                h = attn(sd, f"up.{i}.attn.{j}", h)
        if f"up.{i}.upsample.conv.weight" in sd:
            h = _conv(sd, f"up.{i}.upsample.conv", F.interpolate(h, scale_factor=2.0, mode="nearest"))
    h = _silu(_norm(sd, "norm_out", h))
    return _conv(sd, "conv_out", h)


def shortcuts_of(model) -> Dict[str, bool]:
    """Block name -> in_channels != out_channels of a Model's ResnetBlocks (what the reference tests at run time)."""
    return {n: m.in_channels != m.out_channels for n, m in model.named_modules() if hasattr(m, "temb_proj")}


def alphas(betas: Tensor) -> Tensor:
    """compute_alpha's table (denoising.py:4-7): (1 - cat([0], betas)).cumprod(0), in the dtype of betas."""
    return (1 - torch.cat([torch.zeros(1, dtype=betas.dtype, device=betas.device), betas])).cumprod(0)


def generalized_update(x: Tensor, e: Tensor, noise: Tensor, at: Tensor, at_next: Tensor, eta: float):
    """One update of generalized_steps (denoising.py:21-30), in the reference's operation order.  Returns (x', x0)."""
    x0 = (x - e * (1 - at).sqrt()) / at.sqrt()
    c1 = eta * ((1 - at / at_next) * (1 - at_next) / (1 - at)).sqrt()
    c2 = ((1 - at_next) - c1 ** 2).sqrt()
    return at_next.sqrt() * x0 + c1 * noise + c2 * e, x0


def generalized_steps(eps_fn, x: Tensor, seq, betas: Tensor, eta: float, noises: List[Tensor]):
    """generalized_steps with eps_fn(x, t) as the model and the step noise given (noises[k] for the k-th step in sampling order).
    Returns (xs, x0_preds) as the reference does: x_T first."""
    a = alphas(betas)
    seq_next = [-1] + list(seq[:-1])
    xs, x0s = [x], []
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t = torch.full((x.shape[0],), float(i), dtype=x.dtype)
        e = eps_fn(xs[-1], t)
        xn, x0 = generalized_update(xs[-1], e, noises[k], a[i + 1].view(1), a[j + 1].view(1), eta)
        xs.append(xn)
        x0s.append(x0)
    return xs, x0s


def distinct_vectors(model, seed: int = 1):
    """Adds seeded N(0, 0.01^2) noise to every 1-D parameter of a Model (biases, GroupNorm affine) in parameters() order, so that every
    entry of every parameter is distinct: the pruned-network fixture then records which channels the reference's pruner kept as index
    lists, and prune_like rebuilds the network from them."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(torch.randn(p.shape, generator=g) * 0.01)
    return model


def prune_like(model, keep: Dict[str, tuple]):
    """The reference pruner's slicing (ddpm_exp/torch_pruning/pruner/function.py: conv / linear out and in channels, GroupNorm
    channels): parameter `name` becomes its rows keep[name][0] and columns keep[name][1] (None: all), a new nn.Parameter, and the layer's
    channel counts follow its weight, as the pruner sets them.  The ResnetBlock / AttnBlock ints stay as built, as after the pruner."""
    import torch.nn as nn
    with torch.no_grad():
        for name, (rows, cols) in keep.items():
            mod_name, attr = name.rsplit(".", 1)
            mod = model.get_submodule(mod_name)
            p = getattr(mod, attr)
            if rows is not None:
                p = p[torch.tensor(rows)]
            if cols is not None:
                p = p[:, torch.tensor(cols)]
            setattr(mod, attr, nn.Parameter(p.clone()))
    for mod in model.modules():
        if isinstance(mod, nn.Conv2d):
            mod.out_channels, mod.in_channels = mod.weight.shape[0], mod.weight.shape[1]
        elif isinstance(mod, nn.Linear):
            mod.out_features, mod.in_features = mod.weight.shape
        elif isinstance(mod, nn.GroupNorm):
            mod.num_channels = mod.weight.shape[0]
    return model
