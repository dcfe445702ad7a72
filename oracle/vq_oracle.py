"""ORACLE — test infrastructure only (same rules as unet_oracle.py: tests and scripts, never the product).

A torch functional restatement of the decode side of the LDM's VQ first stage, quantize -> post_quant_conv -> Decoder, evaluated from
a flat state dict in float32 or float64 (the dtype of the weights and the latent it is given).  Each function cites the reference lines
it restates.

Parity pin: tests/test_vq_decoder_host.py checks it against tests/golden/vq_decoder_tiny.pt, written by tools/gen_golden.py from the
UNMODIFIED reference Decoder (`ldm_exp/ldm/modules/diffusionmodules/model.py`).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def nearest_code(z: Tensor, e: Tensor) -> Tensor:
    """The codebook choice dp_vq_quantize makes (include/dpb200.h): per row of z [n, D], argmin over j of the float64 sum
    ((z_0 - e_j0)^2 + (z_1 - e_j1)^2) + ..., the lowest index on a tie (torch.argmin returns the first minimum)."""
    d = None
    for c in range(z.shape[1]):
        t = (z[:, c:c + 1].double() - e[:, c].double()[None]) ** 2
        d = t if d is None else d + t
    return d.argmin(1)


def nearest_code_taming(z: Tensor, e: Tensor) -> Tensor:
    """taming's VectorQuantizer2.forward as recalled (taming-transformers is not in the reference tree): in the dtype of z,
    d = sum(z^2) + sum(e^2) - 2 z e^T through a matmul, then argmin."""
    d = (z ** 2).sum(1, keepdim=True) + (e ** 2).sum(1) - 2 * torch.einsum("bd,dn->bn", z, e.t())
    return d.argmin(1)


def nearest_code_cdist(z: Tensor, e: Tensor) -> Tensor:
    """diffusers/models/vae.py:338 (the in-tree VectorQuantizer): argmin of torch.cdist(z, e)."""
    return torch.cdist(z, e).argmin(1)


def quantize(z: Tensor, e: Tensor, inv_scale: float = 1.0):
    """ddpm.py:713 (`1. / scale_factor * z`, in the dtype of z) then VectorQuantizer2's decode-path output z + (e - z) with the
    nearest_code choice (autoencoder.py:276-277).  z: NCHW.  Returns (z_q NCHW, indices [N, H, W])."""
    z = z * torch.tensor(inv_scale, dtype=z.dtype)
    N, D, H, W = z.shape
    zf = z.permute(0, 2, 3, 1).reshape(-1, D)
    idx = nearest_code(zf, e)
    zq = zf + (e[idx].to(z.dtype) - zf)
    return zq.reshape(N, H, W, D).permute(0, 3, 1, 2), idx.reshape(N, H, W)


def _conv(sd, name, x, pad):
    return F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"], padding=pad)


def _norm(sd, name, x):
    """model.py:38-39: GroupNorm(32, eps 1e-6)."""
    return F.group_norm(x, 32, sd[name + ".weight"], sd[name + ".bias"], eps=1e-6)


def _silu(x):
    """model.py:33-35: x * sigmoid(x)."""
    return x * torch.sigmoid(x)


def resnet_block(sd, p: str, x: Tensor) -> Tensor:
    """model.py:121-141 with temb None (dropout 0): norm1 -> swish -> conv1 -> norm2 -> swish -> conv2 ; + (nin_shortcut(x) | x)."""
    h = _conv(sd, p + "conv1", _silu(_norm(sd, p + "norm1", x)), 1)
    h = _conv(sd, p + "conv2", _silu(_norm(sd, p + "norm2", h)), 1)
    if p + "nin_shortcut.weight" in sd:
        x = _conv(sd, p + "nin_shortcut", x, 0)
    return x + h


def attn_block(sd, p: str, x: Tensor) -> Tensor:
    """model.py:178-202: q k^T over the H*W tokens, times int(c)^-0.5, softmax over the keys, times v, proj_out ; + x."""
    h_ = _norm(sd, p + "norm", x)
    q, k, v = (_conv(sd, p + n, h_, 0) for n in ("q", "k", "v"))
    b, c, h, w = q.shape
    w_ = torch.bmm(q.reshape(b, c, h * w).permute(0, 2, 1), k.reshape(b, c, h * w)) * (int(c) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    h_ = torch.bmm(v.reshape(b, c, h * w), w_.permute(0, 2, 1)).reshape(b, c, h, w)
    return x + _conv(sd, p + "proj_out", h_, 0)


def decoder(sd: Dict[str, Tensor], cfg: dict, z: Tensor) -> Tensor:
    """Decoder.forward (model.py:535-568, give_pre_end / tanh_out False): conv_in -> mid.block_1 / attn_1 / block_2 -> per level from the
    lowest resolution: num_res_blocks + 1 resnet blocks (+ attention), nearest x2 + conv except at level 0 -> norm_out -> swish -> conv_out.
    sd: the Decoder's own state dict (no prefix)."""
    h = _conv(sd, "conv_in", z, 1)
    h = resnet_block(sd, "mid.block_2.", attn_block(sd, "mid.attn_1.", resnet_block(sd, "mid.block_1.", h)))
    for i_level in reversed(range(len(cfg["ch_mult"]))):
        for i_block in range(cfg["num_res_blocks"] + 1):
            h = resnet_block(sd, f"up.{i_level}.block.{i_block}.", h)
            if f"up.{i_level}.attn.{i_block}.q.weight" in sd:
                h = attn_block(sd, f"up.{i_level}.attn.{i_block}.", h)
        if i_level != 0:
            h = _conv(sd, f"up.{i_level}.upsample.conv", F.interpolate(h, scale_factor=2.0, mode="nearest"), 1)
    return _conv(sd, "conv_out", _silu(_norm(sd, "norm_out", h)), 1)


def decode(sd: Dict[str, Tensor], cfg: dict, h: Tensor, force_not_quantize: bool = False, inv_scale: float = 1.0) -> Tensor:
    """VQModelInterface.decode (autoencoder.py:274-282) after decode_first_stage's 1 / scale_factor: quantize (unless
    force_not_quantize) -> post_quant_conv -> decoder.  sd: VQModelInterface's state dict (decoder.*, quantize.embedding.weight,
    post_quant_conv.*); cfg: its ddconfig."""
    if force_not_quantize:
        z = h * torch.tensor(inv_scale, dtype=h.dtype)
    else:
        z, _ = quantize(h, sd["quantize.embedding.weight"], inv_scale)
    z = _conv(sd, "post_quant_conv", z, 0)
    dsd = {k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")}
    return decoder(dsd, cfg, z)


def state_dict_digest(sd: Dict[str, Tensor]) -> str:
    """sha256 over the float32 bytes of the state dict's tensors in key order."""
    import hashlib
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.detach().to(torch.float32).contiguous().numpy().tobytes())
    return h.hexdigest()
