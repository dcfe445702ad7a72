"""ORACLE — test infrastructure only (same rules as oracle/vq_oracle.py: tests and scripts, never the product).

A torch functional restatement of the encode side of the LDM's VQ first stage, Encoder -> quant_conv, evaluated from a flat state dict in
float32 or float64 (the dtype of the weights and the images it is given), on the building blocks of oracle/vq_oracle.py (convolution,
GroupNorm, swish, ResnetBlock, AttnBlock).  Each function cites the reference lines it restates.

Parity pin: tests/test_vq_encoder_host.py checks it against tests/golden/vq_encoder_tiny.pt, written by tools/gen_golden.py from the
UNMODIFIED reference Encoder (`ldm_exp/ldm/modules/diffusionmodules/model.py`) and VQModelInterface.encode (`ldm/models/autoencoder.py`).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle.vq_oracle import _conv, _norm, _silu, attn_block, resnet_block

Tensor = torch.Tensor


def encoder(sd: Dict[str, Tensor], cfg: dict, x: Tensor) -> Tensor:
    """Encoder.forward (model.py:428-460, double_z False): conv_in -> per level: num_res_blocks resnet blocks (+ attention), then, except
    at the last level, Downsample (model.py:72-79: F.pad(x, (0, 1, 0, 1)) and a 3x3 stride-2 convolution without padding) ->
    mid.block_1 / attn_1 / block_2 -> norm_out -> swish -> conv_out.  sd: the Encoder's own state dict (no prefix)."""
    h = _conv(sd, "conv_in", x, 1)
    n = len(cfg["ch_mult"])
    for i_level in range(n):
        for i_block in range(cfg["num_res_blocks"]):
            h = resnet_block(sd, f"down.{i_level}.block.{i_block}.", h)
            if f"down.{i_level}.attn.{i_block}.q.weight" in sd:
                h = attn_block(sd, f"down.{i_level}.attn.{i_block}.", h)
        if i_level != n - 1:
            p = f"down.{i_level}.downsample.conv"
            h = F.conv2d(F.pad(h, (0, 1, 0, 1), mode="constant", value=0), sd[p + ".weight"], sd[p + ".bias"], stride=2)
    h = resnet_block(sd, "mid.block_2.", attn_block(sd, "mid.attn_1.", resnet_block(sd, "mid.block_1.", h)))
    return _conv(sd, "conv_out", _silu(_norm(sd, "norm_out", h)), 1)


def encode(sd: Dict[str, Tensor], cfg: dict, x: Tensor) -> Tensor:
    """VQModelInterface.encode (autoencoder.py:269-272): quant_conv(encoder(x)), no quantisation.  sd: VQModelInterface's state dict
    (encoder.*, quant_conv.*, ...); cfg: its ddconfig."""
    esd = {k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}
    return _conv(sd, "quant_conv", encoder(esd, cfg, x), 0)
