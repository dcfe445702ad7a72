"""The VQ-f4 first stage of the class-conditional LDM (cin256-v2.yaml first_stage_config: VQModelInterface, 8192 x 3 codebook,
Encoder / Decoder ch 128, ch_mult (1, 2, 4), 2 res blocks, no attention resolutions).

Module tree, construction order and parameter names of the reference's `ldm/modules/diffusionmodules/model.py:38-214,368-568`
(Normalize, Upsample, Downsample, ResnetBlock, AttnBlock, Encoder, Decoder) and of `ldm/models/autoencoder.py:14-43,264-282` (VQModel /
VQModelInterface, with taming's VectorQuantizer2 holding `embedding`), so `torch.manual_seed(s); Encoder(**cfg)` / `Decoder(**cfg)`
reproduce the reference modules' parameters and a Lightning checkpoint's `first_stage_model.{encoder,decoder,quantize,quant_conv,
post_quant_conv}.*` load as they are.  The encoder and quant_conv are built on request (with_encoder=True); the loss is not built.

On CUDA, VQModelInterface.decode is the planned sm_90a engine (engine.Plan._build_vq_decoder) behind dp_vq_quantize, and encode the
forward-only encoder plan (engine.Plan._build_vq_encoder), each one CUDA graph per micro-batch; under models.trace_mode() the modules run
as torch ops (structure tests).  No CPU fallback otherwise.
"""
from __future__ import annotations

import gc
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .engine import Plan, _stream, capture_graphs
from .models import tracing

VQ_F4_CONFIG = dict(  # ldm_exp/configs/latent-diffusion/cin256-v2.yaml first_stage_config.params
    embed_dim=3, n_embed=8192,
    ddconfig=dict(double_z=False, z_channels=3, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 4), num_res_blocks=2,
                  attn_resolutions=(), dropout=0.0))

DECODE_MICRO_BATCH = 8    # latents per decoder plan: about 1 GB of activations per 256 x 256 image, plus its 4096^2 attention matrix
ENCODE_MICRO_BATCH = 8    # images per encoder plan


def Normalize(in_channels, num_groups=32):
    """model.py:38-39."""
    return nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


def _silu(x):
    return x * torch.sigmoid(x)


class Upsample(nn.Module):
    """model.py:42-57 (with_conv): nearest x2, then a 3x3 convolution."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        if not with_conv:
            raise NotImplementedError("resamp_with_conv=False")
        self.with_conv = with_conv
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class Downsample(nn.Module):
    """model.py:60-79 (with_conv): F.pad(x, (0, 1, 0, 1)), then a 3x3 stride-2 convolution without padding."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        if not with_conv:
            raise NotImplementedError("resamp_with_conv=False")
        self.with_conv = with_conv
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class ResnetBlock(nn.Module):
    """model.py:82-141 as the encoder and decoder build it: no time embedding (temb_channels 0), a 1x1 nin_shortcut when the width
    changes."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        if temb_channels > 0 or conv_shortcut:
            raise NotImplementedError("the first stage's ResnetBlock has no time embedding and a 1x1 shortcut")
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = Normalize(out_channels)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, x, temb=None):
        h = self.conv1(_silu(self.norm1(x)))
        h = self.conv2(self.dropout(_silu(self.norm2(h))))
        if self.in_channels != self.out_channels:
            x = self.nin_shortcut(x)
        return x + h


class AttnBlock(nn.Module):
    """model.py:150-202: single-head attention over the H*W tokens, q / k / v / proj_out as 1x1 convolutions, the scale c^-0.5 applied
    to the q k^T product."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, x):
        h_ = self.norm(x)
        q, k, v = self.q(h_), self.k(h_), self.v(h_)
        b, c, h, w = q.shape
        w_ = torch.bmm(q.reshape(b, c, h * w).permute(0, 2, 1), k.reshape(b, c, h * w)) * (int(c) ** (-0.5))
        w_ = F.softmax(w_, dim=2)
        h_ = torch.bmm(v.reshape(b, c, h * w), w_.permute(0, 2, 1)).reshape(b, c, h, w)
        return x + self.proj_out(h_)


class Encoder(nn.Module):
    """model.py:368-460 (attn_type "vanilla", double_z False)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels, resolution, z_channels, double_z=True, use_linear_attn=False, attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        if use_linear_attn or attn_type != "vanilla" or double_z:
            raise NotImplementedError("only the vanilla-attention Encoder with double_z=False (the VQ-f4 first stage)")
        self.ch, self.temb_ch = ch, 0
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.resolution, self.in_channels = resolution, in_channels
        self.conv_in = nn.Conv2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
        self.down = nn.ModuleList()
        for i_level in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            down = nn.Module()
            down.block = block
            down.attn = attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, z_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x):
        if not tracing():
            raise RuntimeError("diff_pruning_b200: the Encoder runs on the engine through VQModelInterface.encode (CPU execution exists "
                               "only under models.trace_mode())")
        h = self.conv_in(x)
        for i_level in range(self.num_resolutions):
            for i_block in range(self.num_res_blocks):
                h = self.down[i_level].block[i_block](h)
                if len(self.down[i_level].attn) > 0:
                    h = self.down[i_level].attn[i_block](h)
            if i_level != self.num_resolutions - 1:
                h = self.down[i_level].downsample(h)
        h = self.mid.block_2(self.mid.attn_1(self.mid.block_1(h)))
        return self.conv_out(_silu(self.norm_out(h)))


class Decoder(nn.Module):
    """model.py:462-568 (attn_type "vanilla", give_pre_end False, tanh_out False)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False, use_linear_attn=False, attn_type="vanilla",
                 **ignorekwargs):
        super().__init__()
        if use_linear_attn or attn_type != "vanilla" or give_pre_end or tanh_out:
            raise NotImplementedError("only the vanilla-attention Decoder without give_pre_end / tanh_out (the VQ-f4 first stage)")
        self.ch, self.temb_ch = ch, 0
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.resolution, self.in_channels = resolution, in_channels
        self.give_pre_end, self.tanh_out = give_pre_end, tanh_out
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.conv_in = nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block = block
            up.attn = attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def forward(self, z):
        if not tracing():
            raise RuntimeError("diff_pruning_b200: the Decoder runs on the engine through VQModelInterface.decode (CPU execution exists "
                               "only under models.trace_mode())")
        h = self.mid.block_2(self.mid.attn_1(self.mid.block_1(self.conv_in(z))))
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                h = self.up[i_level].block[i_block](h)
                if len(self.up[i_level].attn) > 0:
                    h = self.up[i_level].attn[i_block](h)
            if i_level != 0:
                h = self.up[i_level].upsample(h)
        return self.conv_out(_silu(self.norm_out(h)))


class _EncodePath(nn.Module):
    """encoder -> quant_conv of a VQModelInterface (its encode()): the module an encoder plan is built from (engine.Plan._build_vq_encoder).
    It shares the interface's parameters and is not part of its module tree or state dict."""

    def __init__(self, encoder, quant_conv):
        super().__init__()
        self.encoder, self.quant_conv = encoder, quant_conv


class VectorQuantizer(nn.Module):
    """taming's VectorQuantizer2 as the decode path uses it: the codebook `embedding` ([n_e, e_dim], initialised U(-1/n_e, 1/n_e)).
    The nearest code is chosen by dp_vq_quantize's fp64 distance (include/dpb200.h); remap / sane_index_shape are not supported."""

    def __init__(self, n_e, e_dim, beta=0.25, remap=None, unknown_index="random", sane_index_shape=False, legacy=True):
        super().__init__()
        if remap is not None or sane_index_shape:
            raise NotImplementedError("VectorQuantizer remap / sane_index_shape")
        self.n_e, self.e_dim, self.beta, self.legacy = n_e, e_dim, beta, legacy
        self.embedding = nn.Embedding(self.n_e, self.e_dim)
        self.embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)


class VQModelInterface(nn.Module):
    """autoencoder.py:264-282 (VQModel's constructor, :14-43): `encoder` (with_encoder=True), `decoder`, `quantize`, `quant_conv`
    (with_encoder=True) and `post_quant_conv` in the reference's construction and state-dict order, so with the encoder a seeded
    VQModelInterface draws the reference's parameters (its loss, torch.nn.Identity for cin256-v2, holds none).  decode() and encode() run
    on the engine in micro-batches of `decode_batch` latents / `encode_batch` images."""

    def __init__(self, embed_dim, ddconfig, lossconfig=None, n_embed=8192, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None, remap=None, sane_index_shape=False, use_ema=False, with_encoder=False, **unused):
        super().__init__()
        if ckpt_path is not None or colorize_nlabels is not None or use_ema:
            raise NotImplementedError("VQModelInterface ckpt_path / colorize_nlabels / use_ema")
        self.embed_dim, self.n_embed, self.image_key = embed_dim, n_embed, image_key
        if with_encoder:
            self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.quantize = VectorQuantizer(n_embed, embed_dim, beta=0.25, remap=remap, sane_index_shape=sane_index_shape)
        if with_encoder:
            self.quant_conv = nn.Conv2d(ddconfig["z_channels"], embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.decode_batch = DECODE_MICRO_BATCH
        self.encode_batch = ENCODE_MICRO_BATCH

    def __getstate__(self):
        d = self.__dict__.copy()
        d.pop("_dpb200_decode", None)
        d.pop("_dpb200_encode", None)
        return d

    use_graph = True     # tests clear it on an instance to run the launch list eagerly

    @torch.no_grad()
    def encode(self, x):
        """autoencoder.py:269-272: quant_conv(encoder(x)), no quantisation.  x: (B, in_channels, H, W) fp32 on CUDA, H and W multiples of
        2^(len(ch_mult) - 1) (the reference's F.pad + stride-2 convolution takes odd sides too; the engine's does not).  Returns
        (B, embed_dim, H / 4, W / 4) for VQ-f4."""
        if not hasattr(self, "encoder"):
            raise NotImplementedError("this VQModelInterface was built without its encoder: pass with_encoder=True")
        if tracing():
            return self.quant_conv(self.encoder(x))
        if not x.is_cuda:
            raise RuntimeError("diff_pruning_b200: VQModelInterface.encode runs on a CUDA device (no CPU fallback)")
        if x.dtype != torch.float32:
            raise TypeError(f"diff_pruning_b200: the encoder computes in fp32; got {x.dtype}")
        f = 2 ** (self.encoder.num_resolutions - 1)
        H, W = x.shape[2:]
        if H % f or W % f:
            raise NotImplementedError(f"the engine's encoder takes images whose sides are multiples of {f}; got {H} x {W}")
        return self._micro_batched(x, self.encode_batch, self.encode_chunk)

    def encode_chunk(self, x) -> SimpleNamespace:
        """Encode up to encode_batch images into the micro-batch plan's output buffer (`.plan.y_out`, padded NHWC) and return the runner.
        A short chunk is padded with zero images, for the reason decode_chunk gives."""
        n, _, H, W = x.shape
        assert 0 < n <= self.encode_batch
        B = self.encode_batch

        def setup(run):        # dp_nchw_to_nhwc of `.x` into the plan's input
            run.x = torch.zeros((B, self.encoder.in_channels, H, W), device=x.device, dtype=torch.float32)
            x_in = run.plan.x_in
            return lambda: L.check(run.lib.dp_nchw_to_nhwc(run.x.data_ptr(), x_in.ptr, x_in.ld, B, x_in.C, H, W, _stream()), "nchw->nhwc")
        run = self._runner("_dpb200_encode", _EncodePath(self.encoder, self.quant_conv), B, H, W, (), x.device, setup)
        return self._run_chunk(run, run.x, x)

    @torch.no_grad()
    def decode(self, h, force_not_quantize=False, inv_scale: float = 1.0):
        """autoencoder.py:274-282: quantize (unless force_not_quantize) -> post_quant_conv -> decoder.  h: (B, embed_dim, H, W) fp32 on
        CUDA; inv_scale multiplies h first, in fp32 (decode_first_stage's 1 / scale_factor).  Returns (B, out_ch, 4H, 4W) for VQ-f4."""
        if tracing():
            return self._decode_traced(h, force_not_quantize, inv_scale)
        if not h.is_cuda:
            raise RuntimeError("diff_pruning_b200: VQModelInterface.decode runs on a CUDA device (no CPU fallback)")
        if h.dtype != torch.float32:
            raise TypeError(f"diff_pruning_b200: the decoder computes in fp32; got {h.dtype}")
        return self._micro_batched(h, self.decode_batch, lambda z: self.decode_chunk(z, force_not_quantize, inv_scale))

    def decode_chunk(self, h, force_not_quantize=False, inv_scale: float = 1.0, indices: bool = False) -> SimpleNamespace:
        """Decode up to decode_batch latents into the micro-batch plan's output buffer (`.plan.y_out`, padded NHWC) and return the
        runner.  A short chunk is padded with zero latents, so nothing of an earlier chunk reaches the per-tensor operand scales of this
        one's tensor-core convolutions: a chunk's images depend on its own latents only.  indices=True also leaves the chosen
        codes in `.indices` ([decode_batch, H, W] int64)."""
        n, _, H, W = h.shape
        assert 0 < n <= self.decode_batch
        B, fnq, inv_scale = self.decode_batch, bool(force_not_quantize), float(inv_scale)

        def setup(run):        # dp_vq_quantize of `.z` into the plan's input, writing `.indices` when asked to
            run.z = torch.zeros((B, self.embed_dim, H, W), device=h.device, dtype=torch.float32)
            run.indices = torch.zeros((B, H, W), device=h.device, dtype=torch.int64)
            run.want_indices = [False]
            emb, x_in = self.quantize.embedding.weight, run.plan.x_in

            def stage():
                idx = run.indices.data_ptr() if (run.want_indices[0] and not fnq) else None
                L.check(run.lib.dp_vq_quantize(run.z.data_ptr(), B, self.embed_dim, H, W, inv_scale, emb.data_ptr(), self.n_embed,
                                               0 if fnq else 1, x_in.ptr, x_in.ld, idx, _stream()), "vq_quantize")
            return stage
        run = self._runner("_dpb200_decode", self, B, H, W, (fnq, inv_scale), h.device, setup)
        run.want_indices[0] = indices
        return self._run_chunk(run, run.z, h, eager=indices)

    def _runner(self, slot, module, B, H, W, extra, device, setup) -> SimpleNamespace:
        """The forward-only plan of `module` at (B, H, W), kept in __dict__[slot], and with use_graph its captured graph.  setup(run)
        allocates the runner's input buffers and returns the staging launch into the plan's input; run.body() is that launch, then the
        forward.  A different request (`extra` holds what else the staging launch depends on), or parameters replaced since, frees the
        old plan first."""
        key = (B, H, W, *extra, str(device), self.use_graph)
        sig = tuple((p.data_ptr(), tuple(p.shape)) for p in module.parameters())
        run = self.__dict__.get(slot)
        if run is not None and run.key == key and run.plan.signature() == sig:
            return run
        self.__dict__.pop(slot, None)
        run = None
        gc.collect()
        torch.cuda.empty_cache()
        plan = Plan(module, B, H, W, device, need_grad=False)
        run = SimpleNamespace(key=key, plan=plan, lib=L.load(), graph=None)
        stage = setup(run)

        def body():
            stage()
            plan.run_forward()
        run.body = body
        plan.ensure_packed()
        if self.use_graph:
            run.graph, = capture_graphs(device, body)
        self.__dict__[slot] = run
        return run

    @staticmethod
    def _run_chunk(run, buf, x, eager=False) -> SimpleNamespace:
        """x into the runner's input buffer, its tail zeroed for a short chunk, then one graph replay (or body() when eager)."""
        n = x.shape[0]
        buf[:n].copy_(x, non_blocking=True)
        if n < buf.shape[0]:
            buf[n:].zero_()
        run.plan.ensure_packed()
        if run.graph is not None and not eager:
            run.graph.replay()
        else:
            run.body()
        return run

    @staticmethod
    def _micro_batched(x, mb, chunk):
        """chunk() over micro-batches of mb along x's batch, each chunk's padded NHWC output gathered into one NCHW tensor."""
        B = x.shape[0]
        out = None
        for s in range(0, B, mb):
            run = chunk(x[s:s + mb])
            y = run.plan.y_out
            if out is None:
                out = torch.empty((B, y.C, y.H, y.W), device=x.device, dtype=torch.float32)
            n = min(mb, B - s)
            L.check(run.lib.dp_nhwc_to_nchw(y.ptr, y.ld, out[s:s + n].data_ptr(), n, y.C, y.H, y.W, 0, _stream()), "nhwc->nchw")
        return out

    def _decode_traced(self, h, force_not_quantize, inv_scale):
        """Host restatement used under models.trace_mode(): the same codebook choice as dp_vq_quantize (fp64 distances, lowest index on
        a tie) and z + (e - z)."""
        z = h * torch.tensor(inv_scale, dtype=h.dtype)
        if not force_not_quantize:
            e = self.quantize.embedding.weight
            zf = z.permute(0, 2, 3, 1).reshape(-1, self.embed_dim)
            d = None
            for c in range(self.embed_dim):
                t = (zf[:, c:c + 1].double() - e[:, c].double()[None]) ** 2
                d = t if d is None else d + t
            idx = d.argmin(1)
            zq = zf + (e[idx] - zf)
            z = zq.reshape(h.shape[0], h.shape[2], h.shape[3], -1).permute(0, 3, 1, 2)
        return self.decoder(self.post_quant_conv(z))
