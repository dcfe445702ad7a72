"""prune_ldm.py's sample-then-score loop (BASELINE configs[4], ldm_exp/prune_ldm.py:105-131) on the engine, in latent space.

ClassEmbedder    — ldm/modules/encoders/modules.py:21-33 (`embedding.weight`), the cin256-v2 conditioning (1001 classes, 1000 = unconditional).
LatentDiffusion  — a thin container of what the loop uses of ldm/models/diffusion/ddpm.py's LatentDiffusion: `model.diffusion_model` (the
                   UNetModel of ldm.py), `cond_stage_model`, the schedule buffers, get_learned_conditioning / apply_model / get_loss_at_t,
                   and load_state_dict of a Lightning checkpoint's `state_dict`.  Not a Lightning module; no EMA; the VQ first
                   stage (`first_stage_model`: decode_first_stage, and encode_first_stage / get_first_stage_encoding when it holds
                   its encoder) when built with first_stage_config.
DDIMSampler      — ldm/models/diffusion/ddim.py: the same `sample(...)` call and results.  The whole S-step sample is ONE CUDA graph: per
                   step a fill of the timestep, the no-grad plan's forward at batch 2B (unconditional | conditional), and dp_ddim_cfg_step,
                   which forms the guided eps, writes x_prev and feeds both halves of the next forward's input.
LDMPruneScorer   — the loop itself: classes -> guided DDIM-20 sample -> get_loss_at_t at t = iteration on the samples with fresh noise ->
                   the stop rule of --pruner diff-pruning / diff0 -> backward into the UNet's gradient arena.  With encode_samples=True it
                   is test_criterion.py's loop instead: the samples go through encode_first_stage before get_loss_at_t.
sample_for_fid   — sample_for_FID.py's render-and-score loop: guided DDIM samples, decode_first_stage on the engine (autoencoder.py), the
                   save_image bytes on the device, FID moments of those bytes and / or the PNG files.

Gradients reach the UNet only: the reference's trainable ClassEmbedder also gets a gradient from loss.backward(), but the pruner looks at
`diffusion_model` alone, and the context enters the engine as a constant input.

Under torch.distributed with W > 1 ranks (one process per GPU, torchrun) both loops shard and return the single-process result on every
rank.  They run in rounds of W consecutive iterations (LDMPruneScorer) or batches (sample_for_fid), rank r taking the r-th of each round.
Rank 0 draws the round's random inputs (class labels, x_T, per-step noise, q_sample noise) in the single-process order and broadcasts
each iteration's draws, so no other rank's random state is read.  LDMPruneScorer all-reduces the round's losses and every rank replays
the stop rule over them in iteration order; the gradient arena is all-reduced once at the end.  sample_for_fid shares the FID moments'
shift (rank 0's first batch) and all-reduces the moments once at the end.  Only all_reduce and broadcast are used, on tensors of the
model's device.  shard=False keeps every rank a replica.
"""
from __future__ import annotations

import os
import random
from contextlib import contextmanager
from types import SimpleNamespace
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib as L
from .autoencoder import VQModelInterface
from .engine import _stream, capture_graphs, frozen_weights, get_plan
from .ldm import CIN256_V2_CONFIG, UNetModel
from .scoring import TaylorScorer, _dist_ready


class ClassEmbedder(nn.Module):
    """modules.py:21-33: batch[key] (B,) class labels -> (B, 1, embed_dim)."""

    def __init__(self, embed_dim: int, n_classes: int = 1001, key: str = "class_label"):
        super().__init__()
        self.key = key
        self.embedding = nn.Embedding(n_classes, embed_dim)

    def forward(self, batch, key=None):
        return self.embedding(batch[self.key if key is None else key][:, None])


class DiffusionWrapper(nn.Module):
    """ddpm.py DiffusionWrapper with conditioning_key 'crossattn': holds `diffusion_model` (the state-dict prefix `model.diffusion_model.`)."""

    def __init__(self, diffusion_model: UNetModel):
        super().__init__()
        self.diffusion_model = diffusion_model
        self.conditioning_key = "crossattn"

    def forward(self, x, t, c_crossattn=None):
        return self.diffusion_model(x, t, context=torch.cat(list(c_crossattn), 1))


def make_ddim_timesteps(num_ddim_timesteps: int, num_ddpm_timesteps: int = 1000) -> np.ndarray:
    """util.py make_ddim_timesteps, 'uniform': range(0, T, T // S) + 1."""
    c = num_ddpm_timesteps // num_ddim_timesteps
    return np.asarray(list(range(0, num_ddpm_timesteps, c))) + 1


def ddim_schedule(alphas_cumprod: torch.Tensor, S: int, eta: float) -> SimpleNamespace:
    """DDIMSampler.make_schedule's DDIM arrays (ddim.py:24-53, util.py make_ddim_sampling_parameters) in the dtypes the reference ends up
    with: alphas = float32 table entries, alphas_prev = float64 array of float32 values, sigmas = float64 (eta times the float64 square root
    of a mix of float64 and float32 terms; pinned bit for bit by tests/test_ldm_sampling_host.py), sqrt(1 - alphas) in float32.  `coefs[index]` are the fp32 scalars p_sample_ddim forms from them
    (ddim.py:190-202): (sqrt(1 - a_t), sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev - sigma^2), sigma)."""
    ac = alphas_cumprod.detach().to("cpu", torch.float32)
    ts = make_ddim_timesteps(S, ac.shape[0])
    alphas = ac[ts]
    alphas_prev = np.asarray([float(ac[0])] + ac[ts[:-1]].tolist())
    ap64 = torch.from_numpy(alphas_prev)
    # (1 - alphas_prev) / (1 - alphas) is ndarray / float32 tensor, which torch evaluates as the float32 reciprocal of the divisor
    # times the float64 numerator; alphas / alphas_prev is float32 / float64, a float64 quotient
    sigmas = eta * torch.sqrt((1 - alphas).reciprocal().double() * (1 - ap64) * (1 - alphas.double() / ap64))
    sqrt_one_minus = torch.sqrt(1. - alphas)
    f32 = lambda v: torch.tensor([float(v)], dtype=torch.float32)        # torch.full((b, 1, 1, 1), v): a float32 fill
    coefs = []
    for i in range(S):
        a_t, a_prev, sigma_t, sb = f32(alphas[i]), f32(alphas_prev[i]), f32(sigmas[i]), f32(sqrt_one_minus[i])
        coefs.append((float(sb), float(a_t.sqrt()), float(a_prev.sqrt()), float((1. - a_prev - sigma_t ** 2).sqrt()), float(sigma_t)))
    return SimpleNamespace(ddim_timesteps=ts, ddim_alphas=alphas, ddim_alphas_prev=alphas_prev, ddim_sigmas=sigmas,
                           ddim_sqrt_one_minus_alphas=sqrt_one_minus, coefs=coefs)


class _MSELoss(torch.autograd.Function):
    """mean((out - target)^2) and its gradient 2 (out - target) / n from one dp_mse_loss_grad launch (the kernel of the fast path)."""

    @staticmethod
    def forward(ctx, out, target):
        lib = L.load()
        o, tg = out.contiguous(), target.contiguous()
        n = o.numel()
        grad = torch.empty_like(o)
        loss = torch.zeros(1, device=o.device, dtype=torch.float32)
        partial = torch.empty(max(1, lib.dp_mse_partials(n)), device=o.device, dtype=torch.float32)
        L.check(lib.dp_mse_loss_grad(o.data_ptr(), tg.data_ptr(), grad.data_ptr(), n, 1.0 / n, 2.0 / n, partial.data_ptr(),
                                     loss.data_ptr(), _stream()), "mse")
        ctx.save_for_backward(grad)
        return loss[0]

    @staticmethod
    def backward(ctx, gout):
        grad, = ctx.saved_tensors
        return grad * gout, None


class LatentDiffusion(nn.Module):
    """What prune_ldm.py uses of ldm/models/diffusion/ddpm.py's LatentDiffusion at the cin256-v2 settings (eps parameterisation, l2 loss,
    l_simple_weight 1, logvar 0, original_elbo_weight 0, linear schedule 0.0015..0.0195 over 1000 steps, class-label cross-attention)."""

    def __init__(self, unet_config: Optional[dict] = None, cond_stage_config: Optional[dict] = None, timesteps: int = 1000,
                 linear_start: float = 0.0015, linear_end: float = 0.0195, cond_stage_key: str = "class_label",
                 first_stage_config: Optional[dict] = None, scale_factor: float = 1.0):
        """first_stage_config: VQModelInterface's parameters (autoencoder.VQ_F4_CONFIG for cin256-v2, plus with_encoder=True for the encode
        side) to hold the first stage as `first_stage_model`; None (the default) leaves it out, as the latent-space loops need it not.
        scale_factor: the config's (cin256-v2 leaves it at 1.0)."""
        super().__init__()
        self.model = DiffusionWrapper(UNetModel(**(unet_config or CIN256_V2_CONFIG)))
        self.scale_factor = scale_factor        # ddpm.py:456-457 (scale_by_std False: a plain attribute, not in the state dict)
        if first_stage_config is not None:
            self.first_stage_model = VQModelInterface(**first_stage_config).eval()
        self.cond_stage_model = ClassEmbedder(**(cond_stage_config or dict(embed_dim=512, n_classes=1001, key=cond_stage_key)))
        self.cond_stage_key = cond_stage_key
        self.parameterization = "eps"
        self.num_timesteps = timesteps
        # ddpm.py:117-145: float64 schedule, stored as float32
        betas = torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2
        ac = torch.cumprod(1.0 - betas, dim=0)
        self.register_buffer("betas", betas.float())
        self.register_buffer("alphas_cumprod", ac.float())
        self.register_buffer("alphas_cumprod_prev", torch.cat([torch.ones(1, dtype=torch.float64), ac[:-1]]).float())

    @property
    def device(self):
        return self.betas.device

    def load_state_dict(self, state_dict, strict: bool = True):
        """A Lightning checkpoint's `state_dict` (prune_ldm.py:21-28): `model.diffusion_model.*`, `cond_stage_model.*` and the three
        schedule buffers are loaded; `first_stage_model.*` (the VQ-f4 autoencoder), `model_ema.*` and the schedule buffers this container
        does not hold are ignored.  With a first stage, its `quantize.*`, `post_quant_conv.*` and `decoder.*` load too, and its
        `encoder.*` and `quant_conv.*` when it was built with its encoder (its loss is not built)."""
        own = set(self.state_dict().keys())
        prefixes = ("model.diffusion_model.", "cond_stage_model.")
        if hasattr(self, "first_stage_model"):
            parts = ("quantize", "post_quant_conv", "decoder")
            if hasattr(self.first_stage_model, "encoder"):
                parts += ("encoder", "quant_conv")
            prefixes += tuple(f"first_stage_model.{m}." for m in parts)
        keep = {k: v for k, v in state_dict.items() if k.startswith(prefixes) or (k in own and "." not in k)}
        return super().load_state_dict(keep, strict=strict)

    @contextmanager
    def ema_scope(self, context=None):
        """ddpm.py:171-184 with use_ema False (cin256-v2): the weights in use are the weights."""
        yield None

    @torch.no_grad()
    def decode_first_stage(self, z, predict_cids=False, force_not_quantize=False):
        """ddpm.py:706-765 without the patch-wise path: z / scale_factor (fp32) -> first_stage_model.decode, on the engine."""
        if predict_cids:
            raise NotImplementedError("decode_first_stage(predict_cids=True)")
        if hasattr(self, "split_input_params"):
            raise NotImplementedError("patch-wise decoding (split_input_params)")
        if not hasattr(self, "first_stage_model"):
            raise RuntimeError("this LatentDiffusion was built without first_stage_config: it holds no decoder")
        inv = float(torch.tensor(1. / self.scale_factor, dtype=torch.float32))   # the fp32 scalar of `1. / self.scale_factor * z`
        return self.first_stage_model.decode(z, force_not_quantize=predict_cids or force_not_quantize, inv_scale=inv)

    @torch.no_grad()
    def encode_first_stage(self, x):
        """ddpm.py:826-863 without the patch-wise path: first_stage_model.encode on the engine (quant_conv(encoder(x)), no quantisation)."""
        if hasattr(self, "split_input_params"):
            raise NotImplementedError("patch-wise encoding (split_input_params)")
        if not hasattr(self, "first_stage_model"):
            raise RuntimeError("this LatentDiffusion was built without first_stage_config: it holds no encoder")
        return self.first_stage_model.encode(x)

    def get_first_stage_encoding(self, encoder_posterior):
        """ddpm.py:542-549 for the VQ first stage, whose encode() returns a tensor: scale_factor * z (the KL first stage's
        DiagonalGaussianDistribution is not built)."""
        if not torch.is_tensor(encoder_posterior):
            raise NotImplementedError(f"encoder_posterior of type '{type(encoder_posterior)}' not yet implemented")
        return self.scale_factor * encoder_posterior

    def get_learned_conditioning(self, c):
        """ddpm.py get_learned_conditioning with the ClassEmbedder: {cond_stage_key: (B,) labels} -> (B, 1, embed_dim)."""
        return self.cond_stage_model(c)

    def apply_model(self, x_noisy, t, cond):
        """ddpm.py:901-924 for crossattn conditioning: the UNet with context = cond (a tensor, or a list / {'c_crossattn': [...]}).
        The context is a constant of the engine's forward (no gradient flows into it)."""
        if isinstance(cond, dict):
            cond = cond["c_crossattn"]
        if isinstance(cond, (list, tuple)):
            cond = torch.cat(list(cond), 1)
        return self.model.diffusion_model(x_noisy, t, context=cond.detach())

    def q_sample(self, x_start, t, noise):
        """ddpm.py:275-278 on the device (dp_add_noise: sqrt of the float32 alphas_cumprod entry, within an ulp of the reference's
        float32-rounded float64 square roots; the fast path uses the same kernel)."""
        x, nz = x_start.contiguous(), noise.contiguous()
        out = torch.empty_like(x)
        B, C_, H, W = x.shape
        tt = t.to(device=x.device, dtype=torch.int64).contiguous()
        acp = self.alphas_cumprod.to(x.device).contiguous()
        L.check(L.load().dp_add_noise(x.data_ptr(), nz.data_ptr(), tt.data_ptr(), acp.data_ptr(), out.data_ptr(), B, C_, H, W, 0, 0,
                                      _stream()), "add_noise")
        return out

    def get_loss_at_t(self, x, c, t, noise=None):
        """ddpm.py:881-889 -> p_losses (:1022-1056) at the cin256-v2 values: the mean over C, H, W per image, then over the batch, of
        (eps_hat - noise)^2 — one mean over all elements, as one kernel forms it with its gradient.  With logvar 0 and
        original_elbo_weight 0 the other terms add exactly 0.  Returns (loss, loss_dict) like the reference."""
        if isinstance(c, dict):
            c = self.get_learned_conditioning(c)
        noise = torch.randn_like(x) if noise is None else noise
        if not torch.is_tensor(t):
            t = torch.full((x.shape[0],), int(t), dtype=torch.long, device=x.device)
        out = self.apply_model(self.q_sample(x.detach(), t, noise), t, c)
        loss = _MSELoss.apply(out, noise)
        prefix = "train" if self.training else "val"
        return loss, {f"{prefix}/loss_simple": loss.detach(), f"{prefix}/loss": loss.detach()}


class DDIMSampler:
    """ldm/models/diffusion/ddim.py on the engine (uniform discretisation, eta, classifier-free guidance).

    x_T (when not given) and the sigma noise are drawn with torch.randn on `generator` (the default generator of the device when None):
    x_T first, then one (B, C, H, W) draw per step.  With eta == 0 no per-step noise is drawn; the reference draws it and multiplies it by
    zero, so after an eta-0 sample the random stream is where the reference's is not."""

    def __init__(self, model: LatentDiffusion, schedule: str = "linear", **kwargs):
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.use_graph = True
        self._graphs: Dict[tuple, SimpleNamespace] = {}
        self.last_run: Optional[SimpleNamespace] = None    # static buffers of the last sample: every step's x_prev / pred_x0

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        if ddim_discretize != "uniform":
            raise NotImplementedError(f"ddim_discretize={ddim_discretize!r}: only the uniform DDIM discretisation is on the engine")
        sch = ddim_schedule(self.model.alphas_cumprod, ddim_num_steps, ddim_eta)
        for k, v in vars(sch).items():
            setattr(self, k, v)

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None, quantize_x0=False,
               eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None, verbose=True,
               x_T=None, log_every_t=100, unconditional_guidance_scale=1., unconditional_conditioning=None, generator=None,
               step_noise=None, **kwargs):
        """ddim.py:55-104 + ddim_sampling (:106-163): returns (samples, {'x_inter': [...], 'pred_x0': [...]}) with x_T first and the
        steps whose index % log_every_t == 0 or index == S - 1 after it.  step_noise: the (S, B, C, H, W) per-step noise drawn
        beforehand, used in place of the S draws on `generator` when eta > 0 (ignored when eta == 0)."""
        unsupported = {"mask / x0": mask is not None or x0 is not None, "quantize_x0": quantize_x0, "score_corrector": score_corrector is not None,
                       "temperature != 1": temperature != 1., "noise_dropout": noise_dropout > 0., "callback / img_callback":
                       callback is not None or img_callback is not None, "ddim_use_original_steps": kwargs.get("ddim_use_original_steps", False),
                       "ddim_discretize != uniform": kwargs.get("ddim_discretize", "uniform") != "uniform"}
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError(f"DDIMSampler options outside prune_ldm's sampling: {bad}")
        if not torch.is_tensor(conditioning):
            raise NotImplementedError("conditioning must be the (B, 1, context_dim) tensor get_learned_conditioning returns")
        self.make_schedule(S, ddim_eta=eta, verbose=verbose)
        unet = self.model.model.diffusion_model
        dev = unet.device
        if dev.type != "cuda":
            raise RuntimeError("diff_pruning_b200: DDIMSampler samples on a CUDA device (no CPU fallback)")
        C_, H, W = shape
        B = batch_size
        guided = unconditional_conditioning is not None and unconditional_guidance_scale != 1.
        gdev = generator.device if generator is not None else dev
        if x_T is None:
            x_T = torch.randn((B, C_, H, W), generator=generator, device=gdev, dtype=torch.float32)
        was_training = unet.training
        unet.eval()
        try:
            frozen = unet.__dict__.get("_dpb200_frozen", False)
            with (_nullctx() if frozen else frozen_weights(unet)):
                plan = get_plan(unet, 2 * B if guided else B, H, W, dev, need_grad=False)
                plan.ensure_packed()
                run = self._run_for(plan, S, float(eta), float(unconditional_guidance_scale), guided, B, C_, H, W)
                run.x_T.copy_(x_T.to(dev, torch.float32).reshape(B, C_, H, W))
                ctx = conditioning.reshape(B, 1, -1)
                if guided:
                    ctx = torch.cat([unconditional_conditioning.reshape(B, 1, -1).to(ctx.device), ctx])
                plan.load_context(ctx)
                if run.noise is not None and step_noise is not None:
                    run.noise.copy_(step_noise.to(dev, torch.float32).reshape(S, B, C_, H, W))
                elif run.noise is not None:
                    for i in range(S):
                        run.noise[i].copy_(torch.randn((B, C_, H, W), generator=generator, device=gdev, dtype=torch.float32))
                if run.graph is not None:
                    run.graph.replay()
                else:
                    run.body()
        finally:
            unet.train(was_training)
        self.last_run = run
        inter = {"x_inter": [run.x_T.clone()], "pred_x0": [run.x_T.clone()]}
        for i in range(S):
            index = S - i - 1
            if index % log_every_t == 0 or index == S - 1:
                inter["x_inter"].append(run.xs[i].clone())
                inter["pred_x0"].append(run.x0s[i].clone())
        return run.xs[S - 1].clone(), inter

    def _run_for(self, plan, S, eta, scale, guided, B, C_, H, W) -> SimpleNamespace:
        """The static buffers and the captured graph of one (plan, S, eta, scale), built on first use."""
        key = (id(plan), S, eta, scale, guided, self.use_graph)
        run = self._graphs.get(key)
        if run is not None and run.plan is plan:
            return run
        lib, dev = L.load(), plan.dev
        run = SimpleNamespace(plan=plan, graph=None)
        run.x_T = torch.empty((B, C_, H, W), device=dev, dtype=torch.float32)
        run.xs = torch.empty((S, B, C_, H, W), device=dev, dtype=torch.float32)      # x_prev of step i
        run.x0s = torch.empty((S, B, C_, H, W), device=dev, dtype=torch.float32)     # pred_x0 of step i
        run.noise = torch.empty((S, B, C_, H, W), device=dev, dtype=torch.float32) if eta > 0 else None
        steps = [(int(step), S - i - 1) for i, step in enumerate(np.flip(self.ddim_timesteps))]
        coefs = list(self.coefs)
        x_in, y_out = plan.x_in, plan.y_out
        half_in = B * H * W * x_in.ld * 4

        def body():
            s = _stream()
            L.check(lib.dp_nchw_to_nhwc(run.x_T.data_ptr(), x_in.ptr, x_in.ld, B, C_, H, W, s), "x_T nchw->nhwc")
            if guided:
                L.check(lib.dp_nchw_to_nhwc(run.x_T.data_ptr(), x_in.ptr + half_in, x_in.ld, B, C_, H, W, s), "x_T nchw->nhwc")
            for i, (step, index) in enumerate(steps):
                plan.t_dev.fill_(step)
                plan.run_forward(s)
                sb, sa, sap, dirc, sigma = coefs[index]
                x = run.x_T if i == 0 else run.xs[i - 1]
                nz = run.noise[i].data_ptr() if (run.noise is not None and sigma != 0.) else None
                L.check(lib.dp_ddim_cfg_step(y_out.ptr, y_out.ld, x.data_ptr(), nz, run.xs[i].data_ptr(), x_in.ptr, x_in.ld,
                                             run.x0s[i].data_ptr(), B, C_, H, W, 1 if guided else 0, scale, sb, sa, sap, dirc, sigma, s),
                        "ddim_cfg_step")
        run.body = body
        if self.use_graph:
            run.x_T.zero_()
            if run.noise is not None:
                run.noise.zero_()
            run.graph, = capture_graphs(dev, body)
        self._graphs[key] = run
        return run


class _nullctx:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


def _world_rank(shard: bool):
    """(world size, rank) of the default process group when `shard` and it has more than one rank; (1, 0) otherwise."""
    if shard and _dist_ready():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def _round_inputs(draw: Callable[[], Dict[str, torch.Tensor]], spec: Dict[str, tuple], n: int, world: int, rank: int, dev):
    """The random inputs of this rank's iteration in a round of n <= world consecutive iterations (None when rank >= n).  Rank 0 calls
    draw() n times, in iteration order, as the single-process loop would, and broadcasts iteration j's draws for rank j; spec gives
    their {name: (shape, dtype)} for the receiving buffers on `dev`.  Rank 0 keeps its own draws where draw() made them."""
    mine = None
    for j in range(n):
        got = draw() if rank == 0 else None
        if j > 0:
            if got is not None:
                bad = {k: tuple(v.shape) for k, v in got.items() if (tuple(v.shape), v.dtype) != (tuple(spec[k][0]), spec[k][1])}
                if bad or set(got) != set(spec):
                    raise RuntimeError(f"drawn inputs {bad or sorted(got)} do not match the broadcast layout {spec}")
                got = {k: v.to(dev) for k, v in got.items()}
            else:
                got = {k: torch.empty(shape, dtype=dtype, device=dev) for k, (shape, dtype) in spec.items()}
            for k in spec:
                dist.broadcast(got[k], 0)
        if j == rank:
            mine = got
    return mine


PRUNE_LDM_THRESHOLDS = {"taylor": None, "diff-pruning": 0.1, "diff0": 0.0}


class PruneLDMStopRule:
    """prune_ldm.py:120-131: max_loss (starting at -1) is updated FIRST, then `diff-pruning` (0.1) / `diff0` (0.0) stop when
    loss / max_loss < thr, BEFORE loss.backward() — the stopping iteration's gradient is not accumulated.  `taylor` never stops.
    The quotient and the comparison are fp32, as on the reference's 0-dim fp32 tensors."""

    def __init__(self, pruner: str):
        if pruner not in PRUNE_LDM_THRESHOLDS:
            raise ValueError(f"pruner must be one of {sorted(PRUNE_LDM_THRESHOLDS)}, got {pruner!r}")
        self.thr = PRUNE_LDM_THRESHOLDS[pruner]
        self.max_loss = np.float32(-1.0)

    def stop(self, loss: float) -> bool:
        l32 = np.float32(loss)
        if l32 > self.max_loss:
            self.max_loss = l32
        if self.thr is None:
            return False
        with np.errstate(divide="ignore", invalid="ignore"):
            return bool(np.float32(l32 / self.max_loss) < np.float32(self.thr))


class LDMPruneScorer:
    """The fast path of prune_ldm.py:105-131: per iteration t = 0, 1, ...: B random classes (`class_sampler(B)`, by default
    random.sample(range(1000), B) on the module-level `random` as the script does), their context, a guided DDIM sample of B latents
    (DDIMSampler: one graph replay), then get_loss_at_t(samples, t, fresh noise) as two graphs — forward + loss, whose loss is read back
    to the host for the stop rule, and the backward, which accumulates into the UNet's Parameter.grad (the plan's gradient arena).

    encode_samples=True runs test_criterion.py:108-135 instead: the same loop with encoded = encode_first_stage(samples) (the encoder
    plan's graph, autoencoder.py) between the sample and get_loss_at_t, which then scores the encoded latents (3 x 16 x 16 for a
    3 x 64 x 64 cin256-v2 sample) at the same t and with the same stop rule.  The model's first stage must hold its encoder."""

    def __init__(self, model: LatentDiffusion, n_samples_per_class: int = 6, ddim_steps: int = 20, scale: float = 3.0, eta: float = 0.0,
                 use_graph: bool = True, encode_samples: bool = False):
        if encode_samples and not hasattr(getattr(model, "first_stage_model", None), "encoder"):
            raise ValueError("encode_samples=True needs a first stage built with its encoder (first_stage_config with_encoder=True)")
        self.encode_samples = encode_samples
        self.model = model
        self.B, self.S, self.scale, self.eta = n_samples_per_class, ddim_steps, float(scale), float(eta)
        self.unet = model.model.diffusion_model
        self.dev = self.unet.device
        cfg = self.unet.config
        self.shape = (cfg.in_channels, cfg.image_size, cfg.image_size)
        self.loss_shape = (self.B,) + self.shape         # the latents get_loss_at_t scores (and its noise)
        if encode_samples:
            fs = model.first_stage_model
            f = 2 ** (fs.encoder.num_resolutions - 1)
            self.loss_shape = (self.B, fs.embed_dim, cfg.image_size // f, cfg.image_size // f)
        self.use_graph = use_graph
        self.sampler = DDIMSampler(model)
        self.sampler.use_graph = use_graph
        self.ts: Optional[TaylorScorer] = None
        self.g_fwd = self.g_bwd = None
        self.stopped_at: Optional[int] = None

    def _draw(self, class_sampler, generator) -> Dict[str, torch.Tensor]:
        """One iteration's random inputs, in the order the loop consumes them: the class labels (`class_sampler(B)`, or random.sample on
        the module-level `random`), then on `generator` x_T, the per-step noise (eta > 0 only) and the q_sample noise."""
        gdev = generator.device if generator is not None else self.dev
        labels = class_sampler(self.B) if class_sampler is not None else random.sample(range(1000), self.B)
        d = {"labels": torch.as_tensor(labels, dtype=torch.long)}
        d["x_T"] = torch.randn((self.B,) + self.shape, generator=generator, device=gdev, dtype=torch.float32)
        if self.eta > 0:
            d["step_noise"] = torch.stack([torch.randn((self.B,) + self.shape, generator=generator, device=gdev, dtype=torch.float32)
                                           for _ in range(self.S)])
        d["noise"] = torch.randn(self.loss_shape, generator=generator, device=gdev, dtype=torch.float32)
        return d

    def _draw_spec(self) -> Dict[str, tuple]:
        spec = {"labels": ((self.B,), torch.long), "x_T": ((self.B,) + self.shape, torch.float32)}
        if self.eta > 0:
            spec["step_noise"] = ((self.S, self.B) + self.shape, torch.float32)
        spec["noise"] = (self.loss_shape, torch.float32)
        return spec

    def _scorer(self, samples, noise, c) -> TaylorScorer:
        if self.ts is None:
            self.ts = TaylorScorer(self.unet, samples, noise, alphas_cumprod=self.model.alphas_cumprod, use_graph=False, context=c)
        else:
            self.ts.clean.copy_(samples)
            self.ts.noise.copy_(noise)
            self.ts.plan.load_context(c)
        return self.ts

    def _fwd(self):
        self.ts._refresh_noise()
        self.ts._forward_loss()

    def _bwd(self):
        self.ts.plan.run_backward(_stream())

    def _forward(self, t: int, d: Dict[str, torch.Tensor], uc: torch.Tensor) -> torch.Tensor:
        """Iteration t up to its stop check: context, guided DDIM sample from d's x_T (and step noise), the encoder with encode_samples,
        then forward + loss at t with d's noise.  Returns the device loss (1,)."""
        model, B = self.model, self.B
        c = model.get_learned_conditioning({model.cond_stage_key: d["labels"].to(self.dev)})
        samples, _ = self.sampler.sample(S=self.S, conditioning=c, batch_size=B, shape=list(self.shape), verbose=False,
                                         unconditional_guidance_scale=self.scale, unconditional_conditioning=uc, eta=self.eta,
                                         x_T=d["x_T"], step_noise=d.get("step_noise"))
        if self.encode_samples:
            samples = model.encode_first_stage(samples)
        if tuple(samples.shape) != self.loss_shape:
            raise RuntimeError(f"the scored latents are {tuple(samples.shape)}, the loss noise was drawn as {self.loss_shape}")
        ts = self._scorer(samples, d["noise"].to(self.dev), c)
        p = ts.plan
        p.check_current()
        p.attach_grads()
        p.ensure_packed()
        p.t_dev.fill_(t)
        if self.use_graph:
            if self.g_fwd is None:
                self.g_fwd, self.g_bwd = capture_graphs(self.dev, self._fwd, self._bwd, restore=(p.grad_arena,))
            self.g_fwd.replay()
        else:
            self._fwd()
        return ts.loss

    def _backward(self):
        if self.use_graph:
            self.g_bwd.replay()
        else:
            self._bwd()

    def _grad_arena(self, uc: torch.Tensor) -> torch.Tensor:
        """The UNet's gradient arena; a rank that ran no iteration (iterations < world) builds the Taylor plan to have one."""
        if self.ts is None:
            z = torch.zeros(self.loss_shape, device=self.dev, dtype=torch.float32)
            self._scorer(z, z, uc)
        p = self.ts.plan
        p.check_current()
        p.attach_grads()
        return p.grad_arena

    def run(self, pruner: str = "taylor", iterations: int = 1000, class_sampler: Optional[Callable[[int], Sequence[int]]] = None,
            generator: Optional[torch.Generator] = None, shard: bool = True) -> torch.Tensor:
        """The loop of prune_ldm.py:105-131 (test_criterion.py:108-135 with encode_samples) for `pruner` in {taylor, diff-pruning,
        diff0}.  Returns the losses of the iterations that ran (with the stopping one last when the rule stopped the loop, its gradient
        not accumulated; self.stopped_at is its index).

        With torch.distributed initialised over W > 1 ranks (and shard=True) the iterations run in rounds of W: rank r runs iteration
        r0 + r on the inputs rank 0 drew for it, the round's losses are all-reduced (each rank fills its own slot of a W-vector) and every
        rank replays the stop rule over them in iteration order; an iteration at or after the stopping one skips its backward.  After the
        last round the gradient arena is all-reduced (SUM) once.  Every rank returns the single-process losses and stopped_at, and holds
        the single-process gradient up to fp32 summation order.  The gradient already in Parameter.grad counts once, rank 0's: the other
        ranks zero theirs first."""
        rule = PruneLDMStopRule(pruner)
        model, B = self.model, self.B
        world, rank = _world_rank(shard and iterations > 0)
        losses: List[float] = []
        self.stopped_at = None
        was_training = self.unet.training
        self.unet.eval()                     # prune_ldm.py:72
        try:
            with torch.no_grad(), frozen_weights(self.unet):
                uc = model.get_learned_conditioning({model.cond_stage_key: torch.full((B,), 1000, dtype=torch.long, device=self.dev)})
                if rank > 0:
                    for p in self.unet.parameters():
                        if p.grad is not None:
                            p.grad.zero_()
                spec = self._draw_spec()
                for r0 in range(0, iterations, world):
                    n = min(world, iterations - r0)
                    d = _round_inputs(lambda: self._draw(class_sampler, generator), spec, n, world, rank, self.dev)
                    rl = torch.zeros(world, device=self.dev, dtype=torch.float32)
                    if d is not None:
                        rl[rank:rank + 1].copy_(self._forward(r0 + rank, d, uc))
                    if world > 1:
                        dist.all_reduce(rl, op=dist.ReduceOp.SUM)      # x + 0 is x: every rank reads the losses bit for bit
                    stop = None
                    for j, loss in enumerate(rl.tolist()[:n]):
                        losses.append(loss)
                        if rule.stop(loss):
                            stop = j
                            break
                    if d is not None and (stop is None or rank < stop):
                        self._backward()
                    if stop is not None:
                        self.stopped_at = r0 + stop
                        break
                if world > 1:
                    dist.all_reduce(self._grad_arena(uc), op=dist.ReduceOp.SUM)
        finally:
            self.unet.train(was_training)
        return torch.tensor(losses, dtype=torch.float32)


@torch.no_grad()
def sample_for_fid(model: LatentDiffusion, classes: Sequence[int] = range(1000), ipc: int = 50, batch_size: int = 50, ddim_steps: int = 250,
                   eta: float = 0., scale: float = 3.0, out_dir: Optional[str] = None, fid_dims: int = 2048, inception=None,
                   generator: Optional[torch.Generator] = None, decode_batch: int = 8, shard: bool = True):
    """sample_for_FID.py:67-100: uc once; then ipc // batch_size rounds over `classes`, each a guided DDIM sample of batch_size latents
    (DDIMSampler, one graph), decode_first_stage in micro-batches of decode_batch (one graph each) and dp_decode_images, which writes
    the bytes tvu.save_image(clamp((x + 1) / 2, 0, 1)) would put in the PNG.  With an Inception model (fid.InceptionV3) the FID moments
    of those bytes accumulate on the device, batch by batch, as fid.calculate_activation_statistics would add the saved files batched
    by batch_size; with out_dir the files `{class_label}_{img_id}.png` are written on the host (img_id counts over the whole run).
    Returns (mu, sigma, n_files): mu / sigma None without an Inception model, n_files 0 without out_dir.

    With torch.distributed initialised over W > 1 ranks (and shard=True), batch k of the single-process order goes to rank k mod W, on
    the x_T (and step noise) rank 0 draws for it; each rank writes its own batches' files under their single-process names (out_dir must
    be one directory all ranks see).  The moments' shift is rank 0's first batch, as in one process; the moments are all-reduced once at
    the end, and every rank returns the same (mu, sigma, n_files), n_files counting the files of all ranks."""
    if inception is None and out_dir is None:
        raise ValueError("sample_for_fid needs an Inception model, an output directory, or both")
    if not hasattr(model, "first_stage_model"):
        raise RuntimeError("sample_for_fid decodes its samples: build the LatentDiffusion with first_stage_config")
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
    dev = model.device
    lib = L.load()
    fs = model.first_stage_model
    cfg = model.model.diffusion_model.config
    shape = [cfg.in_channels, cfg.image_size, cfg.image_size]
    inv = float(torch.tensor(1. / model.scale_factor, dtype=torch.float32))
    key = model.cond_stage_key
    sampler = DDIMSampler(model)
    mom = block = None
    if inception is not None:
        from . import fid
        block = fid._block_of(inception, fid_dims)
        mom = fid.Moments(fid_dims)
    world, rank = _world_rank(shard)
    batches = [class_label for _ in range(ipc // batch_size) for class_label in classes]
    gdev = generator.device if generator is not None else dev
    lat = (batch_size, *shape)
    spec = {"x_T": (lat, torch.float32)}
    if eta > 0:
        spec["step_noise"] = ((ddim_steps,) + lat, torch.float32)

    def draw():      # DDIMSampler.sample's draws: x_T, then one per step when eta > 0
        d = {"x_T": torch.randn(lat, generator=generator, device=gdev, dtype=torch.float32)}
        if eta > 0:
            d["step_noise"] = torch.stack([torch.randn(lat, generator=generator, device=gdev, dtype=torch.float32) for _ in range(ddim_steps)])
        return d
    u8 = None
    n_files = 0
    saved_batch = fs.decode_batch
    fs.decode_batch = decode_batch
    try:
        with model.ema_scope():
            uc = model.get_learned_conditioning({key: torch.tensor(batch_size * [1000]).to(dev)})
            for r0 in range(0, len(batches), world):
                d = _round_inputs(draw, spec, min(world, len(batches) - r0), world, rank, dev)
                feat = None
                if d is not None:
                    k = r0 + rank
                    class_label = batches[k]
                    c = model.get_learned_conditioning({key: torch.tensor(batch_size * [class_label]).to(dev)})
                    samples, _ = sampler.sample(S=ddim_steps, conditioning=c, batch_size=batch_size, shape=shape, verbose=False,
                                                unconditional_guidance_scale=scale, unconditional_conditioning=uc, eta=eta,
                                                x_T=d["x_T"], step_noise=d.get("step_noise"))
                    for s in range(0, batch_size, decode_batch):
                        y = fs.decode_chunk(samples[s:s + decode_batch], inv_scale=inv).plan.y_out
                        if u8 is None:
                            u8 = torch.empty((batch_size, y.H, y.W, y.C), dtype=torch.uint8, device=dev)
                        n = min(decode_batch, batch_size - s)
                        L.check(lib.dp_decode_images(y.ptr, y.ld, n, y.C, y.H, y.W, u8[s:s + n].data_ptr(), None, _stream()),
                                "decode_images")
                    if mom is not None:
                        plan = inception.plan(batch_size, "u8", u8.shape[1:3])
                        plan.load(u8)
                        plan.run()
                        feat = plan.feat[block]
                    if out_dir is not None:
                        from PIL import Image
                        for i, img in enumerate(u8.cpu().numpy()):
                            Image.fromarray(img).save(os.path.join(out_dir, f"{class_label}_{k * batch_size + i}.png"))
                            n_files += 1
                if mom is not None and world > 1 and r0 == 0:
                    if rank == 0:
                        mom.add(feat)          # batch 0 sets the shift, as in one process
                    mom.share_shift(0)
                    if rank > 0 and feat is not None:
                        mom.add(feat)
                elif feat is not None:
                    mom.add(feat)
    finally:
        fs.decode_batch = saved_batch
    if world > 1:
        if mom is not None:
            mom.all_reduce()
        nf = torch.tensor([n_files], dtype=torch.int64, device=dev)
        dist.all_reduce(nf, op=dist.ReduceOp.SUM)
        n_files = int(nf.item())
    mu, sigma = mom.finalize() if mom is not None else (None, None)
    return mu, sigma, n_files
