"""DDIM sampling on the device — SURVEY.md §8(f) item 1: the step right after finetune in BASELINE config 2 and the tail of
ddpm_prune.py:138-147 / ddpm_sample.py.

DDIMScheduler  — diffusers/schedulers/scheduling_ddim.py as MODIFIED by the reference: `skip_type` uniform|quad timestep
                 spacing (:257-266) and `prev_timestep = t - T // S` (:324, kept although it is inconsistent with that spacing).
DDIMPipeline   — diffusers/pipelines/ddim/pipeline_ddim.py:45-122: randn image -> S x [UNet forward, scheduler.step] ->
                 (x/2+0.5).clamp(0,1) -> NHWC numpy.  The UNet forward is the planned engine (no-grad plan), the update is one
                 fused kernel (dp_ddim_step); per-step coefficients are formed in fp32 torch scalars like the reference.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch

from . import _lib as L
from .engine import _stream
from .models import DDPMScheduler, UNet2DModel


class DDIMScheduler:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, beta_schedule="linear", skip_type="uniform",
                 clip_sample=True, set_alpha_to_one=True, steps_offset=0, prediction_type="epsilon", clip_sample_range=1.0,
                 **unused):
        if beta_schedule != "linear" or prediction_type != "epsilon":
            raise NotImplementedError("only the linear-beta epsilon-prediction DDPM family is on the hot path")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, clip_sample=clip_sample, set_alpha_to_one=set_alpha_to_one,
                                      steps_offset=steps_offset, prediction_type=prediction_type,
                                      clip_sample_range=clip_sample_range)
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.skip_type = skip_type
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    @classmethod
    def from_config(cls, config, **kw):
        from . import checkpoint
        d = dict(vars(config)) if not isinstance(config, dict) else dict(config)
        return checkpoint.build_from_config(cls, d, **kw)

    # ---- scheduler_config.json I/O (checkpoint.py); `DDIMScheduler.from_pretrained(save_path, subfolder="scheduler")` re-reads
    # a DDPM scheduler's config, as ddpm_prune.py:140 and ddpm_sample.py:34 do
    def save_pretrained(self, save_directory, **unused):
        from . import checkpoint
        checkpoint.save_config(self, save_directory, checkpoint.SCHEDULER_CONFIG_NAME)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kw):
        from . import checkpoint
        cfg = checkpoint.load_config(pretrained_model_name_or_path, checkpoint.SCHEDULER_CONFIG_NAME, subfolder)
        return checkpoint.build_from_config(cls, cfg, **kw)

    def set_timesteps(self, num_inference_steps: int, device=None):
        T = self.config.num_train_timesteps
        if num_inference_steps > T:
            raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than `self.config.train_timesteps`: {T}")
        self.num_inference_steps = num_inference_steps
        if self.skip_type == "uniform":
            ratio = (T - 1) / (num_inference_steps - 1)
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        elif self.skip_type == "quad":
            ratio = (T - 1) / (num_inference_steps - 1) ** 2
            ts = (np.arange(0, num_inference_steps) ** 2 * ratio).round()[::-1].copy().astype(np.int64)
        else:
            raise NotImplementedError(f"skip_type {self.skip_type} is not implemented")
        self.timesteps = torch.from_numpy(ts) + self.config.steps_offset

    def _coefficients(self, timestep: int, eta: float):
        prev = timestep - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[timestep]
        a_prev = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        variance = ((1 - a_prev) / b_t) * (1 - a_t / a_prev)          # scheduling_ddim.py:194-202
        std = eta * variance ** 0.5
        return (float(b_t ** 0.5), float(a_t ** 0.5), float(a_prev ** 0.5), float((1 - a_prev - std ** 2) ** 0.5), float(std))

    def step(self, model_output, timestep, sample, eta: float = 0.0, use_clipped_model_output=False, generator=None,
             variance_noise=None, return_dict=True):
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if use_clipped_model_output:
            raise NotImplementedError("use_clipped_model_output")
        if not sample.is_cuda:
            raise RuntimeError("diff_pruning_b200: DDIMScheduler.step is a CUDA op (no CPU fallback)")
        sb, sa, sap, dirc, sigma = self._coefficients(int(timestep), eta)
        x, e = sample.contiguous(), model_output.contiguous()
        noise = None
        if eta > 0:
            noise = variance_noise if variance_noise is not None else \
                torch.randn(e.shape, generator=generator, device=generator.device if generator is not None else e.device,
                            dtype=e.dtype)
            noise = noise.to(e.device).contiguous()
        out = torch.empty_like(x)
        clip = float(self.config.clip_sample_range) if self.config.clip_sample else 0.0
        L.check(L.load().dp_ddim_step(x.data_ptr(), e.data_ptr(), noise.data_ptr() if noise is not None else None, out.data_ptr(),
                                      x.numel(), sb, sa, clip, sap, dirc, sigma, _stream()), "ddim_step")
        return SimpleNamespace(prev_sample=out) if return_dict else (out,)


class DDIMPipeline:
    def __init__(self, unet: UNet2DModel, scheduler):
        self.unet = unet
        self.scheduler = DDIMScheduler.from_config(scheduler.config) if not isinstance(scheduler, DDIMScheduler) else scheduler
        self._pbar = {}
        self.use_graph = True        # replay the UNet forward as one CUDA graph per sampling step

    @property
    def device(self):
        return next(self.unet.parameters()).device

    def to(self, device):
        self.unet.to(device)
        return self

    def set_progress_bar_config(self, **kw):
        self._pbar = kw

    # ---- model_index.json + unet/ + scheduler/ (checkpoint.py; pipeline_utils.py:485-560, 563-1000)
    def save_pretrained(self, save_directory, safe_serialization=False, **unused):
        from . import checkpoint
        checkpoint.save_pipeline(self, save_directory, safe_serialization=safe_serialization)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, **kw):
        from . import checkpoint
        return checkpoint.load_pipeline(cls, pretrained_model_name_or_path, **kw)

    @torch.no_grad()
    def __call__(self, batch_size=1, generator=None, eta=0.0, num_inference_steps=50, use_clipped_model_output=None,
                 output_type="pil", return_dict=True):
        """pipeline_ddim.py:45-122.  The UNet forward of the whole loop is ONE captured CUDA graph (static launch plan, the timestep
        lives in device memory) replayed per step, followed by the fused scheduler update (dp_ddim_step): no per-step Python walk over
        the ~400 launches of a forward and no host synchronisation inside the loop."""
        cfg = self.unet.config
        size = cfg.sample_size if isinstance(cfg.sample_size, int) else None
        shape = (batch_size, cfg.in_channels, size, size) if size is not None else (batch_size, cfg.in_channels, *cfg.sample_size)
        gdev = generator.device if generator is not None else self.device
        image = torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32).to(self.device)
        self.scheduler.set_timesteps(num_inference_steps)
        timesteps = self.scheduler.timesteps.tolist()
        if not image.is_cuda:
            raise RuntimeError("diff_pruning_b200: DDIMPipeline samples on a CUDA device (no CPU fallback); call pipeline.to('cuda')")
        from .engine import frozen_weights, get_plan
        was_training = self.unet.training
        self.unet.eval()
        try:
            with frozen_weights(self.unet):       # weights are packed once for the loop (whatever they are NOW: EMA copy_to etc.)
                if self.use_graph:
                    plan = get_plan(self.unet, shape[0], shape[2], shape[3], image.device, need_grad=False)
                    plan.ensure_packed(force=True)
                    x_static, eps = image.clone(), torch.empty_like(image)

                    def body():
                        L.check(L.load().dp_nchw_to_nhwc(x_static.data_ptr(), plan.x_in.ptr, plan.x_in.ld, plan.B, plan.x_in.C, plan.H, plan.W,
                                                         _stream()), "nchw->nhwc")
                        plan.run_forward()
                        L.check(L.load().dp_nhwc_to_nchw(plan.y_out.ptr, plan.y_out.ld, eps.data_ptr(), plan.B, plan.y_out.C, plan.H, plan.W, 0,
                                                         _stream()), "nhwc->nchw")
                    torch.cuda.synchronize(image.device)
                    side = torch.cuda.Stream(device=image.device)
                    side.wait_stream(torch.cuda.current_stream(image.device))
                    with torch.cuda.stream(side):     # warm-up outside capture (lazy module loading)
                        body()
                    torch.cuda.current_stream(image.device).wait_stream(side)
                    torch.cuda.synchronize(image.device)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        body()
                    for t in timesteps:
                        plan.t_dev.fill_(t)
                        graph.replay()
                        x_static.copy_(self.scheduler.step(eps, t, x_static, eta=eta, generator=generator).prev_sample)
                    image = x_static
                else:
                    for t in timesteps:
                        eps = self.unet(image, t).sample
                        image = self.scheduler.step(eps, t, image, eta=eta, generator=generator).prev_sample
        finally:
            self.unet.train(was_training)
        if output_type == "device":   # the raw final sample, NCHW on the device (FID statistics quantise it there, fid.py)
            return SimpleNamespace(images=image) if return_dict else (image,)
        image = (image / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).numpy()
        if output_type == "pil":
            from PIL import Image  # optional dependency, like the reference
            image = [Image.fromarray((im * 255).round().astype("uint8")) for im in image]
        return SimpleNamespace(images=image) if return_dict else (image,)


class DDPMPipeline:
    """Container the reference scripts use to carry (unet, scheduler) to and from disk (`DDPMPipeline.from_pretrained(model_path)`
    at ddpm_prune.py:50, `pipeline.save_pretrained(save_path)` at :132, ddpm_train.py:304-308,498).  Sampling on the hot path is
    DDIM (`DDIMPipeline`, which the scripts build from this pipeline's unet and the re-read scheduler config); the 1000-step
    ancestral sampler of pipeline_ddpm.py is not rebuilt."""

    def __init__(self, unet: UNet2DModel, scheduler):
        self.unet = unet
        self.scheduler = scheduler

    @property
    def device(self):
        return next(self.unet.parameters()).device

    def to(self, device):
        self.unet.to(device)
        return self

    def set_progress_bar_config(self, **kw):
        pass

    def save_pretrained(self, save_directory, safe_serialization=False, **unused):
        from . import checkpoint
        checkpoint.save_pipeline(self, save_directory, safe_serialization=safe_serialization)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, **kw):
        from . import checkpoint
        return checkpoint.load_pipeline(cls, pretrained_model_name_or_path, **kw)

    def __call__(self, *a, **kw):
        raise NotImplementedError("diff_pruning_b200: ancestral DDPM sampling is not on the hot path; build "
                                  "DDIMPipeline(unet=pipeline.unet, scheduler=DDIMScheduler.from_config(pipeline.scheduler.config))")


class DiffusionPipeline:
    """`DiffusionPipeline.from_pretrained(dir)` (pipeline_utils.py:563-1000; imported at ddpm_prune.py:1): reads model_index.json and
    builds the pipeline class it names (DDPMPipeline / DDIMPipeline — the two of this path)."""

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, **kw):
        import json
        import os
        from . import checkpoint
        fn = os.path.join(pretrained_model_name_or_path, checkpoint.MODEL_INDEX_NAME)
        name = json.load(open(fn, encoding="utf-8")).get("_class_name", "DDPMPipeline") if os.path.isfile(fn) else "DDPMPipeline"
        classes = {"DDPMPipeline": DDPMPipeline, "DDIMPipeline": DDIMPipeline}
        if name not in classes:
            raise NotImplementedError(f"diff_pruning_b200: pipeline class {name} is outside the DDPM path")
        return classes[name].from_pretrained(pretrained_model_name_or_path, **kw)
