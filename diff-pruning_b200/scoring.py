"""The two hot loops of the reference as fused, CUDA-graph-replayed device programs.

TaylorScorer   — ddpm_prune.py:94-106: for each timestep  add_noise -> UNet fwd -> mse -> bwd, gradients
                 accumulating into Parameter.grad (no zero_grad between steps).  One graph replay per step.
FinetuneStepper— ddpm_train.py:437-469: add_noise -> fwd -> loss -> bwd -> clip_grad_norm_(1.0) -> Adam -> EMA
                 over flat parameter / gradient / moment / EMA arenas.
taylor_layer_scores / TaylorImportance — torch_pruning TaylorImportance.__call__
                 (ddpm_exp/torch_pruning/importance.py:375-434) on the device via dp_taylor_reduce.

Multi-GPU (SURVEY.md §8(e)): timesteps are sharded t = rank, rank+W, ... with ONE all-reduce(SUM) of the flat
gradient arena at the end of scoring; finetune shards the minibatch and all-reduces the gradient arena each
step (mean), both over NCCL.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from .engine import Plan, _dropout_seed, _stream, arena_offsets, capture_graphs, get_plan, invalidate_packs
from .models import UNet2DModel, ddpm_alphas_cumprod


def _dist_ready():
    import torch.distributed as dist
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class TaylorScorer:
    """Accumulates sum_t dL_t/dW into Parameter.grad for fixed (clean_images, noise) — ddpm_prune.py:90-102."""

    def __init__(self, model: UNet2DModel, clean_images: torch.Tensor, noise: torch.Tensor,
                 num_train_timesteps: int = 1000, alphas_cumprod: Optional[torch.Tensor] = None, use_graph: bool = True,
                 fused_scores: bool = False, context: Optional[torch.Tensor] = None):
        assert clean_images.is_cuda and clean_images.shape == noise.shape and clean_images.dtype == torch.float32
        self.lib = L.load()
        self.model = model
        self.dev = clean_images.device
        B, C_, H, W = clean_images.shape
        self.B, self.C, self.H, self.W = B, C_, H, W
        self.clean = clean_images.contiguous().clone()
        self.noise = noise.contiguous().clone()
        self.acp = (alphas_cumprod if alphas_cumprod is not None else ddpm_alphas_cumprod(num_train_timesteps)).to(self.dev).contiguous()
        was_training = model.training
        model.eval()  # ddpm_prune.py:91
        # fused_scores: the split-K wgrad reduce also accumulates sum_t sum_k W*dW_t per out/in channel of every conv/linear
        # (plan.score_arena, ~78 k floats for C1): the `multivariable=True` importance is |that| — no extra pass over dW,
        # and the multi-GPU exchange can be this small vector instead of the 143 MB gradient arena (SURVEY.md §8e).
        self.plan: Plan = get_plan(model, B, H, W, self.dev, need_grad=True, fused_scores=fused_scores)
        if was_training:
            model.train()
        if hasattr(self.plan, "ctx_in"):      # latent-diffusion UNetModel: cross-attention conditioning.  prune_ldm.py:105-131 draws new
            # classes, hence a new context (and new latents), every iteration: ldm_sampling.LDMPruneScorer reloads it with plan.load_context
            if context is None:
                raise ValueError("the LDM UNetModel needs context=(B, 1, context_dim)")
            self.plan.load_context(context)
        ldo = self.plan.y_out.ld                      # y_out is a C-channel view of a zero-padded ld-channel buffer
        self.noise_nhwc = torch.zeros((B, H, W, ldo), device=self.dev, dtype=torch.float32)
        n = B * C_ * H * W
        self.n = B * H * W * ldo                      # flat extent handed to the loss kernel (pads contribute 0)
        self.partial = torch.empty(max(1, self.lib.dp_mse_partials(self.n)), device=self.dev, dtype=torch.float32)
        self.loss = torch.zeros(1, device=self.dev, dtype=torch.float32)
        self.use_graph = use_graph
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.loss_scale, self.grad_scale = 1.0 / n, 2.0 / n   # F.mse_loss mean reduction, ddpm_prune.py:101
        self._refresh_noise()
        self.plan.attach_grads()
        self.plan.ensure_packed()

    def _refresh_noise(self):
        L.check(self.lib.dp_nchw_to_nhwc(self.noise.data_ptr(), self.noise_nhwc.data_ptr(), self.noise_nhwc.shape[-1], self.B, self.C,
                                         self.H, self.W, _stream()), "noise nchw->nhwc")

    def _forward_loss(self):
        """add_noise -> forward -> loss and its gradient d loss / d y_out: everything of a pass up to the backward."""
        lib, p, s = self.lib, self.plan, _stream()
        L.check(lib.dp_add_noise(self.clean.data_ptr(), self.noise.data_ptr(), p.t_dev.data_ptr(), self.acp.data_ptr(),
                                 p.x_in.ptr, self.B, self.C, self.H, self.W, 1, p.x_in.ld, s), "add_noise")
        p.run_forward(s)
        gy = p.gradof(p.y_out)
        L.check(lib.dp_mse_loss_grad(p.y_out.ptr, self.noise_nhwc.data_ptr(), gy.ptr, self.n, self.loss_scale, self.grad_scale,
                                     self.partial.data_ptr(), self.loss.data_ptr(), s), "mse")

    def _body(self):
        self._forward_loss()
        self.plan.run_backward(_stream())

    def signed_scores(self) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
        """{weight name: (out-channel, in-channel) sum_t sum_k W*dW_t} accumulated by the fused reduce (fused_scores=True)."""
        names = {id(p): n for n, p in self.model.named_parameters()}
        return {names[k]: v for k, v in self.plan.scores.items()}

    def step(self, t) -> torch.Tensor:
        """One pass at timestep(s) t (int, or a (B,) tensor).  Returns the device loss scalar (no sync)."""
        p = self.plan
        p.check_current()
        p.attach_grads()
        p.ensure_packed()
        if torch.is_tensor(t):
            p.t_dev.copy_(t.to(device=self.dev, dtype=torch.int64), non_blocking=True)
        else:
            p.t_dev.fill_(int(t))
        if self.use_graph:
            if self.graph is None:
                self.graph, = capture_graphs(self.dev, self._body,
                                             restore=(p.grad_arena, p.score_arena if p.fused_scores else None, p.t_dev))
            self.graph.replay()
        else:
            self._body()
        return self.loss

    def step_from_host(self, clean_pinned: torch.Tensor, noise_pinned: torch.Tensor, t: int) -> float:
        """End-to-end step through host buffers: H2D of the batch, one pass, D2H of the loss."""
        self.clean.copy_(clean_pinned, non_blocking=True)
        self.noise.copy_(noise_pinned, non_blocking=True)
        self._refresh_noise()
        return float(self.step(t).item())

    def run(self, timesteps: Iterable[int], shard: bool = True, thr: Optional[float] = None) -> torch.Tensor:
        """The whole loop of ddpm_prune.py:97-106; with torch.distributed initialised, timesteps are sharded
        (t_k for k = rank mod world) and the gradient arena is all-reduced (SUM) once at the end.

        `thr` is the `--pruner diff-pruning` rule of ddpm_prune.py:104-106: track the running maximum loss and stop after the
        first timestep whose loss falls below `thr * loss_max` (that timestep's gradient is still accumulated — its backward ran
        before the check).  Returns the losses of the timesteps that were used."""
        ts = list(timesteps)
        world, rank = 1, 0
        if shard and _dist_ready():
            import torch.distributed as dist
            world, rank = dist.get_world_size(), dist.get_rank()
        if thr is not None:
            losses = self._run_thresholded(ts, float(thr), world, rank)
        else:
            losses = torch.zeros(len(ts), device=self.dev, dtype=torch.float32)
            for k, t in enumerate(ts):
                if k % world != rank:
                    continue
                losses[k:k + 1].copy_(self.step(t))
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(self.plan.grad_arena, op=dist.ReduceOp.SUM)
            if thr is None:
                dist.all_reduce(losses, op=dist.ReduceOp.SUM)
            if self.plan.fused_scores:
                dist.all_reduce(self.plan.score_arena, op=dist.ReduceOp.SUM)
        return losses

    def _run_thresholded(self, ts, thr: float, world: int, rank: int) -> torch.Tensor:
        """Rounds of `world` consecutive timesteps (rank r takes the r-th of each round).  The stop rule is sequential, so after
        every round the ranks exchange their losses (one tiny all-reduce; the reference syncs on the loss every step as well) and
        replay the reference's scalar logic; a rank whose timestep lies beyond the stopping one restores the gradient arena from
        the snapshot taken before its speculative pass, so the accumulated gradient is exactly that of the sequential loop."""
        used = []
        loss_max = np.float32(0.0)
        thr32 = np.float32(thr)
        snap = snap_scores = None
        for r0 in range(0, len(ts), world):
            k = r0 + rank
            mine = k < len(ts)
            if world > 1 and mine and rank > 0:      # rank 0's timestep is the first of the round: never undone
                snap = self.plan.grad_arena.clone() if snap is None else snap.copy_(self.plan.grad_arena)
                if self.plan.fused_scores:
                    snap_scores = self.plan.score_arena.clone() if snap_scores is None else snap_scores.copy_(self.plan.score_arena)
            rl = torch.zeros(world, device=self.dev, dtype=torch.float32)
            if mine:
                rl[rank:rank + 1].copy_(self.step(ts[k]))
            if world > 1:
                import torch.distributed as dist
                dist.all_reduce(rl, op=dist.ReduceOp.SUM)
            stop_at = None
            for j, l in enumerate(rl.tolist()[:min(world, len(ts) - r0)]):
                l = np.float32(l)
                if l > loss_max:
                    loss_max = l
                used.append(float(l))
                if l < loss_max * thr32:             # fp32 product, as `loss < loss_max * args.thr` on 0-dim fp32 tensors
                    stop_at = j
                    break
            if stop_at is not None:
                if mine and rank > stop_at:
                    self.plan.grad_arena.copy_(snap)
                    if self.plan.fused_scores:
                        self.plan.score_arena.copy_(snap_scores)
                break
        return torch.tensor(used, device=self.dev, dtype=torch.float32)


def threshold_stop(losses, thr: float) -> int:
    """Number of timesteps the `diff-pruning` loop of ddpm_prune.py:97-106 consumes for a given loss sequence (host helper,
    same fp32 comparisons as TaylorScorer.run(thr=...))."""
    loss_max, thr32 = np.float32(0.0), np.float32(thr)
    for n, l in enumerate(losses, 1):
        l = np.float32(l)
        if l > loss_max:
            loss_max = l
        if l < loss_max * thr32:
            return n
    return len(losses)


# --------------------------------------------------------------------------------------------------------
# Taylor importance on device
# --------------------------------------------------------------------------------------------------------
def taylor_layer_scores(weight: torch.Tensor, grad: torch.Tensor) -> Dict[str, torch.Tensor]:
    """All six per-channel reductions of w*dw for one layer (out/in x signed/abs/sq) via dp_taylor_reduce.
    weight: (O, I, R, S) conv, (O, I) linear, or (C,) GroupNorm gamma."""
    lib = L.load()
    assert weight.is_cuda and grad.is_cuda and weight.shape == grad.shape
    w, g = weight.detach().contiguous().float(), grad.detach().contiguous().float()
    a = L.TaylorArgs()
    if w.dim() == 1:
        O, I, RS = w.numel(), 1, 1
    else:
        O, I = w.shape[0], w.shape[1]
        RS = w.numel() // (O * I)
    a.O, a.I, a.RS = O, I, RS
    a.w, a.dw = w.data_ptr(), g.data_ptr()
    out = torch.empty((3, O), device=w.device, dtype=torch.float32)
    a.out_signed, a.out_abs, a.out_sq = out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr()
    res = {"out_signed": out[0], "out_abs": out[1], "out_sq": out[2]}
    if w.dim() > 1:
        inn = torch.empty((3, I), device=w.device, dtype=torch.float32)
        a.in_signed, a.in_abs, a.in_sq = inn[0].data_ptr(), inn[1].data_ptr(), inn[2].data_ptr()
        res.update({"in_signed": inn[0], "in_abs": inn[1], "in_sq": inn[2]})
    L.check(lib.dp_taylor_reduce(a, _stream()), "taylor_reduce")
    return res


_VARIANT_KEY = {"vendored": "sq", "taylor": "signed", "diff": "abs", "abs": "abs"}
EXP_VARIANTS = ("full1", "full2", "abs", "fisher")   # ddpm_exp/torch_pruning/importance.py:438-781


def group_importance(items: Sequence[Tuple[str, str, Sequence[int]]], named_weights: Dict[str, torch.Tensor],
                     named_grads: Dict[str, torch.Tensor], variant: str = "taylor",
                     cache: Optional[dict] = None) -> Optional[torch.Tensor]:
    """importance.py:375-434 for one group given as (layer_name, kind in {out,in,gn}, idxs) items.
    variant: 'taylor' = |sum_k w dw| (multivariable=True, ddpm_prune.py:60), 'diff' = sum_k |w dw|
    (multivariable=False, :66), 'vendored' = sum_k (w dw)^2 (vendored importance.py:393).  GroupNorm: |w dw| (:416).
    The ddpm_exp criteria go through the same device reductions: 'full1' / 'full2' = FullTaylorImportance(order) (:438-548: signed
    sum_k w dw, + sum_k (w dw)^2 for order 2, abs AFTER the group sum), 'abs' = AbsTaylorImportance (:553-670, = 'diff' per item),
    'fisher' = FisherImportance (:672-781: sum_k dw^2 — dp_taylor_reduce with w := dw — and (w dw)^2 for GroupNorm)."""
    cache = {} if cache is None else cache
    imps = []
    for name, kind, idxs in items:
        w, g = named_weights[name + ".weight"], named_grads[name + ".weight"]
        ck = (name, "fisher") if (variant == "fisher" and kind != "gn") else name
        sc = cache.get(ck)
        if sc is None:
            sc = taylor_layer_scores(g, g) if ck != name else taylor_layer_scores(w, g)
            cache[ck] = sc
        idx = torch.as_tensor(sorted(idxs), device=sc["out_abs"].device, dtype=torch.long)
        if kind == "gn":
            v = {"full1": sc["out_signed"], "full2": sc["out_signed"] + sc["out_sq"], "fisher": sc["out_sq"]}.get(variant, sc["out_abs"])[idx]
        elif variant == "full1":
            v = sc[f"{kind}_signed"][idx]
        elif variant == "full2":
            v = sc[f"{kind}_signed"][idx] + sc[f"{kind}_sq"][idx]
        elif variant == "fisher":
            v = sc[f"{kind}_signed"][idx]            # sum_k dw*dw
        else:
            v = sc[f"{kind}_{_VARIANT_KEY[variant]}"][idx]
            if variant == "taylor":
                v = v.abs()
        imps.append(v)
    if not imps:
        return None
    size = len(imps[0])
    total = torch.stack([i for i in imps if len(i) == size], dim=0).sum(0)
    return total.abs() if variant in ("full1", "full2") else total


def select_pruning_idxs(imp: torch.Tensor, ch_groups: int, n_pruned: int) -> List[int]:
    """metapruner.py:231-249 — host-side integer selection (argsort on CPU like the reference's CPU run)."""
    imp = imp.detach().float().cpu()
    if n_pruned <= 0:
        return []
    if ch_groups > 1:
        size, per, out = len(imp) // ch_groups, n_pruned // ch_groups, []
        for g in range(ch_groups):
            out.append(torch.argsort(imp[g * size:(g + 1) * size])[:per] + g * size)
        return torch.cat(out, 0).tolist()
    return torch.argsort(imp)[: n_pruned // ch_groups].tolist()


# --------------------------------------------------------------------------------------------------------
# Finetune step
# --------------------------------------------------------------------------------------------------------
class FinetuneStepper:
    """ddpm_train.py:437-469 on device.  Parameters are re-pointed into one flat arena (values preserved) so the
    clip + Adam + EMA tail is a single pass over contiguous memory and DDP needs one all-reduce."""

    def __init__(self, model: UNet2DModel, lr: float = 2e-4, betas=(0.9, 0.999), eps: float = 1e-8,
                 ema_decay: float = 0.9999, max_grad_norm: float = 1.0, use_ema: bool = True,
                 num_train_timesteps: int = 1000, use_graph: bool = True, compute: str = "fp32"):
        self.lib = L.load()
        self.model = model
        self.compute = compute      # "fp32": fp32-grade 3 x fp16 split tier | "bf16": single-pass tensor tier (ddpm_train.py --mixed_precision bf16)
        self.dev = next(model.parameters()).device
        assert self.dev.type == "cuda"
        self.lr, self.betas, self.eps = lr, betas, eps
        self.ema_decay, self.max_grad_norm = ema_decay, max_grad_norm
        self.params = list(model.parameters())
        self._offs, total = arena_offsets(self.params)     # the same 256-byte-aligned layout as the plan's gradient arena
        self.n = total
        self.param_arena = torch.zeros(total, device=self.dev, dtype=torch.float32)
        with torch.no_grad():
            for p, o in zip(self.params, self._offs):
                v = self.param_arena[o:o + p.numel()].view_as(p)
                v.copy_(p.data)
                p.data = v
        self.m = torch.zeros(total, device=self.dev, dtype=torch.float32)
        self.v = torch.zeros(total, device=self.dev, dtype=torch.float32)
        self.ema = self.param_arena.clone() if use_ema else None
        self.acp = ddpm_alphas_cumprod(num_train_timesteps).to(self.dev).contiguous()
        self.step_scalars = torch.zeros(2, device=self.dev, dtype=torch.float32)
        self.sumsq = torch.zeros(1, device=self.dev, dtype=torch.float32)
        self.ss_partial = torch.empty(max(1, self.lib.dp_sumsq_partials(total)), device=self.dev, dtype=torch.float32)
        self.loss = torch.zeros(1, device=self.dev, dtype=torch.float32)
        self.steps_done = 0
        self.use_graph = use_graph
        self.plan: Optional[Plan] = None
        self.g_main = self.g_tail = None
        self.world = 1
        if _dist_ready():
            import torch.distributed as dist
            self.world = dist.get_world_size()

    def ema_state(self) -> Dict[str, torch.Tensor]:
        out = {}
        for (name, p), o in zip(self.model.named_parameters(), self._offs):
            out[name] = self.ema[o:o + p.numel()].view_as(p)
        return out

    def _setup(self, B, C_, H, W):
        self.model.train()
        self.plan = get_plan(self.model, B, H, W, self.dev, need_grad=True, compute=self.compute)
        self.B, self.C, self.H, self.W = B, C_, H, W
        self.clean = torch.empty((B, C_, H, W), device=self.dev, dtype=torch.float32)
        self.noise = torch.empty_like(self.clean)
        self.noise_nhwc = torch.zeros((B, H, W, self.plan.y_out.ld), device=self.dev, dtype=torch.float32)
        self.nelem = B * H * W * self.plan.y_out.ld   # flat extent incl. zero pads (contribute 0 to the loss)
        self.partial = torch.empty(max(1, self.lib.dp_mse_partials(self.nelem)), device=self.dev, dtype=torch.float32)
        self.plan.attach_grads()

    def _main(self):
        lib, p, s = self.lib, self.plan, _stream()
        p.run_pack(s)
        L.check(lib.dp_nchw_to_nhwc(self.noise.data_ptr(), self.noise_nhwc.data_ptr(), self.noise_nhwc.shape[-1], self.B, self.C, self.H,
                                    self.W, s), "noise")
        L.check(lib.dp_add_noise(self.clean.data_ptr(), self.noise.data_ptr(), p.t_dev.data_ptr(), self.acp.data_ptr(),
                                 p.x_in.ptr, self.B, self.C, self.H, self.W, 1, p.x_in.ld, s), "add_noise")
        p.run_forward(s)
        gy = p.gradof(p.y_out)
        # loss = (noise - out)^2 .sum(1,2,3).mean(0)  (ddpm_train.py:459)
        L.check(lib.dp_mse_loss_grad(p.y_out.ptr, self.noise_nhwc.data_ptr(), gy.ptr, self.nelem, 1.0 / self.B, 2.0 / self.B,
                                     self.partial.data_ptr(), self.loss.data_ptr(), s), "loss")
        p.grad_arena.zero_()          # optimizer.zero_grad() (:456)
        p.run_backward(s)

    def _tail(self):
        lib, p, s = self.lib, self.plan, _stream()
        L.check(lib.dp_sumsq(p.grad_arena.data_ptr(), self.n, self.ss_partial.data_ptr(), self.sumsq.data_ptr(), s), "sumsq")
        a = L.AdamArgs()
        a.n = self.n
        a.p, a.g, a.m, a.v = self.param_arena.data_ptr(), p.grad_arena.data_ptr(), self.m.data_ptr(), self.v.data_ptr()
        a.ema = self.ema.data_ptr() if self.ema is not None else None
        a.sumsq = self.sumsq.data_ptr() if self.max_grad_norm is not None else None
        a.max_norm = float(self.max_grad_norm or 0.0)
        a.lr, a.beta1, a.beta2, a.eps, a.ema_decay = self.lr, self.betas[0], self.betas[1], self.eps, self.ema_decay
        a.step, a.grad_scale = 1, 1.0 / self.world
        a.step_scalars = self.step_scalars.data_ptr()
        self._adam_args = a
        L.check(lib.dp_adam_clip_ema(a, s), "adam")

    def step(self, clean: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        """One optimisation step; returns the device loss scalar (this rank's minibatch)."""
        B, C_, H, W = clean.shape
        if self.plan is None:
            self._setup(B, C_, H, W)
        p = self.plan
        p.check_current()
        self.clean.copy_(clean, non_blocking=True)
        self.noise.copy_(noise, non_blocking=True)
        p.t_dev.copy_(timesteps.to(device=self.dev, dtype=torch.int64), non_blocking=True)
        self.steps_done += 1
        t = self.steps_done
        bc = torch.tensor([self.lr / (1.0 - self.betas[0] ** t), math.sqrt(1.0 - self.betas[1] ** t)], dtype=torch.float32)
        self.step_scalars.copy_(bc, non_blocking=True)
        p.dropout_seed_dev.fill_(_dropout_seed(t))   # per step AND per rank: data-parallel ranks draw different masks
        if self.use_graph and self.g_main is None:
            self.g_main, self.g_tail = capture_graphs(self.dev, self._main, self._tail,
                                                      restore=(self.param_arena, self.m, self.v, self.ema))
        if self.use_graph:
            self.g_main.replay()
        else:
            self._main()
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(p.grad_arena, op=dist.ReduceOp.SUM)   # mean applied through grad_scale = 1/world
        if self.use_graph:
            self.g_tail.replay()
        else:
            self._tail()
        invalidate_packs(self.model)   # the Adam kernel wrote the parameter arena through raw pointers: other cached plans are stale
        return self.loss
