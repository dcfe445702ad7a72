"""ORACLE of prune_ldm.py's sample-then-score loop — test infrastructure only (tests/ and scripts/time_ldm_prune_loop.py's eager bars).

A float64-capable torch restatement of the reference's DDIM schedule, guided DDIM step and get_loss_at_t, around the functional LDM UNet of
oracle/ldm_oracle.py.  Each function cites the reference lines it restates.  Pinned to the unmodified reference by
tests/golden/ldm_ddim_tiny.pt (tools/gen_golden.py ldm_ddim) in tests/test_ldm_sampling_host.py.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from oracle.ldm_oracle import unet_forward

Tensor = torch.Tensor


def make_schedule(alphas_cumprod: Tensor, S: int, eta: float) -> Tuple[np.ndarray, List[Tuple[float, float, float, float]]]:
    """ddim.py:24-53 with util.py make_ddim_timesteps ('uniform': range(0, T, T // S) + 1) and make_ddim_sampling_parameters (a_t, a_prev
    = alphacums[0] then the previous DDIM step's, sigma = eta sqrt((1 - a_prev) / (1 - a_t) (1 - a_t / a_prev))), in float64 from the
    float32 table.  Returns (timesteps, [(a_t, a_prev, sigma, sqrt(1 - a_t)) per index])."""
    ac = alphas_cumprod.detach().double().cpu()
    T = ac.shape[0]
    ts = np.asarray(list(range(0, T, T // S))) + 1
    a = ac[ts]
    ap = torch.cat([ac[:1], ac[ts[:-1]]])
    sig = eta * torch.sqrt((1 - ap) / (1 - a) * (1 - a / ap))
    return ts, [(float(a[i]), float(ap[i]), float(sig[i]), float(torch.sqrt(1 - a[i]))) for i in range(S)]


def p_sample_ddim(eps_fn: Callable[[Tensor, Tensor, Tensor], Tensor], x: Tensor, c: Tensor, uc: Optional[Tensor], t: int,
                  coef: Tuple[float, float, float, float], scale: float, noise: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
    """ddim.py:165-202 (temperature 1, no corrector / quantisation / noise dropout): one forward of cat([x, x]) with cat([uc, c]),
    e = e_u + s (e_c - e_u) (or one forward of x with c when s == 1 or uc is None); pred_x0 = (x - sqrt(1 - a_t) e) / sqrt(a_t);
    x_prev = sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma^2) e + sigma noise.  Returns (x_prev, pred_x0, e)."""
    b = x.shape[0]
    tt = torch.full((b,), t, dtype=torch.long, device=x.device)
    if uc is None or scale == 1.:
        e = eps_fn(x, tt, c)
    else:
        e_u, e_c = eps_fn(torch.cat([x, x]), torch.cat([tt, tt]), torch.cat([uc, c])).chunk(2)
        e = e_u + scale * (e_c - e_u)
    a_t, a_prev, sigma, sb = coef
    pred_x0 = (x - sb * e) / a_t ** 0.5
    x_prev = a_prev ** 0.5 * pred_x0 + (1. - a_prev - sigma ** 2) ** 0.5 * e
    if noise is not None and sigma != 0:
        x_prev = x_prev + sigma * noise
    return x_prev, pred_x0, e


def sample(eps_fn, alphas_cumprod: Tensor, S: int, x_T: Tensor, c: Tensor, uc: Optional[Tensor], scale: float, eta: float,
           noises: Optional[List[Tensor]] = None) -> Tuple[Tensor, List[Dict[str, Tensor]]]:
    """ddim.py:106-163: the S steps over the flipped DDIM timesteps, index = S - i - 1.  Returns (samples, per-step records)."""
    ts, coefs = make_schedule(alphas_cumprod, S, eta)
    x, steps = x_T, []
    for i, step in enumerate(np.flip(ts)):
        index = S - i - 1
        x, x0, e = p_sample_ddim(eps_fn, x, c, uc, int(step), coefs[index], scale, noises[i] if noises is not None else None)
        steps.append({"x_prev": x, "pred_x0": x0, "e": e})
    return x, steps


def unet_eps(sd: Dict[str, Tensor], cfg: dict):
    """eps_fn of the functional UNet (oracle/ldm_oracle.py) in the state dict's dtype."""
    dt = sd["time_embed.0.weight"].dtype
    return lambda x, t, ctx: unet_forward(sd, cfg, x.to(dt), t, ctx.to(dt))


def get_loss_at_t(sd: Dict[str, Tensor], cfg: dict, alphas_cumprod: Tensor, x0: Tensor, context: Tensor, t: Tensor, noise: Tensor) -> Tensor:
    """ddpm.py:881-889 -> p_losses (:1022-1056) at the cin256-v2 values (eps target, l2, logvar 0, original_elbo_weight 0): q_sample with
    the float32 table's square roots (as the engine forms them), the per-image mean over C, H, W, then the batch mean; backward into the
    state dict's leaves."""
    dt = sd["time_embed.0.weight"].dtype
    ac = alphas_cumprod.to(device=x0.device)
    a = (ac[t] ** 0.5).to(dt).reshape(-1, 1, 1, 1)
    s = ((1 - ac[t]) ** 0.5).to(dt).reshape(-1, 1, 1, 1)
    out = unet_forward(sd, cfg, a * x0.to(dt) + s * noise.to(dt), t, context.to(dt))
    loss = ((out - noise.to(dt)) ** 2).mean([1, 2, 3]).mean()
    loss.backward()
    return loss.detach()
