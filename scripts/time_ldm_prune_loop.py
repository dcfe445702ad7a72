#!/usr/bin/env python
"""Time prune_ldm.py's loop (ldm_exp/prune_ldm.py:105-131) on the engine: C5 cin256-v2 with seeded weights (the zero-initialised
convolutions re-drawn, as bench.py does), batch 6, DDIM-20 with guidance scale 3.

Reports, as one JSON line: ms per DDIM-20 guided sample (one graph replay), ms per Taylor pass (forward + loss graph and backward graph
replays), ms per full loop iteration (LDMPruneScorer.run, class draw and host loss read included), the same iteration run as torch eager
on this GPU with the float32 oracle (tests/ldm_sampling_oracle.py) with cuDNN TF32 allowed and with plain fp32, and the GPU's name, power
limit and SM clock read in the same call.  Writes nothing.

    python scripts/time_ldm_prune_loop.py [--iters 10] [--eager-iters 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402


def c5_latent_diffusion():
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    torch.manual_seed(0)
    ld = LatentDiffusion()              # the UNet is built first: the seed-0 weights of bench.py's C5
    unet = ld.model.diffusion_model
    g = torch.Generator().manual_seed(5)
    for p in unet.parameters():
        if p.dim() > 1 and float(p.detach().abs().sum()) == 0:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.02)
    return ld.cuda()


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def eager_iteration_ms(ld, B, iters, tf32):
    """One loop iteration as torch eager with the float32 oracle: 20 guided steps at batch 2B, then get_loss_at_t + backward at batch B."""
    import ldm_sampling_oracle as orc
    from diff_pruning_b200 import ldm
    cfg = ldm.CIN256_V2_CONFIG
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        sd = {k: v.detach().clone().requires_grad_(True) for k, v in ld.model.diffusion_model.state_dict().items()}
        g = torch.Generator(device="cuda").manual_seed(1)
        emb = ld.cond_stage_model

        def one(t):
            with torch.no_grad():
                c = emb({"class_label": torch.randint(0, 1000, (B,), device="cuda", generator=g)})
                uc = emb({"class_label": torch.full((B,), 1000, device="cuda")})
                x_T = torch.randn(B, 3, 64, 64, device="cuda", generator=g)
                x, _ = orc.sample(orc.unet_eps(sd, cfg), ld.alphas_cumprod, 20, x_T, c, uc, 3.0, 0.0)
            noise = torch.randn(x.shape, device="cuda", generator=g)
            orc.get_loss_at_t(sd, cfg, ld.alphas_cumprod, x, c, torch.full((B,), t, device="cuda", dtype=torch.long), noise)
        one(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(iters):
            one(t + 1)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / iters
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--eager-iters", type=int, default=2)
    ap.add_argument("--batch", type=int, default=6)
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    if not torch.cuda.is_available():
        raise SystemExit("time_ldm_prune_loop.py measures on a CUDA device; none found")
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    B = a.batch
    ld = c5_latent_diffusion()
    unet = ld.model.diffusion_model
    unet.zero_grad()
    sc = LDMPruneScorer(ld, n_samples_per_class=B, ddim_steps=20, scale=3.0, eta=0.0)
    g = torch.Generator(device="cuda").manual_seed(0)
    sc.run("taylor", iterations=2, generator=g)                 # builds both plans and all three graphs
    torch.cuda.synchronize()
    sample_ms = events_ms(sc.sampler.last_run.graph.replay, 5)

    def taylor():
        sc.g_fwd.replay()
        sc.g_bwd.replay()
    taylor_ms = events_ms(taylor, 5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sc.run("taylor", iterations=a.iters, generator=g)
    torch.cuda.synchronize()
    iter_ms = (time.perf_counter() - t0) * 1e3 / a.iters
    info = gpu_info()
    eager_tf32 = eager_iteration_ms(ld, B, a.eager_iters, True)
    eager_fp32 = eager_iteration_ms(ld, B, a.eager_iters, False)
    info_after = gpu_info()
    print(json.dumps({
        "workload": "prune_ldm loop, C5 cin256-v2 (seeded weights), B=%d, DDIM-20 scale 3 eta 0, Taylor pass at t=iteration" % B,
        "sample_ms": round(sample_ms, 3), "taylor_pass_ms": round(taylor_ms, 3), "iteration_ms": round(iter_ms, 3),
        "iterations_per_s": round(1e3 / iter_ms, 3), "sampling_share": round(sample_ms / iter_ms, 4),
        "eager_oracle_iteration_ms_tf32": round(eager_tf32, 1), "eager_oracle_iteration_ms_fp32": round(eager_fp32, 1),
        "speedup_vs_eager_tf32": round(eager_tf32 / iter_ms, 2), "speedup_vs_eager_fp32": round(eager_fp32 / iter_ms, 2),
        "gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock": info.get("clocks.sm"),
        "sm_clock_max": info.get("clocks.max.sm"), "sm_clock_after_eager": info_after.get("clocks.sm")}))


if __name__ == "__main__":
    main()
