#!/usr/bin/env python
"""Time prune.py's Taylor loop for ddpm_exp's Model on the engine: the CIFAR-10 config (configs/cifar10.yml, seeded weights), batch 128
(the script's --taylor_batch_size default), one fixed batch and noise, t = step_k for every image.

Reports, as one JSON line: Taylor passes per second of the engine loop (per step: the forward + loss graph, the host read of the loss
that `--pruner ours` makes, the backward graph; CUDA events around --steps steps after --warmup steps); the same pass as torch eager on
the reference math (the Model's module-by-module torch forward under models.trace_mode() and noise_estimation_loss(...).backward()),
with cuDNN / matmul TF32 allowed and in plain fp32; the three arms alternate in --rounds rounds and each reports its fastest window; and the GPU's name, power limit and SM clocks read in the same
call.  Writes nothing.

    python scripts/time_ddpm_exp_prune.py [--steps 50] [--warmup 5] [--eager-steps 20] [--rounds 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

import torch  # noqa: E402

from time_ldm_decode import events_ms, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--eager-steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ddpm_exp_prune.py measures on a CUDA device")
    import diff_pruning_b200.ddpm_exp as de
    from diff_pruning_b200.models import trace_mode
    from diff_pruning_b200.scoring import TaylorScorer
    cfg = de.dict2namespace(de.CIFAR10_CONFIG)
    B = 128
    torch.manual_seed(0)
    m = de.Model(de.CIFAR10_CONFIG).eval().cuda()
    b = de.beta_schedule(cfg).cuda()
    x = torch.rand(B, 3, 32, 32, device="cuda") * 2 - 1
    e = torch.randn_like(x)
    m.zero_grad()
    ts = TaylorScorer(m, x, e, alphas_cumprod=(1 - b).cumprod(0), reduction="sum_mean")
    k = [0]

    def engine_step():
        loss = ts.forward_loss(k[0] % 1000)
        float(loss.item())
        ts.backward()
        k[0] += 1

    def eager_step():
        with trace_mode():
            de.noise_estimation_loss(m, x, torch.full((B,), k[0] % 1000, dtype=torch.long, device="cuda"), e, b).backward()
        k[0] += 1
    for _ in range(a.warmup):
        engine_step()
    res = {"engine": [], "eager_tf32": [], "eager_fp32": []}
    for _ in range(a.rounds):      # the three arms alternate, so each sees the same clock and thermal state
        res["engine"].append(events_ms(engine_step, a.steps))
        for name, tf32 in (("eager_tf32", True), ("eager_fp32", False)):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            eager_step()
            res[name].append(events_ms(eager_step, a.eager_steps))
    ms = min(res["engine"])
    out = {"what": "ddpm_exp prune.py Taylor loop, CIFAR-10 config, batch 128", "engine_passes_s": 1e3 / ms, "engine_ms_per_pass": ms,
           "steps": a.steps, "eager_steps": a.eager_steps, "rounds": a.rounds, "windows_ms": res}
    for name in ("eager_tf32", "eager_fp32"):
        out[f"{name}_ms_per_pass"] = min(res[name])
        out[f"speedup_vs_{name}"] = min(res[name]) / ms
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
