#!/usr/bin/env python
"""Time ddpm_exp's FID sampling loop on the engine: the CIFAR-10 config (configs/cifar10.yml, seeded weights), batch 64
(sampling.batch_size), 100 quad steps at eta 0 — one sample_image call, i.e. one round of sample_fid without the PNG writes.

Reports, as one JSON line: img/s and ms per step of the engine loop (CUDA events around whole samples after a warm-up sample); the same
100 steps as torch eager with the float32 oracle Model (oracle/ddpm_exp_oracle.py) and generalized_steps' update on this GPU, with cuDNN /
matmul TF32 allowed and with plain fp32; and the GPU's name, power limit and SM clocks read in the same call.  Writes nothing.

    python scripts/time_ddpm_exp_sample.py [--iters 3] [--eager-steps 10]
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
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--eager-steps", type=int, default=10, help="steps of the eager arms timed (ms per step is what is reported)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ddpm_exp_sample.py measures on a CUDA device")
    import diff_pruning_b200.ddpm_exp as de
    from oracle import ddpm_exp_oracle as xo
    cfg = de.dict2namespace(de.CIFAR10_CONFIG)
    B, S = cfg.sampling.batch_size, 100
    torch.manual_seed(0)
    m = de.Model(de.CIFAR10_CONFIG).eval().cuda()
    betas = de.beta_schedule(cfg).cuda()
    x = torch.randn(B, 3, 32, 32, device="cuda")
    de.sample_image(x, m, betas, S, "quad", 0.0)           # builds the plan, captures the graph
    ms = events_ms(lambda: de.sample_image(x, m, betas, S, "quad", 0.0), a.iters)
    out = {"what": "ddpm_exp sample_image, CIFAR-10 config, batch 64, 100 quad steps, eta 0", "engine_img_s": B / (ms / 1e3),
           "engine_ms_per_step": ms / S}

    sd = {k: v.detach() for k, v in m.state_dict().items()}
    seq, seq_next = de.timestep_sequence(1000, S, "quad")
    ac = xo.alphas(betas)
    pairs = list(zip(reversed(seq), reversed(seq_next)))[:a.eager_steps]

    def eager():
        with torch.no_grad():
            xt = x
            for i, j in pairs:
                e = xo.forward(sd, xt, torch.full((B,), float(i), device="cuda"))
                xt, _ = xo.generalized_update(xt, e, torch.randn_like(x), ac[i + 1].view(1), ac[j + 1].view(1), 0.0)
    for name, tf32 in (("eager_tf32", True), ("eager_fp32", False)):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        eager()
        e_ms = events_ms(eager, 2) / len(pairs)
        out[f"{name}_ms_per_step"] = e_ms
        out[f"{name}_img_s"] = B / (e_ms * S / 1e3)
    out["speedup_vs_eager_tf32"] = out["eager_tf32_ms_per_step"] / out["engine_ms_per_step"]
    out["speedup_vs_eager_fp32"] = out["eager_fp32_ms_per_step"] / out["engine_ms_per_step"]
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
