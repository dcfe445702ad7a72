#!/usr/bin/env python
"""Time the LDM's VQ-f4 first-stage encode on the engine (VQModelInterface.encode, 256 x 256 images in [-1, 1] to 64 x 64 latents, seeded
weights) and one iteration of test_criterion.py's loop on cin256-v2 (LDMPruneScorer(encode_samples=True): guided DDIM-20 at batch 6,
encode of the 3 x 64 x 64 samples to 3 x 16 x 16, the Taylor pass).

Reports, as one JSON line: encode img/s at micro-batch 8 (graph replays, CUDA events) with the plan's bytes_allocated; the same encode as
torch eager with the float32 oracle (tests/vq_encoder_oracle.py) on this GPU with cuDNN / matmul TF32 allowed and with plain fp32; the loop's
time per iteration; and the GPU's name, power limit and SM clocks read in the same call.  Writes nothing.

    python scripts/time_ldm_encode.py [--iters 5] [--loop-iters 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import torch  # noqa: E402

from time_ldm_decode import events_ms, gpu_info  # noqa: E402


def seeded_vq_f4():
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    torch.manual_seed(0)
    return VQModelInterface(**VQ_F4_CONFIG, with_encoder=True).eval().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--loop-iters", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ldm_encode.py measures on a CUDA device")
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    import vq_encoder_oracle as eo
    out = {"gpu": gpu_info()}
    m = seeded_vq_f4()
    g = torch.Generator(device="cuda").manual_seed(1)
    mb = m.encode_batch
    x = torch.rand(mb, 3, 256, 256, device="cuda", generator=g) * 2 - 1
    m.encode(x)
    torch.cuda.synchronize()
    ms = events_ms(lambda: m.encode(x), a.iters)
    out[f"engine_mb{mb}"] = {"ms_per_batch": round(ms, 2), "img_per_s": round(mb / ms * 1e3, 2),
                             "plan_gib": round(m.__dict__["_dpb200_encode"].plan.bytes_allocated() / 2 ** 30, 2)}
    m.__dict__.pop("_dpb200_encode", None)
    torch.cuda.empty_cache()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    for tf32 in (True, False):
        prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        try:
            with torch.no_grad():
                eo.encode(sd, VQ_F4_CONFIG["ddconfig"], x)
                torch.cuda.synchronize()
                ms = events_ms(lambda: eo.encode(sd, VQ_F4_CONFIG["ddconfig"], x), max(1, a.iters // 2))
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        out[f"eager_oracle_{'tf32' if tf32 else 'fp32'}_b{mb}"] = {"ms_per_batch": round(ms, 2), "img_per_s": round(mb / ms * 1e3, 2)}
    torch.cuda.empty_cache()
    out["encode_speedup_vs_eager_tf32"] = round(out[f"engine_mb{mb}"]["img_per_s"] / out[f"eager_oracle_tf32_b{mb}"]["img_per_s"], 2)
    print(json.dumps(out), flush=True)
    out["criterion_loop"] = criterion_loop(m, a.loop_iters)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


def criterion_loop(vq, iters, B=6):
    """LDMPruneScorer(encode_samples=True).run('taylor') on cin256-v2 seeded as bench.py's C5: one warm-up iteration (plans and graphs),
    then `iters` iterations timed on the host clock around a synchronised run."""
    from time_ldm_prune_loop import c5_latent_diffusion
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    ld = c5_latent_diffusion()
    ld.first_stage_model = vq
    sc = LDMPruneScorer(ld, n_samples_per_class=B, ddim_steps=20, scale=3.0, encode_samples=True)
    gen = torch.Generator().manual_seed(0)
    sc.run("taylor", iterations=1, generator=gen)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sc.run("taylor", iterations=iters, generator=gen)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    return {"batch": B, "ddim_steps": 20, "iterations": iters, "ms_per_iteration": round((t1 - t0) / iters * 1e3, 1)}


if __name__ == "__main__":
    main()
