#!/usr/bin/env python
"""Time prune_ldm.py's loop (LDMPruneScorer.run) and a fixed slice of sample_for_FID.py's loop (ldm_sampling.sample_for_fid) with both
sharded over the processes of one torchrun launch, one GPU each: cin256-v2 with seeded weights (as scripts/time_ldm_prune_loop.py and
scripts/time_ldm_decode.py build it), the VQ-f4 decoder and a seeded stand-in Inception-v3 (timing does not depend on the weights).

* prune loop: batch 6, guided DDIM-20 at scale 3, eta 0, Taylor pass at t = iteration.  One warm-up run of one round (plans and graphs),
  then a timed run of --iters-per-rank rounds, the final gradient all-reduce included: iterations/s over all ranks.
* sample_for_fid: --batch images per batch, guided DDIM---steps at scale 3, eta 0, decode and FID moments (block 3, 2048 dims), no PNG
  files.  A warm-up call at DDIM-2 builds the plans; then calls with 1 and 2 batches per rank.  Each call captures its sampler's graph
  once (an eager sample), so the steady rate is taken from their difference: W * batch images over T(2) - T(1).

Rank 0 prints one JSON line with the GPUs' name, power limit and SM clock read in the same call.  Writes nothing.

    torchrun --nproc-per-node N scripts/time_ldm_sharded.py [--iters-per-rank 4] [--batch 25] [--steps 250]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def gpu_info():
    q = "index,name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        return []
    return [dict(zip(q.split(","), [v.strip() for v in line.split(",")])) for line in r.stdout.strip().splitlines()]


def timed(fn):
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters-per-rank", type=int, default=4)
    ap.add_argument("--batch", type=int, default=25)
    ap.add_argument("--steps", type=int, default=250)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ldm_sharded.py measures on CUDA devices; none found")
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (("WORLD_SIZE", "1"), ("RANK", "0"), ("LOCAL_RANK", "0")))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import __graft_entry__ as ge
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    ge.build()                          # up to date now: loads the library
    info = gpu_info()
    out = {"world": world, "prune_loop": prune_loop(world, a.iters_per_rank), "sample_for_fid": fid_slice(world, a.batch, a.steps)}
    out["gpus"], out["gpus_after"] = info, gpu_info()
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def prune_loop(world, rounds):
    from time_ldm_prune_loop import c5_latent_diffusion
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    B = 6
    ld = c5_latent_diffusion()
    ld.model.diffusion_model.zero_grad()
    sc = LDMPruneScorer(ld, n_samples_per_class=B, ddim_steps=20, scale=3.0, eta=0.0)
    g = torch.Generator(device="cuda").manual_seed(0)
    sc.run("taylor", iterations=world, generator=g)                 # builds both plans and all three graphs on every rank
    n = rounds * world
    s, _ = timed(lambda: sc.run("taylor", iterations=n, generator=g))
    del sc, ld
    torch.cuda.empty_cache()
    return {"workload": f"C5 cin256-v2 (seeded weights), B={B}, DDIM-20 scale 3 eta 0, Taylor pass at t=iteration",
            "iterations": n, "seconds": round(s, 3), "iterations_per_s": round(n / s, 3), "ms_per_iteration": round(s * 1e3 / n, 1)}


def fid_slice(world, B, steps):
    from time_ldm_decode import seeded_vq_f4
    from time_ldm_prune_loop import c5_latent_diffusion
    from diff_pruning_b200 import fid
    from diff_pruning_b200.ldm_sampling import sample_for_fid
    from oracle import inception_oracle as orc
    lay = json.load(open(os.path.join(ROOT, "tests", "golden", "fid_weights.json")))
    inc = fid.InceptionV3([3], weights=orc.seeded_state_dict(lay["weight_file"], lay["seed"])).cuda()
    ld = c5_latent_diffusion()
    ld.first_stage_model = seeded_vq_f4()

    def call(per_rank, S):
        return sample_for_fid(ld, classes=range(per_rank * world), ipc=B, batch_size=B, ddim_steps=S, inception=inc,
                              generator=torch.Generator(device="cuda").manual_seed(0))
    call(1, 2)                          # plans: the guided UNet at 2 B, the decoder, the Inception pass
    t1, _ = timed(lambda: call(1, steps))
    t2, (mu, _, _) = timed(lambda: call(2, steps))
    return {"workload": f"C5 cin256-v2 + VQ-f4 decoder (seeded weights), batch {B}, guided DDIM-{steps} scale 3 eta 0, decode, FID moments",
            "seconds_1_batch_per_rank": round(t1, 3), "seconds_2_batches_per_rank": round(t2, 3),
            "images_per_s": round(world * B / (t2 - t1), 3), "s_per_batch_per_rank": round(t2 - t1, 3),
            "images_per_s_2_batch_call": round(2 * world * B / t2, 3), "mu_finite": bool(np.isfinite(mu).all())}


if __name__ == "__main__":
    main()
