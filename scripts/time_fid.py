"""Throughput of the FID Inception feature pass (inception.py, all four output blocks) from device buffers at batch 256: the project's
plan (one CUDA graph; convolutions on the general-geometry tensor-core kernel with the ReLU epilogue), the same plan with every
convolution on the exact-fp32 SIMT kernel, and the torch-eager restatement in oracle/inception_oracle.py on the same GPU with cuDNN in
TF32 and in fp32.  Weights are the seeded stand-in of the test fixtures (timing does not depend on them).
Warm-up first, then `--repeats` alternated rounds of `--iters` passes each; medians are printed with the card's name and power limit.
Usage: python scripts/time_fid.py [--batch 256] [--iters 3] [--repeats 3] [--out FILE.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import diff_pruning_b200.fid as fid  # noqa: E402
from oracle import inception_oracle as orc  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fid.py measures on a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    lay = json.load(open(os.path.join(ROOT, "tests", "golden", "fid_weights.json")))
    tv = orc.seeded_state_dict(lay["weight_file"], lay["seed"])
    model = fid.InceptionV3([0, 1, 2, 3], weights=tv).cuda()
    sd = {k: v.cuda() for k, v in fid.convert_torchvision_state_dict(tv).items()}
    B = a.batch
    x = torch.rand(B, 3, 32, 32, device="cuda")          # CIFAR-10 sized samples, resized to 299 x 299 inside the pass
    plan = model.plan(B, "f32", (32, 32))
    plan.load(x)
    simt = fid.FeaturePlan(model, B, "f32", (32, 32), force_simt=True)
    simt.load(x)

    def eager(tf32):
        def f():
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                orc.forward(sd, x, (0, 1, 2, 3))
        return f

    legs = {"plan": plan.run, "plan_all_simt": simt.run, "torch_cudnn_tf32": eager(True), "torch_cudnn_fp32": eager(False)}
    for f in legs.values():          # warm-up: module loading, graph capture, cuDNN algorithm choice
        f()
        f()
    torch.cuda.synchronize()
    err = float(((plan.feat[3] - simt.feat[3]).abs().max() / simt.feat[3].abs().max()))
    times = {k: [] for k in legs}
    for _ in range(a.repeats):
        for k, f in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / 1e3 / a.iters)
    res = {"card": card, "batch": B, "pool3_max_rel_vs_simt": err, "conv_gmac_per_img": plan.macs / B / 1e9, "input": "fp32 NCHW 32x32 -> 299x299"}
    for k, ts in times.items():
        t = statistics.median(ts)
        res[k] = {"img_per_s": B / t, "s_per_batch": t, "conv_tmac_per_s": plan.macs / t / 1e12, "runs": ts}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
