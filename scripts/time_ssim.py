"""Throughput of SSIM evaluation (dp_ssim) on batches of image pairs, from uint8 NHWC (decoded files) and from fp32 NCHW, at 32 x 32
(CIFAR-10) and 256 x 256 (LSUN / CelebA-HQ), against the fp32 torch restatement of pytorch_msssim (oracle/ssim_oracle.py, cuDNN
grouped convolutions) on the same GPU and inputs.  Per-image SSIM and MSE are produced by both.  Warm-up first, then `--repeats`
rounds that alternate the two implementations, `--iters` calls each, timed with CUDA events; medians are printed with the card's name,
power limit and the SM clock read right after the timed rounds.  GB/s counts the input bytes of both images once.
Usage: python scripts/time_ssim.py [--batch 100] [--iters 20] [--repeats 5] [--out FILE.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import diff_pruning_b200.ssim as S  # noqa: E402
from oracle import ssim_oracle as orc  # noqa: E402


def nvsmi(q):
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ssim.py measures on a CUDA device")
    card = nvsmi("name,power.limit,clocks.max.sm")
    torch.backends.cudnn.allow_tf32 = False
    B, rows = a.batch, []
    g = torch.Generator(device="cuda").manual_seed(0)
    for hw in (32, 256):
        u8a = torch.randint(0, 256, (B, hw, hw, 3), dtype=torch.uint8, device="cuda", generator=g)
        u8b = (u8a.int() + torch.randint(-16, 17, u8a.shape, device="cuda", generator=g)).clamp(0, 255).to(torch.uint8)
        fa, fb = (u.permute(0, 3, 1, 2).float().div(255).contiguous() for u in (u8a, u8b))

        def torch_fp32():
            with torch.no_grad():
                s = orc.ssim_per_channel(fa, fb, 1.0).mean(1)
                m = F.mse_loss(fa, fb, reduction="none").mean(dim=(1, 2, 3))
            return s, m
        legs = {"dp_ssim_u8": (lambda: S._scores(u8a, u8b, S.DP_SSIM_U8_NHWC, 1.0), 1),
                "dp_ssim_f32": (lambda: S._scores(fa, fb, S.DP_SSIM_F32_NCHW, 1.0), 4),
                "torch_fp32": (torch_fp32, 4)}
        for f, _ in legs.values():
            f()
            f()
        torch.cuda.synchronize()
        times = {k: [] for k in legs}
        for _ in range(a.repeats):
            for k, (f, _) in legs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    f()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / 1e3 / a.iters)
        clock = nvsmi("clocks.sm")
        ours = S._per_image(S._scores(fa, fb, S.DP_SSIM_F32_NCHW, 1.0)[0])
        ref64 = orc.ssim_per_channel(fa.double(), fb.double(), 1.0).mean(1)
        row = {"hw": hw, "batch": B, "sm_clock_after": clock, "max_abs_err_vs_fp64": {
            "dp_ssim": float((ours - ref64).abs().max()), "torch_fp32": float((torch_fp32()[0].double() - ref64).abs().max())}}
        for k, (f, elem_bytes) in legs.items():
            t = statistics.median(times[k])
            row[k] = {"pairs_per_s": B / t, "us_per_batch": t * 1e6, "GB_per_s": 2 * B * 3 * hw * hw * elem_bytes / t / 1e9,
                      "runs_us": [round(v * 1e6, 1) for v in times[k]]}
        rows.append(row)
        print(json.dumps(row))
    res = {"card": card, "rows": rows}
    print(json.dumps({"card": card}))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
