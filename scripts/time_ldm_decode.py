#!/usr/bin/env python
"""Time the LDM's VQ-f4 first-stage decode on the engine (VQModelInterface.decode, 256 x 256 images from 64 x 64 latents, seeded weights)
and one batch of sample_for_FID.py's loop (ldm_sampling.sample_for_fid: guided DDIM-250 of cin256-v2 at batch 25, decode, save_image bytes;
the reference renders 50 per batch, but a guided cin256-v2 plan takes at most 32 images: its LayerNorm runs over at most 65535 tokens).

Reports, as one JSON line: decode img/s at micro-batch 8 and 16 (graph replays, CUDA events) with each plan's bytes_allocated; the same
decode as torch eager with the float32 oracle (oracle/vq_oracle.py) on this GPU with cuDNN / matmul TF32 allowed and with plain fp32;
one sample_for_fid batch split into its sampling time and its decode (+ bytes) time; and the GPU's name, power limit and SM clocks read
in the same call.  Writes nothing.

    python scripts/time_ldm_decode.py [--iters 5] [--sample-batch 25] [--steps 250]
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


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def seeded_vq_f4():
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    torch.manual_seed(0)
    return VQModelInterface(**VQ_F4_CONFIG).eval().cuda()


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sample-batch", type=int, default=25)
    ap.add_argument("--steps", type=int, default=250)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ldm_decode.py measures on a CUDA device")
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    from oracle import vq_oracle as vo
    out = {"gpu": gpu_info()}
    m = seeded_vq_f4()
    g = torch.Generator(device="cuda").manual_seed(1)
    for mb in (8, 16):
        m.decode_batch = mb
        h = torch.randn(mb, 3, 64, 64, device="cuda", generator=g) * 2e-4
        m.decode(h)
        torch.cuda.synchronize()
        ms = events_ms(lambda: m.decode(h), a.iters)
        out[f"engine_mb{mb}"] = {"ms_per_batch": round(ms, 2), "img_per_s": round(mb / ms * 1e3, 2),
                                 "plan_gib": round(m.__dict__["_dpb200_decode"].plan.bytes_allocated() / 2 ** 30, 2)}
    m.__dict__.pop("_dpb200_decode", None)
    torch.cuda.empty_cache()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    h = torch.randn(8, 3, 64, 64, device="cuda", generator=g) * 2e-4
    for tf32 in (True, False):
        prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        try:
            with torch.no_grad():
                vo.decode(sd, VQ_F4_CONFIG["ddconfig"], h)
                torch.cuda.synchronize()
                ms = events_ms(lambda: vo.decode(sd, VQ_F4_CONFIG["ddconfig"], h), max(1, a.iters // 2))
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        out[f"eager_oracle_{'tf32' if tf32 else 'fp32'}_b8"] = {"ms_per_batch": round(ms, 2), "img_per_s": round(8 / ms * 1e3, 2)}
    torch.cuda.empty_cache()
    out["decode_speedup_vs_eager_tf32"] = round(out["engine_mb8"]["img_per_s"] / out["eager_oracle_tf32_b8"]["img_per_s"], 2)
    print(json.dumps(out), flush=True)
    out["sample_for_fid"] = sample_batch(m, a.sample_batch, a.steps)
    print(json.dumps(out))


def sample_batch(vq, B, steps):
    """One class of sample_for_fid at batch B (cin256-v2 seeded as bench.py's C5, guided DDIM-`steps`), timed as its two halves: the
    DDIMSampler call (one graph replay) and decode + save_image bytes in micro-batches of 8; then the whole sample_for_fid call."""
    import tempfile
    from time_ldm_prune_loop import c5_latent_diffusion
    from diff_pruning_b200 import _lib as L
    from diff_pruning_b200.engine import _stream
    from diff_pruning_b200.ldm_sampling import DDIMSampler, sample_for_fid
    ld = c5_latent_diffusion()
    ld.first_stage_model = vq
    key = ld.cond_stage_key
    uc = ld.get_learned_conditioning({key: torch.full((B,), 1000, device="cuda")})
    c = ld.get_learned_conditioning({key: torch.full((B,), 7, device="cuda")})
    sampler = DDIMSampler(ld)
    vq.decode_batch = 8
    lib = L.load()
    u8 = torch.empty(B, 256, 256, 3, dtype=torch.uint8, device="cuda")

    def sample():
        return sampler.sample(S=steps, conditioning=c, batch_size=B, shape=[3, 64, 64], verbose=False, unconditional_guidance_scale=3.0,
                              unconditional_conditioning=uc, eta=0.0)[0]

    def decode(z):
        for s in range(0, B, 8):
            y = vq.decode_chunk(z[s:s + 8]).plan.y_out
            n = min(8, B - s)
            L.check(lib.dp_decode_images(y.ptr, y.ld, n, 3, y.H, y.W, u8[s:s + n].data_ptr(), None, _stream()), "decode_images")
    z = sample()
    decode(z)              # warm-up: plans built, graphs captured
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    z = sample()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    decode(z)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    with tempfile.TemporaryDirectory() as d:
        t3 = time.perf_counter()
        _, _, n = sample_for_fid(ld, classes=[7], ipc=B, batch_size=B, ddim_steps=steps, out_dir=d)
        torch.cuda.synchronize()
        t4 = time.perf_counter()
    return {"batch": B, "ddim_steps": steps, "sample_s": round(t1 - t0, 3), "decode_s": round(t2 - t1, 3),
            "sample_for_fid_call_s_with_png_writes": round(t4 - t3, 3), "files": n}


if __name__ == "__main__":
    main()
