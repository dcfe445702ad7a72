"""Device time of single fprop / dgrad / attention NT GEMM launches on the persistent tensor-core kernel (conv_tc_ps_kernel) at the
C1 (CIFAR-10, batch 128) and C3 (LSUN-256, batch 4) shapes, plus one general-geometry fprop (Inception-v3, DP_CONV_ANY_GEOMETRY).
A stride-2 dgrad is one call that runs its four parity classes back to back.  Split-K launches get the workspace the engine gives them.
Set DPB200_LIB to time another build of the library, e.g. alternating two builds in one session.
Usage: python scripts/time_tc_shapes.py"""
import ctypes as C
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import diff_pruning_b200  # noqa: F401,E402
from diff_pruning_b200 import _lib as L  # noqa: E402

lib = L.load()
S = lambda: torch.cuda.current_stream().cuda_stream
ITERS = int(os.environ.get("ITERS", "20"))
ANY = 8   # DP_CONV_ANY_GEOMETRY


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / ITERS


def conv(op, N, Cin, K, H, R=3, stride=1, pad=None, flags=0):
    """op 'fprop': x [N][H][H][Cin] -> y [N][H/stride][..][K];  op 'dgrad': dy [N][P][P][K] -> dx [N][H][H][Cin]."""
    pad = R // 2 if pad is None else pad
    P = (H + 2 * pad - R) // stride + 1
    x = torch.randn(N, H, H, Cin, device="cuda")
    y = torch.randn(N, P, P, K, device="cuda")
    w = torch.randn(K, Cin, R, R, device="cuda") / (Cin * R * R) ** 0.5
    Cp, Kp = lib.dp_tc_weight_row(Cin), lib.dp_tc_weight_row(K)
    packs = [torch.empty(n, device="cuda", dtype=torch.float16) for n in (R * R * K * Cp, R * R * K * Cp, R * R * Cin * Kp, R * R * Cin * Kp)]
    slots = torch.zeros(3, dtype=torch.int32, device="cuda")     # [weight, x, dy] amax slots
    assert lib.dp_pack_conv_weight_tc(w.data_ptr(), K, Cin, R, R, *[p.data_ptr() for p in packs], slots.data_ptr(), S()) == 0
    assert lib.dp_amax(x.data_ptr(), Cin, N * H * H, Cin, slots.data_ptr() + 4, S()) == 0
    assert lib.dp_amax(y.data_ptr(), K, N * P * P, K, slots.data_ptr() + 8, S()) == 0
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S = N, H, H, Cin, P, P, K, R, R
    a.stride, a.pad_t, a.pad_l, a.splits, a.flags = stride, pad, pad, 1, flags
    a.x, a.ldx, a.y, a.ldy, a.w = x.data_ptr(), Cin, y.data_ptr(), K, w.data_ptr()
    a.amax_w, a.amax_x, a.amax_y = slots.data_ptr(), slots.data_ptr() + 4, slots.data_ptr() + 8
    if op == "fprop":
        a.w_tc_hi, a.w_tc_lo = packs[0].data_ptr(), packs[1].data_ptr()
        call = lib.dp_conv2d_fprop
    else:
        a.w_tc_hi, a.w_tc_lo = packs[2].data_ptr(), packs[3].data_ptr()
        call = lib.dp_conv2d_dgrad
    n_ws = lib.dp_conv_splitk_workspace_floats(C.byref(a), 0 if op == "fprop" else 1)
    ws = torch.empty(max(n_ws, 1), device="cuda")
    a.workspace = ws.data_ptr() if n_ws else None
    us = timed(lambda: L.check(call(C.byref(a), S())))
    macs = N * P * P * K * Cin * R * R
    tag = f"{op} {R}x{R}{' s2' if stride == 2 else ''} {Cin:4d}->{K:4d} @{H}x{H} N={N}{' (any)' if flags & ANY else ''}{' split-K' if n_ws else ''}"
    return tag, us, macs


def nt_gemm(N, T, inner):
    """Attention logits S = q k^T per image: A = q [N][T][inner] (token grid HxW), B = split(k), C [N][T][T]."""
    hw = int(round(T ** 0.5))
    q = torch.randn(N, T, inner, device="cuda")
    k = torch.randn(N, T, inner, device="cuda")
    out = torch.empty(N, T, T, device="cuda")
    i8 = (inner + 7) // 8 * 8
    hi = torch.empty(N * T * i8, device="cuda", dtype=torch.float16)
    lo = torch.empty_like(hi)
    slots = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert lib.dp_amax(q.data_ptr(), inner, N * T, inner, slots.data_ptr(), S()) == 0
    assert lib.dp_amax(k.data_ptr(), inner, N * T, inner, slots.data_ptr() + 4, S()) == 0
    assert lib.dp_split_h3(k.data_ptr(), inner, T * inner, N, T, inner, 0, slots.data_ptr() + 4, hi.data_ptr(), lo.data_ptr(), S()) == 0
    g = L.GemmNtArgs()
    g.batch, g.H, g.W, g.Kg, g.N = N, hw, hw, inner, T
    g.A, g.ld_a, g.b_hi, g.b_lo, g.C, g.ldc, g.alpha = q.data_ptr(), inner, hi.data_ptr(), lo.data_ptr(), out.data_ptr(), T, inner ** -0.5
    g.amax_a, g.amax_b = slots.data_ptr(), slots.data_ptr() + 4
    us = timed(lambda: L.check(lib.dp_gemm_nt_tc(C.byref(g), S())))
    return f"attn qk^T NT GEMM T={T} d={inner} N={N}", us, N * T * T * inner


CASES = [
    # C1: batch 128, 32x32 / 16x16 / 8x8 / 4x4 levels
    ("C1", lambda: conv("fprop", 128, 128, 128, 32)),
    ("C1", lambda: conv("fprop", 128, 384, 128, 32)),
    ("C1", lambda: conv("fprop", 128, 256, 256, 16)),
    ("C1", lambda: conv("fprop", 128, 256, 256, 8)),
    ("C1", lambda: conv("fprop", 128, 256, 256, 4)),
    ("C1", lambda: conv("fprop", 128, 128, 128, 32, stride=2)),
    ("C1", lambda: conv("dgrad", 128, 128, 128, 32)),
    ("C1", lambda: conv("dgrad", 128, 384, 128, 32)),
    ("C1", lambda: conv("dgrad", 128, 256, 256, 16)),
    ("C1", lambda: conv("dgrad", 128, 256, 256, 4)),
    ("C1", lambda: conv("dgrad", 128, 128, 128, 32, stride=2)),
    ("C1", lambda: conv("dgrad", 128, 256, 256, 16, stride=2)),
    ("C1", lambda: nt_gemm(128, 256, 256)),
    # C3: batch 4, LSUN-256
    ("C3", lambda: conv("fprop", 4, 128, 128, 256)),
    ("C3", lambda: conv("fprop", 4, 256, 256, 64)),
    ("C3", lambda: conv("fprop", 4, 512, 512, 16)),
    ("C3", lambda: conv("dgrad", 4, 128, 128, 256)),
    ("C3", lambda: conv("dgrad", 4, 128, 128, 256, stride=2)),
    ("C3", lambda: conv("dgrad", 4, 512, 512, 16)),
    ("C3", lambda: nt_gemm(4, 256, 512)),
    # Inception-v3 (FID): conv_tc_ps_kernel<true>
    ("FID", lambda: conv("fprop", 100, 64, 96, 35, flags=ANY)),
]

if __name__ == "__main__":
    print(f"{torch.cuda.get_device_name()}  lib {os.environ.get('DPB200_LIB', L.LIB_PATH)}")
    for cfg, case in CASES:
        tag, us, macs = case()
        print(f"{cfg:4s} {tag:52s} {us:9.1f} us  {2.0 * macs / us / 1e6:6.1f} TF algorithmic", flush=True)
        torch.cuda.empty_cache()
