"""Device time of each convolution geometry of the FID Inception pass (the MAC table of one 299 x 299 image, at batch 32): the box
tensor-core kernel where it takes the shape, the general-geometry kernel (DP_CONV_ANY_GEOMETRY), and the exact-fp32 SIMT kernel, all with
the ReLU epilogue except the box kernel (which does not take it).  CUDA events over 10 launches after 3 warm-ups; the card's name and power
limit are printed first.  Usage: python scripts/time_inception_convs.py [--batch 32]"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diff_pruning_b200 import _lib as L  # noqa: E402

# (C, K, R, S, stride, pad_h, pad_w, H, W, convs per image)
GEOMS = [(128, 128, 1, 7, 1, 0, 3, 17, 17, 13), (160, 192, 7, 1, 1, 3, 0, 17, 17, 13), (768, 192, 1, 1, 1, 0, 0, 17, 17, 18),
         (64, 80, 1, 1, 1, 0, 0, 73, 73, 1), (80, 192, 3, 3, 1, 0, 0, 73, 73, 1), (64, 96, 3, 3, 1, 1, 1, 35, 35, 7),
         (32, 64, 3, 3, 1, 1, 1, 147, 147, 1), (288, 384, 3, 3, 2, 0, 0, 35, 35, 2), (1280, 320, 1, 1, 1, 0, 0, 8, 8, 8),
         (48, 64, 5, 5, 1, 2, 2, 35, 35, 3), (288, 64, 1, 1, 1, 0, 0, 35, 35, 13), (32, 32, 3, 3, 1, 0, 0, 149, 149, 1),
         (448, 384, 3, 3, 1, 1, 1, 8, 8, 2), (384, 384, 1, 3, 1, 0, 1, 8, 8, 8), (192, 192, 3, 3, 2, 0, 0, 17, 17, 2),
         (3, 32, 3, 3, 2, 0, 0, 299, 299, 1)]


def box_takes(N, H, W, C, R, S, st, ph, pw, P, Q):
    """The shapes dp_conv2d_fprop's box tensor-core kernel accepts (conv_tc.cu: dp_conv2d_fprop_tc, pick_box)."""
    if R != S or R not in (1, 3) or ph != pw or C % 4:
        return False
    if not ((st == 1 and ph == (R - 1) // 2) or (st == 2 and R == 3 and ph in (0, 1))) or P * st != H or Q * st != W:
        return False
    if Q >= 128:
        return Q % 128 == 0
    if 128 % Q:
        return False
    rem = 128 // Q
    return P % rem == 0 if P >= rem else rem % P == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    N = ap.parse_args().batch
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    lib = L.load()
    S = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    for Cin, K, R, Sw, st, ph, pw, H, W, n in GEOMS:
        P, Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - Sw) // st + 1
        ldx = (Cin + 3) // 4 * 4
        x = torch.randn(N, H, W, ldx, device="cuda")
        w = torch.randn(K, Cin, R, Sw, device="cuda") / (Cin * R * Sw) ** 0.5
        y = torch.empty(N, P, Q, K, device="cuda")
        cp = lib.dp_tc_weight_row(Cin)
        wpk = torch.empty(R * Sw * Cin * K, device="cuda")
        hi, lo = (torch.empty(R * Sw * K * cp, dtype=torch.float16, device="cuda") for _ in range(2))
        slots = torch.zeros(3, dtype=torch.int32, device="cuda")
        assert lib.dp_pack_conv_weight(w.data_ptr(), K, Cin, R, Sw, wpk.data_ptr(), None, S()) == 0
        assert lib.dp_pack_conv_weight_tc(w.data_ptr(), K, Cin, R, Sw, hi.data_ptr(), lo.data_ptr(), None, None, slots.data_ptr(), S()) == 0
        assert lib.dp_amax(x.data_ptr(), ldx, N * H * W, Cin, slots.data_ptr() + 4, S()) == 0
        row = {}
        for name, flags in (("box", 0), ("general", 4 | 8), ("simt", 4 | 2)):
            a = L.ConvArgs()
            a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S = N, H, W, Cin, P, Q, K, R, Sw
            a.stride, a.pad_t, a.pad_l, a.splits, a.flags = st, ph, pw, 1, flags
            a.x, a.ldx, a.y, a.ldy, a.w = x.data_ptr(), ldx, y.data_ptr(), K, wpk.data_ptr()
            a.w_tc_hi, a.w_tc_lo, a.amax_w, a.amax_x, a.amax_out = hi.data_ptr(), lo.data_ptr(), slots.data_ptr(), slots.data_ptr() + 4, slots.data_ptr() + 8
            need = lib.dp_conv_splitk_workspace_floats(C.byref(a), 0)
            ws = torch.empty(max(need, 1), device="cuda")
            a.workspace = ws.data_ptr() if need else None
            if name == "box" and not box_takes(N, H, W, Cin, R, Sw, st, ph, pw, P, Q):
                row[name] = None
                continue
            for _ in range(3):
                assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
            e1.record()
            torch.cuda.synchronize()
            row[name] = e0.elapsed_time(e1) * 100      # us per launch
        macs = N * P * Q * K * Cin * R * Sw
        cells = "  ".join(f"{k} {'   n/a' if v is None else f'{v:8.1f} us {macs / v / 1e6:6.2f} TMAC/s'}" for k, v in row.items())
        print(f"{R}x{Sw} s{st} p({ph},{pw}) {H}x{W} C{Cin:5d} K{K:4d} x{n:2d}/img: {cells}", flush=True)


if __name__ == "__main__":
    main()
