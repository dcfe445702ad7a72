"""Case tables of the dispatch-edge sweep (test_dispatch_edges_gpu.py runs them, test_dispatch_edges_host.py checks on the host that
every dispatch threshold of the kernels' host code has a case on each side), the thresholds as the CUDA sources state them, and
Python restatements of the host-side choices (box, K split, N tile, channel map, row kernels) that predict the path every case takes
at a given SM count.

A case is a dict: `op` names the entry point, the rest its extents and view layout.  `px` / `py` / `pb` / `pr` / `ps` are the 16-byte
phases (in fp32 elements) of x / y / bias / rowadd / residual; `xe` / `ye` widen the pixel pitch beyond the channel count.  A case
either runs (the host admits it and the kernel must compute it within the error model) or carries `refuse`, the exact return code.
"""
from __future__ import annotations

import os
import re

import launch_census as lc

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diff-pruning_b200", "csrc")
DP_ERR_SHAPE, DP_ERR_UNSUPPORTED = -1, -3
ACC, FORCE_SIMT, RELU, ANY = 1, 2, 4, 8


# ---------------------------------------------------------------------------------------------------------------- thresholds
def source(name: str) -> str:
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def const(name: str, file: str) -> int:
    """`constexpr int NAME = value` (alone or in a comma list) from a CUDA source."""
    m = re.search(r"constexpr int (?:[^;]*?,\s*)?" + name + r"\s*=\s*(\d+)", source(file))
    assert m, f"{name} not found in {file}"
    return int(m.group(1))


def thresholds() -> dict:
    """Every dispatch threshold the sweep straddles, read from the sources."""
    tc, nm, bf = source("conv_tc.cu"), source("norm.cu"), source("conv_bf16.cu")
    wr = re.search(r"static int wrow\(int c\) \{ return c > (\d+) \? \(\(c \+ (\d+)\) & ~\d+\) : \(\(c \+ (\d+)\) & ~\d+\); \}", tc)
    assert wr, "wrow rule not found in conv_tc.cu"
    ln = re.search(r"a->C <= (\d+) \* (\d+) \* LN_V", nm)
    assert ln, "ln_fast channel limit not found in norm.cu"
    nt = re.search(r"pl\.n_tiles = \(g\.Nout \+ (\d+)\) / (\d+);", bf)
    assert nt and int(nt.group(1)) + 1 == int(nt.group(2)), "plan_bf16 N-tile rule not found in conv_bf16.cu"
    return {
        "ANY_MIN_C": const("ANY_MIN_C", "conv_tc.cu"), "PS_MAX_SPLIT_STAGES": const("PS_MAX_SPLIT_STAGES", "conv_tc.cu"),
        "BM": const("BM", "conv_tc.cu"), "BK": const("BK", "conv_tc.cu"), "PS_BN": const("PS_BN", "conv_tc.cu"),
        "WROW_SPLIT": int(wr.group(1)), "WROW_LONG": int(wr.group(2)) + 1, "WROW_SHORT": int(wr.group(3)) + 1,
        "NT": const("NT", "norm.cu"), "MAXCPT": const("MAXCPT", "norm.cu"), "GN_FOLD_FWD": const("GN_FOLD_FWD", "norm.cu"),
        "GN_FOLD_BWD": const("GN_FOLD_BWD", "norm.cu"),
        "LN_MAX_C": int(ln.group(1)) * int(ln.group(2)) * const("LN_V", "norm.cu"),
        "WG_PIX": const("WG_PIX", "conv_bf16.cu"), "BF_NTILE": int(nt.group(2)),
        "WG_KPIX": const("WG_KPIX", "conv_tc.cu"),
    }


T = thresholds()


# ---------------------------------------------------------------------------------------------------------------- restatements
def cdiv(a, b):
    return -(-a // b)


def pick_box(npix, H, W):
    """sm90_host.cuh pick_box: (bw, bh, bn) or None."""
    if W >= npix:
        return (npix, 1, 1) if W % npix == 0 else None
    if npix % W:
        return None
    rem = npix // W
    if H >= rem:
        return (W, rem, 1) if H % rem == 0 else None
    if rem % H:
        return None
    return W, H, rem // H


def wrow(c):
    return cdiv(c, T["WROW_LONG"]) * T["WROW_LONG"] if c > T["WROW_SPLIT"] else cdiv(c, T["WROW_SHORT"]) * T["WROW_SHORT"]


def parity_taps(pad_t, pad_l, cls):
    return sum(1 for r in range(3) for s in range(3) if not ((cls >> 1) + pad_t - r) & 1 and not ((cls & 1) + pad_l - s) & 1)


def out_extent(c):
    """(P, Q) of a case: the box kernels' stride-2 grid is the input grid / 2, everything else the usual convolution arithmetic."""
    R, S, s = c["R"], c.get("S", c["R"]), c.get("stride", 1)
    pt, pl_ = c.get("pad", (R - 1) // 2), c.get("pad_l", c.get("pad", (S - 1) // 2))
    if s == 2 and R == S == 3 and pt == pl_ and pt in (0, 1) and not c.get("general"):
        return c["H"] // 2, c["W"] // 2
    return (c["H"] + 2 * pt - R) // s + 1, (c["W"] + 2 * pl_ - S) // s + 1


def al16(phase, ld):
    return phase == 0 and ld % 4 == 0


def box_geometry(c):
    R, S, s = c["R"], c.get("S", c["R"]), c.get("stride", 1)
    pt, pl_ = c.get("pad", (R - 1) // 2), c.get("pad_l", c.get("pad", (S - 1) // 2))
    P, Q = out_extent(c)
    if R != S or R not in (1, 3) or pt != pl_:
        return False
    if not ((s == 1 and pt == (R - 1) // 2) or (s == 2 and R == 3 and pt in (0, 1))):
        return False
    return P * s == c["H"] and Q * s == c["W"]


def conv_path(c, sms):
    """Path of an fp32-grade convolution case: {"kernel": "box" | "any" | "simt" | "wgrad_tc", "gemms": [(ksplit, stages per split,
    work items)], "vec4": bool, "box": (bw, bh, bn) or None, "ws_floats": split-K workspace the library must report, "L": chain}."""
    op, H, W, Cc, K = c["op"], c["H"], c["W"], c["C"], c["K"]
    R, S, s = c["R"], c.get("S", c["R"]), c.get("stride", 1)
    pt, pl_ = c.get("pad", (R - 1) // 2), c.get("pad_l", c.get("pad", (S - 1) // 2))
    P, Q = out_extent(c)
    ldx, ldy = Cc + c.get("xe", 0), K + c.get("ye", 0)
    flags = c.get("flags", 0)
    px, py = c.get("px", 0), c.get("py", 0)
    out = {"kernel": "simt", "gemms": [], "vec4": False, "box": None, "ws_floats": 0}
    N = at_sms(c, sms)["N"]
    if op == "wgrad":
        box = pick_box(T["WG_KPIX"], P, Q)
        ok = box_geometry(c) and al16(px, ldx) and al16(py, ldy) and box is not None and box[0] * s <= 256 and box[1] * s <= 256
        out.update(kernel="wgrad_tc" if ok else "simt", box=box if ok else None)
        sp = c.get("splits", 1)
        out["L"] = lc.chain_wgrad(lc.wgrad_pixels_per_cta(N * P * Q, sp), sp) if ok else None
        return out
    if op == "fprop":
        grids = [(1, N, P, Q, Cc, K, R * S, s)]            # (count, N, Hg, Wg, Kg, Nout, taps, in_stride)
        act_ok, out_ld, out_ph = al16(px, ldx), ldy, py
    elif s == 1:
        grids = [(1, N, H, W, K, Cc, R * S, 1)]
        act_ok, out_ld, out_ph = al16(py, ldy), ldx, px
    else:
        grids = [(1, N, P, Q, K, Cc, parity_taps(pt, pl_, cls), 1) for cls in range(4)]
        act_ok, out_ld, out_ph = al16(py, ldy), ldx, px
    epi = [(out_ph, out_ld)]
    if op == "fprop":
        epi += [(c.get("pb", 0), 0)] if c.get("bias") else []
        epi += [(c.get("pr", 0), K + c.get("re", 0))] if c.get("rowadd") else []
        epi += [(c.get("ps", 0), K + c.get("se", 0))] if c.get("residual") else []
    out["vec4"] = all(al16(ph, ld) for ph, ld in epi)
    ws = c.get("ws", True)
    if op == "fprop":
        box_ok = not flags & RELU and box_geometry(c)
    elif s == 1:
        box_ok = box_geometry(c)
    else:
        box_ok = R == S == 3 and H == 2 * P and W == 2 * Q
    box = pick_box(T["BM"], grids[0][2], grids[0][3]) if box_ok else None
    if box is not None and act_ok and box[0] * grids[0][7] <= 256 and box[1] * grids[0][7] <= 256:
        kernel = "box"
    elif op == "fprop" and flags & ANY and Cc >= T["ANY_MIN_C"] and not c.get("rowadd") and act_ok:
        kernel, box = "any", None
    else:
        out["L"] = R * S * (Cc if op == "fprop" else K)      # sequential fp32 FMAs of the SIMT kernel
        return out
    L = 0
    for _, n, Hg, Wg, Kg, Nout, taps, _s in grids:
        tiles_m = cdiv(n * Hg * Wg, T["BM"]) if kernel == "any" else cdiv(Wg, box[0]) * (Hg // box[1]) * cdiv(n, box[2])
        n_tiles = cdiv(Nout, T["PS_BN"])
        iters = taps * cdiv(Kg, T["BK"])
        ks, ips = pick_ksplit(tiles_m * n_tiles, iters, sms) if ws else (1, iters)
        out["gemms"].append((ks, ips, tiles_m * n_tiles * ks))
        if ks > 1:
            out["ws_floats"] = max(out["ws_floats"], ks * tiles_m * T["BM"] * n_tiles * T["PS_BN"])
        L = max(L, lc.chain_general(ks, ips))
    out.update(kernel=kernel, box=box, L=L)
    return out


def pick_ksplit(tiles, iters, sms):
    """conv_tc.cu pick_ksplit, statement by statement (launch_census.pick_ksplit is the census's own mirror; the host test holds
    the two to each other)."""
    ks = 1
    if tiles * 2 <= sms and iters >= 8:
        ks = sms // tiles
        if ks > iters // 4:
            ks = iters // 4
        if ks > 16:
            ks = 16
    chain_ks = (iters + T["PS_MAX_SPLIT_STAGES"] - 1) // T["PS_MAX_SPLIT_STAGES"]
    if ks < chain_ks:
        ks = chain_ks
    if ks < 2:
        return 1, iters
    ips = (iters + ks - 1) // ks
    return (iters + ips - 1) // ips, ips


def bf16_plan(c):
    """conv_bf16.cu: (eligible, bn_tile or wgrad in-channel tile, box) of a bf16 case, as plan_bf16 / plan_wgrad_bf16 decide."""
    op, N, Cc, K, s = c["op"], c["N"], c["C"], c["K"], c.get("stride", 1)
    P, Q = out_extent(c)
    ldx, ldy = Cc + c.get("xe", 0), K + c.get("ye", 0)
    if not box_geometry(c):
        return False, None, None
    if op == "wgrad":
        box = pick_box(T["WG_PIX"], P, Q)
        if ldx % 8 or ldy % 8 or box is None or N % box[2] or box[0] * s > 256 or box[1] * s > 256:
            return False, None, box
        tiles = cdiv(Cc, 256)
        return True, min(256, cdiv(cdiv(Cc, tiles), 64) * 64), box
    if op == "fprop":
        Hg, Wg, Kg, Nout, ld_act, st = P, Q, Cc, K, ldx, s
    elif s == 1:
        Hg, Wg, Kg, Nout, ld_act, st = c["H"], c["W"], K, Cc, ldy, 1
    else:
        Hg, Wg, Kg, Nout, ld_act, st = P, Q, K, Cc, ldy, 1
    box = pick_box(T["BM"], Hg, Wg)
    if ld_act % 8 or Kg < 8 or box is None or box[0] * st > 256 or box[1] * st > 256:
        return False, None, box
    nt = cdiv(Nout, T["BF_NTILE"])
    return True, min(T["BF_NTILE"], cdiv(cdiv(Nout, nt), 64) * 64), box


def make_map(HW, C):
    NT = T["NT"]
    if C >= NT:
        CT, PL = NT, 1
    else:
        CT = 32
        while CT < C:
            CT <<= 1
        PL = NT // CT
    ppc = min(max(8192 // C, PL), HW)
    ppc = max(ppc, 1)
    return CT, PL, ppc, cdiv(HW, ppc)


def make_map4(HW, C):
    NT = T["NT"]
    c4, CT = C // 4, 8
    while CT < c4:
        CT <<= 1
    PL = NT // CT
    ppc = max(min(max(16384 // C, PL), HW), 1)
    return CT, PL, ppc, cdiv(HW, ppc)


def ln_fast(c):
    return c["HW"] == 1 and c["G"] == 1 and c["C"] % 4 == 0 and c["C"] <= T["LN_MAX_C"]


def gn_path(c):
    """norm.cu: {"ln": row kernels?, "v4": float4 kernels?, "nchunks", "finalize" (forward finalize launch), "reduce" (backward
    reduce launch)} of a GroupNorm / LayerNorm case, or {"refuse": code} when validation turns it down."""
    C, bwd = c["C"], c["op"] == "gn_bwd"
    ph = dict(x=c.get("px", 0), y=c.get("py", 0), dy=c.get("pdy", 0), dx=c.get("pdx", 0), gamma=c.get("pg", 0), beta=c.get("pbeta", 0),
              add=c.get("padd", 0) if c.get("add") else 0, add2=c.get("padd2", 0) if c.get("add2") else 0)
    ld = dict(x=C + c.get("xe", 0), y=C + c.get("ye", 0), dy=C + c.get("dye", 0), dx=C + c.get("dxe", 0), gamma=0, beta=0,
              add=C + c.get("adde", 0), add2=C + c.get("add2e", 0))
    ok = lambda *names: all(al16(ph[n], ld[n]) for n in names)
    rows = ln_fast(c) and ok("x", "gamma") and (ok("dy", "dx", "add", "add2") if bwd else (not c.get("no_y") and ok("y", "beta")))
    if not (C <= T["NT"] * T["MAXCPT"] or rows) or c["G"] > 1024:
        return {"refuse": DP_ERR_UNSUPPORTED}
    if rows:
        return {"ln": True, "v4": True}
    if c["N"] > 65535:
        return {"refuse": DP_ERR_SHAPE}
    v4 = C % 4 == 0 and (ok("x", "dy", "dx", "add", "add2") if bwd else ok("x", "y"))
    nch = (make_map4 if v4 else make_map)(c["HW"], C)[3]
    return {"ln": False, "v4": v4, "nchunks": nch, "finalize": nch > T["GN_FOLD_FWD"], "reduce": nch > T["GN_FOLD_BWD"]}


# ---------------------------------------------------------------------------------------------------------------- the tables
def _cv(op, N, H, W, C, K, R=3, **kw):
    return dict(op=op, N=N, H=H, W=W, C=C, K=K, R=R, **kw)


def at_sms(c, sms):
    """The case on a device of `sms` SMs: a batch given as (a, b) is a * sms + b images (one 128-pixel tile each in the persistent-round
    cases, so the tile count sits at the same edge of the persistent grid on any part)."""
    return dict(c, N=c["N"][0] * sms + c["N"][1]) if isinstance(c["N"], tuple) else c


# fp32-grade convolutions.  Box: pick_box(128, ...) over the GEMM's grid; every other geometry falls to the SIMT kernel (or, with
# DP_CONV_ANY_GEOMETRY, the general-geometry kernel).  K split: see pick_ksplit; the persistent grid is min(work items, SMs).
CONV = [
    # pick_box branches (fprop, stride 1) and their SIMT fallbacks
    _cv("fprop", 2, 2, 128, 64, 64, tag="W == 128: one row per box"),
    _cv("fprop", 2, 2, 256, 64, 64, tag="128 divides W"),
    _cv("fprop", 2, 16, 16, 64, 64, tag="W divides 128, H fits"),
    _cv("fprop", 5, 8, 8, 64, 96, bias=True, tag="box of 2 images, the last past the batch"),
    _cv("fprop", 3, 4, 4, 40, 72, tag="box of 8 images past the batch, Kg / Nout tails"),
    _cv("fprop", 2, 8, 12, 64, 64, tag="W = 12: SIMT"),
    _cv("fprop", 2, 8, 24, 64, 64, tag="W = 24: SIMT"),
    _cv("fprop", 2, 4, 48, 32, 32, tag="W = 48: SIMT"),
    _cv("fprop", 1, 2, 192, 32, 32, tag="W = 192: SIMT"),
    _cv("fprop", 2, 6, 32, 64, 64, tag="W = 32, H = 6: SIMT"),
    # Kg / Nout tails around the 64-channel stage, the wrow split and the 128-channel N tile
    _cv("fprop", 2, 8, 16, 64, 128, R=1, tag="Kg 64, N 128"),
    _cv("fprop", 2, 8, 16, 65, 129, R=1, xe=3, tag="Kg 65 (wrow 128), N 129"),
    _cv("fprop", 2, 8, 16, 127, 256, R=1, xe=1, tag="Kg 127, N 256"),
    _cv("fprop", 2, 8, 16, 128, 257, R=1, tag="Kg 128, N 257"),
    _cv("fprop", 2, 8, 16, 8, 24, R=1, tag="Kg 8: short weight rows"),
    # pick_ksplit: no split (tiles cover half the SMs), split capped by iters / 4, capped at 16, iters 7 / 8, forced chain split
    _cv("fprop", 80, 16, 16, 64, 64, R=1, tag="160 tiles: no split"),
    _cv("fprop", 2, 8, 8, 256, 64, R=1, tag="iters 4 < 8: no split"),
    _cv("fprop", 2, 8, 8, 448, 64, R=1, tag="iters 7: no split"),
    _cv("fprop", 2, 8, 8, 512, 64, R=1, tag="iters 8: split capped at iters / 4"),
    _cv("fprop", 4, 8, 8, 512, 512, tag="split capped at 16"),
    _cv("fprop", 16, 16, 16, 1088, 128, tag="153 stages, 32 tiles: split over the SMs"),
    _cv("fprop", 67, 8, 16, 9408, 64, R=1, tag="147 stages, M fills the machine: no split"),
    _cv("fprop", 67, 8, 16, 9412, 64, R=1, tag="148 stages, M fills the machine: chain split forced"),
    # persistent rounds around the SM count (tile counts sms - 1, sms, sms + 1, 2 sms + 1 at 132 SMs)
    _cv("fprop", (1, -1), 8, 16, 32, 64, R=1, tag="sms - 1 tiles"),
    _cv("fprop", (1, 0), 8, 16, 32, 64, R=1, tag="sms tiles"),
    _cv("fprop", (1, 1), 8, 16, 32, 64, R=1, tag="sms + 1 tiles"),
    _cv("fprop", (2, 1), 8, 16, 32, 64, R=1, tag="2 sms + 1 tiles"),
    # vec4 epilogue: every pointer aligned, then each one off its 16-byte phase; accumulate
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, tag="vec4"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, ye=1, tag="scalar: y pitch"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, py=2, ye=4, tag="scalar: y phase"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, pb=1, tag="scalar: bias phase"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, pr=3, tag="scalar: rowadd phase"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, ps=1, tag="scalar: residual phase"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, ws=False, tag="vec4, no workspace"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, ps=1, ws=False, tag="scalar: residual phase, no workspace"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, rowadd=True, residual=True, pr=2, ws=False, tag="scalar: rowadd phase, no workspace"),
    _cv("fprop", 3, 8, 16, 64, 96, bias=True, residual=True, se=2, flags=ACC, tag="scalar: residual pitch, accumulate"),
    _cv("fprop", 2, 4, 4, 512, 256, bias=True, residual=True, flags=ACC, ye=1, tag="split, scalar epilogue, accumulate"),
    _cv("fprop", 3, 8, 16, 64, 96, px=1, xe=3, tag="x off 16 bytes: SIMT"),
    # stride-2 fprop: pad 0 / 1
    _cv("fprop", 4, 16, 16, 64, 96, stride=2, pad=0, tag="stride 2 pad 0"),
    _cv("fprop", 4, 16, 16, 64, 96, stride=2, pad=1, bias=True, tag="stride 2 pad 1"),
    # dgrad: stride 1, the stride-2 parity classes (pad 0 / 1, P odd / even), box and SIMT, split and not
    _cv("dgrad", 3, 8, 8, 96, 64, tag="dgrad stride 1, box past the batch"),
    _cv("dgrad", 2, 8, 12, 64, 64, tag="dgrad W = 12: SIMT"),
    _cv("dgrad", 3, 16, 16, 64, 96, stride=2, pad=0, tag="dgrad stride 2 pad 0, P even"),
    _cv("dgrad", 3, 16, 16, 64, 96, stride=2, pad=1, flags=ACC, tag="dgrad stride 2 pad 1, accumulate"),
    _cv("dgrad", 2, 18, 18, 64, 64, stride=2, pad=1, tag="dgrad stride 2 P odd: SIMT"),
    _cv("dgrad", 2, 6, 256, 32, 32, stride=2, pad=1, tag="dgrad stride 2 P = 3 on one-row boxes"),
    _cv("dgrad", 3, 2, 128, 32, 64, stride=2, pad=0, tag="dgrad stride 2 P = 1, box past the batch"),
    _cv("dgrad", 64, 16, 16, 64, 64, stride=2, pad=0, xe=1, tag="dgrad stride 2, scalar dx"),
    # general-geometry fprop
    _cv("fprop", 2, 9, 9, 31, 64, flags=ANY, general=True, tag="any: C 31 -> SIMT"),
    _cv("fprop", 2, 9, 9, 32, 64, flags=ANY, general=True, tag="any: C 32"),
    _cv("fprop", 2, 9, 13, 48, 80, R=1, S=7, pad=0, pad_l=3, flags=ANY, general=True, bias=True, tag="any: 1x7"),
    _cv("fprop", 2, 13, 9, 48, 80, R=7, S=1, pad=3, pad_l=0, flags=ANY, general=True, tag="any: 7x1"),
    _cv("fprop", 2, 11, 11, 64, 64, R=5, pad=2, flags=ANY | RELU, general=True, bias=True, residual=True, tag="any: 5x5 ReLU"),
    _cv("fprop", 2, 17, 17, 64, 96, R=3, pad=0, stride=2, flags=ANY | RELU, general=True, bias=True, tag="any: stride 2 valid"),
    _cv("fprop", 2, 8, 8, 64, 64, flags=ANY, rowadd=True, tag="any geometry flag, box shape, rowadd: box"),
    _cv("fprop", 2, 9, 9, 64, 64, flags=ANY, rowadd=True, general=True, tag="any with rowadd: SIMT"),
    _cv("fprop", 2, 8, 8, 64, 64, flags=RELU, bias=True, tag="ReLU: SIMT only"),
    _cv("fprop", 2, 9, 9, 64, 64, flags=ANY, ye=1, general=True, tag="any: scalar epilogue"),
    # weight gradient + dp_conv2d_wgrad_reduce
    _cv("wgrad", 4, 8, 8, 64, 96, splits=1, tag="wgrad box 64 px"),
    _cv("wgrad", 3, 4, 4, 64, 96, splits=1, tag="wgrad box of 4 images past the batch"),
    _cv("wgrad", 4, 16, 16, 96, 64, splits=3, tag="wgrad 3 splits"),
    _cv("wgrad", 2, 8, 12, 64, 64, splits=1, tag="wgrad W = 12: SIMT"),
    _cv("wgrad", 4, 16, 16, 64, 96, stride=2, pad=1, splits=2, tag="wgrad stride 2"),
    _cv("wgrad", 4, 8, 8, 64, 96, splits=1, xe=2, tag="wgrad x pitch: SIMT"),
]
# bf16 tier: N tile 64 / 128 / 192 / 256, ld % 8, Kg 7 / 8, the box past the batch (fprop takes it, the weight gradient refuses)
BF16 = [
    _cv("fprop", 2, 8, 16, 64, 64, R=1, tag="bn_tile 64"),
    _cv("fprop", 2, 8, 16, 64, 65, R=1, tag="bn_tile 128 (65)"),
    _cv("fprop", 2, 8, 16, 64, 192, R=1, bias=True, residual=True, tag="bn_tile 192"),
    _cv("fprop", 2, 8, 16, 64, 256, R=1, tag="bn_tile 256"),
    _cv("fprop", 2, 8, 16, 64, 257, R=1, tag="257: two tiles of 192"),
    _cv("fprop", 2, 8, 16, 64, 448, R=1, ye=1, tag="448: two tiles of 256, scalar epilogue"),
    _cv("fprop", 5, 8, 8, 64, 96, tag="box past the batch"),
    _cv("fprop", 2, 8, 16, 8, 64, R=1, tag="Kg 8"),
    _cv("fprop", 2, 8, 16, 7, 64, R=1, xe=1, refuse=DP_ERR_UNSUPPORTED, tag="Kg 7"),
    _cv("fprop", 2, 8, 16, 60, 64, R=1, xe=2, refuse=DP_ERR_UNSUPPORTED, tag="ld % 8"),
    _cv("fprop", 2, 8, 16, 64, 64, R=1, xe=8, tag="ld 72"),
    _cv("dgrad", 2, 8, 16, 130, 64, tag="dgrad bn_tile 192"),
    _cv("dgrad", 3, 16, 16, 64, 96, stride=2, pad=0, flags=ACC, tag="dgrad stride 2, accumulate"),
    _cv("wgrad", 4, 8, 8, 64, 96, splits=1, tag="wgrad"),
    _cv("wgrad", 4, 8, 8, 320, 64, splits=2, tag="wgrad in-channel tile 192"),
    _cv("wgrad", 3, 4, 4, 64, 96, splits=1, refuse=DP_ERR_UNSUPPORTED, tag="wgrad N % bn != 0"),
    _cv("wgrad", 4, 8, 8, 60, 96, xe=2, splits=1, refuse=DP_ERR_UNSUPPORTED, tag="wgrad ld % 8"),
]


def _gn(op, N, HW, C, G, **kw):
    return dict(op=op, N=N, HW=HW, C=C, G=G, **kw)


# GroupNorm / LayerNorm: the channel map (CT below NT, one to MAXCPT channels per thread above), the pixel chunk and both fold
# thresholds, each float4 condition on its own, the row kernels and their admission
GN = [
    _gn("gn_fwd", 2, 64, 32, 8, tag="C 32"),
    _gn("gn_fwd", 2, 64, 64, 32, silu=1, tag="C 64 SiLU"),
    _gn("gn_fwd", 2, 256, 128, 32, tag="C 128"),
    _gn("gn_fwd", 2, 64, 255, 5, tag="C 255 scalar"),
    _gn("gn_fwd", 2, 64, 256, 32, tag="C 256"),
    _gn("gn_fwd", 2, 64, 257, 1, tag="C 257 scalar"),
    _gn("gn_fwd", 2, 16, 1024, 32, tag="C 1024"),
    _gn("gn_fwd", 2, 16, 1024, 1024, tag="C 1024, G 1024"),
    _gn("gn_fwd", 2, 4096, 128, 32, tag="32 chunks: folded"),
    _gn("gn_fwd", 2, 4224, 128, 32, tag="33 chunks: finalize"),
    _gn("gn_fwd", 1, 8192, 32, 32, xe=1, tag="scalar map, 32 chunks"),
    _gn("gn_fwd", 2, 8448, 32, 8, xe=1, tag="scalar map, 33 chunks"),
    _gn("gn_fwd", 2, 64, 128, 32, px=1, xe=4, tag="x phase: scalar"),
    _gn("gn_fwd", 2, 64, 128, 32, xe=2, tag="x pitch: scalar"),
    _gn("gn_fwd", 2, 64, 128, 32, py=2, ye=4, tag="y phase: scalar"),
    _gn("gn_fwd", 2, 64, 128, 32, ye=1, tag="y pitch: scalar"),
    _gn("gn_bwd", 2, 64, 32, 8, tag="bwd C 32"),
    _gn("gn_bwd", 2, 256, 128, 32, silu=1, tag="bwd C 128 SiLU"),
    _gn("gn_bwd", 2, 64, 255, 5, tag="bwd C 255"),
    _gn("gn_bwd", 2, 64, 257, 1, tag="bwd C 257"),
    _gn("gn_bwd", 2, 16, 1024, 32, tag="bwd C 1024"),
    _gn("gn_bwd", 2, 1024, 128, 32, tag="bwd 8 chunks: folded"),
    _gn("gn_bwd", 2, 1152, 128, 32, fin=True, tag="bwd 9 chunks: reduce, fin form"),
    _gn("gn_bwd", 2, 1152, 128, 32, add=True, add2=True, tag="bwd 9 chunks, addends"),
    _gn("gn_bwd", 2, 64, 128, 32, add=True, alias=True, tag="bwd dx += (addend aliasing dx)"),
    _gn("gn_bwd", 2, 64, 128, 32, add=True, add2=True, padd=1, adde=4, tag="bwd addend phase"),
    _gn("gn_bwd", 2, 64, 128, 32, add=True, add2=True, add2e=2, tag="bwd second addend pitch"),
    _gn("gn_bwd", 300, 1, 1024, 1, add=True, padd=2, adde=4, tag="LN bwd 1024, addend off 16 bytes: GroupNorm kernels"),
    _gn("gn_bwd", 2, 64, 128, 32, px=1, xe=4, tag="bwd x phase"),
    _gn("gn_bwd", 2, 64, 128, 32, dye=1, tag="bwd dy pitch"),
    _gn("gn_bwd", 2, 64, 128, 32, pdx=2, dxe=4, tag="bwd dx phase"),
    # LayerNorm over tokens
    _gn("gn_fwd", 300, 1, 1280, 1, tag="LN 1280: row kernel"),
    _gn("gn_bwd", 300, 1, 1280, 1, tag="LN bwd 1280: row kernel"),
    _gn("gn_fwd", 300, 1, 1028, 1, tag="LN 1028: row kernel"),
    _gn("gn_fwd", 300, 1, 1024, 1, pg=1, tag="LN 1024, gamma off 16 bytes: GroupNorm kernels"),
    _gn("gn_bwd", 300, 1, 1024, 1, pg=1, tag="LN bwd 1024, gamma off 16 bytes: GroupNorm kernels"),
    _gn("gn_fwd", 300, 1, 1022, 1, tag="LN 1022 (C % 4): GroupNorm kernels"),
    _gn("gn_fwd", 65544, 1, 1280, 1, tag="LN beyond 65535 rows: row kernel"),
    # refusals (host validation, nothing launched)
    _gn("gn_fwd", 300, 1, 1281, 1, refuse=DP_ERR_UNSUPPORTED, tag="LN 1281"),
    _gn("gn_fwd", 300, 1, 1280, 1, pg=1, refuse=DP_ERR_UNSUPPORTED, tag="LN 1280, gamma misaligned"),
    _gn("gn_fwd", 300, 1, 1280, 1, pbeta=2, refuse=DP_ERR_UNSUPPORTED, tag="LN 1280, beta misaligned"),
    _gn("gn_fwd", 300, 1, 1280, 1, px=1, xe=4, refuse=DP_ERR_UNSUPPORTED, tag="LN 1280, x misaligned"),
    _gn("gn_fwd", 300, 1, 1280, 1, ye=2, refuse=DP_ERR_UNSUPPORTED, tag="LN 1280, y pitch"),
    _gn("gn_fwd", 300, 1, 1280, 1, no_y=True, refuse=DP_ERR_UNSUPPORTED, tag="LN 1280, bf16 output only"),
    _gn("gn_bwd", 300, 1, 1280, 1, pg=1, refuse=DP_ERR_UNSUPPORTED, tag="LN bwd 1280, gamma misaligned"),
    _gn("gn_bwd", 300, 1, 1280, 1, pdx=1, dxe=4, refuse=DP_ERR_UNSUPPORTED, tag="LN bwd 1280, dx misaligned"),
    _gn("gn_bwd", 300, 1, 1280, 1, add=True, add2=True, padd2=3, add2e=4, refuse=DP_ERR_UNSUPPORTED, tag="LN bwd 1280, second addend misaligned"),
    _gn("gn_fwd", 2, 4, 1280, 32, refuse=DP_ERR_UNSUPPORTED, tag="GroupNorm C 1280"),
    _gn("gn_fwd", 1, 4, 2048, 2048, refuse=DP_ERR_UNSUPPORTED, tag="G 2048 (G <= C: the channel limit refuses it first)"),
    _gn("gn_fwd", 102400, 1, 1022, 1, refuse=DP_ERR_SHAPE, tag="LN 102400 rows, C % 4: off the row kernel"),
    _gn("gn_fwd", 102400, 1, 1024, 1, pg=1, refuse=DP_ERR_SHAPE, tag="LN 102400 rows, gamma misaligned"),
]

# row / pointwise kernels (the census replays at these arguments)
ROWS = [
    ("dp_softmax_fwd", (1, 1)), ("dp_softmax_fwd", (64, 31)), ("dp_softmax_fwd", (64, 32)), ("dp_softmax_fwd", (64, 33)),
    ("dp_softmax_fwd", (16, 4096)), ("dp_softmax_fwd", (16, 4097)),
    ("dp_softmax_bwd", (64, 31)), ("dp_softmax_bwd", (64, 33)), ("dp_softmax_bwd", (16, 4097)),
    # dp_amax: (phase, ld, rows, cols) — dense collapse (ld == cols) vec / scalar, strided vec / scalar
    ("dp_amax", (0, 64, 100, 64)), ("dp_amax", (0, 63, 101, 63)), ("dp_amax", (0, 67, 100, 64)), ("dp_amax", (0, 68, 100, 64)),
    ("dp_amax", (1, 68, 100, 64)), ("dp_amax", (0, 1, 999, 1)),
    # dp_colsum: (phase, ld, rows, cols, seg_rows, acc) — vec / scalar, segments that do not divide the rows
    ("dp_colsum", (0, 64, 256, 64, 64, 0)), ("dp_colsum", (1, 64, 256, 64, 64, 1)), ("dp_colsum", (0, 70, 250, 65, 60, 0)),
    ("dp_colsum", (0, 132, 1000, 129, 1000, 1)),
    # dp_split_h3: (phase, ld, bs, batch, rows, cols, transpose) — float4 loads need x 16-byte aligned with ld and bs multiples of 4; the
    # rows form pads to 8 columns, the transposed form to 8 rows
    ("dp_split_h3", (0, 64, 64 * 50, 3, 50, 64, 0)), ("dp_split_h3", (0, 68, 68 * 50, 3, 50, 65, 0)),
    ("dp_split_h3", (1, 64, 64 * 50, 3, 50, 64, 0)), ("dp_split_h3", (0, 66, 66 * 50, 3, 50, 64, 0)),
    ("dp_split_h3", (0, 64, 64 * 50 + 2, 3, 50, 64, 0)),
    ("dp_split_h3", (0, 72, 72 * 70, 2, 70, 72, 1)), ("dp_split_h3", (0, 45, 45 * 70, 2, 70, 45, 1)),
    ("dp_split_h3", (2, 72, 72 * 65, 2, 65, 72, 1)),
    # dp_transpose_batched: (batch, rows, cols) — float4 when both extents are multiples of 4; 64 x 64 tiles with tails
    ("dp_transpose_batched", (2, 64, 128)), ("dp_transpose_batched", (2, 68, 132)), ("dp_transpose_batched", (2, 70, 45)),
    ("dp_transpose_batched", (3, 65, 64)),
    # dp_gemm_batched: (batch, M, N, Kd, a_cs, b_cs, accumulate) — 128 x 128 x 16 tiles, their tails, the four operand layouts
    ("dp_gemm_batched", (2, 128, 128, 16, 1, 1, 0)), ("dp_gemm_batched", (2, 129, 129, 17, 1, 1, 1)),
    ("dp_gemm_batched", (2, 127, 65, 15, 0, 1, 0)), ("dp_gemm_batched", (2, 65, 127, 33, 1, 0, 1)),
    ("dp_gemm_batched", (3, 257, 100, 64, 0, 0, 0)),
]
