"""Memory footprint of every C-ABI launch kind the plans issue: a captured call (the argument struct, or the scalar arguments as
launch_census.argkinds decodes them) mapped to the exact regions it reads and writes (test_stream_order_host.py checks the region
algebra on the host, test_stream_races_gpu.py checks this table against the kernels on the device).

A region is (ptr, element size, rows, ld, cols): rows of `cols` elements, `ld` elements apart; a flat range is the rows = 1 case.  Two
channel ranges of one concatenated buffer are two regions of the same ld that interleave row by row without sharing a byte.  Modes:
  R   read                      W   written (every byte of the region)
  RW  read and written (+=, accumulate flags, in-place updates)
  A   atomic max into an amax slot (dp_amax semantics): two A accesses of one slot commute, A against any other access does not.
Scratch regions (split-K workspaces, the GroupNorm workspace, reduction partials) are written and read inside one call; their contents
after the call are not an output.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, List, NamedTuple, Optional

import numpy as np

R, W, RW, A = "R", "W", "RW", "A"
WRITES = (W, RW, A)
T_TABLE = 1000          # entries of an alphas_cumprod table: dp_add_noise reads acp[t[b]], t in [0, 1000)


class Region(NamedTuple):
    ptr: int
    esz: int
    rows: int
    ld: int
    cols: int

    @property
    def pitch(self) -> int:
        return self.ld * self.esz

    @property
    def lo(self) -> int:
        return self.ptr

    @property
    def hi(self) -> int:
        """One past the last byte (the bounding range is [lo, hi))."""
        return self.ptr + (self.rows - 1) * self.pitch + self.cols * self.esz

    def intervals(self) -> np.ndarray:
        """[rows, 2] int64 byte intervals [start, end), increasing and disjoint (ld >= cols)."""
        s = self.ptr + np.arange(self.rows, dtype=np.int64) * self.pitch
        return np.stack([s, s + self.cols * self.esz], 1)

    def nbytes(self) -> int:
        return self.rows * self.cols * self.esz


def flat(ptr: int, n: int, esz: int = 4) -> Region:
    return Region(int(ptr), esz, 1, n, n)


def view(ptr: int, rows: int, ld: int, cols: int, esz: int = 4) -> Region:
    if ld == cols or rows == 1:                 # dense: one flat range
        return flat(ptr, rows * cols, esz)
    return Region(int(ptr), esz, int(rows), int(ld), int(cols))


class Access(NamedTuple):
    field: str            # the struct field or argument name
    region: Region
    mode: str
    kind: str = "f32"     # f32 / f16 / bf16 / u8 / i64 / f64 / slot / seed: what the bytes hold (device validation fills by kind)
    scratch: bool = False
    of: str = ""          # amax slots: the field whose operand the slot bounds


# ------------------------------------------------------------------------------------------------------------- region intersection
def _first_same_pitch(a: Region, b: Region):
    """Closed form for two regions of one pitch: rows i of a and i + k of b overlap iff -wb < d + k P < wa (d = b0 - a0)."""
    P, wa, wb, d = a.pitch, a.cols * a.esz, b.cols * b.esz, b.ptr - a.ptr
    # k ranges over the integers with (-wb - d) / P < k < (wa - d) / P; widths <= P leave at most two candidates
    k_lo = (-wb - d) // P + 1
    k_hi = -(-(wa - d) // P) - 1
    best = None
    for k in range(k_lo, k_hi + 1):
        i0, i1 = max(0, -k), min(a.rows, b.rows - k)
        if i0 >= i1:
            continue
        byte = max(a.ptr + i0 * P, b.ptr + (i0 + k) * P)
        cand = (i0, (byte - a.ptr - i0 * P) // a.esz)
        if best is None or cand < best:
            best = cand
    return best


def _first_sweep(a: Region, b: Region):
    """Row-interval sweep for any two regions: for each row interval of a, the first interval of b that ends after it starts."""
    ia, ib = a.intervals(), b.intervals()
    j = np.searchsorted(ib[:, 1], ia[:, 0], side="right")
    ok = j < len(ib)
    jj = np.minimum(j, len(ib) - 1)
    hit = ok & (ib[jj, 0] < ia[:, 1])
    if not hit.any():
        return None
    i = int(np.argmax(hit))
    byte = max(int(ia[i, 0]), int(ib[jj[i], 0]))
    return i, (byte - int(ia[i, 0])) // a.esz


def first_overlap(a: Region, b: Region):
    """(row, element) of a's first byte that b also covers, or None.  Exact: rows interleaving in one wider buffer do not overlap."""
    if a.rows <= 0 or b.rows <= 0 or a.cols <= 0 or b.cols <= 0 or a.hi <= b.lo or b.hi <= a.lo:
        return None
    if a.pitch == b.pitch and a.esz == b.esz and a.rows > 1 and b.rows > 1:
        return _first_same_pitch(a, b)
    return _first_sweep(a, b)


def overlaps(a: Region, b: Region) -> bool:
    return first_overlap(a, b) is not None


def same_region(a: Region, b: Region) -> bool:
    return a == b or (a.nbytes() == b.nbytes() and a.ptr == b.ptr and (a.rows == 1 or b.rows == 1) and
                      ((a.rows == 1 and a.cols * a.esz == b.nbytes() and b.ld == b.cols) or
                       (b.rows == 1 and b.cols * b.esz == a.nbytes() and a.ld == a.cols)))


# ------------------------------------------------------------------------------------------------------------- per-kind footprints
class Ctx:
    """Host queries some footprints need (split-K / GroupNorm workspace sizes, packed weight rows).  Defaults restate the library's rules;
    the GPU test binds the library's own queries."""

    def __init__(self, lib=None):
        self.lib = lib

    def tc_row(self, c: int) -> int:
        return self.lib.dp_tc_weight_row(c) if self.lib else (((c + 63) & ~63) if c > 64 else ((c + 7) & ~7))

    def bf16_row(self, c: int) -> int:
        return self.lib.dp_bf16_weight_row(c) if self.lib else (c + 63) & ~63

    def splitk_floats(self, a, op: int) -> int:
        if self.lib is None:
            return int(getattr(a, "_ws_floats", 0))
        b = type(a)()
        C.memmove(C.byref(b), C.byref(a), C.sizeof(a))
        return int(self.lib.dp_conv_splitk_workspace_floats(C.byref(b), op))

    def gn_ws_bytes(self, a) -> int:
        if self.lib is None:
            return int(getattr(a, "_ws_bytes", 256))
        return int(self.lib.dp_groupnorm_workspace_bytes(a.N, a.HW, a.C, a.G))

    def partials(self, name: str, n: int) -> int:
        per = 4096
        if self.lib is not None:
            return int(getattr(self.lib, name)(n))
        return max(0, -(-n // per))


def _slot(field, ptr, mode, of=""):
    return Access(field, flat(ptr, 1), mode, "slot", of=of)


def _conv(op: str, a, ctx: Ctx) -> List[Access]:
    """dp_conv2d_fprop / dgrad / wgrad (fp32-grade tier, ConvArgs)."""
    acc = a.flags & 1
    x = view(a.x, a.N * a.H * a.W, a.ldx, a.C)
    y = view(a.y, a.N * a.P * a.Q, a.ldy, a.K)
    RS, out = a.R * a.S, []
    if op == "fprop":
        out += [Access("x", x, R), Access("y", y, RW if acc else W)]
        if a.w:
            out.append(Access("w", flat(a.w, RS * a.C * a.K), R))
        if a.w_tc_hi:
            n = RS * a.K * ctx.tc_row(a.C)
            out += [Access("w_tc_hi", flat(a.w_tc_hi, n, 2), R, "f16"), Access("w_tc_lo", flat(a.w_tc_lo, n, 2), R, "f16")]
        if a.bias:
            out.append(Access("bias", flat(a.bias, a.K), R))
        if a.rowadd:
            out.append(Access("rowadd", view(a.rowadd, a.N, a.ld_rowadd, a.K), R))
        if a.residual:
            out.append(Access("residual", view(a.residual, a.N * a.P * a.Q, a.ld_res, a.K), R))
    elif op == "dgrad":
        out += [Access("y", y, R), Access("x", x, RW if acc else W)]
        if a.w:
            out.append(Access("w", flat(a.w, RS * a.C * a.K), R))
        if a.w_tc_hi:
            n = RS * a.C * ctx.tc_row(a.K)
            out += [Access("w_tc_hi", flat(a.w_tc_hi, n, 2), R, "f16"), Access("w_tc_lo", flat(a.w_tc_lo, n, 2), R, "f16")]
    else:   # wgrad: split-K partials of dW (and of the bias gradient) into caller-owned workspaces
        out += [Access("x", x, R), Access("y", y, R),
                Access("workspace", flat(a.workspace, a.splits * a.K * RS * a.C), W)]
        if a.bias_ws:
            out.append(Access("bias_ws", flat(a.bias_ws, a.splits * a.K), W))
    if op != "wgrad" and a.workspace:
        n = ctx.splitk_floats(a, 0 if op == "fprop" else 1)
        if n > 0:
            out.append(Access("workspace", flat(a.workspace, n), W, scratch=True))
    for f, of in (("amax_x", "x"), ("amax_y", "y"), ("amax_w", "w_tc_hi")):
        if getattr(a, f):
            out.append(_slot(f, getattr(a, f), R, of))
    if a.amax_out:
        out.append(_slot("amax_out", a.amax_out, A, "y" if op == "fprop" else "x"))
    return out


def _conv_bf16(op: str, a, ctx: Ctx) -> List[Access]:
    acc = a.flags & 1
    RS, out = a.R * a.S, []
    if op == "fprop":
        out += [Access("x_bf16", view(a.x_bf16, a.N * a.H * a.W, a.ldx, a.C, 2), R, "bf16"),
                Access("w_bf16", flat(a.w_bf16, RS * a.K * ctx.bf16_row(a.C), 2), R, "bf16"),
                Access("out", view(a.out, a.N * a.P * a.Q, a.ld_out, a.K), RW if acc else W)]
        if a.bias:
            out.append(Access("bias", flat(a.bias, a.K), R))
        if a.rowadd:
            out.append(Access("rowadd", view(a.rowadd, a.N, a.ld_rowadd, a.K), R))
        if a.residual:
            out.append(Access("residual", view(a.residual, a.N * a.P * a.Q, a.ld_res, a.K), R))
    elif op == "dgrad":
        out += [Access("dy_bf16", view(a.dy_bf16, a.N * a.P * a.Q, a.lddy, a.K, 2), R, "bf16"),
                Access("w_bf16", flat(a.w_bf16, RS * a.C * ctx.bf16_row(a.K), 2), R, "bf16"),
                Access("out", view(a.out, a.N * a.H * a.W, a.ld_out, a.C), RW if acc else W)]
    else:
        out += [Access("x_bf16", view(a.x_bf16, a.N * a.H * a.W, a.ldx, a.C, 2), R, "bf16"),
                Access("dy_bf16", view(a.dy_bf16, a.N * a.P * a.Q, a.lddy, a.K, 2), R, "bf16"),
                Access("workspace", flat(a.workspace, a.splits * a.K * RS * a.C), W)]
    return out


def _reduce(a, ctx: Ctx) -> List[Access]:
    RS = a.R * a.S
    n = a.K * a.C * RS
    scores = bool(a.w and (a.score_out or a.score_in))
    out = [Access("workspace", flat(a.workspace, a.splits * n), R), Access("dw", flat(a.dw, n), RW)]
    if scores:    # the signed W*dW terms of this pass are parked in the consumed split-0 slab
        out[0] = Access("workspace", flat(a.workspace + 4 * n, (a.splits - 1) * n), R) if a.splits > 1 else None
        out = [o for o in out if o is not None]
        out += [Access("workspace", flat(a.workspace, n), RW), Access("w", flat(a.w, n), R)]
        if a.score_out:
            out.append(Access("score_out", flat(a.score_out, a.K), RW))
        if a.score_in:
            out.append(Access("score_in", flat(a.score_in, a.C), RW))
    if a.bias_ws:
        out += [Access("bias_ws", flat(a.bias_ws, a.splits * a.K), R), Access("db", flat(a.db, a.K), RW)]
    return out


def _al16(p, ld) -> bool:
    return not p or (int(p) % 16 == 0 and ld % 4 == 0)


def _ln_rows(op: str, a) -> bool:
    """Does the call take norm.cu's LayerNorm row kernels (no GroupNorm workspace in the forward, none in a backward without dgamma /
    dbeta)?  norm.cu's ln_fast() and the alignment tests of dp_groupnorm_fwd / dp_groupnorm_bwd that guard them."""
    ln = a.HW == 1 and a.G == 1 and a.C % 4 == 0 and a.C <= 4 * 32 * 8 and not a.silu and a.dropout_p == 0 and not a.y_bf16
    if op == "fwd":
        return (ln and bool(a.y) and _al16(a.x, a.ldx) and _al16(a.y, a.ldy) and _al16(a.gamma, 0) and _al16(a.beta, 0))
    return (ln and _al16(a.x, a.ldx) and _al16(a.dy, a.lddy) and _al16(a.dx, a.lddx) and _al16(a.dx_add, a.ldadd) and
            _al16(a.dx_add2, a.ldadd2) and _al16(a.gamma, 0))


def _gn(op: str, a, ctx: Ctx) -> List[Access]:
    rows = a.N * a.HW
    out = []
    if op == "param":       # dgamma / dbeta += the per-image channel sums a dp_groupnorm_bwd call left in fin
        if not (a.dgamma or a.dbeta):
            return []
        out.append(Access("fin", flat(a.fin, 2 * a.N * a.C), R))
        for f in ("dgamma", "dbeta"):
            if getattr(a, f):
                out.append(Access(f, flat(getattr(a, f), a.C), RW))
        return out
    out += [Access("x", view(a.x, rows, a.ldx, a.C), R), Access("gamma", flat(a.gamma, a.C), R),
            Access("beta", flat(a.beta, a.C), R)]
    if a.dropout_p > 0 and a.dropout_seed_dev:
        out.append(Access("dropout_seed_dev", flat(a.dropout_seed_dev, 1, 8), R, "seed"))
    mean, rstd = flat(a.mean, a.N * a.G), flat(a.rstd, a.N * a.G)
    ln = _ln_rows(op, a)
    if op == "fwd":
        out += [Access("mean", mean, W), Access("rstd", rstd, W)]
        if a.y:
            out.append(Access("y", view(a.y, rows, a.ldy, a.C), W))
        if a.y_bf16:
            out.append(Access("y_bf16", view(a.y_bf16, rows, a.ldyb, a.C, 2), W, "bf16"))
        if a.amax_y:
            out.append(_slot("amax_y", a.amax_y, A, "y"))
        if not ln:
            out.append(Access("workspace", flat(a.workspace, ctx.gn_ws_bytes(a) // 4), W, scratch=True))
        return out
    out += [Access("mean", mean, R), Access("rstd", rstd, R), Access("dy", view(a.dy, rows, a.lddy, a.C), R)]
    dx = view(a.dx, rows, a.lddx, a.C)
    add = view(a.dx_add, rows, a.ldadd, a.C) if a.dx_add else None
    out.append(Access("dx", dx, RW if (add is not None and add == dx) else W))
    if add is not None and add != dx:
        out.append(Access("dx_add", add, R))
    if a.dx_add2:
        out.append(Access("dx_add2", view(a.dx_add2, rows, a.ldadd2, a.C), R))
    if a.amax_dx:
        out.append(_slot("amax_dx", a.amax_dx, A, "dx"))
    if a.fin:
        out.append(Access("fin", flat(a.fin, 2 * a.N * a.C), W))
    elif a.dgamma or a.dbeta:
        for f in ("dgamma", "dbeta"):
            if getattr(a, f):
                out.append(Access(f, flat(getattr(a, f), a.C), RW))
    if ln and not (a.dgamma or a.dbeta):
        return out
    out.append(Access("workspace", flat(a.workspace, ctx.gn_ws_bytes(a) // 4), W, scratch=True))
    return out


def _gemm_operand(ptr, batch, rows_, cols_, rs, cs, bs, esz=4):
    """Regions of a batched strided [rows][cols] operand (one of rs / cs is 1): one region when the batches stack row-contiguously."""
    if cs == 1:
        r, ld, c = rows_, rs, cols_
    else:
        r, ld, c = cols_, cs, rows_
    if batch == 1 or bs == r * ld:
        return [view(ptr, batch * r, ld, c, esz)]
    return [view(ptr + b * bs * esz, r, ld, c, esz) for b in range(batch)]


def _gemm(a, ctx) -> List[Access]:
    out = [Access("A", g, R) for g in _gemm_operand(a.A, a.batch, a.M, a.Kd, a.a_rs, a.a_cs, a.a_bs)]
    out += [Access("B", g, R) for g in _gemm_operand(a.B, a.batch, a.Kd, a.N, a.b_rs, a.b_cs, a.b_bs)]
    out += [Access("C", g, RW if a.accumulate else W) for g in _gemm_operand(a.C, a.batch, a.M, a.N, a.ldc, 1, a.c_bs)]
    return out


def _gemm_nt(a, ctx) -> List[Access]:
    rows, kg8 = a.batch * a.H * a.W, (a.Kg + 7) & ~7
    out = [Access("A", view(a.A, rows, a.ld_a, a.Kg), R),
           # B's tensor map spans the padded row (kg8 = dp_split_h3's zero-filled pitch, conv_tc.cu:686-688): the pads are read
           Access("b_hi", flat(a.b_hi, a.batch * a.N * kg8, 2), R, "f16"),
           Access("b_lo", flat(a.b_lo, a.batch * a.N * kg8, 2), R, "f16"),
           Access("C", view(a.C, rows, a.ldc, a.N), W),
           _slot("amax_a", a.amax_a, R, "A"), _slot("amax_b", a.amax_b, R, "B")]
    if a.amax_out:
        out.append(_slot("amax_out", a.amax_out, A, "C"))
    return out


def _adam(a, ctx) -> List[Access]:
    n = a.n
    out = [Access("p", flat(a.p, n), RW), Access("g", flat(a.g, n), R), Access("m", flat(a.m, n), RW), Access("v", flat(a.v, n), RW)]
    if a.ema:
        out.append(Access("ema", flat(a.ema, n), RW))
    if a.sumsq:
        out.append(Access("sumsq", flat(a.sumsq, 1), R))
    if a.step_scalars:
        out.append(Access("step_scalars", flat(a.step_scalars, 2), R))
    return out


def _taylor(a, ctx) -> List[Access]:
    n = a.O * a.I * a.RS
    out = [Access("w", flat(a.w, n), R), Access("dw", flat(a.dw, n), R)]
    for f in ("out_signed", "out_abs", "out_sq"):
        if getattr(a, f):
            out.append(Access(f, flat(getattr(a, f), a.O), W))
    for f in ("in_signed", "in_abs", "in_sq"):
        if getattr(a, f):
            out.append(Access(f, flat(getattr(a, f), a.I), W))
    return out


def _ssim(a, ctx) -> List[Access]:
    n = a.N * a.C * a.H * a.W
    esz, kind = (1, "u8") if a.format == 0 else (4, "f32")
    return [Access("x", flat(a.x, n, esz), R, kind), Access("y", flat(a.y, n, esz), R, kind),
            Access("ssim_nc", flat(a.ssim_nc, a.N * a.C, 8), W, "f64"), Access("sse_n", flat(a.sse_n, a.N, 8), W, "f64")]


def _moments_sxx(ptr, D):
    return [Access("sxx", Region(int(ptr) + 8 * (i * D + i), 8, 1, D - i, D - i), RW, "f64") for i in range(D)]


# scalar-argument kinds: args are the call's arguments without the stream, in header order
def _s(name: str, args, ctx: Ctx) -> List[Access]:
    g = args
    if name == "dp_pack_conv_weight":
        w, K, Cc, Rr, S, ck, kc = g
        n = K * Cc * Rr * S
        return [Access("w", flat(w, n), R)] + [Access(f, flat(p, n), W) for f, p in (("w_ck", ck), ("w_kc", kc)) if p]
    if name == "dp_pack_conv_weight_tc":
        w, K, Cc, Rr, S, kch, kcl, ckh, ckl, amax = g
        RS = Rr * S
        out = [Access("w", flat(w, K * Cc * RS), R), Access("amax_w", flat(amax, 1), RW, "slot", of="w")]
        if kch:
            n = RS * K * ctx.tc_row(Cc)
            out += [Access("kc_hi", flat(kch, n, 2), W, "f16"), Access("kc_lo", flat(kcl, n, 2), W, "f16")]
        if ckh:
            n = RS * Cc * ctx.tc_row(K)
            out += [Access("ck_hi", flat(ckh, n, 2), W, "f16"), Access("ck_lo", flat(ckl, n, 2), W, "f16")]
        return out
    if name == "dp_pack_conv_weight_bf16":
        w, K, Cc, Rr, S, kc, ck = g
        RS = Rr * S
        out = [Access("w", flat(w, K * Cc * RS), R)]
        if kc:
            out.append(Access("kc", flat(kc, RS * K * ctx.bf16_row(Cc), 2), W, "bf16"))
        if ck:
            out.append(Access("ck", flat(ck, RS * Cc * ctx.bf16_row(K), 2), W, "bf16"))
        return out
    if name == "dp_amax":
        x, ld, rows, cols, slot = g
        return [Access("x", view(x, rows, ld, cols), R), _slot("slot", slot, A, "x")]
    if name == "dp_zero_u32":
        p, n = g
        return [Access("p", flat(p, n), W, "slot")]
    if name == "dp_cvt_bf16":
        src, ld, rows, Cc, dst, ldd = g
        return [Access("src", view(src, rows, ld, Cc), R), Access("dst", view(dst, rows, ldd, ldd, 2), W, "bf16")]
    if name == "dp_split_h3":
        x, ld, bs, batch, rows, cols, tr, amax, hi, lo = g
        if batch == 1 or bs == rows * ld:
            src = [view(x, batch * rows, ld, cols)]
        else:
            src = [view(x + 4 * b * bs, rows, ld, cols) for b in range(batch)]
        n = batch * (cols * ((rows + 7) & ~7) if tr else rows * ((cols + 7) & ~7))
        return [Access("x", r, R) for r in src] + [Access("amax", flat(amax, 1), R, "slot", of="x"),
                                                    Access("hi", flat(hi, n, 2), W, "f16"), Access("lo", flat(lo, n, 2), W, "f16")]
    if name == "dp_transpose_batched":
        i, o, batch, rows, cols = g
        n = batch * rows * cols
        return [Access("in", flat(i, n), R), Access("out", flat(o, n), W)]
    if name == "dp_softmax_fwd":
        s, p, rows, cols = g
        return [Access("s", flat(s, rows * cols), R), Access("p", flat(p, rows * cols), W)]
    if name == "dp_softmax_bwd":
        p, dp, ds, rows, cols, amax = g
        out = [Access("p", flat(p, rows * cols), R), Access("dp", flat(dp, rows * cols), R), Access("ds", flat(ds, rows * cols), W)]
        return out + ([_slot("amax_ds", amax, A, "ds")] if amax else [])
    if name == "dp_silu_fwd":
        x, y, n = g
        return [Access("x", flat(x, n), R), Access("y", flat(y, n), W)]
    if name == "dp_silu_bwd":
        x, dy, dx, n, acc = g
        return [Access("x", flat(x, n), R), Access("dy", flat(dy, n), R), Access("dx", flat(dx, n), RW if acc else W)]
    if name == "dp_geglu_fwd":
        u, ldu, o, ldo, rows, I = g
        return [Access("u", view(u, rows, ldu, 2 * I), R), Access("out", view(o, rows, ldo, I), W)]
    if name == "dp_geglu_bwd":
        u, ldu, do, lddo, du, lddu, rows, I = g
        return [Access("u", view(u, rows, ldu, 2 * I), R), Access("dout", view(do, rows, lddo, I), R),
                Access("du", view(du, rows, lddu, 2 * I), W)]
    if name == "dp_timestep_embedding":
        t, fr, o, B, half, flip = g
        return [Access("t", flat(t, B, 8), R, "i64"), Access("freqs", flat(fr, half), R), Access("out", flat(o, 2 * B * half), W)]
    if name == "dp_add_noise":
        x0, nz, t, acp, o, B, Cc, H, Wd, nhwc, ld = g
        n = B * Cc * H * Wd
        out = [Access("x0", flat(x0, n), R), Access("noise", flat(nz, n), R), Access("t", flat(t, B, 8), R, "i64"),
               Access("acp", flat(acp, T_TABLE), R, "acp")]
        return out + [Access("out", view(o, B * H * Wd, ld or Cc, Cc) if nhwc else flat(o, n), W)]
    if name == "dp_nchw_to_nhwc":
        i, o, ld, N, Cc, H, Wd = g
        return [Access("in", flat(i, N * Cc * H * Wd), R), Access("out", view(o, N * H * Wd, ld, Cc), W)]
    if name == "dp_nhwc_to_nchw":
        i, ld, o, N, Cc, H, Wd, acc = g
        return [Access("in", view(i, N * H * Wd, ld, Cc), R), Access("out", flat(o, N * Cc * H * Wd), RW if acc else W)]
    if name == "dp_mse_loss_grad":
        pred, tgt, grad, n, sl, sg, part, loss = g
        out = [Access("pred", flat(pred, n), R), Access("target", flat(tgt, n), R),
               Access("partial", flat(part, ctx.partials("dp_mse_partials", n)), W, scratch=True), Access("loss_out", flat(loss, 1), W)]
        return out + ([Access("grad", flat(grad, n), W)] if grad else [])
    if name == "dp_upsample2x_fwd":
        x, ldx, y, ldy, N, H, Wd, Cc = g
        return [Access("x", view(x, N * H * Wd, ldx, Cc), R), Access("y", view(y, 4 * N * H * Wd, ldy, Cc), W)]
    if name == "dp_upsample2x_bwd":
        dy, lddy, dx, lddx, N, H, Wd, Cc, acc = g
        return [Access("dy", view(dy, 4 * N * H * Wd, lddy, Cc), R), Access("dx", view(dx, N * H * Wd, lddx, Cc), RW if acc else W)]
    if name == "dp_colsum":
        x, ld, rows, cols, seg, o, ldo, acc = g
        nseg = -(-rows // seg)
        return [Access("x", view(x, rows, ld, cols), R), Access("out", view(o, nseg, ldo, cols), RW if acc else W)]
    if name == "dp_add_views":
        a_, lda, b_, ldb, y, ldy, rows, cols = g
        return [Access("a", view(a_, rows, lda, cols), R), Access("b", view(b_, rows, ldb, cols), R),
                Access("y", view(y, rows, ldy, cols), W)]
    if name == "dp_copy_rows":
        a_, lda, y, ldy, rows, cols = g
        return [Access("a", view(a_, rows, lda, cols), R), Access("y", view(y, rows, ldy, cols), W)]
    if name == "dp_sumsq":
        x, n, part, o = g
        return [Access("x", flat(x, n), R), Access("partial", flat(part, ctx.partials("dp_sumsq_partials", n)), W, scratch=True),
                Access("out", flat(o, 1), W)]
    if name == "dp_ddim_step":
        x, e, nz, o, n, sb, sa, clip, sap, dirc, sigma = g
        out = [Access("x", flat(x, n), R), Access("eps", flat(e, n), R)]
        if sigma != 0 and nz:
            out.append(Access("noise", flat(nz, n), R))
        return out + [Access("out", flat(o, n), W)]
    if name == "dp_ddim_cfg_step":
        e, lde, x, nz, xo, xi, ldi, px0, B, Cc, H, Wd, guided, scale, sb, sa, sap, dirc, sigma = g
        n, rows = B * Cc * H * Wd, (2 if guided else 1) * B * H * Wd
        out = [Access("eps", view(e, rows, lde, Cc), R), Access("x", flat(x, n), R)]
        if sigma != 0 and nz:
            out.append(Access("noise", flat(nz, n), R))
        out += [Access("x_out", flat(xo, n), W), Access("x_in", view(xi, rows, ldi, Cc), W)]
        return out + ([Access("pred_x0", flat(px0, n), W)] if px0 else [])
    if name == "dp_scale":
        x, n, s = g
        return [Access("x", flat(x, n), RW)]
    if name == "dp_fid_input":
        src, u8, q, N, Hs, Ws, o, ldo, Ho, Wo, resize, norm, amax = g
        out = [Access("src", flat(src, N * Hs * Ws * 3, 1 if u8 else 4), R, "u8" if u8 else "f32"),
               Access("out", view(o, N * Ho * Wo, ldo, 3), W)]
        return out + ([_slot("amax_out", amax, A, "out")] if amax else [])
    if name == "dp_pool3x3":
        x, ldx, y, ldy, N, H, Wd, Cc, stride, pad, mode, amax = g
        P, Q = (H + 2 * pad - 3) // stride + 1, (Wd + 2 * pad - 3) // stride + 1
        out = [Access("x", view(x, N * H * Wd, ldx, Cc), R), Access("y", view(y, N * P * Q, ldy, Cc), W)]
        return out + ([_slot("amax_out", amax, A, "y")] if amax else [])
    if name == "dp_global_mean":
        x, ldx, y, ldy, N, H, Wd, Cc = g
        return [Access("x", view(x, N * H * Wd, ldx, Cc), R), Access("y", view(y, N, ldy, Cc), W)]
    if name == "dp_feature_moments":
        f, ld, rows, D, shift, s, sxx = g
        out = [Access("f", view(f, rows, ld, D), R), Access("sum", flat(s, D, 8), RW, "f64")] + _moments_sxx(sxx, D)
        return out + ([Access("shift", flat(shift, D), R)] if shift else [])
    if name == "dp_vq_quantize":
        z, N, D, H, Wd, inv, cb, ne, quant, o, ldo, idx = g
        out = [Access("z", flat(z, N * D * H * Wd), R), Access("out", view(o, N * H * Wd, ldo, D), W)]
        if quant:
            out.append(Access("codebook", flat(cb, ne * D), R))
            if idx:
                out.append(Access("indices", flat(idx, N * H * Wd, 8), W, "i64"))
        return out
    if name == "dp_decode_images":
        y, ld, N, Cc, H, Wd, u8, f32 = g
        out = [Access("y", view(y, N * H * Wd, ld, Cc), R)]
        if u8:
            out.append(Access("u8_nhwc", flat(u8, N * H * Wd * Cc, 1), W, "u8"))
        if f32:
            out.append(Access("f32_nchw", flat(f32, N * Cc * H * Wd), W))
        return out
    raise KeyError(name)


STRUCT_KINDS: Dict[str, Callable] = {
    "dp_conv2d_fprop": lambda a, c: _conv("fprop", a, c), "dp_conv2d_dgrad": lambda a, c: _conv("dgrad", a, c),
    "dp_conv2d_wgrad": lambda a, c: _conv("wgrad", a, c), "dp_conv2d_wgrad_reduce": _reduce,
    "dp_conv2d_fprop_bf16": lambda a, c: _conv_bf16("fprop", a, c), "dp_conv2d_dgrad_bf16": lambda a, c: _conv_bf16("dgrad", a, c),
    "dp_conv2d_wgrad_bf16": lambda a, c: _conv_bf16("wgrad", a, c),
    "dp_groupnorm_fwd": lambda a, c: _gn("fwd", a, c), "dp_groupnorm_bwd": lambda a, c: _gn("bwd", a, c),
    "dp_groupnorm_bwd_param": lambda a, c: _gn("param", a, c),
    "dp_gemm_batched": _gemm, "dp_gemm_nt_tc": _gemm_nt, "dp_adam_clip_ema": _adam, "dp_taylor_reduce": _taylor, "dp_ssim": _ssim,
}
SCALAR_KINDS = ("dp_pack_conv_weight", "dp_pack_conv_weight_tc", "dp_pack_conv_weight_bf16", "dp_amax", "dp_zero_u32", "dp_cvt_bf16",
                "dp_split_h3", "dp_transpose_batched", "dp_softmax_fwd", "dp_softmax_bwd", "dp_silu_fwd", "dp_silu_bwd", "dp_geglu_fwd",
                "dp_geglu_bwd", "dp_timestep_embedding", "dp_add_noise", "dp_nchw_to_nhwc", "dp_nhwc_to_nchw", "dp_mse_loss_grad",
                "dp_upsample2x_fwd", "dp_upsample2x_bwd", "dp_colsum", "dp_add_views", "dp_copy_rows", "dp_sumsq", "dp_ddim_step",
                "dp_ddim_cfg_step", "dp_scale", "dp_fid_input", "dp_pool3x3", "dp_global_mean", "dp_feature_moments",
                "dp_vq_quantize", "dp_decode_images")
KINDS = tuple(STRUCT_KINDS) + SCALAR_KINDS


def footprint(name: str, args, ctx: Optional[Ctx] = None) -> List[Access]:
    """The accesses of one captured call: args as launch_census captures them (a one-element list holding the struct copy, or the
    scalar arguments without the stream)."""
    ctx = ctx or Ctx()
    if name in STRUCT_KINDS:
        a = args[0] if isinstance(args, (list, tuple)) else args
        return [x for x in STRUCT_KINDS[name](a, ctx) if x.region.rows > 0 and x.region.cols > 0]
    return [x for x in _s(name, [0 if v is None else v for v in args], ctx) if x.region.ptr and x.region.rows > 0 and x.region.cols > 0]


# --------------------------------------------------------------------------------------------------------- in-place allowlist
# (kind, written field, read field): the same region exactly, every element read and then written by one thread, through coherent loads
# (an operand read through __ldg / ld.global.nc gets no allowance: the non-coherent path may serve a line another thread rewrote).
IN_PLACE = {
    ("dp_softmax_fwd", "p", "s"): "pointwise.cu softmax_fwd_kernel: no operand is __restrict__ (every load is LDG.E, none .CONSTANT); "
                                  "lane j reads in[j] and then writes out[j] of its own row",
    ("dp_softmax_bwd", "ds", "dp"): "pointwise.cu softmax_bwd_kernel: no operand is __restrict__ (every load is LDG.E, none .CONSTANT); "
                                    "lane j reads dr[j] in both passes, then writes o[j]",
    ("dp_groupnorm_bwd", "dx", "dx_add"): "norm.cu:578 gn_bwd_apply4 (and gn_bwd_apply): dx_add is loaded through a plain pointer of the "
                                          "by-value argument struct by the thread that then writes that element of dx (dx_add2 and dy "
                                          "go through ld4 = __ldg and get no allowance)",
}


def aliasing(name: str, accs: List[Access]):
    """Intra-launch hazards: an R region of one operand overlapping a W / RW region of another, outside the allowlist.  Returns
    [(read field, written field, (row, element))]."""
    bad = []
    for r in accs:
        if r.mode != R:
            continue
        for w in accs:
            if w.mode not in (W, RW) or w.field == r.field:
                continue
            hit = first_overlap(r.region, w.region)
            if hit is None:
                continue
            if (name, w.field, r.field) in IN_PLACE and same_region(r.region, w.region):
                continue
            bad.append((r.field, w.field, hit))
    return bad
