"""Dispatch-edge sweep: every case of dispatch_edges.py at its own shape and view layout, on both sides of each host-side threshold of
the kernels, checked element by element against fp64 on the device with the census's replays (test_launch_census_gpu.py: per-channel
scales 2^U(-6, 6) on one operand, sentinels around every written view, a second run bit-identical, amax_out == max|written|) and
with a witness of the path it took: the kernels torch.profiler records, the launches dp_launch_count counts, and the split-K
workspace the library asks for, all predicted from the device's own SM count by the restatements in dispatch_edges.py.  Cases the host
code refuses must return their exact code and launch nothing."""
import ctypes as C
import re
import zlib

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import dispatch_edges as de
import launch_census as lc
from test_launch_census_gpu import REPLAY, S, _check, _randn, _twice, replay_conv, lib  # noqa: F401  (lib: the module-scoped fixture)

pytestmark = pytest.mark.gpu

BASE = 1 << 20          # fake pointers of the argument structs: the replays take only NULL-or-not and the 16-byte phase from them
_REPORT = {}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ptr(phase=0, esz=4):
    return BASE + phase * esz


def _kernel(name):
    """Bare kernel name from a profiler event: `void (anonymous namespace)::conv_tc_ps_kernel<false>(...)` -> conv_tc_ps_kernel<false>."""
    name = name.replace("(anonymous namespace)::", "")
    m = re.match(r"(?:void\s+)?(?:[\w:]*::)?(\w+(?:<[^()]*>)?)\(", name)
    return m.group(1) if m else name


class Witness:
    """Kernels the block ran (torch.profiler, CUDA activity only) and dp_launch_count per call of the entry points named."""

    def __init__(self, lib, *entries):
        self.lib, self.entries, self.deltas, self.orig = lib, entries, [], {}

    def __enter__(self):
        for e in self.entries:
            fn = self.orig[e] = getattr(self.lib, e)

            def wrapped(*a, fn=fn):
                n0 = self.lib.dp_launch_count()
                rc = fn(*a)
                self.deltas.append((rc, self.lib.dp_launch_count() - n0))
                return rc
            setattr(self.lib, e, wrapped)
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        for e, fn in self.orig.items():
            setattr(self.lib, e, fn)
        self.kernels = {}
        for ev in self.prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = _kernel(ev.name)
                self.kernels[k] = self.kernels.get(k, 0) + 1
        return False

    def count(self, *names):
        return sum(v for k, v in self.kernels.items() if any(k == n or k.startswith(n + "<") for n in names))


def _report(entry, rep):
    for k, v in rep.items():
        _REPORT[k] = max(_REPORT.get(k, 0.0), max(v))


# ---------------------------------------------------------------------------------------------------------------- fp32-grade convolutions
def _conv_args(c):
    from diff_pruning_b200 import _lib as L
    a = L.ConvArgs()
    P, Q = de.out_extent(c)
    R, Sx = c["R"], c.get("S", c["R"])
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S = c["N"], c["H"], c["W"], c["C"], P, Q, c["K"], R, Sx
    a.stride, a.pad_t, a.pad_l = c.get("stride", 1), c.get("pad", (R - 1) // 2), c.get("pad_l", c.get("pad", (Sx - 1) // 2))
    a.flags, a.splits = c.get("flags", 0), c.get("splits", 1)
    a.ldx, a.ldy = c["C"] + c.get("xe", 0), c["K"] + c.get("ye", 0)
    a.x, a.y, a.w = _ptr(c.get("px", 0)), _ptr(c.get("py", 0)), _ptr()
    a.w_tc_hi = a.w_tc_lo = a.amax_w = a.amax_x = a.amax_y = _ptr()
    a.workspace = _ptr() if c.get("ws", True) else None
    if c.get("bias"):
        a.bias = _ptr(c.get("pb", 0))
    if c.get("rowadd"):
        a.rowadd, a.ld_rowadd = _ptr(c.get("pr", 0)), c["K"] + c.get("re", 0)
    if c.get("residual"):
        a.residual, a.ld_res = _ptr(c.get("ps", 0)), c["K"] + c.get("se", 0)
    if c["op"] == "wgrad":
        a.bias_ws = _ptr()
    return a


@pytest.mark.parametrize("c", de.CONV, ids=[c["tag"] for c in de.CONV])
def test_conv_edges(lib, c):
    g = torch.Generator().manual_seed(zlib.crc32(c["tag"].encode()))
    sms = _sms()
    c = de.at_sms(c, sms)
    want = de.conv_path(c, sms)
    a = _conv_args(c)
    op = c["op"]
    entry = {"fprop": "dp_conv2d_fprop", "dgrad": "dp_conv2d_dgrad", "wgrad": "dp_conv2d_wgrad"}[op]
    rep = {}
    seen = {}

    def chain(args, need):
        seen["need"] = need
        return want["L"], want["kernel"] != "simt"
    with Witness(lib, entry) as w:
        if op == "wgrad":
            REPLAY[entry](lib, g, entry, a, rep)
        else:
            ws = replay_conv(lib, g, entry, a, rep, chain=chain)
    runs = 2
    assert all(rc == 0 for rc, _ in w.deltas) and len(w.deltas) == runs, w.deltas
    if op == "wgrad":
        tc = want["kernel"] == "wgrad_tc"
        assert w.count("wgrad_tc_kernel") == (runs if tc else 0), (w.kernels, want)
        assert w.count("gemm_simt_kernel") == (0 if tc else runs), (w.kernels, want)
        assert all(d == (1 if tc else 2) for _, d in w.deltas), w.deltas
    else:
        gem = want["gemms"]
        if want["kernel"] == "simt":
            names = {"gemm_simt_kernel": runs}
        else:
            tk = "conv_tc_ps_kernel<true>" if want["kernel"] == "any" else "conv_tc_ps_kernel<false>"
            ep = "splitk_flat_epilogue_kernel" if want["kernel"] == "any" else "splitk_epilogue_kernel"
            names = {tk: runs * len(gem), ep: runs * sum(1 for gg in gem if gg[0] > 1)}
            assert seen["need"] == want["ws_floats"], (seen["need"], want)
        # the NaN-filled split-K workspace: the split launches wrote their partial sums through it, every other launch left it alone
        if ws is not None:
            assert bool(torch.isnan(ws).all()) == (names.get(ep, 0) == 0 if want["kernel"] != "simt" else True), (want, c["tag"])
        for k in ("gemm_simt_kernel", "conv_tc_ps_kernel<true>", "conv_tc_ps_kernel<false>", "splitk_epilogue_kernel",
                  "splitk_flat_epilogue_kernel"):
            assert w.count(k) == names.get(k, 0), (k, w.kernels, want)
        per_call = 1 if want["kernel"] == "simt" else len(gem) + sum(1 for gg in gem if gg[0] > 1)
        assert all(d == per_call for _, d in w.deltas), (w.deltas, want)
    _report(entry, rep)


# ---------------------------------------------------------------------------------------------------------------- bf16 tier
def _bf16_args(c):
    from diff_pruning_b200 import _lib as L
    a = L.ConvBf16Args()
    P, Q = de.out_extent(c)
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S = c["N"], c["H"], c["W"], c["C"], P, Q, c["K"], c["R"], c["R"]
    a.stride, a.pad_t = c.get("stride", 1), c.get("pad", (c["R"] - 1) // 2)
    a.pad_l, a.flags, a.splits = a.pad_t, c.get("flags", 0), c.get("splits", 1)
    a.ldx, a.lddy = c["C"] + c.get("xe", 0), c["K"] + c.get("ye", 0)
    a.ld_out = a.lddy if c["op"] == "fprop" else a.ldx
    a.x_bf16 = a.dy_bf16 = a.w_bf16 = a.out = a.workspace = _ptr()
    if c.get("bias"):
        a.bias = _ptr()
    if c.get("residual"):
        a.residual, a.ld_res = _ptr(), c["K"]
    return a


@pytest.mark.parametrize("c", de.BF16, ids=[c["tag"] for c in de.BF16])
def test_bf16_edges(lib, c):
    g = torch.Generator().manual_seed(zlib.crc32(c["tag"].encode()))
    a = _bf16_args(c)
    op = {"fprop": 0, "dgrad": 1, "wgrad": 2}[c["op"]]
    ok, tile, _ = de.bf16_plan(c)
    rc = lib.dp_conv_bf16_eligible(C.byref(a), op)
    assert rc == (0 if ok else c["refuse"]), (rc, c)
    entry = {"fprop": "dp_conv2d_fprop_bf16", "dgrad": "dp_conv2d_dgrad_bf16", "wgrad": "dp_conv2d_wgrad_bf16"}[c["op"]]
    if not ok:
        # refused in host planning before anything is encoded or launched; real buffers sized for the views, so that a regression which
        # launched one of these shapes would at least not read or write global memory outside them
        P, Q = de.out_extent(c)
        x = torch.zeros(c["N"] * c["H"] * c["W"] * a.ldx + 8, dtype=torch.bfloat16, device="cuda")
        dy = torch.zeros(c["N"] * P * Q * a.lddy + 8, dtype=torch.bfloat16, device="cuda")
        out = torch.zeros(max(x.numel(), dy.numel(), a.splits * c["K"] * c["C"] * 9), device="cuda")
        wt = torch.zeros(9 * lib.dp_bf16_weight_row(max(c["C"], c["K"])) * max(c["C"], c["K"]), dtype=torch.bfloat16, device="cuda")
        a.x_bf16, a.dy_bf16, a.out, a.workspace, a.w_bf16 = x.data_ptr(), dy.data_ptr(), out.data_ptr(), out.data_ptr(), wt.data_ptr()
        n0 = lib.dp_launch_count()
        assert getattr(lib, entry)(C.byref(a), S()) == c["refuse"]
        torch.cuda.synchronize()
        assert lib.dp_launch_count() == n0
        return
    rep = {}
    with Witness(lib, entry) as w:
        REPLAY[entry](lib, g, entry, a, rep)
    assert all(rc == 0 for rc, _ in w.deltas) and len(w.deltas) == 2, w.deltas
    if c["op"] == "wgrad":
        assert w.count(f"wgrad_bf16_kernel<{tile // 64}>") == 2, w.kernels
    else:
        gemms = 4 if c["op"] == "dgrad" and c.get("stride", 1) == 2 else 1
        assert w.count(f"conv_bf16_kernel<{tile // 64}>") == 2 * gemms, (w.kernels, tile)
        assert w.count("conv_bf16_kernel") == 2 * gemms, w.kernels
    _report(entry, rep)


# ---------------------------------------------------------------------------------------------------------------- GroupNorm / LayerNorm
def _gn_args(c):
    from diff_pruning_b200 import _lib as L
    a = L.GnArgs()
    C_ = c["C"]
    a.N, a.HW, a.C, a.G, a.eps, a.silu = c["N"], c["HW"], C_, c["G"], 1e-5, c.get("silu", 0)
    a.x, a.ldx = _ptr(c.get("px", 0)), C_ + c.get("xe", 0)
    a.gamma, a.beta = _ptr(c.get("pg", 0)), _ptr(c.get("pbeta", 0))
    a.mean = a.rstd = a.workspace = _ptr()
    if c["op"] == "gn_fwd":
        if c.get("no_y"):
            a.y_bf16, a.ldyb = _ptr(), C_ + (-C_) % 8
        else:
            a.y, a.ldy = _ptr(c.get("py", 0)), C_ + c.get("ye", 0)
    else:
        a.dy, a.lddy = _ptr(), C_ + c.get("dye", 0)
        a.dx, a.lddx = _ptr(c.get("pdx", 0)), C_ + c.get("dxe", 0)
        a.dgamma = a.dbeta = _ptr()
        if c.get("fin"):
            a.fin = _ptr()
        if c.get("add"):      # its own address unless the case adds into dx in place (the replay keys the aliasing on equal pointers)
            a.dx_add, a.ldadd = (a.dx, a.lddx) if c.get("alias") else (2 * BASE + 4 * c.get("padd", 0), C_ + c.get("adde", 0))
        if c.get("add2"):
            a.dx_add2, a.ldadd2 = 3 * BASE + 4 * c.get("padd2", 0), C_ + c.get("add2e", 0)
    return a


def _gn_refusal(lib, c, a):
    """The call on real buffers sized for its views: the exact code, and no launch.  The buffers do not make a wrongly admitted shape
    safe: a LayerNorm beyond NT * MAXCPT channels that reached the GroupNorm kernels would still write past their shared memory."""
    N, HW, C_ = c["N"], c["HW"], c["C"]
    rows = N * HW
    bufs = []

    def buf(n, dtype=torch.float32):
        bufs.append(torch.zeros(n + 8, dtype=dtype, device="cuda"))
        return bufs[-1].data_ptr()
    ph = lambda p: (int(p) - BASE) if p else None
    for f, ld in (("x", a.ldx), ("y", a.ldy), ("dy", a.lddy), ("dx", a.lddx)):
        if getattr(a, f):
            setattr(a, f, buf(rows * ld) + ph(getattr(a, f)))
    if a.y_bf16:
        a.y_bf16 = buf(rows * a.ldyb, torch.bfloat16)
    a.gamma, a.beta = buf(C_) + ph(a.gamma), buf(C_) + ph(a.beta)
    a.mean, a.rstd = buf(N * c["G"]), buf(N * c["G"])
    a.workspace = buf(lib.dp_groupnorm_workspace_bytes(N, HW, C_, c["G"]) // 4 + 1)
    if a.dgamma:
        a.dgamma, a.dbeta = buf(C_), buf(C_)
    for f, ld in (("dx_add", a.ldadd), ("dx_add2", a.ldadd2)):
        if getattr(a, f):
            setattr(a, f, buf(rows * ld) + (int(getattr(a, f)) % 16))
    n0 = lib.dp_launch_count()
    fn = lib.dp_groupnorm_fwd if c["op"] == "gn_fwd" else lib.dp_groupnorm_bwd
    assert fn(C.byref(a), S()) == c["refuse"], c["tag"]
    torch.cuda.synchronize()
    assert lib.dp_launch_count() == n0, c["tag"]


@pytest.mark.parametrize("c", de.GN, ids=[c["tag"] for c in de.GN])
def test_norm_edges(lib, c):
    g = torch.Generator().manual_seed(zlib.crc32(c["tag"].encode()))
    want = de.gn_path(c)
    a = _gn_args(c)
    if "refuse" in c:
        return _gn_refusal(lib, c, a)
    entry = "dp_groupnorm_fwd" if c["op"] == "gn_fwd" else "dp_groupnorm_bwd"
    rep = {}
    with Witness(lib, entry) as w:
        REPLAY[entry](lib, g, entry, a, rep)
    assert all(rc == 0 for rc, _ in w.deltas), w.deltas
    runs = 2
    if c["op"] == "gn_fwd":
        if want["ln"]:
            expect = {"ln_fwd_kernel": runs}
        else:
            s = "4" if want["v4"] else ""
            expect = {f"gn_stats{s}_kernel": runs, f"gn_apply{s}_kernel": runs, "gn_finalize_kernel": runs if want["finalize"] else 0}
        names = ("ln_fwd_kernel", "gn_stats_kernel", "gn_stats4_kernel", "gn_apply_kernel", "gn_apply4_kernel", "gn_finalize_kernel")
        calls = [d for _, d in w.deltas]
        assert calls == [sum(expect.values()) // runs] * runs, (calls, expect)
    else:
        # the replay runs the forward once for its statistics (not counted here), then the backward twice
        fwd = de.gn_path(dict(c, op="gn_fwd", py=0, ye=0, pbeta=0))
        if want["ln"]:
            expect = {"ln_bwd_dx_kernel": runs, "ln_bwd_param_partial_kernel": runs, "ln_bwd_param_final_kernel": runs}
        else:
            s = "4" if want["v4"] else ""
            expect = {f"gn_bwd_partial{s}_kernel": runs, f"gn_bwd_apply{s}_kernel": runs, "gn_bwd_reduce_kernel": runs if want["reduce"] else 0,
                      "gn_bwd_param_kernel": runs}
        names = ("ln_bwd_dx_kernel", "ln_bwd_param_partial_kernel", "ln_bwd_param_final_kernel", "gn_bwd_partial_kernel",
                 "gn_bwd_partial4_kernel", "gn_bwd_apply_kernel", "gn_bwd_apply4_kernel", "gn_bwd_reduce_kernel", "gn_bwd_param_kernel")
        calls = [d for _, d in w.deltas]
        assert calls == [sum(expect.values()) // runs - (1 if c.get("fin") else 0)] * runs, (calls, expect)
        assert ("ln_fwd_kernel" in w.kernels) == bool(fwd.get("ln")), (w.kernels, fwd)
    for k in names:
        assert w.count(k) == expect.get(k, 0), (k, w.kernels, want)
    _report(entry, rep)


# ---------------------------------------------------------------------------------------------------------------- rows / pointwise
@pytest.mark.parametrize("name,args", de.ROWS, ids=[f"{n}{a}" for n, a in de.ROWS])
def test_rows_edges(lib, name, args):
    g = torch.Generator().manual_seed(sum(args) + len(name))
    rep = {}
    if name == "dp_softmax_fwd":
        rows, cols = args
        fake = (_ptr(), _ptr(), rows, cols)
        kern = "softmax_fwd_kernel"
    elif name == "dp_softmax_bwd":
        rows, cols = args
        fake = (_ptr(), _ptr(), _ptr(), rows, cols, _ptr())
        kern = "softmax_bwd_kernel"
    elif name == "dp_amax":
        phase, ld, rows, cols = args
        fake = (_ptr(phase), ld, rows, cols, _ptr())
        kern = "amax_kernel"
    elif name == "dp_split_h3":
        phase, ld, bs, b, rows, cols, tr = args
        fake = (_ptr(phase), ld, bs, b, rows, cols, tr, _ptr(), _ptr(), _ptr())
        kern = "split_h3_t_kernel" if tr else "split_h3_rows_kernel"
    elif name == "dp_transpose_batched":
        b, rows, cols = args
        fake = (_ptr(), _ptr(), b, rows, cols)
        kern = "transpose_batched_kernel"
    elif name == "dp_gemm_batched":
        return _gemm_batched(lib, g, *args)
    else:
        return _colsum(lib, g, *args)
    with Witness(lib, name) as w:
        REPLAY[name](lib, g, name, fake, rep)
    assert w.deltas and all(rc == 0 and d == 1 for rc, d in w.deltas), w.deltas
    assert w.count(kern) == len(w.deltas), w.kernels
    _report(name, rep)


def _gemm_batched(lib, g, b, M, N, Kd, a_cs, b_cs, acc):
    """dp_gemm_batched through the census replay: A [b][M][Kd] and B [b][Kd][N], each K-contiguous (cs = 1) or not, into a C view with
    a pitch of N + 3 (sentinel columns beside it) and 1.5 alpha."""
    from diff_pruning_b200 import _lib as L
    a = L.GemmArgs()
    a.M, a.N, a.Kd, a.batch, a.alpha, a.accumulate = M, N, Kd, b, 1.5, acc
    a.a_rs, a.a_cs = (Kd, 1) if a_cs else (1, M)
    a.b_rs, a.b_cs = (N, 1) if b_cs else (1, Kd)
    a.a_bs, a.b_bs = M * Kd + 4, Kd * N + 4
    a.ldc, a.c_bs = N + 3, M * (N + 3) + 4
    a.A, a.B, a.C = _ptr(), _ptr(), _ptr()
    rep = {}
    with Witness(lib, "dp_gemm_batched") as w:
        REPLAY["dp_gemm_batched"](lib, g, "dp_gemm_batched", a, rep)
    assert w.deltas and all(rc == 0 and d == 1 for rc, d in w.deltas), w.deltas
    assert w.count("gemm_simt_kernel") == len(w.deltas), w.kernels
    _report("dp_gemm_batched", rep)


def _colsum(lib, g, phase, ld, rows, cols, seg, acc):
    """dp_colsum with a last segment shorter than seg_rows when seg_rows does not divide the rows: sum_bound per segment, one rounding of
    the old value; the rows past the last segment of the output and the channels beside it hold their sentinel."""
    from test_launch_census_gpu import SENT, Buf
    nseg = de.cdiv(rows, seg)
    x = Buf(_ptr(phase), rows, ld, cols, 3.0)
    x.v.copy_(_randn(g, rows, cols))
    out = Buf(_ptr(), nseg + 1, cols + 3, cols)
    o0 = _randn(g, nseg, cols)

    def reset():
        out.t.fill_(SENT)
        out.v[:nseg].copy_(o0)

    def run():
        assert lib.dp_colsum(x.ptr, ld, rows, cols, seg, out.ptr, cols + 3, acc, S()) == 0
    rep = {}
    with Witness(lib, "dp_colsum") as w:
        got, = _twice(run, reset, [out.v])
    assert w.count("colsum_kernel") == 2 and all(d == 1 for _, d in w.deltas)
    assert bool((got[nseg] == SENT).all()) and out.outside_untouched()
    xs = torch.nn.functional.pad(x.v.double(), (0, 0, 0, nseg * seg - rows)).view(nseg, seg, cols)
    ref = xs.sum(1) + (o0.double() if acc else 0)
    b = lc.sum_bound(xs.pow(2).sum(1).sqrt(), seg) + 2 * lc.U * (o0.double().abs() if acc else 0)
    _check(rep, "dp_colsum", got[:nseg], ref, b, f"{rows}x{cols} seg {seg}")
    _report("dp_colsum", rep)


def test_zz_report():
    """Worst err / bound per entry point over the sweep, and the SM count it ran on."""
    print(f"dispatch edges on {torch.cuda.get_device_name(0)}, {_sms()} SMs")
    for k in sorted(_REPORT):
        print(f"  {k:28s} worst err/bound {_REPORT[k]:.3g}")
    assert all(v <= 1.0 for v in _REPORT.values())
