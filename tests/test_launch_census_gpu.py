"""Launch census: every distinct launch the C1 / C3 / C5 Taylor-scoring plans and the pruned-C1 finetune plans (fp32-grade and bf16)
issue, replayed on fresh seeded buffers at its own geometry and checked element by element against a float64 restatement on the
device, within the error model of launch_census.py.

A plan is built with every kernel-launching entry point of the library wrapped, so both the recorded argument structs (bound when
the plan records them) and the lambda launches (which look the entry point up when called) go through the wrappers; one eager pass
records a copy of every call's arguments.  Launches are deduplicated on launch_census.launch_key.  A replay keeps the extents, the
pixel strides `ld` and each view's 16-byte phase, fills the channels around every written view with a sentinel, gives one operand
of each convolution per-channel scales 2^U(-6, 6), re-queries the split-K workspace, runs the weight gradient at the plan's split
count followed by dp_conv2d_wgrad_reduce, and also asserts: sentinels untouched, a second run bit-identical, amax_out == max|written|.
"""
import ctypes as C
import gc
import math

import pytest
import torch
import torch.nn.functional as F

import launch_census as lc

pytestmark = pytest.mark.gpu

SENT = -777.0
# the split-K reduce runs (and is checked: dW, db, fused scores) right after every replayed weight gradient; every other kind a plan
# issues is replayed on its own
INSIDE = {"dp_conv2d_wgrad_reduce": ("dp_conv2d_wgrad", "dp_conv2d_wgrad_bf16")}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    assert lib.dp_tc_available() and lib.dp_bf16_available()
    return lib


def S():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------- capture
def _capture(lib, run):
    """Calls every kernel-launching entry point receives while run() builds a fresh plan and makes one eager pass: [(name, args)]
    (the stream each call was enqueued on is dropped: the census replays launches one at a time)."""
    calls = []
    with lc.wrap_launches(lib, lambda name, args, stream: calls.append((name, args))):
        run()
        torch.cuda.synchronize()
    return calls


def _unique(calls):
    out = {}
    for name, args in calls:
        key = lc.launch_key(name, lc.argkinds(name), args)
        if key not in out:
            out[key] = (name, args)
    return list(out.values())


# ---------------------------------------------------------------------------------------------------------------------- buffers
class Buf:
    """A [rows][ld] fp32 (or bf16) buffer whose view of `cols` channels starts at the same 16-byte phase as the captured pointer;
    everything around the view holds `fill`."""

    TAIL_ROWS = 128       # rows of `fill` past the view: a box of pixels running past the batch must not store there

    def __init__(self, ptr, rows, ld, cols, fill=SENT, dtype=torch.float32):
        esz = 4 if dtype == torch.float32 else 2
        self.phase = (int(ptr) % 16) // esz
        self.t = torch.full(((rows + self.TAIL_ROWS) * ld + 16 // esz,), fill, device="cuda", dtype=dtype)
        self.v = self.t[self.phase:self.phase + rows * ld].view(rows, ld)[:, :cols]
        self.fill = fill

    @property
    def ptr(self):
        return self.v.data_ptr()

    def outside_untouched(self) -> bool:
        mask = torch.ones_like(self.t, dtype=torch.bool)
        idx = torch.arange(self.v.shape[0], device="cuda")[:, None] * self.v.stride(0) + torch.arange(self.v.shape[1], device="cuda")
        mask[self.phase + idx.reshape(-1)] = False
        return bool((self.t[mask] == self.fill).all())


def _slot(lib, ptr, ld, rows, cols):
    s = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.dp_amax(ptr, ld, rows, cols, s.data_ptr(), S()) == 0
    return s


def _slot_value(s):
    return float(s.view(torch.float32).item())


def _scaled(g, rows, cols):
    """Seeded normal data with per-channel scales 2^U(-6, 6)."""
    return torch.randn(rows, cols, generator=g).mul_(2.0 ** (torch.rand(1, cols, generator=g) * 12 - 6)).cuda()


def _randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _nchw(v, N, H, W):
    return v.double().reshape(N, H, W, -1).permute(0, 3, 1, 2)


def _nhwc_rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


class Conv:
    """fp64 conv2d with explicit top / left padding and the bottom / right padding implied by the output extent (dp_conv_args)."""

    def __init__(self, a):
        self.a = a
        self.pb = max(0, (a.P - 1) * a.stride + a.R - a.H - a.pad_t)
        self.pr = max(0, (a.Q - 1) * a.stride + a.S - a.W - a.pad_l)

    def fwd(self, x, w):
        a = self.a
        return F.conv2d(F.pad(x, (a.pad_l, self.pr, a.pad_t, self.pb)), w, stride=a.stride)[:, :, :a.P, :a.Q]

    def grads(self, x, w, dy):
        x, w = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        dx, dw = torch.autograd.grad(self.fwd(x, w), (x, w), dy)
        return dx, dw


def _fresh(a):
    """A copy of a captured argument struct with every pointer field NULL: a replay sets the ones it uses, nothing of the freed plan
    stays reachable."""
    from diff_pruning_b200.engine import _copy_args
    r = _copy_args(a)
    for name, t in r._fields_:
        if t is C.c_void_p:
            setattr(r, name, None)
    return r


def _check(rep, kind, got, ref, bound, what):
    worst, where = lc.violations(got, ref, bound)
    rep.setdefault(kind, []).append(worst)
    assert not where, f"{kind} {what}: |err| above the bound at {where} (worst err/bound {worst:.3g})"


def _twice(run, reset, outs):
    """Runs the launch twice from the same initial state; returns the first run's outputs after asserting the second is bit-identical."""
    reset()
    run()
    first = [o.clone() for o in outs]
    reset()
    run()
    for a, b in zip(first, outs):
        assert torch.equal(a, b), "a second run from the same state is not bit-identical"
    return first


# ---------------------------------------------------------------------------------------------------------------------- replays
def _conv_weights(lib, g, K, Cin, R, Sx, tc):
    w = (torch.randn(K, Cin, R, Sx, generator=g) / math.sqrt(Cin * R * Sx)).cuda()
    ck, kc = torch.empty(w.numel(), device="cuda"), torch.empty(w.numel(), device="cuda")
    assert lib.dp_pack_conv_weight(w.data_ptr(), K, Cin, R, Sx, ck.data_ptr(), kc.data_ptr(), S()) == 0
    packs = None
    if tc:
        na, nb = R * Sx * K * lib.dp_tc_weight_row(Cin), R * Sx * Cin * lib.dp_tc_weight_row(K)
        packs = [torch.empty(n, device="cuda", dtype=torch.float16) for n in (na, na, nb, nb)] + [torch.zeros(1, dtype=torch.int32, device="cuda")]
        assert lib.dp_pack_conv_weight_tc(w.data_ptr(), K, Cin, R, Sx, *[p.data_ptr() for p in packs], S()) == 0
    return w, ck, kc, packs


def _epilogue(lib, g, a, r, K, rows_out, ref, epi):
    """Fresh bias / per-image row / residual operands of a fprop-type launch `r` (set where the captured `a` has them), added to ref."""
    keep = []
    if a.bias:
        b = _randn(g, K)
        r.bias = b.data_ptr()
        ref += b.double()
        epi += b.double().abs()
        keep.append(b)
    if a.rowadd:
        ra = Buf(a.rowadd, a.N, a.ld_rowadd, K, 0.0)
        ra.v.copy_(_randn(g, a.N, K))
        r.rowadd = ra.ptr
        per = rows_out // a.N
        add = ra.v.double().repeat_interleave(per, 0)
        ref += add
        epi += add.abs()
        keep.append(ra)
    if a.residual:
        rs = Buf(a.residual, rows_out, a.ld_res, K, 0.0)
        rs.v.copy_(_randn(g, rows_out, K))
        r.residual = rs.ptr
        ref += rs.v.double()
        epi += rs.v.double().abs()
        keep.append(rs)
    return keep


DP_CONV_RELU = 4


def replay_conv(lib, g, name, a, rep, chain=None):
    """fprop / dgrad (fp32-grade) at the captured geometry.  With DP_CONV_RELU the fp64 reference takes the ReLU after every epilogue
    term (1-Lipschitz: same bound).  chain(args, split-K workspace floats) -> (L, tensor-core launch?) overrides the box kernel's
    chain length (the general-geometry and SIMT kernels of the evaluation census).  Returns the split-K workspace the launch was
    given, NaN-filled before the first run (None without one)."""
    N, H, W, Cin, P, Q, K, R, Sx = a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S
    tc = bool(a.w_tc_hi)
    w, ck, kc, packs = _conv_weights(lib, g, K, Cin, R, Sx, tc)
    r = _fresh(a)
    cv = Conv(a)
    w64 = w.double()
    rows_in, rows_out = N * H * W, N * P * Q
    acc = bool(a.flags & 1)
    keep = []
    if name == "dp_conv2d_fprop":
        x = Buf(a.x, rows_in, a.ldx, Cin, 3.0)
        x.v.copy_(_scaled(g, rows_in, Cin))
        y = Buf(a.y, rows_out, a.ldy, K)
        r.x, r.y, r.w = x.ptr, y.ptr, ck.data_ptr()
        if tc:
            r.w_tc_hi, r.w_tc_lo, r.amax_w = packs[0].data_ptr(), packs[1].data_ptr(), packs[4].data_ptr()
            sx = _slot(lib, x.ptr, a.ldx, rows_in, Cin)
            r.amax_x = sx.data_ptr()
        x64 = _nchw(x.v, N, H, W)
        ref = _nhwc_rows(cv.fwd(x64, w64))
        s = _nhwc_rows(cv.fwd(x64 ** 2, w64 ** 2)).sqrt()
        epi = torch.zeros_like(ref)
        keep += _epilogue(lib, g, a, r, K, rows_out, ref, epi)
        kg, out, op, launch = Cin, y, 0, lib.dp_conv2d_fprop
    else:
        dy = Buf(a.y, rows_out, a.ldy, K, 3.0)
        dy.v.copy_(_scaled(g, rows_out, K))
        dx = Buf(a.x, rows_in, a.ldx, Cin)
        r.x, r.y, r.w = dx.ptr, dy.ptr, kc.data_ptr()
        if tc:
            r.w_tc_hi, r.w_tc_lo, r.amax_w = packs[2].data_ptr(), packs[3].data_ptr(), packs[4].data_ptr()
            sy = _slot(lib, dy.ptr, a.ldy, rows_out, K)
            r.amax_y = sy.data_ptr()
        x0 = torch.zeros(N, Cin, H, W, dtype=torch.float64, device="cuda")
        dy64 = _nchw(dy.v, N, P, Q)
        ref = _nhwc_rows(cv.grads(x0, w64, dy64)[0])
        s = _nhwc_rows(cv.grads(x0, w64 ** 2, dy64 ** 2)[0]).sqrt()
        epi = torch.zeros_like(ref)
        kg, out, op, launch = K, dx, 1, lib.dp_conv2d_dgrad
    init = _randn(g, out.v.shape[0], out.v.shape[1]) if acc else None
    if acc:
        ref += init.double()
        epi += init.double().abs()
    if a.flags & DP_CONV_RELU:
        ref = ref.clamp_min(0.0)
    r.workspace = None
    ws, need = None, 0
    if a.workspace:
        need = lib.dp_conv_splitk_workspace_floats(C.byref(r), op)
        if need > 0:
            ws = torch.full((need,), float("nan"), device="cuda")
            r.workspace = ws.data_ptr()
    if chain is not None:
        L_, on_tc = chain(a, need)
    else:
        L_, on_tc = lc.chain_fprop(R * Sx, kg, lc.splitk_count(need, out.v.shape[0], out.v.shape[1], R * Sx * -(-kg // 64))), tc
    assert not on_tc or L_ <= lc.L_MAX, f"{name}: chain of {L_} updates, beyond the {lc.L_MAX} at which the bound keeps its teeth"
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if a.amax_out else None
    r.amax_out = so.data_ptr() if so is not None else None

    def reset():
        out.t.fill_(SENT)
        if acc:
            out.v.copy_(init)
        if so is not None:
            so.zero_()

    def run():
        assert launch(C.byref(r), S()) == 0
    got, = _twice(run, reset, [out.v])
    assert out.outside_untouched(), f"{name}: channels around the written view changed"
    _check(rep, name, got, ref, lc.product_bound(s, L_, epi), f"{N}x{H}x{W} {Cin}->{K} {R}x{Sx} s{a.stride} L={L_}")
    if so is not None:
        assert _slot_value(so) == float(got.abs().max()), name
    return ws


def replay_wgrad(lib, g, name, a, rep):
    """dp_conv2d_wgrad (fp32-grade) / dp_conv2d_wgrad_bf16 at the plan's split count, then dp_conv2d_wgrad_reduce into a non-zero dW
    (+=), with the bias gradient (when the launch writes bias_ws) and the fused signed scores."""
    from diff_pruning_b200 import _lib as L
    N, H, W, Cin, P, Q, K, R, Sx, sp = a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.splits
    bf = name.endswith("bf16")
    rows_in, rows_out = N * H * W, N * P * Q
    r = _fresh(a)
    if bf:
        x = Buf(a.x_bf16, rows_in, a.ldx, Cin, 3.0, torch.bfloat16)
        dy = Buf(a.dy_bf16, rows_out, a.lddy, K, 3.0, torch.bfloat16)
        x.v.copy_(_scaled(g, rows_in, Cin))
        dy.v.copy_(_randn(g, rows_out, K))
        r.x_bf16, r.dy_bf16 = x.ptr, dy.ptr
        bws = None
    else:
        x = Buf(a.x, rows_in, a.ldx, Cin, 3.0)
        dy = Buf(a.y, rows_out, a.ldy, K, 3.0)
        x.v.copy_(_scaled(g, rows_in, Cin))
        dy.v.copy_(_randn(g, rows_out, K))
        r.x, r.y = x.ptr, dy.ptr
        if a.amax_x:
            sx, sy = _slot(lib, x.ptr, a.ldx, rows_in, Cin), _slot(lib, dy.ptr, a.ldy, rows_out, K)
            r.amax_x, r.amax_y = sx.data_ptr(), sy.data_ptr()
        bws = torch.full((sp * K,), float("nan"), device="cuda") if a.bias_ws else None
        r.bias_ws = bws.data_ptr() if bws is not None else None
    ws = torch.full((sp * K * R * Sx * Cin,), float("nan"), device="cuda")
    r.workspace = ws.data_ptr()
    w = _randn(g, K, Cin, R, Sx)
    dw0, db0 = _randn(g, K, Cin, R, Sx), _randn(g, K)
    so0, si0 = _randn(g, K), _randn(g, Cin)
    dw, db, so, si = (torch.empty_like(t) for t in (dw0, db0, so0, si0))
    ra = L.WgradReduceArgs()
    ra.K, ra.C, ra.R, ra.S, ra.splits = K, Cin, R, Sx, sp
    ra.workspace, ra.dw = ws.data_ptr(), dw.data_ptr()
    if not bf:       # the fp32-grade plans fuse the signed Taylor scores into the reduce; the bf16 ones do not
        ra.w, ra.score_out, ra.score_in = w.data_ptr(), so.data_ptr(), si.data_ptr()
    if bws is not None:
        ra.bias_ws, ra.db = bws.data_ptr(), db.data_ptr()
    launch = lib.dp_conv2d_wgrad_bf16 if bf else lib.dp_conv2d_wgrad

    def reset():
        for t, t0 in ((dw, dw0), (db, db0), (so, so0), (si, si0)):
            t.copy_(t0)

    def run():
        assert launch(C.byref(r), S()) == 0
        assert lib.dp_conv2d_wgrad_reduce(C.byref(ra), S()) == 0
    got_dw, got_db, got_so, got_si = _twice(run, reset, [dw, db, so, si])
    cv = Conv(a)
    x64, dy64 = _nchw(x.v, N, H, W), _nchw(dy.v, N, P, Q)
    w0 = torch.zeros(K, Cin, R, Sx, dtype=torch.float64, device="cuda")
    dwt = cv.grads(x64, w0, dy64)[1]
    s = cv.grads(x64 ** 2, w0, dy64 ** 2)[1].sqrt()
    L_ = lc.chain_wgrad(lc.wgrad_pixels_per_cta(rows_out, sp), sp)
    assert L_ <= lc.L_MAX or not (bf or a.amax_x), f"{name}: chain of {L_} updates, beyond the {lc.L_MAX} at which the bound keeps its teeth"
    bound = lc.product_bound(s, L_)
    tag = f"{N}x{H}x{W} {Cin}->{K} {R}x{Sx} s{a.stride} splits {sp} L={L_}"
    _check(rep, name, got_dw, dw0.double() + dwt, bound + 2 * lc.U * dw0.double().abs(), tag)
    rep.setdefault("dp_conv2d_wgrad_reduce", []).append(rep[name][-1])
    if bws is not None:
        dyd = dy.v.double()
        _check(rep, name, got_db, db0.double() + dyd.sum(0), lc.product_bound(dyd.pow(2).sum(0).sqrt(), L_, db0.double().abs()), tag + " db")
    if not bf:
        wd = w.double()
        for dims, t0, got in (((1, 2, 3), so0, got_so), ((0, 2, 3), si0, got_si)):
            ref = t0.double() + (wd * dwt).sum(dims)
            b = (wd.abs() * bound).sum(dims) + 2 * lc.U * ((wd * dwt).abs().sum(dims) + t0.double().abs())
            _check(rep, name, got, ref, b, tag + " scores")


def replay_conv_bf16(lib, g, name, a, rep):
    """dp_conv2d_fprop_bf16 / dp_conv2d_dgrad_bf16 against fp64 math on the bf16-rounded operands."""
    N, H, W, Cin, P, Q, K, R, Sx = a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S
    rows_in, rows_out = N * H * W, N * P * Q
    w = (torch.randn(K, Cin, R, Sx, generator=g) / math.sqrt(Cin * R * Sx)).cuda()
    kc = torch.empty(R * Sx * K * lib.dp_bf16_weight_row(Cin), device="cuda", dtype=torch.bfloat16)
    ck = torch.empty(R * Sx * Cin * lib.dp_bf16_weight_row(K), device="cuda", dtype=torch.bfloat16)
    assert lib.dp_pack_conv_weight_bf16(w.data_ptr(), K, Cin, R, Sx, kc.data_ptr(), ck.data_ptr(), S()) == 0
    w64 = w.bfloat16().double()
    r = _fresh(a)
    cv = Conv(a)
    acc = bool(a.flags & 1)
    keep = []
    if name == "dp_conv2d_fprop_bf16":
        x = Buf(a.x_bf16, rows_in, a.ldx, Cin, 3.0, torch.bfloat16)
        x.v.copy_(_scaled(g, rows_in, Cin))
        out = Buf(a.out, rows_out, a.ld_out, K)
        r.x_bf16, r.out, r.w_bf16 = x.ptr, out.ptr, kc.data_ptr()
        x64 = _nchw(x.v, N, H, W)
        ref = _nhwc_rows(cv.fwd(x64, w64))
        s = _nhwc_rows(cv.fwd(x64 ** 2, w64 ** 2)).sqrt()
        epi = torch.zeros_like(ref)
        keep += _epilogue(lib, g, a, r, K, rows_out, ref, epi)
        L_ = lc.chain_fprop(R * Sx, Cin)
        assert L_ <= lc.L_MAX, (name, L_)
        launch = lib.dp_conv2d_fprop_bf16
    else:
        dy = Buf(a.dy_bf16, rows_out, a.lddy, K, 3.0, torch.bfloat16)
        dy.v.copy_(_scaled(g, rows_out, K))
        out = Buf(a.out, rows_in, a.ld_out, Cin)
        r.dy_bf16, r.out, r.w_bf16 = dy.ptr, out.ptr, ck.data_ptr()
        x0 = torch.zeros(N, Cin, H, W, dtype=torch.float64, device="cuda")
        dy64 = _nchw(dy.v, N, P, Q)
        ref = _nhwc_rows(cv.grads(x0, w64, dy64)[0])
        s = _nhwc_rows(cv.grads(x0, w64 ** 2, dy64 ** 2)[0]).sqrt()
        epi = torch.zeros_like(ref)
        L_ = lc.chain_fprop(R * Sx, K)
        assert L_ <= lc.L_MAX, (name, L_)
        launch = lib.dp_conv2d_dgrad_bf16
    init = _randn(g, out.v.shape[0], out.v.shape[1]) if acc else None
    if acc:
        ref += init.double()
        epi += init.double().abs()

    def reset():
        out.t.fill_(SENT)
        if acc:
            out.v.copy_(init)

    def run():
        assert launch(C.byref(r), S()) == 0
    got, = _twice(run, reset, [out.v])
    assert out.outside_untouched(), f"{name}: channels around the written view changed"
    _check(rep, name, got, ref, lc.product_bound(s, L_, epi), f"{N}x{H}x{W} {Cin}->{K} {R}x{Sx} s{a.stride} L={L_}")


def replay_gemm_nt(lib, g, name, a, rep):
    """dp_gemm_nt_tc: C = alpha A B^T per batch, B given as its dp_split_h3 fp16 hi / lo' parts."""
    nb, T, Kg, Nn = a.batch, a.H * a.W, a.Kg, a.N
    r = _fresh(a)
    A = Buf(a.A, nb * T, a.ld_a, Kg, 3.0)
    A.v.copy_(_scaled(g, nb * T, Kg))
    B = _randn(g, nb, Nn, Kg)
    K8 = (Kg + 7) // 8 * 8
    hi, lo = (torch.empty(nb * Nn * K8, device="cuda", dtype=torch.float16) for _ in range(2))
    sb, sa = _slot(lib, B.data_ptr(), Kg, nb * Nn, Kg), _slot(lib, A.ptr, a.ld_a, nb * T, Kg)
    assert lib.dp_split_h3(B.data_ptr(), Kg, Nn * Kg, nb, Nn, Kg, 0, sb.data_ptr(), hi.data_ptr(), lo.data_ptr(), S()) == 0
    out = Buf(a.C, nb * T, a.ldc, Nn)
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if a.amax_out else None
    r.A, r.b_hi, r.b_lo, r.C, r.amax_a, r.amax_b = A.ptr, hi.data_ptr(), lo.data_ptr(), out.ptr, sa.data_ptr(), sb.data_ptr()
    r.amax_out = so.data_ptr() if so is not None else None

    def reset():
        out.t.fill_(SENT)
        if so is not None:
            so.zero_()

    def run():
        assert lib.dp_gemm_nt_tc(C.byref(r), S()) == 0
    got, = _twice(run, reset, [out.v])
    assert out.outside_untouched(), name
    A64, B64 = A.v.double().view(nb, T, Kg), B.double()
    ref = (a.alpha * torch.bmm(A64, B64.transpose(1, 2))).reshape(nb * T, Nn)
    s = (abs(a.alpha) * torch.bmm(A64 ** 2, (B64 ** 2).transpose(1, 2)).sqrt()).reshape(nb * T, Nn)
    L_ = lc.chain_fprop(1, Kg)
    assert L_ <= lc.L_MAX, (name, L_)
    _check(rep, name, got, ref, lc.product_bound(s, L_), f"batch {nb} T {T} Kg {Kg} N {Nn} L={L_}")
    if so is not None:
        assert _slot_value(so) == float(got.abs().max()), name


def _strided(ptr, shape, strides, fill, g=None):
    """A fresh buffer holding a (batch, rows, cols) strided view at the captured pointer's 16-byte phase: (buffer, view, phase)."""
    phase = (int(ptr) % 16) // 4
    n = 1 + sum((s_ - 1) * st for s_, st in zip(shape, strides))
    buf = torch.full((n + 4,), fill, device="cuda")
    v = buf[phase:].as_strided(shape, strides)
    if g is not None:
        v.copy_(_randn(g, *shape))
    return buf, v, phase


def replay_gemm_batched(lib, g, name, a, rep):
    """dp_gemm_batched (exact-fp32 SIMT GEMM of the attention cores whose token count is not a multiple of 128): a sequential fp32
    chain of Kd fused multiply-adds per output."""
    nb, M, Nn, Kd = a.batch, a.M, a.N, a.Kd
    r = _fresh(a)
    _, A, _ = _strided(a.A, (nb, M, Kd), (a.a_bs, a.a_rs, a.a_cs), 3.0, g)
    _, B, _ = _strided(a.B, (nb, Kd, Nn), (a.b_bs, a.b_rs, a.b_cs), 3.0, g)
    cbuf, Cv, cph = _strided(a.C, (nb, M, Nn), (a.c_bs, a.ldc, 1), SENT)
    init = _randn(g, nb, M, Nn) if a.accumulate else None
    r.A, r.B, r.C = A.data_ptr(), B.data_ptr(), Cv.data_ptr()

    def reset():
        cbuf.fill_(SENT)
        if init is not None:
            Cv.copy_(init)

    def run():
        assert lib.dp_gemm_batched(C.byref(r), S()) == 0
    got, = _twice(run, reset, [Cv])
    inside = torch.zeros_like(cbuf, dtype=torch.bool)
    inside[cph:].as_strided((nb, M, Nn), (a.c_bs, a.ldc, 1)).fill_(True)
    assert bool((cbuf[~inside] == SENT).all()), name
    A64, B64 = A.double(), B.double()
    ref = a.alpha * torch.bmm(A64, B64)
    s = abs(a.alpha) * torch.bmm(A64 ** 2, B64 ** 2).sqrt()
    epi = None
    if init is not None:
        ref, epi = ref + init.double(), init.double().abs()
    _check(rep, name, got, ref, lc.product_bound(s, Kd, epi), f"batch {nb} {M}x{Nn}x{Kd}")


def replay_softmax(lib, g, name, args, rep):
    """Row softmax (in place, as the plans run it) within launch_census.softmax_fwd_bound, and its backward ds = p (dp - sum_j dp_j p_j): the
    backward's row sum sum_j dp_j p_j is a fixed-order fp32 sum of <= 1024 terms, 2^-18 * sum_j |dp_j p_j| covers it with room."""
    if name == "dp_softmax_fwd":
        _, _, rows, cols = args
        x = _randn(g, rows, cols, scale=3.0)
        buf = x.clone()
        ref = torch.softmax(x.double(), -1)
        z = x.double() - x.double().amax(-1, keepdim=True)

        def run():
            assert lib.dp_softmax_fwd(buf.data_ptr(), buf.data_ptr(), rows, cols, S()) == 0
        got, = _twice(run, lambda: buf.copy_(x), [buf])
        _check(rep, name, got, ref, lc.softmax_fwd_bound(ref, z, cols), f"{rows}x{cols}")
    else:
        _, _, _, rows, cols, amax = args
        p = torch.softmax(_randn(g, rows, cols, scale=3.0), -1)
        dp = _randn(g, rows, cols)
        buf = dp.clone()
        so = torch.zeros(1, dtype=torch.int32, device="cuda") if amax else None

        def reset():
            buf.copy_(dp)
            if so is not None:
                so.zero_()

        def run():
            assert lib.dp_softmax_bwd(p.data_ptr(), buf.data_ptr(), buf.data_ptr(), rows, cols, so.data_ptr() if so is not None else None, S()) == 0
        got, = _twice(run, reset, [buf])
        p64, dp64 = p.double(), dp.double()
        ref = p64 * (dp64 - (dp64 * p64).sum(-1, keepdim=True))
        bound = 2.0 ** -22 * ref.abs() + p64 * (2.0 ** -22 * dp64.abs() + 2.0 ** -18 * (dp64 * p64).abs().sum(-1, keepdim=True))
        _check(rep, name, got, ref, bound, f"{rows}x{cols}")
        if so is not None:
            assert _slot_value(so) == float(got.abs().max()), name


def replay_groupnorm_fwd(lib, g, name, a, rep):
    """GroupNorm / LayerNorm (+SiLU) forward: y (and its bf16 copy).  Bound: fp32 statistics over a group (relative error of mean and
    rstd below 2^-21 for these sizes), normalisation and affine a few roundings, the special-function sigmoid ~3e-7 relative:
    |y^ - y| <= 2^-19 (|gamma| (|x_hat| + 1) + |beta|)."""
    assert a.dropout_p == 0, "dropout masks are outside this replay"
    N, HW, Cc, G = a.N, a.HW, a.C, a.G
    rows = N * HW
    r = _fresh(a)
    x = Buf(a.x, rows, a.ldx, Cc, 3.0)
    x.v.copy_(_randn(g, rows, Cc, scale=2.0) + 0.5)
    gamma, beta = Buf(a.gamma, 1, Cc, Cc, 0.0), Buf(a.beta, 1, Cc, Cc, 0.0)
    gamma.v.copy_(_randn(g, 1, Cc))
    beta.v.copy_(_randn(g, 1, Cc, scale=0.5))
    stats = torch.empty(2 * N * G, device="cuda")
    wsp = torch.empty((lib.dp_groupnorm_workspace_bytes(N, HW, Cc, G) + 3) // 4 + 1, device="cuda")
    y = Buf(a.y, rows, a.ldy, Cc) if a.y else None
    yb = Buf(a.y_bf16, rows, a.ldyb, Cc, 5.0, torch.bfloat16) if a.y_bf16 else None
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if a.amax_y else None
    r.x, r.gamma, r.beta, r.mean, r.rstd, r.workspace = x.ptr, gamma.ptr, beta.ptr, stats.data_ptr(), stats.data_ptr() + 4 * N * G, wsp.data_ptr()
    r.y = y.ptr if y else None
    r.y_bf16 = yb.ptr if yb else None
    r.amax_y = so.data_ptr() if so is not None else None
    r.dropout_seed_dev = None
    outs = [o.v for o in (y, yb) if o is not None]

    def reset():
        for o in (y, yb):
            if o is not None:
                o.t.fill_(o.fill)
        if so is not None:
            so.zero_()

    def run():
        assert lib.dp_groupnorm_fwd(C.byref(r), S()) == 0
    got = _twice(run, reset, outs)
    x64 = x.v.double().view(N, HW, Cc).permute(0, 2, 1)
    xh = F.group_norm(x64, G, eps=a.eps).permute(0, 2, 1).reshape(rows, Cc)
    ga, be = gamma.v.double(), beta.v.double()
    z = xh * ga + be
    ref = F.silu(z) if a.silu else z
    bound = 2.0 ** -19 * (ga.abs() * (xh.abs() + 1) + be.abs())
    tag = f"N {N} HW {HW} C {Cc} G {G} silu {a.silu}"
    for o, gt in zip([o for o in (y, yb) if o is not None], got):
        assert o.outside_untouched(), name
        extra = 2.0 ** -8 * ref.abs() if o is yb else 0          # bf16 copy: one more RNE rounding to 8 significant bits
        _check(rep, name, gt.double() if o is yb else gt, ref, bound + extra, tag + (" bf16" if o is yb else ""))
    if so is not None:
        assert _slot_value(so) == float(got[0].abs().max()), name


def replay_geglu(lib, g, name, args, rep):
    """GEGLU out = a * gelu(gate) (erf GELU) and its backward.  Bound: erf / exp a few ulp, products two roundings:
    2^-20 relative to the magnitudes of the terms."""
    if name == "dp_geglu_fwd":
        _, ldu, _, ldo, rows, inner = args
        u = Buf(args[0], rows, ldu, 2 * inner, 3.0)
        u.v.copy_(_randn(g, rows, 2 * inner, scale=2.0))
        out = Buf(args[2], rows, ldo, inner)

        def run():
            assert lib.dp_geglu_fwd(u.ptr, ldu, out.ptr, ldo, rows, inner, S()) == 0
        got, = _twice(run, lambda: out.t.fill_(SENT), [out.v])
        assert out.outside_untouched(), name
        av, gv = u.v[:, :inner].double(), u.v[:, inner:].double()
        ref = av * F.gelu(gv)
        _check(rep, name, got, ref, 2.0 ** -20 * av.abs() * (gv.abs() + 1), f"{rows}x{inner}")
    else:
        _, ldu, _, lddo, _, lddu, rows, inner = args
        u = Buf(args[0], rows, ldu, 2 * inner, 3.0)
        u.v.copy_(_randn(g, rows, 2 * inner, scale=2.0))
        do = Buf(args[2], rows, lddo, inner, 3.0)
        do.v.copy_(_randn(g, rows, inner))
        du = Buf(args[4], rows, lddu, 2 * inner)

        def run():
            assert lib.dp_geglu_bwd(u.ptr, ldu, do.ptr, lddo, du.ptr, lddu, rows, inner, S()) == 0
        got, = _twice(run, lambda: du.t.fill_(SENT), [du.v])
        assert du.outside_untouched(), name
        av, gv = (u.v[:, :inner].double().requires_grad_(True), u.v[:, inner:].double().requires_grad_(True))
        d64 = do.v.double()
        ga, gg = torch.autograd.grad(av * F.gelu(gv), (av, gv), d64)
        ref = torch.cat([ga, gg], 1)
        mag = torch.cat([d64.abs() * (gv.abs() + 1), d64.abs() * av.abs() * (1 + gv ** 2)], 1).detach()
        _check(rep, name, got, ref, 2.0 ** -20 * mag, f"{rows}x{inner}")


REPLAY = {
    "dp_conv2d_fprop": replay_conv, "dp_conv2d_dgrad": replay_conv,
    "dp_conv2d_wgrad": replay_wgrad, "dp_conv2d_wgrad_bf16": replay_wgrad,
    "dp_conv2d_fprop_bf16": replay_conv_bf16, "dp_conv2d_dgrad_bf16": replay_conv_bf16,
    "dp_gemm_nt_tc": replay_gemm_nt, "dp_gemm_batched": replay_gemm_batched,
    "dp_softmax_fwd": replay_softmax, "dp_softmax_bwd": replay_softmax,
    "dp_groupnorm_fwd": replay_groupnorm_fwd,
    "dp_geglu_fwd": replay_geglu, "dp_geglu_bwd": replay_geglu,
}


# ------------------------------------------------------------------------------------------- normalisation backward, reductions, pointwise
def _gn_fwd_for(lib, g, a, x, gamma, beta):
    """Runs dp_groupnorm_fwd on the replay's x / gamma / beta (statistics for the backward); returns (args, stats, workspace)."""
    r = _fresh(a)
    N, HW, Cc, G = a.N, a.HW, a.C, a.G
    stats = torch.empty(2 * N * G, device="cuda")
    wsp = torch.empty((lib.dp_groupnorm_workspace_bytes(N, HW, Cc, G) + 3) // 4 + 1, device="cuda")
    y = torch.empty(N * HW, Cc, device="cuda")
    r.x, r.ldx, r.y, r.ldy, r.gamma, r.beta = x.ptr, a.ldx, y.data_ptr(), Cc, gamma.ptr, beta.ptr
    r.mean, r.rstd, r.workspace = stats.data_ptr(), stats.data_ptr() + 4 * N * G, wsp.data_ptr()
    assert lib.dp_groupnorm_fwd(C.byref(r), S()) == 0
    return r, (stats, wsp, y)


def replay_groupnorm_bwd(lib, g, name, a, rep):
    """GroupNorm / LayerNorm (+SiLU) backward at the captured geometry: dx (=, or += through dx_add aliasing dx) + dx_add2, amax_dx,
    and dgamma / dbeta (+=), directly or through `fin` and dp_groupnorm_bwd_param.  Against fp64 autograd of the forward.
    Bound on dx = rstd (gamma dy' - mean_g(gamma dy') - x_hat mean_g(gamma dy' x_hat)), dy' = dy silu'(z): each term a few roundings
    (2^-20 relative to its magnitude, the special-function sigmoid inside silu' included) plus the error of the two group sums
    (sum_bound over the N_g = HW * C / G elements of a group), plus one rounding per addend; dgamma / dbeta: sum_bound over the N * HW
    pixels plus one rounding of the old value."""
    assert a.dropout_p == 0, "dropout masks are outside this replay"
    N, HW, Cc, G = a.N, a.HW, a.C, a.G
    rows, cg = N * HW, Cc // G
    x = Buf(a.x, rows, a.ldx, Cc, 3.0)
    x.v.copy_(_randn(g, rows, Cc, scale=2.0) + 0.5)
    gamma, beta = Buf(a.gamma, 1, Cc, Cc, 0.0), Buf(a.beta, 1, Cc, Cc, 0.0)
    gamma.v.copy_(_randn(g, 1, Cc))
    beta.v.copy_(_randn(g, 1, Cc, scale=0.5))
    from diff_pruning_b200.engine import _copy_args
    f, keep = _gn_fwd_for(lib, g, a, x, gamma, beta)
    r = _copy_args(f)
    r.y = None
    dy = Buf(a.dy, rows, a.lddy, Cc, 3.0)
    dy.v.copy_(_randn(g, rows, Cc))
    alias = bool(a.dx_add) and a.dx_add == a.dx
    dx = Buf(a.dx, rows, a.lddx, Cc)
    dx0 = _randn(g, rows, Cc) if alias else None
    add = add2 = None
    if a.dx_add and not alias:
        add = Buf(a.dx_add, rows, a.ldadd, Cc, 3.0)
        add.v.copy_(_randn(g, rows, Cc))
    if a.dx_add2:
        add2 = Buf(a.dx_add2, rows, a.ldadd2, Cc, 3.0)
        add2.v.copy_(_randn(g, rows, Cc))
    dg, db = Buf(a.dgamma, 1, Cc, Cc, 0.0), Buf(a.dbeta, 1, Cc, Cc, 0.0)
    dg0, db0 = _randn(g, 1, Cc), _randn(g, 1, Cc)
    fin = torch.empty(2 * N * Cc, device="cuda") if a.fin else None
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if a.amax_dx else None
    r.dy, r.lddy, r.dx, r.lddx = dy.ptr, a.lddy, dx.ptr, a.lddx
    r.dx_add = dx.ptr if alias else (add.ptr if add else None)
    r.ldadd = a.lddx if alias else a.ldadd
    r.dx_add2, r.ldadd2 = (add2.ptr if add2 else None), a.ldadd2
    r.dgamma, r.dbeta, r.fin = dg.ptr, db.ptr, (fin.data_ptr() if fin is not None else None)
    r.amax_dx = so.data_ptr() if so is not None else None

    def reset():
        dx.t.fill_(SENT)
        if alias:
            dx.v.copy_(dx0)
        dg.v.copy_(dg0)
        db.v.copy_(db0)
        if so is not None:
            so.zero_()

    def run():
        assert lib.dp_groupnorm_bwd(C.byref(r), S()) == 0
        if fin is not None:
            assert lib.dp_groupnorm_bwd_param(C.byref(r), S()) == 0
    got_dx, got_dg, got_db = _twice(run, reset, [dx.v, dg.v, db.v])
    assert dx.outside_untouched(), name
    x64 = x.v.double().view(N, HW, Cc).permute(0, 2, 1).clone().requires_grad_(True)
    ga = gamma.v.double().reshape(Cc).clone().requires_grad_(True)
    be = beta.v.double().reshape(Cc).clone().requires_grad_(True)
    z = F.group_norm(x64, G, ga, be, a.eps)
    out = F.silu(z) if a.silu else z
    d64 = dy.v.double().view(N, HW, Cc).permute(0, 2, 1)
    gx, gg, gb = torch.autograd.grad(out, (x64, ga, be), d64)
    with torch.no_grad():
        xh = F.group_norm(x64, G, eps=a.eps)
        zz = z.detach()
        sig = torch.sigmoid(zz)
        dyp = d64 * (sig * (1 + zz * (1 - sig))) if a.silu else d64
        mag = ga.view(1, Cc, 1).abs() * (d64.abs() * (1 + zz.abs()) if a.silu else d64.abs())
        rstd = 1 / (x64.reshape(N, G, -1).var(-1, unbiased=False) + a.eps).sqrt()            # [N][G]
        t1 = (ga.view(1, Cc, 1) * dyp).reshape(N, G, -1)
        t2 = (ga.view(1, Cc, 1) * dyp * xh).reshape(N, G, -1)
        ng = cg * HW
        e1 = lc.sum_bound(t1.pow(2).sum(-1).sqrt(), ng) / ng
        e2 = lc.sum_bound(t2.pow(2).sum(-1).sqrt(), ng) / ng
        magg = mag.reshape(N, G, -1)
        b = 2.0 ** -20 * (magg + magg.mean(-1, keepdim=True) + xh.reshape(N, G, -1).abs() * (magg * xh.reshape(N, G, -1).abs()).mean(-1, keepdim=True))
        b = rstd[..., None] * (b + e1[..., None] + xh.reshape(N, G, -1).abs() * e2[..., None])
        bound = b.reshape(N, Cc, HW).permute(0, 2, 1).reshape(rows, Cc)
        ref = gx.permute(0, 2, 1).reshape(rows, Cc)
        for extra in ((dx0 if alias else None), (add.v if add else None), (add2.v if add2 else None)):
            if extra is not None:
                ref = ref + extra.double()
                bound = bound + 2 * lc.U * extra.double().abs()
        tag = f"N {N} HW {HW} C {Cc} G {G} silu {a.silu} add {bool(a.dx_add)} add2 {bool(a.dx_add2)} fin {bool(a.fin)}"
        _check(rep, name, got_dx, ref, bound, tag)
        sg = (dyp * xh).permute(0, 2, 1).reshape(rows, Cc)
        sb = dyp.permute(0, 2, 1).reshape(rows, Cc)
        _check(rep, name, got_dg, dg0.double() + gg, lc.sum_bound(sg.pow(2).sum(0).sqrt(), rows) + 2 * lc.U * (dg0.double().abs() + gg.abs()), tag + " dgamma")
        _check(rep, name, got_db, db0.double() + gb, lc.sum_bound(sb.pow(2).sum(0).sqrt(), rows) + 2 * lc.U * (db0.double().abs() + gb.abs()), tag + " dbeta")
    if so is not None:
        assert _slot_value(so) == float(got_dx.abs().max()), name


def replay_colsum(lib, g, name, args, rep):
    """out[s][c] (=|+=) sum of seg_rows rows of x: sum_bound over seg_rows terms, one rounding of the old value."""
    xp, ld, rows, cols, seg, op, ld_out, acc = args
    x = Buf(xp, rows, ld, cols, 3.0)
    x.v.copy_(_randn(g, rows, cols))
    nseg = rows // seg
    out = Buf(op, nseg, ld_out, cols)
    o0 = _randn(g, nseg, cols)

    def reset():
        out.t.fill_(SENT)
        out.v.copy_(o0)

    def run():
        assert lib.dp_colsum(x.ptr, ld, rows, cols, seg, out.ptr, ld_out, acc, S()) == 0
    got, = _twice(run, reset, [out.v])
    assert out.outside_untouched(), name
    xs = x.v.double().view(nseg, seg, cols)
    ref = xs.sum(1) + (o0.double() if acc else 0)
    _check(rep, name, got, ref, lc.sum_bound(xs.pow(2).sum(1).sqrt(), seg) + 2 * lc.U * (o0.double().abs() if acc else 0), f"{rows}x{cols} seg {seg}")


def _positive_sum_check(rep, name, got, terms, scale, what):
    ref = scale * terms.sum()
    b = abs(scale) * lc.sum_bound(terms.pow(2).sum().sqrt(), terms.numel()) + 2 * lc.U * ref.abs()
    _check(rep, name, got.double().reshape(()), ref, b, what)


def replay_mse(lib, g, name, args, rep):
    """loss = scale_loss sum (pred - target)^2 (sum_bound over n terms, the final scaling one rounding), grad = scale_grad (pred -
    target) (two roundings)."""
    _, _, _, n, sl, sg, _, _ = args
    pred, tgt = _randn(g, n), _randn(g, n)
    grad = torch.full((n + 4,), SENT, device="cuda")
    partial = torch.empty(max(1, lib.dp_mse_partials(n)), device="cuda")
    loss = torch.zeros(1, device="cuda")

    def run():
        assert lib.dp_mse_loss_grad(pred.data_ptr(), tgt.data_ptr(), grad.data_ptr(), n, sl, sg, partial.data_ptr(), loss.data_ptr(), S()) == 0
    got_g, got_l = _twice(run, lambda: grad.fill_(SENT), [grad[:n], loss])
    assert bool((grad[n:] == SENT).all()), name
    d = pred.double() - tgt.double()
    _check(rep, name, got_g, sg * d, 2.0 ** -22 * (sg * d).abs(), f"n {n} grad")
    _positive_sum_check(rep, name, got_l, d * d, sl, f"n {n} loss")


def replay_sumsq(lib, g, name, args, rep):
    _, n, _, _ = args
    x = _randn(g, n)
    partial = torch.empty(max(1, lib.dp_sumsq_partials(n)), device="cuda")
    out = torch.zeros(1, device="cuda")

    def run():
        assert lib.dp_sumsq(x.data_ptr(), n, partial.data_ptr(), out.data_ptr(), S()) == 0
    got, = _twice(run, lambda: out.zero_(), [out])
    _positive_sum_check(rep, name, got, x.double() ** 2, 1.0, f"n {n}")


def replay_adam(lib, g, name, a, rep):
    """Clip + Adam + EMA (torch.optim.Adam's op order, optim.cu) against the same formulas in fp64 on the same fp32 scalars.  Bound:
    the moments a few roundings each (2^-21 relative to their terms), the step 2^-19 relative to the update (the division, square
    root and the moments' errors), one rounding of each parameter and EMA value."""
    from diff_pruning_b200 import _lib as L
    n = a.n
    p0, gr, m0, v0, e0 = _randn(g, n), _randn(g, n, scale=1e-3), _randn(g, n, scale=1e-4), _randn(g, n, scale=1e-8).abs(), _randn(g, n)
    p, m, v, e = p0.clone(), m0.clone(), v0.clone(), e0.clone()
    r = L.AdamArgs()
    r.n, r.max_norm, r.lr, r.beta1, r.beta2, r.eps, r.ema_decay, r.step, r.grad_scale = (
        n, a.max_norm, a.lr, a.beta1, a.beta2, a.eps, a.ema_decay, a.step, a.grad_scale)
    r.p, r.g, r.m, r.v = p.data_ptr(), gr.data_ptr(), m.data_ptr(), v.data_ptr()
    r.ema = e.data_ptr() if a.ema else None
    ss = (gr.double() ** 2).sum().float().reshape(1).cuda()
    r.sumsq = ss.data_ptr() if a.sumsq else None
    scal = torch.tensor([a.lr / (1 - a.beta1 ** 3), math.sqrt(1 - a.beta2 ** 3)], dtype=torch.float32).cuda()
    r.step_scalars = scal.data_ptr() if a.step_scalars else None

    def reset():
        for t, t0 in ((p, p0), (m, m0), (v, v0), (e, e0)):
            t.copy_(t0)

    def run():
        assert lib.dp_adam_clip_ema(C.byref(r), S()) == 0
    gp, gm, gv, ge = _twice(run, reset, [p, m, v, e])
    f32 = lambda z: float(torch.tensor(z, dtype=torch.float32))
    clip = 1.0
    if a.sumsq:
        tot = math.sqrt(float(ss)) * f32(a.grad_scale)
        clip = min(1.0, f32(a.max_norm) / (tot + 1e-6))
    if a.step_scalars:
        step_size, bc2 = float(scal[0]), float(scal[1])
    else:
        step_size, bc2 = f32(a.lr / (1 - a.beta1 ** a.step)), f32(math.sqrt(1 - a.beta2 ** a.step))
    # the derived constants are formed in double on the host and rounded once to fp32 (dp_adam_args), as torch's Python scalars are
    w1, w2, b2, eps, d, d1 = f32(1 - a.beta1), f32(1 - a.beta2), f32(a.beta2), f32(a.eps), f32(a.ema_decay), f32(1 - a.ema_decay)
    G64 = gr.double() * f32(a.grad_scale) * clip
    M = m0.double() + w1 * (G64 - m0.double())
    V = v0.double() * b2 + w2 * G64 ** 2
    denom = V.sqrt() / bc2 + eps
    upd = step_size * M / denom
    P = p0.double() - upd
    bM = 2.0 ** -21 * (m0.double().abs() * (1 + w1) + w1 * G64.abs())
    tag = f"n {n} clip {a.sumsq is not None} ema {a.ema is not None}"
    _check(rep, name, gm, M, bM, tag + " m")
    _check(rep, name, gv, V, 2.0 ** -21 * (v0.double().abs() + w2 * G64 ** 2), tag + " v")
    bp = 2.0 ** -19 * upd.abs() + step_size * bM / denom + 2.0 ** -23 * (P.abs() + p0.double().abs())   # m's error carries into the step
    _check(rep, name, gp, P, bp, tag + " p")
    if a.ema:
        E = d1 * P + d * e0.double()
        _check(rep, name, ge, E, 2.0 ** -22 * (d1 * P.abs() + d * e0.double().abs()) + d1 * bp, tag + " ema")


def replay_silu(lib, g, name, args, rep):
    """SiLU forward / backward (flat): the special-function sigmoid ~3e-7 relative, two more roundings: 2^-20 of the magnitudes."""
    if name == "dp_silu_fwd":
        _, _, n = args
        x, y = _randn(g, n, scale=3.0), torch.full((n + 4,), SENT, device="cuda")

        def run():
            assert lib.dp_silu_fwd(x.data_ptr(), y.data_ptr(), n, S()) == 0
        got, = _twice(run, lambda: y.fill_(SENT), [y[:n]])
        ref = F.silu(x.double())
        _check(rep, name, got, ref, 2.0 ** -20 * x.double().abs(), f"n {n}")
    else:
        _, _, _, n, acc = args
        x, dy, d0 = _randn(g, n, scale=3.0), _randn(g, n), _randn(g, n)
        dx = torch.full((n + 4,), SENT, device="cuda")

        def reset():
            dx.fill_(SENT)
            dx[:n].copy_(d0)

        def run():
            assert lib.dp_silu_bwd(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), n, acc, S()) == 0
        got, = _twice(run, reset, [dx[:n]])
        x64 = x.double()
        sig = torch.sigmoid(x64)
        ref = dy.double() * sig * (1 + x64 * (1 - sig)) + (d0.double() if acc else 0)
        _check(rep, name, got, ref, 2.0 ** -20 * dy.double().abs() * (1 + x64.abs()) + (2 * lc.U * d0.double().abs() if acc else 0), f"n {n} acc {acc}")
    assert bool(((y if name == "dp_silu_fwd" else dx)[n:] == SENT).all()), name


def replay_temb(lib, g, name, args, rep):
    """Sinusoidal timestep embedding: the argument t * f is one fp32 product (its rounding, 2^-24 |t f|, is part of the op), sin / cos
    then a few ulp: 2^-21 + 2^-23 |t f| absolute."""
    _, _, _, B, half, flip = args
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    fr = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half).cuda()
    out = torch.full((B * 2 * half + 4,), SENT, device="cuda")

    def run():
        assert lib.dp_timestep_embedding(t.data_ptr(), fr.data_ptr(), out.data_ptr(), B, half, flip, S()) == 0
    got, = _twice(run, lambda: out.fill_(SENT), [out[:B * 2 * half]])
    arg = t.double()[:, None] * fr.double()[None]
    s_, c_ = arg.sin(), arg.cos()
    ref = torch.cat([c_, s_] if flip else [s_, c_], 1).reshape(-1)
    bnd = (2.0 ** -21 + 2.0 ** -23 * arg.abs()).repeat(1, 2).reshape(-1)
    _check(rep, name, got, ref, bnd, f"B {B} half {half} flip {flip}")


def replay_add_noise(lib, g, name, args, rep):
    """x_t = sqrt(acp[t]) x0 + sqrt(1 - acp[t]) eps, NCHW in, NHWC view out: a few roundings, 2^-21 of the two terms."""
    _, _, _, _, op, B, Cc, H, W, nhwc, ld_out = args
    x0, nz = _randn(g, B, Cc, H, W), _randn(g, B, Cc, H, W)
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    acp = torch.linspace(0.9999, 0.005, 1000).cuda()
    ld = ld_out or Cc
    out = Buf(op, B * H * W, ld, Cc) if nhwc else Buf(op, B * Cc * H * W, 1, 1)

    def run():
        assert lib.dp_add_noise(x0.data_ptr(), nz.data_ptr(), t.data_ptr(), acp.data_ptr(), out.ptr, B, Cc, H, W, nhwc, ld_out, S()) == 0
    got, = _twice(run, lambda: out.t.fill_(SENT), [out.v])
    assert out.outside_untouched(), name
    a_ = acp.double()[t].sqrt().view(B, 1, 1, 1)
    b_ = (1 - acp.double()[t]).sqrt().view(B, 1, 1, 1)
    ref, mag = a_ * x0.double() + b_ * nz.double(), a_ * x0.double().abs() + b_ * nz.double().abs()
    if nhwc:
        ref, mag = _nhwc_rows(ref), _nhwc_rows(mag)
    else:
        ref, mag = ref.reshape(-1, 1), mag.reshape(-1, 1)
    _check(rep, name, got, ref, 2.0 ** -21 * mag, f"B {B} C {Cc} {H}x{W}")


def replay_upsample_bwd(lib, g, name, args, rep):
    """dx (=|+=) sum of the 2x2 children of dy: sum_bound over 4 (5) terms."""
    dyp, lddy, dxp, lddx, N, H, W, Cc, acc = args
    dy = Buf(dyp, N * 4 * H * W, lddy, Cc, 3.0)
    dy.v.copy_(_randn(g, N * 4 * H * W, Cc))
    dx = Buf(dxp, N * H * W, lddx, Cc)
    d0 = _randn(g, N * H * W, Cc)

    def reset():
        dx.t.fill_(SENT)
        dx.v.copy_(d0)

    def run():
        assert lib.dp_upsample2x_bwd(dy.ptr, lddy, dx.ptr, lddx, N, H, W, Cc, acc, S()) == 0
    got, = _twice(run, reset, [dx.v])
    assert dx.outside_untouched(), name
    ch = dy.v.double().view(N, H, 2, W, 2, Cc)
    ref = ch.sum((2, 4)).reshape(-1, Cc) + (d0.double() if acc else 0)
    s2 = ch.pow(2).sum((2, 4)).reshape(-1, Cc) + (d0.double() ** 2 if acc else 0)
    _check(rep, name, got, ref, lc.sum_bound(s2.sqrt(), 5), f"{N}x{H}x{W}x{Cc} acc {acc}")


# ---------------------------------------------------------------------------------------------------- exact ops: checked with torch.equal
def _exact(rep, name, got, ref, what):
    rep.setdefault(name, []).append(0.0)
    assert torch.equal(got, ref), f"{name} {what}: not bit-exact"


def replay_exact(lib, g, name, args, rep):
    """Data movement, layout conversion, rounding to bf16, amax, zeroing and weight packing: their results are exact, so the replay
    asserts equality (and that nothing around the written view changed)."""
    fn = getattr(lib, name)
    if name == "dp_amax":
        xp, ld, rows, cols, _ = args
        x = Buf(xp, rows, ld, cols, 1e30)
        x.v.copy_(_scaled(g, rows, cols))
        slot = torch.zeros(1, dtype=torch.int32, device="cuda")
        _twice(lambda: fn(x.ptr, ld, rows, cols, slot.data_ptr(), S()), lambda: slot.zero_(), [slot])
        _exact(rep, name, slot.view(torch.float32).cpu(), x.v.abs().max().reshape(1).cpu(), f"{rows}x{cols}")
    elif name == "dp_zero_u32":
        _, n = args
        t = torch.full((n + 4,), 7, dtype=torch.int32, device="cuda")
        assert fn(t.data_ptr(), n, S()) == 0
        _exact(rep, name, t, torch.cat([torch.zeros(n, dtype=torch.int32), torch.full((4,), 7, dtype=torch.int32)]).cuda(), f"n {n}")
    elif name == "dp_cvt_bf16":
        sp, ld, rows, Cc, dp_, ldd = args
        src = Buf(sp, rows, ld, Cc, 3.0)
        src.v.copy_(_scaled(g, rows, Cc))
        dst = Buf(dp_, rows, ldd, ldd, 5.0, torch.bfloat16)
        _twice(lambda: fn(src.ptr, ld, rows, Cc, dst.ptr, ldd, S()), lambda: dst.t.fill_(5.0), [dst.v])
        ref = torch.zeros(rows, ldd, dtype=torch.bfloat16, device="cuda")
        ref[:, :Cc] = src.v.bfloat16()
        _exact(rep, name, dst.v, ref, f"{rows}x{Cc}")
        assert dst.outside_untouched(), name
    elif name == "dp_copy_rows":
        ap, lda, yp, ldy, rows, cols = args
        a_ = Buf(ap, rows, lda, cols, 3.0)
        a_.v.copy_(_randn(g, rows, cols))
        y = Buf(yp, rows, ldy, cols)
        _twice(lambda: fn(a_.ptr, lda, y.ptr, ldy, rows, cols, S()), lambda: y.t.fill_(SENT), [y.v])
        _exact(rep, name, y.v, a_.v, f"{rows}x{cols}")
        assert y.outside_untouched(), name
    elif name == "dp_transpose_batched":
        _, _, b, rows, cols = args
        x, y = _randn(g, b, rows, cols), torch.full((b, cols, rows), SENT, device="cuda")
        _twice(lambda: fn(x.data_ptr(), y.data_ptr(), b, rows, cols, S()), lambda: y.fill_(SENT), [y])
        _exact(rep, name, y, x.transpose(1, 2), f"{b}x{rows}x{cols}")
    elif name == "dp_nchw_to_nhwc":
        _, op, ld, N, Cc, H, W = args
        x = _randn(g, N, Cc, H, W)
        y = Buf(op, N * H * W, ld, Cc)
        _twice(lambda: fn(x.data_ptr(), y.ptr, ld, N, Cc, H, W, S()), lambda: y.t.fill_(SENT), [y.v])
        _exact(rep, name, y.v, x.permute(0, 2, 3, 1).reshape(-1, Cc), f"{N}x{Cc}x{H}x{W}")
        assert y.outside_untouched(), name
    elif name == "dp_nhwc_to_nchw":
        ip, ld, _, N, Cc, H, W, acc = args
        x = Buf(ip, N * H * W, ld, Cc, 3.0)
        x.v.copy_(_randn(g, N * H * W, Cc))
        y0 = _randn(g, N, Cc, H, W)
        y = y0.clone()
        _twice(lambda: fn(x.ptr, ld, y.data_ptr(), N, Cc, H, W, acc, S()), lambda: y.copy_(y0), [y])
        ref = x.v.reshape(N, H, W, Cc).permute(0, 3, 1, 2)
        _exact(rep, name, y, (y0 + ref) if acc else ref.contiguous(), f"{N}x{Cc}x{H}x{W} acc {acc}")     # one fp32 add: exact as torch's
    elif name == "dp_upsample2x_fwd":
        xp, ldx, yp, ldy, N, H, W, Cc = args
        x = Buf(xp, N * H * W, ldx, Cc, 3.0)
        x.v.copy_(_randn(g, N * H * W, Cc))
        y = Buf(yp, N * 4 * H * W, ldy, Cc)
        _twice(lambda: fn(x.ptr, ldx, y.ptr, ldy, N, H, W, Cc, S()), lambda: y.t.fill_(SENT), [y.v])
        ref = x.v.reshape(N, H, 1, W, 1, Cc).expand(N, H, 2, W, 2, Cc).reshape(-1, Cc)
        _exact(rep, name, y.v, ref, f"{N}x{H}x{W}x{Cc}")
        assert y.outside_untouched(), name
    elif name == "dp_pack_conv_weight":
        _, K, Cc, R, Sx, ckp, kcp = args
        w = _randn(g, K, Cc, R, Sx)
        ck, kc = torch.full((w.numel(),), SENT, device="cuda"), torch.full((w.numel(),), SENT, device="cuda")
        assert fn(w.data_ptr(), K, Cc, R, Sx, ck.data_ptr() if ckp else None, kc.data_ptr() if kcp else None, S()) == 0
        wt = w.permute(2, 3, 1, 0).reshape(-1)             # [R][S][C][K]
        _exact(rep, name, ck if ckp else wt, wt, f"{K}x{Cc}x{R}x{Sx} ck")
        _exact(rep, name, kc if kcp else w.permute(2, 3, 0, 1).reshape(-1), w.permute(2, 3, 0, 1).reshape(-1), f"{K}x{Cc}x{R}x{Sx} kc")
    elif name == "dp_pack_conv_weight_bf16":
        _, K, Cc, R, Sx, _, _ = args
        w = _randn(g, K, Cc, R, Sx)
        Cp, Kp = lib.dp_bf16_weight_row(Cc), lib.dp_bf16_weight_row(K)
        kc = torch.full((R * Sx * K * Cp,), 5.0, device="cuda", dtype=torch.bfloat16)
        ck = torch.full((R * Sx * Cc * Kp,), 5.0, device="cuda", dtype=torch.bfloat16)
        assert fn(w.data_ptr(), K, Cc, R, Sx, kc.data_ptr(), ck.data_ptr(), S()) == 0
        rk = torch.zeros(R * Sx, K, Cp, dtype=torch.bfloat16, device="cuda")
        rk[..., :Cc] = w.permute(2, 3, 0, 1).reshape(R * Sx, K, Cc).bfloat16()
        rc = torch.zeros(R * Sx, Cc, Kp, dtype=torch.bfloat16, device="cuda")
        rc[..., :K] = w.permute(2, 3, 1, 0).reshape(R * Sx, Cc, K).bfloat16()
        _exact(rep, name, kc, rk.reshape(-1), f"{K}x{Cc}x{R}x{Sx} kc")
        _exact(rep, name, ck, rc.reshape(-1), f"{K}x{Cc}x{R}x{Sx} ck")
    else:
        raise AssertionError(f"no replay for {name}")


def _split_ok(hi, lo, slot, ref, pitch, valid):
    """The 3 x fp16 split reproduces ref to 2^-21 of its maximum, the pad columns are zero and |hi| <= 2^14.  The scale puts every
    scaled value below 2^14 (s |v| < 2^(140 - E) 2^(E - 126)), but fp16 rounds a value within 4 of 2^14 (half its spacing of 8 there) up
    to 2^14 itself: a tensor whose maximum lies within 2^-12 (relative) below a power of two has hi = 2^14 exactly, and lo' carries the
    negative remainder.  2^14 is far from fp16's overflow (65504)."""
    E = (int(slot.item()) >> 23) & 0xFF
    scale = 2.0 ** (140 - E)
    rec = ((hi.double() + lo.double() / 2048.0) / scale).view(-1, pitch)
    err = float((rec[:, :valid] - ref.double().reshape(-1, valid)).abs().max()) / float(ref.abs().max())
    return err <= 2.0 ** -21 and float(rec[:, valid:].abs().sum()) == 0.0 and float(hi.float().abs().max()) <= 2.0 ** 14, err


def replay_split(lib, g, name, args, rep):
    """dp_pack_conv_weight_tc and dp_split_h3: hi + lo' / 2^11 over the slot's scale reproduces the operand to 2^-21 of its maximum
    (22 bits kept), pads zero, and the weight's slot holds max|w| exactly."""
    if name == "dp_pack_conv_weight_tc":
        _, K, Cc, R, Sx = args[:5]
        w = _randn(g, K, Cc, R, Sx)
        Cp, Kp = lib.dp_tc_weight_row(Cc), lib.dp_tc_weight_row(K)
        packs = [torch.empty(n, device="cuda", dtype=torch.float16) for n in (R * Sx * K * Cp,) * 2 + (R * Sx * Cc * Kp,) * 2]
        slot = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
        assert lib.dp_pack_conv_weight_tc(w.data_ptr(), K, Cc, R, Sx, *[p.data_ptr() for p in packs], slot.data_ptr(), S()) == 0
        assert _slot_value(slot) == float(w.abs().max()), name
        ok1, e1 = _split_ok(packs[0], packs[1], slot, w.permute(2, 3, 0, 1), Cp, Cc)
        ok2, e2 = _split_ok(packs[2], packs[3], slot, w.permute(2, 3, 1, 0), Kp, K)
        rep.setdefault(name, []).append(max(e1, e2) / 2.0 ** -21)
        assert ok1 and ok2, (name, e1, e2)
    else:
        xp, ld, bs, b, rows, cols, tr = args[:7]
        x = _strided(xp, (b, rows, cols), (bs, ld, 1), 3.0, g)[1]
        slot = torch.zeros(1, dtype=torch.int32, device="cuda")
        for i in range(b):
            assert lib.dp_amax(x[i].data_ptr(), ld, rows, cols, slot.data_ptr(), S()) == 0
        n8 = (cols + 7) // 8 * 8 if not tr else (rows + 7) // 8 * 8
        hi, lo = (torch.empty(b * (rows if not tr else cols) * n8, device="cuda", dtype=torch.float16) for _ in range(2))
        assert lib.dp_split_h3(x.data_ptr(), ld, bs, b, rows, cols, tr, slot.data_ptr(), hi.data_ptr(), lo.data_ptr(), S()) == 0
        ref = x.transpose(1, 2) if tr else x
        ok, e = _split_ok(hi, lo, slot, ref, n8, cols if not tr else rows)
        rep.setdefault(name, []).append(e / 2.0 ** -21)
        assert ok, (name, e)


REPLAY_MORE = {
    "dp_groupnorm_bwd": replay_groupnorm_bwd, "dp_groupnorm_bwd_param": replay_groupnorm_bwd,
    "dp_colsum": replay_colsum, "dp_mse_loss_grad": replay_mse, "dp_sumsq": replay_sumsq, "dp_adam_clip_ema": replay_adam,
    "dp_silu_fwd": replay_silu, "dp_silu_bwd": replay_silu, "dp_timestep_embedding": replay_temb, "dp_add_noise": replay_add_noise,
    "dp_upsample2x_bwd": replay_upsample_bwd,
    "dp_pack_conv_weight_tc": replay_split, "dp_split_h3": replay_split,
    **{k: replay_exact for k in ("dp_amax", "dp_zero_u32", "dp_cvt_bf16", "dp_copy_rows", "dp_transpose_batched", "dp_nchw_to_nhwc",
                                 "dp_nhwc_to_nchw", "dp_upsample2x_fwd", "dp_pack_conv_weight", "dp_pack_conv_weight_bf16")},
}
REPLAY.update(REPLAY_MORE)


# ---------------------------------------------------------------------------------------------------------------------- plans
def _inputs(b, hw):
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)
    return torch.randn(b, 3, hw, hw, generator=g1).cuda(), torch.randn(b, 3, hw, hw, generator=g2).cuda()


def _scoring_pass(model, B, hw, **kw):
    from diff_pruning_b200.scoring import TaylorScorer

    def run():
        clean, noise = _inputs(B, hw)
        TaylorScorer(model, clean, noise, use_graph=False, **kw).step(500)
    return run


def _finetune_pass(model, compute):
    from diff_pruning_b200.scoring import FinetuneStepper

    def run():
        g = torch.Generator().manual_seed(11)
        clean, noise = torch.randn(8, 3, 32, 32, generator=g), torch.randn(8, 3, 32, 32, generator=g)
        FinetuneStepper(model, use_graph=False, compute=compute).step(clean.cuda(), noise.cuda(), torch.arange(8) * 100)
    return run


def _config(tag):
    import diff_pruning_b200 as dp
    from diff_pruning_b200 import ldm
    if tag == "C1 b128":
        torch.manual_seed(0)
        return _scoring_pass(dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval().cuda(), 128, 32)
    if tag == "C3 b4":
        torch.manual_seed(0)
        return _scoring_pass(dp.UNet2DModel(**dp.LSUN256_DDPM_CONFIG).eval().cuda(), 4, 256)
    if tag == "C5 b6":
        m, cfg = lc.c5_model()
        ctx = torch.randn(6, 1, cfg["context_dim"], generator=torch.Generator().manual_seed(9)).cuda()
        return _scoring_pass(m.cuda(), 6, 64, alphas_cumprod=ldm.ldm_alphas_cumprod(), context=ctx)
    from test_unet_gpu import _pruned_c1
    return _finetune_pass(_pruned_c1().train(), "bf16" if tag.endswith("bf16") else "fp32")


@pytest.mark.parametrize("tag", ["C1 b128", "C3 b4", "C5 b6", "pruned C1 finetune fp32", "pruned C1 finetune bf16"])
def test_launch_census(lib, tag):
    run = _config(tag)
    calls = _capture(lib, run)
    del run
    gc.collect()              # the plan and its model form a reference cycle
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    missing = kinds - set(REPLAY) - set(INSIDE)
    assert not missing, f"{tag}: launch kinds without a replay: {sorted(missing)}"
    uniq = _unique(calls)
    rep, count, failures = {}, {}, []
    g = torch.Generator().manual_seed(2024)
    for name, args in uniq:
        if name in INSIDE:
            continue
        count[name] = count.get(name, 0) + 1
        try:
            REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:          # report every failing launch of the config, not just the first
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print(f"  FAIL {tag}: {f}")
    assert not failures, f"{tag}: {len(failures)} launches failed their checks"
    assert set(rep) == kinds, (tag, sorted(kinds - set(rep)))     # every kind the plan issued was checked
    print(f"\n{tag}: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds, all replayed")
    for name in sorted(rep):
        n = count.get(name, len(rep[name]))
        print(f"  {tag:24s} {name:26s} {n:4d} unique, worst err/bound {max(rep[name]):.3f}")
