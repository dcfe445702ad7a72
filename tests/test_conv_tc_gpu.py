"""wgmma/TMA implicit-GEMM convolution (conv_tc.cu) vs plain torch fp32 CPU convolution.
Tolerance: the 3-product split (3 x fp16 on power-of-two-scaled operands for fprop / dgrad, 3xTF32 for wgrad) keeps 22 bits of every
operand, fp32 accumulation in registers => 1.5e-5 on the tensor."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    if not lib.dp_tc_available():
        pytest.fail("tensor-core path (wgmma/TMA) not available on this device: conv_tc.cu must run on sm_90a")
    return lib


def S():
    return torch.cuda.current_stream().cuda_stream


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().cuda()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous().cpu()


def amax_slot(lib, t, ld=None, rows=None, cols=None, ptr=None):
    """A fresh amax slot holding max|t| of a [rows][cols] view (dense tensor by default) — what engine._amax records per operand."""
    slot = torch.zeros(1, dtype=torch.int32, device="cuda")
    cols = cols or t.shape[-1]
    rows = rows or t.numel() // t.shape[-1]
    assert lib.dp_amax(ptr or t.data_ptr(), ld or t.shape[-1], rows, cols, slot.data_ptr(), S()) == 0
    return slot


def pack_tc(lib, wd, K, Cin, R):
    """fp16 hi / lo' packs of an OIHW weight in both orientations + its amax slot: (kc_hi, kc_lo, ck_hi, ck_lo, slot)."""
    Cp, Kp = lib.dp_tc_weight_row(Cin), lib.dp_tc_weight_row(K)
    packs = [torch.empty(n, device="cuda", dtype=torch.float16) for n in (R * R * K * Cp, R * R * K * Cp, R * R * Cin * Kp, R * R * Cin * Kp)]
    slot = torch.full((1,), 12345, dtype=torch.int32, device="cuda")     # stale content: the pack call resets it
    assert lib.dp_pack_conv_weight_tc(wd.data_ptr(), K, Cin, R, R, *[p.data_ptr() for p in packs], slot.data_ptr(), S()) == 0
    return packs + [slot]


def splitk_ws(lib, args, op):
    """Split-K scratch for a small-M fprop (op 0) / dgrad (op 1) launch, NaN-filled; None when the geometry does not split."""
    need = lib.dp_conv_splitk_workspace_floats(C.byref(args), op)
    if need <= 0:
        return None
    ws = torch.full((need,), float("nan"), device="cuda")
    args.workspace = ws.data_ptr()
    return ws


CASES = [
    # N, C, H, W, K, R, ld_extra_in, ld_extra_out
    (2, 64, 16, 16, 128, 3, 0, 0),
    (2, 32, 16, 16, 32, 3, 0, 0),       # BN=64 kernel, single k-chunk
    (8, 256, 4, 4, 256, 3, 0, 0),       # 4x4 images: 8 images per 128-row box, two N tiles
    (3, 96, 8, 8, 96, 3, 0, 0),         # pruned widths (96): partial N tile, 3 k-chunks; N not a multiple of the box
    (1, 128, 32, 32, 128, 3, 64, 32),   # views inside wider (concat) buffers, 32x32 (box = 4 rows x 32)
    (2, 256, 16, 16, 64, 1, 0, 0),      # 1x1 shortcut
    (4, 40, 8, 8, 200, 1, 0, 0),        # ragged channel counts (K-chunk and N-tile tails)
    (128, 512, 1, 1, 256, 1, 0, 0),     # time_emb_proj as a 1x1 conv over [B,1,1,512]
    (2, 192, 16, 16, 179, 1, 0, 1),     # pruned attention to_q: 192 -> 179 (odd N, output view with a 180-float pitch)
    (2, 179, 16, 16, 192, 1, 1, 0),     # pruned attention to_out: 179 -> 192 (odd GEMM-K: padded weight rows, 180-float pitch)
    (64, 358, 1, 1, 96, 1, 2, 0),       # pruned time_emb_proj: 358 -> 96
    # many pixel tiles: several persistent work items per CTA
    (32, 128, 32, 32, 128, 3, 0, 0),    # 256 tiles -> 128 supertiles, full N tile (64 weight rows per CTA)
    (151, 64, 8, 16, 128, 3, 0, 0),     # ODD tile count (151): the last pair's second tile lies past the batch (TMA zero fill, no store)
    (40, 256, 16, 16, 256, 3, 0, 0),    # two N tiles x 80 pixel-tile pairs
    (10, 96, 64, 64, 96, 3, 0, 0),      # pruned width 96: N = 96 instruction, 48 weight rows from each CTA
    (40, 192, 32, 32, 179, 1, 1, 1),    # odd N (179): second N tile of 51 -> N = 64 instruction, masked store; strided views
    # small-M launches that split their K loop over the idle SMs (dp_conv_splitk_workspace_floats > 0), as do several cases above
    (6, 960, 8, 8, 960, 3, 0, 0),       # LDM 8x8 level: 3 x 8 tiles, 270 stages -> 6 splits of 45
    (4, 512, 8, 8, 512, 3, 0, 0),       # LSUN 8x8 level: 2 x 4 tiles, 144 stages -> 16 splits of 9
    (16, 256, 4, 4, 512, 3, 64, 32),    # 4x4 images, views inside wider buffers
    (5, 179, 8, 8, 358, 3, 1, 2),       # pruned widths, odd pitches (scalar epilogue), last pixel tile half outside the batch
]
MUST_SPLIT = {(6, 960, 8, 960), (4, 512, 8, 512), (16, 256, 4, 512), (5, 179, 8, 358), (8, 256, 4, 256), (3, 96, 8, 96)}


@pytest.mark.parametrize("N,Cin,H,W,K,R,ldx,ldy", CASES)
def test_conv_tc_fprop_dgrad(lib, N, Cin, H, W, K, R, ldx, ldy):
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(N + Cin + K)
    pad = (R - 1) // 2
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(K, Cin, R, R, generator=g) / math.sqrt(Cin * R * R)
    b = torch.randn(K, generator=g)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y_ref = F.conv2d(xr, wr, b, padding=pad)
    rowadd, res = torch.randn(N, K, generator=g), torch.randn(N, K, H, W, generator=g)
    gy = torch.randn(N, K, H, W, generator=g)
    y_ref.backward(gy)
    wd = w.contiguous().cuda()
    C4, K4 = lib.dp_tc_weight_row(Cin), lib.dp_tc_weight_row(K)     # fp16 elements: 8-multiple up to 64 channels, 64-multiple beyond
    assert C4 >= Cin and C4 % 8 == 0 and (Cin <= 64 or C4 % 64 == 0)
    packs = pack_tc(lib, wd, K, Cin, R)
    simt_ck, simt_kc = torch.empty(w.numel(), device="cuda"), torch.empty(w.numel(), device="cuda")
    assert lib.dp_pack_conv_weight(wd.data_ptr(), K, Cin, R, R, simt_ck.data_ptr(), simt_kc.data_ptr(), S()) == 0
    # the slot holds max|w|; (hi + lo' / 2^11) / scale reproduces w to 2^-22 (rows zero-padded), scale = 2^(140 - E) keeps |hi| < 2^14
    wmax = float(w.abs().max())
    assert packs[4].view(torch.float32).item() == wmax
    E = (int(packs[4].item()) >> 23) & 0xFF
    scale = 2.0 ** (140 - E)
    for hi, lo, rows, pitch, valid, ref in ((packs[0], packs[1], K, C4, Cin, simt_kc), (packs[2], packs[3], Cin, K4, K, simt_ck)):
        rec = ((hi.double() + lo.double() / 2048.0) / scale).view(R * R, rows, pitch)
        assert float((rec[..., :valid].reshape(-1) - ref.double()).abs().max()) <= wmax * 2.0 ** -21
        assert float(rec[..., valid:].abs().sum()) == 0.0 and float(hi.float().abs().max()) < 2.0 ** 14
    xb = torch.randn(N, H, W, Cin + ldx, generator=g).cuda()
    xb[..., ldx:] = nhwc(x)
    yb = torch.full((N, H, W, K + ldy), 7.0, device="cuda")
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K = N, H, W, Cin, H, W, K
    a.R = a.S = R
    a.stride, a.pad_t, a.pad_l, a.splits = 1, pad, pad, 1
    a.x, a.ldx, a.y, a.ldy = xb.data_ptr() + 4 * ldx, Cin + ldx, yb.data_ptr() + 4 * ldy, K + ldy
    a.w, a.w_tc_hi, a.w_tc_lo, a.amax_w = simt_ck.data_ptr(), packs[0].data_ptr(), packs[1].data_ptr(), packs[4].data_ptr()
    sx = amax_slot(lib, xb, ld=Cin + ldx, rows=N * H * W, cols=Cin, ptr=xb.data_ptr() + 4 * ldx)
    a.amax_x = sx.data_ptr()
    bd, rd, resd = b.cuda(), rowadd.cuda().contiguous(), nhwc(res)
    a.bias, a.rowadd, a.ld_rowadd, a.residual, a.ld_res = bd.data_ptr(), rd.data_ptr(), K, resd.data_ptr(), K
    n0 = lib.dp_launch_count()
    assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
    torch.cuda.synchronize()
    y_full = y_ref.detach() + rowadd[:, :, None, None] + res
    assert rel_err(nchw(yb[..., ldy:]), y_full) < 1.5e-5
    assert float((yb[..., :ldy] - 7.0).abs().sum()) == 0.0          # neighbours in the wider buffer untouched
    # the same launch with the split-K scratch: K loop spread over idle SMs, fixed-order reduce -> same result to rounding, run to run identical
    ws = splitk_ws(lib, a, 0)
    assert ws is not None or (N, Cin, H, K) not in MUST_SPLIT
    assert ws is None or N * H * W <= 74 * 128                     # never when the pixel tiles alone cover half the SMs
    if ws is not None:
        y_plain = yb.clone()
        outs = []
        for _ in range(2):
            yb.fill_(7.0)
            n1 = lib.dp_launch_count()
            assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
            on_tc = (Cin + ldx) % 4 == 0 and ldx % 4 == 0           # TMA needs 16-byte aligned views; others take the SIMT kernel (1 launch)
            assert lib.dp_launch_count() - n1 == (2 if on_tc else 1)  # persistent kernel + split reduce / epilogue
            outs.append(yb.clone())
        assert torch.equal(outs[0], outs[1])
        assert rel_err(nchw(yb[..., ldy:]), y_full) < 1.5e-5 and rel_err(yb, y_plain) < 1e-5
        assert float((yb[..., :ldy] - 7.0).abs().sum()) == 0.0
        assert bool(torch.isnan(ws).all()) == (not on_tc)          # the split partial sums went through the scratch
    # same call forced onto the SIMT path agrees (and is the exact-fp32 reference on device)
    y2 = torch.zeros(N, H, W, K, device="cuda")
    a2 = L.ConvArgs()
    C.memmove(C.byref(a2), C.byref(a), C.sizeof(a))
    a2.flags, a2.y, a2.ldy = 2, y2.data_ptr(), K
    assert lib.dp_conv2d_fprop(C.byref(a2), S()) == 0
    assert rel_err(yb[..., ldy:], y2) < 1.5e-5
    # accumulate epilogue
    a.flags, a.bias, a.rowadd, a.residual = 1, None, None, None
    assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
    assert rel_err(nchw(yb[..., ldy:]), y_full + (y_ref.detach() - b[None, :, None, None])) < 1.5e-5
    # dgrad (tap-flipped fprop of dy) into a strided view, then accumulate
    gyd = nhwc(gy)
    gxb = torch.zeros(N, H, W, Cin + ldx, device="cuda")
    d = L.ConvArgs()
    C.memmove(C.byref(d), C.byref(a), C.sizeof(a))
    d.flags = 0
    d.x, d.ldx, d.y, d.ldy = gxb.data_ptr() + 4 * ldx, Cin + ldx, gyd.data_ptr(), K
    d.w, d.w_tc_hi, d.w_tc_lo = simt_kc.data_ptr(), packs[2].data_ptr(), packs[3].data_ptr()
    sdy = amax_slot(lib, gyd)
    d.amax_y = sdy.data_ptr()
    d.workspace = None
    wsd = splitk_ws(lib, d, 1)                                      # dgrad and its accumulate run split when the geometry allows
    assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0
    print("fprop err", rel_err(nchw(yb[..., ldy:]), y_full + (y_ref.detach() - b[None, :, None, None])), "dgrad err", rel_err(nchw(gxb[..., ldx:]), xr.grad))
    assert rel_err(nchw(gxb[..., ldx:]), xr.grad) < 1.5e-5
    assert float(gxb[..., :ldx].abs().sum()) == 0.0
    d.flags = 1
    assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0
    assert rel_err(nchw(gxb[..., ldx:]), 2 * xr.grad) < 1.5e-5
    # wgrad (MN-major operands, both split in-kernel), deterministic split-K + reduce into dW (+=)
    pix_chunks = max(1, N * H * W // 64)
    # the tensor core adds every K-block of products into the fp32 accumulator with a truncating rounding, so ONE CTA walking tens of
    # thousands of pixels drifts by a few 1e-5 (7.5e-5 at 32768 pixels).  The engine's wave-aware split-K does not cap a CTA's pixels (up
    # to 18752 in C1 at batch 128); test_launch_census_gpu.py replays the engine's own split counts against a chain-length-aware bound.
    # The large cases here keep a CTA at <= 8192 pixels (the small ones keep their 1 / 3 / 7-way splits incl. the trailing EMPTY split
    # of 7 over 16 chunks)
    base = max(1, -(-(N * H * W) // 8192))
    for splits in sorted({base, min(3 * base, pix_chunks), min(7 * base, pix_chunks)} if base > 1 else {1, min(3, pix_chunks), min(7, pix_chunks)}):
        ws = torch.full((splits * K * R * R * Cin,), float("nan"), device="cuda")
        wg = L.ConvArgs()
        C.memmove(C.byref(wg), C.byref(a), C.sizeof(a))
        wg.flags, wg.splits, wg.y, wg.ldy, wg.workspace, wg.amax_y = 0, splits, gyd.data_ptr(), K, ws.data_ptr(), sdy.data_ptr()
        bws = torch.full((splits * K,), float("nan"), device="cuda")      # the bias gradient falls out of the same pass over dy
        wg.bias_ws = bws.data_ptr()
        assert lib.dp_conv2d_wgrad(C.byref(wg), S()) == 0
        dw, db = torch.ones(K, Cin, R, R, device="cuda"), torch.ones(K, device="cuda")
        r = L.WgradReduceArgs()
        r.K, r.C, r.R, r.S, r.splits = K, Cin, R, R, splits
        r.workspace, r.dw, r.bias_ws, r.db = ws.data_ptr(), dw.data_ptr(), bws.data_ptr(), db.data_ptr()
        assert lib.dp_conv2d_wgrad_reduce(C.byref(r), S()) == 0
        assert rel_err(db.cpu() - 1, gy.sum((0, 2, 3))) < 1e-5, splits
        assert rel_err(dw.cpu() - 1, wr.grad) < (1.5e-5 if N * H * W // splits <= 2048 else 4e-5), splits   # longer per-CTA chains drift (see above)
        # and the SIMT path on the same problem agrees
        ws2, bws2 = torch.empty_like(ws), torch.full_like(bws, float("nan"))
        wg.flags, wg.workspace, wg.bias_ws = 2, ws2.data_ptr(), bws2.data_ptr()
        assert lib.dp_conv2d_wgrad(C.byref(wg), S()) == 0
        assert rel_err(bws2.view(splits, K).sum(0).cpu(), gy.sum((0, 2, 3))) < 1e-5
        assert rel_err(ws.view(splits, -1).sum(0), ws2.view(splits, -1).sum(0)) < (1.5e-5 if N * H * W // splits <= 2048 else 4e-5)


def test_single_pass_tf32_would_not_be_enough(lib):
    """Documents why the split is needed: hi*hi alone (what plain TF32 computes) is ~1e-3 off."""
    g = torch.Generator().manual_seed(0)
    x, w = torch.randn(4096, 256, generator=g), torch.randn(256, 256, generator=g)
    hi = lambda t: (t.view(torch.int32) + 0x1000 & ~0x1FFF).view(torch.float32)
    exact = x.double() @ w.double().t()
    one = (hi(x).double() @ hi(w).double().t())
    three = one + ((x - hi(x)).double() @ hi(w).double().t()) + (hi(x).double() @ (w - hi(w)).double().t())
    assert rel_err(one, exact) > 1e-4 and rel_err(three, exact) < 1e-6


@pytest.mark.parametrize("N,Cin,H,K", [(2, 64, 16, 64), (4, 128, 8, 96), (1, 32, 32, 160), (80, 128, 32, 128)])   # the last: pair kernel
def test_stride2_dgrad_parity_classes(lib, N, Cin, H, K):
    """Downsample2D backward (stride 2, F.pad(0,1,0,1) folded, resnet.py:213-218) as 4 tensor-core parity-class GEMMs."""
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(N + Cin)
    x = torch.randn(N, Cin, H, H, generator=g).requires_grad_(True)
    w = torch.randn(K, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)
    y = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, None, stride=2)
    gy = torch.randn_like(y)
    y.backward(gy)
    P = H // 2
    wd = w.contiguous().cuda()
    packs = pack_tc(lib, wd, K, Cin, 3)
    ck, kc = torch.empty(w.numel(), device="cuda"), torch.empty(w.numel(), device="cuda")
    assert lib.dp_pack_conv_weight(wd.data_ptr(), K, Cin, 3, 3, ck.data_ptr(), kc.data_ptr(), S()) == 0
    gyd = nhwc(gy)
    gx = torch.full((N, H, H, Cin), float("nan"), device="cuda")
    d = L.ConvArgs()
    d.N, d.H, d.W, d.C, d.P, d.Q, d.K = N, H, H, Cin, P, P, K
    d.R = d.S = 3
    d.stride, d.pad_t, d.pad_l, d.splits = 2, 0, 0, 1
    d.x, d.ldx, d.y, d.ldy = gx.data_ptr(), Cin, gyd.data_ptr(), K
    d.w, d.w_tc_hi, d.w_tc_lo, d.amax_w = kc.data_ptr(), packs[2].data_ptr(), packs[3].data_ptr(), packs[4].data_ptr()
    sdy = amax_slot(lib, gyd)
    d.amax_y = sdy.data_ptr()
    n0 = lib.dp_launch_count()
    assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0
    assert lib.dp_launch_count() - n0 == 4          # four parity-class launches, i.e. the tensor-core path was taken
    assert rel_err(nchw(gx), x.grad) < 1.5e-5
    d.flags = 1
    assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0
    assert rel_err(nchw(gx), 2 * x.grad) < 1.5e-5
    if splitk_ws(lib, d, 1) is not None:            # small grids: the classes with enough taps split their K loop (one more launch each)
        gx.fill_(float("nan"))
        d.flags = 0
        n0 = lib.dp_launch_count()
        assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0
        assert 4 < lib.dp_launch_count() - n0 <= 8
        assert rel_err(nchw(gx), x.grad) < 1.5e-5
    else:
        assert (N, Cin, H, K) != (4, 128, 8, 96)


@pytest.mark.parametrize("N,Cin,H,K,pad", [(2, 64, 16, 128, 0), (4, 128, 8, 96, 0), (1, 32, 32, 160, 1), (8, 256, 8, 256, 0), (80, 128, 32, 128, 0)])
def test_stride2_fprop_wgrad_tc(lib, N, Cin, H, K, pad):
    """Downsample2D forward + weight gradient (stride 2; pad 0 with the (0,1,0,1) border folded into TMA zero fill, or pad 1)
    on the tensor-core kernels: the activation boxes are fetched with TMA element strides (2, 2)."""
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(N + Cin + pad)
    x = torch.randn(N, Cin, H, H, generator=g)
    w = (torch.randn(K, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9)).requires_grad_(True)
    b = torch.randn(K, generator=g)
    xin = F.pad(x, (0, 1, 0, 1)) if pad == 0 else x
    y = F.conv2d(xin, w, b, stride=2, padding=pad)
    gy = torch.randn_like(y)
    y.backward(gy)
    P = H // 2
    assert y.shape[-1] == P
    wd = w.detach().contiguous().cuda()
    packs = pack_tc(lib, wd, K, Cin, 3)
    ck, kc = torch.empty(w.numel(), device="cuda"), torch.empty(w.numel(), device="cuda")
    assert lib.dp_pack_conv_weight(wd.data_ptr(), K, Cin, 3, 3, ck.data_ptr(), kc.data_ptr(), S()) == 0
    xd, gyd, bd = nhwc(x), nhwc(gy), b.cuda()
    yd = torch.full((N, P, P, K), float("nan"), device="cuda")
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K = N, H, H, Cin, P, P, K
    a.R = a.S = 3
    a.stride, a.pad_t, a.pad_l, a.splits = 2, pad, pad, 1
    a.x, a.ldx, a.y, a.ldy = xd.data_ptr(), Cin, yd.data_ptr(), K
    a.w, a.w_tc_hi, a.w_tc_lo, a.bias, a.amax_w = ck.data_ptr(), packs[0].data_ptr(), packs[1].data_ptr(), bd.data_ptr(), packs[4].data_ptr()
    sx = amax_slot(lib, xd)
    a.amax_x = sx.data_ptr()
    assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
    assert rel_err(nchw(yd), y.detach()) < 1.5e-5
    y2 = torch.empty_like(yd)                      # the SIMT path (exact fp32) agrees
    a2 = L.ConvArgs()
    C.memmove(C.byref(a2), C.byref(a), C.sizeof(a))
    a2.flags, a2.y = 2, y2.data_ptr()
    assert lib.dp_conv2d_fprop(C.byref(a2), S()) == 0
    assert rel_err(yd, y2) < 1.5e-5
    if splitk_ws(lib, a, 0) is not None:           # split-K variant of the same strided launch
        yd.fill_(float("nan"))
        assert lib.dp_conv2d_fprop(C.byref(a), S()) == 0
        assert rel_err(nchw(yd), y.detach()) < 1.5e-5 and rel_err(yd, y2) < 1.5e-5
    else:
        assert (N, Cin, H, K, pad) not in {(8, 256, 8, 256, 0), (4, 128, 8, 96, 0)}
    chunks = max(1, N * P * P // 64)
    sdy = amax_slot(lib, gyd)
    base = max(1, -(-(N * P * P) // 2048))       # keep a CTA's pixel chain short enough for the 1.5e-5 bound (tensor-core accumulation truncates)
    for splits in sorted({base, min(3 * base, chunks)}):
        ws = torch.full((splits * K * 9 * Cin,), float("nan"), device="cuda")
        wg = L.ConvArgs()
        C.memmove(C.byref(wg), C.byref(a), C.sizeof(a))
        wg.flags, wg.splits, wg.y, wg.ldy, wg.workspace, wg.bias, wg.amax_y = 0, splits, gyd.data_ptr(), K, ws.data_ptr(), None, sdy.data_ptr()
        assert lib.dp_conv2d_wgrad(C.byref(wg), S()) == 0
        dw = torch.zeros(K, Cin, 3, 3, device="cuda")
        r = L.WgradReduceArgs()
        r.K, r.C, r.R, r.S, r.splits = K, Cin, 3, 3, splits
        r.workspace, r.dw = ws.data_ptr(), dw.data_ptr()
        assert lib.dp_conv2d_wgrad_reduce(C.byref(r), S()) == 0
        assert rel_err(dw.cpu(), w.grad) < 1.5e-5


@pytest.mark.parametrize("N,H,W,Kg,Nn", [(3, 16, 16, 256, 256), (2, 16, 16, 179, 256), (2, 16, 16, 256, 179), (2, 8, 16, 64, 128)])
def test_attention_nt_gemm_tc(lib, N, H, W, Kg, Nn):
    """dp_gemm_nt_tc + dp_split_h3 (+transpose) vs torch.bmm: C = alpha * A B^T per image, and the transposed-split form."""
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(N + Kg + Nn)
    T = H * W
    A = torch.randn(N, T, Kg, generator=g)
    B = torch.randn(N, Nn, Kg, generator=g)
    ref = 0.25 * torch.bmm(A, B.transpose(1, 2))
    Ad, Bd = torch.zeros(N, T, (Kg + 3) // 4 * 4, device="cuda"), B.cuda()
    Ad[..., :Kg] = A.cuda()
    K8 = (Kg + 7) // 8 * 8
    hi, lo = (torch.empty(N * Nn * K8, device="cuda", dtype=torch.float16) for _ in range(2))
    sb = amax_slot(lib, Bd)
    scale = 2.0 ** (140 - ((int(sb.item()) >> 23) & 0xFF))

    def check_split():
        rec = ((hi.double() + lo.double() / 2048.0) / scale).view(N, Nn, K8)
        assert float((rec[..., :Kg] - Bd.double()).abs().max()) <= float(Bd.abs().max()) * 2.0 ** -21 and float(rec[..., Kg:].abs().sum()) == 0.0
    assert lib.dp_split_h3(Bd.data_ptr(), Kg, Nn * Kg, N, Nn, Kg, 0, sb.data_ptr(), hi.data_ptr(), lo.data_ptr(), S()) == 0
    check_split()
    Cd = torch.full((N, T, Nn + 4), 5.0, device="cuda")
    sa = amax_slot(lib, Ad, ld=Ad.shape[-1], rows=N * T, cols=Kg)
    a = L.GemmNtArgs()
    a.batch, a.H, a.W, a.Kg, a.N = N, H, W, Kg, Nn
    a.A, a.ld_a, a.b_hi, a.b_lo, a.C, a.ldc, a.alpha = Ad.data_ptr(), Ad.shape[-1], hi.data_ptr(), lo.data_ptr(), Cd.data_ptr(), Nn + 4, 0.25
    a.amax_a, a.amax_b = sa.data_ptr(), sb.data_ptr()
    assert lib.dp_gemm_nt_tc(C.byref(a), S()) == 0
    assert rel_err(Cd[..., :Nn].cpu(), ref) < 1.5e-5 and float((Cd[..., Nn:] - 5.0).abs().sum()) == 0.0
    # operands 2^-20 and 2^+20 times smaller / larger: the power-of-two scales keep the result bit-identical up to that factor
    for fa, fb in ((2.0 ** -20, 2.0 ** 12), (2.0 ** 20, 2.0 ** -30)):
        A2, B2 = Ad * fa, Bd * fb
        s2a, s2b = amax_slot(lib, A2, ld=A2.shape[-1], rows=N * T, cols=Kg), amax_slot(lib, B2)
        hi2, lo2 = torch.empty_like(hi), torch.empty_like(lo)
        assert lib.dp_split_h3(B2.data_ptr(), Kg, Nn * Kg, N, Nn, Kg, 0, s2b.data_ptr(), hi2.data_ptr(), lo2.data_ptr(), S()) == 0
        assert torch.equal(hi2, hi) and torch.equal(lo2, lo)
        C2 = torch.full((N, T, Nn + 4), 5.0, device="cuda")
        a2 = L.GemmNtArgs()
        C.memmove(C.byref(a2), C.byref(a), C.sizeof(a))
        a2.A, a2.b_hi, a2.b_lo, a2.C, a2.amax_a, a2.amax_b = A2.data_ptr(), hi2.data_ptr(), lo2.data_ptr(), C2.data_ptr(), s2a.data_ptr(), s2b.data_ptr()
        assert lib.dp_gemm_nt_tc(C.byref(a2), S()) == 0
        assert torch.equal(C2[..., :Nn], Cd[..., :Nn] * (fa * fb))
    # transposed split: B given as [N][Kg][Nn] (e.g. v: [tokens][inner]) -> operand [N][Nn][Kg8]
    Bt = B.transpose(1, 2).contiguous().cuda()
    assert lib.dp_split_h3(Bt.data_ptr(), Nn, Kg * Nn, N, Kg, Nn, 1, sb.data_ptr(), hi.data_ptr(), lo.data_ptr(), S()) == 0
    check_split()
    # batched transpose
    X = torch.randn(N, 70, 45, generator=g).cuda()
    Y = torch.empty(N, 45, 70, device="cuda")
    assert lib.dp_transpose_batched(X.data_ptr(), Y.data_ptr(), N, 70, 45, S()) == 0
    assert torch.equal(Y, X.transpose(1, 2))


def test_fp16_split_dynamic_range_within_one_tensor(lib):
    """The 3-product fp16 split scales every operand by ONE power of two per tensor.  Elements far below the tensor's maximum keep their
    relative precision as long as the scaled value stays a normal fp16 number (2^28 of range below the 2^14 the maximum is scaled to);
    beyond that the ABSOLUTE error stays at 2^-50 of the maximum.  dgrad of a 1x1 convolution whose dy has output channels scaled by
    2^0 / 2^-12 / 2^-24 / 2^-36: each group of input-gradient contributions is checked against fp64 on its own scale."""
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(5)
    N, H, Cin, K = 4, 16, 128, 128
    w = torch.randn(K, Cin, 1, 1, generator=g) / math.sqrt(Cin)
    gy = torch.randn(N, K, H, H, generator=g)
    scales = (0, -12, -24, -36)
    wd = w.contiguous().cuda()
    packs = pack_tc(lib, wd, K, Cin, 1)
    kc = torch.empty(w.numel(), device="cuda")
    ck = torch.empty(w.numel(), device="cuda")
    assert lib.dp_pack_conv_weight(wd.data_ptr(), K, Cin, 1, 1, ck.data_ptr(), kc.data_ptr(), S()) == 0
    worst = {}
    for e in scales:
        # only the first 32 output channels carry gradient, at scale 2^e; the rest of the tensor holds O(1) values in OTHER pixels' rows,
        # so the tensor's maximum (and with it the scale) stays O(1): zero them where the probe lives to read the probe's contribution alone
        gyp = torch.zeros_like(gy)
        gyp[:, :32] = gy[:, :32] * 2.0 ** e
        big = torch.zeros_like(gy)
        big[0, 64:, 0, 0] = 8.0                                   # one pixel keeps max|dy| = 8 whatever e is
        dyd = nhwc(gyp + big)
        ref = F.conv_transpose2d((gyp + big).double(), w.double())   # dx = dy * W for a 1x1 convolution
        ref_probe = F.conv_transpose2d(gyp.double(), w.double())
        gx = torch.full((N, H, H, Cin), float("nan"), device="cuda")
        d = L.ConvArgs()
        d.N, d.H, d.W, d.C, d.P, d.Q, d.K = N, H, H, Cin, H, H, K
        d.R = d.S = 1
        d.stride, d.pad_t, d.pad_l, d.splits = 1, 0, 0, 1
        d.x, d.ldx, d.y, d.ldy = gx.data_ptr(), Cin, dyd.data_ptr(), K
        sdy = amax_slot(lib, dyd)
        d.w, d.w_tc_hi, d.w_tc_lo, d.amax_w, d.amax_y = kc.data_ptr(), packs[2].data_ptr(), packs[3].data_ptr(), packs[4].data_ptr(), sdy.data_ptr()
        n0 = lib.dp_launch_count()
        assert lib.dp_conv2d_dgrad(C.byref(d), S()) == 0 and lib.dp_launch_count() - n0 == 1
        got = nchw(gx).double()
        assert rel_err(got, ref) < 1.5e-5
        keep = torch.ones(N, 1, H, H, dtype=torch.bool)
        keep[0, 0, 0, 0] = False                                  # the big pixel's own outputs are O(1): fp32 output rounding hides the probe there
        worst[e] = float(((got - ref_probe) * keep).norm() / (ref_probe * keep).norm())
    print("relative error of the 2^e-scaled part on its own scale:", worst)
    assert worst[0] < 1e-6 and worst[-12] < 1e-6 and worst[-24] < 1e-5     # still normal fp16 numbers after scaling: full precision (measured 1e-7, 1e-7, 2e-7)
    assert worst[-36] < 1e-2                                                  # below fp16's range: absolute error ~2^-50 of the maximum (measured 6e-4)
