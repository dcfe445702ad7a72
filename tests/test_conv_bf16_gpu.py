"""bf16 tensor tier (conv_bf16.cu, bf16 wgmma): op-level parity against a torch fp32 convolution of the SAME bf16-rounded
operands (products of bf16 values are exact in fp32, so only the fp32 accumulation order differs: tolerance 2e-5 on the tensor), and
end to end — a finetune step of the engine in compute="bf16" against the oracle, with the tolerance bf16 operand rounding implies
(the reference under `--mixed_precision bf16` = torch.autocast rounds conv OUTPUTS to bf16 as well, so its own distance to fp32 is the
yardstick; both are stated in the test)."""
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
    if not lib.dp_bf16_available():
        pytest.fail("bf16 tensor tier (wgmma / TMA) not available on this device: conv_bf16.cu must run on sm_90a")
    return lib


def S():
    return torch.cuda.current_stream().cuda_stream


def bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def to_bf16_dev(lib, x_nhwc_f32, C_):
    """fp32 [rows][ld] device view -> bf16 [rows][C8] through dp_cvt_bf16."""
    rows = x_nhwc_f32.numel() // x_nhwc_f32.shape[-1]
    ld = (C_ + 7) // 8 * 8
    out = torch.full((rows, ld), 3.0, device="cuda", dtype=torch.bfloat16)
    assert lib.dp_cvt_bf16(x_nhwc_f32.data_ptr(), x_nhwc_f32.shape[-1], rows, C_, out.data_ptr(), ld, S()) == 0
    return out, ld


CASES = [
    # N, C, H, W, K, R, stride, pad
    (8, 128, 32, 32, 128, 3, 1, 1),     # C1's dominant shape
    (4, 96, 32, 32, 96, 3, 1, 1),       # pruned widths: N tile 96, K chunk tail (96 = 64 + 32)
    (4, 192, 16, 16, 179, 1, 1, 0),     # pruned attention to_q: odd N (179 -> N=192 instruction, masked store), 1x1
    (4, 179, 16, 16, 192, 1, 1, 0),     # odd GEMM-K 179: bf16 pitch 184, TMA zero fill of channels 179..191
    (16, 256, 8, 8, 256, 3, 1, 1),      # 8x8 images: two images per 128-pixel box, N tile 256
    (32, 512, 4, 4, 256, 3, 1, 1),      # 4x4 images: 8 images per box, 8 K chunks x 9 taps
    (4, 384, 16, 16, 128, 1, 1, 0),     # up-path shortcut 1x1
    (4, 512, 16, 16, 512, 3, 1, 1),     # two N tiles of 256 (LSUN widths)
    (4, 128, 32, 32, 128, 3, 2, 0),     # Downsample2D: stride 2, (0,1,0,1) zero border from TMA bounds
    (2, 128, 64, 64, 128, 3, 2, 1),     # stride 2 with pad 1
    (1, 128, 256, 256, 128, 3, 1, 1),   # LSUN-256 top level: W = 256 (two 128-pixel boxes per row)
]


@pytest.mark.parametrize("N,Cin,H,W,K,R,stride,pad", CASES)
def test_conv_bf16_fprop_dgrad_wgrad(lib, N, Cin, H, W, K, R, stride, pad):
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(N + Cin + K + R + stride)
    P, Q = H // stride, W // stride
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(K, Cin, R, R, generator=g) / math.sqrt(Cin * R * R)
    b = torch.randn(K, generator=g)
    gy = torch.randn(N, K, P, Q, generator=g)
    # reference: fp32 convolution of the bf16-rounded operands (what the tensor core computes, up to summation order)
    xr, wr = bf(x).requires_grad_(True), bf(w).requires_grad_(True)
    xin = F.pad(xr, (0, 1, 0, 1)) if (stride == 2 and pad == 0) else xr
    y_ref = F.conv2d(xin, wr, b, stride=stride, padding=pad if not (stride == 2 and pad == 0) else 0)
    assert y_ref.shape == (N, K, P, Q)
    rowadd, res = torch.randn(N, K, generator=g), torch.randn(N, K, P, Q, generator=g)
    # dgrad / wgrad references use the bf16-rounded dy
    y_ref.backward(bf(gy))
    gx_ref, gw_ref = xr.grad.float(), wr.grad.float()

    wd = w.contiguous().cuda()
    Cp, Kp = lib.dp_bf16_weight_row(Cin), lib.dp_bf16_weight_row(K)
    assert Cp % 64 == 0 and Cp >= Cin
    kc = torch.empty(R * R * K * Cp, device="cuda", dtype=torch.bfloat16)
    ck = torch.empty(R * R * Cin * Kp, device="cuda", dtype=torch.bfloat16)
    assert lib.dp_pack_conv_weight_bf16(wd.data_ptr(), K, Cin, R, R, kc.data_ptr(), ck.data_ptr(), S()) == 0
    assert torch.equal(kc.view(R * R, K, Cp)[..., :Cin].float().cpu(), bf(w).permute(2, 3, 0, 1).reshape(R * R, K, Cin))
    assert float(kc.view(R * R, K, Cp)[..., Cin:].float().abs().sum()) == 0.0

    x_nhwc = x.permute(0, 2, 3, 1).contiguous().cuda()
    xb, ldxb = to_bf16_dev(lib, x_nhwc, Cin)
    assert torch.equal(xb[:, :Cin].float().cpu(), bf(x).permute(0, 2, 3, 1).reshape(-1, Cin))
    assert float(xb[:, Cin:].float().abs().sum()) == 0.0
    ldy = K + 4
    yb = torch.full((N, P, Q, ldy), 7.0, device="cuda")
    a = L.ConvBf16Args()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K = N, H, W, Cin, P, Q, K
    a.R = a.S = R
    a.stride, a.pad_t, a.pad_l, a.splits = stride, pad, pad, 1
    a.x_bf16, a.ldx = xb.data_ptr(), ldxb
    a.out, a.ld_out = yb.data_ptr() + 16, ldy
    a.w_bf16 = kc.data_ptr()
    bd, rd, resd = b.cuda(), rowadd.cuda().contiguous(), res.permute(0, 2, 3, 1).contiguous().cuda()
    a.bias, a.rowadd, a.ld_rowadd, a.residual, a.ld_res = bd.data_ptr(), rd.data_ptr(), K, resd.data_ptr(), K
    e = L.ConvBf16Args()                  # geometry-only copy for the eligibility query (dgrad writes [.., C]: its pitch must cover C)
    C.memmove(C.byref(e), C.byref(a), C.sizeof(a))
    e.lddy, e.ld_out = (K + 7) // 8 * 8, max(ldy, Cin)
    for op in (0, 1, 2):
        assert lib.dp_conv_bf16_eligible(C.byref(e), op) == 0, op
    assert lib.dp_conv2d_fprop_bf16(C.byref(a), S()) == 0
    torch.cuda.synchronize()
    y_full = (y_ref.detach() + rowadd[:, :, None, None] + res).float()
    got = yb[..., 4:].permute(0, 3, 1, 2).cpu()
    assert rel_err(got, y_full) < 2e-5
    assert float((yb[..., :4] - 7.0).abs().sum()) == 0.0          # neighbours in the wider buffer untouched
    # accumulate epilogue
    a.flags, a.bias, a.rowadd, a.residual = 1, None, None, None
    assert lib.dp_conv2d_fprop_bf16(C.byref(a), S()) == 0
    torch.cuda.synchronize()
    assert rel_err(yb[..., 4:].permute(0, 3, 1, 2).cpu(), y_full + (y_ref.detach() - b[None, :, None, None])) < 2e-5

    # ---- dgrad
    gy_nhwc = gy.permute(0, 2, 3, 1).contiguous().cuda()
    dyb, lddyb = to_bf16_dev(lib, gy_nhwc, K)
    gxb = torch.zeros(N, H, W, Cin, device="cuda")
    d = L.ConvBf16Args()
    C.memmove(C.byref(d), C.byref(a), C.sizeof(a))
    d.flags, d.x_bf16 = 0, None
    d.dy_bf16, d.lddy, d.w_bf16 = dyb.data_ptr(), lddyb, ck.data_ptr()
    d.out, d.ld_out = gxb.data_ptr(), Cin
    assert lib.dp_conv2d_dgrad_bf16(C.byref(d), S()) == 0
    torch.cuda.synchronize()
    assert rel_err(gxb.permute(0, 3, 1, 2).cpu(), gx_ref) < 2e-5
    d.flags = 1
    assert lib.dp_conv2d_dgrad_bf16(C.byref(d), S()) == 0
    torch.cuda.synchronize()
    assert rel_err(gxb.permute(0, 3, 1, 2).cpu(), 2 * gx_ref) < 2e-5

    # ---- wgrad (split-K partials summed by the shared reduce kernel into an OIHW gradient)
    for splits in (1, 3):
        ws = torch.full((splits * K * R * R * Cin,), float("nan"), device="cuda")
        wa = L.ConvBf16Args()
        C.memmove(C.byref(wa), C.byref(a), C.sizeof(a))
        wa.flags, wa.splits, wa.out = 0, splits, None
        wa.x_bf16, wa.ldx, wa.dy_bf16, wa.lddy, wa.workspace = xb.data_ptr(), ldxb, dyb.data_ptr(), lddyb, ws.data_ptr()
        assert lib.dp_conv2d_wgrad_bf16(C.byref(wa), S()) == 0
        dw = torch.zeros(K, Cin, R, R, device="cuda")
        ra = L.WgradReduceArgs()
        ra.K, ra.C, ra.R, ra.S, ra.splits = K, Cin, R, R, splits
        ra.workspace, ra.dw = ws.data_ptr(), dw.data_ptr()
        assert lib.dp_conv2d_wgrad_reduce(C.byref(ra), S()) == 0
        torch.cuda.synchronize()
        assert not torch.isnan(dw).any()
        # the tensor core adds each K=16 product block into the fp32 accumulator with a truncating rounding; one CTA walking all
        # N*P*Q pixels (splits = 1, up to 65536 here = 4096 sequential accumulations) drifts by a few 1e-5 relative — the engine's
        # wave-aware split-K keeps the per-CTA reduction short; either way it is far below bf16 operand rounding (4e-3)
        assert rel_err(dw.cpu(), gw_ref) < (2e-5 if N * P * Q // splits <= 16384 else 2e-4), splits


def test_groupnorm_writes_the_bf16_operand(lib):
    from diff_pruning_b200 import _lib as L
    g = torch.Generator().manual_seed(5)
    N, HW, C_, G = 3, 64, 96, 32
    x = torch.randn(N, HW, C_, generator=g).cuda()
    gamma, beta = torch.randn(C_, generator=g).cuda(), torch.randn(C_, generator=g).cuda()
    y = torch.empty_like(x)
    yb = torch.zeros(N * HW, C_, device="cuda", dtype=torch.bfloat16)
    stats = torch.empty(2 * N * G, device="cuda")
    ws = torch.empty(lib.dp_groupnorm_workspace_bytes(N, HW, C_, G) // 4 + 1, device="cuda")
    a = L.GnArgs()
    a.N, a.HW, a.C, a.G, a.eps, a.silu = N, HW, C_, G, 1e-6, 1
    a.x, a.ldx, a.y, a.ldy = x.data_ptr(), C_, y.data_ptr(), C_
    a.gamma, a.beta, a.mean, a.rstd = gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * N * G
    a.workspace, a.y_bf16, a.ldyb = ws.data_ptr(), yb.data_ptr(), C_
    assert lib.dp_groupnorm_fwd(C.byref(a), S()) == 0
    torch.cuda.synchronize()
    assert torch.equal(yb.float().view(N, HW, C_), y.to(torch.bfloat16).float())
    y2 = y.clone()
    y.fill_(-1.0)
    a.y = None                         # operand only: the fp32 tensor is not written
    yb.zero_()
    assert lib.dp_groupnorm_fwd(C.byref(a), S()) == 0
    torch.cuda.synchronize()
    assert float((y + 1.0).abs().sum()) == 0.0 and torch.equal(yb.float().view(N, HW, C_), y2.to(torch.bfloat16).float())


def _oracle_step(cfg, state, clean, noise, t, autocast):
    from oracle import unet_oracle as orc
    params = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in state.items()}
    ac = orc.alphas_cumprod()
    noisy = orc.add_noise(ac, clean, noise, t)
    with torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
        out = orc.unet_forward(params, cfg, noisy, t)
    loss = (noise - out.float()).square().sum(dim=(1, 2, 3)).mean(dim=0)
    loss.backward()
    return loss.detach(), out.detach().float(), {k: v.grad for k, v in params.items()}


@pytest.mark.parametrize("cfg_name,B,hw", [("TINY_TEST_CONFIG", 8, 16), ("CIFAR10_DDPM_CONFIG", 8, 32)])
def test_bf16_tier_forward_backward_vs_oracle(lib, cfg_name, B, hw):
    """One fwd+bwd of the engine in compute='bf16' (bf16 conv / linear operands, fp32 accumulate, fp32 everywhere else) against the
    oracle in fp32 and under torch.autocast(bf16) — the reference's `--mixed_precision bf16` semantics (ddpm_train.py:255-261).
    Tolerance: eps_hat and the gradient must be as close to the fp32 result as autocast itself is (x1.5 + 2e-3 slack): bf16 operand
    rounding (2^-9 relative per element) is the only error source here, autocast additionally rounds every conv output."""
    import diff_pruning_b200 as dp
    from diff_pruning_b200.engine import get_plan
    from diff_pruning_b200.scoring import FinetuneStepper
    cfg = getattr(dp, cfg_name)
    torch.manual_seed(0)
    m = dp.UNet2DModel(**cfg).cuda().train()
    state = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(21)
    clean, noise = torch.randn(B, 3, hw, hw, generator=g), torch.randn(B, 3, hw, hw, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    l32, e32, g32 = _oracle_step(cfg, state, clean, noise, t, autocast=False)
    lac, eac, gac = _oracle_step(cfg, state, clean, noise, t, autocast=True)
    st = FinetuneStepper(m, lr=0.0, ema_decay=0.9999, max_grad_norm=None, use_graph=False, compute="bf16")   # lr 0: weights stay put
    loss = st.step(clean.cuda(), noise.cuda(), t.cuda())
    assert st.plan.compute == "bf16" and st.plan.n_bf16_convs > 10          # the tensor tier actually ran
    eps = st.plan.output_nchw().cpu()
    err_eps, ref_eps = rel_err(eps, e32), rel_err(eac, e32)
    assert err_eps < 1.5 * ref_eps + 2e-3, (err_eps, ref_eps)
    assert abs(loss.item() - l32.item()) / l32.item() < max(2e-2, 3 * abs(lac.item() - l32.item()) / l32.item())
    ours = torch.cat([p.grad.flatten().cpu() for _, p in m.named_parameters()])
    ref32 = torch.cat([g32[k].flatten() for k, _ in m.named_parameters()])
    refac = torch.cat([gac[k].float().flatten() for k, _ in m.named_parameters()])
    err_g, ref_g = rel_err(ours, ref32), rel_err(refac, ref32)
    assert err_g < 1.5 * ref_g + 2e-3, (err_g, ref_g)
    # and the fp32-grade tier on the same inputs is orders of magnitude closer (the two tiers are really different code paths)
    m2 = dp.UNet2DModel(**cfg).cuda().train()
    m2.load_state_dict(state)
    st2 = FinetuneStepper(m2, lr=0.0, ema_decay=0.9999, max_grad_norm=None, use_graph=False)
    st2.step(clean.cuda(), noise.cuda(), t.cuda())
    assert rel_err(st2.plan.output_nchw().cpu(), e32) < 1e-4 < err_eps * 10
