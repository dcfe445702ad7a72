"""The GroupNorm dropout of the finetune on the GPU, against the host restatement of its keep-mask (tests/dropout_mask.py).

Op level: dp_groupnorm_fwd / dp_groupnorm_bwd with dropout on every kernel path of test_ops_gpu.py's GN_CASES, element by element and
bit for bit: the forward is the p = 0 forward times the restated keep scale, its bf16 operand that value rounded to nearest even, and
the backward is the p = 0 backward of dy times the same factor (the kernel applies it with an uncontracted multiply, so no check here
needs an ulp of slack).  Plan level: the dropout-0.1 finetune plans (TINY, C1, pruned C1 at 0.3; fp32-grade and bf16 tiers) give every
dropout launch its own seed and draw the restated masks; graph replay equals eager mode; and one / two FinetuneStepper steps match
oracle/unet_oracle.py in float64 fed the restated masks.

Not covered: under the reference's set_dropout the attention output projection drops too (Attention.to_out[1]); the engine fuses
to_out[0] with the residual and applies no dropout there, so these tests set only ResnetBlock2D.dropout.p."""
import ctypes as C

import numpy as np
import pytest
import torch

import dropout_mask as dm
from conftest import rel_err, worst_grad_err
from test_ops_gpu import GN_CASES, S, lib  # noqa: F401  (lib: the module-scoped fixture)

pytestmark = pytest.mark.gpu

SEED, SEED_DEV = 0x0123456789ABCDEF, 987654321


def L_():
    from diff_pruning_b200 import _lib as L
    return L


def _amax(slot):
    return slot.view(torch.float32).item()


def _scale_nhwc(seed, p, N, HW, Cc):
    return torch.from_numpy(dm.scale_nhwc(seed, p, N, HW, Cc)).cuda()


class _Buf:
    """A NaN-filled [N][HW][ld] buffer with a [.., C] view at element offset `off`; untouched() checks every element outside the view."""

    def __init__(self, N, HW, Cc, ld, off, dtype=torch.float32, fill=float("nan")):
        self.t = torch.full((N * HW * ld + off + 8,), fill, device="cuda", dtype=dtype)
        self.Cc, self.ld, self.off, self.rows = Cc, ld, off, N * HW
        self.mask = torch.ones_like(self.t, dtype=torch.bool)
        self.mask[off:off + self.rows * ld].view(self.rows, ld)[:, :Cc] = False

    @property
    def ptr(self):
        return self.t.data_ptr() + self.off * self.t.element_size()

    def view(self):
        return self.t[self.off:self.off + self.rows * self.ld].view(self.rows, self.ld)[:, :self.Cc]

    def untouched(self):
        return bool(torch.isnan(self.t[self.mask].float()).all())


def _pitches(Cc, phase):
    """(ldy, y offset, lddy, dy offset, lddx, dx offset) in floats: three different pitches; phase 0 keeps every view 16-byte aligned
    (the float4 kernels stay eligible), phase 1 moves the views off 16 bytes (the scalar kernels)."""
    c4 = (Cc + 3) // 4 * 4
    return c4 + 12, 4 + phase, c4 + 20, 8 + phase, c4 + 4, 4 + 2 * phase


@pytest.mark.parametrize("phase", [0, 1])
@pytest.mark.parametrize("out", ["y", "bf16", "both"])
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("N,H,W,Cc,G,silu,ldx", GN_CASES)
def test_groupnorm_dropout_vs_restatement(lib, N, H, W, Cc, G, silu, ldx, p, out, phase):
    L = L_()
    HW = H * W
    g = torch.Generator().manual_seed(Cc + H + int(10 * p))
    xb = (torch.randn(N, HW, Cc + ldx, generator=g) * 1.5 + 0.3).cuda()
    x_before = xb.clone()
    gm, bt = (torch.randn(Cc, generator=g) * 0.5 + 1).cuda(), torch.randn(Cc, generator=g).cuda()
    stats = torch.empty(2 * N * G, device="cuda")
    ws = torch.empty(lib.dp_groupnorm_workspace_bytes(N, HW, Cc, G) // 4 + 64, device="cuda")
    a = L.GnArgs()
    a.N, a.HW, a.C, a.G, a.eps, a.silu = N, HW, Cc, G, 1e-6, silu
    a.x, a.ldx = xb.data_ptr() + 4 * ldx, Cc + ldx
    a.gamma, a.beta, a.mean, a.rstd, a.workspace = gm.data_ptr(), bt.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * N * G, ws.data_ptr()
    ldy, oy, lddy, ody, lddx, odx = _pitches(Cc, phase)
    y0 = _Buf(N, HW, Cc, ldy, oy)
    a.y, a.ldy = y0.ptr, ldy
    assert lib.dp_groupnorm_fwd(C.byref(a), S()) == 0
    ref_y0 = y0.view().clone()
    k = _scale_nhwc(dm.combined_seed(SEED, SEED_DEV), p, N, HW, Cc).view(N * HW, Cc)
    expect = ref_y0 * k                       # fp32(y_p0 * scale); +-0 where dropped, as the kernel's multiply by 0
    seed_dev = torch.tensor([SEED_DEV], device="cuda", dtype=torch.int64)
    slot = torch.zeros(1, device="cuda", dtype=torch.int32)
    a.dropout_p, a.amax_y = p, slot.data_ptr()
    for dev in (True, False):                 # the device scalar, and the same combined seed with a NULL one
        a.dropout_seed, a.dropout_seed_dev = (SEED, seed_dev.data_ptr()) if dev else (dm.combined_seed(SEED, SEED_DEV), None)
        y = _Buf(N, HW, Cc, ldy, oy) if out in ("y", "both") else None
        yb = _Buf(N, HW, Cc, Cc + (-Cc) % 8 + 8, 8, dtype=torch.bfloat16) if out in ("bf16", "both") else None
        a.y, a.ldy = (y.ptr, ldy) if y else (None, 0)
        a.y_bf16, a.ldyb = (yb.ptr, yb.ld) if yb else (None, 0)
        slot.zero_()
        assert lib.dp_groupnorm_fwd(C.byref(a), S()) == 0
        if y:
            got = y.view()
            assert torch.equal(got, expect) and y.untouched()
            assert bool((got[k == 0] == 0).all())
        if yb:
            assert torch.equal(yb.view().view(torch.int16), expect.to(torch.bfloat16).view(torch.int16)) and yb.untouched()
        assert _amax(slot) == float(expect.abs().max())
    assert torch.equal(xb, x_before)
    kept = float((k != 0).float().mean())
    assert abs(kept - (1 - dm.threshold(p) / 65536)) < 6 * (p * (1 - p) / k.numel()) ** 0.5 + 1e-12

    # backward: dx = the p = 0 backward of dy * mask, dgamma / dbeta likewise, in the one-call form and through `fin`
    a.amax_y, a.y, a.y_bf16, a.ldy = None, y0.ptr, None, ldy
    dyb = _Buf(N, HW, Cc, lddy, ody, fill=0.0)
    dyb.view().copy_(torch.randn(N * HW, Cc, generator=g).cuda())
    dym = _Buf(N, HW, Cc, lddy, ody, fill=0.0)
    dym.view().copy_(dyb.view() * k)
    runs = {}
    for name, drop, dy in (("drop", True, dyb), ("ref", False, dym)):
        for use_fin in (False, True):
            dx = _Buf(N, HW, Cc, lddx, odx)
            dg, db = torch.zeros(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
            fin = torch.full((2 * N * Cc,), float("nan"), device="cuda")
            a.dropout_p = p if drop else 0.0
            a.dropout_seed, a.dropout_seed_dev = SEED, seed_dev.data_ptr()
            a.dy, a.lddy, a.dx, a.lddx = dy.ptr, lddy, dx.ptr, lddx
            a.dgamma, a.dbeta, a.fin, a.amax_dx = dg.data_ptr(), db.data_ptr(), fin.data_ptr() if use_fin else None, slot.data_ptr()
            slot.zero_()
            assert lib.dp_groupnorm_bwd(C.byref(a), S()) == 0
            if use_fin:
                assert bool((dg == 0).all()) and bool((db == 0).all())
                assert lib.dp_groupnorm_bwd_param(C.byref(a), S()) == 0
            assert dx.untouched() and _amax(slot) == float(dx.view().abs().max())
            runs[name, use_fin] = (dx.view().clone(), dg, db)
    for use_fin in (False, True):
        for got, ref in zip(runs["drop", use_fin], runs["ref", use_fin]):
            assert torch.equal(got, ref), use_fin
    for got, ref in zip(runs["drop", True], runs["drop", False]):
        assert torch.equal(got, ref)


def _drop_readback(y, y0):
    """Dropped elements of a forward output against its p = 0 output (elements with y_p0 == 0 read as kept)."""
    return ((y == 0) & (y0 != 0)).cpu().numpy().reshape(-1)


def test_split_tensor_parts_draw_independent_masks(lib):
    """A 2048-channel tensor run as two 1024-channel parts with the engine's part seeds (Plan.gn splits tensors wider than GN_MAX_C
    so): each part's mask, read back from y, is the restated one, and the two are independent (the statistic of test_dropout_host.py)."""
    from diff_pruning_b200.engine import Plan, _dropout_seed, dropout_layer_seed
    L = L_()
    N, HW, Cc, G, p = 2, 1024, 2 * Plan.GN_MAX_C, 32, 0.1
    cp, gp = Cc // 2, G // 2
    x = torch.randn(N, HW, Cc, device="cuda")
    gm, bt = torch.ones(Cc, device="cuda"), torch.full((Cc,), 12.0, device="cuda")     # no SiLU: y_p0 = xhat + 12 > 0 everywhere
    seed_dev = torch.tensor([_dropout_seed(4, 0)], device="cuda", dtype=torch.int64)
    drops = []
    for i in range(2):
        c0 = i * cp
        stats = torch.empty(2 * N * gp, device="cuda")
        ws = torch.empty(lib.dp_groupnorm_workspace_bytes(N, HW, cp, gp) // 4 + 64, device="cuda")
        ys = []
        for pp in (0.0, p):
            y = torch.empty(N, HW, cp, device="cuda")
            a = L.GnArgs()
            a.N, a.HW, a.C, a.G, a.eps, a.silu = N, HW, cp, gp, 1e-6, 0
            a.x, a.ldx, a.y, a.ldy = x.data_ptr() + 4 * c0, Cc, y.data_ptr(), cp
            a.gamma, a.beta = gm.data_ptr() + 4 * c0, bt.data_ptr() + 4 * c0
            a.mean, a.rstd, a.workspace = stats.data_ptr(), stats.data_ptr() + 4 * N * gp, ws.data_ptr()
            a.dropout_p, a.dropout_seed, a.dropout_seed_dev = pp, dropout_layer_seed(1, i), seed_dev.data_ptr()
            assert lib.dp_groupnorm_fwd(C.byref(a), S()) == 0
            ys.append(y)
        assert bool((ys[0] > 0).all())
        d = _drop_readback(ys[1], ys[0])
        seed = dm.combined_seed(dropout_layer_seed(1, i), int(seed_dev.item()))
        assert np.array_equal(d, ~dm.keep(seed, p, d.size))
        drops.append(d)
    q = dm.threshold(p) / 65536.0
    z, s, rate = dm.worst_coincidence_sigma(drops[0], drops[1], q, q)
    assert z < 6.0, (z, s, rate)


# ---------------------------------------------------------------------------------------------------------------------- plans
def _with_dropout(m, p=0.1):
    from diff_pruning_b200.models import ResnetBlock2D
    for mod in m.modules():
        if isinstance(mod, ResnetBlock2D):
            mod.dropout.p = p
    return m


def _net(name):
    import diff_pruning_b200 as dp
    from test_pruned_widths_host import build_pruned
    if name == "pruned C1 0.3":
        m = build_pruned("C1", 0.3)
        cfg = dp.CIFAR10_DDPM_CONFIG
    else:
        cfg = dp.TINY_TEST_CONFIG if name == "TINY" else dp.CIFAR10_DDPM_CONFIG
        torch.manual_seed(0)
        m = dp.UNet2DModel(**cfg)
    hw = 16 if name == "TINY" else 32
    return _with_dropout(m).cuda().train(), cfg, hw


def _inputs(B, hw, step):
    g = torch.Generator().manual_seed(100 + step)
    clean, noise = torch.randn(B, 3, hw, hw, generator=g), torch.randn(B, 3, hw, hw, generator=g)
    return clean, noise, (torch.arange(B) * 131 + 17 * step) % 1000


class _GnRecorder:
    """Sink of launch_census.wrap_launches: every dropout GroupNorm launch, with the forward output read back. Each launch synchronises
    the device before the next one is enqueued, so the previous launch's output is intact when it is read."""

    def __init__(self, lib):
        self.lib, self.fwd, self.bwd, self.pending = lib, [], [], None

    def __call__(self, name, args, stream):
        self.flush()
        if name in ("dp_groupnorm_fwd", "dp_groupnorm_bwd") and args[0].dropout_p > 0:
            a = args[0]
            (self.fwd if name == "dp_groupnorm_fwd" else self.bwd).append(a)
            if name == "dp_groupnorm_fwd":
                self.pending = a

    def flush(self):
        if self.pending is None:
            return
        a, self.pending = self.pending, None
        torch.cuda.synchronize()
        from diff_pruning_b200.engine import _copy_args
        rows, Cc = a.N * a.HW, a.C
        dev = int(_ptr_tensor(a.dropout_seed_dev, 1, torch.int64).item())
        if a.y:
            got = _ptr_tensor(a.y, rows * a.ldy, torch.float32).view(rows, a.ldy)[:, :Cc].clone()
        else:
            got = _ptr_tensor(a.y_bf16, rows * a.ldyb, torch.bfloat16).view(rows, a.ldyb)[:, :Cc].clone()
        # the same launch at p = 0 into fresh buffers (the plan's x, gamma and beta are intact: the plan has not run past this launch)
        r = _copy_args(a)
        y0 = torch.empty(rows, Cc, device="cuda")
        stats = torch.empty(2 * a.N * a.G, device="cuda")
        ws = torch.empty(self.lib.dp_groupnorm_workspace_bytes(a.N, a.HW, Cc, a.G) // 4 + 64, device="cuda")
        r.dropout_p, r.dropout_seed_dev, r.amax_y, r.y_bf16, r.ldyb = 0.0, None, None, None, 0
        r.y, r.ldy, r.mean, r.rstd, r.workspace = y0.data_ptr(), Cc, stats.data_ptr(), stats.data_ptr() + 4 * a.N * a.G, ws.data_ptr()
        assert self.lib.dp_groupnorm_fwd(C.byref(r), S()) == 0
        k = _scale_nhwc(dm.combined_seed(a.dropout_seed, dev), a.dropout_p, a.N, a.HW, Cc).view(rows, Cc)
        expect = y0 * k
        ok = torch.equal(got, expect) if a.y else torch.equal(got.view(torch.int16), expect.to(torch.bfloat16).view(torch.int16))
        a.checked = ok


def _ptr_tensor(ptr, n, dtype):
    """A tensor over n elements of device memory at ptr."""
    class _Cai:
        __cuda_array_interface__ = {"shape": (n,), "typestr": {torch.float32: "<f4", torch.int64: "<i8", torch.bfloat16: "<i2"}[dtype],
                                    "data": (int(ptr), False), "version": 3, "strides": None}
    t = torch.as_tensor(_Cai(), device="cuda")
    return t.view(torch.bfloat16) if dtype == torch.bfloat16 else t


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
@pytest.mark.parametrize("net", ["TINY", "C1", "pruned C1 0.3"])
def test_finetune_plan_draws_restated_masks(lib, net, compute):
    """Every dropout GroupNorm launch of one eager finetune step: one forward per ResnetBlock2D, in forward order, seeded
    dropout_layer_seed(k, 0) plus the step seed on the device, each with its own combined seed; its output, read back, is the p = 0
    output times the restated mask; the backward launches reuse the forward's p and seed; and the masks the plan drew are pairwise
    independent."""
    import launch_census as lc
    from diff_pruning_b200.engine import _dropout_seed, dropout_layer_seed
    from diff_pruning_b200.models import ResnetBlock2D
    from diff_pruning_b200.scoring import FinetuneStepper
    m, cfg, hw = _net(net)
    B = 4
    rec = _GnRecorder(lib)
    with lc.wrap_launches(lib, rec):
        st = FinetuneStepper(m, use_graph=False, compute=compute)
        clean, noise, t = _inputs(B, hw, 0)
        st.step(clean.cuda(), noise.cuda(), t.cuda())
        rec.flush()
    torch.cuda.synchronize()
    n_rb = sum(isinstance(mod, ResnetBlock2D) for mod in m.modules())
    assert len(rec.fwd) == n_rb and len(rec.bwd) == n_rb
    assert [a.dropout_seed for a in rec.fwd] == [dropout_layer_seed(k, 0) for k in range(1, n_rb + 1)]
    assert all(a.dropout_p == pytest.approx(0.1) and a.dropout_seed_dev for a in rec.fwd)
    assert all(a.checked for a in rec.fwd), [i for i, a in enumerate(rec.fwd) if not a.checked]
    assert sorted((a.dropout_seed, a.N, a.HW, a.C) for a in rec.bwd) == sorted((a.dropout_seed, a.N, a.HW, a.C) for a in rec.fwd)
    dev = _dropout_seed(1, 0)
    seeds = [dm.combined_seed(a.dropout_seed, dev) for a in rec.fwd]
    assert len(set(seeds)) == n_rb
    q = dm.threshold(0.1) / 65536.0
    n = min(1 << 20, min(a.N * a.HW * a.C for a in rec.fwd))
    drops = [~dm.keep(s, 0.1, n) for s in seeds]
    worst = max(dm.worst_coincidence_sigma(drops[i], drops[j], q, q)[0] for i in range(n_rb) for j in range(i + 1, n_rb))
    assert worst < 6.0, worst


def test_graph_replay_draws_fresh_masks_and_equals_eager():
    """Three FinetuneStepper steps on TINY with dropout 0.1, captured graph vs eager: the device seed is the step's seed every step, and
    losses, gradient norms, parameters, Adam moments and EMA are bit-identical."""
    from diff_pruning_b200.engine import _dropout_seed
    from diff_pruning_b200.scoring import FinetuneStepper
    out = {}
    for use_graph in (False, True):
        m, _, hw = _net("TINY")
        st = FinetuneStepper(m, use_graph=use_graph)
        res = []
        for step in range(3):
            clean, noise, t = _inputs(4, hw, step)
            res.append(st.step(clean.cuda(), noise.cuda(), t.cuda()).clone())
            res.append(st.sumsq.clone())
            assert int(st.plan.dropout_seed_dev.item()) == _dropout_seed(step + 1, 0)
        out[use_graph] = res + [st.param_arena.clone(), st.m.clone(), st.v.clone(), st.ema.clone()]
    for a, b in zip(out[False], out[True]):
        assert torch.equal(a, b)
    assert len({float(x) for x in out[True][0:6:2]}) == 3


def _oracle_masks(m, B, hw, step, p=0.1):
    """The restated keep scales of every ResnetBlock2D at FinetuneStepper step `step` (rank 0), NCHW float64 on the GPU, in forward
    order: the down blocks, the mid block, the up blocks (the order the plan numbers its dropout layers in)."""
    from diff_pruning_b200.engine import _dropout_seed, dropout_layer_seed
    from diff_pruning_b200.models import ResnetBlock2D
    levels = len(m.down_blocks)
    blocks = []
    for name, mod in m.named_modules():
        if isinstance(mod, ResnetBlock2D):
            part, i = name.split(".")[0], int(name.split(".")[1]) if not name.startswith("mid") else 0
            key = {"down_blocks": 0, "mid_block": 1, "up_blocks": 2}[part]
            res = hw >> {0: i, 1: levels - 1, 2: levels - 1 - i}[key]
            blocks.append(((key, i, int(name.split(".")[-1])), mod.conv1.out_channels, res))
    blocks.sort()
    masks = []
    for k, (_, Cout, res) in enumerate(blocks, start=1):
        seed = dm.combined_seed(dropout_layer_seed(k, 0), _dropout_seed(step, 0))
        sc = torch.from_numpy(dm.scale_nhwc(seed, p, B, res * res, Cout)).view(B, res, res, Cout)
        masks.append(sc.permute(0, 3, 1, 2).double().cuda())
    return masks


@pytest.mark.parametrize("net", ["TINY", "pruned C1 0.3"])
def test_finetune_step_with_dropout_vs_fp64_oracle(net):
    """One fp32-grade FinetuneStepper step with dropout 0.1 against oracle/unet_oracle.py in float64 on the GPU fed the restated masks,
    with the tolerances of test_pruned_census_gpu.py::test_pruned_finetune_step_vs_fp64_oracle (loss, gradient norm) and the per-parameter
    gradient criterion of the Taylor-pass tests."""
    from oracle import unet_oracle as orc
    from diff_pruning_b200.scoring import FinetuneStepper
    m, cfg, hw = _net(net)
    B = 8
    params = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    ac = orc.alphas_cumprod().double().cuda()
    clean, noise, t = (v.cuda() for v in _inputs(B, hw, 0))
    out = orc.unet_forward(params, cfg, orc.add_noise(ac, clean.double(), noise.double(), t), t, masks=_oracle_masks(m, B, hw, 1))
    loss_ref = (noise.double() - out).square().sum(dim=(1, 2, 3)).mean(dim=0)
    loss_ref.backward()
    gn_ref = torch.sqrt(sum((p.grad ** 2).sum() for p in params.values())).item()
    del out
    st = FinetuneStepper(m, lr=2e-4, ema_decay=0.9999, max_grad_norm=1.0, use_graph=False)
    loss = st.step(clean, noise, t).item()
    gn = float(st.sumsq.sqrt())
    print(f"\n{net}: loss {loss:.7f} (fp64 {loss_ref.item():.7f}), grad norm {gn:.6g} (fp64 {gn_ref:.6g})")
    assert loss == pytest.approx(loss_ref.item(), rel=2e-5)
    assert gn == pytest.approx(gn_ref, rel=2e-4)
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), {k: v.grad for k, v in params.items()})
    assert worst < 1e-4, worst


def test_finetune_two_steps_with_dropout_on_pruned_c1_vs_oracle():
    """Two captured FinetuneStepper steps with dropout 0.1 on C1 at ratio 0.3 (Adam, clipping, EMA) against the float64 oracle fed the
    restated masks of steps 1 and 2, with the tolerances of test_unet_gpu.py::test_finetune_two_steps_on_pruned_c1_vs_oracle."""
    from oracle import unet_oracle as orc
    from diff_pruning_b200.scoring import FinetuneStepper
    m, cfg, hw = _net("pruned C1 0.3")
    B = 8
    params = {k: v.detach().double().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    p0 = {k: v.detach().clone() for k, v in params.items()}
    ema = {k: v.detach().clone() for k, v in params.items()}
    opt = torch.optim.Adam(list(params.values()), lr=2e-4, betas=(0.9, 0.999), weight_decay=0.0, eps=1e-8)
    ac = orc.alphas_cumprod().double().cuda()
    st = FinetuneStepper(m, lr=2e-4, ema_decay=0.9999, max_grad_norm=1.0, use_graph=True)
    for step in range(2):
        clean, noise, t = (v.cuda() for v in _inputs(B, hw, step))
        l_ref, gn_ref = orc.finetune_step(params, cfg, ac, clean.double(), noise.double(), t, opt, ema,
                                          masks=_oracle_masks(m, B, hw, step + 1))
        loss = st.step(clean, noise, t)
        assert loss.item() == pytest.approx(l_ref.item(), rel=2e-5), step
        assert float(st.sumsq.sqrt()) == pytest.approx(gn_ref.item(), rel=2e-4), step
    e = st.ema_state()
    lr, steps = 2e-4, 2
    for k, p in m.named_parameters():
        ref, ours = params[k].detach().double().cpu(), p.detach().cpu().double()
        upd = (ref - p0[k].double().cpu()).norm().item()
        if upd < 1e-2 * lr * steps * ref.numel() ** 0.5:
            assert (ours - ref).abs().max().item() <= 1e-2 * lr * steps, k
            continue
        assert (ours - ref).norm().item() <= 3e-2 * upd + 1e-12, (k, (ours - ref).norm().item(), upd)
        if p.dim() >= 2:
            assert rel_err(p, params[k]) < 1e-4, k
        assert rel_err(e[k], ema[k]) < 1e-4 or (e[k].cpu().double() - ema[k].double().cpu()).norm().item() <= 3e-2 * upd, k
