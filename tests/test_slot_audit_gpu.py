"""Amax-slot audit over one instance of every plan kind (slot_audit.py): each plan is built and run eagerly with every launch wrapped, and
before every launch that reads an input slot the slot is compared with max|.| over the view the launch's own arguments describe.

Per plan: every launch naming an input slot was audited (launches flagged DP_CONV_FORCE_SIMT read none and are only counted), no slot
is below its operand's maximum, and the worst looseness slot / max is at most 2^16.  Argument for 2^16: a slot filled by the writer of
exactly the tensor a launch reads is exact (looseness 1); a slot shared by the channel slices of one buffer, or the maximum over the
steps of a sampling loop, is loose by the spread of those maxima; the constant-1 slot of softmax probabilities (the P v product) is loose
by up to T <= 4096 = 2^12 over a row whose probabilities are uniform.  Four more octaves of room are kept; a bound further off than that
comes from another tensor or a stale pass and costs the 3 x fp16 split its low bits.  The worst looseness of each plan is printed.

The audit's self-tests: a slot equal to the maximum of a view inside a wider buffer (larger values outside the view's rows and
channels) passes and the launch runs; half that maximum raises before the library is called, so no kernel is launched.
"""
import ctypes
import gc
import math

import pytest
import torch

import launch_census as lc
import slot_audit as sa
from test_launch_census_gpu import S, _conv_weights, lib  # noqa: F401  (lib: the module-scoped fixture)

pytestmark = pytest.mark.gpu

MAX_LOOSENESS = 2.0 ** 16
FWD, GRAD = {"dp_conv2d_fprop"}, {"dp_conv2d_fprop", "dp_conv2d_dgrad", "dp_conv2d_wgrad"}
ATTN = {"dp_gemm_nt_tc", "dp_split_h3"}
_WORST = {}           # plan -> worst looseness, for the summary


# ---------------------------------------------------------------------------------------------------------------------- self-tests
def _fprop_in_a_wider_buffer(lib):
    """A 3x3 fprop (N 2, 8 x 8, C 64 -> K 64) whose x view is 64 of 96 channels starting 8 rows into its buffer; the rows before and
    after the view and the channels past it hold values 100 x larger than any inside it."""
    g = torch.Generator().manual_seed(41)
    N, H, W, Cc, K, ld, skip = 2, 8, 8, 64, 64, 96, 8
    rows = N * H * W
    buf = torch.full((skip + rows + skip, ld), 300.0, device="cuda")
    inside = torch.randn(rows, Cc, generator=g).clamp_(-3, 3).cuda()
    buf[skip:skip + rows, :Cc] = inside
    w, ck, kc, packs = _conv_weights(lib, g, K, Cc, 3, 3, True)
    y = torch.full((rows, K), -777.0, device="cuda")
    slot = torch.zeros(1, dtype=torch.int32, device="cuda")
    from diff_pruning_b200 import _lib as L
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l, a.flags, a.splits = N, H, W, Cc, H, W, K, 3, 3, 1, 1, 1, 0, 1
    a.x, a.ldx, a.y, a.ldy, a.w = buf[skip].data_ptr(), ld, y.data_ptr(), K, ck.data_ptr()
    a.w_tc_hi, a.w_tc_lo, a.amax_w = packs[0].data_ptr(), packs[1].data_ptr(), packs[4].data_ptr()
    a.amax_x = slot.data_ptr()
    return a, (buf, inside, w, ck, kc, packs, y, slot)


def _launch(lib, a):
    return lib.dp_conv2d_fprop(ctypes.byref(a), S())


def test_audit_passes_a_slot_equal_to_the_views_maximum(lib):
    a, (buf, inside, *_, y, slot) = _fprop_in_a_wider_buffer(lib)
    top = float(inside.abs().max())
    slot.view(torch.float32).fill_(top)
    audit = sa.SlotAudit(raise_now=True)
    with lc.wrap_launches(lib, audit):
        assert _launch(lib, a) == 0
    torch.cuda.synchronize()
    assert audit.audited == 1 and audit.failures == [] and audit.checks[0][0] == 1.0, (audit.audited, audit.checks)
    assert bool((y != -777.0).all()), "the audited launch did not run"
    print(f"\nin-view slot {top} (buffer maximum {float(buf.abs().max())}): passed, looseness {audit.checks[0][0]}")


def test_audit_reports_a_slot_below_the_views_maximum_before_the_launch(lib):
    a, (buf, inside, *_, y, slot) = _fprop_in_a_wider_buffer(lib)
    top = float(inside.abs().max())
    slot.view(torch.float32).fill_(top / 2)
    audit = sa.SlotAudit(raise_now=True)
    torch.cuda.synchronize()
    before = lib.dp_launch_count()
    with lc.wrap_launches(lib, audit):
        with pytest.raises(AssertionError, match=r"dp_conv2d_fprop #1 amax_x: .* below the operand's maximum"):
            _launch(lib, a)
    torch.cuda.synchronize()
    assert lib.dp_launch_count() == before and bool((y == -777.0).all()), "the launch ran although its slot was reported"
    # record mode: the violation is kept and the launch runs
    audit = sa.SlotAudit()
    with lc.wrap_launches(lib, audit):
        assert _launch(lib, a) == 0
    torch.cuda.synchronize()
    assert len(audit.failures) == 1 and lib.dp_launch_count() > before, audit.failures
    print(f"\nhalf-maximum slot reported: {audit.failures[0]}")


# ---------------------------------------------------------------------------------------------------------------------- plans
def _taylor_c1():
    import diff_pruning_b200 as dp
    from diff_pruning_b200 import engine
    from diff_pruning_b200.scoring import TaylorScorer
    from test_launch_census_gpu import _inputs
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval().cuda()
    clean, noise = _inputs(8, 32)

    def run():
        engine.AUDIT_SLOTS = True
        try:
            sc = TaylorScorer(m, clean, noise, use_graph=False)
        finally:
            engine.AUDIT_SLOTS = False
        for t in (3, 600):
            sc.step(t)
        torch.cuda.synchronize()
        log = sc.plan.audit_log
        # the engine's own audit of the same run (the planner's view of each operand) passes too
        assert len(log) > 50 and all(b >= v for b, v in log), len(log)
        return f"engine audit: {len(log)} slots, all bound their operands"
    return run


def _finetune_pruned_c1():
    from diff_pruning_b200.scoring import FinetuneStepper
    from test_unet_gpu import _pruned_c1
    m = _pruned_c1().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.1
    g = torch.Generator().manual_seed(11)
    batches = [(torch.randn(8, 3, 32, 32, generator=g).cuda(), torch.randn(8, 3, 32, 32, generator=g).cuda(), t)
               for t in (torch.arange(8) * 100, torch.arange(8) * 90 + 200)]

    def run():
        st = FinetuneStepper(m, use_graph=False, compute="fp32")
        w0 = m.conv_in.weight.detach().clone()
        for clean, noise, t in batches:
            st.step(clean, noise, t)
        torch.cuda.synchronize()
        assert st.plan.training and st.plan._n_dropout > 0
        assert not torch.equal(w0, m.conv_in.weight.detach()), "the weights did not move between the steps"
        return f"{st.plan._n_dropout} dropout layers, weights moved"
    return run


def _ddim_c1():
    import diff_pruning_b200 as dp
    from diff_pruning_b200.sampling import DDIMPipeline
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval().cuda()

    def run():
        pipe = DDIMPipeline(unet=m, scheduler=dp.DDPMScheduler(num_train_timesteps=1000))
        pipe.use_graph = False
        pipe(batch_size=8, generator=torch.Generator(device="cuda").manual_seed(0), eta=0.5, num_inference_steps=3, output_type="device")
    return run


def _ddim_sampler(family, guided):
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    from test_ldm_sampling_gpu import B0, GOLD, HW0, _c5_ld, _conds, _tiny_ld
    if family == "ldm_tiny":
        ld = _tiny_ld()
        c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
        B, shape, x_T = B0, HW0, GOLD["x_T"].cuda()
    else:
        ld, _ = _c5_ld()
        c, uc = _conds(ld, torch.tensor([25, 992]), torch.full((2,), 1000))
        B, shape, x_T = 2, [3, 64, 64], torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(21)).cuda()

    def run():
        sm = DDIMSampler(ld)
        sm.use_graph = False
        # S = 4: the uniform discretisation range(0, 1000, 1000 // S) + 1 reaches timestep 1000 (past the table) when S does not
        # divide 1000, in the reference's make_ddim_timesteps as here
        sm.sample(S=4, batch_size=B, shape=shape, conditioning=c, eta=0.5, x_T=x_T, unconditional_guidance_scale=3.0 if guided else 1.0,
                  unconditional_conditioning=uc if guided else None, generator=torch.Generator().manual_seed(3))
    return run


def _ldm_prune_scorer():
    from test_ldm_sampling_gpu import _loop, _tiny_ld
    ld = _tiny_ld()

    def run():
        sc, losses, _ = _loop(ld, 3, 2, pruner="taylor", use_graph=False, S_=4)
        assert len(losses) == 2 and bool(torch.isfinite(losses).all())
    return run


def _vq(name):
    from test_vq_decoder_gpu import _vq_f4
    from test_vq_decoder_host import vq_model
    m, h = ((_vq_f4(), torch.randn(2, 3, 64, 64) * 2e-4) if name == "f4" else
            (vq_model("tiny", n_embed=512), torch.randn(2, 3, 8, 8) * 0.01))
    m = m.cuda()
    m.use_graph = False
    m.decode_batch = 2

    def run():
        m.decode_chunk(h.cuda())
    return run


def _fid(batch, src, hw, quantize):
    from diff_pruning_b200 import fid
    from test_eval_census_gpu import _seeded_inception
    model = _seeded_inception()
    g = torch.Generator().manual_seed(13)
    x = (torch.randint(0, 256, (batch, hw[0], hw[1], 3), generator=g, dtype=torch.uint8) if src == "u8" else
         torch.randn(batch, 3, hw[0], hw[1], generator=g) * 0.6).cuda()

    def run():
        plan = fid.FeaturePlan(model, batch, src, hw, quantize=quantize, use_graph=False)
        plan.load(x)
        plan.ensure_packed()
        plan.run_eager()
        plan.run_eager()          # a second pass over the same buffers: the slots are zeroed at its start
    return run


PLANS = {
    "TaylorScorer C1 b8": (_taylor_c1, GRAD | ATTN),
    "FinetuneStepper pruned C1 fp32 dropout 0.1": (_finetune_pruned_c1, GRAD | ATTN),
    "DDIMPipeline C1 b8 eta 0.5": (_ddim_c1, FWD | ATTN),
    "DDIMSampler ldm_tiny guided": (lambda: _ddim_sampler("ldm_tiny", True), FWD),
    "DDIMSampler ldm_tiny unguided": (lambda: _ddim_sampler("ldm_tiny", False), FWD),
    "DDIMSampler cin256-v2 b2 guided": (lambda: _ddim_sampler("cin256-v2", True), FWD | ATTN),
    "DDIMSampler cin256-v2 b2 unguided": (lambda: _ddim_sampler("cin256-v2", False), FWD | ATTN),
    "LDMPruneScorer ldm_tiny taylor": (_ldm_prune_scorer, GRAD),
    "VQ-f4 decode_chunk 64x64 b2": (lambda: _vq("f4"), FWD | ATTN),
    "VQ tiny decode_chunk": (lambda: _vq("tiny"), FWD),
    "FeaturePlan u8 b50 32px": (lambda: _fid(50, "u8", (32, 32), False), FWD),
    "FeaturePlan f32 quantized b128 32px": (lambda: _fid(128, "f32", (32, 32), True), FWD),
    "FeaturePlan u8 b4 256px": (lambda: _fid(4, "u8", (256, 256), False), FWD),
}


@pytest.mark.parametrize("tag", list(PLANS))
def test_amax_slots_bound_the_views_their_launches_read(lib, tag):
    make, must = PLANS[tag]
    run = make()
    audit = sa.SlotAudit()
    with lc.wrap_launches(lib, audit):
        note = run()
        torch.cuda.synchronize()
    del run
    gc.collect()
    torch.cuda.empty_cache()
    for f in audit.failures[:10]:
        print(f"  FAIL {tag}: {f}")
    worst, where = audit.worst()
    print(f"\n{tag}: {audit.launches} launches name an input slot, {audit.audited} audited ({audit.simt} forced onto SIMT), "
          f"{len(audit.checks) + audit.zero} slots checked ({audit.zero} over all-zero operands), {len(audit.failures)} below the maximum; "
          f"kinds {sorted(audit.kinds)}")
    print(f"  worst looseness {worst:.4g} (2^{math.log2(worst) if worst > 0 else float('-inf'):.2f}) at {where}")
    if note:
        print(f"  {note}")
    _WORST[tag] = worst
    assert not audit.failures, f"{tag}: {len(audit.failures)} slots below their operand's maximum; first: {audit.failures[0]}"
    assert audit.audited > 0 and audit.audited + audit.simt == audit.launches, (audit.audited, audit.simt, audit.launches)
    assert must <= audit.kinds, f"{tag}: no audited launch of {sorted(must - audit.kinds)}"
    assert worst <= MAX_LOOSENESS, f"{tag}: looseness {worst:.4g} above 2^16 at {where}"


def test_slot_audit_summary():
    if not _WORST:
        pytest.skip("no plan audited in this session")
    tag = max(_WORST, key=_WORST.get)
    print(f"\nslot audit: {len(_WORST)} plans, largest looseness {_WORST[tag]:.4g} ({tag})")
