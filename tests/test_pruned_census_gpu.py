"""Pruned networks at every width the reference's pruning ratios produce (the sweep of test_pruned_widths_host.py: C1 at 0.05 / 0.15 /
0.2 / 0.3 / 0.5 / 0.7, C3 at 0.3), on the GPU:

* launch census: every distinct launch of the fp32-grade and bf16 finetune plans of every C1 network at batch 128 (bench.py's batch),
  and of the C3-at-0.3 Taylor scoring pass (fused scores), fp32 / bf16 finetune and DDIM sampling at batch 4, replayed with the
  machinery of test_launch_census_gpu.py / test_eval_census_gpu.py.  Launches are deduplicated across the whole sweep;
* the amax-slot audit on the scoring passes of C1 at 0.05 / 0.7 and C3 at 0.3;
* poisoned plans: every plan buffer torch.empty hands out filled with NaN, 1e30 or 0 before the plan is built, and the results of two
  eager Taylor passes / finetune steps / DDIM steps compared bit for bit.  The census replays each launch on fresh buffers, so it
  cannot see a plan that reads memory no launch wrote; this can.  A planted-pad test shows the comparison has teeth;
* two accumulated Taylor passes and one finetune step against oracle/unet_oracle.py in float64 (on the GPU) at pruned widths.
"""
import copy
import gc

import pytest
import torch
import torch.nn.functional as F

import launch_census as lc
from conftest import max_rel, worst_grad_err
from test_eval_census_gpu import EVAL_REPLAY
from test_launch_census_gpu import INSIDE, S, _capture, lib  # noqa: F401  (lib: the module-scoped fixture)
from test_pruned_widths_host import SWEEP, build_pruned, poisoned_alloc

pytestmark = pytest.mark.gpu

C1_RATIOS = [r for f, r in SWEEP if f == "C1"]
HW = {"C1": 32, "C3": 256}
_MODELS = {}


def _model(family, ratio):
    """The host-built network of the sweep (ratio 0: unpruned), on the GPU; callers work on a deepcopy."""
    key = (family, ratio)
    if key not in _MODELS:
        _MODELS[key] = build_pruned(family, ratio).cuda()
    return _MODELS[key]


def _fresh(family, ratio):
    return copy.deepcopy(_model(family, ratio))


def _batch(B, hw, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, hw, hw, generator=g).cuda(), torch.randn(B, 3, hw, hw, generator=g).cuda()


def _cfg(family):
    import diff_pruning_b200 as dp
    return {"C1": dp.CIFAR10_DDPM_CONFIG, "C3": dp.LSUN256_DDPM_CONFIG}[family]


# ---------------------------------------------------------------------------------------------------------------------- runs
def _taylor(m, B, hw, use_graph=False, **kw):
    """Two accumulated Taylor passes (t = 7, 400) with fused scores: {loss, eps_hat, every .grad, the fused scores}."""
    from diff_pruning_b200.scoring import TaylorScorer
    clean, noise = _batch(B, hw)
    m.zero_grad(set_to_none=True)
    sc = TaylorScorer(m, clean, noise, use_graph=use_graph, fused_scores=True, **kw)
    losses = [sc.step(t).clone() for t in (7, 400)]
    out = {"loss": torch.cat(losses), "eps": sc.plan.output_nchw()}
    out.update({"grad " + k: p.grad.clone() for k, p in m.named_parameters()})
    out.update({"scores " + k: torch.cat(v) for k, v in sc.signed_scores().items()})
    return out


def _finetune(m, B, hw, compute, use_graph=False):
    """Two FinetuneStepper steps: {loss, sumsq, parameter arena, m, v, EMA}."""
    from diff_pruning_b200.scoring import FinetuneStepper
    m.train()
    st = FinetuneStepper(m, use_graph=use_graph, compute=compute)
    g = torch.Generator().manual_seed(5)
    out = {}
    for step in range(2):
        clean, noise = torch.randn(B, 3, hw, hw, generator=g).cuda(), torch.randn(B, 3, hw, hw, generator=g).cuda()
        out[f"loss {step}"] = st.step(clean, noise, (torch.arange(B) * (997 // B) + 3 * step) % 1000).clone()
        out[f"sumsq {step}"] = st.sumsq.clone()
    out.update(params=st.param_arena.clone(), m=st.m.clone(), v=st.v.clone(), ema=st.ema.clone())
    return out


def _ddim(m, B, use_graph=False):
    """Two DDIM steps (t = 999, 0) at eta 0.5 from a seeded latent: {samples}."""
    import diff_pruning_b200 as dp
    from diff_pruning_b200.sampling import DDIMPipeline
    pipe = DDIMPipeline(unet=m.eval(), scheduler=dp.DDPMScheduler(num_train_timesteps=1000))
    pipe.use_graph = use_graph
    img = pipe(batch_size=B, generator=torch.Generator(device="cuda").manual_seed(0), eta=0.5, num_inference_steps=2,
               output_type="device").images
    return {"samples": img.clone()}


# ---------------------------------------------------------------------------------------------------------------------- census
def _census_run(family, ratio, B, what):
    m = _fresh(family, ratio)
    hw = HW[family]
    if what == "scoring":
        from diff_pruning_b200.scoring import TaylorScorer

        def run():
            clean, noise = _batch(B, hw)
            TaylorScorer(m, clean, noise, use_graph=False, fused_scores=True).step(500)
    elif what == "ddim":
        def run():
            _ddim(m, B)
    else:
        from diff_pruning_b200.scoring import FinetuneStepper
        m.train()

        def run():
            clean, noise = _batch(B, hw)
            FinetuneStepper(m, use_graph=False, compute=what).step(clean, noise, torch.arange(B) * (997 // B))
    return run


CENSUS = {f"C1 {r} finetune {tier} b128": ("C1", r, 128, tier) for r in C1_RATIOS for tier in ("fp32", "bf16")}
CENSUS.update({f"C3 0.3 {w} b4": ("C3", 0.3, 4, w) for w in ("scoring", "fp32", "bf16", "ddim")})
CENSUS_KINDS = {"fp32": {"dp_conv2d_fprop", "dp_conv2d_dgrad", "dp_conv2d_wgrad", "dp_adam_clip_ema", "dp_mse_loss_grad", "dp_silu_bwd"},
                "bf16": {"dp_conv2d_fprop_bf16", "dp_conv2d_dgrad_bf16", "dp_conv2d_wgrad_bf16", "dp_cvt_bf16", "dp_adam_clip_ema"},
                "scoring": {"dp_conv2d_fprop", "dp_conv2d_wgrad", "dp_gemm_nt_tc", "dp_groupnorm_bwd"},
                "ddim": {"dp_conv2d_fprop", "dp_ddim_step"}}
_SEEN = set()         # launch keys replayed so far, over the whole sweep
_REP = {}             # kind -> err/bound of every replayed launch of the sweep
_COUNT = {}           # kind -> unique launches replayed


@pytest.mark.parametrize("tag", list(CENSUS))
def test_pruned_census(lib, tag):
    family, ratio, B, what = CENSUS[tag]
    run = _census_run(family, ratio, B, what)
    calls = _capture(lib, run)
    del run
    gc.collect()              # the plan and its model form a reference cycle
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert CENSUS_KINDS[what] <= kinds, f"{tag}: the plan no longer issues {sorted(CENSUS_KINDS[what] - kinds)}"
    missing = kinds - set(EVAL_REPLAY) - set(INSIDE)
    assert not missing, f"{tag}: launch kinds without a replay: {sorted(missing)}"
    uniq, new = set(), []
    for name, args in calls:
        key = lc.launch_key(name, lc.argkinds(name), args)
        if key not in uniq:
            uniq.add(key)
            if key not in _SEEN:
                _SEEN.add(key)
                new.append((name, args))
    rep, failures = {}, []
    g = torch.Generator().manual_seed(2026)
    for name, args in new:
        _COUNT[name] = _COUNT.get(name, 0) + 1
        if name in INSIDE:          # checked by the replay of the launch it follows
            continue
        try:
            EVAL_REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:          # report every failing launch of the config, not just the first
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for k, v in rep.items():
        _REP.setdefault(k, []).extend(v)
    for f in failures:
        print(f"  FAIL {tag}: {f}")
    assert not failures, f"{tag}: {len(failures)} launches failed their checks"
    # every kind the plan issued was replayed, by this configuration or by an earlier one of the sweep
    assert kinds <= set(_REP), (tag, sorted(kinds - set(_REP)))
    print(f"\n{tag}: {len(calls)} launches, {len(uniq)} unique, {len([1 for n, _ in new if n not in INSIDE])} not seen earlier in the "
          f"sweep, {len(kinds)} kinds, all replayed")
    for name in sorted(rep):
        print(f"  {tag:28s} {name:26s} {len(rep[name]):4d} checks, worst err/bound {max(rep[name]):.3f}")


def test_pruned_census_sweep_summary():
    if not _REP:
        pytest.skip("no census configuration ran in this session")
    print(f"\nsweep: {len(_SEEN)} unique launches")
    for name in sorted(_REP):
        print(f"  {name:26s} {_COUNT.get(name, 0):5d} unique, worst err/bound {max(_REP[name]):.3f}")
    assert max(max(v) for v in _REP.values()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------- amax slots
@pytest.mark.parametrize("family,ratio,B", [("C1", 0.05, 8), ("C1", 0.7, 8), ("C3", 0.3, 4)])
def test_amax_slots_bound_their_operands_at_pruned_widths(family, ratio, B):
    """test_unet_gpu.py::test_amax_slots_bound_their_operands on the sweep's scoring passes: every slot a tensor-core launch scales by
    is >= torch's max|operand| right before the launch."""
    from diff_pruning_b200 import engine
    from diff_pruning_b200.scoring import TaylorScorer
    engine.AUDIT_SLOTS = True
    try:
        m = _fresh(family, ratio)
        clean, noise = _batch(B, HW[family])
        sc = TaylorScorer(m, clean, noise, use_graph=False, fused_scores=True)
        for t in (3, 600):
            sc.step(t)
        log = sc.plan.audit_log
        assert len(log) > 50, len(log)
        assert all(b >= v for b, v in log)
        standalone = sum(1 for f in sc.plan.fwd + sc.plan.bwd_steps if getattr(f, "what", "") == "amax")
        convs = sum(1 for f in sc.plan.fwd + sc.plan.bwd_steps if getattr(f, "what", "").startswith("conv fprop"))
        assert standalone < 2 * convs, (standalone, convs)
        print(f"\n{family} {ratio}: {len(log)} slot checks, {standalone} dp_amax launches for {convs} convolutions")
    finally:
        engine.AUDIT_SLOTS = False


# ---------------------------------------------------------------------------------------------------------------------- poisoned plans
POISONS = (float("nan"), 1e30, 0.0)


def _same(a, b, what):
    assert a.keys() == b.keys()
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, f"{what}: {len(bad)} outputs differ, first {bad[:6]}"


def _finite(out, what):
    bad = [k for k, v in out.items() if not bool(torch.isfinite(v).all())]
    assert not bad, f"{what}: non-finite outputs {bad[:6]}"


def _poisoned(make, fn, what):
    """fn(fresh model) under each poison; asserts the results bitwise equal (and finite).  Returns the poisoned-allocation counts."""
    outs, counts = [], []
    for v in POISONS:
        m = make()
        with poisoned_alloc(v) as c:
            outs.append(fn(m))
        counts.append(c.n)
        del m
        gc.collect()
        torch.cuda.empty_cache()
    assert all(n > 0 for n in counts), (what, counts)      # the hook was live
    _finite(outs[2], what)
    _same(outs[2], outs[0], f"{what}: NaN-poisoned vs zero-filled")
    _same(outs[2], outs[1], f"{what}: 1e30-poisoned vs zero-filled")
    print(f"\n{what}: {counts[0]} / {counts[1]} / {counts[2]} allocations poisoned (NaN / 1e30 / 0), results bit-identical")
    return counts


POISON_NETS = [("C1", 0.0, 128), ("C3", 0.0, 4)] + [("C1", r, 128) for r in C1_RATIOS] + [("C3", 0.3, 4)]


@pytest.mark.parametrize("run", ["taylor", "finetune fp32", "finetune bf16", "ddim"])
@pytest.mark.parametrize("net", POISON_NETS, ids=[f"{f}-{r}-b{b}" for f, r, b in POISON_NETS])
def test_poisoned_plans_are_bitwise_equal(net, run):
    family, ratio, B = net
    hw = HW[family]
    fn = {"taylor": lambda m: _taylor(m, B, hw), "finetune fp32": lambda m: _finetune(m, B, hw, "fp32"),
          "finetune bf16": lambda m: _finetune(m, B, hw, "bf16"), "ddim": lambda m: _ddim(m, B)}[run]
    _poisoned(lambda: _fresh(family, ratio), fn, f"{family} {ratio} b{B} {run}")


def test_poisoned_c5_taylor_passes_are_bitwise_equal():
    """C5 (cin256-v2, batch 2): FinetuneStepper and DDIMPipeline take the UNet2DModel family only, so the Taylor passes."""
    from diff_pruning_b200 import ldm
    base, cfg = lc.c5_model()
    base = base.cuda()
    ctx = torch.randn(2, 1, cfg["context_dim"], generator=torch.Generator().manual_seed(9)).cuda()
    _poisoned(lambda: copy.deepcopy(base), lambda m: _taylor(m, 2, 64, alphas_cumprod=ldm.ldm_alphas_cumprod(), context=ctx), "C5 b2 taylor")


def test_poisoned_feature_plan_and_ssim_are_bitwise_equal():
    from diff_pruning_b200 import fid
    from diff_pruning_b200.ssim import ssim
    from test_eval_census_gpu import _seeded_inception
    model = _seeded_inception()
    x = torch.randint(0, 256, (50, 32, 32, 3), generator=torch.Generator().manual_seed(13), dtype=torch.uint8).cuda()

    def features(_):
        plan = fid.FeaturePlan(model, 50, "u8", (32, 32), quantize=False, use_graph=False)
        plan.load(x)
        plan.ensure_packed()
        plan.run_eager()
        return {f"feat {k}": v.clone() for k, v in plan.feat.items()}
    _poisoned(lambda: None, features, "FID FeaturePlan u8 b50 32px")
    g = torch.Generator().manual_seed(4)
    X, Y = torch.rand(3, 3, 37, 45, generator=g).cuda(), torch.rand(3, 3, 37, 45, generator=g).cuda()
    _poisoned(lambda: None, lambda _: {"ssim": ssim(X, Y, data_range=1.0, size_average=False)}, "dp_ssim")


@pytest.mark.parametrize("what", ["C1 b128 taylor", "C1 0.3 b128 finetune fp32"])
def test_graph_mode_under_nan_equals_eager_under_zero(what):
    """The path bench.py and the stepper take: a CUDA-graph run whose plan was built under NaN poison against an eager run under 0."""
    ratio = 0.3 if "0.3" in what else 0.0
    fn = (lambda m, g: _taylor(m, 128, 32, use_graph=g)) if "taylor" in what else (lambda m, g: _finetune(m, 128, 32, "fp32", use_graph=g))
    m = _fresh("C1", ratio)
    with poisoned_alloc(0.0):
        eager = fn(m, False)
    m = _fresh("C1", ratio)
    with poisoned_alloc(float("nan")) as c:
        graph = fn(m, True)
    assert c.n > 0
    _finite(eager, what)
    _same(eager, graph, f"{what}: graph under NaN vs eager under 0")


def test_planted_pad_nan_changes_the_result(lib):
    """The plan's one dependency on initialised pads: the pad columns of the fused q / k / v gradient buffer (C1 at 0.3: inner 179, part
    pitch 180) are zeroed once when the plan is built and read by the fused dgrad against zero weight rows.  The buffer is found through
    the arguments of the six fused dgrad launches (K = 3 x 180) of the first pass; NaN written into its pad columns must show in the
    gradients after the second pass, so a plan that stopped zeroing them would fail the poisoned-plan comparison."""
    from diff_pruning_b200.scoring import TaylorScorer
    inner, ip = 179, 180
    outs = []
    for fill in (0.0, float("nan")):
        m = _fresh("C1", 0.3)
        clean, noise = _batch(8, 32)
        made = []      # the plan binds the launch functions when it records them: it is built inside the capture
        calls = _capture(lib, lambda: made.append(TaylorScorer(m, clean, noise, use_graph=False, fused_scores=True)) or made[0].step(7))
        sc, = made
        found = [args[0] for n, args in calls if n == "dp_conv2d_dgrad" and args[0].K == 3 * ip and args[0].R == args[0].S == 1]
        assert len(found) == 6 and all(a.ldy == 3 * ip for a in found), [(a.K, a.ldy) for a in found]
        for a in found:
            rows = a.N * a.H * a.W
            col = torch.full((rows, 1), fill, device="cuda")
            for i in range(3):
                assert lib.dp_copy_rows(col.data_ptr(), 1, a.y + 4 * (i * ip + inner), a.ldy, rows, 1, S()) == 0
        sc.step(400)
        outs.append({"grad " + k: p.grad.clone() for k, p in m.named_parameters()})
        del sc, m, calls, found
        gc.collect()
    _finite(outs[0], "zeros written into the pads")
    bad = [k for k in outs[0] if not torch.equal(outs[0][k], outs[1][k])]
    assert bad, "NaN in the fused q / k / v dy pad columns left every gradient unchanged: the poisoned-plan comparison has no teeth"
    print(f"\nNaN planted in the q / k / v dy pads: {len(bad)} of {len(outs[0])} gradients changed")


# ---------------------------------------------------------------------------------------------------------------------- fp64 end to end
FP64_NETS = [("C1", 0.05, 8), ("C1", 0.7, 8), ("C3", 0.3, 1)]


@pytest.mark.parametrize("family,ratio,B", FP64_NETS)
def test_pruned_two_accumulated_passes_vs_fp64_oracle(family, ratio, B):
    """Two accumulated Taylor passes (t = 7, 400) against oracle/unet_oracle.py evaluated in float64 on the GPU (no TF32 there), with
    the thresholds of the full-width C5 test: loss within 5e-6, eps_hat within 1e-4, worst gradient error below 1e-4, and every
    gradient the oracle gives as exactly zero exactly zero on the device (these networks have none: gradients that vanish in exact
    arithmetic, such as to_k.bias, hold cancellation noise on both sides, which worst_grad_err's absolute criterion covers).
    Measured on an H100 80GB HBM3: loss within 2e-7, eps_hat 2e-6, worst gradient error 7e-6 (C3 at 0.3)."""
    from oracle import unet_oracle as orc
    from diff_pruning_b200.scoring import TaylorScorer
    m = _fresh(family, ratio)
    cfg, hw = _cfg(family), HW[family]
    clean, noise = _batch(B, hw)
    sd = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    ac = orc.alphas_cumprod().double().cuda()
    m.zero_grad(set_to_none=True)
    sc = TaylorScorer(m, clean, noise, use_graph=False)
    for tt in (7, 400):
        t = torch.full((B,), tt, dtype=torch.long, device="cuda")
        out_ref = orc.unet_forward(sd, cfg, orc.add_noise(ac, clean.double(), noise.double(), t), t)
        loss_ref = F.mse_loss(out_ref, noise.double())
        loss_ref.backward()
        loss = sc.step(tt).item()
        eps = max_rel(sc.plan.output_nchw(), out_ref)
        print(f"\n{family} {ratio} t={tt}: loss {loss:.9f} (fp64 oracle {loss_ref.item():.9f}), eps_hat max-rel {eps:.2e}")
        assert loss == pytest.approx(loss_ref.item(), rel=5e-6), tt
        assert eps < 1e-4, tt
        del out_ref, loss_ref
    ref = {k: v.grad for k, v in sd.items()}
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), ref)
    zero = [k for k in ref if float(ref[k].abs().max()) == 0.0]
    print(f"{family} {ratio}: worst gradient error {worst:.2e}, {len(zero)} exactly-zero oracle gradients")
    assert worst < 1e-4, worst
    params = dict(m.named_parameters())
    assert all(float(params[k].grad.abs().max()) == 0.0 for k in zero), zero


@pytest.mark.parametrize("family,ratio,B", FP64_NETS)
def test_pruned_finetune_step_vs_fp64_oracle(family, ratio, B):
    """One fp32-grade FinetuneStepper step (dropout 0) against the float64 oracle on the GPU: loss (ddpm_train.py:459) and the gradient
    norm before clipping, with the tolerances of test_unet_gpu.py::test_finetune_two_steps_on_pruned_c1_vs_oracle."""
    from oracle import unet_oracle as orc
    from diff_pruning_b200.scoring import FinetuneStepper
    m = _fresh(family, ratio).train()
    assert all(mod.p == 0 for mod in m.modules() if isinstance(mod, torch.nn.Dropout))
    cfg, hw = _cfg(family), HW[family]
    params = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    ac = orc.alphas_cumprod().double().cuda()
    g = torch.Generator().manual_seed(11)
    clean, noise = torch.randn(B, 3, hw, hw, generator=g).cuda(), torch.randn(B, 3, hw, hw, generator=g).cuda()
    t = orc.antithetic_timesteps(B, 1000, generator=g).cuda()
    out = orc.unet_forward(params, cfg, orc.add_noise(ac, clean.double(), noise.double(), t), t)
    loss_ref = (noise.double() - out).square().sum(dim=(1, 2, 3)).mean(dim=0)
    loss_ref.backward()
    gn_ref = torch.sqrt(sum((p.grad ** 2).sum() for p in params.values())).item()
    del out
    st = FinetuneStepper(m, lr=2e-4, ema_decay=0.9999, max_grad_norm=1.0, use_graph=False)
    loss = st.step(clean, noise, t).item()
    gn = float(st.sumsq.sqrt())
    print(f"\n{family} {ratio}: loss {loss:.7f} (fp64 {loss_ref.item():.7f}), grad norm {gn:.6g} (fp64 {gn_ref:.6g})")
    assert loss == pytest.approx(loss_ref.item(), rel=2e-5)
    assert gn == pytest.approx(gn_ref, rel=2e-4)
