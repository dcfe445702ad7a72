"""End-to-end parity of the planned CUDA engine (through the C-ABI) against golden fixtures produced by the
unmodified reference, and against the oracle on fresh seeds."""
import copy

import pytest
import torch
import torch.nn.functional as F

from conftest import expand, load_golden, max_rel, rel_err, worst_grad_err
import diff_pruning_b200 as dp
from diff_pruning_b200.scoring import FinetuneStepper, TaylorScorer, group_importance, select_pruning_idxs
from diff_pruning_b200 import pruning

pytestmark = pytest.mark.gpu


def inputs(b, hw):
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)
    return torch.randn(b, 3, hw, hw, generator=g1), torch.randn(b, 3, hw, hw, generator=g2)


def build(cfg, seed=0):
    torch.manual_seed(seed)
    return dp.UNet2DModel(**cfg).eval().cuda()


@pytest.mark.parametrize("use_graph", [False, True])
def test_tiny_two_accumulated_passes(use_graph):
    """grads accumulate over passes (no zero_grad) — ddpm_prune.py:90,97-102."""
    G = load_golden("tiny_unet.pt")
    m = build(G["cfg"])
    clean, noise = inputs(2, 16)
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=use_graph)
    losses = [sc.step(7).item(), sc.step(400).item()]
    assert losses == pytest.approx(G["losses"], rel=2e-6)
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), G["grads"])
    assert worst < 5e-5, worst


def test_tiny_autograd_boundary_matches_scripts_loop():
    """The unchanged script loop: scheduler.add_noise -> model(...).sample -> F.mse_loss -> loss.backward()."""
    G = load_golden("tiny_unet.pt")
    m = build(G["cfg"])
    sched = dp.DDPMScheduler(num_train_timesteps=1000)
    clean, noise = (t.cuda() for t in inputs(2, 16))
    m.zero_grad()
    losses = []
    for tt in (7, 400):
        t = (tt * torch.ones(2, device="cuda")).long()
        out = m(sched.add_noise(clean, noise, t), t).sample
        loss = F.mse_loss(out, noise)
        loss.backward()
        losses.append(loss.item())
    assert losses == pytest.approx(G["losses"], rel=2e-6)
    assert max_rel(out, G["out_last"]) < 1e-5
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), G["grads"])
    assert worst < 5e-5, worst
    with torch.no_grad():   # per-sample timesteps, inference path
        out2 = m(sched.add_noise(clean, noise, G["t2"].cuda()), G["t2"].cuda()).sample
    assert max_rel(out2, G["out_t2"]) < 1e-5
    # python-number timestep like the pipelines pass (pipeline_ddim.py:105)
    with torch.no_grad():
        o3 = m(clean, 5).sample
        o4 = m(clean, torch.tensor(5, device="cuda")).sample
    assert torch.equal(o3, o4)
    # model survives pickling / deepcopy with live plans (ddpm_prune.py:135, op_counter.py:18)
    m2 = copy.deepcopy(m)
    assert "_dpb200_plans" not in m2.__dict__


def test_cifar_eps_and_grads():
    """C1 (CIFAR UNet) seed 0: eps_hat within 1e-4 relative of the reference CPU fp32 (north_star tolerance)."""
    G = load_golden("cifar_fwd.pt")
    m = build(dp.CIFAR10_DDPM_CONFIG)
    sched = dp.DDPMScheduler()
    clean16, noise16 = inputs(16, 32)
    clean, noise = clean16[:2].cuda(), noise16[:2].cuda()
    with torch.no_grad():
        for tt, ref in G["eps_b2"].items():
            t = (tt * torch.ones(2, device="cuda")).long()
            assert max_rel(m(sched.add_noise(clean, noise, t), t).sample, ref) < 1e-4, tt
    m.zero_grad()
    sc = TaylorScorer(m, clean, noise, use_graph=False)
    assert sc.step(500).item() == pytest.approx(G["loss_b2_t500"], rel=5e-6)
    bad = []
    for k, p in m.named_parameters():
        s = G["grad_samples_b2_t500"][k]
        g = p.grad.flatten()[:64].cpu()
        if rel_err(g, s) > 2e-3 and float((g - s).abs().max()) > 1e-7:
            bad.append((k, rel_err(g, s)))
        f = G["grad_fp_b2_t500"][k]
        assert float((p.grad.double() ** 2).sum()) == pytest.approx(f[2], rel=2e-3), k
    assert not bad, bad[:5]


def test_cfg1_scores_and_masks_bit_exact():
    """BASELINE config 1 on the GPU: 100 timesteps B=16, ratio 0.3.  Losses, per-group importance vectors and the
    pruned channel-index sets (all three importance variants) against the unmodified reference; then the pruned
    network's eps_hat."""
    G = load_golden("cifar_cfg1.pt")
    m = build(dp.CIFAR10_DDPM_CONFIG)
    clean, noise = inputs(G["B"], 32)
    m.zero_grad()
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=True)
    losses = sc.run(range(G["n_steps"])).cpu()
    assert rel_err(losses, torch.tensor(G["losses"])) < 5e-6
    for k, p in m.named_parameters():
        assert float((p.grad.double() ** 2).sum()) == pytest.approx(G["grad_fp"][k][2], rel=5e-3), k
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    sched = dp.DDPMScheduler()
    for variant, V in G["variants"].items():
        mv = copy.deepcopy(m)
        for k, p in mv.named_parameters():
            p.grad = grads[k].clone()
        # the whole product pipeline: structural groups in the reference's order -> device-side scores -> selection -> slicing
        rec = pruning.taylor_prune(mv, G["ratio"], variant, ignored_layers=[mv.conv_out])
        assert [r["root"] for r in rec] == [g["root"] for g in V["groups"]]
        worst_imp = 0.0
        for r, g in zip(rec, V["groups"]):
            worst_imp = max(worst_imp, rel_err(r["imp"], g["imp"]))
            assert sorted(r["idxs"]) == sorted(g["idxs"]), (variant, g["root"], worst_imp)   # bit-exact mask
        assert worst_imp < 2e-3, (variant, worst_imp)
        assert {k: list(v.shape) for k, v in mv.state_dict().items()} == V["pruned_shapes"]
        assert sum(p.numel() for p in mv.parameters()) == V["pruned"][1] == 19851157
        with torch.no_grad():
            t = (10 * torch.ones(2, device="cuda")).long()
            out = mv(sched.add_noise(clean[:2].cuda(), noise[:2].cuda(), t), t).sample
        assert max_rel(out, V["pruned_eps_b2_t10"]) < 1e-4, variant
    # the same through the reference's own call sequence (ddpm_prune.py:60,79-87,108-116) on the compat names
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diff-pruning_b200", "compat"))
    import torch_pruning as tp
    from diffusers.models.resnet import Downsample2D, Upsample2D
    mv = copy.deepcopy(m)
    for k, p in mv.named_parameters():
        p.grad = grads[k].clone()
    ex = {"sample": torch.randn(1, 3, 32, 32).cuda(), "timestep": torch.ones((1,)).long().cuda()}
    pr = tp.pruner.MagnitudePruner(mv, ex, importance=tp.importance.TaylorImportance(multivariable=True), iterative_steps=1,
                                   channel_groups={}, ch_sparsity=G["ratio"], ignored_layers=[mv.conv_out])
    got = []
    for g in pr.step(interactive=True):
        got.append(sorted(g.idxs))
        g.prune()
    for mod in mv.modules():
        if isinstance(mod, (Upsample2D, Downsample2D)):
            mod.channels = mod.conv.in_channels
    assert got == [sorted(g["idxs"]) for g in G["variants"]["taylor"]["groups"]]
    assert tp.utils.count_ops_and_params(mv, ex) == (G["variants"]["taylor"]["pruned"][0], 19851157.0)


def test_finetune_two_steps():
    """ddpm_train.py:437-469 (dropout 0): loss, clipped Adam update and EMA after 2 steps vs the reference."""
    G = load_golden("finetune_tiny.pt")
    for use_graph in (False, True):
        torch.manual_seed(0)
        m = dp.UNet2DModel(**G["cfg"]).cuda().train()
        st = FinetuneStepper(m, lr=2e-4, ema_decay=0.9999, max_grad_norm=1.0, use_graph=use_graph)
        for s in G["steps"]:
            loss = st.step(s["clean"].cuda(), s["noise"].cuda(), s["t"].cuda())
            assert loss.item() == pytest.approx(s["loss"], rel=2e-5)
            assert float(st.sumsq.sqrt()) == pytest.approx(s["grad_norm"], rel=2e-4)
        ema = st.ema_state()
        # Adam normalises the step (m/sqrt(v)): a zero-initialised bias moves by ~lr per step, so its relative
        # error after 2 steps equals the gradient's relative rounding error (~1e-5), not 1e-7.
        for k, p in m.named_parameters():
            assert rel_err(p, G["params"][k]) < 5e-5, k
            assert rel_err(ema[k], G["ema"][k]) < 5e-5, k


def test_lsun_family_block_one_pass_vs_oracle():
    """A narrow member of the LSUN-256 family (6 levels, attention at level 4, 64x64 input) vs the oracle."""
    from oracle import unet_oracle as orc
    cfg = dict(dp.LSUN256_DDPM_CONFIG, block_out_channels=(32, 32, 64, 64, 128, 128), sample_size=64)
    torch.manual_seed(3)
    m = dp.UNet2DModel(**cfg).eval()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(9)
    clean, noise = torch.randn(2, 3, 64, 64, generator=g), torch.randn(2, 3, 64, 64, generator=g)
    t = torch.tensor([123, 877])
    ref = orc.taylor_pass(sd, cfg, orc.alphas_cumprod(), clean, noise, t)
    m = m.cuda()
    m.zero_grad()
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=False)
    assert sc.step(t).item() == pytest.approx(ref.item(), rel=5e-6)
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), {k: v.grad for k, v in sd.items()})
    assert worst < 1e-4, worst


def test_fused_signed_scores_fall_out_of_backward():
    """North-star item: the wgrad reduce accumulates sum_t sum_k W*dW_t per channel while it adds dW_t into .grad; the
    `multivariable=True` Taylor score |.| computed from that equals the one computed from the accumulated gradient
    (scores are linear in dW: sum_t and sum_k commute)."""
    from diff_pruning_b200.scoring import taylor_layer_scores
    m = build(dp.TINY_TEST_CONFIG)
    clean, noise = inputs(2, 16)
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=True, fused_scores=True)
    for t in (3, 250, 600, 990):
        sc.step(t)
    fused = sc.signed_scores()
    params = dict(m.named_parameters())
    assert len(fused) == sum(1 for p in params.values() if p.dim() >= 2)
    worst = 0.0
    for name, (so, si) in fused.items():
        ref = taylor_layer_scores(params[name], params[name].grad)
        scale = float(ref["out_abs"].max())          # sum |w dw|: the magnitude of the summands (signed sums can cancel)
        worst = max(worst, float((so - ref["out_signed"]).abs().max()) / scale, float((si - ref["in_signed"]).abs().max()) / scale)
    assert worst < 2e-5, worst


def test_cfg3_lsun256_b4_scores_and_masks_bit_exact():
    """BASELINE config 3 (google/ddpm-ema-bedroom-256 architecture, 113.7 M params, batch 4 x 3x256x256, ratio 0.05, README.md:140-148)
    on the GPU against tests/golden/lsun_cfg3_s3.pt — produced by the UNMODIFIED reference on 3 of the 1000 timesteps (t = 0, 500, 999):
    losses, eps_hat (strided sample) <= 1e-4, accumulated-gradient fingerprints, then for all three importance variants the interactive
    prune sequence: group order, per-group importance vectors, and the pruned channel-index sets BIT-EXACT (at ratio 0.05 the 59
    GroupNorm-coupled groups get a per-GN-group quota of 0 and prune nothing, metapruner.py:237-246; the 12 others carry the mask)."""
    G = load_golden("lsun_cfg3_s3.pt")
    cfg = dp.LSUN256_DDPM_CONFIG
    m = build(cfg)
    assert round(sum(p.numel() for p in m.parameters()) / 1e6, 3) == 113.673
    clean, noise = inputs(G["B"], G["hw"])
    m.zero_grad()
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=False)
    st = G["eps_stride"]
    for t, l_ref, e_ref in zip(G["timesteps"], G["losses"], G["eps_sub"]):
        assert sc.step(t).item() == pytest.approx(l_ref, rel=5e-6), t
        assert max_rel(sc.plan.output_nchw()[:, :, ::st, ::st], e_ref) < 1e-4, t
    for k, p in m.named_parameters():
        assert float((p.grad.double() ** 2).sum()) == pytest.approx(G["grad_fp"][k][2], rel=5e-3), k
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    del sc
    m._dpb200_plans.clear()
    torch.cuda.empty_cache()
    sched = dp.DDPMScheduler()
    for variant, V in G["variants"].items():
        mv = copy.deepcopy(m)
        for k, p in mv.named_parameters():
            p.grad = grads[k].clone()
        rec = pruning.taylor_prune(mv, G["ratio"], variant, ignored_layers=[mv.conv_out])
        assert [r["root"] for r in rec] == [g["root"] for g in V["groups"]]
        worst_imp, n_sel = 0.0, 0
        for r, g in zip(rec, V["groups"]):
            worst_imp = max(worst_imp, rel_err(r["imp"], g["imp"]))
            assert sorted(r["idxs"]) == sorted(g["idxs"]), (variant, g["root"], worst_imp)   # bit-exact mask
            n_sel += len(g["idxs"])
        assert n_sel == 267 and worst_imp < 2e-3, (variant, n_sel, worst_imp)
        assert {k: list(v.shape) for k, v in mv.state_dict().items()} == V["pruned_shapes"]
        assert sum(p.numel() for p in mv.parameters()) == V["pruned"][1] == 112648617
        with torch.no_grad():
            t = (10 * torch.ones(2, device="cuda")).long()
            out = mv(sched.add_noise(clean[:2].cuda(), noise[:2].cuda(), t), t).sample
        assert max_rel(out[:, :, ::st, ::st], V["pruned_eps_b2_t10"]) < 1e-4, variant
        del mv
        torch.cuda.empty_cache()


def _pruned_c1(batch=8):
    """C1 pruned at ratio 0.3 by the product path (3 accumulated scoring passes, taylor_prune): the 19.85 M-parameter architecture."""
    m = build(dp.CIFAR10_DDPM_CONFIG)
    clean, noise = inputs(batch, 32)
    m.zero_grad()
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=False)
    for t in (0, 500, 999):
        sc.step(t)
    del sc
    pruning.taylor_prune(m, 0.3, "taylor", ignored_layers=[m.conv_out])
    m.zero_grad(set_to_none=True)
    assert sum(p.numel() for p in m.parameters()) == 19851157
    return m


def test_finetune_two_steps_on_pruned_c1_vs_oracle():
    """The network bench.py's finetune leg times (C1 at ratio 0.3: widths 96 / 192 / 179 / 358, stale attention scale) through two
    optimisation steps of ddpm_train.py:437-469 (dropout 0) against the CPU oracle: loss, pre-clip gradient norm, parameters and EMA."""
    from oracle import unet_oracle as orc
    m = _pruned_c1().train()
    cfg = dp.CIFAR10_DDPM_CONFIG
    params = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    p0 = {k: v.detach().clone() for k, v in params.items()}
    ema = {k: v.detach().clone() for k, v in params.items()}
    opt = torch.optim.Adam(list(params.values()), lr=2e-4, betas=(0.9, 0.999), weight_decay=0.0, eps=1e-8)
    ac = orc.alphas_cumprod()
    st = FinetuneStepper(m, lr=2e-4, ema_decay=0.9999, max_grad_norm=1.0, use_graph=True)
    g = torch.Generator().manual_seed(11)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    for step in range(2):
        clean, noise = torch.randn(8, 3, 32, 32, generator=g), torch.randn(8, 3, 32, 32, generator=g)
        t = orc.antithetic_timesteps(8, 1000, generator=g)
        l_ref, gn_ref = orc.finetune_step(params, cfg, ac, clean, noise, t, opt, ema)
        loss = st.step(clean.cuda(), noise.cuda(), t.cuda())
        assert loss.item() == pytest.approx(l_ref.item(), rel=2e-5), step
        assert float(st.sumsq.sqrt()) == pytest.approx(gn_ref.item(), rel=2e-4), step
    e = st.ema_state()
    # Adam normalises the step (m / sqrt(v) is O(1) per element whatever the gradient's size), so elements whose gradient is mostly
    # cancellation noise move by an essentially arbitrary fraction of lr: the parameter check is (a) the weights as tensors and (b) the
    # error of the UPDATE relative to the update itself (97 % of every tensor's two-step update must agree with the reference).
    lr, steps = 2e-4, 2
    for k, p in m.named_parameters():
        ref, ours = params[k].detach().double(), p.detach().cpu().double()
        upd = (ref - p0[k].double()).norm().item()
        if upd < 1e-2 * lr * steps * ref.numel() ** 0.5:
            # the reference itself barely moved this tensor: its gradient is identically zero in exact arithmetic (d/d to_k.bias: softmax
            # is invariant to a per-query constant) or pure cancellation, |g| << Adam's eps — both sides hold rounding noise only
            assert (ours - ref).abs().max().item() <= 1e-2 * lr * steps, k
            continue
        assert (ours - ref).norm().item() <= 3e-2 * upd + 1e-12, (k, (ours - ref).norm().item(), upd)
        if p.dim() >= 2:
            assert rel_err(p, params[k]) < 1e-4, k
        assert rel_err(e[k], ema[k]) < 1e-4 or (e[k].cpu().double() - ema[k].double()).norm().item() <= 3e-2 * upd, k


def test_sharded_scoring_equals_sequential_on_two_streams():
    """Timestep sharding (SURVEY.md §8e) exercised on ONE GPU: two replicas of the model act as ranks 0 / 1 on two CUDA streams
    (t = r, r+2, ...), their gradient arenas are summed (what the NCCL all-reduce does) and compared with the sequential loop —
    so the driver's single-GPU box checks sharded == sequential too (tests/test_multi_gpu.py needs 2 GPUs)."""
    m = build(dp.TINY_TEST_CONFIG)
    clean, noise = (x.cuda() for x in inputs(2, 16))
    ts = list(range(0, 1000, 125))
    m.zero_grad()
    seq = TaylorScorer(m, clean, noise, use_graph=False)
    l_seq = seq.run(ts, shard=False)
    reps, streams, losses = [], [torch.cuda.Stream(), torch.cuda.Stream()], {}
    for r in range(2):
        mr = copy.deepcopy(m)
        mr.zero_grad(set_to_none=True)
        reps.append(TaylorScorer(mr, clean, noise, use_graph=False))
    torch.cuda.synchronize()
    for k, t in enumerate(ts):
        with torch.cuda.stream(streams[k % 2]):
            losses[k] = reps[k % 2].step(t).clone()
    torch.cuda.synchronize()
    total = reps[0].plan.grad_arena + reps[1].plan.grad_arena
    assert rel_err(total, seq.plan.grad_arena) < 1e-6
    assert torch.allclose(torch.stack([losses[k] for k in range(len(ts))]).flatten(), l_seq, rtol=1e-6)


def test_diff_pruning_threshold_rule_on_gpu():
    """`--pruner diff-pruning` (ddpm_prune.py:104-106): run(thr=) stops after the first timestep whose loss drops below thr x the running
    maximum; that timestep's gradient is included.  Against the sequential loop replayed step by step on a second replica."""
    from diff_pruning_b200.scoring import threshold_stop
    m = build(dp.TINY_TEST_CONFIG)
    clean, noise = (x.cuda() for x in inputs(2, 16))
    ts = list(range(0, 1000, 40))
    ref = copy.deepcopy(m)
    ref.zero_grad(set_to_none=True)
    rs = TaylorScorer(ref, clean, noise, use_graph=False)
    all_losses = [rs.step(t).item() for t in ts]
    # a threshold the (random-init, nearly flat) loss sequence crosses part-way: scan candidate ratios l_k / running max
    thr = n_used = None
    run_max = 0.0
    for k, l in enumerate(all_losses):
        run_max = max(run_max, l)
        cand = 0.5 * (l / run_max + 1.0) if l < run_max else None
        if cand is not None and 1 < threshold_stop(all_losses, cand) < len(ts):
            thr, n_used = cand, threshold_stop(all_losses, cand)
            break
    if thr is None:     # monotonically rising losses: reverse the order (the rule only sees the sequence it is given)
        ts = ts[::-1]
        all_losses = all_losses[::-1]
        k = len(ts) // 2
        thr = 0.5 * (all_losses[k] + all_losses[k - 1]) / max(all_losses[:k])
        n_used = threshold_stop(all_losses, thr)
    assert 1 < n_used < len(ts), (n_used, thr, all_losses)
    ref.zero_grad(set_to_none=True)
    ref._dpb200_plans.clear()
    rs = TaylorScorer(ref, clean, noise, use_graph=False)
    for t in ts[:n_used]:
        rs.step(t)
    m.zero_grad()
    sc = TaylorScorer(m, clean, noise, use_graph=True)
    used = sc.run(ts, thr=thr)
    assert len(used) == n_used and used.cpu().tolist() == pytest.approx(all_losses[:n_used], rel=1e-6)
    assert rel_err(sc.plan.grad_arena, rs.plan.grad_arena) < 1e-6


def test_fused_scores_match_the_oracle_item_score():
    """fused_scores=True: the wgrad reduce accumulates sum_t sum_k W*dW_t per in/out channel; |.| of it is the `multivariable=True`
    Taylor score of the UNSLICED layer (importance.py:393,407 with the abs outside the sum).  Checked against the oracle's item_score on
    the accumulated gradient.  (Later groups of an interactive prune see already-sliced layers, so the product's taylor_prune re-reads
    W and dW per group; the fused vector is exact for each layer's first evaluation and as the small all-reduce payload.)"""
    from oracle import unet_oracle as orc
    m = build(dp.TINY_TEST_CONFIG)
    clean, noise = inputs(2, 16)
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=True, fused_scores=True)
    for t in (3, 250, 600, 990):
        sc.step(t)
    params = dict(m.named_parameters())
    worst = 0.0
    for name, (so, si) in sc.signed_scores().items():
        w, dw = params[name].detach().cpu(), params[name].grad.detach().cpu()
        ref_o = orc.item_score(w, dw, "out", list(range(w.shape[0])), "taylor")
        ref_i = orc.item_score(w, dw, "in", list(range(w.shape[1])), "taylor")
        scale = float(orc.item_score(w, dw, "out", list(range(w.shape[0])), "diff").max())   # sum |w dw|: size of the summands
        worst = max(worst, float((so.abs().cpu() - ref_o).abs().max()) / scale, float((si.abs().cpu() - ref_i).abs().max()) / scale)
    assert worst < 2e-5, worst


def test_forward_after_finetune_step_uses_current_weights():
    """ADVICE round 1 (high): the Adam kernel writes the parameter arena through raw pointers and `param.data.copy_` (EMAModel.copy_to /
    restore) leaves torch's version counters untouched — a cached no-grad plan must not keep the packs of its first use."""
    from diff_pruning_b200 import engine
    m = build(dp.TINY_TEST_CONFIG).train()
    st = FinetuneStepper(m, lr=1e-2, ema_decay=0.9, max_grad_norm=1.0, use_graph=True)
    g = torch.Generator().manual_seed(3)
    clean, noise = torch.randn(4, 3, 16, 16, generator=g).cuda(), torch.randn(4, 3, 16, 16, generator=g).cuda()
    t = torch.tensor([5, 300, 700, 994]).cuda()
    x = torch.randn(2, 3, 16, 16, generator=g).cuda()

    def fresh(model):       # the same weights through a plan that has never been used
        m2 = copy.deepcopy(model).eval()
        with torch.no_grad():
            return m2(x, 50).sample
    m.eval()
    for it in range(2):
        m.train(); st.step(clean, noise, t); m.eval()
        with torch.no_grad():
            y = m(x, 50).sample
        assert torch.equal(y, fresh(m)), it
    # EMA copy_to-style write (no version bump) followed by sampling inside frozen_weights, then restore
    saved = [p.detach().clone() for p in m.parameters()]
    with torch.no_grad():
        for p, e in zip(m.parameters(), st.ema_state().values()):
            p.data.copy_(e)
    with engine.frozen_weights(m), torch.no_grad():
        y_ema = m(x, 50).sample
        assert torch.equal(y_ema, m(x, 50).sample)
    assert torch.equal(y_ema, fresh(m))
    with torch.no_grad():
        for p, s_ in zip(m.parameters(), saved):
            p.data.copy_(s_)
        assert torch.equal(m(x, 50).sample, y)


def test_autograd_path_guards_and_dropout_stream():
    """ADVICE round 1 (medium): (a) two forwards before one backward must raise instead of producing gradients from overwritten
    activations; (b) an input that requires grad is refused (the engine does not produce dL/dsample); (c) in train mode with dropout
    every forward draws a fresh mask (the unmodified ddpm_train.py loop with --dropout 0.1)."""
    m = build(dp.TINY_TEST_CONFIG)
    x = torch.randn(2, 3, 16, 16, device="cuda")
    y1 = m(x, 10).sample
    y2 = m(x, 20).sample
    with pytest.raises(RuntimeError, match="overwritten"):
        y1.sum().backward()
    y2.sum().backward()
    with pytest.raises(RuntimeError, match="d\\(loss\\)/d\\(sample\\)"):
        m(x.clone().requires_grad_(True), 10)
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.3
    m.train()
    with torch.no_grad():
        a, b = m(x, 10).sample, m(x, 10).sample
    assert not torch.equal(a, b)
    m.eval()
    with torch.no_grad():
        assert torch.equal(m(x, 10).sample, m(x, 10).sample)


def test_ddim_sampling_matches_reference_pipeline():
    """DDIMPipeline + the reference's modified DDIMScheduler (skip_type, prev_timestep rule) on the device: images of a 10-step
    eta=0 uniform run and a 7-step eta=0.5 quad run (CPU generator for the initial latent and the variance noise, like the
    fixture) within 2e-4 of the reference's CPU pipeline (errors of the 1e-5-grade UNet compound over the chain)."""
    G = load_golden("ddim_tiny.pt")
    from diff_pruning_b200.sampling import DDIMPipeline
    m = build(G["cfg"])
    for name in ("uniform_eta0", "quad_eta05"):
        R = G[name]
        pipe = DDIMPipeline(unet=m, scheduler=dp.DDPMScheduler(num_train_timesteps=1000))
        pipe.scheduler.skip_type = R["skip_type"]
        g = torch.Generator().manual_seed(0)
        out = pipe(batch_size=2, generator=g, eta=R["eta"], num_inference_steps=R["steps"], output_type="numpy").images
        assert torch.equal(pipe.scheduler.timesteps, R["timesteps"])
        assert out.shape == tuple(R["images"].shape) and out.min() >= 0.0 and out.max() <= 1.0
        assert float((torch.from_numpy(out) - R["images"]).abs().max()) < 2e-4, name


def test_ddpm_train_loop_through_the_compat_surface_bf16():
    """The body of ddpm_train.py:255-261,320-348,381-401,423-477 driven through compat/ (accelerate shim with mixed_precision="bf16",
    diffusers.optimization.get_scheduler, diffusers.training_utils.EMAModel, DDIMPipeline sampling around the loop) on the GPU: the
    training forwards run on the bf16 tensor tier, evaluation forwards on the fp32-grade tier with the weights that are current at that
    moment (EMA copy_to / restore write through `param.data.copy_`), and the loss goes down."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diff-pruning_b200", "compat"))
    from accelerate import Accelerator
    from accelerate.utils import ProjectConfiguration
    from diffusers import DDIMPipeline, DDIMScheduler, DDPMScheduler
    from diffusers.optimization import get_scheduler
    from diffusers.training_utils import EMAModel
    accelerator = Accelerator(gradient_accumulation_steps=1, mixed_precision="bf16", log_with=None, project_dir="/tmp/dpb200_logs",
                              project_config=ProjectConfiguration())
    torch.manual_seed(0)
    model = dp.UNet2DModel(**dp.TINY_TEST_CONFIG)
    noise_scheduler = DDPMScheduler(num_train_timesteps=1000)
    g = torch.Generator().manual_seed(0)
    data = torch.randn(16, 3, 16, 16, generator=g).clamp(-1, 1)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(data), batch_size=8, shuffle=False)
    ema_model = EMAModel(model.parameters(), decay=0.999, use_ema_warmup=False, inv_gamma=1.0, power=0.75, model_cls=dp.UNet2DModel,
                         model_config=model.config)
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.95, 0.999), weight_decay=0.0, eps=1e-8)
    lr_scheduler = get_scheduler("constant", optimizer=optimizer, num_warmup_steps=0, num_training_steps=100)
    model, optimizer, loader, lr_scheduler = accelerator.prepare(model, optimizer, loader, lr_scheduler)
    ema_model.to(accelerator.device)
    for m_ in model.modules():
        if isinstance(m_, torch.nn.Dropout):
            m_.p = 0.1

    def sample():
        unet = accelerator.unwrap_model(model).eval()
        ema_model.store(unet.parameters())
        ema_model.copy_to(unet.parameters())
        pipe = DDIMPipeline(unet=unet, scheduler=DDIMScheduler(num_train_timesteps=1000))
        pipe.scheduler.set_timesteps(4)
        imgs = pipe(batch_size=2, num_inference_steps=4, output_type="numpy").images
        ema_model.restore(unet.parameters())
        return imgs
    before = sample()
    assert before.shape == (2, 16, 16, 3)
    losses = []
    for epoch in range(6):
        for (clean_images,) in loader:
            model.train()
            noise = torch.randn(clean_images.shape, generator=g).to(clean_images.device)
            bsz = clean_images.shape[0]
            timesteps = torch.randint(0, 1000, (bsz // 2 + 1,), generator=g).to(clean_images.device)
            timesteps = torch.cat([timesteps, 1000 - timesteps - 1], dim=0)[:bsz]
            noisy = noise_scheduler.add_noise(clean_images, noise, timesteps)
            with accelerator.accumulate(model):
                optimizer.zero_grad()
                out = model(noisy, timesteps).sample
                loss = (noise - out).square().sum(dim=(1, 2, 3)).mean(dim=0)
                accelerator.backward(loss)
                if accelerator.sync_gradients:
                    accelerator.clip_grad_norm_(model.parameters(), 1.0)
                optimizer.step()
                lr_scheduler.step()
            ema_model.step(model.parameters())
            losses.append(loss.detach().item())
    plans = model._dpb200_plans
    assert any(pl.compute == "bf16" and pl.training and pl.n_bf16_convs > 5 for pl in plans.values())     # training ran on the bf16 tier
    assert sum(losses[-4:]) < sum(losses[:4]), losses
    after = sample()
    assert float(abs(after - before).max()) > 0            # sampling saw the (EMA of the) updated weights, not the packs of its first use
    model.eval()
    x = torch.randn(2, 3, 16, 16, device="cuda")
    with torch.no_grad():
        y = model(x, 50).sample
        assert torch.equal(y, copy.deepcopy(model)(x, 50).sample)   # and the live weights are back after ema.restore


def test_ldm_unet_two_accumulated_passes_vs_reference():
    """BASELINE configs[4]: the latent-diffusion UNetModel (ResBlocks, SpatialTransformer with LayerNorm / self-attention / one-token
    cross-attention / GEGLU feed-forward, strided-conv down- and nearest+conv up-sampling) through the engine: loss, eps_hat and every
    parameter gradient after two accumulated Taylor passes against the UNMODIFIED reference modules (tests/golden/ldm_tiny.pt);
    the to_q / to_k / norm2 parameters of the cross-attention receive exactly zero gradient on both sides."""
    from test_oracle_golden import ldm_tiny_model
    from diff_pruning_b200 import ldm
    G = load_golden("ldm_tiny.pt")
    for use_graph in (False, True):
        m = ldm_tiny_model(G).cuda()
        clean, noise = inputs(2, 16)
        m.zero_grad()
        sc = TaylorScorer(m, clean.cuda(), noise.cuda(), alphas_cumprod=ldm.ldm_alphas_cumprod(), use_graph=use_graph, context=G["context"].cuda())
        losses = [sc.step(7).item(), sc.step(400).item()]
        assert losses == pytest.approx(G["losses"], rel=5e-6), use_graph
        assert max_rel(sc.plan.output_nchw(), G["out_last"]) < 1e-4
        worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), G["grads"])
        assert worst < 1e-4, (use_graph, worst)
        for k, p in m.named_parameters():
            if float(G["grads"][k].abs().max()) == 0.0:
                assert float(p.grad.abs().max()) == 0.0, k
    # the module-forward path (what prune_ldm.py's model.apply_model reaches): autograd boundary + context argument
    m = ldm_tiny_model(G).cuda()
    ac = ldm.ldm_alphas_cumprod().cuda()
    clean, noise, ctx = clean.cuda(), noise.cuda(), G["context"].cuda()
    m.zero_grad()
    for tt in (7, 400):
        t = torch.full((2,), tt, device="cuda", dtype=torch.long)
        xt = (ac[t] ** 0.5).reshape(-1, 1, 1, 1) * clean + ((1 - ac[t]) ** 0.5).reshape(-1, 1, 1, 1) * noise
        loss = F.mse_loss(m(xt, t, context=ctx), noise)
        loss.backward()
    assert loss.item() == pytest.approx(G["losses"][1], rel=5e-6)
    assert worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), G["grads"]) < 1e-4


def test_ldm_cin256_v2_full_width_two_accumulated_passes_vs_fp64_oracle():
    """C5 at its real widths (cin256-v2, 400.9 M parameters: 192-960 channels, 6 / 18 / 30 channels per GroupNorm group, concatenations
    up to 1920 channels, attention over 1024 tokens on the tensor-core NT GEMM, LayerNorm at 192-960, GEGLU inner widths up to 3840,
    context_dim 512), built as bench.py builds it, batch 2 of 3x64x64 latents: two accumulated Taylor passes (t = 7, 400) against
    oracle/ldm_oracle.py evaluated in float64 on the host, with the same criteria as the ldm_tiny test."""
    from launch_census import c5_model
    from oracle import ldm_oracle as lorc
    from diff_pruning_b200 import ldm
    m, cfg = c5_model()
    B = 2
    ctx = torch.randn(B, 1, cfg["context_dim"], generator=torch.Generator().manual_seed(9))
    clean, noise = inputs(B, 64)
    sd = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    ac = lorc.alphas_cumprod()
    torch.set_num_threads(min(32, torch.get_num_threads()))
    m = m.cuda()
    m.zero_grad()
    sc = TaylorScorer(m, clean.cuda(), noise.cuda(), alphas_cumprod=ldm.ldm_alphas_cumprod(), use_graph=False, context=ctx.cuda())
    for tt in (7, 400):
        t = torch.full((B,), tt, dtype=torch.long)
        out_ref = lorc.unet_forward(sd, cfg, lorc.q_sample(ac, clean.double(), noise.double(), t), t, ctx.double())
        loss_ref = F.mse_loss(out_ref, noise.double())
        loss_ref.backward()
        loss = sc.step(tt).item()
        eps = max_rel(sc.plan.output_nchw(), out_ref)
        print(f"C5 t={tt}: loss {loss:.9f} (fp64 oracle {loss_ref.item():.9f}), eps_hat max-rel {eps:.2e}")
        assert loss == pytest.approx(loss_ref.item(), rel=5e-6), tt
        assert eps < 1e-4, tt
    ref = {k: v.grad for k, v in sd.items()}
    worst = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), ref)
    print(f"C5 worst gradient error {worst:.2e}")
    assert worst < 1e-4, worst
    zero = [k for k, p in m.named_parameters() if float(ref[k].abs().max()) == 0.0]
    assert zero and all(float(dict(m.named_parameters())[k].grad.abs().max()) == 0.0 for k in zero), zero


@pytest.mark.parametrize("family", ["unet2d_c1", "unet2d_lsun_block", "ldm_tiny"])
def test_amax_slots_bound_their_operands(family):
    """Every tensor-core launch scales its operands by the power of two taken from an amax slot.  Most slots are filled by the kernel
    that WROTE the tensor (convolution / GEMM epilogues, GroupNorm, softmax backward) instead of a separate dp_amax pass: with
    engine.AUDIT_SLOTS the plan compares each slot with torch's max|operand| right before the consuming launch (eager pass)."""
    from diff_pruning_b200 import engine
    engine.AUDIT_SLOTS = True
    try:
        if family == "ldm_tiny":
            from test_oracle_golden import ldm_tiny_model
            from diff_pruning_b200 import ldm
            G = load_golden("ldm_tiny.pt")
            m = ldm_tiny_model(G).cuda()
            clean, noise = inputs(2, 16)
            sc = TaylorScorer(m, clean.cuda(), noise.cuda(), alphas_cumprod=ldm.ldm_alphas_cumprod(), use_graph=False, context=G["context"].cuda())
        elif family == "unet2d_c1":
            m = build(dp.CIFAR10_DDPM_CONFIG)
            clean, noise = inputs(8, 32)
            sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=False)
        else:       # six levels, up / down sampling at every resolution from 64x64 to 2x2, attention at level 4
            cfg = dict(dp.LSUN256_DDPM_CONFIG, block_out_channels=(32, 32, 64, 64, 128, 128), sample_size=64)
            m = build(cfg, seed=3)
            clean, noise = inputs(2, 64)
            sc = TaylorScorer(m, clean.cuda(), noise.cuda(), use_graph=False)
        for t in (3, 600):
            sc.step(t)
        log = sc.plan.audit_log
        assert len(log) > 50, len(log)
        # the bounds are tight where the producer wrote the whole tensor, and never more than the tensor they live in allows
        assert all(b >= v for b, v in log)
        standalone = sum(1 for f in sc.plan.fwd + sc.plan.bwd_steps if getattr(f, "what", "") == "amax")
        convs = sum(1 for f in sc.plan.fwd + sc.plan.bwd_steps if getattr(f, "what", "").startswith("conv fprop"))
        assert standalone < 2 * convs, (standalone, convs)
    finally:
        engine.AUDIT_SLOTS = False
