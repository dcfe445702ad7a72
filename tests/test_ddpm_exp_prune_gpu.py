"""prune.py for ddpm_exp's Model on the GPU: the backward plan of Plan._build_ddim_model against the unmodified reference's 1000-step
loop (tests/golden/ddpm_exp_loop_tiny.pt) and its `ours` stop; ddpm_exp.prune for every criterion against the reference's pruner
(tests/golden/ddpm_exp_prune_tiny.pt); a pruned CIFAR-10 Model saved, reloaded through load_model and sampled through sample_fid; the
CIFAR-10 config's gradients against a float64 autograd of the oracle, graph against eager, poisoned allocations, the backward plan's
launch census, the amax-slot audit and the race audit of the two-stream backward, unpruned and pruned at 0.3 / 0.5 by the Model's own
groups (pruned_by_groups: odd widths such as 179 / 358 where no GroupNorm is in the group).

Bounds: the losses and the accumulated-gradient fingerprints use the C1 loop's bounds (tests/test_unet_gpu.py: 5e-6 relative L2 over
the loss sequence, 5e-3 on the squared-gradient sums); float64 gradients use conftest.worst_grad_err's 1e-4."""
import gc

import pytest
import torch

from conftest import load_golden, max_rel, rel_err, worst_grad_err
from oracle import ddpm_exp_oracle as xo

import diff_pruning_b200.ddpm_exp as de

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    return L.load()


def _gold():
    return load_golden("ddpm_exp_loop_tiny.pt")


def _betas(config):
    return de.beta_schedule(de.dict2namespace(config))


def _tiny(g):
    torch.manual_seed(g["seed"])
    return de.Model(g["config"]).eval().cuda()


def _check_fingerprints(m, fps):
    """Squared-gradient sums within 5e-3 relative.  The AttnBlocks' k biases get a gradient that is zero in exact arithmetic (the softmax
    over keys does not see q.b_k), so both sides hold rounding noise there: an absolute 1e-8 of the largest sum covers it."""
    top = max(f[2] for f in fps.values())
    for k, p in m.named_parameters():
        assert float((p.grad.double() ** 2).sum()) == pytest.approx(fps[k][2], rel=5e-3, abs=1e-8 * top), k


# ---------------------------------------------------------------------------------------------------------------------- the reference's loop
def test_tiny_loop_matches_reference(lib):
    g = _gold()
    m = _tiny(g)
    losses, stop = de.taylor_loop(m, g["x"].cuda(), g["e"].cuda(), _betas(g["config"]))
    err = rel_err(losses, g["losses"])
    print(f"tiny 1000-step loop: loss rel-L2 {err:.2e}")
    assert stop is None and losses.shape == (1000,) and err < 5e-6
    _check_fingerprints(m, g["grad_fp"])


def test_tiny_ours_stops_where_reference_stops(lib):
    g = _gold()
    o = g["ours"]
    m = _tiny(g)
    losses, stop = de.taylor_loop(m, g["x"].cuda(), g["e"].cuda(), _betas(g["config"]), pruner="ours", thr=o["thr"])
    print(f"ours: stop {stop} (reference {o['stop']}), ratio margin {o['margin']:.2e}")
    assert stop == o["stop"] and len(losses) == stop + 1 and rel_err(losses, o["losses"]) < 5e-6
    _check_fingerprints(m, o["grad_fp"])       # the stopping step's backward did not run


# ---------------------------------------------------------------------------------------------------------------------- CIFAR-10 config
def pruned_by_groups(model, ratio):
    """The Model pruned at `ratio` by its own pruning groups (pruning.build_groups through the torch_pruning surface, magnitude
    importance, conv_out ignored): the widths prune.py leaves, GroupNorm-coupled groups in whole multiples of 32 channels, q / k / v and
    the time embedding at int(n (1 - ratio)) (179 and 358 at 0.3)."""
    from diff_pruning_b200.compat import torch_pruning as tp
    ex = {"x": torch.zeros(1, 3, 32, 32), "t": torch.ones(1)}
    tp.pruner.MagnitudePruner(model, ex, importance=tp.importance.MagnitudeImportance(), ch_sparsity=ratio,
                              ignored_layers=[model.conv_out]).step()
    return model


def _cifar(ratio=None):
    torch.manual_seed(0)
    m = de.Model(de.CIFAR10_CONFIG).eval()
    if ratio is not None:
        m = pruned_by_groups(m, ratio)
    return m.cuda()


NETS = [None, 0.3, 0.5]


def _inputs(B, seed=6):
    gen = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, 32, 32, generator=gen) * 2 - 1
    return x.cuda(), torch.randn(B, 3, 32, 32, generator=gen).cuda()


@pytest.mark.parametrize("ratio", NETS)
def test_cifar10_gradients_match_float64_autograd(lib, ratio):
    """noise_estimation_loss(model, x, t, e, b).backward() through Model.forward's autograd node at t = 0, 500 and 999 (gradients
    cleared between them), against the same loss on the float64 oracle."""
    m = _cifar(ratio)
    B = 4
    x, e = _inputs(B)
    b = _betas(de.CIFAR10_CONFIG).cuda()
    sd = {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}
    a_all = (1 - b).cumprod(0).double().cpu()
    worst = 0.0
    for step in (0, 500, 999):
        m.zero_grad()
        t = torch.full((B,), step, dtype=torch.long, device="cuda")
        loss = de.noise_estimation_loss(m, x, t, e, b)
        loss.backward()
        for v in sd.values():
            v.grad = None
        a = a_all[step]
        xt = x.double().cpu() * a.sqrt() + e.double().cpu() * (1 - a).sqrt()
        out = xo.forward(sd, xt, t.double().cpu(), shortcuts=xo.shortcuts_of(m))
        ref = (e.double().cpu() - out).square().sum(dim=(1, 2, 3)).mean()
        ref.backward()
        assert float(loss) == pytest.approx(float(ref), rel=1e-5), step
        err = worst_grad_err(((k, p.grad) for k, p in m.named_parameters()), {k: v.grad for k, v in sd.items()})
        worst = max(worst, err)
        print(f"ratio {ratio} t={step}: loss {float(loss):.6f} (float64 {float(ref):.6f}), worst grad err {err:.2e}")
    assert worst < 1e-4


def test_graph_replay_equals_eager(lib):
    x, e = _inputs(8, seed=7)
    b = _betas(de.CIFAR10_CONFIG)
    res = []
    for use_graph in (True, False):
        m = _cifar(0.3)
        losses, _ = de.taylor_loop(m, x, e, b, n_steps=4, use_graph=use_graph)
        res.append((losses, [p.grad.clone() for p in m.parameters()]))
    (la, ga), (lb, gb) = res
    assert torch.equal(la, lb) and all(torch.equal(u, v) for u, v in zip(ga, gb))
    assert bool(torch.isfinite(la).all()) and all(bool(torch.isfinite(u).all()) for u in ga)


def test_loop_bit_identical_under_poisoned_allocations(lib):
    from test_pruned_widths_host import poisoned_alloc
    x, e = _inputs(4, seed=8)
    b = _betas(de.CIFAR10_CONFIG)
    outs = []
    for v in (float("nan"), 1e30, 0.0):
        m = _cifar(0.5)
        with poisoned_alloc(v) as cnt:
            losses, _ = de.taylor_loop(m, x, e, b, n_steps=3)
            outs.append((losses, [p.grad.clone() for p in m.parameters()]))
        assert cnt.n > 0
        del m
        gc.collect()
        torch.cuda.empty_cache()
    ref_l, ref_g = outs[2]
    assert bool(torch.isfinite(ref_l).all()) and all(bool(torch.isfinite(g).all()) for g in ref_g)
    for losses, grads in outs[:2]:
        assert torch.equal(losses, ref_l) and all(torch.equal(u, v) for u, v in zip(grads, ref_g))


# ---------------------------------------------------------------------------------------------------------------------- census, audits
def _loop_run(m, B=16, steps=2):
    x, e = _inputs(B, seed=9)
    b = _betas(de.CIFAR10_CONFIG)
    return lambda: de.taylor_loop(m, x, e, b, n_steps=steps, use_graph=False)


@pytest.mark.parametrize("ratio", NETS)
def test_backward_plan_census(lib, ratio):
    """Every distinct launch of two eager Taylor steps of the CIFAR-10 Model plan at batch 16 replayed on fresh seeded buffers and
    checked against float64 (the bounds of launch_census.py) or bit for bit."""
    from test_launch_census_gpu import INSIDE, REPLAY, _capture, _unique
    calls = _capture(lib, _loop_run(_cifar(ratio)))
    gc.collect()
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert {"dp_conv2d_dgrad", "dp_conv2d_wgrad", "dp_groupnorm_bwd", "dp_mse_loss_grad", "dp_upsample2x_bwd"} <= kinds
    missing = kinds - set(REPLAY) - set(INSIDE)
    assert not missing, f"launch kinds without a replay: {sorted(missing)}"
    rep, failures = {}, []
    g = torch.Generator().manual_seed(2032)
    uniq = _unique(calls)
    for name, args in uniq:
        if name in INSIDE:
            continue
        try:
            REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print("  FAIL", f)
    assert not failures
    assert kinds - set(INSIDE) <= set(rep), sorted(kinds - set(INSIDE) - set(rep))
    print(f"\nddpm_exp Taylor census ratio {ratio}: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds")
    for name in sorted(rep):
        print(f"  {name:26s} worst err/bound {max(rep[name]):.3f}")


@pytest.mark.parametrize("ratio", NETS)
def test_backward_plan_amax_slots_bound_their_operands(lib, ratio):
    import launch_census as lc
    import slot_audit as sa
    from test_slot_audit_gpu import GRAD, MAX_LOOSENESS
    run = _loop_run(_cifar(ratio), B=8)
    audit = sa.SlotAudit()
    with lc.wrap_launches(lib, audit):
        run()
        torch.cuda.synchronize()
    worst, where = audit.worst()
    print(f"\nddpm_exp Taylor ratio {ratio}: {audit.launches} launches name an input slot, {audit.audited} audited ({audit.simt} SIMT), "
          f"{len(audit.failures)} below the maximum; worst looseness {worst:.4g} at {where}")
    assert not audit.failures, audit.failures[:3]
    assert audit.audited > 0 and audit.audited + audit.simt == audit.launches
    assert GRAD <= audit.kinds
    assert worst <= MAX_LOOSENESS


@pytest.mark.parametrize("ratio", NETS)
def test_two_stream_backward_has_no_race(lib, ratio):
    """The race audit of the two-stream backward (stream_order.py over footprint.py's launch footprints) over two eager steps and
    two graph-replayed steps of the loop."""
    from test_stream_races_gpu import Recorded, _check, _plans, _record
    m = _cifar(ratio)
    x, e = _inputs(16, seed=10)
    b = _betas(de.CIFAR10_CONFIG)

    def run():
        de.taylor_loop(m, x, e, b, n_steps=2, use_graph=False)
        return de.taylor_loop(m, x, e, b, n_steps=2, use_graph=True)
    r = Recorded(_record(lib, run), _plans(m))
    _check(f"ddpm_exp Taylor ratio {ratio}", r)


def test_autograd_path_refuses_input_grad_and_dropout(lib):
    m = _cifar()
    x, e = _inputs(2)
    with pytest.raises(RuntimeError):
        m(x.requires_grad_(True), torch.zeros(2, device="cuda"))
    m.train()
    with pytest.raises(RuntimeError):
        m(x.detach(), torch.zeros(2, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------- ddpm_exp.prune
def _selections_agree(got, want, tol=1e-3):
    """The selected channels of one group equal the reference's, or differ only between channels whose reference importance lies within
    `tol` (relative) of the selection boundary of their GroupNorm sub-group: near-ties that the engine's gradient (fp32-grade, another
    summation order) may order either way.  Returns whether the selections are identical."""
    if sorted(got["idxs"]) == sorted(want["idxs"]):
        return True
    imp = want["imp"].double().cpu()
    size = want["channels"] // want["ch_groups"]
    for i in set(got["idxs"]) ^ set(want["idxs"]):
        lo = i // size * size
        sel = [j for j in want["idxs"] if lo <= j < lo + size]
        rest = sorted(set(range(lo, lo + size)) - set(sel))
        thr = (float(imp[sel].max()) + float(imp[rest].min())) / 2
        assert abs(float(imp[i]) - thr) <= tol * abs(thr), (want["root"], i, float(imp[i]), thr)
    return False


@pytest.mark.parametrize("pruner", de.PRUNERS)
def test_prune_matches_reference_for_every_criterion(lib, pruner):
    """ddpm_exp.prune on the tiny Model at the golden's ratio, e the reference's (randn_like replaced for the call): the group order,
    n_pruned, the selected channels (up to near-ties, _selections_agree), MACs and parameters before and after; when every selection is
    identical, the pruned state dict's digest and eps_hat (reinit: its re-drawn weights come from the device generator, so shapes only)."""
    from oracle import vq_oracle as vo
    G = load_golden("ddpm_exp_prune_tiny.pt")
    want = G["criteria"][pruner]
    torch.manual_seed(0)
    m = de.Model(G["config"]).eval().cuda()
    loop = load_golden("ddpm_exp_loop_tiny.pt")
    orig = torch.randn_like
    torch.randn_like = lambda x, *a, **k: G["e"].to(x.device).clone() if x.shape == G["e"].shape else orig(x, *a, **k)
    try:
        res = de.prune(m, G["config"], loop["x01"].cuda(), pruner, G["ratio"], thr=G["thr"], timesteps=4)
    finally:
        torch.randn_like = orig
    assert [g["root"] for g in res.groups] == [w["root"] for w in want["groups"]]
    exact = True
    for got, w in zip(res.groups, want["groups"]):
        assert (got["n_pruned"], got["ch_groups"]) == (w["n_pruned"], w["ch_groups"]), w["root"]
        exact = _selections_agree(got, w) and exact if w["imp"] is not None else (sorted(got["idxs"]) == sorted(w["idxs"]) and exact)
    assert exact or pruner not in ("magnitude", "random", "reinit")
    assert res.macs == pytest.approx((want["base"][0], want["pruned"][0])) and res.params == (want["base"][1], want["pruned"][1])
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    assert {k: list(v.shape) for k, v in sd.items()} == want["shapes"]
    assert res.samples.shape == (G["config"]["sampling"]["batch_size"], 3, 16, 16) and bool(torch.isfinite(res.samples).all())
    if pruner in ("taylor", "ours", "first_order_taylor", "second_order_taylor", "abs_taylor", "fisher"):
        assert res.losses.shape[0] == (1000 if pruner != "ours" else loop["ours"]["stop"] + 1)
    print(f"{pruner}: selections {'identical' if exact else 'equal up to near-ties'}")
    if exact and pruner != "reinit":
        assert vo.state_dict_digest(sd) == want["digest"]
        with torch.no_grad():
            eps = m(G["x"][:2].cuda(), torch.full((2,), 500.0, device="cuda"))
        assert max_rel(eps, want["eps_t500"]) < 1e-4


def test_pruned_cifar10_model_saves_reloads_and_samples(lib, tmp_path):
    from test_ddpm_exp_host import save_as_reference
    torch.manual_seed(0)
    m = de.Model(de.CIFAR10_CONFIG).eval().cuda()
    x01 = torch.rand(4, 3, 32, 32, generator=torch.Generator().manual_seed(12)).cuda()
    res = de.prune(m, de.CIFAR10_CONFIG, x01, "taylor", 0.3, n_steps=4, timesteps=2)
    assert res.params[1] < 0.6 * res.params[0] and res.macs[1] < res.macs[0]
    path = save_as_reference(m.cpu(), tmp_path / "pruned.pth")
    back = de.load_model(de.CIFAR10_CONFIG, pruned=path).cuda()
    assert all(torch.equal(a.cpu(), b) for a, b in zip(back.state_dict().values(), m.state_dict().values()))
    mu, sigma, n = de.sample_fid(back, de.CIFAR10_CONFIG, str(tmp_path / "imgs"), total=4, batch_size=4, timesteps=2)
    assert n == 4 and len(list((tmp_path / "imgs").glob("*.png"))) == 4
