"""prune.py's Taylor loop for ddpm_exp's Model on the host (no GPU): the trace-mode torch forward of Model / ResnetBlock against the
reference's eps_hat, noise_estimation_loss against the reference loop's losses (tests/golden/ddpm_exp_loop_tiny.pt, tools/gen_golden.py),
the `ours` stop rule against the reference's stop index, the loop's refusals; the Model's pruning groups and their order for the tiny and
CIFAR-10 configs, the magnitude and random selections, count_ops_and_params and the pruned pickle through load_model against
tests/golden/ddpm_exp_prune_tiny.pt."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import expand, load_golden
from test_ddpm_exp_host import seeded_tiny

import diff_pruning_b200.ddpm_exp as de
from diff_pruning_b200 import pruning
from diff_pruning_b200.compat import torch_pruning as tp
from diff_pruning_b200.models import trace_mode
from oracle import vq_oracle as vo


def _gold():
    return load_golden("ddpm_exp_loop_tiny.pt")


def test_trace_mode_forward_equals_reference():
    m, g = seeded_tiny()
    with trace_mode(), torch.no_grad():
        for t, want in g["eps"].items():
            assert torch.equal(m(g["x"], torch.full((2,), float(t))), want), t


def test_noise_estimation_loss_equals_reference_losses():
    """functions/losses.py on the trace-mode Model: the reference loop's loss at a few steps (the weights do not change in the loop, so
    every step's loss is that of the initial network), and a backward that reaches every parameter.  The AttnBlocks' k biases are left
    out: their gradient is zero in exact arithmetic (the softmax over keys does not see q.b_k) and holds rounding noise only."""
    g = _gold()
    torch.manual_seed(g["seed"])
    m = de.Model(g["config"]).eval()
    b = de.beta_schedule(de.dict2namespace(g["config"]))
    B = g["x"].shape[0]
    assert torch.equal(g["x"], 2 * g["x01"] - 1.0)
    with trace_mode():
        for step in (0, 1, 500, 999):
            loss = de.noise_estimation_loss(m, g["x"], torch.full((B,), step, dtype=torch.long), g["e"], b)
            assert float(loss) == pytest.approx(float(g["losses"][step]), rel=1e-6), step
        loss.backward()
        per_image = de.noise_estimation_loss(m, g["x"], torch.full((B,), 999, dtype=torch.long), g["e"], b, keepdim=True)
    assert per_image.shape == (B,) and float(per_image.mean()) == pytest.approx(float(loss), rel=1e-6)
    assert all(p.grad is not None and bool(p.grad.abs().sum() > 0) for n, p in m.named_parameters() if not n.endswith(".k.bias"))


def _restated(losses, thr):
    """prune.py:248-253 on 0-dim fp32 tensors, as the reference runs it."""
    max_loss = 0
    for k, l in enumerate(losses):
        loss = torch.tensor(l, dtype=torch.float32)
        if loss > max_loss:
            max_loss = loss
        if loss < max_loss * thr:
            return k
    return None


def _rule(losses, thr):
    rule = de.OursStopRule(thr)
    return next((k for k, l in enumerate(losses) if rule.stop(l)), None)


def test_ours_stop_rule_gives_reference_stop_index():
    g = _gold()
    o = g["ours"]
    losses = g["losses"].tolist()
    assert _rule(losses, o["thr"]) == o["stop"] == _restated(losses, o["thr"])
    assert torch.equal(g["losses"][:o["stop"] + 1], o["losses"])
    # the chosen thr sits mid-way between the stopping ratio and the smallest earlier one
    r = np.float32(o["losses"][-1]) / np.float32(o["losses"].max())
    assert r < o["thr"] and o["thr"] - r == pytest.approx(o["margin"], rel=1e-3)


@pytest.mark.parametrize("losses,thr", [
    ([1.0, 2.0, 1.9, 0.02, 0.01, 5.0], 0.01),          # stops at the first loss below max * thr, not at or above it
    ([0.0, 0.0, 1.0, 0.5], 0.6),                       # max_loss starts at 0: zero losses never stop
    ([1.0, float("nan"), 0.2, 0.1], 0.15),             # a NaN loss neither raises max_loss nor stops
    ([3.0, 2.0, 1.0], 0.0),                            # thr 0 never stops on non-negative losses
    ([1.0, 0.99, 0.98], 0.99),                         # fp32 product: 0.98 < 0.99 (rounded) * 1.0
])
def test_ours_stop_rule_restates_the_reference(losses, thr):
    assert _rule(losses, thr) == _restated(losses, thr)


def test_loop_refusals():
    m, g = seeded_tiny()
    x = torch.zeros(2, 3, 16, 16)
    b = de.beta_schedule(de.dict2namespace(g["config"]))
    with pytest.raises(ValueError):
        de.taylor_loop(m, x, x, b, pruner="magnitude")    # prune.py runs no loop for magnitude / random / reinit
    with pytest.raises(RuntimeError):
        de.taylor_loop(m, x, x, b)
    with pytest.raises(ValueError):
        de.taylor_loop(m, x, x, b, n_steps=1001)           # past the alphas table
    from diff_pruning_b200.scoring import TaylorScorer
    with pytest.raises(ValueError):
        TaylorScorer(m, x, x, reduction="sum")


# ---------------------------------------------------------------------------------------------------------------------- pruning groups
def _prune_gold():
    return load_golden("ddpm_exp_prune_tiny.pt")


def _items(items):
    return {(n, k): expand(i) for n, k, i in items}


def _structure_matches(groups, want):
    assert [g["root"] for g in groups] == [w["root"] for w in want]
    for g, w in zip(groups, want):
        assert (g["channels"], g["ch_groups"]) == (w["channels"], w["ch_groups"]), g["root"]
        assert _items(g["items"]) == _items(w["items"]), g["root"]


def test_tiny_group_structure_and_order_match_reference():
    """Every group of the unpruned tiny Model (root, width, GroupNorm groups, every member with its index map) in the reference's order;
    the q / k / v outputs and proj_out's input form one group, rooted at k as the reference's tracer roots it."""
    m, _ = seeded_tiny()
    _structure_matches(pruning.build_groups(m, [m.conv_out]), _prune_gold()["tiny_groups"])


def test_cifar10_group_structure_and_order_match_reference():
    torch.manual_seed(0)
    m = de.Model(de.CIFAR10_CONFIG).eval()
    g = _prune_gold()
    _structure_matches(pruning.build_groups(m, [m.conv_out]), g["cifar_groups"])
    assert tp.count_ops_and_params(m, {"x": torch.randn(1, 3, 32, 32), "t": torch.ones(1)}) == pytest.approx(g["cifar_counts"])


def _host_prune(pruner_name, ratio):
    """prune.py's pruner step for the criteria that need no gradient, through the torch_pruning surface on the host: seed, the example
    input on the CPU generator, MagnitudePruner, counts, the interactive step, counts."""
    torch.manual_seed(0)
    m = de.Model(_prune_gold()["config"]).eval()
    example = {"x": torch.randn(1, 3, 16, 16), "t": torch.ones(1)}
    imp = tp.importance.MagnitudeImportance() if pruner_name == "magnitude" else tp.importance.RandomImportance()
    mp = tp.pruner.MagnitudePruner(m, example, importance=imp, iterative_steps=1, channel_groups={}, ch_sparsity=ratio,
                                   ignored_layers=[m.conv_out], root_module_types=[nn.Conv2d, nn.Linear])
    base = tp.count_ops_and_params(m, example)
    groups = []
    for grp in mp.step(interactive=True):
        groups.append({"root": grp.root, "n_pruned": grp.n_pruned, "ch_groups": grp.ch_groups, "idxs": list(grp.idxs)})
        grp.prune()
    return m, groups, base, tp.count_ops_and_params(m, example)


@pytest.mark.parametrize("pruner_name", ["magnitude", "random"])
def test_magnitude_and_random_select_what_the_reference_selects(pruner_name):
    g = _prune_gold()
    want = g["criteria"][pruner_name]
    m, groups, base, after = _host_prune(pruner_name, g["ratio"])
    assert [x["root"] for x in groups] == [w["root"] for w in want["groups"]]
    for x, w in zip(groups, want["groups"]):
        assert (x["n_pruned"], x["ch_groups"]) == (w["n_pruned"], w["ch_groups"]) and sorted(x["idxs"]) == sorted(w["idxs"]), x["root"]
    sd = m.state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == want["shapes"] and vo.state_dict_digest(sd) == want["digest"]
    assert base == pytest.approx(want["base"]) and after == pytest.approx(want["pruned"])
    with trace_mode(), torch.no_grad():
        assert torch.allclose(m(g["x"][:2], torch.full((2,), 500.0)), want["eps_t500"], rtol=1e-5, atol=1e-5)


def test_pruned_pickle_round_trips_through_load_model(tmp_path):
    from test_ddpm_exp_host import save_as_reference
    g = _prune_gold()
    m, _, _, _ = _host_prune("magnitude", g["ratio"])
    path = save_as_reference(m, tmp_path / "pruned.pth")
    back = de.load_model(g["config"], pruned=path)
    assert list(back.state_dict()) == list(m.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(back.state_dict().values(), m.state_dict().values()))
    with trace_mode(), torch.no_grad():
        assert torch.equal(back(g["x"][:2], torch.full((2,), 500.0)), m(g["x"][:2], torch.full((2,), 500.0)))
