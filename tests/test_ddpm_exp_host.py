"""ddpm_exp's Model, checkpoints and sampling schedule on the host (no GPU): the module tree against the reference's seeded state dict,
every checkpoint form the runners load (pruned pickle, pruned list with EMA, ckpt.pth list, plain state dict), the uniform / quad
timestep sequences, the frequency table of get_timestep_embedding and the fp32 step scalars of generalized_steps.  The oracle is pinned
on the reference's eps_hat and trajectories (tests/golden/ddpm_exp_tiny.pt, tools/gen_golden.py)."""
import argparse
import contextlib
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import diff_pruning_b200.ddpm_exp as de
from diff_pruning_b200.models import ddpm_exp_frequencies, sinusoidal_frequencies
from oracle import ddpm_exp_oracle as xo
from oracle import vq_oracle as vo

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)


def gold():
    return torch.load(os.path.join(GOLD, "ddpm_exp_tiny.pt"), weights_only=False)


def seeded_tiny():
    g = gold()
    torch.manual_seed(g["seed"])
    return de.Model(g["config"]).eval(), g


REF_CLASSES = ("Model", "ResnetBlock", "AttnBlock", "Downsample", "Upsample")


@contextlib.contextmanager
def reference_class_names():
    """Inside, this package's classes carry the module path the reference's pickles name (models.diffusion.*), so torch.save(model)
    writes what prune.py:281 and runners/diffusion_simple.py:270-283 write.  Loading happens outside, through the allow-list alone."""
    pkg, mod = types.ModuleType("models"), types.ModuleType("models.diffusion")
    pkg.diffusion = mod
    saved = {n: getattr(de, n).__module__ for n in REF_CLASSES}
    old = {k: sys.modules.get(k) for k in ("models", "models.diffusion")}
    for n in REF_CLASSES:
        getattr(de, n).__module__ = "models.diffusion"
        setattr(mod, n, getattr(de, n))
    sys.modules.update({"models": pkg, "models.diffusion": mod})
    try:
        yield
    finally:
        for n in REF_CLASSES:
            getattr(de, n).__module__ = saved[n]
        for k, v in old.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def pruned_tiny(g):
    """The fixture's pruned network, rebuilt from the indices the reference's MagnitudePruner kept, with the reference runner's config
    (an argparse.Namespace carrying `device`)."""
    torch.manual_seed(g["seed"])
    m = xo.prune_like(xo.distinct_vectors(de.Model(g["config"]).eval()), g["pruned_keep"])
    m.config.device = torch.device("cpu")
    return m


def save_as_reference(obj, path):
    with reference_class_names():
        torch.save(obj, path)
    return str(path)


def reference_pickles(g, tmp_path):
    """(pruned pickle, ckpt.pth list [Module, optimizer state, epoch, step, ema_shadow]) as the reference writes them; the shadow is the
    parameters + 0.01."""
    m = pruned_tiny(g)
    shadow = [p.detach().clone() + 0.01 for p in m.parameters()]
    opt = torch.optim.Adam(m.parameters(), lr=2e-4)
    return (save_as_reference(m, tmp_path / "pruned.pth"),
            save_as_reference([m, opt.state_dict(), 3, 1234, shadow], tmp_path / "ckpt.pth"))


def test_state_dict_matches_reference():
    m, g = seeded_tiny()
    sd = m.state_dict()
    assert list(sd.keys()) == g["sd_keys"]
    assert [list(v.shape) for v in sd.values()] == g["sd_shapes"]
    assert vo.state_dict_digest(sd) == g["digest"]
    types = {type(mod) for mod in m.modules() if not list(mod.children()) and not isinstance(mod, torch.nn.ModuleList)}
    assert types <= {torch.nn.Conv2d, torch.nn.Linear, torch.nn.GroupNorm, torch.nn.Dropout}, types


def test_cifar10_config_parameter_count():
    m = de.Model(de.CIFAR10_CONFIG)
    assert sum(p.numel() for p in m.parameters()) == 35746307      # the 35.7 M-parameter CIFAR-10 UNet


def test_oracle_matches_reference_eps():
    m, g = seeded_tiny()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    for t, want in g["eps"].items():
        got = xo.forward(sd, g["x"], torch.full((2,), float(t)))
        assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()), t


def test_oracle_generalized_steps_matches_reference():
    """The oracle's generalized_steps on the oracle forward, with the reference's recorded step noise, follows the reference's 10-step
    quad trajectories at eta 0 and 0.5 (fp32, CPU: only the convolutions' summation order differs)."""
    m, g = seeded_tiny()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    betas = de.beta_schedule(de.dict2namespace(g["config"]))
    for eta, tr in g["traj"].items():
        xs, x0s = xo.generalized_steps(lambda x, t: xo.forward(sd, x, t), tr["x_T"], tr["seq"], betas, eta, list(tr["noise"]))
        assert len(tr["noise"]) == len(tr["seq"])
        got = torch.stack(xs)
        assert float((got - tr["xs"]).abs().max()) <= 1e-4 * float(tr["xs"].abs().max()), eta


def test_frequency_table_bit_identical():
    """The sinusoid frequencies of get_timestep_embedding (diffusion.py:16-18), not diffusers' (which round differently)."""
    for dim in (32, 64, 128, 256):
        half = dim // 2
        ref = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
        assert torch.equal(ddpm_exp_frequencies(dim), ref)
    assert not torch.equal(ddpm_exp_frequencies(128), sinusoidal_frequencies(128, 1))


@pytest.mark.parametrize("S", [10, 100])
@pytest.mark.parametrize("skip_type", ["uniform", "quad"])
def test_timestep_sequences(S, skip_type):
    """runners/diffusion.py:499-511 and denoising.py:13."""
    T = 1000
    if skip_type == "uniform":
        ref = list(range(0, T, T // S))
    else:
        ref = [int(s) for s in list(np.linspace(0, np.sqrt(T * 0.8), S) ** 2)]
    seq, seq_next = de.timestep_sequence(T, S, skip_type)
    assert seq == ref and seq_next == [-1] + ref[:-1]


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_step_scalars_equal_reference_expressions(eta):
    """compute_alpha + generalized_steps' fp32 expressions (denoising.py:4-7, 16-26) evaluated at full batch shape, as the reference
    evaluates them, against the one-element scalars the sampler passes to the step update."""
    betas = de.beta_schedule(de.dict2namespace(de.CIFAR10_CONFIG))
    seq, seq_next = de.timestep_sequence(1000, 100, "quad")
    got = de.step_scalars(betas, seq, seq_next, eta)

    def compute_alpha(beta, t):
        beta = torch.cat([torch.zeros(1).to(beta.device), beta], dim=0)
        return (1 - beta).cumprod(dim=0).index_select(0, t + 1).view(-1, 1, 1, 1)
    for (i, sb, sa, sap, c1, c2), (ri, rj) in zip(got, zip(reversed(seq), reversed(seq_next))):
        at, at_next = compute_alpha(betas, (torch.ones(4) * ri).long()), compute_alpha(betas, (torch.ones(4) * rj).long())
        rc1 = eta * ((1 - at / at_next) * (1 - at_next) / (1 - at)).sqrt()
        rc2 = ((1 - at_next) - rc1 ** 2).sqrt()
        want = [(1 - at).sqrt(), at.sqrt(), at_next.sqrt(), rc1, rc2]
        assert i == ri
        for v, w in zip((sb, sa, sap, c1, c2), want):
            assert torch.equal(torch.full_like(w, v), w), (i, v, w.flatten()[0])


def test_load_pruned_pickle_keeps_widths(tmp_path):
    g = gold()
    pruned, _ = reference_pickles(g, tmp_path)
    assert "models" not in sys.modules
    m = de.load_model(g["config"], pruned=pruned)
    assert type(m) is de.Model and not m.training
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["pruned_shapes"]
    assert xo.shortcuts_of(m) == g["pruned_shortcuts"]
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    for t, want in g["pruned_eps"].items():
        got = xo.forward(sd, g["x"], torch.full((2,), float(t)), xo.shortcuts_of(m))
        assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()), t


@pytest.mark.parametrize("use_ema", [False, True])
def test_load_ckpt_list_and_pruned_list(use_ema, tmp_path):
    g = gold()
    pruned, ckpt = reference_pickles(g, tmp_path)
    base = de.load_model(g["config"], pruned=pruned)
    for kw in ({"path": ckpt}, {"pruned": ckpt}):
        m = de.load_model(g["config"], use_ema=use_ema, **kw)
        assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["pruned_shapes"]
        for p, q in zip(m.parameters(), base.parameters()):
            assert torch.equal(p, q + 0.01 if use_ema else q)


def test_load_plain_state_dict_and_state_dict_list(tmp_path):
    m, g = seeded_tiny()
    sd = m.state_dict()
    torch.save(sd, tmp_path / "plain.pth")
    torch.save([sd, {}, 1, 2, [p.detach().clone() * 2 for p in m.parameters()]], tmp_path / "ckpt.pth")
    a = de.load_model(g["config"], path=str(tmp_path / "plain.pth"))
    assert vo.state_dict_digest(a.state_dict()) == g["digest"]
    b = de.load_model(g["config"], path=str(tmp_path / "ckpt.pth"), use_ema=True)
    for p, q in zip(b.parameters(), m.parameters()):
        assert torch.equal(p, q * 2)
    with pytest.raises(OSError):
        de.load_model(g["config"], path=str(tmp_path / "missing.pth"))


def test_own_pickle_round_trip(tmp_path):
    m, g = seeded_tiny()
    torch.save(m, tmp_path / "m.pth")
    r = de.load_model(g["config"], pruned=str(tmp_path / "m.pth"))
    assert vo.state_dict_digest(r.state_dict()) == g["digest"]


def test_forward_refuses_grad_and_cpu():
    m, g = seeded_tiny()
    with pytest.raises(RuntimeError):
        m(g["x"], torch.zeros(2))
    with torch.no_grad(), pytest.raises(RuntimeError):
        m(g["x"], torch.zeros(2))
