"""Host checks of prune_ldm.py's sample-then-score loop (ldm_sampling.py) against tests/golden/ldm_ddim_tiny.pt, which the unmodified
reference DDIMSampler / UNetModel / ClassEmbedder produced (tools/gen_golden.py ldm_ddim): the DDIM schedule and per-step scalars bit for bit,
the state-dict names and the Lightning-checkpoint load, the stop rule of --pruner diff-pruning / diff0 / taylor, and the float32 oracle
sampler and loss of tests/ldm_sampling_oracle.py against the reference's trajectories."""
import hashlib
import math

import numpy as np
import pytest
import torch

from conftest import load_golden, max_rel



def _unpack(g):
    """The fixture keeps one stacked tensor per field (tools/gen_golden.py gen_ldm_ddim); the tests read per-step records and named
    gradient samples."""
    for r in g["runs"].values():
        st = r["steps"]
        r["steps"] = [] if st is None else [{"t": int(st["t"][i]), "index": int(st["index"][i]), "raw": st["raw"][i],
                                             "x_prev": st["x_prev"][i], "pred_x0": st["pred_x0"][i]} for i in range(len(st["t"]))]
    g["grad_samples"] = {k: v[:int(n)] for k, v, n in zip(g["grad_names"], g["grad_samples"], g["grad_numel"].clamp(max=32))}
    g["grad_fp"] = dict(zip(g["grad_names"], g["grad_fp"].tolist()))
    return g


GOLD = _unpack(load_golden("ldm_ddim_tiny.pt"))
RUNS = list(GOLD["runs"].keys())
SHAPE = tuple(GOLD["x_T"].shape)          # (B, 3, H, W) of the reference's samples


def grad_sample_err(named_grads):
    """Gradients against the fixture's first 32 elements and (sum, sum |g|, sum g^2) of every UNet gradient: the worst over parameters
    of min(relative error of the sample, max-abs error / the largest gradient RMS) (as conftest.worst_grad_err, for the identically-zero
    and pure-cancellation gradients), and of the relative error of sum g^2 against the same floor."""
    fp = GOLD["grad_fp"]
    numel = dict(zip(GOLD["grad_names"], GOLD["grad_numel"].tolist()))
    top = max((f[2] / numel[k]) ** 0.5 for k, f in fp.items())
    worst = 0.0
    for k, g in named_grads:
        ref, got = GOLD["grad_samples"][k].double(), g.detach().double().cpu().flatten()[:32]
        d = float((got - ref).abs().max())
        worst = max(worst, min(d / max(float(ref.abs().max()), 1e-30), d / top))
        sq = float((g.detach().double() ** 2).sum())
        worst = max(worst, abs(sq - fp[k][2]) / max(fp[k][2], top * top * numel[k] * 1e-6))
    return worst


def _f32(v):
    return torch.tensor([float(v)], dtype=torch.float32)


@pytest.mark.parametrize("run", RUNS, ids=[f"S{S}-s{s:g}-eta{e:g}" for S, s, e in RUNS])
def test_schedule_and_step_scalars_equal_the_reference(run):
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import ddim_schedule
    S, _, eta = run
    ref = GOLD["runs"][run]
    sch = ddim_schedule(ldm.ldm_alphas_cumprod(), S, eta)
    rs = ref["sched"]
    assert np.array_equal(sch.ddim_timesteps, rs["ddim_timesteps"]["value"].numpy())
    assert torch.equal(sch.ddim_alphas, rs["ddim_alphas"]["value"])
    assert sch.ddim_alphas.dtype == torch.float32 and rs["ddim_alphas"]["dtype"] == "torch.float32"
    assert np.array_equal(sch.ddim_alphas_prev, rs["ddim_alphas_prev"]["value"].numpy()) and sch.ddim_alphas_prev.dtype == np.float64
    assert torch.equal(sch.ddim_sigmas, rs["ddim_sigmas"]["value"]) and sch.ddim_sigmas.dtype == torch.float64
    assert torch.equal(sch.ddim_sqrt_one_minus_alphas, rs["ddim_sqrt_one_minus_alphas"]["value"])
    full = ref["full"]
    for i in range(S):
        sb, sa, sap, dirc, sigma = sch.coefs[i]
        a_t, a_prev, sig = _f32(full["a_t"][i]), _f32(full["a_prev"][i]), _f32(full["sigma_t"][i])
        assert sb == float(full["sqrt_one_minus_at"][i]) and sigma == float(sig), i
        assert sa == float(a_t.sqrt()) and sap == float(a_prev.sqrt()), i
        assert dirc == float((1. - a_prev - sig ** 2).sqrt()), i


def test_latent_diffusion_schedule_buffers_equal_the_reference():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    m = LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16))
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev"):
        assert torch.equal(getattr(m, k), GOLD["schedule"][k]), k
    assert torch.equal(m.alphas_cumprod, ldm.ldm_alphas_cumprod())
    assert m.num_timesteps == 1000 and m.cond_stage_key == "class_label"


def _tiny_latent_diffusion():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    return LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16))


def test_state_dict_names_match_the_reference():
    from diff_pruning_b200.ldm_sampling import ClassEmbedder
    assert list(ClassEmbedder(16).state_dict().keys()) == GOLD["emb_keys"]
    unet_keys = load_golden("ldm_tiny.pt")["sd_keys"]            # the reference UNetModel's names (gen_ldm_tiny)
    keys = list(_tiny_latent_diffusion().state_dict().keys())
    assert [k[len("model.diffusion_model."):] for k in keys if k.startswith("model.diffusion_model.")] == unet_keys
    assert set(keys) - {"model.diffusion_model." + k for k in unet_keys} == {
        "cond_stage_model.embedding.weight", "betas", "alphas_cumprod", "alphas_cumprod_prev"}


def test_lightning_checkpoint_loads_and_ignores_first_stage_and_ema():
    src = _tiny_latent_diffusion()
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(v.shape, generator=g) if v.is_floating_point() else v for k, v in src.state_dict().items()}
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev"):
        sd[k] = src.state_dict()[k].clone()
    ckpt = dict(sd)
    ckpt.update({"first_stage_model.encoder.conv_in.weight": torch.randn(128, 3, 3, 3), "first_stage_model.quantize.embedding.weight":
                 torch.randn(8192, 3), "model_ema.diffusion_modelinput_blocks00weight": torch.randn(32, 3, 3, 3),
                 "model_ema.num_updates": torch.tensor(7), "sqrt_alphas_cumprod": torch.rand(1000), "logvar": torch.zeros(1000),
                 "posterior_variance": torch.rand(1000)})
    dst = _tiny_latent_diffusion()
    res = dst.load_state_dict({"state_dict": ckpt}["state_dict"])
    assert not res.missing_keys and not res.unexpected_keys
    got = dst.state_dict()
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    del ckpt["model.diffusion_model.out.2.weight"]
    with pytest.raises(RuntimeError):
        _tiny_latent_diffusion().load_state_dict(ckpt)


# ---------------------------------------------------------------------------------------------------------------------- stop rule
def _prune_ldm_loop(losses, pruner):
    """prune_ldm.py:105-131 restated on 0-dim fp32 tensors: the iterations whose backward runs, and the number of forwards."""
    max_loss = -1
    backward = []
    n = 0
    for t, l in enumerate(losses):
        n += 1
        loss = torch.tensor(l, dtype=torch.float32)
        if loss > max_loss:
            max_loss = loss
        thres = 0.1 if pruner == "diff-pruning" else 0.0
        if pruner in ("diff-pruning", "diff0"):
            if loss / max_loss < thres:
                break
        backward.append(t)
    return backward, n


def _scorer_decisions(losses, pruner):
    from diff_pruning_b200.ldm_sampling import PruneLDMStopRule
    rule, backward, n = PruneLDMStopRule(pruner), [], 0
    for t, l in enumerate(losses):
        n += 1
        if rule.stop(l):
            break
        backward.append(t)
    return backward, n


SEQS = {
    "earliest (second iteration)": [0.8, 0.05, 0.7],
    "middle": [0.5, 0.9, 0.4, 0.2, 0.1, 0.089, 0.3],
    "at the threshold": [1.0, 0.1, np.nextafter(np.float32(0.1), np.float32(0)), 0.5],
    "never": [0.3, 0.2, 0.1, 0.5, 0.25, 0.06],
    "zero loss": [0.0, 0.0, 0.4],
}


@pytest.mark.parametrize("pruner", ["diff-pruning", "diff0", "taylor"])
@pytest.mark.parametrize("seq", list(SEQS))
def test_stop_rule_matches_prune_ldm(seq, pruner):
    losses = [float(np.float32(v)) for v in SEQS[seq]]
    assert _scorer_decisions(losses, pruner) == _prune_ldm_loop(losses, pruner)


def test_stop_rule_sequences_cover_first_middle_and_none():
    """The first iteration can never stop (loss / max_loss = 1, or NaN for a zero loss); the sequences above stop on the earliest possible
    iteration, in the middle, and never."""
    stops = {k: _prune_ldm_loop([float(np.float32(v)) for v in s], "diff-pruning")[1] for k, s in SEQS.items()}
    assert stops["earliest (second iteration)"] == 2
    assert 2 < stops["middle"] < len(SEQS["middle"])
    assert stops["never"] == len(SEQS["never"])


# ---------------------------------------------------------------------------------------------------------------------- oracle
def tiny_weights():
    """The tiny LDM UNet as gen_ldm_tiny / gen_ldm_ddim build it: seed 0, the zero-initialised convolutions re-drawn from Generator(5)
    times 0.05, and the ClassEmbedder of seed 1."""
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import ClassEmbedder
    torch.manual_seed(0)
    m = ldm.UNetModel(**ldm.LDM_TINY_CONFIG)
    g = torch.Generator().manual_seed(5)
    for p in m.parameters():
        if float(p.detach().abs().sum()) == 0 and p.dim() > 1:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.05)
    torch.manual_seed(1)
    emb = ClassEmbedder(ldm.LDM_TINY_CONFIG["context_dim"], n_classes=1001)
    return m, emb


def reference_noises(seed, S, shape=SHAPE):
    """The reference's sigma noise: torch.manual_seed(seed), then noise_like = torch.randn(shape) once per step."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(shape, generator=g) for _ in range(S)]


# float32 oracle on the CPU against the reference on the CPU: the same math, other op order (functional vs modules), so rounding noise
# that the S steps carry forward; guidance (s = 3) multiplies the eps error by up to 2 s + 1 = 7 per step.
ORACLE_TOL = {4: 2e-5, 20: 1e-4}


@pytest.mark.parametrize("run", RUNS, ids=[f"S{S}-s{s:g}-eta{e:g}" for S, s, e in RUNS])
def test_oracle_sampler_reproduces_the_reference(run):
    import ldm_sampling_oracle as orc
    from diff_pruning_b200 import ldm
    S, scale, eta = run
    ref = GOLD["runs"][run]
    m, emb = tiny_weights()
    assert hashlib.sha256(emb.embedding.weight.detach().numpy().tobytes()).hexdigest() == GOLD["embedding_sha"]
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    with torch.no_grad():
        c, uc = emb({"class_label": GOLD["labels"]}), emb({"class_label": GOLD["ulabels"]})
        x, steps = orc.sample(orc.unet_eps(sd, ldm.LDM_TINY_CONFIG), ldm.ldm_alphas_cumprod(), S, GOLD["x_T"], c, uc, scale, eta,
                              reference_noises(ref["seed"], S))
    worst = 0.0
    for i, st in enumerate(ref["steps"]):
        worst = max(worst, max_rel(steps[i]["x_prev"], st["x_prev"]), max_rel(steps[i]["pred_x0"], st["pred_x0"]))
    worst = max(worst, max_rel(x, ref["samples"]))
    assert worst < ORACLE_TOL[S], worst


def test_oracle_loss_at_t_reproduces_the_reference():
    import ldm_sampling_oracle as orc
    from diff_pruning_b200 import ldm
    m, emb = tiny_weights()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    with torch.no_grad():
        c = emb({"class_label": GOLD["labels"]})
    x0 = GOLD["runs"][(20, 3.0, 0.0)]["samples"]
    t = torch.full((SHAPE[0],), GOLD["loss_t"], dtype=torch.long)
    loss = orc.get_loss_at_t(sd, ldm.LDM_TINY_CONFIG, ldm.ldm_alphas_cumprod(), x0, c, t, GOLD["loss_noise"])
    assert math.isclose(float(loss), GOLD["loss"], rel_tol=1e-5), (float(loss), GOLD["loss"])
    assert grad_sample_err((k, sd[k].grad) for k in GOLD["grad_names"]) < 1e-4
