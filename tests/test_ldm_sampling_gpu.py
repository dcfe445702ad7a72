"""GPU checks of prune_ldm.py's sample-then-score loop (ldm_sampling.py) on one H100:

1. dp_ddim_cfg_step against a torch fp32 restatement of p_sample_ddim with torch.equal (guided scale 1 / 3 and the batch-B variant, eta 0
   and 0.5, padded pixel strides, B not a multiple of 4, both halves of the next input), and a census of its launches in a guided sample,
   each replayed at its geometry against fp64 (launch_census.ddim_step_ref);
2. the tiny LDM against the reference's DDIMSampler (tests/golden/ldm_ddim_tiny.pt): every step under teacher forcing, and the free-running
   20-step guided trajectory;
3. C5 at full width, batch 2: one 20-step guided sample and one get_loss_at_t pass against the float64 oracle on the GPU;
4. the graph sample against the eager sample, and the sample plus two loop iterations under NaN / 1e30 / 0 poisoned allocations;
5. three LDMPruneScorer iterations against the module-path composition DDIMSampler.sample + get_loss_at_t + loss.backward();
6. the diff-pruning stop rule: a forced stop leaves the arena equal to the iterations before it.
"""
import numpy as np
import pytest
import torch

import launch_census as lc
from conftest import max_rel, worst_grad_err
from test_launch_census_gpu import S, _capture, lib  # noqa: F401  (lib: the module-scoped fixture)
from test_ldm_sampling_host import GOLD, SHAPE, grad_sample_err, reference_noises, tiny_weights

B0, HW0 = SHAPE[0], list(SHAPE[1:])          # batch and (C, H, W) of the reference fixture's samples
from test_pruned_widths_host import poisoned_alloc

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------- kernel
def _torch_step(e_all, x, nz, coef32, scale, guided):
    """p_sample_ddim (ddim.py:170-202) in torch fp32 on the device, coefficients as (B, 1, 1, 1) tensors as the reference forms them."""
    B = x.shape[0]
    a_t, a_prev, sigma_t, sb = (torch.full((B, 1, 1, 1), v, device="cuda") for v in coef32)
    if guided:
        e_u, e_t = e_all.chunk(2)
        e_t = e_u + scale * (e_t - e_u)
    else:
        e_t = e_all[:B]
    pred_x0 = (x - sb * e_t) / a_t.sqrt()
    dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
    noise = sigma_t * nz * 1. if nz is not None else 0.
    return a_prev.sqrt() * pred_x0 + dir_xt + noise, pred_x0


def _kernel_coefs(coef32):
    """(sqrt(1 - a_t), sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev - sigma^2), sigma) in fp32, from (a_t, a_prev, sigma, sqrt(1 - a_t))."""
    a_t, a_prev, sig, sb = (torch.tensor([v], dtype=torch.float32) for v in coef32)
    return float(sb), float(a_t.sqrt()), float(a_prev.sqrt()), float((1. - a_prev - sig ** 2).sqrt()), float(sig)


def _run_kernel(lib, e_all, x, nz, coef32, scale, guided, ld_eps, ld_in, want_x0=True):
    """Lays eps out NHWC at pitch ld_eps (pads 1e30), runs dp_ddim_cfg_step; returns (x_out, x_in [2B or B, H, W, ld_in], pred_x0)."""
    B, C_, H, W = x.shape
    n_e = e_all.shape[0]
    eps = torch.full((n_e, H, W, ld_eps), 1e30, device="cuda")
    eps[..., :C_] = e_all.permute(0, 2, 3, 1)
    x_in = torch.full(((2 if guided else 1) * B, H, W, ld_in), -777.0, device="cuda")
    x_out = torch.full_like(x, -777.0)
    x0 = torch.full_like(x, -777.0) if want_x0 else None
    sb, sa, sap, dirc, sig = _kernel_coefs(coef32)
    assert lib.dp_ddim_cfg_step(eps.data_ptr(), ld_eps, x.data_ptr(), nz.data_ptr() if nz is not None else None, x_out.data_ptr(),
                                x_in.data_ptr(), ld_in, x0.data_ptr() if x0 is not None else None, B, C_, H, W, 1 if guided else 0,
                                scale, sb, sa, sap, dirc, sig, S()) == 0
    torch.cuda.synchronize()
    return x_out, x_in, x0


CASES = [(3, 1.0, 0.0, True, 4, 4), (3, 3.0, 0.0, True, 4, 8), (5, 3.0, 0.5, True, 8, 4), (6, 1.0, 0.5, True, 4, 4),
         (7, 3.0, 0.5, False, 4, 4), (2, 1.0, 0.0, False, 3, 3)]


@pytest.mark.parametrize("B,scale,eta,guided,ld_eps,ld_in", CASES)
def test_ddim_cfg_step_equals_torch_fp32(lib, B, scale, eta, guided, ld_eps, ld_in):
    from diff_pruning_b200 import ldm
    import ldm_sampling_oracle as orc
    g = torch.Generator().manual_seed(B * 10 + int(scale))
    C_, H, W = 3, 9, 7
    _, coefs = orc.make_schedule(ldm.ldm_alphas_cumprod(), 20, eta)
    x = (torch.randn(B, C_, H, W, generator=g) * 3).cuda()
    e_all = torch.randn((2 if guided else 1) * B, C_, H, W, generator=g).cuda()
    nz = torch.randn(B, C_, H, W, generator=g).cuda() if eta > 0 else None
    for index in (0, 7, 19):
        coef32 = tuple(float(torch.tensor([v], dtype=torch.float32)) for v in coefs[index])
        x_out, x_in, x0 = _run_kernel(lib, e_all, x, nz, coef32, scale, guided, ld_eps, ld_in)
        want, want_x0 = _torch_step(e_all, x, nz, coef32, scale, guided)
        assert torch.equal(x_out, want), (index, float((x_out - want).abs().max()))
        assert torch.equal(x0, want_x0), index
        halves = x_in.chunk(2) if guided else (x_in,)
        for h in halves:
            assert torch.equal(h[..., :C_], want.permute(0, 2, 3, 1)), index
            assert bool((h[..., C_:] == -777.0).all()), "pad channels of the next input were written"
        if guided:
            assert torch.equal(halves[0], halves[1])
        x_out2, _, none = _run_kernel(lib, e_all, x, nz, coef32, scale, guided, ld_eps, ld_in, want_x0=False)
        assert none is None and torch.equal(x_out2, x_out)


def _tiny_ld():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    m, emb = tiny_weights()
    ld = LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=ldm.LDM_TINY_CONFIG["context_dim"]))
    ld.model.diffusion_model.load_state_dict(m.state_dict())
    ld.cond_stage_model.load_state_dict(emb.state_dict())
    return ld.cuda()


def _conds(ld, labels, ulabels):
    with torch.no_grad():
        return (ld.get_learned_conditioning({"class_label": labels.cuda()}), ld.get_learned_conditioning({"class_label": ulabels.cuda()}))


def test_ddim_cfg_step_census(lib):
    """Every distinct dp_ddim_cfg_step launch of a guided and an unguided eta-0.5 sample of the tiny LDM (the fixture's x_T), replayed on fresh seeded
    buffers at its geometry: bit-exact against the torch fp32 restatement and within launch_census.ddim_step_ref's fp64 bound."""
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ld = _tiny_ld()
    c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])

    def run():
        for scale in (3.0, 1.0):
            sm = DDIMSampler(ld)
            sm.use_graph = False
            sm.sample(S=4, batch_size=B0, shape=HW0, conditioning=c, eta=0.5, x_T=GOLD["x_T"].cuda(),
                      unconditional_guidance_scale=scale, unconditional_conditioning=uc, generator=torch.Generator().manual_seed(3))
    calls = [(n, a) for n, a in _capture(lib, run) if n == "dp_ddim_cfg_step"]
    assert len(calls) == 8
    seen, rep = {}, {}
    for name, args in calls:
        seen.setdefault(lc.launch_key(name, lc.argkinds(name), args), args)
    g = torch.Generator().manual_seed(17)
    for args in seen.values():
        replay_ddim_cfg_step(lib, g, "dp_ddim_cfg_step", args, rep)
    print(f"\ndp_ddim_cfg_step census: {len(calls)} launches, {len(seen)} distinct, worst err/bound {max(rep['dp_ddim_cfg_step']):.3g}")


def replay_ddim_cfg_step(lib, g, name, args, rep):
    """One captured dp_ddim_cfg_step launch replayed on fresh seeded buffers at its geometry, pitches and fp32 coefficients: bit-exact
    against the torch fp32 restatement, and within launch_census.ddim_step_ref's fp64 bound (err / bound appended to rep[name])."""
    _, ld_eps, _, nzp, _, _, ld_in, _, B, C_, H, W, guided, scale, sb, sa, sap, dirc, sig = args
    x = torch.randn(B, C_, H, W, generator=g).cuda() * 4
    e_all = torch.randn((2 if guided else 1) * B, C_, H, W, generator=g).cuda()
    nz = torch.randn(B, C_, H, W, generator=g).cuda() if nzp else None
    out, _, x0 = _run_kernel_raw(lib, e_all, x, nz, ld_eps, ld_in, guided, scale, (sb, sa, sap, dirc, sig))
    e = e_all[:B] + scale * (e_all[B:] - e_all[:B]) if guided else e_all[:B]
    k = [torch.full((B, 1, 1, 1), v, device="cuda") for v in (sb, sa, sap, dirc, sig)]
    want_x0 = (x - k[0] * e) / k[1]
    want = k[2] * want_x0 + k[3] * e + (k[4] * nz if nz is not None else 0.)
    assert torch.equal(x0, want_x0) and torch.equal(out, want), "dp_ddim_cfg_step is not bit-exact"
    r64, bound = lc.ddim_step_ref(x, e, nz, sb, sa, 0.0, sap, dirc, sig)
    w, where = lc.violations(out, r64, bound)
    assert not where, where
    rep.setdefault(name, []).append(w)


def _run_kernel_raw(lib, e_all, x, nz, ld_eps, ld_in, guided, scale, k):
    B, C_, H, W = x.shape
    eps = torch.full((e_all.shape[0], H, W, ld_eps), 1e30, device="cuda")
    eps[..., :C_] = e_all.permute(0, 2, 3, 1)
    x_in = torch.full(((2 if guided else 1) * B, H, W, ld_in), -777.0, device="cuda")
    x_out, x0 = torch.full_like(x, -777.0), torch.full_like(x, -777.0)
    assert lib.dp_ddim_cfg_step(eps.data_ptr(), ld_eps, x.data_ptr(), nz.data_ptr() if nz is not None else None, x_out.data_ptr(),
                                x_in.data_ptr(), ld_in, x0.data_ptr(), B, C_, H, W, guided, scale, *k, S()) == 0
    torch.cuda.synchronize()
    return x_out, x_in, x0


# ---------------------------------------------------------------------------------------------------------------------- tiny vs reference
RUNS_STEPPED = [k for k, v in GOLD["runs"].items() if v["steps"]]
EPS_TOL = 1e-4          # the eps_hat bound of the engine (BASELINE north star), also for x_prev after one step


@pytest.mark.parametrize("run", RUNS_STEPPED, ids=[f"S{S_}-s{s:g}-eta{e:g}" for S_, s, e in RUNS_STEPPED])
def test_tiny_teacher_forced_steps_match_the_reference(lib, run):
    """Each step from the reference's own x_t: the engine forward at batch 2B (B when unguided), the guided combine and the update by
    dp_ddim_cfg_step, against the reference's raw eps, combine and x_prev / pred_x0."""
    from diff_pruning_b200.ldm_sampling import ddim_schedule
    from diff_pruning_b200 import ldm
    S_, scale, eta = run
    ref = GOLD["runs"][run]
    ld = _tiny_ld()
    unet = ld.model.diffusion_model.eval()
    c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
    guided = scale != 1.0
    sch = ddim_schedule(ldm.ldm_alphas_cumprod(), S_, eta)
    noises = reference_noises(ref["seed"], S_)
    x = GOLD["x_T"].cuda()
    worst = {"eps": 0.0, "e": 0.0, "x_prev": 0.0, "pred_x0": 0.0}
    for i, st in enumerate(ref["steps"]):
        tt = torch.full((2 * B0 if guided else B0,), st["t"], dtype=torch.long, device="cuda")
        with torch.no_grad():
            e_all = unet(torch.cat([x, x]) if guided else x, tt, context=torch.cat([uc, c]) if guided else c)
        raw = st["raw"].cuda()
        worst["eps"] = max(worst["eps"], max_rel(e_all, raw))
        nz = noises[i].cuda() if eta > 0 else None
        out, x_in, x0 = _run_kernel_raw(lib, e_all, x, nz, 4, 4, 1 if guided else 0, scale, sch.coefs[st["index"]])
        e = e_all[:B0] + scale * (e_all[B0:] - e_all[:B0]) if guided else e_all
        e_ref = raw[:B0] + scale * (raw[B0:] - raw[:B0]) if guided else raw
        worst["e"] = max(worst["e"], max_rel(e, e_ref))
        worst["x_prev"] = max(worst["x_prev"], max_rel(out, st["x_prev"]))
        worst["pred_x0"] = max(worst["pred_x0"], max_rel(x0, st["pred_x0"]))
        x = st["x_prev"].cuda()
    print(f"\nteacher-forced {run}: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert max(worst.values()) < EPS_TOL, worst


# Free-running 20-step guided trajectory.  Measured on one H100 with the fixture's 8 x 8 latents: the UNet's eps_hat is within 2.8e-6 of the
# reference's per step, the guided combine e_u + 3 (e_c - e_u) raises that to 8.0e-6 (at worst 2 s + 1 = 7 times), and one update turns it
# into at most 2.2e-6 on x_prev (teacher forcing); run freely, the error does not compound (1.3e-6 at the logged steps from the first to the
# twentieth; C5 at full width ends at 2.7e-6).  The bound is the largest teacher-forced guided combine error with a margin of 2.5: 2e-5.
FREE_TOL = 2e-5


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_tiny_free_running_guided_sample_matches_the_reference(lib, eta):
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ref = GOLD["runs"][(20, 3.0, eta)]
    ld = _tiny_ld()
    c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
    sm = DDIMSampler(ld)
    samples, inter = sm.sample(S=20, batch_size=B0, shape=HW0, conditioning=c, eta=eta, x_T=GOLD["x_T"].cuda(), log_every_t=5,
                               unconditional_guidance_scale=3.0, unconditional_conditioning=uc,
                               generator=torch.Generator().manual_seed(ref["seed"]))
    logged = [i for i in range(20) if (20 - i - 1) % 5 == 0 or i == 0]          # ddim.py:158: index % log_every_t == 0 or the first step
    assert len(inter["x_inter"]) == len(ref["x_inter"]) == len(logged) + 1
    assert torch.equal(inter["x_inter"][0], GOLD["x_T"].cuda()) and len(inter["pred_x0"]) == len(logged) + 1
    assert all(torch.equal(a, sm.last_run.xs[i]) for a, i in zip(inter["x_inter"][1:], logged))
    per_step = [max_rel(a, b) for a, b in zip(inter["x_inter"][1:], ref["x_inter"][1:])]
    print(f"\nfree-running S20 s3 eta {eta}: x_prev max-rel at steps {logged}: " + " ".join(f"{v:.1e}" for v in per_step))
    assert max(per_step) < FREE_TOL and max_rel(samples, ref["samples"]) < FREE_TOL


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_tiny_unguided_sample_matches_the_reference(lib, eta):
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ref = GOLD["runs"][(4, 1.0, eta)]
    ld = _tiny_ld()
    c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
    samples, _ = DDIMSampler(ld).sample(S=4, batch_size=B0, shape=HW0, conditioning=c, eta=eta, x_T=GOLD["x_T"].cuda(),
                                        unconditional_guidance_scale=1.0, unconditional_conditioning=uc,
                                        generator=torch.Generator().manual_seed(ref["seed"]))
    assert max_rel(samples, ref["samples"]) < 4 * EPS_TOL


def test_tiny_get_loss_at_t_matches_the_reference(lib):
    ld = _tiny_ld()
    x0 = GOLD["runs"][(20, 3.0, 0.0)]["samples"].cuda()
    ld.zero_grad()
    t = torch.full((B0,), GOLD["loss_t"], dtype=torch.long, device="cuda")
    loss, _ = ld.get_loss_at_t(x0, {"class_label": GOLD["labels"].cuda()}, t, noise=GOLD["loss_noise"].cuda())
    loss.backward()
    assert float(loss) == pytest.approx(GOLD["loss"], rel=5e-6)
    unet = ld.model.diffusion_model
    assert grad_sample_err((k, p.grad) for k, p in unet.named_parameters()) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------- C5 vs fp64
def _c5_ld():
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    m, cfg = lc.c5_model()
    ld = LatentDiffusion()
    ld.model.diffusion_model.load_state_dict(m.state_dict())
    torch.manual_seed(1)
    ld.cond_stage_model.embedding.weight.data.normal_()
    return ld.cuda(), cfg


def test_c5_guided_sample_and_loss_vs_fp64_oracle(lib):
    """cin256-v2 at full width, batch 2 (4 images per forward): one 20-step scale-3 sample and one get_loss_at_t pass at t = 5 on the
    engine's samples against ldm_sampling_oracle in float64 on the GPU."""
    import ldm_sampling_oracle as orc
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ld, cfg = _c5_ld()
    B = 2
    labels, ulabels = torch.tensor([25, 992]), torch.full((B,), 1000)
    c, uc = _conds(ld, labels, ulabels)
    x_T = torch.randn(B, 3, 64, 64, generator=torch.Generator().manual_seed(21)).cuda()
    samples, _ = DDIMSampler(ld).sample(S=20, batch_size=B, shape=[3, 64, 64], conditioning=c, eta=0.0, x_T=x_T,
                                        unconditional_guidance_scale=3.0, unconditional_conditioning=uc)
    unet = ld.model.diffusion_model
    sd = {k: v.detach().double().clone() for k, v in unet.state_dict().items()}
    with torch.no_grad():
        ref, _ = orc.sample(orc.unet_eps(sd, cfg), ld.alphas_cumprod, 20, x_T.double(), c.double(), uc.double(), 3.0, 0.0)
    lat = max_rel(samples, ref)
    noise = torch.randn(B, 3, 64, 64, generator=torch.Generator().manual_seed(22)).cuda()
    t = torch.full((B,), 5, dtype=torch.long, device="cuda")
    ld.zero_grad()
    loss, _ = ld.get_loss_at_t(samples, {"class_label": labels.cuda()}, t, noise=noise)
    loss.backward()
    sd = {k: v.requires_grad_(True) for k, v in sd.items()}
    loss_ref = orc.get_loss_at_t(sd, cfg, ld.alphas_cumprod, samples.double(), c.double(), t, noise.double())
    grad = worst_grad_err(((k, p.grad) for k, p in unet.named_parameters()), {k: v.grad for k, v in sd.items()})
    print(f"\nC5 b2 DDIM-20 s3: latents max-rel {lat:.2e}; loss {float(loss):.9f} (fp64 {float(loss_ref):.9f}); worst gradient {grad:.2e}")
    assert lat < FREE_TOL
    assert float(loss) == pytest.approx(float(loss_ref), rel=5e-6)
    assert grad < 1e-4


# ---------------------------------------------------------------------------------------------------------------------- graph, poison
def _labels_seq(B):
    seqs = [[3, 998, 17, 400, 5, 999][:B], [250, 1, 77, 930, 12, 600][:B], [8, 8, 500, 42, 990, 2][:B], [100, 200, 300, 400, 500, 600][:B]]
    it = iter(seqs)
    return lambda n: next(it)


def _loop(ld, B, iters, pruner="taylor", use_graph=True, S_=4):
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    unet = ld.model.diffusion_model
    unet.zero_grad()
    sc = LDMPruneScorer(ld, n_samples_per_class=B, ddim_steps=S_, scale=3.0, use_graph=use_graph)
    losses = sc.run(pruner, iterations=iters, class_sampler=_labels_seq(B), generator=torch.Generator().manual_seed(31))
    torch.cuda.synchronize()
    return sc, losses, {k: p.grad.clone() for k, p in unet.named_parameters()}


def test_graph_sample_equals_eager_sample(lib):
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ld = _tiny_ld()
    c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
    outs = []
    for use_graph in (True, False):
        sm = DDIMSampler(ld)
        sm.use_graph = use_graph
        s, inter = sm.sample(S=20, batch_size=B0, shape=HW0, conditioning=c, eta=0.5, x_T=GOLD["x_T"].cuda(),
                             unconditional_guidance_scale=3.0, unconditional_conditioning=uc, generator=torch.Generator().manual_seed(5))
        outs.append((s, sm.last_run.x0s.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


POISONS = (float("nan"), 1e30, 0.0)


@pytest.fixture
def poisoned_runs():
    """fn(poison value) -> {name: tensor} run once under each poison (every torch.empty* buffer filled before the code writes it, both
    plans included); returns the three result dicts."""
    def run(fn):
        outs = []
        for v in POISONS:
            with poisoned_alloc(v) as cnt:
                outs.append(fn())
            assert cnt.n > 0
            torch.cuda.synchronize()
        return outs
    return run


def test_poisoned_sample_and_loop_are_bitwise_equal(lib, poisoned_runs):
    from diff_pruning_b200.ldm_sampling import DDIMSampler

    def fn():
        ld = _tiny_ld()
        c, uc = _conds(ld, GOLD["labels"], GOLD["ulabels"])
        s, _ = DDIMSampler(ld).sample(S=4, batch_size=B0, shape=HW0, conditioning=c, eta=0.5, x_T=GOLD["x_T"].cuda(),
                                      unconditional_guidance_scale=3.0, unconditional_conditioning=uc,
                                      generator=torch.Generator().manual_seed(5))
        _, losses, grads = _loop(ld, 2, 2)
        return {"sample": s.clone(), "losses": losses, **grads}
    outs = poisoned_runs(fn)
    for k in outs[2]:
        assert bool(torch.isfinite(outs[2][k]).all()), k
        assert torch.equal(outs[0][k], outs[2][k]) and torch.equal(outs[1][k], outs[2][k]), k


# ---------------------------------------------------------------------------------------------------------------------- fast vs module path
def test_fast_path_equals_module_path(lib):
    """Three taylor iterations of LDMPruneScorer against DDIMSampler.sample + get_loss_at_t + loss.backward() with the same labels, x_T,
    noise and timesteps: the same kernels on the same values, so the gradients are bit-identical.  (The two losses sum the same squares
    in a different order: the fast path over the padded NHWC output, get_loss_at_t over NCHW.)"""
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    B = 2
    ld = _tiny_ld()
    _, fast_losses, fast = _loop(ld, B, 3)
    unet = ld.model.diffusion_model
    unet.zero_grad()
    sm = DDIMSampler(ld)
    g = torch.Generator().manual_seed(31)
    labels = _labels_seq(B)
    with torch.no_grad():
        uc = ld.get_learned_conditioning({"class_label": torch.full((B,), 1000, device="cuda")})
    losses = []
    for t in range(3):
        xc = torch.tensor(labels(B)).cuda()
        with torch.no_grad():
            c = ld.get_learned_conditioning({"class_label": xc})
        s, _ = sm.sample(S=4, conditioning=c, batch_size=B, shape=[3, 16, 16], verbose=False, unconditional_guidance_scale=3.0,
                         unconditional_conditioning=uc, eta=0.0, generator=g)
        noise = torch.randn(s.shape, generator=g).cuda()
        loss, _ = ld.get_loss_at_t(s, {"class_label": xc}, torch.full((B,), t, device="cuda", dtype=torch.long), noise=noise)
        losses.append(float(loss))
        loss.backward()
    assert np.allclose(losses, fast_losses.tolist(), rtol=1e-6)
    bad = [k for k, p in unet.named_parameters() if not torch.equal(p.grad, fast[k])]
    assert not bad, bad[:8]


def test_forced_stop_leaves_the_gradients_of_the_earlier_iterations(lib, monkeypatch):
    from diff_pruning_b200 import ldm_sampling
    B = 2
    ld = _tiny_ld()
    _, _, two = _loop(ld, B, 2)                           # taylor: iterations 0 and 1 accumulated
    orig = ldm_sampling.PruneLDMStopRule.stop
    calls = []

    def forced(self, loss):
        calls.append(loss)
        return orig(self, loss) or len(calls) == 3         # the third iteration stops (before its backward)
    monkeypatch.setattr(ldm_sampling.PruneLDMStopRule, "stop", forced)
    sc, losses, stopped = _loop(ld, B, 10, pruner="diff-pruning")
    assert sc.stopped_at == 2 and len(losses) == 3
    bad = [k for k in two if not torch.equal(two[k], stopped[k])]
    assert not bad, bad[:8]
