"""ddpm_exp's Model and FID sampling loop on the GPU: the Model plan against the reference's eps_hat (tiny and pruned goldens) and the
CIFAR-10 config against the float64 oracle; the step update (dp_ddim_cfg_step) equal to the reference's fp32 update; the free-running
trajectory; graph against eager; poisoned allocations; the sample_fid draws, PNG bytes and FID moments; the launch census and the amax
slot audit of the CIFAR-10 sampling plan.

Bounds: 1e-4 max-rel is the project's fp32-grade bound for a whole network's output (BASELINE.json north star), used for eps_hat.  The
free-running trajectory divides eps_hat by sqrt(a_t) (down to 0.01 at t = 999) on every step, so its bound is stated per test."""
import gc
import os

import numpy as np
import pytest
import torch

from conftest import max_rel
from oracle import ddpm_exp_oracle as xo
from test_ddpm_exp_host import gold, reference_pickles, seeded_tiny

import diff_pruning_b200.ddpm_exp as de

pytestmark = pytest.mark.gpu


def S():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    return L.load()


def _cifar(seed=0):
    torch.manual_seed(seed)
    return de.Model(de.CIFAR10_CONFIG).eval()


# ---------------------------------------------------------------------------------------------------------------------- forward
def test_tiny_forward_matches_reference(lib):
    m, g = seeded_tiny()
    m = m.cuda()
    with torch.no_grad():
        for t, want in g["eps"].items():
            got = m(g["x"].cuda(), torch.full((2,), float(t), device="cuda"))
            err = max_rel(got, want)
            print(f"tiny t={t}: max-rel {err:.2e}")
            assert err < 1e-4


def test_pruned_forward_matches_reference(lib, tmp_path):
    g = gold()
    m = de.load_model(g["config"], pruned=reference_pickles(g, tmp_path)[0]).cuda()
    with torch.no_grad():
        for t, want in g["pruned_eps"].items():
            err = max_rel(m(g["x"].cuda(), torch.full((2,), float(t), device="cuda")), want)
            print(f"pruned t={t}: max-rel {err:.2e}")
            assert err < 1e-4


def test_cifar10_forward_matches_float64_oracle(lib):
    m = _cifar().cuda()
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(64, 3, 32, 32, generator=gen)
    t = torch.randint(0, 1000, (64,), generator=gen).float()
    with torch.no_grad():
        got = m(x.cuda(), t.cuda())
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    want = xo.forward(sd, x.double(), t.double())
    err = max_rel(got.double().cpu(), want)
    print(f"CIFAR-10 batch 64: max-rel {err:.2e} against float64")
    assert err < 1e-4


# ---------------------------------------------------------------------------------------------------------------------- the step kernel
def _step(lib, e, x, nz, k, ld_eps=5, ld_in=4):
    B, C_, H, W = x.shape
    eps = torch.full((B, H, W, ld_eps), 1e30, device="cuda")
    eps[..., :C_] = e.permute(0, 2, 3, 1)
    x_in = torch.full((B, H, W, ld_in), -777.0, device="cuda")
    out, x0, tmp = torch.full_like(x, -777.0), torch.full_like(x, -777.0), torch.full_like(x, -777.0)
    de.generalized_update(lib, eps.data_ptr(), ld_eps, x, nz, out, tmp, x_in.data_ptr(), ld_in, x0.data_ptr(), *k)
    torch.cuda.synchronize()
    assert torch.equal(x_in[..., :C_], out.permute(0, 2, 3, 1)) and bool((x_in[..., C_:] == -777.0).all())
    return out, x0


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_step_update_equals_reference_update(lib, eta):
    """Teacher-forced: for the same x, eps_hat and noise, every step of a 100-step quad sample equals generalized_steps' fp32 update
    (denoising.py:21-27) evaluated by torch on the same device, value for value (torch.equal), x0 included: at eta 0 one
    dp_ddim_cfg_step launch, otherwise the noise term first and the direction term in a second launch, as the reference adds them."""
    betas = de.beta_schedule(de.dict2namespace(de.CIFAR10_CONFIG)).cuda()
    seq, seq_next = de.timestep_sequence(1000, 100, "quad")
    ac = (1 - torch.cat([torch.zeros(1).to(betas.device), betas], dim=0)).cumprod(dim=0)
    g = torch.Generator(device="cuda").manual_seed(11)
    for (i, *k), j in zip(de.step_scalars(betas, seq, seq_next, eta), reversed(seq_next)):
        x = torch.randn(4, 3, 8, 8, device="cuda", generator=g) * 3
        e, nz = torch.randn(4, 3, 8, 8, device="cuda", generator=g), torch.randn(4, 3, 8, 8, device="cuda", generator=g)
        at, at_next = ac.index_select(0, torch.full((4,), i + 1, device="cuda")).view(-1, 1, 1, 1), \
            ac.index_select(0, torch.full((4,), j + 1, device="cuda")).view(-1, 1, 1, 1)
        want, want_x0 = xo.generalized_update(x, e, nz, at, at_next, eta)
        out, x0 = _step(lib, e, x, nz, k)
        assert torch.equal(x0, want_x0) and torch.equal(out, want), (i, float((out - want).abs().max()))


# ---------------------------------------------------------------------------------------------------------------------- the loop
@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_tiny_trajectory_follows_reference(lib, eta):
    """The free-running 10-step quad sample from the reference's x_T with its recorded step noise: every step's x0 prediction within
    1e-3 max-rel of the reference's (eps_hat's 1e-4 amplified by up to 1 / sqrt(a_t) and carried through the steps), the final sample
    too."""
    m, g = seeded_tiny()
    m = m.cuda()
    tr = g["traj"][eta]
    betas = de.beta_schedule(de.dict2namespace(g["config"]))
    S_ = len(tr["seq"])
    x0s = torch.empty((S_,) + tuple(tr["x_T"].shape), device="cuda")
    noise = iter(tr["noise"].cuda())
    orig = torch.randn_like
    torch.randn_like = lambda x, *a, **k: next(noise).clone()
    try:
        out = de.sample_image(tr["x_T"].cuda(), m, betas, S_, "quad", eta, x0_out=x0s)
    finally:
        torch.randn_like = orig
    errs = [max_rel(x0s[k], tr["x0s"][k]) for k in range(S_)]
    print(f"eta {eta}: per-step x0 max-rel {max(errs):.2e}, final {max_rel(out, tr['xs'][-1]):.2e}")
    assert max(errs) < 1e-3 and max_rel(out, tr["xs"][-1]) < 1e-3


def _sample(m, x, eta=0.5, use_graph=True, steps=10):
    betas = de.beta_schedule(de.dict2namespace(de.CIFAR10_CONFIG))
    torch.cuda.manual_seed(99)
    return de.sample_image(x, m, betas, steps, "quad", eta, use_graph=use_graph)


def test_graph_replay_equals_eager(lib):
    m = _cifar().cuda()
    x = torch.randn(8, 3, 32, 32, generator=torch.Generator().manual_seed(1)).cuda()
    a, b = _sample(m, x, use_graph=True), _sample(m, x, use_graph=False)
    assert bool(torch.isfinite(a).all()) and torch.equal(a, b)


def test_loop_bit_identical_under_poisoned_allocations(lib):
    from test_pruned_widths_host import poisoned_alloc
    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(2)).cuda()
    outs = []
    for v in (float("nan"), 1e30, 0.0):
        m = _cifar().cuda()
        with poisoned_alloc(v) as cnt:
            outs.append(_sample(m, x, steps=5))
        assert cnt.n > 0
        del m
        gc.collect()
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs[2]).all()) and all(torch.equal(o, outs[2]) for o in outs)


def _cfg(n):
    cfg = dict(g for g in gold()["config"].items())
    cfg["sampling"] = {"batch_size": n, "last_only": True}
    return cfg


def test_sample_fid_draws_bytes_and_moments(lib, tmp_path):
    """Two rounds of sample_fid on the tiny Model: (1) each round starts from the x_T a torch restatement of the reference loop draws on
    the same generator after seeding with rank + seed (x_T, then one randn_like per step, eta 0 included); (2) the PNG files hold the
    bytes tvu.save_image writes for the final sample (make_grid of one image, then mul(255).add_(0.5).clamp_(0, 255) to uint8 through
    PIL); (3) the FID moments equal fid.py's statistics over the written files."""
    from PIL import Image
    from diff_pruning_b200 import fid
    m, g = seeded_tiny()
    m = m.cuda()
    cfg = de.dict2namespace(_cfg(3))
    betas = de.beta_schedule(cfg)
    seen = []
    orig = de.sample_image

    def spy(x, *a, **k):
        seen.append(x.clone())
        return orig(x, *a, **k)
    torch.manual_seed(0)
    inc = fid.InceptionV3([fid.InceptionV3.BLOCK_INDEX_BY_DIM[64]], weights=False).cuda()
    de.sample_image = spy
    try:
        mu, sigma, n = de.sample_fid(m, _cfg(3), str(tmp_path / "imgs"), total=6, timesteps=4, seed=5, inception=inc, fid_dims=64)
    finally:
        de.sample_image = orig
    assert n == 6 and len(seen) == 2
    # (1) the reference loop's draws: seed, then per round x_T and one randn_like per step
    torch.manual_seed(5)
    want = []
    for _ in range(2):
        x = torch.randn(3, 3, 16, 16, device="cuda")
        want.append(x)
        for _ in range(4):
            torch.randn_like(x)
    assert all(torch.equal(a, b) for a, b in zip(seen, want))
    # (2) the PNG bytes of the last round
    last = orig(seen[1], m, betas.cuda(), 4, "quad", 0.0)      # redraws the step noise, which eta 0 multiplies by zero
    x = torch.clamp((last + 1.0) / 2.0, 0.0, 1.0)
    for i in range(3):
        arr = x[i].mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()
        got = np.asarray(Image.open(tmp_path / "imgs" / f"{3 + i}.png"))
        assert np.array_equal(got, arr), i
    # (3) the moments of the same bytes against fid.py over the files
    mu_f, sigma_f = fid.calculate_activation_statistics(sorted(str(p) for p in (tmp_path / "imgs").glob("*.png")), inc, batch_size=3,
                                                        dims=64)
    assert np.allclose(mu, mu_f, rtol=1e-6, atol=1e-9) and np.allclose(sigma, sigma_f, rtol=1e-5, atol=1e-9)
    # img_id continues from the files already there
    _, _, n2 = de.sample_fid(m, _cfg(3), str(tmp_path / "imgs"), total=9, timesteps=2, seed=5)
    assert n2 == 3 and os.path.exists(tmp_path / "imgs" / "8.png")


# ---------------------------------------------------------------------------------------------------------------------- census, audit
def _census_run(m):
    x = torch.randn(64, 3, 32, 32, generator=torch.Generator().manual_seed(4)).cuda()
    return lambda: _sample(m, x, eta=0.5, use_graph=False, steps=2)


def test_cifar10_sampling_census(lib):
    """Every distinct launch of two eager eta-0.5 steps of the CIFAR-10 sampling plan at batch 64, replayed on fresh seeded buffers and
    checked against float64 (bounds of launch_census.py) or bit for bit."""
    from test_eval_census_gpu import EVAL_REPLAY, _LOG
    from test_launch_census_gpu import _capture, _unique
    from test_ldm_sampling_gpu import replay_ddim_cfg_step
    _LOG.clear()
    _LOG.update(geoms=set(), tc=[], simt=set())
    replay = dict(EVAL_REPLAY, dp_ddim_cfg_step=replay_ddim_cfg_step)
    m = _cifar().cuda()
    calls = _capture(lib, _census_run(m))
    kinds = {n for n, _ in calls}
    assert {"dp_conv2d_fprop", "dp_groupnorm_fwd", "dp_ddim_cfg_step", "dp_timestep_embedding"} <= kinds
    missing = kinds - set(replay)
    assert not missing, f"launch kinds without a replay: {sorted(missing)}"
    rep, failures = {}, []
    g = torch.Generator().manual_seed(2031)
    uniq = _unique(calls)
    for name, args in uniq:
        try:
            replay[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print("  FAIL", f)
    assert not failures
    print(f"\nddpm_exp CIFAR-10 census: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds")
    for name in sorted(rep):
        print(f"  {name:26s} worst err/bound {max(rep[name]):.3f}")


def test_cifar10_amax_slots_bound_their_operands(lib):
    import launch_census as lc
    import slot_audit as sa
    from test_slot_audit_gpu import MAX_LOOSENESS
    m = _cifar().cuda()
    run = _census_run(m)
    audit = sa.SlotAudit()
    with lc.wrap_launches(lib, audit):
        run()
        torch.cuda.synchronize()
    worst, where = audit.worst()
    print(f"\nddpm_exp CIFAR-10: {audit.launches} launches name an input slot, {audit.audited} audited ({audit.simt} SIMT), "
          f"{len(audit.failures)} below the maximum; worst looseness {worst:.4g} at {where}")
    assert not audit.failures, audit.failures[:3]
    assert audit.audited > 0 and audit.audited + audit.simt == audit.launches
    assert worst <= MAX_LOOSENESS
