"""test_criterion.py's sample-encode-score loop (LDMPruneScorer(encode_samples=True)) on one H100:

1. three taylor iterations on the tiny LDM (with the small VQ encoder) are bit-identical to the module-path composition
   DDIMSampler.sample -> encode_first_stage -> get_loss_at_t -> loss.backward();
2. the loop stops where a host restatement of test_criterion.py's rule over its own losses stops, for diff-pruning, diff0 and taylor;
3. two iterations of cin256-v2 at full width with the VQ-f4 encoder (batch 2, 3 x 64 x 64 samples encoded to 3 x 16 x 16) against the
   float64 oracle (vq_encoder_oracle.encode, ldm_sampling_oracle.get_loss_at_t) for the encoded latents, the losses and the accumulated gradients.
"""
import numpy as np
import pytest
import torch

from conftest import max_rel, worst_grad_err
import vq_encoder_oracle as eo
from test_launch_census_gpu import lib  # noqa: F401  (the module-scoped fixture)
from test_ldm_sampling_gpu import _labels_seq, _tiny_ld
from test_vq_encoder_host import GOLD as EGOLD

pytestmark = pytest.mark.gpu


def _with_encoder(ld, fs_config, seed=0):
    """ld with a seeded first stage that holds its encoder."""
    from diff_pruning_b200.autoencoder import VQModelInterface
    torch.manual_seed(seed)
    ld.first_stage_model = VQModelInterface(**fs_config, with_encoder=True).eval().cuda()
    return ld


def _tiny():
    return _with_encoder(_tiny_ld(), dict(embed_dim=3, n_embed=64, ddconfig=EGOLD["configs"]["tiny"]["ddconfig"]))


def _labels_cycle(B):
    """Labels for loops longer than _labels_seq's four iterations: iteration j draws (17 j + 101 i) mod 1000 for image i."""
    k = iter(range(1 << 30))
    return lambda n: [(17 * next(k) + 101 * i) % 1000 for i in range(n)]


def _loop(ld, B, iters, pruner="taylor", S_=4):
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    unet = ld.model.diffusion_model
    unet.zero_grad()
    sc = LDMPruneScorer(ld, n_samples_per_class=B, ddim_steps=S_, scale=3.0, encode_samples=True)
    sampler = _labels_seq(B) if iters <= 4 else _labels_cycle(B)
    losses = sc.run(pruner, iterations=iters, class_sampler=sampler, generator=torch.Generator().manual_seed(31))
    torch.cuda.synchronize()
    return sc, losses, {k: p.grad.clone() for k, p in unet.named_parameters()}


def test_criterion_loop_equals_module_path(lib):
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    B = 2
    ld = _tiny()
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
        encoded = ld.encode_first_stage(s)
        assert tuple(encoded.shape) == (B, 3, 8, 8)
        noise = torch.randn(encoded.shape, generator=g).cuda()
        loss, _ = ld.get_loss_at_t(encoded, {"class_label": xc}, torch.full((B,), t, device="cuda", dtype=torch.long), noise=noise)
        losses.append(float(loss))
        loss.backward()
    assert np.allclose(losses, fast_losses.tolist(), rtol=1e-6)
    bad = [k for k, p in unet.named_parameters() if not torch.equal(p.grad, fast[k])]
    assert not bad, bad[:8]


def _host_rule(losses, pruner):
    """test_criterion.py:127-133 on fp32 scalars: max_loss from -1, updated first; diff-pruning 0.1 / diff0 0.0 stop when
    loss / max_loss < thres, before the backward; taylor never stops.  Returns the stopping index or None."""
    max_loss = np.float32(-1)
    thres = np.float32(0.1 if pruner == "diff-pruning" else 0.0)
    for i, l in enumerate(losses):
        l = np.float32(l)
        if l > max_loss:
            max_loss = l
        if pruner in ("diff-pruning", "diff0") and np.float32(l / max_loss) < thres:
            return i
    return None


@pytest.mark.parametrize("pruner", ["diff-pruning", "diff0", "taylor"])
def test_criterion_loop_stops_where_the_host_rule_stops(lib, pruner):
    """Eight iterations over t = 0..7, then again with the first loss the rule sees scaled up tenfold (a large first loss, as at small t
    on a trained model), so that the diff-pruning threshold can be reached: the loop stops where the host restatement stops on the same
    losses, or runs to the end where it does not."""
    from diff_pruning_b200 import ldm_sampling
    ld = _tiny()
    iters = 8
    sc, losses, _ = _loop(ld, 2, iters, pruner, S_=4)
    want = _host_rule(losses.tolist(), pruner)
    assert sc.stopped_at == want and len(losses) == (iters if want is None else want + 1)
    seen = []
    orig = ldm_sampling.PruneLDMStopRule.stop

    def boosted(self, loss):
        seen.append(loss * 10 if not seen else loss)
        return orig(self, seen[-1])
    ldm_sampling.PruneLDMStopRule.stop = boosted
    try:
        sc2, _, _ = _loop(ld, 2, iters, pruner, S_=4)
    finally:
        ldm_sampling.PruneLDMStopRule.stop = orig
    want2 = _host_rule(seen, pruner)
    print(f"{pruner}: losses {[f'{l:.4g}' for l in losses.tolist()]}; stops at {sc.stopped_at}, with a boosted first loss at {sc2.stopped_at}")
    assert sc2.stopped_at == want2 and len(seen) == (iters if want2 is None else want2 + 1)


def test_cin256_two_iterations_match_float64_oracle(lib):
    """cin256-v2 at full width, batch 2, DDIM-4 at scale 3, with the VQ-f4 encoder: the samples each iteration encodes are recorded, and
    the fp64 oracle encodes them, forms get_loss_at_t at t = iteration with the same noise and accumulates the gradients of both."""
    import launch_census as lc
    import ldm_sampling_oracle as orc
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    m, cfg = lc.c5_model()
    ld = LatentDiffusion()
    ld.model.diffusion_model.load_state_dict(m.state_dict())
    torch.manual_seed(1)
    ld.cond_stage_model.embedding.weight.data.normal_()
    ld = _with_encoder(ld.cuda(), VQ_F4_CONFIG, seed=2)
    recorded = []
    enc = ld.encode_first_stage

    def recording(x):
        z = enc(x)
        recorded.append((x.clone(), z.clone()))
        return z
    ld.encode_first_stage = recording
    B, iters = 2, 2
    _, losses, grads = _loop(ld, B, iters, "taylor")
    del ld.encode_first_stage
    assert len(recorded) == iters and tuple(recorded[0][1].shape) == (B, 3, 16, 16)
    # the generator's draws per iteration: x_T (B, 3, 64, 64), then the loss noise (B, 3, 16, 16) (eta 0: no step noise)
    g = torch.Generator().manual_seed(31)
    labels = _labels_seq(B)
    unet = ld.model.diffusion_model
    sd = {k: v.detach().double().clone().requires_grad_(True) for k, v in unet.state_dict().items()}
    fs64 = {k: v.detach().double() for k, v in ld.first_stage_model.state_dict().items()}
    worst_z, ref_losses = 0.0, []
    for t, (x, z) in enumerate(recorded):
        torch.randn(B, 3, 64, 64, generator=g)
        noise = torch.randn(B, 3, 16, 16, generator=g).cuda()
        with torch.no_grad():
            z64 = eo.encode(fs64, VQ_F4_CONFIG["ddconfig"], x.double())
            c = ld.get_learned_conditioning({"class_label": torch.tensor(labels(B)).cuda()})
        worst_z = max(worst_z, max_rel(z, z64))
        ref_losses.append(float(orc.get_loss_at_t(sd, cfg, ld.alphas_cumprod, z64, c.double(), torch.full((B,), t, device="cuda"),
                                                  noise.double())))
    err = worst_grad_err(((k, grads[k]) for k, _ in unet.named_parameters()), {k: v.grad for k, v in sd.items()})
    print(f"\ncin256-v2 + VQ-f4 encoder, 2 iterations: encoded max-rel {worst_z:.2e}; losses {losses.tolist()} (fp64 {ref_losses}); "
          f"worst gradient {err:.2e}")
    assert worst_z < 1e-4
    assert np.allclose(losses.tolist(), ref_losses, rtol=1e-5)
    assert err < 1e-4
