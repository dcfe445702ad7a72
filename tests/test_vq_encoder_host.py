"""Host checks of the encode side of the LDM's VQ first stage (autoencoder.py) against tests/golden/vq_encoder_tiny.pt, which the
unmodified reference Encoder and VQModelInterface.encode produced (tools/gen_golden.py vq_encoder): state-dict names and seeded weights,
the float32 oracle and the traced modules against the reference outputs, the Lightning-checkpoint load with and without the encoder, the
options that are rejected, and the encoder plan's launch list at two image sizes."""
import pytest
import torch

from conftest import load_golden, max_rel
import vq_encoder_oracle as eo
from oracle import vq_oracle as vo

GOLD = load_golden("vq_encoder_tiny.pt")
CONFIGS = list(GOLD["configs"])


def seeded_encoder(name):
    from diff_pruning_b200.autoencoder import Encoder
    c = GOLD["configs"][name]
    torch.manual_seed(c["seed"])
    return Encoder(**c["ddconfig"]).eval()


def seeded_vq(name):
    """torch.manual_seed(seed); VQModelInterface(with_encoder=True): the reference VQModelInterface's parameters (fixture digest)."""
    from diff_pruning_b200.autoencoder import VQModelInterface
    c = GOLD["configs"][name]
    torch.manual_seed(c["seed"])
    return VQModelInterface(embed_dim=c["ddconfig"]["z_channels"], n_embed=c["n_embed"], ddconfig=c["ddconfig"], with_encoder=True).eval()


@pytest.mark.parametrize("name", CONFIGS)
def test_encoder_state_dict_names_and_seeded_weights_match_the_reference(name):
    c = GOLD["configs"][name]
    sd = seeded_encoder(name).state_dict()
    assert list(sd.keys()) == c["sd_keys"]
    assert vo.state_dict_digest(sd) == c["digest"]


@pytest.mark.parametrize("name", CONFIGS)
def test_vq_model_with_encoder_draws_the_reference_parameters_in_its_order(name):
    c = GOLD["configs"][name]
    sd = seeded_vq(name).state_dict()
    assert list(sd.keys()) == c["vq_sd_keys"]
    assert vo.state_dict_digest(sd) == c["vq_digest"]


@pytest.mark.parametrize("name", CONFIGS)
def test_float32_oracle_matches_reference_encoder_and_encode(name):
    c = GOLD["configs"][name]
    assert max_rel(eo.encoder(seeded_encoder(name).state_dict(), c["ddconfig"], c["x"]), c["out"]) < 1e-5
    assert max_rel(eo.encode(seeded_vq(name).state_dict(), c["ddconfig"], c["x"]), c["encoded"]) < 1e-5


@pytest.mark.parametrize("name", CONFIGS)
def test_traced_encode_is_the_reference(name):
    import diff_pruning_b200 as dp
    c = GOLD["configs"][name]
    with dp.trace_mode(), torch.no_grad():
        got = seeded_vq(name).encode(c["x"])
    assert max_rel(got, c["encoded"]) < 1e-5


def _ld(with_encoder, first_stage=True):
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    fsc = dict(embed_dim=3, n_embed=64, ddconfig=GOLD["configs"]["tiny"]["ddconfig"], with_encoder=with_encoder)
    return LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16), first_stage_config=fsc if first_stage else None)


def test_lightning_checkpoint_loads_the_encoder_and_quant_conv():
    src = _ld(True)
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(v.shape, generator=g) if v.is_floating_point() else v for k, v in src.state_dict().items()}
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev"):
        sd[k] = src.state_dict()[k].clone()
    assert any(k.startswith("first_stage_model.encoder.") for k in sd) and "first_stage_model.quant_conv.weight" in sd
    ckpt = dict(sd, **{"first_stage_model.loss.logvar": torch.zeros(()), "model_ema.num_updates": torch.tensor(7)})
    dst = _ld(True)
    res = dst.load_state_dict(ckpt)
    assert not res.missing_keys and not res.unexpected_keys
    got = dst.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    # without the encoder the same checkpoint loads the decode side only, as before
    dec_only = _ld(False)
    res = dec_only.load_state_dict(ckpt)
    assert not res.missing_keys and not res.unexpected_keys
    assert not any(k.startswith(("first_stage_model.encoder.", "first_stage_model.quant_conv.")) for k in dec_only.state_dict())
    # an encoder key missing from the checkpoint is an error when the encoder is built
    del ckpt["first_stage_model.quant_conv.bias"]
    with pytest.raises(RuntimeError):
        _ld(True).load_state_dict(ckpt)


def test_unsupported_options_raise():
    from diff_pruning_b200.autoencoder import Downsample, Encoder, VQModelInterface
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    dd = dict(GOLD["configs"]["tiny"]["ddconfig"])
    for bad in (dict(resamp_with_conv=False), dict(use_linear_attn=True), dict(attn_type="linear"), dict(double_z=True)):
        with pytest.raises(NotImplementedError):
            Encoder(**dict(dd, **bad))
    with pytest.raises(NotImplementedError):
        Downsample(8, with_conv=False)
    with pytest.raises(NotImplementedError):                       # the reference Encoder's default is double_z=True
        Encoder(**{k: v for k, v in dd.items() if k != "double_z"})
    with pytest.raises(NotImplementedError):
        VQModelInterface(embed_dim=3, n_embed=64, ddconfig=dd).encode(torch.zeros(1, 3, 16, 16))
    m = VQModelInterface(embed_dim=3, n_embed=64, ddconfig=dd, with_encoder=True)
    with pytest.raises(RuntimeError):
        m.encode(torch.zeros(1, 3, 16, 16))                        # no CPU fallback
    ld = _ld(True)
    ld.split_input_params = {"patch_distributed_vq": True}
    with pytest.raises(NotImplementedError):
        ld.encode_first_stage(torch.zeros(1, 3, 16, 16))
    with pytest.raises(RuntimeError):
        _ld(False, first_stage=False).encode_first_stage(torch.zeros(1, 3, 16, 16))
    with pytest.raises(NotImplementedError):
        _ld(False).encode_first_stage(torch.zeros(1, 3, 16, 16))
    with pytest.raises(ValueError):
        LDMPruneScorer(_ld(False), encode_samples=True)
    with pytest.raises(NotImplementedError):
        ld.get_first_stage_encoding([torch.zeros(1)])


def test_get_first_stage_encoding_is_scale_factor_times_z():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    ld = LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16), scale_factor=0.18215)
    z = torch.randn(2, 3, 4, 4, generator=torch.Generator().manual_seed(1))
    assert torch.equal(ld.get_first_stage_encoding(z), 0.18215 * z)


def _launches(m, hw):
    from diff_pruning_b200.autoencoder import _EncodePath
    from diff_pruning_b200.engine import Plan
    from diff_pruning_b200 import _lib as L
    p = Plan(_EncodePath(m.encoder, m.quant_conv), 2, hw, hw, "cpu", need_grad=False)
    convs = [a for a in p._keep if isinstance(a, L.ConvArgs)]
    return p, [(f.what, f.info.split(" @")[0]) for f in p.fwd], convs


def test_encoder_plan_launch_list_is_the_same_at_two_image_sizes():
    """VQ-f4's forward-only encoder plan at 32 x 32 and 64 x 64 images: the same launches in the same order, only the grids differ;
    27 convolutions, 18 GroupNorms and the three launches of the mid attention (host planning: SIMT, no tensor-core amax launches), the
    two Downsample convolutions as stride 2 with pad_t = pad_l = 0 onto the half grid, and no backward."""
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    torch.manual_seed(0)
    m = VQModelInterface(**VQ_F4_CONFIG, with_encoder=True).eval()
    runs = {hw: _launches(m, hw) for hw in (32, 64)}
    (p32, l32, c32), (p64, l64, c64) = runs[32], runs[64]
    assert l32 == l64
    kinds = [w for w, _ in l64]
    assert (kinds.count("conv fprop"), kinds.count("gn fwd"), len(kinds)) == (27, 18, 48)
    assert [w for w in kinds if w not in ("conv fprop", "gn fwd")] == ["attn qk", "softmax", "attn pv"]
    for hw, convs in ((32, c32), (64, c64)):
        down = [a for a in convs if a.stride == 2]
        assert [(a.H, a.C, a.P, a.pad_t, a.pad_l, a.R) for a in down] == [(hw, 128, hw // 2, 0, 0, 3), (hw // 2, 256, hw // 4, 0, 0, 3)]
    assert tuple(p64.y_out.t.shape) == (2, 16, 16, 4) and p64.y_out.C == 3 and not p64.bwd
