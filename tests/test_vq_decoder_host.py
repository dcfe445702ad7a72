"""Host checks of the LDM's VQ first stage (autoencoder.py) against tests/golden/vq_decoder_tiny.pt, which the unmodified reference
Decoder produced (tools/gen_golden.py vq_decoder): state-dict names and seeded weights, the Lightning-checkpoint load with and without a
first stage, the float32 oracle against the reference outputs, the save_image byte rule against torchvision's, and the argument checks
of dp_vq_quantize / dp_decode_images."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden, max_rel
from oracle import vq_oracle as vo

GOLD = load_golden("vq_decoder_tiny.pt")
CONFIGS = list(GOLD["configs"])


def seeded_decoder(name):
    from diff_pruning_b200.autoencoder import Decoder
    c = GOLD["configs"][name]
    torch.manual_seed(c["seed"])
    return Decoder(**c["ddconfig"]).eval()


def vq_model(name, n_embed=8192, seed=0):
    """A VQModelInterface around the fixture's seeded decoder: post_quant_conv and the codebook drawn from `seed` afterwards."""
    from diff_pruning_b200.autoencoder import VQModelInterface
    c = GOLD["configs"][name]
    torch.manual_seed(seed)
    m = VQModelInterface(embed_dim=c["ddconfig"]["z_channels"], n_embed=n_embed, ddconfig=c["ddconfig"]).eval()
    m.decoder.load_state_dict(seeded_decoder(name).state_dict())
    return m


@pytest.mark.parametrize("name", CONFIGS)
def test_decoder_state_dict_names_and_seeded_weights_match_the_reference(name):
    dec = seeded_decoder(name)
    sd = dec.state_dict()
    assert list(sd.keys()) == GOLD["configs"][name]["sd_keys"]
    assert vo.state_dict_digest(sd) == GOLD["configs"][name]["digest"]       # same construction order: same parameters from a seed


def test_vq_f4_config_is_cin256_v2s_first_stage():
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    m = VQModelInterface(**VQ_F4_CONFIG)
    assert [k for k in m.state_dict() if not k.startswith("decoder.")] == ["quantize.embedding.weight", "post_quant_conv.weight",
                                                                            "post_quant_conv.bias"]
    assert tuple(m.quantize.embedding.weight.shape) == (8192, 3)
    assert round(sum(p.numel() for p in m.decoder.parameters()) / 1e6, 1) == 33.0
    assert float(m.quantize.embedding.weight.detach().abs().max()) <= 1 / 8192


@pytest.mark.parametrize("name", CONFIGS)
def test_float32_oracle_matches_reference_decoder(name):
    c = GOLD["configs"][name]
    got = vo.decoder(seeded_decoder(name).state_dict(), c["ddconfig"], c["z"])
    assert max_rel(got, c["out"]) < 1e-5


def test_traced_decode_is_the_oracle():
    """autoencoder.VQModelInterface.decode under trace_mode (torch ops) and oracle.vq_oracle.decode: the same choice of codes and output."""
    import diff_pruning_b200 as dp
    m = vq_model("tiny", n_embed=64)
    g = torch.Generator().manual_seed(4)
    h = torch.randn(2, 3, 8, 8, generator=g) * 0.02
    sd = m.state_dict()
    with dp.trace_mode(), torch.no_grad():
        got = m.decode(h)
        got_fnq = m.decode(h, force_not_quantize=True)
    assert max_rel(got, vo.decode(sd, GOLD["configs"]["tiny"]["ddconfig"], h)) < 1e-6
    assert max_rel(got_fnq, vo.decode(sd, GOLD["configs"]["tiny"]["ddconfig"], h, force_not_quantize=True)) < 1e-6


def test_recalled_taming_and_cdist_choices_agree_with_the_fp64_contract_up_to_near_ties():
    """The fixture's nearest codes of both reference formulas against the fp64 contract on the same latent: they may differ from it
    only where the two nearest distances are closer than the fp32 rounding of the formula."""
    cd = GOLD["codes"]
    g = torch.Generator().manual_seed(cd["codebook_seed"])
    code = (torch.rand(8192, 3, generator=g) * 2 - 1) / 8192 * 64
    z = torch.randn(4096, 3, generator=g) * 0.004
    assert torch.equal(z, cd["z"])
    exact = vo.nearest_code(z, code)
    d = ((z.double()[:, None] - code.double()[None]) ** 2).sum(-1)
    for formula in ("cdist", "taming"):
        other = cd[formula]
        diff = (other != exact).nonzero().flatten()
        gap = (d[diff, other[diff]] - d[diff, exact[diff]]).abs()
        # |z|^2 + |e|^2 - 2 z.e in fp32 rounds at 2^-24 of the squared norms; cdist's sqrt of a similar sum does no better
        tol = 8 * 2.0 ** -24 * ((z.double()[diff] ** 2).sum(1) + (code.double()[other[diff]] ** 2).sum(1))
        assert bool((gap <= tol).all()), (formula, int(diff.numel()))
        print(f"{formula}: {int(diff.numel())} of {z.shape[0]} pixels choose another code than the fp64 contract, all near ties")


def test_lightning_checkpoint_loads_first_stage_decoder_when_configured():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    fsc = dict(embed_dim=3, n_embed=64, ddconfig=GOLD["configs"]["tiny"]["ddconfig"])

    def make(first_stage):
        return LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16),
                               first_stage_config=fsc if first_stage else None)
    src = make(True)
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(v.shape, generator=g) if v.is_floating_point() else v for k, v in src.state_dict().items()}
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev"):
        sd[k] = src.state_dict()[k].clone()
    ckpt = dict(sd)
    ckpt.update({"first_stage_model.encoder.conv_in.weight": torch.randn(64, 3, 3, 3), "first_stage_model.quant_conv.weight":
                 torch.randn(3, 3, 1, 1), "first_stage_model.loss.logvar": torch.zeros(()), "model_ema.num_updates": torch.tensor(7)})
    dst = make(True)
    res = dst.load_state_dict(ckpt)
    assert not res.missing_keys and not res.unexpected_keys
    got = dst.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert any(k.startswith("first_stage_model.decoder.") for k in got)
    # without first_stage_config the same checkpoint loads the UNet / embedder only, as before
    plain = make(False)
    res = plain.load_state_dict(ckpt)
    assert not res.missing_keys and not res.unexpected_keys
    assert not any(k.startswith("first_stage_model.") for k in plain.state_dict())
    del ckpt["first_stage_model.decoder.conv_out.weight"]
    with pytest.raises(RuntimeError):
        make(True).load_state_dict(ckpt)
    with make(True).ema_scope() as s:
        assert s is None


def test_decode_first_stage_rejects_what_is_not_built():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.autoencoder import Decoder, VQModelInterface
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    m = LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16))
    with pytest.raises(RuntimeError):
        m.decode_first_stage(torch.zeros(1, 3, 8, 8))
    with pytest.raises(NotImplementedError):
        m.decode_first_stage(torch.zeros(1, 3, 8, 8), predict_cids=True)
    dd = dict(GOLD["configs"]["tiny"]["ddconfig"])
    for bad in (dict(tanh_out=True), dict(give_pre_end=True), dict(attn_type="linear"), dict(use_linear_attn=True)):
        with pytest.raises(NotImplementedError):
            Decoder(**dd, **bad)
    with pytest.raises(NotImplementedError):
        VQModelInterface(embed_dim=3, n_embed=64, ddconfig=dd).encode(torch.zeros(1, 3, 16, 16))


# ---------------------------------------------------------------------------------------------------------------------- save_image rule
def device_rule_bytes(x: np.ndarray) -> np.ndarray:
    """image_src.cuh's rule restated in numpy float32 (every operation rounds once): v = clamp((x + 1) / 2, 0, 1), byte =
    trunc(clamp(v * 255 + 0.5, 0, 255))."""
    f = np.float32
    v = np.minimum(np.maximum((x.astype(f) + f(1)) / f(2), f(0)), f(1))
    return np.minimum(np.maximum(v * f(255) + f(0.5), f(0)), f(255)).astype(np.uint8)


def boundary_values() -> np.ndarray:
    """Every decoded value x whose v = (x + 1) / 2 puts v * 255 + 0.5 on, or within a few ulps of, an integer; plus the clamps."""
    f = np.float32
    out = []
    for k in range(0, 257):
        v0 = f((k - 0.5) / 255.0)
        for v in (v0, *[v0 + s * np.spacing(v0) * i for s in (-1, 1) for i in (1, 2, 3)]):
            x0 = f(2) * f(v) - f(1)
            out += [x0 + s * np.spacing(x0) * i for s in (-1, 1) for i in range(4)] + [x0]
    out += [-3.0, -1.0, -0.9999999, 1.0, 1.0000001, 2.5, 0.0]
    return np.asarray(out, dtype=np.float32)


def torchvision_bytes(x: np.ndarray, tmp_path) -> np.ndarray:
    """sample_for_FID.py's chain on the host: clamp((x + 1) / 2, 0, 1) -> tvu.save_image -> PIL -> bytes."""
    from PIL import Image
    from torchvision import utils as tvu
    n = x.size
    img = torch.from_numpy(x).reshape(1, 1, n).expand(3, 1, n).contiguous()
    img = torch.clamp((img + 1.0) / 2.0, min=0.0, max=1.0)
    p = tmp_path / "rule.png"
    tvu.save_image(img, str(p))
    return np.asarray(Image.open(p).convert("RGB"))[0, :, 0]


def test_save_image_rule_matches_torchvision_at_every_rounding_boundary(tmp_path):
    x = boundary_values()
    want = torchvision_bytes(x, tmp_path)
    got = device_rule_bytes(x)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]
    # the rule rounds half up: it differs from the DDPM sampler's rint rule (round half to even) on some of these values
    v = np.minimum(np.maximum((x + np.float32(1)) / np.float32(2), 0), 1).astype(np.float32)
    assert (np.rint(v * np.float32(255)).astype(np.uint8) != got).any()


# ---------------------------------------------------------------------------------------------------------------------- C-ABI
def test_capi_argument_checks():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    p = ctypes.c_void_p(64)          # never dereferenced: argument checks return before any launch
    ok = dict(z=p, N=1, D=3, H=4, W=4, s=1.0, e=p, n=8, q=1, out=p, ld=4, idx=None)

    def vq(**kw):
        a = dict(ok, **kw)
        return lib.dp_vq_quantize(a["z"], a["N"], a["D"], a["H"], a["W"], a["s"], a["e"], a["n"], a["q"], a["out"], a["ld"], a["idx"], None)
    assert vq(z=None) == -5 and vq(out=None) == -5 and vq(e=None) == -5
    assert vq(N=0) == -1 and vq(H=0) == -1 and vq(D=0) == -1 and vq(ld=2) == -1 and vq(n=0) == -1
    assert vq(D=9, ld=12) == -3

    def di(**kw):
        a = dict(dict(y=p, ld=4, N=1, C=3, H=4, W=4, u8=p, f32=None), **kw)
        return lib.dp_decode_images(a["y"], a["ld"], a["N"], a["C"], a["H"], a["W"], a["u8"], a["f32"], None)
    assert di(y=None) == -5 and di(u8=None, f32=None) == -5
    assert di(N=0) == -1 and di(C=0) == -1 and di(ld=2) == -1 and di(H=0) == -1
