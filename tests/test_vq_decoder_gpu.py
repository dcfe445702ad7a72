"""The LDM's VQ first stage on the device: dp_vq_quantize against the fp64 nearest-code contract, dp_decode_images against torchvision's
save_image, the decoder plan against the reference Decoder (tests/golden/vq_decoder_tiny.pt) and the float64 oracle at 256 x 256, the
launch census of every distinct decoder launch, NaN-poisoned plans, graph against eager, micro-batch chunking, and sample_for_fid end to
end on the tiny LDM."""
import gc
import os

import numpy as np
import pytest
import torch

from conftest import max_rel
from oracle import vq_oracle as vo
from test_vq_decoder_host import GOLD, seeded_decoder, vq_model

pytestmark = pytest.mark.gpu


def S():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    return L.load()


def _quantize(lib, z, code, quantize=True, inv_scale=1.0, ld=4):
    N, D, H, W = z.shape
    out = torch.full((N * H * W, ld), -777.0, device="cuda")
    idx = torch.full((N, H, W), -1, dtype=torch.int64, device="cuda")
    assert lib.dp_vq_quantize(z.data_ptr(), N, D, H, W, inv_scale, code.data_ptr(), code.shape[0], int(quantize), out.data_ptr(), ld,
                              idx.data_ptr() if quantize else None, S()) == 0
    torch.cuda.synchronize()
    assert bool((out[:, D:] == -777.0).all()), "a pad channel was written"
    return out[:, :D].cpu(), idx.cpu()


def _contract(z, code):
    """numpy float64: ((z0 - e0)^2 + (z1 - e1)^2) + (z2 - e2)^2, first minimum."""
    zf = z.permute(0, 2, 3, 1).reshape(-1, z.shape[1]).double().numpy()
    e = code.double().numpy()
    d = np.zeros((zf.shape[0], e.shape[0]))
    for c in range(zf.shape[1]):
        d = d + (zf[:, c:c + 1] - e[None, :, c]) ** 2
    return torch.from_numpy(d.argmin(1)), d


def _codebook(g, n=8192, D=3):
    return ((torch.rand(n, D, generator=g) * 2 - 1) / n * 64)


@pytest.mark.parametrize("case", ["seeded", "halfway", "duplicated"])
def test_vq_quantize_matches_fp64_contract_and_straight_through_rounding(lib, case):
    g = torch.Generator().manual_seed({"seeded": 1, "halfway": 2, "duplicated": 3}[case])
    code = _codebook(g)
    z = torch.randn(2, 3, 24, 40, generator=g) * 0.004
    if case == "halfway":        # a pixel exactly between two codes: e_a = z - d, e_b = z + d with d a power of two
        zf = z.permute(0, 2, 3, 1).reshape(-1, 3)
        for i in range(0, zf.shape[0], 7):
            a, b = sorted(torch.randint(0, 8192, (2,), generator=g).tolist())
            if a == b:
                continue
            d = torch.tensor([2.0 ** -12, -2.0 ** -13, 2.0 ** -11])
            code[a], code[b] = zf[i] - d, zf[i] + d
        z = zf.reshape(2, 24, 40, 3).permute(0, 3, 1, 2).contiguous()
    if case == "duplicated":     # repeated rows: the first copy wins
        for j in range(0, 4096, 3):
            code[8191 - j] = code[j].clone()
    want, d = _contract(z, code)
    got_out, got_idx = _quantize(lib, z.cuda(), code.cuda())
    assert torch.equal(got_idx.reshape(-1), want)
    zf = z.permute(0, 2, 3, 1).reshape(-1, 3)
    assert torch.equal(got_out, zf + (code[want] - zf))              # z + (e - z) in fp32, not e
    n_not_e = int((got_out != code[want]).any(1).sum())
    # the two formulas of the reference (recalled taming / in-tree cdist) on the same pixels
    for name, fn in (("taming", vo.nearest_code_taming), ("cdist", vo.nearest_code_cdist)):
        other = fn(zf, code)
        diff = (other != want).nonzero().flatten()
        gap = np.abs(d[diff.numpy(), other[diff].numpy()] - d[diff.numpy(), want[diff].numpy()])
        tol = 8 * 2.0 ** -24 * ((zf.double()[diff] ** 2).sum(1) + (code.double()[other[diff]] ** 2).sum(1)).numpy()
        assert (gap <= tol).all(), (name, case)
        print(f"{case}: {name} picks another code at {int(diff.numel())} of {zf.shape[0]} pixels, every one a near tie; "
              f"z + (e - z) != e at {n_not_e}")


def test_vq_quantize_force_not_quantize_and_scale(lib):
    g = torch.Generator().manual_seed(5)
    z = torch.randn(3, 3, 8, 8, generator=g)
    code = _codebook(g, 64)
    out, _ = _quantize(lib, z.cuda(), code.cuda(), quantize=False, inv_scale=0.18215)
    assert torch.equal(out, (z * torch.tensor(0.18215)).permute(0, 2, 3, 1).reshape(-1, 3))
    out, idx = _quantize(lib, z.cuda(), code.cuda(), inv_scale=0.5)
    want, _ = _contract(z * 0.5, code)
    assert torch.equal(idx.reshape(-1), want)


def test_decode_images_bytes_equal_save_image_and_fp32_the_clamp(lib, tmp_path):
    from PIL import Image
    from torchvision import utils as tvu
    from test_vq_decoder_host import boundary_values
    g = torch.Generator().manual_seed(6)
    N, H, W = 2, 48, 72
    x = torch.randn(N, H, W, 3, generator=g) * 0.8
    b = torch.from_numpy(boundary_values())
    x.view(-1)[:b.numel()] = b
    y = torch.full((N * H * W, 4), 9.0, device="cuda")
    y[:, :3] = x.reshape(-1, 3).cuda()
    u8 = torch.zeros(N, H, W, 3, dtype=torch.uint8, device="cuda")
    f = torch.zeros(N, 3, H, W, device="cuda")
    assert lib.dp_decode_images(y.data_ptr(), 4, N, 3, H, W, u8.data_ptr(), f.data_ptr(), S()) == 0
    torch.cuda.synchronize()
    xc = torch.clamp((x.permute(0, 3, 1, 2) + 1.0) / 2.0, min=0.0, max=1.0)
    assert torch.equal(f.cpu(), xc)
    for i in range(N):
        p = tmp_path / f"{i}.png"
        tvu.save_image(xc[i], str(p))
        assert np.array_equal(np.asarray(Image.open(p)), u8[i].cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------- decoder plan
def _identity_front(m):
    """post_quant_conv = identity, so decode(force_not_quantize=True) is the Decoder alone (x + 0 + 0 is exact)."""
    with torch.no_grad():
        m.post_quant_conv.weight.copy_(torch.eye(3).reshape(3, 3, 1, 1))
        m.post_quant_conv.bias.zero_()
    return m


@pytest.mark.parametrize("name", list(GOLD["configs"]))
def test_decoder_plan_matches_reference_decoder(name):
    c = GOLD["configs"][name]
    m = _identity_front(vq_model(name)).cuda()
    got = m.decode(c["z"].cuda(), force_not_quantize=True)
    err = max_rel(got, c["out"])
    print(f"{name}: max-rel {err:.2e} against the reference Decoder")
    assert err < 1e-4


def _vq_f4(seed=3):
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    torch.manual_seed(seed)
    return VQModelInterface(**VQ_F4_CONFIG).eval()


def test_vq_f4_256px_decode_matches_float64_oracle():
    """VQ-f4 at a 64 x 64 latent (256 x 256 images, 4096 attention tokens) at batch 2, quantised, against the float64 oracle."""
    m = _vq_f4()
    g = torch.Generator().manual_seed(8)
    h = torch.randn(2, 3, 64, 64, generator=g) * 2e-4
    sd64 = {k: v.detach().double().cuda() for k, v in m.state_dict().items()}
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    want = vo.decode(sd64, VQ_F4_CONFIG["ddconfig"], h.double().cuda())
    m = m.cuda()
    m.decode_batch = 2
    got = m.decode(h.cuda())
    err = max_rel(got, want)
    plan = m.__dict__["_dpb200_decode"].plan
    print(f"VQ-f4 256px b2: max-rel {err:.2e} against fp64; plan bytes at micro-batch 2: {plan.bytes_allocated() / 2 ** 30:.2f} GiB")
    assert tuple(got.shape) == (2, 3, 256, 256) and err < 1e-4


def test_decode_in_chunks_and_graph_equal_separate_and_eager():
    """13 latents at micro-batch 8 = the first 8 and the last 5 decoded on their own (the tail chunk is zero-padded); the graph run
    equals the eager launch list."""
    m = _vq_f4().cuda()
    g = torch.Generator().manual_seed(9)
    h = (torch.randn(13, 3, 16, 16, generator=g) * 2e-4).cuda()
    all13 = m.decode(h)
    parts = torch.cat([m.decode(h[:8]), m.decode(h[8:])])
    assert torch.equal(all13, parts)
    m.use_graph = False
    eager = m.decode(h)
    assert torch.equal(all13, eager)


def test_decoder_plan_is_bit_identical_under_poisoned_allocations():
    from test_pruned_widths_host import poisoned_alloc
    g = torch.Generator().manual_seed(10)
    h = (torch.randn(3, 3, 16, 16, generator=g) * 2e-4).cuda()
    outs = []
    for v in (float("nan"), 1e30, 0.0):
        m = _vq_f4().cuda()
        m.decode_batch = 4
        with poisoned_alloc(v) as cnt:
            outs.append(m.decode(h))
        assert cnt.n > 0
        del m
        gc.collect()
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs[2]).all())
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[2])


# ---------------------------------------------------------------------------------------------------------------------- launch census
def _replay_vq(lib, g, name, args, rep):
    from test_launch_census_gpu import _twice
    zp, N, D, H, W, inv, cp, n_embed, q, op, ld, ip = args
    z = (torch.randn(N, D, H, W, generator=g) * 2e-4).cuda()
    code = _codebook(g, n_embed, D).cuda()
    out = torch.full((N * H * W, ld), -777.0, device="cuda")
    idx = torch.full((N * H * W,), -1, dtype=torch.int64, device="cuda")

    def run():
        assert lib.dp_vq_quantize(z.data_ptr(), N, D, H, W, inv, code.data_ptr(), n_embed, q, out.data_ptr(), ld, idx.data_ptr(), S()) == 0
    got, gi = _twice(run, lambda: (out.fill_(-777.0), idx.fill_(-1)), [out, idx])
    zs = (z * torch.tensor(inv, device="cuda")).cpu()
    zf = zs.permute(0, 2, 3, 1).reshape(-1, D)
    if q:
        want, _ = _contract(zs, code.cpu())
        assert torch.equal(gi.cpu(), want), name
        zf = zf + (code.cpu()[want] - zf)
    assert torch.equal(got[:, :D].cpu(), zf) and bool((got[:, D:] == -777.0).all()), name
    rep.setdefault(name, []).append(0.0)


def _replay_decode_images(lib, g, name, args, rep):
    from test_launch_census_gpu import _twice
    yp, ld, N, Cc, H, W, up, fp_ = args
    y = torch.full((N * H * W, ld), 5.0, device="cuda")
    y[:, :Cc] = (torch.randn(N * H * W, Cc, generator=g) * 1.2).cuda()
    u8 = torch.zeros(N, H, W, Cc, dtype=torch.uint8, device="cuda")
    f = torch.zeros(N, Cc, H, W, device="cuda")

    def run():
        assert lib.dp_decode_images(y.data_ptr(), ld, N, Cc, H, W, u8.data_ptr(), f.data_ptr(), S()) == 0
    gu, gf = _twice(run, lambda: (u8.zero_(), f.zero_()), [u8, f])
    x = y[:, :Cc].reshape(N, H, W, Cc).permute(0, 3, 1, 2)
    v = torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0)
    assert torch.equal(gf, v), name
    assert torch.equal(gu, v.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)), name
    rep.setdefault(name, []).append(0.0)


def test_vq_decoder_census(lib):
    """Every distinct launch of VQ-f4 decode at a 64 x 64 latent (batch 2) and of the small config (SIMT attention), plus the byte
    conversion, replayed on fresh seeded buffers and checked against float64 (bounds of launch_census.py) or bit for bit."""
    from test_eval_census_gpu import EVAL_REPLAY, _LOG
    from test_launch_census_gpu import _capture, _unique
    replay = dict(EVAL_REPLAY)
    replay.update({"dp_vq_quantize": _replay_vq, "dp_decode_images": _replay_decode_images})
    _LOG.clear()
    _LOG.update(geoms=set(), tc=[], simt=set())

    def run():
        for m, h in ((_vq_f4(), torch.randn(2, 3, 64, 64) * 2e-4), (vq_model("tiny", n_embed=512), torch.randn(2, 3, 8, 8) * 0.01)):
            m = m.cuda()
            m.use_graph = False
            m.decode_batch = 2
            y = m.decode_chunk(h.cuda()).plan.y_out
            u8 = torch.empty(2, y.H, y.W, 3, dtype=torch.uint8, device="cuda")
            assert lib.dp_decode_images(y.ptr, y.ld, 2, 3, y.H, y.W, u8.data_ptr(), None, S()) == 0
            torch.cuda.synchronize()
    calls = _capture(lib, run)
    gc.collect()
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert {"dp_vq_quantize", "dp_decode_images", "dp_conv2d_fprop", "dp_groupnorm_fwd", "dp_gemm_nt_tc", "dp_gemm_batched",
            "dp_upsample2x_fwd"} <= kinds, sorted(kinds)
    missing = kinds - set(replay)
    assert not missing, f"launch kinds without a replay: {sorted(missing)}"
    rep, failures = {}, []
    g = torch.Generator().manual_seed(2026)
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
    assert set(rep) == kinds
    print(f"\nVQ decoder census: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds")
    for name in sorted(rep):
        print(f"  {name:26s} worst err/bound {max(rep[name]):.3f}")


# ---------------------------------------------------------------------------------------------------------------------- end to end
def _tiny_ldm():
    from diff_pruning_b200 import ldm
    from diff_pruning_b200.ldm_sampling import LatentDiffusion
    torch.manual_seed(0)
    m = LatentDiffusion(unet_config=ldm.LDM_TINY_CONFIG, cond_stage_config=dict(embed_dim=16),
                        first_stage_config=dict(embed_dim=3, n_embed=256, ddconfig=GOLD["configs"]["tiny"]["ddconfig"]))
    g = torch.Generator().manual_seed(5)
    for p in m.model.diffusion_model.parameters():        # a fresh LDM UNet outputs exactly 0: re-draw its zero-initialised layers
        if p.dim() > 1 and float(p.detach().abs().sum()) == 0:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.05)
    m.first_stage_model.decoder.load_state_dict(seeded_decoder("tiny").state_dict())
    return m.cuda().eval()


def test_sample_for_fid_files_and_features_equal_device_bytes(tmp_path):
    from PIL import Image
    from diff_pruning_b200 import fid
    from diff_pruning_b200.ldm_sampling import DDIMSampler, sample_for_fid
    from test_fid_gpu import seeded_model
    model = _tiny_ldm()
    inc = seeded_model((3,))
    kw = dict(classes=[3, 11], ipc=4, batch_size=2, ddim_steps=4, decode_batch=2)
    mu, sigma, n = sample_for_fid(model, out_dir=str(tmp_path), inception=inc, generator=torch.Generator(device="cuda").manual_seed(0), **kw)
    assert n == 8
    files = sorted(os.listdir(tmp_path))
    assert files == sorted(f"{c}_{i}.png" for i, c in enumerate([3, 3, 11, 11, 3, 3, 11, 11]))
    # the same loop by hand: the device bytes, and the torchvision chain on decode_first_stage's output
    from torchvision import utils as tvu
    gen = torch.Generator(device="cuda").manual_seed(0)
    from diff_pruning_b200 import _lib as L
    sampler, key, lib = DDIMSampler(model), model.cond_stage_key, L.load()
    model.first_stage_model.decode_batch = 2          # the micro-batch sample_for_fid decoded with
    uc = model.get_learned_conditioning({key: torch.tensor([1000, 1000]).cuda()})
    img_id, order = 0, []
    for _ in range(2):
        for c in kw["classes"]:
            cond = model.get_learned_conditioning({key: torch.tensor([c, c]).cuda()})
            smp, _ = sampler.sample(S=4, conditioning=cond, batch_size=2, shape=[3, 16, 16], verbose=False, unconditional_guidance_scale=3.0,
                                    unconditional_conditioning=uc, eta=0.0, generator=gen)
            x = torch.clamp((model.decode_first_stage(smp) + 1.0) / 2.0, min=0.0, max=1.0)
            y = model.first_stage_model.decode_chunk(smp).plan.y_out
            u8 = torch.empty(2, y.H, y.W, 3, dtype=torch.uint8, device="cuda")
            assert lib.dp_decode_images(y.ptr, y.ld, 2, 3, y.H, y.W, u8.data_ptr(), None, S()) == 0
            for i in range(2):
                f = tmp_path / f"{c}_{img_id}.png"
                assert np.array_equal(np.asarray(Image.open(f).convert("RGB")), u8[i].cpu().numpy()), f
                p = tmp_path / "tv.png"
                tvu.save_image(x[i], str(p))
                assert np.array_equal(np.asarray(Image.open(p)), u8[i].cpu().numpy()), f
                order.append(f)
                img_id += 1
    os.remove(tmp_path / "tv.png")
    # FID features of the files, batched as the loop batched them (2 per batch, in generation order), equal the device statistics
    mom = fid.Moments(2048)
    for s in range(0, len(order), 2):
        x = fid._decode(order[s:s + 2])
        plan = inc.plan(2, "u8", x.shape[1:3])
        plan.load(x.cuda())
        plan.run()
        mom.add(plan.feat[3])
    mu2, sigma2 = mom.finalize()
    assert np.array_equal(mu, mu2) and np.array_equal(sigma, sigma2)
