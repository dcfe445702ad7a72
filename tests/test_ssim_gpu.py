"""SSIM evaluation on the GPU: dp_ssim against the reference's utils_image.py values and the torch oracle, the three source formats
against each other, determinism and batch independence, the MSE, compute_ssim.py's call sequence through the compat import, and
DDIM pipelines scored from device memory vs. from their PNGs."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, load_golden
from oracle import ssim_oracle as orc
import diff_pruning_b200 as dp
import diff_pruning_b200.ssim as S
from diff_pruning_b200 import pruning
from diff_pruning_b200.scoring import TaylorScorer

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT, "diff-pruning_b200", "compat"))

G64 = orc.window(dtype=torch.float64)


def _u8_nchw(u8):
    return u8.permute(0, 3, 1, 2)


def test_golden_pairs():
    """Within 1e-6 of utils_image.py (fp64 NumPy + cv2) on every fixture pair, from uint8 at data_range 1 and from fp32 0..255 values at
    data_range 255, with the exact-grade taps; an image against itself gives exactly 1."""
    for case in load_golden("ssim_ref.pt"):
        x, y = case["x"][None].cuda(), case["y"][None].cuda()
        routes = {"u8": S._scores(x, y, S.DP_SSIM_U8_NHWC, 1.0, win=G64)[0],
                  "f32_255": S._scores(_u8_nchw(x).float().contiguous(), _u8_nchw(y).float().contiguous(), S.DP_SSIM_F32_NCHW, 255.0,
                                       win=G64)[0]}
        for route, nc in routes.items():
            nc = nc.cpu()[0]
            assert float((nc - case["ssim_c"]).abs().max()) <= 1e-6, (case["name"], route)
            assert abs(float(S._per_image(nc[None])[0]) - case["ssim"]) <= 1e-6, (case["name"], route)
            if case["name"] == "identical":
                assert torch.all(nc == 1.0)
    ident = [c for c in load_golden("ssim_ref.pt") if c["name"] == "identical"][0]
    xi = _u8_nchw(ident["x"][None]).float().div(255).cuda()
    assert float(S.ssim(xi, xi.clone(), data_range=1.0)) == 1.0


def _batches():
    g = torch.Generator().manual_seed(11)
    out = {}
    for hw in (32, 256):
        rnd = torch.rand(6, 3, hw, hw, generator=g)
        out[f"random_{hw}"] = (rnd, torch.rand(6, 3, hw, hw, generator=g))
        base = F.interpolate(torch.rand(6, 3, hw // 8, hw // 8, generator=g), size=(hw, hw), mode="bilinear", align_corners=False)
        out[f"structured_{hw}"] = (base, (base + 0.03 * torch.randn(base.shape, generator=g)).clamp(0, 1))
        # flat regions (sky, walls): a bright constant with a few steps of 1/255, where fp32 moments cancel against C2
        flat = torch.full((6, 3, hw, hw), 0.85)
        bumpy = flat.clone()
        bumpy[:, :, hw // 4: hw // 2, hw // 3:] += 1 / 255
        bumpy[:, :, ::7, ::5] -= 2 / 255
        out[f"flat_{hw}"] = (flat + (torch.rand(flat.shape, generator=g) < 0.02) / 255, bumpy)
    return out


def test_versus_torch_oracle():
    """For every image: |ours - fp64 oracle| <= |fp32 oracle (pytorch_msssim's arithmetic) - fp64 oracle| + 1e-6, with the fp32 taps
    of pytorch_msssim on all three."""
    for name, (x, y) in _batches().items():
        xc, yc = x.cuda(), y.cuda()
        ours = S._per_image(S._scores(xc, yc, S.DP_SSIM_F32_NCHW, 1.0)[0]).cpu()
        ref64 = orc.ssim_per_channel(xc.double(), yc.double(), 1.0).mean(1).cpu()
        ref32 = orc.ssim_per_channel(xc, yc, 1.0).mean(1).double().cpu()
        e_ours, e_32 = (ours - ref64).abs(), (ref32 - ref64).abs()
        print(f"{name}: max |ours - fp64 oracle| {float(e_ours.max()):.3e}, max |fp32 oracle - fp64 oracle| {float(e_32.max()):.3e}")
        assert torch.all(e_ours <= e_32 + 1e-6), name
        # the public surface returns the same values in fp32
        pub = S.ssim(xc, yc, data_range=1.0, size_average=False)
        assert pub.dtype == torch.float32 and pub.is_cuda and torch.equal(pub.cpu(), ours.float())


def test_routes_agree():
    g = torch.Generator().manual_seed(5)
    u8a = torch.randint(0, 256, (5, 40, 36, 3), dtype=torch.uint8, generator=g)
    u8b = (u8a.int() + torch.randint(-20, 21, u8a.shape, generator=g)).clamp(0, 255).to(torch.uint8)
    r_u8 = S._scores(u8a.cuda(), u8b.cuda(), S.DP_SSIM_U8_NHWC, 1.0)
    fa, fb = (_u8_nchw(u).float().div(255).contiguous().cuda() for u in (u8a, u8b))      # ToTensor's values
    r_f32 = S._scores(fa, fb, S.DP_SSIM_F32_NCHW, 1.0)
    assert torch.equal(r_u8[0], r_f32[0]) and torch.equal(r_u8[1], r_f32[1])
    # DDIM-sample-like tensors through the PNG quantisation vs. the PNG bytes sampling.py's PIL path writes
    xa, xb = torch.randn(4, 3, 24, 20, generator=g) * 0.7, torch.randn(4, 3, 24, 20, generator=g) * 0.7
    xa.view(-1)[:6] = torch.tensor([-1.0, 1.0, 3.0, -3.0, 2.0 / 255 - 1, 1.0 / 255 - 1])   # clamps, a .5 tie

    def png(x):
        return torch.from_numpy(np.ascontiguousarray(((x / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")))
    r_q = S._scores(xa.cuda(), xb.cuda(), S.DP_SSIM_F32_NCHW_PNG, 1.0)
    r_png = S._scores(png(xa).cuda(), png(xb).cuda(), S.DP_SSIM_U8_NHWC, 1.0)
    assert torch.equal(r_q[0], r_png[0]) and torch.equal(r_q[1], r_png[1])


def test_deterministic_and_batch_independent():
    g = torch.Generator().manual_seed(9)
    for hw in (32, 256):
        x, y = torch.rand(7, 3, hw, hw, generator=g).cuda(), torch.rand(7, 3, hw, hw, generator=g).cuda()
        a = S._scores(x, y, S.DP_SSIM_F32_NCHW, 1.0)
        b = S._scores(x, y, S.DP_SSIM_F32_NCHW, 1.0)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        for i in (0, 4, 6):
            one = S._scores(x[i:i + 1].contiguous(), y[i:i + 1].contiguous(), S.DP_SSIM_F32_NCHW, 1.0)
            assert torch.equal(one[0][0], a[0][i]) and torch.equal(one[1][0], a[1][i])


def test_mse():
    g = torch.Generator().manual_seed(13)
    x, y = torch.rand(5, 3, 48, 40, generator=g), torch.rand(5, 3, 48, 40, generator=g)
    _, sse = S._scores(x.cuda(), y.cuda(), S.DP_SSIM_F32_NCHW, 1.0)
    mse = (sse / x[0].numel()).cpu()
    ref64 = (x - y).double().pow(2).mean((1, 2, 3))          # fp64 on the fp32 differences
    assert float(((mse - ref64).abs() / ref64).max()) <= 1e-12
    ref = F.mse_loss(x.cuda(), y.cuda(), reduction="none").mean(dim=(1, 2, 3)).double().cpu()     # compute_ssim.py's
    assert float(((mse - ref).abs() / ref).max()) <= 1e-6


def _write_pairs(root, n=7, hw=(32, 28)):
    from PIL import Image
    g = torch.Generator().manual_seed(21)
    for i in range(n):
        a = torch.randint(0, 256, (*hw, 3), dtype=torch.uint8, generator=g)
        b = (a.int() + torch.randint(-30, 31, a.shape, generator=g)).clamp(0, 255).to(torch.uint8)
        for d, im in (("a", a), ("b", b)):
            os.makedirs(root / d, exist_ok=True)
            Image.fromarray(im.numpy()).save(root / d / f"{i}.png")


def test_compat_call_sequence(tmp_path):
    """compute_ssim.py's loop through `import pytorch_msssim`: ToTensor'd batches of the two folders (here in sorted order, which is
    how ssim_of_paths pairs them), ssim(a.cuda(), b.cuda(), data_range=1.0, size_average=False)."""
    import pytorch_msssim
    import torchvision
    from PIL import Image
    _write_pairs(tmp_path)
    ssim_ref, mse_ref = S.ssim_of_paths(tmp_path / "a", tmp_path / "b", batch_size=3)
    tt = torchvision.transforms.ToTensor()
    files = sorted(os.listdir(tmp_path / "a"))
    ssim_list, mse_list = [], []
    with torch.no_grad():
        for s in range(0, len(files), 3):
            img1 = torch.stack([tt(Image.open(tmp_path / "a" / f).convert("RGB")) for f in files[s:s + 3]])
            img2 = torch.stack([tt(Image.open(tmp_path / "b" / f).convert("RGB")) for f in files[s:s + 3]])
            ssim_list.append(pytorch_msssim.ssim(img1.cuda(), img2.cuda(), data_range=1.0, size_average=False).cpu())
            mse_list.append(F.mse_loss(img1.cuda(), img2.cuda(), reduction="none").mean(dim=(1, 2, 3)).cpu())
    got = torch.cat(ssim_list)
    assert got.dtype == torch.float32
    assert np.array_equal(got.numpy(), ssim_ref.astype(np.float32))
    assert np.abs(torch.cat(mse_list).double().numpy() - mse_ref).max() <= 1e-6 * mse_ref.max()
    # batch size does not change per-image results
    s7, m7 = S.ssim_of_paths(tmp_path / "a", tmp_path / "b", batch_size=100)
    assert np.array_equal(s7, ssim_ref) and np.array_equal(m7, mse_ref)


def _tiny_pipelines():
    torch.manual_seed(0)
    unet = dp.UNet2DModel(**dp.TINY_TEST_CONFIG).cuda().eval()
    pruned = copy.deepcopy(unet)
    g = torch.Generator().manual_seed(1)
    clean, noise = torch.randn(4, 3, 16, 16, generator=g), torch.randn(4, 3, 16, 16, generator=g)
    pruned.zero_grad()
    sc = TaylorScorer(pruned, clean.cuda(), noise.cuda(), use_graph=False)
    for t in (0, 500, 999):
        sc.step(t)
    del sc
    pruning.taylor_prune(pruned, 0.3, "taylor", ignored_layers=[pruned.conv_out])
    pruned.zero_grad(set_to_none=True)
    pruned.eval()
    assert sum(p.numel() for p in pruned.parameters()) < sum(p.numel() for p in unet.parameters())
    sched = dp.DDPMScheduler(num_train_timesteps=1000)
    return dp.DDIMPipeline(unet=unet, scheduler=sched), dp.DDIMPipeline(unet=pruned, scheduler=sched)


def test_pipelines_equal_png_folders(tmp_path):
    base, pruned = _tiny_pipelines()
    s, m = S.ssim_of_pipelines(pruned, base, total_samples=8, batch_size=4, num_inference_steps=3, seed=3)
    assert s.shape == (8,) and m.shape == (8,) and s.dtype == np.float64
    # ddpm_sample.py: one generator per run, seeded; files <output_dir>/process_0/<i * batch + j>.png
    for name, pipe in (("pruned", pruned), ("base", base)):
        sub = tmp_path / name / "process_0"
        sub.mkdir(parents=True)
        gen = torch.Generator(device=pipe.device).manual_seed(3)
        for i in range(2):
            for j, im in enumerate(pipe(batch_size=4, num_inference_steps=3, generator=gen).images):
                im.save(sub / f"{i * 4 + j}.png")
    sp, mp = S.ssim_of_paths(tmp_path / "pruned", tmp_path / "base")       # sorted names 0.png .. 7.png: sample order
    assert np.array_equal(s, sp) and np.array_equal(m, mp)
    assert np.all(s < 1.0) and np.all(m > 0.0)
    s0, m0 = S.ssim_of_pipelines(base, base, total_samples=4, batch_size=4, num_inference_steps=3, seed=3)
    assert np.all(s0 == 1.0) and np.all(m0 == 0.0)
    other = dp.DDIMPipeline(unet=dp.UNet2DModel(**{**dp.TINY_TEST_CONFIG, "sample_size": 24}).cuda(), scheduler=base.scheduler)
    with pytest.raises(ValueError):
        S.ssim_of_pipelines(base, other, total_samples=4, batch_size=4, num_inference_steps=3)
