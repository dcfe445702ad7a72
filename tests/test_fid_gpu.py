"""FID evaluation on the GPU: the ReLU convolution epilogue on Inception geometries, the input kernel, pools, fp64 moments, the
end-to-end feature pass against the reference's features, graph replay, and DDIM samples scored from device memory vs. from PNGs."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, load_golden, max_rel, rel_err
from oracle import inception_oracle as orc
import diff_pruning_b200 as dp
import diff_pruning_b200.fid as fid
from diff_pruning_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _s():
    return torch.cuda.current_stream().cuda_stream


def seeded_model(blocks=(0, 1, 2, 3)):
    lay = json.load(open(os.path.join(GOLDEN, "fid_weights.json")))
    return fid.InceptionV3(list(blocks), weights=orc.seeded_state_dict(lay["weight_file"], lay["seed"])).cuda()


# (C, K, R, S, stride, pad_h, pad_w, H, W): every filter / stride / padding class of the Inception pass, at small extents, with
# N*P*Q and K off multiples of 128 and C off multiples of 64
GEOMS = [
    (3, 32, 3, 3, 2, 0, 0, 37, 37), (32, 64, 3, 3, 1, 1, 1, 19, 19), (80, 192, 3, 3, 1, 0, 0, 13, 13), (64, 80, 1, 1, 1, 0, 0, 13, 13),
    (48, 64, 5, 5, 1, 2, 2, 11, 11), (96, 96, 3, 3, 1, 1, 1, 11, 11), (288, 384, 3, 3, 2, 0, 0, 11, 11), (128, 128, 1, 7, 1, 0, 3, 9, 9),
    (160, 192, 7, 1, 1, 3, 0, 9, 9), (768, 192, 1, 1, 1, 0, 0, 9, 9), (192, 320, 3, 3, 2, 0, 0, 9, 9), (384, 384, 1, 3, 1, 0, 1, 8, 8),
    (384, 384, 3, 1, 1, 1, 0, 8, 8), (448, 384, 3, 3, 1, 1, 1, 8, 8), (1280, 320, 1, 1, 1, 0, 0, 8, 8),
]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("relu", [False, True])
def test_conv_relu_inception_geometries(geom, relu):
    C, K, R, S, st, ph, pw, H, W = geom
    N = 3
    P, Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1
    g = torch.Generator().manual_seed(C * 7 + K + R)
    x = torch.randn(N, C, H, W, generator=g)
    w = torch.randn(K, C, R, S, generator=g) / (C * R * S) ** 0.5
    b = torch.randn(K, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), st, (ph, pw)).float()
    if relu:
        ref = F.relu(ref)
    # input and output as channel slices of wider (concatenated) buffers
    xb = torch.zeros(N, H, W, C + 12, device="cuda")
    xb[..., 5:5 + C] = x.permute(0, 2, 3, 1).cuda()
    yb = torch.full((N, P, Q, K + 20), 7.0, device="cuda")
    wpk = torch.empty(R * S * C * K, device="cuda")
    wd, bd = w.cuda().contiguous(), b.cuda()
    L.check(L.load().dp_pack_conv_weight(wd.data_ptr(), K, C, R, S, wpk.data_ptr(), None, _s()), "pack")
    slot = torch.zeros(1, dtype=torch.int32, device="cuda")
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l = N, H, W, C, P, Q, K, R, S, st, ph, pw
    a.flags, a.splits = (fid.DP_CONV_RELU if relu else 0), 1
    a.x, a.ldx, a.y, a.ldy = xb.data_ptr() + 20, C + 12, yb.data_ptr() + 4 * 8, K + 20
    a.w, a.bias, a.amax_out = wpk.data_ptr(), bd.data_ptr(), slot.data_ptr()
    L.check(L.load().dp_conv2d_fprop(ctypes.byref(a), _s()), "fprop")
    torch.cuda.synchronize()
    got = yb[..., 8:8 + K].permute(0, 3, 1, 2).cpu()
    assert rel_err(got, ref) <= 1e-5
    if relu:
        assert float(got.min()) >= 0.0
    assert torch.all(yb[..., :8] == 7.0) and torch.all(yb[..., 8 + K:] == 7.0)
    amax = slot.cpu().view(torch.float32).item()
    assert amax >= float(got.abs().max())


class TcConv:
    """One fprop launch with every operand both kernels take: SIMT packed weight, fp16 hi / lo' pair, amax slots of x and w."""

    def __init__(self, geom, N, seed, ldx_extra=12, ldy_extra=20, x_off=4, y_off=8):
        C, K, R, S, st, ph, pw, H, W = geom
        self.geom, self.N = geom, N
        self.P, self.Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1
        g = torch.Generator().manual_seed(seed)
        self.x = torch.randn(N, C, H, W, generator=g)
        self.w = torch.randn(K, C, R, S, generator=g) / (C * R * S) ** 0.5
        self.b = torch.randn(K, generator=g)
        self.ldx, self.ldy, self.x_off, self.y_off = C + ldx_extra, K + ldy_extra, x_off, y_off   # views inside wider buffers
        self.xb = torch.zeros(N, H, W, self.ldx, device="cuda")
        self.xb[..., x_off:x_off + C] = self.x.permute(0, 2, 3, 1).cuda()
        lib = L.load()
        wd = self.w.cuda().contiguous()
        self.bd = self.b.cuda()
        cp = lib.dp_tc_weight_row(C)
        self.wpk = torch.empty(R * S * C * K, device="cuda")
        self.hi = torch.empty(R * S * K * cp, dtype=torch.float16, device="cuda")
        self.lo = torch.empty_like(self.hi)
        self.slots = torch.zeros(3, dtype=torch.int32, device="cuda")      # w, x, out
        L.check(lib.dp_pack_conv_weight(wd.data_ptr(), K, C, R, S, self.wpk.data_ptr(), None, _s()), "pack")
        L.check(lib.dp_pack_conv_weight_tc(wd.data_ptr(), K, C, R, S, self.hi.data_ptr(), self.lo.data_ptr(), None, None,
                                           self.slots.data_ptr(), _s()), "pack tc")
        L.check(lib.dp_amax(self.xb.data_ptr() + 4 * x_off, self.ldx, N * H * W, C, self.slots.data_ptr() + 4, _s()), "amax")

    def args(self, flags, yb, ws=None):
        C, K, R, S, st, ph, pw, H, W = self.geom
        a = L.ConvArgs()
        a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l = self.N, H, W, C, self.P, self.Q, K, R, S, st, ph, pw
        a.flags, a.splits = flags, 1
        a.x, a.ldx, a.y, a.ldy = self.xb.data_ptr() + 4 * self.x_off, self.ldx, yb.data_ptr() + 4 * self.y_off, self.ldy
        a.w, a.bias, a.w_tc_hi, a.w_tc_lo = self.wpk.data_ptr(), self.bd.data_ptr(), self.hi.data_ptr(), self.lo.data_ptr()
        a.amax_w, a.amax_x, a.amax_out = self.slots.data_ptr(), self.slots.data_ptr() + 4, self.slots.data_ptr() + 8
        a.workspace = ws.data_ptr() if ws is not None else None
        return a

    def run(self, flags, split=False):
        C, K = self.geom[0], self.geom[1]
        lib = L.load()
        yb = torch.full((self.N, self.P, self.Q, self.ldy), 7.0, device="cuda")
        need = lib.dp_conv_splitk_workspace_floats(ctypes.byref(self.args(flags, yb)), 0)
        ws = torch.empty(max(need, 1), device="cuda") if split else None
        self.slots[2] = 0
        L.check(lib.dp_conv2d_fprop(ctypes.byref(self.args(flags, yb, ws)), _s()), "fprop")
        torch.cuda.synchronize()
        assert torch.all(yb[..., :self.y_off] == 7.0) and torch.all(yb[..., self.y_off + K:] == 7.0)
        return yb[..., self.y_off:self.y_off + K].permute(0, 3, 1, 2).cpu(), need

    def ref(self, relu):
        C, K, R, S, st, ph, pw, H, W = self.geom
        r = F.conv2d(self.x.double(), self.w.double(), self.b.double(), st, (ph, pw)).float()
        return F.relu(r) if relu else r


# every row of the Inception MAC table (filter, stride / padding, grid) at batch 2, plus tails: N*P*Q off 128 everywhere, K = 80 / 320,
# C = 48 / 80 / 288 / 1280 (not multiples of 64)
ANY_GEOMS = [
    (128, 128, 1, 7, 1, 0, 3, 17, 17), (160, 192, 7, 1, 1, 3, 0, 17, 17), (768, 192, 1, 1, 1, 0, 0, 17, 17), (64, 192, 3, 3, 1, 0, 0, 37, 37),
    (64, 96, 3, 3, 1, 1, 1, 35, 35), (32, 64, 3, 3, 1, 1, 1, 47, 47), (288, 384, 3, 3, 2, 0, 0, 35, 35), (1280, 320, 1, 1, 1, 0, 0, 8, 8),
    (48, 64, 5, 5, 1, 2, 2, 35, 35), (288, 64, 1, 1, 1, 0, 0, 35, 35), (32, 32, 3, 3, 1, 0, 0, 49, 49), (448, 384, 3, 3, 1, 1, 1, 8, 8),
    (384, 384, 1, 3, 1, 0, 1, 8, 8), (384, 384, 3, 1, 1, 1, 0, 8, 8), (192, 192, 3, 3, 2, 0, 0, 17, 17), (64, 80, 1, 1, 1, 0, 0, 37, 37),
]


@pytest.mark.parametrize("geom", ANY_GEOMS)
@pytest.mark.parametrize("relu", [False, True])
def test_general_geometry_conv(geom, relu):
    t = TcConv(geom, 2, seed=sum(geom))
    flags = fid.DP_CONV_ANY_GEOMETRY | (fid.DP_CONV_RELU if relu else 0)
    ref = t.ref(relu)
    got, need = t.run(flags)
    assert rel_err(got, ref) <= 1e-5
    assert t.slots[2:].cpu().view(torch.float32).item() >= float(got.abs().max())
    if relu:
        assert float(got.min()) >= 0.0
    if need:      # split-K: the same bound, ReLU and amax after the fixed-order sum
        got_s, _ = t.run(flags, split=True)
        assert rel_err(got_s, ref) <= 1e-5
        assert t.slots[2:].cpu().view(torch.float32).item() >= float(got_s.abs().max())
        if relu:
            assert float(got_s.min()) >= 0.0
        got_s2, _ = t.run(flags, split=True)
        assert torch.equal(got_s, got_s2)         # deterministic
    # the general path really ran: SIMT (exact fp32) gives different low bits
    simt, _ = t.run(flags | fid.DP_CONV_FORCE_SIMT)
    assert not torch.equal(simt, got)


def test_general_geometry_split_k_is_exercised():
    t = TcConv((384, 384, 3, 1, 1, 1, 0, 8, 8), 2, seed=3)
    assert L.load().dp_conv_splitk_workspace_floats(ctypes.byref(t.args(fid.DP_CONV_ANY_GEOMETRY, t.xb)), 0) > 0


@pytest.mark.parametrize("geom", [(64, 128, 3, 3, 1, 1, 1, 16, 16), (128, 128, 1, 1, 1, 0, 0, 8, 8), (64, 64, 3, 3, 2, 1, 1, 32, 32)])
def test_box_kernel_routing_unchanged(geom):
    """Geometries the box kernel takes give the same bits with and without DP_CONV_ANY_GEOMETRY (split-K included)."""
    t = TcConv(geom, 2, seed=5, ldx_extra=0, ldy_extra=0, x_off=0, y_off=0)
    for split in (False, True):
        a, _ = t.run(0, split)
        b, _ = t.run(fid.DP_CONV_ANY_GEOMETRY, split)
        assert torch.equal(a, b)


def test_small_channel_counts_stay_on_simt():
    t = TcConv((3, 32, 3, 3, 2, 0, 0, 37, 37), 2, seed=7)
    a, _ = t.run(fid.DP_CONV_ANY_GEOMETRY | fid.DP_CONV_RELU)
    b, _ = t.run(fid.DP_CONV_FORCE_SIMT | fid.DP_CONV_RELU)
    assert torch.equal(a, b)


def test_relu_flag_takes_exact_path_with_tc_operands():
    """A launch that carries tensor-core operands and DP_CONV_RELU runs the exact-fp32 kernel: same bits as with FORCE_SIMT."""
    lib = L.load()
    N, H, W, C, K = 2, 16, 16, 64, 128
    x = torch.randn(N, H, W, C, device="cuda")
    w = torch.randn(K, C, 3, 3, device="cuda") * 0.05
    wpk = torch.empty(9 * C * K, device="cuda")
    Cp = lib.dp_tc_weight_row(C)
    hi, lo = torch.empty(9 * K * Cp, dtype=torch.float16, device="cuda"), torch.empty(9 * K * Cp, dtype=torch.float16, device="cuda")
    sw, sx = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.dp_pack_conv_weight(w.data_ptr(), K, C, 3, 3, wpk.data_ptr(), None, _s()), "pack")
    L.check(lib.dp_pack_conv_weight_tc(w.data_ptr(), K, C, 3, 3, hi.data_ptr(), lo.data_ptr(), None, None, sw.data_ptr(), _s()), "pack tc")
    L.check(lib.dp_amax(x.data_ptr(), C, N * H * W, C, sx.data_ptr(), _s()), "amax")
    outs = []
    for flags in (fid.DP_CONV_RELU, fid.DP_CONV_RELU | 2):
        y = torch.empty(N, H, W, K, device="cuda")
        a = L.ConvArgs()
        a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l = N, H, W, C, H, W, K, 3, 3, 1, 1, 1
        a.flags, a.splits, a.x, a.ldx, a.y, a.ldy, a.w = flags, 1, x.data_ptr(), C, y.data_ptr(), K, wpk.data_ptr()
        a.w_tc_hi, a.w_tc_lo, a.amax_x, a.amax_w = hi.data_ptr(), lo.data_ptr(), sx.data_ptr(), sw.data_ptr()
        L.check(lib.dp_conv2d_fprop(ctypes.byref(a), _s()), "fprop")
        outs.append(y)
    assert torch.equal(outs[0], outs[1]) and float(outs[0].min()) >= 0.0


@pytest.mark.parametrize("hw", [(32, 32), (64, 48), (256, 256)])
def test_input_kernel_u8_matches_interpolate(hw):
    N = 3
    u8 = torch.randint(0, 256, (N, hw[0], hw[1], 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros(N, 299, 299, 4, device="cuda")
    L.check(L.load().dp_fid_input(u8.data_ptr(), 1, 0, N, hw[0], hw[1], out.data_ptr(), 4, 299, 299, 1, 1, None, _s()), "fid_input")
    x = u8.permute(0, 3, 1, 2).float().div(255)
    ref = 2 * F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1
    got = out[..., :3].permute(0, 3, 1, 2)
    assert float((got - ref).abs().max()) <= 2e-6
    assert torch.all(out[..., 3] == 0)


def test_input_kernel_quantisation_equals_png_values():
    N, H, W = 4, 20, 24
    x = torch.randn(N, 3, H, W, device="cuda") * 0.7
    x.view(-1)[:6] = torch.tensor([-1.0, 1.0, 3.0, -3.0, 2.0 / 255 - 1, 1.0 / 255 - 1], device="cuda")   # clamps, a .5 tie
    png = ((x / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")   # sampling.py's PIL path
    png = np.ascontiguousarray(png)        # as PIL holds it: packed HWC rows
    lib = L.load()
    a = torch.zeros(N, H, W, 4, device="cuda")
    b = torch.zeros(N, H, W, 4, device="cuda")
    L.check(lib.dp_fid_input(x.data_ptr(), 0, 1, N, H, W, a.data_ptr(), 4, H, W, 0, 0, None, _s()), "quantise")
    u8 = torch.from_numpy(png).cuda()
    L.check(lib.dp_fid_input(u8.data_ptr(), 1, 0, N, H, W, b.data_ptr(), 4, H, W, 0, 0, None, _s()), "u8")
    assert torch.equal(a, b)
    assert torch.equal((a[..., :3].cpu() * 255).round().to(torch.uint8), torch.from_numpy(png))


@pytest.mark.parametrize("case", [("max", 2, 0), ("avg", 1, 1), ("max", 1, 1)])
def test_pools_match_torch(case):
    kind, st, pad = case
    N, H, W, C = 2, 17, 15, 40
    xb = torch.randn(N, H, W, C + 8, device="cuda")
    x = xb[..., 3:3 + C]
    P, Q = (H + 2 * pad - 3) // st + 1, (W + 2 * pad - 3) // st + 1
    yb = torch.zeros(N, P, Q, C + 4, device="cuda")
    slot = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.load().dp_pool3x3(xb.data_ptr() + 12, C + 8, yb.data_ptr() + 16, C + 4, N, H, W, C, st, pad, 0 if kind == "max" else 1,
                                slot.data_ptr(), _s()), "pool")
    assert slot.cpu().view(torch.float32).item() == float(yb[..., 4:4 + C].abs().max())
    xn = x.permute(0, 3, 1, 2).contiguous()
    ref = F.max_pool2d(xn, 3, st, pad) if kind == "max" else F.avg_pool2d(xn, 3, st, pad, count_include_pad=False)
    assert torch.equal(yb[..., 4:4 + C].permute(0, 3, 1, 2), ref)


def test_global_mean():
    N, H, W, C = 3, 8, 8, 70
    x = torch.randn(N, H, W, C + 2, device="cuda")
    y = torch.zeros(N, C, device="cuda")
    L.check(L.load().dp_global_mean(x.data_ptr(), C + 2, y.data_ptr(), C, N, H, W, C, _s()), "mean")
    ref = x[..., :C].double().mean((1, 2))
    assert max_rel(y, ref) < 1e-6


@pytest.mark.parametrize("offset", [0.0, 100.0])
def test_moments_match_numpy(offset):
    D = 200
    f = torch.relu(torch.randn(300, D + 5, device="cuda")) + 0.1 + offset * torch.rand(D + 5, device="cuda")   # mean / std up to ~100
    mom = fid.Moments(D)
    mom.add(f[:128, :D])
    mom.add(f[128:, :D])         # moments add over batches
    mu, sigma = mom.finalize()
    act = f[:, :D].double().cpu().numpy()
    assert np.abs(mu - act.mean(0)).max() <= 1e-12 * np.abs(act.mean(0)).max()
    ref = np.cov(act, rowvar=False)
    assert np.linalg.norm(sigma - ref) <= 1e-12 * np.linalg.norm(ref)
    assert np.array_equal(sigma, sigma.T)
    again = fid.Moments(D)
    again.add(f[:128, :D])
    again.add(f[128:, :D])
    assert torch.equal(again.sxx, mom.sxx) and torch.equal(again.s, mom.s)     # fixed order: run-to-run identical


def test_features_match_reference_all_blocks():
    model = seeded_model()
    gold = load_golden("fid_features.pt")
    for hw, u8 in gold["images"].items():
        plan = model.plan(u8.shape[0], "u8", u8.shape[1:3])
        plan.load(u8.cuda())
        plan.run()
        for b in range(4):
            assert max_rel(plan.feat[b], gold["features"][hw][b]) <= 1e-4, (hw, b)
        # the module's forward (fp32 NCHW in [0, 1]) gives the same features
        outs = model(u8.permute(0, 3, 1, 2).float().div(255).cuda())
        assert max_rel(orc.pooled(outs[3]), gold["features"][hw][3]) <= 1e-4


def test_graph_replay_equals_eager():
    model = seeded_model((1, 3))
    u8 = torch.randint(0, 256, (5, 40, 40, 3), dtype=torch.uint8, device="cuda")
    eager = fid.FeaturePlan(model, 5, "u8", (40, 40), use_graph=False)
    graph = fid.FeaturePlan(model, 5, "u8", (40, 40), use_graph=True)
    for p in (eager, graph):
        p.load(u8)
        p.run()
    graph.run()           # second replay
    torch.cuda.synchronize()
    for b in (1, 3):
        assert torch.equal(eager.feat[b], graph.feat[b])


def test_short_final_batch_and_partial_rows(tmp_path):
    from PIL import Image
    model = seeded_model((3,))
    imgs = torch.randint(0, 256, (7, 24, 24, 3), dtype=torch.uint8)
    files = []
    for i, im in enumerate(imgs.numpy()):
        p = tmp_path / f"{i:03d}.png"
        Image.fromarray(im).save(p)
        files.append(p)
    act = fid.get_activations(files, model, batch_size=3, dims=2048)
    assert act.shape == (7, 2048)
    again = fid.get_activations(files, model, batch_size=3, dims=2048)
    assert np.array_equal(act, again)          # the zeroed tail: a short batch depends on its own images only
    full = model.plan(7, "u8", (24, 24))
    full.load(imgs.cuda())
    full.run()
    # one batch of 7 vs 3 + 3 + 1: the tensor-core operand scales are per batch, so the features agree to fp32 grade, not bit for bit
    assert max_rel(torch.from_numpy(act), full.feat[3]) <= 1e-5
    mu, sigma = fid.calculate_activation_statistics(files, model, batch_size=3, dims=2048)
    assert np.abs(mu - act.mean(0)).max() <= 1e-12 * np.abs(act).max()
    ref = np.cov(act, rowvar=False)
    assert np.linalg.norm(sigma - ref) <= 1e-10 * np.linalg.norm(ref)


def test_pipeline_features_equal_png_features(tmp_path):
    torch.manual_seed(0)
    unet = dp.UNet2DModel(**dp.TINY_TEST_CONFIG).cuda().eval()
    pipe = dp.DDIMPipeline(unet=unet, scheduler=dp.DDPMScheduler(num_train_timesteps=1000))
    model = seeded_model((3,))
    mu, sigma, feats = fid.statistics_of_pipeline(pipe, total_samples=8, batch_size=4, num_inference_steps=3, seed=3, dims=2048,
                                                   model=model, return_features=True)
    # the same samples as ddpm_sample.py writes them, then scored from the folder
    gen = torch.Generator(device=pipe.device).manual_seed(3)
    for i in range(2):
        for j, im in enumerate(pipe(batch_size=4, num_inference_steps=3, generator=gen).images):
            im.save(tmp_path / f"{i * 4 + j:04d}.png")
    files = fid._image_files(tmp_path)
    assert len(files) == 8
    act = fid.get_activations(files, model, batch_size=4, dims=2048)
    assert np.array_equal(feats, act)
    m2, s2 = fid.compute_statistics_of_path(str(tmp_path), model, 4, 2048)
    assert np.array_equal(mu, m2) and np.array_equal(sigma, s2)
