"""Launch census of the evaluation path: every distinct launch of the FID Inception feature pass (fid.FeaturePlan at the batch sizes and
input formats FID scoring runs: u8 files at batch 50, DDIM samples through the PNG quantisation at batch 128, LSUN-size files) and of DDIM
sampling (DDIMPipeline, C1 and pruned C1 at batch 128), replayed on fresh seeded buffers at its own geometry and checked element by
element against float64 with the census machinery of test_launch_census_gpu.py and the bounds of launch_census.py.

On top of the training census' replays: the ReLU / general-geometry convolutions (their split count recovered from the kernel's rule
and checked against the split-K workspace it asks for; the C = 3 stem on the SIMT kernel with L = R S C), the resize / normalise input
kernel, the 3 x 3 pools, the global mean, the fp64 feature moments and the DDIM update.  Directed edge cases of the input kernel, the
moments and the DDIM update, and the batch-128 pool3 features against the fp64 Inception oracle, follow the census.
"""
import gc
import math

import pytest
import torch
import torch.nn.functional as F

import launch_census as lc
from test_launch_census_gpu import (REPLAY, SENT, Buf, Conv, S, _capture, _check, _nchw, _nhwc_rows, _randn, _scaled, _slot_value,
                                    _twice, _unique, lib, replay_conv, replay_exact, replay_split)

pytestmark = pytest.mark.gpu

DP_CONV_RELU, DP_CONV_ANY_GEOMETRY = 4, 8
ANY_MIN_C = 32           # conv_tc.cu: general-geometry launches with fewer input channels run on the SIMT kernel
FAR = 1e30               # fill around the views a replay reads: a read outside the view shows in the result

# what the replays of one configuration saw: convolution geometries, chain lengths
_LOG = {}


def _num_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------- replays
def replay_eval_conv(lib, g, name, a, rep):
    """fprop with DP_CONV_RELU | DP_CONV_ANY_GEOMETRY (every Inception convolution): replay_conv with the ReLU reference and the chain
    of the kernel the launch runs on.  C >= 32: conv_tc_ps_kernel<true>, its split count from the kernel's own rule (which must ask for
    exactly the split-K workspace the library reports), L = 4 stages per split + splits <= L_MAX.  C < 32: the SIMT kernel, R S C
    sequential fp32 FMAs.  Other convolutions go to replay_conv unchanged."""
    if name != "dp_conv2d_fprop" or not a.flags & (DP_CONV_RELU | DP_CONV_ANY_GEOMETRY):
        return replay_conv(lib, g, name, a, rep)
    assert a.flags & DP_CONV_RELU, "general-geometry launches without the ReLU epilogue are outside the evaluation path"
    geom = (a.C, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l, a.H, a.W)
    if geom not in _LOG["geoms"]:
        # Conv pads the bottom / right by what the last window reaches past the image: the same as torch's symmetric padding
        assert a.P == (a.H + 2 * a.pad_t - a.R) // a.stride + 1 and a.Q == (a.W + 2 * a.pad_l - a.S) // a.stride + 1, geom
        cv = Conv(a)
        assert cv.pb <= a.pad_t and cv.pr <= a.pad_l, geom
        x1 = torch.randn(1, a.C, a.H, a.W, dtype=torch.float64, device="cuda")
        w1 = torch.randn(a.K, a.C, a.R, a.S, dtype=torch.float64, device="cuda")
        want = F.conv2d(x1, w1, stride=a.stride, padding=(a.pad_t, a.pad_l))
        assert torch.allclose(cv.fwd(x1, w1), want, rtol=1e-12, atol=1e-12 * float(want.abs().max())), geom
        _LOG["geoms"].add(geom)

    def chain(a, need):
        if a.C < ANY_MIN_C:
            _LOG["simt"].add(a.R * a.S * a.C)
            return a.R * a.S * a.C, False
        iters = a.R * a.S * -(-a.C // 64)
        ks, ips = lc.general_split(a.N, a.P, a.Q, a.K, a.C, a.R, a.S, _num_sms())
        if a.workspace:
            tile_floats = -(-(a.N * a.P * a.Q) // 128) * 128 * -(-a.K // 128) * 128
            assert need == (ks * tile_floats if ks > 1 else 0), (geom, need, ks)
        else:
            ks, ips = 1, iters
        L_ = lc.chain_general(ks, ips)
        _LOG["tc"].append((L_, ks, geom))
        return L_, True
    replay_conv(lib, g, name, a, rep, chain=chain)


def _exact(rep, name, got, ref, what):
    rep.setdefault(name, []).append(0.0)
    assert torch.equal(got, ref), f"{name} {what}: not bit-exact"


def _source(g, u8, quantize, N, Hs, Ws):
    """A seeded source of dp_fid_input and the [N, 3, Hs, Ws] fp32 values the kernel reads from it: ToTensor's u / 255, or the PNG
    quantisation of a DDIM sample in [-1, 1] (the uint8 the sampler writes, over 255).  The divisions run on the host, where torch
    divides correctly rounded (on the device it multiplies by the reciprocal)."""
    if u8:
        src = torch.randint(0, 256, (N, Hs, Ws, 3), generator=g, dtype=torch.uint8)
        return src.cuda(), (src.permute(0, 3, 1, 2).float() / 255).cuda()
    if not quantize:
        src = torch.rand(N, 3, Hs, Ws, generator=g)
        return src.cuda(), src.cuda()
    src = torch.randn(N, 3, Hs, Ws, generator=g) * 0.7
    edge = torch.tensor([-1.0, 1.0, 3.0, -3.0, 2.0 / 255 - 1, 1.0 / 255 - 1])          # clamps, a .5 tie
    src.view(-1)[:min(6, src.numel())] = edge[:min(6, src.numel())]
    png = ((src / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8)                   # the sampler's PNG write
    return src.cuda(), (png.float() / 255).cuda()


def replay_fid_input(lib, g, name, args, rep):
    """dp_fid_input: the source read (u8, fp32, fp32 through the PNG quantisation) is exact, checked with the resize off into a second
    buffer; without resize the output is exact, with resize it is held to bilinear_ref's bound.  Normalisation 2 v - 1 is one more
    rounding.  The pad channel of a pitch-4 pixel row (outside the written view) keeps its sentinel; the amax slot holds max|written|."""
    _, u8, q, N, Hs, Ws, out_p, ld, Ho, Wo, resize, norm, amax = args
    src, val = _source(g, u8, q, N, Hs, Ws)
    tag = f"u8 {u8} quantize {q} N {N} {Hs}x{Ws} -> {Ho}x{Wo} resize {resize} normalize {norm} ld {ld}"
    if resize:       # the value read, exact (the resize and normalisation off)
        raw = Buf(out_p, N * Hs * Ws, ld, 3)
        assert lib.dp_fid_input(src.data_ptr(), u8, q, N, Hs, Ws, raw.ptr, ld, Hs, Ws, 0, 0, None, S()) == 0
        assert raw.outside_untouched(), name
        _exact(rep, name, raw.v, _nhwc_rows(val), tag + " source read")
    out = Buf(out_p, N * Ho * Wo, ld, 3)
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if amax else None

    def reset():
        out.t.fill_(SENT)
        if so is not None:
            so.zero_()

    def run():
        assert lib.dp_fid_input(src.data_ptr(), u8, q, N, Hs, Ws, out.ptr, ld, Ho, Wo, resize, norm,
                                so.data_ptr() if so is not None else None, S()) == 0
    got, = _twice(run, reset, [out.v])
    assert out.outside_untouched(), f"{name} {tag}: the pad channel / sentinels changed"
    if not resize:
        _exact(rep, name, got, _nhwc_rows(2 * val - 1 if norm else val), tag)
    else:
        ref, bound = lc.bilinear_ref(val.double(), Ho, Wo)
        if norm:
            ref = 2 * ref - 1
            bound = 2 * bound + 2 * lc.U * ref.abs()
        _check(rep, name, got, _nhwc_rows(ref), _nhwc_rows(bound), tag)
    if so is not None:
        assert _slot_value(so) == float(got.abs().max()), name


def replay_pool(lib, g, name, args, rep):
    """dp_pool3x3: max exact; average (padding not counted) within avgpool_ref's bound; amax slot exact."""
    xp, ldx, yp, ldy, N, H, W, Cc, stride, pad, mode, amax = args
    P, Q = (H + 2 * pad - 3) // stride + 1, (W + 2 * pad - 3) // stride + 1
    x = Buf(xp, N * H * W, ldx, Cc, FAR)
    x.v.copy_(_scaled(g, N * H * W, Cc))
    y = Buf(yp, N * P * Q, ldy, Cc)
    so = torch.zeros(1, dtype=torch.int32, device="cuda") if amax else None

    def reset():
        y.t.fill_(SENT)
        if so is not None:
            so.zero_()

    def run():
        assert lib.dp_pool3x3(x.ptr, ldx, y.ptr, ldy, N, H, W, Cc, stride, pad, mode, so.data_ptr() if so is not None else None, S()) == 0
    got, = _twice(run, reset, [y.v])
    assert y.outside_untouched(), name
    x64 = _nchw(x.v, N, H, W)
    tag = f"{'max' if mode == 0 else 'avg'} N {N} {H}x{W}x{Cc} stride {stride} pad {pad}"
    if mode == 0:
        _exact(rep, name, got.double(), _nhwc_rows(F.max_pool2d(x64, 3, stride, pad)), tag)
    else:
        ref, bound = lc.avgpool_ref(x64, stride, pad)
        _check(rep, name, got, _nhwc_rows(ref), _nhwc_rows(bound), tag)
    if so is not None:
        assert _slot_value(so) == float(got.abs().max()), name


def replay_global_mean(lib, g, name, args, rep):
    """dp_global_mean (the pooled features, and the moments' shift as one image of rows x 1 pixels): global_mean_ref's bound."""
    xp, ldx, yp, ldy, N, H, W, Cc = args
    x = Buf(xp, N * H * W, ldx, Cc, FAR)
    x.v.copy_(_scaled(g, N * H * W, Cc).abs_() + 0.25)         # post-ReLU features: non-negative
    y = Buf(yp, N, ldy, Cc)

    def run():
        assert lib.dp_global_mean(x.ptr, ldx, y.ptr, ldy, N, H, W, Cc, S()) == 0
    got, = _twice(run, lambda: y.t.fill_(SENT), [y.v])
    assert y.outside_untouched(), name
    ref, bound = lc.global_mean_ref(_nchw(x.v, N, H, W))
    _check(rep, name, got, ref, bound, f"N {N} {H}x{W}x{Cc}")


def _moments_run(lib, f, ld, rows, D, shift, s, sxx):
    assert lib.dp_feature_moments(f, ld, rows, D, shift.data_ptr() if shift is not None else None, s.data_ptr(), sxx.data_ptr(), S()) == 0


def replay_moments(lib, g, name, args, rep):
    """dp_feature_moments accumulating (+=) into non-zero sum / sxx, with the captured shift and without one: moments_ref's bound on
    the sum and the upper triangle of sxx; the strict lower triangle is never written."""
    fp, ld, rows, D = args[:4]
    f = Buf(fp, rows, ld, D, FAR)
    f.v.copy_(torch.randn(rows, D, generator=g).relu_().mul_(2).add_(0.5).cuda())
    iu = torch.triu(torch.ones(D, D, dtype=torch.bool, device="cuda"))
    for shift in (f.v.mean(0), None):
        s0 = torch.randn(D, generator=g, dtype=torch.float64).cuda()
        sxx0 = torch.randn(D, D, generator=g, dtype=torch.float64).cuda()
        s, sxx = s0.clone(), sxx0.clone()

        def reset():
            s.copy_(s0)
            sxx.copy_(sxx0)
        got_s, got_x = _twice(lambda: _moments_run(lib, f.ptr, ld, rows, D, shift, s, sxx), reset, [s, sxx])
        tag = f"rows {rows} D {D} ld {ld} shift {shift is not None}"
        assert torch.equal(got_x[~iu], sxx0[~iu]), f"{name} {tag}: the strict lower triangle of sxx changed"
        rs, bs, rx, bx = lc.moments_ref(f.v, shift, s0, sxx0)
        _check(rep, name, got_s, rs, bs, tag + " sum")
        _check(rep, name, got_x[iu], rx[iu], bx[iu], tag + " sxx")


def replay_ddim(lib, g, name, args, rep):
    """dp_ddim_step at the captured length and fp32 coefficients, with a sixteenth of the outputs placed so that x0 straddles +-clip:
    ddim_step_ref's bound; nothing past the n outputs is written."""
    _, _, nzp, op, n, sb, sa, clip, sap, dirc, sigma = args
    x, e = _randn(g, n), _randn(g, n)
    k = n // 16
    if clip > 0 and k:
        side = torch.where(torch.rand(k, generator=g) < 0.5, -clip, clip) * (1 + (torch.rand(k, generator=g) - 0.5) * 2.0 ** -18)
        x[:k] = sa * side.cuda() + sb * e[:k]
    nz = _randn(g, n) if nzp else None
    out = Buf(op, n, 1, 1)

    def run():
        assert lib.dp_ddim_step(x.data_ptr(), e.data_ptr(), nz.data_ptr() if nz is not None else None, out.ptr, n, sb, sa, clip, sap,
                                dirc, sigma, S()) == 0
    got, = _twice(run, lambda: out.t.fill_(SENT), [out.v])
    assert out.outside_untouched(), name
    ref, bound = lc.ddim_step_ref(x, e, nz, sb, sa, clip, sap, dirc, sigma)
    _check(rep, name, got.view(-1), ref, bound, f"n {n} sqrt(alpha_t) {sa:.4g} clip {clip} sigma {sigma:.3g}")


EVAL_REPLAY = dict(REPLAY)
EVAL_REPLAY.update({
    "dp_conv2d_fprop": replay_eval_conv, "dp_fid_input": replay_fid_input, "dp_pool3x3": replay_pool,
    "dp_global_mean": replay_global_mean, "dp_feature_moments": replay_moments, "dp_ddim_step": replay_ddim,
    # already exact replays of the training census; listed here because the evaluation plans must reach them
    "dp_zero_u32": replay_exact, "dp_nchw_to_nhwc": replay_exact, "dp_nhwc_to_nchw": replay_exact, "dp_pack_conv_weight": replay_exact,
    "dp_pack_conv_weight_tc": replay_split,
})


# ---------------------------------------------------------------------------------------------------------------------- plans
def _seeded_inception():
    from test_fid_gpu import seeded_model
    return seeded_model((0, 1, 2, 3))


def _fid_pass(batch, src, hw, quantize):
    """One FeaturePlan built and run eagerly (weights packed, input loaded), then the moments of its pool3 features added as the FID
    statistics add every batch."""
    from diff_pruning_b200 import fid
    model = _seeded_inception()
    g = torch.Generator().manual_seed(13)
    x = (torch.randint(0, 256, (batch, hw[0], hw[1], 3), generator=g, dtype=torch.uint8) if src == "u8" else
         torch.randn(batch, 3, hw[0], hw[1], generator=g) * 0.6).cuda()
    info = {}

    def run():
        plan = fid.FeaturePlan(model, batch, src, hw, quantize=quantize, use_graph=False)
        plan.load(x)
        plan.ensure_packed()
        plan.run_eager()
        fid.Moments(2048).add(plan.feat[3])
        info["convs"] = {(a.C, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l, a.H, a.W) for a in plan.conv_args}
        info["n_convs"] = len(plan.conv_args)
    return run, info


def _ddim_pass(pruned, eta):
    """DDIMPipeline, eager (no graph), 2 uniform steps (t = 999, then t = 0 onto the final alpha 1) at batch 128."""
    import diff_pruning_b200 as dp
    from diff_pruning_b200.sampling import DDIMPipeline
    if pruned:
        from test_unet_gpu import _pruned_c1
        m = _pruned_c1().eval()
    else:
        torch.manual_seed(0)
        m = dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval().cuda()

    def run():
        pipe = DDIMPipeline(unet=m, scheduler=dp.DDPMScheduler(num_train_timesteps=1000))
        pipe.use_graph = False
        pipe(batch_size=128, generator=torch.Generator(device="cuda").manual_seed(0), eta=eta, num_inference_steps=2, output_type="device")
    return run, {}


FID_KINDS = {"dp_conv2d_fprop", "dp_fid_input", "dp_pool3x3", "dp_global_mean", "dp_feature_moments", "dp_zero_u32",
             "dp_pack_conv_weight", "dp_pack_conv_weight_tc"}
DDIM_KINDS = {"dp_conv2d_fprop", "dp_ddim_step", "dp_nchw_to_nhwc", "dp_nhwc_to_nchw"}
CONFIGS = {
    "FID u8 b50 32px": (lambda: _fid_pass(50, "u8", (32, 32), False), FID_KINDS),
    "FID f32q b128 32px": (lambda: _fid_pass(128, "f32", (32, 32), True), FID_KINDS),
    "FID u8 b50 256px": (lambda: _fid_pass(50, "u8", (256, 256), False), FID_KINDS),
    "DDIM C1 b128": (lambda: _ddim_pass(False, 0.0), DDIM_KINDS),
    "DDIM pruned C1 b128 eta0.5": (lambda: _ddim_pass(True, 0.5), DDIM_KINDS),
}


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_eval_census(lib, tag):
    make, must = CONFIGS[tag]
    run, info = make()
    _LOG.clear()
    _LOG.update(geoms=set(), tc=[], simt=set())
    calls = _capture(lib, run)
    del run
    gc.collect()              # the plan and its model form a reference cycle
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert must <= kinds, f"{tag}: the plan no longer issues {sorted(must - kinds)}"
    missing = kinds - set(EVAL_REPLAY)
    assert not missing, f"{tag}: launch kinds without a replay: {sorted(missing)}"
    uniq = _unique(calls)
    rep, count, failures = {}, {}, []
    g = torch.Generator().manual_seed(2025)
    for name, args in uniq:
        count[name] = count.get(name, 0) + 1
        try:
            EVAL_REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:          # report every failing launch of the config, not just the first
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print(f"  FAIL {tag}: {f}")
    assert not failures, f"{tag}: {len(failures)} launches failed their checks"
    assert set(rep) == kinds, (tag, sorted(kinds - set(rep)))     # every kind the plan issued was checked
    print(f"\n{tag}: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds, all replayed")
    for name in sorted(rep):
        print(f"  {tag:28s} {name:26s} {count[name]:4d} unique, worst err/bound {max(rep[name]):.3f}")
    if "convs" in info:
        # every convolution of the Inception pass, stem through Mixed_7c, was replayed at its geometry
        assert info["n_convs"] == 94 and info["convs"] <= _LOG["geoms"], sorted(info["convs"] - _LOG["geoms"])
        Ls = sorted({L_ for L_, _, _ in _LOG["tc"]})
        split = sorted({(geom, ks) for _, ks, geom in _LOG["tc"] if ks > 1})
        assert _LOG["tc"] and max(Ls) <= lc.L_MAX and _LOG["simt"] == {27}
        print(f"  tensor-core launches: {len(_LOG['tc'])}, L in {Ls}; K split in {split}; SIMT (C = 3 stem): L = {sorted(_LOG['simt'])}")


# ---------------------------------------------------------------------------------------------------------------- directed edges
@pytest.mark.parametrize("n", [1, 255, 257, 3 * 132 * 32 * 256 + 5])
def test_ddim_step_edges(lib, n):
    """dp_ddim_step at lengths around one block and beyond three sweeps of the grid-stride loop, at t = 999 (division by
    sqrt(alpha_bar) ~ 0.0064) and t = 0 (final alpha 1, where eta gives sigma = 0), eta 0 and 1, clip on and off, x0 straddling +-1."""
    from diff_pruning_b200.sampling import DDIMScheduler
    sch = DDIMScheduler()
    sch.set_timesteps(10)
    rep = {}
    g = torch.Generator().manual_seed(n % 1000)
    for t in (999, 0):
        for eta in (0.0, 1.0):
            sb, sa, sap, dirc, sigma = sch._coefficients(t, eta)
            for clip in (1.0, 0.0):
                replay_ddim(lib, g, "dp_ddim_step", [0, 0, 0x1000 if eta else 0, 0x2004, n, sb, sa, clip, sap, dirc, sigma], rep)
    print(f"\nn {n}: worst err/bound {max(rep['dp_ddim_step']):.3f}")


@pytest.mark.parametrize("case", [
    # (u8, quantize, N, Hs, Ws, Ho, Wo, resize, normalize, ld, 16-byte phase of the output)
    (1, 0, 2, 512, 384, 299, 299, 1, 1, 4, 0),          # downscale, non-square source
    (0, 1, 3, 48, 40, 299, 299, 1, 1, 4, 0),            # DDIM samples through the PNG rule, non-square
    (1, 0, 2, 1, 1, 299, 299, 1, 1, 4, 0),              # a 1 x 1 source
    (0, 0, 2, 37, 53, 299, 299, 1, 0, 7, 1),            # fp32 [0, 1] as the module forward passes it, odd pitch and phase
    (1, 0, 2, 20, 24, 20, 24, 0, 1, 4, 0),              # no resize: exact
    (0, 1, 2, 20, 24, 20, 24, 0, 0, 4, 0),              # no resize, no normalisation: the PNG values themselves
])
def test_fid_input_edges(lib, case):
    u8, q, N, Hs, Ws, Ho, Wo, resize, norm, ld, phase = case
    rep = {}
    replay_fid_input(lib, torch.Generator().manual_seed(sum(case)), "dp_fid_input",
                     [0, u8, q, N, Hs, Ws, 0x1000 + 4 * phase, ld, Ho, Wo, resize, norm, 0x2000], rep)
    print(f"\n{case}: worst err/bound {max(rep['dp_fid_input']):.3f}")
    # in the plan's own pitch-4 buffer the pad channel stays 0
    src, _ = _source(torch.Generator().manual_seed(1), u8, q, N, Hs, Ws)
    out = torch.zeros(N, Ho, Wo, 4, device="cuda")
    assert lib.dp_fid_input(src.data_ptr(), u8, q, N, Hs, Ws, out.data_ptr(), 4, Ho, Wo, resize, norm, None, S()) == 0
    assert torch.equal(out[..., 3], torch.zeros_like(out[..., 3]))


@pytest.mark.parametrize("D", [64, 192, 768, 2048])
@pytest.mark.parametrize("rows", [1, 31, 33, 50])
def test_feature_moments_edges(lib, D, rows):
    """dp_feature_moments at the four FID feature widths, row counts around the kernel's 32-row step, a pitch wider than D; and two
    calls over a split of the rows accumulate to one call over all of them, within the bound (the split call chain has at most twice
    its updates)."""
    rep = {}
    g = torch.Generator().manual_seed(D + rows)
    replay_moments(lib, g, "dp_feature_moments", [0x1000, D + 3, rows, D], rep)
    f = torch.randn(rows, D + 3, generator=g).relu_().add_(0.5).cuda()
    shift = f[:, :D].mean(0)
    s0 = torch.randn(D, generator=g, dtype=torch.float64).cuda()
    sxx0 = torch.randn(D, D, generator=g, dtype=torch.float64).cuda()
    one, two = (s0.clone(), sxx0.clone()), (s0.clone(), sxx0.clone())
    _moments_run(lib, f.data_ptr(), D + 3, rows, D, shift, *one)
    a = rows // 2
    _moments_run(lib, f.data_ptr(), D + 3, a, D, shift, *two)
    _moments_run(lib, f[a:].data_ptr(), D + 3, rows - a, D, shift, *two)
    rs, bs, rx, bx = lc.moments_ref(f[:, :D], shift, s0, sxx0)
    iu = torch.triu(torch.ones(D, D, dtype=torch.bool, device="cuda"))
    for got, ref, b, what in ((one[0], rs, bs, "sum"), (one[1][iu], rx[iu], bx[iu], "sxx")):
        _check(rep, "one call", got, ref, b, what)
    for got, ref, b, what in ((two[0], rs, 2 * bs, "sum"), (two[1][iu], rx[iu], 2 * bx[iu], "sxx")):
        _check(rep, "two calls", got, ref, b, what)
    print(f"\nD {D} rows {rows}: worst err/bound {max(max(v) for v in rep.values()):.3f}")


@pytest.mark.parametrize("hw", [(73, 73), (35, 35), (8, 8)])
def test_global_mean_of_non_negative_maps(lib, hw):
    """Post-ReLU maps, all terms of one sign, at the extents whose means are FID features: within global_mean_ref's bound, which a
    running fp32 sum of the H W terms exceeds (about sqrt(H W) ulps)."""
    H, W = hw
    rep = {}
    replay_global_mean(lib, torch.Generator().manual_seed(H), "dp_global_mean", [0x1000, 70, 0x2004, 66, 3, H, W, 64], rep)
    print(f"\n{H}x{W}: worst err/bound {max(rep['dp_global_mean']):.3f}")


# ---------------------------------------------------------------------------------------------------------------- end to end
def _pool3_error(plan, x, ref):
    plan.load(x)
    plan.run()
    feat = plan.feat[3].double()
    return ((feat - ref).abs().amax(1) / ref.abs().amax(1)).cpu()


def test_pool3_features_at_batch_128_match_fp64_oracle():
    """statistics_of_pipeline's plan (batch 128, DDIM samples through the PNG quantisation, 32 x 32 -> 299) against the Inception
    oracle in float64 on the device, same state dict, conv -> BN -> ReLU unfolded, fed the PNG values resized by torch's fp32 source
    rule: the pool3 features of every image, relative to that image's largest feature.  This covers what the replays cannot: the
    wiring, the channel offsets of the concatenations and the amax slots that concatenated branches share.

    Measured on an H100 80GB HBM3: the tensor-core plan 2.46e-5 (worst image; the median image 2.42e-5), the exact-fp32 SIMT plan
    5.3e-7.  Every tensor-core launch is within its census bound; the gap is the wgmma accumulator's truncating rounding, whose error
    has the sign of the partial sum (up to 253 updates per output here) and so adds up coherently over the 45 layers rather than
    averaging out, which is why every image shows about the same error.  The tensor-core plan is held to 5e-5, twice the measured
    value (a wiring or offset error is O(1); the golden test against the reference's fp32 CPU features allows 1e-4), and the SIMT plan
    to 2e-6, which shows the oracle comparison itself resolves far below that."""
    from oracle import inception_oracle as orc
    from diff_pruning_b200 import fid
    model = _seeded_inception()
    sd = {k: v.detach().to("cuda", torch.float64) for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")}
    xc = torch.randn(128, 3, 32, 32, generator=torch.Generator().manual_seed(12)) * 0.6
    q = ((xc / 2 + 0.5).clamp(0, 1) * 255).round() / 255                    # the PNG values the plan reads (host division: exact)
    x_in = 2 * lc.bilinear_ref(q.double().cuda(), 299, 299)[0] - 1
    with torch.no_grad():
        ref = torch.cat([orc.forward(sd, x_in[i:i + 32], (3,), resize_input=False, normalize_input=False)[0].flatten(1)
                         for i in range(0, 128, 32)])
    x = xc.cuda()
    tc = _pool3_error(fid.FeaturePlan(model, 128, "f32", (32, 32), quantize=True, use_graph=False), x, ref)
    gc.collect()
    simt = _pool3_error(fid.FeaturePlan(model, 128, "f32", (32, 32), quantize=True, use_graph=False, force_simt=True), x, ref)
    for what, per in (("tensor-core plan", tc), ("exact-fp32 SIMT plan", simt)):
        print(f"\npool3 features, batch 128, {what}: max-rel per image worst {float(per.max()):.3g}, median {float(per.median()):.3g}")
    assert math.isfinite(float(tc.max())) and float(tc.max()) <= 5e-5
    assert math.isfinite(float(simt.max())) and float(simt.max()) <= 2e-6
