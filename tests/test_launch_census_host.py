"""The checker of the launch census (launch_census.py) on the host: its element-wise bound rejects the kernel variants it must reject,
reports a planted error where it is, and its dedup key never merges launches that differ in a keyed field."""
import ctypes as C

import torch
import torch.nn.functional as F

import launch_census as lc
from diff_pruning_b200 import _lib as L
from diff_pruning_b200 import engine


def _census_chains():
    """Chain lengths the census meets: a C1 128 -> 128 3x3 fprop, the C1 256 -> 128 3x3 weight gradient at 32x32 and batch 128 with
    the engine's own split count (its longest), and L_MAX, the longest chain any tensor-core launch of the census may have."""
    tiles, rows = 18, 128 * 32 * 32
    sp = engine._wgrad_splits(tiles, rows // 64)
    return {"fprop 128->128 3x3": lc.chain_fprop(9, 128), "wgrad 256->128 3x3 @32x32 b128": lc.chain_wgrad(lc.wgrad_pixels_per_cta(rows, sp), sp),
            "L_MAX": lc.L_MAX}


def test_bound_rejects_one_and_two_product_variants():
    """hi*hi alone (what a plain single-pass fp16 / TF32 kernel computes) and hi*hi + hi*lo' (the split with one correction term
    dropped) violate the bound on most outputs of a realistic convolution at census chain lengths, even with their sums taken
    exactly; the full three-product split passes."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 128, 16, 16, generator=g, dtype=torch.float64).float().double()
    x = x * 2.0 ** (torch.rand(1, 128, 1, 1, generator=g, dtype=torch.float64) * 12 - 6).floor()     # per-channel scales 2^U(-6, 6)
    w = (torch.randn(128, 128, 3, 3, generator=g, dtype=torch.float64) / 34).float().double()
    exact = F.conv2d(x, w, padding=1)
    s = F.conv2d(x * x, w * w, padding=1).sqrt()
    xh, xl, sx = lc.split_h(x)
    wh, wl, sw = lc.split_h(w)
    conv = lambda a, b: F.conv2d(a, b, padding=1) / (sx * sw)
    one = conv(xh, wh)
    two = one + conv(xh, wl) / 2048
    three = two + conv(xl, wh) / 2048
    for tag, L_ in _census_chains().items():
        bound = lc.product_bound(s, L_)
        for name, y in (("hi*hi", one), ("hi*hi + hi*lo'", two)):
            frac = float(((y - exact).abs() > bound).double().mean())
            print(f"{tag}: L = {L_}, {name} violates on {frac:.1%} of the outputs")
            assert frac > 0.5, (tag, name, frac)
        worst, where = lc.violations(three, exact, bound)
        assert not where and worst < 0.25, (tag, worst)


def test_truncating_accumulator_stays_within_the_bound():
    """The complete split with the fp32 accumulator truncating after every 16-deep block (the tensor core's rounding), emulated at the
    census' chain lengths: within (ALPHA + BETA L) 2^-24 s on every output, and using a real part of it (the bound is not slack)."""
    g = torch.Generator().manual_seed(4)
    for L_ in sorted(set(_census_chains().values())):
        M, n = 512, 16 * L_
        a = torch.randn(M, n, generator=g).double()
        b = (torch.randn(M, n, generator=g) * 2.0 ** (torch.rand(1, n, generator=g) * 12 - 6)).double()
        ah, al, sa = lc.split_h(a)
        bh, bl, sb = lc.split_h(b)
        main, corr = (ah * bh).view(M, L_, 16).sum(-1), ((ah * bl + al * bh) / 2048).view(M, L_, 16).sum(-1)
        acc = torch.zeros(M, dtype=torch.float64)
        cor = torch.zeros(M, dtype=torch.float64)
        for j in range(L_):
            acc, cor = _trunc32(acc + main[:, j]), _trunc32(cor + corr[:, j])
        y = (acc + cor).float().double() / (sa * sb)
        exact, s = (a * b).sum(1), ((a * b) ** 2).sum(1).sqrt()
        worst, where = lc.violations(y, exact, lc.product_bound(s, L_))
        print(f"L = {L_}: worst err / bound {worst:.3f}")
        assert not where and 0.1 < worst < 1.0, (L_, worst)


def _trunc32(v: torch.Tensor) -> torch.Tensor:
    """Round float64 values to fp32 toward zero."""
    f = v.float()
    over = f.double().abs() > v.abs()
    f[over] = torch.nextafter(f[over], torch.zeros_like(f[over]))
    return f.double()


def test_planted_error_is_reported_at_its_coordinates():
    g = torch.Generator().manual_seed(5)
    ref = torch.randn(3, 7, 9, 11, generator=g, dtype=torch.float64)
    s = ref.abs() + 1
    bound = lc.product_bound(s, 100)
    got = (ref + (torch.rand(ref.shape, generator=g, dtype=torch.float64) - 0.5) * bound).clone()    # within the bound everywhere
    worst, where = lc.violations(got, ref, bound)
    assert not where and worst <= 0.5
    got[2, 5, 0, 10] = ref[2, 5, 0, 10] + 2 * bound[2, 5, 0, 10]
    worst, where = lc.violations(got, ref, bound)
    assert where == [(2, 5, 0, 10)] and 1.9 < worst < 2.1
    got[1, 1, 1, 1] = float("nan")
    worst, where = lc.violations(got, ref, bound)
    assert where == [(1, 1, 1, 1), (2, 5, 0, 10)] and worst == float("inf")


def test_dedup_key_separates_every_keyed_field():
    base = L.ConvArgs()
    for name, t in base._fields_:
        setattr(base, name, 0x7F0000001000 if t is C.c_void_p else 3)
    kinds = lc.argkinds("dp_conv2d_fprop")
    k0 = lc.launch_key("dp_conv2d_fprop", kinds, [base])
    assert lc.launch_key("dp_conv2d_dgrad", lc.argkinds("dp_conv2d_dgrad"), [base]) != k0
    for name, t in base._fields_:
        a = engine._copy_args(base)
        if t is C.c_void_p:
            for v in (None, 0x7F0000001004, 0x7F0000001008, 0x7F000000100C):      # NULL, and each 16-byte phase of a view
                setattr(a, name, v)
                assert lc.launch_key("dp_conv2d_fprop", kinds, [a]) != k0, (name, v)
            setattr(a, name, 0x7F0000002000)                                       # same phase, another buffer: one launch
            assert lc.launch_key("dp_conv2d_fprop", kinds, [a]) == k0, name
        else:
            setattr(a, name, 4)
            assert lc.launch_key("dp_conv2d_fprop", kinds, [a]) != k0, name
    # bf16 operands: views 2 bytes apart are different launches
    b = L.ConvBf16Args()
    b.x_bf16 = 0x7F0000001000
    kb = lc.argkinds("dp_conv2d_fprop_bf16")
    k1 = lc.launch_key("dp_conv2d_fprop_bf16", kb, [b])
    b.x_bf16 = 0x7F0000001002
    assert lc.launch_key("dp_conv2d_fprop_bf16", kb, [b]) != k1
    # plain-argument entry points: dp_amax(x, ld, rows, cols, slot)
    kinds = lc.argkinds("dp_amax")
    assert kinds == ["p", "i", "i", "i", "p"]
    args = [0x1000, 64, 128, 60, 0x2000]
    k0 = lc.launch_key("dp_amax", kinds, args)
    for i, v in enumerate((0x1004, 68, 129, 61, None)):
        a = list(args)
        a[i] = v
        assert lc.launch_key("dp_amax", kinds, a) != k0, i


# ---------------------------------------------------------------------------------------------------- evaluation path (FID, DDIM)
def _inception_convs():
    """(C, K, R, S, stride, pad_t, pad_l, H, W) of every convolution of the FID Inception pass on its 299 x 299 input, stem through
    Mixed_7c, with the extents fid.FeaturePlan gives them."""
    from diff_pruning_b200 import fid
    out, H, W = [], 299, 299
    size = lambda h, w, k, s, p: ((h + 2 * p[0] - k[0]) // s + 1, (w + 2 * p[1] - k[1]) // s + 1)
    for _, _, layer in fid.LAYERS:
        if layer[0] == "conv":
            _, cin, cout, k, s, p = layer
            out.append((cin, cout, k[0], k[1], s, p[0], p[1], H, W))
            H, W = size(H, W, k, s, p)
        elif layer[0] == "maxpool":
            H, W = size(H, W, (3, 3), 2, (0, 0))
        elif layer[0] == "mixed":
            _, cin, spec = layer
            _, ps, pp = spec["pool"]
            ext, width = {"x": (H, W), "pool": size(H, W, (3, 3), ps, (pp, pp))}, {"x": cin, "pool": cin}
            for name, src, cout, k, s, p in spec["convs"]:
                out.append((width[src], cout, k[0], k[1], s, p[0], p[1]) + ext[src])
                ext[name], width[name] = size(*ext[src], k, s, p), cout
            H, W = ext[spec["out"][0]]
    return out


def test_general_split_count_follows_the_kernel_rule():
    """launch_census.general_split restates conv_tc.cu's pick_ksplit over the general-geometry kernel's tiles and stages: hand-computed
    cases (splits to fill the SMs only where the tiles cover less than half of 132 SMs, capped at 16, at least 4 stages per split; at
    least enough splits that none walks more than MAX_SPLIT_STAGES stages, so that even 16 of them keep the chain within L_MAX; no empty
    split), and on every Inception convolution at batches 50, 128 and 256 the rule's invariants hold and the chain stays within L_MAX."""
    sms = 132
    assert lc.chain_general(16, lc.MAX_SPLIT_STAGES) <= lc.L_MAX
    assert lc.pick_ksplit(1, 100, sms) == (15, 7)        # 16 splits of 7 stages would leave the last one empty
    assert lc.pick_ksplit(4, 9, sms) == (2, 5)
    assert lc.pick_ksplit(66, 8, sms) == (2, 4)
    assert lc.pick_ksplit(67, 100, sms) == (1, 100)      # tiles cover more than half the SMs
    assert lc.pick_ksplit(1, 7, sms) == (1, 7)           # fewer than 8 stages
    assert lc.pick_ksplit(40, 11, sms) == (2, 6)         # 3 SMs per tile, but at least 4 stages per split: 2 splits of 6
    assert lc.pick_ksplit(120, 216, sms) == (2, 108)     # tiles fill the SMs, but 216 stages are longer than one split may walk
    assert lc.pick_ksplit(400, 270, sms) == (2, 135)
    assert lc.pick_ksplit(400, 147, sms) == (1, 147)     # the longest chain that stays whole
    assert lc.pick_ksplit(1, 300, sms) == (16, 19)       # the SM rule already splits further than the chain rule
    convs = _inception_convs()
    assert len(convs) == 94
    geo = {c[:9]: c for c in convs}
    # Mixed_7b / Mixed_7c branch_pool (1x1 over 1280 / 2048 channels at 8x8) and Mixed_7a branch7x7x3_4 (3x3 s2 17 -> 8) split at batch 50
    assert lc.general_split(50, 8, 8, 192, 1280, 1, 1, sms) == (2, 10)
    assert lc.general_split(50, 8, 8, 192, 2048, 1, 1, sms) == (2, 16)
    assert lc.general_split(50, 8, 8, 192, 192, 3, 3, sms) == (2, 14)
    assert lc.general_split(128, 8, 8, 192, 1280, 1, 1, sms) == (1, 20)
    assert lc.general_split(50, 8, 8, 384, 448, 3, 3, sms) == (1, 63)      # the longest chain: 9 taps x 7 stages
    assert lc.general_split(256, 147, 147, 32, 32, 3, 3, sms) == (1, 9)
    assert (448, 384, 3, 3, 1, 1, 1, 8, 8) in geo and (192, 192, 3, 3, 2, 0, 0, 17, 17) in geo
    splits = {}
    for N in (50, 128, 256):
        for C_, K, R, S, st, pt, pl, H, W in convs:
            P, Q = (H + 2 * pt - R) // st + 1, (W + 2 * pl - S) // st + 1
            tiles = -(-(N * P * Q) // 128) * -(-K // 128)
            iters = R * S * -(-C_ // 64)
            ks, ips = lc.general_split(N, P, Q, K, C_, R, S, sms)
            assert 1 <= ks <= 16 and (ks - 1) * ips < iters <= ks * ips
            if ks > 1:
                assert 2 * tiles <= sms and ks * tiles <= sms and ips >= 4
            else:
                assert ips == iters
            assert lc.chain_general(ks, ips) <= lc.L_MAX
            splits[N] = splits.get(N, 0) + (ks > 1)
    print(f"general-geometry launches that split K at batch 50 / 128 / 256: {splits}")
    assert splits[50] > 0 and splits[256] == 0


def _affected_majority(bad: torch.Tensor, affected: torch.Tensor, what: str, need: float = 0.5):
    frac = float(bad[affected].double().mean())
    print(f"{what}: violates the bound on {frac:.1%} of {int(affected.sum())} affected outputs")
    assert int(affected.sum()) > 0 and frac > need, (what, frac)


def _emulate_bilinear_fp32(src32: torch.Tensor, Ho: int, Wo: int) -> torch.Tensor:
    """fid_input_kernel's resize in fp32 on the host (no contraction): the kernel's own arithmetic, as the bound must admit it."""
    h0, h1, a0, a1, _ = lc.bilinear_coords(src32.shape[2], Ho)
    w0, w1, b0, b1, _ = lc.bilinear_coords(src32.shape[3], Wo)
    A0, A1, B0, B1 = a0.float().view(-1, 1), a1.float().view(-1, 1), b0.float().view(1, -1), b1.float().view(1, -1)
    r0, r1 = src32[:, :, h0], src32[:, :, h1]
    return A0 * (B0 * r0[..., w0] + B1 * r0[..., w1]) + A1 * (B0 * r1[..., w0] + B1 * r1[..., w1])


def test_bilinear_bound_rejects_corner_alignment_and_dropped_half_pixel():
    """On seeded u8 images (32 x 32 -> 299, 48 x 40 -> 299 x 299, 512 x 384 -> 299 x 299) the fp32 restatement of the kernel stays
    within bilinear_ref's bound, while align_corners=True and the rule without the half-pixel offset violate it on most of the outputs
    whose source position they move."""
    g = torch.Generator().manual_seed(6)
    for Hs, Ws in ((32, 32), (48, 40), (512, 384)):
        src = (torch.randint(0, 256, (2, 3, Hs, Ws), generator=g).float() / 255)
        ref, bound = lc.bilinear_ref(src.double(), 299, 299)
        worst, where = lc.violations(_emulate_bilinear_fp32(src, 299, 299), ref, bound)
        assert not where and worst < 0.5, (Hs, Ws, worst)
        # align_corners=True: r = dst (n_src - 1) / (n_dst - 1)
        ac = F.interpolate(src.double(), size=(299, 299), mode="bilinear", align_corners=True)
        rh = torch.arange(299, dtype=torch.float64) * (Hs - 1) / 298
        rw = torch.arange(299, dtype=torch.float64) * (Ws - 1) / 298
        th = (torch.arange(299, dtype=torch.float64) + 0.5) * Hs / 299 - 0.5
        tw = (torch.arange(299, dtype=torch.float64) + 0.5) * Ws / 299 - 0.5
        moved = lambda a, b: (a - b.clamp_min(0)).abs() > 1e-3
        aff = moved(rh, th).view(-1, 1) | moved(rw, tw).view(1, -1)
        _affected_majority((ac - ref).abs() > bound, aff.expand_as(ref), f"{Hs}x{Ws} align_corners=True")
        # the half-pixel offset dropped: r = scale dst
        nh, _ = lc.bilinear_ref(src.double(), 299, 299, half_pixel=False)
        aff = moved(torch.arange(299, dtype=torch.float64) * Hs / 299, th).view(-1, 1) | \
            moved(torch.arange(299, dtype=torch.float64) * Ws / 299, tw).view(1, -1)
        _affected_majority((nh - ref).abs() > bound, aff.expand_as(ref), f"{Hs}x{Ws} no half-pixel offset")


def test_avgpool_bound_rejects_counting_padding():
    """3 x 3 / stride 1 / pad 1 average pool: a fixed-order fp32 sum of the taps over the taps inside the image passes avgpool_ref's
    bound; dividing by 9 on the border (count_include_pad=True) violates it on most border outputs."""
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 8, 17, 15, generator=g).float()
    ref, bound = lc.avgpool_ref(x.double(), 1, 1)
    cols = F.unfold(F.pad(x, (1, 1, 1, 1)), 3).view(2, 8, 9, 17, 15)           # padded zeros add nothing to an fp32 sum
    acc = torch.zeros(2, 8, 17, 15)
    for k in range(9):
        acc = acc + cols[:, :, k]
    n = (F.avg_pool2d(torch.ones(1, 1, 17, 15, dtype=torch.float64), 3, 1, 1, count_include_pad=True) * 9).float()
    worst, where = lc.violations(acc / n, ref, bound)
    assert not where and worst < 0.5, worst
    inc = F.avg_pool2d(x.double(), 3, 1, 1, count_include_pad=True)
    border = (n < 9).expand_as(ref)
    _affected_majority((inc - ref).abs() > bound, border, "avg pool counting padding")


def test_moments_bound_rejects_fp32_accumulation():
    """dp_feature_moments' accumulation emulated in fp64 (one row at a time, product then sum) stays within moments_ref's bound, onto
    non-zero old values; the same sums formed in fp32 violate it on most elements of the upper triangle and of the sum."""
    g = torch.Generator().manual_seed(8)
    for rows in (1, 33, 50):
        D = 64
        f = (torch.relu(torch.randn(rows, D, generator=g)) * 3 + 0.2).float()
        shift = f.mean(0).float()
        s0, sxx0 = torch.randn(D, generator=g, dtype=torch.float64), torch.randn(D, D, generator=g, dtype=torch.float64)
        rs, bs, rx, bx = lc.moments_ref(f, shift, s0, sxx0)
        d = f.double() - shift.double()
        acc, sacc = torch.zeros(D, D, dtype=torch.float64), torch.zeros(D, dtype=torch.float64)
        for r in range(rows):
            acc = acc + d[r][:, None] * d[r][None, :]
            sacc = sacc + d[r]
        iu = torch.triu(torch.ones(D, D, dtype=torch.bool))
        worst, where = lc.violations((sxx0 + acc)[iu], rx[iu], bx[iu])
        assert not where and worst < 0.5, (rows, worst)
        worst, where = lc.violations(s0 + sacc, rs, bs)
        assert not where and worst < 0.5, (rows, worst)
        d32 = f - shift
        x32 = (sxx0.float() + d32.T @ d32).double()
        s32 = (s0.float() + d32.sum(0)).double()
        _affected_majority((x32 - rx).abs() > bx, iu, f"rows {rows}: sxx accumulated in fp32")
        _affected_majority((s32 - rs).abs() > bs, torch.ones(D, dtype=torch.bool), f"rows {rows}: sum accumulated in fp32")


def _ddim_coefficients(t: int, eta: float, steps: int = 10):
    from diff_pruning_b200.sampling import DDIMScheduler
    sch = DDIMScheduler()
    sch.set_timesteps(steps)
    return sch._coefficients(t, eta)


def test_ddim_bound_rejects_a_step_without_the_clip():
    """At t = 999 (division by sqrt(alpha_bar) ~ 0.0064) and t = 0 (final alpha 1) the DDIM update evaluated in fp32 stays within
    ddim_step_ref's bound; the same update without the clip of x0 violates it on most outputs whose x0 lies beyond +-1."""
    g = torch.Generator().manual_seed(9)
    for t, eta in ((999, 0.0), (999, 1.0), (0, 0.0)):
        sb, sa, sap, dirc, sigma = _ddim_coefficients(t, eta)
        x, e, nz = (torch.randn(4096, generator=g) for _ in range(3))
        ref, bound = lc.ddim_step_ref(x, e, nz, sb, sa, 1.0, sap, dirc, sigma)
        f = lambda v: torch.tensor(v, dtype=torch.float32)
        x0 = ((x - f(sb) * e) / f(sa)).clamp(-1, 1)
        got = f(sap) * x0 + f(dirc) * e + f(sigma) * nz
        worst, where = lc.violations(got, ref, bound)
        assert not where and worst < 0.5, (t, eta, worst)
        raw = (x.double() - sb * e.double()) / sa
        noclip = sap * raw + dirc * e.double() + sigma * nz.double()
        _affected_majority((noclip - ref).abs() > bound, raw.abs() > 1.0, f"t {t} eta {eta}: no clip")


def test_global_mean_bound_rejects_a_running_fp32_sum():
    """Post-ReLU 73 x 73 maps (all terms of one sign): the mean of an fp64 sum rounded once to fp32 is within global_mean_ref's bound; a
    running fp32 sum over the 5329 terms violates it on most channels."""
    g = torch.Generator().manual_seed(10)
    x = (torch.randn(2, 16, 73, 73, generator=g).abs() + 0.25).float()
    ref, bound = lc.global_mean_ref(x.double())
    worst, where = lc.violations(ref.float(), ref, bound)
    assert not where and worst <= 0.5, worst
    flat = x.flatten(2)
    acc = torch.zeros(2, 16)
    for k in range(flat.shape[2]):
        acc = acc + flat[:, :, k]
    run32 = acc / 73 / 73
    _affected_majority((run32.double() - ref).abs() > bound, torch.ones_like(ref, dtype=torch.bool), "running fp32 sum over 73 x 73")


def _emulate_softmax_fp32(x: torch.Tensor, lanes_summed: int = 32, dtype=torch.float32) -> torch.Tensor:
    """softmax_fwd_kernel on the host: fp32 z = x - max, exp, per-lane sums of every 32nd term in `dtype`, a butterfly over the first
    `lanes_summed` lanes, p = e * (1 / sum)."""
    rows, cols = x.shape
    z = x - x.amax(-1, keepdim=True)
    e = torch.exp(z)
    acc = torch.zeros(rows, 32, dtype=dtype)
    for k in range(cols // 32):
        acc = acc + e[:, 32 * k:32 * k + 32].to(dtype)
    acc = acc.float()[:, :lanes_summed]
    o = lanes_summed // 2
    while o:
        acc = acc + acc[:, torch.arange(lanes_summed) ^ o]
        o //= 2
    return e * (1.0 / acc[:, :1])


def test_softmax_bound_admits_the_kernel_order_and_rejects_a_lost_lane_or_a_half_precision_sum():
    """softmax_fwd_bound at the 4096 columns of the VQ-f4 attention: the kernel's own order of operations in fp32 stays within it, while
    a butterfly that drops half the lanes, or lane sums kept in fp16, violate it on most rows."""
    x = torch.randn(256, 4096, generator=torch.Generator().manual_seed(5)) * 3
    ref = torch.softmax(x.double(), -1)
    bound = lc.softmax_fwd_bound(ref, x.double() - x.double().amax(-1, keepdim=True), 4096)
    worst, where = lc.violations(_emulate_softmax_fp32(x), ref, bound)
    assert not where and worst < 0.5, worst
    for what, got in (("16 lanes", _emulate_softmax_fp32(x, 16)), ("fp16 lane sums", _emulate_softmax_fp32(x, dtype=torch.float16))):
        bad = ((got.double() - ref).abs() > bound).any(-1).double().mean()
        print(f"{what}: violates the bound on {float(bad):.1%} of the rows")
        assert float(bad) > 0.5, what
    print(f"kernel order: worst err/bound {worst:.3f}")
