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
