"""Error model, chain lengths and launch dedup key of the launch census (test_launch_census_gpu.py, checked on the host by
test_launch_census_host.py).

Error model of a product-sum output y_i = sum_k a_k b_k computed by the tensor-core kernels:
  * operands: the 3 x fp16 split keeps 22 bits of each operand and drops lo' * lo' (conv_tc.cu), so every product carries a relative
    error of a few 2^-22 with a random sign; over the sum that is a few 2^-22 * s_i, s_i = sqrt(sum_k (a_k b_k)^2).
  * accumulation: wgmma adds each 16-deep block of products into the fp32 accumulator with a TRUNCATING rounding: every one of the L
    updates of one output loses less than one ulp of the partial sum, ulp(v) <= 2^-23 |v|, and these errors all have the sign of the
    partial sum, so they add up linearly to < 2^-23 L mean_j |partial sum j|.  For the random-sign operands of the census the mean
    magnitude of the partial sums is about 0.53 s_i, s_i = sqrt(sum_k (a_k b_k)^2), and stays below 1.5 s_i: BETA = 2 * 1.5 = 3.
  * epilogue: bias / per-image row / residual / the old value (+=) each cost at most one fp32 rounding of the running value.
Hence  |y^ - y| <= (ALPHA + BETA * L) * 2^-24 * s_i + 2^-23 * sum|epilogue terms|.
ALPHA = 64 covers the operand split (a few 2^-22 s_i with its tail) and the final fp32 rounding of the output.  The bf16 tier is held
to the same bound against fp64 math on the bf16-rounded operands (its products are exact, only the accumulation rounds).

The bound keeps its teeth only while the accumulation term stays below the error of a dropped lo' correction term (about 2^-12.3 s_i):
every tensor-core launch of the census must have L <= L_MAX, the longest chain at which test_launch_census_host.py shows that the
split with one correction term dropped violates the bound on most outputs.

Fixed-order fp32 sums with round-to-nearest (column sums, GroupNorm statistics, loss / norm reductions) are held to
SUM_ALPHA * 2^-24 * s + 8 * sqrt(n) * 2^-24 * s (sum_bound): the n rounding errors are independent, zero-mean and each below 2^-24 of a
partial sum of order s, so their total is of order sqrt(n) 2^-24 s; 8 standard deviations is never reached by chance, while dropping a
single term of typical size s / sqrt(n) exceeds it for every n < 2^21.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
ALPHA, BETA = 64.0, 3.0
L_MAX = 640
SUM_ALPHA = 16.0


def chain_fprop(taps: int, kg: int, ksplit: int = 1) -> int:
    """fp32 accumulator updates of one output of a fprop / dgrad / NT-GEMM launch: taps x ceil(Kg / 64) pipeline stages of 4 wgmma
    k-steps each, divided over ksplit K splits (splitk_count), plus the fixed-order sum of the splits."""
    return -(-taps * -(-kg // 64) * 4 // ksplit) + ksplit


def chain_wgrad(pixels_per_cta: int, splits: int) -> int:
    """fp32 accumulator updates of one weight-gradient element: one per 16 pixels a CTA walks, plus the fixed-order reduce of the
    splits."""
    return -(-pixels_per_cta // 16) + splits


def wgrad_pixels_per_cta(rows: int, splits: int) -> int:
    """Pixels one CTA of dp_conv2d_wgrad walks: the kernel cuts the rows into 64-pixel chunks and gives each split ceil(chunks / splits)."""
    chunks = max(1, rows // 64)
    return -(-chunks // splits) * 64


def product_bound(s: torch.Tensor, L: int, epi_abs=None) -> torch.Tensor:
    """Element-wise bound of a product-sum output (see the module docstring); s and epi_abs in float64."""
    b = (ALPHA + BETA * L) * U * s
    if epi_abs is not None:
        b = b + 2 * U * epi_abs
    return b


def sum_bound(s: torch.Tensor, n: int) -> torch.Tensor:
    """Element-wise bound of a fixed-order fp32 sum of n terms whose squares sum to s^2 (see the module docstring)."""
    return (SUM_ALPHA + 8.0 * math.sqrt(n)) * U * s


def splitk_count(need_floats: int, rows: int, cols: int, stages: int) -> int:
    """K splits of a fprop / dgrad launch from its split-K workspace size, which holds ksplit x [M tiles x 128][N tiles x 128] floats
    (the launch's `stages` = taps x ceil(Kg / 64) pipeline stages are split at most 16 ways, at least 4 stages per split)."""
    if need_floats <= 0:
        return 1
    ks = need_floats // ((-(-rows // 128) * 128) * (-(-cols // 128) * 128))
    return max(1, min(ks, 16, stages // 4))


MAX_SPLIT_STAGES = 147     # conv_tc.cu PS_MAX_SPLIT_STAGES: 4 x 147 = 588 accumulator updates per split, within L_MAX with 16 splits


def pick_ksplit(tiles: int, iters: int, num_sms: int):
    """conv_tc.cu's pick_ksplit: (K splits, pipeline stages per split) of a persistent-kernel launch with `tiles` output tiles of `iters`
    stages each.  To fill the SMs: no split when the tiles already cover half the SMs or there are fewer than 8 stages, otherwise enough
    work items to fill them, at least 4 stages per split, at most 16 splits.  Whatever the tiles, at least ceil(iters / MAX_SPLIT_STAGES)
    splits, so that no chain is longer than MAX_SPLIT_STAGES stages; and no empty split."""
    ks = 1
    if tiles * 2 <= num_sms and iters >= 8:
        ks = min(num_sms // tiles, iters // 4, 16)
    ks = max(ks, -(-iters // MAX_SPLIT_STAGES))
    if ks < 2:
        return 1, iters
    ips = -(-iters // ks)
    return -(-iters // ips), ips


def general_split(N: int, P: int, Q: int, K: int, C: int, R: int, S: int, num_sms: int):
    """(K splits, stages per split) of a general-geometry fprop (conv_tc_ps_kernel<true>): ceil(N P Q / 128) x ceil(K / 128) output
    tiles of R S ceil(C / 64) stages."""
    tiles = -(-(N * P * Q) // 128) * -(-K // 128)
    return pick_ksplit(tiles, R * S * -(-C // 64), num_sms)


def chain_general(ksplit: int, stages_per_split: int) -> int:
    """fp32 accumulator updates of one output of a general-geometry fprop: 4 wgmma k-steps per stage of its split, plus the fixed-order
    sum of the splits."""
    return 4 * stages_per_split + ksplit


# ---------------------------------------------------------------------------------------------------- evaluation path (FID, DDIM)
U53 = 2.0 ** -53


def bilinear_coords(n_src: int, n_dst: int, half_pixel: bool = True):
    """Source rows of a bilinear resize to n_dst, as torch's align_corners=False rule forms them in fp32: scale = n_src / n_dst,
    r = max(scale (dst + 0.5) - 0.5, 0), i0 = trunc(r), i1 = i0 + 1 except on the last row, l1 = r - i0, l0 = 1 - l1 (fp32).
    half_pixel=False drops the half-pixel offset (r = scale dst).  Returns (i0, i1, l0, l1, slack): the weights in float64 and
    slack, two ulps of scale (dst + 0.5), a bound on how far a contracted (fma) evaluation of r can move the weights."""
    f = torch.float32
    d = torch.arange(n_dst, dtype=f)
    scale = torch.tensor(float(n_src), dtype=f) / torch.tensor(float(n_dst), dtype=f)
    prod = scale * (d + 0.5) if half_pixel else scale * d
    r = (prod - 0.5).clamp_min(0.0) if half_pixel else prod
    i0 = r.long()
    i1 = torch.where(i0 < n_src - 1, i0 + 1, i0)
    l1 = r - i0.to(f)
    l0 = 1.0 - l1
    return i0, i1, l0.double(), l1.double(), 2.0 ** -22 * prod.double()


def bilinear_ref(src: torch.Tensor, Ho: int, Wo: int, half_pixel: bool = True):
    """(ref, bound) of a bilinear resize of src [N, C, Hs, Ws] (float64: the values the kernel reads) to Ho x Wo, interpolated in fp64
    from the fp32 weights of bilinear_coords.  The kernel's fp32 interpolation is a convex combination of four values, six roundings:
    8 2^-24 of the largest neighbour covers it.  A weight moved by `slack` moves the result by at most slack x the largest jump between
    neighbouring source values, bounded by 2 max|src| of the image channel (the moved weight may select the next source row)."""
    N, Cc, Hs, Ws = src.shape
    h0, h1, a0, a1, sh = bilinear_coords(Hs, Ho, half_pixel)
    w0, w1, b0, b1, sw = bilinear_coords(Ws, Wo, half_pixel)
    dev = src.device
    h0, h1, w0, w1 = (t.to(dev) for t in (h0, h1, w0, w1))
    A0, A1, sh = (t.to(dev).view(-1, 1) for t in (a0, a1, sh))
    B0, B1, sw = (t.to(dev).view(1, -1) for t in (b0, b1, sw))
    rows0, rows1 = src[:, :, h0], src[:, :, h1]
    v00, v01, v10, v11 = rows0[..., w0], rows0[..., w1], rows1[..., w0], rows1[..., w1]
    ref = A0 * (B0 * v00 + B1 * v01) + A1 * (B0 * v10 + B1 * v11)
    vmax = torch.stack([v00.abs(), v01.abs(), v10.abs(), v11.abs()]).amax(0)
    smax = src.abs().amax((2, 3), keepdim=True)
    return ref, 8 * U * vmax + 2 * smax * (sh + sw)


def avgpool_ref(x: torch.Tensor, stride: int, pad: int):
    """(ref, bound) of the 3 x 3 average pool that does not count padding (count_include_pad=False) of x [N, C, H, W] float64: the
    fixed-order fp32 sum of the n <= 9 taps inside the image (sum_bound), then one rounding of the division by n."""
    ref = F.avg_pool2d(x, 3, stride, pad, count_include_pad=False)
    n = F.avg_pool2d(torch.ones_like(x[:1, :1]), 3, stride, pad, count_include_pad=True) * 9          # taps inside the image
    s = (F.avg_pool2d(x * x, 3, stride, pad, count_include_pad=False) * n).sqrt()
    return ref, (SUM_ALPHA + 8.0 * 3.0) * U * s / n + 2 * U * ref.abs()


def global_mean_ref(x: torch.Tensor):
    """(ref, bound) of the mean over H x W of x [N, C, H, W] float64 as dp_global_mean forms it: an fp64 sum of the H W fp32 terms
    ((H W + 4) 2^-53 sum|x|), one fp64 division and one rounding to fp32 (2^-24 of the mean, doubled for room)."""
    HW = x.shape[2] * x.shape[3]
    ref = x.mean((2, 3))
    return ref, (HW + 4) * U53 * x.abs().mean((2, 3)) + 2 * U * ref.abs()


def moments_ref(f: torch.Tensor, shift, s0: torch.Tensor, sxx0: torch.Tensor):
    """(sum, bound, sxx, bound) of dp_feature_moments accumulating rows of f [rows, D] into s0 [D] / sxx0 [D, D], in float64.
    d = f - shift is exact in fp64; each of the rows fp64 updates of an element rounds once (fma), so with the old value as one more
    term the error is below (rows + 4) 2^-53 (sum_r |d_ri d_rj| + |old|)."""
    d = f.double() - (shift.double() if shift is not None else 0.0)
    rows = d.shape[0]
    k = (rows + 4) * U53
    return (s0 + d.sum(0), k * (d.abs().sum(0) + s0.abs()),
            sxx0 + d.T @ d, k * (d.abs().T @ d.abs() + sxx0.abs()))


def ddim_step_ref(x, e, nz, sb: float, sa: float, clip: float, sap: float, dirc: float, sigma: float):
    """(ref, bound) of one DDIM update from the fp32 coefficients the scheduler passes: x0 = (x - sb e) / sa, clipped to +-clip when
    clip > 0, out = sap x0 + dirc e (+ sigma noise).  x0 carries at most three roundings of |x| + sb |e| (product, difference,
    division), 4 2^-24 (|x| + sb |e|) / sa, which sap scales; the clip is 1-Lipschitz, so a pre-clip x0 within that bound of +-clip
    may land on either side; the update adds a few roundings of its terms."""
    x, e = x.double(), e.double()
    x0 = (x - sb * e) / sa
    ex0 = 4 * U * (x.abs() + sb * e.abs()) / sa
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    ref = sap * x0 + dirc * e
    mag = sap * x0.abs() + dirc * e.abs()
    if nz is not None and sigma != 0:
        ref = ref + sigma * nz.double()
        mag = mag + sigma * nz.double().abs()
    return ref, sap * ex0 + 4 * U * mag


def softmax_fwd_bound(ref, z, cols):
    """Element-wise bound of dp_softmax_fwd (one warp per row: z = x - max in fp32, e = expf(z), per-lane sums of ceil(cols / 32)
    e's, a 5-level butterfly over the lanes, p = e * (1 / sum)), relative to p:
      * its own exponential: expf is within 2 ulp (2^-22 relative), and the fp32 rounding of z moves exp(z) by up to 2^-24 |z|;
      * the row sum: the same exponential errors weighted by the terms, 2^-22 + 2^-24 sum_k p_k |z_k|, and the fixed-order rounding
        of the sum.  Every partial sum is at most the row sum S (the terms are positive) and one lane's chain is ceil(cols / 32)
        additions plus the 5 butterfly levels: sum_bound's model with S for s, (SUM_ALPHA + 8 sqrt(n)) 2^-24 (the lane holding the
        row's largest term adds its other terms to a partial of about S from the start, so its n roundings are each of order 2^-24 S);
      * the reciprocal and the product: one rounding each.
    The argument terms are doubled for room; values below 2^-126 are held to 2^-126 absolute (subnormal exponentials).  An emulation
    of the kernel's order of operations in torch fp32 on an H100 is bit-identical to it; at 2 x 32768 rows of 4096 (the VQ-f4 attention
    at batch 8) its worst row-sum error is 17.4 2^-24, its worst element 35 2^-24, against a bound of 108 2^-24 and more."""
    n = -(-cols // 32) + 5
    rel = (2.0 ** -22 + 2.0 ** -23 * z.abs()) + (2.0 ** -22 + 2.0 ** -23 * (ref * z.abs()).sum(-1, keepdim=True))
    rel = rel + (SUM_ALPHA + 8.0 * math.sqrt(n)) * U + 2 * U
    return rel * ref + 2.0 ** -126


def violations(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, limit: int = 8):
    """(worst err / bound, coordinates of up to `limit` elements where |got - ref| > bound, or where got is not finite)."""
    err = (got.double() - ref.double()).abs()
    bad = ~(err <= bound)
    ratio = (err / bound.clamp_min(1e-300))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not bool(torch.isfinite(got).all()):
        worst = math.inf
    coords = [tuple(int(c) for c in idx) for idx in bad.nonzero()[:limit].tolist()]
    return worst, coords


def argkinds(name: str):
    """'p' / 'i' / 'f' / 's' (struct) per argument of an exported entry point, from its ctypes signature; the trailing stream dropped."""
    from diff_pruning_b200 import _lib as L
    kinds = []
    for t in list(L._SIGS[name][1])[:-1]:
        if t is C.c_void_p:
            kinds.append("p")
        elif t in (C.c_float, C.c_double):
            kinds.append("f")
        elif isinstance(t, type) and issubclass(t, C._Pointer):
            kinds.append("s")
        else:
            kinds.append("i")
    return kinds


_SINKS: list = []      # on_call of every active wrap_launches block, innermost last


class wrap_launches:
    """`with wrap_launches(lib, on_call):` every kernel-launching entry point of the library (the ones taking a stream last) calls
    on_call(name, args, stream) before it runs: args are the arguments without the stream, struct arguments copied as they are at the
    call.  Plans bind struct launches when they record them, so a plan must be built inside such a block; the wrappers it binds report
    to whichever blocks are active when it runs, so a plan built in one block is seen by a later one."""

    def __init__(self, lib, on_call):
        self.lib, self.on_call, self.orig = lib, on_call, {}

    def __enter__(self):
        from diff_pruning_b200 import _lib as L
        from diff_pruning_b200.engine import _copy_args
        _SINKS.append(self.on_call)
        for name, (_, argtypes) in L._SIGS.items():
            if not argtypes or argtypes[-1] is not C.c_void_p:      # launches take the stream last; the rest are host queries
                continue
            fn, kinds = getattr(self.lib, name), argkinds(name)
            if getattr(fn, "_dp_wrapped", False):                  # an outer block wrapped it already
                continue

            def wrapped(*args, fn=fn, kinds=kinds, name=name):
                if _SINKS:
                    snap = [_copy_args(getattr(v, "_obj", v)) if k == "s" else v for k, v in zip(kinds, args[:-1])]
                    for sink in list(_SINKS):
                        sink(name, snap, args[-1])
                return fn(*args)
            wrapped._dp_wrapped = True
            self.orig[name] = fn
            setattr(self.lib, name, wrapped)
        return self

    def __exit__(self, *exc):
        _SINKS.remove(self.on_call)
        for name, fn in self.orig.items():
            setattr(self.lib, name, fn)
        return False


def _ptr_key(v, esz: int = 4):
    """A pointer's part of the key: NULL or not, and its 16-byte alignment phase in elements of `esz` bytes (the element offset of a
    view mod 16 / esz)."""
    return None if not v else (int(v) % 16) // esz


BF16_FIELDS = {"x_bf16", "dy_bf16", "w_bf16", "y_bf16"}   # 2-byte elements in the argument structs


def struct_key(s: C.Structure):
    out = []
    for name, t in s._fields_:
        v = getattr(s, name)
        if t is C.c_void_p:
            out.append((name, _ptr_key(v, 2 if name in BF16_FIELDS else 4)))
        elif hasattr(v, "__len__"):
            out.append((name, tuple(v)))
        else:
            out.append((name, v))
    return tuple(out)


def launch_key(name: str, kinds, args):
    """Dedup key of one captured call: the entry point, every integer / float field or argument (extents, ld, flags, splits ...),
    and for every pointer whether it is set and its 16-byte phase."""
    parts = [name]
    for k, v in zip(kinds, args):
        if k == "s":
            parts.append(struct_key(v))
        elif k == "p":
            parts.append(_ptr_key(v, 2))      # plain pointer arguments: the finer phase (bf16 / fp16 buffers among them)
        else:
            parts.append(v)
    return tuple(parts)


# ---------------------------------------------------------------------------------------------------- host emulation of the split
def split_h(v: torch.Tensor):
    """The 3 x fp16 split of conv_tc.cu on the host: (hi, lo', scale) with s*v = hi + lo' / 2^11, |s*v| < 2^14 (float64 results)."""
    e = math.floor(math.log2(float(v.abs().max()))) + 1
    s = 2.0 ** (14 - e)
    sv = v.double() * s
    hi = sv.half().double()
    lo = ((sv - hi) * 2048).half().double()
    return hi, lo, s


def c5_model():
    """cin256-v2 as bench.py builds it: seed-0 init, the zero-initialised convolutions re-drawn (a fresh LDM UNet outputs exactly 0).
    Returns (model, config)."""
    from diff_pruning_b200 import ldm
    cfg = ldm.CIN256_V2_CONFIG
    torch.manual_seed(0)
    m = ldm.UNetModel(**cfg)
    g = torch.Generator().manual_seed(5)
    for p in m.parameters():
        if p.dim() > 1 and float(p.detach().abs().sum()) == 0:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.02)
    return m, cfg
