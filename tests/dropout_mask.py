"""Host restatement of the GroupNorm dropout keep-mask (include/dpb200.h, dp_gn_args.dropout_*) in numpy uint64 arithmetic, and the
coincidence statistic the independence tests apply to pairs of masks.  Imports no GPU code.

Element `idx` of a dense [N][HW][C] extent (idx = (n * HW + pixel) * C + c, never the pitch) reads 16-bit field idx % 4 of
fmix(m + PHI * (idx // 4 + 1)), with m = fmix(dropout_seed + *dropout_seed_dev) and fmix the splitmix64 finalizer; it is kept iff the
field is >= thr = round(p * 65536) (__float2uint_rn(p * 65536.f)), and survivors are scaled by fp32(65536 / (65536 - thr))."""
import math

import numpy as np

M64 = (1 << 64) - 1
PHI = 0x9E3779B97F4A7C15


def fmix(z):
    """splitmix64's finalizer on a uint64 array (wrap-around multiply)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def combined_seed(dropout_seed: int, seed_dev: int = 0) -> int:
    """dropout_seed + *dropout_seed_dev (mod 2^64); seed_dev 0 stands for a NULL device scalar."""
    return (int(dropout_seed) + int(seed_dev)) & M64


def threshold(p: float) -> int:
    return int(np.rint(np.float32(p) * np.float32(65536.0)))


def keep_scale(p: float) -> np.float32:
    return np.float32(65536.0) / np.float32(65536 - threshold(p))


def fields(seed: int, n: int, start: int = 0, mixed: bool = True) -> np.ndarray:
    """The 16-bit uniforms of elements start .. start + n - 1 (uint32).  mixed=False restates the hash without the seed finalizer (the
    definition before the fix), so a test can show what it catches."""
    m = int(fmix(np.uint64(seed))) if mixed else seed
    g0, g1 = start // 4, (start + n + 3) // 4
    with np.errstate(over="ignore"):
        z = fmix(np.uint64(m) + np.uint64(PHI) * (np.arange(g0, g1, dtype=np.uint64) + np.uint64(1)))
    u = ((z[:, None] >> (np.uint64(16) * np.arange(4, dtype=np.uint64))) & np.uint64(0xFFFF)).astype(np.uint32).reshape(-1)
    return u[start - 4 * g0:start - 4 * g0 + n]


def keep(seed: int, p: float, n: int, start: int = 0, mixed: bool = True) -> np.ndarray:
    """Boolean keep-mask of elements start .. start + n - 1."""
    return fields(seed, n, start, mixed) >= threshold(p)


def keep_nhwc(seed: int, p: float, N: int, HW: int, C: int) -> np.ndarray:
    """The keep-mask of a dense [N][HW][C] tensor."""
    return keep(seed, p, N * HW * C).reshape(N, HW, C)


def scale_nhwc(seed: int, p: float, N: int, HW: int, C: int) -> np.ndarray:
    """The factor the kernel multiplies each element by: fp32(65536 / (65536 - thr)) where kept, 0 where dropped."""
    return np.where(keep_nhwc(seed, p, N, HW, C), keep_scale(p), np.float32(0)).astype(np.float32)


SHIFTS = range(-16, 17)


def coincidences(drop_a: np.ndarray, drop_b: np.ndarray, shift: int) -> tuple:
    """(count of i with drop_a[i] and drop_b[i + shift], number of i compared), over the i where both indices are in range."""
    n = min(len(drop_a), len(drop_b))
    lo, hi = max(0, -shift), min(n, n - shift)
    return int(np.count_nonzero(drop_a[lo:hi] & drop_b[lo + shift:hi + shift])), hi - lo


def worst_coincidence_sigma(drop_a: np.ndarray, drop_b: np.ndarray, q_a: float, q_b: float, shifts=SHIFTS) -> tuple:
    """max over shifts of |coincidences - q_a q_b n| / sigma, sigma the binomial one of independent masks with drop rates q_a / q_b;
    returns (worst sigma, its shift, the coincidence rate there)."""
    worst = (0.0, 0, 0.0)
    q = q_a * q_b
    for s in shifts:
        k, n = coincidences(drop_a, drop_b, s)
        z = abs(k - q * n) / math.sqrt(n * q * (1 - q))
        if z > worst[0]:
            worst = (z, s, k / n)
    return worst
