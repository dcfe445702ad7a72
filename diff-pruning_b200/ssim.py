"""SSIM evaluation on the device: the consistency metric of Diff-Pruning (SSIM and MSE between images of the pruned and of the
pre-trained model drawn from the same initial noise, compute_ssim.py), on one fused fp64 kernel (dp_ssim, ssim.cu).

ssim               pytorch_msssim.ssim for 4-D CUDA fp32 tensors (the only name the reference's scripts use).
ssim_of_paths      compute_ssim.py's two numbers, per image, over two folders of image files paired by relative path.
ssim_of_pipelines  the same numbers for two DDIMPipelines sampled from the same seed, straight from device memory (no PNG written),
                   bit-identical to saving both folders the way ddpm_sample.py does and running ssim_of_paths.

The numeric definition (11-tap Gaussian, sigma 1.5, separable, "valid"; C1 = (0.01 R)^2, C2 = (0.03 R)^2; the map's mean per
channel) is pinned on the reference tree's utils_image.py (tests/golden/ssim_ref.pt).  The pytorch_msssim 1.0 API semantics
restated in `ssim` (default data_range=255, the squeeze of singleton dimensions, the size_average reductions, nonnegative_ssim and
the window taps' fp32 construction) are recalled, not verified against that package, which is not vendored."""
from __future__ import annotations

import ctypes
import os
from typing import Tuple

import numpy as np
import torch

from . import _lib as L
from .engine import _stream

WIN_SIZE = 11
DP_SSIM_U8_NHWC, DP_SSIM_F32_NCHW, DP_SSIM_F32_NCHW_PNG = 0, 1, 2


def gaussian_window(size: int = WIN_SIZE, sigma: float = 1.5, dtype=torch.float32) -> torch.Tensor:
    """pytorch_msssim._fspecial_gauss_1d's taps (recalled), in fp32: exp(-c^2 / (2 sigma^2)) over c = -size//2 .. size//2, divided
    by their sum.  The fp32 taps sum to 1 only to ~1e-7; dtype=torch.float64 gives the exact-grade taps of cv2.getGaussianKernel."""
    coords = torch.arange(size, dtype=dtype)
    coords -= size // 2
    g = torch.exp(-(coords ** 2) / (2 * sigma ** 2))
    g /= g.sum()
    return g


def _scores(x: torch.Tensor, y: torch.Tensor, fmt: int, data_range: float, K=(0.01, 0.03), win: torch.Tensor = None):
    """One dp_ssim launch: (ssim [N, C] float64, sse [N] float64) on the device.  x, y: contiguous uint8 NHWC (fmt 0) or fp32 NCHW."""
    if fmt == DP_SSIM_U8_NHWC:
        N, H, W, C = x.shape
    else:
        N, C, H, W = x.shape
    win = gaussian_window() if win is None else win
    out = torch.empty(N, C, dtype=torch.float64, device=x.device)
    sse = torch.empty(N, dtype=torch.float64, device=x.device)
    a = L.SsimArgs()
    a.x, a.y, a.format, a.N, a.C, a.H, a.W, a.win_size = x.data_ptr(), y.data_ptr(), fmt, N, C, H, W, WIN_SIZE
    for k, v in enumerate(win.tolist()):
        a.win[k] = v
    a.c1, a.c2 = (K[0] * data_range) ** 2, (K[1] * data_range) ** 2
    a.ssim_nc, a.sse_n = out.data_ptr(), sse.data_ptr()
    with torch.cuda.device(x.device):
        L.check(L.load().dp_ssim(ctypes.byref(a), _stream()), "ssim")
    return out, sse


def _per_image(ssim_nc: torch.Tensor) -> torch.Tensor:
    """Mean over channels, in float64: the one reduction every entry point shares, so their per-image values agree bit for bit."""
    return ssim_nc.mean(1)


def ssim(X, Y, data_range=255, size_average=True, win_size=11, win_sigma=1.5, win=None, K=(0.01, 0.03), nonnegative_ssim=False):
    """pytorch_msssim.ssim (1.0 semantics, recalled) on the device.  X, Y: CUDA fp32 [N, C, H, W] (after pytorch_msssim's squeeze of
    singleton dimensions from the last down to dim 2).  Returns a CUDA fp32 tensor: the mean over all (image, channel) values with
    size_average=True, else one value per image, the mean over its channels; nonnegative_ssim applies ReLU to the per-channel values.
    The moments and the map are computed in fp64 (dp_ssim), so values are closer to the exact SSIM than pytorch_msssim's fp32 ones.
    ValueError as pytorch_msssim: different shapes, not 4-D or 5-D, an even window.  NotImplementedError: 5-D (3-D SSIM), CPU tensors
    (no CPU fallback), dtypes other than fp32, win_size other than 11, a user-supplied `win`, images under 11 pixels (pytorch_msssim
    warns and skips the smoothing along that axis; that is not copied)."""
    if not X.shape == Y.shape:
        raise ValueError(f"Input images should have the same dimensions, but got {X.shape} and {Y.shape}.")
    for d in range(len(X.shape) - 1, 1, -1):
        X = X.squeeze(dim=d)
        Y = Y.squeeze(dim=d)
    if len(X.shape) not in (4, 5):
        raise ValueError(f"Input images should be 4-d or 5-d tensors, but got {X.shape}")
    if win is not None:
        win_size = win.shape[-1]
    if not (win_size % 2 == 1):
        raise ValueError("Window size should be odd.")
    if len(X.shape) == 5:
        raise NotImplementedError("diff_pruning_b200.ssim: 3-D (5-d input) SSIM is not implemented")
    if win is not None:
        raise NotImplementedError("diff_pruning_b200.ssim: a user-supplied window is not implemented (only the Gaussian of win_sigma)")
    if win_size != WIN_SIZE:
        raise NotImplementedError(f"diff_pruning_b200.ssim: only win_size={WIN_SIZE} is implemented")
    if not (X.is_cuda and Y.is_cuda and X.device == Y.device):
        raise NotImplementedError("diff_pruning_b200.ssim: inputs must be CUDA tensors on one device (no CPU fallback)")
    if X.dtype != torch.float32 or Y.dtype != torch.float32:
        raise NotImplementedError(f"diff_pruning_b200.ssim: only float32 inputs are implemented, got {X.dtype} / {Y.dtype}")
    if X.shape[2] < WIN_SIZE or X.shape[3] < WIN_SIZE:
        raise NotImplementedError(f"diff_pruning_b200.ssim: images must be at least {WIN_SIZE} x {WIN_SIZE}, got {tuple(X.shape[2:])}")
    ssim_nc, _ = _scores(X.contiguous(), Y.contiguous(), DP_SSIM_F32_NCHW, float(data_range), K, gaussian_window(win_size, win_sigma))
    if nonnegative_ssim:
        ssim_nc = torch.relu(ssim_nc)
    return (ssim_nc.mean() if size_average else _per_image(ssim_nc)).float()


def _relative_files(path) -> dict:
    from .fid import _image_files
    root = os.fspath(path)
    return {os.path.relpath(f, root): f for f in _image_files(root)}


def ssim_of_paths(path1, path2, batch_size: int = 100) -> Tuple[np.ndarray, np.ndarray]:
    """compute_ssim.py over two folders (searched recursively for image files, decoded with PIL as RGB): per-image SSIM at
    data_range 1.0 (the mean of the per-channel values) and MSE (mean of (x - y)^2 over channels and pixels of the ToTensor values),
    float64 arrays in the order of the sorted relative paths.  Files are paired by relative path, and two folders whose sets of
    relative paths differ are an error.  (compute_ssim.py zips two unsorted glob lists, which pairs images by the order the file
    system lists them; pairing by name is what the metric means.)"""
    from .fid import _decode
    f1, f2 = _relative_files(path1), _relative_files(path2)
    if set(f1) != set(f2):
        only1, only2 = sorted(set(f1) - set(f2)), sorted(set(f2) - set(f1))
        raise ValueError(f"image folders do not hold the same relative paths: {len(only1)} only in {path1} (e.g. {only1[:3]}), "
                         f"{len(only2)} only in {path2} (e.g. {only2[:3]})")
    names = sorted(f1)
    dev = torch.device("cuda", torch.cuda.current_device())
    ssims, mses = [], []
    for start in range(0, len(names), batch_size):
        part = names[start:start + batch_size]
        a, b = _decode([f1[n] for n in part]), _decode([f2[n] for n in part])
        if a.shape != b.shape:
            raise ValueError(f"image sizes differ between the folders: {tuple(a.shape[1:3])} vs {tuple(b.shape[1:3])}")
        s, m = _pair_scores(a.to(dev), b.to(dev), DP_SSIM_U8_NHWC)
        ssims.append(s)
        mses.append(m)
    if not names:
        return np.empty(0), np.empty(0)
    return np.concatenate(ssims), np.concatenate(mses)


def _pair_scores(a: torch.Tensor, b: torch.Tensor, fmt: int):
    """(per-image SSIM, per-image MSE) float64 NumPy arrays at data_range 1.0."""
    H, W = (a.shape[1], a.shape[2]) if fmt == DP_SSIM_U8_NHWC else (a.shape[2], a.shape[3])
    if H < WIN_SIZE or W < WIN_SIZE:
        raise NotImplementedError(f"diff_pruning_b200.ssim: images must be at least {WIN_SIZE} x {WIN_SIZE}, got {(H, W)}")
    ssim_nc, sse = _scores(a.contiguous(), b.contiguous(), fmt, 1.0)
    numel = a[0].numel()
    return _per_image(ssim_nc).cpu().numpy(), (sse / numel).cpu().numpy()


@torch.no_grad()
def ssim_of_pipelines(pipeline_a, pipeline_b, total_samples: int, batch_size: int, num_inference_steps: int,
                      seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """The paper's consistency metric without writing PNGs: `total_samples // batch_size` batches from each pipeline, drawn as
    ddpm_sample.py:57-74 draws them (one generator per pipeline on its device, seeded with `seed`, one call per batch), scored pair by
    pair through the PNG quantisation of the samples.  Returns (ssim [n], mse [n]) float64 in sample order, equal bit for bit to
    saving both pipelines' samples as ddpm_sample.py names them and running ssim_of_paths on the two folders."""
    def shape_of(p):
        cfg = p.unet.config
        size = cfg.sample_size if isinstance(cfg.sample_size, int) else tuple(cfg.sample_size)
        return cfg.in_channels, size
    if shape_of(pipeline_a) != shape_of(pipeline_b):
        raise ValueError(f"the pipelines sample different shapes: {shape_of(pipeline_a)} vs {shape_of(pipeline_b)}")
    ga = torch.Generator(device=pipeline_a.device).manual_seed(seed)
    gb = torch.Generator(device=pipeline_b.device).manual_seed(seed)
    ssims, mses = [], []
    for _ in range(total_samples // batch_size):
        xa = pipeline_a(batch_size=batch_size, num_inference_steps=num_inference_steps, generator=ga, output_type="device").images
        xb = pipeline_b(batch_size=batch_size, num_inference_steps=num_inference_steps, generator=gb, output_type="device").images
        s, m = _pair_scores(xa, xb.to(xa.device), DP_SSIM_F32_NCHW_PNG)
        ssims.append(s)
        mses.append(m)
    if not ssims:
        return np.empty(0), np.empty(0)
    return np.concatenate(ssims), np.concatenate(mses)
