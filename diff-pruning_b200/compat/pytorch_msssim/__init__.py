"""`import pytorch_msssim` for compute_ssim.py: `ssim` on diff_pruning_b200.ssim (CUDA fp32 4-D tensors, the fused fp64 kernel).
MS-SSIM and the SSIM / MS_SSIM module classes are not provided; CPU tensors raise NotImplementedError."""
from diff_pruning_b200.ssim import ssim  # noqa: F401

__all__ = ["ssim"]
