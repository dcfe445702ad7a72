// image_src.cuh — how the evaluation kernels (fid.cu, ssim.cu, vq.cu) read or write one image value, so that every image quantisation
// rule lives in one place.
#pragma once
#include <stdint.h>

// The LDM's evaluation path (sample_for_FID.py): a decoded image x in about [-1, 1] becomes v = clamp(fl(x + 1) / 2, 0, 1), and
// torchvision's save_image writes the byte trunc(clamp(fl(fl(v * 255) + 0.5), 0, 255)) (mul(255).add_(0.5).clamp_(0, 255).to(uint8)):
// round half up, not the rint rule of the DDPM sampler's PNG write below.
__device__ __forceinline__ float dp_unit_from_pm1(float x) { return fminf(fmaxf(__fdiv_rn(__fadd_rn(x, 1.0f), 2.0f), 0.0f), 1.0f); }
__device__ __forceinline__ uint8_t dp_save_image_byte(float v) {
  return (uint8_t)fminf(fmaxf(__fadd_rn(__fmul_rn(v, 255.0f), 0.5f), 0.0f), 255.0f);
}

// One source value, as the reference's input tensor holds it.  u8: NHWC [n][H][W][C] bytes of decoded image files, u / 255 correctly
// rounded as ToTensor computes it.  Otherwise fp32 NCHW [n][C][H][W], taken as given, or with `quantize` through the sampler's PNG
// write (clamp(x / 2 + 0.5, 0, 1) -> rint(. * 255) -> / 255; rint rounds half to even, as numpy does), so that a DDIM sample in
// [-1, 1] reads exactly like its saved PNG.  The explicit _rn intrinsics keep nvcc from contracting the quantisation into FMAs, which
// would round differently from the numpy / PIL chain it restates.
__device__ __forceinline__ float dp_image_src(const void* src, int u8, int quantize, int n, int c, int h, int w, int C, int H, int W) {
  if (u8) {
    const uint8_t u = static_cast<const uint8_t*>(src)[(((long long)n * H + h) * W + w) * C + c];
    return __fdiv_rn((float)u, 255.0f);
  }
  const float x = static_cast<const float*>(src)[(((long long)n * C + c) * H + h) * W + w];
  if (!quantize) return x;
  const float v = fminf(fmaxf(__fadd_rn(__fmul_rn(x, 0.5f), 0.5f), 0.0f), 1.0f);
  return __fdiv_rn(rintf(__fmul_rn(v, 255.0f)), 255.0f);
}
