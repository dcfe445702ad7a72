// image_src.cuh — how the evaluation kernels (fid.cu, ssim.cu) read one image value, so that the PNG quantisation rule lives in one place.
#pragma once
#include <stdint.h>

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
