// sm90_host.cuh — host side of the tensor-core tiers (conv_tc.cu: fp32-grade 3 x fp16 split, conv_bf16.cu: bf16): the runtime probe,
// TMA map encoding, and the geometry rules of the box kernels, which run a convolution as implicit GEMMs whose 128-pixel M tiles are
// TMA boxes of an NHWC view.  Device side: sm90.cuh.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "common.cuh"

namespace sm90 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct Runtime {
  EncodeTiledFn encode = nullptr;   // cuTensorMapEncodeTiled; null unless the current device has compute capability 9
  int num_sms = 132;                // H100 SXM until the device is read
};
// Probed once per process; each tier still sets its own kernels' shared-memory attribute before it reports itself available
inline const Runtime& runtime() {
  static const Runtime rt = [] {
    Runtime r;
    int dev = 0, major = 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
        major != 9 || cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
        qres != cudaDriverEntryPointSuccess) {
      (void)cudaGetLastError();
      return r;
    }
    r.encode = (EncodeTiledFn)fn;
    cudaDeviceGetAttribute(&r.num_sms, cudaDevAttrMultiProcessorCount, dev);
    (void)cudaGetLastError();
    return r;
  }();
  return rt;
}

// A tiled map with 128-byte swizzle.  pix_stride > 1 (strided convolution): dims 1 and 2 (W, H) are traversed with that element
// stride, and the box extents count traversed elements (loaded pixels x pix_stride).
inline bool encode_map(CUtensorMap* m, CUtensorMapDataType dtype, const void* base, int rank, const cuuint64_t* dims,
                       const cuuint64_t* strides_bytes, const cuuint32_t* box, int pix_stride = 1) {
  const cuuint32_t estr[5] = {1, (cuuint32_t)pix_stride, (cuuint32_t)pix_stride, 1, 1};
  return runtime().encode(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// `npix` pixels of an [N][H][W] grid as a (bw, bh, bn) box with bw * bh * bn == npix whose boxes tile the grid's rows and images
// (the last box may run past the batch: TMA zero fill)
inline bool pick_box(int npix, int H, int W, int& bw, int& bh, int& bn) {
  if (W >= npix) { if (W % npix) return false; bw = npix; bh = 1; bn = 1; return true; }
  if (npix % W) return false;
  bw = W;
  const int rem = npix / W;
  if (H >= rem) { if (H % rem) return false; bh = rem; bn = 1; return true; }
  if (rem % H) return false;
  bh = H; bn = rem / H;
  return true;
}

// Taps of one GEMM: tap i reads the input at (output pixel * in_stride + (dh, dw)) with weight tap wt
struct TapTable { int n; signed char dh[9], dw[9], wt[9]; };
inline TapTable dense_taps(int R, int S, int pad, bool flip) {
  TapTable t{};
  t.n = R * S;
  for (int r = 0; r < R; ++r)
    for (int s = 0; s < S; ++s) {
      const int i = r * S + s;
      t.dh[i] = (signed char)(r - pad); t.dw[i] = (signed char)(s - pad);
      t.wt[i] = (signed char)(flip ? (R * S - 1 - i) : i);
    }
  return t;
}
// Parity class cls = 2a + b of a stride-2 3x3 dgrad: dx[2i+a, 2j+b] only sees the taps with (a+pad_t-r), (b+pad_l-s) even, read
// from the dy grid (1 / 2 / 2 / 4 taps over the four classes, none wasted on structural zeros)
inline TapTable parity_taps(int pad_t, int pad_l, int cls) {
  TapTable t{};
  for (int r = 0; r < 3; ++r)
    for (int s = 0; s < 3; ++s) {
      const int nh = (cls >> 1) + pad_t - r, nw = (cls & 1) + pad_l - s;
      if ((nh & 1) || (nw & 1)) continue;
      t.dh[t.n] = (signed char)(nh / 2); t.dw[t.n] = (signed char)(nw / 2); t.wt[t.n] = (signed char)(r * 3 + s);
      ++t.n;
    }
  return t;
}

// One implicit GEMM of a convolution: M = the pixels of an [N][H][W] grid (the A operand is sampled at in_stride x pixel + tap
// offset), K = taps x Kg channels, N = Nout channels; grid pixel (n, p, q) writes output pixel (p*os + oa, q*os + ob) of [N][Ho][Wo].
struct ConvGemm {
  TapTable taps;
  int N, H, W, Kg, Nout;
  int os, oa, ob, Ho, Wo;
  int in_stride;
};
// The GEMMs of a fprop (op 0) or dgrad (other op) with R = S in {1, 3}.  fprop: one over the output grid.  Stride-1 dgrad: fprop of dy
// with the taps flipped and the channel roles swapped.  Otherwise the four parity classes of a stride-2 dgrad, run back to back.
template <class A>
int conv_gemms(const A* a, int op, ConvGemm g[4]) {
  if (op == 0) {
    g[0] = {dense_taps(a->R, a->S, a->pad_t, false), a->N, a->P, a->Q, a->C, a->K, 1, 0, 0, a->P, a->Q, a->stride};
    return 1;
  }
  if (a->stride == 1) {
    g[0] = {dense_taps(a->R, a->S, a->pad_t, true), a->N, a->H, a->W, a->K, a->C, 1, 0, 0, a->H, a->W, 1};
    return 1;
  }
  for (int c = 0; c < 4; ++c) g[c] = {parity_taps(a->pad_t, a->pad_l, c), a->N, a->P, a->Q, a->K, a->C, 2, c >> 1, c & 1, a->H, a->W, 1};
  return 4;
}

// Geometry the box kernels take (dp_conv_args / dp_conv_bf16_args): square 1x1 or 3x3 filters, stride 1 with 'same' padding or stride 2
// 3x3 with pad 1, or pad 0 + the (0,1,0,1) zero border of Downsample2D (resnet.py:213-218), which TMA out-of-bounds zero fill provides
// for free; the output grid is the input grid / stride.
template <class A>
bool box_geometry(const A* a) {
  if (a->R != a->S || (a->R != 1 && a->R != 3) || a->pad_l != a->pad_t) return false;
  if (!((a->stride == 1 && a->pad_t == (a->R - 1) / 2) || (a->stride == 2 && a->R == 3 && (a->pad_t == 0 || a->pad_t == 1)))) return false;
  return a->P * a->stride == a->H && a->Q * a->stride == a->W;
}

}  // namespace sm90
