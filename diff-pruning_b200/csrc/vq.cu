// vq.cu — the two ends of the LDM's first-stage decoder on the evaluation path (VQModelInterface.decode, sample_for_FID.py): the
// codebook lookup that turns a sampled latent into the decoder's input, and the clamp / save_image quantisation of the decoded images.
// Both are exact: no result depends on launch geometry or on another image of the batch.
#include <math.h>
#include "common.cuh"
#include "image_src.cuh"

namespace {
constexpr int VQ_NT = 128;
constexpr int VQ_MAX_D = 8;
constexpr int VQ_TILE_FLOATS = 6144;   // codebook rows staged in shared memory per pass (24 KB): 2048 rows of the VQ-f4 codebook

// One thread per latent pixel.  The codebook streams through shared memory a tile at a time; every thread reads the same row at the same
// time (a broadcast).  The distance is formed in fp64 with explicit roundings: the difference of two fp32 values and its square are exact
// there, so only the running sum rounds, in the documented order, and the argmin is reproducible on the host bit for bit.
template <int D>
__global__ void __launch_bounds__(VQ_NT) vq_quantize_kernel(const float* __restrict__ z, int N, int H, int W, float inv_scale,
                                                            const float* __restrict__ codebook, int n_embed, int quantize,
                                                            float* __restrict__ out, long long ld_out, long long* __restrict__ indices) {
  __shared__ float tile[VQ_TILE_FLOATS];
  const long long HW = (long long)H * W, total = (long long)N * HW;
  const long long p = blockIdx.x * (long long)VQ_NT + threadIdx.x;
  const bool live = p < total;
  const long long n = live ? p / HW : 0, hw = live ? p % HW : 0;
  float zv[D];
#pragma unroll
  for (int d = 0; d < D; ++d) zv[d] = live ? __fmul_rn(inv_scale, __ldg(z + (n * D + d) * HW + hw)) : 0.0f;
  if (!quantize) {   // force_not_quantize: the scaled latent itself
    if (live) {
#pragma unroll
      for (int d = 0; d < D; ++d) out[p * ld_out + d] = zv[d];
    }
    return;
  }
  double best = INFINITY;
  int bi = 0;
  constexpr int ROWS = VQ_TILE_FLOATS / D;
  for (int j0 = 0; j0 < n_embed; j0 += ROWS) {
    const int nr = min(ROWS, n_embed - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < nr * D; e += VQ_NT) tile[e] = __ldg(codebook + (long long)j0 * D + e);
    __syncthreads();
    if (!live) continue;
    for (int j = 0; j < nr; ++j) {
      double dist = 0.0;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const double t = __dsub_rn((double)zv[d], (double)tile[j * D + d]);
        dist = __dadd_rn(dist, __dmul_rn(t, t));
      }
      if (dist < best) {   // strict: the lowest index wins a tie
        best = dist;
        bi = j0 + j;
      }
    }
  }
  if (!live) return;
  // the straight-through expression z + (e - z) of VectorQuantizer2.forward, rounded as fp32 torch rounds it (not always e)
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float e = __ldg(codebook + (long long)bi * D + d);
    out[p * ld_out + d] = __fadd_rn(zv[d], __fsub_rn(e, zv[d]));
  }
  if (indices) indices[p] = bi;
}

constexpr int DI_NT = 256;
// one thread per output value (n, h, w, c), channels fastest
__global__ void decode_images_kernel(const float* __restrict__ y, long long ld, int N, int C, int H, int W, uint8_t* __restrict__ u8,
                                     float* __restrict__ f32) {
  const long long HW = (long long)H * W, total = (long long)N * HW * C;
  for (long long i = blockIdx.x * (long long)DI_NT + threadIdx.x; i < total; i += (long long)gridDim.x * DI_NT) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const float v = dp_unit_from_pm1(__ldg(y + pix * ld + c));
    if (u8) u8[i] = dp_save_image_byte(v);
    if (f32) f32[((pix / HW) * C + c) * HW + pix % HW] = v;
  }
}

template <int D>
int launch_vq(const float* z, int N, int H, int W, float inv_scale, const float* codebook, int n_embed, int quantize, float* out,
              long long ld_out, long long* indices, cudaStream_t s) {
  const long long total = (long long)N * H * W;
  vq_quantize_kernel<D><<<(unsigned)((total + VQ_NT - 1) / VQ_NT), VQ_NT, 0, s>>>(z, N, H, W, inv_scale, codebook, n_embed, quantize, out,
                                                                                  ld_out, indices);
  return dp_check_launch();
}
}  // namespace

extern "C" int dp_vq_quantize(const float* z, int32_t N, int32_t D, int32_t H, int32_t W, float inv_scale, const float* codebook,
                              int32_t n_embed, int32_t quantize, float* out, int64_t ld_out, int64_t* indices, dp_stream_t stream) {
  DP_REQUIRE(z && out && (codebook || !quantize), DP_ERR_NULL);
  DP_REQUIRE(N > 0 && H > 0 && W > 0 && D > 0 && ld_out >= D && (n_embed > 0 || !quantize), DP_ERR_SHAPE);
  DP_REQUIRE(D <= VQ_MAX_D, DP_ERR_UNSUPPORTED);
  DP_REQUIRE((long long)N * H * W < (1LL << 40), DP_ERR_SHAPE);
  const int q = quantize ? 1 : 0;
  long long* idx = reinterpret_cast<long long*>(indices);
  cudaStream_t s = (cudaStream_t)stream;
  switch (D) {
    case 1: return launch_vq<1>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 2: return launch_vq<2>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 3: return launch_vq<3>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 4: return launch_vq<4>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 5: return launch_vq<5>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 6: return launch_vq<6>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    case 7: return launch_vq<7>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
    default: return launch_vq<8>(z, N, H, W, inv_scale, codebook, n_embed, q, out, ld_out, idx, s);
  }
}

extern "C" int dp_decode_images(const float* y, int64_t ld, int32_t N, int32_t C, int32_t H, int32_t W, uint8_t* u8_nhwc, float* f32_nchw,
                                dp_stream_t stream) {
  DP_REQUIRE(y && (u8_nhwc || f32_nchw), DP_ERR_NULL);
  DP_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && ld >= C, DP_ERR_SHAPE);
  const long long total = (long long)N * H * W * C;
  long long b = (total + DI_NT - 1) / DI_NT;
  if (b > DP_NUM_SMS * 32) b = DP_NUM_SMS * 32;
  decode_images_kernel<<<(int)b, DI_NT, 0, (cudaStream_t)stream>>>(y, ld, N, C, H, W, u8_nhwc, f32_nchw);
  return dp_check_launch();
}
