// fid.cu — the Inception-v3 feature pass of FID evaluation around its convolutions: the resize / normalise front end, the 3 x 3 pools,
// the global mean, and fp64 feature moments.  Every sum runs in a fixed order, so features and moments are run-to-run identical.
#include <math.h>
#include "common.cuh"
#include "image_src.cuh"

namespace {
constexpr int NT = 256;
static inline int nblocks(long long n, int cap = DP_NUM_SMS * 32) {
  long long b = (n + NT - 1) / NT;
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}

// One RGB source value in [0, 1] (image_src.cuh)
__device__ __forceinline__ float fid_src(const void* src, int u8, int quantize, int n, int c, int h, int w, int Hs, int Ws) {
  return dp_image_src(src, u8, quantize, n, c, h, w, 3, Hs, Ws);
}

// one thread per output pixel (all three channels)
__global__ void fid_input_kernel(const void* __restrict__ src, int u8, int quantize, int N, int Hs, int Ws, float* __restrict__ out, long long ld,
                                 int Ho, int Wo, int resize, int normalize, uint32_t* __restrict__ amax_out) {
  float amax = 0.f;
  const long long total = (long long)N * Ho * Wo;
  // torch's scale for align_corners = False without a scale factor: input / output in fp32
  const float sh = (float)Hs / (float)Ho, sw = (float)Ws / (float)Wo;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    const int ow = (int)(i % Wo);
    const long long t = i / Wo;
    const int oh = (int)(t % Ho), n = (int)(t / Ho);
    float* o = out + i * ld;
    if (!resize) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = fid_src(src, u8, quantize, n, c, oh, ow, Hs, Ws);
        o[c] = normalize ? __fsub_rn(__fmul_rn(2.0f, v), 1.0f) : v;
        amax = fmaxf(amax, fabsf(o[c]));
      }
      continue;
    }
    // source index = scale * (dst + 0.5) - 0.5, clamped at 0; the far neighbour is the same pixel on the last row / column
    const float hr = fmaxf(sh * ((float)oh + 0.5f) - 0.5f, 0.0f), wr = fmaxf(sw * ((float)ow + 0.5f) - 0.5f, 0.0f);
    const int h0 = (int)hr, w0 = (int)wr;
    const int h1 = h0 + (h0 < Hs - 1 ? 1 : 0), w1 = w0 + (w0 < Ws - 1 ? 1 : 0);
    const float lh1 = hr - (float)h0, lh0 = 1.0f - lh1, lw1 = wr - (float)w0, lw0 = 1.0f - lw1;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v00 = fid_src(src, u8, quantize, n, c, h0, w0, Hs, Ws), v01 = fid_src(src, u8, quantize, n, c, h0, w1, Hs, Ws);
      const float v10 = fid_src(src, u8, quantize, n, c, h1, w0, Hs, Ws), v11 = fid_src(src, u8, quantize, n, c, h1, w1, Hs, Ws);
      const float v = lh0 * (lw0 * v00 + lw1 * v01) + lh1 * (lw0 * v10 + lw1 * v11);
      o[c] = normalize ? __fsub_rn(__fmul_rn(2.0f, v), 1.0f) : v;
      amax = fmaxf(amax, fabsf(o[c]));
    }
  }
  if (amax_out) amax_commit(amax_out, amax);
}

// one thread per output element (n, p, q, c), channels fastest: coalesced reads of every tap
__global__ void pool3x3_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ y, long long ldy, int N, int H, int W, int C,
                               int P, int Q, int stride, int pad, int mode, uint32_t* __restrict__ amax_out) {
  const long long total = (long long)N * P * Q * C;
  float amax = 0.f;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int q = (int)(pix % Q);
    const long long t = pix / Q;
    const int p = (int)(t % P), n = (int)(t / P);
    const int h0 = max(p * stride - pad, 0), h1 = min(p * stride - pad + 3, H);
    const int w0 = max(q * stride - pad, 0), w1 = min(q * stride - pad + 3, W);
    const float* xb = x + ((long long)n * H * W) * ldx + c;
    float acc = mode == 0 ? -INFINITY : 0.0f;
    for (int h = h0; h < h1; ++h)
      for (int w = w0; w < w1; ++w) {
        const float v = __ldg(xb + ((long long)h * W + w) * ldx);
        acc = mode == 0 ? fmaxf(acc, v) : acc + v;
      }
    const float v = mode == 0 ? acc : acc / (float)((h1 - h0) * (w1 - w0));
    y[pix * ldy + c] = v;
    amax = fmaxf(amax, fabsf(v));
  }
  if (amax_out) amax_commit(amax_out, amax);
}

// The sum runs in fp64: the maps it averages are post-ReLU (all terms of one sign), where a running fp32 sum of H*W terms loses about
// sqrt(H*W) ulps (73 x 73 maps: ~2e-6 relative); in fp64 the mean is the fp32 rounding of the exact mean, up to 2^-53 H*W.
__global__ void global_mean_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ y, long long ldy, int N, int H, int W, int C) {
  const long long total = (long long)N * C;
  const int HW = H * W;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    const int c = (int)(i % C), n = (int)(i / C);
    const float* xb = x + (long long)n * HW * ldx + c;
    double s = 0.0;
    for (int k = 0; k < HW; ++k) s += (double)__ldg(xb + (long long)k * ldx);
    y[(long long)n * ldy + c] = (float)(s / (double)HW);
  }
}

// Block (bi, bj), bj >= bi: the 32 x 32 tile of sxx with rows 32 bi.., columns 32 bj..; thread (tx, ty) owns column 32 bj + tx and rows
// 32 bi + ty + 8 k.  Rows of f stream through shared memory 32 at a time and every thread adds them in index order.  Products of two
// fp32 values are exact in fp64 (and so are their differences with an fp32 shift), so only the products and running sums round.
constexpr int MT = 32, MR = 32;
__global__ void __launch_bounds__(256) moments_kernel(const float* __restrict__ f, long long ld, long long rows, int D,
                                                      const float* __restrict__ shift, double* __restrict__ sum, double* __restrict__ sxx) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj < bi) return;
  __shared__ double fi[MR][MT], fj[MR][MT];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  double acc[4] = {0.0, 0.0, 0.0, 0.0}, s = 0.0;
  for (long long r0 = 0; r0 < rows; r0 += MR) {
    for (int e = threadIdx.x; e < MR * MT; e += 256) {
      const int rr = e / MT, cc = e % MT;
      const long long r = r0 + rr;
      const int ci = bi * MT + cc, cj = bj * MT + cc;
      fi[rr][cc] = (r < rows && ci < D) ? (double)__ldg(f + r * ld + ci) - (shift ? (double)__ldg(shift + ci) : 0.0) : 0.0;
      fj[rr][cc] = (r < rows && cj < D) ? (double)__ldg(f + r * ld + cj) - (shift ? (double)__ldg(shift + cj) : 0.0) : 0.0;
    }
    __syncthreads();
    const int nr = (int)min((long long)MR, rows - r0);
    for (int rr = 0; rr < nr; ++rr) {
      const double vj = fj[rr][tx];
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] = fma(fi[rr][ty + 8 * k], vj, acc[k]);
      s += vj;
    }
    __syncthreads();
  }
  const int j = bj * MT + tx;
  if (j >= D) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = bi * MT + ty + 8 * k;
    if (i <= j) sxx[(long long)i * D + j] += acc[k];
  }
  if (bi == bj && ty == 0) sum[j] += s;
}
}  // namespace

extern "C" int dp_fid_input(const void* src, int32_t src_u8, int32_t quantize, int32_t N, int32_t Hs, int32_t Ws, float* out, int64_t ld_out,
                            int32_t Ho, int32_t Wo, int32_t resize, int32_t normalize, uint32_t* amax_out, dp_stream_t stream) {
  DP_REQUIRE(src && out, DP_ERR_NULL);
  DP_REQUIRE(N > 0 && Hs > 0 && Ws > 0 && Ho > 0 && Wo > 0 && ld_out >= 3, DP_ERR_SHAPE);
  DP_REQUIRE(resize || (Ho == Hs && Wo == Ws), DP_ERR_SHAPE);
  DP_REQUIRE(!(src_u8 && quantize), DP_ERR_UNSUPPORTED);
  fid_input_kernel<<<nblocks((long long)N * Ho * Wo), NT, 0, (cudaStream_t)stream>>>(src, src_u8 ? 1 : 0, quantize ? 1 : 0, N, Hs, Ws, out,
                                                                                      ld_out, Ho, Wo, resize ? 1 : 0, normalize ? 1 : 0, amax_out);
  return dp_check_launch();
}

extern "C" int dp_pool3x3(const float* x, int64_t ldx, float* y, int64_t ldy, int32_t N, int32_t H, int32_t W, int32_t C, int32_t stride,
                          int32_t pad, int32_t mode, uint32_t* amax_out, dp_stream_t stream) {
  DP_REQUIRE(x && y, DP_ERR_NULL);
  DP_REQUIRE(N > 0 && C > 0 && ldx >= C && ldy >= C && (stride == 1 || stride == 2) && pad >= 0 && pad <= 1, DP_ERR_SHAPE);
  DP_REQUIRE(mode == 0 || mode == 1, DP_ERR_UNSUPPORTED);
  DP_REQUIRE(H + 2 * pad >= 3 && W + 2 * pad >= 3, DP_ERR_SHAPE);
  const int P = (H + 2 * pad - 3) / stride + 1, Q = (W + 2 * pad - 3) / stride + 1;
  pool3x3_kernel<<<nblocks((long long)N * P * Q * C), NT, 0, (cudaStream_t)stream>>>(x, ldx, y, ldy, N, H, W, C, P, Q, stride, pad, mode, amax_out);
  return dp_check_launch();
}

extern "C" int dp_global_mean(const float* x, int64_t ldx, float* y, int64_t ldy, int32_t N, int32_t H, int32_t W, int32_t C, dp_stream_t stream) {
  DP_REQUIRE(x && y, DP_ERR_NULL);
  DP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && ldx >= C && ldy >= C, DP_ERR_SHAPE);
  global_mean_kernel<<<nblocks((long long)N * C), NT, 0, (cudaStream_t)stream>>>(x, ldx, y, ldy, N, H, W, C);
  return dp_check_launch();
}

extern "C" int dp_feature_moments(const float* f, int64_t ld, int64_t rows, int32_t D, const float* shift, double* sum, double* sxx,
                                  dp_stream_t stream) {
  DP_REQUIRE(f && sum && sxx, DP_ERR_NULL);
  DP_REQUIRE(rows >= 0 && D > 0 && ld >= D, DP_ERR_SHAPE);
  if (rows == 0) return DP_OK;
  const int nt = (D + MT - 1) / MT;
  moments_kernel<<<dim3(nt, nt), 256, 0, (cudaStream_t)stream>>>(f, ld, rows, D, shift, sum, sxx);
  return dp_check_launch();
}
