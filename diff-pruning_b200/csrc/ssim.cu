// ssim.cu — SSIM evaluation (compute_ssim.py / pytorch_msssim.ssim): per image pair, the mean SSIM map of every channel and the sum of
// squared differences, in one fused launch.  Filtered moments and the map are fp64; every sum runs in a fixed order and an image's
// results come from its own blocks only, so they are run-to-run identical and independent of the rest of the batch.
#include "common.cuh"
#include "image_src.cuh"

namespace {
constexpr int WIN = DP_SSIM_WIN, HALO = WIN - 1;
// A tile is 32 input columns (one per lane) by IH input rows; it yields TW x TH map values.  Each of the 8 warps filters RPW map rows.
constexpr int NWARP = 8, NT = 32 * NWARP, RPW = 3;
constexpr int IW = 32, TW = IW - HALO, TH = RPW * NWARP, IH = TH + HALO;
constexpr int NMOM = 5;   // mu_x, mu_y, E[x^2], E[y^2], E[xy]

struct SsimParams {
  const void* x; const void* y;
  int C, H, W;
  double g[WIN];
  double c1, c2;
  double* ssim_nc; double* sse_n;
};

template <int FMT>
__device__ __forceinline__ float src(const SsimParams& p, const void* s, int n, int c, int h, int w) {
  return dp_image_src(s, FMT == DP_SSIM_U8_NHWC, FMT == DP_SSIM_F32_NCHW_PNG, n, c, h, w, p.C, p.H, p.W);
}

// Sum of v over the block, in a fixed order (xor-butterfly within warps, then warps in index order); the result is valid in thread 0.
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum_d(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < NWARP; ++i) s += red[i];
  __syncthreads();
  return s;
}

// Block (n, c): channel c of pair n, walking the map in TW x TH tiles in a fixed order.  Per tile: the input tile with its halo in
// shared memory (fp32), the window along H into five fp64 moment rows per column (lane = column, RPW rows per warp), the window along W
// over those rows (lane = map column), the map value in fp64.  Block (n, 0) also sums (x - y)^2 over all channels of pair n.
template <int FMT>
__global__ void __launch_bounds__(NT, 2) ssim_kernel(const SsimParams p) {
  __shared__ float sx[IH][IW], sy[IH][IW];
  __shared__ double sv[NMOM][TH][IW];
  __shared__ double red[NWARP];
  const int n = blockIdx.x, c = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Ho = p.H - HALO, Wo = p.W - HALO;
  double part = 0.0;
  for (int th0 = 0; th0 < Ho; th0 += TH) {
    for (int tw0 = 0; tw0 < Wo; tw0 += TW) {
      for (int e = threadIdx.x; e < IH * IW; e += NT) {
        const int r = e / IW, q = e % IW, h = th0 + r, w = tw0 + q;
        const bool in = h < p.H && w < p.W;      // the zeros only reach map values outside the valid region, which are skipped
        sx[r][q] = in ? src<FMT>(p, p.x, n, c, h, w) : 0.0f;
        sy[r][q] = in ? src<FMT>(p, p.y, n, c, h, w) : 0.0f;
      }
      __syncthreads();
      {
        // along H: x^2, y^2, xy of fp32 values are exact in fp64, as is g x for the fp32 taps pytorch_msssim uses; the running sums round
        double acc[RPW][NMOM];
#pragma unroll
        for (int j = 0; j < RPW; ++j)
#pragma unroll
          for (int m = 0; m < NMOM; ++m) acc[j][m] = 0.0;
#pragma unroll
        for (int i = 0; i < RPW + HALO; ++i) {
          const double xv = sx[warp * RPW + i][lane], yv = sy[warp * RPW + i][lane];
#pragma unroll
          for (int j = 0; j < RPW; ++j) {
            const int k = i - j;
            if (k < 0 || k >= WIN) continue;
            const double gx = __dmul_rn(p.g[k], xv), gy = __dmul_rn(p.g[k], yv);
            acc[j][0] = __dadd_rn(acc[j][0], gx);
            acc[j][1] = __dadd_rn(acc[j][1], gy);
            acc[j][2] = fma(gx, xv, acc[j][2]);
            acc[j][3] = fma(gy, yv, acc[j][3]);
            acc[j][4] = fma(gx, yv, acc[j][4]);
          }
        }
#pragma unroll
        for (int j = 0; j < RPW; ++j)
#pragma unroll
          for (int m = 0; m < NMOM; ++m) sv[m][warp * RPW + j][lane] = acc[j][m];
      }
      __syncthreads();
      if (lane < TW) {
#pragma unroll
        for (int j = 0; j < RPW; ++j) {
          const int r = warp * RPW + j;
          double mo[NMOM];
#pragma unroll
          for (int m = 0; m < NMOM; ++m) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < WIN; ++k) s = fma(p.g[k], sv[m][r][lane + k], s);
            mo[m] = s;
          }
          if (th0 + r < Ho && tw0 + lane < Wo) {
            // explicit roundings: no contraction, so an image scored against itself gives exactly 1 (numerators equal denominators)
            const double mxx = __dmul_rn(mo[0], mo[0]), myy = __dmul_rn(mo[1], mo[1]), mxy = __dmul_rn(mo[0], mo[1]);
            const double sxx = __dsub_rn(mo[2], mxx), syy = __dsub_rn(mo[3], myy), sxy = __dsub_rn(mo[4], mxy);
            const double cs = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, sxy), p.c2), __dadd_rn(__dadd_rn(sxx, syy), p.c2));
            const double l = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, mxy), p.c1), __dadd_rn(__dadd_rn(mxx, myy), p.c1));
            part = __dadd_rn(part, __dmul_rn(l, cs));
          }
        }
      }
      __syncthreads();
    }
  }
  const double total = block_sum(part, red);
  if (threadIdx.x == 0) p.ssim_nc[(long long)n * p.C + c] = total / ((double)Ho * (double)Wo);
  if (c != 0) return;
  // squared error of the whole pair, summed in (c, h, w) order whatever the source layout, so that every format gives the same bits
  // for the same values; the difference rounds in fp32 as F.mse_loss forms it, its square is exact in fp64
  const long long HW = (long long)p.H * p.W, tot = HW * p.C;
  double sse = 0.0;
  for (long long e = threadIdx.x; e < tot; e += NT) {
    const int cc = (int)(e / HW);
    const long long px = e % HW;
    const int h = (int)(px / p.W), w = (int)(px % p.W);
    const double d = (double)__fsub_rn(src<FMT>(p, p.x, n, cc, h, w), src<FMT>(p, p.y, n, cc, h, w));
    sse = fma(d, d, sse);
  }
  const double s = block_sum(sse, red);
  if (threadIdx.x == 0) p.sse_n[n] = s;
}
}  // namespace

extern "C" int dp_ssim(const dp_ssim_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->x && a->y && a->ssim_nc && a->sse_n, DP_ERR_NULL);
  DP_REQUIRE(a->win_size == DP_SSIM_WIN, DP_ERR_UNSUPPORTED);
  DP_REQUIRE(a->N > 0 && a->C > 0 && a->C <= 65535 && a->H >= DP_SSIM_WIN && a->W >= DP_SSIM_WIN, DP_ERR_SHAPE);
  SsimParams p;
  p.x = a->x, p.y = a->y, p.C = a->C, p.H = a->H, p.W = a->W;
  for (int k = 0; k < WIN; ++k) p.g[k] = a->win[k];
  p.c1 = a->c1, p.c2 = a->c2, p.ssim_nc = a->ssim_nc, p.sse_n = a->sse_n;
  const dim3 grid(a->N, a->C);
  cudaStream_t s = (cudaStream_t)stream;
  switch (a->format) {
    case DP_SSIM_U8_NHWC: ssim_kernel<DP_SSIM_U8_NHWC><<<grid, NT, 0, s>>>(p); break;
    case DP_SSIM_F32_NCHW: ssim_kernel<DP_SSIM_F32_NCHW><<<grid, NT, 0, s>>>(p); break;
    case DP_SSIM_F32_NCHW_PNG: ssim_kernel<DP_SSIM_F32_NCHW_PNG><<<grid, NT, 0, s>>>(p); break;
    default: return DP_ERR_UNSUPPORTED;
  }
  return dp_check_launch();
}
