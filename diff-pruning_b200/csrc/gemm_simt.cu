// gemm_simt.cu — fp32 SIMT implicit-GEMM core (CUDA cores, FFMA) for libdpb200.
//
// One templated kernel computes C[M,N] = alpha * A[M,K] x B[K,N] with 128x128x16 tiles, 256 threads, 8x8
// register micro-tiles and a register-prefetch + double-buffered shared-memory pipeline.  The A and B operand
// loaders are compile-time "modes": plain strided (k-contiguous / m|n-contiguous) or an on-the-fly im2col
// GATHER from an NHWC activation view, which turns the same kernel into conv fprop, dgrad and wgrad
// (split-K over pixels, fixed-order reduce => deterministic).  This is the exact-fp32 path: every shape the
// model can take after pruning runs here; the wgmma path (conv_tc.cu) takes over the big regular convs.
#include "common.cuh"

namespace {

constexpr int TM = 128, TN = 128, TK = 16, NTHREADS = 256;

enum { A_KC = 0, A_MC = 1, A_GATHER = 2 };
enum { B_KC = 0, B_NC = 1, B_GATHER = 2 };

struct Gather {
  const float* src;
  long long ld;
  int H, W, C;        // gathered tensor [*][H][W][C]
  int P, Q, PQ;       // pixel-index grid: pix -> (n, p, q)
  int S;              // filter width (tap -> (r, s))
  int sm, sr, off_h, off_w, sds;  // h_num = p*sm + r*sr + off_h ; valid iff (h_num & sds)==0 ; h = h_num >> sds
  int logQ, logPQ;    // >= 0 when Q / PQ are powers of two (fast path), else -1
};

struct GemmParams {
  int M, N, K;
  const float* A; long long a_rs, a_cs, a_bs;
  const float* B; long long b_rs, b_cs, b_bs;
  float* C; long long ldc, c_bs;
  float alpha;
  int accumulate;
  int k_per_split;  // > 0: blockIdx.z is a K-split writing C + z*c_bs ; == 0: blockIdx.z is a batch index
  const float* bias;
  const float* rowadd; long long ld_rowadd; int rows_per_img;
  const float* residual; long long ld_res;
  uint32_t* amax_out;   // optional amax slot of C
  Gather g;
};

template <int AM, int BMODE>
__global__ void __launch_bounds__(NTHREADS) gemm_simt_kernel(const GemmParams p) {
  __shared__ __align__(16) float As[2][TK][TM + 4];
  __shared__ __align__(16) float Bs[2][TK][TN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int z = blockIdx.z;
  int kbeg = 0, kend = p.K;
  const float* __restrict__ A = p.A;
  const float* __restrict__ B = p.B;
  float* __restrict__ C = p.C;
  if (p.k_per_split > 0) {
    kbeg = z * p.k_per_split;
    kend = min(p.K, kbeg + p.k_per_split);
    C += (long long)z * p.c_bs;
  } else {
    A += (long long)z * p.a_bs;
    B += (long long)z * p.b_bs;
    C += (long long)z * p.c_bs;
  }
  const Gather& g = p.g;

  // ---- per-thread operand-load coordinates ----
  // k-contiguous mapping: (k_local = tid & 15, row = (tid >> 4) + 16 j) ; m|n-contiguous: (row = tid & 127, k_local = (tid >> 7) + 2 j)
  const int kc_k = tid & 15, kc_r = tid >> 4;
  const int mc_r = tid & 127, mc_k = tid >> 7;

  // A gather: rows (pixels) are fixed for the whole kernel -> decompose once
  int a_gh[8], a_gw[8], a_gb[8];
  if (AM == A_GATHER) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int m = m0 + kc_r + 16 * j;
      if (m < p.M) {
        int n = m / g.PQ, rem = m - n * g.PQ;
        int pp = rem / g.Q, qq = rem - pp * g.Q;
        a_gh[j] = pp * g.sm + g.off_h;
        a_gw[j] = qq * g.sm + g.off_w;
        a_gb[j] = n * g.H * g.W;
      } else {
        a_gh[j] = -(1 << 28); a_gw[j] = 0; a_gb[j] = 0;
      }
    }
  }
  // B gather: column (tap, channel) fixed for the whole kernel
  int b_dh = 0, b_dw = 0, b_c = 0;
  bool b_nvalid = false;
  if (BMODE == B_GATHER) {
    int tc = n0 + mc_r;
    b_nvalid = tc < p.N;
    int tap = tc / g.C;
    b_c = tc - tap * g.C;
    int r = tap / g.S, s = tap - r * g.S;
    b_dh = r * g.sr + g.off_h;
    b_dw = s * g.sr + g.off_w;
  }

  float ra[8], rb[8];

  auto load_A = [&](int k0) {
    if (AM == A_KC) {
      int k = k0 + kc_k;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int m = m0 + kc_r + 16 * j;
        ra[j] = (m < p.M && k < kend) ? __ldg(A + (long long)m * p.a_rs + k) : 0.f;
      }
    } else if (AM == A_MC) {
      int m = m0 + mc_r;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int k = k0 + mc_k + 2 * j;
        ra[j] = (m < p.M && k < kend) ? __ldg(A + (long long)k * p.a_cs + m) : 0.f;
      }
    } else {
      int k = k0 + kc_k;
      bool kv = k < kend;
      int tap = kv ? k / g.C : 0;
      int c = k - tap * g.C;
      int r = tap / g.S, s = tap - r * g.S;
      int dh = r * g.sr, dw = s * g.sr;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int hn = a_gh[j] + dh, wn = a_gw[j] + dw;
        bool ok = kv && hn >= 0 && wn >= 0 && (((hn | wn) & g.sds) == 0);
        int h = hn >> g.sds, w = wn >> g.sds;
        ok = ok && h < g.H && w < g.W;
        ra[j] = ok ? __ldg(g.src + (long long)(a_gb[j] + h * g.W + w) * g.ld + c) : 0.f;
      }
    }
  };
  auto load_B = [&](int k0) {
    if (BMODE == B_KC) {
      int k = k0 + kc_k;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int n = n0 + kc_r + 16 * j;
        rb[j] = (n < p.N && k < kend) ? __ldg(B + (long long)n * p.b_cs + k) : 0.f;
      }
    } else if (BMODE == B_NC) {
      int n = n0 + mc_r;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int k = k0 + mc_k + 2 * j;
        rb[j] = (n < p.N && k < kend) ? __ldg(B + (long long)k * p.b_rs + n) : 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int pix = k0 + mc_k + 2 * j;
        bool ok = b_nvalid && pix < kend;
        int n, pp, qq;
        if (g.logPQ >= 0 && g.logQ >= 0) {
          n = pix >> g.logPQ;
          int rem = pix & (g.PQ - 1);
          pp = rem >> g.logQ;
          qq = rem & (g.Q - 1);
        } else {
          n = pix / g.PQ;
          int rem = pix - n * g.PQ;
          pp = rem / g.Q;
          qq = rem - pp * g.Q;
        }
        int hn = pp * g.sm + b_dh, wn = qq * g.sm + b_dw;
        ok = ok && hn >= 0 && wn >= 0 && (((hn | wn) & g.sds) == 0);
        int h = hn >> g.sds, w = wn >> g.sds;
        ok = ok && h < g.H && w < g.W;
        rb[j] = ok ? __ldg(g.src + ((long long)(n * g.H + h) * g.W + w) * g.ld + b_c) : 0.f;
      }
    }
  };
  auto store_AB = [&](int buf) {
    if (AM == A_MC) {
#pragma unroll
      for (int j = 0; j < 8; ++j) As[buf][mc_k + 2 * j][mc_r] = ra[j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) As[buf][kc_k][kc_r + 16 * j] = ra[j];
    }
    if (BMODE == B_KC) {
#pragma unroll
      for (int j = 0; j < 8; ++j) Bs[buf][kc_k][kc_r + 16 * j] = rb[j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) Bs[buf][mc_k + 2 * j][mc_r] = rb[j];
    }
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int tx = tid & 15, ty = tid >> 4;
  const int nk = (kend - kbeg + TK - 1) / TK;
  if (nk > 0) {
    load_A(kbeg);
    load_B(kbeg);
    store_AB(0);
  }
  __syncthreads();
  for (int t = 0; t < nk; ++t) {
    const int buf = t & 1;
    if (t + 1 < nk) {
      load_A(kbeg + (t + 1) * TK);
      load_B(kbeg + (t + 1) * TK);
    }
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (t + 1 < nk) store_AB(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue ----
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
    const float* radd = p.rowadd ? p.rowadd + (long long)(m / p.rows_per_img) * p.ld_rowadd : nullptr;
    const float* res = p.residual ? p.residual + (long long)m * p.ld_res : nullptr;
    float* crow = C + (long long)m * p.ldc;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n >= p.N) continue;
      float v = p.alpha * acc[i][j];
      if (p.bias) v += __ldg(p.bias + n);
      if (radd) v += __ldg(radd + n);
      if (res) v += __ldg(res + n);
      if (p.accumulate) v += crow[n];
      crow[n] = v;
      amax = fmaxf(amax, fabsf(v));
    }
  }
  if (p.amax_out) amax_commit(p.amax_out, amax);
}

template <int AM, int BMODE>
int launch_gemm(const GemmParams& p, int zdim, cudaStream_t st) {
  dim3 grid((p.M + TM - 1) / TM, (p.N + TN - 1) / TN, zdim);
  if (grid.y > 65535 || grid.z > 65535) return DP_ERR_SHAPE;
  gemm_simt_kernel<AM, BMODE><<<grid, NTHREADS, 0, st>>>(p);
  return dp_check_launch();
}

void clear_epilogue(GemmParams& p) {
  p.bias = nullptr; p.rowadd = nullptr; p.residual = nullptr; p.ld_rowadd = 0; p.ld_res = 0; p.rows_per_img = 1;
  p.k_per_split = 0; p.alpha = 1.f; p.accumulate = 0; p.amax_out = nullptr;
  p.a_bs = p.b_bs = p.c_bs = 0;
}

int validate_conv(const dp_conv_args* a) {
  DP_REQUIRE(a, DP_ERR_NULL);
  DP_REQUIRE(a->x && a->y, DP_ERR_NULL);
  DP_REQUIRE(a->N > 0 && a->H > 0 && a->W > 0 && a->C > 0 && a->P > 0 && a->Q > 0 && a->K > 0, DP_ERR_SHAPE);
  DP_REQUIRE(a->R > 0 && a->S > 0 && (a->stride == 1 || a->stride == 2), DP_ERR_SHAPE);
  DP_REQUIRE(a->pad_t >= 0 && a->pad_l >= 0, DP_ERR_SHAPE);
  DP_REQUIRE(a->ldx >= a->C && a->ldy >= a->K, DP_ERR_SHAPE);
  // every output pixel's window must start inside the padded input
  DP_REQUIRE((long long)(a->P - 1) * a->stride - a->pad_t < a->H, DP_ERR_SHAPE);
  DP_REQUIRE((long long)(a->Q - 1) * a->stride - a->pad_l < a->W, DP_ERR_SHAPE);
  DP_REQUIRE((long long)a->N * a->H * a->W < (1ll << 31) && (long long)a->N * a->P * a->Q < (1ll << 31), DP_ERR_SHAPE);
  DP_REQUIRE((long long)a->R * a->S * a->C < (1ll << 31), DP_ERR_SHAPE);
  return DP_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
int dp_conv2d_fprop_simt(const dp_conv_args* a, dp_stream_t stream) {
  int rc = validate_conv(a);
  if (rc) return rc;
  DP_REQUIRE(a->w, DP_ERR_NULL);
  GemmParams p{};
  clear_epilogue(p);
  p.M = a->N * a->P * a->Q; p.N = a->K; p.K = a->R * a->S * a->C;
  p.A = nullptr; p.a_rs = p.a_cs = 0;
  p.B = a->w; p.b_rs = a->K; p.b_cs = 1;
  p.C = (float*)a->y; p.ldc = a->ldy;
  p.accumulate = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  p.bias = a->bias; p.rowadd = a->rowadd; p.ld_rowadd = a->ld_rowadd; p.rows_per_img = a->P * a->Q;
  p.residual = a->residual; p.ld_res = a->ld_res;
  p.amax_out = a->amax_out;
  Gather& g = p.g;
  g.src = (const float*)a->x; g.ld = a->ldx; g.H = a->H; g.W = a->W; g.C = a->C;
  g.P = a->P; g.Q = a->Q; g.PQ = a->P * a->Q; g.S = a->S;
  g.sm = a->stride; g.sr = 1; g.off_h = -a->pad_t; g.off_w = -a->pad_l; g.sds = 0;
  g.logQ = ilog2_exact(g.Q); g.logPQ = ilog2_exact(g.PQ);
  return launch_gemm<A_GATHER, B_NC>(p, 1, (cudaStream_t)stream);
}

int dp_conv2d_dgrad_simt(const dp_conv_args* a, dp_stream_t stream) {
  int rc = validate_conv(a);
  if (rc) return rc;
  DP_REQUIRE(a->w, DP_ERR_NULL);
  GemmParams p{};
  clear_epilogue(p);
  // dx[n,h,w,c] = sum_{r,s,k} dy[n,(h+pad_t-r)/stride,(w+pad_l-s)/stride,k] * W[k,c,r,s]
  p.M = a->N * a->H * a->W; p.N = a->C; p.K = a->R * a->S * a->K;
  p.B = a->w; p.b_rs = a->C; p.b_cs = 1;  // packed [R*S][K][C]
  p.C = (float*)a->x; p.ldc = a->ldx;
  p.accumulate = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  p.amax_out = a->amax_out;
  Gather& g = p.g;
  g.src = (const float*)a->y; g.ld = a->ldy; g.H = a->P; g.W = a->Q; g.C = a->K;
  g.P = a->H; g.Q = a->W; g.PQ = a->H * a->W; g.S = a->S;
  g.sm = 1; g.sr = -1; g.off_h = a->pad_t; g.off_w = a->pad_l; g.sds = a->stride - 1;
  g.logQ = ilog2_exact(g.Q); g.logPQ = ilog2_exact(g.PQ);
  return launch_gemm<A_GATHER, B_NC>(p, 1, (cudaStream_t)stream);
}

int dp_conv2d_wgrad_simt(const dp_conv_args* a, dp_stream_t stream) {
  int rc = validate_conv(a);
  if (rc) return rc;
  DP_REQUIRE(a->workspace, DP_ERR_NULL);
  DP_REQUIRE(a->splits >= 1 && a->splits <= 65535, DP_ERR_SHAPE);
  GemmParams p{};
  clear_epilogue(p);
  // ws[z][k][(tap,c)] = sum_{pix in split z} dy[pix][k] * xcol[pix][(tap,c)]
  p.M = a->K; p.N = a->R * a->S * a->C; p.K = a->N * a->P * a->Q;
  p.A = (const float*)a->y; p.a_rs = 1; p.a_cs = a->ldy;  // A(m=k_out, k=pix) = dy[pix*ldy + k_out]
  p.C = a->workspace; p.ldc = p.N; p.c_bs = (long long)p.M * p.N;
  int kper = (p.K + a->splits - 1) / a->splits;
  kper = ((kper + TK - 1) / TK) * TK;
  p.k_per_split = kper;
  Gather& g = p.g;
  g.src = (const float*)a->x; g.ld = a->ldx; g.H = a->H; g.W = a->W; g.C = a->C;
  g.P = a->P; g.Q = a->Q; g.PQ = a->P * a->Q; g.S = a->S;
  g.sm = a->stride; g.sr = 1; g.off_h = -a->pad_t; g.off_w = -a->pad_l; g.sds = 0;
  g.logQ = ilog2_exact(g.Q); g.logPQ = ilog2_exact(g.PQ);
  rc = launch_gemm<A_MC, B_GATHER>(p, a->splits, (cudaStream_t)stream);
  if (rc || !a->bias_ws) return rc;
  // the column sums of dy the tensor-core kernel produces on the way: one column-sum segment per K split (the same pixel ranges)
  const int64_t rows = (int64_t)a->N * a->P * a->Q;
  const int64_t nseg = (rows + kper - 1) / kper;
  if (nseg < a->splits &&
      cudaMemsetAsync(a->bias_ws + nseg * a->K, 0, (size_t)(a->splits - nseg) * a->K * sizeof(float), (cudaStream_t)stream) != cudaSuccess)
    return dp_check_launch();
  return dp_colsum((const float*)a->y, a->ldy, rows, a->K, kper, a->bias_ws, a->K, 0, stream);
}

// ---------------------------------------------------------------------------------------------
extern "C" int dp_gemm_batched(const dp_gemm_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->A && a->B && a->C, DP_ERR_NULL);
  DP_REQUIRE(a->M > 0 && a->N > 0 && a->Kd > 0 && a->batch > 0 && a->batch <= 65535, DP_ERR_SHAPE);
  DP_REQUIRE((a->a_rs == 1 || a->a_cs == 1) && (a->b_rs == 1 || a->b_cs == 1), DP_ERR_UNSUPPORTED);
  GemmParams p{};
  clear_epilogue(p);
  p.M = a->M; p.N = a->N; p.K = a->Kd;
  p.A = a->A; p.a_rs = a->a_rs; p.a_cs = a->a_cs; p.a_bs = a->a_bs;
  p.B = a->B; p.b_rs = a->b_rs; p.b_cs = a->b_cs; p.b_bs = a->b_bs;
  p.C = a->C; p.ldc = a->ldc; p.c_bs = a->c_bs;
  p.alpha = a->alpha; p.accumulate = a->accumulate ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  bool a_kc = (a->a_cs == 1), b_nc = (a->b_cs == 1);
  if (a_kc && b_nc) return launch_gemm<A_KC, B_NC>(p, a->batch, st);
  if (a_kc && !b_nc) return launch_gemm<A_KC, B_KC>(p, a->batch, st);
  if (!a_kc && b_nc) return launch_gemm<A_MC, B_NC>(p, a->batch, st);
  return launch_gemm<A_MC, B_KC>(p, a->batch, st);
}

// ---------------------------------------------------------------------------------------------
// split-K reduce + scatter into the OIHW gradient (+ optional signed Taylor accumulation)
namespace {
// sum of the splits of one workspace element, in the fixed order every variant of this kernel has used: 4 interleaved accumulators,
// (s0 + s1) + (s2 + s3)
__device__ __forceinline__ float split_sum(const float* __restrict__ ws, long long split_stride, int splits) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int z = 0;
  for (; z + 4 <= splits; z += 4) {
    s0 += ws[(z + 0) * split_stride]; s1 += ws[(z + 1) * split_stride];
    s2 += ws[(z + 2) * split_stride]; s3 += ws[(z + 3) * split_stride];
  }
  for (; z < splits; ++z) s0 += ws[z * split_stride];
  return (s0 + s1) + (s2 + s3);
}
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const dp_wgrad_reduce_args a) {
  // block (x = chunk of 256 (tap,c) entries, y = output channel k): coalesced reads of every split, 4 splits in flight.  (One thread per
  // (k, c) writing the R*S contiguous gradient values was measured: better stores, but 9x fewer threads — slower on C1 / C3 weights.)
  const int k = blockIdx.y;
  const int RS = a.R * a.S, TC = RS * a.C;
  const long long split_stride = (long long)a.K * TC;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < TC) {
    const float s = split_sum(a.workspace + (long long)k * TC + i, split_stride, a.splits);
    const int tap = i / a.C, c = i - tap * a.C;
    const long long gi = ((long long)k * a.C + c) * RS + tap;
    a.dw[gi] += s;
    if (a.bias_ws && i == 0) {        // bias gradient: the per-split column sums of dy, summed in split order
      float b = 0.f;
      for (int z2 = 0; z2 < a.splits; ++z2) b += a.bias_ws[(long long)z2 * a.K + k];
      a.db[k] += b;
    }
    // signed first-order Taylor term of this pass, parked in the (already consumed) split-0 slot for the score kernels
    if (a.w && (a.score_out || a.score_in)) const_cast<float*>(a.workspace)[(long long)k * TC + i] = a.w[gi] * s;
  }
}
// R = S = 1 with 16-byte aligned rows (every nn.Linear, 1x1 convolution): the tensor is flat, 4 elements per thread
__global__ void __launch_bounds__(256) wgrad_reduce_flat4_kernel(const dp_wgrad_reduce_args a) {
  const long long n4 = (long long)a.K * a.C / 4, split_stride4 = n4;
  const bool scores = a.w && (a.score_out || a.score_in);
  const float4* ws = reinterpret_cast<const float4*>(a.workspace);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 s0 = make_float4(0, 0, 0, 0), s1 = s0, s2 = s0, s3 = s0;
    auto add = [](float4& acc, const float4 v) { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; };
    int z = 0;
    for (; z + 4 <= a.splits; z += 4) {
      add(s0, ws[(z + 0) * split_stride4 + i]); add(s1, ws[(z + 1) * split_stride4 + i]);
      add(s2, ws[(z + 2) * split_stride4 + i]); add(s3, ws[(z + 3) * split_stride4 + i]);
    }
    for (; z < a.splits; ++z) add(s0, ws[z * split_stride4 + i]);
    const float4 s = make_float4((s0.x + s1.x) + (s2.x + s3.x), (s0.y + s1.y) + (s2.y + s3.y), (s0.z + s1.z) + (s2.z + s3.z), (s0.w + s1.w) + (s2.w + s3.w));
    float4* dst = reinterpret_cast<float4*>(a.dw) + i;
    float4 d = *dst;
    d.x += s.x; d.y += s.y; d.z += s.z; d.w += s.w;
    *dst = d;
    if (scores) {
      const float4 w = reinterpret_cast<const float4*>(a.w)[i];
      const_cast<float4*>(ws)[i] = make_float4(w.x * s.x, w.y * s.y, w.z * s.z, w.w * s.w);
    }
  }
  if (a.bias_ws)
    for (long long k = blockIdx.x * 256ll + threadIdx.x; k < a.K; k += (long long)gridDim.x * 256) {
      float b = 0.f;
      for (int z2 = 0; z2 < a.splits; ++z2) b += a.bias_ws[(long long)z2 * a.K + k];
      a.db[k] += b;
    }
}
__global__ void wgrad_score_out_kernel(const dp_wgrad_reduce_args a) {
  // one block per output channel k: fixed-order sum over (tap, c) of W*dW_t
  const int k = blockIdx.x;
  const int TC = a.R * a.S * a.C;
  float s = 0.f;
  for (int i = threadIdx.x; i < TC; i += blockDim.x) s += a.workspace[(long long)k * TC + i];
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) a.score_out[k] += v;
  }
}
__global__ void wgrad_score_in_kernel(const dp_wgrad_reduce_args a) {
  // one block per input channel c: sum over (k, tap) of the W*dW_t terms left in workspace split 0
  const int c = blockIdx.x;
  const int RS = a.R * a.S, TC = RS * a.C;
  float s = 0.f;
  for (int i = threadIdx.x; i < a.K * RS; i += blockDim.x) {
    int k = i / RS, tap = i - k * RS;
    s += a.workspace[(long long)k * TC + tap * a.C + c];
  }
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) a.score_in[c] += v;
  }
}

__global__ void pack_weight_kernel(const float* __restrict__ w, int K, int C, int RS, float* __restrict__ w_ck,
                                   float* __restrict__ w_kc) {
  long long total = (long long)K * C * RS;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int tap = (int)(i % RS);
    long long kc = i / RS;
    int c = (int)(kc % C), k = (int)(kc / C);
    float v = w[i];
    if (w_ck) w_ck[((long long)tap * C + c) * K + k] = v;
    if (w_kc) w_kc[((long long)tap * K + k) * C + c] = v;
  }
}
}  // namespace

extern "C" int dp_conv2d_wgrad_reduce(const dp_wgrad_reduce_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->workspace && a->dw, DP_ERR_NULL);
  DP_REQUIRE((a->bias_ws == nullptr) == (a->db == nullptr), DP_ERR_NULL);
  DP_REQUIRE(a->K > 0 && a->C > 0 && a->R > 0 && a->S > 0 && a->splits >= 1, DP_ERR_SHAPE);
  cudaStream_t st = (cudaStream_t)stream;
  const int RS = a->R * a->S, TC = RS * a->C;
  const long long kc = (long long)a->K * a->C;
  if (RS == 1 && a->C % 4 == 0 && ((((uintptr_t)a->workspace) | ((uintptr_t)a->dw) | ((uintptr_t)a->w)) & 15) == 0) {
    // flat tensor (every nn.Linear / 1x1 convolution: most of the 400 M LDM parameters): 4 elements per thread, grid-stride
    long long blocks = (kc / 4 + 255) / 256;
    if (blocks > DP_NUM_SMS * 16) blocks = DP_NUM_SMS * 16;
    wgrad_reduce_flat4_kernel<<<(unsigned)(blocks < 1 ? 1 : blocks), 256, 0, st>>>(*a);
  } else {
    DP_REQUIRE(a->K <= 65535, DP_ERR_SHAPE);
    wgrad_reduce_kernel<<<dim3((TC + 255) / 256, a->K), 256, 0, st>>>(*a);
  }
  int rc = dp_check_launch();
  if (rc) return rc;
  if (a->w && a->score_out) {
    wgrad_score_out_kernel<<<a->K, 256, 0, st>>>(*a);
    if ((rc = dp_check_launch())) return rc;
  }
  if (a->w && a->score_in) {
    wgrad_score_in_kernel<<<a->C, 256, 0, st>>>(*a);
    rc = dp_check_launch();
  }
  return rc;
}

extern "C" int dp_pack_conv_weight(const float* w, int32_t K, int32_t C, int32_t R, int32_t S, float* w_ck,
                                   float* w_kc, dp_stream_t stream) {
  DP_REQUIRE(w && (w_ck || w_kc), DP_ERR_NULL);
  DP_REQUIRE(K > 0 && C > 0 && R > 0 && S > 0, DP_ERR_SHAPE);
  long long total = (long long)K * C * R * S;
  int blocks = (int)((total + 255) / 256);
  if (blocks > DP_NUM_SMS * 16) blocks = DP_NUM_SMS * 16;
  pack_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, K, C, R * S, w_ck, w_kc);
  return dp_check_launch();
}
