// pointwise.cu — small fused elementwise / reduction kernels of the Taylor-scoring and finetune path.
// All are HBM- or latency-bound; sums are two-stage with fixed order (deterministic, no atomics); the one atomic is the max of dp_amax,
// which is order-independent.
#include "common.cuh"

namespace {
constexpr int NT = 256;
static inline int nblocks(long long n, int per_block, int cap = DP_NUM_SMS * 32) {
  long long b = (n + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}

// max |x| over a [rows][cols] view, accumulated into an "amax slot" as the BIT PATTERN of the float (monotone for non-negative floats):
// atomicMax on it is order-independent, so the slot — and everything scaled by it — is run-to-run identical although blocks race.
__global__ void amax_kernel(const float* __restrict__ x, long long ld, long long rows, long long cols, int vec, uint32_t* __restrict__ slot) {
  float m = 0.f;
  if (vec) {
    const long long c4 = cols >> 2, total = rows * c4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
      const long long r = i / c4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ld + ((i - r * c4) << 2)));
      m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
  } else {
    const long long total = rows * cols;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
      const long long r = i / cols;
      m = fmaxf(m, fabsf(__ldg(x + r * ld + (i - r * cols))));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(slot, __float_as_uint(m));
}
__global__ void zero_u32_kernel(uint32_t* __restrict__ p, long long n) {
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) p[i] = 0u;
}

__global__ void silu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
    float v = x[i];
    y[i] = v * sigmoidf_acc(v);
  }
}
__global__ void silu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                                long long n, int acc) {
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
    float v = x[i], s = sigmoidf_acc(v);
    float g = dy[i] * s * (1.f + v * (1.f - s));
    dx[i] = acc ? dx[i] + g : g;
  }
}
// GEGLU (ldm/modules/attention.py:37-44): u = [a | gate] per row, out = a * gelu(gate), gelu = exact erf form (F.gelu default)
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * expf(-0.5f * x * x);
}
__global__ void geglu_fwd_kernel(const float* __restrict__ u, long long ldu, float* __restrict__ out, long long ldo, long long rows, int I) {
  const long long total = rows * I;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    const long long r = i / I; const int c = (int)(i - r * I);
    const float a = u[r * ldu + c], g = u[r * ldu + I + c];
    out[r * ldo + c] = a * gelu_erf(g);
  }
}
__global__ void geglu_bwd_kernel(const float* __restrict__ u, long long ldu, const float* __restrict__ dout, long long lddo,
                                 float* __restrict__ du, long long lddu, long long rows, int I) {
  const long long total = rows * I;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    const long long r = i / I; const int c = (int)(i - r * I);
    const float a = u[r * ldu + c], g = u[r * ldu + I + c], d = dout[r * lddo + c];
    du[r * lddu + c] = d * gelu_erf(g);
    du[r * lddu + I + c] = d * a * gelu_erf_grad(g);
  }
}
__global__ void temb_kernel(const int64_t* __restrict__ t, const float* __restrict__ freqs, float* __restrict__ out,
                            int B, int half, int flip) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  int b = i / half, k = i - b * half;
  float arg = (float)t[b] * freqs[k];
  float s = sinf(arg), c = cosf(arg);
  float* o = out + (long long)b * 2 * half;
  if (flip) { o[k] = c; o[half + k] = s; } else { o[k] = s; o[half + k] = c; }
}
__global__ void add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ nz, const int64_t* __restrict__ t,
                                 const float* __restrict__ acp, float* __restrict__ out, int B, int C, int HW, int nhwc, long long ld) {
  long long total = (long long)B * C * HW;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int hw = (int)(i % HW);
    long long bc = i / HW;
    int c = (int)(bc % C), b = (int)(bc / C);
    float ac = acp[t[b]];
    float v = sqrtf(ac) * x0[i] + sqrtf(1.0f - ac) * nz[i];
    if (nhwc) out[((long long)b * HW + hw) * ld + c] = v; else out[i] = v;
  }
}
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, long long ld, int N, int C, int HW) {
  long long total = (long long)N * HW * C;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int c = (int)(i % C);
    long long np = i / C;
    int hw = (int)(np % HW), n = (int)(np / HW);
    out[np * ld + c] = in[((long long)n * C + c) * HW + hw];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, long long ld, float* __restrict__ out, int N, int C, int HW, int acc) {
  long long total = (long long)N * HW * C;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int hw = (int)(i % HW);
    long long nc = i / HW;
    int c = (int)(nc % C), n = (int)(nc / C);
    float v = in[((long long)n * HW + hw) * ld + c];
    out[i] = acc ? out[i] + v : v;
  }
}
constexpr int MSE_PER_BLOCK = 4096;
__global__ void mse_stage1_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, float* __restrict__ grad,
                                  long long n, float sg, float* __restrict__ partial) {
  long long base = (long long)blockIdx.x * MSE_PER_BLOCK;
  float s = 0.f;
  for (int j = threadIdx.x; j < MSE_PER_BLOCK; j += NT) {
    long long i = base + j;
    if (i < n) { float d = pred[i] - tgt[i]; s += d * d; if (grad) grad[i] = sg * d; }
  }
  __shared__ float red[NT / 32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < NT / 32; ++w) t += red[w]; partial[blockIdx.x] = t; }
}
__global__ void sum_stage2_kernel(const float* __restrict__ partial, long long nb, float scale, float* __restrict__ out) {
  __shared__ double red[NT];
  double s = 0;
  for (long long i = threadIdx.x; i < nb; i += NT) s += partial[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) out[0] = (float)(red[0] * (double)scale);
}
__global__ void upsample_fwd_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ y, long long ldy, int N, int H, int W, int C) {
  long long total = (long long)N * 4 * H * W * C;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int c = (int)(i % C);
    long long p = i / C;
    int ow = (int)(p % (2 * W));
    long long q = p / (2 * W);
    int oh = (int)(q % (2 * H)), n = (int)(q / (2 * H));
    y[p * ldy + c] = x[(((long long)n * H + (oh >> 1)) * W + (ow >> 1)) * ldx + c];
  }
}
__global__ void upsample_bwd_kernel(const float* __restrict__ dy, long long lddy, float* __restrict__ dx, long long lddx, int N, int H, int W, int C, int acc) {
  long long total = (long long)N * H * W * C;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int c = (int)(i % C);
    long long p = i / C;
    int w = (int)(p % W);
    long long q = p / W;
    int h = (int)(q % H), n = (int)(q / H);
    long long r0 = ((long long)n * 2 * H + 2 * h) * (2 * W) + 2 * w;
    float s = dy[r0 * lddy + c] + dy[(r0 + 1) * lddy + c] + dy[(r0 + 2 * W) * lddy + c] + dy[(r0 + 2 * W + 1) * lddy + c];
    dx[p * lddx + c] = acc ? dx[p * lddx + c] + s : s;
  }
}
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, long long ld, long long rows, int cols, long long seg_rows,
                                                     float* __restrict__ out, long long ld_out, int acc, int vec) {
  // grid (nseg, ceil(cols/64)), block (16 column quads, 16 row lanes): float4 loads (vec: 16-byte aligned rows), four independent rows in
  // flight per thread, fixed-order tree over the 16 lanes (deterministic)
  __shared__ float red[16][64];
  const long long seg = blockIdx.x;
  const int qx = threadIdx.x, ly = threadIdx.y;
  const int c0 = blockIdx.y * 64 + qx * 4;
  long long r0 = seg * seg_rows, r1 = r0 + seg_rows;
  if (r1 > rows) r1 = rows;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (vec && c0 + 4 <= cols) {
#pragma unroll 4
    for (long long r = r0 + ly; r < r1; r += 16) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ld + c0));
      s0 += v.x; s1 += v.y; s2 += v.z; s3 += v.w;
    }
  } else if (c0 < cols) {
    for (long long r = r0 + ly; r < r1; r += 16) {
      const float* row = x + r * ld + c0;
      s0 += __ldg(row);
      if (c0 + 1 < cols) s1 += __ldg(row + 1);
      if (c0 + 2 < cols) s2 += __ldg(row + 2);
      if (c0 + 3 < cols) s3 += __ldg(row + 3);
    }
  }
  red[ly][qx * 4 + 0] = s0; red[ly][qx * 4 + 1] = s1; red[ly][qx * 4 + 2] = s2; red[ly][qx * 4 + 3] = s3;
  __syncthreads();
  const int t = ly * 16 + qx;          // threads 0..63 finish one column each
  if (t < 64) {
    const int c = blockIdx.y * 64 + t;
    if (c < cols) {
      float tot = 0.f;
#pragma unroll
      for (int l = 0; l < 16; ++l) tot += red[l][t];
      float* o = out + seg * ld_out + c;
      *o = acc ? *o + tot : tot;
    }
  }
}
__global__ void add_views_kernel(const float* __restrict__ a, long long lda, const float* __restrict__ b, long long ldb,
                                 float* __restrict__ y, long long ldy, long long rows, int cols) {
  long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int c = (int)(i % cols);
    long long r = i / cols;
    y[r * ldy + c] = a[r * lda + c] + b[r * ldb + c];
  }
}
__global__ void copy_rows_kernel(const float* __restrict__ a, long long lda, float* __restrict__ y, long long ldy, long long rows, int cols) {
  long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
    int c = (int)(i % cols);
    long long r = i / cols;
    y[r * ldy + c] = a[r * lda + c];
  }
}
// s and p may be one buffer (the engine normalises the attention scores in place): no __restrict__, so the loads stay coherent
// (LDG.E, not ld.global.nc), and lane j reads in[j] before it writes out[j] of its own row
__global__ void softmax_fwd_kernel(const float* s, float* p, long long rows, int cols) {
  long long row = blockIdx.x * (long long)(NT / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  int lane = threadIdx.x & 31;
  const float* in = s + row * cols;
  float* out = p + row * cols;
  float mx = -INFINITY;
  for (int j = lane; j < cols; j += 32) mx = fmaxf(mx, in[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < cols; j += 32) sum += expf(in[j] - mx);
  sum = warp_sum(sum);
  float inv = 1.0f / sum;
  for (int j = lane; j < cols; j += 32) out[j] = expf(in[j] - mx) * inv;
}
// dp and ds may be one buffer (in place, as the engine runs it): no operand is __restrict__, so every load stays coherent; lane j reads dr[j]
// in both passes before it writes o[j]
__global__ void softmax_bwd_kernel(const float* p, const float* dp, float* ds, long long rows, int cols,
                                   uint32_t* __restrict__ amax_ds) {
  __shared__ float wmax[NT / 32];
  const long long row = blockIdx.x * (long long)(NT / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  float amax = 0.f;
  if (row < rows) {
    const float* pr = p + row * cols;
    const float* dr = dp + row * cols;
    float* o = ds + row * cols;
    float dot = 0.f;
    for (int j = lane; j < cols; j += 32) dot += pr[j] * dr[j];
    dot = warp_sum(dot);
    for (int j = lane; j < cols; j += 32) {
      const float v = pr[j] * (dr[j] - dot);
      o[j] = v;
      amax = fmaxf(amax, fabsf(v));
    }
  }
  if (amax_ds) {      // one atomic per block (a row per warp would serialise tens of thousands of them on one address)
    amax = warp_max(amax);
    if (lane == 0) wmax[threadIdx.x >> 5] = amax;
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = 0.f;
      for (int i = 0; i < NT / 32; ++i) m = fmaxf(m, wmax[i]);
      if (m > 0.f) atomicMax(amax_ds, __float_as_uint(m));
    }
  }
}
// The DDIM update of one element, shared by both samplers: x0 = (x - sb e) / sa, then sap x0 + dir e (+ sigma nz).  kRn: every operation
// rounded on its own (no fma contraction), in the order torch evaluates p_sample_ddim (ddim.py:194-202), so the result is bit-identical to
// that fp32 torch code; otherwise the compiler may contract, as dp_ddim_step always has.
template <bool kRn>
__device__ __forceinline__ float ddim_x0(float x, float e, float sb, float sa) {
  if (kRn) return __fdiv_rn(__fsub_rn(x, __fmul_rn(sb, e)), sa);
  return (x - sb * e) / sa;
}
template <bool kRn>
__device__ __forceinline__ float ddim_prev(float x0, float e, float sap, float dir, bool has_nz, float sigma, float nz) {
  if (kRn) {
    float v = __fadd_rn(__fmul_rn(sap, x0), __fmul_rn(dir, e));
    return has_nz ? __fadd_rn(v, __fmul_rn(sigma, nz)) : v;
  }
  float v = sap * x0 + dir * e;
  if (has_nz) v += sigma * nz;
  return v;
}
__global__ void ddim_step_kernel(const float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ nz,
                                 float* __restrict__ out, long long n, float sb, float sa, float clip, float sap, float dir, float sigma) {
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
    float e = eps[i];
    float x0 = ddim_x0<false>(x[i], e, sb, sa);
    if (clip > 0.f) x0 = fminf(fmaxf(x0, -clip), clip);
    out[i] = ddim_prev<false>(x0, e, sap, dir, nz != nullptr, sigma, nz ? nz[i] : 0.f);
  }
}
// Guided DDIM step of the LDM sampler over the NCHW state x [B][C][HW]: eps_hat is read from the UNet's NHWC output (pixel stride ld_eps),
// images 0..B-1 unconditional and B..2B-1 conditional when guided (e = e_u + s (e_c - e_u)), images 0..B-1 as is otherwise.  x_prev goes
// to x_out (NCHW) and to the UNet's NHWC input (pixel stride ld_in), into both halves when guided; pred_x0 (NCHW) when asked for.
__global__ void ddim_cfg_step_kernel(const float* __restrict__ eps, long long ld_eps, const float* __restrict__ x, const float* __restrict__ nz,
                                     float* __restrict__ x_out, float* __restrict__ x_in, long long ld_in, float* __restrict__ pred_x0,
                                     int B, int C, int HW, int guided, float scale, float sb, float sa, float sap, float dir, float sigma) {
  const long long n = (long long)B * C * HW, half_eps = (long long)B * HW * ld_eps, half_in = (long long)B * HW * ld_in;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
    const int c = (int)((i / HW) % C);
    const long long pix = (i / ((long long)C * HW)) * HW + i % HW;       // image * HW + pixel
    float e = eps[pix * ld_eps + c];
    if (guided) e = __fadd_rn(e, __fmul_rn(scale, __fsub_rn(eps[half_eps + pix * ld_eps + c], e)));
    const float x0 = ddim_x0<true>(x[i], e, sb, sa);
    const float v = ddim_prev<true>(x0, e, sap, dir, nz != nullptr, sigma, nz ? nz[i] : 0.f);
    x_out[i] = v;
    x_in[pix * ld_in + c] = v;
    if (guided) x_in[half_in + pix * ld_in + c] = v;
    if (pred_x0) pred_x0[i] = x0;
  }
}
__global__ void scale_kernel(float* __restrict__ x, long long n, float s) {
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) x[i] *= s;
}
}  // namespace

extern "C" int dp_amax(const float* x, int64_t ld, int64_t rows, int32_t cols, uint32_t* slot, dp_stream_t st) {
  DP_REQUIRE(x && slot, DP_ERR_NULL);
  DP_REQUIRE(rows > 0 && cols > 0 && ld >= cols, DP_ERR_SHAPE);
  long long r = rows, c = cols;
  if (ld == cols) { c = r * c; r = 1; }                     // dense: one long row
  const int vec = ((((uintptr_t)x) & 15) == 0 && c % 4 == 0 && (r == 1 || ld % 4 == 0)) ? 1 : 0;
  amax_kernel<<<nblocks(vec ? r * (c >> 2) : r * c, NT * 4, DP_NUM_SMS * 8), NT, 0, (cudaStream_t)st>>>(x, ld, r, c, vec, slot);
  return dp_check_launch();
}
extern "C" int dp_zero_u32(uint32_t* p, int64_t n, dp_stream_t st) {
  DP_REQUIRE(p, DP_ERR_NULL);
  DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  zero_u32_kernel<<<nblocks(n, NT, DP_NUM_SMS), NT, 0, (cudaStream_t)st>>>(p, n);
  return dp_check_launch();
}
extern "C" int dp_silu_fwd(const float* x, float* y, int64_t n, dp_stream_t st) {
  DP_REQUIRE(x && y, DP_ERR_NULL); DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  silu_fwd_kernel<<<nblocks(n, NT), NT, 0, (cudaStream_t)st>>>(x, y, n);
  return dp_check_launch();
}
extern "C" int dp_silu_bwd(const float* x, const float* dy, float* dx, int64_t n, int32_t acc, dp_stream_t st) {
  DP_REQUIRE(x && dy && dx, DP_ERR_NULL); DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  silu_bwd_kernel<<<nblocks(n, NT), NT, 0, (cudaStream_t)st>>>(x, dy, dx, n, acc);
  return dp_check_launch();
}
extern "C" int dp_geglu_fwd(const float* u, int64_t ldu, float* out, int64_t ldo, int64_t rows, int32_t inner, dp_stream_t st) {
  DP_REQUIRE(u && out, DP_ERR_NULL); DP_REQUIRE(rows > 0 && inner > 0 && ldu >= 2 * (int64_t)inner && ldo >= inner, DP_ERR_SHAPE);
  geglu_fwd_kernel<<<nblocks(rows * inner, NT), NT, 0, (cudaStream_t)st>>>(u, ldu, out, ldo, rows, inner);
  return dp_check_launch();
}
extern "C" int dp_geglu_bwd(const float* u, int64_t ldu, const float* dout, int64_t lddo, float* du, int64_t lddu, int64_t rows, int32_t inner,
                            dp_stream_t st) {
  DP_REQUIRE(u && dout && du, DP_ERR_NULL);
  DP_REQUIRE(rows > 0 && inner > 0 && ldu >= 2 * (int64_t)inner && lddu >= 2 * (int64_t)inner && lddo >= inner, DP_ERR_SHAPE);
  geglu_bwd_kernel<<<nblocks(rows * inner, NT), NT, 0, (cudaStream_t)st>>>(u, ldu, dout, lddo, du, lddu, rows, inner);
  return dp_check_launch();
}
extern "C" int dp_timestep_embedding(const int64_t* t, const float* freqs, float* out, int32_t B, int32_t half, int32_t flip, dp_stream_t st) {
  DP_REQUIRE(t && freqs && out, DP_ERR_NULL); DP_REQUIRE(B > 0 && half > 0, DP_ERR_SHAPE);
  temb_kernel<<<(B * half + 127) / 128, 128, 0, (cudaStream_t)st>>>(t, freqs, out, B, half, flip);
  return dp_check_launch();
}
extern "C" int dp_add_noise(const float* x0, const float* noise, const int64_t* t, const float* acp, float* out, int32_t B,
                            int32_t C, int32_t H, int32_t W, int32_t out_nhwc, int64_t ld_out, dp_stream_t st) {
  DP_REQUIRE(x0 && noise && t && acp && out, DP_ERR_NULL); DP_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0, DP_ERR_SHAPE);
  DP_REQUIRE(ld_out == 0 || ld_out >= C, DP_ERR_SHAPE);
  add_noise_kernel<<<nblocks((long long)B * C * H * W, NT), NT, 0, (cudaStream_t)st>>>(x0, noise, t, acp, out, B, C, H * W, out_nhwc,
                                                                                    ld_out ? ld_out : C);
  return dp_check_launch();
}
extern "C" int dp_nchw_to_nhwc(const float* in, float* out, int64_t ld, int32_t N, int32_t C, int32_t H, int32_t W, dp_stream_t st) {
  DP_REQUIRE(in && out, DP_ERR_NULL); DP_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && ld >= C, DP_ERR_SHAPE);
  nchw_to_nhwc_kernel<<<nblocks((long long)N * C * H * W, NT), NT, 0, (cudaStream_t)st>>>(in, out, ld, N, C, H * W);
  return dp_check_launch();
}
extern "C" int dp_nhwc_to_nchw(const float* in, int64_t ld, float* out, int32_t N, int32_t C, int32_t H, int32_t W, int32_t acc, dp_stream_t st) {
  DP_REQUIRE(in && out, DP_ERR_NULL); DP_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && ld >= C, DP_ERR_SHAPE);
  nhwc_to_nchw_kernel<<<nblocks((long long)N * C * H * W, NT), NT, 0, (cudaStream_t)st>>>(in, ld, out, N, C, H * W, acc);
  return dp_check_launch();
}
extern "C" int64_t dp_mse_partials(int64_t n) { return n <= 0 ? 0 : (n + MSE_PER_BLOCK - 1) / MSE_PER_BLOCK; }
extern "C" int dp_mse_loss_grad(const float* pred, const float* target, float* grad, int64_t n, float scale_loss, float scale_grad,
                                float* partial, float* loss_out, dp_stream_t st) {
  DP_REQUIRE(pred && target && partial && loss_out, DP_ERR_NULL); DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  long long nb = dp_mse_partials(n);
  DP_REQUIRE(nb < (1ll << 31), DP_ERR_SHAPE);
  mse_stage1_kernel<<<(unsigned)nb, NT, 0, (cudaStream_t)st>>>(pred, target, grad, n, scale_grad, partial);
  int rc = dp_check_launch();
  if (rc) return rc;
  sum_stage2_kernel<<<1, NT, 0, (cudaStream_t)st>>>(partial, nb, scale_loss, loss_out);
  return dp_check_launch();
}
extern "C" int dp_upsample2x_fwd(const float* x, int64_t ldx, float* y, int64_t ldy, int32_t N, int32_t H, int32_t W, int32_t C, dp_stream_t st) {
  DP_REQUIRE(x && y, DP_ERR_NULL); DP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && ldx >= C && ldy >= C, DP_ERR_SHAPE);
  upsample_fwd_kernel<<<nblocks((long long)N * 4 * H * W * C, NT), NT, 0, (cudaStream_t)st>>>(x, ldx, y, ldy, N, H, W, C);
  return dp_check_launch();
}
extern "C" int dp_upsample2x_bwd(const float* dy, int64_t lddy, float* dx, int64_t lddx, int32_t N, int32_t H, int32_t W, int32_t C, int32_t acc, dp_stream_t st) {
  DP_REQUIRE(dy && dx, DP_ERR_NULL); DP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && lddy >= C && lddx >= C, DP_ERR_SHAPE);
  upsample_bwd_kernel<<<nblocks((long long)N * H * W * C, NT), NT, 0, (cudaStream_t)st>>>(dy, lddy, dx, lddx, N, H, W, C, acc);
  return dp_check_launch();
}
extern "C" int dp_colsum(const float* x, int64_t ld, int64_t rows, int32_t cols, int64_t seg_rows, float* out, int64_t ld_out, int32_t acc, dp_stream_t st) {
  DP_REQUIRE(x && out, DP_ERR_NULL); DP_REQUIRE(rows > 0 && cols > 0 && seg_rows > 0 && ld >= cols && ld_out >= cols, DP_ERR_SHAPE);
  long long nseg = (rows + seg_rows - 1) / seg_rows;
  DP_REQUIRE(nseg < (1ll << 31) && (cols + 63) / 64 <= 65535, DP_ERR_SHAPE);
  const int vec = (((uintptr_t)x & 15) == 0 && ld % 4 == 0) ? 1 : 0;
  colsum_kernel<<<dim3((unsigned)nseg, (cols + 63) / 64), dim3(16, 16), 0, (cudaStream_t)st>>>(x, ld, rows, cols, seg_rows, out, ld_out, acc, vec);
  return dp_check_launch();
}
extern "C" int dp_add_views(const float* a, int64_t lda, const float* b, int64_t ldb, float* y, int64_t ldy, int64_t rows, int32_t cols, dp_stream_t st) {
  DP_REQUIRE(a && b && y, DP_ERR_NULL); DP_REQUIRE(rows > 0 && cols > 0, DP_ERR_SHAPE);
  add_views_kernel<<<nblocks(rows * cols, NT), NT, 0, (cudaStream_t)st>>>(a, lda, b, ldb, y, ldy, rows, cols);
  return dp_check_launch();
}
extern "C" int dp_copy_rows(const float* a, int64_t lda, float* y, int64_t ldy, int64_t rows, int32_t cols, dp_stream_t st) {
  DP_REQUIRE(a && y, DP_ERR_NULL); DP_REQUIRE(rows > 0 && cols > 0 && lda >= cols && ldy >= cols, DP_ERR_SHAPE);
  copy_rows_kernel<<<nblocks(rows * cols, NT), NT, 0, (cudaStream_t)st>>>(a, lda, y, ldy, rows, cols);
  return dp_check_launch();
}
extern "C" int dp_softmax_fwd(const float* s, float* p, int64_t rows, int32_t cols, dp_stream_t st) {
  DP_REQUIRE(s && p, DP_ERR_NULL); DP_REQUIRE(rows > 0 && cols > 0, DP_ERR_SHAPE);
  long long nb = (rows + NT / 32 - 1) / (NT / 32);
  DP_REQUIRE(nb < (1ll << 31), DP_ERR_SHAPE);
  softmax_fwd_kernel<<<(unsigned)nb, NT, 0, (cudaStream_t)st>>>(s, p, rows, cols);
  return dp_check_launch();
}
extern "C" int dp_softmax_bwd(const float* p, const float* dp, float* ds, int64_t rows, int32_t cols, uint32_t* amax_ds, dp_stream_t st) {
  DP_REQUIRE(p && dp && ds, DP_ERR_NULL); DP_REQUIRE(rows > 0 && cols > 0, DP_ERR_SHAPE);
  long long nb = (rows + NT / 32 - 1) / (NT / 32);
  DP_REQUIRE(nb < (1ll << 31), DP_ERR_SHAPE);
  softmax_bwd_kernel<<<(unsigned)nb, NT, 0, (cudaStream_t)st>>>(p, dp, ds, rows, cols, amax_ds);
  return dp_check_launch();
}
extern "C" int dp_ddim_step(const float* x, const float* eps, const float* noise, float* out, int64_t n, float sqrt_beta_t,
                            float sqrt_alpha_t, float clip, float sqrt_alpha_prev, float dir_coef, float sigma, dp_stream_t st) {
  DP_REQUIRE(x && eps && out, DP_ERR_NULL); DP_REQUIRE(n > 0 && sqrt_alpha_t > 0.f, DP_ERR_SHAPE);
  DP_REQUIRE(sigma == 0.f || noise, DP_ERR_NULL);
  ddim_step_kernel<<<nblocks(n, NT), NT, 0, (cudaStream_t)st>>>(x, eps, sigma != 0.f ? noise : nullptr, out, n, sqrt_beta_t, sqrt_alpha_t,
                                                              clip, sqrt_alpha_prev, dir_coef, sigma);
  return dp_check_launch();
}
extern "C" int dp_ddim_cfg_step(const float* eps, int64_t ld_eps, const float* x, const float* noise, float* x_out, float* x_in, int64_t ld_in,
                                float* pred_x0, int32_t B, int32_t C, int32_t H, int32_t W, int32_t guided, float scale,
                                float sqrt_one_minus_at, float sqrt_at, float sqrt_a_prev, float dir_coef, float sigma, dp_stream_t st) {
  DP_REQUIRE(eps && x && x_out && x_in, DP_ERR_NULL);
  DP_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && ld_eps >= C && ld_in >= C && sqrt_at > 0.f, DP_ERR_SHAPE);
  DP_REQUIRE(sigma == 0.f || noise, DP_ERR_NULL);
  const long long n = (long long)B * C * H * W;
  ddim_cfg_step_kernel<<<nblocks(n, NT), NT, 0, (cudaStream_t)st>>>(eps, ld_eps, x, sigma != 0.f ? noise : nullptr, x_out, x_in, ld_in, pred_x0,
                                                                  B, C, H * W, guided ? 1 : 0, scale, sqrt_one_minus_at, sqrt_at, sqrt_a_prev,
                                                                  dir_coef, sigma);
  return dp_check_launch();
}
extern "C" int dp_scale(float* x, int64_t n, float s, dp_stream_t st) {
  DP_REQUIRE(x, DP_ERR_NULL); DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  scale_kernel<<<nblocks(n, NT), NT, 0, (cudaStream_t)st>>>(x, n, s);
  return dp_check_launch();
}
