// optim.cu — Taylor-importance reductions and the fused finetune tail (clip + Adam + EMA) over flat arenas.
#include "common.cuh"

namespace {
constexpr int NT = 256;

__device__ __forceinline__ void block_sum3(float& a, float& b, float& c) {
  __shared__ float red[3][NT / 32];
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; red[2][threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float x = 0, y = 0, z = 0;
    for (int w = 0; w < NT / 32; ++w) { x += red[0][w]; y += red[1][w]; z += red[2][w]; }
    a = x; b = y; c = z;
  }
}
__global__ void taylor_out_kernel(const dp_taylor_args a) {
  const int o = blockIdx.x;
  const long long inner = (long long)a.I * a.RS;
  const float* w = a.w + o * inner;
  const float* d = a.dw + o * inner;
  float s = 0, ab = 0, sq = 0;
  for (long long i = threadIdx.x; i < inner; i += NT) { float p = w[i] * d[i]; s += p; ab += fabsf(p); sq += p * p; }
  block_sum3(s, ab, sq);
  if (threadIdx.x == 0) { if (a.out_signed) a.out_signed[o] = s; if (a.out_abs) a.out_abs[o] = ab; if (a.out_sq) a.out_sq[o] = sq; }
}
__global__ void taylor_in_kernel(const dp_taylor_args a) {
  const int ic = blockIdx.x;
  float s = 0, ab = 0, sq = 0;
  const long long n = (long long)a.O * a.RS;
  for (long long i = threadIdx.x; i < n; i += NT) {
    long long o = i / a.RS; int rs = (int)(i - o * a.RS);
    long long idx = (o * a.I + ic) * a.RS + rs;
    float p = a.w[idx] * a.dw[idx]; s += p; ab += fabsf(p); sq += p * p;
  }
  block_sum3(s, ab, sq);
  if (threadIdx.x == 0) { if (a.in_signed) a.in_signed[ic] = s; if (a.in_abs) a.in_abs[ic] = ab; if (a.in_sq) a.in_sq[ic] = sq; }
}

constexpr int SS_PER_BLOCK = 8192;
__global__ void sumsq_stage1_kernel(const float* __restrict__ x, long long n, float* __restrict__ partial) {
  long long base = (long long)blockIdx.x * SS_PER_BLOCK;
  float s = 0.f;
  for (int j = threadIdx.x; j < SS_PER_BLOCK; j += NT) { long long i = base + j; if (i < n) { float v = x[i]; s += v * v; } }
  __shared__ float red[NT / 32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < NT / 32; ++w) t += red[w]; partial[blockIdx.x] = t; }
}
__global__ void sumsq_stage2_kernel(const float* __restrict__ partial, long long nb, float* __restrict__ out) {
  __shared__ double red[NT];
  double s = 0;
  for (long long i = threadIdx.x; i < nb; i += NT) s += partial[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) out[0] = (float)red[0];
}
struct AdamConsts { float step_size, bc2_sqrt, w1, w2, beta2, eps, max_norm, ema_d, ema_1md; };
__global__ void adam_kernel(const dp_adam_args a, AdamConsts k) {
  // torch.optim.Adam (single-tensor path) op order:
  //   exp_avg.lerp_(g, 1-b1); exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2)
  //   denom = exp_avg_sq.sqrt() / sqrt(bc2) + eps ; p.addcdiv_(exp_avg, denom, value=-lr/bc1)
  float clip = 1.0f;
  if (a.sumsq) {
    float total = sqrtf(*a.sumsq) * a.grad_scale;            // norm of the (scaled) gradient
    float coef = k.max_norm / (total + 1e-6f);               // torch.nn.utils.clip_grad_norm_
    clip = coef < 1.0f ? coef : 1.0f;
  }
  if (a.step_scalars) { k.step_size = a.step_scalars[0]; k.bc2_sqrt = a.step_scalars[1]; }
  const float gs = a.grad_scale * clip;
  for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < a.n; i += (long long)gridDim.x * NT) {
    float g = a.g[i] * gs;
    float m = a.m[i]; m = m + k.w1 * (g - m);
    float v = a.v[i] * k.beta2 + k.w2 * g * g;
    float denom = sqrtf(v) / k.bc2_sqrt + k.eps;
    float p = a.p[i] - k.step_size * (m / denom);
    a.m[i] = m; a.v[i] = v; a.p[i] = p;
    if (a.ema) a.ema[i] = k.ema_1md * p + k.ema_d * a.ema[i];   // training_utils.py:216
  }
}
}  // namespace

extern "C" int dp_taylor_reduce(const dp_taylor_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->w && a->dw, DP_ERR_NULL);
  DP_REQUIRE(a->O > 0 && a->I > 0 && a->RS > 0, DP_ERR_SHAPE);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = DP_OK;
  if (a->out_signed || a->out_abs || a->out_sq) { taylor_out_kernel<<<a->O, NT, 0, st>>>(*a); if ((rc = dp_check_launch())) return rc; }
  if (a->in_signed || a->in_abs || a->in_sq) { taylor_in_kernel<<<a->I, NT, 0, st>>>(*a); rc = dp_check_launch(); }
  return rc;
}
extern "C" int64_t dp_sumsq_partials(int64_t n) { return n <= 0 ? 0 : (n + SS_PER_BLOCK - 1) / SS_PER_BLOCK; }
extern "C" int dp_sumsq(const float* x, int64_t n, float* partial, float* out, dp_stream_t stream) {
  DP_REQUIRE(x && partial && out, DP_ERR_NULL); DP_REQUIRE(n > 0, DP_ERR_SHAPE);
  long long nb = dp_sumsq_partials(n);
  DP_REQUIRE(nb < (1ll << 31), DP_ERR_SHAPE);
  sumsq_stage1_kernel<<<(unsigned)nb, NT, 0, (cudaStream_t)stream>>>(x, n, partial);
  int rc = dp_check_launch();
  if (rc) return rc;
  sumsq_stage2_kernel<<<1, NT, 0, (cudaStream_t)stream>>>(partial, nb, out);
  return dp_check_launch();
}
extern "C" int dp_adam_clip_ema(const dp_adam_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->p && a->g && a->m && a->v, DP_ERR_NULL);
  DP_REQUIRE(a->n > 0 && a->step >= 1, DP_ERR_SHAPE);
  const double bc1 = 1.0 - pow(a->beta1, a->step), bc2 = 1.0 - pow(a->beta2, a->step);
  AdamConsts k;
  k.step_size = (float)(a->lr / bc1); k.bc2_sqrt = (float)sqrt(bc2);
  k.w1 = (float)(1.0 - a->beta1); k.w2 = (float)(1.0 - a->beta2); k.beta2 = (float)a->beta2; k.eps = (float)a->eps;
  k.max_norm = (float)a->max_norm; k.ema_d = (float)a->ema_decay; k.ema_1md = (float)(1.0 - a->ema_decay);
  long long nb = (a->n + NT * 4 - 1) / (NT * 4);
  if (nb > DP_NUM_SMS * 16) nb = DP_NUM_SMS * 16;
  adam_kernel<<<(unsigned)nb, NT, 0, (cudaStream_t)stream>>>(*a, k);
  return dp_check_launch();
}
