// conv_bf16.cu — the single-pass tensor tier: wgmma on BF16 operands, fp32 accumulation in registers.
//
// What it is for: the pruned-UNet finetune step under `--mixed_precision bf16` (ddpm_train.py:200-208,255-261: torch.autocast runs
// conv2d / linear in bf16, GroupNorm / softmax / loss / Adam / EMA in fp32) — BASELINE configs[3].  Operands are rounded to bf16 (RNE)
// at the convolution boundary by their producers (dp_cvt_bf16, or the GroupNorm+SiLU kernel writing bf16 directly); products are exact
// in the tensor core and accumulate in fp32; outputs, the residual stream and all gradients stay fp32.
//
// Unlike the fp32-grade split kernels (conv_tc.cu) nothing has to touch the operands between TMA and the MMA: TMA -> swizzled shared memory ->
// wgmma, no splitting, no proxy fence in the loop.  One pipeline stage = 64 bf16 of GEMM-K = one 128-byte swizzle row.  Warpgroup roles:
// sm90.cuh (TMA producer + two consumer warpgroups of 64 tile rows each).
//   conv_bf16_kernel   fprop / dgrad (stride-1 dgrad = tap-flipped fprop; stride 2 through TMA element strides / parity classes):
//                      persistent, 1 CTA per SM, tile 128 pixels x up to 256 output channels (one N tile covers every layer of the
//                      DDPM configs up to 256 channels, so the activation tile is fetched once).
//   wgrad_bf16_kernel  dW[k][tap][c] = sum_pix dy[pix][k] x[pix@tap][c]: both operands MN-major (pixel-major activations) straight
//                      from TMA (SWIZZLE_128B, 64 channels x 64 pixels per box), tile 128 out-channels x up to 256 in-channels,
//                      split-K over pixels into the fp32 workspace that dp_conv2d_wgrad_reduce sums in fixed order.
// Both are instantiated per N tile width (64, 128, 192, 256): wgmma takes N as an immediate and the accumulators live in registers.
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "sm90.cuh"
#include "sm90_host.cuh"

namespace {
using namespace sm90;

constexpr int BM = 128;            // GEMM-M tile: 128 output pixels (64 per consumer warpgroup)
constexpr int KB = 64;             // bf16 elements of GEMM-K per pipeline stage (one 128-byte swizzle row)
constexpr int A_BYTES = BM * KB * 2;   // 16 KB
constexpr int MAX_SMEM = 227 * 1024;

struct BfParams {
  int Nimg, Nout;
  int kchunks;                 // ceil(Kg / 64)
  int bw, bh, bn, tiles_w, tiles_h;
  float* y; long long ldy;
  const float* bias;
  const float* rowadd; long long ld_rowadd;
  const float* residual; long long ld_res;
  int accumulate, vec4;
  int ntaps;
  signed char dh[9], dw[9], wt[9];
  int os, oa, ob, Ho, Wo;      // output pixel = (p*os + oa, q*os + ob) on an [Ho][Wo] grid
  int in_stride;
  int stages;
};

// ------------------------------------------------------------------------------------------------ fprop / dgrad
// NB = N tile / 64 = rows of the weight box / 64
template <int NB>
__global__ void __launch_bounds__(THREADS, 1)
conv_bf16_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const BfParams p,
                 const int tiles_m, const int total_tiles) {
  constexpr int BNT = 64 * NB;
  constexpr int B_BYTES = BNT * 128;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t pad_to = ((raw + 1023u) & ~1023u) - raw;   // SWIZZLE_128B needs 1024-byte aligned tiles
  const uint32_t sbase = raw + pad_to;
  const int S = p.stages;
  const uint32_t bar0 = sbase + (uint32_t)(S * STAGE_BYTES);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (S + s); };
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }   // one arrival per consumer warp
    mbar_init_fence();
  }
  __syncthreads();
  const int iters_per_tile = p.ntaps * p.kchunks;

  auto tile_coords = [&](int tile, int& q0, int& p0, int& n0, int& nblk) {
    nblk = tile / tiles_m;
    const int tile_m = tile - nblk * tiles_m;
    const int tw = tile_m % p.tiles_w;
    const int th = (tile_m / p.tiles_w) % p.tiles_h;
    const int tn = tile_m / (p.tiles_w * p.tiles_h);
    q0 = tw * p.bw; p0 = th * p.bh; n0 = tn * p.bn;
  };

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      prefetch_map(&mapA); prefetch_map(&mapB);
      int s = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int q0, p0, n0, nblk;
        tile_coords(tile, q0, p0, n0, nblk);
        for (int it = 0; it < iters_per_tile; ++it) {
          mbar_wait(empty_bar(s), ph ^ 1u);
          mbar_expect_tx(full_bar(s), STAGE_BYTES);
          const int tap = it / p.kchunks, kc = it - tap * p.kchunks;
          const uint32_t st = sbase + (uint32_t)(s * STAGE_BYTES);
          tma_load_4d(st, &mapA, full_bar(s), kc * KB, q0 * p.in_stride + p.dw[tap], p0 * p.in_stride + p.dh[tap], n0);
          tma_load_3d(st + A_BYTES, &mapB, full_bar(s), kc * KB, nblk * BNT, p.wt[tap]);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1;                       // consumer warpgroup: tile rows 64c .. 64c + 63
  const int warp = tid >> 5, lane = tid & 31;
  int s = 0; uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    float acc[BNT / 2];
    int prev_s = 0;
    for (int it = 0; it < iters_per_tile; ++it) {
      mbar_wait(full_bar(s), ph);
      const uint32_t st = sbase + (uint32_t)(s * STAGE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KB / 16; ++k)     // wgmma K = 16 bf16 = 32 bytes inside the 128-byte swizzle row
        wgmma_bf16<BNT, 0, 0>(acc, desc_k(st + c * 8192 + k * 32), desc_k(st + A_BYTES + k * 32), (it > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                      // the previous stage's MMAs have read their operands: hand it back to TMA
      if (it > 0 && lane == 0) mbar_arrive(empty_bar(prev_s));
      prev_s = s;
      if (++s == S) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (lane == 0) mbar_arrive(empty_bar(prev_s));

    int q0, p0, n0, nblk;
    tile_coords(tile, q0, p0, n0, nblk);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = 64 * c + 16 * warp + (lane >> 2) + 8 * i;
      const int w_l = row % p.bw, h_l = (row / p.bw) % p.bh, n_l = row / (p.bw * p.bh);
      const int img = n0 + n_l;
      if (img >= p.Nimg) continue;
      const long long m = ((long long)img * p.Ho + ((p0 + h_l) * p.os + p.oa)) * p.Wo + ((q0 + w_l) * p.os + p.ob);
      float* yrow = p.y + m * p.ldy;
      const float* rrow = p.residual ? p.residual + m * p.ld_res : nullptr;
      const float* arow = p.rowadd ? p.rowadd + (long long)img * p.ld_rowadd : nullptr;
#pragma unroll
      for (int j = 0; j < BNT / 8; ++j) {
        const int col = nblk * BNT + 8 * j + 2 * (lane & 3);
        float o[2] = {acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]};
        if (p.vec4 && col + 2 <= p.Nout) {
          if (p.bias) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.bias + col)); o[0] += t.x; o[1] += t.y; }
          if (arow) { const float2 t = __ldg(reinterpret_cast<const float2*>(arow + col)); o[0] += t.x; o[1] += t.y; }
          if (rrow) { const float2 t = __ldg(reinterpret_cast<const float2*>(rrow + col)); o[0] += t.x; o[1] += t.y; }
          float2* dst = reinterpret_cast<float2*>(yrow + col);
          if (p.accumulate) { const float2 t = *dst; o[0] += t.x; o[1] += t.y; }
          *dst = make_float2(o[0], o[1]);
        } else {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int cc = col + e;
            if (cc < p.Nout) {
              float ov = o[e];
              if (p.bias) ov += __ldg(p.bias + cc);
              if (arow) ov += __ldg(arow + cc);
              if (rrow) ov += __ldg(rrow + cc);
              if (p.accumulate) ov += yrow[cc];
              yrow[cc] = ov;
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ wgrad
struct WgBfParams {
  int Nimg, H, W, C, K;          // H, W = dy (output) grid
  int R, S, pad;
  int bw, bh, bn, tiles_w, tiles_h;   // 64-pixel box of the dy grid
  int total_chunks, chunks_per_split;
  int c_tiles, ct_width;         // in-channel tiles of ct_width (= 64 * NB)
  float* ws;
  int in_stride;
  int stages;
};
constexpr int WG_PIX = 64;                 // pixels (GEMM-K) per stage
constexpr int BLK_BYTES = WG_PIX * 128;    // one [64 px][64 ch] bf16 block = 8 KB

// stage: dy blocks 0,1 (out-channels 0-63, 64-127 of the tile: consumer warpgroup c multiplies block c) | x blocks 0..NB-1
template <int NB>
__global__ void __launch_bounds__(THREADS, 1)
wgrad_bf16_kernel(const __grid_constant__ CUtensorMap mapDy, const __grid_constant__ CUtensorMap mapX, const WgBfParams p) {
  constexpr int BNT = 64 * NB;
  constexpr int STAGE_BYTES = (2 + NB) * BLK_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t pad_to = ((raw + 1023u) & ~1023u) - raw;
  const uint32_t sbase = raw + pad_to;
  const int S = p.stages;
  const uint32_t bar0 = sbase + (uint32_t)(S * STAGE_BYTES);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (S + s); };
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
    mbar_init_fence();
  }
  __syncthreads();

  const int T = p.R * p.S;
  int tile = blockIdx.x;
  const int tap = tile % T; tile /= T;
  const int ct = tile % p.c_tiles;
  const int kt = tile / p.c_tiles;
  const int r = tap / p.S, sx = tap - r * p.S;
  const int chunk0 = blockIdx.y * p.chunks_per_split;
  const int chunk1 = min(p.total_chunks, chunk0 + p.chunks_per_split);
  const int num_iters = max(0, chunk1 - chunk0);
  const int c_valid = min(BNT, p.C - ct * BNT);
  const int xb = (c_valid + 63) >> 6;            // 64-channel x blocks that hold valid channels (the others only feed unstored columns)

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      prefetch_map(&mapDy); prefetch_map(&mapX);
      int s = 0; uint32_t ph = 0;
      for (int it = 0; it < num_iters; ++it) {
        mbar_wait(empty_bar(s), ph ^ 1u);
        mbar_expect_tx(full_bar(s), (uint32_t)((2 + xb) * BLK_BYTES));
        const int chunk = chunk0 + it;
        const int tw = chunk % p.tiles_w;
        const int th = (chunk / p.tiles_w) % p.tiles_h;
        const int tn = chunk / (p.tiles_w * p.tiles_h);
        const int q0 = tw * p.bw, p0 = th * p.bh, n0 = tn * p.bn;
        const uint32_t st = sbase + (uint32_t)(s * STAGE_BYTES);
        tma_load_4d(st, &mapDy, full_bar(s), kt * 128, q0, p0, n0);
        tma_load_4d(st + BLK_BYTES, &mapDy, full_bar(s), kt * 128 + 64, q0, p0, n0);
        for (int b = 0; b < xb; ++b)
          tma_load_4d(st + (2 + b) * BLK_BYTES, &mapX, full_bar(s), ct * BNT + b * 64, q0 * p.in_stride + sx - p.pad,
                      p0 * p.in_stride + r - p.pad, n0);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int warp = tid >> 5, lane = tid & 31;
  float acc[BNT / 2];
  int s = 0, prev_s = 0; uint32_t ph = 0;
  for (int it = 0; it < num_iters; ++it) {
    mbar_wait(full_bar(s), ph);
    const uint32_t st = sbase + (uint32_t)(s * STAGE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < WG_PIX / 16; ++k)   // 16 pixels = two 8-pixel K groups = 2048 bytes further into every block
      wgmma_bf16<BNT, 1, 1>(acc, desc_mn(st + c * BLK_BYTES + k * 2048, BLK_BYTES), desc_mn(st + 2 * BLK_BYTES + k * 2048, BLK_BYTES),
                            (it > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0 && lane == 0) mbar_arrive(empty_bar(prev_s));
    prev_s = s;
    if (++s == S) { s = 0; ph ^= 1u; }
  }
  wgmma_wait<0>();
  fence_regs(acc);
  const long long TC_ = (long long)T * p.C;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kout = kt * 128 + 64 * c + 16 * warp + (lane >> 2) + 8 * i;
    if (kout >= p.K) continue;
    float* wrow = p.ws + ((long long)blockIdx.y * p.K + kout) * TC_ + (long long)tap * p.C + (long long)ct * BNT;
#pragma unroll
    for (int j = 0; j < BNT / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * j + 2 * (lane & 3) + e;
        // an empty split accumulated nothing (the registers hold garbage): it contributes zeros
        if (col < c_valid) wrow[col] = num_iters ? acc[4 * j + 2 * i + e] : 0.f;
      }
  }
}

// ------------------------------------------------------------------------------------------------ operand producers
// fp32 NHWC view -> bf16 (RNE) dense rows of `ld_dst` elements (a multiple of 8 = 16-byte pitch); pad columns [C, ld_dst) are zeroed.
__global__ void cvt_bf16_kernel(const float* __restrict__ src, long long ld, long long rows, int C, __nv_bfloat16* __restrict__ dst,
                                long long ld_dst, int vec_ok) {
  const int groups = (int)(ld_dst >> 3);
  const long long total = rows * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long rrow = i / groups;
    const int c0 = (int)(i - rrow * groups) << 3;
    const float* s = src + rrow * ld + c0;
    float v[8];
    if (vec_ok && c0 + 8 <= C) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(s)), b = __ldg(reinterpret_cast<const float4*>(s + 4));
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c0 + j < C) ? __ldg(s + j) : 0.f;
    }
    __nv_bfloat162 o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<uint4*>(dst + rrow * ld_dst + c0) = *reinterpret_cast<const uint4*>(o);
  }
}

// OIHW fp32 -> kc [RS][K][Cp] (fprop B operand) and ck [RS][C][Kp] (dgrad B operand), bf16, rows zero-padded to a multiple of 64
__global__ void pack_bf16_kernel(const float* __restrict__ w, int K, int C, int RS, int Cp, int Kp, __nv_bfloat16* __restrict__ kc,
                                 __nv_bfloat16* __restrict__ ck) {
  const long long na = (long long)RS * K * Cp, nb = (long long)RS * C * Kp;
  const long long total = na > nb ? na : nb;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (kc && i < na) {
      int c = (int)(i % Cp); long long t = i / Cp; int k = (int)(t % K), tap = (int)(t / K);
      kc[i] = __float2bfloat16_rn(c < C ? w[((long long)k * C + c) * RS + tap] : 0.f);
    }
    if (ck && i < nb) {
      int k = (int)(i % Kp); long long t = i / Kp; int c = (int)(t % C), tap = (int)(t / C);
      ck[i] = __float2bfloat16_rn(k < K ? w[((long long)k * C + c) * RS + tap] : 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
int bf_init() {
  static const int ok = [] {
    bool set = runtime().encode != nullptr;
    for (const void* k : {(const void*)conv_bf16_kernel<1>, (const void*)conv_bf16_kernel<2>, (const void*)conv_bf16_kernel<3>,
                          (const void*)conv_bf16_kernel<4>, (const void*)wgrad_bf16_kernel<1>, (const void*)wgrad_bf16_kernel<2>,
                          (const void*)wgrad_bf16_kernel<3>, (const void*)wgrad_bf16_kernel<4>})
      set = set && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM) == cudaSuccess;
    (void)cudaGetLastError();
    return set ? 1 : 0;
  }();
  return ok;
}

int wrow_bf16(int c) { return (c + 63) & ~63; }

// Box, tiles, N tile and pipeline depth of one conv_bf16_kernel launch over an activation of pixel pitch ld_act (bf16 elements)
struct BfPlan { int bw, bh, bn, tiles_m, n_tiles, bn_tile, stages; };
int plan_bf16(const ConvGemm& g, long long ld_act, BfPlan& pl) {
  if (!bf_init()) return DP_ERR_UNSUPPORTED;
  if (ld_act % 8 || g.Kg < 8 || g.Nout < 1 || !pick_box(BM, g.H, g.W, pl.bw, pl.bh, pl.bn)) return DP_ERR_UNSUPPORTED;
  if (pl.bw * g.in_stride > 256 || pl.bh * g.in_stride > 256) return DP_ERR_UNSUPPORTED;
  pl.tiles_m = (g.W / pl.bw) * (g.H / pl.bh) * ((g.N + pl.bn - 1) / pl.bn);
  // N tile: as wide as possible (<= 256) so the activation tile is fetched once; balanced over the tiles it takes, a multiple of 64
  // (one instantiation per width)
  pl.n_tiles = (g.Nout + 255) / 256;
  pl.bn_tile = ((g.Nout + pl.n_tiles - 1) / pl.n_tiles + 63) & ~63;
  if (pl.bn_tile > 256) pl.bn_tile = 256;
  pl.stages = (MAX_SMEM - 2048) / (A_BYTES + pl.bn_tile * 128);     // every tile starts 1024-byte aligned
  if (pl.stages > 8) pl.stages = 8;
  return pl.stages < 2 ? DP_ERR_UNSUPPORTED : DP_OK;
}

// Operands and epilogue of a launch.  A: bf16 [N][H*in_stride][W*in_stride][ld_act] view of the GEMM's input; B: bf16 [T][Nout][wrow_bf16(Kg)];
// out: fp32 [N][Ho][Wo][ld_out] view.
struct BfLaunch {
  const void* act; long long ld_act; const void* w; int T;
  float* out; long long ld_out;
  const float* bias; const float* rowadd; long long ld_rowadd; const float* residual; long long ld_res;
  int accumulate;
};
// A convolution's launch: A = x (fprop) or dy (dgrad), B = its packed weights; the epilogue terms are fprop's
BfLaunch conv_launch(const dp_conv_bf16_args* a, bool dgrad) {
  BfLaunch l{};
  l.act = dgrad ? a->dy_bf16 : a->x_bf16; l.ld_act = dgrad ? a->lddy : a->ldx; l.w = a->w_bf16; l.T = a->R * a->S;
  l.out = a->out; l.ld_out = a->ld_out;
  if (!dgrad) { l.bias = a->bias; l.rowadd = a->rowadd; l.ld_rowadd = a->ld_rowadd; l.residual = a->residual; l.ld_res = a->ld_res; }
  l.accumulate = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  return l;
}

int launch_bf16(const ConvGemm& g, const BfLaunch& l, cudaStream_t st) {
  if (!bf_init()) return DP_ERR_UNSUPPORTED;
  if (!l.act || !l.w || !l.out) return DP_ERR_NULL;
  if (((uintptr_t)l.act & 15) || ((uintptr_t)l.w & 15)) return DP_ERR_UNSUPPORTED;
  BfPlan pl;
  const int rc = plan_bf16(g, l.ld_act, pl);
  if (rc != DP_OK) return rc;
  CUtensorMap mA, mB;
  {
    const int s = g.in_stride;
    const cuuint64_t Hin = (cuuint64_t)g.H * s, Win = (cuuint64_t)g.W * s;
    cuuint64_t dims[4] = {(cuuint64_t)g.Kg, Win, Hin, (cuuint64_t)g.N};
    cuuint64_t str[3] = {(cuuint64_t)l.ld_act * 2, Win * l.ld_act * 2, Hin * Win * l.ld_act * 2};
    cuuint32_t box[4] = {(cuuint32_t)KB, (cuuint32_t)(pl.bw * s), (cuuint32_t)(pl.bh * s), (cuuint32_t)pl.bn};
    if (!encode_map(&mA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, l.act, 4, dims, str, box, s)) return DP_ERR_UNSUPPORTED;
  }
  {
    const cuuint64_t ldb = (cuuint64_t)wrow_bf16(g.Kg);
    cuuint64_t dims[3] = {ldb, (cuuint64_t)g.Nout, (cuuint64_t)l.T};
    cuuint64_t str[2] = {ldb * 2, (cuuint64_t)g.Nout * ldb * 2};
    cuuint32_t box[3] = {(cuuint32_t)KB, (cuuint32_t)pl.bn_tile, 1};
    if (!encode_map(&mB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, l.w, 3, dims, str, box)) return DP_ERR_UNSUPPORTED;
  }
  BfParams p{};
  p.Nimg = g.N; p.Nout = g.Nout;
  p.ntaps = g.taps.n;
  for (int i = 0; i < 9; ++i) { p.dh[i] = g.taps.dh[i]; p.dw[i] = g.taps.dw[i]; p.wt[i] = g.taps.wt[i]; }
  p.os = g.os; p.oa = g.oa; p.ob = g.ob; p.Ho = g.Ho; p.Wo = g.Wo; p.in_stride = g.in_stride;
  p.kchunks = (g.Kg + KB - 1) / KB;
  p.bw = pl.bw; p.bh = pl.bh; p.bn = pl.bn; p.tiles_w = g.W / pl.bw; p.tiles_h = g.H / pl.bh;
  p.y = l.out; p.ldy = l.ld_out; p.bias = l.bias; p.rowadd = l.rowadd; p.ld_rowadd = l.ld_rowadd; p.residual = l.residual; p.ld_res = l.ld_res;
  p.accumulate = l.accumulate;
  p.vec4 = (al16(l.out, l.ld_out) && al16(l.bias, 0) && al16(l.rowadd, l.ld_rowadd) && al16(l.residual, l.ld_res)) ? 1 : 0;
  p.stages = pl.stages;
  const int total = pl.tiles_m * pl.n_tiles, sms = runtime().num_sms, ctas = total < sms ? total : sms;
  const size_t smem = (size_t)pl.stages * (A_BYTES + pl.bn_tile * 128) + 2048;
  switch (pl.bn_tile / 64) {
    case 1: conv_bf16_kernel<1><<<ctas, THREADS, smem, st>>>(mA, mB, p, pl.tiles_m, total); break;
    case 2: conv_bf16_kernel<2><<<ctas, THREADS, smem, st>>>(mA, mB, p, pl.tiles_m, total); break;
    case 3: conv_bf16_kernel<3><<<ctas, THREADS, smem, st>>>(mA, mB, p, pl.tiles_m, total); break;
    default: conv_bf16_kernel<4><<<ctas, THREADS, smem, st>>>(mA, mB, p, pl.tiles_m, total); break;
  }
  return dp_check_launch();
}

bool conv_shape_ok(const dp_conv_bf16_args* a) {
  return a && box_geometry(a) && a->N > 0 && a->H > 0 && a->W > 0 && a->C > 0 && a->K > 0;
}

// The GEMMs of a fprop (op 0) or dgrad (op 1), or 0 when the bf16 kernels do not take the convolution's geometry
int bf16_gemms(const dp_conv_bf16_args* a, int op, ConvGemm g[4]) {
  if (!conv_shape_ok(a)) return 0;
  if (op == 0 ? (a->ldx < a->C || a->ld_out < a->K) : (a->lddy < a->K || a->ld_out < a->C)) return 0;
  return conv_gemms(a, op, g);
}

int conv_bf16(const dp_conv_bf16_args* a, int op, cudaStream_t st) {
  ConvGemm g[4];
  const int n = bf16_gemms(a, op, g);
  if (n == 0) return DP_ERR_UNSUPPORTED;
  const BfLaunch l = conv_launch(a, op != 0);
  for (int c = 0; c < n; ++c) {
    const int rc = launch_bf16(g[c], l, st);
    if (rc != DP_OK) return rc;
  }
  return DP_OK;
}

bool wgrad_geometry(const dp_conv_bf16_args* a) { return conv_shape_ok(a) && a->splits >= 1 && a->ldx >= a->C && a->lddy >= a->K; }

// Box (64 pixels of the dy grid), in-channel tile and pipeline depth of a wgrad_bf16_kernel launch
struct WgBfPlan { int bw, bh, bn, ct_width, stages; };
int plan_wgrad_bf16(const dp_conv_bf16_args* a, WgBfPlan& pl) {
  if (!bf_init() || a->ldx % 8 || a->lddy % 8) return DP_ERR_UNSUPPORTED;
  if (!pick_box(WG_PIX, a->P, a->Q, pl.bw, pl.bh, pl.bn) || a->N % pl.bn) return DP_ERR_UNSUPPORTED;
  if (pl.bw * a->stride > 256 || pl.bh * a->stride > 256) return DP_ERR_UNSUPPORTED;
  pl.ct_width = dp_bf16_wgrad_ctile(a->C);
  pl.stages = (MAX_SMEM - 2048) / ((2 + pl.ct_width / 64) * BLK_BYTES);
  if (pl.stages > 8) pl.stages = 8;
  return DP_OK;
}

int wgrad_bf16(const dp_conv_bf16_args* a, cudaStream_t st) {
  if (!wgrad_geometry(a) || !bf_init()) return DP_ERR_UNSUPPORTED;
  if (!a->x_bf16 || !a->dy_bf16 || !a->workspace) return DP_ERR_NULL;
  if (((uintptr_t)a->x_bf16 & 15) || ((uintptr_t)a->dy_bf16 & 15)) return DP_ERR_UNSUPPORTED;
  WgBfPlan pl;
  const int rc = plan_wgrad_bf16(a, pl);
  if (rc != DP_OK) return rc;
  CUtensorMap mDy, mX;
  {
    cuuint64_t dims[4] = {(cuuint64_t)a->K, (cuuint64_t)a->Q, (cuuint64_t)a->P, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->lddy * 2, (cuuint64_t)a->Q * a->lddy * 2, (cuuint64_t)a->P * a->Q * a->lddy * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)pl.bw, (cuuint32_t)pl.bh, (cuuint32_t)pl.bn};
    if (!encode_map(&mDy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a->dy_bf16, 4, dims, str, box)) return DP_ERR_UNSUPPORTED;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)a->C, (cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->ldx * 2, (cuuint64_t)a->W * a->ldx * 2, (cuuint64_t)a->H * a->W * a->ldx * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(pl.bw * a->stride), (cuuint32_t)(pl.bh * a->stride), (cuuint32_t)pl.bn};
    if (!encode_map(&mX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a->x_bf16, 4, dims, str, box, a->stride)) return DP_ERR_UNSUPPORTED;
  }
  WgBfParams p{};
  p.Nimg = a->N; p.H = a->P; p.W = a->Q; p.C = a->C; p.K = a->K; p.R = a->R; p.S = a->S; p.pad = a->pad_t; p.in_stride = a->stride;
  p.bw = pl.bw; p.bh = pl.bh; p.bn = pl.bn; p.tiles_w = a->Q / pl.bw; p.tiles_h = a->P / pl.bh;
  p.total_chunks = p.tiles_w * p.tiles_h * (a->N / pl.bn);
  p.chunks_per_split = (p.total_chunks + a->splits - 1) / a->splits;
  p.ct_width = pl.ct_width;
  p.c_tiles = (a->C + p.ct_width - 1) / p.ct_width;
  p.ws = a->workspace;
  p.stages = pl.stages;
  const int k_tiles = (a->K + 127) / 128;
  dim3 grid((unsigned)(k_tiles * p.c_tiles * a->R * a->S), (unsigned)a->splits);
  const size_t smem = (size_t)pl.stages * (2 + pl.ct_width / 64) * BLK_BYTES + 2048;
  switch (pl.ct_width / 64) {
    case 1: wgrad_bf16_kernel<1><<<grid, THREADS, smem, st>>>(mDy, mX, p); break;
    case 2: wgrad_bf16_kernel<2><<<grid, THREADS, smem, st>>>(mDy, mX, p); break;
    case 3: wgrad_bf16_kernel<3><<<grid, THREADS, smem, st>>>(mDy, mX, p); break;
    default: wgrad_bf16_kernel<4><<<grid, THREADS, smem, st>>>(mDy, mX, p); break;
  }
  return dp_check_launch();
}

}  // namespace

extern "C" int dp_bf16_available(void) { return bf_init(); }
extern "C" int dp_bf16_weight_row(int channels) { return channels > 0 ? wrow_bf16(channels) : 0; }
// in-channel tile width of the bf16 wgrad: the whole width up to 256, else balanced 64-multiples
extern "C" int dp_bf16_wgrad_ctile(int C) {
  if (C <= 0) return 0;
  const int tiles = (C + 255) / 256;
  int w = (((C + tiles - 1) / tiles) + 63) & ~63;
  return w > 256 ? 256 : w;
}

extern "C" int dp_conv2d_fprop_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return conv_bf16(a, 0, (cudaStream_t)s); }
extern "C" int dp_conv2d_dgrad_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return conv_bf16(a, 1, (cudaStream_t)s); }
extern "C" int dp_conv2d_wgrad_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return wgrad_bf16(a, (cudaStream_t)s); }
// op: 0 fprop, 1 dgrad, 2 wgrad.  DP_OK when the bf16 kernels take this shape (pointers are not needed), else DP_ERR_UNSUPPORTED.
extern "C" int dp_conv_bf16_eligible(const dp_conv_bf16_args* a, int op) {
  if (!a) return DP_ERR_NULL;
  if (op != 0 && op != 1) {
    WgBfPlan pl;
    return wgrad_geometry(a) ? plan_wgrad_bf16(a, pl) : DP_ERR_UNSUPPORTED;
  }
  ConvGemm g[4];
  BfPlan pl;
  // the parity classes of a stride-2 dgrad share their grid and channels: the first stands for all four
  return bf16_gemms(a, op, g) ? plan_bf16(g[0], op == 0 ? a->ldx : a->lddy, pl) : DP_ERR_UNSUPPORTED;
}

extern "C" int dp_cvt_bf16(const float* src, int64_t ld, int64_t rows, int32_t C, void* dst, int64_t ld_dst, dp_stream_t stream) {
  DP_REQUIRE(src && dst, DP_ERR_NULL);
  DP_REQUIRE(rows > 0 && C > 0 && ld >= C && ld_dst >= C && ld_dst % 8 == 0, DP_ERR_SHAPE);
  DP_REQUIRE(((uintptr_t)dst & 15) == 0, DP_ERR_ALIGN);
  const int vec_ok = (((uintptr_t)src & 15) == 0 && ld % 4 == 0) ? 1 : 0;
  const long long total = rows * (ld_dst / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > runtime().num_sms * 32) blocks = runtime().num_sms * 32;
  cvt_bf16_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(src, ld, rows, C, (__nv_bfloat16*)dst, ld_dst, vec_ok);
  return dp_check_launch();
}

extern "C" int dp_pack_conv_weight_bf16(const float* w, int32_t K, int32_t C, int32_t R, int32_t S, void* kc, void* ck, dp_stream_t stream) {
  DP_REQUIRE(w && (kc || ck), DP_ERR_NULL);
  DP_REQUIRE(K > 0 && C > 0 && R > 0 && S > 0, DP_ERR_SHAPE);
  const int Cp = wrow_bf16(C), Kp = wrow_bf16(K);
  long long total = (long long)R * S * ((long long)K * Cp > (long long)C * Kp ? (long long)K * Cp : (long long)C * Kp);
  int blocks = (int)((total + 255) / 256);
  if (blocks > runtime().num_sms * 16) blocks = runtime().num_sms * 16;
  pack_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, K, C, R * S, Cp, Kp, (__nv_bfloat16*)kc, (__nv_bfloat16*)ck);
  return dp_check_launch();
}
