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
#include <mutex>
#include "common.cuh"
#include "sm90.cuh"

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

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
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
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
int g_state = -1;
int g_num_sms = 132;   // H100 SXM; bf_init reads the device's count
std::mutex g_mutex;

int bf_init() {
  std::lock_guard<std::mutex> lk(g_mutex);
  if (g_state >= 0) return g_state;
  g_state = 0;
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess || major != 9) { (void)cudaGetLastError(); return 0; }
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
      qres != cudaDriverEntryPointSuccess) { (void)cudaGetLastError(); return 0; }
  g_encode = (EncodeTiledFn)fn;
  bool ok = true;
  for (const void* k : {(const void*)conv_bf16_kernel<1>, (const void*)conv_bf16_kernel<2>, (const void*)conv_bf16_kernel<3>,
                        (const void*)conv_bf16_kernel<4>, (const void*)wgrad_bf16_kernel<1>, (const void*)wgrad_bf16_kernel<2>,
                        (const void*)wgrad_bf16_kernel<3>, (const void*)wgrad_bf16_kernel<4>})
    ok = ok && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM) == cudaSuccess;
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  if (!ok) { (void)cudaGetLastError(); return 0; }
  g_state = 1;
  return 1;
}

bool make_map_bf16(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                   const cuuint32_t* box, int pix_stride = 1) {
  cuuint32_t estr[5] = {1, (cuuint32_t)pix_stride, (cuuint32_t)pix_stride, 1, 1};
  if (rank == 3) { estr[1] = 1; estr[2] = 1; }
  return g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// a box of `npix` pixels of an [N][H][W] grid as (bw, bh, bn) with bw*bh*bn == npix
bool pick_box(int npix, int H, int W, int& bw, int& bh, int& bn) {
  if (W >= npix) { if (W % npix) return false; bw = npix; bh = 1; bn = 1; return true; }
  if (npix % W) return false;
  bw = W;
  int rem = npix / W;
  if (H >= rem) { if (H % rem) return false; bh = rem; bn = 1; return true; }
  if (rem % H) return false;
  bh = H; bn = rem / H;
  return true;
}

int wrow_bf16(int c) { return (c + 63) & ~63; }

struct TapTable { int n; signed char dh[9], dw[9], wt[9]; };

TapTable dense_taps(int R, int S, int pad, bool flip) {
  TapTable t{};
  t.n = R * S;
  for (int r = 0; r < R; ++r)
    for (int s = 0; s < S; ++s) {
      int i = r * S + s;
      t.dh[i] = (signed char)(r - pad); t.dw[i] = (signed char)(s - pad);
      t.wt[i] = (signed char)(flip ? (R * S - 1 - i) : i);
    }
  return t;
}

// act: bf16 [Nimg][H*in_stride][W*in_stride][ld_act] view with Kg valid channels; w: bf16 [T][Nout][wrow_bf16(Kg)]; out fp32 view.
// dry = 1: only check eligibility.
int launch_bf16(const void* act, long long ld_act, int Nimg, int H, int W, int Kg, const void* w, int Nout, int T, const TapTable& taps,
                int os, int oa, int ob, int Ho, int Wo, float* out, long long ld_out, const float* bias, const float* rowadd,
                long long ld_rowadd, const float* residual, long long ld_res, int accumulate, cudaStream_t st, int in_stride, int dry) {
  if (!bf_init()) return DP_ERR_UNSUPPORTED;
  if (!dry && (!act || !w || !out)) return DP_ERR_NULL;
  if (ld_act % 8 || ((uintptr_t)act & 15) || ((uintptr_t)w & 15) || Kg < 8 || Nout < 1) return DP_ERR_UNSUPPORTED;
  int bw, bh, bn;
  if (!pick_box(BM, H, W, bw, bh, bn)) return DP_ERR_UNSUPPORTED;
  if (bw * in_stride > 256 || bh * in_stride > 256) return DP_ERR_UNSUPPORTED;
  // N tile: as wide as possible (<= 256) so the activation tile is fetched once; balanced over the tiles it takes, a multiple of 64
  // (one instantiation per width)
  const int n_tiles = (Nout + 255) / 256;
  int bn_tile = ((Nout + n_tiles - 1) / n_tiles + 63) & ~63;
  if (bn_tile > 256) bn_tile = 256;
  if (dry) return DP_OK;
  CUtensorMap mA, mB;
  {
    const cuuint64_t Hin = (cuuint64_t)H * in_stride, Win = (cuuint64_t)W * in_stride;
    cuuint64_t dims[4] = {(cuuint64_t)Kg, Win, Hin, (cuuint64_t)Nimg};
    cuuint64_t str[3] = {(cuuint64_t)ld_act * 2, Win * ld_act * 2, Hin * Win * ld_act * 2};
    cuuint32_t box[4] = {(cuuint32_t)KB, (cuuint32_t)(bw * in_stride), (cuuint32_t)(bh * in_stride), (cuuint32_t)bn};
    if (!make_map_bf16(&mA, act, 4, dims, str, box, in_stride)) return DP_ERR_UNSUPPORTED;
  }
  {
    const cuuint64_t ldb = (cuuint64_t)wrow_bf16(Kg);
    cuuint64_t dims[3] = {ldb, (cuuint64_t)Nout, (cuuint64_t)T};
    cuuint64_t str[2] = {ldb * 2, (cuuint64_t)Nout * ldb * 2};
    cuuint32_t box[3] = {(cuuint32_t)KB, (cuuint32_t)bn_tile, 1};
    if (!make_map_bf16(&mB, w, 3, dims, str, box)) return DP_ERR_UNSUPPORTED;
  }
  BfParams p{};
  p.Nimg = Nimg; p.Nout = Nout;
  p.ntaps = taps.n;
  for (int i = 0; i < 9; ++i) { p.dh[i] = taps.dh[i]; p.dw[i] = taps.dw[i]; p.wt[i] = taps.wt[i]; }
  p.os = os; p.oa = oa; p.ob = ob; p.Ho = Ho; p.Wo = Wo; p.in_stride = in_stride;
  p.kchunks = (Kg + KB - 1) / KB;
  p.bw = bw; p.bh = bh; p.bn = bn; p.tiles_w = W / bw; p.tiles_h = H / bh;
  p.y = out; p.ldy = ld_out; p.bias = bias; p.rowadd = rowadd; p.ld_rowadd = ld_rowadd; p.residual = residual; p.ld_res = ld_res;
  p.accumulate = accumulate;
  auto al16 = [](const void* q, long long ld) { return q == nullptr || ((((uintptr_t)q) & 15) == 0 && (ld % 4) == 0); };
  p.vec4 = (al16(out, ld_out) && al16(bias, 0) && al16(rowadd, ld_rowadd) && al16(residual, ld_res)) ? 1 : 0;
  const int stage_bytes = A_BYTES + bn_tile * 128;     // every tile starts 1024-byte aligned
  int stages = (MAX_SMEM - 2048) / stage_bytes;
  if (stages > 8) stages = 8;
  if (stages < 2) return DP_ERR_UNSUPPORTED;
  p.stages = stages;
  const int tiles_n = (Nimg + bn - 1) / bn;
  const int tiles_m = p.tiles_w * p.tiles_h * tiles_n, total = tiles_m * n_tiles;
  const int ctas = total < g_num_sms ? total : g_num_sms;
  const size_t smem = (size_t)stages * stage_bytes + 2048;
  switch (bn_tile / 64) {
    case 1: conv_bf16_kernel<1><<<ctas, THREADS, smem, st>>>(mA, mB, p, tiles_m, total); break;
    case 2: conv_bf16_kernel<2><<<ctas, THREADS, smem, st>>>(mA, mB, p, tiles_m, total); break;
    case 3: conv_bf16_kernel<3><<<ctas, THREADS, smem, st>>>(mA, mB, p, tiles_m, total); break;
    default: conv_bf16_kernel<4><<<ctas, THREADS, smem, st>>>(mA, mB, p, tiles_m, total); break;
  }
  return dp_check_launch();
}

bool conv_shape_ok(const dp_conv_bf16_args* a) {
  if (!a) return false;
  if (a->R != a->S || (a->R != 1 && a->R != 3) || a->pad_l != a->pad_t) return false;
  if (!((a->stride == 1 && a->pad_t == (a->R - 1) / 2) || (a->stride == 2 && a->R == 3 && (a->pad_t == 0 || a->pad_t == 1)))) return false;
  if (a->P * a->stride != a->H || a->Q * a->stride != a->W) return false;
  if (a->N <= 0 || a->H <= 0 || a->W <= 0 || a->C <= 0 || a->K <= 0) return false;
  return true;
}

int fprop_impl(const dp_conv_bf16_args* a, cudaStream_t st, int dry) {
  if (!conv_shape_ok(a) || a->ldx < a->C || a->ld_out < a->K) return DP_ERR_UNSUPPORTED;
  return launch_bf16(a->x_bf16, a->ldx, a->N, a->P, a->Q, a->C, a->w_bf16, a->K, a->R * a->S, dense_taps(a->R, a->S, a->pad_t, false), 1, 0, 0,
                     a->P, a->Q, a->out, a->ld_out, a->bias, a->rowadd, a->ld_rowadd, a->residual, a->ld_res,
                     (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0, st, a->stride, dry);
}

int dgrad_impl(const dp_conv_bf16_args* a, cudaStream_t st, int dry) {
  if (!conv_shape_ok(a) || a->lddy < a->K || a->ld_out < a->C) return DP_ERR_UNSUPPORTED;
  const int acc = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  if (a->stride == 1)
    return launch_bf16(a->dy_bf16, a->lddy, a->N, a->H, a->W, a->K, a->w_bf16, a->C, a->R * a->S, dense_taps(a->R, a->S, a->pad_t, true), 1, 0, 0,
                       a->H, a->W, a->out, a->ld_out, nullptr, nullptr, 0, nullptr, 0, acc, st, 1, dry);
  // stride 2: dx[2i+a, 2j+b] only sees taps with (a+pad-r), (b+pad-s) even -> 4 parity classes, each a dense GEMM over the dy grid
  TapTable cls[4];
  for (int ca = 0; ca < 2; ++ca)
    for (int cb = 0; cb < 2; ++cb) {
      TapTable& t = cls[ca * 2 + cb];
      t = TapTable{};
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
          int nh = ca + a->pad_t - r, nw = cb + a->pad_l - s;
          if ((nh & 1) || (nw & 1)) continue;
          t.dh[t.n] = (signed char)(nh / 2); t.dw[t.n] = (signed char)(nw / 2); t.wt[t.n] = (signed char)(r * 3 + s);
          ++t.n;
        }
      if (t.n == 0) return DP_ERR_UNSUPPORTED;
    }
  for (int ca = 0; ca < 2; ++ca)
    for (int cb = 0; cb < 2; ++cb) {
      int rc = launch_bf16(a->dy_bf16, a->lddy, a->N, a->P, a->Q, a->K, a->w_bf16, a->C, 9, cls[ca * 2 + cb], 2, ca, cb, a->H, a->W, a->out,
                           a->ld_out, nullptr, nullptr, 0, nullptr, 0, acc, st, 1, dry);
      if (rc != DP_OK) return rc;
      if (dry) break;
    }
  return DP_OK;
}

int wgrad_impl(const dp_conv_bf16_args* a, cudaStream_t st, int dry) {
  if (!conv_shape_ok(a) || a->splits < 1 || a->ldx < a->C || a->lddy < a->K) return DP_ERR_UNSUPPORTED;
  if (!bf_init()) return DP_ERR_UNSUPPORTED;
  if (!dry && (!a->x_bf16 || !a->dy_bf16 || !a->workspace)) return DP_ERR_NULL;
  if (a->ldx % 8 || a->lddy % 8 || ((uintptr_t)a->x_bf16 & 15) || ((uintptr_t)a->dy_bf16 & 15)) return DP_ERR_UNSUPPORTED;
  int bw, bh, bn;
  if (!pick_box(WG_PIX, a->P, a->Q, bw, bh, bn)) return DP_ERR_UNSUPPORTED;   // 64-pixel chunks of the dy grid
  if (a->N % bn) return DP_ERR_UNSUPPORTED;
  if (bw * a->stride > 256 || bh * a->stride > 256) return DP_ERR_UNSUPPORTED;
  if (dry) return DP_OK;
  CUtensorMap mDy, mX;
  {
    cuuint64_t dims[4] = {(cuuint64_t)a->K, (cuuint64_t)a->Q, (cuuint64_t)a->P, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->lddy * 2, (cuuint64_t)a->Q * a->lddy * 2, (cuuint64_t)a->P * a->Q * a->lddy * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
    if (!make_map_bf16(&mDy, a->dy_bf16, 4, dims, str, box)) return DP_ERR_UNSUPPORTED;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)a->C, (cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->ldx * 2, (cuuint64_t)a->W * a->ldx * 2, (cuuint64_t)a->H * a->W * a->ldx * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(bw * a->stride), (cuuint32_t)(bh * a->stride), (cuuint32_t)bn};
    if (!make_map_bf16(&mX, a->x_bf16, 4, dims, str, box, a->stride)) return DP_ERR_UNSUPPORTED;
  }
  WgBfParams p{};
  p.Nimg = a->N; p.H = a->P; p.W = a->Q; p.C = a->C; p.K = a->K; p.R = a->R; p.S = a->S; p.pad = a->pad_t; p.in_stride = a->stride;
  p.bw = bw; p.bh = bh; p.bn = bn; p.tiles_w = a->Q / bw; p.tiles_h = a->P / bh;
  p.total_chunks = p.tiles_w * p.tiles_h * (a->N / bn);
  p.chunks_per_split = (p.total_chunks + a->splits - 1) / a->splits;
  p.ct_width = dp_bf16_wgrad_ctile(a->C);
  p.c_tiles = (a->C + p.ct_width - 1) / p.ct_width;
  const int x_blocks = p.ct_width / 64;
  p.ws = a->workspace;
  const int stage_bytes = (2 + x_blocks) * BLK_BYTES;
  int stages = (MAX_SMEM - 2048) / stage_bytes;
  if (stages > 8) stages = 8;
  p.stages = stages;
  const int k_tiles = (a->K + 127) / 128;
  dim3 grid((unsigned)(k_tiles * p.c_tiles * a->R * a->S), (unsigned)a->splits);
  const size_t smem = (size_t)stages * stage_bytes + 2048;
  switch (x_blocks) {
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

extern "C" int dp_conv2d_fprop_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return fprop_impl(a, (cudaStream_t)s, 0); }
extern "C" int dp_conv2d_dgrad_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return dgrad_impl(a, (cudaStream_t)s, 0); }
extern "C" int dp_conv2d_wgrad_bf16(const dp_conv_bf16_args* a, dp_stream_t s) { return wgrad_impl(a, (cudaStream_t)s, 0); }
// op: 0 fprop, 1 dgrad, 2 wgrad.  DP_OK when the bf16 kernels take this shape (pointers are not needed), else DP_ERR_UNSUPPORTED.
extern "C" int dp_conv_bf16_eligible(const dp_conv_bf16_args* a, int op) {
  if (!a) return DP_ERR_NULL;
  dp_conv_bf16_args b = *a;     // alignment checks see aligned dummies
  b.x_bf16 = b.dy_bf16 = b.w_bf16 = nullptr;
  return op == 0 ? fprop_impl(&b, nullptr, 1) : op == 1 ? dgrad_impl(&b, nullptr, 1) : wgrad_impl(&b, nullptr, 1);
}

extern "C" int dp_cvt_bf16(const float* src, int64_t ld, int64_t rows, int32_t C, void* dst, int64_t ld_dst, dp_stream_t stream) {
  DP_REQUIRE(src && dst, DP_ERR_NULL);
  DP_REQUIRE(rows > 0 && C > 0 && ld >= C && ld_dst >= C && ld_dst % 8 == 0, DP_ERR_SHAPE);
  DP_REQUIRE(((uintptr_t)dst & 15) == 0, DP_ERR_ALIGN);
  const int vec_ok = (((uintptr_t)src & 15) == 0 && ld % 4 == 0) ? 1 : 0;
  const long long total = rows * (ld_dst / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > g_num_sms * 32) blocks = g_num_sms * 32;
  cvt_bf16_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(src, ld, rows, C, (__nv_bfloat16*)dst, ld_dst, vec_ok);
  return dp_check_launch();
}

extern "C" int dp_pack_conv_weight_bf16(const float* w, int32_t K, int32_t C, int32_t R, int32_t S, void* kc, void* ck, dp_stream_t stream) {
  DP_REQUIRE(w && (kc || ck), DP_ERR_NULL);
  DP_REQUIRE(K > 0 && C > 0 && R > 0 && S > 0, DP_ERR_SHAPE);
  const int Cp = wrow_bf16(C), Kp = wrow_bf16(K);
  long long total = (long long)R * S * ((long long)K * Cp > (long long)C * Kp ? (long long)K * Cp : (long long)C * Kp);
  int blocks = (int)((total + 255) / 256);
  if (blocks > g_num_sms * 16) blocks = g_num_sms * 16;
  pack_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, K, C, R * S, Cp, Kp, (__nv_bfloat16*)kc, (__nv_bfloat16*)ck);
  return dp_check_launch();
}
