// conv_tc.cu — wgmma / TMA implicit-GEMM convolution for sm_90a, fp32-grade through a THREE-PRODUCT SPLIT.
//
// fprop / dgrad / attention GEMMs (conv_tc_ps_kernel): 3 x FP16.  Every operand is scaled by a power of two taken from its "amax slot"
// (an upper bound of max|v|: dp_amax for activations / gradients, dp_pack_conv_weight_tc for weights) so that |s*v| < 2^14, then
//     s*v = hi + lo,   hi = fp16(s*v) (11 significant bits),  lo' = fp16((s*v - hi) * 2^11)            (22 bits kept, as 3xTF32 does)
//     x*w ~= [hi(x)*hi(w)] + 2^-11 * [hi(x)*lo'(w) + lo'(x)*hi(w)]
// with both brackets accumulated in fp32 registers (main | correction accumulator) by wgmma on fp16 operands — twice the rate of
// tf32 wgmma and half the shared-memory operand bytes.  Elements more than 2^28 below the tensor's maximum lose RELATIVE precision
// (absolute error <= 2^-50 of the maximum): below fp32 round-off of any sum they take part in.
// The weight gradient (wgrad_tc_kernel) uses the same split with both operands scaled by their own slots.
//
// GEMM view: M = N*H*W output pixels (tile of 128 = one TMA box of the NHWC activation), N = output channels, K = taps x input
// channels, one pipeline stage = (one tap, 64 channels).  The activation box is im2col-free: the tap shift is a coordinate offset,
// image borders are TMA out-of-bounds zero fill, stride 2 is a TMA element stride.
//
// Kernels (warpgroup roles: sm90.cuh):
//   conv_tc_ps_kernel     fprop / dgrad / NT GEMM: persistent (1 CTA per SM loops over (tile, K split) work items); each consumer
//                         warpgroup splits its 64 rows of the raw fp32 A boxes IN PLACE into fp16 hi | lo' tiles, B = pre-split fp16
//                         weights by TMA, 3 x 64 KB stages
//   splitk_epilogue_kernel  fixed-order sum of the K splits + the epilogue (small-M launches)
//   wgrad_tc_kernel       weight gradient: dY^T split in registers (wgmma A from registers), X split in place in shared memory
//                         (MN-major B), 64-pixel stages, split-K over pixels
//   pack / split / transpose helpers; dp_gemm_nt_tc runs the attention GEMMs on the persistent kernel.
#include <cuda.h>
#include <cuda_fp16.h>
#include <mutex>
#include "common.cuh"
#include "sm90.cuh"

namespace {
using namespace sm90;

constexpr int BM = 128, BK = 64;          // pixel tile, K elements (channels of one tap) per pipeline stage
constexpr int A_BYTES = BM * 32 * 4;      // 16 KB: one raw fp32 TMA box of 32 channels = one fp16 tile of 64 channels

struct TcParams {
  int Nimg, H, W;
  int Nout;            // GEMM N (valid output channels)
  int kchunks;         // ceil(Kg / 64)
  int bw, bh, bn, tiles_w, tiles_h;
  float* y; long long ldy;
  const float* bias;
  const float* rowadd; long long ld_rowadd;
  const float* residual; long long ld_res;
  int accumulate;
  int vec4;            // all epilogue pointers / strides are 16-byte aligned
  // generalised tap table (stride-2 dgrad runs as 4 parity classes with 1/2/2/4 taps each) and output pixel mapping
  int ntaps;
  signed char dh[9], dw[9], wt[9];
  int os, oa, ob, Ho, Wo;   // output pixel = (p*os + oa, q*os + ob) on an [Ho][Wo] grid
  int in_stride;            // strided fprop: input pixel = in_stride * output pixel + tap offset (the A map traverses W, H with that stride)
  float alpha;              // epilogue scale of the accumulator (attention logits); 1 for convolutions
  int b_from_img;           // batched GEMM: the B tile index is the tile's image (bn == 1) instead of a filter tap
  const uint32_t* amax_a;   // amax slots of the A operand (activation / gradient view) and of the B operand (weights / split activation)
  const uint32_t* amax_b;
  uint32_t* amax_out;       // optional amax slot of the output tensor
  // split-K (persistent kernel, launches with fewer tiles than half the SMs: the 4x4 / 8x8 / 16x16 levels): work item = (tile, K split);
  // a split walks `it_per_split` pipeline stages of the tile and writes its accumulator to ws[split][row][channel]
  // (row = tile_m * 128 + tile row, pitch ws_ld); splitk_epilogue_kernel sums the splits in fixed order and applies the epilogue
  int ksplit, it_per_split;
  float* ws; long long ws_split_stride; int ws_ld;
  // general-geometry fprop (conv_tc_ps_kernel<true>): the M tiles are 128 consecutive flattened output pixels m = (n*P + p)*Q + q of an
  // [N][P][Q] grid (the launcher sets Nimg = Ho = 1, Wo = M, bw = 128, so the epilogue maps row -> m = tile_m*128 + row), and the producer
  // warpgroup gathers each stage's A rows from the NHWC input x [N][H][W][ldx] with cp.async: taps walked arithmetically (r, s) = (tap / S,
  // tap % S), padding and tails as zero fill.  relu: y = max(y, 0) after every epilogue term (DP_CONV_RELU)
  const float* gx; long long gldx;
  int gH, gW, gC, gQ, gPQ, gS, gstride, gpad_t, gpad_l, gM;
  int relu;
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
// 16-byte cp.async with zero fill past src_bytes (0 = nothing read), and the mbarrier arrival that fires when this thread's copies land
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// amax slot -> power-of-two scale.  E = biased exponent of the bound (|v| < 2^(E-126)), clamped so that both factors are normal floats;
// up = 2^(140-E) brings the operand below 2^14 (fp16 overflows at 65504), dn = 2^(E-140) undoes it in the epilogue.
__device__ __forceinline__ int amax_exponent(const uint32_t* slot) {
  const int E = (int)((__ldg(slot) >> 23) & 0xFFu);
  return min(max(E, 14), 254);
}
__device__ __forceinline__ float scale_up(int E) { return __uint_as_float((uint32_t)(267 - E) << 23); }
__device__ __forceinline__ float scale_dn(int E) { return __uint_as_float((uint32_t)(E - 13) << 23); }
constexpr float LO_SCALE = 2048.f, LO_UNSCALE = 1.f / 2048.f;   // lo' = lo * 2^11 keeps the residual in fp16's normal range
// two scaled values -> packed fp16 hi pair and lo' pair (low half = first element = lower address)
__device__ __forceinline__ void split2(float a, float b, uint32_t& h, uint32_t& l) {
  const __half2 hh = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn((a - hf.x) * LO_SCALE, (b - hf.y) * LO_SCALE);
  h = *reinterpret_cast<const uint32_t*>(&hh);
  l = *reinterpret_cast<const uint32_t*>(&ll);
}
// one scaled fp32 value -> fp16 hi and lo' = (v - hi) * 2^11
__device__ __forceinline__ void split1(float v, __half& h, __half& l) {
  h = __float2half_rn(v);
  l = __float2half_rn((v - __half2float(h)) * LO_SCALE);
}

// ------------------------------------------------------------------------------------------------ persistent fprop / dgrad / NT GEMM
// Stage = [A box k 0..31 | A box k 32..63 | b_hi | b_lo'] x 16 KB.  Consumer warpgroup c splits its tile rows 64c .. 64c+63 IN PLACE
// (thread = row, raw box), then main += a_hi b_hi, corr += a_hi b_lo' + a_lo' b_hi per 16-element K step.  One wgmma group stays in
// flight, so a warpgroup splits stage i+1 while the tensor cores run stage i.
constexpr int PS_STAGES = 3, PS_BN = 128;
constexpr int PS_B_BYTES = PS_BN * BK * 2;
constexpr int PS_STAGE_BYTES = 2 * A_BYTES + 2 * PS_B_BYTES;

template <bool ANY>
__global__ void __launch_bounds__(THREADS, 1)
conv_tc_ps_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapBh,
                  const __grid_constant__ CUtensorMap mapBl, const TcParams p, const int tiles_m, const int total_tiles) {
  const int total_work = total_tiles * p.ksplit;     // work item wi = split * total_tiles + tile (the splits of one tile run on different SMs)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t pad_to = ((raw + 1023u) & ~1023u) - raw;
  uint8_t* smem = smem_raw + pad_to;
  const uint32_t sbase = raw + pad_to;
  const uint32_t bar0 = sbase + PS_STAGES * PS_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (PS_STAGES + s); };
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    // full: the TMA thread's expect_tx (+ one cp.async arrival per gathering producer thread); empty: one arrival per consumer warp
    for (int s = 0; s < PS_STAGES; ++s) { mbar_init(full_bar(s), ANY ? 1 + 128 : 1); mbar_init(empty_bar(s), 8); }
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
    if constexpr (ANY) {
      // thread t gathers A row t of every stage: 64 fp32 channels of one input pixel, 16 x 16 bytes, into the two raw boxes at the
      // 128-byte-swizzled positions TMA would have used (chunk j of row t at j ^ (t & 7)), so the consumers are unchanged
      const int t = threadIdx.x;
      if (t == 0) { prefetch_map(&mapBh); prefetch_map(&mapBl); }
      const uint32_t sw = (uint32_t)(t & 7);
      uint32_t g = 0;
      for (int wi = blockIdx.x; wi < total_work; wi += gridDim.x) {
        const int tile = wi % total_tiles, it0 = (wi / total_tiles) * p.it_per_split, it1 = min(iters_per_tile, it0 + p.it_per_split);
        const int nblk = tile / tiles_m, m = (tile - nblk * tiles_m) * BM + t;
        const bool mv = m < p.gM;
        const int n = mv ? m / p.gPQ : 0, rem = m - n * p.gPQ, pq = rem / p.gQ;
        const int hb = pq * p.gstride - p.gpad_t, wb = (rem - pq * p.gQ) * p.gstride - p.gpad_l;
        const float* xn = p.gx + (long long)n * p.gH * p.gW * p.gldx;
        for (int it = it0; it < it1; ++it, ++g) {
          const int s = g % PS_STAGES;
          const uint32_t ph = (g / PS_STAGES) & 1u;
          mbar_wait(empty_bar(s), ph ^ 1u);
          const int tap = it / p.kchunks, kc = it - tap * p.kchunks;
          const int r = tap / p.gS, h = hb + r, w = wb + (tap - r * p.gS);
          const uint32_t st = sbase + s * PS_STAGE_BYTES;
          if (t == 0) {
            mbar_expect_tx(full_bar(s), 2 * PS_B_BYTES);
            tma_load_3d(st + 2 * A_BYTES, &mapBh, full_bar(s), kc * BK, nblk * PS_BN, tap);
            tma_load_3d(st + 2 * A_BYTES + PS_B_BYTES, &mapBl, full_bar(s), kc * BK, nblk * PS_BN, tap);
          }
          const bool v = mv && h >= 0 && h < p.gH && w >= 0 && w < p.gW;
          const int cleft = v ? p.gC - kc * BK : 0;       // valid channels from the stage's first one
          const float* src = v ? xn + ((long long)h * p.gW + w) * p.gldx + kc * BK : p.gx;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int nb = min(max(cleft - 4 * j, 0), 4) * 4;
            cp_async16(st + (j >> 3) * A_BYTES + t * 128 + ((((uint32_t)j & 7u) ^ sw) << 4), nb ? src + 4 * j : p.gx, (uint32_t)nb);
          }
          cp_async_mbar_arrive(full_bar(s));
        }
      }
      return;
    }
    if (threadIdx.x == 0) {
      prefetch_map(&mapA); prefetch_map(&mapBh); prefetch_map(&mapBl);
      uint32_t g = 0;
      for (int wi = blockIdx.x; wi < total_work; wi += gridDim.x) {
        const int tile = wi % total_tiles, it0 = (wi / total_tiles) * p.it_per_split, it1 = min(iters_per_tile, it0 + p.it_per_split);
        int q0, p0, n0, nblk;
        tile_coords(tile, q0, p0, n0, nblk);
        for (int it = it0; it < it1; ++it, ++g) {
          const int s = g % PS_STAGES;
          const uint32_t ph = (g / PS_STAGES) & 1u;
          mbar_wait(empty_bar(s), ph ^ 1u);
          mbar_expect_tx(full_bar(s), PS_STAGE_BYTES);
          const int tap = it / p.kchunks, kc = it - tap * p.kchunks;
          const uint32_t st = sbase + s * PS_STAGE_BYTES;
          const int aw = q0 * p.in_stride + p.dw[tap], ah = p0 * p.in_stride + p.dh[tap];
          tma_load_4d(st, &mapA, full_bar(s), kc * BK, aw, ah, n0);
          tma_load_4d(st + A_BYTES, &mapA, full_bar(s), kc * BK + 32, aw, ah, n0);     // past the last channel: TMA zero fill
          const int tapb = p.b_from_img ? n0 : p.wt[tap];
          tma_load_3d(st + 2 * A_BYTES, &mapBh, full_bar(s), kc * BK, nblk * PS_BN, tapb);
          tma_load_3d(st + 2 * A_BYTES + PS_B_BYTES, &mapBl, full_bar(s), kc * BK, nblk * PS_BN, tapb);
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1;                              // consumer warpgroup: tile rows 64c .. 64c + 63
  const int warp = tid >> 5, lane = tid & 31;
  const int r = 64 * c + (tid & 63), h = tid >> 6;   // splitter task: row r, raw box h (K elements 32h .. 32h + 31 of the stage)
  const uint32_t sw = (uint32_t)(r & 7);             // 128B swizzle: 16-byte chunk j of row r sits at chunk position j ^ (r & 7)
  const float sa = scale_up(amax_exponent(p.amax_a));
  // accumulators hold (s_a s_b) x the products: f1 * f2 undoes the two power-of-two operand scales (two factors: their product may underflow)
  const float f1 = scale_dn(amax_exponent(p.amax_a)), f2 = scale_dn(amax_exponent(p.amax_b)) * p.alpha;
  auto fin = [&](float main, float corr) { return fmaf(corr, LO_UNSCALE, main) * f1 * f2; };
  float amax = 0.f;         // max |value written| by this thread (split launches: splitk_epilogue_kernel writes, and tracks, the outputs)
  uint32_t g = 0;
  for (int wi = blockIdx.x; wi < total_work; wi += gridDim.x) {
    const int tile = wi % total_tiles, it0 = (wi / total_tiles) * p.it_per_split, it1 = min(iters_per_tile, it0 + p.it_per_split);
    float acc[64], cor[64];
    int prev_s = 0;
    for (int it = it0; it < it1; ++it, ++g) {
      const int s = g % PS_STAGES;
      const uint32_t ph = (g / PS_STAGES) & 1u;
      mbar_wait(full_bar(s), ph);
      uint8_t* a0 = smem + s * PS_STAGE_BYTES + r * 128;      // row r of the k 0..31 box  -> row r of a_hi
      uint8_t* a1 = a0 + A_BYTES;                              // row r of the k 32..63 box -> row r of a_lo'
      const uint8_t* src = h ? a1 : a0;
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const float4*>(src + ((j ^ sw) << 4));
      named_sync(1 + c, 128);                                  // both halves of every row of this warpgroup have read it
#pragma unroll
      for (int m = 0; m < 4; ++m) {        // output chunk 4h + m = K elements 32h + 8m .. 32h + 8m + 7
        const float4 x0 = v[2 * m], x1 = v[2 * m + 1];
        uint4 hq, lq;
        split2(x0.x * sa, x0.y * sa, hq.x, lq.x);
        split2(x0.z * sa, x0.w * sa, hq.y, lq.y);
        split2(x1.x * sa, x1.y * sa, hq.z, lq.z);
        split2(x1.z * sa, x1.w * sa, hq.w, lq.w);
        const uint32_t pos = (uint32_t)(((4 * h + m) ^ sw) << 4);
        *reinterpret_cast<uint4*>(a0 + pos) = hq;
        *reinterpret_cast<uint4*>(a1 + pos) = lq;
      }
      fence_proxy_async();
      named_sync(1 + c, 128);                                  // the warpgroup's 64 rows are split
      const uint32_t st = sbase + s * PS_STAGE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {      // one instruction = 16 fp16 along K = 32 bytes of every 128-byte row
        const uint64_t a_hi = desc_k(st + c * 8192 + k * 32), a_lo = desc_k(st + A_BYTES + c * 8192 + k * 32);
        const uint64_t b_hi = desc_k(st + 2 * A_BYTES + k * 32), b_lo = desc_k(st + 2 * A_BYTES + PS_B_BYTES + k * 32);
        const uint32_t first = (it > it0 || k > 0) ? 1u : 0u;
        wgmma_f16_n128<0, 0>(acc, a_hi, b_hi, first);
        wgmma_f16_n128<0, 0>(cor, a_hi, b_lo, first);
        wgmma_f16_n128<0, 0>(cor, a_lo, b_hi, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();                        // the previous stage's MMAs have read their operands: hand it back to TMA
      if (it > it0 && lane == 0) mbar_arrive(empty_bar(prev_s));
      prev_s = s;
    }
    wgmma_wait<0>();
    fence_regs(acc); fence_regs(cor);
    if (lane == 0) mbar_arrive(empty_bar(prev_s));

    int q0, p0, n0, nblk;
    tile_coords(tile, q0, p0, n0, nblk);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = 64 * c + 16 * warp + (lane >> 2) + 8 * i;
      const int cb = 2 * (lane & 3);
      if (p.ksplit > 1) {   // split-K: partial sums into this split's slab of the (padded) workspace; splitk_epilogue_kernel finishes
        float* wrow = p.ws + (long long)(wi / total_tiles) * p.ws_split_stride + ((long long)(tile - nblk * tiles_m) * BM + row) * p.ws_ld + nblk * PS_BN;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *reinterpret_cast<float2*>(wrow + 8 * j + cb) =
              make_float2(fin(acc[4 * j + 2 * i], cor[4 * j + 2 * i]), fin(acc[4 * j + 2 * i + 1], cor[4 * j + 2 * i + 1]));
        continue;
      }
      const int w_l = row % p.bw, h_l = (row / p.bw) % p.bh, n_l = row / (p.bw * p.bh);
      const int img = n0 + n_l;
      if (img >= p.Nimg) continue;
      if constexpr (ANY) { if (q0 + w_l >= p.Wo) continue; }   // the tail of the last flattened tile
      const long long m = ((long long)img * p.Ho + ((p0 + h_l) * p.os + p.oa)) * p.Wo + ((q0 + w_l) * p.os + p.ob);
      float* yrow = p.y + m * p.ldy;
      const float* rrow = p.residual ? p.residual + m * p.ld_res : nullptr;
      const float* arow2 = p.rowadd ? p.rowadd + (long long)img * p.ld_rowadd : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = nblk * PS_BN + 8 * j + cb;
        float o[2] = {fin(acc[4 * j + 2 * i], cor[4 * j + 2 * i]), fin(acc[4 * j + 2 * i + 1], cor[4 * j + 2 * i + 1])};
        if (p.vec4 && col + 2 <= p.Nout) {
          if (p.bias) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.bias + col)); o[0] += t.x; o[1] += t.y; }
          if (arow2) { const float2 t = __ldg(reinterpret_cast<const float2*>(arow2 + col)); o[0] += t.x; o[1] += t.y; }
          if (rrow) { const float2 t = __ldg(reinterpret_cast<const float2*>(rrow + col)); o[0] += t.x; o[1] += t.y; }
          float2* dst = reinterpret_cast<float2*>(yrow + col);
          if (p.accumulate) { const float2 t = *dst; o[0] += t.x; o[1] += t.y; }
          if constexpr (ANY) { if (p.relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); } }
          *dst = make_float2(o[0], o[1]);
          amax = fmaxf(amax, fmaxf(fabsf(o[0]), fabsf(o[1])));
        } else {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int cc = col + e;
            if (cc < p.Nout) {
              float ov = o[e];
              if (p.bias) ov += __ldg(p.bias + cc);
              if (arow2) ov += __ldg(arow2 + cc);
              if (rrow) ov += __ldg(rrow + cc);
              if (p.accumulate) ov += yrow[cc];
              if constexpr (ANY) { if (p.relu) ov = fmaxf(ov, 0.f); }
              yrow[cc] = ov;
              amax = fmaxf(amax, fabsf(ov));
            }
          }
        }
      }
    }
  }
  if (p.amax_out && p.ksplit == 1) amax_commit(p.amax_out, amax);
}

// Sums the K splits of conv_tc_ps_kernel in fixed order (deterministic) and applies its epilogue: bias, per-image row, residual,
// accumulate, the (strided) output pixel mapping.  One thread per (GEMM row, 4 channels).
__global__ void __launch_bounds__(256) splitk_epilogue_kernel(const TcParams p, const int tiles_m) {
  const int c4 = (p.Nout + 3) >> 2;
  const long long total = (long long)tiles_m * BM * c4;
  float amax = 0.f;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long grow = i / c4;
    const int c = (int)(i - grow * c4) << 2;
    const int tile_m = (int)(grow / BM), row = (int)(grow - (long long)tile_m * BM);
    const int tw = tile_m % p.tiles_w, th = (tile_m / p.tiles_w) % p.tiles_h, tn = tile_m / (p.tiles_w * p.tiles_h);
    const int w_l = row % p.bw, h_l = (row / p.bw) % p.bh, n_l = row / (p.bw * p.bh);
    const int img = tn * p.bn + n_l;
    if (img >= p.Nimg) continue;
    const float* src = p.ws + grow * p.ws_ld + c;
    float4 acc = *reinterpret_cast<const float4*>(src);
    for (int ks = 1; ks < p.ksplit; ++ks) {
      const float4 t = *reinterpret_cast<const float4*>(src + ks * p.ws_split_stride);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    float o[4] = {acc.x, acc.y, acc.z, acc.w};     // the splits were written with the operand scales and alpha already undone
    const long long m = ((long long)img * p.Ho + ((th * p.bh + h_l) * p.os + p.oa)) * p.Wo + ((tw * p.bw + w_l) * p.os + p.ob);
    float* yrow = p.y + m * p.ldy;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int cc = c + e;
      if (cc < p.Nout) {
        float v = o[e];
        if (p.bias) v += __ldg(p.bias + cc);
        if (p.rowadd) v += __ldg(p.rowadd + (long long)img * p.ld_rowadd + cc);
        if (p.residual) v += __ldg(p.residual + m * p.ld_res + cc);
        if (p.accumulate) v += yrow[cc];
        yrow[cc] = v;
        amax = fmaxf(amax, fabsf(v));
      }
    }
  }
  if (p.amax_out) amax_commit(p.amax_out, amax);
}

// The same for conv_tc_ps_kernel<true>: workspace row m is output pixel m of the flattened [M][ldy] view (rows past M are tile padding),
// ReLU after the fixed-order sum of the splits.
__global__ void __launch_bounds__(256) splitk_flat_epilogue_kernel(const TcParams p) {
  const int c4 = (p.Nout + 3) >> 2;
  const long long total = (long long)p.gM * c4;
  float amax = 0.f;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long m = i / c4;
    const int c = (int)(i - m * c4) << 2;
    const float* src = p.ws + m * p.ws_ld + c;
    float4 acc = *reinterpret_cast<const float4*>(src);
    for (int ks = 1; ks < p.ksplit; ++ks) {
      const float4 t = *reinterpret_cast<const float4*>(src + ks * p.ws_split_stride);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    const float o[4] = {acc.x, acc.y, acc.z, acc.w};
    float* yrow = p.y + m * p.ldy;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int cc = c + e;
      if (cc < p.Nout) {
        float v = o[e];
        if (p.bias) v += __ldg(p.bias + cc);
        if (p.residual) v += __ldg(p.residual + m * p.ld_res + cc);
        if (p.accumulate) v += yrow[cc];
        if (p.relu) v = fmaxf(v, 0.f);
        yrow[cc] = v;
        amax = fmaxf(amax, fabsf(v));
      }
    }
  }
  if (p.amax_out) amax_commit(p.amax_out, amax);
}

// ------------------------------------------------------------------------------------------------ wgrad
// dW[k][tap][c] = sum_pixels dy[pix][k] * x[pix @ tap][c]: M = out-channels (128 per tile), N = in-channels of one tap (128 per tile),
// GEMM-K = pixels, 64 per pipeline stage.  Both operands are pixel-major fp32 activations, i.e. MN-major for this product.
// A stage holds 8 raw TMA boxes [64 px][32 ch]: dy in [0, 32 KB), x in [32 KB, 64 KB); the x boxes of channels [64j, 64j+32) and
// [64j+32, 64j+64) land where the fp16 blocks x_hi[j] and x_lo'[j] will live ([hi0 | hi1 | lo0 | lo1], MN-major SWIZZLE_128B: LBO = 8 KB
// between 64-channel blocks).  Consumer warpgroup c splits x block c in place (thread = pixel row) and reads its 64 out-channels of dy
// straight into wgmma A fragments, split in registers (dy is never written back; the fragment rows also sum the bias gradient), then
// main += dy_hi[c] x_hi, corr += dy_hi[c] x_lo' + dy_lo'[c] x_hi.
// grid = (k tiles * c tiles * taps, splits): split z covers pixel chunks [z*cps, (z+1)*cps) and writes its partial
// tile to workspace[z][k][tap*C + c]; dp_conv2d_wgrad_reduce sums splits in fixed order (deterministic).
struct WgParams {
  int Nimg, H, W, C, K;
  int R, S, pad;
  int bw, bh, bn, tiles_w, tiles_h;   // 64-pixel box of the dy grid
  int total_chunks, chunks_per_split;
  int c_tiles;
  float* ws;
  int in_stride;             // x pixel = in_stride * dy pixel + tap offset
  const uint32_t* amax_x; const uint32_t* amax_y;
  float* bias_ws;            // optional [splits][K]: column sums of dy over this split's pixels (written by the tap 0 / c-tile 0 CTAs)
};
constexpr int WG_KPIX = 64;                  // pixels per stage
constexpr int WG_BLK = WG_KPIX * 128;        // 8 KB: one raw fp32 box [64 px][32 ch] = one fp16 block [64 px][64 ch]
constexpr int WG_STAGES = 3, WG_STAGE_BYTES = 8 * WG_BLK;

__global__ void __launch_bounds__(THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap mapDy, const __grid_constant__ CUtensorMap mapX, const WgParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t pad_to = ((raw + 1023u) & ~1023u) - raw;
  uint8_t* smem = smem_raw + pad_to;
  const uint32_t sbase = raw + pad_to;
  const uint32_t bar0 = sbase + WG_STAGES * WG_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (WG_STAGES + s); };
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
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
  const int num_iters = max(0, chunk1 - chunk0);   // 0 for a trailing empty split: its workspace tile is zero-filled
  // 32-channel boxes that hold valid channels (pruned widths: 96 / 179 / 358 ...): boxes past the last channel are neither loaded nor
  // split — their accumulator rows / columns are never stored, so whatever the stage buffers still hold there is harmless
  const int dy_boxes = min(4, (p.K - kt * 128 + 31) >> 5), x_boxes = min(4, (p.C - ct * 128 + 31) >> 5);

  if (wg == 0) {
    setmaxnreg_dec<24>();      // the TMA loop fits in 24: consumers get 240 (2 x 32 dy fragments + 128 accumulators + the x split)
    if (threadIdx.x == 0) {
      prefetch_map(&mapDy); prefetch_map(&mapX);
      for (int it = 0; it < num_iters; ++it) {
        const int s = it % WG_STAGES;
        const uint32_t ph = (uint32_t)(it / WG_STAGES) & 1u;
        mbar_wait(empty_bar(s), ph ^ 1u);
        mbar_expect_tx(full_bar(s), (uint32_t)((dy_boxes + x_boxes) * WG_BLK));
        const int chunk = chunk0 + it;
        const int tw = chunk % p.tiles_w;
        const int th = (chunk / p.tiles_w) % p.tiles_h;
        const int tn = chunk / (p.tiles_w * p.tiles_h);
        const int q0 = tw * p.bw, p0 = th * p.bh, n0 = tn * p.bn;
        const uint32_t st = sbase + s * WG_STAGE_BYTES;
        const int xw = q0 * p.in_stride + sx - p.pad, xh = p0 * p.in_stride + r - p.pad;
#pragma unroll
        for (int b = 0; b < 4; ++b) {   // box b = channels [32b, 32b+32) of the tile -> block b >> 1, raw half b & 1
          const uint32_t slot = (uint32_t)((b & 1) * 2 + (b >> 1));
          if (b < dy_boxes) tma_load_4d(st + slot * WG_BLK, &mapDy, full_bar(s), kt * 128 + b * 32, q0, p0, n0);
          if (b < x_boxes) tma_load_4d(st + (4 + slot) * WG_BLK, &mapX, full_bar(s), ct * 128 + b * 32, xw, xh, n0);
        }
      }
    }
    return;
  }
  setmaxnreg_inc<240>();
  const int c = wg - 1;                       // consumer warpgroup: dy block c (out-channels 64c .. 64c+63) and x block c
  const int warp = tid >> 5, lane = tid & 31;
  const int Ey = amax_exponent(p.amax_y), Ex = amax_exponent(p.amax_x);
  const float sy = scale_up(Ey), sxs = scale_up(Ex);
  // dy^T fragment (A from registers): out-channel rows 16 warp + lane/4 (+8) of block c, pixel pairs 2 (lane%4) + {0, 1} (+8) of each
  // 16-pixel step.  Both rows lie in raw box 2c + warp/2 (slot (warp/2) * 2 + c).  Pixel p's 16-byte chunk j sits at j ^ (p & 7), and
  // p & 7 = 2 (lane%4) + e for every step: the per-pixel loads of a warp are bank-conflict free
  const bool dy_valid = 2 * c + (warp >> 1) < dy_boxes;
  // address of (row, pixel 0) in a stage; row + 8 flips chunk bit 1 (XOR 32 B), pixel + 1 flips row bit 0 and chunk bit 0 (XOR 144 B)
  const uint32_t cb = (uint32_t)(16 * (warp & 1) + (lane >> 2)), pe = (uint32_t)(2 * (lane & 3));
  const uint32_t dy_off = (uint32_t)((warp >> 1) * 2 + c) * WG_BLK + pe * 128 + (((cb >> 2) ^ pe) << 4) + (cb & 3) * 4;
  // x task: pixel row xp of block c, raw box xh (channels 32 xh .. 32 xh + 31 of the block)
  const int xp = tid & 63, xh = tid >> 6;
  const bool x_valid = 2 * c + xh < x_boxes;
  const uint32_t xsw = (uint32_t)(xp & 7);
  float bsum[2] = {0.f, 0.f};                 // sums of this thread's pixels of its two out-channel rows over the split (bias gradient)
  float acc[64], cor[64];
  int prev_s = 0;
  // One stage: x block c split in place (B, both warpgroups read both blocks), dy^T fragments of four 16-pixel steps split into
  // fah / fal, then 12 MMAs.  The MMAs of the stage before still read the other fragment set, so stages alternate between two sets.
  auto stage = [&](uint32_t (&fah)[4][4], uint32_t (&fal)[4][4], const int it) {
    const int s = it % WG_STAGES;
    const uint32_t ph = (uint32_t)(it / WG_STAGES) & 1u;
    mbar_wait(full_bar(s), ph);
    uint8_t* stp = smem + s * WG_STAGE_BYTES;
    uint8_t* x0 = stp + 4 * WG_BLK + c * WG_BLK + xp * 128;     // row xp of x_hi[c] (over the raw box of channels 64c .. 64c+31)
    uint8_t* x1 = x0 + 2 * WG_BLK;                              // row xp of x_lo'[c]
    float4 xv[8];
    if (x_valid) {
      const uint8_t* src = xh ? x1 : x0;
#pragma unroll
      for (int j = 0; j < 8; ++j) xv[j] = *reinterpret_cast<const float4*>(src + ((j ^ xsw) << 4));
    }
    named_sync(1 + c, 128);                   // block c of x has been read
    if (x_valid) {
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const float4 u0 = xv[2 * m], u1 = xv[2 * m + 1];
        uint4 hq, lq;
        split2(u0.x * sxs, u0.y * sxs, hq.x, lq.x);
        split2(u0.z * sxs, u0.w * sxs, hq.y, lq.y);
        split2(u1.x * sxs, u1.y * sxs, hq.z, lq.z);
        split2(u1.z * sxs, u1.w * sxs, hq.w, lq.w);
        const uint32_t pos = (uint32_t)(((4 * xh + m) ^ xsw) << 4);
        *reinterpret_cast<uint4*>(x0 + pos) = hq;
        *reinterpret_cast<uint4*>(x1 + pos) = lq;
      }
    }
    fence_proxy_async();
    named_sync(3, 256);                       // both blocks of x are split (each warpgroup's B spans both)
    if (dy_valid) {
#pragma unroll
      for (int k = 0; k < WG_KPIX / 16; ++k)
#pragma unroll
        for (int q = 0; q < 4; ++q) {          // fragment register q: row +8 (q & 1), pixels +8 (q >> 1)
          const uint8_t* d = stp + (16 * k + 8 * (q >> 1)) * 128;
          const float v0 = *reinterpret_cast<const float*>(d + (dy_off ^ (32u * (q & 1))));
          const float v1 = *reinterpret_cast<const float*>(d + (dy_off ^ (32u * (q & 1) + 144u)));
          bsum[q & 1] += v0 + v1;
          split2(v0 * sy, v1 * sy, fah[k][q], fal[k][q]);
        }
    } else {     // channels past the last box: rows that are never stored
#pragma unroll
      for (int k = 0; k < WG_KPIX / 16; ++k)
#pragma unroll
        for (int q = 0; q < 4; ++q) fah[k][q] = fal[k][q] = 0u;
    }
    const uint32_t st = sbase + s * WG_STAGE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < WG_KPIX / 16; ++k) {     // 16 pixels per instruction = two 8-pixel groups (2 KB) further into every block
      const uint64_t b_hi = desc_mn(st + 4 * WG_BLK + k * 2048, WG_BLK), b_lo = desc_mn(st + 6 * WG_BLK + k * 2048, WG_BLK);
      const uint32_t first = (it > 0 || k > 0) ? 1u : 0u;
      wgmma_f16_n128_rs<1>(acc, fah[k], b_hi, first);
      wgmma_f16_n128_rs<1>(cor, fah[k], b_lo, first);
      wgmma_f16_n128_rs<1>(cor, fal[k], b_hi, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0 && lane == 0) mbar_arrive(empty_bar(prev_s));
    prev_s = s;
  };
  // the odd tail stays outside the loop: on every path a set is rewritten only after the group that read it has retired
  uint32_t fah0[4][4], fal0[4][4], fah1[4][4], fal1[4][4];
  int it = 0;
  for (; it + 1 < num_iters; it += 2) {
    stage(fah0, fal0, it);
    stage(fah1, fal1, it + 1);
  }
  if (it < num_iters) stage(fah0, fal0, it);
  wgmma_wait<0>();
  fence_regs(acc); fence_regs(cor);
  // the four lanes of a row hold its pixel columns: fixed-order butterfly, every lane ends with the row's sum
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 1);
    bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 2);
  }
  const float f1 = scale_dn(Ey), f2 = scale_dn(Ex);
  const long long TC_ = (long long)T * p.C;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kout = kt * 128 + 64 * c + 16 * warp + (lane >> 2) + 8 * i;
    if (kout >= p.K) continue;
    if (p.bias_ws && tap == 0 && ct == 0 && (lane & 3) == 0) p.bias_ws[(long long)blockIdx.y * p.K + kout] = bsum[i];   // 0 for an empty split
    float* wrow = p.ws + ((long long)blockIdx.y * p.K + kout) * TC_ + (long long)tap * p.C;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = ct * 128 + 8 * j + 2 * (lane & 3) + e;
        // an empty split accumulated nothing (the registers hold garbage): it contributes zeros
        if (col < p.C) wrow[col] = num_iters ? fmaf(cor[4 * j + 2 * i + e], LO_UNSCALE, acc[4 * j + 2 * i + e]) * f1 * f2 : 0.f;
      }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
int g_tc_state = -1;  // -1 unknown, 0 unavailable, 1 ok
int g_num_sms = 132;   // H100 SXM; tc_init reads the device's count
std::mutex g_tc_mutex;
constexpr int PS_SMEM = PS_STAGES * PS_STAGE_BYTES + 2048;
constexpr int WG_SMEM = WG_STAGES * WG_STAGE_BYTES + 2048;

// Row length (fp16 elements) of the packed weight tiles (dp_pack_conv_weight_tc): rows longer than 64 are zero-padded to a multiple of
// 64 elements (128 B) so that every 64-element TMA box row is exactly one aligned 128-byte line; short rows to a multiple of 8 (the TMA
// 16-byte stride rule).  With 16-byte padding only, pruned widths (90 / 179 input channels) ran 20-25 % slower (round 1, 3xTF32 rows).
static int wrow(int c) { return c > 64 ? ((c + 63) & ~63) : ((c + 7) & ~7); }

int tc_init() {
  std::lock_guard<std::mutex> lk(g_tc_mutex);
  if (g_tc_state >= 0) return g_tc_state;
  g_tc_state = 0;
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess || major != 9) { (void)cudaGetLastError(); return 0; }
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
      qres != cudaDriverEntryPointSuccess) { (void)cudaGetLastError(); return 0; }
  g_encode = (EncodeTiledFn)fn;
  bool ok = cudaFuncSetAttribute(conv_tc_ps_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PS_SMEM) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(conv_tc_ps_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PS_SMEM) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM) == cudaSuccess;
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  if (!ok) { (void)cudaGetLastError(); return 0; }
  (void)cudaGetLastError();
  g_tc_state = 1;
  return 1;
}

// pix_stride > 1 (strided convolution): dims 1 and 2 (W, H) are traversed with that element stride; the caller passes the box
// extents in traversed elements (box = loaded pixels x pix_stride)
bool make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
              const cuuint32_t* box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B, int pix_stride = 1,
              CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT32) {
  cuuint32_t estr[5] = {1, (cuuint32_t)pix_stride, (cuuint32_t)pix_stride, 1, 1};
  CUresult r = g_encode(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// 128-pixel box of an [N][H][W] grid
bool pick_box(int N, int H, int W, int& bw, int& bh, int& bn) {
  if (W >= BM) {
    if (W % BM) return false;
    bw = BM; bh = 1; bn = 1; return true;
  }
  if (BM % W) return false;
  bw = W;
  int rem = BM / W;
  if (H >= rem) {
    if (H % rem) return false;
    bh = rem; bn = 1; return true;
  }
  if (rem % H) return false;
  bh = H; bn = rem / H;
  return true;
}

struct TapTable { int n; signed char dh[9], dw[9], wt[9]; };
// K splits of a persistent-kernel launch with `tiles` output tiles of `iters` pipeline stages each: enough work items to fill the SMs,
// at least 4 stages per split, none when the tiles already cover half the machine
static int pick_ksplit(int tiles, int iters, int& it_per_split) {
  it_per_split = iters;
  if (tiles * 2 > g_num_sms || iters < 8) return 1;
  int ks = g_num_sms / tiles;
  if (ks > iters / 4) ks = iters / 4;
  if (ks > 16) ks = 16;
  if (ks < 2) return 1;
  it_per_split = (iters + ks - 1) / ks;
  return (iters + it_per_split - 1) / it_per_split;      // no empty split
}

// Shared launcher.  act: [Nimg][H][W][Kg] fp32 view (ld_act) = A operand on whose pixel grid the M tiles live, amax_a its amax slot;
// w_hi / w_lo: fp16 [T][Nout][ldb] with the scale of slot amax_b; out: [Nimg][Ho][Wo][Nout] view, output pixel = (p*os+oa, q*os+ob).
// ws: optional split-K workspace (dp_conv_splitk_workspace_floats floats); *ws_need != nullptr: only report the floats a split launch needs
int launch_tc(const float* act, long long ld_act, const uint32_t* amax_a, int Nimg, int H, int W, int Kg, const void* w_hi, const void* w_lo,
              const uint32_t* amax_b, int Nout, int T, const TapTable& taps, int os, int oa, int ob, int Ho, int Wo, float* out,
              long long ld_out, const float* bias, const float* rowadd, long long ld_rowadd, const float* residual, long long ld_res,
              int accumulate, cudaStream_t st, float alpha = 1.0f, int b_from_img = 0, int in_stride = 1, int ldb = -1, float* ws = nullptr,
              long long* ws_need = nullptr, uint32_t* amax_out = nullptr) {
  if (ldb < 0) ldb = wrow(Kg);   // packed conv weights; batched GEMM callers pass their own row pitch
  if (!tc_init()) return DP_ERR_UNSUPPORTED;
  if (!ws_need && (!w_hi || !w_lo || !amax_a || !amax_b)) return DP_ERR_UNSUPPORTED;
  if (!ws_need && (ld_act % 4 || ((uintptr_t)act & 15) || ((uintptr_t)w_hi & 15) || ((uintptr_t)w_lo & 15))) return DP_ERR_UNSUPPORTED;
  int bw, bh, bn;
  if (!pick_box(Nimg, H, W, bw, bh, bn)) return DP_ERR_UNSUPPORTED;
  constexpr int BN = 128;
  if (ws_need) {     // geometry-only query
    *ws_need = 0;
    if (b_from_img) return DP_OK;
    const int tiles_m = (W / bw) * (H / bh) * ((Nimg + bn - 1) / bn), n_tiles = (Nout + 127) / 128;
    int ips;
    const int ks = pick_ksplit(tiles_m * n_tiles, taps.n * ((Kg + BK - 1) / BK), ips);
    if (ks > 1) *ws_need = (long long)ks * tiles_m * BM * n_tiles * 128;
    return DP_OK;
  }
  if (b_from_img && bn != 1) return DP_ERR_UNSUPPORTED;
  CUtensorMap mA, mBh, mBl;
  {
    // strided fprop: the M tiles live on the OUTPUT grid [H][W]; the activation is [H*in_stride][W*in_stride] and the box picks every
    // in_stride-th pixel (TMA element strides), so a tile is still one 128-pixel box
    const cuuint64_t Hin = (cuuint64_t)H * in_stride, Win = (cuuint64_t)W * in_stride;
    cuuint64_t dims[4] = {(cuuint64_t)Kg, Win, Hin, (cuuint64_t)Nimg};
    cuuint64_t str[3] = {(cuuint64_t)ld_act * 4, Win * ld_act * 4, Hin * Win * ld_act * 4};
    cuuint32_t box[4] = {32u, (cuuint32_t)(bw * in_stride), (cuuint32_t)(bh * in_stride), (cuuint32_t)bn};   // two boxes of 32 fp32 channels per stage
    if (box[1] > 256 || box[2] > 256) return DP_ERR_UNSUPPORTED;
    if (!make_map(&mA, act, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, in_stride)) return DP_ERR_UNSUPPORTED;
  }
  {
    const cuuint64_t Kp = (cuuint64_t)ldb;
    if (Kp % 8) return DP_ERR_UNSUPPORTED;
    cuuint64_t dims[3] = {Kp, (cuuint64_t)Nout, (cuuint64_t)T};
    cuuint64_t str[2] = {Kp * 2, (cuuint64_t)Nout * Kp * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BN, 1};
    if (!make_map(&mBh, w_hi, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16) ||
        !make_map(&mBl, w_lo, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16)) return DP_ERR_UNSUPPORTED;
  }
  TcParams p{};
  p.Nimg = Nimg; p.H = H; p.W = W; p.Nout = Nout;
  p.ntaps = taps.n;
  for (int i = 0; i < 9; ++i) { p.dh[i] = taps.dh[i]; p.dw[i] = taps.dw[i]; p.wt[i] = taps.wt[i]; }
  p.os = os; p.oa = oa; p.ob = ob; p.Ho = Ho; p.Wo = Wo;
  p.alpha = alpha; p.b_from_img = b_from_img; p.in_stride = in_stride; p.amax_a = amax_a; p.amax_b = amax_b; p.amax_out = amax_out;
  p.kchunks = (Kg + BK - 1) / BK;
  p.bw = bw; p.bh = bh; p.bn = bn; p.tiles_w = W / bw; p.tiles_h = H / bh;
  p.y = out; p.ldy = ld_out; p.bias = bias; p.rowadd = rowadd; p.ld_rowadd = ld_rowadd; p.residual = residual; p.ld_res = ld_res;
  p.accumulate = accumulate;
  auto al16 = [](const void* q, long long ld) { return q == nullptr || ((((uintptr_t)q) & 15) == 0 && (ld % 4) == 0); };
  p.vec4 = (al16(out, ld_out) && al16(bias, 0) && al16(rowadd, ld_rowadd) && al16(residual, ld_res)) ? 1 : 0;
  const int tiles_n = (Nimg + bn - 1) / bn;
  dim3 grid((unsigned)(p.tiles_w * p.tiles_h * tiles_n), (unsigned)((Nout + BN - 1) / BN));
  p.ksplit = 1; p.it_per_split = p.ntaps * p.kchunks;
  {
    const int tiles_m = (int)grid.x, total = (int)(grid.x * grid.y);
    if (ws && !b_from_img) {
      p.ksplit = pick_ksplit(total, p.ntaps * p.kchunks, p.it_per_split);
      p.ws = ws; p.ws_ld = (int)grid.y * 128; p.ws_split_stride = (long long)tiles_m * BM * p.ws_ld;
    }
    const int work = total * p.ksplit;
    const int ctas = work < g_num_sms ? work : g_num_sms;
    conv_tc_ps_kernel<false><<<ctas, THREADS, PS_SMEM, st>>>(mA, mBh, mBl, p, tiles_m, total);
    if (p.ksplit > 1) {
      int rc = dp_check_launch();
      if (rc) return rc;
      const long long items = (long long)tiles_m * BM * ((Nout + 3) / 4);
      long long blocks = (items + 255) / 256;
      if (blocks > g_num_sms * 8) blocks = g_num_sms * 8;
      splitk_epilogue_kernel<<<(int)blocks, 256, 0, st>>>(p, tiles_m);
    }
  }
  return dp_check_launch();
}

__global__ void pack_tc_kernel(const float* __restrict__ w, int K, int C, int RS, int Cp, int Kp, __half* __restrict__ kc_hi,
                               __half* __restrict__ kc_lo, __half* __restrict__ ck_hi, __half* __restrict__ ck_lo,
                               const uint32_t* __restrict__ amax) {
  // rows are zero-padded to Cp = dp_tc_weight_row(C), Kp = dp_tc_weight_row(K): kc [RS][K][Cp] (fprop B), ck [RS][C][Kp] (dgrad B)
  const float sw = scale_up(amax_exponent(amax));
  const long long na = (long long)RS * K * Cp, nb = (long long)RS * C * Kp;
  const long long total = na > nb ? na : nb;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (i < na && kc_hi) {
      int c = (int)(i % Cp); long long t = i / Cp; int k = (int)(t % K), tap = (int)(t / K);
      split1(c < C ? w[((long long)k * C + c) * RS + tap] * sw : 0.f, kc_hi[i], kc_lo[i]);
    }
    if (i < nb && ck_hi) {
      int k = (int)(i % Kp); long long t = i / Kp; int c = (int)(t % C), tap = (int)(t / C);
      split1(k < K ? w[((long long)k * C + c) * RS + tap] * sw : 0.f, ck_hi[i], ck_lo[i]);
    }
  }
}
// fp16 hi / lo' split of a batched [rows][cols] fp32 matrix, dense output rows of `pitch` = round8(cols) elements: 8 columns per thread
// (two float4 loads, one 16-byte store per output)
__global__ void split_h3_rows_kernel(const float* __restrict__ x, long long ld, long long bs, int rows, int cols, int pitch, int vec,
                                     __half* __restrict__ hi, __half* __restrict__ lo, const uint32_t* __restrict__ amax) {
  const float sx = scale_up(amax_exponent(amax));
  const int groups = pitch >> 3;
  const long long total = (long long)rows * groups;
  const float* xb = x + (long long)blockIdx.y * bs;
  __half* hb = hi + (long long)blockIdx.y * rows * pitch;
  __half* lb = lo + (long long)blockIdx.y * rows * pitch;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long r = i / groups;
    const int c0 = (int)(i - r * groups) << 3;
    const float* src = xb + r * ld + c0;
    float v[8];
    if (vec && c0 + 8 <= cols) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src + 4));
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c0 + j < cols) ? __ldg(src + j) : 0.f;
    }
    uint4 h, l;
    split2(v[0] * sx, v[1] * sx, h.x, l.x); split2(v[2] * sx, v[3] * sx, h.y, l.y);
    split2(v[4] * sx, v[5] * sx, h.z, l.z); split2(v[6] * sx, v[7] * sx, h.w, l.w);
    *reinterpret_cast<uint4*>(hb + r * pitch + c0) = h;
    *reinterpret_cast<uint4*>(lb + r * pitch + c0) = l;
  }
}
// transposed form: out[b][c][r] (rows of round8(rows) elements).  A 64 (r) x 64 (c) tile through shared memory: float4 reads along c
// (256 bytes per 16 threads), then every thread owns one output row segment of 16 consecutive r: two 16-byte stores per array
__global__ void __launch_bounds__(256) split_h3_t_kernel(const float* __restrict__ x, long long ld, long long bs, int rows, int cols, int vec,
                                                         __half* __restrict__ hi, __half* __restrict__ lo, const uint32_t* __restrict__ amax) {
  __shared__ float t[64][65];
  const float sx = scale_up(amax_exponent(amax));
  const int b = blockIdx.z, r0 = blockIdx.y * 64, c0 = blockIdx.x * 64, tid = threadIdx.x;
  const float* xb = x + (long long)b * bs;
  {
    const int cc = (tid & 15) * 4, c = c0 + cc;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = (tid >> 4) + 16 * i, r = r0 + rr;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < rows) {
        const float* src = xb + (long long)r * ld + c;
        if (vec && c + 4 <= cols) v = __ldg(reinterpret_cast<const float4*>(src));
        else {
          if (c < cols) v.x = __ldg(src);
          if (c + 1 < cols) v.y = __ldg(src + 1);
          if (c + 2 < cols) v.z = __ldg(src + 2);
          if (c + 3 < cols) v.w = __ldg(src + 3);
        }
      }
      t[rr][cc] = v.x * sx; t[rr][cc + 1] = v.y * sx; t[rr][cc + 2] = v.z * sx; t[rr][cc + 3] = v.w * sx;
    }
  }
  __syncthreads();
  const int rows8 = (rows + 7) & ~7;
  const int c = c0 + (tid >> 2), rs = (tid & 3) * 16;
  if (c < cols) {
    const long long o = ((long long)b * cols + c) * rows8 + r0 + rs;
#pragma unroll
    for (int h8 = 0; h8 < 2; ++h8) {
      if (r0 + rs + 8 * h8 + 8 <= rows8) {         // rows8 and the segments are multiples of 8: a segment is inside or outside as a whole
        uint4 h, l;
        const int rb = rs + 8 * h8, cl = tid >> 2;
        split2(t[rb][cl], t[rb + 1][cl], h.x, l.x); split2(t[rb + 2][cl], t[rb + 3][cl], h.y, l.y);
        split2(t[rb + 4][cl], t[rb + 5][cl], h.z, l.z); split2(t[rb + 6][cl], t[rb + 7][cl], h.w, l.w);
        *reinterpret_cast<uint4*>(hi + o + 8 * h8) = h;
        *reinterpret_cast<uint4*>(lo + o + 8 * h8) = l;
      }
    }
  }
}
// out[b][c][r] = in[b][r][c]: 64 x 64 tiles, float4 on both sides when the extents allow it
__global__ void __launch_bounds__(256) transpose_batched_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols, int vec) {
  __shared__ float t[64][65];
  const int b = blockIdx.z, r0 = blockIdx.y * 64, c0 = blockIdx.x * 64, tid = threadIdx.x;
  const float* ib = in + (long long)b * rows * cols;
  float* ob = out + (long long)b * rows * cols;
  const int q4 = (tid & 15) * 4, l16 = tid >> 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rr = l16 + 16 * i, r = r0 + rr, c = c0 + q4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < rows) {
      const float* src = ib + (long long)r * cols + c;
      if (vec && c + 4 <= cols) v = __ldg(reinterpret_cast<const float4*>(src));
      else {
        if (c < cols) v.x = __ldg(src);
        if (c + 1 < cols) v.y = __ldg(src + 1);
        if (c + 2 < cols) v.z = __ldg(src + 2);
        if (c + 3 < cols) v.w = __ldg(src + 3);
      }
    }
    t[rr][q4] = v.x; t[rr][q4 + 1] = v.y; t[rr][q4 + 2] = v.z; t[rr][q4 + 3] = v.w;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int cc = l16 + 16 * i, c = c0 + cc, r = r0 + q4;
    if (c < cols) {
      float* dst = ob + (long long)c * rows + r;
      if (vec && r + 4 <= rows) *reinterpret_cast<float4*>(dst) = make_float4(t[q4][cc], t[q4 + 1][cc], t[q4 + 2][cc], t[q4 + 3][cc]);
      else {
        if (r < rows) dst[0] = t[q4][cc];
        if (r + 1 < rows) dst[1] = t[q4 + 1][cc];
        if (r + 2 < rows) dst[2] = t[q4 + 2][cc];
        if (r + 3 < rows) dst[3] = t[q4 + 3][cc];
      }
    }
  }
}
}  // namespace

extern "C" int dp_split_h3(const float* x, int64_t ld, int64_t bs, int32_t batch, int32_t rows, int32_t cols, int32_t transpose,
                           const uint32_t* amax, void* hi, void* lo, dp_stream_t stream) {
  DP_REQUIRE(x && hi && lo && amax, DP_ERR_NULL);
  DP_REQUIRE(batch > 0 && rows > 0 && cols > 0 && ld >= cols && batch <= 65535, DP_ERR_SHAPE);
  if (!transpose) {
    const int pitch = (cols + 7) & ~7;
    const int vec = ((((uintptr_t)x) & 15) == 0 && ld % 4 == 0 && bs % 4 == 0) ? 1 : 0;
    long long blocks = ((long long)rows * (pitch >> 3) + 255) / 256;
    if (blocks > g_num_sms * 8) blocks = g_num_sms * 8;
    split_h3_rows_kernel<<<dim3((unsigned)blocks, (unsigned)batch), 256, 0, (cudaStream_t)stream>>>(x, ld, bs, rows, cols, pitch, vec, (__half*)hi,
                                                                                                (__half*)lo, amax);
  } else {
    // the padded tail of a row (rows8) must be covered by the grid: round the covered extent up
    const int vec = ((((uintptr_t)x) & 15) == 0 && ld % 4 == 0 && bs % 4 == 0) ? 1 : 0;
    DP_REQUIRE((((uintptr_t)hi) & 15) == 0 && (((uintptr_t)lo) & 15) == 0, DP_ERR_ALIGN);
    dim3 grid((cols + 63) / 64, (((rows + 7) & ~7) + 63) / 64, batch);
    split_h3_t_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ld, bs, rows, cols, vec, (__half*)hi, (__half*)lo, amax);
  }
  return dp_check_launch();
}
extern "C" int dp_transpose_batched(const float* in, float* out, int32_t batch, int32_t rows, int32_t cols, dp_stream_t stream) {
  DP_REQUIRE(in && out, DP_ERR_NULL);
  DP_REQUIRE(batch > 0 && rows > 0 && cols > 0 && batch <= 65535, DP_ERR_SHAPE);
  const int vec = ((((uintptr_t)in) & 15) == 0 && (((uintptr_t)out) & 15) == 0 && rows % 4 == 0 && cols % 4 == 0) ? 1 : 0;
  dim3 grid((cols + 63) / 64, (rows + 63) / 64, batch);
  transpose_batched_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, rows, cols, vec);
  return dp_check_launch();
}
extern "C" int dp_gemm_nt_tc(const dp_gemm_nt_args* a, dp_stream_t stream) {
  DP_REQUIRE(a && a->A && a->b_hi && a->b_lo && a->C, DP_ERR_NULL);
  DP_REQUIRE(a->batch > 0 && a->H > 0 && a->W > 0 && a->Kg > 0 && a->N > 0 && a->ld_a >= a->Kg && a->ldc >= a->N, DP_ERR_SHAPE);
  if (a->batch > 127) { /* the B "tap" index travels in a signed char table only for real taps; images use n0 directly */ }
  TapTable t{};
  t.n = 1;
  return launch_tc(a->A, a->ld_a, a->amax_a, a->batch, a->H, a->W, a->Kg, a->b_hi, a->b_lo, a->amax_b, a->N, a->batch, t, 1, 0, 0, a->H,
                   a->W, a->C, a->ldc, nullptr, nullptr, 0, nullptr, 0, 0, (cudaStream_t)stream, a->alpha, 1, 1, (a->Kg + 7) & ~7, nullptr,
                   nullptr, a->amax_out);
}

int dp_tc_runtime_ok() { return tc_init(); }

static TapTable dense_taps(int R, int S, int pad, bool flip) {
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

int dp_conv2d_fprop_tc(const dp_conv_args* a, dp_stream_t stream) {
  if (!a || !a->x || !a->y) return DP_ERR_UNSUPPORTED;   // let the SIMT entry produce the precise error
  if (a->flags & DP_CONV_RELU) return DP_ERR_UNSUPPORTED;  // the ReLU epilogue lives on the SIMT kernel
  if (a->R != a->S || (a->R != 1 && a->R != 3) || a->pad_l != a->pad_t) return DP_ERR_UNSUPPORTED;
  // stride 1: 'same' padding.  stride 2: 3x3 with pad 1, or pad 0 + the (0,1,0,1) zero border of Downsample2D (resnet.py:213-218) which
  // TMA out-of-bounds zero fill provides for free
  if (!((a->stride == 1 && a->pad_t == (a->R - 1) / 2) || (a->stride == 2 && a->R == 3 && (a->pad_t == 0 || a->pad_t == 1)))) return DP_ERR_UNSUPPORTED;
  if (a->P * a->stride != a->H || a->Q * a->stride != a->W) return DP_ERR_UNSUPPORTED;   // stride 2: even extents, out = in / 2 (Downsample2D, pad 1)
  if (a->N <= 0 || a->H <= 0 || a->W <= 0 || a->C <= 0 || a->K <= 0 || a->ldx < a->C || a->ldy < a->K) return DP_ERR_UNSUPPORTED;
  return launch_tc((const float*)a->x, a->ldx, a->amax_x, a->N, a->P, a->Q, a->C, a->w_tc_hi, a->w_tc_lo, a->amax_w, a->K, a->R * a->S,
                   dense_taps(a->R, a->S, a->pad_t, false), 1, 0, 0, a->P, a->Q, (float*)a->y, a->ldy, a->bias, a->rowadd,
                   a->ld_rowadd, a->residual, a->ld_res, (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0, (cudaStream_t)stream, 1.0f, 0, a->stride, -1,
                   a->workspace, nullptr, a->amax_out);
}

// General-geometry fprop (DP_CONV_ANY_GEOMETRY): any R x S, stride 1 or 2, explicit top / left padding, any N x H x W, on
// conv_tc_ps_kernel<true>.  Channel counts below ANY_MIN_C stay on the SIMT kernel: a stage holds 64 input channels, and with fewer than 32
// of them most of every 3 x fp16 product multiplies zero fill (Inception's C = 3 stem).  ws_need: geometry-only workspace query.
constexpr int ANY_MIN_C = 32;
int fprop_tc_any(const dp_conv_args* a, float* ws, long long* ws_need, cudaStream_t st) {
  if (a->N <= 0 || a->H <= 0 || a->W <= 0 || a->C <= 0 || a->K <= 0 || a->P <= 0 || a->Q <= 0 || a->R <= 0 || a->S <= 0) return DP_ERR_UNSUPPORTED;
  if (a->C < ANY_MIN_C || (a->stride != 1 && a->stride != 2) || a->pad_t < 0 || a->pad_l < 0 || a->rowadd) return DP_ERR_UNSUPPORTED;
  if ((long long)a->N * a->P * a->Q >= (1ll << 31) || (long long)a->R * a->S > 65535) return DP_ERR_UNSUPPORTED;
  if (!tc_init()) return DP_ERR_UNSUPPORTED;
  const int M = a->N * a->P * a->Q, tiles_m = (M + BM - 1) / BM, n_tiles = (a->K + PS_BN - 1) / PS_BN;
  const int kchunks = (a->C + BK - 1) / BK, iters = a->R * a->S * kchunks;
  if (ws_need) {
    int ips;
    const int ks = pick_ksplit(tiles_m * n_tiles, iters, ips);
    *ws_need = ks > 1 ? (long long)ks * tiles_m * BM * n_tiles * PS_BN : 0;
    return DP_OK;
  }
  if (!a->x || !a->y || !a->w_tc_hi || !a->w_tc_lo || !a->amax_x || !a->amax_w) return DP_ERR_UNSUPPORTED;
  if (a->ldx % 4 || ((uintptr_t)a->x & 15) || ((uintptr_t)a->w_tc_hi & 15) || ((uintptr_t)a->w_tc_lo & 15)) return DP_ERR_UNSUPPORTED;
  CUtensorMap mBh, mBl;
  {
    const cuuint64_t Kp = (cuuint64_t)wrow(a->C);
    cuuint64_t dims[3] = {Kp, (cuuint64_t)a->K, (cuuint64_t)(a->R * a->S)};
    cuuint64_t str[2] = {Kp * 2, (cuuint64_t)a->K * Kp * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)PS_BN, 1};
    if (!make_map(&mBh, a->w_tc_hi, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16) ||
        !make_map(&mBl, a->w_tc_lo, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16)) return DP_ERR_UNSUPPORTED;
  }
  TcParams p{};
  p.Nimg = 1; p.H = 1; p.W = M; p.Nout = a->K;
  p.ntaps = a->R * a->S; p.kchunks = kchunks;
  p.os = 1; p.oa = 0; p.ob = 0; p.Ho = 1; p.Wo = M;
  p.alpha = 1.0f; p.b_from_img = 0; p.in_stride = 1; p.amax_a = a->amax_x; p.amax_b = a->amax_w; p.amax_out = a->amax_out;
  p.bw = BM; p.bh = 1; p.bn = 1; p.tiles_w = tiles_m; p.tiles_h = 1;
  p.y = (float*)a->y; p.ldy = a->ldy; p.bias = a->bias; p.residual = a->residual; p.ld_res = a->ld_res;
  p.accumulate = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  auto al16 = [](const void* q, long long ld) { return q == nullptr || ((((uintptr_t)q) & 15) == 0 && (ld % 4) == 0); };
  p.vec4 = (al16(a->y, a->ldy) && al16(a->bias, 0) && al16(a->residual, a->ld_res)) ? 1 : 0;
  p.gx = (const float*)a->x; p.gldx = a->ldx; p.gH = a->H; p.gW = a->W; p.gC = a->C; p.gQ = a->Q; p.gPQ = a->P * a->Q; p.gS = a->S;
  p.gstride = a->stride; p.gpad_t = a->pad_t; p.gpad_l = a->pad_l; p.gM = M; p.relu = (a->flags & DP_CONV_RELU) ? 1 : 0;
  const int total = tiles_m * n_tiles;
  p.ksplit = 1; p.it_per_split = iters;
  if (ws) {
    p.ksplit = pick_ksplit(total, iters, p.it_per_split);
    p.ws = ws; p.ws_ld = n_tiles * PS_BN; p.ws_split_stride = (long long)tiles_m * BM * p.ws_ld;
  }
  const int work = total * p.ksplit;
  conv_tc_ps_kernel<true><<<work < g_num_sms ? work : g_num_sms, THREADS, PS_SMEM, st>>>(mBh, mBh, mBl, p, tiles_m, total);
  if (p.ksplit > 1) {
    int rc = dp_check_launch();
    if (rc) return rc;
    long long blocks = ((long long)M * ((a->K + 3) / 4) + 255) / 256;
    if (blocks > g_num_sms * 8) blocks = g_num_sms * 8;
    splitk_flat_epilogue_kernel<<<(int)blocks, 256, 0, st>>>(p);
  }
  return dp_check_launch();
}
int dp_conv2d_fprop_tc_any(const dp_conv_args* a, dp_stream_t stream) {
  if (!a) return DP_ERR_UNSUPPORTED;
  return fprop_tc_any(a, a->workspace, nullptr, (cudaStream_t)stream);
}

// stride-1 dgrad == fprop of dy with the taps flipped and the (K,C) roles swapped: dx[n,h,w,c] = sum dy[n,h+1-r,w+1-s,k] W[k,c,r,s].
// stride-2 dgrad: dx[2i+a, 2j+b] only sees taps with (a+pad-r), (b+pad-s) even -> 4 parity classes, each a dense GEMM over the
// dy grid with 1/2/2/4 taps and a strided output mapping (no MACs wasted on structural zeros).
int dp_conv2d_dgrad_tc(const dp_conv_args* a, dp_stream_t stream) {
  if (!a || !a->x || !a->y) return DP_ERR_UNSUPPORTED;
  if (a->N <= 0 || a->H <= 0 || a->W <= 0 || a->C <= 0 || a->K <= 0 || a->ldx < a->C || a->ldy < a->K) return DP_ERR_UNSUPPORTED;
  if (a->R != a->S || (a->R != 1 && a->R != 3)) return DP_ERR_UNSUPPORTED;
  const int acc = (a->flags & DP_CONV_ACCUMULATE) ? 1 : 0;
  if (a->stride == 1) {
    if (a->pad_t != (a->R - 1) / 2 || a->pad_l != a->pad_t || a->P != a->H || a->Q != a->W) return DP_ERR_UNSUPPORTED;
    return launch_tc((const float*)a->y, a->ldy, a->amax_y, a->N, a->H, a->W, a->K, a->w_tc_hi, a->w_tc_lo, a->amax_w, a->C, a->R * a->S,
                     dense_taps(a->R, a->S, a->pad_t, true), 1, 0, 0, a->H, a->W, (float*)a->x, a->ldx, nullptr, nullptr, 0, nullptr, 0,
                     acc, (cudaStream_t)stream, 1.0f, 0, 1, -1, a->workspace, nullptr, a->amax_out);
  }
  if (a->stride != 2 || a->R != 3 || a->H != 2 * a->P || a->W != 2 * a->Q) return DP_ERR_UNSUPPORTED;
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
      int rc = launch_tc((const float*)a->y, a->ldy, a->amax_y, a->N, a->P, a->Q, a->K, a->w_tc_hi, a->w_tc_lo, a->amax_w, a->C, 9, cls[ca * 2 + cb], 2, ca, cb,
                         a->H, a->W, (float*)a->x, a->ldx, nullptr, nullptr, 0, nullptr, 0, acc, (cudaStream_t)stream, 1.0f, 0, 1, -1,
                         a->workspace, nullptr, a->amax_out);
      if (rc != DP_OK) return (ca == 0 && cb == 0) ? rc : (rc == DP_ERR_UNSUPPORTED ? DP_ERR_SHAPE : rc);
    }
  return DP_OK;
}

// Floats of split-K workspace dp_conv2d_fprop (op 0) / dp_conv2d_dgrad (op 1) can use for this geometry (0: the launch fills the SMs
// without splitting).  With a->workspace == NULL the launch simply does not split.
extern "C" long long dp_conv_splitk_workspace_floats(const dp_conv_args* a, int op) {
  if (a && op == 0 && (a->flags & DP_CONV_ANY_GEOMETRY)) {   // the box kernel's need, or else the general-geometry kernel's
    dp_conv_args b = *a;
    b.flags &= ~DP_CONV_ANY_GEOMETRY;
    long long need = (a->flags & DP_CONV_RELU) ? 0 : dp_conv_splitk_workspace_floats(&b, 0), any = 0;
    if (fprop_tc_any(a, nullptr, &any, nullptr) == DP_OK && any > need) need = any;
    return need;
  }
  if (!a || a->N <= 0 || a->H <= 0 || a->W <= 0 || a->C <= 0 || a->K <= 0 || a->R != a->S || (a->R != 1 && a->R != 3)) return 0;
  long long need = 0;
  TapTable t{};
  if (op == 0) {
    t.n = a->R * a->S;
    launch_tc(nullptr, 0, nullptr, a->N, a->P, a->Q, a->C, nullptr, nullptr, nullptr, a->K, t.n, t, 1, 0, 0, a->P, a->Q, nullptr, 0, nullptr,
              nullptr, 0, nullptr, 0, 0, nullptr, 1.0f, 0, a->stride, -1, nullptr, &need);
  } else if (a->stride == 1) {
    t.n = a->R * a->S;
    launch_tc(nullptr, 0, nullptr, a->N, a->H, a->W, a->K, nullptr, nullptr, nullptr, a->C, t.n, t, 1, 0, 0, a->H, a->W, nullptr, 0, nullptr,
              nullptr, 0, nullptr, 0, 0, nullptr, 1.0f, 0, 1, -1, nullptr, &need);
  } else {
    for (int taps = 1; taps <= 4; taps *= 2) {     // the parity classes of a stride-2 3x3 dgrad have 1 / 2 / 2 / 4 taps and run back to back
      long long n = 0;
      t.n = taps;
      launch_tc(nullptr, 0, nullptr, a->N, a->P, a->Q, a->K, nullptr, nullptr, nullptr, a->C, 9, t, 2, 0, 0, a->H, a->W, nullptr, 0, nullptr,
                nullptr, 0, nullptr, 0, 0, nullptr, 1.0f, 0, 1, -1, nullptr, &n);
      if (n > need) need = n;
    }
  }
  return need;
}

// 64-pixel K-chunk box of an [N][H][W] grid
static bool pick_box64(int H, int W, int& bw, int& bh, int& bn) {
  if (W >= WG_KPIX) { if (W % WG_KPIX) return false; bw = WG_KPIX; bh = 1; bn = 1; return true; }
  if (WG_KPIX % W) return false;
  bw = W;
  int rem = WG_KPIX / W;
  if (H >= rem) { if (H % rem) return false; bh = rem; bn = 1; return true; }
  if (rem % H) return false;
  bh = H; bn = rem / H;
  return true;
}

int dp_conv2d_wgrad_tc(const dp_conv_args* a, dp_stream_t stream) {
  if (!a || !a->x || !a->y || !a->workspace) return DP_ERR_UNSUPPORTED;
  if (!tc_init()) return DP_ERR_UNSUPPORTED;
  if (a->R != a->S || (a->R != 1 && a->R != 3) || a->pad_l != a->pad_t) return DP_ERR_UNSUPPORTED;
  // stride 1: 'same' padding.  stride 2: 3x3 with pad 1, or pad 0 + the (0,1,0,1) zero border of Downsample2D (resnet.py:213-218) which
  // TMA out-of-bounds zero fill provides for free
  if (!((a->stride == 1 && a->pad_t == (a->R - 1) / 2) || (a->stride == 2 && a->R == 3 && (a->pad_t == 0 || a->pad_t == 1)))) return DP_ERR_UNSUPPORTED;
  if (a->P * a->stride != a->H || a->Q * a->stride != a->W || a->splits < 1) return DP_ERR_UNSUPPORTED;
  if (a->ldx % 4 || a->ldy % 4 || ((uintptr_t)a->x & 15) || ((uintptr_t)a->y & 15)) return DP_ERR_UNSUPPORTED;
  int bw, bh, bn;
  if (!a->amax_x || !a->amax_y) return DP_ERR_UNSUPPORTED;
  if (!pick_box64(a->P, a->Q, bw, bh, bn)) return DP_ERR_UNSUPPORTED;   // 64-pixel chunks of the dy (output) grid; images past the batch
  const int img_boxes = (a->N + bn - 1) / bn;                           // in the last box are TMA zero fill: they add nothing
  CUtensorMap mDy, mX;
  {
    cuuint64_t dims[4] = {(cuuint64_t)a->K, (cuuint64_t)a->Q, (cuuint64_t)a->P, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->ldy * 4, (cuuint64_t)a->Q * a->ldy * 4, (cuuint64_t)a->P * a->Q * a->ldy * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
    if (!make_map(&mDy, a->y, 4, dims, str, box)) return DP_ERR_UNSUPPORTED;
  }
  {   // x is sampled at stride * (output pixel) + tap offset: TMA element strides on W, H
    cuuint64_t dims[4] = {(cuuint64_t)a->C, (cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N};
    cuuint64_t str[3] = {(cuuint64_t)a->ldx * 4, (cuuint64_t)a->W * a->ldx * 4, (cuuint64_t)a->H * a->W * a->ldx * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)(bw * a->stride), (cuuint32_t)(bh * a->stride), (cuuint32_t)bn};
    if (box[1] > 256 || box[2] > 256) return DP_ERR_UNSUPPORTED;
    if (!make_map(&mX, a->x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, a->stride)) return DP_ERR_UNSUPPORTED;
  }
  WgParams p{};
  p.Nimg = a->N; p.H = a->P; p.W = a->Q; p.C = a->C; p.K = a->K; p.R = a->R; p.S = a->S; p.pad = a->pad_t; p.in_stride = a->stride;
  p.bw = bw; p.bh = bh; p.bn = bn; p.tiles_w = a->Q / bw; p.tiles_h = a->P / bh;
  p.total_chunks = p.tiles_w * p.tiles_h * img_boxes;
  p.amax_x = a->amax_x; p.amax_y = a->amax_y; p.bias_ws = a->bias_ws;
  p.chunks_per_split = (p.total_chunks + a->splits - 1) / a->splits;
  p.c_tiles = (a->C + 127) / 128;
  p.ws = a->workspace;
  const int k_tiles = (a->K + 127) / 128;
  dim3 grid((unsigned)(k_tiles * p.c_tiles * a->R * a->S), (unsigned)a->splits);
  wgrad_tc_kernel<<<grid, THREADS, WG_SMEM, (cudaStream_t)stream>>>(mDy, mX, p);
  return dp_check_launch();
}

extern "C" int dp_pack_conv_weight_tc(const float* w, int32_t K, int32_t C, int32_t R, int32_t S, void* kc_hi, void* kc_lo,
                                      void* ck_hi, void* ck_lo, uint32_t* amax_w, dp_stream_t stream) {
  DP_REQUIRE(w && amax_w, DP_ERR_NULL);
  DP_REQUIRE((kc_hi == nullptr) == (kc_lo == nullptr) && (ck_hi == nullptr) == (ck_lo == nullptr), DP_ERR_NULL);
  DP_REQUIRE(K > 0 && C > 0 && R > 0 && S > 0, DP_ERR_SHAPE);
  // the weight's own amax slot first (one scale per tensor), then both fp16 hi / lo' orientations with that scale
  if (cudaMemsetAsync(amax_w, 0, sizeof(uint32_t), (cudaStream_t)stream) != cudaSuccess) return dp_check_launch();
  int rc = dp_amax(w, (int64_t)C * R * S, K, C * R * S, amax_w, stream);
  if (rc) return rc;
  const int Cp = wrow(C), Kp = wrow(K);
  long long total = (long long)R * S * ((long long)K * Cp > (long long)C * Kp ? (long long)K * Cp : (long long)C * Kp);
  int blocks = (int)((total + 255) / 256);
  if (blocks > g_num_sms * 16) blocks = g_num_sms * 16;
  pack_tc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, K, C, R * S, Cp, Kp, (__half*)kc_hi, (__half*)kc_lo, (__half*)ck_hi, (__half*)ck_lo,
                                                           amax_w);
  return dp_check_launch();
}

extern "C" int dp_tc_weight_row(int channels) { return channels > 0 ? wrow(channels) : 0; }
