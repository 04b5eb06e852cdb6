// Backbone stem on the tensor cores: conv 7x7 stride 2, 1 -> 128 channels, + folded BatchNorm + ReLU
// (reference src/loftr/backbone/resnet_fpn.py:58-60,101), written as NHWC fp16 hi/lo planes.
//
// As a GEMM the stem is M = output pixels, N = 128, K = 49 (padded to 64): far too little K for the TMA-fed
// gemm_split_kernel, and a single-channel image cannot be im2col'ed by a tensor map (the tap stride would be 2 or 4
// bytes).  So this kernel builds the A tile in software: per 8 x 16 output-pixel tile the 21 x 37 input patch is
// staged in shared memory, every warp writes its rows of the [128 x 64] fp16 hi/lo operand tiles straight into the
// 128-byte-swizzled K-major layout wgmma expects, and each of the two warpgroups issues the wgmma of one 64-channel
// half (rows 0-63 and 64-127 x 4 k-steps x (hi*hi + hi*lo + lo*hi)).  The accumulator is staged row-major in shared
// memory and all 8 warps run the epilogue (BN + ReLU + split, TMA store of 2 x 16 pixel x 32 channel boxes).  The
// weights (128 x 49 fp32) are scaled by a power of two, split and swizzled into shared memory once per CTA.  One
// persistent CTA per SM, 256 threads.
#pragma once
#include "epilogues.cuh"

namespace lb {

struct StemTcParams {
  const float* img;     // [N, 1, H, W]
  int N, H, W;
  const float* wt;      // conv1.weight transposed [49][128]
  const float* scale;   // folded bn1 [128]
  const float* shift;
  OutMaps om;           // NHWC planes [N, H/2, W/2, 128]: 4-D TMA-store maps (box 32 ch x 16 x 2 px)
  int tiles_w, tiles_h; // 16- / 8-pixel tiles of the output grid
};

constexpr int kStemThreads = 256;
constexpr int kStemPatchH = 2 * kConvTileH + 5;    // 21 input rows feed 8 output rows
constexpr int kStemPatchW = 2 * kConvTileW + 5;    // 37
constexpr int kStemPatchPitch = 40;
constexpr int kStemATile = 128 * 128;              // [128 rows][64 fp16] = 16 KB per plane
constexpr int kStemAccStride = 132;                // floats per staged accumulator row (conflict-free row reads)
constexpr int kStemSmemBytes = 2 * kStemATile      // A hi/lo
                               + 2 * kStemATile    // W hi/lo
                               + 128 * kStemAccStride * 4   // staged accumulator
                               + 8 * 4096          // per-warp TMA-store staging
                               + kStemPatchH * kStemPatchPitch * 4 + 2 * 128 * 4 + 64 * 4;

__device__ __forceinline__ uint32_t stem_sw128(int row, int k) {   // byte offset of fp16 element (row, k) in a SW128 K-major tile
  return static_cast<uint32_t>(row * 128 + ((((k >> 3) ^ (row & 7)) << 4) | ((k & 7) << 1)));
}

__global__ void __launch_bounds__(kStemThreads, 1) conv_stem7x7_tc_kernel(const __grid_constant__ StemTcParams p) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the first convolution may set up meanwhile
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) asm volatile("trap;");
  uint8_t* sA = smem;                                   // [hi|lo][16 KB]
  uint8_t* sW = smem + 2 * kStemATile;                  // [hi|lo][16 KB]
  float* sAcc = reinterpret_cast<float*>(smem + 4 * kStemATile);                 // [128][kStemAccStride]
  uint32_t* sStage = reinterpret_cast<uint32_t*>(sAcc + 128 * kStemAccStride);
  float* sPatch = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sStage) + 8 * 4096);   // [21][40]
  float* sScale = sPatch + kStemPatchH * kStemPatchPitch;
  float* sShift = sScale + 128;
  float* sRed = sShift + 128;                           // [64]

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // warp-uniform: keeps the wgmma window convergent

  // ---- weights: power-of-two scale (keeps the fp16 `lo` residuals out of the subnormal range), split, swizzle
  float amax = 0.f;
  for (int i = tid; i < 49 * 128; i += kStemThreads) amax = fmaxf(amax, fabsf(p.wt[i]));
  for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (lane == 0) sRed[warp] = amax;
  __syncthreads();
  amax = sRed[0];
  for (int k = 1; k < kStemThreads / 32; ++k) amax = fmaxf(amax, sRed[k]);
  int e = amax > 0.f ? static_cast<int>(floorf(log2f(4096.f / amax))) : 0;
  e = max(-24, min(24, e));
  const float wmul = exp2f(static_cast<float>(e)), inv = exp2f(static_cast<float>(-e));
  for (int i = tid; i < 128 * 32; i += kStemThreads) {          // (cout n, k pair)
    const int n = i >> 5, k = (i & 31) << 1;
    const float w0 = k < 49 ? p.wt[k * 128 + n] * wmul : 0.f;
    const float w1 = k + 1 < 49 ? p.wt[(k + 1) * 128 + n] * wmul : 0.f;
    uint32_t h, l;
    split_f16x2(w0, w1, h, l);
    *reinterpret_cast<uint32_t*>(sW + stem_sw128(n, k)) = h;
    *reinterpret_cast<uint32_t*>(sW + kStemATile + stem_sw128(n, k)) = l;
  }
  for (int i = tid; i < 2 * kStemATile / 16; i += kStemThreads) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid < 128) {
    sScale[tid] = p.scale[tid] * inv;
    sShift[tid] = p.shift[tid];
  }
  __syncthreads();

  const long tiles_per_img = static_cast<long>(p.tiles_w) * p.tiles_h;
  const long total = tiles_per_img * p.N;
  const int half = warp >> 2;                     // warpgroup = 64-channel half of the accumulator
  const int wt = tid & 127;                       // thread within the warpgroup
  uint32_t* stage = sStage + warp * 1024;

  for (long t = blockIdx.x; t < total; t += gridDim.x) {
    const int n = static_cast<int>(t / tiles_per_img);
    const int rem = static_cast<int>(t - n * tiles_per_img);
    const int ty = rem / p.tiles_w, tx = rem - ty * p.tiles_w;
    // (a) input patch -> shared memory (zero outside the image = the convolution's padding)
    const int iy0 = 2 * ty * kConvTileH - 3, ix0 = 2 * tx * kConvTileW - 3;
    for (int i = tid; i < kStemPatchH * kStemPatchW; i += kStemThreads) {
      const int py = i / kStemPatchW, px = i - py * kStemPatchW;
      const int iy = iy0 + py, ix = ix0 + px;
      float v = 0.f;
      if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) v = p.img[(static_cast<long>(n) * p.H + iy) * p.W + ix];
      sPatch[py * kStemPatchPitch + px] = v;
    }
    __syncthreads();
    // (b) software im2col: warp w writes rows w, w+8, ...; lane = pair of taps (k, k+1)
    if (lane < 25) {
      const int k0 = 2 * lane, k1 = k0 + 1;
      const int ky0 = k0 / 7, kx0 = k0 - ky0 * 7;
      const int ky1 = k1 / 7, kx1 = k1 - ky1 * 7;
      for (int r = warp; r < 128; r += kStemThreads / 32) {
        const int py = r >> 4, px = r & 15;
        const float v0 = sPatch[(2 * py + ky0) * kStemPatchPitch + 2 * px + kx0];
        const float v1 = k1 < 49 ? sPatch[(2 * py + ky1) * kStemPatchPitch + 2 * px + kx1] : 0.f;
        uint32_t h, l;
        split_f16x2(v0, v1, h, l);
        *reinterpret_cast<uint32_t*>(sA + stem_sw128(r, k0)) = h;
        *reinterpret_cast<uint32_t*>(sA + kStemATile + stem_sw128(r, k0)) = l;
      }
    }
    fence_proxy_async();   // generic-proxy operand writes before the wgmma (async proxy) reads them
    __syncthreads();
    // (c) wgmma: warpgroup `half` computes output channels [64 half, 64 half + 64) for all 128 pixels
    float acc[2][32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[0][i] = acc[1][i] = 0.f;
    {
      const uint32_t a0 = smem_u32(sA), w0 = smem_u32(sW) + static_cast<uint32_t>(half * 64 * 128);
      wgmma_fence();
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
        const uint32_t a_off = static_cast<uint32_t>(mh * 64 * 128);
        const uint64_t da_hi = wgmma_desc_k_sw128(a0 + a_off), da_lo = wgmma_desc_k_sw128(a0 + kStemATile + a_off);
        const uint64_t db_hi = wgmma_desc_k_sw128(w0), db_lo = wgmma_desc_k_sw128(w0 + kStemATile);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t adv = static_cast<uint64_t>(k * 2);
          wgmma_f16<64>(acc[mh], da_hi + adv, db_hi + adv, 1u);
          wgmma_f16<64>(acc[mh], da_hi + adv, db_lo + adv, 1u);
          wgmma_f16<64>(acc[mh], da_lo + adv, db_hi + adv, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
    }
    // (d) stage the accumulator row-major: thread holds rows 16 (wt/32) + (wt%32)/4 (+8, +64), columns 8 j + 2 (wt%4)
    {
      const int r0 = 16 * (wt >> 5) + ((wt & 31) >> 2);
      const int c0 = half * 64 + 2 * (wt & 3);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float* q = sAcc + (mh * 64 + r0) * kStemAccStride + c0 + 8 * j;
          *reinterpret_cast<float2*>(q) = make_float2(acc[mh][4 * j], acc[mh][4 * j + 1]);
          *reinterpret_cast<float2*>(q + 8 * kStemAccStride) = make_float2(acc[mh][4 * j + 2], acc[mh][4 * j + 3]);
        }
      }
    }
    __syncthreads();
    // (e) epilogue: warp w drains pixel rows 32 (w%4) + lane, channel groups of its half
    const float* row = sAcc + ((warp & 3) * 32 + lane) * kStemAccStride;
#pragma unroll 1
    for (int c = half * 2; c < half * 2 + 2; ++c) {
      float x[32];
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 v = *reinterpret_cast<const float4*>(row + c * 32 + j);
        x[j] = fmaxf(fmaf(v.x, sScale[c * 32 + j], sShift[c * 32 + j]), 0.f);
        x[j + 1] = fmaxf(fmaf(v.y, sScale[c * 32 + j + 1], sShift[c * 32 + j + 1]), 0.f);
        x[j + 2] = fmaxf(fmaf(v.z, sScale[c * 32 + j + 2], sShift[c * 32 + j + 2]), 0.f);
        x[j + 3] = fmaxf(fmaf(v.w, sScale[c * 32 + j + 3], sShift[c * 32 + j + 3]), 0.f);
      }
      warp_tma_store_planes32(stage, p.om, OutCoord{c * 32, tx * kConvTileW, ty * kConvTileH + (warp & 3) * 2, n}, x);
    }
    __syncthreads();   // the staged accumulator and the operand tile are rewritten by the next tile
  }
  tma_store_wait_all();
}

}  // namespace lb
