// KV = K^T V of the coarse linear attention on the tensor cores (reference linear_attention.py:43:
// `KV = einsum("nshd,nshv->nhdv", K, values)`), fed from the fp16 hi/lo planes the k|v projection epilogue
// (EpiKvProj) writes.
//
// As a GEMM this is D[d, v] = sum_rows K[row, d] * V[row, v]: the contraction runs over the ROWS of two row-major
// matrices, i.e. both operands are "MN-major" for wgmma (imm-trans-a = imm-trans-b = 1).  A TMA box of 64 columns x
// 64 rows of the planes lands in shared memory as [64 k-rows][128 B] with the 128-byte swizzle, which is the canonical
// MN-major SWIZZLE_128B layout: LBO = 8192 B between blocks of 64 d (or v), SBO = 1024 B between groups of 8 k-rows,
// 2048 B per K = 16 step.
//
// One CTA per (k-split, head quartet, image), one consumer warpgroup and one TMA warp.  Only the four diagonal
// 32 x 32 blocks of the quartet's 128 x 128 product are attention state, so the warpgroup computes two m64n64 blocks
// (heads 0-1 x their v, heads 2-3 x their v) and stores them as one partial per (image, split, head).  Split
// precision as everywhere: hi*hi + hi*lo + lo*hi into one fp32 register accumulator.
//
// Ksum = K^T 1 (`K.sum(dim=1)`, linear_attention.py:44) rides along: N = 16 MMAs multiply the K planes with a block of
// ones (1 KB of fp16 1.0 in shared memory -- with every element equal, any descriptor that stays inside the block is a
// valid "ones" operand); masked / out-of-range rows are already zero in the planes.
#pragma once
#include "ptx.cuh"

namespace lb {

struct KvGemmParams {
  float* part;        // [images][splits][H = 8][32*32 + 32]: KV then Ksum, the layout of the final kv state
  int kb_total;       // ceil(rows per image / 64)
  int kb_per_split;
  int splits;
};

constexpr int kKvGemmThreads = 160;                 // warps 0-3 wgmma + epilogue, warp 4 TMA
constexpr int kKvGemmStages = 3;
constexpr int kKvBlock = 64 * 128;                  // one TMA box: 64 k-rows x 128 bytes
constexpr int kKvTile = 2 * kKvBlock;               // 128 d (or v) x 64 k-rows per plane: 16 KB
constexpr int kKvStageBytes = 4 * kKvTile;          // A hi, A lo, B hi, B lo
constexpr int kKvOnesBytes = 1024;
constexpr int kKvGemmSmem = kKvGemmStages * kKvStageBytes + kKvOnesBytes + 256;

// D[64 x 64] += A^T B with both operands MN-major (transposed) in shared memory
__device__ __forceinline__ void wgmma_f16_n64_tt(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
      "%14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b));
}
// D[64 x 16] += A^T B with A MN-major, B K-major (the ones block)
__device__ __forceinline__ void wgmma_f16_n16_tn(float (&d)[8], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(desc_a), "l"(desc_b));
}
// MN-major operand tile, 128-byte swizzle: LBO = 8192 B (next 64 MN elements), SBO = 1024 B (next 8 k-rows)
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(kKvBlock >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// unswizzled K-major descriptor into the ones block: 8-row groups 128 B apart, the two 16-byte K halves 256 B apart
__device__ __forceinline__ uint64_t wgmma_desc_ones(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(256 >> 4) << 16;
  d |= static_cast<uint64_t>(128 >> 4) << 32;
  return d;
}

// tm_hi / tm_lo: the K|V planes [images][rows][512] with box (64 columns, 64 rows, 1); columns as the projection emits
// them: [K of heads 0-3 | V of heads 0-3 | K of heads 4-7 | V of heads 4-7]
__global__ void __launch_bounds__(kKvGemmThreads, 1)
kv_gemm_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, const KvGemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) asm volatile("trap;");
  uint8_t* s_ones = smem + kKvGemmStages * kKvStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_ones + kKvOnesBytes);
  uint64_t* empty_bar = full_bar + kKvGemmStages;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform roles
  const int lane = threadIdx.x & 31;
  const int split = blockIdx.x, quartet = blockIdx.y, image = blockIdx.z;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(kb0 + p.kb_per_split, p.kb_total);
  const int nkb = max(kb1 - kb0, 0);

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_hi);
    tma_prefetch_desc(&tm_lo);
    for (int s = 0; s < kKvGemmStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 128);   // every consumer thread arrives
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < kKvOnesBytes / 4; i += kKvGemmThreads) reinterpret_cast<uint32_t*>(s_ones)[i] = 0x3C003C00u;   // fp16 1.0 x 2
  fence_proxy_async();
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < nkb; ++i) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* st = smem + stage * kKvStageBytes;
        uint64_t* fb = &full_bar[stage];
        mbar_arrive_expect_tx(fb, kKvStageBytes);
        const int row0 = (kb0 + i) * 64;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int ck = quartet * 256 + b * 64, cv = quartet * 256 + 128 + b * 64;
          tma_load_3d(st + b * kKvBlock, &tm_hi, fb, ck, row0, image);
          tma_load_3d(st + kKvTile + b * kKvBlock, &tm_lo, fb, ck, row0, image);
          tma_load_3d(st + 2 * kKvTile + b * kKvBlock, &tm_hi, fb, cv, row0, image);
          tma_load_3d(st + 3 * kKvTile + b * kKvBlock, &tm_lo, fb, cv, row0, image);
        }
        if (++stage == kKvGemmStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ---- consumer warpgroup: block mh = heads (2 mh, 2 mh + 1): d in [64 mh, 64 mh + 64) x v in the same range
    float acc[2][32], ks[2][8];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[0][i] = acc[1][i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) ks[0][i] = ks[1][i] = 0.f;
    const uint64_t ones = wgmma_desc_ones(smem_u32(s_ones));
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st = smem_u32(smem + stage * kKvStageBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t off = static_cast<uint32_t>(k) * 2048u;   // 16 k-rows of 128 bytes
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
          const uint32_t blk = off + static_cast<uint32_t>(mh * kKvBlock);
          const uint64_t a_hi = wgmma_desc_mn_sw128(st + blk), a_lo = wgmma_desc_mn_sw128(st + kKvTile + blk);
          const uint64_t b_hi = wgmma_desc_mn_sw128(st + 2 * kKvTile + blk), b_lo = wgmma_desc_mn_sw128(st + 3 * kKvTile + blk);
          wgmma_f16_n64_tt(acc[mh], a_hi, b_hi);
          wgmma_f16_n64_tt(acc[mh], a_hi, b_lo);
          wgmma_f16_n64_tt(acc[mh], a_lo, b_hi);
          wgmma_f16_n16_tn(ks[mh], a_hi, ones);
          wgmma_f16_n16_tn(ks[mh], a_lo, ones);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-block's MMAs are done: its slot may be refilled
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kKvGemmStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    wgmma_fence_regs(ks[0]);
    wgmma_fence_regs(ks[1]);
    // ---- epilogue: thread holds rows r0, r0 + 8 and columns 8 j + 2 (t % 4) (+1) of each 64 x 64 block; only the
    // diagonal 32 x 32 head blocks are stored (zeros when this split has no rows)
    const int t = threadIdx.x;
    const int r0 = 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int r = r0 + 8 * rr;          // 0..63 inside the block
        const int head = 2 * mh + (r >> 5), d = r & 31;
        float* base = p.part + ((static_cast<long>(image) * p.splits + split) * 8 + quartet * 4 + head) * 1056;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * (t & 3);
          if ((c >> 5) == (r >> 5))
            *reinterpret_cast<float2*>(base + d * 32 + (c & 31)) = make_float2(acc[mh][4 * j + 2 * rr], acc[mh][4 * j + 2 * rr + 1]);
        }
        if ((t & 3) == 0) base[1024 + d] = ks[mh][2 * rr];
      }
    }
  }
}

}  // namespace lb
