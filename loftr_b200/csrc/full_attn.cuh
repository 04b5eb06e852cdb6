// Full (softmax) attention of the coarse transformer on the tensor cores (reference linear_attention.py:56-81,
// `FullAttention`): message = softmax(Q K^T / sqrt(D)) V per (image, head), fused so that the L x S x H score tensor
// never exists (737 MB of fp32 per image and layer call at 640 x 480).
//
// One CTA per (128-query tile, head, image group): two consumer warpgroups of 64 query rows and one TMA producer warp.
// The producer loads Q (hi / lo planes, 128 rows x 64 B, 64-byte swizzle) once and streams K_h / V_h tiles of 64 keys
// through a ring of kFwStages mbarrier-guarded slots; rows past the group arrive as zeros, and the producer writes
// each tile's key bias (0, or -inf for keys past the group or with kv_mask = 0) before the tile's barrier completes.
// Per tile, warpgroup g:
//   S[64 x 64] = Q K^T   wgmma.m64n64k16, both operands K-major from shared memory, hi*hi + hi*lo + lo*hi over two
//                        k-steps (the split-precision product of the GEMM core)
//   softmax              online row max / row sum in fp32, base 2 (exp2f); P = 2^(S log2(e)/sqrt(D) - m) is split
//                        into hi/lo fp16 in registers (the m64nN accumulator layout of a warp is the A-operand layout
//                        of the register form)
//   O[64 x 32] += P V    wgmma.m64n32k16 with P from registers (RS form) and V MN-major (transpose bit), 3 products
// The epilogue divides by the row sum and writes the message as fp16 planes.  Padded queries (q_mask = 0) and rows
// whose keys are all masked write 0 (the reference would produce NaN there; DESIGN.md §5).
//
// Q is read from the same planes the message is written to: every CTA reads only its own (rows, head) block, before it
// writes that block.  Deterministic: no atomics, fixed reduction order.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>
#include "ptx.cuh"
#include "simt_kernels.cuh"

namespace lb {

constexpr int kFaRows = 128;               // query rows per CTA
constexpr int kFaKeys = 64;                // keys per ring slot
constexpr int kFaD = 32;                   // head dimension (coarse: 256 / 8)

constexpr int kFwStages = 3;
constexpr int kFwThreads = 288;                       // warps 0-7 consumers, warp 8 producer
constexpr int kFwQPlane = kFaRows * 64;               // 128 rows x 64 B
constexpr int kFwKvPlane = kFaKeys * 64;              // 64 keys x 64 B
constexpr int kFwStage = 4 * kFwKvPlane;              // K hi, K lo, V hi, V lo
constexpr int kFwSmem = 2 * kFwQPlane + kFwStages * kFwStage + kFwStages * kFaKeys * 4 + 2 * kFwStages * 8 + 8 + 1024;

// D[64 x 32] += A[64 x 16] (registers, fp16x2) * B, B MN-major in shared memory (imm-trans-b = 1)
__device__ __forceinline__ void wgmma_rs_n32_tb(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
      "%14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b));
}
// MN-major operand, 64-byte swizzle: rows of 32 MN elements (64 B) per k; 8-k-row groups 512 B apart (SBO)
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(kFwKvPlane >> 4) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}

struct FullAttnWgParams {
  int Lx, Ls;
  int v_col0;
  long x_base, s_base;
  const uint8_t* mask;
  __half* o_hi;
  __half* o_lo;
  int ld_o;
  float scale_log2;
};

// tm_q_hi/lo: Q planes as [groups][Lx][C], box (32, 128); tm_kv_hi/lo: K|V planes as [groups][Ls][2C], box (32, 64)
__global__ void __launch_bounds__(kFwThreads, 1)
full_attn_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
                       const __grid_constant__ CUtensorMap tm_kv_hi, const __grid_constant__ CUtensorMap tm_kv_lo,
                       const FullAttnWgParams p) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t fw_smem[];
  uint8_t* smem = fw_smem + ((1024u - (smem_u32(fw_smem) & 1023u)) & 1023u);
  uint8_t* s_q = smem;                                              // [hi | lo][128][64 B]
  uint8_t* s_ring = smem + 2 * kFwQPlane;                           // [stage][K hi, K lo, V hi, V lo][64][64 B]
  float* s_bias = reinterpret_cast<float*>(s_ring + kFwStages * kFwStage);   // [stage][64]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_bias + kFwStages * kFaKeys);
  uint64_t* empty_bar = full_bar + kFwStages;
  uint64_t* q_bar = empty_bar + kFwStages;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, grp = blockIdx.z;
  const int n_tiles = (p.Ls + kFaKeys - 1) / kFaKeys;
  const long srow0 = p.s_base + static_cast<long>(grp) * p.Ls;
  const long xrow0 = p.x_base + static_cast<long>(grp) * p.Lx;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_q_hi);
    tma_prefetch_desc(&tm_q_lo);
    tma_prefetch_desc(&tm_kv_hi);
    tma_prefetch_desc(&tm_kv_lo);
    for (int s = 0; s < kFwStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 256);   // every consumer thread arrives
    }
    mbar_init(q_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ---- producer: Q once, then the K / V ring; the key bias of a tile is written before its barrier arrives
    if (lane == 0) {
      mbar_arrive_expect_tx(q_bar, 2 * kFwQPlane);
      tma_load_3d(s_q, &tm_q_hi, q_bar, head * kFaD, qt * kFaRows, grp);
      tma_load_3d(s_q + kFwQPlane, &tm_q_lo, q_bar, head * kFaD, qt * kFaRows, grp);
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = 0; kt < n_tiles; ++kt) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      const int key0 = kt * kFaKeys;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = key0 + lane + 32 * h;
        const bool ok = k < p.Ls && (p.mask == nullptr || p.mask[srow0 + k] != 0);
        s_bias[stage * kFaKeys + lane + 32 * h] = ok ? 0.f : -INFINITY;
      }
      __syncwarp();
      if (lane == 0) {
        uint8_t* st = s_ring + stage * kFwStage;
        uint64_t* fb = &full_bar[stage];
        mbar_arrive_expect_tx(fb, kFwStage);
        tma_load_3d(st, &tm_kv_hi, fb, head * kFaD, key0, grp);
        tma_load_3d(st + kFwKvPlane, &tm_kv_lo, fb, head * kFaD, key0, grp);
        tma_load_3d(st + 2 * kFwKvPlane, &tm_kv_hi, fb, p.v_col0 + head * kFaD, key0, grp);
        tma_load_3d(st + 3 * kFwKvPlane, &tm_kv_lo, fb, p.v_col0 + head * kFaD, key0, grp);
      }
      __syncwarp();
      if (++stage == kFwStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }

  // ---- consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile
  const int wg = warp >> 2, wq = warp & 3;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int r_lo = qt * kFaRows + wg * 64 + wq * 16 + g4, r_hi = r_lo + 8;
  const uint32_t q_hi = smem_u32(s_q) + wg * 64 * 64, q_lo = q_hi + kFwQPlane;
  float o[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  mbar_wait(q_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int kt = 0; kt < n_tiles; ++kt) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t st = smem_u32(s_ring + stage * kFwStage);
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      const uint64_t adv = static_cast<uint64_t>(kk * 2);   // 16 fp16 = 32 bytes along K inside the swizzle row
      const uint64_t ah = wgmma_desc_k_sw64(q_hi) + adv, al = wgmma_desc_k_sw64(q_lo) + adv;
      const uint64_t bh = wgmma_desc_k_sw64(st) + adv, bl = wgmma_desc_k_sw64(st + kFwKvPlane) + adv;
      wgmma_f16<64>(s, ah, bh, 1u);
      wgmma_f16<64>(s, ah, bl, 1u);
      wgmma_f16<64>(s, al, bh, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // ---- scale, mask, online softmax: s[4j + 0..1] row g, s[4j + 2..3] row g + 8, columns 8j + 2t (+1)
    const float* bias = s_bias + stage * kFaKeys;
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float b0 = bias[j * 8 + 2 * t4], b1 = bias[j * 8 + 2 * t4 + 1];
      s[4 * j] = fmaf(s[4 * j], p.scale_log2, b0);
      s[4 * j + 1] = fmaf(s[4 * j + 1], p.scale_log2, b1);
      s[4 * j + 2] = fmaf(s[4 * j + 2], p.scale_log2, b0);
      s[4 * j + 3] = fmaf(s[4 * j + 3], p.scale_log2, b1);
      mx_lo = fmaxf(mx_lo, fmaxf(s[4 * j], s[4 * j + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
    const float mu_lo = mn_lo == -INFINITY ? 0.f : mn_lo, mu_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
    const float corr_lo = exp2f(m_lo - mu_lo), corr_hi = exp2f(m_hi - mu_hi);
    m_lo = mn_lo;
    m_hi = mn_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[4 * j] = exp2f(s[4 * j] - mu_lo);
      s[4 * j + 1] = exp2f(s[4 * j + 1] - mu_lo);
      s[4 * j + 2] = exp2f(s[4 * j + 2] - mu_hi);
      s[4 * j + 3] = exp2f(s[4 * j + 3] - mu_hi);
      sum_lo += s[4 * j] + s[4 * j + 1];
      sum_hi += s[4 * j + 2] + s[4 * j + 3];
    }
    l_lo = fmaf(l_lo, corr_lo, sum_lo);
    l_hi = fmaf(l_hi, corr_hi, sum_hi);
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      o[4 * n] *= corr_lo;
      o[4 * n + 1] *= corr_lo;
      o[4 * n + 2] *= corr_hi;
      o[4 * n + 3] *= corr_hi;
    }
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      split_f16x2(s[8 * kk], s[8 * kk + 1], ph[kk][0], pl[kk][0]);
      split_f16x2(s[8 * kk + 2], s[8 * kk + 3], ph[kk][1], pl[kk][1]);
      split_f16x2(s[8 * kk + 4], s[8 * kk + 5], ph[kk][2], pl[kk][2]);
      split_f16x2(s[8 * kk + 6], s[8 * kk + 7], ph[kk][3], pl[kk][3]);
    }
    // ---- O += P V: k-step kk = keys [16 kk, 16 kk + 16) = 16 rows of 64 B of the V tile
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t off = static_cast<uint32_t>(kk * 16 * 64);
      const uint64_t vh = wgmma_desc_mn_sw64(st + 2 * kFwKvPlane + off);
      const uint64_t vl = wgmma_desc_mn_sw64(st + 3 * kFwKvPlane + off);
      wgmma_rs_n32_tb(o, ph[kk], vh);
      wgmma_rs_n32_tb(o, ph[kk], vl);
      wgmma_rs_n32_tb(o, pl[kk], vh);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    mbar_arrive(&empty_bar[stage]);
    if (++stage == kFwStages) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ---- epilogue: O / rowsum -> fp16 planes; padded queries and rows without a valid key write 0
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = rr ? r_hi : r_lo;
    if (r >= p.Lx) continue;
    const float l = rr ? l_hi : l_lo;
    const bool q_ok = p.mask == nullptr || p.mask[xrow0 + r] != 0;
    const float inv = (q_ok && l > 0.f) ? 1.f / l : 0.f;
    const long off = (xrow0 + r) * p.ld_o + head * kFaD + 2 * t4;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      uint32_t h, lo;
      split_f16x2(o[4 * n + 2 * rr] * inv, o[4 * n + 2 * rr + 1] * inv, h, lo);
      *reinterpret_cast<uint32_t*>(p.o_hi + off + n * 8) = h;
      *reinterpret_cast<uint32_t*>(p.o_lo + off + n * 8) = lo;
    }
  }
}

}  // namespace lb
