// Epilogue functors for gemm_split_kernel.  Each one is the fused tail of a reference op group
// (SURVEY.md §2a G1-G7): the thread that owns accumulator row r applies the
// elementwise / row-wise work that the reference runs as separate eager kernels.
#pragma once
#include <cuda_fp16.h>
#include "gemm_split.cuh"

namespace lb {

constexpr float kNegBig = -1.0e30f;  // finite stand-in for -inf (keeps exp(x - max) NaN-free)
constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exp(x) for x <= 0 (softmax numerators)
__device__ __forceinline__ float exp_fast(float x) { return ex2_approx(x * kLog2e); }
// elu(x) + 1 = x + 1 (x > 0) | exp(x) (x <= 0): the feature map of the linear attention (linear_attention.py:7-8).
// Branch-free: the exponential is always evaluated (ex2.approx of min(x, 0) * log2 e, relative error ~1e-6, the level
// of the split-precision GEMMs around it) and selected.  expf() compiles to a guarded slow path per element.
__device__ __forceinline__ float elu_plus1(float x) {
  const float e = exp_fast(fminf(x, 0.f));
  return x > 0.f ? x + 1.f : e;
}

__device__ __forceinline__ int epi_tid() { return threadIdx.x - kEpiWarp0 * 32; }   // 0..255
__device__ __forceinline__ int epi_row() { return epi_tid() & 127; }                  // accumulator row
__device__ __forceinline__ int epi_half() { return epi_tid() >> 7; }                  // column half of the tile
__device__ __forceinline__ void epi_bar_sync() { epi_group_sync(); }

// x = hi + lo with both halves fp16 (round-to-nearest); |x| must stay below 65504.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}

// Two values at once, packed as (a | b << 16): cvt.rn.f16x2.f32 (F2FP.PACK_AB) and HADD2.F32 run on the full-rate
// ALU, whereas the scalar F2F conversions of split_f16 go through the quarter-rate XU pipe (3 per value: measured as the
// `mio` / `wait` stalls of every plane-writing epilogue).  Bit-identical to split_f16 (round-to-nearest-even both).
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ void store_f32x32(float* p, const float (&x)[32]) {
  float4* q = reinterpret_cast<float4*>(p);
#pragma unroll
  for (int j = 0; j < 8; ++j) q[j] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
}

// 32 consecutive fp32 accumulator columns of this thread's row (acc_row: shared-memory address of the staged row)
__device__ __forceinline__ void load_acc32(uint32_t acc_row, int col, float (&x)[32]) {
  const uint32_t a = acc_row + static_cast<uint32_t>(col) * 4u;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(x[4 * j]), "=f"(x[4 * j + 1]), "=f"(x[4 * j + 2]), "=f"(x[4 * j + 3])
                 : "r"(a + 16u * j)
                 : "memory");
}

__device__ __forceinline__ void load_planes32(const __half* hp, const __half* lp, float (&x)[32]) {
  const uint4* h4 = reinterpret_cast<const uint4*>(hp);
  const uint4* l4 = reinterpret_cast<const uint4*>(lp);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 a = h4[j], b = l4[j];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&aw[k]));
      const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&bw[k]));
      x[j * 8 + 2 * k] = fh.x + fl.x;
      x[j * 8 + 2 * k + 1] = fh.y + fl.y;
    }
  }
}


// ------------------------------------------------------------------------------------------------
// Coalesced epilogue I/O.  An epilogue thread owns one accumulator ROW, so a warp-wide 16-byte store of "my row's
// next 16 bytes" touches 32 different cache lines (32 sectors per request: the L1 tag stage, not DRAM, becomes the
// limiter -- l1tex at 70-75 % in the round-1 ncu captures).  These helpers transpose a [32 rows x 64 B] block through
// a 2 KB per-warp shared-memory scratch (XOR-swizzled, bank-conflict free both ways) so that every global access
// instruction covers 8 rows x 64 contiguous bytes.  Rows are addressed by a per-lane pointer (lane = row; nullptr =
// row not stored / read as zero), so the same code serves row-major matrices and NHWC pixel rows.
// Per-warp 4 KB staging tile at the START of the epilogue area (1024-byte aligned): a [32 rows x 128 B] fp32 block or
// two [32 rows x 64 B] plane blocks (hi at +0, lo at +2048) for TMA stores; its first 2 KB double as the transposer
// scratch of the coalesced load / store helpers below.
constexpr int kEpiScratchBytes = 8 * 4096;   // 8 epilogue warps x 4 KB
__device__ __forceinline__ uint32_t* epi_scratch(uint8_t* base) {
  return reinterpret_cast<uint32_t*>(base + ((epi_tid() >> 5) << 12));
}
template <class T>
__device__ __forceinline__ T* shfl_ptr(T* p, int src_lane) {
  const unsigned long long v = __shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(p), src_lane);
  return reinterpret_cast<T*>(v);
}
// w[16]: 64 bytes of this lane's row -> *(row_ptr + 0..63) for every lane with row_ptr != nullptr
__device__ __forceinline__ void warp_store_rows64(uint32_t* scr, uint8_t* row_ptr, const uint32_t (&w)[16]) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 4; ++q)
    *reinterpret_cast<uint4*>(scr + lane * 16 + ((q ^ ((lane >> 1) & 3)) << 2)) =
        make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
  __syncwarp();
  const int g = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = (lane >> 2) + 8 * i;
    uint8_t* dst = shfl_ptr(row_ptr, r);
    const uint4 v = *reinterpret_cast<const uint4*>(scr + r * 16 + ((g ^ ((r >> 1) & 3)) << 2));
    if (dst) *reinterpret_cast<uint4*>(dst + g * 16) = v;
  }
}
// inverse: 64 bytes at row_ptr (zeros for nullptr) -> w[16] of the owning lane
__device__ __forceinline__ void warp_load_rows64(uint32_t* scr, const uint8_t* row_ptr, uint32_t (&w)[16]) {
  const int lane = threadIdx.x & 31;
  const int g = lane & 3;
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = (lane >> 2) + 8 * i;
    const uint8_t* src = shfl_ptr(row_ptr, r);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (src) v = *reinterpret_cast<const uint4*>(src + g * 16);
    *reinterpret_cast<uint4*>(scr + r * 16 + ((g ^ ((r >> 1) & 3)) << 2)) = v;
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint4 v = *reinterpret_cast<const uint4*>(scr + lane * 16 + ((q ^ ((lane >> 1) & 3)) << 2));
    w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
  }
}
// 32 values of my row as fp16 hi/lo planes: hi_ptr / lo_ptr address (row, first column) or nullptr
__device__ __forceinline__ void warp_store_planes32(uint32_t* scr, __half* hi_ptr, __half* lo_ptr, const float (&x)[32]) {
  uint32_t h[16], l[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    split_f16x2(x[2 * j], x[2 * j + 1], h[j], l[j]);
  }
  warp_store_rows64(scr, reinterpret_cast<uint8_t*>(hi_ptr), h);
  warp_store_rows64(scr, reinterpret_cast<uint8_t*>(lo_ptr), l);
}
__device__ __forceinline__ void warp_store_f32x32(uint32_t* scr, float* ptr, const float (&x)[32]) {
  uint32_t a[16], b[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    a[j] = __float_as_uint(x[j]);
    b[j] = __float_as_uint(x[16 + j]);
  }
  warp_store_rows64(scr, reinterpret_cast<uint8_t*>(ptr), a);
  warp_store_rows64(scr, ptr ? reinterpret_cast<uint8_t*>(ptr) + 64 : nullptr, b);
}
// 32 values of my row from fp16 hi/lo planes, in two steps: `issue` puts the lane's eight 16-byte global loads in flight
// (rows lane/4 + 8i, 16-byte group lane%4), `finish` transposes them through the scratch into this lane's row.  An
// epilogue can issue before it waits for / converts its accumulator group and finish afterwards.
__device__ __forceinline__ void warp_issue_planes32(const __half* hi_ptr, const __half* lo_ptr, uint4 (&vh)[4], uint4 (&vl)[4]) {
  const int lane = threadIdx.x & 31;
  const int g = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = (lane >> 2) + 8 * i;
    const uint8_t* sh = shfl_ptr(reinterpret_cast<const uint8_t*>(hi_ptr), r);
    const uint8_t* sl = shfl_ptr(reinterpret_cast<const uint8_t*>(lo_ptr), r);
    vh[i] = make_uint4(0u, 0u, 0u, 0u);
    vl[i] = make_uint4(0u, 0u, 0u, 0u);
    if (sh) vh[i] = *reinterpret_cast<const uint4*>(sh + g * 16);
    if (sl) vl[i] = *reinterpret_cast<const uint4*>(sl + g * 16);
  }
}
__device__ __forceinline__ void warp_finish_planes32(uint32_t* scr, const uint4 (&vh)[4], const uint4 (&vl)[4], float (&x)[32]) {
  uint32_t h[16], l[16];
  const int lane = threadIdx.x & 31;
  const int g = lane & 3;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = (lane >> 2) + 8 * i;
      *reinterpret_cast<uint4*>(scr + r * 16 + ((g ^ ((r >> 1) & 3)) << 2)) = pass == 0 ? vh[i] : vl[i];
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint4 v = *reinterpret_cast<const uint4*>(scr + lane * 16 + ((q ^ ((lane >> 1) & 3)) << 2));
      if (pass == 0) {
        h[4 * q] = v.x; h[4 * q + 1] = v.y; h[4 * q + 2] = v.z; h[4 * q + 3] = v.w;
      } else {
        l[4 * q] = v.x; l[4 * q + 1] = v.y; l[4 * q + 2] = v.z; l[4 * q + 3] = v.w;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&h[j]));
    const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&l[j]));
    x[2 * j] = fh.x + fl.x;
    x[2 * j + 1] = fh.y + fl.y;
  }
}
__device__ __forceinline__ void warp_load_f32x32(uint32_t* scr, const float* ptr, float (&x)[32]) {
  uint32_t a[16], b[16];
  warp_load_rows64(scr, reinterpret_cast<const uint8_t*>(ptr), a);
  warp_load_rows64(scr, ptr ? reinterpret_cast<const uint8_t*>(ptr) + 64 : nullptr, b);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    x[j] = __uint_as_float(a[j]);
    x[16 + j] = __uint_as_float(b[j]);
  }
}


// ------------------------------------------------------------------------------------------------
// TMA-store epilogue path: the warp stages its 32-row block in shared memory in the tensor map's swizzled box layout
// and ONE lane hands it to the copy engine (cp.async.bulk.tensor ... bulk_group): full-line writes, no per-lane
// address generation, rows / channels beyond the tensor's extent are clipped by the map (no predicates).  The staging
// tile is reused only after the engine has read the previous block (wait_group.read).
struct OutMaps {            // filled on the host (engine.cu make_out_map_*) for the outputs an epilogue writes
  CUtensorMap hi, lo, f32;
  int use;                  // bit 0: planes map set, bit 1: fp32 map set.  The host always sets the bits of the outputs
                            // it passes; EpiLayerNorm and EpiConv keep pointer stores for a clear bit because without
                            // that code ptxas allocates their registers worse (more spills in EpiConv<256, 0>)
  int dims;                 // 3: (col, row, batch) coordinates;  4: NHWC (channel, x, y, image) coordinates
};
struct OutCoord {           // where this warp's 32-row block goes
  int c0, c1, c2, c3;       // dims == 3: (col, row0, batch, -);  dims == 4: (channel, x0, y0, image)
};
__device__ __forceinline__ void tma_store_box(const CUtensorMap* m, const void* src, int dims, const OutCoord& o) {
  if (dims == 4) tma_store_4d(m, src, o.c0, o.c1, o.c2, o.c3);
  else tma_store_3d(m, src, o.c0, o.c1, o.c2);
}
// 32 values of my row -> fp16 hi/lo planes, box = 32 columns (64 B, 64-byte swizzle) x 32 rows
__device__ __forceinline__ void warp_tma_store_planes32(uint32_t* stage, const OutMaps& om, const OutCoord& o, const float (&x)[32]) {
  const int lane = threadIdx.x & 31;
  uint32_t h[16], l[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    split_f16x2(x[2 * j], x[2 * j + 1], h[j], l[j]);
  }
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
  const int sw = (lane >> 1) & 3;   // 64-byte swizzle: 16-byte chunk q of row r lives at q ^ ((r >> 1) & 3)
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    *reinterpret_cast<uint4*>(stage + lane * 16 + ((q ^ sw) << 2)) = make_uint4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]);
    *reinterpret_cast<uint4*>(stage + 512 + lane * 16 + ((q ^ sw) << 2)) = make_uint4(l[4 * q], l[4 * q + 1], l[4 * q + 2], l[4 * q + 3]);
  }
  fence_proxy_async();
  __syncwarp();
  if (lane == 0) {
    tma_store_box(&om.hi, stage, om.dims, o);
    tma_store_box(&om.lo, stage + 512, om.dims, o);
    tma_store_commit();
  }
}
// 32 fp32 values of my row, box = 32 columns (128 B, 128-byte swizzle) x 32 rows
__device__ __forceinline__ void warp_tma_store_f32x32(uint32_t* stage, const OutMaps& om, const OutCoord& o, const float (&x)[32]) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 8; ++q)
    *reinterpret_cast<float4*>(stage + lane * 32 + ((q ^ (lane & 7)) << 2)) = make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]);
  fence_proxy_async();
  __syncwarp();
  if (lane == 0) {
    tma_store_box(&om.f32, stage, om.dims, o);
    tma_store_commit();
  }
}
// The transposer helpers use the first 2 KB of the same tile: wait until the copy engine is done reading it.
__device__ __forceinline__ void stage_quiesce() {
  if ((threadIdx.x & 31) == 0) tma_store_wait_read();
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// out[row, col] = act(acc) * rowmask[row];  act = elu(x)+1 for col < elu_cols, identity otherwise.
// Covers q/k/v projection + feature map + padding mask of LinearAttention
// (reference linear_attention.py:31-39: Q = elu(q)+1, K = elu(k)+1, Q*=q_mask, K*=kv_mask, V*=kv_mask).
template <int BLOCK_N>
struct EpiActStore {
  struct Params {
    float* out;              // [batches*M, ld] (written through om.f32)
    int ld;
    int elu_cols;            // columns [0, elu_cols) get elu+1
    const uint8_t* rowmask;  // optional [batches*M] (1 = valid)
    float acc_scale;         // 2^-e: undoes the power-of-two pre-scaling of the weight planes (exact)
    int skip;                // probe mode (LOFTR_B200_PROBE_NULL_EPI, lb_gemm_split only): 1 = drain nothing, 2 = accumulator loads only
    OutMaps om;              // om.f32: the fp32 output
  };
  static constexpr int kSmemBytes = kEpiScratchBytes;
  const Params& p;
  const GemmShape& s;
  uint32_t* scr;
  __device__ EpiActStore(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), scr(epi_scratch(smem)) {}
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  __device__ void prefetch(int, int, int) {}
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    if (p.skip == 1) return;
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    const long grow = static_cast<long>(batch) * s.M + r;
    float mk = 1.f;
    if (row_ok && p.rowmask) mk = p.rowmask[grow] ? 1.f : 0.f;
    const int c_begin = epi_half() * (BLOCK_N / 64);
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      const int col = n0 + c * 32;
      if (col >= s.N) break;  // warp-uniform
      float x[32];
      load_acc32(acc_row, c * 32, x);
      if (p.skip == 2) {   // keep the loads alive without storing
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) acc += x[j];
        if (acc == 1.2345e-30f) p.out[0] = acc;
        continue;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= p.acc_scale;
      if (col < p.elu_cols) {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = elu_plus1(x[j]);
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= mk;
      warp_tma_store_f32x32(scr, p.om, OutCoord{col, m0 + ((epi_tid() >> 5) & 3) * 32, batch, 0}, x);
    }
  }
};


// ------------------------------------------------------------------------------------------------
// Linear attention fused into the projections (SURVEY.md §2a G1/G2; reference linear_attention.py:31-46).
// The fp32 q / k / v tensors of the reference never reach HBM: the k|v projection writes K and V as planes (EpiKvProj,
// below), kv_gemm_kernel reduces them to KV / Ksum, and the q projection applies them (EpiAttn).
//
// EpiAttn: epilogue of the q projection.  Q = elu(q)+1 (masked), then for the head that owns each 32-column group
//     out[r, h, :] = (Q[r,h,:] . KV[g,h]) / (Q[r,h,:] . Ksum[g,h] + eps)                    (linear_attention.py:44-46)
// with KV / Ksum of the row's group (batch) staged in shared memory, written as fp16 planes = the A operand of the
// merge projection.  Requires N == BLOCK_N == H * D (one n-tile) and a batched launch (batch = group).
template <int BLOCK_N, int D>
struct EpiAttn {
  static_assert(D == 32 && BLOCK_N == 256, "built for the coarse transformer (d_model 256, 8 heads)");
  struct Params {
    const uint8_t* rowmask;  // optional [batches*M]
    float acc_scale;
    const float* kv;         // [batches][H][D*D + D]
    float eps;
    __half* att_hi;          // [batches*M, ld]
    __half* att_lo;
    int ld;
  };
  static constexpr int kH = BLOCK_N / D;
  static constexpr int kPer = D * D + D;
  static constexpr int kSmemBytes = kH * kPer * 4;
  const Params& p;
  const GemmShape& s;
  float* sKV;
  int cur_batch;
  __device__ EpiAttn(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), cur_batch(-1) {
    sKV = reinterpret_cast<float*>(smem);
  }
  __device__ void item_begin(int batch, int, int) {
    if (batch != cur_batch) {   // uniform over the 256 epilogue threads
      epi_bar_sync();           // nobody still reads the previous group's matrices
      const float4* src = reinterpret_cast<const float4*>(p.kv + static_cast<long>(batch) * kH * kPer);
      float4* dst = reinterpret_cast<float4*>(sKV);
      for (int i = epi_tid(); i < kH * kPer / 4; i += kEpiThreads) dst[i] = src[i];
      epi_bar_sync();
      cur_batch = batch;
    }
  }
  __device__ void item_end(int, int, int) {}
  __device__ void prefetch(int, int, int) {}
  __device__ void tile(uint32_t acc_row, int batch, int m0, int) {
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    const long grow = static_cast<long>(batch) * s.M + r;
    float mk = 1.f;
    if (row_ok && p.rowmask) mk = p.rowmask[grow] ? 1.f : 0.f;
    const int c_begin = epi_half() * (BLOCK_N / 64);
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      float q[32];
      load_acc32(acc_row, c * 32, q);
      const float* kvh = sKV + c * kPer;   // head = column group
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float x = q[j] * p.acc_scale;
        q[j] = elu_plus1(x) * mk;
      }
      float zden = p.eps;
#pragma unroll
      for (int d = 0; d < D; ++d) zden = fmaf(q[d], kvh[D * D + d], zden);
      const float z = 1.f / zden;
      __half* hp = p.att_hi + grow * p.ld + c * 32;
      __half* lp = p.att_lo + grow * p.ld + c * 32;
#pragma unroll
      for (int v8 = 0; v8 < D; v8 += 8) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const float4 a = *reinterpret_cast<const float4*>(&kvh[d * D + v8]);
          const float4 b = *reinterpret_cast<const float4*>(&kvh[d * D + v8 + 4]);
          o[0] = fmaf(q[d], a.x, o[0]); o[1] = fmaf(q[d], a.y, o[1]);
          o[2] = fmaf(q[d], a.z, o[2]); o[3] = fmaf(q[d], a.w, o[3]);
          o[4] = fmaf(q[d], b.x, o[4]); o[5] = fmaf(q[d], b.y, o[5]);
          o[6] = fmaf(q[d], b.z, o[6]); o[7] = fmaf(q[d], b.w, o[7]);
        }
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          split_f16x2(o[2 * j] * z, o[2 * j + 1] * z, hw[j], lw[j]);
        }
        if (row_ok) {
          *reinterpret_cast<uint4*>(hp + v8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
          *reinterpret_cast<uint4*>(lp + v8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// y = LayerNorm(acc) * gamma + beta (+ residual) over the full row (requires N == BLOCK_N).
// Covers merge+norm1 and mlp[2]+norm2+residual of LoFTREncoderLayer (reference transformer.py:51-58).
template <int BLOCK_N>
struct EpiLayerNorm {
  struct Params {
    const float* gamma;
    const float* beta;
    float eps;
    const float* residual;  // optional fp32 residual [rows, ld_res]
    int ld_res;
    const __half* res_hi;   // optional residual as fp16 planes [rows, ld_res_pl] (x = hi + lo, exact to 2^-22): the
    const __half* res_lo;   // residual stream then needs no fp32 master copy between layers
    int ld_res_pl;
    float* out_f32;         // optional [rows, ld_f32]
    int ld_f32;
    __half* out_hi;         // optional planes [rows, ld_pl], written at column offset pl_col0
    __half* out_lo;
    int ld_pl;
    int pl_col0;
    float acc_scale;        // 2^-e of the weight planes
    OutMaps om;             // TMA-store maps of (out_hi, out_lo) [based at column pl_col0] and out_f32
  };
  // gamma / beta are read through the read-only cache (2 KB, L1-resident): the shared memory goes to the staging tiles
  static constexpr int kSmemBytes = kEpiScratchBytes + 2 * 128 * 8 + 128 * 4;
  const Params& p;
  const GemmShape& s;
  float* s_red;  // [2 halves][128 rows] float2 + [128] shift
  uint32_t* scr;
  __device__ EpiLayerNorm(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), scr(epi_scratch(smem)) {
    s_red = reinterpret_cast<float*>(smem + kEpiScratchBytes);
  }
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  // pull this thread's residual segments towards L2 while the tensor core is still producing the tile
  __device__ void prefetch(int batch, int m0, int) {
    const int r = m0 + epi_row();
    if (r >= s.M) return;
    const long grow = static_cast<long>(batch) * s.M + r;
    const int c0 = epi_half() * (BLOCK_N / 2);
    if (p.res_hi) {
      for (int c = 0; c < BLOCK_N / 2; c += 64) {   // 64 fp16 = one 128-byte line
        prefetch_l2(p.res_hi + grow * p.ld_res_pl + c0 + c);
        prefetch_l2(p.res_lo + grow * p.ld_res_pl + c0 + c);
      }
    }
    if (p.residual) {
      for (int c = 0; c < BLOCK_N / 2; c += 32) prefetch_l2(p.residual + grow * p.ld_res + c0 + c);
    }
  }
  // the two threads that share a row (column halves) exchange their partial (sum, sum of squares) through smem
  __device__ float2 row_total2(float a, float b) {
    const int row = epi_row(), half = epi_half();
    float2* red = reinterpret_cast<float2*>(s_red);
    red[half * 128 + row] = make_float2(a, b);
    epi_bar_sync();
    const float2 u = red[row], v = red[128 + row];
    epi_bar_sync();
    return make_float2(u.x + v.x, u.y + v.y);
  }
  __device__ void tile(uint32_t acc_row, int batch, int m0, int) {
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    const long grow = static_cast<long>(batch) * s.M + r;
    const int c_begin = epi_half() * (BLOCK_N / 64);
    const int c_end = c_begin + BLOCK_N / 64;
    // one pass over the accumulator for both moments (biased variance E[x^2] - mean^2 in fp32: the normalised inputs
    // are O(1) with |mean| << 1 + std, so the cancellation costs < 1e-6 relative), shifted by the row's first value
    float sum = 0.f, sq = 0.f, shift = 0.f;
#pragma unroll 1
    for (int c = c_begin; c < c_end; ++c) {
      float x[32];
      load_acc32(acc_row, c * 32, x);
      if (c == c_begin) shift = x[0] * p.acc_scale;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float d = x[j] * p.acc_scale - shift;
        sum += d;
        sq = fmaf(d, d, sq);
      }
    }
    // both column halves must use the same shift: re-centre the right half's moments onto the left half's shift
    float* sh_shift = s_red + 2 * 128 * 2;   // [128] behind the float2 exchange area
    if (epi_half() == 0) sh_shift[epi_row()] = shift;
    epi_bar_sync();
    {
      const float delta = shift - sh_shift[epi_row()];     // 0 for the left half
      const float n = static_cast<float>(BLOCK_N / 2);
      sq = sq + 2.f * delta * sum + n * delta * delta;       // sum (d + delta)^2
      sum = sum + n * delta;
      shift -= delta;
    }
    const float2 tot = row_total2(sum, sq);
    const float m1 = tot.x * (1.f / BLOCK_N);
    const float mean = shift + m1;
    const float var = fmaxf(tot.y * (1.f / BLOCK_N) - m1 * m1, 0.f);
    const float rstd = rsqrtf(var + p.eps);
#pragma unroll 1
    for (int c = c_begin; c < c_end; ++c) {
      // residual rows of this 32-column group: requested before the accumulator group is fetched and normalised
      // (18 % of the mlp[2]+norm2 kernel's samples waited on them when they were loaded after the arithmetic)
      uint4 rh[4], rl[4];
      if (p.res_hi)
        warp_issue_planes32(row_ok ? p.res_hi + grow * p.ld_res_pl + c * 32 : nullptr,
                            row_ok ? p.res_lo + grow * p.ld_res_pl + c * 32 : nullptr, rh, rl);
      float x[32];
      load_acc32(acc_row, c * 32, x);
#pragma unroll
      for (int j4 = 0; j4 < 8; ++j4) {
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.gamma + c * 32) + j4);
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.beta + c * 32) + j4);
        x[4 * j4] = (x[4 * j4] * p.acc_scale - mean) * rstd * g4.x + b4.x;
        x[4 * j4 + 1] = (x[4 * j4 + 1] * p.acc_scale - mean) * rstd * g4.y + b4.y;
        x[4 * j4 + 2] = (x[4 * j4 + 2] * p.acc_scale - mean) * rstd * g4.z + b4.z;
        x[4 * j4 + 3] = (x[4 * j4 + 3] * p.acc_scale - mean) * rstd * g4.w + b4.w;
      }
      // warp-cooperative (coalesced) residual loads and stores: every lane takes part, invalid rows pass nullptr
      if (p.om.use && (p.residual || p.res_hi)) stage_quiesce();
      if (p.residual) {
        float r[32];
        warp_load_f32x32(scr, row_ok ? p.residual + grow * p.ld_res + c * 32 : nullptr, r);
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] += r[j];
      }
      if (p.res_hi) {
        float r[32];
        warp_finish_planes32(scr, rh, rl, r);
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] += r[j];
      }
      const OutCoord oc{c * 32, m0 + ((epi_tid() >> 5) & 3) * 32, batch, 0};
      if (p.out_f32) {
        if (p.om.use & 2) warp_tma_store_f32x32(scr, p.om, oc, x);
        else warp_store_f32x32(scr, row_ok ? p.out_f32 + grow * p.ld_f32 + c * 32 : nullptr, x);
      }
      if (p.out_hi) {
        if (p.om.use & 1) {
          warp_tma_store_planes32(scr, p.om, oc, x);
        } else {
          const long off = grow * p.ld_pl + p.pl_col0 + c * 32;
          warp_store_planes32(scr, row_ok ? p.out_hi + off : nullptr, row_ok ? p.out_lo + off : nullptr, x);
        }
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// h = relu(acc) -> fp16 planes (mlp[0]+ReLU, reference transformer.py:22-26,55)
// or, with group_bias: y = acc + gbias[row / group_rows, col] -> fp32 + planes
// (merge_feat over [window | repeated coarse feature], reference fine_preprocess.py:51-56: the
// repeated half of the concatenation contributes one bias vector per window).
template <int BLOCK_N>
struct EpiPlanes {
  struct Params {
    int relu;
    const float* gbias;   // optional [groups, N]
    int group_rows;
    float* out_f32;       // optional
    int ld_f32;
    __half* out_hi;
    __half* out_lo;
    int ld_pl;
    int pl_col0;
    float acc_scale;      // 2^-e of the weight planes
    OutMaps om;           // TMA-store maps of (out_hi, out_lo) [based at column pl_col0] and out_f32
  };
  static constexpr int kSmemBytes = kEpiScratchBytes;
  const Params& p;
  const GemmShape& s;
  uint32_t* scr;
  __device__ EpiPlanes(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), scr(epi_scratch(smem)) {}
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  __device__ void prefetch(int, int, int) {}
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    const long grow = static_cast<long>(batch) * s.M + r;
    const float* gb = nullptr;
    if (p.gbias && row_ok) gb = p.gbias + (grow / p.group_rows) * s.N;
    const int c_begin = epi_half() * (BLOCK_N / 64);
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      const int col = n0 + c * 32;
      if (col >= s.N) break;
      float x[32];
      load_acc32(acc_row, c * 32, x);
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= p.acc_scale;
      if (p.relu) {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = fmaxf(x[j], 0.f);
      }
      if (gb) {
        const float4* bp = reinterpret_cast<const float4*>(gb + col);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 t = bp[j];
          x[4 * j] += t.x;
          x[4 * j + 1] += t.y;
          x[4 * j + 2] += t.z;
          x[4 * j + 3] += t.w;
        }
      }
      const OutCoord oc{col, m0 + ((epi_tid() >> 5) & 3) * 32, batch, 0};
      if (p.out_f32) warp_tma_store_f32x32(scr, p.om, oc, x);
      if (p.out_hi) warp_tma_store_planes32(scr, p.om, oc, x);
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Convolution epilogue (backbone, reference src/loftr/backbone/resnet_fpn.py): the accumulator row r of tile
// (ty, tx) is output pixel (ty*8 + r/16, tx*16 + r%16).
//   y = acc * scale[c] + shift[c]            eval-mode BatchNorm folded to an affine map (BasicBlock :28-40)
//   y += residual[pixel, c]                  BasicBlock skip connection (:35-40)
//   y += bilinear_x2(up_src)[pixel, c]       FPN top-down merge, F.interpolate(scale_factor=2, bilinear,
//                                            align_corners=True) (:107-113)
//   y = relu / leaky_relu(0.01) / identity
// written as NHWC fp16 planes (the next convolution's A operand) and / or NHWC fp32.
//
// kUpMode selects the FPN merge: 0 = none (every other layer: no upsample code, leanest registers), 1 = staged window,
// 2 = per-thread global gathers (any shape).  The engine dispatches 0 and 2: the staged window's shared memory does
// not fit beside the TMA ring and the accumulator staging of gemm_split_kernel.
// kUpMode = 1 (the two FPN lateral 1x1 convolutions): the 6 x 10 source pixels whose bilinear footprints cover the
// 8 x 16 output tile are fetched ONCE per tile by TMA into shared memory (boxes of 200 / 2 x 136 channels: the pixel
// stride of 100 / 68 words keeps the quarter-warp LDS.128 conflict-free) while the tile's MMAs run; the four
// neighbours of a pixel are then shared-memory reads.  With per-thread global loads (kUpMode = 2) the
// kernel is bound by L1 tag lookups: 32 LDG.128 per thread and 32-channel group, each touching ~16 lines.
struct UpMaps {
  CUtensorMap hi, lo;   // upsample source planes [batches, up_h, up_w, C], unswizzled boxes (kUpBoxC, 10, 6, 1)
};
constexpr int kUpW = 10, kUpH = 6;
template <int BLOCK_N, int kUpMode = 0>
struct EpiConv {
  static constexpr bool kNoRowBound = true;      // backbone shapes are static: no device row bound (gemm_split.cuh)
  static constexpr bool kUp = kUpMode == 1;      // staged window
  static constexpr bool kUpAny = kUpMode != 0;
  struct Params {
    const float* scale;   // [N]
    const float* shift;   // [N]
    int act;              // 0 none, 1 relu, 2 leaky relu (0.01)
    const __half* res_hi; // optional residual planes, NHWC, same spatial size, row stride res_ld
    const __half* res_lo;
    int res_ld;
    const __half* up_hi;  // optional x2-upsample source planes [batches, up_h, up_w, up_ld]
    const __half* up_lo;
    int up_ld, up_h, up_w;
    __half* out_hi;       // optional NHWC planes [batches*H*W, out_ld]
    __half* out_lo;
    int out_ld;
    float* out_f32;       // optional NHWC fp32 [batches*H*W, f32_ld]
    int f32_ld;
    int H_out, W_out, tiles_w;
    OutMaps om;           // NHWC TMA-store maps (channel, x, y, image): box 32 channels x 16 x 2 pixels
    UpMaps um;            // kUp only
  };
  static constexpr int kChunks = (BLOCK_N + 31) / 32;        // 32-column groups of the tile (the last may be partial)
  static constexpr int kChunksHalf0 = (kChunks + 1) / 2;     // column half 0 takes the first ones
  static constexpr int kCols = kChunks * 32;
  static constexpr int kUpBoxC = BLOCK_N <= 208 ? 200 : 136; // channels per staged pixel (one box / two boxes at 0, 128)
  static constexpr int kUpBoxes = BLOCK_N <= 208 ? 1 : 2;
  static constexpr int kUpBoxData = kUpH * kUpW * kUpBoxC * 2;          // bytes one TMA box delivers
  static constexpr int kUpBoxBytes = (kUpBoxData + 127) & ~127;         // its (128-byte aligned) slot
  static constexpr int kUpPlaneBytes = kUpBoxes * kUpBoxBytes;
  static constexpr int kUpOffset = kEpiScratchBytes + 2 * kCols * 4;
  // N = 208 has 17.9 KB of shared memory to spare beside its three-stage ring: the residual transposer gets its own
  // 2 KB per warp there instead of aliasing the TMA-store staging tile, so a chunk's residual read no longer waits for
  // the copy engine to finish reading the previous chunk's store (11 us per tile in the layer2 conv2 kernels)
  static constexpr bool kOwnXpose = BLOCK_N == 208 && kUpMode == 0;
  static constexpr int kSmemBytes = kUpOffset + (kUp ? 2 * kUpPlaneBytes + 16 : 0) + (kOwnXpose ? 8 * 2048 : 0);
  static_assert(kUpOffset % 128 == 0 && kUpBoxBytes % 128 == 0, "TMA destinations are 128-byte aligned");
  static_assert(!kUp || BLOCK_N > 128, "the staged upsample is built for the 196- and 256-channel laterals");
  const Params& p;
  const GemmShape& s;
  float* s_scale;
  float* s_shift;
  uint32_t* scr;
  uint32_t* xscr;       // transposer scratch of the residual loads (== scr unless kOwnXpose)
  uint8_t* s_up;        // [hi | lo][box][6][10][kUpBoxC] fp16
  uint64_t* up_bar;
  uint32_t up_phase = 0;
  __device__ EpiConv(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), scr(epi_scratch(smem)) {
    s_scale = reinterpret_cast<float*>(smem + kEpiScratchBytes);
    s_shift = s_scale + kCols;
    s_up = smem + kUpOffset;
    xscr = kOwnXpose ? reinterpret_cast<uint32_t*>(smem + kUpOffset + ((epi_tid() >> 5) << 11)) : scr;
    up_bar = reinterpret_cast<uint64_t*>(smem + kUpOffset + 2 * kUpPlaneBytes);
    if (kUp) {
      if ((smem_u32(s_up) & 127u) != 0) asm volatile("trap;");
      if (epi_tid() == 0) {
        mbar_init(up_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&p.um.hi);
        tma_prefetch_desc(&p.um.lo);
      }
    }
    if (s.n_tiles == 1) {   // every layer of the backbone: one n-tile -> the folded BatchNorm is staged once per CTA
      stage_affine(0);
      epi_bar_sync();
    } else if (kUp) {
      epi_bar_sync();
    }
  }
  // first source row / column of the staged window of tile (ty, tx): the footprint of its first pixel
  __device__ void up_window(int ty, int tx, int& ybase, int& xbase) const {
    const float sh = p.H_out > 1 ? static_cast<float>(p.up_h - 1) / static_cast<float>(p.H_out - 1) : 0.f;
    const float sw = p.W_out > 1 ? static_cast<float>(p.up_w - 1) / static_cast<float>(p.W_out - 1) : 0.f;
    ybase = static_cast<int>(sh * (ty * kConvTileH));
    xbase = static_cast<int>(sw * (tx * kConvTileW));
  }
  __device__ void stage_affine(int n0) {
    for (int j = epi_tid(); j < kCols; j += kEpiThreads) {
      const int c = n0 + j;
      s_scale[j] = c < s.N ? p.scale[c] : 0.f;
      s_shift[j] = c < s.N ? p.shift[c] : 0.f;
    }
  }
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  // residual / FPN-upsample source rows of this thread's pixel -> L2, issued while the tile's MMAs still run
  __device__ void prefetch(int batch, int m0, int n0) {
    if (kUp) {
      // every epilogue thread has finished reading the previous tile's window (it got here); then one thread refills it
      epi_bar_sync();
      if (epi_tid() == 0) {
        const int mt = m0 / kBlockM;
        const int ty = mt / p.tiles_w, tx = mt - ty * p.tiles_w;
        int ybase, xbase;
        up_window(ty, tx, ybase, xbase);
        mbar_arrive_expect_tx(up_bar, 2 * kUpBoxes * kUpBoxData);
#pragma unroll
        for (int b = 0; b < kUpBoxes; ++b) {
          tma_load_4d(s_up + b * kUpBoxBytes, &p.um.hi, up_bar, b * 128, xbase, ybase, batch);
          tma_load_4d(s_up + kUpPlaneBytes + b * kUpBoxBytes, &p.um.lo, up_bar, b * 128, xbase, ybase, batch);
        }
      }
    }
    if (!p.res_hi && (kUp || !p.up_hi)) return;
    const int row = epi_row();
    const int mt = m0 / kBlockM;
    const int ty = mt / p.tiles_w, tx = mt - ty * p.tiles_w;
    const int y = ty * kConvTileH + row / kConvTileW;
    const int x = tx * kConvTileW + row % kConvTileW;
    if (y >= p.H_out || x >= p.W_out) return;
    const int c_lo = n0 + (epi_half() == 0 ? 0 : kChunksHalf0) * 32;
    const int c_hi = min(n0 + (epi_half() == 0 ? kChunksHalf0 : kChunks) * 32, s.N);
    if (p.res_hi) {
      // one request per 128 bytes of the row segment from its first byte (measured: also covering the last, partially
      // used line -- pixel rows of 196 channels are 400 bytes apart -- costs more than it saves: 635 -> 675 us)
      const long pix = (static_cast<long>(batch) * p.H_out + y) * p.W_out + x;
      for (int c = c_lo; c < c_hi; c += 64) {
        prefetch_l2(p.res_hi + pix * p.res_ld + c);
        prefetch_l2(p.res_lo + pix * p.res_ld + c);
      }
    }
    if (kUpMode == 2 && p.up_hi) {
      const float sh = p.H_out > 1 ? static_cast<float>(p.up_h - 1) / static_cast<float>(p.H_out - 1) : 0.f;
      const float sw = p.W_out > 1 ? static_cast<float>(p.up_w - 1) / static_cast<float>(p.W_out - 1) : 0.f;
      const int y0 = static_cast<int>(sh * y), x0 = static_cast<int>(sw * x);
      const int y1 = y0 + (y0 < p.up_h - 1 ? 1 : 0), x1 = x0 + (x0 < p.up_w - 1 ? 1 : 0);
      const long base = static_cast<long>(batch) * p.up_h * p.up_w;
      const long u[4] = {(base + static_cast<long>(y0) * p.up_w + x0) * p.up_ld, (base + static_cast<long>(y0) * p.up_w + x1) * p.up_ld,
                         (base + static_cast<long>(y1) * p.up_w + x0) * p.up_ld, (base + static_cast<long>(y1) * p.up_w + x1) * p.up_ld};
      for (int q = 0; q < 4; ++q)
        for (int c = c_lo; c < c_hi; c += 64) {
          prefetch_l2(p.up_hi + u[q] + c);
          prefetch_l2(p.up_lo + u[q] + c);
        }
    }
  }
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    if (s.n_tiles > 1) {
      stage_affine(n0);
      epi_bar_sync();
    }
    const int row = epi_row();
    const int mt = m0 / kBlockM;
    const int ty = mt / p.tiles_w, tx = mt - ty * p.tiles_w;
    const int y = ty * kConvTileH + row / kConvTileW;
    const int x = tx * kConvTileW + row % kConvTileW;
    const bool ok = y < p.H_out && x < p.W_out;
    const long pix = (static_cast<long>(batch) * p.H_out + y) * p.W_out + x;
    // bilinear source coordinates (PyTorch upsample_bilinear2d, align_corners=True)
    // kUp: u.. are fp16-element offsets of the neighbour pixels inside one staged box, else into the global planes
    long u00 = 0, u01 = 0, u10 = 0, u11 = 0;
    float wy1 = 0.f, wx1 = 0.f;
    if (kUpAny && p.up_hi && ok) {
      const float sh = p.H_out > 1 ? static_cast<float>(p.up_h - 1) / static_cast<float>(p.H_out - 1) : 0.f;
      const float sw = p.W_out > 1 ? static_cast<float>(p.up_w - 1) / static_cast<float>(p.W_out - 1) : 0.f;
      const float fy = sh * y, fx = sw * x;
      const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
      const int y1 = y0 + (y0 < p.up_h - 1 ? 1 : 0), x1 = x0 + (x0 < p.up_w - 1 ? 1 : 0);
      wy1 = fy - y0;
      wx1 = fx - x0;
      if (kUp) {
        int ybase, xbase;
        up_window(ty, tx, ybase, xbase);
        u00 = ((y0 - ybase) * kUpW + (x0 - xbase)) * kUpBoxC;
        u01 = ((y0 - ybase) * kUpW + (x1 - xbase)) * kUpBoxC;
        u10 = ((y1 - ybase) * kUpW + (x0 - xbase)) * kUpBoxC;
        u11 = ((y1 - ybase) * kUpW + (x1 - xbase)) * kUpBoxC;
      } else {
        const long base = static_cast<long>(batch) * p.up_h * p.up_w;
        u00 = (base + static_cast<long>(y0) * p.up_w + x0) * p.up_ld;
        u01 = (base + static_cast<long>(y0) * p.up_w + x1) * p.up_ld;
        u10 = (base + static_cast<long>(y1) * p.up_w + x0) * p.up_ld;
        u11 = (base + static_cast<long>(y1) * p.up_w + x1) * p.up_ld;
      }
    }
    if (kUp) {   // this tile's window has landed
      mbar_wait(up_bar, up_phase);
      up_phase ^= 1u;
    }
    const int c_begin = epi_half() == 0 ? 0 : kChunksHalf0;
    const int c_end = epi_half() == 0 ? kChunksHalf0 : kChunks;
    // launch parameters read once per tile (inside the chunk loop each constant-bank load was an exposed latency)
    const int act = p.act;
    const bool tma_pl = p.out_hi && (p.om.use & 1), tma_f = p.out_f32 && (p.om.use & 2);
#pragma unroll 1
    for (int c = c_begin; c < c_end; ++c) {
      const int col = n0 + c * 32;
      if (col >= s.N) break;
      const int nvalid = min(32, s.N - col);   // warp-uniform
      // residual rows of this 32-channel group: requested before the accumulator is fetched and converted
      const bool res_early = p.res_hi != nullptr && nvalid == 32;
      uint4 rh[4], rl[4];
      if (res_early)
        warp_issue_planes32(ok ? p.res_hi + pix * p.res_ld + col : nullptr, ok ? p.res_lo + pix * p.res_ld + col : nullptr, rh, rl);
      float v[32];
      load_acc32(acc_row, c * 32, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaf(v[j], s_scale[c * 32 + j], s_shift[c * 32 + j]);
      if (nvalid == 32) {
        // full 32-channel group: warp-cooperative (coalesced) loads / stores, pixels outside the image pass nullptr
        if (p.res_hi) {
          if (p.om.use && !kOwnXpose) stage_quiesce();
          float r[32];
          warp_finish_planes32(xscr, rh, rl, r);
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] += r[j];
        }
        if (kUpAny && p.up_hi) {
          // the four bilinear neighbours: plain per-thread loads (two rounds of two neighbours)
          if (ok) {
            // kUp: the staged window (box = column / 128 when the tile spans two boxes), else the global planes
            const __half* uh = p.up_hi + col;
            const __half* ul = p.up_lo + col;
            if (kUp) {
              const int box = kUpBoxes > 1 ? (c * 32) / 128 : 0;
              uh = reinterpret_cast<const __half*>(s_up + box * kUpBoxBytes) + (c * 32 - box * 128);
              ul = reinterpret_cast<const __half*>(s_up + kUpPlaneBytes + box * kUpBoxBytes) + (c * 32 - box * 128);
            }
            float a[32], b[32];
            load_planes32(uh + u00, ul + u00, a);
            load_planes32(uh + u01, ul + u01, b);
            const float wy0 = 1.f - wy1, wx0 = 1.f - wx1;
            float top[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) top[j] = wx0 * a[j] + wx1 * b[j];
            load_planes32(uh + u10, ul + u10, a);
            load_planes32(uh + u11, ul + u11, b);
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += wy0 * top[j] + wy1 * (wx0 * a[j] + wx1 * b[j]);
          }
        }
      } else if (ok) {
        // channel tail (e.g. 196 = 6*32 + 4): scalar path.  Fully unrolled with a predicate: a run-time trip count
        // would index v[] dynamically and push the whole array through local memory (LDL/STL in every chunk)
        const float wy0 = 1.f - wy1, wx0 = 1.f - wx1;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (j >= nvalid) continue;
          if (p.res_hi) {
            const long o = pix * p.res_ld + col + j;
            v[j] += __half2float(p.res_hi[o]) + __half2float(p.res_lo[o]);
          }
          if (kUpAny && p.up_hi) {
            const int box = kUpBoxes > 1 ? (c * 32) / 128 : 0;
            const __half* uh = kUp ? reinterpret_cast<const __half*>(s_up + box * kUpBoxBytes) + (c * 32 - box * 128) : p.up_hi + col;
            const __half* ul = kUp ? reinterpret_cast<const __half*>(s_up + kUpPlaneBytes + box * kUpBoxBytes) + (c * 32 - box * 128)
                                   : p.up_lo + col;
            auto at = [&](long o) { return __half2float(uh[o + j]) + __half2float(ul[o + j]); };
            v[j] += wy0 * (wx0 * at(u00) + wx1 * at(u01)) + wy1 * (wx0 * at(u10) + wx1 * at(u11));
          }
        }
      }
      if (act == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
      } else if (act == 2) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : 0.01f * v[j];
      }
      // the warp's 32 accumulator rows are the 2 x 16 pixel block at (tx*16, ty*8 + 2*quarter); channels / pixels
      // outside the tensor are clipped by the map, so the TMA path also covers the channel tail and image borders
      const OutCoord oc{col, tx * kConvTileW, ty * kConvTileH + ((epi_tid() >> 5) & 3) * 2, batch};
      if (tma_f) warp_tma_store_f32x32(scr, p.om, oc, v);
      if (tma_pl) warp_tma_store_planes32(scr, p.om, oc, v);
      if (nvalid == 32) {
        if (p.out_f32 && !tma_f) warp_store_f32x32(scr, ok ? p.out_f32 + pix * p.f32_ld + col : nullptr, v);
        if (p.out_hi && !tma_pl)
          warp_store_planes32(scr, ok ? p.out_hi + pix * p.out_ld + col : nullptr, ok ? p.out_lo + pix * p.out_ld + col : nullptr, v);
      } else if (ok && !(tma_pl || tma_f)) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (j >= nvalid) continue;
          if (p.out_f32) p.out_f32[pix * p.f32_ld + col + j] = v[j];
          if (p.out_hi) {
            __half hh, ll;
            split_f16(v[j], hh, ll);
            p.out_hi[pix * p.out_ld + col + j] = hh;
            p.out_lo[pix * p.out_ld + col + j] = ll;
          }
        }
      }
    }
    if (s.n_tiles > 1) epi_bar_sync();  // s_scale / s_shift are rewritten by the next tile
  }
};

// ------------------------------------------------------------------------------------------------
// Warp "transpose-reduce": every lane holds v[0..31] (its row's values for 32 columns); afterwards
// lane j holds op over the warp's 32 rows of column j in v[0].  31 shuffles instead of 32*5.
template <class T, class Op>
__device__ __forceinline__ T warp_transpose_reduce(T (&v)[32], Op op) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int step = 16; step >= 1; step >>= 1) {
    const bool up = (lane & step) != 0;
#pragma unroll
    for (int k = 0; k < step; ++k) {
      const T send = up ? v[k] : v[k + step];
      const T keep = up ? v[k + step] : v[k];
      const T recv = __shfl_xor_sync(0xffffffffu, send, step);
      v[k] = op(keep, recv);
    }
  }
  return v[0];
}

struct OpMaxF { __device__ float operator()(float a, float b) const { return fmaxf(a, b); } };
struct OpAddF { __device__ float operator()(float a, float b) const { return a + b; } };
struct OpMaxU64 {
  __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const {
    return a > b ? a : b;
  }
};

// EpiKvProj: epilogue of the k|v projection when K^T V runs on the tensor cores (kv_gemm.cuh).  Column layout of the
// projection (weights permuted on the host, loftr.py): n-tile t = [K of heads 4t..4t+3 (128 columns) | V of the same
// heads (128 columns)].  K = elu(k)+1 and V, both times the padding mask (linear_attention.py:32-39), are written as
// fp16 hi/lo planes (TMA stores) -- the MN-major operands of kv_gemm_kernel.  Rows past the group's end are clipped by
// the store map.
template <int BLOCK_N>
struct EpiKvProj {
  static_assert(BLOCK_N == 256, "built for the coarse transformer (d_model 256, 8 heads)");
  struct Params {
    const uint8_t* rowmask;  // optional [batches*M] (1 = valid)
    float acc_scale;
    OutMaps om;              // planes [batches][M][512]
  };
  static constexpr int kSmemBytes = kEpiScratchBytes;
  const Params& p;
  const GemmShape& s;
  uint32_t* scr;
  __device__ EpiKvProj(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_), scr(epi_scratch(smem)) {}
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  __device__ void prefetch(int, int, int) {}
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    float mk = row_ok ? 1.f : 0.f;
    if (row_ok && p.rowmask) mk = p.rowmask[static_cast<long>(batch) * s.M + r] ? 1.f : 0.f;
    const bool is_k = epi_half() == 0;
    const int quarter = (epi_tid() >> 5) & 3;
    const int c_begin = epi_half() * 4;
#pragma unroll 1
    for (int c = c_begin; c < c_begin + 4; ++c) {
      float x[32];
      load_acc32(acc_row, c * 32, x);
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= p.acc_scale;
      if (is_k) {
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = elu_plus1(x[j]);
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= mk;
      warp_tma_store_planes32(scr, p.om, OutCoord{n0 + c * 32, m0 + quarter * 32, batch, 0}, x);
    }
  }
};

// order-preserving map float -> uint32
__device__ __forceinline__ uint32_t f32_ordered(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_unordered(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// ------------------------------------------------------------------------------------------------
// Pass 1 of the fused coarse matching: z = acc * scale is one 128 x BLOCK_N tile of the similarity
// matrix (reference coarse_matching.py:109-110 / 122).  Emits log-sum-exp partials
//   rows:    (max, sum) over this work item's columns of  z[i,j] + colterm[j]
//   columns: (max, sum) over this tile's 128 rows of      z[i,j] + rowterm[i]
// without ever storing z.  With colterm = rowterm = 0 these are the two softmax normalisers of the
// dual-softmax (coarse_matching.py:119); with the Sinkhorn potentials they are one half-iteration of
// log_sinkhorn_iterations (third_party superglue.py:141-148).  Masked / out-of-range entries carry
// the term kNegBig and therefore vanish from every sum (coarse_matching.py:115-118 fills -1e9).
template <int BLOCK_N, bool kRows, bool kCols>
struct EpiScoreLse {
  struct Params {
    float scale;
    const float* colterm;   // optional [batches*N]; nullptr -> 0
    const float* rowterm;   // optional [batches*M]
    float2* row_part;       // [n_chunks][batches*M]
    float2* col_part;       // [m_tiles][batches*N]
  };
  // colterm staging + per-warp-row-quarter column partials + per-warp column-max broadcast + row merge
  static constexpr int kSmemBytes = BLOCK_N * 4 + 4 * BLOCK_N * 8 + 8 * 32 * 4 + 128 * 8;
  const Params& p;
  const GemmShape& s;
  float* s_ct;       // [BLOCK_N]
  float2* s_cpart;   // [4][BLOCK_N]
  float* s_cmax;     // [8][32]
  float2* s_rmerge;  // [128]
  float row_m, row_l;

  __device__ EpiScoreLse(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_) {
    s_ct = reinterpret_cast<float*>(smem);
    s_cpart = reinterpret_cast<float2*>(smem + BLOCK_N * 4);
    s_cmax = reinterpret_cast<float*>(smem + BLOCK_N * 4 + 4 * BLOCK_N * 8);
    s_rmerge = reinterpret_cast<float2*>(smem + BLOCK_N * 4 + 4 * BLOCK_N * 8 + 8 * 32 * 4);
  }
  __device__ void prefetch(int, int, int) {}
  __device__ void item_begin(int, int, int) {
    row_m = kNegBig;
    row_l = 0.f;
  }
  __device__ void item_end(int batch, int m0, int chunk) {
    if (kRows) {
      // merge the two column halves of each row, then one thread per row writes the partial
      const int row = epi_row();
      if (epi_half() == 1) s_rmerge[row] = make_float2(row_m, row_l);
      epi_bar_sync();
      if (epi_half() == 0) {
        const float2 o = s_rmerge[row];
        const float m = fmaxf(row_m, o.x);
        const float l = row_l * exp_fast(row_m - m) + o.y * exp_fast(o.x - m);
        const int r = m0 + row;
        if (r < s.M) {
          p.row_part[static_cast<long>(chunk) * s.batches * s.M + static_cast<long>(batch) * s.M + r] =
              make_float2(m, l);
        }
      }
      epi_bar_sync();
    }
  }
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    const int t = epi_tid();
    const int w = t >> 5;        // 0..7
    const int q = w & 3;         // row quarter
    const int lane = t & 31;
    const int r = m0 + epi_row();
    // stage column terms of this tile
    for (int j = t; j < BLOCK_N; j += kEpiThreads) {
      const int col = n0 + j;
      float ct = kNegBig;
      if (col < s.N) ct = p.colterm ? p.colterm[static_cast<long>(batch) * s.N + col] : 0.f;
      s_ct[j] = ct;
    }
    float rt = kNegBig;
    if (r < s.M) rt = p.rowterm ? p.rowterm[static_cast<long>(batch) * s.M + r] : 0.f;
    epi_bar_sync();

    const int c_begin = epi_half() * (BLOCK_N / 64);
    // Fast path (dual-softmax without padding masks): rows and columns share ONE exponential per element,
    // e = exp(z - g) with g the maximum of the warp's 32 x 32 block; a (g, sum) pair is a valid partial for both
    // directions.  If any row or column of the block sits more than ~69 nats below g (its sum would lose
    // significant terms to fp32 underflow) the whole block falls back to the per-row / per-column references.
    const bool shared_ref = kRows && kCols && p.colterm == nullptr && p.rowterm == nullptr;
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      if (n0 + c * 32 >= s.N) break;
      float z[32];
      load_acc32(acc_row, c * 32, z);
#pragma unroll
      for (int j = 0; j < 32; ++j) z[j] *= p.scale;

      if (kRows && kCols && shared_ref && n0 + c * 32 + 32 <= s.N) {   // warp-uniform condition
        const bool row_valid = r < s.M;
        float cm = kNegBig;
#pragma unroll
        for (int j = 0; j < 32; ++j) cm = fmaxf(cm, z[j]);
        if (!row_valid) cm = kNegBig;
        float g = cm;
#pragma unroll
        for (int o = 16; o; o >>= 1) g = fmaxf(g, __shfl_xor_sync(0xffffffffu, g, o));
        float v[32];
        float rs = 0.f;
        const float gl = g * kLog2e;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          v[j] = row_valid ? ex2_approx(fmaf(z[j], kLog2e, -gl)) : 0.f;
          rs += v[j];
        }
        const float csum = warp_transpose_reduce(v, OpAddF());   // lane j: sum over the block's rows of column j
        const bool fine = (rs >= 1e-30f || !row_valid) && (csum >= 1e-30f);
        if (__all_sync(0xffffffffu, fine)) {
          const float m_new = fmaxf(row_m, g);
          row_l = row_l * exp_fast(row_m - m_new) + rs * exp_fast(g - m_new);
          row_m = m_new;
          s_cpart[q * BLOCK_N + c * 32 + lane] = make_float2(g, csum);
          continue;
        }
      }

      if (kRows) {
        float cm = kNegBig;
#pragma unroll
        for (int j = 0; j < 32; ++j) cm = fmaxf(cm, z[j] + s_ct[c * 32 + j]);
        const float m_new = fmaxf(row_m, cm);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) acc += exp_fast(z[j] + s_ct[c * 32 + j] - m_new);
        row_l = row_l * exp_fast(row_m - m_new) + acc;
        row_m = m_new;
      }
      if (kCols) {
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          z[j] += rt;
          v[j] = z[j];
        }
        const float cmax = warp_transpose_reduce(v, OpMaxF());  // lane j: max of column c*32+j
        s_cmax[w * 32 + lane] = cmax;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = exp_fast(z[j] - s_cmax[w * 32 + j]);
        __syncwarp();
        const float csum = warp_transpose_reduce(v, OpAddF());
        s_cpart[q * BLOCK_N + c * 32 + lane] = make_float2(cmax, csum);
      }
    }
    if (kCols) {
      epi_bar_sync();
      // merge the four 32-row partials of each column and emit the 128-row partial
      for (int j = t; j < BLOCK_N; j += kEpiThreads) {
        const int col = n0 + j;
        if (col < s.N) {
          float m = kNegBig;
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) m = fmaxf(m, s_cpart[qq * BLOCK_N + j].x);
          float l = 0.f;
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) {
            const float2 pq = s_cpart[qq * BLOCK_N + j];
            l += pq.y * exp_fast(pq.x - m);
          }
          p.col_part[static_cast<long>(m0 / kBlockM) * s.batches * s.N + static_cast<long>(batch) * s.N + col] =
              make_float2(m, l);
        }
      }
    }
    epi_bar_sync();  // s_ct / s_cpart are reused by the next tile
  }
};

// ------------------------------------------------------------------------------------------------
// Optional materialisation of the confidence matrix (reference `data['conf_matrix']`, coarse_matching.py:145;
// its only consumer is the training loss, so the engine writes it on request only):
//   conf[i,j] = exp(alpha*z[i,j] + rowterm[i] + colterm[j] + bias), 0 where a term is disabled (padded /
//   prefiltered rows and columns).  HBM-bound: 4*L*S bytes per pair.
template <int BLOCK_N>
struct EpiConfStore {
  struct Params {
    float scale, alpha, bias;
    const float* rowterm;  // [batches*M]
    const float* colterm;  // [batches*N]
    float* out;            // [batches, M, N]
  };
  static constexpr int kSmemBytes = BLOCK_N * 4;
  const Params& p;
  const GemmShape& s;
  float* s_ct;
  __device__ EpiConfStore(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_) {
    s_ct = reinterpret_cast<float*>(smem);
  }
  __device__ void item_begin(int, int, int) {}
  __device__ void item_end(int, int, int) {}
  __device__ void prefetch(int, int, int) {}
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    const int t = epi_tid();
    for (int j = t; j < BLOCK_N; j += kEpiThreads) {
      const int col = n0 + j;
      s_ct[j] = (col < s.N) ? p.colterm[static_cast<long>(batch) * s.N + col] : kNegBig;
    }
    const int r = m0 + epi_row();
    const bool row_ok = r < s.M;
    const float rt = row_ok ? p.rowterm[static_cast<long>(batch) * s.M + r] : kNegBig;
    const float sa = p.scale * p.alpha;
    epi_bar_sync();
    float* orow = p.out + (static_cast<long>(batch) * s.M + r) * s.N;
    const int c_begin = epi_half() * (BLOCK_N / 64);
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      const int col = n0 + c * 32;
      if (col >= s.N) break;
      float z[32];
      load_acc32(acc_row, c * 32, z);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float ct = s_ct[c * 32 + j];
        z[j] = (rt > -1.0e29f && ct > -1.0e29f) ? expf(z[j] * sa + rt + ct + p.bias) : 0.f;
      }
      if (row_ok) {
        if (col + 32 <= s.N && (s.N & 3) == 0) {
          store_f32x32(orow + col, z);
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (col + j < s.N) orow[col + j] = z[j];   // predicated, not a run-time trip count: z[] stays in registers
        }
      }
    }
    epi_bar_sync();
  }
};

// ------------------------------------------------------------------------------------------------
// Pass 2: recompute the tile and take arg-maxima of the confidence along both directions.
//   row key  = alpha*z[i,j] + colterm[j]   (arg max over j: nearest neighbour of row i)
//   col key  = alpha*z[i,j] + rowterm[i]   (arg max over i: nearest neighbour of column j)
// dual-softmax: alpha=2, colterm=-colLSE, rowterm=-rowLSE (log conf = 2z - rowLSE_i - colLSE_j,
// monotone in the key along each direction); Sinkhorn: alpha=1, terms = potentials v, u.
// Replaces conf.max(dim=2) / conf.max(dim=1) of the mutual-nearest test (coarse_matching.py:187-189).
struct ArgPart {
  float key;
  int idx;
};
template <int BLOCK_N>
struct EpiScoreArgmax {
  struct Params {
    float scale;
    float alpha;
    const float* colterm;  // [batches*N] (kNegBig disables a column)
    const float* rowterm;  // [batches*M]
    ArgPart* row_part;     // [n_chunks][batches*M]
    ArgPart* col_part;     // [m_tiles][batches*N]
  };
  static constexpr int kSmemBytes = BLOCK_N * 4 + 4 * BLOCK_N * 8 + 128 * 8;
  const Params& p;
  const GemmShape& s;
  float* s_ct;
  unsigned long long* s_cpart;  // [4][BLOCK_N]
  ArgPart* s_rmerge;            // [128]
  float best_key;
  int best_j;

  __device__ EpiScoreArgmax(const Params& p_, uint8_t* smem, const GemmShape& s_) : p(p_), s(s_) {
    s_ct = reinterpret_cast<float*>(smem);
    s_cpart = reinterpret_cast<unsigned long long*>(smem + BLOCK_N * 4);
    s_rmerge = reinterpret_cast<ArgPart*>(smem + BLOCK_N * 4 + 4 * BLOCK_N * 8);
  }
  __device__ void prefetch(int, int, int) {}
  __device__ void item_begin(int, int, int) {
    best_key = -3.0e38f;
    best_j = -1;
  }
  __device__ void item_end(int batch, int m0, int chunk) {
    const int row = epi_row();
    if (epi_half() == 1) {
      ArgPart a;
      a.key = best_key;
      a.idx = best_j;
      s_rmerge[row] = a;
    }
    epi_bar_sync();
    if (epi_half() == 0) {
      ArgPart a;
      a.key = best_key;
      a.idx = best_j;
      const ArgPart o = s_rmerge[row];      // right half = larger column indices: strict '>' keeps the first
      if (o.key > a.key) a = o;
      const int r = m0 + row;
      if (r < s.M) p.row_part[static_cast<long>(chunk) * s.batches * s.M + static_cast<long>(batch) * s.M + r] = a;
    }
    epi_bar_sync();
  }
  __device__ void tile(uint32_t acc_row, int batch, int m0, int n0) {
    const int t = epi_tid();
    const int q = (t >> 5) & 3;
    const int lane = t & 31;
    const int r = m0 + epi_row();
    for (int j = t; j < BLOCK_N; j += kEpiThreads) {
      const int col = n0 + j;
      s_ct[j] = (col < s.N) ? p.colterm[static_cast<long>(batch) * s.N + col] : kNegBig;
    }
    const float rt = (r < s.M) ? p.rowterm[static_cast<long>(batch) * s.M + r] : kNegBig;
    const float sa = p.scale * p.alpha;
    epi_bar_sync();

    const int c_begin = epi_half() * (BLOCK_N / 64);
#pragma unroll 1
    for (int c = c_begin; c < c_begin + BLOCK_N / 64; ++c) {
      if (n0 + c * 32 >= s.N) break;
      float z[32];
      load_acc32(acc_row, c * 32, z);
#pragma unroll
      for (int j = 0; j < 32; ++j) z[j] *= sa;
      // row direction: thread-local, strict '>' keeps the first (smallest j) maximum
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float key = z[j] + s_ct[c * 32 + j];
        if (key > best_key) {
          best_key = key;
          best_j = n0 + c * 32 + j;
        }
      }
      // column direction: arg max over the warp's 32 rows; ties -> smallest row
      unsigned long long v[32];
      const unsigned long long tag = 0xFFFFFFFFull - static_cast<unsigned long long>(static_cast<uint32_t>(r));
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] = (static_cast<unsigned long long>(f32_ordered(z[j] + rt)) << 32) | tag;
      }
      const unsigned long long best = warp_transpose_reduce(v, OpMaxU64());
      s_cpart[q * BLOCK_N + c * 32 + lane] = best;
    }
    epi_bar_sync();
    for (int j = t; j < BLOCK_N; j += kEpiThreads) {
      const int col = n0 + j;
      if (col < s.N) {
        unsigned long long b = s_cpart[j];
#pragma unroll
        for (int qq = 1; qq < 4; ++qq) {
          const unsigned long long o = s_cpart[qq * BLOCK_N + j];
          b = o > b ? o : b;
        }
        ArgPart a;
        a.key = f32_unordered(static_cast<uint32_t>(b >> 32));
        a.idx = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(b & 0xFFFFFFFFull));
        p.col_part[static_cast<long>(m0 / kBlockM) * s.batches * s.N + static_cast<long>(batch) * s.N + col] = a;
      }
    }
    epi_bar_sync();
  }
};

}  // namespace lb
