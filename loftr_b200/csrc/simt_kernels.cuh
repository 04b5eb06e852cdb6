// Small CUDA-core kernels of the matching hot path: operand preparation, the linear-attention
// core (KV = K^T V is only H x D x D floats per image), partial merges, match selection and the fine
// level.  They are bandwidth / latency bound; the dense work lives in gemm_split.cuh.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>
#include "epilogues.cuh"

namespace lb {

// Programmatic dependent launch: lets a tensor-core kernel that follows on the stream (launched with the PDL attribute,
// gemm_split.cuh) be scheduled and run its set-up while this grid is still working; it waits for this grid's completion
// before it touches global memory.  A no-op when the next launch is an ordinary one.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// fp32 [rows, cols] (ld_x) -> fp16 hi/lo planes (ld_pl, column offset col0).  Weight packing and tests.
__global__ void split_planes_kernel(const float* __restrict__ x, long rows, int cols, int ld_x,
                                    __half* __restrict__ hi, __half* __restrict__ lo, int ld_pl, int col0) {
  const long total = rows * cols;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / cols;
    const int c = static_cast<int>(i - r * cols);
    __half h, l;
    split_f16(x[r * ld_x + c], h, l);
    hi[r * ld_pl + col0 + c] = h;
    lo[r * ld_pl + col0 + c] = l;
  }
}

// ------------------------------------------------------------------------------------------------
// Coarse prologue: feat_c (backbone output, NCHW [n_img, C, h, w] or NHWC [n_img, h, w, C]) + pe[C, pe_h, pe_w]
// -> token-major x_f32 [n_img*h*w, C] and fp16 planes in columns [0, C) of the [rows, 2C] cat buffer.
// = PositionEncodingSine.forward + rearrange 'n c h w -> n (h w) c' (reference loftr.py:58-59,
// position_encoding.py:37-42).  32x32 smem transpose so both sides are coalesced.
__global__ void coarse_prep_kernel(const float* __restrict__ feat, int nhwc, const float* __restrict__ pe, int C,
                                   int h, int w, int pe_h, int pe_w, float* __restrict__ x_f32,
                                   __half* __restrict__ cat_hi, __half* __restrict__ cat_lo) {
  pdl_trigger();
  __shared__ float tile[32][33];
  const int L = h * w;
  const int img = blockIdx.z;
  const int l0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  // read: threadIdx.x along l (contiguous in the channel-major sources), threadIdx.y along c
  for (int cy = threadIdx.y; cy < 32; cy += blockDim.y) {
    const int c = c0 + cy;
    const int l = l0 + threadIdx.x;
    float v = 0.f;
    if (c < C && l < L) {
      const int y = l / w, x = l - y * w;
      v = pe[(static_cast<long>(c) * pe_h + y) * pe_w + x];
      if (!nhwc) v += feat[(static_cast<long>(img) * C + c) * L + l];
    }
    tile[cy][threadIdx.x] = v;
  }
  __syncthreads();
  // write: threadIdx.x along c (contiguous in NLC)
  for (int ly = threadIdx.y; ly < 32; ly += blockDim.y) {
    const int l = l0 + ly;
    const int c = c0 + threadIdx.x;
    if (c < C && l < L) {
      const long row = static_cast<long>(img) * L + l;
      float v = tile[threadIdx.x][ly];
      if (nhwc) v = feat[row * C + c] + v;
      x_f32[row * C + c] = v;
      __half hh, ll;
      split_f16(v, hh, ll);
      cat_hi[row * (2 * C) + c] = hh;
      cat_lo[row * (2 * C) + c] = ll;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Linear attention, source side (reference linear_attention.py:43-44):
//   KV[g,h,d,v] = sum_s K[s,h,d] * V[s,h,v],   Ksum[g,h,d] = sum_s K[s,h,d]
// over the rows s of group g.  K = elu+1 and the padding mask were already applied by the projection epilogue.  The
// reference's V/S ... *S rescale is an fp16-overflow guard and a mathematical no-op in fp32 (SURVEY.md §9 V3), so it is
// not reproduced.  Atomics-free so the result is bit-reproducible.

// Sum of the per-split partials written by kv_gemm_kernel (coarse level): part [groups][nparts][H*per] ->
// kv [groups][H*per] (fixed order over the splits: bit-reproducible).
__global__ void kv_tile_merge_kernel(const float* __restrict__ part, int nparts, int hper, float* __restrict__ kv,
                                     long total) {
  pdl_trigger();
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  const long g = i / hper;
  const int e = static_cast<int>(i - g * hper);
  const float* src = part + g * nparts * hper + e;
  float acc = 0.f;
  for (int k = 0; k < nparts; ++k) acc += src[static_cast<long>(k) * hper];
  kv[i] = acc;
}

// Window variant for the fine transformer (group = one window of at most 32 rows, D = 16, H = 8): one block per
// window, all heads; writes kv directly.  Only the cross pass between windows of different sizes uses it (with
// attn_apply_kernel<16, 8>); equal windows run window_attn_kernel.
template <int D, int H>
__global__ void __launch_bounds__(256) kv_window_kernel(const float* __restrict__ qkv, int ld, int k_col0,
                                                        int v_col0, long row_base, int rows_per_group,
                                                        float* __restrict__ kv) {
  static_assert(D == 16 && H == 8, "fine head layout");
  constexpr int C = D * H;  // 128
  constexpr int MAXR = 32;
  __shared__ __align__(16) float sK[MAXR][C];
  __shared__ __align__(16) float sV[MAXR][C];
  const int g = blockIdx.x;
  const int tid = threadIdx.x;
  for (int i = tid; i < rows_per_group * (C / 4); i += 256) {
    const int s = i / (C / 4), c4 = (i % (C / 4)) * 4;
    const float* rowp = qkv + (row_base + static_cast<long>(g) * rows_per_group + s) * ld;
    *reinterpret_cast<float4*>(&sK[s][c4]) = *reinterpret_cast<const float4*>(rowp + k_col0 + c4);
    *reinterpret_cast<float4*>(&sV[s][c4]) = *reinterpret_cast<const float4*>(rowp + v_col0 + c4);
  }
  __syncthreads();
  const int hd = tid >> 5;          // 0..7
  const int d = (tid & 31) >> 1;    // 0..15
  const int v0 = (tid & 1) * 8;     // 0 or 8
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  float ks = 0.f;
  for (int s = 0; s < rows_per_group; ++s) {
    const float k = sK[s][hd * D + d];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(k, sV[s][hd * D + v0 + j], acc[j]);
    ks += k;
  }
  float* out = kv + (static_cast<long>(g) * H + hd) * (D * D + D);
#pragma unroll
  for (int j = 0; j < 8; ++j) out[d * D + v0 + j] = acc[j];
  if ((tid & 1) == 0) out[D * D + d] = ks;
}

// ------------------------------------------------------------------------------------------------
// Linear attention, query side (reference linear_attention.py:45-46):
//   out[r,h,:] = (Q[r,h,:] . KV[g,h]) / (Q[r,h,:] . Ksum[g,h] + eps)
// written as fp16 planes = the A operand of the merge projection.  One warp per head, lanes = rows.
template <int D, int H>
__global__ void __launch_bounds__(32 * H) attn_apply_kernel(const float* __restrict__ qkv, int ld, int q_col0,
                                                            long x_row_base, int rows_per_group,
                                                            int rows_per_block, const float* __restrict__ kv,
                                                            float eps, __half* __restrict__ att_hi,
                                                            __half* __restrict__ att_lo, int ld_att) {
  constexpr int PER = D * D + D;
  __shared__ __align__(16) float sKV[H][PER];
  const int g = blockIdx.x;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = min(r_begin + rows_per_block, rows_per_group);
  const int hd = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  {
    const float* src = kv + static_cast<long>(g) * H * PER;
    float* dst = &sKV[0][0];
    for (int i = threadIdx.x; i < H * PER; i += 32 * H) dst[i] = src[i];
  }
  __syncthreads();
  const float* kvh = sKV[hd];
  for (int r0 = r_begin; r0 < r_end; r0 += 32) {
    const int r = r0 + lane;
    if (r < r_end) {
      const long row = x_row_base + static_cast<long>(g) * rows_per_group + r;
      float q[D];
      const float4* qp = reinterpret_cast<const float4*>(qkv + row * ld + q_col0 + hd * D);
#pragma unroll
      for (int j = 0; j < D / 4; ++j) {
        const float4 t = qp[j];
        q[4 * j] = t.x; q[4 * j + 1] = t.y; q[4 * j + 2] = t.z; q[4 * j + 3] = t.w;
      }
      float zden = eps;
#pragma unroll
      for (int d = 0; d < D; ++d) zden = fmaf(q[d], kvh[D * D + d], zden);
      const float z = 1.f / zden;
      __half* hp = att_hi + row * ld_att + hd * D;
      __half* lp = att_lo + row * ld_att + hd * D;
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
        *reinterpret_cast<uint4*>(hp + v8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(lp + v8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fine (window) linear attention in ONE kernel: kv_window_kernel + attn_apply_kernel<16, 8> back to back per window
// (reference linear_attention.py:43-46 on the [M, 25, 128] window sequences of fine_preprocess.py).  One block takes
// windows g, g + gridDim.x, ...; KV[h] = K_h^T V_h and Ksum_h are built in shared memory (never in HBM) and warp h /
// lane r applies them to query row r.  The kernel is latency-bound on the q/k/v reads (ncu: 34 % of the samples wait
// on them), so the NEXT window's K / V rows travel global -> shared with cp.async into the other half of a double
// buffer and its query row into registers while the current window is computed.  Same summation order as the
// two-kernel path: bit-identical output.  Dynamic shared memory: 2 x 2 x rows x 512 B + 8.7 KB (60 KB for 25 rows).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int D, int H>
__global__ void __launch_bounds__(32 * H, 3) window_attn_kernel(const float* __restrict__ qkv, int ld, int q_col0, int k_col0,
                                                                int v_col0, long x_row_base, long s_row_base,
                                                                int rows_per_group, int n_groups, float eps,
                                                                __half* __restrict__ att_hi, __half* __restrict__ att_lo,
                                                                int ld_att, const int* __restrict__ live, int live_cap) {
  pdl_trigger();
  static_assert(D == 16 && H == 8, "fine head layout");
  constexpr int C = D * H;  // 128
  constexpr int PER = D * D + D;
  extern __shared__ __align__(16) float wa_smem[];
  float* sKV = wa_smem;                                   // [H][PER]
  float* sKVbuf = wa_smem + H * PER;                      // [2][K | V][rows][C]
  const int buf_floats = 2 * rows_per_group * C;
  const int tid = threadIdx.x;
  const int hd = tid >> 5, lane = tid & 31;
  const bool has_row = lane < rows_per_group;

  auto issue = [&](int g, int b) {   // K / V rows of window g -> buffer b
    float* dK = sKVbuf + b * buf_floats;
    float* dV = dK + rows_per_group * C;
    for (int i = tid; i < rows_per_group * (C / 4); i += 32 * H) {
      const int r = i / (C / 4), c4 = (i % (C / 4)) * 4;
      const float* rowp = qkv + (s_row_base + static_cast<long>(g) * rows_per_group + r) * ld;
      cp_async16(dK + r * C + c4, rowp + k_col0 + c4);
      cp_async16(dV + r * C + c4, rowp + v_col0 + c4);
    }
  };
  auto load_q = [&](int g, float (&q)[D]) {
    const float4* qp = reinterpret_cast<const float4*>(
        qkv + (x_row_base + static_cast<long>(g) * rows_per_group + lane) * ld + q_col0 + hd * D);
#pragma unroll
    for (int j = 0; j < D / 4; ++j) {
      const float4 t = qp[j];
      q[4 * j] = t.x; q[4 * j + 1] = t.y; q[4 * j + 2] = t.z; q[4 * j + 3] = t.w;
    }
  };

  // Optional device bound (`live` != nullptr): the groups are sets of live_cap windows of which only the first
  // min(*live, live_cap) are filled, i.e. groups [0, n) U [cap, cap + n) U ...  Work item v maps to group
  // (v / n_live) * cap + v % n_live (the identity without a bound).
  int n_items = n_groups, n_live = n_groups, cap = n_groups;
  if (live != nullptr) {
    cap = live_cap;
    n_live = min(max(*live, 0), live_cap);
    n_items = n_live * (n_groups / live_cap);
  }
  auto group_of = [&](int v) { return v / n_live * cap + v % n_live; };

  float q[D], qn[D];
#pragma unroll
  for (int j = 0; j < D; ++j) q[j] = qn[j] = 0.f;
  int v = blockIdx.x;
  if (v < n_items) {
    issue(group_of(v), 0);
    if (has_row) load_q(group_of(v), q);
  }
  cp_async_commit();
  int b = 0;
  for (; v < n_items; v += gridDim.x, b ^= 1) {
    const int g = group_of(v);
    const int vn = v + gridDim.x;
    if (vn < n_items) {
      const int gn = group_of(vn);
      issue(gn, b ^ 1);
      if (has_row) load_q(gn, qn);
    }
    cp_async_commit();
    cp_async_wait<1>();      // this thread's copies of window g have landed ...
    __syncthreads();         // ... and everybody else's
    const float* sK = sKVbuf + b * buf_floats;
    const float* sV = sK + rows_per_group * C;
    // KV[hd][d][v0..v0+7] and Ksum[hd][d] over the window's rows
    {
      const int d = lane >> 1, v0 = (lane & 1) * 8;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      float ks = 0.f;
      for (int r = 0; r < rows_per_group; ++r) {
        const float k = sK[r * C + hd * D + d];
        const float4 a = *reinterpret_cast<const float4*>(&sV[r * C + hd * D + v0]);
        const float4 c = *reinterpret_cast<const float4*>(&sV[r * C + hd * D + v0 + 4]);
        acc[0] = fmaf(k, a.x, acc[0]); acc[1] = fmaf(k, a.y, acc[1]); acc[2] = fmaf(k, a.z, acc[2]); acc[3] = fmaf(k, a.w, acc[3]);
        acc[4] = fmaf(k, c.x, acc[4]); acc[5] = fmaf(k, c.y, acc[5]); acc[6] = fmaf(k, c.z, acc[6]); acc[7] = fmaf(k, c.w, acc[7]);
        ks += k;
      }
      float* out = sKV + hd * PER + d * D + v0;
      *reinterpret_cast<float4*>(out) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      *reinterpret_cast<float4*>(out + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
      if ((lane & 1) == 0) sKV[hd * PER + D * D + d] = ks;
    }
    __syncwarp();   // KV of head hd is produced and consumed by warp hd only
    // message row = (q . KV) / (q . Ksum + eps) -> fp16 planes
    if (has_row) {
      const float* kvh = sKV + hd * PER;
      const long xrow = x_row_base + static_cast<long>(g) * rows_per_group + lane;
      float zden = eps;
#pragma unroll
      for (int d = 0; d < D; ++d) zden = fmaf(q[d], kvh[D * D + d], zden);
      const float z = 1.f / zden;
      __half* hp = att_hi + xrow * ld_att + hd * D;
      __half* lp = att_lo + xrow * ld_att + hd * D;
#pragma unroll
      for (int v8 = 0; v8 < D; v8 += 8) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const float4 a = *reinterpret_cast<const float4*>(&kvh[d * D + v8]);
          const float4 c = *reinterpret_cast<const float4*>(&kvh[d * D + v8 + 4]);
          o[0] = fmaf(q[d], a.x, o[0]); o[1] = fmaf(q[d], a.y, o[1]);
          o[2] = fmaf(q[d], a.z, o[2]); o[3] = fmaf(q[d], a.w, o[3]);
          o[4] = fmaf(q[d], c.x, o[4]); o[5] = fmaf(q[d], c.y, o[5]);
          o[6] = fmaf(q[d], c.z, o[6]); o[7] = fmaf(q[d], c.w, o[7]);
        }
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split_f16x2(o[2 * j] * z, o[2 * j + 1] * z, hw[j], lw[j]);
        *reinterpret_cast<uint4*>(hp + v8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(lp + v8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      }
    }
#pragma unroll
    for (int j = 0; j < D; ++j) q[j] = qn[j];
    __syncthreads();   // buffer b is refilled by the next iteration's copies
  }
  cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// Fine (window) full attention: message = softmax(q k^T / sqrt(D)) v over the rows of one window per head (reference
// linear_attention.py:56-81 on the [M, 25, 128] window sequences), exact fp32 on the CUDA cores.  One block takes
// windows g, g + gridDim.x, ...; the window's K / V rows are staged in shared memory and warp h / lane r computes
// query row r of head h: scores, max, exponentials, sum and the weighted V rows in a fixed order (deterministic).
// Keys with mask 0 get weight 0; padded query rows and rows without a valid key write 0.  Same device bound as
// window_attn_kernel: with `live`, only windows [0, min(*live, live_cap)) of every set of live_cap are visited.
template <int D, int H, int MAXR>
__global__ void __launch_bounds__(32 * H) window_full_attn_kernel(const float* __restrict__ qkv, int ld, int q_col0,
                                                                  int k_col0, int v_col0, long x_row_base,
                                                                  long s_row_base, int rows_per_group, int n_groups,
                                                                  const uint8_t* __restrict__ mask,
                                                                  __half* __restrict__ att_hi,
                                                                  __half* __restrict__ att_lo, int ld_att,
                                                                  const int* __restrict__ live, int live_cap) {
  pdl_trigger();
  static_assert(D % 8 == 0 && MAXR <= 32, "window head layout");
  constexpr int C = D * H;
  __shared__ __align__(16) float sK[MAXR * C];
  __shared__ __align__(16) float sV[MAXR * C];
  __shared__ float sBias[MAXR];
  const int tid = threadIdx.x;
  const int hd = tid >> 5, lane = tid & 31;
  const bool has_row = lane < rows_per_group;
  const float scale = rsqrtf(static_cast<float>(D));

  int n_items = n_groups, n_live = n_groups, cap = n_groups;
  if (live != nullptr) {
    cap = live_cap;
    n_live = min(max(*live, 0), live_cap);
    n_items = n_live * (n_groups / live_cap);
  }
  for (int v = blockIdx.x; v < n_items; v += gridDim.x) {
    const int g = v / n_live * cap + v % n_live;
    const long srow = s_row_base + static_cast<long>(g) * rows_per_group;
    const long xrow = x_row_base + static_cast<long>(g) * rows_per_group + lane;
    for (int i = tid; i < rows_per_group * (C / 4); i += 32 * H) {
      const int r = i / (C / 4), c4 = (i % (C / 4)) * 4;
      const float* rowp = qkv + (srow + r) * ld;
      *reinterpret_cast<float4*>(sK + r * C + c4) = *reinterpret_cast<const float4*>(rowp + k_col0 + c4);
      *reinterpret_cast<float4*>(sV + r * C + c4) = *reinterpret_cast<const float4*>(rowp + v_col0 + c4);
    }
    if (tid < rows_per_group) sBias[tid] = (mask == nullptr || mask[srow + tid] != 0) ? 0.f : -INFINITY;
    float q[D];
    if (has_row) {
      const float4* qp = reinterpret_cast<const float4*>(qkv + xrow * ld + q_col0 + hd * D);
#pragma unroll
      for (int j = 0; j < D / 4; ++j) {
        const float4 t = qp[j];
        q[4 * j] = t.x; q[4 * j + 1] = t.y; q[4 * j + 2] = t.z; q[4 * j + 3] = t.w;
      }
    }
    __syncthreads();
    if (has_row) {
      float s[MAXR];
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < MAXR; ++j) {
        s[j] = -INFINITY;
        if (j < rows_per_group) {
          const float* kr = sK + j * C + hd * D;
          float a = 0.f;
#pragma unroll
          for (int d = 0; d < D; ++d) a = fmaf(q[d], kr[d], a);
          s[j] = a * scale + sBias[j];
          m = fmaxf(m, s[j]);
        }
      }
      float o[D];
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] = 0.f;
      float sum = 0.f;
      if (m != -INFINITY) {
#pragma unroll
        for (int j = 0; j < MAXR; ++j) {
          if (j < rows_per_group) {
            const float pj = expf(s[j] - m);
            sum += pj;
            const float* vr = sV + j * C + hd * D;
#pragma unroll
            for (int d = 0; d < D; ++d) o[d] = fmaf(pj, vr[d], o[d]);
          }
        }
      }
      const bool q_ok = mask == nullptr || mask[xrow] != 0;
      const float inv = (q_ok && sum > 0.f) ? 1.f / sum : 0.f;
      __half* hp = att_hi + xrow * ld_att + hd * D;
      __half* lp = att_lo + xrow * ld_att + hd * D;
#pragma unroll
      for (int v8 = 0; v8 < D; v8 += 8) {
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split_f16x2(o[v8 + 2 * j] * inv, o[v8 + 2 * j + 1] * inv, hw[j], lw[j]);
        *reinterpret_cast<uint4*>(hp + v8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(lp + v8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      }
    }
    __syncthreads();   // the K / V rows are overwritten by the next window
  }
}

// ------------------------------------------------------------------------------------------------
// Merge log-sum-exp partials: out[i] = base - LSE(parts[:, i] U {dustbin term}).
//   dual-softmax:  base = 0, no dustbin   -> out = -LSE (the additive log-normaliser)
//   Sinkhorn:      base = log_mu / log_nu, dustbin term = bin + bin_pot[pair]   (superglue.py:146-147)
// `valid` (optional) marks padded rows / columns: their real entries are -1e9 in the reference
// (coarse_matching.py:115-118,124-127), i.e. only the dustbin term survives (or nothing: kNegBig).
__global__ void lse_merge_kernel(const float2* __restrict__ part, int nparts, long count, float base,
                                 const float* __restrict__ bin, const float* __restrict__ bin_pot, int per,
                                 const uint8_t* __restrict__ valid, float* __restrict__ out) {
  pdl_trigger();
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  const bool use_extra = bin != nullptr;
  float e = 0.f;
  if (use_extra) e = *bin + (bin_pot ? bin_pot[i / per] : 0.f);
  if (valid && !valid[i]) {
    out[i] = use_extra ? base - e : kNegBig;
    return;
  }
  float m = kNegBig;
  for (int k = 0; k < nparts; ++k) m = fmaxf(m, part[k * count + i].x);
  if (use_extra) m = fmaxf(m, e);
  float l = 0.f;
  for (int k = 0; k < nparts; ++k) {
    const float2 p = part[k * count + i];
    l += p.y * expf(p.x - m);
  }
  if (use_extra) l += expf(e - m);
  out[i] = base - (m + logf(l));
}

// Arg-max partial merge; partials are ordered by increasing index range, strict '>' keeps the first.
__global__ void argmax_merge_kernel(const ArgPart* __restrict__ part, int nparts, long count,
                                    float* __restrict__ key, int* __restrict__ idx) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  ArgPart b = part[i];
  for (int k = 1; k < nparts; ++k) {
    const ArgPart o = part[k * count + i];
    if (o.key > b.key) b = o;
  }
  key[i] = b.key;
  idx[i] = b.idx;
}

// ------------------------------------------------------------------------------------------------
// Valid extents of padded masks: h = max over columns of column sums etc.
// (reference coarse_matching.py:37-38: p_m.sum(1).max(-1), p_m.sum(-1).max(-1)).  One block per image.
__global__ void mask_extent_kernel(const uint8_t* __restrict__ mask, int h, int w, int* __restrict__ ext) {
  __shared__ int s_h, s_w;
  if (threadIdx.x == 0) { s_h = 0; s_w = 0; }
  __syncthreads();
  const uint8_t* m = mask + static_cast<long>(blockIdx.x) * h * w;
  for (int x = threadIdx.x; x < w; x += blockDim.x) {
    int c = 0;
    for (int y = 0; y < h; ++y) c += m[y * w + x] ? 1 : 0;
    atomicMax(&s_h, c);
  }
  for (int y = threadIdx.x; y < h; y += blockDim.x) {
    int c = 0;
    for (int x = 0; x < w; ++x) c += m[y * w + x] ? 1 : 0;
    atomicMax(&s_w, c);
  }
  __syncthreads();
  if (threadIdx.x == 0) { ext[2 * blockIdx.x] = s_h; ext[2 * blockIdx.x + 1] = s_w; }
}

// ------------------------------------------------------------------------------------------------
// Mutual-nearest-neighbour test + threshold + border removal for every row i of every pair
// (reference coarse_matching.py:175-196).  flag[i]=1 iff (i, j*(i)) is a coarse match;
// conf = exp(rowkey_best + rowterm_i + bias)  [DS: 2z - colLSE + (-rowLSE);  OT: z + v + u - norm].
struct SelectParams {
  int n_pairs, L, S;
  int h0c, w0c, h1c, w1c;
  int border;
  float thr;
  float conf_bias;
  const float* row_key;     // [n*L] best key along the row
  const int* row_arg;       // [n*L] j*(i)
  const int* col_arg;       // [n*S] i*(j)
  const float* rowterm;     // [n*L]
  const uint8_t* mask0;     // optional [n*L]
  const uint8_t* mask1;     // optional [n*S]
  const int* ext0;          // optional [n,2] (h0s, w0s) valid extents when masks are given
  const int* ext1;
  const uint8_t* row_dead;  // optional [n*L]: Sinkhorn prefilter
  const uint8_t* col_dead;  // optional [n*S]
  uint8_t* flag;            // [n*L]
  float* conf;              // [n*L]
};
__global__ void match_flag_kernel(const SelectParams p) {
  const long gi = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (gi >= static_cast<long>(p.n_pairs) * p.L) return;
  const int b = static_cast<int>(gi / p.L);
  const int i = static_cast<int>(gi - static_cast<long>(b) * p.L);
  uint8_t ok = 0;
  float conf = 0.f;
  const int j = p.row_arg[gi];
  if (j >= 0 && j < p.S && p.row_key[gi] > -1.0e29f) {
    const long gj = static_cast<long>(b) * p.S + j;
    bool good = (p.col_arg[gj] == i);
    if (p.mask0) good = good && p.mask0[gi] && p.mask1[gj];
    if (p.row_dead) good = good && !p.row_dead[gi] && !p.col_dead[gj];
    const int y0 = i / p.w0c, x0 = i - y0 * p.w0c;
    const int y1 = j / p.w1c, x1 = j - y1 * p.w1c;
    if (p.border > 0) {
      int h0 = p.h0c, w0 = p.w0c, h1 = p.h1c, w1 = p.w1c;
      if (p.ext0) { h0 = p.ext0[2 * b]; w0 = p.ext0[2 * b + 1]; h1 = p.ext1[2 * b]; w1 = p.ext1[2 * b + 1]; }
      good = good && y0 >= p.border && x0 >= p.border && y1 >= p.border && x1 >= p.border &&
             y0 < h0 - p.border && x0 < w0 - p.border && y1 < h1 - p.border && x1 < w1 - p.border;
    }
    if (good) {
      conf = expf(p.row_key[gi] + p.rowterm[gi] + p.conf_bias);
      good = conf > p.thr;
    }
    ok = good ? 1 : 0;
  }
  p.flag[gi] = ok;
  p.conf[gi] = conf;
}

// Ordered stream compaction (ascending (b, i) like torch.where, coarse_matching.py:194) + coarse
// keypoints (coarse_matching.py:241-250).
struct CompactParams {
  long total;          // n*L
  int L, S, w0c, w1c;
  float scale;         // hw0_i[0] / hw0_c[0]
  const float* scale0; // optional [n,2]
  const float* scale1;
  const uint8_t* flag;
  const float* conf;
  const int* row_arg;
  long capacity;
  long long* b_ids;
  long long* i_ids;
  long long* j_ids;
  float* mconf;
  float* mkpts0;       // [cap,2]
  float* mkpts1;
  int* count;
};
// Two launches instead of one single-block sweep (which took 0.115 ms at n*L = 38400): per-block flag counts, then
// every block derives its exclusive offset from the counts of the blocks before it (<= a few hundred integers) and
// scatters its rows in order.  The output order is the global row order: ascending (b, i).
constexpr int kCompactBlock = 256;
__global__ void __launch_bounds__(kCompactBlock) match_count_kernel(const uint8_t* __restrict__ flag, long total,
                                                                    int* __restrict__ block_counts) {
  __shared__ int s_warp[kCompactBlock / 32];
  const long gi = blockIdx.x * static_cast<long>(kCompactBlock) + threadIdx.x;
  const int f = (gi < total) ? flag[gi] : 0;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = __popc(bal);
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int k = 0; k < kCompactBlock / 32; ++k) t += s_warp[k];
    block_counts[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(kCompactBlock) match_scatter_kernel(const CompactParams p, const int* __restrict__ block_counts) {
  __shared__ int s_warp[kCompactBlock / 32];
  __shared__ int s_red[kCompactBlock / 32];
  __shared__ int s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // exclusive offset of this block = sum of the counts of all earlier blocks
  int part = 0;
  for (int k = threadIdx.x; k < static_cast<int>(blockIdx.x); k += kCompactBlock) part += block_counts[k];
  for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) s_red[warp] = part;
  const long gi = blockIdx.x * static_cast<long>(kCompactBlock) + threadIdx.x;
  const int f = (gi < p.total) ? p.flag[gi] : 0;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  const int wpre = __popc(bal & ((1u << lane) - 1));
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  if (threadIdx.x == 0) {
    int b = 0;
    for (int k = 0; k < kCompactBlock / 32; ++k) b += s_red[k];
    s_base = b;
  }
  __syncthreads();
  int woff = 0, tot = 0;
  for (int k = 0; k < kCompactBlock / 32; ++k) {
    const int c = s_warp[k];
    if (k < warp) woff += c;
    tot += c;
  }
  if (f) {
    const long pos = static_cast<long>(s_base) + woff + wpre;
    if (pos < p.capacity) {
      const int b = static_cast<int>(gi / p.L);
      const int i = static_cast<int>(gi - static_cast<long>(b) * p.L);
      const int j = p.row_arg[gi];
      p.b_ids[pos] = b;
      p.i_ids[pos] = i;
      p.j_ids[pos] = j;
      p.mconf[pos] = p.conf[gi];
      float s0x = p.scale, s0y = p.scale, s1x = p.scale, s1y = p.scale;
      if (p.scale0) {
        s0x = p.scale * p.scale0[2 * b]; s0y = p.scale * p.scale0[2 * b + 1];
        s1x = p.scale * p.scale1[2 * b]; s1y = p.scale * p.scale1[2 * b + 1];
      }
      p.mkpts0[2 * pos] = static_cast<float>(i % p.w0c) * s0x;
      p.mkpts0[2 * pos + 1] = static_cast<float>(i / p.w0c) * s0y;
      p.mkpts1[2 * pos] = static_cast<float>(j % p.w1c) * s1x;
      p.mkpts1[2 * pos + 1] = static_cast<float>(j / p.w1c) * s1y;
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *p.count = s_base + tot;
}

// ------------------------------------------------------------------------------------------------
// Sinkhorn helpers (log_optimal_transport, third_party/SuperGluePretrainedNetwork/models/superglue.py:
// 141-170; called from coarse_matching.py:130-131).  The (L+1)x(S+1) couplings matrix is never
// built: the dustbin row/column hold the scalar bin_score, so their contribution to each log-sum-exp
// is one extra term handled in lse_merge_kernel, and the dustbin potentials are vector LSEs:
//   out[b] = base - LSE( { bin + pot[b, k] : k < count } U { bin + extra } )
__global__ void bin_lse_kernel(const float* __restrict__ pot, int count, const float* __restrict__ bin,
                               const float* __restrict__ extra, float base, float* __restrict__ out) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* p = pot ? pot + static_cast<long>(b) * count : nullptr;
  const float binv = *bin;
  const float ex = binv + (extra ? extra[b] : 0.f);
  float m = ex;
  for (int k = threadIdx.x; k < count; k += blockDim.x) m = fmaxf(m, binv + (p ? p[k] : 0.f));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int k = 1; k < (blockDim.x >> 5); ++k) m = fmaxf(m, red[k]);
  __syncthreads();
  float l = 0.f;
  for (int k = threadIdx.x; k < count; k += blockDim.x) l += expf(binv + (p ? p[k] : 0.f) - m);
  for (int o = 16; o; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < (blockDim.x >> 5); ++k) t += red[k];
    t += expf(ex - m);
    out[b] = base - (m + logf(t));
  }
}

// Sinkhorn prefilter (coarse_matching.py:136-140): a row is dead when its arg max over S+1 columns is
// the dustbin (strictly larger, since torch.max returns the first maximum and the bin is last).
__global__ void ot_dead_kernel(const float* __restrict__ best_key, const float* __restrict__ bin,
                               const float* __restrict__ other_bin_pot, int per, long count,
                               uint8_t* __restrict__ dead) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= count) return;
  const int b = static_cast<int>(i / per);
  dead[i] = (*bin + other_bin_pot[b] > best_key[i]) ? 1 : 0;
}

__global__ void fill_kernel(float* p, float v, long n) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = v;
}

// term[i] = valid[i] ? src[i] (or 0) : kNegBig ; also used to kill prefiltered rows/columns
__global__ void mask_term_kernel(const float* __restrict__ src, const uint8_t* __restrict__ valid,
                                 const uint8_t* __restrict__ dead, long n, float* __restrict__ out) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  float v = src ? src[i] : 0.f;
  if (valid && !valid[i]) v = kNegBig;
  if (dead && dead[i]) v = kNegBig;
  out[i] = v;
}

// ------------------------------------------------------------------------------------------------
// Fine level.  Gather the 5x5 (W x W) windows of both fine maps around each coarse match
// (reference fine_preprocess.py:40-47: F.unfold(kernel=W, stride, padding=W//2) then index by
// (b, i) / (b, j); SURVEY.md §9 V4: win[k=ky*W+kx, c] = feat_f[c, stride*y - W/2 + ky, stride*x - W/2 + kx],
// zero outside) straight into fp16 planes -- the full im2col is never materialised.
// Row layout of the output: side*M*WW + m*WW + k.  Strides are in elements so NCHW and NHWC both work.
struct FineGatherParams {
  const float* feat0;
  const float* feat1;
  long sn0, sc0, sh0, sw0;
  long sn1, sc1, sh1, sw1;
  int Hf0, Wf0, Hf1, Wf1;
  int w0c, w1c;
  int stride, W, Cf;
  long M;
  const long long* b_ids;
  const long long* i_ids;
  const long long* j_ids;
  __half* out_hi;   // [2*M*WW, ld]
  __half* out_lo;
  int ld;
  const int* live;  // optional device count: windows m >= min(*live, M) of each side are skipped (M = capacity)
};
__global__ void fine_gather_kernel(const FineGatherParams p) {
  const int WW = p.W * p.W;
  const long win = blockIdx.x;             // 0 .. 2M-1
  const int side = win >= p.M ? 1 : 0;
  const long m = side ? win - p.M : win;
  if (p.live != nullptr && m >= *p.live) return;
  const int b = static_cast<int>(p.b_ids[m]);
  const int idx = static_cast<int>(side ? p.j_ids[m] : p.i_ids[m]);
  const int wc = side ? p.w1c : p.w0c;
  const int cy = idx / wc, cx = idx - cy * wc;
  const float* feat = side ? p.feat1 : p.feat0;
  const long sn = side ? p.sn1 : p.sn0, sc = side ? p.sc1 : p.sc0, sh = side ? p.sh1 : p.sh0,
             sw = side ? p.sw1 : p.sw0;
  const int Hf = side ? p.Hf1 : p.Hf0, Wf = side ? p.Wf1 : p.Wf0;
  for (int e = threadIdx.x; e < WW * p.Cf; e += blockDim.x) {
    const int k = e / p.Cf, c = e - k * p.Cf;
    const int ky = k / p.W, kx = k - ky * p.W;
    const int y = p.stride * cy - p.W / 2 + ky;
    const int x = p.stride * cx - p.W / 2 + kx;
    float v = 0.f;
    if (y >= 0 && y < Hf && x >= 0 && x < Wf) v = feat[b * sn + c * sc + y * sh + x * sw];
    __half hh, ll;
    split_f16(v, hh, ll);
    const long row = win * WW + k;
    p.out_hi[row * p.ld + c] = hh;
    p.out_lo[row * p.ld + c] = ll;
  }
}

// Channel-contiguous (NHWC, sc == 1) maps with Cf % 8 == 0: one thread moves 8 channels of one window position --
// two 16-byte loads, packed split, one 16-byte store per plane (the element-wise kernel above issues 2-byte stores).
__global__ void __launch_bounds__(256) fine_gather_vec8_kernel(const FineGatherParams p) {
  const int WW = p.W * p.W;
  const int c8n = p.Cf >> 3;
  const long win = blockIdx.x;             // 0 .. 2M-1
  const int side = win >= p.M ? 1 : 0;
  const long m = side ? win - p.M : win;
  if (p.live != nullptr && m >= *p.live) return;
  const int b = static_cast<int>(p.b_ids[m]);
  const int idx = static_cast<int>(side ? p.j_ids[m] : p.i_ids[m]);
  const int wc = side ? p.w1c : p.w0c;
  const int cy = idx / wc, cx = idx - cy * wc;
  const float* feat = side ? p.feat1 : p.feat0;
  const long sn = side ? p.sn1 : p.sn0, sh = side ? p.sh1 : p.sh0, sw = side ? p.sw1 : p.sw0;
  const int Hf = side ? p.Hf1 : p.Hf0, Wf = side ? p.Wf1 : p.Wf0;
  for (int e = threadIdx.x; e < WW * c8n; e += blockDim.x) {
    const int k = e / c8n, c = (e - k * c8n) << 3;
    const int ky = k / p.W, kx = k - ky * p.W;
    const int y = p.stride * cy - p.W / 2 + ky;
    const int x = p.stride * cx - p.W / 2 + kx;
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
    if (y >= 0 && y < Hf && x >= 0 && x < Wf) {
      const float4* src = reinterpret_cast<const float4*>(feat + b * sn + y * sh + x * sw + c);
      v0 = src[0];
      v1 = src[1];
    }
    uint32_t h[4], l[4];
    split_f16x2(v0.x, v0.y, h[0], l[0]);
    split_f16x2(v0.z, v0.w, h[1], l[1]);
    split_f16x2(v1.x, v1.y, h[2], l[2]);
    split_f16x2(v1.z, v1.w, h[3], l[3]);
    const long o = (win * WW + k) * p.ld + c;
    *reinterpret_cast<uint4*>(p.out_hi + o) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(p.out_lo + o) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// Per-window bias of the merge projection (reference fine_preprocess.py:50-56):
//   c = down_proj(feat_c[b, idx]) ;  gbias = W_merge[:, Cf:2Cf] @ c + b_merge
// (the repeated coarse half of the concatenation is identical for all WW positions of a window).
// Weights arrive TRANSPOSED ([in, out]) so that thread o's reads are coalesced; a block handles
// kFineBiasWin windows so every weight element is read once per kFineBiasWin outputs.
constexpr int kFineBiasWin = 8;
struct FineBiasParams {
  const float* feat_c;     // coarse transformer output x_f32 [rows, Cc]: set 0 rows then set 1 rows
  long set1_row_base;
  int L, S, Cc, Cf;
  long M;
  const long long* b_ids;
  const long long* i_ids;
  const long long* j_ids;
  const float* WdT;        // [Cc, Cf]  down_proj.weight^T
  const float* bd;         // [Cf]
  const float* Wm2T;       // [Cf, Cf]  merge_feat.weight[:, Cf:2Cf]^T
  const float* bm;         // [Cf]
  float* gbias;            // [2M, Cf]
  const int* live;         // optional device count: windows m >= min(*live, M) of each side are skipped
};
__global__ void __launch_bounds__(128) fine_bias_kernel(const FineBiasParams p) {
  pdl_trigger();
  __shared__ float s_fc[kFineBiasWin][256];
  __shared__ float s_c[kFineBiasWin][128];
  const long win0 = static_cast<long>(blockIdx.x) * kFineBiasWin;
  const long nwin = 2 * p.M;
  const long n_live = p.live != nullptr ? min(static_cast<long>(*p.live), p.M) : p.M;
  auto is_live = [&](long win) { return win < nwin && (win >= p.M ? win - p.M : win) < n_live; };
  {
    bool any = false;
    for (int wv = 0; wv < kFineBiasWin; ++wv) any |= is_live(win0 + wv);
    if (!any) return;   // block-uniform
  }
  for (int wv = 0; wv < kFineBiasWin; ++wv) {
    const long win = win0 + wv;
    if (is_live(win)) {
      const int side = win >= p.M ? 1 : 0;
      const long m = side ? win - p.M : win;
      const long b = p.b_ids[m];
      const long row = side ? p.set1_row_base + b * p.S + p.j_ids[m] : b * p.L + p.i_ids[m];
      for (int c = threadIdx.x; c < p.Cc; c += blockDim.x) s_fc[wv][c] = p.feat_c[row * p.Cc + c];
    } else {
      for (int c = threadIdx.x; c < p.Cc; c += blockDim.x) s_fc[wv][c] = 0.f;
    }
  }
  __syncthreads();
  const int o = threadIdx.x;
  if (o < p.Cf) {
    float a[kFineBiasWin];
#pragma unroll
    for (int wv = 0; wv < kFineBiasWin; ++wv) a[wv] = p.bd[o];
    for (int c = 0; c < p.Cc; ++c) {
      const float wgt = p.WdT[static_cast<long>(c) * p.Cf + o];
#pragma unroll
      for (int wv = 0; wv < kFineBiasWin; ++wv) a[wv] = fmaf(wgt, s_fc[wv][c], a[wv]);
    }
#pragma unroll
    for (int wv = 0; wv < kFineBiasWin; ++wv) s_c[wv][o] = a[wv];
  }
  __syncthreads();
  if (o < p.Cf) {
    float a[kFineBiasWin];
#pragma unroll
    for (int wv = 0; wv < kFineBiasWin; ++wv) a[wv] = p.bm[o];
    for (int c = 0; c < p.Cf; ++c) {
      const float wgt = p.Wm2T[static_cast<long>(c) * p.Cf + o];
#pragma unroll
      for (int wv = 0; wv < kFineBiasWin; ++wv) a[wv] = fmaf(wgt, s_c[wv][c], a[wv]);
    }
#pragma unroll
    for (int wv = 0; wv < kFineBiasWin; ++wv)
      if (is_live(win0 + wv)) p.gbias[(win0 + wv) * p.Cf + o] = a[wv];
  }
}

// Fine matching (reference fine_matching.py:43-74): correlate the centre of window 0 with window 1,
// softmax(1/sqrt(C)), spatial expectation on the normalised grid [-1,1]^2 (kornia
// dsnt.spatial_expectation2d with normalized_coordinates=True), std, and the refined keypoint
// mkpts1_f = mkpts1_c + coords * (W//2) * scale1.  One warp per match.
struct FineMatchParams {
  const float* f0;       // [M*WW, C]
  const float* f1;
  int W, C;
  long M;
  float scale;           // hw0_i[0] / hw0_f[0]
  const float* scale1;   // optional [n,2]
  const long long* b_ids;
  const float* mkpts1_c; // [M,2]
  float* expec_f;        // [M,3]
  float* mkpts1_f;       // [M,2]
  const int* live;       // optional device count: matches m >= min(*live, M) are skipped (M = capacity)
};
__global__ void fine_match_kernel(const FineMatchParams p) {
  const long m = (blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (m >= p.M || (p.live != nullptr && m >= *p.live)) return;
  const int WW = p.W * p.W;
  const float* c0 = p.f0 + (m * WW + WW / 2) * p.C;
  const float* w1 = p.f1 + m * WW * p.C;
  // lane r (< WW) gets sim[r]; C <= 128 -> each lane holds 4 channels of the centre
  float sim = kNegBig;
  for (int r = 0; r < WW; ++r) {
    float part = 0.f;
    for (int c = lane; c < p.C; c += 32) part = fmaf(c0[c], w1[r * p.C + c], part);
    for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == r) sim = part;
  }
  const float temp = 1.0f / sqrtf(static_cast<float>(p.C));
  float v = (lane < WW) ? sim * temp : kNegBig;
  float mx = v;
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float e = (lane < WW) ? expf(v - mx) : 0.f;
  float den = e;
  for (int o = 16; o; o >>= 1) den += __shfl_xor_sync(0xffffffffu, den, o);
  const float heat = e / den;
  const int ky = lane / p.W, kx = lane - ky * p.W;
  const float step = 2.f / static_cast<float>(p.W - 1);
  const float gx = (lane < WW) ? -1.f + step * kx : 0.f;
  const float gy = (lane < WW) ? -1.f + step * ky : 0.f;
  float ex = gx * heat, ey = gy * heat, exx = gx * gx * heat, eyy = gy * gy * heat;
  for (int o = 16; o; o >>= 1) {
    ex += __shfl_xor_sync(0xffffffffu, ex, o);
    ey += __shfl_xor_sync(0xffffffffu, ey, o);
    exx += __shfl_xor_sync(0xffffffffu, exx, o);
    eyy += __shfl_xor_sync(0xffffffffu, eyy, o);
  }
  if (lane == 0) {
    const float vx = fmaxf(exx - ex * ex, 1e-10f), vy = fmaxf(eyy - ey * ey, 1e-10f);
    const float sd = sqrtf(vx) + sqrtf(vy);
    p.expec_f[3 * m] = ex;
    p.expec_f[3 * m + 1] = ey;
    p.expec_f[3 * m + 2] = sd;
    float sx = p.scale, sy = p.scale;
    if (p.scale1) {
      const long b = p.b_ids[m];
      sx = p.scale * p.scale1[2 * b];
      sy = p.scale * p.scale1[2 * b + 1];
    }
    const float half_w = static_cast<float>(p.W / 2);
    p.mkpts1_f[2 * m] = p.mkpts1_c[2 * m] + ex * half_w * sx;
    p.mkpts1_f[2 * m + 1] = p.mkpts1_c[2 * m + 1] + ey * half_w * sy;
  }
}

// ------------------------------------------------------------------------------------------------
// Evaluation harness (SURVEY.md §8(f) rank 3): squared symmetric epipolar distance of every match against the
// ground-truth relative pose of its pair (reference src/utils/metrics.py:30-72): E = [t]_x R from T_0to1, points
// normalised by the intrinsics, d = (p1^T E p0)^2 (1 / |(E p0)_xy|^2 + 1 / |(E^T p1)_xy|^2).  One thread per match.
__global__ void epipolar_error_kernel(const float* __restrict__ mk0, const float* __restrict__ mk1,
                                      const long long* __restrict__ bids, long M, int n_pairs,
                                      const float* __restrict__ T_0to1 /*[n,4,4]*/, const float* __restrict__ K0 /*[n,3,3]*/,
                                      const float* __restrict__ K1, float* __restrict__ err) {
  const long m = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (m >= M) return;
  const long b = bids[m];
  if (b < 0 || b >= n_pairs) {
    err[m] = __int_as_float(0x7fc00000);   // NaN: a match that belongs to no pair
    return;
  }
  const float* T = T_0to1 + b * 16;
  const float tx = T[3], ty = T[7], tz = T[11];
  float E[9];   // [t]_x R, row-major
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float r0 = T[c], r1 = T[4 + c], r2 = T[8 + c];
    E[c] = -tz * r1 + ty * r2;
    E[3 + c] = tz * r0 - tx * r2;
    E[6 + c] = -ty * r0 + tx * r1;
  }
  const float* k0 = K0 + b * 9;
  const float* k1 = K1 + b * 9;
  const float x0 = (mk0[2 * m] - k0[2]) / k0[0], y0 = (mk0[2 * m + 1] - k0[5]) / k0[4];
  const float x1 = (mk1[2 * m] - k1[2]) / k1[0], y1 = (mk1[2 * m + 1] - k1[5]) / k1[4];
  const float a0 = E[0] * x0 + E[1] * y0 + E[2];          // E p0
  const float a1 = E[3] * x0 + E[4] * y0 + E[5];
  const float a2 = E[6] * x0 + E[7] * y0 + E[8];
  const float c0 = E[0] * x1 + E[3] * y1 + E[6];          // E^T p1
  const float c1 = E[1] * x1 + E[4] * y1 + E[7];
  const float pep = x1 * a0 + y1 * a1 + a2;
  err[m] = pep * pep * (1.0f / (a0 * a0 + a1 * a1) + 1.0f / (c0 * c0 + c1 * c1));
}

}  // namespace lb
