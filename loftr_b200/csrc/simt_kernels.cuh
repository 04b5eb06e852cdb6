// Small CUDA-core kernels of the matching hot path: operand preparation, the linear-attention
// core (KV = K^T V is only H x D x D floats per image), partial merges, match selection and the fine
// level.  They are bandwidth / latency bound; the dense work lives in gemm_split.cuh.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>
#include "../../include/loftr_b200.h"
#include "epilogues.cuh"

namespace lb {

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
// kIndexed: output image `img` reads source image img_idx[img] of `feat` (a per-image feature bank shared by several
// pairs); otherwise it reads image `img` and img_idx is unused.
template <bool kIndexed>
__global__ void coarse_prep_kernel(const float* __restrict__ feat, int nhwc, const float* __restrict__ pe, int C,
                                   int h, int w, int pe_h, int pe_w, float* __restrict__ x_f32,
                                   __half* __restrict__ cat_hi, __half* __restrict__ cat_lo,
                                   const int* __restrict__ img_idx) {
  pdl_trigger();
  __shared__ float tile[32][33];
  const int L = h * w;
  const int img = blockIdx.z;
  const long src = kIndexed ? img_idx[img] : 0;   // source image (indexed variant)
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
      if (!nhwc) v += feat[((kIndexed ? src : static_cast<long>(img)) * C + c) * L + l];
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
      if (nhwc) v = feat[(kIndexed ? src * L + l : row) * C + c] + v;
      x_f32[row * C + c] = v;
      __half hh, ll;
      split_f16(v, hh, ll);
      cat_hi[row * (2 * C) + c] = hh;
      cat_lo[row * (2 * C) + c] = ll;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Image front end: uint8 source images of any size (grey, or interleaved RGB / BGR) -> the matcher's input
// [n, 1, H, W] fp32 in [0, 1], each image resized to its (h_new, w_new), placed top-left in the H x W canvas and
// zero-padded, plus the 1/8 padding mask.  = imread_gray's colour conversion, cv2.resize (INTER_LINEAR), pad_bottom_right
// and `/ 255` of the reference (src/utils/dataset.py:47-51,94-125,141-157) and the mask subsampling of
// src/datasets/megadepth.py:119-125.  HBM-bound: one pass, no shared memory, no atomics.
//
// Grey level of source pixel (y, x): the byte itself, or OpenCV's 15-bit fixed-point luma of an interleaved pixel.
__device__ __forceinline__ float image_level(const LbImageDesc& d, int y, int x) {
  const uint8_t* p = d.src + static_cast<long>(y) * d.row_stride_bytes + static_cast<long>(x) * d.channels;
  if (d.channels == 1) return static_cast<float>(__ldg(p));
  const int r = __ldg(p + d.r_index), g = __ldg(p + 1), b = __ldg(p + 2 - d.r_index);
  return static_cast<float>((9798 * r + 19235 * g + 3735 * b + 16384) >> 15);
}

constexpr int kPreprocessBlockX = 32;   // threads along x, four output pixels each: a 128-pixel tile row
constexpr int kPreprocessBlockY = 8;
// grid (cdiv(W, 128), cdiv(H, 8), n); descs[img] describes image blockIdx.z.  Bilinear taps with half-pixel centres and
// edge clamp.  The source coordinate is formed in fp64 (in fp32 its rounding at x ~ 1000 would move the weight by 1e-4,
// i.e. the result by up to 1e-4 of full scale on a noisy image); the interpolation itself is fp32 on levels 0..255,
// not rounded to a level, then a true division by 255.  With h_new == h and w_new == w both weights are exactly 0 and
// the output is level / 255 bit for bit.  W is a multiple of 8, so a thread's four pixels lie in one row and its float4
// store is aligned; mask cell (Y, X) is written by the thread that owns pixel (8Y, 8X).
__global__ void __launch_bounds__(kPreprocessBlockX * kPreprocessBlockY)
preprocess_images_kernel(const LbImageDesc* __restrict__ descs, float* __restrict__ out, int H, int W,
                         uint8_t* __restrict__ mask) {
  const int img = blockIdx.z;
  const int x4 = (blockIdx.x * kPreprocessBlockX + threadIdx.x) * 4;
  const int y = blockIdx.y * kPreprocessBlockY + threadIdx.y;
  if (x4 >= W || y >= H) return;
  const LbImageDesc d = descs[img];
  const bool inside = y < d.h_new && x4 < d.w_new;
  float v[4] = {0.f, 0.f, 0.f, 0.f};   // padding is exactly 0
  if (inside) {
    const double sy = (y + 0.5) * (static_cast<double>(d.h) / d.h_new) - 0.5;
    const double sy0 = floor(sy);
    const float fy = static_cast<float>(sy - sy0);
    const int y0 = min(max(static_cast<int>(sy0), 0), d.h - 1);
    const int y1 = min(max(static_cast<int>(sy0) + 1, 0), d.h - 1);
    const double rx = static_cast<double>(d.w) / d.w_new;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = x4 + i;
      if (x >= d.w_new) break;
      const double sx = (x + 0.5) * rx - 0.5;
      const double sx0 = floor(sx);
      const float fx = static_cast<float>(sx - sx0);
      const int x0 = min(max(static_cast<int>(sx0), 0), d.w - 1);
      const int x1 = min(max(static_cast<int>(sx0) + 1, 0), d.w - 1);
      const float a = image_level(d, y0, x0), b = image_level(d, y0, x1);
      const float c = image_level(d, y1, x0), e = image_level(d, y1, x1);
      const float top = a + fx * (b - a);
      const float bot = c + fx * (e - c);
      v[i] = (top + fy * (bot - top)) / 255.0f;
    }
  }
  *reinterpret_cast<float4*>(out + (static_cast<long>(img) * H + y) * W + x4) = make_float4(v[0], v[1], v[2], v[3]);
  if (mask && (y & 7) == 0 && (x4 & 7) == 0)
    mask[(static_cast<long>(img) * (H >> 3) + (y >> 3)) * (W >> 3) + (x4 >> 3)] = inside ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// Rectified matching (DESIGN.md §19): image1 resampled onto image0's canvas through a per-pair homography x1 ~ H x0,
// and points of that canvas mapped back into image1.  H acts on source pixels: network pixel (x, y) of image k sits at
// (x * sx_k, y * sy_k), with (sx_k, sy_k) = scale_k[b], or (1, 1) without scales.
//
// Pair b's model as both kernels apply it, in fp64: the identity when an entry is not finite (a failed estimate), and
// otherwise H times the sign of w at the centre ((W0 - 1) / 2, (H0 - 1) / 2) of image0's canvas (+1 when that w is 0),
// so that H and -H act alike and w <= 0 marks points beyond the horizon.
__device__ __forceinline__ void rectify_model(const float* __restrict__ models, long b, double cx, double cy,
                                              double* h) {
  bool finite = true;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    h[k] = static_cast<double>(models[b * 9 + k]);
    finite = finite && isfinite(h[k]);
  }
  if (!finite) {
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = (k % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  if (h[6] * cx + h[7] * cy + h[8] < 0.0) {
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = -h[k];
  }
}

// (qx, qy, qw) = H (px, py, 1); the one expression both kernels evaluate, so a point and its pixel agree
__device__ __forceinline__ void rectify_apply(const double* h, double px, double py, double& qx, double& qy,
                                              double& qw) {
  qx = h[0] * px + h[1] * py + h[2];
  qy = h[3] * px + h[4] * py + h[5];
  qw = h[6] * px + h[7] * py + h[8];
}

constexpr int kRectifyBlockX = 32;   // threads along x, four output pixels each: a 128-pixel tile row
constexpr int kRectifyBlockY = 8;
// grid (cdiv(W, 128), cdiv(H, 8), n): output pixel (x, y) of pair blockIdx.z takes image1 at
//   (u, v) = (H (x sx0, y sy0, 1))_xy / w / (sx1, sy1)      (image1's network pixels)
// bilinearly, pixel centres at integer coordinates, taps outside [0, W1 - 1] x [0, H1 - 1] read as 0 (grid_sample with
// align_corners=True and zero padding); 0 where w <= 0.  The coordinates are fp64 (as in preprocess_images_kernel: in
// fp32 their rounding would move the weights by ~1e-4 at x ~ 1000) and the interpolation is fp32 with exact weights of
// 0 at integer coordinates, so an identity model with equal sizes and scales copies image1 bit for bit.  No texture
// filtering: its weights have 8 fractional bits.  W is a multiple of 8, so a thread's four pixels lie in one row and
// its float4 store is aligned.
__global__ void __launch_bounds__(kRectifyBlockX * kRectifyBlockY)
rectify_images_kernel(const float* __restrict__ image1, int H1, int W1, const float* __restrict__ models,
                      const float* __restrict__ scale0, const float* __restrict__ scale1, float* __restrict__ out,
                      int H, int W) {
  __shared__ double s_h[9];
  __shared__ double s_scale[4];   // sx0, sy0, sx1, sy1
  const int b = blockIdx.z;
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const double sx0 = scale0 ? scale0[2 * b] : 1.0, sy0 = scale0 ? scale0[2 * b + 1] : 1.0;
    double h[9];
    rectify_model(models, b, 0.5 * (W - 1) * sx0, 0.5 * (H - 1) * sy0, h);
#pragma unroll
    for (int k = 0; k < 9; ++k) s_h[k] = h[k];
    s_scale[0] = sx0;
    s_scale[1] = sy0;
    s_scale[2] = scale1 ? scale1[2 * b] : 1.0;
    s_scale[3] = scale1 ? scale1[2 * b + 1] : 1.0;
  }
  __syncthreads();
  const int x4 = (blockIdx.x * kRectifyBlockX + threadIdx.x) * 4;
  const int y = blockIdx.y * kRectifyBlockY + threadIdx.y;
  if (x4 >= W || y >= H) return;
  double h[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) h[k] = s_h[k];
  const double sx0 = s_scale[0], py = y * s_scale[1], sx1 = s_scale[2], sy1 = s_scale[3];
  const float* src = image1 + static_cast<long>(b) * H1 * W1;
  auto tap = [&](int ix, int iy) {
    return (ix >= 0 && ix < W1 && iy >= 0 && iy < H1) ? __ldg(src + static_cast<long>(iy) * W1 + ix) : 0.f;
  };
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double qx, qy, qw;
    rectify_apply(h, (x4 + i) * sx0, py, qx, qy, qw);
    v[i] = 0.f;
    if (!(qw > 0.0)) continue;
    const double u = qx / qw / sx1, w = qy / qw / sy1;
    if (!(u > -1.0 && u < W1 && w > -1.0 && w < H1)) continue;   // no tap inside (and no int overflow below)
    const double u0 = floor(u), w0 = floor(w);
    const float fx = static_cast<float>(u - u0), fy = static_cast<float>(w - w0);
    const int ix = static_cast<int>(u0), iy = static_cast<int>(w0);
    const float a = tap(ix, iy), c = tap(ix + 1, iy);
    const float d = tap(ix, iy + 1), e = tap(ix + 1, iy + 1);
    const float top = a + fx * (c - a);
    const float bot = d + fx * (e - d);
    v[i] = top + fy * (bot - top);
  }
  *reinterpret_cast<float4*>(out + (static_cast<long>(b) * H + y) * W + x4) = make_float4(v[0], v[1], v[2], v[3]);
}

// Points of the rectified canvas back into image1: point i of pair ids[i] (source pixels of image0's frame) ->
// H p in fp64, rounded once to fp32 (source pixels of image1); NaN with inside 0 where w <= 0, the point is not
// finite or the pair id is out of range.  inside[i]: the mapped point divided by scale1 lies in [0, W1 - 1] x
// [0, H1 - 1] and, with mask1, in a true cell of mask1[b] (cell (floor(v / 8), floor(u / 8)), w1c cells per row).
// Only i < min(*live, m) when live is given.
struct RectifyPointsParams {
  const float* pts;
  const long long* ids;
  long m;
  const int* live;
  const float* models;
  int n_pairs;
  const float* scale0;
  const float* scale1;
  int H0, W0, H1, W1;
  const uint8_t* mask1;
  int w1c;
  float* out;
  uint8_t* inside;
};

__global__ void rectify_points_kernel(const RectifyPointsParams p) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  const long m = p.live ? min(p.m, static_cast<long>(max(*p.live, 0))) : p.m;
  if (i >= m) return;
  const long long b = p.ids[i];
  float ox = __int_as_float(0x7fc00000), oy = ox;   // NaN
  bool in = false;
  if (b >= 0 && b < p.n_pairs) {
    const double sx0 = p.scale0 ? p.scale0[2 * b] : 1.0, sy0 = p.scale0 ? p.scale0[2 * b + 1] : 1.0;
    double h[9];
    rectify_model(p.models, b, 0.5 * (p.W0 - 1) * sx0, 0.5 * (p.H0 - 1) * sy0, h);
    double qx, qy, qw;
    rectify_apply(h, p.pts[2 * i], p.pts[2 * i + 1], qx, qy, qw);
    if (qw > 0.0) {
      const double x = qx / qw, y = qy / qw;
      ox = static_cast<float>(x);
      oy = static_cast<float>(y);
      const double u = x / (p.scale1 ? p.scale1[2 * b] : 1.0), v = y / (p.scale1 ? p.scale1[2 * b + 1] : 1.0);
      in = u >= 0.0 && u <= p.W1 - 1 && v >= 0.0 && v <= p.H1 - 1;
      if (in && p.mask1)
        in = p.mask1[(b * (p.H1 >> 3) + static_cast<long>(floor(v / 8))) * p.w1c + static_cast<long>(floor(u / 8))] != 0;
    }
  }
  p.out[2 * i] = ox;
  p.out[2 * i + 1] = oy;
  if (p.inside) p.inside[i] = in ? 1 : 0;
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

// ------------------------------------------------------------------------------------------------
// Fine (window) linear attention (reference linear_attention.py:43-46 on the [M, 25, 128] window sequences of
// fine_preprocess.py), one kernel per pass:
//   out[r,h,:] = (Q[r,h,:] . KV[g,h]) / (Q[r,h,:] . Ksum[g,h] + eps)
// written as fp16 planes = the A operand of the merge projection.  Query window g has x_rows rows and source window g
// s_rows rows (both <= 32; they differ in a cross pass of the standalone fine transformer with L != S).  One block
// takes windows g, g + gridDim.x, ...; KV[h] = K_h^T V_h and Ksum_h over the s_rows source rows are built in shared
// memory (never in HBM) and warp h / lane r applies them to query row r.  The kernel is latency-bound on the q/k/v
// reads (ncu: 34 % of the samples wait on them), so the NEXT window's K / V rows travel global -> shared with cp.async
// into the other half of a double buffer and its query row into registers while the current window is computed.
// Dynamic shared memory: 2 x 2 x s_rows x 512 B + 8.7 KB (60 KB for 25 rows).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int D, int H>
__global__ void __launch_bounds__(32 * H, 3) window_attn_kernel(const float* __restrict__ qkv, int ld, int q_col0, int k_col0,
                                                                int v_col0, long x_row_base, long s_row_base,
                                                                int x_rows, int s_rows, int n_groups, float eps,
                                                                __half* __restrict__ att_hi, __half* __restrict__ att_lo,
                                                                int ld_att, const int* __restrict__ live, int live_cap) {
  pdl_trigger();
  static_assert(D == 16 && H == 8, "fine head layout");
  constexpr int C = D * H;  // 128
  constexpr int PER = D * D + D;
  extern __shared__ __align__(16) float wa_smem[];
  float* sKV = wa_smem;                                   // [H][PER]
  float* sKVbuf = wa_smem + H * PER;                      // [2][K | V][s_rows][C]
  const int buf_floats = 2 * s_rows * C;
  const int tid = threadIdx.x;
  const int hd = tid >> 5, lane = tid & 31;
  const bool has_row = lane < x_rows;

  auto issue = [&](int g, int b) {   // K / V rows of window g -> buffer b
    float* dK = sKVbuf + b * buf_floats;
    float* dV = dK + s_rows * C;
    for (int i = tid; i < s_rows * (C / 4); i += 32 * H) {
      const int r = i / (C / 4), c4 = (i % (C / 4)) * 4;
      const float* rowp = qkv + (s_row_base + static_cast<long>(g) * s_rows + r) * ld;
      cp_async16(dK + r * C + c4, rowp + k_col0 + c4);
      cp_async16(dV + r * C + c4, rowp + v_col0 + c4);
    }
  };
  auto load_q = [&](int g, float (&q)[D]) {
    const float4* qp = reinterpret_cast<const float4*>(
        qkv + (x_row_base + static_cast<long>(g) * x_rows + lane) * ld + q_col0 + hd * D);
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
    const float* sV = sK + s_rows * C;
    // KV[hd][d][v0..v0+7] and Ksum[hd][d] over the source window's rows
    {
      const int d = lane >> 1, v0 = (lane & 1) * 8;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      float ks = 0.f;
      for (int r = 0; r < s_rows; ++r) {
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
      const long xrow = x_row_base + static_cast<long>(g) * x_rows + lane;
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

// Caller-given points -> the coarse answer of each: image0 points (kSide 0, LoFTR.match_points, DESIGN.md §17) or
// image1 points (kSide 1, §22).  Fields are named by role: "q" is the queried image, "o" the other; the host maps
// rows and columns onto them.  Each query takes the q cell nearest to the point, its arg-max in o, conf and flags as
// match_flag_kernel computes them, and the fine window centres of both images.  One thread per query; queries that are
// not inside get NaN points, conf 0, no flags, ids -1 and fine-stage ids (win) 0, so no later kernel reads through an
// invalid index.  ids, centres and win are written in (image0, image1) order.  Where the sides differ:
//   mutual  side 0: arg_o[answer] == cell; side 1 also needs the answer row to have a valid column.
//   conf    exp((key + term) + conf_bias) of the queried cell, except a mutual answer on side 1, which takes its row's
//           (o) expression, so it equals mconf bit for bit.
//   valid   side 0: flag[i]; side 1: mutual && flag[i], i.e. the forward keeps (b, i, j).
struct QueryParams {
  int n_pairs, Q, L, S;
  int h0c, w0c, h1c, w1c;
  int Hq, Wq;               // queried image (network pixels)
  int Hfq, Wfq;             // fine map of the queried image
  int stride;               // fine pixels per coarse cell
  float s_c, s_f;           // image pixels per coarse / fine pixel
  float conf_bias;
  const float* points_q;    // [n*Q, 2] (x, y), source pixels when the queried image's scale is given
  const uint8_t* valid_q;   // optional [n*Q]
  const float* scale0;      // optional [n, 2]
  const float* scale1;
  const uint8_t* mask_q;    // optional, per queried cell
  const float* key_q;       // per queried cell: best key, arg-max in o, conf term (row_* on side 0, col_* on side 1)
  const int* arg_q;
  const float* term_q;
  const float* key_o;       // per cell of o: the same
  const int* arg_o;
  const float* term_o;
  const uint8_t* flag;      // [n*L] match_flag_kernel's test
  long long* i_ids;         // [n*Q]
  long long* j_ids;
  float* conf;
  uint8_t* mutual;
  uint8_t* valid;
  uint8_t* inside;
  int* centres;             // [2, n*Q, 2] fine-map (x, y) of the image0 / image1 window centres
  long long* win;           // [3, n*Q] (b, i, j) read by the fine stage
  float* pts_qf;            // [n*Q, 2] the query snapped to the queried image's fine grid
  float* pts_oc;            // [n*Q, 2] the window centre in o
};
template <int kSide>
__global__ void coarse_query_kernel(const QueryParams p) {
  constexpr bool k1 = kSide == 1;
  const long q = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  const long nq = static_cast<long>(p.n_pairs) * p.Q;
  if (q >= nq) return;
  const int b = static_cast<int>(q / p.Q);
  const int Nq = k1 ? p.S : p.L, No = k1 ? p.L : p.S;   // cells of q / o
  const int hqc = k1 ? p.h1c : p.h0c, wqc = k1 ? p.w1c : p.w0c, woc = k1 ? p.w0c : p.w1c;
  const float* scale_q = k1 ? p.scale1 : p.scale0;
  const float* scale_o = k1 ? p.scale0 : p.scale1;
  float sxq = 1.f, syq = 1.f, sxo = 1.f, syo = 1.f;
  if (scale_q) { sxq = scale_q[2 * b]; syq = scale_q[2 * b + 1]; sxo = scale_o[2 * b]; syo = scale_o[2 * b + 1]; }
  float px = p.points_q[2 * q], py = p.points_q[2 * q + 1];
  if (scale_q) { px = px / sxq; py = py / syq; }
  // the comparisons are false for NaN, so a NaN coordinate fails here
  bool in = (!p.valid_q || p.valid_q[q]) && px >= 0.f && px <= static_cast<float>(p.Wq - 1) && py >= 0.f &&
            py <= static_cast<float>(p.Hq - 1);
  int cell = 0, ans = 0, cx = 0, cy = 0;
  long gq = 0;
  if (in) {
    cx = min(max(static_cast<int>(floorf(px / p.s_c + 0.5f)), 0), wqc - 1);
    cy = min(max(static_cast<int>(floorf(py / p.s_c + 0.5f)), 0), hqc - 1);
    cell = cy * wqc + cx;
    gq = static_cast<long>(b) * Nq + cell;
    if (p.mask_q && !p.mask_q[gq]) in = false;
  }
  if (in) {
    ans = p.arg_q[gq];
    in = ans >= 0 && ans < No && p.key_q[gq] > -1.0e29f;   // a cell without any valid partner has no answer
  }
  const long nq2 = 2 * nq;
  if (!in) {
    const float nan = __int_as_float(0x7fffffff);
    p.i_ids[q] = -1; p.j_ids[q] = -1;
    p.conf[q] = 0.f;
    p.mutual[q] = 0; p.valid[q] = 0; p.inside[q] = 0;
    p.centres[2 * q] = 0; p.centres[2 * q + 1] = 0; p.centres[2 * (nq + q)] = 0; p.centres[2 * (nq + q) + 1] = 0;
    p.win[q] = b; p.win[nq + q] = 0; p.win[nq2 + q] = 0;
    p.pts_qf[2 * q] = nan; p.pts_qf[2 * q + 1] = nan;
    p.pts_oc[2 * q] = nan; p.pts_oc[2 * q + 1] = nan;
    return;
  }
  const int fxq = min(max(static_cast<int>(floorf(px / p.s_f + 0.5f)), 0), p.Wfq - 1);
  const int fyq = min(max(static_cast<int>(floorf(py / p.s_f + 0.5f)), 0), p.Hfq - 1);
  const int ay = ans / woc, ax = ans - ay * woc;
  const int fxo = p.stride * ax + (fxq - p.stride * cx);
  const int fyo = p.stride * ay + (fyq - p.stride * cy);
  const long go = static_cast<long>(b) * No + ans;
  bool mutual = p.arg_o[go] == cell;
  // a row without any valid column (key kNegBig) has no arg-max, as in match_flag_kernel
  if constexpr (k1) mutual = mutual && p.key_o[go] > -1.0e29f;
  const bool conf_o = k1 && mutual;
  p.conf[q] = expf((conf_o ? p.key_o[go] : p.key_q[gq]) + (conf_o ? p.term_o[go] : p.term_q[gq]) + p.conf_bias);
  p.mutual[q] = mutual ? 1 : 0;
  if constexpr (k1) p.valid[q] = mutual && p.flag[go] ? 1 : 0;
  else p.valid[q] = p.flag[gq];
  p.inside[q] = 1;
  const int i = k1 ? ans : cell, j = k1 ? cell : ans;
  const long cq = 2 * (k1 ? nq + q : q), co = 2 * (k1 ? q : nq + q);   // centres of q / o
  p.i_ids[q] = i; p.j_ids[q] = j;
  p.centres[cq] = fxq; p.centres[cq + 1] = fyq;
  p.centres[co] = fxo; p.centres[co + 1] = fyo;
  p.win[q] = b; p.win[nq + q] = i; p.win[nq2 + q] = j;
  p.pts_qf[2 * q] = static_cast<float>(fxq) * p.s_f * sxq;
  p.pts_qf[2 * q + 1] = static_cast<float>(fyq) * p.s_f * syq;
  p.pts_oc[2 * q] = static_cast<float>(fxo) * p.s_f * sxo;
  p.pts_oc[2 * q + 1] = static_cast<float>(fyo) * p.s_f * syo;
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

// Per-pair cap on the coarse matches (match_coarse.max_matches_per_pair), between the flag pass and the compaction.
// One CTA per pair keeps the k flagged rows with the largest conf (ties at the k-th value: smaller row index first)
// and clears the other flags in place.  conf >= 0 (an exp), so its fp32 bit pattern orders as an unsigned integer:
// the k-th largest key is found by a radix select over 8-bit digits, most significant first, with a shared-memory
// histogram of the flagged rows that share the digits selected so far.  Every pass re-reads flag / conf from global
// memory (n*L*5 bytes, L2-resident), so there is no limit on L.  A pair with at most k matches exits after counting.
constexpr int kCapBlock = 1024;
__global__ void __launch_bounds__(kCapBlock) match_cap_kernel(uint8_t* __restrict__ flag,
                                                              const float* __restrict__ conf, int L, int k) {
  __shared__ int s_hist[256];
  __shared__ int s_warp[kCapBlock / 32];
  __shared__ unsigned s_prefix;
  __shared__ int s_rem;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* f = flag + static_cast<long>(blockIdx.x) * L;
  const float* c = conf + static_cast<long>(blockIdx.x) * L;

  int cnt = 0;
  for (int i = threadIdx.x; i < L; i += kCapBlock) cnt += f[i] ? 1 : 0;
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) s_warp[warp] = cnt;
  __syncthreads();
  int total = 0;
  for (int w = 0; w < kCapBlock / 32; ++w) total += s_warp[w];
  if (total <= k) return;

  // invariant: the k-th largest key starts with the digits in `prefix` (bits above `shift + 8`), and is the rem-th
  // largest of the flagged keys that start with them
  unsigned prefix = 0;
  int rem = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    const unsigned hi_mask = shift == 24 ? 0u : ~0u << (shift + 8);
    if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < L; i += kCapBlock) {
      if (f[i]) {
        const unsigned key = __float_as_uint(c[i]);
        if ((key & hi_mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 0xffu], 1);
      }
    }
    __syncthreads();
    if (warp == 0) {   // lane l scans digits 255-8l down to 248-8l; `above` counts the keys of higher digits
      const int d0 = 255 - 8 * lane;
      int sum = 0;
      for (int d = d0; d > d0 - 8; --d) sum += s_hist[d];
      int above = sum;
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, above, o);
        if (lane >= o) above += v;
      }
      above -= sum;
      for (int d = d0; d > d0 - 8; --d) {
        const int h = s_hist[d];
        if (above < rem && above + h >= rem) {   // exactly one digit of one lane satisfies this
          s_prefix = prefix | (static_cast<unsigned>(d) << shift);
          s_rem = rem - above;
        }
        above += h;
      }
    }
    __syncthreads();
    prefix = s_prefix;
    rem = s_rem;
  }

  // prefix = the k-th largest key; rem = how many rows with exactly that key are kept, the first ones in row order
  int ties_before = 0;
  for (int i0 = 0; i0 < L; i0 += kCapBlock) {
    const int i = i0 + threadIdx.x;
    bool drop = false, tie = false;
    if (i < L && f[i]) {
      const unsigned key = __float_as_uint(c[i]);
      drop = key < prefix;
      tie = key == prefix;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int rank = ties_before + __popc(bal & ((1u << lane) - 1));
    for (int w = 0; w < kCapBlock / 32; ++w) {
      if (w < warp) rank += s_warp[w];
      ties_before += s_warp[w];
    }
    if (drop || (tie && rank >= rem)) f[i] = 0;
    __syncthreads();   // s_warp is rewritten for the next chunk
  }
}

// Rectification search (DESIGN.md §20), between the flag pass and the per-pair cap: the n_pairs "pairs" of the coarse
// stage are N * K candidates, candidate c = b * K + k.  One CTA per pair b counts the flagged rows of each of its K
// candidates (counts[b * K + k]), picks the smallest k with the largest count (choice[b]; 0 when every count is 0) and
// clears the flags of the other K - 1 candidates, so that the cap and the compaction see the winner's rows only.
constexpr int kSearchBlock = 256;
__global__ void __launch_bounds__(kSearchBlock) rectify_search_kernel(uint8_t* __restrict__ flag, int L, int K,
                                                                      int* __restrict__ counts,
                                                                      long long* __restrict__ choice) {
  __shared__ int s_warp[kSearchBlock / 32];
  __shared__ int s_best;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long c0 = static_cast<long>(blockIdx.x) * K;
  int best = 0, best_cnt = -1;   // thread 0's running choice
  for (int k = 0; k < K; ++k) {
    const uint8_t* f = flag + (c0 + k) * L;
    int cnt = 0;
    for (int i = threadIdx.x; i < L; i += kSearchBlock) cnt += f[i] ? 1 : 0;
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_warp[warp] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int total = 0;
      for (int w = 0; w < kSearchBlock / 32; ++w) total += s_warp[w];
      counts[c0 + k] = total;
      if (total > best_cnt) {   // strictly larger: a tie keeps the smaller k
        best_cnt = total;
        best = k;
      }
    }
    __syncthreads();   // s_warp is rewritten for the next candidate
  }
  if (threadIdx.x == 0) {
    choice[blockIdx.x] = best;
    s_best = best;
  }
  __syncthreads();
  const int win = s_best;
  for (int k = 0; k < K; ++k) {
    if (k == win) continue;
    uint8_t* f = flag + (c0 + k) * L;
    for (int i = threadIdx.x; i < L; i += kSearchBlock) f[i] = 0;
  }
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
  const int* img_idx0;  // kIndexed: pair b reads image img_idx0[b] of feat0 / img_idx1[b] of feat1
  const int* img_idx1;
  const int* centres;   // kCentres: [2, M, 2] fine-map (x, y) window centres of side 0 / side 1
  const uint8_t* inside;  // kCentres: [M]; windows m with inside[m] == 0 are written as zeros
};
// Image of `feat0` / `feat1` that pair b's side-`side` windows are read from.
template <bool kIndexed>
__device__ __forceinline__ int fine_gather_image(const FineGatherParams& p, int side, int b) {
  return kIndexed ? (side ? p.img_idx1 : p.img_idx0)[b] : b;
}
// Window m's centre on side `side` is (step * cx, step * cy) on the fine map: step = stride and (cx, cy) the coarse
// cell of i_ids / j_ids, or (kCentres) step = 1 and (cx, cy) read from the centre table.  `answered` is false for a
// kCentres window whose query is not inside.
template <bool kCentres>
__device__ __forceinline__ void fine_gather_centre(const FineGatherParams& p, int side, long m, int& cx, int& cy,
                                                   int& step, bool& answered) {
  if (kCentres) {
    const int* c = p.centres + 2 * (side * p.M + m);
    cx = c[0];
    cy = c[1];
    step = 1;
    answered = p.inside[m] != 0;
  } else {
    const int idx = static_cast<int>(side ? p.j_ids[m] : p.i_ids[m]);
    const int wc = side ? p.w1c : p.w0c;
    cy = idx / wc;
    cx = idx - cy * wc;
    step = p.stride;
    answered = true;
  }
}
template <bool kIndexed, bool kCentres = false>
__global__ void fine_gather_kernel(const FineGatherParams p) {
  const int WW = p.W * p.W;
  const long win = blockIdx.x;             // 0 .. 2M-1
  const int side = win >= p.M ? 1 : 0;
  const long m = side ? win - p.M : win;
  if (p.live != nullptr && m >= *p.live) return;
  const int img = fine_gather_image<kIndexed>(p, side, static_cast<int>(p.b_ids[m]));
  int cx, cy, step;
  bool answered;
  fine_gather_centre<kCentres>(p, side, m, cx, cy, step, answered);
  const float* feat = side ? p.feat1 : p.feat0;
  const long sn = side ? p.sn1 : p.sn0, sc = side ? p.sc1 : p.sc0, sh = side ? p.sh1 : p.sh0,
             sw = side ? p.sw1 : p.sw0;
  const int Hf = side ? p.Hf1 : p.Hf0, Wf = side ? p.Wf1 : p.Wf0;
  for (int e = threadIdx.x; e < WW * p.Cf; e += blockDim.x) {
    const int k = e / p.Cf, c = e - k * p.Cf;
    const int ky = k / p.W, kx = k - ky * p.W;
    const int y = step * cy - p.W / 2 + ky;
    const int x = step * cx - p.W / 2 + kx;
    float v = 0.f;
    if (answered && y >= 0 && y < Hf && x >= 0 && x < Wf) v = feat[img * sn + c * sc + y * sh + x * sw];
    __half hh, ll;
    split_f16(v, hh, ll);
    const long row = win * WW + k;
    p.out_hi[row * p.ld + c] = hh;
    p.out_lo[row * p.ld + c] = ll;
  }
}

// Channel-contiguous (NHWC, sc == 1) maps with Cf % 8 == 0: one thread moves 8 channels of one window position --
// two 16-byte loads, packed split, one 16-byte store per plane (the element-wise kernel above issues 2-byte stores).
template <bool kIndexed, bool kCentres = false>
__global__ void __launch_bounds__(256) fine_gather_vec8_kernel(const FineGatherParams p) {
  const int WW = p.W * p.W;
  const int c8n = p.Cf >> 3;
  const long win = blockIdx.x;             // 0 .. 2M-1
  const int side = win >= p.M ? 1 : 0;
  const long m = side ? win - p.M : win;
  if (p.live != nullptr && m >= *p.live) return;
  const int img = fine_gather_image<kIndexed>(p, side, static_cast<int>(p.b_ids[m]));
  int cx, cy, step;
  bool answered;
  fine_gather_centre<kCentres>(p, side, m, cx, cy, step, answered);
  const float* feat = side ? p.feat1 : p.feat0;
  const long sn = side ? p.sn1 : p.sn0, sh = side ? p.sh1 : p.sh0, sw = side ? p.sw1 : p.sw0;
  const int Hf = side ? p.Hf1 : p.Hf0, Wf = side ? p.Wf1 : p.Wf0;
  for (int e = threadIdx.x; e < WW * c8n; e += blockDim.x) {
    const int k = e / c8n, c = (e - k * c8n) << 3;
    const int ky = k / p.W, kx = k - ky * p.W;
    const int y = step * cy - p.W / 2 + ky;
    const int x = step * cx - p.W / 2 + kx;
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
    if (answered && y >= 0 && y < Hf && x >= 0 && x < Wf) {
      const float4* src = reinterpret_cast<const float4*>(feat + img * sn + y * sh + x * sw + c);
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
