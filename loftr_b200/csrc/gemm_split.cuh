// Split-precision tensor-core contraction core shared by every dense product on the hot path.
//
//   D[b, m, n] = sum_k A[b, m, k] * B[b?, n, k]          (A and B both K-major, "NT" form)
//
// which is exactly the form of nn.Linear (x @ W^T; reference src/loftr/loftr_module/transformer.py:47-49,
// 51,55) and of the coarse score matrix einsum('nlc,nsc->nls') (src/loftr/utils/coarse_matching.py:109).
//
// Precision: the reference computes these products in fp32.  The mconf tolerance (rtol 1e-3 on logits
// of magnitude ~100) rules out single-pass fp16/bf16/tf32 operands (SURVEY.md §7 hard part 1), so each
// operand lives in HBM as two fp16 planes, x = hi + lo (|lo| <= ulp(hi)/2), and every k-step issues
// three wgmma (hi*hi + hi*lo + lo*hi) into one fp32 register accumulator.  The dropped lo*lo term is
// <= 2^-22 relative.
//
// Structure (one persistent CTA per SM, 288 threads: with one CTA per SM every thread may hold up to 224 registers,
// room for the 128-register accumulator next to the epilogue's working set):
//   warps 0-7  : two consumer warpgroups.  Warpgroup h issues the wgmma of the tile's column half h (M = 128 as two
//                m64 instructions, N = BLOCK_N / 2, K = 16), stages its fp32 accumulator in shared memory (row-major,
//                padded rows) and then runs the epilogue on it: thread t owns accumulator row t%128 and column half
//                t/128.  The staging area aliases the TMA ring, so the producer starts the next tile's loads only
//                once the epilogue has released it.
//   warp 8     : TMA producer    (global -> 128B-swizzled smem ring, 4 tiles per stage)
// Everything between the first wgmma of a tile and its last wait_group is warpgroup-uniform (no per-lane branches,
// every consumer thread arrives on the ring's empty barriers): otherwise ptxas serialises the asynchronous MMAs.
#pragma once
#include "ptx.cuh"

namespace lb {

constexpr int kBlockM = 128;
#ifndef LB_BLOCK_K
#define LB_BLOCK_K 64
#endif
// k-block of one pipeline stage: 64 fp16 = one 128-byte swizzle row, or 32 fp16 = one 64-byte swizzle row (twice
// as many, half as large stages in the same shared memory -> deeper TMA pipeline)
constexpr int kBlockK = LB_BLOCK_K;
static_assert(kBlockK == 64 || kBlockK == 32, "supported k-block sizes");
constexpr int kMmaK = 16;
constexpr int kGemmThreads = 288;
constexpr int kEpiThreads = 256;  // two epilogue warpgroups: rows x {left, right} half of the tile's columns
constexpr int kEpiWarp0 = 0;
constexpr int kProducerWarp = 8;
// named barrier 1 over the 256 epilogue threads (also used by the epilogues themselves)
__device__ __forceinline__ void epi_group_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Implicit-GEMM convolution mode: the A operand is an NHWC activation (fp16 planes) read through a 4-D tensor
// map; a 128-row tile is an 8 x 16 patch of output pixels and k-block kb = (tap, 64-channel block) is the same
// patch shifted by the tap offset (out-of-image reads are zero-filled by TMA = the convolution's padding).
constexpr int kConvTileH = 8;
constexpr int kConvTileW = 16;
// Channel remainder (Cin = 64*cin_blocks + r, 0 < r <= 16, e.g. 196 = 3*64 + 4): instead of a fourth, 94 % empty
// 64-channel block per tap, the r channels of every tap travel as 16-channel boxes (32-byte swizzle rows, one K = 16
// MMA step per tap); four taps share one pipeline stage ("remainder group").  K-steps per output for a 3x3 / Cin = 196
// convolution: 9*3*4 + 9 = 117 instead of 9*4*4 = 144.
constexpr int kRemChannels = 16;
constexpr int kRemTapsPerStage = 4;
struct ConvGeom {
  int enabled;     // 0: plain GEMM (3-D maps)
  int tiles_w;     // spatial tiles per tile row; m_tile = ty * tiles_w + tx
  int stride;      // 1 or 2 (also encoded as the map's element stride)
  int pad;
  int taps_w;      // kernel width
  int cin_blocks;  // full 64-channel blocks per tap
  int taps;        // kernel taps (ksize^2)
  int n_main;      // taps * cin_blocks k-blocks of 64 channels
  int rem_groups;  // 0, or ceil(taps / 4) remainder groups that follow the main k-blocks
};

struct GemmShape {
  int batches;      // independent problems along the tensor maps' 3rd dimension
  int M;            // rows of A per batch
  int N;            // rows of B per batch (= output columns)
  int K;            // multiple of 64
  int b_batched;    // 1: B has its own batch slice (score matrix); 0: B shared (weights)
  int m_tiles;      // ceil(M / 128)
  int n_tiles;      // ceil(N / BLOCK_N)
  int n_chunks;     // a work item = (batch, m_tile, chunk); chunk = tiles_per_chunk consecutive n tiles
  int tiles_per_chunk;
  ConvGeom conv;
  // optional device bound on the rows of every batch (capacity-sized buffers whose filled prefix is only known on the
  // device): rows [0, min(*live_count * live_unit_rows, M)) are computed, the m tiles past them are skipped.  nullptr:
  // all M rows.
  const int* live_count;
  int live_unit_rows;
};

// Epilogues that can never run under a device row bound (GemmShape::live_count) declare
// `static constexpr bool kNoRowBound = true;`: the kernel then compiles without the bound's code, so their register
// allocation is exactly that of an unbounded kernel.
template <class Epi, class = void>
struct EpiRowBound {
  static constexpr bool value = true;
};
template <class Epi>
struct EpiRowBound<Epi, decltype(void(Epi::kNoRowBound))> {
  static constexpr bool value = !Epi::kNoRowBound;
};

// K-major operand tile descriptor for the configured k-block (128-byte or 64-byte swizzle rows).
__device__ __forceinline__ uint64_t desc_k(uint32_t smem_addr) {
  return kBlockK == 64 ? wgmma_desc_k_sw128(smem_addr) : wgmma_desc_k_sw64(smem_addr);
}

// Shared memory: [TMA ring | accumulator staging (aliased)][epilogue area][mbarriers].
// The staging tile is 128 rows of BLOCK_N + 4 fp32: a row stride of an odd multiple of 16 bytes keeps the epilogue's
// row-per-lane 16-byte reads free of bank conflicts.  +32 floats: an epilogue's last 32-column group may run past N.
template <int BLOCK_N, int kEpiBytes = 0>
struct GemmSmem {
  static constexpr int kATile = kBlockM * kBlockK * 2;          // 16 KB per plane
  static constexpr int kBTile = BLOCK_N * kBlockK * 2;          // per plane
  static constexpr int kStageBytes = 2 * kATile + 2 * kBTile;   // hi + lo of A and B
  static constexpr int kBarBytes = 256;
  static constexpr int kAccStride = BLOCK_N + 4;                // floats
  static constexpr int kAccBytes = (kBlockM * kAccStride + 32) * 4;
  static constexpr int kFit = (232448 - kBarBytes - kEpiBytes) / kStageBytes;
  static constexpr int kWant = (192 * 1024) / kStageBytes;      // 2 (96 KB) / 3 (64 KB) / 4 (48 KB)
  static constexpr int kStages = kFit < kWant ? kFit : kWant;
  static_assert(kStages >= 2, "the TMA ring needs two stages");
  static constexpr int kRingBytes = kStages * kStageBytes > kAccBytes ? kStages * kStageBytes : kAccBytes;
};

// Epilogue contract (all methods are called by the 256 consumer threads only):
//   struct Params;                               // trivially copyable, passed by value to the kernel
//   static constexpr int kSmemBytes;             // extra dynamic smem the epilogue wants
//   __device__ Epi(const Params&, uint8_t* smem, const GemmShape&);
//   __device__ void item_begin(int batch, int m0, int chunk);
//   __device__ void prefetch(int batch, int m0, int n0);   // called before the tile's main loop: the place to pull
//                                                          // residual / bias data towards L2
//   __device__ void tile(uint32_t acc_row, int batch, int m0, int n0);   // acc_row: shared-memory address of this
//                                                                        // thread's staged accumulator row
//   __device__ void item_end(int batch, int m0, int chunk);
template <int BLOCK_N, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_split_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                  const __grid_constant__ CUtensorMap tm_ar_hi, const __grid_constant__ CUtensorMap tm_ar_lo,
                  const __grid_constant__ CUtensorMap tm_br_hi, const __grid_constant__ CUtensorMap tm_br_lo,
                  const GemmShape shape, const __grid_constant__ typename Epi::Params epi_params) {
  using S = GemmSmem<BLOCK_N, Epi::kSmemBytes>;
  constexpr int kN = BLOCK_N / 2;   // columns per consumer warpgroup
  static_assert(kN % 8 == 0, "wgmma N must be a multiple of 8");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // The swizzled tiles (ring, TMA-store staging) need a 1024-byte aligned base.  With no static shared memory the
  // dynamic window starts 1024-aligned (checked below: a misaligned base traps instead of corrupting tiles); the
  // pointers stay plain offsets of the __shared__ array -- through an integer round trip the compiler loses the
  // address space and every epilogue smem access becomes a generic LD/ST.
  uint8_t* ring = smem_raw;
  uint8_t* epi_smem = smem_raw + S::kRingBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_raw + S::kRingBytes + Epi::kSmemBytes);
  uint64_t* empty_bar = full_bar + S::kStages;
  uint64_t* acc_free = empty_bar + S::kStages;
  static_assert(Epi::kSmemBytes % 16 == 0, "epilogue area must keep the barriers aligned");
  if ((smem_u32(smem_raw) & 1023u) != 0) asm volatile("trap;");

  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below are not divergent paths
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tm_a_hi);
    tma_prefetch_desc(&tm_a_lo);
    tma_prefetch_desc(&tm_b_hi);
    tma_prefetch_desc(&tm_b_lo);
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < S::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kEpiThreads);   // every consumer thread arrives (keeps the MMA window uniform)
    }
    mbar_init(acc_free, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch (engine.cu sets the launch attribute unless LOFTR_B200_PDL=0; without it both
  // instructions are no-ops): the NEXT kernel of the stream may be scheduled as soon as every CTA of this grid got
  // here -- its CTAs take over SMs as ours exit and run their own set-up (barriers, descriptor prefetch) -- while
  // everything below this line first waits until the PREVIOUS grid has completed and flushed.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  // k-blocks of one output tile: K / 64 full blocks (+ the channel-remainder groups of a convolution)
  const int num_kb = shape.conv.enabled ? shape.conv.n_main + shape.conv.rem_groups : shape.K / kBlockK;
  constexpr int kTapBytes = S::kStageBytes / kRemTapsPerStage;   // one tap of a remainder group: A_hi A_lo B_hi B_lo
  constexpr int kRemATile = kBlockM * kRemChannels * 2;           // 4 KB
  constexpr int kRemBTile = S::kBTile / (kBlockK / kRemChannels);
  static_assert(kBlockK != 64 || (kTapBytes == 2 * kRemATile + 2 * kRemBTile && kTapBytes % 256 == 0 &&
                                  kRemBTile % 256 == 0), "remainder group layout");
  // m tiles per batch: all of them, or those that hold live rows.  The count is written by an earlier kernel of the
  // stream, so it is read only here, after griddepcontrol.wait; producer and consumers read the same value.
  int m_tiles = shape.m_tiles;
  if (EpiRowBound<Epi>::value && shape.live_count != nullptr) {
    const long live = min(static_cast<long>(max(*shape.live_count, 0)) * shape.live_unit_rows, static_cast<long>(shape.M));
    m_tiles = min(m_tiles, static_cast<int>((live + kBlockM - 1) / kBlockM));
  }
  // work items (batch, m_tile, chunk), strided over the persistent CTAs
  const int total_items = shape.batches * m_tiles * shape.n_chunks;

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      uint32_t tiles = 0;
      for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        const int chunk = item % shape.n_chunks;
        const int mt = (item / shape.n_chunks) % m_tiles;
        const int batch = item / (shape.n_chunks * m_tiles);
        const int nt_begin = chunk * shape.tiles_per_chunk;
        const int nt_end = min(nt_begin + shape.tiles_per_chunk, shape.n_tiles);
        for (int nt = nt_begin; nt < nt_end; ++nt) {
          if (tiles > 0) mbar_wait(acc_free, (tiles - 1) & 1);   // the previous tile's staged accumulator is consumed
          ++tiles;
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* st = ring + stage * S::kStageBytes;
            uint64_t* fb = &full_bar[stage];
            const bool rem_group = shape.conv.enabled && kb >= shape.conv.n_main;
            if (rem_group) {
              // ---- channel remainder: up to four taps, each a 16-channel box of A (hi, lo) and of the weights
              const ConvGeom& g = shape.conv;
              const int rem_t0 = (kb - g.n_main) * kRemTapsPerStage;
              const int rem_nt = min(kRemTapsPerStage, g.taps - rem_t0);
              mbar_arrive_expect_tx(fb, static_cast<uint32_t>(rem_nt) * kTapBytes);
              const int ty = mt / g.tiles_w, tx = mt - ty * g.tiles_w;
              for (int t = 0; t < rem_nt; ++t) {
                const int tap = rem_t0 + t;
                const int ky = tap / g.taps_w, kx = tap - ky * g.taps_w;
                const int x = tx * kConvTileW * g.stride + kx - g.pad;
                const int y = ty * kConvTileH * g.stride + ky - g.pad;
                uint8_t* base = st + t * kTapBytes;
                const int c0 = g.cin_blocks * kBlockK;
                tma_load_4d(base, &tm_ar_hi, fb, c0, x, y, batch);
                tma_load_4d(base + kRemATile, &tm_ar_lo, fb, c0, x, y, batch);
                tma_load_3d(base + 2 * kRemATile, &tm_br_hi, fb, tap * kRemChannels, nt * BLOCK_N, 0);
                tma_load_3d(base + 2 * kRemATile + kRemBTile, &tm_br_lo, fb, tap * kRemChannels, nt * BLOCK_N, 0);
              }
            } else {
              mbar_arrive_expect_tx(fb, S::kStageBytes);
              // ---- A: 128 rows (or an 8 x 16 pixel patch shifted by the tap)
              if (shape.conv.enabled) {
                const ConvGeom& g = shape.conv;
                const int tap = kb / g.cin_blocks, cb = kb - tap * g.cin_blocks;
                const int ky = tap / g.taps_w, kx = tap - ky * g.taps_w;
                const int ty = mt / g.tiles_w, tx = mt - ty * g.tiles_w;
                const int x = tx * kConvTileW * g.stride + kx - g.pad;
                const int y = ty * kConvTileH * g.stride + ky - g.pad;
                tma_load_4d(st, &tm_a_hi, fb, cb * kBlockK, x, y, batch);
                tma_load_4d(st + S::kATile, &tm_a_lo, fb, cb * kBlockK, x, y, batch);
              } else {
                tma_load_3d(st, &tm_a_hi, fb, kb * kBlockK, mt * kBlockM, batch);
                tma_load_3d(st + S::kATile, &tm_a_lo, fb, kb * kBlockK, mt * kBlockM, batch);
              }
              // ---- B
              const int bb = shape.b_batched ? batch : 0;
              tma_load_3d(st + 2 * S::kATile, &tm_b_hi, fb, kb * kBlockK, nt * BLOCK_N, bb);
              tma_load_3d(st + 2 * S::kATile + S::kBTile, &tm_b_lo, fb, kb * kBlockK, nt * BLOCK_N, bb);
            }
            if (++stage == S::kStages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups: wgmma + epilogue
    const int ct = threadIdx.x - kEpiWarp0 * 32;   // 0..255
    const int h = ct >> 7;                          // column half of the tile
    const int wt = ct & 127;                        // thread within the warpgroup
    Epi epi(epi_params, epi_smem, shape);
    float acc[2][kN / 2];                           // rows [0, 64) and [64, 128) of this warpgroup's column half
    float* stg = reinterpret_cast<float*>(ring);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const int chunk = item % shape.n_chunks;
      const int mt = (item / shape.n_chunks) % m_tiles;
      const int batch = item / (shape.n_chunks * m_tiles);
      const int nt_begin = chunk * shape.tiles_per_chunk;
      const int nt_end = min(nt_begin + shape.tiles_per_chunk, shape.n_tiles);
      epi.item_begin(batch, mt * kBlockM, chunk);
      for (int nt = nt_begin; nt < nt_end; ++nt) {
        epi.prefetch(batch, mt * kBlockM, nt * BLOCK_N);
        // a zeroed accumulator instead of a first MMA with scale-d = 0: the previous tile's values are dead after
        // staging, so the epilogue does not have to keep them in registers
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) acc[0][i] = acc[1][i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t st = smem_u32(ring + stage * S::kStageBytes);
          wgmma_fence();
          if (shape.conv.enabled && kb >= shape.conv.n_main) {
            // remainder group: one K = 16 step per tap, 32-byte swizzle rows (kb > 0 here: always accumulate)
            const int rem_t0 = (kb - shape.conv.n_main) * kRemTapsPerStage;
            const int rem_nt = min(kRemTapsPerStage, shape.conv.taps - rem_t0);
            for (int t = 0; t < rem_nt; ++t) {
              const uint32_t base = st + t * kTapBytes;
              const uint32_t b_off = static_cast<uint32_t>(h * kN * kRemChannels * 2);
#pragma unroll
              for (int mh = 0; mh < 2; ++mh) {
                const uint32_t a_off = static_cast<uint32_t>(mh * 64 * kRemChannels * 2);
                const uint64_t ra_hi = wgmma_desc_k_sw32(base + a_off);
                const uint64_t ra_lo = wgmma_desc_k_sw32(base + kRemATile + a_off);
                const uint64_t rb_hi = wgmma_desc_k_sw32(base + 2 * kRemATile + b_off);
                const uint64_t rb_lo = wgmma_desc_k_sw32(base + 2 * kRemATile + kRemBTile + b_off);
                wgmma_f16<kN>(acc[mh], ra_hi, rb_hi, 1u);
                wgmma_f16<kN>(acc[mh], ra_hi, rb_lo, 1u);
                wgmma_f16<kN>(acc[mh], ra_lo, rb_hi, 1u);
              }
            }
          } else {
            const uint32_t b_off = static_cast<uint32_t>(h * kN * kBlockK * 2);
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
              const uint32_t a_off = static_cast<uint32_t>(mh * 64 * kBlockK * 2);
              const uint64_t da_hi = desc_k(st + a_off);
              const uint64_t da_lo = desc_k(st + S::kATile + a_off);
              const uint64_t db_hi = desc_k(st + 2 * S::kATile + b_off);
              const uint64_t db_lo = desc_k(st + 2 * S::kATile + S::kBTile + b_off);
#pragma unroll
              for (int k = 0; k < kBlockK / kMmaK; ++k) {
                // advance 16 fp16 = 32 bytes along K inside the swizzle row: +2 in 16-byte units
                const uint64_t adv = static_cast<uint64_t>(k * 2);
                wgmma_f16<kN>(acc[mh], da_hi + adv, db_hi + adv, 1u);
                wgmma_f16<kN>(acc[mh], da_hi + adv, db_lo + adv, 1u);
                wgmma_f16<kN>(acc[mh], da_lo + adv, db_hi + adv, 1u);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous k-block's MMAs are done: its slot may be refilled
          if (prev >= 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == S::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        mbar_arrive(&empty_bar[prev]);
        // ---- stage the accumulator (row-major) over the ring, once both warpgroups' MMAs have read it
        epi_group_sync();
        {
          const int r0 = 16 * (wt >> 5) + ((wt & 31) >> 2);
          const int c0 = h * kN + 2 * (wt & 3);
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
            for (int j = 0; j < kN / 8; ++j) {
              float* p = stg + (mh * 64 + r0) * S::kAccStride + c0 + 8 * j;
              *reinterpret_cast<float2*>(p) = make_float2(acc[mh][4 * j], acc[mh][4 * j + 1]);
              *reinterpret_cast<float2*>(p + 8 * S::kAccStride) = make_float2(acc[mh][4 * j + 2], acc[mh][4 * j + 3]);
            }
          }
        }
        epi_group_sync();
        epi.tile(smem_u32(stg + (ct & 127) * S::kAccStride), batch, mt * kBlockM, nt * BLOCK_N);
        fence_proxy_async();   // staging reads / writes (generic proxy) before the next TMA writes into the ring
        epi_group_sync();
        if (ct == 0) mbar_arrive(acc_free);
      }
      epi.item_end(batch, mt * kBlockM, chunk);
    }
    tma_store_wait_all();   // bulk stores issued by this thread (if any) have landed before the CTA may exit
  }
}

}  // namespace lb
