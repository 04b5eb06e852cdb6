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
//                t/128.  The staging area aliases the GemmSmem::kAccStages consecutive ring stages the tile consumed
//                last (GemmSmem::staging_first), so the producer loads the next tile into the other stages while the
//                epilogue runs and waits for the epilogue's release (acc_free) only before it writes a staged one.
//   warp 8     : TMA producer    (global -> swizzled smem ring; a stage holds the A and B tiles, hi and lo planes)
// A ring stage holds GemmSmem::kBK of K: 32 (64-byte swizzle rows) with two planes, 64 (128-byte swizzle rows) with one,
// so a stage is as large either way and 4-6 stages are in flight.  The k16 MMAs run in the same k order at any stage
// depth, so the stage depth does not change a bit of the result.
// Everything between the first wgmma of a tile and its last wait_group is warpgroup-uniform (no per-lane branches,
// every consumer thread arrives on the ring's empty barriers): otherwise ptxas serialises the asynchronous MMAs.
#pragma once
#include "ptx.cuh"

namespace lb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // granularity of K (and of a convolution's channel blocks): 64 fp16 = one 128-byte row
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
// MMA step per tap); GemmSmem::kRemTapsPerStage taps (2 with two planes, 4 with one) share one pipeline stage
// ("remainder group").  K-steps per output for a 3x3 / Cin = 196 convolution: 9*3*4 + 9 = 117 instead of 9*4*4 = 144.
constexpr int kRemChannels = 16;
struct ConvGeom {
  int enabled;     // 0: plain GEMM (3-D maps)
  int tiles_w;     // spatial tiles per tile row; m_tile = ty * tiles_w + tx
  int stride;      // 1 or 2 (also encoded as the map's element stride)
  int pad;
  int taps_w;      // kernel width
  int cin_blocks;  // full 64-channel blocks per tap
  int taps;        // kernel taps (ksize^2)
  int n_main;      // taps * cin_blocks k-blocks of 64 channels
  int rem_groups;  // 0, or the remainder groups (ceil(taps / kRemTapsPerStage)) that follow the main k-blocks
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

// Operand planes of a tensor-core kernel, declared by its epilogue: 2 (the default) = split precision, hi and lo planes
// of A and B and three MMAs per k-step; an epilogue that declares `static constexpr int kOperandPlanes = 1;` runs the
// kernel on single fp16 planes with one MMA per k-step (the fp16 backbone, EpiConvF16).  The ring then carries the hi
// planes only and every stage is half as large.
template <class Epi, class = void>
struct EpiOperandPlanes {
  static constexpr int value = 2;
};
template <class Epi>
struct EpiOperandPlanes<Epi, decltype(void(Epi::kOperandPlanes))> {
  static constexpr int value = Epi::kOperandPlanes;
  static_assert(value == 1 || value == 2, "operands are one or two fp16 planes");
};

// K-major operand tile descriptor of a ring stage holding kBK of K: rows of 128 bytes (kBK = 64, 128-byte swizzle) or
// 64 bytes (kBK = 32, 64-byte swizzle).
template <int kBK>
__device__ __forceinline__ uint64_t desc_k(uint32_t smem_addr) {
  static_assert(kBK == 32 || kBK == 64, "a stage holds 32 or 64 of K");
  return kBK == 64 ? wgmma_desc_k_sw128(smem_addr) : wgmma_desc_k_sw64(smem_addr);
}

// Dynamic shared memory a block may opt in to on the H100 (227 KB).
constexpr int kSmemLimit = 232448;

// Accumulator staging of the persistent kernels (gemm_split_kernel, conv3x3_halo_kernel): 128 rows of BLOCK_N + 4 fp32
// over the dead ring.  A row stride of an odd multiple of 16 bytes keeps the epilogue's row-per-lane 16-byte reads free
// of bank conflicts.  +32 floats: an epilogue's last 32-column group may run past N.
__host__ __device__ constexpr int acc_stride(int block_n) { return block_n + 4; }   // floats
__host__ __device__ constexpr int acc_bytes(int block_n) { return (kBlockM * acc_stride(block_n) + 32) * 4; }

// Shared memory: [TMA ring (the accumulator staging aliases kAccStages consecutive stages)][epilogue area][mbarriers].
// A stage holds kBK of K: 32 with two planes (64-byte swizzle rows), 64 with one, so the stages are as large either way
// and the ring of about 192 KB holds 6 / 4 / 4 of them at N = 128 / 208 / 256 (32 / 42 / 48 KB each).  The staged
// accumulator (acc_bytes) covers 3 of them at every N, which leaves 3 / 1 / 1 stages to the producer while the
// epilogue runs.
template <int BLOCK_N, int kEpiBytes = 0, int kPlanes = 2>
struct GemmSmem {
  static constexpr int kBK = kPlanes == 2 ? kBlockK / 2 : kBlockK;
  static constexpr int kATile = kBlockM * kBK * 2;              // per plane
  static constexpr int kBTile = BLOCK_N * kBK * 2;              // per plane
  static constexpr int kStageBytes = kPlanes * (kATile + kBTile);   // hi (+ lo) of A and B
  static constexpr int kBarBytes = 256;
  static constexpr int kAccBytes = acc_bytes(BLOCK_N);
  static constexpr int kFit = (kSmemLimit - kBarBytes - kEpiBytes) / kStageBytes;
  static constexpr int kWant = (192 * 1024) / kStageBytes;
  static constexpr int kStages = kFit < kWant ? kFit : kWant;
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kAccStages = (kAccBytes + kStageBytes - 1) / kStageBytes;   // stages the staging covers
  static_assert(kAccStages < kStages, "the ring needs a stage beside the staged accumulator");
  static_assert((2 * kStages + 1) * 8 <= kBarBytes, "barrier area");
  // channel remainder: one tap = a 16-channel box of A and of B per plane; kBK / 16 taps per stage
  static constexpr int kRemATile = kBlockM * kRemChannels * 2;   // 4 KB
  static constexpr int kRemBTile = BLOCK_N * kRemChannels * 2;
  static constexpr int kTapBytes = kPlanes * (kRemATile + kRemBTile);
  static constexpr int kRemTapsPerStage = kStageBytes / kTapBytes;
  static_assert(kRemTapsPerStage * kTapBytes == kStageBytes && kTapBytes % 256 == 0 && kRemBTile % 256 == 0,
                "remainder group layout");

  // First ring stage of the staged accumulator of a tile whose last k-stage was in ring stage `last`: the kAccStages
  // stages that end at `last`, so the stages that follow it in ring order (where the next tile's loads go) stay free.
  // When those would wrap around the ring's end, the last kAccStages stages of the ring, the farthest from last + 1.
  // Producer and consumers both place the staging with this function.
  __host__ __device__ static constexpr int staging_first(int last) {
    return last >= kAccStages - 1 ? last - kAccStages + 1 : kStages - kAccStages;
  }
  __host__ __device__ static constexpr bool staged_over(int first, int stage) {
    return stage >= first && stage < first + kAccStages;
  }
};

// ---- pieces shared by the persistent kernels (gemm_split_kernel, conv3x3_halo_kernel)

// Set-up: traps on a misaligned shared-memory base, prefetches the four main tensor-map descriptors, initialises the
// ring barriers, the kernel's own barriers (init_more) and acc_free, then triggers the next grid and waits for the
// previous one.  Returns the warp index broadcast from lane 0: provably warp-uniform, so the role branches on it are
// not divergent paths.
template <int kStages, class InitMore>
__device__ __forceinline__ int persistent_setup(const uint8_t* smem_raw, const CUtensorMap* tm_a_hi,
                                                const CUtensorMap* tm_a_lo, const CUtensorMap* tm_b_hi,
                                                const CUtensorMap* tm_b_lo, uint64_t* full_bar, uint64_t* empty_bar,
                                                uint64_t* acc_free, InitMore init_more) {
  if ((smem_u32(smem_raw) & 1023u) != 0) asm volatile("trap;");
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(tm_a_hi);
    tma_prefetch_desc(tm_a_lo);
    tma_prefetch_desc(tm_b_hi);
    tma_prefetch_desc(tm_b_lo);
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kEpiThreads);   // every consumer thread arrives (keeps the MMA window uniform)
    }
    init_more();
    mbar_init(acc_free, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch (engine.cu sets the launch attribute unless LOFTR_B200_PDL=0): the next kernel's CTAs
  // take over SMs as ours exit and run their own set-up, while everything after this waits for the previous grid.
  pdl_trigger();
  pdl_wait();
  return warp;
}

// Work item `item` = (batch, m tile, chunk of consecutive n tiles); items are strided over the persistent CTAs.
struct WorkItem {
  int batch, mt, chunk, nt_begin, nt_end;
};
__device__ __forceinline__ WorkItem work_item(const GemmShape& s, int m_tiles, int item) {
  WorkItem w;
  w.chunk = item % s.n_chunks;
  w.mt = (item / s.n_chunks) % m_tiles;
  w.batch = item / (s.n_chunks * m_tiles);
  w.nt_begin = w.chunk * s.tiles_per_chunk;
  w.nt_end = min(w.nt_begin + s.tiles_per_chunk, s.n_tiles);
  return w;
}

// Stores an m64nN accumulator (wgmma_f16 fragment layout) row-major with a row stride of `stride` floats: thread t of
// the warpgroup holds rows row0 + 2 step (t / 32) + (t % 32) / 4 and that + step, columns col0 + 8 j + 2 (t % 4) (+1).
template <int N>
__device__ __forceinline__ void stage_acc(float* stg, int stride, const float (&acc)[N / 2], int row0, int step,
                                          int col0) {
  const int t = threadIdx.x & 127;
  const int r = 2 * step * (t >> 5) + ((t & 31) >> 2);
  const int c = col0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    float* p = stg + (row0 + r) * stride + c + 8 * j;
    *reinterpret_cast<float2*>(p) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(p + step * stride) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// Tile end of a consumer thread, after the tile's last wgmma_commit: drain the MMAs, release the ring slots they read
// (release_ring), stage the accumulator at `stg` (stage) once both warpgroups' MMAs are done with the ring, run the
// epilogue on this thread's staged row and hand the staging memory back to the producer (acc_free).  `stg` must be
// memory the producer does not write before acc_free: gemm_split_kernel's producer keeps off the kAccStages ring stages
// from GemmSmem::staging_first until then, conv3x3_halo_kernel's off its whole weight ring (and the halo slots when the
// staging reaches into them).
template <int BLOCK_N, class Epi, class Acc, class Release, class Stage>
__device__ __forceinline__ void finish_tile(Epi& epi, Acc& acc, Release release_ring, Stage stage, const float* stg,
                                            int ct, uint64_t* acc_free, int batch, int m0, int n0) {
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  release_ring();
  epi_group_sync();
  stage();
  epi_group_sync();
  epi.tile(smem_u32(stg + (ct & 127) * acc_stride(BLOCK_N)), batch, m0, n0);
  fence_proxy_async();   // staging reads / writes (generic proxy) before the next TMA writes over them
  epi_group_sync();
  if (ct == 0) mbar_arrive(acc_free);
}

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
  constexpr int kPlanes = EpiOperandPlanes<Epi>::value;   // 1: single fp16 planes, one MMA per k-step
  using S = GemmSmem<BLOCK_N, Epi::kSmemBytes, kPlanes>;
  constexpr int kN = BLOCK_N / 2;   // columns per consumer warpgroup
  static_assert(kN % 8 == 0, "wgmma N must be a multiple of 8");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // The swizzled tiles (ring, TMA-store staging) need a 1024-byte aligned base.  With no static shared memory the
  // dynamic window starts 1024-aligned (checked in persistent_setup: a misaligned base traps instead of corrupting
  // tiles); the pointers stay plain offsets of the __shared__ array -- through an integer round trip the compiler loses
  // the address space and every epilogue smem access becomes a generic LD/ST.
  uint8_t* ring = smem_raw;
  uint8_t* epi_smem = smem_raw + S::kRingBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_raw + S::kRingBytes + Epi::kSmemBytes);
  uint64_t* empty_bar = full_bar + S::kStages;
  uint64_t* acc_free = empty_bar + S::kStages;
  static_assert(Epi::kSmemBytes % 16 == 0, "epilogue area must keep the barriers aligned");
  const int warp = persistent_setup<S::kStages>(smem_raw, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, full_bar, empty_bar,
                                                acc_free, [] {});
  const int lane = threadIdx.x & 31;

  // k-stages (ring stages) of one output tile: K / kBK (+ the channel-remainder groups of a convolution).  A stage of
  // the main loop is part j of k-block ks / kSubs (64 of K: a convolution's (tap, 64-channel block)), K offset ks * kBK.
  constexpr int kBK = S::kBK;
  constexpr int kSubs = kBlockK / kBK;
  const int n_main = shape.conv.enabled ? shape.conv.n_main * kSubs : shape.K / kBK;
  const int num_ks = n_main + (shape.conv.enabled ? shape.conv.rem_groups : 0);
  constexpr int kTapBytes = S::kTapBytes;   // one tap of a remainder group: A_hi (A_lo) B_hi (B_lo)
  constexpr int kRemATile = S::kRemATile;
  constexpr int kRemBTile = S::kRemBTile;
  constexpr int kRemTapsPerStage = S::kRemTapsPerStage;
  // m tiles per batch: all of them, or those that hold live rows.  The count is written by an earlier kernel of the
  // stream, so it is read only here, after griddepcontrol.wait; producer and consumers read the same value.
  int m_tiles = shape.m_tiles;
  if (EpiRowBound<Epi>::value && shape.live_count != nullptr) {
    const long live = min(static_cast<long>(max(*shape.live_count, 0)) * shape.live_unit_rows, static_cast<long>(shape.M));
    m_tiles = min(m_tiles, static_cast<int>((live + kBlockM - 1) / kBlockM));
  }
  const int total_items = shape.batches * m_tiles * shape.n_chunks;

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      RingPos<S::kStages> pos;
      uint32_t tiles = 0;
      int staged = -1;   // first ring stage of the previous tile's staged accumulator until acc_free is waited on
      for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        const WorkItem w = work_item(shape, m_tiles, item);
        for (int nt = w.nt_begin; nt < w.nt_end; ++nt) {
          int last = 0;
          for (int ks = 0; ks < num_ks; ++ks) {
            // The previous tile's epilogue must release its staging before a stage under it is refilled.  The wait
            // comes at the latest before this tile's last load: the consumers cannot finish this tile before it, so
            // acc_free never runs two phases ahead of the parity waited on.
            if (staged >= 0 && (S::staged_over(staged, pos.stage) || ks == num_ks - 1)) {
              mbar_wait(acc_free, (tiles - 1) & 1);
              staged = -1;
            }
            mbar_wait(&empty_bar[pos.stage], pos.phase ^ 1);
            uint8_t* st = ring + pos.stage * S::kStageBytes;
            uint64_t* fb = &full_bar[pos.stage];
            const bool rem_group = ks >= n_main;
            if (rem_group) {
              // ---- channel remainder: up to kRemTapsPerStage taps, each a 16-channel box of A (hi, lo) and of the
              // weights
              const ConvGeom& g = shape.conv;
              const int rem_t0 = (ks - n_main) * kRemTapsPerStage;
              const int rem_nt = min(kRemTapsPerStage, g.taps - rem_t0);
              mbar_arrive_expect_tx(fb, static_cast<uint32_t>(rem_nt) * kTapBytes);
              const int ty = w.mt / g.tiles_w, tx = w.mt - ty * g.tiles_w;
              for (int t = 0; t < rem_nt; ++t) {
                const int tap = rem_t0 + t;
                const int ky = tap / g.taps_w, kx = tap - ky * g.taps_w;
                const int x = tx * kConvTileW * g.stride + kx - g.pad;
                const int y = ty * kConvTileH * g.stride + ky - g.pad;
                uint8_t* base = st + t * kTapBytes;
                const int c0 = g.cin_blocks * kBlockK;
                tma_load_4d(base, &tm_ar_hi, fb, c0, x, y, w.batch);
                if constexpr (kPlanes == 2) tma_load_4d(base + kRemATile, &tm_ar_lo, fb, c0, x, y, w.batch);
                tma_load_3d(base + kPlanes * kRemATile, &tm_br_hi, fb, tap * kRemChannels, nt * BLOCK_N, 0);
                if constexpr (kPlanes == 2)
                  tma_load_3d(base + 2 * kRemATile + kRemBTile, &tm_br_lo, fb, tap * kRemChannels, nt * BLOCK_N, 0);
              }
            } else {
              mbar_arrive_expect_tx(fb, S::kStageBytes);
              // ---- A: 128 rows (or an 8 x 16 pixel patch shifted by the tap)
              const int k0 = ks * kBK;
              if (shape.conv.enabled) {
                const ConvGeom& g = shape.conv;
                const int kb = ks / kSubs;
                const int tap = kb / g.cin_blocks, cb = kb - tap * g.cin_blocks;
                const int ky = tap / g.taps_w, kx = tap - ky * g.taps_w;
                const int ty = w.mt / g.tiles_w, tx = w.mt - ty * g.tiles_w;
                const int x = tx * kConvTileW * g.stride + kx - g.pad;
                const int y = ty * kConvTileH * g.stride + ky - g.pad;
                const int c0 = cb * kBlockK + (ks - kb * kSubs) * kBK;
                tma_load_4d(st, &tm_a_hi, fb, c0, x, y, w.batch);
                if constexpr (kPlanes == 2) tma_load_4d(st + S::kATile, &tm_a_lo, fb, c0, x, y, w.batch);
              } else {
                tma_load_3d(st, &tm_a_hi, fb, k0, w.mt * kBlockM, w.batch);
                if constexpr (kPlanes == 2) tma_load_3d(st + S::kATile, &tm_a_lo, fb, k0, w.mt * kBlockM, w.batch);
              }
              // ---- B (a convolution's weight planes hold k-block (tap, cb) at (tap * cin_blocks + cb) * 64)
              const int bb = shape.b_batched ? w.batch : 0;
              tma_load_3d(st + kPlanes * S::kATile, &tm_b_hi, fb, k0, nt * BLOCK_N, bb);
              if constexpr (kPlanes == 2)
                tma_load_3d(st + 2 * S::kATile + S::kBTile, &tm_b_lo, fb, k0, nt * BLOCK_N, bb);
            }
            last = pos.stage;
            pos.advance();
          }
          staged = S::staging_first(last);
          ++tiles;
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups: wgmma + epilogue
    const int ct = threadIdx.x - kEpiWarp0 * 32;   // 0..255
    const int h = ct >> 7;                          // column half of the tile
    Epi epi(epi_params, epi_smem, shape);
    float acc[2][kN / 2];                           // rows [0, 64) and [64, 128) of this warpgroup's column half
    RingPos<S::kStages> pos;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const WorkItem w = work_item(shape, m_tiles, item);
      epi.item_begin(w.batch, w.mt * kBlockM, w.chunk);
      for (int nt = w.nt_begin; nt < w.nt_end; ++nt) {
        epi.prefetch(w.batch, w.mt * kBlockM, nt * BLOCK_N);
        // a zeroed accumulator instead of a first MMA with scale-d = 0: the previous tile's values are dead after
        // staging, so the epilogue does not have to keep them in registers
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) acc[0][i] = acc[1][i] = 0.f;
        int prev = -1;
        for (int ks = 0; ks < num_ks; ++ks) {
          mbar_wait(&full_bar[pos.stage], pos.phase);
          const uint32_t st = smem_u32(ring + pos.stage * S::kStageBytes);
          wgmma_fence();
          if (ks >= n_main) {
            // remainder group: one K = 16 step per tap, 32-byte swizzle rows (ks > 0 here: always accumulate)
            const int rem_t0 = (ks - n_main) * kRemTapsPerStage;
            const int rem_nt = min(kRemTapsPerStage, shape.conv.taps - rem_t0);
            for (int t = 0; t < rem_nt; ++t) {
              const uint32_t base = st + t * kTapBytes;
              const uint32_t b_off = static_cast<uint32_t>(h * kN * kRemChannels * 2);
#pragma unroll
              for (int mh = 0; mh < 2; ++mh) {
                const uint32_t a_off = static_cast<uint32_t>(mh * 64 * kRemChannels * 2);
                const uint64_t ra_hi = wgmma_desc_k_sw32(base + a_off);
                const uint64_t ra_lo = wgmma_desc_k_sw32(base + kRemATile + a_off);
                const uint64_t rb_hi = wgmma_desc_k_sw32(base + kPlanes * kRemATile + b_off);
                const uint64_t rb_lo = wgmma_desc_k_sw32(base + 2 * kRemATile + kRemBTile + b_off);
                wgmma_split<kN, kPlanes>(acc[mh], ra_hi, ra_lo, rb_hi, rb_lo);
              }
            }
          } else {
            const uint32_t b_off = static_cast<uint32_t>(h * kN * kBK * 2);
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
              const uint32_t a_off = static_cast<uint32_t>(mh * 64 * kBK * 2);
              const uint64_t da_hi = desc_k<kBK>(st + a_off);
              const uint64_t da_lo = desc_k<kBK>(st + S::kATile + a_off);
              const uint64_t db_hi = desc_k<kBK>(st + kPlanes * S::kATile + b_off);
              const uint64_t db_lo = desc_k<kBK>(st + 2 * S::kATile + S::kBTile + b_off);
#pragma unroll
              for (int k = 0; k < kBK / kMmaK; ++k) {
                // advance 16 fp16 = 32 bytes along K inside the swizzle row: +2 in 16-byte units
                const uint64_t adv = static_cast<uint64_t>(k * 2);
                wgmma_split<kN, kPlanes>(acc[mh], da_hi + adv, da_lo + adv, db_hi + adv, db_lo + adv);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous k-stage's MMAs are done: its slot may be refilled
          if (prev >= 0) mbar_arrive(&empty_bar[prev]);
          prev = pos.stage;
          pos.advance();
        }
        float* stg = reinterpret_cast<float*>(ring + S::staging_first(prev) * S::kStageBytes);
        finish_tile<BLOCK_N>(
            epi, acc, [&] { mbar_arrive(&empty_bar[prev]); },
            [&] {
              stage_acc<kN>(stg, acc_stride(BLOCK_N), acc[0], 0, 8, h * kN);
              stage_acc<kN>(stg, acc_stride(BLOCK_N), acc[1], 64, 8, h * kN);
            },
            stg, ct, acc_free, w.batch, w.mt * kBlockM, nt * BLOCK_N);
      }
      epi.item_end(w.batch, w.mt * kBlockM, w.chunk);
    }
    tma_store_wait_all();   // bulk stores issued by this thread (if any) have landed before the CTA may exit
  }
}

}  // namespace lb
