// Stride-1 3x3 convolution on the split-precision core with the input patch resident in shared memory.
//
// gemm_split_kernel's convolution mode loads one 8 x 16 pixel patch per (tap, 64-channel block), so the nine taps of a
// 3x3 convolution bring every input pixel from L2 to shared memory 6.4 times (1,152 pixels for a 10 x 18 patch of 180).
// Here the producer loads the 10 x 18 halo of an output tile once per channel block and the nine taps become nine
// shifted shared-memory descriptors over it; only the weights stream through the per-tap pipeline ring.
//
// Halo layout (wgmma no-swizzle K-major core matrices): [8-channel chunk][halo pixel (row-major, 18 wide)][16 bytes].
// Consumer warpgroup h computes x-half h of the 8 x 16 tile (output rows y = 0..7, columns x = 8h..8h+7) over all
// BLOCK_N channels: one m64nBLOCK_Nk16 instruction per product and k-step, so each A core matrix is read by one
// warpgroup and a 196-channel output runs as a 200-wide tile (200 / 2 is no wgmma N).  For tap (ky, kx) the
// instruction's 8-row group y is the 8 consecutive halo pixels from (y + ky) * 18 + 8 * h + kx -- one 128-byte core
// matrix -- so
//   start = ((ky * 18) + 8 * h + kx) * 16,   SBO = 18 * 16 (next y),   LBO = chunk stride (next 8 channels along K),
// and k-step k of a 64-channel block starts 2k chunks further.  Row r of warpgroup h is therefore tile pixel
// (r / 8) * 16 + 8 * h + r % 8; the accumulator is staged row-major by pixel, exactly as gemm_split_kernel stages it,
// so the epilogue (EpiConv) is unchanged.
//
// Each halo plane is loaded as eight 8-channel boxes of a 4-D NHWC map whose channel extent is Cin: TMA zero-fills
// the image border (the padding) and every channel at or past Cin, so the row-stride padding of a Cin = 196 plane
// (channels 196..199 are never written) cannot reach the MMAs.  Chunks sit 2,944 bytes apart (2,880 rounded up to the
// 128-byte alignment of a TMA destination).
//
// K order: with at most two halos per tile (Cin <= 128) both stay resident and the taps run tap-major, the order of
// gemm_split_kernel's convolution mode, so those layers produce the same bits.  Wider inputs run channel-block-major
// (nine taps per halo, the next block's halo loading into the other slot meanwhile); the channel remainder
// (Cin = 64 * cin_blocks + r, r <= 16) is a last 16-channel halo with one K = 16 step per tap.
//
// Warp roles, the epilogue contract, the set-up, the work split and the tile end (drain, accumulator staging over the
// dead ring / halo memory, epilogue, hand-off) are gemm_split.cuh's shared pieces.  Where the staging fits in the
// weight ring (N = 128) the next tile's first halos load while the epilogue runs.
#pragma once
#include "gemm_split.cuh"

namespace lb {

constexpr int kHaloW = kConvTileW + 2;
constexpr int kHaloH = kConvTileH + 2;
constexpr int kHaloChunkBytes = 2944;                      // 180 pixels x 16 bytes = 2,880, 128-byte aligned
constexpr int kHaloPlaneBytes = (kBlockK / 8) * kHaloChunkBytes;
constexpr int kHaloTaps = 9;
static_assert(kHaloW * kHaloH * 16 <= kHaloChunkBytes && kHaloChunkBytes % 128 == 0, "halo chunk layout");

// Shared memory: [weight ring | two halo slots (accumulator staging aliases both)][epilogue area][mbarriers].
// A weight stage is one tap of a 64-channel block (kBK = 64, 128-byte swizzle rows) when three of them fit beside the
// halo slots, else half a tap (kBK = 32, 64-byte swizzle rows): three or more stages in flight at every N.  N = 200
// gets four stages of 25,600 bytes because EpiConv<200> shares the residual transposer with the TMA-store staging
// (EpiConv::kOwnXpose): its own transposer would take the fourth stage, and three stages made the 196-channel
// layers 13-14 % slower on an H100 at 700 W.
// With single fp16 planes (kPlanes = 1: EpiConvF16) the halo slots and the weight stages are half as large and the same
// rule gives kBK = 64 and 6 / 5 / 4 stages at N = 128 / 200 / 256 (two planes: 3 / 4 / 3).
template <int BLOCK_N, int kEpiBytes, int kPlanes = 2>
struct HaloSmem {
  static constexpr int kHaloSlotBytes = kPlanes * kHaloPlaneBytes;   // hi (+ lo) planes of one channel block
  static constexpr int kBarBytes = 256;
  static constexpr int kFree = kSmemLimit - kBarBytes - kEpiBytes - 2 * kHaloSlotBytes;
  static constexpr int kBK = kFree / (kPlanes * BLOCK_N * kBlockK * 2) >= 3 ? kBlockK : kBlockK / 2;
  static constexpr int kBTile = BLOCK_N * kBK * 2;        // per plane
  static constexpr int kStageBytes = kPlanes * kBTile;
  static constexpr int kStages = kFree / kStageBytes < 6 ? kFree / kStageBytes : 6;
  static_assert(kStages >= 3, "the weight ring needs three stages");
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kAccBytes = acc_bytes(BLOCK_N);
  static constexpr int kMainBytes = kRingBytes + 2 * kHaloSlotBytes;
  static_assert(kMainBytes >= kAccBytes && kMainBytes % 1024 == 0 && kRingBytes % 1024 == 0, "halo smem layout");
  static constexpr int kTotalBytes = kMainBytes + kEpiBytes + kBarBytes;
};

// No-swizzle K-major descriptor: lbo / sbo = byte distance between core matrices adjacent along K / along M or N.
__device__ __forceinline__ uint64_t wgmma_desc_k_noswz(uint32_t a, uint32_t lbo, uint32_t sbo) {
  uint64_t d = static_cast<uint64_t>((a >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(lbo >> 4) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  return d;
}

// tm_a_*: 4-D NHWC maps (C = Cin, W, H, N), box 8 channels x 18 x 10 x 1, no swizzle.
// tm_b_*: main weight planes [Cout, 9 * cin_blocks * 64], box kBK x BLOCK_N.  tm_br_*: remainder weight planes
// [Cout, 9 * 16], box 16 x BLOCK_N (copies of tm_b_* when Cin has no remainder).
// shape.conv: tiles_w, cin_blocks and rem_groups (> 0: a channel remainder) are read; stride 1, pad 1 are implied.
template <int BLOCK_N, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                    const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                    const __grid_constant__ CUtensorMap tm_br_hi, const __grid_constant__ CUtensorMap tm_br_lo,
                    const GemmShape shape, const __grid_constant__ typename Epi::Params epi_params) {
  constexpr int kPlanes = EpiOperandPlanes<Epi>::value;   // 1: single fp16 planes, one MMA per k-step
  using S = HaloSmem<BLOCK_N, Epi::kSmemBytes, kPlanes>;
  constexpr int kHaloSlotBytes = S::kHaloSlotBytes;
  constexpr int kBK = S::kBK;
  constexpr int kSubs = kBlockK / kBK;                       // weight stages per (tap, 64-channel block)
  constexpr int kRemBTile = BLOCK_N * kRemChannels * 2;      // per plane
  constexpr bool kStagingInRing = S::kAccBytes <= S::kRingBytes;   // N = 128: the halo slots stay free at the tile end
  static_assert(BLOCK_N % 8 == 0 && BLOCK_N <= 256, "one wgmma spans the tile: N a multiple of 8, at most 256");
  static_assert(kPlanes * kRemBTile <= S::kStageBytes && kRemBTile % 256 == 0, "remainder weight stage");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* ring = smem_raw;
  uint8_t* halo = smem_raw + S::kRingBytes;
  uint8_t* epi_smem = smem_raw + S::kMainBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_raw + S::kMainBytes + Epi::kSmemBytes);
  uint64_t* empty_bar = full_bar + S::kStages;
  uint64_t* halo_full = empty_bar + S::kStages;
  uint64_t* halo_empty = halo_full + 2;
  uint64_t* acc_free = halo_empty + 2;
  static_assert(Epi::kSmemBytes % 16 == 0, "epilogue area must keep the barriers aligned");
  static_assert((2 * S::kStages + 5) * 8 <= S::kBarBytes, "barrier area");
  const int warp = persistent_setup<S::kStages>(smem_raw, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, full_bar, empty_bar,
                                                acc_free, [&] {
                                                  for (int s = 0; s < 2; ++s) {
                                                    mbar_init(&halo_full[s], 1);
                                                    mbar_init(&halo_empty[s], kEpiThreads);
                                                  }
                                                });
  const int lane = threadIdx.x & 31;

  const ConvGeom& g = shape.conv;
  const int n_halo = g.cin_blocks + (g.rem_groups > 0 ? 1 : 0);   // halos (channel blocks) per output tile
  const bool tap_major = n_halo <= 2;                               // every halo of the tile resident at once
  const int n_steps = kHaloTaps * n_halo;                           // (tap, halo) steps of a tile
  const int total_items = shape.batches * shape.m_tiles * shape.n_chunks;

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      RingPos<S::kStages> pos;
      uint32_t tiles = 0;
      int halos = 0;   // halo loads issued so far: load i goes to slot i & 1
      for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        const WorkItem w = work_item(shape, shape.m_tiles, item);
        const int ty = w.mt / g.tiles_w, tx = w.mt - ty * g.tiles_w;
        const int x0 = tx * kConvTileW - 1, y0 = ty * kConvTileH - 1;
        for (int nt = w.nt_begin; nt < w.nt_end; ++nt) {
          // the previous tile's staged accumulator must be consumed before the ring (and, when the staging reaches
          // past the ring, the halo slots) is refilled
          bool staged = tiles > 0;
          const uint32_t staged_parity = (tiles - 1) & 1;
          ++tiles;
          auto wait_staged = [&]() {
            if (staged) mbar_wait(acc_free, staged_parity);
            staged = false;
          };
          // ---- the halo of channel block hh
          auto load_halo = [&](int hh) {
            if (!kStagingInRing) wait_staged();
            const int hi = halos + hh, slot = hi & 1;
            mbar_wait(&halo_empty[slot], ((hi >> 1) & 1) ^ 1);
            const int chunks = (hh == g.cin_blocks ? kRemChannels : kBlockK) / 8;
            uint64_t* fb = &halo_full[slot];
            mbar_arrive_expect_tx(fb, static_cast<uint32_t>(chunks) * kPlanes * kHaloW * kHaloH * 16);
            uint8_t* dst = halo + slot * kHaloSlotBytes;
            for (int c = 0; c < chunks; ++c) {
              const int ch = hh * kBlockK + 8 * c;
              tma_load_4d(dst + c * kHaloChunkBytes, &tm_a_hi, fb, ch, x0, y0, w.batch);
              if constexpr (kPlanes == 2)
                tma_load_4d(dst + kHaloPlaneBytes + c * kHaloChunkBytes, &tm_a_lo, fb, ch, x0, y0, w.batch);
            }
          };
          // the halos needed first are issued before the weights (with kStagingInRing: while the previous tile's
          // epilogue still runs); the others at their first tap
          const int preload = tap_major ? n_halo : 1;
          for (int hh = 0; hh < preload; ++hh) load_halo(hh);
          for (int s = 0; s < n_steps; ++s) {
            const int hh = tap_major ? s % n_halo : s / kHaloTaps;
            const int tap = tap_major ? s / n_halo : s % kHaloTaps;
            const bool rem = hh == g.cin_blocks;
            if (tap == 0 && hh >= preload) load_halo(hh);
            // ---- the weights of (tap, hh): kSubs stages, or one 16-channel stage for the remainder
            for (int j = 0; j < (rem ? 1 : kSubs); ++j) {
              wait_staged();
              mbar_wait(&empty_bar[pos.stage], pos.phase ^ 1);
              uint8_t* st = ring + pos.stage * S::kStageBytes;
              uint64_t* fb = &full_bar[pos.stage];
              if (rem) {
                mbar_arrive_expect_tx(fb, kPlanes * kRemBTile);
                tma_load_3d(st, &tm_br_hi, fb, tap * kRemChannels, nt * BLOCK_N, 0);
                if constexpr (kPlanes == 2) tma_load_3d(st + kRemBTile, &tm_br_lo, fb, tap * kRemChannels, nt * BLOCK_N, 0);
              } else {
                // the main weight planes keep gemm_split_kernel's K layout: k-block (tap, cb) at (tap * cin_blocks + cb) * 64
                const int k0 = (tap * g.cin_blocks + hh) * kBlockK + j * kBK;
                mbar_arrive_expect_tx(fb, S::kStageBytes);
                tma_load_3d(st, &tm_b_hi, fb, k0, nt * BLOCK_N, 0);
                if constexpr (kPlanes == 2) tma_load_3d(st + S::kBTile, &tm_b_lo, fb, k0, nt * BLOCK_N, 0);
              }
              pos.advance();
            }
          }
          halos += n_halo;
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups: wgmma + epilogue
    const int ct = threadIdx.x - kEpiWarp0 * 32;
    const int h = (warp - kEpiWarp0) >> 2;   // == ct >> 7, from the shuffled warp index: the compiler sees it uniform
    Epi epi(epi_params, epi_smem, shape);
    float acc[BLOCK_N / 2];                         // x-half h of the tile, all BLOCK_N columns
    float* stg = reinterpret_cast<float*>(ring);
    const uint32_t ring_u32 = smem_u32(ring);
    const uint32_t halo_u32 = smem_u32(halo);
    RingPos<S::kStages> pos;
    int halos = 0;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const WorkItem w = work_item(shape, shape.m_tiles, item);
      epi.item_begin(w.batch, w.mt * kBlockM, w.chunk);
      for (int nt = w.nt_begin; nt < w.nt_end; ++nt) {
        epi.prefetch(w.batch, w.mt * kBlockM, nt * BLOCK_N);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
        int prev = -1;        // ring stage of the previous weight stage
        int prev_halo = -1;   // halo slot whose last tap was the previous weight stage, else -1
        for (int s = 0; s < n_steps; ++s) {
          const int hh = tap_major ? s % n_halo : s / kHaloTaps;
          const int tap = tap_major ? s / n_halo : s % kHaloTaps;
          const bool rem = hh == g.cin_blocks;
          const int hi = halos + hh, slot = hi & 1;
          if (tap == 0) mbar_wait(&halo_full[slot], (hi >> 1) & 1);
          const int ky = tap / 3, kx = tap - ky * 3;
          // halo pixel of row group y = 0 of x-half h for this tap
          const uint32_t a_tap = halo_u32 + slot * kHaloSlotBytes + (ky * kHaloW + kx) * 16 + h * 8 * 16;
          const int subs = rem ? 1 : kSubs;
          for (int j = 0; j < subs; ++j) {
            mbar_wait(&full_bar[pos.stage], pos.phase);
            const uint32_t st = ring_u32 + pos.stage * S::kStageBytes;
            wgmma_fence();
            if (rem) {
              const uint64_t rb_hi = wgmma_desc_k_sw32(st);
              const uint64_t rb_lo = wgmma_desc_k_sw32(st + kRemBTile);
              const uint64_t ra_hi = wgmma_desc_k_noswz(a_tap, kHaloChunkBytes, kHaloW * 16);
              const uint64_t ra_lo = wgmma_desc_k_noswz(a_tap + kHaloPlaneBytes, kHaloChunkBytes, kHaloW * 16);
              wgmma_split<BLOCK_N, kPlanes>(acc, ra_hi, ra_lo, rb_hi, rb_lo);
            } else {
              const uint64_t db_hi = kBK == 64 ? wgmma_desc_k_sw128(st) : wgmma_desc_k_sw64(st);
              const uint64_t db_lo = kBK == 64 ? wgmma_desc_k_sw128(st + S::kBTile) : wgmma_desc_k_sw64(st + S::kBTile);
              const uint32_t a = a_tap + j * (kBK / kMmaK) * 2 * kHaloChunkBytes;
              const uint64_t da_hi = wgmma_desc_k_noswz(a, kHaloChunkBytes, kHaloW * 16);
              const uint64_t da_lo = wgmma_desc_k_noswz(a + kHaloPlaneBytes, kHaloChunkBytes, kHaloW * 16);
#pragma unroll
              for (int k = 0; k < kBK / kMmaK; ++k) {
                // A: 16 channels = two chunks further; B: 32 bytes further inside the swizzle row (16-byte units)
                const uint64_t a_adv = static_cast<uint64_t>(k * 2 * kHaloChunkBytes / 16);
                const uint64_t b_adv = static_cast<uint64_t>(k * 2);
                wgmma_split<BLOCK_N, kPlanes>(acc, da_hi + a_adv, da_lo + a_adv, db_hi + b_adv, db_lo + b_adv);
              }
            }
            wgmma_commit();
            wgmma_wait<1>();   // the previous stage's MMAs are done: its weight slot (and halo, if last) may be refilled
            if (prev >= 0) mbar_arrive(&empty_bar[prev]);
            if (prev_halo >= 0) mbar_arrive(&halo_empty[prev_halo]);
            prev = pos.stage;
            prev_halo = (tap == kHaloTaps - 1 && j == subs - 1) ? slot : -1;
            pos.advance();
          }
        }
        halos += n_halo;
        // the accumulator is staged by tile pixel: row r of warpgroup h is pixel (r / 8) * 16 + 8 * h + r % 8
        finish_tile<BLOCK_N>(
            epi, acc,
            [&] {
              mbar_arrive(&empty_bar[prev]);
              if (prev_halo >= 0) mbar_arrive(&halo_empty[prev_halo]);
            },
            [&] { stage_acc<BLOCK_N>(stg, acc_stride(BLOCK_N), acc, 8 * h, 16, 0); }, stg, ct, acc_free, w.batch,
            w.mt * kBlockM, nt * BLOCK_N);
      }
      epi.item_end(w.batch, w.mt * kBlockM, w.chunk);
    }
    tma_store_wait_all();
  }
}

}  // namespace lb
