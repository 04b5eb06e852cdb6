// Host side of the C ABI (include/loftr_b200.h): tensor-map construction, kernel launches and the
// per-stage orchestration of the matching hot path.  No torch types; raw device pointers + a stream.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/loftr_b200.h"
#include "epilogues.cuh"
#include "gemm_split.cuh"
#include "conv_halo.cuh"
#include "simt_kernels.cuh"
#include "kv_gemm.cuh"
#include "full_attn.cuh"
#include "stem_tc.cuh"
#include "comm.cuh"
#include "geometry.cuh"

namespace lb {

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

#define LB_CUDA(expr)                                                                      \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

#define LB_TRY(expr)          \
  do {                        \
    int r__ = (expr);         \
    if (r__ != 0) return r__; \
  } while (0)

static inline int cdiv(long a, long b) { return static_cast<int>((a + b - 1) / b); }

// CUDA's limit on gridDim.y and gridDim.z.  Entry points whose launches put a caller's count there refuse larger
// counts before launching anything (DESIGN.md §4.3).
constexpr int kMaxGridYZ = 65535;

// ------------------------------------------------------------------------------------------------ timing hook
// Optional per-launch CUDA-event timing of the tensor-core kernels (bench.py's roofline leg), of the per-pair match
// cap and the rectification search, of the point queries, of the image front end, of the rectifying warp and of the
// geometry estimator (its three launches as one record): events are recorded on the launching stream right around the
// kernels, and only while timing is enabled.  TAG_NONE: not timed.
enum Tag { TAG_NONE = -1, TAG_GEMM_TEST = 0, TAG_PROJ, TAG_MERGE_LN, TAG_MLP1, TAG_MLP2_LN, TAG_SCORE_LSE,
           TAG_SCORE_ARGMAX, TAG_FINE_MERGE, TAG_CONV, TAG_KV, TAG_QATTN, TAG_FULL_ATTN, TAG_MATCH_CAP, TAG_PREPROCESS,
           TAG_GEOMETRY, TAG_MATCH_QUERY, TAG_RECTIFY, TAG_MATCH_SEARCH, TAG_COUNT };
static const char* kTagNames[TAG_COUNT] = {"gemm_test", "proj_act", "merge_ln", "mlp1_relu", "mlp2_ln_res",
                                           "score_lse", "score_argmax", "fine_merge", "backbone_conv",
                                           "tf_kv_proj_fused", "tf_q_attn_fused", "tf_full_attn", "match_cap",
                                           "preprocess", "geometry", "match_query", "rectify", "match_search"};
struct TimingRec {
  cudaEvent_t e0, e1;
  int tag;
};
static bool g_timing = false;
static std::vector<TimingRec> g_recs;
static std::mutex g_timing_mu;
// One timing record over the launches issued on `st` between begin() and end(); events are only created and recorded
// while timing is enabled, and never for TAG_NONE.
struct TimedRange {
  TimingRec rec{nullptr, nullptr, TAG_NONE};
  cudaStream_t st = nullptr;
  int begin(int tag, cudaStream_t stream) {
    if (!g_timing || tag == TAG_NONE) return 0;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaError_t e = cudaStreamIsCapturing(stream, &cs);
    if (e != cudaSuccess) return fail("cudaStreamIsCapturing failed: %s", cudaGetErrorString(e));
    if (cs != cudaStreamCaptureStatusNone)
      return fail("kernel timing is enabled (lb_timing_enable) but the stream is being captured into a CUDA graph: "
                  "timing events cannot be recorded into a graph; disable timing before capture");
    if (cudaEventCreate(&rec.e0) != cudaSuccess || cudaEventCreate(&rec.e1) != cudaSuccess ||
        cudaEventRecord(rec.e0, stream) != cudaSuccess)
      return fail("timing event set-up failed");
    rec.tag = tag;
    st = stream;
    return 0;
  }
  int end() {
    if (rec.tag == TAG_NONE) return 0;
    if (cudaEventRecord(rec.e1, st) != cudaSuccess) return fail("timing event record failed");
    std::lock_guard<std::mutex> lk(g_timing_mu);
    g_recs.push_back(rec);
    return 0;
  }
};

// Every kernel launch: `kern` over grid x block with `smem` bytes of dynamic shared memory on `st`, counted by
// lb_launch_count() and, with a tag, timed as one record.  kPdl: programmatic dependent launch (the kernel's set-up
// overlaps the previous kernel's tail).
template <bool kPdl = false, class... Params, class... Args>
static int launch(int tag, void (*kern)(Params...), dim3 grid, dim3 block, int smem, cudaStream_t st, Args&&... args) {
  TimedRange t;
  LB_TRY(t.begin(tag, st));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = kPdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);   // its error is returned and cleared by cudaGetLastError
  g_launches.fetch_add(1);
  LB_CUDA(cudaGetLastError());
  return t.end();
}

// The library carries its own (static) CUDA runtime, whose notion of "current device" is independent of the
// caller's (e.g. torch's).  Every entry point therefore binds the calling thread to the device that owns the
// buffers it was given -- otherwise a process working on cuda:1 would launch on device 0 through the legacy
// default stream.
// The previous device of the calling thread is restored when the entry point returns (RAII), so a caller whose
// current device differs from the buffers' device is left undisturbed.  Binding also checks that the device is an
// sm_90 one and gives its SM count (`sms`).
constexpr int kMaxDevices = 64;
struct DeviceScope {
  int sms = 0;
  int bind(const void* dev_ptr) {
    if (!dev_ptr) return fail("null device pointer");
    cudaPointerAttributes attr;
    cudaError_t e = cudaPointerGetAttributes(&attr, dev_ptr);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail("no usable CUDA device for this buffer (%s); loftr_b200 has no CPU fallback", cudaGetErrorString(e));
    }
    if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)
      return fail("expected a CUDA device pointer; loftr_b200 has no CPU fallback");
    return bind_device(attr.device);
  }
  int bind_device(int device) {
    LB_CUDA(cudaGetDevice(&prev));
    if (prev != device) {
      LB_CUDA(cudaSetDevice(device));
      switched = true;
    }
    if (device < 0 || device >= kMaxDevices) return fail("device index %d out of range", device);
    static std::mutex mu;
    static int count[kMaxDevices] = {0};
    std::lock_guard<std::mutex> lk(mu);
    if (count[device] == 0) {
      cudaDeviceProp prop;
      cudaError_t e = cudaGetDeviceProperties(&prop, device);
      if (e != cudaSuccess) return fail("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
      if (prop.major != 9 || prop.minor != 0)
        return fail("loftr_b200 requires an sm_90 (H100) device, found sm_%d%d; there is no fallback", prop.major,
                    prop.minor);
      count[device] = prop.multiProcessorCount;
    }
    sms = count[device];
    return 0;
  }
  ~DeviceScope() {
    if (switched) cudaSetDevice(prev);
  }

 private:
  int prev = -1;
  bool switched = false;
};

// Allows `Kernel` up to `bytes` of dynamic shared memory on the current device (needed above 48 KB); the attribute is
// set on the first launch per device.
template <auto Kernel>
static int set_max_dynamic_smem(int bytes) {
  static bool configured[kMaxDevices] = {false};
  int dev = 0;
  LB_CUDA(cudaGetDevice(&dev));
  if (!configured[dev]) {
    LB_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    configured[dev] = true;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ TMA maps
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
  });
  return fn;
}

// One tiled tensor map over `rank` dims (innermost first) of fp16 or fp32 elements: byte strides of dims 1..rank-1,
// box and element strides per dim (estr nullptr: all 1).  Out-of-range elements read as zero.
static int encode_map(CUtensorMap* m, const char* what, const void* base, bool f32, int rank, const cuuint64_t* dims,
                      const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swz,
                      CUtensorMapL2promotion l2) {
  auto enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("%s: base pointer not 16-byte aligned", what);
  for (int i = 0; i + 1 < rank; ++i)
    if (strides[i] % 16 != 0)
      return fail("%s: stride of %llu bytes is not a multiple of 16", what, static_cast<unsigned long long>(strides[i]));
  const cuuint32_t ones[4] = {1, 1, 1, 1};
  CUresult r = enc(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank,
                   const_cast<void*>(base), dims, strides, box, estr ? estr : ones, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (%s) failed with CUresult %d", what, static_cast<int>(r));
  return 0;
}
static cuuint64_t u64(long v) { return static_cast<cuuint64_t>(v); }

// fp16 plane viewed as [batches][rows][K] with row stride ld and batch stride bs (elements; 0 -> rows * ld);
// box = box_k x box_rows x 1, swizzled rows of box_k elements.
static CUtensorMapSwizzle swizzle_for(int box_k) {
  return box_k * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : box_k * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}
static int make_map(CUtensorMap* m, const void* base, long K, long rows, long batches, long ld, long bs,
                    int box_rows, int box_k = kBlockK) {
  const cuuint64_t dims[3] = {u64(K), u64(rows), u64(batches)};
  const cuuint64_t strides[2] = {u64(ld * 2), u64((bs > 0 ? bs : rows * ld) * 2)};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_k), static_cast<cuuint32_t>(box_rows), 1};
  return encode_map(m, "plane", base, false, 3, dims, strides, box, nullptr, swizzle_for(box_k),
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// NHWC fp16 plane viewed as [N][H][W][C] (pixel stride ld elements); box = box_c channels x (16*stride) x (8*stride)
// x 1 with element strides (1, stride, stride, 1): an 8 x 16 patch of (strided) pixels per load.
static int make_map_nhwc(CUtensorMap* m, const void* base, int C, int W, int H, int N, long ld, int stride,
                         int box_c = kBlockK) {
  const cuuint64_t dims[4] = {u64(C), u64(W), u64(H), u64(N)};
  const cuuint64_t px = u64(ld * 2), strides[3] = {px, px * W, px * W * H};
  const cuuint32_t box[4] = {static_cast<cuuint32_t>(box_c), static_cast<cuuint32_t>(kConvTileW * stride),
                             static_cast<cuuint32_t>(kConvTileH * stride), 1};
  const cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1};
  return encode_map(m, "NHWC", base, false, 4, dims, strides, box, estr, swizzle_for(box_c),
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// NHWC fp16 plane [N][H][W][C] for conv3x3_halo_kernel: box = 8 channels x 18 x 10 pixels x 1, no swizzle (one
// 8-channel chunk of a 10 x 18 halo).  The channel extent is C, so channels at or past C read as zeros.
static int make_map_halo(CUtensorMap* m, const void* base, int C, int W, int H, int N, long ld) {
  const cuuint64_t dims[4] = {u64(C), u64(W), u64(H), u64(N)};
  const cuuint64_t px = u64(ld * 2), strides[3] = {px, px * W, px * W * H};
  const cuuint32_t box[4] = {8, static_cast<cuuint32_t>(kHaloW), static_cast<cuuint32_t>(kHaloH), 1};
  return encode_map(m, "halo", base, false, 4, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// ---- output tensor maps for the TMA-store epilogues (epilogues.cuh OutMaps): 64-byte swizzle for fp16 planes,
// 128-byte swizzle for fp32
static CUtensorMapSwizzle out_swizzle(bool f32) { return f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B; }
// [batches][rows][cols] matrix (row stride ld, batch stride bs elements; bs = 0 -> rows * ld): box 32 x 32 x 1
static int make_out_map(CUtensorMap* m, const void* base, bool f32, long cols, long rows, long batches, long ld, long bs) {
  const int esz = f32 ? 4 : 2;
  const cuuint64_t dims[3] = {u64(cols), u64(rows), u64(batches)};
  const cuuint64_t strides[2] = {u64(ld * esz), u64((bs > 0 ? bs : rows * ld) * esz)};
  const cuuint32_t box[3] = {32, 32, 1};
  return encode_map(m, "output", base, f32, 3, dims, strides, box, nullptr, out_swizzle(f32),
                    CU_TENSOR_MAP_L2_PROMOTION_NONE);
}
// NHWC [N][H][W][C] (pixel stride ld elements): box 32 channels x 16 x 2 pixels x 1 image
static int make_out_map_nhwc(CUtensorMap* m, const void* base, bool f32, int C, int W, int H, int N, long ld) {
  const cuuint64_t dims[4] = {u64(C), u64(W), u64(H), u64(N)};
  const cuuint64_t px = u64(ld * (f32 ? 4 : 2)), strides[3] = {px, px * W, px * W * H};
  const cuuint32_t box[4] = {32, static_cast<cuuint32_t>(kConvTileW), 2, 1};
  return encode_map(m, "NHWC output", base, f32, 4, dims, strides, box, nullptr, out_swizzle(f32),
                    CU_TENSOR_MAP_L2_PROMOTION_NONE);
}

// The map `make` builds over the hi plane and, for data held as two planes, the one over the lo plane.  With one plane
// the lo map is a copy of the hi map, which the kernels never read (lo may be null).
template <auto make, class... Args>
static int map_planes(int planes, CUtensorMap* m_hi, CUtensorMap* m_lo, const void* hi, const void* lo, Args... args) {
  LB_TRY(make(m_hi, hi, args...));
  if (planes == 2) return make(m_lo, lo, args...);
  *m_lo = *m_hi;
  return 0;
}

// planes (+ optional fp32) of a [batches][rows][cols] output
static int fill_out_maps(OutMaps* om, const void* hi, const void* lo, long ld_pl, const float* f32, long ld_f32, long cols,
                         long rows, long batches) {
  memset(om, 0, sizeof(*om));
  om->dims = 3;
  if (hi) {
    LB_TRY(map_planes<make_out_map>(2, &om->hi, &om->lo, hi, lo, false, cols, rows, batches, ld_pl, 0L));
    om->use |= 1;
  }
  if (f32) {
    LB_TRY(make_out_map(&om->f32, f32, true, cols, rows, batches, ld_f32, 0));
    om->use |= 2;
  }
  return 0;
}
// `planes` fp16 planes (+ optional fp32) of an NHWC [N][H][W][C] output
static int fill_out_maps_nhwc(OutMaps* om, int planes, const void* hi, const void* lo, long ld_pl, const float* f32,
                              long ld_f32, int C, int W, int H, int N) {
  memset(om, 0, sizeof(*om));
  om->dims = 4;
  if (hi) {
    LB_TRY(map_planes<make_out_map_nhwc>(planes, &om->hi, &om->lo, hi, lo, false, C, W, H, N, ld_pl));
    om->use |= 1;
  }
  if (f32) {
    LB_TRY(make_out_map_nhwc(&om->f32, f32, true, C, W, H, N, ld_f32));
    om->use |= 2;
  }
  return 0;
}

struct Planes {
  const void* hi;
  const void* lo;
  long ld;            // elements
  long batch_stride;  // elements, 0 = not batched
};

// ------------------------------------------------------------------------------------------------ GEMM launch
struct GemmMaps {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;      // boxes one ring stage deep along K (GemmSmem::kBK)
  CUtensorMap ar_hi, ar_lo, br_hi, br_lo;  // convolution channel remainder (16-element boxes); copies of the above if unused
};

// One persistent CTA per SM (at most one per work item) of a tensor-core kernel with the GemmShape work split.
template <auto kern, class... Args>
static int launch_persistent(int tag, const GemmShape& s, int smem_bytes, int sms, cudaStream_t st, Args... args) {
  LB_TRY(set_max_dynamic_smem<kern>(smem_bytes));
  const long items = static_cast<long>(s.batches) * s.m_tiles * s.n_chunks;
  const int grid = static_cast<int>(items < sms ? items : sms);
  // programmatic dependent launch of the tensor-core kernels (gemm_split.cuh): the next kernel's set-up overlaps this
  // one's tail.  LOFTR_B200_PDL=0 disables it.
  static const bool pdl = [] {
    const char* e = getenv("LOFTR_B200_PDL");
    return !e || atoi(e) != 0;
  }();
  return pdl ? launch<true>(tag, kern, grid, kGemmThreads, smem_bytes, st, args...)
             : launch<false>(tag, kern, grid, kGemmThreads, smem_bytes, st, args...);
}

template <int BN, class Epi>
static int launch_raw(int tag, const GemmMaps& maps, const GemmShape& s, const typename Epi::Params& ep, int sms,
                      cudaStream_t st) {
  using S = GemmSmem<BN, Epi::kSmemBytes, EpiOperandPlanes<Epi>::value>;
  constexpr int smem_bytes = S::kRingBytes + S::kBarBytes + Epi::kSmemBytes;
  static_assert(smem_bytes <= kSmemLimit, "shared memory budget exceeded");
  return launch_persistent<&gemm_split_kernel<BN, Epi>>(tag, s, smem_bytes, sms, st, maps.a_hi, maps.a_lo, maps.b_hi,
                                                          maps.b_lo, maps.ar_hi, maps.ar_lo, maps.br_hi, maps.br_lo, s, ep);
}

// The work split of `batches` M x N x K products in BN-wide n tiles: each work item sweeps one chunk of n tiles, with
// the n tiles split into n_chunks chunks (0: one tile per chunk).  b_batched: B holds one matrix per batch.
// live / live_unit_rows: optional device bound on the rows of every batch (GemmShape::live_count).
template <int BN>
static GemmShape gemm_shape(int batches, int M, int N, int K, bool b_batched = false, int n_chunks = 0,
                            const int* live = nullptr, int live_unit_rows = 0) {
  GemmShape s;
  s.batches = batches;
  s.M = M;
  s.N = N;
  s.K = K;
  s.b_batched = b_batched ? 1 : 0;
  s.m_tiles = cdiv(M, kBlockM);
  s.n_tiles = cdiv(N, BN);
  if (n_chunks <= 0 || n_chunks > s.n_tiles) n_chunks = s.n_tiles;
  s.tiles_per_chunk = n_chunks > 0 ? cdiv(s.n_tiles, n_chunks) : 1;   // no n tiles: nothing is launched
  s.n_chunks = cdiv(s.n_tiles, s.tiles_per_chunk);
  s.conv = ConvGeom{0, 0, 0, 0, 0, 0, 0, 0, 0};
  s.live_count = live;
  s.live_unit_rows = live_unit_rows;
  return s;
}

template <int BN, class Epi>
static int launch_gemm(int tag, const Planes& A, const Planes& B, const GemmShape& s, const typename Epi::Params& ep,
                       int sms, cudaStream_t st) {
  if (s.K % kBlockK != 0 || s.K <= 0) return fail("K=%d must be a positive multiple of %d", s.K, kBlockK);
  if (s.M <= 0 || s.N <= 0 || s.batches <= 0) return 0;  // nothing to do
  if (s.live_count && !EpiRowBound<Epi>::value) return fail("this GEMM epilogue is built without a device row bound");
  constexpr int kP = EpiOperandPlanes<Epi>::value;
  constexpr int kBK = GemmSmem<BN, Epi::kSmemBytes, kP>::kBK;
  GemmMaps mp;
  LB_TRY(map_planes<make_map>(kP, &mp.a_hi, &mp.a_lo, A.hi, A.lo, s.K, s.M, s.batches, A.ld, A.batch_stride, kBlockM,
                              kBK));
  const int bb = s.b_batched ? s.batches : 1;
  LB_TRY(map_planes<make_map>(kP, &mp.b_hi, &mp.b_lo, B.hi, B.lo, s.K, s.N, bb, B.ld, B.batch_stride, BN, kBK));
  mp.ar_hi = mp.a_hi; mp.ar_lo = mp.a_lo; mp.br_hi = mp.b_hi; mp.br_lo = mp.b_lo;
  return launch_raw<BN, Epi>(tag, mp, s, ep, sms, st);
}

// Implicit-GEMM convolution launch: in = NHWC planes [N, H_in, W_in, ld_in] with Cin valid channels; weights =
// main planes [Cout, taps * cin_blocks * 64] (+ remainder planes [Cout, taps * 16], see lb_conv_layout); out pixel
// grid H_out x W_out; cin_blocks / rem: the K layout of conv_layout.
struct ConvDesc {
  int N, H_in, W_in, Cin, H_out, W_out, Cout, ksize, stride, pad;
  int cin_blocks, rem;
};
// K layout of a convolution's implicit GEMM: `cin_blocks` 64-channel blocks per tap, plus `rem` (<= 16) remainder
// channels per tap that travel as 16-channel boxes (gemm_split.cuh ConvGeom).
static void conv_layout(int cin, int* cin_blocks, int* rem) {
  const int r = cin % kBlockK;
  if (cin > kBlockK && r > 0 && r <= kRemChannels) {
    *cin_blocks = cin / kBlockK;
    *rem = r;
  } else {
    *cin_blocks = (cin + kBlockK - 1) / kBlockK;
    *rem = 0;
  }
}
// The implicit GEMM of convolution d with BN-wide n tiles (one per work item), and the output geometry its epilogue
// reads.  lo: the weights have lo planes (split precision).  rem_taps_per_group: taps of one remainder group
// (ConvGeom::rem_groups).
template <int BN, class Params>
static int conv_shape(const ConvDesc& d, const Planes& wgt_rem, bool lo, int rem_taps_per_group, GemmShape* s,
                      Params* ep) {
  if (d.rem && (!wgt_rem.hi || (lo && !wgt_rem.lo)))
    return fail("convolution with Cin=%d needs remainder weight planes", d.Cin);
  const int taps = d.ksize * d.ksize;
  const int tiles_h = (d.H_out + kConvTileH - 1) / kConvTileH;
  const int tiles_w = (d.W_out + kConvTileW - 1) / kConvTileW;
  const int m_tiles = tiles_h * tiles_w, n_tiles = (d.Cout + BN - 1) / BN;
  if (n_tiles != 1)   // EpiConvImpl stages the folded BatchNorm of one n-tile per CTA
    return fail("convolution with Cout=%d needs one %d-wide n-tile, got %d", d.Cout, BN, n_tiles);
  const int rem_groups = d.rem ? (taps + rem_taps_per_group - 1) / rem_taps_per_group : 0;
  *s = GemmShape{d.N, m_tiles * kBlockM, d.Cout, taps * d.cin_blocks * kBlockK, /*b_batched=*/0, m_tiles, n_tiles,
                 /*n_chunks=*/n_tiles, /*tiles_per_chunk=*/1,
                 ConvGeom{1, tiles_w, d.stride, d.pad, d.ksize, d.cin_blocks, taps, taps * d.cin_blocks, rem_groups},
                 /*live_count=*/nullptr, 0};
  ep->H_out = d.H_out;
  ep->W_out = d.W_out;
  ep->tiles_w = tiles_w;
  return 0;
}

// Epi: EpiConv<BN, .> (hi / lo planes: operands, weights and outputs) or EpiConvF16<BN, .> (hi planes only; the lo
// maps are copies of the hi ones and never loaded)
template <int BN, class Epi>
static int launch_conv(const Planes& in, const Planes& wgt, const Planes& wgt_rem, const ConvDesc& d,
                       const typename Epi::Params& ep_in, int sms, cudaStream_t st) {
  constexpr int kP = EpiOperandPlanes<Epi>::value;
  using S = GemmSmem<BN, Epi::kSmemBytes, kP>;
  GemmShape s;
  typename Epi::Params ep = ep_in;
  LB_TRY(conv_shape<BN>(d, wgt_rem, kP == 2, S::kRemTapsPerStage, &s, &ep));
  GemmMaps mp;
  LB_TRY(map_planes<make_map_nhwc>(kP, &mp.a_hi, &mp.a_lo, in.hi, in.lo, d.Cin, d.W_in, d.H_in, d.N, in.ld, d.stride,
                                   S::kBK));
  LB_TRY(map_planes<make_map>(kP, &mp.b_hi, &mp.b_lo, wgt.hi, wgt.lo, s.K, d.Cout, 1, wgt.ld, 0, BN, S::kBK));
  if (d.rem) {
    LB_TRY(map_planes<make_map_nhwc>(kP, &mp.ar_hi, &mp.ar_lo, in.hi, in.lo, d.Cin, d.W_in, d.H_in, d.N, in.ld,
                                     d.stride, kRemChannels));
    LB_TRY(map_planes<make_map>(kP, &mp.br_hi, &mp.br_lo, wgt_rem.hi, wgt_rem.lo, s.conv.taps * kRemChannels, d.Cout,
                                1, wgt_rem.ld, 0, BN, kRemChannels));
  } else {
    mp.ar_hi = mp.a_hi; mp.ar_lo = mp.a_lo; mp.br_hi = mp.b_hi; mp.br_lo = mp.b_lo;
  }
  return launch_raw<BN, Epi>(TAG_CONV, mp, s, ep, sms, st);
}

// Stride-1 3x3 convolution through conv3x3_halo_kernel (same operands, weights and epilogue as launch_conv).
template <int BN, class Epi>
static int launch_conv_halo(const Planes& in, const Planes& wgt, const Planes& wgt_rem, const ConvDesc& d,
                            const typename Epi::Params& ep_in, int sms, cudaStream_t st) {
  constexpr int kP = EpiOperandPlanes<Epi>::value;
  using S = HaloSmem<BN, Epi::kSmemBytes, kP>;
  static_assert(S::kTotalBytes <= kSmemLimit, "shared memory budget exceeded");
  if (d.ksize != 3 || d.stride != 1 || d.pad != 1) return fail("the halo convolution is built for 3x3, stride 1, pad 1");
  GemmShape s;
  typename Epi::Params ep = ep_in;
  LB_TRY(conv_shape<BN>(d, wgt_rem, kP == 2, kHaloTaps, &s, &ep));   // the remainder is one 16-channel halo
  CUtensorMap a_hi, a_lo, b_hi, b_lo, br_hi, br_lo;
  LB_TRY(map_planes<make_map_halo>(kP, &a_hi, &a_lo, in.hi, in.lo, d.Cin, d.W_in, d.H_in, d.N, in.ld));
  LB_TRY(map_planes<make_map>(kP, &b_hi, &b_lo, wgt.hi, wgt.lo, s.K, d.Cout, 1, wgt.ld, 0, BN, S::kBK));
  if (d.rem) {
    LB_TRY(map_planes<make_map>(kP, &br_hi, &br_lo, wgt_rem.hi, wgt_rem.lo, kHaloTaps * kRemChannels, d.Cout, 1,
                                wgt_rem.ld, 0, BN, kRemChannels));
  } else {
    br_hi = b_hi;
    br_lo = b_lo;
  }
  return launch_persistent<&conv3x3_halo_kernel<BN, Epi>>(TAG_CONV, s, S::kTotalBytes, sms, st, a_hi, a_lo, b_hi, b_lo,
                                                            br_hi, br_lo, s, ep);
}

// number of n-chunks that gives every SM a few work items when a CTA must sweep many n tiles
static int pick_chunks(int row_items, int n_tiles, int sms) {
  int c = 1;
  while (static_cast<long>(row_items) * c < 40L * sms && c < n_tiles) ++c;   // fine-grained items: <3 % tail
  return c;
}

// ------------------------------------------------------------------------------------------------ workspace
struct Bump {
  uint8_t* base;
  size_t size;
  size_t off = 0;
  bool ok = true;
  template <class T>
  T* take(size_t count) {
    const size_t bytes = (count * sizeof(T) + 255) & ~size_t(255);
    if (!base) {  // sizing pass
      off += bytes;
      return nullptr;
    }
    if (off + bytes > size) {
      ok = false;
      return nullptr;
    }
    T* p = reinterpret_cast<T*>(base + off);
    off += bytes;
    return p;
  }
};

// ------------------------------------------------------------------------------------------------ transformer
struct TfWs {
  float* qkv;       // fine only: [R, 3C]
  __half* att_hi;   // [R, C]
  __half* att_lo;
  __half* h_hi;     // [R, 2C]
  __half* h_lo;
  float* kv;        // coarse only: [2*n_groups, H, D*D + D]
  float* kv_part;   // coarse only: [2*n_groups, KvSplits::parts, H, per] (K^T V split partials)
};
// The row splits over which kv_gemm_kernel sums K^T V for n_groups groups of group_rows rows on `sms` SMs (64-row
// blocks, kb_per of them per split).  parts = max(m_tiles, kKvSplits) bounds `splits` on every device and sizes
// TfWs::kv_part; the workspace size needs only `parts` and passes sms = 0.  `splits` fixes the summation order of
// K^T V, so changing this plan changes the output bits.
constexpr int kKvSplits = 8;
struct KvSplits {
  int parts, kb_total, kb_per, splits;
};
static KvSplits kv_splits(int group_rows, int n_groups, int sms) {
  const int m_tiles = cdiv(group_rows, kBlockM);
  KvSplits k{m_tiles > kKvSplits ? m_tiles : kKvSplits, cdiv(group_rows, 64), 0, 0};
  if (sms <= 0) return k;
  int splits = sms / (2 * n_groups);
  if (splits < 1) splits = 1;
  if (splits > k.kb_total) splits = k.kb_total;
  if (splits > k.parts) splits = k.parts;
  k.kb_per = cdiv(k.kb_total, splits);
  k.splits = cdiv(k.kb_total, k.kb_per);
  return k;
}

// Operand planes of the transformer and score-matrix products: 2 = split precision (hi*hi + hi*lo + lo*hi), 1 = the hi
// planes only, one fp16 MMA per product (match_precision "fp16": lb_transformer_forward_fp16 / lb_coarse_match_fp16,
// DESIGN.md §16).  The epilogues are the same; only the kernels' main loops read and multiply less.
template <class Epi, int kP>
using Operands = std::conditional_t<kP == 2, Epi, EpiF16Operands<Epi>>;

static void carve_tf(Bump& b, TfWs& w, int C, int H, long R, int n_groups, bool coarse, int max_group_rows) {
  const int D = C / H;
  // fp32 q|k|v of the fine (window) transformer; the coarse projections write planes
  w.qkv = coarse ? nullptr : b.take<float>(static_cast<size_t>(R) * 3 * C);
  w.att_hi = b.take<__half>(static_cast<size_t>(R) * C);
  w.att_lo = b.take<__half>(static_cast<size_t>(R) * C);
  w.h_hi = b.take<__half>(static_cast<size_t>(R) * 2 * C);
  w.h_lo = b.take<__half>(static_cast<size_t>(R) * 2 * C);
  w.kv = coarse ? b.take<float>(static_cast<size_t>(2) * n_groups * H * (D * D + D)) : nullptr;
  const size_t parts = static_cast<size_t>(kv_splits(max_group_rows, n_groups, 0).parts);
  w.kv_part = coarse ? b.take<float>(static_cast<size_t>(2) * n_groups * H * parts * (D * D + D)) : nullptr;
}

// ------------------------------------------------------------------------------------------------ backbone
// ResNetFPN_8_2 forward (reference src/loftr/backbone/resnet_fpn.py:43-118) on tensor cores: every 3x3 / 1x1
// convolution is an implicit GEMM through gemm_split_kernel<., EpiConv>, the stride-1 3x3 ones through
// conv3x3_halo_kernel<., EpiConv> (BatchNorm, ReLU / LeakyReLU, residual add and the FPN upsample-add fused in the
// epilogue); activations live as NHWC fp16 hi/lo planes.  The fp16 backbone (lb_backbone_forward_fp16) runs the same
// network on single fp16 planes (planes = 1: lo == nullptr) with one MMA per product after the stem (EpiConvF16).
struct BbBuf {
  __half* hi;
  __half* lo;
  int ld;
};
static inline int pad8(int c) { return (c + 7) & ~7; }
static BbBuf bb_take(Bump& b, long pixels, int C, int planes) {
  BbBuf r;
  r.ld = pad8(C);
  r.hi = b.take<__half>(static_cast<size_t>(pixels) * r.ld);
  r.lo = planes == 2 ? b.take<__half>(static_cast<size_t>(pixels) * r.ld) : nullptr;
  return r;
}
struct BbWs {
  BbBuf s0, t1, a1, x1;                 // 1/2 resolution, d1 channels
  BbBuf t2, dn2, a2, x2;                // 1/4, d2
  BbBuf t3, dn3, a3, x3, x3o;           // 1/8, d3
  BbBuf x2l, m2, x2o;                   // 1/4: d3, d3, d2
  BbBuf x1l, m1;                        // 1/2: d2, d2
};
static void carve_bb(Bump& b, BbWs& w, int N, int H, int W, int d1, int d2, int d3, int planes) {
  const long p2 = static_cast<long>(N) * (H / 2) * (W / 2), p4 = static_cast<long>(N) * (H / 4) * (W / 4),
             p8 = static_cast<long>(N) * (H / 8) * (W / 8);
  auto take = [&](long pixels, int C) { return bb_take(b, pixels, C, planes); };
  w.s0 = take(p2, d1); w.t1 = take(p2, d1); w.a1 = take(p2, d1); w.x1 = take(p2, d1);
  w.t2 = take(p4, d2); w.dn2 = take(p4, d2); w.a2 = take(p4, d2); w.x2 = take(p4, d2);
  w.t3 = take(p8, d3); w.dn3 = take(p8, d3); w.a3 = take(p8, d3); w.x3 = take(p8, d3);
  w.x3o = take(p8, d3);
  w.x2l = take(p4, d3); w.m2 = take(p4, d3); w.x2o = take(p4, d2);
  w.x1l = take(p2, d2); w.m1 = take(p2, d2);
}

struct ConvRun {
  const LbConvWeights* w;
  BbBuf in;
  int H_in, W_in;
  int act;
  const BbBuf* res;
  const BbBuf* up;
  int up_h, up_w;
  const BbBuf* out;     // outputs (planes and / or fp32): run_conv builds the epilogue's store maps over them
  float* out_f32;
  int f32_ld;
};
// The kernel of a convolution and its output-channel tile BN.  Stride-1 3x3 convolutions (none of them carries the FPN
// upsample-add) run conv3x3_halo_kernel, which loads each input patch once per channel block; the others the implicit
// GEMM.  BN is the smallest built N that covers Cout: 196 -> 200 in the halo kernel (one m64n200 wgmma per x-half);
// 208 in gemm_split_kernel, whose two column halves need N / 2 to be a wgmma N (104 = 13 x 8).  0: none is built.
struct ConvKernel {
  bool halo;
  int bn;
};
static ConvKernel conv_kernel(const LbConvWeights& w, bool up) {
  const bool halo = w.ksize == 3 && w.stride == 1 && !up;
  const int mid = halo ? 200 : 208;
  return {halo, w.cout <= 128 ? 128 : w.cout <= mid ? mid : w.cout <= 256 ? 256 : 0};
}

// One convolution on the kernel and tile conv_kernel picked; the epilogue type of the tile width and FPN mode also
// selects the kernels' operand planes.
template <int kPlanes, bool kHalo, int BN, bool kUp>
static int launch_conv_on(const ConvRun& r, const ConvDesc& d, const OutMaps& om, int sms, cudaStream_t st) {
  using Epi = std::conditional_t<kPlanes == 2, EpiConv<BN, kUp>, EpiConvF16<BN, kUp>>;
  const LbConvWeights& w = *r.w;
  const int taps = w.ksize * w.ksize;
  const Planes in{r.in.hi, r.in.lo, r.in.ld, 0};
  const Planes wg{w.w_hi, w.w_lo, static_cast<long>(taps) * d.cin_blocks * kBlockK, 0};
  const Planes wr{w.wr_hi, w.wr_lo, static_cast<long>(taps) * kRemChannels, 0};
  typename Epi::Params ep{w.scale, w.shift, r.act, r.res ? r.res->hi : nullptr, r.res ? r.res->lo : nullptr,
                          r.res ? r.res->ld : 0, r.up ? r.up->hi : nullptr, r.up ? r.up->lo : nullptr,
                          r.up ? r.up->ld : 0, r.up_h, r.up_w, 0, 0, 0, om};
  if constexpr (kHalo) return launch_conv_halo<BN, Epi>(in, wg, wr, d, ep, sms, st);
  else return launch_conv<BN, Epi>(in, wg, wr, d, ep, sms, st);
}

// kPlanes = 2: the split-precision convolution (EpiConv); 1: single fp16 planes (EpiConvF16, w_lo / wr_lo unused)
template <int kPlanes>
static int run_conv(const ConvRun& r, int N, int sms, cudaStream_t st) {
  const LbConvWeights& w = *r.w;
  ConvDesc d;
  d.N = N; d.H_in = r.H_in; d.W_in = r.W_in; d.Cin = w.cin;
  d.ksize = w.ksize; d.stride = w.stride; d.pad = w.ksize / 2;
  d.H_out = (r.H_in + 2 * d.pad - w.ksize) / w.stride + 1;
  d.W_out = (r.W_in + 2 * d.pad - w.ksize) / w.stride + 1;
  d.Cout = w.cout;
  conv_layout(w.cin, &d.cin_blocks, &d.rem);
  // NHWC output maps of the TMA-store epilogue (planes and / or fp32 feature map)
  OutMaps om;
  LB_TRY(fill_out_maps_nhwc(&om, kPlanes, r.out ? r.out->hi : nullptr, r.out ? r.out->lo : nullptr,
                            r.out ? r.out->ld : 0, r.out_f32, r.f32_ld, d.Cout, d.W_out, d.H_out, N));
  const ConvKernel k = conv_kernel(w, r.up != nullptr);
  if (k.halo) {
    switch (k.bn) {
      case 128: return launch_conv_on<kPlanes, true, 128, false>(r, d, om, sms, st);
      case 200: return launch_conv_on<kPlanes, true, 200, false>(r, d, om, sms, st);
      case 256: return launch_conv_on<kPlanes, true, 256, false>(r, d, om, sms, st);
    }
  } else if (r.up) {
    switch (k.bn) {
      case 128: return launch_conv_on<kPlanes, false, 128, true>(r, d, om, sms, st);
      case 208: return launch_conv_on<kPlanes, false, 208, true>(r, d, om, sms, st);
      case 256: return launch_conv_on<kPlanes, false, 256, true>(r, d, om, sms, st);
    }
  } else {
    switch (k.bn) {
      case 128: return launch_conv_on<kPlanes, false, 128, false>(r, d, om, sms, st);
      case 208: return launch_conv_on<kPlanes, false, 208, false>(r, d, om, sms, st);
      case 256: return launch_conv_on<kPlanes, false, 256, false>(r, d, om, sms, st);
    }
  }
  return fail("convolutions with more than 256 output channels are not built");
}

}  // namespace lb

using namespace lb;

// Steps 1-3 of a coarse (D = 32) encoder-layer call with full (softmax) attention: the message planes att[x rows] =
// softmax(Q K^T / sqrt(D)) V per group and head            [transformer.py:47-50, linear_attention.py:56-81]
// Projections carry no feature map and no row zeroing: masks act inside the attention (key weight 0, padded query 0).
// Q goes to the att planes [R, C] (overwritten in place by the message), K|V to the MLP hidden planes [R, 2C], which
// are dead at this point of the layer; full_attn_wgmma_kernel (full_attn.cuh) reads both through tensor maps.
template <int BN, int kP>
static int tf_full_attention_coarse(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st,
                                    const TfWs& w, long x_base, long x_rows, int x_group_rows, long s_base,
                                    long s_rows, int s_group_rows, int n_groups_x, bool self_pass, int sms,
                                    cudaStream_t stream) {
  const long ldc = 2L * C;
  const __half* cat_hi = static_cast<const __half*>(st.cat_hi);
  const __half* cat_lo = static_cast<const __half*>(st.cat_lo);
  const int n_groups_s = static_cast<int>(s_rows / s_group_rows);
  if (C != 256 || H != 8) return fail("full attention of the coarse transformer is built for d_model 256, 8 heads");
  if (n_groups_x != n_groups_s && !self_pass) return fail("query / source group counts differ");
  const __half* wq_hi = static_cast<const __half*>(lw.wqkv_hi);
  const __half* wq_lo = static_cast<const __half*>(lw.wqkv_lo);
  const long wkv_off = static_cast<long>(C) * C;   // k_proj, v_proj rows of wqkv
  {
    using Epi = Operands<EpiPlanes<BN>, kP>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, 0};
    Planes B{wq_hi, wq_lo, C, 0};
    typename Epi::Params ep{0, nullptr, 1, lw.s_qkv, {}};
    LB_TRY(fill_out_maps(&ep.om, w.att_hi + x_base * C, w.att_lo + x_base * C, C, nullptr, 0, C, x_rows, 1));
    LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, gemm_shape<BN>(1, static_cast<int>(x_rows), C, C), ep, sms, stream)));
  }
  {
    using Epi = Operands<EpiPlanes<BN>, kP>;
    Planes A{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, 0};
    Planes B{wq_hi + wkv_off, wq_lo + wkv_off, C, 0};
    typename Epi::Params ep{0, nullptr, 1, lw.s_qkv, {}};
    LB_TRY(fill_out_maps(&ep.om, w.h_hi + s_base * ldc, w.h_lo + s_base * ldc, ldc, nullptr, 0, 2 * C, s_rows, 1));
    LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, gemm_shape<BN>(1, static_cast<int>(s_rows), 2 * C, C), ep, sms,
                                 stream)));
  }
  const long qbs = static_cast<long>(x_group_rows) * C, kvbs = static_cast<long>(s_group_rows) * ldc;
  CUtensorMap tq_hi, tq_lo, tkv_hi, tkv_lo;
  LB_TRY(map_planes<make_map>(kP, &tq_hi, &tq_lo, w.att_hi + x_base * C, w.att_lo + x_base * C, C, x_group_rows,
                              n_groups_x, C, qbs, kFaRows, kFaD));
  LB_TRY(map_planes<make_map>(kP, &tkv_hi, &tkv_lo, w.h_hi + s_base * ldc, w.h_lo + s_base * ldc, 2 * C, s_group_rows,
                              n_groups_s, ldc, kvbs, kFaKeys, kFaD));
  constexpr auto kernel = kP == 2 ? &full_attn_wgmma_kernel : &full_attn_wgmma_fp16_kernel;
  LB_TRY(set_max_dynamic_smem<kernel>(fw_smem_bytes(kP)));
  FullAttnWgParams wp;
  wp.Lx = x_group_rows;
  wp.Ls = s_group_rows;
  wp.v_col0 = C;
  wp.x_base = x_base;
  wp.s_base = s_base;
  wp.mask = st.mask;
  wp.o_hi = w.att_hi;
  wp.o_lo = w.att_lo;
  wp.ld_o = C;
  wp.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(kFaD));
  const dim3 grid(cdiv(x_group_rows, kFaRows), H, n_groups_x);
  return launch(TAG_FULL_ATTN, kernel, grid, kFwThreads, fw_smem_bytes(kP), stream, tq_hi, tq_lo, tkv_hi, tkv_lo, wp);
}

// Steps 1-3 of a coarse (D = 32) encoder-layer call with linear attention (SURVEY.md §2a G1/G2): the k|v projection
// writes K = elu(k)+1 and V as planes, kv_gemm_kernel reduces them to K^T V and Ksum on the tensor cores, and the q
// projection applies the attention in its epilogue; q, k, v never reach HBM.
//                                                   [transformer.py:47-50, linear_attention.py:31-46]
template <int kP>
static int tf_linear_attention_coarse(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st,
                                      const TfWs& w, long x_base, int x_group_rows, long s_base, int s_group_rows,
                                      int n_groups_x, int n_groups_s, int sms, cudaStream_t stream) {
  if (!lw.wkv_hi || (kP == 2 && !lw.wkv_lo))
    return fail("linear attention of the coarse transformer needs the fused k|v weight planes (wkv_hi / wkv_lo)");
  const int D = C / H;
  const int per = D * D + D;
  const long ldc = 2L * C;
  const __half* cat_hi = static_cast<const __half*>(st.cat_hi);
  const __half* cat_lo = static_cast<const __half*>(st.cat_lo);
  const uint8_t* mask = st.mask;
  __half* kvp_hi = w.h_hi + s_base * ldc;   // the MLP hidden planes [R, 2C] are free at this point of the layer
  __half* kvp_lo = w.h_lo + s_base * ldc;
  {
    using Epi = Operands<EpiKvProj<256>, kP>;
    Planes A{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, static_cast<long>(s_group_rows) * ldc};
    Planes B{lw.wkv_hi, lw.wkv_lo, C, 0};
    typename Epi::Params ep;
    ep.rowmask = mask ? mask + s_base : nullptr;
    ep.acc_scale = lw.s_qkv;
    LB_TRY(fill_out_maps(&ep.om, kvp_hi, kvp_lo, ldc, nullptr, 0, 2 * C, s_group_rows, n_groups_s));
    LB_TRY((launch_gemm<256, Epi>(TAG_KV, A, B, gemm_shape<256>(n_groups_s, s_group_rows, 2 * C, C), ep, sms, stream)));
  }
  {
    CUtensorMap tm_hi, tm_lo;
    LB_TRY(map_planes<make_map>(kP, &tm_hi, &tm_lo, kvp_hi, kvp_lo, 2 * C, s_group_rows, n_groups_s, ldc,
                                static_cast<long>(s_group_rows) * ldc, 64, 64));
    const KvSplits ks = kv_splits(s_group_rows, n_groups_s, sms);
    constexpr auto kernel = kP == 2 ? &kv_gemm_kernel : &kv_gemm_fp16_kernel;
    LB_TRY(set_max_dynamic_smem<kernel>(kv_gemm_smem(kP)));
    KvGemmParams kp{w.kv_part, ks.kb_total, ks.kb_per, ks.splits};
    LB_TRY(launch(TAG_NONE, kernel, dim3(ks.splits, 2, n_groups_s), kKvGemmThreads, kv_gemm_smem(kP), stream, tm_hi,
                  tm_lo, kp));
    const long total = static_cast<long>(n_groups_s) * H * per;
    LB_TRY(launch(TAG_NONE, kv_tile_merge_kernel, cdiv(total, 256), 256, 0, stream, w.kv_part, ks.splits, H * per, w.kv,
                  total));
  }
  {
    using Epi = Operands<EpiAttn<256, 32>, kP>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, static_cast<long>(x_group_rows) * ldc};
    Planes B{lw.wqkv_hi, lw.wqkv_lo, C, 0};
    typename Epi::Params ep{mask ? mask + x_base : nullptr, lw.s_qkv, w.kv, 1e-6f, w.att_hi + x_base * C,
                            w.att_lo + x_base * C, C};
    LB_TRY((launch_gemm<256, Epi>(TAG_QATTN, A, B, gemm_shape<256>(n_groups_x, x_group_rows, C, C), ep, sms, stream)));
  }
  return 0;
}

// Runs one encoder-layer call `x <- layer(x, source)` for the row range x (queries) / s (source).
// self_pass: x range == source range (q, k, v in one projection launch).
template <int BN, int kP>
static int tf_layer_pass(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st, const TfWs& w,
                         long x_base, long x_rows, int x_group_rows, long s_base, long s_rows, int s_group_rows,
                         int n_groups_x, bool self_pass, bool write_f32, int sms, cudaStream_t stream, const int* live,
                         int live_cap, bool full) {
  const int D = C / H;
  const long ldc = 2L * C;
  const __half* cat_hi = static_cast<const __half*>(st.cat_hi);
  const __half* cat_lo = static_cast<const __half*>(st.cat_lo);
  const uint8_t* mask = st.mask;
  const int n_groups_s = static_cast<int>(s_rows / s_group_rows);
  if (n_groups_x != n_groups_s && !self_pass) return fail("query / source group counts differ");
  // Device-bounded window transformer (`live` != nullptr): every set of live_cap windows is one GEMM batch of
  // live_cap * group_rows rows whose live prefix is read on the device, so a self pass over both sets is a two-batch
  // GEMM.  Without a bound every row range is one batch (xb = sb = 1).
  const int xb = live ? static_cast<int>(x_rows / (static_cast<long>(live_cap) * x_group_rows)) : 1;
  const int sb = live ? static_cast<int>(s_rows / (static_cast<long>(live_cap) * s_group_rows)) : 1;
  const int xM = static_cast<int>(x_rows / xb), sM = static_cast<int>(s_rows / sb);
  const long xbs = xb > 1 ? static_cast<long>(xM) * ldc : 0, sbs = sb > 1 ? static_cast<long>(sM) * ldc : 0;
  const long xbs_a = xb > 1 ? static_cast<long>(xM) * C : 0;       // attention planes [R, C]
  if (live && (D != 16 || x_group_rows != s_group_rows))
    return fail("device-bounded group counts are built for the fine (window) transformer only");

  // 1-3. attention message -> att planes [x rows, C]
  if (D == 32 && !full) {
    LB_TRY(tf_linear_attention_coarse<kP>(lw, C, H, st, w, x_base, x_group_rows, s_base, s_group_rows, n_groups_x,
                                      n_groups_s, sms, stream));
  } else if (D == 32) {
    LB_TRY((tf_full_attention_coarse<BN, kP>(lw, C, H, st, w, x_base, x_rows, x_group_rows, s_base, s_rows, s_group_rows,
                                        n_groups_x, self_pass, sms, stream)));
  } else {
    // windows of the fine transformer (D = 16, H = 8): the window kernels give every query / source row one lane
    if (x_group_rows > 32 || s_group_rows > 32)
      return fail("window transformer supports at most 32 rows per window (got %d query and %d source rows)",
                  x_group_rows, s_group_rows);
    if (full && x_group_rows != s_group_rows) return fail("full window attention is built for equal window sizes");
    // q|k|v projection (linear: + elu+1 feature map + padding mask; full: plain, the window kernel applies the mask)
    //                                                                 [transformer.py:47-49, linear_attention.py:31-39]
    const int elu_self = full ? 0 : 2 * C, elu_q = full ? 0 : C, elu_kv = full ? 0 : C;
    const uint8_t* pmask = full ? nullptr : mask;
    using Epi = Operands<EpiActStore<BN>, kP>;
    if (self_pass) {
      Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
      Planes B{lw.wqkv_hi, lw.wqkv_lo, C, 0};
      OutMaps om;
      LB_TRY(fill_out_maps(&om, nullptr, nullptr, 0, w.qkv + x_base * 3 * C, 3 * C, 3 * C, xM, xb));
      typename Epi::Params ep{elu_self, pmask ? pmask + x_base : nullptr, lw.s_qkv, om};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, gemm_shape<BN>(xb, xM, 3 * C, C, false, 0, live, x_group_rows), ep,
                                   sms, stream)));
    } else {
      Planes Aq{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
      Planes Bq{lw.wqkv_hi, lw.wqkv_lo, C, 0};
      OutMaps omq, omk;
      LB_TRY(fill_out_maps(&omq, nullptr, nullptr, 0, w.qkv + x_base * 3 * C, 3 * C, C, xM, xb));
      LB_TRY(fill_out_maps(&omk, nullptr, nullptr, 0, w.qkv + s_base * 3 * C + C, 3 * C, 2 * C, sM, sb));
      typename Epi::Params eq{elu_q, pmask ? pmask + x_base : nullptr, lw.s_qkv, omq};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, Aq, Bq, gemm_shape<BN>(xb, xM, C, C, false, 0, live, x_group_rows), eq,
                                   sms, stream)));
      Planes Ak{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, sbs};
      Planes Bk{static_cast<const __half*>(lw.wqkv_hi) + static_cast<long>(C) * C,
                static_cast<const __half*>(lw.wqkv_lo) + static_cast<long>(C) * C, C, 0};
      typename Epi::Params ek{elu_kv, pmask ? pmask + s_base : nullptr, lw.s_qkv, omk};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, Ak, Bk, gemm_shape<BN>(sb, sM, 2 * C, C, false, 0, live, s_group_rows), ek,
                                   sms, stream)));
    }
    if (full) {
      // full (softmax) attention of the windows, exact fp32                      [linear_attention.py:56-81]
      const int grid = n_groups_x < 4 * sms ? n_groups_x : 4 * sms;
      LB_TRY(launch(TAG_NONE, window_full_attn_kernel<16, 8, 32>, grid, 256, 0, stream, w.qkv, 3 * C, 0, C, 2 * C,
                    x_base, s_base, x_group_rows, n_groups_x, mask, w.att_hi, w.att_lo, C, live, live_cap));
    } else {
      // linear attention, one kernel per pass: KV stays in shared memory      [linear_attention.py:43-46]
      const int grid = n_groups_x < 3 * sms ? n_groups_x : 3 * sms;   // 3 resident blocks per SM (60 KB, <= 85 registers)
      const int wa_smem = (H * (D * D + D) + 4 * s_group_rows * C) * static_cast<int>(sizeof(float));
      LB_TRY((set_max_dynamic_smem<&window_attn_kernel<16, 8>>(
          (8 * (16 * 16 + 16) + 4 * 32 * 128) * static_cast<int>(sizeof(float)))));   // largest (32-row) window
      LB_TRY(launch(TAG_NONE, window_attn_kernel<16, 8>, grid, 256, wa_smem, stream, w.qkv, 3 * C, 0, C, 2 * C, x_base,
                    s_base, x_group_rows, s_group_rows, n_groups_x, 1e-6f, w.att_hi, w.att_lo, C, live, live_cap));
    }
  }
  // 4. merge + norm1 -> cat[:, C:2C]                            [transformer.py:51-52]
  {
    using Epi = Operands<EpiLayerNorm<BN>, kP>;
    Planes A{w.att_hi + x_base * C, w.att_lo + x_base * C, C, xbs_a};
    Planes B{lw.wm_hi, lw.wm_lo, C, 0};
    typename Epi::Params ep{lw.ln1_g, lw.ln1_b, 1e-5f, nullptr, nullptr, 0, lw.s_m, {}};
    LB_TRY(fill_out_maps(&ep.om, static_cast<__half*>(st.cat_hi) + x_base * ldc + C,
                         static_cast<__half*>(st.cat_lo) + x_base * ldc + C, ldc, nullptr, 0, C, xM, xb));
    LB_TRY((launch_gemm<BN, Epi>(TAG_MERGE_LN, A, B, gemm_shape<BN>(xb, xM, C, C, false, 0, live, x_group_rows), ep,
                                 sms, stream)));
  }
  // 5. mlp[0] + ReLU on cat([x, message]) -> h planes           [transformer.py:55, mlp 22-26]
  {
    using Epi = Operands<EpiPlanes<BN>, kP>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
    Planes B{lw.w1_hi, lw.w1_lo, 2 * C, 0};
    typename Epi::Params ep{1, nullptr, 1, lw.s_1, {}};
    LB_TRY(fill_out_maps(&ep.om, w.h_hi + x_base * ldc, w.h_lo + x_base * ldc, ldc, nullptr, 0, 2 * C, xM, xb));
    LB_TRY((launch_gemm<BN, Epi>(TAG_MLP1, A, B, gemm_shape<BN>(xb, xM, 2 * C, 2 * C, false, 0, live, x_group_rows), ep,
                                 sms, stream)));
  }
  // 6. mlp[2] + norm2 + residual -> cat[:, 0:C] (and x_f32 after the last layer)   [transformer.py:55-58]
  // The residual stream lives in the fp16 planes (x = hi + lo, exact to 2^-22 relative): no fp32 master copy is read
  // or written between layers.
  {
    using Epi = Operands<EpiLayerNorm<BN>, kP>;
    Planes A{w.h_hi + x_base * ldc, w.h_lo + x_base * ldc, ldc, xbs};
    Planes B{lw.w2_hi, lw.w2_lo, 2 * C, 0};
    float* xf = write_f32 ? st.x_f32 + x_base * C : nullptr;
    typename Epi::Params ep{lw.ln2_g, lw.ln2_b, 1e-5f, cat_hi + x_base * ldc, cat_lo + x_base * ldc,
                            static_cast<int>(ldc), lw.s_2, {}};
    LB_TRY(fill_out_maps(&ep.om, static_cast<__half*>(st.cat_hi) + x_base * ldc,
                         static_cast<__half*>(st.cat_lo) + x_base * ldc, ldc, xf, C, C, xM, xb));
    LB_TRY((launch_gemm<BN, Epi>(TAG_MLP2_LN, A, B, gemm_shape<BN>(xb, xM, C, 2 * C, false, 0, live, x_group_rows), ep,
                                 sms, stream)));
  }
  return 0;
}

// The test hooks of the contraction core: gemm_split_kernel<BN, Operands<EpiActStore<BN>, kP>> at BN 256 / 128, the
// instantiations the transformers run (kP = 1 reads the hi planes only: a_lo / b_lo may be null).
template <int kP>
static int gemm_test(const char* who, const void* a_hi, const void* a_lo, long lda, long a_batch_stride,
                     const void* b_hi, const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo,
                     long o_batch_stride, int batches, int M, int N, int K, void* stream) {
  if (N % 32 != 0) return fail("%s: N must be a multiple of 32", who);
  DeviceScope dev;
  LB_TRY(dev.bind(out));
  if (batches > 1 && o_batch_stride != static_cast<long>(M) * ldo)
    return fail("%s: output batches must be densely stacked (o_batch_stride == M*ldo)", who);
  Planes A{a_hi, a_lo, lda, batches > 1 ? a_batch_stride : 0};
  Planes B{b_hi, b_lo, ldb, b_batch_stride};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  OutMaps om;
  LB_TRY(fill_out_maps(&om, nullptr, nullptr, 0, out, ldo, N, M, batches));
  if (N % 256 == 0 || N > 128) {
    using Epi = Operands<EpiActStore<256>, kP>;
    typename Epi::Params ep{0, nullptr, 1.f, om};
    return launch_gemm<256, Epi>(TAG_GEMM_TEST, A, B, gemm_shape<256>(batches, M, N, K, b_batch_stride > 0), ep,
                                 dev.sms, st);
  }
  using Epi = Operands<EpiActStore<128>, kP>;
  typename Epi::Params ep{0, nullptr, 1.f, om};
  return launch_gemm<128, Epi>(TAG_GEMM_TEST, A, B, gemm_shape<128>(batches, M, N, K, b_batch_stride > 0), ep, dev.sms,
                               st);
}

extern "C" {

int lb_version(void) { return 110; }
int lb_block_k(void) { return kBlockK; }
int lb_conv_layout(int cin, int* cin_blocks, int* rem_channels) {
  if (!cin_blocks || !rem_channels || cin <= 0) return fail("lb_conv_layout: bad arguments");
  conv_layout(cin, cin_blocks, rem_channels);
  return 0;
}
const char* lb_last_error(void) { return g_err; }
long long lb_launch_count(void) { return g_launches.load(); }

int lb_timing_enable(int on) {
  std::lock_guard<std::mutex> lk(g_timing_mu);
  for (auto& r : g_recs) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  g_recs.clear();
  g_timing = on != 0;
  return 0;
}
int lb_timing_num_tags(void) { return TAG_COUNT; }
const char* lb_timing_tag_name(int tag) { return (tag >= 0 && tag < TAG_COUNT) ? kTagNames[tag] : ""; }
int lb_timing_collect(double* total_ms, long long* counts, int n) {
  std::lock_guard<std::mutex> lk(g_timing_mu);
  for (int i = 0; i < n; ++i) {
    total_ms[i] = 0.0;
    counts[i] = 0;
  }
  for (auto& r : g_recs) {
    LB_CUDA(cudaEventSynchronize(r.e1));
    float ms = 0.f;
    LB_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
    if (r.tag < n) {
      total_ms[r.tag] += ms;
      counts[r.tag] += 1;
    }
  }
  return 0;
}

int lb_split_planes(const float* x, long rows, int cols, int ld_x, void* hi, void* lo, int ld_pl, int col0,
                    void* stream) {
  if (rows <= 0 || cols <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(x));
  const long total = rows * cols;
  const int grid = static_cast<int>(total / 256 + 1 < 4096 ? total / 256 + 1 : 4096);
  return launch(TAG_NONE, split_planes_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), x, rows, cols, ld_x,
                static_cast<__half*>(hi), static_cast<__half*>(lo), ld_pl, col0);
}

int lb_gemm_split(const void* a_hi, const void* a_lo, long lda, long a_batch_stride, const void* b_hi,
                  const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo, long o_batch_stride,
                  int batches, int M, int N, int K, void* stream) {
  return gemm_test<2>("lb_gemm_split", a_hi, a_lo, lda, a_batch_stride, b_hi, b_lo, ldb, b_batch_stride, out, ldo,
                      o_batch_stride, batches, M, N, K, stream);
}

int lb_gemm_fp16(const void* a_hi, const void* a_lo, long lda, long a_batch_stride, const void* b_hi,
                 const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo, long o_batch_stride,
                 int batches, int M, int N, int K, void* stream) {
  return gemm_test<1>("lb_gemm_fp16", a_hi, a_lo, lda, a_batch_stride, b_hi, b_lo, ldb, b_batch_stride, out, ldo,
                      o_batch_stride, batches, M, N, K, stream);
}

int lb_preprocess_images(const LbImageDesc* descs, int n_images, float* out, int H, int W, uint8_t* mask,
                         void* stream) {
  if (H <= 0 || W <= 0 || H % 8 != 0 || W % 8 != 0)
    return fail("lb_preprocess_images: canvas %dx%d must be positive and divisible by 8", H, W);
  if (n_images < 0 || n_images > 65535) return fail("lb_preprocess_images: n_images=%d must be in [0, 65535]", n_images);
  if (!descs || !out) return fail("lb_preprocess_images: descs and out are required");
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0) return fail("lb_preprocess_images: out is not 16-byte aligned");
  if (n_images == 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(out));
  dim3 grid(cdiv(W, kPreprocessBlockX * 4), cdiv(H, kPreprocessBlockY), n_images);
  return launch(TAG_PREPROCESS, preprocess_images_kernel, grid, dim3(kPreprocessBlockX, kPreprocessBlockY), 0,
                static_cast<cudaStream_t>(stream), descs, out, H, W, mask);
}

int lb_rectify_images(const float* image1, int n, int H1, int W1, const float* models, const float* scale0,
                      const float* scale1, float* out, int H, int W, void* stream) {
  if (H <= 0 || W <= 0 || H % 8 != 0 || W % 8 != 0)
    return fail("lb_rectify_images: canvas %dx%d must be positive and divisible by 8", H, W);
  if (n < 0 || n > 65535) return fail("lb_rectify_images: n=%d must be in [0, 65535]", n);
  if (H1 <= 0 || W1 <= 0) return fail("lb_rectify_images: image1 size %dx%d must be positive", H1, W1);
  if (!image1 || !models || !out) return fail("lb_rectify_images: image1, models and out are required");
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0) return fail("lb_rectify_images: out is not 16-byte aligned");
  if (n == 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(out));
  dim3 grid(cdiv(W, kRectifyBlockX * 4), cdiv(H, kRectifyBlockY), n);
  return launch(TAG_RECTIFY, rectify_images_kernel, grid, dim3(kRectifyBlockX, kRectifyBlockY), 0,
                static_cast<cudaStream_t>(stream), image1, H1, W1, models, scale0, scale1, out, H, W);
}

int lb_rectify_points(const float* pts, const long long* pair_ids, long m, const int* M_live, const float* models,
                      int n_pairs, const float* scale0, const float* scale1, int H0, int W0, int H1, int W1,
                      const uint8_t* mask1, int w1c, float* out, uint8_t* inside, void* stream) {
  if (m < 0 || n_pairs < 0) return fail("lb_rectify_points: m=%ld and n_pairs=%d must not be negative", m, n_pairs);
  if (H0 <= 0 || W0 <= 0 || H1 <= 0 || W1 <= 0)
    return fail("lb_rectify_points: image sizes %dx%d and %dx%d must be positive", H0, W0, H1, W1);
  if (mask1 && (H1 % 8 != 0 || W1 % 8 != 0 || w1c != W1 / 8))
    return fail("lb_rectify_points: mask1 needs image1 sides divisible by 8 and w1c = W1 / 8 (got %dx%d, w1c=%d)", H1,
                W1, w1c);
  if (m == 0) return 0;
  if (!pts || !pair_ids || !models || !out) return fail("lb_rectify_points: pts, pair_ids, models and out are required");
  DeviceScope dev;
  LB_TRY(dev.bind(out));
  const RectifyPointsParams p{pts, pair_ids, m, M_live, models, n_pairs, scale0, scale1, H0, W0, H1, W1, mask1, w1c,
                              out, inside};
  return launch(TAG_NONE, rectify_points_kernel, cdiv(m, 256), 256, 0, static_cast<cudaStream_t>(stream), p);
}

// n_out output images; with img_idx, output image b reads image img_idx[b] of feat
static int coarse_prep(const float* feat, int nhwc, const float* pe, const int* img_idx, int n_out, int C, int h,
                       int w, int pe_h, int pe_w, float* x_f32, void* cat_hi, void* cat_lo, void* stream) {
  if (n_out > kMaxGridYZ) return fail("coarse_prep: n_out=%d images exceed the grid.z limit %d", n_out, kMaxGridYZ);
  if (n_out <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(x_f32));
  if (h > pe_h || w > pe_w) return fail("feature map %dx%d exceeds the position-encoding table %dx%d", h, w, pe_h, pe_w);
  dim3 grid(cdiv(static_cast<long>(h) * w, 32), cdiv(C, 32), n_out);
  return launch(TAG_NONE, img_idx ? coarse_prep_kernel<true> : coarse_prep_kernel<false>, grid, dim3(32, 8), 0,
                static_cast<cudaStream_t>(stream), feat, nhwc, pe, C, h, w, pe_h, pe_w, x_f32,
                static_cast<__half*>(cat_hi), static_cast<__half*>(cat_lo), img_idx);
}

int lb_coarse_prep(const float* feat, int nhwc, const float* pe, int n_img, int C, int h, int w, int pe_h, int pe_w,
                   float* x_f32, void* cat_hi, void* cat_lo, void* stream) {
  return coarse_prep(feat, nhwc, pe, nullptr, n_img, C, h, w, pe_h, pe_w, x_f32, cat_hi, cat_lo, stream);
}

int lb_coarse_prep_indexed(const float* feat, int nhwc, const float* pe, const int* img_idx, int n_out, int C, int h,
                           int w, int pe_h, int pe_w, float* x_f32, void* cat_hi, void* cat_lo, void* stream) {
  if (n_out > 0 && !img_idx) return fail("lb_coarse_prep_indexed: img_idx is null");
  return coarse_prep(feat, nhwc, pe, img_idx, n_out, C, h, w, pe_h, pe_w, x_f32, cat_hi, cat_lo, stream);
}

size_t lb_transformer_workspace_bytes(int d_model, int nhead, int n_groups, int group_rows0, int group_rows1) {
  Bump b{nullptr, 0};
  TfWs w;
  const long R = static_cast<long>(n_groups) * (group_rows0 + group_rows1);
  carve_tf(b, w, d_model, nhead, R, n_groups, d_model / nhead == 32, group_rows0 > group_rows1 ? group_rows0 : group_rows1);
  return b.off + 256;
}

}  // extern "C"

// kP: operand planes of every tensor-core product (Operands)
template <int kP>
static int transformer_forward(const LbEncoderLayerWeights* layers, const int* kinds, int n_layers, int d_model,
                               int nhead, const LbTransformerState* st, void* ws, size_t ws_bytes, void* stream) {
  if (st->n_groups <= 0) return 0;
  const int C = d_model, H = nhead;
  const bool coarse = (C == 256 && H == 8);
  // the coarse attention kernels put the images of a pass in grid.z (kv_gemm_kernel, full_attn_wgmma_kernel)
  if (coarse && st->n_groups > kMaxGridYZ)
    return fail("coarse transformer: n_groups=%d pairs exceed the grid.z limit %d", st->n_groups, kMaxGridYZ);
  DeviceScope dev;
  LB_TRY(dev.bind(st->x_f32));
  const bool fine = (C == 128 && H == 8);
  if (!coarse && !fine) return fail("unsupported transformer shape d_model=%d nhead=%d (built: 256/8 and 128/8)", C, H);
  const int* live = st->n_groups_live;
  if (live && !fine) return fail("n_groups_live is built for the fine (window) transformer only");
  const long rows0 = static_cast<long>(st->n_groups) * st->group_rows0;
  const long rows1 = static_cast<long>(st->n_groups) * st->group_rows1;
  if (!ws) return fail("workspace pointer is null");
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  TfWs w;
  carve_tf(b, w, C, H, rows0 + rows1, st->n_groups, coarse,
           st->group_rows0 > st->group_rows1 ? st->group_rows0 : st->group_rows1);
  if (!b.ok) return fail("transformer workspace too small: need %zu bytes", lb_transformer_workspace_bytes(C, H, st->n_groups, st->group_rows0, st->group_rows1));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // One self pass over both sets doubles the images in grid.z: above kMaxGridYZ / 2 coarse pairs the sets get a pass
  // each.  Groups are independent and the pass's splits (kv_splits) are 1 at these counts, so the bits are the same.
  const bool same_groups =
      st->group_rows0 == st->group_rows1 && (!coarse || 2L * st->n_groups <= kMaxGridYZ);
  for (int l = 0; l < n_layers; ++l) {
    const LbEncoderLayerWeights& lw = layers[l];
    const bool last = l == n_layers - 1;   // the fp32 copy of the features is only written after the last layer
    const int kind = kinds[l];
    const bool full = kind == LB_LAYER_SELF_FULL || kind == LB_LAYER_CROSS_FULL;
    auto pass = [&](long xb, long xr, int xg, long sb, long sr, int sg, int ng, bool self_pass) -> int {
      return coarse ? tf_layer_pass<256, kP>(lw, C, H, *st, w, xb, xr, xg, sb, sr, sg, ng, self_pass, last, dev.sms, s,
                                             nullptr, 0, full)
                    : tf_layer_pass<128, kP>(lw, C, H, *st, w, xb, xr, xg, sb, sr, sg, ng, self_pass, last, dev.sms, s,
                                             live, st->n_groups, full);
    };
    if (kind == LB_LAYER_SELF || kind == LB_LAYER_SELF_FULL) {
      // feat0 = layer(feat0, feat0); feat1 = layer(feat1, feat1)  [transformer.py:93-94]; same weights,
      // independent -> one pass over both sets when the group sizes agree.
      if (same_groups) {
        LB_TRY(pass(0, rows0 + rows1, st->group_rows0, 0, rows0 + rows1, st->group_rows0, 2 * st->n_groups, true));
      } else {
        LB_TRY(pass(0, rows0, st->group_rows0, 0, rows0, st->group_rows0, st->n_groups, true));
        LB_TRY(pass(rows0, rows1, st->group_rows1, rows0, rows1, st->group_rows1, st->n_groups, true));
      }
    } else if (kind == LB_LAYER_CROSS || kind == LB_LAYER_CROSS_FULL) {
      // feat0 = layer(feat0, feat1); feat1 = layer(feat1, feat0_new)  [transformer.py:96-97]
      LB_TRY(pass(0, rows0, st->group_rows0, rows0, rows1, st->group_rows1, st->n_groups, false));
      LB_TRY(pass(rows0, rows1, st->group_rows1, 0, rows0, st->group_rows0, st->n_groups, false));
    } else {
      return fail("unknown layer kind %d", kind);
    }
  }
  return 0;
}

extern "C" {

int lb_transformer_forward(const LbEncoderLayerWeights* layers, const int* kinds, int n_layers, int d_model,
                           int nhead, const LbTransformerState* st, void* ws, size_t ws_bytes, void* stream) {
  return transformer_forward<2>(layers, kinds, n_layers, d_model, nhead, st, ws, ws_bytes, stream);
}

int lb_transformer_forward_fp16(const LbEncoderLayerWeights* layers, const int* kinds, int n_layers, int d_model,
                                int nhead, const LbTransformerState* st, void* ws, size_t ws_bytes, void* stream) {
  return transformer_forward<1>(layers, kinds, n_layers, d_model, nhead, st, ws, ws_bytes, stream);
}

}  // extern "C"

// Workspace of the backbone with `planes` fp16 planes per activation
static size_t backbone_workspace_bytes(const LbBackboneWeights* w, int N, int H, int W, int planes) {
  Bump b{nullptr, 0};
  BbWs ws;
  carve_bb(b, ws, N, H, W, w->l1[0].cout, w->l2[0].cout, w->l3[0].cout, planes);
  return b.off + 256;
}

// ResNetFPN_8_2 forward with split-precision (kPlanes = 2) or single fp16 (kPlanes = 1) activations and products
template <int kPlanes>
static int backbone_forward(const LbBackboneWeights* w, const float* images, int N, int H, int W, float* feat_c_nhwc,
                            float* feat_f_nhwc, void* ws, size_t ws_bytes, void* stream) {
  if (N <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(images));
  const int sms = dev.sms;
  if (H % 8 != 0 || W % 8 != 0) return fail("image size %dx%d must be divisible by 8", H, W);
  if (!ws) return fail("workspace pointer is null");
  const int d1 = w->l1[0].cout, d2 = w->l2[0].cout, d3 = w->l3[0].cout;
  if (w->stem_cout != 128 || d1 != w->stem_cout) return fail("backbone stem built for initial_dim = block_dims[0] = 128");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  BbWs B;
  carve_bb(b, B, N, H, W, d1, d2, d3, kPlanes);
  if (!b.ok)
    return fail("backbone workspace too small: need %zu bytes", backbone_workspace_bytes(w, N, H, W, kPlanes));
  const int H2 = H / 2, W2 = W / 2, H4 = H / 4, W4 = W / 4, H8 = H / 8, W8 = W / 8;

  // stem: conv 7x7 s2 + BN + ReLU on the tensor cores, software im2col (stem_tc.cuh)  [resnet_fpn.py:101]
  {
    StemTcParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.img = images; sp.N = N; sp.H = H; sp.W = W;
    sp.wt = w->stem_wt; sp.scale = w->stem_scale; sp.shift = w->stem_shift;
    sp.tiles_w = cdiv(W2, kConvTileW); sp.tiles_h = cdiv(H2, kConvTileH);
    LB_TRY(fill_out_maps_nhwc(&sp.om, kPlanes, B.s0.hi, B.s0.lo, B.s0.ld, nullptr, 0, 128, W2, H2, N));
    constexpr auto kStem = kPlanes == 2 ? &conv_stem7x7_tc_kernel : &conv_stem7x7_tc_fp16_kernel;
    LB_TRY(set_max_dynamic_smem<kStem>(kStemSmemBytes));
    const long tiles = static_cast<long>(sp.tiles_w) * sp.tiles_h * N;
    const int grid = static_cast<int>(tiles < sms ? tiles : sms);
    LB_TRY(launch(TAG_NONE, kStem, grid, kStemThreads, kStemSmemBytes, st, sp));
  }
  auto conv = [&](const LbConvWeights& cw, const BbBuf& in, int hin, int win, int act, const BbBuf* res,
                  const BbBuf* up, int uph, int upw, const BbBuf* out, float* of32, int f32ld) -> int {
    ConvRun r{&cw, in, hin, win, act, res, up, uph, upw, out, of32, f32ld};
    return run_conv<kPlanes>(r, N, sms, st);
  };
  // layer1 (1/2)                                                                    [resnet_fpn.py:102]
  LB_TRY(conv(w->l1[0], B.s0, H2, W2, 1, nullptr, nullptr, 0, 0, &B.t1, nullptr, 0));
  LB_TRY(conv(w->l1[1], B.t1, H2, W2, 1, &B.s0, nullptr, 0, 0, &B.a1, nullptr, 0));
  LB_TRY(conv(w->l1[2], B.a1, H2, W2, 1, nullptr, nullptr, 0, 0, &B.t1, nullptr, 0));
  LB_TRY(conv(w->l1[3], B.t1, H2, W2, 1, &B.a1, nullptr, 0, 0, &B.x1, nullptr, 0));
  // layer2 (1/4): first block strided with a projected skip                         [resnet_fpn.py:103]
  LB_TRY(conv(w->l2[0], B.x1, H2, W2, 1, nullptr, nullptr, 0, 0, &B.t2, nullptr, 0));
  LB_TRY(conv(w->l2_down, B.x1, H2, W2, 0, nullptr, nullptr, 0, 0, &B.dn2, nullptr, 0));
  LB_TRY(conv(w->l2[1], B.t2, H4, W4, 1, &B.dn2, nullptr, 0, 0, &B.a2, nullptr, 0));
  LB_TRY(conv(w->l2[2], B.a2, H4, W4, 1, nullptr, nullptr, 0, 0, &B.t2, nullptr, 0));
  LB_TRY(conv(w->l2[3], B.t2, H4, W4, 1, &B.a2, nullptr, 0, 0, &B.x2, nullptr, 0));
  // layer3 (1/8)                                                                    [resnet_fpn.py:104]
  LB_TRY(conv(w->l3[0], B.x2, H4, W4, 1, nullptr, nullptr, 0, 0, &B.t3, nullptr, 0));
  LB_TRY(conv(w->l3_down, B.x2, H4, W4, 0, nullptr, nullptr, 0, 0, &B.dn3, nullptr, 0));
  LB_TRY(conv(w->l3[1], B.t3, H8, W8, 1, &B.dn3, nullptr, 0, 0, &B.a3, nullptr, 0));
  LB_TRY(conv(w->l3[2], B.a3, H8, W8, 1, nullptr, nullptr, 0, 0, &B.t3, nullptr, 0));
  LB_TRY(conv(w->l3[3], B.t3, H8, W8, 1, &B.a3, nullptr, 0, 0, &B.x3, nullptr, 0));
  // FPN                                                                             [resnet_fpn.py:107-116]
  // The x2 bilinear upsampling of the coarser level is gathered inside the lateral 1x1 convolution's epilogue.
  LB_TRY(conv(w->l3_out, B.x3, H8, W8, 0, nullptr, nullptr, 0, 0, &B.x3o, feat_c_nhwc, d3));
  LB_TRY(conv(w->l2_out, B.x2, H4, W4, 0, nullptr, &B.x3o, H8, W8, &B.x2l, nullptr, 0));
  LB_TRY(conv(w->l2_out2[0], B.x2l, H4, W4, 2, nullptr, nullptr, 0, 0, &B.m2, nullptr, 0));
  LB_TRY(conv(w->l2_out2[1], B.m2, H4, W4, 0, nullptr, nullptr, 0, 0, &B.x2o, nullptr, 0));
  LB_TRY(conv(w->l1_out, B.x1, H2, W2, 0, nullptr, &B.x2o, H4, W4, &B.x1l, nullptr, 0));
  LB_TRY(conv(w->l1_out2[0], B.x1l, H2, W2, 2, nullptr, nullptr, 0, 0, &B.m1, nullptr, 0));
  LB_TRY(conv(w->l1_out2[1], B.m1, H2, W2, 0, nullptr, nullptr, 0, 0, nullptr, feat_f_nhwc, w->l1_out2[1].cout));
  return 0;
}

extern "C" {

size_t lb_backbone_workspace_bytes(const LbBackboneWeights* w, int N, int H, int W) {
  return backbone_workspace_bytes(w, N, H, W, 2);
}
int lb_backbone_forward(const LbBackboneWeights* w, const float* images, int N, int H, int W, float* feat_c_nhwc,
                        float* feat_f_nhwc, void* ws, size_t ws_bytes, void* stream) {
  return backbone_forward<2>(w, images, N, H, W, feat_c_nhwc, feat_f_nhwc, ws, ws_bytes, stream);
}
size_t lb_backbone_workspace_bytes_fp16(const LbBackboneWeights* w, int N, int H, int W) {
  return backbone_workspace_bytes(w, N, H, W, 1);
}
int lb_backbone_forward_fp16(const LbBackboneWeights* w, const float* images, int N, int H, int W, float* feat_c_nhwc,
                             float* feat_f_nhwc, void* ws, size_t ws_bytes, void* stream) {
  return backbone_forward<1>(w, images, N, H, W, feat_c_nhwc, feat_f_nhwc, ws, ws_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ coarse matching
struct CmWs {
  float2* row_part;  // [n_chunks][n*L]
  float2* col_part;  // [m_tiles][n*S]
  ArgPart* row_apart;
  ArgPart* col_apart;
  float *row_t, *col_t;          // additive terms used by the argmax pass (-LSE or potentials, masked)
  float *row_u, *col_v;          // true potentials (sinkhorn)
  float *row_key, *col_key;
  int *row_arg, *col_arg;
  float *bin_u, *bin_v;          // dustbin potentials [n]
  uint8_t *row_dead, *col_dead;
  uint8_t* flag;
  float* conf;
  int *ext0, *ext1;
  int* blk_counts;               // per-block match counts of the ordered compaction
};
constexpr int kMaxChunks = 32;

static void carve_cm(Bump& b, CmWs& w, int n, int L, int S) {
  const size_t nl = static_cast<size_t>(n) * L, ns = static_cast<size_t>(n) * S;
  const int m_tiles = (L + kBlockM - 1) / kBlockM;
  w.row_part = b.take<float2>(nl * kMaxChunks);
  w.col_part = b.take<float2>(ns * m_tiles);
  w.row_apart = b.take<ArgPart>(nl * kMaxChunks);
  w.col_apart = b.take<ArgPart>(ns * m_tiles);
  w.row_t = b.take<float>(nl);
  w.col_t = b.take<float>(ns);
  w.row_u = b.take<float>(nl);
  w.col_v = b.take<float>(ns);
  w.row_key = b.take<float>(nl);
  w.col_key = b.take<float>(ns);
  w.row_arg = b.take<int>(nl);
  w.col_arg = b.take<int>(ns);
  w.bin_u = b.take<float>(n);
  w.bin_v = b.take<float>(n);
  w.row_dead = b.take<uint8_t>(nl);
  w.col_dead = b.take<uint8_t>(ns);
  w.flag = b.take<uint8_t>(nl);
  w.conf = b.take<float>(nl);
  w.ext0 = b.take<int>(2 * static_cast<size_t>(n));
  w.ext1 = b.take<int>(2 * static_cast<size_t>(n));
  w.blk_counts = b.take<int>((nl + kCompactBlock - 1) / kCompactBlock + 1);
}

size_t lb_coarse_match_workspace_bytes(int n_pairs, int L, int S) {
  Bump b{nullptr, 0};
  CmWs w;
  carve_cm(b, w, n_pairs, L, S);
  return b.off + 256;
}

}  // extern "C"

// The coarse quantities of every row of every pair (n_pairs > 0), shared by lb_coarse_match* and lb_coarse_query: the
// score passes, the Sinkhorn iterations and prefilter, the optional conf_matrix, and match_flag_kernel's flag / conf.
// On return `w` holds them in the workspace and `sp` describes them.
// kP: operand planes of the score products (Operands); every pass recomputes the same logits.
// kG: guided (DESIGN.md §18): every score pass and the conf_matrix take the guided epilogue, with `guide` beside its
// arguments; the passes between them and match_flag_kernel are the same launches.
template <bool kG, class Plain, class Guided>
using GuideSel = std::conditional_t<kG, Guided, Plain>;
template <class Epi>
static typename Epi::Params epi_params(const typename Epi::Args& args, const GuideParams* guide) {
  if constexpr (std::is_same_v<typename Epi::Params, typename Epi::Args>) return args;
  else return typename Epi::Params{args, *guide};
}

template <int kP, bool kG>
static int coarse_rows(const LbCoarseMatchArgs* a, const GuideParams* guide, const DeviceScope& dev, void* ws,
                       size_t ws_bytes, cudaStream_t st, CmWs& w, SelectParams& sp) {
  const int n = a->n_pairs, L = a->L, S = a->S, C = a->C;
  if (L != a->h0c * a->w0c || S != a->h1c * a->w1c) return fail("L/S do not match the coarse grid sizes");
  if (C % kBlockK != 0) return fail("C=%d must be a multiple of %d", C, kBlockK);
  if ((a->mask0 == nullptr) != (a->mask1 == nullptr)) return fail("mask0 and mask1 must be given together");
  if (!ws) return fail("workspace pointer is null");
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  carve_cm(b, w, n, L, S);
  if (!b.ok) return fail("coarse-match workspace too small: need %zu bytes", lb_coarse_match_workspace_bytes(n, L, S));

  // the score products: row partials per chunk of n tiles (score.n_chunks), column partials per m tile
  constexpr int BN = 256;
  const long nl = static_cast<long>(n) * L, ns = static_cast<long>(n) * S;
  int chunks = pick_chunks(n * cdiv(L, kBlockM), cdiv(S, BN), dev.sms);
  if (chunks > kMaxChunks) chunks = kMaxChunks;
  const GemmShape score = gemm_shape<BN>(n, L, S, C, /*b_batched=*/true, chunks);
  const int n_chunks = score.n_chunks, m_tiles = score.m_tiles;

  Planes A{a->f0_hi, a->f0_lo, a->ld, static_cast<long>(L) * a->ld};
  Planes B{a->f1_hi, a->f1_lo, a->ld, static_cast<long>(S) * a->ld};
  const bool masked = a->mask0 != nullptr;
  if (masked) {
    LB_TRY(launch(TAG_NONE, mask_extent_kernel, n, 128, 0, st, a->mask0, a->h0c, a->w0c, w.ext0));
    LB_TRY(launch(TAG_NONE, mask_extent_kernel, n, 128, 0, st, a->mask1, a->h1c, a->w1c, w.ext1));
  }
  const int TB = 256;
  float conf_bias = 0.f;
  float alpha = 1.f;
  float scale = 1.f;
  const float* rowterm_for_conf = nullptr;

  if (a->match_type == LB_MATCH_DUAL_SOFTMAX) {
    // sim = <f0/sqrt(C), f1/sqrt(C)> / T                                    [coarse_matching.py:106-110]
    scale = 1.f / (static_cast<float>(C) * a->temperature);
    alpha = 2.f;
    const float* ct = nullptr;
    const float* rt = nullptr;
    if (masked) {  // padded rows / columns leave every normaliser      [coarse_matching.py:115-118]
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(ns, TB), TB, 0, st, nullptr, a->mask1, nullptr, ns, w.col_t));
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(nl, TB), TB, 0, st, nullptr, a->mask0, nullptr, nl, w.row_t));
      ct = w.col_t;
      rt = w.row_t;
    }
    using Epi = Operands<GuideSel<kG, EpiScoreLse<BN, true, true>, EpiScoreLseGuided<BN, true, true>>, kP>;
    const auto ep = epi_params<Epi>({scale, ct, rt, w.row_part, w.col_part}, guide);
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, score, ep, dev.sms, st)));
    // row_t = -rowLSE, col_t = -colLSE (kNegBig on padded entries)              [coarse_matching.py:119]
    LB_TRY(launch(TAG_NONE, lse_merge_kernel, cdiv(nl, TB), TB, 0, st, w.row_part, n_chunks, nl, 0.f, nullptr, nullptr,
                  L, a->mask0, w.row_t));
    LB_TRY(launch(TAG_NONE, lse_merge_kernel, cdiv(ns, TB), TB, 0, st, w.col_part, m_tiles, ns, 0.f, nullptr, nullptr,
                  S, a->mask1, w.col_t));
    rowterm_for_conf = w.row_t;
  } else if (a->match_type == LB_MATCH_SINKHORN) {
    // sim = <f0, f1> / C ; log-domain Sinkhorn with dustbins              [coarse_matching.py:121-131]
    if (!a->bin_score) return fail("sinkhorn matching needs bin_score");
    scale = 1.f / static_cast<float>(C);
    alpha = 1.f;
    const float norm = -logf(static_cast<float>(L + S));
    const float log_mu_bin = logf(static_cast<float>(S)) + norm;  // dustbin row mass   [superglue.py:161]
    const float log_nu_bin = logf(static_cast<float>(L)) + norm;  // dustbin column mass [superglue.py:162]
    // v = 0 (kNegBig on padded columns for the masked variant), bin_v = 0
    LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(ns, TB), TB, 0, st, nullptr, a->mask1, nullptr, ns, w.col_t));
    LB_TRY(launch(TAG_NONE, fill_kernel, cdiv(ns, TB), TB, 0, st, w.col_v, 0.f, ns));
    LB_TRY(launch(TAG_NONE, fill_kernel, cdiv(n, TB), TB, 0, st, w.bin_v, 0.f, n));
    // u = 0 (only observable with skh_iters == 0)
    LB_TRY(launch(TAG_NONE, fill_kernel, cdiv(nl, TB), TB, 0, st, w.row_u, 0.f, nl));
    LB_TRY(launch(TAG_NONE, fill_kernel, cdiv(n, TB), TB, 0, st, w.bin_u, 0.f, n));
    LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(nl, TB), TB, 0, st, nullptr, a->mask0, nullptr, nl, w.row_t));
    for (int it = 0; it < a->skh_iters; ++it) {
      // u_i = log_mu_i - LSE_j(Z_ij + v_j), j over S real columns + the dustbin column   [superglue.py:146]
      {
        using Epi = Operands<GuideSel<kG, EpiScoreLse<BN, true, false>, EpiScoreLseGuided<BN, true, false>>, kP>;
        const auto ep = epi_params<Epi>({scale, w.col_t, nullptr, w.row_part, w.col_part}, guide);
        LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, score, ep, dev.sms, st)));
        LB_TRY(launch(TAG_NONE, lse_merge_kernel, cdiv(nl, TB), TB, 0, st, w.row_part, n_chunks, nl, norm, a->bin_score,
                      w.bin_v, L, a->mask0, w.row_u));
      }
      // dustbin row: u_L = log_mu_L - LSE_j(bin + v_j, bin + bin_v)                         [superglue.py:146]
      LB_TRY(launch(TAG_NONE, bin_lse_kernel, n, 256, 0, st, w.col_v, S, a->bin_score, w.bin_v, log_mu_bin, w.bin_u));
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(nl, TB), TB, 0, st, w.row_u, a->mask0, nullptr, nl, w.row_t));
      // v_j = log_nu_j - LSE_i(Z_ij + u_i), i over L real rows + the dustbin row            [superglue.py:147]
      {
        using Epi = Operands<GuideSel<kG, EpiScoreLse<BN, false, true>, EpiScoreLseGuided<BN, false, true>>, kP>;
        const auto ep = epi_params<Epi>({scale, nullptr, w.row_t, w.row_part, w.col_part}, guide);
        LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, score, ep, dev.sms, st)));
        LB_TRY(launch(TAG_NONE, lse_merge_kernel, cdiv(ns, TB), TB, 0, st, w.col_part, m_tiles, ns, norm, a->bin_score,
                      w.bin_u, S, a->mask1, w.col_v));
      }
      LB_TRY(launch(TAG_NONE, bin_lse_kernel, n, 256, 0, st, w.row_u, L, a->bin_score, w.bin_u, log_nu_bin, w.bin_v));
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(ns, TB), TB, 0, st, w.col_v, a->mask1, nullptr, ns, w.col_t));
    }
    // assignment = exp(Z + u + v - norm)                                      [superglue.py:148,168-169]
    conf_bias = -norm;
    rowterm_for_conf = w.row_u;
  } else {
    return fail("unknown match_type %d", a->match_type);
  }

  // arg-maxima of the confidence along both directions                       [coarse_matching.py:187-189]
  const uint8_t* row_dead = nullptr;
  const uint8_t* col_dead = nullptr;
  const int passes = (a->match_type == LB_MATCH_SINKHORN && a->skh_prefilter) ? 2 : 1;
  for (int pass = 0; pass < passes; ++pass) {
    using Epi = Operands<GuideSel<kG, EpiScoreArgmax<BN>, EpiScoreArgmaxGuided<BN>>, kP>;
    const auto ep = epi_params<Epi>({scale, alpha, w.col_t, w.row_t, w.row_apart, w.col_apart}, guide);
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_ARGMAX, A, B, score, ep, dev.sms, st)));
    LB_TRY(launch(TAG_NONE, argmax_merge_kernel, cdiv(nl, TB), TB, 0, st, w.row_apart, n_chunks, nl, w.row_key,
                  w.row_arg));
    LB_TRY(launch(TAG_NONE, argmax_merge_kernel, cdiv(ns, TB), TB, 0, st, w.col_apart, m_tiles, ns, w.col_key,
                  w.col_arg));
    if (passes == 2 && pass == 0) {
      // prefilter: rows / columns whose best partner is the dustbin are zeroed  [coarse_matching.py:136-140]
      LB_TRY(launch(TAG_NONE, ot_dead_kernel, cdiv(nl, TB), TB, 0, st, w.row_key, a->bin_score, w.bin_v, L, nl,
                    w.row_dead));
      LB_TRY(launch(TAG_NONE, ot_dead_kernel, cdiv(ns, TB), TB, 0, st, w.col_key, a->bin_score, w.bin_u, S, ns,
                    w.col_dead));
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(nl, TB), TB, 0, st, w.row_u, a->mask0, w.row_dead, nl, w.row_t));
      LB_TRY(launch(TAG_NONE, mask_term_kernel, cdiv(ns, TB), TB, 0, st, w.col_v, a->mask1, w.col_dead, ns, w.col_t));
      row_dead = w.row_dead;
      col_dead = w.col_dead;
    }
  }

  if (a->conf_matrix) {   // opt-in materialisation of data['conf_matrix']         [coarse_matching.py:145]
    using Epi = Operands<GuideSel<kG, EpiConfStore<BN>, EpiConfStoreGuided<BN>>, kP>;
    // row_t / col_t hold -LSE (dual-softmax) or the Sinkhorn potentials, with padded / prefiltered entries disabled
    const auto ep = epi_params<Epi>({scale, alpha, conf_bias, w.row_t, w.col_t, a->conf_matrix}, guide);
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_ARGMAX, A, B, gemm_shape<BN>(n, L, S, C, /*b_batched=*/true), ep, dev.sms,
                                 st)));
  }

  sp.n_pairs = n; sp.L = L; sp.S = S;
  sp.h0c = a->h0c; sp.w0c = a->w0c; sp.h1c = a->h1c; sp.w1c = a->w1c;
  sp.border = a->border_rm;
  sp.thr = a->thr;
  sp.conf_bias = conf_bias;
  sp.row_key = w.row_key; sp.row_arg = w.row_arg; sp.col_arg = w.col_arg;
  sp.rowterm = rowterm_for_conf;
  sp.mask0 = a->mask0; sp.mask1 = a->mask1;
  sp.ext0 = masked ? w.ext0 : nullptr; sp.ext1 = masked ? w.ext1 : nullptr;
  sp.row_dead = row_dead; sp.col_dead = col_dead;
  sp.flag = w.flag; sp.conf = w.conf;
  return launch(TAG_NONE, match_flag_kernel, cdiv(nl, TB), TB, 0, st, sp);
}

// max_per_pair: 0 = every match; otherwise each pair keeps its max_per_pair most confident matches (match_cap_kernel).
// guide: NULL, or the guide of lb_coarse_match_guided.  search: NULL, or the search of lb_coarse_match_search
// (a->n_pairs a multiple of search->K): rectify_search_kernel keeps only the flags of each pair's winning candidate,
// before the cap.
template <int kP>
static int coarse_match(const LbCoarseMatchArgs* a, int max_per_pair, const GuideParams* guide, void* ws,
                        size_t ws_bytes, void* stream, const LbCoarseSearch* search = nullptr) {
  DeviceScope dev;
  LB_TRY(dev.bind(a->count));
  const int n = a->n_pairs, L = a->L, S = a->S;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0) {
    LB_CUDA(cudaMemsetAsync(a->count, 0, sizeof(int), st));
    return 0;
  }
  CmWs w;
  SelectParams sp;
  LB_TRY((guide ? coarse_rows<kP, true>(a, guide, dev, ws, ws_bytes, st, w, sp)
                : coarse_rows<kP, false>(a, nullptr, dev, ws, ws_bytes, st, w, sp)));
  const long nl = static_cast<long>(n) * L;
  if (search) {
    LB_TRY(launch(TAG_MATCH_SEARCH, rectify_search_kernel, n / search->K, kSearchBlock, 0, st, w.flag, L, search->K,
                  search->counts, search->choice));
  }
  if (max_per_pair > 0) {
    LB_TRY(launch(TAG_MATCH_CAP, match_cap_kernel, n, kCapBlock, 0, st, w.flag, w.conf, L, max_per_pair));
  }

  CompactParams cp;
  cp.total = nl; cp.L = L; cp.S = S; cp.w0c = a->w0c; cp.w1c = a->w1c;
  cp.scale = a->img_scale; cp.scale0 = a->scale0; cp.scale1 = a->scale1;
  cp.flag = w.flag; cp.conf = w.conf; cp.row_arg = w.row_arg;
  cp.capacity = a->capacity;
  cp.b_ids = a->b_ids; cp.i_ids = a->i_ids; cp.j_ids = a->j_ids;
  cp.mconf = a->mconf; cp.mkpts0 = a->mkpts0_c; cp.mkpts1 = a->mkpts1_c; cp.count = a->count;
  const int cblocks = cdiv(nl, kCompactBlock);
  LB_TRY(launch(TAG_NONE, match_count_kernel, cblocks, kCompactBlock, 0, st, w.flag, nl, w.blk_counts));
  LB_TRY(launch(TAG_NONE, match_scatter_kernel, cblocks, kCompactBlock, 0, st, cp, w.blk_counts));
  return 0;
}

// The guide of a guided entry (`who`), checked -> gp with the coarse keypoints' scales of `a`.
static int guide_params(const char* who, const LbCoarseMatchArgs* a, const LbCoarseGuide* g, GuideParams& gp) {
  if (!g || !g->model) return fail("%s: the guide model is null", who);
  if (g->kind != LB_GUIDE_HOMOGRAPHY && g->kind != LB_GUIDE_FUNDAMENTAL)
    return fail("%s: unknown guide kind %d", who, g->kind);
  if (!std::isfinite(g->radius) || !(g->radius > 0.f))
    return fail("%s: the radius must be finite and positive (got %g)", who, g->radius);
  gp = GuideParams{g->kind, g->model, g->radius, a->img_scale, a->scale0, a->scale1, a->w0c, a->w1c};
  return 0;
}

// The query arguments every query entry (`who`) checks before it launches anything.
static int check_query(const char* who, const LbCoarseQueryArgs* q) {
  if (!q->points0) return fail("%s: points0 is null", who);
  if (q->stride <= 0 || q->fine_scale <= 0.f || q->Hf0 <= 0 || q->Wf0 <= 0)
    return fail("%s: bad fine grid (stride %d, fine_scale %g, %d x %d)", who, q->stride, q->fine_scale, q->Hf0,
                q->Wf0);
  return 0;
}

// The query kernel of `side` on the coarse quantities coarse_rows left in `w`: coarse_query_kernel<0> for image0
// points, coarse_query_kernel<1> for image1 points.  conf = exp(key + term + bias) with the terms and the bias
// coarse_rows gives match_flag_kernel (DESIGN.md §22): -LSE and 0 for dual-softmax, the Sinkhorn potentials and
// log(L + S) for Sinkhorn.
static int query_launch(int side, const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, const CmWs& w,
                        cudaStream_t st) {
  const bool ot = a->match_type == LB_MATCH_SINKHORN;
  const float* rowterm = ot ? w.row_u : w.row_t;
  const float* colterm = ot ? w.col_v : w.col_t;
  const bool s1 = side == 1;
  QueryParams qp;
  qp.n_pairs = a->n_pairs; qp.Q = q->Q; qp.L = a->L; qp.S = a->S;
  qp.h0c = a->h0c; qp.w0c = a->w0c; qp.h1c = a->h1c; qp.w1c = a->w1c;
  // the *0 fields of `q` describe the queried image on either side, pts0_f receives the snapped query and pts1_c the
  // other image's window centre; centres and win_ids keep the (image0, image1) order
  qp.Hq = q->H0; qp.Wq = q->W0; qp.Hfq = q->Hf0; qp.Wfq = q->Wf0;
  qp.stride = q->stride; qp.s_c = a->img_scale; qp.s_f = q->fine_scale;
  qp.conf_bias = ot ? logf(static_cast<float>(a->L + a->S)) : 0.f;   // coarse_rows' -norm
  qp.points_q = q->points0; qp.valid_q = q->valid0;
  qp.scale0 = a->scale0; qp.scale1 = a->scale1; qp.mask_q = s1 ? a->mask1 : a->mask0;
  qp.key_q = s1 ? w.col_key : w.row_key; qp.arg_q = s1 ? w.col_arg : w.row_arg; qp.term_q = s1 ? colterm : rowterm;
  qp.key_o = s1 ? w.row_key : w.col_key; qp.arg_o = s1 ? w.row_arg : w.col_arg; qp.term_o = s1 ? rowterm : colterm;
  qp.flag = w.flag;
  qp.i_ids = q->i_ids; qp.j_ids = q->j_ids; qp.conf = q->conf;
  qp.mutual = q->mutual; qp.valid = q->valid; qp.inside = q->inside;
  qp.centres = q->centres; qp.win = q->win_ids; qp.pts_qf = q->pts0_f; qp.pts_oc = q->pts1_c;
  const long nq = static_cast<long>(a->n_pairs) * q->Q;
  return s1 ? launch(TAG_MATCH_QUERY, coarse_query_kernel<1>, cdiv(nq, 256), 256, 0, st, qp)
            : launch(TAG_MATCH_QUERY, coarse_query_kernel<0>, cdiv(nq, 256), 256, 0, st, qp);
}

// What a query entry does before the query kernel: the coarse rows, unguided or under a guide, or none (reuse).
enum QueryRows { kRowsPlain, kRowsGuided, kRowsReuse };

// The body of the query entries; `who` names the entry in the messages.  `g` is checked when `rows` is kRowsGuided,
// and `operand_planes` unless it is kRowsReuse.  The argument checks come before the return for Q = 0 or no pairs, so
// they hold on machines without a device; reuse checks everything before it binds one.
static int coarse_query(const char* who, const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, QueryRows rows,
                        const LbCoarseGuide* g, int side, int operand_planes, void* ws, size_t ws_bytes,
                        void* stream) {
  if (side != 0 && side != 1) return fail("%s: side must be 0 (image0) or 1 (image1) (got %d)", who, side);
  if (rows != kRowsReuse && operand_planes != 1 && operand_planes != 2)
    return fail("%s: operand_planes must be 1 (fp16) or 2 (split) (got %d)", who, operand_planes);
  GuideParams gp;
  if (rows == kRowsGuided) LB_TRY(guide_params(who, a, g, gp));
  if (q->Q <= 0 || a->n_pairs <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceScope dev;
  CmWs w;
  if (rows == kRowsReuse) {   // the workspace a preceding query entry filled for the same args on the same stream
    LB_TRY(check_query(who, q));
    if (a->L != a->h0c * a->w0c || a->S != a->h1c * a->w1c)
      return fail("%s: L/S do not match the coarse grid sizes", who);
    if (a->match_type != LB_MATCH_DUAL_SOFTMAX && a->match_type != LB_MATCH_SINKHORN)
      return fail("%s: unknown match_type %d", who, a->match_type);
    if (!ws) return fail("%s: workspace pointer is null", who);
    Bump b{static_cast<uint8_t*>(ws), ws_bytes};
    carve_cm(b, w, a->n_pairs, a->L, a->S);
    if (!b.ok)
      return fail("%s: workspace of %zu bytes is too small for %d pairs of %d x %d cells (need %zu)", who, ws_bytes,
                  a->n_pairs, a->L, a->S, lb_coarse_match_workspace_bytes(a->n_pairs, a->L, a->S));
    LB_TRY(dev.bind(q->i_ids));
  } else {
    LB_TRY(dev.bind(q->i_ids));
    LB_TRY(check_query(who, q));
    using Rows = int (*)(const LbCoarseMatchArgs*, const GuideParams*, const DeviceScope&, void*, size_t,
                         cudaStream_t, CmWs&, SelectParams&);
    static constexpr Rows kRows[2][2] = {{coarse_rows<1, false>, coarse_rows<1, true>},
                                         {coarse_rows<2, false>, coarse_rows<2, true>}};
    const bool guided = rows == kRowsGuided;
    SelectParams sp;
    LB_TRY(kRows[operand_planes - 1][guided](a, guided ? &gp : nullptr, dev, ws, ws_bytes, st, w, sp));
  }
  return query_launch(side, a, q, w, st);
}

extern "C" {

int lb_coarse_match(const LbCoarseMatchArgs* a, void* ws, size_t ws_bytes, void* stream) {
  return coarse_match<2>(a, 0, nullptr, ws, ws_bytes, stream);
}

int lb_coarse_match_capped(const LbCoarseMatchArgs* a, int max_per_pair, void* ws, size_t ws_bytes, void* stream) {
  if (max_per_pair < 1) return fail("lb_coarse_match_capped: max_per_pair must be at least 1 (got %d)", max_per_pair);
  return coarse_match<2>(a, max_per_pair, nullptr, ws, ws_bytes, stream);
}

int lb_coarse_match_fp16(const LbCoarseMatchArgs* a, int max_per_pair, void* ws, size_t ws_bytes, void* stream) {
  if (max_per_pair < 0) return fail("lb_coarse_match_fp16: max_per_pair must be 0 (no cap) or at least 1 (got %d)", max_per_pair);
  return coarse_match<1>(a, max_per_pair, nullptr, ws, ws_bytes, stream);
}

int lb_coarse_match_guided(const LbCoarseMatchArgs* a, const LbCoarseGuide* g, int max_per_pair, int fp16, void* ws,
                           size_t ws_bytes, void* stream) {
  GuideParams gp;
  LB_TRY(guide_params("lb_coarse_match_guided", a, g, gp));
  if (max_per_pair < 0)
    return fail("lb_coarse_match_guided: max_per_pair must be 0 (no cap) or at least 1 (got %d)", max_per_pair);
  if (fp16 != 0 && fp16 != 1) return fail("lb_coarse_match_guided: fp16 must be 0 (split) or 1 (got %d)", fp16);
  return fp16 ? coarse_match<1>(a, max_per_pair, &gp, ws, ws_bytes, stream)
              : coarse_match<2>(a, max_per_pair, &gp, ws, ws_bytes, stream);
}

int lb_coarse_match_search(const LbCoarseMatchArgs* a, const LbCoarseSearch* s, int max_per_pair, int fp16, void* ws,
                           size_t ws_bytes, void* stream) {
  if (!s || (a->n_pairs > 0 && (!s->counts || !s->choice)))
    return fail("lb_coarse_match_search: the search and its counts and choice outputs are required");
  if (s->K < 1) return fail("lb_coarse_match_search: K=%d must be at least 1", s->K);
  if (a->n_pairs % s->K != 0)
    return fail("lb_coarse_match_search: n_pairs=%d is not a multiple of K=%d", a->n_pairs, s->K);
  if (max_per_pair < 0)
    return fail("lb_coarse_match_search: max_per_pair must be 0 (no cap) or at least 1 (got %d)", max_per_pair);
  if (fp16 != 0 && fp16 != 1) return fail("lb_coarse_match_search: fp16 must be 0 (split) or 1 (got %d)", fp16);
  return fp16 ? coarse_match<1>(a, max_per_pair, nullptr, ws, ws_bytes, stream, s)
              : coarse_match<2>(a, max_per_pair, nullptr, ws, ws_bytes, stream, s);
}

int lb_coarse_query(const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, int operand_planes, void* ws,
                    size_t ws_bytes, void* stream) {
  return coarse_query("lb_coarse_query", a, q, kRowsPlain, nullptr, 0, operand_planes, ws, ws_bytes, stream);
}

int lb_coarse_query_guided(const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, const LbCoarseGuide* g,
                           int operand_planes, void* ws, size_t ws_bytes, void* stream) {
  return coarse_query("lb_coarse_query_guided", a, q, kRowsGuided, g, 0, operand_planes, ws, ws_bytes, stream);
}

int lb_coarse_query_side(const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, const LbCoarseGuide* g, int side,
                         int operand_planes, void* ws, size_t ws_bytes, void* stream) {
  return coarse_query("lb_coarse_query_side", a, q, g ? kRowsGuided : kRowsPlain, g, side, operand_planes, ws,
                      ws_bytes, stream);
}

int lb_coarse_query_reuse(const LbCoarseMatchArgs* a, const LbCoarseQueryArgs* q, int side, void* ws,
                          size_t ws_bytes, void* stream) {
  return coarse_query("lb_coarse_query_reuse", a, q, kRowsReuse, nullptr, side, 0, ws, ws_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ fine level
struct FpWs {
  __half* win_hi;   // [2*M*W*W, Cf] gathered windows
  __half* win_lo;
  float* gbias;     // [2*M, Cf] per-window bias of the merge
};
static void carve_fp(Bump& b, FpWs& w, long M, int W, int Cf) {
  const size_t rows = static_cast<size_t>(2) * M * W * W;
  w.win_hi = b.take<__half>(rows * Cf);
  w.win_lo = b.take<__half>(rows * Cf);
  w.gbias = b.take<float>(static_cast<size_t>(2) * M * Cf);
}

size_t lb_fine_preprocess_workspace_bytes(long M, int W, int Cf) {
  Bump b{nullptr, 0};
  FpWs w;
  carve_fp(b, w, M, W, Cf);
  return b.off + 256;
}

// img_idx0 / img_idx1: NULL, or pair b's windows are read from image img_idx0[b] of feat_f0 / img_idx1[b] of feat_f1.
// centres / inside: NULL, or the window centres come from the centre table (lb_fine_preprocess_centres); with img_idx0
// as well, from the table on bank images (lb_fine_preprocess_centres_indexed).
static int fine_preprocess(const LbFinePreprocessArgs* a, const int* img_idx0, const int* img_idx1, const int* centres,
                           const uint8_t* inside, void* ws, size_t ws_bytes, void* stream) {
  if (a->M <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(a->x_f32));
  if (a->Cf != 128 || a->Cc > 256) return fail("fine preprocess built for Cf=128, Cc<=256 (got %d, %d)", a->Cf, a->Cc);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int WW = a->W * a->W;
  const long rows = 2 * a->M * WW;
  if (!ws) return fail("workspace pointer is null");
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  FpWs w;
  carve_fp(b, w, a->M, a->W, a->Cf);
  if (!b.ok) return fail("fine-preprocess workspace too small");

  FineGatherParams g;
  g.feat0 = a->feat_f0; g.feat1 = a->feat_f1;
  g.sn0 = a->sn0; g.sc0 = a->sc0; g.sh0 = a->sh0; g.sw0 = a->sw0;
  g.sn1 = a->sn1; g.sc1 = a->sc1; g.sh1 = a->sh1; g.sw1 = a->sw1;
  g.Hf0 = a->Hf0; g.Wf0 = a->Wf0; g.Hf1 = a->Hf1; g.Wf1 = a->Wf1;
  g.w0c = a->w0c; g.w1c = a->w1c; g.stride = a->stride; g.W = a->W; g.Cf = a->Cf; g.M = a->M;
  g.b_ids = a->b_ids; g.i_ids = a->i_ids; g.j_ids = a->j_ids;
  g.out_hi = w.win_hi; g.out_lo = w.win_lo; g.ld = a->Cf;
  g.live = a->M_live;
  g.img_idx0 = img_idx0; g.img_idx1 = img_idx1;
  g.centres = centres; g.inside = inside;
  const bool vec8 = a->sc0 == 1 && a->sc1 == 1 && a->Cf % 8 == 0 && g.ld % 8 == 0 && a->sw0 % 4 == 0 && a->sw1 % 4 == 0 &&
                    a->sh0 % 4 == 0 && a->sh1 % 4 == 0 && a->sn0 % 4 == 0 && a->sn1 % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(a->feat_f0) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->feat_f1) & 15) == 0;
  const unsigned wins = static_cast<unsigned>(2 * a->M);
  const auto gather = centres && img_idx0 ? (vec8 ? fine_gather_vec8_kernel<true, true> : fine_gather_kernel<true, true>)
                      : centres          ? (vec8 ? fine_gather_vec8_kernel<false, true> : fine_gather_kernel<false, true>)
                      : img_idx0         ? (vec8 ? fine_gather_vec8_kernel<true> : fine_gather_kernel<true>)
                                         : (vec8 ? fine_gather_vec8_kernel<false> : fine_gather_kernel<false>);
  LB_TRY(launch(TAG_NONE, gather, wins, 256, 0, st, g));

  FineBiasParams fb;
  fb.feat_c = a->feat_c;
  fb.set1_row_base = static_cast<long>(a->n_pairs) * a->L;
  fb.L = a->L; fb.S = a->S; fb.Cc = a->Cc; fb.Cf = a->Cf; fb.M = a->M;
  fb.b_ids = a->b_ids; fb.i_ids = a->i_ids; fb.j_ids = a->j_ids;
  fb.WdT = a->down_wt; fb.bd = a->down_b; fb.Wm2T = a->merge_w2t; fb.bm = a->merge_b;
  fb.gbias = w.gbias;
  fb.live = a->M_live;
  LB_TRY(launch(TAG_NONE, fine_bias_kernel, static_cast<unsigned>(cdiv(2 * a->M, kFineBiasWin)), 128, 0, st, fb));

  // merge_feat over [window | coarse] = window @ Wm[:, :Cf]^T + per-window bias     [fine_preprocess.py:52-56]
  // With a device bound each side is one GEMM batch of M*WW rows (M = capacity) with its own live prefix.
  using Epi = EpiPlanes<128>;
  const int nb = a->M_live ? 2 : 1;
  const long rows_b = rows / nb;
  Planes A{w.win_hi, w.win_lo, a->Cf, nb > 1 ? rows_b * a->Cf : 0};
  Planes B{a->merge_w_hi, a->merge_w_lo, a->Cf, 0};
  Epi::Params ep{0, w.gbias, WW, a->merge_acc_scale, {}};
  LB_TRY(fill_out_maps(&ep.om, a->cat_hi, a->cat_lo, 2 * a->Cf, a->x_f32, a->Cf, a->Cf, rows_b, nb));
  return launch_gemm<128, Epi>(TAG_FINE_MERGE, A, B,
                               gemm_shape<128>(nb, static_cast<int>(rows_b), a->Cf, a->Cf, false, 0, a->M_live, WW),
                               ep, dev.sms, st);
}

int lb_fine_preprocess(const LbFinePreprocessArgs* a, void* ws, size_t ws_bytes, void* stream) {
  return fine_preprocess(a, nullptr, nullptr, nullptr, nullptr, ws, ws_bytes, stream);
}

int lb_fine_preprocess_indexed(const LbFinePreprocessArgs* a, const int* img_idx0, const int* img_idx1, void* ws,
                               size_t ws_bytes, void* stream) {
  if (a->M > 0 && (!img_idx0 || !img_idx1)) return fail("lb_fine_preprocess_indexed: img_idx0 and img_idx1 are required");
  return fine_preprocess(a, img_idx0, img_idx1, nullptr, nullptr, ws, ws_bytes, stream);
}

int lb_fine_preprocess_centres(const LbFinePreprocessArgs* a, const int* centres, const uint8_t* inside, void* ws,
                               size_t ws_bytes, void* stream) {
  if (a->M > 0 && (!centres || !inside)) return fail("lb_fine_preprocess_centres: centres and inside are required");
  if (a->M_live) return fail("lb_fine_preprocess_centres: M_live is not supported (every query has a window)");
  return fine_preprocess(a, nullptr, nullptr, centres, inside, ws, ws_bytes, stream);
}

int lb_fine_preprocess_centres_indexed(const LbFinePreprocessArgs* a, const int* centres, const uint8_t* inside,
                                       const int* img_idx0, const int* img_idx1, void* ws, size_t ws_bytes,
                                       void* stream) {
  if (a->M > 0 && (!centres || !inside || !img_idx0 || !img_idx1))
    return fail("lb_fine_preprocess_centres_indexed: centres, inside, img_idx0 and img_idx1 are required");
  if (a->M_live) return fail("lb_fine_preprocess_centres_indexed: M_live is not supported (every query has a window)");
  return fine_preprocess(a, img_idx0, img_idx1, centres, inside, ws, ws_bytes, stream);
}

int lb_fine_match(const LbFineMatchArgs* a, void* stream) {
  if (a->M <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(a->expec_f));
  if (a->W * a->W > 32) return fail("fine window %dx%d exceeds one warp", a->W, a->W);
  FineMatchParams p;
  p.f0 = a->f0; p.f1 = a->f1; p.W = a->W; p.C = a->C; p.M = a->M;
  p.scale = a->img_scale; p.scale1 = a->scale1; p.b_ids = a->b_ids;
  p.mkpts1_c = a->mkpts1_c; p.expec_f = a->expec_f; p.mkpts1_f = a->mkpts1_f;
  p.live = a->M_live;
  const int warps_per_block = 8;
  return launch(TAG_NONE, fine_match_kernel, cdiv(a->M, warps_per_block), warps_per_block * 32, 0,
                static_cast<cudaStream_t>(stream), p);
}

// ------------------------------------------------------------------------------------------------ evaluation
int lb_epipolar_errors(const float* mkpts0_f, const float* mkpts1_f, const long long* m_bids, long M, int n_pairs,
                       const float* T_0to1, const float* K0, const float* K1, float* epi_errs, void* stream) {
  if (M <= 0) return 0;
  DeviceScope dev;
  LB_TRY(dev.bind(epi_errs));
  if (!mkpts0_f || !mkpts1_f || !m_bids || !T_0to1 || !K0 || !K1) return fail("lb_epipolar_errors: null input");
  return launch(TAG_NONE, epipolar_error_kernel, cdiv(M, 256), 256, 0, static_cast<cudaStream_t>(stream), mkpts0_f,
                mkpts1_f, m_bids, M, n_pairs, T_0to1, K0, K1, epi_errs);
}

// ------------------------------------------------------------------------------------------------ two-view geometry
static size_t geometry_ws_layout(int B, int K, int iterations, size_t* off_col, size_t* off_n, size_t* off_best) {
  const size_t bk = static_cast<size_t>(B) * K;
  const size_t n_tiles = static_cast<size_t>(cdiv(iterations, kGeoHypPerBlock));
  *off_col = bk * sizeof(float4);
  *off_n = *off_col + ((bk * sizeof(int) + 15) & ~size_t(15));
  *off_best = *off_n + ((static_cast<size_t>(B) * sizeof(int) + 15) & ~size_t(15));
  return *off_best + static_cast<size_t>(B) * n_tiles * sizeof(GeoBest);
}

size_t lb_geometry_workspace_bytes(int B, int K, int iterations) {
  if (B <= 0 || K <= 0 || iterations <= 0) return 0;
  size_t a, b, c;
  return geometry_ws_layout(B, K, iterations, &a, &b, &c);
}

int lb_estimate_geometry(const float* pts0, const float* pts1, const uint8_t* valid, const int* pair_ids, int B, int K,
                         int model, float threshold, int iterations, unsigned long long seed, float* model_out,
                         uint8_t* mask_out, int* count_out, int* best_out, int* samples_out, void* ws, size_t ws_bytes,
                         void* stream) {
  if (model != LB_GEOMETRY_HOMOGRAPHY && model != LB_GEOMETRY_FUNDAMENTAL)
    return fail("lb_estimate_geometry: unknown model %d", model);
  const int s = model == LB_GEOMETRY_HOMOGRAPHY ? 4 : 8;
  if (B < 0 || B > 65535) return fail("lb_estimate_geometry: B=%d must be in [0, 65535]", B);
  if (K < s) return fail("lb_estimate_geometry: K=%d is below the minimal sample size %d", K, s);
  if (!(threshold > 0.0f) || !std::isfinite(threshold))
    return fail("lb_estimate_geometry: threshold must be a positive number of pixels");
  if (iterations <= 0) return fail("lb_estimate_geometry: iterations=%d must be positive", iterations);
  if (B == 0) return 0;
  if (!pts0 || !pts1 || !model_out || !mask_out || !count_out || !ws)
    return fail("lb_estimate_geometry: pts0, pts1, model_out, mask_out, count_out and ws are required");
  if ((reinterpret_cast<uintptr_t>(pts0) & 7) || (reinterpret_cast<uintptr_t>(pts1) & 7) ||
      (reinterpret_cast<uintptr_t>(ws) & 15))
    return fail("lb_estimate_geometry: points must be 8-byte and the workspace 16-byte aligned");
  size_t off_col, off_n, off_best;
  const size_t need = geometry_ws_layout(B, K, iterations, &off_col, &off_n, &off_best);
  if (ws_bytes < need) return fail("lb_estimate_geometry: workspace of %zu bytes, %zu needed", ws_bytes, need);
  DeviceScope dev;
  LB_TRY(dev.bind(model_out));
  GeoParams p;
  p.pts0 = pts0; p.pts1 = pts1; p.valid = valid; p.pair_ids = pair_ids;
  p.B = B; p.K = K; p.model = model; p.iterations = iterations; p.n_tiles = cdiv(iterations, kGeoHypPerBlock);
  p.seed = seed;
  p.thr2 = static_cast<double>(threshold) * threshold;
  char* w = static_cast<char*>(ws);
  p.compact = reinterpret_cast<float4*>(w);
  p.compact_col = reinterpret_cast<int*>(w + off_col);
  p.n_valid = reinterpret_cast<int*>(w + off_n);
  p.tile_best = reinterpret_cast<GeoBest*>(w + off_best);
  p.model_out = model_out; p.mask_out = mask_out; p.count_out = count_out;
  p.best_out = best_out; p.samples_out = samples_out;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TimedRange timed;   // the three launches are one record
  LB_TRY(timed.begin(TAG_GEOMETRY, st));
  LB_TRY(launch(TAG_NONE, geometry_compact_kernel, B, kGeoRefitThreads, 0, st, p));
  LB_TRY(launch(TAG_NONE, geometry_score_kernel, dim3(p.n_tiles, B), kGeoHypPerBlock, 0, st, p));
  LB_TRY(launch(TAG_NONE, geometry_refit_kernel, B, kGeoRefitThreads, 0, st, p));
  return timed.end();
}

// ------------------------------------------------------------------------------------------------ multi-GPU
int lb_comm_unique_id(char* id_out, const char* nccl_lib_path) {
  NcclApi* api = nccl_api(nccl_lib_path);
  if (!api) return fail("NCCL library not found (dlopen of libnccl.so.2 failed; set LOFTR_B200_NCCL_LIB)");
  NcclApi::UniqueId id;
  const int rc = api->GetUniqueId(&id);
  if (rc != 0) return fail("ncclGetUniqueId failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  memcpy(id_out, id.internal, LB_NCCL_UNIQUE_ID_BYTES);
  return 0;
}

int lb_comm_init(const char* id_bytes, int rank, int world, int device, const char* nccl_lib_path, void** comm_out) {
  if (!id_bytes || !comm_out || world <= 0 || rank < 0 || rank >= world) return fail("lb_comm_init: bad arguments");
  NcclApi* api = nccl_api(nccl_lib_path);
  if (!api) return fail("NCCL library not found (dlopen of libnccl.so.2 failed; set LOFTR_B200_NCCL_LIB)");
  DeviceScope dev;
  LB_TRY(dev.bind_device(device));
  NcclApi::UniqueId id;
  memcpy(id.internal, id_bytes, LB_NCCL_UNIQUE_ID_BYTES);
  void* nccl = nullptr;
  const int rc = api->CommInitRank(&nccl, world, id, rank);
  if (rc != 0) return fail("ncclCommInitRank failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  *comm_out = new LbComm{nccl, rank, world, device};
  return 0;
}

int lb_comm_destroy(void* comm) {
  if (!comm) return 0;
  LbComm* c = static_cast<LbComm*>(comm);
  NcclApi* api = nccl_api(nullptr);
  if (api && c->nccl) api->CommDestroy(c->nccl);
  delete c;
  return 0;
}

int lb_pack_matches(const float* mkpts0_f, const float* mkpts1_f, const float* mconf, const long long* m_bids,
                    long count, int pair_offset, float* wire, long capacity, void* stream) {
  DeviceScope dev;
  LB_TRY(dev.bind(wire));
  if (count > capacity) return fail("lb_pack_matches: %ld matches exceed the wire capacity %ld", count, capacity);
  if (count > 0 && (!mkpts0_f || !mkpts1_f || !mconf || !m_bids)) return fail("lb_pack_matches: null input");
  const long n = count > 0 ? count : 1;
  return launch(TAG_NONE, pack_matches_kernel, cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream), mkpts0_f,
                mkpts1_f, mconf, m_bids, count, pair_offset, wire, capacity);
}

int lb_allgather_matches(void* comm, const float* wire_send, float* wire_recv, long capacity, void* stream) {
  if (!comm) return fail("lb_allgather_matches: null communicator");
  LbComm* c = static_cast<LbComm*>(comm);
  DeviceScope dev;
  LB_TRY(dev.bind(wire_recv));
  NcclApi* api = nccl_api(nullptr);
  if (!api) return fail("NCCL library not loaded");
  const size_t count = static_cast<size_t>(1 + capacity) * kWireCols;
  const int rc = api->AllGather(wire_send, wire_recv, count, kNcclFloat32, c->nccl, static_cast<cudaStream_t>(stream));
  if (rc != 0) return fail("ncclAllGather failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  return 0;
}

int lb_unpack_matches(const float* wire_recv, int world, long capacity, float* mkpts0_f, float* mkpts1_f, float* mconf,
                      long long* m_bids, long out_capacity, int* counts_out, void* stream) {
  DeviceScope dev;
  LB_TRY(dev.bind(wire_recv));
  if (world <= 0 || capacity < 0) return fail("lb_unpack_matches: bad arguments");
  const long n = capacity > 0 ? capacity : 1;
  return launch(TAG_NONE, unpack_matches_kernel, dim3(cdiv(n, 256), world), 256, 0, static_cast<cudaStream_t>(stream),
                wire_recv, world, capacity, mkpts0_f, mkpts1_f, mconf, m_bids, out_capacity, counts_out);
}

}  // extern "C"
