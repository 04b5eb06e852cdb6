// Host side of the C ABI (include/loftr_b200.h): tensor-map construction, kernel launches and the
// per-stage orchestration of the matching hot path.  No torch types; raw device pointers + a stream.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/loftr_b200.h"
#include "epilogues.cuh"
#include "gemm_split.cuh"
#include "simt_kernels.cuh"
#include "kv_gemm.cuh"
#include "full_attn.cuh"
#include "stem_tc.cuh"
#include "comm.cuh"

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

#define LB_LAUNCHED()                 \
  do {                                \
    g_launches.fetch_add(1);          \
    LB_CUDA(cudaGetLastError());      \
  } while (0)

// ------------------------------------------------------------------------------------------------ timing hook
// Optional per-launch CUDA-event timing of the tensor-core kernels (bench.py's roofline leg): events are
// recorded on the launching stream right around the kernel, and only while timing is enabled.
enum Tag { TAG_GEMM_TEST = 0, TAG_PROJ, TAG_MERGE_LN, TAG_MLP1, TAG_MLP2_LN, TAG_SCORE_LSE, TAG_SCORE_ARGMAX,
           TAG_FINE_MERGE, TAG_CONV, TAG_KV, TAG_QATTN, TAG_FULL_ATTN, TAG_COUNT };
static const char* kTagNames[TAG_COUNT] = {"gemm_test", "proj_act", "merge_ln", "mlp1_relu", "mlp2_ln_res",
                                           "score_lse", "score_argmax", "fine_merge", "backbone_conv",
                                           "tf_kv_proj_fused", "tf_q_attn_fused", "tf_full_attn"};
struct TimingRec {
  cudaEvent_t e0, e1;
  int tag;
};
static bool g_timing = false;
static std::vector<TimingRec> g_recs;
static std::mutex g_timing_mu;
// Around a launch on `st`: events are only created and recorded while timing is enabled.
static int timing_begin(TimingRec& rec, cudaStream_t st) {
  if (!g_timing) return 0;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaError_t e = cudaStreamIsCapturing(st, &cs);
  if (e != cudaSuccess) return fail("cudaStreamIsCapturing failed: %s", cudaGetErrorString(e));
  if (cs != cudaStreamCaptureStatusNone)
    return fail("kernel timing is enabled (lb_timing_enable) but the stream is being captured into a CUDA graph: "
                "timing events cannot be recorded into a graph; disable timing before capture");
  if (cudaEventCreate(&rec.e0) != cudaSuccess || cudaEventCreate(&rec.e1) != cudaSuccess ||
      cudaEventRecord(rec.e0, st) != cudaSuccess)
    return fail("timing event set-up failed");
  return 0;
}
static int timing_end(const TimingRec& rec, cudaStream_t st) {
  if (!g_timing) return 0;
  if (cudaEventRecord(rec.e1, st) != cudaSuccess) return fail("timing event record failed");
  std::lock_guard<std::mutex> lk(g_timing_mu);
  g_recs.push_back(rec);
  return 0;
}

// The library carries its own (static) CUDA runtime, whose notion of "current device" is independent of the
// caller's (e.g. torch's).  Every entry point therefore binds the calling thread to the device that owns the
// buffers it was given -- otherwise a process working on cuda:1 would launch on device 0 through the legacy
// default stream.
// The previous device of the calling thread is restored when the entry point returns (RAII), so a caller whose
// current device differs from the buffers' device is left undisturbed.
constexpr int kMaxDevices = 64;
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
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
    LB_CUDA(cudaGetDevice(&prev));
    if (prev != attr.device) {
      LB_CUDA(cudaSetDevice(attr.device));
      switched = true;
    }
    return 0;
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

static int device_check(int* sm_count) {
  static std::mutex mu;
  static int sms[kMaxDevices] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail("no CUDA device: %s", cudaGetErrorString(e));
  if (dev < 0 || dev >= kMaxDevices) return fail("device index %d out of range", dev);
  std::lock_guard<std::mutex> lk(mu);
  if (sms[dev] == 0) {
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return fail("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
      return fail("loftr_b200 requires an sm_90 (H100) device, found sm_%d%d; there is no fallback", prop.major,
                  prop.minor);
    sms[dev] = prop.multiProcessorCount;
  }
  *sm_count = sms[dev];
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

// fp16 plane viewed as [batches][rows][K] with row stride ld and batch stride bs (elements);
// box = 64 (K) x box_rows x 1, 128-byte swizzle, out-of-range elements read as zero.
static CUtensorMapSwizzle swizzle_for(int box_k) {
  return box_k * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : box_k * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}
static int make_map(CUtensorMap* m, const void* base, long K, long rows, long batches, long ld, long bs,
                    int box_rows, int box_k = kBlockK) {
  auto enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("plane pointer not 16-byte aligned");
  if ((ld * 2) % 16 != 0 || (bs * 2) % 16 != 0) return fail("plane strides must be multiples of 8 elements");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(batches)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld * 2), static_cast<cuuint64_t>((bs > 0 ? bs : rows * ld) * 2)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box_k), static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(box_k),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult %d", static_cast<int>(r));
  return 0;
}

// NHWC fp16 plane viewed as [N][H][W][C] (row stride ld elements); box = 64 channels x (16*stride) x (8*stride)
// x 1 with element strides (1, stride, stride, 1): an 8 x 16 patch of (strided) pixels per load.
static int make_map_nhwc(CUtensorMap* m, const void* base, int C, int W, int H, int N, long ld, int stride,
                         int box_c = kBlockK) {
  auto enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("plane pointer not 16-byte aligned");
  if ((ld * 2) % 16 != 0) return fail("NHWC channel stride must be a multiple of 8 elements (got %ld)", ld);
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(ld * 2), static_cast<cuuint64_t>(ld * 2 * W),
                           static_cast<cuuint64_t>(ld * 2 * W) * H};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(box_c), static_cast<cuuint32_t>(kConvTileW * stride),
                       static_cast<cuuint32_t>(kConvTileH * stride), 1};
  cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(box_c),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (NHWC) failed with CUresult %d", static_cast<int>(r));
  return 0;
}

// ---- output tensor maps for the TMA-store epilogues (epilogues.cuh OutMaps)
// [batches][rows][cols] matrix (row stride ld, batch stride bs elements; bs = 0 -> rows * ld): box 32 x 32 x 1,
// 64-byte swizzle for fp16 planes, 128-byte swizzle for fp32
static int make_out_map(CUtensorMap* m, const void* base, bool f32, long cols, long rows, long batches, long ld, long bs) {
  auto enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
  const int esz = f32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * esz) % 16 != 0 || (bs * esz) % 16 != 0)
    return fail("TMA-store output not 16-byte aligned");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(batches)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld * esz), static_cast<cuuint64_t>((bs > 0 ? bs : rows * ld) * esz)};
  cuuint32_t box[3] = {32, 32, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (output) failed with CUresult %d", static_cast<int>(r));
  return 0;
}
// NHWC [N][H][W][C] (pixel stride ld elements): box 32 channels x 16 x 2 pixels x 1 image
static int make_out_map_nhwc(CUtensorMap* m, const void* base, bool f32, int C, int W, int H, int N, long ld) {
  auto enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
  const int esz = f32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * esz) % 16 != 0) return fail("TMA-store NHWC output not 16-byte aligned");
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(ld * esz), static_cast<cuuint64_t>(ld * esz) * W,
                           static_cast<cuuint64_t>(ld * esz) * W * H};
  cuuint32_t box[4] = {32, static_cast<cuuint32_t>(kConvTileW), 2, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (NHWC output) failed with CUresult %d", static_cast<int>(r));
  return 0;
}
// planes (+ optional fp32) of a [batches][rows][cols] output
static int fill_out_maps(OutMaps* om, const void* hi, const void* lo, long ld_pl, const float* f32, long ld_f32, long cols,
                         long rows, long batches) {
  memset(om, 0, sizeof(*om));
  om->dims = 3;
  if (hi) {
    LB_TRY(make_out_map(&om->hi, hi, false, cols, rows, batches, ld_pl, 0));
    LB_TRY(make_out_map(&om->lo, lo, false, cols, rows, batches, ld_pl, 0));
    om->use |= 1;
  }
  if (f32) {
    LB_TRY(make_out_map(&om->f32, f32, true, cols, rows, batches, ld_f32, 0));
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
  CUtensorMap a_hi, a_lo, b_hi, b_lo;      // 64-element k-blocks
  CUtensorMap ar_hi, ar_lo, br_hi, br_lo;  // convolution channel remainder (16-element boxes); copies of the above if unused
};

template <int BN, class Epi>
static int launch_raw(int tag, const GemmMaps& maps, const GemmShape& s, const typename Epi::Params& ep, int sms,
                      cudaStream_t st) {
  using S = GemmSmem<BN, Epi::kSmemBytes>;
  constexpr int smem_bytes = S::kRingBytes + S::kBarBytes + Epi::kSmemBytes;
  static_assert(smem_bytes <= 232448, "shared memory budget exceeded");
  auto kern = gemm_split_kernel<BN, Epi>;
  static bool configured[kMaxDevices] = {false};  // per instantiation and device
  int dev = 0;
  LB_CUDA(cudaGetDevice(&dev));
  if (!configured[dev]) {
    LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    configured[dev] = true;
  }
  const long items = static_cast<long>(s.batches) * s.m_tiles * s.n_chunks;
  const int grid = static_cast<int>(items < sms ? items : sms);
  TimingRec rec{nullptr, nullptr, tag};
  LB_TRY(timing_begin(rec, st));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  cfg.attrs = attr;
  cfg.numAttrs = 0;
  // programmatic dependent launch of the tensor-core kernels (gemm_split.cuh): the next kernel's set-up overlaps this
  // one's tail.  LOFTR_B200_PDL=0 disables it.
  static int pdl = -1;
  if (pdl < 0) {
    const char* e = getenv("LOFTR_B200_PDL");
    pdl = e ? (atoi(e) != 0 ? 1 : 0) : 1;
  }
  if (pdl) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 1;
  }
  LB_CUDA(cudaLaunchKernelEx(&cfg, kern, maps.a_hi, maps.a_lo, maps.b_hi, maps.b_lo, maps.ar_hi, maps.ar_lo, maps.br_hi,
                             maps.br_lo, s, ep));
  LB_LAUNCHED();
  return timing_end(rec, st);
}

// live / live_unit_rows: optional device bound on the rows of every batch (GemmShape::live_count)
template <int BN, class Epi>
static int launch_gemm(int tag, const Planes& A, const Planes& B, int batches, int M, int N, int K, int n_chunks,
                       const typename Epi::Params& ep, cudaStream_t st, const int* live = nullptr,
                       int live_unit_rows = 0) {
  int sms = 0;
  LB_TRY(device_check(&sms));
  if (K % kBlockK != 0 || K <= 0) return fail("K=%d must be a positive multiple of %d", K, kBlockK);
  if (M <= 0 || N <= 0 || batches <= 0) return 0;  // nothing to do
  if (live && !EpiRowBound<Epi>::value) return fail("this GEMM epilogue is built without a device row bound");
  GemmShape s;
  s.batches = batches;
  s.M = M;
  s.N = N;
  s.K = K;
  s.b_batched = B.batch_stride > 0 ? 1 : 0;
  s.m_tiles = (M + kBlockM - 1) / kBlockM;
  s.n_tiles = (N + BN - 1) / BN;
  if (n_chunks <= 0 || n_chunks > s.n_tiles) n_chunks = s.n_tiles;
  s.tiles_per_chunk = (s.n_tiles + n_chunks - 1) / n_chunks;
  s.n_chunks = (s.n_tiles + s.tiles_per_chunk - 1) / s.tiles_per_chunk;
  s.conv = ConvGeom{0, 0, 0, 0, 0, 0, 0, 0, 0};
  s.live_count = live;
  s.live_unit_rows = live_unit_rows;

  GemmMaps mp;
  LB_TRY(make_map(&mp.a_hi, A.hi, K, M, batches, A.ld, A.batch_stride, kBlockM));
  LB_TRY(make_map(&mp.a_lo, A.lo, K, M, batches, A.ld, A.batch_stride, kBlockM));
  const int bb = s.b_batched ? batches : 1;
  LB_TRY(make_map(&mp.b_hi, B.hi, K, N, bb, B.ld, B.batch_stride, BN));
  LB_TRY(make_map(&mp.b_lo, B.lo, K, N, bb, B.ld, B.batch_stride, BN));
  mp.ar_hi = mp.a_hi; mp.ar_lo = mp.a_lo; mp.br_hi = mp.b_hi; mp.br_lo = mp.b_lo;
  return launch_raw<BN, Epi>(tag, mp, s, ep, sms, st);
}

// Implicit-GEMM convolution launch: in = NHWC planes [N, H_in, W_in, ld_in] with Cin valid channels; weights =
// main planes [Cout, taps * cin_blocks * 64] (+ remainder planes [Cout, taps * 16], see lb_conv_layout); out pixel
// grid H_out x W_out.
struct ConvDesc {
  int N, H_in, W_in, Cin, H_out, W_out, Cout, ksize, stride, pad;
};
// K layout of a convolution's implicit GEMM: `cin_blocks` 64-channel blocks per tap, plus `rem` (<= 16) remainder
// channels per tap that travel as 16-channel boxes (gemm_split.cuh ConvGeom).
static void conv_layout(int cin, int* cin_blocks, int* rem) {
  const int r = cin % kBlockK;
  if (kBlockK == 64 && cin > kBlockK && r > 0 && r <= kRemChannels) {
    *cin_blocks = cin / kBlockK;
    *rem = r;
  } else {
    *cin_blocks = (cin + kBlockK - 1) / kBlockK;
    *rem = 0;
  }
}
template <int BN, int kUpMode = 0>
static int launch_conv(const Planes& in, const Planes& wgt, const Planes& wgt_rem, const ConvDesc& d,
                       const typename EpiConv<BN, kUpMode>::Params& ep_in, cudaStream_t st) {
  using Epi = EpiConv<BN, kUpMode>;
  int sms = 0;
  LB_TRY(device_check(&sms));
  GemmShape s;
  int cin_blocks = 0, rem = 0;
  conv_layout(d.Cin, &cin_blocks, &rem);
  const int taps = d.ksize * d.ksize;
  const int tiles_h = (d.H_out + kConvTileH - 1) / kConvTileH;
  const int tiles_w = (d.W_out + kConvTileW - 1) / kConvTileW;
  s.batches = d.N;
  s.M = tiles_h * tiles_w * kBlockM;
  s.N = d.Cout;
  s.K = taps * cin_blocks * kBlockK;
  s.b_batched = 0;
  s.m_tiles = tiles_h * tiles_w;
  s.n_tiles = (d.Cout + BN - 1) / BN;
  s.n_chunks = s.n_tiles;
  s.tiles_per_chunk = 1;
  const int rem_groups = rem ? (taps + kRemTapsPerStage - 1) / kRemTapsPerStage : 0;
  s.conv = ConvGeom{1, tiles_w, d.stride, d.pad, d.ksize, cin_blocks, taps, taps * cin_blocks, rem_groups};
  s.live_count = nullptr;
  s.live_unit_rows = 0;
  if (rem && (!wgt_rem.hi || !wgt_rem.lo)) return fail("convolution with Cin=%d needs remainder weight planes", d.Cin);
  GemmMaps mp;
  LB_TRY(make_map_nhwc(&mp.a_hi, in.hi, d.Cin, d.W_in, d.H_in, d.N, in.ld, d.stride));
  LB_TRY(make_map_nhwc(&mp.a_lo, in.lo, d.Cin, d.W_in, d.H_in, d.N, in.ld, d.stride));
  LB_TRY(make_map(&mp.b_hi, wgt.hi, s.K, d.Cout, 1, wgt.ld, 0, BN));
  LB_TRY(make_map(&mp.b_lo, wgt.lo, s.K, d.Cout, 1, wgt.ld, 0, BN));
  if (rem) {
    LB_TRY(make_map_nhwc(&mp.ar_hi, in.hi, d.Cin, d.W_in, d.H_in, d.N, in.ld, d.stride, kRemChannels));
    LB_TRY(make_map_nhwc(&mp.ar_lo, in.lo, d.Cin, d.W_in, d.H_in, d.N, in.ld, d.stride, kRemChannels));
    LB_TRY(make_map(&mp.br_hi, wgt_rem.hi, taps * kRemChannels, d.Cout, 1, wgt_rem.ld, 0, BN, kRemChannels));
    LB_TRY(make_map(&mp.br_lo, wgt_rem.lo, taps * kRemChannels, d.Cout, 1, wgt_rem.ld, 0, BN, kRemChannels));
  } else {
    mp.ar_hi = mp.a_hi; mp.ar_lo = mp.a_lo; mp.br_hi = mp.b_hi; mp.br_lo = mp.b_lo;
  }
  typename Epi::Params ep = ep_in;
  ep.H_out = d.H_out;
  ep.W_out = d.W_out;
  ep.tiles_w = tiles_w;
  return launch_raw<BN, Epi>(TAG_CONV, mp, s, ep, sms, st);
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

static inline int cdiv(long a, long b) { return static_cast<int>((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------------ transformer
struct TfWs {
  float* qkv;       // fine only: [R, 3C]
  __half* att_hi;   // [R, C]
  __half* att_lo;
  __half* h_hi;     // [R, 2C]
  __half* h_lo;
  float* kv;        // [2*n_groups, H, D*D + D]
  float* kv_part;   // coarse only: [2*n_groups, max(m_tiles, kKvSplits), H, per] (K^T V split partials)
};
// kv_gemm_kernel sums K^T V over at most max(m_tiles, kKvSplits) row splits per group.  That bound sizes kv_part here
// and caps `splits` in tf_linear_attention_coarse; `splits` fixes the summation order of K^T V, so changing either
// formula changes the output bits.
constexpr int kKvSplits = 8;

static void carve_tf(Bump& b, TfWs& w, int C, int H, long R, int n_groups, bool coarse, int max_group_rows) {
  const int D = C / H;
  // fp32 q|k|v of the fine (window) transformer; the coarse projections write planes
  w.qkv = coarse ? nullptr : b.take<float>(static_cast<size_t>(R) * 3 * C);
  w.att_hi = b.take<__half>(static_cast<size_t>(R) * C);
  w.att_lo = b.take<__half>(static_cast<size_t>(R) * C);
  w.h_hi = b.take<__half>(static_cast<size_t>(R) * 2 * C);
  w.h_lo = b.take<__half>(static_cast<size_t>(R) * 2 * C);
  w.kv = b.take<float>(static_cast<size_t>(2) * n_groups * H * (D * D + D));
  const size_t tiles = static_cast<size_t>((max_group_rows + kBlockM - 1) / kBlockM);
  const size_t parts = tiles > static_cast<size_t>(kKvSplits) ? tiles : static_cast<size_t>(kKvSplits);
  w.kv_part = coarse ? b.take<float>(static_cast<size_t>(2) * n_groups * H * parts * (D * D + D)) : nullptr;
}

template <int BN>
static int tf_layer_pass(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st, const TfWs& w,
                         long x_base, long x_rows, int x_group_rows, long s_base, long s_rows, int s_group_rows,
                         int n_groups_x, bool self_pass, bool write_f32, cudaStream_t stream, const int* live,
                         int live_cap, bool full);


// ------------------------------------------------------------------------------------------------ backbone
// ResNetFPN_8_2 forward (reference src/loftr/backbone/resnet_fpn.py:43-118) on tensor cores: every 3x3 / 1x1
// convolution is an implicit GEMM through gemm_split_kernel<., EpiConv> (BatchNorm, ReLU / LeakyReLU, residual
// add and the FPN upsample-add fused in the epilogue); activations live as NHWC fp16 hi/lo planes.
struct BbBuf {
  __half* hi;
  __half* lo;
  int ld;
};
static inline int pad8(int c) { return (c + 7) & ~7; }
static BbBuf bb_take(Bump& b, long pixels, int C) {
  BbBuf r;
  r.ld = pad8(C);
  r.hi = b.take<__half>(static_cast<size_t>(pixels) * r.ld);
  r.lo = b.take<__half>(static_cast<size_t>(pixels) * r.ld);
  return r;
}
struct BbWs {
  BbBuf s0, t1, a1, x1;                 // 1/2 resolution, d1 channels
  BbBuf t2, dn2, a2, x2;                // 1/4, d2
  BbBuf t3, dn3, a3, x3, x3o;           // 1/8, d3
  BbBuf x2l, m2, x2o;                   // 1/4: d3, d3, d2
  BbBuf x1l, m1;                        // 1/2: d2, d2
};
static void carve_bb(Bump& b, BbWs& w, int N, int H, int W, int d1, int d2, int d3) {
  const long p2 = static_cast<long>(N) * (H / 2) * (W / 2), p4 = static_cast<long>(N) * (H / 4) * (W / 4),
             p8 = static_cast<long>(N) * (H / 8) * (W / 8);
  w.s0 = bb_take(b, p2, d1); w.t1 = bb_take(b, p2, d1); w.a1 = bb_take(b, p2, d1); w.x1 = bb_take(b, p2, d1);
  w.t2 = bb_take(b, p4, d2); w.dn2 = bb_take(b, p4, d2); w.a2 = bb_take(b, p4, d2); w.x2 = bb_take(b, p4, d2);
  w.t3 = bb_take(b, p8, d3); w.dn3 = bb_take(b, p8, d3); w.a3 = bb_take(b, p8, d3); w.x3 = bb_take(b, p8, d3);
  w.x3o = bb_take(b, p8, d3);
  w.x2l = bb_take(b, p4, d3); w.m2 = bb_take(b, p4, d3); w.x2o = bb_take(b, p4, d2);
  w.x1l = bb_take(b, p2, d2); w.m1 = bb_take(b, p2, d2);
}

struct ConvRun {
  const LbConvWeights* w;
  BbBuf in;
  int H_in, W_in;
  int act;
  const BbBuf* res;
  const BbBuf* up;
  int up_h, up_w;
  const BbBuf* out;
  float* out_f32;
  int f32_ld;
};
static int run_conv(const ConvRun& r, int N, cudaStream_t st) {
  const LbConvWeights& w = *r.w;
  ConvDesc d;
  d.N = N; d.H_in = r.H_in; d.W_in = r.W_in; d.Cin = w.cin;
  d.ksize = w.ksize; d.stride = w.stride; d.pad = w.ksize / 2;
  d.H_out = (r.H_in + 2 * d.pad - w.ksize) / w.stride + 1;
  d.W_out = (r.W_in + 2 * d.pad - w.ksize) / w.stride + 1;
  d.Cout = w.cout;
  int cin_blocks = 0, rem = 0;
  conv_layout(w.cin, &cin_blocks, &rem);
  const int taps = w.ksize * w.ksize;
  Planes in{r.in.hi, r.in.lo, r.in.ld, 0};
  Planes wg{w.w_hi, w.w_lo, static_cast<long>(taps) * cin_blocks * kBlockK, 0};
  Planes wr{w.wr_hi, w.wr_lo, static_cast<long>(taps) * kRemChannels, 0};
  // NHWC output maps of the TMA-store epilogue (planes and / or fp32 feature map)
  OutMaps om;
  memset(&om, 0, sizeof(om));
  om.dims = 4;
  if (r.out) {
    LB_TRY(make_out_map_nhwc(&om.hi, r.out->hi, false, d.Cout, d.W_out, d.H_out, N, r.out->ld));
    LB_TRY(make_out_map_nhwc(&om.lo, r.out->lo, false, d.Cout, d.W_out, d.H_out, N, r.out->ld));
    om.use |= 1;
  }
  if (r.out_f32) {
    LB_TRY(make_out_map_nhwc(&om.f32, r.out_f32, true, d.Cout, d.W_out, d.H_out, N, r.f32_ld));
    om.use |= 2;
  }
#define LB_CONV_CASE_UP(BN, UP)                                                                                       \
  {                                                                                                                   \
    EpiConv<BN, UP>::Params ep{w.scale, w.shift, r.act, r.res ? r.res->hi : nullptr, r.res ? r.res->lo : nullptr,     \
                               r.res ? r.res->ld : 0, r.up ? r.up->hi : nullptr, r.up ? r.up->lo : nullptr,          \
                               r.up ? r.up->ld : 0, r.up_h, r.up_w, r.out ? r.out->hi : nullptr,                      \
                               r.out ? r.out->lo : nullptr, r.out ? r.out->ld : 0, r.out_f32, r.f32_ld, 0, 0, 0, om, \
                               um};                                                                                   \
    return launch_conv<BN, UP>(in, wg, wr, d, ep, st);                                                                \
  }
#define LB_CONV_CASE(BN)                                                                                              \
  {                                                                                                                   \
    if (r.up) LB_CONV_CASE_UP(BN, 2)                                                                                  \
    LB_CONV_CASE_UP(BN, 0)                                                                                            \
  }
  UpMaps um;
  memset(&um, 0, sizeof(um));
  // output-channel tile: the smallest built N that covers Cout (196 -> 208: 13 x 16, no MMAs on 60 padding columns)
  if (w.cout <= 128) LB_CONV_CASE(128)
  if (w.cout <= 208) LB_CONV_CASE(208)
  if (w.cout <= 256) LB_CONV_CASE(256)
#undef LB_CONV_CASE
#undef LB_CONV_CASE_UP
  return fail("convolutions with more than 256 output channels are not built");
}

}  // namespace lb

using namespace lb;

// Steps 1-3 of a coarse (D = 32) encoder-layer call with full (softmax) attention: the message planes att[x rows] =
// softmax(Q K^T / sqrt(D)) V per group and head            [transformer.py:47-50, linear_attention.py:56-81]
// Projections carry no feature map and no row zeroing: masks act inside the attention (key weight 0, padded query 0).
// Q goes to the att planes [R, C] (overwritten in place by the message), K|V to the MLP hidden planes [R, 2C], which
// are dead at this point of the layer; full_attn_wgmma_kernel (full_attn.cuh) reads both through tensor maps.
template <int BN>
static int tf_full_attention_coarse(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st,
                                    const TfWs& w, long x_base, long x_rows, int x_group_rows, long s_base,
                                    long s_rows, int s_group_rows, int n_groups_x, bool self_pass, cudaStream_t stream) {
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
    using Epi = EpiPlanes<BN>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, 0};
    Planes B{wq_hi, wq_lo, C, 0};
    OutMaps om;
    LB_TRY(fill_out_maps(&om, w.att_hi + x_base * C, w.att_lo + x_base * C, C, nullptr, 0, C, x_rows, 1));
    typename Epi::Params ep{0, nullptr, 1, nullptr, 0, w.att_hi + x_base * C, w.att_lo + x_base * C, C, 0, lw.s_qkv, om};
    LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, 1, static_cast<int>(x_rows), C, C, 0, ep, stream)));
  }
  {
    using Epi = EpiPlanes<BN>;
    Planes A{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, 0};
    Planes B{wq_hi + wkv_off, wq_lo + wkv_off, C, 0};
    OutMaps om;
    LB_TRY(fill_out_maps(&om, w.h_hi + s_base * ldc, w.h_lo + s_base * ldc, ldc, nullptr, 0, 2 * C, s_rows, 1));
    typename Epi::Params ep{0, nullptr, 1, nullptr, 0, w.h_hi + s_base * ldc, w.h_lo + s_base * ldc,
                            static_cast<int>(ldc), 0, lw.s_qkv, om};
    LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, 1, static_cast<int>(s_rows), 2 * C, C, 0, ep, stream)));
  }
  const long qbs = static_cast<long>(x_group_rows) * C, kvbs = static_cast<long>(s_group_rows) * ldc;
  CUtensorMap tq_hi, tq_lo, tkv_hi, tkv_lo;
  LB_TRY(make_map(&tq_hi, w.att_hi + x_base * C, C, x_group_rows, n_groups_x, C, qbs, kFaRows, kFaD));
  LB_TRY(make_map(&tq_lo, w.att_lo + x_base * C, C, x_group_rows, n_groups_x, C, qbs, kFaRows, kFaD));
  LB_TRY(make_map(&tkv_hi, w.h_hi + s_base * ldc, 2 * C, s_group_rows, n_groups_s, ldc, kvbs, kFaKeys, kFaD));
  LB_TRY(make_map(&tkv_lo, w.h_lo + s_base * ldc, 2 * C, s_group_rows, n_groups_s, ldc, kvbs, kFaKeys, kFaD));
  static bool configured[kMaxDevices] = {false};
  int dev = 0;
  LB_CUDA(cudaGetDevice(&dev));
  if (!configured[dev]) {
    LB_CUDA(cudaFuncSetAttribute(full_attn_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwSmem));
    configured[dev] = true;
  }
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
  TimingRec rec{nullptr, nullptr, TAG_FULL_ATTN};
  LB_TRY(timing_begin(rec, stream));
  full_attn_wgmma_kernel<<<grid, kFwThreads, kFwSmem, stream>>>(tq_hi, tq_lo, tkv_hi, tkv_lo, wp);
  LB_LAUNCHED();
  LB_TRY(timing_end(rec, stream));
  return 0;
}

// Steps 1-3 of a coarse (D = 32) encoder-layer call with linear attention (SURVEY.md §2a G1/G2): the k|v projection
// writes K = elu(k)+1 and V as planes, kv_gemm_kernel reduces them to K^T V and Ksum on the tensor cores, and the q
// projection applies the attention in its epilogue; q, k, v never reach HBM.
//                                                   [transformer.py:47-50, linear_attention.py:31-46]
static int tf_linear_attention_coarse(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st,
                                      const TfWs& w, long x_base, int x_group_rows, long s_base, int s_group_rows,
                                      int n_groups_x, int n_groups_s, cudaStream_t stream) {
  if (!lw.wkv_hi || !lw.wkv_lo)
    return fail("linear attention of the coarse transformer needs the fused k|v weight planes (wkv_hi / wkv_lo)");
  const int D = C / H;
  const int per = D * D + D;
  const long ldc = 2L * C;
  const __half* cat_hi = static_cast<const __half*>(st.cat_hi);
  const __half* cat_lo = static_cast<const __half*>(st.cat_lo);
  const uint8_t* mask = st.mask;
  int sms = 0;
  LB_TRY(device_check(&sms));
  __half* kvp_hi = w.h_hi + s_base * ldc;   // the MLP hidden planes [R, 2C] are free at this point of the layer
  __half* kvp_lo = w.h_lo + s_base * ldc;
  {
    using Epi = EpiKvProj<256>;
    Planes A{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, static_cast<long>(s_group_rows) * ldc};
    Planes B{lw.wkv_hi, lw.wkv_lo, C, 0};
    typename Epi::Params ep;
    ep.rowmask = mask ? mask + s_base : nullptr;
    ep.acc_scale = lw.s_qkv;
    LB_TRY(fill_out_maps(&ep.om, kvp_hi, kvp_lo, ldc, nullptr, 0, 2 * C, s_group_rows, n_groups_s));
    LB_TRY((launch_gemm<256, Epi>(TAG_KV, A, B, n_groups_s, s_group_rows, 2 * C, C, 0, ep, stream)));
  }
  {
    CUtensorMap tm_hi, tm_lo;
    LB_TRY(make_map(&tm_hi, kvp_hi, 2 * C, s_group_rows, n_groups_s, ldc, static_cast<long>(s_group_rows) * ldc, 64, 64));
    LB_TRY(make_map(&tm_lo, kvp_lo, 2 * C, s_group_rows, n_groups_s, ldc, static_cast<long>(s_group_rows) * ldc, 64, 64));
    const int kb_total = cdiv(s_group_rows, 64);
    const int m_tiles_s = cdiv(s_group_rows, kBlockM);
    const int parts_cap = m_tiles_s > kKvSplits ? m_tiles_s : kKvSplits;   // capacity of kv_part (see kKvSplits)
    int splits = sms / (2 * n_groups_s);
    if (splits < 1) splits = 1;
    if (splits > kb_total) splits = kb_total;
    if (splits > parts_cap) splits = parts_cap;
    const int kb_per = cdiv(kb_total, splits);
    splits = cdiv(kb_total, kb_per);
    static bool configured[kMaxDevices] = {false};
    int dev = 0;
    LB_CUDA(cudaGetDevice(&dev));
    if (!configured[dev]) {
      LB_CUDA(cudaFuncSetAttribute(kv_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kKvGemmSmem));
      configured[dev] = true;
    }
    KvGemmParams kp{w.kv_part, kb_total, kb_per, splits};
    kv_gemm_kernel<<<dim3(splits, 2, n_groups_s), kKvGemmThreads, kKvGemmSmem, stream>>>(tm_hi, tm_lo, kp);
    LB_LAUNCHED();
    const long total = static_cast<long>(n_groups_s) * H * per;
    kv_tile_merge_kernel<<<cdiv(total, 256), 256, 0, stream>>>(w.kv_part, splits, H * per, w.kv, total);
    LB_LAUNCHED();
  }
  {
    using Epi = EpiAttn<256, 32>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, static_cast<long>(x_group_rows) * ldc};
    Planes B{lw.wqkv_hi, lw.wqkv_lo, C, 0};
    typename Epi::Params ep{mask ? mask + x_base : nullptr, lw.s_qkv, w.kv, 1e-6f, w.att_hi + x_base * C,
                            w.att_lo + x_base * C, C};
    LB_TRY((launch_gemm<256, Epi>(TAG_QATTN, A, B, n_groups_x, x_group_rows, C, C, 0, ep, stream)));
  }
  return 0;
}

// Runs one encoder-layer call `x <- layer(x, source)` for the row range x (queries) / s (source).
// self_pass: x range == source range (q, k, v in one projection launch).
template <int BN>
static int lb::tf_layer_pass(const LbEncoderLayerWeights& lw, int C, int H, const LbTransformerState& st,
                             const TfWs& w, long x_base, long x_rows, int x_group_rows, long s_base, long s_rows,
                             int s_group_rows, int n_groups_x, bool self_pass, bool write_f32, cudaStream_t stream,
                             const int* live, int live_cap, bool full) {
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
    LB_TRY(tf_linear_attention_coarse(lw, C, H, st, w, x_base, x_group_rows, s_base, s_group_rows, n_groups_x,
                                      n_groups_s, stream));
  } else if (D == 32) {
    LB_TRY(tf_full_attention_coarse<BN>(lw, C, H, st, w, x_base, x_rows, x_group_rows, s_base, s_rows, s_group_rows,
                                        n_groups_x, self_pass, stream));
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
    using Epi = EpiActStore<BN>;
    if (self_pass) {
      Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
      Planes B{lw.wqkv_hi, lw.wqkv_lo, C, 0};
      OutMaps om;
      LB_TRY(fill_out_maps(&om, nullptr, nullptr, 0, w.qkv + x_base * 3 * C, 3 * C, 3 * C, xM, xb));
      typename Epi::Params ep{w.qkv + x_base * 3 * C, 3 * C, elu_self, pmask ? pmask + x_base : nullptr, lw.s_qkv, 0, om};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, A, B, xb, xM, 3 * C, C, 0, ep, stream, live, x_group_rows)));
    } else {
      Planes Aq{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
      Planes Bq{lw.wqkv_hi, lw.wqkv_lo, C, 0};
      OutMaps omq, omk;
      LB_TRY(fill_out_maps(&omq, nullptr, nullptr, 0, w.qkv + x_base * 3 * C, 3 * C, C, xM, xb));
      LB_TRY(fill_out_maps(&omk, nullptr, nullptr, 0, w.qkv + s_base * 3 * C + C, 3 * C, 2 * C, sM, sb));
      typename Epi::Params eq{w.qkv + x_base * 3 * C, 3 * C, elu_q, pmask ? pmask + x_base : nullptr, lw.s_qkv, 0, omq};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, Aq, Bq, xb, xM, C, C, 0, eq, stream, live, x_group_rows)));
      Planes Ak{cat_hi + s_base * ldc, cat_lo + s_base * ldc, ldc, sbs};
      Planes Bk{static_cast<const __half*>(lw.wqkv_hi) + static_cast<long>(C) * C,
                static_cast<const __half*>(lw.wqkv_lo) + static_cast<long>(C) * C, C, 0};
      typename Epi::Params ek{w.qkv + s_base * 3 * C + C, 3 * C, elu_kv, pmask ? pmask + s_base : nullptr, lw.s_qkv, 0, omk};
      LB_TRY((launch_gemm<BN, Epi>(TAG_PROJ, Ak, Bk, sb, sM, 2 * C, C, 0, ek, stream, live, s_group_rows)));
    }
    int sms = 0;
    LB_TRY(device_check(&sms));
    if (full) {
      // full (softmax) attention of the windows, exact fp32                      [linear_attention.py:56-81]
      const int grid = n_groups_x < 4 * sms ? n_groups_x : 4 * sms;
      window_full_attn_kernel<16, 8, 32><<<grid, 256, 0, stream>>>(w.qkv, 3 * C, 0, C, 2 * C, x_base, s_base,
                                                                   x_group_rows, n_groups_x, mask, w.att_hi, w.att_lo,
                                                                   C, live, live_cap);
    } else if (x_group_rows == s_group_rows) {
      // linear attention, one kernel per pass: KV stays in shared memory      [linear_attention.py:43-46]
      const int grid = n_groups_x < 3 * sms ? n_groups_x : 3 * sms;   // 3 resident blocks per SM (60 KB, <= 85 registers)
      const int wa_smem = (H * (D * D + D) + 4 * x_group_rows * C) * static_cast<int>(sizeof(float));
      static bool wa_configured[kMaxDevices] = {false};
      int dev = 0;
      LB_CUDA(cudaGetDevice(&dev));
      if (!wa_configured[dev]) {
        LB_CUDA(cudaFuncSetAttribute(window_attn_kernel<16, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (8 * (16 * 16 + 16) + 4 * 32 * 128) * static_cast<int>(sizeof(float))));
        wa_configured[dev] = true;
      }
      window_attn_kernel<16, 8><<<grid, 256, wa_smem, stream>>>(w.qkv, 3 * C, 0, C, 2 * C, x_base, s_base, x_group_rows,
                                                                n_groups_x, 1e-6f, w.att_hi, w.att_lo, C, live, live_cap);
    } else {
      // linear attention between windows of different sizes (a cross pass of the standalone fine transformer): KV and
      // Ksum per source window through HBM, then one 32-row block per query window   [linear_attention.py:43-46]
      kv_window_kernel<16, 8><<<n_groups_s, 256, 0, stream>>>(w.qkv, 3 * C, C, 2 * C, s_base, s_group_rows, w.kv);
      LB_LAUNCHED();
      attn_apply_kernel<16, 8><<<dim3(n_groups_x, 1), 256, 0, stream>>>(w.qkv, 3 * C, 0, x_base, x_group_rows, 32,
                                                                        w.kv, 1e-6f, w.att_hi, w.att_lo, C);
    }
    LB_LAUNCHED();
  }
  // 4. merge + norm1 -> cat[:, C:2C]                            [transformer.py:51-52]
  {
    using Epi = EpiLayerNorm<BN>;
    Planes A{w.att_hi + x_base * C, w.att_lo + x_base * C, C, xbs_a};
    Planes B{lw.wm_hi, lw.wm_lo, C, 0};
    OutMaps om;
    LB_TRY(fill_out_maps(&om, static_cast<__half*>(st.cat_hi) + x_base * ldc + C, static_cast<__half*>(st.cat_lo) + x_base * ldc + C,
                         ldc, nullptr, 0, C, xM, xb));
    typename Epi::Params ep{lw.ln1_g, lw.ln1_b, 1e-5f, nullptr, 0, nullptr, nullptr, 0, nullptr, 0,
                            static_cast<__half*>(st.cat_hi) + x_base * ldc,
                            static_cast<__half*>(st.cat_lo) + x_base * ldc, static_cast<int>(ldc), C, lw.s_m, om};
    LB_TRY((launch_gemm<BN, Epi>(TAG_MERGE_LN, A, B, xb, xM, C, C, 0, ep, stream, live, x_group_rows)));
  }
  // 5. mlp[0] + ReLU on cat([x, message]) -> h planes           [transformer.py:55, mlp 22-26]
  {
    using Epi = EpiPlanes<BN>;
    Planes A{cat_hi + x_base * ldc, cat_lo + x_base * ldc, ldc, xbs};
    Planes B{lw.w1_hi, lw.w1_lo, 2 * C, 0};
    OutMaps om;
    LB_TRY(fill_out_maps(&om, w.h_hi + x_base * ldc, w.h_lo + x_base * ldc, ldc, nullptr, 0, 2 * C, xM, xb));
    typename Epi::Params ep{1, nullptr, 1, nullptr, 0, w.h_hi + x_base * ldc, w.h_lo + x_base * ldc,
                            static_cast<int>(ldc), 0, lw.s_1, om};
    LB_TRY((launch_gemm<BN, Epi>(TAG_MLP1, A, B, xb, xM, 2 * C, 2 * C, 0, ep, stream, live, x_group_rows)));
  }
  // 6. mlp[2] + norm2 + residual -> cat[:, 0:C] (and x_f32 after the last layer)   [transformer.py:55-58]
  // The residual stream lives in the fp16 planes (x = hi + lo, exact to 2^-22 relative): no fp32 master copy is read
  // or written between layers.
  {
    using Epi = EpiLayerNorm<BN>;
    Planes A{w.h_hi + x_base * ldc, w.h_lo + x_base * ldc, ldc, xbs};
    Planes B{lw.w2_hi, lw.w2_lo, 2 * C, 0};
    float* xf = write_f32 ? st.x_f32 + x_base * C : nullptr;
    OutMaps om;
    LB_TRY(fill_out_maps(&om, static_cast<__half*>(st.cat_hi) + x_base * ldc, static_cast<__half*>(st.cat_lo) + x_base * ldc, ldc, xf,
                         C, C, xM, xb));
    typename Epi::Params ep{lw.ln2_g, lw.ln2_b, 1e-5f, nullptr, 0, cat_hi + x_base * ldc, cat_lo + x_base * ldc,
                            static_cast<int>(ldc), xf, C,
                            static_cast<__half*>(st.cat_hi) + x_base * ldc,
                            static_cast<__half*>(st.cat_lo) + x_base * ldc, static_cast<int>(ldc), 0, lw.s_2, om};
    LB_TRY((launch_gemm<BN, Epi>(TAG_MLP2_LN, A, B, xb, xM, C, 2 * C, 0, ep, stream, live, x_group_rows)));
  }
  return 0;
}

extern "C" {

int lb_version(void) { return 103; }
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
  int sms;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(x));
  LB_TRY(device_check(&sms));
  const long total = rows * cols;
  const int grid = static_cast<int>(total / 256 + 1 < 4096 ? total / 256 + 1 : 4096);
  split_planes_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, rows, cols, ld_x, static_cast<__half*>(hi), static_cast<__half*>(lo), ld_pl, col0);
  LB_LAUNCHED();
  return 0;
}

int lb_gemm_split(const void* a_hi, const void* a_lo, long lda, long a_batch_stride, const void* b_hi,
                  const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo, long o_batch_stride,
                  int batches, int M, int N, int K, void* stream) {
  if (N % 32 != 0) return fail("lb_gemm_split: N must be a multiple of 32");
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(out));
  if (batches > 1 && o_batch_stride != static_cast<long>(M) * ldo)
    return fail("lb_gemm_split: output batches must be densely stacked (o_batch_stride == M*ldo)");
  Planes A{a_hi, a_lo, lda, batches > 1 ? a_batch_stride : 0};
  Planes B{b_hi, b_lo, ldb, b_batch_stride};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* pe = getenv("LOFTR_B200_PROBE_NULL_EPI");   // measurement probe of the main loop (tools/gemm_probe.py)
  const int skip = pe ? atoi(pe) : 0;
  OutMaps om;
  LB_TRY(fill_out_maps(&om, nullptr, nullptr, 0, out, ldo, N, M, batches));
  if (N % 256 == 0 || N > 128) {
    using Epi = EpiActStore<256>;
    Epi::Params ep{out, static_cast<int>(ldo), 0, nullptr, 1.f, skip, om};
    return launch_gemm<256, Epi>(TAG_GEMM_TEST, A, B, batches, M, N, K, 0, ep, st);
  }
  using Epi = EpiActStore<128>;
  Epi::Params ep{out, static_cast<int>(ldo), 0, nullptr, 1.f, skip, om};
  return launch_gemm<128, Epi>(TAG_GEMM_TEST, A, B, batches, M, N, K, 0, ep, st);
}

int lb_coarse_prep(const float* feat, int nhwc, const float* pe, int n_img, int C, int h, int w, int pe_h, int pe_w,
                   float* x_f32, void* cat_hi, void* cat_lo, void* stream) {
  int sms;
  if (n_img <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(x_f32));
  LB_TRY(device_check(&sms));
  if (h > pe_h || w > pe_w) return fail("feature map %dx%d exceeds the position-encoding table %dx%d", h, w, pe_h, pe_w);
  if (n_img <= 0) return 0;
  dim3 grid(cdiv(static_cast<long>(h) * w, 32), cdiv(C, 32), n_img);
  coarse_prep_kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      feat, nhwc, pe, C, h, w, pe_h, pe_w, x_f32, static_cast<__half*>(cat_hi), static_cast<__half*>(cat_lo));
  LB_LAUNCHED();
  return 0;
}

size_t lb_transformer_workspace_bytes(int d_model, int nhead, int n_groups, int group_rows0, int group_rows1) {
  Bump b{nullptr, 0};
  TfWs w;
  const long R = static_cast<long>(n_groups) * (group_rows0 + group_rows1);
  carve_tf(b, w, d_model, nhead, R, n_groups, d_model / nhead == 32, group_rows0 > group_rows1 ? group_rows0 : group_rows1);
  return b.off + 256;
}

int lb_transformer_forward(const LbEncoderLayerWeights* layers, const int* kinds, int n_layers, int d_model,
                           int nhead, const LbTransformerState* st, void* ws, size_t ws_bytes, void* stream) {
  int sms;
  if (st->n_groups <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(st->x_f32));
  LB_TRY(device_check(&sms));
  const int C = d_model, H = nhead;
  const bool coarse = (C == 256 && H == 8);
  const bool fine = (C == 128 && H == 8);
  if (!coarse && !fine) return fail("unsupported transformer shape d_model=%d nhead=%d (built: 256/8 and 128/8)", C, H);
  if (st->n_groups <= 0) return 0;
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
  const bool same_groups = st->group_rows0 == st->group_rows1;
  for (int l = 0; l < n_layers; ++l) {
    const LbEncoderLayerWeights& lw = layers[l];
    const bool last = l == n_layers - 1;   // the fp32 copy of the features is only written after the last layer
    const int kind = kinds[l];
    const bool full = kind == LB_LAYER_SELF_FULL || kind == LB_LAYER_CROSS_FULL;
    auto pass = [&](long xb, long xr, int xg, long sb, long sr, int sg, int ng, bool self_pass) -> int {
      return coarse ? tf_layer_pass<256>(lw, C, H, *st, w, xb, xr, xg, sb, sr, sg, ng, self_pass, last, s, nullptr, 0,
                                         full)
                    : tf_layer_pass<128>(lw, C, H, *st, w, xb, xr, xg, sb, sr, sg, ng, self_pass, last, s, live,
                                         st->n_groups, full);
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


size_t lb_backbone_workspace_bytes(const LbBackboneWeights* w, int N, int H, int W) {
  Bump b{nullptr, 0};
  BbWs ws;
  carve_bb(b, ws, N, H, W, w->l1[0].cout, w->l2[0].cout, w->l3[0].cout);
  return b.off + 256;
}

int lb_backbone_forward(const LbBackboneWeights* w, const float* images, int N, int H, int W, float* feat_c_nhwc,
                        float* feat_f_nhwc, void* ws, size_t ws_bytes, void* stream) {
  int sms;
  if (N <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(images));
  LB_TRY(device_check(&sms));
  if (H % 8 != 0 || W % 8 != 0) return fail("image size %dx%d must be divisible by 8", H, W);
  if (!ws) return fail("workspace pointer is null");
  const int d1 = w->l1[0].cout, d2 = w->l2[0].cout, d3 = w->l3[0].cout;
  if (w->stem_cout != 128 || d1 != w->stem_cout) return fail("backbone stem built for initial_dim = block_dims[0] = 128");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  BbWs B;
  carve_bb(b, B, N, H, W, d1, d2, d3);
  if (!b.ok) return fail("backbone workspace too small: need %zu bytes", lb_backbone_workspace_bytes(w, N, H, W));
  const int H2 = H / 2, W2 = W / 2, H4 = H / 4, W4 = W / 4, H8 = H / 8, W8 = W / 8;

  // stem: conv 7x7 s2 + BN + ReLU on the tensor cores, software im2col (stem_tc.cuh)  [resnet_fpn.py:101]
  {
    StemTcParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.img = images; sp.N = N; sp.H = H; sp.W = W;
    sp.wt = w->stem_wt; sp.scale = w->stem_scale; sp.shift = w->stem_shift;
    sp.tiles_w = cdiv(W2, kConvTileW); sp.tiles_h = cdiv(H2, kConvTileH);
    sp.om.dims = 4;
    LB_TRY(make_out_map_nhwc(&sp.om.hi, B.s0.hi, false, 128, W2, H2, N, B.s0.ld));
    LB_TRY(make_out_map_nhwc(&sp.om.lo, B.s0.lo, false, 128, W2, H2, N, B.s0.ld));
    sp.om.use = 1;
    static bool configured[kMaxDevices] = {false};
    int dev = 0;
    LB_CUDA(cudaGetDevice(&dev));
    if (!configured[dev]) {
      LB_CUDA(cudaFuncSetAttribute(conv_stem7x7_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStemSmemBytes));
      configured[dev] = true;
    }
    const long tiles = static_cast<long>(sp.tiles_w) * sp.tiles_h * N;
    const int grid = static_cast<int>(tiles < sms ? tiles : sms);
    conv_stem7x7_tc_kernel<<<grid, kStemThreads, kStemSmemBytes, st>>>(sp);
    LB_LAUNCHED();
  }
  auto conv = [&](const LbConvWeights& cw, const BbBuf& in, int hin, int win, int act, const BbBuf* res,
                  const BbBuf* up, int uph, int upw, const BbBuf* out, float* of32, int f32ld) -> int {
    ConvRun r{&cw, in, hin, win, act, res, up, uph, upw, out, of32, f32ld};
    return run_conv(r, N, st);
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

int lb_coarse_match(const LbCoarseMatchArgs* a, void* ws, size_t ws_bytes, void* stream) {
  int sms;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(a->count));
  LB_TRY(device_check(&sms));
  const int n = a->n_pairs, L = a->L, S = a->S, C = a->C;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0) {
    LB_CUDA(cudaMemsetAsync(a->count, 0, sizeof(int), st));
    return 0;
  }
  if (L != a->h0c * a->w0c || S != a->h1c * a->w1c) return fail("L/S do not match the coarse grid sizes");
  if (C % kBlockK != 0) return fail("C=%d must be a multiple of %d", C, kBlockK);
  if ((a->mask0 == nullptr) != (a->mask1 == nullptr)) return fail("mask0 and mask1 must be given together");
  if (!ws) return fail("workspace pointer is null");
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  CmWs w;
  carve_cm(b, w, n, L, S);
  if (!b.ok) return fail("coarse-match workspace too small: need %zu bytes", lb_coarse_match_workspace_bytes(n, L, S));

  constexpr int BN = 256;
  const long nl = static_cast<long>(n) * L, ns = static_cast<long>(n) * S;
  const int m_tiles = (L + kBlockM - 1) / kBlockM;
  const int n_tiles = (S + BN - 1) / BN;
  int chunks = pick_chunks(n * m_tiles, n_tiles, sms);
  if (chunks > kMaxChunks) chunks = kMaxChunks;
  // launch_gemm re-derives (tiles_per_chunk, n_chunks) from this request; mirror it to size the merges
  const int tpc = (n_tiles + chunks - 1) / chunks;
  const int n_chunks = (n_tiles + tpc - 1) / tpc;

  Planes A{a->f0_hi, a->f0_lo, a->ld, static_cast<long>(L) * a->ld};
  Planes B{a->f1_hi, a->f1_lo, a->ld, static_cast<long>(S) * a->ld};
  const bool masked = a->mask0 != nullptr;
  if (masked) {
    mask_extent_kernel<<<n, 128, 0, st>>>(a->mask0, a->h0c, a->w0c, w.ext0);
    LB_LAUNCHED();
    mask_extent_kernel<<<n, 128, 0, st>>>(a->mask1, a->h1c, a->w1c, w.ext1);
    LB_LAUNCHED();
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
      mask_term_kernel<<<cdiv(ns, TB), TB, 0, st>>>(nullptr, a->mask1, nullptr, ns, w.col_t);
      LB_LAUNCHED();
      mask_term_kernel<<<cdiv(nl, TB), TB, 0, st>>>(nullptr, a->mask0, nullptr, nl, w.row_t);
      LB_LAUNCHED();
      ct = w.col_t;
      rt = w.row_t;
    }
    using Epi = EpiScoreLse<BN, true, true>;
    Epi::Params ep{scale, ct, rt, w.row_part, w.col_part};
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, n, L, S, C, chunks, ep, st)));
    // row_t = -rowLSE, col_t = -colLSE (kNegBig on padded entries)              [coarse_matching.py:119]
    lse_merge_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_part, n_chunks, nl, 0.f, nullptr, nullptr, L, a->mask0, w.row_t);
    LB_LAUNCHED();
    lse_merge_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_part, m_tiles, ns, 0.f, nullptr, nullptr, S, a->mask1, w.col_t);
    LB_LAUNCHED();
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
    mask_term_kernel<<<cdiv(ns, TB), TB, 0, st>>>(nullptr, a->mask1, nullptr, ns, w.col_t);
    LB_LAUNCHED();
    fill_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_v, 0.f, ns);
    LB_LAUNCHED();
    fill_kernel<<<cdiv(n, TB), TB, 0, st>>>(w.bin_v, 0.f, n);
    LB_LAUNCHED();
    fill_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_u, 0.f, nl);   // u = 0 (only observable with skh_iters == 0)
    LB_LAUNCHED();
    fill_kernel<<<cdiv(n, TB), TB, 0, st>>>(w.bin_u, 0.f, n);
    LB_LAUNCHED();
    mask_term_kernel<<<cdiv(nl, TB), TB, 0, st>>>(nullptr, a->mask0, nullptr, nl, w.row_t);
    LB_LAUNCHED();
    for (int it = 0; it < a->skh_iters; ++it) {
      // u_i = log_mu_i - LSE_j(Z_ij + v_j), j over S real columns + the dustbin column   [superglue.py:146]
      {
        using Epi = EpiScoreLse<BN, true, false>;
        Epi::Params ep{scale, w.col_t, nullptr, w.row_part, w.col_part};
        LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, n, L, S, C, chunks, ep, st)));
        lse_merge_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_part, n_chunks, nl, norm, a->bin_score, w.bin_v, L,
                                                      a->mask0, w.row_u);
        LB_LAUNCHED();
      }
      // dustbin row: u_L = log_mu_L - LSE_j(bin + v_j, bin + bin_v)                         [superglue.py:146]
      bin_lse_kernel<<<n, 256, 0, st>>>(w.col_v, S, a->bin_score, w.bin_v, log_mu_bin, w.bin_u);
      LB_LAUNCHED();
      mask_term_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_u, a->mask0, nullptr, nl, w.row_t);
      LB_LAUNCHED();
      // v_j = log_nu_j - LSE_i(Z_ij + u_i), i over L real rows + the dustbin row            [superglue.py:147]
      {
        using Epi = EpiScoreLse<BN, false, true>;
        Epi::Params ep{scale, nullptr, w.row_t, w.row_part, w.col_part};
        LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_LSE, A, B, n, L, S, C, chunks, ep, st)));
        lse_merge_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_part, m_tiles, ns, norm, a->bin_score, w.bin_u, S,
                                                      a->mask1, w.col_v);
        LB_LAUNCHED();
      }
      bin_lse_kernel<<<n, 256, 0, st>>>(w.row_u, L, a->bin_score, w.bin_u, log_nu_bin, w.bin_v);
      LB_LAUNCHED();
      mask_term_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_v, a->mask1, nullptr, ns, w.col_t);
      LB_LAUNCHED();
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
    using Epi = EpiScoreArgmax<BN>;
    Epi::Params ep{scale, alpha, w.col_t, w.row_t, w.row_apart, w.col_apart};
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_ARGMAX, A, B, n, L, S, C, chunks, ep, st)));
    argmax_merge_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_apart, n_chunks, nl, w.row_key, w.row_arg);
    LB_LAUNCHED();
    argmax_merge_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_apart, m_tiles, ns, w.col_key, w.col_arg);
    LB_LAUNCHED();
    if (passes == 2 && pass == 0) {
      // prefilter: rows / columns whose best partner is the dustbin are zeroed  [coarse_matching.py:136-140]
      ot_dead_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_key, a->bin_score, w.bin_v, L, nl, w.row_dead);
      LB_LAUNCHED();
      ot_dead_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_key, a->bin_score, w.bin_u, S, ns, w.col_dead);
      LB_LAUNCHED();
      mask_term_kernel<<<cdiv(nl, TB), TB, 0, st>>>(w.row_u, a->mask0, w.row_dead, nl, w.row_t);
      LB_LAUNCHED();
      mask_term_kernel<<<cdiv(ns, TB), TB, 0, st>>>(w.col_v, a->mask1, w.col_dead, ns, w.col_t);
      LB_LAUNCHED();
      row_dead = w.row_dead;
      col_dead = w.col_dead;
    }
  }

  if (a->conf_matrix) {   // opt-in materialisation of data['conf_matrix']         [coarse_matching.py:145]
    using Epi = EpiConfStore<BN>;
    // row_t / col_t hold -LSE (dual-softmax) or the Sinkhorn potentials, with padded / prefiltered entries disabled
    Epi::Params ep{scale, alpha, conf_bias, w.row_t, w.col_t, a->conf_matrix};
    LB_TRY((launch_gemm<BN, Epi>(TAG_SCORE_ARGMAX, A, B, n, L, S, C, 0, ep, st)));
  }

  SelectParams sp;
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
  match_flag_kernel<<<cdiv(nl, TB), TB, 0, st>>>(sp);
  LB_LAUNCHED();

  CompactParams cp;
  cp.total = nl; cp.L = L; cp.S = S; cp.w0c = a->w0c; cp.w1c = a->w1c;
  cp.scale = a->img_scale; cp.scale0 = a->scale0; cp.scale1 = a->scale1;
  cp.flag = w.flag; cp.conf = w.conf; cp.row_arg = w.row_arg;
  cp.capacity = a->capacity;
  cp.b_ids = a->b_ids; cp.i_ids = a->i_ids; cp.j_ids = a->j_ids;
  cp.mconf = a->mconf; cp.mkpts0 = a->mkpts0_c; cp.mkpts1 = a->mkpts1_c; cp.count = a->count;
  const int cblocks = cdiv(nl, kCompactBlock);
  match_count_kernel<<<cblocks, kCompactBlock, 0, st>>>(w.flag, nl, w.blk_counts);
  LB_LAUNCHED();
  match_scatter_kernel<<<cblocks, kCompactBlock, 0, st>>>(cp, w.blk_counts);
  LB_LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------------------ fine level
size_t lb_fine_preprocess_workspace_bytes(long M, int W, int Cf) {
  Bump b{nullptr, 0};
  const size_t rows = static_cast<size_t>(2) * M * W * W;
  b.take<__half>(rows * Cf);
  b.take<__half>(rows * Cf);
  b.take<float>(static_cast<size_t>(2) * M * Cf);
  return b.off + 256;
}

int lb_fine_preprocess(const LbFinePreprocessArgs* a, void* ws, size_t ws_bytes, void* stream) {
  int sms;
  if (a->M <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(a->x_f32));
  LB_TRY(device_check(&sms));
  if (a->Cf != 128 || a->Cc > 256) return fail("fine preprocess built for Cf=128, Cc<=256 (got %d, %d)", a->Cf, a->Cc);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int WW = a->W * a->W;
  const long rows = 2 * a->M * WW;
  if (!ws) return fail("workspace pointer is null");
  Bump b{static_cast<uint8_t*>(ws), ws_bytes};
  __half* win_hi = b.take<__half>(static_cast<size_t>(rows) * a->Cf);
  __half* win_lo = b.take<__half>(static_cast<size_t>(rows) * a->Cf);
  float* gbias = b.take<float>(static_cast<size_t>(2) * a->M * a->Cf);
  if (!b.ok) return fail("fine-preprocess workspace too small");

  FineGatherParams g;
  g.feat0 = a->feat_f0; g.feat1 = a->feat_f1;
  g.sn0 = a->sn0; g.sc0 = a->sc0; g.sh0 = a->sh0; g.sw0 = a->sw0;
  g.sn1 = a->sn1; g.sc1 = a->sc1; g.sh1 = a->sh1; g.sw1 = a->sw1;
  g.Hf0 = a->Hf0; g.Wf0 = a->Wf0; g.Hf1 = a->Hf1; g.Wf1 = a->Wf1;
  g.w0c = a->w0c; g.w1c = a->w1c; g.stride = a->stride; g.W = a->W; g.Cf = a->Cf; g.M = a->M;
  g.b_ids = a->b_ids; g.i_ids = a->i_ids; g.j_ids = a->j_ids;
  g.out_hi = win_hi; g.out_lo = win_lo; g.ld = a->Cf;
  g.live = a->M_live;
  const bool vec8 = a->sc0 == 1 && a->sc1 == 1 && a->Cf % 8 == 0 && g.ld % 8 == 0 && a->sw0 % 4 == 0 && a->sw1 % 4 == 0 &&
                    a->sh0 % 4 == 0 && a->sh1 % 4 == 0 && a->sn0 % 4 == 0 && a->sn1 % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(a->feat_f0) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->feat_f1) & 15) == 0;
  if (vec8) fine_gather_vec8_kernel<<<static_cast<unsigned>(2 * a->M), 256, 0, st>>>(g);
  else fine_gather_kernel<<<static_cast<unsigned>(2 * a->M), 256, 0, st>>>(g);
  LB_LAUNCHED();

  FineBiasParams fb;
  fb.feat_c = a->feat_c;
  fb.set1_row_base = static_cast<long>(a->n_pairs) * a->L;
  fb.L = a->L; fb.S = a->S; fb.Cc = a->Cc; fb.Cf = a->Cf; fb.M = a->M;
  fb.b_ids = a->b_ids; fb.i_ids = a->i_ids; fb.j_ids = a->j_ids;
  fb.WdT = a->down_wt; fb.bd = a->down_b; fb.Wm2T = a->merge_w2t; fb.bm = a->merge_b;
  fb.gbias = gbias;
  fb.live = a->M_live;
  fine_bias_kernel<<<static_cast<unsigned>(cdiv(2 * a->M, kFineBiasWin)), 128, 0, st>>>(fb);
  LB_LAUNCHED();

  // merge_feat over [window | coarse] = window @ Wm[:, :Cf]^T + per-window bias     [fine_preprocess.py:52-56]
  // With a device bound each side is one GEMM batch of M*WW rows (M = capacity) with its own live prefix.
  using Epi = EpiPlanes<128>;
  const int nb = a->M_live ? 2 : 1;
  const long rows_b = rows / nb;
  Planes A{win_hi, win_lo, a->Cf, nb > 1 ? rows_b * a->Cf : 0};
  Planes B{a->merge_w_hi, a->merge_w_lo, a->Cf, 0};
  OutMaps om;
  LB_TRY(fill_out_maps(&om, a->cat_hi, a->cat_lo, 2 * a->Cf, a->x_f32, a->Cf, a->Cf, rows_b, nb));
  Epi::Params ep{0, gbias, WW, a->x_f32, a->Cf, static_cast<__half*>(a->cat_hi), static_cast<__half*>(a->cat_lo),
                 2 * a->Cf, 0, a->merge_acc_scale, om};
  return launch_gemm<128, Epi>(TAG_FINE_MERGE, A, B, nb, static_cast<int>(rows_b), a->Cf, a->Cf, 0, ep, st, a->M_live, WW);
}

int lb_fine_match(const LbFineMatchArgs* a, void* stream) {
  int sms;
  if (a->M <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(a->expec_f));
  LB_TRY(device_check(&sms));
  if (a->W * a->W > 32) return fail("fine window %dx%d exceeds one warp", a->W, a->W);
  FineMatchParams p;
  p.f0 = a->f0; p.f1 = a->f1; p.W = a->W; p.C = a->C; p.M = a->M;
  p.scale = a->img_scale; p.scale1 = a->scale1; p.b_ids = a->b_ids;
  p.mkpts1_c = a->mkpts1_c; p.expec_f = a->expec_f; p.mkpts1_f = a->mkpts1_f;
  p.live = a->M_live;
  const int warps_per_block = 8;
  fine_match_kernel<<<cdiv(a->M, warps_per_block), warps_per_block * 32, 0, static_cast<cudaStream_t>(stream)>>>(p);
  LB_LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------------------ evaluation
int lb_epipolar_errors(const float* mkpts0_f, const float* mkpts1_f, const long long* m_bids, long M, int n_pairs,
                       const float* T_0to1, const float* K0, const float* K1, float* epi_errs, void* stream) {
  if (M <= 0) return 0;
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(epi_errs));
  int sms;
  LB_TRY(device_check(&sms));
  if (!mkpts0_f || !mkpts1_f || !m_bids || !T_0to1 || !K0 || !K1) return fail("lb_epipolar_errors: null input");
  epipolar_error_kernel<<<cdiv(M, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(mkpts0_f, mkpts1_f, m_bids, M, n_pairs,
                                                                                      T_0to1, K0, K1, epi_errs);
  LB_LAUNCHED();
  return 0;
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
  int prev = -1;
  LB_CUDA(cudaGetDevice(&prev));
  LB_CUDA(cudaSetDevice(device));
  int sms;
  int rc0 = device_check(&sms);
  if (rc0) {
    cudaSetDevice(prev);
    return rc0;
  }
  NcclApi::UniqueId id;
  memcpy(id.internal, id_bytes, LB_NCCL_UNIQUE_ID_BYTES);
  void* nccl = nullptr;
  const int rc = api->CommInitRank(&nccl, world, id, rank);
  cudaSetDevice(prev);
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
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(wire));
  if (count > capacity) return fail("lb_pack_matches: %ld matches exceed the wire capacity %ld", count, capacity);
  if (count > 0 && (!mkpts0_f || !mkpts1_f || !mconf || !m_bids)) return fail("lb_pack_matches: null input");
  const long n = count > 0 ? count : 1;
  pack_matches_kernel<<<cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(mkpts0_f, mkpts1_f, mconf, m_bids, count,
                                                                                    pair_offset, wire, capacity);
  LB_LAUNCHED();
  return 0;
}

int lb_allgather_matches(void* comm, const float* wire_send, float* wire_recv, long capacity, void* stream) {
  if (!comm) return fail("lb_allgather_matches: null communicator");
  LbComm* c = static_cast<LbComm*>(comm);
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(wire_recv));
  NcclApi* api = nccl_api(nullptr);
  if (!api) return fail("NCCL library not loaded");
  const size_t count = static_cast<size_t>(1 + capacity) * kWireCols;
  const int rc = api->AllGather(wire_send, wire_recv, count, kNcclFloat32, c->nccl, static_cast<cudaStream_t>(stream));
  if (rc != 0) return fail("ncclAllGather failed: %s", api->GetErrorString ? api->GetErrorString(rc) : "?");
  return 0;
}

int lb_unpack_matches(const float* wire_recv, int world, long capacity, float* mkpts0_f, float* mkpts1_f, float* mconf,
                      long long* m_bids, long out_capacity, int* counts_out, void* stream) {
  DeviceGuard dev_guard;
  LB_TRY(dev_guard.bind(wire_recv));
  if (world <= 0 || capacity < 0) return fail("lb_unpack_matches: bad arguments");
  const long n = capacity > 0 ? capacity : 1;
  unpack_matches_kernel<<<dim3(cdiv(n, 256), world), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      wire_recv, world, capacity, mkpts0_f, mkpts1_f, mconf, m_bids, out_capacity, counts_out);
  LB_LAUNCHED();
  return 0;
}

}  // extern "C"
