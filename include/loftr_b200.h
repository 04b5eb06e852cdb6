/*
 * loftr_b200 -- C ABI of the H100-native LoFTR matching hot path.
 *
 * Every entry point replaces one `forward` of the reference (zju3dv/LoFTR, paths relative to the
 * reference root) and is what a binding from the reference side would call:
 *
 *   lb_coarse_prep            <- PositionEncodingSine.forward + rearrange   src/loftr/utils/position_encoding.py:37-42,
 *                                                                           src/loftr/loftr.py:58-59
 *   lb_transformer_forward    <- LocalFeatureTransformer.forward            src/loftr/loftr_module/transformer.py:80-101
 *                                (LoFTREncoderLayer.forward :35-58, LinearAttention.forward linear_attention.py:20-47,
 *                                 FullAttention.forward :56-81 for the *_FULL layer kinds)
 *   lb_coarse_match           <- CoarseMatching.forward + get_coarse_match  src/loftr/utils/coarse_matching.py:87-148,150-261
 *                                (Sinkhorn branch: log_optimal_transport, third_party/SuperGluePretrainedNetwork/
 *                                 models/superglue.py:141-170)
 *   lb_fine_preprocess        <- FinePreprocess.forward                     src/loftr/loftr_module/fine_preprocess.py:29-59
 *   lb_fine_match             <- FineMatching.forward + get_fine_match      src/loftr/utils/fine_matching.py:15-74
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless a parameter says "host".  No torch / C++ types cross this
 *     boundary; `stream` is a cudaStream_t passed as void*.
 *   - Functions enqueue work on `stream` and return without synchronising.  Return value 0 = success,
 *     non-zero = error (lb_last_error() gives the message for the calling thread).
 *   - Workspaces are caller-provided; query the size with the matching *_workspace_bytes function.
 *   - "planes": an fp32 matrix x kept as two fp16 matrices hi, lo with x ~= hi + lo (see DESIGN.md).
 *     A "cat buffer" is a [rows, 2C] pair of planes; columns [0, C) hold the token features.
 *   - There is no CPU fallback: on a machine without an sm_90 (H100) device every compute entry point fails.
 */
#ifndef LOFTR_B200_H_
#define LOFTR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB_MATCH_DUAL_SOFTMAX 0
#define LB_MATCH_SINKHORN 1
#define LB_LAYER_SELF 0
#define LB_LAYER_CROSS 1
/* full (softmax) attention layers (reference FullAttention, linear_attention.py:50-81): the same weights and token
 * state as the linear kinds.  Libraries before version 102 reject these kinds ("unknown layer kind"). */
#define LB_LAYER_SELF_FULL 2
#define LB_LAYER_CROSS_FULL 3

/* 101: device-count fields appended to LbTransformerState / LbFinePreprocessArgs / LbFineMatchArgs;
 * 102: full-attention layer kinds; 103: lb_selftest removed (no structure changes). */
int lb_version(void);
/* k-block (in elements) the library was built with: convolution weight planes pad Cin per tap to a multiple of it */
int lb_block_k(void);
/* K layout of a convolution with `cin` input channels: `cin_blocks` 64-channel blocks per tap in the main weight
 * planes, plus `rem_channels` (0, or 1..16 when cin = 64*cin_blocks + rem, e.g. 196 = 3*64 + 4) channels per tap that
 * go into the remainder planes of LbConvWeights. */
int lb_conv_layout(int cin, int* cin_blocks /*host*/, int* rem_channels /*host*/);
const char* lb_last_error(void);
/* number of kernels this library has launched in this process (for bench.py's gpu_launches) */
long long lb_launch_count(void);

/* Optional per-launch CUDA-event timing of the tensor-core kernels (events recorded on the launching
 * stream around each kernel while enabled).  lb_timing_enable(1) clears old records and starts recording,
 * lb_timing_collect synchronises the recorded events and returns per-tag total milliseconds and launch counts
 * (arrays of lb_timing_num_tags() entries; names via lb_timing_tag_name).  Timed launches cannot be recorded into a
 * CUDA graph: while timing is enabled, a launch on a capturing stream fails. */
int lb_timing_enable(int on);
int lb_timing_num_tags(void);
const char* lb_timing_tag_name(int tag);
int lb_timing_collect(double* total_ms /*host*/, long long* counts /*host*/, int n);

/* fp32 [rows, cols] (row stride ld_x) -> fp16 planes written at column offset col0 of [rows, ld_pl] buffers. */
int lb_split_planes(const float* x, long rows, int cols, int ld_x, void* hi, void* lo, int ld_pl, int col0,
                    void* stream);

/* Test hook for the contraction core: out[b, m, n] = sum_k A[b, m, k] * B[b?, n, k] (fp32 out).
 * b_batch_stride == 0 shares B across batches. */
int lb_gemm_split(const void* a_hi, const void* a_lo, long lda, long a_batch_stride, const void* b_hi,
                  const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo, long o_batch_stride,
                  int batches, int M, int N, int K, void* stream);

/* feat fp32 (NCHW [n_img, C, h, w], or NHWC [n_img, h, w, C] when nhwc != 0) + pe [C, pe_h, pe_w]
 * -> x_f32 [n_img*h*w, C], cat planes [rows, 2C] cols [0,C). */
int lb_coarse_prep(const float* feat, int nhwc, const float* pe, int n_img, int C, int h, int w, int pe_h, int pe_w,
                   float* x_f32, void* cat_hi, void* cat_lo, void* stream);

/* ResNetFPN_8_2 local-feature CNN on tensor cores (reference src/loftr/backbone/resnet_fpn.py:43-118; SURVEY.md
 * §8(f) rank 1).  One LbConvWeights per Conv2d(+BatchNorm2d in eval mode, folded to scale/shift; scale = 1,
 * shift = 0 for a bare convolution).  Weight planes (fp16 hi/lo, tap-major), with (cin_blocks, rem) =
 * lb_conv_layout(cin): main [cout, k*k * cin_blocks*64] = for every tap the first cin_blocks*64 channels (zero padded
 * when rem == 0 and cin is not a multiple of 64); remainder [cout, k*k * 16] = for every tap channels
 * cin_blocks*64 .. cin-1 zero-padded to 16 (NULL when rem == 0). */
typedef struct LbConvWeights {
  const void* w_hi;
  const void* w_lo;
  const void* wr_hi;   /* remainder planes or NULL */
  const void* wr_lo;
  const float* scale;  /* [cout] */
  const float* shift;  /* [cout] */
  int cin, cout, ksize, stride;
} LbConvWeights;

typedef struct LbBackboneWeights {
  const float* stem_wt;    /* conv1.weight [cout,1,7,7] stored transposed as [49, cout] fp32 */
  const float* stem_scale; /* bn1 folded */
  const float* stem_shift;
  int stem_cout;
  LbConvWeights l1[4];     /* layer1.{0,1}.{conv1,conv2} (+bn1/bn2) */
  LbConvWeights l2[4];     /* layer2.{0,1}.{conv1,conv2}; l2[0] has stride 2 */
  LbConvWeights l2_down;   /* layer2.0.downsample.{0,1} */
  LbConvWeights l3[4];
  LbConvWeights l3_down;
  LbConvWeights l3_out;    /* layer3_outconv */
  LbConvWeights l2_out;    /* layer2_outconv */
  LbConvWeights l2_out2[2];/* layer2_outconv2.{0(+1 BN, LeakyReLU), 3} */
  LbConvWeights l1_out;    /* layer1_outconv */
  LbConvWeights l1_out2[2];/* layer1_outconv2.{0(+1), 3} */
} LbBackboneWeights;

size_t lb_backbone_workspace_bytes(const LbBackboneWeights* w /*host*/, int N, int H, int W);
/* images [N,1,H,W] fp32 -> feat_c NHWC fp32 [N,H/8,W/8,block_dims[2]], feat_f NHWC fp32 [N,H/2,W/2,block_dims[0]] */
int lb_backbone_forward(const LbBackboneWeights* w /*host*/, const float* images, int N, int H, int W,
                        float* feat_c_nhwc, float* feat_f_nhwc, void* ws, size_t ws_bytes, void* stream);

/* Weights of one LoFTREncoderLayer (state_dict names in comments), as fp16 planes of the [out, in] matrices.
 * Each weight matrix may be pre-scaled by a power of two 2^e before it is split (keeps the fp16 `lo` plane out of
 * the subnormal range, see DESIGN.md §2); s_* = 2^-e is applied to the fp32 accumulator (exact). */
typedef struct LbEncoderLayerWeights {
  const void* wqkv_hi; /* [3C, C]: rows = q_proj.weight, k_proj.weight, v_proj.weight */
  const void* wqkv_lo;
  const void* wkv_hi;  /* optional (coarse, D = 32) [2C, C]: the k and v rows of wqkv regrouped in blocks of 4 heads, */
  const void* wkv_lo;  /* [k heads 0-3; v heads 0-3; k heads 4-7; v heads 4-7]: B operand of the fused k|v projection */
  const void* wm_hi;   /* [C, C]   merge.weight */
  const void* wm_lo;
  const void* w1_hi;   /* [2C, 2C] mlp.0.weight */
  const void* w1_lo;
  const void* w2_hi;   /* [C, 2C]  mlp.2.weight */
  const void* w2_lo;
  const float* ln1_g;  /* norm1.weight / bias, norm2.weight / bias  [C] */
  const float* ln1_b;
  const float* ln2_g;
  const float* ln2_b;
  float s_qkv, s_m, s_1, s_2;
} LbEncoderLayerWeights;

/* Token state of a LocalFeatureTransformer run over two token sets (feat0 rows first, then feat1 rows). */
typedef struct LbTransformerState {
  float* x_f32;         /* [rows0 + rows1, C]   in/out */
  void* cat_hi;         /* [rows0 + rows1, 2C]  in/out (cols [0,C) = features, cols [C,2C) scratch) */
  void* cat_lo;
  const uint8_t* mask;  /* optional [rows0 + rows1], 1 = valid (mask0 then mask1 flattened) */
  int n_groups;         /* images (coarse) or windows (fine) per set */
  int group_rows0;      /* L  (or 25) */
  int group_rows1;      /* S  (or 25) */
  /* optional device int (fine / window transformer only): live windows per set.  NULL = all n_groups.  When set,
   * n_groups is the capacity that fixes the buffer layout and the grids; only windows [0, min(*n_groups_live,
   * n_groups)) of each set are computed, read on the device (no host synchronisation). */
  const int* n_groups_live;
} LbTransformerState;

size_t lb_transformer_workspace_bytes(int d_model, int nhead, int n_groups, int group_rows0, int group_rows1);
int lb_transformer_forward(const LbEncoderLayerWeights* layers /*host*/, const int* kinds /*host*/, int n_layers,
                           int d_model, int nhead, const LbTransformerState* st /*host*/, void* ws,
                           size_t ws_bytes, void* stream);

typedef struct LbCoarseMatchArgs {
  const void* f0_hi;   /* planes of feat_c0 [n_pairs*L, >=C] */
  const void* f0_lo;
  const void* f1_hi;   /* planes of feat_c1 [n_pairs*S, >=C] */
  const void* f1_lo;
  int ld;              /* row stride (elements) of the planes */
  int n_pairs, L, S, C;
  int h0c, w0c, h1c, w1c;
  int match_type;      /* LB_MATCH_* */
  float temperature;   /* dsmax_temperature */
  float thr;
  int border_rm;
  const float* bin_score; /* device scalar (sinkhorn) */
  int skh_iters;
  int skh_prefilter;
  const uint8_t* mask0;   /* optional [n_pairs*L] */
  const uint8_t* mask1;   /* optional [n_pairs*S] */
  float img_scale;        /* hw0_i[0] / hw0_c[0] */
  const float* scale0;    /* optional [n_pairs, 2] */
  const float* scale1;
  long capacity;          /* entries available in the outputs below (n_pairs*L always suffices) */
  long long* b_ids;
  long long* i_ids;
  long long* j_ids;
  float* mconf;
  float* mkpts0_c;        /* [capacity, 2] */
  float* mkpts1_c;
  int* count;             /* device int: number of matches M */
  float* conf_matrix;     /* optional [n_pairs, L, S] fp32: the reference's data['conf_matrix'] (opt-in) */
} LbCoarseMatchArgs;

size_t lb_coarse_match_workspace_bytes(int n_pairs, int L, int S);
int lb_coarse_match(const LbCoarseMatchArgs* args /*host*/, void* ws, size_t ws_bytes, void* stream);

typedef struct LbFinePreprocessArgs {
  const float* feat_f0;   /* fine maps, any strides (elements): index = n*sn + c*sc + y*sh + x*sw */
  const float* feat_f1;
  long sn0, sc0, sh0, sw0;
  long sn1, sc1, sh1, sw1;
  int Hf0, Wf0, Hf1, Wf1;
  int w0c, w1c;
  int stride;             /* hw0_f[0] // hw0_c[0] */
  int W;                  /* fine_window_size */
  int Cf, Cc;             /* fine / coarse d_model */
  const float* feat_c;    /* coarse transformer output x_f32: n_pairs*L rows then n_pairs*S rows, [.., Cc] */
  int n_pairs, L, S;
  long M;                 /* number of coarse matches */
  const long long* b_ids;
  const long long* i_ids;
  const long long* j_ids;
  const float* down_wt;   /* fine_preprocess.down_proj.weight TRANSPOSED [Cc, Cf], bias [Cf] */
  const float* down_b;
  const float* merge_w2t; /* fine_preprocess.merge_feat.weight[:, Cf:2Cf] TRANSPOSED [Cf, Cf] (fp32) */
  const float* merge_b;   /* fine_preprocess.merge_feat.bias [Cf] */
  const void* merge_w_hi; /* planes of merge_w[:, 0:Cf] * 2^e  -> [Cf, Cf] */
  const void* merge_w_lo;
  float merge_acc_scale;  /* 2^-e */
  /* outputs: fine transformer state, rows = side*M*W*W + m*W*W + k */
  float* x_f32;           /* [2*M*W*W, Cf] */
  void* cat_hi;           /* [2*M*W*W, 2Cf] */
  void* cat_lo;
  /* optional device int: live match count.  NULL = M.  When set, M is the capacity (layout and grids as above) and
   * only windows m < min(*M_live, M) of each side are gathered and merged. */
  const int* M_live;
} LbFinePreprocessArgs;

size_t lb_fine_preprocess_workspace_bytes(long M, int W, int Cf);
int lb_fine_preprocess(const LbFinePreprocessArgs* args /*host*/, void* ws, size_t ws_bytes, void* stream);

typedef struct LbFineMatchArgs {
  const float* f0;        /* [M*W*W, C] fine transformer output, window side 0 */
  const float* f1;        /* side 1 */
  int W, C;
  long M;
  float img_scale;        /* hw0_i[0] / hw0_f[0] */
  const float* scale1;    /* optional [n_pairs, 2] */
  const long long* b_ids;
  const float* mkpts1_c;  /* [M, 2] */
  float* expec_f;         /* [M, 3] */
  float* mkpts1_f;        /* [M, 2] */
  const int* M_live;      /* optional device int: live match count (NULL = M; when set, M is the capacity) */
} LbFineMatchArgs;

int lb_fine_match(const LbFineMatchArgs* args /*host*/, void* stream);

/* ---- evaluation harness (SURVEY.md §8(f) rank 3).  Squared symmetric epipolar distance of every match against the
 * ground-truth relative pose of its pair: replaces compute_symmetrical_epipolar_errors / symmetric_epipolar_distance
 * (src/utils/metrics.py:30-72).  T_0to1 [n_pairs,4,4], K0 / K1 [n_pairs,3,3] fp32 row-major, m_bids[m] = pair of
 * match m; epi_errs [M] out. */
int lb_epipolar_errors(const float* mkpts0_f, const float* mkpts1_f, const long long* m_bids, long M, int n_pairs,
                       const float* T_0to1, const float* K0, const float* K1, float* epi_errs, void* stream);

/* ---- multi-GPU: all-gather of the match lists.  Pairs are sharded over ranks (one process per GPU); every rank ends
 * with the global list.  Replaces the reference's gather() (src/utils/comm.py:113-176, called from
 * src/lightning/lightning_loftr.py:235,241: a size exchange plus a padded pickled-object all_gather on a gloo side
 * group) with ONE static-shape ncclAllGather on the compute stream between a pack and an unpack kernel.
 * Wire buffer per rank: float32 [1 + capacity][6]; row 0 = (count, 0...), row 1+k = (x0, y0, x1, y1, mconf, global
 * pair id).  NCCL is bound at run time (dlopen of libnccl.so.2; `nccl_lib_path` / LOFTR_B200_NCCL_LIB override it). */
#define LB_NCCL_UNIQUE_ID_BYTES 128
/* rank 0: create the rendezvous id (host buffer of LB_NCCL_UNIQUE_ID_BYTES), ship it to the other ranks out of band */
int lb_comm_unique_id(char* id_out /*host*/, const char* nccl_lib_path /*host, optional*/);
int lb_comm_init(const char* id_bytes /*host*/, int rank, int world, int device, const char* nccl_lib_path /*host, optional*/,
                 void** comm_out /*host*/);
int lb_comm_destroy(void* comm);
/* this rank's matcher outputs (`count` rows; pair ids are offset by `pair_offset`) -> wire buffer */
int lb_pack_matches(const float* mkpts0_f, const float* mkpts1_f, const float* mconf, const long long* m_bids,
                    long count, int pair_offset, float* wire, long capacity, void* stream);
/* wire_send [1 + capacity][6] of every rank -> wire_recv [world][1 + capacity][6] on every rank */
int lb_allgather_matches(void* comm, const float* wire_send, float* wire_recv, long capacity, void* stream);
/* wire_recv -> concatenated lists in rank order (= ascending (pair, i) for contiguous pair blocks); counts_out
 * [world + 1] device ints: the per-rank counts as sent (a count > capacity signals overflow) and the stored total */
int lb_unpack_matches(const float* wire_recv, int world, long capacity, float* mkpts0_f, float* mkpts1_f, float* mconf,
                      long long* m_bids, long out_capacity, int* counts_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LOFTR_B200_H_ */
