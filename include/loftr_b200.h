/*
 * loftr_b200 -- C ABI of the H100-native LoFTR matching hot path.
 *
 * Every entry point replaces one `forward` of the reference (zju3dv/LoFTR, paths relative to the
 * reference root) and is what a binding from the reference side would call:
 *
 *   lb_preprocess_images      <- read_megadepth_gray / read_scannet_gray    src/utils/dataset.py:94-125,141-157,
 *                                (grey, resize, pad, / 255) + the 1/8 mask    src/datasets/megadepth.py:119-125
 *   lb_coarse_prep            <- PositionEncodingSine.forward + rearrange   src/loftr/utils/position_encoding.py:37-42,
 *                                                                           src/loftr/loftr.py:58-59
 *                                (lb_coarse_prep_indexed / lb_fine_preprocess_indexed: the same stages reading the
 *                                 backbone output of a per-image feature bank through a pair -> image index)
 *   lb_transformer_forward    <- LocalFeatureTransformer.forward            src/loftr/loftr_module/transformer.py:80-101
 *                                (LoFTREncoderLayer.forward :35-58, LinearAttention.forward linear_attention.py:20-47,
 *                                 FullAttention.forward :56-81 for the *_FULL layer kinds)
 *   lb_coarse_match           <- CoarseMatching.forward + get_coarse_match  src/loftr/utils/coarse_matching.py:87-148,150-261
 *                                (Sinkhorn branch: log_optimal_transport, third_party/SuperGluePretrainedNetwork/
 *                                 models/superglue.py:141-170)
 *   lb_fine_preprocess        <- FinePreprocess.forward                     src/loftr/loftr_module/fine_preprocess.py:29-59
 *   lb_fine_match             <- FineMatching.forward + get_fine_match      src/loftr/utils/fine_matching.py:15-74
 *
 * lb_estimate_geometry has no counterpart in the reference: it fits a homography or a fundamental matrix to each
 * pair's matches (batched RANSAC), the step callers otherwise run on the host after matching.
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
 * 102: full-attention layer kinds; 103: lb_selftest removed (no structure changes);
 * 104: lb_coarse_prep_indexed / lb_fine_preprocess_indexed (pairs read from a per-image feature bank);
 * 105: lb_coarse_match_capped (at most k matches per pair, chosen by confidence);
 * 106: lb_preprocess_images (uint8 images of any size -> the matcher's padded fp32 input and 1/8 mask);
 * 107: lb_estimate_geometry (batched RANSAC homography / fundamental matrix per pair);
 * 108: lb_backbone_workspace_bytes_fp16 / lb_backbone_forward_fp16 (single-pass fp16 backbone);
 * 109: lb_transformer_forward_fp16 / lb_coarse_match_fp16 (single-pass fp16 transformers and coarse matching);
 * 110: lb_gemm_fp16 (test hook of the contraction core on single fp16 planes).
 * Entries added without a version step (a caller finds them by name: a build that lacks one does not export it):
 * lb_coarse_query / lb_fine_preprocess_centres (matching caller-given image0 points);
 * lb_coarse_match_guided (coarse matching restricted to a band around a homography or fundamental matrix);
 * lb_rectify_images / lb_rectify_points (image1 warped into image0's frame through a homography, matches mapped back);
 * lb_coarse_match_search (coarse matching of K candidate warps per pair, keeping the best candidate's matches);
 * lb_coarse_query_guided / lb_fine_preprocess_centres_indexed (caller-given points on bank pairs, with a guide);
 * lb_coarse_query_side / lb_coarse_query_reuse (caller-given image1 points, and round trips on one coarse pass). */
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

/* Optional per-launch CUDA-event timing of the tensor-core kernels, the per-pair match cap, the image front end and
 * the geometry estimator (events recorded on the launching stream around each kernel while enabled).  lb_timing_enable(1) clears old records and starts recording,
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
/* The same product on the hi planes only, one fp16 MMA per k-step with fp32 accumulation (version 110): the kernels of
 * match_precision "fp16" (DESIGN.md §16).  Same arguments as lb_gemm_split; a_lo and b_lo are not read and may be NULL. */
int lb_gemm_fp16(const void* a_hi, const void* a_lo, long lda, long a_batch_stride, const void* b_hi,
                 const void* b_lo, long ldb, long b_batch_stride, float* out, long ldo, long o_batch_stride,
                 int batches, int M, int N, int K, void* stream);

/* ---- image front end.  Replaces, for a whole batch in one launch, the per-image host work of the reference's dataset
 * readers (src/utils/dataset.py: imread_gray's colour conversion :47-51, get_resized_wh / get_divisible_wh are the
 * caller's, cv2.resize + pad_bottom_right + `/ 255` of read_megadepth_gray :94-125 and read_scannet_gray :141-157) and
 * the 1/8 mask of src/datasets/megadepth.py:119-125.  One descriptor per image, in DEVICE memory. */
typedef struct LbImageDesc {
  const uint8_t* src;    /* device: pixel (y, x), channel c at src[y*row_stride_bytes + x*channels + c] */
  int h, w;              /* source size, both >= 1 */
  int row_stride_bytes;  /* >= w*channels: a cropped view or a row-padded decoder buffer needs no copy */
  int channels;          /* 1 (grey) or 3 (interleaved colour) */
  int r_index;           /* 3 channels: position of red, 0 = RGB, 2 = BGR (green is 1); ignored for 1 channel */
  int h_new, w_new;      /* size after the resize, 1 <= h_new <= H, 1 <= w_new <= W */
} LbImageDesc;

/* Image i is converted to grey at source resolution (OpenCV's Y = (9798 R + 19235 G + 3735 B + 16384) >> 15), resized
 * to h_new x w_new (bilinear, half-pixel centres, edge clamp, no antialiasing: cv2.resize INTER_LINEAR, except that
 * the fp32 result is not rounded to a grey level), divided by 255 and written top-left into out[i] ([n_images, 1, H, W]
 * fp32, 16-byte aligned); the rest of the canvas is 0.  With h_new == h and w_new == w, out is level / 255 exactly.
 * mask: NULL, or [n_images, H/8, W/8] bytes, cell (Y, X) = (8Y < h_new && 8X < w_new).  H and W must be positive
 * multiples of 8 and n_images at most 65535.  The descriptors are read on the device and not checked there: the caller
 * guarantees the ranges above.  One launch (timing tag "preprocess"), no workspace, no atomics. */
int lb_preprocess_images(const LbImageDesc* descs, int n_images, float* out, int H, int W, uint8_t* mask,
                         void* stream);

/* ---- rectified matching (found by name, see lb_version; DESIGN.md §19).  models: [n][9] f32, device, row-major
 * homography per pair, x1 ~ H x0 in source pixels: network pixel (x, y) of image k sits at (x * sx, y * sy) with
 * (sx, sy) = scale_k[b] ([n, 2] f32, device), or (1, 1) when scale_k is NULL.  Both entries apply H in fp64 as follows:
 * a model with a non-finite entry is replaced by the identity; otherwise H is multiplied by the sign of its w at the
 * centre ((W0 - 1) / 2 * sx0, (H0 - 1) / 2 * sy0) of image0's canvas (+1 when that w is 0).
 *
 * lb_rectify_images: out [n, 1, H, W] f32 (16-byte aligned; H, W positive multiples of 8 = image0's canvas), pixel
 * (x, y) of pair b = image1[b] ([n, 1, H1, W1] f32, contiguous) sampled at (H (x sx0, y sy0, 1))_xy / w / (sx1, sy1):
 * bilinear, pixel centres at integer coordinates, taps outside the image read as 0, i.e. grid_sample(mode="bilinear",
 * padding_mode="zeros", align_corners=True); 0 where w <= 0.  Coordinates in fp64, interpolation in fp32.  n at most
 * 65535.  One launch (timing tag "rectify"), no workspace. */
int lb_rectify_images(const float* image1, int n, int H1, int W1, const float* models, const float* scale0,
                      const float* scale1, float* out, int H, int W, void* stream);
/* lb_rectify_points: pts [m, 2] f32 (x, y) in source pixels of the rectified frame (image0's); pair_ids [m] int64.
 * out [m, 2] = (H p)_xy / w in fp64, rounded once to fp32: source pixels of image1; NaN where w <= 0, p is not finite
 * or the pair id is outside [0, n_pairs).  inside (NULL, or [m] bytes): 1 when out / (sx1, sy1) lies in
 * [0, W1 - 1] x [0, H1 - 1] and, with mask1 ([n_pairs, H1/8, w1c] bytes, w1c = W1/8), its cell (floor(v/8), floor(u/8))
 * is non-zero.  H0 x W0: image0's canvas (the sign rule above).  M_live: NULL, or a device int: only points
 * i < min(*M_live, m) are written.  One launch, no workspace. */
int lb_rectify_points(const float* pts, const long long* pair_ids, long m, const int* M_live, const float* models,
                      int n_pairs, const float* scale0, const float* scale1, int H0, int W0, int H1, int W1,
                      const uint8_t* mask1, int w1c, float* out, uint8_t* inside, void* stream);

/* ---- two-view geometry.  Robust fit of one model per pair to matches in a padded layout: pts0 / pts1 [B, K, 2] fp32
 * (x, y) pixels, 8-byte aligned; valid [B, K] bytes (non-zero: a match) or NULL (all K are matches).
 * model LB_GEOMETRY_HOMOGRAPHY: x1 ~ H x0, 4-point normalised DLT hypotheses, symmetric transfer error (the mean of
 * the squared forward and backward transfer distances); LB_GEOMETRY_FUNDAMENTAL: x1^T F x0 = 0, normalised 8-point
 * hypotheses with rank 2 enforced, squared Sampson distance.  A match is an inlier when its error is below
 * threshold^2 (threshold in pixels).
 * Per pair: `iterations` hypotheses, hypothesis h drawn from Philox4x32-10 with counter (h, pair id, block, 0) and key
 * seed (pair id: pair_ids[b], or b when pair_ids is NULL), so that a pair's result depends on its matches, its id, the
 * seed and the budget only; degenerate samples are skipped; the best hypothesis has the most inliers, then the lowest
 * MSAC cost (sum of min(error, threshold^2)), then the lowest index; the model is refitted by Hartley-normalised least
 * squares on its inliers and the inliers are recomputed once.  All geometry in fp64.
 * Outputs: model_out [B, 3, 3] fp32 (H scaled to H[2][2] = 1; F to unit Frobenius norm, largest entry positive), NaN
 * when the pair has fewer valid matches than the sample size or only degenerate samples; mask_out [B, K] bytes (1:
 * inlier of the returned model; padding and invalid entries 0); count_out [B] int32 (0 with a NaN model);
 * best_out [B] (or NULL): the best hypothesis, -1 when none; samples_out [B, iterations, 4 or 8] (or NULL): every
 * hypothesis' sample as columns of K, ascending, -1 when the pair is too small (a debugging output).
 * Three launches, no host synchronisation (capturable in a CUDA graph), timing tag "geometry". */
#define LB_GEOMETRY_HOMOGRAPHY 0
#define LB_GEOMETRY_FUNDAMENTAL 1
size_t lb_geometry_workspace_bytes(int B, int K, int iterations);
int lb_estimate_geometry(const float* pts0, const float* pts1, const uint8_t* valid, const int* pair_ids, int B, int K,
                         int model, float threshold, int iterations, unsigned long long seed, float* model_out,
                         uint8_t* mask_out, int* count_out, int* best_out, int* samples_out, void* ws, size_t ws_bytes,
                         void* stream);

/* feat fp32 (NCHW [n_img, C, h, w], or NHWC [n_img, h, w, C] when nhwc != 0) + pe [C, pe_h, pe_w]
 * -> x_f32 [n_img*h*w, C], cat planes [rows, 2C] cols [0,C). */
int lb_coarse_prep(const float* feat, int nhwc, const float* pe, int n_img, int C, int h, int w, int pe_h, int pe_w,
                   float* x_f32, void* cat_hi, void* cat_lo, void* stream);
/* lb_coarse_prep over a feature bank: `feat` holds the bank's images, output image b (of n_out) is bank image
 * img_idx[b] (device int [n_out], every entry in [0, images in the bank); not checked on the device).  The same image
 * may appear at several b. */
int lb_coarse_prep_indexed(const float* feat, int nhwc, const float* pe, const int* img_idx, int n_out, int C, int h,
                           int w, int pe_h, int pe_w, float* x_f32, void* cat_hi, void* cat_lo, void* stream);

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
/* The same network with single fp16 activations and one fp16 MMA per product (version 108; DESIGN.md §15).  The stem
 * keeps its split product; every later convolution multiplies the stored fp16 activation by the hi weight planes
 * (w_hi, wr_hi: fp16(w * 2^e) in the layout above) with fp32 accumulation, and the epilogue (x 2^-e, BatchNorm,
 * residual, FPN upsample-add, activation) stores one fp16 plane, rounded to nearest even.  w_lo / wr_lo are ignored
 * and may be NULL.  feat_c / feat_f are fp32 as above.  The workspace holds one plane per activation (about half of
 * lb_backbone_workspace_bytes).  Separate entry points rather than a flag: DESIGN.md §12. */
size_t lb_backbone_workspace_bytes_fp16(const LbBackboneWeights* w /*host*/, int N, int H, int W);
int lb_backbone_forward_fp16(const LbBackboneWeights* w /*host*/, const float* images, int N, int H, int W,
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
/* The same layers with one fp16 MMA per tensor-core product (version 109; DESIGN.md §16): every projection, merge and
 * MLP product, K^T V / Ksum of the coarse linear attention and S = Q K^T, P V of the coarse full attention multiply the
 * hi planes of their operands only (P rounded once to fp16), with fp32 accumulation.  Epilogues, LayerNorm, residuals
 * (read as hi + lo), masks, the stored hi / lo planes, the fp32 window-attention kernels and the workspace
 * (lb_transformer_workspace_bytes) are those of lb_transformer_forward.  The *_lo weight planes are not read and may
 * be NULL. */
int lb_transformer_forward_fp16(const LbEncoderLayerWeights* layers /*host*/, const int* kinds /*host*/, int n_layers,
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
/* lb_coarse_match keeping at most max_per_pair (>= 1) matches per pair: the ones with the largest mconf, a tie at the
 * max_per_pair-th value going to the smaller row index i.  Pairs with at most max_per_pair matches are unchanged; the
 * outputs stay in ascending (b, i) order, and a capacity of n_pairs*max_per_pair always suffices.  conf_matrix is not
 * affected.  One more launch than lb_coarse_match (timing tag "match_cap"); same workspace. */
int lb_coarse_match_capped(const LbCoarseMatchArgs* args /*host*/, int max_per_pair, void* ws, size_t ws_bytes,
                           void* stream);
/* Coarse matching with the score matrix computed as hi(f0) . hi(f1), one fp16 MMA per product (version 109;
 * DESIGN.md §16), in every pass (log-sum-exp, Sinkhorn iterations, arg-maxima, prefilter, conf_matrix), so all passes
 * see the same logits.  f0_lo / f1_lo are not read and may be NULL.  max_per_pair: 0 = no cap (as lb_coarse_match),
 * >= 1 as lb_coarse_match_capped; negative values are an error.  Same workspace. */
int lb_coarse_match_fp16(const LbCoarseMatchArgs* args /*host*/, int max_per_pair, void* ws, size_t ws_bytes,
                         void* stream);

/* Guided coarse matching (found by name, see lb_version; DESIGN.md §18).  A separate structure, not new fields of LbCoarseMatchArgs:
 * DESIGN.md §12. */
#define LB_GUIDE_HOMOGRAPHY 0
#define LB_GUIDE_FUNDAMENTAL 1
typedef struct LbCoarseGuide {
  int kind;            /* LB_GUIDE_* */
  const float* model;  /* [n_pairs][9] f32, device: row-major 3x3 T per pair, in the coordinates of mkpts0_c / mkpts1_c
                        * (source pixels when scale0 / scale1 are given); a pair whose T has a non-finite entry is
                        * unguided */
  float radius;        /* finite, > 0: pixels of image1's output coordinates */
} LbCoarseGuide;
/* lb_coarse_match / lb_coarse_match_capped (fp16 = 0) or lb_coarse_match_fp16 (fp16 = 1) with every score entry of an
 * inadmissible cell pair left out of the normalisers (the reference's -1e9 fill) and given conf 0 before the
 * threshold, border and mutual-nearest tests, in the dual-softmax and the Sinkhorn branch; conf_matrix is 0 there too.
 * Cell pair (i, j) of pair b is admissible when p0 = mkpts0_c(i), p1 = mkpts1_c(j) satisfy, in fp32:
 *   LB_GUIDE_FUNDAMENTAL  l = T (p0, 1):  |l . (p1, 1)| <= radius * sqrt(l0^2 + l1^2)  (l0 = l1 = 0: none)
 *   LB_GUIDE_HOMOGRAPHY   q = T (p0, 1):  q2 != 0 and |q01 / q2 - p1| <= radius
 * max_per_pair: 0 = no cap, >= 1 as lb_coarse_match_capped.  Errors: a NULL guide or model, an unknown kind, a radius
 * that is not finite and positive.  Same workspace as lb_coarse_match. */
int lb_coarse_match_guided(const LbCoarseMatchArgs* args /*host*/, const LbCoarseGuide* guide /*host*/,
                           int max_per_pair, int fp16, void* ws, size_t ws_bytes, void* stream);

/* Rectification search (found by name, see lb_version; DESIGN.md §20).  A separate structure, not new fields of
 * LbCoarseMatchArgs: DESIGN.md §12.  args->n_pairs = N * K candidates, candidate c = b * K + k of pair b. */
typedef struct LbCoarseSearch {
  int K;               /* >= 1 candidates per pair; args->n_pairs must be a multiple of K */
  int* counts;         /* [N, K] int32, device: the candidate's flagged rows (mutual, masks, border, > thr, Sinkhorn
                        * prefilter), before any per-pair cap */
  long long* choice;   /* [N] int64, device: the smallest k with the largest count (0 when every count is 0) */
} LbCoarseSearch;
/* lb_coarse_match / lb_coarse_match_capped (fp16 = 0) or lb_coarse_match_fp16 (fp16 = 1) over the N * K candidates,
 * with one more launch between the flag pass and the cap (timing tag "match_search", one CTA per pair): it writes
 * counts and choice and clears the flags of every candidate but (b, choice[b]).  The cap (max_per_pair: 0 = no cap,
 * >= 1 as lb_coarse_match_capped) and the compaction then see the winners' rows only: b_ids hold candidate ids c, and
 * a capacity of the N-pair bound (N * min(L, S), N * L with masks, N * min(max_per_pair, that) with a cap) always
 * suffices.  Errors: a NULL search, NULL counts or choice with n_pairs > 0, K < 1, n_pairs not a multiple of K.  Same
 * workspace as lb_coarse_match. */
int lb_coarse_match_search(const LbCoarseMatchArgs* args /*host*/, const LbCoarseSearch* search /*host*/,
                           int max_per_pair, int fp16, void* ws, size_t ws_bytes, void* stream);

/* Caller-given image0 points of every pair (found by name, see lb_version; LoFTR.match_points, DESIGN.md §17).  A separate structure, not
 * new fields of LbCoarseMatchArgs: DESIGN.md §12.  Outputs are per query, q = b*Q + k. */
typedef struct LbCoarseQueryArgs {
  int Q;                  /* queries per pair */
  const float* points0;   /* [n_pairs, Q, 2] (x, y) f32: image0 pixels, or source pixels when args->scale0 is given */
  const uint8_t* valid0;  /* optional [n_pairs, Q]: 0 = not a query */
  int H0, W0;             /* image0 size (hw0_i) */
  int Hf0, Wf0;           /* fine map of image0 (hw0_f) */
  int stride;             /* fine pixels per coarse cell (hw0_f / hw0_c) */
  float fine_scale;       /* image pixels per fine pixel (hw0_i / hw0_f) */
  long long* i_ids;       /* [n_pairs*Q] the query's cell in image0, -1 when it is not inside */
  long long* j_ids;       /* [n_pairs*Q] the row arg-max of that cell in image1, -1 when not inside */
  float* conf;            /* [n_pairs*Q] mconf's expression for (b, i, j); 0 when not inside */
  uint8_t* mutual;        /* [n_pairs*Q] i is the column arg-max of j */
  uint8_t* valid;         /* [n_pairs*Q] the forward would keep (b, i, j) before any per-pair cap */
  uint8_t* inside;        /* [n_pairs*Q] the query was answered */
  int* centres;           /* [2, n_pairs*Q, 2] fine-map (x, y) centres of the image0 / image1 windows */
  long long* win_ids;     /* [3, n_pairs*Q] (b, i, j) for lb_fine_preprocess_centres / lb_fine_match: i = j = 0 when
                           * the query is not inside, so every id is in range */
  float* pts0_f;          /* [n_pairs*Q, 2] fine-grid image0 point (source pixels); NaN when not inside */
  float* pts1_c;          /* [n_pairs*Q, 2] image1 window centre (source pixels): mkpts1_c of lb_fine_match */
} LbCoarseQueryArgs;

/* The coarse stage of lb_coarse_match (operand_planes 2) or lb_coarse_match_fp16 (1), answered for the points of
 * `query` instead of as a match list.  A query is inside when valid0 allows it, its point (divided by scale0) is finite
 * and in [0, W0 - 1] x [0, H0 - 1], its cell cx = clamp(floor(x / img_scale + 0.5)) (and y) is unmasked, and the row
 * of that cell has a valid column.  Fine centres: f0 = clamp(floor(p / fine_scale + 0.5)) on the fine map, f1 =
 * stride * (jx, jy) + f0 - stride * (cx, cy).  The match-list outputs of `args` (capacity, b_ids .. count) are not
 * read or written; conf_matrix is written when given.  Same workspace as lb_coarse_match; one more launch after its
 * flag pass (timing tag "match_query"), no per-pair cap and no compaction. */
int lb_coarse_query(const LbCoarseMatchArgs* args /*host*/, const LbCoarseQueryArgs* query /*host*/,
                    int operand_planes, void* ws, size_t ws_bytes, void* stream);
/* lb_coarse_query on the guided coarse quantities of lb_coarse_match_guided (found by name; DESIGN.md §21): every
 * score pass takes the guide's predicate, so j is the row arg-max over the admissible cells of the query's row, valid
 * is lb_coarse_match_guided's flag test and a row without an admissible, unmasked column has no answer (not inside).
 * Errors: those of lb_coarse_query, and a NULL guide or model, an unknown kind or a radius that is not finite and
 * positive, as lb_coarse_match_guided.  Same workspace as lb_coarse_match. */
int lb_coarse_query_guided(const LbCoarseMatchArgs* args /*host*/, const LbCoarseQueryArgs* query /*host*/,
                           const LbCoarseGuide* guide /*host*/, int operand_planes, void* ws, size_t ws_bytes,
                           void* stream);

/* Point queries from either image (found by name; DESIGN.md §22).  side 0: lb_coarse_query, or with a non-NULL guide
 * lb_coarse_query_guided.  side 1: the queries are image1 points, and `query` is read with the roles swapped: points0 /
 * valid0 hold the image1 points (source pixels when args->scale1 is given), H0 / W0 image1's size, Hf0 / Wf0 its fine
 * map; pts0_f receives the query snapped to image1's fine grid and pts1_c the image0 window centre.  A query is inside
 * when valid0 allows it, its point (divided by scale1) is finite and in [0, W0 - 1] x [0, H0 - 1], its cell j is
 * unmasked and the column of j has a valid row; i is that column's arg-max.  i_ids / j_ids, centres and win_ids keep
 * the (image0, image1) order.  f1 = clamp(floor(p / fine_scale + 0.5)), f0 = stride * (ix, iy) + f1 - stride * (jx, jy).
 * mutual: row_arg[i] == j and row i has a valid column; valid: mutual and the forward's flag of (b, i); conf: mconf's
 * expression when mutual, else exp((col_key[j] + colterm[j]) + bias).  Errors: those of lb_coarse_query_guided when a
 * guide is given, a side that is not 0 or 1, operand_planes not 1 or 2.  Same workspace as lb_coarse_match. */
int lb_coarse_query_side(const LbCoarseMatchArgs* args /*host*/, const LbCoarseQueryArgs* query /*host*/,
                         const LbCoarseGuide* guide /*host, NULL: unguided*/, int side, int operand_planes, void* ws,
                         size_t ws_bytes, void* stream);
/* The query launch of lb_coarse_query_side alone (one launch, timing tag "match_query"; no score pass): `ws` must hold
 * what a preceding query entry computed for the same args (guide and operand planes included) on the same stream.
 * Errors: a side that is not 0 or 1, the query checks of lb_coarse_query, L / S that do not match the coarse grids, an
 * unknown match_type, a NULL workspace or one smaller than lb_coarse_match_workspace_bytes.  Q <= 0 or n_pairs <= 0
 * launch nothing. */
int lb_coarse_query_reuse(const LbCoarseMatchArgs* args /*host*/, const LbCoarseQueryArgs* query /*host*/, int side,
                          void* ws, size_t ws_bytes, void* stream);

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
/* lb_fine_preprocess with feat_f0 / feat_f1 holding feature banks: the windows of pair b (b_ids) are read from image
 * img_idx0[b] of feat_f0 and image img_idx1[b] of feat_f1 (device ints [n_pairs], each in range of its bank; sn0 / sn1
 * step from one bank image to the next).  feat_c stays pair-major.  Same workspace as lb_fine_preprocess. */
int lb_fine_preprocess_indexed(const LbFinePreprocessArgs* args /*host*/, const int* img_idx0, const int* img_idx1,
                               void* ws, size_t ws_bytes, void* stream);
/* lb_fine_preprocess with the window centres read from `centres` ([2, M, 2] fine-map (x, y) of side 0 then side 1,
 * as lb_coarse_query writes them) instead of stride * (the cell of i_ids / j_ids) (found by name).  Windows m with
 * inside[m] == 0 are gathered as zeros; b_ids / i_ids / j_ids still select the image and the coarse-feature bias and
 * must be in range for every m.  M_live must be NULL.  Same workspace as lb_fine_preprocess. */
int lb_fine_preprocess_centres(const LbFinePreprocessArgs* args /*host*/, const int* centres, const uint8_t* inside,
                               void* ws, size_t ws_bytes, void* stream);
/* lb_fine_preprocess_centres with feat_f0 / feat_f1 holding feature banks, read as lb_fine_preprocess_indexed reads
 * them: pair b's windows come from image img_idx0[b] of feat_f0 and img_idx1[b] of feat_f1, centred on the table's
 * fine pixels (found by name; DESIGN.md §21).  Errors: NULL centres, inside, img_idx0 or img_idx1 with M > 0, and a
 * non-NULL M_live.  Same workspace as lb_fine_preprocess. */
int lb_fine_preprocess_centres_indexed(const LbFinePreprocessArgs* args /*host*/, const int* centres,
                                       const uint8_t* inside, const int* img_idx0, const int* img_idx1, void* ws,
                                       size_t ws_bytes, void* stream);

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
