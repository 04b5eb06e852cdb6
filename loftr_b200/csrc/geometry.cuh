// Robust two-view geometry for matched pairs: batched RANSAC (MSAC scoring) of a homography or a fundamental matrix
// per pair, followed by one least-squares refit on the best hypothesis' inliers.  Three launches per call, no host
// synchronisation, no atomics:
//   geometry_compact_kernel  one block per pair: the valid matches of the padded [B, K] layout, in order, as float4
//                            (x0, y0, x1, y1) plus their column in K;
//   geometry_score_kernel    one thread per hypothesis, kGeoHypPerBlock hypotheses per block: draw a minimal sample
//                            (Philox keyed on (seed, pair id, hypothesis)), solve it in fp64, score it against every
//                            valid match of its pair staged through shared memory, reduce to the block's best;
//   geometry_refit_kernel    one block per pair: best over the tiles, inlier statistics, Hartley-normalised least
//                            squares on all inliers (smallest eigenvector by cyclic Jacobi), final inlier mask.
// Everything geometric runs in fp64 (the H100 has full-rate fp64 next to fp32): the results then agree with a float64
// NumPy implementation of the same algorithm to rounding, hypothesis for hypothesis.
//
// The hypothesis budget is fixed per call.  Adaptive early stopping (fewer iterations once an inlier ratio is
// established) is deliberately not implemented: its data-dependent trip count would make each pair's work depend on
// its own data and break the single static batched launch that makes the estimator capturable in a CUDA graph.
#pragma once
#include <cstdint>
#include <cmath>
#include "../../include/loftr_b200.h"

namespace lb {

constexpr int kGeoHypPerBlock = 64;    // hypotheses (threads) per scoring block
constexpr int kGeoStage = 1024;        // matches staged in shared memory per round of the scoring loop (16 KB)
constexpr int kGeoRefitThreads = 256;
constexpr int kGeoMaxSample = 8;
constexpr double kGeoCollinearEps = 1e-5;  // |cross| of three normalised sample points below which H is degenerate
constexpr double kGeoPivotEps = 1e-10;     // smallest usable pivot of the normalised 8x8 DLT system
constexpr double kGeoRankEps = 1e-12;      // F: second-smallest / largest eigenvalue of A^T A below which the sample
                                           // does not determine F (collinear points, planar sample)
constexpr int kGeoJacobiSweeps = 30;

struct GeoBest {        // a scored hypothesis; count -1: degenerate or absent
  double sum;           // MSAC cost: sum over valid matches of min(err, thr^2)
  int count;            // inliers: err < thr^2
  int hyp;
};

__host__ __device__ __forceinline__ bool geo_better(const GeoBest& a, const GeoBest& b) {
  if (a.count != b.count) return a.count > b.count;
  if (a.sum != b.sum) return a.sum < b.sum;
  return a.hyp < b.hyp;
}

// ---------------------------------------------------------------------------------------------- Philox4x32-10
__device__ __forceinline__ void philox4x32_10(uint32_t ctr[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t c0 = hi1 ^ ctr[1] ^ k0, c1 = lo1, c2 = hi0 ^ ctr[3] ^ k1, c3 = lo0;
    ctr[0] = c0; ctr[1] = c1; ctr[2] = c2; ctr[3] = c3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

// s distinct indices in [0, n), ascending, for hypothesis `hyp` of pair `pair_id`.  Draw j is word j % 4 of the Philox
// block with counter (hyp, pair_id, j / 4, 0) and key (seed low, seed high): r = (word * (n - j)) >> 32 picks the r-th
// index not drawn yet.  Exactly s draws, no rejection loop, and sorted samples (a set drawn twice gives one model).
__device__ __forceinline__ void geo_sample(unsigned long long seed, uint32_t pair_id, uint32_t hyp, int n, int s,
                                           int* idx) {
  uint32_t w[8];
#pragma unroll
  for (int blk = 0; blk < 2; ++blk) {
    uint32_t c[4] = {hyp, pair_id, static_cast<uint32_t>(blk), 0u};
    philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
#pragma unroll
    for (int q = 0; q < 4; ++q) w[blk * 4 + q] = c[q];
  }
  for (int j = 0; j < s; ++j) {
    int r = static_cast<int>((static_cast<unsigned long long>(w[j]) * static_cast<unsigned>(n - j)) >> 32);
    int pos = 0;
    for (; pos < j && idx[pos] <= r; ++pos) ++r;   // skip the drawn indices at or below r (ascending)
    for (int q = j; q > pos; --q) idx[q] = idx[q - 1];
    idx[pos] = r;
  }
}

// ---------------------------------------------------------------------------------------------- small linear algebra
// Hartley normalisation of a point set from its sums: centroid to the origin, RMS distance sqrt(2).
// t = {scale, -scale*cx, -scale*cy}; false when the points coincide.
__host__ __device__ __forceinline__ bool geo_norm_from_sums(double n, double sx, double sy, double sq, double t[3]) {
  const double cx = sx / n, cy = sy / n;
  const double d2 = sq / n - (cx * cx + cy * cy);
  if (!(d2 > 1e-24 * (sq / n) + 1e-300)) return false;
  const double s = sqrt(2.0 / d2);
  t[0] = s; t[1] = -s * cx; t[2] = -s * cy;
  return true;
}

// Cyclic Jacobi on the symmetric N x N matrix a (destroyed): eigenvalues on its diagonal, eigenvectors in the columns
// of v.  Sweeps stop when the off-diagonal mass vanishes against the diagonal, or after kGeoJacobiSweeps.
template <int N>
__device__ void geo_jacobi(double (&a)[N][N], double (&v)[N][N]) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) v[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kGeoJacobiSweeps; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < N; ++i) {
      diag += a[i][i] * a[i][i];
      for (int j = i + 1; j < N; ++j) off += a[i][j] * a[i][j];
    }
    if (off <= 1e-36 * diag || off == 0.0) break;
    for (int p = 0; p < N - 1; ++p) {
      for (int q = p + 1; q < N; ++q) {
        const double apq = a[p][q];
        if (apq == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {   // a <- a J (columns p, q)
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {   // a <- J^T a (rows p, q)
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq;
          v[k][q] = s * vkp + c * vkq;
        }
      }
    }
  }
}

// Smallest eigenvector of the symmetric 9 x 9 matrix m (row-major, destroyed) into x; rank_ok: the second-smallest
// eigenvalue is above kGeoRankEps of the largest (the null space is one-dimensional).
__device__ void geo_null9(double (&m)[9][9], double x[9], bool* rank_ok) {
  double v[9][9];
  geo_jacobi<9>(m, v);
  int i0 = 0;
  double lmax = m[0][0];
  for (int i = 1; i < 9; ++i) {
    if (m[i][i] < m[i0][i0]) i0 = i;
    lmax = fmax(lmax, m[i][i]);
  }
  double l2 = INFINITY;
  for (int i = 0; i < 9; ++i)
    if (i != i0) l2 = fmin(l2, m[i][i]);
  *rank_ok = l2 > kGeoRankEps * lmax;
  for (int i = 0; i < 9; ++i) x[i] = v[i][i0];
}

// F <- F (I - v v^T), v the right singular vector of F's smallest singular value: the closest rank-2 matrix.
__device__ void geo_rank2(double f[9]) {
  double g[3][3], v[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) g[i][j] = f[i] * f[j] + f[3 + i] * f[3 + j] + f[6 + i] * f[6 + j];
  geo_jacobi<3>(g, v);
  int i0 = 0;
  for (int i = 1; i < 3; ++i)
    if (g[i][i] < g[i0][i0]) i0 = i;
  const double v0 = v[0][i0], v1 = v[1][i0], v2 = v[2][i0];
  for (int r = 0; r < 3; ++r) {
    const double fv = f[3 * r] * v0 + f[3 * r + 1] * v1 + f[3 * r + 2] * v2;
    f[3 * r] -= fv * v0;
    f[3 * r + 1] -= fv * v1;
    f[3 * r + 2] -= fv * v2;
  }
}

// Pixel-space model from the normalised one: H = T1^-1 Hn T0, F = T1^T Fn T0 (t0, t1 from geo_norm_from_sums).
__host__ __device__ __forceinline__ void geo_denormalise(int model, const double mn[9], const double t0[3],
                                                         const double t1[3], double out[9]) {
  double a[9];   // Mn T0: column j scaled by s0, column 2 gets the translation
  for (int r = 0; r < 3; ++r) {
    a[3 * r] = mn[3 * r] * t0[0];
    a[3 * r + 1] = mn[3 * r + 1] * t0[0];
    a[3 * r + 2] = mn[3 * r] * t0[1] + mn[3 * r + 1] * t0[2] + mn[3 * r + 2];
  }
  if (model == 0) {   // T1^-1 = [[1/s, 0, -tx/s], [0, 1/s, -ty/s], [0, 0, 1]]
    const double is = 1.0 / t1[0];
    for (int c = 0; c < 3; ++c) {
      out[c] = is * (a[c] - t1[1] * a[6 + c]);
      out[3 + c] = is * (a[3 + c] - t1[2] * a[6 + c]);
      out[6 + c] = a[6 + c];
    }
  } else {            // T1^T = [[s, 0, 0], [0, s, 0], [tx, ty, 1]]
    for (int c = 0; c < 3; ++c) {
      out[c] = t1[0] * a[c];
      out[3 + c] = t1[0] * a[3 + c];
      out[6 + c] = t1[1] * a[c] + t1[2] * a[3 + c] + a[6 + c];
    }
  }
}

// inverse through the adjugate; false when singular or not finite
__device__ __forceinline__ bool geo_inverse3(const double m[9], double inv[9]) {
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  if (!(fabs(det) > 0.0) || !isfinite(det)) return false;
  const double id = 1.0 / det;
  inv[0] = c00 * id; inv[1] = (m[2] * m[7] - m[1] * m[8]) * id; inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  inv[3] = c01 * id; inv[4] = (m[0] * m[8] - m[2] * m[6]) * id; inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  inv[6] = c02 * id; inv[7] = (m[1] * m[6] - m[0] * m[7]) * id; inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  return true;
}

// Squared pixel error of match (x0, y0) <-> (x1, y1):
//   homography (model 0): symmetric transfer error, the mean of |x1 - H x0|^2 and |x0 - H^-1 x1|^2;
//   fundamental (model 1): Sampson error (x1^T F x0)^2 / ((F x0)_1^2 + (F x0)_2^2 + (F^T x1)_1^2 + (F^T x1)_2^2).
// A point mapped to infinity, or a zero denominator, gives inf or NaN: never an inlier (callers test err < thr^2).
__device__ __forceinline__ double geo_error(int model, const double m[9], const double mi[9], double x0, double y0,
                                            double x1, double y1) {
  if (model == 0) {
    const double pw = m[6] * x0 + m[7] * y0 + m[8];
    const double px = (m[0] * x0 + m[1] * y0 + m[2]) / pw - x1;
    const double py = (m[3] * x0 + m[4] * y0 + m[5]) / pw - y1;
    const double qw = mi[6] * x1 + mi[7] * y1 + mi[8];
    const double qx = (mi[0] * x1 + mi[1] * y1 + mi[2]) / qw - x0;
    const double qy = (mi[3] * x1 + mi[4] * y1 + mi[5]) / qw - y0;
    return 0.5 * (px * px + py * py + qx * qx + qy * qy);
  }
  const double f0 = m[0] * x0 + m[1] * y0 + m[2];
  const double f1 = m[3] * x0 + m[4] * y0 + m[5];
  const double f2 = m[6] * x0 + m[7] * y0 + m[8];
  const double g0 = m[0] * x1 + m[3] * y1 + m[6];
  const double g1 = m[1] * x1 + m[4] * y1 + m[7];
  const double e = x1 * f0 + y1 * f1 + f2;
  return e * e / (f0 * f0 + f1 * f1 + g0 * g0 + g1 * g1);
}

// ---------------------------------------------------------------------------------------------- minimal solvers
// Homography from 4 matches: normalised DLT with h33 = 1, an 8 x 8 solve by Gaussian elimination with partial
// pivoting.  Degenerate: three collinear points in either image (|cross| < kGeoCollinearEps after normalisation) or
// a pivot below kGeoPivotEps.
__device__ bool geo_solve_h4(const float4* p, double h[9]) {
  double sx0 = 0, sy0 = 0, sq0 = 0, sx1 = 0, sy1 = 0, sq1 = 0;
  for (int i = 0; i < 4; ++i) {
    sx0 += p[i].x; sy0 += p[i].y; sq0 += (double)p[i].x * p[i].x + (double)p[i].y * p[i].y;
    sx1 += p[i].z; sy1 += p[i].w; sq1 += (double)p[i].z * p[i].z + (double)p[i].w * p[i].w;
  }
  double t0[3], t1[3];
  if (!geo_norm_from_sums(4.0, sx0, sy0, sq0, t0) || !geo_norm_from_sums(4.0, sx1, sy1, sq1, t1)) return false;
  double u[4], v[4], u2[4], v2[4];
  for (int i = 0; i < 4; ++i) {
    u[i] = t0[0] * p[i].x + t0[1]; v[i] = t0[0] * p[i].y + t0[2];
    u2[i] = t1[0] * p[i].z + t1[1]; v2[i] = t1[0] * p[i].w + t1[2];
  }
  for (int a = 0; a < 4; ++a)           // every triple, in both images
    for (int b = a + 1; b < 4; ++b)
      for (int c = b + 1; c < 4; ++c) {
        const double c0 = (u[b] - u[a]) * (v[c] - v[a]) - (v[b] - v[a]) * (u[c] - u[a]);
        const double c1 = (u2[b] - u2[a]) * (v2[c] - v2[a]) - (v2[b] - v2[a]) * (u2[c] - u2[a]);
        if (!(fabs(c0) >= kGeoCollinearEps) || !(fabs(c1) >= kGeoCollinearEps)) return false;
      }
  double A[8][9];
  for (int i = 0; i < 4; ++i) {
    double* r0 = A[2 * i];
    double* r1 = A[2 * i + 1];
    r0[0] = u[i]; r0[1] = v[i]; r0[2] = 1; r0[3] = 0; r0[4] = 0; r0[5] = 0;
    r0[6] = -u[i] * u2[i]; r0[7] = -v[i] * u2[i]; r0[8] = u2[i];
    r1[0] = 0; r1[1] = 0; r1[2] = 0; r1[3] = u[i]; r1[4] = v[i]; r1[5] = 1;
    r1[6] = -u[i] * v2[i]; r1[7] = -v[i] * v2[i]; r1[8] = v2[i];
  }
  for (int c = 0; c < 8; ++c) {
    int piv = c;
    for (int r = c + 1; r < 8; ++r)
      if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
    if (!(fabs(A[piv][c]) >= kGeoPivotEps)) return false;
    if (piv != c)
      for (int k = c; k < 9; ++k) {
        const double t = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = t;
      }
    const double ip = 1.0 / A[c][c];
    for (int r = c + 1; r < 8; ++r) {
      const double f = A[r][c] * ip;
      for (int k = c; k < 9; ++k) A[r][k] -= f * A[c][k];
    }
  }
  double hn[9];
  hn[8] = 1.0;
  for (int c = 7; c >= 0; --c) {
    double s = A[c][8];
    for (int k = c + 1; k < 8; ++k) s -= A[c][k] * hn[k];
    hn[c] = s / A[c][c];
  }
  geo_denormalise(0, hn, t0, t1, h);
  for (int i = 0; i < 9; ++i)
    if (!isfinite(h[i])) return false;
  return true;
}

// Accumulates the upper triangle of a a^T for one row a of the homogeneous system into m
__device__ __forceinline__ void geo_accum_row(double (&m)[9][9], const double a[9]) {
  for (int i = 0; i < 9; ++i)
    for (int j = i; j < 9; ++j) m[i][j] += a[i] * a[j];
}

// Rows of the homogeneous systems in normalised coordinates (u, v) -> (u2, v2):
//   F: x1^T F x0 = 0, a = kron((u2, v2, 1), (u, v, 1));
//   H: the two DLT rows of (u2, v2, 1) x H (u, v, 1) = 0.
__device__ __forceinline__ void geo_f_row(double u, double v, double u2, double v2, double a[9]) {
  a[0] = u2 * u; a[1] = u2 * v; a[2] = u2; a[3] = v2 * u; a[4] = v2 * v; a[5] = v2; a[6] = u; a[7] = v; a[8] = 1.0;
}
__device__ __forceinline__ void geo_h_rows(double u, double v, double u2, double v2, double a[9], double b[9]) {
  a[0] = -u; a[1] = -v; a[2] = -1.0; a[3] = 0.0; a[4] = 0.0; a[5] = 0.0; a[6] = u2 * u; a[7] = u2 * v; a[8] = u2;
  b[0] = 0.0; b[1] = 0.0; b[2] = 0.0; b[3] = -u; b[4] = -v; b[5] = -1.0; b[6] = v2 * u; b[7] = v2 * v; b[8] = v2;
}

// Solves the normalised homogeneous system m (upper triangle filled) for the model; false when rank-deficient (F
// minimal sample) or not finite.  F gets its rank-2 constraint in normalised coordinates, then both are denormalised.
__device__ bool geo_solve_system(int model, double (&m)[9][9], const double t0[3], const double t1[3], bool need_rank,
                                 double out[9]) {
  for (int i = 0; i < 9; ++i)
    for (int j = 0; j < i; ++j) m[i][j] = m[j][i];
  double x[9];
  bool rank_ok;
  geo_null9(m, x, &rank_ok);
  if (need_rank && !rank_ok) return false;
  if (model == 1) geo_rank2(x);
  geo_denormalise(model, x, t0, t1, out);
  for (int i = 0; i < 9; ++i)
    if (!isfinite(out[i])) return false;
  return true;
}

// Fundamental matrix from 8 matches: normalised 8-point (null vector of A^T A), rank 2 enforced.
__device__ bool geo_solve_f8(const float4* p, double f[9]) {
  double sx0 = 0, sy0 = 0, sq0 = 0, sx1 = 0, sy1 = 0, sq1 = 0;
  for (int i = 0; i < 8; ++i) {
    sx0 += p[i].x; sy0 += p[i].y; sq0 += (double)p[i].x * p[i].x + (double)p[i].y * p[i].y;
    sx1 += p[i].z; sy1 += p[i].w; sq1 += (double)p[i].z * p[i].z + (double)p[i].w * p[i].w;
  }
  double t0[3], t1[3];
  if (!geo_norm_from_sums(8.0, sx0, sy0, sq0, t0) || !geo_norm_from_sums(8.0, sx1, sy1, sq1, t1)) return false;
  double m[9][9];
  for (int i = 0; i < 9; ++i)
    for (int j = 0; j < 9; ++j) m[i][j] = 0.0;
  for (int i = 0; i < 8; ++i) {
    double a[9];
    geo_f_row(t0[0] * p[i].x + t0[1], t0[0] * p[i].y + t0[2], t1[0] * p[i].z + t1[1], t1[0] * p[i].w + t1[2], a);
    geo_accum_row(m, a);
  }
  return geo_solve_system(1, m, t0, t1, true, f);
}

// Hypothesis `hyp` of a pair with n >= s compacted matches pts: its sample (ascending compacted indices) and model;
// false when degenerate.
__device__ bool geo_hypothesis(int model, const float4* __restrict__ pts, int n, unsigned long long seed,
                               uint32_t pair_id, int hyp, int* idx, double m[9]) {
  const int s = model == 0 ? 4 : 8;
  geo_sample(seed, pair_id, static_cast<uint32_t>(hyp), n, s, idx);
  float4 p[kGeoMaxSample];
  for (int i = 0; i < s; ++i) p[i] = pts[idx[i]];
  return model == 0 ? geo_solve_h4(p, m) : geo_solve_f8(p, m);
}

// ---------------------------------------------------------------------------------------------- kernels
struct GeoParams {
  const float* pts0;         // [B, K, 2]
  const float* pts1;         // [B, K, 2]
  const uint8_t* valid;      // [B, K] or null (all valid)
  const int* pair_ids;       // [B] RNG key per pair, or null (the pair's index)
  int B, K, model, iterations, n_tiles;
  unsigned long long seed;
  double thr2;
  float4* compact;           // ws [B, K]
  int* compact_col;          // ws [B, K]
  int* n_valid;              // ws [B]
  GeoBest* tile_best;        // ws [B, n_tiles]
  float* model_out;          // [B, 9]
  uint8_t* mask_out;         // [B, K]
  int* count_out;            // [B]
  int* best_out;             // [B] or null: index of the best hypothesis, -1 when none
  int* samples_out;          // [B, iterations, s] or null: each hypothesis' sample as columns of K, -1 when n < s
};

__device__ __forceinline__ uint32_t geo_pair_id(const GeoParams& p, int b) {
  return static_cast<uint32_t>(p.pair_ids ? p.pair_ids[b] : b);
}

// One block per pair: valid matches of row b in column order -> compact[b, 0..n), compact_col, n_valid[b].
__global__ void __launch_bounds__(kGeoRefitThreads) geometry_compact_kernel(GeoParams p) {
  const int b = blockIdx.x;
  __shared__ int warp_n[kGeoRefitThreads / 32];
  __shared__ int base;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const long row = static_cast<long>(b) * p.K;
  for (int k0 = 0; k0 < p.K; k0 += kGeoRefitThreads) {
    const int k = k0 + threadIdx.x;
    const bool v = k < p.K && (p.valid == nullptr || p.valid[row + k] != 0);
    const unsigned bal = __ballot_sync(0xffffffffu, v);
    if (lane == 0) warp_n[wid] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < wid; ++w) off += warp_n[w];
    off += __popc(bal & ((1u << lane) - 1u));
    if (v) {
      const float2 a = reinterpret_cast<const float2*>(p.pts0)[row + k];
      const float2 c = reinterpret_cast<const float2*>(p.pts1)[row + k];
      p.compact[row + off] = make_float4(a.x, a.y, c.x, c.y);
      p.compact_col[row + off] = k;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 0; w < kGeoRefitThreads / 32; ++w) base += warp_n[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) p.n_valid[b] = base;
}

__device__ __forceinline__ GeoBest geo_shfl_best(const GeoBest& a, int delta) {
  GeoBest o;
  o.sum = __shfl_down_sync(0xffffffffu, a.sum, delta);
  o.count = __shfl_down_sync(0xffffffffu, a.count, delta);
  o.hyp = __shfl_down_sync(0xffffffffu, a.hyp, delta);
  return o;
}

// grid (n_tiles, B): thread t of tile j scores hypothesis j * kGeoHypPerBlock + t of pair blockIdx.y.
__global__ void __launch_bounds__(kGeoHypPerBlock) geometry_score_kernel(GeoParams p) {
  __shared__ float4 stage[kGeoStage];
  __shared__ GeoBest warp_best[kGeoHypPerBlock / 32];
  const int b = blockIdx.y;
  const int hyp = blockIdx.x * kGeoHypPerBlock + threadIdx.x;
  const int n = p.n_valid[b];
  const int s = p.model == 0 ? 4 : 8;
  const long row = static_cast<long>(b) * p.K;
  const float4* pts = p.compact + row;
  double m[9], mi[9];
  int idx[kGeoMaxSample];
  bool ok = false;
  if (hyp < p.iterations && n >= s) {
    ok = geo_hypothesis(p.model, pts, n, p.seed, geo_pair_id(p, b), hyp, idx, m);
    if (ok && p.model == 0) ok = geo_inverse3(m, mi);
  }
  if (p.samples_out != nullptr && hyp < p.iterations) {
    int* so = p.samples_out + (static_cast<long>(b) * p.iterations + hyp) * s;
    for (int i = 0; i < s; ++i) so[i] = n >= s ? p.compact_col[row + idx[i]] : -1;
  }
  GeoBest best{0.0, -1, hyp};
  if (ok) best.count = 0;
  double sum_in = 0.0;
  for (int c0 = 0; c0 < n; c0 += kGeoStage) {
    const int cn = min(kGeoStage, n - c0);
    __syncthreads();
    for (int i = threadIdx.x; i < cn; i += kGeoHypPerBlock) stage[i] = pts[c0 + i];
    __syncthreads();
    if (ok) {
      int cnt = 0;
      double sm = 0.0;
#pragma unroll 4
      for (int i = 0; i < cn; ++i) {
        const float4 q = stage[i];
        const double e = geo_error(p.model, m, mi, q.x, q.y, q.z, q.w);
        if (e < p.thr2) {
          ++cnt;
          sm += e;
        }
      }
      best.count += cnt;
      sum_in += sm;
    }
  }
  if (ok) best.sum = sum_in + static_cast<double>(n - best.count) * p.thr2;
  // block argmax under geo_better: warp shuffles, then the warps' winners in order
  for (int d = 16; d > 0; d >>= 1) {
    const GeoBest o = geo_shfl_best(best, d);
    if (geo_better(o, best)) best = o;
  }
  if ((threadIdx.x & 31) == 0) warp_best[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    GeoBest bb = warp_best[0];
    for (int w = 1; w < kGeoHypPerBlock / 32; ++w)
      if (geo_better(warp_best[w], bb)) bb = warp_best[w];
    p.tile_best[static_cast<long>(b) * p.n_tiles + blockIdx.x] = bb;
  }
}

// Block-wide sum of N doubles per thread (fixed order: warp trees, then the warps in order); the result is valid in
// thread 0.  red: shared [kGeoRefitThreads / 32][N].
template <int N>
__device__ void geo_block_sum(double (&v)[N], double (*red)[N]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i = 0; i < N; ++i) {
    double x = v[i];
    for (int d = 16; d > 0; d >>= 1) x += __shfl_down_sync(0xffffffffu, x, d);
    if (lane == 0) red[wid][i] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 0; i < N; ++i) {
      double x = red[0][i];
      for (int w = 1; w < kGeoRefitThreads / 32; ++w) x += red[w][i];
      v[i] = x;
    }
  __syncthreads();
}

// One block per pair: the best hypothesis over the tiles, least squares on its inliers, the final inlier mask.
__global__ void __launch_bounds__(kGeoRefitThreads) geometry_refit_kernel(GeoParams p) {
  __shared__ double model_s[9], inv_s[9];
  __shared__ int state_s;     // 0: no model, 1: model in model_s / inv_s
  __shared__ double red6[kGeoRefitThreads / 32][6];
  __shared__ double red45[kGeoRefitThreads / 32][45];
  __shared__ double red1[kGeoRefitThreads / 32][1];
  __shared__ double t_s[6];
  const int b = blockIdx.x;
  const int n = p.n_valid[b];
  const int s = p.model == 0 ? 4 : 8;
  const long row = static_cast<long>(b) * p.K;
  const float4* pts = p.compact + row;
  if (threadIdx.x == 0) {
    GeoBest best{0.0, -1, -1};
    for (int t = 0; t < p.n_tiles; ++t) {
      const GeoBest c = p.tile_best[static_cast<long>(b) * p.n_tiles + t];
      if (c.count >= 0 && (best.count < 0 || geo_better(c, best))) best = c;
    }
    state_s = 0;
    if (n >= s && best.count >= 0) {
      int idx[kGeoMaxSample];
      double m[9], mi[9];
      if (geo_hypothesis(p.model, pts, n, p.seed, geo_pair_id(p, b), best.hyp, idx, m)) {
        if (p.model == 1 || geo_inverse3(m, mi)) {
          for (int i = 0; i < 9; ++i) {
            model_s[i] = m[i];
            inv_s[i] = p.model == 0 ? mi[i] : 0.0;
          }
          state_s = 1;
        }
      }
    }
    if (p.best_out) p.best_out[b] = state_s ? best.hyp : -1;
  }
  for (int k = threadIdx.x; k < p.K; k += kGeoRefitThreads) p.mask_out[row + k] = 0;
  __syncthreads();
  if (state_s == 0) {
    if (threadIdx.x < 9) p.model_out[b * 9 + threadIdx.x] = __int_as_float(0x7fc00000);   // NaN
    if (threadIdx.x == 0) p.count_out[b] = 0;
    return;
  }
  double m[9], mi[9];
  for (int i = 0; i < 9; ++i) {
    m[i] = model_s[i];
    mi[i] = inv_s[i];
  }
  // 1. Hartley normalisation of the inliers of both images
  double st[6] = {0, 0, 0, 0, 0, 0};   // sx0, sy0, sq0, sx1, sy1, sq1
  double cnt[1] = {0};
  for (int i = threadIdx.x; i < n; i += kGeoRefitThreads) {
    const float4 q = pts[i];
    if (geo_error(p.model, m, mi, q.x, q.y, q.z, q.w) < p.thr2) {
      cnt[0] += 1.0;
      st[0] += q.x; st[1] += q.y; st[2] += (double)q.x * q.x + (double)q.y * q.y;
      st[3] += q.z; st[4] += q.w; st[5] += (double)q.z * q.z + (double)q.w * q.w;
    }
  }
  geo_block_sum<6>(st, red6);
  geo_block_sum<1>(cnt, red1);
  if (threadIdx.x == 0) {
    double t0[3], t1[3];
    const bool ok = cnt[0] >= s && geo_norm_from_sums(cnt[0], st[0], st[1], st[2], t0) &&
                    geo_norm_from_sums(cnt[0], st[3], st[4], st[5], t1);
    state_s = ok ? 2 : 1;     // 2: refit
    for (int i = 0; i < 3; ++i) {
      t_s[i] = ok ? t0[i] : 0.0;
      t_s[3 + i] = ok ? t1[i] : 0.0;
    }
  }
  __syncthreads();
  if (state_s == 2) {
    // 2. normal equations of all inliers, upper triangle packed row by row
    double acc[45];
    for (int i = 0; i < 45; ++i) acc[i] = 0.0;
    const double s0 = t_s[0], a0 = t_s[1], b0 = t_s[2], s1 = t_s[3], a1 = t_s[4], b1 = t_s[5];
    for (int i = threadIdx.x; i < n; i += kGeoRefitThreads) {
      const float4 q = pts[i];
      if (!(geo_error(p.model, m, mi, q.x, q.y, q.z, q.w) < p.thr2)) continue;
      const double u = s0 * q.x + a0, v = s0 * q.y + b0, u2 = s1 * q.z + a1, v2 = s1 * q.w + b1;
      double r0[9], r1[9];
      int nr = 1;
      if (p.model == 0) {
        geo_h_rows(u, v, u2, v2, r0, r1);
        nr = 2;
      } else {
        geo_f_row(u, v, u2, v2, r0);
      }
      for (int r = 0; r < nr; ++r) {
        const double* a = r == 0 ? r0 : r1;
        int k = 0;
        for (int ii = 0; ii < 9; ++ii)
          for (int jj = ii; jj < 9; ++jj) acc[k++] += a[ii] * a[jj];
      }
    }
    geo_block_sum<45>(acc, red45);
    if (threadIdx.x == 0) {
      double mm[9][9];
      int k = 0;
      for (int ii = 0; ii < 9; ++ii)
        for (int jj = ii; jj < 9; ++jj) mm[ii][jj] = acc[k++];
      const double t0[3] = {s0, a0, b0}, t1[3] = {s1, a1, b1};
      double r[9], ri[9];
      if (geo_solve_system(p.model, mm, t0, t1, false, r) && (p.model == 1 || geo_inverse3(r, ri)))
        for (int i = 0; i < 9; ++i) {
          model_s[i] = r[i];
          inv_s[i] = p.model == 0 ? ri[i] : 0.0;
        }
    }
    __syncthreads();
    for (int i = 0; i < 9; ++i) {
      m[i] = model_s[i];
      mi[i] = inv_s[i];
    }
  }
  // 3. final inlier mask and count under the returned model
  double fin[1] = {0};
  for (int i = threadIdx.x; i < n; i += kGeoRefitThreads) {
    const float4 q = pts[i];
    if (geo_error(p.model, m, mi, q.x, q.y, q.z, q.w) < p.thr2) {
      p.mask_out[row + p.compact_col[row + i]] = 1;
      fin[0] += 1.0;
    }
  }
  geo_block_sum<1>(fin, red1);
  if (threadIdx.x == 0) {
    // output scale: H with H[2][2] = 1 (unit Frobenius norm when |H[2][2]| is negligible); F with unit Frobenius
    // norm and its largest-magnitude entry positive
    double nrm = 0.0;
    int imax = 0;
    for (int i = 0; i < 9; ++i) {
      nrm += m[i] * m[i];
      if (fabs(m[i]) > fabs(m[imax])) imax = i;
    }
    nrm = sqrt(nrm);
    double d = m[imax] < 0.0 ? -nrm : nrm;
    if (p.model == 0 && fabs(m[8]) > 1e-12 * nrm) d = m[8];
    for (int i = 0; i < 9; ++i) p.model_out[b * 9 + i] = static_cast<float>(m[i] / d);
    p.count_out[b] = static_cast<int>(fin[0]);
  }
}

}  // namespace lb
