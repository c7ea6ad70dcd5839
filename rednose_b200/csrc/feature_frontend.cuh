// rednose_b200 -- MSCKF front-end kernels: batched feature-track triangulation and track bookkeeping (sm_90a).
//
// Replaces, for a batch of independent tracks / camera frames,
//   rednose/templates/compute_pos.c:10-27   gauss_newton()   (Eigen 2K x 3 least squares, <= 30 iterations)
//   rednose/templates/compute_pos.c:30-52   compute_pos()    (initial guess, camera -> ECEF transform)
//   rednose/templates/feature_handler.c:1-21   sane()
//   rednose/templates/feature_handler.c:23-56  merge_features()
// Included at the end of the generated features_<K>.cu, after `struct feature_model` (pose_term = one pose's residual
// pair + Jacobian rows, generated from sympy by rednose_b200/features.py).
//
// compute_pos_thread: one thread per track.  The track's K poses (7K doubles) and K image positions (2K doubles) are
// staged once through shared memory with coalesced loads (row pitch odd: conflict-free thread-per-row reads); every
// Gauss-Newton iteration loops over the poses accumulating the 3 x 3 normal equations J^T J and J^T E (the 2K x 3
// Jacobian of compute_pos.c:12 is never stored), solves them with the closed-form 3 x 3 inverse (what Eigen's
// fixed-size .inverse() does) and stops on |delta|^2 <= 1e-4 or 30 iterations, like the reference.
// Algorithmic bytes per track: 8 * (9K + 9 + 6) read/written = 840 B for K = 10.
//
// merge_features_cta: one CTA per camera frame (instance).  The reference loop is sequential over 3000 features because
// (a) two features may point at the same track (only the first may extend it) and (b) unmatched features take
// consecutive entries of empty_idxs.  Here (a) is an atomicMin per track over feature indices, (b) an exclusive block
// scan; if a new track's slot collides with a matched track or with another new track (the only cases where the
// sequential order changes the result) the instance falls back to an in-order single-thread pass, so results are
// bit-identical to the reference in every case.
#pragma once
#include <cuda_runtime.h>
#include <climits>
#include <cstdio>
#include <mutex>
#include "ekf_common.cuh"

namespace rnb {

// ------------------------------------------------------------------------------------------ triangulation ---
template <class FM>
__host__ __device__ __forceinline__ int gauss_newton_track(const double* poses, int pstride, const double* img, int istride, double* x) {
  constexpr int K = FM::K;
  const double* p0 = poses + (K - 1) * 7 * pstride;   // "pose 0" of the residual = the LAST pose (compute_pos.c:41-44 uses the same one)
  double p0r[7];
#pragma unroll
  for (int c = 0; c < 7; ++c) p0r[c] = p0[c * pstride];
  int counter = 0;
  double d2 = 0.0;
  while ((d2 > 0.0001 && counter < 30) || counter == 0) {   // compute_pos.c:18
    double A00 = 0, A01 = 0, A02 = 0, A11 = 0, A12 = 0, A22 = 0, g0 = 0, g1 = 0, g2 = 0;
#pragma unroll 1
    for (int i = 0; i < K; ++i) {
      double pi[7], uv[2], r[2], j[6];
#pragma unroll
      for (int c = 0; c < 7; ++c) pi[c] = poses[(i * 7 + c) * pstride];
      uv[0] = img[(2 * i) * istride]; uv[1] = img[(2 * i + 1) * istride];
      FM::pose_term(x, pi, p0r, uv, r, j);
#pragma unroll
      for (int a = 0; a < 2; ++a) {   // J^T J and J^T E, rows in the reference's order (2i, 2i+1)
        const double j0 = j[a * 3], j1 = j[a * 3 + 1], j2 = j[a * 3 + 2], e = r[a];
        A00 = fma(j0, j0, A00); A01 = fma(j0, j1, A01); A02 = fma(j0, j2, A02);
        A11 = fma(j1, j1, A11); A12 = fma(j1, j2, A12); A22 = fma(j2, j2, A22);
        g0 = fma(j0, e, g0); g1 = fma(j1, e, g1); g2 = fma(j2, e, g2);
      }
    }
    // delta = (J^T J)^-1 J^T E   (compute_pos.c:22): adjugate / determinant of the symmetric 3 x 3
    const double c00 = A11 * A22 - A12 * A12, c01 = A02 * A12 - A01 * A22, c02 = A01 * A12 - A02 * A11;
    const double c11 = A00 * A22 - A02 * A02, c12 = A01 * A02 - A00 * A12, c22 = A00 * A11 - A01 * A01;
    const double det = A00 * c00 + A01 * c01 + A02 * c02;
    const double id = 1.0 / det;
    const double d0 = (c00 * g0 + c01 * g1 + c02 * g2) * id;
    const double d1 = (c01 * g0 + c11 * g1 + c12 * g2) * id;
    const double d2_ = (c02 * g0 + c12 * g1 + c22 * g2) * id;
    x[0] -= d0; x[1] -= d1; x[2] -= d2_;
    d2 = d0 * d0 + d1 * d1 + d2_ * d2_;
    ++counter;
  }
  return counter;
}

// camera frame -> ECEF (compute_pos.c:36-51): rot = R(q_last normalised) * to_c^T
__host__ __device__ __forceinline__ void camera_to_ecef(const double* to_c, const double* last_pose, int pstride, const double* param, double* pos) {
  double qw = last_pose[3 * pstride], qx = last_pose[4 * pstride], qy = last_pose[5 * pstride], qz = last_pose[6 * pstride];
  const double n = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
  qw /= n; qx /= n; qy /= n; qz /= n;
  // Eigen::Quaternion::toRotationMatrix
  const double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx, tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  const double v[3] = {param[0] / param[2], param[1] / param[2], 1.0 / param[2]};
  double cam[3];   // to_c^T v
#pragma unroll
  for (int i = 0; i < 3; ++i) cam[i] = to_c[0 * 3 + i] * v[0] + to_c[1 * 3 + i] * v[1] + to_c[2 * 3 + i] * v[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) pos[i] = R[i * 3] * cam[0] + R[i * 3 + 1] * cam[1] + R[i * 3 + 2] * cam[2] + last_pose[i * pstride];
}

constexpr int CP_THREADS = 64;

template <class FM>
__global__ void __launch_bounds__(CP_THREADS) compute_pos_thread(const double* __restrict__ to_c, const double* __restrict__ poses, const double* __restrict__ img,
                                                                  double* __restrict__ param, double* __restrict__ pos, int* __restrict__ iters, long long B, double fallback_depth) {
  constexpr int K = FM::K, REC = 9 * K, PITCH = REC | 1;
  extern __shared__ double sm[];
  const long long b0 = (long long)blockIdx.x * CP_THREADS;
  const int nb = (int)((B - b0 < CP_THREADS) ? (B - b0) : CP_THREADS);
  // coalesced staging: poses rows then image rows of the block's tracks
  for (int idx = threadIdx.x; idx < nb * 7 * K; idx += CP_THREADS) {
    const int t = idx / (7 * K), c = idx - t * 7 * K;
    sm[t * PITCH + c] = poses[b0 * 7 * K + idx];
  }
  for (int idx = threadIdx.x; idx < nb * 2 * K; idx += CP_THREADS) {
    const int t = idx / (2 * K), c = idx - t * 2 * K;
    sm[t * PITCH + 7 * K + c] = img[b0 * 2 * K + idx];
  }
  __syncthreads();
  if ((int)threadIdx.x >= nb) return;
  const double* mp = sm + threadIdx.x * PITCH;
  const double* mi = mp + 7 * K;
  double x[3] = {mi[2 * K - 2], mi[2 * K - 1], 0.1};   // compute_pos.c:31-33
  int it = gauss_newton_track<FM>(mp, 1, mi, 1, x);
  double p[3];
  double tc[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) tc[i] = __ldg(to_c + i);
  camera_to_ecef(tc, mp + (K - 1) * 7, 1, x, p);
  // optional guard (fallback_depth > 0; the reference has none): a track whose Gauss-Newton hit the iteration cap or left
  // the finite range gets a finite stand-in on the optical axis of the last camera and iters = -iterations, so that the
  // caller / the filter's Mahalanobis gate can reject it instead of a NaN reaching the state
  if (fallback_depth > 0.0 && (it >= 30 || !(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2])))) {
    x[0] = 0.0; x[1] = 0.0; x[2] = 1.0 / fallback_depth;
    camera_to_ecef(tc, mp + (K - 1) * 7, 1, x, p);
    it = -it;
  }
  const long long b = b0 + threadIdx.x;
#pragma unroll
  for (int i = 0; i < 3; ++i) { param[b * 3 + i] = x[i]; pos[b * 3 + i] = p[i]; }
  if (iters) iters[b] = it;
}

// One LANE per (track, pose): the K pose terms of a Gauss-Newton iteration are independent, so a group of LPT >= K lanes
// evaluates them at once and butterfly-reduces the 9 sums of the normal equations (every lane of the group ends with
// bit-identical sums: the xor tree is symmetric and IEEE addition commutes), then every lane solves the same 3 x 3.  The
// dependent chain of an iteration is one pose term instead of K of them, at the 10 000 tracks of config 5
// where the thread-per-track kernel is pure latency.  The sums are formed in
// tree order instead of the reference's row order (compute_pos.c:22): same algorithm, last-bit differences.
template <class FM, int LPT>
__global__ void __launch_bounds__(128) compute_pos_lanes(const double* __restrict__ to_c, const double* __restrict__ poses, const double* __restrict__ img,
                                                         double* __restrict__ param, double* __restrict__ pos, int* __restrict__ iters, long long B, double fallback_depth) {
  constexpr int K = FM::K;
  static_assert(K <= LPT && (LPT == 8 || LPT == 16 || LPT == 32), "one lane per pose");
  const long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long b = gt / LPT;
  const int i = (int)(gt % LPT);
  if (b >= B) return;   // whole groups leave together (LPT divides the block size)
  const unsigned gmask = (LPT == 32) ? 0xffffffffu : (((1u << LPT) - 1u) << (((threadIdx.x & 31) / LPT) * LPT));
  const bool act = i < K;
  const double* tp = poses + b * 7 * K;
  const double* ti = img + b * 2 * K;
  double pi[7], p0[7], uv[2];
#pragma unroll
  for (int c = 0; c < 7; ++c) { pi[c] = tp[(act ? i : 0) * 7 + c]; p0[c] = tp[(K - 1) * 7 + c]; }
  uv[0] = ti[2 * (act ? i : 0)]; uv[1] = ti[2 * (act ? i : 0) + 1];
  double x[3] = {ti[2 * K - 2], ti[2 * K - 1], 0.1};   // compute_pos.c:31-33
  int counter = 0;
  double d2 = 0.0;
  while ((d2 > 0.0001 && counter < 30) || counter == 0) {   // compute_pos.c:18 (uniform inside the group)
    double r[2], j[6];
    FM::pose_term(x, pi, p0, uv, r, j);
    double sums[9];
    {
      const double w = act ? 1.0 : 0.0;   // idle lanes contribute exact zeros
      const double j0 = j[0] * w, j1 = j[1] * w, j2 = j[2] * w, j3 = j[3] * w, j4 = j[4] * w, j5 = j[5] * w, e0 = r[0] * w, e1 = r[1] * w;
      sums[0] = fma(j0, j0, j3 * j3); sums[1] = fma(j0, j1, j3 * j4); sums[2] = fma(j0, j2, j3 * j5);
      sums[3] = fma(j1, j1, j4 * j4); sums[4] = fma(j1, j2, j4 * j5); sums[5] = fma(j2, j2, j5 * j5);
      sums[6] = fma(j0, e0, j3 * e1); sums[7] = fma(j1, e0, j4 * e1); sums[8] = fma(j2, e0, j5 * e1);
    }
#pragma unroll
    for (int off = LPT / 2; off >= 1; off >>= 1) {
#pragma unroll
      for (int q = 0; q < 9; ++q) sums[q] += __shfl_xor_sync(gmask, sums[q], off);
    }
    const double A00 = sums[0], A01 = sums[1], A02 = sums[2], A11 = sums[3], A12 = sums[4], A22 = sums[5], g0 = sums[6], g1 = sums[7], g2 = sums[8];
    const double c00 = A11 * A22 - A12 * A12, c01 = A02 * A12 - A01 * A22, c02 = A01 * A12 - A02 * A11;
    const double c11 = A00 * A22 - A02 * A02, c12 = A01 * A02 - A00 * A12, c22 = A00 * A11 - A01 * A01;
    const double id = 1.0 / (A00 * c00 + A01 * c01 + A02 * c02);
    const double d0 = (c00 * g0 + c01 * g1 + c02 * g2) * id;
    const double d1 = (c01 * g0 + c11 * g1 + c12 * g2) * id;
    const double d2_ = (c02 * g0 + c12 * g1 + c22 * g2) * id;
    x[0] -= d0; x[1] -= d1; x[2] -= d2_;
    d2 = d0 * d0 + d1 * d1 + d2_ * d2_;
    ++counter;
  }
  if (i != 0) return;
  double tc[9], p[3];
#pragma unroll
  for (int q = 0; q < 9; ++q) tc[q] = __ldg(to_c + q);
  camera_to_ecef(tc, p0, 1, x, p);
  int it = counter;
  if (fallback_depth > 0.0 && (it >= 30 || !(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2])))) {   // see compute_pos_thread
    x[0] = 0.0; x[1] = 0.0; x[2] = 1.0 / fallback_depth;
    camera_to_ecef(tc, p0, 1, x, p);
    it = -it;
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) { param[b * 3 + q] = x[q]; pos[b * 3 + q] = p[q]; }
  if (iters) iters[b] = it;
}

// ------------------------------------------------------------------------------------------ track bookkeeping ---
// feature_handler.c:1-21 on one track [K + 1][5] (row 0 is the header)
template <int K>
__host__ __device__ __forceinline__ bool track_sane(const double* track) {
  double px = 0.0, py = 0.0;
  for (int i = 0; i < K - 1; ++i) {
    const double dx = fabs(track[(i + 2) * 5 + 2] - track[(i + 1) * 5 + 2]);
    const double dy = fabs(track[(i + 2) * 5 + 3] - track[(i + 1) * 5 + 3]);
    if (i >= 1) {
      if (((dx > 0.05 || px > 0.05) && (dx > 2 * px || dx < .5 * px)) || ((dy > 0.05 || py > 0.05) && (dy > 2 * py || dy < .5 * py))) return false;
    }
    px = dx; py = dy;
  }
  return true;
}

// one feature in program order (the body of the loop feature_handler.c:33-54); returns 1 if it consumed an empty slot.
// Writes outside the track table / the K + 1 rows of a track, which the reference would perform (undefined behaviour),
// are skipped.
template <int K>
__host__ __device__ __forceinline__ int merge_one(double* tracks, const double* feat, const long long* empty_idxs, int empty_idx, int n_tracks) {
  constexpr int TS = (K + 1) * 5;
  const int match = (int)feat[4];
  const bool in_range = match >= 0 && match < n_tracks;
  double* t = tracks + (long long)(in_range ? match : 0) * TS;
  if (in_range && t[1] == (double)match && t[2] == 0.0) {
    t[0] = t[0] + 1; t[1] = feat[1]; t[2] = 1;
    const int idx = (int)t[0];
    if (idx >= 0 && idx <= K) for (int c = 0; c < 5; ++c) t[idx * 5 + c] = feat[c];
    if (idx == K) {
      t[3] = 1;
      if (track_sane<K>(t)) t[4] = 1;
    }
    return 0;
  }
  const long long s = empty_idxs[empty_idx];
  if (s >= 0 && s < n_tracks) {
    double* n = tracks + s * TS;
    n[0] = 1; n[1] = feat[1]; n[2] = 1;
    for (int c = 0; c < 5; ++c) n[5 + c] = feat[c];
  }
  return 1;
}

constexpr int MF_THREADS = 256;

template <int K>
__global__ void __launch_bounds__(MF_THREADS) merge_features_cta(double* __restrict__ tracks_all, const double* __restrict__ feats_all, const long long* __restrict__ empty_all,
                                                                  int n_features, int n_tracks, int* __restrict__ fallbacks) {
  constexpr int TS = (K + 1) * 5;
  extern __shared__ int first[];              // [n_tracks]: smallest feature index whose match is this (extendable) track; then slot claims
  __shared__ int s_scan[MF_THREADS];
  __shared__ int s_conflict;
  const long long b = blockIdx.x;
  double* tracks = tracks_all + b * (long long)n_tracks * TS;
  const double* feats = feats_all + b * (long long)n_features * 5;
  const long long* empty_idxs = empty_all + b * (long long)n_features;
  const int tid = threadIdx.x;
  for (int t = tid; t < n_tracks; t += MF_THREADS) first[t] = INT_MAX;
  if (tid == 0) s_conflict = 0;
  __syncthreads();
  // (a) candidates: the header test of feature_handler.c:35 against the ORIGINAL headers
  for (int i = tid; i < n_features; i += MF_THREADS) {
    const int match = (int)feats[i * 5 + 4];
    if (match >= 0 && match < n_tracks) {
      const double* t = tracks + (long long)match * TS;
      if (t[1] == (double)match && t[2] == 0.0) atomicMin(&first[match], i);
    }
  }
  __syncthreads();
  // (b) each thread owns a contiguous chunk of features (program order inside the chunk), counts its unmatched ones
  const int per = (n_features + MF_THREADS - 1) / MF_THREADS;
  const int i0 = tid * per, i1 = (i0 + per < n_features) ? i0 + per : n_features;
  int cnt = 0;
  for (int i = i0; i < i1; ++i) {
    const int match = (int)feats[i * 5 + 4];
    const bool m = match >= 0 && match < n_tracks && first[match] == i;
    cnt += m ? 0 : 1;
  }
  s_scan[tid] = cnt;
  __syncthreads();
  for (int off = 1; off < MF_THREADS; off <<= 1) {   // inclusive Hillis-Steele scan
    const int v = (tid >= off) ? s_scan[tid - off] : 0;
    __syncthreads();
    s_scan[tid] += v;
    __syncthreads();
  }
  int e = s_scan[tid] - cnt;   // exclusive prefix: index into empty_idxs of this chunk's first new track
  // (c) conflicts: a new track's slot that is also an extended track, or claimed twice, or outside the table
  {
    int ee = e;
    for (int i = i0; i < i1; ++i) {
      const int match = (int)feats[i * 5 + 4];
      const bool m = match >= 0 && match < n_tracks && first[match] == i;
      if (!m) {
        const long long s = empty_idxs[ee++];
        if (s < 0 || s >= n_tracks) s_conflict = 1;
        else if (atomicExch(&first[(int)s], -1) != INT_MAX) s_conflict = 1;   // -1 = claimed by a new track
      }
    }
  }
  __syncthreads();
  if (s_conflict) {   // rare: replay in program order, exactly the reference loop
    if (tid == 0) {
      int ei = 0;
      for (int i = 0; i < n_features; ++i) ei += merge_one<K>(tracks, feats + i * 5, empty_idxs, ei, n_tracks);
      if (fallbacks) atomicAdd(fallbacks, 1);
    }
    return;
  }
  // (d) apply: every feature touches a distinct track now.  `first` has been overwritten by the claims only at new
  // slots, which no matched feature refers to (else s_conflict), so the match test is still valid.
  for (int i = i0; i < i1; ++i) {
    const double* f = feats + i * 5;
    const int match = (int)f[4];
    const bool m = match >= 0 && match < n_tracks && first[match] == i;
    if (m) {
      double* t = tracks + (long long)match * TS;
      const double cntr = t[0] + 1;
      t[0] = cntr; t[1] = f[1]; t[2] = 1;
      const int idx = (int)cntr;
      if (idx >= 0 && idx <= K) {
#pragma unroll
        for (int c = 0; c < 5; ++c) t[idx * 5 + c] = f[c];
      }
      if (idx == K) {
        t[3] = 1;
        if (track_sane<K>(t)) t[4] = 1;
      }
    } else {
      double* n = tracks + empty_idxs[e++] * TS;
      n[0] = 1; n[1] = f[1]; n[2] = 1;
#pragma unroll
      for (int c = 0; c < 5; ++c) n[5 + c] = f[c];
    }
  }
}

template <int K>
__global__ void sane_thread(const double* __restrict__ tracks, int* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = track_sane<K>(tracks + i * (K + 1) * 5) ? 1 : 0;
}

// leaf entry points res_fun / jac_fun in the template's full-K shape (one thread)
template <class FM>
__global__ void res_jac_kernel(const double* x, const double* poses, const double* img, double* res, double* jac) {
  constexpr int K = FM::K;
  if (threadIdx.x != 0) return;
  for (int i = 0; i < K; ++i) {
    double r[2], j[6];
    FM::pose_term(x, poses + 7 * i, poses + 7 * (K - 1), img + 2 * i, r, j);
    if (res) { res[2 * i] = r[0]; res[2 * i + 1] = r[1]; }
    if (jac) for (int c = 0; c < 6; ++c) jac[6 * i + c] = j[c];
  }
}

// ------------------------------------------------------------------------------------------------- host side ---
struct FeatureHost {
  std::mutex mu;
  // device scratch of the single-instance entry points, one per device
  double* d[32] = {nullptr}; size_t cap[32] = {0};
  double* scratch(size_t bytes) {
    int dev = 0; cudaGetDevice(&dev); if (dev < 0 || dev >= 32) dev = 0;
    if (bytes > cap[dev]) {
      if (d[dev]) cudaFree(d[dev]);
      d[dev] = nullptr; cap[dev] = 0;
      if (!check(cudaMalloc(&d[dev], bytes), "cudaMalloc(feature scratch)")) return nullptr;
      cap[dev] = bytes;
    }
    return d[dev];
  }
};
inline FeatureHost& fhost() { static FeatureHost h; return h; }

template <class FM>
inline void launch_compute_pos(const double* to_c, const double* poses, const double* img, double* param, double* pos, int* iters, long long B, cudaStream_t st, double fallback_depth = 0.0) {
  if (B <= 0) return;
  if constexpr (FM::K <= 32) {
    // lane-per-pose kernel (default): groups of LPT lanes per track
    constexpr int LPT = FM::K <= 8 ? 8 : (FM::K <= 16 ? 16 : 32);
    const long long threads = B * LPT;
    compute_pos_lanes<FM, LPT><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(to_c, poses, img, param, pos, iters, B, fallback_depth);
  } else {
    constexpr size_t smem = sizeof(double) * CP_THREADS * ((9 * FM::K) | 1);
    if (smem > 48 * 1024) cudaFuncSetAttribute(compute_pos_thread<FM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    compute_pos_thread<FM><<<(unsigned)((B + CP_THREADS - 1) / CP_THREADS), CP_THREADS, smem, st>>>(to_c, poses, img, param, pos, iters, B, fallback_depth);
  }
  check(cudaGetLastError(), "compute_pos launch");
}

template <class FM>
inline void launch_merge_features(double* tracks, const double* feats, const long long* empty_idxs, int nf, int nt, long long B, int* fallbacks, cudaStream_t st) {
  if (B <= 0) return;
  const size_t smem = sizeof(int) * (size_t)nt;
  if (smem > 200 * 1024) { fprintf(stderr, "[rednose_b200] merge_features: n_tracks %d too large for the shared-memory index\n", nt); last_status() = (int)cudaErrorInvalidValue; return; }
  if (smem > 48 * 1024) cudaFuncSetAttribute(merge_features_cta<FM::K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  merge_features_cta<FM::K><<<(unsigned)B, MF_THREADS, smem, st>>>(tracks, feats, empty_idxs, nf, nt, fallbacks);
  check(cudaGetLastError(), "merge_features launch");
}

}  // namespace rnb

// ------------------------------------------------------------------------------------------------- C-ABI ---
extern "C" {
int features_k(void) { return feature_model::K; }
int features_cuda_status(void) { int s = rnb::last_status(); rnb::last_status() = 0; return s; }

void compute_pos_batch(const double* to_c, const double* poses, const double* img_positions, double* param, double* pos, int* iters, long long B, double fallback_depth, void* stream) {
  rnb::launch_compute_pos<feature_model>(to_c, poses, img_positions, param, pos, iters, B, (cudaStream_t)stream, fallback_depth);
}
void merge_features_batch(double* tracks, const double* features, const long long* empty_idxs, int n_features, int n_tracks, long long B, int* fallbacks, void* stream) {
  rnb::launch_merge_features<feature_model>(tracks, features, empty_idxs, n_features, n_tracks, B, fallbacks, (cudaStream_t)stream);
}
void sane_batch(const double* tracks, int* out, long long n, void* stream) {
  if (n <= 0) return;
  rnb::sane_thread<feature_model::K><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(tracks, out, n);
  rnb::check(cudaGetLastError(), "sane launch");
}

// host pointers, one instance: rednose/templates/compute_pos.c:30 (same arguments: param and pos are outputs)
void compute_pos(double* to_c, double* poses, double* img_positions, double* param, double* pos) {
  constexpr int K = feature_model::K;
  auto& h = rnb::fhost();
  std::lock_guard<std::mutex> lk(h.mu);
  double* d = h.scratch(sizeof(double) * (9 + 9 * K + 6));
  if (!d) return;
  double stage[9 + 9 * K];
  memcpy(stage, to_c, sizeof(double) * 9); memcpy(stage + 9, poses, sizeof(double) * 7 * K); memcpy(stage + 9 + 7 * K, img_positions, sizeof(double) * 2 * K);
  if (!rnb::check(cudaMemcpy(d, stage, sizeof(stage), cudaMemcpyHostToDevice), "compute_pos memcpy")) return;
  rnb::launch_compute_pos<feature_model>(d, d + 9, d + 9 + 7 * K, d + 9 + 9 * K, d + 9 + 9 * K + 3, nullptr, 1, nullptr);
  double out[6];
  if (!rnb::check(cudaMemcpy(out, d + 9 + 9 * K, sizeof(out), cudaMemcpyDeviceToHost), "compute_pos memcpy back")) return;
  memcpy(param, out, sizeof(double) * 3); memcpy(pos, out + 3, sizeof(double) * 3);
}

static void res_jac_host(double* abr, double* poses, double* img, double* res, double* jac) {
  constexpr int K = feature_model::K;
  auto& h = rnb::fhost();
  std::lock_guard<std::mutex> lk(h.mu);
  double* d = h.scratch(sizeof(double) * (3 + 9 * K + 8 * K));
  if (!d) return;
  double stage[3 + 9 * K];
  memcpy(stage, abr, sizeof(double) * 3); memcpy(stage + 3, poses, sizeof(double) * 7 * K); memcpy(stage + 3 + 7 * K, img, sizeof(double) * 2 * K);
  if (!rnb::check(cudaMemcpy(d, stage, sizeof(stage), cudaMemcpyHostToDevice), "res_jac memcpy")) return;
  rnb::res_jac_kernel<feature_model><<<1, 32>>>(d, d + 3, d + 3 + 7 * K, d + 3 + 9 * K, d + 3 + 11 * K);
  rnb::check(cudaGetLastError(), "res_jac launch");
  if (res) rnb::check(cudaMemcpy(res, d + 3 + 9 * K, sizeof(double) * 2 * K, cudaMemcpyDeviceToHost), "res memcpy back");
  if (jac) rnb::check(cudaMemcpy(jac, d + 3 + 11 * K, sizeof(double) * 6 * K, cudaMemcpyDeviceToHost), "jac memcpy back");
}
void res_fun(double* abr, double* poses, double* img_positions, double* out) { res_jac_host(abr, poses, img_positions, out, nullptr); }
void jac_fun(double* abr, double* poses, double* img_positions, double* out) { res_jac_host(abr, poses, img_positions, nullptr, out); }

// host pointers, one camera frame with the template's fixed sizes: rednose/templates/feature_handler.c:23
void merge_features(double* tracks, double* features, long long* empty_idxs) {
  constexpr int K = feature_model::K, NF = 3000, NT = 6000;
  const size_t tb = sizeof(double) * NT * (K + 1) * 5, fb = sizeof(double) * NF * 5, eb = sizeof(long long) * NF;
  auto& h = rnb::fhost();
  std::lock_guard<std::mutex> lk(h.mu);
  char* d = (char*)h.scratch(tb + fb + eb);
  if (!d) return;
  if (!rnb::check(cudaMemcpy(d, tracks, tb, cudaMemcpyHostToDevice), "merge_features memcpy")) return;
  cudaMemcpy(d + tb, features, fb, cudaMemcpyHostToDevice);
  cudaMemcpy(d + tb + fb, empty_idxs, eb, cudaMemcpyHostToDevice);
  rnb::launch_merge_features<feature_model>((double*)d, (const double*)(d + tb), (const long long*)(d + tb + fb), NF, NT, 1, nullptr, nullptr);
  rnb::check(cudaMemcpy(tracks, d, tb, cudaMemcpyDeviceToHost), "merge_features memcpy back");
}
}  // extern "C"
