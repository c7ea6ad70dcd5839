// rednose_b200 -- common device/host helpers for the batched EKF kernels (sm_90a).
//
// Hot path being replaced: rednose/templates/ekf_c.c:8-33 (predict) and :37-121 (update),
// plus the driver-level quaternion normalisation rednose/helpers/ekf_sym.cc:69-77.
// All arithmetic is IEEE float64, all matrices row-major (ekf_c.c:4-6).
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <mutex>
#include <set>
#include <utility>

namespace rnb {

constexpr int MAX_QUAT = 8;

// runtime flags of a batched step
enum : int {
  FLAG_NORM_AFTER_PREDICT = 1,  // ekf_sym.cc:207 (the C++ driver does, the python driver does not)
  FLAG_NORM_AFTER_UPDATE  = 2,  // ekf_sym.cc:213 / ekf_sym.py:521
  FLAG_Q_DIAG             = 4,  // caller promises Q is diagonal (only its diagonal is read)
  FLAG_SHARED_R           = 8,  // R points at ONE [ZDIM, ZDIM] matrix used by every filter / observation
  FLAG_AUGMENT            = 16, // MSCKF: shift the clone window after the (last) update, in the same launch (ekf_sym.py:527-528 -> :365-391); CTA kernel only
};

// One argument block per launch, passed by value (lives in the kernel parameter
// constant bank: every field is warp-uniform).  NG = number of global_vars.
template <int NG>
struct StepArgs {
  double* x;             // [B, DIM]        in/out
  double* P;             // [B, EDIM, EDIM] in/out, row-major, symmetric
  const double* Q;       // [EDIM, EDIM]    batch-shared process noise (ekf_c.c:21,28)
  const double* dt_arr;  // [B] or nullptr -> use dt
  double dt;
  double* z;             // [B, n_obs, ZDIM] in/out: overwritten with the innovation y (ekf_c.c:120)
  const double* R;       // [B, n_obs, ZDIM, ZDIM]
  const double* ea;      // [B, n_obs, EADIM] or nullptr
  int n_obs;
  int ea_dim;            // doubles of extra args per observation (0 if unused)
  long long B;           // number of ENTRIES processed by this launch
  // optional gather list: entry e works on filter idx[e] of x / P / history, while z, R, ea, dt_arr stay
  // entry-indexed (compact).  nullptr = entry e is filter e.  Used by the ragged scheduler (per-tick kind buckets).
  const int* idx;
  int flags;
  int n_quat;
  int quat_idx[MAX_QUAT];
  // optional history slabs for the RTS smoother (ekf_sym.py:510,523): written when non-null
  double* hx_pred;       // [B, DIM]        x_{k|k-1}
  double* hP_pred;       // [B, EDIM, EDIM] P_{k|k-1}
  double* hx_filt;       // [B, DIM]        x_{k|k}
  double* hP_filt;       // [B, EDIM, EDIM] P_{k|k}
  double gv[NG > 0 ? NG : 1];
};

// ---------------------------------------------------------------------------
// Small symmetric solve used for S = H P H^T + R (ZDIM <= ~8 here).
// The reference uses Eigen fullPivLu (ekf_c.c:89,101); S is symmetric positive
// definite for any valid R, so an LDL^T factorisation (no square roots, Z
// reciprocals) gives the same solution to rounding.  Everything is unrolled at
// compile time so L/D live in registers.
// ---------------------------------------------------------------------------
template <int Z>
struct LDL {
  double L[Z][Z];   // unit lower (only i>j used)
  double D[Z];
  double Dinv[Z];

  __device__ __forceinline__ void factor(const double (&S)[Z][Z]) {
#pragma unroll
    for (int j = 0; j < Z; ++j) {
      double d = S[j][j];
#pragma unroll
      for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k] * D[k];
      D[j] = d;
      Dinv[j] = 1.0 / d;
#pragma unroll
      for (int i = j + 1; i < Z; ++i) {
        double s = S[i][j];
#pragma unroll
        for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k] * D[k];
        L[i][j] = s * Dinv[j];
      }
    }
  }
  // in-place solve S w = v
  __device__ __forceinline__ void solve(double (&v)[Z]) const {
#pragma unroll
    for (int i = 1; i < Z; ++i) {
#pragma unroll
      for (int k = 0; k < i; ++k) v[i] -= L[i][k] * v[k];
    }
#pragma unroll
    for (int i = 0; i < Z; ++i) v[i] *= Dinv[i];
#pragma unroll
    for (int i = Z - 2; i >= 0; --i) {
#pragma unroll
      for (int k = i + 1; k < Z; ++k) v[i] -= L[k][i] * v[k];
    }
  }
};

// Closed-form symmetric inverse for Z <= 3 (one reciprocal, cofactors computed independently: short dependency
// chain), LDL^T otherwise.  Same interface as LDL: factor(S), solve(v).  S is SPD with modest condition number
// (it is the innovation covariance H P H^T + R), so the adjugate is accurate to ~cond(S) * eps.
template <int Z>
struct SmallSym {
  LDL<Z> ldl;
  __device__ __forceinline__ void factor(const double (&S)[Z][Z]) { ldl.factor(S); }
  __device__ __forceinline__ void solve(double (&v)[Z]) const { ldl.solve(v); }
};
template <>
struct SmallSym<1> {
  double i00;
  __device__ __forceinline__ void factor(const double (&S)[1][1]) { i00 = 1.0 / S[0][0]; }
  __device__ __forceinline__ void solve(double (&v)[1]) const { v[0] *= i00; }
};
template <>
struct SmallSym<2> {
  double i00, i01, i11;
  __device__ __forceinline__ void factor(const double (&S)[2][2]) {
    const double r = 1.0 / fma(S[0][0], S[1][1], -S[0][1] * S[0][1]);
    i00 = S[1][1] * r; i01 = -S[0][1] * r; i11 = S[0][0] * r;
  }
  __device__ __forceinline__ void solve(double (&v)[2]) const {
    const double a = v[0], b = v[1];
    v[0] = fma(i00, a, i01 * b); v[1] = fma(i01, a, i11 * b);
  }
};
template <>
struct SmallSym<3> {
  double i00, i01, i02, i11, i12, i22;
  __device__ __forceinline__ void factor(const double (&S)[3][3]) {
    const double a = S[0][0], b = S[0][1], c = S[0][2], d = S[1][1], e = S[1][2], f = S[2][2];
    const double c00 = fma(d, f, -e * e), c01 = fma(c, e, -b * f), c02 = fma(b, e, -c * d);
    const double c11 = fma(a, f, -c * c), c12 = fma(b, c, -a * e), c22 = fma(a, d, -b * b);
    const double r = 1.0 / fma(a, c00, fma(b, c01, c * c02));
    i00 = c00 * r; i01 = c01 * r; i02 = c02 * r; i11 = c11 * r; i12 = c12 * r; i22 = c22 * r;
  }
  __device__ __forceinline__ void solve(double (&v)[3]) const {
    const double a = v[0], b = v[1], c = v[2];
    v[0] = fma(i00, a, fma(i01, b, i02 * c));
    v[1] = fma(i01, a, fma(i11, b, i12 * c));
    v[2] = fma(i02, a, fma(i12, b, i22 * c));
  }
};

#ifndef RNB_SMALLSYM
#define RNB_SMALLSYM 0   // 1 = closed-form adjugate inverse for Z <= 3: ~1 % faster, ~10x larger rounding error on ill-conditioned S; off
#endif
#if RNB_SMALLSYM
template <int Z> using SolverZ = SmallSym<Z>;
#else
template <int Z> using SolverZ = LDL<Z>;
#endif

// quaternion normalisation of x[idx..idx+4) -- division, like Eigen's normalize()
__device__ __forceinline__ void normalize4(double* q) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}

// ------------------------------------------------------------------ host ---
// C-ABI entry points return void (like the reference); failures are recorded
// here, printed, and surfaced by <name>_cuda_status() so bindings can raise.
inline int& last_status() { static int s = 0; return s; }

inline bool check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  last_status() = (int)e;
  fprintf(stderr, "[rednose_b200] CUDA failure in %s: %s\n", what, cudaGetErrorString(e));
  if (getenv("REDNOSE_B200_ABORT_ON_ERROR")) abort();
  return false;
}


// true exactly once per (device, kernel address): the caller then sets the kernel's shared-memory attributes, which
// are per device.  Entry points may be called from several host threads and for several devices in one process.
inline bool first_launch_of(const void* kern) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> configured;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(mu);
  return configured.insert({dev, kern}).second;
}

// stream-ordered scratch (cudaMallocAsync).  The default memory pool gives its memory back to the OS at every
// synchronisation; raising the release threshold once per device keeps it, so a per-call workspace costs microseconds.
inline void* stream_alloc(size_t bytes, cudaStream_t st, const char* what) {
  static std::mutex mu;
  static std::set<int> tuned;
  int dev = 0;
  cudaGetDevice(&dev);
  {
    std::lock_guard<std::mutex> lk(mu);
    if (tuned.insert(dev).second) {
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      }
    }
  }
  void* p = nullptr;
  if (!check(cudaMallocAsync(&p, bytes, st), what)) return nullptr;
  return p;
}

}  // namespace rnb
