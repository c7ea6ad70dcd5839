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

constexpr int MAX_QUAT = 16;   // the MSCKF normalises 11 (main state + 10 clones)

// runtime flags of a batched step
enum : int {
  FLAG_NORM_AFTER_PREDICT = 1,  // ekf_sym.cc:207 (the C++ driver does, the python driver does not)
  FLAG_NORM_AFTER_UPDATE  = 2,  // ekf_sym.cc:213 / ekf_sym.py:521
  FLAG_Q_DIAG             = 4,  // caller promises Q is diagonal (only its diagonal is read)
  FLAG_SHARED_R           = 8,  // R points at ONE [ZDIM, ZDIM] matrix used by every filter / observation
  FLAG_AUGMENT            = 16, // MSCKF: shift the clone window after the (last) update, in the same launch (ekf_sym.py:527-528 -> :365-391); CTA kernel only
  FLAG_PACKED_P           = 32, // P is [B, packed_doubles(EDIM)] in the packed lower-block-triangle layout (ekf_packed.cuh); pair kernel only
  FLAG_PACKED_HIST        = 64, // hP_pred / hP_filt hold packed_doubles(EDIM) per filter in that layout; pair kernel only
  FLAG_MAIN_HIST          = 128,// hP_pred holds the MEDIM x MEDIM main block per filter, hP_pred_last the full newest P_{k+1|k};
                                // set by the <name>_batch_mainhist_step_<kind> entry points, CTA kernel (EDIM > 32) only
};

// A filter model whose covariance HISTORY slabs are packed (FLAG_PACKED_HIST, ekf_packed.cuh).  The kernels that record
// and smooth histories are instantiated with PackedHist<M> in place of M, so that the instantiations without packed
// history keep their symbols and their machine code.
template <class M>
struct PackedHist : M {
  static constexpr bool PACKED_HIST = true;
};
template <class M, class = void>
struct PackedHistOf { static constexpr bool value = false; };
template <class M>
struct PackedHistOf<M, decltype(void(M::PACKED_HIST))> { static constexpr bool value = M::PACKED_HIST; };
template <class M>
constexpr bool packed_hist() { return PackedHistOf<M>::value; }

// A filter model (EDIM > 32) whose PREDICTED covariance history keeps only the MEDIM x MEDIM main block per step
// (FLAG_MAIN_HIST): the RTS recursion reads nothing else of P_{k+1|k} (ekf_sym.py:677-686).  The full newest prediction,
// which the smoother copies to its last output row, goes to a separate [B, EDIM, EDIM] buffer.  Instantiated in place
// of M, like PackedHist, so the full-layout kernels keep their symbols and machine code.
template <class M>
struct MainHist : M {
  static constexpr bool MAIN_HIST = true;
};
template <class M, class = void>
struct MainHistOf { static constexpr bool value = false; };
template <class M>
struct MainHistOf<M, decltype(void(M::MAIN_HIST))> { static constexpr bool value = M::MAIN_HIST; };
template <class M>
constexpr bool main_hist() { return MainHistOf<M>::value; }

// A filter model (EDIM <= 32) whose ragged history holds one SEGMENT of each filter's rows (RtsArgs::term / k0s): the
// ragged smoothers are instantiated with RaggedSeg<M> (or RaggedSeg<PackedHist<M>>) in place of M, like PackedHist, so
// the whole-history instantiations keep their symbols and machine code.
template <class M>
struct RaggedSeg : M {
  static constexpr bool RAGGED_SEG = true;
};
template <class M, class = void>
struct RaggedSegOf { static constexpr bool value = false; };
template <class M>
struct RaggedSegOf<M, decltype(void(M::RAGGED_SEG))> { static constexpr bool value = M::RAGGED_SEG; };
template <class M>
constexpr bool ragged_seg() { return RaggedSegOf<M>::value; }

// One argument block per launch, passed by value (lives in the kernel parameter
// constant bank: every field is warp-uniform).  NG = number of global_vars.
template <int NG>
struct StepArgs {
  double* x;             // [B, DIM]        in/out
  double* P;             // [B, EDIM, EDIM] in/out, row-major, symmetric (lower triangle read); [B, packed_doubles(EDIM)] with FLAG_PACKED_P
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
  double* hP_pred;       // [B, EDIM, EDIM] P_{k|k-1}; [B, packed_doubles(EDIM)] with FLAG_PACKED_HIST
  double* hx_filt;       // [B, DIM]        x_{k|k}
  double* hP_filt;       // [B, EDIM, EDIM] P_{k|k}; [B, packed_doubles(EDIM)] with FLAG_PACKED_HIST
  double gv[NG > 0 ? NG : 1];
  // ragged histories (gather list only): entry e records at slab element hist_row[e] * hist_B + idx[e] instead of
  // idx[e]; a negative row steps without recording.  nullptr = the slabs are indexed by filter.  Kept behind the
  // existing fields so that the launches without a gather list see the argument block they always had.
  // FLAG_MAIN_HIST, which is refused with a gather list, uses the same slot for hP_pred_last: [B, EDIM, EDIM], the full
  // P_{k+1|k} of this step (hP_pred is then [B, MEDIM, MEDIM]).  Sharing it keeps the block's size, and so the offsets
  // of the kernel parameters behind it, unchanged.
  union {
    const int* hist_row;
    double* hP_pred_last;
  };
  long long hist_B;      // filter stride of the history slabs
};

// slab element entry e of a gather list records at (-1: nothing recorded)
template <int NG>
__device__ __forceinline__ long long hist_slot(const StepArgs<NG>& a, long long e, long long fid) {
  if (!a.hist_row) return fid;
  const int r = a.hist_row[e];
  return r < 0 ? -1 : (long long)r * a.hist_B + fid;
}

// ---------------------------------------------------------------------------
// Small symmetric solve used for S = H P H^T + R (ZDIM <= ~8 here).
// The reference uses Eigen fullPivLu (ekf_c.c:89,101); S is symmetric positive
// definite for any valid R, so an LDL^T factorisation (no square roots, Z
// reciprocals) gives the same solution to rounding.  Everything is unrolled at
// compile time so L/D live in registers.  A closed-form adjugate inverse for
// Z <= 3 was about 1 % faster but has about 10x the rounding error on
// ill-conditioned S.
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

// Runs an entry point and returns the cudaError_t it latched (0 = ok).  A status latched before the call is kept when the
// call succeeds, so <name>_cuda_status() still reports it.
template <class F>
inline int call_status(F&& f) {
  const int before = last_status();
  last_status() = 0;
  f();
  const int st = last_status();
  if (st == 0) last_status() = before;
  return st;
}

// The quaternion index list is copied into every launch's argument block and dereferenced in shared memory by the
// kernels, so it is validated on the host before anything is launched: 0 <= n_quat <= MAX_QUAT and every
// quaternion [idx, idx + 4) inside the DIM-long state.  On failure nothing runs and the status is cudaErrorInvalidValue.
inline bool check_quat_idxs(const int* quat_idxs, int n_quat, int dim) {
  if (n_quat < 0 || n_quat > MAX_QUAT || (n_quat > 0 && !quat_idxs)) {
    fprintf(stderr, "[rednose_b200] n_quat = %d: at most %d quaternion indices are supported\n", n_quat, MAX_QUAT);
    last_status() = (int)cudaErrorInvalidValue;
    return false;
  }
  for (int i = 0; i < n_quat; ++i) {
    if (quat_idxs[i] < 0 || quat_idxs[i] > dim - 4) {
      fprintf(stderr, "[rednose_b200] quaternion index %d does not fit a state of %d entries\n", quat_idxs[i], dim);
      last_status() = (int)cudaErrorInvalidValue;
      return false;
    }
  }
  return true;
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
