// rednose_b200 -- host-side templates behind the generated C-ABI of one filter library.
//
// The generated lib<name>.so exports (a) the reference's own symbol set
// (rednose/helpers/ekf_sym.py:149-171: <name>_predict, <name>_update_<kind>, leaf
// functions, <name>_set_<var>) operating on HOST pointers for ONE filter, and (b)
// batched additions (<name>_batch_*) operating on DEVICE pointers.  Both run the same
// CUDA kernels; there is no CPU implementation in this library.
#pragma once
#include "ekf_common.cuh"
#include "ekf_thread.cuh"
#include "ekf_warp2.cuh"
#include "ekf_cta.cuh"
#include "ekf_rts.cuh"
#include "ekf_rts_mma.cuh"
#include "ekf_augment.cuh"
#include <cstring>
#include <mutex>
#include <type_traits>
#include <unordered_set>

namespace rnb {

// placeholder kind for predict-only instantiations
struct NullKind {
  static constexpr int KIND = -1, ZDIM = 1, YDIM = 1, EADIM = 0, NH = 0;
  static constexpr bool MAHA = false, HAS_HE = false;
  static constexpr double MAHA_THRESH = 0.0;
  template <class HV> static __device__ __forceinline__ void obs_leaf(const double*, const double*, const double*, double (&)[1], HV&) {}
  template <class HV, class V> static __device__ __forceinline__ void Herr_apply(const HV&, const V&, double (&hp)[1]) { hp[0] = 0.0; }
  template <class HV, class A> static __device__ __forceinline__ void S_accum(const HV&, A, double (&)[1][1]) {}
};

template <int NG>
struct GV { double v[NG > 0 ? NG : 1]; };

// Per-library host context: global_vars (ekf_sym.py:129-132 keeps them as file
// statics; here they are copied into every launch's argument block) and a small
// device scratch used by the single-filter host-pointer entry points.
constexpr int MAX_DEVICES = 32;
inline int current_device() { int d = 0; cudaGetDevice(&d); return (d >= 0 && d < MAX_DEVICES) ? d : 0; }

template <class M>
struct HostCtx {
  GV<M::NG> gv{};
  std::mutex mu;
  // device scratch / pinned staging / private stream of the single-filter entry points, ONE SET PER DEVICE (a process may
  // drive several GPUs; a pointer or stream created on device 0 must never be used while device 1 is current)
  struct PerDevice {
    double* d_scratch = nullptr;
    size_t scratch_doubles = 0;
    double* h_pinned = nullptr;      // pinned host staging: one copy in, one copy out
    size_t pinned_doubles = 0;
    cudaStream_t stream = nullptr;
  };
  PerDevice dev[MAX_DEVICES];

  double* scratch(size_t n) {
    PerDevice& p = dev[current_device()];
    if (n > p.scratch_doubles) {
      if (p.d_scratch) cudaFree(p.d_scratch);
      p.d_scratch = nullptr; p.scratch_doubles = 0;
      if (!check(cudaMalloc(&p.d_scratch, n * sizeof(double)), "cudaMalloc(scratch)")) return nullptr;
      p.scratch_doubles = n;
    }
    return p.d_scratch;
  }
  double* pinned(size_t n) {
    PerDevice& p = dev[current_device()];
    if (n > p.pinned_doubles) {
      if (p.h_pinned) cudaFreeHost(p.h_pinned);
      p.h_pinned = nullptr; p.pinned_doubles = 0;
      if (!check(cudaMallocHost((void**)&p.h_pinned, n * sizeof(double)), "cudaMallocHost(staging)")) return nullptr;
      p.pinned_doubles = n;
    }
    return p.h_pinned;
  }
  cudaStream_t single_stream() {
    PerDevice& p = dev[current_device()];
    if (!p.stream) check(cudaStreamCreateWithFlags(&p.stream, cudaStreamNonBlocking), "cudaStreamCreate(single)");
    return p.stream;
  }
};

constexpr int THREAD_MAX_EDIM = 6;

// true when the steps of filter M serve its covariance with the pair kernel (ekf_warp2.cuh), the only kernel that reads
// and writes the packed layout.  A filter with a feature-track kind is never served whole by the pair kernel (its feature
// kinds run on the CTA kernel, which reads the full layout), so its P stays full
template <class M>
constexpr bool pair_may_serve() { return M::EDIM > THREAD_MAX_EDIM && use_pair<M>() && !M::HAS_FEATURE_KIND; }

// doubles per filter of the packed covariance layout, 0 when the pair kernel does not serve this filter
template <class M>
constexpr int packed_P_doubles() { return pair_may_serve<M>() ? packed_doubles(M::EDIM) : 0; }

// FLAG_PACKED_P or FLAG_PACKED_HIST on a launch that the pair kernel would not run: rejected before any CUDA call
template <class M, bool FEATURE_KIND>
inline bool check_packed_flag(int flags, const char* what) {
  if (!(flags & (FLAG_PACKED_P | FLAG_PACKED_HIST)) || (!FEATURE_KIND && pair_may_serve<M>())) return true;
  fprintf(stderr, "[rednose_b200] %s: the packed covariance layout (%s) exists only for the two-filters-per-warp kernel "
                  "(even EDIM <= 32, no feature kinds)\n", what,
          (flags & FLAG_PACKED_P) ? "P" : "history slabs");
  last_status() = (int)cudaErrorNotSupported;
  return false;
}

// FLAG_MAIN_HIST exists for the fused step of a filter above EDIM 32 (the CTA-per-filter kernel), without a gather list
// and in the full covariance layout: anything else is rejected before any CUDA call
template <class M, bool FUSED>
inline bool check_main_hist_flag(const StepArgs<M::NG>& a, const char* what) {
  if (!(a.flags & FLAG_MAIN_HIST)) return true;
  const char* why = nullptr;
  if (M::EDIM <= 32) why = "exists only above EDIM 32";
  else if (!FUSED) why = "is recorded by the fused predict + update step only";
  else if (a.flags & (FLAG_PACKED_P | FLAG_PACKED_HIST)) why = "cannot be combined with the packed covariance layouts";
  else if (a.idx) why = "cannot be combined with a gather list";   // history rows (hist_row) come only with one
  if (!why) return true;
  fprintf(stderr, "[rednose_b200] %s: the main-block prediction history %s\n", what, why);
  last_status() = (int)cudaErrorNotSupported;
  return false;
}

template <class M, class K, bool PRED, bool UPD>
inline void launch_step(const StepArgs<M::NG>& a, cudaStream_t st) {
  if (!check_packed_flag<M, K::HAS_HE>(a.flags, "ekf_step")) return;
  if (!check_main_hist_flag<M, PRED && UPD>(a, "ekf_step")) return;
  if (a.B <= 0) return;
  if ((a.flags & FLAG_AUGMENT) && !(M::EDIM > 32 || K::HAS_HE)) {
    fprintf(stderr, "[rednose_b200] the fused augment exists only in the CTA-per-filter kernel (EDIM > 32): call <name>_batch_augment\n");
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  // feature-track kinds (left-null-space projection with He, ekf_c.c:66-76) exist only in the CTA kernel: they go there
  // whatever the state size
  // per-entry history rows come only with the fused gather step (batch_step_hist): the thread and CTA kernels take them
  // through their own instantiation, the warp kernels on their gather path
  constexpr bool FUSED = PRED && UPD;
  if constexpr (M::EDIM <= THREAD_MAX_EDIM && !K::HAS_HE) {
    const unsigned grid = (unsigned)((a.B + 127) / 128);
    if constexpr (FUSED) {
      if (a.hist_row) ekf_step_thread<M, K, PRED, UPD, true><<<grid, 128, 0, st>>>(a);
      else ekf_step_thread<M, K, PRED, UPD><<<grid, 128, 0, st>>>(a);
    } else {
      ekf_step_thread<M, K, PRED, UPD><<<grid, 128, 0, st>>>(a);
    }
  } else if constexpr (M::EDIM <= 32 && !K::HAS_HE) {
    if constexpr (use_pair<M>()) {
      // two filters per warp (ekf_warp2.cuh): 128-bit accesses to every covariance array
      if (reinterpret_cast<uintptr_t>(a.P) & 15u) {
        fprintf(stderr, "[rednose_b200] P must be 16-byte aligned (bulk-copy staging of covariance tiles)\n");
        last_status() = (int)cudaErrorMisalignedAddress;
        return;
      }
      if ((reinterpret_cast<uintptr_t>(a.hP_pred) | reinterpret_cast<uintptr_t>(a.hP_filt)) & 15u) {
        fprintf(stderr, "[rednose_b200] covariance history slabs must be 16-byte aligned\n");
        last_status() = (int)cudaErrorMisalignedAddress;
        return;
      }
      constexpr int G = PAIR_GROUP;
      const bool packed = a.flags & FLAG_PACKED_P, phist = a.flags & FLAG_PACKED_HIST;
      const size_t smem = packed ? pair_smem_bytes<M, K, G, true>() : pair_smem_bytes<M, K, G, false>();
      const unsigned grid = (unsigned)((a.B + G - 1) / G);
      auto run = [&](void (*kern)(const StepArgs<M::NG>)) {
        if (first_launch_of((const void*)kern)) {
          cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
          cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
        kern<<<grid, 32, smem, st>>>(a);
      };
      // the packed-history kernels (FLAG_PACKED_HIST) of gather list GA, for either layout of P; instantiated only for the
      // filters the pair kernel may serve (check_packed_flag refused the flag for the others)
      auto phist_kernel = [&](auto ga) -> void (*)(const StepArgs<M::NG>) {
        constexpr bool GA = decltype(ga)::value;
        using MH = PackedHist<M>;
        if constexpr (pair_may_serve<M>())
          return packed ? ekf_step_pair<MH, K, PRED, UPD, G, GA, true> : ekf_step_pair<MH, K, PRED, UPD, G, GA, false>;
        else return nullptr;
      };
      if constexpr (PRED && UPD) {
        if (phist) run(a.idx ? phist_kernel(std::true_type{}) : phist_kernel(std::false_type{}));
        else if (a.idx) run(packed ? ekf_step_pair<M, K, PRED, UPD, G, true, true> : ekf_step_pair<M, K, PRED, UPD, G, true, false>);
        else run(packed ? ekf_step_pair<M, K, PRED, UPD, G, false, true> : ekf_step_pair<M, K, PRED, UPD, G, false, false>);
      } else {
        if (a.idx) {
          fprintf(stderr, "[rednose_b200] gather lists are only supported by the fused predict+update step\n");
          last_status() = (int)cudaErrorNotSupported;
          return;
        }
        if (phist) run(phist_kernel(std::false_type{}));
        else run(packed ? ekf_step_pair<M, K, PRED, UPD, G, false, true> : ekf_step_pair<M, K, PRED, UPD, G, false, false>);
      }
    } else {
      constexpr int G = WARP_GROUP, W = WARP_CTA_WARPS;
      constexpr size_t smem = warp_smem_bytes<M, K, G, W>();
      const long long per_cta = (long long)G * W;
      const unsigned grid = (unsigned)((a.B + per_cta - 1) / per_cta);
      auto run = [&](void (*kern)(const StepArgs<M::NG>)) {
        if (first_launch_of((const void*)kern)) {
          cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
          cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
        kern<<<grid, W * 32, smem, st>>>(a);
      };
      if constexpr (PRED && UPD) {
        // the gather-list variant exists only for the fused step (what the ragged scheduler issues)
        if (a.idx) run(ekf_step_warp<M, K, PRED, UPD, G, W, true>);
        else run(ekf_step_warp<M, K, PRED, UPD, G, W, false>);
      } else {
        if (a.idx) {
          fprintf(stderr, "[rednose_b200] gather lists are only supported by the fused predict+update step\n");
          last_status() = (int)cudaErrorNotSupported;
          return;
        }
        run(ekf_step_warp<M, K, PRED, UPD, G, W, false>);
      }
    }
  } else {
    if constexpr (FUSED) {
      bool main_hist = false;   // checked first: hP_pred_last shares hist_row's slot
      if constexpr (M::EDIM > 32) main_hist = a.flags & FLAG_MAIN_HIST;
      if (main_hist) {
        if constexpr (M::EDIM > 32) launch_step_cta<M, K, PRED, UPD, false, true>(a, st);
      } else if (a.hist_row) launch_step_cta<M, K, PRED, UPD, true>(a, st);
      else launch_step_cta<M, K, PRED, UPD>(a, st);
    } else {
      launch_step_cta<M, K, PRED, UPD>(a, st);
    }
  }
  check(cudaGetLastError(), "ekf_step launch");
}

// false (and nothing filled) when the quaternion list is invalid: the caller launches nothing
template <class M>
inline bool fill_common(StepArgs<M::NG>& a, HostCtx<M>& ctx, long long B, const int* quat_idxs, int n_quat, int flags) {
  if (!check_quat_idxs(quat_idxs, n_quat, M::DIM)) return false;
  memset(&a, 0, sizeof(a));
  a.B = B;
  a.flags = flags;
  a.n_quat = n_quat;
  for (int i = 0; i < n_quat; ++i) a.quat_idx[i] = quat_idxs[i];
  for (int i = 0; i < (M::NG > 0 ? M::NG : 1); ++i) a.gv[i] = ctx.gv.v[i];
  a.n_obs = 1;
  return true;
}

// ----------------------------------------------------------- batched (device) ---
template <class M>
inline void batch_predict(HostCtx<M>& ctx, double* x, double* P, const double* Q, const double* dt_arr, double dt,
                          long long B, const int* quat_idxs, int n_quat, int flags,
                          double* hx_pred, double* hP_pred, void* stream) {
  StepArgs<M::NG> a;
  if (!fill_common<M>(a, ctx, B, quat_idxs, n_quat, flags)) return;
  a.x = x; a.P = P; a.Q = Q; a.dt_arr = dt_arr; a.dt = dt;
  a.hx_pred = hx_pred; a.hP_pred = hP_pred;
  launch_step<M, NullKind, true, false>(a, (cudaStream_t)stream);
}

template <class M, class K, bool PRED>
inline void batch_step(HostCtx<M>& ctx, double* x, double* P, const double* Q, const double* dt_arr, double dt,
                       double* z, const double* R, const double* ea, int n_obs, long long B,
                       const int* quat_idxs, int n_quat, int flags,
                       double* hx_pred, double* hP_pred, double* hx_filt, double* hP_filt, void* stream,
                       const int* idx = nullptr, const int* hist_row = nullptr, long long hist_B = 0,
                       double* hP_pred_last = nullptr) {
  StepArgs<M::NG> a;
  if (!fill_common<M>(a, ctx, B, quat_idxs, n_quat, flags)) return;
  a.idx = idx;
  a.hist_row = hist_row; a.hist_B = hist_B;
  if (hP_pred_last) a.hP_pred_last = hP_pred_last;   // shares hist_row's slot (StepArgs); the main-block step has no rows
  a.x = x; a.P = P; a.Q = Q; a.dt_arr = dt_arr; a.dt = dt;
  a.z = z; a.R = R; a.ea = (K::EADIM > 0) ? ea : nullptr; a.ea_dim = K::EADIM; a.n_obs = n_obs;
  a.hx_pred = hx_pred; a.hP_pred = hP_pred; a.hx_filt = hx_filt; a.hP_filt = hP_filt;
  launch_step<M, K, PRED, true>(a, (cudaStream_t)stream);
}

// fused gather step that records entry e at row hist_row[e] of [T, hist_B, ...] history slabs (ragged histories)
template <class M, class K>
inline void batch_step_hist(HostCtx<M>& ctx, double* x, double* P, const double* Q, const double* dt_arr, double dt,
                            double* z, const double* R, const double* ea, int n_obs, long long B,
                            const int* quat_idxs, int n_quat, int flags,
                            double* hx_pred, double* hP_pred, double* hx_filt, double* hP_filt,
                            const int* idx, const int* hist_row, long long hist_B, void* stream) {
  if (!idx || !hist_row || hist_B <= 0) {
    fprintf(stderr, "[rednose_b200] batch_step_hist: a gather list, its history rows and a positive slab stride are required\n");
    last_status() = (int)cudaErrorInvalidValue;
    return;
  }
  batch_step<M, K, true>(ctx, x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags,
                         hx_pred, hP_pred, hx_filt, hP_filt, stream, idx, hist_row, hist_B);
}

// fused step that records one row of a main-block prediction history (FLAG_MAIN_HIST): hP_pred [B, MEDIM, MEDIM] gets
// the main block of P_{k+1|k}, hP_pred_last [B, EDIM, EDIM] the whole of it
template <class M, class K>
inline void batch_step_mainhist(HostCtx<M>& ctx, double* x, double* P, const double* Q, const double* dt_arr, double dt,
                                double* z, const double* R, const double* ea, int n_obs, long long B,
                                const int* quat_idxs, int n_quat, int flags,
                                double* hx_pred, double* hP_pred, double* hx_filt, double* hP_filt, double* hP_pred_last,
                                void* stream) {
  batch_step<M, K, true>(ctx, x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags | FLAG_MAIN_HIST,
                         hx_pred, hP_pred, hx_filt, hP_filt, stream, nullptr, nullptr, 0, hP_pred_last);
}

}  // namespace rnb
#include "ekf_maha.cuh"
namespace rnb {

// Mahalanobis distances of B observations of one kind (ekf_sym.py:626-649); out [B] on the device
template <class M, class K>
inline void batch_maha(HostCtx<M>& ctx, const double* x, const double* P, const double* z, const double* R, const double* ea,
                       long long B, int flags, double* out, void* stream) {
  if (!check_packed_flag<M, false>(flags, "batch_maha")) return;
  if (B <= 0) return;
  // per-call scratch, allocated and released in stream order (no buffer shared between streams or devices)
  double* scratch = (double*)stream_alloc(sizeof(double) * (size_t)B * K::ZDIM * M::EDIM, (cudaStream_t)stream, "cudaMallocAsync(maha scratch)");
  if (!scratch) return;
  ekf_maha_thread<M, K><<<(unsigned)((B + 127) / 128), 128, 0, (cudaStream_t)stream>>>(x, P, z, R, ea, B, flags, ctx.gv, out, scratch);
  check(cudaGetLastError(), "ekf_maha launch");
  check(cudaFreeAsync(scratch, (cudaStream_t)stream), "cudaFreeAsync(maha scratch)");
}

// PH: the covariance slabs (hP_pred, hP_filt, Ps and P_term) are packed; only where the pair kernel records them so
template <class M, bool PH>
inline bool check_packed_hist(const char* what) {
  if constexpr (PH) return check_packed_flag<M, false>(FLAG_PACKED_HIST, what);
  else return true;
}

// MH: a main-block prediction history (FLAG_MAIN_HIST, EDIM > 32): hP_pred is [T, B, MEDIM, MEDIM] and, without a
// terminal estimate, the recursion starts from hP_pred_last [B, EDIM, EDIM], the full prediction of the newest row
template <class M, bool PH = false, bool MH = false>
inline void batch_rts(HostCtx<M>& ctx, const double* hx_pred, const double* hP_pred, const double* hx_filt, const double* hP_filt,
                      const double* t, int t_per_filter, double* xs, double* Ps, int T, long long B,
                      const int* quat_idxs, int n_quat, int norm_quats, void* stream,
                      const double* x_term = nullptr, const double* P_term = nullptr, long long k0 = 0,
                      const double* hP_pred_last = nullptr) {
  static_assert(!(PH && MH), "main-block prediction histories are in the full layout");
  if (!check_packed_hist<M, PH>("batch_rts_packed")) return;
  if constexpr (MH && M::EDIM <= 32) {
    fprintf(stderr, "[rednose_b200] batch_rts_mainhist: main-block prediction histories exist only above EDIM 32\n");
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  if (!check_quat_idxs(quat_idxs, n_quat, M::DIM)) return;
  if (MH && B > 0 && !(x_term && P_term) && !hP_pred_last) {
    fprintf(stderr, "[rednose_b200] batch_rts_mainhist: without a terminal estimate the newest full prediction (hP_pred_last) is required\n");
    last_status() = (int)cudaErrorInvalidValue;
    return;
  }
  RtsArgs<M::NG> a;
  memset(&a, 0, sizeof(a));
  a.x_term = (x_term && P_term) ? x_term : nullptr; a.P_term = (x_term && P_term) ? P_term : nullptr; a.k0 = k0;
  a.hP_pred_last = MH ? hP_pred_last : nullptr;
  a.hx_pred = hx_pred; a.hP_pred = hP_pred; a.hx_filt = hx_filt; a.hP_filt = hP_filt;
  a.t = t; a.t_per_filter = t_per_filter; a.xs = xs; a.Ps = Ps; a.T = T; a.B = B; a.norm_quats = norm_quats;
  a.n_quat = n_quat;
  for (int i = 0; i < n_quat; ++i) a.quat_idx[i] = quat_idxs[i];
  for (int i = 0; i < (M::NG > 0 ? M::NG : 1); ++i) a.gv[i] = ctx.gv.v[i];
  if constexpr (PH && !pair_may_serve<M>()) return;   // refused above
  else {
    if constexpr (M::EDIM > 32) {
      // above 32 the kernels write only the main block of Ps[0 .. T-2]; everything else there is P_{k|k}: nothing to do in
      // place, one copy of those rows of hP_filt otherwise (row T-1 the kernel writes in full, or not at all for a segment)
      if (B > 0 && T >= 2 && Ps != hP_filt &&
          !check(cudaMemcpyAsync(Ps, hP_filt, sizeof(double) * (size_t)(T - 1) * (size_t)B * M::EDIM * M::EDIM,
                                 cudaMemcpyDeviceToDevice, (cudaStream_t)stream), "cudaMemcpyAsync(RTS P_{k|k})"))
        return;
    }
    if constexpr (!MH) launch_rts_auto<M, PH>(a, (cudaStream_t)stream);
    else if constexpr (M::EDIM > 32) launch_rts_auto<MainHist<M>>(a, (cudaStream_t)stream);   // refused above otherwise
  }
}

// RTS over a ragged history: filter b smooths rows 0 .. len[b] - 1 of [T, B, ...] slabs with its own times t [T, B]
template <class M, bool PH = false>
inline void batch_rts_ragged(HostCtx<M>& ctx, const double* hx_pred, const double* hP_pred, const double* hx_filt, const double* hP_filt,
                             const double* t, const int* len, double* xs, double* Ps, int T, long long B,
                             const int* quat_idxs, int n_quat, int norm_quats, void* stream) {
  if (!check_packed_hist<M, PH>("batch_rts_ragged_packed")) return;
  if (M::EDIM > 32) {
    fprintf(stderr, "[rednose_b200] batched RTS for EDIM=%d > 32 is not built into this library\n", M::EDIM);
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  if (!t || !len || T <= 0) {
    fprintf(stderr, "[rednose_b200] batch_rts_ragged: per-filter times, per-filter lengths and T >= 1 are required\n");
    last_status() = (int)cudaErrorInvalidValue;
    return;
  }
  if (!check_quat_idxs(quat_idxs, n_quat, M::DIM)) return;
  RtsArgs<M::NG> a;
  memset(&a, 0, sizeof(a));
  a.hx_pred = hx_pred; a.hP_pred = hP_pred; a.hx_filt = hx_filt; a.hP_filt = hP_filt;
  a.t = t; a.t_per_filter = 1; a.len = len; a.xs = xs; a.Ps = Ps; a.T = T; a.B = B; a.norm_quats = norm_quats;
  a.n_quat = n_quat;
  for (int i = 0; i < n_quat; ++i) a.quat_idx[i] = quat_idxs[i];
  for (int i = 0; i < (M::NG > 0 ? M::NG : 1); ++i) a.gv[i] = ctx.gv.v[i];
  if constexpr (PH && !pair_may_serve<M>()) return;   // refused above
  else launch_rts_auto<M, PH>(a, (cudaStream_t)stream);
}

// RTS over one SEGMENT of a ragged history: filter b smooths rows 0 .. len[b] - 1, the global rows k0[b] .. of its
// stream; with term[b] != 0 row len[b] - 1 is the first row of the filter's segment behind (only its predicted state and
// time are read) and the recursion starts from x_term[b] / P_term[b], that row's smoothed estimate.  packed: every
// covariance slab, P_term included, is in the packed layout
template <class M>
inline void batch_rts_ragged_segment(HostCtx<M>& ctx, const double* hx_pred, const double* hP_pred, const double* hx_filt,
                                     const double* hP_filt, const double* t, const int* len, const unsigned char* term,
                                     const long long* k0, const double* x_term, const double* P_term, double* xs, double* Ps,
                                     int T, long long B, const int* quat_idxs, int n_quat, int norm_quats, int packed,
                                     void* stream) {
  if (packed && !check_packed_hist<M, true>("batch_rts_ragged_segment")) return;
  if constexpr (M::EDIM > 32) {
    fprintf(stderr, "[rednose_b200] batch_rts_ragged_segment: ragged histories exist only up to EDIM 32 (EDIM = %d)\n", M::EDIM);
    last_status() = (int)cudaErrorNotSupported;
  } else {
    if (B < 0 || (B > 0 && (!t || !len || !term || !k0 || !x_term || !P_term || T <= 0))) {
      fprintf(stderr, "[rednose_b200] batch_rts_ragged_segment: B >= 0 and, for B > 0, per-filter times, lengths, terminal "
                      "flags, first rows, terminal estimates and T >= 1 are required\n");
      last_status() = (int)cudaErrorInvalidValue;
      return;
    }
    if (!check_quat_idxs(quat_idxs, n_quat, M::DIM)) return;
    RtsArgs<M::NG> a;
    memset(&a, 0, sizeof(a));
    a.hx_pred = hx_pred; a.hP_pred = hP_pred; a.hx_filt = hx_filt; a.hP_filt = hP_filt;
    a.t = t; a.t_per_filter = 1; a.len = len; a.term = term; a.k0s = k0; a.x_term = x_term; a.P_term = P_term;
    a.xs = xs; a.Ps = Ps; a.T = T; a.B = B; a.norm_quats = norm_quats;
    a.n_quat = n_quat;
    for (int i = 0; i < n_quat; ++i) a.quat_idx[i] = quat_idxs[i];
    for (int i = 0; i < (M::NG > 0 ? M::NG : 1); ++i) a.gv[i] = ctx.gv.v[i];
    if (!packed) launch_rts_ragged_segment<M, false>(a, (cudaStream_t)stream);
    else if constexpr (pair_may_serve<M>()) launch_rts_ragged_segment<M, true>(a, (cudaStream_t)stream);   // refused above otherwise
  }
}

// ------------------------------------------------------ covariance layout conversion ---
// Entry e of the compact full-layout buffer `full` [n, EDIM, EDIM] <-> filter idx[e] (e without a list) of the packed
// batch `packed` [*, packed_doubles(EDIM)].  Packing reads only the lower triangle; unpacking writes its exact mirror.
template <int E>
__global__ void __launch_bounds__(256) convert_P_kernel(double* __restrict__ full, double* __restrict__ packed, const int* __restrict__ idx,
                                                        long long n, int to_packed) {
  constexpr int PD = packed_doubles(E);
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * (E * E)) return;
  const long long e = t / (E * E);
  const int r = (int)(t - e * (E * E)), i = r / E, j = r - i * E;
  double* pk = packed + (idx ? (long long)idx[e] : e) * PD;
  if (to_packed) {
    // every slot of the lower block triangle once, the diagonal blocks' upper slot from its lower mirror
    if ((i >> 1) >= (j >> 1)) pk[packed_block(i >> 1, j >> 1) + 2 * (i & 1) + (j & 1)] = full[e * (E * E) + (i >= j ? i * E + j : j * E + i)];
  } else {
    full[t] = pk[packed_index(i, j)];
  }
}

template <class M>
inline int convert_P(double* full, double* packed, const int* idx, long long n, int to_packed, void* stream) {
  constexpr int E = M::EDIM;
  if constexpr (E % 2 == 0 && E <= 32) {
    if (n <= 0) return 0;
    const long long threads = n * (E * E);
    convert_P_kernel<E><<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(full, packed, idx, n, to_packed);
    const cudaError_t err = cudaGetLastError();
    check(err, "convert_P launch");
    return (int)err;
  } else {
    fprintf(stderr, "[rednose_b200] convert_P: no packed covariance layout for EDIM = %d\n", E);
    last_status() = (int)cudaErrorNotSupported;
    return (int)cudaErrorNotSupported;
  }
}

// ------------------------------------------------------ restore filters from history rows ---
// Filter idx[e] of the resident x [*, D] / P <- slab element hist_row[e] * hist_B + idx[e] of hx_filt / hP_filt (the
// addressing of the recording steps, hist_slot); an entry with a negative row is skipped.  PH: the history covariances
// are packed, PP: the resident P is.  One thread per destination double.  Across layouts the copy is the one convert_P
// makes: into the packed layout from the lower triangle, out of it as the exact mirror.
template <int D, int E, bool PH, bool PP>
__global__ void __launch_bounds__(256) restore_hist_kernel(const double* __restrict__ hx, const double* __restrict__ hP,
                                                           const int* __restrict__ idx, const int* __restrict__ hist_row,
                                                           long long n, long long hist_B, double* __restrict__ x, double* __restrict__ P) {
  constexpr int SH = PH ? packed_doubles(E) : E * E, SP = PP ? packed_doubles(E) : E * E, W = D + SP;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * W) return;
  const long long e = t / W;
  const int r = hist_row[e];
  if (r < 0) return;
  const long long f = idx[e], s = (long long)r * hist_B + f;
  const int c = (int)(t - e * W);
  if (c < D) {
    x[f * D + c] = hx[s * D + c];
    return;
  }
  const int k = c - D;
  int src = k;
  if constexpr (PP && !PH) {
    int i, j;
    packed_element(E, k, i, j);
    src = i >= j ? i * E + j : j * E + i;
  } else if constexpr (PH && !PP) {
    src = packed_index(k / E, k % E);
  }
  P[f * SP + k] = hP[s * SH + src];
}

template <class M>
inline void batch_restore_hist(const double* hx_filt, const double* hP_filt, const int* idx, const int* hist_row, long long n,
                               long long hist_B, double* x, double* P, int flags, void* stream) {
  if (!check_packed_flag<M, false>(flags, "batch_restore_hist")) return;
  if constexpr (M::EDIM > 32) {
    fprintf(stderr, "[rednose_b200] batch_restore_hist: ragged histories exist only up to EDIM 32 (EDIM = %d)\n", M::EDIM);
    last_status() = (int)cudaErrorNotSupported;
  } else {
    if (n < 0 || hist_B <= 0 || (n > 0 && (!hx_filt || !hP_filt || !idx || !hist_row || !x || !P))) {
      fprintf(stderr, "[rednose_b200] batch_restore_hist: n >= 0, a positive slab stride and, for n > 0, every pointer are required\n");
      last_status() = (int)cudaErrorInvalidValue;
      return;
    }
    if (n == 0) return;
    constexpr int D = M::DIM, E = M::EDIM;
    const bool ph = flags & FLAG_PACKED_HIST, pp = flags & FLAG_PACKED_P;
    auto run = [&](auto kern, int w) {
      kern<<<(unsigned)((n * w + 255) / 256), 256, 0, (cudaStream_t)stream>>>(hx_filt, hP_filt, idx, hist_row, n, hist_B, x, P);
    };
    if constexpr (pair_may_serve<M>()) {
      constexpr int PD = packed_doubles(E);
      if (ph && pp) run(restore_hist_kernel<D, E, true, true>, D + PD);
      else if (ph) run(restore_hist_kernel<D, E, true, false>, D + E * E);
      else if (pp) run(restore_hist_kernel<D, E, false, true>, D + PD);
      else run(restore_hist_kernel<D, E, false, false>, D + E * E);
    } else {
      run(restore_hist_kernel<D, E, false, false>, D + E * E);   // check_packed_flag refused the packed flags
    }
    check(cudaGetLastError(), "batch_restore_hist launch");
  }
}

// --------------------------------------------- batched, HOST buffers (stateless) ---
// Full round trip: x,P,z,R(,ea) host -> device, fused step, x,P,y device -> host, in
// chunks on alternating streams so copies overlap the kernel when the host
// buffers are pinned.  This is the batched analogue of calling the reference's
// <name>_predict + <name>_update_<kind> on caller-owned host arrays.
template <class M, class K>
inline void host_step(HostCtx<M>& ctx, double* x, double* P, const double* Q, const double* dt_arr, double dt,
                      double* z, const double* R, const double* ea, int n_obs, long long B,
                      const int* quat_idxs, int n_quat, int flags) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM, EA = K::EADIM;
  if (!check_quat_idxs(quat_idxs, n_quat, D)) return;   // before any stream, allocation or copy
  if (flags & (FLAG_PACKED_P | FLAG_PACKED_HIST)) {
    fprintf(stderr, "[rednose_b200] host_step: host buffers hold the full [B, EDIM, EDIM] covariance; FLAG_PACKED_P and FLAG_PACKED_HIST are not accepted\n");
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  if (B <= 0) return;
  const long long per = D + E * E + 1 + (long long)n_obs * (Z + Z * Z + EA) + 1;
  constexpr long long PAD = 8;   // each of the six sub-buffers below is rounded up to an even number of doubles
  long long chunk = (64ll << 20) / (per * 8);  // ~64 MiB of device staging per stream
  if (chunk < 1) chunk = 1;
  if (chunk > B) chunk = B;
  constexpr int NS = 3;
  struct Stage { cudaStream_t streams[NS] = {nullptr, nullptr, nullptr}; double* dbuf[NS] = {nullptr, nullptr, nullptr}; long long dcap = 0; double* dQ = nullptr; };
  static Stage stages[MAX_DEVICES];   // streams and staging buffers belong to the device that is current
  std::lock_guard<std::mutex> lk(ctx.mu);
  Stage& sg = stages[current_device()];
  cudaStream_t* streams = sg.streams;
  double** dbuf = sg.dbuf;
  long long& dcap = sg.dcap;
  double*& dQ = sg.dQ;
  for (int i = 0; i < NS; ++i)
    if (!streams[i] && !check(cudaStreamCreateWithFlags(&streams[i], cudaStreamNonBlocking), "cudaStreamCreate")) return;
  if (!dQ && !check(cudaMalloc(&dQ, sizeof(double) * E * E), "cudaMalloc(Q)")) return;
  if (chunk * per + PAD > dcap) {
    for (int i = 0; i < NS; ++i) {
      if (dbuf[i]) cudaFree(dbuf[i]);
      dbuf[i] = nullptr;
      if (!check(cudaMalloc(&dbuf[i], sizeof(double) * (chunk * per + PAD)), "cudaMalloc(stage)")) return;
    }
    dcap = chunk * per + PAD;
  }
  if (!check(cudaMemcpy(dQ, Q, sizeof(double) * E * E, cudaMemcpyHostToDevice), "memcpy Q")) return;
  int si = 0;
  for (long long b0 = 0; b0 < B; b0 += chunk, si = (si + 1) % NS) {
    const long long nb = (B - b0 < chunk) ? (B - b0) : chunk;
    cudaStream_t st = streams[si];
    auto up2 = [](long long n) { return (n + 1) & ~1ll; };  // keep every sub-buffer 16-byte aligned (bulk copies)
    double* dx = dbuf[si];
    double* dP = dx + up2(nb * D);
    double* ddt = dP + up2(nb * E * E);
    double* dz = ddt + up2(nb);
    double* dR = dz + up2(nb * n_obs * Z);
    double* dea = dR + up2(nb * n_obs * Z * Z);
    cudaMemcpyAsync(dx, x + b0 * D, sizeof(double) * nb * D, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(dP, P + b0 * E * E, sizeof(double) * nb * E * E, cudaMemcpyHostToDevice, st);
    if (dt_arr) cudaMemcpyAsync(ddt, dt_arr + b0, sizeof(double) * nb, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(dz, z + b0 * n_obs * Z, sizeof(double) * nb * n_obs * Z, cudaMemcpyHostToDevice, st);
    if (flags & FLAG_SHARED_R) cudaMemcpyAsync(dR, R, sizeof(double) * Z * Z, cudaMemcpyHostToDevice, st);
    else cudaMemcpyAsync(dR, R + b0 * n_obs * Z * Z, sizeof(double) * nb * n_obs * Z * Z, cudaMemcpyHostToDevice, st);
    if (EA > 0 && ea) cudaMemcpyAsync(dea, ea + b0 * n_obs * EA, sizeof(double) * nb * n_obs * EA, cudaMemcpyHostToDevice, st);
    StepArgs<M::NG> a;
    fill_common<M>(a, ctx, nb, quat_idxs, n_quat, flags);   // validated above: cannot fail
    a.x = dx; a.P = dP; a.Q = dQ; a.dt_arr = dt_arr ? ddt : nullptr; a.dt = dt;
    a.z = dz; a.R = dR; a.ea = (EA > 0 && ea) ? dea : nullptr; a.ea_dim = EA; a.n_obs = n_obs;
    launch_step<M, K, true, true>(a, st);
    cudaMemcpyAsync(x + b0 * D, dx, sizeof(double) * nb * D, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(P + b0 * E * E, dP, sizeof(double) * nb * E * E, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(z + b0 * n_obs * Z, dz, sizeof(double) * nb * n_obs * Z, cudaMemcpyDeviceToHost, st);
  }
  for (int i = 0; i < NS; ++i) check(cudaStreamSynchronize(streams[i]), "host_step sync");
}

// --------------------------------------------- single filter, HOST pointers ---
// The reference's own entry points (<name>_predict / <name>_update_<kind> on caller-owned host arrays, one filter).  All
// inputs are packed into ONE pinned staging buffer and travel in one asynchronous copy each way on a private stream
// (round 1 issued 3-5 synchronous pageable cudaMemcpy per direction): copy in, launch with B = 1, copy out, one wait.
template <class M>
inline void single_predict(HostCtx<M>& ctx, double* x, double* P, const double* Q, double dt) {
  constexpr int D = M::DIM, E = M::EDIM;
  std::lock_guard<std::mutex> lk(ctx.mu);
  constexpr int DA = (D + 1) & ~1;   // P starts 16-byte aligned behind x (covariance tiles move by bulk copy / 128-bit accesses)
  constexpr size_t N = DA + 2 * E * E;
  double* d = ctx.scratch(N);
  double* h = ctx.pinned(N);
  cudaStream_t st = ctx.single_stream();
  if (!d || !h || !st) return;
  memcpy(h, x, sizeof(double) * D); memcpy(h + DA, P, sizeof(double) * E * E); memcpy(h + DA + E * E, Q, sizeof(double) * E * E);
  if (!check(cudaMemcpyAsync(d, h, sizeof(double) * N, cudaMemcpyHostToDevice, st), "memcpy in")) return;
  StepArgs<M::NG> a;
  fill_common<M>(a, ctx, 1, nullptr, 0, 0);
  a.x = d; a.P = d + DA; a.Q = d + DA + E * E; a.dt = dt;
  launch_step<M, NullKind, true, false>(a, st);
  cudaMemcpyAsync(h, d, sizeof(double) * (DA + E * E), cudaMemcpyDeviceToHost, st);
  if (!check(cudaStreamSynchronize(st), "single_predict")) return;
  memcpy(x, h, sizeof(double) * D); memcpy(P, h + DA, sizeof(double) * E * E);
}

template <class M, class K>
inline void single_update(HostCtx<M>& ctx, double* x, double* P, double* z, const double* R, const double* ea) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM, EA = K::EADIM;
  std::lock_guard<std::mutex> lk(ctx.mu);
  constexpr int DA = (D + 1) & ~1;   // see single_predict
  constexpr size_t OZ = DA + E * E, OR_ = OZ + Z, OEA = OR_ + Z * Z, N = OEA + (EA > 0 ? EA : 1);
  double* d = ctx.scratch(N);
  double* h = ctx.pinned(N);
  cudaStream_t st = ctx.single_stream();
  if (!d || !h || !st) return;
  memcpy(h, x, sizeof(double) * D); memcpy(h + DA, P, sizeof(double) * E * E); memcpy(h + OZ, z, sizeof(double) * Z);
  memcpy(h + OR_, R, sizeof(double) * Z * Z);
  if (EA > 0 && ea) memcpy(h + OEA, ea, sizeof(double) * EA);
  if (!check(cudaMemcpyAsync(d, h, sizeof(double) * N, cudaMemcpyHostToDevice, st), "memcpy in")) return;
  StepArgs<M::NG> a;
  fill_common<M>(a, ctx, 1, nullptr, 0, 0);
  a.x = d; a.P = d + DA; a.z = d + OZ; a.R = d + OR_; a.ea = (EA > 0 && ea) ? d + OEA : nullptr; a.ea_dim = EA;
  launch_step<M, K, false, true>(a, st);
  cudaMemcpyAsync(h, d, sizeof(double) * (OZ + Z), cudaMemcpyDeviceToHost, st);
  if (!check(cudaStreamSynchronize(st), "single_update")) return;
  memcpy(x, h, sizeof(double) * D); memcpy(P, h + DA, sizeof(double) * E * E);
  // ekf_c.c:120: the innovation overwrites z (K::YDIM entries: ZDIM, or ZDIM-EADIM after projection)
  memcpy(z, h + OZ, sizeof(double) * K::YDIM);
}

// leaf functions exported with host pointers (ekf_sym.py:155-161): one-thread kernels
template <class M, class Kern>
inline void run_leaf(HostCtx<M>& ctx, Kern kern, const double* in0, int n0, const double* in1, int n1, double s,
                     double* out, int nout) {
  std::lock_guard<std::mutex> lk(ctx.mu);
  double* d = ctx.scratch((size_t)n0 + n1 + nout + 2);
  if (!d) return;
  double* d0 = d; double* d1 = d + n0; double* dout = d1 + n1;
  if (n0 > 0 && !check(cudaMemcpy(d0, in0, sizeof(double) * n0, cudaMemcpyHostToDevice), "leaf memcpy")) return;
  if (n1 > 0 && in1) cudaMemcpy(d1, in1, sizeof(double) * n1, cudaMemcpyHostToDevice);
  kern<<<1, 32>>>(d0, d1, s, ctx.gv, dout);
  check(cudaGetLastError(), "leaf launch");
  check(cudaMemcpy(out, dout, sizeof(double) * nout, cudaMemcpyDeviceToHost), "leaf memcpy back");
}

}  // namespace rnb

#define RNB_LEAF_KERNEL(KNAME, NGV, CALL)                                                              \
  __global__ void KNAME(const double* in0, const double* in1, double s, rnb::GV<NGV> gvs, double* out) { \
    const double* gv = gvs.v; (void)gv; (void)in1; (void)s;                                            \
    if (threadIdx.x == 0) { CALL; }                                                                    \
  }
