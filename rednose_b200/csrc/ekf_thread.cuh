// rednose_b200 -- thread-per-filter fused predict+update kernel for tiny states
// (EDIM <= 6, e.g. the kinematic example: DIM=EDIM=2, examples/kinematic_kf.py:31-47).
//
// One thread owns one filter: x and the whole P live in registers, every loop is
// unrolled at compile time, F / H_err sparsity comes from the generated model
// (MODEL::F_apply, KIND::Herr_apply).  The batch is laid out AoS ([B,DIM],
// [B,EDIM,EDIM]); a thread's record is contiguous, so a warp reads 32 consecutive
// records = one fully used run of sectors (16-byte vector accesses when the
// record size allows).  Memory-bound by design: 128 B/step for the kinematic model.
//
// Reference semantics: ekf_c.c:8-33 (predict), :37-121 (update, He==NULL path),
// normalisation ekf_sym.cc:69-77,207,213.
#pragma once
#include "ekf_common.cuh"

namespace rnb {

template <int W>
__device__ __forceinline__ void load_rec(const double* __restrict__ g, double (&r)[W]) {
  if constexpr (W % 2 == 0) {
    const double2* g2 = reinterpret_cast<const double2*>(g);
#pragma unroll
    for (int i = 0; i < W / 2; ++i) { double2 v = g2[i]; r[2 * i] = v.x; r[2 * i + 1] = v.y; }
  } else {
#pragma unroll
    for (int i = 0; i < W; ++i) r[i] = g[i];
  }
}

template <int W>
__device__ __forceinline__ void store_rec(double* __restrict__ g, const double (&r)[W]) {
  if constexpr (W % 2 == 0) {
    double2* g2 = reinterpret_cast<double2*>(g);
#pragma unroll
    for (int i = 0; i < W / 2; ++i) g2[i] = make_double2(r[2 * i], r[2 * i + 1]);
  } else {
#pragma unroll
    for (int i = 0; i < W; ++i) g[i] = r[i];
  }
}

// HIST: gather list with per-entry history rows (StepArgs::hist_row); the other instantiations are the kernel as it was
template <class M, class K, bool PRED, bool UPD, bool HIST = false>
__global__ void __launch_bounds__(128) ekf_step_thread(const StepArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;

  const long long fb = a.idx ? (long long)a.idx[b] : b;   // filter this entry works on
  long long hb = fb;                                       // history slab element of this entry (-1: not recorded)
  if constexpr (HIST) hb = hist_slot(a, b, fb);
  const bool rec = !HIST || hb >= 0;
  double x[D];
  double P[E * E];
  load_rec<D>(a.x + fb * D, x);
  load_rec<E * E>(a.P + fb * E * E, P);

  if constexpr (PRED) {
    const double dt = a.dt_arr ? a.dt_arr[b] : a.dt;
    double xn[D];
    double fv[M::NF > 0 ? M::NF : 1];
    M::predict_leaf(x, dt, a.gv, xn, fv);
    // P <- F P      (column by column: (FP)[:,j] = F P[:,j])
#pragma unroll
    for (int j = 0; j < E; ++j) {
      double v[E];
#pragma unroll
      for (int i = 0; i < E; ++i) v[i] = P[i * E + j];
      M::F_apply(fv, v);
#pragma unroll
      for (int i = 0; i < E; ++i) P[i * E + j] = v[i];
    }
    // P <- P F^T    (row by row: (M F^T)[i,:]^T = F M[i,:]^T)
#pragma unroll
    for (int i = 0; i < E; ++i) {
      double v[E];
#pragma unroll
      for (int j = 0; j < E; ++j) v[j] = P[i * E + j];
      M::F_apply(fv, v);
#pragma unroll
      for (int j = 0; j < E; ++j) P[i * E + j] = v[j];
    }
#pragma unroll
    for (int i = 0; i < E * E; ++i) P[i] = fma(dt, __ldg(a.Q + i), P[i]);
#pragma unroll
    for (int i = 0; i < D; ++i) x[i] = xn[i];
    if (a.flags & FLAG_NORM_AFTER_PREDICT)
      for (int q = 0; q < a.n_quat; ++q) {
        // dynamic index into a register array would spill; D is tiny here so select
        double qv[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          qv[c] = 0.0;
#pragma unroll
          for (int i = 0; i < D; ++i) if (i == a.quat_idx[q] + c) qv[c] = x[i];
        }
        normalize4(qv);
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int i = 0; i < D; ++i) if (i == a.quat_idx[q] + c) x[i] = qv[c];
      }
    if (a.hx_pred && rec) store_rec<D>(a.hx_pred + hb * D, x);
    if (a.hP_pred && rec) store_rec<E * E>(a.hP_pred + hb * E * E, P);
  }

  if constexpr (UPD) {
    for (int o = 0; o < a.n_obs; ++o) {
      const long long bo = b * a.n_obs + o;
      double zz[Z], R[Z][Z];
#pragma unroll
      for (int i = 0; i < Z; ++i) zz[i] = a.z[bo * Z + i];
#pragma unroll
      for (int i = 0; i < Z; ++i)
#pragma unroll
        for (int j = 0; j < Z; ++j) R[i][j] = a.R[((a.flags & FLAG_SHARED_R) ? 0 : bo * Z * Z) + i * Z + j];
      const double* ea = a.ea ? a.ea + bo * a.ea_dim : nullptr;

      double hx[Z];
      double hv[K::NH > 0 ? K::NH : 1];
      K::obs_leaf(x, ea, a.gv, hx, hv);
      double y[Z];
#pragma unroll
      for (int i = 0; i < Z; ++i) y[i] = zz[i] - hx[i];

      // HP[a][j] = sum_k Herr[a][k] P[k][j]
      double HP[Z][E];
#pragma unroll
      for (int j = 0; j < E; ++j) {
        double v[E], hp[Z];
#pragma unroll
        for (int i = 0; i < E; ++i) v[i] = P[i * E + j];
        K::Herr_apply(hv, v, hp);
#pragma unroll
        for (int c = 0; c < Z; ++c) HP[c][j] = hp[c];
      }
      double S[Z][Z];
#pragma unroll
      for (int i = 0; i < Z; ++i)
#pragma unroll
        for (int j = 0; j < Z; ++j) S[i][j] = 0.0;
      K::S_accum(hv, [&](int c, int k) { return HP[c][k]; }, S);

      LDL<Z> ldl;
      if constexpr (K::MAHA) {
        // ekf_c.c:88-94: gate = inflate R by 1e16 and still run the update
        double Sg[Z][Z];
#pragma unroll
        for (int i = 0; i < Z; ++i)
#pragma unroll
          for (int j = 0; j < Z; ++j) Sg[i][j] = S[i][j] + R[i][j];
        ldl.factor(Sg);
        double u[Z];
#pragma unroll
        for (int i = 0; i < Z; ++i) u[i] = y[i];
        ldl.solve(u);
        double d = 0.0;
#pragma unroll
        for (int i = 0; i < Z; ++i) d += y[i] * u[i];
        if (d > K::MAHA_THRESH) {
#pragma unroll
          for (int i = 0; i < Z; ++i)
#pragma unroll
            for (int j = 0; j < Z; ++j) R[i][j] *= 1.0e16;
        }
      }
#pragma unroll
      for (int i = 0; i < Z; ++i)
#pragma unroll
        for (int j = 0; j < Z; ++j) S[i][j] += R[i][j];
      ldl.factor(S);

      // W = S^-1 HP  (column j of W is row j of K);  dx = K y
      double dx[E];
#pragma unroll
      for (int j = 0; j < E; ++j) {
        double w[Z];
#pragma unroll
        for (int c = 0; c < Z; ++c) w[c] = HP[c][j];
        ldl.solve(w);
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < Z; ++c) s = fma(w[c], y[c], s);
        dx[j] = s;
        // P[:,j] -= HP^T w   == Joseph form when K is the exact gain (see DESIGN.md)
#pragma unroll
        for (int i = 0; i < E; ++i) {
          double acc = P[i * E + j];
#pragma unroll
          for (int c = 0; c < Z; ++c) acc = fma(-HP[c][i], w[c], acc);
          P[i * E + j] = acc;
        }
      }
      double xn[D];
      M::err_fun(x, dx, a.gv, xn);
#pragma unroll
      for (int i = 0; i < D; ++i) x[i] = xn[i];
      if (a.flags & FLAG_NORM_AFTER_UPDATE)
        for (int q = 0; q < a.n_quat; ++q) {
          double qv[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            qv[c] = 0.0;
#pragma unroll
            for (int i = 0; i < D; ++i) if (i == a.quat_idx[q] + c) qv[c] = x[i];
          }
          normalize4(qv);
#pragma unroll
          for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int i = 0; i < D; ++i) if (i == a.quat_idx[q] + c) x[i] = qv[c];
        }
#pragma unroll
      for (int i = 0; i < Z; ++i) a.z[bo * Z + i] = y[i];
    }
    if (a.hx_filt && rec) store_rec<D>(a.hx_filt + hb * D, x);
    if (a.hP_filt && rec) store_rec<E * E>(a.hP_filt + hb * E * E, P);
  }

  store_rec<D>(a.x + fb * D, x);
  store_rec<E * E>(a.P + fb * E * E, P);
}

}  // namespace rnb
