// rednose_b200 -- CTA-per-filter predict / update for large error states (EDIM > 32), e.g. an MSCKF
// with 10 cloned camera poses: DIM 93, EDIM 82, MEDIM 22, feature-track kind ZDIM 20 / EADIM 3.
//
// The covariance (EDIM^2 doubles = 53.8 kB at EDIM 82) does not fit a warp's registers, so one CTA owns one
// filter with P resident in shared memory (odd leading dimension: rows and columns are both conflict-free)
// and thread j working on column j.  A step is two launches:
//
//   ekf_leaf_thread   thread-per-filter: x_pred = f(x, dt), the F value slots, y = z - h(x_pred), the H_err
//                     value slots and (feature kinds) He = dh/d(ea) -> a small per-filter workspace in HBM.
//                     (Same reason as the warp kernel's phase A: scalar generated code wants one filter per
//                     lane, not one filter per CTA.)
//   ekf_step_cta      CTA-per-filter: P <- F P F^T + dt Q on the MEDIM main block only (ekf_c.c:23-26),
//                     left-null-space projection of (y, H_err, R) with Householder reflectors of He
//                     (ekf_c.c:66-76 uses fullPivLu().kernel(); x and P do not depend on the basis),
//                     Mahalanobis gate (ekf_c.c:88-94), S = LDL^T, gain, P <- P - (HP)^T S^-1 (HP), inject.
//
// Exploited structure: H_err of a feature kind has 6 non-zeros per row (one clone each), so H_err P goes
// through the generated sparse KIND::Herr_apply, and the projection is applied to the small ZDIM-vectors
// (Q^T (H_err P) = (Q^T H_err) P) instead of densifying H_err.
#pragma once
#include "ekf_common.cuh"
#include "ekf_warp.cuh"
#include "ekf_rts_mma.cuh"   // dmma884

namespace rnb {

template <class M, class K>
struct CtaWs {  // per-filter workspace record (doubles)
  static constexpr int OFF_X = 0;
  static constexpr int OFF_FV = OFF_X + M::DIM;
  static constexpr int OFF_DT = OFF_FV + (M::NF > 0 ? M::NF : 1);
  static constexpr int OFF_Y = OFF_DT + 1;
  static constexpr int OFF_HV = OFF_Y + K::ZDIM;
  static constexpr int OFF_HE = OFF_HV + (K::NH > 0 ? K::NH : 1);
  // feature kinds: Householder vectors V [NR][Z] of He (NR = EADIM) followed by the NR scalars beta
  static constexpr int SIZE = OFF_HE + (K::HAS_HE ? K::ZDIM * K::EADIM + K::EADIM : 0);
};

// ------------------------------------------------------------------ leaf kernel ---
template <class M, class K, bool PRED, bool UPD>
__global__ void __launch_bounds__(64) ekf_leaf_thread(const StepArgs<M::NG> a, int o, double* __restrict__ ws_all) {
  constexpr int D = M::DIM, Z = K::ZDIM;
  using W = CtaWs<M, K>;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  double* ws = ws_all + b * W::SIZE;
  const long long fb = a.idx ? (long long)a.idx[b] : b;   // filter this entry works on
  double x[D];
  if (PRED || o == 0) {
#pragma unroll
    for (int i = 0; i < D; ++i) x[i] = a.x[fb * D + i];
  } else {
#pragma unroll
    for (int i = 0; i < D; ++i) x[i] = ws[W::OFF_X + i];
  }
  if constexpr (PRED) {
    const double dt = a.dt_arr ? a.dt_arr[b] : a.dt;
    double xn[D];
    double fv[M::NF > 0 ? M::NF : 1];
    M::predict_leaf(x, dt, a.gv, xn, fv);
#pragma unroll
    for (int i = 0; i < (M::NF > 0 ? M::NF : 1); ++i) ws[W::OFF_FV + i] = fv[i];
    ws[W::OFF_DT] = dt;
#pragma unroll
    for (int i = 0; i < D; ++i) ws[W::OFF_X + i] = xn[i];
    if ((a.flags & FLAG_NORM_AFTER_PREDICT) && a.n_quat > 0) {
      for (int q = 0; q < a.n_quat; ++q) normalize4(ws + W::OFF_X + a.quat_idx[q]);
    }
#pragma unroll
    for (int i = 0; i < D; ++i) x[i] = ws[W::OFF_X + i];
    if (a.hx_pred) {
#pragma unroll
      for (int i = 0; i < D; ++i) a.hx_pred[fb * D + i] = x[i];
    }
    if (!UPD) {
#pragma unroll
      for (int i = 0; i < D; ++i) a.x[fb * D + i] = x[i];
    }
  } else if (o == 0) {
#pragma unroll
    for (int i = 0; i < D; ++i) ws[W::OFF_X + i] = x[i];
  }
  if constexpr (UPD) {
    const long long bo = b * a.n_obs + o;
    const double* ea = a.ea ? a.ea + bo * a.ea_dim : nullptr;
    double hx[Z];
    K::obs_leaf(x, ea, a.gv, hx, *reinterpret_cast<double(*)[K::NH > 0 ? K::NH : 1]>(ws + W::OFF_HV));
#pragma unroll
    for (int i = 0; i < Z; ++i) ws[W::OFF_Y + i] = a.z[bo * Z + i] - hx[i];
    if constexpr (K::HAS_HE) {
      // Householder QR of He (Z x EA) done here, one filter per thread: Q = H_1 .. H_EA, the left null space of
      // He is spanned by the last Z - EA columns of Q (ekf_c.c:66-76 takes fullPivLu().kernel() of He^T instead)
      constexpr int EA = K::EADIM;
      double He[Z * EA];
      K::He_dense(x, ea, a.gv, He);
#pragma unroll
      for (int r = 0; r < EA; ++r) {
        double nrm = 0.0;
#pragma unroll
        for (int i = r; i < Z; ++i) nrm = fma(He[i * EA + r], He[i * EA + r], nrm);
        nrm = sqrt(nrm);
        const double a0 = He[r * EA + r];
        const double alpha = (a0 >= 0.0) ? -nrm : nrm;
        double v[Z];
#pragma unroll
        for (int i = 0; i < Z; ++i) v[i] = (i < r) ? 0.0 : He[i * EA + r];
        v[r] = a0 - alpha;
        double vn = 0.0;
#pragma unroll
        for (int i = r; i < Z; ++i) vn = fma(v[i], v[i], vn);
        const double beta = (vn > 0.0) ? 2.0 / vn : 0.0;
#pragma unroll
        for (int c = r + 1; c < EA; ++c) {
          double w = 0.0;
#pragma unroll
          for (int i = r; i < Z; ++i) w = fma(v[i], He[i * EA + c], w);
          w *= beta;
#pragma unroll
          for (int i = r; i < Z; ++i) He[i * EA + c] = fma(-w, v[i], He[i * EA + c]);
        }
#pragma unroll
        for (int i = 0; i < Z; ++i) ws[W::OFF_HE + r * Z + i] = v[i];
        ws[W::OFF_HE + EA * Z + r] = beta;
      }
    }
  }
}

// ------------------------------------------------------------------ CTA kernel ---
// Shared-memory plan of one CTA (= one filter), 3 warps, thread j <-> column j of the covariance:
//   Ppk   the symmetric covariance, PACKED lower-triangular row-major (E (E + 1) / 2 doubles: 27.2 kB at EDIM 82 instead
//         of 53.8 kB) -- this is what lets 4 CTAs share an SM instead of 2, so that the serial sections of one filter
//         (the small factorisation, the projections) overlap the wide sections of three others;
//   U     [column][k]: first H_err P (unprojected, for S), later U = L^-1 (A^T H_err P) of S = L D L^T; the rank-m
//         covariance update is P -= U^T D^-1 U, which needs ONE operand buffer and no backward substitution
//         (ekf_c.c:105,115 with K the exact gain reduce to this); during the predict its first rows hold the
//         NFROWS x E exchange rows of F P;
//   S/LT, Rm, small vectors.
template <class M, class K>
struct CtaSmem {
  static constexpr int E = M::EDIM, Z = K::ZDIM, Y = K::YDIM;
  static constexpr int NPK = E * (E + 1) / 2;
  static constexpr int HL = (Z + 3) & ~3;          // leading dimension of U ([column][k]); multiple of the mma k = 4
  static constexpr int SL = Z | 1;
  static constexpr int NU = (E * HL > M::NFROWS * E) ? E * HL : M::NFROWS * E;
  double Ppk[NPK];
  double U[NU];
  double S[Z * SL];                                // H_err P H_err^T (projected in place); then LT: the L D L^T factor, transposed
  double Rm[Z * SL];                               // R (projected in place)
  double dinv[HL];                                 // 1 / D[k], zero padded to HL
  double yt[HL];                                   // L^-1 y
  double V[(K::HAS_HE ? K::EADIM : 1) * Z];        // Householder vectors of He
  double beta[K::HAS_HE ? K::EADIM : 1];
  double y[Z];
  double hv[K::NH > 0 ? K::NH : 1];
  double fv[M::NF > 0 ? M::NF : 1];
  double x[M::DIM], xo[M::DIM], dx[E];
  double dt;
  int gated;
};

template <int Z>
struct SmemCol {  // read-only view of one shared-memory column / row as a vector
  const double* p;
  int stride;
  __device__ __forceinline__ double operator[](int i) const { return p[i * stride]; }
};

// element (i, j) of the packed lower-triangular storage
__device__ __forceinline__ int pk_idx(int i, int j) { return (i >= j) ? (i * (i + 1) / 2 + j) : (j * (j + 1) / 2 + i); }

struct PackedCol {  // column `col` of the packed symmetric matrix as a vector (generated code indexes it with constants)
  const double* p;
  int col, tcol;    // tcol = col (col + 1) / 2
  __device__ __forceinline__ double operator[](int i) const { return (i >= col) ? p[i * (i + 1) / 2 + col] : p[tcol + i]; }
};

// packed index -> (row, column)
__device__ __forceinline__ void pk_unpack(int idx, int& i, int& j) {
  i = (int)((sqrtf(8.0f * (float)idx + 1.0f) - 1.0f) * 0.5f);
  while (i * (i + 1) / 2 > idx) --i;
  while ((i + 1) * (i + 2) / 2 <= idx) ++i;
  j = idx - i * (i + 1) / 2;
}

// apply Q^T = H_r ... H_1 (Householder reflectors, vectors V[r][:], scalars beta[r]) to a Z-vector in registers
template <int Z, int NR>
__device__ __forceinline__ void apply_reflectors(const double* V, const double* beta, double (&u)[Z]) {
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    double w0 = 0.0, w1 = 0.0;   // two partial sums: half the dependent-FMA chain
#pragma unroll
    for (int i = 0; i < Z; i += 2) {
      w0 = fma(V[r * Z + i], u[i], w0);
      if (i + 1 < Z) w1 = fma(V[r * Z + i + 1], u[i + 1], w1);
    }
    const double w = (w0 + w1) * beta[r];
#pragma unroll
    for (int i = 0; i < Z; ++i) u[i] = fma(-w, V[r * Z + i], u[i]);
  }
}

template <class M>
constexpr int cta_threads() { return ((M::EDIM + 31) / 32) * 32; }   // one thread per column
#ifndef RNB_CTA_MIN_BLOCKS
#define RNB_CTA_MIN_BLOCKS 4
#endif

template <class M, class K, bool PRED, bool UPD>
__global__ void __launch_bounds__(cta_threads<M>(), RNB_CTA_MIN_BLOCKS) ekf_step_cta(const StepArgs<M::NG> a, int o, const double* __restrict__ ws_all) {
  constexpr int D = M::DIM, E = M::EDIM, ME = M::MEDIM, Z = K::ZDIM, Y = K::YDIM, NR = Z - Y;
  using SM = CtaSmem<M, K>;
  using W = CtaWs<M, K>;
  constexpr int HL = SM::HL, SL = SM::SL, NPK = SM::NPK;
  static_assert(ME <= 32, "FROW_MASK covers a main block of at most 32 error states");
  static_assert(Y + 1 <= 32, "the innovation covariance is factored by one warp (one lane per column + one for y)");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SM& s = *reinterpret_cast<SM*>(smem_raw);
  const int tid = threadIdx.x, nth = blockDim.x;
  const int col = tid;
  const long long b = blockIdx.x;
  const double* ws = ws_all + b * W::SIZE;
  const long long fb = a.idx ? (long long)a.idx[b] : b;   // filter this entry works on
  double* Pg = a.P + fb * (long long)(E * E);
  const bool own = col < E;            // this thread is attached to column `col`
  const PackedCol pc{s.Ppk, own ? col : 0, own ? col * (col + 1) / 2 : 0};

  // ---- stage: lower triangle of the covariance (the matrix is symmetric: half the read traffic), leaf values.
  //      Warp w takes rows w, w + nw, ...; lanes run along the row (coalesced). ----
  const int lane = tid & 31, warp = tid >> 5, nw = nth >> 5;
  constexpr int NC = (E + 31) / 32;     // 32-column chunks of a row
  // cp.async (LDGSTS, 8 bytes per element: a packed row starts 16-byte aligned only every other row): no registers are
  // held, so the whole triangle is in flight at once -- ONE global round trip, overlapped with the leaf-value loads below
  // (the register-staged version needed four and spent a large share of the kernel waiting on them)
  for (int i = warp; i < E; i += nw) {
    const int ti = i * (i + 1) / 2;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int j = lane + 32 * c;
      if (j <= i) {
        const unsigned dst = (unsigned)__cvta_generic_to_shared(&s.Ppk[ti + j]);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(Pg + i * E + j) : "memory");
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  // packed -> full row-major matrix in global memory (P itself and the history slabs): coalesced rows, no divisions
  int tj[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) tj[c] = (lane + 32 * c) * (lane + 32 * c + 1) / 2;
  bool aug = false;   // set below when this launch also shifts the clone window
  auto store_full = [&](double* __restrict__ dst) {
    for (int i = warp; i < E; i += nw) {
      const int ti = i * (i + 1) / 2;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int j = lane + 32 * c;
        if (j < E) dst[i * E + j] = s.Ppk[(j <= i) ? ti + j : tj[c] + i];
      }
    }
  };
  for (int i = tid; i < D; i += nth) s.x[i] = ws[W::OFF_X + i];
  if constexpr (PRED) {
    for (int i = tid; i < (M::NF > 0 ? M::NF : 1); i += nth) s.fv[i] = ws[W::OFF_FV + i];
    if (tid == 0) s.dt = ws[W::OFF_DT];
  }
  if constexpr (UPD) {
    for (int i = tid; i < (K::NH > 0 ? K::NH : 1); i += nth) s.hv[i] = ws[W::OFF_HV + i];
    for (int i = tid; i < Z; i += nth) s.y[i] = ws[W::OFF_Y + i];
    if constexpr (K::HAS_HE) {
      for (int i = tid; i < Z * K::EADIM; i += nth) s.V[i] = ws[W::OFF_HE + i];
      for (int i = tid; i < K::EADIM; i += nth) s.beta[i] = ws[W::OFF_HE + Z * K::EADIM + i];
    }
    const double* Rg = a.R + ((a.flags & FLAG_SHARED_R) ? 0 : (b * a.n_obs + o) * (long long)(Z * Z));
    for (int idx = tid; idx < Z * Z; idx += nth) s.Rm[(idx / Z) * SL + idx % Z] = Rg[idx];
    for (int i = tid; i < HL; i += nth) { s.dinv[i] = 0.0; s.yt[i] = 0.0; }
    if (tid == 0) s.gated = 0;
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  // =============================== predict: P <- F P F^T + dt Q (main block) ===============================
  if constexpr (PRED) {
    double* T = s.U;                   // exchange rows: T[slot][column] = (F P)[frow(slot)][column]
    if (own) {                         // column col of F P: only the rows of F that differ from the identity change
      double v[ME];
#pragma unroll
      for (int i = 0; i < ME; ++i) v[i] = pc[i];
      M::F_apply(s.fv, v);
      M::frows_store(v, &T[col], E);
    }
    __syncthreads();
    if (own && col < ME && ((M::FROW_MASK >> col) & 1u)) {   // row col of (F P) F^T, columns of the main block
      const int slot = __popc(M::FROW_MASK & ((1u << col) - 1u));
      double v[ME];
#pragma unroll
      for (int k = 0; k < ME; ++k) {
        // (F P)[col][k]: an exchange row if k is itself a changed row, else (symmetry of P) the exchange row's own entry
        v[k] = T[slot * E + k];
      }
      M::F_apply(s.fv, v);
      M::frows_scatter(v, &T[slot * E], 1);   // only the NFROWS x NFROWS block differs from T
    }
    __syncthreads();
    if (own) {
      int slot = 0;
#pragma unroll
      for (int r = 0; r < ME; ++r) {
        if ((M::FROW_MASK >> r) & 1u) {
          // element {r, col}: when both indices are changed rows it is visited from both sides -- the larger column writes
          const bool other_side = (col < r) && ((M::FROW_MASK >> col) & 1u);
          if (!other_side) s.Ppk[pk_idx(r, col)] = T[slot * E + col];
          ++slot;
        }
      }
    }
    __syncthreads();
    {
      const double dt = s.dt;
      if (a.flags & FLAG_Q_DIAG) {
        if (own) s.Ppk[pc.tcol + col] += dt * __ldg(a.Q + col * E + col);
      } else {
        for (int i = 0; i < E; ++i)
          for (int j = tid; j <= i; j += nth) s.Ppk[i * (i + 1) / 2 + j] = fma(dt, __ldg(a.Q + i * E + j), s.Ppk[i * (i + 1) / 2 + j]);
      }
    }
    __syncthreads();
    if (a.hP_pred) store_full(a.hP_pred + fb * (long long)(E * E));
  }

  if constexpr (UPD) {
    // ---- HP_raw[:, col] = H_err P[:, col] (sparse) ----
    double hp[Z];
    if (own) {
      K::Herr_apply(s.hv, pc, hp);
#pragma unroll
      for (int c = 0; c < Z; ++c) s.U[col * HL + c] = hp[c];  // unprojected, for S
    }
    __syncthreads();
    // S_raw[:, t] = H_err (HP_raw[t, :])^T   (P symmetric)
    if (tid < Z) {
      SmemCol<Z> hr{&s.U[tid], HL};
      double sc[Z];
      K::Herr_apply(s.hv, hr, sc);
#pragma unroll
      for (int c = 0; c < Z; ++c) s.S[c * SL + tid] = sc[c];
    }
    __syncthreads();
    if constexpr (K::HAS_HE) {
      // project S and R on both sides, y and HP on the left; S and R are handled by two different warps
      const int w = warp, t = lane;
      for (int mx = w; mx < 2; mx += nw) {
        if (t < Z) {  // columns
          double* Mx = (mx == 0) ? s.S : s.Rm;
          double u[Z];
#pragma unroll
          for (int c = 0; c < Z; ++c) u[c] = Mx[c * SL + t];
          apply_reflectors<Z, NR>(s.V, s.beta, u);
#pragma unroll
          for (int c = 0; c < Z; ++c) Mx[c * SL + t] = u[c];
        }
      }
      if (own) apply_reflectors<Z, NR>(s.V, s.beta, hp);
      __syncthreads();
      for (int mx = w; mx < 2; mx += nw) {
        if (t < Z) {  // rows
          double* Mx = (mx == 0) ? s.S : s.Rm;
          double u[Z];
#pragma unroll
          for (int c = 0; c < Z; ++c) u[c] = Mx[t * SL + c];
          apply_reflectors<Z, NR>(s.V, s.beta, u);
#pragma unroll
          for (int c = 0; c < Z; ++c) Mx[t * SL + c] = u[c];
        }
      }
      if (tid == nth - 1) {  // the innovation (the last thread has no column when E is not a multiple of 32)
        double u[Z];
#pragma unroll
        for (int c = 0; c < Z; ++c) u[c] = s.y[c];
        apply_reflectors<Z, NR>(s.V, s.beta, u);
#pragma unroll
        for (int c = 0; c < Z; ++c) s.y[c] = u[c];
      }
      __syncthreads();
    }
    // from here on only the trailing Y x Y block / Y entries are used (offset NR)

    // ---- factor S + R = L D L^T by warp 0: lane j < Y = column j, lane Y carries y through the same eliminations
    //      (so it ends as L^-1 y: the Mahalanobis distance and the state correction need nothing else).  The loop over
    //      pivots is fully unrolled: register arrays are indexed statically and only rows below the pivot are touched.
    //      Gate (ekf_c.c:88-94): if y^T S^-1 y exceeds the threshold, R is inflated by 1e16 and the factorisation redone.
    if (tid < 32) {
      const int j = tid < Y ? tid : 0;
      double A0[Y], A1[K::MAHA ? Y : 1];
#pragma unroll
      for (int i = 0; i < Y; ++i) {
        const double sv = s.S[(NR + i) * SL + NR + j], rv = s.Rm[(NR + i) * SL + NR + j], yv = s.y[NR + i];
        A0[i] = (tid == Y) ? yv : sv + rv;
        if constexpr (K::MAHA) A1[i] = (tid == Y) ? yv : fma(1.0e16, rv, sv);   // ekf_c.c:92
      }
      __syncwarp();   // S is dead from here: its storage becomes LT
      double* LT = s.S;
#pragma unroll 1
      for (int pass = 0; pass < (K::MAHA ? 2 : 1); ++pass) {
        double A[Y];
#pragma unroll
        for (int i = 0; i < Y; ++i) A[i] = (K::MAHA && pass == 1) ? A1[K::MAHA ? i : 0] : A0[i];
#pragma unroll
        for (int kk = 0; kk < Y; ++kk) {
          // the pivot's reciprocal (the long pole of a step) starts from a register shuffle, before the column's round
          // trip through shared memory
          const double di = 1.0 / __shfl_sync(0xffffffffu, A[kk], kk);
          if (tid == kk) {   // lane kk publishes its (unscaled) column: rows kk .. Y-1
#pragma unroll
            for (int i = kk; i < Y; ++i) LT[kk * SL + i] = A[i];
            s.dinv[kk] = di;
          }
          __syncwarp();
          // L[lane][kk] = c[lane] / D[kk] (symmetry: c[lane] is the lane's own A[kk]); the y lane uses its own entry
          const double cj = ((tid == Y) ? A[kk] : LT[kk * SL + j]) * di;
#pragma unroll
          for (int i = kk + 1; i < Y; ++i) A[i] = fma(-LT[kk * SL + i], cj, A[i]);
        }
        __syncwarp();
        bool gate = false;
        if (tid == Y) {
          double d = 0.0;   // y^T S^-1 y = sum_k (L^-1 y)_k^2 / D_k
#pragma unroll
          for (int i = 0; i < Y; ++i) { d = fma(A[i] * s.dinv[i], A[i], d); s.yt[i] = A[i]; }
          gate = K::MAHA && pass == 0 && d > K::MAHA_THRESH;
          if (gate) s.gated = 1;
        }
        gate = __shfl_sync(0xffffffffu, (int)gate, Y) != 0;
        if (!gate) break;
        __syncwarp();
      }
    }
    __syncthreads();

    // ---- U[:, col] = L^-1 (A^T H_err P)[:, col]; state correction dx = U^T D^-1 (L^-1 y) ----
    if (own) {
      const double* LT = s.S;
      double u[Y];
#pragma unroll
      for (int c = 0; c < Y; ++c) u[c] = hp[NR + c];
#pragma unroll
      for (int kk = 0; kk < Y; ++kk) {
        const double uk = u[kk] * s.dinv[kk];
#pragma unroll
        for (int i = kk + 1; i < Y; ++i) u[i] = fma(-LT[kk * SL + i], uk, u[i]);
      }
      double d0 = 0.0, d1 = 0.0;
#pragma unroll
      for (int c = 0; c < Y; c += 2) {
        d0 = fma(u[c] * s.dinv[c], s.yt[c], d0);
        if (c + 1 < Y) d1 = fma(u[c + 1] * s.dinv[c + 1], s.yt[c + 1], d1);
      }
      s.dx[col] = d0 + d1;
#pragma unroll
      for (int c = 0; c < HL; ++c) s.U[col * HL + c] = (c < Y) ? u[c < Y ? c : 0] : 0.0;
    }
    __syncthreads();
    // ---- P -= U^T D^-1 U on the FP64 tensor path: lower-triangle 8 x 8 tiles only, k = Y padded to a multiple of 4 ----
    {
      constexpr int NTE = (E + 7) / 8, NKY = HL / 4;
      const int fg = lane >> 2, ft = lane & 3;
      double nd[NKY];   // -1 / D[k] for this lane's k of every k-step
#pragma unroll
      for (int kq = 0; kq < NKY; ++kq) nd[kq] = -s.dinv[kq * 4 + ft];
      // lower-triangle tiles (mi >= ni) dealt to the warps round-robin in packed order: tile t = tri(mi) + ni goes to warp t % NW
      constexpr int NW = cta_threads<M>() / 32;
      for (int mi = 0; mi < NTE; ++mi)
      for (int ni = ((warp - mi * (mi + 1) / 2) % NW + NW) % NW; ni <= mi; ni += NW) {
        const int r = mi * 8 + fg, c = ni * 8 + 2 * ft, n = ni * 8 + fg;
        const bool ok0 = r < E && c <= r, ok1 = r < E && c + 1 <= r;   // inside the matrix and the lower triangle
        const int p0 = r * (r + 1) / 2 + c;
        double c0 = ok0 ? s.Ppk[p0] : 0.0;
        double c1 = ok1 ? s.Ppk[p0 + 1] : 0.0;
        double av[NKY], bv[NKY];
#pragma unroll
        for (int kq = 0; kq < NKY; ++kq) {
          av[kq] = (r < E) ? s.U[r * HL + kq * 4 + ft] * nd[kq] : 0.0;   // A[m][k] = -U[k][m] / D[k]
          bv[kq] = (n < E) ? s.U[n * HL + kq * 4 + ft] : 0.0;            // B[k][n] = U[k][n]
        }
#pragma unroll
        for (int kq = 0; kq < NKY; ++kq) dmma884(c0, c1, av[kq], bv[kq]);
        if (ok0) s.Ppk[p0] = c0;
        if (ok1) s.Ppk[p0 + 1] = c1;
      }
    }
    __syncthreads();
    const bool last = (o == a.n_obs - 1);
    aug = (a.flags & FLAG_AUGMENT) && last && M::EAUG > 0;
    // state injection, normalisation and the small outputs by warp 0 while the other warps start writing P back
    if (tid < 32) {
      M::err_fun(s.x, s.dx, a.gv, s.xo);   // every lane evaluates the small generated function; identical values
      __syncwarp();
      if ((a.flags & FLAG_NORM_AFTER_UPDATE) && a.n_quat > 0) {
        if (tid < a.n_quat) normalize4(s.xo + a.quat_idx[tid]);
        __syncwarp();
      }
      for (int i = tid; i < D; i += 32) {
        const double v = s.xo[i];
        if (last) {
          // fused augment (ekf_sym.py:368-370): [main | clone_1 .. clone_N] -> [main | clone_2 .. clone_N | main[:DAUG]]
          const int si = (!aug || i < M::DMAIN) ? i : (i < D - M::DAUG ? i + M::DAUG : i - (D - M::DAUG));
          a.x[fb * D + i] = s.xo[si];
        }
        const_cast<double*>(ws_all)[b * W::SIZE + W::OFF_X + i] = v;  // next observation of this batch starts here
        if (last && a.hx_filt) a.hx_filt[fb * D + i] = v;              // the history keeps the estimate BEFORE the window shifts (ekf_sym.py:523-528)
      }
      // innovation overwrites z (ekf_c.c:120): the first YDIM entries
      for (int i = tid; i < Y; i += 32) a.z[(b * a.n_obs + o) * Z + i] = s.y[NR + i];
    }
    if (last && a.hP_filt) store_full(a.hP_filt + fb * (long long)(E * E));
  }

  if (!aug) {
    store_full(Pg);
  } else {
    // fused augment (ekf_sym.py:372-389): the same selection on rows and columns, src(i) = i for the main block,
    // i + EAUG for the surviving clones, i - (E - EAUG) (= the first EAUG main error states) for the new clone
    auto src = [&](int i) { return i < ME ? i : (i < E - M::EAUG ? i + M::EAUG : i - (E - M::EAUG)); };
    for (int i = warp; i < E; i += nw) {
      const int sr = src(i);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int j = lane + 32 * c;
        if (j < E) Pg[i * E + j] = s.Ppk[pk_idx(sr, src(j))];
      }
    }
  }
}

template <class M, class K, bool PRED, bool UPD>
inline void launch_step_cta(const StepArgs<M::NG>& a, cudaStream_t st) {
  using W = CtaWs<M, K>;
  // leaf-value workspace of THIS call, allocated and released in stream order (calls on different streams / devices
  // never share it)
  double* ws = (double*)stream_alloc(sizeof(double) * (size_t)a.B * W::SIZE, st, "cudaMallocAsync(cta workspace)");
  if (!ws) return;
  constexpr size_t smem = sizeof(CtaSmem<M, K>);
  if (first_launch_of((const void*)ekf_step_cta<M, K, PRED, UPD>))
    check(cudaFuncSetAttribute(ekf_step_cta<M, K, PRED, UPD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "smem attribute");
  if (first_launch_of((const void*)ekf_step_cta<M, K, false, UPD>))
    check(cudaFuncSetAttribute(ekf_step_cta<M, K, false, UPD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "smem attribute");
  constexpr int threads = cta_threads<M>();
  const int n_obs = UPD ? a.n_obs : 1;
  for (int o = 0; o < n_obs; ++o) {
    const unsigned lgrid = (unsigned)((a.B + 63) / 64);
    if (o == 0) {
      ekf_leaf_thread<M, K, PRED, UPD><<<lgrid, 64, 0, st>>>(a, o, ws);
      ekf_step_cta<M, K, PRED, UPD><<<(unsigned)a.B, threads, smem, st>>>(a, o, ws);
    } else {
      ekf_leaf_thread<M, K, false, UPD><<<lgrid, 64, 0, st>>>(a, o, ws);
      ekf_step_cta<M, K, false, UPD><<<(unsigned)a.B, threads, smem, st>>>(a, o, ws);
    }
  }
  check(cudaFreeAsync(ws, st), "cudaFreeAsync(cta workspace)");
}

}  // namespace rnb
