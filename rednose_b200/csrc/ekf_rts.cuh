// rednose_b200 -- batched Rauch-Tung-Striebel backward pass (warp-per-filter, MEDIM <= 32).
//
// Reference: EKF_sym.rts_smooth, rednose/helpers/ekf_sym.py:651-690 (Python + numpy, one filter).  Per
// filter the recursion over the stored history is strictly sequential, so one warp walks one filter's
// history backwards while the batch supplies the parallelism.  For k = T-2 .. 0 (n = MEDIM main block):
//
//   F   = F_fun(x_{k|k}, t_{k+1} - t_k)                                         :672-673
//   C   = ( P_{k+1|k}^-1  F P_{k|k}^T )^T                                       :677
//   d   = inv_err_fun(x_{k+1|k}, x_{k+1|N});  d[:n] = C d[:n]                   :679-681
//   x_{k|N}[:dim_main] = err_fun(x_{k|k}, d)[:dim_main]                         :682-684
//   P_{k|N}[:n,:n] = P_{k|k} + C (P_{k+1|N} - P_{k+1|k}) C^T                    :686
//
// with the reference's quirks kept: the recursion starts from the PREDICTED last state
// (:658-659), and with norm_quats every smoothed state that is used as x_{k+1|N} has its
// quaternion normalised in place, i.e. all outputs except index 0 (:666-667).
//
// Mapping: lane j owns column j of the symmetric n x n matrices.
//   G = F P_{k|k}           lane-local (generated sparse MODEL::F_apply on the column)
//   P_{k+1|k} = L D L^T     right-looking LDL^T across lanes; column k of L is broadcast through
//                           shared memory (stored transposed so rows are read with 128-bit loads)
//   X = P_{k+1|k}^-1 G      forward / backward substitution, lane-local on the lane's column of G
//   C = X^T, so  C d = X^T d is a lane-local dot product and
//   C dP C^T = X^T (dP X):  two dense n x n x n products with one operand broadcast from shared memory.
// The smoothed covariance P_{k+1|N} is carried in registers between steps; per step the kernel
// reads P_{k+1|k}, P_{k|k} and writes P_{k|N}: 3 EDIM^2 + 3 DIM doubles (SURVEY.md section 8d).
//
// Above EDIM 32 (an MSCKF, whose main block is at most 32 wide) a lane cannot own a column of the full covariance: lanes
// < MEDIM read and write only the main block (row stride EDIM), other lanes load no covariance, and the rest of Ps[k] is
// P_{k|k} before the launch (in place, or copied there by batch_rts): 3 MEDIM^2 + 3 DIM doubles per step.  Only whole and
// segment histories in the full layout are smoothed there.
#pragma once
#include "ekf_common.cuh"
#include "ekf_warp.cuh"
#include "ekf_packed.cuh"

namespace rnb {

// Covariance slabs (hP_pred, hP_filt, Ps, P_term) are full [.., EDIM, EDIM] or, in the kernels' PH (packed history)
// instantiations, [.., packed_doubles(EDIM)] in the layout of ekf_packed.cuh.
template <int NG>
struct RtsArgs {
  const double* hx_pred;  // [T, B, DIM]         x_{k|k-1}
  const double* hP_pred;  // [T, B, EDIM, EDIM]  P_{k|k-1}
  const double* hx_filt;  // [T, B, DIM]         x_{k|k}
  const double* hP_filt;  // [T, B, EDIM, EDIM]  P_{k|k}
  const double* t;        // [T] or [T, B] observation times
  int t_per_filter;
  double* xs;             // [T, B, DIM]         smoothed states (may alias hx_filt)
  double* Ps;             // [T, B, EDIM, EDIM]  smoothed covariances (may alias hP_filt)
  int T;
  long long B;
  int norm_quats;
  int n_quat;
  int quat_idx[MAX_QUAT];
  // segment continuation (checkpointed smoothing of long histories): when x_term / P_term are given, the slabs hold
  // the steps k0 .. k0 + T - 1 of a longer history, entry T - 1 only contributes its PREDICTED state, and the recursion
  // starts from x_term [B, DIM] / P_term [B, EDIM, EDIM] = the smoothed estimate of step k0 + T - 1 produced by the
  // segment behind it (instead of the reference's start from the predicted last state, ekf_sym.py:658-659); entry T - 1
  // of xs / Ps is then not written.  k0 only decides which outputs get their quaternion normalised (all but global
  // index 0, ekf_sym.py:666-667).
  const double* x_term;
  const double* P_term;
  long long k0;
  double gv[NG > 0 ? NG : 1];
  // ragged histories: filter b smooths rows 0 .. len[b] - 1 only (with t [T, B]) and leaves its rows >= len[b] of xs / Ps
  // untouched; nullptr = every filter has T rows.  Combined with segment continuation only through RaggedSeg (below).
  const int* len;
  // M = MainHist<model> (EDIM > 32): hP_pred is [T, B, MEDIM, MEDIM], the main block of each P_{k|k-1}, and the recursion
  // starts (without x_term / P_term) from this [B, EDIM, EDIM] full P_{T-1|T-2}
  const double* hP_pred_last;
  // M = RaggedSeg<model> (a ragged history holding one segment of each filter's rows, with len): term[b] != 0 makes row
  // len[b] - 1 of filter b the first row of its segment behind, which contributes only its predicted state and time, and
  // the recursion of filter b starts from x_term[b] / P_term[b], the smoothed estimate of that row (row len[b] - 1 of
  // xs / Ps is then not written); term[b] == 0 smooths filter b as a whole ragged history does.  k0s[b] is the global
  // row index of filter b's row 0 (normalisation: every output but global row 0).  Read only by those instantiations.
  const unsigned char* term;
  const long long* k0s;
};

// rows filter b smooths: T, or len[b] clamped to [0, T] for a ragged history
template <bool RAGGED, int NG>
__device__ __forceinline__ long long rts_rows(const RtsArgs<NG>& a, long long b) {
  if constexpr (!RAGGED) return a.T;
  const long long n = a.len[b];
  return n < 0 ? 0 : (n > a.T ? a.T : n);
}

// Elements (r, c), (r, c + 1), c even, of a packed covariance Pb, read the way the pair kernel reads its tiles: P is
// defined by its lower triangle.  Below the block diagonal the pair is one 128-bit load of block (r / 2, c / 2); above it
// it is the transposed pair, column r of block (c / 2, r / 2); on a diagonal block the upper element is its lower mirror.
__device__ __forceinline__ double2 packed_pair(const double* Pb, int r, int c) {
  const int R = r >> 1, C = c >> 1;
  if (R > C) return *reinterpret_cast<const double2*>(Pb + packed_block(R, C) + 2 * (r & 1));
  if (R < C) {
    const double* q = Pb + packed_block(C, R) + (r & 1);
    return make_double2(q[0], q[2]);
  }
  const double* q = Pb + packed_block(R, R);
  return (r & 1) ? *reinterpret_cast<const double2*>(q + 2) : make_double2(q[0], q[2]);
}

constexpr int RTS_WARPS = 2;
constexpr int RTS_MIN_CTAS = 6;

template <class M>
struct RtsScratch {
  static constexpr int N = M::MEDIM;
  static constexpr int LD = (N + 3) & ~1;             // even leading dimension (128-bit rows), not a multiple of 32 banks
  alignas(16) double LT[N * LD];                      // LT[k][i] = unscaled column k of the trailing matrix = D[k] L[i][k] (i >= k)
  alignas(16) double DP[N * LD];                      // dP = P_{k+1|N} - P_{k+1|k}; later X (row-major)
  // y = dP X (column per lane) lives in the LT buffer: L is dead once the substitutions are done
  alignas(16) double xf[(M::DIM + 1) & ~1];           // x_{k|k}
  alignas(16) double xp[(M::DIM + 1) & ~1];           // x_{k+1|k}
  alignas(16) double xn[(M::DIM + 1) & ~1];           // x_{k+1|N} -> x_{k|N}
  alignas(16) double xt[(M::DIM + 1) & ~1];           // err_fun output
  alignas(16) double dl[(M::EDIM + 1) & ~1];          // error-state delta
  alignas(16) double dinv[(N + 1) & ~1];              // 1 / D[k]
};

// M = PackedHist<model>: every covariance slab (hP_pred, hP_filt, Ps, P_term) is packed
template <class M, bool RAGGED = false>
__global__ void __launch_bounds__(RTS_WARPS * 32, RTS_MIN_CTAS) ekf_rts_warp(const RtsArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, N = M::MEDIM, D1 = M::DMAIN;
  constexpr bool PH = packed_hist<M>(), MH = main_hist<M>();
  using SC = RtsScratch<M>;
  constexpr int LD = SC::LD;
  static_assert(N <= 32, "warp-per-filter RTS needs MEDIM <= 32");
  static_assert(E <= 32 || (!PH && !RAGGED), "above EDIM 32 only whole and segment histories in the full layout");
  static_assert(!PH || E % 2 == 0, "the packed layout needs an even EDIM");
  static_assert(!ragged_seg<M>() || (RAGGED && E <= 32), "ragged segments are ragged histories, EDIM <= 32");
  static_assert(!MH || E > 32, "main-block prediction histories exist only above EDIM 32");
  constexpr int PS = PH ? packed_doubles(E) : E * E;   // doubles of one filter's covariance in the slabs
  constexpr int PPS = MH ? N * N : PS, PLD = MH ? N : E;   // the same, and the row stride, in the hP_pred slab
  __shared__ SC s_all[RTS_WARPS];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long b = (long long)blockIdx.x * RTS_WARPS + wib;
  if (b >= a.B) return;
  const long long T = rts_rows<RAGGED>(a, b);   // warp-uniform; the warps of a CTA never synchronise with each other
  if (RAGGED && T == 0) return;
  SC& s = s_all[wib];
  const bool act = lane < N;        // owns a column of the main block
  const bool actE = lane < E;       // owns a column of the full covariance
  const int col = actE ? lane : 0;
  const long long BP = a.B * (long long)PS, BPP = a.B * (long long)PPS, BX = a.B * (long long)D;

  auto normalize_xn = [&]() {
    for (int q = 0; q < a.n_quat; ++q) {
      double* qp = s.xn + a.quat_idx[q];
      const double nrm = sqrt(qp[0] * qp[0] + qp[1] * qp[1] + qp[2] * qp[2] + qp[3] * qp[3]);
      __syncwarp();
      if (lane < 4) qp[lane] = qp[lane] / nrm;
      __syncwarp();
    }
  };

  // ---- start: x_{T-1|N} = x_{T-1|T-2} (predicted), P likewise (ekf_sym.py:658-659) ----
  double pn[N];  // column `lane` of the carried smoothed covariance (main block)
  {
    const long long k = T - 1;
    const bool seg = ragged_seg<M>() ? a.term[b] != 0 : a.x_term != nullptr;
    if constexpr (PH) {
      const double* Pg = seg ? a.P_term + b * (long long)PS : a.hP_pred + k * BP + b * (long long)PS;
      double* Po = a.Ps + k * BP + b * (long long)PS;
#pragma unroll
      for (int i = 0; i < N; ++i) pn[i] = Pg[packed_index(i, col)];
      if (!seg) for (int t = lane; t < PS; t += 32) Po[t] = Pg[t];
    } else if constexpr (E > 32) {
      const double* Pg = seg ? a.P_term + b * (long long)(E * E)
                             : (MH ? a.hP_pred_last + b * (long long)(E * E) : a.hP_pred + k * BP + b * (long long)(E * E));
      double* Po = a.Ps + k * BP + b * (long long)(E * E);
#pragma unroll
      for (int i = 0; i < N; ++i) pn[i] = act ? Pg[i * E + lane] : 0.0;
      if (!seg) for (int t = lane; t < E * E; t += 32) Po[t] = Pg[t];
    } else {
    const double* Pg = (seg ? a.P_term + b * (long long)(E * E) : a.hP_pred + k * BP + b * (long long)(E * E)) + col;
    double* Po = a.Ps + k * BP + b * (long long)(E * E) + col;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const double v = Pg[i * E];
      if (i < N) pn[i] = v;
      if (actE && !seg) Po[i * E] = v;
    }
    }
    for (int i = lane; i < D; i += 32) s.xn[i] = seg ? a.x_term[b * D + i] : a.hx_pred[k * BX + b * D + i];
    __syncwarp();
    if (!seg) {
      if (a.norm_quats && (ragged_seg<M>() ? a.k0s[b] : a.k0) + T - 1 >= 1) normalize_xn();   // every output but global index 0, as in the loop
      for (int i = lane; i < D; i += 32) a.xs[k * BX + b * D + i] = s.xn[i];
    }
  }

#pragma unroll 1
  for (long long k = T - 2; k >= 0; --k) {
    const double* Pf_b = a.hP_filt + k * BP + b * (long long)PS;
    const double* Pp_b = a.hP_pred + (k + 1) * BPP + b * (long long)PPS;
    const double* Pf_g = Pf_b + col;
    const double* Pp_g = Pp_b + col;
    // element i of the lane's column of a covariance (row stride ld): P is defined by its lower triangle
    auto el = [&](const double* Pb, const double* Pg, int i, int ld = M::EDIM) {
      if constexpr (E > 32) return act ? Pg[i * ld] : 0.0;   // main block only
      else return PH ? Pb[packed_index(i, col)] : Pg[i * E];
    };
    double g[N];
#pragma unroll
    for (int i = 0; i < N; ++i) g[i] = el(Pf_b, Pf_g, i);
    for (int i = lane; i < D; i += 32) {
      s.xf[i] = a.hx_filt[k * BX + b * D + i];
      s.xp[i] = a.hx_pred[(k + 1) * BX + b * D + i];
    }
    const double dt = a.t_per_filter ? (a.t[(k + 1) * a.B + b] - a.t[k * a.B + b]) : (a.t[k + 1] - a.t[k]);
    __syncwarp();

    // G[:,lane] = F P_{k|k}[:,lane]   (F evaluated at the filtered state)
    {
      double fv[M::NF > 0 ? M::NF : 1];
      M::F_vals(s.xf, dt, a.gv, fv);
      M::F_apply(fv, g);
    }
    asm volatile("" ::: "memory");  // scheduling fence: keep the next loads below the leaf code (register pressure)

    // A = column of P_{k+1|k};  dP column = P_{k+1|N} - P_{k+1|k} (pn is dead afterwards)
    double A[N];
#pragma unroll
    for (int i = 0; i < N; ++i) A[i] = el(Pp_b, Pp_g, i, PLD);
    if (act) {
#pragma unroll
      for (int i = 0; i < N; ++i) s.DP[i * LD + lane] = pn[i] - A[i];
    }

    // ---- P_{k+1|k} = L D L^T : right-looking, one (unscaled) column broadcast per step.  The outer loop is
    //      NOT unrolled (code size); register arrays are only indexed statically: lane kk publishes its
    //      column c = A_kk[:], every lane then needs c[lane] (= its own A[kk] by symmetry) and c[i]. ----
#pragma unroll 1
    for (int kk = 0; kk < N; ++kk) {
      if (lane == kk) {
#pragma unroll
        for (int i = 0; i < N; ++i) s.LT[kk * LD + i] = A[i];
      }
      __syncwarp();
      const double di = 1.0 / s.LT[kk * LD + kk];
      if (lane == 0) s.dinv[kk] = di;
      const double cj = s.LT[kk * LD + (act ? lane : 0)] * di;   // D[kk] L[lane][kk] / D[kk] ... = L[lane][kk]
      // rows i <= kk of A are final (already published) and never read again, so the update needs no
      // predicate: it may clobber them freely
#pragma unroll
      for (int i = 0; i < N; i += 2) {
        const double2 c2 = *reinterpret_cast<const double2*>(&s.LT[kk * LD + i]);
        A[i] = fma(-c2.x, cj, A[i]);
        if (i + 1 < N) A[i + 1] = fma(-c2.y, cj, A[i + 1]);
      }
    }
    __syncwarp();
    // ---- X[:,lane] = (L D L^T)^-1 G[:,lane];  L[i][kk] = LT[kk][i] * dinv[kk] ----
#pragma unroll
    for (int kk = 0; kk < N; ++kk) {
      const double gk = g[kk] * s.dinv[kk];
#pragma unroll
      for (int i = kk + 1; i < N; ++i) g[i] = fma(-s.LT[kk * LD + i], gk, g[i]);
      asm volatile("" ::: "memory");  // keep ptxas from hoisting every row of L into registers at once
    }
#pragma unroll
    for (int i = 0; i < N; ++i) g[i] *= s.dinv[i];
    // re-read L through a laundered pointer: otherwise ptxas keeps every row of L loaded by the forward sweep
    // alive in registers for the backward sweep (1.4 kB of spills); laundering keeps the 128-bit loads
    const double* LTv = s.LT;
    asm volatile("" : "+l"(LTv));
#pragma unroll
    for (int kk = N - 2; kk >= 0; --kk) {
      double acc = 0.0;
#pragma unroll
      for (int i = kk + 1; i < N; ++i) acc = fma(LTv[kk * LD + i], g[i], acc);
      g[kk] = fma(-acc, s.dinv[kk], g[kk]);
      asm volatile("" ::: "memory");
    }
    // g = X[:,lane] = row `lane` of C

    // ---- state: d = inv_err(x_{k+1|k}, x_{k+1|N}); d[:n] = C d[:n]; x_{k|N} = err(x_{k|k}, d) ----
    M::inv_err_fun(s.xp, s.xn, a.gv, s.dl);  // every lane writes identical values
    __syncwarp();
    double cd = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) cd = fma(g[i], s.dl[i], cd);
    __syncwarp();
    if (act) s.dl[lane] = cd;
    __syncwarp();
    M::err_fun(s.xf, s.dl, a.gv, s.xt);
    __syncwarp();
    for (int i = lane; i < D; i += 32) s.xn[i] = (i < D1) ? s.xt[i] : s.xf[i];
    __syncwarp();
    if (a.norm_quats && k + (ragged_seg<M>() ? a.k0s[b] : a.k0) >= 1) normalize_xn();
    for (int i = lane; i < D; i += 32) a.xs[k * BX + b * D + i] = s.xn[i];

    // ---- covariance: P_{k|N} = P_{k|k} + X^T (dP X) ----
#pragma unroll 1
    for (int i = 0; i < N; ++i) {   // y[i] = dP[i,:] . X[:,lane]
      double acc = 0.0;
#pragma unroll
      for (int c = 0; c < N; c += 2) {
        const double2 d2 = *reinterpret_cast<const double2*>(&s.DP[i * LD + c]);
        acc = fma(d2.x, g[c], acc);
        if (c + 1 < N) acc = fma(d2.y, g[c + 1], acc);
      }
      if (act) s.LT[i * LD + lane] = acc;
    }
    __syncwarp();
    if (act) {  // X row-major into the dP buffer: XS[r][lane] = X[r][lane]
#pragma unroll
      for (int i = 0; i < N; ++i) s.DP[i * LD + lane] = g[i];
    }
    __syncwarp();
    // out = P_{k|k}[:, lane] + sum_r X[r][:] y[r]
#pragma unroll
    for (int i = 0; i < N; ++i) pn[i] = el(Pf_b, Pf_g, i);
#pragma unroll 1
    for (int r = 0; r < N; ++r) {
      const double yr = s.LT[r * LD + (act ? lane : 0)];
#pragma unroll
      for (int i = 0; i < N; i += 2) {
        const double2 x2 = *reinterpret_cast<const double2*>(&s.DP[r * LD + i]);
        pn[i] = fma(x2.x, yr, pn[i]);
        if (i + 1 < N) pn[i + 1] = fma(x2.y, yr, pn[i + 1]);
      }
    }
    // lanes / rows outside the main block keep P_{k|k} (only the main block is smoothed, ekf_sym.py:686)
    if constexpr (PH) {
      // packed: the lane writes the lower part of its column, i >= col, and an even column also the upper corner of its
      // diagonal block, the mirror of element (col + 1, col)
      if (actE) {
        double* Po = a.Ps + k * BP + b * (long long)PS;
#pragma unroll
        for (int i = 0; i < E; ++i) {
          if (i >= col) {
            const double v = (act && i < N) ? pn[i < N ? i : 0] : Pf_b[packed_index(i, col)];
            Po[packed_index(i, col)] = v;
            if (i == col + 1 && !(col & 1)) Po[packed_block(col >> 1, col >> 1) + 1] = v;
          }
        }
      }
      __syncwarp();
      // carry P_{k|N} as stored, by its lower triangle (see ekf_rts_warp_mma)
      const double* Pk = a.Ps + k * BP + b * (long long)PS;
#pragma unroll
      for (int i = 0; i < N; ++i) pn[i] = Pk[packed_index(i, col)];
    } else if constexpr (E > 32) {
      if (act) {
        double* Po = a.Ps + k * BP + b * (long long)(E * E) + lane;
#pragma unroll
        for (int i = 0; i < N; ++i) Po[i * E] = pn[i];
      }
    } else {
    if (actE) {
      const double* Pfull = a.hP_filt + k * BP + b * (long long)(E * E) + col;
      double* Po = a.Ps + k * BP + b * (long long)(E * E) + col;
#pragma unroll
      for (int i = 0; i < E; ++i) Po[i * E] = (act && i < N) ? pn[i < N ? i : 0] : Pfull[i * E];
    }
    }
    __syncwarp();
  }
}

// PH: the covariance slabs are packed (only instantiated for an even EDIM <= 32).  Above EDIM 32 the rest of Ps outside
// the main block must already hold P_{k|k} (batch_rts), and ragged histories are refused by their caller.
template <class M, bool PH = false>
inline void launch_rts(const RtsArgs<M::NG>& a, cudaStream_t st) {
  if (a.B <= 0 || a.T <= 0) return;
  if constexpr (M::EDIM > 32 && M::MEDIM <= 32 && !PH) {
    ekf_rts_warp<M><<<(unsigned)((a.B + RTS_WARPS - 1) / RTS_WARPS), RTS_WARPS * 32, 0, st>>>(a);
    check(cudaGetLastError(), "ekf_rts launch");
  } else if constexpr (M::EDIM <= 32) {
    const unsigned grid = (unsigned)((a.B + RTS_WARPS - 1) / RTS_WARPS);
    if constexpr (PH) {
      if (a.len) ekf_rts_warp<PackedHist<M>, true><<<grid, RTS_WARPS * 32, 0, st>>>(a);
      else ekf_rts_warp<PackedHist<M>><<<grid, RTS_WARPS * 32, 0, st>>>(a);
    } else {
      if (a.len) ekf_rts_warp<M, true><<<grid, RTS_WARPS * 32, 0, st>>>(a);
      else ekf_rts_warp<M><<<grid, RTS_WARPS * 32, 0, st>>>(a);
    }
    check(cudaGetLastError(), "ekf_rts launch");
  } else {
    fprintf(stderr, "[rednose_b200] batched RTS for EDIM=%d, MEDIM=%d is not built into this library\n", M::EDIM, M::MEDIM);
    last_status() = (int)cudaErrorNotSupported;
  }
}

}  // namespace rnb
