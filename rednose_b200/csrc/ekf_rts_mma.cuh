// rednose_b200 -- RTS backward pass, variant whose two dense n x n x n products run on the FP64 tensor path
// (mma.sync.aligned.m8n8k4.f64, SASS DMMA).  Same recursion, same factorisation / substitution code as
// ekf_rts_warp (ekf_rts.cuh); only  P_{k|N} = P_{k|k} + X^T (dP X)  changes:
//
//   * the scalar version broadcasts every row of dP and of X to all lanes from shared memory (2 wavefronts per
//     128-bit broadcast load): ~1000 of the ~2000 L1TEX wavefronts per step, the kernel's limiter (72 % of the
//     shared-memory pipe at 15 % of the HBM roofline);
//   * here dP, X and Y = dP X are read as m8n8k4 fragments (one 64-bit element per lane, 36 loads per product
//     instead of 242) and the smoothed covariance is carried between steps in accumulator-fragment layout
//     (row = lane / 4, columns 2 (lane % 4) + {0, 1} of every 8 x 8 tile), which is also the layout it is
//     loaded from / stored to global memory in (aligned 128-bit accesses).
//
// n is padded to a multiple of 8 with zeros (22 -> 24 for live_kf).  FP64 mma is IEEE fused multiply-add, so
// results agree with the scalar kernel to rounding (different summation order).  Above EDIM 32 (an MSCKF) only the main
// block of the slabs is read and written, as in ekf_rts_warp.
#pragma once
#include <type_traits>
#include "ekf_rts.cuh"

namespace rnb {

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

template <class M>
struct RtsMmaScratch {
  static constexpr int N = M::MEDIM;
  static constexpr int NP = (N + 7) & ~7;             // padded extent
  static constexpr int LD = (N + 3) & ~1;             // factor buffer (as in the scalar kernel)
  static constexpr int LP = NP + 2;                   // fragment buffers: even (128-bit rows), spreads rows over banks
  alignas(16) double LT[(N * LD > NP * LP) ? N * LD : NP * LP];   // L during the solve, then Y = dP X
  alignas(16) double DP[NP * LP];                     // dP, row-major, zero padded
  alignas(16) double XS[NP * LP];                     // X, row-major, zero padded
  alignas(16) double xf[(M::DIM + 1) & ~1];
  alignas(16) double xp[(M::DIM + 1) & ~1];
  alignas(16) double xn[(M::DIM + 1) & ~1];
  alignas(16) double xt[(M::DIM + 1) & ~1];
  alignas(16) double dl[(M::EDIM + 1) & ~1];
  alignas(16) double dinv[(N + 1) & ~1];
};

// M = PackedHist<model>: every covariance slab is packed (ekf_packed.cuh); fragments are read with packed_pair and only
// the lower blocks of Ps are written
template <class M, bool RAGGED = false>
__global__ void __launch_bounds__(RTS_WARPS * 32, RTS_MIN_CTAS) ekf_rts_warp_mma(const RtsArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, N = M::MEDIM, D1 = M::DMAIN;
  constexpr bool PH = packed_hist<M>(), MH = main_hist<M>();
  using SC = RtsMmaScratch<M>;
  constexpr int LD = SC::LD, NP = SC::NP, LP = SC::LP, NT = NP / 8, NK = NP / 4;
  static_assert(E % 2 == 0 && N <= 32, "fragment I/O needs an even EDIM and MEDIM <= 32");
  static_assert(E <= 32 || (!PH && !RAGGED), "above EDIM 32 only whole and segment histories in the full layout");
  static_assert(!MH || E > 32, "main-block prediction histories exist only above EDIM 32");
  static_assert(!ragged_seg<M>() || (RAGGED && E <= 32), "ragged segments are ragged histories, EDIM <= 32");
  constexpr int PS = PH ? packed_doubles(E) : E * E;   // doubles of one filter's covariance in the slabs
  constexpr int PPS = MH ? N * N : PS, PLD = MH ? N : E;   // the same, and the row stride, in the hP_pred slab
  // dynamic: from a main block of 25 (NP = 32) the RTS_WARPS scratch blocks pass the 48 KB static limit
  extern __shared__ __align__(16) unsigned char rts_smem_raw[];
  SC* s_all = reinterpret_cast<SC*>(rts_smem_raw);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long b = (long long)blockIdx.x * RTS_WARPS + wib;
  if (b >= a.B) return;
  const long long T = rts_rows<RAGGED>(a, b);   // warp-uniform; the warps of a CTA never synchronise with each other
  if (RAGGED && T == 0) return;
  SC& s = s_all[wib];
  const bool act = lane < N, actE = lane < E;
  const int col = actE ? lane : 0;
  const int fg = lane >> 2, ft = lane & 3;   // fragment coordinates: row fg, k / column pair ft
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
  // element pair (r, c), (r, c+1) of tile (mi, ni) in accumulator layout
  auto frag_rc = [&](int mi, int ni, int& r, int& c) { r = mi * 8 + fg; c = ni * 8 + 2 * ft; };
  // elements (r, c), (r, c + 1) of the covariance at Pb (row stride ld)
  auto pair_at = [&](const double* Pb, int r, int c, int ld = M::EDIM) {
    if constexpr (PH) return packed_pair(Pb, r, c);
    else return *reinterpret_cast<const double2*>(Pb + r * ld + c);
  };
  // elements (r, c), (r, c + 1) of P_{k+1|k}.  A main-block slab of odd MEDIM (an even EDIM with position clones, EAUG 3)
  // has rows of odd length: its pairs are not 16-byte aligned, and (r, MEDIM) is not in the row.  That element only
  // meets the zero padding of X (row MEDIM), so 0 stands in for it; the products come out as from the full slab.
  auto pred_pair = [&](const double* Pb, int r, int c) {
    if constexpr (MH && N % 2 == 1) return make_double2(Pb[r * N + c], c + 1 < N ? Pb[r * N + c + 1] : 0.0);
    else return pair_at(Pb, r, c, PLD);
  };

  // ---- start: smoothed = predicted at T-1 (ekf_sym.py:658-659); carried in fragment layout ----
  double pn[NT * NT * 2];
  {
    const long long k = T - 1;
    const bool seg = ragged_seg<M>() ? a.term[b] != 0 : a.x_term != nullptr;   // segment continuation: start from the smoothed estimate handed in
    const double* Pg = seg ? a.P_term + b * (long long)PS
                           : (MH ? a.hP_pred_last + b * (long long)PS : a.hP_pred + k * BP + b * (long long)PS);
    double* Po = a.Ps + k * BP + b * (long long)PS;
    if (!seg) for (int idx = lane; idx < PS; idx += 32) Po[idx] = Pg[idx];
#pragma unroll
    for (int mi = 0; mi < NT; ++mi)
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        int r, c; frag_rc(mi, ni, r, c);
        double2 v = make_double2(0.0, 0.0);
        if (r < N && c < N) v = pair_at(Pg, r, c);
        pn[(mi * NT + ni) * 2] = v.x; pn[(mi * NT + ni) * 2 + 1] = v.y;
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
    // every global load of the step is issued here, before any dependent work (one latency round trip per step)
    double g[N], A[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if constexpr (PH) { g[i] = Pf_b[packed_index(i, col)]; A[i] = Pp_b[packed_index(i, col)]; }   // lower triangle
      else if constexpr (E > 32) { g[i] = act ? Pf_g[i * E] : 0.0; A[i] = act ? Pp_g[i * PLD] : 0.0; }   // main block only
      else { g[i] = Pf_g[i * E]; A[i] = Pp_g[i * E]; }
    }
    // P_{k|k} once more, in accumulator layout (the C operand of the last product): fetched here with everything
    // else -- inside the product loop each tile's load sat behind the previous tile's store to Ps (may alias) and
    // paid its own L2 round trip
    double pf[NT * NT * 2];
#pragma unroll
    for (int mi = 0; mi < NT; ++mi)
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        int r, c; frag_rc(mi, ni, r, c);
        double2 v = make_double2(0.0, 0.0);
        if (r < N && c < N) v = pair_at(Pf_b, r, c);
        pf[(mi * NT + ni) * 2] = v.x; pf[(mi * NT + ni) * 2 + 1] = v.y;
      }
    // the next step's history slabs go into L2 while this step computes
    if constexpr (E > 32) {   // the main block's rows: lane r touches every 128-byte line of row r (points <= 16 doubles apart)
      auto prefetch_row = [&](const double* r) {
#pragma unroll
        for (int o = 0; o < N; o += 16) prefetch_l2(r + o);
        prefetch_l2(r + N - 1);
      };
      if (k > 0 && act) {
        prefetch_row(Pf_b - BP + lane * E);
        prefetch_row(a.hP_pred + k * BPP + b * (long long)PPS + lane * PLD);
      }
      if (k > 0 && lane < (D - 1) / 16 + 2) {   // x rows likewise: points at most 16 doubles apart, the last one included
        const int xo = lane * 16 < D ? lane * 16 : D - 1;
        prefetch_l2(a.hx_filt + (k - 1) * BX + b * D + xo);
        prefetch_l2(a.hx_pred + k * BX + b * D + xo);
      }
    } else if (k > 0) {   // step k-1 reads P_{k-1|k-1}, P_{k|k-1}, x_{k-1|k-1}, x_{k|k-1}: one 128-byte line per lane
      constexpr int TB = PS * (int)sizeof(double);
      const int off = (lane * 128 < TB - 8) ? lane * 128 : TB - 8;
      prefetch_l2(reinterpret_cast<const char*>(Pf_b - BP) + off);
      prefetch_l2(reinterpret_cast<const char*>(a.hP_pred + k * BP + b * (long long)PS) + off);
      if (lane < 2) {
        constexpr int XB = D * (int)sizeof(double);
        const int xo = (lane * 128 < XB - 8) ? lane * 128 : XB - 8;
        prefetch_l2(reinterpret_cast<const char*>(a.hx_filt + (k - 1) * BX + b * D) + xo);
        prefetch_l2(reinterpret_cast<const char*>(a.hx_pred + k * BX + b * D) + xo);
      }
    }
    // dP = P_{k+1|N} - P_{k+1|k} in fragment layout -> shared memory (zero padded)
#pragma unroll
    for (int mi = 0; mi < NT; ++mi)
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        int r, c; frag_rc(mi, ni, r, c);
        double2 v = make_double2(0.0, 0.0);
        if (r < N && c < N) {
          const double2 pp = pred_pair(Pp_b, r, c);
          v.x = pn[(mi * NT + ni) * 2] - pp.x;
          v.y = pn[(mi * NT + ni) * 2 + 1] - pp.y;
        }
        *reinterpret_cast<double2*>(&s.DP[r * LP + c]) = v;
      }

    for (int i = lane; i < D; i += 32) {
      s.xf[i] = a.hx_filt[k * BX + b * D + i];
      s.xp[i] = a.hx_pred[(k + 1) * BX + b * D + i];
    }
    const double dt = a.t_per_filter ? (a.t[(k + 1) * a.B + b] - a.t[k * a.B + b]) : (a.t[k + 1] - a.t[k]);
    __syncwarp();
    {
      double fv[M::NF > 0 ? M::NF : 1];
      M::F_vals(s.xf, dt, a.gv, fv);
      M::F_apply(fv, g);   // G[:,lane] = F P_{k|k}[:,lane]
    }

    // ---- P_{k+1|k} = L D L^T, right-looking, FULLY UNROLLED: register arrays are indexed statically, only the rows
    //      below the pivot are published / updated (231 instead of 484 FMAs), and the reciprocal of the pivot -- the long
    //      pole of every step -- is started from a register shuffle BEFORE the column makes its round trip through shared
    //      memory, so the two latencies overlap instead of adding up. ----
#pragma unroll
    for (int kk = 0; kk < N; ++kk) {
      const double piv = __shfl_sync(0xffffffffu, A[kk], kk);   // lane kk's diagonal entry is final
      const double di = 1.0 / piv;
      if (lane == kk) {   // publish the (unscaled) column below the pivot; rows <= kk of this buffer row are never read
#pragma unroll
        for (int i = kk + 1; i < N; ++i) s.LT[kk * LD + i] = A[i];
        s.dinv[kk] = di;
      }
      __syncwarp();
      // L[lane][kk] = c[lane] / D[kk]: read from the published column (not the lane's own A[kk]) so that L is exactly
      // the factor the substitutions below use; lanes <= kk own finished columns and update nothing
      const double cj = ((lane > kk && act) ? s.LT[kk * LD + lane] : 0.0) * di;
#pragma unroll
      for (int i = kk + 1; i < N; ++i) A[i] = fma(-s.LT[kk * LD + i], cj, A[i]);
    }
    __syncwarp();
    // ---- X[:,lane] = (L D L^T)^-1 G[:,lane];  L[i][kk] = LT[kk][i] * dinv[kk] ----
#pragma unroll
    for (int kk = 0; kk < N; ++kk) {
      const double gk = g[kk] * s.dinv[kk];
#pragma unroll
      for (int i = kk + 1; i < N; ++i) g[i] = fma(-s.LT[kk * LD + i], gk, g[i]);
      asm volatile("" ::: "memory");
    }
#pragma unroll
    for (int i = 0; i < N; ++i) g[i] *= s.dinv[i];
    const double* LTv = s.LT;
    asm volatile("" : "+l"(LTv));
#pragma unroll
    for (int kk = N - 2; kk >= 0; --kk) {
      double acc0 = 0.0, acc1 = 0.0;   // two partial sums: half the dependent-FMA chain of the dot product
#pragma unroll
      for (int i = kk + 1; i < N; i += 2) {
        acc0 = fma(LTv[kk * LD + i], g[i], acc0);
        if (i + 1 < N) acc1 = fma(LTv[kk * LD + i + 1], g[i + 1], acc1);
      }
      g[kk] = fma(-(acc0 + acc1), s.dinv[kk], g[kk]);
      asm volatile("" ::: "memory");
    }
    // g = X[:,lane]

    // ---- state ----
    M::inv_err_fun(s.xp, s.xn, a.gv, s.dl);
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

    // ---- X into shared memory, row-major, zero padded (lane j writes column j) ----
    if (lane < NP) {
#pragma unroll
      for (int i = 0; i < NP; ++i) s.XS[i * LP + lane] = (act && i < N) ? g[i < N ? i : 0] : 0.0;
    }
    __syncwarp();

    // X fragments (B operand of dP X, and A operand of X^T Y): xb[kq][t] = X[kq*4 + ft][t*8 + fg]
    double xb[NK][NT];
#pragma unroll
    for (int kq = 0; kq < NK; ++kq)
#pragma unroll
      for (int t = 0; t < NT; ++t) xb[kq][t] = s.XS[(kq * 4 + ft) * LP + t * 8 + fg];

    // ---- Y = dP X  (accumulator fragments), then to shared memory (L's buffer: L is dead) ----
#pragma unroll
    for (int mi = 0; mi < NT; ++mi) {
      double ad[NK];
#pragma unroll
      for (int kq = 0; kq < NK; ++kq) ad[kq] = s.DP[(mi * 8 + fg) * LP + kq * 4 + ft];
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        double c0 = 0.0, c1 = 0.0;
#pragma unroll
        for (int kq = 0; kq < NK; ++kq) dmma884(c0, c1, ad[kq], xb[kq][ni]);
        int r, c; frag_rc(mi, ni, r, c);
        *reinterpret_cast<double2*>(&s.LT[r * LP + c]) = make_double2(c0, c1);
      }
    }
    __syncwarp();

    // ---- P_{k|N} = P_{k|k} + X^T Y : A[m][k] = X[k][m] = xb[kq][mi], B[k][n] = Y[k][n] ----
#pragma unroll
    for (int ni = 0; ni < NT; ++ni) {
      double yb[NK];
#pragma unroll
      for (int kq = 0; kq < NK; ++kq) yb[kq] = s.LT[(kq * 4 + ft) * LP + ni * 8 + fg];
#pragma unroll
      for (int mi = 0; mi < NT; ++mi) {
        int r, c; frag_rc(mi, ni, r, c);
        double c0 = pf[(mi * NT + ni) * 2], c1 = pf[(mi * NT + ni) * 2 + 1];
#pragma unroll
        for (int kq = 0; kq < NK; ++kq) dmma884(c0, c1, xb[kq][mi], yb[kq]);
        pn[(mi * NT + ni) * 2] = c0; pn[(mi * NT + ni) * 2 + 1] = c1;
        if constexpr (PH) {
          // lower blocks only: below the block diagonal one 128-bit store; on a diagonal block row r + 1 stores the
          // block's lower row and, into the upper corner, the mirror of its element (r + 1, r); row r stores (r, r)
          if (r < N && c < N && (r >> 1) >= (c >> 1)) {
            double* q = a.Ps + k * BP + b * (long long)PS + packed_block(r >> 1, c >> 1);
            if ((r >> 1) > (c >> 1) || (r & 1)) *reinterpret_cast<double2*>(q + 2 * (r & 1)) = make_double2(c0, c1);
            else q[0] = c0;
            if ((r >> 1) == (c >> 1) && (r & 1)) q[1] = c0;
          }
        } else {
          if (r < N && c < N) *reinterpret_cast<double2*>(a.Ps + k * BP + b * (long long)(E * E) + r * E + c) = make_double2(c0, c1);
        }
      }
    }
    // rows / columns outside the main block keep P_{k|k} (ekf_sym.py:686 smooths the main block only)
    if constexpr (E > N && E <= 32) {   // above 32 batch_rts leaves P_{k|k} there before the launch
      double* Po = a.Ps + k * BP + b * (long long)PS;
      for (int idx = lane; idx < PS; idx += 32) {
        int i, j;
        if constexpr (PH) packed_element(E, idx, i, j);
        else { i = idx / E; j = idx - i * E; }
        if (i >= N || j >= N) Po[idx] = Pf_b[idx];
      }
    }
    __syncwarp();
    if constexpr (PH) {
      // carry P_{k|N} as stored, by its lower triangle: the next step (or the segment smoothed after this one, from its
      // terminal estimate) then starts from the same matrix, bit for bit
      const double* Pk = a.Ps + k * BP + b * (long long)PS;
#pragma unroll
      for (int mi = 0; mi < NT; ++mi)
#pragma unroll
        for (int ni = 0; ni < NT; ++ni) {
          int r, c; frag_rc(mi, ni, r, c);
          if (r < N && c < N) {
            const double2 v = packed_pair(Pk, r, c);
            pn[(mi * NT + ni) * 2] = v.x; pn[(mi * NT + ni) * 2 + 1] = v.y;
          }
        }
    }
  }
}

// dense products of the smoother on the FP64 tensor path (DMMA) where the fragment layout fits; the scalar broadcast
// kernel otherwise.  PH: the covariance slabs are packed (callers check that the pair kernel serves M)
template <class M, bool PH = false>
inline void launch_rts_auto(const RtsArgs<M::NG>& a, cudaStream_t st) {
  if (a.len && a.x_term) {
    fprintf(stderr, "[rednose_b200] RTS: per-filter lengths and segment continuation cannot be combined\n");
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  if (a.B <= 0 || a.T <= 0) return;
  if constexpr (M::EDIM % 2 == 0 && M::MEDIM >= 8 && M::MEDIM <= 32 && (M::EDIM <= 32 || !PH)) {
    const unsigned grid = (unsigned)((a.B + RTS_WARPS - 1) / RTS_WARPS);
    constexpr size_t smem = sizeof(RtsMmaScratch<M>) * RTS_WARPS;   // 55 296 B at EDIM 32, 32 192 B for live_kf
    auto run = [&](void (*kern)(const RtsArgs<M::NG>)) {
      if (first_launch_of((const void*)kern)) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<grid, RTS_WARPS * 32, smem, st>>>(a);
    };
    if constexpr (M::EDIM > 32) run(ekf_rts_warp_mma<M, false>);   // ragged histories are refused above 32 by their caller
    else if constexpr (PH) run(a.len ? ekf_rts_warp_mma<PackedHist<M>, true> : ekf_rts_warp_mma<PackedHist<M>, false>);
    else run(a.len ? ekf_rts_warp_mma<M, true> : ekf_rts_warp_mma<M, false>);
    check(cudaGetLastError(), "ekf_rts_mma launch");
  } else if constexpr (PH && !(M::EDIM <= 32 && M::EDIM % 2 == 0)) {
    fprintf(stderr, "[rednose_b200] RTS: no packed covariance layout for EDIM = %d\n", M::EDIM);
    last_status() = (int)cudaErrorNotSupported;
  } else {
    launch_rts<M, PH>(a, st);
  }
}

// one segment of a ragged history (a.len, a.term, a.k0s, a.x_term / a.P_term; EDIM <= 32): the RaggedSeg instantiations
// of the kernel launch_rts_auto picks for M.  PH: the covariance slabs are packed (callers check that the pair kernel
// serves M)
template <class M, bool PH>
inline void launch_rts_ragged_segment(const RtsArgs<M::NG>& a, cudaStream_t st) {
  static_assert(M::EDIM <= 32, "ragged histories exist only up to EDIM 32");
  if (a.B <= 0 || a.T <= 0) return;
  using MS = RaggedSeg<std::conditional_t<PH, PackedHist<M>, M>>;
  const unsigned grid = (unsigned)((a.B + RTS_WARPS - 1) / RTS_WARPS);
  if constexpr (M::EDIM % 2 == 0 && M::MEDIM >= 8 && M::MEDIM <= 32) {
    constexpr size_t smem = sizeof(RtsMmaScratch<MS>) * RTS_WARPS;
    auto kern = ekf_rts_warp_mma<MS, true>;
    if (first_launch_of((const void*)kern)) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, RTS_WARPS * 32, smem, st>>>(a);
    check(cudaGetLastError(), "ekf_rts_mma launch");
  } else {
    ekf_rts_warp<MS, true><<<grid, RTS_WARPS * 32, 0, st>>>(a);
    check(cudaGetLastError(), "ekf_rts launch");
  }
}

}  // namespace rnb
