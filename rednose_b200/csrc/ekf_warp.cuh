// rednose_b200 -- warp-per-filter fused predict+update kernel (odd EDIM 7..31).
//
// Even-EDIM filters (e.g. live_kf: DIM 23 / EDIM 22, examples/live_kf.py:97-124) run ekf_step_pair (ekf_warp2.cuh: two
// filters per warp, same phases and arithmetic, built on the primitives of this file); this kernel serves odd EDIM.
//
// A warp owns a GROUP of G consecutive filters and walks through three phases:
//
//  A  (thread-per-filter)  lane l evaluates the generated leaf code of filter l of the group:
//       x_pred = f(x, dt), the NF non-trivial entries of F, h(x_pred), the NH non-zeros of
//       H_err = H * H_mod, y = z - h.  Results go to a per-filter ROW in shared memory.  The leaf
//       code is scalar and branch-free, so 32 lanes = 32 different filters run it at full SIMT
//       efficiency -- evaluating it redundantly in every lane of a warp-per-filter kernel was the
//       dominant cost of the first version.
//  B  (warp-per-filter)    for each filter of the group in turn: lane j holds COLUMN j of the
//       symmetric covariance P in registers.  With that ownership
//         (F P)[:,j] = F P[:,j]            lane-local  (generated sparse MODEL::F_apply)
//         (H P)[:,j] = H_err P[:,j]        lane-local  (generated sparse KIND::Herr_apply)
//         W[:,j]     = S^-1 (H P)[:,j]     lane-local  (row j of the gain K)
//         P'[:,j]    = P[:,j] - (H P)^T W[:,j]         needs (H P) broadcast through shared memory
//       F P F^T needs a transposition only for the rows of F that differ from the identity (9 of
//       22 for live_kf): column j of F P F^T = F (row j of F P)^T, and row j of F P equals column j
//       of P (symmetry) unless j is such a row; those rows go through a [NFROWS][33] exchange.
//       Leaf values are read from the filter's row as warp-uniform broadcasts.
//  C  (thread-per-filter)  lane l injects the correction: x = err_fun(x_pred, K y), normalises
//       quaternions and writes the state back.
//
// Reference semantics: ekf_c.c:8-33 (predict), :37-121 (update, He==NULL path), normalisation
// ekf_sym.cc:69-77,207,213.  P is assumed symmetric on entry (it is a covariance; the
// reference's own arithmetic keeps it symmetric to rounding).
#pragma once
#include "ekf_common.cuh"

namespace rnb {

constexpr int WARP_GROUP = 14;   // filters per warp group (leaf phase uses WARP_GROUP of the 32 lanes)
constexpr int WARP_CTA_WARPS = 1;   // warps per CTA (warps never synchronise with each other)

constexpr int even_up(int n) { return (n + 1) & ~1; }

// ---- TMA (cp.async.bulk) + mbarrier primitives (ekf_step_pair's tile ring and staging); SASS: UBLKCP / SYNCS ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Per-filter row in shared memory.  Every section starts on an even index (16-byte aligned) so
// rows are moved with 128-bit accesses; the row stride is = 2 (mod 4) doubles, which makes lane-
// strided 128-bit stores/loads (phase A/C: lane l touches row l) bank-conflict free.
template <class M, class K>
struct RowLayout {
  static constexpr int NFp = even_up(M::NF > 0 ? M::NF : 1);
  static constexpr int NHp = even_up(K::NH > 0 ? K::NH : 1);
  static constexpr int Zp = even_up(K::ZDIM);
  static constexpr int ZZp = even_up(K::ZDIM * K::ZDIM);
  static constexpr int Dp = even_up(M::DIM);
  static constexpr int Ep = even_up(M::EDIM);
  static constexpr int OFF_FV = 0;                  // F value slots; reused for dx = K y once F is dead
  static constexpr int FVDX = NFp > Ep ? NFp : Ep;
  static constexpr int OFF_HV = OFF_FV + FVDX;      // H_err value slots
  static constexpr int OFF_Y = OFF_HV + NHp;        // innovation
  static constexpr int OFF_R = OFF_Y + Zp;          // measurement noise
  static constexpr int OFF_X = OFF_R + ZZp;         // predicted state
  static constexpr int OFF_DT = OFF_X + Dp;         // dt of this filter (+1 pad)
  static constexpr int OFF_HID = OFF_DT + 1;        // the pad: history slab element of a gather entry (ekf_step_pair)
  static constexpr int RAW = OFF_DT + 2;
  static constexpr int STRIDE = RAW + ((2 - RAW % 4) + 4) % 4;  // = 2 (mod 4)
};

template <int N>
__device__ __forceinline__ void vec_store(double* dst, const double (&v)[N]) {
  static_assert(N % 2 == 0, "even");
#pragma unroll
  for (int i = 0; i < N; i += 2) *reinterpret_cast<double2*>(dst + i) = make_double2(v[i], v[i + 1]);
}
template <int N>
__device__ __forceinline__ void vec_load(const double* src, double (&v)[N]) {
  static_assert(N % 2 == 0, "even");
#pragma unroll
  for (int i = 0; i < N; i += 2) { const double2 t = *reinterpret_cast<const double2*>(src + i); v[i] = t.x; v[i + 1] = t.y; }
}

template <class M, class K, int G>
struct WarpScratch {
  using L = RowLayout<M, K>;
  alignas(16) double rows[G * L::STRIDE];
  // exchange row stride = 2 (mod 4) doubles: rows start 16-byte aligned and the lanes that read a whole row each
  // (128-bit accesses, one row per lane) hit distinct bank groups; the column writes (lane l -> element l) are
  // conflict free for any stride
  static constexpr int EXS = ((M::EDIM + 3) & ~3) + 2;
  static constexpr int EXN = (M::NFROWS > 0 ? M::NFROWS : 1) * EXS + 32;
  static constexpr int HPN = K::ZDIM * 32;
  // one buffer, two lives: row exchange for F P F^T during the predict, then (H P)[c][k] during the update
  alignas(16) double exhp[EXN > HPN ? EXN : HPN];
};

// normalise quaternions of a state held in shared memory (private to the calling lane)
template <int NG>
__device__ __forceinline__ void lane_normalize(double* xs, const StepArgs<NG>& a) {
  for (int q = 0; q < a.n_quat; ++q) normalize4(xs + a.quat_idx[q]);
}

// Cooperative, coalesced copies between a contiguous global block of ng records of width WD and the per-filter
// rows in shared memory (record f -> rows[f * STRIDE + off .. + WD)).  The inbound direction is split into a load
// half and a store half so that the kernel can put the loads of SEVERAL record types (x, z, R) in flight before the
// first dependent shared-memory store: one global round trip per group.  gather_load is the same for records
// scattered in global memory: record f lives at g + fid(f) * WD, fid held by lane f.
template <int WD, int G>
struct StageRegs { static constexpr int NIT = (G * WD + 31) / 32; double v[NIT]; };
template <int WD, int G>
__device__ __forceinline__ void stage_load(const double* __restrict__ g, StageRegs<WD, G>& r, int ng, int lane) {
#pragma unroll
  for (int it = 0; it < StageRegs<WD, G>::NIT; ++it) {
    const int idx = it * 32 + lane;
    r.v[it] = (idx < ng * WD) ? g[idx] : 0.0;
  }
}
template <int WD, int G>
__device__ __forceinline__ void gather_load(const double* __restrict__ g, StageRegs<WD, G>& r, int ng, int lane, long long myfid) {
#pragma unroll
  for (int it = 0; it < StageRegs<WD, G>::NIT; ++it) {
    const int idx = it * 32 + lane;
    const bool ok = idx < ng * WD;
    const int f = ok ? idx / WD : 0, i = idx - f * WD;
    const long long fid = __shfl_sync(0xffffffffu, myfid, f);
    r.v[it] = ok ? g[fid * WD + i] : 0.0;
  }
}
template <int WD, int STRIDE, int G>
__device__ __forceinline__ void stage_store(const StageRegs<WD, G>& r, double* rows, int off, int ng, int lane) {
#pragma unroll
  for (int it = 0; it < StageRegs<WD, G>::NIT; ++it) {
    const int idx = it * 32 + lane;
    const int f = idx / WD, i = idx - f * WD;
    if (idx < ng * WD) rows[f * STRIDE + off + i] = r.v[it];
  }
}
template <int WD, int STRIDE>
__device__ __forceinline__ void stage_out(double* __restrict__ g, const double* rows, int off, int ng, int lane) {
  for (int idx = lane; idx < ng * WD; idx += 32) {
    const int f = idx / WD, i = idx - f * WD;
    g[idx] = rows[f * STRIDE + off + i];
  }
}

// scattered counterpart of stage_out; with SKIP_NEG a record whose destination index is negative is not written
template <int WD, int STRIDE, bool SKIP_NEG = false>
__device__ __forceinline__ void scatter_out(double* __restrict__ g, const double* rows, int off, int ng, int lane, long long myfid) {
  for (int base = 0; base < ng * WD; base += 32) {
    const int idx = base + lane;
    const bool ok = idx < ng * WD;
    const int f = ok ? idx / WD : 0, i = idx - f * WD;
    const long long fid = __shfl_sync(0xffffffffu, myfid, f);
    if (ok && (!SKIP_NEG || fid >= 0)) g[fid * WD + i] = rows[f * STRIDE + off + i];
  }
}

constexpr int WARP_MIN_WARPS = 12;   // resident warps per SM the register allocator must allow (170 registers per thread)

template <class M, class K, bool PRED, bool UPD, int G, int W, bool GATHER>
__global__ void __launch_bounds__(W * 32, WARP_MIN_WARPS / W) ekf_step_warp(const StepArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  using L = RowLayout<M, K>;
  constexpr int RS = L::STRIDE;
  constexpr int EXS = WarpScratch<M, K, G>::EXS;
  static_assert(E <= 32 && E % 2 == 1, "warp-per-filter kernel: odd EDIM <= 32 (even EDIM runs ekf_step_pair)");
  static_assert(G <= 32, "group size");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WarpScratch<M, K, G>& s = reinterpret_cast<WarpScratch<M, K, G>*>(smem_raw)[threadIdx.x >> 5];

  const int lane = threadIdx.x & 31;
  const long long b0 = ((long long)blockIdx.x * W + (threadIdx.x >> 5)) * G;  // first ENTRY of the group
  if (b0 >= a.B) return;  // whole warp exits together
  const int ng = (a.B - b0 < G) ? (int)(a.B - b0) : G;
  const bool act = lane < E;
  const int col = act ? lane : 0;
  double* myrow = s.rows + (lane < G ? lane : 0) * RS;
  const bool mine = lane < ng;
  // filter this lane's entry works on (gather list, ragged scheduler) -- entry index when there is no list
  constexpr bool gathered = GATHER;
  long long myfid = b0 + (mine ? lane : 0);
  long long myhid = 0;       // gather lists: history slab element of this lane's entry (-1: not recorded)
  if constexpr (GATHER) {
    myhid = myfid;
    if (mine) {
      myfid = (long long)a.idx[b0 + lane];
      myhid = hist_slot(a, b0 + lane, myfid);
    }
  }
  // filter id of entry f of the group: a shuffle only when a gather list is in use
  auto fid_of = [&](int f) -> long long {
    if constexpr (GATHER) return __shfl_sync(0xffffffffu, myfid, f);
    else return b0 + f;
  };
  auto hid_of = [&](int f) -> long long { return __shfl_sync(0xffffffffu, myhid, f); };   // gather lists only

  // diagonal process noise: this lane's entry, fetched once per warp
  double qdiag = 0.0;
  if (PRED && (a.flags & FLAG_Q_DIAG)) qdiag = __ldg(a.Q + col * E + col);

  const int n_obs = UPD ? a.n_obs : 1;
  for (int o = 0; o < n_obs; ++o) {
    const bool do_pred = PRED && o == 0;

    // ---- stage this group's small per-filter records into the rows (coalesced) ----
    // every global load of the block (x, z, R, dt) is issued before the first shared-memory store that depends on
    // one of them: the group pays ONE global round trip here instead of one per record type (four serialised
    // long-scoreboard waits otherwise)
    double dt_lane = a.dt;
    {
      StageRegs<D, G> rx;
      StageRegs<Z, G> rz;
      StageRegs<Z * Z, G> rR;
      const bool shared_R = UPD && (a.flags & FLAG_SHARED_R);
      const bool bulk_obs = UPD && a.n_obs == 1;
      if (o == 0) {
        if (gathered) gather_load<D, G>(a.x, rx, ng, lane, myfid);
        else stage_load<D, G>(a.x + b0 * D, rx, ng, lane);
      }
      if constexpr (UPD) {
        if (bulk_obs) {
          stage_load<Z, G>(a.z + b0 * Z, rz, ng, lane);
          if (!shared_R) stage_load<Z * Z, G>(a.R + b0 * (Z * Z), rR, ng, lane);
        }
      }
      if (do_pred && mine && a.dt_arr) dt_lane = a.dt_arr[b0 + lane];
      if (o == 0) stage_store<D, RS, G>(rx, s.rows, L::OFF_X, ng, lane);
      if constexpr (UPD) {
        if (bulk_obs) {
          stage_store<Z, RS, G>(rz, s.rows, L::OFF_Y, ng, lane);
          if (!shared_R) stage_store<Z * Z, RS, G>(rR, s.rows, L::OFF_R, ng, lane);
        } else if (mine) {
          const long long bo = (b0 + lane) * a.n_obs + o;
#pragma unroll
          for (int i = 0; i < Z; ++i) myrow[L::OFF_Y + i] = a.z[bo * Z + i];
          if (!shared_R) {
#pragma unroll
            for (int i = 0; i < Z * Z; ++i) myrow[L::OFF_R + i] = a.R[bo * (Z * Z) + i];
          }
        }
        if (shared_R && mine) {
#pragma unroll
          for (int i = 0; i < Z * Z; ++i) myrow[L::OFF_R + i] = __ldg(a.R + i);
        }
      }
    }
    __syncwarp();

    // ================= phase A: leaf evaluation, one filter per lane =================
    if (mine) {
      double xp[L::Dp];
      vec_load(myrow + L::OFF_X, xp);
      if (do_pred) {
        const double dt = dt_lane;
        double fv[L::NFp];
        double xn[L::Dp];
        M::predict_leaf(xp, dt, a.gv, xn, fv);
        if constexpr (L::NFp > M::NF) fv[L::NFp - 1] = 0.0;
        if constexpr (L::Dp > D) xn[L::Dp - 1] = 0.0;
        vec_store(myrow + L::OFF_FV, fv);
        myrow[L::OFF_DT] = dt;
        vec_store(myrow + L::OFF_X, xn);
        if ((a.flags & FLAG_NORM_AFTER_PREDICT) && a.n_quat > 0) lane_normalize(myrow + L::OFF_X, a);
        vec_load(myrow + L::OFF_X, xp);
      }
      if constexpr (UPD) {
        const double* ea = a.ea ? a.ea + ((b0 + lane) * a.n_obs + o) * a.ea_dim : nullptr;
        double hx[Z];
        double hv[L::NHp];
        K::obs_leaf(xp, ea, a.gv, hx, hv);
        if constexpr (L::NHp > K::NH) hv[L::NHp - 1] = 0.0;
        vec_store(myrow + L::OFF_HV, hv);
#pragma unroll
        for (int i = 0; i < Z; ++i) myrow[L::OFF_Y + i] -= hx[i];  // innovation y = z - h(x)
      }
    }
    __syncwarp();
    if (do_pred && a.hx_pred) {
      if (gathered) scatter_out<D, RS, true>(a.hx_pred, s.rows, L::OFF_X, ng, lane, myhid);
      else stage_out<D, RS>(a.hx_pred + b0 * D, s.rows, L::OFF_X, ng, lane);
    }
    if constexpr (UPD) {
      // the innovation overwrites z (ekf_c.c:120)
      if (a.n_obs == 1) {
        stage_out<Z, RS>(a.z + b0 * Z, s.rows, L::OFF_Y, ng, lane);
      } else if (mine) {
        const long long bo = (b0 + lane) * a.n_obs + o;
#pragma unroll
        for (int i = 0; i < Z; ++i) a.z[bo * Z + i] = myrow[L::OFF_Y + i];
      }
    }

    // ================= phase B: covariance, one filter per warp iteration =================
#pragma unroll 1
    for (int f = 0; f < ng; ++f) {
      const long long b = fid_of(f);   // filter id of this iteration
      long long hb = b;                // its history slab element
      bool rec = true;
      if constexpr (GATHER) { hb = hid_of(f); rec = hb >= 0; }
      double* row = s.rows + f * RS;
      double p[E];
      double fv[L::NFp];
      // column `lane` of P straight from global memory: an odd-EDIM tile is no multiple of the 16 bytes a bulk copy moves
      const double* Pg = a.P + b * (long long)(E * E) + col;
#pragma unroll
      for (int i = 0; i < E; ++i) p[i] = Pg[i * E];

      if (do_pred) {
        vec_load(row + L::OFF_FV, fv);
        const double dt = row[L::OFF_DT];
        // rows of F P that are not rows of P (F's non-identity rows) go through the exchange; every other
        // row j of F P equals column j of P (symmetry), which the lane already holds
        if constexpr (M::NFROWS > 0) {
          {
            double m[E];
#pragma unroll
            for (int i = 0; i < E; ++i) m[i] = p[i];
            M::F_apply(fv, m);                      // only the non-identity rows of m are computed / used
            if (act) M::frows_store(m, s.exhp + lane, EXS);   // stride < 32: idle lanes must not spill into the next row
          }
          __syncwarp();
          const bool in_rf = (M::FROW_MASK >> lane) & 1u;
          const int slot_rf = __popc(M::FROW_MASK & ((1u << lane) - 1u));
          if (in_rf) {  // this lane's row of F P replaces its column of P
            const double* xr = s.exhp + slot_rf * EXS;
#pragma unroll
            for (int i = 0; i + 1 < E; i += 2) {
              const double2 t = *reinterpret_cast<const double2*>(xr + i);
              p[i] = t.x; p[i + 1] = t.y;
            }
            if constexpr (E % 2) p[E - 1] = xr[E - 1];
          }
          M::F_apply(fv, p);                        // column `lane` of F (F P)^T = F P F^T
          __syncwarp();
        } else {
          M::F_apply(fv, p);
        }
        if (a.flags & FLAG_Q_DIAG) {
          // diagonal process noise: only P[lane][lane] changes
          const double dq = dt * qdiag;
          // one predicated DADD per element (a select costs ISETP + 2 FSEL + DADD; an `if` compiles to branches)
#pragma unroll
          for (int i = 0; i < E; ++i)
            asm("{\n .reg .pred q;\n setp.eq.s32 q, %2, %3;\n @q add.f64 %0, %0, %1;\n}" : "+d"(p[i]) : "d"(dq), "r"(lane), "r"(i));
        } else {
          const double* Qg = a.Q + col;
#pragma unroll
          for (int i = 0; i < E; ++i) p[i] = fma(dt, __ldg(Qg + i * E), p[i]);
        }
        if (a.hP_pred && act && rec) {
          double* Hg = a.hP_pred + hb * (long long)(E * E) + col;
#pragma unroll
          for (int i = 0; i < E; ++i) Hg[i * E] = p[i];
        }
      }

      if constexpr (UPD) {
        double hp[Z];
        double S[Z][Z];
        {
          double hv[L::NHp];
          vec_load(row + L::OFF_HV, hv);
          K::Herr_apply(hv, p, hp);  // (H P)[:,lane]
#pragma unroll
          for (int c = 0; c < Z; ++c) s.exhp[c * 32 + lane] = act ? hp[c] : 0.0;
          __syncwarp();
          // S = H_err (H P)^T + R, warp-uniform
#pragma unroll
          for (int i = 0; i < Z; ++i)
#pragma unroll
            for (int j = 0; j < Z; ++j) S[i][j] = 0.0;
          K::S_accum(hv, [&](int c, int k) { return s.exhp[c * 32 + k]; }, S);
        }
        double y[L::Zp], R[L::ZZp];
        vec_load(row + L::OFF_Y, y);
        vec_load(row + L::OFF_R, R);

        LDL<Z> ldl;
        if constexpr (K::MAHA) {
          double Sg[Z][Z];
#pragma unroll
          for (int i = 0; i < Z; ++i)
#pragma unroll
            for (int j = 0; j < Z; ++j) Sg[i][j] = S[i][j] + R[i * Z + j];
          ldl.factor(Sg);
          double u[Z];
#pragma unroll
          for (int i = 0; i < Z; ++i) u[i] = y[i];
          ldl.solve(u);
          double d = 0.0;
#pragma unroll
          for (int i = 0; i < Z; ++i) d += y[i] * u[i];
          if (d > K::MAHA_THRESH) {  // warp-uniform predicate (ekf_c.c:91-93)
#pragma unroll
            for (int i = 0; i < Z * Z; ++i) R[i] *= 1.0e16;
          }
        }
#pragma unroll
        for (int i = 0; i < Z; ++i)
#pragma unroll
          for (int j = 0; j < Z; ++j) S[i][j] += R[i * Z + j];
        ldl.factor(S);

        // w = S^-1 hp: row `lane` of the Kalman gain;  dx[lane] = K[lane,:] y
        ldl.solve(hp);
        double dxl = 0.0;
#pragma unroll
        for (int c = 0; c < Z; ++c) dxl = fma(hp[c], y[c], dxl);
        if (act) row[L::OFF_FV + lane] = dxl;  // F values are dead: reuse for dx

        // P[:,lane] -= (H P)^T w
#pragma unroll
        for (int i = 0; i < E; i += 2) {
          double a0 = p[i], a1 = (i + 1 < E) ? p[i + 1] : 0.0;
#pragma unroll
          for (int c = 0; c < Z; ++c) {
            const double2 h2 = *reinterpret_cast<const double2*>(&s.exhp[c * 32 + i]);
            a0 = fma(-h2.x, hp[c], a0);
            a1 = fma(-h2.y, hp[c], a1);
          }
          p[i] = a0;
          if (i + 1 < E) p[i + 1] = a1;
        }
        __syncwarp();
        if (a.hP_filt && act && rec && o == n_obs - 1) {
          double* Hg = a.hP_filt + hb * (long long)(E * E) + col;
#pragma unroll
          for (int i = 0; i < E; ++i) Hg[i * E] = p[i];
        }
      }

      if (act) {
        double* Pg = a.P + b * (long long)(E * E) + col;
#pragma unroll
        for (int i = 0; i < E; ++i) Pg[i * E] = p[i];
      }
    }
    __syncwarp();

    // ================= phase C: inject the correction, one filter per lane =================
    if constexpr (UPD) {
      if (mine) {
        double xp[L::Dp], dx[L::Ep], xn[L::Dp];
        vec_load(myrow + L::OFF_X, xp);
        vec_load(myrow + L::OFF_FV, dx);
        M::err_fun(xp, dx, a.gv, xn);
        if constexpr (L::Dp > D) xn[L::Dp - 1] = 0.0;
        vec_store(myrow + L::OFF_X, xn);
        if ((a.flags & FLAG_NORM_AFTER_UPDATE) && a.n_quat > 0) lane_normalize(myrow + L::OFF_X, a);
      }
      __syncwarp();
    }
    if (o == n_obs - 1) {
      if (gathered) scatter_out<D, RS>(a.x, s.rows, L::OFF_X, ng, lane, myfid);
      else stage_out<D, RS>(a.x + b0 * D, s.rows, L::OFF_X, ng, lane);
      if (UPD && a.hx_filt) {
        if (gathered) scatter_out<D, RS, true>(a.hx_filt, s.rows, L::OFF_X, ng, lane, myhid);
        else stage_out<D, RS>(a.hx_filt + b0 * D, s.rows, L::OFF_X, ng, lane);
      }
    }
    __syncwarp();
  }
}

template <class M, class K, int G, int W>
constexpr size_t warp_smem_bytes() { return sizeof(WarpScratch<M, K, G>) * W; }

}  // namespace rnb
