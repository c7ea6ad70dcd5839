// rednose_b200 -- fused predict+update kernel, TWO filters per warp (even EDIM <= 32, e.g. live_kf 22).
//
// Same three phases and the same arithmetic as ekf_step_warp (ekf_warp.cuh: A leaf per lane, B covariance per
// warp, C inject per lane; reference semantics ekf_c.c:8-33, :37-121), different lane mapping in phase B:
//
//   half-warp h (lanes 16h .. 16h+15) works on filter f + h of the group; lane hl of the half owns the ADJACENT
//   columns 2 hl and 2 hl + 1 of that filter's covariance.
//
// Why: ekf_step_warp is bound by the L1TEX data pipe (shared-memory wavefronts per filter).  Most of those are warp-uniform ("broadcast") loads of per-filter
// values -- F slots, H slots, the rows of H P for the rank-m update -- and a broadcast costs one wavefront per
// 8 bytes no matter how many lanes listen.  Here one such instruction fetches the value of filter f for half 0 and
// of filter f+1 for half 1, and serves two columns per lane: broadcast wavefronts per filter halve.  Adjacent
// columns also turn the tile reads, the exchange stores and the global stores of P into 128-bit accesses
// (22 STG.128 per filter PAIR instead of 22 STG.64 per filter).
//
// Cost: two columns + the F slots live at once = ~200 registers, so 8 warps per SM (16 filters in flight per SM
// instead of 12) and two independent dependency chains per lane.
#pragma once
#include "ekf_warp.cuh"
#include <cstdlib>

namespace rnb {

#ifndef RNB_PAIR
#define RNB_PAIR 1        // 1: even-EDIM filters use ekf_step_pair; 0: always ekf_step_warp
#endif
#ifndef RNB_PAIR_GROUP
#define RNB_PAIR_GROUP 16 // filters per warp group (leaf phase: one filter per lane)
#endif
#ifndef RNB_PAIR_MIN_WARPS
#define RNB_PAIR_MIN_WARPS 8
#endif
#ifndef RNB_PAIR_FV_EARLY
#define RNB_PAIR_FV_EARLY 0    // 1: F value slots are fetched before the tile wait instead of after it
#endif
#ifndef RNB_PAIR_WAR_FIX
#define RNB_PAIR_WAR_FIX 1   // ordering of the tile reads before the slot refill: 1 = proxy fence (deterministic over 250 x 6.3e6 filter-steps), 2 = wait on the last load only (NOT sufficient: 66 of 250 runs differed), 3 = both
#endif
#ifndef RNB_PAIR_LATE_REFILL
#define RNB_PAIR_LATE_REFILL 0   // 1: in fused-predict instantiations the fence + refill move behind the exchange stores of F P (the tile loads have long landed there)
#endif
#ifndef RNB_PAIR_TMA_STAGE
#define RNB_PAIR_TMA_STAGE 1   // x / z / R / dt blocks of a full group arrive by bulk copy (one mbarrier wait, no registers held)
#endif

template <class M, class K, int G>
struct PairScratch {
  using L = RowLayout<M, K>;
  static constexpr int E = M::EDIM;
  static constexpr int NST = RNB_STAGES;
  alignas(128) double tile[NST * 2 * E * E];          // covariance tile PAIRS (TMA ring)
  alignas(8) uint64_t full[NST];
  alignas(16) double rows[G * L::STRIDE];
  static constexpr int EXS = ((E + 3) & ~3) + 2;      // exchange row stride, = 2 (mod 4): see WarpScratch
  static constexpr int HPS = 32;                      // (H P)[c][k] row stride
  // exchange row of slot s: every 8th row is skewed by 16 bytes -- with a stride = 2 (mod 4) doubles, rows s and s+8
  // would start in the same bank group, and the lanes that read one whole row each hold rows 0, 2, 4, 6, 8 (live_kf)
  static constexpr int exrow(int sl) { return sl * EXS + 2 * (sl >> 3); }
  static constexpr int EXN = exrow(M::NFROWS > 0 ? M::NFROWS : 1) + 32;
  static constexpr int HPN = K::ZDIM * HPS;
  // staging area for the group's x / z / R / dt blocks (bulk-copied, consumed by phase A before the exchange
  // buffers come into use): offsets in doubles, each 16-byte aligned
  static constexpr int STG_X = 0;
  static constexpr int STG_Z = STG_X + even_up(G * M::DIM);
  static constexpr int STG_R = STG_Z + even_up(G * K::ZDIM);
  static constexpr int STG_DT = STG_R + even_up(G * K::ZDIM * K::ZDIM);
  static constexpr int STG_N = STG_DT + even_up(G);
  static constexpr int XN0 = ((EXN > HPN ? EXN : HPN) + 3) & ~1;  // per half
  static constexpr int XN1 = (STG_N + 1) / 2;
  static constexpr int XN = (((XN0 > XN1 ? XN0 : XN1) + 1) & ~1) | 2;   // even, = 2 (mod 4): the halves sit on different banks
  alignas(16) double exhp[2 * XN];
  alignas(8) uint64_t stg;                            // "staging blocks landed" mbarrier
};

template <class M, class K, bool PRED, bool UPD, int G, bool GATHER>
__global__ void __launch_bounds__(32, RNB_PAIR_MIN_WARPS) ekf_step_pair(const StepArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  using L = RowLayout<M, K>;
  using SC = PairScratch<M, K, G>;
  constexpr int RS = L::STRIDE, HPS = SC::HPS, XN = SC::XN;
  static_assert(E <= 32 && E % 2 == 0, "pair kernel: even EDIM <= 32");
  static_assert(G <= 32 && G % 2 == 0, "group size");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SC& s = *reinterpret_cast<SC*>(smem_raw);

  const int lane = threadIdx.x & 31;
  const long long b0 = (long long)blockIdx.x * G;   // first ENTRY of the group
  if (b0 >= a.B) return;
  const int ng = (a.B - b0 < G) ? (int)(a.B - b0) : G;
  const int h = lane >> 4;                  // half-warp = which filter of the pair
  const int hl_raw = lane & 15;
  const bool act = hl_raw < E / 2;          // lane owns two real columns
  const int hl = act ? hl_raw : E / 2 - 1;  // idle lanes mirror the last active lane (same quarter-warp: a broadcast, not a bank conflict)
  const int c0 = 2 * hl;                    // owned columns c0, c0 + 1
  double* myrow = s.rows + (lane < G ? lane : 0) * RS;
  const bool mine = lane < ng;
  long long myfid = b0 + (mine ? lane : 0);
  if constexpr (GATHER) { if (mine) myfid = (long long)a.idx[b0 + lane]; }
  auto fid_of = [&](int f) -> long long {
    if constexpr (GATHER) return __shfl_sync(0xffffffffu, myfid, f);
    else return b0 + f;
  };
  double* exh = s.exhp + h * XN;            // this half's exchange / (H P) buffer

  constexpr int NST = RNB_STAGES;
  constexpr uint32_t TILE_BYTES = E * E * sizeof(double);
  uint32_t it = 0;
  if (lane == 0) {
#pragma unroll
    for (int st = 0; st < NST; ++st) mbar_init(&s.full[st], 1);
    mbar_init(&s.stg, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_async_smem();
  }
  __syncwarp();
  // one elected lane arms the barrier and issues the bulk copies of pair (f, f+1)
  auto issue_pair = [&](int f, uint32_t slot, long long fidA, long long fidB) {
    const int np = (ng - f >= 2) ? 2 : 1;
    mbar_expect_tx(&s.full[slot], np * TILE_BYTES);
    double* dst = s.tile + slot * (2 * E * E);
    if constexpr (GATHER) {
      tma_load_1d(dst, a.P + fidA * (long long)(E * E), TILE_BYTES, &s.full[slot]);
      if (np == 2) tma_load_1d(dst + E * E, a.P + fidB * (long long)(E * E), TILE_BYTES, &s.full[slot]);
    } else {
      tma_load_1d(dst, a.P + fidA * (long long)(E * E), np * TILE_BYTES, &s.full[slot]);   // consecutive filters: one copy
    }
  };

  // diagonal process noise entries of the two owned columns
  double qd0 = 0.0, qd1 = 0.0;
  if (PRED && (a.flags & FLAG_Q_DIAG)) { qd0 = __ldg(a.Q + c0 * E + c0); qd1 = __ldg(a.Q + (c0 + 1) * E + c0 + 1); }

  const int n_obs = UPD ? a.n_obs : 1;
  for (int o = 0; o < n_obs; ++o) {
    const bool do_pred = PRED && o == 0;
    if (o > 0) {
      asm volatile("fence.proxy.async;" ::: "memory");   // our plain stores of P -> visible to the bulk-copy engine
      __syncwarp();
    }
#pragma unroll
    for (int k = 0; k < NST; ++k) {
      const long long fa = fid_of(2 * k < ng ? 2 * k : 0), fb = fid_of(2 * k + 1 < ng ? 2 * k + 1 : 0);
      if (lane == 0 && 2 * k < ng) issue_pair(2 * k, (it + k) % NST, fa, fb);
    }

    // ---- stage x, z, R, dt of the group ----
    double dt_lane = a.dt;
    bool staged = false;
    if constexpr (RNB_PAIR_TMA_STAGE && !GATHER) {
      // full group, 16-byte aligned arrays, one observation per filter: the blocks are contiguous -> bulk copies into
      // the (still idle) exchange buffers, one mbarrier wait; used at most once per kernel (o == 0), so parity 0
      const bool ok = o == 0 && ng == G && (!UPD || a.n_obs == 1) &&
          !((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.z) | reinterpret_cast<uintptr_t>(a.R) |
             reinterpret_cast<uintptr_t>(a.dt_arr)) & 15u);
      if (ok) {
        staged = true;
        const bool shared_R = UPD && (a.flags & FLAG_SHARED_R);
        const bool want_dt = do_pred && a.dt_arr;
        double* stg = s.exhp;
        if (lane == 0) {
          uint32_t bytes = G * D * 8;
          if (UPD) bytes += G * Z * 8 + (shared_R ? 0 : G * Z * Z * 8);
          if (want_dt) bytes += G * 8;
          mbar_expect_tx(&s.stg, bytes);
          tma_load_1d(stg + SC::STG_X, a.x + b0 * D, G * D * 8, &s.stg);
          if (UPD) {
            tma_load_1d(stg + SC::STG_Z, a.z + b0 * Z, G * Z * 8, &s.stg);
            if (!shared_R) tma_load_1d(stg + SC::STG_R, a.R + b0 * (Z * Z), G * Z * Z * 8, &s.stg);
          }
          if (want_dt) tma_load_1d(stg + SC::STG_DT, a.dt_arr + b0, G * 8, &s.stg);
        }
        mbar_wait(&s.stg, 0);
        if (mine) {   // ng == G: every lane < G owns a record; odd record strides -> conflict-free lane-strided reads
#pragma unroll
          for (int i = 0; i < D; ++i) myrow[L::OFF_X + i] = stg[SC::STG_X + lane * D + i];
          if constexpr (UPD) {
#pragma unroll
            for (int i = 0; i < Z; ++i) myrow[L::OFF_Y + i] = stg[SC::STG_Z + lane * Z + i];
#pragma unroll
            for (int i = 0; i < Z * Z; ++i) myrow[L::OFF_R + i] = shared_R ? __ldg(a.R + i) : stg[SC::STG_R + lane * (Z * Z) + i];
          }
          if (want_dt) dt_lane = stg[SC::STG_DT + lane];
        }
      }
    }
    if (!staged) {
      // register path: every global load of the block before the first dependent shared-memory store
      StageRegs<D, G> rx;
      StageRegs<Z, G> rz;
      StageRegs<Z * Z, G> rR;
      const bool shared_R = UPD && (a.flags & FLAG_SHARED_R);
      const bool bulk_obs = UPD && a.n_obs == 1;
      if (o == 0) {
        if (GATHER) gather_load<D, G>(a.x, rx, ng, lane, myfid);
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
        double fv[L::NFp];
        double xn[L::Dp];
        M::predict_leaf(xp, dt_lane, a.gv, xn, fv);
        if constexpr (L::NFp > M::NF) fv[L::NFp - 1] = 0.0;
        if constexpr (L::Dp > D) xn[L::Dp - 1] = 0.0;
        vec_store(myrow + L::OFF_FV, fv);
        myrow[L::OFF_DT] = dt_lane;
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
      if (GATHER) scatter_out<D, RS>(a.hx_pred, s.rows, L::OFF_X, ng, lane, myfid);
      else stage_out<D, RS>(a.hx_pred + b0 * D, s.rows, L::OFF_X, ng, lane);
    }
    if constexpr (UPD) {
      if (a.n_obs == 1) {
        stage_out<Z, RS>(a.z + b0 * Z, s.rows, L::OFF_Y, ng, lane);   // the innovation overwrites z (ekf_c.c:120)
      } else if (mine) {
        const long long bo = (b0 + lane) * a.n_obs + o;
#pragma unroll
        for (int i = 0; i < Z; ++i) a.z[bo * Z + i] = myrow[L::OFF_Y + i];
      }
    }

    // ================= phase B: covariance, one filter PAIR per warp iteration =================
#pragma unroll 1
    for (int f = 0; f < ng; f += 2) {
      const bool valid = f + h < ng;              // half 1 idles on an odd tail (computes on stale data, writes nothing)
      const int fi = valid ? f + h : f;
      const bool wr = valid && act;
      const long long b = fid_of(fi);
      double* row = s.rows + fi * RS;
      const uint32_t slot = it % NST;
      const double* tile = s.tile + slot * (2 * E * E) + (valid ? h : 0) * (E * E);
      double p0[E], p1[E];                        // columns c0 and c0 + 1
      double fv[L::NFp];
      if (RNB_PAIR_FV_EARLY && do_pred) vec_load(row + L::OFF_FV, fv);

      mbar_wait(&s.full[slot], (it / NST) & 1u);
      // row i of the tile holds P[i][c0], P[i][c0+1] side by side: one 128-bit load per row feeds both columns
#pragma unroll
      for (int i = 0; i < E; ++i) {
        const double2 t = *reinterpret_cast<const double2*>(tile + i * E + c0);
        p0[i] = t.x; p1[i] = t.y;
      }
      const int fn = f + 2 * NST;
      const long long fa = fid_of(fn < ng ? fn : 0), fb = fid_of(fn + 1 < ng ? fn + 1 : 0);
      constexpr bool LATE = RNB_PAIR_LATE_REFILL && (M::NFROWS > 0);
      if (!(LATE && do_pred)) {
        // WAR across proxies: the 128-bit shared loads above are generic-proxy reads that may still be queued when this
        // point is reached (a load is "issued", not "performed"); the bulk copy that refills the slot writes through the
        // async proxy.  The proxy fence orders the reads before it -- without it about one filter-step in 1e7 saw the last
        // tile rows of the NEXT pair (found as run-to-run differences of 10 000-step histories, scripts/dbg_rts_race.py).
        if constexpr (RNB_PAIR_WAR_FIX & 1) fence_async_smem();
        if constexpr (RNB_PAIR_WAR_FIX & 2) {   // experiment kept for the record: waiting on the LAST load of the sequence is NOT enough
          const double landed = p0[E - 1] + p1[E - 1];
          asm volatile("" ::"d"(landed));
        }
        __syncwarp();   // every lane holds its columns before the slot is refilled
        if (lane == 0 && fn < ng) issue_pair(fn, slot, fa, fb);
      }
      ++it;

      if (do_pred) {
        if (!RNB_PAIR_FV_EARLY) vec_load(row + L::OFF_FV, fv);
        const double dt = row[L::OFF_DT];
        if constexpr (M::NFROWS > 0) {
          {
            // rows of F P that differ from rows of P, for both columns, into the exchange (one 128-bit store per row)
            double m0[E], m1[E];
#pragma unroll
            for (int i = 0; i < E; ++i) { m0[i] = p0[i]; m1[i] = p1[i]; }
            M::F_apply(fv, m0);
            M::F_apply(fv, m1);
            if (act) {
              int sl = 0;
#pragma unroll
              for (int r = 0; r < E; ++r) {
                if ((M::FROW_MASK >> r) & 1u) {
                  *reinterpret_cast<double2*>(exh + SC::exrow(sl) + c0) = make_double2(m0[r], m1[r]);
                  ++sl;
                }
              }
            }
          }
          if constexpr (LATE) fence_async_smem();   // late refill: the tile loads landed long ago, the fence costs nothing here
          __syncwarp();
          if constexpr (LATE) { if (lane == 0 && fn < ng) issue_pair(fn, slot, fa, fb); }
          // a column whose index is a non-identity row of F is replaced by that row of F P (symmetry gives the rest)
          if ((M::FROW_MASK >> c0) & 1u) {
            const double* xr = exh + SC::exrow(__popc(M::FROW_MASK & ((1u << c0) - 1u)));
#pragma unroll
            for (int i = 0; i < E; ++i) p0[i] = xr[i];   // 64-bit loads: p0[i] shares a register quad with p1[i], not p0[i+1]
          }
          if ((M::FROW_MASK >> (c0 + 1)) & 1u) {
            const double* xr = exh + SC::exrow(__popc(M::FROW_MASK & ((2u << c0) - 1u)));
#pragma unroll
            for (int i = 0; i < E; ++i) p1[i] = xr[i];
          }
          M::F_apply(fv, p0);                     // columns c0, c0+1 of F (F P)^T
          M::F_apply(fv, p1);
          __syncwarp();
        } else {
          M::F_apply(fv, p0);
          M::F_apply(fv, p1);
        }
        if (a.flags & FLAG_Q_DIAG) {
          const double dq0 = dt * qd0, dq1 = dt * qd1;
#pragma unroll
          for (int i = 0; i < E; i += 2) {        // c0 is even: p0 takes its diagonal at an even i, p1 at the odd one
            asm("{\n .reg .pred q;\n setp.eq.s32 q, %2, %3;\n @q add.f64 %0, %0, %1;\n}" : "+d"(p0[i]) : "d"(dq0), "r"(c0), "r"(i));
            asm("{\n .reg .pred q;\n setp.eq.s32 q, %2, %3;\n @q add.f64 %0, %0, %1;\n}" : "+d"(p1[i + 1]) : "d"(dq1), "r"(c0), "r"(i));
          }
        } else {
          const double* Qg = a.Q + c0;
#pragma unroll
          for (int i = 0; i < E; ++i) {
            p0[i] = fma(dt, __ldg(Qg + i * E), p0[i]);
            p1[i] = fma(dt, __ldg(Qg + i * E + 1), p1[i]);
          }
        }
        if (a.hP_pred && wr) {
          double* Hg = a.hP_pred + b * (long long)(E * E) + c0;
#pragma unroll
          for (int i = 0; i < E; ++i) *reinterpret_cast<double2*>(Hg + i * E) = make_double2(p0[i], p1[i]);
        }
      }

      if constexpr (UPD) {
        double hp0[Z], hp1[Z];
        double S[Z][Z];
        {
          double hv[L::NHp];
          vec_load(row + L::OFF_HV, hv);
          K::Herr_apply(hv, p0, hp0);             // (H P)[:, c0], (H P)[:, c0+1]
          K::Herr_apply(hv, p1, hp1);
#pragma unroll
          for (int c = 0; c < Z; ++c) {
            if (hl_raw < HPS / 2)
              *reinterpret_cast<double2*>(exh + c * HPS + 2 * hl_raw) = act ? make_double2(hp0[c], hp1[c]) : make_double2(0.0, 0.0);
          }
          __syncwarp();
#pragma unroll
          for (int i = 0; i < Z; ++i)
#pragma unroll
            for (int j = 0; j < Z; ++j) S[i][j] = 0.0;
          K::S_accum(hv, [&](int c, int k) { return exh[c * HPS + k]; }, S);   // uniform within the half
        }
        double y[L::Zp], R[L::ZZp];
        vec_load(row + L::OFF_Y, y);
        vec_load(row + L::OFF_R, R);

        SolverZ<Z> ldl;
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
          const double infl = (d > K::MAHA_THRESH) ? 1.0e16 : 1.0;   // per half: a select, not a branch (ekf_c.c:91-93)
#pragma unroll
          for (int i = 0; i < Z * Z; ++i) R[i] *= infl;
        }
#pragma unroll
        for (int i = 0; i < Z; ++i)
#pragma unroll
          for (int j = 0; j < Z; ++j) S[i][j] += R[i * Z + j];
        ldl.factor(S);

        // w = S^-1 hp: rows c0, c0+1 of the Kalman gain;  dx = K y
        ldl.solve(hp0);
        ldl.solve(hp1);
        double dx0 = 0.0, dx1 = 0.0;
#pragma unroll
        for (int c = 0; c < Z; ++c) { dx0 = fma(hp0[c], y[c], dx0); dx1 = fma(hp1[c], y[c], dx1); }
        if (wr) *reinterpret_cast<double2*>(row + L::OFF_FV + c0) = make_double2(dx0, dx1);  // F slots are dead: reuse for dx

        // P[:, c] -= (H P)^T w_c for both columns: every broadcast load of (H P) feeds four FMAs
#pragma unroll
        for (int i = 0; i < E; i += 2) {
          double a0 = p0[i], a1 = p0[i + 1], b0v = p1[i], b1v = p1[i + 1];
#pragma unroll
          for (int c = 0; c < Z; ++c) {
            const double2 h2 = *reinterpret_cast<const double2*>(exh + c * HPS + i);
            a0 = fma(-h2.x, hp0[c], a0);
            a1 = fma(-h2.y, hp0[c], a1);
            b0v = fma(-h2.x, hp1[c], b0v);
            b1v = fma(-h2.y, hp1[c], b1v);
          }
          p0[i] = a0; p0[i + 1] = a1; p1[i] = b0v; p1[i + 1] = b1v;
        }
        __syncwarp();
        if (a.hP_filt && wr && o == n_obs - 1) {
          double* Hg = a.hP_filt + b * (long long)(E * E) + c0;
#pragma unroll
          for (int i = 0; i < E; ++i) *reinterpret_cast<double2*>(Hg + i * E) = make_double2(p0[i], p1[i]);
        }
      }

      if (wr) {
        double* Pg = a.P + b * (long long)(E * E) + c0;
#pragma unroll
        for (int i = 0; i < E; ++i) *reinterpret_cast<double2*>(Pg + i * E) = make_double2(p0[i], p1[i]);
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
      if (GATHER) scatter_out<D, RS>(a.x, s.rows, L::OFF_X, ng, lane, myfid);
      else stage_out<D, RS>(a.x + b0 * D, s.rows, L::OFF_X, ng, lane);
      if (UPD && a.hx_filt) {
        if (GATHER) scatter_out<D, RS>(a.hx_filt, s.rows, L::OFF_X, ng, lane, myfid);
        else stage_out<D, RS>(a.hx_filt + b0 * D, s.rows, L::OFF_X, ng, lane);
      }
    }
    __syncwarp();
  }
}

template <class M, class K, int G>
constexpr size_t pair_smem_bytes() { return sizeof(PairScratch<M, K, G>); }

template <class M>
constexpr bool use_pair() { return RNB_PAIR && RNB_TMA && M::EDIM % 2 == 0 && M::EDIM <= 32; }

// run-time escape hatch (and the way the tests reach ekf_step_warp on an even-EDIM filter):
// REDNOSE_B200_WARP_KERNEL=single selects the one-filter-per-warp kernel; read at every launch (a getenv is
// nothing next to a kernel launch) so that a test can flip it inside one process
inline bool pair_enabled() {
  const char* e = getenv("REDNOSE_B200_WARP_KERNEL");
  return !(e && e[0] == 's');
}

}  // namespace rnb
