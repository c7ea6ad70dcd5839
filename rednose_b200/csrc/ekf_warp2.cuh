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
#include "ekf_packed.cuh"

namespace rnb {

constexpr int PAIR_GROUP = 16;   // filters per warp group (leaf phase: one filter per lane)
constexpr int PAIR_MIN_WARPS = 8;   // ~200 live values per lane: 255 registers, 8 one-warp CTAs per SM

// Depth of the covariance tile ring (pairs in flight per warp).  A packed pair (live_kf: 4 224 B) is little more than half
// a full one (7 744 B), so with the packed layout two slots cost about what one full slot does and the warp keeps two
// pairs in flight at 8 warps per SM; the full layout (unflagged ABI, host_step) keeps one slot of its size.
template <bool PACKED>
constexpr int pair_stages() { return PACKED ? 2 : 1; }

template <class M, class K, int G, bool PACKED>
struct PairScratch {
  using L = RowLayout<M, K>;
  static constexpr int E = M::EDIM;
  static constexpr int NST = pair_stages<PACKED>();
  static constexpr int TS = PACKED ? packed_doubles(E) : E * E;   // doubles of one filter's covariance tile
  alignas(128) double tile[NST * 2 * TS];             // covariance tile PAIRS (TMA ring)
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

// doubles of one filter's entry in the history slabs hP_pred / hP_filt
template <class M>
constexpr int hist_doubles() { return packed_hist<M>() ? packed_doubles(M::EDIM) : M::EDIM * M::EDIM; }

// M = PackedHist<model>: the history slabs hP_pred / hP_filt are packed (FLAG_PACKED_HIST).  (packed_hist<M>() and
// hist_doubles<M>() are not held in local constants: such a local moves the register allocation of the other instantiations.)
template <class M, class K, bool PRED, bool UPD, int G, bool GATHER, bool PACKED>
__global__ void __launch_bounds__(32, PAIR_MIN_WARPS) ekf_step_pair(const StepArgs<M::NG> a) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  using L = RowLayout<M, K>;
  using SC = PairScratch<M, K, G, PACKED>;
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
  if constexpr (GATHER) {
    if (mine) {
      myfid = (long long)a.idx[b0 + lane];
      // the entry's history slab element waits in its row (no register held through the kernel: the gather
      // instantiations are at the 8-warps-per-SM register limit)
      *reinterpret_cast<long long*>(myrow + L::OFF_HID) = hist_slot(a, b0 + lane, myfid);
    }
  }
  auto fid_of = [&](int f) -> long long {
    if constexpr (GATHER) return __shfl_sync(0xffffffffu, myfid, f);
    else return b0 + f;
  };
  // gather lists: history slab element of this lane's entry (-1: not recorded)
  auto my_hid = [&]() -> long long { return mine ? *reinterpret_cast<const long long*>(myrow + L::OFF_HID) : 0; };
  double* exh = s.exhp + h * XN;            // this half's exchange / (H P) buffer

  constexpr int NST = SC::NST;
  constexpr int TS = SC::TS;                // doubles of one filter's covariance in a.P
  constexpr uint32_t TILE_BYTES = TS * sizeof(double);
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
    double* dst = s.tile + slot * (2 * TS);
    if constexpr (GATHER) {
      tma_load_1d(dst, a.P + fidA * (long long)TS, TILE_BYTES, &s.full[slot]);
      if (np == 2) tma_load_1d(dst + TS, a.P + fidB * (long long)TS, TILE_BYTES, &s.full[slot]);
    } else {
      tma_load_1d(dst, a.P + fidA * (long long)TS, np * TILE_BYTES, &s.full[slot]);   // consecutive filters: one copy
    }
  };
  // full row-major a.P (without FLAG_PACKED_P) and hP_filt: the lane writes its lower blocks (I, hl), I >= hl, and their
  // transposes, so that the stored matrix is the exact mirror of its lower triangle
  // hP_pred, read only by the RTS backward pass: the lane writes its two columns, one coalesced 128-bit store per row.  Its
  // lower triangle is what store_full writes, its upper triangle the lane's own values (the mirror up to rounding).  The
  // transposed stores of store_full hit a different row per lane: on both slabs they made the forward pass with history
  // 1.5x slower.
  auto store_cols = [&](double* Pm, const double (&q0)[E], const double (&q1)[E]) {
#pragma unroll
    for (int i = 0; i < E; ++i) *reinterpret_cast<double2*>(Pm + i * E + c0) = make_double2(q0[i], q1[i]);
  };
  auto store_full = [&](double* Pm, const double (&q0)[E], const double (&q1)[E]) {
#pragma unroll
    for (int I = 0; I < E / 2; ++I) {
      if (I >= hl) {
        *reinterpret_cast<double2*>(Pm + 2 * I * E + c0) = make_double2(q0[2 * I], I == hl ? q0[2 * I + 1] : q1[2 * I]);
        *reinterpret_cast<double2*>(Pm + (2 * I + 1) * E + c0) = make_double2(q0[2 * I + 1], q1[2 * I + 1]);
      }
      if (I > hl) {
        *reinterpret_cast<double2*>(Pm + c0 * E + 2 * I) = make_double2(q0[2 * I], q0[2 * I + 1]);
        *reinterpret_cast<double2*>(Pm + (c0 + 1) * E + 2 * I) = make_double2(q1[2 * I], q1[2 * I + 1]);
      }
    }
  };
  // packed layout (a.P with FLAG_PACKED_P, both history slabs with FLAG_PACKED_HIST): the lane's blocks (I, hl), I >= hl,
  // one 32-byte block per iteration, two 128-bit stores.  For hP_pred this is the lower triangle of what store_cols writes.
  auto store_packed = [&](double* Pg, const double (&q0)[E], const double (&q1)[E]) {
#pragma unroll
    for (int I = 0; I < E / 2; ++I) {
      if (I >= hl) {
        double* q = Pg + packed_block(I, hl);
        *reinterpret_cast<double2*>(q) = make_double2(q0[2 * I], I == hl ? q0[2 * I + 1] : q1[2 * I]);
        *reinterpret_cast<double2*>(q + 2) = make_double2(q0[2 * I + 1], q1[2 * I + 1]);
      }
    }
  };
  auto store_hpred = [&](double* Pm, const double (&q0)[E], const double (&q1)[E]) {
    if constexpr (packed_hist<M>()) store_packed(Pm, q0, q1);
    else store_cols(Pm, q0, q1);
  };
  auto store_hfilt = [&](double* Pm, const double (&q0)[E], const double (&q1)[E]) {
    if constexpr (packed_hist<M>()) store_packed(Pm, q0, q1);
    else store_full(Pm, q0, q1);
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
    if constexpr (!GATHER) {
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
      if (GATHER) scatter_out<D, RS, true>(a.hx_pred, s.rows, L::OFF_X, ng, lane, my_hid());
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
      // gather lists: history slab element of this half's filter, read from its row where it is stored at each use (a
      // register held across the iteration spills)
      auto hist_el = [&]() -> long long { return *reinterpret_cast<const long long*>(s.rows + fi * RS + L::OFF_HID); };
      double* row = s.rows + fi * RS;
      const uint32_t slot = it % NST;
      const double* tile = s.tile + slot * (2 * TS) + (valid ? h : 0) * TS;
      double p0[E], p1[E];                        // columns c0 and c0 + 1
      double fv[L::NFp];   // loaded after the tile wait: loaded before it, the F slots spill inside the loop

      mbar_wait(&s.full[slot], (it / NST) & 1u);
      // P is defined by its lower triangle.  Rows 2I, 2I+1 of the owned columns are the 2x2 block (I, hl) when I >= hl and
      // the transpose of block (hl, I) when I < hl; either way the block arrives as two 128-bit loads u = first row,
      // v = second row, and only the two off-diagonal values swap places.  On the diagonal block (I == hl) the upper
      // element P[c0][c0+1] is taken from its lower mirror v.x.
#pragma unroll
      for (int I = 0; I < E / 2; ++I) {
        const int mx = I > hl ? I : hl, mn = I > hl ? hl : I;
        const double* pb = tile + (PACKED ? packed_block(mx, mn) : 2 * mx * E + 2 * mn);
        const double2 u = *reinterpret_cast<const double2*>(pb);
        const double2 v = *reinterpret_cast<const double2*>(pb + (PACKED ? 2 : E));
        p0[2 * I] = u.x;
        p1[2 * I] = I > hl ? u.y : v.x;
        p0[2 * I + 1] = I >= hl ? v.x : u.y;
        p1[2 * I + 1] = v.y;
      }
      const int fn = f + 2 * NST;
      const long long fa = fid_of(fn < ng ? fn : 0), fb = fid_of(fn + 1 < ng ? fn + 1 : 0);
      // WAR across proxies: the 128-bit shared loads above are generic-proxy reads that may still be queued when this
      // point is reached (a load is "issued", not "performed"); the bulk copy that refills the slot writes through the
      // async proxy.  The proxy fence orders the reads before it -- without it about one filter-step in 1e7 saw the last
      // tile rows of the NEXT pair (found as run-to-run differences of 10 000-step histories, scripts/dbg_rts_race.py).
      // Waiting on the register of the last load instead is not sufficient (66 of 250 runs still differed).
      fence_async_smem();
      __syncwarp();   // every lane holds its columns before the slot is refilled
      if (lane == 0 && fn < ng) issue_pair(fn, slot, fa, fb);
      ++it;

      if (do_pred) {
        vec_load(row + L::OFF_FV, fv);
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
          __syncwarp();
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
        if constexpr (GATHER) {
          const long long hb = hist_el();
          if (a.hP_pred && wr && hb >= 0) store_hpred(a.hP_pred + hb * (long long)hist_doubles<M>(), p0, p1);
        }
        else { if (a.hP_pred && wr) store_hpred(a.hP_pred + b * (long long)hist_doubles<M>(), p0, p1); }
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
        if constexpr (!GATHER) { if (a.hP_filt && wr && o == n_obs - 1) store_hfilt(a.hP_filt + b * (long long)hist_doubles<M>(), p0, p1); }   // = the state, bit for bit
        else {
          const long long hb = hist_el();
          if (a.hP_filt && wr && hb >= 0 && o == n_obs - 1) store_hfilt(a.hP_filt + hb * (long long)hist_doubles<M>(), p0, p1);
        }
      }

      const long long bp = GATHER ? fid_of(fi) : b;   // gather lists: shuffled again here rather than held through the update
      if (wr) {
        if constexpr (PACKED) {
          store_packed(a.P + bp * (long long)TS, p0, p1);
        } else {
          store_full(a.P + bp * (long long)(E * E), p0, p1);
        }
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
        if (GATHER) scatter_out<D, RS, true>(a.hx_filt, s.rows, L::OFF_X, ng, lane, my_hid());
        else stage_out<D, RS>(a.hx_filt + b0 * D, s.rows, L::OFF_X, ng, lane);
      }
    }
    __syncwarp();
  }
}

template <class M, class K, int G, bool PACKED>
constexpr size_t pair_smem_bytes() { return sizeof(PairScratch<M, K, G, PACKED>); }

template <class M>
constexpr bool use_pair() { return M::EDIM % 2 == 0 && M::EDIM <= 32; }

}  // namespace rnb
