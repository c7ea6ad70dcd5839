"""Histories recorded under RewindingScheduler on the device: streams with late observations, rewound and replayed per
filter, recorded into a RaggedHistory and RTS-smoothed.

6. With and without a history the scheduler computes the same x, P, clocks, innovations and counters, bit for bit.
7. The rewound history equals the one RaggedScheduler records from the same observations in time order, bit for bit,
   and so do their smoothed rows.
8. restore_from_history of the row a filter just recorded gives back its resident x and P, bit for bit, in every layout
   pair (on live also the packed history into a full P, through the C-ABI).
9. Live at 65 536 filters with a packed history: rewound == in order, and sampled filters against the oracle.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME as MSCKF_BY_NAME, batch as msckf_batch, observe as msckf_observe
from tests.shapes import BY_NAME as SHAPE_BY_NAME, batch as shape_batch, observe as shape_observe
from tests.util import LIVE_R, Oracle, cov_err, kinematic_batch, live_batch, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
PACKED_HIST = 64
CASES = ["live", "live_packed", "kinematic", "shape_e7", "shape_e31", "msckf_e18", "msckf_e28"]


def _case(name):
  """(engine factory, kinds {kind: (ZDIM, EADIM)}, per-filter observations {kind: (z [B, Z], R [B, Z, Z], ea [B, EA] or
  None)}, packed history, quaternion indices) of one kernel path."""
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  gv = None
  if name.startswith("live"):
    from rednose_b200.filters.live import LiveKalman
    cls, B, q = LiveKalman, 45, [3]
    x, P, Q = live_batch(B, seed=3)
    rng = np.random.default_rng(4)
    obs = {4: (rng.normal(0, 0.01, (B, 3)), None), 10: (rng.normal(0, 0.1, (B, 3)) + [0, 0, -9.8], None),
           12: (x[:, :3] + rng.normal(0, 5.0, (B, 3)), None)}
    obs = {k: (z, np.tile(np.diag(LIVE_R[k]), (B, 1, 1)), ea) for k, (z, ea) in obs.items()}
  elif name == "kinematic":
    from rednose_b200.filters.kinematic import KinematicKalman
    cls, B, q = KinematicKalman, 300, []
    x, P, Q, z, R = kinematic_batch(B, seed=4)
    obs = {1: (z, R, None)}
  else:
    msckf = name in MSCKF_BY_NAME
    cls = MSCKF_BY_NAME[name] if msckf else SHAPE_BY_NAME[name]
    m = hiprec.model_of(cls)
    m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
    gv = {g: m.gv[i] for i, g in enumerate(cls.global_names())}
    B, q = 2 * cls.group() + 1, cls.quat_idxs()
    x, P, Q, _ = (msckf_batch if msckf else shape_batch)(cls, B, seed=5)
    kinds = [k for k, v in cls.kinds().items() if not v[2] or (msckf and v[3])]
    obs = {k: (msckf_observe if msckf else shape_observe)(cls, m, k, x, seed=k) for k in kinds}
  folder = ensure_generated(cls)

  def engine():
    return BatchedEKF(folder, cls.name, Q, x, P, quaternion_idxs=q, global_vars=gv)
  kinds = {k: (z.shape[-1], 0 if ea is None else ea.shape[-1]) for k, (z, R, ea) in obs.items()}
  return engine, kinds, obs, name == "live_packed", q


def _stream(B, kinds, obs, seed, ticks=40):
  """Per tick: (ids, t, kinds, z_by_kind, R_by_kind, ea_by_kind), at most one observation per filter.  After tick 5 about
  15 % of the observations are 11-60 ms late (a rewind over 1-6 checkpoints, never before the filter's first one) and
  5 % are 3 s late, ignored.  Also returns each filter's applied observations in time order [(t, kind, z, R, ea)] and the
  number of ignored ones."""
  rng = np.random.default_rng(seed)
  first = np.full(B, np.nan)
  applied = [[] for _ in range(B)]
  out, ignored = [], 0
  ks = sorted(kinds)
  for tick in range(ticks):
    now = 0.01 * (tick + 1)
    ent = []
    for b in range(B):
      if rng.random() < 0.25:
        continue
      u, tb, k = rng.random(), now + 1e-5 * b, ks[int(rng.integers(len(ks)))]
      late = tick > 5 and not np.isnan(first[b])
      if late and u < 0.15:
        tb = max(tb - rng.uniform(0.011, 0.06), first[b] + 1e-6)
      z, R, ea = obs[k]
      zb = z[b] + 0.01 * rng.normal(size=z.shape[-1]) * np.sqrt(np.diagonal(R[b]))
      if late and 0.15 <= u < 0.20:
        ent.append((b, tb - 3.0, k, zb))
        ignored += 1
        continue
      if np.isnan(first[b]):
        first[b] = tb
      ent.append((b, tb, k, zb))
      applied[b].append((tb, k, zb, R[b], None if ea is None else ea[b]))
    if not ent:
      continue
    ids = np.array([e[0] for e in ent]); ts = np.array([e[1] for e in ent]); kk = np.array([e[2] for e in ent])
    zk, Rk, eak = {}, {}, {}
    for k in ks:
      s = [i for i, e in enumerate(ent) if e[2] == k]
      if not s:
        continue
      zk[k] = np.array([ent[i][3] for i in s]); Rk[k] = obs[k][1][ids[s]]
      if obs[k][2] is not None:
        eak[k] = obs[k][2][ids[s]]
    out.append((ids, ts, kk, zk, Rk, eak or None))
  for a in applied:
    a.sort(key=lambda v: v[0])
  return out, applied, ignored


def _in_order_ticks(applied, kinds):
  """Each filter's applied observations in time order, one per tick: tick j holds the j-th of every filter."""
  out = []
  for j in range(max(len(a) for a in applied)):
    bs = [b for b, a in enumerate(applied) if len(a) > j]
    ev = [applied[b][j] for b in bs]
    ids, ts, kk = np.array(bs), np.array([e[0] for e in ev]), np.array([e[1] for e in ev])
    zk, Rk, eak = {}, {}, {}
    for k in kinds:
      s = [i for i, e in enumerate(ev) if e[1] == k]
      if s:
        zk[k] = np.array([ev[i][2] for i in s]); Rk[k] = np.array([ev[i][3] for i in s])
        if ev[s[0]][4] is not None:
          eak[k] = np.array([ev[i][4] for i in s])
    out.append((ids, ts, kk, zk, Rk, eak or None))
  return out


def _rewinding(engine, kinds, history=None):
  from rednose_b200.scheduler import RewindingScheduler
  return RewindingScheduler(engine, {k: v[0] for k, v in kinds.items()}, depth=64, max_rewind_age=0.5,
                            ea_dims={k: v[1] for k, v in kinds.items() if v[1]}, history=history)


def _rows_equal(h1, h2):
  assert torch.equal(h1.n, h2.n)
  T, B = h1.t.shape
  below = torch.arange(T, device=h1.n.device)[:, None] < h1.n[None, :].long()
  for a1, a2 in ((h1.t, h2.t), (h1.x_pred, h2.x_pred), (h1.x_filt, h2.x_filt), (h1.P_pred, h2.P_pred), (h1.P_filt, h2.P_filt)):
    assert torch.equal(a1[below], a2[below])


def _smoothed(e, h, q):
  xs, Ps = torch.zeros_like(h.x_filt), torch.zeros_like(h.P_filt)     # rows >= n[b] stay 0 in both
  e.rts_smooth(h, norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,), out=(xs, Ps))
  return xs, Ps


@pytest.mark.parametrize("case", CASES)
def test_rewinding_with_history_equals_without_and_equals_in_order(case):
  """6: RewindingScheduler with and without a history, torch.equal on x, P, t_filter, every tick's innovations and the
  counters.  7: its history against RaggedScheduler's over the applied observations in time order, torch.equal on n, t,
  the four slabs below n and the smoothed rows."""
  from rednose_b200.scheduler import RaggedScheduler
  engine, kinds, obs, packed, q = _case(case)
  a, b, c = engine(), engine(), engine()
  T = 64
  h1 = b.new_ragged_history(T, packed=packed)
  s0, s1 = _rewinding(a, kinds), _rewinding(b, kinds, history=h1)
  ticks, applied, ignored = _stream(a.B, kinds, obs, seed=21)
  for tk in ticks:
    y0, y1 = s0.tick(*tk), s1.tick(*tk)
    assert y0.keys() == y1.keys()
    for k in y0:
      assert torch.equal(y0[k][0], y1[k][0]) and torch.equal(y0[k][1], y1[k][1]), k
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P) and torch.equal(s0.t_filter, s1.t_filter)
  assert (s0.rewinds, s0.replayed, s0.dropped) == (s1.rewinds, s1.replayed, s1.dropped)
  assert s1.rewinds > 10 and s1.replayed > s1.rewinds and s1.dropped == ignored > 0 and s1.unrecorded == 0
  assert h1.overflowed() == 0 and h1.n.tolist() == [len(v) for v in applied]
  # 7. the same observations in time order
  h2 = c.new_ragged_history(T, packed=packed)
  s2 = RaggedScheduler(c, history=h2)
  for tk in _in_order_ticks(applied, kinds):
    s2.tick(*tk)
  assert s2.dropped == 0 and torch.equal(b.x, c.x) and torch.equal(b.P, c.P)
  _rows_equal(h1, h2)
  xs1, Ps1 = _smoothed(b, h1, q)
  xs2, Ps2 = _smoothed(c, h2, q)
  assert torch.equal(xs1, xs2) and torch.equal(Ps1, Ps2)


@pytest.mark.parametrize("case", CASES)
def test_restore_of_the_row_just_recorded_gives_back_the_resident_state(case):
  """8: every filter steps twice with recording; x and P are then overwritten, and restore_from_history of each
  filter's last row (one entry with row -1 left untouched) brings them back bit for bit."""
  engine, kinds, obs, packed, q = _case(case)
  e = engine()
  B = e.B
  h = e.new_ragged_history(4, packed=packed)
  k = sorted(kinds)[0]
  z, R, ea = obs[k]
  ids = torch.arange(B, dtype=torch.int32, device="cuda")
  dev = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()   # noqa: E731
  for j in range(2):
    e.step_indexed(k, ids, torch.full((B,), 0.01 * j, dtype=torch.float64, device="cuda"), dev(z).clone(), dev(R), dev(ea),
                   hist=h, t=0.01 * j)
  x0, P0 = e.x.clone(), e.P.clone()
  rows = torch.ones(B, dtype=torch.int32, device="cuda")
  rows[B // 2] = -1
  e.x.zero_()
  e.set_P_rows(ids, torch.zeros(B, e.dim_err, e.dim_err, dtype=torch.float64, device="cuda"))
  e.restore_from_history(h, ids, rows)
  keep = torch.ones(B, dtype=torch.bool, device="cuda"); keep[B // 2] = False
  assert torch.equal(e.x[keep], x0[keep]) and torch.equal(e.P[keep], P0[keep])
  assert not e.x[B // 2].any() and not e.P[B // 2].any()


def test_live_restore_through_the_c_abi_in_the_full_resident_layout():
  """8, the pairs the engine does not produce on live: history (packed or full) into a full [B, EDIM, EDIM] P, against
  unpack_P of the packed rows and the full rows themselves."""
  engine, kinds, obs, _, _ = _case("live")
  e = engine()
  B, D, E = e.B, e.dim_x, e.dim_err
  hp, hf = e.new_ragged_history(3, packed=True), e.new_ragged_history(3)
  ids = torch.arange(B, dtype=torch.int32, device="cuda")
  z, R, _ = obs[12]
  for h in (hp, hf):
    e2 = engine()
    for j in range(3):
      e2.step_indexed(12, ids, torch.full((B,), 0.01, dtype=torch.float64, device="cuda"),
                      torch.as_tensor(z).cuda().clone(), torch.as_tensor(R).cuda(), hist=h, t=0.01 * j)
  sel = torch.tensor([3, 0, 17, B - 1, 8], dtype=torch.int32, device="cuda")
  rows = torch.tensor([2, 0, -1, 1, 2], dtype=torch.int32, device="cuda")
  for h, flag in ((hp, PACKED_HIST), (hf, 0)):
    x = torch.full((B, D), -1.0, dtype=torch.float64, device="cuda")
    P = torch.full((B, E, E), -1.0, dtype=torch.float64, device="cuda")
    st = e._lib.live_batch_restore_hist(e._cp(h.x_filt), e._cp(h.P_filt), e._ffi.cast("const int *", sel.data_ptr()),
                                        e._ffi.cast("const int *", rows.data_ptr()), 5, B, e._p(x), e._p(P), flag, e._stream())
    torch.cuda.synchronize()
    assert st == 0 and e._lib.live_cuda_status() == 0
    s, r = sel[rows >= 0].long(), rows[rows >= 0].long()
    want = e.unpack_P(h.P_filt[r, s]) if flag else h.P_filt[r, s]
    assert torch.equal(x[s], h.x_filt[r, s]) and torch.equal(P[s], want)
    untouched = torch.ones(B, dtype=torch.bool, device="cuda"); untouched[s] = False
    assert bool((x[untouched] == -1.0).all()) and bool((P[untouched] == -1.0).all())


# ------------------------------------------------------------------------------------------------------------ 9. scale ---
def _live_gnss_late(B, ticks, rng):
  """Config-3-like live streams: every 10 ms tick each filter observes its gyro (4) or accelerometer (10), alternating
  with a per-filter phase, ~3 % missing; one position fix (12) per filter, time-stamped in 0.06-0.15 s and arriving
  50-300 ms later, in place of that tick's IMU sample.  Returns per tick (ids, t, kinds) as arrays."""
  ph = rng.integers(0, 2, B)
  jit = rng.uniform(0, 0.005, B)
  tg = rng.uniform(0.06, 0.15, B)
  arrive = np.minimum(((tg + rng.uniform(0.05, 0.3, B)) / 0.01).astype(int), ticks - 1)
  out = []
  for j in range(ticks):
    t = 0.01 * (j + 1) + jit
    kind = np.where((j + ph) % 2 == 0, 4, 10)
    keep = (rng.random(B) >= 0.03) | (j < 5)       # every filter has checkpointed before its fix's time stamp
    g = arrive == j
    t = np.where(g, tg, t)
    kind = np.where(g, 12, kind)
    keep |= g
    out.append((np.flatnonzero(keep), t[keep], kind[keep]))
  return out


def test_live_65536_filters_packed_history_rewound_equals_in_order(oracle_dir):
  from oracle.rts_numpy import rts_smooth
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RaggedScheduler
  o = Oracle(oracle_dir, "live")
  B, ticks, T = 65536, 45, 52
  rng = np.random.default_rng(31)
  x, P, Q = live_batch(B, seed=31)
  folder = ensure_generated(LiveKalman)
  a, c = (BatchedEKF(folder, "live", Q, x, P, quaternion_idxs=[3]) for _ in range(2))
  zf = {4: rng.normal(0, 0.01, (B, 3)), 10: rng.normal(0, 0.1, (B, 3)) + [0, 0, -9.8], 12: x[:, :3] + rng.normal(0, 5.0, (B, 3))}
  Rk = {k: np.diag(LIVE_R[k]) for k in (4, 10, 12)}
  stream = _live_gnss_late(B, ticks, rng)
  h1 = a.new_ragged_history(T, packed=True)
  s1 = _rewinding(a, {4: (3, 0), 10: (3, 0), 12: (3, 0)}, history=h1)
  applied = [[] for _ in range(B)]
  for ids, t, kinds in stream:
    zt = {k: zf[k][ids[kinds == k]] + 1e-3 * t[kinds == k, None] for k in (4, 10, 12) if (kinds == k).any()}
    s1.tick(ids, t, kinds, zt, {k: np.tile(Rk[k], (len(zt[k]), 1, 1)) for k in zt})
    for k in zt:
      for b, tb, zb in zip(ids[kinds == k], t[kinds == k], zt[k]):
        applied[b].append((tb, k, zb))
  assert s1.dropped == 0 and s1.unrecorded == 0 and s1.rewinds > B // 2 and h1.overflowed() == 0
  for v in applied:
    v.sort(key=lambda e: e[0])
  h2 = c.new_ragged_history(T, packed=True)
  s2 = RaggedScheduler(c, history=h2)
  for j in range(max(len(v) for v in applied)):
    bs = np.array([b for b in range(B) if len(applied[b]) > j])
    ev = [applied[b][j] for b in bs]
    kk = np.array([e[1] for e in ev])
    zk = {k: np.array([e[2] for e, kind in zip(ev, kk) if kind == k]) for k in (4, 10, 12) if (kk == k).any()}
    s2.tick(bs, np.array([e[0] for e in ev]), kk, zk, {k: np.tile(Rk[k], (len(zk[k]), 1, 1)) for k in zk})
  assert torch.equal(a.x, c.x) and torch.equal(a.P, c.P)
  _rows_equal(h1, h2)
  xs1, Ps1 = _smoothed(a, h1, [3])
  xs2, Ps2 = _smoothed(c, h2, [3])
  assert torch.equal(xs1, xs2) and torch.equal(Ps1, Ps2)
  # 16 sampled filters: per-filter oracle driving in time order, and oracle/rts_numpy over their rows
  n = h1.n.cpu().numpy()
  xk, Pk = a.state(), a.covs()
  for b in np.random.default_rng(32).choice(B, 16, replace=False):
    xr, Pr, tl = x[b:b + 1], P[b:b + 1], None
    for tb, k, zb in applied[b]:
      xr, Pr, _ = o.batch_step(k, xr, Pr, Q, 0.0 if tl is None else tb - tl, zb[None], Rk[k][None], quat_idxs=[3], flags=3)
      tl = tb
    assert state_err(xk[b], xr[0]) < TIGHT and cov_err(Pk[b], Pr[0]) < TIGHT, b
    k = int(n[b])
    slabs = [s[:k, b].cpu().numpy() for s in (h1.x_pred, h1.x_filt)] + [a.unpack_P(s[:k, b]).cpu().numpy() for s in (h1.P_pred, h1.P_filt)]
    xo, Po = rts_smooth(o, *slabs, h1.t[:k, b].cpu().numpy(), 23, 22, norm_quats=True)
    ex, eP = state_err(xs1[:k, b].cpu().numpy(), xo), cov_err(a.unpack_P(Ps1[:k, b]).cpu().numpy(), Po)
    assert ex < TIGHT and eP < TIGHT, (b, ex, eP)
