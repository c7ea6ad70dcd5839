"""Ragged histories on the device: every filter records its own steps (RaggedScheduler / step_indexed with a
RaggedHistory) and is RTS-smoothed over its own rows and times (rts_smooth(RaggedHistory)).

1. A lockstep stream recorded this way is bit-identical to step_recorded + rts_smooth(History) on every kernel path.
2. Ragged streams at every tests/shapes.py shape and at the MSCKF shapes with a smoother, against the 40-digit reference
   of tests/hiprec.py.
3. Live IMU + GNSS streams on per-filter clocks, against per-filter oracle driving and oracle/rts_numpy.
4. A filter that outruns the history keeps stepping; the smoother refuses the history and says how many steps were lost.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME as MSCKF_BY_NAME, batch as msckf_batch, observe as msckf_observe
from tests.shapes import SHAPES, batch as shape_batch, observe as shape_observe
from tests.util import LIVE_R, Oracle, cov_err, kinematic_batch, live_batch, live_obs, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9


def _engine(folder, name, x, P, Q, quats, global_vars=None):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(folder, name, Q, x, P, quaternion_idxs=quats, global_vars=global_vars)


def _dev(a):
  return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------------- 1. lockstep ---
def _lockstep_case(name):
  """(folder, engine name, x, P, Q, quats, [(kind, z, R, ea)] per tick) of one kernel path."""
  from rednose_b200.filters import ensure_generated
  if name == "live":
    from rednose_b200.filters.live import LiveKalman
    x, P, Q = live_batch(45, seed=3)
    ticks = []
    for k, kind in enumerate([4, 10, 12, 4, 10]):
      R = np.tile(np.diag(LIVE_R[kind]), (45, 1, 1))
      z = np.random.default_rng(k).normal(0, 0.05, (45, 3)) + (x[:, :3] if kind == 12 else [0, 0, -9.8] if kind == 10 else 0)
      ticks.append((kind, z, R, None))
    return ensure_generated(LiveKalman), "live", x, P, Q, [3], ticks
  if name == "kinematic":
    from rednose_b200.filters.kinematic import KinematicKalman
    x, P, Q, z, R = kinematic_batch(300, seed=4)
    ticks = [(1, z + 0.01 * k, R, None) for k in range(5)]
    return ensure_generated(KinematicKalman), "kinematic", x, P, Q, [], ticks
  if name == "shape_e7":
    from tests.shapes import BY_NAME
    cls = BY_NAME[name]
    m = hiprec.model_of(cls)
    m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
    x, P, Q, _ = shape_batch(cls, 2 * cls.group() + 1, seed=5)
    kinds = [k for k, (_, _, g) in cls.kinds().items() if not g]
    ticks = [(kinds[k % len(kinds)],) + shape_observe(cls, m, kinds[k % len(kinds)], x, seed=k) for k in range(5)]
    return ensure_generated(cls), cls.name, x, P, Q, cls.quat_idxs(), ticks
  cls = MSCKF_BY_NAME[name]
  m = hiprec.model_of(cls)
  x, P, Q, _ = msckf_batch(cls, 9, seed=6)
  fk = cls.feature_kinds()[0]
  plain = [k for k, v in cls.kinds().items() if not v[3]][0]
  ticks = [(kind,) + msckf_observe(cls, m, kind, x, seed=k) for k, kind in enumerate([fk, plain, fk])]
  return ensure_generated(cls), cls.name, x, P, Q, cls.quat_idxs(), ticks


@pytest.mark.parametrize("case", ["live", "kinematic", "shape_e7", "msckf_e18", "msckf_e28"])
def test_lockstep_stream_equals_lockstep_recording_bit_for_bit(case):
  """Every filter observes every tick with the same kind and time: RaggedScheduler(history=) + rts_smooth(ragged) ==
  step_recorded + rts_smooth(History), torch.equal on x, P, the four slabs and the smoothed rows."""
  from rednose_b200.scheduler import RaggedScheduler
  folder, name, x, P, Q, q, ticks = _lockstep_case(case)
  B, T = x.shape[0], len(ticks)
  a, b = _engine(folder, name, x, P, Q, q), _engine(folder, name, x, P, Q, q)
  h = a.new_history(T)
  rh = b.new_ragged_history(T)
  sch = RaggedScheduler(b, history=rh)
  ids = np.arange(B)
  for k, (kind, z, R, ea) in enumerate(ticks):
    t = 0.02 * k + 0.005 * (k % 2)
    a.step_recorded(h, kind, t, z, R, ea)
    sch.tick(ids, t, np.full(B, kind), {kind: z}, {kind: R}, None if ea is None else {kind: ea})
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)
  for s1, s2 in ((h.x_pred, rh.x_pred), (h.P_pred, rh.P_pred), (h.x_filt, rh.x_filt), (h.P_filt, rh.P_filt)):
    assert torch.equal(s1, s2)
  assert rh.n.tolist() == [T] * B and torch.equal(rh.t, h.t.new_tensor(h.t_host)[:, None].expand(T, B))
  kw = dict(norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
  xs1, Ps1 = a.rts_smooth(h, **kw)
  xs2, Ps2 = b.rts_smooth(rh, **kw)
  assert torch.equal(xs1, xs2) and torch.equal(Ps1, Ps2)


# ------------------------------------------------------------------------------------------- 2. every shape, hiprec ---
RAGGED_SHAPES = SHAPES + [MSCKF_BY_NAME[n] for n in ("msckf_e18", "msckf_e27", "msckf_e28")]


@pytest.mark.parametrize("cls", RAGGED_SHAPES, ids=[c.name for c in RAGGED_SHAPES])
def test_ragged_streams_against_the_40_digit_reference(cls):
  """B = 2G + 1 filters with 0 .. T recorded steps each, mixed kinds, irregular times, zero-dt pairs, one entry with two
  observations.  Final x / P of sampled filters against a per-filter 40-digit replay; their smoothed rows against
  hiprec.rts over their own rows and times (with and without quaternion normalisation); rows past n[b] untouched.
  An MSCKF (EDIM <= 32) also runs its gated feature kind on the CTA kernel and is smoothed on its main block."""
  from rednose_b200.filters import ensure_generated
  msckf = cls in MSCKF_BY_NAME.values()
  batch, observe = (msckf_batch, msckf_observe) if msckf else (shape_batch, shape_observe)
  G = cls.group()
  B, T = 2 * G + 1, 5
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  x, P, Q, _ = batch(cls, B, seed=90)
  q = cls.quat_idxs()
  kinds = [k for k, v in cls.kinds().items() if not v[2] or (msckf and v[3])]
  rng = np.random.default_rng(91)
  mask = rng.random((B, T)) < 0.6
  mask[0] = False                       # no step at all
  mask[1] = False; mask[1, 2] = True    # exactly one step
  mask[2] = True                        # every row used
  t_b = np.cumsum(rng.uniform(0.005, 0.04, (B, T)), axis=1)
  t_b[2, 3] = t_b[2, 2]                 # zero-dt pair
  t_b[G, 1:] = t_b[G, 0]; mask[G, :2] = True
  two = 3; mask[two, 1] = True          # filter 3's entry at tick 1 carries two observations
  obs = {k: observe(cls, m, k, x, seed=92 + k, n_obs=2) for k in kinds}    # [B, 2, ...] per kind
  e = _engine(ensure_generated(cls), cls.name, x, P, Q, q, {g: m.gv[i] for i, g in enumerate(cls.global_names())})
  rh = e.new_ragged_history(T)
  entries = [[] for _ in range(B)]      # per filter: (kind, dt, z, R, ea) as applied
  t_last = np.full(B, np.nan)
  for k in range(T):
    act = np.flatnonzero(mask[:, k])
    kind_of = rng.choice(kinds, act.size)
    for kind in kinds:
      sel = act[kind_of == kind]
      for grp in ([s for s in sel if not (s == two and k == 1)], [s for s in sel if s == two and k == 1]):
        if not grp:
          continue
        grp = np.array(grp)
        nobs = 2 if (grp[0] == two and k == 1) else 1
        z, R, ea = obs[kind]
        zg, Rg = z[grp, :nobs], R[grp, :nobs]
        eag = None if ea is None else ea[grp, :nobs]
        tk = t_b[grp, k]
        dt = np.where(np.isnan(t_last[grp]), 0.0, tk - t_last[grp])
        t_last[grp] = tk
        e.step_indexed(kind, _dev(grp.astype(np.int32)), _dev(dt), zg.copy(), Rg, eag, hist=rh, t=_dev(tk))
        for i, b in enumerate(grp):
          entries[b].append((kind, dt[i], zg[i], Rg[i], None if eag is None else eag[i]))
  n = rh.n.cpu().numpy()
  assert n.tolist() == [len(v) for v in entries] and n[0] == 0 and n[1] == 1 and n[2] == T
  sel = sorted({1, 2, two, G - 1, G, B - 1})
  xk, Pk = e.state(), e.covs()
  for b in sel:   # final state of a per-filter replay
    xr, Pr = x[b:b + 1], P[b:b + 1]
    for kind, dt, z, R, ea in entries[b]:
      xr, Pr, _ = hiprec.step(m, kind, xr, Pr, Q, dt, z[None], R[None], None if ea is None else ea[None], quat_idxs=q)
    ex, eP = state_err(xk[b], xr[0]), cov_err(Pk[b], Pr[0])
    assert ex < TIGHT and eP < TIGHT, (b, ex, eP)
  slabs = [s.cpu().numpy() for s in (rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt)]
  tt = rh.t.cpu().numpy()
  for norm in ([False, True] if q else [False]):
    xs, Ps = (torch.full_like(s, float("nan")) for s in (rh.x_filt, rh.P_filt))
    e.rts_smooth(rh, norm_quats=norm, quaternion_idxs=tuple(q) or (0,), out=(xs, Ps))
    xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
    for b in range(B):
      assert np.isnan(xs[n[b]:, b]).all() and np.isnan(Ps[n[b]:, b]).all()
      assert not np.isnan(xs[:n[b], b]).any()
    for b in sel:
      k = int(n[b])
      xr, Pr = hiprec.rts(m, *[s[:k, b:b + 1] for s in slabs], tt[:k, b], quat_idxs=q, norm_quats=norm)
      ex, eP = state_err(xs[:k, b], xr[:, 0]), cov_err(Ps[:k, b], Pr[:, 0])
      print(f"{cls.name} ragged rts filter {b} ({k} rows, norm {norm}): state {ex:.1e} cov {eP:.1e}")
      assert ex < TIGHT and eP < TIGHT, (b, norm, ex, eP)


# -------------------------------------------------------------------------------------- 3. live IMU + GNSS, oracle ---
def _imu_gnss_streams(B, seconds, rng):
  """Config-3 streams on per-filter clocks: 100 Hz gyro (4) and accelerometer (10), 1 Hz position (12), each filter
  with its own phase, ~3 % of the samples missing.  Returns a time-ordered list of (t, filter, kind)."""
  ev = []
  for b in range(B):
    ph = rng.uniform(0, 0.01)
    for i in range(int(seconds * 100)):
      for kind, off in ((4, 0.0), (10, 0.004)):
        if rng.random() > 0.03:
          ev.append((ph + 0.01 * i + off, b, kind))
    gph = rng.uniform(0, min(1.0, seconds))
    for i in range(int(seconds) + 1):
      if gph + i < seconds:
        ev.append((gph + i, b, 12))
  ev.sort()
  return ev


def _run_live_streams(B, T, seconds, seed, oracle_dir):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RaggedScheduler
  o = Oracle(oracle_dir, "live")
  rng = np.random.default_rng(seed)
  x, P, Q = live_batch(B, seed=seed)
  e = _engine(ensure_generated(LiveKalman), "live", x, P, Q, [3])
  rh = e.new_ragged_history(T)
  sch = RaggedScheduler(e, history=rh)
  xr, Pr = x.copy(), P.copy()
  t_ref = np.full(B, np.nan)
  ev = _imu_gnss_streams(B, seconds, rng)
  # ticks of 10 ms: at most one observation per filter per tick (the earliest; the rest wait for the next tick)
  pending, tick_end = list(ev), 0.01
  while pending:
    taken, rest, seen = [], [], set()
    for item in pending:
      if item[0] < tick_end and item[1] not in seen:
        taken.append(item); seen.add(item[1])
      else:
        rest.append(item)
    pending, tick_end = rest, tick_end + 0.01
    if not taken:
      continue
    t_obs = np.array([a[0] for a in taken]); ids = np.array([a[1] for a in taken]); kinds = np.array([a[2] for a in taken])
    zs, Rs = {}, {}
    for k in (4, 10, 12):
      s = kinds == k
      if not s.any():
        continue
      f = ids[s]
      zk, Rk = live_obs(o, k, xr[f], seed=int(tick_end * 1000))
      zs[k], Rs[k] = zk, Rk
      dt = np.where(np.isnan(t_ref[f]), 0.0, t_obs[s] - t_ref[f])
      xr[f], Pr[f], _ = o.batch_step(k, xr[f], Pr[f], Q, dt, zk, Rk, quat_idxs=[3], flags=3)
      t_ref[f] = t_obs[s]
    sch.tick(ids, t_obs, kinds, zs, Rs)
  assert sch.dropped == 0
  return o, e, rh, xr, Pr


def test_live_imu_gnss_streams_against_the_oracle(oracle_dir):
  from oracle.rts_numpy import rts_smooth
  B, T = 2000, 64
  o, e, rh, xr, Pr = _run_live_streams(B, T, 0.3, 11, oracle_dir)
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT
  n = rh.n.cpu().numpy()
  assert rh.overflowed() == 0 and n.min() >= 40 and n.max() <= T and len(set(n.tolist())) > 3
  xs, Ps = e.rts_smooth(rh, norm_quats=True)
  for b in (0, 1, 777, B - 1):
    k = int(n[b])
    slabs = [s[:k, b].cpu().numpy() for s in (rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt)]
    xo, Po = rts_smooth(o, *slabs, rh.t[:k, b].cpu().numpy(), 23, 22, norm_quats=True)
    ex, eP = state_err(xs[:k, b].cpu().numpy(), xo), cov_err(Ps[:k, b].cpu().numpy(), Po)
    print(f"live ragged rts filter {b} ({k} rows): state {ex:.1e} cov {eP:.1e}")
    assert ex < TIGHT and eP < TIGHT, (b, ex, eP)


# ------------------------------------------------------------------------------------------------------ 4. overflow ---
def test_overflowing_filter_keeps_stepping_and_the_smoother_refuses(oracle_dir):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  o = Oracle(oracle_dir, "live")
  B, T = 3, 4
  x, P, Q = live_batch(B, seed=12)
  e = _engine(ensure_generated(LiveKalman), "live", x, P, Q, [3])
  rh = e.new_ragged_history(T)
  xr, Pr = x.copy(), P.copy()
  first = None
  for k in range(T + 3):                    # filter 0 steps T + 3 times, filter 1 twice, filter 2 never
    ids = np.array([0, 1]) if k < 2 else np.array([0])
    z, R = live_obs(o, 4, xr[ids], seed=k)
    dt = 0.0 if k == 0 else 0.01
    e.step_indexed(4, _dev(ids.astype(np.int32)), _dev(np.full(ids.size, dt)), z.copy(), R, hist=rh, t=0.01 * k)
    xr[ids], Pr[ids], _ = o.batch_step(4, xr[ids], Pr[ids], Q, dt, z, R, quat_idxs=[3], flags=3)
    if k == T - 1:
      first = [s[:, 0].clone() for s in (rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt)]
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT
  assert rh.n.tolist() == [T, 2, 0] and rh.overflowed() == 3
  for s, f in zip((rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt), first):
    assert torch.equal(s[:, 0], f)          # the first T rows are intact
  assert rh.t[:, 0].tolist() == [0.0, 0.01, 0.02, 0.03]
  with pytest.raises(RuntimeError, match="overflow: 3 step"):
    e.rts_smooth(rh)
