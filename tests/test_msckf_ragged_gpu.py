"""MSCKF filters on their own clocks: clone-window shifts of listed filters (augment(ids), step_indexed(augment=)), through
RaggedScheduler, RewindingScheduler and RaggedCheckpointedSmoother.

1. augment(ids) at every MSCKF shape: listed filters are augment_np of their state, the others untouched, bit for bit.
2. step_indexed(augment=mask), a feature kind and a plain kind: bit for bit step_indexed + augment_np of the flagged
   filters; recorded rows are the estimates before the shift.
3. Per-filter MSCKF streams with shifting camera frames through RaggedScheduler against the 40-digit reference of
   tests/hiprec.py (smoothed rows too where a ragged smoother exists), and the shipped msckf against the oracle.
4. Lockstep streams with shifts: RaggedScheduler(history=) + rts_smooth == step_recorded(augment=True) + rts_smooth.
5. RewindingScheduler with frames 50-300 ms late == RaggedScheduler fed the same observations in time order.
6. RaggedCheckpointedSmoother with shifting ticks == one whole ragged pass, bit for bit.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME, MSCKF_SHAPES, augment_np, batch, observe
from tests.util import cov_err, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
IDS = [c.name for c in MSCKF_SHAPES]
SMOOTHED = ("msckf_e18", "msckf_e27", "msckf_e28")


def _engine(cls, x, P, Q, m=None):
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  gv = {} if m is None else {g: m.gv[i] for i, g in enumerate(cls.global_names())}
  return BatchedEKF(ensure_generated(cls), cls.name, Q, x, P, quaternion_idxs=cls.quat_idxs(), global_vars=gv)


def _model(cls):
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  return m


def _dev(a):
  return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _plain(cls):
  return [k for k, v in cls.kinds().items() if not v[3] and not v[2]][0]


# ---------------------------------------------------------------------------------------------------- 1. augment ---
@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_augment_listed_filters(cls):
  B = 70
  x, P, Q, _ = batch(cls, B, seed=10)
  e = _engine(cls, x, P, Q)
  ids = np.random.default_rng(11).permutation(B)[:41]                 # unordered, 29 filters not listed
  e.augment(_dev(ids.astype(np.int32)))
  xa, Pa = augment_np(cls, x[ids], P[ids])
  rest = np.setdiff1d(np.arange(B), ids)
  assert np.array_equal(e.state()[ids], xa) and np.array_equal(e.covs()[ids], Pa)
  assert np.array_equal(e.state()[rest], x[rest]) and np.array_equal(e.covs()[rest], P[rest])
  launches = e.launches
  e.augment(np.zeros(0, dtype=np.int32))                              # empty: nothing happens
  e.augment(torch.zeros(0, dtype=torch.int32, device="cuda"))
  assert e.launches == launches
  assert np.array_equal(e.state()[ids], xa) and np.array_equal(e.state()[rest], x[rest])
  e.augment(ids.tolist())                                             # host ids
  xb, Pb = augment_np(cls, xa, Pa)
  assert np.array_equal(e.state()[ids], xb) and np.array_equal(e.covs()[ids], Pb)


# ------------------------------------------------------------------------------------------ 2. step_indexed(augment) ---
@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_step_indexed_with_a_mixed_augment_mask(cls):
  m = _model(cls)
  B = 70
  x, P, Q, dt = batch(cls, B, seed=20)
  n = 66
  idx = np.random.default_rng(21).permutation(B)[:n].astype(np.int32)
  mask = np.random.default_rng(22).random(n) < 0.5
  for kind in (cls.feature_kinds()[0], _plain(cls)):
    z, R, ea = observe(cls, m, kind, x[idx], seed=23 + kind)
    a, b = _engine(cls, x, P, Q, m), _engine(cls, x, P, Q, m)
    ya = a.step_indexed(kind, _dev(idx), _dev(dt[:n]), z.copy(), R, ea)
    yb = b.step_indexed(kind, _dev(idx), _dev(dt[:n]), z.copy(), R, ea, augment=_dev(mask))
    assert torch.equal(ya, yb), kind                                  # innovations in the order of idx
    xa, Pa = a.state(), a.covs()
    xs, Ps = augment_np(cls, xa[idx[mask]], Pa[idx[mask]])
    xa[idx[mask]], Pa[idx[mask]] = xs, Ps
    assert np.array_equal(b.state(), xa) and np.array_equal(b.covs(), Pa), kind
    # recorded: rows hold the estimate before the shift
    c, d = _engine(cls, x, P, Q, m), _engine(cls, x, P, Q, m)
    hc, hd = c.new_ragged_history(2), d.new_ragged_history(2)
    c.step_indexed(kind, _dev(idx), _dev(dt[:n]), z.copy(), R, ea, hist=hc, t=0.5)
    d.step_indexed(kind, _dev(idx), _dev(dt[:n]), z.copy(), R, ea, hist=hd, t=_dev(np.full(n, 0.5)), augment=_dev(mask))
    for s1, s2 in ((hc.x_pred, hd.x_pred), (hc.P_pred, hd.P_pred), (hc.x_filt, hd.x_filt), (hc.P_filt, hd.P_filt)):
      assert torch.equal(s1[:1, idx], s2[:1, idx]), kind
    assert torch.equal(hc.n, hd.n) and torch.equal(hc.t, hd.t)
    assert np.array_equal(d.state(), xa) and np.array_equal(d.covs(), Pa), kind
  e = _engine(cls, x, P, Q, m)                                        # all flagged, and a scalar True
  z, R, ea = observe(cls, m, _plain(cls), x[idx], seed=40)
  e.step_indexed(_plain(cls), _dev(idx), _dev(dt[:n]), z.copy(), R, ea, augment=True)
  f = _engine(cls, x, P, Q, m)
  f.step_indexed(_plain(cls), _dev(idx), _dev(dt[:n]), z.copy(), R, ea)
  f.augment(_dev(idx))
  assert torch.equal(e.x, f.x) and torch.equal(e.P, f.P)


# ------------------------------------------------------------------------------------------- 3. streams, hiprec ---
def _frame_streams(cls, m, B, n_ticks, seed):
  """Per filter: a plain kind at every tick but frame ticks, a feature frame (augment) every 3 ticks at a per-filter phase;
  filters 0 and 1 have no frames; about 10 % of the samples are missing.  Returns the ticks as RaggedScheduler.tick
  arguments."""
  rng = np.random.default_rng(seed)
  plain, feat = _plain(cls), cls.feature_kinds()[0]
  phase = rng.integers(0, 3, B)
  phase[:2] = -1
  x, _, _, _ = batch(cls, B, seed=seed)
  obs = {k: observe(cls, m, k, x, seed=seed + k, n_obs=n_ticks) for k in (plain, feat)}
  times = 0.01 * np.arange(1, n_ticks + 1)[None, :] + rng.uniform(0, 0.005, (B, 1))
  ticks = []
  for j in range(n_ticks):
    ids, kinds, aug = [], [], []
    for b in range(B):
      frame = phase[b] >= 0 and j % 3 == phase[b]
      if not frame and rng.random() < 0.1:
        continue
      ids.append(b); kinds.append(feat if frame else plain); aug.append(bool(frame))
    ids, kinds = np.array(ids), np.array(kinds)
    z, R, ea = {}, {}, {}
    for k in (plain, feat):
      s = ids[kinds == k]
      if s.size:
        zk, Rk, eak = obs[k]
        z[k], R[k] = zk[s, j].copy(), Rk[s, j]
        if eak is not None:
          ea[k] = eak[s, j]
    ticks.append((ids, times[ids, j], kinds, z, R, ea or None, np.array(aug)))
  return ticks


def _replay(cls, m, x, P, Q, ticks, b):
  """Filter b's stream through hiprec, augment_np after each frame: (final x, P)."""
  q = cls.quat_idxs()
  xr, Pr, tl = x[b:b + 1], P[b:b + 1], None
  for ids, t, kinds, z, R, ea, aug in ticks:
    w = np.flatnonzero(ids == b)
    if not w.size:
      continue
    w = int(w[0]); k = int(kinds[w]); pos = int(np.sum(kinds[:w] == k))
    dt = 0.0 if tl is None else t[w] - tl
    tl = t[w]
    eak = None if (ea is None or k not in ea) else ea[k][pos:pos + 1]
    xr, Pr, _ = hiprec.step(m, k, xr, Pr, Q, dt, z[k][pos:pos + 1], R[k][pos:pos + 1], eak, quat_idxs=q)
    if aug[w]:
      xr, Pr = augment_np(cls, xr, Pr)
  return xr[0], Pr[0]


@pytest.mark.parametrize("name", SMOOTHED + ("msckf_e33", "msckf_e64"))
def test_frame_streams_against_the_40_digit_reference(name):
  """Final x / P of sampled filters against a per-filter 40-digit replay; at EDIM <= 32 also their smoothed rows."""
  from rednose_b200.scheduler import RaggedScheduler
  cls = BY_NAME[name]
  m = _model(cls)
  smooth = name in SMOOTHED
  B, n_ticks = (2 * cls.group() + 1, 7) if smooth else (9, 5)
  x, P, Q, _ = batch(cls, B, seed=300)
  ticks = _frame_streams(cls, m, B, n_ticks, seed=301)
  e = _engine(cls, x, P, Q, m)
  rh = e.new_ragged_history(n_ticks) if smooth else None
  s = RaggedScheduler(e, history=rh)
  for tk in ticks:
    s.tick(*tk)
  sel = sorted({0, 2, 3, 4, B - 1} | ({cls.group() - 1, cls.group()} if smooth else set()))
  xk, Pk = e.state(), e.covs()
  for b in sel:
    xr, Pr = _replay(cls, m, x, P, Q, ticks, b)
    ex, eP = state_err(xk[b], xr), cov_err(Pk[b], Pr)
    print(f"{name} filter {b}: state {ex:.1e} cov {eP:.1e}")
    assert ex < TIGHT and eP < TIGHT, (b, ex, eP)
  if not smooth:
    return
  q = cls.quat_idxs()
  n = rh.n.cpu().numpy()
  slabs = [a.cpu().numpy() for a in (rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt)]
  tt = rh.t.cpu().numpy()
  for norm in ([False, True] if q else [False]):
    xs, Ps = (a.cpu().numpy() for a in e.rts_smooth(rh, norm_quats=norm, quaternion_idxs=tuple(q) or (0,)))
    for b in sel:
      k = int(n[b])
      xr, Pr = hiprec.rts(m, *[a[:k, b:b + 1] for a in slabs], tt[:k, b], quat_idxs=q, norm_quats=norm)
      ex, eP = state_err(xs[:k, b], xr[:, 0]), cov_err(Ps[:k, b], Pr[:, 0])
      print(f"{name} rts filter {b} ({k} rows, norm {norm}): state {ex:.1e} cov {eP:.1e}")
      assert ex < TIGHT and eP < TIGHT, (b, norm, ex, eP)


QUATS = [3] + [23 + 3 + 7 * c for c in range(10)]


def _msckf_shipped(oracle_dir):
  import os
  from oracle import build_ref
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.msckf import MsckfKalman
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  return ensure_generated(MsckfKalman)


def _shipped_streams(x, point, o, n_ticks, seed):
  """Shipped msckf: a gyro sample (kind 4) at every tick but frame ticks, a camera frame (kind 17, augment) every 4 ticks
  at a per-filter phase, filter 0 without frames.  Returns ticks as RaggedScheduler.tick arguments."""
  from tests.util import LIVE_R, msckf_feature_obs
  B = x.shape[0]
  rng = np.random.default_rng(seed)
  phase = rng.integers(0, 4, B)
  phase[0] = -1
  zf, Rf, _ = msckf_feature_obs(o, x, point, seed=seed)
  R4 = np.diag(LIVE_R[4])
  ticks = []
  for j in range(n_ticks):
    frame = (phase >= 0) & (j % 4 == phase)
    ids = np.arange(B)
    kinds = np.where(frame, 17, 4)
    t = 0.01 * (j + 1) + 1e-4 * ids
    z = {4: rng.normal(0, 0.01, (int((~frame).sum()), 3))}
    R = {4: np.tile(R4, (int((~frame).sum()), 1, 1))}
    ea = None
    if frame.any():
      z[17] = zf[frame] + rng.normal(0, 1e-4, (int(frame.sum()), 20))
      R[17], ea = Rf[frame], {17: point[frame]}
    ticks.append((ids, t, kinds, z, R, ea, frame))
  return ticks


def test_shipped_msckf_frame_streams_against_the_oracle(oracle_dir):
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.scheduler import RaggedScheduler
  from tests.util import Oracle, msckf_batch
  folder = _msckf_shipped(oracle_dir)
  o = Oracle(oracle_dir, "msckf")
  B, n_ticks = 12, 12
  x, P, Q, point = msckf_batch(B, seed=400)
  ticks = _shipped_streams(x, point, o, n_ticks, seed=401)
  e = BatchedEKF(folder, "msckf", Q, x, P, quaternion_idxs=QUATS)
  s = RaggedScheduler(e)
  for tk in ticks:
    s.tick(*tk)
  xr, Pr = x.copy(), P.copy()
  tl = None
  for ids, t, kinds, z, R, ea, frame in ticks:
    dt = np.zeros(B) if tl is None else t - tl
    tl = t
    for k in (4, 17):
      s_ = np.flatnonzero(kinds == k)
      if s_.size:
        xo, Po, _ = o.batch_step(k, xr[s_], Pr[s_], Q, dt[s_], z[k], R[k], None if k == 4 else ea[17], quat_idxs=QUATS, flags=3)
        xr[s_], Pr[s_] = xo, Po
    f = np.flatnonzero(frame)
    if f.size:
      xr[f], Pr[f] = _shift_np(xr[f], Pr[f])
  ex, eP = state_err(e.state(), xr), cov_err(e.covs(), Pr)
  print(f"msckf frame streams vs oracle: state {ex:.1e} cov {eP:.1e}")
  assert ex < 1e-9 and eP < 1e-9


def _shift_np(x, P):
  from rednose_b200.filters.msckf import DIM_AUGMENT as d3, DIM_AUGMENT_ERR as d4
  x = x.copy()
  x[:, 23:-d3] = x[:, 23 + d3:].copy()
  x[:, -d3:] = x[:, :d3]
  src = np.r_[0:22, 22 + d4:P.shape[1], 0:d4]
  return x, P[:, src][:, :, src]


# ------------------------------------------------------------------------------------------- 4. lockstep, shifts ---
@pytest.mark.parametrize("name", ["msckf_e18", "msckf_e28"])
def test_lockstep_stream_with_shifts_equals_lockstep_recording_bit_for_bit(name):
  from rednose_b200.scheduler import RaggedScheduler
  cls = BY_NAME[name]
  m = _model(cls)
  B = 9
  x, P, Q, _ = batch(cls, B, seed=6)
  fk, plain = cls.feature_kinds()[0], _plain(cls)
  kinds, augs = [fk, plain, fk, plain, fk], [True, False, True, False, True]
  ticks = [(kind,) + observe(cls, m, kind, x, seed=k) for k, kind in enumerate(kinds)]
  T = len(ticks)
  a, b = _engine(cls, x, P, Q, m), _engine(cls, x, P, Q, m)
  h, rh = a.new_history(T), b.new_ragged_history(T)
  sch = RaggedScheduler(b, history=rh)
  ids = np.arange(B)
  for k, ((kind, z, R, ea), aug) in enumerate(zip(ticks, augs)):
    t = 0.02 * k + 0.005 * (k % 2)
    a.step_recorded(h, kind, t, z, R, ea, augment=aug)
    sch.tick(ids, t, np.full(B, kind), {kind: z}, {kind: R}, None if ea is None else {kind: ea}, np.full(B, aug))
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)
  for s1, s2 in ((h.x_pred, rh.x_pred), (h.P_pred, rh.P_pred), (h.x_filt, rh.x_filt), (h.P_filt, rh.P_filt)):
    assert torch.equal(s1, s2)
  q = cls.quat_idxs()
  kw = dict(norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
  xs1, Ps1 = a.rts_smooth(h, **kw)
  xs2, Ps2 = b.rts_smooth(rh, **kw)
  assert torch.equal(xs1, xs2) and torch.equal(Ps1, Ps2)


# ------------------------------------------------------------------------------------ 5. rewinding, late frames ---
def _late_frames(plain_obs, frame_obs, B, n_ticks, seed, ea_of=None):
  """A plain kind at 100 Hz and camera frames at 20 Hz with a per-filter phase (filter 0 without frames); after tick 10
  each frame arrives 50-300 ms late with p = 0.6 (the filter's plain samples go on).  plain_obs(b, j) / frame_obs(b, j)
  -> (kind, z, R, ea).  Returns (arrival ticks, per-filter observation lists (t, kind, z, R, ea, aug))."""
  rng = np.random.default_rng(seed)
  phase = rng.integers(0, 5, B)
  phase[0] = -1
  arrivals = [[] for _ in range(n_ticks + 40)]
  per_filter = [[] for _ in range(B)]
  for b in range(B):
    for j in range(n_ticks):
      t = 0.01 * (j + 1) + 1e-4 * b
      if phase[b] >= 0 and j % 5 == phase[b]:
        o = (t,) + frame_obs(b, j) + (True,)
        at = j + int(rng.integers(5, 31)) if (j > 10 and rng.random() < 0.6) else j
      else:
        o, at = (t,) + plain_obs(b, j) + (False,), j
      per_filter[b].append(o)
      arrivals[at].append((b, o))
  return arrivals, per_filter


def _tick_args(entries, zdims):
  """RaggedScheduler.tick arguments of [(filter, (t, kind, z, R, ea, aug))], at most one entry per filter."""
  ids = np.array([b for b, _ in entries])
  t = np.array([o[0] for _, o in entries])
  kinds = np.array([o[1] for _, o in entries])
  z = {k: np.array([o[2] for _, o in entries if o[1] == k]) for k in zdims if (kinds == k).any()}
  R = {k: np.array([o[3] for _, o in entries if o[1] == k]) for k in zdims if (kinds == k).any()}
  ea = {k: np.array([o[4] for _, o in entries if o[1] == k]) for k in zdims
        if any(o[1] == k and o[4] is not None for _, o in entries)}
  return ids, t, kinds, z, R, ea or None, np.array([o[5] for _, o in entries])


def _rewinding_vs_in_order(e_rw, e_io, arrivals, per_filter, zdims, ea_dims, history_T=None):
  """Drive e_rw by arrival (RewindingScheduler, depth 48, max_rewind_age 1 s) and e_io by time order (RaggedScheduler);
  with history_T both record.  Returns (rewinding scheduler, its history, in-order history)."""
  from rednose_b200.scheduler import RaggedScheduler, RewindingScheduler
  hr = e_rw.new_ragged_history(history_T) if history_T else None
  hi = e_io.new_ragged_history(history_T) if history_T else None
  rw = RewindingScheduler(e_rw, zdims, depth=48, max_rewind_age=1.0, ea_dims=ea_dims, history=hr)
  for entries in arrivals:
    # one observation per filter and tick: a filter with two arrivals gets the later one next tick
    while entries:
      seen, now, later = set(), [], []
      for b, o in entries:
        (later if b in seen else now).append((b, o))
        seen.add(b)
      rw.tick(*_tick_args(now, zdims))
      entries = later
  io = RaggedScheduler(e_io, history=hi)
  srt = [sorted(obs, key=lambda o: o[0]) for obs in per_filter]
  for j in range(max(len(s) for s in srt)):
    io.tick(*_tick_args([(b, s[j]) for b, s in enumerate(srt) if j < len(s)], zdims))
  assert rw.dropped == 0 and io.dropped == 0 and rw.rewinds > 3 and rw.replayed > rw.rewinds
  return rw, hr, hi


@pytest.mark.parametrize("name,history", [("msckf_e18", False), ("msckf_e18", True), ("msckf_e28", True)])
def test_rewinding_late_frames_equal_the_in_order_stream(name, history):
  cls = BY_NAME[name]
  m = _model(cls)
  B, n_ticks = 9, 40
  x, P, Q, _ = batch(cls, B, seed=500)
  plain, feat = _plain(cls), cls.feature_kinds()[0]
  op = observe(cls, m, plain, x, seed=501, n_obs=n_ticks)
  of = observe(cls, m, feat, x, seed=502, n_obs=n_ticks)
  zd = {plain: cls.kinds()[plain][0], feat: cls.kinds()[feat][0]}
  ead = {k: cls.kinds()[k][1] for k in zd if cls.kinds()[k][1]}
  pick = lambda obs, k, b, j: (k, obs[0][b, j], obs[1][b, j], None if obs[2] is None else obs[2][b, j])   # noqa: E731
  arrivals, per_filter = _late_frames(lambda b, j: pick(op, plain, b, j), lambda b, j: pick(of, feat, b, j), B, n_ticks, 503)
  a, b = _engine(cls, x, P, Q, m), _engine(cls, x, P, Q, m)
  rw, hr, hi = _rewinding_vs_in_order(a, b, arrivals, per_filter, zd, ead, history_T=n_ticks if history else None)
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)
  if history:
    assert torch.equal(hr.n, hi.n) and hr.overflowed() == 0
    for s1, s2 in ((hr.x_pred, hi.x_pred), (hr.P_pred, hi.P_pred), (hr.x_filt, hi.x_filt), (hr.P_filt, hi.P_filt), (hr.t, hi.t)):
      for f in range(B):
        k = int(hi.n[f])
        assert torch.equal(s1[:k, f], s2[:k, f]), f
    q = cls.quat_idxs()
    kw = dict(norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
    xs1, Ps1 = a.rts_smooth(hr, **kw)
    xs2, Ps2 = b.rts_smooth(hi, **kw)
    assert torch.equal(xs1.nan_to_num(), xs2.nan_to_num()) and torch.equal(Ps1.nan_to_num(), Ps2.nan_to_num())


def test_rewinding_late_frames_shipped_msckf(oracle_dir):
  from rednose_b200.batched import BatchedEKF
  from tests.util import LIVE_R, Oracle, msckf_batch, msckf_feature_obs
  folder = _msckf_shipped(oracle_dir)
  o = Oracle(oracle_dir, "msckf")
  B, n_ticks = 6, 40
  x, P, Q, point = msckf_batch(B, seed=600)
  zf, Rf, _ = msckf_feature_obs(o, x, point, seed=601)
  rng = np.random.default_rng(602)
  gyro = rng.normal(0, 0.01, (B, n_ticks, 3))
  fn = rng.normal(0, 1e-4, (B, n_ticks, 20))
  R4 = np.diag(LIVE_R[4])
  arrivals, per_filter = _late_frames(lambda b, j: (4, gyro[b, j], R4, None), lambda b, j: (17, zf[b] + fn[b, j], Rf[b], point[b]),
                                      B, n_ticks, 603)
  a = BatchedEKF(folder, "msckf", Q, x, P, quaternion_idxs=QUATS)
  b = BatchedEKF(folder, "msckf", Q, x, P, quaternion_idxs=QUATS)
  _rewinding_vs_in_order(a, b, arrivals, per_filter, {4: 3, 17: 20}, {17: 3})
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)


# ------------------------------------------------------------------------------------ 6. checkpointed smoother ---
@pytest.mark.parametrize("name", ["msckf_e18", "msckf_e28"])
def test_checkpointed_smoother_with_shifts_equals_the_whole_ragged_pass(name):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.scheduler import RaggedScheduler
  from rednose_b200.smoothing import RaggedCheckpointedSmoother
  cls = BY_NAME[name]
  m = _model(cls)
  B, n_ticks = 2 * cls.group() + 1, 24
  x, P, Q, _ = batch(cls, B, seed=700)
  ticks = _frame_streams(cls, m, B, n_ticks, seed=701)
  q = cls.quat_idxs()
  kw = dict(norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
  e = _engine(cls, x, P, Q, m)
  rh = e.new_ragged_history(n_ticks)
  s = RaggedScheduler(e, history=rh)
  for tk in ticks:
    s.tick(*tk)
  xw, Pw = (a.cpu().numpy() for a in e.rts_smooth(rh, **kw))
  n = rh.n.cpu().numpy()

  def tick_fn(j, lo, hi):
    ids, t, kinds, z, R, ea, aug = ticks[j]
    assert (lo, hi) == (0, B)
    return ids, t, kinds, {k: v.copy() for k, v in z.items()}, R, ea, aug

  for segment in (1, 5, 16):
    cs = RaggedCheckpointedSmoother(ensure_generated(cls), cls.name, Q, x.shape[1], P.shape[1], quaternion_idxs=q, segment=segment)
    got_x, got_P = np.full_like(xw, np.nan), np.full_like(Pw, np.nan)
    count = np.zeros(B, dtype=np.int64)

    def sink(lo, hi, k0, n_rows, xs, Ps):
      k0, n_rows, xs, Ps = k0.cpu().numpy(), n_rows.cpu().numpy(), xs.cpu().numpy(), Ps.cpu().numpy()
      for f in range(hi - lo):
        k, r = int(k0[f]), int(n_rows[f])
        got_x[k:k + r, lo + f], got_P[k:k + r, lo + f] = xs[:r, f], Ps[:r, f]
        count[lo + f] += r

    cs.run(x, P, n_ticks, tick_fn, sink, norm_quats=bool(q))
    assert count.tolist() == n.tolist(), segment
    for f in range(B):
      r = int(n[f])
      assert np.array_equal(got_x[:r, f], xw[:r, f]) and np.array_equal(got_P[:r, f], Pw[:r, f]), (segment, f)
