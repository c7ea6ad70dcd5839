"""Packed covariance histories (BatchedEKF.new_history(T, packed=True), REDNOSE_PACKED_HIST) on the device, at live_kf
and at every pair-kernel shape of tests/shapes.py.

The pair kernel writes P_{k|k} packed exactly as it writes the resident packed P, and P_{k|k-1} as the lower triangle of
the full slab it writes otherwise, so recording is checked bit for bit against a full history.  The smoothers read the
packed slabs by the lower triangle only; against the 40-digit reference they hold the tolerance test_shapes_gpu.py
asserts.  Against smoothing of the full history they differ by rounding: the full P_{k|k-1} slab's upper triangle is its
lower triangle's mirror only up to rounding, and the full smoothers read both.

Worst values measured on one H100 80GB HBM3 (power limit 700 W): against the 40-digit reference state 2.6e-12 (live;
8.1e-16 at the synthetic shapes; 5.9e-12 on the ragged live streams), covariance 7.4e-14; packed against full smoothing
state 0, covariance 6.2e-15 (bound PACKED_VS_FULL = 1e-12).
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.shapes import BY_NAME, batch as shape_batch, observe as shape_observe, sample
from tests.util import LIVE_R, cov_err, live_batch, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9            # the smoother tolerance of tests/test_shapes_gpu.py against the 40-digit reference
PACKED_VS_FULL = 1e-12  # packed against full smoothing, same units (state_err / cov_err)
CASES = ["live", "shape_e8", "shape_e16", "shape_e24", "shape_e28", "shape_e32"]


def _live_ticks(x, T):
  B = x.shape[0]
  ticks = []
  for k in range(T):
    kind = (4, 10, 12)[k % 3]
    R = np.tile(np.diag(LIVE_R[kind]), (B, 1, 1))
    z = np.random.default_rng(k).normal(0, 0.05, (B, 3)) + (x[:, :3] if kind == 12 else [0, 0, -9.8] if kind == 10 else 0)
    ticks.append((kind, z, R, None))
  return ticks


def _case(name, T=6):
  """(folder, name, x, P, Q, quats, global values, hiprec model, sampled filters, [(kind, z, R, ea)] per step)."""
  from rednose_b200.filters import ensure_generated
  if name == "live":
    from rednose_b200.filters.live import LiveKalman
    x, P, Q = live_batch(45, seed=21)
    return ensure_generated(LiveKalman), "live", x, P, Q, [3], {}, hiprec.model_of(LiveKalman), [0, 15, 16, 31, 32, 44], _live_ticks(x, T)
  cls = BY_NAME[name]
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  B = 2 * cls.group() + 1
  x, P, Q, _ = shape_batch(cls, B, seed=22)
  kinds = sorted(k for k, (_, _, gated) in cls.kinds().items() if not gated)
  ticks = [(kinds[k % len(kinds)],) + shape_observe(cls, m, kinds[k % len(kinds)], x, seed=30 + k) for k in range(T)]
  gv = {g: m.gv[i] for i, g in enumerate(cls.global_names())}
  return ensure_generated(cls), cls.name, x, P, Q, cls.quat_idxs(), gv, m, sample(cls, B), ticks


def _engine(folder, name, x, P, Q, q, gv):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q, global_vars=gv)


def _tril(P):
  return torch.tril(P)


def _record(e, hist, ticks, after=None):
  for k, (kind, z, R, ea) in enumerate(ticks):
    e.step_recorded(hist, kind, 0.02 * k + 0.005 * (k % 2), z.copy(), R, ea)
    if after:
      after(k)


@pytest.mark.parametrize("case", CASES)
def test_packed_history_recording_and_smoothing(case):
  """(a) lockstep recording, packed against full; (b) packed P_{k|k} == the resident packed P after every step; (c) the
  packed smoother against the 40-digit reference; (d) packed against full smoothing; (h) a second identical packed run
  is bit-identical."""
  folder, name, x, P, Q, q, gv, m, sel, ticks = _case(case)
  T = len(ticks)
  full, pk, pk2 = (_engine(folder, name, x, P, Q, q, gv) for _ in range(3))
  h = full.new_history(T)
  hp = pk.new_history(T, packed=True)
  PD = pk._packed_doubles
  assert hp.packed and hp.P_pred.shape == hp.P_filt.shape == (T, x.shape[0], PD)

  def resident(k):   # (b)
    assert not pk._full_owns and torch.equal(hp.P_filt[k], pk._Pk), k
  _record(full, h, ticks)
  _record(pk, hp, ticks, resident)
  # (a)
  assert torch.equal(h.x_pred, hp.x_pred) and torch.equal(h.x_filt, hp.x_filt)
  assert torch.equal(pk.unpack_P(hp.P_filt), h.P_filt)
  assert torch.equal(_tril(pk.unpack_P(hp.P_pred)), _tril(h.P_pred))
  assert torch.equal(full.P, pk.P)
  kw = dict(norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
  xs, Ps = pk.rts_smooth(hp, **kw)
  assert Ps.shape == hp.P_filt.shape
  Psf = pk.unpack_P(Ps)
  # (c)
  slabs = [hp.x_pred.cpu().numpy(), hp.x_filt.cpu().numpy(), pk.unpack_P(hp.P_pred).cpu().numpy(), pk.unpack_P(hp.P_filt).cpu().numpy()]
  xr, Pr = hiprec.rts(m, *slabs, hp.t_host, quat_idxs=q, norm_quats=bool(q), sel=sel)
  ex, eP = state_err(xs.cpu().numpy()[:, sel], xr), cov_err(Psf.cpu().numpy()[:, sel], Pr)
  # (d)
  xs_f, Ps_f = full.rts_smooth(h, **kw)
  dx, dP = state_err(xs.cpu().numpy(), xs_f.cpu().numpy()), cov_err(Psf.cpu().numpy(), Ps_f.cpu().numpy())
  print(f"{name} packed rts: vs 40 digits state {ex:.1e} cov {eP:.1e}; vs full smoothing state {dx:.1e} cov {dP:.1e}")
  assert ex < TIGHT and eP < TIGHT, (ex, eP)
  assert dx < PACKED_VS_FULL and dP < PACKED_VS_FULL, (dx, dP)
  assert torch.equal(Psf, Psf.transpose(-1, -2))      # what the smoother wrote is a lower triangle, unpacked symmetric
  # (h)
  hp2 = pk2.new_history(T, packed=True)
  _record(pk2, hp2, ticks)
  xs2, Ps2 = pk2.rts_smooth(hp2, **kw)
  assert torch.equal(hp.P_pred, hp2.P_pred) and torch.equal(hp.P_filt, hp2.P_filt)
  assert torch.equal(xs, xs2) and torch.equal(Ps, Ps2)


def test_packed_rows_of_predict_update_and_step():
  """predict(hist=), update(hist=) and step(hist_pred=, hist_filt=) take the layout from the slab shape; an in-place
  smoothing (Ps aliasing P_filt), out= and terminal= keep the packed layout."""
  folder, name, x, P, Q, q, gv, m, sel, ticks = _case("live", T=3)
  a, b = _engine(folder, name, x, P, Q, q, gv), _engine(folder, name, x, P, Q, q, gv)
  B, E, PD = x.shape[0], 22, b._packed_doubles
  hxa, hxb = (torch.empty(B, 23, dtype=torch.float64, device="cuda") for _ in range(2))
  fa = torch.empty(B, E, E, dtype=torch.float64, device="cuda")
  fb = torch.empty(B, PD, dtype=torch.float64, device="cuda")
  a.predict(0.01, hist=(hxa, fa)); b.predict(0.01, hist=(hxb, fb))
  assert torch.equal(hxa, hxb) and torch.equal(_tril(b.unpack_P(fb)), _tril(fa))
  kind, z, R, _ = ticks[2]
  a.update(kind, z.copy(), R, hist=(hxa, fa)); b.update(kind, z.copy(), R, hist=(hxb, fb))
  assert torch.equal(hxa, hxb) and torch.equal(b.unpack_P(fb), fa) and torch.equal(fb, b._Pk)
  with pytest.raises(AssertionError):
    b.predict(0.01, hist=(hxb, fb[:, :PD - 4]))
  h, hp = a.new_history(3), b.new_history(3, packed=True)
  _record(a, h, ticks); _record(b, hp, ticks)
  xs, Ps = b.rts_smooth(hp, norm_quats=True)
  out = (torch.empty_like(hp.x_filt), torch.empty_like(hp.P_filt))
  b.rts_smooth(hp, norm_quats=True, out=out)
  assert torch.equal(out[1], Ps)
  with pytest.raises(AssertionError):
    b.rts_smooth(hp, out=(torch.empty_like(h.x_filt), torch.empty_like(h.P_filt)))
  # segment continuation: the last two rows smoothed from a packed terminal estimate == rows of the whole smoothing
  seg = b.new_history(2, packed=True)
  for s1, s2 in ((seg.x_pred, hp.x_pred), (seg.x_filt, hp.x_filt), (seg.P_pred, hp.P_pred), (seg.P_filt, hp.P_filt)):
    s1.copy_(s2[1:3])
  seg.t_host[:] = hp.t_host[1:3]
  seg.n = 2
  xo, Po = torch.empty_like(seg.x_filt), torch.empty_like(seg.P_filt)
  b.rts_smooth(seg, norm_quats=True, out=(xo, Po), terminal=(xs[2].contiguous(), Ps[2].contiguous()), k0=1)
  assert torch.equal(xo[0], xs[1]) and torch.equal(Po[0], Ps[1])
  with pytest.raises(AssertionError):
    b.rts_smooth(seg, out=(xo, Po), terminal=(xs[2].contiguous(), b.unpack_P(Ps[2])), k0=1)
  xi, Pi = b.rts_smooth(hp, norm_quats=True, in_place=True)
  assert Pi.data_ptr() == hp.P_filt.data_ptr() and torch.equal(xi, xs) and torch.equal(Pi, Ps)


@pytest.mark.parametrize("norm_quats", [False, True])
def test_checkpointed_packed_equals_whole_history_packed(norm_quats):
  """(e) CheckpointedSmoother(packed_history=True) == TiledSmoother(packed_history=True) over the whole history, bit for
  bit; both sinks receive packed covariances."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother
  folder = ensure_generated(LiveKalman)
  B, T = 29, 37
  x, P, Q = live_batch(B, seed=310)
  ticks = _live_ticks(x, T)

  def obs_fn(k, lo, hi):
    kind, z, R, _ = ticks[k]
    return 0.01 * (k + 1), kind, z[lo:hi].copy(), R[lo:hi]

  ref = {}
  ts = TiledSmoother(folder, "live", Q, 23, 22, quaternion_idxs=[3], tile=64, packed_history=True)
  ts.run(x, P, T, obs_fn, lambda lo, hi, xs, Ps: ref.update(a=(xs.cpu().numpy().copy(), Ps.cpu().numpy().copy())), norm_quats=norm_quats)
  PD = ref["a"][1].shape[-1]
  assert PD == 264
  for segment, tile in ((8, 16), (5, 64)):
    xs_all, Ps_all = np.full((T, B, 23), np.nan), np.full((T, B, PD), np.nan)

    def sink(lo, hi, k0, xs, Ps):
      n = xs.shape[0]
      assert np.isnan(xs_all[k0:k0 + n, lo:hi]).all()
      xs_all[k0:k0 + n, lo:hi], Ps_all[k0:k0 + n, lo:hi] = xs.cpu().numpy(), Ps.cpu().numpy()
    cs = CheckpointedSmoother(folder, "live", Q, 23, 22, quaternion_idxs=[3], segment=segment, tile=tile, packed_history=True)
    cs.run(x, P, T, obs_fn, sink, norm_quats=norm_quats)
    assert np.array_equal(xs_all, ref["a"][0]) and np.array_equal(Ps_all, ref["a"][1]), (segment, tile)
  full = cs.unpack_P(torch.as_tensor(Ps_all[:2, :3]).cuda())
  assert full.shape == (2, 3, 22, 22) and torch.equal(full, full.transpose(-1, -2))


def test_ragged_packed_history_through_the_scheduler():
  """(f) live IMU + GNSS kinds through RaggedScheduler with a packed RaggedHistory: lockstep streams are bit-identical
  to step_recorded with a packed History; ragged streams against the 40-digit reference."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RaggedScheduler
  folder = ensure_generated(LiveKalman)
  B, T = 45, 6
  x, P, Q = live_batch(B, seed=40)
  ticks = _live_ticks(x, T)
  a, b = _engine(folder, "live", x, P, Q, [3], {}), _engine(folder, "live", x, P, Q, [3], {})
  h, rh = a.new_history(T, packed=True), b.new_ragged_history(T, packed=True)
  sch = RaggedScheduler(b, history=rh)
  ids = np.arange(B)
  for k, (kind, z, R, _) in enumerate(ticks):
    t = 0.02 * k + 0.005 * (k % 2)
    a.step_recorded(h, kind, t, z.copy(), R)
    sch.tick(ids, t, np.full(B, kind), {kind: z.copy()}, {kind: R})
  for s1, s2 in ((h.x_pred, rh.x_pred), (h.P_pred, rh.P_pred), (h.x_filt, rh.x_filt), (h.P_filt, rh.P_filt)):
    assert torch.equal(s1, s2)
  xs1, Ps1 = a.rts_smooth(h, norm_quats=True)
  xs2, Ps2 = b.rts_smooth(rh, norm_quats=True)
  assert torch.equal(xs1, xs2) and torch.equal(Ps1, Ps2)
  # ragged: each filter observes on its own subset of ticks
  m = hiprec.model_of(LiveKalman)
  c = _engine(folder, "live", x, P, Q, [3], {})
  rc = c.new_ragged_history(T, packed=True)
  sch = RaggedScheduler(c, history=rc)
  rng = np.random.default_rng(41)
  mask = rng.random((B, T)) < 0.6
  mask[0] = True
  mask[1] = False; mask[1, 3] = True
  t_b = np.cumsum(rng.uniform(0.005, 0.03, (B, T)), axis=1)
  for k, (kind, z, R, _) in enumerate(ticks):
    act = np.flatnonzero(mask[:, k])
    if act.size:
      sch.tick(act, t_b[act, k], np.full(act.size, kind), {kind: z[act].copy()}, {kind: R[act]})
  n = rc.n.cpu().numpy()
  assert n.tolist() == mask.sum(1).tolist()
  xs, Ps = c.rts_smooth(rc, norm_quats=True)
  Psf = c.unpack_P(Ps)
  slabs = [rc.x_pred.cpu().numpy(), rc.x_filt.cpu().numpy(), c.unpack_P(rc.P_pred).cpu().numpy(), c.unpack_P(rc.P_filt).cpu().numpy()]
  tt = rc.t.cpu().numpy()
  for f in (0, 1, 16, B - 1):
    k = int(n[f])
    if k == 0:
      continue
    xr, Pr = hiprec.rts(m, *[s[:k, f:f + 1] for s in slabs], tt[:k, f], quat_idxs=[3], norm_quats=True)
    ex, eP = state_err(xs[:k, f].cpu().numpy(), xr[:, 0]), cov_err(Psf[:k, f].cpu().numpy(), Pr[:, 0])
    print(f"live ragged packed rts filter {f} ({k} rows): state {ex:.1e} cov {eP:.1e}")
    assert ex < TIGHT and eP < TIGHT, (f, ex, eP)


def test_packed_history_refused():
  """(g) ValueError from new_history / new_ragged_history where the filter has no packed layout: kinematic (thread
  kernel), shape_e7 (odd EDIM) and an MSCKF with a feature kind (CTA kernel)."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.kinematic import KinematicKalman
  from tests.msckf_shapes import BY_NAME as MSCKF_BY_NAME, batch as msckf_batch
  from tests.util import kinematic_batch
  xk, Pk, Qk, _, _ = kinematic_batch(4, seed=1)
  cls7 = BY_NAME["shape_e7"]
  x7, P7, Q7, _ = shape_batch(cls7, 4, seed=1)
  mcls = MSCKF_BY_NAME["msckf_e18"]
  xm, Pm, Qm, _ = msckf_batch(mcls, 4, seed=1)
  cases = [(ensure_generated(KinematicKalman), "kinematic", xk, Pk, Qk, []),
           (ensure_generated(cls7), cls7.name, x7, P7, Q7, cls7.quat_idxs()),
           (ensure_generated(mcls), mcls.name, xm, Pm, Qm, mcls.quat_idxs())]
  for folder, name, x, P, Q, q in cases:
    e = _engine(folder, name, x, P, Q, q, {})
    assert e._packed_doubles == 0
    with pytest.raises(ValueError, match="two-filters-per-warp"):
      e.new_history(3, packed=True)
    with pytest.raises(ValueError, match="two-filters-per-warp"):
      e.new_ragged_history(3, packed=True)
