"""Ragged streams longer than one history: RaggedCheckpointedSmoother (checkpoints per segment of ticks, segments
re-filtered through RaggedScheduler(history=...) and smoothed last to first with <name>_batch_rts_ragged_segment) must
give every filter's smoothed rows bit for bit as one whole RaggedHistory + rts_smooth does.

1. Live config-3 streams (gyro, accelerometer, GNSS on per-filter clocks, samples missing) over many segments, full and
   packed, segments of 1, 5 and 16 ticks, quaternions normalised: a filter with no rows at all, one whose first row is
   in the last segments, one with no rows over several whole segments.
2. Every tests/shapes.py shape and the MSCKF shapes with a ragged smoother, feature kinds with extra arguments included.
3. One ragged segment through the entry point alone against the 40-digit reference of tests/hiprec.py.
4. Several tiles give the rows of one tile.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME as MSCKF_BY_NAME, batch as msckf_batch, observe as msckf_observe
from tests.shapes import SHAPES, batch as shape_batch, observe as shape_observe
from tests.util import LIVE_R, cov_err, live_batch, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9


class _Stream:
  """Ticks of B filters: entries (filter, time, kind) per tick and one observation per (kind, tick, filter), so that
  tick_fn returns the same tick every time it is asked."""

  def __init__(self, mask, kind_of, times, obs):
    self.mask, self.kind_of, self.times, self.obs = mask, kind_of, times, obs   # obs[kind] = (z [T, B, Z], R [B, Z, Z], ea)

  def tick(self, j, lo, hi):
    f = np.flatnonzero(self.mask[lo:hi, j]) + lo
    kinds = self.kind_of[f, j]
    z, R, ea = {}, {}, {}
    for k in sorted(set(kinds.tolist())):
      s = f[kinds == k]
      zk, Rk, eak = self.obs[k]
      z[k], R[k] = zk[j, s].copy(), Rk[s]
      if eak is not None:
        ea[k] = eak[j, s]
    return (f - lo, self.times[f, j], kinds, z, R) + ((ea,) if ea else ())


def _mask(B, n_ticks, rng, p):
  mask = rng.random((B, n_ticks)) < p
  mask[0] = False                                  # a filter without any row
  mask[1, :int(0.85 * n_ticks)] = False            # first row in the last segments
  mask[2, n_ticks // 4:n_ticks // 2] = False       # no rows over several whole segments
  mask[3] = True
  return mask


def _live_stream(B, n_ticks, seed):
  """Config-3 streams: 100 Hz gyro (4) and accelerometer (10) alternating, a GNSS fix (12) every 20 ticks at a
  per-filter phase, ~3 % of the samples missing, every filter on its own clock."""
  rng = np.random.default_rng(seed)
  x, P, Q = live_batch(B, seed=seed)
  mask = _mask(B, n_ticks, rng, 0.97)
  gph = rng.integers(0, 20, B)
  kind_of = np.where((np.arange(n_ticks)[None, :] - gph[:, None]) % 20 == 0, 12, np.where(np.arange(n_ticks) % 2 == 0, 4, 10)[None, :])
  times = 0.01 * np.arange(n_ticks)[None, :] + rng.uniform(0, 0.01, (B, 1))
  obs = {4: rng.normal(0, 0.01, (n_ticks, B, 3)), 10: rng.normal(0, 0.1, (n_ticks, B, 3)) + [0, 0, -9.8],
         12: x[None, :, :3] + rng.normal(0, 1.0, (n_ticks, B, 3))}
  obs = {k: (z, np.tile(np.diag(LIVE_R[k]), (B, 1, 1)), None) for k, z in obs.items()}
  return x, P, Q, _Stream(mask, kind_of, times, obs)


def _shape_case(cls, n_ticks, seed):
  """(folder, x, P, Q, quats, globals, stream, model) of a tests/shapes.py or MSCKF shape: 2G + 1 filters (at least 9)."""
  from rednose_b200.filters import ensure_generated
  msckf = cls in MSCKF_BY_NAME.values()
  batch, observe = (msckf_batch, msckf_observe) if msckf else (shape_batch, shape_observe)
  B = max(2 * cls.group() + 1, 9)
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  x, P, Q, _ = batch(cls, B, seed=seed)
  kinds = [k for k, v in cls.kinds().items() if not v[2] or (msckf and v[3])]
  rng = np.random.default_rng(seed + 1)
  mask = _mask(B, n_ticks, rng, 0.6)
  kind_of = rng.choice(kinds, (B, n_ticks))
  times = np.cumsum(rng.uniform(0.005, 0.04, (B, n_ticks)), axis=1)
  obs = {}
  for k in kinds:
    z, R, ea = observe(cls, m, k, x, seed=seed + 2 + k, n_obs=n_ticks)      # [B, n_ticks, ...]: one per tick
    obs[k] = (np.ascontiguousarray(z.swapaxes(0, 1)), R[:, 0], None if ea is None else np.ascontiguousarray(ea.swapaxes(0, 1)))
  gv = {g: m.gv[i] for i, g in enumerate(cls.global_names())}
  return ensure_generated(cls), x, P, Q, cls.quat_idxs(), gv, _Stream(mask, kind_of, times, obs), m


def _whole(folder, name, x, P, Q, q, gv, stream, n_ticks, norm, packed):
  """One RaggedHistory of n_ticks rows (a filter records at most one row per tick) + rts_smooth: (xs, Ps, n, history)."""
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.scheduler import RaggedScheduler
  e = BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q, global_vars=gv)
  rh = e.new_ragged_history(n_ticks, packed=packed)
  s = RaggedScheduler(e, history=rh)
  for j in range(n_ticks):
    s.tick(*stream.tick(j, 0, x.shape[0]))
  xs, Ps = e.rts_smooth(rh, norm_quats=norm, quaternion_idxs=tuple(q) or (0,))
  return xs.cpu().numpy(), Ps.cpu().numpy(), rh.n.cpu().numpy(), rh, e


def _checkpointed(folder, name, x, P, Q, q, stream, n_ticks, norm, packed, segment, tile=None):
  """RaggedCheckpointedSmoother's rows reassembled per filter: (xs [n_ticks, B, ...], Ps, rows per filter, smoother)."""
  from rednose_b200.smoothing import RaggedCheckpointedSmoother
  B = x.shape[0]
  cs = RaggedCheckpointedSmoother(folder, name, Q, x.shape[1], P.shape[1], quaternion_idxs=q, segment=segment, tile=tile,
                                  packed_history=packed)
  got_x = got_P = None
  count = np.zeros(B, dtype=np.int64)

  def sink(lo, hi, k0, n_rows, xs, Ps):
    nonlocal got_x, got_P
    if got_x is None:
      got_x = np.full((n_ticks, B) + tuple(xs.shape[2:]), np.nan)
      got_P = np.full((n_ticks, B) + tuple(Ps.shape[2:]), np.nan)
    k0, n_rows, xs, Ps = k0.cpu().numpy(), n_rows.cpu().numpy(), xs.cpu().numpy(), Ps.cpu().numpy()
    for b in range(hi - lo):
      k, r = int(k0[b]), int(n_rows[b])
      assert np.isnan(got_x[k:k + r, lo + b]).all()          # every row delivered once
      got_x[k:k + r, lo + b], got_P[k:k + r, lo + b] = xs[:r, b], Ps[:r, b]
      count[lo + b] += r

  cs.run(x, P, n_ticks, stream.tick, sink, norm_quats=norm)
  return got_x, got_P, count, cs


def _assert_rows_equal(got_x, got_P, count, xw, Pw, n, what):
  assert count.tolist() == n.tolist(), what
  for b in range(len(n)):
    r = int(n[b])
    same = np.array_equal(got_x[:r, b], xw[:r, b]) and np.array_equal(got_P[:r, b], Pw[:r, b])
    assert same, f"{what}: filter {b} ({r} rows) differs from the whole history"
    assert np.isnan(got_x[r:, b]).all()


# ----------------------------------------------------------------------------------------------- 1. live, config 3 ---
@pytest.mark.parametrize("packed", [False, True])
def test_live_streams_over_many_segments_equal_the_whole_history(packed):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  B, n_ticks = 33, 48
  x, P, Q, stream = _live_stream(B, n_ticks, seed=501)
  folder = ensure_generated(LiveKalman)
  xw, Pw, n, _, _ = _whole(folder, "live", x, P, Q, [3], None, stream, n_ticks, True, packed)
  assert n[0] == 0 and 0 < n[1] <= 0.15 * n_ticks + 1 and n[3] == n_ticks and len(set(n.tolist())) > 3
  for segment in (1, 5, 16):
    got_x, got_P, count, cs = _checkpointed(folder, "live", x, P, Q, [3], stream, n_ticks, True, packed, segment)
    assert cs.stats["segments"] == (n_ticks + segment - 1) // segment and cs.stats["segment_rows"] <= segment
    _assert_rows_equal(got_x, got_P, count, xw, Pw, n, f"live packed={packed} segment={segment}")


# --------------------------------------------------------------------------------------------------- 2. every shape ---
CASES = SHAPES + [MSCKF_BY_NAME[n] for n in ("msckf_e18", "msckf_e27", "msckf_e28")]


@pytest.mark.parametrize("cls", CASES, ids=[c.name for c in CASES])
def test_every_shape_equals_the_whole_ragged_pass(cls):
  n_ticks = 11
  folder, x, P, Q, q, gv, stream, _ = _shape_case(cls, n_ticks, seed=520)
  norm = bool(q)
  xw, Pw, n, _, _ = _whole(folder, cls.name, x, P, Q, q, gv, stream, n_ticks, norm, False)
  for segment in (1, 3):
    got_x, got_P, count, _ = _checkpointed(folder, cls.name, x, P, Q, q, stream, n_ticks, norm, False, segment)
    _assert_rows_equal(got_x, got_P, count, xw, Pw, n, f"{cls.name} segment={segment}")


# ------------------------------------------------------------------------------------------ 3. the entry point alone ---
def test_one_ragged_segment_against_the_40_digit_reference():
  """Filter b's rows k0[b] .. k0[b] + L[b] - 1 of a recorded ragged history, plus the next row where it has one (term),
  smoothed from that row's smoothed estimate: the rows equal the whole pass bit for bit and the 40-digit reference at
  TIGHT; the carried row and the rows past it are not written."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  B, n_ticks, L = 33, 10, 4
  x, P, Q, stream = _live_stream(B, n_ticks, seed=540)
  xw, Pw, n, rh, e = _whole(ensure_generated(LiveKalman), "live", x, P, Q, [3], None, stream, n_ticks, True, False)
  k0 = np.minimum(n, np.arange(B) % 7)
  rows = np.minimum(n - k0, L)
  term = (k0 + rows < n).astype(np.uint8)
  seg = e.new_ragged_history(L + 1)
  for a in ("x_pred", "x_filt", "P_pred", "P_filt", "t"):
    src, dst = getattr(rh, a), getattr(seg, a)
    for b in range(B):
      m = int(rows[b] + term[b])
      dst[:m, b] = src[k0[b]:k0[b] + m, b]
  seg.n.copy_(torch.as_tensor(rows + term, dtype=torch.int32))
  xt = torch.zeros(B, x.shape[1], dtype=torch.float64, device="cuda")
  Pt = torch.zeros(B, 22, 22, dtype=torch.float64, device="cuda")
  for b in np.flatnonzero(term):
    xt[b] = torch.as_tensor(xw[k0[b] + rows[b], b]); Pt[b] = torch.as_tensor(Pw[k0[b] + rows[b], b])
  xs, Ps = e.rts_smooth_ragged_segment(seg, torch.as_tensor(term).cuda(), torch.as_tensor(k0).cuda(), (xt, Pt),
                                       norm_quats=True, quaternion_idxs=(3,))
  xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
  assert term.any() and (~term.astype(bool) & (rows > 0)).any() and (k0 == 0).any() and (k0 > 0).any()
  for b in range(B):
    r = int(rows[b])
    assert np.array_equal(xs[:r, b], xw[k0[b]:k0[b] + r, b]) and np.array_equal(Ps[:r, b], Pw[k0[b]:k0[b] + r, b]), b
    assert np.isnan(xs[r:, b]).all() and np.isnan(Ps[r:, b]).all(), b
  slabs = [s.cpu().numpy() for s in (rh.x_pred, rh.x_filt, rh.P_pred, rh.P_filt)]
  tt = rh.t.cpu().numpy()
  m = hiprec.live_model()
  for b in sorted({int(np.flatnonzero(term)[0]), int(np.flatnonzero(~term.astype(bool) & (rows > 0))[0]), 3}):
    k = int(n[b])
    xr, Pr = hiprec.rts(m, *[s[:k, b:b + 1] for s in slabs], tt[:k, b], quat_idxs=[3], norm_quats=True)
    sl = slice(int(k0[b]), int(k0[b] + rows[b]))
    ex, eP = state_err(xs[:rows[b], b], xr[sl, 0]), cov_err(Ps[:rows[b], b], Pr[sl, 0])
    print(f"live ragged segment filter {b} (rows {sl.start} .. {sl.stop - 1} of {k}, term {term[b]}): state {ex:.1e} cov {eP:.1e}")
    assert ex < TIGHT and eP < TIGHT, (b, ex, eP)


# ----------------------------------------------------------------------------------------------------------- 4. tiles ---
def test_several_tiles_give_the_rows_of_one_tile():
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  B, n_ticks = 33, 24
  x, P, Q, stream = _live_stream(B, n_ticks, seed=560)
  folder = ensure_generated(LiveKalman)
  one = _checkpointed(folder, "live", x, P, Q, [3], stream, n_ticks, True, True, 4)
  many = _checkpointed(folder, "live", x, P, Q, [3], stream, n_ticks, True, True, 4, tile=10)
  assert one[3].plan(B, n_ticks) == (B, 1) and many[3].plan(B, n_ticks) == (9, 4) and many[3].stats["tiles"] == 4
  assert one[2].tolist() == many[2].tolist()
  assert np.array_equal(one[0], many[0], equal_nan=True) and np.array_equal(one[1], many[1], equal_nan=True)
