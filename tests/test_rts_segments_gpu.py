"""Segment-continued smoothing (<name>_batch_rts_segment: terminal x / P and k0, and CheckpointedSmoother) at every shape a
smoother serves: it must give the whole-history result bit for bit.

1. Kernel level, at all ten tests/shapes.py shapes, live, kinematic and the MSCKF shapes with a smoother (main block only):
   one recorded history of T = 7 steps is smoothed whole, then again as chained segments of S = 1, 2, 3, 4, T and T + 2
   steps, last segment first, each handing its smoothed first row to the segment in front.  T - 1 is a multiple of 1, 2
   and 3, so those chains end in a segment of a single row.  Rows a segment does not deliver stay unwritten, and on a
   sample of filters the result matches the 40-digit reference of tests/hiprec.py at TIGHT = 1e-9.
2. End to end, at one shape per step kernel (thread, single-warp, pair) and live: CheckpointedSmoother against
   TiledSmoother over T = 37 steps, segments 4 and 12 (a one-row last segment) and 5, ragged last tiles.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests import msckf_shapes, shapes
from tests.util import LIVE_R, cov_err, kinematic_batch, live_batch, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
T = 7
CASES = [c.name for c in shapes.SHAPES] + ["live", "kinematic", "msckf_e18", "msckf_e27", "msckf_e28"]
GV = [1.0, 1.25]


def _engine(folder, name, x, P, Q, q, gv=None):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q, global_vars=gv)


def _kinematic_model():
  """hiprec model of the kinematic filter (its generator builds the sympy inline; the same expressions here)."""
  import sympy as sp
  state = sp.MatrixSymbol('state', 2, 1)
  dt = sp.Symbol('dt')
  return hiprec.HiPrecModel(sp.Matrix([state[0, 0] + dt * state[1, 0], state[1, 0]]), dt, state,
                            [[sp.Matrix([state[0, 0]]), 1, None]], 2, 2)


def _live_obs(kind, x, rng):
  """Gyro (4), accelerometer (10) or position (12) observations near what the live model predicts, with its R."""
  z = rng.normal(0, 0.05, (x.shape[0], 3)) + (x[:, :3] if kind == 12 else [0, 0, -9.8] if kind == 10 else 0)
  return z, np.tile(np.diag(LIVE_R[kind]), (x.shape[0], 1, 1))


def _inputs(name):
  """(folder, engine name, model, x, P, Q, quats, globals, group, obs(k, x) -> (kind, z, R, ea)) of one case."""
  from rednose_b200.filters import ensure_generated
  if name == "live":
    from rednose_b200.filters.live import LiveKalman
    x, P, Q = live_batch(2 * 16 + 1, seed=301)
    rng = np.random.default_rng(302)
    kinds = [4, 10, 12]
    return (ensure_generated(LiveKalman), name, hiprec.live_model(), x, P, Q, [3], None, 16,
            lambda k, xb: (kinds[k % 3],) + _live_obs(kinds[k % 3], xb, rng) + (None,))
  if name == "kinematic":
    from rednose_b200.filters.kinematic import KinematicKalman
    x, P, Q, z, R = kinematic_batch(2 * 128 + 1, seed=303)
    return (ensure_generated(KinematicKalman), name, _kinematic_model(), x, P, Q, [], None, 128,
            lambda k, xb: (1, z + 0.02 * k, R, None))
  mod = msckf_shapes if name.startswith("msckf") else shapes
  cls = mod.BY_NAME[name]
  m = hiprec.model_of(cls)
  m.gv = GV[:len(m.gvars)]
  x, P, Q, _ = mod.batch(cls, 2 * cls.group() + 1, seed=304)
  kinds = sorted(cls.kinds())
  gv = {g: GV[i] for i, g in enumerate(cls.global_names())}
  return (ensure_generated(cls), name, m, x, P, Q, cls.quat_idxs(), gv, cls.group(),
          lambda k, xb: (kinds[k % len(kinds)],) + mod.observe(cls, m, kinds[k % len(kinds)], xb, seed=310 + k))


SLABS = ("x_pred", "x_filt", "P_pred", "P_filt")


def _chained(e, h, S, kw):
  """Smooth h as segments of S steps, last first: rows k0 .. k0 + S of h go into a history of S + 1 rows, smoothed with
  k0 and the smoothed row k0 + S from the segment behind (none for the last segment)."""
  nan = float("nan")
  xs = torch.full_like(h.x_filt[:h.n], nan)
  Ps = torch.full_like(h.P_filt[:h.n], nan)
  seg = e.new_history(S + 1)
  term = None
  for k0 in reversed(range(0, h.n, S)):
    n = min(S + 1, h.n - k0)
    for a in SLABS:
      getattr(seg, a)[:n].copy_(getattr(h, a)[k0:k0 + n])
    seg.t_host[:n] = h.t_host[k0:k0 + n]
    seg.n = n
    out = (torch.full_like(seg.x_filt, nan), torch.full_like(seg.P_filt, nan))
    e.rts_smooth(seg, out=out, terminal=term, k0=k0, **kw)
    m = n - (term is not None)         # with a terminal, the last row only gives its predicted state
    assert not torch.isnan(out[0][:m]).any() and not torch.isnan(out[1][:m]).any(), (S, k0)
    assert torch.isnan(out[0][m:]).all() and torch.isnan(out[1][m:]).all(), (S, k0)   # not delivered: not written
    xs[k0:k0 + m], Ps[k0:k0 + m] = out[0][:m], out[1][:m]
    term = (out[0][0].clone(), out[1][0].clone())
  return xs, Ps


def _rows_that_differ(a, b):
  """{row: max |a - b|} over the rows where a and b are not identical."""
  d = (a - b).abs().flatten(1).amax(1).cpu().numpy()
  same = torch.eq(a, b).flatten(1).all(1).cpu().numpy()
  return {k: float(d[k]) for k in range(len(d)) if not same[k]}


@pytest.mark.parametrize("case", CASES)
def test_chained_segments_equal_the_whole_history(case):
  folder, name, m, x, P, Q, q, gv, G, obs = _inputs(case)
  B = x.shape[0]
  sel = [0, G, B - 1]
  e = _engine(folder, name, x, P, Q, q, gv)
  h = e.new_history(T)
  t = np.cumsum(np.random.default_rng(305).uniform(0.005, 0.04, T))
  for k in range(T):
    kind, z, R, ea = obs(k, e.state())
    e.step_recorded(h, kind, float(t[k]), z, R, ea)
  slabs = [getattr(h, a).cpu().numpy() for a in SLABS]
  for norm in ([False, True] if q else [False]):
    kw = dict(norm_quats=norm, quaternion_idxs=tuple(q) or (0,))
    xw, Pw = e.rts_smooth(h, **kw)
    xr, Pr = hiprec.rts(m, *slabs, h.t_host, quat_idxs=q, norm_quats=norm, sel=sel)
    for S in (1, 2, 3, 4, T, T + 2):
      xs, Ps = _chained(e, h, S, kw)
      dx, dP = _rows_that_differ(xs, xw), _rows_that_differ(Ps, Pw)
      assert not dx and not dP, f"{case} S={S} norm={norm}: rows of xs {dx}, of Ps {dP} differ from the whole history"
      ex, eP = state_err(xs.cpu().numpy()[:, sel], xr), cov_err(Ps.cpu().numpy()[:, sel], Pr)
      assert ex < TIGHT and eP < TIGHT, (S, norm, ex, eP)
    print(f"{case} chained segments (norm {norm}): state {ex:.1e} cov {eP:.1e}")


E2E = ["shape_e6", "shape_e31", "shape_e16", "live"]   # thread, single-warp and pair step kernels, and live


@pytest.mark.parametrize("norm_quats", [False, True])
@pytest.mark.parametrize("case", E2E)
def test_checkpointed_smoother_equals_tiled_smoother(case, norm_quats):
  """CheckpointedSmoother (checkpoints, segments re-filtered with history and smoothed last to first) == TiledSmoother
  (one backward pass over the whole stored history), bit for bit, over T = 37 steps of kinds without extra arguments."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother
  TT = 37
  if case == "live":
    from rednose_b200.filters.live import LiveKalman
    folder, G, q = ensure_generated(LiveKalman), 16, [3]
    x, P, Q = live_batch(2 * G + 1, seed=320)
    rng = np.random.default_rng(321)
    kinds = [12 if k % 7 == 0 else (4 if k % 2 else 10) for k in range(TT)]
    zR = [_live_obs(kind, x, rng) for kind in kinds]
  else:
    cls = shapes.BY_NAME[case]
    folder, G, q = ensure_generated(cls), cls.group(), cls.quat_idxs()
    m = hiprec.model_of(cls)
    x, P, Q, _ = shapes.batch(cls, 2 * G + 1, seed=320)
    plain = [k for k, (_, ea, _) in cls.kinds().items() if not ea]
    kinds = [plain[k % len(plain)] for k in range(TT)]
    zR = [shapes.observe(cls, m, kind, x, seed=330 + k)[:2] for k, kind in enumerate(kinds)]
  B, D, E = x.shape[0], x.shape[1], P.shape[1]
  t = 0.01 * np.arange(1, TT + 1) + 0.003 * (np.arange(TT) % 3)

  def obs_fn(k, lo, hi):
    return float(t[k]), kinds[k], zR[k][0][lo:hi].copy(), zR[k][1][lo:hi]

  want_x, want_P = np.full((TT, B, D), np.nan), np.full((TT, B, E, E), np.nan)

  def tiled_sink(lo, hi, xs, Ps):
    want_x[:, lo:hi], want_P[:, lo:hi] = xs.cpu().numpy(), Ps.cpu().numpy()

  TiledSmoother(folder, case, Q, D, E, quaternion_idxs=q, tile=G).run(x, P, TT, obs_fn, tiled_sink, norm_quats=norm_quats)
  assert not np.isnan(want_x).any()
  for segment, tile in ((4, G + 4), (12, B), (5, G + 4)):
    got_x, got_P = np.full_like(want_x, np.nan), np.full_like(want_P, np.nan)

    def sink(lo, hi, k0, xs, Ps):
      n = xs.shape[0]
      assert np.isnan(got_x[k0:k0 + n, lo:hi]).all()          # every (step, filter) delivered exactly once
      got_x[k0:k0 + n, lo:hi], got_P[k0:k0 + n, lo:hi] = xs.cpu().numpy(), Ps.cpu().numpy()

    cs = CheckpointedSmoother(folder, case, Q, D, E, quaternion_idxs=q, segment=segment, tile=tile)
    assert cs.plan(B, TT)[1] == (1 if tile == B else 2)
    cs.run(x, P, TT, obs_fn, sink, norm_quats=norm_quats)
    bad = sorted({int(k) for k in np.argwhere(got_x != want_x)[:, 0]} | {int(k) for k in np.argwhere(got_P != want_P)[:, 0]})
    assert not bad, f"{case} segment {segment}: steps {bad} differ from the whole history"
