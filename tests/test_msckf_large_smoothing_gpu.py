"""RTS smoothing of MSCKFs above EDIM 32 (main block only) against the 40-digit reference of tests/hiprec.py.

Above EDIM 32 a lane cannot own a column of the covariance, so ekf_rts_warp_mma (msckf_e64, e68, e166 and the shipped
msckf) and ekf_rts_warp (odd EDIM: msckf_e33, e73) read and write only the main block, which is at most 32 wide.  The
rest of Ps[0 .. T-2] is P_{k|k}: left in place, or copied into an output buffer before the launch.  The clone part of xs
is x_{k|k} (ekf_sym.py:651-690).

Each case records T = 8 steps of B = 7 filters (odd: the last CTA of RTS_WARPS = 2 smooths one filter), plain and feature
kinds at irregular times, with the clone window shifted inside one recording step (step_recorded(..., augment=True)).
The reference replays every recorded row of the sampled filters (the first, the first of the second CTA, the last;
only the first and the last at EDIM 166 and the shipped msckf) and smooths them, state per component and covariance in correlation
units at TIGHT = 1e-9.  The other checks are bit for bit over the whole batch: in place against out of place, hP_pred
outside the main block never read, chained segments against the whole pass, and histories of one and two steps.  At the
shipped msckf the smoothed rows are also compared with oracle/rts_numpy driven by the reference generator's C, where
oracle/_ref/libmsckf.so is built.

The 40-digit arithmetic on the host dominates the runtime: about 10 minutes on an H100 machine, 2.5 of them at the
shipped msckf (mostly building its reference model) and the most at msckf_e166.
"""
import os

import numpy as np
import pytest
import torch

from tests import hiprec, msckf_shapes
from tests.msckf_shapes import MsckfShape, augment_np
from tests.test_rts_segments_gpu import SLABS, _chained, _rows_that_differ
from tests.util import cov_err, msckf_batch, quat_norm_err, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
T, AUG, B = 8, 3, 7
GV = [1.0, 1.25]
CASES = ["msckf_e33", "msckf_e64", "msckf_e68", "msckf_e73", "msckf_e166", "msckf"]
SEL = {"msckf_e166": [0, B - 1], "msckf": [0, B - 1]}   # elsewhere [0, 2, B - 1]


class _Msckf(MsckfShape):
  """The shipped msckf with the facts of a tests/msckf_shapes.py shape: main block 23 / 22, ten pose clones, the plain
  kind 12 (ECEF position) and the feature kind 17 (ten views of one point, the point as extra arguments)."""
  name = "msckf"
  spec = dict(medim=22, eskf=True, n_clones=10, clone='pose', features=[])

  @classmethod
  def kinds(cls):
    return {12: (3, 0, False, False), 17: (20, 3, True, True)}


def _observe(cls, m, kind, x, point, seed):
  """(z, R, ea) of one observation per filter; the msckf's feature kind looks at `point`, noise 1e-3 (5 for kind 12)."""
  if cls is not _Msckf:
    return msckf_shapes.observe(cls, m, kind, x, seed=seed)
  rng = np.random.default_rng(seed)
  sd = 1e-3 if kind == 17 else 5.0
  z = np.stack([m.np_leaf(('h', kind), x[b], *([point[b]] if kind == 17 else [])) for b in range(x.shape[0])])
  z = z + sd * rng.normal(size=z.shape)
  R = np.tile(np.eye(z.shape[1]) * sd ** 2, (x.shape[0], 1, 1))
  return z, R, (point if kind == 17 else None)


@pytest.fixture(scope="module", params=CASES)
def rec(request):
  """One recorded history per case: engine, history, observations, host slabs and the reference model."""
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  name = request.param
  if name == "msckf":
    from rednose_b200.filters.msckf import MsckfKalman
    cls, folder = _Msckf, ensure_generated(MsckfKalman)
    m = hiprec.model_of(MsckfKalman)
    x, P, Q, point = msckf_batch(B, seed=400)
  else:
    cls = msckf_shapes.BY_NAME[name]
    folder, m = ensure_generated(cls), hiprec.model_of(cls)
    x, P, Q, _ = msckf_shapes.batch(cls, B, seed=400)
    point = None
  m.gv = GV[:len(m.gvars)]
  gv = {g: GV[i] for i, g in enumerate(cls.global_names())}
  q = cls.quat_idxs()
  e = BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q, global_vars=gv)
  plain, feat = [k for k, v in cls.kinds().items() if not v[3]][0], cls.feature_kinds()[0]
  kinds = [plain, feat, feat, feat, plain, feat, plain, feat]
  t = np.cumsum(np.random.default_rng(401).uniform(0.005, 0.04, T))
  h = e.new_history(T)
  obs = []
  for k in range(T):
    obs.append(_observe(cls, m, kinds[k], e.state(), point, seed=410 + k))
    e.step_recorded(h, kinds[k], float(t[k]), *obs[k], augment=(k == AUG))
  slabs = [getattr(h, a).cpu().numpy() for a in SLABS]
  return dict(cls=cls, m=m, e=e, h=h, x0=x, P0=P, Q=Q, q=q, kinds=kinds, obs=obs, slabs=slabs,
              sel=SEL.get(name, [0, 2, B - 1]), norms=[False, True] if q else [False])


def _kw(r, norm):
  return dict(norm_quats=norm, quaternion_idxs=tuple(r["q"]) or (0,))


def _copy(r, n=None):
  """A new history holding the first n rows of the recorded one."""
  h = r["h"]
  n = h.n if n is None else n
  c = r["e"].new_history(n)
  for a in SLABS:
    getattr(c, a).copy_(getattr(h, a)[:n])
  c.t_host[:] = h.t_host[:n]
  c.n = n
  return c


def _check(tag, x, P, xr, Pr):
  ex, eP = state_err(x, xr), cov_err(P, Pr)
  print(f"{tag}: state {ex:.1e} cov {eP:.1e}")
  assert ex < TIGHT and eP < TIGHT, (tag, ex, eP)


def _outside_main_block_is_filtered(r, xs, Ps, norm):
  """Rows 0 .. T-2 outside the main block: P_{k|k} bit for bit; the clone part of x likewise, except a listed clone
  quaternion, which is normalised in rows >= 1.  The last row is the predicted estimate, where the recursion starts."""
  cls, q = r["cls"], r["q"]
  xp, xf, Pp, Pf = (a[:xs.shape[0]] for a in r["slabs"])
  ME, DM, n = cls.medim(), cls.dmain(), xs.shape[0]
  assert np.array_equal(Ps[:-1, :, ME:], Pf[:-1, :, ME:]) and np.array_equal(Ps[:-1, :, :, ME:], Pf[:-1, :, :, ME:])
  assert np.array_equal(Ps[-1], Pp[-1])
  renorm = [i + c for i in q if i >= DM for c in range(4)] if norm else []
  keep = [i for i in range(DM, cls.dim()) if i not in renorm]
  assert np.array_equal(xs[:-1, :, keep], xf[:-1, :, keep])
  assert np.array_equal(xs[0, :, DM:], xf[0, :, DM:])
  if renorm and n > 2:
    want = xf[1:-1, :, renorm].reshape(n - 2, B, -1, 4)
    want = want / np.linalg.norm(want, axis=-1, keepdims=True)
    assert state_err(xs[1:-1, :, renorm], want.reshape(n - 2, B, -1)) < 1e-15
  if norm and n > 1:
    assert quat_norm_err(xs[1:], q) <= 1e-15


def test_recorded_rows_and_the_smoothed_main_block_match_the_reference(rec):
  r = rec
  cls, m, sel, q, kinds = r["cls"], r["m"], r["sel"], r["q"], r["kinds"]
  xp, xf, Pp, Pf = r["slabs"]
  t = r["h"].t_host
  xa, Pa = augment_np(cls, xf[AUG], Pf[AUG])   # the recorded x_{AUG|AUG} is the estimate before the clone shift
  xk, Pk = r["x0"][sel], r["P0"][sel]
  for k in range(T):
    if k:
      xk, Pk = (xa[sel], Pa[sel]) if k - 1 == AUG else (xf[k - 1, sel], Pf[k - 1, sel])
    z, R, ea = (None if a is None else a[sel] for a in r["obs"][k])
    xr, Pr = hiprec.predict(m, xk, Pk, r["Q"], t[k] - t[k - 1] if k else 0.0, quat_idxs=q)
    _check(f"{cls.name} row {k} predicted", xp[k, sel], Pp[k, sel], xr, Pr)
    xr, Pr, _ = hiprec.update(m, kinds[k], xp[k, sel], Pp[k, sel], z, R, ea, quat_idxs=q)
    _check(f"{cls.name} row {k} filtered (kind {kinds[k]})", xf[k, sel], Pf[k, sel], xr, Pr)
  for norm in r["norms"]:
    xs, Ps = (a.cpu().numpy() for a in r["e"].rts_smooth(r["h"], **_kw(r, norm)))
    xr, Pr = hiprec.rts(m, *r["slabs"], t, quat_idxs=q, norm_quats=norm, sel=sel)
    _check(f"{cls.name} rts (norm {norm})", xs[:, sel], Ps[:, sel], xr, Pr)
    _outside_main_block_is_filtered(r, xs, Ps, norm)
    assert state_err(xs[:-1, :, :cls.dmain()], xf[:-1, :, :cls.dmain()]) > 1e-9   # the main block is smoothed


def test_in_place_and_out_of_place_are_identical(rec):
  """A new buffer, a preallocated out= (NaN, one row longer than the history) and in place give the same bits; in place
  leaves every element of P_{k|k} outside the main block as it was."""
  r, ME = rec, rec["cls"].medim()
  for norm in r["norms"]:
    xs, Ps = r["e"].rts_smooth(r["h"], **_kw(r, norm))
    out = (torch.full((T + 1,) + xs.shape[1:], float("nan"), dtype=torch.float64, device=xs.device),
           torch.full((T + 1,) + Ps.shape[1:], float("nan"), dtype=torch.float64, device=xs.device))
    xo, Po = r["e"].rts_smooth(r["h"], out=out, **_kw(r, norm))
    assert torch.isnan(out[0][T]).all() and torch.isnan(out[1][T]).all()
    c = _copy(r)
    before = c.P_filt.clone()
    xi, Pi = r["e"].rts_smooth(c, in_place=True, **_kw(r, norm))
    assert xi.data_ptr() == c.x_filt.data_ptr() and Pi.data_ptr() == c.P_filt.data_ptr()
    for a, b in ((xo, xs), (Po, Ps), (xi, xs), (Pi, Ps)):
      assert torch.equal(a, b), norm
    assert torch.equal(Pi[:-1, :, ME:], before[:-1, :, ME:]) and torch.equal(Pi[:-1, :, :, ME:], before[:-1, :, :, ME:])


def test_only_the_main_block_of_the_predicted_covariance_is_read(rec):
  """NaN in hP_pred outside the main block of rows 1 .. T-2 and in all of row 0 changes no bit of the result."""
  r, ME = rec, rec["cls"].medim()
  c = _copy(r)
  c.P_pred[0] = float("nan")
  c.P_pred[1:-1, :, ME:] = float("nan")
  c.P_pred[1:-1, :, :, ME:] = float("nan")
  for norm in r["norms"]:
    xw, Pw = r["e"].rts_smooth(r["h"], **_kw(r, norm))
    xs, Ps = r["e"].rts_smooth(c, **_kw(r, norm))
    assert torch.equal(xs, xw) and torch.equal(Ps, Pw), norm


def test_chained_segments_equal_the_whole_history(rec):
  """Segments of S = 1, 2, 3, T and T + 2 steps, last first, each started from the smoothed first row of the one behind
  it (P_term full [B, EDIM, EDIM]), give the whole-history pass bit for bit; rows a segment does not deliver stay
  unwritten."""
  r = rec
  for norm in r["norms"]:
    xw, Pw = r["e"].rts_smooth(r["h"], **_kw(r, norm))
    for S in (1, 2, 3, T, T + 2):
      xs, Ps = _chained(r["e"], r["h"], S, _kw(r, norm))
      dx, dP = _rows_that_differ(xs, xw), _rows_that_differ(Ps, Pw)
      assert not dx and not dP, f"{r['cls'].name} S={S} norm={norm}: rows of xs {dx}, of Ps {dP} differ"


@pytest.mark.parametrize("n", [1, 2])
def test_one_and_two_step_histories(rec, n):
  """T = 1: the predicted estimate, unnormalised (global step 0).  T = 2: one backward step, against the reference."""
  r = rec
  cls, sel = r["cls"], r["sel"]
  c = _copy(r, n)
  xp, xf, Pp, Pf = (a[:n] for a in r["slabs"])
  for norm in r["norms"]:
    xs, Ps = (a.cpu().numpy() for a in r["e"].rts_smooth(c, **_kw(r, norm)))
    assert xs.shape[0] == n and Ps.shape[0] == n
    if n == 1:
      assert np.array_equal(xs[0], xp[0]) and np.array_equal(Ps[0], Pp[0])
      continue
    xr, Pr = hiprec.rts(r["m"], xp, xf, Pp, Pf, c.t_host, quat_idxs=r["q"], norm_quats=norm, sel=sel)
    _check(f"{cls.name} T = 2 rts (norm {norm})", xs[:, sel], Ps[:, sel], xr, Pr)
    _outside_main_block_is_filtered(r, xs, Ps, norm)


def test_shipped_msckf_agrees_with_the_reference_recursion(rec):
  """At the shipped msckf: rts_numpy (the reference's recursion in float64) over the recorded slabs, driven by the
  reference generator's leaf C; the attitude at 3 normalised or not, as the reference's hard-coded slice does."""
  r = rec
  if r["cls"] is not _Msckf:
    pytest.skip("the shipped msckf only")
  from oracle import build_ref
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  from oracle.rts_numpy import rts_smooth
  from rednose_b200.filters.live import DIM_STATE, DIM_STATE_ERR
  from tests.util import Oracle
  o = Oracle(build_ref.OUT, "msckf")
  for norm in (False, True):
    xs, Ps = (a.cpu().numpy() for a in r["e"].rts_smooth(r["h"], norm_quats=norm, quaternion_idxs=(3,)))
    for b in r["sel"]:
      xo, Po = rts_smooth(o, *[a[:, b] for a in r["slabs"]], r["h"].t_host, DIM_STATE, DIM_STATE_ERR, norm_quats=norm)
      _check(f"msckf filter {b} against rts_numpy (norm {norm})", xs[:, b], Ps[:, b], xo, Po)
