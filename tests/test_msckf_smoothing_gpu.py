"""RTS smoothing of MSCKF histories (EDIM <= 32: main block only) against the 40-digit reference of tests/hiprec.py.

An MSCKF with EDIM <= 32 is smoothed by ekf_rts_warp_mma (even EDIM, MEDIM >= 8) or ekf_rts_warp (otherwise), on its main
block only: the clone rows and columns of Ps are P_{k|k}, and the clone part of xs is x_{k|k} (ekf_sym.py:651-690).  The
three shapes reach both kernels with a main block smaller than the state: msckf_e18 (MEDIM 6: scalar kernel although
EDIM is even), msckf_e27 (odd EDIM: scalar kernel) and msckf_e28 (tensor-core kernel, a pose clone whose quaternion the
smoother normalises).

Each shape runs B = 2G + 1 filters (G: the group of the kernel that runs its plain kinds) and the reference is evaluated on
the first and last filter and on both sides of every group boundary.  The history mixes plain kinds (pair or single-warp
kernel) with feature kinds (CTA kernel), irregular times and one clone-window shift between two recorded steps.  State
per component and covariance in correlation units, at TIGHT = 1e-9.
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME, augment_np, batch, observe
from tests.shapes import sample
from tests.util import cov_err, quat_norm_err, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
SMOOTHED = [BY_NAME[n] for n in ("msckf_e18", "msckf_e27", "msckf_e28")]
IDS = [c.name for c in SMOOTHED]


def _engine(cls, x, P, Q):
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  return BatchedEKF(ensure_generated(cls), cls.name, Q, x, P, quaternion_idxs=cls.quat_idxs())


def _check(tag, x, P, xr, Pr):
  ex, eP = state_err(x, xr), cov_err(P, Pr)
  print(f"{tag}: state {ex:.1e} cov {eP:.1e}")
  assert ex < TIGHT and eP < TIGHT, (tag, ex, eP)


@pytest.mark.parametrize("cls", SMOOTHED, ids=IDS)
def test_whole_history_smoothed_on_the_main_block(cls):
  """step_recorded over T = 8 steps (plain and feature kinds, irregular times, augment() after step 3), every recorded row
  of the sampled filters against a 40-digit replay from the row before, then rts_smooth with and without quaternion
  normalisation against the main-block reference, and the clone part of xs / Ps against x_{k|k} / P_{k|k} bit for bit."""
  m = hiprec.model_of(cls)
  B = 2 * cls.group() + 1
  sel = sample(cls, B)
  x, P, Q, _ = batch(cls, B, seed=200)
  q, DM, ME, T, AUG = cls.quat_idxs(), cls.dmain(), cls.medim(), 8, 3
  plain, feat = [k for k, v in cls.kinds().items() if not v[3]][0], cls.feature_kinds()[0]
  kinds = [plain, feat, feat, plain, feat, plain, feat, feat]
  t = np.cumsum(np.random.default_rng(201).uniform(0.005, 0.04, T))
  e = _engine(cls, x, P, Q)
  h = e.new_history(T)
  obs = []
  for k in range(T):
    obs.append(observe(cls, m, kinds[k], e.state(), seed=210 + k))
    e.step_recorded(h, kinds[k], float(t[k]), *obs[k])
    if k == AUG:
      e.augment()
  slabs = [s.cpu().numpy() for s in (h.x_pred, h.x_filt, h.P_pred, h.P_filt)]
  xp, xf, Pp, Pf = slabs
  xa, Pa = augment_np(cls, xf[AUG], Pf[AUG])
  xk, Pk = x[sel], P[sel]
  for k in range(T):   # the row before: the initial state, or x_{k-1|k-1} (shifted after step AUG)
    if k:
      xk, Pk = (xa[sel], Pa[sel]) if k - 1 == AUG else (xf[k - 1, sel], Pf[k - 1, sel])
    z, R, ea = (None if a is None else a[sel] for a in obs[k])
    xr, Pr = hiprec.predict(m, xk, Pk, Q, t[k] - t[k - 1] if k else 0.0, quat_idxs=q)
    _check(f"{cls.name} row {k} predicted", xp[k, sel], Pp[k, sel], xr, Pr)
    xr, Pr, _ = hiprec.update(m, kinds[k], xp[k, sel], Pp[k, sel], z, R, ea, quat_idxs=q)
    _check(f"{cls.name} row {k} filtered (kind {kinds[k]})", xf[k, sel], Pf[k, sel], xr, Pr)
  for norm in ([False, True] if q else [False]):
    xs, Ps = (a.cpu().numpy() for a in e.rts_smooth(h, norm_quats=norm, quaternion_idxs=tuple(q) or (0,)))
    xr, Pr = hiprec.rts(m, *slabs, h.t_host, quat_idxs=q, norm_quats=norm, sel=sel)
    _check(f"{cls.name} rts ({cls.rts_kernel()}, norm {norm})", xs[:, sel], Ps[:, sel], xr, Pr)
    # outside the main block: P_{k|k} (the last row: P_{T-1|T-2}, where the recursion starts), bit for bit
    assert np.array_equal(Ps[:-1, :, ME:], Pf[:-1, :, ME:]) and np.array_equal(Ps[:-1, :, :, ME:], Pf[:-1, :, :, ME:])
    assert np.array_equal(Ps[-1], Pp[-1])
    # the clone part of x: x_{k|k} bit for bit, except a listed clone quaternion, which is normalised in rows >= 1
    renorm = [i + c for i in q if i >= DM for c in range(4)] if norm else []
    keep = [i for i in range(DM, cls.dim()) if i not in renorm]
    assert np.array_equal(xs[:-1, :, keep], xf[:-1, :, keep])
    assert np.array_equal(xs[0, :, DM:], xf[0, :, DM:])
    if renorm:
      want = xf[1:-1, :, renorm].reshape(T - 2, B, -1, 4)
      want = want / np.linalg.norm(want, axis=-1, keepdims=True)
      assert state_err(xs[1:-1, :, renorm], want.reshape(T - 2, B, -1)) < 1e-15
    if norm:
      assert quat_norm_err(xs[1:], q) <= 1e-15
