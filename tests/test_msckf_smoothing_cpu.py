"""MSCKF smoothing without a GPU: the main-block RTS of the 40-digit reference (tests/hiprec.py) is itself right, and the
smoother each MSCKF shape with EDIM <= 32 is served by is pinned.

The reference smooths only the main block of an MSCKF (ekf_sym.py:651-690 with dim_main / dim_main_err).  It is checked
against oracle/rts_numpy.rts_smooth, the reference's recursion restated in float64, driven here by the model's own leaf
functions in float64 and, at the shipped msckf, by the reference generator's C where that oracle library is built."""
import os
import re

import numpy as np
import pytest

from tests import hiprec
from tests.msckf_shapes import BY_NAME, MSCKF_SHAPES, augment_np, batch, observe
from tests.util import cov_err, state_err

SMOOTHED = [BY_NAME[n] for n in ("msckf_e18", "msckf_e27", "msckf_e28")]
IDS = [c.name for c in SMOOTHED]


class _Leaves:
  """The leaf interface rts_numpy drives (``leaf(name, *inputs, out)``) over HiPrecModel.np_leaf, in float64."""
  KEYS = {"F_fun": "F", "err_fun": "err", "inv_err_fun": "inv_err"}

  def __init__(self, m):
    self.m = m

  def leaf(self, fn, *args):
    *inputs, out = args
    out[...] = self.m.np_leaf(self.KEYS[fn], *inputs).reshape(out.shape)


def _f64_history(cls, m, T, seed, augment_after=2):
  """One filter's recorded history in float64: every kind in turn, irregular times, and the clone-window shift after
  step `augment_after` (x_{k|k} is recorded before the shift, as predict_and_update_batch(augment=True) records it)."""
  x, P, Q, _ = batch(cls, 1, seed=seed)
  x, P = x[0], P[0]
  q, E = cls.quat_idxs(), cls.edim()
  rng = np.random.default_rng(seed)
  t = np.cumsum(rng.uniform(0.005, 0.04, T))
  kinds = sorted(cls.kinds())
  rows = [[], [], [], []]
  for k in range(T):
    dt = t[k] - t[k - 1] if k else 0.0
    F = m.np_leaf('F', x, dt).reshape(E, E)
    x = m.np_leaf('f', x, dt)
    for i in q:
      x[i:i + 4] /= np.linalg.norm(x[i:i + 4])
    P = F @ P @ F.T + dt * Q
    rows[0].append(x); rows[2].append(P)
    kind = kinds[k % len(kinds)]
    z, R, ea = observe(cls, m, kind, x[None], seed=seed + k)
    x, P, _ = m.step_f64(kind, x, P, None, 0.0, z[0], R[0], quat_idxs=q, ea=None if ea is None else ea[0], predict=False)
    rows[1].append(x); rows[3].append(P)
    if k == augment_after:
      xa, Pa = augment_np(cls, x[None], P[None])
      x, P = xa[0], Pa[0]
  x_pred, x_filt, P_pred, P_filt = (np.stack(r) for r in rows)
  return x_pred, x_filt, P_pred, P_filt, t


# norm_quats only where state 3 starts a quaternion (msckf_e27 has none: rts_numpy would normalise four plain states)
@pytest.mark.parametrize("cls, norm_quats", [(c, n) for c in SMOOTHED for n in ([False, True] if c.quat_idxs() else [False])],
                         ids=[f"{c.name}-{n}" for c in SMOOTHED for n in ([False, True] if c.quat_idxs() else [False])])
def test_main_block_reference_agrees_with_rts_numpy(cls, norm_quats):
  """hiprec.rts in main-block mode == rts_numpy.rts_smooth(dim_main, dim_main_err) to 1e-12, with the quaternion at 3
  (rts_numpy's hard-coded slice) normalised or not.  The clone part of the smoothed state and every covariance entry
  outside the main block are x_{k|k} / P_{k|k} in both."""
  from oracle.rts_numpy import rts_smooth
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  slabs = _f64_history(cls, m, 6, seed=5)
  t = slabs[-1]
  xo, Po = rts_smooth(_Leaves(m), *slabs, cls.dmain(), cls.medim(), norm_quats=norm_quats)
  xr, Pr = hiprec.rts(m, *[s[:, None] for s in slabs[:4]], t, quat_idxs=(3,), norm_quats=norm_quats)
  xr, Pr = xr[:, 0], Pr[:, 0]
  ex, eP = state_err(xo, xr), cov_err(Po, Pr)
  print(f"{cls.name} norm {norm_quats}: state {ex:.1e} cov {eP:.1e}")
  assert ex < 1e-12 and eP < 1e-12, (ex, eP)
  x_filt, P_filt, ME, DM = slabs[1], slabs[3], cls.medim(), cls.dmain()
  assert np.array_equal(xr[:-1, DM:], x_filt[:-1, DM:])       # the normalised slice 3:7 lies in the main block
  assert np.array_equal(Pr[:-1, ME:], P_filt[:-1, ME:]) and np.array_equal(Pr[:-1, :, ME:], P_filt[:-1, :, ME:])
  assert state_err(xr[:-1, :DM], x_filt[:-1, :DM]) > 1e-6     # the main block is smoothed


def test_main_block_reference_agrees_with_the_oracle_at_the_shipped_msckf():
  """At the shipped msckf (EDIM 82: main block 23 / 22, ten pose clones): hiprec.rts against rts_numpy driven by the
  reference generator's own leaf C, over a history filtered by the oracle."""
  from oracle import build_ref
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  from oracle.rts_numpy import rts_smooth
  from rednose_b200.filters.live import DIM_STATE, DIM_STATE_ERR
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.util import Oracle, msckf_batch, msckf_feature_obs
  o = Oracle(build_ref.OUT, "msckf")
  m = hiprec.model_of(MsckfKalman)
  x, P, Q, point = msckf_batch(1, seed=7)
  T, t = 4, np.array([0.0, 0.01, 0.025, 0.03])
  rows = [[], [], [], []]
  for k in range(T):
    x, P = o.predict(x, P, Q, t[k] - t[k - 1] if k else 0.0)
    rows[0].append(x[0].copy()); rows[2].append(P[0].copy())
    z, R, _ = msckf_feature_obs(o, x, point, seed=8 + k)
    x, P, _ = o.update(MsckfKalman.feature_kind, x, P, z, R, ea=point)
    rows[1].append(x[0].copy()); rows[3].append(P[0].copy())
  slabs = [np.stack(r) for r in rows]
  xo, Po = rts_smooth(o, *slabs, t, DIM_STATE, DIM_STATE_ERR, norm_quats=True)
  xr, Pr = hiprec.rts(m, *[s[:, None] for s in slabs], t, quat_idxs=(3,), norm_quats=True)
  ex, eP = state_err(xo, xr[:, 0]), cov_err(Po, Pr[:, 0])
  print(f"msckf: state {ex:.1e} cov {eP:.1e}")
  assert ex < 1e-9 and eP < 1e-9, (ex, eP)


def test_smoother_kernel_of_every_msckf_shape():
  """launch_rts_auto: the tensor-core smoother for even EDIM <= 32 with MEDIM >= 8, the scalar one for any other EDIM <= 32,
  none above.  msckf_e18 is even but its main block has 6 error states, so it runs the scalar kernel.  The EDIM / MEDIM
  the rule reads are those of the generated model."""
  from rednose_b200.filters import ensure_generated
  want = {"msckf_e18": "scalar", "msckf_e27": "scalar", "msckf_e28": "mma"}
  assert {c.name: c.rts_kernel() for c in MSCKF_SHAPES} == {c.name: want.get(c.name) for c in MSCKF_SHAPES}
  for cls in SMOOTHED:
    src = open(os.path.join(ensure_generated(cls), f"{cls.name}.cu"), encoding="utf-8").read()
    edim, medim = (int(re.search(rf"\b{k} = (\d+)", src).group(1)) for k in ("EDIM", "MEDIM"))
    assert (edim, medim) == (cls.edim(), cls.medim()), cls.name
