"""CPU tests of the parity metrics in tests/util.py and of the high-precision reference in tests/hiprec.py.

The metrics must see an error in a small component (a quaternion, a bias, a 1e-4 variance) even when the state also
holds 4e6 m ECEF positions, and must not depend on the units of the state.  The high-precision reference must agree
with the float64 oracle to float64 rounding on well-conditioned inputs, so that it can arbitrate where two float64
implementations legitimately differ."""
import numpy as np
import pytest

from tests.util import LIVE_KINDS, Oracle, cov_err, live_batch, live_obs, quat_norm_err, state_err


def test_cov_err_is_invariant_under_rescaling_of_the_state_units():
  rng = np.random.default_rng(0)
  _, A, _ = live_batch(8, seed=1, well_conditioned=False)
  B = A * (1 + 1e-4 * rng.normal(size=A.shape))   # the difference keeps ~12 significant digits
  B = 0.5 * (B + np.transpose(B, (0, 2, 1)))
  d = np.exp(rng.uniform(-8, 8, 22))
  D = d[:, None] * d[None, :]
  e, eD = cov_err(B, A), cov_err(D * B, D * A)
  assert e > 0 and abs(eD - e) <= 1e-10 * e, (e, eD)


def test_state_err_is_invariant_under_rescaling_of_columns():
  rng = np.random.default_rng(1)
  x, _, _ = live_batch(16, seed=2)
  y = x * (1 + 1e-4 * rng.normal(size=x.shape))
  s = np.exp(rng.uniform(-10, 10, 23))
  e, es = state_err(y, x), state_err(y * s, x * s)
  assert e > 0 and abs(es - e) <= 1e-10 * e, (e, es)


@pytest.mark.parametrize("col", [3, 4, 5, 6, 13, 20])
def test_small_component_error_is_seen_next_to_ecef_positions(col):
  """A 1e-6 relative error in one quaternion / bias component of one filter is reported as >= 1e-6 although the
  positions of the same state are 4e6 m (a whole-array max-norm ratio would report ~1e-13 here)."""
  x, _, _ = live_batch(64, seed=3)
  y = x.copy()
  b = int(np.argmax(np.abs(x[:, col])))
  y[b, col] *= 1 + 1e-6
  assert state_err(y, x) >= 1e-6 * (1 - 1e-9)
  assert np.max(np.abs(y - x)) / np.max(np.abs(x)) < 1e-12        # what the old metric saw


def test_smallest_variance_error_is_seen_next_to_the_position_block():
  _, P, _ = live_batch(8, seed=4, well_conditioned=False)      # variances 1e8 .. 1e-4
  i = int(np.argmin(np.diagonal(P[0])))
  Q = P.copy()
  Q[0, i, i] *= 1 + 1e-6
  assert cov_err(Q, P) >= 1e-6 * (1 - 1e-9)
  assert np.max(np.abs(Q - P)) / np.max(np.abs(P)) < 1e-16


def test_cov_err_rejects_a_non_positive_reference_diagonal():
  _, P, _ = live_batch(2, seed=5)
  P[1, 7, 7] = 0.0
  with pytest.raises(AssertionError):
    cov_err(P, P)


def test_state_err_compares_all_zero_components_absolutely():
  want = np.zeros((4, 3))
  want[:, 0] = 5.0
  got = want.copy()
  got[2, 1] = 3e-9
  assert state_err(got, want) == pytest.approx(3e-9, rel=1e-12)


def test_quat_norm_err_covers_every_listed_index():
  x = np.zeros((5, 20))
  x[:, 2] = 1.0
  x[:, 9] = 1.0
  assert quat_norm_err(x, [2, 9]) == 0.0
  x[3, 10] = 1e-3                                                # second quaternion off unit norm
  assert quat_norm_err(x, [2]) == 0.0 and quat_norm_err(x, [2, 9]) == pytest.approx(np.hypot(1, 1e-3) - 1, rel=1e-9)


# ------------------------------------------------------------------ the high-precision reference vs the oracle ---
# Measured on well-conditioned live_batch inputs (8 kinds x 3 filters): the float64 oracle is within 1.0e-14 (state and
# innovation, per component) and 7.5e-16 (covariance, correlation units) of the 40-digit result; bounds 10x that.
# The exception is anything computed from a difference of ECEF positions: a 4.2e6 m coordinate carries an absolute
# rounding of up to 4.7e-10 m, so the innovation of a position fix (a few metres) and the corrections it drives, and
# the RTS increments inv_err_fun(x_pred, x_smooth), are only defined to ~1e-10 relative in float64 (measured 8.5e-11
# and 5.8e-11); those are held to 1e-9.  The RTS covariance measured 5.6e-15 and is held to 1e-13.
HIPREC_X, HIPREC_P, HIPREC_POS = 1e-13, 1e-14, 1e-9


@pytest.mark.parametrize("kind", sorted(LIVE_KINDS))
def test_hiprec_fused_step_matches_the_oracle(oracle_dir, kind):
  from tests import hiprec
  o = Oracle(oracle_dir, "live")
  x, P, Q = live_batch(3, seed=40 + kind)
  z, R = live_obs(o, kind, x, seed=7)
  xr, Pr, yr = o.batch_step(kind, x, P, Q, 0.01, z, R, quat_idxs=[3], flags=3, nthreads=1)
  xh, Ph, yh = hiprec.live_step(kind, x, P, Q, 0.01, z, R, quat_idxs=[3], flags=3)
  ex, eP, ey = state_err(xr, xh), cov_err(Pr, Ph), state_err(yr, yh)
  tol_x = HIPREC_POS if kind == 12 else HIPREC_X
  assert ex < tol_x and eP < HIPREC_P and ey < tol_x, (ex, eP, ey)
  assert quat_norm_err(xh, [3]) <= 1e-15


def test_hiprec_rts_matches_the_oracle(oracle_dir):
  from oracle.rts_numpy import rts_smooth
  from tests import hiprec
  o = Oracle(oracle_dir, "live")
  B, T = 2, 10
  x, P, Q = live_batch(B, seed=60)
  hist = {k: [] for k in ("xp", "xf", "Pp", "Pf")}
  t = 0.01 * np.arange(1, T + 1)
  for k in range(T):
    kind = 12 if k % 5 == 0 else (4 if k % 2 else 10)
    z, R = live_obs(o, kind, x, seed=70 + k)
    xp, Pp = o.predict(x, P, Q, 0.01)
    for q in xp:
      q[3:7] /= np.linalg.norm(q[3:7])
    x, P, _ = o.update(kind, xp, Pp, z, R)
    for q in x:
      q[3:7] /= np.linalg.norm(q[3:7])
    for key, v in zip(("xp", "xf", "Pp", "Pf"), (xp, x, Pp, P)):
      hist[key].append(v.copy())
  h = {k: np.stack(v) for k, v in hist.items()}
  for b in range(B):
    args = (h["xp"][:, b], h["xf"][:, b], h["Pp"][:, b], h["Pf"][:, b], t)
    xr, Pr = rts_smooth(o, *args, 23, 22, norm_quats=True)
    xh, Ph = hiprec.live_rts(*args, norm_quats=True)
    ex, eP = state_err(xr, xh), cov_err(Pr, Ph)
    assert ex < HIPREC_POS and eP < 10 * HIPREC_P, (b, ex, eP)
