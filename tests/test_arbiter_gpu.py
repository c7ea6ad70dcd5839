"""The high-precision reference (tests/hiprec.py) as the arbiter where the CUDA path and the oracle legitimately differ.

The kernels factor S with LDL^T and update P in the structured rank-m form P - (HP)^T S^-1 (HP); the oracle uses
full-pivot LU and dense Joseph products.  On the example's own ill-conditioned P0 (variances 1e8 .. 1e-4) the two
float64 results differ by more than rounding, and neither is "the" answer.  Here each is measured against the
40-digit result on the same float64 inputs, per component, and the CUDA path must not be much worse than the
oracle:  err(GPU, exact) <= C * err(oracle, exact) + FLOOR  for every state component / covariance entry.
"""
import numpy as np
import pytest

from tests import hiprec
from tests.util import LIVE_KINDS, Oracle, cov_err, live_batch, live_obs, quat_norm_err, state_err

pytestmark = pytest.mark.gpu
C = 10.0
FLOOR = 1e-12
# Covariances.  The kernels' rank-m update P - (HP)^T S^-1 (HP) subtracts a term as large as the prior and is first-order
# sensitive to rounding in the gain, where the oracle's Joseph form is not.  So a covariance entry loses about the
# digits by which the update shrinks its variances: eps * sqrt(prior_ii prior_jj / (post_ii post_jj)).  Measured on an
# H100 (700 W), single steps from the example's P0: 3.2e-9 for kind 9 (R = 0.00025^2 shrinks the rate variances
# 1.6e7-fold; 0.9 eps x that amplification), 1.1e-9 for kind 12, 1.0e-12 on entries the update barely changes; 6.2e-11
# after 50 IMU steps.  The Joseph form stays at 1e-15 .. 3e-11 on the same inputs.  The covariance floor is therefore
# 16 eps x the amplification (summed over the steps of a stream), and never below FLOOR_P = 1e-10.
FLOOR_P = 1e-10
EPS = np.finfo(np.float64).eps


def _engine(gen_dir, x, P, Q):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(gen_dir, "live", Q, x, P, quaternion_idxs=[3])


def _amplification(P_prior, P_post):
  """[n, n]: max over filters of sqrt(prior_ii prior_jj / (post_ii post_jj))."""
  s = np.sqrt(np.diagonal(P_prior, axis1=-2, axis2=-1) / np.diagonal(P_post, axis1=-2, axis2=-1))
  return (s[:, :, None] * s[:, None, :]).max(axis=0)


def _judge(what, got, oracle, exact, cov=False, floor=FLOOR):
  f = cov_err if cov else state_err
  eg, eo = f(got, exact, per_component=True), f(oracle, exact, per_component=True)
  bad = eg > C * eo + np.maximum(floor, FLOOR)
  ratio = float(np.max(eg / np.maximum(eo, 1e-17)))
  print(f"arbiter {what}: err(GPU) {eg.max():.2e}  err(oracle) {eo.max():.2e}  worst ratio {ratio:.1f}")
  assert not bad.any(), (what, np.argwhere(bad)[:5].tolist(), float(eg.max()), float(eo.max()))


@pytest.mark.parametrize("kind", sorted(LIVE_KINDS))
def test_arbiter_single_fused_step_ill_conditioned(gen_dir, oracle_dir, kind):
  o = Oracle(oracle_dir, "live")
  x, P, Q = live_batch(6, seed=700 + kind, well_conditioned=False)
  z, R = live_obs(o, kind, x, seed=3)
  xo, Po, yo = o.batch_step(kind, x, P, Q, 0.01, z, R, quat_idxs=[3], flags=3, nthreads=1)
  e = _engine(gen_dir, x, P, Q)
  yg = e.step(kind, 0.01, z, R).cpu().numpy()[:, 0]
  xh, Ph, yh = hiprec.live_step(kind, x, P, Q, 0.01, z, R, quat_idxs=[3], flags=3)
  _judge(f"kind {kind} x", e.state(), xo, xh)
  _judge(f"kind {kind} y", yg, yo, yh)
  _judge(f"kind {kind} P", e.covs(), Po, Ph, cov=True, floor=np.maximum(FLOOR_P, 16 * EPS * _amplification(P, Ph)))
  assert quat_norm_err(e.state(), [3]) <= 1e-15


def test_arbiter_imu_stream_and_rts_ill_conditioned(gen_dir, oracle_dir):
  """A 50-step gyro / accelerometer stream (no position fix: cond(P) stays ~1e12), then RTS over the GPU's history."""
  from oracle.rts_numpy import rts_smooth
  o = Oracle(oracle_dir, "live")
  B, T = 4, 50
  x, P, Q = live_batch(B, seed=710, well_conditioned=False)
  e = _engine(gen_dir, x, P, Q)
  e.filter_time = 0.0                       # the first step predicts over 0.01 s, like the oracle's
  hist = e.new_history(T)
  xo, Po = x.copy(), P.copy()
  xh, Ph = x.copy(), P.copy()
  amp = np.zeros((22, 22))
  for k in range(T):
    kind = 4 if k % 2 else 10
    z, R = live_obs(o, kind, xo, seed=720 + k)
    xo, Po, _ = o.batch_step(kind, xo, Po, Q, 0.01, z, R, quat_idxs=[3], flags=3, nthreads=1)
    P_prior = Ph
    xh, Ph, _ = hiprec.live_step(kind, xh, Ph, Q, 0.01, z, R, quat_idxs=[3], flags=3)
    amp += _amplification(P_prior, Ph)
    e.step_recorded(hist, kind, 0.01 * (k + 1), z, R)
    if k in (9, T - 1):
      _judge(f"stream step {k} x", e.state(), xo, xh)
      _judge(f"stream step {k} P", e.covs(), Po, Ph, cov=True, floor=np.maximum(FLOOR_P, 16 * EPS * amp))
  assert quat_norm_err(hist.x_filt.cpu().numpy(), [3]) <= 1e-15
  # RTS: all three smooth the SAME recorded history
  hx_p, hx_f = hist.x_pred.cpu().numpy(), hist.x_filt.cpu().numpy()
  hP_p, hP_f = hist.P_pred.cpu().numpy(), hist.P_filt.cpu().numpy()
  t = hist.t_host.copy()
  xs, Ps = e.rts_smooth(hist, norm_quats=True)
  xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
  ro = [rts_smooth(o, hx_p[:, b], hx_f[:, b], hP_p[:, b], hP_f[:, b], t, 23, 22, norm_quats=True) for b in range(B)]
  rh = [hiprec.live_rts(hx_p[:, b], hx_f[:, b], hP_p[:, b], hP_f[:, b], t, norm_quats=True) for b in range(B)]
  # the RTS gain solves with P_{k+1|k} (cond ~1e12 here): LDL^T and LU forward errors differ by more than 1e-12
  # (measured on an H100: 5.5e-12 for the kernel, 7.7e-13 for numpy on one gyro-bias component), so FLOOR_P applies
  _judge("rts x", xs, np.stack([r[0] for r in ro], 1), np.stack([r[0] for r in rh], 1), floor=FLOOR_P)
  _judge("rts P", Ps, np.stack([r[1] for r in ro], 1), np.stack([r[1] for r in rh], 1), cov=True, floor=FLOOR_P)
