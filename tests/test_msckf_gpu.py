"""GPU parity tests of the CTA-per-filter path (EDIM 82): synthetic MSCKF with 10 cloned poses, feature-track
updates with left-null-space projection and Mahalanobis gating, state augmentation."""
import numpy as np
import pytest
import torch

from tests.util import Oracle, cov_err, live_obs, msckf_batch, msckf_feature_obs, quat_norm_err, state_err

pytestmark = pytest.mark.gpu
QUATS = [3] + [23 + 3 + 7 * c for c in range(10)]   # the main attitude and the 10 clone attitudes
QN = 1e-15       # | |q| - 1 | after a normalising step: a few ulp


@pytest.fixture(scope="module")
def msckf_dirs(gen_dir, oracle_dir):
  import os
  from oracle import build_ref
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.msckf import MsckfKalman
  ensure_generated(MsckfKalman)
  if build_ref.reference_available():
    build_ref.build("msckf", "rednose_b200.filters.msckf:MsckfKalman")
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  return gen_dir, oracle_dir


def _engine(gen_dir, x, P, Q, **kw):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(gen_dir, "msckf", Q, x, P, quaternion_idxs=QUATS, **kw)


def test_msckf_predict_block_structure(msckf_dirs):
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  x, P, Q, _ = msckf_batch(37, seed=1)
  xr, Pr = o.predict(x, P, Q, 0.05)
  e = _engine(gen_dir, x, P, Q, norm_after_predict=False, norm_after_update=False)
  e.predict(0.05)
  assert state_err(e.state(), xr) < 1e-12 and cov_err(e.covs(), Pr) < 1e-9
  # clones are static: their block of P is untouched by the predict (ekf_c.c:23-26)
  assert np.array_equal(e.covs()[:, 22:, 22:], P[:, 22:, 22:])


def test_msckf_plain_kind_on_the_big_state(msckf_dirs):
  gen_dir, oracle_dir = msckf_dirs
  o, ol = Oracle(oracle_dir, "msckf"), Oracle(oracle_dir, "live")
  x, P, Q, _ = msckf_batch(41, seed=2)
  z, R = live_obs(ol, 12, x[:, :23])
  xr, Pr, yr = o.batch_step(12, x, P, Q, 0.01, z, R, quat_idxs=QUATS, flags=3)
  e = _engine(gen_dir, x, P, Q)
  y = e.step(12, 0.01, z, R)
  assert state_err(e.state(), xr) < 1e-9 and cov_err(e.covs(), Pr) < 1e-9 and state_err(y.cpu().numpy()[:, 0], yr) < 1e-9
  assert quat_norm_err(e.state(), QUATS) <= QN


@pytest.mark.parametrize("outlier_frac", [0.0, 0.3])
def test_msckf_feature_update_nullspace_and_gate(msckf_dirs, outlier_frac):
  """x and P are invariant to the null-space basis (ekf_c.c:71 fullPivLu().kernel() vs Householder here);
  the returned innovation is basis dependent and only its norm is compared."""
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  B = 48
  x, P, Q, point = msckf_batch(B, seed=3)
  z, R, out = msckf_feature_obs(o, x, point, seed=4, outlier_frac=outlier_frac)
  xr, Pr, yr = o.update(17, x, P, z, R, ea=point)
  e = _engine(gen_dir, x, P, Q, norm_after_update=False)
  y = e.update(17, z, R, ea=point).cpu().numpy()[:, 0]
  ex, eP = state_err(e.state(), xr), cov_err(e.covs(), Pr)
  assert ex < 1e-9 and eP < 1e-9, (ex, eP)
  if outlier_frac:
    # gated filters keep (essentially) their prior covariance; the others shrink it
    shrink = np.trace(e.covs(), axis1=1, axis2=2) / np.trace(P, axis1=1, axis2=2)
    gated = shrink > 1 - 1e-9
    assert gated.any() and (~gated).any() and np.all(out[gated])   # the gate fired, and only on gross outliers


def test_msckf_fused_step_with_feature_kind(msckf_dirs):
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  B = 33
  x, P, Q, point = msckf_batch(B, seed=5)
  xp, _ = o.predict(x, P, Q, 0.01)
  z, R, _ = msckf_feature_obs(o, xp, point, seed=6)
  xr, Pr, _ = o.batch_step(17, x, P, Q, 0.01, z, R, ea=point, quat_idxs=QUATS, flags=3)
  e = _engine(gen_dir, x, P, Q)
  e.step(17, 0.01, z, R, ea=point)
  ex, eP = state_err(e.state(), xr), cov_err(e.covs(), Pr)
  assert ex < 1e-9 and eP < 1e-9, (ex, eP)
  assert quat_norm_err(e.state(), QUATS) <= QN


def test_batched_augment_equals_reference_selection(msckf_dirs):
  """K3 vs the selection-matrix formulation of ekf_sym.py:365-391 written out in numpy."""
  gen_dir, _ = msckf_dirs
  x, P, Q, _ = msckf_batch(19, seed=7)
  e = _engine(gen_dir, x, P, Q)
  e.augment()
  d1, d2, d3, d4, n = 23, 22, 7, 6, 82
  xr = x.copy()
  xr[:, d1:-d3] = x[:, d1 + d3:]
  xr[:, -d3:] = x[:, :d3]
  to_mult = np.zeros((n, n - d4))
  to_mult[:-d4, :] = np.eye(n - d4)
  to_mult[-d4:, :d4] = np.eye(d4)
  Pr = np.stack([to_mult @ np.delete(np.delete(Pb, np.s_[d2:d2 + d4], axis=1), np.s_[d2:d2 + d4], axis=0) @ to_mult.T for Pb in P])
  assert np.array_equal(e.state(), xr) and np.array_equal(e.covs(), Pr)


def test_msckf_two_observations_per_predict_and_gather_list(msckf_dirs):
  """CTA path: n_obs = 2 (leaf + CTA kernels re-launched per observation) and the gather-list variant."""
  gen_dir, oracle_dir = msckf_dirs
  o, ol = Oracle(oracle_dir, "msckf"), Oracle(oracle_dir, "live")
  B = 21
  x, P, Q, _ = msckf_batch(B, seed=11)
  z1, R1 = live_obs(ol, 12, x[:, :23], seed=1)
  z2, R2 = live_obs(ol, 12, x[:, :23], seed=2)
  xr, Pr = o.predict(x, P, Q, 0.02)
  xr, Pr, _ = o.update(12, xr, Pr, z1, R1)
  xr, Pr, _ = o.update(12, xr, Pr, z2, R2)
  e = _engine(gen_dir, x, P, Q, norm_after_predict=False, norm_after_update=False)
  e.step(12, 0.02, np.stack([z1, z2], 1), np.stack([R1, R2], 1))
  assert state_err(e.state(), xr) < 1e-9 and cov_err(e.covs(), Pr) < 1e-9
  # gather list: only the odd filters step; the even ones must stay bit-identical
  e2 = _engine(gen_dir, x, P, Q)
  idx = torch.arange(1, B, 2, dtype=torch.int32, device="cuda")
  sel = idx.cpu().numpy()
  e2.step_indexed(12, idx, 0.02, z1[sel], R1[sel])
  xs, Ps, _ = o.batch_step(12, x[sel], P[sel], Q, 0.02, z1[sel], R1[sel], quat_idxs=QUATS, flags=3)
  got_x, got_P = e2.state(), e2.covs()
  assert state_err(got_x[sel], xs) < 1e-9 and cov_err(got_P[sel], Ps) < 1e-9
  assert quat_norm_err(got_x[sel], QUATS) <= QN
  keep = np.setdiff1d(np.arange(B), sel)
  assert np.array_equal(got_x[keep], x[keep]) and np.array_equal(got_P[keep], P[keep])


def test_msckf_he_leaf_matches_reference_generated_c(msckf_dirs):
  """The exported He_<kind> leaf (d h / d point, ekf_sym.py:86-87) against the reference generator's own C."""
  from rednose_b200.ekf_sym import EKF_sym
  from rednose_b200.filters.msckf import MsckfKalman
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  x, P, Q, point = msckf_batch(5, seed=21)
  kf = EKF_sym(gen_dir, "msckf", Q, x[0], P[0], 23, 22, N=10, dim_augment=7, dim_augment_err=6, maha_test_kinds=[17], quaternion_idxs=QUATS)
  for b in range(5):
    want, got = np.zeros(60), np.zeros(60)
    o.leaf("He_17", np.ascontiguousarray(x[b]), np.ascontiguousarray(point[b]), want)
    kf.Hes[17](np.ascontiguousarray(x[b]), np.ascontiguousarray(point[b]), got)
    assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))


def test_msckf_projected_innovation_is_pinned_basis_invariantly(msckf_dirs):
  """The innovation returned by a feature kind is expressed in a basis of the left null space of He (Eigen's
  fullPivLu().kernel() in the reference, ekf_c.c:71; orthonormal Householder columns here), so its entries differ;
  its length does not: for an orthonormal basis A, |A^T y|^2 = |(I - He He^+) y|^2, computed here from the reference
  generator's own h_17 / He_17."""
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  B = 64
  x, P, Q, point = msckf_batch(B, seed=23)
  z, R, _ = msckf_feature_obs(o, x, point, seed=24, sigma=2e-3)
  e = _engine(gen_dir, x, P, Q, norm_after_update=False)
  y = e.update(17, z, R, ea=point).cpu().numpy()[:, 0]
  for b in range(B):
    hx, He = np.zeros(20), np.zeros(60)
    o.leaf("h_17", np.ascontiguousarray(x[b]), np.ascontiguousarray(point[b]), hx)
    o.leaf("He_17", np.ascontiguousarray(x[b]), np.ascontiguousarray(point[b]), He)
    He = He.reshape(20, 3)
    yr = z[b] - hx
    proj = yr - He @ np.linalg.lstsq(He, yr, rcond=None)[0]
    assert abs(np.linalg.norm(y[b, :17]) - np.linalg.norm(proj)) <= 1e-9 * np.linalg.norm(proj)


def test_msckf_baseline_size_10k_gate_fires_on_the_oracle_set(msckf_dirs):
  """BASELINE.json config 5 at size: 10 000 filters, 5 % gross outliers (x50 noise), fused predict + gated feature
  update + augment.  Every filter is compared with the oracle (16 host threads' worth of work: a few seconds); the set
  of gated filters -- read off the covariance, which a gated update leaves essentially untouched -- must be the oracle's."""
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  B = 10_000
  x, P, Q, point = msckf_batch(B, seed=31)
  xp, Pp = o.predict(x[:256], P[:256], Q, 0.01)
  z, R, out = msckf_feature_obs(o, x, point, seed=32, sigma=1e-3, outlier_frac=0.05)
  xr, Pr, _ = o.batch_step(17, x, P, Q, 0.01, z, R, ea=point, quat_idxs=QUATS, flags=3)
  e = _engine(gen_dir, x, P, Q)
  e.step(17, 0.01, z, R, ea=point)
  gx, gP = e.state(), e.covs()
  # per component over all 10 000 filters, and per filter for the covariance (correlation units)
  ex, eP = state_err(gx, xr), cov_err(gP, Pr)
  assert ex < 1e-9 and eP < 1e-9, (ex, eP)
  assert quat_norm_err(gx, QUATS) <= QN
  tr = lambda A: np.trace(A[:, 22:, 22:], axis1=1, axis2=2)
  o_gated = tr(Pr) > tr(P) * (1 - 1e-9)          # clone block untouched (the predict does not change it, ekf_c.c:23-26)
  g_gated = tr(gP) > tr(P) * (1 - 1e-9)
  assert np.array_equal(o_gated, g_gated) and 100 < o_gated.sum() < 1500 and np.all(out[o_gated])
  e.augment()
  assert np.array_equal(e.covs()[:, -6:, -6:], gP[:, :6, :6])   # the new clone is the main pose (ekf_sym.py:384-389)


def test_msckf_feature_kind_single_filter_host_entry_point(msckf_dirs):
  """Single-filter host-pointer entry point <name>_update_<feature kind> (B = 1 launch of the CTA kernel, the only
  kernel with the He projection: feature kinds are routed there whatever EDIM is, ekf_abi.cuh launch_step)."""
  from rednose_b200.ekf_sym import EKF_sym
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  x, P, Q, point = msckf_batch(3, seed=41)
  z, R, _ = msckf_feature_obs(o, x, point, seed=42)
  xr, Pr, _ = o.update(17, x, P, z, R, ea=point)
  for b in range(3):
    kf = EKF_sym(gen_dir, "msckf", Q, x[b], P[b], 23, 22, N=10, dim_augment=7, dim_augment_err=6, maha_test_kinds=[17], quaternion_idxs=QUATS)
    xb, Pb, zb = x[b].copy(), P[b].copy(), z[b].copy()
    kf._update(xb, Pb, 17, zb, np.ascontiguousarray(R[b]), np.ascontiguousarray(point[b]))
    assert state_err(xb, xr[b]) < 1e-9 and cov_err(Pb, Pr[b]) < 1e-9


def test_msckf_fused_augment_equals_step_then_augment(msckf_dirs):
  """predict_and_update_batch(..., augment=True) (ekf_sym.py:527-528): the clone-window shift done inside the CTA kernel's
  write-back is the same permutation as the separate <name>_batch_augment launch, bit for bit; the history slabs keep the
  estimate from before the shift."""
  gen_dir, oracle_dir = msckf_dirs
  o = Oracle(oracle_dir, "msckf")
  B = 37
  x, P, Q, point = msckf_batch(B, seed=51)
  z, R, _ = msckf_feature_obs(o, x, point, seed=52, outlier_frac=0.2)
  e1, e2 = _engine(gen_dir, x, P, Q), _engine(gen_dir, x, P, Q)
  hx, hP = torch.empty(B, 93, dtype=torch.float64, device="cuda"), torch.empty(B, 82, 82, dtype=torch.float64, device="cuda")
  e1.step(17, 0.01, z, R, ea=point)
  pre_x, pre_P = e1.state().copy(), e1.covs().copy()
  e1.augment()
  e2.step(17, 0.01, z, R, ea=point, augment=True, hist_filt=(hx, hP))
  assert np.array_equal(e2.state(), e1.state()) and np.array_equal(e2.covs(), e1.covs())
  assert np.array_equal(hx.cpu().numpy(), pre_x) and np.array_equal(hP.cpu().numpy(), pre_P)
  # a plain kind on the big state, two observations per predict: the shift happens once, after the last one
  ol = Oracle(oracle_dir, "live")
  z1, R1 = live_obs(ol, 12, x[:, :23], seed=1)
  z2, R2 = live_obs(ol, 12, x[:, :23], seed=2)
  e3, e4 = _engine(gen_dir, x, P, Q), _engine(gen_dir, x, P, Q)
  e3.step(12, 0.02, np.stack([z1, z2], 1), np.stack([R1, R2], 1)); e3.augment()
  e4.step(12, 0.02, np.stack([z1, z2], 1), np.stack([R1, R2], 1), augment=True)
  assert np.array_equal(e4.state(), e3.state()) and np.array_equal(e4.covs(), e3.covs())


def test_more_quaternions_than_supported_raise(msckf_dirs):
  """A quaternion list the kernels cannot honour (17 > MAX_QUAT, or an index past the state) is refused before any
  launch and BatchedEKF raises; the state is left untouched."""
  gen_dir, _ = msckf_dirs
  x, P, Q, _ = msckf_batch(3, seed=61)
  for quats in (QUATS + [23 + 7 * c for c in range(6)], [3, 90]):
    from rednose_b200.batched import BatchedEKF
    e = BatchedEKF(gen_dir, "msckf", Q, x, P, quaternion_idxs=quats)
    with pytest.raises(RuntimeError, match="CUDA error 1 "):
      e.predict(0.01)
    assert np.array_equal(e.state(), x) and np.array_equal(e.covs(), P)
