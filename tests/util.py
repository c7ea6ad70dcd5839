"""Shared helpers for the parity tests: oracle access (test infrastructure) and synthetic inputs."""

import numpy as np

from oracle.handle import Oracle  # noqa: F401

LIVE_KINDS = {3: 1, 4: 3, 9: 3, 10: 3, 12: 3, 13: 3, 14: 3, 19: 3}  # kind -> ZDIM (gen/live.cpp:1780-1802)
LIVE_R = {3: [0.2**2], 4: [0.025**2] * 3, 9: [0.00025**2] * 3, 10: [0.5**2] * 3, 12: [5.0**2] * 3,
          13: [0.1**2] * 3, 14: [0.05**2] * 3, 19: [0.05**2] * 3}


def state_err(got, want, per_component=False):
  """Worst per-component relative error of states / innovations / history slabs [..., n].

  For every last-axis component i: max |got - want| over all leading axes, divided by max |want[..., i]| over the
  same axes (absolute where the reference component is identically zero).  A 4e6 m position no longer sets the scale
  of a unit quaternion or a 1e-2 accelerometer bias.  per_component=True returns the [n] vector instead of its max."""
  got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
  assert got.shape == want.shape, (got.shape, want.shape)
  n = want.shape[-1] if want.ndim else 1
  d = np.abs(got - want).reshape(-1, n).max(axis=0)
  s = np.abs(want).reshape(-1, n).max(axis=0)
  e = np.where(s > 0, d / np.where(s > 0, s, 1.0), d)
  return e if per_component else float(np.max(e))


def cov_err(got, want, per_component=False):
  """Worst covariance error in correlation units: max |got_ij - want_ij| / sqrt(want_ii want_jj) per matrix [..., n, n].

  Invariant under a rescaling of the state units (D P D for a positive diagonal D), so a 1e-4 variance block is held
  to the same standard as the 1e8 position block.  per_component=True returns the [n, n] maximum over the leading axes."""
  got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
  assert got.shape == want.shape and want.shape[-1] == want.shape[-2], (got.shape, want.shape)
  dg = np.diagonal(want, axis1=-2, axis2=-1)
  assert np.all(dg > 0), "reference covariance has a non-positive diagonal entry"
  sd = np.sqrt(dg)
  e = np.abs(got - want) / (sd[..., :, None] * sd[..., None, :])
  n = want.shape[-1]
  return e.reshape(-1, n, n).max(axis=0) if per_component else float(np.max(e))


def quat_norm_err(x, idxs):
  """max | |q| - 1 | over every quaternion x[..., i:i + 4], i in idxs, and every filter / step."""
  x = np.asarray(x, dtype=np.float64)
  return float(max(np.max(np.abs(np.linalg.norm(x[..., i:i + 4], axis=-1) - 1.0)) for i in idxs))


def live_batch(B, seed=0, well_conditioned=True):
  """Random but physically plausible live_kf states / covariances (SURVEY.md section 8d, config 3)."""
  from rednose_b200.filters.live import LiveKalman
  rng = np.random.default_rng(seed)
  x = np.tile(LiveKalman.initial_x, (B, 1))
  x[:, 0:3] += rng.normal(0, 100.0, (B, 3))
  q = rng.normal(size=(B, 4))
  x[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
  x[:, 7:10] = rng.normal(0, 5.0, (B, 3))
  x[:, 10:13] = rng.normal(0, 0.1, (B, 3))
  x[:, 13:16] = rng.normal(0, 0.01, (B, 3))
  x[:, 16] = 1.0 + rng.normal(0, 0.01, B)
  x[:, 17:20] = rng.normal(0, 1.0, (B, 3))
  x[:, 20:23] = rng.normal(0, 0.01, (B, 3))
  if well_conditioned:
    s = np.sqrt(np.array([25.0] * 3 + [0.05**2] * 3 + [1.0] * 3 + [0.1**2] * 3 + [0.01**2] * 3 + [0.01**2] + [0.5**2] * 3 + [0.01**2] * 3))
  else:
    s = np.sqrt(LiveKalman.initial_P_diag)
  L = np.eye(22)[None] + 0.2 * np.tril(rng.normal(size=(B, 22, 22)), -1)
  L = s[None, :, None] * L
  P = L @ np.transpose(L, (0, 2, 1))
  P = 0.5 * (P + np.transpose(P, (0, 2, 1)))
  return x, P, LiveKalman.Q.copy()


def live_obs(oracle, kind, x, seed=1, noise_scale=1.0):
  """z = h_kind(x) + N(0, R) with the default R of the kind; uses the oracle's leaf h (reference-generated C)."""
  rng = np.random.default_rng(seed + kind)
  m = LIVE_KINDS[kind]
  B = x.shape[0]
  R = np.tile(np.diag(LIVE_R[kind]), (B, 1, 1))
  z = np.zeros((B, m))
  dummy = np.zeros(1)
  for b in range(B):
    oracle.leaf(f"h_{kind}", np.ascontiguousarray(x[b]), dummy, z[b])
  z += noise_scale * rng.normal(size=(B, m)) * np.sqrt(np.array(LIVE_R[kind]))[None, :]
  return z, R


def kinematic_batch(B, seed=0):
  from rednose_b200.filters.kinematic import KinematicKalman
  rng = np.random.default_rng(seed)
  x = np.tile(KinematicKalman.initial_x, (B, 1)) + rng.normal(size=(B, 2))
  L = np.eye(2)[None] + 0.3 * np.tril(rng.normal(size=(B, 2, 2)), -1)
  P = L @ np.transpose(L, (0, 2, 1))
  z = x[:, :1] + rng.normal(0, 0.1, (B, 1))
  R = np.tile(np.array([[0.1**2]]), (B, 1, 1))
  return x, P, KinematicKalman.Q.copy(), z, R


def msckf_batch(B, seed=0, outlier_frac=0.0):
  """Synthetic MSCKF states: live main state, 10 clones = the main pose displaced along a short track,
  one 3-D point 10-50 m ahead seen from every clone (SURVEY.md section 8d, config 5)."""
  from rednose_b200.filters.msckf import DIM, DIM_AUGMENT, EDIM, N_CLONES, MsckfKalman
  from rednose_b200.filters.live import DIM_STATE
  from rednose_b200.geometry import quat2rot
  rng = np.random.default_rng(seed)
  xm, _, _ = live_batch(B, seed=seed)
  x = np.zeros((B, DIM))
  x[:, :DIM_STATE] = xm
  Rm = quat2rot(xm[:, 3:7])                       # device -> ecef
  fwd = Rm[:, :, 0]
  for c in range(N_CLONES):
    o = DIM_STATE + c * DIM_AUGMENT
    x[:, o:o + 3] = xm[:, 0:3] - fwd * 0.5 * (N_CLONES - c) + rng.normal(0, 0.02, (B, 3))
    q = xm[:, 3:7] + rng.normal(0, 0.002, (B, 4))
    x[:, o + 3:o + 7] = q / np.linalg.norm(q, axis=1, keepdims=True)
  s = np.sqrt(np.concatenate([[25.0] * 3 + [0.05**2] * 3 + [1.0] * 3 + [0.1**2] * 3 + [0.01**2] * 3 + [0.01**2] + [0.5**2] * 3 + [0.01**2] * 3]
                             + [[1.0] * 3 + [0.02**2] * 3] * N_CLONES))
  L = np.eye(EDIM)[None] + 0.05 * np.tril(rng.normal(size=(B, EDIM, EDIM)), -1)
  L = s[None, :, None] * L
  P = L @ np.transpose(L, (0, 2, 1))
  P = 0.5 * (P + np.transpose(P, (0, 2, 1)))
  local = np.stack([rng.uniform(10, 50, B), rng.uniform(-5, 5, B), rng.uniform(-3, 3, B)], 1)
  point = xm[:, 0:3] + np.einsum('bij,bj->bi', Rm, local)
  return x, P, MsckfKalman.Q.copy(), point


def msckf_feature_obs(oracle, x, point, seed=1, sigma=1e-3, outlier_frac=0.0):
  rng = np.random.default_rng(seed)
  B = x.shape[0]
  z = np.zeros((B, 20))
  for b in range(B):
    oracle.leaf("h_17", np.ascontiguousarray(x[b]), np.ascontiguousarray(point[b]), z[b])
  noise = rng.normal(0, sigma, (B, 20))
  out = rng.random(B) < outlier_frac
  noise[out] *= 50.0
  R = np.tile(np.eye(20) * sigma**2, (B, 1, 1))
  return z + noise, R, out
