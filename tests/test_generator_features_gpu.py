"""GPU parity for generator features the shipped examples do not exercise: global_vars / <name>_set_<var>,
extra_routines, a gated kind with extra arguments (thread-per-filter kernel, EDIM 3)."""
import os

import numpy as np
import pytest

from tests.util import Oracle, cov_err, state_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dirs(gen_dir, oracle_dir):
  from oracle import build_ref
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.pendulum import PendulumKalman
  ensure_generated(PendulumKalman)
  if build_ref.reference_available():
    build_ref.build("pendulum", "rednose_b200.filters.pendulum:PendulumKalman")
  if not os.path.exists(os.path.join(build_ref.OUT, "libpendulum.so")):
    pytest.skip("oracle/_ref/libpendulum.so not built")
  return gen_dir, oracle_dir


def _batch(B, seed):
  rng = np.random.default_rng(seed)
  x = np.stack([rng.uniform(-1, 1, B), rng.normal(0, 0.5, B), rng.normal(0, 0.02, B)], 1)
  L = np.eye(3)[None] + 0.3 * np.tril(rng.normal(size=(B, 3, 3)), -1)
  L = np.array([0.1, 0.5, 0.05])[None, :, None] * L
  P = L @ np.transpose(L, (0, 2, 1))
  return x, 0.5 * (P + np.transpose(P, (0, 2, 1)))


def test_global_vars_extra_routine_and_gated_kind(dirs):
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.ekf_sym_pyx import EKF_sym_pyx
  from rednose_b200.filters.pendulum import PendulumKalman as F
  gen_dir, oracle_dir = dirs
  o = Oracle(oracle_dir, "pendulum")
  B = 5003
  x, P = _batch(B, 1)
  for grav, damp in ((9.81, 0.1), (1.62, 0.0)):
    o.lib.pendulum_set_grav(grav); o.lib.pendulum_set_damp(damp)
    e = BatchedEKF(gen_dir, "pendulum", F.Q, x, P, global_vars={"grav": grav, "damp": damp})
    # kind 1 (m = 1), fused step
    rng = np.random.default_rng(2)
    z1 = (x[:, 0] + x[:, 2])[:, None] + rng.normal(0, 0.01, (B, 1))
    R1 = np.tile(np.array([[1e-4]]), (B, 1, 1))
    xr, Pr, yr = o.batch_step(1, x, P, F.Q, 0.02, z1, R1)
    y = e.step(1, 0.02, z1, R1)
    assert state_err(e.state(), xr) < 1e-12 and cov_err(e.covs(), Pr) < 1e-10 and state_err(y.cpu().numpy()[:, 0], yr) < 1e-10
    # kind 2 (m = 2, extra args, Mahalanobis gated) with 20 % gross outliers
    pivot = rng.normal(0, 1.0, (B, 2))
    x2 = e.state()
    h = np.stack([pivot[:, 0] + F.LENGTH * np.sin(x2[:, 0]), pivot[:, 1] - F.LENGTH * np.cos(x2[:, 0])], 1)
    noise = rng.normal(0, 0.01, (B, 2))
    out = rng.random(B) < 0.2
    noise[out] += 5.0
    z2, R2 = h + noise, np.tile(np.eye(2) * 1e-4, (B, 1, 1))
    xr2, Pr2, yr2 = o.update(2, xr, Pr, z2, R2, ea=pivot)
    y2 = e.update(2, z2, R2, ea=pivot)
    assert state_err(e.state(), xr2) < 1e-10 and cov_err(e.covs(), Pr2) < 1e-9 and state_err(y2.cpu().numpy()[:, 0], yr2) < 1e-10
    gated = np.trace(e.covs(), axis1=1, axis2=2) > np.trace(Pr, axis1=1, axis2=2) * (1 - 1e-9)
    assert gated[out].all() and gated[~out].mean() < 0.15   # gross outliers always gated; ~5 % false positives at the 0.95 quantile
  # extra routine + set_global through the drop-in driver
  kf = EKF_sym_pyx(gen_dir, "pendulum", F.Q, F.initial_x, np.diag(F.initial_P_diag), 3, 3, global_vars=["grav", "damp"])
  kf.set_global("grav", 9.81)
  xs = np.ascontiguousarray(x[0])
  got, want = np.zeros(1), np.zeros(1)
  ffi, lib = kf._ffi, kf._lib
  lib.pendulum_energy(ffi.cast("double *", xs.ctypes.data), ffi.cast("double *", got.ctypes.data))
  o.lib.pendulum_set_grav(9.81)
  o.leaf("energy", xs, want)
  assert abs(got[0] - want[0]) < 1e-14 * max(1.0, abs(want[0])) and got[0] != 0.0
  with pytest.raises(KeyError):
    kf.set_global("nope", 1.0)
