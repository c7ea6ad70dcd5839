"""CPU tests: the ORACLE (restated ekf_c.c + reference-generated leaf C, and the restated RTS) against
golden vectors produced by the reference's own Python maths (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from tests.util import LIVE_KINDS, Oracle, cov_err, quat_norm_err, state_err

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference.npz")


@pytest.fixture(scope="module")
def gold():
  return np.load(GOLD)


def test_oracle_matches_reference_python_maths_on_live(oracle_dir, gold):
  """Forward filter, 40 steps over all 8 kinds: restated C core == reference numpy predict/update."""
  o = Oracle(oracle_dir, "live")
  Q, kinds, ts = gold["Q"], gold["kinds"], gold["t"]
  x, P = gold["x0"].copy(), gold["P0"].copy()
  t_prev = ts[0]
  for k, kind in enumerate(kinds):
    m = LIVE_KINDS[int(kind)]
    z = np.stack([gold[f"z{b}"][k, :m] for b in range(2)])
    R = np.stack([gold[f"R{b}"][k, :m, :m] for b in range(2)])
    # python-driver semantics (ekf_sym.py:505-522): predict, update, then normalise
    x, P, y = o.batch_step(int(kind), x, P, Q, ts[k] - t_prev, z, R, quat_idxs=[3], flags=2, nthreads=1)
    t_prev = ts[k]
    ex = state_err(x, np.stack([gold[f"x_filt{b}"][k] for b in range(2)]))
    eP = cov_err(P, np.stack([gold[f"P_filt{b}"][k] for b in range(2)]))
    ey = state_err(y, np.stack([gold[f"y{b}"][k, :m] for b in range(2)]))
    assert ex < 1e-10 and eP < 1e-9 and ey < 1e-7, (k, kind, ex, eP, ey)
    assert quat_norm_err(x, [3]) <= 1e-15


def test_restated_rts_matches_reference_rts(oracle_dir, gold):
  from oracle.rts_numpy import rts_smooth
  o = Oracle(oracle_dir, "live")
  for b in range(2):
    xs, Ps = rts_smooth(o, gold[f"x_pred{b}"], gold[f"x_filt{b}"], gold[f"P_pred{b}"], gold[f"P_filt{b}"], gold["t"], 23, 22, norm_quats=True)
    assert state_err(xs, gold[f"xs{b}"]) < 1e-12 and cov_err(Ps, gold[f"Ps{b}"]) < 1e-12


def _msckf_gold():
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "msckf_reference.npz"))


def test_oracle_matches_reference_python_maths_on_msckf(oracle_dir):
  """MSCKF pieces: block predict, feature update through the left-null-space projection (reference numpy: SVD null(),
  oracle: restated fullPivLu().kernel(), ekf_c.c:66-76) with the Mahalanobis gate armed, augment.  x and P are
  basis-invariant and must agree at every step (tests/golden/make_golden_msckf.py)."""
  if not os.path.exists(os.path.join(oracle_dir, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  from rednose_b200.ekf_sym import EKF_sym
  from rednose_b200.filters.live import DIM_STATE, DIM_STATE_ERR
  from rednose_b200.filters.msckf import DIM_AUGMENT, DIM_AUGMENT_ERR, N_CLONES, MsckfKalman
  g = _msckf_gold()
  feat = int(MsckfKalman.feature_kind)
  quats = [3] + [DIM_STATE + 3 + 7 * c for c in range(N_CLONES)]
  for b in range(2):
    kf = EKF_sym(oracle_dir, "msckf", g["Q"], g["x0"][b], g["P0"][b], DIM_STATE, DIM_STATE_ERR, N=N_CLONES, dim_augment=DIM_AUGMENT,
                 dim_augment_err=DIM_AUGMENT_ERR, maha_test_kinds=[feat], quaternion_idxs=quats)
    for k, kind in enumerate(g["kinds"]):
      kind = int(kind)
      m = 2 * N_CLONES if kind == feat else 3
      z, R = g[f"z{b}"][k, :m], np.diag(g[f"Rdiag{b}"][k, :m])
      r = kf.predict_and_update_batch(float(g["t"][k]), kind, z[None], R[None], extra_args=[g["point"][b]] if kind == feat else [[]],
                                      augment=bool(g["augment"][k]))
      assert r is not None
      ex, eP = state_err(kf.state(), g[f"xk{b}"][k]), cov_err(kf.covs(), g[f"Pk{b}"][k])
      assert ex < 1e-10 and eP < 1e-8, (b, k, kind, ex, eP)
      assert quat_norm_err(kf.state(), quats) <= 1e-15, (b, k)
