"""CPU tests of the drop-in surface: filter scripts written against the reference's surface generate and run through this
package.  The reference's UNMODIFIED example scripts import `rednose.helpers.*`, which this repository provides as a
shim over rednose_b200; what they generate through it is stored in tests/golden/dropin_reference.json (written by
tests/golden/make_golden_support.py) and compared here with what this repository's own filter scripts generate.
Running goes through this package's EKF_sym_pyx (native driver) -- pointed at the oracle's CPU build of the same C-ABI,
since there is no GPU here."""
import hashlib
import json
import os
import re
import runpy
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FILTERS = os.path.join(os.path.dirname(HERE), "rednose_b200", "filters")
with open(os.path.join(HERE, "golden", "dropin_reference.json"), encoding="utf-8") as _f:
  GOLDEN_GEN = json.load(_f)


def _protos_sha256(path):
  with open(path, encoding="utf-8") as f:
    protos = sorted(re.sub(r"\s+", " ", ln) for ln in f.read().split("\n") if ln.startswith("void "))
  return hashlib.sha256("\n".join(protos).encode()).hexdigest()


def _sig(path):
  with open(path, encoding="utf-8") as f:
    return re.findall(r"static constexpr int (?:NF|KIND) = [^;]*;", f.read())


@pytest.mark.parametrize("script,name", [("kinematic_kf.py", "kinematic"), ("live_kf.py", "live")])
def test_reference_generator_scripts_run_unchanged(tmp_path, monkeypatch, gen_dir, script, name):
  """`python <filter>.py <target> <output_dir>` (site_scons/site_tools/rednose_filter.py:13) through this package
  generates what the reference's examples/<script> generates through it (stored in GOLDEN_GEN[name])."""
  import rednose
  assert "rednose_b200" in open(os.path.join(os.path.dirname(rednose.__file__), "helpers", "ekf_sym.py")).read()
  monkeypatch.setenv("REDNOSE_B200_NO_COMPILE", "1")
  monkeypatch.setattr(sys, "argv", [f"{name}.py", name, str(tmp_path)])
  runpy.run_path(os.path.join(FILTERS, f"{name}.py"), run_name="__main__")
  assert os.path.exists(tmp_path / f"{name}.cu") and os.path.exists(tmp_path / f"{name}.h")
  for d in (str(tmp_path), gen_dir):
    # same C-ABI as the reference's example script generates
    assert _protos_sha256(os.path.join(d, f"{name}.h")) == GOLDEN_GEN[name]["protos_sha256"]
    # same structure: the sparsity signature of F / H_err survives (33 F slots, per-kind non-zeros)
    assert _sig(os.path.join(d, f"{name}.cu")) == GOLDEN_GEN[name]["sig"]


def test_reference_kinematic_example_on_the_dropin_driver(oracle_dir):
  """examples/test_kinematic_kf.py:10-55 with this package's KinematicKalman (the example's model on the KalmanFilter
  surface); GOLDEN are the reference test's own expected values."""
  from rednose_b200.filters import kinematic as mod
  from tests.test_oracle_cpu import GOLDEN
  np.random.seed(0)
  kf = mod.KinematicKalman(oracle_dir)
  assert type(kf.filter).__module__ == "rednose_b200.ekf_sym_pyx"
  dt = 0.01
  ts = np.arange(0, 5, step=dt)
  x = 0.0
  for t, v in zip(ts, np.sin(ts * 5)):
    kf.predict_and_observe(t, mod.ObservationKind.POSITION, [np.random.normal(x, 0.1)])
    x += v * dt
  got = (kf.x[0], np.sqrt(kf.P[0, 0]), kf.x[1], np.sqrt(kf.P[1, 1]))
  for g, want in zip(got, GOLDEN):
    assert abs(g - want) < 5e-8


def test_reference_live_example_on_the_dropin_driver(oracle_dir):
  """The usage of examples/live_kf.py's LiveKalman (live_kf.py:269-306) on this package's LiveKalman: the quaternion
  normalisation written through the filter's live (DIM, 1) view, .t, rts_smooth."""
  from rednose_b200.filters import live as mod
  K = mod.ObservationKind
  kf = mod.LiveKalman(oracle_dir)
  rng = np.random.default_rng(0)
  estimates = []
  t = 0.0
  for k in range(30):
    t += 0.01
    if k % 10 == 0:
      r = kf.predict_and_observe(t, K.ECEF_POS, [kf.x[:3] + rng.normal(0, 1.0, 3)])
    elif k % 10 == 5:
      r = kf.predict_and_observe(t, K.CAMERA_ODO_TRANSLATION, [np.concatenate([rng.normal(0, 0.1, 3), [0.1, 0.1, 0.1]])])
    elif k % 10 == 7:
      r = kf.predict_and_observe(t, K.ODOMETRIC_SPEED, [[0.0]])
    else:
      r = kf.predict_and_observe(t, K.PHONE_GYRO, [rng.normal(0, 0.01, 3)])
    assert r is not None
    estimates.append(r)
    assert abs(np.linalg.norm(kf.x[3:7]) - 1.0) < 1e-12   # the example's own normalisation wrote through .x
    assert abs(kf.t - t) < 1e-12
  xs, Ps = kf.rts_smooth(estimates)
  assert xs.shape == (30, 23) and Ps.shape == (30, 22, 22) and np.isfinite(xs).all() and np.isfinite(Ps).all()
  assert Ps[10, 0, 0] <= estimates[10][3][0, 0] * (1 + 1e-9)
