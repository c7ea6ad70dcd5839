"""The synthetic shape filters (tests/shapes.py) without a GPU: every one generates and cross-compiles for sm_90a, reports
the dispatch facts of its shape, and its 40-digit reference (tests/hiprec.py) is itself right.  A model whose main error
block is larger than the kernels serve is refused by gen_code before nvcc runs."""
import os

import numpy as np
import pytest

from tests import hiprec
from tests.shapes import SHAPES, batch, observe, synthetic_model
from tests.util import cov_err, state_err

IDS = [c.name for c in SHAPES]


def _load(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_shape_library_builds(cls):
  ffi, lib = _load(cls)
  kinds = sorted(int(s.rsplit("_", 1)[1]) for s in dir(lib) if s.startswith(f"{cls.name}_batch_step_") and not s.endswith("_idx"))
  assert kinds == sorted(cls.kinds())
  assert hasattr(lib, f"{cls.name}_batch_rts")
  for g in cls.global_names():
    assert hasattr(lib, f"{cls.name}_set_{g}")


def test_main_block_above_32_is_refused_before_nvcc(tmp_path):
  from rednose_b200.codegen import gen_code
  with pytest.raises(ValueError, match="main error block of 33 states.*at most 32"):
    gen_code(str(tmp_path), "shape_e33", **synthetic_model(33, zdims=(1, 3)), compile_lib=True)
  assert os.listdir(tmp_path) == []                 # nothing generated, nvcc never ran


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_dispatch_facts(cls):
  _, lib = _load(cls)
  E = cls.edim
  want = 4 * (E // 2) * (E // 2 + 1) // 2 if cls.step_kernel() == "pair" else 0
  assert getattr(lib, f"{cls.name}_packed_P_doubles")() == want


def _fd(fun, x0, h=1e-6):
  x0 = np.asarray(x0, dtype=np.float64)
  cols = []
  for i in range(x0.shape[0]):
    e = np.zeros_like(x0)
    e[i] = h
    cols.append((fun(x0 + e) - fun(x0 - e)) / (2 * h))
  return np.stack(cols, 1)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_reference_jacobians_match_finite_differences(cls):
  """F = d f_err / d x_err and H, H H_mod as the reference derives them, against central differences of the leaf
  functions: F of the exact error map inv_err(f(x), f(x [+] d)) (x [-] x and x [+] 0 are exact for a unit quaternion)."""
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  x, _, _, dt = batch(cls, 3, seed=1)
  E, D = cls.edim, cls.dim()
  for b in range(3):
    fx = m.np_leaf('f', x[b], dt[b])
    F = m.np_leaf('F', x[b], dt[b]).reshape(E, E)
    Fd = _fd(lambda d: m.np_leaf('inv_err', fx, m.np_leaf('f', m.np_leaf('err', x[b], d), dt[b])), np.zeros(E))
    assert np.max(np.abs(F - Fd)) < 1e-8 * max(1.0, np.max(np.abs(F))), (b, np.max(np.abs(F - Fd)))
    Hm = m.np_leaf('H_mod', x[b]).reshape(D, E)
    rng = np.random.default_rng(b)
    for kind, (Z, EA, _) in cls.kinds().items():
      ea = [rng.normal(size=EA)] if EA else []
      H = m.np_leaf(('H', kind), x[b], *ea).reshape(Z, D)
      Hd = _fd(lambda v: m.np_leaf(('h', kind), v, *ea), x[b])
      assert np.max(np.abs(H - Hd)) < 1e-8 * max(1.0, np.max(np.abs(H))), (kind, np.max(np.abs(H - Hd)))
      He = _fd(lambda d: m.np_leaf(('h', kind), m.np_leaf('err', x[b], d), *ea), np.zeros(E))
      assert np.max(np.abs(H @ Hm - He)) < 1e-8 * max(1.0, np.max(np.abs(He))), (kind, np.max(np.abs(H @ Hm - He)))


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_reference_step_agrees_with_a_float64_step(cls):
  """On well-conditioned inputs the 40-digit step and a plain float64 step from the same leaf functions agree to 1e-12
  (so neither the reference's algebra nor its lambdified leaves can be off by more than float64 rounding)."""
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  x, P, Q, dt = batch(cls, 2, seed=2)
  q = cls.quat_idxs()
  for kind in cls.kinds():
    z, R, ea = observe(cls, m, kind, x, seed=3)
    xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=q, gate=False)
    for b in range(2):
      xf, Pf, yf = m.step_f64(kind, x[b], P[b], Q, dt[b], z[b], R[b], quat_idxs=q, ea=None if ea is None else ea[b])
      # innovations as the predicted observation z - y: y itself cancels to ~1e-5 of z in some components
      ex, ey = state_err(xf, xr[b]), state_err(z[b] - yf, z[b] - yr[b])
      assert ex < 1e-12 and ey < 1e-12, (kind, ex, ey)
      assert cov_err(Pf, Pr[b]) < 1e-12, (kind, cov_err(Pf, Pr[b]))
