"""The CTA-per-filter path (ekf_leaf_thread + ekf_step_cta, the augment kernels, ekf_maha_thread above EDIM 32) at every
MSCKF shape it claims to serve (tests/msckf_shapes.py), against the 40-digit reference of tests/hiprec.py.

Each shape runs B = 70 filters, so the leaf kernel (64 filters per block) has two blocks; the reference is evaluated on
the first and last filter and on both sides of the leaf block boundary (63, 64), and on every planted outlier.  x is
compared per component and P in correlation units, at TIGHT = 1e-9.  A feature kind's innovation is expressed in a basis
of the left null space of He that the kernel and the reference choose differently, so it is compared by its norm; plain
kinds compare the predicted observation z - y.  After a normalising step every listed quaternion is within 1e-15 of unit
norm.

Worst values measured on one H100 80GB HBM3 (power limit 700 W) over all eight shapes, all against TIGHT; the
innovation column is relative, of |y| for a feature kind and per component of z - y otherwise:

| check | state | covariance | innovation |
|---|---|---|---|
| fused step, every kind | 3.1e-15 | 1.7e-14 | 2.5e-15 |
| predict / update / two observations | 2.8e-14 | 2.7e-14 | 6.8e-15 |
| step_indexed | 2.9e-15 | 1.2e-14 | 4.3e-14 |
| gated kind with outliers | 7.4e-16 | 2.0e-14 | 3.1e-15 |
| second global values | 1.1e-15 | 2.4e-15 | 2.4e-16 |
| host entry point, feature kind | 5.9e-16 | 7.7e-15 | |
| Mahalanobis distance, relative | 1.0e-14 | | |

The file takes about six minutes, nearly all of it the 40-digit reference on the host (EDIM 166 costs ~3 s a step).
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.msckf_shapes import BY_NAME, MSCKF_SHAPES, augment_np, batch, observe
from tests.util import cov_err, quat_norm_err, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
B = 70
SEL = [0, 63, 64, B - 1]                 # first, last, and both sides of the ekf_leaf_thread block boundary
IDS = [c.name for c in MSCKF_SHAPES]
GV0, GV1 = [1.0, 1.25], [1.6, 0.7]       # global variable values: at construction, then after <name>_set_<var>


def _folder(cls):
  from rednose_b200.filters import ensure_generated
  return ensure_generated(cls)


def _model(cls, gv=GV0):
  m = hiprec.model_of(cls)
  m.gv = list(gv[:len(m.gvars)])
  return m


def _engine(cls, x, P, Q, gv=GV0, **kw):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(_folder(cls), cls.name, Q, x, P, quaternion_idxs=cls.quat_idxs(),
                    global_vars={g: gv[i] for i, g in enumerate(cls.global_names())}, **kw)


def _dev(a):
  return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _innovation_err(cls, kind, z, y, yr):
  """z, y: the kernel's observation and returned innovation [n, (k,) Z]; yr: the reference's [n, (k,) Y]."""
  Z, EA, _, feat = cls.kinds()[kind]
  if feat:
    nk, nr = np.linalg.norm(y[..., :Z - EA], axis=-1), np.linalg.norm(yr, axis=-1)
    return float(np.max(np.abs(nk - nr) / nr))
  return state_err(z - y, z - yr)


def _check(cls, tag, x, P, xr, Pr, ey=0.0, normalised=True):
  ex, eP = state_err(x, xr), cov_err(P, Pr)
  print(f"{cls.name} {tag}: state {ex:.1e} cov {eP:.1e} innovation {ey:.1e}")
  assert ex < TIGHT and ey < TIGHT, (tag, ex, ey)
  assert eP < TIGHT, (tag, eP)
  if cls.quat_idxs() and normalised:
    assert quat_norm_err(x, cls.quat_idxs()) <= 1e-15


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_fused_step_every_kind(cls):
  m = _model(cls)
  for kind in cls.kinds():
    x, P, Q, dt = batch(cls, B, seed=10 + kind)
    z, R, ea = observe(cls, m, kind, x, seed=kind)
    e = _engine(cls, x, P, Q)
    y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
    xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=SEL)
    _check(cls, f"step kind {kind}", e.state()[SEL], e.covs()[SEL], xr, Pr, _innovation_err(cls, kind, z[SEL], y[SEL], yr))


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_predict_update_and_two_observations(cls):
  """Predict alone leaves the clone block of x and P bit-identical (F is the identity there, Q is zero; quaternions are
  normalised only after updates here); then a feature update, then a fused step with two feature observations at one
  timestamp (extra arguments at offset b * n_obs + o)."""
  m = _model(cls)
  x, P, Q, dt = batch(cls, B, seed=20)
  q, ME, DM = cls.quat_idxs(), cls.medim(), cls.dmain()
  e = _engine(cls, x, P, Q, norm_after_predict=False)
  e.predict(_dev(dt))
  xk, Pk = e.state(), e.covs()
  assert np.array_equal(xk[:, DM:], x[:, DM:]) and np.array_equal(Pk[:, ME:, ME:], P[:, ME:, ME:])
  xp, Pp = hiprec.predict(m, x, P, Q, dt, quat_idxs=q, flags=2, sel=SEL)
  _check(cls, "predict", xk[SEL], Pk[SEL], xp, Pp, normalised=False)
  kind = cls.feature_kinds()[0]
  z, R, ea = observe(cls, m, kind, xk, seed=21)
  y = e.update(kind, z, R, ea)[:, 0].cpu().numpy()
  xr, Pr, yr = hiprec.update(m, kind, xk, Pk, z, R, ea, quat_idxs=q, flags=2, sel=SEL)
  _check(cls, f"update kind {kind}", e.state()[SEL], e.covs()[SEL], xr, Pr, _innovation_err(cls, kind, z[SEL], y[SEL], yr))
  x2, P2 = e.state(), e.covs()
  z, R, ea = observe(cls, m, kind, x2, seed=22, n_obs=2)
  y = e.step(kind, _dev(dt), z, R, ea).cpu().numpy()
  xr, Pr, yr = hiprec.step(m, kind, x2, P2, Q, dt, z, R, ea, quat_idxs=q, flags=2, sel=SEL)
  _check(cls, f"two observations kind {kind}", e.state()[SEL], e.covs()[SEL], xr, Pr, _innovation_err(cls, kind, z[SEL], y[SEL], yr))


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_step_indexed_unordered(cls):
  m = _model(cls)
  x, P, Q, dt = batch(cls, B, seed=30)
  n = 66                                           # two leaf blocks; four filters are not listed
  idx = np.random.default_rng(31).permutation(B)[:n].astype(np.int32)
  kind = cls.feature_kinds()[-1]
  z, R, ea = observe(cls, m, kind, x[idx], seed=32)
  e = _engine(cls, x, P, Q)
  y = e.step_indexed(kind, _dev(idx), _dev(dt[:n]), z, R, ea)[:, 0].cpu().numpy()
  rest = np.setdiff1d(np.arange(B), idx)
  assert np.array_equal(e.state()[rest], x[rest]) and np.array_equal(e.covs()[rest], P[rest])   # untouched, bit for bit
  ent = [0, 63, 64, n - 1]
  xr, Pr, yr = hiprec.step(m, kind, x[idx], P[idx], Q, dt[:n], z, R, ea, quat_idxs=cls.quat_idxs(), sel=ent)
  _check(cls, f"step_indexed kind {kind}", e.state()[idx[ent]], e.covs()[idx[ent]], xr, Pr,
         _innovation_err(cls, kind, z[ent], y[ent], yr))


def _f64_projected_maha(m, cls, kind, x, P, Q, dt, z, R, ea):
  """y'^T S'^-1 y' of every filter after the predict, in float64: the distance the gate of a feature kind thresholds."""
  E, D = m.dim_err, m.dim_x
  Z, EA = cls.kinds()[kind][:2]
  out = []
  for b in range(x.shape[0]):
    F = m.np_leaf('F', x[b], dt[b]).reshape(E, E)
    xb = m.np_leaf('f', x[b], dt[b])
    for i in cls.quat_idxs():
      xb[i:i + 4] /= np.linalg.norm(xb[i:i + 4])
    Pb = F @ P[b] @ F.T + dt[b] * Q
    He = m.np_leaf(('H', kind), xb, ea[b]).reshape(Z, D) @ m.np_leaf('H_mod', xb).reshape(D, E)
    A = np.linalg.qr(m.np_leaf(('He', kind), xb, ea[b]).reshape(Z, EA), mode='complete')[0][:, EA:]
    y, H = A.T @ (z[b] - m.np_leaf(('h', kind), xb, ea[b])), A.T @ He
    out.append(float(y @ np.linalg.solve(H @ Pb @ H.T + A.T @ R[b] @ A, y)))
  return np.array(out)


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_gate_fires_on_exactly_the_reference_set(cls):
  m = _model(cls)
  kind = next(k for k, v in cls.kinds().items() if v[2] and v[3])   # the gated feature kind
  x, P, Q, dt = batch(cls, B, seed=40)
  outliers = [5, 63, 64, 66]
  xp = np.stack([m.np_leaf('f', x[b], dt[b]) for b in range(B)])      # float64 predicted states
  for i in cls.quat_idxs():
    xp[:, i:i + 4] /= np.linalg.norm(xp[:, i:i + 4], axis=1, keepdims=True)
  z, R, ea = observe(cls, m, kind, xp, seed=41, noise=0.1, outliers=outliers)   # inliers: distance ~0.01 Y
  thr = float(m.maha_thresh(kind))
  d = _f64_projected_maha(m, cls, kind, x, P, Q, dt, z, R, ea)
  assert np.min(np.abs(d - thr)) > 1e-6 * thr      # no distance near the threshold: the set is well defined
  want = set(np.flatnonzero(d > thr).tolist())
  assert want == set(outliers)
  e = _engine(cls, x, P, Q)
  y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
  xk = e.state()
  # a gated update moves x by ~1e-12 from the predicted state, any other by ~1e-3
  got = set(np.flatnonzero(np.max(np.abs(xk - xp), axis=1) < 1e-8).tolist())
  assert got == want, sorted(got ^ want)
  sel = sorted(set(SEL) | set(outliers))
  xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=sel)
  _check(cls, f"gated kind {kind}", xk[sel], e.covs()[sel], xr, Pr, _innovation_err(cls, kind, z[sel], y[sel], yr))


@pytest.mark.parametrize("cls", [c for c in MSCKF_SHAPES if c.global_names()], ids=lambda c: c.name)
def test_global_variables_take_effect(cls):
  x, P, Q, dt = batch(cls, B, seed=50)
  kind = min(k for k, v in cls.kinds().items() if not v[3])          # f and this kind's h use the globals
  z, R, ea = observe(cls, _model(cls), kind, x, seed=51)
  e = _engine(cls, x, P, Q)
  for i, g in enumerate(cls.global_names()):
    getattr(e._lib, f"{cls.name}_set_{g}")(GV1[i])
  y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
  m1 = _model(cls, GV1)
  xr, Pr, yr = hiprec.step(m1, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=SEL)
  _check(cls, "second global values", e.state()[SEL], e.covs()[SEL], xr, Pr, _innovation_err(cls, kind, z[SEL], y[SEL], yr))
  x0, _, _ = hiprec.step(_model(cls, GV0), kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=SEL)
  assert state_err(e.state()[SEL], x0) > 1e-6      # the first values would give a different answer


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_mahalanobis_query_is_unprojected(cls):
  """maha_dist of every kind, a feature kind included, is y^T (H_err P H_err^T + R)^-1 y with the full ZDIM innovation
  (ekf_sym.py:626-649 does not project)."""
  m = _model(cls)
  for kind in cls.kinds():
    x, P, Q, dt = batch(cls, B, seed=70 + kind)
    z, R, ea = observe(cls, m, kind, x, seed=71, outliers=[3, 64])
    e = _engine(cls, x, P, Q)
    d = e.maha_dist(kind, z, R, ea).cpu().numpy()
    dr = hiprec.maha(m, kind, x, P, z, R, ea, sel=SEL + [3])
    err = float(np.max(np.abs(d[SEL + [3]] - dr) / dr))
    print(f"{cls.name} maha kind {kind}: relative {err:.1e}")
    assert err < TIGHT, (kind, err)


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_fused_augment_equals_step_then_augment(cls):
  """step(..., augment=True) (the shift inside the CTA kernel's write-back above EDIM 32, a second launch below) is
  bit-identical to step + augment(), and both are the selection of ekf_sym.py:365-391 applied to the stepped state."""
  m = _model(cls)
  kind = cls.feature_kinds()[0]
  x, P, Q, dt = batch(cls, B, seed=90)
  z, R, ea = observe(cls, m, kind, x, seed=91, outliers=[7])
  e1, e2 = _engine(cls, x, P, Q), _engine(cls, x, P, Q)
  e1.step(kind, _dev(dt), z, R, ea)
  pre_x, pre_P = e1.state().copy(), e1.covs().copy()
  e1.augment()
  e2.step(kind, _dev(dt), z, R, ea, augment=True)
  xa, Pa = augment_np(cls, pre_x, pre_P)
  assert np.array_equal(e1.state(), xa) and np.array_equal(e1.covs(), Pa)
  assert np.array_equal(e2.state(), xa) and np.array_equal(e2.covs(), Pa)


def test_feature_kind_single_filter_host_entry_point():
  """<name>_update_<feature kind> on host arrays (one B = 1 launch of the CTA kernel), at EDIM 33: the reference's
  update, and bit for bit what the batched engine computes for the same filter."""
  cls = BY_NAME["msckf_e33"]
  m = _model(cls)
  kind = cls.feature_kinds()[0]
  x, P, Q, _ = batch(cls, 3, seed=100)
  z, R, ea = observe(cls, m, kind, x, seed=101, outliers=[1])
  e = _engine(cls, x, P, Q, norm_after_update=False)
  e.update(kind, z, R, ea)
  ffi, lib = e._ffi, e._lib
  pp = lambda a: ffi.cast("double *", a.ctypes.data)
  xs, Ps = [], []
  for b in range(3):
    xb, Pb, zb = x[b].copy(), P[b].copy(), z[b].copy()
    getattr(lib, f"{cls.name}_update_{kind}")(pp(xb), pp(Pb), pp(zb), pp(np.ascontiguousarray(R[b])), pp(np.ascontiguousarray(ea[b])))
    assert getattr(lib, f"{cls.name}_cuda_status")() == 0
    xs.append(xb); Ps.append(Pb)
  xs, Ps = np.stack(xs), np.stack(Ps)
  assert np.array_equal(xs, e.state()) and np.array_equal(Ps, e.covs())
  xr, Pr, _ = hiprec.update(m, kind, x, P, z, R, ea, flags=0)
  _check(cls, f"host update kind {kind}", xs, Ps, xr, Pr, normalised=False)
