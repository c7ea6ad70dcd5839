"""Every step, query and smoother entry point at every filter shape the kernels claim to serve (tests/shapes.py), against
the 40-digit reference of tests/hiprec.py.

Each shape runs a ragged batch of B = 2G + 1 filters for the group size G of the kernel that serves it, so the last
group holds one filter; the reference is evaluated on the first and last filter and on both sides of every group
boundary (tests/shapes.sample).  Inputs are well conditioned (prior / posterior variance at most ~100), so the kernels'
rank-m covariance update loses at most ~1e-14 and every check holds at TIGHT = 1e-9.  Innovations are compared as the
predicted observation z - y, since y cancels to ~1e-5 of z in some components.

Worst values measured on one H100 80GB HBM3 (power limit 400 W) over all ten shapes, against TIGHT unless noted:

| check | state | covariance | innovation |
|---|---|---|---|
| fused step, every kind | 7.4e-16 | 2.5e-14 | 4.5e-16 |
| predict / update / two observations | 6.0e-16 | 1.5e-14 | 2.1e-16 |
| step_indexed | 4.5e-16 | 1.5e-14 | 2.2e-16 |
| gated kind with outliers | 2.6e-16 | 3.4e-15 | 2.6e-16 |
| second global values | 2.2e-16 | 1.1e-15 | 1.8e-16 |
| RTS (scalar and tensor-core) | 4.5e-16 | 4.2e-14 | |
| Mahalanobis distance, relative | 6.8e-15 | | |
"""
import numpy as np
import pytest
import torch

from tests import hiprec
from tests.shapes import EA_KIND, SHAPES, batch, observe, sample
from tests.util import cov_err, quat_norm_err, state_err

pytestmark = pytest.mark.gpu

TIGHT = 1e-9
IDS = [c.name for c in SHAPES]
GV0, GV1 = [1.0, 1.25], [1.6, 0.7]   # global variable values: at construction, then after <name>_set_<var>


def _folder():
  from tests.shapes import ensure_all
  return ensure_all()


def _model(cls, gv=GV0):
  m = hiprec.model_of(cls)
  m.gv = list(gv[:len(m.gvars)])
  return m


def _engine(cls, x, P, Q, gv=GV0):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(_folder(), cls.name, Q, x, P, quaternion_idxs=cls.quat_idxs(),
                    global_vars={g: gv[i] for i, g in enumerate(cls.global_names())})


def _dev(a):
  return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _check(cls, tag, x, P, xr, Pr, z=None, y=None, yr=None, state_tol=TIGHT, cov_tol=TIGHT, normalised=True):
  """x, P, z, y: the kernel's values of the sampled filters; xr, Pr, yr: the reference's."""
  ex, eP = state_err(x, xr), cov_err(P, Pr)
  ey = state_err(z - y, z - yr) if y is not None else 0.0
  print(f"{cls.name} {tag}: state {ex:.1e} cov {eP:.1e} innovation {ey:.1e}")
  assert ex < state_tol and ey < state_tol, (tag, ex, ey)
  assert eP < cov_tol, (tag, eP)
  if cls.quat_idxs() and normalised:
    assert quat_norm_err(x, cls.quat_idxs()) <= 1e-15


def _setup(cls, seed, B=None):
  B = B or 2 * cls.group() + 1
  x, P, Q, dt = batch(cls, B, seed=seed)
  return _model(cls), x, P, Q, dt, sample(cls, B)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_fused_step_every_kind(cls):
  for kind in cls.kinds():
    m, x, P, Q, dt, sel = _setup(cls, seed=10 + kind)
    z, R, ea = observe(cls, m, kind, x, seed=kind)
    e = _engine(cls, x, P, Q)
    y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
    xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=sel)
    _check(cls, f"step kind {kind}", e.state()[sel], e.covs()[sel], xr, Pr, z[sel], y[sel], yr)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_predict_update_and_two_observations(cls):
  m, x, P, Q, dt, sel = _setup(cls, seed=20)
  q = cls.quat_idxs()
  e = _engine(cls, x, P, Q)
  e.predict(_dev(dt))
  xp, Pp = hiprec.predict(m, x, P, Q, dt, quat_idxs=q, sel=sel)
  _check(cls, "predict", e.state()[sel], e.covs()[sel], xp, Pp)
  kind = sorted(cls.kinds())[0]
  x1, P1 = e.state(), e.covs()
  z, R, ea = observe(cls, m, kind, x1, seed=21)
  y = e.update(kind, z, R, ea)[:, 0].cpu().numpy()
  xr, Pr, yr = hiprec.update(m, kind, x1, P1, z, R, ea, quat_idxs=q, sel=sel)
  _check(cls, f"update kind {kind}", e.state()[sel], e.covs()[sel], xr, Pr, z[sel], y[sel], yr)
  # two observations at one timestamp, on the extra-argument kind where there is one (its ea offset is b * n_obs + o)
  kind = EA_KIND if EA_KIND in cls.kinds() else kind
  x2, P2 = e.state(), e.covs()
  z, R, ea = observe(cls, m, kind, x2, seed=22, n_obs=2)
  y = e.step(kind, _dev(dt), z, R, ea).cpu().numpy()
  xr, Pr, yr = hiprec.step(m, kind, x2, P2, Q, dt, z, R, ea, quat_idxs=q, sel=sel)
  _check(cls, f"two observations kind {kind}", e.state()[sel], e.covs()[sel], xr, Pr, z[sel], y[sel], yr)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_step_indexed_unordered_with_ragged_tail(cls):
  m, x, P, Q, dt, _ = _setup(cls, seed=30)
  B, G = x.shape[0], cls.group()
  n = G + G // 2 + 1                               # one full group and a ragged one
  idx = np.random.default_rng(31).permutation(B)[:n].astype(np.int32)
  kind = EA_KIND if EA_KIND in cls.kinds() else sorted(cls.kinds())[-1]
  z, R, ea = observe(cls, m, kind, x[idx], seed=32)
  e = _engine(cls, x, P, Q)
  x0, P0 = e.x.clone(), e.P.clone()
  y = e.step_indexed(kind, _dev(idx), _dev(dt[:n]), z, R, ea)[:, 0].cpu().numpy()
  rest = torch.as_tensor(np.setdiff1d(np.arange(B), idx)).cuda()
  assert torch.equal(e.x[rest], x0[rest]) and torch.equal(e.P[rest], P0[rest])   # untouched, bit for bit
  ent = sorted({0, G - 1, G, n - 1})                # entries on both sides of the group boundary and the last
  xr, Pr, yr = hiprec.step(m, kind, x[idx], P[idx], Q, dt[:n], z, R, ea, quat_idxs=cls.quat_idxs(), sel=ent)
  _check(cls, f"step_indexed kind {kind}", e.state()[idx[ent]], e.covs()[idx[ent]], xr, Pr, z[ent], y[ent], yr)


def _f64_predicted_maha(m, kind, x, P, Q, dt, z, R, ea, q):
  """Mahalanobis distance of every filter after the predict, in float64 (decides the gate for the whole batch)."""
  E, D = m.dim_err, m.dim_x
  out = []
  for b in range(x.shape[0]):
    F = m.np_leaf('F', x[b], dt[b]).reshape(E, E)
    xb = m.np_leaf('f', x[b], dt[b])
    for i in q:
      xb[i:i + 4] /= np.linalg.norm(xb[i:i + 4])
    Pb = F @ P[b] @ F.T + dt[b] * Q
    args = [ea[b]] if ea is not None else []
    He = m.np_leaf(('H', kind), xb, *args).reshape(-1, D) @ m.np_leaf('H_mod', xb).reshape(D, E)
    y = z[b] - m.np_leaf(('h', kind), xb, *args)
    out.append(float(y @ np.linalg.solve(He @ Pb @ He.T + R[b], y)))
  return np.array(out)


@pytest.mark.parametrize("cls", [c for c in SHAPES if any(g for _, _, g in c.kinds().values())], ids=lambda c: c.name)
def test_gate_fires_on_exactly_the_reference_set(cls):
  m, x, P, Q, dt, sel = _setup(cls, seed=40)
  B = x.shape[0]
  kind = next(k for k, (_, _, g) in cls.kinds().items() if g)
  outliers = sorted({b for b in range(B) if b % 3 == 1} | {B - 1})
  xp = np.stack([m.np_leaf('f', x[b], dt[b]) for b in range(B)])      # float64 predicted states
  for i in cls.quat_idxs():
    xp[:, i:i + 4] /= np.linalg.norm(xp[:, i:i + 4], axis=1, keepdims=True)
  z, R, ea = observe(cls, m, kind, xp, seed=41, noise=0.1, outliers=outliers)   # inliers: distance ~0.01 Z
  thr = float(m.maha_thresh(kind))
  d = _f64_predicted_maha(m, kind, x, P, Q, dt, z, R, ea, cls.quat_idxs())
  assert np.min(np.abs(d - thr)) > 1e-6 * thr      # no distance near the threshold: the set is well defined
  want = set(np.flatnonzero(d > thr).tolist())
  assert want == set(outliers)
  e = _engine(cls, x, P, Q)
  y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
  xk = e.state()
  # the filters the kernel gated: a gated update moves x by ~1e-12 from the predicted state, any other by ~1e-2
  moved = np.max(np.abs(xk - xp), axis=1)
  got = set(np.flatnonzero(moved < 1e-8).tolist())
  assert got == want, sorted(got ^ want)
  xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=sel)
  _check(cls, f"gated kind {kind}", xk[sel], e.covs()[sel], xr, Pr, z[sel], y[sel], yr)


@pytest.mark.parametrize("cls", [c for c in SHAPES if c.global_names()], ids=lambda c: c.name)
def test_global_variables_take_effect(cls):
  m, x, P, Q, dt, sel = _setup(cls, seed=50)
  kind = sorted(cls.kinds())[0]                    # f and this kind's h use the globals
  z, R, ea = observe(cls, m, kind, x, seed=51)
  e = _engine(cls, x, P, Q)
  for i, g in enumerate(cls.global_names()):
    getattr(e._lib, f"{cls.name}_set_{g}")(GV1[i])
  y = e.step(kind, _dev(dt), z, R, ea)[:, 0].cpu().numpy()
  m1 = _model(cls, GV1)
  xr, Pr, yr = hiprec.step(m1, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=sel)
  _check(cls, "second global values", e.state()[sel], e.covs()[sel], xr, Pr, z[sel], y[sel], yr)
  m0 = _model(cls, GV0)
  x0, _, _ = hiprec.step(m0, kind, x, P, Q, dt, z, R, ea, quat_idxs=cls.quat_idxs(), sel=sel)
  assert state_err(e.state()[sel], x0) > 1e-6      # the first values would give a different answer


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_edge_batches_and_the_last_history_slab(cls):
  """B = 0 (no launch, no error) and B = 1 against the reference; over a recorded history the last filtered slab is the
  state bit for bit, and the predicted slab differs from it."""
  m, x, P, Q, dt, _ = _setup(cls, seed=90)
  kind = sorted(cls.kinds())[0]
  z, R, ea = observe(cls, m, kind, x[:1], seed=91)
  e = _engine(cls, x[:0], P[:0], Q)
  y = e.step(kind, _dev(dt[:0]), z[:0], R[:0], None if ea is None else ea[:0])
  assert y.shape[0] == 0 and e.state().shape[0] == 0
  e = _engine(cls, x[:1], P[:1], Q)
  y = e.step(kind, _dev(dt[:1]), z, R, ea)[:, 0].cpu().numpy()
  xr, Pr, yr = hiprec.step(m, kind, x[:1], P[:1], Q, dt[:1], z, R, ea, quat_idxs=cls.quat_idxs(), sel=[0])
  _check(cls, f"B = 1 kind {kind}", e.state(), e.covs(), xr, Pr, z, y, yr)
  e = _engine(cls, x, P, Q)
  T = 3
  h = e.new_history(T)
  kinds = sorted(cls.kinds())
  for k in range(T):
    kind = kinds[k % len(kinds)]
    z, R, ea = observe(cls, m, kind, e.state(), seed=92 + k)
    e.step_recorded(h, kind, 0.02 * (k + 1), z, R, ea)
  assert torch.equal(h.x_filt[T - 1], e.x) and torch.equal(h.P_filt[T - 1], e.P)
  assert not torch.equal(h.P_pred[T - 1], e.P)


@pytest.mark.parametrize("cls", [c for c in SHAPES if c.step_kernel() == "pair"], ids=lambda c: c.name)
def test_pair_layouts_and_host_step(cls):
  """Packed engine, full-layout ABI and host entry point: bit-identical."""
  m, x, P, Q, dt, _ = _setup(cls, seed=60)
  B, E = x.shape[0], cls.edim
  for kind in cls.kinds():
    outliers = [b for b in range(B) if b % 5 == 2] if cls.kinds()[kind][2] else []
    z, R, ea = observe(cls, m, kind, x, seed=61, outliers=outliers)
    a, b = _engine(cls, x, P, Q), _engine(cls, x, P, Q)
    assert a._Pk is not None and a._packed_doubles == 4 * (E // 2) * (E // 2 + 1) // 2
    b._Pf, b._Pk, b._full_owns = b.P.clone(), None, True
    ya, yb = a.step(kind, _dev(dt), z, R, ea), b.step(kind, _dev(dt), z, R, ea)
    assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P) and torch.equal(ya, yb)
    assert torch.equal(a.P, a.P.transpose(1, 2))
    hx, hP, hz = x.copy(), P.copy(), z.copy()
    ffi, lib = a._ffi, a._lib
    pp = lambda t: ffi.cast("double *", t.ctypes.data) if t is not None else ffi.NULL
    qi = cls.quat_idxs()
    getattr(lib, f"{cls.name}_host_step_{kind}")(pp(hx), pp(hP), pp(Q), pp(dt), 0.0, pp(hz), pp(np.ascontiguousarray(R)),
                                                 pp(None if ea is None else np.ascontiguousarray(ea)), 1, B,
                                                 ffi.new("int[]", qi or [0]), len(qi), a.flags)
    assert getattr(lib, f"{cls.name}_cuda_status")() == 0
    assert np.array_equal(hx, a.state()) and np.array_equal(hP, a.covs()) and np.array_equal(hz, ya.cpu().numpy()[:, 0])


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_mahalanobis_query(cls):
  for kind, (Z, _, _) in cls.kinds().items():
    m, x, P, Q, dt, sel = _setup(cls, seed=70 + kind)
    B = x.shape[0]
    outliers = [b for b in range(B) if b % 4 == 3]
    z, R, ea = observe(cls, m, kind, x, seed=71, outliers=outliers)
    e = _engine(cls, x, P, Q)
    d = e.maha_dist(kind, z, R, ea).cpu().numpy()
    dr = hiprec.maha(m, kind, x, P, z, R, ea, sel=sel)
    err = float(np.max(np.abs(d[sel] - dr) / dr))
    print(f"{cls.name} maha kind {kind}: relative {err:.1e}")
    assert err < TIGHT, (kind, err)                  # worst (H100): 6.8e-15
    from rednose_b200.chi2 import chi2_ppf
    thr = float(chi2_ppf(0.95, Z))
    assert np.min(np.abs(d - thr)) > 1e-6 * thr
    passed = e.maha_test(kind, z, R, ea).cpu().numpy()
    assert np.array_equal(passed, d <= thr) and not passed[outliers].any()
    assert np.array_equal(passed[sel], dr <= thr)


@pytest.mark.parametrize("cls", SHAPES, ids=IDS)
def test_smoother_over_a_mixed_kind_history(cls):
  """step_recorded over 6 steps cycling through every kind, then rts_smooth (ekf_rts_warp_mma for even EDIM 8-32,
  ekf_rts_warp otherwise), against the reference's RTS on the same recorded slabs."""
  m, x, P, Q, _, sel = _setup(cls, seed=80)
  q = cls.quat_idxs()
  e = _engine(cls, x, P, Q)
  T = 6
  h = e.new_history(T)
  kinds = sorted(cls.kinds())
  for k in range(T):
    kind = kinds[k % len(kinds)]
    z, R, ea = observe(cls, m, kind, e.state(), seed=80 + k)
    e.step_recorded(h, kind, 0.03 * k + 0.007 * (k % 2), z, R, ea)
  xs, Ps = e.rts_smooth(h, norm_quats=bool(q), quaternion_idxs=tuple(q) or (0,))
  slabs = [t.cpu().numpy() for t in (h.x_pred, h.x_filt, h.P_pred, h.P_filt)]
  xr, Pr = hiprec.rts(m, *slabs, h.t_host, quat_idxs=q, norm_quats=bool(q), sel=sel)
  _check(cls, f"rts ({cls.rts_kernel()})", xs.cpu().numpy()[:, sel], Ps.cpu().numpy()[:, sel], xr, Pr,
         normalised=False)   # the smoother leaves step 0 unnormalised, as the reference does
