"""GPU parity tests: the CUDA path (through the C-ABI) against the oracle on identical inputs.

Metrics (tests/util.py): state_err is the worst per-component relative error of states and innovations, cov_err
the worst covariance error in correlation units.  Tolerances are set from the errors measured on an H100 with
about 10x headroom; TIGHT (1e-9) wherever that holds.
"""
import numpy as np
import pytest
import torch

from tests.test_oracle_cpu import GOLDEN, P0, Q, X0, run_kinematic_procedure
from tests.util import LIVE_KINDS, Oracle, cov_err, kinematic_batch, live_batch, live_obs, quat_norm_err, state_err

pytestmark = pytest.mark.gpu
TOL = 1e-6       # the contract
TIGHT = 1e-9     # what the implementation achieves on well-conditioned inputs
QN = 1e-15       # | |q| - 1 | after a normalising step: a few ulp


def _engine(gen_dir, name, x, P, Qm, **kw):
  from rednose_b200.batched import BatchedEKF
  return BatchedEKF(gen_dir, name, Qm, x, P, **kw)


def test_kinematic_golden_through_the_dropin_class(gen_dir):
  """examples/test_kinematic_kf.py run through EKF_sym_pyx -> C-ABI -> CUDA kernels."""
  from rednose_b200.filters.kinematic import KinematicKalman
  kf = KinematicKalman(gen_dir)
  got = run_kinematic_procedure(kf.filter)
  for g, want in zip(got, GOLDEN):
    assert abs(g - want) < 5e-8
    assert abs(g - want) < 1e-12


def test_compare_procedure_on_gpu(gen_dir):
  from rednose_b200.ekf_sym import EKF_sym
  from rednose_b200.ekf_sym_pyx import EKF_sym_pyx
  np.random.seed(0)
  a = EKF_sym_pyx(gen_dir, "kinematic", Q, X0, P0, 2, 2)
  b = EKF_sym(gen_dir, "kinematic", Q, X0, P0, 2, 2)
  ts = np.arange(0, 1, step=0.01)
  ts[20], ts[40] = ts[40], ts[20]
  for t in ts:
    z, R = np.array([[np.random.normal(0, 0.1)]]), np.array([[[0.1**2]]])
    a.predict_and_update_batch(t, 1, z, R)
    b.predict_and_update_batch(t, 1, z, R)
    assert np.allclose(a.state(), b.state()) and np.allclose(a.covs(), b.covs())


def test_kinematic_batched_step(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "kinematic")
  B = 10007  # ragged: not a multiple of the CTA size
  x, P, Qm, z, R = kinematic_batch(B)
  dt = np.random.default_rng(5).uniform(0.005, 0.02, B)
  xr, Pr, yr = o.batch_step(1, x, P, Qm, dt, z, R)
  e = _engine(gen_dir, "kinematic", x, P, Qm)
  y = e.step(1, torch.as_tensor(dt), z, R)
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT and state_err(y.cpu().numpy()[:, 0], yr) < TIGHT


@pytest.mark.parametrize("kind", sorted(LIVE_KINDS))
def test_live_fused_step_every_kind(gen_dir, oracle_dir, kind):
  o = Oracle(oracle_dir, "live")
  B = 1031
  x, P, Qm = live_batch(B, seed=kind)
  z, R = live_obs(o, kind, x)
  xr, Pr, yr = o.batch_step(kind, x, P, Qm, 0.01, z, R, quat_idxs=[3], flags=3)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  y = e.step(kind, 0.01, z, R)
  ex, eP, ey = state_err(e.state(), xr), cov_err(e.covs(), Pr), state_err(y.cpu().numpy()[:, 0], yr)
  assert ex < TIGHT and eP < TIGHT and ey < TIGHT, (ex, eP, ey)
  assert quat_norm_err(e.state(), [3]) <= QN


def test_live_predict_and_update_separately(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  B = 257
  x, P, Qm = live_batch(B, seed=11)
  xr, Pr = o.predict(x, P, Qm, 0.02)
  e = _engine(gen_dir, "live", x, P, Qm, norm_after_predict=False, norm_after_update=False)
  e.predict(0.02)
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT
  z, R = live_obs(o, 13, xr)
  xr2, Pr2, yr = o.update(13, xr, Pr, z, R)
  y = e.update(13, z, R)
  assert state_err(e.state(), xr2) < TIGHT and cov_err(e.covs(), Pr2) < TIGHT and state_err(y.cpu().numpy()[:, 0], yr) < TIGHT


def test_live_stream_300_steps(gen_dir, oracle_dir):
  """IMU at 100 Hz alternating gyro / accel, a position fix at t0 and every 100 steps (SURVEY.md 8d config 3)."""
  o = Oracle(oracle_dir, "live")
  B = 64
  x, P, Qm = live_batch(B, seed=21, well_conditioned=False)  # starts from the example's own P0 scale (cond ~1e12)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  xr, Pr = x.copy(), P.copy()
  for k in range(300):
    kind = 12 if k % 100 == 0 else (4 if k % 2 else 10)
    z, R = live_obs(o, kind, xr, seed=100 + k)
    xr, Pr, yr = o.batch_step(kind, xr, Pr, Qm, 0.01, z, R, quat_idxs=[3], flags=3)
    y = e.step(kind, 0.01, z, R)
    if k in (0, 1, 50, 299):   # measured on an H100: worst 8.1e-10 (state), 1.4e-9 (covariance)
      assert state_err(e.state(), xr) < 1e-8 and cov_err(e.covs(), Pr) < 1e-8, k
      assert quat_norm_err(e.state(), [3]) <= QN, k
  assert state_err(e.state(), xr) < 1e-8 and cov_err(e.covs(), Pr) < 1e-8


def test_multiple_observations_per_predict(gen_dir, oracle_dir):
  """n observations of one kind at one timestamp: predict once, update n times (ekf_sym.cc:174-180)."""
  o = Oracle(oracle_dir, "live")
  B, n = 129, 3
  x, P, Qm = live_batch(B, seed=31)
  zs, Rs = zip(*[live_obs(o, 4, x, seed=40 + i) for i in range(n)])
  xr, Pr = o.predict(x, P, Qm, 0.01)
  for i in range(n):
    xr, Pr, _ = o.update(4, xr, Pr, zs[i], Rs[i])
  e = _engine(gen_dir, "live", x, P, Qm, norm_after_predict=False, norm_after_update=False)
  e.step(4, 0.01, np.stack(zs, 1), np.stack(Rs, 1))
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT


def test_leaf_functions_match_reference_generated_c(gen_dir, oracle_dir):
  from rednose_b200.ekf_sym import EKF_sym
  from rednose_b200.filters.live import LiveKalman
  o = Oracle(oracle_dir, "live")
  kf = EKF_sym(gen_dir, "live", LiveKalman.Q, LiveKalman.initial_x, np.diag(LiveKalman.initial_P_diag), 23, 22)
  x, _, _ = live_batch(4, seed=7)
  rng = np.random.default_rng(0)
  got, want = {}, {}     # every output entry is compared per entry, scaled by its largest value over the 4 states

  def put(key, a, r):
    got.setdefault(key, []).append(a.copy()); want.setdefault(key, []).append(r.copy())

  for b in range(4):
    xb = np.ascontiguousarray(x[b])
    for fn, shape, args in [("f_fun", 23, (0.01,)), ("F_fun", 22 * 22, (0.01,))]:
      a, r = np.zeros(shape), np.zeros(shape)
      getattr(kf, "f" if fn == "f_fun" else "F")(xb, 0.01, a)
      o.leaf(fn, xb, 0.01, r)
      put(fn, a, r)
    a, r = np.zeros(23 * 22), np.zeros(23 * 22)
    kf.H_mod(xb, a); o.leaf("H_mod_fun", xb, r)
    put("H_mod_fun", a, r)
    d = rng.normal(0, 0.01, 22)
    a, r = np.zeros(23), np.zeros(23)
    kf.err_function(xb, d, a); o.leaf("err_fun", xb, d, r)
    put("err_fun", a, r)
    a2, r2 = np.zeros(22), np.zeros(22)
    kf.inv_err_function(xb, a, a2); o.leaf("inv_err_fun", xb, r, r2)
    put("inv_err_fun", a2, r2)
    assert np.max(np.abs(a2 - d)) < 1e-3 * np.max(np.abs(d))     # inv_err_fun inverts err_fun to first order
    dummy = np.zeros(1)
    for k, m in LIVE_KINDS.items():
      a, r = np.zeros(m), np.zeros(m)
      kf.hs[k](xb, dummy, a); o.leaf(f"h_{k}", xb, dummy, r)
      put(f"h_{k}", a, r)
      a, r = np.zeros(m * 23), np.zeros(m * 23)
      kf.Hs[k](xb, dummy, a); o.leaf(f"H_{k}", xb, dummy, r)
      put(f"H_{k}", a, r)
  for key in got:
    err = state_err(np.stack(got[key]), np.stack(want[key]))
    assert err < (1e-9 if key == "inv_err_fun" else 1e-13), (key, err)


def test_host_buffer_entry_point_equals_device_path(gen_dir):
  """<name>_host_step_<kind> (host pointers, copies inside) == <name>_batch_step_<kind> (device pointers)."""
  from rednose_b200.loader import load_code
  B = 20011
  x, P, Qm = live_batch(B, seed=3)
  rng = np.random.default_rng(9)
  z = x[:, 0:3] + rng.normal(0, 5.0, (B, 3))
  R = np.tile(np.diag([25.0] * 3), (B, 1, 1))
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  y = e.step(12, 0.01, z, R).cpu().numpy()[:, 0]
  ffi, lib = load_code(gen_dir, "live")
  hx, hP, hz = x.copy(), P.copy(), z.copy()
  qi = ffi.new("int[]", [3])
  p = lambda a: ffi.cast("double *", a.ctypes.data)
  lib.live_host_step_12(p(hx), p(hP), ffi.cast("const double *", Qm.ctypes.data), ffi.NULL, 0.01, p(hz),
                        ffi.cast("const double *", R.ctypes.data), ffi.NULL, 1, B, qi, 1, e.flags)
  assert lib.live_cuda_status() == 0
  assert np.array_equal(hx, e.state()) and np.array_equal(hP, e.covs()) and np.array_equal(hz, y)


def test_full_size_properties_1m_live(gen_dir, oracle_dir):
  """BASELINE.json full size (1M live filters): size-independent properties + a sampled oracle check."""
  o = Oracle(oracle_dir, "live")
  Bu = 4096
  x, P, Qm = live_batch(Bu, seed=77)
  z, R = live_obs(o, 4, x)
  reps = 256  # 4096 * 256 = 1,048,576 filters: every replica must produce bit-identical results
  B = Bu * reps
  e = _engine(gen_dir, "live", np.tile(x, (reps, 1)), np.tile(P, (reps, 1, 1)), Qm, quaternion_idxs=[3])
  y = e.step(4, 0.01, torch.as_tensor(np.tile(z, (reps, 1))), torch.as_tensor(np.tile(R, (reps, 1, 1))))
  xs = e.x.view(reps, Bu, 23)
  Ps = e.P.view(reps, Bu, 22, 22)
  assert bool((xs == xs[0:1]).all()) and bool((Ps == Ps[0:1]).all())       # position independence
  asym = (e.P - e.P.transpose(1, 2)).abs().amax() / e.P.abs().amax()
  assert float(asym) < 1e-12                                                # covariance stays symmetric
  qn = e.x[:, 3:7].norm(dim=1)
  assert float((qn - 1).abs().max()) < 1e-14                                # quaternion normalised
  xr, Pr, yr = o.batch_step(4, x, P, Qm, 0.01, z, R, quat_idxs=[3], flags=3)
  assert state_err(xs[-1].cpu().numpy(), xr) < TIGHT and cov_err(Ps[-1].cpu().numpy(), Pr) < TIGHT
  assert B == 1048576


def _record_live_history(gen_dir, o, B, T, seed, well_conditioned=True):
  x, P, Qm = live_batch(B, seed=seed, well_conditioned=well_conditioned)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  hist = e.new_history(T)
  xr = x.copy()
  for k in range(T):
    kind = 12 if k % 10 == 0 else (4 if k % 2 else 10)
    z, R = live_obs(o, kind, e.state() if k else xr, seed=500 + k)
    e.step_recorded(hist, kind, 0.01 * (k + 1), z, R)
  return e, hist


@pytest.mark.parametrize("norm_quats", [False, True])
def test_rts_smoother_matches_reference_recursion(gen_dir, oracle_dir, norm_quats):
  """K2: the batched backward kernel vs the restated ekf_sym.py:651-690 on the SAME recorded history."""
  from oracle.rts_numpy import rts_smooth
  o = Oracle(oracle_dir, "live")
  B, T = 33, 40
  e, hist = _record_live_history(gen_dir, o, B, T, seed=61)
  hx_p, hx_f = hist.x_pred.cpu().numpy(), hist.x_filt.cpu().numpy()
  hP_p, hP_f = hist.P_pred.cpu().numpy(), hist.P_filt.cpu().numpy()
  t = hist.t_host.copy()
  xs, Ps = e.rts_smooth(hist, norm_quats=norm_quats)
  xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
  worst_x = worst_P = 0.0
  for b in range(0, B, 4):
    xr, Pr = rts_smooth(o, hx_p[:, b], hx_f[:, b], hP_p[:, b], hP_f[:, b], t, 23, 22, norm_quats=norm_quats)
    worst_x = max(worst_x, state_err(xs[:, b], xr))
    worst_P = max(worst_P, cov_err(Ps[:, b], Pr))
  assert worst_x < TIGHT and worst_P < TIGHT, (worst_x, worst_P)
  # smoothing must not increase the position variance of interior points
  assert np.all(Ps[5, :, 0, 0] <= hP_f[5, :, 0, 0] * (1 + 1e-9))


def test_history_slabs_equal_separate_predict_update(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  e, hist = _record_live_history(gen_dir, o, 17, 3, seed=71)
  # the last filtered slab is the live state; the predicted slab differs from it
  assert torch.equal(hist.x_filt[2], e.x) and torch.equal(hist.P_filt[2], e.P)
  assert not torch.equal(hist.P_pred[2], e.P)


def test_cuda_path_reproduces_reference_golden_vectors(gen_dir):
  """tests/golden/live_reference.npz: forward filter (all 8 kinds) and RTS smoother produced by the
  reference's own Python maths; the CUDA path must reproduce them through the batched C-ABI."""
  import os
  g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference.npz"))
  kinds, ts = g["kinds"], g["t"]
  T = len(kinds)
  # python-driver semantics: no normalisation after the predict (ekf_sym.py:508), after the update yes (:521)
  e = _engine(gen_dir, "live", g["x0"], g["P0"], g["Q"], quaternion_idxs=[3], norm_after_predict=False)
  hist = e.new_history(T)
  e.filter_time = float(ts[0])
  for k, kind in enumerate(kinds):
    m = LIVE_KINDS[int(kind)]
    z = np.stack([g[f"z{b}"][k, :m] for b in range(2)])
    R = np.stack([g[f"R{b}"][k, :m, :m] for b in range(2)])
    y = e.step_recorded(hist, int(kind), float(ts[k]), z, R).cpu().numpy()[:, 0]
    ex = state_err(e.state(), np.stack([g[f"x_filt{b}"][k] for b in range(2)]))
    eP = cov_err(e.covs(), np.stack([g[f"P_filt{b}"][k] for b in range(2)]))
    assert ex < TIGHT and eP < TIGHT, (k, kind, ex, eP)
    assert quat_norm_err(e.state(), [3]) <= QN
    ey = state_err(y, np.stack([g[f"y{b}"][k, :m] for b in range(2)]))
    assert ey < TIGHT, (k, kind, ey)
  for b in range(2):
    assert cov_err(hist.P_pred[:, b].cpu().numpy(), g[f"P_pred{b}"]) < TIGHT
  xs, Ps = e.rts_smooth(hist, norm_quats=True)
  for b in range(2):
    assert state_err(xs[:, b].cpu().numpy(), g[f"xs{b}"]) < TIGHT and cov_err(Ps[:, b].cpu().numpy(), g[f"Ps{b}"]) < TIGHT


def test_shared_R_equals_replicated_R(gen_dir):
  B = 513
  x, P, Qm = live_batch(B, seed=81)
  rng = np.random.default_rng(1)
  z = x[:, 0:3] + rng.normal(0, 5.0, (B, 3))
  R1 = np.diag([25.0, 16.0, 9.0])
  a = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  b = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  ya = a.step(12, 0.01, z, np.tile(R1, (B, 1, 1)))
  yb = b.step(12, 0.01, z, R1)
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P) and torch.equal(ya, yb)


def test_host_streamer_equals_direct_stepping(gen_dir):
  """The overlapped host<->device front-end returns, for every step, exactly what direct stepping produces."""
  from rednose_b200.streaming import HostStreamer
  B, T = 4099, 7
  x, P, Qm = live_batch(B, seed=91)
  rng = np.random.default_rng(2)
  R = {12: torch.as_tensor(np.diag([25.0] * 3)).cuda(), 4: torch.as_tensor(np.diag([0.025**2] * 3)).cuda()}
  zs = [(12 if k % 3 == 0 else 4, torch.as_tensor((x[:, 0:3] if k % 3 == 0 else np.zeros((B, 3))) + rng.normal(0, 0.01, (B, 3))).pin_memory())
        for k in range(T)]
  a = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  b = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  st = HostStreamer(b, {12: 3, 4: 3})
  a.filter_time = b.filter_time = 0.0
  tickets, want = [], []
  for k, (kind, z) in enumerate(zs):
    t = 0.01 * (k + 1)
    xa, ya = a.predict_and_update_batch(t, kind, z, R[kind])
    want.append((xa.cpu().clone(), ya.cpu()[:, 0].clone()))
    tickets.append(st.submit(t, kind, z, R[kind]))
    if k >= 1:  # results of the previous step are still retrievable (depth 2)
      xh, yh = st.result(tickets[k - 1], zs[k - 1][0])
      assert torch.equal(xh, want[k - 1][0]) and torch.equal(yh, want[k - 1][1])
  xh, yh = st.result(tickets[-1], zs[-1][0])
  assert torch.equal(xh, want[-1][0]) and torch.equal(yh, want[-1][1])
  assert torch.equal(a.P, b.P)


def test_ragged_scheduler_matches_per_filter_driving(gen_dir, oracle_dir):
  """Every filter gets its own observation stream (different kinds, different times, gaps); the scheduler's
  bucketed indexed launches must equal driving each filter on its own (oracle predict + update per observation)."""
  from rednose_b200.scheduler import RaggedScheduler
  o = Oracle(oracle_dir, "live")
  B, ticks = 301, 12
  x, P, Qm = live_batch(B, seed=123)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  sch = RaggedScheduler(e)
  rng = np.random.default_rng(7)
  xr, Pr = x.copy(), P.copy()
  t_ref = np.full(B, np.nan)
  kinds_all = [4, 10, 12, 3]
  for tick in range(ticks):
    active = np.flatnonzero(rng.random(B) < 0.6)                   # ~40 % of the filters see nothing this tick
    t_obs = 0.01 * (tick + 1) + rng.uniform(0, 0.004, active.size)  # per-filter observation times
    kinds = rng.choice(kinds_all, active.size)
    zs, Rs = {}, {}
    for k in kinds_all:
      sel = active[kinds == k]
      if sel.size == 0:
        continue
      zk, Rk = live_obs(o, k, xr[sel], seed=1000 + tick)
      zs[k], Rs[k] = zk, Rk
      # reference: drive each selected filter on its own
      dt = np.where(np.isnan(t_ref[sel]), 0.0, t_obs[kinds == k] - t_ref[sel])
      xs, Ps, _ = o.batch_step(k, xr[sel], Pr[sel], Qm, dt, zk, Rk, quat_idxs=[3], flags=3)
      xr[sel], Pr[sel] = xs, Ps
      t_ref[sel] = t_obs[kinds == k]
    sch.tick(active, t_obs, kinds, zs, Rs)
  assert sch.dropped == 0
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT
  assert quat_norm_err(e.state(), [3]) <= QN
  assert np.allclose(sch.t_filter.cpu().numpy(), t_ref, equal_nan=True)
  # a late observation is dropped, not applied
  before = e.state().copy()
  sch.tick(np.array([0]), np.array([1e-6]), np.array([12]), {12: x[:1, 0:3]}, {12: np.diag([25.0] * 3)})
  assert sch.dropped == 1 and np.array_equal(before, e.state())


def test_edge_batches_empty_single_and_ragged_tail(gen_dir, oracle_dir):
  """B = 0 (no launch, no error), B = 1, and a batch one short / one over a multiple of the warp group."""
  o = Oracle(oracle_dir, "live")
  for B in (0, 1, 13, 15, 29):
    x, P, Qm = live_batch(max(B, 1), seed=200 + B)
    x, P = x[:B], P[:B]
    z, R = (live_obs(o, 12, x) if B else (np.zeros((0, 3)), np.zeros((0, 3, 3))))
    e = _engine(gen_dir, "live", x if B else np.zeros((0, 23)), P if B else np.zeros((0, 22, 22)), Qm, quaternion_idxs=[3])
    y = e.step(12, 0.01, z, R)
    assert y.shape[0] == B
    if B:
      xr, Pr, yr = o.batch_step(12, x, P, Qm, 0.01, z, R, quat_idxs=[3], flags=3)
      assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT


def test_tiled_smoother_equals_untiled(gen_dir, oracle_dir):
  """Config 4 in miniature: forward + RTS over a history, tiled over filters because the history does not fit."""
  from rednose_b200.smoothing import TiledSmoother, history_bytes_per_filter
  o = Oracle(oracle_dir, "live")
  B, T = 37, 12
  x, P, Qm = live_batch(B, seed=300)
  kinds = [12 if k % 5 == 0 else 4 for k in range(T)]
  zs = [live_obs(o, kinds[k], x, seed=400 + k) for k in range(T)]

  def obs_fn(k, lo, hi):
    return 0.01 * (k + 1), kinds[k], zs[k][0][lo:hi], zs[k][1][lo:hi]

  got = {}
  def sink(lo, hi, xs, Ps):
    got[(lo, hi)] = (xs.cpu().numpy().copy(), Ps.cpu().numpy().copy())

  assert history_bytes_per_filter(23, 22, 10_000) == 8 * (2 * 484 + 46) * 10_000   # 81 MB per live filter over 10k steps
  ts = TiledSmoother(gen_dir, "live", Qm, 23, 22, quaternion_idxs=[3], tile=16)
  assert ts.run(x, P, T, obs_fn, sink, norm_quats=True) == 3
  ref = {}
  TiledSmoother(gen_dir, "live", Qm, 23, 22, quaternion_idxs=[3], tile=64).run(x, P, T, obs_fn, lambda lo, hi, xs, Ps: ref.update(a=(xs.cpu().numpy().copy(), Ps.cpu().numpy().copy())), norm_quats=True)
  xs_t = np.concatenate([got[k][0] for k in sorted(got)], axis=1)
  Ps_t = np.concatenate([got[k][1] for k in sorted(got)], axis=1)
  assert np.array_equal(xs_t, ref["a"][0]) and np.array_equal(Ps_t, ref["a"][1])


def test_batched_maha_query_matches_reference_formula(gen_dir, oracle_dir):
  """(f)-2: batched maha_test vs ekf_sym.py:626-649 written out with the oracle's leaf functions."""
  o = Oracle(oracle_dir, "live")
  B = 211
  x, P, Qm = live_batch(B, seed=500)
  for kind, m in ((4, 3), (3, 1), (12, 3)):
    z, R = live_obs(o, kind, x, seed=600 + kind, noise_scale=3.0)
    e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
    d = e.maha_dist(kind, z, R).cpu().numpy()
    want = np.zeros(B)
    dummy = np.zeros(1)
    for b in range(B):
      xb = np.ascontiguousarray(x[b])
      h, H, Hm = np.zeros(m), np.zeros(m * 23), np.zeros(23 * 22)
      o.leaf(f"h_{kind}", xb, dummy, h); o.leaf(f"H_{kind}", xb, dummy, H); o.leaf("H_mod_fun", xb, Hm)
      He = H.reshape(m, 23) @ Hm.reshape(23, 22)
      y = z[b] - h
      want[b] = y @ np.linalg.inv(He @ P[b] @ He.T + R[b]) @ y
    assert state_err(d[:, None], want[:, None]) < 1e-9, kind
    assert torch.equal(e.x.cpu(), torch.as_tensor(x))   # a query: state untouched
    passed = e.maha_test(kind, z, R).cpu().numpy()
    from rednose_b200.chi2 import chi2_ppf
    assert np.array_equal(passed, want <= chi2_ppf(0.95, m))


def test_batched_kalmanfilter_front_end(gen_dir, oracle_dir):
  """(f)-2: KalmanFilter.predict_and_observe for a whole batch (shared per-kind noise from obs_noise)."""
  from rednose_b200.filter_base import BatchedKalmanFilter
  from rednose_b200.filters.kinematic import KinematicKalman
  o = Oracle(oracle_dir, "kinematic")
  B = 1000
  x, P, Qm, z, R = kinematic_batch(B, seed=9)

  class BatchedKinematic(BatchedKalmanFilter):
    obs_noise = KinematicKalman.obs_noise

    def __init__(self):
      self.filter = _engine(gen_dir, "kinematic", x, P, Qm)

  kf = BatchedKinematic()
  kf.predict_and_observe(0.0, 1, z)
  kf.predict_and_observe(0.05, 1, z)
  xr, Pr, _ = o.batch_step(1, x, P, Qm, 0.0, z, R)
  xr, Pr, _ = o.batch_step(1, xr, Pr, Qm, 0.05, z, R)
  assert state_err(kf.x, xr) < TIGHT and cov_err(kf.P, Pr) < TIGHT and kf.t == 0.05
  assert kf.maha_test(1, z).shape == (B,)


def test_gather_list_on_the_thread_kernel(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "kinematic")
  B = 1001
  x, P, Qm, z, R = kinematic_batch(B, seed=77)
  e = _engine(gen_dir, "kinematic", x, P, Qm)
  idx = torch.as_tensor(np.random.default_rng(0).permutation(B)[:400].astype(np.int32)).cuda()   # unordered subset
  sel = idx.cpu().numpy()
  dt = torch.linspace(0.001, 0.02, 400, dtype=torch.float64)
  e.step_indexed(1, idx, dt, z[sel], R[sel])
  xr, Pr, _ = o.batch_step(1, x[sel], P[sel], Qm, dt.numpy(), z[sel], R[sel])
  gx, gP = e.state(), e.covs()
  assert state_err(gx[sel], xr) < TIGHT and cov_err(gP[sel], Pr) < TIGHT
  keep = np.setdiff1d(np.arange(B), sel)
  assert np.array_equal(gx[keep], x[keep]) and np.array_equal(gP[keep], P[keep])


def test_live_long_stream_2000_steps(gen_dir, oracle_dir):
  """Drift check: 2000 fused steps (20 s of 100 Hz IMU + 1 Hz fixes) stay within the contract of the oracle."""
  o = Oracle(oracle_dir, "live")
  B = 16
  x, P, Qm = live_batch(B, seed=2000, well_conditioned=False)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  xr, Pr = x.copy(), P.copy()
  worst = 0.0
  for k in range(2000):
    kind = 12 if k % 100 == 0 else (4 if k % 2 else 10)
    z, R = live_obs(o, kind, xr, seed=5000 + k)
    xr, Pr, _ = o.batch_step(kind, xr, Pr, Qm, 0.01, z, R, quat_idxs=[3], flags=3, nthreads=1)
    e.step(kind, 0.01, z, R)
    if k % 250 == 249:
      worst = max(worst, state_err(e.state(), xr), cov_err(e.covs(), Pr))
      assert quat_norm_err(e.state(), [3]) <= QN
  assert worst < 2e-8, worst       # measured on an H100: 1.8e-9


def test_rts_scalar_fallback_on_the_kinematic_model(gen_dir, oracle_dir):
  """Filters with MEDIM < 8 smooth through the scalar RTS kernel (ekf_rts_warp), not the DMMA variant."""
  from oracle.rts_numpy import rts_smooth
  o = Oracle(oracle_dir, "kinematic")
  B, T = 40, 25
  x, P, Qm, _, _ = kinematic_batch(B, seed=88)
  e = _engine(gen_dir, "kinematic", x, P, Qm)
  hist = e.new_history(T)
  rng = np.random.default_rng(1)
  for k in range(T):
    z = e.state()[:, :1] + rng.normal(0, 0.1, (B, 1))
    e.step_recorded(hist, 1, 0.01 * (k + 1), z, np.array([[0.01]]))
  xs, Ps = e.rts_smooth(hist, norm_quats=False)
  xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
  hx_p, hx_f = hist.x_pred.cpu().numpy(), hist.x_filt.cpu().numpy()
  hP_p, hP_f = hist.P_pred.cpu().numpy(), hist.P_filt.cpu().numpy()
  t = hist.t_host.copy()
  for b in range(0, B, 7):
    xr, Pr = rts_smooth(o, hx_p[:, b], hx_f[:, b], hP_p[:, b], hP_f[:, b], t, 2, 2)
    assert state_err(xs[:, b], xr) < 1e-9 and cov_err(Ps[:, b], Pr) < 1e-9


def test_dense_process_noise(gen_dir, oracle_dir):
  """A Q with off-diagonal terms takes the dense dt*Q path of the kernels (the diagonal fast path is what every
  other live test runs, examples/live_kf.py's Q being diagonal); ekf_c.c:27-28."""
  o = Oracle(oracle_dir, "live")
  B = 131
  x, P, Qm = live_batch(B, seed=17)
  A = np.random.default_rng(4).normal(size=(22, 22)) * 1e-3
  Qd = Qm + A @ A.T
  z, R = live_obs(o, 4, x)
  xr, Pr, yr = o.batch_step(4, x, P, Qd, 0.01, z, R, quat_idxs=[3], flags=3)
  e = _engine(gen_dir, "live", x, P, Qd, quaternion_idxs=[3])
  y = e.step(4, 0.01, z, R)
  assert state_err(e.state(), xr) < TIGHT and cov_err(e.covs(), Pr) < TIGHT and state_err(y.cpu().numpy()[:, 0], yr) < TIGHT


def test_live_single_filter_dropin_path(gen_dir, oracle_dir):
  """The reference's own calling pattern on the 23-state filter: one filter, host arrays, `live_predict` +
  `live_update_<k>` through both drivers (native EKF_sym_pyx and the Python EKF_sym), CUDA library against the
  reference-generated CPU library on the same stream (rednose/helpers/ekf_sym.py:258-343, ekf_sym.cc:125-215)."""
  from rednose_b200.ekf_sym import EKF_sym
  from rednose_b200.filters.live import LiveKalman, ObservationKind as K
  for filter_cls in (None, EKF_sym):
    gpu, cpu = LiveKalman(gen_dir, filter_cls), LiveKalman(oracle_dir, filter_cls)
    rng = np.random.default_rng(3)
    t = 0.0
    for k in range(40):
      t += 0.01
      if k % 10 == 0:
        kind, data = K.ECEF_POS, [cpu.x[:3] + rng.normal(0, 1.0, 3)]
      elif k % 10 == 5:
        kind, data = K.CAMERA_ODO_TRANSLATION, [np.concatenate([rng.normal(0, 0.1, 3), [0.1, 0.1, 0.1]])]
      elif k % 10 == 7:
        kind, data = K.ODOMETRIC_SPEED, [[0.0]]
      else:
        kind, data = (K.PHONE_GYRO if k % 2 else K.PHONE_ACCEL), [rng.normal(0, 0.01, 3) + (0.0 if k % 2 else np.array([0, 0, -9.8]))]
      rg, rc = gpu.predict_and_observe(t, kind, data), cpu.predict_and_observe(t, kind, data)
      assert rg is not None and rc is not None
      # measured on an H100: worst 1.1e-9 (state), 2.4e-10 (covariance)
      assert state_err(gpu.x, cpu.x) < 1e-8 and cov_err(gpu.P, cpu.P) < 1e-8, (k, int(kind))


def test_rewinding_scheduler_on_the_device(gen_dir, oracle_dir, monkeypatch):
  """Late observations rewind and fast-forward per filter (rednose/helpers/ekf_sym.py:418-482) through the device ring
  of RewindingScheduler; reference: one Python-driver instance per filter on the reference-generated CPU library.
  (tests/test_scheduler_cpu.py runs the same stream bit-for-bit against the CPU oracle engine.)"""
  import rednose_b200.ekf_sym as drv
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RewindingScheduler
  depth = 32
  monkeypatch.setattr(drv, "REWIND_TO_KEEP", depth)
  B, zd = 5, {3: 1, 4: 3, 10: 3, 12: 3}
  rng = np.random.default_rng(7)
  x0 = np.tile(LiveKalman.initial_x, (B, 1)); x0[:, :3] += rng.normal(0, 10.0, (B, 3))
  P0 = np.tile(np.diag(LiveKalman.initial_P_diag), (B, 1, 1))
  Rk = {3: np.array([[0.2**2]]), 4: np.eye(3) * 0.025**2, 10: np.eye(3) * 0.5**2, 12: np.eye(3) * 25.0}
  refs = [drv.EKF_sym(oracle_dir, "live", LiveKalman.Q, x0[b], P0[b], 23, 22, quaternion_idxs=[3], max_rewind_age=0.5) for b in range(B)]
  e = _engine(gen_dir, "live", x0, P0, LiveKalman.Q, quaternion_idxs=[3], norm_after_predict=False)
  s = RewindingScheduler(e, zd, depth=depth, max_rewind_age=0.5)
  ref_dropped = 0
  for tick in range(70):
    now = 0.01 * (tick + 1)
    ids, ts, ks, zs = [], [], [], {k: [] for k in zd}
    for b in range(B):
      if rng.random() < 0.25:
        continue
      u, tb = rng.random(), now + 1e-4 * b
      if tick > 5 and u < 0.15:
        tb -= rng.uniform(0.011, 0.06)
      elif tick > 5 and u < 0.20:
        tb -= 3.0
      k = int(rng.choice([4, 10, 10, 4, 3 if tick > 12 else 4, 12]))
      zb = {3: np.array([0.1]), 4: rng.normal(0, 0.01, 3), 10: rng.normal(0, 0.1, 3) + [0, 0, -9.8], 12: refs[b].state()[:3] + rng.normal(0, 1.0, 3)}[k]
      ids.append(b); ts.append(tb); ks.append(k); zs[k].append(zb)
      if refs[b].predict_and_update_batch(tb, k, zb[None], Rk[k][None]) is None:
        ref_dropped += 1
    if ids:
      s.tick(np.array(ids), np.array(ts), np.array(ks), {k: np.array(v) for k, v in zs.items() if v}, Rk)
  assert s.dropped == ref_dropped and s.rewinds > 10 and s.replayed > s.rewinds
  ex = state_err(e.state(), np.stack([r.state() for r in refs]))
  eP = cov_err(e.covs(), np.stack([r.covs() for r in refs]))
  assert ex < 2e-9 and eP < 2e-9, (ex, eP)     # measured on an H100: 1.8e-10, 1.7e-10
  for b in range(B):
    assert int(s.cnt[b]) == len(refs[b].rewind_t) and abs(float(s.t_filter[b]) - refs[b].filter_time) < 1e-12


def test_msckf_cuda_path_reproduces_reference_golden_vectors(gen_dir):
  """tests/golden/msckf_reference.npz (reference numpy maths: block predict, SVD null-space projection + gate, augment):
  the CTA-per-filter kernels (Householder projection) must land on the same x and P at every step, through the
  batched C-ABI with the Python driver's normalisation order (ekf_sym.py:505-531)."""
  import os
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import DIM_STATE
  from rednose_b200.filters.msckf import N_CLONES, MsckfKalman
  d = ensure_generated(MsckfKalman)
  g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "msckf_reference.npz"))
  feat = int(MsckfKalman.feature_kind)
  quats = [3] + [DIM_STATE + 3 + 7 * c for c in range(N_CLONES)]
  e = BatchedEKF(d, "msckf", g["Q"], g["x0"], g["P0"], quaternion_idxs=quats, norm_after_predict=False)
  t_prev = float(g["t"][0])
  for k, kind in enumerate(g["kinds"]):
    kind = int(kind)
    m = 2 * N_CLONES if kind == feat else 3
    z = np.stack([g[f"z{b}"][k, :m] for b in range(2)])
    R = np.stack([np.diag(g[f"Rdiag{b}"][k, :m]) for b in range(2)])
    e.step(kind, float(g["t"][k]) - t_prev, z, R, ea=g["point"] if kind == feat else None)
    t_prev = float(g["t"][k])
    if g["augment"][k]:
      e.augment()
    ex = state_err(e.state(), np.stack([g[f"xk{b}"][k] for b in range(2)]))
    eP = cov_err(e.covs(), np.stack([g[f"Pk{b}"][k] for b in range(2)]))
    assert ex < TIGHT and eP < TIGHT, (k, kind, ex, eP)
    assert quat_norm_err(e.state(), quats) <= QN, k          # the main quaternion and all 10 clones


@pytest.mark.parametrize("norm_quats", [False, True])
def test_checkpointed_smoother_equals_full_history(gen_dir, oracle_dir, norm_quats):
  """BASELINE config 4's plan in miniature: checkpoints every `segment` steps, segments re-filtered with history and
  smoothed last to first through <name>_batch_rts_segment == one backward pass over the whole stored history, bit for bit."""
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother
  o = Oracle(oracle_dir, "live")
  B, T = 29, 37
  x, P, Qm = live_batch(B, seed=310)
  kinds = [12 if k % 7 == 0 else (4 if k % 2 else 10) for k in range(T)]
  zs = [live_obs(o, kinds[k], x, seed=700 + k) for k in range(T)]

  def obs_fn(k, lo, hi):
    return 0.01 * (k + 1), kinds[k], zs[k][0][lo:hi].copy(), zs[k][1][lo:hi]

  ref = {}
  TiledSmoother(gen_dir, "live", Qm, 23, 22, quaternion_idxs=[3], tile=64).run(
    x, P, T, obs_fn, lambda lo, hi, xs, Ps: ref.update(a=(xs.cpu().numpy().copy(), Ps.cpu().numpy().copy())), norm_quats=norm_quats)
  for segment, tile in ((8, 16), (5, 64), (64, 64)):
    xs_all, Ps_all = np.full((T, B, 23), np.nan), np.full((T, B, 22, 22), np.nan)
    def sink(lo, hi, k0, xs, Ps):
      n = xs.shape[0]
      assert np.isnan(xs_all[k0:k0 + n, lo:hi]).all()                     # every (step, filter) delivered exactly once
      xs_all[k0:k0 + n, lo:hi], Ps_all[k0:k0 + n, lo:hi] = xs.cpu().numpy(), Ps.cpu().numpy()
    cs = CheckpointedSmoother(gen_dir, "live", Qm, 23, 22, quaternion_idxs=[3], segment=segment, tile=tile)
    cs.run(x, P, T, obs_fn, sink, norm_quats=norm_quats)
    assert np.array_equal(xs_all, ref["a"][0]) and np.array_equal(Ps_all, ref["a"][1]), (segment, tile)
  assert cs.bytes_per_filter(10_000) < 81_200_000 / 20                     # vs 81 MB of full history per live filter


def test_tiled_smoother_two_passes_equal_two_oracle_passes(gen_dir, oracle_dir):
  """README.md:41-45 "multiple forward and backwards passes": pass 2 restarts the forward filter from pass 1's smoothed
  first step.  Oracle: forward (restated ekf_c.c) + backward (restated ekf_sym.py:651-690), twice."""
  from oracle.rts_numpy import rts_smooth
  from rednose_b200.smoothing import TiledSmoother
  o = Oracle(oracle_dir, "live")
  B, T = 6, 14
  x, P, Qm = live_batch(B, seed=320)
  kinds = [12 if k % 5 == 0 else (4 if k % 2 else 10) for k in range(T)]
  zs = [live_obs(o, kinds[k], x, seed=800 + k) for k in range(T)]
  ts = [0.01 * (k + 1) for k in range(T)]

  def oracle_pass(x0, P0):
    xp, Pp, xf, Pf = [], [], [], []
    xc, Pc, t_prev = x0.copy(), P0.copy(), 0.0
    for k in range(T):
      a, b_ = o.predict(xc, Pc, Qm, ts[k] - t_prev)
      for q in a:
        q[3:7] /= np.linalg.norm(q[3:7])
      xp.append(a.copy()); Pp.append(b_.copy())
      xc, Pc, _ = o.update(kinds[k], a, b_, zs[k][0], zs[k][1])
      for q in xc:
        q[3:7] /= np.linalg.norm(q[3:7])
      xf.append(xc.copy()); Pf.append(Pc.copy())
      t_prev = ts[k]
    xs, Ps = zip(*[rts_smooth(o, np.stack(xp)[:, b], np.stack(xf)[:, b], np.stack(Pp)[:, b], np.stack(Pf)[:, b], np.array(ts), 23, 22, norm_quats=True) for b in range(B)])
    return np.stack(xs, 1), np.stack(Ps, 1)

  xs1, Ps1 = oracle_pass(x, P)
  xs2, Ps2 = oracle_pass(xs1[0], Ps1[0])
  got = {}
  ts_ = TiledSmoother(gen_dir, "live", Qm, 23, 22, quaternion_idxs=[3], tile=8)
  ts_.run(x, P, T, lambda k, lo, hi: (ts[k], kinds[k], zs[k][0][lo:hi].copy(), zs[k][1][lo:hi]),
          lambda lo, hi, xs, Ps: got.update(a=(xs.cpu().numpy().copy(), Ps.cpu().numpy().copy())), norm_quats=True, passes=2)
  assert state_err(got["a"][0], xs2) < TIGHT and cov_err(got["a"][1], Ps2) < TIGHT
  assert state_err(xs2, xs1) > 1e-9                                        # the second pass did change the estimate


def test_rts_on_an_ill_conditioned_history(gen_dir, oracle_dir):
  """SURVEY.md section 7.4: from the example's own P0 (variances 1e8 .. 1e-4) and an IMU-only stretch (no position fix)
  cond(P_{k+1|k}) ~ 1e12; LDL^T here vs numpy's LU in the oracle are both backward stable but differ at the 1e-7 level
  there.  Tolerances are therefore reported separately: per-array max-norm 1e-5 on this stretch (the reference's own
  np.allclose rtol, examples/test_compare.py:119-120) against 1e-6 on well-conditioned histories."""
  from oracle.rts_numpy import rts_smooth
  o = Oracle(oracle_dir, "live")
  B, T = 12, 60
  x, P, Qm = live_batch(B, seed=330, well_conditioned=False)
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  hist = e.new_history(T)
  for k in range(T):
    kind = 4 if k % 2 else 10                                              # gyro / accelerometer only
    z, R = live_obs(o, kind, e.state() if k else x, seed=900 + k)
    e.step_recorded(hist, kind, 0.01 * (k + 1), z, R)
  hx_p, hx_f = hist.x_pred.cpu().numpy(), hist.x_filt.cpu().numpy()
  hP_p, hP_f = hist.P_pred.cpu().numpy(), hist.P_filt.cpu().numpy()
  cond = max(np.linalg.cond(hP_p[k, b]) for k in (1, T // 2, T - 1) for b in range(B))
  assert cond > 1e10, cond
  xs, Ps = e.rts_smooth(hist, norm_quats=True)
  xs, Ps = xs.cpu().numpy(), Ps.cpu().numpy()
  worst_x = worst_P = 0.0
  for b in range(B):
    xr, Pr = rts_smooth(o, hx_p[:, b], hx_f[:, b], hP_p[:, b], hP_f[:, b], hist.t_host.copy(), 23, 22, norm_quats=True)
    worst_x, worst_P = max(worst_x, state_err(xs[:, b], xr)), max(worst_P, cov_err(Ps[:, b], Pr))
  print(f"ill-conditioned RTS (cond {cond:.1e}): x {worst_x:.2e} P {worst_P:.2e}")
  assert worst_x < TIGHT and worst_P < TIGHT, (worst_x, worst_P)   # measured on an H100: 5.4e-11, 1.2e-10
  assert np.isfinite(Ps).all() and np.all(np.diagonal(Ps, axis1=2, axis2=3) > 0)


def test_full_size_1m_kinematic_sampled_oracle(gen_dir, oracle_dir):
  """BASELINE.json config 2 at size: 1 048 576 kinematic filters, 20 fused steps; every 997th filter against the oracle."""
  o = Oracle(oracle_dir, "kinematic")
  B = 1 << 20
  x, P, Qm, _, R = kinematic_batch(B, seed=91)
  e = _engine(gen_dir, "kinematic", x, P, Qm)
  sel = np.arange(0, B, 997)
  xr, Pr = x[sel].copy(), P[sel].copy()
  rng = np.random.default_rng(92)
  Rd = torch.as_tensor(R).cuda()
  for k in range(20):
    z = rng.normal(0.5, 0.3, (B, 1))
    e.step(1, 0.01, torch.as_tensor(z).cuda(), Rd)
    xr, Pr, _ = o.batch_step(1, xr, Pr, Qm, 0.01, z[sel], R[sel])
  gx, gP = e.state(), e.covs()
  assert state_err(gx[sel], xr) < TIGHT and cov_err(gP[sel], Pr) < TIGHT
  assert np.isfinite(gx).all() and np.all(gP[:, 0, 0] > 0) and np.all(gP[:, 1, 1] > 0)
  assert float(np.max(np.abs(gP[:, 0, 1] - gP[:, 1, 0]))) < 1e-12


def test_cuda_graph_replay_equals_eager_stepping(gen_dir, oracle_dir):
  """BatchedEKF.capture: a captured sequence of fused steps (live, kinds 4 / 10 / 12; kinematic) replays bit-identically."""
  o = Oracle(oracle_dir, "live")
  B = 3000
  x, P, Qm = live_batch(B, seed=410)
  kinds = [12, 4, 10, 4, 10, 4]
  zs = {k: live_obs(o, k, x[:64], seed=20 + k) for k in set(kinds)}
  zd = {k: torch.as_tensor(np.tile(zs[k][0], (B // 64 + 1, 1))[:B]).cuda() for k in zs}
  Rd = {k: torch.as_tensor(np.diag(np.diag(zs[k][1][0]))).cuda() for k in zs}
  dt = torch.full((B,), 0.01, dtype=torch.float64, device="cuda")

  def run(e, zw):
    for k in kinds:
      zw[k][:, 0, :].copy_(zd[k])
      e.step(k, dt, zw[k], Rd[k])

  e1 = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  e2 = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  zw1 = {k: torch.empty(B, 1, 3, dtype=torch.float64, device="cuda") for k in zs}
  zw2 = {k: torch.empty(B, 1, 3, dtype=torch.float64, device="cuda") for k in zs}
  run(e1, zw1); run(e1, zw1)
  x0, P0 = e2.x.clone(), e2.P.clone()
  g = e2.capture(lambda: run(e2, zw2))
  e2.x.copy_(x0); e2.P.copy_(P0)
  g.replay(); g.replay()
  torch.cuda.synchronize()
  assert torch.equal(e1.x, e2.x) and torch.equal(e1.P, e2.P) and all(torch.equal(zw1[k], zw2[k]) for k in zs)


def test_host_streamer_selected_columns_and_decimation(gen_dir):
  """HostStreamer(out_cols=..., every=...): only the asked-for state columns come back, and only every `every`-th step;
  the filter itself is unaffected (same P and x as direct stepping)."""
  from rednose_b200.streaming import HostStreamer
  B, T = 2053, 6
  x, P, Qm = live_batch(B, seed=93)
  rng = np.random.default_rng(4)
  R4 = torch.as_tensor(np.diag([0.025**2] * 3)).cuda()
  zs = [torch.as_tensor(rng.normal(0, 0.01, (B, 3))).pin_memory() for _ in range(T)]
  a = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  b = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  cols = [0, 1, 2, 3, 4, 5, 6]
  st = HostStreamer(b, {4: 3}, out_cols=cols, every=2)
  a.filter_time = b.filter_time = 0.0
  for k, z in enumerate(zs):
    t = 0.01 * (k + 1)
    xa, ya = a.predict_and_update_batch(t, 4, z, R4)
    tk = st.submit(t, 4, z, R4)
    xh, yh = st.result(tk, 4)
    assert xh.shape == (B, 7) and torch.equal(yh, ya.cpu()[:, 0])
    if k % 2 == 0:
      assert torch.equal(xh, xa.cpu()[:, cols])
  assert torch.equal(a.P, b.P) and torch.equal(a.x, b.x)
  assert st.d2h_bytes == 8 * B * (7 * 3 + 3 * T)


def test_forward_filter_is_bit_reproducible_run_to_run(gen_dir):
  """Regression for a cross-proxy write-after-read race found in round 2: the bulk copy (async proxy) that refills a
  covariance-tile slot could overtake the still-queued shared-memory loads (generic proxy) of the previous pair, about
  once in 1e7 filter-steps -- invisible to single-step parity tests, visible as run-to-run differences of long histories
  (and, rarely, a non-finite smoothed covariance).  65 536 filters x 100 steps x 6 runs: every run must equal the first."""
  B, T = 65536, 100
  rng = np.random.default_rng(5)
  x, P, Qm = live_batch(4096, seed=500)
  x, P = np.tile(x, (16, 1)), np.tile(P, (16, 1, 1))
  e = _engine(gen_dir, "live", x, P, Qm, quaternion_idxs=[3])
  x0, P0 = e.x.clone(), e.P.clone()
  z = {4: torch.as_tensor(rng.normal(0, 0.02, (2, B, 3))).cuda(), 10: torch.as_tensor(rng.normal(0, 0.3, (2, B, 3)) + [0, 0, -9.8]).cuda(),
       12: (e.x[:, :3] + torch.as_tensor(rng.normal(0, 3.0, (B, 3))).cuda())[None].repeat(2, 1, 1)}
  R = {4: torch.eye(3, dtype=torch.float64, device="cuda") * 0.025**2, 10: torch.eye(3, dtype=torch.float64, device="cuda") * 0.25,
       12: torch.eye(3, dtype=torch.float64, device="cuda") * 25.0}
  def run():
    e.x.copy_(x0); e.P.copy_(P0)
    for k in range(T):
      kind = 12 if k % 50 == 0 else (4 if k % 2 else 10)
      e.step(kind, 0.01, z[kind][k % 2].clone(), R[kind])
    return e.x.clone(), e.P.clone()

  torch.cuda.empty_cache()
  ref = run()
  assert bool(torch.isfinite(ref[1]).all())
  for r in range(5):
    got = run()
    for name, a, b in zip(("x", "P"), ref, got):   # a glitch anywhere changes the rest of that filter's trajectory
      assert torch.equal(a, b), (r, name, (a != b).nonzero()[0].tolist())
