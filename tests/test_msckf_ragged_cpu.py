"""MSCKF clone-window shifts for filters on their own clocks, without a GPU: the C-ABI of <name>_batch_augment_idx (which
libraries export it, its refusals, all made before any CUDA call), the schedulers' bookkeeping of augment flags, and
RewindingScheduler with and without a history over MSCKF streams with late camera frames, against a per-filter driver
that follows the reference's rewind rules except that a replayed observation keeps its augment flag."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from tests import msckf_long_shapes
from tests.msckf_shapes import MSCKF_SHAPES
from tests.shapes import SHAPES

CUDA_INVALID_VALUE, CUDA_NOT_SUPPORTED = 1, 801
PACKED_P, PACKED_HIST = 32, 64
QUATS = [3] + [23 + 3 + 7 * c for c in range(10)]     # shipped msckf: the main attitude and the 10 clone attitudes


def _filters():
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  from rednose_b200.filters.pendulum import PendulumKalman
  return ([KinematicKalman, LiveKalman, MsckfKalman, PendulumKalman] + list(SHAPES) + list(MSCKF_SHAPES)
          + list(msckf_long_shapes.SHAPES))


def _is_msckf(cls):
  from rednose_b200.filters.msckf import MsckfKalman
  return cls is MsckfKalman or cls in MSCKF_SHAPES or cls in msckf_long_shapes.SHAPES


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


# ------------------------------------------------------------------------------------------------------------ C-ABI ---
@pytest.mark.parametrize("cls", _filters(), ids=lambda c: c.name)
def test_msckf_headers_declare_and_libraries_export_augment_idx(cls):
  from rednose_b200.filters import ensure_generated
  folder = ensure_generated(cls)
  with open(os.path.join(folder, f"{cls.name}.h"), encoding="utf-8") as f:
    protos = [ln for ln in f.read().split("\n") if re.match(rf"(void|int) {cls.name}_batch_augment_idx\(", ln)]
  exported = hasattr(ctypes.CDLL(os.path.join(folder, f"lib{cls.name}.so")), f"{cls.name}_batch_augment_idx")
  if _is_msckf(cls):
    assert protos == [f"int {cls.name}_batch_augment_idx(double *x, double *P, const int *idx, long long n, int flags, void *stream);"]
    assert exported
  else:
    assert protos == [] and not exported


def test_include_header_declares_the_augment_idx_typedef_in_c(tmp_path):
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "t.c"
  src.write_text('#include "rednose_b200.h"\n'
                 "int main(void){ rednose_batch_augment_idx_fn f = 0; (void)f; return 0; }\n")
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{INCLUDE_DIR}", "-c", str(src), "-o", str(tmp_path / "t.o")], check=True)


def _augment_idx(cls, **kw):
  """Call <name>_batch_augment_idx with one-entry arguments overridden by `kw`; returns (status, latched status).  The
  pointers are host memory or NULL: every case here is decided before any CUDA call."""
  ffi, lib = _lib(cls)
  name = cls.name
  getattr(lib, f"{name}_cuda_status")()
  buf = ffi.new("double[]", 8)
  a = dict(x=buf, P=buf, idx=ffi.new("int[]", [0]), n=1, flags=0)
  a.update({k: (ffi.NULL if v is None else v) for k, v in kw.items()})
  st = getattr(lib, f"{name}_batch_augment_idx")(a["x"], a["P"], a["idx"], a["n"], a["flags"], ffi.NULL)
  return st, getattr(lib, f"{name}_cuda_status")()


@pytest.mark.parametrize("name", ["msckf", "msckf_e18", "msckf_e33"])
def test_augment_idx_rejects_bad_arguments_before_any_cuda_call(name):
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.msckf_shapes import BY_NAME
  cls = MsckfKalman if name == "msckf" else BY_NAME[name]
  assert _augment_idx(cls, n=-1) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  for arg in ("x", "P", "idx"):
    assert _augment_idx(cls, **{arg: None}) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE), arg
  for flags in (PACKED_P, PACKED_HIST, PACKED_P | PACKED_HIST):
    assert _augment_idx(cls, flags=flags) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED), flags
  assert _augment_idx(cls, n=0, x=None, P=None, idx=None) == (0, 0)       # valid and empty: nothing to launch


# ------------------------------------------------------------------------------------ scheduler bookkeeping (stub) ---
class _CallLog:
  """An engine surface that records every step_indexed call (kind, ids, keyword names, augment mask) and steps nothing.
  With `accepts_augment=False` its step_indexed has today's signature, without augment."""

  def __init__(self, B, accepts_augment=True):
    self.B, self.device, self.calls = B, torch.device("cpu"), []
    self.x, self.P = torch.zeros(B, 2, dtype=torch.float64), torch.zeros(B, 2, 2, dtype=torch.float64)
    if not accepts_augment:
      self.step_indexed = self._step_plain

  def _record(self, kind, idx, z, kw):
    self.calls.append((kind, idx.tolist(), sorted(kw), kw["augment"].tolist() if "augment" in kw else None))
    return z.reshape(z.shape[0], 1, -1)

  def step_indexed(self, kind, idx, dt, z, R, ea=None, **kw):
    return self._record(kind, idx, z, kw)

  def _step_plain(self, kind, idx, dt, z, R, ea=None, hist=None, t=None):
    return self._record(kind, idx, z, {} if hist is None else dict(hist=hist, t=t))


def _tick(s, t, augment=None):
  ids = np.array([0, 1, 2, 3, 4])
  kinds = np.array([4, 17, 4, 17, 17])
  z = {4: np.zeros((2, 3)), 17: np.zeros((3, 20))}
  R = {4: np.eye(3), 17: np.eye(20)}
  kw = {} if augment is None else dict(augment=augment)
  return s.tick(ids, t, kinds, z, R, {17: np.zeros((3, 3))}, **kw)


def test_unflagged_ticks_make_todays_calls():
  from rednose_b200.scheduler import RaggedScheduler
  for augment in (None, np.zeros(5, dtype=bool)):
    e = _CallLog(5, accepts_augment=False)
    s = RaggedScheduler(e)
    _tick(s, 0.1, augment)
    _tick(s, 0.2, augment)
    assert e.calls == [(4, [0, 2], [], None), (17, [1, 3, 4], [], None)] * 2


def test_flagged_entries_reach_their_kind_bucket_aligned():
  from rednose_b200.scheduler import RaggedScheduler
  e = _CallLog(5)
  s = RaggedScheduler(e)
  _tick(s, 0.1, np.array([False, True, False, False, True]))
  assert e.calls == [(4, [0, 2], [], None), (17, [1, 3, 4], ["augment"], [True, False, True])]


def test_dropped_observations_neither_step_nor_shift():
  from rednose_b200.scheduler import RaggedScheduler
  e = _CallLog(5)
  s = RaggedScheduler(e)
  _tick(s, np.array([0.2, 0.2, 0.2, 0.2, 0.2]))
  e.calls.clear()
  t = np.array([0.3, 0.1, 0.3, 0.3, 0.3])                           # filter 1's frame is late: dropped
  _tick(s, t, np.array([False, True, False, True, False]))
  assert s.dropped == 1
  assert e.calls == [(4, [0, 2], [], None), (17, [3, 4], ["augment"], [True, False])]
  e.calls.clear()
  _tick(s, np.array([0.4, 0.1, 0.4, 0.4, 0.4]), np.array([False, True, False, False, False]))   # the only flag dropped
  assert e.calls == [(4, [0, 2], [], None), (17, [3, 4], [], None)]


def test_rewinding_ring_keeps_the_augment_flags():
  from rednose_b200.scheduler import RewindingScheduler
  e = _CallLog(5)
  s = RewindingScheduler(e, {4: 3, 17: 20}, depth=4, ea_dims={17: 3})
  assert s.ring_aug.shape == (5, 4) and s.ring_aug.dtype == torch.bool
  _tick(s, 0.1, np.array([False, True, False, False, True]))
  assert s.ring_aug[:, 0].tolist() == [False, True, False, False, True]
  _tick(s, 0.2)                                                       # unflagged: today's calls, flags cleared
  assert s.ring_aug[:, 1].tolist() == [False] * 5 and all(c[2] == [] for c in e.calls[-2:])


# --------------------------------------------------------------------- RewindingScheduler against the driver (oracle) ---
@pytest.fixture(scope="module")
def msckf_oracle(oracle_dir):
  from oracle import build_ref
  if build_ref.reference_available():
    build_ref.build("msckf", "rednose_b200.filters.msckf:MsckfKalman")
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  return oracle_dir


def _shift(x, P):
  """The clone-window shift of the shipped msckf (ekf_sym.py:365-391) on one filter, as EKF_sym.augment does it."""
  from rednose_b200.filters.msckf import DIM_AUGMENT as d3, DIM_AUGMENT_ERR as d4
  d1, d2, E = 23, 22, P.shape[0]
  xr = x.clone()
  xr[d1:-d3] = x[d1 + d3:]
  xr[-d3:] = x[:d3]
  src = np.r_[0:d2, d2 + d4:E, 0:d4]
  return xr, P[np.ix_(src, src)].clone()


class _MsckfOracleEngine:
  """BatchedEKF's surface for an MSCKF (x, P, step_indexed with hist= and augment=, augment(ids), restore_from_history)
  computing on the CPU oracle one filter at a time with the driver's calls: predict, update, normalise every quaternion,
  then the shift of the flagged filters; a recorded row keeps the estimate before the shift."""

  def __init__(self, oracle, x, P, Q):
    self.o, self.Q = oracle, Q
    self.x, self.P = torch.as_tensor(x.copy()), torch.as_tensor(P.copy())
    self.B, self.dim_err, self.device = x.shape[0], P.shape[1], torch.device("cpu")
    self.shifts = self.restores = 0

  def step_indexed(self, kind, idx, dt, z, R, ea=None, hist=None, t=None, augment=False):
    if idx.numel() == 0:
      return None
    rows = hist.reserve(idx, t) if hist is not None else None
    aug = torch.as_tensor(augment).to(torch.bool).expand(idx.shape[0])
    ys = []
    for e, b in enumerate(idx.tolist()):
      xp, Pp = self.o.predict(self.x[b].numpy()[None], self.P[b].numpy()[None], self.Q, float(dt[e]))
      Re = R.numpy() if R.ndim == 2 else R[e].numpy()
      xf, Pf, y = self.o.update(kind, xp, Pp, z[e].numpy().reshape(1, -1), Re[None], None if ea is None else ea[e].numpy()[None])
      for q in QUATS:
        xf[0, q:q + 4] /= np.linalg.norm(xf[0, q:q + 4])
      if rows is not None and int(rows[e]) >= 0:
        r = int(rows[e])
        hist.x_pred[r, b], hist.P_pred[r, b] = torch.as_tensor(xp[0]), torch.as_tensor(Pp[0])
        hist.x_filt[r, b], hist.P_filt[r, b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      self.x[b], self.P[b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      if bool(aug[e]):
        self.x[b], self.P[b] = _shift(self.x[b], self.P[b])
      ys.append(y[0])
    return torch.as_tensor(np.array(ys)).reshape(len(ys), 1, -1)

  def augment(self, ids):
    for b in torch.as_tensor(ids).tolist():
      self.x[b], self.P[b] = _shift(self.x[b], self.P[b])
    self.shifts += 1

  def restore_from_history(self, hist, ids, rows):
    for b, r in zip(ids.tolist(), rows.tolist()):
      if r >= 0:
        self.x[b], self.P[b] = hist.x_filt[r, b], hist.P_filt[r, b]
    self.restores += 1


def _keep_flag_driver(folder, x0, P0):
  """The per-filter reference driver (rednose_b200.ekf_sym.EKF_sym), except that each checkpoint keeps its observation's
  augment flag, so a replay after a rewind shifts again where the observation did."""
  import rednose_b200.ekf_sym as drv
  from rednose_b200.filters.msckf import MsckfKalman

  class KeepFlag(drv.EKF_sym):
    def _predict_and_update_batch(self, t, kind, z, R, extra_args, augment=False):
      self._aug = augment
      return super()._predict_and_update_batch(t, kind, z, R, extra_args, augment)

    def checkpoint(self, obs):
      super().checkpoint(tuple(obs) + (self._aug,))

  return KeepFlag(folder, "msckf", MsckfKalman.Q, x0, P0, 23, 22, N=10, dim_augment=7, dim_augment_err=6,
                  maha_test_kinds=[17], quaternion_idxs=QUATS, max_rewind_age=0.5)


ZD, EAD = {4: 3, 17: 20}, {17: 3}
R4 = np.eye(3) * 0.025**2


def _run_rewinding(folder, depth, monkeypatch, seed, n_ticks=80, T=128):
  """Four msckf filters: a gyro sample (kind 4) at most ticks of 10 ms, a camera frame (kind 17, augment) every 5 ticks
  with a per-filter phase (filter 3 has none); after tick 8 half the frames arrive 1-3 ticks late, so each rewinds over
  gyro samples and sometimes over an earlier frame, and a quarter of the gyro samples 1-3 ticks late, some of them to the
  checkpoint of a frame.  Drives the keep-flag driver, RewindingScheduler without a history
  and RewindingScheduler with one, and checks that both schedulers return the same innovations every tick.  Returns
  (drivers, applied observations per filter, (scheduler, engine) x 2, history, x0, P0)."""
  import rednose_b200.ekf_sym as drv
  from rednose_b200.batched import RaggedHistory
  from rednose_b200.scheduler import RewindingScheduler
  from tests.util import Oracle, msckf_batch, msckf_feature_obs
  monkeypatch.setattr(drv, "REWIND_TO_KEEP", depth)
  B = 4
  rng = np.random.default_rng(seed)
  x0, P0, Q, point = msckf_batch(B, seed=seed)
  o = Oracle(folder, "msckf")
  zf, Rf, _ = msckf_feature_obs(o, x0, point, seed=seed, sigma=1e-3)
  refs = [_keep_flag_driver(folder, x0[b], P0[b]) for b in range(B)]
  e0, e1 = _MsckfOracleEngine(o, x0, P0, Q), _MsckfOracleEngine(o, x0, P0, Q)
  s0 = RewindingScheduler(e0, ZD, depth=depth, max_rewind_age=0.5, ea_dims=EAD)
  s1 = RewindingScheduler(e1, ZD, depth=depth, max_rewind_age=0.5, ea_dims=EAD, history=RaggedHistory(T, B, 93, 82, "cpu"))
  phase = [0, 2, 4, None]
  pending = [[] for _ in range(B)]
  applied = [[] for _ in range(B)]
  for tick in range(n_ticks):
    now = 0.01 * (tick + 1)
    obs = []
    for b in range(B):
      due = [p for p in pending[b] if p[0] <= tick]
      if due:
        pending[b].remove(due[0])
        obs.append((b,) + due[0][1:])
        continue
      if phase[b] is not None and tick % 5 == phase[b]:
        fr = (now + 1e-4 * b, 17, zf[b] + rng.normal(0, 1e-4, 20), Rf[b], point[b], True)
        if tick > 8 and rng.random() < 0.5:
          pending[b].append((tick + int(rng.integers(1, 4)),) + fr)
        else:
          obs.append((b,) + fr)
      elif rng.random() < 0.8:
        g = (now + 1e-4 * b, 4, rng.normal(0, 0.01, 3), R4, None, False)
        if tick > 8 and rng.random() < 0.25:                          # late too: it may rewind to a frame's checkpoint
          pending[b].append((tick + int(rng.integers(1, 4)),) + g)
        else:
          obs.append((b,) + g)
    if not obs:
      continue
    for b, tb, k, zb, Rb, eab, ab in obs:
      ea = [eab] if eab is not None else [[]]
      if refs[b].predict_and_update_batch(tb, k, zb[None], Rb[None], ea, augment=ab) is not None:
        applied[b].append((tb, k, zb, Rb, eab, ab))
    ids = np.array([o_[0] for o_ in obs])
    ts = np.array([o_[1] for o_ in obs])
    ks = np.array([o_[2] for o_ in obs])
    z = {k: np.array([o_[3] for o_ in obs if o_[2] == k]) for k in ZD if (ks == k).any()}
    R = {k: np.array([o_[4] for o_ in obs if o_[2] == k]) for k in ZD if (ks == k).any()}
    ea = {17: np.array([o_[5] for o_ in obs if o_[2] == 17])} if (ks == 17).any() else None
    aug = np.array([o_[6] for o_ in obs])
    y0, y1 = s0.tick(ids, ts, ks, z, R, ea, aug), s1.tick(ids, ts, ks, z, R, ea, aug)
    assert y0.keys() == y1.keys()
    for k in y0:
      assert torch.equal(y0[k][0], y1[k][0]) and torch.equal(y0[k][1], y1[k][1])
  return refs, applied, (s0, e0), (s1, e1), s1.history, x0, P0


def _close(got, want, tol=1e-12):
  return np.max(np.abs(np.asarray(got) - want)) <= tol * max(np.max(np.abs(want)), 1e-300)


@pytest.mark.parametrize("seed,depth", [(3, 64), (5, 4)])
def test_rewinding_msckf_stream_equals_the_keep_flag_driver(msckf_oracle, monkeypatch, seed, depth):
  """Without a history the final x / P of every filter equal the driver's; with one they are the same bit for bit, and
  each filter's rows equal the driver fed the same applied observations in time order (x_{k|k} before the shift)."""
  refs, applied, (s0, e0), (s1, e1), hist, x0, P0 = _run_rewinding(msckf_oracle, depth, monkeypatch, seed)
  assert s0.rewinds >= 4 and s0.replayed > s0.rewinds and s1.unrecorded == 0
  assert e0.shifts == 0 and e1.shifts > 0 and e1.restores > 0       # rewinds to a frame's checkpoint shift again
  assert (s0.rewinds, s0.replayed, s0.dropped) == (s1.rewinds, s1.replayed, s1.dropped)
  assert torch.equal(e0.x, e1.x) and torch.equal(e0.P, e1.P) and torch.equal(s0.t_filter, s1.t_filter)
  for b, ref in enumerate(refs):
    assert _close(e0.x[b].numpy(), ref.state()) and _close(e0.P[b].numpy(), ref.covs()), b
  assert hist.overflowed() == 0
  for b in range(4):
    ref = _keep_flag_driver(msckf_oracle, x0[b], P0[b])
    est = [ref.predict_and_update_batch(t, k, z[None], R[None], [ea] if ea is not None else [[]], augment=a)
           for t, k, z, R, ea, a in sorted(applied[b], key=lambda a: a[0])]
    k = int(hist.n[b])
    assert k == len(est)
    assert np.array_equal(hist.t[:k, b].numpy(), [e[4] for e in est])
    for r, e in enumerate(est):
      for got, want in zip((hist.x_pred, hist.x_filt, hist.P_pred, hist.P_filt), e[:4]):
        assert _close(got[r, b].numpy(), want), (b, r)
