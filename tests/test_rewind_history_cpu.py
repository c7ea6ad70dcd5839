"""Histories recorded under RewindingScheduler, without a GPU: the C-ABI of the restore-from-history entry point and its
argument checks (all made before any CUDA call), RaggedHistory.rewind, and the scheduler's semantics with a history --
same state and counters as without one, and per-filter rows equal to what the reference driver returns for the same
observations in time order -- against a CPU stand-in engine that records and restores like the kernels."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from rednose_b200.batched import BatchedEKF
from tests.shapes import SHAPES

CUDA_INVALID_VALUE, CUDA_NOT_SUPPORTED = 1, 801
PACKED_P, PACKED_HIST = 32, 64


def _filters():
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  return [KinematicKalman, LiveKalman] + list(SHAPES)


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


# ------------------------------------------------------------------------------------------------------------ C-ABI ---
@pytest.mark.parametrize("cls", _filters(), ids=lambda c: c.name)
def test_headers_declare_and_libraries_export_restore_hist(cls):
  from rednose_b200.filters import ensure_generated
  folder = ensure_generated(cls)
  with open(os.path.join(folder, f"{cls.name}.h"), encoding="utf-8") as f:
    protos = [ln for ln in f.read().split("\n") if re.match(rf"(void|int) {cls.name}_batch_restore_hist\(", ln)]
  assert protos == [f"int {cls.name}_batch_restore_hist(const double *hx_filt, const double *hP_filt, const int *idx, "
                    "const int *hist_row, long long n, long long hist_B, double *x, double *P, int flags, void *stream);"]
  assert hasattr(ctypes.CDLL(os.path.join(folder, f"lib{cls.name}.so")), f"{cls.name}_batch_restore_hist")


def test_include_header_declares_the_restore_typedef_in_c(tmp_path):
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "t.c"
  src.write_text('#include "rednose_b200.h"\n'
                 "int main(void){ rednose_batch_restore_hist_fn f = 0; (void)f; return 0; }\n")
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{INCLUDE_DIR}", "-c", str(src), "-o", str(tmp_path / "t.o")], check=True)


def _restore(cls, **kw):
  """Call <name>_batch_restore_hist with valid one-entry arguments overridden by `kw`; returns (status, latched status)."""
  ffi, lib = _lib(cls)
  name = cls.name
  getattr(lib, f"{name}_cuda_status")()
  buf = ffi.new("double[]", 64 * 64)
  a = dict(hx=buf, hP=buf, idx=ffi.new("int[]", [0]), rows=ffi.new("int[]", [0]), n=1, hist_B=1, x=buf, P=buf, flags=0)
  a.update({k: (ffi.NULL if v is None else v) for k, v in kw.items()})
  st = getattr(lib, f"{name}_batch_restore_hist")(a["hx"], a["hP"], a["idx"], a["rows"], a["n"], a["hist_B"], a["x"], a["P"],
                                                  a["flags"], ffi.NULL)
  return st, getattr(lib, f"{name}_cuda_status")()


def test_restore_rejects_bad_arguments_before_any_cuda_call():
  """Every case returns its status without touching the device (so it runs here without one) and latches it."""
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.shapes import BY_NAME
  for cls in (KinematicKalman, BY_NAME["shape_e7"]):        # the pair kernel does not serve these: no packed layouts
    for flags in (PACKED_P, PACKED_HIST, PACKED_P | PACKED_HIST):
      assert _restore(cls, flags=flags) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED), (cls.name, flags)
  assert _restore(MsckfKalman) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED)   # EDIM 82: ragged histories are refused
  assert _restore(MsckfKalman, n=0) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED)
  for arg in ("hx", "hP", "idx", "rows", "x", "P"):
    assert _restore(LiveKalman, **{arg: None}) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE), arg
  assert _restore(LiveKalman, hist_B=0) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  assert _restore(LiveKalman, n=-1) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  none = dict(hx=None, hP=None, idx=None, rows=None, x=None, P=None)
  for cls, flags in ((LiveKalman, PACKED_P | PACKED_HIST), (LiveKalman, 0), (KinematicKalman, 0)):
    assert _restore(cls, n=0, flags=flags, **none) == (0, 0)   # valid and empty: nothing to launch


def test_ragged_history_rewind_sets_n_and_keeps_overflow():
  from rednose_b200.batched import RaggedHistory
  h = RaggedHistory(3, 4, 2, 2, "cpu")
  for _ in range(4):
    h.reserve(torch.tensor([0, 1]), 0.5)
  h.reserve(torch.tensor([2]), 0.5)
  assert h.n.tolist() == [3, 3, 1, 0] and h.overflowed() == 2
  h.rewind(torch.tensor([1, 2]), torch.tensor([0, 0], dtype=torch.int32))
  assert h.n.tolist() == [3, 1, 1, 0] and h.n.dtype == torch.int32 and h.overflowed() == 2
  assert h.reserve(torch.tensor([1, 0]), 0.75).tolist() == [1, -1]                # the next row after the rewound one


# --------------------------------------------------------------------------------------------- scheduler semantics ---
class _RecordingOracleEngine:
  """BatchedEKF's surface (x, P, step_indexed with and without hist=, restore_from_history) computing on the CPU oracle
  library one filter at a time with the reference driver's calls (predict, update, normalise after the update),
  writing the history slabs at the rows RaggedHistory.reserve hands out and restoring x / P from x_filt / P_filt rows
  -- what the recording and restoring kernels do on the device.  rts_smooth is BatchedEKF's own: with a RaggedHistory
  that overflowed it raises before any launch."""
  rts_smooth = BatchedEKF.rts_smooth
  _rts_smooth_ragged = BatchedEKF._rts_smooth_ragged

  def __init__(self, oracle, x, P, Q):
    self.o, self.Q = oracle, Q
    self.x, self.P = torch.as_tensor(x.copy()), torch.as_tensor(P.copy())
    self.B, self.dim_err, self.device = x.shape[0], P.shape[1], torch.device("cpu")
    self.restores = 0

  def step_indexed(self, kind, idx, dt, z, R, ea=None, hist=None, t=None):
    if idx.numel() == 0:
      return None
    rows = hist.reserve(idx, t) if hist is not None else None
    ys = []
    for e, b in enumerate(idx.tolist()):
      xp, Pp = self.o.predict(self.x[b].numpy()[None], self.P[b].numpy()[None], self.Q, float(dt[e]))
      Re = R.numpy() if R.ndim == 2 else R[e].numpy()
      xf, Pf, y = self.o.update(kind, xp, Pp, z[e].numpy().reshape(1, -1), Re[None])
      xf[0, 3:7] /= np.linalg.norm(xf[0, 3:7])
      if rows is not None and int(rows[e]) >= 0:
        r = int(rows[e])
        hist.x_pred[r, b], hist.P_pred[r, b] = torch.as_tensor(xp[0]), torch.as_tensor(Pp[0])
        hist.x_filt[r, b], hist.P_filt[r, b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      self.x[b], self.P[b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      ys.append(y[0])
    return torch.as_tensor(np.array(ys)).reshape(len(ys), 1, -1)

  def restore_from_history(self, hist, ids, rows):
    for b, r in zip(ids.tolist(), rows.tolist()):
      if r >= 0:
        self.x[b], self.P[b] = hist.x_filt[r, b], hist.P_filt[r, b]
    self.restores += 1


ZD = {3: 1, 4: 3, 10: 3, 12: 3}
RK = {3: np.array([[0.2**2]]), 4: np.eye(3) * 0.025**2, 10: np.eye(3) * 0.5**2, 12: np.eye(3) * 25.0}


def _initial(B, seed):
  """The rng and initial states of the live stream of the rewinding-scheduler tests."""
  from rednose_b200.filters.live import LiveKalman
  rng = np.random.default_rng(seed)
  x0 = np.tile(LiveKalman.initial_x, (B, 1)); x0[:, :3] += rng.normal(0, 10.0, (B, 3))
  P0 = np.tile(np.diag(LiveKalman.initial_P_diag), (B, 1, 1))
  return rng, x0, P0


def _run(oracle_dir, depth, monkeypatch, seed, T=256):
  """The live stream of the rewinding-scheduler tests (per tick each filter observes, with p = 0.75, one of kinds 3 / 4 /
  10 / 12; after tick 5 about 15 % of the observations are 11-60 ms late, a rewind over 1-6 checkpoints, and 5 % are 3 s
  late, ignored) through a per-filter reference driver, RewindingScheduler without a history and RewindingScheduler with
  one, checking that every tick returns the same innovations from both.  Returns (drivers, applied observations per filter, (scheduler, engine) x 2, history)."""
  import rednose_b200.ekf_sym as drv
  from rednose_b200.batched import RaggedHistory
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RewindingScheduler
  from tests.util import Oracle
  monkeypatch.setattr(drv, "REWIND_TO_KEEP", depth)          # the reference keeps 512 (ekf_sym.py:447); same ring size on both sides
  B = 5
  rng, x0, P0 = _initial(B, seed)
  o = Oracle(oracle_dir, "live")
  refs = [drv.EKF_sym(oracle_dir, "live", LiveKalman.Q, x0[b], P0[b], 23, 22, quaternion_idxs=[3], max_rewind_age=0.5) for b in range(B)]
  e0, e1 = _RecordingOracleEngine(o, x0, P0, LiveKalman.Q), _RecordingOracleEngine(o, x0, P0, LiveKalman.Q)
  hist = RaggedHistory(T, B, 23, 22, "cpu")
  s0 = RewindingScheduler(e0, ZD, depth=depth, max_rewind_age=0.5)
  s1 = RewindingScheduler(e1, ZD, depth=depth, max_rewind_age=0.5, history=hist)
  applied = [[] for _ in range(B)]                          # (t, kind, z) the reference driver applied, in arrival order
  for tick in range(70):
    now = 0.01 * (tick + 1)
    ids, ts, ks, zs = [], [], [], {k: [] for k in ZD}
    for b in range(B):
      if rng.random() < 0.25:
        continue
      u = rng.random()
      tb = now + 1e-4 * b
      if tick > 5 and u < 0.15:
        tb -= rng.uniform(0.011, 0.06)
      elif tick > 5 and u < 0.20:
        tb -= 3.0
      k = int(rng.choice([4, 10, 10, 4, 3 if tick > 12 else 4, 12]))   # the speed observation is singular at v = 0
      zb = {3: np.array([0.1]), 4: rng.normal(0, 0.01, 3), 10: rng.normal(0, 0.1, 3) + [0, 0, -9.8], 12: refs[b].state()[:3] + rng.normal(0, 1.0, 3)}[k]
      ids.append(b); ts.append(tb); ks.append(k); zs[k].append(zb)
      if refs[b].predict_and_update_batch(tb, k, zb[None], RK[k][None]) is not None:
        applied[b].append((tb, k, zb))
    if ids:
      args = (np.array(ids), np.array(ts), np.array(ks), {k: np.array(v) for k, v in zs.items() if v}, RK)
      y0, y1 = s0.tick(*args), s1.tick(*args)
      assert y0.keys() == y1.keys()
      for k in y0:
        assert torch.equal(y0[k][0], y1[k][0]) and torch.equal(y0[k][1], y1[k][1])
  return refs, applied, (s0, e0), (s1, e1), hist


def _in_order_estimates(oracle_dir, x0, P0, applied):
  """EKF_sym.predict_and_update_batch over one filter's applied observations sorted by time (stably: an observation
  that arrived later at the same time goes after, as bisect_right puts a late one behind its checkpoint)."""
  import rednose_b200.ekf_sym as drv
  from rednose_b200.filters.live import LiveKalman
  ref = drv.EKF_sym(oracle_dir, "live", LiveKalman.Q, x0, P0, 23, 22, quaternion_idxs=[3], max_rewind_age=0.5)
  est = [ref.predict_and_update_batch(t, k, z[None], RK[k][None]) for t, k, z in sorted(applied, key=lambda a: a[0])]
  assert all(e is not None for e in est)
  return ref, est


@pytest.mark.parametrize("seed,depth", [(7, 64), (11, 4)])
def test_rewinding_history_equals_the_in_order_reference(oracle_dir, monkeypatch, seed, depth):
  """State, clocks, ring and counters equal the scheduler without a history (innovations of every tick too), and each
  filter's rows, smoothed by oracle/rts_numpy, equal the reference driver fed the same observations in time order."""
  from oracle.rts_numpy import rts_smooth
  from tests.util import Oracle
  refs, applied, (s0, e0), (s1, e1), hist = _run(oracle_dir, depth, monkeypatch, seed)
  assert s1.rewinds > 5 and s1.replayed > s1.rewinds and s1.dropped > 3 and s1.unrecorded == 0
  assert (s0.rewinds, s0.replayed, s0.dropped) == (s1.rewinds, s1.replayed, s1.dropped)
  assert e1.restores > 0 and torch.equal(e0.x, e1.x) and torch.equal(e0.P, e1.P)
  assert torch.equal(s0.t_filter, s1.t_filter) and torch.equal(s0.cnt, s1.cnt) and torch.equal(s0.head, s1.head)
  assert not hasattr(s1, "ring_x") and not hasattr(s1, "ring_P") and s1.ring_row.dtype == torch.int32
  assert hist.overflowed() == 0
  o = Oracle(oracle_dir, "live")
  _, x0, P0 = _initial(5, seed)
  for b in range(5):
    ref, est = _in_order_estimates(oracle_dir, x0[b], P0[b], applied[b])
    k = int(hist.n[b])
    assert k == len(est) == len(applied[b])
    assert np.array_equal(hist.t[:k, b].numpy(), [e[4] for e in est])
    slabs = [a[:k, b].numpy() for a in (hist.x_pred, hist.x_filt, hist.P_pred, hist.P_filt)]
    for r, e in enumerate(est):          # x_{k|k-1}, x_{k|k}, P_{k|k-1}, P_{k|k}: the driver's 9-tuple starts with them
      for got, want in zip(slabs, e[:4]):
        assert np.max(np.abs(got[r] - want)) <= 1e-12 * np.max(np.abs(want)), (b, r)
    xs, Ps = rts_smooth(o, *slabs, hist.t[:k, b].numpy(), 23, 22, norm_quats=True)
    xr, Pr = ref.rts_smooth([tuple(np.copy(a) if isinstance(a, np.ndarray) else a for a in e) for e in est], norm_quats=True)
    ex = np.max(np.abs(xs - xr)) / np.max(np.abs(xr))
    eP = np.max(np.abs(Ps - Pr)) / np.max(np.abs(Pr))
    assert ex < 1e-12 and eP < 1e-12, (b, ex, eP)


def test_history_with_packed_ring_or_another_batch_is_refused():
  from rednose_b200.batched import RaggedHistory
  from rednose_b200.scheduler import RewindingScheduler

  class Eng:
    B, dim_err, device, x = 3, 2, torch.device("cpu"), torch.zeros(3, 2)

  with pytest.raises(ValueError, match="packed"):
    RewindingScheduler(Eng(), {1: 2}, history=RaggedHistory(4, 3, 2, 2, "cpu"), packed=True)
  with pytest.raises(ValueError, match="4 filters"):
    RewindingScheduler(Eng(), {1: 2}, history=RaggedHistory(4, 4, 2, 2, "cpu"))
  s = RewindingScheduler(Eng(), {1: 2}, history=RaggedHistory(4, 3, 2, 2, "cpu"))
  assert s.ring_row.shape == (3, 16) and not hasattr(s, "ring_x")


def test_late_observation_behind_the_full_history_is_ignored_and_counted(oracle_dir):
  """Filter 0 fills its T rows, keeps stepping, then gets an observation late enough to rewind to a checkpoint stepped
  after the rows ran out: ignored (counted in .unrecorded, not .dropped).  One late enough for a recorded checkpoint is
  still applied.  rts_smooth refuses the history because it overflowed."""
  from rednose_b200.batched import RaggedHistory
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RewindingScheduler
  from tests.util import Oracle
  B, T = 2, 4
  x0 = np.tile(LiveKalman.initial_x, (B, 1))
  P0 = np.tile(np.diag(LiveKalman.initial_P_diag), (B, 1, 1))
  e = _RecordingOracleEngine(Oracle(oracle_dir, "live"), x0, P0, LiveKalman.Q)
  hist = RaggedHistory(T, B, 23, 22, "cpu")
  s = RewindingScheduler(e, ZD, depth=16, max_rewind_age=0.5, history=hist)
  z4 = np.array([[0.001, 0.002, 0.003]])
  for j in range(T + 3):                                    # rows 0 .. T-1 recorded, then 3 unrecorded steps
    s.tick([0], 0.01 * (j + 1), [4], {4: z4}, RK)
  assert hist.n.tolist() == [T, 0] and hist.overflowed() == 3
  assert s.ring_row[0, :T + 3].tolist() == [0, 1, 2, 3, -1, -1, -1]
  x_before, P_before = e.x.clone(), e.P.clone()
  s.tick([0], 0.055, [4], {4: z4}, RK)                       # checkpoint at 0.05: stepped with no row left
  assert s.unrecorded == 1 and s.dropped == 0 and s.rewinds == 0 and e.restores == 0
  assert torch.equal(e.x, x_before) and torch.equal(e.P, P_before) and hist.n.tolist() == [T, 0]
  s.tick([0], 0.035, [4], {4: z4}, RK)                       # checkpoint at 0.03: row 2
  assert s.unrecorded == 1 and s.rewinds == 1 and e.restores == 1 and s.replayed == 4
  assert hist.n.tolist() == [T, 0] and hist.overflowed() == 3 + 4   # rows 3 .. then four more steps with no row left
  with pytest.raises(RuntimeError, match="overflow"):
    e.rts_smooth(hist)
