"""Ragged histories without a GPU: the C-ABI of the per-filter recording step and the per-filter RTS pass, their
argument checks (all made before any CUDA call), RaggedHistory's row bookkeeping, and the row semantics of a history
recorded by RaggedScheduler, pinned to the reference driver (EKF_sym.predict_and_update_batch + rts_smooth per filter)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from tests.shapes import SHAPES

CUDA_INVALID_VALUE, CUDA_MISALIGNED, CUDA_NOT_SUPPORTED = 1, 716, 801


def _protos(folder, name):
  with open(os.path.join(folder, f"{name}.h"), encoding="utf-8") as f:
    return [ln for ln in f.read().split("\n") if ln.startswith(("void ", "int "))]


def _filters():
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  return [KinematicKalman, LiveKalman] + list(SHAPES)


@pytest.mark.parametrize("cls", _filters(), ids=lambda c: c.name)
def test_headers_declare_and_libraries_export_the_ragged_entry_points(cls):
  from rednose_b200.filters import ensure_generated
  folder = ensure_generated(cls)
  protos = _protos(folder, cls.name)
  lib = ctypes.CDLL(os.path.join(folder, f"lib{cls.name}.so"))
  steps = {int(m.group(1)) for p in protos if (m := re.match(rf"void {cls.name}_batch_step_(\d+)\(", p))}
  assert steps
  for k in steps:
    p = next(p for p in protos if p.startswith(f"int {cls.name}_batch_step_{k}_hist_idx("))   # int: the void set stays the reference's
    assert p.endswith("const int *idx, const int *hist_row, long long hist_B, void *stream);")
    assert hasattr(lib, f"{cls.name}_batch_step_{k}_hist_idx")
  p = next(p for p in protos if p.startswith(f"int {cls.name}_batch_rts_ragged("))
  assert "const double *t, const int *len, double *xs, double *Ps, int T, long long B" in p
  assert hasattr(lib, f"{cls.name}_batch_rts_ragged")


def test_include_header_declares_the_ragged_typedefs_in_c(tmp_path):
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "t.c"
  src.write_text('#include "rednose_b200.h"\n'
                 "int main(void){ rednose_batch_step_hist_idx_fn s = 0; rednose_batch_rts_ragged_fn r = 0; (void)s; (void)r; return 0; }\n")
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{INCLUDE_DIR}", "-c", str(src), "-o", str(tmp_path / "t.o")], check=True)


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


def test_recording_step_rejects_bad_arguments_before_any_cuda_call():
  """Every case returns its status without touching the device (so it runs here without one)."""
  from rednose_b200.filters.live import LiveKalman
  ffi, lib = _lib(LiveKalman)
  assert lib.live_cuda_status() == 0
  x, P, Q, z, R = (ffi.new("double[]", n) for n in (24, 22 * 22, 22 * 22, 4, 10))
  hx, hP = ffi.new("double[]", 24), ffi.new("double[]", 22 * 22 + 2)
  idx, rows = ffi.new("int[]", [0]), ffi.new("int[]", [0])
  good_q, bad_q = ffi.new("int[]", [3]), ffi.new("int[]", [20])

  def step(idx=idx, rows=rows, hist_B=1, q=good_q, hP_pred=hP, B=1):
    st = lib.live_batch_step_12_hist_idx(x, P, Q, ffi.NULL, 0.01, z, R, ffi.NULL, 1, B, q, 1, 3, hx, hP_pred, hx, hP, idx,
                                         rows, hist_B, ffi.NULL)
    assert lib.live_cuda_status() == st                   # returned and latched
    return st

  assert step(idx=ffi.NULL) == CUDA_INVALID_VALUE
  assert step(rows=ffi.NULL) == CUDA_INVALID_VALUE
  assert step(hist_B=0) == CUDA_INVALID_VALUE
  assert step(q=bad_q) == CUDA_INVALID_VALUE
  # the pair kernel stores covariance history rows with 128-bit accesses
  misaligned = ffi.cast("double *", int(ffi.cast("uintptr_t", hP)) + 8)
  assert step(hP_pred=misaligned) == CUDA_MISALIGNED
  assert step(B=0) == 0                                   # valid and empty: nothing to launch
  assert lib.live_cuda_status() == 0


def test_ragged_smoother_rejects_bad_arguments_before_any_cuda_call():
  from rednose_b200.filters.live import LiveKalman
  from tests.msckf_shapes import MSCKF_SHAPES
  ffi, lib = _lib(LiveKalman)
  x, P = ffi.new("double[]", 2 * 23), ffi.new("double[]", 2 * 22 * 22)
  t, n = ffi.new("double[]", 2), ffi.new("int[]", [2])
  good_q, bad_q = ffi.new("int[]", [3]), ffi.new("int[]", [-1])

  def rts(t=t, n=n, T=2, q=good_q, nq=1):
    st = lib.live_batch_rts_ragged(x, P, x, P, t, n, x, P, T, 1, q, nq, 1, ffi.NULL)
    assert lib.live_cuda_status() == st
    return st

  assert rts(n=ffi.NULL) == CUDA_INVALID_VALUE
  assert rts(t=ffi.NULL) == CUDA_INVALID_VALUE
  assert rts(T=0) == CUDA_INVALID_VALUE
  assert rts(q=bad_q) == CUDA_INVALID_VALUE
  assert rts(nq=17) == CUDA_INVALID_VALUE
  assert lib.live_cuda_status() == 0
  big = next(c for c in MSCKF_SHAPES if c.edim() > 32)    # smoothing serves EDIM <= 32 only
  ffi_m, lib_m = _lib(big)
  st = getattr(lib_m, f"{big.name}_batch_rts_ragged")(ffi_m.NULL, ffi_m.NULL, ffi_m.NULL, ffi_m.NULL, ffi_m.new("double[]", 1),
                                                      ffi_m.new("int[]", [1]), ffi_m.NULL, ffi_m.NULL, 1, 1, ffi_m.NULL, 0, 0, ffi_m.NULL)
  assert st == CUDA_NOT_SUPPORTED and getattr(lib_m, f"{big.name}_cuda_status")() == CUDA_NOT_SUPPORTED


def test_reserve_hands_out_rows_times_and_counts_overflow():
  from rednose_b200.batched import RaggedHistory
  h = RaggedHistory(3, 5, 2, 2, "cpu")
  assert h.reserve(torch.tensor([0, 2, 4]), 0.5).tolist() == [0, 0, 0]
  assert h.reserve(torch.tensor([4, 0]), torch.tensor([0.75, 0.6], dtype=torch.float64)).tolist() == [1, 1]
  assert h.reserve(torch.tensor([1]), 0.8).tolist() == [0]                      # an entry list that skips filters
  assert h.reserve(torch.tensor([4, 3]), torch.tensor([0.9, 0.9], dtype=torch.float64)).tolist() == [2, 0]
  assert h.reserve(torch.tensor([2, 4]), torch.tensor([1.0, 1.1], dtype=torch.float64)).tolist() == [1, -1]   # 4 is full
  assert h.reserve(torch.tensor([4]), 1.2).tolist() == [-1]
  assert h.n.tolist() == [2, 1, 2, 1, 3] and h.n.dtype == torch.int32
  assert h.overflowed() == 2
  t = h.t.numpy()
  assert t[:, 4].tolist() == [0.5, 0.75, 0.9]                                    # overflow leaves the rows as they were
  assert t[:2, 0].tolist() == [0.5, 0.6] and t[:2, 2].tolist() == [0.5, 1.0] and t[0, 1] == 0.8 and t[0, 3] == 0.9
  assert t[2, 0] == 0.0 and t[1, 1] == 0.0


class _RecordingOracleEngine:
  """BatchedEKF's surface (x, P, step_indexed with hist=) computing on the CPU oracle library, one filter at a time with
  the reference driver's own calls (predict, update, normalise after the update), writing the history slabs at the rows
  RaggedHistory.reserve hands out -- what the recording kernels do on the device."""

  def __init__(self, oracle, x, P, Q):
    self.o, self.Q = oracle, Q
    self.x, self.P = torch.as_tensor(x.copy()), torch.as_tensor(P.copy())
    self.B, self.device = x.shape[0], torch.device("cpu")

  def step_indexed(self, kind, idx, dt, z, R, ea=None, hist=None, t=None):
    if idx.numel() == 0:                                # BatchedEKF launches nothing for an empty list
      return None
    rows = hist.reserve(idx, t)
    ys = []
    for e, b in enumerate(idx.tolist()):
      xp, Pp = self.o.predict(self.x[b].numpy()[None], self.P[b].numpy()[None], self.Q, float(dt[e]))
      Re = R.numpy() if R.ndim == 2 else R[e].numpy()
      xf, Pf, y = self.o.update(kind, xp, Pp, z[e].numpy().reshape(1, -1), Re[None])
      xf[0, 3:7] /= np.linalg.norm(xf[0, 3:7])
      r = int(rows[e])
      if r >= 0:
        hist.x_pred[r, b], hist.P_pred[r, b] = torch.as_tensor(xp[0]), torch.as_tensor(Pp[0])
        hist.x_filt[r, b], hist.P_filt[r, b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      self.x[b], self.P[b] = torch.as_tensor(xf[0]), torch.as_tensor(Pf[0])
      ys.append(y[0])
    return torch.as_tensor(np.array(ys)).reshape(len(ys), 1, -1)


def test_scheduler_history_rows_smooth_like_the_reference_driver(oracle_dir):
  """5 live filters on random interleaved streams (kinds 4, 10, 12, own clocks, gaps, late drops).  The history rows
  RaggedScheduler records, smoothed per filter by oracle/rts_numpy, equal EKF_sym.rts_smooth over the estimates the
  reference driver returns for the same stream, to 1e-12."""
  import rednose_b200.ekf_sym as drv
  from oracle.rts_numpy import rts_smooth
  from rednose_b200.batched import RaggedHistory
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RaggedScheduler
  from tests.util import Oracle
  B, T = 5, 64
  rng = np.random.default_rng(3)
  x0 = np.tile(LiveKalman.initial_x, (B, 1)); x0[:, :3] += rng.normal(0, 10.0, (B, 3))
  P0 = np.tile(np.diag(LiveKalman.initial_P_diag), (B, 1, 1))
  Rk = {4: np.eye(3) * 0.025**2, 10: np.eye(3) * 0.5**2, 12: np.eye(3) * 25.0}
  o = Oracle(oracle_dir, "live")
  refs = [drv.EKF_sym(oracle_dir, "live", LiveKalman.Q, x0[b], P0[b], 23, 22, quaternion_idxs=[3]) for b in range(B)]
  est = [[] for _ in range(B)]
  eng = _RecordingOracleEngine(o, x0, P0, LiveKalman.Q)
  hist = RaggedHistory(T, B, 23, 22, "cpu")
  s = RaggedScheduler(eng, history=hist)
  for tick in range(40):
    ids, ts, ks, zs = [], [], [], {k: [] for k in Rk}
    for b in range(B):
      if b == 4 and tick >= 3:                          # filter 4 stops after three steps
        continue
      if b < 4 and rng.random() < 0.3:
        continue
      late = b < 4 and tick > 0 and rng.random() < 0.1  # some late observations: dropped
      tb = 0.01 * tick + 0.003 * b - (0.05 if late else 0.0)
      k = int(rng.choice([4, 10, 12]))
      zb = {4: rng.normal(0, 0.01, 3), 10: rng.normal(0, 0.1, 3) + [0, 0, -9.8], 12: refs[b].state()[:3] + rng.normal(0, 1.0, 3)}[k]
      ids.append(b); ts.append(tb); ks.append(k); zs[k].append(zb)
      if refs[b].filter_time is None or tb >= refs[b].filter_time:   # what RaggedScheduler applies (it drops, never rewinds)
        est[b].append(refs[b].predict_and_update_batch(tb, k, zb[None], Rk[k][None]))
    if ids:
      s.tick(np.array(ids), np.array(ts), np.array(ks), {k: np.array(v) for k, v in zs.items() if v}, Rk)
  assert s.dropped > 0 and hist.overflowed() == 0
  n = hist.n.numpy()
  assert n.tolist() == [len(e) for e in est] and n[4] == 3 and n[:4].min() > 10
  for b in range(B):
    k = int(n[b])
    slabs = [a[:k, b].numpy() for a in (hist.x_pred, hist.x_filt, hist.P_pred, hist.P_filt)]
    assert np.array_equal(hist.t[:k, b].numpy(), [e[4] for e in est[b]])
    for r, e in enumerate(est[b]):                                     # the recorded rows are the driver's estimates
      assert np.max(np.abs(slabs[0][r] - e[0])) < 1e-12 * np.max(np.abs(e[0])) and np.max(np.abs(slabs[1][r] - e[1])) < 1e-12 * np.max(np.abs(e[1]))
    xs, Ps = rts_smooth(o, *slabs, hist.t[:k, b].numpy(), 23, 22, norm_quats=True)
    xr, Pr = refs[b].rts_smooth([tuple(np.copy(a) if isinstance(a, np.ndarray) else a for a in e) for e in est[b]], norm_quats=True)
    ex = np.max(np.abs(xs - xr)) / np.max(np.abs(xr))
    eP = np.max(np.abs(Ps - Pr)) / np.max(np.abs(Pr))
    assert ex < 1e-12 and eP < 1e-12, (b, ex, eP)
