"""Main-block prediction histories and the MSCKF stream of the smoothers, without a GPU: which libraries carry the
entry points, the refusals that return before any CUDA call, the byte and tile arithmetic of long histories, and the
smoothers' handling of 4- and 6-tuple observations."""
import os
import re

import pytest

from tests.msckf_long_shapes import SHAPES as ODD_MAIN
from tests.msckf_shapes import MSCKF_SHAPES

CUDA_INVALID_VALUE, CUDA_NOT_SUPPORTED = 1, 801
MAIN_HIST, PACKED_P, PACKED_HIST = 128, 32, 64
LARGE = [c for c in MSCKF_SHAPES if c.edim() > 32] + ODD_MAIN   # msckf_e36: even EDIM, odd MEDIM
SMALL = [c for c in MSCKF_SHAPES if c.edim() <= 32]


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


def _msckf():
  from rednose_b200.filters.msckf import MsckfKalman
  return MsckfKalman


def _protos(cls):
  from rednose_b200.filters import ensure_generated
  with open(os.path.join(ensure_generated(cls), f"{cls.name}.h"), encoding="utf-8") as f:
    return [ln for ln in f.read().split("\n") if ln.startswith(("void ", "int "))]


@pytest.mark.parametrize("cls", LARGE + [_msckf()] + SMALL, ids=lambda c: c.name)
def test_entry_points_exist_only_above_edim_32(cls):
  """Above EDIM 32: one int _batch_mainhist_step_<kind> per kind and the two int smoothers, taking hP_pred_last before the
  stream; none of them at or below 32.  <name>_main_pred_doubles is MEDIM^2 above 32, 0 elsewhere."""
  _, lib = _lib(cls)
  protos = _protos(cls)
  names = [re.match(r"\w+ (\w+)\(", p).group(1) for p in protos]
  mainhist = sorted(n for n in names if "mainhist" in n)
  kinds = sorted(int(n.rsplit("_", 1)[1]) for n in names if re.fullmatch(rf"{cls.name}_batch_step_\d+", n))
  edim, medim = _dims(cls, "EDIM", "MEDIM")
  if edim > 32:
    want = sorted([f"{cls.name}_batch_mainhist_step_{k}" for k in kinds] + [f"{cls.name}_batch_rts_mainhist", f"{cls.name}_batch_rts_segment_mainhist"])
    assert mainhist == want
    assert all(p.startswith("int ") and p.endswith("double *hP_pred_last, void *stream);") for p in protos if "mainhist" in p)
    assert getattr(lib, f"{cls.name}_main_pred_doubles")() == medim * medim
  else:
    assert mainhist == []
    assert getattr(lib, f"{cls.name}_main_pred_doubles")() == 0


def _dims(cls, *keys):
  from rednose_b200.filters import ensure_generated
  src = open(os.path.join(ensure_generated(cls), f"{cls.name}.cu"), encoding="utf-8").read()
  return tuple(int(re.search(rf"\b{k} = (\d+)", src).group(1)) for k in keys)


def _bufs(ffi):
  x, P, Q, z, R, ea = (ffi.new("double[]", n) for n in (256, 256 * 256, 256 * 256, 64, 64 * 64, 8))
  return x, P, Q, z, R, ea, ffi.new("int[]", [3])


@pytest.mark.parametrize("cls", LARGE + [_msckf()], ids=lambda c: c.name)
def test_main_block_step_refusals(cls):
  """The main-block step is refused with the packed layouts (cudaErrorNotSupported), and FLAG_MAIN_HIST on the gather-list
  launches (_idx, _hist_idx) likewise; B = 0 otherwise returns status 0.  Device pointers are never dereferenced: these
  return before any CUDA call."""
  ffi, lib = _lib(cls)
  name = cls.name
  status = getattr(lib, f"{name}_cuda_status")
  x, P, Q, z, R, ea, qi = _bufs(ffi)
  n = ffi.NULL
  kinds = sorted(int(s.rsplit("_", 1)[1]) for s in dir(lib) if re.fullmatch(rf"{name}_batch_mainhist_step_\d+", s))
  assert kinds
  idx, rows = ffi.new("int[]", [0, 1, 2]), ffi.new("int[]", [0, 0, 0])
  for k in kinds:
    fn = getattr(lib, f"{name}_batch_mainhist_step_{k}")
    assert fn(x, P, Q, n, 0.01, z, R, ea, 1, 0, qi, 1, 3, n, n, n, n, n, n) == 0
    for flag in (PACKED_P, PACKED_HIST):
      assert fn(x, P, Q, n, 0.01, z, R, ea, 1, 3, qi, 1, 3 | flag, n, n, n, n, n, n) == CUDA_NOT_SUPPORTED
    getattr(lib, f"{name}_batch_step_{k}_idx")(x, P, Q, n, 0.01, z, R, ea, 1, 3, qi, 1, 3 | MAIN_HIST, n, n, n, n, idx, n)
    assert status() == CUDA_NOT_SUPPORTED
    st = getattr(lib, f"{name}_batch_step_{k}_hist_idx")(x, P, Q, n, 0.01, z, R, ea, 1, 3, qi, 1, 3 | MAIN_HIST, n, n, n, n,
                                                         idx, rows, 3, n)
    assert st == CUDA_NOT_SUPPORTED
    getattr(lib, f"{name}_batch_update_{k}")(x, P, z, R, ea, 1, 3, qi, 1, 3 | MAIN_HIST, n, n, n)   # no prediction to record
    assert status() == CUDA_NOT_SUPPORTED
  assert status() == 0


@pytest.mark.parametrize("cls", SMALL, ids=lambda c: c.name)
def test_main_block_flag_refused_at_or_below_edim_32(cls):
  """At EDIM <= 32 FLAG_MAIN_HIST is refused on every step entry point before any CUDA call."""
  ffi, lib = _lib(cls)
  status = getattr(lib, f"{cls.name}_cuda_status")
  x, P, Q, z, R, ea, qi = _bufs(ffi)
  n = ffi.NULL
  for k in cls.kinds():
    getattr(lib, f"{cls.name}_batch_step_{k}")(x, P, Q, n, 0.01, z, R, ea, 1, 3, qi, 1, 3 | MAIN_HIST, n, n, n, n, n)
    assert status() == CUDA_NOT_SUPPORTED, k
  assert status() == 0


@pytest.mark.parametrize("cls", LARGE + [_msckf()], ids=lambda c: c.name)
def test_main_block_smoother_arguments_are_checked_before_any_cuda_call(cls):
  """B = 0 is valid; a bad quaternion index is refused with cudaErrorInvalidValue; the whole-history smoother (and a
  segment without a terminal estimate) needs hP_pred_last, the segment with a terminal does not read it."""
  ffi, lib = _lib(cls)
  status = getattr(lib, f"{cls.name}_cuda_status")
  rts, seg = getattr(lib, f"{cls.name}_batch_rts_mainhist"), getattr(lib, f"{cls.name}_batch_rts_segment_mainhist")
  n = ffi.NULL
  t = ffi.new("double[]", 4)
  dim, = _dims(cls, "DIM")
  good_q, bad_q = ffi.new("int[]", [3]), ffi.new("int[]", [dim - 3])
  assert rts(n, n, n, n, t, 0, n, n, 4, 0, good_q, 1, 1, n, n) == 0
  assert rts(n, n, n, n, t, 0, n, n, 4, 3, bad_q, 1, 1, n, n) == CUDA_INVALID_VALUE
  assert rts(n, n, n, n, t, 0, n, n, 4, 3, good_q, 1, 1, n, n) == CUDA_INVALID_VALUE          # no hP_pred_last
  assert seg(n, n, n, n, t, 0, n, n, 4, 3, good_q, 1, 1, n, n, 2, n, n) == CUDA_INVALID_VALUE  # last segment: likewise
  assert seg(n, n, n, n, t, 0, n, n, 4, 0, bad_q, 1, 1, n, n, 2, n, n) == CUDA_INVALID_VALUE
  assert status() == CUDA_INVALID_VALUE and status() == 0   # the last refusal stays latched until it is read


# ------------------------------------------------------------------------------------------- byte and tile arithmetic
MSCKF_DIM, MSCKF_EDIM, MSCKF_MEDIM = 93, 82, 22


def test_msckf_history_step_bytes():
  """A msckf history step: 8 (2 * 82^2 + 2 * 93) = 109 072 bytes in full, 8 (82^2 + 22^2 + 2 * 93) = 59 152 with the main
  block of the prediction, plus 53 792 bytes once for the full newest prediction."""
  from rednose_b200.smoothing import history_bytes_per_filter
  full = history_bytes_per_filter(MSCKF_DIM, MSCKF_EDIM, 1)
  assert full == 109_072
  main = history_bytes_per_filter(MSCKF_DIM, MSCKF_EDIM, 10, main_pred_doubles=MSCKF_MEDIM ** 2)
  assert main == 10 * 59_152 + 53_792
  assert history_bytes_per_filter(MSCKF_DIM, MSCKF_EDIM, 10, smoothed_in_place=False, main_pred_doubles=MSCKF_MEDIM ** 2) == \
    10 * (59_152 + 8 * (MSCKF_EDIM ** 2 + MSCKF_DIM)) + 53_792


def _smoother(kind, **kw):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother
  cls = {"checkpointed": CheckpointedSmoother, "tiled": TiledSmoother}[kind]
  return cls(ensure_generated(_msckf()), "msckf", None, MSCKF_DIM, MSCKF_EDIM, **kw)


def test_worked_example_tiles():
  """10 000 msckf filters, T = 1 000, segment 64, the default 60 GiB budget: 8.13 MB per filter and two tiles in full,
  4.93 MB (the full newest prediction included) and one tile with main-block predictions.  TiledSmoother at T = 512
  fits 1.83x the filters per tile."""
  full, main = _smoother("checkpointed"), _smoother("checkpointed", main_pred=True)
  assert full.bytes_per_filter(1000) == 8_125_864
  assert main.bytes_per_filter(1000) == 4_934_856
  assert full.plan(10_000, 1000) == (5_000, 2)
  assert main.plan(10_000, 1000) == (10_000, 1)
  tf, tm = _smoother("tiled").tile_size(512), _smoother("tiled", main_pred=True).tile_size(512)
  assert 1.83 < tm / tf < 1.84, (tf, tm)


def test_main_block_history_refusals_in_the_smoothers():
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother
  small = MSCKF_SHAPES[0]
  assert small.edim() <= 32
  for S in (CheckpointedSmoother, TiledSmoother):
    with pytest.raises(ValueError, match="above EDIM 32"):
      S(ensure_generated(small), small.name, None, small.dim(), small.edim(), main_pred=True)
    with pytest.raises(ValueError, match="above EDIM 32"):
      S(ensure_generated(LiveKalman), "live", None, 23, 22, main_pred=True)
    with pytest.raises(ValueError, match="full covariance layout"):
      S(ensure_generated(_msckf()), "msckf", None, MSCKF_DIM, MSCKF_EDIM, main_pred=True, packed_history=True)


# -------------------------------------------------------------------------------------------------- observation tuples
def test_four_and_six_tuple_observations():
  """obs_fn may return (t, kind, z, R) -- ea None, no shift -- or (t, kind, z, R, ea, augment)."""
  from rednose_b200.smoothing import _observation
  assert _observation(lambda k, lo, hi: (0.5, 12, "z", "R"), 0, 0, 1) == (0.5, 12, "z", "R", None, False)
  assert _observation(lambda k, lo, hi: (0.5, 17, "z", "R", "ea", k == 3), 3, 0, 1) == (0.5, 17, "z", "R", "ea", True)


class _Engine:
  """Stands in for BatchedEKF in the smoothers' loops: records what each call received."""

  def __init__(self, calls, dim_x, dim_err, B):
    import torch
    self.calls, self.B = calls, B
    self.x = torch.zeros(B, dim_x, dtype=torch.float64)
    self.P = torch.zeros(B, dim_err, dim_err, dtype=torch.float64)
    self.filter_time = None

  def init_state(self, x, P, filter_time=None):
    self.filter_time = filter_time

  def new_history(self, T, packed=False, main_pred=False):
    import torch

    class H:
      pass
    h = H()
    h.T, h.n, h.main_pred = T, 0, main_pred
    h.P_filt = torch.zeros(T, self.B, self.P.shape[1], self.P.shape[1], dtype=torch.float64)
    self.calls.append(("new_history", T, main_pred))
    return h

  def predict_and_update_batch(self, t, kind, z, R, extra_args=None, augment=False):
    self.calls.append(("forward", t, kind, extra_args, augment))
    self.filter_time = t

  def step_recorded(self, hist, kind, t, z, R, ea=None, augment=False):
    self.calls.append(("recorded", t, kind, ea, augment))
    hist.n += 1

  def rts_smooth(self, hist, **kw):
    import torch
    T = hist.n
    return torch.zeros(T, self.B, self.x.shape[1], dtype=torch.float64), hist.P_filt[:T]


@pytest.mark.parametrize("six", [False, True])
def test_smoothers_pass_the_observation_tuple_through(monkeypatch, six):
  """Both smoothers hand a 4-tuple on as ea = None, augment = False, and a 6-tuple's ea and augment unchanged: in
  CheckpointedSmoother to the first forward pass and to the re-forward with history."""
  import torch
  from rednose_b200 import smoothing
  calls = []
  B, T = 3, 5
  monkeypatch.setattr(smoothing, "BatchedEKF", lambda folder, name, Q, x0, P0, **kw: _Engine(calls, MSCKF_DIM, MSCKF_EDIM, x0.shape[0]))

  class _Event:
    def __init__(self, **kw): pass
    def record(self): pass
    def synchronize(self): pass
    def elapsed_time(self, other): return 0.0
  monkeypatch.setattr(torch.cuda, "Event", _Event)

  def obs_fn(k, lo, hi):
    base = (0.1 * (k + 1), 17, torch.zeros(hi - lo, 20), torch.zeros(hi - lo, 20, 20))
    return base + (f"ea{k}", k == 2) if six else base

  x0, P0 = torch.zeros(B, MSCKF_DIM), torch.zeros(B, MSCKF_EDIM, MSCKF_EDIM)
  want = {k: ((f"ea{k}", k == 2) if six else (None, False)) for k in range(T)}
  for main in (False, True):
    calls.clear()
    sm = _smoother("checkpointed", segment=2, main_pred=main, device="cpu")
    sm.run(x0, P0, T, obs_fn, lambda *a: None)
    fwd = [c for c in calls if c[0] == "forward"]
    rec = [c for c in calls if c[0] == "recorded"]
    assert [c[3:] for c in fwd] == [want[k] for k in range(T)]
    assert sorted(set((round(c[1] * 10) - 1, c[3], c[4]) for c in rec)) == [(k, *want[k]) for k in range(T)]
    assert ("new_history", 3, main) in calls
    calls.clear()
    sm = _smoother("tiled", main_pred=main, device="cpu")
    sm.run(x0, P0, T, obs_fn, lambda *a: None)
    assert [c[3:] for c in calls if c[0] == "recorded"] == [want[k] for k in range(T)]
    assert ("new_history", T, main) in calls
