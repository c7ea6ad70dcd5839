"""Ragged streams longer than one history, without a GPU: the C-ABI of <name>_batch_rts_ragged_segment (which libraries
export it, its refusals, all made before any CUDA call) and RaggedCheckpointedSmoother's byte and tile arithmetic."""
import ctypes
import os
import re

import pytest

from tests.msckf_shapes import MSCKF_SHAPES
from tests.shapes import BY_NAME, SHAPES

CUDA_INVALID_VALUE, CUDA_NOT_SUPPORTED = 1, 801
ARGS = ("(const double *hx_pred, const double *hP_pred, const double *hx_filt, const double *hP_filt, const double *t, "
        "const int *len, const unsigned char *term, const long long *k0, const double *x_term, const double *P_term, "
        "double *xs, double *Ps, int T, long long B, const int *quat_idxs, int n_quat, int norm_quats, int packed, void *stream);")


def _filters():
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  return [KinematicKalman, LiveKalman, MsckfKalman] + list(SHAPES) + list(MSCKF_SHAPES)


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


@pytest.mark.parametrize("cls", _filters(), ids=lambda c: c.name)
def test_headers_declare_and_libraries_export_the_segment_smoother(cls):
  from rednose_b200.filters import ensure_generated
  folder = ensure_generated(cls)
  with open(os.path.join(folder, f"{cls.name}.h"), encoding="utf-8") as f:
    protos = [ln for ln in f.read().split("\n") if re.match(rf"(void|int) {cls.name}_batch_rts_ragged_segment\w*\(", ln)]
  assert protos == [f"int {cls.name}_batch_rts_ragged_segment{ARGS}"]
  assert hasattr(ctypes.CDLL(os.path.join(folder, f"lib{cls.name}.so")), f"{cls.name}_batch_rts_ragged_segment")


def test_include_header_declares_the_segment_typedef_in_c(tmp_path):
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "t.c"
  src.write_text('#include "rednose_b200.h"\n'
                 "int main(void){ rednose_batch_rts_ragged_segment_fn f = 0; (void)f; return 0; }\n")
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{INCLUDE_DIR}", "-c", str(src), "-o", str(tmp_path / "t.o")], check=True)


def _segment(cls, **kw):
  """Call <name>_batch_rts_ragged_segment with B = 0 and valid arguments overridden by `kw`; returns (status, latched
  status).  Nothing is dereferenced on the device: every outcome here is decided before any CUDA call."""
  ffi, lib = _lib(cls)
  name = cls.name
  getattr(lib, f"{name}_cuda_status")()
  buf = ffi.new("double[]", 64)
  a = dict(t=buf, len=ffi.new("int[]", [1]), term=ffi.new("unsigned char[]", [0]), k0=ffi.new("long long[]", [0]), x_term=buf,
           P_term=buf, T=1, B=0, q=ffi.NULL, nq=0, packed=0)
  a.update({k: (ffi.NULL if v is None else v) for k, v in kw.items()})
  st = getattr(lib, f"{name}_batch_rts_ragged_segment")(buf, buf, buf, buf, a["t"], a["len"], a["term"], a["k0"], a["x_term"],
                                                         a["P_term"], buf, buf, a["T"], a["B"], a["q"], a["nq"], 0, a["packed"],
                                                         ffi.NULL)
  return st, getattr(lib, f"{name}_cuda_status")()


def test_segment_smoother_refusals_before_any_cuda_call():
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  for cls in (KinematicKalman, BY_NAME["shape_e7"]):          # the pair kernel does not serve these: no packed layout
    assert _segment(cls, packed=1) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED), cls.name
    assert _segment(cls, packed=1, B=1) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED), cls.name
  big = [MsckfKalman] + [c for c in MSCKF_SHAPES if c.edim() > 32]   # EDIM > 32: ragged histories are refused
  for cls in big:
    for packed in (0, 1):
      assert _segment(cls, packed=packed) == (CUDA_NOT_SUPPORTED, CUDA_NOT_SUPPORTED), (cls.name, packed)
  none = dict(t=None, len=None, term=None, k0=None, x_term=None, P_term=None)
  for cls, packed in ((LiveKalman, 0), (LiveKalman, 1), (KinematicKalman, 0), (BY_NAME["shape_e7"], 0), (BY_NAME["shape_e16"], 1)):
    assert _segment(cls, packed=packed) == (0, 0), (cls.name, packed)          # valid and empty: nothing to launch
    assert _segment(cls, packed=packed, **none) == (0, 0), (cls.name, packed)
  for arg in none:                                            # a non-empty batch needs every per-filter array
    assert _segment(LiveKalman, B=1, **{arg: None}) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE), arg
  assert _segment(LiveKalman, B=1, T=0) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  assert _segment(LiveKalman, B=-1) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  ffi, lib = _lib(LiveKalman)
  assert _segment(LiveKalman, q=ffi.new("int[]", [21]), nq=1) == (CUDA_INVALID_VALUE, CUDA_INVALID_VALUE)
  assert lib.live_cuda_status() == 0


# ------------------------------------------------------------------------------------------- byte and tile arithmetic
def test_whole_ragged_history_row_bytes():
  """A row of a whole RaggedHistory costs 8 120 bytes per live filter (8 112 of slabs + its time), 4 600 packed; an hour
  of 100 Hz IMU (360 000 rows) is 2.9 GB per filter."""
  from rednose_b200.smoothing import ragged_history_bytes_per_filter
  assert ragged_history_bytes_per_filter(23, 22, 1) == 8_120 + 4
  assert ragged_history_bytes_per_filter(23, 22, 1, packed_doubles=264) == 4_600 + 4
  assert ragged_history_bytes_per_filter(23, 22, 360_000) == 360_000 * 8_120 + 4


def test_checkpointed_ragged_bytes_and_tiles():
  """Live, 360 000 ticks, segments of 64 ticks: 5 625 checkpoints of 4 076 bytes (x, P, clock, rows so far, rows in the
  segment), a 65-row segment history (527 804 bytes) and pass 1's one-row history (8 124), the carried row and terminal
  estimate (8 120) and the resident state (3 x 4 056 + 16): 23 483 732 bytes per filter, so the default 60 GiB budget
  takes 2 743 filters per tile and 16 384 filters go in 6 equal tiles of 2 731.  Segments of 256 ticks: 7 850 204
  bytes, 2 tiles of 8 192."""
  from rednose_b200.smoothing import RaggedCheckpointedSmoother
  s = RaggedCheckpointedSmoother("unused", "live", None, 23, 22, segment=64)
  assert s.bytes_per_filter(360_000) == 5_625 * 4_076 + 527_804 + 8_124 + 8_120 + 3 * 4_056 + 16 == 23_483_732
  assert s.tile_size(360_000) == (60 << 30) // 23_483_732 == 2_743
  assert s.plan(16_384, 360_000) == (2_731, 6)
  s = RaggedCheckpointedSmoother("unused", "live", None, 23, 22, segment=256)
  assert s.bytes_per_filter(360_000) == 7_850_204 and s.plan(16_384, 360_000) == (8_192, 2)
  assert RaggedCheckpointedSmoother("unused", "live", None, 23, 22, tile=10).plan(33, 100) == (9, 4)


def test_packed_segment_history_needs_a_packed_layout():
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.smoothing import RaggedCheckpointedSmoother
  with pytest.raises(ValueError, match="packed histories are not available"):
    RaggedCheckpointedSmoother(ensure_generated(KinematicKalman), "kinematic", None, 2, 2, packed_history=True)
  s = RaggedCheckpointedSmoother(ensure_generated(LiveKalman), "live", None, 23, 22, segment=64, packed_history=True)
  full = RaggedCheckpointedSmoother("unused", "live", None, 23, 22, segment=64)
  per_row = 8 * (2 * (484 - 264))                             # two covariance slabs per history row, packed
  assert full.bytes_per_filter(64) - s.bytes_per_filter(64) == (65 + 1) * per_row + 8 * 2 * (484 - 264)
