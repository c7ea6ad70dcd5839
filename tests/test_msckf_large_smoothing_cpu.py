"""RTS smoothing of MSCKFs above EDIM 32 without a GPU: which smoother each library carries, and the argument checks of
<name>_batch_rts / _batch_rts_segment, which return before any CUDA call.

Above EDIM 32 a filter is smoothed on its main block (at most 32 wide) by the same warp-per-filter kernels as below it:
ekf_rts_warp_mma for an even EDIM with MEDIM >= 8, ekf_rts_warp otherwise.  Only the whole-history instantiation exists
there: ragged and packed histories stay refused."""
import os
import re
import subprocess

import pytest

from tests.msckf_shapes import MSCKF_SHAPES

CUDA_INVALID_VALUE = 1
LARGE = [c for c in MSCKF_SHAPES if c.edim() > 32]
# the smoother launch_rts_auto picks above EDIM 32 (tests/msckf_shapes.py's MsckfShape.rts_kernel covers EDIM <= 32)
WANT = {"msckf_e33": "scalar", "msckf_e64": "mma", "msckf_e68": "mma", "msckf_e73": "scalar", "msckf_e166": "mma",
        "msckf": "mma"}


def _classes():
  from rednose_b200.filters.msckf import MsckfKalman
  return LARGE + [MsckfKalman]


def _dims(folder, name):
  src = open(os.path.join(folder, f"{name}.cu"), encoding="utf-8").read()
  return tuple(int(re.search(rf"\b{k} = (\d+)", src).group(1)) for k in ("EDIM", "MEDIM"))


def test_every_msckf_above_edim_32_has_an_expected_smoother():
  assert sorted(c.name for c in _classes()) == sorted(WANT)


@pytest.mark.parametrize("cls", _classes(), ids=lambda c: c.name)
def test_library_carries_the_expected_smoother_kernel(cls):
  """`cuobjdump -symbols` of lib<name>.so lists exactly one smoother entry: the whole-history (not ragged) instantiation of
  the kernel the rule gives for the generated EDIM / MEDIM."""
  from rednose_b200 import build
  from rednose_b200.filters import ensure_generated
  folder = ensure_generated(cls)
  edim, medim = _dims(folder, cls.name)
  assert edim > 32 and medim <= 32
  assert WANT[cls.name] == ("mma" if edim % 2 == 0 and medim >= 8 else "scalar")
  cuobjdump = os.path.join(os.path.dirname(build.nvcc_path()), "cuobjdump")
  out = subprocess.run([cuobjdump, "-symbols", os.path.join(folder, f"lib{cls.name}.so")], check=True, capture_output=True,
                       text=True).stdout
  kernels = sorted(set(re.findall(r"_ZN3rnb\d+(ekf_rts_warp(?:_mma)?)I\w+?L(b[01])EEEvNS_7RtsArgs", out)))
  want = "ekf_rts_warp_mma" if WANT[cls.name] == "mma" else "ekf_rts_warp"
  assert kernels == [(want, "b0")], kernels


def _lib(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


def _dim(cls):
  from rednose_b200.filters import ensure_generated
  src = open(os.path.join(ensure_generated(cls), f"{cls.name}.cu"), encoding="utf-8").read()
  return int(re.search(r"\bDIM = (\d+)", src).group(1))


@pytest.mark.parametrize("cls", _classes(), ids=lambda c: c.name)
def test_smoother_arguments_are_checked_before_any_cuda_call(cls):
  """B = 0 is valid and launches nothing; a quaternion index that does not fit the state is refused with
  cudaErrorInvalidValue, in both the whole-history and the segment entry point.  No device is touched (the slabs are
  null pointers), so this runs without one."""
  ffi, lib = _lib(cls)
  status = getattr(lib, f"{cls.name}_cuda_status")
  rts, seg = getattr(lib, f"{cls.name}_batch_rts"), getattr(lib, f"{cls.name}_batch_rts_segment")
  n = ffi.NULL
  t = ffi.new("double[]", 4)
  good_q, bad_q = ffi.new("int[]", [3]), ffi.new("int[]", [_dim(cls) - 3])
  assert status() == 0

  def call(fn, B, q, *segment):
    fn(n, n, n, n, t, 0, n, n, 4, B, q, 1, 1, *segment, ffi.NULL)
    return status()

  for fn, segment in ((rts, ()), (seg, (n, n, 2))):
    assert call(fn, 0, good_q, *segment) == 0
    assert call(fn, 0, bad_q, *segment) == CUDA_INVALID_VALUE     # checked before the empty batch returns
    assert call(fn, 3, bad_q, *segment) == CUDA_INVALID_VALUE
  assert status() == 0

