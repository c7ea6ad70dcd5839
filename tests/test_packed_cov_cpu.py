"""The packed covariance layout of the two-filters-per-warp kernel (rednose_b200/csrc/ekf_packed.cuh), without a GPU.

The block-offset header is compiled for the host with g++ and every offset here comes from it, so these tests check the
one definition the kernels use.  Also checked: which filters get the layout, and that the flag is refused, before any
CUDA call, wherever the pair kernel would not run."""
import subprocess

import numpy as np
import pytest
from cffi import FFI

EVEN_EDIMS = list(range(2, 33, 2))
CUDA_NOT_SUPPORTED = 801
PACKED_P = 32

SHIM = r"""
#include "ekf_packed.cuh"
extern "C" int rnb_packed_doubles(int E) { return rnb::packed_doubles(E); }
extern "C" int rnb_packed_block(int I, int J) { return rnb::packed_block(I, J); }
extern "C" int rnb_packed_index(int i, int j) { return rnb::packed_index(i, j); }
static_assert(rnb::packed_doubles(22) == 264 && rnb::packed_block(10, 10) == 260, "constexpr on the host");
"""


@pytest.fixture(scope="module")
def layout(tmp_path_factory):
  from rednose_b200.build import CSRC_DIR
  d = tmp_path_factory.mktemp("packed")
  (d / "shim.cc").write_text(SHIM)
  so = d / "libpacked.so"
  subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-fPIC", "-shared", f"-I{CSRC_DIR}", str(d / "shim.cc"), "-o", str(so)], check=True)
  ffi = FFI()
  ffi.cdef("int rnb_packed_doubles(int E); int rnb_packed_block(int I, int J); int rnb_packed_index(int i, int j);")
  return ffi.dlopen(str(so))


def _index_map(layout, E):
  return np.array([[layout.rnb_packed_index(i, j) for j in range(E)] for i in range(E)])


def _pack(layout, P):
  """What the conversion kernel does: every slot of the lower block triangle from P[max][min]."""
  E = P.shape[0]
  out = np.full(layout.rnb_packed_doubles(E), np.nan)
  for i in range(E):
    for j in range(E):
      if i // 2 >= j // 2:
        out[layout.rnb_packed_block(i // 2, j // 2) + 2 * (i & 1) + (j & 1)] = P[max(i, j), min(i, j)]
  return out


def _unpack(layout, pk, E):
  return pk[_index_map(layout, E)]


@pytest.mark.parametrize("E", EVEN_EDIMS)
def test_block_offsets_are_a_bijection_of_aligned_blocks(layout, E):
  nb = E // 2
  n = layout.rnb_packed_doubles(E)
  assert n == 4 * nb * (nb + 1) // 2
  slots = []
  for I in range(nb):
    for J in range(I + 1):
      b = layout.rnb_packed_block(I, J)
      assert b % 4 == 0                      # 32-byte aligned blocks
      slots += range(b, b + 4)
  assert sorted(slots) == list(range(n))
  # element map: the lower triangle covers every slot except the upper corner of each diagonal block, which is its mirror
  idx = _index_map(layout, E)
  assert np.array_equal(idx, idx.T)
  lower = sorted(idx[np.tril_indices(E)].tolist())
  assert len(set(lower)) == len(lower) == E * (E + 1) // 2
  assert sorted(set(range(n)) - set(lower)) == [layout.rnb_packed_block(I, I) + 1 for I in range(nb)]


@pytest.mark.parametrize("E", [2, 6, 22, 32])
def test_pack_unpack_round_trip_and_mirror(layout, E):
  rng = np.random.default_rng(E)
  A = rng.normal(size=(E, E))
  S = A @ A.T
  assert np.array_equal(_unpack(layout, _pack(layout, S), E), S)
  # an asymmetric input: unpacking gives the mirror of its lower triangle, whatever the upper triangle held
  L = np.tril(A) + np.tril(A, -1).T
  U = A.copy()
  U[np.triu_indices(E, 1)] = 1e300
  got = _unpack(layout, _pack(layout, U), E)
  assert np.array_equal(got, L) and np.array_equal(got, got.T)


def _bank_conflicts(layout, E, packed):
  """Worst number of distinct 16-byte addresses in one bank group, per 128-bit tile read step of ekf_step_pair (the
  quarter-warp of 8 lanes is the unit a 128-bit shared load is served in).  Lane hl (idle lanes mirror E/2 - 1) of half
  h reads block (max(I, hl), min(I, hl)) of its half's tile as two 16-byte loads."""
  nb = E // 2
  ts = layout.rnb_packed_doubles(E) if packed else E * E
  worst = []
  for I in range(nb):
    w = 0
    for h in (0, 1):
      for quarter in (0, 1):
        for second in (0, 1):
          groups = {}
          for lane in range(8 * quarter, 8 * quarter + 8):
            hl = min(lane, nb - 1)
            mx, mn = max(I, hl), min(I, hl)
            off = layout.rnb_packed_block(mx, mn) + 2 * second if packed else 2 * mx * E + 2 * mn + E * second
            a = h * ts + off                                # doubles from the (128-byte aligned) slot
            groups.setdefault((a // 2) % 8, set()).add(a)
          w = max(w, max(len(v) for v in groups.values()))
    worst.append(w)
  return worst


def test_tile_read_bank_groups(layout):
  """Not conflict-free: block rows start 2I(I+1) doubles apart, so for live_kf (EDIM 22) 9 of the 11 read steps are
  2-way and steps 2 and 6 are 3-way.  This pins that measured worst case (the full layout's transposed reads, used for
  history-free callers of the unflagged ABI, are no better), so a layout change that makes it worse shows up here."""
  packed = _bank_conflicts(layout, 22, True)
  assert packed == [2, 2, 3, 2, 2, 2, 3, 2, 2, 2, 2]
  assert max(_bank_conflicts(layout, 22, False)) == 3
  assert all(max(_bank_conflicts(layout, E, True)) <= 4 for E in EVEN_EDIMS)


def _gen(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  d = ensure_generated(cls)
  return load_code(d, cls.name)


def test_packed_doubles_per_filter(gen_dir):
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  _, live = _gen(LiveKalman)
  _, kin = _gen(KinematicKalman)
  _, msckf = _gen(MsckfKalman)
  assert live.live_packed_P_doubles() == 264
  assert kin.kinematic_packed_P_doubles() == 0       # EDIM 2: thread-per-filter kernel
  assert msckf.msckf_packed_P_doubles() == 0         # EDIM > 32: CTA kernel


def _step(ffi, lib, name, kind, E, flags, B=0):
  x, P, Q, z, R = (ffi.new("double[]", n) for n in (64, E * E, E * E, 64, 64 * 64))
  qi = ffi.new("int[]", [0])
  getattr(lib, f"{name}_batch_step_{kind}")(x, P, Q, ffi.NULL, 0.01, z, R, ffi.NULL, 1, B, qi, 0, flags, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL)
  return getattr(lib, f"{name}_cuda_status")()


def test_flag_rejected_where_the_pair_kernel_does_not_run(gen_dir):
  """B = 0: an accepted launch returns before any CUDA call, so acceptance is checkable without a GPU too."""
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.shapes import BY_NAME
  ffi, live = _gen(LiveKalman)
  assert _step(ffi, live, "live", 12, 22, 3 | PACKED_P) == 0
  ffi_k, kin = _gen(KinematicKalman)
  assert _step(ffi_k, kin, "kinematic", 1, 2, PACKED_P) == CUDA_NOT_SUPPORTED
  ffi_m, msckf = _gen(MsckfKalman)
  kinds = sorted(int(s.rsplit("_", 1)[1]) for s in dir(msckf) if s.startswith("msckf_batch_step_") and not s.endswith("_idx"))
  for k in kinds:                                     # EDIM > 32 and the feature kinds: CTA kernel
    assert _step(ffi_m, msckf, "msckf", k, 64, PACKED_P) == CUDA_NOT_SUPPORTED
  x, P, z, R, out = (ffi.new("double[]", n) for n in (23, 484, 3, 9, 1))
  qi = ffi.new("int[]", [3])
  # host buffers are always full
  live.live_host_step_12(x, P, P, ffi.NULL, 0.01, z, R, ffi.NULL, 1, 1, qi, 1, PACKED_P)
  assert live.live_cuda_status() == CUDA_NOT_SUPPORTED
  ffi_7, e7 = _gen(BY_NAME["shape_e7"])               # odd EDIM: one filter per warp
  assert _step(ffi_7, e7, "shape_e7", 1, 7, PACKED_P) == CUDA_NOT_SUPPORTED
  x, P, z, R, out = (ffi_7.new("double[]", n) for n in (7, 49, 1, 1, 1))
  qi = ffi_7.new("int[]", [0])
  e7.shape_e7_batch_predict(x, P, P, ffi_7.NULL, 0.01, 0, qi, 0, PACKED_P, ffi_7.NULL, ffi_7.NULL, ffi_7.NULL)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED
  e7.shape_e7_batch_update_1(x, P, z, R, ffi_7.NULL, 1, 0, qi, 0, PACKED_P, ffi_7.NULL, ffi_7.NULL, ffi_7.NULL)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED
  e7.shape_e7_batch_maha_1(x, P, z, R, ffi_7.NULL, 0, PACKED_P, out, ffi_7.NULL)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED
  assert e7.shape_e7_cuda_status() == 0
