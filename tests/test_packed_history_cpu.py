"""Packed covariance histories (REDNOSE_PACKED_HIST), without a GPU: the C-ABI the generator emits, the refusals that
happen before any CUDA call, the byte accounting and tile planning, and the smoother's packed addressing restated on the
host against the one definition of the layout (csrc/ekf_packed.cuh, compiled here with g++)."""
import re
import subprocess

import numpy as np
import pytest
from cffi import FFI

CUDA_NOT_SUPPORTED = 801
PACKED_P, PACKED_HIST = 32, 64
PAIR_EDIMS = (8, 16, 22, 24, 28, 32)

SHIM = r"""
#include "ekf_packed.cuh"
extern "C" int rnb_packed_doubles(int E) { return rnb::packed_doubles(E); }
extern "C" int rnb_packed_block(int I, int J) { return rnb::packed_block(I, J); }
extern "C" int rnb_packed_index(int i, int j) { return rnb::packed_index(i, j); }
extern "C" void rnb_packed_element(int E, int t, int* i, int* j) { rnb::packed_element(E, t, *i, *j); }
"""


@pytest.fixture(scope="module")
def layout(tmp_path_factory):
  from rednose_b200.build import CSRC_DIR
  d = tmp_path_factory.mktemp("packed_hist")
  (d / "shim.cc").write_text(SHIM)
  so = d / "libpacked.so"
  subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-fPIC", "-shared", f"-I{CSRC_DIR}", str(d / "shim.cc"), "-o", str(so)], check=True)
  ffi = FFI()
  ffi.cdef("int rnb_packed_doubles(int E); int rnb_packed_block(int I, int J); int rnb_packed_index(int i, int j);"
           "void rnb_packed_element(int E, int t, int* i, int* j);")
  return ffi, ffi.dlopen(str(so))


def _gen(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  d = ensure_generated(cls)
  return d, load_code(d, cls.name)


def _protos(folder, name):
  with open(f"{folder}/{name}.h", encoding="utf-8") as f:
    return [ln for ln in f.read().split("\n") if ln.startswith(("void ", "int "))]


def test_packed_smoother_prototypes(gen_dir):
  from rednose_b200.filters.live import LiveKalman
  folder, _ = _gen(LiveKalman)
  protos = _protos(folder, "live")
  args = {re.match(r"\w+ (\w+)\(", p).group(1): p[p.index("("):] for p in protos}
  for base in ("batch_rts", "batch_rts_segment", "batch_rts_ragged"):
    assert f"int live_{base}_packed{args[f'live_{base}']}" in protos      # same arguments, int result
  # the reference-compatible `void ` set gains nothing
  assert not [p for p in protos if p.startswith("void ") and "packed" in p]
  assert len([p for p in protos if p.startswith("int ") and p.split("(")[0].endswith("_packed")]) == 3


def _step(ffi, lib, name, kind, E, flags, B=0):
  x, P, Q, z, R, h = (ffi.new("double[]", n) for n in (64, E * E, E * E, 64, 64 * 64, E * E))
  qi = ffi.new("int[]", [0])
  getattr(lib, f"{name}_batch_step_{kind}")(x, P, Q, ffi.NULL, 0.01, z, R, ffi.NULL, 1, B, qi, 0, flags, ffi.NULL, h, ffi.NULL, h, ffi.NULL)
  return getattr(lib, f"{name}_cuda_status")()


def _rts(ffi, lib, name, which, D=64, E=64):
  xs, Ps, t = ffi.new("double[]", D), ffi.new("double[]", E * E), ffi.new("double[]", 2)
  ln = ffi.new("int[]", [0])
  qi = ffi.new("int[]", [0])
  if which == "rts":
    return getattr(lib, f"{name}_batch_rts_packed")(xs, Ps, xs, Ps, t, 0, xs, Ps, 1, 0, qi, 0, 0, ffi.NULL)
  if which == "rts_segment":
    return getattr(lib, f"{name}_batch_rts_segment_packed")(xs, Ps, xs, Ps, t, 0, xs, Ps, 1, 0, qi, 0, 0, xs, Ps, 0, ffi.NULL)
  return getattr(lib, f"{name}_batch_rts_ragged_packed")(xs, Ps, xs, Ps, t, ln, xs, Ps, 1, 0, qi, 0, 0, ffi.NULL)


RTS = ("rts", "rts_segment", "rts_ragged")


def test_packed_history_refused_where_the_pair_kernel_does_not_run(gen_dir):
  """B = 0: an accepted launch returns before any CUDA call, so acceptance is checkable without a GPU too."""
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.shapes import BY_NAME
  _, (ffi, live) = _gen(LiveKalman)
  for flags in (PACKED_HIST, PACKED_HIST | PACKED_P):
    assert _step(ffi, live, "live", 12, 22, 3 | flags) == 0
  assert all(_rts(ffi, live, "live", w) == 0 for w in RTS)
  _, (ffi_k, kin) = _gen(KinematicKalman)                 # EDIM 2: thread kernel
  assert _step(ffi_k, kin, "kinematic", 1, 2, PACKED_HIST) == CUDA_NOT_SUPPORTED
  assert all(_rts(ffi_k, kin, "kinematic", w) == CUDA_NOT_SUPPORTED for w in RTS)
  _, (ffi_7, e7) = _gen(BY_NAME["shape_e7"])             # odd EDIM: one filter per warp
  assert _step(ffi_7, e7, "shape_e7", 1, 7, PACKED_HIST) == CUDA_NOT_SUPPORTED
  x7, P7, z7, R7 = (ffi_7.new("double[]", n) for n in (7, 49, 1, 1))
  q7 = ffi_7.new("int[]", [0])
  e7.shape_e7_batch_predict(x7, P7, P7, ffi_7.NULL, 0.01, 0, q7, 0, PACKED_HIST, ffi_7.NULL, P7, ffi_7.NULL)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED
  e7.shape_e7_batch_update_1(x7, P7, z7, R7, ffi_7.NULL, 1, 0, q7, 0, PACKED_HIST, ffi_7.NULL, P7, ffi_7.NULL)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED
  assert all(_rts(ffi_7, e7, "shape_e7", w) == CUDA_NOT_SUPPORTED for w in RTS)
  assert e7.shape_e7_cuda_status() == CUDA_NOT_SUPPORTED   # a refused call also latches its status, like _hist_idx
  assert e7.shape_e7_cuda_status() == 0
  _, (ffi_m, msckf) = _gen(MsckfKalman)                   # EDIM > 32 and feature kinds: CTA kernel
  kinds = sorted(int(s.rsplit("_", 1)[1]) for s in dir(msckf) if s.startswith("msckf_batch_step_") and not s.endswith("_idx"))
  for k in kinds:
    assert _step(ffi_m, msckf, "msckf", k, 64, PACKED_HIST) == CUDA_NOT_SUPPORTED
  assert all(_rts(ffi_m, msckf, "msckf", w) == CUDA_NOT_SUPPORTED for w in RTS)
  x, P, z, R = (ffi.new("double[]", n) for n in (23, 484, 3, 9))
  qi = ffi.new("int[]", [3])
  live.live_host_step_12(x, P, P, ffi.NULL, 0.01, z, R, ffi.NULL, 1, 1, qi, 1, PACKED_HIST)   # host buffers are always full
  assert live.live_cuda_status() == CUDA_NOT_SUPPORTED
  assert live.live_cuda_status() == 0


def test_history_bytes_and_tile_planning(gen_dir):
  import torch
  from rednose_b200.batched import History, RaggedHistory
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.smoothing import CheckpointedSmoother, TiledSmoother, history_bytes_per_filter
  folder, (_, live) = _gen(LiveKalman)
  D, E, PD = 23, 22, live.live_packed_P_doubles()
  assert PD == 264
  assert history_bytes_per_filter(D, E, 1) == 8112 and history_bytes_per_filter(D, E, 1, packed_doubles=PD) == 4592
  assert history_bytes_per_filter(D, E, 10, smoothed_in_place=False, packed_doubles=PD) == 10 * 8 * (3 * PD + 3 * D)
  T, B = 5, 7
  for packed in (False, True):
    h = History(T, B, D, E, "cpu", PD if packed else 0)
    assert h.packed == packed and h.P_pred.shape == h.P_filt.shape == ((T, B, PD) if packed else (T, B, E, E))
    assert h.bytes() == B * history_bytes_per_filter(D, E, T, packed_doubles=PD if packed else 0) + 8 * T
    r = RaggedHistory(T, B, D, E, "cpu", PD if packed else 0)
    assert r.packed == packed and r.P_filt.shape == h.P_filt.shape
    assert r.bytes() == B * history_bytes_per_filter(D, E, T, packed_doubles=PD if packed else 0) + 8 * T * B + 4 * B
  Q = torch.eye(E)
  budget = 40 << 30
  full = TiledSmoother(folder, "live", Q, D, E, hbm_budget_bytes=budget)
  pk = TiledSmoother(folder, "live", Q, D, E, hbm_budget_bytes=budget, packed_history=True)
  state = 8 * (E * E + D)
  assert pk.tile_size(1000) == budget // (1000 * 4592 + state) and full.tile_size(1000) == budget // (1000 * 8112 + state)
  assert 1.76 < pk.tile_size(1000) / full.tile_size(1000) < 1.77
  cf = CheckpointedSmoother(folder, "live", Q, D, E, hbm_budget_bytes=budget)
  cp = CheckpointedSmoother(folder, "live", Q, D, E, hbm_budget_bytes=budget, packed_history=True)
  assert cf.bytes_per_filter(10_000) - cp.bytes_per_filter(10_000) == 65 * (8112 - 4592)   # checkpoints stay full
  assert cp.plan(1_000_000, 10_000)[1] <= cf.plan(1_000_000, 10_000)[1]
  from rednose_b200.filters.kinematic import KinematicKalman
  kfolder, _ = _gen(KinematicKalman)
  for cls in (TiledSmoother, CheckpointedSmoother):
    with pytest.raises(ValueError, match="packed"):
      cls(kfolder, "kinematic", torch.eye(2), 2, 2, packed_history=True)


def _pair(layout, E, r, c):
  """packed_pair (csrc/ekf_rts.cuh) restated: the slots it reads for elements (r, c), (r, c + 1), c even."""
  _, L = layout
  R, C = r >> 1, c >> 1
  if R > C:
    b = L.rnb_packed_block(R, C) + 2 * (r & 1)
    return b, b + 1
  if R < C:
    b = L.rnb_packed_block(C, R) + (r & 1)
    return b, b + 2
  b = L.rnb_packed_block(R, R)
  return (b + 2, b + 3) if r & 1 else (b, b + 2)


def _mma_store(layout, r, c):
  """Slots the tensor-core smoother stores fragment pair (r, c), (r, c + 1) to, as {slot: 0 or 1 (which element)}."""
  _, L = layout
  R, C = r >> 1, c >> 1
  if R < C:
    return {}
  q = L.rnb_packed_block(R, C)
  if R > C or (r & 1):
    out = {q + 2 * (r & 1): 0, q + 2 * (r & 1) + 1: 1}
  else:
    out = {q: 0}
  if R == C and (r & 1):
    out[q + 1] = 0
  return out


@pytest.mark.parametrize("E", PAIR_EDIMS)
def test_smoother_packed_addressing(layout, E):
  ffi, L = layout
  PD = L.rnb_packed_doubles(E)
  # reads: every fragment pair of the main block resolves to P[max][min] of both elements, the lower triangle
  for r in range(E):
    for c in range(0, E, 2):
      for slot, (i, j) in zip(_pair(layout, E, r, c), ((r, c), (r, c + 1))):
        assert slot == L.rnb_packed_index(max(i, j), min(i, j)), (E, r, c)
  # mma stores (N = E): every slot exactly once, each with a lower element (the diagonal corner with its mirror)
  written = {}
  for r in range(E):
    for c in range(0, E, 2):
      for slot, which in _mma_store(layout, r, c).items():
        i, j = r, c + which
        assert slot not in written, (E, r, c)
        written[slot] = (i, j)
        assert i >= j and L.rnb_packed_index(i, j) == slot or (slot == L.rnb_packed_block(i >> 1, i >> 1) + 1 and j == i - 1)
  assert sorted(written) == list(range(PD))
  # scalar smoother stores: lane `col` writes rows i >= col of its column, an even column also the diagonal corner
  cover = []
  for col in range(E):
    for i in range(col, E):
      cover.append(L.rnb_packed_index(i, col))
      if i == col + 1 and col % 2 == 0:
        cover.append(L.rnb_packed_block(col >> 1, col >> 1) + 1)
  assert sorted(cover) == list(range(PD))
  # the rows outside a main block of N are found from each slot's element (packed_element inverts packed_index)
  i, j = ffi.new("int*"), ffi.new("int*")
  elems = []
  for t in range(PD):
    L.rnb_packed_element(E, t, i, j)
    elems.append((i[0], j[0]))
    corner = i[0] < j[0]
    assert (t == L.rnb_packed_block(i[0] >> 1, i[0] >> 1) + 1 and j[0] == i[0] + 1) if corner else L.rnb_packed_index(i[0], j[0]) == t
  assert sorted(set(elems)) == sorted(elems)
  assert [e for e in elems if e[0] < e[1]] == [(2 * I, 2 * I + 1) for I in range(E // 2)]


def test_unpack_of_a_packed_history_row_is_its_lower_triangle_mirrored(layout):
  """What unpack_P gives for a row of a packed P_pred slab: the lower triangle of the full store_cols slab, mirrored."""
  _, L = layout
  E = 22
  rng = np.random.default_rng(3)
  cols = rng.normal(size=(E, E))              # a store_cols slab: not symmetric to the last bit
  pk = np.empty(L.rnb_packed_doubles(E))
  for I in range(E // 2):
    for hl in range(I + 1):                   # the pair kernel's store_packed for lane hl, columns c0 = 2 hl, c0 + 1
      c0, q = 2 * hl, L.rnb_packed_block(I, hl)
      pk[q:q + 4] = cols[2 * I, c0], (cols[2 * I + 1, c0] if I == hl else cols[2 * I, c0 + 1]), cols[2 * I + 1, c0], cols[2 * I + 1, c0 + 1]
  full = pk[np.array([[L.rnb_packed_index(i, j) for j in range(E)] for i in range(E)])]
  low = np.tril(cols)
  assert np.array_equal(full, low + np.tril(low, -1).T)
