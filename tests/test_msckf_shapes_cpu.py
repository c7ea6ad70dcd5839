"""The synthetic MSCKF shapes (tests/msckf_shapes.py) without a GPU: every one generates and cross-compiles for sm_90a,
keeps its covariance in the layout the CTA kernel reads, fits the shared memory its kernels need, and its 40-digit
reference (tests/hiprec.py) is itself right: against a float64 restatement at every shape, and against the reference
generator's own C at the shipped msckf where that oracle is built.  An MSCKF whose augment kernel would not fit in one
CTA's shared memory is refused by gen_code before nvcc runs."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests import hiprec
from tests.msckf_shapes import MSCKF_SHAPES, augment_np, batch, msckf_model, observe
from tests.util import cov_err, state_err

IDS = [c.name for c in MSCKF_SHAPES]
CUDA_NOT_SUPPORTED = 801
PACKED_P = 32


def _load(cls):
  from rednose_b200.filters import ensure_generated
  from rednose_b200.loader import load_code
  return load_code(ensure_generated(cls), cls.name)


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_msckf_shape_library_builds(cls):
  _, lib = _load(cls)
  kinds = sorted(int(s.rsplit("_", 1)[1]) for s in dir(lib) if s.startswith(f"{cls.name}_batch_step_") and not s.endswith("_idx"))
  assert kinds == sorted(cls.kinds())
  assert hasattr(lib, f"{cls.name}_batch_augment")
  for k in cls.feature_kinds():
    assert hasattr(lib, f"{cls.name}_He_{k}")
  for g in cls.global_names():
    assert hasattr(lib, f"{cls.name}_set_{g}")


def _step(ffi, lib, name, kind, flags, B=0):
  x, P, Q, z, R, ea = (ffi.new("double[]", n) for n in (256, 256 * 256, 256 * 256, 64, 64 * 64, 4))
  qi = ffi.new("int[]", [3])
  getattr(lib, f"{name}_batch_step_{kind}")(x, P, Q, ffi.NULL, 0.01, z, R, ea, 1, B, qi, 1, flags, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL)
  return getattr(lib, f"{name}_cuda_status")()


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_full_covariance_layout_under_the_engines_flags(cls):
  """A filter with a feature-track kind keeps P full: the CTA kernel, which runs its feature kinds, reads only that
  layout.  Every kind is accepted with the flags BatchedEKF passes (B = 0: an accepted launch returns before any CUDA
  call), and the packed flag stays refused for feature kinds."""
  ffi, lib = _load(cls)
  packed = getattr(lib, f"{cls.name}_packed_P_doubles")()
  assert packed == 0, packed
  pflag = PACKED_P if packed else 0                   # what BatchedEKF._P_arg adds to every launch
  for kind in cls.kinds():
    assert _step(ffi, lib, cls.name, kind, 3 | pflag) == 0, kind
  for kind in cls.feature_kinds():
    assert _step(ffi, lib, cls.name, kind, 3 | PACKED_P) == CUDA_NOT_SUPPORTED


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_reference_step_and_augment_agree_with_float64(cls):
  """The 40-digit step and a plain float64 step from the same leaf functions agree to 1e-12 on every kind (a feature
  kind's innovation by its norm: the two use different null-space bases); the 40-digit augment is the float64
  selection-matrix products exactly."""
  m = hiprec.model_of(cls)
  m.gv = [1.0 + 0.25 * i for i in range(len(m.gvars))]
  x, P, Q, dt = batch(cls, 1, seed=2)
  q = cls.quat_idxs()
  for kind, (_, _, _, feat) in cls.kinds().items():
    z, R, ea = observe(cls, m, kind, x, seed=3)
    xr, Pr, yr = hiprec.step(m, kind, x, P, Q, dt, z, R, ea, quat_idxs=q, gate=False)
    xf, Pf, yf = m.step_f64(kind, x[0], P[0], Q, dt[0], z[0], R[0], quat_idxs=q, ea=None if ea is None else ea[0])
    ex, eP = state_err(xf, xr[0]), cov_err(Pf, Pr[0])
    if feat:
      assert yr.shape == (1, cls.kinds()[kind][0] - cls.kinds()[kind][1])
      ey = abs(np.linalg.norm(yf) - np.linalg.norm(yr[0])) / np.linalg.norm(yr[0])
    else:
      ey = state_err(z[0] - yf, z[0] - yr[0])
    assert ex < 1e-12 and eP < 1e-12 and ey < 1e-12, (kind, ex, eP, ey)
  xa, Pa = hiprec.augment(m, x, P)
  xn, Pn = augment_np(cls, x, P)
  assert np.array_equal(xa, xn) and np.array_equal(Pa, Pn)


def test_reference_agrees_with_the_oracle_at_the_shipped_msckf():
  """hiprec's feature update (its own null-space basis) against the reference generator's C (Eigen's fullPivLu kernel)
  at the shipped msckf, EDIM 82: x and P do not depend on the basis."""
  from oracle import build_ref
  if not os.path.exists(os.path.join(build_ref.OUT, "libmsckf.so")):
    pytest.skip("oracle/_ref/libmsckf.so not built")
  from rednose_b200.filters.msckf import MsckfKalman
  from tests.util import Oracle, msckf_batch, msckf_feature_obs
  o = Oracle(build_ref.OUT, "msckf")
  m = hiprec.model_of(MsckfKalman)
  x, P, Q, point = msckf_batch(2, seed=3)
  z, R, _ = msckf_feature_obs(o, x, point, seed=4)
  xo, Po, _ = o.update(17, x, P, z, R, ea=point)
  xr, Pr, yr = hiprec.update(m, 17, x, P, z, R, point, gate=False)
  assert yr.shape == (2, 17)
  assert state_err(xo, xr) < 1e-9 and cov_err(Po, Pr) < 1e-9, (state_err(xo, xr), cov_err(Po, Pr))


SIZE_PROBE = r"""
#include <cstdio>
#include "ekf_cta.cuh"
@STRUCTS@
int main() {
@PRINTS@
  return 0;
}
"""


def _constants(src, struct):
  """The `static constexpr` integers and booleans of one generated struct."""
  body = src[src.index(f"struct {struct} {{"):]
  body = body[:body.index("\n};")]
  out = {}
  for decl in re.findall(r"static constexpr (?:int|bool) ([^;]*);", body):
    for item in decl.split(","):
      k, v = (s.strip() for s in item.split("="))
      out[k] = v
  return out


@pytest.fixture(scope="module")
def smem_sizes(tmp_path_factory):
  """sizeof(CtaSmem<M, K>) of ekf_cta.cuh for every shape and kind (and the predict-only kind), from an nvcc-built host
  program whose model and kind structs carry the constants of the generated sources."""
  from rednose_b200 import build
  from rednose_b200.filters import ensure_generated
  # the predict-only kind of ekf_abi.cuh (rnb::NullKind), with its constants
  structs = ["struct NullK { static constexpr int ZDIM = 1, YDIM = 1, EADIM = 0, NH = 0; static constexpr bool HAS_HE = false; };"]
  prints = []
  for cls in MSCKF_SHAPES:
    src = open(os.path.join(ensure_generated(cls), f"{cls.name}.cu"), encoding="utf-8").read()
    mc = _constants(src, f"{cls.name}_model")
    structs.append(f"struct M_{cls.name} {{ static constexpr int DIM = {mc['DIM']}, EDIM = {mc['EDIM']}, NF = {mc['NF']}, NFROWS = {mc['NFROWS']}; }};")
    for kind in list(cls.kinds()) + [None]:
      k = "NullK" if kind is None else f"K_{cls.name}_{kind}"
      if kind is not None:
        kc = _constants(src, f"{cls.name}_kind_{kind}")
        structs.append(f"struct {k} {{ static constexpr int ZDIM = {kc['ZDIM']}, YDIM = {kc['YDIM']}, EADIM = {kc['EADIM']}, NH = {kc['NH']}; "
                       f"static constexpr bool HAS_HE = {kc['HAS_HE']}; }};")
      prints.append(f'  printf("{cls.name} {kind} %zu\\n", sizeof(rnb::CtaSmem<M_{cls.name}, {k}>));')
  d = tmp_path_factory.mktemp("smem")
  (d / "probe.cu").write_text(SIZE_PROBE.replace("@STRUCTS@", "\n".join(structs)).replace("@PRINTS@", "\n".join(prints)))
  exe = d / "probe"
  subprocess.run([build.nvcc_path(), "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                  f"-I{build.CSRC_DIR}", f"-I{build.INCLUDE_DIR}", "-o", str(exe), str(d / "probe.cu")], check=True)
  out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
  sizes = {}
  for line in out.splitlines():
    name, kind, n = line.split()
    sizes[(name, None if kind == "None" else int(kind))] = int(n)
  return sizes


@pytest.mark.parametrize("cls", MSCKF_SHAPES, ids=IDS)
def test_kernels_fit_shared_memory(cls, smem_sizes):
  """Every launch of the CTA step kernel (each kind, and the predict) and the augment kernel fits the 227 KB one CTA can
  opt in to; gen_code bounds an MSCKF by the augment kernel's need, which is the larger of the two from EDIM ~120 on."""
  from rednose_b200.codegen import MAX_SMEM_PER_BLOCK, augment_smem_bytes
  step = {kind: smem_sizes[(cls.name, kind)] for kind in list(cls.kinds()) + [None]}
  aug = augment_smem_bytes(cls.edim(), cls.dim())
  print(f"{cls.name}: step {max(step.values())} B, augment {aug} B")
  assert max(step.values()) <= MAX_SMEM_PER_BLOCK and aug <= MAX_SMEM_PER_BLOCK, (step, aug)
  if cls.edim() >= 128:
    assert max(step.values()) < aug


def test_msckf_over_the_augment_envelope_is_refused_before_nvcc(tmp_path):
  """EDIM 166 (25 clones of 6 states) is the largest this layout's augment kernel fits; a 26th clone is refused."""
  from rednose_b200.codegen import MAX_SMEM_PER_BLOCK, augment_smem_bytes, gen_code
  assert augment_smem_bytes(166, 166) <= MAX_SMEM_PER_BLOCK < augment_smem_bytes(172, 172)
  spec = dict(medim=16, eskf=False, n_clones=26, clone='plain6', features=[(3, range(16, 26), True)], zdims=(3,))
  with pytest.raises(ValueError, match="EDIM 172.*ekf_augment_cta.*238048 bytes"):
    gen_code(str(tmp_path), "msckf_e172", **msckf_model(**spec), compile_lib=True)
  assert os.listdir(tmp_path) == []                 # nothing generated, nvcc never ran
