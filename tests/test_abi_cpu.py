"""CPU tests (no GPU): the generated CUDA libraries build for sm_90a, load, and export every
symbol their headers declare; the plugin descriptor is readable.  No compute calls."""
import ctypes
import os
import re

import pytest


def _protos(header_path):
  with open(header_path, encoding="utf-8") as f:
    return [ln for ln in f.read().split("\n") if re.match(r"^(void|int|void\*) \w+\(", ln)]


@pytest.mark.parametrize("name", ["kinematic", "live"])
def test_library_exports_every_declared_symbol(gen_dir, name):
  lib = ctypes.CDLL(os.path.join(gen_dir, f"lib{name}.so"))
  protos = _protos(os.path.join(gen_dir, f"{name}.h"))
  assert len(protos) > 10
  for p in protos:
    sym = re.match(r"^(?:void|int|void\*) (\w+)\(", p).group(1)
    assert hasattr(lib, sym), sym


@pytest.mark.parametrize("name,dims,kinds", [("kinematic", (2, 2, 2), [1]), ("live", (23, 22, 22), [3, 4, 9, 10, 12, 13, 14, 19])])
def test_reference_symbol_set_and_descriptor(gen_dir, name, dims, kinds):
  """The reference's C symbol set (rednose/helpers/ekf_sym.py:149-171) is present under the same names."""
  lib = ctypes.CDLL(os.path.join(gen_dir, f"lib{name}.so"))
  for s in ["predict", "f_fun", "F_fun", "err_fun", "inv_err_fun", "H_mod_fun"]:
    assert hasattr(lib, f"{name}_{s}")
  for k in kinds:
    for s in ("update", "h", "H", "batch_update", "batch_step", "host_step"):
      assert hasattr(lib, f"{name}_{s}_{k}")

  class Desc(ctypes.Structure):
    _fields_ = [("abi_version", ctypes.c_int), ("name", ctypes.c_char_p), ("dim", ctypes.c_int), ("edim", ctypes.c_int),
                ("medim", ctypes.c_int), ("n_kinds", ctypes.c_int), ("kinds", ctypes.POINTER(ctypes.c_int))]
  lib.ekf_get.restype = ctypes.POINTER(Desc)
  d = lib.ekf_get().contents
  assert d.abi_version == 1 and d.name.decode() == name
  assert (d.dim, d.edim, d.medim) == dims
  assert [d.kinds[i] for i in range(d.n_kinds)] == kinds


def test_header_is_parseable_by_the_reference_loader_rule(gen_dir):
  """rednose/helpers/__init__.py:27 keeps only lines starting with 'void ' and feeds them to cffi.cdef."""
  from cffi import FFI
  with open(os.path.join(gen_dir, "live.h"), encoding="utf-8") as f:
    header = "\n".join(ln for ln in f.read().split("\n") if ln.startswith("void "))
  ffi = FFI()
  ffi.cdef(header)
  lib = ffi.dlopen(os.path.join(gen_dir, "liblive.so"))
  assert lib.live_update_12 and lib.live_batch_step_12


def test_include_header_compiles_as_c(tmp_path):
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "t.c"
  src.write_text('#include "rednose_b200.h"\nint main(void){ rednose_ekf_desc d; (void)d; return 0; }\n')
  subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{INCLUDE_DIR}", "-c", str(src), "-o", str(tmp_path / "t.o")], check=True)


def test_generator_features_symbols(gen_dir):
  """global_vars -> <name>_set_<var>, extra_routines -> <name>_<routine> (ekf_sym.py:94-95,166-171)."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.pendulum import PendulumKalman
  d = ensure_generated(PendulumKalman)
  lib = ctypes.CDLL(os.path.join(d, "libpendulum.so"))
  for sym in ("pendulum_set_grav", "pendulum_set_damp", "pendulum_energy", "pendulum_update_2", "pendulum_batch_step_2"):
    assert hasattr(lib, sym)


@pytest.mark.parametrize("quats", [list(range(0, 17)), [3, 20], [-1]], ids=["n_quat=MAX_QUAT+1", "idx=20", "idx=-1"])
def test_invalid_quaternion_list_is_rejected_before_any_launch(gen_dir, quats):
  """More than MAX_QUAT (16) quaternion indices, or a quaternion that does not fit the 23-entry state, is refused on the
  host: a message, status cudaErrorInvalidValue (1), and no CUDA call at all (so this runs without a GPU).  Accepting
  it would mean normalising only some quaternions or writing outside the state in shared memory."""
  from rednose_b200.loader import load_code
  ffi, lib = load_code(gen_dir, "live")
  assert lib.live_cuda_status() == 0
  x, P, Q, z, R = (ffi.new("double[]", n) for n in (23, 22 * 22, 22 * 22, 3, 9))
  qi = ffi.new("int[]", quats)
  n = len(quats)
  lib.live_batch_step_12(x, P, Q, ffi.NULL, 0.01, z, R, ffi.NULL, 1, 1, qi, n, 3, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL)
  assert lib.live_cuda_status() == 1
  lib.live_batch_predict(x, P, Q, ffi.NULL, 0.01, 1, qi, n, 3, ffi.NULL, ffi.NULL, ffi.NULL)
  assert lib.live_cuda_status() == 1
  lib.live_host_step_12(x, P, Q, ffi.NULL, 0.01, z, R, ffi.NULL, 1, 1, qi, n, 3)
  assert lib.live_cuda_status() == 1
  t = ffi.new("double[]", 2)
  lib.live_batch_rts(x, P, x, P, t, 0, x, P, 2, 1, qi, n, 1, ffi.NULL)
  assert lib.live_cuda_status() == 1
  assert lib.live_cuda_status() == 0     # reading the status clears it


ADAPTER_PROGRAM = r"""
// host program of a maintainer of the reference: its own `struct EKF` (field list of rednose/helpers/ekf.h:14-33, minus
// the Eigen include this image lacks), the adapter header of this repository, and a loader that is
// rednose/helpers/ekf_load.cc:22-39 with the one changed line.
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>
#include <dlfcn.h>
typedef void (*extra_routine_t)(double *, double *);
struct EKF {
  std::string name;
  std::vector<int> kinds;
  std::vector<int> feature_kinds;
  void (*f_fun)(double *, double, double *);
  void (*F_fun)(double *, double, double *);
  void (*err_fun)(double *, double *, double *);
  void (*inv_err_fun)(double *, double *, double *);
  void (*H_mod_fun)(double *, double *);
  void (*predict)(double *, double *, double *, double);
  std::unordered_map<int, void (*)(double *, double *, double *)> hs = {};
  std::unordered_map<int, void (*)(double *, double *, double *)> Hs = {};
  std::unordered_map<int, void (*)(double *, double *, double *, double *, double *)> updates = {};
  std::unordered_map<int, void (*)(double *, double *, double *)> Hes = {};
  std::unordered_map<std::string, void (*)(double)> sets = {};
  std::unordered_map<std::string, extra_routine_t> extra_routines = {};
};
#include "rednose_b200_ekf_adapter.h"

int main(int argc, char** argv) {
  void* handle = dlopen(argv[1], RTLD_NOW);
  assert(handle);
  void* (*ekf_get)() = (void* (*)())dlsym(handle, "ekf_get");
  assert(ekf_get != NULL);
  const EKF* ekf = rednose_b200_adapt((const rednose_ekf_desc*)ekf_get());   // the changed line
  assert(ekf && ekf->name == argv[2]);
  // drive one predict + update through the adapted table, like EKFSym does (ekf_sym.cc:206,212)
  const int kind = ekf->kinds.at(0);
  double x[2] = {0.5, 0.0}, P[4] = {1, 0, 0, 1}, Q[4] = {0.01, 0, 0, 4.0}, z[1] = {0.7}, R[1] = {0.01}, ea[1] = {0};
  ekf->predict(x, P, Q, 0.1);
  ekf->updates.at(kind)(x, P, z, R, ea);
  // the same two calls through the library's C symbols
  typedef void (*pred_t)(double*, double*, double*, double);
  typedef void (*upd_t)(double*, double*, double*, double*, double*);
  std::string n = argv[2];
  pred_t pr = (pred_t)dlsym(handle, (n + "_predict").c_str());
  upd_t up = (upd_t)dlsym(handle, (n + "_update_" + std::to_string(kind)).c_str());
  double x2[2] = {0.5, 0.0}, P2[4] = {1, 0, 0, 1}, z2[1] = {0.7};
  pr(x2, P2, Q, 0.1); up(x2, P2, z2, R, ea);
  assert(memcmp(x, x2, sizeof(x)) == 0 && memcmp(P, P2, sizeof(P)) == 0 && z[0] == z2[0]);
  double h[1]; ekf->hs.at(kind)(x, ea, h);
  printf("%s kinds=%zu feature_kinds=%zu x=%.17g %.17g h=%.17g y=%.17g\n", ekf->name.c_str(), ekf->kinds.size(), ekf->feature_kinds.size(), x[0], x[1], h[0], z[0]);
  return 0;
}
"""


def test_struct_ekf_adapter_drives_a_library(tmp_path, oracle_dir):
  """SURVEY.md section 8 row a13: include/rednose_b200_ekf_adapter.h turns the plain-C descriptor behind ekf_get() into the
  reference's C++ `struct EKF`; compiled here with g++ against a struct with the reference's field list and driven
  through predict / update / h.  The library is the CPU oracle build (same descriptor type, no GPU needed); the
  generated CUDA libraries export the identical descriptor (test_reference_symbol_set_and_descriptor)."""
  import subprocess
  from rednose_b200.build import INCLUDE_DIR
  src = tmp_path / "adapter_host.cc"
  src.write_text(ADAPTER_PROGRAM)
  exe = tmp_path / "adapter_host"
  subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", f"-I{INCLUDE_DIR}", str(src), "-o", str(exe), "-ldl"], check=True)
  out = subprocess.run([str(exe), os.path.join(oracle_dir, "libkinematic.so"), "kinematic"], check=True, capture_output=True, text=True).stdout
  assert out.startswith("kinematic kinds=1 feature_kinds=0")
  # known answer: predict(dt = 0.1) then update with z = 0.7, R = 0.01 on x = [0.5, 0], P = I, Q = diag(0.01, 4)
  vals = [float(v.split("=")[1]) if "=" in v else float(v) for v in out.split()[3:]]
  P00 = 1 + 0.01 + 0.1 * 0.01            # (F P F^T)[0,0] + dt Q[0,0] with F = [[1, dt], [0, 1]]
  K0 = P00 / (P00 + 0.01)
  assert abs(vals[0] - (0.5 + K0 * 0.2)) < 1e-12 and abs(vals[3] - 0.2) < 1e-15
