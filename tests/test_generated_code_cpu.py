"""The GENERATED model code (sparse F / H_err slots, CSE'd leaf functions, F_apply / Herr_apply / S_accum) compiled for
the HOST and driven through the column-wise algorithm of the warp kernels (rednose_b200/csrc/ekf_warp.cuh phase B:
lane j = column j of P, exchange of the non-identity rows of F P, rank-m update), checked against the oracle on CPU.

The device functions the generator emits are plain C++ behind `__device__ __forceinline__`; defining those away lets
g++ build them.  This runs in the CPU suite every round, so a generator regression (sparsity pattern, slot numbering,
symbolic H * H_mod) is caught without a GPU; the kernels proper are covered by tests/test_parity_gpu.py."""
import os
import re
import subprocess

import numpy as np
import pytest
from cffi import FFI

from tests.util import LIVE_KINDS, Oracle, cov_err, live_batch, live_obs, quat_norm_err, state_err

HARNESS = r"""
#include <cmath>
#include <cstring>
#define __device__
#define __forceinline__ inline
#define __restrict__
using std::fma; using std::sqrt; using std::sin; using std::cos;
%(structs)s

static void solve_small(int n, double* A, double* b, int nrhs) {   // Gaussian elimination with partial pivoting, A n x n row-major, b n x nrhs
  for (int k = 0; k < n; ++k) {
    int piv = k;
    for (int i = k + 1; i < n; ++i) if (std::fabs(A[i * n + k]) > std::fabs(A[piv * n + k])) piv = i;
    if (piv != k) { for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[piv * n + j]); for (int j = 0; j < nrhs; ++j) std::swap(b[k * nrhs + j], b[piv * nrhs + j]); }
    for (int i = k + 1; i < n; ++i) {
      const double f = A[i * n + k] / A[k * n + k];
      for (int j = k; j < n; ++j) A[i * n + j] -= f * A[k * n + j];
      for (int j = 0; j < nrhs; ++j) b[i * nrhs + j] -= f * b[k * nrhs + j];
    }
  }
  for (int k = n - 1; k >= 0; --k)
    for (int j = 0; j < nrhs; ++j) {
      double v = b[k * nrhs + j];
      for (int i = k + 1; i < n; ++i) v -= A[k * n + i] * b[i * nrhs + j];
      b[k * nrhs + j] = v / A[k * n + k];
    }
}
static void norm4(double* q) { const double n = sqrt(q[0]*q[0] + q[1]*q[1] + q[2]*q[2] + q[3]*q[3]); for (int i = 0; i < 4; ++i) q[i] /= n; }

// one fused predict + update of one filter, column by column like phase B of the warp kernels
template <class M, class K>
static void step_cols(double* x, double* P, const double* Q, double dt, double* z, const double* R, const double* ea, int quat, int flags) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  double xn[D + 1], fv[M::NF + 2], dx[E + 1];
  M::predict_leaf(x, dt, nullptr, xn, fv);
  if ((flags & 1) && quat >= 0) norm4(xn + quat);
  static double p[E][E], ex[E][E];                       // p[j] = column j of P
  for (int j = 0; j < E; ++j) for (int i = 0; i < E; ++i) p[j][i] = P[i * E + j];
  for (int j = 0; j < E; ++j) {                          // rows of F P that differ from rows of P -> exchange
    double m[E];
    std::memcpy(m, p[j], sizeof(m));
    M::F_apply(fv, m);
    int sl = 0;
    for (int r = 0; r < E; ++r) if ((M::FROW_MASK >> r) & 1u) ex[sl++][j] = m[r];
  }
  for (int j = 0; j < E; ++j) {
    if ((M::FROW_MASK >> j) & 1u) {
      int sl = 0;
      for (int r = 0; r < j; ++r) sl += (M::FROW_MASK >> r) & 1u;
      std::memcpy(p[j], ex[sl], sizeof(double) * E);     // row j of F P (every other row of F P is a column of P: symmetry)
    }
    M::F_apply(fv, p[j]);                                // column j of F (F P)^T
    for (int i = 0; i < E; ++i) p[j][i] = fma(dt, Q[i * E + j], p[j][i]);
  }
  double hx[Z], hv[K::NH + 2], y[Z], HP[Z][E], S[Z][Z], A[Z * Z], W[Z][E];
  K::obs_leaf(xn, ea, nullptr, hx, hv);
  for (int i = 0; i < Z; ++i) y[i] = z[i] - hx[i];
  for (int j = 0; j < E; ++j) { double hp[Z]; K::Herr_apply(hv, p[j], hp); for (int c = 0; c < Z; ++c) HP[c][j] = hp[c]; }
  for (int i = 0; i < Z; ++i) for (int j = 0; j < Z; ++j) S[i][j] = 0.0;
  K::S_accum(hv, [&](int c, int k) { return HP[c][k]; }, S);
  for (int i = 0; i < Z; ++i) for (int j = 0; j < Z; ++j) A[i * Z + j] = S[i][j] + R[i * Z + j];
  double rhs[Z * E];
  for (int c = 0; c < Z; ++c) for (int j = 0; j < E; ++j) rhs[c * E + j] = HP[c][j];
  solve_small(Z, A, rhs, E);                             // W = S^-1 (H P): column j = row j of the gain
  for (int c = 0; c < Z; ++c) for (int j = 0; j < E; ++j) W[c][j] = rhs[c * E + j];
  for (int j = 0; j < E; ++j) {
    double d = 0.0;
    for (int c = 0; c < Z; ++c) d = fma(W[c][j], y[c], d);
    dx[j] = d;
    for (int i = 0; i < E; ++i) for (int c = 0; c < Z; ++c) p[j][i] = fma(-HP[c][i], W[c][j], p[j][i]);
  }
  double xo[D + 1];
  M::err_fun(xn, dx, nullptr, xo);
  if ((flags & 2) && quat >= 0) norm4(xo + quat);
  std::memcpy(x, xo, sizeof(double) * D);
  for (int j = 0; j < E; ++j) for (int i = 0; i < E; ++i) P[i * E + j] = p[j][i];
  for (int i = 0; i < Z; ++i) z[i] = y[i];
}
extern "C" {
%(entries)s
}
"""


@pytest.fixture(scope="module")
def emu(gen_dir, tmp_path_factory):
  src = open(os.path.join(gen_dir, "live.cu"), encoding="utf-8").read()
  structs = src[src.index("struct live_model {"):src.index('extern "C" {')]
  kinds = [int(k) for k in re.findall(r"struct live_kind_(\d+) \{", structs)]
  entries = "\n".join(
    f"void emu_step_{k}(double* x, double* P, const double* Q, double dt, double* z, const double* R, int quat, int flags) "
    f"{{ step_cols<live_model, live_kind_{k}>(x, P, Q, dt, z, R, nullptr, quat, flags); }}" for k in kinds)
  d = tmp_path_factory.mktemp("emu")
  cpp = os.path.join(d, "emu.cc")
  with open(cpp, "w", encoding="utf-8") as f:
    f.write(HARNESS % dict(structs=structs, entries=entries))
  lib = os.path.join(d, "libemu.so")
  subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", lib, cpp], check=True)
  ffi = FFI()
  ffi.cdef("\n".join(f"void emu_step_{k}(double*, double*, const double*, double, double*, const double*, int, int);" for k in kinds))
  return ffi, ffi.dlopen(lib), kinds


@pytest.mark.parametrize("kind", sorted(LIVE_KINDS))
def test_generated_sparse_code_through_the_column_algorithm(emu, oracle_dir, kind):
  ffi, lib, kinds = emu
  assert kind in kinds
  o = Oracle(oracle_dir, "live")
  B = 24
  x, P, Q = live_batch(B, seed=100 + kind)
  A = np.random.default_rng(kind).normal(size=(22, 22)) * 1e-3
  Q = Q + A @ A.T                                        # dense Q: every F / Q term of the predict is exercised
  z, R = live_obs(o, kind, x)
  xr, Pr, yr = o.batch_step(kind, x, P, Q, 0.02, z, R, quat_idxs=[3], flags=3)
  xe, Pe, ze = x.copy(), P.copy(), np.ascontiguousarray(z, dtype=np.float64).copy()
  Qc, Rc = np.ascontiguousarray(Q), np.ascontiguousarray(R)
  p = lambda a: ffi.cast("double *", a.ctypes.data)
  for b in range(B):
    getattr(lib, f"emu_step_{kind}")(p(xe[b]), p(Pe[b]), ffi.cast("const double *", Qc.ctypes.data), 0.02, p(ze[b]),
                                     ffi.cast("const double *", Rc[b].ctypes.data), 3, 3)
  ex, eP, ey = state_err(xe, xr), cov_err(Pe, Pr), state_err(ze.reshape(yr.shape), yr)
  assert ex < 1e-9 and eP < 1e-9 and ey < 1e-9, (ex, eP, ey)
  # the column algorithm keeps P symmetric to rounding of its update P - (HP)^T S^-1 (HP): that form cancels where the
  # update is strong (kind 9, R = 0.00025^2, shrinks the rate variances ~1e7-fold), measured 1.7e-11 there, 1e-15 elsewhere
  assert cov_err(Pe, np.transpose(Pe, (0, 2, 1))) < 1e-10
  assert quat_norm_err(xe, [3]) <= 1e-15
