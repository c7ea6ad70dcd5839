"""Filter code generator: sympy filter definition -> ``{name}.cu`` + ``{name}.h`` -> ``lib{name}.so``.

Keeps the call signature and the build-time maths of the reference's ``gen_code``
(rednose/helpers/ekf_sym.py:29-217: F = d f_err / d x_err at x_err = 0 (:76-80),
H_k = d h_k / d x (:85), He_k = d h_k / d ea for feature kinds (:86-87), Mahalanobis
thresholds chi2_ppf(0.95, dim_z) (:144)) but emits CUDA for sm_90a instead of C + Eigen:

* a ``<name>_model`` struct of ``__device__`` leaf functions (CSE'd, sparsity aware),
* one ``<name>_kind_<k>`` struct per observation kind,
* ``extern "C"`` wrappers instantiating the hand-written kernels in ``csrc/``.

The generated header stays parseable by the reference's cffi loader, which keeps only
lines starting with ``void `` (rednose/helpers/__init__.py:27).
"""
from __future__ import annotations

import os

import numpy as np
import sympy as sp

from rednose_b200.chi2 import chi2_ppf
from rednose_b200.codegen.symbolic import CudaPrinter, cse_block, normalise, sparse_pattern
from rednose_b200 import build as _build

ABI_VERSION = 1


def _arr(n):  # C array extent that is never zero
  return n if n > 0 else 1


def _matsym_name(m):
  return str(m.name) if hasattr(m, 'name') else str(m)


# dynamic shared memory one CTA may opt in to on sm_90 (227 KB)
MAX_SMEM_PER_BLOCK = 232448


def augment_smem_bytes(edim, dim):
  """Dynamic shared memory of ekf_augment_cta (csrc/ekf_augment.cuh): the whole covariance and state of one filter.
  It bounds an MSCKF's size: ekf_step_cta keeps only the lower triangle plus a ZDIM-wide panel (ZDIM <= 31 + EADIM), which
  is the larger of the two only below EDIM ~120, where both need less than half the limit."""
  return 8 * (edim * edim + dim)


def _fma_chain(terms, init=None):
  """terms: [(coef_c, var_c)] -> nested fma expression string."""
  acc = init
  for coef, var in terms:
    if acc is None:
      acc = f"{coef}*{var}"
    else:
      acc = f"fma({coef}, {var}, {acc})"
  return acc if acc is not None else "0.0"


def gen_code(folder, name, f_sym, dt_sym, x_sym, obs_eqs, dim_x, dim_err, eskf_params=None, msckf_params=None,  # pylint: disable=dangerous-default-value
             maha_test_kinds=[], quaternion_idxs=[], global_vars=None, extra_routines=[], compile_lib=None):
  """Generate (and by default compile) the CUDA library of one filter.

  Arguments as in the reference (ekf_sym.py:29-30).  ``compile_lib=None`` compiles
  unless the environment sets ``REDNOSE_B200_NO_COMPILE=1`` (the reference leaves
  compilation to SCons, site_scons/site_tools/rednose_filter.py:27-37).
  """
  # ---- ESKF / plain EKF (ekf_sym.py:36-53) ----
  if eskf_params:
    err_eqs, inv_err_eqs, H_mod_sym, f_err_sym, x_err_sym = eskf_params[:5]
  else:
    nom_x = sp.MatrixSymbol('nom_x', dim_x, 1)
    true_x = sp.MatrixSymbol('true_x', dim_x, 1)
    delta_x = sp.MatrixSymbol('delta_x', dim_x, 1)
    err_eqs = [sp.Matrix(nom_x + delta_x), nom_x, delta_x]
    inv_err_eqs = [sp.Matrix(true_x - nom_x), nom_x, true_x]
    H_mod_sym = sp.eye(dim_x)
    f_err_sym = f_sym
    x_err_sym = x_sym

  # ---- MSCKF layout (ekf_sym.py:57-73) ----
  if msckf_params:
    msckf = True
    dim_main, dim_augment, dim_main_err, dim_augment_err, N, feature_track_kinds = msckf_params[:6]
    assert dim_main + dim_augment * N == dim_x
    assert dim_main_err + dim_augment_err * N == dim_err
  else:
    msckf = False
    dim_main, dim_augment, dim_main_err, dim_augment_err, N, feature_track_kinds = dim_x, 0, dim_err, 0, 0, []
  if int(dim_main_err) > 32:
    raise ValueError(f"filter '{name}': main error block of {int(dim_main_err)} states; the kernels serve at most 32 (the "
                     f"rows of F that differ from the identity are one 32-bit mask).  A larger state needs an MSCKF layout "
                     f"(msckf_params) whose main block is at most 32.")
  if msckf and augment_smem_bytes(int(dim_err), int(dim_x)) > MAX_SMEM_PER_BLOCK:
    raise ValueError(f"filter '{name}': EDIM {int(dim_err)}, DIM {int(dim_x)}: the clone-window shift (ekf_augment_cta) "
                     f"stages the whole covariance and state of a filter in shared memory, "
                     f"{augment_smem_bytes(int(dim_err), int(dim_x))} bytes, over the {MAX_SMEM_PER_BLOCK} bytes one CTA "
                     f"can have.  Use fewer or smaller clones.")

  f_sym = sp.Matrix(f_sym)
  H_mod_sym = sp.Matrix(H_mod_sym)
  gvars = list(global_vars) if global_vars is not None else []
  NG = len(gvars)

  # ---- Jacobians (ekf_sym.py:76-89) ----
  F_sym = sp.Matrix(f_err_sym).jacobian(sp.Matrix(x_err_sym))
  if eskf_params:
    F_sym = F_sym.subs({s: 0 for s in sp.Matrix(x_err_sym)})
  assert dt_sym in F_sym.free_symbols
  F_sym = F_sym.applyfunc(normalise)

  kinds = []
  for eq in obs_eqs:
    h_sym, kind, ea_sym = sp.Matrix(eq[0]), int(eq[1]), eq[2]
    H_sym = h_sym.jacobian(sp.Matrix(x_sym))
    feature = msckf and kind in feature_track_kinds
    He_sym = h_sym.jacobian(sp.Matrix(ea_sym)) if feature else None
    kinds.append(dict(kind=kind, h=h_sym, ea=ea_sym, H=H_sym, He=He_sym, feature=feature,
                      maha=kind in maha_test_kinds, zdim=int(h_sym.shape[0]),
                      eadim=int(ea_sym.shape[0]) if ea_sym is not None else 0))

  # ---- printers ----
  scal = {str(dt_sym): 'dt'}
  for i, g in enumerate(gvars):
    scal[str(g)] = f"gv[{i}]"

  def printer(arrays):
    return CudaPrinter(arrays, scal)

  xname = _matsym_name(x_sym)
  model = f"{name}_model"
  DIM, EDIM, MEDIM = int(dim_x), int(dim_err), int(dim_main_err)
  out = []
  out.append(f"// generated by rednose_b200.codegen (ABI {ABI_VERSION}) for filter '{name}' -- do not edit\n")
  out.append('#include "ekf_abi.cuh"\n#include "rednose_b200.h"\n\n')

  # =========================================================== model struct ==
  out.append(f"struct {model} {{\n")
  out.append(f"  static constexpr int DIM = {DIM}, EDIM = {EDIM}, MEDIM = {MEDIM}, DMAIN = {int(dim_main)}, NG = {NG};\n")
  out.append(f"  static constexpr int DAUG = {int(dim_augment) if msckf else 0}, EAUG = {int(dim_augment_err) if msckf else 0};   // clone size (state / error state), ekf_sym.py:57-66\n")
  out.append(f"  static constexpr bool HAS_FEATURE_KIND = {'true' if any(kd['feature'] for kd in kinds) else 'false'};   // a feature kind runs on the CTA kernel: P stays in the full layout\n")

  # f_fun, F_dense, H_mod_dense, err_fun, inv_err_fun: reference-shaped leaf functions
  pr = printer({xname: 'state'})
  out.append("  static __device__ __forceinline__ void f_fun(const double* __restrict__ state, double dt, const double* __restrict__ gv, double* __restrict__ out) {\n")
  out.append(cse_block([(f"out[{i}]", f_sym[i]) for i in range(DIM)], pr))
  out.append("  }\n")
  out.append("  static __device__ __forceinline__ void F_dense(const double* __restrict__ state, double dt, const double* __restrict__ gv, double* __restrict__ out) {\n")
  out.append(cse_block([(f"out[{i * EDIM + j}]", F_sym[i, j]) for i in range(EDIM) for j in range(EDIM)], pr))
  out.append("  }\n")
  out.append("  static __device__ __forceinline__ void H_mod_dense(const double* __restrict__ state, const double* __restrict__ gv, double* __restrict__ out) {\n")
  out.append(cse_block([(f"out[{i * EDIM + j}]", H_mod_sym[i, j]) for i in range(DIM) for j in range(EDIM)], pr))
  out.append("  }\n")
  pr_err = printer({_matsym_name(err_eqs[1]): 'nom_x', _matsym_name(err_eqs[2]): 'delta_x'})
  out.append("  static __device__ __forceinline__ void err_fun(const double* __restrict__ nom_x, const double* __restrict__ delta_x, const double* __restrict__ gv, double* __restrict__ out) {\n")
  out.append(cse_block([(f"out[{i}]", sp.Matrix(err_eqs[0])[i]) for i in range(DIM)], pr_err))
  out.append("  }\n")
  pr_inv = printer({_matsym_name(inv_err_eqs[1]): 'nom_x', _matsym_name(inv_err_eqs[2]): 'true_x'})
  out.append("  static __device__ __forceinline__ void inv_err_fun(const double* __restrict__ nom_x, const double* __restrict__ true_x, const double* __restrict__ gv, double* __restrict__ out) {\n")
  out.append(cse_block([(f"out[{i}]", sp.Matrix(inv_err_eqs[0])[i]) for i in range(EDIM)], pr_inv))
  out.append("  }\n")

  # structured F over the main block: value slots + straight-line application
  F_main = F_sym[:MEDIM, :MEDIM]
  f_nz = sparse_pattern(F_main)
  rows = {}
  for i, j, e in f_nz:
    rows.setdefault(i, []).append((j, e))
  slots = []           # expressions of the value slots
  row_terms = {}       # row -> (has_unit_diag, [(slot, col)])
  for i in range(MEDIM):
    ents = rows.get(i, [])
    unit_diag = any(j == i and e == 1 for j, e in ents)
    others = [(j, e) for j, e in ents if not (j == i and e == 1)]
    if unit_diag and not others:
      continue  # identity row
    terms = []
    for j, e in others:
      slots.append(e)
      terms.append((len(slots) - 1, j))
    row_terms[i] = (unit_diag, terms)
  NF = len(slots)
  frows = sorted(row_terms)
  out.append(f"  static constexpr int NF = {NF}, NFROWS = {len(frows)};\n")
  out.append(f"  static constexpr unsigned FROW_MASK = 0x{sum(1 << r for r in frows if r < 32):x}u;  // rows of F that differ from the identity\n")
  out.append(f"  // fused leaf of the predict: x_new = f(x, dt) and the {NF} non-trivial entries of F (ekf_c.c:15-16)\n")
  out.append("  template <class FV> static __device__ __forceinline__ void predict_leaf(const double* __restrict__ state, double dt, const double* __restrict__ gv, double* __restrict__ xout, FV& fv) {\n")
  out.append(cse_block([(f"xout[{i}]", f_sym[i]) for i in range(DIM)] + [(f"fv[{s}]", e) for s, e in enumerate(slots)], pr))
  out.append("  }\n")
  out.append("  template <class FV> static __device__ __forceinline__ void F_vals(const double* __restrict__ state, double dt, const double* __restrict__ gv, FV& fv) {\n")
  out.append(cse_block([(f"fv[{s}]", e) for s, e in enumerate(slots)], pr))
  out.append("  }\n")
  out.append(f"  // v <- F v for one column/row held in registers; only the MEDIM main block is touched (ekf_c.c:23-26)\n")
  out.append("  template <class FV, class V> static __device__ __forceinline__ void F_apply(const FV& fv, V& v) {\n")
  for i in frows:
    unit_diag, terms = row_terms[i]
    expr = _fma_chain([(f"fv[{s}]", f"v[{j}]") for s, j in terms], init=f"v[{i}]" if unit_diag else None)
    out.append(f"    const double n{i} = {expr};\n")
  for i in frows:
    out.append(f"    v[{i}] = n{i};\n")
  out.append("  }\n")
  out.append("  static __device__ __forceinline__ void frows_store(const double* v, double* dst, int stride) {\n")
  for s, i in enumerate(frows):
    out.append(f"    dst[{s} * stride] = v[{i}];\n")
  out.append("  }\n")
  out.append("  // v[row] -> dst[row * stride] for the rows of F that differ from the identity\n")
  out.append("  template <class V> static __device__ __forceinline__ void frows_scatter(const V& v, double* dst, int stride) {\n")
  for i in frows:
    out.append(f"    dst[{i} * stride] = v[{i}];\n")
  out.append("  }\n")
  out.append("};\n\n")

  # ============================================================ kind structs ==
  Herr_syms = {}
  for kd in kinds:
    k = kd['kind']
    ks = f"{name}_kind_{k}"
    Z, EA = kd['zdim'], kd['eadim']
    ydim = Z - EA if kd['feature'] else Z
    arrays = {xname: 'state'}
    if kd['ea'] is not None:
      arrays[_matsym_name(kd['ea'])] = 'ea'
    prk = printer(arrays)
    Herr = (kd['H'] * H_mod_sym).applyfunc(normalise)
    Herr_syms[k] = Herr
    h_nz = sparse_pattern(Herr)
    NH = len(h_nz)
    thresh = float(chi2_ppf(0.95, Z))  # the generated C uses dim(h) even for projected kinds (ekf_sym.py:144)
    out.append(f"struct {ks} {{\n")
    out.append(f"  static constexpr int KIND = {k}, ZDIM = {Z}, YDIM = {ydim}, EADIM = {EA}, NH = {NH};\n")
    out.append(f"  static constexpr bool MAHA = {'true' if kd['maha'] else 'false'}, HAS_HE = {'true' if kd['feature'] else 'false'};\n")
    out.append(f"  static constexpr double MAHA_THRESH = {thresh!r};\n")
    sig = "(const double* __restrict__ state, const double* __restrict__ ea, const double* __restrict__ gv, double* __restrict__ out)"
    out.append(f"  static __device__ __forceinline__ void h_fun{sig} {{\n")
    out.append(cse_block([(f"out[{i}]", kd['h'][i]) for i in range(Z)], prk))
    out.append("  }\n")
    out.append(f"  static __device__ __forceinline__ void H_dense{sig} {{\n")
    out.append(cse_block([(f"out[{i * DIM + j}]", kd['H'][i, j]) for i in range(Z) for j in range(DIM)], prk))
    out.append("  }\n")
    if kd['feature']:
      out.append(f"  static __device__ __forceinline__ void He_dense{sig} {{\n")
      out.append(cse_block([(f"out[{i * EA + j}]", kd['He'][i, j]) for i in range(Z) for j in range(EA)], prk))
      out.append("  }\n")
      out.append(f"  // dense H_err = H * H_mod (ZDIM x EDIM), input of the left-null-space projection (ekf_c.c:66-85)\n")
      out.append(f"  static __device__ __forceinline__ void Herr_dense{sig} {{\n")
      out.append(cse_block([(f"out[{i * EDIM + j}]", Herr[i, j]) for i in range(Z) for j in range(EDIM)], prk))
      out.append("  }\n")
    out.append(f"  // fused leaf of the update: h(x) and the {NH} non-zeros of H_err = H * H_mod (ekf_c.c:59-60,83-85)\n")
    out.append(f"  template <class HV> static __device__ __forceinline__ void obs_leaf(const double* __restrict__ state, const double* __restrict__ ea, const double* __restrict__ gv, double (&hx)[{Z}], HV& hv) {{\n")
    out.append(cse_block([(f"hx[{i}]", kd['h'][i]) for i in range(Z)] + [(f"hv[{s}]", e) for s, (_, _, e) in enumerate(h_nz)], prk))
    out.append("  }\n")
    out.append(f"  // hp = H_err v  (v = one column of P)\n")
    out.append(f"  template <class HV, class V> static __device__ __forceinline__ void Herr_apply(const HV& hv, const V& v, double (&hp)[{Z}]) {{\n")
    for a in range(Z):
      terms = [(f"hv[{s}]", f"v[{j}]") for s, (i, j, _) in enumerate(h_nz) if i == a]
      out.append(f"    hp[{a}] = {_fma_chain(terms)};\n")
    out.append("  }\n")
    out.append(f"  // S += (H_err P) H_err^T given an accessor hp(c, k) = (H_err P)[c][k]; upper triangle then mirrored\n")
    out.append(f"  template <class HV, class A> static __device__ __forceinline__ void S_accum(const HV& hv, A hp, double (&S)[{Z}][{Z}]) {{\n")
    for s, (b, kcol, _) in enumerate(h_nz):
      for a in range(b + 1):
        out.append(f"    S[{a}][{b}] = fma(hv[{s}], hp({a}, {kcol}), S[{a}][{b}]);\n")
    for b in range(Z):
      for a in range(b):
        out.append(f"    S[{b}][{a}] = S[{a}][{b}];\n")
    out.append("  }\n")
    out.append("};\n\n")

  # ======================================================= extra routines ==
  extras = []
  for ename, eexpr, eargs in extra_routines:
    eexpr = sp.Matrix(eexpr)
    ptr_args = [a for a in eargs if a is not None]
    if len(ptr_args) > 2 or any(not hasattr(a, 'shape') for a in ptr_args):
      raise NotImplementedError(f"extra routine {ename}: only up to two matrix arguments are supported")
    arrays = {_matsym_name(a): f"in{i}" for i, a in enumerate(ptr_args)}
    sizes = [int(np.prod(a.shape)) for a in ptr_args] + [0, 0]
    nout = int(np.prod(eexpr.shape))
    out.append(f"static __device__ __forceinline__ void {name}_extra_{ename}(const double* __restrict__ in0, const double* __restrict__ in1, const double* __restrict__ gv, double* __restrict__ out) {{\n")
    out.append(cse_block([(f"out[{i}]", eexpr[i]) for i in range(nout)], printer(arrays)))
    out.append("}\n")
    extras.append((ename, len(ptr_args), sizes[0], sizes[1], nout))

  # ============================================================ C-ABI ==
  hdr = []   # header lines (every prototype is a single line starting with 'void ')
  c = []     # wrapper code
  c.append(f"static rnb::HostCtx<{model}>& ctx_() {{ static rnb::HostCtx<{model}> c; return c; }}\n\n")

  def leaf(sym_name, call, proto, hostcall):
    c.append(f"RNB_LEAF_KERNEL(k_{name}_{sym_name}, {NG}, {call})\n")
    hdr.append(f"void {name}_{sym_name}({proto});")
    c.append(f'extern "C" void {name}_{sym_name}({proto}) {{ rnb::run_leaf(ctx_(), k_{name}_{sym_name}, {hostcall}); }}\n')

  # update wrappers first, like the reference header (ekf_sym.py:149)
  for kd in kinds:
    k = kd['kind']
    ks = f"{name}_kind_{k}"
    hdr.append(f"void {name}_update_{k}(double *in_x, double *in_P, double *in_z, double *in_R, double *in_ea);")
    c.append(f'extern "C" void {name}_update_{k}(double *in_x, double *in_P, double *in_z, double *in_R, double *in_ea) {{ rnb::single_update<{model}, {ks}>(ctx_(), in_x, in_P, in_z, in_R, in_ea); }}\n')
  for ename, nptr, n0, n1, nout in extras:
    if nptr == 2:
      leaf(ename, f"{name}_extra_{ename}(in0, in1, gv, out)", "double *in0, double *in1, double *out", f"in0, {n0}, in1, {n1}, 0.0, out, {nout}")
    else:
      leaf(ename, f"{name}_extra_{ename}(in0, in1, gv, out)", "double *in0, double *out", f"in0, {n0}, nullptr, 0, 0.0, out, {nout}")
  leaf("err_fun", f"{model}::err_fun(in0, in1, gv, out)", "double *nom_x, double *delta_x, double *out", f"nom_x, {DIM}, delta_x, {EDIM}, 0.0, out, {DIM}")
  leaf("inv_err_fun", f"{model}::inv_err_fun(in0, in1, gv, out)", "double *nom_x, double *true_x, double *out", f"nom_x, {DIM}, true_x, {DIM}, 0.0, out, {EDIM}")
  leaf("H_mod_fun", f"{model}::H_mod_dense(in0, gv, out)", "double *state, double *out", f"state, {DIM}, nullptr, 0, 0.0, out, {DIM * EDIM}")
  leaf("f_fun", f"{model}::f_fun(in0, s, gv, out)", "double *state, double dt, double *out", f"state, {DIM}, nullptr, 0, dt, out, {DIM}")
  leaf("F_fun", f"{model}::F_dense(in0, s, gv, out)", "double *state, double dt, double *out", f"state, {DIM}, nullptr, 0, dt, out, {EDIM * EDIM}")
  for kd in kinds:
    k, Z, EA = kd['kind'], kd['zdim'], kd['eadim']
    ks = f"{name}_kind_{k}"
    ea_arg = "ea" if EA > 0 else "unused"
    leaf(f"h_{k}", f"{ks}::h_fun(in0, in1, gv, out)", f"double *state, double *{ea_arg}, double *out", f"state, {DIM}, {ea_arg}, {EA}, 0.0, out, {Z}")
    leaf(f"H_{k}", f"{ks}::H_dense(in0, in1, gv, out)", f"double *state, double *{ea_arg}, double *out", f"state, {DIM}, {ea_arg}, {EA}, 0.0, out, {Z * DIM}")
    if kd['feature']:
      leaf(f"He_{k}", f"{ks}::He_dense(in0, in1, gv, out)", f"double *state, double *{ea_arg}, double *out", f"state, {DIM}, {ea_arg}, {EA}, 0.0, out, {Z * EA}")
  hdr.append(f"void {name}_predict(double *in_x, double *in_P, double *in_Q, double dt);")
  c.append(f'extern "C" void {name}_predict(double *in_x, double *in_P, double *in_Q, double dt) {{ rnb::single_predict<{model}>(ctx_(), in_x, in_P, in_Q, dt); }}\n')
  for i, g in enumerate(gvars):
    hdr.append(f"void {name}_set_{g}(double x);")
    c.append(f'extern "C" void {name}_set_{g}(double x) {{ ctx_().gv.v[{i}] = x; }}\n')

  # ---- batched additions (device pointers) ----
  bp = "double *x, double *P, const double *Q, const double *dt_arr, double dt, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_pred, double *hP_pred, void *stream"
  hdr.append(f"void {name}_batch_predict({bp});")
  c.append(f'extern "C" void {name}_batch_predict({bp}) {{ rnb::batch_predict<{model}>(ctx_(), x, P, Q, dt_arr, dt, B, quat_idxs, n_quat, flags, hx_pred, hP_pred, stream); }}\n')
  bu = "double *x, double *P, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_filt, double *hP_filt, void *stream"
  bs = "double *x, double *P, const double *Q, const double *dt_arr, double dt, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_pred, double *hP_pred, double *hx_filt, double *hP_filt, void *stream"
  hs = "double *x, double *P, const double *Q, const double *dt_arr, double dt, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags"
  for kd in kinds:
    k = kd['kind']
    ks = f"{name}_kind_{k}"
    hdr.append(f"void {name}_batch_update_{k}({bu});")
    c.append(f'extern "C" void {name}_batch_update_{k}({bu}) {{ rnb::batch_step<{model}, {ks}, false>(ctx_(), x, P, nullptr, nullptr, 0.0, z, R, ea, n_obs, B, quat_idxs, n_quat, flags, nullptr, nullptr, hx_filt, hP_filt, stream); }}\n')
    hdr.append(f"void {name}_batch_step_{k}({bs});")
    c.append(f'extern "C" void {name}_batch_step_{k}({bs}) {{ rnb::batch_step<{model}, {ks}, true>(ctx_(), x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags, hx_pred, hP_pred, hx_filt, hP_filt, stream); }}\n')
    bi = bs.replace(", void *stream", ", const int *idx, void *stream")
    hdr.append(f"void {name}_batch_step_{k}_idx({bi});")
    c.append(f'extern "C" void {name}_batch_step_{k}_idx({bi}) {{ rnb::batch_step<{model}, {ks}, true>(ctx_(), x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags, hx_pred, hP_pred, hx_filt, hP_filt, stream, idx); }}\n')
    # ragged history: entry e records at row hist_row[e] of [T, hist_B, ...] slabs.  Returns the call's cudaError_t (an
    # int, so the reference-compatible set of `void ` prototypes is unchanged), and its name ends in _idx like its
    # sibling, so readers that list the kinds from the <name>_batch_step_<kind> symbols skip both.
    bh = bi.replace(", void *stream", ", const int *hist_row, long long hist_B, void *stream")
    hdr.append(f"int {name}_batch_step_{k}_hist_idx({bh});")
    c.append(f'extern "C" int {name}_batch_step_{k}_hist_idx({bh}) {{ return rnb::call_status([&] {{ rnb::batch_step_hist<{model}, {ks}>(ctx_(), x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags, hx_pred, hP_pred, hx_filt, hP_filt, idx, hist_row, hist_B, stream); }}); }}\n')
    if EDIM > 32:
      # main-block prediction history (FLAG_MAIN_HIST): hP_pred is one row [B, MEDIM, MEDIM], hP_pred_last [B, EDIM, EDIM]
      # the full prediction.  int result (see _hist_idx); named so that <name>_batch_step_<kind> still lists the kinds
      bmh = bs.replace(", void *stream", ", double *hP_pred_last, void *stream")
      hdr.append(f"int {name}_batch_mainhist_step_{k}({bmh});")
      c.append(f'extern "C" int {name}_batch_mainhist_step_{k}({bmh}) {{ return rnb::call_status([&] {{ rnb::batch_step_mainhist<{model}, {ks}>(ctx_(), x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags, hx_pred, hP_pred, hx_filt, hP_filt, hP_pred_last, stream); }}); }}\n')
    bm = "const double *x, const double *P, const double *z, const double *R, const double *ea, long long B, int flags, double *out, void *stream"
    hdr.append(f"void {name}_batch_maha_{k}({bm});")
    c.append(f'extern "C" void {name}_batch_maha_{k}({bm}) {{ rnb::batch_maha<{model}, {ks}>(ctx_(), x, P, z, R, ea, B, flags, out, stream); }}\n')
    hdr.append(f"void {name}_host_step_{k}({hs});")
    c.append(f'extern "C" void {name}_host_step_{k}({hs}) {{ rnb::host_step<{model}, {ks}>(ctx_(), x, P, Q, dt_arr, dt, z, R, ea, n_obs, B, quat_idxs, n_quat, flags); }}\n')

  # packed covariance layout of the pair kernel (csrc/ekf_packed.cuh): these two return int, so the reference-compatible
  # set of `void ` prototypes is unchanged
  hdr.append(f"int {name}_packed_P_doubles(void);")
  c.append(f'extern "C" int {name}_packed_P_doubles(void) {{ return rnb::packed_P_doubles<{model}>(); }}\n')
  cp = "double *full, double *packed, const int *idx, long long n, int to_packed, void *stream"
  hdr.append(f"int {name}_convert_P({cp});")
  c.append(f'extern "C" int {name}_convert_P({cp}) {{ return rnb::convert_P<{model}>(full, packed, idx, n, to_packed, stream); }}\n')

  br = "const double *hx_pred, const double *hP_pred, const double *hx_filt, const double *hP_filt, const double *t, int t_per_filter, double *xs, double *Ps, int T, long long B, const int *quat_idxs, int n_quat, int norm_quats, void *stream"
  hdr.append(f"void {name}_batch_rts({br});")
  c.append(f'extern "C" void {name}_batch_rts({br}) {{ rnb::batch_rts<{model}>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, t_per_filter, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream); }}\n')
  # one SEGMENT [k0, k0 + T - 1) of a longer history: starts from the smoothed estimate (x_term, P_term) of step k0 + T - 1
  brs = br.replace(", void *stream", ", const double *x_term, const double *P_term, long long k0, void *stream")
  hdr.append(f"void {name}_batch_rts_segment({brs});")
  c.append(f'extern "C" void {name}_batch_rts_segment({brs}) {{ rnb::batch_rts<{model}>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, t_per_filter, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream, x_term, P_term, k0); }}\n')
  # ragged history: filter b smooths its first len[b] rows, times t [T, B]; returns the call's cudaError_t (see _hist_idx)
  brr = "const double *hx_pred, const double *hP_pred, const double *hx_filt, const double *hP_filt, const double *t, const int *len, double *xs, double *Ps, int T, long long B, const int *quat_idxs, int n_quat, int norm_quats, void *stream"
  hdr.append(f"int {name}_batch_rts_ragged({brr});")
  c.append(f'extern "C" int {name}_batch_rts_ragged({brr}) {{ return rnb::call_status([&] {{ rnb::batch_rts_ragged<{model}>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, len, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream); }}); }}\n')
  # one SEGMENT of a ragged history: filter b's rows are its global rows k0[b] ..; with term[b] its row len[b] - 1 is the
  # first row of its segment behind and the recursion starts from (x_term[b], P_term[b]).  packed selects the packed
  # covariance layout (an argument, not a _packed name).  int result (see _hist_idx); refused above EDIM 32
  brg = ("const double *hx_pred, const double *hP_pred, const double *hx_filt, const double *hP_filt, const double *t, const int *len, "
         "const unsigned char *term, const long long *k0, const double *x_term, const double *P_term, double *xs, double *Ps, int T, "
         "long long B, const int *quat_idxs, int n_quat, int norm_quats, int packed, void *stream")
  hdr.append(f"int {name}_batch_rts_ragged_segment({brg});")
  c.append(f'extern "C" int {name}_batch_rts_ragged_segment({brg}) {{ return rnb::call_status([&] {{ rnb::batch_rts_ragged_segment<{model}>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, len, term, k0, x_term, P_term, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, packed, stream); }}); }}\n')
  # the three smoothers over packed histories (REDNOSE_PACKED_HIST): hP_pred, hP_filt, Ps and P_term are
  # [.., <name>_packed_P_doubles()]; int results like the ragged ones, refused where the pair kernel does not record them
  for suffix, args, call in (("rts", br, f"batch_rts<{model}, true>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, t_per_filter, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream)"),
                             ("rts_segment", brs, f"batch_rts<{model}, true>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, t_per_filter, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream, x_term, P_term, k0)"),
                             ("rts_ragged", brr, f"batch_rts_ragged<{model}, true>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, len, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream)")):
    hdr.append(f"int {name}_batch_{suffix}_packed({args});")
    c.append(f'extern "C" int {name}_batch_{suffix}_packed({args}) {{ return rnb::call_status([&] {{ rnb::{call}; }}); }}\n')
  # restore filters idx[e] of the resident x / P from row hist_row[e] of a ragged history's x_filt / P_filt slabs (a
  # rewind); flags: REDNOSE_PACKED_HIST / REDNOSE_PACKED_P give the two layouts.  int result (see _hist_idx)
  rh = "const double *hx_filt, const double *hP_filt, const int *idx, const int *hist_row, long long n, long long hist_B, double *x, double *P, int flags, void *stream"
  hdr.append(f"int {name}_batch_restore_hist({rh});")
  c.append(f'extern "C" int {name}_batch_restore_hist({rh}) {{ return rnb::call_status([&] {{ rnb::batch_restore_hist<{model}>(hx_filt, hP_filt, idx, hist_row, n, hist_B, x, P, flags, stream); }}); }}\n')
  # doubles per filter and step of a main-block prediction history (MEDIM^2), 0 where it does not exist (EDIM <= 32)
  hdr.append(f"int {name}_main_pred_doubles(void);")
  c.append(f'extern "C" int {name}_main_pred_doubles(void) {{ return {MEDIM * MEDIM if EDIM > 32 else 0}; }}\n')
  if EDIM > 32:
    # the two smoothers over a main-block prediction history: hP_pred [T, B, MEDIM, MEDIM]; without a terminal estimate
    # the recursion starts from hP_pred_last [B, EDIM, EDIM], the full prediction of the newest row
    for suffix, args, tail in (("rts", br, ""), ("rts_segment", brs, ", x_term, P_term, k0")):
      args = args.replace(", void *stream", ", const double *hP_pred_last, void *stream")
      hdr.append(f"int {name}_batch_{suffix}_mainhist({args});")
      c.append(f'extern "C" int {name}_batch_{suffix}_mainhist({args}) {{ return rnb::call_status([&] {{ rnb::batch_rts<{model}, false, true>(ctx_(), hx_pred, hP_pred, hx_filt, hP_filt, t, t_per_filter, xs, Ps, T, B, quat_idxs, n_quat, norm_quats, stream{tail if tail else ", nullptr, nullptr, 0"}, hP_pred_last); }}); }}\n')

  if msckf:
    ba = "double *x, double *P, long long B, void *stream"
    hdr.append(f"void {name}_batch_augment({ba});")
    c.append(f'extern "C" void {name}_batch_augment({ba}) {{ rnb::launch_augment<{model}>(x, P, B, {int(dim_augment)}, {int(dim_augment_err)}, (cudaStream_t)stream); }}\n')
    # the shift of the n filters idx[e] (distinct) only, for filters on their own clocks; full covariance layout (packed
    # flags refused).  int result (see _hist_idx)
    bai = "double *x, double *P, const int *idx, long long n, int flags, void *stream"
    hdr.append(f"int {name}_batch_augment_idx({bai});")
    c.append(f'extern "C" int {name}_batch_augment_idx({bai}) {{ return rnb::call_status([&] {{ rnb::launch_augment_idx<{model}>(x, P, idx, n, flags, {int(dim_augment)}, {int(dim_augment_err)}, (cudaStream_t)stream); }}); }}\n')

  # ---- descriptor + ekf_get (rednose/helpers/ekf.h:16-42) ----
  kl = [kd['kind'] for kd in kinds]
  def arr(ctype, vals):
    return f"{{ {', '.join(str(v) for v in vals)} }}" if vals else "{ 0 }"
  c.append("\nnamespace {\n")
  c.append(f"const int kinds_[] = {arr('int', kl)};\n")
  c.append(f"const int zdims_[] = {arr('int', [kd['zdim'] for kd in kinds])};\n")
  c.append(f"const int eadims_[] = {arr('int', [kd['eadim'] for kd in kinds])};\n")
  c.append(f"const int feature_[] = {arr('int', [int(kd['feature']) for kd in kinds])};\n")
  c.append(f"const int maha_[] = {arr('int', [int(kd['maha']) for kd in kinds])};\n")
  c.append(f"const rednose_leaf3_fn hs_[] = {arr('', [f'{name}_h_{k}' for k in kl])};\n")
  c.append(f"const rednose_leaf3_fn Hs_[] = {arr('', [f'{name}_H_{k}' for k in kl])};\n")
  c.append(f"const rednose_leaf3_fn Hes_[] = {arr('', [(f'{name}_He_{kd['kind']}' if kd['feature'] else 'nullptr') for kd in kinds])};\n")
  c.append(f"const rednose_update_fn updates_[] = {arr('', [f'{name}_update_{k}' for k in kl])};\n")
  c.append(f"const rednose_batch_update_fn batch_updates_[] = {arr('', [f'{name}_batch_update_{k}' for k in kl])};\n")
  c.append(f"const rednose_batch_step_fn batch_steps_[] = {arr('', [f'{name}_batch_step_{k}' for k in kl])};\n")
  c.append(f"const rednose_host_step_fn host_steps_[] = {arr('', [f'{name}_host_step_{k}' for k in kl])};\n")
  set_names = ', '.join(f'"{g}"' for g in gvars) if gvars else 'nullptr'
  set_fns = ', '.join(f'{name}_set_{g}' for g in gvars) if gvars else 'nullptr'
  c.append(f"const char* const set_names_[] = {{ {set_names} }};\n")
  c.append(f"const rednose_set_fn sets_[] = {{ {set_fns} }};\n")
  ex_names = ', '.join(f'"{e[0]}"' for e in extras) if extras else 'nullptr'
  ex_fns = ', '.join(f'(void*){name}_{e[0]}' for e in extras) if extras else 'nullptr'
  c.append(f"const char* const extra_names_[] = {{ {ex_names} }};\n")
  c.append(f"void* const extra_fns_[] = {{ {ex_fns} }};\n")
  c.append("const rednose_ekf_desc desc_ = {\n")
  c.append(f"  {ABI_VERSION}, \"{name}\", {DIM}, {EDIM}, {MEDIM}, {len(kl)}, kinds_, zdims_, eadims_, feature_, maha_,\n")
  c.append(f"  {name}_f_fun, {name}_F_fun, {name}_err_fun, {name}_inv_err_fun, {name}_H_mod_fun, {name}_predict,\n")
  c.append("  hs_, Hs_, Hes_, updates_,\n")
  c.append(f"  {NG}, set_names_, sets_, {len(extras)}, extra_names_, extra_fns_,\n")
  c.append(f"  {name}_batch_predict, batch_updates_, batch_steps_, host_steps_, {name}_batch_rts,\n")
  c.append("};\n}  // namespace\n")
  c.append('extern "C" void* ekf_get() { return (void*)&desc_; }\n')
  c.append(f'extern "C" int {name}_cuda_status() {{ int s = rnb::last_status(); rnb::last_status() = 0; return s; }}\n')
  c.append('static void __attribute__((constructor)) rnb_self_register_() { rednose_b200_register_weak(&desc_); }\n')

  header = "#pragma once\n#include \"rednose_b200.h\"\n#ifdef __cplusplus\nextern \"C\" {\n#endif\n"
  header += "\n".join(hdr) + "\n"
  header += f"int {name}_cuda_status(void);\nvoid* ekf_get(void);\n"
  header += "#ifdef __cplusplus\n}\n#endif\n"

  os.makedirs(folder, exist_ok=True)
  cu_path = os.path.join(folder, f"{name}.cu")
  with open(os.path.join(folder, f"{name}.h"), 'w', encoding='utf-8') as f:
    f.write(header)
  with open(cu_path, 'w', encoding='utf-8') as f:
    f.write("".join(out))
    f.write('extern "C" {\n' + "\n".join(h for h in hdr) + "\n}\n")
    f.write("".join(c))

  if compile_lib is None:
    compile_lib = os.environ.get("REDNOSE_B200_NO_COMPILE", "0") != "1"
  if compile_lib:
    _build.compile_filter(folder, name)
  return cu_path
