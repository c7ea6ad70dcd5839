"""High-precision reference for one filter: predict, update and RTS step in mpmath at 40 significant digits.

The same operations as oracle/ekf_oracle_core.h (predict F P F^T + dt Q; update with S, gain, optional Mahalanobis
gate that inflates R by 1e16, Joseph form, err_fun injection) and oracle/rts_numpy.py (the backward recursion), with
quaternion normalisation after predict / update as set by the step flags.  The leaf functions are lambdified with
modules="mpmath" from the filter's own sympy definition, with F, H and H_mod derived the way codegen.gen_code derives
them, so nothing is rounded to float64 between the float64 inputs and the result.  The result is therefore the
exact answer to rounding at 1e-40, against which float64 implementations (the CUDA kernels, the CPU oracle) can each
be measured.

Pure Python: a 22x22 product costs about 10 ms, so keep it to a few filters and a few dozen steps.
It needs neither the reference checkout nor any compiled library.
"""
import functools

import numpy as np
import sympy as sp
from mpmath import mp

DPS = 40


def _lam(args, exprs):
  return sp.lambdify(args, list(exprs), modules="mpmath")


@functools.lru_cache(maxsize=None)
def live_model():
  from rednose_b200.filters.live import LiveKalman
  return HiPrecModel(**LiveKalman.symbolic_model())


class HiPrecModel:
  """Leaf functions of one ESKF model (the arguments gen_code receives), evaluated in mpmath."""

  def __init__(self, f_sym, dt_sym, x_sym, obs_eqs, dim_x, dim_err, eskf_params, maha_test_kinds=(), **_):
    self.dim_x, self.dim_err = int(dim_x), int(dim_err)
    inject, invert, H_mod_sym, f_err_sym, x_err_sym = eskf_params[:5]
    err = sp.Matrix(x_err_sym)
    F_sym = sp.Matrix(f_err_sym).jacobian(err).subs({s: 0 for s in err})   # gen_code: F = d f_err / d x_err at x_err = 0
    self._f = _lam([x_sym, dt_sym], sp.Matrix(f_sym))
    self._F = _lam([x_sym, dt_sym], F_sym)
    self._H_mod = _lam([x_sym], sp.Matrix(H_mod_sym))
    self._err = _lam([inject[1], inject[2]], sp.Matrix(inject[0]))
    self._inv_err = _lam([invert[1], invert[2]], sp.Matrix(invert[0]))
    self._h, self._H, self.zdim = {}, {}, {}
    for h_sym, kind, ea_sym in obs_eqs:
      h_sym = sp.Matrix(h_sym)
      args = [x_sym] + ([ea_sym] if ea_sym is not None else [])
      self._h[int(kind)] = _lam(args, h_sym)
      self._H[int(kind)] = _lam(args, h_sym.jacobian(sp.Matrix(x_sym)))
      self.zdim[int(kind)] = int(h_sym.shape[0])
    self.maha_test_kinds = set(int(k) for k in maha_test_kinds)

  # ---- leaf functions on mp.matrix column vectors ----
  def f(self, x, dt):
    return mp.matrix(self._f(x, dt))

  def F(self, x, dt):
    return _reshape(self._F(x, dt), self.dim_err, self.dim_err)

  def H_mod(self, x):
    return _reshape(self._H_mod(x), self.dim_x, self.dim_err)

  def h(self, kind, x, ea=None):
    return mp.matrix(self._h[kind](x, *([ea] if ea is not None else [])))

  def H(self, kind, x, ea=None):
    return _reshape(self._H[kind](x, *([ea] if ea is not None else [])), self.zdim[kind], self.dim_x)

  def err_fun(self, nom, delta):
    return mp.matrix(self._err(nom, delta))

  def inv_err_fun(self, nom, true):
    return mp.matrix(self._inv_err(nom, true))

  # ---- one filter ----
  def predict(self, x, P, Q, dt):
    F = self.F(x, dt)
    return self.f(x, dt), F * P * F.T + dt * Q

  def update(self, kind, x, P, z, R, ea=None, maha_thresh=None):
    """Returns (x, P, y).  maha_thresh: the gate of a Mahalanobis-tested kind (None: no gate)."""
    y = z - self.h(kind, x, ea)
    He = self.H(kind, x, ea) * self.H_mod(x)
    S = He * P * He.T + R
    if maha_thresh is not None and (y.T * mp.inverse(S) * y)[0, 0] > maha_thresh:
      R = R * mp.mpf(10) ** 16
      S = He * P * He.T + R
    K = (mp.inverse(S) * He * P.T).T                               # K^T = S^-1 (He P^T), as the oracle forms it
    IKH = mp.eye(self.dim_err) - K * He
    P = IKH * P * IKH.T + K * R * K.T
    return self.err_fun(x, K * y), P, y

  @staticmethod
  def normalize(x, quat_idxs):
    x = x.copy()
    for i in quat_idxs:
      n = mp.sqrt(sum(x[i + c] ** 2 for c in range(4)))
      for c in range(4):
        x[i + c] = x[i + c] / n
    return x

  def step(self, kind, x, P, Q, dt, z, R, quat_idxs=(), flags=3, maha_thresh=None):
    """Fused predict + update with the step flags of the kernels (1: normalise after predict, 2: after update)."""
    x, P = self.predict(x, P, Q, dt)
    if flags & 1:
      x = self.normalize(x, quat_idxs)
    x, P, y = self.update(kind, x, P, z, R, maha_thresh=maha_thresh)
    if flags & 2:
      x = self.normalize(x, quat_idxs)
    return x, P, y

  def rts(self, x_pred, x_filt, P_pred, P_filt, t, norm_quats=False):
    """oracle/rts_numpy.rts_smooth for one filter (lists of mp matrices); returns (xs, Ps) in time order."""
    T = len(x_pred)
    xk_n, Pk_n = x_pred[-1].copy(), P_pred[-1].copy()
    xs, Ps = [xk_n], [Pk_n]
    for k in range(T - 2, -1, -1):
      xk1_n = self.normalize(xk_n, [3]) if norm_quats else xk_n    # the reference's hard-coded slice 3:7
      if norm_quats:
        xs[-1] = xk1_n
      Pk1_n = Pk_n
      xk1_k, Pk1_k, xk_k, Pk_k = x_pred[k + 1], P_pred[k + 1], x_filt[k], P_filt[k]
      F = self.F(xk_k, t[k + 1] - t[k])
      C = (mp.inverse(Pk1_k) * F * Pk_k.T).T                      # solve(Pk1_k, F Pk_k^T)^T
      xk_n = self.err_fun(xk_k, C * self.inv_err_fun(xk1_k, xk1_n))
      Pk_n = Pk_k + C * (Pk1_n - Pk1_k) * C.T
      xs.append(xk_n)
      Ps.append(Pk_n)
    return xs[::-1], Ps[::-1]


def _reshape(flat, m, n):
  A = mp.matrix(m, n)
  for i in range(m):
    for j in range(n):
      A[i, j] = flat[i * n + j]
  return A


def to_mp(a):
  """float64 array -> mp.matrix (a 1-D array becomes a column); every float64 is exact in mpmath."""
  a = np.asarray(a, dtype=np.float64)
  if a.ndim == 1:
    return mp.matrix([mp.mpf(float(v)) for v in a])
  return mp.matrix([[mp.mpf(float(v)) for v in row] for row in a])


def to_np(A):
  """mp.matrix -> float64 array (a column vector becomes 1-D), rounded once to nearest."""
  out = np.array([[float(A[i, j]) for j in range(A.cols)] for i in range(A.rows)])
  return out[:, 0] if A.cols == 1 else out


class workdps:
  """with workdps(): evaluate at DPS significant digits."""

  def __enter__(self):
    self._ctx = mp.workdps(DPS)
    self._ctx.__enter__()

  def __exit__(self, *exc):
    return self._ctx.__exit__(*exc)


def live_step(kind, x, P, Q, dt, z, R, quat_idxs=(3,), flags=3):
  """One fused step of the live model per filter, on float64 batches [B, ...]; returns float64 (x, P, y)."""
  m = live_model()
  xs, Ps, ys = [], [], []
  with workdps():
    Qm = to_mp(Q)
    for b in range(x.shape[0]):
      xb, Pb, yb = m.step(kind, to_mp(x[b]), to_mp(P[b]), Qm, mp.mpf(float(dt)), to_mp(z[b]), to_mp(R[b]), quat_idxs, flags)
      xs.append(to_np(xb)); Ps.append(to_np(Pb)); ys.append(to_np(yb))
  return np.stack(xs), np.stack(Ps), np.stack(ys)


def live_rts(x_pred, x_filt, P_pred, P_filt, t, norm_quats=True):
  """RTS over the float64 history of ONE filter ([T, DIM], [T, EDIM, EDIM], t [T]); returns float64 (xs, Ps)."""
  m = live_model()
  with workdps():
    args = [[to_mp(a) for a in arr] for arr in (x_pred, x_filt, P_pred, P_filt)]
    xs, Ps = m.rts(*args, [mp.mpf(float(v)) for v in t], norm_quats=norm_quats)
    return np.stack([to_np(v) for v in xs]), np.stack([to_np(v) for v in Ps])
