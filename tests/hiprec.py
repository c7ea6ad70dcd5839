"""High-precision reference for one filter: predict, update and RTS step in mpmath at 40 significant digits.

The same operations as oracle/ekf_oracle_core.h (predict F P F^T + dt Q; update with S, gain, optional Mahalanobis
gate that inflates R by 1e16, err_fun injection; the covariance as P - K H P, which at 40 digits equals the oracle's Joseph
form far below float64 rounding) and oracle/rts_numpy.py (the backward recursion), with
quaternion normalisation after predict / update as set by the step flags.  The leaf functions are lambdified with
modules="mpmath" from the filter's own sympy definition, with F, H and H_mod derived the way codegen.gen_code derives
them (for a plain EKF: identity injection and H_mod = I), so nothing is rounded to float64 between the float64 inputs
and the result.  The result is therefore the exact answer to rounding at 1e-40, against which float64 implementations
(the CUDA kernels, the CPU oracle) can each be measured.

Any model gen_code accepts works: ESKF or plain, observation kinds with extra arguments, global variables
(``HiPrecModel.gv``), and the MSCKF layout (``msckf_params``): a feature-track kind is projected on an orthonormal basis
of the left null space of He = dh/d(ea), computed at 40 digits, and ``augment`` is the clone-window shift.  x and P do not
depend on the basis; the projected innovation does, so only its norm can be compared.  The batch helpers (``step``,
``predict``, ``update``, ``maha``, ``augment``, ``rts``) take float64 arrays over filters and return float64 arrays.

Pure Python: a 22x22 product costs about 10 ms, so keep it to a few filters and a few dozen steps.
It needs neither the reference checkout nor any compiled library.
"""
import functools

import numpy as np
import sympy as sp
from mpmath import mp

DPS = 40


def _lam(args, exprs, modules="mpmath"):
  return sp.lambdify(args, list(exprs), modules=modules)


@functools.lru_cache(maxsize=None)
def live_model():
  from rednose_b200.filters.live import LiveKalman
  return HiPrecModel(**LiveKalman.symbolic_model())


@functools.lru_cache(maxsize=None)
def model_of(filter_cls):
  """The HiPrecModel of a filter class with ``symbolic_model()`` (cached: lambdifying a 32-state model takes seconds)."""
  return HiPrecModel(**filter_cls.symbolic_model())


class HiPrecModel:
  """Leaf functions of one model (the arguments gen_code receives), evaluated in mpmath."""

  def __init__(self, f_sym, dt_sym, x_sym, obs_eqs, dim_x, dim_err, eskf_params=None, maha_test_kinds=(), global_vars=None,
               msckf_params=None, **_):
    self.dim_x, self.dim_err = int(dim_x), int(dim_err)
    # MSCKF layout (ekf_sym.py:57-73): (DIM_MAIN, DAUG, MEDIM, EAUG, N, feature-track kinds)
    self.msckf = [int(v) for v in msckf_params[:5]] if msckf_params else None
    self.feature_kinds = set(int(k) for k in msckf_params[5]) if msckf_params else set()
    if eskf_params:
      inject, invert, H_mod_sym, f_err_sym, x_err_sym = eskf_params[:5]
      err = sp.Matrix(x_err_sym)
      F_sym = sp.Matrix(f_err_sym).jacobian(err).subs({s: 0 for s in err})   # gen_code: F = d f_err / d x_err at x_err = 0
    else:                                                                      # gen_code's plain EKF (codegen/__init__.py)
      nom_x = sp.MatrixSymbol('nom_x', dim_x, 1)
      true_x = sp.MatrixSymbol('true_x', dim_x, 1)
      delta_x = sp.MatrixSymbol('delta_x', dim_x, 1)
      inject = [sp.Matrix(nom_x + delta_x), nom_x, delta_x]
      invert = [sp.Matrix(true_x - nom_x), nom_x, true_x]
      H_mod_sym = sp.eye(dim_x)
      F_sym = sp.Matrix(f_sym).jacobian(sp.Matrix(x_sym))
    self.gvars = list(global_vars) if global_vars is not None else []
    self.gv = [0.0] * len(self.gvars)                                          # the library's values before any set
    g = self.gvars
    self._sym = dict(f=([x_sym, dt_sym] + g, sp.Matrix(f_sym)), F=([x_sym, dt_sym] + g, F_sym),
                     H_mod=([x_sym] + g, sp.Matrix(H_mod_sym)), err=([inject[1], inject[2]] + g, sp.Matrix(inject[0])),
                     inv_err=([invert[1], invert[2]] + g, sp.Matrix(invert[0])))
    self.zdim, self.eadim = {}, {}
    for h_sym, kind, ea_sym in obs_eqs:
      h_sym = sp.Matrix(h_sym)
      args = [x_sym] + ([ea_sym] if ea_sym is not None else []) + g
      self._sym[('h', int(kind))] = (args, h_sym)
      self._sym[('H', int(kind))] = (args, h_sym.jacobian(sp.Matrix(x_sym)))
      if int(kind) in self.feature_kinds:
        self._sym[('He', int(kind))] = (args, h_sym.jacobian(sp.Matrix(ea_sym)))
      self.zdim[int(kind)] = int(h_sym.shape[0])
      self.eadim[int(kind)] = int(ea_sym.shape[0]) if ea_sym is not None else 0
    self.maha_test_kinds = set(int(k) for k in maha_test_kinds)
    self._fns = {}

  def _fn(self, key, modules="mpmath"):
    if (key, modules) not in self._fns:
      args, expr = self._sym[key]
      self._fns[(key, modules)] = _lam(args, expr, modules)
    return self._fns[(key, modules)]

  def _g(self):
    return [mp.mpf(float(v)) for v in self.gv]

  def maha_thresh(self, kind):
    """The gate of a Mahalanobis-tested kind as the generated code holds it (float64 chi2_ppf(0.95, ZDIM)), else None."""
    from rednose_b200.chi2 import chi2_ppf
    return mp.mpf(float(chi2_ppf(0.95, self.zdim[kind]))) if kind in self.maha_test_kinds else None

  # ---- leaf functions on mp.matrix column vectors ----
  def f(self, x, dt):
    return mp.matrix(self._fn('f')(x, dt, *self._g()))

  def F(self, x, dt):
    return _reshape(self._fn('F')(x, dt, *self._g()), self.dim_err, self.dim_err)

  def H_mod(self, x):
    return _reshape(self._fn('H_mod')(x, *self._g()), self.dim_x, self.dim_err)

  def h(self, kind, x, ea=None):
    return mp.matrix(self._fn(('h', kind))(x, *([ea] if ea is not None else []), *self._g()))

  def H(self, kind, x, ea=None):
    return _reshape(self._fn(('H', kind))(x, *([ea] if ea is not None else []), *self._g()), self.zdim[kind], self.dim_x)

  def He(self, kind, x, ea):
    """d h / d ea of a feature-track kind (ZDIM x EADIM)."""
    return _reshape(self._fn(('He', kind))(x, ea, *self._g()), self.zdim[kind], self.eadim[kind])

  def err_fun(self, nom, delta):
    return mp.matrix(self._fn('err')(nom, delta, *self._g()))

  def inv_err_fun(self, nom, true):
    return mp.matrix(self._fn('inv_err')(nom, true, *self._g()))

  # ---- one filter ----
  def predict(self, x, P, Q, dt):
    F = self.F(x, dt)
    # F (F P)^T, transposed: the sparse F is the left operand of both products (an MSCKF's F is the identity on the
    # clones, so this costs ~nnz(F) E instead of E^3 products)
    return self.f(x, dt), _mul(F, _mul(F, P).T).T + dt * Q

  def maha(self, kind, x, P, z, R, ea=None):
    """y^T S^-1 y of one observation (no state change; a feature kind is not projected, ekf_sym.py:626-649)."""
    y = z - self.h(kind, x, ea)
    He = _mul(self.H(kind, x, ea), self.H_mod(x))
    return (y.T * mp.inverse(_mul(He, P) * He.T + R) * y)[0, 0]

  def null_basis(self, kind, x, ea):
    """An orthonormal basis A (ZDIM x (ZDIM - EADIM)) of the left null space of He = dh/d(ea): the trailing columns of
    the full QR factor of He at 40 digits."""
    Qf, _ = mp.qr(self.He(kind, x, ea), mode='full')
    Z, EA = self.zdim[kind], self.eadim[kind]
    return Qf[:, EA:Z] if Z - EA > 1 else mp.matrix([[Qf[i, EA]] for i in range(Z)])

  def update(self, kind, x, P, z, R, ea=None, maha_thresh=None):
    """Returns (x, P, y).  maha_thresh: the gate of a Mahalanobis-tested kind (None: no gate).  A feature-track kind is
    projected on the left null space of He (ekf_c.c:66-85): y' = A^T y, H' = A^T H_err, R' = A^T R A, and y is y'."""
    y = z - self.h(kind, x, ea)
    He = _mul(self.H(kind, x, ea), self.H_mod(x))
    if kind in self.feature_kinds:
      A = self.null_basis(kind, x, ea)
      y, He, R = A.T * y, _mul(A.T, He), A.T * R * A
    HP = _mul(He, P)
    S = HP * He.T + R
    if maha_thresh is not None and (y.T * mp.inverse(S) * y)[0, 0] > maha_thresh:
      R = R * mp.mpf(10) ** 16
      S = HP * He.T + R
    K = (mp.inverse(S) * _mul(He, P.T)).T                          # K^T = S^-1 (He P^T), as the oracle forms it
    # P - K (He P): with the exact gain this equals the oracle's Joseph form (I - K He) P (I - K He)^T + K R K^T, and
    # at 40 digits the two differ by ~1e-38 x cond(S), far below float64; it costs E Z E instead of 2 E^3 products
    P = P - K * HP
    return self.err_fun(x, K * y), P, y

  def augment(self, x, P):
    """The MSCKF clone-window shift (ekf_sym.py:365-391): drop the oldest clone, append a copy of the first DAUG main
    states; the same selection on the rows and columns of P (the reference's selection-matrix products, whose every
    entry is one product by 1)."""
    d1, d3, d2, d4, _ = self.msckf
    D, E = self.dim_x, self.dim_err
    sx = list(range(d1)) + list(range(d1 + d3, D)) + list(range(d3))
    se = list(range(d2)) + list(range(d2 + d4, E)) + list(range(d4))
    xo = mp.matrix([x[i] for i in sx])
    Po = mp.matrix(E, E)
    for i in range(E):
      for j in range(E):
        Po[i, j] = P[se[i], se[j]]
    return xo, Po

  @staticmethod
  def normalize(x, quat_idxs):
    x = x.copy()
    for i in quat_idxs:
      n = mp.sqrt(sum(x[i + c] ** 2 for c in range(4)))
      for c in range(4):
        x[i + c] = x[i + c] / n
    return x

  def step(self, kind, x, P, Q, dt, z, R, quat_idxs=(), flags=3, maha_thresh=None, ea=None):
    """Fused predict + update with the step flags of the kernels (1: normalise after predict, 2: after update).
    z, R, ea may be lists: several observations of one kind at one timestamp, applied in order."""
    x, P = self.predict(x, P, Q, dt)
    if flags & 1:
      x = self.normalize(x, quat_idxs)
    obs = list(zip(z, R, ea if ea is not None else [None] * len(z))) if isinstance(z, list) else [(z, R, ea)]
    ys = []
    for zo, Ro, eo in obs:
      x, P, y = self.update(kind, x, P, zo, Ro, eo, maha_thresh=maha_thresh)
      ys.append(y)
      if flags & 2:
        x = self.normalize(x, quat_idxs)
    return x, P, (ys if isinstance(z, list) else ys[0])

  def rts(self, x_pred, x_filt, P_pred, P_filt, t, norm_quats=False, quat_idxs=(3,)):
    """oracle/rts_numpy.rts_smooth for one filter (lists of mp matrices); returns (xs, Ps) in time order.

    With ``msckf_params`` only the main block is smoothed (ekf_sym.py:651-690 with dim_main / dim_main_err): C is formed
    from the main blocks of F, P_{k|k} and P_{k+1|k}, only delta[:d2] of the full inv_err delta is replaced by C delta[:d2],
    x_{k|N} is x_{k|k} with [:d1] taken from err_fun(x_{k|k}, delta), and P_{k|N} is P_{k|k} with the main block
    replaced.  Every quaternion in `quat_idxs` is normalised, clones included."""
    d1, d2 = (self.msckf[0], self.msckf[2]) if self.msckf else (self.dim_x, self.dim_err)
    T = len(x_pred)
    xk_n, Pk_n = x_pred[-1].copy(), P_pred[-1].copy()
    xs, Ps = [xk_n], [Pk_n]
    for k in range(T - 2, -1, -1):
      xk1_n = self.normalize(xk_n, quat_idxs) if norm_quats else xk_n    # the reference's hard-coded slice 3:7 by default
      if norm_quats:
        xs[-1] = xk1_n
      Pk1_n = Pk_n
      xk1_k, Pk1_k, xk_k, Pk_k = x_pred[k + 1], P_pred[k + 1], x_filt[k], P_filt[k]
      F = _block(self.F(xk_k, t[k + 1] - t[k]), d2)
      Pk1_k_m, Pk_k_m = _block(Pk1_k, d2), _block(Pk_k, d2)
      C = _mul(mp.inverse(Pk1_k_m), _mul(F, Pk_k_m.T)).T          # solve(Pk1_k, F Pk_k^T)^T on the main block
      delta = self.inv_err_fun(xk1_k, xk1_n)
      cd = C * mp.matrix([delta[i] for i in range(d2)])
      for i in range(d2):
        delta[i] = cd[i]
      xe = self.err_fun(xk_k, delta)
      xk_n = xk_k.copy()
      for i in range(d1):
        xk_n[i] = xe[i]
      Pm = Pk_k_m + _mul(_mul(C, _block(Pk1_n, d2) - Pk1_k_m), C.T)
      Pk_n = Pk_k.copy()
      for i in range(d2):
        for j in range(d2):
          Pk_n[i, j] = Pm[i, j]
      xs.append(xk_n)
      Ps.append(Pk_n)
    return xs[::-1], Ps[::-1]

  # ---- the same step in plain float64 numpy, from the same leaf functions (a check of the reference itself) ----
  def np_leaf(self, key, *args):
    """Leaf `key` ('f', 'F', 'H_mod', 'err', 'inv_err', ('h', kind), ('H', kind)) in float64; vectors are 1-D arrays,
    scalars (dt) stay scalars.  Returns the flat float64 output."""
    conv = [np.asarray(a, dtype=np.float64).reshape(-1, 1) if np.ndim(a) else float(a) for a in args]
    return np.array(self._fn(key, "numpy")(*conv, *self.gv), dtype=np.float64).reshape(-1)

  def step_f64(self, kind, x, P, Q, dt, z, R, quat_idxs=(), flags=3, ea=None, predict=True):
    """Fused step in float64 (no gate, Joseph form), x [DIM], P [E, E]; returns (x, P, y).  predict=False: the update
    alone (Q, dt unused)."""
    E, D = self.dim_err, self.dim_x
    if predict:
      F = self.np_leaf('F', x, dt).reshape(E, E)
      x = self.np_leaf('f', x, dt)
      P = F @ P @ F.T + dt * Q
    if predict and flags & 1:
      x = _np_normalize(x, quat_idxs)
    ea_args = [ea] if ea is not None else []
    He = self.np_leaf(('H', kind), x, *ea_args).reshape(self.zdim[kind], D) @ self.np_leaf('H_mod', x).reshape(D, E)
    y = z - self.np_leaf(('h', kind), x, *ea_args)
    if kind in self.feature_kinds:            # left-null-space projection with numpy's own (complete) QR basis
      Hea = self.np_leaf(('He', kind), x, ea).reshape(self.zdim[kind], self.eadim[kind])
      A = np.linalg.qr(Hea, mode='complete')[0][:, self.eadim[kind]:]
      y, He, R = A.T @ y, A.T @ He, A.T @ R @ A
    S = He @ P @ He.T + R
    K = np.linalg.solve(S, He @ P.T).T
    IKH = np.eye(E) - K @ He
    P = IKH @ P @ IKH.T + K @ R @ K.T
    x = self.np_leaf('err', x, K @ y)
    if flags & 2:
      x = _np_normalize(x, quat_idxs)
    return x, P, y


def _np_normalize(x, quat_idxs):
  x = x.copy()
  for i in quat_idxs:
    x[i:i + 4] /= np.linalg.norm(x[i:i + 4])
  return x


def _mul(A, B):
  """A B for mp matrices, skipping the zero entries of A (F, H_err and I - K H_err are sparse or block sparse); several
  times faster than mp.matrix's own product, with the same correctly rounded dot products (mp.fdot)."""
  cols = [[B[k, j] for k in range(B.rows)] for j in range(B.cols)]
  out = mp.matrix(A.rows, B.cols)
  for i in range(A.rows):
    nz = [(k, A[i, k]) for k in range(A.cols) if A[i, k]]
    if nz:
      for j in range(B.cols):
        c = cols[j]
        out[i, j] = mp.fdot((a, c[k]) for k, a in nz)
  return out


def _block(A, n):
  """The leading n x n block of an mp matrix (A itself when it is n x n)."""
  if A.rows == n and A.cols == n:
    return A
  out = mp.matrix(n, n)
  for i in range(n):
    for j in range(n):
      out[i, j] = A[i, j]
  return out


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


def to_np(A, matrix=False):
  """mp.matrix -> float64 array (a column vector becomes 1-D unless `matrix`), rounded once to nearest."""
  out = np.array([[float(A[i, j]) for j in range(A.cols)] for i in range(A.rows)])
  return out[:, 0] if A.cols == 1 and not matrix else out


class workdps:
  """with workdps(): evaluate at DPS significant digits."""

  def __enter__(self):
    self._ctx = mp.workdps(DPS)
    self._ctx.__enter__()

  def __exit__(self, *exc):
    return self._ctx.__exit__(*exc)


# ---- batch helpers: float64 arrays over the filters `sel` of a batch in, float64 arrays out ----
def _per_obs(z, R, ea, b):
  """Observations of filter b as mp lists: z / ea [B, n, m] or [B, m]; R [Z, Z] (shared), [B, Z, Z] or [B, n, Z, Z]."""
  zb = np.asarray(z)[b]
  multi = zb.ndim == 2
  zl = [zb[o] for o in range(zb.shape[0])] if multi else [zb]
  R = np.asarray(R)
  if R.ndim == 2:
    Rl = [R] * len(zl)
  elif R.ndim == 3:
    Rl = [R[b]] * len(zl)
  else:
    Rl = [R[b, o] for o in range(R.shape[1])]
  if ea is None:
    el = [None] * len(zl)
  else:
    eb = np.asarray(ea)[b]
    el = [eb[o] for o in range(eb.shape[0])] if eb.ndim == 2 else [eb]
  return multi, [to_mp(v) for v in zl], [to_mp(v) for v in Rl], [to_mp(v) if v is not None else None for v in el]


def step(m, kind, x, P, Q, dt, z, R, ea=None, quat_idxs=(), flags=3, sel=None, predict=True, update=True, gate=True):
  """Fused step of model m on the filters `sel` (default all) of a float64 batch: x [B, DIM], P [B, E, E], dt scalar or
  [B], z [B, (n,) Z], R shared [Z, Z] or per filter [B, (n,) Z, Z], ea [B, (n,) EA].  Returns float64 (x, P, y) for
  the selected filters, y shaped like their z.  gate=False skips the Mahalanobis gate of a gated kind (the result the
  kernel must give for a filter the gate lets through)."""
  sel = range(x.shape[0]) if sel is None else sel
  thresh = m.maha_thresh(kind) if (update and gate) else None
  xs, Ps, ys = [], [], []
  with workdps():
    Qm = to_mp(Q) if predict else None
    for b in sel:
      xb, Pb = to_mp(x[b]), to_mp(P[b])
      if predict:
        dtb = mp.mpf(float(np.asarray(dt)[b] if np.ndim(dt) else dt))
        xb, Pb = m.predict(xb, Pb, Qm, dtb)
        if flags & 1:
          xb = m.normalize(xb, quat_idxs)
      yb = None
      if update:
        multi, zl, Rl, el = _per_obs(z, R, ea, b)
        yl = []
        for zo, Ro, eo in zip(zl, Rl, el):
          xb, Pb, y = m.update(kind, xb, Pb, zo, Ro, eo, maha_thresh=thresh)
          yl.append(to_np(y))
          if flags & 2:
            xb = m.normalize(xb, quat_idxs)
        yb = np.stack(yl) if multi else yl[0]
      xs.append(to_np(xb)); Ps.append(to_np(Pb, matrix=True)); ys.append(yb)
  return np.stack(xs), np.stack(Ps), (np.stack(ys) if update else None)


def predict(m, x, P, Q, dt, quat_idxs=(), flags=3, sel=None):
  xs, Ps, _ = step(m, None, x, P, Q, dt, None, None, quat_idxs=quat_idxs, flags=flags, sel=sel, update=False)
  return xs, Ps


def update(m, kind, x, P, z, R, ea=None, quat_idxs=(), flags=3, sel=None, gate=True):
  return step(m, kind, x, P, None, 0.0, z, R, ea, quat_idxs, flags, sel, predict=False, gate=gate)


def maha(m, kind, x, P, z, R, ea=None, sel=None):
  """Mahalanobis distances [len(sel)] of one observation per filter."""
  sel = range(x.shape[0]) if sel is None else sel
  out = []
  with workdps():
    for b in sel:
      _, zl, Rl, el = _per_obs(z, R, ea, b)
      out.append(float(m.maha(kind, to_mp(x[b]), to_mp(P[b]), zl[0], Rl[0], el[0])))
  return np.array(out)


def augment(m, x, P, sel=None):
  """The clone-window shift of the filters `sel` of a float64 batch; returns float64 (x, P)."""
  sel = range(x.shape[0]) if sel is None else sel
  xs, Ps = [], []
  for b in sel:
    xb, Pb = m.augment(to_mp(x[b]), to_mp(P[b]))
    xs.append(to_np(xb)); Ps.append(to_np(Pb, matrix=True))
  return np.stack(xs), np.stack(Ps)


def rts(m, x_pred, x_filt, P_pred, P_filt, t, quat_idxs=(), norm_quats=False, sel=None):
  """RTS over time-major float64 histories [T, B, ...] for the filters `sel`; returns (xs [T, n, DIM], Ps [T, n, E, E])."""
  sel = range(x_pred.shape[1]) if sel is None else sel
  X, Pl = [], []
  with workdps():
    tm = [mp.mpf(float(v)) for v in t]
    for b in sel:
      args = [[to_mp(a[k, b]) for k in range(a.shape[0])] for a in (x_pred, x_filt, P_pred, P_filt)]
      xs, Ps = m.rts(*args, tm, norm_quats=norm_quats, quat_idxs=quat_idxs)
      X.append(np.stack([to_np(v) for v in xs])); Pl.append(np.stack([to_np(v, matrix=True) for v in Ps]))
  return np.stack(X, 1), np.stack(Pl, 1)


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
