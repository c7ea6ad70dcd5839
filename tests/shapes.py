"""Synthetic filters at the shapes the step, query and smoother kernels claim to serve (test infrastructure).

``launch_step`` routes a filter by its error-state size EDIM (thread kernel for EDIM <= 6, two filters per warp for even
EDIM 8-32, one filter per warp for odd EDIM 7-31, CTA kernel above 32) and ``launch_rts_auto`` picks the tensor-core
smoother for even EDIM with a main block of at least 8.  ``SHAPES`` holds one filter per side of every boundary;
``__graft_entry__.build()`` generates and compiles them next to the shipped filters, and tests/test_shapes_*.py check
them against the 40-digit reference of tests/hiprec.py.

Every model comes from ``synthetic_model``: f is nonlinear in the state and depends on dt, with deterministic
pseudo-random coefficients, and its F has identity rows, rows with a non-unit diagonal, sparse coupled rows and dense
rows; the last row is always dense, so at EDIM 32 row 31 (the top ``FROW_MASK`` bit) differs from the identity.
"""
import numpy as np

GATED_KIND = 20   # the Mahalanobis-gated kind (ZDIM 3, or EDIM when smaller)
EA_KIND = 30      # the kind with extra arguments (ZDIM 2, EADIM 2)
EADIM = 2


def synthetic_model(edim, zdims, eskf=False, maha_kinds=(), ea_kind=None, n_globals=0, seed=0):
  """gen_code arguments of a synthetic filter with error-state size `edim`.

  zdims: one plain kind per entry, kind id = its ZDIM.  maha_kinds: ZDIMs of Mahalanobis-gated kinds (ids GATED_KIND,
  GATED_KIND + 1, ...).  ea_kind: ZDIM of a kind with EADIM extra arguments (id EA_KIND), or None.  n_globals: global
  variables g0, g1, ... (used in f and in the first plain kind).  eskf: the first four states are a quaternion with a
  three-dimensional error (DIM = EDIM + 1), injected multiplicatively; otherwise a plain EKF (DIM = EDIM).
  """
  import sympy as sp
  from rednose_b200.geometry import quat_matrix_r, quat_rotate
  rng = np.random.default_rng(1000 + 97 * edim + seed)
  coef = lambda lo=-1.0, hi=1.0: sp.Float(float(np.round(rng.uniform(lo, hi), 6)))   # 6-digit literals
  nq = 4 if eskf else 0
  dim = edim + 1 if eskf else edim
  nv = dim - nq                      # additive states after the quaternion
  assert nv >= 1 and (not eskf or nv >= 3)
  state_sym = sp.MatrixSymbol('state', dim, 1)
  st = sp.Matrix(state_sym)
  dt = sp.Symbol('dt')
  gvars = [sp.Symbol(f'g{i}') for i in range(n_globals)]
  q = st[:nq, :] if eskf else None

  dense = {nv - 1, nv // 2}
  fc = [[coef() for _ in range(nv)] if i in dense else [coef(0.2, 1.5), coef(), coef()] for i in range(nv)]   # drawn once

  def f_v(s):
    """The additive part of f on a full state vector s (sympy Matrix)."""
    v = s[nq:, :]
    Rq = quat_rotate(*s[:nq, :]) if eskf else None
    out = []
    for i in range(nv):
      j, k, c = (i + 1) % nv, (i + 2) % nv, fc[i]
      if i in dense:                                   # dense row: every additive state, nonlinear
        out.append(v[i] + dt * sum((c[l] * sp.sin(v[l]) for l in range(nv)), sp.Integer(0)) * sp.Rational(1, 4))
      elif i % 3 == 0:                                 # identity row
        out.append(v[i])
      elif i % 3 == 1:                                 # non-unit diagonal plus one nonlinear coupling
        g = gvars[i % len(gvars)] if gvars else 1
        out.append(v[i] * (1 - c[0] * dt) + dt * g * c[1] * sp.sin(v[j]))
      else:                                            # sparse nonlinear coupling, through the attitude with a quaternion
        term = c[1] * v[j] * v[k] / 2
        if eskf:
          term += c[2] * (Rq * sp.Matrix(v[:3]))[i % 3]
        out.append(v[i] + dt * term)
    return sp.Matrix(out)

  f_sym = sp.Matrix(list(q) + list(f_v(st))) if eskf else f_v(st)

  eskf_params = None
  if eskf:
    err_sym = sp.MatrixSymbol('state_err', edim, 1)
    er = sp.Matrix(err_sym)
    nom_x = sp.MatrixSymbol('nom_x', dim, 1)
    true_x = sp.MatrixSymbol('true_x', dim, 1)
    delta_x = sp.MatrixSymbol('delta_x', edim, 1)

    def inject(nom, dl):
      dq = sp.Matrix([1] + list(sp.Rational(1, 2) * dl[:3, :]))
      return sp.Matrix(list(quat_matrix_r(nom[:4, :]) * dq) + list(nom[4:, :] + dl[3:, :]))

    nom, tru = sp.Matrix(nom_x), sp.Matrix(true_x)
    inj = inject(nom, sp.Matrix(delta_x))
    inv = sp.Matrix(list(2 * (quat_matrix_r(nom[:4, :]).T * tru[:4, :])[1:, :]) + list(tru[4:, :] - nom[4:, :]))
    # error dynamics: exactly inv_err(f(x), f(x [+] e)) for a unit quaternion (f keeps the attitude)
    f_err_sym = sp.Matrix(list(er[:3, :]) + list(f_v(inject(st, er)) - f_v(st)))
    H_mod = sp.zeros(dim, edim)
    H_mod[:4, :3] = sp.Rational(1, 2) * quat_matrix_r(q)[:, 1:]
    H_mod[4:, 3:] = sp.eye(nv)
    eskf_params = [[inj, nom_x, delta_x], [inv, nom_x, true_x], H_mod, f_err_sym, err_sym]

  def obs(z, salt):
    r = np.random.default_rng(7 * z + salt + seed)
    idx = r.permutation(dim)
    h = []
    for a in range(z):
      p, s_, t = int(idx[a % dim]), int(r.integers(dim)), int(r.integers(dim))
      h.append(st[p] + coef(0.1, 0.5) * sp.sin(st[s_]) * st[t])
    if eskf and z >= 3:                                 # an attitude-dependent block
      rot = quat_rotate(*q).T * sp.Matrix(st[nq:nq + 3, :])
      for a in range(3):
        h[a] += rot[a]
    return h

  obs_eqs = []
  for z in zdims:
    h = obs(z, 1)
    if gvars and z == zdims[0]:
      h[0] = h[0] + gvars[-1] * st[dim - 1] ** 2 / 2
    obs_eqs.append([sp.Matrix(h), z, None])
  for i, z in enumerate(maha_kinds):
    obs_eqs.append([sp.Matrix(obs(z, 2)), GATED_KIND + i, None])
  if ea_kind is not None:
    anchor = sp.MatrixSymbol('anchor', EADIM, 1)
    h = obs(ea_kind, 3)
    for a in range(ea_kind):
      h[a] = anchor[a % EADIM, 0] + anchor[(a + 1) % EADIM, 0] * h[a]
    obs_eqs.append([sp.Matrix(h), EA_KIND, anchor])
  return dict(f_sym=f_sym, dt_sym=dt, x_sym=state_sym, obs_eqs=obs_eqs, dim_x=dim, dim_err=edim, eskf_params=eskf_params,
              maha_test_kinds=[GATED_KIND + i for i in range(len(maha_kinds))], global_vars=gvars or None)


class ShapeFilter:
  """One synthetic filter: ``name``, ``symbolic_model()`` and ``generate_code(folder)`` as the shipped filters have."""
  name = None
  edim = None
  spec = {}

  @classmethod
  def symbolic_model(cls):
    return synthetic_model(cls.edim, **cls.spec)

  @classmethod
  def generate_code(cls, generated_dir, name=None):
    from rednose_b200.codegen import gen_code
    gen_code(generated_dir, name or cls.name, **cls.symbolic_model())

  # ---- facts the tests use ----
  @classmethod
  def eskf(cls):
    return bool(cls.spec.get('eskf'))

  @classmethod
  def dim(cls):
    return cls.edim + 1 if cls.eskf() else cls.edim

  @classmethod
  def quat_idxs(cls):
    return [0] if cls.eskf() else []

  @classmethod
  def kinds(cls):
    """kind -> (ZDIM, EADIM, gated)"""
    out = {z: (z, 0, False) for z in cls.spec['zdims']}
    out.update({GATED_KIND + i: (z, 0, True) for i, z in enumerate(cls.spec.get('maha_kinds', ()))})
    if cls.spec.get('ea_kind') is not None:
      out[EA_KIND] = (cls.spec['ea_kind'], EADIM, False)
    return out

  @classmethod
  def global_names(cls):
    return [f'g{i}' for i in range(cls.spec.get('n_globals', 0))]

  @classmethod
  def step_kernel(cls):
    e = cls.edim
    return 'thread' if e <= 6 else ('pair' if e % 2 == 0 else 'warp')

  @classmethod
  def group(cls):
    """Filters per kernel group of the kernel that serves this shape (thread block, pair-kernel or warp-kernel group)."""
    return {'thread': 128, 'pair': 16, 'warp': 14}[cls.step_kernel()]

  @classmethod
  def rts_kernel(cls):
    return 'mma' if cls.edim % 2 == 0 and 8 <= cls.edim <= 32 else 'scalar'


def batch(cls, B, seed=0):
  """Well-conditioned float64 inputs: x [B, DIM] (unit quaternion for an ESKF), P [B, E, E] (standard deviations
  0.1-0.5, correlated), Q [E, E] (diagonal for an ESKF, dense otherwise), dt [B] in 0.01-0.05."""
  rng = np.random.default_rng(seed)
  E, D = cls.edim, cls.dim()
  x = rng.normal(0, 0.5, (B, D))
  if cls.eskf():
    q = rng.normal(size=(B, 4))
    x[:, :4] = q / np.linalg.norm(q, axis=1, keepdims=True)
  s = rng.uniform(0.1, 0.5, (B, E))
  L = s[:, :, None] * (np.eye(E)[None] + 0.1 * np.tril(rng.normal(size=(B, E, E)), -1))
  P = L @ np.transpose(L, (0, 2, 1))
  P = 0.5 * (P + np.transpose(P, (0, 2, 1)))
  if cls.eskf():
    Q = np.diag(rng.uniform(0.5, 2.0, E) * 1e-2)
  else:
    A = rng.normal(size=(E, E))
    Q = 1e-3 * (A @ A.T) / E + np.diag(rng.uniform(0.5, 2.0, E) * 1e-2)
  return x, P, Q, rng.uniform(0.01, 0.05, B)


def observe(cls, m, kind, x, seed=1, n_obs=None, outliers=(), noise=1.0):
  """z = h(x) + noise x N(0, R), per-filter diagonal R (standard deviations 0.05-0.3) and extra arguments for a kind;
  the filters in `outliers` get 1e3 standard deviations added (Mahalanobis distance ~1e6).  n_obs: [B, n, ...] arrays."""
  rng = np.random.default_rng(seed * 131 + kind)
  Z, EA, _ = cls.kinds()[kind]
  B = x.shape[0]
  n = n_obs or 1
  ea = rng.normal(0, 1.0, (B, n, EA)) if EA else None
  sd = rng.uniform(0.05, 0.3, (B, n, Z))
  z = np.empty((B, n, Z))
  for b in range(B):
    for o in range(n):
      z[b, o] = m.np_leaf(('h', kind), x[b], *([ea[b, o]] if EA else []))
  z += noise * sd * rng.normal(size=(B, n, Z))
  z[list(outliers)] += 1e3 * sd[list(outliers)]
  R = np.einsum('bni,ij->bnij', sd ** 2, np.eye(Z))
  if n_obs is None:
    return z[:, 0], R[:, 0], (ea[:, 0] if EA else None)
  return z, R, ea


def sample(cls, B):
  """Filters a check compares against the 40-digit reference: the first and the last, and both sides of every boundary
  of the serving kernel's groups."""
  G = cls.group()
  s = {0, B - 1}
  for g in range(G, B, G):
    s |= {g - 1, g}
  return sorted(s)


def _shape(edim, **spec):
  spec.setdefault('seed', 0)
  return type(f'Shape{edim}', (ShapeFilter,), dict(name=f'shape_e{edim}', edim=edim, spec=spec, __module__=__name__))


# one filter per dispatch boundary: thread (1, 4, 6), one filter per warp (odd 7, 31), pair (8, 16, 24, 28, 32)
SHAPES = [
  _shape(1, zdims=(1,), maha_kinds=(1,)),
  _shape(4, zdims=(1, 3, 4), maha_kinds=(3,), ea_kind=2, n_globals=1),
  _shape(6, zdims=(1, 3, 6), eskf=True, maha_kinds=(3,)),                          # even EDIM, MEDIM < 8: scalar RTS
  _shape(7, zdims=(1, 3, 7), maha_kinds=(3,), ea_kind=2, n_globals=2),
  _shape(8, zdims=(1, 3, 8), maha_kinds=(3,), ea_kind=2),                          # smallest pair / RTS-MMA shape
  _shape(16, zdims=(1, 3, 16), eskf=True, ea_kind=2),                              # ZDIM 16 on the pair kernel
  _shape(24, zdims=(1, 3, 8), eskf=True, maha_kinds=(3,), ea_kind=2, n_globals=2),  # FROW_MASK bits 22-23, NP 24
  _shape(28, zdims=(1, 3, 8), maha_kinds=(3,)),                                    # NP 32 smoother
  _shape(31, zdims=(1, 3, 8), eskf=True, maha_kinds=(3,), ea_kind=2),
  _shape(32, zdims=(1, 3, 8), maha_kinds=(3,), ea_kind=2, n_globals=1),            # every pair lane active
]
BY_NAME = {c.name: c for c in SHAPES}


def ensure_all(folder=None, jobs=None):
  """Generate and compile every shape library (concurrently: nvcc is single-threaded); returns the folder."""
  import os
  from concurrent.futures import ThreadPoolExecutor
  from rednose_b200.build import GENERATED_DIR
  from rednose_b200.filters import ensure_generated
  folder = folder or GENERATED_DIR
  with ThreadPoolExecutor(max_workers=jobs or min(len(SHAPES), os.cpu_count() or 1)) as ex:
    for f in [ex.submit(ensure_generated, cls, folder) for cls in SHAPES]:
      f.result()
  return folder
