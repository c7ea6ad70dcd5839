"""Synthetic MSCKF filters at the shapes the CTA-per-filter kernels claim to serve (test infrastructure).

An MSCKF state is a main block followed by N clones; a clone is a copy of the first DAUG main states and of the first
EAUG main error states (ekf_sym.py:365-391), so every main block here begins with what is cloned: a position (3/3), a
position and attitude quaternion (7/6, ESKF main block), or the first six states of a plain main block (6/6).  The main
block is ``tests.shapes.synthetic_model`` with its states reordered so that the position comes first.  Clones are static
(identity rows of F, no process noise) and are observed by feature-track kinds: a point ``p = BASE + DIRS[:, :EADIM] ea``
about 20 units ahead, seen from each clone as two normalised image coordinates (ZDIM = 2 x the clones it sees), which
the kernels project on the left null space of He = dh/d(ea).

``MSCKF_SHAPES`` holds one filter per boundary of ``ekf_cta.cuh`` (and the two even shapes below EDIM 32, where feature
kinds still go to the CTA kernel while plain kinds go to the pair kernel); ``__graft_entry__.build()`` compiles them
next to ``tests.shapes.SHAPES`` and tests/test_msckf_shapes_*.py check them against tests/hiprec.py.
"""
import numpy as np

from tests.shapes import EA_KIND, GATED_KIND, EADIM as PLAIN_EADIM, synthetic_model

FEATURE_KIND = 40    # feature-track kinds: ids 40, 41, ...
BASE = (20.0, 0.0, 0.0)
DIRS = ((1.0, 0.0, 0.0), (0.3, 1.0, 0.0), (-0.2, 0.1, 1.0))   # columns of the map ea -> point


def msckf_model(medim, eskf, n_clones, clone, features, zdims=(), maha_kinds=(), ea_kind=None, n_globals=0, seed=0):
  """gen_code arguments of a synthetic MSCKF.

  medim: main error states.  eskf: quaternion main block (DIM_MAIN = medim + 1).  clone: 'position' (3/3), 'pose'
  (7/6, ESKF only: position + quaternion) or 'plain6' (6/6, plain main block only: position + small-angle rotation).
  features: one feature kind per entry (eadim, seen clones (indices), gated).  zdims / maha_kinds / ea_kind / n_globals:
  plain kinds and globals on the main block, as in ``synthetic_model``."""
  import sympy as sp
  from rednose_b200.geometry import quat_matrix_r, quat_rotate
  daug, eaug = {'position': (3, 3), 'pose': (7, 6), 'plain6': (6, 6)}[clone]
  assert eskf or daug == eaug, "a plain main block takes clones with DAUG = EAUG"
  assert clone != 'pose' or eskf, "a pose clone needs an ESKF main block"
  main = synthetic_model(medim, zdims, eskf=eskf, maha_kinds=maha_kinds, ea_kind=ea_kind, n_globals=n_globals, seed=seed)
  dm = main['dim_x']
  # new index -> index in synthetic_model's layout (quaternion first there, position first here)
  px = list(range(4, 7)) + list(range(4)) + list(range(7, dm)) if eskf else list(range(dm))
  pe = list(range(3, 6)) + list(range(3)) + list(range(6, medim)) if eskf else list(range(medim))
  D, E = dm + n_clones * daug, medim + n_clones * eaug
  state_sym = sp.MatrixSymbol('state', D, 1)
  st = sp.Matrix(state_sym)

  def lift(expr, old, new, perm):
    """Substitute old[perm[i]] -> new[i]."""
    return expr.xreplace({old[perm[i], 0]: new[i, 0] for i in range(len(perm))})

  old_x = main['x_sym']
  f_main = sp.Matrix(main['f_sym'])
  f_sym = sp.Matrix(st)                                            # clones are static
  for i in range(dm):
    f_sym[i] = lift(f_main[px[i]], old_x, state_sym, px)

  eskf_params = None
  if eskf:
    (m_inj, m_nom, m_delta), (m_inv, _, m_true), m_Hmod, m_ferr, m_err = main['eskf_params']
    err_sym = sp.MatrixSymbol('state_err', E, 1)
    nom_x, true_x = sp.MatrixSymbol('nom_x', D, 1), sp.MatrixSymbol('true_x', D, 1)
    delta_x = sp.MatrixSymbol('delta_x', E, 1)
    er, nom, tru, dl = sp.Matrix(err_sym), sp.Matrix(nom_x), sp.Matrix(true_x), sp.Matrix(delta_x)
    m_inj, m_inv, m_Hmod, m_ferr = sp.Matrix(m_inj), sp.Matrix(m_inv), sp.Matrix(m_Hmod), sp.Matrix(m_ferr)
    f_err = sp.Matrix(er)
    for i in range(medim):
      f_err[i] = lift(lift(m_ferr[pe[i]], old_x, state_sym, px), m_err, err_sym, pe)
    H_mod = sp.zeros(D, E)
    inject, invert = sp.zeros(D, 1), sp.zeros(E, 1)
    for i in range(dm):
      for j in range(medim):
        H_mod[i, j] = lift(m_Hmod[px[i], pe[j]], old_x, state_sym, px)
      inject[i] = lift(lift(m_inj[px[i]], m_nom, nom_x, px), m_delta, delta_x, pe)
    for i in range(medim):
      invert[i] = lift(lift(m_inv[pe[i]], m_nom, nom_x, px), m_true, true_x, px)
    for c in range(n_clones):
      o, oe = dm + c * daug, medim + c * eaug
      H_mod[o:o + 3, oe:oe + 3] = sp.eye(3)
      inject[o:o + 3, :] = nom[o:o + 3, :] + dl[oe:oe + 3, :]
      invert[oe:oe + 3, :] = tru[o:o + 3, :] - nom[o:o + 3, :]
      if clone == 'pose':
        H_mod[o + 3:o + 7, oe + 3:oe + 6] = sp.Rational(1, 2) * quat_matrix_r(st[o + 3:o + 7, :])[:, 1:]
        dq = sp.Matrix([1] + list(sp.Rational(1, 2) * dl[oe + 3:oe + 6, :]))
        inject[o + 3:o + 7, :] = quat_matrix_r(nom[o + 3:o + 7, :]) * dq
        invert[oe + 3:oe + 6, :] = 2 * (quat_matrix_r(nom[o + 3:o + 7, :]).T * tru[o + 3:o + 7, :])[1:, :]
    eskf_params = [[inject, nom_x, delta_x], [invert, nom_x, true_x], H_mod, f_err, err_sym]

  obs_eqs = [[lift(sp.Matrix(h), old_x, state_sym, px), kind, ea] for h, kind, ea in main['obs_eqs']]
  feature_kinds = []
  maha = list(main['maha_test_kinds'])
  for fi, (ea_dim, seen, gated) in enumerate(features):
    ea = sp.MatrixSymbol('point', ea_dim, 1)
    p = sp.Matrix([sp.Float(BASE[r]) + sum((sp.Float(DIRS[r][k]) * ea[k, 0] for k in range(ea_dim)), sp.Integer(0))
                   for r in range(3)])
    rows = []
    for c in seen:
      o = dm + c * daug
      d = p - st[o:o + 3, :]
      if clone == 'pose':
        pc = quat_rotate(*st[o + 3:o + 7, :]).T * d
      elif clone == 'plain6':
        r = st[o + 3:o + 6, :]
        pc = d - r.cross(d) / 4                                    # a small rotation by -r / 4
      else:
        pc = d
      rows += [pc[1] / pc[0], pc[2] / pc[0]]
    kind = FEATURE_KIND + fi
    obs_eqs.append([sp.Matrix(rows), kind, ea])
    feature_kinds.append(kind)
    if gated:
      maha.append(kind)
  msckf_params = [dm, daug, medim, eaug, n_clones, feature_kinds]
  return dict(f_sym=f_sym, dt_sym=main['dt_sym'], x_sym=state_sym, obs_eqs=obs_eqs, dim_x=D, dim_err=E,
              eskf_params=eskf_params, msckf_params=msckf_params, maha_test_kinds=maha, global_vars=main['global_vars'])


class MsckfShape:
  """One synthetic MSCKF: ``name``, ``symbolic_model()`` and ``generate_code(folder)`` as the shipped filters have."""
  name = None
  spec = {}

  @classmethod
  def symbolic_model(cls):
    return msckf_model(**{k: v for k, v in cls.spec.items() if k != 'dense_q'})

  @classmethod
  def generate_code(cls, generated_dir, name=None):
    from rednose_b200.codegen import gen_code
    gen_code(generated_dir, name or cls.name, **cls.symbolic_model())

  # ---- facts the tests use ----
  @classmethod
  def eskf(cls):
    return bool(cls.spec['eskf'])

  @classmethod
  def medim(cls):
    return cls.spec['medim']

  @classmethod
  def dmain(cls):
    return cls.medim() + 1 if cls.eskf() else cls.medim()

  @classmethod
  def aug(cls):
    """(DAUG, EAUG)"""
    return {'position': (3, 3), 'pose': (7, 6), 'plain6': (6, 6)}[cls.spec['clone']]

  @classmethod
  def n(cls):
    return cls.spec['n_clones']

  @classmethod
  def dim(cls):
    return cls.dmain() + cls.n() * cls.aug()[0]

  @classmethod
  def edim(cls):
    return cls.medim() + cls.n() * cls.aug()[1]

  @classmethod
  def quat_idxs(cls):
    """The main attitude and every clone attitude (at most MAX_QUAT = 16 in all)."""
    if not cls.eskf():
      return []
    q = [3]
    if cls.spec['clone'] == 'pose':
      q += [cls.dmain() + 7 * c + 3 for c in range(cls.n())]
    return q

  @classmethod
  def kinds(cls):
    """kind -> (ZDIM, EADIM, gated, feature)"""
    out = {z: (z, 0, False, False) for z in cls.spec.get('zdims', ())}
    out.update({GATED_KIND + i: (z, 0, True, False) for i, z in enumerate(cls.spec.get('maha_kinds', ()))})
    if cls.spec.get('ea_kind') is not None:
      out[EA_KIND] = (cls.spec['ea_kind'], PLAIN_EADIM, False, False)
    for i, (ea, seen, gated) in enumerate(cls.spec['features']):
      out[FEATURE_KIND + i] = (2 * len(seen), ea, gated, True)
    return out

  @classmethod
  def feature_kinds(cls):
    return [k for k, v in cls.kinds().items() if v[3]]

  @classmethod
  def global_names(cls):
    return [f'g{i}' for i in range(cls.spec.get('n_globals', 0))]

  @classmethod
  def group(cls):
    """Filters per group of the kernel that runs the plain kinds at EDIM <= 32 (pair kernel for even EDIM, single-warp
    kernel for odd), as ``tests.shapes.ShapeFilter.group``."""
    return 16 if cls.edim() % 2 == 0 else 14

  @classmethod
  def rts_kernel(cls):
    """The smoother launch_rts_auto picks (main block only): 'mma' for even EDIM <= 32 with MEDIM >= 8, 'scalar' for
    any other EDIM <= 32, None above (not built)."""
    e = cls.edim()
    if e > 32:
      return None
    return 'mma' if e % 2 == 0 and cls.medim() >= 8 else 'scalar'


def batch(cls, B, seed=0):
  """Well-conditioned float64 inputs: x [B, DIM] (attitudes near the identity, so every clone sees the point ~20 units
  ahead), P [B, E, E] (standard deviations 0.05-0.3, correlated), Q [E, E] (zero on the clone block; dense on the main
  block when ``spec['dense_q']``), dt [B] in 0.01-0.05."""
  rng = np.random.default_rng(seed)
  E, D, dm, ME = cls.edim(), cls.dim(), cls.dmain(), cls.medim()
  x = rng.normal(0, 0.5, (B, D))
  for i in cls.quat_idxs():
    q = np.array([1.0, 0, 0, 0]) + rng.normal(0, 0.1 if i == 3 else 0.03, (B, 4))
    x[:, i:i + 4] = q / np.linalg.norm(q, axis=1, keepdims=True)
  if cls.spec['clone'] == 'plain6':
    for c in range(cls.n()):
      o = dm + 6 * c
      x[:, o + 3:o + 6] *= 0.2
  s = rng.uniform(0.05, 0.3, (B, E))
  L = s[:, :, None] * (np.eye(E)[None] + 0.1 * np.tril(rng.normal(size=(B, E, E)), -1))
  P = L @ np.transpose(L, (0, 2, 1))
  P = 0.5 * (P + np.transpose(P, (0, 2, 1)))
  Q = np.zeros((E, E))
  Q[:ME, :ME] = np.diag(rng.uniform(0.5, 2.0, ME) * 1e-2)
  if cls.spec.get('dense_q'):
    A = rng.normal(size=(ME, ME))
    Q[:ME, :ME] += 1e-3 * (A @ A.T) / ME
  return x, P, Q, rng.uniform(0.01, 0.05, B)


def observe(cls, m, kind, x, seed=1, n_obs=None, outliers=(), noise=1.0):
  """z = h(x) + noise x N(0, R), per-filter diagonal R (standard deviations 0.01-0.03 for a feature kind, 0.05-0.3
  otherwise) and extra arguments (the point: N(0, 1) around BASE); the filters in `outliers` get 1e3 standard deviations
  added.  n_obs: [B, n, ...] arrays."""
  rng = np.random.default_rng(seed * 131 + kind)
  Z, EA, _, feat = cls.kinds()[kind]
  B, n = x.shape[0], n_obs or 1
  ea = rng.normal(0, 1.0, (B, n, EA)) if EA else None
  sd = rng.uniform(0.01, 0.03, (B, n, Z)) if feat else rng.uniform(0.05, 0.3, (B, n, Z))
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


def augment_np(cls, x, P):
  """The clone-window shift of ekf_sym.py:365-391 as its selection-matrix products, in float64 numpy."""
  (d3, d4), d1, d2, n = cls.aug(), cls.dmain(), cls.medim(), cls.edim()
  xr = x.copy()
  xr[:, d1:-d3] = x[:, d1 + d3:]
  xr[:, -d3:] = x[:, :d3]
  to_mult = np.zeros((n, n - d4))
  to_mult[:-d4, :] = np.eye(n - d4)
  to_mult[-d4:, :d4] = np.eye(d4)
  Pr = np.stack([to_mult @ np.delete(np.delete(Pb, np.s_[d2:d2 + d4], axis=1), np.s_[d2:d2 + d4], axis=0) @ to_mult.T for Pb in P])
  return xr, Pr


def _msckf(name, **spec):
  spec.setdefault('seed', 0)
  return type(f'Msckf_{name}', (MsckfShape,), dict(name=f'msckf_{name}', spec=spec, __module__=__name__))


# one filter per boundary of the CTA-per-filter kernels (ekf_cta.cuh)
MSCKF_SHAPES = [
  # EDIM 18: a feature kind on an even EDIM <= 32 (one-warp CTA); the plain kind goes to the pair kernel
  _msckf('e18', medim=6, eskf=True, n_clones=4, clone='position', features=[(3, range(4), True)], zdims=(3,)),
  # EDIM 27: a feature kind next to the single-warp kernel, EADIM 2
  _msckf('e27', medim=9, eskf=False, n_clones=3, clone='plain6', features=[(2, range(3), True)], zdims=(3,)),
  # EDIM 33: NC = 2, E not a multiple of 8, one column in warp 1
  _msckf('e33', medim=9, eskf=True, n_clones=4, clone='pose', features=[(3, range(4), True)], zdims=(3,)),
  # EDIM 64: the innovation thread owns column 63; dense Q, globals, a plain kind with extra arguments
  _msckf('e64', medim=22, eskf=True, n_clones=7, clone='pose', features=[(3, range(7), True), (1, range(5, 7), False)],
         zdims=(3,), ea_kind=2, n_globals=2, dense_q=True),
  # EDIM 68: FROW_MASK bit 31; a plain kind with ZDIM 31 (Y + 1 = 32)
  _msckf('e68', medim=32, eskf=True, n_clones=6, clone='pose', features=[(3, range(6), True)], zdims=(31,)),
  # EDIM 73: a point seen from 17 clones, ZDIM 34 / Y 31; only the main attitude is a quaternion
  _msckf('e73', medim=22, eskf=True, n_clones=17, clone='position', features=[(3, range(17), True)], zdims=(3,)),
  # EDIM 28: one clone, which the augment overwrites; a single view with EADIM 1
  _msckf('e28', medim=22, eskf=True, n_clones=1, clone='pose', features=[(1, range(1), True)], zdims=(3,)),
  # EDIM 166: 6 warps (register cap of __launch_bounds__(192, 4)); the largest EDIM of this layout the augment kernel fits
  _msckf('e166', medim=16, eskf=False, n_clones=25, clone='plain6', features=[(3, range(15, 25), True)], zdims=(3,)),
]
BY_NAME = {c.name: c for c in MSCKF_SHAPES}


def ensure_all(folder=None, jobs=None):
  """Generate and compile every MSCKF shape library (concurrently); returns the folder."""
  import os
  from concurrent.futures import ThreadPoolExecutor
  from rednose_b200.build import GENERATED_DIR
  from rednose_b200.filters import ensure_generated
  folder = folder or GENERATED_DIR
  with ThreadPoolExecutor(max_workers=jobs or min(len(MSCKF_SHAPES), os.cpu_count() or 1)) as ex:
    for f in [ex.submit(ensure_generated, cls, folder) for cls in MSCKF_SHAPES]:
      f.result()
  return folder
