"""Long MSCKF streams through the smoothers: main-block prediction histories and the feature-kind stream (extra arguments
and the fused clone-window shift) in TiledSmoother and CheckpointedSmoother.

Above EDIM 32 a history may keep only the main block of each P_{k+1|k} (BatchedEKF.new_history(T, main_pred=True)) plus
the full prediction of the newest step: everything the smoother reads.  Each case records the same stream of T = 8
steps of B = 5 filters (plain and feature kinds at irregular times, the clone window shifted after step AUG) into a full
and a main-block history from the same start, and checks bit for bit:

- recording: x_pred, x_filt and P_filt equal; each main-block row is the main block of the full row, and P_pred_last
  is the newest full row;
- smoothing: the main-block history gives the full history's xs and Ps in a new buffer, with out=, in place, as chained
  segments, and for histories of one and two steps;
- CheckpointedSmoother (segment 1, a segment that does not divide T, more than one tile) and TiledSmoother (uneven tiles,
  passes=2), in both layouts, against whole-history smoothing of the same stream.

msckf_e36 (tests/msckf_long_shapes.py) has an even EDIM with an odd main block, whose slab rows the tensor-core smoother
reads without 16-byte pairs.  msckf_e33 and msckf_e36 are also checked against the 40-digit main-block RTS of
tests/hiprec.py.  Filters at EDIM <= 32 (msckf_e18,
e27, e28) run the same stream through both smoothers in the full layout.  Observations come from the libraries' own
h leaf functions, so no 40-digit model is built except those two."""
import numpy as np
import pytest
import torch

from tests import hiprec, msckf_long_shapes, msckf_shapes
from tests.util import cov_err, msckf_batch, state_err

pytestmark = pytest.mark.gpu

T, AUG, B = 8, 3, 5
GV = [1.0, 1.25]
LARGE = ["msckf_e33", "msckf_e36", "msckf_e64", "msckf_e68", "msckf_e73", "msckf_e166", "msckf"]
SMALL = ["msckf_e18", "msckf_e27", "msckf_e28"]
SLABS = ("x_pred", "x_filt", "P_filt")


def _setup(name):
  """(folder, x0, P0, Q, quaternion indices, global vars, plain kind, feature kind, ea sampler, medim)."""
  from rednose_b200.filters import ensure_generated
  if name == "msckf":
    from rednose_b200.filters.msckf import MsckfKalman
    x, P, Q, point = msckf_batch(B, seed=500)
    from tests.test_msckf_large_smoothing_gpu import _Msckf
    return ensure_generated(MsckfKalman), x, P, Q, _Msckf.quat_idxs(), {}, 12, 17, (lambda rng: point), 22
  cls = {**msckf_shapes.BY_NAME, **msckf_long_shapes.BY_NAME}[name]
  x, P, Q, _ = msckf_shapes.batch(cls, B, seed=500)
  plain = [k for k, v in cls.kinds().items() if not v[3]][0]
  feat = cls.feature_kinds()[0]
  EA = cls.kinds()[feat][1]
  gv = {g: GV[i] for i, g in enumerate(cls.global_names())}
  return ensure_generated(cls), x, P, Q, cls.quat_idxs(), gv, plain, feat, (lambda rng: rng.normal(0, 1.0, (B, EA))), cls.medim()


@pytest.fixture(scope="module", params=LARGE + SMALL)
def rec(request):
  from rednose_b200.batched import BatchedEKF
  name = request.param
  folder, x, P, Q, q, gv, plain, feat, ea_of, ME = _setup(name)
  zdim = _zdims(folder, name)
  rng = np.random.default_rng(501)
  kinds = [plain, feat, feat, feat, plain, feat, plain, feat]
  t = 0.1 + np.cumsum(rng.uniform(0.005, 0.04, T))
  large = name in LARGE
  e = BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q, global_vars=gv)   # sets the library's globals for every engine
  em = BatchedEKF(folder, name, Q, x, P, quaternion_idxs=q) if large else None
  h = e.new_history(T)
  hm = em.new_history(T, main_pred=True) if large else None
  obs = []
  for k in range(T):
    kind = kinds[k]
    ea = ea_of(rng) if kind == feat else None
    xs = e.state()
    Z = zdim[kind]
    z = np.stack([_h(e, kind, xs[b], None if ea is None else ea[b], Z) for b in range(B)])
    sd = (5.0 if (name == "msckf" and kind == 12) else 1e-2)
    z = z + sd * rng.normal(size=z.shape)
    R = np.tile(np.eye(Z) * sd ** 2, (B, 1, 1))
    obs.append((float(t[k]), kind, z, R, ea, k == AUG))
    e.step_recorded(h, kind, float(t[k]), z, R, ea, augment=(k == AUG))
    if large:
      em.step_recorded(hm, kind, float(t[k]), z, R, ea, augment=(k == AUG))
  return dict(name=name, folder=folder, e=e, em=em, h=h, hm=hm, x0=x, P0=P, Q=Q, q=q, obs=obs, ME=ME, t=t,
              norms=[False, True] if q else [False])


def _zdims(folder, name):
  import re
  src = open(f"{folder}/{name}.cu", encoding="utf-8").read()
  return {int(k): int(z) for k, z in re.findall(r"struct \w+_kind_(\d+) \{\s*static constexpr int KIND = \d+, ZDIM = (\d+)", src)}


def _h(e, kind, x, ea, Z):
  ffi, lib = e._ffi, e._lib
  xb = np.ascontiguousarray(x, dtype=np.float64)
  eb = np.ascontiguousarray(ea if ea is not None else np.zeros(1), dtype=np.float64)
  out = np.zeros(Z)
  getattr(lib, f"{e.name}_h_{kind}")(ffi.cast("double *", xb.ctypes.data), ffi.cast("double *", eb.ctypes.data),
                                     ffi.cast("double *", out.ctypes.data))
  return out


def _kw(r, norm):
  return dict(norm_quats=norm, quaternion_idxs=tuple(r["q"]) or (0,))


def _obs_fn(r):
  def fn(k, lo, hi):
    t, kind, z, R, ea, aug = r["obs"][k]
    return t, kind, z[lo:hi].copy(), R[lo:hi], (None if ea is None else ea[lo:hi]), aug
  return fn


def _large(r):
  if r["hm"] is None:
    pytest.skip("main-block prediction histories exist only above EDIM 32")


def _copy(r, n, main):
  """A new history holding the first n rows of the recorded one (main: of the main-block history, with the full
  prediction of row n - 1 as its newest)."""
  e, src = (r["em"], r["hm"]) if main else (r["e"], r["h"])
  c = e.new_history(n, main_pred=main)
  for a in SLABS + ("P_pred",):
    getattr(c, a).copy_(getattr(src, a)[:n])
  if main:
    c.P_pred_last.copy_(r["h"].P_pred[n - 1])
  c.t_host[:] = src.t_host[:n]
  c.n = n
  return c


def test_main_block_recording_matches_the_full_layout(rec):
  r = rec
  _large(r)
  h, hm, ME = r["h"], r["hm"], r["ME"]
  assert tuple(hm.P_pred.shape) == (T, B, ME, ME) and tuple(hm.P_pred_last.shape) == h.P_pred.shape[1:]
  for a in SLABS:
    assert torch.equal(getattr(hm, a), getattr(h, a)), a
  assert torch.equal(hm.P_pred, h.P_pred[:, :, :ME, :ME])
  assert torch.equal(hm.P_pred_last, h.P_pred[T - 1])
  assert torch.equal(r["em"].x, r["e"].x) and torch.equal(r["em"].P, r["e"].P)
  assert hm.bytes() == h.bytes() - 8 * T * B * (h.P_pred.shape[-1] ** 2 - ME * ME) + 8 * B * h.P_pred.shape[-1] ** 2


def test_main_block_smoothing_matches_the_full_history(rec):
  """New buffers, out= (one row longer, NaN), in place, and histories of one and two steps."""
  r = rec
  _large(r)
  e, em = r["e"], r["em"]
  for norm in r["norms"]:
    xw, Pw = e.rts_smooth(r["h"], **_kw(r, norm))
    xs, Ps = em.rts_smooth(r["hm"], **_kw(r, norm))
    assert torch.equal(xs, xw) and torch.equal(Ps, Pw), norm
    out = (torch.full((T + 1,) + xw.shape[1:], float("nan"), dtype=torch.float64, device=xw.device),
           torch.full((T + 1,) + Pw.shape[1:], float("nan"), dtype=torch.float64, device=xw.device))
    xo, Po = em.rts_smooth(r["hm"], out=out, **_kw(r, norm))
    assert torch.equal(xo, xw) and torch.equal(Po, Pw) and torch.isnan(out[1][T]).all()
    c = _copy(r, T, True)
    xi, Pi = em.rts_smooth(c, in_place=True, **_kw(r, norm))
    assert xi.data_ptr() == c.x_filt.data_ptr() and torch.equal(xi, xw) and torch.equal(Pi, Pw)
    for n in (1, 2):
      xf, Pf = e.rts_smooth(_copy(r, n, False), **_kw(r, norm))
      xm, Pm = em.rts_smooth(_copy(r, n, True), **_kw(r, norm))
      assert torch.equal(xm, xf) and torch.equal(Pm, Pf), (norm, n)


def _chained(e, src, S, kw, main, full):
  """Smooth src as segments of S steps, last first (tests/test_rts_segments_gpu.py's _chained for either layout)."""
  nan = float("nan")
  xs, Ps = torch.full_like(src.x_filt, nan), torch.full_like(src.P_filt, nan)
  seg = e.new_history(S + 1, main_pred=main)
  term = None
  for k0 in reversed(range(0, src.n, S)):
    n = min(S + 1, src.n - k0)
    for a in SLABS + ("P_pred",):
      getattr(seg, a)[:n].copy_(getattr(src, a)[k0:k0 + n])
    if main:
      seg.P_pred_last.copy_(full.P_pred[k0 + n - 1])
    seg.t_host[:n] = src.t_host[k0:k0 + n]
    seg.n = n
    out = (torch.full_like(seg.x_filt, nan), torch.full_like(seg.P_filt, nan))
    e.rts_smooth(seg, out=out, terminal=term, k0=k0, **kw)
    m = n - (term is not None)
    xs[k0:k0 + m], Ps[k0:k0 + m] = out[0][:m], out[1][:m]
    term = (out[0][0].clone(), out[1][0].clone())
  return xs, Ps


def test_main_block_chained_segments_equal_the_whole_history(rec):
  r = rec
  _large(r)
  for norm in r["norms"]:
    xw, Pw = r["e"].rts_smooth(r["h"], **_kw(r, norm))
    for S in (1, 3, T):
      xs, Ps = _chained(r["em"], r["hm"], S, _kw(r, norm), True, r["h"])
      assert torch.equal(xs, xw) and torch.equal(Ps, Pw), (norm, S)


def _collect_checkpointed(r, main, segment, tile):
  from rednose_b200.smoothing import CheckpointedSmoother
  xs = torch.full_like(r["h"].x_filt, float("nan"))
  Ps = torch.full_like(r["h"].P_filt, float("nan"))

  def sink(lo, hi, k0, x, P):
    xs[k0:k0 + x.shape[0], lo:hi] = x
    Ps[k0:k0 + x.shape[0], lo:hi] = P

  dim_x, dim_err = r["x0"].shape[1], r["P0"].shape[1]
  sm = CheckpointedSmoother(r["folder"], r["name"], r["Q"], dim_x, dim_err, quaternion_idxs=r["q"], segment=segment, tile=tile,
                            main_pred=main)
  tiles = sm.run(r["x0"], r["P0"], T, _obs_fn(r), sink, norm_quats=bool(r["q"]), t0=r["obs"][0][0])
  return tiles, xs, Ps


@pytest.mark.parametrize("segment,tile", [(1, None), (3, None), (3, 2)])
def test_checkpointed_smoother_runs_the_msckf_stream(rec, segment, tile):
  """Segment 1, a segment that does not divide T, and tiles of 2, 2 and 1 filters: in both layouts (the full one only at
  EDIM <= 32), bit for bit the whole-history pass of the same stream."""
  r = rec
  xw, Pw = r["e"].rts_smooth(r["h"], **_kw(r, bool(r["q"])))
  for main in ([False, True] if r["hm"] is not None else [False]):
    tiles, xs, Ps = _collect_checkpointed(r, main, segment, tile)
    assert tiles == (1 if tile is None else 3)
    assert torch.equal(xs, xw) and torch.equal(Ps, Pw), (main, segment, tile)


def _collect_tiled(r, main, tile, passes):
  from rednose_b200.smoothing import TiledSmoother
  xs = torch.full_like(r["h"].x_filt, float("nan"))
  Ps = torch.full_like(r["h"].P_filt, float("nan"))

  def sink(lo, hi, x, P):
    xs[:, lo:hi] = x
    Ps[:, lo:hi] = P

  dim_x, dim_err = r["x0"].shape[1], r["P0"].shape[1]
  sm = TiledSmoother(r["folder"], r["name"], r["Q"], dim_x, dim_err, quaternion_idxs=r["q"], tile=tile, main_pred=main)
  tiles = sm.run(r["x0"], r["P0"], T, _obs_fn(r), sink, norm_quats=bool(r["q"]), t0=r["obs"][0][0], passes=passes)
  return tiles, xs, Ps


def _whole_passes(r, passes):
  """`passes` whole forward + backward passes of the stream, each further one started from x_{0|N}, P_{0|N}."""
  from rednose_b200.batched import BatchedEKF
  kw = _kw(r, bool(r["q"]))
  x0, P0 = r["x0"], r["P0"]
  for _ in range(passes):
    e = BatchedEKF(r["folder"], r["name"], r["Q"], x0, P0, quaternion_idxs=r["q"])
    h = e.new_history(T)
    for k in range(T):
      t, kind, z, R, ea, aug = r["obs"][k]
      e.step_recorded(h, kind, t, z.copy(), R, ea, augment=aug)
    xs, Ps = e.rts_smooth(h, **kw)
    x0, P0 = xs[0].clone(), Ps[0].clone()
  return xs, Ps


def test_tiled_smoother_runs_the_msckf_stream(rec):
  """Tiles of 2, 2 and 1 filters equal the untiled pass; passes=2 equals two whole passes; both layouts."""
  r = rec
  xw, Pw = _whole_passes(r, 1)
  x2, P2 = _whole_passes(r, 2)
  for main in ([False, True] if r["hm"] is not None else [False]):
    tiles, xs, Ps = _collect_tiled(r, main, 2, 1)
    assert tiles == 3 and torch.equal(xs, xw) and torch.equal(Ps, Pw), main
    tiles, xs, Ps = _collect_tiled(r, main, None, 2)
    assert tiles == 1 and torch.equal(xs, x2) and torch.equal(Ps, P2), main


def test_main_block_smoothing_matches_the_40_digit_reference(rec):
  """msckf_e33 and msckf_e36: the main-block history's smoothed rows against tests/hiprec.py's main-block RTS over the
  recorded full slabs, state per component and covariance in correlation units, at 1e-9."""
  r = rec
  if r["name"] not in ("msckf_e33", "msckf_e36"):
    pytest.skip("two shapes")
  cls = {**msckf_shapes.BY_NAME, **msckf_long_shapes.BY_NAME}[r["name"]]
  m = hiprec.model_of(cls)
  m.gv = GV[:len(m.gvars)]
  slabs = [getattr(r["h"], a).cpu().numpy() for a in ("x_pred", "x_filt", "P_pred", "P_filt")]
  sel = [0, B - 1]
  for norm in r["norms"]:
    xs, Ps = (a.cpu().numpy() for a in r["em"].rts_smooth(r["hm"], **_kw(r, norm)))
    xr, Pr = hiprec.rts(m, *slabs, r["h"].t_host, quat_idxs=r["q"], norm_quats=norm, sel=sel)
    ex, eP = state_err(xs[:, sel], xr), cov_err(Ps[:, sel], Pr)
    assert ex < 1e-9 and eP < 1e-9, (norm, ex, eP)
