"""The packed resident covariance of the two-filters-per-warp kernel on the GPU.

P is defined by its lower triangle, and every P the kernel writes is the exact mirror of it, in either layout.  So the
packed engine, the full-layout ABI and the stateless host entry point give bit-identical x, P and y (torch.equal), and
nothing depends on the upper triangle of the input."""
import numpy as np
import pytest
import torch

from tests.util import LIVE_KINDS, Oracle, cov_err, live_batch, live_obs, state_err

pytestmark = pytest.mark.gpu


def _engines(gen_dir, x, P, Qm, **kw):
  """(packed engine, full-layout engine): the second drives the unflagged ABI on a full [B, EDIM, EDIM] buffer."""
  from rednose_b200.batched import BatchedEKF
  a = BatchedEKF(gen_dir, "live", Qm, x, P, quaternion_idxs=[3], **kw)
  b = BatchedEKF(gen_dir, "live", Qm, x, P, quaternion_idxs=[3], **kw)
  assert a._Pk is not None and a._packed_doubles == 264
  b._Pf, b._Pk, b._full_owns = b.P.clone(), None, True
  return a, b


def _same(a, b, ya=None, yb=None):
  assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)
  if ya is not None:
    assert torch.equal(ya, yb)
  assert torch.equal(a.P, a.P.transpose(1, 2))


@pytest.mark.parametrize("kind", sorted(LIVE_KINDS))
def test_packed_equals_full_abi_and_host_step(gen_dir, oracle_dir, kind):
  o = Oracle(oracle_dir, "live")
  B = 1031                                          # odd: the last pair of the last group is half empty
  x, P, Qm = live_batch(B, seed=100 + kind)
  z, R = live_obs(o, kind, x)
  a, b = _engines(gen_dir, x, P, Qm)
  dt = torch.as_tensor(np.random.default_rng(kind).uniform(0.005, 0.02, B)).cuda()
  ya = a.step(kind, dt, z, R)
  yb = b.step(kind, dt, z, R)
  _same(a, b, ya, yb)
  # the stateless host entry point: same kernel on the full layout, host buffers
  hx, hP, hz = x.copy(), P.copy(), z.copy()
  ffi, lib = a._ffi, a._lib
  pp = lambda t: ffi.cast("double *", t.ctypes.data)
  Rc, dtc = np.ascontiguousarray(R), dt.cpu().numpy()
  getattr(lib, f"live_host_step_{kind}")(pp(hx), pp(hP), pp(Qm), pp(dtc), 0.0, pp(hz), pp(Rc), ffi.NULL, 1, B, ffi.new("int[]", [3]), 1, a.flags)
  assert lib.live_cuda_status() == 0
  assert np.array_equal(hx, a.state()) and np.array_equal(hP, a.covs()) and np.array_equal(hz, ya.cpu().numpy()[:, 0])


def test_two_observations_predict_update_and_history(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  B = 777
  x, P, Qm = live_batch(B, seed=7)
  a, b = _engines(gen_dir, x, P, Qm)
  z1, R1 = live_obs(o, 4, x, seed=1)
  z2, R2 = live_obs(o, 4, x, seed=2)
  z = np.stack([z1, z2], 1)
  R = np.stack([R1, R2], 1)
  _same(a, b, a.step(4, 0.01, z, R), b.step(4, 0.01, z, R))          # n_obs = 2
  a.predict(0.02); b.predict(0.02)
  _same(a, b)
  _same(a, b, a.update(10, *live_obs(o, 10, x, seed=3)), b.update(10, *live_obs(o, 10, x, seed=3)))
  ha, hb = a.new_history(2), b.new_history(2)
  for k, t in ((12, 0.05), (4, 0.06)):
    zk, Rk = live_obs(o, k, x, seed=int(t * 100))
    _same(a, b, a.step_recorded(ha, k, t, zk, Rk), b.step_recorded(hb, k, t, zk, Rk))
  for sa, sb in ((ha.P_pred, hb.P_pred), (ha.P_filt, hb.P_filt), (ha.x_pred, hb.x_pred), (ha.x_filt, hb.x_filt)):
    assert torch.equal(sa, sb)
  # the filtered slab is the state, an exact mirror; the predicted slab holds the kernel's columns, symmetric to rounding
  assert torch.equal(ha.P_filt[1], a.P) and torch.equal(ha.P_filt, ha.P_filt.transpose(2, 3))
  assert float((ha.P_pred - ha.P_pred.transpose(2, 3)).abs().max()) <= 1e-12 * float(ha.P_pred.abs().max())


def test_gather_list_with_ragged_tail(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  B = 1000
  x, P, Qm = live_batch(B, seed=8)
  a, b = _engines(gen_dir, x, P, Qm)
  idx = torch.as_tensor(np.random.default_rng(3).permutation(B)[:333].astype(np.int32)).cuda()   # 333 = 20 groups + 13
  z, R = live_obs(o, 12, x[idx.cpu().numpy()])
  dt = torch.full((333,), 0.01, dtype=torch.float64, device="cuda")
  _same(a, b, a.step_indexed(12, idx, dt, z.copy(), R), b.step_indexed(12, idx, dt, z.copy(), R))


def test_upper_triangle_of_the_input_is_never_read(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  B = 515
  x, P, Qm = live_batch(B, seed=9)
  z, R = live_obs(o, 12, x)
  Pu = P.copy()
  iu = np.triu_indices(22, 1)
  Pu[:, iu[0], iu[1]] += 1.0                         # a gross perturbation: would change every result if read
  a, b = _engines(gen_dir, x, P, Qm)
  c, d = _engines(gen_dir, x, Pu, Qm)
  ya, yb, yc, yd = (e.step(12, 0.01, z, R) for e in (a, b, c, d))
  _same(a, b, ya, yb)
  _same(a, c, ya, yc)
  _same(a, d, ya, yd)
  da = a.maha_dist(12, z, R)
  assert torch.equal(da, b.maha_dist(12, z, R)) and torch.equal(da, d.maha_dist(12, z, R))


def test_row_accessors_and_graph_replay(gen_dir, oracle_dir):
  o = Oracle(oracle_dir, "live")
  B = 300
  x, P, Qm = live_batch(B, seed=10)
  a, b = _engines(gen_dir, x, P, Qm)
  z, R = live_obs(o, 4, x)
  zd, Rd = torch.as_tensor(z).cuda(), torch.as_tensor(R).cuda()
  a.step(4, 0.01, zd.clone(), Rd)
  ids = torch.tensor([5, 299, 0, 42], device="cuda")
  rows = a.get_P_rows(ids)
  assert not a._full_owns                           # rows only: the batch stays packed
  assert torch.equal(rows, a.P[ids])
  new = torch.as_tensor(live_batch(4, seed=11)[1]).cuda()
  a.step(4, 0.01, zd.clone(), Rd)                   # repacks after the read above
  a.set_P_rows(ids, new)
  assert not a._full_owns and torch.equal(a.get_P_rows(ids), new) and torch.equal(a.P[ids], new)
  # capture / replay: the graph reads and writes the P a caller sees
  zw = torch.empty(B, 1, 3, dtype=torch.float64, device="cuda")

  def run(e):
    for _ in range(3):
      zw[:, 0].copy_(zd)
      e.step(4, 0.01, zw, Rd)
  x0, P0 = a.x.clone(), a.P.clone()
  g = a.capture(lambda: run(a))
  a.x.copy_(x0); a.P.copy_(P0)
  g.replay()
  b.x.copy_(x0); b.P.copy_(P0)
  run(b)
  _same(a, b)
  a.step(4, 0.01, zd.clone(), Rd); b.step(4, 0.01, zd.clone(), Rd)   # eager between replays
  g.replay(); run(b)
  torch.cuda.synchronize()
  _same(a, b)


def test_million_filter_step_against_the_oracle(gen_dir, oracle_dir):
  from rednose_b200.batched import BatchedEKF
  o = Oracle(oracle_dir, "live")
  B = 1 << 20
  x1, P1, Qm = live_batch(1024, seed=12)
  x = np.tile(x1, (B // 1024, 1))
  e = BatchedEKF(gen_dir, "live", Qm, x, torch.as_tensor(P1).cuda().repeat(B // 1024, 1, 1), quaternion_idxs=[3])
  z1, R1 = live_obs(o, 4, x1)
  y = e.step(4, 0.01, np.tile(z1, (B // 1024, 1)), R1[0])
  sel = np.random.default_rng(0).choice(B, 2048, replace=False)
  xr, Pr, yr = o.batch_step(4, x[sel], P1[sel % 1024], Qm, 0.01, z1[sel % 1024], np.tile(R1[:1], (2048, 1, 1)), quat_idxs=[3], flags=3)
  st = torch.as_tensor(sel).cuda()
  assert state_err(e.x[st].cpu().numpy(), xr) < 1e-9
  assert cov_err(e.P[st].cpu().numpy(), Pr) < 1e-9
  assert state_err(y[st, 0].cpu().numpy(), yr) < 1e-9
