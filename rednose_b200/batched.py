"""Batched EKF engine: B independent filter instances resident in H100 HBM.

This is the batched counterpart of the reference's per-instance driver
(rednose/helpers/ekf_sym.cc:158-219 / ekf_sym.py:484-531): the state ``x[B, DIM]`` and
covariance ``P[B, EDIM, EDIM]`` (float64, row-major, AoS per filter) live on the device as
torch tensors -- torch is only the allocator / stream provider -- and every step is ONE launch of
the generated library's fused ``<name>_batch_step_<kind>`` kernel through its C-ABI.

Semantics follow the C++ driver: predict(dt) -> [normalise quaternions] -> update(kind) ->
[normalise] (ekf_sym.cc:162,207,213); the innovation overwrites ``z`` (ekf_c.c:120).

Filters served by the two-filters-per-warp kernel (even EDIM <= 32, e.g. live_kf) keep P resident in that kernel's packed
layout, the lower block triangle of 2x2 blocks (csrc/ekf_packed.cuh: 264 instead of 484 doubles per live filter), which
halves the covariance traffic of a step.  ``P`` still reads as the full ``[B, EDIM, EDIM]`` tensor; see ``BatchedEKF.P``.
For the same filters a history may record its covariances in that layout too (``new_history(T, packed=True)``), which
shrinks a live history step from 8 112 to 4 592 bytes; ``unpack_P`` turns any packed slab back into full matrices.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from rednose_b200.loader import load_code, raise_on_cuda_error

NORM_AFTER_PREDICT = 1
NORM_AFTER_UPDATE = 2
Q_IS_DIAGONAL = 4
SHARED_R = 8
AUGMENT = 16   # fused clone-window shift (CTA kernel only)
PACKED_P = 32  # P is in the packed lower-block-triangle layout (two-filters-per-warp kernel only)
PACKED_HIST = 64  # the covariance history slabs are in that layout (same kernel only)
MAIN_HIST = 128   # the predicted-covariance history slab keeps the main block only (EDIM > 32; set by the _mainhist entry points)

PACKED_REFUSED = ("packed covariances exist only where the two-filters-per-warp kernel serves the filter (even EDIM <= 32, "
                  "no feature-track kind)")
MAIN_PRED_REFUSED = "main-block prediction histories exist only above EDIM 32 (an MSCKF smoothed on its main block)"


def main_pred_doubles(folder, name):
  """Doubles per filter-step of the main-block prediction history of filter `name` (MEDIM^2), 0 where it does not exist
  (EDIM <= 32)."""
  _, lib = load_code(folder, name)
  return int(getattr(lib, f"{name}_main_pred_doubles")())


def packed_P_doubles(folder, name):
  """Doubles per filter of the packed covariance layout of filter `name` (csrc/ekf_packed.cuh), 0 where it is not used."""
  _, lib = load_code(folder, name)
  return int(getattr(lib, f"{name}_packed_P_doubles")())


def _as_device(t, device, dtype=torch.float64):
  if isinstance(t, torch.Tensor):
    return t.to(device=device, dtype=dtype, non_blocking=True).contiguous()
  return torch.as_tensor(np.ascontiguousarray(t, dtype=np.float64)).to(device, non_blocking=True)


class BatchedEKF:
  def __init__(self, folder, name, Q, x_initial, P_initial, batch=None, device="cuda", quaternion_idxs=(),
               norm_after_predict=True, norm_after_update=True, global_vars=None):
    """x_initial: [DIM] (broadcast to `batch` filters) or [B, DIM]; P_initial: [EDIM, EDIM] or [B, EDIM, EDIM]."""
    if not torch.cuda.is_available():
      raise RuntimeError("rednose_b200.BatchedEKF needs a CUDA device (no CPU fallback exists)")
    self.name = name
    self.device = torch.device(device)
    self._ffi, self._lib = load_code(folder, name)
    ffi = self._ffi
    # single states / covariances are broadcast ON THE DEVICE (a 1M x 22 x 22 tile is 3.9 GB: never built on the host)
    x0 = _as_device(x_initial, self.device)
    P0 = _as_device(P_initial, self.device)
    if x0.ndim == 1:
      assert batch is not None, "batch size needed when broadcasting a single initial state"
      x0 = x0.expand(batch, -1)
    B = x0.shape[0]
    if P0.ndim == 2:
      P0 = P0.expand(B, -1, -1)
    self.B, self.dim_x, self.dim_err = B, x0.shape[1], P0.shape[1]
    self.x = x0.contiguous().clone()
    # covariance storage: the full buffer `_Pf` and, when the pair kernel serves this filter, the packed resident buffer
    # `_Pk`; `_full_owns` says which of the two holds the current P
    self._packed_doubles = int(getattr(self._lib, f"{name}_packed_P_doubles")())
    # MEDIM^2 above EDIM 32 (a main-block prediction history is available), 0 elsewhere
    self._main_pred_doubles = int(getattr(self._lib, f"{name}_main_pred_doubles")())
    self._Pf = P0.contiguous().clone()
    self._full_owns = True
    self._Pk = None
    if self._packed_doubles:
      self._Pk = torch.empty(B, self._packed_doubles, dtype=torch.float64, device=self.device)
      self._sync_packed()
      self._Pf = None            # a million live covariances are 3.9 GB in full: allocated again only when P is read
    self.Q = _as_device(Q, self.device)
    assert self.Q.shape == (self.dim_err, self.dim_err)
    self.filter_time = None  # scalar time shared by the batch, or a [B] tensor
    self._quat = ffi.new("int[]", list(quaternion_idxs) or [0])
    self._nquat = len(quaternion_idxs)
    self.flags = (NORM_AFTER_PREDICT if norm_after_predict else 0) | (NORM_AFTER_UPDATE if norm_after_update else 0)
    Qh = np.asarray(Q, dtype=np.float64) if not isinstance(Q, torch.Tensor) else Q.detach().cpu().numpy()
    if np.count_nonzero(Qh - np.diag(np.diagonal(Qh))) == 0:
      self.flags |= Q_IS_DIAGONAL  # lets the kernels skip the dense dt*Q read
    self.kinds = sorted(int(s[len(name) + 12:]) for s in dir(self._lib) if s.startswith(f"{name}_batch_step_") and not s.endswith("_idx"))
    # feature-track kinds (those with an He leaf): the CTA-per-filter kernel runs them at any EDIM
    self._feature_kinds = {k for k in self.kinds if hasattr(self._lib, f"{name}_He_{k}")}
    self._zdim = {}
    self.launches = 0  # kernels launched through this object (bench.py reports it)
    for g, v in (global_vars or {}).items():
      getattr(self._lib, f"{name}_set_{g}")(float(v))

  # -------------------------------------------------------------- covariance ---
  @property
  def P(self):
    """The covariances as a [B, EDIM, EDIM] tensor.  With the packed resident layout this unpacks into a full buffer
    that is kept allocated; from then on that buffer is the state (the caller may write through it), and the next step
    packs it again.  So a handle taken from ``P`` is a snapshot of the moment it was read, not live storage: read ``P``
    again after stepping."""
    if self._Pk is not None and not self._full_owns:
      if self._Pf is None:
        self._Pf = torch.empty(self.B, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device)
      self._convert(self._Pf, None, self.B, to_packed=False)
      self._full_owns = True
    return self._Pf

  @P.setter
  def P(self, value):
    value = _as_device(value, self.device)
    assert value.shape == (self.B, self.dim_err, self.dim_err)
    self._Pf = value
    self._full_owns = True

  def _convert(self, full, idx, n, to_packed):
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_convert_P")(
        self._p(full), self._p(self._Pk), self._ffi.cast("const int *", idx.data_ptr()) if idx is not None else self._ffi.NULL,
        int(n), 1 if to_packed else 0, self._stream())
    self._check("convert_P")

  def _sync_packed(self):
    if self._full_owns:
      self._convert(self._Pf, None, self.B, to_packed=True)
      self._full_owns = False

  def _P_arg(self):
    """(pointer to the covariance a launch reads and writes, layout flag)."""
    if self._Pk is None:
      return self._p(self._Pf), 0
    self._sync_packed()
    return self._p(self._Pk), PACKED_P

  def get_P_rows(self, ids):
    """P of the filters `ids` as a new [n, EDIM, EDIM] tensor, without converting the rest of the batch."""
    ids = torch.as_tensor(ids, device=self.device)
    if self._Pk is None or self._full_owns:
      return self._Pf[ids]
    out = torch.empty(int(ids.shape[0]), self.dim_err, self.dim_err, dtype=torch.float64, device=self.device)
    if out.shape[0]:
      self._convert(out, ids.to(torch.int32).contiguous(), out.shape[0], to_packed=False)
    return out

  def set_P_rows(self, ids, P):
    """Overwrite P of the filters `ids` (distinct) with P [n, EDIM, EDIM]; only their lower triangles are kept in the
    packed layout."""
    ids = torch.as_tensor(ids, device=self.device)
    if self._Pk is None or self._full_owns:
      self._Pf[ids] = P
      return
    P = _as_device(P, self.device)
    if P.shape[0]:
      self._convert(P, ids.to(torch.int32).contiguous(), P.shape[0], to_packed=True)

  # ----------------------------------------------------------------- helpers ---
  def _p(self, t):
    return self._ffi.cast("double *", t.data_ptr()) if t is not None else self._ffi.NULL

  def _cp(self, t):
    return self._ffi.cast("const double *", t.data_ptr()) if t is not None else self._ffi.NULL

  def _stream(self):
    return self._ffi.cast("void *", torch.cuda.current_stream(self.device).cuda_stream)

  def _check(self, what):
    raise_on_cuda_error(self._lib, self.name, what)

  def _hist_flag(self, *slabs):
    """PACKED_HIST when the covariance history slabs (or rows of them) are packed [..., packed doubles], 0 when they are
    full [..., EDIM, EDIM]; all of them must be in the same layout."""
    packed = set()
    for s in slabs:
      if s is None:
        continue
      if tuple(s.shape[-2:]) == (self.dim_err, self.dim_err):
        packed.add(False)
      else:
        assert self._packed_doubles and s.shape[-1] == self._packed_doubles, \
          f"covariance history slab of shape {tuple(s.shape)}: neither [..., {self.dim_err}, {self.dim_err}] nor packed [..., {self._packed_doubles}]"
        packed.add(True)
    assert len(packed) <= 1, "the covariance history slabs of one launch must share one layout"
    return PACKED_HIST if True in packed else 0

  def unpack_P(self, packed):
    """Full [..., EDIM, EDIM] covariances of packed ones [..., packed doubles] (a packed history slab, a row of one, or
    the smoothed Ps of a packed history); a new tensor."""
    assert self._packed_doubles and packed.shape[-1] == self._packed_doubles, (tuple(packed.shape), self._packed_doubles)
    packed = packed.contiguous()
    out = torch.empty(*packed.shape[:-1], self.dim_err, self.dim_err, dtype=torch.float64, device=packed.device)
    n = packed.numel() // self._packed_doubles
    if n:
      with torch.cuda.device(self.device):
        getattr(self._lib, f"{self.name}_convert_P")(self._p(out), self._p(packed), self._ffi.NULL, n, 0, self._stream())
      self._check("convert_P")
    return out

  def _dt_args(self, dt):
    if isinstance(dt, torch.Tensor):
      dt = dt.to(self.device, torch.float64).contiguous()
      assert dt.shape == (self.B,)
      return dt, self._cp(dt), 0.0
    return None, self._ffi.NULL, float(dt)

  # ------------------------------------------------------------------- steps ---
  def predict(self, dt, hist=None):
    """P <- F P F^T + dt Q, x <- f(x, dt) for the whole batch (ekf_c.c:8-33)."""
    keep, dt_ptr, dt_s = self._dt_args(dt)
    hx, hP = (hist if hist is not None else (None, None))
    hflag = self._hist_flag(hP)
    P, pflag = self._P_arg()
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_predict")(
        self._p(self.x), P, self._cp(self.Q), dt_ptr, dt_s, self.B, self._quat, self._nquat, self.flags | pflag | hflag,
        self._p(hx), self._p(hP), self._stream())
    self.launches += 1
    self._check("batch_predict")

  def _obs_args(self, z, R, ea):
    z = _as_device(z, self.device)
    R = _as_device(R, self.device)
    if z.ndim == 2:
      z = z.unsqueeze(1)
    flags = self.flags
    if R.ndim == 2:   # one noise matrix for the whole batch (what KalmanFilter.get_R replicates, kalmanfilter.py:37-43)
      assert R.shape[0] == R.shape[1] == z.shape[2]
      flags |= SHARED_R
    else:
      if R.ndim == 3:
        R = R.unsqueeze(1)
      assert R.shape[:2] == z.shape[:2] and R.shape[2] == R.shape[3] == z.shape[2]
    assert z.shape[0] == self.B
    ea = _as_device(ea, self.device) if ea is not None else None
    return z, R, ea, z.shape[1], flags

  def update(self, kind, z, R, ea=None, hist=None):
    """Measurement update of one kind for the whole batch (ekf_c.c:37-121); returns the innovations y [B, n, m]."""
    z, R, ea, n_obs, flags = self._obs_args(z, R, ea)
    hx, hP = (hist if hist is not None else (None, None))
    hflag = self._hist_flag(hP)
    P, pflag = self._P_arg()
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_update_{kind}")(
        self._p(self.x), P, self._p(z), self._cp(R), self._cp(ea), n_obs, self.B,
        self._quat, self._nquat, flags | pflag | hflag, self._p(hx), self._p(hP), self._stream())
    self.launches += 1
    self._check(f"batch_update_{kind}")
    return z

  def step_indexed(self, kind, idx, dt, z, R, ea=None, hist=None, t=None, augment=False):
    """Fused predict + update of `kind` for the filters listed in `idx` only ([n] int32, device): entry e uses
    z[e], R[e] (or one shared R), dt[e] and works on filter idx[e].  Filters not listed are untouched.  This is the
    building block of the ragged scheduler (per-tick kind buckets).

    With a RaggedHistory `hist`, entry e also records its step at filter idx[e]'s next row, with time t[e] (scalar
    or [n]); a filter whose T rows are used up still steps and counts an overflow.

    augment (MSCKF): True, or an [n] bool mask aligned with `idx`: the flagged filters shift their clone window after
    their update, as predict_and_update_batch(..., augment=True) (ekf_sym.py:527-528); a recorded row keeps the estimate
    before the shift.  Kinds the CTA-per-filter kernel runs (EDIM > 32, or a feature-track kind) shift inside their own
    gather launch (the fused shift); the others step in one launch and shift the flagged filters in a second one.  The
    innovations keep the order of `idx`."""
    if augment is None or augment is False:
      return self._step_indexed(kind, idx, dt, z, R, ea, hist, t)
    idx = idx.to(device=self.device, dtype=torch.int32).contiguous()
    n = int(idx.shape[0])
    mask = torch.as_tensor(augment, device=self.device).to(torch.bool).expand(n)
    if not bool(mask.any()):
      return self._step_indexed(kind, idx, dt, z, R, ea, hist, t)
    if not (self.dim_err > 32 or kind in self._feature_kinds):
      y = self._step_indexed(kind, idx, dt, z, R, ea, hist, t)
      self.augment(idx[mask])
      return y
    # the fused shift: the flagged entries in a gather launch of their own with the AUGMENT flag
    z = _as_device(z, self.device)
    if z.ndim == 2:
      z = z.unsqueeze(1)
    R = _as_device(R, self.device)
    ea = _as_device(ea, self.device) if ea is not None else None
    if t is not None and torch.as_tensor(t).ndim == 1:
      t = torch.as_tensor(t, dtype=torch.float64, device=self.device)
    for sel, aug in (((~mask).nonzero(as_tuple=True)[0], 0), (mask.nonzero(as_tuple=True)[0], AUGMENT)):
      if sel.numel() == 0:
        continue
      dt_s = dt.to(self.device)[sel] if isinstance(dt, torch.Tensor) else dt
      t_s = t[sel] if isinstance(t, torch.Tensor) and t.ndim == 1 else t
      y = self._step_indexed(kind, idx[sel], dt_s, z[sel], R if R.ndim == 2 else R[sel], None if ea is None else ea[sel],
                             hist, t_s, extra_flags=aug)
      z[sel] = y
    return z

  def _step_indexed(self, kind, idx, dt, z, R, ea=None, hist=None, t=None, extra_flags=0):
    idx = idx.to(device=self.device, dtype=torch.int32).contiguous()
    n = int(idx.shape[0])
    if n == 0:
      return None
    z = _as_device(z, self.device)
    if z.ndim == 2:
      z = z.unsqueeze(1)
    R = _as_device(R, self.device)
    flags = self.flags | extra_flags
    if R.ndim == 2:
      flags |= SHARED_R
    elif R.ndim == 3:
      R = R.unsqueeze(1)
    assert z.shape[0] == n
    ea = _as_device(ea, self.device) if ea is not None else None
    if isinstance(dt, torch.Tensor):
      dt = dt.to(self.device, torch.float64).contiguous()
      assert dt.shape == (n,)
      dt_ptr, dt_s = self._cp(dt), 0.0
    else:
      dt_ptr, dt_s = self._ffi.NULL, float(dt)
    P, pflag = self._P_arg()
    idx_p = self._ffi.cast("const int *", idx.data_ptr())
    with torch.cuda.device(self.device):
      if hist is None:
        getattr(self._lib, f"{self.name}_batch_step_{kind}_idx")(
          self._p(self.x), P, self._cp(self.Q), dt_ptr, dt_s, self._p(z), self._cp(R), self._cp(ea),
          z.shape[1], n, self._quat, self._nquat, flags | pflag, self._ffi.NULL, self._ffi.NULL, self._ffi.NULL, self._ffi.NULL,
          idx_p, self._stream())
      else:
        assert t is not None, "a recorded step needs its time"
        assert hist.B == self.B, (hist.B, self.B)
        hflag = self._hist_flag(hist.P_pred, hist.P_filt)
        assert bool(hflag) == hist.packed
        rows = hist.reserve(idx, t)
        getattr(self._lib, f"{self.name}_batch_step_{kind}_hist_idx")(
          self._p(self.x), P, self._cp(self.Q), dt_ptr, dt_s, self._p(z), self._cp(R), self._cp(ea),
          z.shape[1], n, self._quat, self._nquat, flags | pflag | hflag,
          self._p(hist.x_pred), self._p(hist.P_pred), self._p(hist.x_filt), self._p(hist.P_filt),
          idx_p, self._ffi.cast("const int *", rows.data_ptr()), hist.B, self._stream())
    self.launches += 1
    self._check(f"batch_step_{kind}_idx")
    return z

  def step(self, kind, dt, z, R, ea=None, hist_pred=None, hist_filt=None, augment=False, hist_pred_last=None):
    """Fused predict(dt) + update(kind): one kernel launch, P read and written once.  augment=True also shifts the MSCKF
    clone window (predict_and_update_batch(..., augment=True), ekf_sym.py:527-528): inside the same launch for filters on
    the CTA-per-filter kernel (EDIM > 32), as a second launch otherwise.

    hist_pred_last [B, EDIM, EDIM] (EDIM > 32): record a main-block prediction history -- hist_pred's covariance row is
    then [B, MEDIM, MEDIM] and receives the main block of P_{k+1|k}, hist_pred_last the whole of it."""
    keep, dt_ptr, dt_s = self._dt_args(dt)
    z, R, ea, n_obs, flags = self._obs_args(z, R, ea)
    fused_aug = bool(augment) and self.dim_err > 32
    if fused_aug:
      flags |= AUGMENT
    hxp, hPp = (hist_pred if hist_pred is not None else (None, None))
    hxf, hPf = (hist_filt if hist_filt is not None else (None, None))
    if hist_pred_last is None:
      hflag = self._hist_flag(hPp, hPf)
      fn, last = f"{self.name}_batch_step_{kind}", ()
    else:
      me = self._main_block_dim()
      assert hPp is None or tuple(hPp.shape[-2:]) == (me, me), (tuple(hPp.shape), me)
      assert tuple(hist_pred_last.shape) == (self.B, self.dim_err, self.dim_err), tuple(hist_pred_last.shape)
      hflag = self._hist_flag(hPf)
      fn, last = f"{self.name}_batch_mainhist_step_{kind}", (self._p(hist_pred_last),)
    P, pflag = self._P_arg()
    with torch.cuda.device(self.device):
      getattr(self._lib, fn)(
        self._p(self.x), P, self._cp(self.Q), dt_ptr, dt_s, self._p(z), self._cp(R), self._cp(ea),
        n_obs, self.B, self._quat, self._nquat, flags | pflag | hflag, self._p(hxp), self._p(hPp), self._p(hxf), self._p(hPf),
        *last, self._stream())
    self.launches += 1
    self._check(f"batch_step_{kind}")
    if augment and not fused_aug:
      self.augment()
    return z

  # driver-style entry point: time in, observations in (host or device), innovations out
  def predict_and_update_batch(self, t, kind, z, R, extra_args=None, augment=False):
    """All B filters observe `kind` at time t (scalar or [B]); returns (x [B,DIM] device, y [B,n,m] device)."""
    if self.filter_time is None:
      self.filter_time = t
    dt = t - self.filter_time
    if not isinstance(dt, torch.Tensor):
      assert dt >= 0
    y = self.step(kind, dt, z, R, extra_args, augment=augment)
    self.filter_time = t
    return self.x, y

  # ------------------------------------------------------------- CUDA graphs ---
  def capture(self, fn, warmup=1):
    """Capture the launches `fn()` makes -- steps of this engine on DEVICE-resident arguments (no host copies, no
    allocations) -- into a CUDA graph and return it; `graph.replay()` then re-issues the whole sequence with one driver
    call.  For small states (kinematic: 28 us per launch of a million filters) the per-launch driver cost is comparable
    to the kernel, and a captured loop removes it.  `fn` is run `warmup` times first, uncaptured, so that one-time kernel
    attribute setup does not land inside the capture.

    With the packed resident layout the graph packs ``P`` before the captured launches and unpacks it after them, so a
    replay reads and writes the full ``P`` a caller sees (``eng.P.copy_(P0); graph.replay()`` restarts from P0)."""
    side = torch.cuda.Stream(self.device)
    side.wait_stream(torch.cuda.current_stream(self.device))
    with torch.cuda.stream(side):
      for _ in range(max(1, int(warmup))):
        fn()
      if self._Pk is not None:
        self.P                # the full buffer exists and holds the current state before the capture starts
    torch.cuda.current_stream(self.device).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
      if self._Pk is not None:
        self._convert(self._Pf, None, self.B, to_packed=True)
        self._full_owns = False
      fn()
      if self._Pk is not None:
        self._convert(self._Pf, None, self.B, to_packed=False)
        self._full_owns = True
    return g if self._Pk is None else _PackedGraph(g, self)

  # -------------------------------------------------------------- host access ---
  def state(self):
    return self.x.cpu().numpy()

  def covs(self):
    return self.P.cpu().numpy()

  def init_state(self, x, P, filter_time=None):
    self.x.copy_(_as_device(x, self.device).expand_as(self.x))
    if self._Pf is None:
      self._Pf = torch.empty(self.B, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device)
    self._Pf.copy_(_as_device(P, self.device).expand_as(self._Pf))   # overwrites every filter: nothing to unpack first
    self._full_owns = True
    self.filter_time = filter_time

  def maha_dist(self, kind, z, R, ea=None):
    """Mahalanobis distance y^T (H P H^T + R)^-1 y of one observation per filter, without touching the state
    (the quantity EKF_sym.maha_test thresholds, ekf_sym.py:626-649).  Returns a [B] device tensor."""
    z = _as_device(z, self.device).reshape(self.B, -1).contiguous()
    R = _as_device(R, self.device)
    flags = SHARED_R if R.ndim == 2 else 0
    ea = _as_device(ea, self.device) if ea is not None else None
    out = torch.empty(self.B, dtype=torch.float64, device=self.device)
    P, pflag = self._P_arg()
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_maha_{kind}")(
        self._cp(self.x), P, self._cp(z), self._cp(R), self._cp(ea), self.B, flags | pflag, self._p(out), self._stream())
    self.launches += 1
    self._check(f"batch_maha_{kind}")
    return out

  def maha_test(self, kind, z, R, ea=None, maha_thresh=0.95):
    """True where the observation passes the chi-square gate at `maha_thresh` (batched EKF_sym.maha_test)."""
    from rednose_b200.chi2 import chi2_ppf
    d = self.maha_dist(kind, z, R, ea)
    return d <= float(chi2_ppf(maha_thresh, z.shape[-1] if hasattr(z, "shape") else len(z[0])))

  def augment(self, ids=None):
    """MSCKF clone window shift (ekf_sym.py:365-391), one launch: for the whole batch, or with `ids` ([m] int, distinct,
    device or host) for those filters only.  The shift works on the full covariance: a packed resident P is unpacked
    first (reading ``P``)."""
    if ids is None:
      with torch.cuda.device(self.device):
        getattr(self._lib, f"{self.name}_batch_augment")(self._p(self.x), self._p(self.P), self.B, self._stream())
      self.launches += 1
      self._check("batch_augment")
      return
    ids = torch.as_tensor(ids, device=self.device).to(torch.int32).contiguous()
    if ids.numel() == 0:
      return
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_augment_idx")(
        self._p(self.x), self._p(self.P), self._ffi.cast("const int *", ids.data_ptr()), int(ids.shape[0]), 0, self._stream())
    self.launches += 1
    self._check("batch_augment_idx")

  # ------------------------------------------------------- history + smoothing ---
  def _history_doubles(self, packed):
    if not packed:
      return 0
    if not self._packed_doubles:
      raise ValueError(f"filter '{self.name}': packed histories are not available: {PACKED_REFUSED}")
    return self._packed_doubles

  def _main_block_dim(self):
    return math.isqrt(self._main_pred_doubles)

  def new_history(self, T, packed=False, main_pred=False):
    """Device slabs for a T-step history, time-major: what the reference keeps as the list of
    9-tuples returned by predict_and_update_batch (ekf_sym.py:531): x_{k|k-1}, x_{k|k}, P_{k|k-1}, P_{k|k}, t.

    packed=True records the covariances in the packed layout of the resident P ([T, B, packed doubles]: 57 % of the
    bytes of a live history step); raises ValueError where this filter has no packed layout.

    main_pred=True (EDIM > 32, an MSCKF) keeps only the main block of each predicted covariance, P_pred [T, B, MEDIM,
    MEDIM], plus the full prediction of the newest step, P_pred_last [B, EDIM, EDIM]: all the smoother reads of them
    (59 152 instead of 109 072 bytes per msckf step).  Raises ValueError at EDIM <= 32 and together with packed=True."""
    if main_pred:
      if packed:
        raise ValueError("a main-block prediction history is in the full covariance layout: packed=True does not apply")
      if not self._main_pred_doubles:
        raise ValueError(f"filter '{self.name}': EDIM {self.dim_err}: {MAIN_PRED_REFUSED}")
      return History(T, self.B, self.dim_x, self.dim_err, self.device, main_block=self._main_block_dim())
    return History(T, self.B, self.dim_x, self.dim_err, self.device, self._history_doubles(packed))

  def new_ragged_history(self, T, packed=False):
    """Device slabs for up to T recorded steps PER FILTER, each filter on its own clock (step_indexed(..., hist=)):
    row k of filter b is the k-th step that filter recorded.  packed: as in new_history."""
    return RaggedHistory(T, self.B, self.dim_x, self.dim_err, self.device, self._history_doubles(packed))

  def restore_from_history(self, hist, ids, rows):
    """Set x and P of the filters `ids` ([m] distinct) to x_filt / P_filt of row rows[e] ([m] int32) of the RaggedHistory
    `hist`: the estimate filter ids[e] recorded there.  One launch; an entry with a negative row is skipped."""
    ids = torch.as_tensor(ids, device=self.device).to(torch.int32).contiguous()
    rows = torch.as_tensor(rows, device=self.device).to(torch.int32).contiguous()
    assert hist.B == self.B and ids.shape == rows.shape, (hist.B, self.B, tuple(ids.shape), tuple(rows.shape))
    hflag = self._hist_flag(hist.P_filt)
    P, pflag = self._P_arg()
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_restore_hist")(
        self._cp(hist.x_filt), self._cp(hist.P_filt), self._ffi.cast("const int *", ids.data_ptr()),
        self._ffi.cast("const int *", rows.data_ptr()), int(ids.shape[0]), hist.B, self._p(self.x), P, pflag | hflag,
        self._stream())
    self.launches += 1
    self._check("batch_restore_hist")

  def step_recorded(self, hist, kind, t, z, R, ea=None, augment=False):
    """predict_and_update_batch that also appends this step to `hist` (the kernel writes the slabs itself).  augment=True
    shifts the MSCKF clone window after the update, as step(augment=True); the recorded x_{k|k} / P_{k|k} are the
    estimate before the shift, as predict_and_update_batch(augment=True) returns it (ekf_sym.py:522-530)."""
    k = hist.n
    assert k < hist.T, "history is full"
    if self.filter_time is None:
      self.filter_time = t
    dt = t - self.filter_time
    y = self.step(kind, dt, z, R, ea, hist_pred=(hist.x_pred[k], hist.P_pred[k]), hist_filt=(hist.x_filt[k], hist.P_filt[k]),
                  augment=augment, hist_pred_last=hist.P_pred_last)
    self.filter_time = t
    hist.t_host[k] = float(t)
    hist.n += 1
    return y

  def rts_smooth(self, hist, norm_quats=False, quaternion_idxs=(3,), in_place=False, out=None, terminal=None, k0=0):
    """Batched RTS backward pass over a recorded history (ekf_sym.py:651-690, one launch for all filters).

    Returns (xs [T, B, DIM], Ps [T, B, EDIM, EDIM]) on the device.  `norm_quats` normalises the quaternion(s)
    at `quaternion_idxs` the way the reference normalises its hard-coded slice 3:7.  A packed history (new_history(T,
    packed=True)) gives packed Ps [T, B, packed doubles] (see unpack_P), and `out` / `terminal` covariances are packed
    like it.  A main-block prediction history (new_history(T, main_pred=True)) gives full Ps, bit for bit those of the
    full history, and takes full `out` / `terminal` covariances.

    `terminal=(x [B, DIM], P [B, EDIM, EDIM])` smooths one SEGMENT of a longer history (steps k0 .. k0 + T - 2): the
    recursion starts from that smoothed estimate of step k0 + T - 1, whose history entry (the last one recorded) only
    contributes its predicted state; its row of xs / Ps is not written.

    With a RaggedHistory every filter is smoothed over its own n[b] rows and times, and (xs, Ps) are [T, B, ...]: row k
    of filter b is the smoothed estimate of its k-th recorded step; rows >= n[b] are not written (NaN in a new buffer).
    Raises if a filter outran the history.
    """
    if isinstance(hist, RaggedHistory):
      return self._rts_smooth_ragged(hist, norm_quats, quaternion_idxs, in_place, out, terminal, k0)
    T = hist.n
    assert T >= 1
    hist.sync_times()
    if out is not None:
      xs, Ps = out                      # caller-provided [T, B, DIM] / [T, B, EDIM, EDIM] (packed: [T, B, PD]) buffers
      assert xs.shape[0] >= T and Ps.shape[0] >= T and xs.shape[1:] == hist.x_filt.shape[1:] and Ps.shape[1:] == hist.P_filt.shape[1:], \
        ("out must match the history's layout", tuple(xs.shape), tuple(Ps.shape), tuple(hist.P_filt.shape))
    else:
      xs = hist.x_filt if in_place else torch.empty_like(hist.x_filt)
      Ps = hist.P_filt if in_place else torch.empty_like(hist.P_filt)
    qi = self._ffi.new("int[]", list(quaternion_idxs) or [0])
    sfx = "_packed" if hist.packed else ("_mainhist" if hist.main_pred else "")
    last = (self._cp(hist.P_pred_last),) if hist.main_pred else ()
    with torch.cuda.device(self.device):
      if terminal is None and not k0:
        getattr(self._lib, f"{self.name}_batch_rts{sfx}")(
          self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t), 0,
          self._p(xs), self._p(Ps), T, self.B, qi, len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0, *last,
          self._stream())
      else:
        xt, Pt = terminal if terminal is not None else (None, None)   # the LAST segment of a history has k0 > 0 but no terminal
        assert xt is None or (xt.is_contiguous() and Pt.is_contiguous() and xt.shape == (self.B, self.dim_x) and Pt.shape == hist.P_filt.shape[1:]), \
          "terminal=(x [B, DIM], P [B, EDIM, EDIM] or, for a packed history, [B, packed doubles])"
        getattr(self._lib, f"{self.name}_batch_rts_segment{sfx}")(
          self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t), 0,
          self._p(xs), self._p(Ps), T, self.B, qi, len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0,
          self._cp(xt), self._cp(Pt), int(k0), *last, self._stream())
    self.launches += 1
    self._check("batch_rts")
    return xs[:T], Ps[:T]

  def _rts_smooth_ragged(self, hist, norm_quats, quaternion_idxs, in_place, out, terminal, k0):
    if terminal is not None or k0:
      raise ValueError("a ragged history is smoothed whole: segment continuation (terminal, k0) does not apply")
    lost = hist.overflowed()
    if lost:
      raise RuntimeError(f"ragged history overflow: {lost} step(s) found their filter's {hist.T} rows used up and were "
                         f"not recorded; record into a longer history")
    if out is not None:
      xs, Ps = out
      assert xs.shape == hist.x_filt.shape and Ps.shape == hist.P_filt.shape and xs.is_contiguous() and Ps.is_contiguous()
    elif in_place:
      xs, Ps = hist.x_filt, hist.P_filt
    else:
      xs = torch.full_like(hist.x_filt, float("nan"))
      Ps = torch.full_like(hist.P_filt, float("nan"))
    qi = self._ffi.new("int[]", list(quaternion_idxs) or [0])
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_rts_ragged{'_packed' if hist.packed else ''}")(
        self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t),
        self._ffi.cast("const int *", hist.n.data_ptr()), self._p(xs), self._p(Ps), hist.T, self.B, qi,
        len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0, self._stream())
    self.launches += 1
    self._check("batch_rts_ragged")
    return xs, Ps

  def rts_smooth_ragged_segment(self, hist, term, k0, terminal, norm_quats=False, quaternion_idxs=(3,), in_place=False,
                                out=None):
    """RTS backward pass over one SEGMENT of per-filter streams too long for one RaggedHistory (RaggedCheckpointedSmoother
    in rednose_b200/smoothing.py drives it).  Filter b's n[b] rows of `hist` are its global rows k0[b] .. k0[b] + n[b] - 1
    (k0 [B] int64): every smoothed state but that of global row 0 has its quaternions normalised, as in a whole pass.

    term [B] (bool or uint8): where set, filter b's last row (n[b] - 1) is the first row of its segment behind, of which only
    the predicted state and time are read, and the recursion starts from terminal = (x [B, DIM], P [B, EDIM, EDIM], packed
    like the history), that row's smoothed estimate; row n[b] - 1 of xs / Ps is then not written.  Elsewhere filter b is
    smoothed as rts_smooth(hist) smooths it.  Returns (xs, Ps) [T, B, ...] like rts_smooth(hist)."""
    lost = hist.overflowed()
    if lost:
      raise RuntimeError(f"ragged history overflow: {lost} step(s) found their filter's {hist.T} rows used up and were "
                         f"not recorded; record into a longer history")
    term = torch.as_tensor(term, device=self.device).to(torch.uint8).contiguous()
    k0 = torch.as_tensor(k0, device=self.device).to(torch.int64).contiguous()
    xt, Pt = terminal
    assert term.shape == (self.B,) and k0.shape == (self.B,), (tuple(term.shape), tuple(k0.shape))
    assert xt.is_contiguous() and Pt.is_contiguous() and xt.shape == (self.B, self.dim_x) and Pt.shape == hist.P_filt.shape[1:], \
      "terminal=(x [B, DIM], P [B, EDIM, EDIM] or, for a packed history, [B, packed doubles])"
    if out is not None:
      xs, Ps = out
      assert xs.shape == hist.x_filt.shape and Ps.shape == hist.P_filt.shape and xs.is_contiguous() and Ps.is_contiguous()
    elif in_place:
      xs, Ps = hist.x_filt, hist.P_filt
    else:
      xs = torch.full_like(hist.x_filt, float("nan"))
      Ps = torch.full_like(hist.P_filt, float("nan"))
    qi = self._ffi.new("int[]", list(quaternion_idxs) or [0])
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_rts_ragged_segment")(
        self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t),
        self._ffi.cast("const int *", hist.n.data_ptr()), self._ffi.cast("const unsigned char *", term.data_ptr()),
        self._ffi.cast("const long long *", k0.data_ptr()), self._cp(xt), self._cp(Pt), self._p(xs), self._p(Ps), hist.T,
        self.B, qi, len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0, 1 if hist.packed else 0,
        self._stream())
    self.launches += 1
    self._check("batch_rts_ragged_segment")
    return xs, Ps


class _PackedGraph:
  """A captured graph of an engine with packed resident P: the graph reads and writes the full buffer, so before a
  replay that buffer is brought up to date (a no-op unless the engine was stepped eagerly since), and after it the full
  buffer holds the state."""

  def __init__(self, graph, engine):
    self.graph, self._e = graph, engine

  def replay(self):
    self._e.P                 # noqa: B018 -- unpacks only if eager steps ran since the last replay
    self.graph.replay()
    self._e._full_owns = True

  def __getattr__(self, name):
    return getattr(self.graph, name)


def _cov_shape(dim_err, packed_doubles):
  return (packed_doubles,) if packed_doubles else (dim_err, dim_err)


class History:
  """Time-major device buffers of a forward pass, consumed by the RTS kernel.  `packed`: the covariance slabs are
  [T, B, packed_doubles] in the packed layout (BatchedEKF.new_history(T, packed=True)) instead of [T, B, EDIM, EDIM].
  `main_pred` (main_block = MEDIM > 0): P_pred is [T, B, MEDIM, MEDIM] and P_pred_last [B, EDIM, EDIM] holds the full
  prediction of the newest recorded step (BatchedEKF.new_history(T, main_pred=True)); P_pred_last is None otherwise."""

  def __init__(self, T, B, dim_x, dim_err, device, packed_doubles=0, main_block=0):
    assert not (packed_doubles and main_block)
    kw = dict(dtype=torch.float64, device=device)
    self.T, self.B, self.n = T, B, 0
    self.packed = bool(packed_doubles)
    self.main_pred = bool(main_block)
    self.x_pred = torch.empty(T, B, dim_x, **kw)
    self.x_filt = torch.empty(T, B, dim_x, **kw)
    self.P_pred = torch.empty(T, B, *((main_block, main_block) if main_block else _cov_shape(dim_err, packed_doubles)), **kw)
    self.P_pred_last = torch.empty(B, dim_err, dim_err, **kw) if main_block else None
    self.P_filt = torch.empty(T, B, *_cov_shape(dim_err, packed_doubles), **kw)
    self.t = torch.zeros(T, **kw)
    self.t_host = np.zeros(T)          # step times are collected on the host and uploaded once, before the backward pass
    self._t_pinned = None

  def sync_times(self):
    self.t.copy_(torch.as_tensor(self.t_host))

  def bytes(self):
    return sum(t.numel() * 8 for t in (self.x_pred, self.x_filt, self.P_pred, self.P_pred_last, self.P_filt, self.t) if t is not None)


class RaggedHistory:
  """Per-filter histories of a batch whose filters step on their own clocks (BatchedEKF.step_indexed with hist=).

  Slabs are [T, B, ...] in the full covariance layout (or, with `packed`, the packed one), like History, but row k of
  filter b is the k-th step THAT filter recorded: `n [B]` (int32) counts the rows each filter has used and `t [T, B]`
  holds their times.  A step of a filter whose T rows are used up is not recorded; `overflow` counts those steps.  All
  bookkeeping stays on the device (no host synchronisation per tick)."""

  def __init__(self, T, B, dim_x, dim_err, device, packed_doubles=0):
    assert T >= 1
    kw = dict(dtype=torch.float64, device=device)
    self.T, self.B = int(T), int(B)
    self.packed = bool(packed_doubles)
    self.x_pred = torch.empty(T, B, dim_x, **kw)
    self.x_filt = torch.empty(T, B, dim_x, **kw)
    self.P_pred = torch.empty(T, B, *_cov_shape(dim_err, packed_doubles), **kw)
    self.P_filt = torch.empty(T, B, *_cov_shape(dim_err, packed_doubles), **kw)
    self.t = torch.zeros(T, B, **kw)
    self.n = torch.zeros(B, dtype=torch.int32, device=device)
    self.overflow = torch.zeros((), dtype=torch.int64, device=device)

  def reserve(self, ids, t):
    """Hand each filter in `ids` (distinct, [m]) its next row, store its time t (scalar or [m]) there and count the row.
    Returns the rows ([m] int32, on the history's device), -1 for filters that had no row left (counted in overflow)."""
    dev = self.n.device
    ids = torch.as_tensor(ids, device=dev).to(torch.int64)
    t = torch.as_tensor(t, dtype=torch.float64, device=dev).expand(ids.shape[0])
    k = self.n[ids]
    full = k >= self.T
    kc = k.clamp(max=self.T - 1).to(torch.int64)
    self.t[kc, ids] = torch.where(full, self.t[kc, ids], t)
    self.n[ids] = k + (~full).to(torch.int32)
    self.overflow += full.sum()
    return torch.where(full, -1, k).to(torch.int32)

  def rewind(self, ids, rows):
    """Make row rows[e] the newest row of filter ids[e] (distinct): n[ids] = rows + 1.  The rows above are stale and are
    overwritten as the filter records again; the smoother never reads them.  `overflow` is left as it is."""
    dev = self.n.device
    ids = torch.as_tensor(ids, device=dev).to(torch.int64)
    self.n[ids] = torch.as_tensor(rows, device=dev).to(torch.int32) + 1

  def overflowed(self):
    """Steps not recorded because their filter's rows were used up (synchronises with the device)."""
    return int(self.overflow)

  def bytes(self):
    return sum(t.numel() * t.element_size() for t in (self.x_pred, self.x_filt, self.P_pred, self.P_filt, self.t, self.n))
