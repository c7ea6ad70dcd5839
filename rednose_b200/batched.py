"""Batched EKF engine: B independent filter instances resident in H100 HBM.

This is the batched counterpart of the reference's per-instance driver
(rednose/helpers/ekf_sym.cc:158-219 / ekf_sym.py:484-531): the state ``x[B, DIM]`` and
covariance ``P[B, EDIM, EDIM]`` (float64, row-major, AoS per filter) live on the device as
torch tensors -- torch is only the allocator / stream provider -- and every step is ONE launch of
the generated library's fused ``<name>_batch_step_<kind>`` kernel through its C-ABI.

Semantics follow the C++ driver: predict(dt) -> [normalise quaternions] -> update(kind) ->
[normalise] (ekf_sym.cc:162,207,213); the innovation overwrites ``z`` (ekf_c.c:120).
"""
from __future__ import annotations

import numpy as np
import torch

from rednose_b200.loader import load_code, raise_on_cuda_error

NORM_AFTER_PREDICT = 1
NORM_AFTER_UPDATE = 2
Q_IS_DIAGONAL = 4
SHARED_R = 8
AUGMENT = 16   # fused clone-window shift (CTA kernel only)


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
    self.P = P0.contiguous().clone()
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
    self._zdim = {}
    self.launches = 0  # kernels launched through this object (bench.py reports it)
    for g, v in (global_vars or {}).items():
      getattr(self._lib, f"{name}_set_{g}")(float(v))

  # ----------------------------------------------------------------- helpers ---
  def _p(self, t):
    return self._ffi.cast("double *", t.data_ptr()) if t is not None else self._ffi.NULL

  def _cp(self, t):
    return self._ffi.cast("const double *", t.data_ptr()) if t is not None else self._ffi.NULL

  def _stream(self):
    return self._ffi.cast("void *", torch.cuda.current_stream(self.device).cuda_stream)

  def _check(self, what):
    raise_on_cuda_error(self._lib, self.name, what)

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
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_predict")(
        self._p(self.x), self._p(self.P), self._cp(self.Q), dt_ptr, dt_s, self.B, self._quat, self._nquat, self.flags,
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
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_update_{kind}")(
        self._p(self.x), self._p(self.P), self._p(z), self._cp(R), self._cp(ea), n_obs, self.B,
        self._quat, self._nquat, flags, self._p(hx), self._p(hP), self._stream())
    self.launches += 1
    self._check(f"batch_update_{kind}")
    return z

  def step_indexed(self, kind, idx, dt, z, R, ea=None):
    """Fused predict + update of `kind` for the filters listed in `idx` only ([n] int32, device): entry e uses
    z[e], R[e] (or one shared R), dt[e] and works on filter idx[e].  Filters not listed are untouched.  This is the
    building block of the ragged scheduler (per-tick kind buckets)."""
    idx = idx.to(device=self.device, dtype=torch.int32).contiguous()
    n = int(idx.shape[0])
    if n == 0:
      return None
    z = _as_device(z, self.device)
    if z.ndim == 2:
      z = z.unsqueeze(1)
    R = _as_device(R, self.device)
    flags = self.flags
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
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_step_{kind}_idx")(
        self._p(self.x), self._p(self.P), self._cp(self.Q), dt_ptr, dt_s, self._p(z), self._cp(R), self._cp(ea),
        z.shape[1], n, self._quat, self._nquat, flags, self._ffi.NULL, self._ffi.NULL, self._ffi.NULL, self._ffi.NULL,
        self._ffi.cast("const int *", idx.data_ptr()), self._stream())
    self.launches += 1
    self._check(f"batch_step_{kind}_idx")
    return z

  def step(self, kind, dt, z, R, ea=None, hist_pred=None, hist_filt=None, augment=False):
    """Fused predict(dt) + update(kind): one kernel launch, P read and written once.  augment=True also shifts the MSCKF
    clone window (predict_and_update_batch(..., augment=True), ekf_sym.py:527-528): inside the same launch for filters on
    the CTA-per-filter kernel (EDIM > 32), as a second launch otherwise."""
    keep, dt_ptr, dt_s = self._dt_args(dt)
    z, R, ea, n_obs, flags = self._obs_args(z, R, ea)
    fused_aug = bool(augment) and self.dim_err > 32
    if fused_aug:
      flags |= AUGMENT
    hxp, hPp = (hist_pred if hist_pred is not None else (None, None))
    hxf, hPf = (hist_filt if hist_filt is not None else (None, None))
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_step_{kind}")(
        self._p(self.x), self._p(self.P), self._cp(self.Q), dt_ptr, dt_s, self._p(z), self._cp(R), self._cp(ea),
        n_obs, self.B, self._quat, self._nquat, flags, self._p(hxp), self._p(hPp), self._p(hxf), self._p(hPf),
        self._stream())
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
    attribute setup does not land inside the capture."""
    side = torch.cuda.Stream(self.device)
    side.wait_stream(torch.cuda.current_stream(self.device))
    with torch.cuda.stream(side):
      for _ in range(max(1, int(warmup))):
        fn()
    torch.cuda.current_stream(self.device).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
      fn()
    return g

  # -------------------------------------------------------------- host access ---
  def state(self):
    return self.x.cpu().numpy()

  def covs(self):
    return self.P.cpu().numpy()

  def init_state(self, x, P, filter_time=None):
    self.x.copy_(_as_device(x, self.device).expand_as(self.x))
    self.P.copy_(_as_device(P, self.device).expand_as(self.P))
    self.filter_time = filter_time

  def maha_dist(self, kind, z, R, ea=None):
    """Mahalanobis distance y^T (H P H^T + R)^-1 y of one observation per filter, without touching the state
    (the quantity EKF_sym.maha_test thresholds, ekf_sym.py:626-649).  Returns a [B] device tensor."""
    z = _as_device(z, self.device).reshape(self.B, -1).contiguous()
    R = _as_device(R, self.device)
    flags = SHARED_R if R.ndim == 2 else 0
    ea = _as_device(ea, self.device) if ea is not None else None
    out = torch.empty(self.B, dtype=torch.float64, device=self.device)
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_maha_{kind}")(
        self._cp(self.x), self._cp(self.P), self._cp(z), self._cp(R), self._cp(ea), self.B, flags, self._p(out), self._stream())
    self.launches += 1
    self._check(f"batch_maha_{kind}")
    return out

  def maha_test(self, kind, z, R, ea=None, maha_thresh=0.95):
    """True where the observation passes the chi-square gate at `maha_thresh` (batched EKF_sym.maha_test)."""
    from rednose_b200.chi2 import chi2_ppf
    d = self.maha_dist(kind, z, R, ea)
    return d <= float(chi2_ppf(maha_thresh, z.shape[-1] if hasattr(z, "shape") else len(z[0])))

  def augment(self):
    """MSCKF clone window shift for the whole batch (ekf_sym.py:365-391), one launch."""
    with torch.cuda.device(self.device):
      getattr(self._lib, f"{self.name}_batch_augment")(self._p(self.x), self._p(self.P), self.B, self._stream())
    self.launches += 1
    self._check("batch_augment")

  # ------------------------------------------------------- history + smoothing ---
  def new_history(self, T):
    """Device slabs for a T-step history, time-major: what the reference keeps as the list of
    9-tuples returned by predict_and_update_batch (ekf_sym.py:531): x_{k|k-1}, x_{k|k}, P_{k|k-1}, P_{k|k}, t."""
    return History(T, self.B, self.dim_x, self.dim_err, self.device)

  def step_recorded(self, hist, kind, t, z, R, ea=None):
    """predict_and_update_batch that also appends this step to `hist` (the kernel writes the slabs itself)."""
    k = hist.n
    assert k < hist.T, "history is full"
    if self.filter_time is None:
      self.filter_time = t
    dt = t - self.filter_time
    y = self.step(kind, dt, z, R, ea, hist_pred=(hist.x_pred[k], hist.P_pred[k]), hist_filt=(hist.x_filt[k], hist.P_filt[k]))
    self.filter_time = t
    hist.t_host[k] = float(t)
    hist.n += 1
    return y

  def rts_smooth(self, hist, norm_quats=False, quaternion_idxs=(3,), in_place=False, out=None, terminal=None, k0=0):
    """Batched RTS backward pass over a recorded history (ekf_sym.py:651-690, one launch for all filters).

    Returns (xs [T, B, DIM], Ps [T, B, EDIM, EDIM]) on the device.  `norm_quats` normalises the quaternion(s)
    at `quaternion_idxs` the way the reference normalises its hard-coded slice 3:7.

    `terminal=(x [B, DIM], P [B, EDIM, EDIM])` smooths one SEGMENT of a longer history (steps k0 .. k0 + T - 2): the
    recursion starts from that smoothed estimate of step k0 + T - 1, whose history entry (the last one recorded) only
    contributes its predicted state; its row of xs / Ps is not written.
    """
    T = hist.n
    assert T >= 1
    hist.sync_times()
    if out is not None:
      xs, Ps = out                      # caller-provided [T, B, DIM] / [T, B, EDIM, EDIM] buffers
    else:
      xs = hist.x_filt if in_place else torch.empty_like(hist.x_filt)
      Ps = hist.P_filt if in_place else torch.empty_like(hist.P_filt)
    qi = self._ffi.new("int[]", list(quaternion_idxs) or [0])
    with torch.cuda.device(self.device):
      if terminal is None and not k0:
        getattr(self._lib, f"{self.name}_batch_rts")(
          self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t), 0,
          self._p(xs), self._p(Ps), T, self.B, qi, len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0, self._stream())
      else:
        xt, Pt = terminal if terminal is not None else (None, None)   # the LAST segment of a history has k0 > 0 but no terminal
        assert xt is None or (xt.is_contiguous() and Pt.is_contiguous() and xt.shape == (self.B, self.dim_x) and Pt.shape == (self.B, self.dim_err, self.dim_err))
        getattr(self._lib, f"{self.name}_batch_rts_segment")(
          self._cp(hist.x_pred), self._cp(hist.P_pred), self._cp(hist.x_filt), self._cp(hist.P_filt), self._cp(hist.t), 0,
          self._p(xs), self._p(Ps), T, self.B, qi, len(quaternion_idxs) if norm_quats else 0, 1 if norm_quats else 0,
          self._cp(xt), self._cp(Pt), int(k0), self._stream())
    self.launches += 1
    self._check("batch_rts")
    return xs[:T], Ps[:T]


class History:
  """Time-major device buffers of a forward pass, consumed by the RTS kernel."""

  def __init__(self, T, B, dim_x, dim_err, device):
    kw = dict(dtype=torch.float64, device=device)
    self.T, self.B, self.n = T, B, 0
    self.x_pred = torch.empty(T, B, dim_x, **kw)
    self.x_filt = torch.empty(T, B, dim_x, **kw)
    self.P_pred = torch.empty(T, B, dim_err, dim_err, **kw)
    self.P_filt = torch.empty(T, B, dim_err, dim_err, **kw)
    self.t = torch.zeros(T, **kw)
    self.t_host = np.zeros(T)          # step times are collected on the host and uploaded once, before the backward pass
    self._t_pinned = None

  def sync_times(self):
    self.t.copy_(torch.as_tensor(self.t_host))

  def bytes(self):
    return sum(t.numel() * 8 for t in (self.x_pred, self.x_filt, self.P_pred, self.P_filt, self.t))
