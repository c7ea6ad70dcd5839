"""Ragged observation scheduler: independent filters with DIFFERENT observation streams.

In the reference every filter instance is driven on the host, one `predict_and_update_batch(t, kind, z, R)`
call per observation (rednose/helpers/ekf_sym.py:464-531, ekf_sym.cc:83-117).  With a batch of filters the
streams interleave: at a given tick some filters see a gyro sample, some a position fix, some nothing.  The
scheduler buckets the observations of one tick by kind and issues ONE indexed fused launch per kind
(`<name>_batch_step_<kind>_idx`), keeping a per-filter clock on the device so each filter is predicted over
its own dt = t_obs - t_filter.  Filters without an observation in the tick are not touched.

RaggedScheduler drops (and counts) late observations (t_obs < t_filter); RewindingScheduler below keeps a per-filter ring
of checkpoints on the device and rewinds / fast-forwards like the single-filter drivers (ekf_sym.cc:125-156).  Both can
record what they apply into a per-filter history (a RaggedHistory) for RTS smoothing.
"""
from __future__ import annotations

import torch


class RaggedScheduler:
  def __init__(self, engine, history=None):
    """history: a RaggedHistory (engine.new_ragged_history(T)) that records every applied observation at its filter's
    next row, for a per-filter RTS pass afterwards (engine.rts_smooth(history)); dropped observations are not recorded."""
    self.e = engine
    self.history = history
    self.t_filter = torch.full((engine.B,), float("nan"), dtype=torch.float64, device=engine.device)
    self.dropped = 0

  def tick(self, filter_ids, t, kinds, z_by_kind, R_by_kind, ea_by_kind=None, augment=None):
    """One scheduling tick.

    filter_ids [n] int, t [n] float64 (or scalar), kinds [n] int: the observations of this tick, at most one per
    filter.  z_by_kind[k] is [n_k, m_k] in the order the entries of kind k appear in `filter_ids`;
    R_by_kind[k] is [m_k, m_k] (shared) or [n_k, m_k, m_k].  augment [n] bool (MSCKF), aligned with `filter_ids`: the
    flagged filters shift their clone window after their observation (a camera frame: predict_and_update_batch(...,
    augment=True)); a dropped observation neither steps nor shifts.  Returns {kind: (filter_ids_k, innovations_k)}.
    """
    dev = self.e.device
    fid = torch.as_tensor(filter_ids, device=dev).to(torch.int64)
    kinds = torch.as_tensor(kinds, device=dev)
    t = torch.as_tensor(t, dtype=torch.float64, device=dev).expand(fid.shape[0])
    aug = None if augment is None else torch.as_tensor(augment, device=dev).to(torch.bool).expand(fid.shape[0])
    out = {}
    for k in sorted(z_by_kind):
      sel = (kinds == k).nonzero(as_tuple=True)[0]
      if sel.numel() == 0:
        continue
      ids, tk = fid[sel], t[sel]
      ak = None if aug is None else aug[sel]
      tf = self.t_filter[ids]
      tf = torch.where(torch.isnan(tf), tk, tf)          # first observation initialises the clock (ekf_sym.py:502-503)
      dt = tk - tf
      ok = dt >= 0
      z = torch.as_tensor(z_by_kind[k], device=dev, dtype=torch.float64)
      R = torch.as_tensor(R_by_kind[k], device=dev, dtype=torch.float64)
      ea = None if not ea_by_kind or k not in ea_by_kind else torch.as_tensor(ea_by_kind[k], device=dev, dtype=torch.float64)
      if not bool(ok.all()):                              # too old: ignored, like ekf_sym.py:468-471
        self.dropped += int((~ok).sum())
        ids, tk, dt, z = ids[ok], tk[ok], dt[ok], z[ok]
        if R.ndim == 3:
          R = R[ok]
        if ea is not None:
          ea = ea[ok]
        if ak is not None:
          ak = ak[ok]
      rec = {} if self.history is None else dict(hist=self.history, t=tk)
      if ak is not None and bool(ak.any()):               # only then: engines without clone windows take no augment=
        rec["augment"] = ak
      y = self.e.step_indexed(k, ids.to(torch.int32), dt, z.clone(), R, ea, **rec)
      self.t_filter[ids] = tk
      out[k] = (ids, None if y is None else y[:, 0])
    return out


class RewindingScheduler(RaggedScheduler):
  """RaggedScheduler + the reference's out-of-order handling, per filter, on the device.

  Reference semantics (rednose/helpers/ekf_sym.py:418-482, C++ twin ekf_sym.cc:119-156): every applied observation
  checkpoints (filter time, x, P, the observation) into a buffer of the last REWIND_TO_KEEP = 512 entries
  (ekf_sym.py:447, ekf_sym.h:18).  An observation older than the filter rewinds to the last checkpoint at or before
  its time, is applied, and the observations rewound over are re-applied in order; it is ignored when the buffer is
  empty, when it predates the buffer, or when it is more than `max_rewind_age` older than the newest checkpoint.

  Here the buffer is a per-filter ring on the device: `depth` snapshots of x and P plus the observation cache
  (B * depth * (EDIM^2 + DIM + ...) doubles -- pick `depth` for the memory at hand; the reference's 512 is
  affordable for thousands of filters, not for a million).  A tick restores the rewinding filters with indexed copies,
  applies the new observations of all filters (one indexed fused launch per kind), then replays the rewound
  observations round by round (round r = the r-th rewound observation of every filter that has one, again one launch
  per kind).  No new kernel: the ring is plumbing around `<name>_batch_step_<kind>_idx`.

  With a history (a RaggedHistory of the engine's batch) every apply, replays included, records at its filter's next
  row, and the ring keeps no x / P snapshots: a checkpoint is the row its observation was recorded at, whose x_filt /
  P_filt are the state right after it, and a rewind restores the filter from that row (engine.restore_from_history) and
  makes it the filter's newest row.  The replay then records the rows after it again, so at the end of a stream each
  filter's rows are what RaggedScheduler would have recorded had the same observations arrived in time order:
  engine.rts_smooth(history) smooths them.  A late observation whose checkpoint was stepped while the filter's rows were
  used up cannot be restored: it is ignored and counted in `.unrecorded` (the history has overflowed anyway).

  MSCKF clone windows (tick(..., augment=)): each checkpoint keeps its observation's augment flag (`ring_aug`).  Without
  a history the snapshot is the state after the shift, as the reference's checkpoint is (ekf_sym.py:525-529).  With one,
  the checkpoint's row holds the estimate before the shift, so a rewind to a checkpoint whose observation shifted
  restores from the row and shifts again (engine.augment(ids)); the shift is a permutation, so that is the reference's
  checkpoint bit for bit.  Replays re-apply each observation's recorded shift.  This deliberately differs from the
  reference, whose drivers drop the flag on replay (ekf_sym.py keeps (t, kind, z, R, extra_args) in its cache, ekf_sym.cc:110
  replays with augment = false) and so leave the clone window one frame behind after a rewind over a camera frame.
  Re-applying it keeps the rows recorded under rewinds equal to those RaggedScheduler records for the same observations
  in time order.
  """

  def __init__(self, engine, zdims, depth=16, max_rewind_age=1.0, ea_dims=None, packed=False, history=None):
    """packed=True stores the covariance snapshots as their lower triangle (EDIM (EDIM + 1) / 2 doubles instead of EDIM^2:
    half the ring -- the reference's 512-deep ring then fits 100 000 live filters in one H100's HBM); a restored covariance
    is then exactly symmetric (upper := lower), which differs from the stored one by the kernels' last-bit asymmetry.

    history: a RaggedHistory of the engine's batch (engine.new_ragged_history(T), full or packed) to record into; the
    ring then holds history rows instead of snapshots, so `packed` does not apply."""
    if history is not None:
      if packed:
        raise ValueError("with a history the ring keeps no covariance snapshots: packed=True does not apply")
      if history.B != engine.B:
        raise ValueError(f"the history holds {history.B} filters, the engine {engine.B}")
    super().__init__(engine, history=history)
    B, dev = engine.B, engine.device
    self.N, self.max_rewind_age = int(depth), float(max_rewind_age)
    self.zdims = {int(k): int(m) for k, m in zdims.items()}
    self.ea_dims = {int(k): int(m) for k, m in (ea_dims or {}).items()}
    zmax, eamax = max(self.zdims.values()), max(list(self.ea_dims.values()) + [0])
    f64 = dict(dtype=torch.float64, device=dev)
    self.ring_t = torch.full((B, self.N), float("nan"), **f64)
    E = self.E = engine.dim_err if hasattr(engine, "dim_err") else engine.P.shape[1]
    self.packed = bool(packed)
    if history is not None:
      self.ring_row = torch.full((B, self.N), -1, dtype=torch.int32, device=dev)   # history row of each checkpoint
    else:
      self.ring_x = torch.zeros(B, self.N, engine.x.shape[1], **f64)
      if self.packed:
        tr = torch.tril_indices(E, E, device=dev)
        self._tri_r, self._tri_c = tr[0], tr[1]
        ii, jj = torch.meshgrid(torch.arange(E, device=dev), torch.arange(E, device=dev), indexing="ij")
        hi, lo = torch.maximum(ii, jj), torch.minimum(ii, jj)
        self._unpack = (hi * (hi + 1) // 2 + lo).reshape(-1)      # full (i, j) -> packed index of (max, min)
        self.ring_P = torch.zeros(B, self.N, E * (E + 1) // 2, **f64)
      else:
        self.ring_P = torch.zeros(B, self.N, E, E, **f64)
    self.ring_kind = torch.zeros(B, self.N, dtype=torch.int64, device=dev)
    self.ring_aug = torch.zeros(B, self.N, dtype=torch.bool, device=dev)     # the observation shifted the clone window
    self._augmenting = False                       # a tick has passed augment=: rewinds and replays look at ring_aug
    self.ring_z = torch.zeros(B, self.N, zmax, **f64)
    self.ring_R = torch.zeros(B, self.N, zmax, zmax, **f64)
    self.ring_ea = torch.zeros(B, self.N, eamax, **f64) if eamax else None
    self.head = torch.zeros(B, dtype=torch.int64, device=dev)   # physical slot of the oldest checkpoint
    self.cnt = torch.zeros(B, dtype=torch.int64, device=dev)    # checkpoints held
    self.rewinds = 0                                             # observations that arrived late and were rewound for
    self.replayed = 0                                            # observations re-applied during fast-forward
    self.unrecorded = 0                                          # late observations whose checkpoint has no history row

  # -- ring -----------------------------------------------------------------------------------------------------------
  # rows of P through the engine's row accessors when it has them (BatchedEKF: touches only those filters of its
  # resident covariance), else by indexing a plain P tensor
  def _get_P(self, ids):
    return self.e.get_P_rows(ids) if hasattr(self.e, "get_P_rows") else self.e.P[ids]

  def _set_P(self, ids, P):
    if hasattr(self.e, "set_P_rows"):
      self.e.set_P_rows(ids, P)
    else:
      self.e.P[ids] = P

  def _push(self, ids, t, kind, z, R, ea, rows, aug):
    """Checkpoint the CURRENT state of filters `ids` together with the observation just applied (ekf_sym.py:437-450);
    with a history the state is the one recorded at `rows` (before the shift of the entries flagged in `aug`)."""
    full = self.cnt[ids] == self.N
    pos = torch.where(full, self.head[ids], (self.head[ids] + self.cnt[ids]) % self.N)
    m = z.shape[-1]
    self.ring_t[ids, pos] = t
    if self.history is not None:
      self.ring_row[ids, pos] = rows
    else:
      self.ring_x[ids, pos] = self.e.x[ids]
      P = self._get_P(ids)
      self.ring_P[ids, pos] = P[:, self._tri_r, self._tri_c] if self.packed else P
    self.ring_kind[ids, pos] = kind
    self.ring_aug[ids, pos] = False if aug is None else aug
    self.ring_z[ids, pos, :m] = z
    self.ring_R[ids, pos, :m, :m] = R
    if ea is not None and self.ring_ea is not None:
      self.ring_ea[ids, pos, :ea.shape[-1]] = ea
    self.head[ids] = torch.where(full, (self.head[ids] + 1) % self.N, self.head[ids])
    self.cnt[ids] = torch.where(full, self.cnt[ids], self.cnt[ids] + 1)

  def _apply(self, ids, t, kinds, z, R, ea, aug, want_y):
    """Predict to t + update (+ clone-window shift where `aug`, [n] bool or None) + checkpoint for entries (ids, t, kinds)
    with padded z / R / ea rows: one launch per kind (and kernel)."""
    out = {}
    for k in torch.unique(kinds).tolist():
      sel = (kinds == k).nonzero(as_tuple=True)[0]
      m = self.zdims[int(k)]
      idk, tk = ids[sel], t[sel]
      zk = z[sel, :m].contiguous()
      Rk = R[sel, :m, :m].contiguous()
      eak = ea[sel, :self.ea_dims[int(k)]].contiguous() if (ea is not None and int(k) in self.ea_dims) else None
      tf = self.t_filter[idk]
      tf = torch.where(torch.isnan(tf), tk, tf)            # first observation initialises the clock (ekf_sym.py:502-503)
      rows, rec = None, {}
      if self.history is not None:                         # the row reserve() hands out; it saturates n, so read it first
        n = self.history.n[idk]
        rows, rec = torch.where(n < self.history.T, n, -1), dict(hist=self.history, t=tk)
      ak = None if aug is None else aug[sel]
      if ak is not None and bool(ak.any()):                # only then: engines without clone windows take no augment=
        rec["augment"] = ak
      y = self.e.step_indexed(int(k), idk.to(torch.int32), (tk - tf).contiguous(), zk.clone(), Rk, eak, **rec)
      self.t_filter[idk] = tk
      self._push(idk, tk, int(k), zk, Rk, eak, rows, ak)
      if want_y:
        out[int(k)] = (idk, None if y is None else y[:, 0])
    return out

  # -- one tick ---------------------------------------------------------------------------------------------------------
  def tick(self, filter_ids, t, kinds, z_by_kind, R_by_kind, ea_by_kind=None, augment=None):
    """Same arguments and return value as RaggedScheduler.tick; late observations rewind instead of being dropped
    (those that the reference would ignore are counted in `.dropped` and absent from the result).  A late observation
    flagged in `augment` shifts when it is applied, and every observation replayed after it shifts again if it did."""
    dev, N = self.e.device, self.N
    fid = torch.as_tensor(filter_ids, device=dev).to(torch.int64)
    kinds = torch.as_tensor(kinds, device=dev).to(torch.int64)
    n = int(fid.shape[0])
    t = torch.as_tensor(t, dtype=torch.float64, device=dev).expand(n).contiguous()
    aug = None if augment is None else torch.as_tensor(augment, device=dev).to(torch.bool).expand(n).contiguous()
    self._augmenting |= aug is not None
    zmax = self.ring_z.shape[-1]
    z = torch.zeros(n, zmax, dtype=torch.float64, device=dev)
    R = torch.zeros(n, zmax, zmax, dtype=torch.float64, device=dev)
    ea = torch.zeros(n, self.ring_ea.shape[-1], dtype=torch.float64, device=dev) if self.ring_ea is not None else None
    for k in z_by_kind:                                   # scatter the per-kind blocks into per-entry padded rows
      sel = (kinds == int(k)).nonzero(as_tuple=True)[0]
      if sel.numel() == 0:
        continue
      m = self.zdims[int(k)]
      z[sel, :m] = torch.as_tensor(z_by_kind[k], dtype=torch.float64, device=dev).reshape(-1, m)
      Rk = torch.as_tensor(R_by_kind[k], dtype=torch.float64, device=dev)
      R[sel, :m, :m] = Rk if Rk.ndim == 3 else Rk.expand(sel.numel(), m, m)
      if ea is not None and ea_by_kind and k in ea_by_kind:
        eak = torch.as_tensor(ea_by_kind[k], dtype=torch.float64, device=dev)
        ea[sel, :eak.shape[-1]] = eak

    tf = self.t_filter[fid]
    late = (~torch.isnan(tf)) & (t < tf)
    keep = torch.ones(n, dtype=torch.bool, device=dev)
    replay = None
    if bool(late.any()):
      li = late.nonzero(as_tuple=True)[0]
      lf, lt = fid[li], t[li]
      ar = torch.arange(N, device=dev)
      phys = (self.head[lf][:, None] + ar[None, :]) % N                  # logical -> physical slots, oldest first
      tl = self.ring_t[lf].gather(1, phys)
      cnt = self.cnt[lf]
      valid = ar[None, :] < cnt[:, None]
      newest = tl.gather(1, (cnt - 1).clamp(min=0)[:, None])[:, 0]
      too_old = (cnt == 0) | (lt < tl[:, 0]) | (lt < newest - self.max_rewind_age)   # ekf_sym.py:469
      self.dropped += int(too_old.sum())
      keep[li[too_old]] = False
      ok = ~too_old
      if bool(ok.any()):
        li, lf, lt, phys, tl, cnt, valid = li[ok], lf[ok], lt[ok], phys[ok], tl[ok], cnt[ok], valid[ok]
        idx = ((tl <= lt[:, None]) & valid).sum(1)                       # bisect_right(rewind_t, t), >= 1 here
        src = phys.gather(1, (idx - 1)[:, None])[:, 0]
        if self.history is not None:
          row = self.ring_row[lf, src]
          lost = row < 0                        # stepped while the filter's rows were used up: nothing to restore from
          self.unrecorded += int(lost.sum())
          keep[li[lost]] = False
          lf, phys, cnt, idx, src, row = (v[~lost] for v in (lf, phys, cnt, idx, src, row))
        if lf.numel():
          if self.history is not None:
            self.e.restore_from_history(self.history, lf, row)           # ekf_sym.py:425-427, from the recorded row
            self.history.rewind(lf, row)
            shifted = self.ring_aug[lf, src] if self._augmenting else None   # the row holds the estimate before the shift
            if shifted is not None and bool(shifted.any()):
              self.e.augment(lf[shifted])
          else:
            self.e.x[lf] = self.ring_x[lf, src]                          # ekf_sym.py:425-427
            if self.packed:
              E = self.E
              self._set_P(lf, self.ring_P[lf, src][:, self._unpack].reshape(-1, E, E))
            else:
              self._set_P(lf, self.ring_P[lf, src])
          self.t_filter[lf] = self.ring_t[lf, src]
          # the observations rewound over (logical idx .. cnt-1), copied out before the ring is reused
          n_rep = cnt - idx
          lp = (idx[:, None] + ar[None, :]).clamp(max=N - 1)             # logical positions idx, idx+1, ...
          pp = phys.gather(1, lp)
          replay = dict(f=lf, n=n_rep, t=self.ring_t[lf[:, None], pp], kind=self.ring_kind[lf[:, None], pp],
                        z=self.ring_z[lf[:, None], pp], R=self.ring_R[lf[:, None], pp],
                        ea=None if self.ring_ea is None else self.ring_ea[lf[:, None], pp], aug=self.ring_aug[lf[:, None], pp] if self._augmenting else None)
          self.cnt[lf] = idx                                             # throw away the old future (ekf_sym.py:432-435)
          self.rewinds += int(lf.shape[0])

    out = {}
    if bool(keep.any()):
      ks = keep.nonzero(as_tuple=True)[0]
      out = self._apply(fid[ks], t[ks], kinds[ks], z[ks], R[ks], None if ea is None else ea[ks], None if aug is None else aug[ks], True)
    if replay is not None:                                               # fast-forward (ekf_sym.py:479-480)
      for r in range(int(replay["n"].max())):
        sel = (replay["n"] > r).nonzero(as_tuple=True)[0]
        self._apply(replay["f"][sel], replay["t"][sel, r].contiguous(), replay["kind"][sel, r], replay["z"][sel, r],
                    replay["R"][sel, r], None if replay["ea"] is None else replay["ea"][sel, r],
                    None if replay["aug"] is None else replay["aug"][sel, r], False)
        self.replayed += int(sel.shape[0])
    return out
