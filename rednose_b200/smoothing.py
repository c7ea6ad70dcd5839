"""Forward filter + RTS smoother over long histories, tiled over filters.

The smoother needs x_{k|k-1}, x_{k|k}, P_{k|k-1}, P_{k|k} of every step (rednose/helpers/ekf_sym.py:651-690
walks the list of tuples returned by predict_and_update_batch): 2*EDIM^2 + 2*DIM + 1 doubles per filter-step,
8.1 kB for live_kf.  BASELINE.json config 4 (1M filters x 10k steps) would be 81 TB, so the batch is cut into
TILES of filters whose whole history fits the HBM budget; each tile runs forward-store-then-backward-consume and
hands its smoothed track to a sink before the next tile reuses the buffers (SURVEY.md section 7, hard part 3).
Tiles are independent, so multi-GPU use is: shard the filters over ranks first, tile within a rank.

Both smoothers take ``packed_history=True`` for filters with a packed covariance layout (BatchedEKF.new_history(T,
packed=True)): the history then stores each covariance as its packed lower block triangle (4 592 instead of 8 112 bytes
per live filter-step, so 1.77x the filters per tile), and the sink receives the smoothed covariances packed,
[..., packed doubles]; ``unpack_P`` turns them into full matrices.

For an MSCKF (EDIM > 32), ``main_pred=True`` keeps only the main block of each predicted covariance in the history
(BatchedEKF.new_history(T, main_pred=True)): the smoother reads nothing else of it.  A msckf step then takes 59 152
instead of 109 072 bytes; the smoothed covariances stay full and bit-identical.

``obs_fn(k, lo, hi)`` returns ``(t, kind, z, R)`` or ``(t, kind, z, R, ea, augment)``: ``ea`` are the extra arguments of
the kind (the triangulated landmark of a feature-track kind, [hi - lo, EADIM] or None) and ``augment`` shifts the MSCKF
clone window after the update (predict_and_update_batch(..., augment=True)).
"""
from __future__ import annotations

import torch

from rednose_b200.batched import MAIN_PRED_REFUSED, PACKED_REFUSED, BatchedEKF, main_pred_doubles, packed_P_doubles


def history_bytes_per_filter(dim_x, dim_err, T, smoothed_in_place=True, packed_doubles=0, main_pred_doubles=0):
  """Bytes of a T-step history of one filter; packed_doubles > 0: its covariances are in the packed layout of that many
  doubles (BatchedEKF.new_history(T, packed=True)); main_pred_doubles > 0: its predicted covariances keep only their
  main block of that many doubles, plus one full copy of the newest prediction (BatchedEKF.new_history(T,
  main_pred=True))."""
  cov = packed_doubles or dim_err * dim_err
  per_step = cov + (main_pred_doubles or cov) + 2 * dim_x
  if not smoothed_in_place:
    per_step += cov + dim_x
  return 8 * per_step * T + (8 * dim_err * dim_err if main_pred_doubles else 0)


def _history_doubles(folder, name, packed_history):
  if not packed_history:
    return 0
  pd = packed_P_doubles(folder, name)
  if not pd:
    raise ValueError(f"filter '{name}': packed histories are not available: {PACKED_REFUSED}")
  return pd


def _main_pred_doubles(folder, name, main_pred, packed_history):
  if not main_pred:
    return 0
  if packed_history:
    raise ValueError("a main-block prediction history is in the full covariance layout: packed_history does not apply")
  md = main_pred_doubles(folder, name)
  if not md:
    raise ValueError(f"filter '{name}': {MAIN_PRED_REFUSED}")
  return md


def _observation(obs_fn, k, lo, hi):
  """(t, kind, z, R, ea, augment) of step k: obs_fn returns the first four, or all six."""
  obs = obs_fn(k, lo, hi)
  return tuple(obs) if len(obs) == 6 else (*obs, None, False)


class TiledSmoother:
  """Forward filter + RTS smoother, one tile of filters with its whole history at a time.  With packed_history=True the
  history and the smoothed covariances the sink receives are packed [T, n, packed doubles]; unpack_P(Ps) gives them full."""

  def __init__(self, folder, name, Q, dim_x, dim_err, quaternion_idxs=(), device="cuda", hbm_budget_bytes=60 << 30, tile=None,
               packed_history=False, main_pred=False):
    self.folder, self.name, self.Q = folder, name, Q
    self.dim_x, self.dim_err = dim_x, dim_err
    self.quat = tuple(quaternion_idxs)
    self.device = torch.device(device)
    self.budget = hbm_budget_bytes
    self.tile = tile
    self.main_pred_doubles = _main_pred_doubles(folder, name, main_pred, packed_history)
    self.packed_doubles = _history_doubles(folder, name, packed_history)
    self._engine = None
    self._hist = None

  def tile_size(self, T):
    if self.tile:
      return self.tile
    per = history_bytes_per_filter(self.dim_x, self.dim_err, T, packed_doubles=self.packed_doubles,
                                   main_pred_doubles=self.main_pred_doubles) + 8 * (self.dim_err**2 + self.dim_x)
    return max(1, int(self.budget // per))

  def unpack_P(self, Ps):
    """Full [..., EDIM, EDIM] covariances of packed smoothed ones (the sink's Ps with packed_history=True)."""
    return self._engine.unpack_P(Ps)

  def run(self, x0, P0, T, obs_fn, sink, norm_quats=False, t0=0.0, passes=1):
    """x0 [B, DIM], P0 [B, EDIM, EDIM] (host or device).  obs_fn(k, lo, hi) -> (t, kind, z [hi-lo, m], R) or (t, kind, z,
    R, ea, augment) gives the observation of step k for filters lo..hi.  sink(lo, hi, xs [T, n, DIM], Ps [T, n, EDIM, EDIM], or [T, n, packed
    doubles] with packed_history) receives device views that are only valid during the call.  Returns the number of
    tiles.

    passes > 1: "multiple forward and backwards passes of the data" (reference README.md:41-45) -- each further pass
    restarts the forward filter of the tile from the previous pass's smoothed estimate at the first step
    (x_{0|N}, P_{0|N}), which removes the dependence on a poor initialisation; the sink sees the last pass."""
    B = x0.shape[0]
    n_tile = min(self.tile_size(T), B)
    tiles = 0
    for lo in range(0, B, n_tile):
      hi = min(lo + n_tile, B)
      n = hi - lo
      if self._engine is None or self._engine.B != n:
        self._engine = BatchedEKF(self.folder, self.name, self.Q, x0[lo:hi], P0[lo:hi], device=self.device, quaternion_idxs=self.quat)
        self._hist = (self._engine.new_history(T, packed=bool(self.packed_doubles), main_pred=bool(self.main_pred_doubles))
                      if (self._hist is None or self._hist.B != n or self._hist.T != T) else self._hist)
      else:
        self._engine.init_state(x0[lo:hi], P0[lo:hi], None)
      eng, hist = self._engine, self._hist
      for p in range(max(1, int(passes))):
        if p > 0:   # the smoothed slabs alias the history buffers the next forward pass overwrites: copy step 0 out first
          eng.init_state(xs[0].clone(), eng.unpack_P(Ps[0]) if self.packed_doubles else Ps[0].clone(), None)
        hist.n = 0
        eng.filter_time = t0
        for k in range(T):
          t, kind, z, R, ea, aug = _observation(obs_fn, k, lo, hi)
          eng.step_recorded(hist, kind, t, z, R, ea, augment=aug)
        xs, Ps = eng.rts_smooth(hist, norm_quats=norm_quats, quaternion_idxs=self.quat or (3,), in_place=True)
      sink(lo, hi, xs, Ps)
      tiles += 1
    return tiles


class CheckpointedSmoother:
  """Forward filter + RTS smoother over histories too long to store, for LARGE tiles of filters.

  Tiling over filters alone (TiledSmoother) trades history length for batch size: BASELINE.json config 4 (10 000 steps)
  would leave ~1 500 filters per launch, which cannot fill 132 SMs.  Here only a CHECKPOINT (x, P: 4 kB per live filter)
  is kept every `segment` steps of a first forward pass; the backward sweep then visits the segments last to first,
  re-runs the forward filter of one segment from its checkpoint WITH history (segment + 1 steps: the extra one is the
  first step of the segment behind it, whose predicted state the recursion needs) and smooths it starting from the
  smoothed estimate handed over by that segment (`<name>_batch_rts_segment`).  Memory per filter is
  T / segment checkpoints + one segment of history instead of T steps of history, so ~100k live filters fit one tile;
  the price is a second forward pass.  The kernels are deterministic, so the result is bit-identical to smoothing the
  whole history at once (tests/test_parity_gpu.py::test_checkpointed_smoother_equals_full_history).

  packed_history=True: the segment history, the smoothed estimate handed between segments and the covariances the sink
  receives are packed ([..., packed doubles]; unpack_P gives them full); the checkpoints stay full.

  main_pred=True (EDIM > 32): the segment history keeps the main block of each predicted covariance only (see the module
  docstring); checkpoints, the estimate handed between segments and the sink's covariances stay full."""

  def __init__(self, folder, name, Q, dim_x, dim_err, quaternion_idxs=(), device="cuda", hbm_budget_bytes=60 << 30, segment=64, tile=None,
               packed_history=False, main_pred=False):
    self.folder, self.name, self.Q = folder, name, Q
    self.dim_x, self.dim_err = dim_x, dim_err
    self.quat = tuple(quaternion_idxs)
    self.device = torch.device(device)
    self.budget, self.segment, self.tile = hbm_budget_bytes, int(segment), tile
    self.main_pred_doubles = _main_pred_doubles(folder, name, main_pred, packed_history)
    self.packed_doubles = _history_doubles(folder, name, packed_history)
    self._engine = self._hist = self._ck = None
    self.stats = {}

  def bytes_per_filter(self, T):
    nseg = (T + self.segment - 1) // self.segment
    state = 8 * (self.dim_err**2 + self.dim_x)
    return nseg * state + history_bytes_per_filter(self.dim_x, self.dim_err, self.segment + 1, packed_doubles=self.packed_doubles,
                                                   main_pred_doubles=self.main_pred_doubles) + 3 * state

  def unpack_P(self, Ps):
    """Full [..., EDIM, EDIM] covariances of packed smoothed ones (the sink's Ps with packed_history=True)."""
    return self._engine.unpack_P(Ps)

  def tile_size(self, T):
    return self.tile or max(1, int(self.budget // self.bytes_per_filter(T)))

  def plan(self, B, T):
    """(filters per tile, tiles): the batch is cut into EQUAL tiles no larger than tile_size(T), so that one engine and
    one set of history / checkpoint buffers serve every tile."""
    cap = min(self.tile_size(T), B)
    ntiles = (B + cap - 1) // cap
    return (B + ntiles - 1) // ntiles, ntiles

  def run(self, x0, P0, T, obs_fn, sink, norm_quats=False, t0=0.0):
    """obs_fn(k, lo, hi) -> (t, kind, z, R) or (t, kind, z, R, ea, augment) must return the SAME observation every time it
    is asked for step k (each step is filtered twice) in a buffer the kernel may overwrite.  sink(lo, hi, k0, xs [n, tile, DIM], Ps [n, tile, EDIM, EDIM])
    receives the smoothed steps k0 .. k0 + n - 1 of filters lo..hi (segments arrive last to first; views valid during
    the call only; Ps [n, tile, packed doubles] with packed_history).  Returns the number of tiles."""
    B, S = x0.shape[0], self.segment
    n_tile, _ = self.plan(B, T)
    nseg = (T + S - 1) // S
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fwd_ms = refwd_ms = bwd_ms = 0.0
    tiles = 0
    for lo in range(0, B, n_tile):
      hi = min(lo + n_tile, B)
      n = hi - lo
      if self._engine is None or self._engine.B != n:
        self._engine = self._hist = self._ck = self._term = None   # release the previous tile's buffers before allocating
        self._engine = BatchedEKF(self.folder, self.name, self.Q, x0[lo:hi], P0[lo:hi], device=self.device, quaternion_idxs=self.quat)
        self._hist = self._engine.new_history(S + 1, packed=bool(self.packed_doubles), main_pred=bool(self.main_pred_doubles))
        self._ck = (torch.empty(nseg, n, self.dim_x, dtype=torch.float64, device=self.device),
                    torch.empty(nseg, n, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device))
        self._term = (torch.empty(n, self.dim_x, dtype=torch.float64, device=self.device),
                      torch.empty(n, *self._hist.P_filt.shape[2:], dtype=torch.float64, device=self.device))
      else:
        self._engine.init_state(x0[lo:hi], P0[lo:hi], None)
      eng, hist, (ck_x, ck_P), (tx, tP) = self._engine, self._hist, self._ck, self._term
      if ck_x.shape[0] != nseg:
        ck_x = torch.empty(nseg, n, self.dim_x, dtype=torch.float64, device=self.device)
        ck_P = torch.empty(nseg, n, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device)
        self._ck = (ck_x, ck_P)
      ck_t = [t0] * nseg
      # ---- pass 1: forward without history, checkpoint before the first step of every segment ----
      eng.filter_time = t0
      ev[0].record()
      for k in range(T):
        if k % S == 0:
          ck_x[k // S].copy_(eng.x); ck_P[k // S].copy_(eng.P); ck_t[k // S] = eng.filter_time
        t, kind, z, R, ea, aug = _observation(obs_fn, k, lo, hi)
        eng.predict_and_update_batch(t, kind, z, R, ea, augment=aug)
      ev[1].record(); ev[1].synchronize(); fwd_ms += ev[0].elapsed_time(ev[1])
      # ---- pass 2: segments last to first: forward with history from the checkpoint, then backward ----
      have_term = False
      for j in range(nseg - 1, -1, -1):
        k0 = j * S
        k1 = min(k0 + S + 1, T)          # one step past the segment unless it is the last
        eng.x.copy_(ck_x[j]); eng.P.copy_(ck_P[j]); eng.filter_time = ck_t[j]
        hist.n = 0
        ev[0].record()
        for k in range(k0, k1):
          t, kind, z, R, ea, aug = _observation(obs_fn, k, lo, hi)
          eng.step_recorded(hist, kind, t, z, R, ea, augment=aug)
        ev[1].record(); ev[1].synchronize(); refwd_ms += ev[0].elapsed_time(ev[1])
        ev[0].record()
        xs, Ps = eng.rts_smooth(hist, norm_quats=norm_quats, quaternion_idxs=self.quat or (3,), in_place=True,
                                terminal=(tx, tP) if have_term else None, k0=k0)
        ev[1].record(); ev[1].synchronize(); bwd_ms += ev[0].elapsed_time(ev[1])
        n_valid = (k1 - k0) - (1 if have_term else 0)
        tx.copy_(xs[0]); tP.copy_(Ps[0])   # smoothed estimate of step k0: where the segment in front of this one starts
        have_term = True
        sink(lo, hi, k0, xs[:n_valid], Ps[:n_valid])
      tiles += 1
    self.stats = {"tiles": tiles, "tile_filters": n_tile, "segments": nseg, "segment_steps": S, "forward_ms": fwd_ms, "reforward_with_history_ms": refwd_ms,
                  "backward_ms": bwd_ms, "bytes_per_filter": self.bytes_per_filter(T)}
    return tiles


def ragged_history_bytes_per_filter(dim_x, dim_err, T, packed_doubles=0):
  """Bytes of one filter's share of a RaggedHistory of T rows (BatchedEKF.new_ragged_history(T)): the four slabs, the
  per-filter times and the row count."""
  return history_bytes_per_filter(dim_x, dim_err, T, packed_doubles=packed_doubles) + 8 * T + 4


class RaggedCheckpointedSmoother(CheckpointedSmoother):
  """Forward filter + RTS smoother over RAGGED streams (filters on their own clocks, RaggedScheduler) too long for one
  RaggedHistory, in equal tiles of filters planned from the HBM budget like CheckpointedSmoother.

  A whole RaggedHistory is padded to the longest stream (T * B * 8 120 bytes for live, 4 600 packed).  Here the stream is
  cut into segments of `segment` TICKS.  Pass 1 runs RaggedScheduler without a history and, before the first tick of
  every segment, checkpoints each filter's x, P, clock and rows so far (it steps through the same recording kernels as
  the re-forward, into a history of one row); it also counts each filter's rows per segment,
  whose maximum (+ 1) sizes the one segment history, so no tick waits for the host.  The backward sweep then visits the
  segments last to first: it restores the checkpoint, replays the segment's ticks through RaggedScheduler(history=...),
  appends to each filter the first row of its next segment that has rows (its predicted state and time; the carried
  row), and smooths every filter over its own rows from the smoothed estimate of that carried row
  (BatchedEKF.rts_smooth_ragged_segment).  A filter's row 0 then becomes its carried row and terminal estimate for the
  segments in front; a filter without rows in a segment keeps the one it carries.  Each filter's rows come out bit for
  bit as one whole RaggedHistory + rts_smooth would give them (the kernels are deterministic).  Memory per filter is one
  checkpoint per segment plus a segment history; the price is a second forward pass.

  Observations that arrive late are dropped by RaggedScheduler, as in a single pass.  Streams with late observations are
  for RewindingScheduler, which records the rows RaggedScheduler would record for the same observations in time-stamp
  order (DESIGN.md section 4.7): for offline smoothing, sort such a stream by time stamp first and smooth it here.
  MSCKF streams whose camera frames shift the clone window pass the ticks' augment flags (RaggedScheduler.tick's
  `augment`); pass 1 and the re-forward both apply them.  Above EDIM 32 the smoothing step is refused
  (rts_smooth_ragged_segment), so such filters are not smoothed here.

  packed_history=True: the segment history, the carried rows and terminal estimates and the covariances the sink receives
  are packed ([..., packed doubles]; unpack_P gives them full); the checkpoints stay full."""

  def __init__(self, folder, name, Q, dim_x, dim_err, quaternion_idxs=(), device="cuda", hbm_budget_bytes=60 << 30, segment=64, tile=None,
               packed_history=False):
    super().__init__(folder, name, Q, dim_x, dim_err, quaternion_idxs=quaternion_idxs, device=device,
                     hbm_budget_bytes=hbm_budget_bytes, segment=segment, tile=tile, packed_history=packed_history)

  def bytes_per_filter(self, n_ticks):
    """Per filter: a checkpoint per segment (x, P, clock, rows so far, rows in the segment), a segment history of at most
    `segment` + 1 rows (a filter records at most one row per tick, + the carried row) and pass 1's history of one row,
    the carried row and terminal estimate, and the resident state with its scheduler clock."""
    nseg = (n_ticks + self.segment - 1) // self.segment
    state = 8 * (self.dim_err**2 + self.dim_x)
    cov = self.packed_doubles or self.dim_err**2
    hist = sum(ragged_history_bytes_per_filter(self.dim_x, self.dim_err, T, self.packed_doubles) for T in (self.segment + 1, 1))
    return nseg * (state + 8 + 8 + 4) + hist + 8 * (2 * self.dim_x + 2 * cov + 1) + 3 * state + 2 * 8

  def run(self, x0, P0, n_ticks, tick_fn, sink, norm_quats=False):
    """x0 [B, DIM], P0 [B, EDIM, EDIM] (host or device).  tick_fn(j, lo, hi) returns tick j of filters lo..hi as the
    arguments of RaggedScheduler.tick, with filter ids local to the tile: (filter_ids, t, kinds, z_by_kind, R_by_kind),
    those and ea_by_kind, or those and augment (ea_by_kind may be None).  It must return the same tick every time it is
    asked for j (each tick is filtered twice).

    sink(lo, hi, k0 [n], n_rows [n], xs [rows, n, DIM], Ps [rows, n, EDIM, EDIM]) receives, segment by segment (last to
    first), the smoothed rows of filters lo..hi: rows 0 .. n_rows[b] - 1 of filter b are its global rows k0[b] .. (its
    k-th applied observation is its global row k).  Device views, valid during the call only; Ps [rows, n, packed doubles]
    with packed_history.  Returns the number of tiles."""
    from rednose_b200.scheduler import RaggedScheduler
    B, S = x0.shape[0], self.segment
    n_tile, _ = self.plan(B, n_ticks)
    nseg = (n_ticks + S - 1) // S
    dev, f64 = self.device, dict(dtype=torch.float64, device=self.device)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fwd_ms = refwd_ms = bwd_ms = 0.0
    tiles, max_rows = 0, 0
    for lo in range(0, B, n_tile):
      hi = min(lo + n_tile, B)
      n = hi - lo
      if self._engine is None or self._engine.B != n:
        self._engine = self._hist = self._ck = None     # release the previous tile's buffers before allocating
        self._engine = BatchedEKF(self.folder, self.name, self.Q, x0[lo:hi], P0[lo:hi], device=dev, quaternion_idxs=self.quat)
      else:
        self._engine.init_state(x0[lo:hi], P0[lo:hi], None)
      eng = self._engine
      if self._ck is None or self._ck[0].shape[0] != nseg:
        self._ck = None
        self._ck = (torch.empty(nseg, n, self.dim_x, **f64), torch.empty(nseg, n, self.dim_err, self.dim_err, **f64),
                    torch.empty(nseg, n, **f64), torch.empty(nseg, n, dtype=torch.int64, device=dev),
                    torch.empty(nseg, n, dtype=torch.int32, device=dev))
      ck_x, ck_P, ck_t, ck_k0, rows = self._ck
      rows.zero_()
      # ---- pass 1: forward; checkpoint before the first tick of every segment, count rows per segment.  It steps through
      # the recording gather kernels like the re-forward, so that the checkpoints are bit for bit the states the re-forward
      # reaches (the gather kernels with and without history rows are separate instantiations, which need not round
      # alike); into a history of one row, which every later step finds used up and does not record into ----
      sched = RaggedScheduler(eng, history=eng.new_ragged_history(1, packed=bool(self.packed_doubles)))
      done = torch.zeros(n, dtype=torch.int64, device=dev)
      ev[0].record()
      for j in range(nseg):
        ck_x[j].copy_(eng.x); ck_P[j].copy_(eng.P); ck_t[j].copy_(sched.t_filter); ck_k0[j].copy_(done)
        for tick in range(j * S, min((j + 1) * S, n_ticks)):
          for ids, _ in sched.tick(*tick_fn(tick, lo, hi)).values():
            rows[j].index_add_(0, ids, torch.ones_like(ids, dtype=torch.int32))
        done += rows[j]
      ev[1].record(); ev[1].synchronize(); fwd_ms += ev[0].elapsed_time(ev[1])
      T = int(rows.max()) + 1                           # the longest segment of any filter + its carried row
      max_rows = max(max_rows, T - 1)
      if self._hist is None or self._hist.T != T:
        self._hist = None
        self._hist = eng.new_ragged_history(T, packed=bool(self.packed_doubles))
      hist = self._hist
      cov = hist.P_filt.shape[2:]
      # the carried row (x_pred, P_pred, t) of every filter and its smoothed estimate (the terminal)
      cx, cP, ct = torch.empty(n, self.dim_x, **f64), torch.empty(n, *cov, **f64), torch.empty(n, **f64)
      tx, tP = torch.empty(n, self.dim_x, **f64), torch.empty(n, *cov, **f64)
      carry = torch.zeros(n, dtype=torch.bool, device=dev)
      ar = torch.arange(n, device=dev)
      sched = RaggedScheduler(eng, history=hist)
      # ---- backward sweep: segments last to first, each re-filtered with history from its checkpoint, then smoothed ----
      for j in range(nseg - 1, -1, -1):
        eng.x.copy_(ck_x[j]); eng.P.copy_(ck_P[j]); sched.t_filter.copy_(ck_t[j])
        hist.n.zero_(); hist.overflow.zero_()
        ev[0].record()
        for tick in range(j * S, min((j + 1) * S, n_ticks)):
          sched.tick(*tick_fn(tick, lo, hi))
        ev[1].record(); ev[1].synchronize(); refwd_ms += ev[0].elapsed_time(ev[1])
        lost = hist.overflowed()
        if lost:
          raise RuntimeError(f"segment {j} (ticks {j * S} .. {min((j + 1) * S, n_ticks) - 1}) overflowed its history of {T} "
                             f"rows by {lost} step(s): the stream differs from pass 1; use a shorter segment")
        nr = hist.n.clone()
        term = carry & (nr > 0)
        r = nr.clamp(max=T - 1).to(torch.int64)         # row n[b]: the carried row of the filters with a terminal
        hist.x_pred[r, ar] = torch.where(term[:, None], cx, hist.x_pred[r, ar])
        hist.P_pred[r, ar] = torch.where(term.view(-1, *[1] * len(cov)), cP, hist.P_pred[r, ar])
        hist.t[r, ar] = torch.where(term, ct, hist.t[r, ar])
        hist.n += term.to(torch.int32)
        ev[0].record()
        xs, Ps = eng.rts_smooth_ragged_segment(hist, term, ck_k0[j], (tx, tP), norm_quats=norm_quats,
                                               quaternion_idxs=self.quat or (3,), in_place=True)
        ev[1].record(); ev[1].synchronize(); bwd_ms += ev[0].elapsed_time(ev[1])
        has = nr > 0                                    # row 0 hands over to the segments in front
        cx.copy_(torch.where(has[:, None], hist.x_pred[0], cx))
        cP.copy_(torch.where(has.view(-1, *[1] * len(cov)), hist.P_pred[0], cP))
        ct.copy_(torch.where(has, hist.t[0], ct))
        tx.copy_(torch.where(has[:, None], xs[0], tx))
        tP.copy_(torch.where(has.view(-1, *[1] * len(cov)), Ps[0], tP))
        carry |= has
        sink(lo, hi, ck_k0[j], nr, xs, Ps)
      tiles += 1
    self.stats = {"tiles": tiles, "tile_filters": n_tile, "segments": nseg, "segment_ticks": S, "segment_rows": max_rows,
                  "forward_ms": fwd_ms, "reforward_with_history_ms": refwd_ms, "backward_ms": bwd_ms,
                  "bytes_per_filter": self.bytes_per_filter(n_ticks)}
    return tiles
