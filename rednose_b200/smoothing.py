"""Forward filter + RTS smoother over long histories, tiled over filters.

The smoother needs x_{k|k-1}, x_{k|k}, P_{k|k-1}, P_{k|k} of every step (rednose/helpers/ekf_sym.py:651-690
walks the list of tuples returned by predict_and_update_batch): 2*EDIM^2 + 2*DIM + 1 doubles per filter-step,
8.1 kB for live_kf.  BASELINE.json config 4 (1M filters x 10k steps) would be 81 TB, so the batch is cut into
TILES of filters whose whole history fits the HBM budget; each tile runs forward-store-then-backward-consume and
hands its smoothed track to a sink before the next tile reuses the buffers (SURVEY.md section 7, hard part 3).
Tiles are independent, so multi-GPU use is: shard the filters over ranks first, tile within a rank.
"""
from __future__ import annotations

import torch

from rednose_b200.batched import BatchedEKF


def history_bytes_per_filter(dim_x, dim_err, T, smoothed_in_place=True):
  per_step = 2 * dim_err * dim_err + 2 * dim_x
  if not smoothed_in_place:
    per_step += dim_err * dim_err + dim_x
  return 8 * per_step * T


class TiledSmoother:
  def __init__(self, folder, name, Q, dim_x, dim_err, quaternion_idxs=(), device="cuda", hbm_budget_bytes=60 << 30, tile=None):
    self.folder, self.name, self.Q = folder, name, Q
    self.dim_x, self.dim_err = dim_x, dim_err
    self.quat = tuple(quaternion_idxs)
    self.device = torch.device(device)
    self.budget = hbm_budget_bytes
    self.tile = tile
    self._engine = None
    self._hist = None

  def tile_size(self, T):
    if self.tile:
      return self.tile
    per = history_bytes_per_filter(self.dim_x, self.dim_err, T) + 8 * (self.dim_err**2 + self.dim_x)
    return max(1, int(self.budget // per))

  def run(self, x0, P0, T, obs_fn, sink, norm_quats=False, t0=0.0, passes=1):
    """x0 [B, DIM], P0 [B, EDIM, EDIM] (host or device).  obs_fn(k, lo, hi) -> (t, kind, z [hi-lo, m], R) gives the
    observation of step k for filters lo..hi.  sink(lo, hi, xs [T, n, DIM], Ps [T, n, EDIM, EDIM]) receives device
    views that are only valid during the call.  Returns the number of tiles.

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
        self._hist = self._engine.new_history(T) if (self._hist is None or self._hist.B != n or self._hist.T != T) else self._hist
      else:
        self._engine.init_state(x0[lo:hi], P0[lo:hi], None)
      eng, hist = self._engine, self._hist
      for p in range(max(1, int(passes))):
        if p > 0:   # the smoothed slabs alias the history buffers the next forward pass overwrites: copy step 0 out first
          eng.init_state(xs[0].clone(), Ps[0].clone(), None)
        hist.n = 0
        eng.filter_time = t0
        for k in range(T):
          t, kind, z, R = obs_fn(k, lo, hi)
          eng.step_recorded(hist, kind, t, z, R)
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
  whole history at once (tests/test_parity_gpu.py::test_checkpointed_smoother_equals_full_history)."""

  def __init__(self, folder, name, Q, dim_x, dim_err, quaternion_idxs=(), device="cuda", hbm_budget_bytes=60 << 30, segment=64, tile=None):
    self.folder, self.name, self.Q = folder, name, Q
    self.dim_x, self.dim_err = dim_x, dim_err
    self.quat = tuple(quaternion_idxs)
    self.device = torch.device(device)
    self.budget, self.segment, self.tile = hbm_budget_bytes, int(segment), tile
    self._engine = self._hist = self._ck = None
    self.stats = {}

  def bytes_per_filter(self, T):
    nseg = (T + self.segment - 1) // self.segment
    state = 8 * (self.dim_err**2 + self.dim_x)
    return nseg * state + history_bytes_per_filter(self.dim_x, self.dim_err, self.segment + 1) + 3 * state

  def tile_size(self, T):
    return self.tile or max(1, int(self.budget // self.bytes_per_filter(T)))

  def plan(self, B, T):
    """(filters per tile, tiles): the batch is cut into EQUAL tiles no larger than tile_size(T), so that one engine and
    one set of history / checkpoint buffers serve every tile."""
    cap = min(self.tile_size(T), B)
    ntiles = (B + cap - 1) // cap
    return (B + ntiles - 1) // ntiles, ntiles

  def run(self, x0, P0, T, obs_fn, sink, norm_quats=False, t0=0.0):
    """obs_fn(k, lo, hi) -> (t, kind, z, R) must return the SAME observation every time it is asked for step k (each step
    is filtered twice) in a buffer the kernel may overwrite.  sink(lo, hi, k0, xs [n, tile, DIM], Ps [n, tile, EDIM, EDIM])
    receives the smoothed steps k0 .. k0 + n - 1 of filters lo..hi (segments arrive last to first; views valid during
    the call only).  Returns the number of tiles."""
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
        self._hist = self._engine.new_history(S + 1)
        self._ck = (torch.empty(nseg, n, self.dim_x, dtype=torch.float64, device=self.device),
                    torch.empty(nseg, n, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device))
        self._term = (torch.empty(n, self.dim_x, dtype=torch.float64, device=self.device),
                      torch.empty(n, self.dim_err, self.dim_err, dtype=torch.float64, device=self.device))
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
        t, kind, z, R = obs_fn(k, lo, hi)
        eng.predict_and_update_batch(t, kind, z, R)
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
          t, kind, z, R = obs_fn(k, lo, hi)
          eng.step_recorded(hist, kind, t, z, R)
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
