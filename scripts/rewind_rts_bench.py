"""What late observations cost when the stream is recorded for smoothing: RewindingScheduler with and without a history.

Workload: B live_kf filters (default 16 384), a ragged history of T rows per filter (default 256).  Every filter sees a
200 Hz IMU stream, gyro (kind 4) and accelerometer (kind 10) alternating with a per-filter phase (each kind at 100 Hz),
~3 % of the samples missing, and a 1 Hz position fix (kind 12) with a per-filter phase.  Each fix arrives 50-300 ms after
its time stamp, in the 5 ms tick of its arrival: the tick applies the IMU samples, then the fixes, which rewind their
filters to the last checkpoint at or before the fix and replay the samples after it.  max_rewind_age 0.5 s and a ring
of 96 checkpoints, so no fix is lost to the depth.

Modes, in one process, alternated for --rounds rounds after one warm-up round; medians are reported:
  (a) RewindingScheduler without a history: forward only (the ring keeps x / P snapshots);
  (b) with a full RaggedHistory: forward, then rts_smooth;
  (c) with a packed RaggedHistory: forward, then rts_smooth;
  (d) RaggedScheduler with a full RaggedHistory, fed each filter's observations in time order (one per tick): the same
      stream without lateness.
Forward and backward times are host clocks between two device synchronisations.  The restore time is the device time
(CUDA events) of the rewinds' restores, re-issued after the pass with the same per-tick filter lists: (a) the gather of
the x / P snapshots and set_P_rows, (b) / (c) one restore_from_history launch per tick.

Checks: (b) and (d) give bit-identical smoothed rows, and so do (c) and (d) recorded into a packed history (in the
warm-up round): every row below n of every filter through a position-weighted fingerprint of the raw bits, and 256
sampled filters compared exactly.  One JSON line, with the card's name, power limit and maximum SM clock (nvidia-smi,
read only).  Nothing is written to disk.

  python scripts/rewind_rts_bench.py [--filters 16384] [--rows 256] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KINDS = (4, 10, 12)
TICK = 0.005


def gpu_card():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30, check=True).stdout.strip().split("\n")[0]
  return [s.strip() for s in out.split(",")]


def make_stream(B, ticks, seed):
  """Host arrays of every observation: filter, time, kind, arrival tick (numpy)."""
  rng = np.random.default_rng(seed)
  ph, jit = rng.integers(0, 2, B), rng.uniform(0, 0.004, B)
  f, t, k, arr = [], [], [], []
  for j in range(ticks):
    keep = (rng.random(B) >= 0.03) | (j < 4)           # every filter checkpoints before its first fix's time stamp
    b = np.flatnonzero(keep)
    f.append(b); t.append(TICK * (j + 1) + jit[b]); k.append(np.where((j + ph[b]) % 2 == 0, 4, 10)); arr.append(np.full(b.size, j))
  gph = rng.uniform(0.03, 1.0, B)
  for i in range(int(ticks * TICK) + 1):
    tg = gph + i
    a = np.ceil((tg + rng.uniform(0.05, 0.3, B)) / TICK).astype(np.int64) - 1
    b = np.flatnonzero(a < ticks)
    f.append(b); t.append(tg[b]); k.append(np.full(b.size, 12)); arr.append(a[b])
  return tuple(np.concatenate(v) for v in (f, t, k, arr))


def device_ticks(sel_groups, f, t, k, z, R, dev):
  """[(ids, t, kinds, z_by_kind, R_by_kind)] device tensors, one per group of observation indices."""
  out = []
  for s in sel_groups:
    ids = torch.as_tensor(f[s], device=dev)
    kk = torch.as_tensor(k[s], device=dev)
    zk, Rk = {}, {}
    for kind in KINDS:
      m = k[s] == kind
      if m.any():
        fk = torch.as_tensor(f[s][m], device=dev)
        zk[kind] = z[kind][fk]
        Rk[kind] = R[kind].expand(int(m.sum()), 3, 3).contiguous()
    out.append((ids, torch.as_tensor(t[s], device=dev), kk, zk, Rk))
  return out


def fingerprint(xs, Ps, n):
  """Position-weighted sum of the raw bits of every row below n[b] (int64 arithmetic wraps)."""
  acc = torch.zeros((), dtype=torch.int64, device=xs.device)
  for r in range(xs.shape[0]):
    live = (n > r)[:, None]
    for v in (xs[r].reshape(xs.shape[1], -1), Ps[r].reshape(Ps.shape[1], -1)):
      w = torch.arange(1, v.numel() + 1, device=v.device, dtype=torch.int64).reshape(v.shape) * (2 * r + 1)
      acc += torch.where(live, v.view(torch.int64) * w, 0).sum()
  return int(acc)


def ms_events(pairs):
  torch.cuda.synchronize()
  return sum(a.elapsed_time(b) for a, b in pairs)


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=16384)
  ap.add_argument("--rows", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=5)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("rewind_rts_bench needs a CUDA device")
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.scheduler import RaggedScheduler, RewindingScheduler
  from tests.util import LIVE_R, live_batch
  dev = torch.device("cuda:0")
  B, T = a.filters, a.rows
  ticks = T - 16                                       # IMU rows + up to two fixes stay below T
  x0, P0, Q = live_batch(B, seed=1)
  eng = BatchedEKF(ensure_generated(LiveKalman), "live", Q, x0, P0, device=dev, quaternion_idxs=[3])
  g = torch.Generator(device=dev).manual_seed(5)
  z = {4: torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 0.01,
       10: torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 0.1 + torch.tensor([0.0, 0.0, -9.8], device=dev, dtype=torch.float64),
       12: torch.as_tensor(x0[:, :3], device=dev) + torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 5.0}
  R = {k: torch.diag(torch.tensor(LIVE_R[k], device=dev, dtype=torch.float64)) for k in KINDS}
  f, t, k, arr = make_stream(B, ticks, seed=2)
  # arrival order: per tick the IMU samples, then the fixes (a second tick() call)
  late_groups, arrival = [], []
  for j in range(ticks):
    imu = np.flatnonzero((arr == j) & (k != 12))
    fix = np.flatnonzero((arr == j) & (k == 12))
    arrival.append(imu)
    if fix.size:
      arrival.append(fix)
      late_groups.append(torch.as_tensor(f[fix], device=dev))
  arrival_ticks = device_ticks(arrival, f, t, k, z, R, dev)
  order = np.lexsort((t, f))                           # each filter's observations in time order
  start = np.searchsorted(f[order], np.arange(B))
  rank = np.arange(order.size) - start[f[order]]
  in_order_ticks = device_ticks([order[rank == j] for j in range(rank.max() + 1)], f, t, k, z, R, dev)
  n_expect = np.bincount(f, minlength=B)
  assert n_expect.max() <= T
  zd = {kind: 3 for kind in KINDS}
  sample = torch.as_tensor(np.random.default_rng(3).choice(B, 256, replace=False), device=dev)

  def rewinding(history):
    return RewindingScheduler(eng, zd, depth=96, max_rewind_age=0.5, history=history)

  def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)

  def run_ticks(s, tk):
    for ids, tt, kk, zk, Rk in tk:
      s.tick(ids, tt, kk, {q: v.clone() for q, v in zk.items()}, Rk)

  def restore_ms(s, h):
    ev = []
    for lf in late_groups:
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      if h is None:
        src = (s.head[lf] + s.cnt[lf] - 1) % s.N
        eng.x[lf] = s.ring_x[lf, src]
        eng.set_P_rows(lf, s.ring_P[lf, src])
      else:
        eng.restore_from_history(h, lf, torch.zeros(lf.shape[0], dtype=torch.int32, device=dev))
      e1.record()
      ev.append((e0, e1))
    return ms_events(ev)

  def ring_bytes(s):
    names = ("ring_t", "ring_x", "ring_P", "ring_kind", "ring_z", "ring_R", "ring_ea", "ring_row", "head", "cnt")
    return sum(v.numel() * v.element_size() for v in (getattr(s, q, None) for q in names) if v is not None)

  res = {m: {"forward_ms": [], "backward_ms": [], "restore_ms": []} for m in "abcd"}
  facts, prints = {}, {}
  for r in range(a.rounds + 1):                        # round 0 warms every launch shape up, checks, and is not reported
    for m in "abcd":
      eng.init_state(x0, P0)
      h = None if m == "a" else eng.new_ragged_history(T, packed=(m == "c"))
      s = RaggedScheduler(eng, history=h) if m == "d" else rewinding(h)
      tf = timed(lambda: run_ticks(s, in_order_ticks if m == "d" else arrival_ticks))
      tb = 0.0
      if h is not None:
        assert h.overflowed() == 0 and torch.equal(h.n.cpu(), torch.as_tensor(n_expect, dtype=torch.int32))
        tb = timed(lambda: eng.rts_smooth(h, norm_quats=True, in_place=True))
      if m != "d":
        assert s.dropped == 0 and s.unrecorded == 0 and s.rewinds == sum(int(v.numel()) for v in late_groups)
        facts[m] = dict(rewinds=s.rewinds, replayed=s.replayed, ring_bytes=ring_bytes(s))
      if h is not None:
        facts[m] = dict(facts.get(m, {}), history_bytes=h.bytes())
      if r == 0 and h is not None:
        Ps = eng.unpack_P(h.P_filt[:, sample]) if h.packed else h.P_filt[:, sample]
        prints[m] = (fingerprint(h.x_filt, h.P_filt, h.n), h.x_filt[:, sample].cpu(), Ps.cpu(), h.n[sample].cpu())
      if m != "d":
        tr = restore_ms(s, h)
        if r > 0:
          res[m]["restore_ms"].append(tr)
      print(f"round {r} mode {m}: forward {tf:.0f} ms, backward {tb:.0f} ms", file=sys.stderr, flush=True)
      if r > 0:
        res[m]["forward_ms"].append(tf)
        res[m]["backward_ms"].append(tb)
      del s, h
    if r == 0:                                         # (c) against the in-order stream recorded packed
      eng.init_state(x0, P0)
      h = eng.new_ragged_history(T, packed=True)
      run_ticks(RaggedScheduler(eng, history=h), in_order_ticks)
      eng.rts_smooth(h, norm_quats=True, in_place=True)
      Ps = eng.unpack_P(h.P_filt[:, sample])
      prints["d_packed"] = (fingerprint(h.x_filt, h.P_filt, h.n), h.x_filt[:, sample].cpu(), Ps.cpu(), h.n[sample].cpu())
      del h

      def same(p, q):
        ns = p[3]
        rows = torch.arange(T)[:, None] < ns[None, :].long()
        return p[0] == q[0] and torch.equal(p[3], q[3]) and torch.equal(p[1][rows], q[1][rows]) and torch.equal(p[2][rows], q[2][rows])
      assert same(prints["b"], prints["d"]), "full history: rewound != in order"
      assert same(prints["c"], prints["d_packed"]), "packed history: rewound != in order"
  name, power, sm = gpu_card()
  out = {"workload": f"live_kf, {B} filters, {T}-row ragged history, config-3 streams (4 / 10 at 100 Hz, 12 at 1 Hz "
                     f"arriving 50-300 ms late, 3 % missing), {ticks} ticks of 5 ms",
         "gpu": name, "power_limit": power, "max_sm_clock": sm, "rounds": a.rounds,
         "recorded_steps": int(n_expect.sum()), "smoothed_rows_identical": True}
  for m in "abcd":
    for key, v in res[m].items():
      if v:
        out[f"{m}_{key}"] = round(statistics.median(v), 3)
    for key, v in facts.get(m, {}).items():
      out[f"{m}_{key}"] = v
  print(json.dumps(out))


if __name__ == "__main__":
  main()
