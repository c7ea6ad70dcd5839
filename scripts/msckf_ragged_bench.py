"""MSCKF fleets on their own clocks: RaggedScheduler with clone-window shifts, against the lockstep step(augment=True).

Workload: B msckf filters (default 10 000; EDIM 82, ten pose clones) for 2 s of stream at 100 Hz ticks.  Every filter
sees a gyro sample (kind 4, a plain kind) at every tick, except that at 20 Hz, at a per-filter random phase, a camera
frame (kind 17, the gated feature-track kind, 20 coordinates, its 3-D point as extra arguments) takes its place and
shifts the clone window (RaggedScheduler.tick(..., augment=)).  So every tick mixes both kinds: 8 000 gyro samples and
2 000 shifting frames at the default size.  Initial states are 64 distinct msckf states tiled over the batch; each frame
observes h(x0) of its filter plus 1e-4 noise.

Reported (one JSON line), best of the rounds after a warm-up round:
- ragged: ticks/s and filter-steps/s of RaggedScheduler over the whole stream (wall time between two device
  synchronisations, host issue included);
- lockstep: filter-steps/s of the same step count in lockstep, BatchedEKF.step over the whole batch with the same kind
  sequence, frames with augment=True (the shift fused into the CTA kernel's write-back);
- augment: device time (CUDA events, median of the rounds) of <name>_batch_augment_idx on half the batch against
  <name>_batch_augment on all of it, with the bytes each moves (x and P read and written once per shifted filter).
Plus the card's name, power limit and maximum SM clock (nvidia-smi, read only).  Nothing is written to disk.

  python scripts/msckf_ragged_bench.py [--filters 10000] [--seconds 2] [--rounds 3]
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

QUATS = [3] + [23 + 3 + 7 * c for c in range(10)]   # the main attitude and the 10 clone attitudes


def gpu_card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    return [s.strip() for s in out.split(",")]
  except (OSError, subprocess.SubprocessError):
    return ["unknown", "unknown", "unknown"]


def timed(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=10_000)
  ap.add_argument("--seconds", type=float, default=2.0)
  ap.add_argument("--rounds", type=int, default=3)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("msckf_ragged_bench needs a CUDA device")
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.msckf import DIM, EDIM, MsckfKalman
  from rednose_b200.scheduler import RaggedScheduler
  from tests.util import LIVE_R, msckf_batch
  dev = torch.device("cuda:0")
  B, n_ticks = a.filters, int(round(a.seconds * 100))
  xs, Ps, Q, pts = msckf_batch(64, seed=1)
  tile = np.arange(B) % 64
  x0, P0, point = xs[tile], Ps[tile], pts[tile]
  eng = BatchedEKF(ensure_generated(MsckfKalman), "msckf", Q, x0, P0, device=dev, quaternion_idxs=QUATS)
  h = np.zeros((64, 20))
  for i in range(64):                                   # h_17 of the 64 distinct states (host entry point)
    xi, pi, hi = (np.ascontiguousarray(v) for v in (xs[i], pts[i], h[i]))
    eng._lib.msckf_h_17(eng._ffi.cast("double *", xi.ctypes.data), eng._ffi.cast("double *", pi.ctypes.data),
                        eng._ffi.cast("double *", hi.ctypes.data))
    h[i] = hi
  g = torch.Generator(device=dev).manual_seed(2)
  phase = torch.randint(0, 5, (B,), device=dev, generator=g)
  zf = torch.as_tensor(h[tile], device=dev) + 1e-4 * torch.randn(B, 20, device=dev, dtype=torch.float64, generator=g)
  Rf = torch.eye(20, device=dev, dtype=torch.float64) * 1e-3 ** 2
  zg = torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 0.01
  Rg = torch.diag(torch.tensor(LIVE_R[4], device=dev, dtype=torch.float64))
  pt = torch.as_tensor(point, device=dev)
  ids = torch.arange(B, device=dev)
  jit = torch.rand(B, device=dev, dtype=torch.float64, generator=g) * 0.005
  ticks = []                                            # RaggedScheduler.tick arguments, prepared on the device
  for j in range(n_ticks):
    frame = (j % 5) == phase
    kinds = torch.where(frame, 17, 4)
    ticks.append((ids, 0.01 * j + jit, kinds, {4: zg[~frame], 17: zf[frame]}, {4: Rg, 17: Rf}, {17: pt[frame]}, frame))
  frames = sum(int(t[6].sum()) for t in ticks)
  steps = B * n_ticks

  def ragged():
    s = RaggedScheduler(eng)
    for tk in ticks:
      s.tick(*tk)

  def lockstep():
    for j in range(n_ticks):
      if j % 5 == 0:
        eng.step(17, 0.01, zf.clone(), Rf, ea=pt, augment=True)
      else:
        eng.step(4, 0.01, zg.clone(), Rg)

  half = torch.randperm(B, device=dev, generator=g)[:B // 2].to(torch.int32)
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
  res = {"ragged": [], "lockstep": [], "augment_idx_ms": [], "augment_all_ms": []}
  for r in range(a.rounds + 1):                         # round 0 warms every launch shape up and is not reported
    eng.init_state(x0, P0)
    tr = timed(ragged)
    eng.init_state(x0, P0)
    tl = timed(lockstep)
    ev[0].record(); eng.augment(half); ev[1].record()
    ev[2].record(); eng.augment(); ev[3].record()
    torch.cuda.synchronize()
    if r > 0:
      res["ragged"].append(tr); res["lockstep"].append(tl)
      res["augment_idx_ms"].append(ev[0].elapsed_time(ev[1])); res["augment_all_ms"].append(ev[2].elapsed_time(ev[3]))
  name, power, sm = gpu_card()
  per_filter = 2 * 8 * (DIM + EDIM * EDIM)             # x and P read and written once
  out = {"workload": f"msckf (EDIM {EDIM}), {B} filters, {a.seconds:g} s at 100 Hz ticks: gyro (4) every tick, a shifting "
                     f"frame (17) at 20 Hz per-filter phase in its place",
         "gpu": name, "power_limit": power, "max_sm_clock": sm, "rounds": a.rounds, "ticks": n_ticks,
         "filter_steps": steps, "shifting_frames": frames,
         "ragged_ticks_per_s": n_ticks / min(res["ragged"]), "ragged_filter_steps_per_s": steps / min(res["ragged"]),
         "lockstep_filter_steps_per_s": steps / min(res["lockstep"]),
         "augment_idx_filters": B // 2, "augment_idx_ms": statistics.median(res["augment_idx_ms"]),
         "augment_all_filters": B, "augment_all_ms": statistics.median(res["augment_all_ms"]),
         "augment_bytes_per_filter": per_filter}
  out["augment_idx_GBps"] = per_filter * (B // 2) / (out["augment_idx_ms"] * 1e-3) / 1e9
  out["augment_all_GBps"] = per_filter * B / (out["augment_all_ms"] * 1e-3) / 1e9
  print(json.dumps(out))


if __name__ == "__main__":
  main()
