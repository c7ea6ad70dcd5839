"""What raggedness costs: live_kf filters recording config-3 streams on their own clocks, then smoothed per filter.

Workload: B live filters (default 16 384), a history of T rows per filter (default 256: 34 GB of slabs at 8 120 B per
filter-row).  Every filter sees a 100 Hz gyro (kind 4) and a 100 Hz accelerometer (kind 10) interleaved, 200 samples a
second, and a 1 Hz position fix (kind 12) in place of one of them, each filter with its own phase (so every tick mixes
all three kinds) and ~3 % of its samples missing.  The forward pass issues one recording gather launch per kind per
tick (`step_indexed(..., hist=)`, the launches RaggedScheduler makes, with the per-kind buckets prepared on the device
beforehand); the backward pass is one `rts_smooth(RaggedHistory)` launch.

In the same process, alternating with it, the lockstep path on the same batch and row count: every filter observes
the same kind at the same time (aligned phases), `step_recorded` + `rts_smooth(History)`.

Reported (one JSON line): filter-steps/s of each pass = recorded steps (ragged: sum of n[b]) over the wall time between
two device synchronisations, best of the rounds, plus the card's name, power limit and maximum SM clock (nvidia-smi,
read only).  The forward ragged time includes the host-side issue of RaggedHistory.reserve (a few small torch kernels
per launch).  Nothing is written to disk.

  python scripts/ragged_rts_bench.py [--filters 16384] [--rows 256] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KINDS = (4, 10, 12)


def gpu_card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    return [s.strip() for s in out.split(",")]
  except (OSError, subprocess.SubprocessError):
    return ["unknown", "unknown", "unknown"]


def kind_at(phase_tick):
  """Kind observed at tick `phase_tick` of a filter's own 200 Hz sample clock."""
  return torch.where(phase_tick % 200 == 0, 12, torch.where(phase_tick % 2 == 0, 4, 10))


def ragged_plan(B, T, dev, seed):
  """Per tick, per kind: (ids int32, dt, t) device tensors of the filters that observe that kind in that tick."""
  g = torch.Generator(device=dev).manual_seed(seed)
  off = torch.randint(0, 200, (B,), device=dev, generator=g)            # per-filter phase, in samples
  jit = torch.rand(B, device=dev, dtype=torch.float64, generator=g) * 0.005
  t_last = torch.full((B,), float("nan"), device=dev, dtype=torch.float64)
  plan, steps = [], 0
  for j in range(T):
    ph = j + off
    t = ph.to(torch.float64) * 0.005 + jit
    keep = torch.rand(B, device=dev, generator=g) >= 0.03
    kinds = kind_at(ph)
    tick = []
    for k in KINDS:
      ids = ((kinds == k) & keep).nonzero(as_tuple=True)[0]
      if ids.numel() == 0:
        continue
      tk = t[ids]
      tl = t_last[ids]
      dt = torch.where(torch.isnan(tl), torch.zeros_like(tk), tk - tl)
      t_last[ids] = tk
      tick.append((k, ids.to(torch.int32), dt.contiguous(), tk.contiguous()))
      steps += int(ids.numel())
    plan.append(tick)
  return plan, steps


def observations(x0, dev):
  from tests.util import LIVE_R
  B = x0.shape[0]
  g = torch.Generator(device=dev).manual_seed(5)
  z = {4: torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 0.01,
       10: torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 0.1 + torch.tensor([0.0, 0.0, -9.8], device=dev, dtype=torch.float64),
       12: torch.as_tensor(x0[:, :3], device=dev) + torch.randn(B, 3, device=dev, dtype=torch.float64, generator=g) * 5.0}
  R = {k: torch.diag(torch.tensor(LIVE_R[k], device=dev, dtype=torch.float64)) for k in KINDS}
  return z, R


def timed(fn):
  """Wall time of fn() between two device synchronisations; its result is dropped (it may hold 17 GB of views)."""
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=16384)
  ap.add_argument("--rows", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=3)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("ragged_rts_bench needs a CUDA device")
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from tests.util import live_batch
  dev = torch.device("cuda:0")
  B, T = a.filters, a.rows
  x0, P0, Q = live_batch(B, seed=1)
  eng = BatchedEKF(ensure_generated(LiveKalman), "live", Q, x0, P0, device=dev, quaternion_idxs=[3])
  z, R = observations(x0, dev)
  plan, ragged_steps = ragged_plan(B, T, dev, seed=2)
  zr = [[z[k][ids.long()] for k, ids, _, _ in tick] for tick in plan]
  lock_kinds = [int(kind_at(torch.tensor(j))) for j in range(T)]

  def ragged_forward(h):
    for tick, zt in zip(plan, zr):
      for (k, ids, dt, tk), zk in zip(tick, zt):
        eng.step_indexed(k, ids, dt, zk.clone(), R[k], hist=h, t=tk)

  def lockstep_forward(h):
    for j, k in enumerate(lock_kinds):
      eng.step_recorded(h, k, 0.005 * j, z[k].clone(), R[k])

  res = {"ragged_forward": [], "ragged_backward": [], "lockstep_forward": [], "lockstep_backward": []}
  for r in range(a.rounds + 1):                   # round 0 warms every launch shape up and is not reported
    for path in ("ragged", "lockstep"):
      eng.init_state(x0, P0)
      if path == "ragged":
        h = eng.new_ragged_history(T)
        tf = timed(lambda: ragged_forward(h))
        assert int(h.n.sum()) == ragged_steps and h.overflowed() == 0
        tb = timed(lambda: eng.rts_smooth(h, norm_quats=True, in_place=True))
        steps = ragged_steps
      else:
        h = eng.new_history(T)
        tf = timed(lambda: lockstep_forward(h))
        tb = timed(lambda: eng.rts_smooth(h, norm_quats=True, in_place=True))
        steps = B * T
      del h
      if r > 0:
        res[f"{path}_forward"].append(steps / tf)
        res[f"{path}_backward"].append(steps / tb)
  name, power, sm = gpu_card()
  out = {"workload": f"live_kf, {B} filters, {T}-row history, config-3 streams (4 / 10 at 100 Hz, 12 at 1 Hz, 3 % missing)",
         "gpu": name, "power_limit": power, "max_sm_clock": sm, "rounds": a.rounds,
         "ragged_recorded_steps": ragged_steps, "lockstep_recorded_steps": B * T,
         "history_bytes": 2 * T * B * 8 * (23 + 22 * 22)}
  for key, v in res.items():
    out[f"{key}_filter_steps_per_s"] = max(v)
    out[f"{key}_spread"] = (max(v) - min(v)) / max(v)
  print(json.dumps(out))


if __name__ == "__main__":
  main()
