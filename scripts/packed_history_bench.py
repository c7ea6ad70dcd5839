"""Packed against full covariance histories: forward pass with history, backward pass and history bytes, live_kf.

Two workloads, each run in one process with the full and the packed history alternating round by round (medians over
the rounds are reported):

* lockstep: B live filters (default 65 536), T steps (default 16) of `step_recorded` cycling through the gyro (4),
  accelerometer (10) and position (12) kinds, then one `rts_smooth(History)` into preallocated buffers;
* ragged: the configuration of scripts/ragged_rts_bench.py (16 384 filters, 256 rows, config-3 streams on per-filter
  clocks, `step_indexed(..., hist=RaggedHistory)` per kind per tick), then one in-place `rts_smooth(RaggedHistory)`.

Times are wall time between two device synchronisations.  Reported (one JSON line): per workload and layout the median
forward and backward milliseconds, filter-steps/s and `bytes()` of the history, plus the card's name, power limit and
maximum SM clock (nvidia-smi, read only).  Nothing is written to disk.

  python scripts/packed_history_bench.py [--filters 65536] [--steps 16] [--ragged-filters 16384] [--rows 256] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from ragged_rts_bench import KINDS, gpu_card, observations, ragged_plan, timed  # noqa: E402


def lockstep(eng, B, T, rounds, dev):
  z, R = observations(eng.x.cpu().numpy(), dev)
  x0, P0 = eng.x.clone(), eng.P.clone()
  hist = {False: eng.new_history(T), True: eng.new_history(T, packed=True)}
  out = {p: (torch.empty_like(h.x_filt), torch.empty_like(h.P_filt)) for p, h in hist.items()}
  res = {p: {"forward_ms": [], "backward_ms": []} for p in hist}

  def forward(h):
    eng.init_state(x0, P0)
    h.n = 0
    for k in range(T):
      kind = KINDS[k % 3]
      eng.step_recorded(h, kind, 0.005 * (k + 1), z[kind].clone(), R[kind])

  for r in range(rounds + 1):          # round 0 warms up every launch shape
    for p, h in hist.items():
      f = timed(lambda: forward(h))
      b = timed(lambda: eng.rts_smooth(h, norm_quats=True, out=out[p]))
      if r:
        res[p]["forward_ms"].append(1e3 * f)
        res[p]["backward_ms"].append(1e3 * b)
  return {("packed" if p else "full"): _summary(res[p], B * T, hist[p].bytes()) for p in hist}


def ragged(eng, B, T, rounds, dev):
  z, R = observations(eng.x.cpu().numpy(), dev)
  x0, P0 = eng.x.clone(), eng.P.clone()
  plan, steps = ragged_plan(B, T, dev, seed=2)
  zr = [[z[k][ids.long()] for k, ids, _, _ in tick] for tick in plan]
  res = {p: {"forward_ms": [], "backward_ms": []} for p in (False, True)}
  nbytes = {}
  for r in range(rounds + 1):
    for p in (False, True):
      h = eng.new_ragged_history(T, packed=p)
      nbytes[p] = h.bytes()
      eng.init_state(x0, P0)

      def forward():
        for tick, zt in zip(plan, zr):
          for (k, ids, dt, tk), zk in zip(tick, zt):
            eng.step_indexed(k, ids, dt, zk.clone(), R[k], hist=h, t=tk)
      f = timed(forward)
      b = timed(lambda: eng.rts_smooth(h, norm_quats=True, in_place=True))
      del h
      if r:
        res[p]["forward_ms"].append(1e3 * f)
        res[p]["backward_ms"].append(1e3 * b)
  return {("packed" if p else "full"): _summary(res[p], steps, nbytes[p]) for p in res}


def _summary(r, steps, nbytes):
  f, b = statistics.median(r["forward_ms"]), statistics.median(r["backward_ms"])
  return {"forward_ms": round(f, 3), "backward_ms": round(b, 3), "forward_steps_per_s": round(steps / f * 1e3),
          "backward_steps_per_s": round(steps / b * 1e3), "history_bytes": nbytes,
          "forward_ms_all": [round(v, 3) for v in r["forward_ms"]], "backward_ms_all": [round(v, 3) for v in r["backward_ms"]]}


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=65536)
  ap.add_argument("--steps", type=int, default=16)
  ap.add_argument("--ragged-filters", type=int, default=16384)
  ap.add_argument("--rows", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=5)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("packed_history_bench needs a CUDA device")
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from tests.util import live_batch
  dev = torch.device("cuda:0")
  folder = ensure_generated(LiveKalman)
  card = gpu_card()
  out = {"card": card[0], "power_limit": card[1], "max_sm_clock": card[2], "rounds": a.rounds}
  x0, P0, Q = live_batch(a.filters, seed=1)
  eng = BatchedEKF(folder, "live", Q, x0, P0, device=dev, quaternion_idxs=[3])
  out["lockstep"] = dict(filters=a.filters, steps=a.steps, **lockstep(eng, a.filters, a.steps, a.rounds, dev))
  del eng
  torch.cuda.empty_cache()
  x0, P0, Q = live_batch(a.ragged_filters, seed=1)
  eng = BatchedEKF(folder, "live", Q, x0, P0, device=dev, quaternion_idxs=[3])
  out["ragged"] = dict(filters=a.ragged_filters, rows=a.rows, **ragged(eng, a.ragged_filters, a.rows, a.rounds, dev))
  print(json.dumps(out))


if __name__ == "__main__":
  main()
