"""Smoothing ragged streams far longer than one history: live_kf filters on their own clocks, RaggedCheckpointedSmoother.

Workload (the ragged_rts_bench.py configuration): B live filters (default 16 384), every one with a 100 Hz gyro (kind 4)
and a 100 Hz accelerometer (kind 10) interleaved, 200 samples a second, and a 1 Hz position fix (kind 12) in place of
one of them, each filter with its own phase (every tick mixes all three kinds) and ~3 % of its samples missing.  The
stream runs for --ticks ticks of 5 ms (default 4 096: 20 s, ~4 000 rows per filter), which as one whole RaggedHistory
would take 8 120 bytes per filter-row (545 GB at the defaults); here it is cut into segments of --segment ticks.

Timed, per phase (CUDA events inside the smoother, so host issue between launches is included): pass 1 (RaggedScheduler
without history, checkpoints), the re-forward of every segment with history, and the backward pass (the
<name>_batch_rts_ragged_segment launches).  Reported as one JSON line with filter-steps/s per phase (recorded steps over
the phase's time, best of the rounds), the bytes per filter the smoother plans with against a whole RaggedHistory, and
the card's name, power limit and maximum SM clock (nvidia-smi, read only).  A short run of two segments warms every
launch shape up first.  Nothing is written to disk.

  python scripts/ragged_long_smoothing_bench.py [--filters 16384] [--ticks 4096] [--segment 256] [--rounds 2]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.ragged_rts_bench import KINDS, gpu_card, kind_at, observations  # noqa: E402


def tick_plan(B, n_ticks, dev, seed):
  """Per tick: (filter ids [m] int64, times [m], kinds [m]) on the device, grouped by kind; and the number of samples."""
  g = torch.Generator(device=dev).manual_seed(seed)
  off = torch.randint(0, 200, (B,), device=dev, generator=g)            # per-filter phase, in samples
  jit = torch.rand(B, device=dev, dtype=torch.float64, generator=g) * 0.005
  plan, steps = [], 0
  for j in range(n_ticks):
    ph = j + off
    t = ph.to(torch.float64) * 0.005 + jit
    keep = torch.rand(B, device=dev, generator=g) >= 0.03
    kinds = kind_at(ph)
    ids = torch.cat([((kinds == k) & keep).nonzero(as_tuple=True)[0] for k in KINDS])
    plan.append((ids, t[ids].contiguous(), kinds[ids].contiguous()))
    steps += int(ids.numel())
  return plan, steps


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=16384)
  ap.add_argument("--ticks", type=int, default=4096)
  ap.add_argument("--segment", type=int, default=256)
  ap.add_argument("--rounds", type=int, default=2)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("ragged_long_smoothing_bench needs a CUDA device")
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  from rednose_b200.smoothing import RaggedCheckpointedSmoother, ragged_history_bytes_per_filter
  from tests.util import live_batch
  dev = torch.device("cuda:0")
  B, N, S = a.filters, a.ticks, a.segment
  x0, P0, Q = live_batch(B, seed=1)
  z, R = observations(x0, dev)
  plan, steps = tick_plan(B, N, dev, seed=2)

  def tick_fn(j, lo, hi):
    ids, t, kinds = plan[j]
    if lo or hi != B:                  # tile-local ids (one tile at the defaults)
      sel = (ids >= lo) & (ids < hi)
      ids, t, kinds = ids[sel], t[sel], kinds[sel]
    return ids - lo, t, kinds, {k: z[k][ids[kinds == k]] for k in KINDS}, R

  def sink(lo, hi, k0, n_rows, xs, Ps):
    pass

  cs = RaggedCheckpointedSmoother(ensure_generated(LiveKalman), "live", Q, 23, 22, quaternion_idxs=[3], device=dev, segment=S)
  cs.run(x0, P0, min(N, 2 * S), tick_fn, sink, norm_quats=True)      # warm-up: every launch shape once
  res = {"pass1": [], "reforward_with_history": [], "backward": []}
  for _ in range(a.rounds):
    cs.run(x0, P0, N, tick_fn, sink, norm_quats=True)
    st = cs.stats
    res["pass1"].append(st["forward_ms"])
    res["reforward_with_history"].append(st["reforward_with_history_ms"])
    res["backward"].append(st["backward_ms"])
  name, power, sm = gpu_card()
  out = {"workload": f"live_kf, {B} filters, {N} ticks of 5 ms in segments of {S}, config-3 streams (4 / 10 at 100 Hz, "
                     f"12 at 1 Hz, 3 % missing)",
         "gpu": name, "power_limit": power, "max_sm_clock": sm, "rounds": a.rounds, "recorded_steps": steps,
         "tiles": st["tiles"], "segments": st["segments"], "segment_history_rows": st["segment_rows"] + 1,
         "bytes_per_filter": st["bytes_per_filter"],
         "whole_ragged_history_bytes_per_filter": ragged_history_bytes_per_filter(23, 22, N)}
  for key, v in res.items():
    out[f"{key}_ms"] = min(v)
    out[f"{key}_filter_steps_per_s"] = steps / (min(v) * 1e-3)
    out[f"{key}_spread"] = (max(v) - min(v)) / max(v)
  print(json.dumps(out))


if __name__ == "__main__":
  main()
