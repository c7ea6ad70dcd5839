"""Checkpointed RTS smoothing of a long config-5 stream for the shipped MSCKF (DIM 93 / EDIM 82, main block 22), with
full and with main-block prediction histories.

Workload: B msckf filters (default 10 000), T camera frames (default 128), CheckpointedSmoother with segments of
`--segment` steps (default 64) under the default 60 GiB history budget.  Each frame is bench.py's msckf step: a landmark
seen from the ten clones (5 % gross outliers), triangulated by the feature front-end, then the fused predict + gated
feature update + clone-window shift (kind 17 with `ea` and `augment=True`).  The stream is generated once, before the
timed runs, by a forward pass of its own (the smoother asks for every frame twice and must get the same observation).

The two layouts are alternated within one run: `full` records P_{k+1|k} whole (109 072 bytes per filter-step),
`main_pred` only its main block plus the newest full prediction (59 152 bytes per filter-step).  With the defaults the
planner cuts the full layout into two tiles of 5 000 filters (7.36 MB per filter) and keeps the main-block layout in one
tile of 10 000 (4.17 MB), as at T = 1 000.  The default T stays short because the state of this synthetic stream, which
feeds the filter nothing but feature tracks, is no longer finite after 1 000 frames.
Round 0 warms up both; the JSON line reports per layout the tiles, `bytes_per_filter` and the medians over the rounds of
the smoother's own `stats` (CUDA-event times of the first forward pass, the re-forward with history and the backward
passes) and of the wall time of `run`, plus the card's name, power limit and maximum SM clock (nvidia-smi, read only).
The smoothed results of the two layouts are compared bit for bit on the first round.  Nothing is written to disk.

  python scripts/msckf_long_smoothing_bench.py [--filters 10000] [--steps 128] [--segment 64] [--rounds 2]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from msckf_rts_bench import DT, FEATURE_KIND, QUATS, SIGMA, initial_state, observation  # noqa: E402
from ragged_rts_bench import gpu_card  # noqa: E402


def make_stream(folder, B, T, dev):
  """z [T, B, 20] and the triangulated landmarks [T, B, 3] of T frames, from a forward pass of their own."""
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.features import FeatureFrontend, to_c_matrix
  from rednose_b200.filters.msckf import MsckfKalman
  g = torch.Generator(device=dev)
  g.manual_seed(77)
  x0, P0 = initial_state(B, dev, g)
  P0 = P0.expand(B, -1, -1)              # [B, EDIM, EDIM]: the smoothers slice it by tile
  eng = BatchedEKF(folder, "msckf", MsckfKalman.Q, x0, P0, device=dev, quaternion_idxs=QUATS)
  fe = FeatureFrontend(10)
  to_c = torch.as_tensor(to_c_matrix().reshape(9)).to(dev)
  Rk = torch.eye(20, dtype=torch.float64, device=dev) * SIGMA**2
  zs = torch.empty(T, B, 20, dtype=torch.float64, device=dev)
  eas = torch.empty(T, B, 3, dtype=torch.float64, device=dev)
  for k in range(T):
    z = observation(eng, B, g)
    pos, _, _ = fe.compute_pos_batch(to_c, eng.x[:, 23:].contiguous(), z, fallback_depth=30.0)
    zs[k], eas[k] = z, pos
    eng.predict_and_update_batch(DT * (k + 1), FEATURE_KIND, z, Rk, pos, augment=True)
  assert bool(torch.isfinite(eng.x).all()), "the MSCKF diverged while generating the stream"
  del eng
  return x0, P0, zs, eas, Rk


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=10000)
  ap.add_argument("--steps", type=int, default=128)
  ap.add_argument("--segment", type=int, default=64)
  ap.add_argument("--rounds", type=int, default=2)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("msckf_long_smoothing_bench needs a CUDA device")
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.msckf import DIM, EDIM, MsckfKalman
  from rednose_b200.smoothing import CheckpointedSmoother
  B, T, dev = a.filters, a.steps, torch.device("cuda:0")
  folder = ensure_generated(MsckfKalman)
  x0, P0, zs, eas, Rk = make_stream(folder, B, T, dev)

  def obs_fn(k, lo, hi):
    return DT * (k + 1), FEATURE_KIND, zs[k, lo:hi].clone(), Rk, eas[k, lo:hi], True

  smoothers = {m: CheckpointedSmoother(folder, "msckf", MsckfKalman.Q, DIM, EDIM, quaternion_idxs=QUATS, device=dev,
                                       segment=a.segment, main_pred=(m == "main_pred")) for m in ("full", "main_pred")}
  res = {m: {"forward_ms": [], "reforward_with_history_ms": [], "backward_ms": [], "run_s": []} for m in smoothers}
  info = {}
  check = {}
  for r in range(a.rounds + 1):                     # round 0 warms up both layouts
    for m in (list(smoothers) if r % 2 == 0 else list(reversed(list(smoothers)))):
      sm = smoothers[m]
      # one filter's smoothed track (first and last filter) is kept on the first round to compare the layouts
      keep = {} if r == 0 else None

      def sink(lo, hi, k0, xs, Ps, keep=keep):
        if keep is not None:
          for b in (0, B - 1):
            if lo <= b < hi:
              keep[(b, k0)] = (xs[:, b - lo].clone(), Ps[:, b - lo].clone())

      torch.cuda.synchronize()
      t0 = time.perf_counter()
      tiles = sm.run(x0, P0, T, obs_fn, sink, norm_quats=True, t0=0.0)
      torch.cuda.synchronize()
      wall = time.perf_counter() - t0
      sm._engine = sm._hist = sm._ck = sm._term = None      # release this layout's buffers before the other one runs
      torch.cuda.empty_cache()
      if r == 0:
        check[m] = keep
        info[m] = {"tiles": tiles, "tile_filters": sm.stats["tile_filters"], "segments": sm.stats["segments"],
                   "bytes_per_filter": sm.stats["bytes_per_filter"]}
      else:
        for key in ("forward_ms", "reforward_with_history_ms", "backward_ms"):
          res[m][key].append(sm.stats[key])
        res[m]["run_s"].append(wall)
  same = check["full"].keys() == check["main_pred"].keys() and all(
    torch.equal(check["full"][k][0], check["main_pred"][k][0]) and torch.equal(check["full"][k][1], check["main_pred"][k][1])
    for k in check["full"])
  card = gpu_card()
  line = {"filters": B, "steps": T, "segment": a.segment, "rounds": a.rounds, "bit_identical": bool(same)}
  for m in smoothers:
    line[m] = dict(info[m], **{k: round(statistics.median(v), 3) for k, v in res[m].items()},
                   run_s_all=[round(v, 3) for v in res[m]["run_s"]])
  line.update(card=card[0], power_limit=card[1], max_sm_clock=card[2])
  print(json.dumps(line))


if __name__ == "__main__":
  main()
