"""RTS smoothing of the shipped MSCKF (DIM 93 / EDIM 82, main block 23 / 22, ten pose clones) over recorded histories.

Workload: B msckf filters (default 10 000), T steps (default 16) of the config-5 camera-frame step of bench.py's msckf
workload: a device-generated observation of a new landmark from the ten clones (5 % gross outliers), triangulated by
the feature front-end, then the fused predict + gated feature update + clone-window shift, recorded with
`step_recorded(17, ..., augment=True)` (the history holds the estimate before the shift).  Then the backward pass, one
`rts_smooth(History)` launch, which smooths the 22-wide main block (ekf_sym.py:651-690):

* in place: the smoothed estimate overwrites x_{k|k} / P_{k|k}; outside the main block P_{k|k} already is the result;
* out=: into preallocated buffers, which first receive a copy of P_{k|k} (rows 0 .. T-2) and then the main blocks.

Each round records the history again and smooths it one way; the two modes alternate, and the first round of each warms
up.  Forward: CUDA events around each recording step (the observation is generated outside them), ms per step.
Backward: wall time between two device synchronisations.  Reported (one JSON line): medians over the rounds, backward
filter-steps/s (T - 1 recursion steps per filter), the algorithmic bytes of one backward step computed from the shapes
and the bandwidth they give, `History.bytes()`, and the card's name, power limit and maximum SM clock (nvidia-smi, read
only).  Nothing is written to disk.

  python scripts/msckf_rts_bench.py [--filters 10000] [--steps 16] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from ragged_rts_bench import gpu_card, timed  # noqa: E402

FEATURE_KIND, DT, SPEED, SIGMA = 17, 0.05, 10.0, 1e-3
QUATS = [3] + [26 + 7 * c for c in range(10)]   # main and clone attitudes


def step_bytes(dim, edim, medim):
  """Bytes one backward step must move: in place it reads P_{k+1|k} and P_{k|k} and writes P_{k|N} on the main block,
  reads x_{k|k} and x_{k+1|k}, writes x_{k|N} and reads one time; out of place it also copies the rest of P_{k|k}."""
  in_place = 8 * (3 * medim * medim + 3 * dim + 1)
  return in_place, in_place + 16 * (edim * edim - medim * medim)


def quat2rot(q):
  w, x, y, z = q.unbind(-1)
  return torch.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (w * y + x * z),
                      2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
                      2 * (x * z - w * y), 2 * (w * x + y * z), w * w - x * x - y * y + z * z], -1).reshape(q.shape[:-1] + (3, 3))


def initial_state(B, dev, g):
  """bench.py's msckf start: driving forward at 10 m/s, a camera frame every 0.05 s, clones 0.5 m apart."""
  from rednose_b200.filters.msckf import MsckfKalman
  f64 = dict(dtype=torch.float64, device=dev)
  x0 = torch.as_tensor(MsckfKalman.initial_x).to(dev).repeat(B, 1)
  q = torch.randn(B, 4, generator=g, **f64)
  q = q / q.norm(dim=1, keepdim=True)
  Rm = quat2rot(q)
  x0[:, 0:3] += torch.randn(B, 3, generator=g, **f64) * 100.0
  x0[:, 3:7] = q
  x0[:, 7:10] = Rm[:, :, 0] * SPEED
  for c in range(10):
    o = 23 + 7 * c
    x0[:, o:o + 3] = x0[:, 0:3] - Rm[:, :, 0] * (SPEED * DT) * (10 - c)
    x0[:, o + 3:o + 7] = q
  pd = np.concatenate([[25.0] * 3 + [0.05**2] * 3 + [1.0] * 3 + [0.1**2] * 3 + [0.01**2] * 3 + [0.01**2] + [0.5**2] * 3
                       + [0.01**2] * 3] + [[1.0] * 3 + [0.02**2] * 3] * 10)
  return x0, torch.as_tensor(np.diag(pd)).to(dev)


def observation(eng, B, g):
  """A landmark 15-50 m ahead of the newest clone seen from the ten clones (+ noise, 5 % gross outliers), as bench.py."""
  f64 = dict(dtype=torch.float64, device=eng.x.device)
  clones = eng.x[:, 23:].reshape(B, 10, 7)
  local = torch.stack([torch.rand(B, generator=g, **f64) * 35 + 15, torch.rand(B, generator=g, **f64) * 10 - 5,
                       torch.rand(B, generator=g, **f64) * 6 - 3], 1)
  point = clones[:, 9, 0:3] + torch.einsum('bij,bj->bi', quat2rot(clones[:, 9, 3:7]), local)
  pc = torch.einsum('bcji,bcj->bci', quat2rot(clones[:, :, 3:7]), point[:, None, :] - clones[:, :, 0:3])
  z = torch.stack([pc[:, :, 1] / pc[:, :, 0], pc[:, :, 2] / pc[:, :, 0]], -1).reshape(B, 20)
  noise = torch.randn(B, 20, generator=g, **f64) * SIGMA
  noise[torch.rand(B, generator=g, device=eng.x.device) < 0.05] *= 50.0
  return (z + noise).contiguous()


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--filters", type=int, default=10000)
  ap.add_argument("--steps", type=int, default=16)
  ap.add_argument("--rounds", type=int, default=5)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("msckf_rts_bench needs a CUDA device")
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.features import FeatureFrontend, to_c_matrix
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import DIM_STATE_ERR as MEDIM
  from rednose_b200.filters.msckf import DIM, EDIM, MsckfKalman
  B, T, dev = a.filters, a.steps, torch.device("cuda:0")
  assert T >= 2
  hist_bytes = 8 * T * (B * (2 * DIM + 2 * EDIM * EDIM) + 1)
  out_bytes = 8 * T * B * (DIM + EDIM * EDIM)
  print(f"msckf_rts_bench: allocating {hist_bytes / 1e9:.1f} GB of history and {out_bytes / 1e9:.1f} GB of out= buffers",
        file=sys.stderr, flush=True)
  folder = ensure_generated(MsckfKalman)
  fe = FeatureFrontend(10)
  to_c = torch.as_tensor(to_c_matrix().reshape(9)).to(dev)
  g = torch.Generator(device=dev)
  g.manual_seed(77)
  x0, P0 = initial_state(B, dev, g)
  eng = BatchedEKF(folder, "msckf", MsckfKalman.Q, x0, P0, device=dev, quaternion_idxs=QUATS)
  Rk = torch.eye(20, dtype=torch.float64, device=dev) * SIGMA**2
  hist = eng.new_history(T)
  assert hist.bytes() == hist_bytes
  out = (torch.empty_like(hist.x_filt), torch.empty_like(hist.P_filt))
  kw = dict(norm_quats=True, quaternion_idxs=tuple(QUATS))

  def forward():
    eng.init_state(x0, P0)
    hist.n = 0
    ms = 0.0
    for k in range(T):
      z = observation(eng, B, g)
      pos, _, _ = fe.compute_pos_batch(to_c, eng.x[:, 23:].contiguous(), z, fallback_depth=30.0)
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      eng.step_recorded(hist, FEATURE_KIND, DT * (k + 1), z, Rk, ea=pos, augment=True)
      e1.record()
      e1.synchronize()
      ms += e0.elapsed_time(e1)
    assert bool(torch.isfinite(hist.P_filt).all()), "the MSCKF diverged while recording"
    return ms / T

  modes = {"in_place": dict(in_place=True), "out": dict(out=out)}
  res = {m: {"forward_ms_per_step": [], "backward_ms": []} for m in modes}
  for r in range(a.rounds + 1):                     # round 0 warms up every launch shape
    for m in (modes if r % 2 == 0 else reversed(list(modes))):
      f = forward()
      b = timed(lambda: eng.rts_smooth(hist, **kw, **modes[m]))
      if r:
        res[m]["forward_ms_per_step"].append(f)
        res[m]["backward_ms"].append(1e3 * b)
  card = gpu_card()
  bytes_in, bytes_out = step_bytes(DIM, EDIM, MEDIM)
  line = {"filters": B, "steps": T, "rounds": a.rounds, "history_bytes": hist.bytes(),
          "forward_ms_per_step": round(statistics.median(res["in_place"]["forward_ms_per_step"]
                                                         + res["out"]["forward_ms_per_step"]), 4)}
  for m, nbytes in (("in_place", bytes_in), ("out", bytes_out)):
    ms = statistics.median(res[m]["backward_ms"])
    line[m] = {"backward_ms": round(ms, 3), "backward_steps_per_s": round(B * (T - 1) / ms * 1e3),
               "bytes_per_step": nbytes, "achieved_GB_per_s": round(nbytes * B * (T - 1) / ms * 1e-6, 1),
               "backward_ms_all": [round(v, 3) for v in res[m]["backward_ms"]]}
  line.update(card=card[0], power_limit=card[1], max_sm_clock=card[2])
  print(json.dumps(line))


if __name__ == "__main__":
  main()
