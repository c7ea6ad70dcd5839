"""Per-kind launch time of the live pair kernel (ekf_step_pair) against the card's own read+write copy ceiling.

For each batch size the live filter is stepped with kinds 4, 10 and 12 separately: every launch is bracketed by CUDA
events (the observation refresh before it is not), and the mean over --iters launches after --warmup is reported with
its GB/s at the bytes a packed fused step moves.  The ceiling is `dst.copy_(src)` on two float64 tensors of about
--copy-gb each, counted as read + write, which is a 50/50 mix like the kernel's.  The card's name, power limit and
maximum SM clock are read in the same run.

  python scripts/pair_kernel_timing.py [--batch 1048576 100000] [--iters 50] [--out result.json]

Prints one JSON line.  Needs a GPU; it writes nothing unless --out is given.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
  sys.path.insert(0, REPO)

KINDS = (4, 10, 12)


def packed_step_bytes(dim, edim, m):
  """Bytes of one fused step with the packed covariance: P (lower block triangle) and x read and written, z and R read,
  y written, dt read (csrc/ekf_packed.cuh: EDIM / 2 block rows of 2x2 blocks)."""
  nb = edim // 2
  packed = 2 * nb * (nb + 1)
  return 8 * (2 * packed + 2 * dim + m + m * m + m + 1)


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else None
  except (OSError, subprocess.TimeoutExpired):
    return None


def time_events(fn, iters, warmup, pre=None):
  import torch
  for _ in range(warmup):
    if pre:
      pre()
    fn()
  torch.cuda.synchronize()
  ms = []
  for _ in range(iters):
    if pre:
      pre()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    ms.append(e0.elapsed_time(e1))
  return ms


def copy_ceiling(gb, iters, warmup):
  import torch
  n = int(gb * 1e9) // 8
  src = torch.rand(n, dtype=torch.float64, device="cuda")
  dst = torch.empty_like(src)
  ms = time_events(lambda: dst.copy_(src), iters, warmup)
  del src, dst
  torch.cuda.empty_cache()
  return 2 * n * 8 / (float(np.median(ms)) * 1e-3) / 1e9, float(np.median(ms))


def kernel_times(B, iters, warmup):
  import torch
  from bench import make_problem
  from rednose_b200.batched import BatchedEKF
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  dev = torch.device("cuda")
  lib_dir = ensure_generated(LiveKalman)
  x0, P0, Q, pools, (dim, edim), quat = make_problem("live", B, seed=1234, lib_dir=lib_dir)
  eng = BatchedEKF(lib_dir, "live", Q, x0, P0, device=dev, quaternion_idxs=quat)
  dt_arr = torch.full((B,), 0.01, dtype=torch.float64, device=dev)
  out = {}
  for k in KINDS:
    zp, R = (torch.as_tensor(v).to(dev) for v in pools[k])
    z = torch.empty(B, 1, zp.shape[-1], dtype=torch.float64, device=dev)
    ms = time_events(lambda: eng.step(k, dt_arr, z, R), iters, warmup, pre=lambda: z[:, 0, :].copy_(zp[0]))
    nbytes = packed_step_bytes(dim, edim, zp.shape[-1]) * B
    med = float(np.median(ms))
    out[str(k)] = {"ms_median": med, "ms_mean": float(np.mean(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)),
                   "GBps": nbytes / (med * 1e-3) / 1e9, "bytes_per_step": nbytes // B}
  assert bool(torch.isfinite(eng.x).all())
  del eng
  torch.cuda.empty_cache()
  return out


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--batch", type=int, nargs="+", default=[1 << 20, 100000])
  ap.add_argument("--iters", type=int, default=50)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--copy-gb", type=float, default=2.5, help="size of each copy tensor")
  ap.add_argument("--out", default=None, help="also write the JSON result to this file")
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit("pair_kernel_timing.py needs a CUDA device")
  ceil_GBps, ceil_ms = copy_ceiling(args.copy_gb, args.iters, args.warmup)
  res = {"card": card(), "device": torch.cuda.get_device_name(0),
         "copy_ceiling": {"GBps": ceil_GBps, "ms_median": ceil_ms, "bytes_per_tensor": int(args.copy_gb * 1e9) // 8 * 8},
         "batches": {}}
  for B in args.batch:
    kt = kernel_times(B, args.iters, args.warmup)
    for v in kt.values():
      v["frac_of_copy_ceiling"] = v["GBps"] / ceil_GBps
    res["batches"][str(B)] = kt
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, "w", encoding="utf-8") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
