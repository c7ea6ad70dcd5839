"""Resources of the live pair kernel (ekf_step_pair), cross-compiled for sm_90a without a GPU.

The kernel runs 8 one-warp CTAs per SM, which needs at most 255 registers per thread (8 x 32 x 255 = 65 280 of the SM's
65 536) and at most (228 KiB - 8 x 1 KiB reserved) / 8 = 28 160 bytes of shared memory per CTA, in both covariance
layouts: the packed layout spends what its smaller tiles save on a second tile slot.  The small spill frames are pinned at
what nvcc 12.9 gives today, so that a change which grows them is noticed (DESIGN.md section 4.2b).
"""
import os
import re
import subprocess

import pytest

SMEM_PER_CTA = (228 * 1024 - 8 * 1024) // 8
LIVE_FUSED_KINDS = (3, 4, 9, 10, 12, 13, 14, 19)
# (stack, spill stores, spill loads) in bytes, at most, of the fused packed non-gather instantiations bench.py runs
PINNED = {4: (48, 8, 8), 10: (96, 56, 56), 12: (8, 8, 8)}
ANY = (96, 52, 76)   # every other fused live instantiation (full layout, gather lists)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
  from rednose_b200 import build
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.live import LiveKalman
  folder = ensure_generated(LiveKalman)
  tmp = tmp_path_factory.mktemp("pair_res")
  src = tmp / "sizes.cu"
  src.write_text(
    f'#include "{os.path.join(folder, "live.cu")}"\n'
    "#include <cstdio>\n"
    "template <class K> void show(int k) {\n"
    "  printf(\"%d %zu %zu\\n\", k, rnb::pair_smem_bytes<live_model, K, rnb::PAIR_GROUP, true>(),\n"
    "         rnb::pair_smem_bytes<live_model, K, rnb::PAIR_GROUP, false>());\n"
    "}\n"
    "int main() {\n" + "".join(f"  show<live_kind_{k}>({k});\n" for k in LIVE_FUSED_KINDS) + "  return 0;\n}\n")
  exe = tmp / "sizes"
  cmd = [build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
         "-Xptxas", "-v", f"-I{build.CSRC_DIR}", f"-I{build.INCLUDE_DIR}", "-o", str(exe), str(src)]
  res = subprocess.run(cmd, capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  sizes = {}
  for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n"):
    if line.strip():
      k, packed, full = (int(v) for v in line.split())
      sizes[k] = (packed, full)
  return res.stdout + res.stderr, sizes


def _pair_kernels(log):
  """{(kind, gather, packed): (registers, stack, spill stores, spill loads)} of the fused live ekf_step_pair."""
  out = {}
  for block in re.split(r"Compiling entry function '", log)[1:]:
    name = block.split("'")[0]
    m = re.match(r"_ZN3rnb13ekf_step_pairI10live_model\d+live_kind_(\d+)Lb1ELb1ELi16ELb([01])ELb([01])E", name)
    if not m:
      continue
    regs = re.search(r"Used (\d+) registers", block)
    st = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
    out[(int(m.group(1)), m.group(2) == "1", m.group(3) == "1")] = (int(regs.group(1)),) + tuple(int(v) for v in st.groups())
  return out


def test_fused_live_pair_kernels_fit_8_warps_per_sm(compiled):
  k = _pair_kernels(compiled[0])
  assert sorted({kind for kind, _, _ in k}) == list(LIVE_FUSED_KINDS)
  assert len(k) == 4 * len(LIVE_FUSED_KINDS)
  for key, (regs, stack, st, ld) in k.items():
    assert regs <= 255, (key, regs)
    kind, gather, packed = key
    lim = PINNED[kind] if (packed and not gather and kind in PINNED) else ANY
    assert stack <= lim[0] and st <= lim[1] and ld <= lim[2], (key, (stack, st, ld), lim)


def test_pair_scratch_fits_8_ctas_per_sm(compiled):
  sizes = compiled[1]
  assert sorted(sizes) == list(LIVE_FUSED_KINDS)
  for kind, (packed, full) in sizes.items():
    assert packed <= SMEM_PER_CTA and full <= SMEM_PER_CTA, (kind, packed, full, SMEM_PER_CTA)
