"""nvcc build driver for generated filter libraries and the runtime library.

Stands in for the reference's SCons tool (site_scons/site_tools/rednose_filter.py:27-37:
run the generator, then link ``lib{target}.so``) with a direct nvcc invocation for
sm_90a.  Everything is built in-tree.
"""
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
INCLUDE_DIR = os.path.abspath(os.path.join(PKG_DIR, "..", "include"))
GENERATED_DIR = os.environ.get("REDNOSE_B200_GENERATED_DIR") or os.path.join(PKG_DIR, "generated")

NVCC_FLAGS = [
  "-gencode", "arch=compute_90a,code=sm_90a",
  "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
  "-Xcompiler", "-fPIC", "-shared",
]


def nvcc_path():
  p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  if not os.path.exists(p):
    raise RuntimeError("nvcc not found: rednose_b200 needs the CUDA toolkit to build filter libraries")
  return p


def _newer(target, sources):
  if not os.path.exists(target):
    return False
  t = os.path.getmtime(target)
  return all(os.path.getmtime(s) <= t for s in sources if os.path.exists(s))


def csrc_sources():
  # what a generated filter library depends on (the runtime library is built separately)
  return [os.path.join(CSRC_DIR, f) for f in sorted(os.listdir(CSRC_DIR)) if f != "runtime.cc"] + [os.path.join(INCLUDE_DIR, "rednose_b200.h")]


def compile_filter(folder, name, force=False, verbose=False):
  """``{folder}/{name}.cu`` -> ``{folder}/lib{name}.so`` (sm_90a)."""
  src = os.path.join(folder, f"{name}.cu")
  lib = os.path.join(folder, f"lib{name}.so")
  if not force and _newer(lib, [src] + csrc_sources()):
    return lib
  import fcntl
  with open(os.path.join(folder, f".{name}.lock"), "w") as lock:   # concurrent builders (one process per GPU) serialise here
    fcntl.flock(lock, fcntl.LOCK_EX)
    if not force and _newer(lib, [src] + csrc_sources()):
      return lib
    return _compile_filter_locked(folder, name, src, lib, verbose)


def _compile_filter_locked(folder, name, src, lib, verbose):
  tmp = lib + f".tmp{os.getpid()}"
  cmd = [nvcc_path()] + NVCC_FLAGS + ["-Xptxas", "-v", f"-I{CSRC_DIR}", f"-I{INCLUDE_DIR}", "-o", tmp, src]
  res = subprocess.run(cmd, capture_output=True, text=True)
  with open(os.path.join(folder, f"{name}.ptxas.log"), "w", encoding="utf-8") as f:
    f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
  if res.returncode != 0:
    raise RuntimeError(f"nvcc failed for {src}:\n{res.stderr[-4000:]}")
  os.replace(tmp, lib)   # atomic: a reader never sees a half-written library
  if verbose:
    print(res.stderr)
  return lib


def compile_runtime(force=False):
  """csrc/runtime.cc -> rednose_b200/librednose_b200.so (registry + native driver)."""
  src = os.path.join(CSRC_DIR, "runtime.cc")
  lib = os.path.join(PKG_DIR, "librednose_b200.so")
  deps = [src, os.path.join(INCLUDE_DIR, "rednose_b200.h")]
  if not force and _newer(lib, deps):
    return lib
  import fcntl
  with open(os.path.join(PKG_DIR, ".runtime.lock"), "w") as lock:   # one process per GPU: ranks serialise here
    fcntl.flock(lock, fcntl.LOCK_EX)
    if not force and _newer(lib, deps):
      return lib
    cxx = shutil.which("g++") or "g++"
    tmp = lib + f".tmp{os.getpid()}"
    cmd = [cxx, "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", f"-I{INCLUDE_DIR}", "-o", tmp, src, "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
      raise RuntimeError(f"g++ failed for {src}:\n{res.stderr[-4000:]}")
    os.replace(tmp, lib)   # atomic: a concurrent dlopen never sees a half-written library
  return lib
