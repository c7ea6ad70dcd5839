"""Loading of generated filter libraries (mirror of rednose/helpers/__init__.py:9-35).

``load_code`` keeps the reference contract: parse ``{folder}/{name}.h`` keeping only the
lines that start with ``void `` (the only thing cffi's cdef can digest without a
preprocessor) and ``dlopen`` ``{folder}/lib{name}.so``.  The generated header also carries the
batched ``<name>_batch_*`` prototypes in the same single-line form, so the very same call
exposes them.
"""
import os
import platform

from cffi import FFI

from rednose_b200.build import CSRC_DIR as TEMPLATE_DIR  # kernels play the role of the C templates


class KalmanError(Exception):
  pass


def write_code(folder, name, code, header):
  os.makedirs(folder, exist_ok=True)
  with open(os.path.join(folder, f"{name}.cu"), 'w', encoding='utf-8') as f:
    f.write(code)
  with open(os.path.join(folder, f"{name}.h"), 'w', encoding='utf-8') as f:
    f.write(header)


def load_code(folder, name):
  ext = "dylib" if platform.system() == "Darwin" else "so"
  lib_path = os.path.join(folder, f"lib{name}.{ext}")
  with open(os.path.join(folder, f"{name}.h"), encoding='utf-8') as f:
    text = f.read()
  protos = [ln for ln in text.split("\n") if ln.startswith("void ") and not ln.startswith("void* ")]
  ffi = FFI()
  status_proto = f"int {name}_cuda_status(void);"
  ffi.cdef("\n".join(protos) + ("\n" + status_proto + "\n" if status_proto in text else "\n"))
  if not os.path.exists(lib_path):
    raise FileNotFoundError(f"{lib_path} is missing: run the filter's generator (gen_code) first")
  return ffi, ffi.dlopen(lib_path)


def raise_on_cuda_error(lib, name, what=""):
  try:
    status_fn = getattr(lib, f"{name}_cuda_status")
  except AttributeError:  # a library without the CUDA status hook (e.g. a CPU build of the same C-ABI in tests)
    return
  status = status_fn()
  if status != 0:
    raise RuntimeError(f"rednose_b200: CUDA error {status} in {name} {what} (no CPU fallback exists; an H100 is required)")
