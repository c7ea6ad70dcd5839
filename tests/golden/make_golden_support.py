#!/usr/bin/env python3
"""Golden data for tests/test_support_cpu.py and tests/test_dropin_cpu.py, from the REFERENCE ITSELF (run where the
reference is present; its location is oracle.build_ref.REF, overridable with REDNOSE_REFERENCE).

Stores, in tests/golden/support_reference.npz:
  chi2_p, chi2_interp[dim, i]  np.interp(chi2_p[i], arange(.01, .99, .01), chi2_lookup_table.npy[dim]) of the
                               reference's shipped table, for every dim of the table (row 0 unused)
  sym_<name>                   srepr of the reference's sympy_helpers.<name> on the symbols the test uses
and, in tests/golden/dropin_reference.json, what the reference's unmodified examples/<name>_kf.py generate through this
package's gen_code: the SHA-256 of their sorted `void ` prototypes and their F / kind sparsity signature.
"""
import hashlib
import importlib.util
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import sympy as sp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
from oracle.build_ref import REF  # noqa: E402

CHI2_P = np.array([0.5, 0.9, 0.95, 0.975, 0.123])


def main():
  t = np.load(os.path.join(REF, "rednose", "helpers", "chi2_lookup_table.npy"))
  grid = np.arange(.01, .99, .01)
  interp = np.array([[np.interp(p, grid, t[dim]) for p in CHI2_P] for dim in range(t.shape[0])])
  spec = importlib.util.spec_from_file_location("ref_sympy_helpers", os.path.join(REF, "rednose", "helpers", "sympy_helpers.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  r, p, y = sp.symbols("r p y")
  q = sp.symbols("q0:4")
  out = {"chi2_p": CHI2_P, "chi2_interp": interp}
  for name, args in (("euler_rotate", (r, p, y)), ("quat_rotate", q), ("quat_matrix_r", (q,)), ("quat_matrix_l", (q,))):
    out[f"sym_{name}"] = np.array(sp.srepr(sp.Matrix(getattr(mod, name)(*args))))
  np.savez_compressed(os.path.join(HERE, "support_reference.npz"), **out)
  dropin = {}
  for name in ("kinematic", "live"):
    with tempfile.TemporaryDirectory() as d:
      env = dict(os.environ, PYTHONPATH=REPO, REDNOSE_B200_NO_COMPILE="1")   # `rednose` resolves to this package's shim
      subprocess.run([sys.executable, os.path.join(REF, "examples", f"{name}_kf.py"), name, d], check=True, env=env, cwd=d)
      dropin[name] = {"protos_sha256": protos_sha256(os.path.join(d, f"{name}.h")), "sig": sparsity_sig(os.path.join(d, f"{name}.cu"))}
  with open(os.path.join(HERE, "dropin_reference.json"), "w", encoding="utf-8") as f:
    json.dump(dropin, f)


def protos_sha256(header):
  with open(header, encoding="utf-8") as f:
    protos = sorted(re.sub(r"\s+", " ", ln) for ln in f.read().split("\n") if ln.startswith("void "))
  return hashlib.sha256("\n".join(protos).encode()).hexdigest()


def sparsity_sig(src):
  with open(src, encoding="utf-8") as f:
    return re.findall(r"static constexpr int (?:NF|KIND) = [^;]*;", f.read())


if __name__ == "__main__":
  main()
