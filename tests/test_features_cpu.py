"""MSCKF front-end (SURVEY.md section 8f-3) on CPU: the oracle's restatement of rednose/templates/compute_pos.c and
feature_handler.c pinned by domain properties (the reference holds no test or fixture for these templates), the
generated per-pose residual + the kernels' Gauss-Newton / merge code compiled for the HOST against that oracle, and the
C-ABI of libfeatures_<K>.so (load + symbols only; no compute without a GPU)."""
import os
import subprocess

import numpy as np
import pytest
from cffi import FFI

from rednose_b200.features import N_FEATURES, N_TRACKS, ensure_features, to_c_matrix
from rednose_b200.geometry import quat2rot

K = 10


@pytest.fixture(scope="module")
def feat_oracle():
  from oracle import build_ref
  if build_ref.reference_available():
    build_ref.build_features(K)
  lib = os.path.join(build_ref.OUT, f"libfeatures_{K}.so")
  if not os.path.exists(lib):
    pytest.skip("oracle/_ref/libfeatures not built and the reference checkout is not present")
  ffi = FFI()
  with open(os.path.join(build_ref.OUT, f"features_{K}.h"), encoding="utf-8") as f:
    ffi.cdef(f.read())
  return ffi, ffi.dlopen(lib)


def synth_tracks(B, seed=0, noise=0.0):
  """K camera poses along a short forward track + one point 10-50 m ahead; image positions = its projections."""
  rng = np.random.default_rng(seed)
  to_c = to_c_matrix()
  poses = np.zeros((B, K, 7))
  q0 = rng.normal(size=(B, 4)); q0 /= np.linalg.norm(q0, axis=1, keepdims=True)
  p0 = rng.normal(0, 100.0, (B, 3)) + np.array([-2.7e6, -4.26e6, 3.88e6])
  R0 = quat2rot(q0)
  for i in range(K):
    q = q0 + rng.normal(0, 0.01, (B, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    poses[:, i, 3:7] = q
    poses[:, i, 0:3] = p0 + R0[:, :, 0] * 0.8 * i + rng.normal(0, 0.05, (B, 3))
  local = np.stack([rng.uniform(10, 50, B), rng.uniform(-5, 5, B), rng.uniform(-3, 3, B)], 1)
  point = poses[:, K - 1, 0:3] + np.einsum('bij,bj->bi', quat2rot(poses[:, K - 1, 3:7]), local)
  img = np.zeros((B, K, 2))
  for i in range(K):
    cam = np.einsum('ij,bjk,bk->bi', to_c, np.transpose(quat2rot(poses[:, i, 3:7]), (0, 2, 1)), point - poses[:, i, 0:3])
    img[:, i, 0], img[:, i, 1] = cam[:, 0] / cam[:, 2], cam[:, 1] / cam[:, 2]
  img += rng.normal(0, noise, img.shape) if noise else 0.0
  return to_c, poses.reshape(B, 7 * K), img.reshape(B, 2 * K), point


def oracle_compute_pos(fo, to_c, poses, img):
  ffi, lib = fo
  B = poses.shape[0]
  pos, param = np.zeros((B, 3)), np.zeros((B, 3))
  p = lambda a: ffi.cast("double *", a.ctypes.data)
  tc = np.ascontiguousarray(to_c)
  for b in range(B):
    lib.compute_pos(p(tc), p(poses[b]), p(img[b]), p(param[b]), p(pos[b]))
  return pos, param


def test_oracle_triangulation_recovers_the_point(feat_oracle):
  to_c, poses, img, point = synth_tracks(64, seed=1)
  pos, param = oracle_compute_pos(feat_oracle, to_c, poses, img)
  # exact projections; the reference stops as soon as |delta|^2 <= 1e-4 in (alpha, beta, 1/depth) units (compute_pos.c:18),
  # so the last (quadratically small) correction is what remains: decimetres at 10-50 m range
  err = np.linalg.norm(pos - point, axis=1)
  assert err.max() < 1.0 and np.median(err) < 0.2
  ffi, lib = feat_oracle
  p = lambda a: ffi.cast("double *", a.ctypes.data)
  for b in range(8):                                                  # one more Gauss-Newton step from the result is tiny, and lands on the point
    res, jac = np.zeros(2 * K), np.zeros(6 * K)
    lib.res_fun(p(param[b]), p(poses[b]), p(img[b]), p(res)); lib.jac_fun(p(param[b]), p(poses[b]), p(img[b]), p(jac))
    J = jac.reshape(2 * K, 3)
    d = np.linalg.solve(J.T @ J, J.T @ res)
    assert np.linalg.norm(d) < 1e-2 and np.max(np.abs(res)) < 5e-3
    x2 = param[b] - d
    P = poses[b].reshape(K, 7)
    cam = np.array([x2[0] / x2[2], x2[1] / x2[2], 1 / x2[2]])
    assert np.linalg.norm(quat2rot(P[K - 1, 3:7]) @ to_c.T @ cam + P[K - 1, 0:3] - point[b]) < 0.05 * max(1.0, err[b] * 10)


def test_oracle_noisy_tracks_stationary_point(feat_oracle):
  to_c, poses, img, point = synth_tracks(32, seed=2, noise=2e-3)
  pos, param = oracle_compute_pos(feat_oracle, to_c, poses, img)
  ffi, lib = feat_oracle
  p = lambda a: ffi.cast("double *", a.ctypes.data)
  for b in range(32):   # Gauss-Newton stops on |delta|^2 <= 1e-4 (compute_pos.c:18): the gradient is small, not zero
    res, jac = np.zeros(2 * K), np.zeros(6 * K)
    lib.res_fun(p(param[b]), p(poses[b]), p(img[b]), p(res)); lib.jac_fun(p(param[b]), p(poses[b]), p(img[b]), p(jac))
    J = jac.reshape(2 * K, 3)
    assert np.linalg.norm(np.linalg.solve(J.T @ J, J.T @ res)) < 1e-2
  assert np.median(np.linalg.norm(pos - point, axis=1)) < 5.0


def py_sane(track):
  dx = [abs(track[i + 2][2] - track[i + 1][2]) for i in range(K - 1)]
  dy = [abs(track[i + 2][3] - track[i + 1][3]) for i in range(K - 1)]
  for i in range(1, K - 1):
    if (((dx[i] > 0.05 or dx[i - 1] > 0.05) and (dx[i] > 2 * dx[i - 1] or dx[i] < .5 * dx[i - 1])) or
        ((dy[i] > 0.05 or dy[i - 1] > 0.05) and (dy[i] > 2 * dy[i - 1] or dy[i] < .5 * dy[i - 1]))):
      return False
  return True


def py_merge(tracks, features, empty_idxs):
  """Straight transcription of rednose/templates/feature_handler.c:23-56."""
  e = 0
  for i in range(features.shape[0]):
    m = int(features[i, 4])
    if tracks[m, 0, 1] == m and tracks[m, 0, 2] == 0:
      tracks[m, 0, 0] += 1; tracks[m, 0, 1] = features[i, 1]; tracks[m, 0, 2] = 1
      idx = int(tracks[m, 0, 0])
      tracks[m, idx] = features[i]
      if idx == K:
        tracks[m, 0, 3] = 1
        if py_sane(tracks[m]):
          tracks[m, 0, 4] = 1
    else:
      s = empty_idxs[e]
      tracks[s, 0, 0] = 1; tracks[s, 0, 1] = features[i, 1]; tracks[s, 0, 2] = 1
      tracks[s, 1] = features[i]
      e += 1
  return tracks


def synth_frame(nt, nf, seed, smooth=True, collide=False):
  """A track table with live tracks of random length (header: count, own id, 0, 0, 0), empty slots, and a frame of
  features: most extend a live track, some are duplicates of one, the rest start new tracks."""
  rng = np.random.default_rng(seed)
  tracks = np.zeros((nt, K + 1, 5))
  live = rng.choice(np.arange(1, nt), size=nt // 2, replace=False)
  for t in live:
    n = rng.integers(1, K)           # rows already filled: 1 .. K-1
    tracks[t, 0, 0], tracks[t, 0, 1] = n, t
    step = rng.uniform(0.0, 0.08, 2)
    base = rng.uniform(-0.5, 0.5, 2)
    for r in range(1, n + 1):
      jitter = 0.0 if smooth else rng.normal(0, 0.05, 2)
      tracks[t, r] = [rng.integers(1, 1e6), t, base[0] + step[0] * r + (jitter if smooth else jitter[0]), base[1] + step[1] * r + (0.0 if smooth else jitter[1]), t]
  empty = np.setdiff1d(np.arange(nt), live)
  empty = empty[empty != 0]
  feats = np.zeros((nf, 5))
  for i in range(nf):
    u = rng.random()
    if u < 0.6:
      t = rng.choice(live)
      n = int(tracks[t, 0, 0])
      feats[i] = [i + 1, 10_000_000 + i, tracks[t, n, 2] + 0.04 + (0 if smooth else rng.normal(0, 0.06)), tracks[t, n, 3] + 0.02, t]
    else:
      feats[i] = [i + 1, 10_000_000 + i, rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.choice(empty) if u > 0.9 else 0]
  empty_idxs = rng.permutation(empty)[:nf].astype(np.int64)
  if collide:   # a new track lands on a live track that a LATER feature wants to extend -> order matters
    tgt = int(feats[nf - 1, 4]) if feats[nf - 1, 4] in live else int(live[0])
    feats[nf - 1, 4] = tgt
    empty_idxs[0] = tgt
  if len(empty_idxs) < nf:
    empty_idxs = np.concatenate([empty_idxs, np.full(nf - len(empty_idxs), empty[0], dtype=np.int64)])
  return tracks, feats, empty_idxs


@pytest.mark.parametrize("smooth,collide", [(True, False), (False, False), (True, True)])
def test_oracle_merge_features_equals_transcription(feat_oracle, smooth, collide):
  ffi, lib = feat_oracle
  for seed in range(4):
    tracks, feats, empty = synth_frame(200, 90, seed, smooth, collide)
    want = py_merge(tracks.copy(), feats, empty)
    got = tracks.copy()
    lib.merge_features_n(ffi.cast("double *", got.ctypes.data), ffi.cast("double *", feats.ctypes.data), ffi.cast("long long *", empty.ctypes.data), 90, 200)
    assert np.array_equal(got, want)
    assert (want[:, 0, 3] == 1).sum() > 0                       # some tracks completed ...
    assert 0 < (want[:, 0, 4] == 1).sum() or not smooth         # ... and passed sane() when the motion is smooth


HOST_HARNESS = r"""
#include "%(src)s"
extern "C" void host_compute_pos(const double* to_c, const double* poses, const double* img, double* param, double* pos, int* iters, long long B) {
  constexpr int K = feature_model::K;
  for (long long b = 0; b < B; ++b) {
    const double* mi = img + b * 2 * K;
    double x[3] = {mi[2 * K - 2], mi[2 * K - 1], 0.1};
    iters[b] = rnb::gauss_newton_track<feature_model>(poses + b * 7 * K, 1, mi, 1, x);
    rnb::camera_to_ecef(to_c, poses + b * 7 * K + (K - 1) * 7, 1, x, pos + b * 3);
    for (int i = 0; i < 3; ++i) param[b * 3 + i] = x[i];
  }
}
extern "C" void host_merge(double* tracks, const double* feats, const long long* empty_idxs, int nf, int nt) {
  int e = 0;
  for (int i = 0; i < nf; ++i) e += rnb::merge_one<feature_model::K>(tracks, feats + i * 5, empty_idxs, e, nt);
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
  """The generated pose_term + the kernels' own Gauss-Newton / merge_one code, compiled by nvcc for the HOST."""
  from rednose_b200 import build
  folder = ensure_features(K)
  d = tmp_path_factory.mktemp("feat_host")
  src = d / "harness.cu"
  src.write_text(HOST_HARNESS % dict(src=os.path.join(folder, f"features_{K}.cu")))
  lib = d / "libharness.so"
  subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
                  f"-I{build.CSRC_DIR}", f"-I{build.INCLUDE_DIR}", "-o", str(lib), str(src)], check=True)
  ffi = FFI()
  ffi.cdef("void host_compute_pos(const double*, const double*, const double*, double*, double*, int*, long long);"
           "void host_merge(double*, const double*, const long long*, int, int);")
  return ffi, ffi.dlopen(str(lib))


def test_generated_pose_term_and_gauss_newton_match_the_oracle(feat_oracle, host_lib):
  ffi, lib = host_lib
  for noise in (0.0, 2e-3):
    to_c, poses, img, _ = synth_tracks(200, seed=7, noise=noise)
    pos_r, param_r = oracle_compute_pos(feat_oracle, to_c, poses, img)
    pos, param, iters = np.zeros((200, 3)), np.zeros((200, 3)), np.zeros(200, dtype=np.int32)
    c = lambda a: ffi.cast("const double *", a.ctypes.data)
    lib.host_compute_pos(c(np.ascontiguousarray(to_c)), c(poses), c(img), ffi.cast("double *", param.ctypes.data), ffi.cast("double *", pos.ctypes.data),
                         ffi.cast("int *", iters.ctypes.data), 200)
    assert np.max(np.abs(param - param_r) / np.max(np.abs(param_r))) < 1e-9
    assert np.max(np.abs(pos - pos_r)) / np.max(np.abs(pos_r)) < 1e-12
    assert iters.min() >= 1 and iters.max() <= 30


def test_merge_one_in_order_equals_the_oracle(feat_oracle, host_lib):
  ffi, lib = host_lib
  fo_ffi, fo = feat_oracle
  for seed, collide in ((0, False), (1, True)):
    tracks, feats, empty = synth_frame(300, 120, seed, True, collide)
    want = tracks.copy()
    fo.merge_features_n(fo_ffi.cast("double *", want.ctypes.data), fo_ffi.cast("double *", feats.ctypes.data), fo_ffi.cast("long long *", empty.ctypes.data), 120, 300)
    got = tracks.copy()
    lib.host_merge(ffi.cast("double *", got.ctypes.data), ffi.cast("const double *", feats.ctypes.data), ffi.cast("const long long *", empty.ctypes.data), 120, 300)
    assert np.array_equal(got, want)


def test_features_library_loads_and_exports_the_declared_symbols():
  folder = ensure_features(K)
  with open(os.path.join(folder, f"features_{K}.h"), encoding="utf-8") as f:
    protos = [ln for ln in f.read().split("\n") if ln.startswith(("void ", "int "))]
  ffi = FFI()
  ffi.cdef("\n".join(protos))
  lib = ffi.dlopen(os.path.join(folder, f"libfeatures_{K}.so"))
  for name in ("compute_pos", "res_fun", "jac_fun", "merge_features", "compute_pos_batch", "merge_features_batch", "sane_batch", "features_cuda_status"):
    assert getattr(lib, name)
  assert lib.features_k() == K and (N_FEATURES, N_TRACKS) == (3000, 6000)
