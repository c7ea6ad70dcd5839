// rednose_b200 -- batched Mahalanobis query: d = y^T (H_err P H_err^T + R)^-1 y with y = z - h(x), no state change.
// Reference: EKF_sym.maha_test, rednose/helpers/ekf_sym.py:626-649 (h, H, H_mod, S^-1 with numpy; no null-space
// projection even for feature kinds).  A query, not a hot loop: one thread per filter, any EDIM, P read in place
// through a view of its lower triangle (full or packed layout, so both give the same distance); the generated sparse KIND::Herr_apply does both H_err P and (H_err P) H_err^T.
#pragma once
#include "ekf_common.cuh"
#include "ekf_packed.cuh"

namespace rnb {

template <int E>
struct GlobalCol {  // column j of one filter's covariance in global memory as a vector, read from the lower triangle
  const double* P;  // the filter's covariance: row-major [E, E], or packed (ekf_packed.cuh)
  int j;
  bool packed;
  __device__ __forceinline__ double operator[](int i) const {
    if constexpr (E % 2 == 0) {
      if (packed) return __ldg(P + packed_index(i, j));
    }
    return __ldg(P + (i >= j ? i * E + j : j * E + i));
  }
};

struct ScratchRow {  // written by this very thread earlier in the kernel: plain (coherent) loads, never __ldg
  const double* p;
  __device__ __forceinline__ double operator[](int i) const { return p[i]; }
};

template <class M, class K>
__global__ void __launch_bounds__(128) ekf_maha_thread(const double* __restrict__ x, const double* __restrict__ P, const double* __restrict__ z,
                                                       const double* __restrict__ R, const double* __restrict__ ea, long long B, int flags,
                                                       GV<M::NG> gvs, double* __restrict__ out, double* scratch) {
  constexpr int D = M::DIM, E = M::EDIM, Z = K::ZDIM;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double hx[Z];
  double hv[K::NH > 0 ? K::NH : 1];
  K::obs_leaf(x + b * D, (K::EADIM > 0 && ea) ? ea + b * K::EADIM : nullptr, gvs.v, hx, hv);
  double y[Z];
#pragma unroll
  for (int i = 0; i < Z; ++i) y[i] = z[b * Z + i] - hx[i];
  // HP[c][j] for all columns j -> per-thread scratch (Z x E doubles), then S[:, t] = H_err HP[t, :]^T
  double* hpw = scratch + b * (long long)(Z * E);
  const bool packed = (E % 2 == 0) && (flags & FLAG_PACKED_P);
  const double* Pb = P + b * (long long)(packed ? packed_doubles(E) : E * E);
  for (int j = 0; j < E; ++j) {
    GlobalCol<E> pc{Pb, j, packed};
    double hp[Z];
    K::Herr_apply(hv, pc, hp);
#pragma unroll
    for (int c = 0; c < Z; ++c) hpw[c * E + j] = hp[c];
  }
  double S[Z][Z];
  const double* Rb = R + ((flags & FLAG_SHARED_R) ? 0 : b * (long long)(Z * Z));
#pragma unroll
  for (int t = 0; t < Z; ++t) {
    ScratchRow hr{hpw + t * E};
    double sc[Z];
    K::Herr_apply(hv, hr, sc);
#pragma unroll
    for (int c = 0; c < Z; ++c) S[c][t] = sc[c] + Rb[c * Z + t];
  }
  LDL<Z> ldl;
  ldl.factor(S);
  double u[Z];
#pragma unroll
  for (int i = 0; i < Z; ++i) u[i] = y[i];
  ldl.solve(u);
  double d = 0.0;
#pragma unroll
  for (int i = 0; i < Z; ++i) d = fma(y[i], u[i], d);
  out[b] = d;
}

}  // namespace rnb
