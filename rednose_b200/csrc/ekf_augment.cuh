// rednose_b200 -- batched MSCKF state augmentation (K3): drop the oldest clone, append a copy of the
// first dim_augment main states; the same selection on rows and columns of P.
// Reference: EKF_sym.augment, rednose/helpers/ekf_sym.py:365-391, which builds a selection matrix and does
// two dense products; here it is the permutation/copy it really is.  One CTA per filter, P staged in
// shared memory so the in-place rewrite is safe.
#pragma once
#include "ekf_common.cuh"

namespace rnb {

// the shift of one filter's state xg [D] and covariance Pg [E, E] by one CTA
template <class M>
__device__ __forceinline__ void augment_one(double* __restrict__ xg, double* __restrict__ Pg, int d3, int d4) {
  constexpr int D = M::DIM, E = M::EDIM, d1 = M::DMAIN, d2 = M::MEDIM;
  extern __shared__ __align__(16) double tile[];  // E*E + D
  double* xs = tile + E * E;
  for (int i = threadIdx.x; i < E * E; i += blockDim.x) tile[i] = Pg[i];
  for (int i = threadIdx.x; i < D; i += blockDim.x) xs[i] = xg[i];
  __syncthreads();
  // state: [main | clone_1 .. clone_N] -> [main | clone_2 .. clone_N | main[:d3]]
  for (int i = threadIdx.x + d1; i < D; i += blockDim.x) xg[i] = (i < D - d3) ? xs[i + d3] : xs[i - (D - d3)];
  // covariance: src(i) = i for the main block, i + d4 for the surviving clones, i - (E - d4) for the new clone
  auto src = [&](int i) { return i < d2 ? i : (i < E - d4 ? i + d4 : i - (E - d4)); };
  for (int idx = threadIdx.x; idx < E * E; idx += blockDim.x) {
    const int i = idx / E, j = idx - i * E;
    Pg[idx] = tile[src(i) * E + src(j)];
  }
}

template <class M>
__global__ void __launch_bounds__(128) ekf_augment_cta(double* __restrict__ x, double* __restrict__ P, long long B, int d3, int d4) {
  const long long b = blockIdx.x;
  if (b >= B) return;
  augment_one<M>(x + b * M::DIM, P + b * (long long)(M::EDIM * M::EDIM), d3, d4);
}

// gather-list variant: CTA e shifts filter idx[e] (distinct entries); filters not listed are untouched
template <class M, bool GA>
__global__ void __launch_bounds__(128) ekf_augment_cta(double* __restrict__ x, double* __restrict__ P, const int* __restrict__ idx,
                                                       long long n, int d3, int d4) {
  static_assert(GA, "the whole-batch shift is ekf_augment_cta<M>");
  const long long e = blockIdx.x;
  if (e >= n) return;
  const long long b = idx[e];
  augment_one<M>(x + b * M::DIM, P + b * (long long)(M::EDIM * M::EDIM), d3, d4);
}

template <class M>
inline void launch_augment(double* x, double* P, long long B, int dim_augment, int dim_augment_err, cudaStream_t st) {
  if (B <= 0) return;
  const size_t smem = sizeof(double) * (M::EDIM * M::EDIM + M::DIM);
  if (first_launch_of((const void*)ekf_augment_cta<M>))   // per (device, kernel)
    cudaFuncSetAttribute(ekf_augment_cta<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ekf_augment_cta<M><<<(unsigned)B, 128, smem, st>>>(x, P, B, dim_augment, dim_augment_err);
  check(cudaGetLastError(), "ekf_augment launch");
}

// the shift of the n filters idx[e] (distinct) of the full-layout x [*, DIM] / P [*, EDIM, EDIM]; every refusal is made
// before any CUDA call and latched
template <class M>
inline void launch_augment_idx(double* x, double* P, const int* idx, long long n, int flags, int dim_augment, int dim_augment_err,
                               cudaStream_t st) {
  if (n < 0 || (n > 0 && (!x || !P || !idx))) {
    fprintf(stderr, "[rednose_b200] batch_augment_idx: n >= 0 and, for n > 0, x, P and the gather list are required\n");
    last_status() = (int)cudaErrorInvalidValue;
    return;
  }
  if (flags & (FLAG_PACKED_P | FLAG_PACKED_HIST)) {
    fprintf(stderr, "[rednose_b200] batch_augment_idx: the clone-window shift works on the full covariance layout\n");
    last_status() = (int)cudaErrorNotSupported;
    return;
  }
  if (n == 0) return;
  const size_t smem = sizeof(double) * (M::EDIM * M::EDIM + M::DIM);
  if (first_launch_of((const void*)ekf_augment_cta<M, true>))
    cudaFuncSetAttribute(ekf_augment_cta<M, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ekf_augment_cta<M, true><<<(unsigned)n, 128, smem, st>>>(x, P, idx, n, dim_augment, dim_augment_err);
  check(cudaGetLastError(), "ekf_augment_idx launch");
}

}  // namespace rnb
