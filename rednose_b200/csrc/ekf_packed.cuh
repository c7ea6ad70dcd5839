// rednose_b200 -- resident packed-symmetric covariance of the pair kernel (ekf_warp2.cuh): the one definition of the layout.
//
// P (EDIM x EDIM, EDIM even) is stored as its LOWER BLOCK TRIANGLE of 2x2 blocks, block rows first:
//
//   block (I, J), I >= J, starts at double  2 I (I + 1) + 4 J   and holds  P[2I][2J], P[2I][2J+1], P[2I+1][2J], P[2I+1][2J+1]
//
// nb = EDIM / 2 block rows, nb (nb + 1) / 2 blocks of 32 bytes each (live_kf: 66 blocks = 264 doubles = 2 112 B instead of
// 3 872 B).  The one upper element of a diagonal block, P[2I][2I+1], is stored as the mirror of P[2I+1][2I] and never read:
// P is defined by its lower triangle.  Included by the CUDA kernels and, unchanged, by host C++ (the CPU tests).
#pragma once

#if defined(__CUDACC__)
#define RNB_HD __host__ __device__ __forceinline__
#else
#define RNB_HD inline
#endif

namespace rnb {

// doubles of one packed covariance of an E x E matrix (E even)
RNB_HD constexpr int packed_doubles(int E) { return 2 * (E / 2) * (E / 2 + 1); }

// first double of block (I, J), I >= J
RNB_HD constexpr int packed_block(int I, int J) { return 2 * I * (I + 1) + 4 * J; }

// the double that holds P[i][j] as the lower triangle defines it (P[max][min])
RNB_HD constexpr int packed_index(int i, int j) {
  return i >= j ? packed_block(i >> 1, j >> 1) + 2 * (i & 1) + (j & 1) : packed_block(j >> 1, i >> 1) + 2 * (j & 1) + (i & 1);
}

// the element (i, j) that double t of a packed E x E covariance holds; the upper corner of diagonal block I is (2I, 2I + 1)
RNB_HD void packed_element(int E, int t, int& i, int& j) {
  int I = 0;
  while (I + 1 < E / 2 && packed_block(I + 1, 0) <= t) ++I;
  const int w = t - packed_block(I, 0);
  i = 2 * I + ((w >> 1) & 1);
  j = 2 * (w >> 2) + (w & 1);
}

}  // namespace rnb
