// numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src, pairwise_sum) of m float64 terms term(0..m-1), which
// np.sum and np.mean use on a contiguous vector: fewer than 8 terms add left to right from 0; a run of at most 128 (numpy's
// PW_BLOCKSIZE) keeps eight strided partial sums, adds them as a tree, then adds the tail; a longer run splits at m/2 rounded
// down to a multiple of 8 and adds the two halves' sums.  `Depth` is how many nested splits the caller's m can need (0: m <= 128,
// 1: m <= 144, 4: m <= 1010).  Every add is __dadd_rn, which nvcc never contracts, so the result is numpy's bit for bit
// whenever the terms are.
#pragma once

template <class Term>
__device__ __forceinline__ double pairwise_block(const Term& term, int i0, int m) {
  if (m < 8) {
    double res = 0.0;
    for (int i = 0; i < m; ++i) res = __dadd_rn(res, term(i0 + i));
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = term(i0 + j);
  const int m8 = m - m % 8;
  for (int i = 8; i < m8; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], term(i0 + i + j));
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (int i = m8; i < m; ++i) res = __dadd_rn(res, term(i0 + i));
  return res;
}

template <int Depth, class Term>
__device__ __forceinline__ double pairwise_sum(const Term& term, int i0, int m) {
  if constexpr (Depth > 0) {
    if (m > 128) {
      const int h = (m / 2) - (m / 2) % 8;
      return __dadd_rn(pairwise_sum<Depth - 1>(term, i0, h), pairwise_sum<Depth - 1>(term, i0 + h, m - h));
    }
  }
  return pairwise_block(term, i0, m);
}
