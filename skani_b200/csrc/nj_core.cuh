// nj_core.cuh -- per-element arithmetic of sk_neighbor_joining (nj.cu) as __host__ __device__ functions, so that the same
// code runs inside the CUDA kernels and inside tests/emu/emu_nj.cpp on the host (see sk_core.cuh).
//
// Every operation is rounded on its own (no FMA contraction): on the device through the _rn intrinsics, which nvcc never
// contracts, on the host as plain operators in a build with -ffp-contract=off.  Together with the exact initial distances
// (1 - ani is a multiple of 2^-27) and row sums (exact for n < 2^26, so any summation order gives the same bits) this makes
// every Q, branch length and updated distance a function of the contract alone, equal bit for bit to tests/nj_ref.py.
#pragma once
#include <stdint.h>

#include "sk_core.cuh"

namespace sk {

// R of a slot that holds no live node: every Q it enters is +inf, so it is never the minimum while a live pair is left
constexpr double NJ_DEAD = -__builtin_huge_val();

SK_HD double nj_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SK_HD double nj_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
SK_HD double nj_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
SK_HD double nj_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// initial distance of an edge's ANI (0.1 < ani <= 1)
SK_HD double nj_dist(float ani) { return nj_sub(1.0, (double)ani); }

// Q of the live pair (i, j) when m nodes are live
SK_HD double nj_q(uint32_t m, double dij, double ri, double rj) { return nj_sub(nj_sub(nj_mul((double)(m - 2), dij), ri), rj); }

// (q1, k1) before (q2, k2): the smaller Q, ties to the smaller key (i << 32 | j in id order).  Q is compared as a double, so
// -0 equals +0.
SK_HD bool nj_before(double q1, uint64_t k1, double q2, uint64_t k2) { return q1 < q2 || (q1 == q2 && k1 < k2); }

// branch length from the new node to i; the one to j is dij - delta_i
SK_HD double nj_delta_i(uint32_t m, double dij, double ri, double rj) {
  return nj_add(nj_mul(0.5, dij), nj_div(nj_sub(ri, rj), nj_mul(2.0, (double)(m - 2))));
}

// distance from the new node to another live k
SK_HD double nj_duk(double dik, double djk, double dij) { return nj_mul(0.5, nj_sub(nj_add(dik, djk), dij)); }

// R of another live k after the join
SK_HD double nj_rk(double rk, double dik, double djk, double duk) { return nj_add(nj_sub(nj_sub(rk, dik), djk), duk); }

// R of the new node: the closed form of sum_k d_uk
SK_HD double nj_ru(uint32_t m, double ri, double rj, double dij) { return nj_mul(0.5, nj_sub(nj_add(ri, rj), nj_mul((double)m, dij))); }

}  // namespace sk
