// Division of a 32-bit quad index by the quads per row, by multiply-high with a precomputed reciprocal.  Shared by
// the row-wise fast kernel (ew.cuh) and a host-only test driver (tests/c/rowdiv_check.cu), so both run this code.
//
// With magic = ceil(2^64 / qpr) = (2^64 + e) / qpr, 0 <= e < qpr:
//     Q * magic / 2^64 = Q / qpr + Q * e / (qpr * 2^64),
// and the second term is below 1/qpr whenever Q * e < 2^64, which Q, qpr < 2^32 guarantees.  The fractional part of
// Q / qpr is at most (qpr - 1) / qpr, so the floor of the sum is floor(Q / qpr): exact for EVERY 32-bit Q.
// (A 2^40 reciprocal is exact only while Q * qpr < 2^40 and its product Q * magic wraps 64 bits from row 2^24 on.)
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define TSDE_HD __host__ __device__ __forceinline__
#else
#define TSDE_HD inline
#endif

namespace tsde {

// ceil(2^64 / qpr) for 2 <= qpr < 2^32.  (For a power of two this is exactly 2^64 / qpr, which is also exact.)
TSDE_HD uint64_t rowdiv_magic(uint64_t qpr) { return ~0ull / qpr + 1ull; }

// floor(Q / qpr) given magic = rowdiv_magic(qpr).
TSDE_HD uint32_t rowdiv_row(uint32_t Q, uint64_t magic) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__umul64hi((uint64_t)Q, magic);
#else
  return (uint32_t)(((unsigned __int128)Q * magic) >> 64);
#endif
}

// Q mod qpr given its row.
TSDE_HD uint32_t rowdiv_quad(uint32_t Q, uint32_t row, uint32_t qpr) { return Q - row * qpr; }

}  // namespace tsde
