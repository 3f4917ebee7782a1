// Host-only check of the row division of the row-wise fast kernel (torchsde_b200/csrc/rowdiv.cuh) against plain
// integer division.  Built and run by tests/test_row_division.py; prints the first mismatches and exits non-zero on
// any.  The fast kernel takes 32-bit quad indices Q < 2^31 (fewer than 2^31 quads per launch) with any quads-per-row
// qpr that is not a power of two; the checks go a little beyond that, to every 32-bit Q.
#include <stdint.h>
#include <stdio.h>

#include "../../torchsde_b200/csrc/rowdiv.cuh"

static long long g_checks = 0, g_bad = 0;

static void check(uint32_t qpr, uint64_t magic, uint64_t Q) {
  if (Q > 0xFFFFFFFFull) return;
  ++g_checks;
  const uint32_t row = tsde::rowdiv_row((uint32_t)Q, magic);
  const uint32_t quad = tsde::rowdiv_quad((uint32_t)Q, row, qpr);
  if (row != (uint32_t)(Q / qpr) || quad != (uint32_t)(Q % qpr)) {
    if (g_bad < 10)
      printf("mismatch qpr=%u Q=%llu: row %u quad %u, expected row %llu quad %llu\n", qpr, (unsigned long long)Q, row,
             quad, (unsigned long long)(Q / qpr), (unsigned long long)(Q % qpr));
    ++g_bad;
  }
}

// Q = r*qpr - 1, r*qpr, r*qpr + 1 and r*qpr + qpr - 1 for the rows r around `r0`.
static void around_row(uint32_t qpr, uint64_t magic, uint64_t r0) {
  for (int64_t dr = -2; dr <= 2; ++dr) {
    const int64_t r = (int64_t)r0 + dr;
    if (r < 0) continue;
    const uint64_t b = (uint64_t)r * qpr;
    if (b > 0) check(qpr, magic, b - 1);
    check(qpr, magic, b);
    check(qpr, magic, b + 1);
    check(qpr, magic, b + qpr - 1);
  }
}

static void check_qpr(uint32_t qpr) {
  if ((qpr & (qpr - 1)) == 0) return;  // powers of two take the shift
  const uint64_t magic = tsde::rowdiv_magic(qpr);
  const uint64_t last_fast_row = ((1ull << 31) - 1) / qpr;  // largest row of a launch with < 2^31 quads
  const uint64_t last_row = 0xFFFFFFFFull / qpr;             // largest row of any 32-bit Q
  const uint64_t rows[] = {0, 1, 1ull << 23, 1ull << 24, (1ull << 24) + 1, (1ull << 25), (1ull << 31) / qpr,
                           last_fast_row, last_row};
  for (uint64_t r : rows) around_row(qpr, magic, r);
  for (uint64_t Q = 0; Q < 4 * (uint64_t)qpr && Q < 20000; ++Q) check(qpr, magic, Q);
  // a spread of Q over the whole 32-bit range (an odd stride, so every residue class is visited)
  for (uint64_t Q = 12345; Q <= 0xFFFFFFFFull; Q += 0x00F0F0F1ull) check(qpr, magic, Q);
}

int main() {
  for (uint32_t qpr = 3; qpr <= 4096; ++qpr) check_qpr(qpr);
  // a sample of larger quads-per-row, up to the fast path's limit (qpr <= nquads < 2^31)
  uint64_t s = 0x9E3779B97F4A7C15ull;
  for (int i = 0; i < 3000; ++i) {
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;  // xorshift64
    const int bits = 13 + (int)(s % 19);        // 2^13 .. 2^31
    uint32_t qpr = (uint32_t)((s >> 20) & ((1ull << bits) - 1));
    if (qpr < 3) qpr = 3;
    check_qpr(qpr);
  }
  for (uint32_t qpr : {0x7FFFFFFFu, 0x7FFFFFFEu, 0x40000001u, 0x55555555u, 0xFFFFFFFFu, 0x80000001u}) check_qpr(qpr);
  printf("%lld checks, %lld mismatches\n", g_checks, g_bad);
  return g_bad == 0 ? 0 : 1;
}
