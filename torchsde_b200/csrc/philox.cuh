// Counter-based normal generator used by every kernel of the library.
//
// Replaces the reference's per-node `torch.Generator(device).manual_seed(seed)` +
// `torch.randn` (torchsde/_brownian/brownian_interval.py:30-32, 243-255) whose seeds come
// from `numpy.random.SeedSequence` (:336-339, :551-552).  That stream is not pinned by any
// reference test (SURVEY.md §8c), so the bit-level definition below *is* the specification;
// oracle/philox.py restates it in numpy and tests/ pins the two against each other and
// against the Random123 known-answer vectors.
//
// Definition.  For a Brownian object with 64-bit key K, a tree-node / cell id I (64 bit),
// a stream tag S (which normal of the node), global row r and channel c:
//     q    = c / 4,  lane = c % 4
//     ctr  = ( q | S << 24 | call << 31,  r_lo32,  I_lo32,  I_hi32 )        call = 0 (fp32)
//     x[4] = Philox4x32-10(ctr, K)
//   fp32:  pairs (x_0, x_1) and (x_2, x_3) each give two normals by Box-Muller:
//            a = fp32( fma(float(x_a), 2^-32, 2^-33) )      radius uniform in (0, 1], 32-bit resolution
//            b = (x_b >> 9) * 2^-23                           angle fraction in [0, 1), 23-bit resolution
//            n_even = sqrt(-2 ln a) cos(2 pi b),  n_odd = sqrt(-2 ln a) sin(2 pi b);   normal = n[lane]
//          (evaluated with SFU approximations, see below; the oracle evaluates the same formula in
//           float64 — agreement ~1e-6 absolute per normal)
//   fp64:  two calls (call = 0,1); call k serves lanes 2k, 2k+1:
//          u_a = ((x_0 * 2^32 + x_1) >> 11 + 0.5) * 2^-53 ; u_b likewise from x_2,x_3
//          n_{2k}, n_{2k+1} = BoxMuller(u_a, u_b)
//   BoxMuller(a, b) = sqrt(-2 ln a) * (cos(2 pi b), sin(2 pi b))
// Rows are independent streams, so sharding the batch over GPUs (row_offset) cannot change
// any trajectory.
#pragma once
#include <stdint.h>

namespace tsde {

enum : uint32_t {
  STREAM_W = 0,   // cell increment normal          (brownian_interval.py:553-554)
  STREAM_H = 1,   // cell space-time Levy normal    (:555-558)
  STREAM_X1 = 2,  // bridge normal X1               (:211)
  STREAM_X2 = 3,  // bridge normal X2               (:212)
  STREAM_A = 4    // Davie/Foster Levy-area noise   (:88, 252-255)
};

struct Key {
  uint32_t lo, hi;
};

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;  // round multipliers
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;  // key increments (Weyl sequence)

__device__ __forceinline__ uint4 philox_round(uint4 c, uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(kPhiloxM0, c.x), lo0 = kPhiloxM0 * c.x;
  const uint32_t hi1 = __umulhi(kPhiloxM1, c.z), lo1 = kPhiloxM1 * c.z;
  return make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
}

// (round i XORs in the key words (k0 + i W0, k1 + i W1))
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    c = philox_round(c, k0, k1);
    k0 += kPhiloxW0;
    k1 += kPhiloxW1;
  }
  return c;
}

// Philox4x32-10 of the counters (x, y, z, w) of one thread that share words x and y: its draws of one stream and row
// on successive cells.  The key schedule and the part of round 0 that reads x and y alone are formed once
// (philox_xy); each draw (philox_zw) forms the rest.  XOR is associative, so the words are philox4x32_10's.
struct PhiloxXY {
  uint32_t k0[10], k1[10];  // the key words of each round
  uint32_t yk;              // y ^ k0[0]:               round 0's first word is umulhi(M1, z) ^ yk
  uint32_t hx;              // umulhi(M0, x) ^ k1[0]:   its third is hx ^ w
  uint32_t lx;              // M0 x:                    its fourth
};

__device__ __forceinline__ PhiloxXY philox_xy(uint32_t x, uint32_t y, uint32_t k0, uint32_t k1) {
  PhiloxXY s;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    s.k0[i] = k0;
    s.k1[i] = k1;
    k0 += kPhiloxW0;
    k1 += kPhiloxW1;
  }
  s.yk = y ^ s.k0[0];
  s.hx = __umulhi(kPhiloxM0, x) ^ s.k1[0];
  s.lx = kPhiloxM0 * x;
  return s;
}

__device__ __forceinline__ uint4 philox_zw(const PhiloxXY& s, uint32_t z, uint32_t w) {
  uint4 c = make_uint4(__umulhi(kPhiloxM1, z) ^ s.yk, kPhiloxM1 * z, s.hx ^ w, s.lx);
#pragma unroll
  for (int i = 1; i < 10; ++i) c = philox_round(c, s.k0[i], s.k1[i]);
  return c;
}

// ---- fp32 -------------------------------------------------------------------------------
// The Brownian kernels are HBM-bound only if the normals are cheap (the pure-RNG kernels are limited by the
// instruction COUNT per normal, not by any one pipe), so the fp32 path
//   * uses the SFU (MUFU.LG2 / MUFU.SQRT / MUFU.SIN / MUFU.COS) instead of libm;
//   * radius:  r^2 = -2 ln a.  MUFU.LG2 has ~2^-22 *absolute* error, which would hurt only for a -> 1 (tiny r);
//     there (x >= 0xFF000000, v = 1 - a < 2^-8, exact in fp32)  -ln(1 - v) = v (1 + v/2 + v^2/3 + ...) is used;
//   * angle:   the fraction b is built straight into a float's mantissa, fb = as_float(x >> 9 | 0x3f800000) in
//     [1, 2) — one funnel shift instead of an int->float conversion and a multiply — and
//     theta = 2 pi (fb - 1.5) = 2 pi b - pi lies in [-pi, pi) where sin/cos.approx are accurate (~5e-7 abs);
//     cos(2 pi b) = -cos(theta), sin(2 pi b) = -sin(theta);
//   * evaluates the two pairs of a quad side by side, with explicitly rounded operations.
// Agreement with the float64 oracle: a few 1e-7 relative on r, <= ~1e-6 absolute on a normal.
__device__ __forceinline__ float mufu_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float mufu_sqrt(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float mufu_sin(float x) {
  float y;
  asm("sin.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float mufu_cos(float x) {
  float y;
  asm("cos.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// four normals from one Philox output: (x.x, x.y) -> n0, n1 ; (x.z, x.w) -> n2, n3.  The two pairs go side by side,
// one explicitly rounded operation of each per line (never contracted or reassociated, whatever -fmad says).
__device__ __forceinline__ void box_muller4(const uint4 x, float (&n)[4]) {
  const float k2m32 = 2.3283064365386963e-10f, k2m33 = 1.1641532182693481e-10f;
  // radius uniforms a = fma(float(x), 2^-32, 2^-33)
  const float x0 = __uint2float_rn(x.x), x1 = __uint2float_rn(x.z);
  const float a0 = __fmaf_rn(x0, k2m32, k2m33), a1 = __fmaf_rn(x1, k2m32, k2m33);
  // r^2 through the SFU ...
  const float lg0 = mufu_lg2(a0), lg1 = mufu_lg2(a1);
  const float l0 = __fmul_rn(lg0, -1.3862943611198906f), l1 = __fmul_rn(lg1, -1.3862943611198906f);
  // ... and through the series in v = 1 - a (exact), used where a is within 2^-8 of 1
  const float na0 = __fmul_rn(a0, -1.0f), na1 = __fmul_rn(a1, -1.0f);
  const float v0 = __fadd_rn(1.0f, na0), v1 = __fadd_rn(1.0f, na1);
  const float q0 = __fmaf_rn(v0, 0.33333334f, 0.5f), q1 = __fmaf_rn(v1, 0.33333334f, 0.5f);
  const float p0 = __fmaf_rn(v0, q0, 1.0f), p1 = __fmaf_rn(v1, q1, 1.0f);
  const float d0 = __fadd_rn(v0, v0), d1 = __fadd_rn(v1, v1);
  const float s0 = __fmul_rn(d0, p0), s1 = __fmul_rn(d1, p1);
  const float r0 = mufu_sqrt(x.x >= 0xFF000000u ? s0 : l0);
  const float r1 = mufu_sqrt(x.z >= 0xFF000000u ? s1 : l1);
  // angles: mantissa construction, theta = 2 pi (fb - 1.5) in [-pi, pi); fb - 1.5 is exact, so theta carries one
  // rounding and the rounding of the constant (<= 2.7e-7 absolute)
  const float fb0 = __uint_as_float(__funnelshift_r(x.y, 0x7Fu, 9)), fb1 = __uint_as_float(__funnelshift_r(x.w, 0x7Fu, 9));
  const float c0 = __fadd_rn(fb0, -1.5f), c1 = __fadd_rn(fb1, -1.5f);
  const float t0 = __fmul_rn(c0, 6.2831853071795865f), t1 = __fmul_rn(c1, 6.2831853071795865f);
  const float cos0 = mufu_cos(t0), sin0 = mufu_sin(t0);
  const float n0 = __fmul_rn(cos0, -r0), n1 = __fmul_rn(sin0, -r0);
  const float cos1 = mufu_cos(t1), sin1 = mufu_sin(t1);
  const float n2 = __fmul_rn(cos1, -r1), n3 = __fmul_rn(sin1, -r1);
  n[0] = n0;
  n[1] = n1;
  n[2] = n2;
  n[3] = n3;
}

// four normals for channels 4q..4q+3 of (row, id, stream)
__device__ __forceinline__ void normal4(Key k, uint64_t id, uint32_t stream, uint32_t row,
                                        uint32_t q, float (&n)[4]) {
  const uint4 x = philox4x32_10(
      make_uint4(q | (stream << 24), row, (uint32_t)id, (uint32_t)(id >> 32)), k.lo, k.hi);
  box_muller4(x, n);
}

// ---- fp64 -------------------------------------------------------------------------------
__device__ __forceinline__ double u01d(uint32_t hi, uint32_t lo) {
  const uint64_t v = (((uint64_t)hi << 32) | lo) >> 11;
  return ((double)v + 0.5) * 1.1102230246251565e-16;  // 2^-53
}

__device__ __forceinline__ void box_muller(double a, double b, double& n0, double& n1) {
  const double r = sqrt(-2.0 * log(a));
  double s, c;
  sincospi(2.0 * b, &s, &c);
  n0 = r * c;
  n1 = r * s;
}

__device__ __forceinline__ void normal4(Key k, uint64_t id, uint32_t stream, uint32_t row,
                                        uint32_t q, double (&n)[4]) {
#pragma unroll
  for (uint32_t call = 0; call < 2; ++call) {
    const uint4 x = philox4x32_10(
        make_uint4(q | (stream << 24) | (call << 31), row, (uint32_t)id, (uint32_t)(id >> 32)),
        k.lo, k.hi);
    box_muller(u01d(x.x, x.y), u01d(x.z, x.w), n[2 * call], n[2 * call + 1]);
  }
}

__device__ __forceinline__ Key load_key(const void* p) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  return Key{v.x, v.y};
}

}  // namespace tsde
