// Fused row-wise tableau kernel framework (diagonal noise, and every purely element-wise
// stage).  One thread owns one "quad": 4 consecutive channels of one trajectory, which is
// exactly what one Philox4x32 call yields in fp32 — so the Brownian increment of the quad is
// produced in registers and never touches HBM (north star: "dW in registers").
//
// HBM plan (H100 SXM: 132 SMs, 3.35 TB/s HBM3 on the data sheet): each input tensor is read
// once with 128-bit loads, each output written once with 128-bit stores; every thread issues
// all of its loads before the first dependent use (NIN independent LDG.128 in flight per
// thread).  The fast kernel gives each CTA one chunk of U x 256 quads (see ew_fast_kernel); the
// generic kernel's grid is one resident wave (SM count x occupancy), each CTA owning an equal
// contiguous slice of the quads.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "host.cuh"
#include "pw_device.cuh"

namespace tsde {

constexpr int kBlocksPerSM = 8;  // 2048 threads / SM

template <int NIN, int NOUT>
struct EwP {
  const void* in[NIN > 0 ? NIN : 1];
  void* out[NOUT];
  int64_t rows;
  int64_t d;
  int64_t qpr;     // quads per row
  int64_t nquads;  // rows * qpr
  int32_t vec;     // all pointers 16B-aligned (8B for a 16-bit Mixed operand) and d % 4 == 0
  int32_t qshift;  // log2(qpr) if qpr is a power of two, else -1
  int32_t small;   // nquads < 2^31: 32-bit index arithmetic
  uint64_t qmagic; // rowdiv_magic(qpr) = ceil(2^64 / qpr): row = umulhi(Q, qmagic), exact for every 32-bit Q
};

// streaming variants (ld.global.cs: evict-first) for operands that are dead after this kernel
__device__ __forceinline__ void ld4cs(const float* p, float (&v)[4]) {
  const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4cs(const double* p, double (&v)[4]) {
  const double2 a = __ldcs(reinterpret_cast<const double2*>(p));
  const double2 b = __ldcs(reinterpret_cast<const double2*>(p + 2));
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}

template <typename Op, typename = void>
struct streams_inputs { static constexpr bool value = false; };
template <typename Op>
struct streams_inputs<Op, decltype((void)Op::STREAM_INPUTS)> { static constexpr bool value = Op::STREAM_INPUTS; };

// ---- 16-bit SDE outputs (TSDE_FMT_*, float32 state only) ----------------------------------------------------------
// Mixed<Op> is Op with the storage format of each input (and output) as a launch argument, two bits per tensor in
// the op's order.  The kernels instantiated for it load a 16-bit quad with one 64-bit load instead of a 128-bit one,
// widen it exactly and run Op's float32 arithmetic unchanged, so the result equals the float32 launch on widened
// copies bit for bit.  The formats ride in the op rather than in EwP / GenP so that the parameter layout, and hence
// the SASS, of every all-float32 / float64 instantiation stays exactly what it was.
template <typename Op>
struct Mixed : Op {
  static constexpr bool MIXED = true;
  uint32_t fmt;   // inputs
  uint32_t ofmt;  // outputs (only tsde_milstein_vjp_seed writes a 16-bit one: go in g's format)
};
template <typename Op, typename = void>
struct is_mixed { static constexpr bool value = false; };
template <typename Op>
struct is_mixed<Op, decltype((void)Op::MIXED)> { static constexpr bool value = Op::MIXED; };

__host__ __device__ inline uint32_t operand_fmt(uint32_t fmt, int i) { return (fmt >> (2 * i)) & 3u; }

__device__ __forceinline__ float widen16(uint32_t bits, uint32_t f) {  // exact
  return f == TSDE_FMT_BF16 ? __uint_as_float(bits << 16) : __half2float(__ushort_as_half((unsigned short)bits));
}
__device__ __forceinline__ uint32_t narrow16(float x, uint32_t f) {  // round to nearest even, as torch's .to()
  return f == TSDE_FMT_BF16 ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x))
                            : (uint32_t)__half_as_ushort(__float2half_rn(x));
}
// Loads return raw bits and widening is a separate step: a thread issues all of its loads first and converts after,
// as the float32 kernels do (a load whose widening sat next to it would be consumed before the next load issued).
// element i of a tensor in format f
__device__ __forceinline__ uint32_t ld1raw(const void* p, int64_t i, uint32_t f) {
  return f == TSDE_FMT_STATE ? static_cast<const uint32_t*>(p)[i] : (uint32_t)static_cast<const uint16_t*>(p)[i];
}
__device__ __forceinline__ float widen1(uint32_t r, uint32_t f) {
  return f == TSDE_FMT_STATE ? __uint_as_float(r) : widen16(r, f);
}
__device__ __forceinline__ float ld1f(const void* p, int64_t i, uint32_t f) { return widen1(ld1raw(p, i, f), f); }
__device__ __forceinline__ void st1f(void* p, int64_t i, uint32_t f, float x) {
  if (f == TSDE_FMT_STATE) static_cast<float*>(p)[i] = x;
  else static_cast<uint16_t*>(p)[i] = (uint16_t)narrow16(x, f);
}
// elements i..i+3: one 128-bit load (16-byte aligned float32) or one 64-bit load (8-byte aligned 16-bit, in .x, .y);
// CS: evict-first
template <bool CS>
__device__ __forceinline__ uint4 ld4raw(const void* p, int64_t i, uint32_t f) {
  if (f == TSDE_FMT_STATE) {
    const uint4* q = reinterpret_cast<const uint4*>(static_cast<const float*>(p) + i);
    return CS ? __ldcs(q) : *q;
  }
  const uint2* q = reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(p) + i);
  const uint2 h = CS ? __ldcs(q) : *q;
  return make_uint4(h.x, h.y, 0u, 0u);
}
__device__ __forceinline__ void widen4(const uint4 r, uint32_t f, float (&v)[4]) {
  if (f == TSDE_FMT_STATE) {
    v[0] = __uint_as_float(r.x); v[1] = __uint_as_float(r.y); v[2] = __uint_as_float(r.z); v[3] = __uint_as_float(r.w);
    return;
  }
  v[0] = widen16(r.x & 0xffffu, f);
  v[1] = widen16(r.x >> 16, f);
  v[2] = widen16(r.y & 0xffffu, f);
  v[3] = widen16(r.y >> 16, f);
}
__device__ __forceinline__ void st4f(void* p, int64_t i, uint32_t f, const float (&v)[4]) {
  if (f == TSDE_FMT_STATE) {
    st4(static_cast<float*>(p) + i, v);
    return;
  }
  *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p) + i) =
      make_uint2(narrow16(v[0], f) | (narrow16(v[1], f) << 16), narrow16(v[2], f) | (narrow16(v[3], f) << 16));
}
// raw bits of one quad in format f (vector path: ld4raw; otherwise element by element, in .x .. .w)
__device__ __forceinline__ uint4 load_quad_raw(const void* p, int64_t base, bool vec, int nvalid, uint32_t f) {
  if (vec) return ld4raw<false>(p, base, f);
  uint32_t r[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) r[j] = j < nvalid ? ld1raw(p, base + j, f) : 0u;
  return make_uint4(r[0], r[1], r[2], r[3]);
}
__device__ __forceinline__ void widen_quad(const uint4 r, bool vec, uint32_t f, float (&v)[4]) {
  if (vec) {
    widen4(r, f, v);
  } else {
    v[0] = widen1(r.x, f); v[1] = widen1(r.y, f); v[2] = widen1(r.z, f); v[3] = widen1(r.w, f);
  }
}
__device__ __forceinline__ void store_quad_fmt(void* p, int64_t base, bool vec, int nvalid, uint32_t f,
                                               const float (&v)[4]) {
  if (vec) {
    st4f(p, base, f, v);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < nvalid) st1f(p, base + j, f, v[j]);
  }
}
// the host's fast-path alignment: 16 bytes for a float32 / float64 operand, 8 for a 16-bit one
inline bool aligned_for(const void* p, uint32_t f) {
  return (reinterpret_cast<uintptr_t>(p) & (f == TSDE_FMT_STATE ? 15u : 7u)) == 0;
}


// ---- the kernel -----------------------------------------------------------------------------
// Op: struct with  static constexpr int NIN, NOUT; static constexpr bool USES_NOISE, WANT_U;
//     template<T> __device__ void operator()(const T (&in)[NIN], T w, T u, T (&out)[NOUT]) const
// (Mixed<Op>: the raw bits of all NIN operands stay live across the increment's draw, and then their widened values;
// at 4 resident CTAs (64 registers) the 8-input ops would spill, so the bound is 2 CTAs for them)
template <typename T, typename Op, int SRC>
__global__ void __launch_bounds__(kThreads, is_mixed<Op>::value ? 2 : 4)
ew_kernel(const EwP<Op::NIN, Op::NOUT> p, const NoiseP<T> nz, const Op op) {
  constexpr int NIN = Op::NIN, NOUT = Op::NOUT;
  Key key{0u, 0u};
  if (Op::USES_NOISE && (SRC == TSDE_SRC_COUNTER || SRC == kSrcCounterMulti)) key = load_key(nz.key);
  const bool vec = p.vec != 0;
  // Each CTA owns one contiguous slice of the quads, slices differ by at most one quad: with
  // gridDim = SMs x resident CTAs every SM gets the same amount of work (no tail wave, no
  // ceil(trip count) imbalance between SMs).
  const int64_t q_begin = (p.nquads * (int64_t)blockIdx.x) / gridDim.x;
  const int64_t q_end = (p.nquads * ((int64_t)blockIdx.x + 1)) / gridDim.x;
  for (int64_t Q = q_begin + threadIdx.x; Q < q_end; Q += kThreads) {
    int64_t row, q;
    if (p.qshift >= 0) {
      row = Q >> p.qshift;
      q = Q & ((1 << p.qshift) - 1);
    } else if (p.small) {
      const uint32_t r32 = (uint32_t)Q / (uint32_t)p.qpr;
      row = r32;
      q = (uint32_t)Q - r32 * (uint32_t)p.qpr;
    } else {
      row = Q / p.qpr;
      q = Q - row * p.qpr;
    }
    const int64_t base = row * p.d + 4 * q;
    const int64_t rem = p.d - 4 * q;
    const int nvalid = rem < 4 ? (int)rem : 4;
    T in[NIN > 0 ? NIN : 1][4];
    uint4 raw[NIN > 0 ? NIN : 1];  // (Mixed: every load issued before the first widening)
#pragma unroll
    for (int i = 0; i < NIN; ++i) {
      if constexpr (is_mixed<Op>::value) raw[i] = load_quad_raw(p.in[i], base, vec, nvalid, operand_fmt(op.fmt, i));
      else load_quad(reinterpret_cast<const T*>(p.in[i]), base, vec, nvalid, in[i]);
    }
    T w[4], u[4];
    if (Op::USES_NOISE) {
      quad_noise<T, SRC, Op::WANT_U>(nz, key, row, q, vec, nvalid, w, u);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) { w[j] = T(0); u[j] = T(0); }
    }
    if constexpr (is_mixed<Op>::value) {
#pragma unroll
      for (int i = 0; i < NIN; ++i) widen_quad(raw[i], vec, operand_fmt(op.fmt, i), in[i]);
    }
    T out[NOUT][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      T a[NIN > 0 ? NIN : 1], b[NOUT];
#pragma unroll
      for (int i = 0; i < NIN; ++i) a[i] = in[i][j];
      op(a, w[j], u[j], b);
#pragma unroll
      for (int i = 0; i < NOUT; ++i) out[i][j] = b[i];
    }
#pragma unroll
    for (int i = 0; i < NOUT; ++i) {
      if constexpr (is_mixed<Op>::value) store_quad_fmt(p.out[i], base, vec, nvalid, operand_fmt(op.ofmt, i), out[i]);
      else store_quad(reinterpret_cast<T*>(p.out[i]), base, vec, nvalid, out[i]);
    }
  }
}

// ---- fast variant: the shapes the headline path uses -------------------------------------------
// Preconditions checked on the host: 128-bit aligned tensors with d % 4 == 0 (vector path), noise not
// broadcast, fewer than 2^31 quads.  The row of a quad is a shift when quads-per-row is a power of two, else a
// multiply-high by a 64-bit reciprocal (rowdiv.cuh), exact for every 32-bit quad index.
// Everything is 32-bit index arithmetic and there is no per-quad branching.
//
// (Tried and rejected: software-pipelining the integer half of iteration i+1's noise (Philox) next to the float
// half of iteration i (Box-Muller) was slower on every RNG-bound kernel: the carried Philox state costs more than the
// pipe mixing gains.)
// Light ops (at most 3 tensors per quad: the Milstein vjp seed, the Brownian materialisation, the
// predictor stages) are NOT HBM-bound per thread: the Philox + Box-Muller chain (~150 dependent-ish
// instructions per quad) dominates and one 128-bit load per thread does not cover the HBM latency-bandwidth
// product (the kernel is issue-bound with every pipe far from saturation).  Those ops
// process U = 2 quads per thread: the two independent Philox chains interleave, and both loads are issued
// before the first use (2x ILP, 2x bytes in flight per thread).  Heavy ops (>= 4 tensors) keep U = 1: their
// loads already cover the latency and the extra registers would cost occupancy.
template <typename T, typename Op>
struct quads_per_iter { static constexpr int value = (sizeof(T) == 4 && Op::NIN + Op::NOUT <= 3) ? 2 : 1; };

template <typename T, typename Op>
struct FastCtx {
  const EwP<Op::NIN, Op::NOUT>& p;
  const NoiseP<T>& nz;
  const Op& op;
  Key key;
  uint32_t q_end, qshift, qmask, qpr32, row_off;
  uint64_t qmagic;
  bool pow2;
  __device__ __forceinline__ uint32_t row_of(uint32_t Q) const {
    return pow2 ? (Q >> qshift) : rowdiv_row(Q, qmagic);
  }
  __device__ __forceinline__ uint32_t quad_of(uint32_t Q, uint32_t row) const {
    return pow2 ? (Q & qmask) : rowdiv_quad(Q, row, qpr32);
  }
  __device__ __forceinline__ void rng(uint32_t Q, T (&w)[4], T (&u)[4]) const {
    const uint32_t r = row_of(Q);
    counter_noise<T, Op::WANT_U, false>(nz, key, r + row_off, quad_of(Q, r), w, u);
  }
};

// A thread's U quads Q, Q + kThreads, ... (each warp access stays one contiguous 512-byte run).
// Counter noise was produced ahead of the dependency wait and is passed in (w0, u0).
template <typename T, typename Op, int SRC, int U>
__device__ __forceinline__ void ew_fast_body(const FastCtx<T, Op>& c, uint32_t Q, const T (&w0)[U][4],
                                             const T (&u0)[U][4]) {
  constexpr int NIN = Op::NIN, NOUT = Op::NOUT;
  bool ok[U];
  T in[U][NIN > 0 ? NIN : 1][4];
  uint4 raw[U][NIN > 0 ? NIN : 1];  // (Mixed: raw bits, widened once every load has been issued)
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const uint32_t Qk = Q + (uint32_t)k * kThreads;
    ok[k] = k == 0 || Qk < c.q_end;
    const size_t base = (size_t)Qk * 4;  // d == 4 * qpr: quads are laid out contiguously
    if constexpr (is_mixed<Op>::value) {
#pragma unroll
      for (int i = 0; i < NIN; ++i) raw[k][i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (ok[k]) {
#pragma unroll
      for (int i = 0; i < NIN; ++i) {
        if constexpr (is_mixed<Op>::value)
          raw[k][i] = ld4raw<streams_inputs<Op>::value>(c.p.in[i], (int64_t)base, operand_fmt(c.op.fmt, i));
        else if (streams_inputs<Op>::value)
          ld4cs(reinterpret_cast<const T*>(c.p.in[i]) + base, in[k][i]);
        else
          ld4(reinterpret_cast<const T*>(c.p.in[i]) + base, in[k][i]);
      }
    }
  }
  T w[U][4], u[U][4];
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const uint32_t Qk = Q + (uint32_t)k * kThreads;
    const size_t base = (size_t)Qk * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) { w[k][j] = T(0); u[k][j] = T(0); }
    if (Op::USES_NOISE) {
      if (SRC == TSDE_SRC_COUNTER) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { w[k][j] = w0[k][j]; u[k][j] = Op::WANT_U ? u0[k][j] : T(0); }
      } else if (SRC == TSDE_SRC_MEMORY) {
        if (ok[k]) {
          ld4(c.nz.w + base, w[k]);
          if (Op::WANT_U) ld4(c.nz.u + base, u[k]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) { w[k][j] = T(1); u[k][j] = T(0); }
      }
    }
  }
  if constexpr (is_mixed<Op>::value) {
#pragma unroll
    for (int k = 0; k < U; ++k) {
#pragma unroll
      for (int i = 0; i < NIN; ++i) widen4(raw[k][i], operand_fmt(c.op.fmt, i), in[k][i]);
    }
  }
#pragma unroll
  for (int k = 0; k < U; ++k) {
    if (!ok[k]) continue;
    const size_t base = (size_t)(Q + (uint32_t)k * kThreads) * 4;
    T out[NOUT][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      T a[NIN > 0 ? NIN : 1], b[NOUT];
#pragma unroll
      for (int i = 0; i < NIN; ++i) a[i] = in[k][i][j];
      c.op(a, w[k][j], u[k][j], b);
#pragma unroll
      for (int i = 0; i < NOUT; ++i) out[i][j] = b[i];
    }
#pragma unroll
    for (int i = 0; i < NOUT; ++i) {
      if constexpr (is_mixed<Op>::value) st4f(c.p.out[i], (int64_t)base, operand_fmt(c.op.ofmt, i), out[i]);
      else st4(reinterpret_cast<T*>(c.p.out[i]) + base, out[i]);
    }
  }
}

// One chunk of U * kThreads quads per CTA (CTA b owns chunk b), not a persistent grid of contiguous slices: the chunk
// grid needs no loop, so the Milstein tableau and vjp seed take 38 and 32 registers instead of 56 and 61 and more of
// their CTAs are resident; both kernels got faster on the H100 (DESIGN §3, which also records the descending and
// round-robin chunk orders that were measured and rejected).
template <typename T, typename Op>
inline uint32_t fast_chunks(uint32_t nquads) {
  constexpr uint32_t chunk = quads_per_iter<T, Op>::value * kThreads;
  return (nquads + chunk - 1) / chunk;
}

template <typename T, typename Op, int SRC>
__global__ void __launch_bounds__(kThreads, 4)
ew_fast_kernel(const EwP<Op::NIN, Op::NOUT> p, const NoiseP<T> nz, const Op op) {
  constexpr int U = quads_per_iter<T, Op>::value;
  constexpr bool COUNTER = Op::USES_NOISE && SRC == TSDE_SRC_COUNTER;
  const uint32_t nquads = (uint32_t)p.nquads;
  const bool pow2 = p.qshift >= 0;
  const uint32_t qshift = pow2 ? (uint32_t)p.qshift : 0u;
  const FastCtx<T, Op> c{p, nz, op, COUNTER ? load_key(nz.key) : Key{0u, 0u}, nquads, qshift, (1u << qshift) - 1u,
                         (uint32_t)p.qpr, (uint32_t)nz.row_offset, p.qmagic, pow2};
  // Programmatic dependent launch: this grid may start while its predecessor in the stream/graph is
  // still draining.  Everything that does not touch the predecessor's outputs — the Philox/Box-Muller
  // work of the thread's U quads — runs before `griddepcontrol.wait`; all loads and stores come after.
  T w0[U][4], u0[U][4];
  const uint32_t Q0 = blockIdx.x * (uint32_t)(U * kThreads) + threadIdx.x;
  if (COUNTER) {
#pragma unroll
    for (int k = 0; k < U; ++k) {
      c.rng(Q0 + (uint32_t)k * kThreads, w0[k], u0[k]);
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q0 >= nquads) return;
  ew_fast_body<T, Op, SRC, U>(c, Q0, w0, u0);
}

// ---- host-side launcher -----------------------------------------------------------------------
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename T>
inline int fill_noise(const tsde_launch* L, const tsde_noise* nz, bool bcast, NoiseP<T>& out) {
  out = NoiseP<T>{};
  out.m = bcast ? 1 : L->m;
  out.bcast = bcast ? 1 : 0;
  if (L->rows + (nz ? nz->row_offset : 0) > kMaxGlobalRows) return TSDE_EINVAL;
  if (!nz) return 0;
  out.w = reinterpret_cast<const T*>(nz->w);
  out.u = reinterpret_cast<const T*>(nz->u);
  out.key = nz->key;
  out.cell_id = nz->cell_id;
  out.row_offset = nz->row_offset;
  out.n_cells = nz->n_cells < 1 ? 1 : nz->n_cells;
  out.h = nz->h;
  out.cell_h = nz->cell_h;
  out.h_total = nz->h_total;
  out.sqrt_h = (T)sqrt(nz->h);
  out.sqrt_h12 = (T)sqrt(nz->h / 12.0);
  out.ht = (T)nz->h_total;
  if (nz->source == TSDE_SRC_MEMORY && !nz->w) return TSDE_EINVAL;
  if (nz->source == TSDE_SRC_MEMORY && nz->want_u && !nz->u) return TSDE_EINVAL;
  if (nz->source == TSDE_SRC_COUNTER && !nz->key) return TSDE_EINVAL;
  // the channels drawn: m (the row-wise kernels draw one per column of d, d = m for diagonal noise)
  if (nz->source == TSDE_SRC_COUNTER && !bcast &&
      (L->m > kMaxCounterChannels || (L->noise_type == TSDE_NOISE_DIAGONAL && L->d > kMaxCounterChannels)))
    return TSDE_EINVAL;
  return 0;
}

// How a flat quad index maps to (row, quad of the row) over (rows, d): the d, qpr, nquads, qshift, small and qmagic
// members of a kernel parameter struct (EwP, and the whole-step kernels of pointwise.cu).
template <typename P>
inline void fill_quad_map(int64_t rows, int64_t d, P& p) {
  p.d = d;
  p.qpr = (d + 3) / 4;
  p.nquads = rows * p.qpr;
  p.qshift = -1;
  if ((p.qpr & (p.qpr - 1)) == 0 && p.qpr < (1ll << 30)) {
    int sh = 0;
    while ((1ll << sh) < p.qpr) ++sh;
    p.qshift = sh;
  }
  p.small = p.nquads < (1ll << 31) ? 1 : 0;
  p.qmagic = p.qshift < 0 ? rowdiv_magic((uint64_t)p.qpr) : 0;
}

template <typename T, typename Op>
inline int launch_ew(const tsde_launch* L, const tsde_noise* nz, bool bcast,
                     const void* const* ins, void* const* outs, const Op& op) {
  EwP<Op::NIN, Op::NOUT> p{};
  bool vec = (L->d % 4) == 0;
  uint32_t fmt = 0, ofmt = 0;
  if constexpr (is_mixed<Op>::value) {
    fmt = op.fmt;
    ofmt = op.ofmt;
  }
  for (int i = 0; i < Op::NIN; ++i) {
    if (!ins[i]) return TSDE_EINVAL;
    p.in[i] = ins[i];
    vec = vec && aligned_for(ins[i], operand_fmt(fmt, i));
  }
  for (int i = 0; i < Op::NOUT; ++i) {
    if (!outs[i]) return TSDE_EINVAL;
    p.out[i] = outs[i];
    vec = vec && aligned_for(outs[i], operand_fmt(ofmt, i));
  }
  NoiseP<T> np;
  if (int e = fill_noise<T>(L, Op::USES_NOISE ? nz : nullptr, bcast, np)) return e;
  const int src = (Op::USES_NOISE && nz) ? nz->source : TSDE_SRC_UNIT;
  if (Op::USES_NOISE && !nz) return TSDE_EINVAL;
  if (src == TSDE_SRC_MEMORY && !bcast) {
    vec = vec && aligned16(np.w) && (!Op::WANT_U || aligned16(np.u));
    if (L->noise_type == TSDE_NOISE_DIAGONAL && L->m != L->d) return TSDE_EINVAL;
  }
  p.rows = L->rows;
  p.vec = vec ? 1 : 0;
  fill_quad_map(L->rows, L->d, p);
  // (every quads-per-row divides exactly on the fast path: its quad indices are 32-bit, see rowdiv.cuh)
  const bool fast = p.vec && !bcast && p.small && np.n_cells == 1 &&
                    (L->rows + (nz ? nz->row_offset : 0)) < kMaxGlobalRows;
  const cudaStream_t stream = reinterpret_cast<cudaStream_t>(L->stream);
  auto go = [&](auto kernel) -> int {
    // Persistent, balanced grid: small problems get one quad per thread, large ones one wave of resident CTAs, each
    // owning an equal contiguous slice.
    int per_sm = resident_ctas(reinterpret_cast<const void*>(kernel), kThreads, 0);
    if (per_sm < 1) per_sm = 1;
    return launch_kernel(kernel, capped_grid(p.nquads, kThreads, per_sm), kThreads, 0, stream, false, p, np, op);
  };
  auto go_fast = [&](auto kernel) -> int {  // programmatic dependent launch (see ew_fast_kernel)
    return launch_kernel(kernel, fast_chunks<T, Op>((uint32_t)p.nquads), kThreads, 0, stream, true, p, np, op);
  };
  if constexpr (!Op::USES_NOISE) {
    if (fast) return go_fast(ew_fast_kernel<T, Op, TSDE_SRC_UNIT>);
    return go(ew_kernel<T, Op, TSDE_SRC_UNIT>);
  } else {
    if (fast) {
      switch (src) {
        case TSDE_SRC_MEMORY: return go_fast(ew_fast_kernel<T, Op, TSDE_SRC_MEMORY>);
        case TSDE_SRC_COUNTER: return go_fast(ew_fast_kernel<T, Op, TSDE_SRC_COUNTER>);
        case TSDE_SRC_UNIT: return go_fast(ew_fast_kernel<T, Op, TSDE_SRC_UNIT>);
        default: return TSDE_EINVAL;
      }
    }
    switch (src) {
      case TSDE_SRC_MEMORY:
        return go(ew_kernel<T, Op, TSDE_SRC_MEMORY>);
      case TSDE_SRC_COUNTER:
        if (np.n_cells > 1) return go(ew_kernel<T, Op, kSrcCounterMulti>);
        return go(ew_kernel<T, Op, TSDE_SRC_COUNTER>);
      case TSDE_SRC_UNIT:
        return go(ew_kernel<T, Op, TSDE_SRC_UNIT>);
      default:
        return TSDE_EINVAL;
    }
  }
}

}  // namespace tsde
