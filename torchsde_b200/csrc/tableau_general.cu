// Step tableaus for general / additive noise: g:(rows,d,m), dW:(rows,m).
//
// The batched matrix-vector product of the reference (`misc.batch_mvp` = torch.bmm(g, v[...,None]),
// torchsde/_core/misc.py:62-63, reached through base_sde.py:101-102) is fused with the tableau's
// element-wise combination: g — the only large operand, used exactly once (0.5 flop/byte, HBM
// bound; tensor cores cannot help, SURVEY.md fact 5) — is streamed once, and the Brownian
// increments of the rows a CTA owns are produced once (Philox, or a load of the user's tensor)
// into shared memory, so they are not regenerated d times.  `launch_gen` picks the kernel by shape:
//   * m / 4 a power of two <= 32, every g quad-aligned (memory noise: W / U 16-byte aligned):
//     gen_tma_kernel (TMA-staged, persistent) for 32/64-bit operands at m = 64, or m = 16 with one
//     g operand, when d is a power of two, g is not batch-broadcast and the batch fills its
//     pipeline; gen_cta_kernel (one 128-thread CTA per 32 / (m/4) rows, 128-bit loads) otherwise.
//   * every other shape whose row of increments fits in 40 KiB of shared memory: gen_kernel, one
//     thread per (row, d) output walking its m-run of g;
//   * rows wider than that: gen_wide_kernel, one CTA per row walking m in chunks.
//
// Summation order: fixed per kernel (see each kernel) and independent of batch sharding, so results
// are bitwise reproducible; they agree with torch.bmm to rounding (bmm's own order is
// unspecified), which is how the parity tests treat them.
#include <atomic>
#include <type_traits>

#include "ew.cuh"

namespace tsde {

constexpr int kMaxRowsPerBlock = 64;

template <int NE, int NG, int NO>
struct GenP {
  const void* e[NE > 0 ? NE : 1];
  const void* g[NG];
  void* o[NO];
  int64_t rows, d, m;
  int32_t mq;    // m / 4 (gen_cta_kernel)
  int32_t rb;    // rows per block
  int32_t vec;   // m % 4 == 0 and every g aligned for quad loads (gen_wide_kernel)
  int32_t gbcast;  // every g operand is ONE (d, m) block shared by all rows (row stride 0): additive noise whose
                   // diffusion does not depend on y, returned as `sigma.expand(B, d, m)`.  Nothing of size
                   // (rows, d, m) exists then; the block (d*m*s bytes, KiBs) is served from L1/L2.
};

// Op interface:
//   static constexpr int NE, NG, NP, NO;  static constexpr bool WANT_U;
//   T gval(int p, const T (&g)[NG]) const;      value contracted in product p
//   T weight(int p, T w, T u) const;            weight of product p for this Brownian channel
//   void combine(const T (&e)[NE], const T (&gp)[NP], T (&o)[NO]) const;

// ---- pieces the kernels share --------------------------------------------------------------------------------------
// Quad q of row `row` of the increments (W, and U when WANT_U) -> shared memory at sw / su + r * m + 4 * q, one 128-bit
// store per tensor: drawn on the channel-quad counters (MULTI: merging nz.n_cells primary cells when there are several)
// or, for memory noise, one 128-bit load of the user's (rows, m) tensors.
template <bool WANT_U, int SRC, bool MULTI, typename T>
__device__ __forceinline__ void stage_quad(const NoiseP<T>& nz, Key key, int64_t row, int m, int r, int q, T* sw,
                                           T* su) {
  T w[4], u[4];
  if (SRC == TSDE_SRC_MEMORY) {
    const int64_t base = row * m + 4 * q;
    ld4(nz.w + base, w);
    if (WANT_U) ld4(nz.u + base, u);
  } else {
    counter_noise<T, WANT_U, MULTI>(nz, key, (uint32_t)(row + nz.row_offset), (uint32_t)q, w, u);
  }
  st4(sw + r * m + 4 * q, w);
  if (WANT_U) st4(su + r * m + 4 * q, u);
}

// The element-wise operands at eoff (Mixed<Op>: raw bits, converted by widen_e).
template <typename T, typename Op, int N>
__device__ __forceinline__ void load_e(const GenP<Op::NE, Op::NG, Op::NO>& p, const Op& op, int64_t eoff,
                                       T (&e)[N]) {
#pragma unroll
  for (int i = 0; i < Op::NE; ++i) {
    if constexpr (is_mixed<Op>::value) e[i] = __uint_as_float(ld1raw(p.e[i], eoff, operand_fmt(op.fmt, i)));
    else e[i] = reinterpret_cast<const T*>(p.e[i])[eoff];
  }
}
template <typename Op, int N>
__device__ __forceinline__ void widen_e(const Op& op, float (&e)[N]) {
#pragma unroll
  for (int i = 0; i < Op::NE; ++i) e[i] = widen1(__float_as_uint(e[i]), operand_fmt(op.fmt, i));
}

// Epilogue of one (row, d) output: its element-wise operands at eoff, the tableau on the contracted products gp, the
// outputs stored at eoff.
template <typename T, typename Op, int NP>
__device__ __forceinline__ void epilogue(const GenP<Op::NE, Op::NG, Op::NO>& p, const Op& op, int64_t eoff,
                                         const T (&gp)[NP]) {
  T e[Op::NE > 0 ? Op::NE : 1], o[Op::NO];
  load_e(p, op, eoff, e);
  if constexpr (is_mixed<Op>::value) widen_e(op, e);
  op.combine(e, gp, o);
#pragma unroll
  for (int i = 0; i < Op::NO; ++i) reinterpret_cast<T*>(p.o[i])[eoff] = o[i];
}

// ---- generic path: any m, any alignment ----------------------------------------------------------------------------
// rb rows per CTA.  Their increments are staged in shared memory element by element (row r at r * m, for any m); then
// one thread per (row, d) output walks its m-run of g left to right, one separately rounded multiply-add per channel.
template <typename T, typename Op, int SRC>
__global__ void __launch_bounds__(kThreads)
gen_kernel(const GenP<Op::NE, Op::NG, Op::NO> p, const NoiseP<T> nz, const Op op) {
  constexpr int NE = Op::NE, NG = Op::NG, NP = Op::NP;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* sw = reinterpret_cast<T*>(smem_raw);
  T* su = sw + (size_t)p.rb * p.m;

  const int64_t row0 = (int64_t)blockIdx.x * p.rb;
  const int nrows = (int)((p.rows - row0) < p.rb ? (p.rows - row0) : p.rb);
  const int64_t m = p.m, d = p.d;

  // ---- phase 1: Brownian increments of this block's rows -> shared memory ------------------
  {
    Key key{0u, 0u};
    if (SRC == TSDE_SRC_COUNTER) key = load_key(nz.key);
    const int qpr = (int)((m + 3) / 4);
    for (int i = threadIdx.x; i < nrows * qpr; i += kThreads) {
      const int r = i / qpr, q = i - r * qpr;
      const int64_t rem = m - 4 * q;
      const int nvalid = rem < 4 ? (int)rem : 4;
      T w[4], u[4];
      if (SRC == TSDE_SRC_COUNTER) {
        counter_noise<T, Op::WANT_U>(nz, key, (uint32_t)(row0 + r + nz.row_offset), (uint32_t)q, w, u);
      } else {
        const int64_t base = (row0 + r) * m + 4 * q;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          w[j] = j < nvalid ? nz.w[base + j] : T(0);
          u[j] = (Op::WANT_U && j < nvalid) ? nz.u[base + j] : T(0);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < nvalid) {
          sw[r * m + 4 * q + j] = w[j];
          if (Op::WANT_U) su[r * m + 4 * q + j] = u[j];
        }
    }
  }
  __syncthreads();

  // ---- phase 2: stream g, contract, combine ----------------------------------------------------
  const int64_t total = (int64_t)nrows * d;
  for (int64_t c = threadIdx.x; c < total; c += kThreads) {
    const int r = (int)(c / d);
    const int64_t dd = c - (int64_t)r * d;
    const int64_t goff = ((p.gbcast ? 0 : (row0 + r) * d) + dd) * m;
    T part[NP];
#pragma unroll
    for (int k = 0; k < NP; ++k) part[k] = T(0);
    for (int64_t mm = 0; mm < m; ++mm) {
      const T w = sw[r * m + mm];
      const T u = Op::WANT_U ? su[r * m + mm] : T(0);
      T gj[NG];
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if constexpr (is_mixed<Op>::value)
          gj[i] = __uint_as_float(ld1raw(p.g[i], goff + mm, operand_fmt(op.fmt, NE + i)));
        else gj[i] = reinterpret_cast<const T*>(p.g[i])[goff + mm];
      }
      if constexpr (is_mixed<Op>::value) {
#pragma unroll
        for (int i = 0; i < NG; ++i) gj[i] = widen1(__float_as_uint(gj[i]), operand_fmt(op.fmt, NE + i));
      }
#pragma unroll
      for (int k = 0; k < NP; ++k) part[k] = part[k] + op.gval(k, gj) * op.weight(k, w, u);
    }
    epilogue(p, op, (row0 + r) * d + dd, part);
  }
}

// ---- fast path (m % 4 == 0, m/4 a power of two <= 32) ------------------------------------------
// One small CTA (128 threads) per group of RW = 32 / (m/4) consecutive rows: the first warp
// produces the group's RW x m increments (one Philox quad per lane) into shared memory, then
// all four warps stream the group's g tile (RW x d x m contiguous floats) with kGenUnroll
// independent 128-bit loads per thread in flight.  Many small CTAs keep the whole tile set in
// flight at once, which is what matters at the batch sizes of general-noise SDEs (tens of MiB).
constexpr int kGenUnroll = 4;
constexpr int kGenThreads = 128;

template <typename T, typename Op, int SRC>
__global__ void __launch_bounds__(kGenThreads)
gen_cta_kernel(const GenP<Op::NE, Op::NG, Op::NO> p, const NoiseP<T> nz, const Op op) {
  constexpr int NE = Op::NE, NG = Op::NG, NP = Op::NP, NO = Op::NO;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x;
  const int m = (int)p.m, mq = p.mq, rw = p.rb;  // rb = rows per group here
  const int mq_shift = __ffs(mq) - 1;
  T* sw = reinterpret_cast<T*>(smem_raw);
  T* su = sw + rw * m;
  const int per_row = (int)p.d * mq;
  const int64_t row0 = (int64_t)blockIdx.x * rw;
  const int nrows = (int)((p.rows - row0) < rw ? (p.rows - row0) : rw);
  // Programmatic dependent launch: the counter-based increments do not depend on the predecessor
  // kernel's outputs, so they are produced before `griddepcontrol.wait`; user-supplied increments
  // (MEMORY source) and all of g / e are read after it.
  if (SRC == TSDE_SRC_MEMORY) asm volatile("griddepcontrol.wait;" ::: "memory");
  // phase 1: increments of the group's rows (<= 32 quads)
  if (tid < nrows * mq) {
    Key key{0u, 0u};
    if (SRC == TSDE_SRC_COUNTER) key = load_key(nz.key);
    const int r = tid >> mq_shift, q = tid & (mq - 1);
    stage_quad<Op::WANT_U, SRC, true>(nz, key, row0 + r, m, r, q, sw, su);
  }
  if (SRC != TSDE_SRC_MEMORY) asm volatile("griddepcontrol.wait;" ::: "memory");
  // Streaming sweep over the group's g tile (contiguous: element offset = tile0 + 4 * chunk).
  // Index arithmetic is hoisted: a thread's Brownian quad `mc` never changes (128 % mq == 0), its
  // (row, d) position advances by a constant number of (row, d) slots per load, tracked incrementally.
  const int total = nrows * per_row;
  const int64_t tile0 = row0 * p.d * m;          // first g element of the group
  const int64_t slot0 = row0 * p.d;               // first (row, d) slot of the group
  const int mc = tid & (mq - 1);
  const int d = (int)p.d;
  const int slots_per_load = kGenThreads >> mq_shift;
  int slot = tid >> mq_shift;                      // (row, d) slot of this thread's next chunk
  int r = slot / d;                                // row inside the group (one division per thread)
  int dd = slot - r * d;
  bool synced = false;
  for (int base = 0; base < total; base += kGenThreads * kGenUnroll) {  // CTA-uniform trip count
    const int c0 = base + tid;
    T gv[kGenUnroll][NG][4];
    T ev[kGenUnroll][NE > 0 ? NE : 1];  // element-wise operands, fetched together with g (not after the reduce)
    uint4 graw[kGenUnroll][NG];  // (Mixed: raw bits, widened once every load of the pass has been issued)
    int rr[kGenUnroll], slots[kGenUnroll];
    bool valid[kGenUnroll];
#pragma unroll
    for (int un = 0; un < kGenUnroll; ++un) {
      const int c = c0 + un * kGenThreads;
      valid[un] = c < total;
      rr[un] = r;
      slots[un] = slot;
      // element offset of this chunk inside a g operand: contiguous tile, or — batch-broadcast g — the chunk's
      // position inside the one shared (d, m) block
      const int64_t goff = p.gbcast ? (int64_t)4 * (dd * mq + mc) : tile0 + 4 * (int64_t)c;
      if (valid[un] && mc == 0) load_e(p, op, slot0 + slot, ev[un]);
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if (valid[un]) {
          if constexpr (is_mixed<Op>::value) {
            const uint32_t f = operand_fmt(op.fmt, NE + i);
            if (streams_inputs<Op>::value && !p.gbcast) graw[un][i] = ld4raw<true>(p.g[i], goff, f);
            else graw[un][i] = ld4raw<false>(p.g[i], goff, f);
          } else if (streams_inputs<Op>::value && !p.gbcast) {
            ld4cs(reinterpret_cast<const T*>(p.g[i]) + goff, gv[un][i]);
          } else {
            ld4(reinterpret_cast<const T*>(p.g[i]) + goff, gv[un][i]);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) gv[un][i][j] = T(0);
          if constexpr (is_mixed<Op>::value) graw[un][i] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      slot += slots_per_load;
      dd += slots_per_load;
      while (dd >= d) { dd -= d; ++r; }
    }
    if (!synced) { __syncthreads(); synced = true; }  // increments visible (first pass is uniform)
    if constexpr (is_mixed<Op>::value) {
#pragma unroll
      for (int un = 0; un < kGenUnroll; ++un) {
#pragma unroll
        for (int i = 0; i < NG; ++i) widen4(graw[un][i], operand_fmt(op.fmt, NE + i), gv[un][i]);
        widen_e(op, ev[un]);
      }
    }
#pragma unroll
    for (int un = 0; un < kGenUnroll; ++un) {
      T part[NP];
#pragma unroll
      for (int k = 0; k < NP; ++k) part[k] = T(0);
      T w4[4], u4[4];
      const int rs = valid[un] ? rr[un] : 0;
      ld4(sw + rs * m + 4 * mc, w4);
      if (Op::WANT_U) ld4(su + rs * m + 4 * mc, u4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        T gj[NG];
#pragma unroll
        for (int i = 0; i < NG; ++i) gj[i] = gv[un][i][j];
#pragma unroll
        for (int k = 0; k < NP; ++k)  // fused multiply-add: the contraction's rounding is not pinned (bmm)
          part[k] = fma(op.gval(k, gj), op.weight(k, w4[j], Op::WANT_U ? u4[j] : T(0)), part[k]);
      }
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        if (off < mq) {  // uniform
#pragma unroll
          for (int k = 0; k < NP; ++k) part[k] = part[k] + __shfl_xor_sync(0xffffffffu, part[k], off);
        }
      }
      if (valid[un] && mc == 0) {
        const int64_t eoff = slot0 + slots[un];
        T e[NE > 0 ? NE : 1], o[NO];
#pragma unroll
        for (int i = 0; i < NE; ++i) e[i] = ev[un][i];
        op.combine(e, part, o);
#pragma unroll
        for (int i = 0; i < NO; ++i) reinterpret_cast<T*>(p.o[i])[eoff] = o[i];
      }
    }
  }
  if (!synced) __syncthreads();
}

// ---- TMA-staged persistent path (large batches) -------------------------------------------------
// For g tensors much larger than what one wave of small CTAs keeps in flight, the tile stream is
// driven by the copy engine instead of by per-thread loads: a persistent CTA owns a contiguous
// range of row groups ("tiles": rs rows, i.e. rs*d*m contiguous elements of every g operand and
// rs*d of every element-wise operand) and keeps kTmaStages tiles in flight with 1-D bulk copies
// (`cp.async.bulk.shared::cluster.global`, completion counted in bytes on an mbarrier per stage).
// Warp-specialised: a producer warp arms each stage's `full` barrier, issues the copies (one lane)
// and produces the tile's Brownian increments into the same stage (all lanes, Philox in registers);
// eight consumer warps wait on the barrier's phase parity, contract out of shared memory with the
// same chunk -> lane mapping and summation order as `gen_cta_kernel` (so both paths are
// bit-identical), and hand the stage back through an `empty` barrier (one arrive per warp).  There
// is no CTA-wide barrier in the steady state.
// Consumer: two phases without shuffles (lane-per-chunk partial dot products to a shared scratch array, then
// lane-per-output pairwise tree + coalesced epilogue), bit-identical to gen_cta_kernel's xor-shuffle tree.

constexpr int kTmaThreads = 256;
constexpr int kTmaStages = 4;
constexpr int kTmaUnroll = 4;

struct TmaP {
  int64_t n_tiles;
  int32_t rs;            // rows per tile
  uint32_t g_stride;     // bytes between the g operands of one stage (128-byte multiple)
  uint32_t e_stride;     // bytes between the element-wise operands of one stage
  uint32_t w_stride;     // bytes of one increment buffer (rs x m elements, 128-byte multiple)
  int32_t d_shift;       // log2(d)
  uint32_t stage_stride; // bytes per stage
  uint32_t scratch_np_stride;  // bytes of one array of per-chunk partial dot products (one per product of the tableau)
  uint32_t scratch_stride;     // bytes of one scratch buffer (NP arrays); two buffers follow the stages
};

__device__ __forceinline__ uint32_t smem_u32(const void* ptr) {
  return (uint32_t)__cvta_generic_to_shared(ptr);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void lds4(uint32_t addr, float (&v)[4]) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "r"(addr));
}
__device__ __forceinline__ void lds4(uint32_t addr, double (&v)[4]) {
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v[0]), "=d"(v[1]) : "r"(addr));
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v[2]), "=d"(v[3]) : "r"(addr + 16u));
}
template <typename T>
__device__ __forceinline__ T lds1(uint32_t addr);
template <>
__device__ __forceinline__ float lds1<float>(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
template <>
__device__ __forceinline__ double lds1<double>(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts1(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void sts1(uint32_t addr, double v) {
  asm volatile("st.shared.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
template <bool EVICT_FIRST>
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
  if (EVICT_FIRST) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
  } else {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
  }
}

template <typename T, typename Op, int SRC, int MQ_SHIFT>
__global__ void __launch_bounds__(kTmaThreads + 32)
gen_tma_kernel(const GenP<Op::NE, Op::NG, Op::NO> p, const NoiseP<T> nz, const Op op, const TmaP tp) {
  constexpr int NE = Op::NE, NG = Op::NG, NP = Op::NP, NO = Op::NO;
  constexpr bool kEvictFirst = streams_inputs<Op>::value;
  constexpr int kConsumerWarps = kTmaThreads / 32;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw);  // [kTmaStages] tile + increments have landed
  uint64_t* empty = full + kTmaStages;                      // [kTmaStages] every consumer warp is done
  unsigned char* stages = smem_raw + 128;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  constexpr int mq = 1 << MQ_SHIFT, mq_shift = MQ_SHIFT;  // m / 4, compile-time: the shuffle tree is static
  const int m = (int)p.m, d = (int)p.d, rs = tp.rs;
  const int d_shift = tp.d_shift;                          // d is a power of two on this path
  const int64_t t_begin = (tp.n_tiles * blockIdx.x) / gridDim.x;
  const int64_t t_end = (tp.n_tiles * (blockIdx.x + 1)) / gridDim.x;
  const int n_my = (int)(t_end - t_begin);
  auto rows_of = [&](int64_t t) -> int {
    const int64_t left = p.rows - t * rs;
    return left < rs ? (int)left : rs;
  };
  // stage layout: NG g tiles | NE element-wise tiles | increments W (rs x m) | U (rs x m, if wanted)
  auto stage_ptr = [&](int s) -> unsigned char* { return stages + (size_t)s * tp.stage_stride; };
  const uint32_t w_off = NG * tp.g_stride + NE * tp.e_stride;
  const uint32_t u_off = w_off + tp.w_stride;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kTmaStages; ++s) {
      mbar_init(&full[s], 2);                 // the copy-issuing arrive (+ its byte count) and the increments' arrive
      mbar_init(&empty[s], kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ---------------- producer warp: bulk copies (lane 0) and Brownian increments (all lanes) ----------
    Key key{0u, 0u};
    if (SRC == TSDE_SRC_COUNTER) key = load_key(nz.key);
    uint64_t policy = 0;
    if (kEvictFirst) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
    bool waited = false;  // griddepcontrol.wait once, before the first read of global memory
    for (int it = 0; it < n_my; ++it) {
      const int s = it % kTmaStages;
      const int64_t t = t_begin + it;
      const int nr = rows_of(t);
      unsigned char* sp = stage_ptr(s);
      if (it >= kTmaStages) mbar_wait(&empty[s], (uint32_t)(((it / kTmaStages) - 1) & 1));
      if (!waited) { asm volatile("griddepcontrol.wait;" ::: "memory"); waited = true; }
      // copies first (asynchronous), then the increments while the bytes are in flight
      if (lane == 0) {
        const uint32_t gb = (uint32_t)((size_t)nr * d * m * sizeof(T));
        const uint32_t eb = (uint32_t)((size_t)nr * d * sizeof(T));
        mbar_arrive_expect_tx(&full[s], NG * gb + NE * eb);
#pragma unroll
        for (int i = 0; i < NG; ++i)
          bulk_g2s<kEvictFirst>(sp + (size_t)i * tp.g_stride,
                                reinterpret_cast<const T*>(p.g[i]) + t * rs * (int64_t)d * m, gb, &full[s], policy);
#pragma unroll
        for (int i = 0; i < NE; ++i)
          bulk_g2s<false>(sp + (size_t)NG * tp.g_stride + (size_t)i * tp.e_stride,
                          reinterpret_cast<const T*>(p.e[i]) + t * rs * (int64_t)d, eb, &full[s], 0);
      }
      T* swb = reinterpret_cast<T*>(sp + w_off);
      T* sub = reinterpret_cast<T*>(sp + u_off);
      for (int i = lane; i < nr * mq; i += 32) {  // one Philox quad per lane and pass
        const int r = i >> mq_shift, q = i & (mq - 1);
        stage_quad<Op::WANT_U, SRC, true>(nz, key, t * rs + r, m, r, q, swb, sub);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[s]);  // increments written (ordered by __syncwarp; arrive releases)
    }
    return;
  }

  // ---------------- consumer warps: contract out of shared memory, combine, store ----------------------
  // Two phases per tile, both with consecutive lanes on consecutive shared-memory words (conflict-free):
  //   1. lane-per-chunk: chunk c (4 consecutive elements of the tile, (row, d) slot c >> MQ_SHIFT, Brownian
  //      quad c & (mq - 1)) -> its 4-term dot product with the increments (the same FMA chain as
  //      gen_cta_kernel), written to a scratch array in shared memory;
  //   2. lane-per-output: slot s sums its mq partials with the same pairwise tree as gen_cta_kernel's
  //      xor-shuffle (so the result is bit-identical), applies the tableau and stores — coalesced.
  // No shuffles, no predicated epilogue in the hot loop: ~12 instructions per 16-byte chunk instead of ~65.
  // The scratch array is double-buffered, so one consumer-wide named barrier per tile suffices.
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the predecessor's reads of our outputs are complete
  const uint32_t stage0_addr = smem_u32(stages);
  const uint32_t scratch0_addr = stage0_addr + (uint32_t)kTmaStages * tp.stage_stride;
  const uint32_t mcq = (uint32_t)(tid & (mq - 1)) * 4u * (uint32_t)sizeof(T);  // byte offset of this lane's quad in a row of W
  for (int it = 0; it < n_my; ++it) {
    const int s = it % kTmaStages;
    const int64_t t = t_begin + it;
    const int nrows = rows_of(t);
    const int nslots = nrows << d_shift;                 // (row, d) outputs of this tile
    const int total = nslots << mq_shift;                // chunks in this tile
    const int64_t slot0 = (t * rs) << d_shift;           // first (row, d) slot of the tile
    const uint32_t sp = stage0_addr + (uint32_t)s * tp.stage_stride;
    const uint32_t e_addr = sp + NG * tp.g_stride;
    const uint32_t w_addr = sp + w_off + mcq;
    const uint32_t u_addr = w_addr + tp.w_stride;
    const uint32_t scr = scratch0_addr + (uint32_t)(it & 1) * tp.scratch_stride;  // [NP][chunks] partials
    mbar_wait(&full[s], (uint32_t)((it / kTmaStages) & 1));
    // ---- phase 1 ----
    for (int base = 0; base < total; base += kTmaThreads * kTmaUnroll) {
      T gv[kTmaUnroll][NG][4];
#pragma unroll
      for (int un = 0; un < kTmaUnroll; ++un) {
        const int c = base + un * kTmaThreads + tid;
        if (c < total) {
#pragma unroll
          for (int i = 0; i < NG; ++i) lds4(sp + (uint32_t)i * tp.g_stride + (uint32_t)c * 4u * (uint32_t)sizeof(T), gv[un][i]);
        }
      }
#pragma unroll
      for (int un = 0; un < kTmaUnroll; ++un) {
        const int c = base + un * kTmaThreads + tid;
        if (c < total) {
          const uint32_t row = ((uint32_t)c >> mq_shift) >> d_shift;
          T w4[4], u4[4];
          lds4(w_addr + row * (uint32_t)m * (uint32_t)sizeof(T), w4);
          if (Op::WANT_U) lds4(u_addr + row * (uint32_t)m * (uint32_t)sizeof(T), u4);
          T part[NP];
#pragma unroll
          for (int k = 0; k < NP; ++k) part[k] = T(0);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            T gj[NG];
#pragma unroll
            for (int i = 0; i < NG; ++i) gj[i] = gv[un][i][j];
#pragma unroll
            for (int k = 0; k < NP; ++k)
              part[k] = fma(op.gval(k, gj), op.weight(k, w4[j], Op::WANT_U ? u4[j] : T(0)), part[k]);
          }
#pragma unroll
          for (int k = 0; k < NP; ++k)
            sts1(scr + ((uint32_t)k * tp.scratch_np_stride) + (uint32_t)c * (uint32_t)sizeof(T), part[k]);
        }
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kTmaThreads) : "memory");  // consumer warps only: partials visible
    // ---- phase 2 ----
    for (int slot = tid; slot < nslots; slot += kTmaThreads) {
      T gp[NP];
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        T pp[mq];
        const uint32_t a = scr + (uint32_t)k * tp.scratch_np_stride + ((uint32_t)slot << mq_shift) * (uint32_t)sizeof(T);
        if (mq >= 4) {
#pragma unroll
          for (int q = 0; q < mq / 4; ++q) {
            T v[4];
            lds4(a + (uint32_t)q * 4u * (uint32_t)sizeof(T), v);
#pragma unroll
            for (int j = 0; j < 4; ++j) pp[(4 * q + j) & (mq - 1)] = v[j];
          }
        } else {
#pragma unroll
          for (int q = 0; q < mq; ++q) pp[q] = lds1<T>(a + (uint32_t)q * (uint32_t)sizeof(T));
        }
        // pairwise tree in natural order == the xor-shuffle tree seen from lane 0
#pragma unroll
        for (int w = 1; w < mq; w <<= 1) {
#pragma unroll
          for (int i = 0; i + w < mq; i += 2 * w) pp[i] = pp[i] + pp[i + w];
        }
        gp[k] = pp[0];
      }
      T e[NE > 0 ? NE : 1], o[NO];
#pragma unroll
      for (int i = 0; i < NE; ++i) e[i] = lds1<T>(e_addr + (uint32_t)i * tp.e_stride + (uint32_t)slot * (uint32_t)sizeof(T));
      op.combine(e, gp, o);
#pragma unroll
      for (int i = 0; i < NO; ++i) reinterpret_cast<T*>(p.o[i])[slot0 + slot] = o[i];
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);  // this warp no longer reads stage s
  }
}

// Which tiles take the TMA-staged kernel, when the batch fills the pipeline: m = 64 always, and m = 16 for tableaus
// with ONE g operand (with two g operands the per-thread-load kernel already keeps enough bytes in flight); m = 8 and
// m = 32 stay on the per-thread-load kernel.  Both kernels are bit-identical (tests/test_gpu_general_tma.py), so the
// route never changes results.  gen_tma_kernel is instantiated for exactly these (op, m / 4) pairs.
template <typename Op>
constexpr bool tma_route(int64_t mq) { return mq == 16 || (Op::NG == 1 && mq == 4); }

constexpr int kTmaNotEligible = -12345;

template <typename T, typename Op>
static int launch_gen_tma(const tsde_launch* L, const tsde_noise* nz, GenP<Op::NE, Op::NG, Op::NO> p,
                          const NoiseP<T>& np, const Op& op, cudaStream_t st) {
  // Eligibility: bulk copies need 16-byte aligned, 16-byte-multiple extents for every operand tile.
  if (L->d % 4 != 0 || (L->d & (L->d - 1)) != 0 || L->d > (1 << 20)) return kTmaNotEligible;  // d = 2^k >= 4
  for (int i = 0; i < Op::NE; ++i) if (!aligned16(p.e[i])) return kTmaNotEligible;
  const int64_t mq = L->m / 4;
  const size_t row_bytes = (size_t)L->d * L->m * sizeof(T);
  // 16 KiB of every g operand per stage (several resident CTAs per SM keep the ring full; the 200 KiB cap below stays
  // within the 227 KiB of shared memory one CTA may use)
  constexpr size_t kStageTarget = (size_t)Op::NG * 16 * 1024;
  if (Op::NG * row_bytes > 32 * 1024 && Op::NG * row_bytes > kStageTarget) return kTmaNotEligible;
  int64_t rs = (int64_t)(kStageTarget / (Op::NG * row_bytes));
  if (rs < 1) rs = 1;
  if (rs > kTmaThreads / mq) rs = kTmaThreads / mq;
  auto up128 = [](size_t x) { return (x + 127) & ~(size_t)127; };
  TmaP tp{};
  tp.rs = (int32_t)rs;
  for (tp.d_shift = 0; (1ll << tp.d_shift) < L->d; ++tp.d_shift) {}
  tp.g_stride = (uint32_t)up128((size_t)rs * row_bytes);
  tp.e_stride = (uint32_t)up128((size_t)rs * L->d * sizeof(T));
  tp.w_stride = (uint32_t)up128((size_t)rs * L->m * sizeof(T));
  tp.stage_stride = (uint32_t)(Op::NG * tp.g_stride + Op::NE * tp.e_stride + (Op::WANT_U ? 2 : 1) * tp.w_stride);
  tp.n_tiles = (L->rows + rs - 1) / rs;
  tp.scratch_np_stride = (uint32_t)up128((size_t)rs * L->d * mq * sizeof(T));
  tp.scratch_stride = (uint32_t)(Op::NP * tp.scratch_np_stride);
  const size_t smem = 128 + (size_t)kTmaStages * tp.stage_stride + 2 * (size_t)tp.scratch_stride;
  if (smem > 200 * 1024) return kTmaNotEligible;
  p.rb = (int32_t)rs;
  auto go = [&](auto kernel) -> int {
    const int resident = resident_ctas(reinterpret_cast<const void*>(kernel), kTmaThreads + 32, smem);
    if (resident < 1) return kTmaNotEligible;
    const int64_t cap = (int64_t)sm_count() * resident;
    if (tp.n_tiles < 2 * kTmaStages * cap) return kTmaNotEligible;  // too small to fill the pipeline
    g_launches[TSDE_KERNEL_GEN_TMA].fetch_add(1, std::memory_order_relaxed);
    return launch_kernel(kernel, tp.n_tiles < cap ? tp.n_tiles : cap, kTmaThreads + 32, smem, st, true, p, np, op,
                         tp);
  };
  const bool mem = nz->source == TSDE_SRC_MEMORY;
  if constexpr (Op::NG == 1) {
    if (mq == 4) return mem ? go(gen_tma_kernel<T, Op, TSDE_SRC_MEMORY, 2>) : go(gen_tma_kernel<T, Op, TSDE_SRC_COUNTER, 2>);
  }
  return mem ? go(gen_tma_kernel<T, Op, TSDE_SRC_MEMORY, 4>) : go(gen_tma_kernel<T, Op, TSDE_SRC_COUNTER, 4>);  // m = 64
}

// ---- wide rows: one row's increments do not fit in shared memory ---------------------------------------------------
// Taken exactly where `gen_kernel` cannot stage even one row (m * s * (WANT_U ? 2 : 1) > 40 KiB), for any m the
// Brownian source accepts.  One CTA per row walks m in chunks of kWideChunkBytes: the threads produce the chunk's
// increments (one Philox quad per thread and pass, on the channel-quad counters of every other kernel, or a coalesced
// load of the user's W / U) into shared memory once, then each warp takes whole (row, d) outputs and streams their g
// run over the chunk, lanes along the contiguous m axis: quad q of the chunk is lane q % 32's, one 128-bit load per
// operand when g is aligned and m % 4 == 0, else four scalar loads of the same quad.  The running sums of up to
// kWideOutputs outputs stay in shared memory across the chunks; a row with a larger d is walked once per block of
// kWideOutputs outputs, drawing its increments again each time (one extra draw per kWideOutputs g runs).
//
// Summation order, per output and product: a lane sums its quads in increasing order, each quad's four channels left
// to right with fused multiply-adds; the 32 lane sums of a chunk are combined by the xor-tree (offsets 16, 8, 4, 2, 1)
// and the chunk sums are added left to right.  It depends on m alone: the same bits for aligned and unaligned
// operands, for any batch size and for any split of the batch by row_offset.
constexpr int kWideThreads = 256;
constexpr int kWideLoads = 4;               // g quads per lane in flight (over all g operands)
constexpr int kWideChunkBytes = 8 * 1024;   // one chunk of W (and one of U) in shared memory
constexpr int kWideOutputs = 1024;          // outputs per block: their running sums stay in shared memory

template <typename T, typename Op, int SRC>
__global__ void __launch_bounds__(kWideThreads, 1)
gen_wide_kernel(const GenP<Op::NE, Op::NG, Op::NO> p, const NoiseP<T> nz, const Op op) {
  constexpr int NE = Op::NE, NG = Op::NG, NP = Op::NP, NO = Op::NO;
  constexpr int CW = kWideChunkBytes / (int)sizeof(T);  // channels per chunk, a multiple of 4 * 32
  constexpr int UN = kWideLoads / NG;                    // quads per lane and pass
  constexpr int kWarps = kWideThreads / 32;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* sw = reinterpret_cast<T*>(smem_raw);
  T* su = sw + CW;
  T* tot = sw + (Op::WANT_U ? 2 : 1) * CW;  // [NP][outputs of the block]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t row = blockIdx.x, m = p.m, d = p.d;
  const bool vec = p.vec != 0;
  Key key{0u, 0u};
  if (SRC != TSDE_SRC_MEMORY) key = load_key(nz.key);
  const uint32_t grow = (uint32_t)(row + nz.row_offset);
  const int64_t slot_g = p.gbcast ? 0 : row * d;  // first (d, m) run of this row's g
  for (int64_t d0 = 0; d0 < d; d0 += kWideOutputs) {
    const int nout = (int)(d - d0 < kWideOutputs ? d - d0 : kWideOutputs);
    for (int64_t c0 = 0; c0 < m; c0 += CW) {
      const int len = (int)(m - c0 < CW ? m - c0 : CW);
      const int nq = (len + 3) / 4;
      __syncthreads();  // the previous chunk's increments have been read
      if (SRC != TSDE_SRC_MEMORY) {
        for (int q = tid; q < nq; q += kWideThreads) {
          T w[4], u[4];
          counter_noise<T, Op::WANT_U, SRC == kSrcCounterMulti>(nz, key, grow, (uint32_t)(c0 / 4 + q), w, u);
          st4(sw + 4 * q, w);
          if (Op::WANT_U) st4(su + 4 * q, u);
        }
      } else {
        const int64_t base = row * m + c0;
        for (int i = tid; i < len; i += kWideThreads) {
          sw[i] = nz.w[base + i];
          if (Op::WANT_U) su[i] = nz.u[base + i];
        }
      }
      __syncthreads();
      for (int j = warp; j < nout; j += kWarps) {
        const int64_t goff = (slot_g + d0 + j) * m + c0;
        T part[NP];
#pragma unroll
        for (int k = 0; k < NP; ++k) part[k] = T(0);
        for (int b = 0; b < nq; b += 32 * UN) {
          T gv[UN][NG][4];
          uint4 graw[UN][NG];  // (Mixed: every g load of the pass issued before the first widening)
#pragma unroll
          for (int un = 0; un < UN; ++un) {
            const int q = b + 32 * un + lane;
            const int nv = len - 4 * q;  // valid channels of the quad (<= 0: past the chunk)
#pragma unroll
            for (int i = 0; i < NG; ++i) {
              if constexpr (is_mixed<Op>::value) {
                const uint32_t f = operand_fmt(op.fmt, NE + i);
                if (q >= nq) graw[un][i] = make_uint4(0u, 0u, 0u, 0u);
                else if (vec && streams_inputs<Op>::value && !p.gbcast) graw[un][i] = ld4raw<true>(p.g[i], goff + 4 * q, f);
                else if (vec) graw[un][i] = ld4raw<false>(p.g[i], goff + 4 * q, f);
                else graw[un][i] = load_quad_raw(p.g[i], goff + 4 * q, false, nv, f);
              } else {
                const T* g = reinterpret_cast<const T*>(p.g[i]);
                if (q >= nq) {
#pragma unroll
                  for (int jj = 0; jj < 4; ++jj) gv[un][i][jj] = T(0);
                } else if (vec && streams_inputs<Op>::value && !p.gbcast) {
                  ld4cs(g + goff + 4 * q, gv[un][i]);
                } else {
                  load_quad(g, goff + 4 * q, vec, nv, gv[un][i]);
                }
              }
            }
          }
          if constexpr (is_mixed<Op>::value) {
#pragma unroll
            for (int un = 0; un < UN; ++un) {
#pragma unroll
              for (int i = 0; i < NG; ++i) widen_quad(graw[un][i], vec, operand_fmt(op.fmt, NE + i), gv[un][i]);
            }
          }
#pragma unroll
          for (int un = 0; un < UN; ++un) {
            const int q = b + 32 * un + lane;
            if (q < nq) {
              const int nv = len - 4 * q;
              T w4[4], u4[4];
              ld4(sw + 4 * q, w4);
              if (Op::WANT_U) ld4(su + 4 * q, u4);
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                if (jj < nv) {
                  T gj[NG];
#pragma unroll
                  for (int i = 0; i < NG; ++i) gj[i] = gv[un][i][jj];
#pragma unroll
                  for (int k = 0; k < NP; ++k)
                    part[k] = fma(op.gval(k, gj), op.weight(k, w4[jj], Op::WANT_U ? u4[jj] : T(0)), part[k]);
                }
              }
            }
          }
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
#pragma unroll
          for (int k = 0; k < NP; ++k) part[k] = part[k] + __shfl_xor_sync(0xffffffffu, part[k], off);
        }
        if (lane == 0) {
#pragma unroll
          for (int k = 0; k < NP; ++k) tot[k * nout + j] = c0 == 0 ? part[k] : tot[k * nout + j] + part[k];
        }
      }
    }
    __syncthreads();  // the block's sums are complete
    for (int j = tid; j < nout; j += kWideThreads) {
      const int64_t eoff = row * d + d0 + j;
      T e[NE > 0 ? NE : 1], gp[NP], o[NO];
#pragma unroll
      for (int i = 0; i < NE; ++i) {
        if constexpr (is_mixed<Op>::value) e[i] = __uint_as_float(ld1raw(p.e[i], eoff, operand_fmt(op.fmt, i)));
        else e[i] = reinterpret_cast<const T*>(p.e[i])[eoff];
      }
      if constexpr (is_mixed<Op>::value) {
#pragma unroll
        for (int i = 0; i < NE; ++i) e[i] = widen1(__float_as_uint(e[i]), operand_fmt(op.fmt, i));
      }
#pragma unroll
      for (int k = 0; k < NP; ++k) gp[k] = tot[k * nout + j];
      op.combine(e, gp, o);
#pragma unroll
      for (int i = 0; i < NO; ++i) reinterpret_cast<T*>(p.o[i])[eoff] = o[i];
    }
  }
}

template <typename T, typename Op>
static int launch_gen(const tsde_launch* L, const tsde_noise* nz,
                      std::initializer_list<const void*> es, std::initializer_list<const void*> gs,
                      std::initializer_list<void*> os, const Op& op) {
  if (!nz) return TSDE_EINVAL;
  if (nz->source != TSDE_SRC_MEMORY && nz->source != TSDE_SRC_COUNTER)
    return TSDE_EINVAL;  // (a user-supplied product, TSDE_SRC_UNIT, goes through the element-wise entry points)
  GenP<Op::NE, Op::NG, Op::NO> p{};
  bool vec = (L->m % 4) == 0;  // and every g aligned for quad loads: p.vec
  uint32_t fmt = 0;
  if constexpr (is_mixed<Op>::value) fmt = op.fmt;
  int i = 0;
  for (const void* q : es) { if (!q) return TSDE_EINVAL; p.e[i++] = q; }
  i = 0;
  for (const void* q : gs) {
    if (!q) return TSDE_EINVAL;
    vec = vec && aligned_for(q, operand_fmt(fmt, Op::NE + i));
    p.g[i++] = q;
  }
  i = 0;
  for (void* q : os) { if (!q) return TSDE_EINVAL; p.o[i++] = q; }
  NoiseP<T> np;
  if (int e = fill_noise<T>(L, nz, false, np)) return e;
  const int64_t mq = L->m / 4;
  const bool mem = nz->source == TSDE_SRC_MEMORY;
  const int64_t smem_per_row = L->m * (int64_t)sizeof(T) * (Op::WANT_U ? 2 : 1);
  // the tile kernels: m / 4 a power of two <= 32, g and (memory noise) W / U loadable as quads (gen_route)
  const int route =
      gen_route(L->m, vec && (!mem || (aligned16(np.w) && (!Op::WANT_U || aligned16(np.u)))), smem_per_row);
  const bool tile = route == TSDE_GEN_TILE;
  p.rows = L->rows; p.d = L->d; p.m = L->m;
  p.mq = (int32_t)mq;
  p.vec = vec ? 1 : 0;
  p.gbcast = (nz->flags & TSDE_FLAG_G_BROADCAST) ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  if (tile) {
    // (a broadcast g has no tile stream to stage; 16-bit operands are not staged by the TMA kernel)
    if constexpr (!is_mixed<Op>::value) {
      if (!p.gbcast && tma_route<Op>(mq)) {
        int rc = launch_gen_tma<T, Op>(L, nz, p, np, op, st);
        if (rc != kTmaNotEligible) return rc;
      }
    }
    // one 128-thread CTA per group of rw rows
    const int64_t rw = 32 / mq;
    p.rb = (int32_t)rw;
    const int64_t ngroups = (L->rows + rw - 1) / rw;
    if (ngroups > 0x7fffffffll) return TSDE_EINVAL;
    const size_t smem = (size_t)rw * L->m * sizeof(T) * (Op::WANT_U ? 2 : 1);
    g_launches[TSDE_KERNEL_GEN_CTA].fetch_add(1, std::memory_order_relaxed);
    return launch_kernel(mem ? gen_cta_kernel<T, Op, TSDE_SRC_MEMORY> : gen_cta_kernel<T, Op, TSDE_SRC_COUNTER>,
                         ngroups, kGenThreads, smem, st, true, p, np, op);
  }
  // generic path: rows per block ~16 work items per thread, bounded by shared memory for the increments
  const int64_t per_row = L->d;
  int64_t rb = (16 * kThreads + per_row - 1) / per_row;
  if (rb < 1) rb = 1;
  if (rb > kMaxRowsPerBlock) rb = kMaxRowsPerBlock;
  while (rb > 1 && rb * smem_per_row > 40 * 1024) rb >>= 1;
  if (route == TSDE_GEN_WIDE) {  // not even one row's increments fit: walk m in chunks, one CTA per row
    if (L->rows > 0x7fffffffll) return TSDE_EINVAL;
    p.rb = 1;
    const int64_t outs = L->d < kWideOutputs ? L->d : kWideOutputs;
    const size_t smem = ((Op::WANT_U ? 2 : 1) * (size_t)(kWideChunkBytes / sizeof(T)) + Op::NP * (size_t)outs) * sizeof(T);
    g_launches[TSDE_KERNEL_GEN_WIDE].fetch_add(1, std::memory_order_relaxed);
    const auto kernel = mem                ? gen_wide_kernel<T, Op, TSDE_SRC_MEMORY>
                        : np.n_cells > 1 ? gen_wide_kernel<T, Op, kSrcCounterMulti>
                                         : gen_wide_kernel<T, Op, TSDE_SRC_COUNTER>;
    return launch_kernel(kernel, L->rows, kWideThreads, smem, st, false, p, np, op);
  }
  // keep every SM busy on small batches
  while (rb > 1 && (L->rows + rb - 1) / rb < 2 * sm_count()) rb >>= 1;
  p.rb = (int32_t)rb;
  const int64_t blocks = (L->rows + rb - 1) / rb;
  if (blocks > 0x7fffffffll) return TSDE_EINVAL;
  return launch_kernel(mem ? gen_kernel<T, Op, TSDE_SRC_MEMORY> : gen_kernel<T, Op, TSDE_SRC_COUNTER>, blocks,
                       kThreads, (size_t)(rb * smem_per_row), st, false, p, np, op);
}

// A launch that declares 16-bit SDE outputs (float32 state only, see dispatch_fmt) takes the Mixed<Op> tile kernels;
// `fmt` covers the element-wise operands, then the g operands, in the entry point's order.
template <typename T, typename Op>
static int launch_gen_fmt(const tsde_launch* L, const tsde_noise* nz, std::initializer_list<const void*> es,
                          std::initializer_list<const void*> gs, std::initializer_list<void*> os, const Op& op,
                          uint32_t fmt) {
  if constexpr (std::is_same<T, float>::value) {
    if (fmt) return launch_gen<T>(L, nz, es, gs, os, Mixed<Op>{op, fmt, 0u});
  }
  return launch_gen<T>(L, nz, es, gs, os, op);
}

// ---- ops ---------------------------------------------------------------------------------------
// (GEulerOp, GMidpointPredictOp, GSraStageOp, GSraFinalOp, GEulerHeunPredictOp, GEulerHeunOp, GRevHeunZOp and
// GRevHeunOp: pw_device.cuh, which the run-time compiled general-noise kernels include too)
// y1 = y0 + (dt*(f+f') + g.dW + g'.dW) * 0.5                                     methods/heun.py:46
template <typename T>
struct GHeunOp {
  static constexpr int NE = 3, NG = 2, NP = 2, NO = 1;
  static constexpr bool WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: the g tiles are dead afterwards
  T dt;
  __device__ __forceinline__ T gval(int p, const T (&g)[2]) const { return g[p]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[3], const T (&gp)[2], T (&o)[1]) const {
    o[0] = e[0] + ((dt * (e[1] + e[2]) + gp[0]) + gp[1]) * T(0.5);
  }
};
// ---- outer-product bookkeeping of the reversible-Heun adjoint (g-shaped element-wise) ----------
// out[b,dd,mm] = (base ? base[b,dd,mm] : 0) + a1[b,dd]*(c1*w[b,mm]) (+ a2[b,dd]*(c2*w[b,mm]))
// reversible_heun.py:95-96,105,115 (a) and :114,140 (b)
template <typename T, int SRC>
__global__ void __launch_bounds__(kThreads)
outer_kernel(const NoiseP<T> nz, int64_t rows, int64_t d, int64_t m, const T* base, const T* a1,
             T c1, const T* a2, T c2, T* out) {
  Key key{0u, 0u};
  if (SRC == TSDE_SRC_COUNTER) key = load_key(nz.key);
  const int64_t qpr = (m + 3) / 4;
  const int64_t total = rows * d * qpr;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x; c < total; c += stride) {
    const int64_t bd = c / qpr;
    const int64_t q = c - bd * qpr;
    const int64_t row = bd / d;
    const int64_t rem = m - 4 * q;
    const int nvalid = rem < 4 ? (int)rem : 4;
    T w[4], u[4];
    if (SRC == TSDE_SRC_COUNTER) {
      // d-fold redundant Philox work; this g-shaped pass is off the headline path.
      counter_noise<T, false>(nz, key, (uint32_t)(row + nz.row_offset), (uint32_t)q, w, u);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = j < nvalid ? nz.w[row * m + 4 * q + j] : T(0);
    }
    const T x1 = a1[bd];
    const T x2 = a2 ? a2[bd] : T(0);
    const int64_t off = bd * m + 4 * q;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < nvalid) {
        T v = x1 * (c1 * w[j]);
        if (base) v = base[off + j] + v;
        if (a2) v = v + x2 * (c2 * w[j]);
        out[off + j] = v;
      }
    }
  }
}

template <typename T>
static int launch_outer(const tsde_launch* L, const tsde_noise* nz, const void* base,
                        const void* a1, double c1, const void* a2, double c2, void* out) {
  if (!nz || !a1 || !out) return TSDE_EINVAL;
  if (nz->source != TSDE_SRC_MEMORY && nz->source != TSDE_SRC_COUNTER) return TSDE_EINVAL;
  NoiseP<T> np;
  if (int e = fill_noise<T>(L, nz, false, np)) return e;
  const int64_t total = L->rows * L->d * ((L->m + 3) / 4);
  const auto kernel =
      nz->source == TSDE_SRC_MEMORY ? outer_kernel<T, TSDE_SRC_MEMORY> : outer_kernel<T, TSDE_SRC_COUNTER>;
  return launch_kernel(kernel, capped_grid(total, kThreads, kBlocksPerSM), kThreads, 0,
                       reinterpret_cast<cudaStream_t>(L->stream), false, np, L->rows, L->d, L->m, (const T*)base,
                       (const T*)a1, (T)c1, (const T*)a2, (T)c2, (T*)out);
}

// element-wise (rows,d) parts of the adjoint
template <typename T>
struct AdjAElemOp {  // adj_f0' = adj_f0 + adj_y0*half_dt
  static constexpr int NIN = 2, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[2], T, T, T (&out)[1]) const {
    out[0] = in[1] + in[0] * half_dt;
  }
};
template <typename T>
struct AdjBElemOp {  // in: adj_y0, adj_z0, vjp_z -> adj_y1, adj_z1, adj_f1
  static constexpr int NIN = 3, NOUT = 3;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T dt, half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[3], T, T, T (&out)[3]) const {
    const T adj_y0 = in[0];
    const T adj_z0 = in[1] + in[2];                  // :130
    out[0] = adj_y0 + T(2) * adj_z0;                 // :137
    out[1] = -adj_z0;                                // :138
    out[2] = adj_y0 * half_dt + adj_z0 * dt;         // :112,139
  }
};

// ---- entry points ---------------------------------------------------------------------------------------------------
// The routes of cabi.cu for general noise with m > 1.
int general_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                       double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_euler, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f}, {g}, {y1}, GEulerOp<T>{(T)dt}, fmt);
  });
}

int general_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* fp,
                      const void* g, const void* gp, double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f, fp}, {g, gp}, {y1}, GHeunOp<T>{(T)dt}, fmt);
  });
}

int general_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                             const void* g, double half_dt, void* yp) {
  return dispatch_fmt(L, sde_out::midpoint_predict, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f}, {g}, {yp}, GMidpointPredictOp<T>{(T)half_dt}, fmt);
  });
}

int general_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* g, void* yp) {
  return dispatch_fmt(L, sde_out::euler_heun_predict, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0}, {g}, {yp}, GEulerHeunPredictOp<T>{}, fmt);
  });
}

int general_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                            const void* g, const void* gp, double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_euler_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f}, {g, gp}, {y1}, GEulerHeunOp<T>{(T)dt}, fmt);
  });
}

// The reversible-Heun pair rejects launch flags: its g operands are saved and differentiated, so always dense.
int general_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                              const void* f0, const void* g0, double dt, void* z1) {
  if (nz && nz->flags) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::reversible_heun_z, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, z0, f0}, {g0}, {z1}, GRevHeunZOp<T>{(T)dt, 0}, fmt);
  });
}

int general_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                 const void* f1, const void* g0, const void* g1, double half_dt, void* y1) {
  if (nz && nz->flags) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::step_reversible_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f0, f1}, {g0, g1}, {y1}, GRevHeunOp<T>{(T)half_dt, 0}, fmt);
  });
}

int general_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                                      const void* f0, const void* g0, const void* adj_y0, const void* adj_f0,
                                      const void* adj_g0, double dt, double half_dt, void* z1, void* adj_f0_out,
                                      void* adj_g0_out) {
  if (nz && nz->flags) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::adjoint_a, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    // z1 = 2*y0 - z0 - f0*dt - g0.dW                                              :109
    if (int e = launch_gen_fmt<T>(L, nz, {y0, z0, f0}, {g0}, {z1}, GRevHeunZOp<T>{(T)dt, 1}, fmt)) return e;
    // adj_f0' = adj_f0 + adj_y0*half_dt                                            :104,113
    tsde_launch r = *L;
    r.noise_type = TSDE_NOISE_DIAGONAL;
    r.m = r.d;
    const void* ins[2] = {adj_y0, adj_f0};
    void* outs[1] = {adj_f0_out};
    if (int e = launch_ew<T>(&r, nullptr, false, ins, outs, AdjAElemOp<T>{(T)half_dt})) return e;
    // adj_g0' = adj_g0 + adj_y0 (x) half_dW                                        :105,115
    return launch_outer<T>(L, nz, adj_g0, adj_y0, 0.5, nullptr, 0.0, adj_g0_out);
  });
}

int general_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                      const void* f1, const void* g0, const void* g1, const void* adj_y0,
                                      const void* adj_z0, const void* vjp_z, double dt, double half_dt, void* y1,
                                      void* adj_y1, void* adj_z1, void* adj_f1, void* adj_g1) {
  if (nz && nz->flags) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::adjoint_b, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    // y1 = y0 - (f0+f1)*half_dt - (g0+g1).half_dW                                   :134-135
    if (int e = launch_gen_fmt<T>(L, nz, {y0, f0, f1}, {g0, g1}, {y1}, GRevHeunOp<T>{(T)half_dt, 1}, fmt)) return e;
    // element-wise part: adj_y1, adj_z1 = -(adj_z0 + vjp_z), adj_f1
    tsde_launch r = *L;
    r.noise_type = TSDE_NOISE_DIAGONAL;
    r.m = r.d;
    const void* ins[3] = {adj_y0, adj_z0, vjp_z};
    void* outs[3] = {adj_y1, adj_z1, adj_f1};
    if (int e = launch_ew<T>(&r, nullptr, false, ins, outs, AdjBElemOp<T>{(T)dt, (T)half_dt})) return e;
    // adj_g1 = adj_y0 (x) half_dW + adj_z0' (x) dW = adj_y0 (x) (0.5 dW) + adj_z1 (x) (-1 dW)   :114,140
    return launch_outer<T>(L, nz, nullptr, adj_y0, 0.5, adj_z1, -1.0, adj_g1);
  });
}

}  // namespace tsde

using namespace tsde;

// Exported entry points that exist for additive noise only.
TSDE_EXPORT int tsde_srk_additive_stage(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                        const void* ga, double dt, double rdt, void* h0_1) {
  if (!L || L->noise_type != TSDE_NOISE_GENERAL) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::srk_additive_stage, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f0}, {ga}, {h0_1}, GSraStageOp<T>{(T)dt, (T)rdt}, fmt);
  });
}

TSDE_EXPORT int tsde_step_srk_additive(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                       const void* f1, const void* ga, const void* gb, double dt, double rdt,
                                       void* y1) {
  if (!L || L->noise_type != TSDE_NOISE_GENERAL) return TSDE_EINVAL;
  return dispatch_fmt(L, sde_out::step_srk_additive, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return launch_gen_fmt<T>(L, nz, {y0, f0, f1}, {ga, gb}, {y1},
                             GSraFinalOp<T>{(T)dt, (T)rdt, (T)(1.0 / 3), (T)(2.0 / 3)}, fmt);
  });
}

TSDE_EXPORT int64_t tsde_kernel_launches(int32_t family) {
  if (family < 0 || family >= kKernelFamilies) return -1;
  return g_launches[family].load(std::memory_order_relaxed);
}
