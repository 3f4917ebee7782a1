// Log-ODE / Levy-area method support: the batched product  GA = g A  of torchsde/_core/base_sde.py:170,191
// (`ga = torch.bmm(g, a)` inside dg_ga_jvp_column_sum_v1/_v2), g:(rows,d,m), A:(rows,m,m) -> (rows,d,m).
//
// 2 d m^2 flops over (2 d m + m^2) s bytes per row — 3 flop/byte at (d, m) = (32, 16), far below the fp32 ridge
// of the machine (~10 flop/byte): an HBM-bound stream, so plain fp32 FFMA (no tensor cores: they would buy
// nothing and TF32 would cost accuracy the method's jvp tangents need).  Layout of the work:
//   * a warp-sized group of threads owns one row; thread <-> state channel dd: it keeps its g row (m values,
//     read once with 128-bit loads; a warp reads one contiguous run of 32 m s bytes) in registers,
//   * the row's A (m x m) is staged once in shared memory with coalesced loads and read back as broadcasts
//     (every thread of the row needs the same A[k][l]),
//   * the result is stored TRANSPOSED, out[l][row][dd]: the consumer takes one column l at a time as the tangent
//     of a jvp through the user's g (base_sde.py:173-184), and a contiguous (rows, d) slab per column is exactly
//     what it wants; for fixed l a warp writes 32 consecutive floats (coalesced).
// Summation over k ascending with FMA; agrees with torch.bmm to rounding (its order is unspecified).
#include "ew.cuh"

namespace tsde {

constexpr int kBmmThreads = 256;

template <typename T, int M>
__global__ void __launch_bounds__(kBmmThreads, (M <= 16 && sizeof(T) == 4) ? 4 : 1)
bmm_ga_kernel(int64_t rows, int d, const T* __restrict__ g, const T* __restrict__ a, T* __restrict__ out,
              int rows_per_cta) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sA = reinterpret_cast<T*>(smem_raw);                       // [rows_per_cta][M*M]
  const int64_t row0 = (int64_t)blockIdx.x * rows_per_cta;
  const int nrows = (int)((rows - row0) < rows_per_cta ? (rows - row0) : rows_per_cta);
  // the thread's first g row goes into registers BEFORE the A tiles are staged: both global-memory latencies of the
  // CTA (g, then A -> shared -> barrier) overlap instead of following each other
  T gk[M];
  auto load_g = [&](int idx) {
    const T* gp = g + (row0 * d + idx) * M;                       // (row0 + r) * d + dd = row0 * d + idx
    if (M % 4 == 0) {
#pragma unroll
      for (int k = 0; k < M; k += 4) {
        T v[4];
        ld4(gp + k, v);
        gk[k] = v[0]; gk[k + 1] = v[1]; gk[k + 2] = v[2]; gk[k + 3] = v[3];
      }
    } else {
#pragma unroll
      for (int k = 0; k < M; ++k) gk[k] = gp[k];
    }
  };
  if ((int)threadIdx.x < nrows * d) load_g(threadIdx.x);
  // stage the group's A matrices (contiguous in global memory)
  {
    const int64_t base = row0 * (M * M);
    const int total = nrows * M * M;
    if (M % 4 == 0) {
#pragma unroll 2
      for (int e = 4 * threadIdx.x; e < total; e += 4 * kBmmThreads) {
        T v[4];
        ld4(a + base + e, v);
        st4(sA + e, v);
      }
    } else {
      for (int e = threadIdx.x; e < total; e += kBmmThreads) sA[e] = a[base + e];
    }
  }
  __syncthreads();
  const int64_t plane = rows * (int64_t)d;                        // elements per output column
  for (int idx = threadIdx.x; idx < nrows * d; idx += kBmmThreads) {
    const int r = idx / d, dd = idx - r * d;
    const int64_t row = row0 + r;
    if (idx != (int)threadIdx.x) load_g(idx);
    const T* A = sA + r * (M * M);
    // all M results of the thread accumulate at once, k ascending for each (the order of the one-result-at-a-time
    // loop): A[k][.] then comes out of shared memory as 128-bit broadcasts, M*M/4 loads instead of M*M
    T acc[M];
#pragma unroll
    for (int l = 0; l < M; ++l) acc[l] = T(0);
#pragma unroll
    for (int k = 0; k < M; ++k) {
      if (M % 4 == 0) {
#pragma unroll
        for (int l = 0; l < M; l += 4) {
          T a4[4];
          ld4(A + k * M + l, a4);
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[l + j] = fma(gk[k], a4[j], acc[l + j]);
        }
      } else {
#pragma unroll
        for (int l = 0; l < M; ++l) acc[l] = fma(gk[k], A[k * M + l], acc[l]);
      }
    }
#pragma unroll
    for (int l = 0; l < M; ++l) out[(int64_t)l * plane + row * d + dd] = acc[l];
  }
}

// any m: one thread per output element (row, dd, l), A and g read through the caches
template <typename T>
__global__ void __launch_bounds__(kThreads)
bmm_ga_generic_kernel(int64_t rows, int64_t d, int64_t m, const T* __restrict__ g, const T* __restrict__ a,
                      T* __restrict__ out) {
  const int64_t total = rows * d * m, plane = rows * d;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += stride) {
    const int64_t l = e / plane;
    const int64_t rd = e - l * plane;
    const int64_t row = rd / d;
    const T* gp = g + rd * m;
    const T* ap = a + row * m * m + l;
    T acc = T(0);
    for (int64_t k = 0; k < m; ++k) acc = fma(gp[k], ap[k * m], acc);
    out[e] = acc;
  }
}

template <typename T>
static int bmm_ga_impl(const tsde_launch* L, const void* g, const void* a, void* out) {
  if (!g || !a || !out) return TSDE_EINVAL;
  if (L->noise_type != TSDE_NOISE_GENERAL) return TSDE_EINVAL;
  const int64_t rows = L->rows, d = L->d, m = L->m;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  const bool al = aligned16(g) && aligned16(a);
  auto tiled = [&](auto kernel, int M) -> int {
    // rows per CTA: ~256 (row, dd) work items, A tiles within 32 KiB of shared memory
    int64_t rpc = (kBmmThreads + d - 1) / d;
    if (rpc < 1) rpc = 1;
    const int64_t fit = (32 * 1024) / ((int64_t)M * M * (int64_t)sizeof(T));
    if (rpc > fit) rpc = fit;
    if (rpc < 1) return TSDE_EINVAL;
    const int64_t blocks = (rows + rpc - 1) / rpc;
    if (blocks > 0x7fffffffll) return TSDE_EINVAL;
    return launch_kernel(kernel, blocks, kBmmThreads, (size_t)rpc * M * M * sizeof(T), st, false, rows, (int)d,
                         (const T*)g, (const T*)a, (T*)out, (int)rpc);
  };
  if (d <= (1 << 20) && (al || m % 4 != 0)) {
    switch (m) {
      case 2: return tiled(bmm_ga_kernel<T, 2>, 2);
      case 3: return tiled(bmm_ga_kernel<T, 3>, 3);
      case 4: return tiled(bmm_ga_kernel<T, 4>, 4);
      case 8: return tiled(bmm_ga_kernel<T, 8>, 8);
      case 16: return tiled(bmm_ga_kernel<T, 16>, 16);
      case 32: return tiled(bmm_ga_kernel<T, 32>, 32);
      default: break;
    }
  }
  return launch_kernel(bmm_ga_generic_kernel<T>, capped_grid(rows * d * m, kThreads, 16), kThreads, 0, st, false,
                       rows, d, m, (const T*)g, (const T*)a, (T*)out);
}

}  // namespace tsde

using namespace tsde;

TSDE_EXPORT int tsde_bmm_ga(const tsde_launch* L, const void* g, const void* a, void* out_t) {
  return dispatch(L, [&](auto t) { return bmm_ga_impl<decltype(t)>(L, g, a, out_t); });
}

// ---- logqp: KL-integrand augmentation, diagonal noise ---------------------------------------------------------
// torchsde/_core/base_sde.py:266-283 (SDELogqp.f_and_g_diagonal) + misc.py:66-68 (stable_division):
//     u = (f - h) / where(|g| > eps, g, eps * sign(g));   f_aug = [f, 0.5 * sum_d u^2];   g_aug = [g, 0]
// The reference does this with ~10 ATen launches (sub, abs, where, full_like, sign, mul, div, pow, sum, 2 x cat);
// here one warp per row streams f, g, h once, reduces u^2 with shuffles and writes both augmented rows.
namespace tsde {

template <typename T>
__global__ void __launch_bounds__(kThreads)
logqp_augment_kernel(int64_t rows, int d, const T* __restrict__ f, const T* __restrict__ g, const T* __restrict__ h,
                     T eps, T* __restrict__ f_aug, T* __restrict__ g_aug) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * kThreads) >> 5;
  for (int64_t row = (((int64_t)blockIdx.x * kThreads) + threadIdx.x) >> 5; row < rows; row += warps) {
    const T* fr = f + row * d;
    const T* gr = g + row * d;
    const T* hr = h + row * d;
    T* fo = f_aug + row * (d + 1);
    T* go = g_aug + row * (d + 1);
    T acc = T(0);
    for (int c = lane; c < d; c += 32) {
      const T fv = fr[c], gv = gr[c];
      const T ag = gv < T(0) ? -gv : gv;
      const T sgn = gv > T(0) ? T(1) : (gv < T(0) ? T(-1) : T(0));
      const T safe = ag > eps ? gv : eps * sgn;
      const T u = (fv - hr[c]) / safe;
      acc = acc + u * u;
      fo[c] = fv;
      go[c] = gv;
    }
    for (int off = 16; off > 0; off >>= 1) acc = acc + __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) {
      fo[d] = T(0.5) * acc;
      go[d] = T(0);
    }
  }
}

template <typename T>
static int logqp_augment_impl(const tsde_launch* L, const void* f, const void* g, const void* h, double eps,
                              void* f_aug, void* g_aug) {
  if (!f || !g || !h || !f_aug || !g_aug) return TSDE_EINVAL;
  if (L->noise_type != TSDE_NOISE_DIAGONAL || L->d > (1 << 24)) return TSDE_EINVAL;
  // one warp per row
  return launch_kernel(logqp_augment_kernel<T>, capped_grid(L->rows * 32, kThreads, kBlocksPerSM), kThreads, 0,
                       reinterpret_cast<cudaStream_t>(L->stream), false, L->rows, (int)L->d, (const T*)f,
                       (const T*)g, (const T*)h, (T)eps, (T*)f_aug, (T*)g_aug);
}

}  // namespace tsde

TSDE_EXPORT int tsde_logqp_augment(const tsde_launch* L, const void* f, const void* g, const void* h, double eps,
                                   void* f_aug, void* g_aug) {
  return tsde::dispatch(L, [&](auto t) {
    return tsde::logqp_augment_impl<decltype(t)>(L, f, g, h, eps, f_aug, g_aug);
  });
}
