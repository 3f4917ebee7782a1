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

// ---- logqp: KL-integrand augmentation, general / additive / scalar noise ---------------------------------------
// torchsde/_core/base_sde.py:285-306 (SDELogqp.f_and_g_general):
//     u = pinverse(g) (f - h);   f_aug = [f, 0.5 |u|^2];   g_aug = [g ; 0]      g:(d, m) per row, rcond = 1e-15
// The reference runs a batched SVD (cuSOLVER, with a host synchronisation) on every drift evaluation.  Here one
// group of warps per row runs a one-sided (Hestenes) Jacobi SVD on the row's matrix in shared memory; neither U nor V
// is stored, only what |u|^2 needs:
//   * tall, d >= m: the m columns of g (length d) are orthogonalised, G V = U S.  With c_i = (G V)_i . r and
//     s_i^2 = |(G V)_i|^2:  |u|^2 = sum_i c_i^2 / s_i^4  (V is orthogonal, so it drops out of the norm);
//   * wide, d < m: the d columns of g^T (the rows of g, length m) are orthogonalised, g^T V = U S, and every rotation
//     of the pair (i, j) is applied to (r_i, r_j) too, so r ends as V^T r:  |u|^2 = sum_i r'_i^2 / s_i^2.
// Singular values are kept as pinverse keeps them: s_i > rcond * s_max.  A structurally zero column (or row) of g
// stays exactly zero under the rotations and contributes nothing.
// Pairs are visited in round-robin (tournament) order: n/2 disjoint pairs per round, one warp per pair, dot products
// reduced with shuffles and the rotation applied in place.  A sweep in which no pair of any row of the CTA rotated
// ends the loop (a CTA-wide vote), at most kLqMaxSweeps sweeps: extra sweeps of a converged row rotate nothing, so
// its result does not depend on which rows share its CTA.  A pair is rotated only if |a_i.a_j| > tol |a_i| |a_j|,
// so NaN / Inf never rotate; a row with a non-finite g or f - h gets a NaN rate, as the torch path's SVD gives.
namespace tsde {

constexpr int kLqMaxSweeps = 30;
constexpr int kLqWarps = 8;  // warps per CTA

// Per-row shared-memory layout (elements of T): A[n*k] | r[d] | s2[n] | c[n], padded to an even count.
__host__ __device__ inline int lq_stride(int d, int m) {
  const int n = d < m ? d : m, k = d < m ? m : d;
  return (n * k + d + 2 * n + 1) & ~1;
}

template <typename T>
__global__ void __launch_bounds__(kLqWarps * 32)
logqp_augment_general_kernel(int64_t rows, int d, int m, const T* __restrict__ f, const T* __restrict__ g,
                             const T* __restrict__ h, T rcond, T* __restrict__ f_aug, T* __restrict__ g_aug,
                             int rows_per_cta, int warps_per_row) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const bool tall = d >= m;
  const int n = tall ? m : d, k = tall ? d : m;
  const int n2 = n + (n & 1);                         // even number of players (one idle for odd n)
  const int stride = lq_stride(d, m);
  const int group_threads = warps_per_row * 32;
  const int grp = threadIdx.x / group_threads, t = threadIdx.x - grp * group_threads;
  const int w = t >> 5, lane = t & 31;
  T* A = reinterpret_cast<T*>(smem_raw) + (size_t)grp * stride;
  T* r = A + n * k;
  T* s2 = r + d;
  T* cc = s2 + n;
  int* bad = reinterpret_cast<int*>(reinterpret_cast<T*>(smem_raw) + (size_t)rows_per_cta * stride);
  const int64_t row = (int64_t)blockIdx.x * rows_per_cta + grp;
  const bool active = row < rows;
  constexpr T u = sizeof(T) == 4 ? T(5.9604644775390625e-8) : T(1.1102230246251565e-16);
  // below the rounding error of the dot products themselves: a (k/32)-term chain per lane, then 5 shuffle levels
  const T tol = T((k + 31) / 32 + 5) * u;

  if (t == 0) bad[grp] = 0;
  __syncthreads();
  if (active) {
    const int64_t dm = (int64_t)d * m;
    const T* gr = g + row * dm;
    T* go = g_aug + row * (dm + m);
    bool nf = false;
    for (int e = t; e < d * m; e += group_threads) {
      const T v = gr[e];
      go[e] = v;
      nf |= !isfinite(v);
      if (tall) {
        const int i = e / m, j = e - i * m;
        A[j * k + i] = v;                                // column j of g
      } else {
        A[e] = v;                                        // row i of g = column i of g^T
      }
    }
    for (int e = t; e < m; e += group_threads) go[dm + e] = T(0);
    const T* fr = f + row * d;
    const T* hr = h + row * d;
    T* fo = f_aug + row * (d + 1);
    for (int e = t; e < d; e += group_threads) {
      const T fv = fr[e];
      fo[e] = fv;
      const T rv = fv - hr[e];
      r[e] = rv;
      nf |= !isfinite(rv);
    }
    if (__any_sync(0xffffffffu, nf) && lane == 0) atomicOr(&bad[grp], 1);
  }
  __syncthreads();
  const bool live = active && !bad[grp];

  for (int sweep = 0; sweep < kLqMaxSweeps; ++sweep) {
    int rotated = 0;
    for (int round = 0; round < n2 - 1; ++round) {
      for (int p = w; p < n2 / 2; p += warps_per_row) {
        // circle method: slot 0 holds player 0, slots 1..n2-1 hold the others shifted by `round`; pair p is the
        // players of slots p and n2-1-p
        const int a = p == 0 ? 0 : (p - 1 + round) % (n2 - 1) + 1;
        const int b = (n2 - 2 - p + round) % (n2 - 1) + 1;
        if (!live || a >= n || b >= n) continue;
        T* x = A + a * k;
        T* y = A + b * k;
        T app = T(0), aqq = T(0), apq = T(0);
        for (int i = lane; i < k; i += 32) {
          const T xv = x[i], yv = y[i];
          app = fma(xv, xv, app);
          aqq = fma(yv, yv, aqq);
          apq = fma(xv, yv, apq);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          app += __shfl_xor_sync(0xffffffffu, app, off);
          aqq += __shfl_xor_sync(0xffffffffu, aqq, off);
          apq += __shfl_xor_sync(0xffffffffu, apq, off);
        }
        // (false for NaN / Inf: such a pair is never rotated)
        if (!(fabs(apq) > tol * sqrt(app) * sqrt(aqq))) continue;
        const T zeta = (aqq - app) / (T(2) * apq);
        const T az = fabs(zeta);
        const T root = az < T(1e8) ? sqrt(T(1) + zeta * zeta) : az;
        const T tn = (zeta < T(0) ? T(-1) : T(1)) / (az + root);
        const T cs = T(1) / sqrt(T(1) + tn * tn), sn = cs * tn;
        for (int i = lane; i < k; i += 32) {
          const T xv = x[i], yv = y[i];
          x[i] = cs * xv - sn * yv;
          y[i] = sn * xv + cs * yv;
        }
        if (!tall && lane == 0) {
          const T ra = r[a], rb = r[b];
          r[a] = cs * ra - sn * rb;
          r[b] = sn * ra + cs * rb;
        }
        rotated = 1;
      }
      __syncthreads();
    }
    if (!__syncthreads_or(rotated)) break;
  }

  if (active) {
    for (int j = w; j < n; j += warps_per_row) {
      const T* x = A + j * k;
      T ss = T(0), c = T(0);
      for (int i = lane; i < k; i += 32) {
        ss = fma(x[i], x[i], ss);
        if (tall) c = fma(x[i], r[i], c);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, off);
        c += __shfl_xor_sync(0xffffffffu, c, off);
      }
      if (lane == 0) {
        s2[j] = ss;
        cc[j] = tall ? c : r[j];
      }
    }
  }
  __syncthreads();
  if (active && w == 0) {
    const T qnan = sizeof(T) == 4 ? T(__int_as_float(0x7fc00000)) : T(__longlong_as_double(0x7ff8000000000000ll));
    T smax = T(0);
    for (int j = lane; j < n; j += 32) smax = fmax(smax, sqrt(s2[j]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) smax = fmax(smax, __shfl_xor_sync(0xffffffffu, smax, off));
    const T cut = rcond * smax;
    T acc = T(0);
    for (int j = lane; j < n; j += 32) {
      const T s = sqrt(s2[j]);
      if (s > cut) {
        const T q = tall ? (cc[j] / s) / s : cc[j] / s;
        acc = fma(q, q, acc);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) f_aug[row * (d + 1) + d] = bad[grp] ? qnan : T(0.5) * acc;
  }
}

// One row's tall-orientation matrix (min(d,m) x max(d,m)) plus r = f - h within TSDE_LOGQP_GENERAL_MAX elements.
// (d, m <= the bound first: then neither the product nor d + 1 can overflow.)
inline bool logqp_general_fits(int64_t d, int64_t m) {
  if (d > TSDE_LOGQP_GENERAL_MAX || m > TSDE_LOGQP_GENERAL_MAX) return false;
  return (d < m ? d : m) * (d < m ? m : d) + d <= TSDE_LOGQP_GENERAL_MAX;
}

template <typename T>
static int logqp_augment_general_impl(const tsde_launch* L, const void* f, const void* g, const void* h,
                                      double rcond, void* f_aug, void* g_aug) {
  if (!f || !g || !h || !f_aug || !g_aug) return TSDE_EINVAL;
  const int64_t rows = L->rows, d = L->d, m = L->m;
  if (!logqp_general_fits(d, m)) return TSDE_EINVAL;
  if (rows > INT64_MAX / ((d + 1) * m)) return TSDE_EINVAL;   // element offsets of g_aug
  const int n = (int)(d < m ? d : m);
  const int pairs = (n + 1) / 2;
  const int wpr = pairs < kLqWarps ? pairs : kLqWarps;
  const size_t row_bytes = (size_t)lq_stride((int)d, (int)m) * sizeof(T);
  // small rows share a CTA (up to kLqWarps warps, at most 48 KiB of shared memory); a large row has one to itself
  int rpc = kLqWarps / wpr;
  while (rpc > 1 && rpc * row_bytes > 48 * 1024) --rpc;
  const int64_t blocks = (rows + rpc - 1) / rpc;
  if (blocks > 0x7fffffffll) return TSDE_EINVAL;
  const size_t smem = rpc * row_bytes + rpc * sizeof(int);
  const int threads = rpc * wpr * 32;
  auto kernel = logqp_augment_general_kernel<T>;
  if (resident_ctas(reinterpret_cast<const void*>(kernel), threads, smem) == 0) return (int)cudaErrorInvalidConfiguration;
  return launch_kernel(kernel, blocks, threads, smem, reinterpret_cast<cudaStream_t>(L->stream), false, rows, (int)d,
                       (int)m, (const T*)f, (const T*)g, (const T*)h, (T)rcond, (T*)f_aug, (T*)g_aug, rpc, wpr);
}

}  // namespace tsde

TSDE_EXPORT int tsde_logqp_augment(const tsde_launch* L, const void* f, const void* g, const void* h, double eps,
                                   void* f_aug, void* g_aug) {
  return tsde::dispatch(L, [&](auto t) {
    if (L->noise_type == TSDE_NOISE_GENERAL)
      return tsde::logqp_augment_general_impl<decltype(t)>(L, f, g, h, eps, f_aug, g_aug);
    return tsde::logqp_augment_impl<decltype(t)>(L, f, g, h, eps, f_aug, g_aug);
  });
}
