// Brownian source kernels: materialise increments of whole cells, Brownian-bridge descent,
// interval merges, Davie/Foster Levy area.  Replaces the tensor arithmetic of
// torchsde/_brownian/brownian_interval.py (the interval *tree* stays on the host,
// torchsde_b200/_brownian/interval.py).
#include "ew.cuh"

namespace tsde {

// ---- cells -> (W, U, H) ---------------------------------------------------------------------
// Variant that also exposes H itself (the bridge descent consumes it).
template <typename T>
__device__ __forceinline__ void counter_wh(const NoiseP<T>& nz, Key key, uint32_t row, uint32_t q,
                                           T (&w)[4], T (&hh)[4]) {
  double len0 = nz.cell_h ? nz.cell_h[0] : nz.h;
  T n[4];
  normal4(key, nz.cell_id, STREAM_W, row, q, n);
  const T s = (T)sqrt(len0);
#pragma unroll
  for (int j = 0; j < 4; ++j) w[j] = n[j] * s;
  normal4(key, nz.cell_id, STREAM_H, row, q, n);
  const T s12 = (T)sqrt(len0 / 12.0);
#pragma unroll
  for (int j = 0; j < 4; ++j) hh[j] = n[j] * s12;
  double elapsed = len0;
  for (int c = 1; c < nz.n_cells; ++c) {
    const double len = nz.cell_h ? nz.cell_h[c] : nz.h;
    T wi[4];
    normal4(key, nz.cell_id + (uint64_t)c, STREAM_W, row, q, n);
    const T si = (T)sqrt(len);
#pragma unroll
    for (int j = 0; j < 4; ++j) wi[j] = n[j] * si;
    normal4(key, nz.cell_id + (uint64_t)c, STREAM_H, row, q, n);
    const T s12i = (T)sqrt(len / 12.0);
    const T tl = (T)len, te = (T)elapsed, tt = (T)(elapsed + len);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const T hi = n[j] * s12i;
      const T term1 = tl * (hi + T(0.5) * w[j]);
      const T term2 = te * (hh[j] - T(0.5) * wi[j]);
      hh[j] = (term1 + term2) / tt;
      w[j] = w[j] + wi[j];
    }
    elapsed += len;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
cells_wh_kernel(NoiseP<T> nz, int64_t rows, int64_t m, int64_t qpr, int vec, T* out_w, T* out_u,
                T* out_h) {
  const Key key = load_key(nz.key);
  const int64_t nquads = rows * qpr;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const T ht = (T)nz.h_total;
  for (int64_t Q = (int64_t)blockIdx.x * kThreads + threadIdx.x; Q < nquads; Q += stride) {
    const int64_t row = Q / qpr, q = Q - row * qpr;
    const int64_t base = row * m + 4 * q;
    const int64_t rem = m - 4 * q;
    const int nvalid = rem < 4 ? (int)rem : 4;
    T w[4], hh[4];
    counter_wh<T>(nz, key, (uint32_t)(row + nz.row_offset), (uint32_t)q, w, hh);
    store_quad(out_w, base, vec != 0, nvalid, w);
    if (out_h) store_quad(out_h, base, vec != 0, nvalid, hh);
    if (out_u) {
      T u[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) u[j] = ht * (T(0.5) * w[j] + hh[j]);
      store_quad(out_u, base, vec != 0, nvalid, u);
    }
  }
}

// W (and U) of a run of cells through the row-wise framework (specialised kernel + PDL when it applies)
template <typename T, bool WANT>
struct CellsOp {
  static constexpr int NIN = 0, NOUT = WANT ? 2 : 1;
  static constexpr bool USES_NOISE = true, WANT_U = WANT;
  __device__ __forceinline__ void operator()(const T (&)[1], T w, T u, T (&out)[NOUT]) const {
    out[0] = w;
    if (WANT) out[NOUT - 1] = u;
  }
};

// The Brownian tensors are (rows, m); reuse the row-wise framework with d := m.
static tsde_launch as_rows_m(const tsde_launch* L) {
  tsde_launch r = *L;
  r.d = L->m;
  r.noise_type = TSDE_NOISE_DIAGONAL;
  return r;
}

template <typename T>
static int cells_impl(const tsde_launch* L, const tsde_noise* nz, void* out_w, void* out_u,
                      void* out_h) {
  if (!nz || nz->source != TSDE_SRC_COUNTER || !out_w) return TSDE_EINVAL;
  if (!out_h) {
    const tsde_launch r = as_rows_m(L);
    tsde_noise z = *nz;
    if (out_u) {
      z.want_u = 1;
      void* outs[2] = {out_w, out_u};
      return launch_ew<T>(&r, &z, false, nullptr, outs, CellsOp<T, true>{});
    }
    void* outs[1] = {out_w};
    return launch_ew<T>(&r, &z, false, nullptr, outs, CellsOp<T, false>{});
  }
  NoiseP<T> np;
  if (int e = fill_noise<T>(L, nz, false, np)) return e;
  const int64_t m = L->m, rows = L->rows, qpr = (m + 3) / 4, nquads = rows * qpr;
  const bool vec = (m % 4 == 0) && aligned16(out_w) && (!out_u || aligned16(out_u)) && aligned16(out_h);
  return launch_kernel(cells_wh_kernel<T>, capped_grid(nquads, kThreads, kBlocksPerSM), kThreads, 0,
                       reinterpret_cast<cudaStream_t>(L->stream), false, np, rows, m, qpr, vec, (T*)out_w,
                       (T*)out_u, (T*)out_h);
}

// ---- Brownian bridge descent ------------------------------------------------------------------
constexpr int kMaxBridgeDepth = 24;
struct BridgeLevel {
  uint64_t id;
  double k[6];
};
struct BridgeP {
  BridgeLevel lv[kMaxBridgeDepth];
  int32_t depth;
  int32_t have_h;
};

template <typename T, bool HAVE_H>
__global__ void __launch_bounds__(kThreads)
bridge_kernel(const __grid_constant__ BridgeP bp, const void* keyp, int64_t row_offset, int64_t rows,
              int64_t m, int64_t qpr, int vec, const T* in_w, const T* in_h, T* out_w, T* out_h) {
  const Key key = load_key(keyp);
  const int64_t nquads = rows * qpr;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t Q = (int64_t)blockIdx.x * kThreads + threadIdx.x; Q < nquads; Q += stride) {
    const int64_t row = Q / qpr, q = Q - row * qpr;
    const int64_t base = row * m + 4 * q;
    const int64_t rem = m - 4 * q;
    const int nvalid = rem < 4 ? (int)rem : 4;
    const uint32_t grow = (uint32_t)(row + row_offset);
    T w[4], hh[4];
    load_quad(in_w, base, vec != 0, nvalid, w);
    if (HAVE_H) load_quad(in_h, base, vec != 0, nvalid, hh);
    for (int l = 0; l < bp.depth; ++l) {
      const BridgeLevel& lv = bp.lv[l];
      T x1[4];
      normal4(key, lv.id, STREAM_X1, grow, (uint32_t)q, x1);
      if (HAVE_H) {
        // brownian_interval.py:199-225
        T x2[4];
        normal4(key, lv.id, STREAM_X2, grow, (uint32_t)q, x2);
        const T k1 = (T)lv.k[0], k2 = (T)lv.k[1], k3 = (T)lv.k[2], k4 = (T)lv.k[3],
                k5 = (T)lv.k[4], k6 = (T)lv.k[5];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const T ow = (k1 * w[j] + k2 * hh[j]) + k3 * x1[j];
          const T oh = (k4 * hh[j] + k5 * x1[j]) + k6 * x2[j];
          w[j] = ow;
          hh[j] = oh;
        }
      } else {
        // brownian_interval.py:226-237 ; k0 = left_diff, k1 = h_reciprocal, k2 = sqrt(var),
        // k3 = 1 for the left child, 0 for the right child
        const T ld = (T)lv.k[0], hr = (T)lv.k[1], sd = (T)lv.k[2];
        const bool left = lv.k[3] != 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const T left_w = (ld * w[j]) * hr + sd * x1[j];
          w[j] = left ? left_w : (w[j] - left_w);
        }
      }
    }
    store_quad(out_w, base, vec != 0, nvalid, w);
    if (HAVE_H) store_quad(out_h, base, vec != 0, nvalid, hh);
  }
}

template <typename T>
static int bridge_impl(const tsde_launch* L, const void* key, int64_t row_offset, int32_t depth,
                       const uint64_t* ids, const int32_t* is_left, const double* times,
                       const void* in_w, const void* in_h, void* out_w, void* out_h) {
  if (!key || !in_w || !out_w || depth < 0 || (depth > 0 && (!ids || !is_left || !times)))
    return TSDE_EINVAL;
  const bool have_h = in_h != nullptr;
  if (have_h && !out_h) return TSDE_EINVAL;
  const int64_t m = L->m, rows = L->rows, qpr = (m + 3) / 4, nquads = rows * qpr;
  if (rows + row_offset > kMaxGlobalRows || m > kMaxCounterChannels) return TSDE_EINVAL;
  const bool vec = (m % 4 == 0) && aligned16(in_w) && aligned16(out_w) &&
                   (!have_h || (aligned16(in_h) && aligned16(out_h)));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  const auto kernel = have_h ? bridge_kernel<T, true> : bridge_kernel<T, false>;
  const void* cur_w = in_w;
  const void* cur_h = in_h;
  int done = 0;
  do {
    BridgeP bp{};
    const int n = depth - done < kMaxBridgeDepth ? depth - done : kMaxBridgeDepth;
    bp.depth = n;
    bp.have_h = have_h;
    for (int l = 0; l < n; ++l) {
      const int i = done + l;
      const double start = times[3 * i], mid = times[3 * i + 1], end = times[3 * i + 2];
      const double h_rec = 1.0 / (end - start);
      const double ld = mid - start, rd = end - mid;
      BridgeLevel& lv = bp.lv[l];
      lv.id = ids[i];
      if (have_h) {
        const double ld2 = ld * ld, rd2 = rd * rd;
        const double ld3 = ld * ld2, rd3 = rd * rd2;
        const double v = 0.5 * sqrt(ld * rd / (ld3 + rd3));
        const double a = v * ld2 * h_rec;
        const double b = v * rd2 * h_rec;
        const double c = v * 0.57735026918962584;  // 1/sqrt(3)
        const double third = 2 * (a * ld + b * rd) * h_rec;
        if (is_left[i]) {
          const double first = ld * h_rec;
          const double second = 6 * first * rd * h_rec;
          lv.k[0] = first; lv.k[1] = second; lv.k[2] = third;
          lv.k[3] = first * first; lv.k[4] = -a; lv.k[5] = c * rd;
        } else {
          const double first = rd * h_rec;
          const double second = 6 * first * ld * h_rec;
          lv.k[0] = first; lv.k[1] = -second; lv.k[2] = -third;
          lv.k[3] = first * first; lv.k[4] = -b; lv.k[5] = -(c * ld);
        }
      } else {
        lv.k[0] = ld; lv.k[1] = h_rec; lv.k[2] = sqrt(ld * rd * h_rec);
        lv.k[3] = is_left[i] ? 1.0 : 0.0;
      }
    }
    if (int e = launch_kernel(kernel, capped_grid(nquads, kThreads, kBlocksPerSM), kThreads, 0, st, false, bp, key,
                              row_offset, rows, m, qpr, vec, (const T*)cur_w, (const T*)cur_h, (T*)out_w,
                              (T*)out_h))
      return e;
    done += n;
    cur_w = out_w;  // further chunks continue in place
    cur_h = out_h;
  } while (done < depth);
  return 0;
}

// ---- merges ------------------------------------------------------------------------------------
// brownian_interval.py:649-672
template <typename T>
struct MergeWHOp {
  static constexpr int NIN = 4, NOUT = 2;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T len1, len0, tot;
  __device__ __forceinline__ void operator()(const T (&in)[4], T, T, T (&out)[2]) const {
    const T w = in[0], h = in[1], wi = in[2], hi = in[3];
    const T term1 = len1 * (hi + T(0.5) * w);
    const T term2 = len0 * (h - T(0.5) * wi);
    out[1] = (term1 + term2) / tot;
    out[0] = w + wi;
  }
};
template <typename T>
struct AddOp {
  static constexpr int NIN = 2, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  __device__ __forceinline__ void operator()(const T (&in)[2], T, T, T (&out)[1]) const {
    out[0] = in[0] + in[1];
  }
};
template <typename T>
struct HToUOp {
  static constexpr int NIN = 2, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T h;
  __device__ __forceinline__ void operator()(const T (&in)[2], T, T, T (&out)[1]) const {
    out[0] = h * (T(0.5) * in[0] + in[1]);
  }
};

// ---- Davie / Foster Levy area                                   brownian_interval.py:78-99
// A = H (x) W - W (x) H + std * (N - N^T).  The reference draws a full (m x m) matrix N of iid normals and
// antisymmetrises it (:88-90); only the antisymmetric part enters, and N_ij - N_ji ~ N(0, 2) independently for
// every pair i < j.  The counter-based source therefore draws ONE normal z per pair (m(m-1)/2 instead of m^2:
// for m = 16, 30 Philox calls per row instead of 64) and defines
//     N_ij = z_ij / sqrt(2),  N_ji = -N_ij  (i < j),  N_ii = 0        =>   N - N^T has the reference's law;
// pair p = (i, j), i < j, in row-major upper-triangular order, is channel p of stream STREAM_A of node `a_id`
// (oracle/brownian.py levy_noise restates this).  The kernel is a write-bound stream of (m x m) tiles:
// one warp per row — lanes draw the row's pair normals (one Philox quad = 4 pairs per lane), form the upper
// triangle, mirror it (A is antisymmetric, exactly: this translation unit is compiled without FMA contraction)
// into a warp-private shared tile, and the warp stores the tile with fully coalesced 128-bit writes.
// Foster's std needs one square root per pair: fp32 takes the SFU's (MUFU.SQRT, ~1 ulp; the IEEE-rounded `sqrtf`
// is a ~10-instruction Newton sequence and the kernel is issue-bound), fp64 the correctly rounded one.  The SFU flushes
// a subnormal operand to zero, and Foster's variance ~0.027 h^2 is subnormal for h below ~2^-60, where the noise term
// is as large as the cross term: such an operand is scaled by 2^64 first and the root by 2^-32 after (both exact).
__device__ __forceinline__ float levy_sqrt(float x) {
  const bool tiny = x < 1.17549435e-38f;   // FLT_MIN
  const float r = mufu_sqrt(tiny ? x * 18446744073709551616.0f : x);
  return tiny ? r * 2.3283064365386963e-10f : r;
}
__device__ __forceinline__ double levy_sqrt(double x) { return sqrt(x); }

template <typename T, bool FOSTER>
__device__ __forceinline__ T levy_pair_value_t(T wi, T wj, T hi, T hj, T z, T tenth_h, T davie_std) {
  const T a = hi * wj - wi * hj;
  // N_ij = z / sqrt(2), N_ji = -N_ij: N_ij - N_ji = 2 N_ij.  One multiplication by 2 fl(1/sqrt 2) gives exactly
  // twice fl(z fl(1/sqrt 2)) (scaling by two commutes with rounding), i.e. the bits of n - (-n).
  const T noise = z * (T(2) * T(0.70710678118654752440));
  const T std_ = FOSTER ? levy_sqrt(tenth_h * ((tenth_h + hi * hi) + hj * hj)) : davie_std;
  return a + std_ * noise;
}
template <typename T>
__device__ __forceinline__ T levy_pair_value(T wi, T wj, T hi, T hj, T z, T tenth_h, T davie_std, int foster) {
  return foster ? levy_pair_value_t<T, true>(wi, wj, hi, hj, z, tenth_h, davie_std)
                : levy_pair_value_t<T, false>(wi, wj, hi, hj, z, tenth_h, davie_std);
}

constexpr int kLevyWarps = 8;
// Register budget of the fp32 compile-time-m instantiations, as the minimum number of resident CTAs per SM they are
// compiled for (65536 / (256 n) registers per thread).  n = 2 leaves the compiler the registers it takes when it may:
// the issue-bound kernel prefers the longer instruction schedule to more resident warps.
constexpr int kLevyCtasF32 = 2;

// Rows a warp handles per pass in the generating mode: the W and H normals of one row are only m/2 Philox quads, so
// one warp-wide pass draws them for 32 / (m/2) rows at once (m = 16: 4 rows) instead of leaving most lanes idle.
__host__ __device__ constexpr int levy_group_rows(int m, bool gen) {
  return (gen && m >= 4 && 64 / m >= 1) ? 64 / m : 1;
}
// floats per warp in shared memory: padded A tile | (W | H) x rows per pass | one scratch word (16-byte multiple)
__host__ __device__ constexpr int levy_tile_elems(int m, bool gen) {
  return (m * (m + 1) + 2 * m * levy_group_rows(m, gen) + 1 + 3) & ~3;
}

// The four pairs of one Philox quad: operands through per-lane shared-memory pointers looked up once per kernel
// (slots past the last pair point at the scratch word, so the pass has no per-pair branch).
// fp32: two pairs side by side (both pairs' operands are loaded before either result is stored), one explicitly
// rounded operation of each per line (never contracted).  The cross term H_i W_j - W_i H_j keeps its three roundings (the subtraction
// is fma(x, -1, y): the product by -1 is exact).  The sum of squares under the root and the final std * noise + cross
// term are fused multiply-adds, written out as such, so the source says what runs.  The result differs from the
// scalar pass (fp64, m > 16) by at most an ulp of the noise term; the area's noise is a fresh draw per query and
// pinned to the oracle by tolerance, A = -A^T stays exact.
template <bool FOSTER>
__device__ __forceinline__ void levy_quad_pairs_f32(const float* const (&pw_i)[4], const float* const (&pw_j)[4],
                                                    int off, int m, float* const (&pa)[4], float* const (&pb)[4],
                                                    const float (&z)[4], float tenth_h, float davie_std) {
  const float c2 = 2.0f * 0.70710678118654752440f;
#pragma unroll
  for (int k = 0; k < 4; k += 2) {
    const float wi0 = pw_i[k][off], wi1 = pw_i[k + 1][off];
    const float wj0 = pw_j[k][off], wj1 = pw_j[k + 1][off];
    const float hi0 = pw_i[k][off + m], hi1 = pw_i[k + 1][off + m];
    const float hj0 = pw_j[k][off + m], hj1 = pw_j[k + 1][off + m];
    // a = hi wj - wi hj
    const float x0 = __fmul_rn(wi0, hj0), x1 = __fmul_rn(wi1, hj1);
    const float y0 = __fmul_rn(hi0, wj0), y1 = __fmul_rn(hi1, wj1);
    const float a0 = __fmaf_rn(x0, -1.0f, y0), a1 = __fmaf_rn(x1, -1.0f, y1);
    const float n0 = __fmul_rn(z[k], c2), n1 = __fmul_rn(z[k + 1], c2);
    float sd0 = davie_std, sd1 = davie_std;
    if (FOSTER) {
      const float e0 = __fmaf_rn(hi0, hi0, tenth_h), e1 = __fmaf_rn(hi1, hi1, tenth_h);
      const float f0 = __fmaf_rn(hj0, hj0, e0), f1 = __fmaf_rn(hj1, hj1, e1);
      const float s0 = __fmul_rn(tenth_h, f0), s1 = __fmul_rn(tenth_h, f1);
      sd0 = levy_sqrt(s0);
      sd1 = levy_sqrt(s1);
    }
    const float v0 = __fmaf_rn(sd0, n0, a0), v1 = __fmaf_rn(sd1, n1, a1);
    *pa[k] = v0;
    *pb[k] = -v0;
    *pa[k + 1] = v1;
    *pb[k + 1] = -v1;
  }
}

template <typename T, bool FOSTER>
__device__ __forceinline__ void levy_quad_pairs(const T* const (&pw_i)[4], const T* const (&pw_j)[4], int off, int m,
                                                T* const (&pa)[4], T* const (&pb)[4], const T (&z)[4], T tenth_h,
                                                T davie_std) {
  if constexpr (sizeof(T) == 4) {
    levy_quad_pairs_f32<FOSTER>(pw_i, pw_j, off, m, pa, pb, z, tenth_h, davie_std);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const T v = levy_pair_value_t<T, FOSTER>(pw_i[k][off], pw_j[k][off], pw_i[k][off + m], pw_j[k][off + m], z[k],
                                               tenth_h, davie_std);
      *pa[k] = v;
      *pb[k] = -v;
    }
  }
}

// GEN: the row's W and H are not read but drawn from the counter (primary cell `cell_id` of length h: W = sqrt(h) N_W,
// H = sqrt(h/12) N_H, as counter_noise does), and W and U = h (W/2 + H) are written out as well: one launch answers a
// whole-cell query bm(ta, tb, return_U=True, return_A=True) (brownian_interval.py:589-687).
// MT: the channel count as a compile-time constant (0 = run-time `m_rt`); with it the tile stride, the pair count
// and the copy-out pattern fold into immediates.
template <typename T, bool GEN, int MT>
__global__ void __launch_bounds__(kLevyWarps * 32, (MT && sizeof(T) == 4) ? kLevyCtasF32 : 3)
levy_tile_kernel(const void* keyp, int64_t row_offset, uint64_t a_id, int64_t rows, int m_rt, int warps,
                 const T* __restrict__ w, const T* __restrict__ hh, T tenth_h, T davie_std, int foster,
                 T* __restrict__ out, int vec, uint64_t cell_id, T sqrt_h, T sqrt_h12, T ht, T* __restrict__ out_w,
                 T* __restrict__ out_u) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int m = MT ? MT : m_rt;
  const int mm = m * m;
  const int npairs = (m * (m - 1)) >> 1;
  const int ld = m + 1;                                   // padded row stride of the shared tile: the mirrored stores
                                                          // sA[j][i] of consecutive lanes then fall into different banks
                                                          // (with stride m = 16 they are 16-way conflicts)
  const int tile = levy_tile_elems(m, GEN);
  const int R = levy_group_rows(m, GEN);                   // rows per pass (1 unless generating)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char* pairs_i = smem_raw;                       // [npairs] row index of pair p
  unsigned char* pairs_j = pairs_i + npairs;               // [npairs] column index
  T* tiles = reinterpret_cast<T*>(smem_raw + (((size_t)2 * npairs + 15) & ~(size_t)15));
  T* sA = tiles + (size_t)warp * tile;
  T* sW = sA + m * ld;                                     // row r of the pass: W at sW + 2 m r, H at sW + 2 m r + m
  T* scratch = sW + 2 * m * R;
  // pair table (shared by the CTA) and the tile's zero diagonal (written once: rows never touch it)
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    int p = i * m - (i * (i + 1)) / 2;                     // first pair of row i
    for (int j = i + 1; j < m; ++j, ++p) { pairs_i[p] = (unsigned char)i; pairs_j[p] = (unsigned char)j; }
  }
  if (warp < warps) for (int i = lane; i < m; i += 32) sA[i * ld + i] = T(0);
  __syncthreads();
  if (warp >= warps) return;
  const Key key = load_key(keyp);
  const int nq = (npairs + 3) >> 2;
  const int64_t row_stride = (int64_t)gridDim.x * warps;
  // A lane's pairs do not depend on the row when one pass covers them (nq <= 32, i.e. m <= 16): look them up once.
  const bool one_pass = nq <= 32;
  const T* pw_i[4];
  const T* pw_j[4];
  T* pa[4];
  T* pb[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int p = 4 * lane + k;
    const bool ok = one_pass && p < npairs;
    const int i = ok ? pairs_i[p] : 0, j = ok ? pairs_j[p] : 0;
    pw_i[k] = sW + i;
    pw_j[k] = sW + j;
    pa[k] = ok ? sA + i * ld + j : scratch;   // A_ij
    pb[k] = ok ? sA + j * ld + i : scratch;   // A_ji
  }
  // likewise the (up to two, m <= 16) groups of 4 consecutive output elements a lane copies out per row
  const bool copy_cached = vec && mm <= 256;
  int src_off[2], dst_off[2];
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int e = 4 * lane + 128 * t;
    const int i = e / m;
    dst_off[t] = (copy_cached && e < mm) ? e : -1;
    src_off[t] = i * ld + (e - i * m);
  }
  // W | H of a row: element c of the 2m-vector (c < m: W_c, else H_{c-m}) is loaded by lane c % 32; the next row's
  // elements are fetched while the current row is worked on.
  T pre[4] = {T(0), T(0), T(0), T(0)};
  const T* wh_src[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int c = lane + 32 * t;
    wh_src[t] = (c < m) ? w + c : hh + (c - m);
  }
  int64_t base = ((int64_t)blockIdx.x * warps + warp) * R;
  if (!GEN && base < rows) {
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (lane + 32 * t < 2 * m) pre[t] = wh_src[t][base * m];
  }
  for (; base < rows; base += row_stride * R) {
    if (GEN) {
      const int mq = m >> 2, gq = 2 * mq;                  // (host guarantees m % 4 == 0 in this mode)
      for (int t = lane; t < R * gq; t += 32) {            // one trip: R gq <= 32
        const int rg = t / gq, tq = t - rg * gq;
        const bool is_h = tq >= mq;
        const int q = is_h ? tq - mq : tq;
        const int64_t row = base + rg;                     // rows past the end are drawn but not stored
        T n[4], v[4];
        normal4(key, cell_id, is_h ? STREAM_H : STREAM_W, (uint32_t)(row + row_offset), (uint32_t)q, n);
        const T sc = is_h ? sqrt_h12 : sqrt_h;
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = n[j] * sc;
        st4(sW + 2 * m * rg + (is_h ? m : 0) + 4 * q, v);
        if (!is_h && row < rows) st4(out_w + row * m + 4 * q, v);
      }
      __syncwarp();
      for (int t = lane; t < R * mq; t += 32) {
        const int rg = t / mq, q = t - rg * mq;
        const int64_t row = base + rg;
        if (row < rows) {
          T a4[4], b4[4], u4[4];
          ld4(sW + 2 * m * rg + 4 * q, a4);
          ld4(sW + 2 * m * rg + m + 4 * q, b4);
#pragma unroll
          for (int j = 0; j < 4; ++j) u4[j] = ht * (T(0.5) * a4[j] + b4[j]);   // _H_to_U :102-103
          st4(out_u + row * m + 4 * q, u4);
        }
      }
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (lane + 32 * t < 2 * m) sW[lane + 32 * t] = pre[t];
      __syncwarp();
      const int64_t nxt = base + row_stride;
      if (nxt < rows) {
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (lane + 32 * t < 2 * m) pre[t] = wh_src[t][nxt * m];
      }
    }
#pragma unroll 1
    for (int rg = 0; rg < R; ++rg) {
      const int64_t row = base + rg;
      if (GEN && row >= rows) break;
      const int off = GEN ? 2 * m * rg : 0;
      const uint32_t grow = (uint32_t)(row + row_offset);
      if (one_pass) {
        if (lane < nq) {
          T z[4];
          normal4(key, a_id, STREAM_A, grow, (uint32_t)lane, z);
          if (foster) levy_quad_pairs<T, true>(pw_i, pw_j, off, m, pa, pb, z, tenth_h, davie_std);
          else levy_quad_pairs<T, false>(pw_i, pw_j, off, m, pa, pb, z, tenth_h, davie_std);
        }
      } else {
        const T* rW = sW + off;
        const T* rH = rW + m;
        for (int q = lane; q < nq; q += 32) {
          T z[4];
          normal4(key, a_id, STREAM_A, grow, (uint32_t)q, z);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int p = 4 * q + k;
            if (p < npairs) {
              const int i = pairs_i[p], j = pairs_j[p];
              const T v = levy_pair_value(rW[i], rW[j], rH[i], rH[j], z[k], tenth_h, davie_std, foster);
              sA[i * ld + j] = v;
              sA[j * ld + i] = -v;
            }
          }
        }
      }
      __syncwarp();
      T* dst = out + row * (int64_t)mm;
      if (copy_cached) {
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          if (dst_off[t] >= 0) {
            const T* src = sA + src_off[t];
            const T v4[4] = {src[0], src[1], src[2], src[3]};
            st4(dst + dst_off[t], v4);
          }
        }
      } else if (vec) {   // m % 4 == 0: a lane gathers 4 consecutive columns of one tile row, one 128-bit store
        for (int e = 4 * lane; e < mm; e += 128) {
          const int i = e / m, j0 = e - i * m;
          const T* src = sA + i * ld + j0;
          const T v4[4] = {src[0], src[1], src[2], src[3]};
          st4(dst + e, v4);
        }
      } else {
        for (int e = lane; e < mm; e += 32) {
          const int i = e / m;
          dst[e] = sA[i * ld + (e - i * m)];
        }
      }
      // Reading mode: no barrier here — the next row's tile stores come after the barrier that follows its W | H
      // stores, and those only overwrite what was last read before the barrier above.  Generating mode: the next
      // row of the pass writes the tile straight away.
      if (GEN) __syncwarp();
    }
  }
}

// Fallback for Brownian motions with more than 64 channels (the tile would not fit): one thread per element.
template <typename T>
__global__ void __launch_bounds__(kThreads)
levy_area_kernel(const void* keyp, int64_t row_offset, uint64_t a_id, int64_t rows, int64_t m,
                 const T* w, const T* hh, T tenth_h, T davie_std, int foster, T* out) {
  const Key key = load_key(keyp);
  const int64_t mm = m * m, total = rows * mm;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += stride) {
    const int64_t row = e / mm;
    const int64_t ij = e - row * mm;
    const int64_t i = ij / m, j = ij - i * m;
    if (i == j) { out[e] = T(0); continue; }
    const int64_t lo = i < j ? i : j, hi_ = i < j ? j : i;
    const int64_t p = lo * m - (lo * (lo + 1)) / 2 + (hi_ - lo - 1);
    T n4[4];
    normal4(key, a_id, STREAM_A, (uint32_t)(row + row_offset), (uint32_t)(p >> 2), n4);
    const T v = levy_pair_value(w[row * m + lo], w[row * m + hi_], hh[row * m + lo], hh[row * m + hi_], n4[p & 3],
                                tenth_h, davie_std, foster);
    out[e] = i < j ? v : -v;
  }
}

// A <- A + Ai + 0.5 (W (x) Wi - Wi (x) W)                         brownian_interval.py:671
template <typename T>
__global__ void __launch_bounds__(kThreads)
merge_area_kernel(int64_t rows, int64_t m, T* a0, const T* a1, const T* w0, const T* w1) {
  const int64_t mm = m * m, total = rows * mm;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += stride) {
    const int64_t row = e / mm;
    const int64_t ij = e - row * mm;
    const int64_t i = ij / m, j = ij - i * m;
    const T x = w0[row * m + i] * w1[row * m + j] - w1[row * m + i] * w0[row * m + j];
    a0[e] = (a0[e] + a1[e]) + T(0.5) * x;
  }
}

}  // namespace tsde

using namespace tsde;

constexpr int kLevyNoTile = -54321;

template <typename T, bool GEN>
static int launch_levy_tiles(const tsde_launch* L, const void* key, int64_t row_offset, uint64_t a_id, const void* w,
                             const void* hh, double h, int32_t foster, void* out_a, uint64_t cell_id, void* out_w,
                             void* out_u, cudaStream_t st) {
  const int64_t m = L->m;
  const int npairs = (int)(m * (m - 1) / 2);
  const size_t tile = (size_t)levy_tile_elems((int)m, GEN) * sizeof(T);
  const size_t table = ((size_t)2 * npairs + 15) & ~(size_t)15;
  int warps = (int)((46 * 1024 - table) / tile);
  if (warps > kLevyWarps) warps = kLevyWarps;
  if (warps < 1) return kLevyNoTile;
  const size_t smem = table + (size_t)warps * tile;
  const int vec = (m % 4 == 0 && aligned16(out_a)) ? 1 : 0;   // groups of 4 consecutive columns of one row
  const auto kernel = m == 16 ? levy_tile_kernel<T, GEN, 16>
                      : m == 8 ? levy_tile_kernel<T, GEN, 8>
                               : levy_tile_kernel<T, GEN, 0>;
  // persistent: exactly the CTAs that are resident at once (one wave), rows strided over them
  int per_sm = resident_ctas(reinterpret_cast<const void*>(kernel), kLevyWarps * 32, smem);
  if (per_sm < 1) per_sm = 1;
  const int64_t per_cta = (int64_t)warps * levy_group_rows((int)m, GEN);
  return launch_kernel(kernel, capped_grid(L->rows, per_cta, per_sm), kLevyWarps * 32, smem, st, false, key,
                       row_offset, a_id, L->rows, (int)m, warps, (const T*)w, (const T*)hh, (T)(0.1 * h),
                       (T)sqrt((1.0 / 12.0) * h * h), foster, (T*)out_a, vec, cell_id, (T)sqrt(h), (T)sqrt(h / 12.0),
                       (T)h, (T*)out_w, (T*)out_u);
}

// One launch for a whole-cell query with Levy area: W, U and A of primary cell nz->cell_id.
template <typename T>
static int cell_levy_impl(const tsde_launch* L, const tsde_noise* nz, uint64_t a_id, int32_t foster, void* out_w,
                          void* out_u, void* out_a) {
  if (!nz || nz->source != TSDE_SRC_COUNTER || !nz->key || nz->n_cells != 1 || !out_w || !out_u || !out_a)
    return TSDE_EINVAL;
  const int64_t m = L->m;
  if (m < 4 || m > 64 || (m % 4) != 0 || !aligned16(out_w) || !aligned16(out_u)) return TSDE_EINVAL;
  if (L->rows + nz->row_offset > kMaxGlobalRows) return TSDE_EINVAL;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  const int rc = launch_levy_tiles<T, true>(L, nz->key, nz->row_offset, a_id, nullptr, nullptr, nz->h, foster, out_a,
                                            nz->cell_id, out_w, out_u, st);
  return rc == kLevyNoTile ? TSDE_EINVAL : rc;
}

template <typename T>
static int levy_impl(const tsde_launch* L, const void* key, int64_t row_offset, uint64_t a_id,
                     const void* w, const void* hh, double h, int32_t foster, void* out_a) {
  if (!key || !w || !hh || !out_a) return TSDE_EINVAL;
  if (L->rows + row_offset > kMaxGlobalRows) return TSDE_EINVAL;
  if (L->m * L->m > (1ll << 26)) return TSDE_EINVAL;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  const double r12 = 1.0 / 12.0;
  const int64_t m = L->m;
  if (m >= 2 && m <= 64) {
    const int rc = launch_levy_tiles<T, false>(L, key, row_offset, a_id, w, hh, h, foster, out_a, 0, nullptr, nullptr, st);
    if (rc != kLevyNoTile) return rc;
  }
  return launch_kernel(levy_area_kernel<T>, capped_grid(L->rows * m * m, kThreads, kBlocksPerSM), kThreads, 0, st,
                       false, key, row_offset, a_id, L->rows, m, (const T*)w, (const T*)hh, (T)(0.1 * h),
                       (T)sqrt(r12 * h * h), foster, (T*)out_a);
}

template <typename T>
static int merge_area_impl(const tsde_launch* L, void* a0, const void* a1, const void* w0,
                           const void* w1) {
  if (!a0 || !a1 || !w0 || !w1) return TSDE_EINVAL;
  return launch_kernel(merge_area_kernel<T>, capped_grid(L->rows * L->m * L->m, kThreads, kBlocksPerSM), kThreads,
                       0, reinterpret_cast<cudaStream_t>(L->stream), false, L->rows, L->m, (T*)a0, (const T*)a1,
                       (const T*)w0, (const T*)w1);
}


TSDE_EXPORT int tsde_brownian_cells(const tsde_launch* L, const tsde_noise* nz, void* out_w, void* out_u,
                                    void* out_h) {
  return dispatch(L, [&](auto t) { return cells_impl<decltype(t)>(L, nz, out_w, out_u, out_h); });
}

TSDE_EXPORT int tsde_brownian_cell_levy(const tsde_launch* L, const tsde_noise* nz, uint64_t a_id, int32_t foster,
                                        void* out_w, void* out_u, void* out_a) {
  return dispatch(L, [&](auto t) { return cell_levy_impl<decltype(t)>(L, nz, a_id, foster, out_w, out_u, out_a); });
}

TSDE_EXPORT int tsde_brownian_bridge(const tsde_launch* L, const void* key, int64_t row_offset, int32_t depth,
                                     const uint64_t* ids, const int32_t* is_left, const double* times,
                                     const void* in_w, const void* in_h, void* out_w, void* out_h) {
  return dispatch(L, [&](auto t) {
    return bridge_impl<decltype(t)>(L, key, row_offset, depth, ids, is_left, times, in_w, in_h, out_w, out_h);
  });
}

TSDE_EXPORT int tsde_brownian_merge(const tsde_launch* L, void* w0, void* h0, const void* w1, const void* h1,
                                    double len0, double len1, double tot) {
  return dispatch(L, [&](auto t) {
    using T = decltype(t);
    const tsde_launch r = as_rows_m(L);
    if (h0 && h1) {
      const void* ins[4] = {w0, h0, w1, h1};
      void* outs[2] = {w0, h0};
      return launch_ew<T>(&r, nullptr, false, ins, outs, MergeWHOp<T>{(T)len1, (T)len0, (T)tot});
    }
    const void* ins[2] = {w0, w1};
    void* outs[1] = {w0};
    return launch_ew<T>(&r, nullptr, false, ins, outs, AddOp<T>{});
  });
}

TSDE_EXPORT int tsde_brownian_h_to_u(const tsde_launch* L, const void* w, const void* hh, double h, void* out_u) {
  return dispatch(L, [&](auto t) {
    using T = decltype(t);
    const tsde_launch r = as_rows_m(L);
    const void* ins[2] = {w, hh};
    void* outs[1] = {out_u};
    return launch_ew<T>(&r, nullptr, false, ins, outs, HToUOp<T>{(T)h});
  });
}

TSDE_EXPORT int tsde_brownian_levy_area(const tsde_launch* L, const void* key, int64_t row_offset, uint64_t a_id,
                                        const void* w, const void* hh, double h, int32_t foster, void* out_a) {
  return dispatch(L, [&](auto t) {
    return levy_impl<decltype(t)>(L, key, row_offset, a_id, w, hh, h, foster, out_a);
  });
}

TSDE_EXPORT int tsde_brownian_merge_area(const tsde_launch* L, void* a0, const void* a1, const void* w0,
                                         const void* w1) {
  return dispatch(L, [&](auto t) { return merge_area_impl<decltype(t)>(L, a0, a1, w0, w1); });
}

// ---- adaptive step-size control: error estimate --------------------------------------------------
// Sum over all elements of ((y11 - y12) / tol)^2 with tol = clamp_min(rtol*max(|y11|,|y12|) + atol, eps):
// the reduction inside compute_error / _rms of torchsde/_core/adaptive_stepping.py:42-76 (the host
// finishes with sqrt(sum / numel).clamp_min(eps)).  Two deterministic stages, double accumulation.
namespace tsde {

// A fixed partial count, not derived from the SM count: the summation order (and so every accept / reject decision of
// adaptive stepping) is the same on every device.  592 CTAs of 256 threads are one resident wave on 132 SMs.
constexpr int kErrBlocks = 592;

template <typename T>
__global__ void __launch_bounds__(kThreads)
err_partial_kernel(const T* __restrict__ a, const T* __restrict__ b, int64_t n, T rtol, T atol, T eps,
                   double* __restrict__ partial) {
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const T x = a[i], y = b[i];
    const T ax = x < T(0) ? -x : x, ay = y < T(0) ? -y : y;
    T tol = rtol * (ax > ay ? ax : ay) + atol;
    tol = tol < eps ? eps : tol;
    const T r = (x - y) / tol;
    acc += (double)(r * r);
  }
  __shared__ double sh[kThreads / 32];
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < kThreads / 32 ? sh[threadIdx.x] : 0.0;
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    if (threadIdx.x == 0) partial[blockIdx.x] = v;
  }
}

__global__ void err_final_kernel(const double* __restrict__ partial, int nb, double* __restrict__ out) {
  double v = 0.0;
  for (int i = threadIdx.x; i < nb; i += 32) v += partial[i];
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
  if (threadIdx.x == 0) out[0] = v;
}

template <typename T>
static int err_impl(const tsde_launch* L, const void* y11, const void* y12, double rtol, double atol,
                    double eps, void* scratch, void* out) {
  if (!y11 || !y12 || !scratch || !out) return TSDE_EINVAL;
  const int64_t n = L->rows * L->d;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(L->stream);
  int nb = (int)((n + kThreads - 1) / kThreads);
  if (nb > kErrBlocks) nb = kErrBlocks;
  if (int e = launch_kernel(err_partial_kernel<T>, nb, kThreads, 0, st, false, (const T*)y11, (const T*)y12, n,
                            (T)rtol, (T)atol, (T)eps, (double*)scratch))
    return e;
  return launch_kernel(err_final_kernel, 1, 32, 0, st, false, (const double*)scratch, nb, (double*)out);
}

}  // namespace tsde

TSDE_EXPORT int tsde_adaptive_error_sumsq(const tsde_launch* L, const void* y11, const void* y12, double rtol,
                                          double atol, double eps, void* scratch, void* out) {
  return tsde::dispatch(L, [&](auto t) {
    return tsde::err_impl<decltype(t)>(L, y11, y12, rtol, atol, eps, scratch, out);
  });
}
