// Host-side plumbing shared by every entry point: what the library exports, what a valid launch is, the dtype
// dispatch, and how kernels are sized and launched.  Nothing in this header runs on the device.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <utility>

#include "../../include/torchsde_b200.h"

// The library is compiled with -fvisibility=hidden: the definitions of the public header's functions, and nothing
// else, carry this.
#define TSDE_EXPORT extern "C" __attribute__((visibility("default")))

namespace tsde {

constexpr int kSMs = 132;  // H100 SXM; only a fallback, sm_count() asks the device

// Global rows (local row + row_offset) are one 32-bit word of the Philox counter.
constexpr int64_t kMaxGlobalRows = 0xFFFFFFFFll;
// A channel quad (channel / 4) is the low 24 bits of another word, with the stream tag above it (philox.cuh): past
// 2^26 channels one stream's normals would be another stream's.
constexpr int64_t kMaxCounterChannels = 1ll << 26;

// Launches issued per kernel family (TSDE_KERNEL_*), read by tsde_kernel_launches.
constexpr int kKernelFamilies = 10;
inline std::atomic<int64_t> g_launches[kKernelFamilies];

// The contraction of a GENERAL-noise launch with m channels: cabi.cu sends m == 1 to the row-wise kernels (one product
// g * dW), launch_gen picks among the others (tableau_general.cu describes each kernel's summation order), and the
// element-wise general kernels (pointwise.cu) sum in the order of the route this gives them.  `quads`: g (and memory
// noise) loadable as 16-byte quads; `row_bytes`: one row of increments (W, and U when the op wants it) in shared memory.
enum { TSDE_GEN_ROWWISE = 0, TSDE_GEN_TILE = 1, TSDE_GEN_GENERIC = 2, TSDE_GEN_WIDE = 3 };
inline int gen_route(int64_t m, bool quads, int64_t row_bytes) {
  if (m == 1) return TSDE_GEN_ROWWISE;
  const int64_t mq = m / 4;
  if (quads && m % 4 == 0 && mq >= 1 && mq <= 32 && (mq & (mq - 1)) == 0) return TSDE_GEN_TILE;
  return row_bytes > 40 * 1024 ? TSDE_GEN_WIDE : TSDE_GEN_GENERIC;
}

// A launch descriptor every entry point can rely on: non-null, non-negative row count, positive widths.
inline bool valid_launch(const tsde_launch* L) { return L && L->rows >= 0 && L->d > 0 && L->m > 0; }

// The checks every entry point makes, in this order: a valid launch descriptor and a known dtype, else TSDE_EINVAL;
// then an empty batch is a no-op (its tensors have no storage, so their pointers are null).  Otherwise `body` runs
// with a value of the element type, float{} or double{}, and its result is returned.
template <typename F>
inline int dispatch(const tsde_launch* L, F&& body) {
  if (!valid_launch(L) || (L->dtype != TSDE_F32 && L->dtype != TSDE_F64)) return TSDE_EINVAL;
  if (L->rows == 0) return 0;
  return L->dtype == TSDE_F32 ? body(float{}) : body(double{});
}

// dispatch() for the entry points whose SDE outputs may be 16-bit (TSDE_FMT_*).  Bit i of `sde_outputs` marks input
// i as an SDE output.  Format bits anywhere else, with an F64 state, or of value 3 are TSDE_EINVAL (checked before
// the empty-batch no-op).  `body` gets the element type of the state and the launch's format word (dtype >> 8; 0 for
// an all-state-dtype launch, always 0 with an F64 state).
template <typename F>
inline int dispatch_fmt(const tsde_launch* L, uint32_t sde_outputs, F&& body) {
  if (!valid_launch(L)) return TSDE_EINVAL;
  const int32_t state = L->dtype & 0xff;
  const uint32_t fmt = (uint32_t)L->dtype >> 8;
  if (state != TSDE_F32 && state != TSDE_F64) return TSDE_EINVAL;
  if (fmt && state != TSDE_F32) return TSDE_EINVAL;
  for (int i = 0; i < 12; ++i) {
    const uint32_t f = (fmt >> (2 * i)) & 3u;
    if (f == 3u || (f && !((sde_outputs >> i) & 1u))) return TSDE_EINVAL;
  }
  if (L->rows == 0) return 0;
  return state == TSDE_F32 ? body(float{}, fmt) : body(double{}, 0u);
}

inline int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) cudaGetLastError();
  return dev;
}

// SMs of the current device, asked once per device.
inline int sm_count() {
  static std::atomic<int> cache[64];
  const int dev = current_device();
  std::atomic<int>* slot = dev >= 0 && dev < 64 ? &cache[dev] : nullptr;
  int n = slot ? slot->load(std::memory_order_relaxed) : 0;
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = kSMs;
    }
    if (slot) slot->store(n, std::memory_order_relaxed);
  }
  return n;
}

struct ResidencyKey {  // (a type of this library, so the map's code is hidden like the rest: see TSDE_EXPORT)
  const void* kernel;
  int device;
  size_t smem;
  bool operator<(const ResidencyKey& o) const {
    if (kernel != o.kernel) return kernel < o.kernel;
    return device != o.device ? device < o.device : smem < o.smem;
  }
};

// Resident CTAs per SM of `kernel` at `threads` threads and `smem` bytes of dynamic shared memory on the current
// device, asked once per (kernel, device, smem); 0 if it cannot run there.  A kernel that needs more dynamic shared
// memory than it may use by default is opted in first.  The opt-in only ever grows, so every size asked for before
// stays launchable.
inline int resident_ctas(const void* kernel, int threads, size_t smem) {
  static std::mutex mu;
  static std::map<ResidencyKey, int> cache;
  const ResidencyKey key{kernel, current_device(), smem};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  int n = 0;
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess ||
      (smem > (size_t)fa.maxDynamicSharedSizeBytes &&
       cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem) != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  cache.emplace(key, n);
  return n;
}

// ceil(n / per_block) CTAs, at most ctas_per_sm on every SM of the current device.
inline int64_t capped_grid(int64_t n, int64_t per_block, int64_t ctas_per_sm) {
  const int64_t blocks = (n + per_block - 1) / per_block, cap = (int64_t)sm_count() * ctas_per_sm;
  return blocks < cap ? blocks : cap;
}

// Enqueue `kernel` on `st`.  `pdl` lets it start while its predecessor in the stream is still draining
// (programmatic dependent launch; the kernel orders itself with griddepcontrol.wait).  Returns the launch's
// cudaError_t and leaves no error state behind.
template <typename... P, typename... A>
inline int launch_kernel(void (*kernel)(P...), int64_t grid, int block, size_t smem, cudaStream_t st, bool pdl,
                         A&&... args) {
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  if (e != cudaSuccess) cudaGetLastError();
  return (int)e;
}

// launch_kernel for a kernel handle of a library loaded at run time (cudaLibraryGetKernel): `args` points at each of its
// parameters.  No dynamic shared memory.
inline int launch_kernel_handle(cudaKernel_t kernel, int64_t grid, int block, cudaStream_t st, void** args) {
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(block);
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kernel), args);
  if (e != cudaSuccess) cudaGetLastError();
  return (int)e;
}

// Why the last run-time compilation of an element-wise program failed (pointwise.cu; tsde_error_string(TSDE_ECOMPILE))
std::string pw_compile_error();

// ---- which inputs of an entry point are SDE outputs (dispatch_fmt): bit i = input i of its declaration -------------
namespace sde_out {
constexpr uint32_t step_euler = 0b110;              // y0, f, g
constexpr uint32_t milstein_vjp_seed = 0b1;         // g
constexpr uint32_t step_milstein = 0b0110;          // y0, f, g, gdg
constexpr uint32_t milstein_gf_predict = 0b110;     // y0, f, g
constexpr uint32_t step_milstein_gf = 0b1110;       // y0, f, g, gp
constexpr uint32_t step_heun = 0b11110;             // y0, f, fp, g, gp
constexpr uint32_t midpoint_predict = 0b110;        // y0, f, g
constexpr uint32_t euler_heun_predict = 0b10;       // y0, g
constexpr uint32_t step_euler_heun = 0b1110;        // y0, f, g, gp
constexpr uint32_t reversible_heun_z = 0b1100;      // y0, z0, f0, g0
constexpr uint32_t step_reversible_heun = 0b11110;  // y0, f0, f1, g0, g1
constexpr uint32_t adjoint_a = 0b1100;              // y0, z0, f0, g0, adj_y0, adj_f0, adj_g0
constexpr uint32_t adjoint_b = 0b11110;             // y0, f0, f1, g0, g1, adj_y0, adj_z0, vjp_z
constexpr uint32_t srk_diag_stage1 = 0b110;         // y0, f0, g0
constexpr uint32_t srk_diag_stage2 = 0b11110;       // y0, f0, g0, f1, g1
constexpr uint32_t srk_diag_stage3 = 0b11110;       // y0, g0, g1, f2, g2
constexpr uint32_t step_srk_diag = 0b11111110;      // y0, f0, f1, f2, g0, g1, g2, g3
constexpr uint32_t srk_additive_stage = 0b110;      // y0, f0, ga
constexpr uint32_t step_srk_additive = 0b11110;     // y0, f0, f1, ga, gb
}  // namespace sde_out

// ---- noise-layout routing of the tableau entry points (cabi.cu) ----------------------------------------------------
// Row-wise kernels (tableau_diag.cu): DIAGONAL noise, and GENERAL noise with a single Brownian channel.
int diag_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                    double dt, void* y1);
int diag_milstein_vjp_seed(const tsde_launch* L, const tsde_noise* nz, const void* g, double dt, int32_t ito,
                           void* go);
int diag_step_milstein(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                       const void* gdg, double dt, void* y1);
int diag_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* fp,
                   const void* g, const void* gp, double dt, void* y1);
int diag_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                          double half_dt, void* yp);
int diag_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* g, void* yp);
int diag_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                         const void* gp, double dt, void* y1);
int diag_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                           const void* f0, const void* g0, double dt, void* z1);
int diag_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                              const void* f1, const void* g0, const void* g1, double half_dt, void* y1);
int diag_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                                   const void* f0, const void* g0, const void* adj_y0, const void* adj_f0,
                                   const void* adj_g0, double dt, double half_dt, void* z1, void* adj_f0_out,
                                   void* adj_g0_out);
int diag_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                   const void* f1, const void* g0, const void* g1, const void* adj_y0,
                                   const void* adj_z0, const void* vjp_z, double dt, double half_dt, void* y1,
                                   void* adj_y1, void* adj_z1, void* adj_f1, void* adj_g1);
// (rows, d, m) tile kernels (tableau_general.cu): GENERAL noise with m > 1.
int general_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                       double dt, void* y1);
int general_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* fp,
                      const void* g, const void* gp, double dt, void* y1);
int general_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                             const void* g, double half_dt, void* yp);
int general_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* g, void* yp);
int general_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                            const void* g, const void* gp, double dt, void* y1);
int general_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                              const void* f0, const void* g0, double dt, void* z1);
int general_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                 const void* f1, const void* g0, const void* g1, double half_dt, void* y1);
int general_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                                      const void* f0, const void* g0, const void* adj_y0, const void* adj_f0,
                                      const void* adj_g0, double dt, double half_dt, void* z1, void* adj_f0_out,
                                      void* adj_g0_out);
int general_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                      const void* f1, const void* g0, const void* g1, const void* adj_y0,
                                      const void* adj_z0, const void* vjp_z, double dt, double half_dt, void* y1,
                                      void* adj_y1, void* adj_z1, void* adj_f1, void* adj_g1);

}  // namespace tsde
