// Exported C ABI (include/torchsde_b200.h): noise-layout dispatch.
//   DIAGONAL, or GENERAL with a single Brownian channel (scalar noise)  -> tableau_diag.cu
//   GENERAL with m > 1 (general / additive noise)                        -> tableau_general.cu
#include "host.cuh"

using namespace tsde;

static inline bool rowwise(const tsde_launch* L) {
  return L->noise_type == TSDE_NOISE_DIAGONAL || gen_route(L->m, false, 0) == TSDE_GEN_ROWWISE;
}

// A valid launch of a known noise layout (diagonal noise has m == d), with launch flags the routed kernels understand:
// unknown bits are a contract violation, and a batch-broadcast g is only understood by the (rows,d,m) tile kernels
// (the row-wise kernels address g per row).
static inline bool routable(const tsde_launch* L, const tsde_noise* nz) {
  if (!valid_launch(L)) return false;
  if (L->noise_type == TSDE_NOISE_DIAGONAL ? L->m != L->d : L->noise_type != TSDE_NOISE_GENERAL) return false;
  if (!nz) return true;
  if (nz->flags & ~TSDE_FLAG_G_BROADCAST) return false;
  return !((nz->flags & TSDE_FLAG_G_BROADCAST) && rowwise(L));
}

TSDE_EXPORT int tsde_abi_version(void) { return TSDE_ABI_VERSION; }

TSDE_EXPORT const char* tsde_error_string(int code) {
  if (code == TSDE_EINVAL) return "torchsde_b200: invalid argument (contract violation)";
  if (code == TSDE_ECOMPILE) {
    static thread_local std::string msg;
    msg = pw_compile_error();
    return msg.c_str();
  }
  return cudaGetErrorString((cudaError_t)code);
}

TSDE_EXPORT int tsde_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                                const void* g, double dt, void* y1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_step_euler(L, nz, y0, f, g, dt, y1) : general_step_euler(L, nz, y0, f, g, dt, y1);
}

TSDE_EXPORT int tsde_milstein_vjp_seed(const tsde_launch* L, const tsde_noise* nz, const void* g, double dt,
                                       int32_t ito, void* go) {
  if (!routable(L, nz) || !rowwise(L)) return TSDE_EINVAL;  // milstein.py:25: additive/diagonal/scalar only
  return diag_milstein_vjp_seed(L, nz, g, dt, ito, go);
}

TSDE_EXPORT int tsde_step_milstein(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                                   const void* g, const void* gdg, double dt, void* y1) {
  if (!routable(L, nz) || !rowwise(L)) return TSDE_EINVAL;
  return diag_step_milstein(L, nz, y0, f, g, gdg, dt, y1);
}

TSDE_EXPORT int tsde_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                               const void* fp, const void* g, const void* gp, double dt, void* y1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_step_heun(L, nz, y0, f, fp, g, gp, dt, y1)
                    : general_step_heun(L, nz, y0, f, fp, g, gp, dt, y1);
}

TSDE_EXPORT int tsde_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                                      const void* g, double half_dt, void* yp) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_midpoint_predict(L, nz, y0, f, g, half_dt, yp)
                    : general_midpoint_predict(L, nz, y0, f, g, half_dt, yp);
}

TSDE_EXPORT int tsde_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* g,
                                        void* yp) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_euler_heun_predict(L, nz, y0, g, yp) : general_euler_heun_predict(L, nz, y0, g, yp);
}

TSDE_EXPORT int tsde_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                                     const void* g, const void* gp, double dt, void* y1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_step_euler_heun(L, nz, y0, f, g, gp, dt, y1)
                    : general_step_euler_heun(L, nz, y0, f, g, gp, dt, y1);
}

TSDE_EXPORT int tsde_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                                       const void* f0, const void* g0, double dt, void* z1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_reversible_heun_z(L, nz, y0, z0, f0, g0, dt, z1)
                    : general_reversible_heun_z(L, nz, y0, z0, f0, g0, dt, z1);
}

TSDE_EXPORT int tsde_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                                          const void* f0, const void* f1, const void* g0, const void* g1,
                                          double half_dt, void* y1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_step_reversible_heun(L, nz, y0, f0, f1, g0, g1, half_dt, y1)
                    : general_step_reversible_heun(L, nz, y0, f0, f1, g0, g1, half_dt, y1);
}

TSDE_EXPORT int tsde_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                                               const void* z0, const void* f0, const void* g0, const void* adj_y0,
                                               const void* adj_f0, const void* adj_g0, double dt, double half_dt,
                                               void* z1, void* adj_f0_out, void* adj_g0_out) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_adjoint_reversible_heun_a(L, nz, y0, z0, f0, g0, adj_y0, adj_f0, adj_g0, dt, half_dt,
                                                     z1, adj_f0_out, adj_g0_out)
                    : general_adjoint_reversible_heun_a(L, nz, y0, z0, f0, g0, adj_y0, adj_f0, adj_g0, dt, half_dt,
                                                        z1, adj_f0_out, adj_g0_out);
}

TSDE_EXPORT int tsde_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                                               const void* f0, const void* f1, const void* g0, const void* g1,
                                               const void* adj_y0, const void* adj_z0, const void* vjp_z, double dt,
                                               double half_dt, void* y1, void* adj_y1, void* adj_z1, void* adj_f1,
                                               void* adj_g1) {
  if (!routable(L, nz)) return TSDE_EINVAL;
  return rowwise(L) ? diag_adjoint_reversible_heun_b(L, nz, y0, f0, f1, g0, g1, adj_y0, adj_z0, vjp_z, dt, half_dt,
                                                     y1, adj_y1, adj_z1, adj_f1, adj_g1)
                    : general_adjoint_reversible_heun_b(L, nz, y0, f0, f1, g0, g1, adj_y0, adj_z0, vjp_z, dt,
                                                        half_dt, y1, adj_y1, adj_z1, adj_f1, adj_g1);
}
