// Step tableaus for diagonal noise (g:(rows,d), dW:(rows,d)) and for every stage that is
// purely element-wise: one kernel per op of tableau_diag_ops.cuh, which restates the `.step`
// bodies of torchsde/_core/methods/*.py with the reference's evaluation order (one IEEE
// rounding per ATen op, no FMA: this translation unit is compiled with -fmad=false).
//
// Scalar noise (g:(rows,d,1), dW:(rows,1)) also lands here: the contraction over a single
// Brownian channel is one product per element, so it is the diagonal formula with the
// increment broadcast along d (`bcast`).
#include <type_traits>

#include "tableau_diag_ops.cuh"

namespace tsde {

template <typename T, typename Op>
static int run(const tsde_launch* L, const tsde_noise* nz, std::initializer_list<const void*> ins,
               std::initializer_list<void*> outs, const Op& op) {
  const bool bcast = L->noise_type != TSDE_NOISE_DIAGONAL;  // scalar noise: one shared channel
  if (bcast && Op::USES_NOISE && L->m != 1) return TSDE_EINVAL;
  return launch_ew<T, Op>(L, nz, bcast, ins.begin(), outs.begin(), op);
}

// Entry points whose SDE outputs may be 16-bit: a launch that declares formats (float32 state only, see
// dispatch_fmt) takes the Mixed<Op> kernels, every other launch the ones it always took.
template <typename T, typename Op>
static int run_fmt(const tsde_launch* L, const tsde_noise* nz, std::initializer_list<const void*> ins,
                   std::initializer_list<void*> outs, const Op& op, uint32_t fmt, uint32_t ofmt = 0) {
  if constexpr (std::is_same<T, float>::value) {
    if (fmt) return run<T>(L, nz, ins, outs, Mixed<Op>{op, fmt, ofmt});
  }
  return run<T>(L, nz, ins, outs, op);
}

// ---- entry points ---------------------------------------------------------------------------------------------------
// The routes of cabi.cu for row-wise noise (the (rows,d,m) contractions of general noise live in tableau_general.cu).
int diag_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                    double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_euler, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, g}, {y1}, EulerOp<T>{(T)dt}, fmt);
  });
}

int diag_milstein_vjp_seed(const tsde_launch* L, const tsde_noise* nz, const void* g, double dt, int32_t ito,
                           void* go) {
  return dispatch_fmt(L, sde_out::milstein_vjp_seed, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {g}, {go}, MilsteinSeedOp<T>{(T)dt, ito}, fmt, fmt);
  });
}

int diag_step_milstein(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                       const void* gdg, double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_milstein, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, g, gdg}, {y1}, MilsteinOp<T>{(T)dt}, fmt);
  });
}

int diag_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* fp,
                   const void* g, const void* gp, double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, fp, g, gp}, {y1}, HeunOp<T>{(T)dt}, fmt);
  });
}

int diag_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                          double half_dt, void* yp) {
  return dispatch_fmt(L, sde_out::midpoint_predict, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, g}, {yp}, MidpointPredictOp<T>{(T)half_dt}, fmt);
  });
}

int diag_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* g, void* yp) {
  return dispatch_fmt(L, sde_out::euler_heun_predict, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, g}, {yp}, EulerHeunPredictOp<T>{}, fmt);
  });
}

int diag_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f, const void* g,
                         const void* gp, double dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_euler_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, g, gp}, {y1}, EulerHeunOp<T>{(T)dt}, fmt);
  });
}

int diag_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                           const void* f0, const void* g0, double dt, void* z1) {
  return dispatch_fmt(L, sde_out::reversible_heun_z, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, z0, f0, g0}, {z1}, RevHeunZOp<T>{(T)dt}, fmt);
  });
}

int diag_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                              const void* f1, const void* g0, const void* g1, double half_dt, void* y1) {
  return dispatch_fmt(L, sde_out::step_reversible_heun, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f0, f1, g0, g1}, {y1}, RevHeunOp<T>{(T)half_dt}, fmt);
  });
}

int diag_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* z0,
                                   const void* f0, const void* g0, const void* adj_y0, const void* adj_f0,
                                   const void* adj_g0, double dt, double half_dt, void* z1, void* adj_f0_out,
                                   void* adj_g0_out) {
  return dispatch_fmt(L, sde_out::adjoint_a, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, z0, f0, g0, adj_y0, adj_f0, adj_g0}, {z1, adj_f0_out, adj_g0_out},
                  AdjRevHeunAOp<T>{(T)dt, (T)half_dt}, fmt);
  });
}

int diag_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                   const void* f1, const void* g0, const void* g1, const void* adj_y0,
                                   const void* adj_z0, const void* vjp_z, double dt, double half_dt, void* y1,
                                   void* adj_y1, void* adj_z1, void* adj_f1, void* adj_g1) {
  return dispatch_fmt(L, sde_out::adjoint_b, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f0, f1, g0, g1, adj_y0, adj_z0, vjp_z}, {y1, adj_y1, adj_z1, adj_f1, adj_g1},
                  AdjRevHeunBOp<T>{(T)dt, (T)half_dt}, fmt);
  });
}

}  // namespace tsde

using namespace tsde;

// Exported entry points that are row-wise for every noise type they are called with.
TSDE_EXPORT int tsde_milstein_gf_predict(const tsde_launch* L, const void* y0, const void* f, const void* g,
                                         double dt, double sqrt_dt, int32_t ito, void* yp) {
  return dispatch_fmt(L, sde_out::milstein_gf_predict, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nullptr, {y0, f, g}, {yp}, MilsteinGfPredictOp<T>{(T)dt, (T)sqrt_dt, ito}, fmt);
  });
}

TSDE_EXPORT int tsde_step_milstein_gf(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                                      const void* g, const void* gp, double dt, double two_sqrt_dt, int32_t ito,
                                      void* y1) {
  return dispatch_fmt(L, sde_out::step_milstein_gf, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f, g, gp}, {y1}, MilsteinGfOp<T>{(T)dt, (T)two_sqrt_dt, ito}, fmt);
  });
}

TSDE_EXPORT int tsde_srk_diag_stage1(const tsde_launch* L, const void* y0, const void* f0, const void* g0, double dt,
                                     double sqrt_dt, void* h0_1, void* h1_1) {
  return dispatch_fmt(L, sde_out::srk_diag_stage1, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nullptr, {y0, f0, g0}, {h0_1, h1_1}, SrkDiagStage1Op<T>{(T)dt, (T)sqrt_dt}, fmt);
  });
}

TSDE_EXPORT int tsde_srk_diag_stage2(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                     const void* g0, const void* f1, const void* g1, double dt, double rdt,
                                     double sqrt_dt, void* h0_2, void* h1_2) {
  return dispatch_fmt(L, sde_out::srk_diag_stage2, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f0, g0, f1, g1}, {h0_2, h1_2}, SrkDiagStage2Op<T>{(T)dt, (T)rdt, (T)sqrt_dt}, fmt);
  });
}

TSDE_EXPORT int tsde_srk_diag_stage3(const tsde_launch* L, const void* y0, const void* g0, const void* g1,
                                     const void* f2, const void* g2, double dt, double sqrt_dt, void* h1_3) {
  return dispatch_fmt(L, sde_out::srk_diag_stage3, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nullptr, {y0, g0, g1, f2, g2}, {h1_3}, SrkDiagStage3Op<T>{(T)dt, (T)sqrt_dt}, fmt);
  });
}

TSDE_EXPORT int tsde_step_srk_diag(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f0,
                                   const void* f1, const void* f2, const void* g0, const void* g1, const void* g2,
                                   const void* g3, double dt, double rdt, double sqrt_dt, double three_dt,
                                   void* y1) {
  return dispatch_fmt(L, sde_out::step_srk_diag, [&](auto t, uint32_t fmt) {
    using T = decltype(t);
    return run_fmt<T>(L, nz, {y0, f0, f1, f2, g0, g1, g2, g3}, {y1}, make_srk_final<T>(dt, rdt, sqrt_dt, three_dt), fmt);
  });
}

TSDE_EXPORT int tsde_linear_interp(const tsde_launch* L, const void* y0, const void* y1, double w0, double w1,
                                   void* out) {
  return dispatch(L, [&](auto t) {
    using T = decltype(t);
    return run<T>(L, nullptr, {y0, y1}, {out}, LerpOp<T>{(T)w0, (T)w1});
  });
}
