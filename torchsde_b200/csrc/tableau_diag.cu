// Step tableaus for diagonal noise (g:(rows,d), dW:(rows,d)) and for every stage that is
// purely element-wise.  Each op restates one `.step` body of torchsde/_core/methods/*.py with
// the reference's evaluation order (one IEEE rounding per ATen op, no FMA: this translation
// unit is compiled with -fmad=false).
//
// Scalar noise (g:(rows,d,1), dW:(rows,1)) also lands here: the contraction over a single
// Brownian channel is one product per element, so it is the diagonal formula with the
// increment broadcast along d (`bcast`).
#include <type_traits>

#include "ew.cuh"

namespace tsde {

// ----------------------------------------------------------------------------------------------
// y1 = y0 + f*dt + g*dW                                                     methods/euler.py:36
template <typename T>
struct EulerOp {
  static constexpr int NIN = 3, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T dt;
  __device__ __forceinline__ void operator()(const T (&in)[3], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2];
    out[0] = (y0 + f * dt) + g * w;
  }
};

// go = g * (0.5 * v)                       methods/milstein.py:56,69,80-81,90-91 base_sde.py:142-155
template <typename T>
struct MilsteinSeedOp {
  static constexpr int NIN = 1, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T dt;
  int ito;
  __device__ __forceinline__ void operator()(const T (&in)[1], T w, T, T (&out)[1]) const {
    const T v = ito ? (w * w - dt) : (w * w);
    out[0] = in[0] * (T(0.5) * v);
  }
};

// y1 = y0 + f*dt + g*dW + gdg                                               methods/milstein.py:72
template <typename T>
struct MilsteinOp {
  static constexpr int NIN = 4, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // y0, f, g, gdg are all dead after the step's last kernel
  T dt;
  __device__ __forceinline__ void operator()(const T (&in)[4], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2], gdg = in[3];
    out[0] = ((y0 + f * dt) + g * w) + gdg;
  }
};

// y' = y0 + (dt*f | 0.) + g*sqrt_dt                                          methods/milstein.py:63
template <typename T>
struct MilsteinGfPredictOp {
  static constexpr int NIN = 3, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T dt, sqrt_dt;
  int ito;
  __device__ __forceinline__ void operator()(const T (&in)[3], T, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2];
    const T fac = ito ? dt * f : T(0);
    out[0] = (y0 + fac) + g * sqrt_dt;
  }
};

// y1 = y0 + f*dt + g*dW + ((g'-g)*v)/(2*sqrt_dt)                             methods/milstein.py:65-72
template <typename T>
struct MilsteinGfOp {
  static constexpr int NIN = 4, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: every operand is dead afterwards
  T dt, two_sqrt_dt;
  int ito;
  __device__ __forceinline__ void operator()(const T (&in)[4], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2], gp = in[3];
    const T v = ito ? (w * w - dt) : (w * w);
    const T gdg = ((gp - g) * v) / two_sqrt_dt;
    out[0] = ((y0 + f * dt) + g * w) + gdg;
  }
};

// y1 = y0 + (dt*(f+f') + g*dW + g'*dW) * 0.5                                 methods/heun.py:46
template <typename T>
struct HeunOp {
  static constexpr int NIN = 5, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: every operand is dead afterwards
  T dt;
  __device__ __forceinline__ void operator()(const T (&in)[5], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], fp = in[2], g = in[3], gp = in[4];
    out[0] = y0 + ((dt * (f + fp) + g * w) + gp * w) * T(0.5);
  }
};

// y' = y0 + half_dt*f + 0.5*(g*dW)                                           methods/midpoint.py:38
template <typename T>
struct MidpointPredictOp {
  static constexpr int NIN = 3, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[3], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2];
    out[0] = (y0 + half_dt * f) + T(0.5) * (g * w);
  }
};

// y' = y0 + g*dW                                                             methods/euler_heun.py:36
template <typename T>
struct EulerHeunPredictOp {
  static constexpr int NIN = 2, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  __device__ __forceinline__ void operator()(const T (&in)[2], T w, T, T (&out)[1]) const {
    out[0] = in[0] + in[1] * w;
  }
};

// y1 = y0 + dt*f + (g*dW + g'*dW)*0.5                                        methods/euler_heun.py:40
template <typename T>
struct EulerHeunOp {
  static constexpr int NIN = 4, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: every operand is dead afterwards
  T dt;
  __device__ __forceinline__ void operator()(const T (&in)[4], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f = in[1], g = in[2], gp = in[3];
    out[0] = (y0 + dt * f) + (g * w + gp * w) * T(0.5);
  }
};

// z1 = 2*y0 - z0 + f0*dt + g0*dW                                             methods/reversible_heun.py:69
template <typename T>
struct RevHeunZOp {
  static constexpr int NIN = 4, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T dt;
  __device__ __forceinline__ void operator()(const T (&in)[4], T w, T, T (&out)[1]) const {
    const T y0 = in[0], z0 = in[1], f0 = in[2], g0 = in[3];
    out[0] = ((T(2) * y0 - z0) + f0 * dt) + g0 * w;
  }
};

// y1 = y0 + (f0+f1)*(0.5*dt) + (g0+g1)*(0.5*dW)                              methods/reversible_heun.py:71
template <typename T>
struct RevHeunOp {
  static constexpr int NIN = 5, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[5], T w, T, T (&out)[1]) const {
    const T y0 = in[0], f0 = in[1], f1 = in[2], g0 = in[3], g1 = in[4];
    out[0] = (y0 + (f0 + f1) * half_dt) + (g0 + g1) * (T(0.5) * w);
  }
};

// ---- SRK srid2, diagonal / scalar noise                   methods/srk.py:57-88, tableaus/srid2.py
// The accumulation `H0s + A*f*dt + B*g*I_k0*rdt` (srk.py:74-75) is evaluated as
// (H0s + (A*f)*dt) + ((B*g)*I_k0)*rdt ; rows whose coefficient is 0 add an exact 0.
template <typename T>
struct SrkDiagStage1Op {  // s = 1
  static constexpr int NIN = 3, NOUT = 2;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T dt, sqrt_dt;
  __device__ __forceinline__ void operator()(const T (&in)[3], T, T, T (&out)[2]) const {
    const T y0 = in[0], f0 = in[1], g0 = in[2];
    out[0] = y0 + (T(1) * f0) * dt;                                     // A0[1][0]=1, B0[1][0]=0
    out[1] = (y0 + (T(0.25) * f0) * dt) + (T(-0.5) * g0) * sqrt_dt;     // A1=1/4, B1=-1/2
  }
};
template <typename T>
struct SrkDiagStage2Op {  // s = 2
  static constexpr int NIN = 5, NOUT = 2;
  static constexpr bool USES_NOISE = true, WANT_U = true;
  T dt, rdt, sqrt_dt;
  __device__ __forceinline__ void operator()(const T (&in)[5], T, T u, T (&out)[2]) const {
    const T y0 = in[0], f0 = in[1], g0 = in[2], f1 = in[3], g1 = in[4];
    // j=0: A0=1/4 B0=1 ; A1=1 B1=1      j=1: A0=1/4 B0=1/2 ; A1=0 B1=0
    T h0 = (y0 + (T(0.25) * f0) * dt) + ((T(1) * g0) * u) * rdt;
    T h1 = (y0 + (T(1) * f0) * dt) + (T(1) * g0) * sqrt_dt;
    h0 = (h0 + (T(0.25) * f1) * dt) + ((T(0.5) * g1) * u) * rdt;
    out[0] = h0;
    out[1] = h1;
  }
};
template <typename T>
struct SrkDiagStage3Op {  // s = 3 : A0 = B0 = 0 -> H0_3 = y0 ; A1=(0,0,1/4) B1=(2,-1,1/2)
  static constexpr int NIN = 5, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T dt, sqrt_dt;
  __device__ __forceinline__ void operator()(const T (&in)[5], T, T, T (&out)[1]) const {
    const T y0 = in[0], g0 = in[1], g1 = in[2], f2 = in[3], g2 = in[4];
    T h1 = y0 + (T(2) * g0) * sqrt_dt;
    h1 = h1 + (T(-1) * g1) * sqrt_dt;
    h1 = (h1 + (T(0.25) * f2) * dt) + (T(0.5) * g2) * sqrt_dt;
    out[0] = h1;
  }
};
template <typename T>
struct SrkDiagFinalOp {
  static constexpr int NIN = 8, NOUT = 1;
  static constexpr bool USES_NOISE = true, WANT_U = true;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: every operand is dead afterwards
  T dt, rdt, sqrt_dt;
  T three_dt;              // 3*dt as the reference's 0-d tensor product (srk.py:64)
  T alpha[3];
  T b1[3], b2[3], b3[3], b4[4];
  __device__ __forceinline__ void operator()(const T (&in)[8], T w, T u, T (&out)[1]) const {
    const T y0 = in[0];
    const T f[3] = {in[1], in[2], in[3]};
    const T g[4] = {in[4], in[5], in[6], in[7]};
    const T ikk = (w * w - dt) * T(0.5);                       // srk.py:63
    const T r6 = (T)(1.0 / 6.0);
    const T i3 = ((w * w) * w - three_dt * w) * r6;           // srk.py:64
    T y1 = y0;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const T gw = ((b1[s] * w + (b2[s] * ikk) / sqrt_dt) + (b3[s] * u) * rdt) + (b4[s] * i3) * rdt;
      y1 = (y1 + (alpha[s] * f[s]) * dt) + g[s] * gw;
    }
    {  // s = 3: alpha = 0, beta = (0,0,0,1)
      const T gw = (b4[3] * i3) * rdt;
      y1 = y1 + g[3] * gw;
    }
    out[0] = y1;
  }
};

// ---- linear interpolation                                                  _core/interp.py:17
template <typename T>
struct LerpOp {
  static constexpr int NIN = 2, NOUT = 1;
  static constexpr bool USES_NOISE = false, WANT_U = false;
  T w0, w1;
  __device__ __forceinline__ void operator()(const T (&in)[2], T, T, T (&out)[1]) const {
    out[0] = w0 * in[0] + w1 * in[1];
  }
};

// ---- reversible-Heun adjoint, diagonal noise                     methods/reversible_heun.py:98-144
template <typename T>
struct AdjRevHeunAOp {
  static constexpr int NIN = 7, NOUT = 3;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T dt, half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[7], T w, T, T (&out)[3]) const {
    const T y0 = in[0], z0 = in[1], f0 = in[2], g0 = in[3];
    const T adj_y0 = in[4], adj_f0 = in[5], adj_g0 = in[6];
    const T half_dw = T(0.5) * w;                                   // :102
    out[0] = ((T(2) * y0 - z0) - f0 * dt) - g0 * w;                  // :109
    out[1] = adj_f0 + adj_y0 * half_dt;                              // :104,113
    out[2] = adj_g0 + adj_y0 * half_dw;                              // :105,115
  }
};
template <typename T>
struct AdjRevHeunBOp {
  static constexpr int NIN = 8, NOUT = 5;
  static constexpr bool USES_NOISE = true, WANT_U = false;
  T dt, half_dt;
  __device__ __forceinline__ void operator()(const T (&in)[8], T w, T, T (&out)[5]) const {
    const T y0 = in[0], f0 = in[1], f1 = in[2], g0 = in[3], g1 = in[4];
    const T adj_y0 = in[5], adj_z0_in = in[6], vjp_z = in[7];
    const T half_dw = T(0.5) * w;
    const T adj_z0 = adj_z0_in + vjp_z;                              // :130
    out[0] = (y0 - (f0 + f1) * half_dt) - (g0 + g1) * half_dw;       // :134-135
    out[1] = adj_y0 + T(2) * adj_z0;                                 // :137
    out[2] = -adj_z0;                                                // :138
    out[3] = adj_y0 * half_dt + adj_z0 * dt;                         // :112,139
    out[4] = adj_y0 * half_dw + adj_z0 * w;                          // :114,140
  }
};

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

template <typename T>
static SrkDiagFinalOp<T> make_srk_final(double dt, double rdt, double sqrt_dt, double three_dt) {
  SrkDiagFinalOp<T> op;
  op.dt = (T)dt;
  op.rdt = (T)rdt;
  op.sqrt_dt = (T)sqrt_dt;
  op.three_dt = (T)three_dt;
  // methods/tableaus/srid2.py:50-54
  const double alpha[3] = {1.0 / 6, 1.0 / 6, 2.0 / 3};
  const double b1[3] = {-1, 4.0 / 3, 2.0 / 3};
  const double b2[3] = {1, -4.0 / 3, 1.0 / 3};
  const double b3[3] = {2, -4.0 / 3, -2.0 / 3};
  const double b4[4] = {-2, 5.0 / 3, -2.0 / 3, 1};
  for (int i = 0; i < 3; ++i) {
    op.alpha[i] = (T)alpha[i];
    op.b1[i] = (T)b1[i];
    op.b2[i] = (T)b2[i];
    op.b3[i] = (T)b3[i];
  }
  for (int i = 0; i < 4; ++i) op.b4[i] = (T)b4[i];
  return op;
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

// ---- a whole Milstein step of an element-wise SDE (tsde_step_milstein_pointwise) ------------------------------------
// One thread per quad, as ew_fast_kernel: the increment is drawn before the dependency wait, then y0 is read, the
// program's f / g part runs, MilsteinSeedOp forms go, the vjp part runs and MilsteinOp writes y1.  Only y0 and y1 (and
// the program's device operands) touch memory: 2 tensors per step instead of the 13 of the unfused step.
//
// The program's registers live in shared memory as 16-byte vectors laid out [reg][plane][thread] (a float quad is one
// plane, a double quad two): a warp's 128-bit access is 512 contiguous bytes, conflict-free.  A dynamically indexed
// per-thread array would live in local memory instead.  y0, go, f, g and the increment stay in registers.
template <typename T>
struct PwP {
  const T* y0;
  T* y1;
  const T* t0;
  int64_t d, qpr, nquads;
  uint64_t qmagic;  // rowdiv_magic(qpr) when qpr is not a power of two
  int32_t qshift;   // log2(qpr), or -1
  int32_t small;    // nquads < 2^31
  int32_t vec;      // d % 4 == 0 and every tensor 16-byte aligned
  T dt;
  int32_t ito;
};

__device__ __forceinline__ void pw_sload(const void* s, int r, float (&v)[4]) {
  const float4 x = static_cast<const float4*>(s)[r * kThreads + threadIdx.x];
  v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
}
__device__ __forceinline__ void pw_sstore(void* s, int r, const float (&v)[4]) {
  static_cast<float4*>(s)[r * kThreads + threadIdx.x] = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void pw_sload(const void* s, int r, double (&v)[4]) {
  const double2* p = static_cast<const double2*>(s) + 2 * r * kThreads + threadIdx.x;
  const double2 a = p[0], b = p[kThreads];
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void pw_sstore(void* s, int r, const double (&v)[4]) {
  double2* p = static_cast<double2*>(s) + 2 * r * kThreads + threadIdx.x;
  p[0] = make_double2(v[0], v[1]);
  p[kThreads] = make_double2(v[2], v[3]);
}

template <typename T>
struct PwQuad {  // where this thread's quad lives, and the values a program source may name besides registers
  int64_t base, chan;
  int nvalid;
  bool vec;
  T y[4], go[4];
};

template <typename T>
__device__ __forceinline__ void pw_fetch(const tsde_pointwise& pg, const PwP<T>& p, const PwQuad<T>& c,
                                         const void* regs, uint32_t s, T (&v)[4]) {
  if (s == TSDE_PW_SRC_Y || s == TSDE_PW_SRC_GO) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = s == TSDE_PW_SRC_Y ? c.y[j] : c.go[j];
    return;
  }
  if (s < (uint32_t)TSDE_PW_OPERAND(0)) {
    pw_sload(regs, (int)s, v);
    return;
  }
  const tsde_pw_operand& o = pg.operand[s - TSDE_PW_OPERAND(0)];
  if (o.kind == TSDE_PW_CHANNEL || o.kind == TSDE_PW_ROW) {
    load_quad(static_cast<const T*>(o.ptr), o.kind == TSDE_PW_ROW ? c.base : c.chan, c.vec, c.nvalid, v);
    return;
  }
  const T x = o.kind == TSDE_PW_IMM ? (T)o.imm : *(o.kind == TSDE_PW_T0 ? p.t0 : static_cast<const T*>(o.ptr));
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = x;
}

// instructions [i0, i1): one warp-uniform dispatch per instruction, one IEEE rounding per element (-fmad=false)
template <typename T>
__device__ __forceinline__ void pw_run(const tsde_pointwise& pg, const PwP<T>& p, const PwQuad<T>& c, void* regs,
                                       int i0, int i1) {
  for (int i = i0; i < i1; ++i) {
    const tsde_pw_instr in = pg.instr[i];
    T a[4], b[4], r[4];
    pw_fetch(pg, p, c, regs, in.a, a);
    if (in.op != TSDE_PW_NEG && in.op != TSDE_PW_SQRT) pw_fetch(pg, p, c, regs, in.b, b);
    switch (in.op) {
      case TSDE_PW_MUL:
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = a[j] * b[j];
        break;
      case TSDE_PW_ADD:
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = a[j] + b[j];
        break;
      case TSDE_PW_SUB:
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = a[j] - b[j];
        break;
      case TSDE_PW_DIV:
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = a[j] / b[j];
        break;
      case TSDE_PW_NEG:
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = -a[j];
        break;
      default:  // TSDE_PW_SQRT
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = sqrt(a[j]);
        break;
    }
    pw_sstore(regs, in.dst, r);
  }
}

template <typename T, int SRC>
__global__ void __launch_bounds__(kThreads)
pw_milstein_kernel(const __grid_constant__ tsde_pointwise pg, const PwP<T> p, const NoiseP<T> nz) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  const int64_t Q = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  int64_t row, q;
  if (p.qshift >= 0) {
    row = Q >> p.qshift;
    q = Q & ((1ll << p.qshift) - 1);
  } else if (p.small) {
    const uint32_t r32 = rowdiv_row((uint32_t)Q, p.qmagic);
    row = r32;
    q = (int64_t)rowdiv_quad((uint32_t)Q, r32, (uint32_t)p.qpr);
  } else {
    row = Q / p.qpr;
    q = Q - row * p.qpr;
  }
  PwQuad<T> c;
  c.chan = 4 * q;
  c.base = row * p.d + c.chan;
  const int64_t rem = p.d - c.chan;
  c.nvalid = rem < 4 ? (int)rem : 4;
  c.vec = p.vec != 0;
  // the increment depends on no predecessor: drawn while the previous kernel drains (programmatic dependent launch)
  T w[4], u[4];
  quad_noise<T, SRC, false>(nz, load_key(nz.key), row, q, c.vec, c.nvalid, w, u);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.nquads) return;
  load_quad(p.y0, c.base, c.vec, c.nvalid, c.y);
#pragma unroll
  for (int j = 0; j < 4; ++j) c.go[j] = T(0);
  pw_run(pg, p, c, pw_regs, 0, pg.n_fg);
  T f[4], g[4];
  pw_fetch(pg, p, c, pw_regs, pg.f_src, f);
  pw_fetch(pg, p, c, pw_regs, pg.g_src, g);
  const MilsteinSeedOp<T> seed{p.dt, p.ito};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    seed({g[j]}, w[j], u[j], o);
    c.go[j] = o[0];
  }
  pw_run(pg, p, c, pw_regs, pg.n_fg, pg.n_instr);
  T gdg[4], y1[4];
  pw_fetch(pg, p, c, pw_regs, pg.gdg_src, gdg);
  const MilsteinOp<T> step{p.dt};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    step({c.y[j], f[j], g[j], gdg[j]}, w[j], u[j], o);
    y1[j] = o[0];
  }
  store_quad(p.y1, c.base, c.vec, c.nvalid, y1);
}

// ---- a whole SRK step of an element-wise SDE (tsde_step_srk_diag_pointwise) -----------------------------------------
// One thread per quad again: W and U are drawn before the dependency wait, y0 is read, and the seven SDE evaluations
// (the f program at three (t, y), the g program at four) alternate with the unfused step's own stage ops.  y0 and y1
// are the only tensors the step moves, against 22 reads and 6 writes of the unfused step (41 with f and g).
//
// At the last update ten quads are live (y0, f0..f2, g0..g3, W, U).  In fp64 that is 80 registers before the
// interpreter's own, so there f0..f2 and g0..g2 wait in the shared-memory register file, in the kPwSrkStash slots
// past the program's registers; in fp32 they stay in registers.
constexpr int kPwSrkStash = TSDE_PW_MAX_REGS - TSDE_PW_SRK_MAX_REGS;  // six: f0..f2, g0..g2

template <typename T>
struct PwSrkP {
  PwP<T> base;    // y0, y1, the quad mapping; base.t0 unused
  const T* t[4];  // t_0, t_1, t_q, t_h
  SrkDiagStage1Op<T> s1;
  SrkDiagStage2Op<T> s2;
  SrkDiagStage3Op<T> s3;
  SrkDiagFinalOp<T> fin;
};

template <typename T>
struct PwSrkStash {
  static constexpr bool kShared = sizeof(T) == 8;
  T r[kShared ? 1 : kPwSrkStash][4];
  int slot0;  // first shared-memory register past the program's
  __device__ __forceinline__ void put(void* regs, int k, const T (&x)[4]) {
    if constexpr (kShared) {
      pw_sstore(regs, slot0 + k, x);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) r[k][j] = x[j];
    }
  }
  __device__ __forceinline__ void get(const void* regs, int k, T (&x)[4]) const {
    if constexpr (kShared) {
      pw_sload(regs, slot0 + k, x);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = r[k][j];
    }
  }
};

// f (program [0, n_fg), result f_src) or g (program [n_fg, n_instr), result g_src) at (t, y)
template <typename T>
__device__ __forceinline__ void pw_srk_eval(const tsde_pointwise& pg, const PwSrkP<T>& p, PwQuad<T>& c, void* regs,
                                            bool g, const T* t, const T (&y)[4], T (&out)[4]) {
  PwP<T> at = p.base;
  at.t0 = t;
#pragma unroll
  for (int j = 0; j < 4; ++j) c.y[j] = y[j];
  pw_run(pg, at, c, regs, g ? pg.n_fg : 0, g ? pg.n_instr : pg.n_fg);
  pw_fetch(pg, at, c, regs, g ? pg.g_src : pg.f_src, out);
}

template <typename T, int SRC>
__global__ void __launch_bounds__(kThreads)
pw_srk_kernel(const __grid_constant__ tsde_pointwise pg, const PwSrkP<T> p, const NoiseP<T> nz) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  const PwP<T>& b = p.base;
  const int64_t Q = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  int64_t row, q;
  if (b.qshift >= 0) {
    row = Q >> b.qshift;
    q = Q & ((1ll << b.qshift) - 1);
  } else if (b.small) {
    const uint32_t r32 = rowdiv_row((uint32_t)Q, b.qmagic);
    row = r32;
    q = (int64_t)rowdiv_quad((uint32_t)Q, r32, (uint32_t)b.qpr);
  } else {
    row = Q / b.qpr;
    q = Q - row * b.qpr;
  }
  PwQuad<T> c;
  c.chan = 4 * q;
  c.base = row * b.d + c.chan;
  const int64_t rem = b.d - c.chan;
  c.nvalid = rem < 4 ? (int)rem : 4;
  c.vec = b.vec != 0;
  T w[4], u[4];
  quad_noise<T, SRC, true>(nz, load_key(nz.key), row, q, c.vec, c.nvalid, w, u);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= b.nquads) return;
  T y0[4];
  load_quad(b.y0, c.base, c.vec, c.nvalid, y0);
#pragma unroll
  for (int j = 0; j < 4; ++j) c.go[j] = T(0);
  PwSrkStash<T> st;
  st.slot0 = pg.n_regs;
  enum { F0, F1, F2, G0, G1, G2 };
  T f[4], g[4], h0[4], h1[4], x[4], z[4];
  // s = 0: f0, g0 at (t0, y0); H0_1, H1_1
  pw_srk_eval(pg, p, c, pw_regs, false, p.t[0], y0, f);
  pw_srk_eval(pg, p, c, pw_regs, true, p.t[0], y0, g);
  st.put(pw_regs, F0, f);
  st.put(pw_regs, G0, g);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[2];
    p.s1({y0[j], f[j], g[j]}, w[j], u[j], o);
    h0[j] = o[0];
    h1[j] = o[1];
  }
  // s = 1: f1 at (t0 + dt, H0_1), g1 at (t0 + dt/4, H1_1); H0_2, H1_2
  pw_srk_eval(pg, p, c, pw_regs, false, p.t[1], h0, f);
  pw_srk_eval(pg, p, c, pw_regs, true, p.t[2], h1, g);
  st.put(pw_regs, F1, f);
  st.put(pw_regs, G1, g);
  st.get(pw_regs, F0, x);
  st.get(pw_regs, G0, z);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[2];
    p.s2({y0[j], x[j], z[j], f[j], g[j]}, w[j], u[j], o);
    h0[j] = o[0];
    h1[j] = o[1];
  }
  // s = 2: f2 at (t0 + dt/2, H0_2), g2 at (t0 + dt, H1_2); H1_3
  pw_srk_eval(pg, p, c, pw_regs, false, p.t[3], h0, f);
  pw_srk_eval(pg, p, c, pw_regs, true, p.t[1], h1, g);
  st.put(pw_regs, F2, f);
  st.put(pw_regs, G2, g);
  st.get(pw_regs, G0, x);
  st.get(pw_regs, G1, z);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    p.s3({y0[j], x[j], z[j], f[j], g[j]}, w[j], u[j], o);
    h1[j] = o[0];
  }
  // s = 3: g3 at (t0 + dt/4, H1_3); y1
  pw_srk_eval(pg, p, c, pw_regs, true, p.t[2], h1, g);
  T f0[4], f1[4], f2[4], g0[4], g1[4], g2[4], y1[4];
  st.get(pw_regs, F0, f0);
  st.get(pw_regs, F1, f1);
  st.get(pw_regs, F2, f2);
  st.get(pw_regs, G0, g0);
  st.get(pw_regs, G1, g1);
  st.get(pw_regs, G2, g2);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    p.fin({y0[j], f0[j], f1[j], f2[j], g0[j], g1[j], g2[j], g[j]}, w[j], u[j], o);
    y1[j] = o[0];
  }
  store_quad(b.y1, c.base, c.vec, c.nvalid, y1);
}

// A program the kernel can run as given: instruction, register and operand indices in range, every register
// written before it is read, device operands present (and 16-byte aligned for the vector path).  `two`: the SRK
// layout, an f program [0, n_fg) and a g program [n_fg, n_instr) that each define their own registers.
static bool pw_valid(const tsde_pointwise& pg, bool* vec, bool two = false) {
  if (pg.n_instr < 0 || pg.n_instr > TSDE_PW_MAX_INSTR || pg.n_fg < 0 || pg.n_fg > pg.n_instr ||
      pg.n_regs < 0 || pg.n_regs > TSDE_PW_MAX_REGS || pg.n_operands < 0 || pg.n_operands > TSDE_PW_MAX_OPERANDS)
    return false;
  if (two && pg.n_regs > TSDE_PW_SRK_MAX_REGS) return false;
  for (int k = 0; k < pg.n_operands; ++k) {
    const tsde_pw_operand& o = pg.operand[k];
    if (o.kind < TSDE_PW_IMM || o.kind > TSDE_PW_ROW) return false;
    if (o.kind >= TSDE_PW_SCALAR && !o.ptr) return false;
    if (o.kind >= TSDE_PW_CHANNEL) *vec = *vec && aligned16(o.ptr);
  }
  uint64_t written = 0;  // registers defined so far
  auto source_ok = [&](uint32_t s, bool vjp) {
    if (s == TSDE_PW_SRC_Y) return true;
    if (s == TSDE_PW_SRC_GO) return vjp;
    if (s >= (uint32_t)TSDE_PW_OPERAND(0)) return (int)(s - TSDE_PW_OPERAND(0)) < pg.n_operands;
    return (int)s < pg.n_regs && ((written >> s) & 1u);
  };
  for (int i = 0; i <= pg.n_instr; ++i) {
    if (i == pg.n_fg) {
      if (!source_ok(pg.f_src, false) || !(two || source_ok(pg.g_src, false))) return false;
      if (two) written = 0;
    }
    if (i == pg.n_instr) break;
    const tsde_pw_instr& in = pg.instr[i];
    const bool vjp = !two && i >= pg.n_fg;
    if (in.op > TSDE_PW_SQRT || (int)in.dst >= pg.n_regs || !source_ok(in.a, vjp)) return false;
    if (in.op != TSDE_PW_NEG && in.op != TSDE_PW_SQRT && !source_ok(in.b, vjp)) return false;
    written |= 1ull << in.dst;
  }
  return two ? source_ok(pg.g_src, false) : source_ok(pg.gdg_src, true);
}

// The quad mapping of a pointwise step over (rows, d) and its noise; TSDE_EINVAL for a launch it cannot serve.
template <typename T>
static int pw_prepare(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog, const void* y0,
                      void* y1, bool two, PwP<T>& p, NoiseP<T>& np) {
  if (!nz || nz->source != TSDE_SRC_COUNTER || nz->flags || !prog || !y0 || !y1) return TSDE_EINVAL;
  bool vec = L->d % 4 == 0 && aligned16(y0) && aligned16(y1);
  if (!pw_valid(*prog, &vec, two)) return TSDE_EINVAL;
  if (int e = fill_noise<T>(L, nz, false, np)) return e;
  p = PwP<T>{};
  p.y0 = static_cast<const T*>(y0);
  p.y1 = static_cast<T*>(y1);
  p.d = L->d;
  p.qpr = (L->d + 3) / 4;
  p.nquads = L->rows * p.qpr;
  p.qshift = -1;
  if ((p.qpr & (p.qpr - 1)) == 0) {
    int sh = 0;
    while ((1ll << sh) < p.qpr) ++sh;
    p.qshift = sh;
  }
  p.small = p.nquads < (1ll << 31) ? 1 : 0;
  p.qmagic = p.qshift < 0 ? rowdiv_magic((uint64_t)p.qpr) : 0;
  p.vec = vec ? 1 : 0;
  return 0;
}

}  // namespace tsde

using namespace tsde;

TSDE_EXPORT int tsde_step_milstein_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                             const void* y0, const void* t0, double dt, int32_t ito, void* y1) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    using T = decltype(t);
    if (!t0) return TSDE_EINVAL;
    PwP<T> p;
    NoiseP<T> np;
    if (int e = pw_prepare<T>(L, nz, prog, y0, y1, false, p, np)) return e;
    p.t0 = static_cast<const T*>(t0);
    p.dt = (T)dt;
    p.ito = ito;
    const size_t smem = (size_t)prog->n_regs * kThreads * 4 * sizeof(T);
    auto kernel = np.n_cells > 1 ? pw_milstein_kernel<T, kSrcCounterMulti> : pw_milstein_kernel<T, TSDE_SRC_COUNTER>;
    if (resident_ctas(reinterpret_cast<const void*>(kernel), kThreads, smem) < 1) return TSDE_EINVAL;
    const int64_t grid = (p.nquads + kThreads - 1) / kThreads;
    const int e = launch_kernel(kernel, grid, kThreads, smem, reinterpret_cast<cudaStream_t>(L->stream), true, *prog,
                                p, np);
    if (e == 0) g_launches[TSDE_KERNEL_PW_MILSTEIN].fetch_add(1, std::memory_order_relaxed);
    return e;
  });
}

TSDE_EXPORT int tsde_step_srk_diag_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                             const void* y0, const void* t_0, const void* t_1, const void* t_q,
                                             const void* t_h, double dt, double rdt, double sqrt_dt, double three_dt,
                                             void* y1) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    using T = decltype(t);
    if (!t_0 || !t_1 || !t_q || !t_h) return TSDE_EINVAL;
    PwSrkP<T> p;
    NoiseP<T> np;
    if (int e = pw_prepare<T>(L, nz, prog, y0, y1, true, p.base, np)) return e;
    const void* times[4] = {t_0, t_1, t_q, t_h};
    for (int i = 0; i < 4; ++i) p.t[i] = static_cast<const T*>(times[i]);
    // the coefficients of tsde_srk_diag_stage1/2/3 and tsde_step_srk_diag
    p.s1 = SrkDiagStage1Op<T>{(T)dt, (T)sqrt_dt};
    p.s2 = SrkDiagStage2Op<T>{(T)dt, (T)rdt, (T)sqrt_dt};
    p.s3 = SrkDiagStage3Op<T>{(T)dt, (T)sqrt_dt};
    p.fin = make_srk_final<T>(dt, rdt, sqrt_dt, three_dt);
    const int slots = prog->n_regs + (PwSrkStash<T>::kShared ? kPwSrkStash : 0);
    const size_t smem = (size_t)slots * kThreads * 4 * sizeof(T);
    auto kernel = np.n_cells > 1 ? pw_srk_kernel<T, kSrcCounterMulti> : pw_srk_kernel<T, TSDE_SRC_COUNTER>;
    if (resident_ctas(reinterpret_cast<const void*>(kernel), kThreads, smem) < 1) return TSDE_EINVAL;
    const int64_t grid = (p.base.nquads + kThreads - 1) / kThreads;
    const int e = launch_kernel(kernel, grid, kThreads, smem, reinterpret_cast<cudaStream_t>(L->stream), true, *prog,
                                p, np);
    if (e == 0) g_launches[TSDE_KERNEL_PW_SRK].fetch_add(1, std::memory_order_relaxed);
    return e;
  });
}

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
