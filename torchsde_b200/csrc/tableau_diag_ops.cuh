// The element-wise ops of the diagonal-noise step tableaus.  Each op restates one `.step` body of
// torchsde/_core/methods/*.py with the reference's evaluation order (one IEEE rounding per ATen op, no FMA: every
// translation unit that includes this header is compiled with -fmad=false).  tableau_diag.cu launches them one kernel
// per op; pointwise.cu runs the Milstein and SRK ones inside its whole-step kernels, so both compute the same bits.
#pragma once

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

// (MilsteinSeedOp, MilsteinOp: pw_device.cuh, which the run-time compiled Milstein kernels include too)

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

}  // namespace tsde
