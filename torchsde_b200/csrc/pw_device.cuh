// Device code that both the library's nvcc build and its run-time compiler (NVRTC, pointwise.cu) compile: the
// quad-per-thread layout, the Brownian increment of one quad, the Milstein step's two ops, and the chunked Milstein
// step loop of an element-wise program compiled into its own kernel.  Nothing here includes a host header: NVRTC has
// none, so the library hands it this file, philox.cuh, rowdiv.cuh, the public header and a <stdint.h> of its own
// (build() embeds them into the library as strings; the library never reads csrc/ at run time).
#pragma once
#include <stdint.h>

#include "../../include/torchsde_b200.h"
#include "philox.cuh"
#include "rowdiv.cuh"

namespace tsde {

constexpr int kThreads = 256;

template <typename T>
struct NoiseP {
  const T* w;         // MEMORY
  const T* u;         // MEMORY
  const void* key;    // COUNTER
  uint64_t cell_id;
  int64_t row_offset;
  int32_t n_cells;
  int32_t bcast;      // noise has a single channel shared by all d (scalar noise, squeezed g)
  double h;           // uniform cell length
  const double* cell_h;  // device, or nullptr
  double h_total;     // tb - ta of the whole query (for U)
  int64_t m;          // channels of the noise tensor
  T sqrt_h;           // (T)sqrt(h), (T)sqrt(h/12), (T)h_total: host-rounded once (single-cell path)
  T sqrt_h12;
  T ht;
};

// ---- vector load / store helpers ---------------------------------------------------------
__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const double* p, double (&v)[4]) {
  const double2 a = *reinterpret_cast<const double2*>(p);
  const double2 b = *reinterpret_cast<const double2*>(p + 2);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4(double* p, const double (&v)[4]) {
  *reinterpret_cast<double2*>(p) = make_double2(v[0], v[1]);
  *reinterpret_cast<double2*>(p + 2) = make_double2(v[2], v[3]);
}

template <typename T>
__device__ __forceinline__ void load_quad(const T* p, int64_t base, bool vec, int nvalid,
                                          T (&v)[4]) {
  if (vec) {
    ld4(p + base, v);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < nvalid ? p[base + j] : T(0);
  }
}
template <typename T>
__device__ __forceinline__ void store_quad(T* p, int64_t base, bool vec, int nvalid,
                                           const T (&v)[4]) {
  if (vec) {
    st4(p + base, v);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < nvalid) p[base + j] = v[j];
  }
}

// ---- Brownian increment of one quad --------------------------------------------------------
// Counter mode: merge of n_cells primary cells, left to right, with the reference's
// aggregation rule (brownian_interval.py:643-672):
//     H <- ( len_i (H_i + W/2) + (start_i - ta)(H - W_i/2) ) / (end_i - ta) ;  W <- W + W_i
// Lengths are host doubles rounded once to T (python-float * tensor semantics).
constexpr int kSrcCounterMulti = 3;  // internal: COUNTER source merging several primary cells

template <typename T, bool WANT_U, bool MULTI = true>
__device__ __forceinline__ void counter_noise(const NoiseP<T>& nz, Key key, uint32_t row,
                                              uint32_t q, T (&w)[4], T (&u)[4]) {
  T hh[4];
  if (!MULTI || nz.n_cells == 1) {
    // the solver's own grid: one primary cell per step, scales rounded once on the host
    T n[4];
    normal4(key, nz.cell_id, STREAM_W, row, q, n);
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = n[j] * nz.sqrt_h;
    if (WANT_U) {
      normal4(key, nz.cell_id, STREAM_H, row, q, n);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        hh[j] = n[j] * nz.sqrt_h12;
        u[j] = nz.ht * (T(0.5) * w[j] + hh[j]);  // _H_to_U :102-103
      }
    }
    return;
  }
  if (!MULTI) return;  // (unreachable; lets the compiler drop the merge loop from single-cell kernels)
  double len0 = nz.cell_h ? nz.cell_h[0] : nz.h;
  {
    T n[4];
    normal4(key, nz.cell_id, STREAM_W, row, q, n);
    const T s = (T)sqrt(len0);
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = n[j] * s;
    if (WANT_U) {
      normal4(key, nz.cell_id, STREAM_H, row, q, n);
      const T s12 = (T)sqrt(len0 / 12.0);
#pragma unroll
      for (int j = 0; j < 4; ++j) hh[j] = n[j] * s12;
    }
  }
  double elapsed = len0;  // start_i - ta
  for (int c = 1; c < nz.n_cells; ++c) {
    const double len = nz.cell_h ? nz.cell_h[c] : nz.h;
    T n[4], wi[4];
    normal4(key, nz.cell_id + (uint64_t)c, STREAM_W, row, q, n);
    const T s = (T)sqrt(len);
#pragma unroll
    for (int j = 0; j < 4; ++j) wi[j] = n[j] * s;
    if (WANT_U) {
      normal4(key, nz.cell_id + (uint64_t)c, STREAM_H, row, q, n);
      const T s12 = (T)sqrt(len / 12.0);
      const T tl = (T)len, te = (T)elapsed, tt = (T)(elapsed + len);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const T hi = n[j] * s12;
        const T term1 = tl * (hi + T(0.5) * w[j]);
        const T term2 = te * (hh[j] - T(0.5) * wi[j]);
        hh[j] = (term1 + term2) / tt;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = w[j] + wi[j];
    elapsed += len;
  }
  if (WANT_U) {
    const T ht = (T)nz.h_total;
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = ht * (T(0.5) * w[j] + hh[j]);  // _H_to_U :102-103
  }
}

template <typename T, int SRC, bool WANT_U>
__device__ __forceinline__ void quad_noise(const NoiseP<T>& nz, Key key, int64_t row, int64_t q,
                                           bool vec, int nvalid, T (&w)[4], T (&u)[4]) {
  if (SRC == TSDE_SRC_UNIT) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { w[j] = T(1); u[j] = T(0); }
  } else if (SRC == TSDE_SRC_MEMORY) {
    if (nz.bcast) {
      const T a = nz.w[row];
      const T b = WANT_U ? nz.u[row] : T(0);
#pragma unroll
      for (int j = 0; j < 4; ++j) { w[j] = a; u[j] = b; }
    } else {
      const int64_t base = row * nz.m + 4 * q;
      load_quad(nz.w, base, vec, nvalid, w);
      if (WANT_U) load_quad(nz.u, base, vec, nvalid, u);
    }
  } else {
    constexpr bool MULTI = SRC == kSrcCounterMulti;
    const uint32_t grow = (uint32_t)(row + nz.row_offset);
    if (nz.bcast) {
      T w4[4], u4[4];
      counter_noise<T, WANT_U, MULTI>(nz, key, grow, 0u, w4, u4);
#pragma unroll
      for (int j = 0; j < 4; ++j) { w[j] = w4[0]; u[j] = WANT_U ? u4[0] : T(0); }
    } else {
      counter_noise<T, WANT_U, MULTI>(nz, key, grow, (uint32_t)q, w, u);
    }
  }
}

// ---- the Milstein step's ops (tableau_diag_ops.cuh holds the others) --------------------------
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

// ---- the whole-step kernels' parameters (pointwise.cu) --------------------------------------
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

template <typename T>
struct PwOperand {
  const T* ptr;  // SCALAR, CHANNEL, ROW; null for IMM
  T imm;
};

struct PwQuad {  // where this thread's quad lives
  int64_t base, chan;
  int nvalid;
  bool vec;
};

// The flat index Q of this thread's quad (past the last quad when Q >= p.nquads), the row and quad of the row, and `c`.
template <typename T>
__device__ __forceinline__ void pw_locate(const PwP<T>& p, PwQuad& c, int64_t& Q, int64_t& row, int64_t& q) {
  Q = (int64_t)blockIdx.x * kThreads + threadIdx.x;
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
  c.chan = 4 * q;
  c.base = row * p.d + c.chan;
  const int64_t rem = p.d - c.chan;
  c.nvalid = rem < 4 ? (int)rem : 4;
  c.vec = p.vec != 0;
}

// A chunk of consecutive steps (tsde_solve_milstein_pointwise, tsde_solve_euler_pointwise, ...): one thread runs up to
// kPwMaxSteps steps of its quad.
constexpr int kPwMaxSteps = TSDE_PW_MAX_STEPS;

template <typename T>
struct PwStep {  // one step of a chunk, as tsde_pw_step with its scalars rounded to T on the host
  uint64_t cell;   // Brownian cell (the kSrcCounterMulti kernel merges nz.n_cells cells from here)
  const T* t0;     // what TSDE_PW_T0 reads during this step
  T* y1;           // destination of this step's y1, or null
  T sqrt_h, dt;    // (T)sqrt(h) of the cell, (T)dt
};
template <typename T>
struct PwSteps {  // by value: a captured launch carries the whole table
  int32_t n;
  PwStep<T> s[kPwMaxSteps];
  // A uniform grid (pw_steps): every step drawn from one Brownian cell, cell s[0].cell + j, stored to
  // s[0].y1 + j y1_stride, run at s[0].t0 + j t0_stride, with s[0]'s sqrt_h and dt; the noise is not broadcast and
  // every quad is whole (p.vec).  pw_milstein_steps runs such a chunk without reading the table step by step.
  int32_t uniform;
  int64_t y1_stride, t0_stride;  // in elements
};

// ---- consecutive Milstein steps of a compiled program ----------------------------------------
// The operands of a compiled program, in the caller's order: IMM values and device pointers are launch parameters,
// so one compiled kernel serves every value and address of its program's structure.
template <typename T>
struct PwOperands {
  PwOperand<T> k[TSDE_PW_MAX_OPERANDS];
};

// One Milstein step of a compiled program on this thread's quad: the program's f / g part runs on y at s.t0,
// MilsteinSeedOp forms go from the increment w, the vjp part runs and MilsteinOp forms y1, which replaces y.
template <typename T, typename Prog>
__device__ __forceinline__ void pw_milstein_step(Prog& prog, const PwOperands<T>& ops, const PwQuad& c,
                                                 const PwStep<T>& s, int32_t ito, const T (&w)[4], T (&y)[4]) {
  T f[4], g[4], go[4], gdg[4];
  prog.fg(ops, c, s, y, f, g);
  const MilsteinSeedOp<T> seed{s.dt, ito};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    T o[1];
    seed({g[i]}, w[i], T(0), o);
    go[i] = o[0];
  }
  prog.vjp(ops, c, s, y, go, gdg);
  const MilsteinOp<T> step{s.dt};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    T o[1];
    step({y[i], f[i], g[i], gdg[i]}, w[i], T(0), o);
    y[i] = o[0];
  }
}

// A program compiled as relocatable device code calls its transcendental ops out of line (pointwise.cu, kPwHelpers),
// and every register live across a call is saved to the stack around it: a second step loop, with the Philox
// schedule live across the calls, would grow its kernels' call frame.  Its chunks all run through the step table.
#ifdef __CUDACC_RDC__
constexpr bool kPwCalls = true;
#else
constexpr bool kPwCalls = false;
#endif

// pw_milstein_steps on a uniform grid (st.uniform), with `ito` fixed: the launch constants are read once, and the loop
// has one back-edge, no per-step branch and no indexed read of the step table.  Step j's PwStep is built in registers
// (the program reads it as it reads a table entry) and its increment is drawn as counter_noise draws it; in fp32 on a
// Philox whose key schedule and the counter words fixed for the thread are formed once (philox_xy).
template <typename T, typename Prog, int ITO>
__device__ __forceinline__ void pw_milstein_uniform(const PwOperands<T>& ops, const PwP<T>& p, const NoiseP<T>& nz,
                                                    const PwSteps<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p, c, Q, row, q);
  c.vec = true;
  const Key key = load_key(nz.key);
  const uint32_t grow = (uint32_t)(row + nz.row_offset);
  const PhiloxXY ph = philox_xy((uint32_t)q | (STREAM_W << 24), grow, key.lo, key.hi);
  PwStep<T> s = st.s[0];
  T w[4], y[4];
  auto draw = [&]() {
    T n[4];
    if constexpr (sizeof(T) == 4)
      box_muller4(philox_zw(ph, (uint32_t)s.cell, (uint32_t)(s.cell >> 32)), n);
    else  // (fp64 draws two counters per quad, which differ in word x)
      normal4(key, s.cell, STREAM_W, grow, (uint32_t)q, n);
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i] = n[i] * s.sqrt_h;
  };
  draw();  // the first increment is drawn while the previous kernel drains
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.nquads) return;
  Prog prog;
  ld4(p.y0 + c.base, y);
  prog.load(ops, c);
  T* y1 = s.y1 + c.base;
  for (int j = 1;; ++j) {
    pw_milstein_step<T>(prog, ops, c, s, ITO, w, y);
    st4(y1, y);
    if (j == st.n) break;
    ++s.cell;
    s.t0 += st.t0_stride;
    y1 += st.y1_stride;
    draw();
  }
}

// Per step: pw_milstein_step on the state the step before left in registers.  A quad's trajectory depends on nothing but its own state (element-wise SDE, diagonal noise), so one thread runs the
// whole chunk: y0 is read once, y stays in registers from one step to the next and is stored only where the step table
// gives it a destination (an output row, the chunk's last state).  The unfused step moves 13 tensors; a chunk moves one
// read and the stores it is asked for.
//
// `Prog` is the program, generated by the library as straight-line code (pw_milstein_source in pointwise.cu):
//   load(ops, c)                    its operands, after the dependency wait (CHANNEL / ROW quads it keeps in registers)
//   fg(ops, c, s, y, f, g)          instructions [0, n_fg) at (s.t0, y), and the f and g results
//   vjp(ops, c, s, y, go, gdg)      instructions [n_fg, n_instr), and the gdg result
// Its registers are members: values of the f / g part that the vjp part reads carry over.
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_milstein_steps(const PwOperands<T>& ops, const PwP<T>& p, const NoiseP<T>& nz,
                                                  const PwSteps<T>& st) {
  if (SRC == TSDE_SRC_COUNTER && !kPwCalls && st.uniform) {
    if (p.ito)
      pw_milstein_uniform<T, Prog, 1>(ops, p, nz, st);
    else
      pw_milstein_uniform<T, Prog, 0>(ops, p, nz, st);
    return;
  }
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p, c, Q, row, q);
  const Key key = load_key(nz.key);
  Prog prog;
  T y[4];
  for (int j = 0; j < st.n; ++j) {
    const PwStep<T>& s = st.s[j];
    T w[4], u[4];
    NoiseP<T> z = nz;  // this step's cell
    z.cell_id = s.cell;
    z.sqrt_h = s.sqrt_h;
    quad_noise<T, SRC, false>(z, key, row, q, c.vec, c.nvalid, w, u);
    if (j == 0) {  // the first increment is drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      if (Q >= p.nquads) return;
      load_quad(p.y0, c.base, c.vec, c.nvalid, y);
      prog.load(ops, c);
    }
    pw_milstein_step<T>(prog, ops, c, s, p.ito, w, y);
    if (s.y1) store_quad(s.y1, c.base, c.vec, c.nvalid, y);
  }
}

// ---- an adaptive solve's step-doubling proposal (tsde_adaptive_proposal_pointwise) -----------------------------------
// Three sub-steps of one method on increments read from memory: the full step from y0, the first half step from y0
// and the second half step from the midpoint state, which stays in registers.  Only the full step's and the second
// half step's results are stored.
template <typename T>
struct PwSub {
  PwStep<T> s;     // s.t0 (the time the program runs at) and s.dt; cell, sqrt_h and y1 unused
  const T* w;      // (rows, d) increment
  const T* u;      // (rows, d) space-time Levy area (SRK), or null
  const T* t[4];   // the sub-step's other times (SRK's stage times; the predictor-corrector's t_p in t[1])
  T half_dt;       // midpoint's predictor scalar
};
template <typename T>
struct PwSubs {  // by value: the three sub-steps, in order full, first half, second half
  PwSub<T> sub[3];
};

// The compiled Milstein variant: y_full and y_next as pw_milstein_step gives them from the increments sub[k].w.
template <typename T, typename Prog>
__device__ __forceinline__ void pw_milstein_proposal(const PwOperands<T>& ops, const PwP<T>& p, T* y_next,
                                                     const PwSubs<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p, c, Q, row, q);
  // the increments are the Brownian queries that precede the launch: everything is read after the wait
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.nquads) return;
  Prog prog;
  T y0[4], y[4], w[4];
  load_quad(p.y0, c.base, c.vec, c.nvalid, y0);
  prog.load(ops, c);
#pragma unroll
  for (int i = 0; i < 4; ++i) y[i] = y0[i];
  load_quad(st.sub[0].w, c.base, c.vec, c.nvalid, w);
  pw_milstein_step<T>(prog, ops, c, st.sub[0].s, p.ito, w, y);
  store_quad(p.y1, c.base, c.vec, c.nvalid, y);
  load_quad(st.sub[1].w, c.base, c.vec, c.nvalid, w);
  pw_milstein_step<T>(prog, ops, c, st.sub[1].s, p.ito, w, y0);
  load_quad(st.sub[2].w, c.base, c.vec, c.nvalid, w);
  pw_milstein_step<T>(prog, ops, c, st.sub[2].s, p.ito, w, y0);
  store_quad(y_next, c.base, c.vec, c.nvalid, y0);
}

// ---- general-noise tableau ops that the element-wise general kernels share with tableau_general.cu -----------------
// (the Op interface of tableau_general.cu: gval, weight, combine)
// y1 = y0 + f*dt + g.dW                                                         methods/euler.py:36
template <typename T>
struct GEulerOp {
  static constexpr int NE = 2, NG = 1, NP = 1, NO = 1;
  static constexpr bool WANT_U = false;
  T dt;
  __device__ __forceinline__ T gval(int, const T (&g)[1]) const { return g[0]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[2], const T (&gp)[1], T (&o)[1]) const {
    o[0] = (e[0] + e[1] * dt) + gp[0];
  }
};
// y' = y0 + half_dt*f + 0.5*(g.dW)                                               methods/midpoint.py:38
template <typename T>
struct GMidpointPredictOp {
  static constexpr int NE = 2, NG = 1, NP = 1, NO = 1;
  static constexpr bool WANT_U = false;
  T half_dt;
  __device__ __forceinline__ T gval(int, const T (&g)[1]) const { return g[0]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[2], const T (&gp)[1], T (&o)[1]) const {
    o[0] = (e[0] + half_dt * e[1]) + T(0.5) * gp[0];
  }
};
// SRA1 stage: H0_1 = y0 + (3/4 f0) dt + gA.((3/2 U) rdt)             methods/srk.py:100-105, sra1.py:24-36
template <typename T>
struct GSraStageOp {
  static constexpr int NE = 2, NG = 1, NP = 1, NO = 1;
  static constexpr bool WANT_U = true;
  T dt, rdt;
  __device__ __forceinline__ T gval(int, const T (&g)[1]) const { return g[0]; }
  __device__ __forceinline__ T weight(int, T, T u) const { return (T(1.5) * u) * rdt; }
  __device__ __forceinline__ void combine(const T (&e)[2], const T (&gp)[1], T (&o)[1]) const {
    o[0] = (e[0] + (T(0.75) * e[1]) * dt) + gp[0];
  }
};
// SRA1 final: y1 = y0 + (1/3 f0) dt + gA.(W + (-U) rdt) + (2/3 f1) dt + gB.(0*W + U rdt)   srk.py:107-110
template <typename T>
struct GSraFinalOp {
  static constexpr int NE = 3, NG = 2, NP = 2, NO = 1;
  static constexpr bool WANT_U = true;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: the g tiles are dead afterwards
  T dt, rdt, third, two_thirds;
  __device__ __forceinline__ T gval(int p, const T (&g)[2]) const { return g[p]; }
  __device__ __forceinline__ T weight(int p, T w, T u) const {
    return p == 0 ? (T(1) * w + (T(-1) * u) * rdt) : (T(0) * w + (T(1) * u) * rdt);
  }
  __device__ __forceinline__ void combine(const T (&e)[3], const T (&gp)[2], T (&o)[1]) const {
    T y1 = (e[0] + (third * e[1]) * dt) + gp[0];
    y1 = (y1 + (two_thirds * e[2]) * dt) + gp[1];
    o[0] = y1;
  }
};
// y' = y0 + g.dW                                                                 methods/euler_heun.py:36
template <typename T>
struct GEulerHeunPredictOp {
  static constexpr int NE = 1, NG = 1, NP = 1, NO = 1;
  static constexpr bool WANT_U = false;
  __device__ __forceinline__ T gval(int, const T (&g)[1]) const { return g[0]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[1], const T (&gp)[1], T (&o)[1]) const {
    o[0] = e[0] + gp[0];
  }
};
// y1 = y0 + dt*f + (g.dW + g'.dW)*0.5                                            methods/euler_heun.py:40
template <typename T>
struct GEulerHeunOp {
  static constexpr int NE = 2, NG = 2, NP = 2, NO = 1;
  static constexpr bool WANT_U = false;
  static constexpr bool STREAM_INPUTS = true;  // last kernel of the step: the g tiles are dead afterwards
  T dt;
  __device__ __forceinline__ T gval(int p, const T (&g)[2]) const { return g[p]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[2], const T (&gp)[2], T (&o)[1]) const {
    o[0] = (e[0] + dt * e[1]) + (gp[0] + gp[1]) * T(0.5);
  }
};
// z1 = 2*y0 - z0 + f0*dt + g0.dW                                                 reversible_heun.py:69
// sign = -1 gives the adjoint's reconstruction z1 = 2*y0 - z0 - f0*dt - g0.dW    reversible_heun.py:109
template <typename T>
struct GRevHeunZOp {
  static constexpr int NE = 3, NG = 1, NP = 1, NO = 1;
  static constexpr bool WANT_U = false;
  T dt;
  int backward;
  __device__ __forceinline__ T gval(int, const T (&g)[1]) const { return g[0]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return w; }
  __device__ __forceinline__ void combine(const T (&e)[3], const T (&gp)[1], T (&o)[1]) const {
    const T a = T(2) * e[0] - e[1];
    o[0] = backward ? ((a - e[2] * dt) - gp[0]) : ((a + e[2] * dt) + gp[0]);
  }
};
// y1 = y0 + (f0+f1)*half_dt + (g0+g1).(0.5*dW)                                   reversible_heun.py:71
// backward: y1 = y0 - (f0+f1)*half_dt - (g0+g1).half_dW                          reversible_heun.py:134-135
template <typename T>
struct GRevHeunOp {
  static constexpr int NE = 3, NG = 2, NP = 1, NO = 1;
  static constexpr bool WANT_U = false;
  T half_dt;
  int backward;
  __device__ __forceinline__ T gval(int, const T (&g)[2]) const { return g[0] + g[1]; }
  __device__ __forceinline__ T weight(int, T w, T) const { return T(0.5) * w; }
  __device__ __forceinline__ void combine(const T (&e)[3], const T (&gp)[1], T (&o)[1]) const {
    const T fd = (e[1] + e[2]) * half_dt;
    o[0] = backward ? ((e[0] - fd) - gp[0]) : ((e[0] + fd) + gp[0]);
  }
};

// ---- general / additive noise with an element-wise f and g (tsde_solve_euler_general_pointwise, ...) ---------------
// One thread per (row, quad of d), as above.  The thread draws all m increments of its row (MQ channel quads on the
// counters of the general-noise kernels; the d/4 threads of a row draw the same ones) and never forms g in memory:
// `Prog` (generated by pw_general_source in pointwise.cu) evaluates g_ij channel by channel in registers and contracts
// it with the increments in the order of the unfused launch's route (gen_route), so that its g.dW is the unfused one:
//   load(ops, c)                  the operands kept in registers, after the dependency wait
//   f(ops, c, t, y, f)            the f program at (*t, y)
//   gp(ops, c, t, y, w, gp)       the g program at (*t, y), contracted with w[0, 4 MQ)
// and, in the reversible-Heun unit, whose g values stay in registers (gs[j][k]: lane j, channel k < M):
//   dot(op, gs, w, gp)                  op.gval(0, {gs_k}) contracted with w
//   gstep(ops, c, t, y, op, w, gs, gp)  the g program at (*t, y), g1_k; op.gval(0, {gs_k, g1_k}) contracted with w,
//                                       and gs_k <- g1_k

// The increments of this thread's row: channel k in w[k], and with WANT_U its U in u[k]
template <typename T, int SRC, int MQ, bool WANT_U>
__device__ __forceinline__ void pw_general_noise(const NoiseP<T>& nz, Key key, int64_t row, T (&w)[4 * MQ],
                                                 T (&u)[4 * MQ]) {
  const uint32_t grow = (uint32_t)(row + nz.row_offset);
#pragma unroll
  for (int q = 0; q < MQ; ++q) {
    T w4[4], u4[4];
    counter_noise<T, WANT_U, SRC == kSrcCounterMulti>(nz, key, grow, (uint32_t)q, w4, u4);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      w[4 * q + j] = w4[j];
      if (WANT_U) u[4 * q + j] = u4[j];
    }
  }
}
template <typename T, int SRC, int MQ>
__device__ __forceinline__ void pw_general_noise(const NoiseP<T>& nz, Key key, int64_t row, T (&w)[4 * MQ]) {
  T u[4 * MQ];
  pw_general_noise<T, SRC, MQ, false>(nz, key, row, w, u);
}

// Consecutive Euler steps, as pw_milstein_steps: y1 = GEulerOp{dt} on (y, f, g.dW)
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_euler_steps(const PwOperands<T>& ops, const PwP<T>& p, const NoiseP<T>& nz,
                                                       const PwSteps<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p, c, Q, row, q);
  const Key key = load_key(nz.key);
  Prog prog;
  T y[4];
  for (int j = 0; j < st.n; ++j) {
    const PwStep<T>& s = st.s[j];
    NoiseP<T> z = nz;  // this step's cell
    z.cell_id = s.cell;
    z.sqrt_h = s.sqrt_h;
    T w[4 * Prog::MQ];
    pw_general_noise<T, SRC, Prog::MQ>(z, key, row, w);
    if (j == 0) {  // the first increments are drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      if (Q >= p.nquads) return;
      load_quad(p.y0, c.base, c.vec, c.nvalid, y);
      prog.load(ops, c);
    }
    T f[4], gp[4];
    prog.f(ops, c, s.t0, y, f);
    prog.gp(ops, c, s.t0, y, w, gp);
    const GEulerOp<T> op{s.dt};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const T e[2] = {y[i], f[i]}, g1[1] = {gp[i]};
      T o[1];
      op.combine(e, g1, o);
      y[i] = o[0];
    }
    if (s.y1) store_quad(s.y1, c.base, c.vec, c.nvalid, y);
  }
}

template <typename T>
struct PwGeneralMidP {
  PwP<T> base;   // y0, y1, the quad mapping, t0 and dt
  const T* t_p;  // the time of the second evaluation, t0 + half_dt
  T half_dt;
};

// One midpoint step: y' = GMidpointPredictOp{half_dt} on (y0, f, g.dW) at (t0, y0); y1 = GEulerOp{dt} on
// (y0, f', g'.dW) at (t_p, y')
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_midpoint(const PwOperands<T>& ops, const PwGeneralMidP<T>& p,
                                                    const NoiseP<T>& nz) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  T w[4 * Prog::MQ];
  pw_general_noise<T, SRC, Prog::MQ>(nz, load_key(nz.key), row, w);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.base.nquads) return;
  Prog prog;
  T y0[4], yp[4], f[4], gp[4];
  load_quad(p.base.y0, c.base, c.vec, c.nvalid, y0);
  prog.load(ops, c);
  prog.f(ops, c, p.base.t0, y0, f);
  prog.gp(ops, c, p.base.t0, y0, w, gp);
  const GMidpointPredictOp<T> predict{p.half_dt};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[2] = {y0[i], f[i]}, g1[1] = {gp[i]};
    T o[1];
    predict.combine(e, g1, o);
    yp[i] = o[0];
  }
  prog.f(ops, c, p.t_p, yp, f);
  prog.gp(ops, c, p.t_p, yp, w, gp);
  const GEulerOp<T> step{p.base.dt};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[2] = {y0[i], f[i]}, g1[1] = {gp[i]};
    T o[1];
    step.combine(e, g1, o);
    yp[i] = o[0];
  }
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, yp);
}

template <typename T>
struct PwGeneralSraP {
  PwP<T> base;                // y0, y1, the quad mapping and t0 = t_00, the time of f0 and gB
  const T* t_1;               // the time of gA, t0 + dt
  const T* t_34;              // the time of f1, t0 + 3/4 dt
  GSraStageOp<T> stage;       // as tsde_srk_additive_stage and tsde_step_srk_additive build them
  GSraFinalOp<T> final_op;
};

// One sra1 step (methods/srk.py:90-111): f0 = f(t_00, y0); H0_1 = GSraStageOp on (y0, f0, gA.wS) with gA = g(t_1, y0);
// f1 = f(t_34, H0_1); y1 = GSraFinalOp on (y0, f0, f1, gA.w0, gB.w1) with gB = g(t_00, y0).  Each weight vector is the
// op's weight(p, W_k, U_k) per channel, exactly as the unfused launches form it next to the contraction.
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_sra1(const PwOperands<T>& ops, const PwGeneralSraP<T>& p,
                                                const NoiseP<T>& nz) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  T w[4 * Prog::MQ], u[4 * Prog::MQ];
  pw_general_noise<T, SRC, Prog::MQ, true>(nz, load_key(nz.key), row, w, u);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.base.nquads) return;
  Prog prog;
  T y0[4], f0[4], h[4], ga[4], gb[4], wt[4 * Prog::MQ];
  load_quad(p.base.y0, c.base, c.vec, c.nvalid, y0);
  prog.load(ops, c);
  prog.f(ops, c, p.base.t0, y0, f0);
#pragma unroll
  for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = p.stage.weight(0, w[k], u[k]);
  prog.gp(ops, c, p.t_1, y0, wt, ga);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[2] = {y0[i], f0[i]}, g1[1] = {ga[i]};
    T o[1];
    p.stage.combine(e, g1, o);
    h[i] = o[0];
  }
#pragma unroll
  for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = p.final_op.weight(0, w[k], u[k]);
  prog.gp(ops, c, p.t_1, y0, wt, ga);
#pragma unroll
  for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = p.final_op.weight(1, w[k], u[k]);
  prog.gp(ops, c, p.base.t0, y0, wt, gb);
  T f1[4];
  prog.f(ops, c, p.t_34, h, f1);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[3] = {y0[i], f0[i], f1[i]}, g2[2] = {ga[i], gb[i]};
    T o[1];
    p.final_op.combine(e, g2, o);
    h[i] = o[0];
  }
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, h);
}

// One Euler-Heun step (methods/euler_heun.py:34-40), with the parameters of a midpoint step (half_dt unused):
// f = f(t0, y0) and g.dW at (t0, y0); y' = GEulerHeunPredictOp on (y0, g.dW); g'.dW at (t_p, y');
// y1 = GEulerHeunOp{dt} on (y0, f, g.dW, g'.dW).  The unfused predict launch and the final one see the same g operand
// (g and g' come from one program: both dense, or both the user's DM block) and stage m increments per row, so their
// routes are one and the predictor's g.dW is the final launch's first product.
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_euler_heun(const PwOperands<T>& ops, const PwGeneralMidP<T>& p,
                                                      const NoiseP<T>& nz) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  T w[4 * Prog::MQ];
  pw_general_noise<T, SRC, Prog::MQ>(nz, load_key(nz.key), row, w);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (Q >= p.base.nquads) return;
  Prog prog;
  T y0[4], yp[4], f[4], gp[4], gq[4];
  load_quad(p.base.y0, c.base, c.vec, c.nvalid, y0);
  prog.load(ops, c);
  prog.f(ops, c, p.base.t0, y0, f);
  prog.gp(ops, c, p.base.t0, y0, w, gp);
  const GEulerHeunPredictOp<T> predict{};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[1] = {y0[i]}, g1[1] = {gp[i]};
    T o[1];
    predict.combine(e, g1, o);
    yp[i] = o[0];
  }
  prog.gp(ops, c, p.t_p, yp, w, gq);
  const GEulerHeunOp<T> step{p.base.dt};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T e[2] = {y0[i], f[i]}, g2[2] = {gp[i], gq[i]};
    T o[1];
    step.combine(e, g2, o);
    yp[i] = o[0];
  }
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, yp);
}

template <typename T>
struct PwGeneralRevHeunP {
  PwP<T> base;            // y0, the quad mapping (base.y1, t0, dt and ito unused: the step table has them)
  const T *z0, *f0, *g0;  // the solver state the chunk starts from: z and f (rows, d), g (rows, d, m)
  T *z1, *f1, *g1;        // and where the chunk leaves it
  int32_t gvec;           // m % 4 == 0 and g0, g1 16-byte aligned: g moves as quads
};

// This thread's values of a (rows, d, m) tensor: lane j's run of M channels at (c.base + j) * M, a padding lane
// reading lane 0's (as Prog's G does)
template <typename T, int M>
__device__ __forceinline__ void pw_load_g(const T* g, const PwQuad& c, bool vec, T (&gs)[4][M]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t base = (c.base + (j < c.nvalid ? j : 0)) * M;
    if (M % 4 == 0 && vec) {
#pragma unroll
      for (int q = 0; q < M / 4; ++q) {
        T v[4];
        ld4(g + base + 4 * q, v);
#pragma unroll
        for (int i = 0; i < 4; ++i) gs[j][4 * q + i] = v[i];
      }
    } else {
#pragma unroll
      for (int k = 0; k < M; ++k) gs[j][k] = g[base + k];
    }
  }
}
template <typename T, int M>
__device__ __forceinline__ void pw_store_g(T* g, const PwQuad& c, bool vec, const T (&gs)[4][M]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j >= c.nvalid) continue;
    const int64_t base = (c.base + j) * M;
    if (M % 4 == 0 && vec) {
#pragma unroll
      for (int q = 0; q < M / 4; ++q) {
        const T v[4] = {gs[j][4 * q], gs[j][4 * q + 1], gs[j][4 * q + 2], gs[j][4 * q + 3]};
        st4(g + base + 4 * q, v);
      }
    } else {
#pragma unroll
      for (int k = 0; k < M; ++k) g[base + k] = gs[j][k];
    }
  }
}

// Consecutive reversible-Heun steps, as pw_general_euler_steps (reversible_heun.py:64-73); st.s[j].t0 is the step's t1:
//   z1 = GRevHeunZOp{dt} on (y, z, f, g.dW);  f1 at (t1, z1);
//   g1 at (t1, z1), channel by channel, contracted as GRevHeunOp's (g + g1) . (0.5 dW) and left in place of g;
//   y1 = GRevHeunOp{T(0.5) * dt} on (y, f, f1, that product);  (y, z, f) <- (y1, z1, f1)
// The solver state (z, f, g) is read once at the chunk's start and stored once at its end, to pointers the chunk does
// not read; each lane's m values of g stay in registers in between.  Both contractions take the weights the unfused
// launches form (the op's weight per channel) and the route of their dense g operands (Prog, pw_general_source).
// With its 4 M values of g, this kernel holds the most registers of the general ones; m = 32 spills (DESIGN §4).
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_reversible_heun_steps(const PwOperands<T>& ops,
                                                                 const PwGeneralRevHeunP<T>& p, const NoiseP<T>& nz,
                                                                 const PwSteps<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  const Key key = load_key(nz.key);
  Prog prog;
  T y[4], z[4], f[4], g[4][Prog::M];
  for (int j = 0; j < st.n; ++j) {
    const PwStep<T>& s = st.s[j];
    NoiseP<T> n = nz;  // this step's cell
    n.cell_id = s.cell;
    n.sqrt_h = s.sqrt_h;
    T w[4 * Prog::MQ], wt[4 * Prog::MQ];
    pw_general_noise<T, SRC, Prog::MQ>(n, key, row, w);
    if (j == 0) {  // the first increments are drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      if (Q >= p.base.nquads) return;
      load_quad(p.base.y0, c.base, c.vec, c.nvalid, y);
      load_quad(p.z0, c.base, c.vec, c.nvalid, z);
      load_quad(p.f0, c.base, c.vec, c.nvalid, f);
      pw_load_g<T, Prog::M>(p.g0, c, p.gvec != 0, g);
      prog.load(ops, c);
    }
    T gp[4], f1[4];
    const GRevHeunZOp<T> zop{s.dt, 0};
#pragma unroll
    for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = zop.weight(0, w[k], T(0));
    prog.dot(zop, g, wt, gp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const T e[3] = {y[i], z[i], f[i]}, g1[1] = {gp[i]};
      T o[1];
      zop.combine(e, g1, o);
      z[i] = o[0];
    }
    prog.f(ops, c, s.t0, z, f1);
    const GRevHeunOp<T> step{T(0.5) * s.dt, 0};
#pragma unroll
    for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = step.weight(0, w[k], T(0));
    prog.gstep(ops, c, s.t0, z, step, wt, g, gp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const T e[3] = {y[i], f[i], f1[i]}, g1[1] = {gp[i]};
      T o[1];
      step.combine(e, g1, o);
      y[i] = o[0];
      f[i] = f1[i];
    }
    if (s.y1) store_quad(s.y1, c.base, c.vec, c.nvalid, y);
  }
  store_quad(p.z1, c.base, c.vec, c.nvalid, z);
  store_quad(p.f1, c.base, c.vec, c.nvalid, f);
  pw_store_g<T, Prog::M>(p.g1, c, p.gvec != 0, g);
}

// ---- the reversible-Heun adjoint's backward sweep (TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN) -----------------------
// The augmented state of a backward step, in the order of the entry point's state_in / state_out
enum { kAdjY = 0, kAdjZ, kAdjF, kAdjG, kAdjAdjY, kAdjAdjF, kAdjAdjG, kAdjAdjZ, kAdjState };

template <typename T>
struct PwAdjStep {  // one backward step, from tsde_pw_step with its scalars rounded to T on the host
  uint64_t cell;    // Brownian cell
  const T* t1;      // forward time of the step's end: f and g run at (t1, z1)
  int64_t out;      // >= 0: the step ends an output interval (y <- ys[out], adj_y <- adj_y + grad_ys[out]); else -1
  T sqrt_h, dt;
};
template <typename T>
struct PwAdjSteps {  // by value: a captured launch carries the whole table
  int32_t n;
  PwAdjStep<T> s[kPwMaxSteps];
};
template <typename T>
struct PwAdjP {
  PwP<T> base;                          // the quad mapping; base.t0 the time of the first step's forward values
  const T* in[kAdjState];               // the state the chunk starts from
  T* out[kAdjState];                    // where it leaves it (no pointer of in[])
  const T *ys, *gys;                    // the output series and its cotangent, (n_out, rows, d)
  int64_t plane;                        // rows * d
  T* part[TSDE_PW_ADJ_MAX_PARAMS];      // each parameter's (rows, d) partial sum of contributions
};

// Consecutive backward steps of AdjointReversibleHeun (reversible_heun.py:98-144) in reversed time, one thread per
// quad, in the order of the unfused sweep (_BackwardEngine._sweep):
//   z1, adj_f_mid, adj_g_mid = AdjRevHeunAOp (y, z, f, g, adj_y, adj_f, adj_g);
//   vjp_z and the contributions = the vjp with seeds (adj_f_mid, adj_g_mid) of the forward values at z;
//   f1, g1 at (t1, z1);  y, adj_y, adj_z, adj_f, adj_g = AdjRevHeunBOp (y, f, f1, g, g1, adj_y, adj_z, vjp_z);
// and, at an output interval's end, y <- ys[out], adj_y <- adj_y + grad_ys[out].  The forward values the vjp
// differentiates are the program's registers: the evaluation at (t1, z1) of one step is the next step's (the unfused
// sweep keeps that graph as `pending`), and the chunk's first step evaluates them at (base.t0, z).  Each contribution
// is summed over the chunk's steps in a register accumulator and added to its partial once, at the end.
// `Prog` (pw_adjoint_source in pointwise.cu):
//   load(ops, c)                                  the operands kept in registers, after the dependency wait
//   fg(ops, c, t, y, f, g)                        instructions [0, n_fg) at (*t, y), and the f and g results
//   vjp(ops, c, t, y, go, go2, vz, acc)           instructions [n_fg, n_instr) with seeds go (f) and go2 (g), vjp_z
//                                                 into vz, each contribution added to acc[k]
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_adjoint_reversible_heun_steps(const PwOperands<T>& ops, const PwAdjP<T>& p,
                                                                 const NoiseP<T>& nz, const PwAdjSteps<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  const Key key = load_key(nz.key);
  Prog prog;
  T x[kAdjState][4], acc[Prog::NP][4];
  const T* tv = p.base.t0;  // the time of the forward values in the program's registers
  for (int j = 0; j < st.n; ++j) {
    const PwAdjStep<T>& s = st.s[j];
    T w[4], u[4];
    NoiseP<T> n = nz;  // this step's cell
    n.cell_id = s.cell;
    n.sqrt_h = s.sqrt_h;
    quad_noise<T, SRC, false>(n, key, row, q, c.vec, c.nvalid, w, u);
    if (j == 0) {  // the first increment is drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      if (Q >= p.base.nquads) return;
#pragma unroll
      for (int k = 0; k < kAdjState; ++k) load_quad(p.in[k], c.base, c.vec, c.nvalid, x[k]);
      prog.load(ops, c);
      T f0[4], g0[4];
      prog.fg(ops, c, tv, x[kAdjZ], f0, g0);
#pragma unroll
      for (int k = 0; k < Prog::NP; ++k)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[k][i] = T(0);
    }
    const T dt = s.dt, half_dt = T(0.5) * dt;
    T z1[4], afm[4], agm[4];
    const AdjRevHeunAOp<T> a{dt, half_dt};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      T o[3];
      a({x[kAdjY][i], x[kAdjZ][i], x[kAdjF][i], x[kAdjG][i], x[kAdjAdjY][i], x[kAdjAdjF][i], x[kAdjAdjG][i]}, w[i],
        T(0), o);
      z1[i] = o[0];
      afm[i] = o[1];
      agm[i] = o[2];
    }
    T vz[4], f1[4], g1[4];
    prog.vjp(ops, c, tv, x[kAdjZ], afm, agm, vz, acc);
    prog.fg(ops, c, s.t1, z1, f1, g1);
    tv = s.t1;
    const AdjRevHeunBOp<T> b{dt, half_dt};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      T o[5];
      b({x[kAdjY][i], x[kAdjF][i], f1[i], x[kAdjG][i], g1[i], x[kAdjAdjY][i], x[kAdjAdjZ][i], vz[i]}, w[i], T(0), o);
      x[kAdjY][i] = o[0];
      x[kAdjAdjY][i] = o[1];
      x[kAdjAdjZ][i] = o[2];
      x[kAdjAdjF][i] = o[3];
      x[kAdjAdjG][i] = o[4];
      x[kAdjZ][i] = z1[i];
      x[kAdjF][i] = f1[i];
      x[kAdjG][i] = g1[i];
    }
    if (s.out >= 0) {  // adjoint.py:114-116
      T gy[4];
      load_quad(p.ys + s.out * p.plane, c.base, c.vec, c.nvalid, x[kAdjY]);
      load_quad(p.gys + s.out * p.plane, c.base, c.vec, c.nvalid, gy);
#pragma unroll
      for (int i = 0; i < 4; ++i) x[kAdjAdjY][i] = x[kAdjAdjY][i] + gy[i];
    }
  }
#pragma unroll
  for (int k = 0; k < kAdjState; ++k) store_quad(p.out[k], c.base, c.vec, c.nvalid, x[k]);
#pragma unroll
  for (int k = 0; k < Prog::NP; ++k) {
    if (!p.part[k]) continue;  // (NP is 1 for a program without parameters)
    T v[4];
    load_quad(p.part[k], c.base, c.vec, c.nvalid, v);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = v[i] + acc[k][i];
    store_quad(p.part[k], c.base, c.vec, c.nvalid, v);
  }
}

// Consecutive backward steps of a general- or additive-noise SDE (TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN), in
// the order of the unfused sweep with kernels A and B on a GENERAL launch (general_adjoint_reversible_heun_a / _b):
//   z1 = GRevHeunZOp{dt, backward} on (y, z, f, g0.dW);  adj_f_mid = adj_f + adj_y * half_dt;
//   adj_g_mid_k = adj_g_k + adj_y * (0.5 dW_k), and the vjp with seeds (adj_f_mid, adj_g_mid) at (tv, z);
//   f1, g1 at (t1, z1);  y1 = GRevHeunOp{half_dt, backward} on (y, f, f1, (g0 + g1).(0.5 dW));
//   adj_z' = adj_z + vjp_z; adj_y1 = adj_y + 2 adj_z'; adj_z1 = -adj_z'; adj_f1 = adj_y * half_dt + adj_z' * dt;
//   adj_g1_k = adj_y * (0.5 dW_k) + adj_z1 * (-1 dW_k)
// No (d, m) block stays in registers: g_k at (t, z) is re-evaluated from the program whenever it is read (it is
// deterministic, so it equals the g the unfused step stored), and adj_g is carried as kernel B's rank-2 form: per lane
// (ra, rb) = (adj_y, adj_z1) of the previous step, per thread its increments wp.  Only the chunk's first step reads g0
// and adj_g from memory; the chunk stores both once at its end.  `Prog` (pw_general_adjoint_source in pointwise.cu)
// runs each channel pass.  A per-channel contribution is added to its (rows, d, m) partial at every step by the thread
// that owns the element; a (rows, d) one is summed in registers and added to its partial once, as for diagonal noise.
template <typename T, int SRC, typename Prog>
__device__ __forceinline__ void pw_general_adjoint_reversible_heun_steps(const PwOperands<T>& ops, const PwAdjP<T>& p,
                                                                         const NoiseP<T>& nz,
                                                                         const PwAdjSteps<T>& st) {
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  const Key key = load_key(nz.key);
  Prog prog;
  T y[4], z[4], f[4], ay[4], af[4], az[4], ra[4], rb[4], acc[Prog::NP][4], nn[Prog::NN][4], wp[4 * Prog::MQ];
  const T* tv = p.base.t0;  // the time of z, at which nn holds the forward (rows, d) values
  for (int j = 0; j < st.n; ++j) {
    const PwAdjStep<T>& s = st.s[j];
    NoiseP<T> n = nz;  // this step's cell
    n.cell_id = s.cell;
    n.sqrt_h = s.sqrt_h;
    T w[4 * Prog::MQ];
    pw_general_noise<T, SRC, Prog::MQ>(n, key, row, w);
    if (j == 0) {  // the first increments are drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      if (Q >= p.base.nquads) return;
      load_quad(p.in[kAdjY], c.base, c.vec, c.nvalid, y);
      load_quad(p.in[kAdjZ], c.base, c.vec, c.nvalid, z);
      load_quad(p.in[kAdjF], c.base, c.vec, c.nvalid, f);
      load_quad(p.in[kAdjAdjY], c.base, c.vec, c.nvalid, ay);
      load_quad(p.in[kAdjAdjF], c.base, c.vec, c.nvalid, af);
      load_quad(p.in[kAdjAdjZ], c.base, c.vec, c.nvalid, az);
      prog.load(ops, c);
      T f0[4];
      prog.fwd(ops, c, tv, z, nn, f0);
#pragma unroll
      for (int k = 0; k < Prog::NP; ++k)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[k][i] = T(0);
#pragma unroll
      for (int i = 0; i < 4; ++i) ra[i] = rb[i] = T(0);
#pragma unroll
      for (int k = 0; k < 4 * Prog::MQ; ++k) wp[k] = T(0);
    }
    const bool first = j == 0;
    const T dt = s.dt, half_dt = T(0.5) * dt;
    T afm[4], zc[4], vz[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) afm[i] = af[i] + ay[i] * half_dt;  // AdjAElemOp
    prog.vjp(ops, c, tv, z, nn, w, wp, first, p.in[kAdjG], p.in[kAdjAdjG], ay, ra, rb, afm, zc, vz, acc, p.part);
    T z1[4], f1[4], nn1[Prog::NN][4];
    const GRevHeunZOp<T> zop{dt, 1};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const T e[3] = {y[i], z[i], f[i]}, g1[1] = {zc[i]};
      T o[1];
      zop.combine(e, g1, o);
      z1[i] = o[0];
    }
    prog.fwd(ops, c, s.t1, z1, nn1, f1);
    const GRevHeunOp<T> yop{half_dt, 1};
    T wt[4 * Prog::MQ], yc[4];
#pragma unroll
    for (int k = 0; k < 4 * Prog::MQ; ++k) wt[k] = yop.weight(0, w[k], T(0));
    prog.ystep(ops, c, tv, z, nn, s.t1, z1, nn1, wt, first, p.in[kAdjG], yc);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const T e[3] = {y[i], f[i], f1[i]}, g1[1] = {yc[i]};
      T o[1];
      yop.combine(e, g1, o);
      y[i] = o[0];
      const T adj_z0 = az[i] + vz[i];  // AdjBElemOp
      ra[i] = ay[i];
      af[i] = ay[i] * half_dt + adj_z0 * dt;
      ay[i] = ay[i] + T(2) * adj_z0;
      az[i] = -adj_z0;
      rb[i] = az[i];
      z[i] = z1[i];
      f[i] = f1[i];
#pragma unroll
      for (int k = 0; k < Prog::NN; ++k) nn[k][i] = nn1[k][i];
    }
#pragma unroll
    for (int k = 0; k < 4 * Prog::MQ; ++k) wp[k] = w[k];
    tv = s.t1;
    if (s.out >= 0) {  // adjoint.py:114-116
      T gy[4];
      load_quad(p.ys + s.out * p.plane, c.base, c.vec, c.nvalid, y);
      load_quad(p.gys + s.out * p.plane, c.base, c.vec, c.nvalid, gy);
#pragma unroll
      for (int i = 0; i < 4; ++i) ay[i] = ay[i] + gy[i];
    }
  }
  store_quad(p.out[kAdjY], c.base, c.vec, c.nvalid, y);
  store_quad(p.out[kAdjZ], c.base, c.vec, c.nvalid, z);
  store_quad(p.out[kAdjF], c.base, c.vec, c.nvalid, f);
  store_quad(p.out[kAdjAdjY], c.base, c.vec, c.nvalid, ay);
  store_quad(p.out[kAdjAdjF], c.base, c.vec, c.nvalid, af);
  store_quad(p.out[kAdjAdjZ], c.base, c.vec, c.nvalid, az);
  prog.gstore(ops, c, tv, z, nn, p.out[kAdjG]);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j >= c.nvalid) continue;
#pragma unroll
    for (int k = 0; k < Prog::M; ++k)  // launch_outer (tableau_general.cu): adj_y (x) (0.5 dW) + adj_z1 (x) (-1 dW)
      p.out[kAdjAdjG][(c.base + j) * Prog::M + k] = ra[j] * (T(0.5) * wp[k]) + rb[j] * (T(-1) * wp[k]);
  }
#pragma unroll
  for (int k = 0; k < Prog::NP; ++k) {
    if (!p.part[k] || Prog::pc(k)) continue;  // (NP is 1 for a program without parameters)
    T v[4];
    load_quad(p.part[k], c.base, c.vec, c.nvalid, v);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = v[i] + acc[k][i];
    store_quad(p.part[k], c.base, c.vec, c.nvalid, v);
  }
}

}  // namespace tsde
