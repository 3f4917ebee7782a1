// Whole steps of an element-wise SDE as one kernel: tsde_step_milstein_pointwise (and tsde_solve_milstein_pointwise,
// up to TSDE_PW_MAX_STEPS consecutive Milstein steps in one kernel), tsde_step_srk_diag_pointwise,
// tsde_step_predictor_corrector_pointwise, and tsde_solve_euler_pointwise and tsde_solve_reversible_heun_pointwise
// (up to TSDE_PW_MAX_STEPS Euler or reversible-Heun steps in one kernel), and tsde_adaptive_proposal_pointwise (an
// adaptive solve's full step and two half steps in one kernel) (include/torchsde_b200.h describes the tsde_pointwise
// program and its two layouts).
//
// The SDE's f and g (and for Milstein the vjp of g) arrive as a small program of element-wise instructions.  The SRK,
// predictor-corrector and Euler / reversible-Heun kernels interpret it between the unfused step's own ops
// (tableau_diag_ops.cuh), one IEEE rounding per element (this translation unit is compiled with -fmad=false, as the
// tableaus are), so a fused step equals the unfused one bit for bit.  A Milstein program, and a general-noise one, is
// compiled instead, at run time, into a kernel of its own with the same roundings (pw_milstein_source,
// pw_general_source, NVRTC).  The file holds, in this order: the decoded program, its register file and interpreter,
// the validation every program passes before a launch and the decoding that follows it, the prologue the kernels
// share, the program emitter the two code generators share, the compiled units (kPwUnits) and their kernel cache, the
// interpreting kernels with the layout each accepts, the host steps every launch shares (pw_fill, pw_steps,
// pw_launch, pw_launch_compiled), and the launches.
//
// One thread per quad, as ew_fast_kernel.  The program's registers live in shared memory as 16-byte vectors laid
// out [reg][plane][thread] (a float quad is one plane, a double quad two): a warp's 128-bit access is 512 contiguous
// bytes, conflict-free.  A dynamically indexed per-thread array would live in local memory instead.  The state, go,
// the SDE's results and the increments stay in registers; the program reads y and go from their own slots.
#include <dlfcn.h>
#include <nvrtc.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <string>
#include <type_traits>

#include "tableau_diag_ops.cuh"

namespace tsde {

// pw_device.cuh and the headers it includes, as NVRTC is given them: their names as pw_device.cuh includes them, and
// their text (embedded by build() into a generated source of the library)
constexpr int kPwHeaderCount = 4;  // pw_device.cuh, philox.cuh, rowdiv.cuh, include/torchsde_b200.h
extern const char* const kPwHeaderNames[kPwHeaderCount];
extern const char* const kPwHeaderSources[kPwHeaderCount];

// ---- the decoded program --------------------------------------------------------------------------------------------
// pw_prepare decodes the caller's tsde_pointwise once per launch into a PwProg, in which every source is a slot of the
// shared-memory register file:
//   [0, n_regs)  the program's registers
//   y            the state the program runs at, stored there before each evaluation
//   go           the Milstein seed (Milstein layout only)
//   t0           the evaluation's time, stored once per evaluation (when a TSDE_PW_T0 operand is read)
//   u            the launch-uniform values: IMM and SCALAR operands, one per "thread" lane of the slot, written once
//                per launch after the dependency wait
//   hoisted      one slot per CHANNEL / ROW operand, this thread's quad of it, loaded once per launch after the wait
//   end          the first slot past the layout (SRK's fp64 stash starts there)
// A source is then one 16-byte-vector load at (slot, lane): lane = threadIdx.x, or the entry's lane of the u slot (a
// broadcast).  CHANNEL / ROW operands past kPwHoistSlots are read from global memory at every use instead.
//
// An instruction is one word: op in bits [0, 3), dst in [3, 8), source a in [8, 20), source b in [20, 32) (b = a for
// NEG, SQRT and ABS).  A source is a slot in bits [0, 5), with kPwSrcUniform its lane in bits [6, 11); or kPwSrcGlobal
// and the index of its operand in bits [0, 5).  A program with comparison and selection ops (PwProg::ext) needs a
// fourth op bit: its words keep it in bit 31, and its sources are 11 bits, a global operand being kPwExtGlobal (the
// uniform bit with lane 31, which no uniform operand has).  SEL's third source, its condition, is the dst slot.  The
// six-op programs keep the encoding, and the loop, they always had.
constexpr uint32_t kPwSrcUniform = 1u << 5, kPwSrcGlobal = 1u << 11, kPwExtGlobal = kPwSrcUniform | 31u << 6;

// CHANNEL / ROW operands are hoisted into slots only while the layout stays within kPwHoistSlots slots, the footprint
// of a program of TSDE_PW_MAX_REGS registers: hoisting never raises a program's shared memory past what the library's
// largest program takes.  Registers, y, go, t0 and u always have their slots, at most TSDE_PW_MAX_REGS + 4.
constexpr int kPwHoistSlots = TSDE_PW_MAX_REGS;
constexpr int kPwMaxSlots = TSDE_PW_MAX_REGS + 4;
static_assert(kPwMaxSlots * kThreads * 4 * sizeof(double) <= 227 * 1024,
              "every accepted program's fp64 register file fits one CTA's shared memory");
static_assert(kPwMaxSlots <= 32 && TSDE_PW_MAX_OPERANDS <= 31, "slots, operand indices and lanes fit five bits");

template <typename T>
struct PwProg {
  int32_t n_fg, n_instr;
  uint16_t f_src, g_src, gdg_src;    // (gdg_src, go: the Milstein layout's, which runs compiled instead: y and -1)
  int8_t y, go, t0, u, hoist, end;  // slots (t0: -1 when no operand reads the time)
  int8_t n_uniform, n_hoisted;      // operand[0, n_uniform) fill the u slot, the next n_hoisted the hoisted slots
  int8_t n_global;                  // the operands past those, read from global memory at every use
  int8_t ext;                       // some instruction has an opcode past TSDE_PW_SQRT
  uint32_t row;                     // bit k: operand[k] is a ROW operand (else CHANNEL)
  uint32_t instr[TSDE_PW_MAX_INSTR];
  PwOperand<T> operand[TSDE_PW_MAX_OPERANDS];
};

// ---- the interpreter ------------------------------------------------------------------------------------------------
// slot r, lane l: float4 r * kThreads + l; a double quad is the double2 pair 2 r kThreads + l and that + kThreads
__device__ __forceinline__ void pw_sload(const void* s, int r, int l, float (&v)[4]) {
  const float4 x = static_cast<const float4*>(s)[r * kThreads + l];
  v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
}
__device__ __forceinline__ void pw_sstore(void* s, int r, int l, const float (&v)[4]) {
  static_cast<float4*>(s)[r * kThreads + l] = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void pw_sload(const void* s, int r, int l, double (&v)[4]) {
  const double2* p = static_cast<const double2*>(s) + 2 * r * kThreads + l;
  const double2 a = p[0], b = p[kThreads];
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void pw_sstore(void* s, int r, int l, const double (&v)[4]) {
  double2* p = static_cast<double2*>(s) + 2 * r * kThreads + l;
  p[0] = make_double2(v[0], v[1]);
  p[kThreads] = make_double2(v[2], v[3]);
}
template <typename T>
__device__ __forceinline__ void pw_sstore(void* s, int r, const T (&v)[4]) {
  pw_sstore(s, r, threadIdx.x, v);
}

// GLOBAL: the source may be a CHANNEL / ROW operand that did not fit the slots, read from global memory; EXT: the
// source is in the encoding of a program with comparison and selection ops
template <bool GLOBAL = true, bool EXT = false, typename T>
__device__ __forceinline__ void pw_fetch(const PwProg<T>& pg, const PwQuad& c, const void* regs, uint32_t s,
                                         T (&v)[4]) {
  if (GLOBAL && (EXT ? (s & kPwExtGlobal) == kPwExtGlobal : (s & kPwSrcGlobal) != 0)) {
    const int k = s & 31;
    load_quad(pg.operand[k].ptr, (pg.row >> k) & 1 ? c.base : c.chan, c.vec, c.nvalid, v);
    return;
  }
  pw_sload(regs, s & 31, s & kPwSrcUniform ? s >> 6 : threadIdx.x, v);
}

// instructions [i0, i1): one warp-uniform dispatch per instruction, one IEEE rounding per element (-fmad=false).  EXT:
// the program has comparison and selection ops (opcodes past TSDE_PW_SQRT), which round nothing; each case is the
// expression of the ATen CUDA kernel it restates (::max / ::min are fmax / fmin), so NaN payloads and signed zeros come
// out as ATen's do.  Programs without them run the six-op loop.
template <bool GLOBAL, bool EXT, typename T>
__device__ __forceinline__ void pw_loop(const PwProg<T>& pg, const PwQuad& c, void* regs, int i0, int i1) {
  for (int i = i0; i < i1; ++i) {
    const uint32_t in = pg.instr[i];
    T a[4], b[4], r[4];
    pw_fetch<GLOBAL, EXT>(pg, c, regs, (in >> 8) & 0xFFF, a);
    pw_fetch<GLOBAL, EXT>(pg, c, regs, EXT ? (in >> 20) & 0x7FF : in >> 20, b);
    if (EXT && (in >> 31)) {  // (opcodes 8 to 14)
      const int dst = (in >> 3) & 31;
      switch ((in & 7) | 8) {
        case TSDE_PW_LT:  // lt, and gt with the operands swapped
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = a[j] < b[j] ? T(1) : T(0);
          break;
        case TSDE_PW_LE:  // le, ge with the operands swapped, threshold_backward's x <= threshold
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = a[j] <= b[j] ? T(1) : T(0);
          break;
        case TSDE_PW_EQ:
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = a[j] == b[j] ? T(1) : T(0);
          break;
        case TSDE_PW_MAXIMUM:  // maximum_kernel_cuda
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = a[j] != a[j] ? a[j] : b[j] != b[j] ? b[j] : ::max(a[j], b[j]);
          break;
        case TSDE_PW_MINIMUM:  // minimum_kernel_cuda
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = a[j] != a[j] ? a[j] : b[j] != b[j] ? b[j] : ::min(a[j], b[j]);
          break;
        case TSDE_PW_ABS:
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = fabs(a[j]);
          break;
        default:  // TSDE_PW_SEL: where_kernel, masked_fill; the condition is the destination (read into r)
          pw_sload(regs, dst, threadIdx.x, r);
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = r[j] != T(0) ? a[j] : b[j];
          break;
      }
      pw_sstore(regs, dst, r);
      continue;
    }
    switch (in & 7) {
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
    pw_sstore(regs, (in >> 3) & 31, r);
  }
}

// The loop that reads only shared memory unless the program has operands in global memory, which is rare (see
// kPwHoistSlots).  EXT: the program has comparison and selection ops; those programs run in kernels of their own (the
// *_ext_kernel instantiations), so that the six-op programs run the code, and the registers, they always ran.
template <bool EXT, typename T>
__device__ __forceinline__ void pw_run(const PwProg<T>& pg, const PwQuad& c, void* regs, int i0, int i1) {
  if (EXT)
    pw_loop<true, true>(pg, c, regs, i0, i1);
  else if (pg.n_global)
    pw_loop<true, false>(pg, c, regs, i0, i1);
  else
    pw_loop<false, false>(pg, c, regs, i0, i1);
}

// The launch-uniform values into the u slot; every thread of the CTA calls it (it ends in a barrier), after the
// dependency wait.
template <typename T>
__device__ __forceinline__ void pw_load_uniform(const PwProg<T>& pg, void* regs) {
  if ((int)threadIdx.x < pg.n_uniform) {
    const PwOperand<T>& o = pg.operand[threadIdx.x];
    const T x = o.ptr ? *o.ptr : o.imm;
    const T v[4] = {x, x, x, x};
    pw_sstore(regs, pg.u, threadIdx.x, v);
  }
  __syncthreads();
}

// This thread's quads of the hoisted operands into their slots, after the dependency wait
template <typename T>
__device__ __forceinline__ void pw_load_hoisted(const PwProg<T>& pg, const PwQuad& c, void* regs) {
  for (int h = 0; h < pg.n_hoisted; ++h) {
    const int k = pg.n_uniform + h;
    T v[4];
    load_quad(pg.operand[k].ptr, (pg.row >> k) & 1 ? c.base : c.chan, c.vec, c.nvalid, v);
    pw_sstore(regs, pg.hoist + h, v);
  }
}

// The state an evaluation runs at and, when the program reads it, its time
template <typename T>
__device__ __forceinline__ void pw_set_state(const PwProg<T>& pg, void* regs, const T* t, const T (&y)[4]) {
  pw_sstore(regs, pg.y, y);
  if (pg.t0 >= 0) {
    const T x = *t;
    const T v[4] = {x, x, x, x};
    pw_sstore(regs, pg.t0, v);
  }
}

// ---- validation -----------------------------------------------------------------------------------------------------
// A program the kernels can run as given: counts, register and operand indices in range, every register written
// before it is read, device operands present (and 16-byte aligned for the vector path).  This is all that stands
// between a caller's program and an out-of-range shared-memory index.  The parts common to both layouts are here;
// which instructions and results may read what is spelt out per layout, beside the kernel that reads them so.

// the counts and the operand table (kinds up to `max_kind`: TSDE_PW_M in the general layout); clears *vec when a
// CHANNEL or ROW operand, which the kernels read as quads, is not 16-byte aligned
static bool pw_valid_tables(const tsde_pointwise& pg, bool* vec, int max_kind = TSDE_PW_ROW) {
  if (pg.n_instr < 0 || pg.n_instr > TSDE_PW_MAX_INSTR || pg.n_fg < 0 || pg.n_fg > pg.n_instr ||
      pg.n_regs < 0 || pg.n_regs > TSDE_PW_MAX_REGS || pg.n_operands < 0 || pg.n_operands > TSDE_PW_MAX_OPERANDS)
    return false;
  for (int k = 0; k < pg.n_operands; ++k) {
    const tsde_pw_operand& o = pg.operand[k];
    if (o.kind < TSDE_PW_IMM || o.kind > max_kind) return false;
    if (o.kind >= TSDE_PW_SCALAR && !o.ptr) return false;
    if (o.kind == TSDE_PW_CHANNEL || o.kind == TSDE_PW_ROW) *vec = *vec && aligned16(o.ptr);
  }
  return true;
}

// a source that can be read when the registers in `written` are defined and `seeds` seeds exist (1: go; 2: go and
// go2, the adjoint layout's vjp part)
static bool pw_valid_source(const tsde_pointwise& pg, uint32_t s, int seeds, uint64_t written) {
  if (s == TSDE_PW_SRC_Y) return true;
  if (s == TSDE_PW_SRC_GO) return seeds >= 1;
  if (s == TSDE_PW_SRC_GO2) return seeds >= 2;
  if (s >= (uint32_t)TSDE_PW_OPERAND(0)) return (int)(s - TSDE_PW_OPERAND(0)) < pg.n_operands;
  return (int)s < pg.n_regs && ((written >> s) & 1u);
}

// the transcendental opcodes, which only the compiled layouts run (pw_milstein_source, pw_general_source)
static bool pw_transcendental(int op) { return op >= TSDE_PW_EXP && op <= TSDE_PW_SIGMOID_BACKWARD; }

// NEG, SQRT, ABS and the transcendental ops of one argument read source a only
static bool pw_unary(int op) {
  return op == TSDE_PW_NEG || op == TSDE_PW_SQRT || op == TSDE_PW_ABS || (op >= TSDE_PW_EXP && op <= TSDE_PW_SIGMOID);
}

// instructions [i0, i1), run in order from the registers in `written`, which gains the ones they define; `compiled`:
// the layout is compiled, so the transcendental opcodes are valid too (POW's exponent an IMM operand); `csum`: the
// general adjoint's vjp part, where CSUM (source a only) is valid too
static bool pw_valid_range(const tsde_pointwise& pg, int i0, int i1, int seeds, uint64_t& written,
                           bool compiled = false, bool csum = false) {
  for (int i = i0; i < i1; ++i) {
    const tsde_pw_instr& in = pg.instr[i];
    const bool sum = csum && in.op == TSDE_PW_CSUM;
    if (!(compiled && pw_transcendental(in.op)) && !sum &&
        ((in.op > TSDE_PW_SQRT && in.op < TSDE_PW_LT) || in.op > TSDE_PW_SEL))
      return false;
    if ((int)in.dst >= pg.n_regs || !pw_valid_source(pg, in.a, seeds, written)) return false;
    if (!pw_unary(in.op) && !sum && !pw_valid_source(pg, in.b, seeds, written)) return false;
    if (in.op == TSDE_PW_POW && (in.b < TSDE_PW_OPERAND(0) || in.b >= TSDE_PW_SRC_GO2 ||
                                 pg.operand[in.b - TSDE_PW_OPERAND(0)].kind != TSDE_PW_IMM))
      return false;
    if (in.op == TSDE_PW_SEL && !((written >> in.dst) & 1u)) return false;  // the condition
    written |= 1ull << in.dst;
  }
  return true;
}

// ---- decoding -------------------------------------------------------------------------------------------------------
// The PwProg of a two-program layout that passed validation, with `extra` slots past the layout (SRK's fp64 stash)
// counted against kPwHoistSlots.  Returns the slots a launch takes, extra included.
template <typename T>
static int pw_decode(const tsde_pointwise& in, int extra, PwProg<T>& pg) {
  pg = PwProg<T>{};
  for (int i = 0; i < in.n_instr; ++i) pg.ext = pg.ext || in.instr[i].op > TSDE_PW_SQRT;
  pg.n_fg = in.n_fg;
  pg.n_instr = in.n_instr;
  int n_uniform = 0, n_local = 0;
  bool t0 = false;
  for (int k = 0; k < in.n_operands; ++k) {
    const int kind = in.operand[k].kind;
    t0 = t0 || kind == TSDE_PW_T0;
    n_uniform += kind == TSDE_PW_IMM || kind == TSDE_PW_SCALAR;
    n_local += kind >= TSDE_PW_CHANNEL;
  }
  int slot = in.n_regs;
  pg.y = slot++;
  pg.go = -1;
  pg.t0 = t0 ? slot++ : -1;
  pg.u = n_uniform ? slot++ : -1;
  pg.hoist = slot;
  pg.n_uniform = n_uniform;
  pg.n_hoisted = std::min(n_local, std::max(kPwHoistSlots - slot - extra, 0));
  pg.n_global = n_local - pg.n_hoisted;
  slot += pg.n_hoisted;
  pg.end = slot;
  // the operand table in decoded order (uniform, hoisted, global), and the source that names each caller operand
  uint32_t src[TSDE_PW_MAX_OPERANDS];
  int n_u = 0, n_l = 0;
  for (int k = 0; k < in.n_operands; ++k) {
    const tsde_pw_operand& o = in.operand[k];
    if (o.kind == TSDE_PW_T0) {
      src[k] = pg.t0;
      continue;
    }
    const bool local = o.kind >= TSDE_PW_CHANNEL;
    const int j = local ? n_uniform + n_l++ : n_u++;
    pg.operand[j] = PwOperand<T>{o.kind == TSDE_PW_IMM ? nullptr : static_cast<const T*>(o.ptr), (T)o.imm};
    if (o.kind == TSDE_PW_ROW) pg.row |= 1u << j;
    if (!local)
      src[k] = pg.u | kPwSrcUniform | (uint32_t)j << 6;
    else if (j - n_uniform < pg.n_hoisted)
      src[k] = pg.hoist + (j - n_uniform);
    else
      src[k] = (pg.ext ? kPwExtGlobal : kPwSrcGlobal) | j;
  }
  auto source = [&](uint32_t s) -> uint32_t {
    if (s == TSDE_PW_SRC_Y) return pg.y;
    return s >= (uint32_t)TSDE_PW_OPERAND(0) ? src[s - TSDE_PW_OPERAND(0)] : s;
  };
  for (int i = 0; i < in.n_instr; ++i) {
    const tsde_pw_instr& x = in.instr[i];
    const uint32_t a = source(x.a), b = pw_unary(x.op) ? a : source(x.b);
    pg.instr[i] = (x.op & 7u) | (uint32_t)x.dst << 3 | a << 8 | b << 20 | (uint32_t)(x.op >> 3) << 31;
  }
  pg.f_src = source(in.f_src);
  pg.g_src = source(in.g_src);
  pg.gdg_src = pg.y;  // (the two-program layouts have no gdg)
  return slot + extra;
}

// ---- what every kernel starts with ----------------------------------------------------------------------------------
// This thread's quad `c`, its increments and its y0, and the program's operands in their slots.  The increments
// depend on no predecessor: they are drawn while the previous kernel drains (programmatic dependent launch); y0 and
// the operands are read after the dependency wait.  False for a thread past the last quad.
template <typename T, int SRC, bool WANT_U>
__device__ __forceinline__ bool pw_begin(const PwProg<T>& pg, const PwP<T>& p, const NoiseP<T>& nz, void* regs,
                                         PwQuad& c, T (&w)[4], T (&u)[4], T (&y0)[4]) {
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
  c.chan = 4 * q;
  c.base = row * p.d + c.chan;
  const int64_t rem = p.d - c.chan;
  c.nvalid = rem < 4 ? (int)rem : 4;
  c.vec = p.vec != 0;
  quad_noise<T, SRC, WANT_U>(nz, load_key(nz.key), row, q, c.vec, c.nvalid, w, u);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  pw_load_uniform(pg, regs);
  if (Q >= p.nquads) return false;
  load_quad(p.y0, c.base, c.vec, c.nvalid, y0);
  pw_load_hoisted(pg, c, regs);
  return true;
}

// ---- compiled programs (tsde_solve_milstein_pointwise, tsde_step_milstein_pointwise, GENERAL launches) -------------
// A Milstein program is not interpreted: once validated, it is written out as one CUDA translation unit
// (pw_milstein_source) whose kernels run pw_milstein_steps (pw_device.cuh) with the program inlined as straight-line
// register code, compiled at run time by NVRTC to an sm_90a cubin and loaded as a CUDA library.  Each instruction is
// the expression of the matching `case` of pw_loop (pw_expression), one statement per lane, and the translation unit
// is compiled with the library's IEEE options (-fmad=false, NVRTC's default -prec-div=true, -prec-sqrt=true,
// -ftz=false), so a compiled step equals the unfused one bit for bit.  Operand values and addresses are not in the
// source: IMM values and SCALAR / CHANNEL / ROW pointers are the kernel's PwOperands parameter, so the source is a
// function of the program's structure alone (instruction words, n_regs, n_fg, result sources, operand kinds, dtype),
// and it is the key of the process-wide cache of loaded kernels: SDEs that differ only in parameter values share one
// compiled kernel.  The general-noise programs (pw_general_source) are written out from the same parts.

// CHANNEL / ROW operand quads a compiled program keeps in registers for the whole chunk (loaded once per launch after
// the dependency wait); any past these are loaded again at every step.  Within the launch bounds below, cfg2's program
// (two CHANNEL operands) takes 54 registers in fp32.
constexpr int kPwJitHoistQuads[2] = {4, 2};  // float, double

// The compiled kernels run at the resident CTAs per SM the interpreted Milstein kernel had (58-59 registers in fp32,
// 88-92 in fp64): pointwise.py's _RESIDENT_CTAS and chunk_length count on it.
constexpr int kPwJitCtas[2] = {4, 2};

// (const: concatenating two temporaries would instantiate std::operator+(string&&, string&&) out of line, an exported
// symbol of the library)
static const std::string num(int x) {
  char b[16];
  snprintf(b, sizeof(b), "%d", x);
  return b;
}

// The concatenation of `parts` (built by appending, for the reason above)
static std::string pw_cat(std::initializer_list<std::string> parts) {
  std::string s;
  for (const std::string& x : parts) s += x;
  return s;
}

// ---- the transcendental ops (TSDE_PW_EXP .. TSDE_PW_SIGMOID_BACKWARD) -----------------------------------------------
// libdevice's exp, log, sin, ... are not correctly rounded, and their code, like a * (1 - b * b), compiles to other
// instructions when FMA contraction is on: ATen's kernels, built by nvcc with its default -fmad=true, contract; the
// program translation units, compiled with -fmad=false, must not.  So each op is a __noinline__ function of a fixed
// translation unit of its own, kPwHelpers, whose body is the lambda of the ATen CUDA kernel it restates (opmath is the
// dtype itself for float and double), compiled by the same NVRTC with -fmad=true -rdc=true.  A program that uses one is
// compiled with -rdc=true and calls it, and the two relocatable cubins are linked by nvJitLink without LTO, which would
// recompile both under one fmad setting (pw_loaded).  Programs without these ops keep their source and the plain path.
static const char kPwHelpers[] =
    "// The transcendental ops of torchsde_b200's compiled element-wise programs, each as its ATen CUDA kernel's\n"
    "// lambda; compiled with -fmad=true, as ATen is\n"
    "namespace tsde {\n"
    "#define TSDE_PW_OP1(name, ff, fd) \\\n"
    "  __device__ __noinline__ float pw_##name(float a) { return ff; } \\\n"
    "  __device__ __noinline__ double pw_##name(double a) { return fd; }\n"
    "#define TSDE_PW_OP2(name, e) \\\n"
    "  __device__ __noinline__ float pw_##name(float a, float b) { typedef float T; return e; } \\\n"
    "  __device__ __noinline__ double pw_##name(double a, double b) { typedef double T; return e; }\n"
    "TSDE_PW_OP1(exp, expf(a), exp(a))\n"        // exp_kernel_cuda
    "TSDE_PW_OP1(log, logf(a), log(a))\n"        // log_kernel_cuda
    "TSDE_PW_OP1(sin, sinf(a), sin(a))\n"        // sin_kernel_cuda
    "TSDE_PW_OP1(cos, cosf(a), cos(a))\n"        // cos_kernel_cuda
    "TSDE_PW_OP1(tanh, tanhf(a), tanh(a))\n"     // tanh_kernel_cuda
    "TSDE_PW_OP1(log1p, log1pf(a), log1p(a))\n"  // log1p_kernel_cuda
    "TSDE_PW_OP1(expm1, expm1f(a), expm1(a))\n"  // expm1_kernel_cuda
    "TSDE_PW_OP1(rsqrt, rsqrtf(a), rsqrt(a))\n"  // rsqrt_kernel_cuda
    "TSDE_PW_OP1(sigmoid, 1.0f / (1.0f + expf(-a)), 1.0 / (1.0 + exp(-a)))\n"  // sigmoid_kernel_cuda
    "TSDE_PW_OP2(pow, pow(a, b))\n"                          // pow_tensor_scalar_kernel: pow_(base, exp)
    "TSDE_PW_OP2(tanh_backward, a * (T(1) - b * b))\n"       // tanh_backward_kernel_cuda
    "TSDE_PW_OP2(sigmoid_backward, a * (T(1) - b) * b)\n"    // sigmoid_backward_kernel_cuda
    "}  // namespace tsde\n";

static const char* const kPwHelperNames[] = {"exp",   "log",   "sin",     "cos", "tanh",          "log1p",
                                             "expm1", "rsqrt", "sigmoid", "pow", "tanh_backward", "sigmoid_backward"};

// The call of transcendental instruction op on sources a and b (b for POW and the backward ops only)
static std::string pw_helper_call(int op, const std::string& a, const std::string& b) {
  const std::string call = std::string("pw_") + kPwHelperNames[op - TSDE_PW_EXP] + "(" + a;
  return pw_unary(op) ? call + ")" : call + ", " + b + ")";
}

// The declarations of kPwHelpers' functions of dtype `T` when the program calls one, or "" when it calls none (its
// source is then the one it always was)
static std::string pw_helper_declarations(const tsde_pointwise& in, const char* T) {
  bool any = false;
  for (int i = 0; i < in.n_instr; ++i) any = any || pw_transcendental(in.instr[i].op);
  if (!any) return "";
  std::string o = "namespace tsde {  // kPwHelpers, linked in\n";
  for (int op = TSDE_PW_EXP; op <= TSDE_PW_SIGMOID_BACKWARD; ++op)
    o += std::string("__device__ ") + T + " pw_" + kPwHelperNames[op - TSDE_PW_EXP] + "(" + T +
         (pw_unary(op) ? "" : std::string(", ") + T) + ");\n";
  return o + "}  // namespace tsde\n\n";
}

// ---- the program emitter --------------------------------------------------------------------------------------------
// The expression of instruction x on sources a and b in dtype f64 / float, as pw_loop's case of its opcode (a
// transcendental op: the call of its helper).  d is the destination, SEL's condition.
static const std::string pw_expression(const tsde_pw_instr& x, const std::string& a, const std::string& b,
                                       const std::string& d, bool f64) {
  if (pw_transcendental(x.op)) return pw_helper_call(x.op, a, b);
  const char* f = f64 ? "" : "f";
  switch (x.op) {
    case TSDE_PW_MUL: return a + " * " + b;
    case TSDE_PW_ADD: return a + " + " + b;
    case TSDE_PW_SUB: return a + " - " + b;
    case TSDE_PW_DIV: return a + " / " + b;
    case TSDE_PW_NEG: return "-" + a;
    case TSDE_PW_SQRT: return pw_cat({"sqrt", f, "(", a, ")"});
    case TSDE_PW_LT: return a + " < " + b + " ? T(1) : T(0)";
    case TSDE_PW_LE: return a + " <= " + b + " ? T(1) : T(0)";
    case TSDE_PW_EQ: return a + " == " + b + " ? T(1) : T(0)";
    case TSDE_PW_MAXIMUM:  // maximum_kernel_cuda (::max is fmax)
      return pw_cat({a, " != ", a, " ? ", a, " : ", b, " != ", b, " ? ", b, " : fmax", f, "(", a, ", ", b, ")"});
    case TSDE_PW_MINIMUM:  // minimum_kernel_cuda (::min is fmin)
      return pw_cat({a, " != ", a, " ? ", a, " : ", b, " != ", b, " ? ", b, " : fmin", f, "(", a, ", ", b, ")"});
    case TSDE_PW_ABS: return pw_cat({"fabs", f, "(", a, ")"});
    default: return d + " != T(0) ? " + a + " : " + b;  // TSDE_PW_SEL: the condition is the destination
  }
}

static bool pw_per_channel_kind(int kind) { return kind == TSDE_PW_DM || kind == TSDE_PW_M; }

// Source s names an operand (not y, a seed or a register)
static bool pw_operand_source(uint8_t s) {
  return s >= TSDE_PW_OPERAND(0) && s != TSDE_PW_SRC_Y && s != TSDE_PW_SRC_GO && s != TSDE_PW_SRC_GO2;
}

// The CHANNEL / ROW operands a unit keeps in its Prog (k<k>[4], loaded once per launch): the first `max` of them.  A
// part loads the others where it reads them (x<k>[4]).
static void pw_hoist(const tsde_pointwise& in, int max, bool (&hoisted)[TSDE_PW_MAX_OPERANDS]) {
  for (int k = 0, n = 0; k < in.n_operands; ++k) {
    const int kind = in.operand[k].kind;
    hoisted[k] = (kind == TSDE_PW_CHANNEL || kind == TSDE_PW_ROW) && n++ < max;
  }
}

// The value of source s in lane j: y, go, register s, or an operand (a DM or M operand at channel k of the lane's d
// index i, for m channels)
static const std::string pw_value(const tsde_pointwise& in, uint8_t s, const bool (&hoisted)[TSDE_PW_MAX_OPERANDS],
                                  int64_t m = 0) {
  if (s == TSDE_PW_SRC_Y) return "y[j]";
  if (s == TSDE_PW_SRC_GO) return "go[j]";
  if (s == TSDE_PW_SRC_GO2) return "go2[j]";
  if (!pw_operand_source(s)) return pw_cat({"r", num(s), "[j]"});
  const int k = s - TSDE_PW_OPERAND(0);
  const std::string n = num(k);
  switch (in.operand[k].kind) {
    case TSDE_PW_IMM: return pw_cat({"ops.k[", n, "].imm"});
    case TSDE_PW_T0: return "t0";
    case TSDE_PW_SCALAR: return "u" + n;
    case TSDE_PW_DM: return pw_cat({"ops.k[", n, "].ptr[i * ", num((int)m), " + k]"});
    case TSDE_PW_M: return pw_cat({"ops.k[", n, "].ptr[k]"});
    default: return pw_cat({hoisted[k] ? "k" : "x", n, "[j]"});
  }
}

// The statement that loads this thread's quad of CHANNEL / ROW operand k into <var>k
static std::string pw_load_operand(const tsde_pointwise& in, int k, const char* var) {
  const std::string n = num(k);
  return pw_cat({"    load_quad(ops.k[", n, "].ptr, c.", in.operand[k].kind == TSDE_PW_ROW ? "base" : "chan",
                 ", c.vec, c.nvalid, ", var, n, ");\n"});
}

// A unit's text up to its Prog's members: the `title` comment, the helper declarations, and `struct Prog {` with
// `members` (the layout's own), each SCALAR operand's value u<k>, the `hoisted` quads k<k>[4], and load(), which
// fills them after the dependency wait.
static std::string pw_prog_head(const tsde_pointwise& in, bool f64, const char* title, const std::string& members,
                                const bool (&hoisted)[TSDE_PW_MAX_OPERANDS]) {
  const char* T = f64 ? "double" : "float";
  std::string o = title;
  o += "#include \"pw_device.cuh\"\n\n";
  o += pw_helper_declarations(in, T);
  o += pw_cat({"namespace tsde {\nnamespace {\ntypedef ", T, " T;\n\nstruct Prog {\n", members});
  for (int k = 0; k < in.n_operands; ++k) {
    if (in.operand[k].kind == TSDE_PW_SCALAR) o += pw_cat({"  T u", num(k), ";\n"});
    if (hoisted[k]) o += pw_cat({"  T k", num(k), "[4];\n"});
  }
  o += "  __device__ __forceinline__ void load(const PwOperands<T>& ops, const PwQuad& c) {\n";
  for (int k = 0; k < in.n_operands; ++k) {
    if (in.operand[k].kind == TSDE_PW_SCALAR) o += pw_cat({"    u", num(k), " = *ops.k[", num(k), "].ptr;\n"});
    if (hoisted[k]) o += pw_load_operand(in, k, "k");
  }
  return o + "  }\n";
}

// ---- the compiled units ---------------------------------------------------------------------------------------------
// Each unit's extern "C" kernels, as its source spells them and as pw_loaded looks them up.  A kernel with `cells` has
// two: <name>_single draws each step from one Brownian cell (TSDE_SRC_COUNTER), <name>_multi sums the cells of a step
// that spans several (kSrcCounterMulti).
struct PwKernelText {
  const char* name;
  bool cells;
  const char* params;  // the wrapper's parameter list, as written
  const char* driver;  // the pw_device.cuh function it calls, with
  const char* args;    // these arguments
};

struct PwUnit {
  bool jit_ctas;           // launch bounds (kThreads, kPwJitCtas[f64]); else (kThreads, 1)
  PwKernelText kernel[2];  // (a unit of one kernel: the second has no name)
};

// The units, by index: Milstein, the four general ones by their layout tag, the Milstein adaptive proposal and the
// reversible-Heun adjoint's backward steps, of diagonal and of general noise
enum { kPwUnitMilstein = 0, kPwUnitAdaptive = TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN + 1, kPwUnitAdjoint,
       kPwUnitGeneralAdjoint };
static_assert(TSDE_PW_LAYOUT_GENERAL == 1 && TSDE_PW_LAYOUT_GENERAL_SRA == 2 &&
                  TSDE_PW_LAYOUT_GENERAL_EULER_HEUN == 3 && TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN == 4,
              "a general unit's index is its layout tag");
enum { kPwGeneralEuler = 0, kPwGeneralMidpoint = 1 };  // the kernels of the TSDE_PW_LAYOUT_GENERAL unit

static const PwUnit kPwUnits[] = {
    {true,
     {{"tsde_pw_milstein", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const tsde::PwP<tsde::T> p,\n"
       "    const tsde::NoiseP<tsde::T> nz, const __grid_constant__ tsde::PwSteps<tsde::T> st) {\n",
       "pw_milstein_steps", "(ops, p, nz, st)"}}},
    {false,
     {{"tsde_pw_general_euler", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const tsde::PwP<tsde::T> p,\n"
       "    const tsde::NoiseP<tsde::T> nz, const __grid_constant__ tsde::PwSteps<tsde::T> st) {\n",
       "pw_general_euler_steps", "(ops, p, nz, st)"},
      {"tsde_pw_general_midpoint", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const tsde::PwGeneralMidP<tsde::T> p,\n"
       "    const tsde::NoiseP<tsde::T> nz) {\n",
       "pw_general_midpoint", "(ops, p, nz)"}}},
    {false,
     {{"tsde_pw_general_sra1", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops,\n"
       "    const __grid_constant__ tsde::PwGeneralSraP<tsde::T> p, const tsde::NoiseP<tsde::T> nz) {\n",
       "pw_general_sra1", "(ops, p, nz)"}}},
    {false,
     {{"tsde_pw_general_euler_heun", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops,\n"
       "    const tsde::PwGeneralMidP<tsde::T> p, const tsde::NoiseP<tsde::T> nz) {\n",
       "pw_general_euler_heun", "(ops, p, nz)"}}},
    {false,
     {{"tsde_pw_general_reversible_heun", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops,\n"
       "    const tsde::PwGeneralRevHeunP<tsde::T> p, const tsde::NoiseP<tsde::T> nz,\n"
       "    const __grid_constant__ tsde::PwSteps<tsde::T> st) {\n",
       "pw_general_reversible_heun_steps", "(ops, p, nz, st)"}}},
    {true,
     {{"tsde_pw_milstein_adaptive", false,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const tsde::PwP<tsde::T> p,\n"
       "    tsde::T* y_next, const __grid_constant__ tsde::PwSubs<tsde::T> st) {\n",
       "pw_milstein_proposal", "(ops, p, y_next, st)"}}},
    {false,
     {{"tsde_pw_adjoint_reversible_heun", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const __grid_constant__ tsde::PwAdjP<tsde::T> p,\n"
       "    const tsde::NoiseP<tsde::T> nz, const __grid_constant__ tsde::PwAdjSteps<tsde::T> st) {\n",
       "pw_adjoint_reversible_heun_steps", "(ops, p, nz, st)"}}},
    {false,
     {{"tsde_pw_general_adjoint_reversible_heun", true,
       "(const __grid_constant__ tsde::PwOperands<tsde::T> ops, const __grid_constant__ tsde::PwAdjP<tsde::T> p,\n"
       "    const tsde::NoiseP<tsde::T> nz, const __grid_constant__ tsde::PwAdjSteps<tsde::T> st) {\n",
       "pw_general_adjoint_reversible_heun_steps", "(ops, p, nz, st)"}}},
};

static const char* const kPwCellSuffix[2] = {"_single", "_multi"};

// (the general kernels' launch bounds: one resident CTA per SM at least, so that ptxas never spills the increments;
// pointwise.py's _RESIDENT_CTAS counts on one)
static_assert(sizeof(PwOperands<double>) + sizeof(PwP<double>) + sizeof(NoiseP<double>) + sizeof(PwSteps<double>) <=
                  4096,
              "the compiled Milstein and general Euler kernels' parameters fit the 4 KiB parameter space");
static_assert(sizeof(PwOperands<double>) + sizeof(PwGeneralMidP<double>) + sizeof(NoiseP<double>) <= 4096,
              "the compiled general midpoint and Euler-Heun kernels' parameters fit the 4 KiB parameter space");
static_assert(sizeof(PwOperands<double>) + sizeof(PwGeneralSraP<double>) + sizeof(NoiseP<double>) <= 4096,
              "the compiled sra1 kernel's parameters fit the 4 KiB parameter space");
static_assert(sizeof(PwOperands<double>) + sizeof(PwGeneralRevHeunP<double>) + sizeof(NoiseP<double>) +
                      sizeof(PwSteps<double>) <=
                  4096,
              "the compiled general reversible-Heun kernel's parameters fit the 4 KiB parameter space");
static_assert(sizeof(PwOperands<double>) + sizeof(PwAdjP<double>) + sizeof(NoiseP<double>) +
                      sizeof(PwAdjSteps<double>) <=
                  4096,
              "the compiled adjoint kernel's parameters fit the 4 KiB parameter space");

// The end of unit `unit`'s source: the close of its Prog and namespaces, then its kernels
static std::string pw_unit_tail(int unit, bool f64) {
  const PwUnit& u = kPwUnits[unit];
  const std::string bounds = pw_cat({"__launch_bounds__(", num(kThreads), ", ", num(u.jit_ctas ? kPwJitCtas[f64] : 1),
                                     ")"});
  std::string o = "};\n}  // namespace\n}  // namespace tsde\n";
  for (const PwKernelText& k : u.kernel)
    for (int multi = 0; k.name && multi < (k.cells ? 2 : 1); ++multi)
      o += pw_cat({"\nextern \"C\" __global__ void ", bounds, "\n", k.name, k.cells ? kPwCellSuffix[multi] : "",
                   k.params, "  tsde::", k.driver, "<tsde::T, ",
                   k.cells ? (multi ? "tsde::kSrcCounterMulti, " : "TSDE_SRC_COUNTER, ") : "", "tsde::Prog>", k.args,
                   ";\n}\n"});
  return o;
}

// The body of a compiled program's part: instructions [i0, i1) and then `results`, each a statement `prefix` followed
// by the value of its source; the time (*`time`) and the operands not kept in registers (`hoisted`) that they read
// are loaded first.
static std::string pw_part(const tsde_pointwise& in, bool f64, const bool (&hoisted)[TSDE_PW_MAX_OPERANDS], int i0,
                           int i1, const std::pair<std::string, uint8_t>* results, int n_results, const char* time) {
  uint8_t reads[2 * TSDE_PW_MAX_INSTR + 2 + TSDE_PW_ADJ_MAX_PARAMS];
  int n = 0;
  for (int i = i0; i < i1; ++i) {
    reads[n++] = in.instr[i].a;
    if (!pw_unary(in.instr[i].op)) reads[n++] = in.instr[i].b;
  }
  for (int r = 0; r < n_results; ++r) reads[n++] = results[r].second;
  std::string o;
  bool t0 = false, x[TSDE_PW_MAX_OPERANDS] = {};
  for (int i = 0; i < n; ++i) {
    const uint8_t s = reads[i];
    if (!pw_operand_source(s)) continue;
    const int k = s - TSDE_PW_OPERAND(0), kind = in.operand[k].kind;
    if (kind == TSDE_PW_T0 && !t0) {
      t0 = true;
      o += pw_cat({"    const T t0 = *", time, ";\n"});
    } else if (kind >= TSDE_PW_CHANNEL && !hoisted[k] && !x[k]) {
      x[k] = true;
      o += pw_cat({"    T x", num(k), "[4];\n"});
      o += pw_load_operand(in, k, "x");
    }
  }
  o += "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
  for (int i = i0; i < i1; ++i) {
    const tsde_pw_instr& ins = in.instr[i];
    const std::string a = pw_value(in, ins.a, hoisted), b = pw_unary(ins.op) ? a : pw_value(in, ins.b, hoisted);
    const std::string d = pw_cat({"r", num(ins.dst), "[j]"});
    o += pw_cat({"      ", d, " = ", pw_expression(ins, a, b, d, f64), ";\n"});
  }
  for (int r = 0; r < n_results; ++r)
    o += pw_cat({"      ", results[r].first, pw_value(in, results[r].second, hoisted), ";\n"});
  return o + "    }\n";
}

// The translation unit of a program that passed pw_valid_tables and pw_valid_milstein, for dtype `f64`: the Milstein
// unit (the kernels of consecutive steps) or the adaptive one (the kernel of an adaptive solve's proposal).
static std::string pw_milstein_source(const tsde_pointwise& in, bool f64, int unit = kPwUnitMilstein) {
  bool hoisted[TSDE_PW_MAX_OPERANDS];
  pw_hoist(in, kPwJitHoistQuads[f64], hoisted);
  std::string regs;
  for (int r = 0; r < in.n_regs; ++r) regs += pw_cat({"  T r", num(r), "[4];\n"});
  std::string o = pw_prog_head(in, f64, "// A Milstein program of torchsde_b200, generated by pw_milstein_source\n",
                               regs, hoisted);
  o += "  __device__ __forceinline__ void fg(const PwOperands<T>& ops, const PwQuad& c, const PwStep<T>& s,\n"
       "                                     const T (&y)[4], T (&f)[4], T (&g)[4]) {\n";
  const std::pair<std::string, uint8_t> fg[2] = {{"f[j] = ", in.f_src}, {"g[j] = ", in.g_src}};
  o += pw_part(in, f64, hoisted, 0, in.n_fg, fg, 2, "s.t0");
  o += "  }\n  __device__ __forceinline__ void vjp(const PwOperands<T>& ops, const PwQuad& c, const PwStep<T>& s,\n"
       "                                      const T (&y)[4], const T (&go)[4], T (&gdg)[4]) {\n";
  const std::pair<std::string, uint8_t> gdg[1] = {{"gdg[j] = ", in.gdg_src}};
  o += pw_part(in, f64, hoisted, in.n_fg, in.n_instr, gdg, 1, "s.t0");
  o += "  }\n";
  o += pw_unit_tail(unit, f64);
  return o;
}

// The translation unit of an adjoint program that passed pw_valid_adjoint, for dtype `f64`: the Milstein layout's f / g
// part at a time pointer, and a vjp part with two seeds whose results are vjp_z and the contributions, each added to
// its accumulator (pw_adjoint_reversible_heun_steps).  The CHANNEL / ROW operands stay in registers as Milstein's do.
static std::string pw_adjoint_source(const tsde_pw_adjoint& ad, bool f64) {
  const tsde_pointwise& in = ad.prog;
  bool hoisted[TSDE_PW_MAX_OPERANDS];
  pw_hoist(in, kPwJitHoistQuads[f64], hoisted);
  std::string members = pw_cat({"  static constexpr int NP = ", num(ad.n_params > 0 ? ad.n_params : 1), ";\n"});
  for (int r = 0; r < in.n_regs; ++r) members += pw_cat({"  T r", num(r), "[4];\n"});
  std::string o = pw_prog_head(
      in, f64, "// A reversible-Heun adjoint program of torchsde_b200, generated by pw_adjoint_source\n", members,
      hoisted);
  o += "  __device__ __forceinline__ void fg(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
       "                                     T (&f)[4], T (&g)[4]) {\n";
  const std::pair<std::string, uint8_t> fg[2] = {{"f[j] = ", in.f_src}, {"g[j] = ", in.g_src}};
  o += pw_part(in, f64, hoisted, 0, in.n_fg, fg, 2, "tp");
  o += "  }\n  __device__ __forceinline__ void vjp(const PwOperands<T>& ops, const PwQuad& c, const T* tp,\n"
       "                                      const T (&y)[4], const T (&go)[4], const T (&go2)[4], T (&vz)[4],\n"
       "                                      T (&acc)[NP][4]) {\n";
  std::pair<std::string, uint8_t> results[1 + TSDE_PW_ADJ_MAX_PARAMS] = {{"vz[j] = ", in.gdg_src}};
  for (int k = 0; k < ad.n_params; ++k)
    results[1 + k] = {pw_cat({"acc[", num(k), "][j] = acc[", num(k), "][j] + "}), ad.param_src[k]};
  o += pw_part(in, f64, hoisted, in.n_fg, in.n_instr, results, 1 + ad.n_params, "tp");
  o += "  }\n";
  o += pw_unit_tail(kPwUnitAdjoint, f64);
  return o;
}

// ---- the general-noise programs (GENERAL launches) ------------------------------------------------------------------
// The two-program layout with per-channel values.  A g program runs m times per output, so it is compiled, never
// interpreted (an interpreted instruction costs about 30 SASS instructions, DESIGN §4): pw_general_source writes it
// out as a `Prog` for pw_general_euler_steps / pw_general_midpoint, or, by the program's tag, for pw_general_sra1
// (TSDE_PW_LAYOUT_GENERAL_SRA), pw_general_euler_heun (_EULER_HEUN) or pw_general_reversible_heun_steps
// (_REVERSIBLE_HEUN) (pw_device.cuh), with the IEEE options and the cache of the Milstein kernels.  A g
// instruction is per channel when one of its sources is (a DM or M operand, or a per-channel value); the others are
// per (row, d) element, evaluated once per lane before the channel loop.  The contraction of each lane's m values with
// the increments is written out for the route the unfused step takes (gen_route), as that kernel sums:
//   TSDE_GEN_ROWWISE   g * w                                       (the row-wise kernels' single product)
//   TSDE_GEN_TILE      per channel quad an fma chain from 0; the quad sums as the xor-butterfly adds them, a pairwise
//                      tree in natural order                       (gen_cta_kernel, gen_tma_kernel)
//   TSDE_GEN_GENERIC   left to right from 0, a rounded multiply and a rounded add per channel    (gen_kernel)
// (the sra1 launches never take the row-wise kernels: their m == 1 route is TSDE_GEN_GENERIC, pw_general_program).
// Register use stays bounded: m <= TSDE_PW_GENERAL_MAX_M increments per thread, and the tree keeps at most
// log2(m / 4) + 1 partial sums.

// Lane j's `acc`: the values val(k) of m channels contracted with the weights w[k] in the order of route `route`;
// pre(k) / post(k) are the statements before / after channel k's term.
static std::string pw_contraction(int route, int64_t m, bool f64, const std::function<std::string(int)>& val,
                                  const std::function<std::string(int)>& pre,
                                  const std::function<std::string(int)>& post) {
  const std::string fma = f64 ? "fma" : "fmaf";
  const int mq = (int)((m + 3) / 4);
  std::string s;
  if (route == TSDE_GEN_ROWWISE) {
    s += pw_cat({pre(0), "      const T acc = ", val(0), " * w[0];\n", post(0)});
  } else if (route == TSDE_GEN_GENERIC) {
    s += "      T acc = T(0);\n";
    for (int k = 0; k < m; ++k) s += pw_cat({pre(k), "      acc = acc + ", val(k), " * w[", num(k), "];\n", post(k)});
  } else {
    std::string level[TSDE_PW_GENERAL_MAX_M / 4];  // the partial sums of the tree's current level
    for (int q = 0; q < mq; ++q) {
      const std::string sq = pw_cat({"s", num(q)});
      const int k0 = 4 * q;
      s += pw_cat({pre(k0), "      T ", sq, " = ", fma, "(", val(k0), ", w[", num(k0), "], T(0));\n", post(k0)});
      for (int j = 1; j < 4; ++j)
        s += pw_cat({pre(k0 + j), "      ", sq, " = ", fma, "(", val(k0 + j), ", w[", num(k0 + j), "], ", sq, ");\n",
                     post(k0 + j)});
      level[q] = sq;
    }
    for (int l = 0, n = mq; n > 1; ++l, n /= 2) {
      for (int p = 0; p < n; p += 2) {
        const std::string a = pw_cat({"a", num(l), "_", num(p / 2)});
        s += pw_cat({"      const T ", a, " = ", level[p], " + ", level[p + 1], ";\n"});
        level[p / 2] = a;
      }
    }
    s += pw_cat({"      const T acc = ", level[0], ";\n"});
  }
  return s;
}

// The translation unit of a program that passed pw_general_program, for m channels and contraction `route`: the
// unit of its layout tag `layout` (Euler and midpoint kernels for TSDE_PW_LAYOUT_GENERAL).
static std::string pw_general_source(const tsde_pointwise& in, bool f64, int64_t m, int route, int layout) {
  const std::string M = num((int)m);
  const int mq = (int)((m + 3) / 4);
  bool hoisted[TSDE_PW_MAX_OPERANDS];
  pw_hoist(in, TSDE_PW_MAX_OPERANDS, hoisted);
  std::string members = pw_cat({"  static constexpr int MQ = ", num(mq), ";\n"});
  if (layout == TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN) members += pw_cat({"  static constexpr int M = ", M, ";\n"});
  std::string o = pw_prog_head(
      in, f64, "// An element-wise general-noise program of torchsde_b200, generated by pw_general_source\n", members,
      hoisted);
  // f: instructions [0, n_fg) on registers r<n>[4], as the Milstein kernels run them
  o += "  __device__ __forceinline__ void f(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
       "                                    T (&out)[4]) {\n    const T t0 = *tp;\n    (void)t0;\n";
  for (int r = 0; r < in.n_regs; ++r) o += pw_cat({"    T r", num(r), "[4];\n"});
  o += "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
  for (int i = 0; i < in.n_fg; ++i) {
    const tsde_pw_instr& x = in.instr[i];
    const std::string a = pw_value(in, x.a, hoisted, m), b = pw_unary(x.op) ? a : pw_value(in, x.b, hoisted, m);
    const std::string d = pw_cat({"r", num(x.dst), "[j]"});
    o += pw_cat({"      ", d, " = ", pw_expression(x, a, b, d, f64), ";\n"});
  }
  o += pw_cat({"      out[j] = ", pw_value(in, in.f_src, hoisted, m), ";\n    }\n  }\n"});
  // g: instruction i is n<i>[4] (per element, before the channel loop) or v<i> (per channel, inside G(k)); a register
  // names the instruction that last wrote it
  int def[TSDE_PW_MAX_REGS];
  bool wide[TSDE_PW_MAX_INSTR] = {};
  for (int r = 0; r < TSDE_PW_MAX_REGS; ++r) def[r] = -1;
  auto is_wide = [&](uint8_t s) {
    if (s == TSDE_PW_SRC_Y) return false;
    if (pw_operand_source(s)) return pw_per_channel_kind(in.operand[s - TSDE_PW_OPERAND(0)].kind);
    return wide[def[s]];
  };
  auto gsrc = [&](uint8_t s) -> std::string {
    if (s == TSDE_PW_SRC_Y || pw_operand_source(s)) return pw_value(in, s, hoisted, m);
    return wide[def[s]] ? "v" + num(def[s]) : pw_cat({"n", num(def[s]), "[j]"});
  };
  std::string narrow, per_channel;
  for (int i = in.n_fg; i < in.n_instr; ++i) {
    const tsde_pw_instr& x = in.instr[i];
    const bool sel = x.op == TSDE_PW_SEL;
    wide[i] = is_wide(x.a) || (!pw_unary(x.op) && is_wide(x.b)) || (sel && is_wide(x.dst));
    const std::string a = gsrc(x.a), b = pw_unary(x.op) ? a : gsrc(x.b), d = sel ? gsrc(x.dst) : "";
    if (wide[i])
      per_channel += pw_cat({"        const T v", num(i), " = ", pw_expression(x, a, b, d, f64), ";\n"});
    else
      narrow += pw_cat({"      n", num(i), "[j] = ", pw_expression(x, a, b, d, f64), ";\n"});
    def[x.dst] = i;
  }
  // the g program at (*tp, y), up to lane j's channel values G(k)
  std::string g_head = "    const T t0 = *tp;\n    (void)t0;\n";
  for (int i = in.n_fg; i < in.n_instr; ++i)
    if (!wide[i]) g_head += "    T n" + num(i) + "[4];\n";
  g_head += "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
  g_head += narrow;
  g_head += "    }\n#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n"
            "      const int64_t i = c.chan + (j < c.nvalid ? j : 0);  // (the d index of the lane; padding lanes read lane 0's)\n"
            "      (void)i;\n      auto G = [&](int k) -> T {\n        (void)k;\n";
  g_head += per_channel;
  g_head += "        return ";
  g_head += gsrc(in.g_src);
  g_head += ";\n      };\n";
  auto contraction = [&](auto val, auto pre, auto post) {
    return pw_contraction(route, m, f64, val, pre, post) + "      out[j] = acc;\n    }\n  }\n";
  };
  auto none = [](int) { return std::string(); };
  if (layout == TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN) {
    // the state's g values gs[j][k] stay in registers: z's contraction reads them, y's contracts (gs + g1) and leaves
    // g1 in their place (pw_general_reversible_heun_steps)
    o += "  template <typename Op>\n"
         "  __device__ __forceinline__ void dot(const Op& op, const T (&gs)[4][M], const T (&w)[4 * MQ], T (&out)[4]) {\n"
         "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
    o += contraction([&](int k) { return pw_cat({"op.gval(0, {gs[j][", num(k), "]})"}); }, none, none);
    o += "  template <typename Op>\n"
         "  __device__ __forceinline__ void gstep(const PwOperands<T>& ops, const PwQuad& c, const T* tp,\n"
         "                                        const T (&y)[4], const Op& op, const T (&w)[4 * MQ], T (&gs)[4][M],\n"
         "                                        T (&out)[4]) {\n";
    o += g_head;
    o += contraction([&](int k) { return pw_cat({"op.gval(0, {gs[j][", num(k), "], h", num(k), "})"}); },
                     [&](int k) { return pw_cat({"      const T h", num(k), " = G(", num(k), ");\n"}); },
                     [&](int k) { return pw_cat({"      gs[j][", num(k), "] = h", num(k), ";\n"}); });
  } else {
    o += "  __device__ __forceinline__ void gp(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
         "                                     const T (&w)[4 * MQ], T (&out)[4]) {\n";
    o += g_head;
    o += contraction([&](int k) { return pw_cat({"G(", num(k), ")"}); }, none, none);
  }
  o += pw_unit_tail(layout, f64);
  return o;
}

// ---- the general-noise adjoint (TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN) --------------------------------------
// What each instruction of a general adjoint program is, derived from its sources alone: per channel (`wide`: a DM or M
// operand, GO2 or a per-channel value is a source; a CSUM never is), and for a (rows, d) instruction of the vjp part,
// `late` when it reads a channel sum (it runs after the channel loop).  def_*: the instruction that last wrote a
// register source when the instruction runs (-1: not a register), dst_def that of SEL's condition; nidx: a forward
// (rows, d) instruction's index in the Prog's nn[][4] values.  res_def: the instruction of each result's register.
struct PwGAdjShape {
  int def_a[TSDE_PW_MAX_INSTR], def_b[TSDE_PW_MAX_INSTR], dst_def[TSDE_PW_MAX_INSTR], nidx[TSDE_PW_MAX_INSTR];
  bool wide[TSDE_PW_MAX_INSTR], late[TSDE_PW_MAX_INSTR];
  int nn;
  int f_def, g_def, vz_def, p_def[TSDE_PW_ADJ_MAX_PARAMS];
};

// (a range-for over a [begin, end) pair)
template <typename I>
struct PwRange {
  I b, e;
  I begin() const { return b; }
  I end() const { return e; }
};
template <typename I>
static PwRange<I> range(std::pair<I, I> p) {
  return {p.first, p.second};
}

// The shape of a program whose tables and ranges are valid; false if the layout cannot run it: a CSUM of a (rows, d)
// value or in the forward part, a per-channel instruction that reads a channel sum, f or vjp_z per channel.
static bool pw_gadj_shape(const tsde_pw_adjoint& ad, PwGAdjShape& sh) {
  const tsde_pointwise& in = ad.prog;
  int def[TSDE_PW_MAX_REGS];
  for (int r = 0; r < TSDE_PW_MAX_REGS; ++r) def[r] = -1;
  auto reg = [&](uint8_t s) { return s < TSDE_PW_MAX_REGS ? def[s] : -1; };
  auto wide = [&](uint8_t s, int d) {
    if (s == TSDE_PW_SRC_GO2) return true;
    if (pw_operand_source(s)) return pw_per_channel_kind(in.operand[s - TSDE_PW_OPERAND(0)].kind);
    return d >= 0 && sh.wide[d];
  };
  auto late = [&](int d) { return d >= 0 && sh.late[d]; };
  sh.nn = 0;
  for (int i = 0; i < in.n_instr; ++i) {
    const tsde_pw_instr& x = in.instr[i];
    const bool un = pw_unary(x.op) || x.op == TSDE_PW_CSUM, sel = x.op == TSDE_PW_SEL;
    sh.def_a[i] = reg(x.a);
    sh.def_b[i] = un ? -1 : reg(x.b);
    sh.dst_def[i] = sel ? def[x.dst] : -1;
    const bool wa = wide(x.a, sh.def_a[i]), wb = !un && wide(x.b, sh.def_b[i]), wc = sel && wide(x.dst, sh.dst_def[i]);
    const bool la = late(sh.def_a[i]), lb = late(sh.def_b[i]), lc = late(sh.dst_def[i]);
    if (x.op == TSDE_PW_CSUM) {
      if (i < in.n_fg || !wa) return false;
      sh.wide[i] = false;
      sh.late[i] = true;
    } else {
      sh.wide[i] = wa || wb || wc;
      if (sh.wide[i] && (la || lb || lc)) return false;
      sh.late[i] = !sh.wide[i] && (la || lb || lc);
    }
    sh.nidx[i] = i < in.n_fg && !sh.wide[i] ? sh.nn++ : -1;
    def[x.dst] = i;
    if (i + 1 == in.n_fg) {
      sh.f_def = reg(in.f_src);
      sh.g_def = reg(in.g_src);
    }
  }
  if (in.n_fg == 0) sh.f_def = sh.g_def = -1;
  sh.vz_def = reg(in.gdg_src);
  for (int k = 0; k < ad.n_params; ++k) sh.p_def[k] = reg(ad.param_src[k]);
  return !wide(in.f_src, sh.f_def) && !wide(in.gdg_src, sh.vz_def);
}

// The translation unit of a general adjoint program that passed pw_general_adjoint_program, for m channels and the
// contraction order `route` of the unfused kernels A and B.  Its Prog, for pw_general_adjoint_reversible_heun_steps:
//   fwd(ops, c, tp, y, nn, f)    the forward (rows, d) values at (*tp, y) into nn, and f
//   gk(ops, c, t0, y, nn, j, k)  g's channel k of lane j at (t0, y), from the (rows, d) values nn
//   vjp(...)                     kernel A's g0.dW and adj_g_mid, and the vjp, in one pass over the channels
//   ystep(...)                   kernel B's (g0 + g1).(0.5 dW), g0 at (t0, y0) and g1 at (t1, y1)
//   gstore(ops, c, tp, y, nn, g) g at (*tp, y), stored
// and pc(k): whether parameter k's contribution is per channel.
static std::string pw_general_adjoint_source(const tsde_pw_adjoint& ad, bool f64, int64_t m, int route) {
  const tsde_pointwise& in = ad.prog;
  PwGAdjShape sh;
  pw_gadj_shape(ad, sh);
  const std::string M = num((int)m);
  const int mq = (int)((m + 3) / 4), P = (int)(m >= 32 ? 32 : m >= 16 ? 16 : m >= 8 ? 8 : m >= 4 ? 4 : 2);
  bool hoisted[TSDE_PW_MAX_OPERANDS];
  pw_hoist(in, TSDE_PW_MAX_OPERANDS, hoisted);
  std::string members = pw_cat({"  static constexpr int M = ", M, ", MQ = ", num(mq), ", NN = ", num(sh.nn > 0 ? sh.nn : 1),
                                ", NP = ", num(ad.n_params > 0 ? ad.n_params : 1), ";\n"});
  // a contribution is per channel when its source is: a per-channel value, GO2 (a parameter that g broadcasts as it
  // is, S.expand) or a DM / M operand
  auto per_channel = [&](int p) {
    const uint8_t s = ad.param_src[p];
    if (s == TSDE_PW_SRC_GO2) return true;
    if (pw_operand_source(s)) return pw_per_channel_kind(in.operand[s - TSDE_PW_OPERAND(0)].kind);
    return sh.p_def[p] >= 0 && sh.wide[sh.p_def[p]];
  };
  std::string pc = "false";
  for (int k = 0; k < ad.n_params; ++k)
    if (per_channel(k)) pc += pw_cat({" || k == ", num(k)});
  members += pw_cat({"  __host__ __device__ static constexpr bool pc(int k) { return ", pc, "; }\n"});
  std::string o = pw_prog_head(
      in, f64, "// A general-noise reversible-Heun adjoint program of torchsde_b200, generated by pw_general_adjoint_source\n",
      members, hoisted);
  // source s (last written by instruction d) in lane j: a per-channel value v<d>, a forward (rows, d) value nn[][j], a
  // vjp one e<d>[j], the seeds, y or an operand (a DM / M one at the lane's d index i and channel k)
  auto src = [&](uint8_t s, int d) -> std::string {
    if (s == TSDE_PW_SRC_GO2) return "agm";
    if (s == TSDE_PW_SRC_Y || s == TSDE_PW_SRC_GO || pw_operand_source(s)) return pw_value(in, s, hoisted, m);
    if (sh.wide[d]) return "v" + num(d);
    if (d < in.n_fg) return pw_cat({"nn[", num(sh.nidx[d]), "][j]"});
    return pw_cat({"e", num(d), "[j]"});
  };
  auto expr = [&](int i) {
    const tsde_pw_instr& x = in.instr[i];
    const std::string a = src(x.a, sh.def_a[i]);
    const std::string b = pw_unary(x.op) ? a : src(x.b, sh.def_b[i]);
    return pw_expression(x, a, b, x.op == TSDE_PW_SEL ? src(x.dst, sh.dst_def[i]) : "", f64);
  };
  const std::string lane = "      const int64_t i = c.chan + (j < c.nvalid ? j : 0);  // (padding lanes read lane 0's)\n"
                           "      (void)i;\n";
  const std::string own = "(c.base + (j < c.nvalid ? j : 0)) * M + k";
  // per-channel forward values of channel k (in a scope that defines k)
  std::string fwd_wide;
  for (int i = 0; i < in.n_fg; ++i)
    if (sh.wide[i]) fwd_wide += pw_cat({"        const T v", num(i), " = ", expr(i), ";\n"});
  const std::string gval = src(in.g_src, sh.g_def);
  // fwd
  o += "  __device__ __forceinline__ void fwd(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
       "                                      T (&nn)[NN][4], T (&f)[4]) {\n    const T t0 = *tp;\n    (void)t0;\n"
       "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
  for (int i = 0; i < in.n_fg; ++i)
    if (!sh.wide[i]) o += pw_cat({"      nn[", num(sh.nidx[i]), "][j] = ", expr(i), ";\n"});
  o += pw_cat({"      f[j] = ", src(in.f_src, sh.f_def), ";\n    }\n  }\n"});
  // gk
  o += "  __device__ __forceinline__ T gk(const PwOperands<T>& ops, const PwQuad& c, const T t0, const T (&y)[4],\n"
       "                                  const T (&nn)[NN][4], const int j, const int k) {\n    (void)t0;\n"
       "    const int64_t i = c.chan + (j < c.nvalid ? j : 0);\n    (void)i;\n";
  o += fwd_wide;
  o += pw_cat({"    return ", gval, ";\n  }\n"});
  // vjp: per lane, the early (rows, d) ops, then the channels (A's contraction, adj_g_mid, the per-channel vjp ops,
  // the channel sums in ATen's order and the per-channel contributions), then the late (rows, d) ops
  o += "  __device__ __forceinline__ void vjp(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
       "                                      const T (&nn)[NN][4], const T (&w)[4 * MQ], const T (&wp)[4 * MQ],\n"
       "                                      const bool first, const T* gin, const T* ain, const T (&ay)[4],\n"
       "                                      const T (&ra)[4], const T (&rb)[4], const T (&go)[4], T (&zc)[4],\n"
       "                                      T (&vz)[4], T (&pacc)[NP][4], T* const (&part)[TSDE_PW_ADJ_MAX_PARAMS]) {\n"
       "    const T t0 = *tp;\n    (void)t0;\n";
  int csum_at[TSDE_PW_MAX_INSTR], n_csum = 0;
  for (int i = in.n_fg; i < in.n_instr; ++i) {
    if (!sh.wide[i]) o += pw_cat({"    T e", num(i), "[4];\n"});
    if (in.instr[i].op == TSDE_PW_CSUM) csum_at[n_csum++] = i;
  }
  const auto csums = [&]() { return std::pair<const int*, const int*>(csum_at, csum_at + n_csum); };
  o += "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n" + lane;
  for (int i = in.n_fg; i < in.n_instr; ++i)
    if (!sh.wide[i] && !sh.late[i]) o += pw_cat({"      e", num(i), "[j] = ", expr(i), ";\n"});
  for (int cs : range(csums()))
    for (int x = 0; x < P; ++x) o += pw_cat({"      T q", num(cs), "_0_", num(x), ";\n"});
  // ATen's sum over the last dimension (Reduce.cuh, for m <= 32 values per output): P = the largest power of two <= m
  // threads, thread x summing (0 + v_x) + (0 + v_{x+P}) (or 0 + v_x), the P sums then added as the shfl_down
  // butterfly adds them (offsets P/2, P/4, ..., 1: node (l, x) = (l-1, x) + (l-1, x + P/2^l)); emitted as each node
  // completes
  auto leaf_done = [&](int x) { return x + P < m ? x + P : x; };
  auto pre = [&](int k) {
    std::string s = pw_cat({"      T h", num(k), ";\n      {\n        const int k = ", num(k), ";\n"});
    s += fwd_wide;
    s += pw_cat({"        const T g0 = first ? gin[", own, "] : ", gval, ";\n"});
    s += pw_cat({"        const T adg = first ? ain[", own, "] : ra[j] * (T(0.5) * wp[", num(k), "]) + rb[j] * (T(-1) * wp[",
                 num(k), "]);\n"});
    s += pw_cat({"        const T agm = adg + ay[j] * (T(0.5) * w[", num(k), "]);\n        (void)agm;\n"});
    for (int i = in.n_fg; i < in.n_instr; ++i)
      if (sh.wide[i]) s += pw_cat({"        const T v", num(i), " = ", expr(i), ";\n"});
    for (int cs : range(csums())) {
      const std::string v = src(in.instr[cs].a, sh.def_a[cs]);
      if (k < P)
        s += pw_cat({"        q", num(cs), "_0_", num(k), " = T(0) + ", v, ";\n"});
      else
        s += pw_cat({"        q", num(cs), "_0_", num(k - P), " = q", num(cs), "_0_", num(k - P), " + (T(0) + ", v, ");\n"});
    }
    for (int p = 0; p < ad.n_params; ++p)
      if (per_channel(p))
        s += pw_cat({"        if (j < c.nvalid) {\n          T* const pp = part[", num(p), "] + (c.base + j) * M + k;\n"
                     "          *pp = *pp + ", src(ad.param_src[p], sh.p_def[p]), ";\n        }\n"});
    return s + pw_cat({"        h", num(k), " = g0;\n      }\n"});
  };
  auto post = [&](int k) {
    std::string s;
    for (int l = 1, n = P / 2; n >= 1; ++l, n /= 2)
      for (int x = 0; x < n; ++x) {
        int last = 0;  // (the node sums leaves x + i n, i < 2^l)
        for (int leaf = x; leaf < P; leaf += n) last = std::max(last, leaf_done(leaf));
        if (last != k) continue;
        for (int cs : range(csums()))
          s += pw_cat({"      const T q", num(cs), "_", num(l), "_", num(x), " = q", num(cs), "_", num(l - 1), "_",
                       num(x), " + q", num(cs), "_", num(l - 1), "_", num(x + n), ";\n"});
      }
    return s;
  };
  o += pw_contraction(route, m, f64, [&](int k) { return "h" + num(k); }, pre, post);
  o += "      zc[j] = acc;\n";
  int levels = 0;
  while ((1 << levels) < P) ++levels;
  for (int cs : range(csums())) o += pw_cat({"      e", num(cs), "[j] = q", num(cs), "_", num(levels), "_0;\n"});
  for (int i = in.n_fg; i < in.n_instr; ++i)
    if (sh.late[i] && in.instr[i].op != TSDE_PW_CSUM) o += pw_cat({"      e", num(i), "[j] = ", expr(i), ";\n"});
  o += pw_cat({"      vz[j] = ", src(in.gdg_src, sh.vz_def), ";\n"});
  for (int p = 0; p < ad.n_params; ++p)
    if (!per_channel(p))
      o += pw_cat({"      pacc[", num(p), "][j] = pacc[", num(p), "][j] + ", src(ad.param_src[p], sh.p_def[p]), ";\n"});
  o += "    }\n  }\n";
  // ystep
  o += "  __device__ __forceinline__ void ystep(const PwOperands<T>& ops, const PwQuad& c, const T* tp0, const T (&y0)[4],\n"
       "                                        const T (&n0)[NN][4], const T* tp1, const T (&y1)[4], const T (&n1)[NN][4],\n"
       "                                        const T (&w)[4 * MQ], const bool first, const T* gin, T (&out)[4]) {\n"
       "    const T ta = *tp0, tb = *tp1;\n#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n";
  o += pw_contraction(
      route, m, f64, [&](int k) { return "h" + num(k); },
      [&](int k) {
        const std::string K = num(k);
        return pw_cat({"      const T h", K, " = (first ? gin[(c.base + (j < c.nvalid ? j : 0)) * M + ", K,
                       "] : gk(ops, c, ta, y0, n0, j, ", K, ")) + gk(ops, c, tb, y1, n1, j, ", K, ");\n"});
      },
      [](int) { return std::string(); });
  o += "      out[j] = acc;\n    }\n  }\n";
  // gstore
  o += "  __device__ __forceinline__ void gstore(const PwOperands<T>& ops, const PwQuad& c, const T* tp, const T (&y)[4],\n"
       "                                         const T (&nn)[NN][4], T* g) {\n    const T t0 = *tp;\n"
       "#pragma unroll\n    for (int j = 0; j < 4; ++j) {\n      if (j >= c.nvalid) continue;\n"
       "#pragma unroll\n      for (int k = 0; k < M; ++k) g[(c.base + j) * M + k] = gk(ops, c, t0, y, nn, j, k);\n"
       "    }\n  }\n";
  o += pw_unit_tail(kPwUnitGeneralAdjoint, f64);
  return o;
}

// ---- NVRTC --------------------------------------------------------------------------------------------------------
// libnvrtc.so.12 is opened the first time a program is compiled, not linked: the library loads where NVRTC is missing
// (and every other entry point works there).  torchsde_b200/_cabi.py preloads it from the nvidia-cuda-nvrtc package
// that PyTorch installs.
struct Nvrtc {
  decltype(&nvrtcCreateProgram) create;
  decltype(&nvrtcCompileProgram) compile;
  decltype(&nvrtcGetProgramLogSize) log_size;
  decltype(&nvrtcGetProgramLog) log;
  decltype(&nvrtcGetCUBINSize) cubin_size;
  decltype(&nvrtcGetCUBIN) cubin;
  decltype(&nvrtcDestroyProgram) destroy;
  decltype(&nvrtcGetErrorString) error;
};

static const Nvrtc* nvrtc() {
  static const Nvrtc* api = []() -> const Nvrtc* {
    void* h = dlopen("libnvrtc.so.12", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return nullptr;
    static Nvrtc n;
    bool ok = true;
    auto sym = [&](auto& fn, const char* name) {
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
      ok = ok && fn;
    };
    sym(n.create, "nvrtcCreateProgram");
    sym(n.compile, "nvrtcCompileProgram");
    sym(n.log_size, "nvrtcGetProgramLogSize");
    sym(n.log, "nvrtcGetProgramLog");
    sym(n.cubin_size, "nvrtcGetCUBINSize");
    sym(n.cubin, "nvrtcGetCUBIN");
    sym(n.destroy, "nvrtcDestroyProgram");
    sym(n.error, "nvrtcGetErrorString");
    return ok ? &n : nullptr;
  }();
  return api;
}

// NVRTC has no <stdint.h>
static const char kPwStdint[] =
    "#pragma once\n"
    "typedef signed char int8_t; typedef short int16_t; typedef int int32_t; typedef long long int64_t;\n"
    "typedef unsigned char uint8_t; typedef unsigned short uint16_t; typedef unsigned int uint32_t;\n"
    "typedef unsigned long long uint64_t; typedef unsigned long long uintptr_t;\n";

static std::mutex g_pw_error_mu;
static std::string g_pw_error;  // why the last compilation failed (tsde_error_string(TSDE_ECOMPILE))

static int pw_compile_failed(const std::string& why) {
  std::lock_guard<std::mutex> lock(g_pw_error_mu);
  g_pw_error = "torchsde_b200: the element-wise Milstein program could not be compiled: " + why;
  return TSDE_ECOMPILE;
}

std::string pw_compile_error() {
  std::lock_guard<std::mutex> lock(g_pw_error_mu);
  return g_pw_error;
}

// The sm_90a cubin of `source`, or TSDE_ECOMPILE with the compiler's log.  `rdc`: a relocatable cubin, for nvJitLink;
// `fmad`: FMA contraction on (kPwHelpers only)
static int pw_nvrtc(const std::string& source, std::string& cubin, bool rdc = false, bool fmad = false) {
  const Nvrtc* nv = nvrtc();
  if (!nv) return pw_compile_failed("libnvrtc.so.12 (NVRTC) was not found");
  const char* names[kPwHeaderCount + 1];
  const char* bodies[kPwHeaderCount + 1];
  for (int i = 0; i < kPwHeaderCount; ++i) {
    names[i] = kPwHeaderNames[i];
    bodies[i] = kPwHeaderSources[i];
  }
  names[kPwHeaderCount] = "stdint.h";
  bodies[kPwHeaderCount] = kPwStdint;
  nvrtcProgram prog;
  nvrtcResult r = nv->create(&prog, source.c_str(), "tsde_pw_milstein.cu", kPwHeaderCount + 1, bodies, names);
  if (r != NVRTC_SUCCESS) return pw_compile_failed(nv->error(r));
  // straight to SASS (no PTX for the driver to JIT); the public header's declarations are host functions, which NVRTC
  // refuses unless unannotated functions are taken as device ones
  const char* opts[] = {"-arch=sm_90a", "-std=c++17", fmad ? "-fmad=true" : "-fmad=false", "-prec-div=true",
                        "-prec-sqrt=true", "-ftz=false", "-default-device", "-rdc=true"};
  r = nv->compile(prog, (int)(sizeof(opts) / sizeof(opts[0])) - (rdc ? 0 : 1), opts);
  std::string log;
  size_t n = 0;
  if (nv->log_size(prog, &n) == NVRTC_SUCCESS && n > 1) {
    log.resize(n);
    nv->log(prog, &log[0]);
    log.resize(n - 1);
  }
  if (r == NVRTC_SUCCESS && nv->cubin_size(prog, &n) == NVRTC_SUCCESS) {
    cubin.resize(n);
    r = nv->cubin(prog, &cubin[0]);
  }
  nv->destroy(&prog);
  if (r != NVRTC_SUCCESS) return pw_compile_failed(std::string(nv->error(r)) + "\n" + log);
  return 0;
}

// nvJitLink, opened like NVRTC when the first program with a transcendental op is linked (torchsde_b200/_cabi.py's
// nvjitlink() preloads it from the nvidia-nvjitlink package PyTorch installs when such an op is recorded).  Its entry points are versioned; the 12.0 ones are in
// every CUDA 12 release.
struct NvJitLink {
  typedef int (*Create)(void** h, uint32_t n, const char** opts);
  typedef int (*AddData)(void* h, int kind, const void* data, size_t size, const char* name);
  typedef int (*Handle)(void* h);
  typedef int (*Size)(void* h, size_t* n);
  typedef int (*Get)(void* h, void* out);
  typedef int (*Destroy)(void** h);
  Create create;
  AddData add;
  Handle complete;
  Size cubin_size, log_size;
  Get cubin, log;
  Destroy destroy;
};

static const NvJitLink* nvjitlink() {
  static const NvJitLink* api = []() -> const NvJitLink* {
    void* h = dlopen("libnvJitLink.so.12", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return nullptr;
    static NvJitLink n;
    bool ok = true;
    auto sym = [&](auto& fn, const char* name) {
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
      ok = ok && fn;
    };
    sym(n.create, "__nvJitLinkCreate_12_0");
    sym(n.add, "__nvJitLinkAddData_12_0");
    sym(n.complete, "__nvJitLinkComplete_12_0");
    sym(n.cubin_size, "__nvJitLinkGetLinkedCubinSize_12_0");
    sym(n.cubin, "__nvJitLinkGetLinkedCubin_12_0");
    sym(n.log_size, "__nvJitLinkGetErrorLogSize_12_0");
    sym(n.log, "__nvJitLinkGetErrorLog_12_0");
    sym(n.destroy, "__nvJitLinkDestroy_12_0");
    return ok ? &n : nullptr;
  }();
  return api;
}

// The sm_90a cubin of program `source`, which calls kPwHelpers: both compiled relocatable and linked without LTO.
static int pw_nvrtc_linked(const std::string& source, std::string& cubin) {
  static std::string helpers;  // (compiled once; callers hold pw_loaded's lock)
  if (helpers.empty())
    if (int e = pw_nvrtc(kPwHelpers, helpers, true, true)) return e;
  std::string prog;
  if (int e = pw_nvrtc(source, prog, true)) return e;
  const NvJitLink* nj = nvjitlink();
  if (!nj) return pw_compile_failed("libnvJitLink.so.12 (nvJitLink) was not found");
  const int kCubin = 1;  // NVJITLINK_INPUT_CUBIN
  const char* opts[] = {"-arch=sm_90a"};
  void* h = nullptr;
  if (nj->create(&h, 1, opts) != 0) return pw_compile_failed("nvJitLinkCreate failed");
  int r = nj->add(h, kCubin, prog.data(), prog.size(), "program");
  if (r == 0) r = nj->add(h, kCubin, helpers.data(), helpers.size(), "helpers");
  if (r == 0) r = nj->complete(h);
  size_t n = 0;
  if (r == 0) r = nj->cubin_size(h, &n);
  if (r == 0) {
    cubin.resize(n);
    r = nj->cubin(h, &cubin[0]);
  }
  std::string log;
  if (r != 0 && nj->log_size(h, &n) == 0 && n > 1) {
    log.resize(n);
    nj->log(h, &log[0]);
    log.resize(n - 1);
  }
  nj->destroy(&h);
  if (r != 0) return pw_compile_failed("nvJitLink error " + num(r) + "\n" + log);
  return 0;
}

struct PwCompiled {
  cudaKernel_t kernel[2][2];  // [the unit's kernel][its multi-cell variant] (kPwUnits; a kernel without: [k][0])
};

// The kernels of unit `unit` of `source`, compiled and loaded on first use.  Libraries are context-independent: one
// entry serves every device.  A program of `prog` with a transcendental op is linked with kPwHelpers.
static int pw_loaded(const tsde_pointwise& prog, int unit, std::string source, PwCompiled& out) {
  static std::mutex mu;
  static std::map<std::string, PwCompiled> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(source);
  if (it != cache.end()) {
    out = it->second;
    return 0;
  }
  bool link = false;
  for (int i = 0; i < prog.n_instr; ++i) link = link || pw_transcendental(prog.instr[i].op);
  std::string cubin;
  if (int e = link ? pw_nvrtc_linked(source, cubin) : pw_nvrtc(source, cubin)) return e;
  cudaLibrary_t lib;
  cudaError_t e = cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  const bool loaded = e == cudaSuccess;
  for (int i = 0; i < 2; ++i) {
    const PwKernelText& k = kPwUnits[unit].kernel[i];
    for (int multi = 0; k.name && multi < (k.cells ? 2 : 1) && e == cudaSuccess; ++multi)
      e = cudaLibraryGetKernel(&out.kernel[i][multi], lib,
                               (std::string(k.name) + (k.cells ? kPwCellSuffix[multi] : "")).c_str());
  }
  if (e != cudaSuccess && loaded) cudaLibraryUnload(lib);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return (int)e;
  }
  cache.emplace(std::move(source), out);
  return 0;
}

// The Milstein layout, in the order the kernel reads it: go exists from the vjp part on, registers carry over.
static bool pw_valid_milstein(const tsde_pointwise& pg) {
  uint64_t written = 0;
  return pw_valid_range(pg, 0, pg.n_fg, false, written, true) &&
         pw_valid_source(pg, pg.f_src, false, written) && pw_valid_source(pg, pg.g_src, false, written) &&
         pw_valid_range(pg, pg.n_fg, pg.n_instr, true, written, true) &&
         pw_valid_source(pg, pg.gdg_src, true, written);
}

// ---- a whole SRK step (tsde_step_srk_diag_pointwise) ----------------------------------------------------------------
// W and U are drawn, y0 is read, and the seven SDE evaluations (the f program at three (t, y), the g program at four)
// alternate with the unfused step's own stage ops.  y0 and y1 are the only tensors the step moves, against 22 reads
// and 6 writes of the unfused step (41 with f and g).
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
  int slot0;  // first slot past the program's layout (PwProg::end)
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
      pw_sload(regs, slot0 + k, threadIdx.x, x);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = r[k][j];
    }
  }
};

// One SDE evaluation of the two-program layout (SRK, predictor-corrector): f (program [0, n_fg), result f_src) or g
// (program [n_fg, n_instr), result g_src) at (t, y)
template <bool EXT, typename T>
__device__ __forceinline__ void pw_eval(const PwProg<T>& pg, const PwQuad& c, void* regs, bool g, const T* t,
                                        const T (&y)[4], T (&out)[4]) {
  pw_set_state(pg, regs, t, y);
  pw_run<EXT>(pg, c, regs, g ? pg.n_fg : 0, g ? pg.n_instr : pg.n_fg);
  pw_fetch<true, EXT>(pg, c, regs, g ? pg.g_src : pg.f_src, out);
}

// One SRK step from y0 on the increments (w, u) at the stage times t[4] with the stage ops of the step: y1
template <bool EXT, typename T>
__device__ __forceinline__ void pw_srk_step(const PwProg<T>& pg, const PwQuad& c, void* pw_regs,
                                            const T* const (&t)[4], const SrkDiagStage1Op<T>& s1,
                                            const SrkDiagStage2Op<T>& s2, const SrkDiagStage3Op<T>& s3,
                                            const SrkDiagFinalOp<T>& fin, const T (&w)[4], const T (&u)[4],
                                            const T (&y0)[4], T (&y1)[4]) {
  PwSrkStash<T> st;
  st.slot0 = pg.end;
  enum { F0, F1, F2, G0, G1, G2 };
  T f[4], g[4], h0[4], h1[4], x[4], z[4];
  // s = 0: f0, g0 at (t0, y0); H0_1, H1_1
  pw_eval<EXT>(pg, c, pw_regs, false, t[0], y0, f);
  pw_eval<EXT>(pg, c, pw_regs, true, t[0], y0, g);
  st.put(pw_regs, F0, f);
  st.put(pw_regs, G0, g);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[2];
    s1({y0[j], f[j], g[j]}, w[j], u[j], o);
    h0[j] = o[0];
    h1[j] = o[1];
  }
  // s = 1: f1 at (t0 + dt, H0_1), g1 at (t0 + dt/4, H1_1); H0_2, H1_2
  pw_eval<EXT>(pg, c, pw_regs, false, t[1], h0, f);
  pw_eval<EXT>(pg, c, pw_regs, true, t[2], h1, g);
  st.put(pw_regs, F1, f);
  st.put(pw_regs, G1, g);
  st.get(pw_regs, F0, x);
  st.get(pw_regs, G0, z);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[2];
    s2({y0[j], x[j], z[j], f[j], g[j]}, w[j], u[j], o);
    h0[j] = o[0];
    h1[j] = o[1];
  }
  // s = 2: f2 at (t0 + dt/2, H0_2), g2 at (t0 + dt, H1_2); H1_3
  pw_eval<EXT>(pg, c, pw_regs, false, t[3], h0, f);
  pw_eval<EXT>(pg, c, pw_regs, true, t[1], h1, g);
  st.put(pw_regs, F2, f);
  st.put(pw_regs, G2, g);
  st.get(pw_regs, G0, x);
  st.get(pw_regs, G1, z);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    s3({y0[j], x[j], z[j], f[j], g[j]}, w[j], u[j], o);
    h1[j] = o[0];
  }
  // s = 3: g3 at (t0 + dt/4, H1_3); y1
  pw_eval<EXT>(pg, c, pw_regs, true, t[2], h1, g);
  T f0[4], f1[4], f2[4], g0[4], g1[4], g2[4];
  st.get(pw_regs, F0, f0);
  st.get(pw_regs, F1, f1);
  st.get(pw_regs, F2, f2);
  st.get(pw_regs, G0, g0);
  st.get(pw_regs, G1, g1);
  st.get(pw_regs, G2, g2);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    fin({y0[j], f0[j], f1[j], f2[j], g0[j], g1[j], g2[j], g[j]}, w[j], u[j], o);
    y1[j] = o[0];
  }
}

template <typename T, int SRC, bool EXT>
__device__ __forceinline__ void pw_srk(const PwProg<T>& pg, const PwSrkP<T> p, const NoiseP<T> nz) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  PwQuad c;
  T w[4], u[4], y0[4], y1[4];
  if (!pw_begin<T, SRC, true>(pg, p.base, nz, pw_regs, c, w, u, y0)) return;
  pw_srk_step<EXT>(pg, c, pw_regs, p.t, p.s1, p.s2, p.s3, p.fin, w, u, y0, y1);
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, y1);
}

template <typename T, int SRC>
__global__ void __launch_bounds__(kThreads)
pw_srk_kernel(const __grid_constant__ PwProg<T> pg, const PwSrkP<T> p, const NoiseP<T> nz) {
  pw_srk<T, SRC, false>(pg, p, nz);
}
template <typename T, int SRC>
__global__ void __launch_bounds__(kThreads)
pw_srk_ext_kernel(const __grid_constant__ PwProg<T> pg, const PwSrkP<T> p, const NoiseP<T> nz) {
  pw_srk<T, SRC, true>(pg, p, nz);
}

// The two-program layout (SRK, predictor-corrector): an f program and a g program that each start with no register
// defined; go is never a source.  At most MAX_REGS registers: SRK keeps the ones past TSDE_PW_SRK_MAX_REGS for its
// stash.  COMPILED: the layout's kernels are compiled (the general layouts), not interpreted.
template <int MAX_REGS, bool COMPILED = false>
static bool pw_valid_two(const tsde_pointwise& pg) {
  if (pg.n_regs > MAX_REGS) return false;
  uint64_t written = 0;
  if (!pw_valid_range(pg, 0, pg.n_fg, false, written, COMPILED) || !pw_valid_source(pg, pg.f_src, false, written))
    return false;
  written = 0;
  return pw_valid_range(pg, pg.n_fg, pg.n_instr, false, written, COMPILED) &&
         pw_valid_source(pg, pg.g_src, false, written);
}

// ---- a whole Heun, midpoint or Euler-Heun step (tsde_step_predictor_corrector_pointwise) ----------------------------
// W is drawn, y0 is read, f0 and g0 are evaluated at (t0, y0), the method's predictor forms y', the second evaluation
// runs at (t_p, y') (g only for Euler-Heun) and the method's final op writes y1: the unfused step's own ops with the
// scalars its kernels take, so the step equals the unfused one bit for bit.  Five quads are live at most (y0, W, f0,
// g0, y'), which fits registers in fp64 too: no stash.  The minimum of one resident CTA in the launch bounds lets
// ptxas keep them there; without it, it caps some instantiations at 64 or 80 registers and spills.
template <typename T>
struct PwPcP {
  PwP<T> base;   // y0, y1, the quad mapping, t0 and dt
  const T* t_p;  // the time of the second evaluation
  T half_dt;
};

// One predictor-corrector step of METHOD from y0 on the increment w, evaluated at t0 and t_p: y1
template <int METHOD, bool EXT, typename T>
__device__ __forceinline__ void pw_pc_step(const PwProg<T>& pg, const PwQuad& c, void* pw_regs, const T* t0,
                                           const T* t_p, T dt, T half_dt, const T (&w)[4], const T (&y0)[4],
                                           T (&y1)[4]) {
  const T u[4] = {};  // (the ops take no U)
  T f0[4], g0[4], yp[4];
  pw_eval<EXT>(pg, c, pw_regs, false, t0, y0, f0);
  pw_eval<EXT>(pg, c, pw_regs, true, t0, y0, g0);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    if constexpr (METHOD == TSDE_PC_HEUN) {
      EulerOp<T>{dt}({y0[j], f0[j], g0[j]}, w[j], u[j], o);                  // heun.py:42
    } else if constexpr (METHOD == TSDE_PC_MIDPOINT) {
      MidpointPredictOp<T>{half_dt}({y0[j], f0[j], g0[j]}, w[j], u[j], o);    // midpoint.py:38
    } else {
      EulerHeunPredictOp<T>{}({y0[j], g0[j]}, w[j], u[j], o);                // euler_heun.py:36
    }
    yp[j] = o[0];
  }
  T f[4], g[4];
  if constexpr (METHOD != TSDE_PC_EULER_HEUN) pw_eval<EXT>(pg, c, pw_regs, false, t_p, yp, f);
  pw_eval<EXT>(pg, c, pw_regs, true, t_p, yp, g);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T o[1];
    if constexpr (METHOD == TSDE_PC_HEUN) {
      HeunOp<T>{dt}({y0[j], f0[j], f[j], g0[j], g[j]}, w[j], u[j], o);       // heun.py:46
    } else if constexpr (METHOD == TSDE_PC_MIDPOINT) {
      EulerOp<T>{dt}({y0[j], f[j], g[j]}, w[j], u[j], o);                    // midpoint.py:43
    } else {
      EulerHeunOp<T>{dt}({y0[j], f0[j], g0[j], g[j]}, w[j], u[j], o);        // euler_heun.py:40
    }
    y1[j] = o[0];
  }
}

template <typename T, int SRC, int METHOD, bool EXT>
__device__ __forceinline__ void pw_pc(const PwProg<T>& pg, const PwPcP<T> p, const NoiseP<T> nz) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  PwQuad c;
  T w[4], u[4], y0[4], y1[4];
  if (!pw_begin<T, SRC, false>(pg, p.base, nz, pw_regs, c, w, u, y0)) return;
  pw_pc_step<METHOD, EXT>(pg, c, pw_regs, p.base.t0, p.t_p, p.base.dt, p.half_dt, w, y0, y1);
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, y1);
}

template <typename T, int SRC, int METHOD>
__global__ void __launch_bounds__(kThreads, 1)
pw_pc_kernel(const __grid_constant__ PwProg<T> pg, const PwPcP<T> p, const NoiseP<T> nz) {
  pw_pc<T, SRC, METHOD, false>(pg, p, nz);
}
template <typename T, int SRC, int METHOD>
__global__ void __launch_bounds__(kThreads, 1)
pw_pc_ext_kernel(const __grid_constant__ PwProg<T> pg, const PwPcP<T> p, const NoiseP<T> nz) {
  pw_pc<T, SRC, METHOD, true>(pg, p, nz);
}

// ---- consecutive Euler or reversible-Heun steps (tsde_solve_euler_pointwise, tsde_solve_reversible_heun_pointwise) --
// The chunked loop of pw_milstein_kernel around the two-program layout: one thread runs up to kPwMaxSteps steps of
// its quad, draws step j's increment from st.s[j].cell, and stores y1 only where st.s[j].y1 is given.  Per step:
//   Euler            f, g at (t, y);  y <- EulerOp{dt}                                       (euler.py:36)
//   reversible Heun  z1 = RevHeunZOp{dt}(y, z, f, g);  f1, g1 at (t, z1);
//                    y1 = RevHeunOp{dt/2}(y, f, f1, g, g1);  (y, z, f, g) <- (y1, z1, f1, g1) (reversible_heun.py:69-71)
// where t is st.s[j].t0, the time the program runs at: the step's t0 for Euler, its t1 for reversible Heun.  dt/2 is
// T(0.5) * dt, which equals the host-rounded (T)(0.5 * dt) of the unfused step whenever that is a normal number (the
// caller checks).  Reversible Heun's solver state (z, f, g) is read once at the chunk's start and stored once at its
// end, to pointers the chunk does not read: its whole state stays in registers in between.
enum { kPwEuler = 0, kPwReversibleHeun = 1 };

template <typename T>
struct PwChunkP {
  PwP<T> base;           // y0, the quad mapping (base.y1, t0, dt and ito unused: the step table has them)
  const T *z0, *f0, *g0;  // reversible Heun: the solver state the chunk starts from
  T *z1, *f1, *g1;        // and where the chunk leaves it
};
static_assert(sizeof(PwProg<double>) + sizeof(PwChunkP<double>) + sizeof(NoiseP<double>) + sizeof(PwSteps<double>) <=
                  4096,
              "the chunk kernel's parameters fit the 4 KiB parameter space");

template <typename T, int SRC, int METHOD, bool EXT>
__device__ __forceinline__ void pw_chunk_steps(const PwProg<T>& pg, const PwChunkP<T> p, const NoiseP<T> nz,
                                               const PwSteps<T>& st) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  const Key key = load_key(nz.key);
  T y[4], z[4], f[4], g[4];
  for (int j = 0; j < st.n; ++j) {
    const PwStep<T>& s = st.s[j];
    T w[4], u[4];
    NoiseP<T> n = nz;  // this step's cell
    n.cell_id = s.cell;
    n.sqrt_h = s.sqrt_h;
    quad_noise<T, SRC, false>(n, key, row, q, c.vec, c.nvalid, w, u);
    if (j == 0) {  // the first increment is drawn while the previous kernel drains; the rest is read after the wait
      asm volatile("griddepcontrol.wait;" ::: "memory");
      pw_load_uniform(pg, pw_regs);
      if (Q >= p.base.nquads) return;
      load_quad(p.base.y0, c.base, c.vec, c.nvalid, y);
      if constexpr (METHOD == kPwReversibleHeun) {
        load_quad(p.z0, c.base, c.vec, c.nvalid, z);
        load_quad(p.f0, c.base, c.vec, c.nvalid, f);
        load_quad(p.g0, c.base, c.vec, c.nvalid, g);
      }
      pw_load_hoisted(pg, c, pw_regs);
    }
    if constexpr (METHOD == kPwEuler) {
      pw_eval<EXT>(pg, c, pw_regs, false, s.t0, y, f);
      pw_eval<EXT>(pg, c, pw_regs, true, s.t0, y, g);
      const EulerOp<T> step{s.dt};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        T o[1];
        step({y[i], f[i], g[i]}, w[i], u[i], o);
        y[i] = o[0];
      }
    } else {
      const RevHeunZOp<T> zop{s.dt};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        T o[1];
        zop({y[i], z[i], f[i], g[i]}, w[i], u[i], o);
        z[i] = o[0];
      }
      T f1[4], g1[4];
      pw_eval<EXT>(pg, c, pw_regs, false, s.t0, z, f1);
      pw_eval<EXT>(pg, c, pw_regs, true, s.t0, z, g1);
      const RevHeunOp<T> step{T(0.5) * s.dt};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        T o[1];
        step({y[i], f[i], f1[i], g[i], g1[i]}, w[i], u[i], o);
        y[i] = o[0];
        f[i] = f1[i];
        g[i] = g1[i];
      }
    }
    if (s.y1) store_quad(s.y1, c.base, c.vec, c.nvalid, y);
  }
  if constexpr (METHOD == kPwReversibleHeun) {
    store_quad(p.z1, c.base, c.vec, c.nvalid, z);
    store_quad(p.f1, c.base, c.vec, c.nvalid, f);
    store_quad(p.g1, c.base, c.vec, c.nvalid, g);
  }
}

template <typename T, int SRC, int METHOD>
__global__ void __launch_bounds__(kThreads, 1)
pw_chunk_kernel(const __grid_constant__ PwProg<T> pg, const PwChunkP<T> p, const NoiseP<T> nz,
                const __grid_constant__ PwSteps<T> st) {
  pw_chunk_steps<T, SRC, METHOD, false>(pg, p, nz, st);
}
template <typename T, int SRC, int METHOD>
__global__ void __launch_bounds__(kThreads, 1)
pw_chunk_ext_kernel(const __grid_constant__ PwProg<T> pg, const PwChunkP<T> p, const NoiseP<T> nz,
                    const __grid_constant__ PwSteps<T> st) {
  pw_chunk_steps<T, SRC, METHOD, true>(pg, p, nz, st);
}

// ---- an adaptive solve's proposal (tsde_adaptive_proposal_pointwise) ------------------------------------------------
// The full step and the two half steps of Euler, SRK or a predictor-corrector method, each the step body of the
// method's own kernel above, on increments read from memory (pw_milstein_proposal in pw_device.cuh is Milstein's).
template <typename T>
struct PwSrkOps {  // the stage ops of one SRK sub-step
  SrkDiagStage1Op<T> s1;
  SrkDiagStage2Op<T> s2;
  SrkDiagStage3Op<T> s3;
  SrkDiagFinalOp<T> fin;
};

template <typename T>
struct PwProposalP {
  PwP<T> base;  // y0, y1 (y_full), the quad mapping
  T* y_next;
  PwSubs<T> st;
  PwSrkOps<T> srk[3];  // (SRK only)
};

// Sub-step k from y0: y1
template <int METHOD, bool EXT, typename T>
__device__ __forceinline__ void pw_sub_step(const PwProg<T>& pg, const PwQuad& c, void* pw_regs,
                                            const PwProposalP<T>& p, int k, const T (&y0)[4], T (&y1)[4]) {
  const PwSub<T>& s = p.st.sub[k];
  T w[4];
  load_quad(s.w, c.base, c.vec, c.nvalid, w);
  if constexpr (METHOD == TSDE_PROPOSAL_SRK) {
    T u[4];
    load_quad(s.u, c.base, c.vec, c.nvalid, u);
    const PwSrkOps<T>& o = p.srk[k];
    pw_srk_step<EXT>(pg, c, pw_regs, s.t, o.s1, o.s2, o.s3, o.fin, w, u, y0, y1);
  } else if constexpr (METHOD == TSDE_PROPOSAL_EULER) {
    // (pw_chunk_steps' Euler step)
    T f[4], g[4];
    pw_eval<EXT>(pg, c, pw_regs, false, s.s.t0, y0, f);
    pw_eval<EXT>(pg, c, pw_regs, true, s.s.t0, y0, g);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      T o[1];
      EulerOp<T>{s.s.dt}({y0[j], f[j], g[j]}, w[j], T(0), o);
      y1[j] = o[0];
    }
  } else {
    constexpr int PC = METHOD == TSDE_PROPOSAL_HEUN       ? TSDE_PC_HEUN
                       : METHOD == TSDE_PROPOSAL_MIDPOINT ? TSDE_PC_MIDPOINT
                                                          : TSDE_PC_EULER_HEUN;
    pw_pc_step<PC, EXT>(pg, c, pw_regs, s.s.t0, s.t[1], s.s.dt, s.half_dt, w, y0, y1);
  }
}

template <typename T, int METHOD, bool EXT>
__device__ __forceinline__ void pw_proposal(const PwProg<T>& pg, const PwProposalP<T>& p) {
  extern __shared__ __align__(16) unsigned char pw_regs[];
  PwQuad c;
  int64_t Q, row, q;
  pw_locate(p.base, c, Q, row, q);
  // the increments are the Brownian queries that precede the launch: everything is read after the wait
  asm volatile("griddepcontrol.wait;" ::: "memory");
  pw_load_uniform(pg, pw_regs);
  if (Q >= p.base.nquads) return;
  T y0[4], y[4], ym[4];
  load_quad(p.base.y0, c.base, c.vec, c.nvalid, y0);
  pw_load_hoisted(pg, c, pw_regs);
  pw_sub_step<METHOD, EXT>(pg, c, pw_regs, p, 0, y0, y);
  store_quad(p.base.y1, c.base, c.vec, c.nvalid, y);
  pw_sub_step<METHOD, EXT>(pg, c, pw_regs, p, 1, y0, ym);
  pw_sub_step<METHOD, EXT>(pg, c, pw_regs, p, 2, ym, y);
  store_quad(p.y_next, c.base, c.vec, c.nvalid, y);
}

template <typename T, int METHOD, bool EXT>
__global__ void __launch_bounds__(kThreads, 1)
pw_proposal_kernel(const __grid_constant__ PwProg<T> pg, const __grid_constant__ PwProposalP<T> p) {
  pw_proposal<T, METHOD, EXT>(pg, p);
}
static_assert(sizeof(PwProg<double>) + sizeof(PwProposalP<double>) <= 4096,
              "the proposal kernel's parameters fit the 4 KiB parameter space");

// ---- launch ---------------------------------------------------------------------------------------------------------
// What every launch of a step program checks and fills before anything is compiled or launched: counter noise without
// flags (np), y0, and the part of the kernel parameters every pointwise step has (y0, y1, the quad mapping, vec for
// y0, y1 and the program's CHANNEL / ROW operands).  y1 is null for a chunk, whose step table holds the destinations
// (pw_steps).  `prog` has passed its layout's validation.
template <typename T>
static int pw_fill(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise& prog, const void* y0, void* y1,
                   PwP<T>& p, NoiseP<T>& np) {
  if (!nz || nz->source != TSDE_SRC_COUNTER || nz->flags || !y0) return TSDE_EINVAL;
  bool vec = L->d % 4 == 0 && aligned16(y0) && (!y1 || aligned16(y1));
  pw_valid_tables(prog, &vec, TSDE_PW_M);
  if (int e = fill_noise<T>(L, nz, false, np)) return e;
  p = PwP<T>{};
  p.y0 = static_cast<const T*>(y0);
  p.y1 = static_cast<T*>(y1);
  fill_quad_map(L->rows, L->d, p);
  p.vec = vec ? 1 : 0;
  return 0;
}

// The step table of the chunk steps[0, n_steps), after pw_fill: 1 to kPwMaxSteps steps, each with its time, the last
// with a destination.  A step that merges several Brownian cells (np.n_cells > 1) runs alone, in the kSrcCounterMulti
// kernel, which reads the first cell and the uniform length from the noise descriptor.  Clears p.vec for a destination
// that is not 16-byte aligned.
template <typename T>
static int pw_steps(const tsde_pw_step* steps, int32_t n_steps, PwP<T>& p, NoiseP<T>& np, PwSteps<T>& st) {
  if (!steps || n_steps < 1 || n_steps > kPwMaxSteps || !steps[n_steps - 1].y1) return TSDE_EINVAL;
  if (np.n_cells > 1 && n_steps > 1) return TSDE_EINVAL;
  st = PwSteps<T>{};
  st.n = n_steps;
  for (int j = 0; j < n_steps; ++j) {
    const tsde_pw_step& s = steps[j];
    if (!s.t0) return TSDE_EINVAL;
    if (s.y1 && !aligned16(s.y1)) p.vec = 0;
    st.s[j] = PwStep<T>{s.cell_id, static_cast<const T*>(s.t0), static_cast<T*>(s.y1), (T)sqrt(s.h), (T)s.dt};
  }
  // a uniform grid (PwSteps::uniform): consecutive cells, one sqrt_h and dt, and evenly spaced times and
  // destinations, every step stored
  const tsde_pw_step& s0 = steps[0];
  const auto at = [](const void* x) { return (intptr_t)x; };
  const intptr_t dy = n_steps > 1 ? at(steps[1].y1) - at(s0.y1) : 0, dt0 = n_steps > 1 ? at(steps[1].t0) - at(s0.t0) : 0;
  bool uniform = np.n_cells == 1 && !np.bcast && p.vec && dy % (intptr_t)sizeof(T) == 0 &&
                 dt0 % (intptr_t)sizeof(T) == 0;
  for (int j = 0; j < n_steps && uniform; ++j) {
    const tsde_pw_step& s = steps[j];
    uniform = s.y1 && s.cell_id == s0.cell_id + (uint64_t)j && !memcmp(&st.s[j].sqrt_h, &st.s[0].sqrt_h, sizeof(T)) &&
              !memcmp(&st.s[j].dt, &st.s[0].dt, sizeof(T)) && at(s.y1) == at(s0.y1) + j * dy &&
              at(s.t0) == at(s0.t0) + j * dt0;
  }
  st.uniform = uniform ? 1 : 0;
  st.y1_stride = dy / (intptr_t)sizeof(T);
  st.t0_stride = dt0 / (intptr_t)sizeof(T);
  np.cell_id = steps[0].cell_id;
  np.h = steps[0].h;
  return 0;
}

// The decoded program `pg` of an interpreted launch, with the shared-memory slots it takes (`extra` past its layout),
// and pw_fill's parameters, for a program that passes `layout`; TSDE_EINVAL for a launch the kernels cannot serve.
template <typename T>
static int pw_prepare(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog, const void* y0,
                      void* y1, bool (*layout)(const tsde_pointwise&), int extra, PwProg<T>& pg, int& slots,
                      PwP<T>& p, NoiseP<T>& np) {
  bool vec = true;
  if (!prog || !pw_valid_tables(*prog, &vec) || !layout(*prog)) return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, y1, p, np)) return e;
  slots = pw_decode<T>(*prog, extra, pg);
  return 0;
}

// f(std::integral_constant<int, M>{}) for the M of METHODS that `method` is (the caller has checked that one is)
template <int... METHODS, typename F>
static int pw_method(int method, F&& f) {
  int e = TSDE_EINVAL;
  (void)((method == METHODS && ((e = f(std::integral_constant<int, METHODS>{})), true)) || ...);
  return e;
}

// f(std::true_type{}) for a program with comparison and selection ops (PwProg::ext), else f(std::false_type{})
template <typename F>
static int pw_ext(bool ext, F&& f) {
  return ext ? f(std::true_type{}) : f(std::false_type{});
}

// The interpreted kernels of a program with comparison and selection ops (EXT) or without, for Brownian source SRC
template <typename T, int SRC, bool EXT>
constexpr auto pw_srk_of = EXT ? pw_srk_ext_kernel<T, SRC> : pw_srk_kernel<T, SRC>;
template <typename T, int SRC, int METHOD, bool EXT>
constexpr auto pw_pc_of = EXT ? pw_pc_ext_kernel<T, SRC, METHOD> : pw_pc_kernel<T, SRC, METHOD>;
template <typename T, int SRC, int METHOD, bool EXT>
constexpr auto pw_chunk_of = EXT ? pw_chunk_ext_kernel<T, SRC, METHOD> : pw_chunk_kernel<T, SRC, METHOD>;

// One thread per quad, `slots` shared-memory registers per thread; `single` draws from one Brownian cell, `multi` sums
// the cells of a step that spans several.  `x` are the kernel's parameters past the noise (a chunk's step table).
template <typename T, typename P, typename... X>
static int pw_launch(const tsde_launch* L, const PwProg<T>& prog,
                     void (*single)(PwProg<T>, P, NoiseP<T>, X...),
                     void (*multi)(PwProg<T>, P, NoiseP<T>, X...), const P& p, const NoiseP<T>& np,
                     int64_t nquads, int slots, int family, const X&... x) {
  const size_t smem = (size_t)slots * kThreads * 4 * sizeof(T);
  auto kernel = np.n_cells > 1 ? multi : single;
  if (resident_ctas(reinterpret_cast<const void*>(kernel), kThreads, smem) < 1) return TSDE_EINVAL;
  const int64_t grid = (nquads + kThreads - 1) / kThreads;
  const int e = launch_kernel(kernel, grid, kThreads, smem, reinterpret_cast<cudaStream_t>(L->stream), true, prog, p,
                              np, x...);
  if (e == 0) g_launches[family].fetch_add(1, std::memory_order_relaxed);
  return e;
}

// The PwOperands parameter of a compiled kernel: the IMM values and device pointers of `prog`'s operands
template <typename T>
static PwOperands<T> pw_operands(const tsde_pointwise* prog) {
  PwOperands<T> ops{};
  for (int k = 0; k < prog->n_operands; ++k)
    ops.k[k] = PwOperand<T>{static_cast<const T*>(prog->operand[k].ptr), (T)prog->operand[k].imm};
  return ops;
}

// One launch of kernel `entry` of unit `unit` of `source` (compiled here if this is the first launch of its
// structure), its multi-cell variant for a step of several Brownian cells, with parameters (the operands of `prog`,
// x...), one thread per quad of `nquads`, counted under `family`
template <typename T, typename... X>
static int pw_launch_compiled(const tsde_launch* L, const tsde_pointwise* prog, int unit, std::string source,
                              int entry, bool multi, int64_t nquads, int family, X&... x) {
  PwCompiled kc;
  if (int e = pw_loaded(*prog, unit, std::move(source), kc)) return e;
  PwOperands<T> ops = pw_operands<T>(prog);
  void* args[] = {&ops, &x...};
  const int e = launch_kernel_handle(kc.kernel[entry][multi], (nquads + kThreads - 1) / kThreads, kThreads,
                                     reinterpret_cast<cudaStream_t>(L->stream), args);
  if (e == 0) g_launches[family].fetch_add(1, std::memory_order_relaxed);
  return e;
}

// tsde_pointwise_source's result: `src` copied into the caller's buffer (at most size - 1 bytes and a NUL), and its
// length
static int64_t pw_copy_source(const std::string& src, char* buf, int64_t size) {
  if (buf && size > 0) {
    const size_t n = std::min(src.size(), (size_t)size - 1);
    memcpy(buf, src.data(), n);
    buf[n] = 0;
  }
  return (int64_t)src.size();
}

}  // namespace tsde

using namespace tsde;

// A Milstein program the launches `L` may run (tsde_solve_milstein_pointwise's checks of L and prog)
static bool pw_milstein_program(const tsde_launch* L, const tsde_pointwise* prog) {
  bool vec = true;
  return L->noise_type == TSDE_NOISE_DIAGONAL && L->m == L->d && prog && pw_valid_tables(*prog, &vec) &&
         pw_valid_milstein(*prog);
}

// The chunk `steps[0, n_steps)` from y0 (both entry points): one launch of the program's compiled kernel (compiled
// here if this is the first launch of its structure).
template <typename T>
static int pw_milstein_chunk(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog, const void* y0,
                             const tsde_pw_step* steps, int32_t n_steps, int32_t ito) {
  PwP<T> p;
  NoiseP<T> np;
  PwSteps<T> st;
  if (!pw_milstein_program(L, prog)) return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, nullptr, p, np)) return e;
  if (int e = pw_steps<T>(steps, n_steps, p, np, st)) return e;
  p.ito = ito;
  return pw_launch_compiled<T>(L, prog, kPwUnitMilstein, pw_milstein_source(*prog, sizeof(T) == 8), 0,
                               np.n_cells > 1, p.nquads, TSDE_KERNEL_PW_MILSTEIN, p, np, st);
}

// ---- the reversible-Heun adjoint's backward sweep (TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN) -----------------------
// An adjoint program the launches `L` may run: tagged TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN, the Milstein layout's
// checks, with two seeds in the vjp part, vjp_z in gdg_src and each parameter's contribution read at the end
static bool pw_adjoint_program(const tsde_launch* L, const tsde_pw_adjoint* ad) {
  bool vec = true;
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d || !ad ||
      ad->prog.reserved != TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN || ad->n_params < 0 ||
      ad->n_params > TSDE_PW_ADJ_MAX_PARAMS || !pw_valid_tables(ad->prog, &vec))
    return false;
  const tsde_pointwise& pg = ad->prog;
  uint64_t written = 0;
  if (!pw_valid_range(pg, 0, pg.n_fg, 0, written, true) || !pw_valid_source(pg, pg.f_src, 0, written) ||
      !pw_valid_source(pg, pg.g_src, 0, written) || !pw_valid_range(pg, pg.n_fg, pg.n_instr, 2, written, true) ||
      !pw_valid_source(pg, pg.gdg_src, 2, written))
    return false;
  for (int k = 0; k < ad->n_params; ++k)
    if (!pw_valid_source(pg, ad->param_src[k], 2, written)) return false;
  return true;
}

// ---- the general-noise adjoint (TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN) --------------------------------------
// A general adjoint program the GENERAL launches `L` may run, with `route` the contraction order of the unfused kernels
// A and B (dense aligned g, gen_route) for dtype size `s`: the general layout's tables and f / g part, the vjp part with
// two seeds and CSUM, 2 <= m <= TSDE_PW_GENERAL_MAX_M, and a shape pw_gadj_shape accepts.
static bool pw_general_adjoint_program(const tsde_launch* L, const tsde_pw_adjoint* ad, int64_t s, int& route) {
  bool vec = true;
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_GENERAL || L->m < 2 || L->m > TSDE_PW_GENERAL_MAX_M || !ad ||
      ad->prog.reserved != TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN || ad->n_params < 0 ||
      ad->n_params > TSDE_PW_ADJ_MAX_PARAMS || !pw_valid_tables(ad->prog, &vec, TSDE_PW_M))
    return false;
  const tsde_pointwise& pg = ad->prog;
  uint64_t written = 0;
  if (!pw_valid_range(pg, 0, pg.n_fg, 0, written, true) || !pw_valid_source(pg, pg.f_src, 0, written) ||
      !pw_valid_source(pg, pg.g_src, 0, written) || !pw_valid_range(pg, pg.n_fg, pg.n_instr, 2, written, true, true) ||
      !pw_valid_source(pg, pg.gdg_src, 2, written))
    return false;
  for (int k = 0; k < ad->n_params; ++k)
    if (!pw_valid_source(pg, ad->param_src[k], 2, written)) return false;
  PwGAdjShape sh;
  if (!pw_gadj_shape(*ad, sh)) return false;
  route = gen_route(L->m, true, L->m * s);
  return route == TSDE_GEN_TILE || route == TSDE_GEN_GENERIC;
}

// The general adjoint program of a tagged tsde_pointwise (the first member of its tsde_pw_adjoint), or null
static const tsde_pw_adjoint* pw_general_adjoint_of(const tsde_pointwise* prog) {
  return prog && prog->reserved == TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN
             ? reinterpret_cast<const tsde_pw_adjoint*>(prog)
             : nullptr;
}

// tsde_solve_reversible_heun_pointwise for an adjoint program: the chunk steps[0, n_steps) from the state (y, z, f, g)
// of the arguments and (adj_y, adj_f, adj_g, adj_z) of the program's launch buffers, as one launch of its compiled
// kernel (compiled here if this is the first launch of its structure).  `general`: a general adjoint program on a
// GENERAL launch, whose g and adj_g (in and out) are (rows, d, m) and read element by element, as is a per-channel
// parameter's partial.
template <typename T>
static int pw_adjoint_chunk(const tsde_launch* L, const tsde_noise* nz, const tsde_pw_adjoint* ad,
                            const void* const (&in4)[4], const tsde_pw_step* steps, int32_t n_steps,
                            void* const (&out3)[3], bool general = false) {
  int route = 0;
  if (!(general ? pw_general_adjoint_program(L, ad, sizeof(T), route) : pw_adjoint_program(L, ad)) || !ad->t0 ||
      !ad->y1 || !ad->ys || !ad->grad_ys)
    return TSDE_EINVAL;
  const void* const in[kAdjState] = {in4[0], in4[1], in4[2], in4[3], ad->adj_in[0], ad->adj_in[1], ad->adj_in[2],
                                     ad->adj_in[3]};
  void* const out[kAdjState] = {ad->y1, out3[0], out3[1], out3[2], ad->adj_out[0], ad->adj_out[1], ad->adj_out[2],
                                ad->adj_out[3]};
  PwAdjP<T> p{};
  NoiseP<T> np;
  if (int e = pw_fill<T>(L, nz, ad->prog, in[0], nullptr, p.base, np)) return e;
  p.base.t0 = static_cast<const T*>(ad->t0);
  bool vec = p.base.vec != 0 && aligned16(ad->ys) && aligned16(ad->grad_ys);
  for (int k = 0; k < kAdjState; ++k) {
    if (!in[k] || !out[k]) return TSDE_EINVAL;
    if (!general || (k != kAdjG && k != kAdjAdjG)) vec = vec && aligned16(in[k]) && aligned16(out[k]);
    p.in[k] = static_cast<const T*>(in[k]);
    p.out[k] = static_cast<T*>(out[k]);
  }
  for (int k = 0; k < ad->n_params; ++k) {
    if (!ad->partial[k]) return TSDE_EINVAL;
    vec = vec && aligned16(ad->partial[k]);
    p.part[k] = static_cast<T*>(ad->partial[k]);
  }
  p.base.vec = vec ? 1 : 0;
  p.ys = static_cast<const T*>(ad->ys);
  p.gys = static_cast<const T*>(ad->grad_ys);
  p.plane = L->rows * L->d;
  if (!steps || n_steps < 1 || n_steps > kPwMaxSteps || (np.n_cells > 1 && n_steps > 1)) return TSDE_EINVAL;
  PwAdjSteps<T> st{};
  st.n = n_steps;
  const intptr_t plane = (intptr_t)(p.plane * (int64_t)sizeof(T));
  for (int j = 0; j < n_steps; ++j) {
    const tsde_pw_step& s = steps[j];
    int64_t row = -1;  // the output the step ends on: steps[j].y1 = ys + row * rows * d
    if (s.y1) {
      const intptr_t off = (intptr_t)s.y1 - (intptr_t)ad->ys;
      if (off < 0 || off % plane || off / plane >= ad->n_out) return TSDE_EINVAL;
      row = off / plane;
    }
    if (!s.t0) return TSDE_EINVAL;
    st.s[j] = PwAdjStep<T>{s.cell_id, static_cast<const T*>(s.t0), row, (T)sqrt(s.h), (T)s.dt};
  }
  np.cell_id = steps[0].cell_id;
  np.h = steps[0].h;
  if (general)
    return pw_launch_compiled<T>(L, &ad->prog, kPwUnitGeneralAdjoint,
                                 pw_general_adjoint_source(*ad, sizeof(T) == 8, L->m, route), 0, np.n_cells > 1,
                                 p.base.nquads, TSDE_KERNEL_PW_ADJOINT, p, np, st);
  return pw_launch_compiled<T>(L, &ad->prog, kPwUnitAdjoint, pw_adjoint_source(*ad, sizeof(T) == 8), 0,
                               np.n_cells > 1, p.base.nquads, TSDE_KERNEL_PW_ADJOINT, p, np, st);
}

// The adjoint program of a tagged tsde_pointwise (the first member of its tsde_pw_adjoint), or null
static const tsde_pw_adjoint* pw_adjoint_of(const tsde_pointwise* prog) {
  return prog && prog->reserved == TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN
             ? reinterpret_cast<const tsde_pw_adjoint*>(prog)
             : nullptr;
}

// The chunk `steps[0, n_steps)` of Euler or reversible Heun from y0 (and, for reversible Heun, from the solver state
// in[] = z0, f0, g0, left in out[] = z1, f1, g1): one launch of pw_chunk_kernel, under the rules of
// pw_milstein_chunk.
template <typename T, int METHOD>
static int pw_chunk(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog, const void* y0,
                    const tsde_pw_step* steps, int32_t n_steps, const void* const (&in)[3], void* const (&out)[3]) {
  PwProg<T> pg;
  int slots;
  PwChunkP<T> p{};
  NoiseP<T> np;
  PwSteps<T> st;
  if (int e = pw_prepare<T>(L, nz, prog, y0, nullptr, pw_valid_two<TSDE_PW_MAX_REGS>, 0, pg, slots, p.base, np))
    return e;
  if (int e = pw_steps<T>(steps, n_steps, p.base, np, st)) return e;
  if constexpr (METHOD == kPwReversibleHeun) {
    for (int i = 0; i < 3; ++i) {
      if (!in[i] || !out[i]) return TSDE_EINVAL;
      if (!aligned16(in[i]) || !aligned16(out[i])) p.base.vec = 0;
    }
    p.z0 = static_cast<const T*>(in[0]);
    p.f0 = static_cast<const T*>(in[1]);
    p.g0 = static_cast<const T*>(in[2]);
    p.z1 = static_cast<T*>(out[0]);
    p.f1 = static_cast<T*>(out[1]);
    p.g1 = static_cast<T*>(out[2]);
  }
  return pw_ext(pg.ext, [&](auto ext) {
    return pw_launch<T>(L, pg, pw_chunk_of<T, TSDE_SRC_COUNTER, METHOD, decltype(ext)::value>,
                        pw_chunk_of<T, kSrcCounterMulti, METHOD, decltype(ext)::value>, p, np, p.base.nquads, slots,
                        TSDE_KERNEL_PW_CHUNK, st);
  });
}

// ---- general / additive noise (GENERAL launches) -------------------------------------------------------------------
// The general layout (tagged TSDE_PW_LAYOUT_GENERAL): the two-program layout with DM / M operands read by g only.
static bool pw_valid_general(const tsde_pointwise& pg) {
  if (!pw_valid_two<TSDE_PW_MAX_REGS, true>(pg)) return false;
  auto per_channel = [&](uint8_t s) {
    return pw_operand_source(s) && pw_per_channel_kind(pg.operand[s - TSDE_PW_OPERAND(0)].kind);
  };
  for (int i = 0; i < pg.n_fg; ++i)
    if (per_channel(pg.instr[i].a) || (!pw_unary(pg.instr[i].op) && per_channel(pg.instr[i].b))) return false;
  return !per_channel(pg.f_src);
}

// A launch and program of layout tag `layout` the general kernels serve; `route` is the contraction order (gen_route)
// for dtype size `s`.
static bool pw_general_program(const tsde_launch* L, const tsde_pointwise* prog, int64_t s, int& route,
                               int layout = TSDE_PW_LAYOUT_GENERAL) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_GENERAL || L->m > TSDE_PW_GENERAL_MAX_M || !prog ||
      prog->reserved != layout)
    return false;
  bool vec = true;
  if (!pw_valid_tables(*prog, &vec, TSDE_PW_M) || !pw_valid_general(*prog)) return false;
  // the unfused step's g is a new contiguous tensor (aligned), or the user's (d, m) block itself when g is a DM operand;
  // the reversible-Heun pair densifies every g it reads (its solver state)
  bool quads = true;
  const uint8_t g = prog->g_src;
  if (layout != TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN && g >= TSDE_PW_OPERAND(0) && g != TSDE_PW_SRC_Y &&
      g != TSDE_PW_SRC_GO && prog->operand[g - TSDE_PW_OPERAND(0)].kind == TSDE_PW_DM)
    quads = aligned16(prog->operand[g - TSDE_PW_OPERAND(0)].ptr);
  if (layout == TSDE_PW_LAYOUT_GENERAL_SRA) {
    // the sra1 launches call launch_gen directly, which stages U too, and take gen_kernel where cabi.cu would take the
    // row-wise kernels (m == 1: the sum 0 + g * w, which turns a -0 product into +0)
    route = gen_route(L->m, quads, 2 * L->m * s);
    if (route == TSDE_GEN_ROWWISE) route = TSDE_GEN_GENERIC;
  } else {
    route = gen_route(L->m, quads, L->m * s);
  }
  return route != TSDE_GEN_WIDE;
}

// pw_launch_compiled of kernel `entry` of a general program that passed pw_general_program with contraction `route`
// and tag `layout`
template <typename T, typename... X>
static int pw_general_launch(const tsde_launch* L, const tsde_pointwise* prog, int route, int layout, int entry,
                             const NoiseP<T>& np, int64_t nquads, X&... x) {
  return pw_launch_compiled<T>(L, prog, layout, pw_general_source(*prog, sizeof(T) == 8, L->m, route, layout), entry,
                               np.n_cells > 1, nquads, TSDE_KERNEL_PW_GENERAL, x...);
}

// tsde_solve_euler_pointwise for a GENERAL launch: the chunk `steps[0, n_steps)` from y0 as one launch of the
// program's compiled Euler kernel, under the rules of pw_milstein_chunk.
template <typename T>
static int pw_general_euler(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog, const void* y0,
                            const tsde_pw_step* steps, int32_t n_steps) {
  int route;
  PwP<T> p;
  NoiseP<T> np;
  PwSteps<T> st;
  if (!pw_general_program(L, prog, sizeof(T), route)) return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, nullptr, p, np)) return e;
  if (int e = pw_steps<T>(steps, n_steps, p, np, st)) return e;
  return pw_general_launch<T>(L, prog, route, TSDE_PW_LAYOUT_GENERAL, kPwGeneralEuler, np, p.nquads, p, np, st);
}

// tsde_step_predictor_corrector_pointwise for a GENERAL launch: one midpoint step as one launch of the program's
// compiled midpoint kernel, or one Euler-Heun step of an EULER_HEUN-tagged program.
template <typename T>
static int pw_general_pc_step(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                              const void* y0, const void* t0, const void* t_p, int32_t method, double dt,
                              double half_dt, void* y1) {
  int route;
  const bool euler_heun = method == TSDE_PC_EULER_HEUN;
  const int layout = euler_heun ? TSDE_PW_LAYOUT_GENERAL_EULER_HEUN : TSDE_PW_LAYOUT_GENERAL;
  PwGeneralMidP<T> p{};
  NoiseP<T> np;
  if ((method != TSDE_PC_MIDPOINT && !euler_heun) || !t0 || !t_p || !y1 ||
      !pw_general_program(L, prog, sizeof(T), route, layout))
    return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, y1, p.base, np)) return e;
  p.base.t0 = static_cast<const T*>(t0);
  p.base.dt = (T)dt;
  p.t_p = static_cast<const T*>(t_p);
  p.half_dt = (T)half_dt;
  // (the Euler-Heun unit's one kernel, or the general unit's midpoint kernel)
  return pw_general_launch<T>(L, prog, route, layout, euler_heun ? 0 : kPwGeneralMidpoint, np, p.base.nquads, p, np);
}

// tsde_solve_reversible_heun_pointwise for a GENERAL launch: the chunk `steps[0, n_steps)` from y0 and the solver state
// in[] = z0, f0, g0 (g of shape (rows, d, m)), left in out[] = z1, f1, g1, as one launch of the REVERSIBLE_HEUN-tagged
// program's compiled kernel, under the rules of pw_general_euler.
template <typename T>
static int pw_general_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                      const void* y0, const void* const (&in)[3], const tsde_pw_step* steps,
                                      int32_t n_steps, void* const (&out)[3]) {
  int route;
  PwGeneralRevHeunP<T> p{};
  NoiseP<T> np;
  PwSteps<T> st;
  if (!pw_general_program(L, prog, sizeof(T), route, TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN)) return TSDE_EINVAL;
  for (int i = 0; i < 3; ++i)
    if (!in[i] || !out[i]) return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, nullptr, p.base, np)) return e;
  if (int e = pw_steps<T>(steps, n_steps, p.base, np, st)) return e;
  for (int i = 0; i < 2; ++i)  // z, f
    if (!aligned16(in[i]) || !aligned16(out[i])) p.base.vec = 0;
  p.z0 = static_cast<const T*>(in[0]);
  p.f0 = static_cast<const T*>(in[1]);
  p.g0 = static_cast<const T*>(in[2]);
  p.z1 = static_cast<T*>(out[0]);
  p.f1 = static_cast<T*>(out[1]);
  p.g1 = static_cast<T*>(out[2]);
  p.gvec = L->m % 4 == 0 && aligned16(in[2]) && aligned16(out[2]) ? 1 : 0;
  return pw_general_launch<T>(L, prog, route, TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN, 0, np, p.base.nquads, p, np,
                              st);
}

// tsde_step_srk_diag_pointwise for a GENERAL launch: one sra1 step as one launch of the SRA-tagged program's
// compiled kernel.
template <typename T>
static int pw_general_sra1_step(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                const void* y0, const void* t_1, const void* t_34, const void* t_00, double dt,
                                double rdt, void* y1) {
  int route;
  PwGeneralSraP<T> p{};
  NoiseP<T> np;
  if (!t_1 || !t_34 || !t_00 || !y1 || !pw_general_program(L, prog, sizeof(T), route, TSDE_PW_LAYOUT_GENERAL_SRA))
    return TSDE_EINVAL;
  if (int e = pw_fill<T>(L, nz, *prog, y0, y1, p.base, np)) return e;
  p.base.t0 = static_cast<const T*>(t_00);
  p.base.dt = (T)dt;
  p.t_1 = static_cast<const T*>(t_1);
  p.t_34 = static_cast<const T*>(t_34);
  p.stage = GSraStageOp<T>{(T)dt, (T)rdt};
  p.final_op = GSraFinalOp<T>{(T)dt, (T)rdt, (T)(1.0 / 3), (T)(2.0 / 3)};
  return pw_general_launch<T>(L, prog, route, TSDE_PW_LAYOUT_GENERAL_SRA, 0, np, p.base.nquads, p, np);
}

// The unit (its layout tag) and source a GENERAL launch of tsde_pointwise_compile / tsde_pointwise_source serves
// `prog` with: that of its SRA, EULER_HEUN or REVERSIBLE_HEUN tag, else the Euler / midpoint unit (which refuses every
// other tag); false if the general kernels cannot serve it.
template <typename T>
static bool pw_general_unit(const tsde_launch* L, const tsde_pointwise* prog, int& layout, std::string& source) {
  int route;
  const int tag = prog ? prog->reserved : 0;
  layout = tag >= TSDE_PW_LAYOUT_GENERAL_SRA && tag <= TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN ? tag
                                                                                              : TSDE_PW_LAYOUT_GENERAL;
  if (!pw_general_program(L, prog, sizeof(T), route, layout)) return false;
  source = pw_general_source(*prog, sizeof(T) == 8, L->m, route, layout);
  return true;
}

// ---- the entry points -----------------------------------------------------------------------------------------------
TSDE_EXPORT int tsde_solve_euler_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                           const void* y0, const tsde_pw_step* steps, int32_t n_steps) {
  if (valid_launch(L) && L->noise_type == TSDE_NOISE_GENERAL)
    return dispatch(L, [&](auto t) -> int { return pw_general_euler<decltype(t)>(L, nz, prog, y0, steps, n_steps); });
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  const void* const in[3] = {};
  void* const out[3] = {};
  return dispatch(L, [&](auto t) -> int {
    return pw_chunk<decltype(t), kPwEuler>(L, nz, prog, y0, steps, n_steps, in, out);
  });
}

TSDE_EXPORT int tsde_solve_reversible_heun_pointwise(const tsde_launch* L, const tsde_noise* nz,
                                                     const tsde_pointwise* prog, const void* y0, const void* z0,
                                                     const void* f0, const void* g0, const tsde_pw_step* steps,
                                                     int32_t n_steps, void* z1, void* f1, void* g1) {
  const void* const in[3] = {z0, f0, g0};
  void* const out[3] = {z1, f1, g1};
  if (valid_launch(L) && L->noise_type == TSDE_NOISE_GENERAL && pw_general_adjoint_of(prog)) {
    const tsde_pw_adjoint* ad = pw_general_adjoint_of(prog);
    const void* const in4[4] = {y0, z0, f0, g0};
    return dispatch(L, [&](auto t) -> int {
      return pw_adjoint_chunk<decltype(t)>(L, nz, ad, in4, steps, n_steps, out, true);
    });
  }
  if (valid_launch(L) && L->noise_type == TSDE_NOISE_GENERAL)
    return dispatch(L, [&](auto t) -> int {
      return pw_general_reversible_heun<decltype(t)>(L, nz, prog, y0, in, steps, n_steps, out);
    });
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  if (const tsde_pw_adjoint* ad = pw_adjoint_of(prog)) {
    const void* const in4[4] = {y0, z0, f0, g0};
    return dispatch(L, [&](auto t) -> int {
      return pw_adjoint_chunk<decltype(t)>(L, nz, ad, in4, steps, n_steps, out);
    });
  }
  return dispatch(L, [&](auto t) -> int {
    return pw_chunk<decltype(t), kPwReversibleHeun>(L, nz, prog, y0, steps, n_steps, in, out);
  });
}

TSDE_EXPORT int tsde_step_milstein_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                             const void* y0, const void* t0, double dt, int32_t ito, void* y1) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    using T = decltype(t);
    if (!t0 || !nz) return TSDE_EINVAL;
    const tsde_pw_step step{nz->cell_id, nz->h, dt, t0, y1};  // a chunk of one
    return pw_milstein_chunk<T>(L, nz, prog, y0, &step, 1, ito);
  });
}

TSDE_EXPORT int tsde_solve_milstein_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                              const void* y0, const tsde_pw_step* steps, int32_t n_steps,
                                              int32_t ito) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int { return pw_milstein_chunk<decltype(t)>(L, nz, prog, y0, steps, n_steps, ito); });
}

TSDE_EXPORT int tsde_step_srk_diag_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                             const void* y0, const void* t_0, const void* t_1, const void* t_q,
                                             const void* t_h, double dt, double rdt, double sqrt_dt, double three_dt,
                                             void* y1) {
  if (valid_launch(L) && L->noise_type == TSDE_NOISE_GENERAL)  // additive noise: sra1, t_q = t0 + 3/4 dt
    return dispatch(L, [&](auto t) -> int {
      return pw_general_sra1_step<decltype(t)>(L, nz, prog, y0, t_1, t_q, t_0, dt, rdt, y1);
    });
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    using T = decltype(t);
    if (!t_0 || !t_1 || !t_q || !t_h || !y1) return TSDE_EINVAL;
    PwProg<T> pg;
    int slots;
    PwSrkP<T> p;
    NoiseP<T> np;
    if (int e = pw_prepare<T>(L, nz, prog, y0, y1, pw_valid_two<TSDE_PW_SRK_MAX_REGS>,
                              PwSrkStash<T>::kShared ? kPwSrkStash : 0, pg, slots, p.base, np))
      return e;
    const void* times[4] = {t_0, t_1, t_q, t_h};
    for (int i = 0; i < 4; ++i) p.t[i] = static_cast<const T*>(times[i]);
    // the coefficients of tsde_srk_diag_stage1/2/3 and tsde_step_srk_diag
    p.s1 = SrkDiagStage1Op<T>{(T)dt, (T)sqrt_dt};
    p.s2 = SrkDiagStage2Op<T>{(T)dt, (T)rdt, (T)sqrt_dt};
    p.s3 = SrkDiagStage3Op<T>{(T)dt, (T)sqrt_dt};
    p.fin = make_srk_final<T>(dt, rdt, sqrt_dt, three_dt);
    return pw_ext(pg.ext, [&](auto ext) {
      return pw_launch<T>(L, pg, pw_srk_of<T, TSDE_SRC_COUNTER, decltype(ext)::value>,
                          pw_srk_of<T, kSrcCounterMulti, decltype(ext)::value>, p, np, p.base.nquads, slots,
                          TSDE_KERNEL_PW_SRK);
    });
  });
}

TSDE_EXPORT int tsde_step_predictor_corrector_pointwise(const tsde_launch* L, const tsde_noise* nz,
                                                        const tsde_pointwise* prog, const void* y0, const void* t0,
                                                        const void* t_p, int32_t method, double dt, double half_dt,
                                                        void* y1) {
  if (valid_launch(L) && L->noise_type == TSDE_NOISE_GENERAL)
    return dispatch(L, [&](auto t) -> int {
      return pw_general_pc_step<decltype(t)>(L, nz, prog, y0, t0, t_p, method, dt, half_dt, y1);
    });
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    using T = decltype(t);
    if (!t0 || !t_p || !y1 || method < TSDE_PC_HEUN || method > TSDE_PC_EULER_HEUN) return TSDE_EINVAL;
    PwProg<T> pg;
    int slots;
    PwPcP<T> p;
    NoiseP<T> np;
    if (int e = pw_prepare<T>(L, nz, prog, y0, y1, pw_valid_two<TSDE_PW_MAX_REGS>, 0, pg, slots, p.base, np))
      return e;
    p.base.t0 = static_cast<const T*>(t0);
    p.base.dt = (T)dt;
    p.t_p = static_cast<const T*>(t_p);
    p.half_dt = (T)half_dt;
    return pw_method<TSDE_PC_HEUN, TSDE_PC_MIDPOINT, TSDE_PC_EULER_HEUN>(method, [&](auto m) {
      return pw_ext(pg.ext, [&](auto ext) {
        constexpr int M = decltype(m)::value;
        constexpr bool X = decltype(ext)::value;
        return pw_launch<T>(L, pg, pw_pc_of<T, TSDE_SRC_COUNTER, M, X>, pw_pc_of<T, kSrcCounterMulti, M, X>, p, np,
                            p.base.nquads, slots, TSDE_KERNEL_PW_PC);
      });
    });
  });
}

TSDE_EXPORT int tsde_pointwise_compile(const tsde_launch* L, const tsde_pointwise* prog) {
  return dispatch(L, [&](auto t) -> int {
    PwCompiled kc;
    if (L->noise_type == TSDE_NOISE_GENERAL && pw_general_adjoint_of(prog)) {
      int route;
      const tsde_pw_adjoint* ad = pw_general_adjoint_of(prog);
      if (!pw_general_adjoint_program(L, ad, sizeof(t), route)) return TSDE_EINVAL;
      return pw_loaded(*prog, kPwUnitGeneralAdjoint, pw_general_adjoint_source(*ad, sizeof(t) == 8, L->m, route), kc);
    }
    if (L->noise_type == TSDE_NOISE_GENERAL) {
      int layout;
      std::string source;
      if (!pw_general_unit<decltype(t)>(L, prog, layout, source)) return TSDE_EINVAL;
      return pw_loaded(*prog, layout, std::move(source), kc);
    }
    if (const tsde_pw_adjoint* ad = pw_adjoint_of(prog)) {
      if (!pw_adjoint_program(L, ad)) return TSDE_EINVAL;
      return pw_loaded(*prog, kPwUnitAdjoint, pw_adjoint_source(*ad, sizeof(t) == 8), kc);
    }
    if (!pw_milstein_program(L, prog)) return TSDE_EINVAL;
    return pw_loaded(*prog, kPwUnitMilstein, pw_milstein_source(*prog, sizeof(t) == 8), kc);
  });
}

TSDE_EXPORT int64_t tsde_pointwise_source(const tsde_launch* L, const tsde_pointwise* prog, char* buf, int64_t size) {
  return dispatch(L, [&](auto t) -> int64_t {
    if (L->noise_type == TSDE_NOISE_GENERAL && pw_general_adjoint_of(prog)) {
      int route;
      const tsde_pw_adjoint* ad = pw_general_adjoint_of(prog);
      if (!pw_general_adjoint_program(L, ad, sizeof(t), route)) return TSDE_EINVAL;
      return pw_copy_source(pw_general_adjoint_source(*ad, sizeof(t) == 8, L->m, route), buf, size);
    }
    if (L->noise_type == TSDE_NOISE_GENERAL) {
      int layout;
      std::string source;
      if (!pw_general_unit<decltype(t)>(L, prog, layout, source)) return TSDE_EINVAL;
      return pw_copy_source(source, buf, size);
    }
    if (const tsde_pw_adjoint* ad = pw_adjoint_of(prog)) {
      if (!pw_adjoint_program(L, ad)) return TSDE_EINVAL;
      return pw_copy_source(pw_adjoint_source(*ad, sizeof(t) == 8), buf, size);
    }
    if (!pw_milstein_program(L, prog)) return TSDE_EINVAL;
    return pw_copy_source(pw_milstein_source(*prog, sizeof(t) == 8), buf, size);
  });
}

// ---- an adaptive solve's proposal -----------------------------------------------------------------------------------
// The proposal's checks, made before anything is compiled or launched: a known method, sub-steps with the increments,
// and the times, its method reads, a program of its method's layout.  Fills the sub-step table `st`.
template <typename T>
static int pw_proposal_table(const tsde_launch* L, const tsde_pointwise* prog, int32_t method, const void* y0,
                             const tsde_pw_substep* subs, void* y_full, void* y_next, bool& vec, PwSubs<T>& st) {
  if (method < TSDE_PROPOSAL_EULER || method > TSDE_PROPOSAL_EULER_HEUN || !prog || !y0 || !subs || !y_full ||
      !y_next)
    return TSDE_EINVAL;
  const bool milstein = method == TSDE_PROPOSAL_MILSTEIN_ITO || method == TSDE_PROPOSAL_MILSTEIN_STRATONOVICH;
  const int n_times = method == TSDE_PROPOSAL_SRK ? 4 : method >= TSDE_PROPOSAL_HEUN ? 2 : 1;
  vec = L->d % 4 == 0 && aligned16(y0) && aligned16(y_full) && aligned16(y_next);
  st = PwSubs<T>{};
  for (int k = 0; k < 3; ++k) {
    const tsde_pw_substep& s = subs[k];
    if (!s.w || (method == TSDE_PROPOSAL_SRK && !s.u)) return TSDE_EINVAL;
    for (int i = 0; i < n_times; ++i)
      if (!s.t[i]) return TSDE_EINVAL;
    vec = vec && aligned16(s.w) && (method != TSDE_PROPOSAL_SRK || aligned16(s.u));
    PwSub<T>& d = st.sub[k];
    d.s = PwStep<T>{0, static_cast<const T*>(s.t[0]), nullptr, T(0), (T)s.dt};
    d.w = static_cast<const T*>(s.w);
    d.u = method == TSDE_PROPOSAL_SRK ? static_cast<const T*>(s.u) : nullptr;
    for (int i = 0; i < 4; ++i) d.t[i] = i < n_times ? static_cast<const T*>(s.t[i]) : nullptr;
    d.half_dt = (T)s.s[0];
  }
  if (!pw_valid_tables(*prog, &vec)) return TSDE_EINVAL;
  const bool layout = milstein                       ? pw_valid_milstein(*prog)
                      : method == TSDE_PROPOSAL_SRK ? pw_valid_two<TSDE_PW_SRK_MAX_REGS>(*prog)
                                                     : pw_valid_two<TSDE_PW_MAX_REGS>(*prog);
  return layout ? 0 : TSDE_EINVAL;
}

template <typename T>
static int pw_proposal_launch(const tsde_launch* L, const tsde_pointwise* prog, int32_t method, const void* y0,
                              const tsde_pw_substep* subs, void* y_full, void* y_next) {
  bool vec;
  PwProposalP<T> p{};
  if (int e = pw_proposal_table<T>(L, prog, method, y0, subs, y_full, y_next, vec, p.st)) return e;
  p.base.y0 = static_cast<const T*>(y0);
  p.base.y1 = static_cast<T*>(y_full);
  fill_quad_map(L->rows, L->d, p.base);
  p.base.vec = vec ? 1 : 0;
  p.y_next = static_cast<T*>(y_next);
  if (method == TSDE_PROPOSAL_MILSTEIN_ITO || method == TSDE_PROPOSAL_MILSTEIN_STRATONOVICH) {
    p.base.ito = method == TSDE_PROPOSAL_MILSTEIN_ITO ? 1 : 0;
    return pw_launch_compiled<T>(L, prog, kPwUnitAdaptive, pw_milstein_source(*prog, sizeof(T) == 8, kPwUnitAdaptive),
                                 0, false, p.base.nquads, TSDE_KERNEL_PW_ADAPTIVE, p.base, p.y_next, p.st);
  }
  if (method == TSDE_PROPOSAL_SRK) {
    for (int k = 0; k < 3; ++k) {
      const tsde_pw_substep& s = subs[k];
      const double dt = s.dt, rdt = s.s[0], sqrt_dt = s.s[1], three_dt = s.s[2];
      // the coefficients of tsde_srk_diag_stage1/2/3 and tsde_step_srk_diag
      p.srk[k] = PwSrkOps<T>{SrkDiagStage1Op<T>{(T)dt, (T)sqrt_dt}, SrkDiagStage2Op<T>{(T)dt, (T)rdt, (T)sqrt_dt},
                             SrkDiagStage3Op<T>{(T)dt, (T)sqrt_dt}, make_srk_final<T>(dt, rdt, sqrt_dt, three_dt)};
    }
  }
  PwProg<T> pg;
  const int slots = pw_decode<T>(*prog, method == TSDE_PROPOSAL_SRK && PwSrkStash<T>::kShared ? kPwSrkStash : 0, pg);
  const size_t smem = (size_t)slots * kThreads * 4 * sizeof(T);
  return pw_method<TSDE_PROPOSAL_EULER, TSDE_PROPOSAL_SRK, TSDE_PROPOSAL_HEUN, TSDE_PROPOSAL_MIDPOINT,
                   TSDE_PROPOSAL_EULER_HEUN>(method, [&](auto m) {
    return pw_ext(pg.ext, [&](auto ext) {
      auto kernel = pw_proposal_kernel<T, decltype(m)::value, decltype(ext)::value>;
      if (resident_ctas(reinterpret_cast<const void*>(kernel), kThreads, smem) < 1) return TSDE_EINVAL;
      const int e = launch_kernel(kernel, (p.base.nquads + kThreads - 1) / kThreads, kThreads, smem,
                                  reinterpret_cast<cudaStream_t>(L->stream), true, pg, p);
      if (e == 0) g_launches[TSDE_KERNEL_PW_ADAPTIVE].fetch_add(1, std::memory_order_relaxed);
      return e;
    });
  });
}

TSDE_EXPORT int tsde_adaptive_proposal_pointwise(const tsde_launch* L, const tsde_pointwise* prog, int32_t method,
                                                 const void* y0, const tsde_pw_substep* subs, void* y_full,
                                                 void* y_next) {
  if (!valid_launch(L) || L->noise_type != TSDE_NOISE_DIAGONAL || L->m != L->d) return TSDE_EINVAL;
  return dispatch(L, [&](auto t) -> int {
    return pw_proposal_launch<decltype(t)>(L, prog, method, y0, subs, y_full, y_next);
  });
}

TSDE_EXPORT int tsde_adaptive_pointwise_compile(const tsde_launch* L, const tsde_pointwise* prog) {
  return dispatch(L, [&](auto t) -> int {
    if (!pw_milstein_program(L, prog)) return TSDE_EINVAL;
    PwCompiled kc;
    return pw_loaded(*prog, kPwUnitAdaptive, pw_milstein_source(*prog, sizeof(t) == 8, kPwUnitAdaptive), kc);
  });
}

