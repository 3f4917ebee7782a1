/*
 * torchsde_b200 — C ABI of the H100 (sm_90a) SDE-integration hot path.
 *
 * This header is the drop-in boundary of the package.  Every entry point is a
 * plain `extern "C"` function taking raw device pointers, sizes, scalars and a
 * CUDA stream handle; no torch type crosses it.  The Python host
 * (torchsde_b200/_cabi.py, ctypes) is the only caller inside this repository;
 * INTEGRATION.md shows the binding a torchsde maintainer would add.
 *
 * Each function replaces one "kernel-equivalent call site" of the reference
 * (google-research/torchsde v0.2.6).  The reference file:line a function
 * follows is cited above its declaration; paths are relative to the
 * reference tree (`torchsde/...`).
 *
 * Conventions
 *   - All tensors are dense, row-major, contiguous device buffers.
 *       state-like    : (rows, d)
 *       diagonal g    : (rows, d)          (d == m)
 *       general g     : (rows, d, m)       (scalar noise: m == 1; additive: same layout)
 *       noise W, U    : (rows, m)
 *   - `dtype` is TSDE_F32 or TSDE_F64 and applies to every tensor of a call,
 *     except the 16-bit SDE outputs a float32 launch may declare (TSDE_FMT_*).
 *   - Scalars (dt, coefficients) are passed as double and rounded ONCE to the
 *     tensor dtype on the host side of the kernel launch, which is what the
 *     reference's `tensor * python_scalar` / `tensor * 0-d tensor` does.
 *   - Arithmetic inside a tableau follows the reference's left-to-right
 *     evaluation order with separate IEEE roundings (no FMA contraction), so
 *     a diagonal-noise step fed identical inputs is bit-identical to the
 *     reference's sequence of ATen elementwise ops.
 *   - Every function enqueues work on `stream` and returns immediately; it
 *     never allocates and never synchronises, so it may be captured in a
 *     CUDA graph.  Return value: 0 on success, otherwise the cudaError_t of
 *     the launch (or TSDE_EINVAL for a contract violation).
 */
#ifndef TORCHSDE_B200_H_
#define TORCHSDE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSDE_ABI_VERSION 1
#define TSDE_EINVAL (-22)
#define TSDE_ECOMPILE (-38) /* an element-wise program could not be compiled (tsde_pointwise_compile) */

enum { TSDE_F32 = 0, TSDE_F64 = 1 };

/*
 * 16-bit SDE outputs (a drift / diffusion evaluated under torch.autocast).  Bits 0-7 of tsde_launch.dtype are the
 * state dtype; above them, two bits per tensor input of the call, in declaration order, give that input's storage
 * format.  Only inputs that hold what the user's SDE returned may be 16-bit: the f*, fp, g*, gp, ga and gb
 * arguments of the step tableaus, predictors and stages, tsde_milstein_vjp_seed and the two reversible-Heun adjoint
 * halves (g also when it holds a user g_prod, TSDE_SRC_UNIT).  The kernels widen such an operand exactly to float32
 * and run the float32 arithmetic unchanged, so a launch equals the float32 launch on widened copies bit for bit.
 * TSDE_EINVAL: format bits on any other input or entry point, with a TSDE_F64 state, or the value 3.
 * tsde_milstein_vjp_seed writes go in g's format (round to nearest even).
 */
enum { TSDE_FMT_STATE = 0, TSDE_FMT_BF16 = 1, TSDE_FMT_F16 = 2 };
#define TSDE_OPERAND_FMT(i, fmt) ((int32_t)(fmt) << (8 + 2 * (i)))

/* noise layouts (torchsde/settings.py:41-45 NOISE_TYPES) */
enum {
  TSDE_NOISE_DIAGONAL = 0, /* g:(rows,d)      W:(rows,d)                   base_sde.py:98-99   */
  TSDE_NOISE_GENERAL  = 1  /* g:(rows,d,m)    W:(rows,m)   also additive   base_sde.py:101-102 */
                           /* scalar noise is GENERAL with m == 1                               */
};

/* where a kernel takes the Brownian increment from */
enum {
  TSDE_SRC_MEMORY  = 0, /* read W (and U) from device buffers (any BaseBrownian)         */
  TSDE_SRC_COUNTER = 1, /* regenerate in registers from the Philox counter (fast path)   */
  TSDE_SRC_UNIT    = 2  /* W == 1: `g` already holds the user's g_prod (base_sde.py:51-56) */
};

/* Launch flags (tsde_noise.flags).
 * TSDE_FLAG_G_BROADCAST: every (rows,d,m) diffusion operand of this launch is ONE dense (d,m) block shared by
 * all rows (row stride 0) — what `sigma.expand(B, d, m)` is for additive noise whose diffusion does not depend on
 * y (the reference's own additive test problem materialises it with `repeat`, tests/problems.py:113-116; the
 * product base_sde.py:101-102 / misc.py:62-63 only ever reads it).  Honoured by the general-noise entry points
 * (noise_type GENERAL, m > 1); the pointer then addresses d*m elements. */
#define TSDE_FLAG_G_BROADCAST 1

/* Shape / stream descriptor shared by all launches. */
typedef struct tsde_launch {
  int32_t dtype;      /* TSDE_F32 | TSDE_F64, | TSDE_OPERAND_FMT(i, TSDE_FMT_*) for 16-bit SDE outputs */
  int32_t noise_type; /* TSDE_NOISE_*                              */
  int64_t rows;       /* trajectories held by this rank; 0 is a valid launch that does nothing (operand pointers
                         of an empty batch may be NULL)            */
  int64_t d;          /* state channels                            */
  int64_t m;          /* Brownian channels                         */
  void*   stream;     /* cudaStream_t                              */
} tsde_launch;

/*
 * Brownian increment over one solver step.
 *
 * Counter mode restates what BrownianInterval hands the solver
 * (torchsde/_brownian/brownian_interval.py:589-687) for an interval that is
 * the merge of `n_cells` consecutive primary cells of a grid node:
 *     W_c = sqrt(h_c) * N_W(key; cell_id + c; row; channel)          (:553-554)
 *     H_c = sqrt(h_c / 12) * N_H(key; cell_id + c; row; channel)     (:555-558)
 * merged left to right with the reference's aggregation rule (:643-672) and
 * returned as W and U = h (W/2 + H) (:102-103).  N_* are Philox4x32-10
 * Box-Muller normals; see torchsde_b200/csrc/philox.cuh for the bit-level
 * definition and oracle/philox.py for its CPU restatement.
 */
typedef struct tsde_noise {
  int32_t     source;     /* TSDE_SRC_*                                                    */
  int32_t     want_u;     /* also produce U (space-time Levy area, srk.py:61)              */
  const void* w;          /* MEMORY: (rows, m) increments                                  */
  const void* u;          /* MEMORY: (rows, m) U = h(W/2 + H), or NULL                     */
  const void* key;        /* COUNTER: device pointer to the 64-bit Philox key              */
  uint64_t    cell_id;    /* COUNTER: counter words 2,3 of the first cell                  */
  int64_t     row_offset; /* COUNTER: global index of local row 0 (batch sharding)         */
  int32_t     n_cells;    /* COUNTER: number of consecutive cells merged (>= 1)            */
  int32_t     flags;      /* TSDE_FLAG_* of this launch (0 = none)                         */
  double      h;          /* COUNTER: length of each cell when cell_h == NULL              */
  const double* cell_h;   /* COUNTER: DEVICE pointer to n_cells lengths, or NULL (uniform) */
  double      h_total;    /* COUNTER: tb - ta of the whole step (U = h_total (W/2 + H))    */
} tsde_noise;

int tsde_abi_version(void);
/* Last CUDA error string of this library's runtime instance (for diagnostics). */
const char* tsde_error_string(int code);
/* Diagnostics: how many launches of a kernel family this process has issued so far (tests use it to
   check which general-noise tile kernel a shape was routed to). */
#define TSDE_KERNEL_GEN_CTA 0  /* per-thread-load tile kernel                       */
#define TSDE_KERNEL_GEN_TMA 1  /* TMA-staged persistent tile kernel (bulk copies)   */
#define TSDE_KERNEL_GEN_WIDE 2 /* chunked tile kernel for rows whose increments exceed shared memory */
#define TSDE_KERNEL_PW_MILSTEIN 3 /* whole Milstein step with an element-wise SDE (tsde_step_milstein_pointwise) */
#define TSDE_KERNEL_PW_SRK 4      /* whole SRK step with an element-wise SDE (tsde_step_srk_diag_pointwise)     */
#define TSDE_KERNEL_PW_PC 5       /* whole Heun / midpoint / Euler-Heun step with an element-wise SDE
                                     (tsde_step_predictor_corrector_pointwise)                                  */
#define TSDE_KERNEL_PW_CHUNK 6    /* Euler / reversible-Heun steps with an element-wise SDE, up to
                                     TSDE_PW_MAX_STEPS per launch (tsde_solve_euler_pointwise,
                                     tsde_solve_reversible_heun_pointwise)                                      */
#define TSDE_KERNEL_PW_ADAPTIVE 7 /* an adaptive solve's proposal with an element-wise SDE, the full step and both
                                     half steps in one launch (tsde_adaptive_proposal_pointwise)                */
#define TSDE_KERNEL_PW_GENERAL 8  /* general / additive-noise Euler or reversible-Heun steps, a midpoint or
                                     Euler-Heun step or an additive-noise SRK step with an element-wise SDE
                                     (GENERAL launches of tsde_solve_euler_pointwise,
                                     tsde_solve_reversible_heun_pointwise, tsde_step_predictor_corrector_pointwise
                                     and tsde_step_srk_diag_pointwise)                                           */
#define TSDE_KERNEL_PW_ADJOINT 9  /* backward steps of the reversible-Heun adjoint with an element-wise SDE, up to
                                     TSDE_PW_MAX_STEPS per launch (tsde_solve_reversible_heun_pointwise with a
                                     TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN program)                            */
int64_t tsde_kernel_launches(int32_t family);


/* ------------------------------------------------------------------------ */
/* Brownian source  (replaces torchsde/_brownian/brownian_interval.py)       */
/* ------------------------------------------------------------------------ */

/*
 * Materialise the increment described by `nz` (COUNTER source) into device
 * buffers: out_w (rows,m) always; out_u (rows,m) = U if non-NULL; out_h
 * (rows,m) = H if non-NULL.  Replaces BrownianInterval.__call__ for an
 * interval made of whole cells: brownian_interval.py:589-687 (_randn :30-32,
 * top-level draw :551-558, merge :643-672, _H_to_U :102-103).
 */
int tsde_brownian_cells(const tsde_launch* L, const tsde_noise* nz,
                        void* out_w, void* out_u, void* out_h);

/*
 * Brownian-bridge descent: given the (W,H) of an ancestor interval in
 * in_w/in_h (in_h may be NULL when no Levy area is tracked), walk `depth`
 * binary splits down to a descendant and write its (W,H).
 * Level l uses node id ids[l] for its two normals X1,X2, `is_left[l]`, and the
 * split geometry (parent start/mid/end) times[3*l..3*l+2] (host doubles).
 * Replaces _Interval._increment_and_space_time_levy_area,
 * brownian_interval.py:188-241 (with H :199-225, W only :226-237).
 */
int tsde_brownian_bridge(const tsde_launch* L, const void* key, int64_t row_offset,
                         int32_t depth, const uint64_t* ids, const int32_t* is_left,
                         const double* times, const void* in_w, const void* in_h,
                         void* out_w, void* out_h);

/*
 * Merge the increment of [s,u] (w0,h0) with that of the adjacent [u,t]
 * (w1,h1): W = W0 + W1, H per brownian_interval.py:649-658, in place into
 * (w0,h0).  len0 = u - s, len1 = t - u, tot = t - s (each as the host computed it).
 * h pointers may be NULL.
 */
int tsde_brownian_merge(const tsde_launch* L, void* w0, void* h0, const void* w1,
                        const void* h1, double len0, double len1, double tot);

/*
 * One launch for the query pattern of the Levy-area methods on a solver grid: W (rows,m), U = h (W/2 + H) (rows,m)
 * and the Davie / Foster area A (rows,m,m) of ONE primary cell (nz: COUNTER source, n_cells == 1, cell nz->cell_id of
 * length nz->h), with H drawn from the counter as well and never materialised.  Replaces BrownianInterval.__call__
 * (ta, tb, return_U=True, return_A=True) for a whole cell: brownian_interval.py:589-687 with _randn :30-32, the
 * top-level law :551-558, _davie_foster_approximation :78-99 and _H_to_U :102-103.  Requires m % 4 == 0, 4 <= m <= 64.
 */
int tsde_brownian_cell_levy(const tsde_launch* L, const tsde_noise* nz, uint64_t a_id, int32_t foster, void* out_w,
                            void* out_u, void* out_a);

/*
 * `logqp=True`: the KL-integrand augmentation of SDELogqp.f_and_g_* (base_sde.py:240-306).  d (and m) count the
 * state channels WITHOUT the log-ratio channel; f, h are (rows,d) and f_aug is (rows,d+1).
 *   DIAGONAL (f_and_g_diagonal :266-283, misc.py:66-68):  u = (f - h) / stable(g),  f_aug = [f, 0.5 sum_d u^2],
 *     g_aug = [g, 0];  g is (rows,d), g_aug (rows,d+1), d == m, and `eps` is stable_division's epsilon.
 *   GENERAL, also additive and scalar noise (f_and_g_general :285-306):  u = pinverse(g, rcond) (f - h),
 *     f_aug = [f, 0.5 |u|^2],  g_aug = [g ; 0] (a zero row appended);  g is a dense (rows,d,m), g_aug (rows,d+1,m),
 *     and `eps` is pinverse's rcond (singular values s <= rcond * s_max are dropped).  Per row, a one-sided Jacobi
 *     SVD in shared memory: min(d,m) * max(d,m) + d must not exceed TSDE_LOGQP_GENERAL_MAX, else TSDE_EINVAL.
 *     A row whose g or f - h holds a NaN / Inf gets a NaN rate.
 */
#define TSDE_LOGQP_GENERAL_MAX 16384
int tsde_logqp_augment(const tsde_launch* L, const void* f, const void* g, const void* h, double eps,
                       void* f_aug, void* g_aug);

/*
 * GA = g A for the log-ODE correction (base_sde.py:170,191: `ga = torch.bmm(g, a)` inside
 * dg_ga_jvp_column_sum_v1/_v2; used by methods/log_ode.py:39-56).  g is (rows,d,m), a is (rows,m,m) (the Levy
 * area of the step), out_t is (m, rows, d): column l of g A as a contiguous (rows,d) slab, which is what the
 * column-wise jvp's through the user's g consume (base_sde.py:173-184).  noise_type must be GENERAL.
 */
int tsde_bmm_ga(const tsde_launch* L, const void* g, const void* a, void* out_t);

/* U = h (W/2 + H)   brownian_interval.py:102-103 */
int tsde_brownian_h_to_u(const tsde_launch* L, const void* w, const void* hh, double h, void* out_u);

/*
 * Davie / Foster Levy-area approximation of one interval
 * (brownian_interval.py:78-99): A = H (x) W - W (x) H + std * (N - N^T); foster != 0 selects Foster's std.
 * The antisymmetric noise N - N^T is drawn as one Philox normal per pair i < j of counter id `a_id`
 * (N_ij = z_ij / sqrt 2 = -N_ji: the law of the reference's antisymmetrised iid matrix, half the draws).
 * out_a is (rows, m, m).
 */
int tsde_brownian_levy_area(const tsde_launch* L, const void* key, int64_t row_offset,
                            uint64_t a_id, const void* w, const void* hh, double h,
                            int32_t foster, void* out_a);

/* A-merge of two adjacent intervals, brownian_interval.py:659-671, in place into a0. */
int tsde_brownian_merge_area(const tsde_launch* L, void* a0, const void* a1,
                             const void* w0, const void* w1);

/* ------------------------------------------------------------------------ */
/* Step tableaus  (replace torchsde/_core/methods/<name>.py  .step bodies)        */
/* `g*` arguments are (rows,d) for DIAGONAL and (rows,d,m) for GENERAL.      */
/* GENERAL accepts any d and any m the Brownian source accepts (counter     */
/* noise: m <= 2^26), whether or not one row's increments fit in shared     */
/* memory.                                                                  */
/* ------------------------------------------------------------------------ */

/* y1 = y0 + f*dt + g.dW                    methods/euler.py:36
 * also Heun predictor heun.py:42, midpoint corrector midpoint.py:43,
 * additive-noise Milstein milstein.py:72 with gdg == 0 (base_sde.py:157-158) */
int tsde_step_euler(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                    const void* f, const void* g, double dt, void* y1);

/* grad_outputs of Milstein's vjp: go = g * (0.5 * v), v = dW^2 - dt (Ito) or dW^2
 * (Stratonovich).  methods/milstein.py:56,69,80-81,90-91; base_sde.py:127-155.
 * DIAGONAL: go (rows,d).  GENERAL (scalar noise): go (rows,d,m) = g * v2[:,None,:]. */
int tsde_milstein_vjp_seed(const tsde_launch* L, const tsde_noise* nz, const void* g,
                           double dt, int32_t ito, void* go);

/* y1 = y0 + f*dt + g.dW + gdg              methods/milstein.py:72 */
int tsde_step_milstein(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                       const void* f, const void* g, const void* gdg, double dt, void* y1);

/*
 * A whole diagonal-noise Milstein step (milstein.py:68-72) for an SDE whose f(t, y), g(t, y) and the vjp of g
 * are element-wise programs: one launch reads y0, draws dW, evaluates
 *     f, g (program), go = g * (0.5 * v) (as tsde_milstein_vjp_seed), gdg = vjp(go) (program),
 *     y1 = ((y0 + f*dt) + g*dW) + gdg (as tsde_step_milstein)
 * in registers and writes y1.  The program restates ATen ops one IEEE rounding each, in the order they ran, so
 * the step equals the unfused one bit for bit.
 *
 * Program: `n_instr` instructions; [0, n_fg) compute f and g, [n_fg, n_instr) the vjp.  An instruction writes
 * register `dst` (< n_regs <= TSDE_PW_MAX_REGS) from sources `a`, `b` (b unused by NEG / SQRT / ABS).  A source
 * is a register, TSDE_PW_SRC_Y (y0), TSDE_PW_SRC_GO (the seed go, vjp part only) or TSDE_PW_OPERAND(k).  f_src,
 * g_src (read after n_fg instructions) and gdg_src (read at the end) name the three results.  Opcodes, each the
 * expression of the ATen CUDA kernel it restates, in the state dtype T:
 *   MUL a * b   ADD a + b   SUB a - b   DIV a / b   NEG -a   SQRT sqrt(a)    (6, 7: reserved, invalid)
 *   LT  a < b ? 1 : 0    LE a <= b ? 1 : 0    EQ a == b ? 1 : 0    (a boolean is T(0) or T(1))
 *   MAXIMUM  isnan(a) ? a : isnan(b) ? b : max(a, b)    (torch.maximum; clamp with a non-NaN lower bound)
 *   MINIMUM  isnan(a) ? a : isnan(b) ? b : min(a, b)    (torch.minimum; clamp with a non-NaN upper bound)
 *   ABS  fabs(a)
 *   SEL  dst = dst != 0 ? a : b: the condition is the destination register itself, which must have been written
 *        (torch.where, masked_fill).
 * Transcendental opcodes (16 and up), valid only in the programs the library compiles (this Milstein layout, its
 * adaptive proposal, and the general layouts TSDE_PW_LAYOUT_GENERAL, _SRA, _EULER_HEUN and _REVERSIBLE_HEUN); the
 * interpreted entry points refuse them.  Each is the lambda of the ATen CUDA kernel it restates, in T, compiled apart from the
 * program with FMA contraction on, as ATen's kernels are (libdevice's exp, log, ... of T):
 *   EXP exp(a)   LOG log(a)   SIN sin(a)   COS cos(a)   TANH tanh(a)   LOG1P log1p(a)   EXPM1 expm1(a)
 *   RSQRT rsqrt(a)   SIGMOID 1 / (1 + exp(-a))   (unary: b unused)
 *   POW  pow(a, b), b an IMM operand (torch.pow with a scalar exponent off ATen's special cases)
 *   TANH_BACKWARD  a * (1 - b * b)   SIGMOID_BACKWARD  a * (1 - b) * b   (a the gradient, b the forward result)
 *   IMM      value `imm` (a value of the state dtype, stored as double)
 *   T0       the 0-d step time `t0` of the call (state dtype)
 *   SCALAR   ptr[0]                 (a one-element device tensor)
 *   CHANNEL  ptr[channel]           (a (d,) tensor broadcast over the rows)
 *   ROW      ptr[row * d + channel] (a (rows, d) tensor)
 * Device operands are read at every launch, after the kernel's dependency wait.  The struct is passed by value
 * to the kernel (it fits the 4 KiB parameter space), so a captured launch carries it.
 * Requires DIAGONAL noise, counter noise (nz->source == TSDE_SRC_COUNTER) and no 16-bit formats.
 */
#define TSDE_PW_MAX_INSTR 96
#define TSDE_PW_MAX_OPERANDS 24
#define TSDE_PW_MAX_REGS 24
#define TSDE_PW_SRC_Y 0xFE
#define TSDE_PW_SRC_GO 0xFF
#define TSDE_PW_OPERAND(k) (0x80 + (k))
enum { TSDE_PW_MUL = 0, TSDE_PW_ADD = 1, TSDE_PW_SUB = 2, TSDE_PW_DIV = 3, TSDE_PW_NEG = 4, TSDE_PW_SQRT = 5 };
enum { TSDE_PW_LT = 8, TSDE_PW_LE = 9, TSDE_PW_EQ = 10, TSDE_PW_MAXIMUM = 11, TSDE_PW_MINIMUM = 12, TSDE_PW_ABS = 13,
       TSDE_PW_SEL = 14 };
enum { TSDE_PW_EXP = 16, TSDE_PW_LOG = 17, TSDE_PW_SIN = 18, TSDE_PW_COS = 19, TSDE_PW_TANH = 20,
       TSDE_PW_LOG1P = 21, TSDE_PW_EXPM1 = 22, TSDE_PW_RSQRT = 23, TSDE_PW_SIGMOID = 24, TSDE_PW_POW = 25,
       TSDE_PW_TANH_BACKWARD = 26, TSDE_PW_SIGMOID_BACKWARD = 27 };
enum { TSDE_PW_IMM = 0, TSDE_PW_T0 = 1, TSDE_PW_SCALAR = 2, TSDE_PW_CHANNEL = 3, TSDE_PW_ROW = 4 };
typedef struct tsde_pw_instr {
  uint8_t op, dst, a, b;
} tsde_pw_instr;
typedef struct tsde_pw_operand {
  int32_t kind;
  int32_t reserved;
  const void* ptr;
  double imm;
} tsde_pw_operand;
typedef struct tsde_pointwise {
  int32_t n_instr, n_fg, n_regs, n_operands;
  uint8_t f_src, g_src, gdg_src, reserved;
  tsde_pw_instr instr[TSDE_PW_MAX_INSTR];
  tsde_pw_operand operand[TSDE_PW_MAX_OPERANDS];
} tsde_pointwise;
int tsde_step_milstein_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                 const void* y0, const void* t0, double dt, int32_t ito, void* y1);

/*
 * `n_steps` consecutive steps of tsde_step_milstein_pointwise as one launch: each thread reads its quad of y0 once,
 * runs step j = 0 .. n_steps-1 on the state the step before left in its registers, and stores step j's y1 only to
 * steps[j].y1 (an output row, the last state); a step whose y1 is NULL is not stored.  Step j draws its increment
 * from the one Brownian cell steps[j].cell_id of length steps[j].h (W = sqrt(h) N, the square root rounded once to
 * the state dtype, as for tsde_noise), runs the program at the 0-d time steps[j].t0 and uses steps[j].dt; every
 * stored y1 equals what tsde_step_milstein_pointwise gives step by step, bit for bit.  `nz` gives the key, the row
 * offset and the source (COUNTER); its cell_id and h are the first step's.  A step that spans several cells
 * (nz->n_cells > 1, merged as tsde_noise describes from steps[0].cell_id) must run alone (n_steps == 1).
 * TSDE_EINVAL: n_steps outside [1, TSDE_PW_MAX_STEPS], a null steps[j].t0, a null last y1, and whatever
 * tsde_step_milstein_pointwise refuses.  The step table is passed by value, so a captured launch carries it.
 */
#define TSDE_PW_MAX_STEPS 64
typedef struct tsde_pw_step {
  uint64_t    cell_id;  /* the step's Brownian cell                                     */
  double      h;        /* that cell's length                                           */
  double      dt;       /* the step's dt                                                */
  const void* t0;       /* DEVICE 0-d time of the step (state dtype), read by TSDE_PW_T0 */
  void*       y1;       /* where the step's y1 is stored, or NULL (not stored)          */
} tsde_pw_step;
int tsde_solve_milstein_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                  const void* y0, const tsde_pw_step* steps, int32_t n_steps, int32_t ito);

/*
 * The Milstein entry points above do not interpret `prog`: each program structure is compiled at run time into a
 * kernel of its own, with the program as straight-line register code (NVRTC, sm_90a, the IEEE options of the library
 * build), and loaded into a process-wide cache.  The structure is everything but the operand values and addresses
 * (instructions, n_regs, n_fg, the result sources, the operand kinds) and the dtype: programs that differ only in
 * IMM values or device pointers share one kernel, which reads those as launch parameters.  A program is compiled on
 * its first launch unless tsde_pointwise_compile compiled it before.
 *
 * tsde_pointwise_compile compiles and loads the kernels of Milstein program `prog` for the launches `L` describes
 * (its dtype; DIAGONAL noise, m == d) without launching anything: call it before a stream capture, since a capture
 * should not load modules.  Returns 0 (also for an empty launch, which compiles nothing), TSDE_EINVAL for a launch or
 * program tsde_solve_milstein_pointwise refuses, TSDE_ECOMPILE when NVRTC (libnvrtc.so.12) is not found or the
 * compilation fails (tsde_error_string(TSDE_ECOMPILE) then holds the compiler's log), or the cudaError_t of loading
 * the kernels.
 * tsde_pointwise_source writes the source compiled for such a program (at most `size` bytes, NUL-terminated, when
 * `buf` is given) and returns its length, or TSDE_EINVAL (0 for an empty launch); it needs no device.  Two programs
 * share a kernel exactly when their sources are equal.
 */
int tsde_pointwise_compile(const tsde_launch* L, const tsde_pointwise* prog);
int64_t tsde_pointwise_source(const tsde_launch* L, const tsde_pointwise* prog, char* buf, int64_t size);

/*
 * A whole diagonal-noise SRK (srid2) step (srk.py:57-88) for an SDE whose f(t, y) and g(t, y) are element-wise
 * programs: one launch reads y0, draws W and U, and evaluates the step's seven SDE calls and four tableau stages
 *     f0 = f(t_0, y0), g0 = g(t_0, y0); H0_1, H1_1 as tsde_srk_diag_stage1;
 *     f1 = f(t_1, H0_1), g1 = g(t_q, H1_1); H0_2, H1_2 as tsde_srk_diag_stage2;
 *     f2 = f(t_h, H0_2), g2 = g(t_1, H1_2); H1_3 as tsde_srk_diag_stage3; g3 = g(t_q, H1_3);
 *     y1 as tsde_step_srk_diag
 * in registers and writes y1.  t_0, t_1, t_q, t_h are the 0-d stage times t0 + 0*dt, t0 + dt, t0 + dt/4 and
 * t0 + dt/2 (state dtype), read at every launch; dt, rdt, sqrt_dt, three_dt are the scalars tsde_step_srk_diag
 * takes.  The step equals the unfused one bit for bit.
 *
 * Program: the tsde_pointwise layout above holds two programs.  Instructions [0, n_fg) are f, whose result is f_src;
 * [n_fg, n_instr) are g, whose result is g_src; gdg_src is unused.  Each program starts with no register defined
 * and reads only its own; TSDE_PW_SRC_Y is the state it is evaluated at, TSDE_PW_T0 its time, TSDE_PW_SRC_GO is
 * not a source.  The operand table is shared.  n_regs <= TSDE_PW_SRK_MAX_REGS: the kernel may keep six stage values
 * in the rest of the register file.
 * Requires DIAGONAL noise (a GENERAL launch runs an additive-noise sra1 step instead: TSDE_PW_LAYOUT_GENERAL_SRA
 * below), counter noise (nz->source == TSDE_SRC_COUNTER) and no 16-bit formats.
 */
#define TSDE_PW_SRK_MAX_REGS 18
int tsde_step_srk_diag_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                 const void* y0, const void* t_0, const void* t_1, const void* t_q,
                                 const void* t_h, double dt, double rdt, double sqrt_dt, double three_dt, void* y1);

/*
 * A whole diagonal-noise Stratonovich predictor-corrector step for an SDE whose f(t, y) and g(t, y) are element-wise
 * programs: one launch reads y0, draws dW, evaluates f0 = f(t0, y0) and g0 = g(t0, y0), and then, by `method`,
 *     TSDE_PC_HEUN        y' as tsde_step_euler (dt);         f', g' at (t_p, y'); y1 as tsde_step_heun (dt)
 *                         (heun.py:40-46, t_p = t1)
 *     TSDE_PC_MIDPOINT    y' as tsde_midpoint_predict (half_dt); f', g' at (t_p, y'); y1 as tsde_step_euler on
 *                         (y0, f', g') (dt)  (midpoint.py:34-43, t_p = t0 + half_dt)
 *     TSDE_PC_EULER_HEUN  y' as tsde_euler_heun_predict;       g' at (t_p, y');      y1 as tsde_step_euler_heun (dt)
 *                         (euler_heun.py:34-40, t_p = t1)
 * in registers and writes y1.  t0 and t_p are 0-d device times (state dtype), read at every launch; dt and half_dt
 * are the scalars the unfused kernels take (half_dt is read by TSDE_PC_MIDPOINT only).  The step equals the unfused
 * one bit for bit.
 *
 * Program: the two-program layout of tsde_step_srk_diag_pointwise (f in [0, n_fg), g in [n_fg, n_instr), gdg_src
 * unused, the operand table shared, TSDE_PW_SRC_GO not a source), with n_regs <= TSDE_PW_MAX_REGS.
 * Requires DIAGONAL noise, counter noise (nz->source == TSDE_SRC_COUNTER) and no 16-bit formats.  An unknown
 * `method` or a null time is TSDE_EINVAL.
 */
enum { TSDE_PC_HEUN = 0, TSDE_PC_MIDPOINT = 1, TSDE_PC_EULER_HEUN = 2 };
int tsde_step_predictor_corrector_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                            const void* y0, const void* t0, const void* t_p, int32_t method,
                                            double dt, double half_dt, void* y1);

/*
 * `n_steps` consecutive diagonal-noise Euler-Maruyama steps (euler.py:34-37) of an SDE whose f(t, y) and g(t, y) are
 * element-wise programs, as one launch: each thread reads its quad of y0 once and per step evaluates f and g at
 * (steps[j].t0, y) and forms y1 as tsde_step_euler (steps[j].dt), in registers.  The step table, the noise, what is
 * stored and the rule for steps that span several cells are those of tsde_solve_milstein_pointwise; a single step is
 * a chunk of one.  Every stored y1 equals the unfused step's bit for bit.
 * Program: the two-program layout of tsde_step_predictor_corrector_pointwise (n_regs <= TSDE_PW_MAX_REGS).
 * TSDE_EINVAL: whatever tsde_step_predictor_corrector_pointwise refuses, n_steps outside [1, TSDE_PW_MAX_STEPS], a
 * null steps[j].t0, a null last y1, and a step that spans several cells in a chunk of more than one.  An empty batch
 * is a no-op.
 */
int tsde_solve_euler_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                               const void* y0, const tsde_pw_step* steps, int32_t n_steps);

/*
 * `n_steps` consecutive diagonal-noise reversible Heun steps (reversible_heun.py:64-73) as one launch, under the rules
 * of tsde_solve_euler_pointwise.  The chunk starts from y0 and the solver state (z0, f0, g0), each read once, and per
 * step forms
 *     z1 as tsde_reversible_heun_z (dt);  f1, g1 at (steps[j].t0, z1);  y1 as tsde_step_reversible_heun on
 *     (y, f, f1, g, g1) with half_dt = 0.5 * dt rounded once to the state dtype;  (y, z, f, g) <- (y1, z1, f1, g1)
 * in registers.  steps[j].t0 is the time the program runs at, the step's t1.  The state after the last step is stored
 * once, to z1, f1 and g1, which must not overlap z0, f0 or g0.  Every stored value equals the unfused steps' bit for
 * bit when (state dtype) 0.5 * (state dtype) dt equals the unfused step's half_dt, which holds unless it is subnormal.
 * TSDE_EINVAL: as tsde_solve_euler_pointwise, and any null z0, f0, g0, z1, f1 or g1.
 */
int tsde_solve_reversible_heun_pointwise(const tsde_launch* L, const tsde_noise* nz, const tsde_pointwise* prog,
                                         const void* y0, const void* z0, const void* f0, const void* g0,
                                         const tsde_pw_step* steps, int32_t n_steps, void* z1, void* f1, void* g1);

/*
 * One proposal of an adaptive solve's step doubling, for an SDE whose f(t, y) and g(t, y) are element-wise programs:
 * one launch reads y0 and runs `method`'s step three times in registers,
 *     subs[0]  the full step from y0, stored to y_full;
 *     subs[1]  the first half step from y0, to the midpoint state (not stored);
 *     subs[2]  the second half step from the midpoint state, stored to y_next.
 * Each sub-step reads its increment from memory: w, and for SRK the space-time Levy area u, both (rows, d) tensors of
 * the state dtype (the Brownian motion's answers to the sub-step's query).  It runs the program at the 0-d device
 * times t[] (state dtype, read at every launch) and takes dt and the scalars s[] the unfused step takes:
 *     TSDE_PROPOSAL_EULER                    t[0] = t0; as tsde_solve_euler_pointwise
 *     TSDE_PROPOSAL_MILSTEIN_ITO / _STRATONOVICH
 *                                            t[0] = t0; as tsde_step_milstein_pointwise (Milstein layout; the
 *                                            program is compiled into a kernel of its own, as for that entry point)
 *     TSDE_PROPOSAL_SRK                      t[0..3] = t_0, t_1, t_q, t_h; s = (rdt, sqrt_dt, three_dt); as
 *                                            tsde_step_srk_diag_pointwise
 *     TSDE_PROPOSAL_HEUN, _MIDPOINT, _EULER_HEUN
 *                                            t[0] = t0, t[1] = t_p; midpoint: s[0] = half_dt; as
 *                                            tsde_step_predictor_corrector_pointwise
 * Both stored states equal the three unfused steps' bit for bit.  Requires DIAGONAL noise (m == d) and no 16-bit
 * formats.  TSDE_EINVAL: an unknown method, a null y0, subs, y_full or y_next, a null w (u for SRK) or time the
 * method reads, and a program of another layout than its method's; all checked before anything is compiled or
 * launched.  An empty batch is a no-op.
 *
 * tsde_adaptive_pointwise_compile compiles and loads the proposal kernel of Milstein program `prog` without
 * launching anything, under the rules of tsde_pointwise_compile; the proposal compiles it on first use otherwise.
 */
enum { TSDE_PROPOSAL_EULER = 0, TSDE_PROPOSAL_MILSTEIN_ITO = 1, TSDE_PROPOSAL_MILSTEIN_STRATONOVICH = 2,
       TSDE_PROPOSAL_SRK = 3, TSDE_PROPOSAL_HEUN = 4, TSDE_PROPOSAL_MIDPOINT = 5, TSDE_PROPOSAL_EULER_HEUN = 6 };
typedef struct tsde_pw_substep {
  const void* w;     /* DEVICE (rows, d) increment                                  */
  const void* u;     /* DEVICE (rows, d) space-time Levy area (SRK), else unused     */
  const void* t[4];  /* DEVICE 0-d times (state dtype); unused entries may be NULL   */
  double      dt;    /* the sub-step's dt                                            */
  double      s[3];  /* the method's scalars                                         */
} tsde_pw_substep;
int tsde_adaptive_proposal_pointwise(const tsde_launch* L, const tsde_pointwise* prog, int32_t method,
                                     const void* y0, const tsde_pw_substep* subs, void* y_full, void* y_next);
int tsde_adaptive_pointwise_compile(const tsde_launch* L, const tsde_pointwise* prog);

/*
 * General and additive noise.  tsde_solve_euler_pointwise, tsde_step_predictor_corrector_pointwise with
 * TSDE_PC_MIDPOINT, tsde_pointwise_compile and tsde_pointwise_source also take a GENERAL launch with
 * 1 <= L->m <= TSDE_PW_GENERAL_MAX_M, for an SDE whose f(t, y) is a (rows, d) element-wise program and whose g(t, y)
 * is a (rows, d, m) one, built from the same ops:
 *   tsde_solve_euler_pointwise               consecutive Euler steps, y1 = (y0 + f*dt) + g.dW as tsde_step_euler;
 *   tsde_step_predictor_corrector_pointwise  one midpoint step: y' as tsde_midpoint_predict (half_dt) at (t0, y0), y1
 *                                            as tsde_step_euler (dt) on f, g at (t_p, y'); other methods: TSDE_EINVAL.
 * Each thread owns a quad of d of one row; it draws the row's m increments on the channel-quad counters of the
 * general-noise kernels, evaluates g_ij in registers, channel by channel, and contracts it with them in the order the
 * unfused tsde_step_euler / tsde_midpoint_predict launch takes for a contiguous g (aligned unless g is a TSDE_PW_DM
 * operand at an unaligned address):
 *   m == 1                              one product g * dW (the row-wise kernels);
 *   m / 4 a power of two <= 32          per channel quad a fused multiply-add chain from 0, the quad sums added as a
 *                                       pairwise tree in natural order (the tile kernels);
 *   otherwise                           left to right from 0, one rounded multiply and add per channel;
 * so g never exists in memory and every stored state equals the unfused step's bit for bit.  The launches count
 * under TSDE_KERNEL_PW_GENERAL.
 *
 * Program: the two-program layout of tsde_step_predictor_corrector_pointwise, tagged reserved =
 * TSDE_PW_LAYOUT_GENERAL (an untagged program on a GENERAL launch is TSDE_EINVAL), with two more operand kinds that
 * only the g program may read:
 *   DM  ptr[channel * m + k]   (a dense (d, m) tensor broadcast over the rows)
 *   M   ptr[k]                 (an (m,) tensor broadcast over the rows and d)
 * where k is the Brownian channel.  A value computed from a DM or M operand is per channel; every other value, f's
 * result among them, is per (row, d) element and broadcast along m.  g_src may be any source, an operand included
 * (additive noise, `sigma.expand(rows, d, m)`).  As a Milstein program, it is compiled at run time into kernels of its
 * own (one translation unit per structure, dtype, m and contraction order, holding both methods' kernels), which
 * tsde_pointwise_compile compiles and loads and tsde_pointwise_source writes out for a GENERAL launch.  Counter noise
 * only, no 16-bit formats and no launch flags.  TSDE_EINVAL additionally: m outside [1, TSDE_PW_GENERAL_MAX_M] and a
 * DM or M operand read by f.
 */
#define TSDE_PW_GENERAL_MAX_M 32
enum { TSDE_PW_DM = 5, TSDE_PW_M = 6 };
#define TSDE_PW_LAYOUT_GENERAL 1 /* tsde_pointwise.reserved of a general-layout program (0 for the diagonal layouts) */

/*
 * Additive noise, SRA1 (methods/srk.py:90-111).  tsde_step_srk_diag_pointwise on a GENERAL launch with
 * 1 <= L->m <= TSDE_PW_GENERAL_MAX_M runs one SRK step of an element-wise SDE as one launch, for a program of the
 * general layout tagged reserved = TSDE_PW_LAYOUT_GENERAL_SRA.  t_0, t_1 and t_q are the 0-d times t0, t0 + dt and
 * t0 + 3/4 dt (state dtype); dt and rdt as tsde_step_srk_additive takes them; t_h, sqrt_dt and three_dt are unused.
 * The kernel evaluates f0 = f(t_0, y0), gA = g(t_1, y0) and gB = g(t_0, y0); H0_1 as tsde_srk_additive_stage on
 * (y0, f0, gA); f1 = f(t_q, H0_1); y1 as tsde_step_srk_additive on (y0, f0, f1, gA, gB).  It draws W and U on the
 * counters of those launches, forms each product's weights per channel as they do and contracts g with them in their
 * order: the orders above, except that m == 1 sums left to right from 0 (those launches take the generic kernel there,
 * whose 0 + g*w turns a -0 product into +0).  g never exists in memory and y1 equals the unfused step's bit for bit.
 * The launches count under TSDE_KERNEL_PW_GENERAL.  tsde_pointwise_compile and tsde_pointwise_source compile and
 * write out the program's sra1 kernels (a translation unit of their own) for a GENERAL launch and an SRA-tagged
 * program.  Counter noise only, no 16-bit formats and no launch flags.  TSDE_EINVAL additionally: a program without
 * the SRA tag and null times.  The Euler and midpoint GENERAL launches refuse an SRA-tagged program.
 */
#define TSDE_PW_LAYOUT_GENERAL_SRA 2 /* tsde_pointwise.reserved of a general-layout program for the sra1 step */

/*
 * General and additive noise, Stratonovich Euler-Heun and reversible Heun.  Two more tags of the general layout, each
 * compiled into a translation unit of its own by tsde_pointwise_compile and written out by tsde_pointwise_source:
 *   tsde_step_predictor_corrector_pointwise with TSDE_PC_EULER_HEUN on a GENERAL launch, for a program tagged
 *     TSDE_PW_LAYOUT_GENERAL_EULER_HEUN: one Euler-Heun step, f and g.dW at (t0, y0), y' as tsde_euler_heun_predict,
 *     g'.dW at (t_p, y') and y1 as tsde_step_euler_heun (dt);
 *   tsde_solve_reversible_heun_pointwise on a GENERAL launch, for a program tagged
 *     TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN: consecutive reversible-Heun steps as for diagonal noise, with g0 and g1
 *     the (rows, d, m) state (contiguous, not overlapping); each thread keeps its lanes' m values of g in registers.
 * Each contraction sums in the order the unfused launch takes, as above.  Euler-Heun's two launches see the same g
 * operand, so they take one order.  The reversible-Heun pair always reads a dense g (it refuses launch flags), so its
 * order is that of a contiguous aligned g, whatever the program's g source.  Every stored value equals the unfused
 * steps' bit for bit (reversible Heun: under the half-step condition of the diagonal chunk).  The launches count under
 * TSDE_KERNEL_PW_GENERAL.  TSDE_EINVAL, before anything is compiled or launched: a program with another tag (the
 * Euler / midpoint and sra1 programs among them), other predictor-corrector methods, m outside
 * [1, TSDE_PW_GENERAL_MAX_M], noise other than counter noise, launch flags, null times or state pointers, and what
 * the diagonal entry points refuse.
 */
#define TSDE_PW_LAYOUT_GENERAL_EULER_HEUN 3      /* tsde_pointwise.reserved for the general Euler-Heun step     */
#define TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN 4 /* tsde_pointwise.reserved for general reversible-Heun chunks */

/*
 * The backward sweep of the reversible-Heun adjoint (reversible_heun.py:98-144, adjoint.py:97-119) for a diagonal-noise
 * SDE whose f(t, y) and g(t, y) are element-wise programs.  tsde_solve_reversible_heun_pointwise on a DIAGONAL launch,
 * for a program tagged reserved = TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN (the `prog` member of a tsde_pw_adjoint, whose
 * other members it reads), runs `n_steps` consecutive backward steps as one launch.  Each thread reads its quad of the
 * augmented state once, (y, z, f, g) from y0, z0, f0, g0 and (adj_y, adj_f, adj_g, adj_z) from adj_in[], and per
 * step, in reversed time,
 *     z1, adj_f_mid, adj_g_mid as tsde_adjoint_reversible_heun_a (dt, half_dt);
 *     vjp_z and one contribution per parameter: the program's vjp with seeds (adj_f_mid, adj_g_mid) of f and g at the
 *       state z the step starts from (evaluated at (steps[j-1].t0, z), or (t0, z) for the chunk's first step);
 *     f1, g1 at (steps[j].t0, z1): steps[j].t0 is the forward time of the step's end;
 *     y, adj_y, adj_z, adj_f, adj_g as tsde_adjoint_reversible_heun_b (dt, half_dt); (z, f, g) <- (z1, f1, g1);
 *     when steps[j].y1 is not NULL (the step ends an output interval; it points at row k of ys, ys + k rows d):
 *       y <- ys[k], adj_y <- adj_y + grad_ys[k]
 * in registers, with half_dt = 0.5 * dt rounded once to the state dtype.  The state after the last step is stored
 * once, to y1, z1, f1, g1 and adj_out[], which must not overlap what the chunk reads.  Every stored value equals the
 * unfused sweep's (kernels A and B around the user's f, g and torch.autograd.grad) bit for bit when (state dtype) 0.5 *
 * (state dtype) dt is the unfused step's half_dt, which holds unless it is subnormal.  Parameter gradients are not
 * formed here: the chunk sums each parameter's contributions over its steps in registers, in step order, and adds that
 * sum to partial[k], a (rows, d) tensor, once, element-wise; the caller reduces each partial over the batch once per
 * sweep.  Nothing is accumulated with atomics, so every result is the same from run to run.  ys and grad_ys are
 * contiguous (n_out, rows, d) series of the state dtype.  The noise is that of tsde_solve_milstein_pointwise
 * (steps[j].cell_id, h; a step spanning several cells runs alone), on the global row (nz->row_offset).  The launches
 * count under TSDE_KERNEL_PW_ADJOINT.
 *
 * Program: prog holds f and g in [0, n_fg) with results f_src and g_src, as the Milstein layout; [n_fg, n_instr) is the
 * vjp, whose seeds are TSDE_PW_SRC_GO (f's cotangent) and TSDE_PW_SRC_GO2 (g's), with vjp_z in gdg_src and parameter
 * k's contribution in param_src[k] (0 <= n_params <= TSDE_PW_ADJ_MAX_PARAMS).  A contribution is the (rows, d) value
 * whose batch reduction is that parameter's gradient: the value itself for a (rows, d) parameter.  The program is
 * compiled at run time into a kernel of its own, as the Milstein programs are (one translation unit per structure,
 * n_params and dtype), with the library's IEEE options; tsde_pointwise_compile compiles and loads it for a DIAGONAL
 * launch without launching (call it before a stream capture) and tsde_pointwise_source writes out its source.
 *
 * Launch: 256 threads per CTA, bounded at one resident CTA per SM (__launch_bounds__(256, 1)), no shared memory.  The
 * kernel holds 8 state quads, the program's registers and one accumulator quad per parameter.  Measured on sm_90a
 * (ptxas of CUDA 12.9 on the generated source, DESIGN section 3): the program of profiles/adjoint_pointwise_probe.py
 * (f = mu*y - sigma*(sigma*(0.5*y)), g = sigma*y, (d,) mu and sigma) takes 121 / 102 registers (single- / multi-cell
 * kernel) in fp32 and 198 / 190 in fp64, with no spills.
 * TSDE_EINVAL, before anything is compiled or launched: a launch that is not DIAGONAL with m == d, noise other than
 * counter noise or with flags, 16-bit formats, an invalid program (tsde_pointwise_compile's checks with the second
 * seed, a bad n_params or param_src), n_steps outside [1, TSDE_PW_MAX_STEPS], a step spanning several cells in a chunk
 * of more than one, a null t0, steps[j].t0, state pointer, ys, grad_ys or partial[k], and a steps[j].y1 that is not one
 * of the n_out rows of ys.  The tag is valid only on the `prog` member of a tsde_pw_adjoint: the library reads the
 * whole struct behind a program so tagged.  An empty batch is a no-op.
 */
#define TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN 5 /* tsde_pointwise.reserved of a tsde_pw_adjoint's program */
#define TSDE_PW_ADJ_MAX_PARAMS 8
#define TSDE_PW_SRC_GO2 0xFD
/*
 * General and additive noise.  tsde_solve_reversible_heun_pointwise on a GENERAL launch with 2 <= L->m <=
 * TSDE_PW_GENERAL_MAX_M, for the `prog` member of a tsde_pw_adjoint tagged reserved =
 * TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN, runs the same backward steps with g, adj_g and their kernels A and B
 * as tsde_adjoint_reversible_heun_a / _b take them on a GENERAL launch: g0 (the g argument) and adj_in[2] are
 * (rows, d, m), and so are the chunk's g1 and adj_out[2] (contiguous, 16-byte aligned, not overlapping).  Each thread
 * runs one quad of d and keeps no (d, m) block in registers: g at (t, z) is re-evaluated channel by channel from the
 * program, and adj_g is carried in kernel B's rank-2 form (adj_y and adj_z per lane, the step's m increments per
 * thread); only the chunk's first step reads g0 and adj_in[2].  Each contraction with the increments sums in the order
 * of the unfused launch's route, and vjp_z's channel sums in the order of ATen's CUDA sum over the last dimension, so
 * every stored value equals the unfused sweep's bit for bit under the half-step condition above.
 *
 * Program: the general layout's f and g in [0, n_fg) (g per channel, with DM and M operands), and the vjp in
 * [n_fg, n_instr) with seeds TSDE_PW_SRC_GO ((rows, d)) and TSDE_PW_SRC_GO2 (per channel, adj_g_mid).  An instruction
 * is per channel when one of its sources is; TSDE_PW_CSUM (source a only, valid in this layout only) is the channel
 * sum of a per-channel value, a (rows, d) value.  A per-channel instruction may not read a value computed from a
 * channel sum.  f_src and gdg_src (vjp_z) are (rows, d) values; param_src[k] may be either: a (rows, d) contribution is
 * summed over the chunk in registers and added to partial[k], (rows, d), once; a per-channel one is added to
 * partial[k], (rows, d, m), at every step, element by element, by the thread that owns the element.  The launches count
 * under TSDE_KERNEL_PW_ADJOINT; tsde_pointwise_compile and tsde_pointwise_source compile and write out the program on
 * a GENERAL launch.  TSDE_EINVAL, before anything is compiled or launched: m outside [2, TSDE_PW_GENERAL_MAX_M], noise
 * other than counter noise or with flags, an invalid program, and what the diagonal tag refuses.
 */
#define TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN 6 /* ... of a general-noise tsde_pw_adjoint's program */
enum { TSDE_PW_CSUM = 28 };

typedef struct tsde_pw_adjoint {
  tsde_pointwise prog;
  int32_t n_params;
  int32_t reserved;
  uint8_t param_src[TSDE_PW_ADJ_MAX_PARAMS];
  /* DEVICE buffers of a launch */
  const void* t0;                             /* 0-d forward time of the chunk's first forward values (state dtype) */
  const void* adj_in[4];                      /* adj_y, adj_f, adj_g, adj_z the chunk starts from                   */
  void*       y1;                             /* where the chunk leaves y                                           */
  void*       adj_out[4];                     /* and adj_y, adj_f, adj_g, adj_z                                     */
  const void* ys;                             /* the output series and its cotangent, (n_out, rows, d)              */
  const void* grad_ys;
  int64_t     n_out;
  void*       partial[TSDE_PW_ADJ_MAX_PARAMS];
} tsde_pw_adjoint;

/* derivative-free Milstein, predictor: y' = y0 + (Ito ? dt*f : 0) + g*sqrt_dt
 * methods/milstein.py:58-63,83-84,93-94.  g is (rows,d) also for scalar noise (squeezed). */
int tsde_milstein_gf_predict(const tsde_launch* L, const void* y0, const void* f,
                             const void* g, double dt, double sqrt_dt, int32_t ito, void* yp);

/* derivative-free Milstein, corrector:
 * y1 = y0 + f*dt + g.dW + ((g'-g).v) / (2*sqrt_dt)      methods/milstein.py:64-72 */
int tsde_step_milstein_gf(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                          const void* f, const void* g, const void* gp, double dt,
                          double two_sqrt_dt, int32_t ito, void* y1);

/* y1 = y0 + (dt*(f+f') + g.dW + g'.dW) * 0.5             methods/heun.py:46 */
int tsde_step_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0, const void* f,
                   const void* fp, const void* g, const void* gp, double dt, void* y1);

/* y' = y0 + half_dt*f + 0.5*(g.dW)                        methods/midpoint.py:36-38 */
int tsde_midpoint_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                          const void* f, const void* g, double half_dt, void* yp);

/* y' = y0 + g.dW                                          methods/euler_heun.py:36 */
int tsde_euler_heun_predict(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                            const void* g, void* yp);

/* y1 = y0 + dt*f + (g.dW + g'.dW)*0.5                     methods/euler_heun.py:40 */
int tsde_step_euler_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                         const void* f, const void* g, const void* gp, double dt, void* y1);

/* z1 = 2*y0 - z0 + f0*dt + g0.dW                          methods/reversible_heun.py:69 */
int tsde_reversible_heun_z(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                           const void* z0, const void* f0, const void* g0, double dt, void* z1);

/* y1 = y0 + (f0+f1)*(0.5*dt) + (g0+g1).(0.5*dW)           methods/reversible_heun.py:71 */
int tsde_step_reversible_heun(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                              const void* f0, const void* f1, const void* g0, const void* g1,
                              double half_dt, void* y1);

/*
 * Roessler SRI2 (srid2), diagonal or scalar noise: methods/srk.py:57-88 with
 * methods/tableaus/srid2.py:19-54.  The reference re-evaluates earlier stages;
 * only 3 distinct f and 4 distinct g evaluations exist (rows with zero
 * coefficients add exact zeros).  g arguments are (rows,d) (squeezed for scalar).
 *   stage1: H0_1 = y0 + f0*dt ; H1_1 = y0 + 1/4 f0 dt - 1/2 g0 sqrt_dt          (srk.py:74-75, s=1)
 *   stage2: H0_2 = y0 + 1/4 f0 dt + g0 U/dt + 1/4 f1 dt + 1/2 g1 U/dt ;
 *           H1_2 = y0 + f0 dt + g0 sqrt_dt                                      (s=2)
 *   stage3: H1_3 = y0 + 2 g0 sqrt_dt - g1 sqrt_dt + 1/4 f2 dt + 1/2 g2 sqrt_dt  (s=3)
 *   final : y1 = y0 + sum_s alpha_s f_s dt + g_s * gw_s                         (srk.py:80-87)
 */
int tsde_srk_diag_stage1(const tsde_launch* L, const void* y0, const void* f0, const void* g0,
                         double dt, double sqrt_dt, void* h0_1, void* h1_1);
int tsde_srk_diag_stage2(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                         const void* f0, const void* g0, const void* f1, const void* g1,
                         double dt, double rdt, double sqrt_dt, void* h0_2, void* h1_2);
int tsde_srk_diag_stage3(const tsde_launch* L, const void* y0, const void* g0, const void* g1,
                         const void* f2, const void* g2, double dt, double sqrt_dt, void* h1_3);
int tsde_step_srk_diag(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                       const void* f0, const void* f1, const void* f2, const void* g0,
                       const void* g1, const void* g2, const void* g3, double dt, double rdt,
                       double sqrt_dt, double three_dt, void* y1);

/*
 * Roessler SRA1, additive noise: methods/srk.py:90-111 with tableaus/sra1.py:19-36.
 *   stage : H0_1 = y0 + 3/4 f0 dt + gA.(3/2 U/dt)            gA = g(t1, y0)
 *   final : y1 = y0 + 1/3 f0 dt + gA.(W - U/dt) + 2/3 f1 dt + gB.(U/dt)   gB = g(t0, y0)
 */
int tsde_srk_additive_stage(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                            const void* f0, const void* ga, double dt, double rdt, void* h0_1);
int tsde_step_srk_additive(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                           const void* f0, const void* f1, const void* ga, const void* gb,
                           double dt, double rdt, void* y1);

/* ys[i] = (t1-t)/(t1-t0)*y0 + (t-t0)/(t1-t0)*y1     _core/interp.py:15-18; w0,w1 host-computed */
int tsde_linear_interp(const tsde_launch* L, const void* y0, const void* y1, double w0,
                       double w1, void* out);

/* Adaptive stepping: out[0] (double) = sum over all (rows*d) elements of ((y11 - y12)/tol)^2 with
 * tol = clamp_min(rtol*max(|y11|,|y12|) + atol, eps)   _core/adaptive_stepping.py:42-76 (compute_error, _rms).
 * scratch: device buffer of >= 592 doubles.  The host finishes with sqrt(out/numel).clamp_min(eps). */
int tsde_adaptive_error_sumsq(const tsde_launch* L, const void* y11, const void* y12, double rtol,
                              double atol, double eps, void* scratch, void* out);

/* ------------------------------------------------------------------------ */
/* Reversible-Heun adjoint  (methods/reversible_heun.py:98-144)              */
/* ------------------------------------------------------------------------ */

/* First half (:103-115): z1 = 2*y0 - z0 - f0*dt - g0.dW ;
 *   adj_f0' = adj_f0 + adj_y0*half_dt ; adj_g0' = adj_g0 + adj_of_prod(adj_y0, half_dW).
 * adj_g* are (rows,d) for DIAGONAL and (rows,d,m) otherwise (outer product :95-96). */
int tsde_adjoint_reversible_heun_a(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                                   const void* z0, const void* f0, const void* g0,
                                   const void* adj_y0, const void* adj_f0, const void* adj_g0,
                                   double dt, double half_dt, void* z1, void* adj_f0_out,
                                   void* adj_g0_out);

/* Second half (:130-140): adj_z0' = adj_z0 + vjp_z ;
 *   y1 = y0 - (f0+f1)*half_dt - (g0+g1).half_dW ; adj_y1 = adj_y0 + 2*adj_z0' ;
 *   adj_z1 = -adj_z0' ; adj_f1 = adj_y0*half_dt + adj_z0'*dt ;
 *   adj_g1 = adj_of_prod(adj_y0, half_dW) + adj_of_prod(adj_z0', dW). */
int tsde_adjoint_reversible_heun_b(const tsde_launch* L, const tsde_noise* nz, const void* y0,
                                   const void* f0, const void* f1, const void* g0,
                                   const void* g1, const void* adj_y0, const void* adj_z0,
                                   const void* vjp_z, double dt, double half_dt, void* y1,
                                   void* adj_y1, void* adj_z1, void* adj_f1, void* adj_g1);

#ifdef __cplusplus
}
#endif
#endif /* TORCHSDE_B200_H_ */
