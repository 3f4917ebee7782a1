"""Element-wise tapes of the user's SDE: a diagonal-noise Milstein, SRK, Heun, midpoint, Euler-Heun, Euler or
reversible-Heun step as one kernel, and an adaptive solve's proposal (a full step and two half steps) as one kernel.

When the SDE's callables are made only of element-wise ATen ops whose CUDA result is one IEEE rounding per element,
a whole step is one launch that reads y0 and writes y1 (include/torchsde_b200.h, csrc/pointwise.cu) instead of the
user's ATen launches and the tableau kernels between them.  How the program is obtained: the first step of the solve
runs the ordinary way under a recorder, a TorchDispatchMode that sees every ATen op that actually runs, and the tape
is compiled (dead-code elimination, linear-scan register allocation) into a tsde_pointwise program that every later
step runs.

What a tape may hold, for both methods.  The tape accepts only

    mul; add / sub / rsub with alpha = +-1 (any other alpha lets ATen contract to an FMA); neg; sqrt;
    div by a tensor; div by a CPU scalar (ATen computes a * (1/b), with 1/b rounded in the state dtype);
    pow(x, 2) (ATen computes x * x); aliasing views that keep every element where it is (no-ops);

and the ops that do not round, or round once, each restated as its ATen CUDA kernel computes it, NaN and signed zeros
included:

    abs; sign / sgn ((0 < x) - (x < 0)); reciprocal (1 / x); maximum / minimum (NaN-propagating); clamp, clamp_min,
    clamp_max with scalar bounds that are not NaN or with tensor bounds (maximum with the lower bound, then minimum
    with the upper one), relu (clamp_min(x, 0)); lt / le / gt / ge / eq / ne (.Scalar and .Tensor); where.self;
    masked_fill(_).Scalar; logical_and / or / not and their bitwise forms on bools (and in place); threshold_backward
    (x <= threshold ? 0 : grad); scalar_tensor (an immediate: autograd's clamp and where backward emit it),

on operands that are the state y, the 0-d time t the callable was given, Python numbers and CPU 0-d tensors
(immediates, rounded to the state dtype as ATen rounds them), one-element device tensors, (d,)-shaped device tensors
broadcast over the rows and (rows, d) device tensors, all of the state dtype, on y's device and contiguous.  Anything
else — another op, a reduction, `.item()`, an in-place op on anything the tape did not produce, a read of a tensor
whose storage was written in place through another tensor (a view, `detach()`, `.data`), an operand that shares
storage with a value of the tape, a 16-bit result, a tensor created by a factory — rejects the tape, and the solve
keeps its ordinary step.

Transcendental ops, with options={'transcendental': True} only (`Recorder.transcendental`, `_allow`):

    exp, log, sin, cos, tanh, log1p, expm1, rsqrt, sigmoid; tanh_backward and sigmoid_backward (what autograd emits
    for tanh and sigmoid in Milstein's vjp); pow with a scalar exponent as ATen's CUDA kernel dispatches it (`_pow`:
    0.5 sqrt, -0.5 rsqrt, -1 reciprocal, then the exponent rounded to the state dtype: 2 and 3 products, -2 one over
    the square, any other a pow, 0 and 1 rejected).

They are libdevice code, not correctly rounded, and ATen's kernels contract their arithmetic into FMAs: the library
compiles each as a function of its own with ATen's lambda as its body and FMA contraction on, and links it to the
program (csrc/pointwise.cu, kPwHelpers), so only the compiled layouts take them: Milstein (fixed-step and adaptive)
and the general / additive-noise Euler, midpoint, sra1, Euler-Heun and reversible-Heun kernels.  The interpreted ones (`SrkRecorder` on diagonal
noise: SRK, Heun, midpoint, Euler-Heun, Euler, reversible Heun) reject such a tape with the reason.  So does every
recorder when the NVRTC the library compiles with is not the CUDA release PyTorch was built with (`nvrtc_mismatch`),
or when there is no nvJitLink to link with (loaded only then, `_cabi.nvjitlink`).
Without the option the tapes hold what they always held: the default keeps the unfused step for these SDEs.

Bools.  A comparison or logical result is a bool tensor; in the program it is a register holding 0 or 1 of the state
dtype (logical_and is then a product, logical_or a maximum, logical_not 1 - c, ne 1 - eq, gt / ge lt / le with the
operands swapped, all exact).  A bool may only be the condition of where / masked_fill or an operand of a logical op:
one used as a number (in arithmetic, a comparison, `.float()`), returned as f, g or the vjp, or a bool tensor from
outside the tape (a user mask) rejects the tape.  where(c, a, b) compiles to SEL, whose condition is its destination
register: c's own register when this is c's last read, else a copy of it (`_allocate`).

Device operands are passed by address and read at every launch: in-place updates of parameters (optimiser steps) are
followed, exactly as by a captured CUDA graph; f and g must not depend on anything else (the purity contract of
graph capture, README).  SDEs whose callables have side effects say so with options={'overlap': False}, and keep
calling them every step.

Milstein (`Recorder`, tsde_step_milstein_pointwise).  The unfused step runs five full-batch passes: the user's f and
g, the vjp seed, autograd's vjp of g and the tableau (methods.BaseMilstein._step).  The tape has three segments:
f(t0, y), g(t0, y) and torch.autograd.grad(g, y, go), in which the seed go is one more operand.  The vjp is not
derived symbolically: autograd's own op sequence (`grad * other`, the `add` that accumulates a twice-used `y`, ...)
is what decides the bits, so it is what gets recorded.  The three segments are one program: the vjp part may read
what the f / g part computed.  When the batch fills the GPU, up to TSDE_PW_MAX_STEPS consecutive steps run as one
launch of tsde_solve_milstein_pointwise with the state in registers (`plan_chunks`, `chunk_length`, `solve_chunk`).
The library does not interpret a Milstein program: it writes it out as CUDA with the program as straight-line register
code and compiles it at run time (NVRTC, sm_90a, the IEEE options of its own build), one kernel per program structure
and dtype, shared by every SDE of that structure whatever its parameter values.  The step compiles it right after
`Recorder.finish` (`compile_milstein`, tsde_pointwise_compile), on the recording step: the warm-up and capture of a
graph solve come later and never load a module.  If it cannot be compiled (no NVRTC, or a compiler error) the tape is
rejected with the compiler's reason and the solve keeps the ordinary step.

SRK (`SrkRecorder`, tsde_step_srk_diag_pointwise).  The step's seven evaluations, f at three (t, y) and g at four
(methods.SRK._diagonal_or_scalar_step), are recorded one by one; a value of one evaluation is not an operand of
another.  The tape is accepted when the three f evaluations are the same ops on the same operands and so are the four
g evaluations; the first of each is compiled, as two programs that share an operand table.

Heun, midpoint and Euler-Heun (`SrkRecorder` with pattern 'fgfg' or 'fgg', tsde_step_predictor_corrector_pointwise).
The Stratonovich predictor-corrector steps (methods.Heun, Midpoint, EulerHeun) evaluate f and g at (t0, y0) and again
at the predicted state (g only for Euler-Heun).  They are recorded and compiled as SRK's are, with the full register
bound.  Only SDEs whose f and g the step calls as two separate callables are recorded (`pc_recorder`): a user
`f_and_g`, `g_prod` or `f_and_g_prod`, and the adjoint SDE of `sdeint_adjoint`'s backward, keep the ordinary step.

Euler and reversible Heun (`pc_recorder` with pattern 'fg', tsde_solve_euler_pointwise,
tsde_solve_reversible_heun_pointwise).  Both evaluate f and g once per step: Euler at (t0, y0), reversible Heun at
(t1, z1), after its z kernel (methods.Euler, ReversibleHeun).  They are recorded as Heun is and run as Milstein does:
up to TSDE_PW_MAX_STEPS steps per launch once the batch fills the GPU, a single step being a chunk of one.
Reversible Heun's solver state (f, g, z) stays in registers inside a chunk and is stored at its end, alternately to
two sets of solver-owned buffers; its half step T(0.5) * T(dt) must equal the unfused step's half_dt at every step
(`halves_exactly`), and the state it starts from must be tensors of the state dtype of the shapes the kernel reads
(`state_fits`), else
the solve keeps the ordinary step.  `sdeint_adjoint`'s forward solve is a no-grad solve, so the reversible pair's
forward steps fuse too.

Adaptive (`proposing`, `propose`, tsde_adaptive_proposal_pointwise).  An adaptive solve proposes a full step and two
half steps and compares them (BaseSDESolver._integrate_adaptive, `_propose`).  Its Brownian motion is queried at
data-dependent times, so it is never bound to a grid and the kernels above, which draw counter noise, do not apply.
For Euler, Milstein, SRK, Heun, midpoint and Euler-Heun, the first proposal runs unfused and its full step records
the program with the method's usual recorder (Milstein compiles the proposal kernel of its program instead of the
fixed-step ones, `compile_milstein`).  Every later proposal makes the three Brownian queries the unfused steps make,
in the same order and with the same arguments, and then one launch reads y0, runs the method's step three times on
those increments (the midpoint state stays in registers) and writes y_full and y_next.  The error reduction
(tsde_adaptive_error_sumsq) and the host's accept / reject logic are unchanged, so the solve's outputs, its accepted
steps and its queries are the unfused solve's, bit for bit.  The conditions are those of `eligible`, with a Brownian
motion whose answers have the state's shape in place of the grid binding; gradients through the solve and the
backward solve of `sdeint_adjoint` keep the unfused steps.  Reversible Heun keeps them too: its solver state carries
over from one proposal to the next.

General and additive noise (`GeneralRecorder`, `general`, `compile_general`).  Fixed-step Euler and midpoint solves
with 1 <= m <= TSDE_PW_GENERAL_MAX_M Brownian channels record f as above and g as a (rows, d, m) value of the same ops,
with per-channel operands ((d, m) and (m,) tensors) and `y.unsqueeze(-1)`; the program is compiled into kernels of its
own that evaluate g_ij in registers and contract it with the increments in the unfused launch's summation order, and
they run on the solver's GENERAL launch of tsde_solve_euler_pointwise (chunks, as Euler's) and
tsde_step_predictor_corrector_pointwise (midpoint).  A fixed-step additive-noise SRK solve (sra1) records its step's
four evaluations f0, gA, gB, f1 the same way (pattern 'fggf'); its program is tagged PW_LAYOUT_GENERAL_SRA and every
later step is one launch of tsde_step_srk_diag_pointwise on the solver's GENERAL launch, which draws W and U and
contracts g three times, with the weights of the unfused stage and final launches.  Fixed-step Euler-Heun ('fgg') and
reversible Heun ('fg' at (t1, z1)) record the same way; their programs are tagged PW_LAYOUT_GENERAL_EULER_HEUN and
_REVERSIBLE_HEUN (the solver's `_pw_layout`: reversible Heun's pattern is Euler's) and run as one launch of
tsde_step_predictor_corrector_pointwise per Euler-Heun step, and as chunks of tsde_solve_reversible_heun_pointwise whose
solver state holds g as (rows, d, m), kept in registers within a chunk; `sdeint_adjoint`'s forward solve fuses too.
Heun and every other method keep diagonal-only tapes.

The reversible adjoint's backward sweep (`AdjointRecorder`, `compile_adjoint`, `solve_adjoint_chunk`), with
`sdeint_adjoint(..., adjoint_options={'fused_backward': True})`.  Its first backward step runs the ordinary way under
the recorder in three segments: f and g at (t0, z0); torch.autograd.grad of both with respect to z0 and the parameters
with two seeds (GO, f's cotangent, and GO2, g's); f and g at (t1, z1), which must be the first segment's program.  The
program's results are f, g, vjp_z and one contribution per parameter: the (rows, d) value whose batch reduction autograd
returns as that parameter's gradient (on a parameter's path the tape holds autograd's sum_to reductions, views and the
`add` of two of them, nothing else).  It is tagged PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN, compiled right after recording,
and every step of the sweep then runs in chunks of tsde_solve_reversible_heun_pointwise, each contribution summed in
registers and added once per chunk to a (rows, d) partial that the sweep reduces over the batch once at its end
(adjoint._BackwardEngine._fused_sweep).  y, the adjoint state and y0's gradient are the unfused sweep's bits; parameter
gradients differ by summation order only.  Only diagonal noise on a bound grid, without logqp, autocast, overlap=False,
adjoint_adaptive, create_graph or a user f_and_g (`adjoint_refusal`); anything else keeps the unfused sweep and warns.
"""
import ctypes
import numbers
import weakref

import numpy as np
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from .. import _cabi
from ..settings import NOISE_TYPES

aten = torch.ops.aten

# op -> (opcode, swap operands)
_BINARY = {
    aten.mul.Tensor: (_cabi.PW_MUL, False), aten.mul.Scalar: (_cabi.PW_MUL, False),
    aten.add.Tensor: (_cabi.PW_ADD, False), aten.add.Scalar: (_cabi.PW_ADD, False),
    aten.sub.Tensor: (_cabi.PW_SUB, False), aten.sub.Scalar: (_cabi.PW_SUB, False),
    aten.rsub.Tensor: (_cabi.PW_SUB, True), aten.rsub.Scalar: (_cabi.PW_SUB, True),
    aten.div.Tensor: (_cabi.PW_DIV, False), aten.div.Scalar: (_cabi.PW_DIV, False),
}
_UNARY = {aten.neg.default: _cabi.PW_NEG, aten.sqrt.default: _cabi.PW_SQRT, aten.abs.default: _cabi.PW_ABS}
# comparisons: op -> (opcode, swap operands); gt / ge are lt / le with the operands swapped, exactly (NaN included)
_COMPARE = {}
for _name, _entry in (('lt', (_cabi.PW_LT, False)), ('le', (_cabi.PW_LE, False)), ('gt', (_cabi.PW_LT, True)),
                      ('ge', (_cabi.PW_LE, True)), ('eq', (_cabi.PW_EQ, False)), ('ne', (_cabi.PW_EQ, False))):
    for _overload in ('Tensor', 'Scalar'):
        _COMPARE[getattr(getattr(aten, _name), _overload)] = _entry
_NEGATED = {aten.ne.Tensor, aten.ne.Scalar}  # 1 - eq
# logical ops of comparison results (0 or 1): and is a product, or a maximum, not 1 - c (`&`, `|`, `~` of bool
# tensors are the bitwise ops)
_LOGICAL = {aten.logical_and.default: _cabi.PW_MUL, aten.bitwise_and.Tensor: _cabi.PW_MUL,
            aten.logical_or.default: _cabi.PW_MAXIMUM, aten.bitwise_or.Tensor: _cabi.PW_MAXIMUM,
            aten.logical_not.default: _cabi.PW_SUB, aten.bitwise_not.default: _cabi.PW_SUB}
_IN_PLACE = {aten.mul_.Tensor: aten.mul.Tensor, aten.add_.Tensor: aten.add.Tensor,
             aten.sub_.Tensor: aten.sub.Tensor, aten.div_.Tensor: aten.div.Tensor,
             aten.masked_fill_.Scalar: aten.masked_fill.Scalar, aten.logical_and_.default: aten.logical_and.default,
             aten.logical_or_.default: aten.logical_or.default, aten.bitwise_and_.Tensor: aten.bitwise_and.Tensor,
             aten.bitwise_or_.Tensor: aten.bitwise_or.Tensor}
# the transcendental ops (options={'transcendental': True}; the compiled layouts only): op -> opcode, with the unary
# ones' operand in source a and the backward ops' gradient in a, their forward result in b
_TRANSCENDENTAL = {aten.exp.default: _cabi.PW_EXP, aten.log.default: _cabi.PW_LOG, aten.sin.default: _cabi.PW_SIN,
                   aten.cos.default: _cabi.PW_COS, aten.tanh.default: _cabi.PW_TANH,
                   aten.log1p.default: _cabi.PW_LOG1P, aten.expm1.default: _cabi.PW_EXPM1,
                   aten.rsqrt.default: _cabi.PW_RSQRT, aten.sigmoid.default: _cabi.PW_SIGMOID}
_BACKWARD = {aten.tanh_backward.default: _cabi.PW_TANH_BACKWARD,
             aten.sigmoid_backward.default: _cabi.PW_SIGMOID_BACKWARD}
_ALIAS = {aten.view.default, aten._unsafe_view.default, aten.expand.default, aten.unsqueeze.default,
          aten.detach.default, aten.alias.default}

Y, GO, GO2, T0 = ('y',), ('go',), ('go2',), ('t0',)
STALE = ('stale',)  # a tensor whose storage was written in place through another tensor
FOREIGN = ('foreign',)  # a value bound by an earlier evaluation of an SRK step


class Reject(Exception):
    pass


def nvrtc_mismatch():
    """Why the transcendental ops cannot be compiled to ATen's bits here, or None.  They are libdevice code, which is
    not correctly rounded: the program's NVRTC must be the CUDA release (major.minor) PyTorch was built with."""
    have, want = _cabi.nvrtc_version(), torch.version.cuda
    if have is None:
        return "no NVRTC to compile the transcendental ops with"
    if want is None or tuple(int(x) for x in want.split('.')[:2]) != have:
        return (f"NVRTC {have[0]}.{have[1]} is not the CUDA {want} that PyTorch was built with: its libdevice may "
                f"compute the transcendental ops otherwise")
    return None


def transcendental(solver):
    """Whether `solver` fuses the transcendental ops (options={'transcendental': True})."""
    return bool(solver.options.get('transcendental', False))


def _strip(shape):
    """Shape without its leading ones: the element mapping of a tensor broadcast right-aligned to (rows, d)."""
    shape = tuple(shape)
    while shape and shape[0] == 1:
        shape = shape[1:]
    return shape


def _allocate(instrs, reads):
    """Dead-code elimination and register allocation of one tape.  `instrs` are (opcode, value id, source, source,
    condition), the condition being SEL's (else None); `reads` are the (position, source) at which the kernel reads a
    result: after the instructions before `position` have run, so the value is kept until then.  Returns the
    instructions that remain as (position in `instrs`, opcode, register, code, code), the code of each read's source,
    and the number of registers."""
    last = {}
    for pos, v in reads:
        if v[0] == 'v':
            last[v] = max(last.get(v, -1), pos)
    live = []
    for i in range(len(instrs) - 1, -1, -1):
        op, v, *srcs = instrs[i]
        if v not in last:
            continue
        live.append(i)
        for s in srcs:
            if s is not None and s[0] == 'v':
                last[s] = max(last.get(s, -1), i)
    live.reverse()
    # registers: linear scan; a register whose value was last read by this instruction may be its destination
    reg, held, free, n_regs = {}, [], [], 0  # value -> its register; the values whose register is in use

    def code(s):
        if s == Y:
            return _cabi.PW_SRC_Y
        if s == GO:
            return _cabi.PW_SRC_GO
        if s == GO2:
            return _cabi.PW_SRC_GO2
        if s[0] == 'k':
            return _cabi.PW_OPERAND0 + s[1]
        return reg[s]

    def fresh():
        nonlocal n_regs
        if free:
            return free.pop()
        n_regs += 1
        return n_regs - 1

    out = []
    for i in live:
        op, v, a, b, c = instrs[i]
        ca, cb = code(a), code(b) if b is not None else 0
        if c is not None:
            # SEL reads its condition from its destination: the condition's own register when this is its last read,
            # else a copy (maximum(c, c) is c exactly), made before the sources below are released
            if last[c] <= i:
                held.remove(c)
                reg[v] = reg[c]
            else:
                reg[v] = fresh()
                out.append((i, _cabi.PW_MAXIMUM, reg[v], reg[c], reg[c]))
        # (the kernel reads both sources before it writes the destination)
        for s in [s for s in held if last[s] <= i]:
            held.remove(s)
            free.append(reg[s])
        if c is None:
            reg[v] = fresh()
        held.append(v)
        out.append((i, op, reg[v], ca, cb))
    return out, [code(s) for _, s in reads], n_regs


class Recorder(TorchDispatchMode):
    """Records the element-wise tape of one Milstein step; `finish` turns it into a tsde_pointwise program.  With
    `transcendental`, the tape may hold the transcendental ops too (`_TRANSCENDENTAL`, `_BACKWARD`, `_pow`): the
    library compiles this recorder's programs (`compiled`)."""

    compiled = True

    def __init__(self, y, t0, transcendental=False):
        super().__init__()
        self.transcendental = transcendental
        self.rows, self.d = y.shape
        self.dtype, self.device = y.dtype, y.device
        self.ok, self.reason = True, None
        self.instrs = []       # (opcode, value id, source, source, condition of a SEL or None)
        self._bools = set()    # the values that are comparison results (0 or 1 in the state dtype)
        self.n_fg = None
        self.operands = []     # (kind, ptr, imm)
        self._operand_ix = {}
        self._keep = []        # every tensor seen: no address is reused while recording
        self._by_obj = {}      # id(tensor) -> source
        self._by_addr = {}     # (data_ptr, shape, stride) -> source
        self._storage = {}     # id(tensor) / address key -> storage of every bound tensor
        self._shapes = {(), _strip((self.d,)), _strip((self.rows, self.d))}
        self._at(y, t0)

    def _at(self, y=None, t=None):
        """From here on `y` is what the user's function calls the state and `t` the time."""
        if y is not None:
            self._bind(y, Y)
        if t is not None and t.dtype == self.dtype and t.device == self.device:  # (else an op on t rejects the tape)
            self._bind(t, T0)

    def _run(self, fn, y=None, t=None):
        """fn() at (t, y) with its ATen ops recorded."""
        self._at(y, t)
        with self:
            return fn()

    # -- the three segments ---------------------------------------------------------------------------------------
    def segment(self, fn, y=None, go=None):
        """fn() with its ATen ops recorded.  `y` is the tensor the segment calls the state (a detached alias of the
        state for g), `go` the vjp seed (vjp segment)."""
        if go is not None:
            self._bind(go, GO)
            self.n_fg = len(self.instrs)
        return self._run(fn, y)

    def reject(self, reason):
        if self.ok:
            self.ok, self.reason = False, reason

    def _isolate(self):
        """Make every value bound so far (a state, a time, an intermediate) foreign to what is recorded next; a view of
        an operand is an operand again."""
        for table in (self._by_obj, self._by_addr):
            for key, src in list(table.items()):
                if src[0] == 'k':
                    del table[key]
                    self._storage.pop(key, None)
                else:
                    table[key] = FOREIGN

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        if self.ok:
            try:
                self._record(func, args, kwargs, out)
            except Exception as e:  # (anything the recorder cannot account for keeps the ordinary step)
                self.reject(f"{type(e).__name__}: {e}")
        return out

    # -- values ------------------------------------------------------------------------------------------------
    @staticmethod
    def _addr(t):
        return (t.data_ptr(), tuple(t.shape), tuple(t.stride()), t.dtype)

    def _bind(self, t, src):
        self._keep.append(t)
        self._by_obj[id(t)] = src
        self._by_addr[self._addr(t)] = src
        self._storage[id(t)] = self._storage[self._addr(t)] = t.untyped_storage().data_ptr()

    def _written(self, t):
        """`t` is about to be written in place: every other tensor bound to its storage (a view, `detach()`,
        `.data`) would keep the old value, so reading one of them rejects the tape."""
        st, own = t.untyped_storage().data_ptr(), (id(t), self._addr(t))
        for key, s in self._storage.items():
            if s == st and key not in own:
                (self._by_addr if isinstance(key, tuple) else self._by_obj)[key] = STALE

    def _operand(self, kind, ptr, imm):
        key = (kind, ptr, float(imm).hex())
        if key not in self._operand_ix:
            self._operand_ix[key] = len(self.operands)
            self.operands.append(key[:2] + (imm,))
        return ('k', self._operand_ix[key])

    def _immediate(self, x):
        if isinstance(x, bool) or not isinstance(x, numbers.Real):
            raise Reject(f"unsupported scalar {x!r}")
        return float(np.asarray(x).astype(self._np))

    @property
    def _np(self):
        return np.float32 if self.dtype == torch.float32 else np.float64

    def _source(self, x):
        """What an op input is: a value of the tape, y, go, or an operand."""
        if not torch.is_tensor(x):
            return self._operand(_cabi.PW_IMM, None, self._immediate(x))
        src = self._by_obj.get(id(x))
        if src is None:
            src = self._by_addr.get(self._addr(x))
        if src == T0:
            return self._operand(_cabi.PW_T0, None, 0.0)
        if src == STALE:
            raise Reject("a tensor aliasing one written in place is read")
        if src is not None:
            return src
        if x.device.type == 'cpu' and x.dim() == 0 and x.device != self.device:
            return self._operand(_cabi.PW_IMM, None, self._immediate(x.item()))
        if x.device != self.device or x.dtype != self.dtype or x.requires_grad and x.grad_fn is not None:
            raise Reject(f"operand {tuple(x.shape)} {x.dtype} on {x.device}")
        if not x.is_contiguous():
            raise Reject(f"non-contiguous operand {tuple(x.shape)}")
        if x.untyped_storage().data_ptr() in self._storage.values():
            raise Reject("an operand shares storage with a value of the tape")
        if x.numel() == 1:
            kind = _cabi.PW_SCALAR
        elif _strip(x.shape) == (self.d,):
            kind = _cabi.PW_CHANNEL
        elif tuple(x.shape) == (self.rows, self.d):
            kind = _cabi.PW_ROW
        else:
            raise Reject(f"operand of shape {tuple(x.shape)}")
        self._keep.append(x)
        return self._operand(kind, x.data_ptr(), 0.0)

    def _number(self, x):
        """The source of an op input that is a number: a comparison result is a condition only."""
        src = self._source(x)
        if src in self._bools:
            raise Reject("a comparison result is used as a number")
        return src

    def _condition(self, x):
        """The source of a condition (of where, masked_fill, a logical op): a comparison result of the tape."""
        src = self._source(x)
        if src not in self._bools:
            raise Reject("a condition is not a comparison result of the tape")
        return src

    def _result(self, out, boolean=False):
        want = torch.bool if boolean else self.dtype
        if not torch.is_tensor(out) or out.dtype != want or out.device != self.device:
            raise Reject("result is not a tensor of the state dtype")
        if _strip(out.shape) not in self._shapes:
            raise Reject(f"result of shape {tuple(out.shape)}")

    def _value(self, op, a, b=None, cond=None, boolean=False):
        v = ('v', len(self.instrs))
        self.instrs.append((op, v, a, b, cond))
        if boolean:
            self._bools.add(v)
        return v

    def _emit(self, op, a, b, out, cond=None, boolean=False):
        self._result(out, boolean)
        self._bind(out, self._value(op, a, b, cond, boolean))

    def _one(self):
        return self._operand(_cabi.PW_IMM, None, 1.0)

    def _bound(self, x):
        """A scalar clamp bound as an immediate: clamp restates as maximum / minimum only when it is not NaN."""
        imm = self._immediate(x)
        if imm != imm:
            raise Reject("a NaN clamp bound")
        return self._operand(_cabi.PW_IMM, None, imm)

    def _record_select(self, func, args, kwargs, out):
        """The comparison and selection ops; False for any other op."""
        if func in _COMPARE:
            op, swap = _COMPARE[func]
            a, b = self._number(args[0]), self._number(args[1])
            if func in _NEGATED:
                self._emit(_cabi.PW_SUB, self._one(), self._value(op, a, b, boolean=True), out, boolean=True)
            else:
                self._emit(op, *((b, a) if swap else (a, b)), out, boolean=True)
        elif func in _LOGICAL:
            c = self._condition(args[0])
            if _LOGICAL[func] == _cabi.PW_SUB:
                self._emit(_cabi.PW_SUB, self._one(), c, out, boolean=True)
            else:
                self._emit(_LOGICAL[func], c, self._condition(args[1]), out, boolean=True)
        elif func is aten.where.self:
            self._emit(_cabi.PW_SEL, self._number(args[1]), self._number(args[2]), out, self._condition(args[0]))
        elif func is aten.masked_fill.Scalar:
            self._emit(_cabi.PW_SEL, self._operand(_cabi.PW_IMM, None, self._immediate(args[2])),
                       self._number(args[0]), out, self._condition(args[1]))
        elif func in (aten.maximum.default, aten.minimum.default, aten.clamp_min.Tensor, aten.clamp_max.Tensor):
            op = _cabi.PW_MAXIMUM if func in (aten.maximum.default, aten.clamp_min.Tensor) else _cabi.PW_MINIMUM
            self._emit(op, self._number(args[0]), self._number(args[1]), out)
        elif func in (aten.clamp.default, aten.clamp.Tensor, aten.clamp_min.default, aten.clamp_max.default,
                      aten.relu.default):
            # clamp is maximum with the lower bound, then minimum with the upper one: exactly ATen's clamp kernels
            # when a scalar bound is not NaN (relu is clamp_min(y, 0)); a tensor bound propagates NaN as maximum does
            x, scalar = self._number(args[0]), func in (aten.clamp.default, aten.clamp_min.default,
                                                          aten.clamp_max.default)
            lo = kwargs.get('min', args[1] if len(args) > 1 else None)
            hi = kwargs.get('max', args[2] if len(args) > 2 else None)
            if func is aten.clamp_max.default:
                lo, hi = None, args[1]
            elif func is aten.relu.default:
                lo = 0
            bounds = [(op, b) for op, b in ((_cabi.PW_MAXIMUM, lo), (_cabi.PW_MINIMUM, hi)) if b is not None]
            if not bounds:
                raise Reject(f"{func} without bounds")
            for k, (op, b) in enumerate(bounds):
                src = self._bound(b) if scalar else self._number(b)
                if k + 1 < len(bounds):
                    x = self._value(op, x, src)
                else:
                    self._emit(op, x, src, out)
        elif func is aten.threshold_backward.default:  # x <= threshold ? 0 : grad
            c = self._value(_cabi.PW_LE, self._number(args[1]), self._bound(args[2]), boolean=True)
            self._emit(_cabi.PW_SEL, self._operand(_cabi.PW_IMM, None, 0.0), self._number(args[0]), out, c)
        elif func in (aten.sign.default, aten.sgn.default):  # (0 < x) - (x < 0)
            x, zero = self._number(args[0]), self._operand(_cabi.PW_IMM, None, 0.0)
            pos = self._value(_cabi.PW_LT, zero, x, boolean=True)
            self._emit(_cabi.PW_SUB, pos, self._value(_cabi.PW_LT, x, zero, boolean=True), out)
        elif func is aten.reciprocal.default:  # 1 / x
            self._emit(_cabi.PW_DIV, self._one(), self._number(args[0]), out)
        elif func is aten.scalar_tensor.default:  # an immediate, rounded to its own dtype, then to the state's
            dtype = kwargs.get('dtype') or torch.get_default_dtype()
            if dtype not in (torch.float32, torch.float64) or isinstance(args[0], bool) or \
                    not isinstance(args[0], numbers.Real):
                raise Reject(f"scalar_tensor({args[0]!r}) of {dtype}")
            own = (np.float32 if dtype == torch.float32 else np.float64)(args[0])
            self._bind(out, self._operand(_cabi.PW_IMM, None, self._immediate(float(own))))
        else:
            return False
        return True

    def _record(self, func, args, kwargs, out):
        if func in _ALIAS:
            self._result(out, self._source(args[0]) in self._bools)
            if _strip(args[0].shape) != _strip(out.shape) and not (
                    func is aten.expand.default and _strip(out.shape) == (self.rows, self.d)):
                raise Reject(f"{func} moves elements")
            self._bind(out, self._source(args[0]))
            return
        if func in _IN_PLACE:
            if self._source(args[0])[0] != 'v':
                raise Reject(f"{func} writes a tensor the tape did not produce")
            self._written(args[0])
            func = _IN_PLACE[func]
        elif func._schema.is_mutable or 'out' in kwargs:
            raise Reject(f"{func} mutates its arguments")
        if self._record_select(func, args, kwargs, out):
            return
        if func in _UNARY:
            self._emit(_UNARY[func], self._number(args[0]), None, out)
            return
        if func in _TRANSCENDENTAL:
            self._allow(func)
            self._emit(_TRANSCENDENTAL[func], self._number(args[0]), None, out)
            return
        if func in _BACKWARD:
            self._allow(func)
            self._emit(_BACKWARD[func], self._number(args[0]), self._number(args[1]), out)
            return
        if func is aten.pow.Tensor_Scalar:
            self._pow(args[0], args[1], out)
            return
        if func not in _BINARY:
            raise Reject(f"{func} is not an element-wise op the kernel restates")
        op, swap = _BINARY[func]
        alpha = kwargs.get('alpha', args[2] if len(args) > 2 else 1)
        if op in (_cabi.PW_MUL, _cabi.PW_DIV) and (len(args) > 2 or kwargs):
            raise Reject(f"{func} with {kwargs}")
        if op in (_cabi.PW_ADD, _cabi.PW_SUB):
            if isinstance(alpha, bool) or alpha not in (1, -1):
                raise Reject(f"{func} with alpha={alpha!r}")
            if alpha == -1:
                op = _cabi.PW_SUB if op == _cabi.PW_ADD else _cabi.PW_ADD
        a, b = (args[1], args[0]) if swap else (args[0], args[1])
        if op == _cabi.PW_DIV and (not torch.is_tensor(b) or b.device.type == 'cpu' and b.dim() == 0
                                   and b.device != self.device):
            # ATen: a CPU-scalar divisor becomes a multiplication by its reciprocal, rounded in the state dtype
            inv = self._np(1) / self._np(self._immediate(b.item() if torch.is_tensor(b) else b))
            self._emit(_cabi.PW_MUL, self._number(a), self._operand(_cabi.PW_IMM, None, float(inv)), out)
            return
        self._emit(op, self._number(a), self._number(b), out)

    def _allow(self, what):
        """A transcendental op is about to be recorded: reject the tape unless this solve fuses them and can."""
        if not self.transcendental:
            raise Reject(f"{what} is not an element-wise op the kernel restates")
        if not self.compiled:
            raise Reject(f"{what} is fused by the compiled kernels only (Milstein, and Euler, midpoint and SRK on "
                         f"general or additive noise), not by this method's")
        reason = nvrtc_mismatch() or (None if _cabi.nvjitlink() else "no nvJitLink to link the transcendental ops")
        if reason:
            raise Reject(reason)

    def _pow(self, x, p, out):
        """pow(x, p) with a scalar exponent, as ATen's CUDA kernel dispatches it: p == 2 is x * x (always); with
        `transcendental`, 0.5 is sqrt, -0.5 rsqrt, -1 reciprocal, and p rounded to the state dtype e then gives
        x * x * x for 3, 1 / (x * x) for -2 (computed in double by ATen for float: one division rounded twice, first
        to double, which gives the float quotient exactly) and pow(x, e) otherwise.  Exponents 0 and 1 are a fill and a
        copy in ATen and reject the tape."""
        if isinstance(p, bool) or not isinstance(p, numbers.Real) or p != 2 and (not self.transcendental or p in (0, 1)):
            raise Reject(f"pow with exponent {p!r}")
        a = self._number(x)
        if p == 0.5:
            self._emit(_cabi.PW_SQRT, a, None, out)
        elif p == -1:
            self._emit(_cabi.PW_DIV, self._one(), a, out)
        elif p == -0.5:
            self._allow(f"pow with exponent {p!r}")
            self._emit(_cabi.PW_RSQRT, a, None, out)
        else:
            e = self._immediate(p)
            if e == 2:
                self._emit(_cabi.PW_MUL, a, a, out)
            elif e == 3:
                self._emit(_cabi.PW_MUL, self._value(_cabi.PW_MUL, a, a), a, out)
            elif e == -2:
                self._emit(_cabi.PW_DIV, self._one(), self._value(_cabi.PW_MUL, a, a), out)
            else:
                self._allow(f"pow with exponent {p!r}")
                self._emit(_cabi.PW_POW, a, self._operand(_cabi.PW_IMM, None, e), out)

    # -- the program -----------------------------------------------------------------------------------------------
    def _step_result(self, t, allow_go=False):
        """The source of `t`, a tensor the step takes as f, g or the vjp of g."""
        if not torch.is_tensor(t) or tuple(t.shape) != (self.rows, self.d) or t.dtype != self.dtype:
            raise Reject("a result is not a (rows, d) tensor of the state dtype")
        src = self._source(t)
        if src[0] == 'k' or src in (GO, GO2) and not allow_go:
            raise Reject("a result is not computed from the state")
        return src

    def _program(self, code, n_fg, results, n_regs, max_regs):
        """The tsde_pointwise of allocated instructions `code` (_allocate), of which the first `n_fg` come before the
        boundary, with `results` (f_src, g_src, gdg_src) and the recorder's operand table; and the tensors it reads."""
        if len(code) > _cabi.PW_MAX_INSTR or len(self.operands) > _cabi.PW_MAX_OPERANDS:
            raise Reject("program too long")
        if n_regs > max_regs:
            raise Reject("too many live values")
        prog = _cabi.Pointwise()
        prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands = len(code), n_fg, n_regs, len(self.operands)
        prog.f_src, prog.g_src, prog.gdg_src = results
        for j, (_, op, dst, a, b) in enumerate(code):
            ins = prog.instr[j]
            ins.op, ins.dst, ins.a, ins.b = op, dst, a, b
        for k, (kind, ptr, imm) in enumerate(self.operands):
            prog.operand[k].kind, prog.operand[k].ptr, prog.operand[k].imm = kind, ptr, imm
        return prog, tuple(t for t in self._keep if self._by_obj.get(id(t), 'k')[0] == 'k')

    def finish(self, f, g, gdg):
        """The tsde_pointwise program of the recorded step (and the tensors it reads), or None if it was rejected."""
        if self.ok and self.n_fg is None:
            self.reject("no vjp segment")
        if not self.ok:
            return None
        try:
            # the kernel reads f and g at the boundary, gdg at the end
            reads = [(self.n_fg, self._step_result(f)), (self.n_fg, self._step_result(g)),
                     (len(self.instrs), self._step_result(gdg, allow_go=True))]
            code, results, n_regs = _allocate(self.instrs, reads)
            n_fg = sum(1 for c in code if c[0] < self.n_fg)
            return self._program(code, n_fg, results, n_regs, _cabi.PW_MAX_REGS)
        except Exception as e:
            self.reject(f"{type(e).__name__}: {e}")
            return None


# library -> the sources (tsde_pointwise_source) of the Milstein programs it compiled in this process
_COMPILED = weakref.WeakKeyDictionary()
COMPILES = 0  # how many of them were compiled: SDEs of one structure share the first one's kernels


def compile_milstein(rec, res, adaptive=False):
    """`res`, what `rec.finish` returned, once its program's kernels are compiled and loaded (tsde_pointwise_compile;
    with `adaptive`, the proposal kernel of an adaptive solve, tsde_adaptive_pointwise_compile); None if `res` is, or
    if the library cannot compile the program (the tape is then rejected with the compiler's reason).  Called on the
    recording step, so a graph solve's warm-up and capture, and an adaptive solve's fused proposals, never compile or
    load a module.  A program whose source (its structure: values and addresses are launch parameters) was compiled
    before is not compiled again."""
    global COMPILES
    if res is None:
        return None
    prog = res[0]
    src = _cabi.pointwise_source(prog, rec.dtype)
    if src is None:
        rec.reject("the library refuses the program")
        return None
    done = _COMPILED.setdefault(_cabi.lib(), set())
    if (adaptive, src) not in done:
        err = (_cabi.compile_adaptive_pointwise if adaptive else _cabi.compile_pointwise)(prog, rec.dtype)
        if err != 0:
            rec.reject(_cabi.lib().tsde_error_string(err).decode())
            return None
        done.add((adaptive, src))
        COMPILES += 1
    return res


_COUNT = 'zero one two three four five six seven'.split()


class SrkRecorder(Recorder):
    """Records the SDE evaluations of one step whose kernel takes an f program and a g program: by default the seven
    of a diagonal-noise SRK step (methods.SRK._diagonal_or_scalar_step), f at three (t, y), g at four; `pattern`
    names another step's evaluations in order ('fgfg' for Heun and midpoint, 'fgg' for Euler-Heun) and `max_regs`
    its kernel's register bound.  Each evaluation is a segment of its own, with its own state and 0-d time.  `finish`
    accepts the tape when the f segments are one program (same ops, operands and order) and so are the g segments,
    and compiles the first of each into the two-program layout of tsde_step_srk_diag_pointwise and
    tsde_step_predictor_corrector_pointwise.  A Python-side branch between evaluations (or any other difference)
    therefore keeps the ordinary step.  Its kernels interpret the programs, so a transcendental op rejects the tape
    (`compiled`)."""

    compiled = False

    def __init__(self, y, t, pattern='fgfgfgg', max_regs=_cabi.PW_SRK_MAX_REGS, transcendental=False):
        super().__init__(y, t, transcendental)
        self.pattern, self.max_regs = pattern, max_regs
        self.segments = []  # (kind, first instruction, end, result source)

    def evaluation(self, kind, fn, t, y):
        """fn(), the SDE's f (`kind` 'f') or g ('g') at (t, y), with its ATen ops recorded.  Every value bound by an
        earlier evaluation (its state, its time, its intermediates) is foreign to this one; a view of an operand is
        an operand again."""
        self._isolate()
        start = len(self.instrs)
        out = self._run(fn, y, t)
        if self.ok:
            try:
                self.segments.append((kind, start, len(self.instrs), self._step_result(out)))
            except Exception as e:
                self.reject(f"{type(e).__name__}: {e}")
        return out

    def _source(self, x):
        src = super()._source(x)
        if src == FOREIGN:
            raise Reject("a value of another evaluation is read")
        return src

    def _tape(self, start, end, src):
        """Instructions [start, end) and the result, with value ids relative to the segment."""
        def rel(s):
            return ('v', s[1] - start) if s is not None and s[0] == 'v' else s
        return [(op, *map(rel, srcs)) for op, *srcs in self.instrs[start:end]], rel(src)

    def finish(self):
        """The tsde_pointwise program of the recorded step (and the tensors it reads), or None if it was rejected."""
        if not self.ok:
            return None
        try:
            if ''.join(s[0] for s in self.segments) != self.pattern:
                raise Reject(f"not the {_COUNT[len(self.pattern)]} evaluations {self.pattern!r} of the step")
            parts = []
            for kind in 'fg':
                segs = [s for s in self.segments if s[0] == kind]
                tapes = [self._tape(*s[1:]) for s in segs]
                if any(tp != tapes[0] for tp in tapes[1:]):
                    raise Reject(f"the {kind} evaluations differ")
                # each program starts with no register defined; its result is read when it ends
                _, start, end, src = segs[0]
                parts.append(_allocate(self.instrs[start:end], [(end - start, src)]))
            (code_f, (f_src,), regs_f), (code_g, (g_src,), regs_g) = parts
            return self._program(code_f + code_g, len(code_f), (f_src, g_src, 0), max(regs_f, regs_g), self.max_regs)
        except Exception as e:
            self.reject(f"{type(e).__name__}: {e}")
            return None


SRA_PATTERN = 'fggf'  # an additive-noise SRK step's evaluations, in the order methods.SRK._additive_step makes them


def _pad3(shape):
    return (1,) * (3 - len(shape)) + tuple(shape)


class GeneralRecorder(SrkRecorder):
    """Records the f and g evaluations of a general- or additive-noise Euler ('fg') or midpoint ('fgfg') step, or of an
    additive-noise SRK step ('fggf': f0, gA, gB, f1, methods.SRK._additive_step), whose g is (rows, d, m).  A value is
    either of the (rows, d) class of the diagonal tapes or per channel: computed by an op whose result is
    three-dimensional, or not of a (rows, d) shape, or that reads a per-channel value (`_wide`).
    Per-channel ops broadcast as torch does, right-aligned on (rows, d, m), and may read
      * per-channel values;
      * (rows, d)-class values only through `unsqueeze(-1)` (`y[..., None]`), as (rows, d, 1), or when they have one
        element: a lifted tensor (`_lifted`) keeps the element mapping of its value, broadcast along m;
      * device tensors by their layout broadcast to (rows, d, m): one element (SCALAR), a (d, 1) column (CHANNEL),
        an (m,) row (M), a dense (d, m) block (DM); a (rows, d, m) tensor from outside the tape rejects it.
    f must be of the (rows, d) class; g must have the shape (rows, d, m) and may be any of those (an operand's
    `expand` is additive noise).  The kernel derives which instructions are per channel from their sources alone.  The
    program is tagged with its step's layout `layout`, the solver's `_pw_layout` (Euler's and reversible Heun's
    pattern 'fg' is the same); without one, PW_LAYOUT_GENERAL_SRA for SRK's pattern, else PW_LAYOUT_GENERAL.  Its
    kernels are compiled, so with `transcendental` it takes the transcendental ops."""

    compiled = True

    def __init__(self, y, t, pattern, m, transcendental=False, layout=None):
        self.m = m
        if layout is None:
            layout = _cabi.PW_LAYOUT_GENERAL_SRA if pattern == SRA_PATTERN else _cabi.PW_LAYOUT_GENERAL
        self.layout = layout
        self._wide = set()     # the per-channel values
        self._lifted = set()   # id() of (rows, d)-class tensors viewed as (..., 1)
        self._w3 = False       # the op being recorded is per channel
        self._kind = None      # the evaluation being recorded, 'f' or 'g'
        super().__init__(y, t, pattern, _cabi.PW_MAX_REGS, transcendental)

    # -- the op's class ------------------------------------------------------------------------------------------
    def _is_bound(self, x):
        return torch.is_tensor(x) and (id(x) in self._by_obj or self._addr(x) in self._by_addr)

    def _per_channel_input(self, x):
        if not torch.is_tensor(x):
            return False
        src = self._by_obj.get(id(x)) or self._by_addr.get(self._addr(x))
        return src in self._wide or (src is None and x.dim() == 3)

    def _record(self, func, args, kwargs, out):
        tensors = [a for a in list(args) + list(kwargs.values()) if torch.is_tensor(a)]
        self._w3 = torch.is_tensor(out) and (out.dim() == 3 or _strip(out.shape) not in self._shapes or
                                             any(self._per_channel_input(a) for a in tensors))
        if func in _ALIAS and self._w3:
            self._alias3(args[0], out)
            return
        super()._record(func, args, kwargs, out)

    def _alias3(self, x, out):
        """A view in a per-channel context: a view of an unbound tensor is classified where it is read; a view of a
        value keeps the value's element mapping when it only adds broadcast axes."""
        if not self._is_bound(x):
            return
        src = SrkRecorder._source(self, x)  # (the view decides below how the tensor may be read)
        if src[0] == 'k':
            return
        lifted = src not in self._wide
        if lifted:
            if id(x) in self._lifted:
                old = _pad3(x.shape)
            elif tuple(out.shape) == tuple(x.shape) + (1,) and _strip(x.shape) in self._shapes:
                old = _pad3(tuple(x.shape) + (1,))  # unsqueeze(-1): the (rows, d) class as (rows, d, 1)
            elif x.numel() == 1:
                old = (1, 1, 1)
            else:
                raise Reject(f"a (rows, d) value viewed as {tuple(out.shape)}")
        else:
            old = _pad3(x.shape)
        if out.dim() > 3 or any(a not in (1, b) for a, b in zip(old, _pad3(out.shape))):
            raise Reject(f"a view {tuple(x.shape)} -> {tuple(out.shape)} that moves elements")
        self._result(out, src in self._bools)
        self._bind(out, src)
        if lifted:
            self._lifted.add(id(out))

    def _result(self, out, boolean=False):
        if not self._w3:
            return super()._result(out, boolean)
        want = torch.bool if boolean else self.dtype
        if not torch.is_tensor(out) or out.dtype != want or out.device != self.device:
            raise Reject("result is not a tensor of the state dtype")
        if out.dim() > 3 or any(a not in (1, b) for a, b in zip(_pad3(out.shape), (self.rows, self.d, self.m))):
            raise Reject(f"result of shape {tuple(out.shape)}")

    def _value(self, op, a, b=None, cond=None, boolean=False):
        v = super()._value(op, a, b, cond, boolean)
        if self._w3:
            self._wide.add(v)
        return v

    def _source(self, x):
        if not self._w3 or not torch.is_tensor(x):
            return super()._source(x)
        src = self._by_obj.get(id(x)) or self._by_addr.get(self._addr(x))
        if src is None and not (x.device.type == 'cpu' and x.dim() == 0):
            return self._operand3(x)
        src = super()._source(x)
        if src in self._wide or src[0] == 'k' or x.numel() == 1 or id(x) in self._lifted:
            return src
        raise Reject(f"a (rows, d) value of shape {tuple(x.shape)} is read per channel")

    def _operand3(self, x):
        """A device tensor read per channel, by its layout broadcast right-aligned to (rows, d, m)."""
        if x.device != self.device or x.dtype != self.dtype or x.requires_grad and x.grad_fn is not None:
            raise Reject(f"operand {tuple(x.shape)} {x.dtype} on {x.device}")
        if x.dim() > 3:
            raise Reject(f"operand of shape {tuple(x.shape)}")
        if x.untyped_storage().data_ptr() in self._storage.values():
            raise Reject("an operand shares storage with a value of the tape")
        shape, stride = _pad3(x.shape), (0,) * (3 - x.dim()) + tuple(x.stride())
        (a, b, c), (_, sb, sc) = shape, [s if n > 1 else 0 for n, s in zip(shape, stride)]
        if a > 1 and stride[0] != 0 or b not in (1, self.d) or c not in (1, self.m):
            raise Reject(f"operand of shape {tuple(x.shape)} read per channel")
        if b > 1 and c > 1:
            kind, ok = _cabi.PW_DM, sb == c and sc == 1
        elif b > 1:
            kind, ok = _cabi.PW_CHANNEL, sb == 1
        elif c > 1:
            kind, ok = _cabi.PW_M, sc == 1
        else:
            kind, ok = _cabi.PW_SCALAR, True
        if not ok:
            raise Reject(f"operand of shape {tuple(x.shape)} and strides {tuple(x.stride())} is not dense")
        self._keep.append(x)
        return self._operand(kind, x.data_ptr(), 0.0)

    # -- the results -------------------------------------------------------------------------------------------
    def evaluation(self, kind, fn, t, y):
        self._w3, self._kind = False, kind
        return super().evaluation(kind, fn, t, y)

    def _program(self, code, n_fg, results, n_regs, max_regs):
        prog, keep = super()._program(code, n_fg, results, n_regs, max_regs)
        prog.reserved = self.layout
        return prog, keep

    def _step_result(self, t, allow_go=False):
        if self._kind == 'f':
            self._w3 = False
            src = super()._step_result(t)
            if src in self._wide:
                raise Reject("f is computed per channel")
            return src
        if tuple(t.shape) != (self.rows, self.d, self.m) or t.dtype != self.dtype:
            raise Reject("g is not a (rows, d, m) tensor of the state dtype")
        self._w3 = True
        return self._source(t)


def recording(solver):
    """Whether this step of `solver` (its `_pw` is the program, None before the first step, False once rejected)
    is the one to record: the first diagonal-noise step of an `eligible` solve (for reversible Heun, the first whose
    solver state the chunk kernel can read, methods.ReversibleHeun), or the first general- or additive-noise step of
    one that `general` serves."""
    return solver._pw is None and (solver.sde.noise_type == NOISE_TYPES.diagonal or general(solver)) and \
        eligible(solver)


def general(solver):
    """Whether `solver` runs general- or additive-noise steps that the element-wise general kernels serve: a fixed-step
    Euler, midpoint, Euler-Heun, reversible-Heun or (additive-noise) SRK solve (`_pw_general`, whose kernels are those
    of its `_pw_layout`) with 1 <= m <= TSDE_PW_GENERAL_MAX_M Brownian channels."""
    return (getattr(solver, '_pw_general', False) and not solver.adaptive
            and solver.sde.noise_type in (NOISE_TYPES.general, NOISE_TYPES.additive)
            and 1 <= solver.m <= _cabi.PW_GENERAL_MAX_M)


def pc_recorder(solver, y, t, pattern):
    """The recorder of this step of a Heun, midpoint, Euler-Heun, Euler or additive-noise SRK `solver` (evaluations
    `pattern`), or None when it is not the one to record.  Only an SDE whose f and g the step calls as the user's two
    callables is recorded: not one with a user f_and_g (one call yields both), g_prod or f_and_g_prod, and not an
    adjoint SDE."""
    sde = solver.sde
    if (not recording(solver) or sde.f_and_g_prod_mode != 'fused' or sde.g_prod_mode != 'fused'
            or getattr(sde, 'user_f_and_g', True) or getattr(sde, 'is_adjoint_sde', False)):
        return None
    if sde.noise_type != NOISE_TYPES.diagonal:
        return GeneralRecorder(y, t, pattern, solver.m, transcendental(solver), solver._pw_layout)
    return SrkRecorder(y, t, pattern, _cabi.PW_MAX_REGS, transcendental(solver))


def compile_general(solver, rec, res):
    """`res`, what a GeneralRecorder's `finish` returned, once the Euler and midpoint kernels of its program (the sra1,
    Euler-Heun or reversible-Heun kernels of a program with that tag) are compiled and loaded (tsde_pointwise_compile on the solver's GENERAL launch), on the
    recording step as for
    `compile_milstein`; None if `res` is, or if the library refuses or cannot compile the program (the tape is then
    rejected with the reason)."""
    global COMPILES
    if res is None:
        return None
    err = _cabi.compile_general_pointwise(res[0], rec.dtype, solver.d, solver.m)
    if err != 0:
        rec.reject(_cabi.lib().tsde_error_string(err).decode())
        return None
    COMPILES += 1
    return res


def finish(solver, rec):
    """The end of a recording step of `solver` other than Milstein's: what becomes its `_pw`, the program of `rec`'s
    tape (a GeneralRecorder's once `compile_general` has compiled it), or False if the tape was rejected."""
    if isinstance(rec, GeneralRecorder):
        return compile_general(solver, rec, rec.finish()) or False
    return rec.finish() or False


def ready(solver):
    """Whether `solver` has a program and the counter noise its kernel draws from."""
    return bool(solver._pw) and solver._feed.binding is not None


def launch(solver, name, nz, y0, args, out):
    """One step y0 -> out of the library's whole-step function `name` on the solver's program."""
    prog, _ = solver._pw
    out = out if out is not None else torch.empty_like(y0)
    solver._feed._nz.flags = 0  # (an unfused general step may have left TSDE_FLAG_G_BROADCAST; g is not an operand)
    fn = getattr(solver._lib, name)
    _cabi.check(fn(solver._L, nz, ctypes.byref(prog), y0.data_ptr(), *args, out.data_ptr()), name)
    return out


def plan_chunks(first, n_steps, interpolated=(), multi_cell=(), max_steps=_cabi.PW_MAX_STEPS):
    """Steps [first, n_steps) of a fixed-step solve grouped into the launches of its element-wise program (Milstein,
    Euler, reversible Heun), as (k0, k1) ranges of at most `max_steps` consecutive steps.  Inside a chunk a state lives
    in registers only, so a chunk ends where a step's state has to be in memory for someone else:
      * a step in `multi_cell` (it spans several Brownian cells; the chunk kernels draw one cell per step) runs alone;
      * a step in `interpolated` (a non-aligned output falls inside it) runs alone, and the step before it ends a
        chunk: the interpolation reads the states before and after the step.
    Aligned outputs do not end a chunk: the kernel stores those rows as it passes them."""
    solo = set(interpolated) | set(multi_cell)
    out, k0 = [], first
    for k in range(first, n_steps):
        if k + 1 == n_steps or k in solo or k + 1 in solo or k + 1 - k0 == max_steps:
            out.append((k0, k + 1))
            k0 = k + 1
    return out


# Resident CTAs (256 threads) per SM of each chunked kernel, (float32, float64), from its registers (-Xptxas -v,
# sm_90a: 64 K registers per SM): Milstein's compiled kernels are pinned there by their launch bounds (256, 4) and
# (256, 2) (cfg2's program: 54 registers in fp32); Euler at 54 and 88-96; reversible Heun at 72 and 110-120.
# The compiled general-noise Euler and reversible-Heun kernels are bounded at (256, 1): at least one resident CTA,
# whatever m; so is the reversible-Heun adjoint's backward-step kernel, whatever its parameters.
_RESIDENT_CTAS = {'milstein': (4, 2), 'euler': (4, 2), 'reversible_heun': (3, 2), 'euler_general': (1, 1),
                  'reversible_heun_general': (1, 1), 'adjoint_reversible_heun': (1, 1)}


def chunk_length(solver):
    """Steps per launch of the solver's element-wise program (`solver._pw_method`: 'milstein', 'euler' or
    'reversible_heun'): TSDE_PW_MAX_STEPS when the batch fills the GPU with at least one wave of its chunk kernel's
    CTAs (256 quads each, _RESIDENT_CTAS per SM), else 1.  A smaller grid leaves SMs idle; consecutive one-step kernels
    fill them by overlapping one step's tail with the next one's start (programmatic dependent launch), which a chunk,
    whose steps are sequential per thread, cannot.  (On an H100 at B = 4096, D = 64, fp32, Milstein, one session
    alternating the two: 3.3 us per step one step per launch, 4.3 in chunks of 64.)"""
    if solver.device.type != 'cuda':  # (the host-side dry run of the tests; a solve always runs on a CUDA device)
        return _cabi.PW_MAX_STEPS
    ctas = solver.rows * ((solver.d + 3) // 4) / 256
    method = solver._pw_method + ('_general' if solver.sde.noise_type != NOISE_TYPES.diagonal else '')
    wave = torch.cuda.get_device_properties(solver.device).multi_processor_count * (
        _RESIDENT_CTAS[method][0 if solver.dtype == torch.float32 else 1])
    return _cabi.PW_MAX_STEPS if ctas >= wave else 1


def solve_chunk(solver, ctxs, y0, outs, method, ito=0, state=None):
    """Consecutive single-cell steps `ctxs` of `method` ('milstein', 'euler' or 'reversible_heun') from y0 as one
    launch of its tsde_solve_*_pointwise on the solver's program.  Step j's y1 is stored to outs[j] (None: kept in
    registers only; the last must be given).  `ito` is Milstein's; `state` is reversible Heun's ((z0, f0, g0) the chunk
    starts from, (z1, f1, g1) where it leaves its state)."""
    prog, _ = solver._pw
    feed = solver._feed
    nz = feed.get(ctxs[0])
    feed._nz.flags = 0  # (an unfused general step may have left TSDE_FLAG_G_BROADCAST; g is not an operand)
    steps = (_cabi.PwStep * len(ctxs))()
    for s, c, out in zip(steps, ctxs, outs):
        s.cell_id, s.h, _ = feed.binding.cell(c.k)
        # the time the program runs at: reversible Heun evaluates f and g at t1 (reversible_heun.py:70)
        t = c.t1 if method == 'reversible_heun' else c.t0
        s.dt, s.t0, s.y1 = c.dt, t.data_ptr(), None if out is None else out.data_ptr()
    lib, args = solver._lib, (solver._L, nz, ctypes.byref(prog), y0.data_ptr())
    name = f'tsde_solve_{method}_pointwise'
    if method == 'milstein':
        code = lib.tsde_solve_milstein_pointwise(*args, steps, len(ctxs), ito)
    elif method == 'euler':  # (diagonal, or general / additive noise on the solver's GENERAL launch)
        code = lib.tsde_solve_euler_pointwise(*args, steps, len(ctxs))
    else:
        state_in, state_out = state
        code = lib.tsde_solve_reversible_heun_pointwise(*args, *(x.data_ptr() for x in state_in), steps, len(ctxs),
                                                         *(x.data_ptr() for x in state_out))
    _cabi.check(code, name)
    return outs[-1]


def halves_exactly(dtype, ctxs):
    """Whether every step of `ctxs` has the half step reversible Heun's chunk kernel forms, T(0.5) * T(dt) in the state
    dtype T, equal to the unfused step's half_dt (0.5 * dt rounded once to T).  Halving is exact, so the two differ
    only where the result is subnormal in T; a solve with such a step keeps the ordinary step."""
    t = np.float32 if dtype == torch.float32 else np.float64
    return all(t(0.5) * t(c.dt) == t(c.scalars['half_dt']) for c in ctxs)


def state_fits(solver, tensors):
    """Whether reversible Heun's solver state (f, g, z) is what a chunk kernel reads: contiguous tensors of the state
    dtype on the state's device, of shape (rows, d), except a general- or additive-noise g, of shape (rows, d, m) and
    16-byte aligned (the unfused pair reads such a g as quads: the summation order the kernel was compiled for)."""
    rows_d = (solver.rows, solver.d)
    general = solver.sde.noise_type != NOISE_TYPES.diagonal
    shapes = (rows_d, rows_d + (solver.m,) if general else rows_d, rows_d)
    return len(tensors) == 3 and all(
        torch.is_tensor(x) and tuple(x.shape) == shape and x.dtype == solver.dtype and x.device == solver.device
        and x.is_contiguous() for x, shape in zip(tensors, shapes)) and (not general or tensors[1].data_ptr() % 16 == 0)


def eligible(solver):
    """Whether a Milstein, SRK, Heun, midpoint, Euler-Heun, Euler or reversible-Heun solve may run its diagonal-noise
    steps as element-wise programs: no gradients (the forward solve of `sdeint_adjoint` has none), `overlap` not
    False, no logqp, no autocast, and
      * a fixed-step solve: a Brownian motion bound to the solver grid (counter noise);
      * an adaptive one: a Brownian motion whose answers have the state's (rows, d) shape, and not the adjoint SDE of
        `sdeint_adjoint`'s backward solve (its proposals are `proposing`)."""
    from .base_sde import SDELogqp
    sde = solver.sde
    obj = sde
    while hasattr(obj, '_base_sde'):
        obj = obj._base_sde
        if isinstance(obj, SDELogqp):
            return False
    if solver.adaptive:
        noise = (not getattr(sde, 'is_adjoint_sde', False)
                 and tuple(solver.bm.shape) == (solver.rows, solver.d))
    else:
        feed = getattr(solver, '_feed', None)
        noise = feed is not None and feed.binding is not None
    overlap = solver.options.get('overlap')
    return (not solver._autograd and noise and (overlap is None or bool(overlap))
            and not torch.is_autocast_enabled('cuda'))


def proposing(solver):
    """Whether this proposal of an adaptive `solver` runs as one launch of its element-wise program (`propose`): the
    solve is `eligible` and its first proposal recorded the program."""
    return solver.adaptive and bool(solver._pw) and eligible(solver)


def propose(solver, method, curr_t, next_t, midpoint_t, y0):
    """One proposal of an adaptive solve, (y_full, y_next): the Brownian motion is queried for the full step, the first
    half step and the second half step, in that order and exactly as the three unfused steps query it (with U for
    SRK), and one launch of tsde_adaptive_proposal_pointwise (`method`, a TSDE_PROPOSAL_*) runs the three sub-steps
    on those increments.  Each sub-step's times and scalars are the ones the unfused step computes
    (BaseSDESolver._context)."""
    from .base_solver import NoiseFeed
    prog, _ = solver._pw
    solver._refresh_stream()
    feed = solver._feed = NoiseFeed(solver, solver.bm, None)
    subs, keep = (_cabi.PwSubstep * 3)(), []
    for sub, (ta, tb) in zip(subs, ((curr_t, next_t), (curr_t, midpoint_t), (midpoint_t, next_t))):
        c = solver._context(ta, tb)
        w, u = feed.tensors(c, method == _cabi.PROPOSAL_SRK)
        keep.append((c, w, u))
        sub.w, sub.u, sub.dt = w.data_ptr(), None if u is None else u.data_ptr(), c.dt
        if method == _cabi.PROPOSAL_SRK:
            times, scalars = c.aux_t, (c.scalars['rdt'], c.scalars['sqrt_dt'], c.scalars['three_dt'])
        elif method == _cabi.PROPOSAL_MIDPOINT:
            times, scalars = (c.t0, c.aux_t[0]), (c.scalars['half_dt'],)
        elif method in (_cabi.PROPOSAL_HEUN, _cabi.PROPOSAL_EULER_HEUN):
            times, scalars = (c.t0, c.t1), ()
        else:
            times, scalars = (c.t0,), ()
        for i, t in enumerate(times):
            sub.t[i] = t.data_ptr()
        for i, x in enumerate(scalars):
            sub.s[i] = x
    y_full, y_next = torch.empty_like(y0), torch.empty_like(y0)
    _cabi.check(solver._lib.tsde_adaptive_proposal_pointwise(solver._L, ctypes.byref(prog), method, y0.data_ptr(),
                                                             subs, y_full.data_ptr(), y_next.data_ptr()),
                "tsde_adaptive_proposal_pointwise")
    return y_full, y_next


# ---- the reversible-Heun adjoint's backward sweep --------------------------------------------------------------------
# How a parameter's gradient leaves the vjp: reduced over the rows (a (d,) parameter), over everything (one element),
# or not at all (a (rows, d) parameter)
REDUCE_ROWS, REDUCE_ALL, REDUCE_NONE = 'rows', 'all', 'none'
_SUMS = (aten.sum.dim_IntList, aten.sum.default)


class AdjointRecorder(Recorder):
    """Records the first backward step of `sdeint_adjoint`'s reversible pair (adjoint._BackwardEngine) in three
    segments: f and g at (t0, z0) (`forward`); torch.autograd.grad of [f, g] with respect to [z0] + params with seeds
    GO (f's) and GO2 (g's) (`vjp`); f and g at (t1, z1) (`again`), which must be the first segment's program.  The
    program is the first two: its results are f, g, vjp_z and one contribution per parameter, the (rows, d) value whose
    batch reduction autograd returns as that parameter's gradient.  On a parameter's path the tape accepts only
      * sum.dim_IntList / sum.default of a (rows, d) value over the rows or over everything (autograd's sum_to of a
        (d,) or one-element parameter's gradient), views of that reduction, and `add` of two such reductions (a
        parameter used twice), which becomes the element-wise sum of their contributions;
      * a (rows, d) value itself, the gradient of a (rows, d) parameter;
      * None, a parameter the step does not reach: no contribution.
    Any other op on a reduced value (a parameter transformed before it is broadcast), more than
    TSDE_PW_ADJ_MAX_PARAMS parameters, or anything the Milstein recorder rejects, rejects the tape."""

    def __init__(self, z0, t0, n_params, transcendental=False):
        super().__init__(z0, t0, transcendental)
        self.reduced = []      # ('r', j) -> (kind, [contribution sources])
        self.fg = self.fg3 = self.results = None
        self._in_vjp = False   # a sum is a parameter's batch reduction only in the vjp segment
        if n_params > _cabi.PW_ADJ_MAX_PARAMS:
            self.reject(f"{n_params} parameters: at most {_cabi.PW_ADJ_MAX_PARAMS} are fused")

    # -- the three segments ---------------------------------------------------------------------------------------
    def _results(self, tensors):
        try:
            return [self._step_result(t) for t in tensors]
        except Exception as e:
            self.reject(f"{type(e).__name__}: {e}")
            return None

    def forward(self, fn):
        """fn() = (f, g) at the state and time the recorder was made with."""
        out = self._run(fn)
        if self.ok:
            self.fg = self._results(out)
        self.n_fg = len(self.instrs)
        return out

    def vjp(self, fn, go, go2, params):
        """fn() = autograd's gradients of [z0] + `params`, with seeds go and go2."""
        for t, src in ((go, GO), (go2, GO2)):
            self._bind(t, src)
        self._in_vjp = True
        try:
            grads = self._run(fn)
        finally:
            self._in_vjp = False
        if self.ok:
            try:
                self.results = self._contributions(grads, params)
            except Exception as e:
                self.reject(f"{type(e).__name__}: {e}")
        self.n_vjp = len(self.instrs)
        return grads

    def again(self, fn, t1, z1):
        """fn() = (f, g) at (t1, z1), with every value of the first two segments foreign."""
        self._isolate()
        self.start3 = len(self.instrs)
        self._at(z1, t1)
        out = self._run(fn)
        if self.ok:
            self.fg3 = self._results(out)
        return out

    def _contributions(self, grads, params):
        """(vjp_z's source, [(reduction, contribution source) or None per parameter]); a parameter with several
        contributions gets their sum, appended to the tape."""
        vz = grads[0]
        vz = self._operand(_cabi.PW_IMM, None, 0.0) if vz is None else self._step_result(vz, allow_go=True)
        out = []
        for p, gp in zip(params, grads[1:]):
            if gp is None:
                out.append(None)
                continue
            src = self._lookup(gp)
            if src is not None and src[0] == 'r':
                kind, srcs = self.reduced[src[1]]
            elif tuple(gp.shape) == (self.rows, self.d) and tuple(p.shape) == (self.rows, self.d):
                kind, srcs = REDUCE_NONE, [self._step_result(gp, allow_go=True)]
            else:
                raise Reject(f"the gradient of a {tuple(p.shape)} parameter is not a batch reduction of the tape")
            acc = srcs[0]
            for s in srcs[1:]:
                acc = self._value(_cabi.PW_ADD, acc, s)
            out.append((kind, acc))
        return vz, out

    # -- the ops on a parameter's path ----------------------------------------------------------------------------
    def _lookup(self, x):
        if not torch.is_tensor(x):
            return None
        src = self._by_obj.get(id(x))
        return src if src is not None else self._by_addr.get(self._addr(x))

    def _source(self, x):
        src = super()._source(x)
        if src == FOREIGN:
            raise Reject("a value of another evaluation is read")
        if src[0] == 'r':
            raise Reject("a parameter's gradient is transformed after its batch reduction")
        return src

    def _record(self, func, args, kwargs, out):
        if func in _SUMS and self._in_vjp:  # (a sum in f or g is rejected as any other reduction is)
            self._reduce(args, kwargs, out)
            return
        tensors = [a for a in list(args) + list(kwargs.values()) if torch.is_tensor(a)]
        reds = [self._lookup(a) for a in tensors]
        reds = [r for r in reds if r is not None and r[0] == 'r']
        if not reds:
            return super()._record(func, args, kwargs, out)
        if func in _ALIAS:
            self._bind(out, reds[0])
            return
        alpha = kwargs.get('alpha', args[2] if len(args) > 2 else 1)
        if func in (aten.add.Tensor, aten.add_.Tensor) and len(reds) == 2 == len(tensors) and alpha == 1 \
                and not isinstance(alpha, bool):
            (ka, a), (kb, b) = (self.reduced[r[1]] for r in reds)
            if ka != kb:
                raise Reject("two reductions of one parameter's gradient differ")
            self.reduced.append((ka, a + b))
            v = ('r', len(self.reduced) - 1)
            if func is aten.add_.Tensor:
                self._written(args[0])
                self._bind(args[0], v)
            self._bind(out, v)
            return
        raise Reject("a parameter's gradient is transformed after its batch reduction")

    def _reduce(self, args, kwargs, out):
        x = args[0]
        if kwargs.get('dtype') is not None:
            raise Reject("a reduction with a dtype")
        src = self._number(x)
        if tuple(x.shape) != (self.rows, self.d):
            raise Reject(f"a reduction of a {tuple(x.shape)} value")
        if out.numel() == 1:
            kind = REDUCE_ALL
        elif len(args) > 1 and sorted(int(k) % 2 for k in args[1]) == [0] and out.numel() == self.d:
            kind = REDUCE_ROWS
        else:
            raise Reject(f"a reduction to {tuple(out.shape)}")
        self._keep.append(out)
        self.reduced.append((kind, [src]))
        self._bind(out, ('r', len(self.reduced) - 1))

    # -- the program -----------------------------------------------------------------------------------------------
    def finish(self):
        """(the tsde_pw_adjoint program, the tensors it reads, each parameter's reduction or None), or None if the tape
        was rejected."""
        if self.ok and (self.fg is None or self.results is None or self.fg3 is None):
            self.reject("not the three segments of a backward step")
        if not self.ok:
            return None
        try:
            def rel(src, start):
                return ('v', src[1] - start) if src is not None and src[0] == 'v' else src

            def tape(start, end):
                return [(op, *(rel(x, start) for x in srcs)) for op, *srcs in self.instrs[start:end]]
            if tape(0, self.n_fg) != tape(self.start3, len(self.instrs)) or \
                    [rel(x, 0) for x in self.fg] != [rel(x, self.start3) for x in self.fg3]:
                raise Reject("the evaluations at (t0, z0) and (t1, z1) differ")
            vz, contribs = self.results
            live = [c for c in contribs if c is not None]
            reads = [(self.n_fg, self.fg[0]), (self.n_fg, self.fg[1]), (self.n_vjp, vz)] + \
                [(self.n_vjp, src) for _, src in live]
            code, results, n_regs = _allocate(self.instrs[:self.n_vjp], reads)
            n_fg = sum(1 for c in code if c[0] < self.n_fg)
            prog, keep = self._program(code, n_fg, results[:3], n_regs, _cabi.PW_MAX_REGS)
            ad = _cabi.PwAdjoint()
            ad.prog = prog
            ad.prog.reserved = _cabi.PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN
            ad.n_params = len(live)
            for k, src in enumerate(results[3:]):
                ad.param_src[k] = src
            return ad, keep, [None if c is None else c[0] for c in contribs]
        except Exception as e:
            self.reject(f"{type(e).__name__}: {e}")
            return None


def compile_adjoint(rec, res):
    """`res`, what `rec.finish` returned, once its backward-step kernels are compiled and loaded
    (tsde_pointwise_compile of the tagged program), on the recording step as for `compile_milstein`; None if `res` is,
    or if the library refuses or cannot compile the program (the tape is then rejected with the reason)."""
    global COMPILES
    if res is None:
        return None
    ad = res[0]
    src = _cabi.pointwise_source(ad.prog, rec.dtype)
    if src is None:
        rec.reject("the library refuses the program")
        return None
    done = _COMPILED.setdefault(_cabi.lib(), set())
    if ('adjoint', src) not in done:
        err = _cabi.compile_pointwise(ad.prog, rec.dtype)
        if err != 0:
            rec.reject(_cabi.lib().tsde_error_string(err).decode())
            return None
        done.add(('adjoint', src))
        COMPILES += 1
    return res


def adjoint_refusal(engine, options, differentiable=False, adaptive=False):
    """Why the backward sweep of `engine` (adjoint._BackwardEngine) with adjoint_options `options` keeps its unfused
    steps although options={'fused_backward': True} asks for chunks, or None if it may record its first step."""
    from .base_sde import SDELogqp
    sde = engine.sde
    obj = sde
    while hasattr(obj, '_base_sde'):
        obj = obj._base_sde
        if isinstance(obj, SDELogqp):
            return "logqp"
    if differentiable:
        return "create_graph (double backward)"
    if adaptive:
        return "adjoint_adaptive"
    if sde.noise_type != NOISE_TYPES.diagonal:
        return f"{sde.noise_type} noise (diagonal only)"
    if getattr(engine, 'binding', None) is None:
        return "the Brownian motion is not a BrownianInterval bound to the solver grid"
    if options.get('overlap') is not None and not options['overlap']:
        return "overlap=False"
    if torch.is_autocast_enabled('cuda'):
        return "autocast"
    if sde.f_and_g_prod_mode != 'fused' or sde.g_prod_mode != 'fused' or getattr(sde, 'user_f_and_g', True):
        return "f and g are not two separate callables (a user f_and_g, g_prod or f_and_g_prod)"
    if not halves_exactly(engine.dtype, engine.ctxs):
        return "a half step is subnormal in the state dtype"
    return None


def solve_adjoint_chunk(engine, ks, t0, state_in, state_out, ys, grad_ys, partials):
    """Backward steps `ks` (consecutive, single-cell unless alone) of `engine` as one launch of
    tsde_solve_reversible_heun_pointwise on its adjoint program, from the forward values at (t0, z); step k ends on
    output row engine._out[k] (-1: none).  `state_in` / `state_out` are (y, z, f, g, adj_y, adj_f, adj_g, adj_z)."""
    ad = engine._pw[0]
    feed = engine._feed
    nz = feed.get(engine.ctxs[ks[0]])
    feed._nz.flags = 0
    steps = (_cabi.PwStep * len(ks))()
    row = ys.stride(0) * ys.element_size()  # (ys is contiguous: output k starts k rows of bytes past ys)
    for s, k in zip(steps, ks):
        c = engine.ctxs[k]
        s.cell_id, s.h, _ = feed.binding.cell(c.k)
        s.dt, s.t0 = c.dt, c.aux_t[1].data_ptr()
        s.y1 = None if engine._out[k] < 0 else ys.data_ptr() + engine._out[k] * row
    ad.t0, ad.ys, ad.grad_ys, ad.n_out = t0.data_ptr(), ys.data_ptr(), grad_ys.data_ptr(), ys.shape[0]
    ad.y1 = state_out[0].data_ptr()
    for i in range(4):
        ad.adj_in[i], ad.adj_out[i] = state_in[4 + i].data_ptr(), state_out[4 + i].data_ptr()
    for i, x in enumerate(partials):
        ad.partial[i] = x.data_ptr()
    y, z, f, g = (x.data_ptr() for x in state_in[:4])
    _cabi.check(engine._lib.tsde_solve_reversible_heun_pointwise(
        engine._L, nz, ctypes.byref(ad.prog), y, z, f, g, steps, len(ks),
        *(x.data_ptr() for x in state_out[1:4])), 'tsde_solve_reversible_heun_pointwise')
