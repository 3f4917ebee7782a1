"""The element-wise tapes on random SDEs, on the CPU (tests/pointwise_fuzz.py draws them).

For every recorder (Milstein's; SRK's, Heun / midpoint's, Euler-Heun's and Euler's two-program tapes; the general-noise
Euler, midpoint and sra1 tapes), in float32 and float64, a corpus of seeded cases of every size class:

  * acceptance is predicted: a tape drawn from the layout's vocabulary is accepted, or rejected as too long or too wide
    only when it was drawn at the limits;
  * the recorded program, run by a numpy restatement of the kernels' interpreter, gives for f and g at every recorded
    evaluation the bits of the case's numpy evaluator, which restates each torch op as ATen's CUDA kernel computes it
    (cases with a transcendental op are skipped here: numpy has no exact libdevice); Milstein's vjp, which has no
    independent restatement, matches torch's autograd to 4 eps;
  * the allocation is sound: run symbolically, with value terms in the registers, every register is written before it
    is read, every SEL finds its condition in its destination, n_regs is within the kernel's bound, and f, g (and the
    vjp) are the recorded tape's values, so no register was overwritten before its value's last read;
  * every accepted Milstein and general-noise program compiles with NVRTC as the library compiles it;
  * and the checks bite: with `_allocate` freeing a source one instruction early, with a division by a Python number
    recorded as a true division, or with SEL's condition copy dropped, some Milstein case, some case of the
    interpreted layouts and some general-noise case fail.

A failing case prints its `repr` (a `Case(...)` call) and its torch source; `pointwise_fuzz.case(seed, layout)`
rebuilds it."""
import concurrent.futures
import inspect
import textwrap

import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import pointwise_fuzz as fz
from . import test_host_pointwise_compile as compile_
from . import test_host_pointwise_transcendental as transcendental

SEEDS = 200  # per layout, half of them in each dtype
COMPILED = 12  # the seeds per compiled layout whose programs are compiled, besides those at the limits
TOO_BIG = ('program too long', 'too many live values')
UNARY = {_cabi.PW_NEG, _cabi.PW_SQRT, _cabi.PW_ABS, _cabi.PW_EXP, _cabi.PW_LOG, _cabi.PW_SIN, _cabi.PW_COS,
         _cabi.PW_TANH, _cabi.PW_LOG1P, _cabi.PW_EXPM1, _cabi.PW_RSQRT, _cabi.PW_SIGMOID}


def _dtype(seed):
    return torch.float32 if seed % 2 == 0 else torch.float64


def _npt(dtype):
    return np.float32 if dtype == torch.float32 else np.float64


class Recorded:
    """One case recorded as its step records it: the recorder, what `finish` returned, the evaluations
    (kind, t, y, result) and Milstein's vjp seed and result."""

    def __init__(self, case, dtype, rows=fz.ROWS, d=fz.D, m=fz.M):
        self.case, self.dtype = case, dtype
        recorder, pattern, _ = fz.LAYOUTS[case.layout]
        self.p = fz.torch_params(case, rows, d, m, dtype, 'cpu', cpu_scalars=False)
        gen = torch.Generator().manual_seed(case.seed)
        ys = [(torch.rand(rows, d, generator=gen, dtype=torch.float64) * 3 - 1.5).to(dtype) for _ in pattern]
        if case.size == 'edge':
            ys[0] = fz.edge_state(rows, d, dtype, case.seed)
        ts = [torch.tensor(0.375 + 0.0625 * i, dtype=dtype) for i in range(len(pattern))]
        fns = {'f': (case.f, case.f_out), 'g': (case.g, case.g_out)}
        self.evals, self.go, self.gdg = [], None, None
        if recorder == 'milstein':
            y0, t0 = ys[0], ts[0]
            rec = pointwise.Recorder(y0, t0, case.transcendental)
            fv = rec.segment(lambda: fz.run_torch(*fns['f'], t0, y0, self.p))
            with torch.enable_grad():
                y = y0.detach().requires_grad_(True)
                gv = rec.segment(lambda: fz.run_torch(*fns['g'], t0, y, self.p), y=y)
                self.go = (torch.rand(rows, d, generator=gen, dtype=torch.float64) - 0.5).to(dtype)
                if gv.requires_grad:
                    self.gdg, = rec.segment(lambda: torch.autograd.grad(gv, y, grad_outputs=self.go.view_as(gv),
                                                                         allow_unused=True), go=self.go)
            self.res = rec.finish(fv, gv, self.gdg)
            self.evals = [('f', t0, y0, fv), ('g', t0, y0, gv)]
            self.srcs = None
            if self.res is not None:
                self.srcs = [rec._source(fv), rec._source(gv), rec._source(self.gdg)]
        else:
            if recorder == 'general':
                rec = pointwise.GeneralRecorder(ys[0], ts[0], pattern, m, case.transcendental)
            else:
                rec = pointwise.SrkRecorder(ys[0], ts[0], pattern,
                                            _cabi.PW_SRK_MAX_REGS if pattern == 'fgfgfgg' else _cabi.PW_MAX_REGS,
                                            case.transcendental)
            for kind, t, y in zip(pattern, ts, ys):
                out = rec.evaluation(kind, lambda: fz.run_torch(*fns[kind], t, y, self.p), t, y)
                self.evals.append((kind, t, y, out))
            self.res = rec.finish()
        self.rec = rec

    def __str__(self):
        return f'{self.case!r}\n{self.case.source()}\nin {self.dtype}: {self.rec.reason}'


_CORPUS = {}


def corpus(layout):
    """The recorded cases of `layout`, recorded once per session."""
    if layout not in _CORPUS:
        _CORPUS[layout] = [Recorded(fz.case(s, layout), _dtype(s)) for s in range(SEEDS)]
    return _CORPUS[layout]


# -- the numpy interpreter of the kernels ------------------------------------------------------------------------------
def _operand(o, npt, rows, d, m, general):
    if o.kind == _cabi.PW_IMM:
        return npt(o.imm)
    shape = {_cabi.PW_SCALAR: (1,), _cabi.PW_CHANNEL: (d, 1) if general else (d,),
             _cabi.PW_ROW: (rows, d, 1) if general else (rows, d), _cabi.PW_DM: (d, m), _cabi.PW_M: (m,)}[o.kind]
    n = int(np.prod(shape))
    raw = (np.ctypeslib.ctypes.c_byte * (n * np.dtype(npt).itemsize)).from_address(o.ptr)
    return np.ctypeslib.as_array(raw).view(npt).reshape(shape).copy()


def interpret(prog, lo, hi, y, t, go, npt, general=False, m=1, regs=None):
    """Instructions [lo, hi) of a program in numpy, one rounding per instruction in the state dtype.  General-noise
    programs run on (rows, d, 1)-shaped states, every operand broadcast as the kernel reads it.  Returns `fetch`."""
    rows, d = y.shape
    yy = y[..., None] if general else y
    regs = regs if regs is not None else [None] * prog.n_regs

    def fetch(s):
        if s == _cabi.PW_SRC_Y:
            return yy
        if s == _cabi.PW_SRC_GO:
            assert go is not None
            return go
        if s < _cabi.PW_OPERAND0:
            assert regs[s] is not None
            return regs[s]
        o = prog.operand[s - _cabi.PW_OPERAND0]
        return np.asarray(t, dtype=npt) if o.kind == _cabi.PW_T0 else _operand(o, npt, rows, d, m, general)

    with np.errstate(all='ignore'):
        for i in range(lo, hi):
            ins = prog.instr[i]
            a = fetch(ins.a)
            b = None if ins.op in UNARY else fetch(ins.b)
            r = {_cabi.PW_MUL: lambda: a * b, _cabi.PW_ADD: lambda: a + b, _cabi.PW_SUB: lambda: a - b,
                 _cabi.PW_DIV: lambda: a / b, _cabi.PW_NEG: lambda: -a, _cabi.PW_SQRT: lambda: np.sqrt(a),
                 _cabi.PW_LT: lambda: (a < b).astype(npt), _cabi.PW_LE: lambda: (a <= b).astype(npt),
                 _cabi.PW_EQ: lambda: (a == b).astype(npt), _cabi.PW_MAXIMUM: lambda: fz.np_maximum(a, b),
                 _cabi.PW_MINIMUM: lambda: fz.np_minimum(a, b), _cabi.PW_ABS: lambda: np.abs(a),
                 _cabi.PW_SEL: lambda: np.where(regs[ins.dst] != 0, a, b)}[ins.op]()
            regs[ins.dst] = np.asarray(r, dtype=npt)
    return fetch


def _bits(x, shape, npt):
    return np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=npt), shape)).view(
        np.uint32 if npt == np.float32 else np.uint64)


# -- the checks ------------------------------------------------------------------------------------------------------
def check_accepted(r):
    if r.res is None:
        assert r.case.size == 'limits' and any(why in (r.rec.reason or '') for why in TOO_BIG), str(r)


def check_restated(r):
    """f and g of every evaluation: the program's bits are the numpy evaluator's."""
    if r.res is None or not r.case.exact:
        return
    prog, _ = r.res
    npt, case, general = _npt(r.dtype), r.case, r.case.general
    p = fz.numpy_params(r.p, npt)
    m = fz.M if general else 1
    for kind, t, y, out in r.evals:
        yn, tn = y.numpy(), t.numpy()
        want = fz.run_numpy(case.f if kind == 'f' else case.g, case.f_out if kind == 'f' else case.g_out, tn, yn, p,
                            npt)
        shape = tuple(out.shape)
        if fz.LAYOUTS[case.layout][0] == 'milstein':
            fetch = interpret(prog, 0, prog.n_fg, yn, tn, None, npt)
            got = fetch(prog.f_src if kind == 'f' else prog.g_src)
        else:
            lo, hi, src = (0, prog.n_fg, prog.f_src) if kind == 'f' else (prog.n_fg, prog.n_instr, prog.g_src)
            got = interpret(prog, lo, hi, yn, tn, None, npt, general, m)(src)
            if general and kind == 'f':
                got = got[..., 0] if np.ndim(got) == 3 else got
        assert np.array_equal(_bits(got, shape, npt), _bits(want, shape, npt)), f'{kind} differs\n{r}'
        # (and the numpy evaluator is torch's CPU result but for the rounding of ops ATen's CPU kernels vectorise
        # otherwise: a wrong restatement of an op's semantics shows here)
        w = np.broadcast_to(want, shape).astype(np.float64)
        o = out.detach().numpy().astype(np.float64)
        fin = np.isfinite(w) & np.isfinite(o)
        assert np.array_equal(np.isnan(w), np.isnan(o)), f'{kind}: NaN where torch has none\n{r}'
        np.testing.assert_allclose(o[fin], w[fin], rtol=1e-3, atol=1e-3, err_msg=str(r))
    if r.gdg is not None:
        regs = [None] * prog.n_regs
        yn, tn = r.evals[0][2].numpy(), r.evals[0][1].numpy()
        interpret(prog, 0, prog.n_fg, yn, tn, None, npt, regs=regs)
        got = interpret(prog, prog.n_fg, prog.n_instr, yn, tn, r.go.numpy(), npt, regs=regs)(prog.gdg_src)
        want = r.gdg.detach().numpy()
        got = np.broadcast_to(got, want.shape)
        # (torch's CPU kernels round a division by a Python number and sqrt otherwise than the CUDA ones)
        np.testing.assert_allclose(got, want, rtol=4 * np.finfo(npt).eps, atol=4 * np.finfo(npt).eps,
                                   err_msg=f'vjp\n{r}')


class _Terms:
    """Hash-consed value terms: equal ids are equal values."""

    def __init__(self):
        self.ids = {}

    def __call__(self, *key):
        if key[0] == _cabi.PW_MAXIMUM and key[1] == key[2]:  # maximum(c, c) is c: SEL's condition copy
            return key[1]
        return self.ids.setdefault(key, len(self.ids))


def _tape_terms(rec, terms):
    """The term of every value of the recorder's tape."""
    out = {}

    def term(s):
        if s is None:
            return None
        if s[0] == 'v':
            return out[s]
        return terms('leaf', s)
    for op, v, a, b, c in rec.instrs:
        out[v] = terms('sel', term(a), term(b), term(c)) if c is not None else \
            terms(op, term(a), None if op in UNARY else term(b))
    return out, term


def _program_terms(prog, lo, hi, terms, regs, bools):
    """Run instructions [lo, hi) on terms; returns `fetch`.  Checks write-before-read, the register bound and that
    every SEL's destination holds a condition."""
    def fetch(s):
        if s == _cabi.PW_SRC_Y:
            return terms('leaf', pointwise.Y)
        if s == _cabi.PW_SRC_GO:
            return terms('leaf', pointwise.GO)
        if s >= _cabi.PW_OPERAND0:
            return terms('leaf', ('k', s - _cabi.PW_OPERAND0))
        assert s < prog.n_regs and regs[s] is not None, f'register {s} read before it is written'
        return regs[s]
    for i in range(lo, hi):
        ins = prog.instr[i]
        assert ins.dst < prog.n_regs
        a = fetch(ins.a)
        if ins.op == _cabi.PW_SEL:
            cond = regs[ins.dst]
            assert cond is not None and cond in bools, f'SEL {i} does not find its condition in its destination'
            regs[ins.dst] = terms('sel', a, fetch(ins.b), cond)
        else:
            regs[ins.dst] = terms(ins.op, a, None if ins.op in UNARY else fetch(ins.b))
    return fetch


def check_allocation(r):
    if r.res is None:
        return
    prog, _ = r.res
    rec, terms = r.rec, _Terms()
    bound = _cabi.PW_SRK_MAX_REGS if fz.LAYOUTS[r.case.layout][1] == 'fgfgfgg' else _cabi.PW_MAX_REGS
    assert 0 <= prog.n_regs <= bound and prog.n_instr <= _cabi.PW_MAX_INSTR, str(r)
    values, term = _tape_terms(rec, terms)
    bools = {values[v] for v in rec._bools}
    if fz.LAYOUTS[r.case.layout][0] == 'milstein':
        regs = [None] * prog.n_regs
        fetch = _program_terms(prog, 0, prog.n_fg, terms, regs, bools)
        got = [fetch(prog.f_src), fetch(prog.g_src)]
        fetch = _program_terms(prog, prog.n_fg, prog.n_instr, terms, regs, bools)
        got.append(fetch(prog.gdg_src))
        assert got == [term(s) for s in r.srcs], f'a register was overwritten before its last read\n{r}'
        return
    for kind in 'fg':
        seg = next(s for s in rec.segments if s[0] == kind)
        lo, hi, src = (0, prog.n_fg, prog.f_src) if kind == 'f' else (prog.n_fg, prog.n_instr, prog.g_src)
        got = _program_terms(prog, lo, hi, terms, [None] * prog.n_regs, bools)(src)
        assert got == term(seg[3]), f'{kind}: a register was overwritten before its last read\n{r}'


def check(r):
    check_accepted(r)
    check_restated(r)
    check_allocation(r)


LAYOUTS = list(fz.LAYOUTS)


@pytest.mark.parametrize('layout', LAYOUTS)
def test_fuzzed_tapes_are_accepted_restated_and_soundly_allocated(layout):
    cases = corpus(layout)
    for r in cases:
        check(r)
    accepted = [r for r in cases if r.res is not None]
    sizes = {s: sum(1 for r in accepted if r.case.size == s) for s in fz.SIZES}
    print(f'{layout}: {len(accepted)} of {len(cases)} accepted {sizes}; '
          f'{sum(1 for r in accepted if r.case.exact)} restated exactly')
    # every size class is represented among the accepted, and the limits class reaches the kernels' bounds
    assert all(sizes[s] > 0 for s in fz.SIZES), sizes
    bound = _cabi.PW_SRK_MAX_REGS if fz.LAYOUTS[layout][1] == 'fgfgfgg' else _cabi.PW_MAX_REGS
    assert max(r.res[0].n_regs for r in accepted) >= bound - 2


def _compile(r):
    prog, _ = r.res
    if r.case.general:
        src = _cabi.general_pointwise_source(prog, r.dtype, fz.D, fz.M)
    else:
        src = _cabi.pointwise_source(prog, r.dtype)
    assert src is not None, str(r)
    if r.case.exact:
        compile_.compile_source(src)
    else:  # (the transcendental helpers are linked in: relocatable device code, as the library compiles them)
        transcendental._cubin(src, transcendental.LIBRARY + ['-fmad=false'])
    return src


@pytest.mark.parametrize('layout', [k for k, v in fz.LAYOUTS.items() if v[2]])
def test_accepted_compiled_programs_compile(layout):
    """The accepted programs of the first COMPILED seeds and those at the limits among the first 8 * COMPILED
    (NVRTC takes a fraction of a second per program)."""
    compile_._nvrtc()
    seen, todo = set(), []
    for r in corpus(layout):
        if r.res is None or r.case.seed >= COMPILED and (r.case.size != 'limits' or r.case.seed >= 8 * COMPILED):
            continue
        prog = r.res[0]
        src = (_cabi.general_pointwise_source(prog, r.dtype, fz.D, fz.M) if r.case.general else
               _cabi.pointwise_source(prog, r.dtype))
        assert src is not None, str(r)
        if src not in seen:
            seen.add(src)
            todo.append(r)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        list(ex.map(_compile, todo))
    assert todo


# -- the checks bite ------------------------------------------------------------------------------------------------
def _mutated(fn, old, new):
    """`fn` with one line of its source replaced, compiled in its module's namespace."""
    src = textwrap.dedent(inspect.getsource(fn))
    assert src.count(old) == 1, old
    ns = {}
    exec(compile(src.replace(old, new), inspect.getsourcefile(fn), 'exec'), vars(pointwise), ns)
    return ns[fn.__name__]


MUTATIONS = {
    'free_early': (lambda: ('_allocate', _mutated(pointwise._allocate, 'for s in [s for s in held if last[s] <= i]:',
                                                  'for s in [s for s in held if last[s] <= i + 1]:'))),
    'true_division': (lambda: ('Recorder._record', _mutated(
        pointwise.Recorder._record, "if op == _cabi.PW_DIV and (not torch.is_tensor(b)",
        "if False and (not torch.is_tensor(b)"))),
    'no_condition_copy': (lambda: ('_allocate', _mutated(
        pointwise._allocate, 'out.append((i, _cabi.PW_MAXIMUM, reg[v], reg[c], reg[c]))', 'pass'))),
}


@pytest.mark.parametrize('mutation', sorted(MUTATIONS))
def test_the_corpus_catches_a_mutated_compiler(mutation, monkeypatch):
    where, fn = MUTATIONS[mutation]()
    if where == '_allocate':
        monkeypatch.setattr(pointwise, '_allocate', fn)
    else:
        monkeypatch.setattr(pointwise.Recorder, '_record', fn)
    caught = {}
    for layout in LAYOUTS:
        for s in range(0, SEEDS, 4):
            r = Recorded(fz.case(s, layout), _dtype(s))
            try:
                check(r)
            except AssertionError:
                caught[layout] = caught.get(layout, 0) + 1
    print(mutation, caught)
    # in the compiled program (Milstein's) and in the interpreted and the general-noise ones
    assert caught.get('milstein') and caught.keys() & {'srk', 'pc', 'euler_heun', 'euler'} and \
        caught.keys() & {'general_euler', 'general_midpoint', 'sra'}, caught
