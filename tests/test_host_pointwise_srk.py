"""The element-wise tape of an SRK step (torchsde_b200/_core/pointwise.py, SrkRecorder) on the CPU: which SDEs it
accepts, and that the f and g programs it compiles compute what each of the seven recorded evaluations computed.  The
programs are run by a numpy restatement of the kernel's interpreter (tsde_step_srk_diag_pointwise), one rounding per
instruction in the state dtype; the GPU suite compares the kernel with the unfused step
(tests/test_gpu_pointwise_srk.py)."""
import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from .test_host_pointwise import ACCEPTED, REJECTED, ROWS, D, _params, _record as _record_milstein

KINDS = 'fgfgfgg'           # f0, g0, f1, g1, f2, g2, g3 (methods.SRK._diagonal_or_scalar_step)
TIMES = [0, 0, 1, 2, 3, 1, 2]  # index into (t0 + 0*dt, t0 + dt, t0 + dt/4, t0 + dt/2)
STATES = [0, 0, 1, 2, 3, 4, 5]  # y0, y0, H0_1, H1_1, H0_2, H1_2, H1_3


def _record(f, g, dtype):
    """The seven evaluations of one step under the recorder, each at its own state and stage time."""
    p = _params(dtype)
    gen = torch.Generator().manual_seed(1)
    states = [torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.25 for _ in range(6)]
    table = torch.tensor([0.375, 0.5, 0.40625, 0.4375], dtype=dtype)
    times = [table[i] for i in range(4)]
    rec = pointwise.SrkRecorder(states[0], times[0])
    outs, at = [], []
    for kind, ti, yi in zip(KINDS, TIMES, STATES):
        fn, t, y = (f if kind == 'f' else g), times[ti], states[yi]
        outs.append(rec.evaluation(kind, lambda: fn(t, y, p), t, y))
        at.append((t, y))
    return rec, rec.finish(), at, outs


def _interpret(prog, kind, t, y, dtype):
    """numpy restatement of one evaluation in the kernel: the f program [0, n_fg) or the g program [n_fg, n_instr),
    from no defined register, every register and operand as a (rows, d) array."""
    npt = np.float32 if dtype == torch.float32 else np.float64
    y, t = y.numpy(), t.numpy()
    regs = [None] * prog.n_regs

    def fetch(s):
        assert s != _cabi.PW_SRC_GO
        if s == _cabi.PW_SRC_Y:
            return y
        if s < _cabi.PW_OPERAND0:
            assert regs[s] is not None
            return regs[s]
        o = prog.operand[s - _cabi.PW_OPERAND0]
        if o.kind == _cabi.PW_IMM:
            return np.full((ROWS, D), npt(o.imm))
        if o.kind == _cabi.PW_T0:
            return np.full((ROWS, D), t)
        n = {_cabi.PW_SCALAR: 1, _cabi.PW_CHANNEL: D, _cabi.PW_ROW: ROWS * D}[o.kind]
        flat = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_byte * (n * np.dtype(npt).itemsize)).from_address(o.ptr))
        vals = flat.view(npt)
        return np.broadcast_to(vals[0] if n == 1 else vals.reshape(-1, D), (ROWS, D))

    lo, hi = (0, prog.n_fg) if kind == 'f' else (prog.n_fg, prog.n_instr)
    with np.errstate(all='ignore'):
        for i in range(lo, hi):
            ins = prog.instr[i]
            a = fetch(ins.a)
            b = fetch(ins.b) if ins.op not in (_cabi.PW_NEG, _cabi.PW_SQRT) else None
            r = {_cabi.PW_MUL: lambda: a * b, _cabi.PW_ADD: lambda: a + b, _cabi.PW_SUB: lambda: a - b,
                 _cabi.PW_DIV: lambda: a / b, _cabi.PW_NEG: lambda: -a, _cabi.PW_SQRT: lambda: np.sqrt(a)}[ins.op]()
            regs[ins.dst] = np.asarray(r, dtype=npt)
        return fetch(prog.f_src if kind == 'f' else prog.g_src).copy()


SRK_ACCEPTED = sorted(set(ACCEPTED) - {'f_value_in_vjp'})


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', SRK_ACCEPTED)
def test_accepted_tapes_restate_all_seven_evaluations(name, dtype):
    rec, res, at, outs = _record(*ACCEPTED[name], dtype)
    assert res is not None, rec.reason
    prog, _ = res
    assert 0 < prog.n_instr <= _cabi.PW_MAX_INSTR and prog.n_regs <= _cabi.PW_SRK_MAX_REGS
    assert len(rec.segments) == 7
    for k, (kind, (t, y), want) in enumerate(zip(KINDS, at, outs)):
        got = _interpret(prog, kind, t, y, dtype)
        w = np.ascontiguousarray(want.detach().numpy())
        assert got.dtype == w.dtype
        if name in ('div', 'sqrt_rsub') and kind == 'g':
            # a Python-number divisor: ATen's CUDA kernel (restated by the tape) multiplies by the reciprocal, its CPU
            # kernel divides; PyTorch's CPU sqrt is not correctly rounded on AVX-512 hosts (methods._ieee_sqrt).  The
            # GPU suite checks the bits.
            np.testing.assert_allclose(got, w, rtol=4 * np.finfo(w.dtype).eps)
        else:
            assert np.array_equal(got.view(np.uint8), w.view(np.uint8)), (k, kind)


def test_stage_times_are_read_per_evaluation():
    """f and g depend on t differently: each evaluation's T0 operand is its own stage time, not the step's t0."""
    rec, (prog, _), at, outs = _record(lambda t, y, p: t * y, lambda t, y, p: (t * t + 1) * y, torch.float64)
    vals = [a[0].item() for a in at]
    assert len(set(vals)) == 4
    for kind, (t, y), want in zip(KINDS, at, outs):
        assert np.array_equal(_interpret(prog, kind, t, y, torch.float64), want.numpy())


@pytest.mark.parametrize('name', sorted(REJECTED))
def test_rejected_tapes(name):
    rec, res, _, _ = _record(*REJECTED[name], torch.float32)
    assert res is None and rec.reason


def _nth_call_differs(which, n):
    """An SDE whose `which` callable takes another branch on its n-th call (counted in Python)."""
    calls = []

    def f(t, y, p):
        calls.append(0) if which == 'f' else None
        return y * p['a'] if which == 'f' and len(calls) == n else p['a'] * y

    def g(t, y, p):
        calls.append(0) if which == 'g' else None
        return (p['b'] * y) * 1 if which == 'g' and len(calls) == n else p['b'] * y
    return f, g


@pytest.mark.parametrize('which,n', [('f', 2), ('f', 3), ('g', 2), ('g', 4)])
def test_evaluations_that_differ_reject(which, n):
    rec, res, _, _ = _record(*_nth_call_differs(which, n), torch.float32)
    assert res is None and 'differ' in rec.reason


def test_values_of_another_evaluation_reject():
    """g reading f's intermediate, or f reading the state of an earlier evaluation, is not one evaluation's program."""
    rec, res, _, _ = _record(*ACCEPTED['f_value_in_vjp'], torch.float32)
    assert res is None and 'another evaluation' in rec.reason
    first = {}

    def f(t, y, p):
        first.setdefault('y', y)
        return p['a'] * first['y']
    rec, res, _, _ = _record(f, lambda t, y, p: p['b'] * y, torch.float32)
    assert res is None and 'another evaluation' in rec.reason


def test_missing_evaluation_rejects():
    p = _params(torch.float32)
    y, t = torch.rand(ROWS, D), torch.tensor(0.5)
    rec = pointwise.SrkRecorder(y, t)
    for kind in KINDS[:-1]:
        rec.evaluation(kind, lambda: p['a'] * y, t, y)
    assert rec.finish() is None and 'seven' in rec.reason


def test_cfg2_srk_program_is_one_multiplication_each():
    rec, (prog, _), _, _ = _record(*ACCEPTED['gbm_ito'], torch.float32)
    assert (prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands) == (2, 1, 1, 2)
    assert [(prog.instr[i].op, prog.instr[i].dst, prog.instr[i].b) for i in range(2)] == \
        [(_cabi.PW_MUL, 0, _cabi.PW_SRC_Y), (_cabi.PW_MUL, 0, _cabi.PW_SRC_Y)]
    assert (prog.f_src, prog.g_src) == (0, 0)
    assert prog.operand[prog.instr[0].a - _cabi.PW_OPERAND0].ptr != prog.operand[prog.instr[1].a - _cabi.PW_OPERAND0].ptr


def test_cfg2_milstein_program_is_unchanged():
    """The Milstein program of the headline SDE: f = mu*y, g = sigma*y, then autograd's `grad * sigma`, three
    multiplications in two registers."""
    rec, (prog, _), _, _ = _record_milstein(*ACCEPTED['gbm_ito'], torch.float32)
    ins = [(prog.instr[i].op, prog.instr[i].dst, prog.instr[i].a, prog.instr[i].b) for i in range(prog.n_instr)]
    k0, k1 = _cabi.PW_OPERAND0, _cabi.PW_OPERAND0 + 1
    assert (prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands) == (3, 2, 2, 2)
    assert ins == [(_cabi.PW_MUL, 0, k0, _cabi.PW_SRC_Y), (_cabi.PW_MUL, 1, k1, _cabi.PW_SRC_Y),
                   (_cabi.PW_MUL, 1, _cabi.PW_SRC_GO, k1)]
    assert (prog.f_src, prog.g_src, prog.gdg_src) == (0, 1, 1)
