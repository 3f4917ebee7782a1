"""Comparison and selection ops in the element-wise tapes (torchsde_b200/_core/pointwise.py) on the CPU: clamp, relu,
abs, sign, maximum / minimum, where, masked_fill, comparisons, logical ops and reciprocal.  Which tapes the Milstein,
SRK and predictor-corrector recorders accept and reject, that the programs they compile compute what the recorded ops
computed (a numpy restatement of the kernel's interpreter with the new opcodes), and what the library refuses before a
launch.  The states include negative values, so every bound and branch is taken; the GPU suite compares the kernels
with the unfused step on the bits, signed zeros and NaN included (tests/test_gpu_pointwise_select.py)."""
import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from . import test_host_pointwise as milstein
from . import test_host_pointwise_pc as pc
from . import test_host_pointwise_srk as srk
from .test_host_pointwise_validation import DEVICE, GO, _Step, _all, _milstein, _set, _srk

# (f, g) as functions of (t, y, params); the states of the host tests lie in [0.25, 1.25), y - 0.75 has either sign
ACCEPTED = {
    'cir_clamp': (lambda t, y, p: p['a'] * (p['b'] - (y - .75).clamp(min=0)),
                  lambda t, y, p: p['s'] * torch.sqrt((y - .75).clamp(min=0))),
    'cir_relu': (lambda t, y, p: p['a'] * (p['b'] - torch.relu(y - .75)),
                 lambda t, y, p: p['s'] * torch.sqrt(torch.relu(y - .75))),
    'reflection': (lambda t, y, p: p['a'] * (p['b'] - y), lambda t, y, p: p['b'] * torch.sqrt((y - .75).abs())),
    'abs': (lambda t, y, p: (y - .75).abs(), lambda t, y, p: p['b'] * (y - .75).abs()),
    'clamp_both': (lambda t, y, p: (y - .75).clamp(-0.2, 0.3), lambda t, y, p: p['b'] * y.clamp(0.5, 1.0)),
    'clamp_min_max': (lambda t, y, p: torch.clamp_min(y - .75, 0.0) + y, lambda t, y, p: torch.clamp_max(y, 0.9)),
    'clamp_tensor': (lambda t, y, p: torch.clamp(y, min=p['a']),
                     lambda t, y, p: torch.clamp(y, min=p['a'] - .5, max=p['b']) * p['s']),
    'maximum_minimum': (lambda t, y, p: torch.maximum(y, p['a']), lambda t, y, p: torch.minimum(y, p['b']) * p['s']),
    'where': (lambda t, y, p: torch.where(y > .75, p['a'] * y, 2 * y),
              lambda t, y, p: torch.where(y > p['b'] - .25, y, 0.0)),
    'where_masks': (lambda t, y, p: torch.where((y > .5) & (y <= 1.0) | ~(y >= p['a']), y, -y),
                    lambda t, y, p: torch.where(y != p['b'], y * p['s'], y) + torch.where(y < .6, y, p['s'])),
    'reciprocal': (lambda t, y, p: torch.reciprocal(y) * p['a'], lambda t, y, p: torch.reciprocal(y + 1)),
}
SIGN = (lambda t, y, p: p['a'] * y, lambda t, y, p: torch.sign(y - .75) * y)  # its vjp is a zeros_like factory
MASK = torch.arange(milstein.D) % 2 == 0  # a user mask: a bool tensor the tape did not produce


def _mask(t, y, p):
    return torch.where(MASK, y, -y)


REJECTED = {
    'bool_arithmetic': (lambda t, y, p: (y > .75) * y, lambda t, y, p: p['b'] * y),
    'float_of_a_mask': (lambda t, y, p: (y > .75).float() * y, lambda t, y, p: p['b'] * y),
    'user_mask': (_mask, lambda t, y, p: p['b'] * y),
    'comparison_as_f': (lambda t, y, p: y > .75, lambda t, y, p: p['b'] * y),
    'comparison_of_masks': (lambda t, y, p: torch.where((y > .75) == (y < 1.0), y, -y), lambda t, y, p: p['b'] * y),
    'nan_clamp_bound': (lambda t, y, p: y.clamp(min=float('nan')), lambda t, y, p: p['b'] * y),
    'leaky_relu': (lambda t, y, p: torch.nn.functional.leaky_relu(y - .75), lambda t, y, p: p['b'] * y),
}
MILSTEIN_REJECTED = dict(REJECTED, **{
    'comparison_as_g': (lambda t, y, p: p['a'] * y, lambda t, y, p: y > .75),
    'sign': SIGN,
    'pow_half': (lambda t, y, p: p['a'] * y, lambda t, y, p: y ** 0.5),
})


def _ops(prog):
    return {prog.instr[i].op for i in range(prog.n_instr)}


def _run(prog, i0, i1, y, t, go, regs, npt):
    """Instructions [i0, i1) of the kernel's interpreter in numpy, every register and operand a (rows, d) array."""
    rows, d = y.shape

    def fetch(s):
        if s == _cabi.PW_SRC_Y:
            return y
        if s == _cabi.PW_SRC_GO:
            assert go is not None
            return go
        if s < _cabi.PW_OPERAND0:
            assert regs[s] is not None
            return regs[s]
        o = prog.operand[s - _cabi.PW_OPERAND0]
        if o.kind == _cabi.PW_IMM:
            return np.full((rows, d), npt(o.imm))
        if o.kind == _cabi.PW_T0:
            return np.full((rows, d), t)
        n = {_cabi.PW_SCALAR: 1, _cabi.PW_CHANNEL: d, _cabi.PW_ROW: rows * d}[o.kind]
        flat = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_byte * (n * np.dtype(npt).itemsize)).from_address(o.ptr))
        return np.broadcast_to(flat.view(npt).reshape(-1, d) if n == rows * d else flat.view(npt), (rows, d))

    def nan_first(a, b, pick):
        return np.where(np.isnan(a), a, np.where(np.isnan(b), b, pick(a, b)))

    with np.errstate(all='ignore'):
        for i in range(i0, i1):
            ins = prog.instr[i]
            a = fetch(ins.a)
            b = None if ins.op in (_cabi.PW_NEG, _cabi.PW_SQRT, _cabi.PW_ABS) else fetch(ins.b)
            r = {_cabi.PW_MUL: lambda: a * b, _cabi.PW_ADD: lambda: a + b, _cabi.PW_SUB: lambda: a - b,
                 _cabi.PW_DIV: lambda: a / b, _cabi.PW_NEG: lambda: -a, _cabi.PW_SQRT: lambda: np.sqrt(a),
                 _cabi.PW_LT: lambda: (a < b).astype(npt), _cabi.PW_LE: lambda: (a <= b).astype(npt),
                 _cabi.PW_EQ: lambda: (a == b).astype(npt),
                 _cabi.PW_MAXIMUM: lambda: nan_first(a, b, np.maximum),
                 _cabi.PW_MINIMUM: lambda: nan_first(a, b, np.minimum), _cabi.PW_ABS: lambda: np.abs(a),
                 _cabi.PW_SEL: lambda: np.where(regs[ins.dst] != 0, a, b)}[ins.op]()
            regs[ins.dst] = np.asarray(r, dtype=npt)
    return fetch


def _npt(dtype):
    return np.float32 if dtype == torch.float32 else np.float64


def _same(got, want):
    w = np.ascontiguousarray(want.detach().numpy())
    assert got.dtype == w.dtype
    # (torch's CPU kernels vectorise sqrt and division by a Python number differently from the CUDA ones the programs
    # restate; the GPU suite checks the bits)
    np.testing.assert_allclose(got, w, rtol=4 * np.finfo(w.dtype).eps, atol=0)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', sorted(ACCEPTED))
def test_milstein_tapes_restate_f_g_and_the_vjp(name, dtype):
    rec, res, (y0, t0, go), (f, g, gdg) = milstein._record(*ACCEPTED[name], dtype)
    assert res is not None, rec.reason
    prog, _ = res
    assert _ops(prog) - set(range(6)) or name == 'reciprocal'  # (1 / y is a division)
    assert prog.n_regs <= _cabi.PW_MAX_REGS
    npt, regs = _npt(dtype), [None] * prog.n_regs
    fetch = _run(prog, 0, prog.n_fg, y0.numpy(), t0.numpy(), None, regs, npt)
    _same(fetch(prog.f_src).copy(), f)
    _same(fetch(prog.g_src).copy(), g)
    fetch = _run(prog, prog.n_fg, prog.n_instr, y0.numpy(), t0.numpy(), go.numpy(), regs, npt)
    _same(fetch(prog.gdg_src), gdg)


def _two_program(name, dtype, record):
    """Record under a two-program recorder and check every evaluation against its program."""
    f, g = SIGN if name == 'sign' else ACCEPTED[name]
    rec, res, at, outs = record(f, g, dtype)
    assert res is not None, rec.reason
    prog, _ = res
    assert _ops(prog) - set(range(6)) or name == 'reciprocal'
    npt = _npt(dtype)
    for (kind, *_), (t, y), want in zip(rec.segments, at, outs):
        i0, i1, src = (0, prog.n_fg, prog.f_src) if kind == 'f' else (prog.n_fg, prog.n_instr, prog.g_src)
        _same(_run(prog, i0, i1, y.numpy(), t.numpy(), None, [None] * prog.n_regs, npt)(src), want)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', sorted(ACCEPTED) + ['sign'])
def test_srk_tapes_restate_every_evaluation(name, dtype):
    _two_program(name, dtype, srk._record)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', sorted(ACCEPTED) + ['sign'])
@pytest.mark.parametrize('method', ['heun', 'euler_heun'])
def test_predictor_corrector_tapes_restate_every_evaluation(method, name, dtype):
    _two_program(name, dtype, lambda f, g, dt: pc._record(f, g, dt, method))


@pytest.mark.parametrize('name', sorted(MILSTEIN_REJECTED))
def test_milstein_rejects(name):
    rec, res, _, _ = milstein._record(*MILSTEIN_REJECTED[name], torch.float32)
    assert res is None and rec.reason


@pytest.mark.parametrize('name', sorted(REJECTED))
def test_srk_rejects(name):
    rec, res, _, _ = srk._record(*REJECTED[name], torch.float32)
    assert res is None and rec.reason


def test_clamp_is_maximum_then_minimum_with_bounds_rounded_to_the_state_dtype():
    rec, (prog, _), _, _ = srk._record(lambda t, y, p: y.clamp(0.1, 2.0), lambda t, y, p: p['b'] * y, torch.float32)
    assert [prog.instr[i].op for i in range(prog.n_fg)] == [_cabi.PW_MAXIMUM, _cabi.PW_MINIMUM]
    lo, hi = (prog.operand[prog.instr[i].b - _cabi.PW_OPERAND0].imm for i in range(2))
    assert (lo, hi) == (float(np.float32(0.1)), 2.0)


def test_a_condition_that_stays_live_is_copied_into_the_selection():
    """where(c, a, b) reads c from its destination: c's register when this is c's last read, else a copy."""
    def f(t, y, p):
        c = y > .75
        return torch.where(c, y, -y) * torch.where(c, p['a'], y)
    rec, (prog, _), _, _ = srk._record(f, lambda t, y, p: p['b'] * y, torch.float32)
    ops = [prog.instr[i].op for i in range(prog.n_fg)]
    assert ops.count(_cabi.PW_SEL) == 2 and ops.count(_cabi.PW_MAXIMUM) == 1
    copy = ops.index(_cabi.PW_MAXIMUM)
    assert prog.instr[copy].a == prog.instr[copy].b and ops[copy + 1] == _cabi.PW_SEL
    assert prog.instr[copy + 1].dst == prog.instr[copy].dst


SEL, LT, ABS = _cabi.PW_SEL, _cabi.PW_LT, _cabi.PW_ABS
MALFORMED = {
    'opcode 7': _set('instr.0.op', 7),
    'opcode 15': _set('instr.0.op', SEL + 1),
    'SEL reading an unwritten condition': _set('instr.0.op', SEL),
    'LT source past the register file': _all(_set('instr.0.op', LT), _set('instr.0.b', _cabi.PW_MAX_REGS)),
    'ABS source past the register file': _all(_set('instr.0.op', ABS), _set('instr.0.a', _cabi.PW_MAX_REGS)),
    'SEL source past the register file': _all(_set('instr.1.op', SEL), _set('instr.1.dst', 0),
                                              _set('instr.1.b', _cabi.PW_MAX_REGS)),
}
MILSTEIN_MALFORMED = dict(MALFORMED, **{
    'SEL condition past n_regs': _all(_set('instr.2.op', SEL), _set('instr.2.dst', 3), _set('n_regs', 4),
                                      _set('gdg_src', 3)),
    'go in a comparison of the f / g part': _all(_set('instr.1.op', LT), _set('instr.1.a', GO)),
})
SRK_MALFORMED = dict(MALFORMED, **{
    'SEL condition written only by the f program': _set('instr.1.op', SEL),
})


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method,name', [('milstein', n) for n in MILSTEIN_MALFORMED] +
                         [('srk', n) for n in SRK_MALFORMED])
def test_malformed_programs_with_the_new_opcodes_are_refused_without_a_launch(method, name, dtype):
    step = _Step(dtype, DEVICE)
    prog = (_milstein if method == 'milstein' else _srk)(step.mem)
    (MILSTEIN_MALFORMED if method == 'milstein' else SRK_MALFORMED)[name](prog)
    before = step.launches()
    assert getattr(step, method)(prog) == _cabi.EINVAL
    assert step.launches() == before

