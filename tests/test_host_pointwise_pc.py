"""The element-wise tapes of a Heun, midpoint or Euler-Heun step on the CPU (torchsde_b200/_core/pointwise.py,
SrkRecorder with the patterns 'fgfg' and 'fgg'): which SDEs the recorder accepts, that the f and g programs it
compiles compute what every recorded evaluation computed (numpy restatement of the kernel's interpreter,
tests/test_host_pointwise_srk.py), what tsde_step_predictor_corrector_pointwise refuses before any CUDA call, and a
dry run of the solvers' launch sequence.  The GPU suite compares the kernel with the unfused step
(tests/test_gpu_pointwise_pc.py)."""
import ctypes

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import problems
from .test_host_dry_run import dry  # noqa: F401  (fixture)
from .test_host_pointwise import ACCEPTED, REJECTED, ROWS, D, _params
from .test_host_pointwise_srk import SRK_ACCEPTED, _interpret, _nth_call_differs
from .test_host_pointwise_validation import BOTH, DEVICE, GO, _Step, _all, _set, _srk

# method -> (evaluation pattern, state index of each evaluation, time index of each evaluation)
PATTERNS = {
    'heun': ('fgfg', [0, 0, 1, 1], [0, 0, 1, 1]),          # (t0, y0) twice, then (t1, y')
    'midpoint': ('fgfg', [0, 0, 1, 1], [0, 0, 2, 2]),      # (t0, y0) twice, then (t0 + dt/2, y')
    'euler_heun': ('fgg', [0, 0, 1], [0, 0, 1]),           # (t0, y0) twice, then g at (t1, y')
}


def _record(f, g, dtype, method, pattern=None):
    """The evaluations of one step of `method` under the recorder, each at its own state and time; `pattern`
    records another sequence of evaluations."""
    want, states_ix, times_ix = PATTERNS[method]
    kinds = pattern or want
    p = _params(dtype)
    gen = torch.Generator().manual_seed(2)
    states = [torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.25 for _ in range(2)]
    table = torch.tensor([0.375, 0.4375, 0.40625], dtype=dtype)
    rec = pointwise.SrkRecorder(states[0], table[0], want, _cabi.PW_MAX_REGS)
    outs, at = [], []
    for k, kind in enumerate(kinds):
        k = min(k, len(want) - 1)  # (a longer wrong pattern repeats the last evaluation's point)
        fn, t, y = (f if kind == 'f' else g), table[times_ix[k]], states[states_ix[k]]
        outs.append(rec.evaluation(kind, lambda: fn(t, y, p), t, y))
        at.append((t, y))
    return rec, rec.finish(), at, outs


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', SRK_ACCEPTED)
@pytest.mark.parametrize('method', sorted(PATTERNS))
def test_accepted_tapes_restate_every_evaluation(method, name, dtype):
    rec, res, at, outs = _record(*ACCEPTED[name], dtype, method)
    assert res is not None, rec.reason
    prog, _ = res
    assert 0 < prog.n_instr <= _cabi.PW_MAX_INSTR and prog.n_regs <= _cabi.PW_MAX_REGS
    kinds = PATTERNS[method][0]
    assert ''.join(s[0] for s in rec.segments) == kinds
    for k, (kind, (t, y), want) in enumerate(zip(kinds, at, outs)):
        got = _interpret(prog, kind, t, y, dtype)
        w = np.ascontiguousarray(want.detach().numpy())
        assert got.dtype == w.dtype
        if name in ('div', 'sqrt_rsub') and kind == 'g':
            # (a Python-number divisor and torch's CPU sqrt: see tests/test_host_pointwise_srk.py)
            np.testing.assert_allclose(got, w, rtol=4 * np.finfo(w.dtype).eps)
        else:
            assert np.array_equal(got.view(np.uint8), w.view(np.uint8)), (k, kind)


@pytest.mark.parametrize('method', sorted(PATTERNS))
def test_each_evaluation_reads_its_own_time(method):
    rec, (prog, _), at, outs = _record(lambda t, y, p: t * y, lambda t, y, p: (t * t + 1) * y, torch.float64, method)
    assert len({a[0].item() for a in at}) == 2
    for kind, (t, y), want in zip(PATTERNS[method][0], at, outs):
        assert np.array_equal(_interpret(prog, kind, t, y, torch.float64), want.numpy())


@pytest.mark.parametrize('name', sorted(REJECTED))
@pytest.mark.parametrize('method', ['heun', 'euler_heun'])
def test_rejected_tapes(method, name):
    rec, res, _, _ = _record(*REJECTED[name], torch.float32, method)
    assert res is None and rec.reason


@pytest.mark.parametrize('method,which,n', [('heun', 'f', 2), ('heun', 'g', 2), ('midpoint', 'f', 2),
                                            ('euler_heun', 'g', 2)])
def test_evaluations_that_differ_reject(method, which, n):
    rec, res, _, _ = _record(*_nth_call_differs(which, n), torch.float32, method)
    assert res is None and 'differ' in rec.reason


@pytest.mark.parametrize('method,pattern', [('heun', 'fgg'), ('heun', 'fgfgg'), ('euler_heun', 'fgfg'),
                                            ('euler_heun', 'gfg')])
def test_the_wrong_pattern_rejects(method, pattern):
    rec, res, _, _ = _record(*ACCEPTED['gbm_strat'], torch.float32, method, pattern)
    assert res is None and 'evaluations' in rec.reason


def _wide(t, y, p):
    """Twenty values live at once: 20 registers."""
    xs = [y * float(k + 1) for k in range(20)]
    out = xs[0]
    for x in xs[1:]:
        out = out + x
    return out


def test_the_register_bound_is_the_recorders():
    """The predictor-corrector kernels keep no stash: their programs may use every register SRK leaves to its own."""
    rec, res, _, _ = _record(_wide, lambda t, y, p: p['b'] * y, torch.float32, 'heun')
    assert res is not None, rec.reason
    assert _cabi.PW_SRK_MAX_REGS < res[0].n_regs <= _cabi.PW_MAX_REGS
    p = _params(torch.float32)
    y, t = torch.rand(ROWS, D) + 0.25, torch.tensor(0.5)
    srk = pointwise.SrkRecorder(y, t)
    for kind in 'fgfgfgg':
        srk.evaluation(kind, (lambda: _wide(t, y, p)) if kind == 'f' else (lambda: p['b'] * y), t, y)
    assert srk.finish() is None and 'live values' in srk.reason


# ---- what the C entry point refuses --------------------------------------------------------------------------------
PC = dict(BOTH, **{
    'n_regs 25': _set('n_regs', _cabi.PW_MAX_REGS + 1),
    'g reads a register only f wrote': _set('instr.1.dst', 1),
    'go in the f program': _set('instr.0.b', GO),
    'go in the g program': _set('instr.2.b', GO),
    'go as the f result': _set('f_src', GO),
    'go as the g result': _set('g_src', GO),
    'g result in a register only f wrote': _all(_set('instr.1.dst', 1), _set('instr.2.a', 1), _set('g_src', 0)),
})
METHODS = [_cabi.PC_HEUN, _cabi.PC_MIDPOINT, _cabi.PC_EULER_HEUN]


def _pc(step, prog, method=_cabi.PC_HEUN, t0=True, t_p=True):
    return step.lib.tsde_step_predictor_corrector_pointwise(
        ctypes.byref(step.L), ctypes.byref(step.nz), ctypes.byref(prog), step.y0.data_ptr(),
        step.t.data_ptr() if t0 else None, step.t[1:].data_ptr() if t_p else None, method, 0.125, 0.0625,
        step.y1.data_ptr())


def _launches(step):
    return step.lib.tsde_kernel_launches(_cabi.KERNEL_PW_PC)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('name', sorted(PC))
def test_malformed_programs_are_refused_without_a_launch(name, method, dtype):
    step = _Step(dtype, DEVICE)
    prog = _srk(step.mem)
    PC[name](prog)
    before = _launches(step)
    assert _pc(step, prog, method) == _cabi.EINVAL
    assert _launches(step) == before


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('case', ['method -1', 'method 3', 'null t0', 'null t_p', 'memory noise'])
def test_bad_calls_are_refused_without_a_launch(case, dtype):
    step = _Step(dtype, DEVICE)
    prog = _srk(step.mem)
    kw = {'method -1': {'method': -1}, 'method 3': {'method': 3}, 'null t0': {'t0': False},
          'null t_p': {'t_p': False}}.get(case, {})
    if case == 'memory noise':
        step.nz.source, step.nz.w = _cabi.SRC_MEMORY, step.y0.data_ptr()
    before = _launches(step)
    assert _pc(step, prog, **kw) == _cabi.EINVAL
    assert _launches(step) == before


# ---- dry run: the launch sequence of a solve -----------------------------------------------------------------------
class _Log:
    """The dry-run library, with every C-ABI call logged as (name, args)."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in _cabi.SIGNATURES:
            return fn

        def entry(*args):
            self.calls.append((name, args))
            return fn(*args)
        return entry


TS, DT = [0.0, 0.09375, 0.25], 0.0625  # four steps; the middle output is interpolated


@pytest.mark.parametrize('method,code', [('heun', _cabi.PC_HEUN), ('midpoint', _cabi.PC_MIDPOINT),
                                         ('euler_heun', _cabi.PC_EULER_HEUN)])
def test_from_the_second_step_on_a_step_is_one_launch(dry, monkeypatch, method, code):  # noqa: F811
    log = _Log(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    sde = problems.make('gbm', 3, 3, 'stratonovich', dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 3), dtype=torch.float32, device='cpu')
    with torch.no_grad():
        ys = tsde.sdeint(sde, torch.ones(4, 3), TS, bm=bm, method=method, dt=DT)
    assert ys.shape == (3, 4, 3)
    names = [n for n, _ in log.calls]
    name = 'tsde_step_predictor_corrector_pointwise'
    first = names.index(name)
    # the recorded first step ran the unfused kernels; every later step is the one kernel (and the output between
    # two grid points is interpolated)
    assert {'tsde_step_heun', 'tsde_step_euler', 'tsde_midpoint_predict', 'tsde_euler_heun_predict',
            'tsde_step_euler_heun'} & set(names[:first])
    assert names.count(name) == 3 and set(names[first:]) == {name, 'tsde_linear_interp'}
    assert all(args[6] == code for n, args in log.calls if n == name)
