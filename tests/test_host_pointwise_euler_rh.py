"""Euler and reversible-Heun solves whose steps run as element-wise programs, several per kernel
(tsde_solve_euler_pointwise, tsde_solve_reversible_heun_pointwise; pointwise.pc_recorder with pattern 'fg') on the
CPU: which tapes the recorder accepts, the half-step check of reversible Heun, what the two C entry points refuse
before any CUDA call, and a dry run of the launch sequence of a solve.  The GPU suite compares the kernels with the
unfused steps (tests/test_gpu_pointwise_euler_rh.py)."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import problems
from .test_host_dry_run import dry  # noqa: F401  (fixture)
from .test_host_pointwise import ACCEPTED, REJECTED, ROWS, D, _params
from .test_host_pointwise_pc import PC, _Log
from .test_host_pointwise_srk import SRK_ACCEPTED, _interpret
from .test_host_pointwise_validation import DEVICE, _Step, _srk


def _record(f, g, dtype, kinds='fg'):
    """The evaluations `kinds` of one step under the recorder, at one state and time (Euler: (t0, y0); reversible
    Heun: (t1, z1))."""
    p = _params(dtype)
    y = torch.rand(ROWS, D, generator=torch.Generator().manual_seed(4), dtype=dtype) + 0.25
    t = torch.tensor(0.4375, dtype=dtype)
    rec = pointwise.SrkRecorder(y, t, 'fg', _cabi.PW_MAX_REGS)
    outs = [rec.evaluation(kind, lambda fn=(f if kind == 'f' else g): fn(t, y, p), t, y) for kind in kinds]
    return rec, rec.finish(), (t, y), outs


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', SRK_ACCEPTED)
def test_accepted_tapes_restate_both_evaluations(name, dtype):
    rec, res, (t, y), outs = _record(*ACCEPTED[name], dtype)
    assert res is not None, rec.reason
    prog, _ = res
    assert 0 < prog.n_instr <= _cabi.PW_MAX_INSTR and prog.n_regs <= _cabi.PW_MAX_REGS
    for kind, want in zip('fg', outs):
        got = _interpret(prog, kind, t, y, dtype)
        w = np.ascontiguousarray(want.detach().numpy())
        if name in ('div', 'sqrt_rsub') and kind == 'g':
            # (a Python-number divisor and torch's CPU sqrt: see tests/test_host_pointwise_srk.py)
            np.testing.assert_allclose(got, w, rtol=4 * np.finfo(w.dtype).eps)
        else:
            assert np.array_equal(got.view(np.uint8), w.view(np.uint8)), kind


@pytest.mark.parametrize('name', sorted(REJECTED))
def test_rejected_tapes(name):
    rec, res, _, _ = _record(*REJECTED[name], torch.float32)
    assert res is None and rec.reason


@pytest.mark.parametrize('kinds', ['ff', 'gg', 'gf', 'fgf', 'fgg', 'f'])
def test_evaluations_that_differ_from_the_step_reject(kinds):
    rec, res, _, _ = _record(*ACCEPTED['gbm_strat'], torch.float32, kinds)
    assert res is None and 'evaluations' in rec.reason


def test_a_result_that_is_an_operand_rejects():
    """g returning a parameter itself (no op of the state): not a value the program computes."""
    rec, res, _, _ = _record(lambda t, y, p: p['a'] * y, lambda t, y, p: p['r'], torch.float32)
    assert res is None and 'not computed from the state' in rec.reason
    rec, res, _, _ = _record(lambda t, y, p: p['a'] * y, lambda t, y, p: p['b'], torch.float32)
    assert res is None and rec.reason


# ---- reversible Heun's half step -----------------------------------------------------------------------------------
def _ctx(dt, half_dt):
    return SimpleNamespace(dt=dt, scalars={'half_dt': half_dt})


def test_the_half_step_is_exact_on_ordinary_grids():
    for dtype in (torch.float32, torch.float64):
        for dt in (2.0 ** -10, 0.3, 1e-3, 0.1 + 2.0 ** -40, 7.0):
            assert pointwise.halves_exactly(dtype, [_ctx(dt, 0.5 * dt)])


def test_a_subnormal_half_step_that_rounds_differently_keeps_the_ordinary_step():
    # a float64 dt just above float32's least normal number: rounding it to float32 and halving rounds twice, the
    # unfused step's (float32)(0.5 * dt) once, and the two differ in the last subnormal bit
    dt = 2.0 ** -126 * (1 + 2.0 ** -23 + 2.0 ** -30)
    half = np.float32(0.5 * dt)
    assert np.float32(0.5) * np.float32(dt) != half and half < np.finfo(np.float32).tiny
    assert not pointwise.halves_exactly(torch.float32, [_ctx(2.0 ** -10, 2.0 ** -11), _ctx(dt, 0.5 * dt)])
    assert pointwise.halves_exactly(torch.float64, [_ctx(dt, 0.5 * dt)])
    # a subnormal half step that both round alike is accepted
    assert pointwise.halves_exactly(torch.float32, [_ctx(2.0 ** -126, 2.0 ** -127)])


# ---- what the C entry points refuse --------------------------------------------------------------------------------
ENTRIES = ['euler', 'reversible_heun']
EXTRAS = ['z0', 'f0', 'g0', 'z1', 'f1', 'g1']


def _table(step, n, t_null=None, last_null=False):
    steps = (_cabi.PwStep * max(n, 1))()
    for j, s in enumerate(steps):
        s.cell_id, s.h, s.dt = j, 0.125, 0.125
        s.t0 = None if j == t_null else step.t[1:].data_ptr()
        s.y1 = step.y1.data_ptr() if j == len(steps) - 1 and not last_null else None
    return steps


def _solve(entry, step, prog, n=2, steps=None, null=None):
    steps = _table(step, n) if steps is None else steps
    args = (ctypes.byref(step.L), ctypes.byref(step.nz), ctypes.byref(prog), step.y0.data_ptr())
    if entry == 'euler':
        return step.lib.tsde_solve_euler_pointwise(*args, steps, n)
    extra = {k: None if k == null else x.data_ptr() for k, x in zip(EXTRAS, step.extra)}
    return step.lib.tsde_solve_reversible_heun_pointwise(*args, extra['z0'], extra['f0'], extra['g0'], steps, n,
                                                         extra['z1'], extra['f1'], extra['g1'])


def _step(dtype):
    step = _Step(dtype, DEVICE)
    step.extra = [torch.zeros_like(step.y0) for _ in EXTRAS]
    return step


def _launches(step):
    return step.lib.tsde_kernel_launches(_cabi.KERNEL_PW_CHUNK)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('name', sorted(PC))
def test_malformed_programs_are_refused_without_a_launch(name, entry, dtype):
    step = _step(dtype)
    prog = _srk(step.mem)
    PC[name](prog)
    before = _launches(step)
    assert _solve(entry, step, prog) == _cabi.EINVAL
    assert _launches(step) == before


CALLS = ['n_steps 0', 'n_steps 65', 'null table', 'null t0 in a middle step', 'null last y1', 'multi-cell chunk',
         'memory noise', 'general noise', 'm != d', '16-bit format']


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('case', CALLS)
def test_bad_calls_are_refused_without_a_launch(case, entry, dtype):
    step = _step(dtype)
    prog = _srk(step.mem)
    kw = {}
    if case == 'n_steps 0':
        kw = {'n': 0}
    elif case == 'n_steps 65':
        kw = {'n': _cabi.PW_MAX_STEPS + 1, 'steps': _table(step, _cabi.PW_MAX_STEPS + 1)}
    elif case == 'null table':
        kw = {'steps': ctypes.POINTER(_cabi.PwStep)()}
    elif case == 'null t0 in a middle step':
        kw = {'n': 3, 'steps': _table(step, 3, t_null=1)}
    elif case == 'null last y1':
        kw = {'steps': _table(step, 2, last_null=True)}
    elif case == 'multi-cell chunk':
        step.nz.n_cells = 2
    elif case == 'memory noise':
        step.nz.source, step.nz.w = _cabi.SRC_MEMORY, step.y0.data_ptr()
    elif case == 'general noise':
        step.L.noise_type = _cabi.NOISE_GENERAL
    elif case == 'm != d':
        step.L.m = D + 1
    elif case == '16-bit format':
        step.L.dtype = _cabi.dtype_code(dtype) | (_cabi.FMT_BF16 << 8)
    before = _launches(step)
    assert _solve(entry, step, prog, **kw) == _cabi.EINVAL
    assert _launches(step) == before


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('null', EXTRAS)
def test_reversible_heun_refuses_a_null_state_pointer(null, dtype):
    step = _step(dtype)
    before = _launches(step)
    assert _solve('reversible_heun', step, _srk(step.mem), null=null) == _cabi.EINVAL
    assert _launches(step) == before


@pytest.mark.parametrize('entry', ENTRIES)
def test_an_empty_batch_is_a_no_op(entry):
    step = _step(torch.float32)
    step.L.rows = 0
    before = _launches(step)
    assert _solve(entry, step, _srk(step.mem)) == 0
    assert _launches(step) == before


# ---- dry run: the launch sequence of a solve -----------------------------------------------------------------------
TS, DT = [0.0, 0.09375, 0.25], 0.0625  # four steps; step 1 holds the interpolated output
# method -> (chunk entry point, argument index of its step table, of its n_steps)
CHUNK = {'euler': ('tsde_solve_euler_pointwise', 4, 5), 'reversible_heun': ('tsde_solve_reversible_heun_pointwise', 7, 8)}
TABLE_AT = {name: (at, n_at) for name, at, n_at in CHUNK.values()}


class _TableLog(_Log):
    """_Log that also reads each chunk's step table while the call is made: (time, dt, stored) per step, the time
    read through its device pointer (a CPU tensor in the dry run)."""

    def __init__(self, lib):
        super().__init__(lib)
        self.tables = []

    def __getattr__(self, name):
        fn = super().__getattr__(name)
        if name not in TABLE_AT:
            return fn

        def entry(*args):
            at, n_at = TABLE_AT[name]
            steps, n = args[at], args[n_at]
            self.tables.append([(ctypes.c_float.from_address(s.t0).value, s.dt, s.y1 is not None)
                                for s in steps[:n]])
            return fn(*args)
        return entry


@pytest.mark.parametrize('method', sorted(CHUNK))
def test_from_the_second_step_on_steps_are_chunks(dry, monkeypatch, method):  # noqa: F811
    log = _TableLog(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    sde_type = 'ito' if method == 'euler' else 'stratonovich'
    sde = problems.make('gbm', 3, 3, sde_type, dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 3), dtype=torch.float32, device='cpu')
    with torch.no_grad():
        ys, extra = tsde.sdeint(sde, torch.ones(4, 3), TS, bm=bm, method=method, dt=DT, extra=True)
    assert ys.shape == (3, 4, 3)
    name, _, n_at = CHUNK[method]
    names = [n for n, _ in log.calls]
    first = names.index(name)
    # the recorded first step ran the unfused kernels; the interpolated step 1 is a chunk of one, steps 2-3 one chunk
    unfused = {'euler': {'tsde_step_euler'}, 'reversible_heun': {'tsde_reversible_heun_z', 'tsde_step_reversible_heun'}}
    assert unfused[method] <= set(names[:first])
    assert names[first:] == [name, 'tsde_linear_interp', name]
    chunks = [args for n, args in log.calls if n == name]
    assert [args[n_at] for args in chunks] == [1, 2]
    # each step's program runs at its t0 (Euler) or t1 (reversible Heun); only the last state of a chunk is stored,
    # as the output rows here lie at the chunk ends
    t = (lambda k: k * DT) if method == 'euler' else (lambda k: (k + 1) * DT)
    assert log.tables == [[(t(1), DT, True)], [(t(2), DT, False), (t(3), DT, True)]]
    if method == 'reversible_heun':
        assert len(extra) == 3 and all(x.shape == (4, 3) for x in extra)
        ins = [tuple(args[4:7]) for args in chunks]
        outs = [tuple(args[9:12]) for args in chunks]
        for i, o in zip(ins, outs):
            assert not set(i) & set(o)          # the chunk never writes what it reads
        assert ins[1] == outs[0]                 # the second chunk starts from the state the first one left
        assert outs[1] == (extra[2].data_ptr(), extra[0].data_ptr(), extra[1].data_ptr())  # (z, f, g) = the result
    else:
        assert extra == ()
