"""An adaptive solve's proposals as one kernel (tsde_adaptive_proposal_pointwise, pointwise.propose) on the CPU: which
adaptive solves record their element-wise program and fuse their proposals, and which keep the unfused steps; that a
fused solve queries the Brownian motion exactly as the unfused one does; that each fused proposal is one proposal
launch and one error reduction; that its sub-step table holds the times, dt and scalars the three unfused steps
compute; and what the library refuses before any launch.  The GPU suite compares the fused solves with the unfused
ones bit for bit (tests/test_gpu_pointwise_adaptive.py)."""
import ctypes

import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import base_solver, pointwise
from . import problems
from .test_host_dry_run import dry  # noqa: F401  (fixture)
from .test_host_pointwise_pc import PC, _Log
from .test_host_pointwise_validation import DEVICE, MILSTEIN, SRK, _milstein, _srk, _Step

PROPOSAL = 'tsde_adaptive_proposal_pointwise'
# method -> (sde_type, levy area, TSDE_PROPOSAL_*)
METHODS = {
    'euler': ('ito', 'none', _cabi.PROPOSAL_EULER),
    'milstein': ('ito', 'none', _cabi.PROPOSAL_MILSTEIN_ITO),
    'milstein_strat': ('stratonovich', 'none', _cabi.PROPOSAL_MILSTEIN_STRATONOVICH),
    'srk': ('ito', 'space-time', _cabi.PROPOSAL_SRK),
    'heun': ('stratonovich', 'none', _cabi.PROPOSAL_HEUN),
    'midpoint': ('stratonovich', 'none', _cabi.PROPOSAL_MIDPOINT),
    'euler_heun': ('stratonovich', 'none', _cabi.PROPOSAL_EULER_HEUN),
}
TS = [0.0, 0.09375, 0.25]
DT = 0.0625


class _LoggedBM:
    """A Brownian motion that logs every query (ta, tb, return_U) and answers it from a BrownianInterval."""

    def __init__(self, bm, log):
        self._bm, self._log = bm, log

    def __getattr__(self, name):
        return getattr(self._bm, name)

    def __call__(self, ta, tb=None, return_U=False, return_A=False):
        self._log.append((float(ta), float(tb), return_U))
        return self._bm(ta, tb, return_U=return_U, return_A=return_A)


def _solve(dry, monkeypatch, method, kind='gbm', fused=True, queries=None, **kw):  # noqa: F811
    """An adaptive no-grad solve of `method` on the dry-run library; the C-ABI calls it made, as (name, args)."""
    log = _Log(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    if not fused:
        monkeypatch.setattr(pointwise, 'proposing', lambda solver: False)
    sde_type, levy, _ = METHODS[method]
    m = 3 if kind == 'gbm' else 2
    sde = problems.make(kind, 3, m, sde_type, dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, m), dtype=torch.float32, device='cpu',
                               levy_area_approximation=levy)
    if queries is not None:
        bm = _LoggedBM(bm, queries)
    with torch.no_grad():
        ys = tsde.sdeint(sde, torch.ones(4, 3), TS, bm=bm, method=method.replace('_strat', ''), dt=DT,
                         adaptive=True, **kw)
    assert ys.shape == (3, 4, 3)
    return log.calls


def _proposals(calls):
    """The solver's launches between two error reductions (Brownian queries and interpolations left out)."""
    out, cur = [], []
    for name, _ in calls:
        if name.startswith('tsde_brownian') or name == 'tsde_linear_interp':
            continue
        cur.append(name)
        if name == 'tsde_adaptive_error_sumsq':
            out.append(cur)
            cur = []
    return out


@pytest.mark.parametrize('method', sorted(METHODS))
def test_the_first_proposal_records_and_every_later_one_is_one_launch(dry, monkeypatch, method):  # noqa: F811
    calls = _solve(dry, monkeypatch, method)
    props = _proposals(calls)
    assert len(props) >= 3
    # the first proposal runs the three unfused steps (the full step records the program) ...
    assert PROPOSAL not in props[0] and len(props[0]) > 3
    # ... every later one is the proposal kernel and the error reduction
    assert all(p == [PROPOSAL, 'tsde_adaptive_error_sumsq'] for p in props[1:]), props
    code = METHODS[method][2]
    assert all(args[2] == code for name, args in calls if name == PROPOSAL)
    names = [name for name, _ in calls]
    # an adaptive solve never takes the counter-noise entry points
    assert not any(n.endswith('_pointwise') and n != PROPOSAL for n in names)
    if method.startswith('milstein'):
        # the proposal kernel is compiled on the recording step; the fixed-step kernels are not
        assert names.count('tsde_adaptive_pointwise_compile') == 1 and 'tsde_pointwise_compile' not in names
        assert names.index('tsde_adaptive_pointwise_compile') < names.index(PROPOSAL)


@pytest.mark.parametrize('method', sorted(METHODS))
def test_the_fused_solve_queries_the_brownian_motion_as_the_unfused_one(dry, monkeypatch, method):  # noqa: F811
    fused, unfused = [], []
    _solve(dry, monkeypatch, method, queries=fused)
    _solve(dry, monkeypatch, method, fused=False, queries=unfused)
    assert fused == unfused and len(fused) >= 9
    assert all(u == (method == 'srk') for _, _, u in fused)


def _read(ptr, dtype=torch.float32):
    return (ctypes.c_float if dtype == torch.float32 else ctypes.c_double).from_address(ptr).value


@pytest.mark.parametrize('method', sorted(METHODS))
def test_the_sub_step_table_is_what_the_unfused_steps_compute(dry, monkeypatch, method):  # noqa: F811
    """Sub-step j of proposal k carries the times, dt and scalars of unfused step 3 k + j of the same solve."""
    code = METHODS[method][2]
    tables = []

    class _Tables(_Log):
        def __getattr__(self, name):
            fn = super().__getattr__(name)
            if name != PROPOSAL:
                return fn

            def entry(*args):
                subs = args[4]
                tables.append([(tuple(_read(t) for t in s.t if t), s.dt, tuple(s.s)) for s in subs])
                assert all(s.w for s in subs) and all(bool(s.u) == (code == _cabi.PROPOSAL_SRK) for s in subs)
                return fn(*args)
            return entry

    steps = []
    real = base_solver.BaseSDESolver._context

    def context(self, t0, t1):
        c = real(self, t0, t1)
        steps.append(c)
        return c

    monkeypatch.setattr(base_solver.BaseSDESolver, '_context', context)
    log = _Tables(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    sde_type, levy, _ = METHODS[method]
    sde = problems.make('gbm', 3, 3, sde_type, dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 3), dtype=torch.float32, device='cpu',
                               levy_area_approximation=levy)
    with torch.no_grad():
        tsde.sdeint(sde, torch.ones(4, 3), TS, bm=bm, method=method.replace('_strat', ''), dt=DT, adaptive=True)
    fused_steps = steps
    steps = []
    monkeypatch.setattr(pointwise, 'proposing', lambda solver: False)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 3), dtype=torch.float32, device='cpu',
                               levy_area_approximation=levy)
    with torch.no_grad():
        tsde.sdeint(sde, torch.ones(4, 3), TS, bm=bm, method=method.replace('_strat', ''), dt=DT, adaptive=True)
    assert tables and len(steps) == len(fused_steps) == 3 * (len(tables) + 1)

    def want(c):
        s = c.scalars
        if code == _cabi.PROPOSAL_SRK:
            return tuple(float(t) for t in c.aux_t), c.dt, (s['rdt'], s['sqrt_dt'], s['three_dt'])
        if code == _cabi.PROPOSAL_MIDPOINT:
            return (float(c.t0), float(c.aux_t[0])), c.dt, (s['half_dt'], 0.0, 0.0)
        if code in (_cabi.PROPOSAL_HEUN, _cabi.PROPOSAL_EULER_HEUN):
            return (float(c.t0), float(c.t1)), c.dt, (0.0, 0.0, 0.0)
        return (float(c.t0),), c.dt, (0.0, 0.0, 0.0)

    for k, table in enumerate(tables):
        assert table == [want(c) for c in steps[3 * (k + 1):3 * (k + 2)]], k


def _count(calls):
    return sum(1 for name, _ in calls if name == PROPOSAL)


@pytest.mark.parametrize('case', ['reversible_heun', 'grad', 'logqp', 'overlap False', 'autocast', 'general noise',
                                  'additive srk', 'grad-free milstein', 'user f_and_g'])
def test_what_keeps_the_unfused_proposals(dry, monkeypatch, case):  # noqa: F811
    log = _Log(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    method, kind, sde_type, levy, kw = 'euler', 'gbm', 'ito', 'none', {}
    grad = case == 'grad'
    if case == 'reversible_heun':
        method, sde_type = 'reversible_heun', 'stratonovich'
    elif case == 'logqp':
        kw = {'logqp': True}
    elif case == 'overlap False':
        kw = {'options': {'overlap': False}}
    elif case == 'autocast':
        monkeypatch.setattr(torch, 'is_autocast_enabled', lambda *a: True)
    elif case == 'general noise':
        kind = 'general'
    elif case == 'additive srk':
        method, kind, levy = 'srk', 'additive', 'space-time'
    elif case == 'grad-free milstein':
        method, kw = 'milstein', {'options': {'grad_free': True}}
    m = 3 if kind == 'gbm' else 2
    sde = problems.make(kind, 3, m, sde_type, dtype=torch.float32)
    if case == 'logqp':
        sde.h = lambda t, y: 0 * y
    if case == 'user f_and_g':
        method, sde_type = 'heun', 'stratonovich'
        sde = problems.make(kind, 3, m, sde_type, dtype=torch.float32)
        sde.f_and_g = lambda t, y: (sde.f(t, y), sde.g(t, y))
    # (logqp=True integrates the augmented state, one column wider)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, m + (case == 'logqp')), dtype=torch.float32, device='cpu',
                               levy_area_approximation=levy)
    y0 = torch.ones(4, 3).requires_grad_(grad)
    with torch.set_grad_enabled(grad):
        out = tsde.sdeint(sde, y0, TS, bm=bm, method=method, dt=DT, adaptive=True, **kw)
    ys = out[0] if isinstance(out, tuple) else out
    assert ys.shape == (3, 4, 3) and 'tsde_adaptive_error_sumsq' in [n for n, _ in log.calls]
    assert _count(log.calls) == 0


def test_sdeint_adjoint_fuses_its_forward_solve_only(dry, monkeypatch):  # noqa: F811
    log = _Log(dry)
    monkeypatch.setattr(_cabi, '_lib', log)
    monkeypatch.setattr(_cabi, 'lib', lambda: log)
    sde = problems.make('gbm', 3, 3, 'ito', dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 3), dtype=torch.float32, device='cpu')
    y0 = torch.ones(4, 3).requires_grad_()
    ys = tsde.sdeint_adjoint(sde, y0, TS, bm=bm, method='milstein', dt=DT, adaptive=True, adjoint_adaptive=True,
                             adjoint_method='milstein')
    forward = _count(log.calls)
    assert forward > 0
    del log.calls[:]
    ys.sum().backward()
    assert y0.grad is not None and 'tsde_adaptive_error_sumsq' in [n for n, _ in log.calls]
    assert _count(log.calls) == 0


# ---- what the C entry point refuses ---------------------------------------------------------------------------------
def _proposal(step, prog, method, y0=True, subs=True, y_full=True, y_next=True, drop=None):
    """tsde_adaptive_proposal_pointwise on _Step's tensors; `drop` = (sub-step, field) set to null."""
    table = (_cabi.PwSubstep * 3)()
    for s in table:
        s.w, s.u, s.dt = step.y1.data_ptr(), step.y1.data_ptr(), 0.125
        for i in range(4):
            s.t[i] = step.t[i:].data_ptr()
        s.s[0], s.s[1], s.s[2] = 8.0, 0.125 ** 0.5, 0.375
    if drop is not None:
        k, field = drop
        if field.startswith('t'):
            table[k].t[int(field[1:])] = None
        else:
            setattr(table[k], field, None)
    return step.lib.tsde_adaptive_proposal_pointwise(
        ctypes.byref(step.L), ctypes.byref(prog), method, step.y0.data_ptr() if y0 else None,
        table if subs else None, step.y1.data_ptr() if y_full else None, step.y0.data_ptr() if y_next else None)


def _launches(step):
    return step.lib.tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE)


def _layout(code):
    if code in (_cabi.PROPOSAL_MILSTEIN_ITO, _cabi.PROPOSAL_MILSTEIN_STRATONOVICH):
        return _milstein, MILSTEIN
    return _srk, SRK if code == _cabi.PROPOSAL_SRK else PC


CODES = sorted(c for _, _, c in METHODS.values())


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('code,name', [(c, n) for c in CODES for n in sorted(_layout(c)[1])])
def test_malformed_programs_are_refused_without_a_launch(code, name, dtype):
    step = _Step(dtype, DEVICE)
    make, table = _layout(code)
    prog = make(step.mem)
    table[name](prog)
    before = _launches(step)
    assert _proposal(step, prog, code) == _cabi.EINVAL
    assert _launches(step) == before


@pytest.mark.parametrize('code', CODES)
def test_a_program_of_another_layout_is_refused(code):
    step = _Step(torch.float32, DEVICE)
    other = _srk if _layout(code)[0] is _milstein else _milstein
    assert _proposal(step, other(step.mem), code) == _cabi.EINVAL


def _needs(code):
    """The sub-step fields a method reads."""
    times = 4 if code == _cabi.PROPOSAL_SRK else 2 if code >= _cabi.PROPOSAL_HEUN else 1
    return ['w'] + (['u'] if code == _cabi.PROPOSAL_SRK else []) + [f't{i}' for i in range(times)]


BAD = [(c, f'null {f} of sub-step {k}') for c in CODES for f in _needs(c) for k in range(3)] + \
      [(c, case) for c in CODES for case in ('null y0', 'null subs', 'null y_full', 'null y_next')] + \
      [(-1, 'method -1'), (7, 'method 7')]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('code,case', BAD)
def test_bad_calls_are_refused_without_a_launch(code, case, dtype):
    step = _Step(dtype, DEVICE)
    prog = _layout(max(code, 0) if code < 7 else 0)[0](step.mem)
    kw = {}
    if case.startswith('null') and ' of sub-step ' in case:
        field, k = case[5:].split(' of sub-step ')
        kw['drop'] = (int(k), field)
    elif case.startswith('null'):
        kw[case[5:]] = False
    before = _launches(step)
    assert _proposal(step, prog, code, **kw) == _cabi.EINVAL
    assert _launches(step) == before
