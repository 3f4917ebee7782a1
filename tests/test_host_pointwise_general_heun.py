"""General- and additive-noise Euler-Heun and reversible-Heun element-wise steps on the host (no GPU): the layout tag
each general method's recorder gives its program, the translation units of the two new tags, the contraction order
each of their sums spells out for every m (Euler-Heun's predict and final products share one; reversible Heun's z and
y products follow the dense g of the unfused pair whatever the g source), the calls the library refuses before
launching anything, and dry runs of the solvers reaching the GENERAL launches with (rows, d, m) solver state."""
import ctypes

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import methods, pointwise
from .test_host_dry_run import dry  # noqa: F401  (the fixture)
from .test_host_pointwise_general import B, D, _contraction, _expected_contraction, _route, accepted

EH, RH = _cabi.PW_LAYOUT_GENERAL_EULER_HEUN, _cabi.PW_LAYOUT_GENERAL_REVERSIBLE_HEUN
KERNELS = ['tsde_pw_general_euler_single', 'tsde_pw_general_euler_multi', 'tsde_pw_general_midpoint_single',
           'tsde_pw_general_midpoint_multi', 'tsde_pw_general_sra1_single', 'tsde_pw_general_sra1_multi',
           'tsde_pw_general_euler_heun_single', 'tsde_pw_general_euler_heun_multi',
           'tsde_pw_general_reversible_heun_single', 'tsde_pw_general_reversible_heun_multi']


def record(f, g, m, layout, dtype=torch.float32):
    """GeneralRecorder over one step of the method of `layout`: f, g, g for Euler-Heun, f, g for reversible Heun."""
    pattern = 'fgg' if layout == EH else 'fg'
    y = torch.rand(B, D, dtype=dtype) + 0.1
    t = torch.tensor(0.25, dtype=dtype)
    rec = pointwise.GeneralRecorder(y, t, pattern, m, False, layout)
    for kind in pattern:
        rec.evaluation(kind, (lambda: f(t, y)) if kind == 'f' else (lambda: g(t, y)), t, y)
    return rec, rec.finish()


def test_the_method_classes_carry_their_layouts():
    assert methods.Euler._pw_layout == methods.Midpoint._pw_layout == _cabi.PW_LAYOUT_GENERAL
    assert methods.SRK._pw_layout == _cabi.PW_LAYOUT_GENERAL_SRA
    assert methods.EulerHeun._pw_layout == EH and methods.ReversibleHeun._pw_layout == RH
    assert all(c._pw_general for c in (methods.Euler, methods.Midpoint, methods.SRK, methods.EulerHeun,
                                       methods.ReversibleHeun))
    assert not getattr(methods.Heun, '_pw_general', False)


@pytest.mark.parametrize('layout', [EH, RH])
@pytest.mark.parametrize('kind', sorted(accepted()))
def test_each_tag_has_its_own_unit(kind, layout):
    rec, res = record(*accepted()[kind], 16, layout)
    assert res is not None, rec.reason
    assert res[0].reserved == layout
    src = _cabi.general_pointwise_source(res[0], torch.float32, D, 16)
    name = 'euler_heun' if layout == EH else 'reversible_heun'
    mine = {f'tsde_pw_general_{name}_single', f'tsde_pw_general_{name}_multi'}
    assert {k for k in KERNELS if f'void __launch_bounds__(256, 1)\n{k}(' in src} == mine
    # Euler-Heun evaluates g as the midpoint unit does; reversible Heun keeps g in registers instead
    assert ('void gp(' in src) == (layout == EH)
    assert ('void dot(' in src and 'void gstep(' in src and 'static constexpr int M = 16;' in src) == (layout == RH)


def test_the_existing_units_keep_their_text():
    """Re-tagging a program changes only the translation unit, and the Euler / midpoint and sra1 units' Prog are the
    Euler-Heun unit's."""
    _, res = record(*accepted(8)['correlated_gbm'], 8, EH)
    prog = res[0]
    units = {}
    for tag in (_cabi.PW_LAYOUT_GENERAL, _cabi.PW_LAYOUT_GENERAL_SRA, EH):
        p = _cabi.Pointwise.from_buffer_copy(prog)
        p.reserved = tag
        units[tag] = _cabi.general_pointwise_source(p, torch.float32, D, 8).split('\nextern "C"')[0]
    assert units[_cabi.PW_LAYOUT_GENERAL] == units[_cabi.PW_LAYOUT_GENERAL_SRA] == units[EH]


def _function(src, name):
    """The lines of Prog member `name` of a generated unit."""
    lines = [ln.strip() for ln in src.splitlines()]
    start = next(i for i, ln in enumerate(lines) if f' void {name}(' in ln)
    return lines[start:lines.index('out[j] = acc;', start) + 1]


def _rh_contractions(src):
    """The statements of reversible Heun's z product (dot) and y product (gstep, after its G lambda)."""
    dot = _function(src, 'dot')
    dot = dot[dot.index('for (int j = 0; j < 4; ++j) {') + 1:-1]
    gstep = _function(src, 'gstep')
    return dot, gstep[gstep.index('};', gstep.index('auto G = [&](int k) -> T {')) + 1:-1]


def _substituted(lines, value, pre=None, post=None):
    """The statements of a route with G(k) replaced by value(k), and pre(k) / post(k) around channel k's term."""
    out = []
    for ln in lines:
        ks = [k for k in range(_cabi.PW_GENERAL_MAX_M) if f'G({k})' in ln]
        if not ks:
            out.append(ln)
            continue
        k, = ks
        out += ([pre(k)] if pre else []) + [ln.replace(f'G({k})', value(k))] + ([post(k)] if post else [])
    return out


def _expected_rh(route, m, fs):
    exp = _expected_contraction(route, m, fs)
    dot = _substituted(exp, lambda k: f'op.gval(0, {{gs[j][{k}]}})')
    gstep = _substituted(exp, lambda k: f'op.gval(0, {{gs[j][{k}], h{k}}})', lambda k: f'const T h{k} = G({k});',
                         lambda k: f'gs[j][{k}] = h{k};')
    return dot, gstep


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', list(range(1, _cabi.PW_GENERAL_MAX_M + 1)))
def test_the_generated_contractions_follow_the_route(m, dtype):
    fs = 'f' if dtype == torch.float32 else ''
    # Euler-Heun: the predict and the final launch both contract g.dW with one route (the final one's first product
    # is the predictor's): the unit's one gp
    rec, res = record(*accepted(m, dtype)['correlated_gbm'], m, EH, dtype)
    assert res is not None, rec.reason
    assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
        _route(m, True), m, fs)
    rec, res = record(*accepted(m, dtype)['where_clamp'], m, RH, dtype)
    assert res is not None, rec.reason
    assert _rh_contractions(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_rh(
        _route(m, True), m, fs)
    # a DM operand as g: Euler-Heun's launches read the user's block where it is (a misaligned one takes gen_kernel's
    # order); the reversible-Heun pair reads its densified solver state, so the block's address does not matter
    store = torch.zeros(D * m + 1, dtype=dtype)
    for S, quads in ((torch.rand(D, m, dtype=dtype), True), (store[1:].view(D, m), False)):
        aligned = S.data_ptr() % 16 == 0
        rec, res = record(lambda t, y: -y, lambda t, y: S.expand(B, D, m), m, EH, dtype)
        assert res is not None, rec.reason
        assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
            _route(m, quads and aligned), m, fs)
        rec, res = record(lambda t, y: -y, lambda t, y: S.expand(B, D, m), m, RH, dtype)
        assert res is not None, rec.reason
        assert _rh_contractions(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_rh(
            _route(m, True), m, fs)


def test_bad_calls_are_refused_without_a_launch():
    lib = _cabi.lib()
    _, res = record(*accepted(4)['correlated_gbm'], 4, EH)
    eh = res[0]
    _, res = record(*accepted(4)['correlated_gbm'], 4, RH)
    rh = res[0]
    n0 = lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL)
    nz = _cabi.Noise()
    nz.source = _cabi.SRC_COUNTER
    memory = _cabi.Noise()
    memory.source = _cabi.SRC_MEMORY
    flagged = _cabi.Noise()
    flagged.source, flagged.flags = _cabi.SRC_COUNTER, _cabi.FLAG_G_BROADCAST
    general = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, 4, None)
    wide = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, _cabi.PW_GENERAL_MAX_M + 1, None)
    half = _cabi.Launch(_cabi.F32 | _cabi.FMT_BF16 << 8, _cabi.NOISE_GENERAL, 4, D, 4, None)

    def retag(p, tag):
        q = _cabi.Pointwise.from_buffer_copy(p)
        q.reserved = tag
        return q

    def pc(L, p, method=_cabi.PC_EULER_HEUN, noise=nz, times=(16, 16), y=(16, 32)):
        return lib.tsde_step_predictor_corrector_pointwise(ctypes.byref(L), ctypes.byref(noise), ctypes.byref(p), y[0],
                                                           *times, method, 0.1, 0.05, y[1])

    for L in (wide, half):
        assert pc(L, eh) == _cabi.EINVAL
    assert pc(general, eh, noise=memory) == _cabi.EINVAL
    assert pc(general, eh, noise=flagged) == _cabi.EINVAL
    for times in ((None, 16), (16, None)):
        assert pc(general, eh, times=times) == _cabi.EINVAL
    for y in ((None, 32), (16, None)):
        assert pc(general, eh, y=y) == _cabi.EINVAL
    # Heun stays unfused; Euler-Heun and midpoint each take their own tag only
    assert pc(general, eh, _cabi.PC_HEUN) == _cabi.EINVAL
    assert pc(general, eh, _cabi.PC_MIDPOINT) == _cabi.EINVAL
    for tag in (0, _cabi.PW_LAYOUT_GENERAL, _cabi.PW_LAYOUT_GENERAL_SRA, RH):
        assert pc(general, retag(eh, tag)) == _cabi.EINVAL

    steps = (_cabi.PwStep * 1)()
    steps[0].t0, steps[0].y1 = 16, 32

    def chunk(L, p, noise=nz, n_steps=1, y0=16, state=(48, 64, 80), out=(96, 112, 128)):
        return lib.tsde_solve_reversible_heun_pointwise(ctypes.byref(L), ctypes.byref(noise), ctypes.byref(p), y0,
                                                        *state, steps, n_steps, *out)

    for L in (wide, half):
        assert chunk(L, rh) == _cabi.EINVAL
    assert chunk(general, rh, noise=memory) == _cabi.EINVAL
    assert chunk(general, rh, noise=flagged) == _cabi.EINVAL
    for n_steps in (0, _cabi.PW_MAX_STEPS + 1):
        assert chunk(general, rh, n_steps=n_steps) == _cabi.EINVAL
    assert chunk(general, rh, y0=None) == _cabi.EINVAL
    for i in range(3):
        state, out = [48, 64, 80], [96, 112, 128]
        state[i] = None
        assert chunk(general, rh, state=tuple(state)) == _cabi.EINVAL
        out[i] = None
        assert chunk(general, rh, out=tuple(out)) == _cabi.EINVAL
    for tag in (0, _cabi.PW_LAYOUT_GENERAL, _cabi.PW_LAYOUT_GENERAL_SRA, EH):
        assert chunk(general, retag(rh, tag)) == _cabi.EINVAL
    # and the Euler, midpoint and sra1 entries refuse both new tags
    for p in (eh, rh):
        assert lib.tsde_solve_euler_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(p), 16, steps,
                                              1) == _cabi.EINVAL
        assert pc(general, p, _cabi.PC_MIDPOINT) == _cabi.EINVAL
        assert lib.tsde_step_srk_diag_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(p), 16, 16, 16,
                                                16, None, 0.1, 10.0, 0.0, 0.0, 32) == _cabi.EINVAL
        assert _cabi.general_pointwise_source(p, torch.float32, D, _cabi.PW_GENERAL_MAX_M + 1) is None
    assert lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL) == n0


# ---- dry runs ---------------------------------------------------------------------------------------------------------
class GBM(nn.Module):
    """Correlated multi-asset GBM (general noise), or OU with an additive `expand`."""

    def __init__(self, d, m, sde_type, additive=False):
        super().__init__()
        self.sde_type, self.noise_type = sde_type, 'additive' if additive else 'general'
        self.mu, self.S = nn.Parameter(torch.rand(d) - 0.5), nn.Parameter(torch.rand(d, m))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        if self.noise_type == 'additive':
            return self.S.expand(y.size(0), *self.S.shape)
        return y.unsqueeze(-1) * self.S


class _Spy:
    """The recording stand-in library, keeping every call's arguments."""

    def __init__(self, lib):
        self.lib, self.args = lib, {}

    def __getattr__(self, name):
        fn = getattr(self.lib, name)

        def entry(*a):
            self.args.setdefault(name, []).append(a)
            return fn(*a)
        return entry


@pytest.fixture
def spy(dry, monkeypatch):  # noqa: F811
    s = _Spy(dry)
    monkeypatch.setattr(_cabi, '_lib', s)
    monkeypatch.setattr(_cabi, 'lib', lambda: s)
    tags = []
    real = pointwise.compile_general

    def compile_general(solver, rec, res):
        tags.append((type(solver).__name__, None if res is None else res[0].reserved))
        return real(solver, rec, res)
    monkeypatch.setattr(pointwise, 'compile_general', compile_general)
    s.tags = tags
    return s


def _solve(method, sde_type, m=3, d=5, additive=False, adjoint=False, options=None):
    sde = GBM(d, m, sde_type, additive)
    bm = tsde.BrownianInterval(0.0, 0.25, size=(4, m), dtype=torch.float32, device='cpu',
                               levy_area_approximation='space-time' if method == 'srk' else 'none')
    y0 = torch.ones(4, d)
    ts = torch.tensor([0.0, 0.125, 0.25])
    if adjoint:
        y0.requires_grad_(True)
        ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method=method, dt=0.0625, options=dict(options or {}))
        ys.sum().backward()
        return ys
    with torch.no_grad():
        return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=0.0625, options=dict(options or {}))


def _general_launches(spy, name, m):
    calls = spy.args.get(name, [])
    return [a for a in calls if a[0]._obj.noise_type == _cabi.NOISE_GENERAL and a[0]._obj.m == m]


def test_the_five_general_methods_tag_their_programs(spy):
    for method, sde_type, additive in (('euler', 'ito', False), ('midpoint', 'stratonovich', False),
                                       ('srk', 'ito', True), ('euler_heun', 'stratonovich', False),
                                       ('reversible_heun', 'stratonovich', False)):
        _solve(method, sde_type, additive=additive)
    assert spy.tags == [('Euler', _cabi.PW_LAYOUT_GENERAL), ('Midpoint', _cabi.PW_LAYOUT_GENERAL),
                        ('SRK', _cabi.PW_LAYOUT_GENERAL_SRA), ('EulerHeun', EH), ('ReversibleHeun', RH)]


@pytest.mark.parametrize('additive', [False, True])
@pytest.mark.parametrize('options', [{}, {'cuda_graph': True}])
def test_a_euler_heun_solve_reaches_the_fused_step(spy, options, additive):
    m = 3
    _solve('euler_heun', 'stratonovich', m, additive=additive, options=options)
    assert spy.tags == [('EulerHeun', EH)]
    fused = _general_launches(spy, 'tsde_step_predictor_corrector_pointwise', m)
    assert fused and all(a[6] == _cabi.PC_EULER_HEUN for a in fused)
    assert all(len(a) == len(_cabi.SIGNATURES['tsde_step_predictor_corrector_pointwise']) for a in fused)
    # the recording step ran the unfused pair
    assert len(spy.args['tsde_euler_heun_predict']) >= 1 and len(spy.args['tsde_step_euler_heun']) >= 1


@pytest.mark.parametrize('adjoint', [False, True])
@pytest.mark.parametrize('options', [{}, {'cuda_graph': True}])
def test_a_reversible_heun_solve_chunks_with_general_state(spy, monkeypatch, options, adjoint):
    m, d = 3, 5
    states = []
    real = pointwise.solve_chunk

    def solve_chunk(solver, ctxs, y0, outs, method, ito=0, state=None):
        states.append(state)
        return real(solver, ctxs, y0, outs, method, ito, state)
    monkeypatch.setattr(pointwise, 'solve_chunk', solve_chunk)
    _solve('reversible_heun', 'stratonovich', m, d, adjoint=adjoint, options=options)
    assert spy.tags == [('ReversibleHeun', RH)]
    fused = _general_launches(spy, 'tsde_solve_reversible_heun_pointwise', m)
    assert fused and len(fused) == len(states)
    # (z, f, g) in and out: g is (rows, d, m), and a chunk never stores to the set it reads
    for (z0, f0, g0), (z1, f1, g1) in states:
        assert tuple(z0.shape) == tuple(f0.shape) == tuple(z1.shape) == tuple(f1.shape) == (4, d)
        assert tuple(g0.shape) == tuple(g1.shape) == (4, d, m)
        assert {x.data_ptr() for x in (z0, f0, g0)}.isdisjoint(x.data_ptr() for x in (z1, f1, g1))
    # the recording step ran the unfused pair; the adjoint's backward keeps its own kernels
    assert len(spy.args['tsde_reversible_heun_z']) >= 1
    if adjoint:
        assert len(spy.args['tsde_adjoint_reversible_heun_a']) >= 1


def test_state_fits_reads_the_general_state_shape():
    class Solver:
        rows, d, m, dtype, device = 4, 5, 3, torch.float32, torch.device('cpu')
        sde = GBM(5, 3, 'stratonovich')
    s = Solver()
    f, z, g = torch.zeros(4, 5), torch.zeros(4, 5), torch.zeros(4, 5, 3)
    assert pointwise.state_fits(s, (f, g, z))
    assert not pointwise.state_fits(s, (f, torch.zeros(4, 5), z))
    assert not pointwise.state_fits(s, (f, g.transpose(1, 2).contiguous().transpose(1, 2), z))
    # a g the unfused pair would not read as quads
    store = torch.zeros(4 * 5 * 3 + 1)
    assert not pointwise.state_fits(s, (f, store[1:].view(4, 5, 3), z))
