"""A diagonal-noise Heun, midpoint or Euler-Heun step as one kernel (tsde_step_predictor_corrector_pointwise,
torchsde_b200/_core/pointwise.py pc_recorder).

The fused step must give the unfused step's bits.  The unfused reference is the same solve with the tape rejected
(SrkRecorder.finish patched to return None); the route is confirmed by the launch counter TSDE_KERNEL_PW_PC.  Covered,
for each of the three methods: the Stratonovich SDEs of tests/test_gpu_pointwise.py and one whose f and g depend on t
differently, float32 and float64, eager, graph and row_split; stage times; multi-cell steps; shards past global row
2^24 at d = 12; the element path (d = 7, a misaligned parameter); a cfg2-sized graph solve; an in-place parameter
update between replays; the solves that keep the unfused step; and a float64 solve against the numpy oracle on the
oracle's increments.  `sdeint` without a method fuses a Stratonovich element-wise SDE (midpoint)."""
import contextlib

import numpy as np
import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from oracle import solvers
from . import helpers, problems
from .test_gpu_pointwise import MODES, SDE, Nonlinear, same_bits
from .test_gpu_pointwise_srk import Unbound

pytestmark = pytest.mark.gpu
DEV = 'cuda'
METHODS = ['heun', 'midpoint', 'euler_heun']


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_PC)


@contextlib.contextmanager
def unfused():
    """The tape is always rejected: every step runs the user's ops and the unfused kernels."""
    finish = pointwise.SrkRecorder.finish
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.SrkRecorder.finish = finish


class TimeSDE(SDE):
    """f and g read t differently: a stage time taken from the wrong slot changes the bits."""

    def __init__(self, B, d, dtype):
        super().__init__('gbm', 'stratonovich', B, d, dtype)

    def f(self, t, y):
        return (t * self.mu) * y

    def g(self, t, y):
        return (t * t + self.sigma) * y


def make_sde(kind, B, d, dtype):
    return (TimeSDE(B, d, dtype) if kind == 'time2' else SDE(kind, 'stratonovich', B, d, dtype)).to(DEV)


def solve(sde, y0, T, dt, method, options=None, row_offset=0, cell=None, entropy=11):
    B, m = y0.shape
    bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy,
                               **({'dt': cell} if cell else {}))
    if row_offset:
        bm.shard_rows(row_offset)
    ts = torch.arange(T + 1, dtype=y0.dtype, device=DEV) * dt
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options or {}))
    graph.drop_plans(sde)
    return ys


def check_fused(sde, y0, T, dt, method, options=None, **kw):
    n0 = fused_launches()
    ys = solve(sde, y0, T, dt, method, options, **kw)
    assert fused_launches() > n0, "the step was not fused"
    with unfused():
        n1 = fused_launches()
        ref = solve(sde, y0, T, dt, method, options, **kw)
        assert fused_launches() == n1
    assert same_bits(ys, ref)
    return ys


KINDS = ['gbm', 'div', 'in_place', 'time2']  # the Stratonovich SDEs of test_gpu_pointwise.py, and TimeSDE


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('method', METHODS)
def test_small_solves_are_bit_identical(method, kind, dtype, mode):
    B, d = 96, 16
    sde = make_sde(kind, B, d, dtype)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    check_fused(sde, y0, 12, 2.0 ** -6, method, MODES[mode])


@pytest.mark.parametrize('method', ['heun', 'midpoint'])
def test_stage_times_matter(method):
    """The second evaluation runs at t1 (Heun) or t0 + dt/2 (midpoint): moving f's time moves the fused bits, and the
    fused solve still equals the unfused one."""
    B, d, dt = 32, 8, 2.0 ** -5
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    a = check_fused(make_sde('time2', B, d, torch.float64), y0, 4, dt, method)
    shifted = TimeSDE(B, d, torch.float64).to(DEV)
    shifted.f = lambda t, y: ((t + dt / 4) * shifted.mu) * y
    b = check_fused(shifted, y0, 4, dt, method)
    assert not torch.equal(a, b)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_multi_cell_steps(method, dtype):
    B, d, dt = 40, 8, 2.0 ** -5
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    check_fused(make_sde('time2', B, d, dtype), y0, 5, dt, method, cell=dt / 4)


@pytest.mark.parametrize('method', METHODS)
def test_cfg2_sized_graph_solve_is_bit_identical(method):
    B, d = 65536, 64
    y0 = torch.full((B, d), 0.1, device=DEV)
    check_fused(make_sde('gbm', B, d, torch.float32), y0, 8, 2.0 ** -10, method,
                {'cuda_graph': True, 'static_output': False})


@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_shards_past_row_2_24_at_a_width_of_three_quads(method, dtype, mode):
    B, d = 300, 12
    sde = make_sde('gbm', B, d, dtype)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ys = check_fused(sde, y0, 6, 2.0 ** -5, method, MODES[mode], row_offset=(1 << 24) + 5)
    other = check_fused(sde, y0, 6, 2.0 ** -5, method, MODES[mode], row_offset=(1 << 24) + 6)
    assert not torch.equal(ys[-1], other[-1])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_element_path_odd_width_and_misaligned_parameter(method, dtype):
    B = 50
    sde = make_sde('div', B, 7, dtype)
    check_fused(sde, torch.full((B, 7), 0.4, dtype=dtype, device=DEV), 5, 2.0 ** -5, method, {'cuda_graph': True})
    sde = make_sde('gbm', B, 8, dtype)
    with torch.no_grad():
        store = torch.zeros(9, dtype=dtype, device=DEV)
        store[1:].copy_(sde.sigma)
        sde.sigma = nn.Parameter(store[1:])
    assert sde.sigma.data_ptr() % 16
    check_fused(sde, torch.full((B, 8), 0.4, dtype=dtype, device=DEV), 5, 2.0 ** -5, method)


@pytest.mark.parametrize('method', METHODS)
def test_in_place_parameter_update_between_replays_is_followed(method):
    B, d = 64, 8
    sde = make_sde('time2', B, d, torch.float32)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(5, device=DEV) * 2.0 ** -5

    def run():
        bm = tsde.BrownianInterval(0.0, 4 * 2.0 ** -5, size=(B, d), device=DEV, entropy=3)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -5, options={'cuda_graph': True})

    first = run()
    with torch.no_grad():
        sde.sigma.mul_(1.5)
        sde.mu.add_(0.25)
    second = run()                # a replay of the same plan
    graph.drop_plans(sde)
    with unfused():
        want = run()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


def test_the_default_stratonovich_method_is_fused():
    """`sdeint` without `method` solves a Stratonovich SDE with midpoint: a diagonal element-wise one is fused."""
    B, d, T, dt = 64, 8, 6, 2.0 ** -5
    sde = make_sde('gbm', B, d, torch.float32)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * dt

    def run():
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, d), device=DEV, entropy=7)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, dt=dt)

    n0 = fused_launches()
    ys = run()
    assert fused_launches() == n0 + T - 1
    with unfused():
        assert same_bits(ys, run())
    assert same_bits(ys, solve(sde, y0, T, dt, 'midpoint', entropy=7))


class Branching(SDE):
    """g takes another (equally element-wise) branch on its second call: the tapes of one step differ."""

    def __init__(self, B, d):
        super().__init__('gbm', 'stratonovich', B, d, torch.float32)
        self.calls = 0

    def g(self, t, y):
        self.calls += 1
        return (self.sigma * y) * 1 if self.calls == 2 else self.sigma * y


FALLBACKS = ['sigmoid', 'exp', 'item', 'f_and_g', 'g_prod', 'scalar', 'additive', 'general', 'grad', 'logqp',
             'autocast', 'overlap', 'unbound', 'branch']


@pytest.mark.parametrize('case', FALLBACKS)
@pytest.mark.parametrize('method', METHODS)
def test_unfusable_solves_keep_the_unfused_step(method, case):
    B, d, T, dt = 32, 8, 6, 2.0 ** -5
    if case == 'branch':
        sde = Branching(B, d).to(DEV)
    else:
        sde = Nonlinear(case, B, d).to(DEV)
        sde.sde_type = 'stratonovich'
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * dt
    kw, ctx, m = {}, contextlib.nullcontext, d
    if case == 'logqp':
        kw['logqp'], m = True, d + 1
    if case == 'autocast':
        ctx = lambda: torch.autocast('cuda', dtype=torch.bfloat16)  # noqa: E731
    if case == 'overlap':
        kw['options'] = {'overlap': False}
    if case == 'f_and_g':   # f and g from one user call (f and g exist too: Euler-Heun's second evaluation calls g)
        sde.f_and_g = lambda t, y: (sde.f(t, y), sde.g(t, y))
    if case == 'g_prod':
        sde.g_prod = lambda t, y, v: sde.g(t, y) * v
    if case == 'scalar':
        sde.noise_type, m = 'scalar', 1
        sde.g = lambda t, y: (sde.sigma * y).unsqueeze(-1)
    if case == 'additive':
        sde.noise_type = 'additive'
        sde.g = lambda t, y: torch.full((B, d, d), 0.1, device=DEV)
    if case == 'general':
        sde.noise_type, m = 'general', 2
        sde.g = lambda t, y: torch.stack([sde.sigma * y, 0.5 * sde.sigma * y], dim=-1)

    def run():
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), device=DEV, entropy=5)
        if case == 'unbound':
            bm = Unbound(bm)
        if case == 'branch':
            sde.calls = 0
        with (torch.enable_grad() if case == 'grad' else torch.no_grad()), ctx():
            y = y0.clone().requires_grad_(case == 'grad')
            out = tsde.sdeint(sde, y, ts, bm=bm, method=method, dt=dt, **kw)
        out = out if isinstance(out, tuple) else (out,)
        return tuple(o.detach() for o in out)

    n0 = fused_launches()
    out = run()
    assert fused_launches() == n0
    with unfused():
        ref = run()
    for x, r in zip(out, ref):
        assert same_bits(x, r)


@pytest.mark.parametrize('method', ['heun', 'midpoint'])
def test_the_adjoint_backward_keeps_the_unfused_step(method):
    """`sdeint_adjoint`: the forward pass is an ordinary no-grad solve of the user's SDE and is fused; the backward
    solve of the adjoint SDE (adjoint_method = method) is not.  Solutions and gradients equal those of the same solve
    with the tape rejected."""
    B, d, T, dt = 32, 8, 6, 2.0 ** -5
    ts = torch.arange(T + 1, device=DEV) * dt
    out = []
    for ctx in (contextlib.nullcontext, unfused):
        with ctx():
            sde = SDE('gbm', 'stratonovich', B, d, torch.float32).to(DEV)
            y0 = torch.full((B, d), 0.2, device=DEV, requires_grad=True)
            bm = tsde.BrownianInterval(0.0, T * dt, size=(B, d), device=DEV, entropy=9)
            n0 = fused_launches()
            ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method=method, adjoint_method=method, dt=dt)
            n1 = fused_launches()
            ys.pow(2).sum().backward()
            assert fused_launches() == n1
            assert (n1 > n0) == (ctx is contextlib.nullcontext)
            out.append([ys.detach(), y0.grad, sde.sigma.grad, sde.mu.grad])
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize('method', METHODS)
def test_a_fused_solve_matches_the_oracle_on_its_increments(method):
    """float64 against oracle/solvers.py on the oracle's Philox increments (sampled rows)."""
    B, d, dt = 512, 8, 2.0 ** -4
    sde = problems.GBMDiagonal(d, 'stratonovich', seed=3, dtype=torch.float64).to(DEV)
    y0 = torch.full((B, d), 0.5, dtype=torch.float64, device=DEV)
    ts = torch.tensor([0.0, 0.25, 0.5], dtype=torch.float64, device=DEV)
    bm = tsde.BrownianInterval(0.0, 0.5, size=(B, d), dtype=torch.float64, device=DEV, entropy=404)
    n0 = fused_launches()
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt)
    assert fused_launches() > n0
    rows = np.arange(0, B, 7)
    sde_cpu = problems.GBMDiagonal(d, 'stratonovich', seed=3, dtype=torch.float64)
    ref, _ = solvers.make(method, problems.NumpySDE(sde_cpu), helpers.oracle_grid_bm(bm, rows, d, np.float64, False),
                          dt).integrate(y0[torch.from_numpy(rows).to(DEV)].cpu().numpy(), ts.cpu().numpy())
    np.testing.assert_allclose(ys[:, torch.from_numpy(rows).to(DEV)].cpu().numpy(), ref, rtol=1e-9, atol=1e-12)
