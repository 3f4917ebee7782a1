"""Euler and reversible-Heun solves whose steps run as element-wise programs, several per kernel
(tsde_solve_euler_pointwise, tsde_solve_reversible_heun_pointwise; torchsde_b200/_core/pointwise.py).

Every fused solve must give the unfused solve's bits: ys, and for reversible Heun the final solver state (f, g, z).
The unfused reference is the same solve with the tape rejected (SrkRecorder.finish patched to return None); the route
is confirmed by the launch counter TSDE_KERNEL_PW_CHUNK.  Covered, for both methods: float32 and float64; eager, graph
and row_split (reversible Heun carries a solver state and so runs a graph without row blocks); the grids of
tests/test_gpu_pointwise_chunks.py; multi-cell steps; d = 7 and a misaligned parameter; shards past row 2^24; a
time-dependent drift; in-place parameter updates between replays; user-supplied solver state, left unmodified;
backward-in-time solves on a ReverseBrownian; `sdeint_adjoint` with the reversible pair, eager and captured; the launch
count of a cfg2-shaped plan and of a batch below one wave; and the solves that keep the unfused step."""
import contextlib

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from .test_gpu_pointwise import MODES, SDE, Nonlinear, same_bits
from .test_gpu_pointwise_chunks import DT, GRIDS
from .test_gpu_pointwise_pc import TimeSDE, unfused
from .test_gpu_pointwise_srk import Unbound

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
METHODS = ['euler', 'reversible_heun']
SDE_TYPE = {'euler': 'ito', 'reversible_heun': 'stratonovich'}
CHUNK_LENGTH = pointwise.chunk_length


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_CHUNK)


@pytest.fixture(autouse=True)
def full_chunks(monkeypatch):
    """Chunks of TSDE_PW_MAX_STEPS also for the small batches of these tests (which the solver runs one step per
    launch: pointwise.chunk_length), except in the tests of that choice."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)


def make_sde(kind, method, B, d, dtype):
    if kind == 'time2':
        sde = TimeSDE(B, d, dtype)
        sde.sde_type = SDE_TYPE[method]
        return sde.to(DEV)
    return SDE(kind, SDE_TYPE[method], B, d, dtype).to(DEV)


def run(sde, y0, ts, dt, method, options=None, row_offset=0, bm_dt=None, entropy=5, **kw):
    B, m = y0.shape
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy, dt=bm_dt)
    if row_offset:
        bm.shard_rows(row_offset)
    with torch.no_grad():
        out = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options or {}), extra=True, **kw)
    plan = graph.LAST_PLAN
    graph.drop_plans(sde)
    ys, extra = out
    return [ys, *extra], plan


def check(sde, y0, ts, dt, method, options=None, **kw):
    """The fused solve (at least one chunk launch) and the unfused one (none) give the same ys and final state."""
    n0 = fused_launches()
    out, plan = run(sde, y0, ts, dt, method, options, **kw)
    assert fused_launches() > n0, "the steps were not fused"
    with unfused():
        n1 = fused_launches()
        ref, _ = run(sde, y0, ts, dt, method, options, **kw)
        assert fused_launches() == n1
    assert len(out) == len(ref) == (4 if method == 'reversible_heun' else 1)
    for a, b in zip(out, ref):
        assert same_bits(a, b)
    return out, plan


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('grid', sorted(GRIDS))
@pytest.mark.parametrize('method', METHODS)
def test_chunked_solves_are_bit_identical(method, grid, dtype, mode):
    B, d = 96, 16
    sde = make_sde('gbm', method, B, d, dtype)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    check(sde, y0, GRIDS[grid].to(dtype=dtype, device=DEV), DT, method, MODES[mode])


@pytest.mark.parametrize('kind', ['time2', 'div', 'in_place', 'ou', 'square'])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('method', METHODS)
def test_kinds_over_chunk_boundaries(method, mode, kind):
    B, d = 64, 8
    sde = make_sde(kind, method, B, d, torch.float32)
    y0 = torch.full((B, d), 0.3, device=DEV)
    check(sde, y0, GRIDS['not_a_multiple'].to(DEV), DT, method, MODES[mode])


@pytest.mark.parametrize('method', METHODS)
def test_the_program_runs_at_the_steps_time(method):
    """Euler evaluates f and g at t0, reversible Heun at t1: moving the drift's time moves the bits, and the fused solve
    still equals the unfused one."""
    B, d = 32, 8
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    ts = GRIDS['K_plus_one'].to(dtype=torch.float64, device=DEV)
    a, _ = check(make_sde('time2', method, B, d, torch.float64), y0, ts, DT, method)
    shifted = make_sde('time2', method, B, d, torch.float64)
    shifted.f = lambda t, y: ((t + DT / 4) * shifted.mu) * y
    b, _ = check(shifted, y0, ts, DT, method)
    assert not torch.equal(a[0], b[0])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_steps_that_span_several_cells_run_alone(method, dtype):
    B, d, T = 64, 8, K + 10
    sde = make_sde('time2', method, B, d, dtype)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = (torch.arange(T + 1) * DT).to(dtype).to(DEV)
    check(sde, y0, ts, DT, method, MODES['eager'], bm_dt=DT / 2)
    _, plan = check(sde, y0, ts, DT, method, MODES['graph'], bm_dt=DT / 2)
    assert plan.abi_launches == T


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_element_path_odd_width_and_misaligned_parameter(method, dtype):
    B = 50
    ts = GRIDS['non_aligned'].to(dtype=dtype, device=DEV)
    check(make_sde('div', method, B, 7, dtype), torch.full((B, 7), 0.4, dtype=dtype, device=DEV), ts, DT, method,
          {'cuda_graph': True})
    sde = make_sde('gbm', method, B, 8, dtype)
    with torch.no_grad():
        store = torch.zeros(9, dtype=dtype, device=DEV)
        store[1:].copy_(sde.sigma)
        sde.sigma = nn.Parameter(store[1:])
    assert sde.sigma.data_ptr() % 16
    check(sde, torch.full((B, 8), 0.4, dtype=dtype, device=DEV), ts, DT, method)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_shards_past_row_2_24(method, dtype):
    B, d = 300, 12
    sde = make_sde('gbm', method, B, d, dtype)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = GRIDS['every_5'].to(dtype=dtype, device=DEV)
    ys, _ = check(sde, y0, ts, DT, method, {'cuda_graph': True}, row_offset=(1 << 24) + 5)
    other, _ = check(sde, y0, ts, DT, method, {'cuda_graph': True}, row_offset=(1 << 24) + 6)
    assert not torch.equal(ys[0][-1], other[0][-1])


@pytest.mark.parametrize('method', METHODS)
def test_in_place_parameter_update_between_replays_is_followed(method):
    B, d = 64, 8
    sde = make_sde('time2', method, B, d, torch.float32)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = GRIDS['not_a_multiple'].to(DEV)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), device=DEV, entropy=3)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=DT, options={'cuda_graph': True})

    first = solve()
    with torch.no_grad():
        sde.sigma.mul_(1.5)
        sde.mu.add_(0.25)
    second = solve()                # a replay of the same plan
    graph.drop_plans(sde)
    with unfused():
        want = solve()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_a_user_supplied_solver_state_is_read_and_left_alone(dtype, mode):
    B, d = 64, 8
    sde = make_sde('gbm', 'reversible_heun', B, d, dtype)
    gen = torch.Generator(device=DEV).manual_seed(1)
    state = tuple(torch.rand((B, d), generator=gen, dtype=dtype, device=DEV) for _ in range(3))
    kept = tuple(x.clone() for x in state)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    out, _ = check(sde, y0, GRIDS['K_plus_one'].to(dtype=dtype, device=DEV), DT, 'reversible_heun', MODES[mode],
                   extra_solver_state=state)
    assert all(torch.equal(a, b) for a, b in zip(state, kept))
    assert not any(x.data_ptr() in {s.data_ptr() for s in state} for x in out[1:])


class Backward(nn.Module):
    """The SDE of a solve backwards in time (tests/test_gpu_adjoint.py::test_reversibility), with f and g separate."""
    noise_type, sde_type = 'diagonal', 'stratonovich'

    def __init__(self, sde):
        super().__init__()
        self.sde = sde

    def f(self, t, y):
        return -self.sde.f(-t, y)

    def g(self, t, y):
        return -self.sde.g(-t, y)


@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_backward_in_time_on_a_reverse_brownian(mode):
    B, d, dt = 64, 8, 2.0 ** -5
    fwd = make_sde('time2', 'reversible_heun', B, d, torch.float64)
    sde = Backward(fwd)
    ts = -(torch.arange(2 * K + 4, dtype=torch.float64, device=DEV) * dt).flip(0)
    y0 = torch.full((B, d), 0.3, dtype=torch.float64, device=DEV)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(-ts[0]), size=(B, d), dtype=torch.float64, device=DEV, entropy=8)
        with torch.no_grad():
            ys, extra = tsde.sdeint(sde, y0, ts, bm=tsde.ReverseBrownian(bm), method='reversible_heun', dt=dt,
                                    extra=True, options=MODES[mode])
        graph.drop_plans(sde)
        return [ys, *extra]

    n0 = fused_launches()
    out = solve()
    assert fused_launches() > n0
    with unfused():
        ref = solve()
    assert all(same_bits(a, b) for a, b in zip(out, ref))


@pytest.mark.parametrize('graphs', [False, True])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_sdeint_adjoint_with_the_reversible_pair(dtype, graphs):
    """`sdeint_adjoint`'s forward solve is a no-grad reversible-Heun solve and fuses; its backward sweep does not.
    ys, y0's gradient and every parameter's gradient equal those of the same solve with the tape rejected."""
    B, d = 64, 8
    ts = GRIDS['not_a_multiple'].to(dtype=dtype, device=DEV)
    opts = {'options': {'cuda_graph': True}, 'adjoint_options': {'cuda_graph': True}} if graphs else {}
    out = []
    for ctx in (contextlib.nullcontext, unfused):
        with ctx():
            sde = make_sde('time2', 'reversible_heun', B, d, dtype)
            y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV, requires_grad=True)
            bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), dtype=dtype, device=DEV, entropy=9)
            n0 = fused_launches()
            ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=DT, **opts)
            n1 = fused_launches()
            ys.pow(2).sum().backward()
            assert fused_launches() == n1
            assert (n1 > n0) == (ctx is contextlib.nullcontext)
            out.append([ys.detach(), y0.grad] + [p.grad for p in sde.parameters()])
            graph.drop_plans(sde)
    assert out[0][1] is not None
    for a, b in zip(*out):
        assert (a is None) == (b is None) and (a is None or same_bits(a, b))


@pytest.mark.parametrize('method', METHODS)
def test_cfg2_shaped_plan_launches_one_kernel_per_chunk(method, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, T = 65536, 64, 200
    sde = make_sde('gbm', method, B, d, torch.float32)
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(sde, y0, ts, 2.0 ** -10, method, {'cuda_graph': True, 'static_output': False})
    # the recorded step runs before capture; the captured steps 0 .. T-1 are chunks, and reversible Heun's z kernel
    # and final kernel of the recorded step are not part of the plan
    assert plan.abi_launches == -(-T // K)


@pytest.mark.parametrize('method', METHODS)
def test_a_batch_below_one_wave_runs_one_step_per_launch(method, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, T = 2048, 64, 100
    sde = make_sde('gbm', method, B, d, torch.float32)
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(sde, y0, ts, 2.0 ** -10, method, {'cuda_graph': True, 'static_output': False})
    assert plan.abi_launches == T


FALLBACKS = ['sigmoid', 'exp', 'item', 'f_and_g', 'g_prod', 'scalar', 'additive', 'general', 'grad', 'logqp',
             'autocast', 'overlap', 'unbound']


@pytest.mark.parametrize('case', FALLBACKS)
@pytest.mark.parametrize('method', METHODS)
def test_unfusable_solves_keep_the_unfused_step(method, case):
    B, d, T, dt = 32, 8, 6, 2.0 ** -5
    sde = Nonlinear(case, B, d).to(DEV)
    sde.sde_type = SDE_TYPE[method]
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * dt
    kw, ctx, m = {}, contextlib.nullcontext, d
    if case == 'logqp':
        kw['logqp'], m = True, d + 1
    if case == 'autocast':
        ctx = lambda: torch.autocast('cuda', dtype=torch.bfloat16)  # noqa: E731
    if case == 'overlap':
        kw['options'] = {'overlap': False}
    if case == 'f_and_g':
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


@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_a_subnormal_half_step_keeps_the_unfused_step(mode, monkeypatch):
    """A solve where one step's T(0.5) * T(dt) differs from the unfused step's half_dt is not fused at all."""
    monkeypatch.setattr(pointwise, 'halves_exactly', lambda dtype, ctxs: False)
    B, d = 64, 8
    sde = make_sde('gbm', 'reversible_heun', B, d, torch.float32)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = GRIDS['K_plus_one'].to(DEV)
    n0 = fused_launches()
    out, _ = run(sde, y0, ts, DT, 'reversible_heun', MODES[mode])
    assert fused_launches() == n0
    with unfused():
        ref, _ = run(sde, y0, ts, DT, 'reversible_heun', MODES[mode])
    assert all(same_bits(a, b) for a, b in zip(out, ref))
