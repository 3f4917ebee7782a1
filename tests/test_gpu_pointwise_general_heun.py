"""General- and additive-noise Euler-Heun and reversible-Heun solves whose steps run as element-wise programs (GENERAL
launches of tsde_step_predictor_corrector_pointwise and tsde_solve_reversible_heun_pointwise; pointwise.py,
GeneralRecorder with the PW_LAYOUT_GENERAL_EULER_HEUN / _REVERSIBLE_HEUN tags).

Every fused solve must give the unfused solve's bits: the reference is the same solve with the tape rejected, and
TSDE_KERNEL_PW_GENERAL confirms the route (test_gpu_pointwise_general.check).  Covered, for both methods: m in
{1, 3, 4, 8, 16, 32} (row-wise, generic and tile orders), float32 and float64, correlated GBM, OU `expand`, a
time-dependent additive g and a torch.where / clamp g, d = 7, eager and graph solves, the chunk-boundary,
interpolated-output and final-only grids, multi-cell steps, TanhGeneral with the transcendental ops, and random
programs (tests/test_gpu_pointwise_fuzz.sweep).  Reversible Heun also: the final (f, g, z) of extra=True,
sdeint_adjoint's ys and gradients, the launch count of a cfg3-shaped plan and of a batch below one wave, and an fp64
solve against oracle/solvers.py on the oracle's increments.  And the solves that keep the unfused step."""
import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from oracle import solvers
from . import helpers, pointwise_fuzz as fz, problems
from .test_gpu_pointwise import same_bits
from .test_gpu_pointwise_chunks import DT, GRIDS
from .test_gpu_pointwise_fuzz import sweep
from .test_gpu_pointwise_general import SDE, Tanh, check, fused_launches
from .test_gpu_pointwise_pc import unfused

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
METHODS = ['euler_heun', 'reversible_heun']
CHUNK_LENGTH = pointwise.chunk_length


@pytest.fixture(autouse=True)
def full_chunks(monkeypatch):
    """Chunks of TSDE_PW_MAX_STEPS also for the small batches of these tests, except in the tests of that choice."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)


def make(kind, d, m, dtype):
    return SDE(kind, 'stratonovich', d, m, dtype).to(DEV)


@pytest.mark.parametrize('m', [1, 3, 4, 8, 16, 32])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_every_contraction_order_is_bit_identical(method, dtype, m):
    B, d = 96, 8
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    check(make('gbm', d, m, dtype), y0, GRIDS['not_a_multiple'].to(dtype=dtype, device=DEV), DT, method, m)


@pytest.mark.parametrize('m', [3, 4, 16])
@pytest.mark.parametrize('kind', ['gbm', 'ou', 'time_additive', 'where'])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('method', METHODS)
def test_kinds_eager_and_graph(method, mode, kind, m):
    B, d = 64, 7  # d not a multiple of 4
    y0 = torch.rand(B, d, dtype=torch.float32, device=DEV, generator=torch.Generator(DEV).manual_seed(1)) + 0.1
    options = {'cuda_graph': True} if mode == 'graph' else {}
    check(make(kind, d, m, torch.float32), y0, GRIDS['every_5'].to(DEV), DT, method, m, options)


@pytest.mark.parametrize('grid', ['K_plus_one', 'non_aligned', 'short_last_step', 'final_only'])
@pytest.mark.parametrize('method', METHODS)
def test_grids_chunk_boundaries_and_interpolated_outputs(method, grid):
    B, d, m = 80, 16, 8
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    check(make('gbm', d, m, torch.float64), y0, GRIDS[grid].to(dtype=torch.float64, device=DEV), DT, method, m,
          {'cuda_graph': True})


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', METHODS)
def test_steps_that_span_several_cells(method, dtype):
    B, d, m, T = 64, 8, 4, K + 10
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = (torch.arange(T + 1) * DT).to(dtype).to(DEV)
    check(make('time_additive', d, m, dtype), y0, ts, DT, method, m, bm_dt=DT / 2)


@pytest.mark.parametrize('method', METHODS)
def test_transcendental_general(method):
    B, d, m = 64, 8, 4
    sde = problems.TanhGeneral(d, m, 'stratonovich', dtype=torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.3, device=DEV)
    check(sde, y0, GRIDS['every_5'].to(DEV), DT, method, m, {'transcendental': True})


def _with_extra(sde, y0, ts, m, options=None):
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(y0.shape[0], m), dtype=y0.dtype, device=DEV, entropy=8)
    with torch.no_grad():
        out = tsde.sdeint(sde, y0, ts, bm=bm, method='reversible_heun', dt=DT, extra=True,
                          options=dict(options or {}))
    graph.drop_plans(sde)
    return out


@pytest.mark.parametrize('options', [{}, {'cuda_graph': True}])
def test_reversible_heun_final_solver_state(options):
    B, d, m = 64, 8, 16
    sde = make('where', d, m, torch.float32)
    y0 = torch.full((B, d), 0.3, device=DEV)
    ts = GRIDS['K_plus_one'].to(DEV)
    n0 = fused_launches()
    ys, (f, g, z) = _with_extra(sde, y0, ts, m, options)
    assert fused_launches() > n0 and tuple(g.shape) == (B, d, m)
    with unfused():
        ref_ys, ref = _with_extra(sde, y0, ts, m, options)
    assert same_bits(ys, ref_ys)
    for a, b in zip((f, g, z), ref):
        assert same_bits(a, b.contiguous())


def _adjoint(sde, y0, ts, m):
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(y0.shape[0], m), dtype=y0.dtype, device=DEV, entropy=21)
    y = y0.clone().requires_grad_(True)
    ys = tsde.sdeint_adjoint(sde, y, ts, bm=bm, method='reversible_heun', dt=DT)
    grads = torch.autograd.grad((ys * ys).sum(), [y] + list(sde.parameters()), allow_unused=True)
    graph.drop_plans(sde)
    return ys.detach(), grads


@pytest.mark.parametrize('kind', ['gbm', 'ou'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_sdeint_adjoint_forward_fuses_and_keeps_every_bit(kind, dtype):
    B, d, m = 64, 8, 4
    sde = make(kind, d, m, dtype)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = GRIDS['every_5'].to(dtype=dtype, device=DEV)
    n0 = fused_launches()
    ys, grads = _adjoint(sde, y0, ts, m)
    assert fused_launches() > n0, "the forward solve was not fused"
    with unfused():
        n1 = fused_launches()
        ref, ref_grads = _adjoint(sde, y0, ts, m)
        assert fused_launches() == n1
    assert same_bits(ys, ref)
    for a, b in zip(grads, ref_grads):
        assert (a is None) == (b is None)
        if a is not None:
            assert same_bits(a, b)


def test_cfg3_shaped_plan_launches_one_kernel_per_chunk(monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, m, T = 8192, 32, 16, 200
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(make('gbm', d, m, torch.float32), y0, ts, 2.0 ** -10, 'reversible_heun', m,
                    {'cuda_graph': True, 'static_output': False})
    # the recorded step runs before capture; the captured steps 0 .. T-1 are chunks
    assert plan.abi_launches == -(-T // K)


def test_a_batch_below_one_wave_runs_one_step_per_launch(monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, m, T = 1024, 64, 16, 50
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(make('gbm', d, m, torch.float32), y0, ts, 2.0 ** -10, 'reversible_heun', m,
                    {'cuda_graph': True, 'static_output': False})
    assert plan.abi_launches == T


@pytest.mark.parametrize('m', [1, 3, 4, 5, 16, 32])
@pytest.mark.parametrize('method', METHODS)
def test_random_programs(method, m):
    sweep('general_euler', [m, m + 40, m + 80], method, 'stratonovich', [_cabi.KERNEL_PW_GENERAL], m=m)


def test_fp64_reversible_heun_matches_the_oracle_on_its_increments():
    """As test_gpu_pointwise_fuzz's oracle comparison: a small case's fused fp64 solve against oracle/solvers.py on the
    oracle's increments of the same Brownian motion, at a sample of the rows."""
    B, d, m = 64, 5, 3
    seed = next(s for s in range(100) if not fz.case(s, 'general_euler', 'small', transcendental=False).transcendental
                and fz.case(s, 'general_euler', 'small', transcendental=False).f_out != 'y')
    case = fz.case(seed, 'general_euler', 'small', transcendental=False)
    sde = fz.FuzzSDE(case, 'stratonovich', B, d, m, torch.float64, DEV)
    gen = torch.Generator().manual_seed(seed)
    y0 = (torch.rand(B, d, generator=gen, dtype=torch.float64) - 0.5).to(DEV)
    ts = torch.tensor([0.0, 4 * DT, 8 * DT], dtype=torch.float64, device=DEV)
    bm = tsde.BrownianInterval(0.0, 8 * DT, size=(B, m), dtype=torch.float64, device=DEV, entropy=404)
    n0 = fused_launches()
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='reversible_heun', dt=DT)
    assert fused_launches() > n0, f'{case!r} was not fused'
    cpu = fz.FuzzSDE(case, 'stratonovich', B, d, m, torch.float64, 'cpu')
    ref, _ = solvers.make('reversible_heun', problems.NumpySDE(cpu),
                          helpers.oracle_grid_bm(bm, np.arange(B), m, np.float64, False), DT).integrate(
        y0.cpu().numpy(), ts.cpu().numpy())
    got = ys.cpu().numpy()
    rows = np.arange(0, B, 5)
    assert np.isfinite(got).all() and np.abs(got[-1] - got[0]).max() > 1e-3
    np.testing.assert_allclose(got[:, rows], ref[:, rows], rtol=1e-9, atol=1e-9, err_msg=f'{case!r}\n{case.source()}')


class GProd(SDE):
    def g_prod(self, t, y, v):
        return (y.unsqueeze(-1) * self.S * v.unsqueeze(1)).sum(-1)


@pytest.mark.parametrize('case', ['grad', 'adaptive', 'g_prod', 'overlap', 'autocast', 'wide', 'subnormal_half',
                                  'tanh'])
@pytest.mark.parametrize('method', METHODS)
def test_solves_that_keep_the_unfused_step(method, case, monkeypatch):
    """No general launch, and the unfused bits: gradients through the solve, an adaptive solve, a user g_prod,
    overlap=False, autocast, m past TSDE_PW_GENERAL_MAX_M, a step whose kernel half step T(0.5) * T(dt) would differ
    from the unfused half_dt (subnormal; reversible Heun), and a transcendental op without the option."""
    B, d, m = 32, 8, 40 if case == 'wide' else 4
    if case == 'adaptive' and method == 'reversible_heun':
        pytest.skip('reversible Heun has no adaptive solve')
    if case == 'subnormal_half':
        if method != 'reversible_heun':
            pytest.skip('only reversible Heun halves dt in the kernel')
        monkeypatch.setattr(pointwise, 'halves_exactly', lambda dtype, ctxs: False)
    cls = GProd if case == 'g_prod' else Tanh if case == 'tanh' else SDE
    sde = cls('gbm', 'stratonovich', d, m, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.3, device=DEV, requires_grad=case == 'grad')
    dt, options = 2.0 ** -5, {}
    if case == 'overlap':
        options['overlap'] = False
    ts = torch.tensor([0.0, 0.25, 0.5], device=DEV)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), device=DEV, entropy=3)
        with torch.set_grad_enabled(case == 'grad'), torch.autocast('cuda', enabled=case == 'autocast'):
            ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, adaptive=case == 'adaptive',
                             options=dict(options))
        graph.drop_plans(sde)
        return ys.detach()
    n0 = fused_launches()
    ys = solve()
    assert fused_launches() == n0
    with unfused():
        ref = solve()
    assert torch.isfinite(ys).all() and same_bits(ys, ref)
