"""General- and additive-noise Euler and midpoint solves whose steps run as element-wise programs
(tsde_solve_euler_general_pointwise, tsde_step_midpoint_general_pointwise; torchsde_b200/_core/pointwise.py,
GeneralRecorder).

Every fused solve must give the unfused solve's bits.  The unfused reference is the same solve with the tape rejected
(SrkRecorder.finish patched to return None, which GeneralRecorder inherits); the route is confirmed by the launch
counter TSDE_KERNEL_PW_GENERAL.  Covered: Euler (Ito) and midpoint (Stratonovich); float32 and float64; correlated
GBM, OU with an additive `expand`, a time-dependent additive g and a torch.where / clamp g; m in {1, 3, 4, 8, 16, 32},
which takes the row-wise, generic and tile contraction orders; d = 7; eager and graph solves, chunk boundaries,
interpolated outputs, multi-cell steps; the launch count of a cfg3-shaped plan and of a batch below one wave; and
the solves that keep the unfused step."""
import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from .test_gpu_pointwise import same_bits
from .test_gpu_pointwise_chunks import DT, GRIDS
from .test_gpu_pointwise_pc import unfused

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
SDE_TYPE = {'euler': 'ito', 'midpoint': 'stratonovich'}
CHUNK_LENGTH = pointwise.chunk_length


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL)


@pytest.fixture(autouse=True)
def full_chunks(monkeypatch):
    """Chunks of TSDE_PW_MAX_STEPS also for the small batches of these tests, except in the tests of that choice."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)


class SDE(nn.Module):
    def __init__(self, kind, sde_type, d, m, dtype, seed=0):
        super().__init__()
        self.kind, self.sde_type = kind, sde_type
        self.noise_type = 'additive' if kind in ('ou', 'time_additive') else 'general'
        gen = torch.Generator().manual_seed(seed)

        def param(*shape, lo=0.1, hi=0.6):
            return nn.Parameter((torch.rand(shape, generator=gen, dtype=torch.float64) * (hi - lo) + lo).to(dtype))
        self.mu, self.b = param(d, lo=-0.5, hi=0.5), param(d)
        self.S, self.a = param(d, m), param(d, m)

    def f(self, t, y):
        if self.kind == 'ou':
            return self.mu - y
        if self.kind == 'time_additive':
            return self.b / torch.sqrt(1. + t) - y / (2. + 2. * t)
        return self.mu * y

    def g(self, t, y):
        B = y.size(0)
        if self.kind == 'gbm':  # correlated multi-asset GBM
            return y.unsqueeze(-1) * self.S
        if self.kind == 'ou':
            return self.S.expand(B, *self.S.shape)
        if self.kind == 'time_additive':
            return (self.a * (self.b / torch.sqrt(1. + t)).unsqueeze(-1)).unsqueeze(0).expand(B, -1, -1)
        if self.kind == 'where':
            yy = y[..., None]
            return torch.where(yy > 0.25, yy * self.S, torch.clamp(self.a, 0.2, 0.4))
        raise ValueError(self.kind)


def run(sde, y0, ts, dt, method, m, options=None, bm_dt=None, entropy=5):
    B = y0.shape[0]
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy, dt=bm_dt)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options or {}))
    plan = graph.LAST_PLAN
    graph.drop_plans(sde)
    return ys, plan


def check(sde, y0, ts, dt, method, m, options=None, **kw):
    """The fused solve (at least one general launch) and the unfused one (none) give the same ys."""
    n0 = fused_launches()
    out, plan = run(sde, y0, ts, dt, method, m, options, **kw)
    assert fused_launches() > n0, "the steps were not fused"
    with unfused():
        n1 = fused_launches()
        ref, _ = run(sde, y0, ts, dt, method, m, options, **kw)
        assert fused_launches() == n1
    assert same_bits(out, ref)
    return out, plan


def make(kind, method, d, m, dtype):
    return SDE(kind, SDE_TYPE[method], d, m, dtype).to(DEV)


@pytest.mark.parametrize('m', [1, 3, 4, 8, 16, 32])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', ['euler', 'midpoint'])
def test_every_contraction_order_is_bit_identical(method, dtype, m):
    B, d = 96, 8
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    check(make('gbm', method, d, m, dtype), y0, GRIDS['not_a_multiple'].to(dtype=dtype, device=DEV), DT, method, m)


@pytest.mark.parametrize('m', [3, 4, 16])
@pytest.mark.parametrize('kind', ['gbm', 'ou', 'time_additive', 'where'])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('method', ['euler', 'midpoint'])
def test_kinds_eager_and_graph(method, mode, kind, m):
    B, d = 64, 7  # d not a multiple of 4
    y0 = torch.rand(B, d, dtype=torch.float32, device=DEV, generator=torch.Generator(DEV).manual_seed(1)) + 0.1
    options = {'cuda_graph': True} if mode == 'graph' else {}
    check(make(kind, method, d, m, torch.float32), y0, GRIDS['every_5'].to(DEV), DT, method, m, options)


@pytest.mark.parametrize('grid', ['K_plus_one', 'non_aligned', 'short_last_step', 'final_only'])
@pytest.mark.parametrize('method', ['euler', 'midpoint'])
def test_grids_chunk_boundaries_and_interpolated_outputs(method, grid):
    B, d, m = 80, 16, 8
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    check(make('gbm', method, d, m, torch.float64), y0, GRIDS[grid].to(dtype=torch.float64, device=DEV), DT, method,
          m, {'cuda_graph': True})


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', ['euler', 'midpoint'])
def test_steps_that_span_several_cells(method, dtype):
    B, d, m, T = 64, 8, 4, K + 10
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = (torch.arange(T + 1) * DT).to(dtype).to(DEV)
    check(make('time_additive', method, d, m, dtype), y0, ts, DT, method, m, bm_dt=DT / 2)


def test_cfg3_shaped_plan_launches_one_kernel_per_chunk(monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, m, T = 8192, 32, 16, 200
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(make('gbm', 'euler', d, m, torch.float32), y0, ts, 2.0 ** -10, 'euler', m,
                    {'cuda_graph': True, 'static_output': False})
    # the recorded step runs before capture; the captured steps 0 .. T-1 are chunks
    assert plan.abi_launches == -(-T // K)


def test_a_batch_below_one_wave_runs_one_step_per_launch(monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, m, T = 2048, 64, 16, 50
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(make('gbm', 'euler', d, m, torch.float32), y0, ts, 2.0 ** -10, 'euler', m,
                    {'cuda_graph': True, 'static_output': False})
    assert plan.abi_launches == T


class Tanh(SDE):
    def g(self, t, y):
        return torch.tanh(y).unsqueeze(-1) * self.S


@pytest.mark.parametrize('case', ['tanh', 'wide', 'heun', 'adaptive', 'grad'])
def test_solves_that_keep_the_unfused_step(case):
    """No general launch where fusion is not expected: an op outside the set, m past TSDE_PW_GENERAL_MAX_M, a method
    other than Euler and midpoint, an adaptive solve, gradients through the solve."""
    B, d, m = 32, 8, 4
    method = 'heun' if case == 'heun' else 'euler'
    sde_type = 'stratonovich' if case == 'heun' else 'ito'
    if case == 'tanh':
        sde = Tanh('gbm', sde_type, d, m, torch.float32).to(DEV)
    else:
        m = 40 if case == 'wide' else m
        sde = SDE('gbm', sde_type, d, m, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.3, device=DEV, requires_grad=case == 'grad')
    ts = torch.tensor([0.0, 0.25, 0.5], device=DEV)
    bm = tsde.BrownianInterval(0.0, 0.5, size=(B, m), device=DEV, entropy=3)
    n0 = fused_launches()
    with torch.set_grad_enabled(case == 'grad'):
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -5, adaptive=case == 'adaptive')
    assert fused_launches() == n0
    assert torch.isfinite(ys).all()
