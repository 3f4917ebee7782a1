"""Additive-noise SRK (sra1) solves whose steps run as one kernel each (a GENERAL launch of
tsde_step_srk_diag_pointwise; torchsde_b200/_core/pointwise.py, GeneralRecorder with the 'fggf' pattern).

Every fused solve must give the unfused solve's bits.  The unfused reference is the same solve with the tape rejected
(`unfused()`, SrkRecorder.finish patched to return None, which GeneralRecorder inherits); the route is confirmed by
the launch counter TSDE_KERNEL_PW_GENERAL.  Covered: m in {1, 3, 4, 8, 16, 32} (generic order at m = 1 and 3, the
tile order otherwise), float32 and float64; an OU `S.expand`, the time-additive g and a torch.where / clamp g in which
f and g read t; d = 7 and a misaligned (d, m) operand; eager and graph solves; the three Levy approximations;
multi-cell steps and interpolated outputs; shards past global row 2^24; an in-place parameter update between graph
replays; the launch count of a cfg3-shaped plan; the solves that keep the unfused step; and one fp64 solve against
the numpy oracle's SRK on the oracle's increments."""
import contextlib

import numpy as np
import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph
from oracle import solvers
from . import helpers, problems
from .test_gpu_pointwise import same_bits
from .test_gpu_pointwise_chunks import DT as CHUNK_DT, GRIDS
from .test_gpu_pointwise_srk import unfused

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DT = 2.0 ** -5


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL)


class SDE(nn.Module):
    noise_type, sde_type = 'additive', 'ito'

    def __init__(self, kind, d, m, dtype, seed=0):
        super().__init__()
        self.kind = kind
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
        return (t * self.mu) * y - y  # 'where': f reads t too

    def g(self, t, y):
        B = y.size(0)
        if self.kind == 'ou':
            return self.S.expand(B, *self.S.shape)
        if self.kind == 'time_additive':
            return (self.a * (self.b / torch.sqrt(1. + t)).unsqueeze(-1)).unsqueeze(0).expand(B, -1, -1)
        if self.kind == 'where':  # per-channel selection on t and y: a stage time in the wrong slot changes the bits
            yy = y[..., None]
            return torch.where(yy > 0.25 + t, (t + 0.5) * self.S, torch.clamp(self.a * t, 0.02, 0.3))
        raise ValueError(self.kind)


def make(kind, d, m, dtype=torch.float32):
    return SDE(kind, d, m, dtype).to(DEV)


def run(sde, y0, ts, dt, m, options=None, levy='space-time', bm_dt=None, row_offset=0, entropy=5):
    B = y0.shape[0]
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy,
                               levy_area_approximation=levy, dt=bm_dt)
    if row_offset:
        bm.shard_rows(row_offset)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='srk', dt=dt, options=dict(options or {}))
    plan = graph.LAST_PLAN
    graph.drop_plans(sde)
    return ys, plan


def check(sde, y0, ts, dt, m, options=None, **kw):
    """The fused solve (at least one sra1 launch) and the unfused one (none) give the same ys."""
    n0 = fused_launches()
    out, plan = run(sde, y0, ts, dt, m, options, **kw)
    assert fused_launches() > n0, "the steps were not fused"
    with unfused():
        n1 = fused_launches()
        ref, _ = run(sde, y0, ts, dt, m, options, **kw)
        assert fused_launches() == n1
    assert same_bits(out, ref)
    return out, plan


def grid(T, dtype=torch.float32):
    return (torch.arange(T + 1) * DT).to(dtype).to(DEV)


@pytest.mark.parametrize('m', [1, 3, 4, 8, 16, 32])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_every_contraction_order_is_bit_identical(dtype, m):
    B, d = 96, 8
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    check(make('where', d, m, dtype), y0, grid(9, dtype), DT, m)


@pytest.mark.parametrize('m', [1, 3, 4, 16])
@pytest.mark.parametrize('kind', ['ou', 'time_additive', 'where'])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_kinds_eager_and_graph(mode, kind, m):
    B, d = 64, 7  # d not a multiple of 4
    y0 = torch.rand(B, d, dtype=torch.float32, device=DEV, generator=torch.Generator(DEV).manual_seed(1)) + 0.1
    options = {'cuda_graph': True} if mode == 'graph' else {}
    check(make(kind, d, m), y0, grid(7), DT, m, options)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', [4, 16])
def test_a_misaligned_dm_operand(m, dtype):
    """g is the user's (d, m) block at an address that is not 16-byte aligned: the unfused launches take gen_kernel's
    order, and so must the fused one."""
    B, d = 40, 8
    sde = make('ou', d, m, dtype)
    with torch.no_grad():
        store = torch.zeros(d * m + 1, dtype=dtype, device=DEV)
        store[1:].copy_(sde.S.reshape(-1))
        sde.S = nn.Parameter(store[1:].view(d, m))
    assert sde.S.data_ptr() % 16
    check(sde, torch.full((B, d), 0.4, dtype=dtype, device=DEV), grid(5, dtype), DT, m, {'cuda_graph': True})


@pytest.mark.parametrize('levy', ['space-time', 'davie', 'foster'])
@pytest.mark.parametrize('cells', [1, 2])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_levy_approximations_and_multi_cell_steps(dtype, cells, levy):
    B, d, m = 48, 8, 4
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    check(make('where', d, m, dtype), y0, grid(6, dtype), DT, m, levy=levy, bm_dt=DT / cells if cells > 1 else None)


@pytest.mark.parametrize('grid_name', ['non_aligned', 'short_last_step'])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_interpolated_outputs(mode, grid_name):
    B, d, m = 80, 16, 8
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    options = {'cuda_graph': True} if mode == 'graph' else {}
    check(make('time_additive', d, m, torch.float64), y0, GRIDS[grid_name].to(dtype=torch.float64, device=DEV),
          CHUNK_DT, m, options)


def test_stage_times_matter():
    """The time-dependent SDE's solution moves when a stage time does: a wrong slot would show in the bits."""
    B, d, m = 32, 8, 4
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=DEV)
    a, _ = check(make('where', d, m, torch.float64), y0, grid(4, torch.float64), DT, m)
    shifted = make('where', d, m, torch.float64)
    g = shifted.g
    shifted.g = lambda t, y: g(t + DT / 4, y)  # g read at a later time
    b, _ = check(shifted, y0, grid(4, torch.float64), DT, m)
    assert not torch.equal(a, b)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_shards_past_row_2_24(mode, dtype):
    B, d, m = 300, 12, 3
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    options = {'cuda_graph': True} if mode == 'graph' else {}
    ys, _ = check(make('ou', d, m, dtype), y0, grid(6, dtype), DT, m, options, row_offset=(1 << 24) + 5)
    other, _ = check(make('ou', d, m, dtype), y0, grid(6, dtype), DT, m, options, row_offset=(1 << 24) + 6)
    assert not torch.equal(ys[-1], other[-1])


def test_in_place_parameter_update_between_replays_is_followed():
    B, d, m = 64, 8, 4
    sde = make('where', d, m)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = grid(4)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), device=DEV, entropy=3,
                                   levy_area_approximation='space-time')
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method='srk', dt=DT, options={'cuda_graph': True})

    n0 = fused_launches()
    first = solve()
    with torch.no_grad():
        sde.S.mul_(1.5)
        sde.mu.add_(0.25)
    second = solve()                # a replay of the same plan
    assert fused_launches() > n0
    graph.drop_plans(sde)
    with unfused():
        want = solve()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


def test_cfg3_shaped_plan_launches_one_kernel_per_step():
    B, d, m, T = 8192, 32, 16, 100
    sde = problems.make('additive_expand', d, m, 'ito', dtype=torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(sde, y0, ts, 2.0 ** -10, m, {'cuda_graph': True, 'static_output': False})
    # the recorded step runs before capture; every captured step is one launch
    assert plan.abi_launches == T


class Repeat(SDE):
    def g(self, t, y):
        return self.S.unsqueeze(0).repeat(y.size(0), 1, 1)


FALLBACKS = ['wide', 'adaptive', 'grad', 'g_prod', 'overlap', 'autocast', 'repeat']


@pytest.mark.parametrize('case', FALLBACKS)
def test_solves_that_keep_the_unfused_step(case):
    """No sra1 launch where fusion is not expected, and the same bits as the solve with the tape rejected."""
    B, d, m, T = 32, 8, 40 if case == 'wide' else 4, 6
    sde = (Repeat if case == 'repeat' else SDE)('ou', d, m, torch.float32).to(DEV)
    if case == 'g_prod':
        sde.g_prod = lambda t, y, v: (sde.g(t, y) @ v.unsqueeze(-1)).squeeze(-1)
    kw = {'adaptive': True} if case == 'adaptive' else {}
    if case == 'overlap':
        kw['options'] = {'overlap': False}
    ctx = (lambda: torch.autocast('cuda', dtype=torch.bfloat16)) if case == 'autocast' else contextlib.nullcontext
    y0 = torch.full((B, d), 0.3, device=DEV)
    ts = grid(T)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), device=DEV, entropy=3,
                                   levy_area_approximation='space-time')
        with (torch.enable_grad() if case == 'grad' else torch.no_grad()), ctx():
            y = y0.clone().requires_grad_(case == 'grad')
            out = tsde.sdeint(sde, y, ts, bm=bm, method='srk', dt=DT, **kw)
        return out.detach()

    n0 = fused_launches()
    out = solve()
    assert fused_launches() == n0
    graph.drop_plans(sde)
    with unfused():
        ref = solve()
    assert same_bits(out, ref)


def test_a_fused_solve_matches_the_oracle_on_its_increments():
    """sra1, float64, against oracle/solvers.py on the oracle's Philox increments (sampled rows)."""
    B, d, m, dt = 512, 8, 4, 2.0 ** -4
    sde = problems.make('additive_expand', d, m, 'ito', dtype=torch.float64, seed=3).to(DEV)
    y0 = torch.full((B, d), 0.5, dtype=torch.float64, device=DEV)
    ts = torch.tensor([0.0, 0.25, 0.5], dtype=torch.float64, device=DEV)
    bm = tsde.BrownianInterval(0.0, 0.5, size=(B, m), dtype=torch.float64, device=DEV, entropy=404,
                               levy_area_approximation='space-time')
    n0 = fused_launches()
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='srk', dt=dt)
    assert fused_launches() > n0
    rows = np.arange(0, B, 7)
    sde_cpu = problems.make('additive_expand', d, m, 'ito', dtype=torch.float64, seed=3)
    ref, _ = solvers.make('srk', problems.NumpySDE(sde_cpu), helpers.oracle_grid_bm(bm, rows, m, np.float64, True),
                          dt).integrate(y0[torch.from_numpy(rows).to(DEV)].cpu().numpy(), ts.cpu().numpy())
    np.testing.assert_allclose(ys[:, torch.from_numpy(rows).to(DEV)].cpu().numpy(), ref, rtol=1e-9, atol=1e-12)
