"""Element-wise Milstein solves whose steps run several per kernel (tsde_solve_milstein_pointwise, pointwise.plan_chunks)
give the unfused solve's bits: chunks longer than, equal to and shorter than TSDE_PW_MAX_STEPS, outputs every few
steps, non-aligned outputs, a short last step, a multi-cell step in the middle, eager / graph / row_split, float32 and
float64, d % 4 != 0 with a misaligned parameter, shards past row 2^24, a time-dependent drift, in-place parameter
updates between replays and per-trajectory parameters.  A captured cfg2-shaped plan issues one launch per chunk."""
import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise

from .test_gpu_pointwise import SDE, MODES, fused_launches, same_bits, unfused

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
CHUNK_LENGTH = pointwise.chunk_length


@pytest.fixture(autouse=True)
def full_chunks(monkeypatch):
    """Chunks of TSDE_PW_MAX_STEPS also for the small batches of these tests (which the solver runs one step per
    launch: pointwise.chunk_length), except in the test of that choice."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)


def run(sde, y0, ts, dt, options=None, row_offset=0, bm_dt=None):
    B, m = y0.shape
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=y0.dtype, device=DEV, entropy=5, dt=bm_dt)
    if row_offset:
        bm.shard_rows(row_offset)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=dt, options=dict(options or {}))
    plan = graph.LAST_PLAN
    graph.drop_plans(sde)
    return ys, plan


def check(sde, y0, ts, dt, options=None, row_offset=0, bm_dt=None):
    n0 = fused_launches()
    ys, plan = run(sde, y0, ts, dt, options, row_offset, bm_dt)
    assert fused_launches() > n0, "the steps were not fused"
    with unfused():
        ref, _ = run(sde, y0, ts, dt, options, row_offset, bm_dt)
    assert same_bits(ys, ref)
    return ys, plan


DT = 2.0 ** -7
GRIDS = {
    'below_K': torch.arange(K // 2 + 1) * DT,
    'K_plus_one': torch.arange(K + 2) * DT,           # the recorded step, then exactly K
    'not_a_multiple': torch.arange(2 * K + 12) * DT,
    'every_5': torch.arange(0, 3 * K + 1, 5) * DT,
    'final_only': torch.tensor([0.0, (2 * K + 3) * DT]),
    'non_aligned': torch.tensor([0.0, 2.5, 3.25, 70.1, 150.0]) * DT,
    'short_last_step': torch.tensor([0.0, (K + 20.4) * DT]),
}


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('grid', sorted(GRIDS))
def test_chunked_solves_are_bit_identical(grid, dtype, mode):
    B, d = 96, 16
    sde = SDE('gbm', 'ito', B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    check(sde, y0, GRIDS[grid].to(dtype=dtype, device=DEV), DT, MODES[mode])


@pytest.mark.parametrize('kind,sde_type', [('time', 'ito'), ('pertraj', 'stratonovich'), ('ou', 'ito'),
                                           ('square', 'ito'), ('div', 'stratonovich')])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_kinds_over_chunk_boundaries(kind, sde_type, mode):
    B, d = 64, 8
    sde = SDE(kind, sde_type, B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.3, device=DEV)
    check(sde, y0, GRIDS['not_a_multiple'].to(DEV), DT, MODES[mode])


def test_steps_that_span_several_cells_run_alone():
    # a Brownian grid twice as fine as the solver's: every step merges two cells, so every step is a launch of its own
    # (the planner's CPU test puts one such step between chunks)
    B, d, T = 64, 8, K + 10
    sde = SDE('gbm', 'stratonovich', B, d, torch.float64).to(DEV)
    y0 = torch.full((B, d), 0.3, dtype=torch.float64, device=DEV)
    ts = (torch.arange(T + 1) * DT).to(torch.float64).to(DEV)
    check(sde, y0, ts, DT, MODES['eager'], bm_dt=DT / 2)
    _, plan = check(sde, y0, ts, DT, MODES['graph'], bm_dt=DT / 2)
    assert plan.abi_launches == T


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_element_path_odd_width_and_misaligned_parameter(dtype):
    B = 50
    ts = GRIDS['non_aligned'].to(dtype=dtype, device=DEV)
    check(SDE('ou', 'ito', B, 7, dtype).to(DEV), torch.full((B, 7), 0.4, dtype=dtype, device=DEV), ts, DT,
          {'cuda_graph': True})
    sde = SDE('gbm', 'ito', B, 8, dtype).to(DEV)
    with torch.no_grad():
        store = torch.zeros(9, dtype=dtype, device=DEV)
        store[1:].copy_(sde.sigma)
        sde.sigma = nn.Parameter(store[1:])
    assert sde.sigma.data_ptr() % 16
    check(sde, torch.full((B, 8), 0.4, dtype=dtype, device=DEV), ts, DT)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_shards_past_row_2_24(dtype):
    B, d = 300, 12
    sde = SDE('gbm', 'stratonovich', B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ts = GRIDS['every_5'].to(dtype=dtype, device=DEV)
    ys, _ = check(sde, y0, ts, DT, {'cuda_graph': True}, row_offset=(1 << 24) + 5)
    other, _ = check(sde, y0, ts, DT, {'cuda_graph': True}, row_offset=(1 << 24) + 6)
    assert not torch.equal(ys[-1], other[-1])


def test_in_place_parameter_update_between_replays_is_followed():
    B, d = 64, 8
    sde = SDE('gbm', 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = GRIDS['not_a_multiple'].to(DEV)

    def solve():
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), device=DEV, entropy=3)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=DT, options={'cuda_graph': True})

    first = solve()
    with torch.no_grad():
        sde.sigma.mul_(1.5)
        sde.mu.add_(0.25)
    second = solve()
    graph.drop_plans(sde)
    with unfused():
        want = solve()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


@pytest.mark.parametrize('kind', ['gbm', 'pertraj'])
def test_cfg2_shaped_plan_launches_one_kernel_per_chunk(kind, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, T = 65536, 64, 200
    sde = SDE(kind, 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(sde, y0, ts, 2.0 ** -10, {'cuda_graph': True, 'static_output': False})
    # the recorded step runs before capture; the captured steps 0 .. T-1 have no boundary singles
    assert plan.abi_launches == -(-T // K)


def test_a_batch_below_one_wave_runs_one_step_per_launch(monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', CHUNK_LENGTH)
    B, d, T = 4096, 64, 100
    sde = SDE('gbm', 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.1, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * 2.0 ** -10
    _, plan = check(sde, y0, ts, 2.0 ** -10, {'cuda_graph': True, 'static_output': False})
    assert plan.abi_launches == T
