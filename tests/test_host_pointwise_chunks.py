"""How a solve whose Milstein steps run as an element-wise program is cut into launches (pointwise.plan_chunks): at
most TSDE_PW_MAX_STEPS consecutive steps per launch, a step that spans several Brownian cells alone, a step with a
non-aligned output alone and the step before it ending a chunk, aligned outputs anywhere inside a chunk."""
import pytest

from torchsde_b200 import _cabi
from torchsde_b200._core import schedule
from torchsde_b200._core.pointwise import plan_chunks

import torch

K = _cabi.PW_MAX_STEPS


def _check_cover(chunks, first, n):
    assert chunks[0][0] == first and chunks[-1][1] == n
    for (a, b), (c, _) in zip(chunks, chunks[1:]):
        assert b == c
    assert all(0 < b - a <= K for a, b in chunks)


@pytest.mark.parametrize('n', [1, 2, K - 1, K, K + 1, 2 * K, 3 * K + 7, 1000])
def test_steps_below_at_and_above_the_chunk_length(n):
    chunks = plan_chunks(0, n)
    _check_cover(chunks, 0, n)
    assert len(chunks) == -(-n // K)
    assert all(b - a == K for a, b in chunks[:-1])


def test_the_recorded_first_step_is_not_planned():
    chunks = plan_chunks(1, 1001)
    _check_cover(chunks, 1, 1001)
    assert len(chunks) == -(-1000 // K)


def _interpolated(sched):
    return [k for k, os in sched.outputs_after.items() if any(not o.aligned for o in os)]


def test_outputs_every_few_steps_do_not_end_a_chunk():
    sched = schedule.build_schedule(torch.arange(0, 201, 5, dtype=torch.float64) * 2.0 ** -8, 2.0 ** -8)
    assert sched.n_steps == 200 and not _interpolated(sched)
    assert plan_chunks(1, 200, _interpolated(sched)) == [(1, 1 + K), (1 + K, 1 + 2 * K), (1 + 2 * K, 1 + 3 * K),
                                                          (1 + 3 * K, 200)]


def test_non_aligned_outputs_run_alone_after_a_chunk_end():
    # dt = 1/16 on outputs at 0.09375 and 0.25: steps [0, .0625], [.0625, .125] (holds 0.09375), [.125, .1875],
    # [.1875, .25]
    sched = schedule.build_schedule(torch.tensor([0.0, 0.09375, 0.25]), 0.0625)
    assert _interpolated(sched) == [1]
    assert plan_chunks(1, 4, _interpolated(sched)) == [(1, 2), (2, 4)]
    # from step 0 on: the step before an interpolated one ends its chunk
    assert plan_chunks(0, 4, _interpolated(sched)) == [(0, 1), (1, 2), (2, 4)]
    # several interpolated steps in a long solve
    ts = torch.tensor([0.0, 1.3, 7.5, 7.7, 100.0, 200.0], dtype=torch.float64) * 2.0 ** -6
    sched = schedule.build_schedule(ts, 2.0 ** -6)
    interp = _interpolated(sched)
    assert interp == [1, 7]
    chunks = plan_chunks(1, sched.n_steps, interp)
    _check_cover(chunks, 1, sched.n_steps)
    assert (1, 2) in chunks and (7, 8) in chunks and (2, 7) in chunks


def test_a_short_last_step():
    sched = schedule.build_schedule(torch.tensor([0.0, 1.0], dtype=torch.float64), 0.3)
    assert sched.n_steps == 4 and not _interpolated(sched)  # 0.3, 0.6, 0.9, 1.0
    assert plan_chunks(1, 4, _interpolated(sched)) == [(1, 4)]


def test_a_multi_cell_step_in_the_middle_runs_alone():
    assert plan_chunks(1, 300, (), [100]) == [(1, 1 + K), (1 + K, 100), (100, 101), (101, 101 + K),
                                              (101 + K, 101 + 2 * K), (101 + 2 * K, 101 + 3 * K), (101 + 3 * K, 300)]
    assert plan_chunks(0, 5, [2], [3]) == [(0, 2), (2, 3), (3, 4), (4, 5)]


def test_chunk_table_fits_the_header_limit():
    assert K == 64
    hdr = open(__file__.replace('tests/test_host_pointwise_chunks.py', 'include/torchsde_b200.h')).read()
    assert f'#define TSDE_PW_MAX_STEPS {K}' in hdr
