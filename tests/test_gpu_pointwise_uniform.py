"""The compiled Milstein kernel's loop for a uniform grid (csrc/pw_device.cuh, pw_milstein_uniform): a chunk whose steps
all store their state to evenly spaced rows of the output series runs it; a chunk that stores only its last state runs
the step-table loop.  The two give the same final state, bit for bit, for programs that read the time and that do not,
Itô and Stratonovich, in both dtypes, over chunks of several steps (the second chunk starting mid-grid)."""
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200._core import graph, pointwise
from .test_gpu_pointwise import SDE, fused_launches, same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def final_state(sde, y0, ts, dt):
    B, m = y0.shape
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=y0.dtype, device=DEV, entropy=3)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=dt)
    graph.drop_plans(sde)
    return ys[-1]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('kind,sde_type', [('gbm', 'ito'), ('time', 'ito'), ('gbm', 'stratonovich')])
def test_uniform_loop_matches_the_step_table_loop(kind, sde_type, dtype, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: 16)
    B, d, T, dt = 96, 16, 24, 2.0 ** -6
    sde = SDE(kind, sde_type, B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    n0 = fused_launches()
    every = final_state(sde, y0, torch.arange(T + 1, dtype=dtype, device=DEV) * dt, dt)
    last = final_state(sde, y0, torch.tensor([0.0, T * dt], dtype=dtype, device=DEV), dt)
    assert fused_launches() > n0, "the steps were not fused"
    assert same_bits(every, last)
