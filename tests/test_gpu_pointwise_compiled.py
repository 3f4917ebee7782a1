"""Milstein programs compiled at run time into kernels of their own (csrc/pointwise.cu, pw_milstein_source).

A compiled solve, eager and captured, gives the unfused solve's bytes on cfg2's SDE (f = mu*y, g = sigma*y) and on
full-truncation CIR (clamp and sqrt, a program with comparison ops); a parameter updated in place between graph
replays is followed, since operand addresses are launch parameters; an SDE of the same structure with other
parameters reuses the compiled kernel (one compilation, counted by pointwise.COMPILES); and when compilation
fails the tape is rejected and the solve keeps the unfused step."""
import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from .test_gpu_pointwise import SDE, check_fused, fused_launches, same_bits, solve, unfused
from .test_gpu_pointwise_select import SDE as SelectSDE

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MODES = {'eager': {}, 'graph': {'cuda_graph': True}}


def compiles():
    return pointwise.COMPILES


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('kind', ['cfg2', 'cir_clamp'])
def test_compiled_solve_is_byte_identical_to_the_unfused_one(kind, mode):
    B, d = 16384, 64  # enough CTAs for chunks of 64 steps (pointwise.chunk_length)
    if kind == 'cfg2':
        sde = SDE('gbm', 'ito', B, d, torch.float32).to(DEV)
        y0 = torch.full((B, d), 0.1, device=DEV)
    else:
        sde = SelectSDE('cir_clamp', 'ito', d, torch.float32).to(DEV)
        y0 = torch.full((B, d), 0.04, device=DEV)
    check_fused(sde, y0, 70, 2.0 ** -10, MODES[mode])  # a chunk of 64 steps and one of 6


def test_in_place_parameter_update_between_replays_is_followed():
    B, d = 256, 16
    sde = SDE('ou', 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(9, device=DEV) * 2.0 ** -5

    def run():
        bm = tsde.BrownianInterval(0.0, 8 * 2.0 ** -5, size=(B, d), device=DEV, entropy=5)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=2.0 ** -5, options={'cuda_graph': True})

    first = run()
    with torch.no_grad():
        sde.theta.mul_(1.5)  # a SCALAR operand
        sde.mu.add_(0.25)    # a CHANNEL operand
    second = run()           # a replay of the same plan
    graph.drop_plans(sde)
    with unfused():
        want = run()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


class Chain(nn.Module):
    """f = mu * y * theta * ... * theta (`links` factors of theta), g = sigma * y: a program structure of this test's own,
    which no other test of the process compiles before it, so the compilations it counts are its own."""
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, links, d, seed):
        super().__init__()
        gen = torch.Generator().manual_seed(seed)
        self.links = links
        self.mu = nn.Parameter(torch.rand(d, generator=gen, dtype=torch.float64) - 0.5)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen, dtype=torch.float64) * 0.5 + 0.1)
        self.theta = nn.Parameter(torch.rand(1, generator=gen, dtype=torch.float64) * 0.2 + 0.9)

    def f(self, t, y):
        out = self.mu * y
        for _ in range(self.links):
            out = out * self.theta
        return out

    def g(self, t, y):
        return self.sigma * y


def test_same_structure_reuses_the_compiled_kernel():
    B, d = 128, 24
    y0 = torch.full((B, d), 0.3, dtype=torch.float64, device=DEV)
    n0 = compiles()
    check_fused(Chain(11, d, seed=7).to(DEV), y0, 5, 2.0 ** -5)  # compiled on its first solve
    assert compiles() == n0 + 1
    check_fused(Chain(11, d, seed=8).to(DEV), y0, 5, 2.0 ** -5)  # other values, other addresses: the same kernel
    assert compiles() == n0 + 1
    check_fused(Chain(12, d, seed=9).to(DEV), y0, 5, 2.0 ** -5)  # another structure
    assert compiles() == n0 + 2


def test_a_failed_compilation_keeps_the_unfused_step(monkeypatch):
    B, d = 96, 16
    sde = SDE('square', 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.2, device=DEV)
    monkeypatch.setattr(_cabi, 'compile_pointwise', lambda prog, dtype: _cabi.ECOMPILE)
    monkeypatch.setattr(pointwise, '_COMPILED', {})  # (as if no program of this structure had been compiled)
    n0 = fused_launches()
    ys = solve(sde, y0, 6, 2.0 ** -5, {'cuda_graph': True})
    assert fused_launches() == n0
    monkeypatch.undo()
    with unfused():
        ref = solve(sde, y0, 6, 2.0 ** -5, {'cuda_graph': True})
    assert same_bits(ys, ref)
