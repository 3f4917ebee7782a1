"""The backward sweep of `sdeint_adjoint`'s reversible pair for general and additive noise as chunks of one kernel each
(adjoint_options={'fused_backward': True}; pointwise.GeneralAdjointRecorder, the
TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN program of tsde_solve_reversible_heun_pointwise on a GENERAL launch).

Against the unfused sweep of the same solve: ys, y0's gradient and the gradients of the extra solver state (f0, g0 as
(rows, d, m), z0) have the same bits; each parameter gradient differs by summation order only, within
(n_steps + B + 2) u S, S the sum of |x| over every reduction of the unfused sweep.  The channel sum the kernel emits
for vjp_z (ATen's CUDA order of sum(-1, keepdim=True) for m <= 32) is restated here op by op and compared with
torch.sum bit for bit.  Run to run and eager against captured, every result has the same bits, also after an in-place
update of a parameter.  Against float64 central differences of the forward solve (tests/gradient_ref.py).  Index paths
past row 2^24 and the shard ending at the last drawable row; a sharded sweep against the whole one; and the launches of
a cfg-shaped captured plan.  Unless a test says otherwise, the chunks are TSDE_PW_MAX_STEPS long whatever the batch
(chunk_length patched), so g re-evaluated from z, adj_g carried in rank-2 form and the end-of-chunk stores run."""
import math

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import adjoint, pointwise
from . import gradient_ref
from .test_gpu_pointwise import same_bits
from .test_gpu_pointwise_adjoint import _Scale, adjoint_launches, compare

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS


@pytest.fixture(autouse=True)
def long_chunks(monkeypatch):
    """Chunks of up to TSDE_PW_MAX_STEPS steps at every batch size (a test may patch chunk_length again)."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)


class General(nn.Module):
    """Stratonovich SDEs with general / additive noise: correlated GBM (g = y (x) S), multi-factor OU
    (g = S expanded) and a transcendental one (g = tanh(y) (x) S)."""
    sde_type, noise_type = 'stratonovich', 'general'

    def __init__(self, kind, B, d, m, dtype):
        super().__init__()
        gen = torch.Generator().manual_seed(3)
        self.kind, self.B, self.m = kind, B, m
        r = lambda *s: torch.rand(*s, generator=gen, dtype=dtype)  # noqa: E731
        if kind == 'ou':
            self.kappa, self.theta = nn.Parameter(r(1) + 0.5), nn.Parameter(r(1) - 0.5)
        else:
            self.mu = nn.Parameter(r(d) - 0.5)
        self.S = nn.Parameter((r(d, m) - 0.5) * (0.6 / m ** 0.5))

    def f(self, t, y):
        if self.kind == 'ou':
            return self.kappa * (self.theta - y)
        if self.kind == 'tanh':
            return self.mu * torch.tanh(y)
        return self.mu * y

    def g(self, t, y):
        if self.kind == 'ou':
            return self.S.expand(y.shape[0], *self.S.shape)
        if self.kind == 'tanh':
            return torch.tanh(y).unsqueeze(-1) * self.S
        return y.unsqueeze(-1) * self.S


def solve(sde, B, d, m, dtype, ts, dt, fused, graphs=False, scale=None, transcendental=False, drop=True,
          row_offset=0, y0=None, w=None):
    gen = torch.Generator(device=DEV).manual_seed(11)
    if y0 is None:
        y0 = 0.5 + torch.rand(B, d, generator=gen, dtype=dtype, device=DEV)
    y0 = y0.detach().clone().requires_grad_()
    with torch.no_grad():
        extras = [sde.f(ts[0], y0).clone(), sde.g(ts[0], y0).contiguous().clone(), y0.clone()]
    extras = [e.requires_grad_() for e in extras]
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=dtype, device=DEV, entropy=7)
    if row_offset:
        bm.shard_rows(row_offset)
    opts = {'fused_backward': True} if fused else {}
    if graphs:
        opts['cuda_graph'] = True
    if transcendental:
        opts['transcendental'] = True
    for p in sde.parameters():
        p.grad = None
    n0 = adjoint_launches()
    ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=dt, adjoint_options=opts,
                             extra_solver_state=tuple(extras))
    if w is None:
        w = torch.rand(ys.shape, generator=gen, dtype=dtype, device=DEV) - 0.5
    if scale is not None:
        with scale:
            (w * ys).sum().backward()
    else:
        (w * ys).sum().backward()
    torch.cuda.synchronize()
    out = (ys.detach(), y0.grad, [e.grad for e in extras], [p.grad.clone() for p in sde.parameters()],
           adjoint_launches() - n0)
    if drop:
        adjoint.drop_plans(sde)
    return out


GRIDS = {'dense': (16, 2.0 ** -6, 1), 'sparse': (72, 2.0 ** -6, 12)}


def grid(name, dtype):
    n, dt, every = GRIDS[name]
    return torch.arange(0, n + 1, every, dtype=dtype, device=DEV) * dt, dt, n


def check(kind, m, dtype, graphs, grid_name, B=97, d=6):
    ts, dt, n = grid(grid_name, dtype)
    tr = kind == 'tanh'
    if tr and (pointwise.nvrtc_mismatch() or not _cabi.nvjitlink()):
        pytest.skip("no NVRTC / nvJitLink of PyTorch's CUDA release")
    scale = _Scale()
    ref = solve(General(kind, B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, False, scale=scale, transcendental=tr)
    got = solve(General(kind, B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, True, graphs, transcendental=tr)
    assert ref[4] == 0 and got[4] > 0
    if pointwise.chunk_length(None) == K:  # (chunks of several steps ran: fewer launches than steps)
        assert got[4] < n
    return compare(got, ref, n, B, dtype, scale.total)


@pytest.mark.parametrize('chunk', [1, K])
@pytest.mark.parametrize('graphs', [False, True])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', [2, 3, 5, 12, 4, 8, 16, 32])  # (generic route, then tile route)
def test_correlated_gbm_against_the_unfused_sweep(m, dtype, graphs, chunk, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: chunk)
    worst = check('gbm', m, dtype, graphs, 'dense')
    print(f"gbm m={m} {dtype} graphs={graphs}: worst parameter error / bound {worst:.3g}")


@pytest.mark.parametrize('grid_name', ['dense', 'sparse'])
@pytest.mark.parametrize('kind', ['gbm', 'ou', 'tanh'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_every_kind_on_both_grids(kind, dtype, grid_name):
    check(kind, 5, dtype, False, grid_name)
    check(kind, 16, dtype, True, grid_name)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('rows', [1, 97, 65536])
def test_the_restated_channel_sum_is_torch_sum(rows, dtype):
    gen = torch.Generator(device=DEV).manual_seed(5)
    for m in range(2, _cabi.PW_GENERAL_MAX_M + 1):
        d = 3
        mag = torch.exp2(torch.randint(-30, 30, (rows, d, m), generator=gen, device=DEV).to(dtype))
        x = (torch.rand(rows, d, m, generator=gen, dtype=dtype, device=DEV) - 0.5) * mag
        h = rows // 2 + 1
        x[:h, :, 1::2] = -x[:h, :, 0::2][..., :m // 2]  # (values that cancel)
        x[0, 0] = -0.0  # (signed zeros)
        x[-1, -1, :m // 2] = 0.0
        x[-1, -1, m // 2:] = -0.0
        want = torch.sum(x, -1, keepdim=True)
        assert same_bits(pointwise.channel_sum(x), want), m


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_run_to_run_and_eager_against_captured(dtype):
    B, d, m = 97, 6, 12
    ts, dt, n = grid('sparse', dtype)
    sde = General('gbm', B, d, m, dtype).to(DEV)
    runs = [solve(sde, B, d, m, dtype, ts, dt, True, graphs, drop=False) for graphs in (False, False, True, True)]
    with torch.no_grad():
        sde.S.mul_(1.25)  # (an optimiser step: the captured plan reads the parameter in place)
    runs += [solve(sde, B, d, m, dtype, ts, dt, True, graphs, drop=False) for graphs in (False, True)]
    adjoint.drop_plans(sde)
    assert all(r[4] < 72 for r in runs)  # (chunks of several steps)
    for a, b in ((runs[0], runs[1]), (runs[0], runs[2]), (runs[2], runs[3]), (runs[4], runs[5])):
        for x, y in zip([a[0], a[1]] + a[2] + a[3], [b[0], b[1]] + b[2] + b[3]):
            assert same_bits(x, y)
    assert not same_bits(runs[0][3][1], runs[4][3][1])


@pytest.mark.parametrize('kind', ['gbm', 'ou'])
@pytest.mark.parametrize('B,d,m', [(1, 5, 3), (97, 3, 4), (4099, 6, 16)])
@pytest.mark.parametrize('every', [1, 3])
def test_gradients_against_central_differences(kind, B, d, m, every):
    """float64: y0's and every parameter's gradient along random directions within gradient_ref.RTOL of the central
    difference of the forward solve."""
    dtype = torch.float64
    n, dt = 12, 2.0 ** -5
    ts = torch.arange(0, n + 1, every, dtype=dtype, device=DEV) * dt
    sde = General(kind, B, d, m, dtype).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    y0 = (0.5 + torch.rand(B, d, generator=gen, dtype=dtype, device=DEV)).requires_grad_()
    w = torch.rand(ts.numel(), B, d, generator=gen, dtype=dtype, device=DEV) - 0.5

    def bm():
        return tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=dtype, device=DEV, entropy=3)
    n0 = adjoint_launches()
    ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm(), method='reversible_heun', dt=dt,
                             adjoint_options={'fused_backward': True})
    (w * ys).sum().backward()
    assert adjoint_launches() > n0
    grads = [y0.grad] + [p.grad for p in sde.parameters()]
    inputs = [y0] + list(sde.parameters())

    def fn():
        return tsde.sdeint(sde, y0, ts, bm=bm(), method='reversible_heun', dt=dt)
    for i, (x, g) in enumerate(zip(inputs, grads)):
        v = torch.randn(x.shape, generator=gen, dtype=dtype, device=DEV)
        dirs = [None] * len(inputs)
        dirs[i] = v
        D, L = gradient_ref.directional(fn, inputs, dirs, w)
        got = float((g * v).sum())
        assert bool(gradient_ref.within(got, D, L)), (i, got, D, L)


@pytest.mark.parametrize('d,m', [(3, 4), (5, 3)])
def test_rows_past_2_24(d, m):
    """B = 2^24 + 4099: the fused sweep against the unfused one, bit for bit where the guarantees say so; neighbouring
    rows differ (each row draws its own noise)."""
    B, dtype = 2 ** 24 + 4099, torch.float32
    ts, dt, n = torch.tensor([0.0, 2.0 ** -6, 2.0 ** -5], device=DEV), 2.0 ** -6, 2
    scale = _Scale()
    ref = solve(General('gbm', B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, False, scale=scale)
    got = solve(General('gbm', B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, True)
    compare(got, ref, n, B, dtype, scale.total)
    rows = got[1][-4099:]
    assert not same_bits(rows[:-1], rows[1:])


def test_the_top_shard():
    """A shard whose last global row is 2^32 - 2, the last row a launch may draw."""
    B, d, m, dtype = 4099, 5, 4, torch.float32
    ts, dt, n = grid('dense', dtype)
    scale = _Scale()
    kw = dict(row_offset=(1 << 32) - 1 - B)
    ref = solve(General('gbm', B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, False, scale=scale, **kw)
    got = solve(General('gbm', B, d, m, dtype).to(DEV), B, d, m, dtype, ts, dt, True, **kw)
    compare(got, ref, n, B, dtype, scale.total)


def test_a_sharded_sweep_gives_the_whole_sweeps_rows():
    """Two shards (bm.shard_rows) against the whole batch: every per-row result has the whole sweep's bits, and the
    parameter gradients summed over the shards are within the bound of the unfused whole sweep's."""
    B, d, m, dtype = 4099, 7, 5, torch.float32
    ts, dt, n = grid('sparse', dtype)
    gen = torch.Generator(device=DEV).manual_seed(2)
    y0 = 0.5 + torch.rand(B, d, generator=gen, device=DEV)
    w = torch.rand(ts.numel(), B, d, generator=gen, device=DEV) - 0.5
    sde = General('gbm', B, d, m, dtype).to(DEV)
    scale = _Scale()
    ref = solve(sde, B, d, m, dtype, ts, dt, False, y0=y0, w=w, scale=scale)
    whole = solve(sde, B, d, m, dtype, ts, dt, True, y0=y0, w=w)
    cut = 1500
    parts = [solve(sde, rows, d, m, dtype, ts, dt, True, y0=y0[a:a + rows], w=w[:, a:a + rows], row_offset=a)
             for a, rows in ((0, cut), (cut, B - cut))]
    assert all(p[4] > 0 for p in parts)
    assert same_bits(torch.cat([p[0] for p in parts], 1), whole[0])
    assert same_bits(torch.cat([p[1] for p in parts], 0), whole[1])
    for k in range(3):
        assert same_bits(torch.cat([p[2][k] for p in parts], 0), whole[2][k])
    summed = (whole[0], whole[1], whole[2], [a + b for a, b in zip(parts[0][3], parts[1][3])], whole[4])
    compare(summed, ref, n, B, dtype, scale.total)


def test_a_cfg_shaped_captured_plan_launches_one_kernel_per_chunk(monkeypatch):
    """Correlated GBM at B = 8192, d = 32, m = 16, 200 steps, captured, with the library's own chunk length: one
    compiled kernel per chunk and nothing else from the library."""
    monkeypatch.undo()
    B, d, m, T, dt, dtype = 8192, 32, 16, 200, 2.0 ** -10, torch.float32
    ts = torch.arange(T + 1, device=DEV) * dt
    sde = General('gbm', B, d, m, dtype).to(DEV)
    counts = {}
    real = adjoint._BackwardEngine.sweep

    def sweep(self, ys, *a, **k):
        if ys.shape[0] != T + 1:  # (the warm-up sweep)
            return real(self, ys, *a, **k)
        n0, c0 = adjoint_launches(), _cabi.LAUNCHES
        out = real(self, ys, *a, **k)
        counts['chunks'], counts['abi'] = adjoint_launches() - n0, _cabi.LAUNCHES - c0
        counts['length'] = pointwise.chunk_length(self)
        return out
    monkeypatch.setattr(adjoint._BackwardEngine, 'sweep', sweep)
    solve(sde, B, d, m, dtype, ts, dt, True, graphs=True)
    assert counts['chunks'] == counts['abi'] == math.ceil(T / counts['length'])
