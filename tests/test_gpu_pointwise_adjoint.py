"""The backward sweep of `sdeint_adjoint`'s reversible pair as chunks of one kernel each
(adjoint_options={'fused_backward': True}; pointwise.AdjointRecorder, the TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN
program of tsde_solve_reversible_heun_pointwise).

Against the unfused sweep of the same solve: ys, y0's gradient and the gradients of the extra solver state (f0, g0, z0)
have the same bits; each parameter gradient differs by summation order only, within
(n_steps + B + 2) u S, S the sum of |contribution| over every step and row (what the unfused sweep reduces, measured
while it runs).  Against float64 central differences of the forward solve (tests/gradient_ref.py), in float64.  Run to
run and eager against captured, every result has the same bits, also after an in-place update of a parameter.  Index
paths past row 2^24 and the shard ending at the last drawable row, 2^32 - 2; a sharded sweep against the whole one;
and the launches of a cfg-shaped captured plan."""
import math

import pytest
import torch
from torch import nn
from torch.utils._python_dispatch import TorchDispatchMode

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import adjoint, pointwise
from . import gradient_ref
from .test_gpu_pointwise import same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
FUSED = {'fused_backward': True}
aten = torch.ops.aten


class Diag(nn.Module):
    """Element-wise Stratonovich SDEs: GBM with (d,) mu and sigma, OU with 0-d kappa and theta and a time-dependent
    drift, GBM with a per-trajectory (B, d) sigma, and a parameter used in both f and g."""
    sde_type, noise_type = 'stratonovich', 'diagonal'

    def __init__(self, kind, B, d, dtype):
        super().__init__()
        gen = torch.Generator().manual_seed(3)
        self.kind = kind
        r = lambda *s: torch.rand(*s, generator=gen, dtype=dtype)  # noqa: E731
        if kind == 'gbm':
            self.mu, self.sigma = nn.Parameter(r(d) - 0.5), nn.Parameter(0.5 * r(d) + 0.1)
        elif kind == 'ou':
            self.kappa, self.theta = nn.Parameter(r(()) + 0.5), nn.Parameter(r(()) - 0.5)
            self.sigma = nn.Parameter(0.3 * r(d) + 0.1)
        elif kind == 'pertraj':
            self.mu, self.sigma = nn.Parameter(r(d) - 0.5), nn.Parameter(0.5 * r(B, d) + 0.1)
        else:  # 'shared'
            self.a, self.b = nn.Parameter(0.5 * r(d) + 0.1), nn.Parameter(r(1) - 0.5)

    def f(self, t, y):
        if self.kind == 'ou':
            return self.kappa * (self.theta - y) * t
        if self.kind == 'shared':
            return self.a * y + self.b
        return self.mu * y

    def g(self, t, y):
        if self.kind == 'shared':
            return self.a * y
        return self.sigma * y


class _Scale(TorchDispatchMode):
    """S of the module docstring: the sum of |x| over every batch reduction (autograd's sum_to of a parameter's
    gradient) and every in-place accumulation (adj_param += v) of the unfused sweep."""

    def __init__(self):
        super().__init__()
        self.total = 0.0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        if func in (aten.sum.dim_IntList, aten.sum.default):
            self.total += float(args[0].detach().abs().double().sum())
        elif func is aten.add_.Tensor:
            self.total += float(args[1].detach().abs().double().sum())
        return func(*args, **(kwargs or {}))


def adjoint_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADJOINT)


def solve(sde, B, d, dtype, ts, dt, fused, graphs=False, entropy=7, bm_dt=None, row_offset=0, y0=None, scale=None,
          w=None, drop=True):
    """sdeint_adjoint and backward of sum(w * ys): (ys, y0.grad, extras' grads, parameter grads, the launches of the
    fused sweep's kernel)."""
    gen = torch.Generator(device=DEV).manual_seed(11)
    if y0 is None:
        y0 = 0.5 + torch.rand(B, d, generator=gen, dtype=dtype, device=DEV)
    y0 = y0.detach().clone().requires_grad_()
    t0 = ts[0]
    with torch.no_grad():
        extras = [sde.f(t0, y0).clone(), sde.g(t0, y0).clone(), y0.clone()]
    extras = [e.requires_grad_() for e in extras]
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), dtype=dtype, device=DEV, entropy=entropy, dt=bm_dt)
    if row_offset:
        bm.shard_rows(row_offset)
    opts = dict(FUSED) if fused else {}
    if graphs:
        opts['cuda_graph'] = True
    for p in sde.parameters():
        p.grad = None
    n0 = adjoint_launches()  # (a captured sweep launches its chunks when the forward pass captures it)
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


def compare(fused, unfused, n_steps, B, dtype, S):
    """The module docstring's guarantees; the worst ratio of a parameter's difference to its bound."""
    assert same_bits(fused[0], unfused[0]) and same_bits(fused[1], unfused[1])
    for a, b in zip(fused[2], unfused[2]):
        assert same_bits(a, b)
    u = torch.finfo(dtype).eps / 2
    tol = (n_steps + B + 2) * u * S
    worst = 0.0
    for a, b in zip(fused[3], unfused[3]):
        err = float((a.double() - b.double()).abs().max())
        worst = max(worst, err / tol if tol > 0 else 0.0)
        assert err <= tol, (err, tol)
    return worst


GRIDS = {'dense': (16, 2.0 ** -6, 1), 'sparse': (72, 2.0 ** -6, 12)}  # (steps, dt, steps per output interval)


def grid(name, dtype):
    n, dt, every = GRIDS[name]
    return torch.arange(0, n + 1, every, dtype=dtype, device=DEV) * dt, dt, n


@pytest.mark.parametrize('graphs', [False, True])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('kind', ['gbm', 'ou', 'pertraj', 'shared'])
@pytest.mark.parametrize('grid_name', ['dense', 'sparse'])
def test_the_fused_sweep_against_the_unfused_one(kind, dtype, graphs, grid_name):
    B, d = 97, 6
    ts, dt, n = grid(grid_name, dtype)
    scale = _Scale()
    # (S is measured on the eager sweep: a replay dispatches no ops; the unfused sweep's bits are the same captured)
    ref = solve(Diag(kind, B, d, dtype).to(DEV), B, d, dtype, ts, dt, False, scale=scale)
    got = solve(Diag(kind, B, d, dtype).to(DEV), B, d, dtype, ts, dt, True, graphs)
    assert ref[4] == 0 and got[4] > 0
    worst = compare(got, ref, n, B, dtype, scale.total)
    print(f"{kind} {dtype} graphs={graphs} {grid_name}: worst parameter error / bound {worst:.3g}")


def test_one_module_alternating_the_option_keeps_one_plan_each():
    """Captured sweeps of one module, with and without fused_backward in turn, the plans kept between the calls: each
    setting has its own plan, so the unfused solve keeps the unfused bits, parameters included, and the fused one
    launches its chunks."""
    B, d, dtype = 97, 6, torch.float32
    ts, dt, _ = grid('dense', dtype)
    sde = Diag('gbm', B, d, dtype).to(DEV)
    runs = [solve(sde, B, d, dtype, ts, dt, fused, True, drop=False) for fused in (False, True, False, True)]
    adjoint.drop_plans(sde)
    assert runs[0][4] == 0 and runs[1][4] > 0
    for a, b in ((runs[0], runs[2]), (runs[1], runs[3])):
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
        for x, y in zip(a[2] + a[3], b[2] + b[3]):
            assert same_bits(x, y)
    reference = solve(Diag('gbm', B, d, dtype).to(DEV), B, d, dtype, ts, dt, False)
    for x, y in zip(runs[2][3], reference[3]):
        assert same_bits(x, y)


@pytest.mark.parametrize('B,d', [(1, 5), (97, 3), (97, 1), (4099, 33)])
@pytest.mark.parametrize('every', [1, 3])
@pytest.mark.parametrize('cells', [1, 2])
def test_gradients_against_central_differences(B, d, every, cells):
    """float64: y0's and every parameter's gradient along random directions within gradient_ref.RTOL of the central
    difference of the forward solve; `cells` Brownian cells per step (a step of several runs alone)."""
    dtype = torch.float64
    n, dt = 12, 2.0 ** -5
    ts = torch.arange(0, n + 1, every, dtype=dtype, device=DEV) * dt
    sde = Diag('gbm', B, d, dtype).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    y0 = (0.5 + torch.rand(B, d, generator=gen, dtype=dtype, device=DEV)).requires_grad_()
    w = torch.rand(ts.numel(), B, d, generator=gen, dtype=dtype, device=DEV) - 0.5
    bm_dt = dt / cells

    def bm():
        return tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), dtype=dtype, device=DEV, entropy=3, dt=bm_dt)
    n0 = adjoint_launches()
    ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm(), method='reversible_heun', dt=dt, adjoint_options=dict(FUSED))
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


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_run_to_run_and_eager_against_captured(dtype):
    B, d = 4099, 12
    ts, dt, _ = grid('sparse', dtype)
    sde = Diag('ou', B, d, dtype).to(DEV)
    for update in (False, True):
        if update:
            with torch.no_grad():  # an optimiser-style step: the program reads the parameters by address
                for p in sde.parameters():
                    p.mul_(0.75)
        runs = [solve(sde, B, d, dtype, ts, dt, True, graphs) for graphs in (False, False, True, True)]
        for r in runs[1:]:
            assert same_bits(r[0], runs[0][0]) and same_bits(r[1], runs[0][1])
            for a, b in zip(r[2] + r[3], runs[0][2] + runs[0][3]):
                assert same_bits(a, b)
        if update:
            assert not same_bits(runs[0][3][0], before[3][0])
        before = runs[0]


@pytest.mark.parametrize('d', [12, 11])
def test_rows_past_2_24(d, monkeypatch):
    """B = 2^24 + 4099: the fused sweep against the unfused one, bit for bit where the guarantees say so; neighbouring
    rows differ (each row draws its own noise)."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)
    B, dtype = 2 ** 24 + 4099, torch.float32
    ts, dt, n = torch.tensor([0.0, 2.0 ** -6, 2.0 ** -5], device=DEV), 2.0 ** -6, 2
    scale = _Scale()
    ref = solve(Diag('gbm', B, d, dtype).to(DEV), B, d, dtype, ts, dt, False, scale=scale)
    got = solve(Diag('gbm', B, d, dtype).to(DEV), B, d, dtype, ts, dt, True)
    compare(got, ref, n, B, dtype, scale.total)
    rows = got[1][-4099:]
    assert not same_bits(rows[:-1], rows[1:])


def test_the_top_shard(monkeypatch):
    """A shard whose last global row is 2^32 - 2, the last row a launch may draw (as in
    tests/test_gpu_pointwise_index_paths.py)."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)
    B, d, dtype = 4099, 5, torch.float32
    ts, dt, n = grid('dense', dtype)
    scale = _Scale()
    kw = dict(row_offset=(1 << 32) - 1 - B)
    ref = solve(Diag('gbm', B, d, dtype).to(DEV), B, d, dtype, ts, dt, False, scale=scale, **kw)
    got = solve(Diag('gbm', B, d, dtype).to(DEV), B, d, dtype, ts, dt, True, **kw)
    compare(got, ref, n, B, dtype, scale.total)


def test_a_sharded_sweep_gives_the_whole_sweeps_rows(monkeypatch):
    """Two shards (bm.shard_rows) against the whole batch: every per-row result has the whole sweep's bits, and the
    parameter gradients summed over the shards are within the bound of the unfused whole sweep's."""
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: K)
    B, d, dtype = 4099, 7, torch.float32
    ts, dt, n = grid('sparse', dtype)
    gen = torch.Generator(device=DEV).manual_seed(2)
    y0 = 0.5 + torch.rand(B, d, generator=gen, device=DEV)
    w = torch.rand(ts.numel(), B, d, generator=gen, device=DEV) - 0.5
    sde = Diag('gbm', B, d, dtype).to(DEV)
    scale = _Scale()
    ref = solve(sde, B, d, dtype, ts, dt, False, y0=y0, w=w, scale=scale)
    whole = solve(sde, B, d, dtype, ts, dt, True, y0=y0, w=w)
    cut = 1500
    parts = [solve(sde, n_rows, d, dtype, ts, dt, True, y0=y0[a:a + n_rows], w=w[:, a:a + n_rows], row_offset=a)
             for a, n_rows in ((0, cut), (cut, B - cut))]
    assert all(p[4] > 0 for p in parts)
    assert same_bits(torch.cat([p[0] for p in parts], 1), whole[0])
    assert same_bits(torch.cat([p[1] for p in parts], 0), whole[1])
    for k in range(3):
        assert same_bits(torch.cat([p[2][k] for p in parts], 0), whole[2][k])
    summed = (whole[0], whole[1], whole[2], [a + b for a, b in zip(parts[0][3], parts[1][3])], whole[4])
    compare(summed, ref, n, B, dtype, scale.total)


def test_a_cfg_shaped_captured_plan_launches_one_kernel_per_chunk():
    B, d, T, dt, dtype = 65536, 64, 200, 2.0 ** -10, torch.float32
    ts = torch.arange(T + 1, device=DEV) * dt
    sde = Diag('gbm', B, d, dtype).to(DEV)
    counts = {}
    real = adjoint._BackwardEngine.sweep

    class _Ops(TorchDispatchMode):
        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            counts['ops'] = counts.get('ops', 0) + 1
            return func(*args, **(kwargs or {}))

    def sweep(self, ys, *a, **k):
        if ys.shape[0] != T + 1:  # (the warm-up sweep)
            return real(self, ys, *a, **k)
        n0, c0 = adjoint_launches(), _cabi.LAUNCHES
        with _Ops():
            out = real(self, ys, *a, **k)
        counts['chunks'], counts['abi'] = adjoint_launches() - n0, _cabi.LAUNCHES - c0
        return out
    adjoint._BackwardEngine.sweep = sweep
    try:
        solve(sde, B, d, dtype, ts, dt, True, graphs=True)
    finally:
        adjoint._BackwardEngine.sweep = real
    assert counts['chunks'] == counts['abi'] == math.ceil(T / K)
    # the torch ops of the captured sweep (buffers, the per-parameter reductions) do not grow with the steps
    assert counts['ops'] < 60, counts
