"""A diagonal-noise Milstein step as one kernel (tsde_step_milstein_pointwise, torchsde_b200/_core/pointwise.py).

The fused step must give the unfused step's bits.  The unfused reference is the same solve with the tape rejected
(the recorder's `finish` patched to return None).  The route is confirmed by the kernel family's launch counter
(TSDE_KERNEL_PW_MILSTEIN).  Covered: GBM Ito / Stratonovich, per-trajectory GBM, OU, a time-dependent drift, division
by a tensor and by a Python number, g = y*y (whose vjp accumulates with add), a drift written in place, in float32 and float64, eager, graph and
row_split; a cfg2-sized graph solve; batch shards past global row 2^24 at d = 12 (d/4 is not a power of two); the
element path (d % 4 != 0, a misaligned parameter); in-place parameter updates between replays; every whitelisted op
on signed zeros, subnormals, infinities, NaN and extreme magnitudes; and the SDEs and solves that keep the unfused
step (among them a drift written in place through a `detach()` alias)."""
import contextlib

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PW = _cabi.KERNEL_PW_MILSTEIN


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(PW)


@contextlib.contextmanager
def unfused():
    """The tape is always rejected: every step runs the user's ops and the unfused kernels."""
    finish = pointwise.Recorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    try:
        yield
    finally:
        pointwise.Recorder.finish = finish


class SDE(nn.Module):
    noise_type = 'diagonal'

    def __init__(self, kind, sde_type, B, d, dtype, seed=0):
        super().__init__()
        self.kind, self.sde_type = kind, sde_type
        gen = torch.Generator().manual_seed(seed)
        shape = (B, d) if kind == 'pertraj' else (d,)
        self.sigma = nn.Parameter((torch.rand(shape, generator=gen, dtype=torch.float64) * 0.5 + 0.1).to(dtype))
        self.mu = nn.Parameter((torch.rand(shape, generator=gen, dtype=torch.float64) - 0.5).to(dtype))
        self.theta = nn.Parameter(torch.rand(1, generator=gen, dtype=torch.float64).to(dtype) + 0.5)

    def f(self, t, y):
        k = self.kind
        if k in ('gbm', 'pertraj'):
            return self.mu * y if self.sde_type == 'ito' else self.mu * y - .5 * (self.sigma ** 2) * y
        if k == 'ou':
            return self.theta * (self.mu - y)
        if k == 'time':
            return t * y
        if k == 'div':
            return y / (self.sigma + 1)
        if k == 'square':
            return -y
        if k == 'in_place':
            a = self.mu * y
            a.add_(1)
            return a
        raise AssertionError(k)

    def g(self, t, y):
        if self.kind == 'div':
            return self.sigma * y / 3
        if self.kind == 'square':
            return y * y
        return self.sigma * y


KINDS = [('gbm', 'ito'), ('gbm', 'stratonovich'), ('pertraj', 'ito'), ('ou', 'ito'), ('time', 'ito'),
         ('div', 'stratonovich'), ('square', 'ito'), ('in_place', 'stratonovich')]


def solve(sde, y0, T, dt, options=None, row_offset=0, entropy=11, method='milstein'):
    B, m = y0.shape
    bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy)
    if row_offset:
        bm.shard_rows(row_offset)
    ts = torch.arange(T + 1, dtype=y0.dtype, device=DEV) * dt
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options or {}))
    graph.drop_plans(sde)
    return ys


def same_bits(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    ia = a.view(torch.int32 if a.dtype == torch.float32 else torch.int64)
    ib = b.view(torch.int32 if b.dtype == torch.float32 else torch.int64)
    return bool(torch.equal(ia, ib))


def check_fused(sde, y0, T, dt, options=None, row_offset=0):
    n0 = fused_launches()
    ys = solve(sde, y0, T, dt, options, row_offset)
    assert fused_launches() > n0, "the step was not fused"
    with unfused():
        n1 = fused_launches()
        ref = solve(sde, y0, T, dt, options, row_offset)
        assert fused_launches() == n1
    assert same_bits(ys, ref)
    return ys


MODES = {'eager': {}, 'graph': {'cuda_graph': True}, 'row_split': {'cuda_graph': True, 'row_split': 3}}


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('kind,sde_type', KINDS)
def test_small_solves_are_bit_identical(kind, sde_type, dtype, mode):
    if kind == 'pertraj' and mode == 'row_split':
        pytest.skip("per-trajectory parameters do not broadcast over a row block")
    B, d = 96, 16
    sde = SDE(kind, sde_type, B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    check_fused(sde, y0, 12, 2.0 ** -6, MODES[mode])


@pytest.mark.parametrize('kind', ['gbm', 'pertraj'])
def test_cfg2_sized_graph_solve_is_bit_identical(kind):
    B, d = 65536, 64
    sde = SDE(kind, 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.1, device=DEV)
    check_fused(sde, y0, 8, 2.0 ** -10, {'cuda_graph': True, 'static_output': False})


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('mode', ['eager', 'graph'])
def test_shards_past_row_2_24_at_a_width_of_three_quads(dtype, mode):
    B, d = 300, 12
    sde = SDE('gbm', 'stratonovich', B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    ys = check_fused(sde, y0, 6, 2.0 ** -5, MODES[mode], row_offset=(1 << 24) + 5)
    other = check_fused(sde, y0, 6, 2.0 ** -5, MODES[mode], row_offset=(1 << 24) + 6)
    assert not torch.equal(ys[-1], other[-1])  # the rows draw their global index's increments


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_element_path_odd_width_and_misaligned_parameter(dtype):
    B = 50
    sde = SDE('ou', 'ito', B, 7, dtype).to(DEV)
    check_fused(sde, torch.full((B, 7), 0.4, dtype=dtype, device=DEV), 5, 2.0 ** -5, {'cuda_graph': True})
    sde = SDE('gbm', 'ito', B, 8, dtype).to(DEV)
    with torch.no_grad():
        store = torch.zeros(9, dtype=dtype, device=DEV)
        store[1:].copy_(sde.sigma)
        sde.sigma = nn.Parameter(store[1:])  # 4 or 8 bytes past a 16-byte boundary
    assert sde.sigma.data_ptr() % 16
    check_fused(sde, torch.full((B, 8), 0.4, dtype=dtype, device=DEV), 5, 2.0 ** -5)


def test_in_place_parameter_update_between_replays_is_followed():
    B, d = 64, 8
    sde = SDE('gbm', 'ito', B, d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(5, device=DEV) * 2.0 ** -5

    def run():
        bm = tsde.BrownianInterval(0.0, 4 * 2.0 ** -5, size=(B, d), device=DEV, entropy=3)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=2.0 ** -5, options={'cuda_graph': True})

    first = run()
    with torch.no_grad():
        sde.sigma.mul_(1.5)       # what an optimiser step does: same storage
        sde.mu.add_(0.25)
    second = run()                # a replay of the same plan
    graph.drop_plans(sde)
    with unfused():
        want = run()
    graph.drop_plans(sde)
    assert not torch.equal(first, second) and same_bits(second, want)


SPECIAL = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, 1.1754944e-38, 5e-324, 2.2250738585072014e-308, 1.0, -1.0, 3.0,
           -0.1, 3.4028235e38, -3.4028235e38, 1.7976931348623157e308, 1e-30, 1e30, float('inf'), float('-inf'),
           float('nan')]
OPS = {
    'mul': lambda a, b: a * b, 'add': lambda a, b: a + b, 'sub': lambda a, b: a - b, 'div': lambda a, b: a / b,
    'div_scalar': lambda a, b: a / 3, 'div_scalar_7': lambda a, b: a / 7.0, 'mul_scalar': lambda a, b: 0.1 * a,
    'neg': lambda a, b: -a, 'pow2': lambda a, b: a ** 2, 'sqrt': lambda a, b: torch.sqrt(a),
    'rsub': lambda a, b: 2.5 - a, 'add_scalar': lambda a, b: a + 1e-3,
}


class OpSDE(nn.Module):
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, op, a, b):
        super().__init__()
        self.op, self.a, self.b = op, nn.Parameter(a), nn.Parameter(b)

    def f(self, t, y):
        return OPS[self.op](self.a, self.b) + y

    def g(self, t, y):
        return 0.0 * y


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('op', sorted(OPS))
def test_each_op_matches_aten_on_special_values(op, dtype):
    """y0 = 0, dt = 1, g = 0*y: y1 = f, which is the op on every pair of special values (rows x channels)."""
    vals = torch.tensor(SPECIAL, dtype=torch.float64).to(dtype)
    n = len(vals)
    a, b = vals.repeat_interleave(n).reshape(n * n // 4, 4), vals.repeat(n).reshape(n * n // 4, 4)
    sde = OpSDE(op, a.to(DEV), b.to(DEV))
    y0 = torch.zeros_like(sde.a)
    ys = check_fused(sde, y0, 1, 1.0, {'cuda_graph': True})
    want = OPS[op](sde.a.detach(), sde.b.detach())
    got = ys[-1]
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan], want[~nan])   # (== : a -0 result may come out +0 after adding g*dW = 0)


# ---- SDEs and solves that keep the unfused step ------------------------------------------------------------------
class Nonlinear(SDE):
    def __init__(self, kind, B, d):
        super().__init__('gbm', 'ito', B, d, torch.float32)
        self.what = kind

    def f(self, t, y):
        if self.what == 'sigmoid':
            return torch.sigmoid(y) * self.mu
        if self.what == 'matmul':
            return y @ torch.eye(y.shape[1], device=y.device) * self.mu
        if self.what == 'item':
            return self.mu * y * float(self.theta.item())
        if self.what == 'alias_write':  # `a` keeps its storage's old value for the recorder: must not be fused
            a = self.mu * y
            a.detach().add_(1)
            return a
        return self.mu * y

    def g(self, t, y):
        if self.what == 'exp':
            return self.sigma * torch.exp(-y)
        return self.sigma * y

    def h(self, t, y):
        return self.mu * y * 0.5


FALLBACKS = ['sigmoid', 'exp', 'matmul', 'item', 'alias_write', 'logqp', 'autocast', 'grad_free', 'overlap', 'unbound', 'additive']


@pytest.mark.parametrize('case', FALLBACKS)
def test_unfusable_solves_keep_the_unfused_step(case):
    B, d, T, dt = 32, 8, 6, 2.0 ** -5
    sde = Nonlinear(case, B, d).to(DEV)
    y0 = torch.full((B, d), 0.2, device=DEV)
    ts = torch.arange(T + 1, device=DEV) * dt
    kw, ctx, m = {}, contextlib.nullcontext, d
    if case == 'logqp':
        kw['logqp'], m = True, d + 1
    if case == 'autocast':
        ctx = lambda: torch.autocast('cuda', dtype=torch.bfloat16)  # noqa: E731
    if case in ('grad_free', 'overlap'):
        kw['options'] = {case: False if case == 'overlap' else True}
    if case == 'additive':
        sde.noise_type = 'additive'
        sde.g = lambda t, y: torch.full((B, d, d), 0.1, device=DEV)

    def run():
        if case == 'unbound':   # a Brownian motion that cannot bind the solver grid: increments are materialised
            bm = tsde.BrownianPath(t0=0.0, w0=torch.zeros(B, d, device=DEV))
        else:
            bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), device=DEV, entropy=5)
        with torch.no_grad(), ctx():
            out = tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=dt, **kw)
        return out if isinstance(out, tuple) else (out,)

    n0 = fused_launches()
    out = run()
    assert fused_launches() == n0
    if case == 'unbound':
        return  # (its increments come from torch's generator: two solves differ)
    with unfused():
        ref = run()
    for x, r in zip(out, ref):
        assert same_bits(x, r)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_multi_cell_steps_are_fused(dtype):
    """A Brownian grid three times finer than the solver's: every step merges three cells."""
    B, d, T, dt = 40, 8, 5, 2.0 ** -5
    sde = SDE('gbm', 'ito', B, d, dtype).to(DEV)
    y0 = torch.full((B, d), 0.2, dtype=dtype, device=DEV)
    ts = torch.arange(T + 1, dtype=dtype, device=DEV) * dt

    def run():
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, d), dtype=dtype, device=DEV, entropy=5, dt=dt / 4)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=dt)

    n0 = fused_launches()
    ys = run()
    assert fused_launches() > n0
    with unfused():
        assert same_bits(ys, run())


def test_gradients_and_the_adjoint_backward_keep_the_unfused_step():
    """Gradients through `sdeint`: every launch is an autograd node, nothing is fused.  `sdeint_adjoint`: its forward
    pass is an ordinary no-grad solve of the user's SDE and is fused; the backward solve of the adjoint SDE is not.
    Solutions and gradients equal those of the same solves with the tape rejected."""
    B, d, T, dt = 32, 8, 6, 2.0 ** -5
    ts = torch.arange(T + 1, device=DEV) * dt
    grads = []
    for ctx in (contextlib.nullcontext, unfused):
        with ctx():
            out = []
            for adjoint in (False, True):
                sde = SDE('gbm', 'ito', B, d, torch.float32).to(DEV)
                y0 = torch.full((B, d), 0.2, device=DEV, requires_grad=True)
                bm = tsde.BrownianInterval(0.0, T * dt, size=(B, d), device=DEV, entropy=9)
                fn = tsde.sdeint_adjoint if adjoint else tsde.sdeint
                n0 = fused_launches()
                ys = fn(sde, y0, ts, bm=bm, method='milstein', dt=dt)
                n1 = fused_launches()
                ys.pow(2).sum().backward()
                assert fused_launches() == n1          # no backward step is fused
                fused_forward = adjoint and ctx is contextlib.nullcontext
                assert (n1 > n0) == fused_forward      # gradients through sdeint: every launch an autograd node
                out += [ys.detach(), y0.grad, sde.sigma.grad]
            grads.append(out)
    for a, b in zip(*grads):
        assert torch.equal(a, b)
