"""Element-wise SDEs with clamp, relu, abs, maximum / minimum, torch.where, masked_fill, comparisons and reciprocal
fused into one kernel per step or chunk (torchsde_b200/_core/pointwise.py, csrc/pointwise.cu).

Every fused solve must give the unfused solve's bits; the unfused reference is the same solve with the tape rejected
(Recorder.finish and SrkRecorder.finish patched to return None), and the launch counters of the element-wise kernel
families confirm the route.  Covered: every fixed-step method that fuses (Milstein Ito and Stratonovich, SRK, Heun,
midpoint, Euler-Heun, Euler, reversible Heun) on CIR with full truncation (clamp and relu), reflection (sqrt of abs),
maximum / minimum against a per-channel parameter, clamp with (d,) tensor bounds, a piecewise torch.where drift and
diffusion and a reciprocal, in float32 and float64, eager, graph and row_split; every new op on every pair of special
values (signed zeros, subnormals, infinities, NaN, extremes) through f and through the vjp of g; a cfg2-sized CIR graph
solve in chunks; and `sdeint_adjoint` with the reversible pair."""
import contextlib

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from .test_gpu_pointwise import SPECIAL, same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda'
FAMILIES = (_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_SRK, _cabi.KERNEL_PW_PC, _cabi.KERNEL_PW_CHUNK)


def fused_launches():
    return sum(_cabi.lib().tsde_kernel_launches(k) for k in FAMILIES)


@contextlib.contextmanager
def unfused():
    """The tape is always rejected: every step runs the user's ops and the unfused kernels."""
    saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


class SDE(nn.Module):
    noise_type = 'diagonal'

    def __init__(self, kind, sde_type, d, dtype, seed=0):
        super().__init__()
        self.kind, self.sde_type = kind, sde_type
        gen = torch.Generator().manual_seed(seed)

        def param(shape, lo, hi):
            return nn.Parameter((torch.rand(shape, generator=gen, dtype=torch.float64) * (hi - lo) + lo).to(dtype))
        self.kappa, self.theta, self.xi = param(d, 0.5, 2.0), param(d, 0.02, 0.1), param(d, 0.2, 0.6)
        self.floor = param(d, -0.05, 0.05)

    def f(self, t, y):
        k = self.kind
        if k == 'cir_clamp':
            return self.kappa * (self.theta - y.clamp(min=0))
        if k == 'cir_relu':
            return self.kappa * (self.theta - torch.relu(y))
        if k in ('reflection', 'maximum'):
            return self.kappa * (self.theta - y)
        if k == 'clamp_tensor':
            return self.kappa * (self.theta - torch.clamp(y, min=self.floor, max=self.theta))
        if k == 'where':
            return torch.where(y > self.theta, -self.kappa * y, self.kappa * (self.theta - y))
        if k == 'reciprocal':
            return self.kappa * torch.reciprocal(1 + y * y)
        raise AssertionError(k)

    def g(self, t, y):
        k = self.kind
        if k == 'cir_clamp':
            return self.xi * torch.sqrt(y.clamp(min=0))
        if k == 'cir_relu':
            return self.xi * torch.sqrt(torch.relu(y))
        if k == 'reflection':
            return self.xi * torch.sqrt(y.abs())
        if k == 'maximum':
            return self.xi * torch.maximum(y, self.floor) - 0.1 * torch.minimum(y, self.theta)
        if k == 'clamp_tensor':
            return self.xi * torch.clamp(y, min=self.floor)
        if k == 'where':
            return torch.where(y > 0, self.xi * y, 0.0) + torch.where(y < self.floor, 0.01, self.xi * 0.1)
        if k == 'reciprocal':
            return self.xi * y * torch.reciprocal(1 + y.abs())
        raise AssertionError(k)


KINDS = ['cir_clamp', 'cir_relu', 'reflection', 'maximum', 'clamp_tensor', 'where', 'reciprocal']
METHODS = {'milstein_ito': ('milstein', 'ito'), 'milstein_strat': ('milstein', 'stratonovich'), 'srk': ('srk', 'ito'),
           'heun': ('heun', 'stratonovich'), 'midpoint': ('midpoint', 'stratonovich'),
           'euler_heun': ('euler_heun', 'stratonovich'), 'euler': ('euler', 'ito'),
           'reversible_heun': ('reversible_heun', 'stratonovich')}
MODES = {'eager': {}, 'graph': {'cuda_graph': True}, 'row_split': {'cuda_graph': True, 'row_split': 3}}


def solve(sde, y0, T, dt, method, options=None, entropy=11):
    B, m = y0.shape
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), dtype=y0.dtype, device=DEV, entropy=entropy,
                               levy_area_approximation=levy)
    ts = torch.arange(T + 1, dtype=y0.dtype, device=DEV) * dt
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options or {}))
    graph.drop_plans(sde)
    return ys


def check_fused(sde, y0, T, dt, method, options=None):
    n0 = fused_launches()
    ys = solve(sde, y0, T, dt, method, options)
    assert fused_launches() > n0, "the step was not fused"
    with unfused():
        n1 = fused_launches()
        ref = solve(sde, y0, T, dt, method, options)
        assert fused_launches() == n1
    assert same_bits(ys, ref)
    return ys, ref


@pytest.mark.parametrize('mode', sorted(MODES))
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method', sorted(METHODS))
@pytest.mark.parametrize('kind', KINDS)
def test_small_solves_are_bit_identical(kind, method, dtype, mode):
    B, d = 96, 16
    name, sde_type = METHODS[method]
    sde = SDE(kind, sde_type, d, dtype).to(DEV)
    # starts on both sides of zero and of the bounds: every branch is taken
    y0 = (torch.linspace(-0.1, 0.2, B * d, dtype=torch.float64).reshape(B, d)).to(dtype=dtype, device=DEV)
    check_fused(sde, y0, 12, 2.0 ** -5, name, MODES[mode])


# ---- every new op on every pair of special values -------------------------------------------------------------------
OPS = {
    'abs': lambda a, b: a.abs(),
    'relu': lambda a, b: torch.relu(a),
    'clamp_min0': lambda a, b: a.clamp(min=0),
    'clamp_min_negzero': lambda a, b: torch.clamp_min(a, -0.0),
    'clamp_both': lambda a, b: a.clamp(-1.0, 3.0),
    'clamp_max': lambda a, b: torch.clamp_max(a, 1e-30),
    'clamp_tensor_min': lambda a, b: torch.clamp(a, min=b),
    'clamp_tensor_both': lambda a, b: torch.clamp(a, min=b, max=-b),
    'maximum': lambda a, b: torch.maximum(a, b),
    'minimum': lambda a, b: torch.minimum(a, b),
    'where_gt': lambda a, b: torch.where(a > b, a, b),
    'where_ge': lambda a, b: torch.where(a >= b, b, a),
    'where_lt_scalar': lambda a, b: torch.where(a < 1.0, a, 0.0),
    'where_le': lambda a, b: torch.where(a <= b, a, -a),
    'where_eq': lambda a, b: torch.where(a == b, a, b),
    'where_ne': lambda a, b: torch.where(a != b, a, 2.5),
    'where_logical': lambda a, b: torch.where((a > b) & ~(a < 0) | (b == 1), a, b),
    'masked_fill': lambda a, b: a.masked_fill(a < b, 2.0),
    'reciprocal': lambda a, b: torch.reciprocal(a),
    'sign': lambda a, b: torch.sign(a),
}
NO_VJP = {'sign'}  # autograd's vjp of sign is a zeros_like factory: the Milstein tape rejects it


class OpSDE(nn.Module):
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, op, where, a, b):
        super().__init__()
        self.op, self.where, self.a, self.b = op, where, nn.Parameter(a), nn.Parameter(b)

    def f(self, t, y):
        if self.where == 'g':
            return -y
        r = OPS[self.op](self.a, self.b)
        # a zero's sign survives the step's additions as the sign of an infinity
        return torch.reciprocal(r) + y if self.where == 'reciprocal_of_f' else r + y

    def g(self, t, y):
        return OPS[self.op](y, self.b) if self.where == 'g' else 0.0 * y


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('where', ['f', 'reciprocal_of_f', 'g'])
@pytest.mark.parametrize('op', sorted(OPS))
def test_each_new_op_matches_aten_on_special_values(op, where, dtype):
    """f: y0 = 0, dt = 1, g = 0*y, so y1 is f, the op on every pair of special values (rows x channels).  g: y0 is the
    grid of special values and the op is g, so y1 carries its value and autograd's vjp of it (Milstein Ito)."""
    if where == 'g' and op in NO_VJP:
        pytest.skip("the tape is rejected")
    vals = torch.tensor(SPECIAL, dtype=torch.float64).to(dtype)
    n = len(vals)
    a, b = vals.repeat_interleave(n).reshape(n * n // 4, 4), vals.repeat(n).reshape(n * n // 4, 4)
    sde = OpSDE(op, where, a.to(DEV), b.to(DEV))
    y0 = sde.a.detach().clone() if where == 'g' else torch.zeros_like(sde.a)
    ys, _ = check_fused(sde, y0, 1, 1.0, 'milstein', {'cuda_graph': True})
    if where == 'f':
        want = OPS[op](sde.a.detach(), sde.b.detach())
        got = ys[-1]
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan)
        assert torch.equal(got[~nan], want[~nan])  # (== : a -0 result comes out +0 after adding g*dW = 0)


# ---- at scale, and the adjoint ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('method', ['milstein', 'euler'])
def test_cfg2_sized_cir_graph_solve_in_chunks_is_bit_identical(method):
    B, d = 65536, 64
    sde = SDE('cir_clamp', 'ito', d, torch.float32).to(DEV)
    y0 = torch.full((B, d), 0.04, device=DEV)
    n0 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_MILSTEIN if method == 'milstein' else _cabi.KERNEL_PW_CHUNK)
    ys, _ = check_fused(sde, y0, 130, 2.0 ** -8, method, {'cuda_graph': True})
    n1 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_MILSTEIN if method == 'milstein' else _cabi.KERNEL_PW_CHUNK)
    assert 0 < n1 - n0 < 130  # chunks of up to TSDE_PW_MAX_STEPS steps
    assert (ys[-1] < 0).any()  # the truncation is reached


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_sdeint_adjoint_with_the_reversible_pair_on_cir(dtype):
    """`sdeint_adjoint`'s forward solve fuses, its backward sweep does not; ys and every gradient equal those of the
    same solve with the tape rejected."""
    B, d, T, dt = 64, 8, 20, 2.0 ** -5
    ts = torch.arange(T + 1, dtype=dtype, device=DEV) * dt
    out = []
    for ctx in (contextlib.nullcontext, unfused):
        with ctx():
            sde = SDE('cir_relu', 'stratonovich', d, dtype).to(DEV)
            y0 = torch.full((B, d), 0.05, dtype=dtype, device=DEV, requires_grad=True)
            bm = tsde.BrownianInterval(0.0, T * dt, size=(B, d), dtype=dtype, device=DEV, entropy=9)
            n0 = fused_launches()
            ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=dt)
            n1 = fused_launches()
            ys.pow(2).sum().backward()
            assert fused_launches() == n1
            assert (n1 > n0) == (ctx is contextlib.nullcontext)
            out.append([ys.detach(), y0.grad] + [p.grad for p in sde.parameters()])
            graph.drop_plans(sde)
    assert out[0][1] is not None
    for a, b in zip(*out):
        assert (a is None) == (b is None) and (a is None or same_bits(a, b))
