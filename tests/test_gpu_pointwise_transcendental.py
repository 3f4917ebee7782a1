"""Transcendental ops in the compiled element-wise kernels (options={'transcendental': True}; pointwise.py `_allow`,
csrc/pointwise.cu kPwHelpers).

Each op must give ATen's CUDA result bit for bit.  Per op, through both code generators: a program f = op(x) + 0 * y
with x a (rows, d) operand and g = 0 * y (Milstein) or (0 * y)[..., None] * S (general Euler, m = 1) is launched once at
y0 = 0, dt = 1, so y1 is op(x) exactly (a -0 read as +0), and compared with torch's op on the GPU: float32 over all
2^32 bit patterns, float64 over 2^26 random patterns and the specials; pow over the ladder's exponents and random
ones, and the backward ops over random pairs.  Then whole solves against the unfused ones (the tape rejected, the
route confirmed by the launch counters): Milstein with each op in f and in g, chunks of 1 and 64 steps, adaptive
Milstein, TanhGeneral and TanhMixedGeneral with Euler and midpoint, sra1, float32 and float64, eager and captured; and
the solves that must keep the unfused step: the same SDEs without the option, and the interpreted methods with it."""
import contextlib
import ctypes

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from . import problems
from .test_gpu_pointwise import same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ON = {'transcendental': True}

UNARY = {'exp': torch.exp, 'log': torch.log, 'sin': torch.sin, 'cos': torch.cos, 'tanh': torch.tanh,
         'log1p': torch.log1p, 'expm1': torch.expm1, 'rsqrt': torch.rsqrt, 'sigmoid': torch.sigmoid}
BACKWARD = {'tanh_backward': torch.ops.aten.tanh_backward.default,
            'sigmoid_backward': torch.ops.aten.sigmoid_backward.default}
POWERS = [0.5, -0.5, -1, 2, 3, -2, 2.5, -3, 1.7, 0.3, -1.25, 7.0, 1e-3]


class _Kernel:
    """One fused step of a program recorded from fn(*xs) + 0 * y on (rows, d) operands xs, launched directly on other
    operands of that shape: Milstein (tsde_step_milstein_pointwise) or general Euler (tsde_solve_euler_pointwise, m =
    1, g = (0 * y)[..., None] * S)."""

    def __init__(self, fn, n_args, rows, d, dtype, layout):
        self.rows, self.d, self.dtype, self.layout = rows, d, dtype, layout
        self.lib = _cabi.lib()
        y = torch.zeros(rows, d, dtype=dtype, device=DEV)
        t = torch.zeros((), dtype=dtype, device=DEV)
        xs = [torch.rand(rows, d, dtype=dtype, device=DEV) + 0.5 for _ in range(n_args)]
        S = None
        if layout == 'milstein':
            rec = pointwise.Recorder(y, t, True)
            fv = rec.segment(lambda: fn(*xs) + 0 * y)
            with torch.enable_grad():
                yg = y.detach().requires_grad_(True)
                gv = rec.segment(lambda: 0 * yg, y=yg)
                go = torch.ones_like(y)
                gdg, = rec.segment(lambda: torch.autograd.grad(gv, yg, grad_outputs=go), go=go)
            res = pointwise.compile_milstein(rec, rec.finish(fv, gv, gdg))
        else:
            S = torch.ones(d, 1, dtype=dtype, device=DEV)
            rec = pointwise.GeneralRecorder(y, t, 'fg', 1, True)
            rec.evaluation('f', lambda: fn(*xs) + 0 * y, t, y)
            rec.evaluation('g', lambda: (0 * y)[..., None] * S, t, y)
            res = rec.finish()
            if res is not None:
                assert _cabi.compile_general_pointwise(res[0], dtype, d, 1) == 0
        assert res is not None, rec.reason
        self.prog, self.keep = res[0], (xs, S)
        # the operands that are the xs, in order
        ptrs = [x.data_ptr() for x in xs]
        self.slots = [next(k for k in range(self.prog.n_operands) if self.prog.operand[k].ptr == p) for p in ptrs]
        self.y0, self.t = y, t
        self.key = torch.zeros(2, dtype=torch.int32, device=DEV)
        self.nz = _cabi.Noise(source=_cabi.SRC_COUNTER, key=self.key.data_ptr(), n_cells=1, h=1.0, h_total=1.0)
        noise = _cabi.NOISE_DIAGONAL if layout == 'milstein' else _cabi.NOISE_GENERAL
        self.L = _cabi.Launch(_cabi.dtype_code(dtype), noise, rows, d, d if layout == 'milstein' else 1,
                              torch.cuda.current_stream().cuda_stream)

    def __call__(self, *xs):
        for k, x in zip(self.slots, xs):
            assert x.shape == (self.rows, self.d) and x.is_contiguous()
            self.prog.operand[k].ptr = x.data_ptr()
        y1 = torch.empty_like(self.y0)
        if self.layout == 'milstein':
            code = self.lib.tsde_step_milstein_pointwise(ctypes.byref(self.L), ctypes.byref(self.nz),
                                                         ctypes.byref(self.prog), self.y0.data_ptr(),
                                                         self.t.data_ptr(), 1.0, 1, y1.data_ptr())
        else:
            steps = (_cabi.PwStep * 1)()
            steps[0].cell_id, steps[0].h, steps[0].dt = 0, 1.0, 1.0
            steps[0].t0, steps[0].y1 = self.t.data_ptr(), y1.data_ptr()
            code = self.lib.tsde_solve_euler_pointwise(ctypes.byref(self.L), ctypes.byref(self.nz),
                                                       ctypes.byref(self.prog), self.y0.data_ptr(), steps, 1)
        assert code == 0
        return y1


def _same_values(got, want):
    """Equal bits, with -0 read as +0 (y1 = 0 + op(x)) and every NaN equal to every NaN."""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    g, w = torch.where(nan, 0, got) + 0, torch.where(nan, 0, want) + 0  # (+ 0: -0 -> +0)
    it = torch.int32 if want.dtype == torch.float32 else torch.int64
    bad = (g.view(it) != w.view(it)).nonzero()
    assert bad.numel() == 0, (bad.shape[0], [(w[tuple(i)].item(), g[tuple(i)].item()) for i in bad[:4]])


def _specials(dtype):
    fi = torch.finfo(dtype)
    vals = [0.0, -0.0, float('inf'), -float('inf'), float('nan'), fi.tiny, -fi.tiny, fi.max, -fi.max, fi.eps,
            fi.tiny * fi.eps, -fi.tiny * fi.eps, 1.0, -1.0, 0.5, 88.72, -87.33, 709.78, -708.4, 710.0, 1e-300,
            3.141592653589793, 1e22, 1e300]
    return torch.tensor(vals, dtype=torch.float64).to(dtype)


ROWS32, D32 = 1 << 16, 1024  # a chunk of 2^26 float32 patterns


def _fp32_chunks():
    n = ROWS32 * D32
    for c in range((1 << 32) // n):
        bits = torch.arange(c * n, (c + 1) * n, dtype=torch.int64, device=DEV).to(torch.int32)
        yield bits.view(torch.float32).view(ROWS32, D32)


def _random_bits(shape, dtype, g):
    """Values of uniformly random bit patterns of `dtype`."""
    n = 1
    for s in shape:
        n *= s
    words = torch.randint(-(1 << 31), (1 << 31) - 1, (n * (dtype.itemsize // 4),), dtype=torch.int32, device=DEV,
                          generator=g)
    return words.view(dtype).view(shape)


def _fp64_inputs(n=1 << 26):
    x = _random_bits((n,), torch.float64, torch.Generator(DEV).manual_seed(7))
    s = _specials(torch.float64).to(DEV)
    x[:s.numel()] = s
    return x.view(-1, 1024)


@pytest.mark.parametrize('layout', ['milstein', 'general'])
@pytest.mark.parametrize('op', sorted(UNARY))
def test_each_op_is_aten_exactly_float32_every_pattern(op, layout):
    k = _Kernel(UNARY[op], 1, ROWS32, D32, torch.float32, layout)
    for x in _fp32_chunks():
        _same_values(k(x), UNARY[op](x))


@pytest.mark.parametrize('layout', ['milstein', 'general'])
@pytest.mark.parametrize('op', sorted(UNARY))
def test_each_op_is_aten_exactly_float64(op, layout):
    x = _fp64_inputs()
    k = _Kernel(UNARY[op], 1, x.shape[0], x.shape[1], torch.float64, layout)
    _same_values(k(x), UNARY[op](x))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('layout', ['milstein', 'general'])
def test_pow_over_the_ladder_and_other_exponents(layout, dtype):
    g = torch.Generator(DEV).manual_seed(3)
    rows, d = 4096, 1024
    x = torch.cat([torch.rand(rows // 2, d, device=DEV, generator=g, dtype=dtype) * 8,
                   torch.randn(rows // 2, d, device=DEV, generator=g, dtype=dtype) * 4])
    x.view(-1)[:24] = _specials(dtype).to(DEV)
    exps = POWERS + [float(e) for e in (torch.rand(6, generator=torch.Generator().manual_seed(5)) * 10 - 5)]
    for p in exps:
        k = _Kernel(lambda a, p=p: a ** p, 1, rows, d, dtype, layout)
        _same_values(k(x), x ** p)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('layout', ['milstein', 'general'])
@pytest.mark.parametrize('op', sorted(BACKWARD))
def test_the_backward_ops_over_random_pairs(op, layout, dtype):
    g = torch.Generator(DEV).manual_seed(4)
    rows, d = 16384, 1024
    a = _random_bits((rows, d), dtype, g)
    b = torch.cat([torch.rand(rows // 2, d, device=DEV, generator=g, dtype=dtype) * 2 - 1,
                   _random_bits((rows // 2, d), dtype, g)])
    k = _Kernel(BACKWARD[op], 2, rows, d, dtype, layout)
    _same_values(k(a, b), BACKWARD[op](a, b))


# -- whole solves ---------------------------------------------------------------------------------------------------
def launches(kernel):
    return _cabi.lib().tsde_kernel_launches(kernel)


@contextlib.contextmanager
def unfused():
    """Every tape rejected: each step runs the user's ops and the unfused kernels."""
    finish, srk_finish = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = finish, srk_finish


class Diagonal(nn.Module):
    noise_type = 'diagonal'

    def __init__(self, op, where, sde_type, d, dtype):
        super().__init__()
        self.op, self.where, self.sde_type = op, where, sde_type
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter((torch.rand(d, generator=gen, dtype=torch.float64) - 0.5).to(dtype))
        self.sigma = nn.Parameter((torch.rand(d, generator=gen, dtype=torch.float64) * 0.3 + 0.1).to(dtype))

    def _fn(self, y):
        return (lambda a: a ** 1.5)(y) if self.op == 'pow' else UNARY[self.op](y)

    def f(self, t, y):
        return self.mu * self._fn(y) if self.where == 'f' else self.mu * y

    def g(self, t, y):
        return self.sigma * self._fn(y) if self.where == 'g' else self.sigma * y


def _solve(sde, y0, T, dt, method, options, m=None, adaptive=False):
    B, d = y0.shape
    size = (B, m if m is not None else d)
    levy = 'space-time' if method == 'srk' else 'none'  # (SRK needs the space-time Levy area)
    bm = tsde.BrownianInterval(0.0, T * dt, size=size, dtype=y0.dtype, device=DEV, entropy=11,
                               levy_area_approximation=levy)
    ts = torch.arange(T + 1, dtype=y0.dtype, device=DEV) * dt
    with torch.no_grad():
        kw = dict(adaptive=True, rtol=1e-3, atol=1e-4) if adaptive else {}
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=dict(options), **kw)
    graph.drop_plans(sde)
    return ys


def check(kernels, sde, y0, T, dt, method, options, **kw):
    n0 = sum(launches(k) for k in kernels)
    ys = _solve(sde, y0, T, dt, method, options, **kw)
    assert sum(launches(k) for k in kernels) > n0, "the steps were not fused"
    with unfused():
        ref = _solve(sde, y0, T, dt, method, options, **kw)
    assert same_bits(ys, ref)


MILSTEIN_OPS = sorted(UNARY) + ['pow']


@pytest.mark.parametrize('chunk', [1, 64])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('where', ['f', 'g'])
@pytest.mark.parametrize('op', MILSTEIN_OPS)
def test_milstein_solves_are_bit_identical(op, where, dtype, chunk, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: chunk)
    B, d = 96, 16
    y0 = torch.full((B, d), 0.4, dtype=dtype, device=DEV)
    for mode in ({}, {'cuda_graph': True}):
        check([_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_CHUNK], Diagonal(op, where, 'ito', d, dtype).to(DEV), y0, 70, 2.0 ** -7, 'milstein', dict(ON, **mode))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('op', ['tanh', 'sigmoid', 'sin'])
def test_adaptive_milstein_is_bit_identical(op, dtype):
    B, d = 64, 8
    y0 = torch.full((B, d), 0.4, dtype=dtype, device=DEV)
    check([_cabi.KERNEL_PW_ADAPTIVE], Diagonal(op, 'g', 'stratonovich', d, dtype).to(DEV), y0, 16, 2.0 ** -4,
          'milstein', ON, adaptive=True)


@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', [1, 3, 16, 32])
@pytest.mark.parametrize('method', ['euler', 'midpoint'])
@pytest.mark.parametrize('kind', ['TanhGeneral', 'TanhMixedGeneral'])
def test_tanh_general_solves_are_bit_identical(kind, method, m, dtype, mode):
    B, d = 96, 8
    sde_type = 'ito' if method == 'euler' else 'stratonovich'
    sde = getattr(problems, kind)(d, m, sde_type, dtype=dtype).to(DEV)
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    options = dict(ON, cuda_graph=True) if mode == 'graph' else ON
    check([_cabi.KERNEL_PW_GENERAL], sde, y0, 70, 2.0 ** -7, method, options, m=m)


class ExpAdditive(nn.Module):
    noise_type, sde_type = 'additive', 'ito'

    def __init__(self, d, m, dtype):
        super().__init__()
        gen = torch.Generator().manual_seed(1)
        self.a = nn.Parameter((torch.rand(d, m, generator=gen, dtype=torch.float64) * 0.5).to(dtype))
        self.mu = nn.Parameter((torch.rand(d, generator=gen, dtype=torch.float64) - 0.5).to(dtype))

    def f(self, t, y):
        return self.mu * torch.sin(y)

    def g(self, t, y):
        return (self.a * torch.exp(-t)).expand(y.shape[0], *self.a.shape)


@pytest.mark.parametrize('mode', ['eager', 'graph'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_sra1_is_bit_identical(dtype, mode):
    B, d, m = 64, 8, 3
    y0 = torch.full((B, d), 0.3, dtype=dtype, device=DEV)
    options = dict(ON, cuda_graph=True) if mode == 'graph' else ON
    check([_cabi.KERNEL_PW_GENERAL], ExpAdditive(d, m, dtype).to(DEV), y0, 20, 2.0 ** -5, 'srk', options, m=m)


ALL = [_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_SRK, _cabi.KERNEL_PW_PC, _cabi.KERNEL_PW_CHUNK,
       _cabi.KERNEL_PW_ADAPTIVE, _cabi.KERNEL_PW_GENERAL]


@pytest.mark.parametrize('case', ['milstein', 'general', 'srk', 'heun', 'euler', 'reversible_heun', 'euler_heun'])
@pytest.mark.parametrize('option', [False, True])
def test_the_solves_that_keep_the_unfused_step(case, option):
    """Without the option nothing fuses; with it the interpreted methods still keep the unfused step, bit for bit."""
    if case in ('milstein', 'general') and option:
        pytest.skip('fused with the option (above)')
    B, d, m = 64, 8, 4
    options = ON if option else {}
    y0 = torch.full((B, d), 0.3, device=DEV)
    if case == 'general':
        sde, method, mm = problems.TanhGeneral(d, m, 'ito', dtype=torch.float32).to(DEV), 'euler', m
    else:
        method = case
        sde_type = 'ito' if case in ('milstein', 'srk', 'euler') else 'stratonovich'
        sde, mm = Diagonal('tanh', 'g', sde_type, d, torch.float32).to(DEV), None
    before = [launches(k) for k in ALL]
    ys = _solve(sde, y0, 12, 2.0 ** -5, method, options, m=mm)
    assert [launches(k) for k in ALL] == before
    with unfused():
        ref = _solve(sde, y0, 12, 2.0 ** -5, method, options, m=mm)
    assert same_bits(ys, ref)
