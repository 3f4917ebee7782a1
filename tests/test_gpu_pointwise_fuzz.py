"""Fused element-wise solves of random SDEs (tests/pointwise_fuzz.py) against the same solves unfused, on the bits.

For a fixed list of seeds per layout, each case's solve runs fused and then with every tape rejected (`unfused`: the
recorders' `finish` return None), and the two must have the same bits, NaN, infinities and signed zeros included.  The
launch counter of the layout's kernel family confirms the fused route; a case whose tape is rejected (drawn at the
limits: too long or too wide) must still give the unfused bits, and at most REJECTED_SHARE of a layout's cases may be
rejected.  Covered: Milstein Ito and Stratonovich in chunks of 1 and TSDE_PW_MAX_STEPS; SRK, Heun, midpoint and
Euler-Heun; Euler and reversible Heun in chunks; the adaptive proposals of Euler, Milstein, SRK, Heun, midpoint and
Euler-Heun; general-noise Euler and midpoint at m in {1, 3, 4, 5, 16, 32}; additive-noise SRK (sra1); float32 and
float64; in every fixed-step sweep each d in {1, 2, 3, 5, 7, 12, 16, 33} (1 to 9 quads per row, both row-index paths,
every tail, the vector and element loads) in both dtypes, with a batch that is not a multiple of 256 quads; eager and
cuda_graph solves, a Brownian grid finer than the step and interpolated outputs on a subset; and row_split graph
solves of cases without (rows, d) parameters.  And one plain high-precision reference: fp64 Euler, Milstein, midpoint,
SRK and sra1 solves of small cases against oracle/solvers.py on the oracle's increments of the same Brownian motion."""
import contextlib

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph, pointwise
from oracle import solvers
from . import helpers, problems
from . import pointwise_fuzz as fz
from .test_gpu_pointwise import same_bits

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DT = 2.0 ** -5
T = 12
DIMS = [1, 2, 3, 5, 7, 12, 16, 33]
TOO_BIG = ('program too long', 'too many live values')
REJECTED_SHARE = 0.25  # of a layout's cases: the limits class is 15 % of the draws, and some of it fits
# (row_split solves run apart, on cases without (rows, d) parameters: test_row_split_graph_solves)
MODES = [{}, {}, {'cuda_graph': True}, {}, {'cuda_graph': True, 'static_output': False}, {}]


@contextlib.contextmanager
def unfused():
    """Every tape rejected: each step runs the user's ops and the unfused kernels."""
    saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


def launches(kernels):
    return sum(_cabi.lib().tsde_kernel_launches(k) for k in kernels)


def _y0(case, B, d, dtype):
    if case.size == 'edge':
        return fz.edge_state(B, d, dtype, case.seed).to(DEV)
    gen = torch.Generator().manual_seed(case.seed)
    return (torch.rand(B, d, generator=gen, dtype=torch.float64) * 3 - 1.5).to(dtype=dtype, device=DEV)


def _solve(sde, y0, method, options, m=None, adaptive=False, bm_dt=None, interpolated=False):
    B, d = y0.shape
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, T * DT, size=(B, m or d), dtype=y0.dtype, device=DEV, entropy=13,
                               levy_area_approximation=levy, dt=bm_dt)
    if interpolated:
        ts = torch.tensor([0.0, 3.5 * DT, 7.25 * DT, T * DT], dtype=y0.dtype, device=DEV)
    else:
        ts = torch.arange(T + 1, dtype=y0.dtype, device=DEV) * DT
    kw = dict(adaptive=True, rtol=1e-3, atol=1e-4, dt_min=1e-4) if adaptive else {}
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=DT, options=dict(options), **kw)
    graph.drop_plans(sde)
    return ys


@contextlib.contextmanager
def reasons():
    """The reasons the recorders give for rejecting a tape, in order."""
    seen, reject = [], pointwise.Recorder.reject

    def logged(self, reason):
        seen.append(reason)
        reject(self, reason)
    pointwise.Recorder.reject = logged
    try:
        yield seen
    finally:
        pointwise.Recorder.reject = reject


def run(case, method, sde_type, kernels, dtype, d, B, m=None, options=(), **kw):
    """The case's solve fused and unfused: same bits; returns (whether it was fused, the rejection reasons)."""
    options = dict(options, **({'transcendental': True} if case.transcendental else {}))
    sde = fz.FuzzSDE(case, sde_type, B, d, m, dtype, DEV)
    y0 = _y0(case, B, d, dtype)
    n0 = launches(kernels)
    with reasons() as why:
        ys = _solve(sde, y0, method, options, m, **kw)
    fused = launches(kernels) > n0
    with unfused():
        n1 = launches(kernels)
        ref = _solve(sde, y0, method, options, m, **kw)
        assert launches(kernels) == n1
    assert same_bits(ys, ref), f'{case!r}\n{case.source()}\n{method} {dtype} d={d} B={B} m={m} {options} {kw}'
    return fused, why


def sweep(layout, seeds, method, sde_type, kernels, extra=lambda i: {}, m=None, cover=False, row_params=True):
    """Cases `seeds` of `layout` through `method`, the i-th at d = DIMS[i % 8] and in float32 or float64 as i and
    i // 8 say, so 16 seeds run every d in both dtypes (`cover` asserts that they did), and the modes in turn; asserts
    the rejected share."""
    rejected, ran = 0, set()
    for i, seed in enumerate(seeds):
        case = fz.case(seed, layout, row_params=row_params)
        d = DIMS[i % len(DIMS)]
        dtype = torch.float32 if (i + i // len(DIMS)) % 2 == 0 else torch.float64
        B = 306 + 12 * i  # (twice an odd number: B * quads per row is not a multiple of 256; a multiple of 3)
        kw = dict(options=MODES[i % len(MODES)])
        kw.update(extra(i))
        fused, why = run(case, method, sde_type, kernels, dtype, d, B, m, **kw)
        ran.add((d, dtype))
        if not fused:
            rejected += 1
            assert case.size == 'limits' and any(w in str(why) for w in TOO_BIG), \
                f'{case!r}\n{case.source()}\nwas not fused: {why} ({method} {dtype} d={d} B={B} m={m} {kw})'
    assert rejected <= max(1, int(REJECTED_SHARE * len(seeds))), rejected
    if cover:
        assert ran == {(d, t) for d in DIMS for t in (torch.float32, torch.float64)}, sorted(ran, key=str)


SEEDS = list(range(16))  # every d of DIMS in both dtypes
CHUNK = _cabi.PW_MAX_STEPS


@pytest.mark.parametrize('chunk', [1, CHUNK])
@pytest.mark.parametrize('sde_type', ['ito', 'stratonovich'])
def test_milstein(sde_type, chunk, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: chunk)
    sweep('milstein', SEEDS, 'milstein', sde_type, [_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_CHUNK], cover=True)


def _subset(i):
    """A finer Brownian grid on one case in four, interpolated outputs on another (eager solves)."""
    return {'bm_dt': DT / 2} if i % 4 == 1 else {'interpolated': True} if i % 4 == 3 else {}


@pytest.mark.parametrize('method,layout,sde_type,kernel', [
    ('srk', 'srk', 'ito', _cabi.KERNEL_PW_SRK), ('heun', 'pc', 'stratonovich', _cabi.KERNEL_PW_PC),
    ('midpoint', 'pc', 'stratonovich', _cabi.KERNEL_PW_PC),
    ('euler_heun', 'euler_heun', 'stratonovich', _cabi.KERNEL_PW_PC)])
def test_interpreted_steps(method, layout, sde_type, kernel):
    sweep(layout, SEEDS, method, sde_type, [kernel], _subset, cover=True)


@pytest.mark.parametrize('method,sde_type', [('euler', 'ito'), ('reversible_heun', 'stratonovich')])
def test_euler_and_reversible_heun_chunks(method, sde_type, monkeypatch):
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: CHUNK)
    sweep('euler', SEEDS, method, sde_type, [_cabi.KERNEL_PW_CHUNK], _subset, cover=True)


@pytest.mark.parametrize('method,layout,sde_type,kernel', [
    ('milstein', 'milstein', 'ito', _cabi.KERNEL_PW_MILSTEIN), ('srk', 'srk', 'ito', _cabi.KERNEL_PW_SRK),
    ('heun', 'pc', 'stratonovich', _cabi.KERNEL_PW_PC), ('euler', 'euler', 'ito', _cabi.KERNEL_PW_CHUNK),
    ('reversible_heun', 'euler', 'stratonovich', _cabi.KERNEL_PW_CHUNK)])
def test_row_split_graph_solves(method, layout, sde_type, kernel):
    """Captured solves split into three row blocks, on cases without (rows, d) parameters (a block's f and g read a
    block of the state, so a batch-sized parameter would not broadcast)."""
    sweep(layout, [200, 201, 202, 203], method, sde_type, [kernel, _cabi.KERNEL_PW_CHUNK],
          lambda i: {'options': {'cuda_graph': True, 'row_split': 3}}, row_params=False)


@pytest.mark.parametrize('method,layout,sde_type', [
    ('euler', 'euler', 'ito'), ('milstein', 'milstein', 'ito'), ('srk', 'srk', 'ito'), ('heun', 'pc', 'stratonovich'),
    ('midpoint', 'pc', 'stratonovich'), ('euler_heun', 'euler_heun', 'stratonovich')])
def test_adaptive_proposals(method, layout, sde_type):
    seeds = [s for s in range(40) if fz.case(s, layout).size in ('small', 'medium')][:4]
    sweep(layout, seeds, method, sde_type, [_cabi.KERNEL_PW_ADAPTIVE], lambda i: {'adaptive': True, 'options': {}})


@pytest.mark.parametrize('m', [1, 3, 4, 5, 16, 32])
@pytest.mark.parametrize('method,layout,sde_type', [('euler', 'general_euler', 'ito'),
                                                    ('midpoint', 'general_midpoint', 'stratonovich')])
def test_general_noise(method, layout, sde_type, m):
    sweep(layout, [m, m + 40, m + 80], method, sde_type, [_cabi.KERNEL_PW_GENERAL], m=m)


@pytest.mark.parametrize('m', [1, 3, 4, 5, 16, 32])
def test_additive_sra1(m):
    sweep('sra', [m, m + 40], 'srk', 'ito', [_cabi.KERNEL_PW_GENERAL],
          lambda i: {'bm_dt': DT / 2} if i == 1 else {}, m=m)


# -- against the oracle ---------------------------------------------------------------------------------------------
ORACLE = {'euler': ('euler', 'ito', 'euler'), 'milstein': ('milstein', 'ito', 'milstein'),
          'midpoint': ('pc', 'stratonovich', 'midpoint'), 'srk': ('srk', 'ito', 'srk'), 'sra1': ('sra', 'ito', 'srk')}


@pytest.mark.parametrize('name', sorted(ORACLE))
def test_fp64_solves_match_the_oracle_on_its_increments(name):
    """Every value of a small case is bounded (|v| <= 8) and its ops are Lipschitz between branch points, so the fused
    fp64 solve and the oracle's float64 one, which round the same ops in other orders (the solver's tableau, ATen's CPU
    kernels), differ by a few hundred roundings of 2^-53 at most, amplified by the case's Lipschitz bound (at most 8^3
    over a step): well below the 1e-9 tolerance, and far below the step's effect on y."""
    layout, sde_type, method = ORACLE[name]
    B, d, m = 64, 5, (3 if layout == 'sra' else None)
    seed = next(s for s in range(100) if not fz.case(s, layout, 'small', transcendental=False).transcendental
                and fz.case(s, layout, 'small', transcendental=False).f_out != 'y')
    case = fz.case(seed, layout, 'small', transcendental=False)
    sde = fz.FuzzSDE(case, sde_type, B, d, m, torch.float64, DEV)
    gen = torch.Generator().manual_seed(seed)
    y0 = (torch.rand(B, d, generator=gen, dtype=torch.float64) - 0.5).to(DEV)
    ts = torch.tensor([0.0, 4 * DT, 8 * DT], dtype=torch.float64, device=DEV)
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, 8 * DT, size=(B, m or d), dtype=torch.float64, device=DEV, entropy=404,
                               levy_area_approximation=levy)
    kernels = [_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_SRK, _cabi.KERNEL_PW_PC, _cabi.KERNEL_PW_CHUNK,
               _cabi.KERNEL_PW_GENERAL]
    n0 = launches(kernels)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=DT)
    assert launches(kernels) > n0, f'{case!r} was not fused'
    rows = np.arange(B)
    cpu = fz.FuzzSDE(case, sde_type, B, d, m, torch.float64, 'cpu')
    ref, _ = solvers.make(method, problems.NumpySDE(cpu), helpers.oracle_grid_bm(bm, rows, m or d, np.float64,
                                                                                  method == 'srk'),
                          DT).integrate(y0.cpu().numpy(), ts.cpu().numpy())
    got = ys.cpu().numpy()
    assert np.isfinite(got).all() and np.abs(got[-1] - got[0]).max() > 1e-3
    np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9, err_msg=f'{case!r}\n{case.source()}')
