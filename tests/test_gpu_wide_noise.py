"""General-noise entry points at Brownian widths whose increments do not fit in shared memory.

`gen_kernel` stages one row's W (and U) in 40 KiB of shared memory, so m * s * (U ? 2 : 1) > 40 KiB takes
`gen_wide_kernel` (csrc/tableau_general.cu), which walks m in chunks.  Its first m per column:

    state     without U (Euler, Heun, midpoint, Euler-Heun, reversible Heun, adjoint halves)   with U (SRK additive)
    float32   10241                                                                            5121
    float64   5121                                                                             2561

Checked with the float64 harness of test_gpu_general_paths.py (every row within 4 (m + 16) u S of the entry point's
formula on the oracle's increments, every slot written, sentinels intact), the route confirmed by the launch counters
(TSDE_KERNEL_GEN_WIDE advanced, neither tile kernel); then bit-exact batch sharding, 16-bit operands equal to the
widened float32 launch, and whole solves through `sdeint` / `sdeint_adjoint`.
"""
import ctypes
import warnings

import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from . import helpers
from . import problems
from .helpers import GENERAL_OPS
from .test_gpu_general_paths import (CELL, KEY, NONE, _Report, _run_shapes, bound, formula, increments,  # noqa: F401
                                     operands)
from .test_gpu_mixed_precision import HALF, _assert_pair, _run_pair

pytestmark = pytest.mark.gpu

DEV = 'cuda'
GEN_WIDE = 2                                     # TSDE_KERNEL_GEN_WIDE
ALL = list(GENERAL_OPS)
U_OPS = [op for op in ALL if GENERAL_OPS[op].want_u]
W_OPS = [op for op in ALL if not GENERAL_OPS[op].want_u]
# the first wide m and the last m gen_kernel stages, per (dtype, U)
FIRST_WIDE = {(torch.float32, False): 10244, (torch.float32, True): 5124,
              (torch.float64, False): 5124, (torch.float64, True): 2564}
LAST_STAGED = {(torch.float32, False): 10240, (torch.float32, True): 5120,
               (torch.float64, False): 5120, (torch.float64, True): 2560}
DTYPES = pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])


def wide_launches():
    return _cabi.lib().tsde_kernel_launches(GEN_WIDE)


def _run_wide(label, dtype, shapes, report, bad, wide=True, **kw):
    """_run_shapes, one shape at a time, also checking that every tile launch took gen_wide_kernel (or, wide=False,
    that none did)."""
    for shape in shapes:
        B, d, m, ops, expect, g_shift, w_shift = shape
        n_src = 1 if w_shift else len(kw.get('sources', ('counter1', 'counter3', 'memory')))
        before = wide_launches()
        _run_shapes(label, dtype, [shape], report, bad, **kw)
        got, want = wide_launches() - before, n_src * len(ops) if wide else 0
        if got != want:
            bad.append(f'{label} B={B} d={d} m={m}: {got} gen_wide_kernel launches, expected {want}')


def _wide_shapes(dtype):
    mw, mu = FIRST_WIDE[(dtype, False)], FIRST_WIDE[(dtype, True)]
    return [(37, 7, mw, ALL, NONE, 0, 0), (37, 7, mu, U_OPS, NONE, 0, 0),
            (1, 300, mw, ALL, NONE, 0, 0), (1000, 1, mw, ALL, NONE, 0, 0),
            (2, 1100, mw, ALL, NONE, 0, 0),            # more outputs than one block's running sums: two d blocks
            (37, 7, 10243, ALL, NONE, 0, 0),           # prime m: the last quad partial, scalar g loads
            (5, 3, 262147, ALL, NONE, 0, 0),           # many chunks, small d
            (37, 7, mw, ALL, NONE, 1, 0),              # g one element off 16-byte alignment
            (21, 7, mw, ALL, NONE, 0, 1)]              # memory-noise W / U one element off alignment


@DTYPES
def test_wide_route_vs_formula(dtype):
    """Every entry point at the first wide m of its column, a prime m, a very wide m, d in {1, 7, 300, 1100},
    B in {1, 37, 1000}, every noise source, unaligned g and W / U: within the bound, on gen_wide_kernel."""
    report, bad = _Report(), []
    _run_wide('wide', dtype, _wide_shapes(dtype), report, bad)
    report.print()
    assert not bad, '\n'.join(bad)


@DTYPES
def test_last_staged_width_keeps_gen_kernel(dtype):
    """The widest rows gen_kernel can stage stay on it: no tile-kernel counter advances (CTA, TMA or wide)."""
    report, bad = _Report(), []
    shapes = [(37, 7, LAST_STAGED[(dtype, False)], W_OPS, NONE, 0, 0),
              (37, 7, LAST_STAGED[(dtype, True)], U_OPS, NONE, 0, 0)]
    _run_wide('staged', dtype, shapes, report, bad, wide=False)
    report.print()
    assert not bad, '\n'.join(bad)


@DTYPES
def test_wide_broadcast_g_and_row_offset_vs_formula(dtype):
    """A batch-broadcast g (one (d, m) block) for the entry points that accept it, and row_offset = 2^32 - 1 - B."""
    report, bad = _Report(), []
    mw, mu = FIRST_WIDE[(dtype, False)], FIRST_WIDE[(dtype, True)]
    ops = helpers.GENERAL_BROADCAST_OPS
    _run_wide('wide+bcast', dtype, [(37, 7, mw, ops, NONE, 0, 0), (1000, 5, mu, [o for o in ops if o in U_OPS], NONE,
                                                                   0, 0)], report, bad, bcast=True)
    _run_wide('wide@2^32', dtype, [(37, 7, mw, ALL, NONE, 0, 0)], report, bad, near_limit=True)
    report.print()
    assert not bad, '\n'.join(bad)


# ---- batch sharding ------------------------------------------------------------------------------------------------
def _launch(op, dtype, rows, d, m, ins, outs, nz):
    helpers.general_call(op, dtype, rows, d, m, [x.data_ptr() for x in ins], nz, [o.data_ptr() for o in outs])


@DTYPES
@pytest.mark.parametrize('op', ALL)
def test_wide_sharding_is_bit_exact(op, dtype):
    """One launch over B rows equals two launches over rows [0, k) and [k, B) with row_offset advanced by k, bit for
    bit (counter noise over three cells): the summation order depends on m alone."""
    spec = GENERAL_OPS[op]
    B, d, k = 9, 5, 4
    m = FIRST_WIDE[(dtype, spec.want_u)] + 3
    E, G = operands(B, d, m, dtype, DEV, seed=17)
    it_e, it_g = iter(E), iter(G)
    ins = [next(it_e) if a == 'e' else next(it_g) for a in spec.args]
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    cell_h = torch.tensor([2.0 ** -8, 3 * 2.0 ** -8, 2.0 ** -7], dtype=torch.float64, device=DEV)
    shape = {'e': (B, d), 'g': (B, d, m)}
    one = [torch.full(shape[o], float('nan'), device=DEV, dtype=dtype) for o in spec.outs]
    two = [torch.full(shape[o], float('nan'), device=DEV, dtype=dtype) for o in spec.outs]
    R0 = 1000

    def noise(offset):
        return helpers.general_noise(key=key, cell_id=CELL, h=2.0 ** -8, h_total=2.0 ** -6, cell_h=cell_h,
                                     row_offset=offset, want_u=spec.want_u)

    before = wide_launches()
    _launch(op, dtype, B, d, m, ins, one, noise(R0))
    for lo, hi in ((0, k), (k, B)):
        _launch(op, dtype, hi - lo, d, m, [x[lo:hi] for x in ins], [o[lo:hi] for o in two], noise(R0 + lo))
    torch.cuda.synchronize()
    assert wide_launches() - before == 3
    for a, b in zip(one, two):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)


# ---- 16-bit f / g ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('src', ['counter', 'memory'])
@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name', ALL)
def test_wide_16bit_equals_widened_launch(name, half, src):
    """Mixed<Op> on gen_wide_kernel: 16-bit f / g, 8-byte aligned (64-bit quad loads) and 2-byte aligned (scalar
    loads), and a broadcast g where the entry point accepts one, equal the float32 launch on widened copies."""
    m = FIRST_WIDE[(torch.float32, GENERAL_OPS[name].want_u)] + 4
    cases = [dict(), dict(misalign=1)]
    if name in helpers.GENERAL_BROADCAST_OPS:
        cases.append(dict(bcast=True))
    for kw in cases:
        before = wide_launches()
        _assert_pair(_run_pair(name, half, src, ('wide', 'general', 33, 5, m), **kw), (name, kw))
        assert wide_launches() - before == 2, (name, kw)


# ---- whole solves ----------------------------------------------------------------------------------------------------
def _tanh_general(d, m, sde_type, dtype):
    """TanhGeneral with S scaled by 1/sqrt(m): the noise term of a step stays O(1) at any width."""
    sde = problems.make('general', d, m, sde_type, dtype=dtype, seed=4).to(DEV)
    with torch.no_grad():
        sde.S.mul_(m ** -0.5)
    return sde


def _solve(sde, y0, ts, m, method, levy='none', options=None):
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(y0.shape[0], m), dtype=y0.dtype, device=DEV, entropy=7,
                               levy_area_approximation=levy)
    return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -4, options=options)


SOLVES = [('euler', 'ito', 'general', torch.float32, 10244, 'none'),
          ('midpoint', 'stratonovich', 'general', torch.float32, 10244, 'none'),
          ('srk', 'ito', 'additive_expand', torch.float64, 2564, 'space-time')]


@pytest.mark.parametrize('method,sde_type,kind,dtype,m,levy', SOLVES, ids=[s[0] for s in SOLVES])
def test_wide_solve(method, sde_type, kind, dtype, m, levy):
    """Eager equals the CUDA graph bit for bit with no fallback warning, both on gen_wide_kernel, and both agree with
    the grad-tracked solve (g.dW formed with torch.bmm) to rounding."""
    B, d = 64, 8
    sde = _tanh_general(d, m, sde_type, dtype) if kind == 'general' else \
        problems.make(kind, d, m, sde_type, dtype=dtype, seed=4).to(DEV)
    y0 = torch.rand(B, d, dtype=dtype, device=DEV)
    ts = torch.tensor([0.0, 0.25, 0.5], dtype=dtype, device=DEV)
    before = wide_launches()
    with torch.no_grad():
        eager = _solve(sde, y0, ts, m, method, levy)
    assert wide_launches() > before
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter('always')
        with torch.no_grad():
            graph = _solve(sde, y0, ts, m, method, levy, options={'cuda_graph': True})
    assert not [w for w in seen if 'torchsde_b200' in str(w.message)], [str(w.message) for w in seen]
    assert torch.equal(eager, graph)
    tracked = _solve(sde, y0.clone().requires_grad_(), ts, m, method, levy).detach()
    tol = dict(rtol=1e-4, atol=1e-4) if dtype == torch.float32 else dict(rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(eager, tracked, **tol)


def test_wide_adjoint_reversible_heun_equals_backprop():
    """sdeint_adjoint with the reversible pair at a wide m (both adjoint halves on gen_wide_kernel): the gradients
    equal those of backpropagating through sdeint, to rounding."""
    B, d, m = 5, 4, FIRST_WIDE[(torch.float64, False)]
    sde = _tanh_general(d, m, 'stratonovich', torch.float64)
    params = list(sde.parameters())
    y0 = (0.2 + 0.3 * torch.rand(B, d, dtype=torch.float64, device=DEV)).requires_grad_(True)
    ts = torch.tensor([0.0, 0.125, 0.25], dtype=torch.float64, device=DEV)
    out = []
    for adjoint in (True, False):
        bm = tsde.BrownianInterval(0.0, 0.25, size=(B, m), dtype=torch.float64, device=DEV, entropy=21)
        before = wide_launches()
        if adjoint:
            ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun',
                                     adjoint_method='adjoint_reversible_heun', dt=2.0 ** -4)
        else:
            ys = tsde.sdeint(sde, y0, ts, bm=bm, method='reversible_heun', dt=2.0 ** -4)
        grads = torch.autograd.grad((ys ** 2).sum(), [y0] + params)
        if adjoint:
            assert wide_launches() > before
        out.append((ys.detach(), grads))
    torch.testing.assert_close(out[0][0], out[1][0], rtol=1e-12, atol=1e-12)
    for a, b in zip(out[0][1], out[1][1]):
        torch.testing.assert_close(a, b, rtol=1e-8, atol=1e-10)


def test_wide_empty_batch_is_a_noop():
    """B = 0 at a wide m launches nothing and returns success (its operand pointers may be NULL)."""
    before = wide_launches()
    for op in ALL:
        spec = GENERAL_OPS[op]
        key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
        nz = helpers.general_noise(key=key, cell_id=CELL, want_u=spec.want_u)
        L = _cabi.make_launch(torch.float32, _cabi.NOISE_GENERAL, 0, 7, 20000)
        rc = getattr(_cabi.lib(), op)(ctypes.byref(L), ctypes.byref(nz), *([None] * len(spec.args)), *spec.scalars,
                                      *([None] * len(spec.outs)))
        assert rc == 0, op
    assert wide_launches() == before
