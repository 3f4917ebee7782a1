"""An adaptive solve's proposals as one kernel (tsde_adaptive_proposal_pointwise, pointwise.propose).

Every output of a fused adaptive solve must have the bits of the same solve with the tape rejected (the recorders'
`finish` patched to return None), so its accept / reject history and its Brownian queries are the unfused solve's
too.  The route is confirmed by the proposal kernel's launch counter (TSDE_KERNEL_PW_ADAPTIVE), which must stay
still on the unfused solve.  Covered: Euler, Milstein (Ito and Stratonovich), SRK, Heun, midpoint and Euler-Heun, in
float32 and float64, on GBM, OU with (d,) parameters, full-truncation CIR (clamp) and a torch.where drift; tolerances
that reject proposals; outputs between accepted steps (interpolated); a solve that hits dt_min; BrownianInterval,
BrownianTree and BrownianPath; and `sdeint_adjoint(adaptive=True)`, whose solution and gradients must equal the
unfused ones."""
import contextlib
import warnings

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import base_solver, pointwise
from .test_gpu_pointwise import SDE as BasicSDE, same_bits
from .test_gpu_pointwise_select import SDE as SelectSDE

pytestmark = pytest.mark.gpu
DEV = 'cuda'
# method -> (sdeint method, sde_type)
METHODS = {'euler': ('euler', 'ito'), 'milstein_ito': ('milstein', 'ito'),
           'milstein_strat': ('milstein', 'stratonovich'), 'srk': ('srk', 'ito'), 'heun': ('heun', 'stratonovich'),
           'midpoint': ('midpoint', 'stratonovich'), 'euler_heun': ('euler_heun', 'stratonovich')}
KINDS = ['gbm', 'ou', 'cir_clamp', 'where']


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE)


@contextlib.contextmanager
def unfused():
    """The tape is always rejected: every proposal runs the user's ops and the unfused kernels three times."""
    saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


@contextlib.contextmanager
def errors():
    """The error estimate of every proposal, in order."""
    seen, real = [], base_solver.BaseSDESolver._error_estimate

    def estimate(self, y_full, y_half):
        err = real(self, y_full, y_half)
        seen.append(err)
        return err
    base_solver.BaseSDESolver._error_estimate = estimate
    try:
        yield seen
    finally:
        base_solver.BaseSDESolver._error_estimate = real


def make_sde(kind, sde_type, B, d, dtype):
    if kind in ('gbm', 'ou'):
        return BasicSDE(kind, sde_type, B, d, dtype).to(DEV)
    return SelectSDE(kind, sde_type, d, dtype).to(DEV)


def make_bm(which, B, d, dtype, T, levy):
    if which == 'interval':
        return tsde.BrownianInterval(0.0, T, size=(B, d), dtype=dtype, device=DEV, entropy=7,
                                     levy_area_approximation=levy)
    w0 = torch.zeros(B, d, dtype=dtype, device=DEV)
    if which == 'tree':
        return tsde.BrownianTree(t0=0.0, w0=w0, t1=T, entropy=7)
    np.random.seed(7)  # (BrownianPath draws its entropy from numpy)
    return tsde.BrownianPath(t0=0.0, w0=w0)


def solve(kind, method, dtype, B=64, d=16, ts=(0.0, 0.13, 0.25), dt=0.25, rtol=1e-3, atol=1e-4, dt_min=1e-5,
          bm='interval', y0=0.2):
    name, sde_type = METHODS[method]
    sde = make_sde(kind, sde_type, B, d, dtype)
    levy = 'space-time' if method == 'srk' else 'none'
    ts = torch.tensor(ts, dtype=dtype, device=DEV)
    y = torch.full((B, d), y0, dtype=dtype, device=DEV)
    with torch.no_grad(), errors() as errs:
        ys = tsde.sdeint(sde, y, ts, bm=make_bm(bm, B, d, dtype, float(ts[-1]), levy), method=name, dt=dt,
                         adaptive=True, rtol=rtol, atol=atol, dt_min=dt_min)
    return ys, errs


def check_fused(*args, **kw):
    n0 = fused_launches()
    ys, errs = solve(*args, **kw)
    assert fused_launches() > n0, "the proposals were not fused"
    with unfused():
        n1 = fused_launches()
        ref, ref_errs = solve(*args, **kw)
        assert fused_launches() == n1
    assert errs == ref_errs
    assert same_bits(ys, ref)
    return ys, errs


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('method', sorted(METHODS))
def test_adaptive_solves_are_bit_identical(method, kind, dtype):
    ys, errs = check_fused(kind, method, dtype)
    assert any(e > 1 for e in errs), "no proposal was rejected"
    assert torch.isfinite(ys).all()


@pytest.mark.parametrize('which', ['interval', 'tree', 'path'])
@pytest.mark.parametrize('method', ['euler', 'milstein_ito', 'heun'])
def test_every_brownian_motion(method, which):
    check_fused('gbm', method, torch.float32, bm=which)


@pytest.mark.parametrize('method', sorted(METHODS))
def test_a_solve_that_hits_dt_min(method):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        check_fused('gbm', method, torch.float64, rtol=1e-9, atol=1e-9, dt_min=0.02, ts=(0.0, 0.13, 0.2))
    assert any('minimum allowed step size' in str(w.message) for w in caught)


def test_a_batch_that_fills_the_gpu():
    check_fused('gbm', 'milstein_ito', torch.float32, B=16384, d=64)


@pytest.mark.parametrize('method', ['euler', 'milstein_ito', 'heun'])
def test_the_unfusable_solves_keep_the_unfused_proposals(method):
    name, sde_type = METHODS[method]
    B, d = 32, 8
    n0 = fused_launches()
    # gradients through the solve
    sde = make_sde('gbm', sde_type, B, d, torch.float32)
    y0 = torch.full((B, d), 0.2, device=DEV, requires_grad=True)
    bm = make_bm('interval', B, d, torch.float32, 0.5, 'none')
    ys = tsde.sdeint(sde, y0, torch.tensor([0.0, 0.5], device=DEV), bm=bm, method=name, dt=0.05, adaptive=True)
    ys.sum().backward()
    # overlap False
    with torch.no_grad():
        tsde.sdeint(sde, y0.detach(), torch.tensor([0.0, 0.5], device=DEV), bm=make_bm('interval', B, d, torch.float32,
                    0.5, 'none'), method=name, dt=0.05, adaptive=True, options={'overlap': False})
    assert fused_launches() == n0


@pytest.mark.parametrize('method', ['milstein_ito', 'euler', 'midpoint'])
def test_sdeint_adjoint_adaptive(method):
    name, sde_type = METHODS[method]
    B, d = 32, 8
    ts = torch.tensor([0.0, 0.3, 0.5], device=DEV)

    def run():
        sde = make_sde('gbm', sde_type, B, d, torch.float32)
        y0 = torch.full((B, d), 0.2, device=DEV, requires_grad=True)
        bm = make_bm('interval', B, d, torch.float32, 0.5, 'none')
        ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method=name, dt=0.05, adaptive=True, rtol=1e-3, atol=1e-4,
                                 adjoint_method=name)
        (ys * ys).sum().backward()
        return ys.detach(), [y0.grad] + [p.grad for p in sde.parameters()]

    n0 = fused_launches()
    ys, grads = run()
    assert fused_launches() > n0
    with unfused():
        n1 = fused_launches()
        ref, ref_grads = run()
        assert fused_launches() == n1
    assert same_bits(ys, ref)
    assert all(same_bits(a, b) for a, b in zip(grads, ref_grads))
