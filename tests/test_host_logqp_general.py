"""CPU tests of the general-noise `logqp=True` path: which solves take `tsde_logqp_augment` (dry runs against the
recording stand-in of the C library), the library's validation of general-noise launches, the float64 restatement of
the kernel's formula against the live reference, and that the GPU test's error bound tells wrong formulas apart."""
import ctypes
import os
import re
import warnings

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import base_sde
from . import logqp_general_ref as lg
from .test_host_dry_run import dry  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TS = [0.0, 0.125, 0.25]
DT = 0.0625
N_STEPS = 4


@pytest.fixture
def rec(dry, monkeypatch):  # noqa: F811
    """The recording library, also logging (noise_type, rows, d, m, eps) of every tsde_logqp_augment call."""
    class Lib:
        launches = []

        def __getattr__(self, name):
            return getattr(dry, name)

        def tsde_logqp_augment(self, L, *args):
            o = L._obj
            self.launches.append((o.noise_type, o.rows, o.d, o.m, args[3]))
            return dry.tsde_logqp_augment(L, *args)
    lib = Lib()
    lib.launches = []
    monkeypatch.setattr(_cabi, '_lib', lib)
    monkeypatch.setattr(_cabi, 'lib', lambda: lib)
    return lib


class Counting(torch.nn.Module):
    def __init__(self, sde):
        super().__init__()
        self.sde, self.noise_type, self.sde_type = sde, sde.noise_type, sde.sde_type
        self.f_calls = 0

    def f(self, t, y):
        self.f_calls += 1
        return self.sde.f(t, y)

    def g(self, t, y):
        return self.sde.g(t, y)

    def h(self, t, y):
        return self.sde.h(t, y)


KINDS = [('general', 3, 2, 'ito', 'euler'), ('general', 2, 5, 'stratonovich', 'midpoint'),
         ('additive', 3, 2, 'ito', 'srk'), ('additive', 3, 2, 'ito', 'euler'), ('scalar', 3, 1, 'ito', 'euler'),
         ('general', 3, 2, 'stratonovich', 'reversible_heun')]


def _solve(kind, d, m, sde_type, method, B=4, grad=False, options=None):
    sde = Counting(lg.LatentGeneral(d, m, kind, sde_type, dtype=torch.float32))
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(B, m), dtype=torch.float32, device='cpu', levy_area_approximation=levy)
    y0 = torch.full((B, d), 0.2, requires_grad=grad)
    with torch.set_grad_enabled(grad):
        ys, logqp = tsde.sdeint(sde, y0, TS, bm=bm, method=method, dt=DT, logqp=True, options=options)
    assert ys.shape == (3, B, d) and logqp.shape == (2, B)
    return sde, ys, logqp


@pytest.mark.parametrize('kind,d,m,sde_type,method', KINDS)
def test_no_grad_solves_take_the_kernel_once_per_drift_evaluation(rec, kind, d, m, sde_type, method):
    sde, _, _ = _solve(kind, d, m, sde_type, method)
    assert sde.f_calls >= N_STEPS
    assert len(rec.launches) == sde.f_calls
    assert all(lq == (_cabi.NOISE_GENERAL, 4, d, m, 1e-15) for lq in rec.launches), rec.launches[:2]


@pytest.mark.parametrize('kind,d,m,sde_type,method', KINDS)
def test_differentiated_solves_keep_the_torch_path(rec, kind, d, m, sde_type, method, monkeypatch):
    # (the stand-in library computes nothing, so the states are arbitrary memory: the torch formula is replaced by
    # a counting stub that cannot fail on them)
    torch_calls = []

    def kl_rate(f, g, h, diagonal):
        torch_calls.append(diagonal)
        return (0.0 * f).sum(dim=1, keepdim=True)
    monkeypatch.setattr(base_sde, '_kl_rate', kl_rate)
    sde, ys, _ = _solve(kind, d, m, sde_type, method, grad=True)
    assert sde.f_calls >= N_STEPS and ys.requires_grad and rec.launches == []
    assert len(torch_calls) == sde.f_calls and not any(torch_calls)


def test_adjoint_forward_takes_the_kernel_and_backward_does_not(rec, monkeypatch):
    # (arbitrary states under the stand-in library: the backward pass's torch formula is a differentiable stub)
    monkeypatch.setattr(base_sde, '_kl_rate', lambda f, g, h, diagonal: (0.0 * f).sum(dim=1, keepdim=True)
                        + 0.0 * g.sum(dim=(1, 2))[:, None])
    sde = Counting(lg.LatentGeneral(3, 4, 'general', 'stratonovich', dtype=torch.float32))
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 4), dtype=torch.float32, device='cpu')
    y0 = torch.full((4, 3), 0.2, requires_grad=True)
    ys, logqp = tsde.sdeint_adjoint(sde, y0, TS, bm=bm, method='reversible_heun', dt=DT, logqp=True)
    forward = len(rec.launches)
    assert 0 < forward <= sde.f_calls and all(lq[0] == _cabi.NOISE_GENERAL for lq in rec.launches)
    (ys.sum() + logqp.sum()).backward()
    assert len(rec.launches) == forward and y0.grad is not None


@pytest.mark.parametrize('d,m', [(1, 16383), (8192, 1), (127, 127), (1, 16384), (8193, 1), (128, 128), (2, 8192)])
def test_bound_routes_shapes(rec, d, m):
    fits = min(d, m) * max(d, m) + d <= _cabi.LOGQP_GENERAL_MAX
    assert fits == _cabi.logqp_general_fits(d, m)
    assert fits == ((d, m) in ((1, 16383), (8192, 1), (127, 127)))
    sde = base_sde.SDELogqp(lg.LatentGeneral(d, m, 'general', dtype=torch.float32))
    y = torch.full((2, d + 1), 0.3)
    with torch.no_grad():
        f_aug, g_aug = sde.f_and_g(torch.tensor(0.0), y)
    assert f_aug.shape == (2, d + 1) and g_aug.shape == (2, d + 1, m)
    assert len(rec.launches) == (1 if fits else 0)


def test_header_bound_is_mirrored():
    text = open(os.path.join(ROOT, 'include', 'torchsde_b200.h')).read()
    assert int(re.search(r'#define TSDE_LOGQP_GENERAL_MAX (\d+)', text).group(1)) == _cabi.LOGQP_GENERAL_MAX


def test_cuda_graph_captures_once_then_replays(rec):
    from torchsde_b200._core import graph
    sde = lg.LatentGeneral(3, 2, 'general', 'stratonovich', dtype=torch.float32)
    y0 = torch.full((4, 3), 0.2)
    captures, replays = rec.graph_cls.captures, rec.graph_cls.replays
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        for _ in range(3):
            bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, 2), dtype=torch.float32, device='cpu')
            with torch.no_grad():
                tsde.sdeint(sde, y0, TS, bm=bm, method='midpoint', dt=DT, logqp=True, options={'cuda_graph': True})
    assert not [w for w in caught if 'captured' in str(w.message)]
    assert rec.graph_cls.captures == captures + 1 and rec.graph_cls.replays == replays + 3
    assert len(graph._PLANS[sde]) == 1 and rec.launches and all(lq[0] == _cabi.NOISE_GENERAL for lq in rec.launches)


# ---- the library's validation (ctypes, no device: every case returns before any CUDA call) ----------------------
def _lib_or_skip():
    try:
        return _cabi.lib()
    except _cabi.LibraryNotBuilt:
        pytest.skip('CUDA library not built')


@pytest.mark.parametrize('dtype', [_cabi.F32, _cabi.F64])
def test_general_launch_validation(dtype):
    lib = _lib_or_skip()
    p = ctypes.c_void_p(256)

    def call(rows, d, m, ptrs=(p,) * 5):
        L = _cabi.Launch(dtype, _cabi.NOISE_GENERAL, rows, d, m, None)
        f, g, h, fa, ga = ptrs
        return lib.tsde_logqp_augment(ctypes.byref(L), f, g, h, 1e-15, fa, ga)
    assert call(0, 4, 3, (None,) * 5) == 0                       # empty batch: a no-op
    for i in range(5):
        ptrs = [p] * 5
        ptrs[i] = None
        assert call(3, 4, 3, ptrs) == _cabi.EINVAL
    for d, m in ((1, 16384), (8193, 1), (128, 128), (2, 8192), (1 << 40, 1), (1, 1 << 40), (1 << 62, 1 << 62)):
        assert call(3, d, m) == _cabi.EINVAL, (d, m)
    assert call(1 << 62, 4, 3) == _cabi.EINVAL                   # (d + 1) m rows overflows the element offsets
    L = _cabi.Launch(dtype | (_cabi.FMT_BF16 << 10), _cabi.NOISE_GENERAL, 3, 4, 3, None)
    assert lib.tsde_logqp_augment(ctypes.byref(L), p, p, p, 1e-15, p, p) == _cabi.EINVAL


# ---- the float64 restatement and the bound ---------------------------------------------------------------------
def test_restatement_equals_torch_pinverse_with_its_cutoff():
    """pinverse drops s <= rcond * s_max and inverts anything above it; the restatement keeps the same rule."""
    rng = np.random.default_rng(0)
    for d, m in ((4, 3), (3, 4), (5, 5), (6, 1), (1, 6)):
        g = rng.standard_normal((64, d, m))
        g[::4, :, -1] = 0.0
        if d > 1:
            g[1::4, 0, :] = 0.0
        f, h = rng.standard_normal((64, d)), rng.standard_normal((64, d))
        gt = torch.from_numpy(g)
        u = torch.bmm(gt.pinverse(), torch.from_numpy(f - h).unsqueeze(-1)).squeeze(-1)
        want = (0.5 * (u ** 2).sum(1)).numpy()
        np.testing.assert_allclose(lg.kl_rate(f, g, h), want, rtol=1e-10, atol=1e-14)
    f = np.array([[1.0, 2.0]])
    h = np.zeros_like(f)
    g = np.array([[[1.0, 0.0], [0.0, 1e-15]]])
    assert lg.kl_rate(f, g, h)[0] == 0.5                          # at the cutoff: dropped
    g[0, 1, 1] = 1.0000001e-15
    assert lg.kl_rate(f, g, h)[0] > 1e30                          # just above: inverted
    g[0, 0, 0] = np.nan
    assert np.isnan(lg.kl_rate(f, g, h)[0])


REFERENCE = os.path.join(ROOT, 'oracle', '_ref', 'site')


@pytest.mark.parametrize('kind,d,m,zc,zr', [('general', 4, 3, None, None), ('general', 3, 5, None, None),
                                            ('general', 4, 4, None, None), ('scalar', 4, 1, None, None),
                                            ('additive', 4, 3, None, None), ('general', 4, 3, 1, None),
                                            ('general', 3, 5, None, 1)])
def test_restatement_equals_the_live_reference(kind, d, m, zc, zr):
    if not os.path.isdir(os.path.join(REFERENCE, 'torchsde')):
        pytest.skip("reference not staged under oracle/_ref: golden vectors stand in")
    import sys
    for p in (REFERENCE, os.path.join(ROOT, 'oracle', 'refshim')):
        if p not in sys.path:
            sys.path.insert(0, p)
    from torchsde._core import base_sde as ref_base
    sde = lg.LatentGeneral(d, m, kind, 'ito', seed=3, zero_col=zc, zero_row=zr)
    ref = ref_base.SDELogqp(sde)
    y = torch.cat([0.2 + torch.rand(9, d, generator=torch.Generator().manual_seed(5), dtype=torch.float64),
                   torch.zeros(9, 1, dtype=torch.float64)], dim=1)
    t = torch.tensor(0.3, dtype=torch.float64)
    with torch.no_grad():
        fr, gr = ref.f_and_g_general(t, y)
        state = y[:, :-1]
        f, g, h = sde.f(t, state), sde.g(t, state), sde.h(t, state)
    np.testing.assert_allclose(lg.kl_rate(f.numpy(), g.numpy(), h.numpy()), fr[:, -1].numpy(), rtol=1e-10, atol=1e-15)
    assert torch.equal(gr[:, :-1], g) and float(gr[:, -1].abs().max()) == 0.0


def _rows(rng, B, d, m, zero_col=False):
    g = 0.2 + rng.random((B, d, m)) * rng.choice([0.1, 1.0, 10.0], size=(B, 1, 1))
    g = g + 0.5 * rng.standard_normal((B, d, m))
    if zero_col:
        g[:, :, rng.integers(m)] = 0.0
    f, h = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    return (x.astype(np.float32).astype(np.float64) for x in (f, g, h))


@pytest.mark.parametrize('variant,shapes,zero_col', [
    ('swapped', [(4, 4), (16, 16)], False), ('sigma', [(4, 3), (3, 4), (16, 16)], False),
    ('no_cutoff', [(4, 3), (4, 4), (8, 2)], True),   # (a zero column makes a zero singular value when d >= m) ('plus', [(4, 3), (3, 4), (8, 8)], False),
    ('neighbour', [(4, 3), (3, 4), (8, 8)], False)])
def test_bound_rejects_wrong_formulas(variant, shapes, zero_col):
    """The float32 bound of the GPU test (the looser one) must fail each mistake on at least 75 % of the rows."""
    rng = np.random.default_rng(11)
    for d, m in shapes:
        f, g, h = _rows(rng, 400, d, m, zero_col)
        want = lg.kl_rate(f, g, h)
        wrong = lg.kl_rate(f, g, h, variant=variant)
        tol = lg.bound(f, g, h, np.float32)
        assert np.isfinite(want).all() and (np.abs(want - want) <= tol).all()
        with np.errstate(invalid='ignore'):
            rejected = ~(np.abs(wrong - want) <= tol)
        assert rejected.mean() >= 0.75, (variant, d, m, rejected.mean())
