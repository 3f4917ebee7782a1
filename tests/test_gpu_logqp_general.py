"""tsde_logqp_augment for general, additive and scalar noise on the GPU: the kernel against the float64 restatement of
tests/logqp_general_ref.py within a derived bound, golden replays of the reference, and whole latent-SDE solves
(eager vs CUDA graph, no torch pseudo-inverse involved, log-ratio vs the differentiated torch path)."""
import ctypes
import json
import warnings

import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from . import helpers, logqp_general_ref as lg

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SENTINEL = 12345.0
PAD = 64
WORST = {}          # dtype -> worst err / bound over this file's kernel cases


def _launch(f, g, h, rcond=lg.RCOND):
    """The raw entry point, outputs prefilled with NaN and guarded by PAD sentinels on both sides."""
    B, d, m = g.shape
    fa = torch.full((B * (d + 1) + 2 * PAD,), SENTINEL, dtype=f.dtype, device=DEV)
    ga = torch.full((B * (d + 1) * m + 2 * PAD,), SENTINEL, dtype=f.dtype, device=DEV)
    fa[PAD:-PAD] = float('nan')
    ga[PAD:-PAD] = float('nan')
    L = _cabi.make_launch(f.dtype, _cabi.NOISE_GENERAL, B, d, m, device=f.device)
    item = f.element_size()
    code = _cabi.lib().tsde_logqp_augment(ctypes.byref(L), f.data_ptr(), g.data_ptr(), h.data_ptr(), rcond,
                                          fa.data_ptr() + PAD * item, ga.data_ptr() + PAD * item)
    torch.cuda.synchronize()
    return code, fa, ga


def _inputs(B, d, m, dtype, kind, seed):
    rng = np.random.default_rng(seed)
    if kind.startswith('kappa'):
        g = lg.conditioned(rng, B, d, m, float(kind[5:]))
    else:
        g = 0.5 * rng.standard_normal((B, d, m))
    f, h = rng.standard_normal((B, d)), 0.5 * rng.standard_normal((B, d))
    if B and kind == 'zero':                     # a zero column and a zero row in alternate rows
        g[::2, :, m // 2] = 0.0
        g[1::2, d // 2, :] = 0.0
    if B and kind == 'nonfinite':
        for i, (arr, idx, v) in enumerate([(g, (0, 0, 0), np.nan), (g, (0, d - 1, m - 1), np.inf), (f, (0, 0), np.inf),
                                           (h, (0, d - 1), -np.inf), (f, (0, 0), np.nan)]):
            row = (3 * i + 1) % B
            arr[(row,) + idx[1:]] = v
    npdt = np.float32 if dtype == torch.float32 else np.float64
    return [torch.from_numpy(x.astype(npdt)).to(DEV) for x in (f, g, h)]


def _check(f, g, h, dtype):
    B, d, m = g.shape
    code, fa, ga = _launch(f, g, h)
    assert code == 0
    for buf in (fa, ga):
        assert bool((buf[:PAD] == SENTINEL).all()) and bool((buf[-PAD:] == SENTINEL).all())
    fa = fa[PAD:-PAD].view(B, d + 1)
    ga = ga[PAD:-PAD].view(B, d + 1, m)
    bits = torch.int32 if dtype == torch.float32 else torch.int64      # bit copies, NaN payloads included
    assert torch.equal(fa[:, :d].view(bits), f.view(bits)) and torch.equal(ga[:, :d].view(bits), g.view(bits))
    assert bool((ga[:, d] == 0).all()) and not bool(torch.signbit(ga[:, d]).any())
    fn, gn, hn = (x.double().cpu().numpy() for x in (f, g, h))
    want = lg.kl_rate(fn, gn, hn)
    got = fa[:, d].double().cpu().numpy()
    assert np.array_equal(np.isfinite(got), np.isfinite(want))
    ok = np.isfinite(want)
    tol = lg.bound(fn, gn, hn, dtype)
    err = np.abs(got[ok] - want[ok])
    with np.errstate(divide='ignore', invalid='ignore'):
        ratio = np.where(tol[ok] > 0, err / tol[ok], np.where(err > 0, np.inf, 0.0))
    assert (err <= tol[ok]).all(), (d, m, float(ratio.max()))
    if ratio.size:
        WORST[str(dtype)] = max(WORST.get(str(dtype), 0.0), float(ratio.max()))


SHAPES = [(1, 1), (4, 3), (3, 4), (16, 16), (32, 8), (8, 32), (64, 64), (5000, 1), (1, 257)]
DTYPES = [torch.float32, torch.float64]


@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f64'])
@pytest.mark.parametrize('d,m', SHAPES)
@pytest.mark.parametrize('kind', ['random', 'zero', 'kappa1e3', 'kappa1e6', 'nonfinite'])
def test_kernel_against_restatement(d, m, dtype, kind):
    if kind == 'kappa1e6' and dtype == torch.float32:
        pytest.skip('kappa 1e6 is beyond float32')
    # (with d == 1 or m == 1 the zero row / column is all of g in some rows: their rate is exactly 0)
    _check(*_inputs(33, d, m, dtype, kind, seed=d * 1000 + m), dtype)


@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f64'])
@pytest.mark.parametrize('B', [0, 1, 33, 65536])
@pytest.mark.parametrize('d,m', [(4, 3), (3, 4), (16, 16)])
def test_batch_sizes(B, d, m, dtype):
    f, g, h = _inputs(B, d, m, dtype, 'random', seed=B + 7)
    if B == 0:
        code, fa, ga = _launch(f, g, h)
        assert code == 0 and bool((fa == SENTINEL).sum() == 2 * PAD)
        return
    _check(f, g, h, dtype)


@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f64'])
def test_bound_shapes(dtype):
    """The largest shapes within TSDE_LOGQP_GENERAL_MAX run (tall, wide, square); one element over is TSDE_EINVAL."""
    for d, m in ((8192, 1), (1, 16383), (127, 127)):
        assert _cabi.logqp_general_fits(d, m)
        _check(*_inputs(3, d, m, dtype, 'random', seed=d + m), dtype)
    for d, m in ((8193, 1), (1, 16384), (128, 128)):
        assert not _cabi.logqp_general_fits(d, m)
        code, fa, ga = _launch(*_inputs(2, d, m, dtype, 'random', seed=1))
        assert code == _cabi.EINVAL and bool(fa[PAD:-PAD].isnan().all())


def test_report_worst_ratio():
    """(runs after the kernel cases) the worst err / bound per dtype, written for the design notes."""
    if not WORST:
        pytest.skip('no kernel case ran')
    print('worst err/bound', json.dumps(WORST))
    assert all(v <= 1.0 for v in WORST.values())


# ---- golden replays ----------------------------------------------------------------------------------------------
def _replay(case):
    from . import problems
    Ws = [torch.from_numpy(w).to(DEV) for w in case['W']]
    Us = [torch.from_numpy(u).to(DEV) for u in case['U']] if 'U' in case else None
    bm = problems.ReplayBM(case['ta'], case['tb'], Ws, Us, levy='space-time' if 'U' in case else 'none')
    bm.dtype, bm.device = Ws[0].dtype, Ws[0].device
    return bm


@pytest.mark.parametrize('path', helpers.golden_files('logqpgen_'), ids=helpers.case_id)
def test_golden_replay(path, monkeypatch):
    import torchsde_b200 as tsde
    case = helpers.load(path)
    name = str(case['name'])
    d, m, noise, sde_type, method, adjoint, zc, zr = lg.GOLDEN_CASES[name]
    sde = lg.LatentGeneral(d, m, noise, sde_type, seed=int(case['seed']), zero_col=zc, zero_row=zr).to(DEV)
    y0 = torch.from_numpy(case['y0']).to(DEV)
    ts = torch.from_numpy(case['ts']).to(DEV)
    dt = float(case['dt'])
    if not adjoint:
        monkeypatch.setattr(torch.Tensor, 'pinverse', _forbidden)
        monkeypatch.setattr(torch.linalg, 'pinv', _forbidden)
        with torch.no_grad():
            ys, logqp = tsde.sdeint(sde, y0, ts, bm=_replay(case), method=method, dt=dt, logqp=True)
        np.testing.assert_allclose(ys.cpu().numpy(), case['ys'], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(logqp.cpu().numpy(), case['logqp'], rtol=1e-10, atol=1e-12)
        return
    y0.requires_grad_(True)
    ys, logqp = tsde.sdeint_adjoint(sde, y0, ts, bm=_replay(case), method=method, dt=dt, logqp=True)
    np.testing.assert_allclose(ys.detach().cpu().numpy(), case['ys'], rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(logqp.detach().cpu().numpy(), case['logqp'], rtol=1e-10, atol=1e-12)
    wy, wl = torch.from_numpy(case['wy']).to(DEV), torch.from_numpy(case['wl']).to(DEV)
    ((ys * wy).sum() + (logqp * wl).sum()).backward()
    np.testing.assert_allclose(y0.grad.cpu().numpy(), case['grad_y0'], rtol=1e-8, atol=1e-10)
    for n, p in sde.named_parameters():
        got = np.zeros_like(case['grad.' + n]) if p.grad is None else p.grad.cpu().numpy()
        np.testing.assert_allclose(got, case['grad.' + n], rtol=1e-8, atol=1e-10, err_msg=n)


def _forbidden(*a, **k):
    raise AssertionError('the torch pseudo-inverse was called')


# ---- whole solves ------------------------------------------------------------------------------------------------
SOLVES = [('general', 6, 4, 'ito', 'euler', False), ('general', 4, 6, 'stratonovich', 'midpoint', False),
          ('additive', 6, 4, 'ito', 'srk', False), ('scalar', 6, 1, 'ito', 'euler', False),
          ('general', 6, 4, 'stratonovich', 'reversible_heun', True)]


def _solve(sde, y0, ts, m, method, adjoint, options, levy, grad=False):
    import torchsde_b200 as tsde
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(y0.shape[0], m), dtype=torch.float32, device=DEV,
                               entropy=21, levy_area_approximation=levy)
    if adjoint:   # (the forward pass; the backward sweep differentiates the torch path and is not captured)
        return tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -5, logqp=True, options=options)
    with torch.set_grad_enabled(grad):
        return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -5, logqp=True, options=options)


@pytest.mark.parametrize('noise,d,m,sde_type,method,adjoint', SOLVES)
def test_solve_eager_equals_graph_without_pinverse(noise, d, m, sde_type, method, adjoint, monkeypatch):
    B = 257
    sde = lg.LatentGeneral(d, m, noise, sde_type, seed=9, dtype=torch.float32).to(DEV)
    y0 = (0.1 + 0.5 * torch.rand(B, d, generator=torch.Generator().manual_seed(4))).to(DEV)
    ts = torch.tensor([0.0, 0.25, 0.5], device=DEV)
    levy = 'space-time' if method == 'srk' else 'none'
    outs = []
    with monkeypatch.context() as mp, warnings.catch_warnings():
        warnings.simplefilter('error')
        mp.setattr(torch.Tensor, 'pinverse', _forbidden)
        mp.setattr(torch.linalg, 'pinv', _forbidden)
        for opts in (None, {'cuda_graph': True}, {'cuda_graph': True}):
            with torch.no_grad():
                outs.append(_solve(sde, y0, ts, m, method, adjoint, opts, levy))
    for ys, lq in outs[1:]:
        assert torch.equal(ys, outs[0][0]) and torch.equal(lq, outs[0][1])
    ys, lq = outs[0]
    assert bool(torch.isfinite(lq).all()) and bool((lq >= 0).all())
    # the differentiated torch path (pinverse) on the same increments
    ys_t, lq_t = _solve(sde, y0.clone().requires_grad_(True), ts, m, method, False, None, levy, grad=True)
    ys_t, lq_t = ys_t.detach(), lq_t.detach()
    torch.testing.assert_close(ys, ys_t, rtol=1e-5, atol=1e-6)
    # per interval, sum over its steps of dt * bound(rate): bound taken at the worst state the output series shows
    with torch.no_grad():
        states = ys.reshape(-1, d)
        t0 = torch.tensor(0.0, device=DEV)
        f, g, h = sde.f(t0, states), sde.g(t0, states), sde.h(t0, states)
        if g.dim() == 3 and g.shape[0] != states.shape[0]:
            g = g.expand(states.shape[0], -1, -1)
    fn, gn, hn = (x.double().cpu().numpy() for x in (f, g, h))
    per_rate = lg.bound(fn, gn, hn, torch.float32).reshape(ys.shape[0], B).max(axis=0)
    tol = torch.from_numpy(4.0 * per_rate * 0.25 + 1e-6 * lq_t.abs().max(0).values.cpu().numpy()).to(DEV)
    assert bool(((lq - lq_t).abs() <= tol).all()), float(((lq - lq_t).abs() - tol).max())
