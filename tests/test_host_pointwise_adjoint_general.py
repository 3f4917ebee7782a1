"""The fused backward sweep of `sdeint_adjoint`'s reversible pair for general and additive noise
(adjoint_options={'fused_backward': True}; pointwise.GeneralAdjointRecorder, the
TSDE_PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN program of tsde_solve_reversible_heun_pointwise on a GENERAL launch) on
the CPU: which first-step tapes the recorder accepts, with which reductions, why it rejects the others, and a dry run
of a sweep's launch sequence.  The GPU suite compares the kernel with the unfused sweep
(tests/test_gpu_pointwise_adjoint_general.py)."""
import warnings

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from .test_host_dry_run import dry  # noqa: F401  (fixture)

ROWS, D, M = 6, 5, 3


def record(f, g, params, m=M, dtype=torch.float32, transcendental=False):
    """The three segments of a first backward step of f and g (callables of (t, y)) under the general recorder."""
    gen = torch.Generator().manual_seed(1)
    z0 = (torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.5).requires_grad_()
    z1 = (torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.5).requires_grad_()
    t0, t1 = torch.tensor(0.5, dtype=dtype), torch.tensor(0.375, dtype=dtype)
    go, go2 = torch.rand(ROWS, D, generator=gen, dtype=dtype), torch.rand(ROWS, D, m, generator=gen, dtype=dtype)
    rec = pointwise.GeneralAdjointRecorder(z0, t0, len(params), m, transcendental)
    fo, gout = rec.forward(lambda: (f(t0, z0), g(t0, z0)))
    rec.vjp(lambda: torch.autograd.grad([fo, gout], [z0] + list(params), [go, go2.view_as(gout)],
                                        allow_unused=True), go, go2, params)
    rec.again(lambda: (f(t1, z1), g(t1, z1)), t1, z1)
    return rec, rec.finish()


def P(*shape):
    return torch.rand(shape, generator=torch.Generator().manual_seed(len(shape) + 7)).requires_grad_()


def source(res, m=M):
    return _cabi.general_pointwise_source(res[0].prog, torch.float32, D, m)


def test_correlated_gbm():
    mu, S = P(D), P(D, M)
    rec, res = record(lambda t, y: mu * y, lambda t, y: y.unsqueeze(-1) * S, [mu, S])
    assert res is not None, rec.reason
    ad, _, kinds = res
    assert kinds == [pointwise.REDUCE_ROWS, pointwise.REDUCE_CHANNEL_ROWS] and ad.n_params == 2
    assert ad.prog.reserved == _cabi.PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN
    ops = [ad.prog.instr[i].op for i in range(ad.prog.n_instr)]
    assert ops.count(_cabi.PW_CSUM) == 1
    src = source(res)
    assert src is not None and 'pc(int k) { return false || k == 1; }' in src
    assert 'T(0) + ' in src and 'agm' in src


def test_multi_factor_ou():
    kappa, theta, S = P(1), P(1), P(D, M)
    rec, res = record(lambda t, y: kappa * (theta - y), lambda t, y: S.expand(ROWS, D, M), [kappa, theta, S])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ALL, pointwise.REDUCE_ALL, pointwise.REDUCE_CHANNEL_ROWS]
    assert res[0].param_src[2] == _cabi.PW_SRC_GO2  # (S's contribution is the seed itself)
    # its partial is (rows, d, m): the kernel adds to it per channel and never as a (rows, d) quad
    assert 'pc(int k) { return false || k == 2; }' in source(res)


def test_channel_loadings_and_a_one_element_scale():
    mu, w, s = P(D), P(M), P(1)
    rec, res = record(lambda t, y: mu * y, lambda t, y: (s * y).unsqueeze(-1) * w, [mu, w, s])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS, pointwise.REDUCE_CHANNEL_ROWS_D, pointwise.REDUCE_ALL]


@pytest.mark.skipif(pointwise.nvrtc_mismatch() is not None or not _cabi.nvjitlink(),
                    reason="no NVRTC / nvJitLink of PyTorch's CUDA release")
def test_tanh_mixed_general_with_transcendental():
    mu, S = P(D), P(D, M)
    rec, res = record(lambda t, y: mu * torch.tanh(y), lambda t, y: torch.tanh(y).unsqueeze(-1) * S, [mu, S],
                      transcendental=True)
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS, pointwise.REDUCE_CHANNEL_ROWS]
    assert source(res) is not None


def test_tanh_without_the_option_is_refused():
    S = P(D, M)
    rec, res = record(lambda t, y: -y, lambda t, y: torch.tanh(y).unsqueeze(-1) * S, [S])
    assert res is None and 'tanh' in rec.reason


def test_a_parameter_in_f_and_g_sums_its_contributions():
    a, S = P(D), P(D, M)
    rec, res = record(lambda t, y: a * y, lambda t, y: (a * y).unsqueeze(-1) * S, [a, S])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS, pointwise.REDUCE_CHANNEL_ROWS] and res[0].n_params == 2


@pytest.mark.parametrize('case', ['m1', 'm33', 'transformed', 'foreign', 'non_channel_sum'])
def test_rejected_tapes(case):
    S = P(D, M)
    if case in ('m1', 'm33'):
        m = 1 if case == 'm1' else _cabi.PW_GENERAL_MAX_M + 1
        Sm = P(D, m)
        rec, res = record(lambda t, y: -y, lambda t, y: y.unsqueeze(-1) * Sm, [Sm], m=m)
        assert 'general noise' in rec.reason and 'Brownian channels' in rec.reason
    elif case == 'transformed':
        rec, res = record(lambda t, y: -y, lambda t, y: y.unsqueeze(-1) * (S * S), [S])
        assert 'after its batch reduction' in rec.reason
    elif case == 'foreign':  # a (rows, d, m) tensor from outside the tape
        big = torch.rand(ROWS, D, M)
        rec, res = record(lambda t, y: -y, lambda t, y: y.unsqueeze(-1) * big * S, [S])
        assert 'read per channel' in rec.reason
    else:  # the vjp sums a per-channel value over the rows and the channels: a (d, 1) parameter read per channel
        p = P(D, 1)
        rec, res = record(lambda t, y: -y, lambda t, y: y.unsqueeze(-1) * S * p, [S, p])
        assert 'a reduction over dims (0, 2) of a per-channel value' in rec.reason
    assert res is None


def test_the_library_refuses_a_broken_program():
    mu, S = P(D), P(D, M)
    rec, res = record(lambda t, y: mu * y, lambda t, y: y.unsqueeze(-1) * S, [mu, S])
    ad = res[0]
    assert _cabi.general_pointwise_source(ad.prog, torch.float32, D, 1) is None  # m = 1
    ad.prog.reserved = _cabi.PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN  # the diagonal tag on a GENERAL launch
    assert _cabi.general_pointwise_source(ad.prog, torch.float32, D, M) is None
    ad.prog.reserved = _cabi.PW_LAYOUT_GENERAL_ADJOINT_REVERSIBLE_HEUN
    csum = next(i for i in range(ad.prog.n_instr) if ad.prog.instr[i].op == _cabi.PW_CSUM)
    ad.prog.instr[csum].a = _cabi.PW_SRC_Y  # the channel sum of a (rows, d) value
    assert _cabi.general_pointwise_source(ad.prog, torch.float32, D, M) is None


# ---- sweeps ------------------------------------------------------------------------------------------------------------
class CorrelatedGBM(nn.Module):
    sde_type, noise_type = 'stratonovich', 'general'

    def __init__(self, m=M):
        super().__init__()
        self.mu, self.S = nn.Parameter(torch.rand(D) - 0.5), nn.Parameter(torch.rand(D, m) * 0.2)

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return y.unsqueeze(-1) * self.S


def sweep(ts, options, sde=None):
    sde = CorrelatedGBM() if sde is None else sde
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(ROWS, sde.S.shape[1]), dtype=torch.float32, device='cpu')
    y0 = torch.ones(ROWS, D, requires_grad=True)
    ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=0.0625, adjoint_options=dict(options))
    ys.sum().backward()


DENSE = torch.arange(9) * 0.0625
SPARSE = torch.tensor([0.0, 0.25, 0.5])


@pytest.fixture
def chunks(monkeypatch):
    """The output rows of the steps of every chunk launched (pointwise.solve_adjoint_chunk)."""
    outs = []
    real = pointwise.solve_adjoint_chunk

    def chunk(engine, ks, *a):
        outs.append([engine._out[k] for k in ks])
        return real(engine, ks, *a)
    monkeypatch.setattr(pointwise, 'solve_adjoint_chunk', chunk)
    return outs


@pytest.mark.parametrize('max_steps', [3, _cabi.PW_MAX_STEPS])
@pytest.mark.parametrize('ts', [DENSE, SPARSE], ids=['dense', 'sparse'])
def test_with_the_option_one_recording_step_then_chunks(dry, chunks, monkeypatch, ts, max_steps):  # noqa: F811
    monkeypatch.setattr(pointwise, 'chunk_length', lambda solver: max_steps)
    n0 = []
    real = tsde.sdeint_adjoint

    def forward(*a, **k):  # (the forward solve's own reversible-Heun chunks use the same entry point)
        out = real(*a, **k)
        n0.append(dry.calls.get('tsde_solve_reversible_heun_pointwise', 0))
        return out
    monkeypatch.setattr(tsde, 'sdeint_adjoint', forward)
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        sweep(ts, {'fused_backward': True})
    assert dry.calls['tsde_adjoint_reversible_heun_a'] == 1 and 'tsde_adjoint_reversible_heun_b' not in dry.calls
    n = dry.calls['tsde_solve_reversible_heun_pointwise'] - n0[0]
    assert n == len(chunks) == len(pointwise.plan_chunks(0, 8, max_steps=max_steps))
    flat = [o for c in chunks for o in c]
    every = 8 // (len(ts) - 1)
    assert flat == [len(ts) - 2 - k // every if (k + 1) % every == 0 else -1 for k in range(8)]


def test_without_the_option_every_step_runs_kernels_a_and_b(dry, chunks):  # noqa: F811
    sweep(SPARSE, {})
    assert dry.calls['tsde_adjoint_reversible_heun_a'] == dry.calls['tsde_adjoint_reversible_heun_b'] == 8
    assert not chunks
