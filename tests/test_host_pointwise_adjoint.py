"""The fused backward sweep of `sdeint_adjoint`'s reversible pair (adjoint_options={'fused_backward': True};
pointwise.AdjointRecorder, the TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN program of tsde_solve_reversible_heun_pointwise)
on the CPU: which first-step tapes the recorder accepts and why it rejects the others, which sweeps keep their unfused
steps (with the reason, once), and a dry run of the launch sequence of a sweep with and without the option.  The GPU
suite compares the kernel with the unfused sweep and with central differences (tests/test_gpu_pointwise_adjoint.py)."""
import warnings

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import adjoint, pointwise
from .test_host_dry_run import dry  # noqa: F401  (fixture)

ROWS, D = 6, 5


def record(f, g, params, dtype=torch.float32, transcendental=False):
    """The three segments of a first backward step of f and g (callables of (t, y)) under the recorder."""
    gen = torch.Generator().manual_seed(1)
    z0 = (torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.5).requires_grad_()
    z1 = (torch.rand(ROWS, D, generator=gen, dtype=dtype) + 0.5).requires_grad_()
    t0, t1 = torch.tensor(0.5, dtype=dtype), torch.tensor(0.375, dtype=dtype)
    go, go2 = torch.rand(ROWS, D, generator=gen, dtype=dtype), torch.rand(ROWS, D, generator=gen, dtype=dtype)
    rec = pointwise.AdjointRecorder(z0, t0, len(params), transcendental)
    fo, gout = rec.forward(lambda: (f(t0, z0), g(t0, z0)))
    rec.vjp(lambda: torch.autograd.grad([fo, gout], [z0] + list(params), [go, go2], allow_unused=True), go, go2,
            params)
    rec.again(lambda: (f(t1, z1), g(t1, z1)), t1, z1)
    return rec, rec.finish()


def P(*shape):
    return torch.rand(shape, generator=torch.Generator().manual_seed(len(shape) + 7)).requires_grad_()


def test_gbm_with_channel_parameters():
    mu, sigma = P(D), P(D)
    rec, res = record(lambda t, y: mu * y, lambda t, y: sigma * y, [mu, sigma])
    assert res is not None, rec.reason
    ad, _, kinds = res
    assert kinds == [pointwise.REDUCE_ROWS] * 2 and ad.n_params == 2
    assert ad.prog.n_regs <= _cabi.PW_MAX_REGS and 0 < ad.prog.n_fg < ad.prog.n_instr
    assert ad.prog.reserved == _cabi.PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN
    src = _cabi.pointwise_source(ad.prog, torch.float32)
    assert src is not None and 'go2[j]' in src and 'acc[1][j] = acc[1][j] + ' in src


def test_ou_with_scalar_parameters_and_a_time_dependent_drift():
    kappa, theta, sigma = P(), P(), P(D)
    rec, res = record(lambda t, y: kappa * (theta - y) * t, lambda t, y: sigma * y, [kappa, theta, sigma])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ALL, pointwise.REDUCE_ALL, pointwise.REDUCE_ROWS]
    assert any(op.kind == _cabi.PW_T0 for op in res[0].prog.operand[:res[0].prog.n_operands])


def test_a_per_trajectory_parameter():
    mu, sigma = P(D), P(ROWS, D)
    rec, res = record(lambda t, y: mu * y, lambda t, y: sigma * y, [mu, sigma])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS, pointwise.REDUCE_NONE]


def test_a_parameter_used_in_f_and_g_sums_its_contributions():
    a = P(D)
    rec, res = record(lambda t, y: a * y, lambda t, y: a * y * y, [a])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS] and res[0].n_params == 1


def test_an_unused_parameter_contributes_nothing():
    mu, unused = P(D), P(D)
    rec, res = record(lambda t, y: mu * y, lambda t, y: mu * y, [mu, unused])
    assert res is not None, rec.reason
    assert res[2] == [pointwise.REDUCE_ROWS, None] and res[0].n_params == 1


@pytest.mark.parametrize('case', ['transformed', 'too_many', 'transcendental', 'evaluations_differ', 'batch_sum'])
def test_rejected_tapes(case):
    if case == 'transformed':  # the gradient of a parameter transformed before it is broadcast
        mu = P(D)
        rec, res = record(lambda t, y: (mu * mu) * y, lambda t, y: y * 0.5, [mu])
        assert 'after its batch reduction' in rec.reason
    elif case == 'too_many':
        ps = [P(D) for _ in range(_cabi.PW_ADJ_MAX_PARAMS + 1)]
        rec, res = record(lambda t, y: sum(p * y for p in ps), lambda t, y: y * 0.5, ps)
        assert 'parameters' in rec.reason
    elif case == 'transcendental':
        mu = P(D)
        rec, res = record(lambda t, y: mu * torch.exp(y), lambda t, y: y * 0.5, [mu])
        assert 'exp' in rec.reason
    elif case == 'batch_sum':  # a reduction in f itself is not a parameter's gradient: the ordinary reason
        mu = P(D)
        rec, res = record(lambda t, y: mu * (y - y.sum(0, keepdim=True)), lambda t, y: y * 0.5, [mu])
        assert 'sum' in rec.reason and 'batch reduction' not in rec.reason
    else:  # f computed otherwise at (t1, z1) than at (t0, z0), as a Python branch would
        mu, calls = P(D), []

        def f(t, y):
            calls.append(t)
            return mu * y if len(calls) == 1 else mu + y
        rec, res = record(f, lambda t, y: y * 0.5, [mu])
        assert 'differ' in rec.reason
    assert res is None


# ---- sweeps ------------------------------------------------------------------------------------------------------------
class GBM(nn.Module):
    sde_type = 'stratonovich'

    def __init__(self, noise='diagonal', fused=False):
        super().__init__()
        self.noise_type = noise
        self.mu, self.sigma = nn.Parameter(torch.rand(D) - 0.5), nn.Parameter(torch.rand(D))
        if fused:
            self.f_and_g = lambda t, y: (self.f(t, y), self.g(t, y))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return self.sigma * y if self.noise_type == 'diagonal' else (self.sigma * y).unsqueeze(-1)

    def h(self, t, y):  # (the prior drift of logqp)
        return -y


def sweep(ts, options, sde=None, create_graph=False, logqp=False, **kw):
    sde = GBM() if sde is None else sde
    m = 1 if sde.noise_type == 'general' else D + 1 if logqp else D  # (logqp augments the state by one channel)
    bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(ROWS, m), dtype=torch.float32, device='cpu')
    y0 = torch.ones(ROWS, D, requires_grad=True)
    out = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=0.0625,
                              adjoint_options=dict(options), logqp=logqp, **kw)
    ys = out[0] if logqp else out
    if create_graph:
        torch.autograd.grad(ys.sum(), [y0], create_graph=True)
    else:
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


@pytest.mark.parametrize('ts', [DENSE, SPARSE], ids=['dense', 'sparse'])
def test_without_the_option_every_step_runs_kernels_a_and_b(dry, chunks, ts):  # noqa: F811
    sweep(ts, {})
    assert dry.calls['tsde_adjoint_reversible_heun_a'] == dry.calls['tsde_adjoint_reversible_heun_b'] == 8
    assert not chunks


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
    outs = chunks
    assert dry.calls['tsde_adjoint_reversible_heun_a'] == 1 and 'tsde_adjoint_reversible_heun_b' not in dry.calls
    n = dry.calls['tsde_solve_reversible_heun_pointwise'] - n0[0]
    assert n == len(outs) == len(pointwise.plan_chunks(0, 8, max_steps=max_steps))
    # output rows are flagged in the step table, newest first; they do not cut a chunk
    flat = [o for c in outs for o in c]
    every = 8 // (len(ts) - 1)
    assert flat == [len(ts) - 2 - k // every if (k + 1) % every == 0 else -1 for k in range(8)]


@pytest.mark.parametrize('case', ['f_and_g', 'general', 'logqp', 'adjoint_adaptive', 'create_graph'])
def test_sweeps_that_keep_their_unfused_steps_say_why(dry, chunks, monkeypatch, case):  # noqa: F811
    monkeypatch.setattr(adjoint, '_WARNED', set())
    kw = {}
    sde = None
    if case == 'f_and_g':
        sde, want = GBM(fused=True), 'f_and_g'
    elif case == 'general':
        sde, want = GBM('general'), 'general noise'
    elif case == 'logqp':
        kw, want = {'logqp': True}, 'logqp'
    elif case == 'adjoint_adaptive':
        kw, want = {'adjoint_adaptive': True}, 'adjoint_adaptive'
    else:
        kw, want = {'create_graph': True}, 'create_graph'
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        sweep(SPARSE, {'fused_backward': True}, sde, **kw)
    said = [str(w.message) for w in caught if 'unfused steps' in str(w.message)]
    assert len(said) == 1 and want in said[0], said
    assert not chunks
