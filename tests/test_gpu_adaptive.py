"""`sdeint(adaptive=True)` on counter noise against tests/adaptive_ref.py, proposal by proposal.

An adaptive solve queries the BrownianInterval at data-dependent, non-dyadic times (bridges deeper than any grid asks
for, merges across grid cells, SRK's U), forms each proposal's tableau scalars from a step size that is not a power of
two, and decides on the host from `tsde_adaptive_error_sumsq`.  A wrong increment in a rejected proposal crashes
nothing: it moves the step size.  So the GPU solve is recorded (`spy`: every proposal's times, error estimate, step
size and decision, every Brownian query, and on request the proposal's states) and compared with the restatement of
the reference's loop on the same Brownian motion (adaptive_ref's docstring says where its increments come from).

  * float64, free mode: the restatement makes its own decisions.  Histories must be identical: the same number of
    proposals, every (ta, tb) query the same bits in the same order, the same accept decisions and dt_min hits, error
    estimates within a relative 1e-9 and ys (and the logqp log-ratio) within 1e-9 scale(ref).  The step size is a
    continuous function of the error estimate, which the GPU sums in another order, so the restatement adopts the
    GPU's next_t when its own lies within a relative 1e-12 of it (adaptive_ref.SNAP_REL).
  * float32, driven mode: the restatement follows the GPU's history, and y_full, y_half of every proposal and ys must
    be within e n K u scale(ref) (test_gpu_generic_adjoint.f32_bound; n the queries of the solve).  Its own error
    estimate must be within the bound that implies (`err_bound`); where it falls on the other side of 1 from the GPU's
    decision, |err_ref - 1| must be within that bound.
  * full batch: B = 2^20 + 3, d = 3 in float32, fused and unfused.  Every error estimate equals its recomputation from
    the GPU's own y_full / y_half: to a relative 1e-12 when each element's ratio is formed in float32, as the kernel
    and the reference's compute_error do, and accumulated in float64; within 8 u of a pure float64 recomputation.
    Rows 0, 1, B-2, B-1 and 256 random rows match the driven restatement on the oracle's normals of those rows.
  * gradients: with its history fixed, a float64 adaptive solve is a smooth function of y0 and the parameters:
    y0.grad and the parameter gradients of a weighted loss must match central differences of the driven restatement
    (tests/gradient_ref.py).
  * the comparisons must be able to fail: four monkeypatched errors of the restatement (a half step served the other
    half's increment, the error estimate divided by numel - 1, the interpolation weights swapped, one row served its
    neighbour's increments) each make the float64 comparison fail.

Every case's route is confirmed by the proposal kernel's launch counter (TSDE_KERNEL_PW_ADAPTIVE): it moves on a solve
of an element-wise diagonal SDE by a method with a fused proposal, and stays still otherwise (`Coupled` adds a row
reduction that keeps f's value and makes the SDE not element-wise).  Every case's history must hold a rejection and
an accepted step with error in (0.1, 1], so no case passes vacuously.  The worst err/bound per (method, dtype) is
printed at the end (`-s`).
"""
import collections
import contextlib
import math
import warnings

import numpy as np
import pytest
import torch
from torch import nn

from oracle import solvers
from torchsde_b200 import _cabi
from torchsde_b200._brownian import interval as iv
from torchsde_b200._core import base_solver, methods

from . import adaptive_ref, adjoint_ref, gradient_ref, helpers, problems
from .test_gpu_generic_adjoint import f32_bound

pytestmark = pytest.mark.gpu
DEV = 'cuda'
U32 = 2.0 ** -24
RTOL64 = adjoint_ref.RTOL64
NP = {torch.float32: np.float32, torch.float64: np.float64}
FUSED_METHODS = ('euler', 'milstein', 'srk', 'heun', 'midpoint', 'euler_heun')
WORST = {}


def _tsde():
    import torchsde_b200
    return torchsde_b200


def fused_launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE)


class Coupled(nn.Module):
    """The same SDE with a row reduction in its drift: f + 0 sum(y) has f's value, but is not an element-wise program,
    so an adaptive solve takes the unfused proposals."""

    def __init__(self, base):
        super().__init__()
        self.base = base
        self.noise_type, self.sde_type = base.noise_type, base.sde_type

    def f(self, t, y):
        return self.base.f(t, y) + 0.0 * y.sum(dim=1, keepdim=True)

    def g(self, t, y):
        return self.base.g(t, y)


# ---- the spy ---------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def spy(rows=None, on_error=None):
    """Records, inside the block, every proposal of an adaptive solve (times, and the `rows` of y_full / y_half), its
    error estimate (handed to `on_error(y_full, y_half, err)` too), the step size the controller returned, and every
    query of a BrownianInterval."""
    seen = collections.defaultdict(list)
    depth = [0]
    base_propose, mixin_propose = base_solver.BaseSDESolver._propose, methods._ProposalMixin._propose
    real_error, real_update = base_solver.BaseSDESolver._error_estimate, base_solver.BaseSDESolver._update_step_size
    real_call = iv.BrownianInterval.__call__

    def wrap(real):
        def propose(self, curr_t, next_t, midpoint_t, curr_y, curr_extra):
            depth[0] += 1
            try:
                out = real(self, curr_t, next_t, midpoint_t, curr_y, curr_extra)
            finally:
                depth[0] -= 1
            if depth[0] == 0:   # (the fused proposal falls back to the base class's until it has its program)
                seen['props'].append((float(curr_t), float(next_t), float(midpoint_t)))
                if rows is not None:
                    idx = torch.as_tensor(rows, device=out[0].device)
                    seen['full'].append(out[0].detach()[idx].double().cpu().numpy())
                    seen['half'].append(out[1].detach()[idx].double().cpu().numpy())
            return out
        return propose

    def error(self, y_full, y_half):
        err = real_error(self, y_full, y_half)
        seen['errs'].append(err)
        if on_error is not None:
            on_error(self, y_full, y_half, err)
        return err

    def update(**kw):
        out = real_update(**kw)
        seen['steps'].append(float(out[0]))
        return out

    def call(self, ta, tb=None, return_U=False, return_A=False):
        seen['queries'].append((float(ta), float(tb)))
        return real_call(self, ta, tb, return_U=return_U, return_A=return_A)

    base_solver.BaseSDESolver._propose, methods._ProposalMixin._propose = wrap(base_propose), wrap(mixin_propose)
    base_solver.BaseSDESolver._error_estimate = error
    base_solver.BaseSDESolver._update_step_size = staticmethod(update)
    iv.BrownianInterval.__call__ = call
    try:
        yield seen
    finally:
        base_solver.BaseSDESolver._propose, methods._ProposalMixin._propose = base_propose, mixin_propose
        base_solver.BaseSDESolver._error_estimate = real_error
        base_solver.BaseSDESolver._update_step_size = staticmethod(real_update)
        iv.BrownianInterval.__call__ = real_call


def gpu_history(seen, dt_min):
    """The GPU's proposals as adaptive_ref.Proposal: a proposal was accepted iff the next one starts at its next_t (the
    last one ends the solve); it hit dt_min iff the controller returned a step below dt_min."""
    props, errs, steps = seen['props'], seen['errs'], seen['steps']
    assert len(props) == len(errs) == len(steps), (len(props), len(errs), len(steps))
    out = []
    for k, (a, b, mid) in enumerate(props):
        accepted = k == len(props) - 1 or props[k + 1][0] == b
        assert accepted or props[k + 1][0] == a, f'proposal {k + 1} starts neither at {a!r} nor at {b!r}'
        out.append(adaptive_ref.Proposal(a, b, mid, errs[k], accepted, steps[k] < dt_min))
    return out


# ---- cases -----------------------------------------------------------------------------------------------------------
Case = collections.namedtuple('Case', 'method st kind opts coupled dtype B d m ts dt rtol atol dt_min bm_dt logqp '
                                      'graph dt_tensor seed vacuous')


def case(method, st, kind, opts=None, coupled=False, dtype=torch.float64, B=3, d=None, m=None, ts=(0.0, 0.25, 0.5),
         dt=0.5, rtol=1e-4, atol=1e-4, dt_min=1e-5, bm_dt=None, logqp=False, graph=False, dt_tensor=False, seed=0,
         vacuous=True):
    d = d or {'gbm': 4, 'scalar': 3, 'additive': 3, 'general': 4}[kind]
    m = m or {'gbm': d, 'scalar': 1, 'additive': 2, 'general': 3}[kind]
    return Case(method, st, kind, opts, coupled, dtype, B, d, m, tuple(ts), dt, rtol, atol, dt_min, bm_dt, logqp,
                graph, dt_tensor, seed, vacuous)


def case_id(c):
    s = f"{c.st[:5]}-{c.method}{'_gf' if c.opts else ''}-{c.kind}{'-coupled' if c.coupled else ''}"
    return s + f"-B{c.B}d{c.d}"


def expect_fused(c):
    return (c.method in FUSED_METHODS and c.kind == 'gbm' and not c.coupled and not c.logqp and not c.opts)


_ALL = ('gbm', 'scalar', 'additive', 'general')
_DIAG = ('gbm', 'scalar', 'additive')
# every (method, options, sde_type, noise kinds) the reference's adaptive solve accepts (its compatibility matrix,
# check_contract and methods/*.py)
MATRIX = [('euler', None, 'ito', _ALL)] + \
    [('milstein', o, st, _DIAG) for st in ('ito', 'stratonovich') for o in (None, {'grad_free': True})] + \
    [('srk', None, 'ito', _DIAG)] + \
    [(meth, None, 'stratonovich', _ALL) for meth in ('heun', 'midpoint', 'euler_heun', 'reversible_heun')]
MATRIX_CASES = [case(meth, st, kind, opts=o, seed=i) for i, (meth, o, st, kinds) in enumerate(MATRIX)
                for kind in kinds]
# and the unfused route of every method with a fused proposal, on the same element-wise SDE behind a reduction
MATRIX_CASES += [case(meth, st, 'gbm', coupled=True, seed=40 + i) for i, (meth, o, st, kinds) in enumerate(MATRIX)
                 if meth in FUSED_METHODS and o is None]


class Run:
    pass


def problem(c, dtype):
    if c.logqp:
        noise = 'diagonal' if c.kind == 'gbm' else 'general'
        base = problems.LatentPrior(c.d, c.m, noise, c.st, seed=c.seed, dtype=dtype)
    else:
        base = problems.make(c.kind, c.d, c.m, c.st, dtype=dtype, seed=c.seed)
    return Coupled(base) if c.coupled else base


def gpu_solve(c, rows=None, on_error=None, graph=None):
    """The GPU solve of case c under the spy."""
    tsde = _tsde()
    r = Run()
    r.dev = problem(c, c.dtype).to(DEV)
    cpu = problem(c, c.dtype).double()
    r.module = adjoint_ref.Logqp(cpu.base if c.coupled else cpu) if c.logqp else cpu
    bm_m = (c.d + 1 if c.kind == 'gbm' else c.m) if c.logqp else c.m
    gen = torch.Generator().manual_seed(100 + c.seed)
    y0 = (0.1 + 0.5 * torch.rand(c.B, c.d, generator=gen, dtype=torch.float64)).to(c.dtype)
    r.y0_ref = y0.double().numpy()
    if c.logqp:
        r.y0_ref = np.concatenate([r.y0_ref, np.zeros((c.B, 1))], axis=1)
    r.ts_np = np.asarray(c.ts, dtype=NP[c.dtype])
    tst = torch.from_numpy(r.ts_np).to(DEV)
    levy = 'space-time' if c.method == 'srk' else 'none'
    r.bm = tsde.BrownianInterval(float(r.ts_np[0]), float(r.ts_np[-1]), size=(c.B, bm_m), dtype=c.dtype, device=DEV,
                                 entropy=7 + c.seed, levy_area_approximation=levy, dt=c.bm_dt)
    dt = torch.tensor(c.dt, dtype=torch.float64) if c.dt_tensor else c.dt
    options = dict(c.opts or {})
    if c.graph if graph is None else graph:
        options['cuda_graph'] = True
    n0 = fused_launches()
    with torch.no_grad(), spy(rows, on_error) as seen, warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        out = tsde.sdeint(r.dev, y0.to(DEV), tst, bm=r.bm, method=c.method, dt=dt, adaptive=True, rtol=c.rtol,
                          atol=c.atol, dt_min=c.dt_min, options=options, logqp=c.logqp)
        torch.cuda.synchronize()
    r.fused = fused_launches() > n0
    r.warned = any('minimum allowed step size' in str(w.message) for w in caught)
    r.ys, r.lr = (out[0], out[1]) if c.logqp else (out, None)
    r.hist = gpu_history(seen, c.dt_min)
    r.queries = list(seen['queries'])
    r.full, r.half = seen['full'], seen['half']
    return r


def restatement(c, r, query):
    return solvers.make(c.method, problems.NumpySDE(r.module), query, float(c.dt), dict(c.opts or {}))


def _excess(got, ref, bound):
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    if got.shape != ref.shape:
        return math.inf
    return float(np.max(adjoint_ref.excess(got, ref, bound * adjoint_ref.scale(ref)), initial=0.0))


def _note(key, r):
    if key is not None:
        WORST[key] = max(WORST.get(key, 0.0), r)


def check_route_and_history(c, r, bad):
    if r.fused != expect_fused(c):
        bad.append(f"route: the proposal kernel {'ran' if r.fused else 'did not run'}")
    if r.hist and (r.hist[-1].next_t != float(r.ts_np[-1])):
        bad.append(f'the last proposal ends at {r.hist[-1].next_t!r}, not ts[-1]')
    if c.vacuous:
        if all(h.accepted for h in r.hist):
            bad.append('vacuous: no proposal was rejected')
        if not any(h.accepted and 0.1 < h.error <= 1 for h in r.hist):
            bad.append('vacuous: no accepted proposal with error in (0.1, 1]')


def compare_free(c, r, bad, key):
    """float64: the restatement's own history against the GPU's."""
    query, asked = adaptive_ref.increments(r.bm, np.float64)
    try:
        res = adaptive_ref.integrate_adaptive(restatement(c, r, query), r.y0_ref, r.ts_np, c.rtol, c.atol,
                                              c.dt_min, snap=r.hist)
    except AssertionError as e:   # (the tree oracle answers only queries the GPU solve made)
        bad.append(f'the restatement left the GPU history at query {len(asked)} {asked[-1:]}: {str(e)[:80]}')
        return None
    if len(res.history) != len(r.hist):
        bad.append(f'{len(r.hist)} GPU proposals, {len(res.history)} in the restatement')
    if asked != r.queries:
        k = next((i for i, (a, b) in enumerate(zip(asked, r.queries)) if a != b), min(len(asked), len(r.queries)))
        bad.append(f'queries differ from query {k} on (GPU {r.queries[k:k + 1]}, restatement {asked[k:k + 1]})')
    worst = 0.0
    for k, (g, h) in enumerate(zip(r.hist, res.history)):
        if (g.accepted, g.hit_dt_min) != (h.accepted, h.hit_dt_min):
            bad.append(f'proposal {k}: GPU accepted={g.accepted} hit={g.hit_dt_min}, restatement accepted='
                       f'{h.accepted} hit={h.hit_dt_min}')
            break
        e = abs(g.error - h.error) / (RTOL64 * h.error)
        worst = max(worst, e)
        if e > 1:
            bad.append(f'proposal {k}: error estimate {g.error!r}, restatement {h.error!r}')
            break
    ys_ref = res.ys[..., :-1] if c.logqp else res.ys
    worst = max(worst, _excess(r.ys, ys_ref, RTOL64))
    if c.logqp:
        lr_ref = (res.ys[1:, :, -1] - res.ys[:-1, :, -1])
        worst = max(worst, _excess(r.lr, lr_ref, RTOL64))
    _note(key, worst)
    if worst > 1:
        bad.append(f'worst err/bound {worst:.3g} (errors and ys)')
    return res


def check_free(c, expect_pass=True):
    r = gpu_solve(c)
    bad = []
    check_route_and_history(c, r, bad)
    compare_free(c, r, bad, (c.method + ('_gf' if c.opts else ''), 'float64') if expect_pass else None)
    if expect_pass:
        assert not bad, f'{case_id(c)} {c}: ' + '; '.join(bad)
    return r, bad


def err_bound(ref_full, ref_half, state_bound, c, err_ref):
    """How far an error estimate can move when y_full and y_half each move by up to d = state_bound scale: every
    ratio x = (y11 - y12) / tol moves by at most d (2 + rtol |x|) / tol, so the RMS by at most that with tol's least
    value; plus the float32 rounding of the GPU's per-element ratios (8 u relative)."""
    dlt = state_bound * max(adjoint_ref.scale(ref_full), adjoint_ref.scale(ref_half))
    tol = np.maximum(c.rtol * np.maximum(np.abs(ref_full), np.abs(ref_half)) + c.atol, adaptive_ref.EPS)
    x = np.abs(ref_full - ref_half) / tol
    return float(np.max(dlt * (2 + c.rtol * x) / tol)) + 8 * U32 * err_ref


def compare_driven32(c, r, query, asked, bad, key, rows=None, errors=True):
    """float32: the restatement follows the GPU's history; states, ys, errors and decisions within the f32 bound."""
    y0_ref = r.y0_ref if rows is None else r.y0_ref[rows]
    try:
        res = adaptive_ref.integrate_adaptive(restatement(c, r, query), y0_ref, r.ts_np, c.rtol, c.atol, c.dt_min,
                                              driven=r.hist, keep_states=True)
    except AssertionError as e:
        bad.append(f'the restatement could not follow the GPU history: {str(e)[:120]}')
        return
    if asked != r.queries:
        bad.append(f'{len(asked)} restatement queries differ from the {len(r.queries)} GPU queries')
    bound = f32_bound(len(asked))
    worst = 0.0
    for k, ((gf, gh), (hf, hh), g, h) in enumerate(zip(zip(r.full, r.half), res.states, r.hist, res.history)):
        w = max(_excess(gf, hf, bound), _excess(gh, hh, bound))
        worst = max(worst, w)
        if w > 1:
            bad.append(f'proposal {k} [{g.curr_t!r}, {g.next_t!r}]: y_full / y_half err/bound {w:.3g}')
            break
        if not errors:
            continue
        eb = err_bound(hf, hh, bound, c, h.error)
        e = abs(g.error - h.error) / eb
        worst = max(worst, e)
        if e > 1:
            bad.append(f'proposal {k}: error estimate {g.error!r}, restatement {h.error!r}, bound {eb:.3g}')
            break
        own = h.error <= 1 or g.hit_dt_min
        if own != g.accepted and not abs(h.error - 1) <= eb:
            bad.append(f'proposal {k} [{g.curr_t!r}, {g.next_t!r}]: GPU accepted={g.accepted} with error '
                       f'{g.error!r}; the restatement\'s error {h.error!r} is {abs(h.error - 1):.3g} from 1, beyond '
                       f'the bound {eb:.3g}')
            break
    got = r.ys if rows is None else r.ys[:, torch.as_tensor(rows, device=r.ys.device)]
    worst = max(worst, _excess(got, res.ys[..., :-1] if c.logqp else res.ys, bound))
    if c.logqp:
        worst = max(worst, _excess(r.lr, res.ys[1:, :, -1] - res.ys[:-1, :, -1], bound))
    _note(key, worst)
    if worst > 1:
        bad.append(f'worst err/bound {worst:.3g}')


def check_driven32(c):
    r = gpu_solve(c, rows=np.arange(c.B))
    bad = []
    check_route_and_history(c, r, bad)
    query, asked = adaptive_ref.increments(r.bm, np.float32)
    compare_driven32(c, r, query, asked, bad, (c.method + ('_gf' if c.opts else ''), 'float32'))
    assert not bad, f'{case_id(c)} {c}: ' + '; '.join(bad)


# ---- float64, free mode ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('c', MATRIX_CASES, ids=case_id)
def test_matrix_float64(c):
    check_free(c)


VARIANTS = {
    # outputs between accepted steps (interpolated) and a ts[-1] that clamps next_t
    'off-step outputs': case('milstein', 'ito', 'gbm', ts=(0.0, 0.13, 0.29, 0.5), seed=60),
    'off-step outputs unfused': case('heun', 'stratonovich', 'general', ts=(0.0, 0.13, 0.29, 0.5), seed=61),
    'grid dt': case('euler', 'ito', 'gbm', bm_dt=2.0 ** -6, seed=62),
    'grid dt srk': case('srk', 'ito', 'additive', bm_dt=2.0 ** -6, seed=63),
    'grid dt reversible': case('reversible_heun', 'stratonovich', 'scalar', bm_dt=0.03, seed=64),
    'dt tensor': case('midpoint', 'stratonovich', 'gbm', dt_tensor=True, seed=65),
    'logqp diagonal': case('euler', 'ito', 'gbm', d=3, logqp=True, seed=66),
    'logqp general': case('midpoint', 'stratonovich', 'general', d=3, m=2, logqp=True, seed=67),
    'logqp heun': case('heun', 'stratonovich', 'gbm', d=3, logqp=True, seed=68),
    'B=5 d=1': case('milstein', 'ito', 'gbm', B=5, d=1, seed=69),
    'B=5 d=3': case('srk', 'ito', 'gbm', B=5, d=3, seed=70),
    'B=5 d=5': case('euler_heun', 'stratonovich', 'gbm', B=5, d=5, seed=71),
    'B=7 d=3 unfused': case('euler', 'ito', 'gbm', B=7, d=3, coupled=True, seed=72),
    'B=6 d=5 reversible': case('reversible_heun', 'stratonovich', 'gbm', B=6, d=5, seed=73),
}


@pytest.mark.parametrize('name', list(VARIANTS))
def test_variants_float64(name):
    r, _ = check_free(VARIANTS[name])
    if 'off-step' in name:
        accepted_ends = {h.next_t for h in r.hist if h.accepted}
        assert any(float(t) not in accepted_ends for t in r.ts_np[1:-1]), 'no output fell between accepted steps'
        assert any(h.next_t == float(r.ts_np[-1]) and h.next_t - h.curr_t < 0.5 for h in r.hist)


@pytest.mark.parametrize('method,st', [('euler', 'ito'), ('milstein', 'ito'), ('heun', 'stratonovich'),
                                       ('reversible_heun', 'stratonovich')])
def test_a_solve_that_hits_dt_min(method, st):
    """A warning, then every proposal accepted at dt_min whatever its error."""
    c = case(method, st, 'gbm', rtol=1e-9, atol=1e-9, dt_min=0.02, ts=(0.0, 0.13, 0.2), dt=0.2, seed=80,
             vacuous=False)
    r, _ = check_free(c)
    assert r.warned
    assert any(h.hit_dt_min for h in r.hist) and any(h.accepted and h.error > 1 for h in r.hist)


@pytest.mark.parametrize('method,st,kind', [('milstein', 'ito', 'gbm'), ('srk', 'ito', 'scalar'),
                                            ('reversible_heun', 'stratonovich', 'general')])
def test_cuda_graph_option_gives_the_eager_bits(method, st, kind):
    """options={'cuda_graph': True} with adaptive=True runs the eager loop: the same bits and history."""
    c = case(method, st, kind, ts=(0.0, 0.2, 0.5), seed=90)
    eager = gpu_solve(c, graph=False)
    r, _ = check_free(c._replace(graph=True))
    assert torch.equal(eager.ys, r.ys)
    assert eager.hist == r.hist and eager.queries == r.queries


# ---- float32, driven mode --------------------------------------------------------------------------------------------
F32_CASES = [c._replace(dtype=torch.float32, B=5) for c in MATRIX_CASES] + [
    case('milstein', 'ito', 'gbm', dtype=torch.float32, B=5, d=1, ts=(0.0, 0.13, 0.29, 0.5), seed=100),
    case('euler', 'ito', 'gbm', dtype=torch.float32, B=6, d=3, bm_dt=2.0 ** -6, seed=101),
    case('heun', 'stratonovich', 'gbm', dtype=torch.float32, B=7, d=5, ts=(0.0, 0.13, 0.29, 0.5), seed=102),
    case('midpoint', 'stratonovich', 'gbm', dtype=torch.float32, B=5, d=3, logqp=True, seed=103),
]


@pytest.mark.parametrize('c', F32_CASES, ids=lambda c: case_id(c) + ('-logqp' if c.logqp else ''))
def test_float32_driven(c):
    check_driven32(c)


# ---- full batch ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('coupled', [False, True], ids=['fused', 'unfused'])
def test_full_batch_float32(coupled):
    B, d = 2 ** 20 + 3, 3
    need = 4 << 30
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f'{free} bytes of device memory free, {need} needed')
    c = case('milstein', 'ito', 'gbm', coupled=coupled, dtype=torch.float32, B=B, d=d, ts=(0.0, 0.2, 0.4), dt=0.4,
             seed=110)
    rows = np.unique(np.r_[helpers.sample_rows(B, 256, seed=110), 1, B - 2])
    sums = []

    def recompute(solver, y_full, y_half, err):
        a, b = y_full.reshape(-1), y_half.reshape(-1)
        tol = (torch.maximum(a.abs(), b.abs()) * solver.rtol + solver.atol).clamp_min(adaptive_ref.EPS)
        x = (a - b) / tol
        spec = math.sqrt(float((x * x).double().sum()) / a.numel())
        a64, b64 = a.double(), b.double()
        tol64 = (torch.maximum(a64.abs(), b64.abs()) * solver.rtol + solver.atol).clamp_min(adaptive_ref.EPS)
        f64 = math.sqrt(float((((a64 - b64) / tol64) ** 2).sum()) / a.numel())
        sums.append((err, max(spec, adaptive_ref.EPS), max(f64, adaptive_ref.EPS)))

    r = gpu_solve(c, rows=rows, on_error=recompute)
    bad = []
    check_route_and_history(c, r, bad)
    for k, (err, spec, f64) in enumerate(sums):
        if abs(err - spec) > 1e-12 * spec:
            bad.append(f'proposal {k}: error estimate {err!r}, its float32-ratio recomputation {spec!r}')
        if abs(err - f64) > 8 * U32 * f64:
            bad.append(f'proposal {k}: error estimate {err!r}, its float64 recomputation {f64!r}')
    query, asked = adaptive_ref.increments(r.bm, np.float32, rows=rows)
    compare_driven32(c, r, query, asked, bad, ('milstein full batch', 'float32'), rows=rows, errors=False)
    print(f'full batch {"unfused" if coupled else "fused"}: {len(r.hist)} proposals, {len(rows)} rows restated')
    assert not bad, '; '.join(bad[:8])


# ---- gradients through an adaptive solve ------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['gbm', 'additive'])
@pytest.mark.parametrize('method', ['euler', 'milstein', 'srk', 'heun', 'midpoint'])
def test_gradients_against_central_differences(method, kind):
    tsde = _tsde()
    st = 'stratonovich' if method in ('heun', 'midpoint') else 'ito'
    c = case(method, st, kind, B=2, d=3, seed=120)
    dev = problem(c, torch.float64).to(DEV)
    cpu = problem(c, torch.float64)
    y0 = 0.1 + 0.5 * torch.rand(c.B, c.d, generator=torch.Generator().manual_seed(120), dtype=torch.float64)
    ts_np = np.asarray(c.ts)
    bm = tsde.BrownianInterval(0.0, float(ts_np[-1]), size=(c.B, c.m), dtype=torch.float64, device=DEV, entropy=9,
                               levy_area_approximation='space-time' if method == 'srk' else 'none')
    y0_dev = y0.to(DEV).requires_grad_()
    w = torch.linspace(0.5, 1.5, len(ts_np) * c.B * c.d, dtype=torch.float64).reshape(len(ts_np), c.B, c.d)
    with spy() as seen, warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ys = tsde.sdeint(dev, y0_dev, torch.from_numpy(ts_np).to(DEV), bm=bm, method=method, dt=c.dt, adaptive=True,
                         rtol=c.rtol, atol=c.atol, dt_min=c.dt_min)
        (ys * w.to(DEV)).sum().backward()
    hist = gpu_history(seen, c.dt_min)
    assert any(not h.accepted for h in hist), 'no proposal was rejected'
    query, _ = adaptive_ref.increments(bm, np.float64)
    y0_cpu = y0.clone()

    def fn():
        solver = solvers.make(method, problems.NumpySDE(cpu), query, c.dt, {})
        return torch.from_numpy(adaptive_ref.integrate_adaptive(solver, y0_cpu.numpy(), ts_np, c.rtol, c.atol,
                                                                c.dt_min, driven=hist).ys)
    params = list(cpu.parameters())
    out, jacs = gradient_ref.central_jacobian(fn, [y0_cpu] + params)
    assert _excess(ys, out.numpy(), RTOL64) <= 1
    grads = [y0_dev.grad.cpu()] + [p.grad.cpu() for p in dev.parameters()]
    bad = gradient_ref.check_vjp(out, jacs, w, grads, label=f'{method} {kind}')
    assert not bad, '; '.join(bad)


# ---- the comparisons must be able to fail -----------------------------------------------------------------------------
MUTATION_CASE = case('euler', 'ito', 'gbm', ts=(0.0, 0.13, 0.29, 0.5), seed=130)


def _first_half_gets_second_half(real):
    def propose(solver, curr_t, next_t, midpoint_t, y, extra):
        bm = solver.bm

        def served(ta, tb, return_U=False):
            if (float(ta), float(tb)) == (float(curr_t), float(midpoint_t)):
                ta, tb = midpoint_t, next_t
            return bm(ta, tb, return_U)
        solver.bm = served
        try:
            return real(solver, curr_t, next_t, midpoint_t, y, extra)
        finally:
            solver.bm = bm
    return propose


def _divisor_short_by_one(y11, y12, rtol, atol, eps=adaptive_ref.EPS):
    y11, y12 = np.asarray(y11, np.float64), np.asarray(y12, np.float64)
    tol = np.maximum(rtol * np.maximum(np.abs(y11), np.abs(y12)) + atol, eps)
    x = (y11 - y12) / tol
    return float(max(np.sqrt((x ** 2).sum() / (x.size - 1)), eps))


def _weights_swapped(t0, y0, t1, y1, t):
    w0 = (t1 - t) / (t1 - t0)
    w1 = (t - t0) / (t1 - t0)
    return y0.dtype.type(w1) * y0 + y0.dtype.type(w0) * y1


def _neighbour_row(real):
    def increments(bm, npdt, rows=None):
        query, asked = real(bm, npdt, rows)

        def neighbour(x):
            x = np.array(x, copy=True)
            x[0] = x[1]
            return x

        def served(ta, tb, return_U=False):
            out = query(ta, tb, return_U)
            return tuple(neighbour(x) for x in out) if return_U else neighbour(out)
        return served, asked
    return increments


MUTATIONS = {
    'first half step gets the second half step increment': ('propose', _first_half_gets_second_half),
    'error estimate divided by numel - 1': ('error_estimate', lambda real: _divisor_short_by_one),
    'interpolation weights swapped': ('linear_interp', lambda real: _weights_swapped),
    'row 0 gets row 1 increments': ('increments', _neighbour_row),
}


def test_the_mutation_case_passes_unmutated():
    check_free(MUTATION_CASE)


@pytest.mark.parametrize('name', list(MUTATIONS))
def test_mutation_fails_the_comparison(name, monkeypatch):
    attr, make = MUTATIONS[name]
    monkeypatch.setattr(adaptive_ref, attr, make(getattr(adaptive_ref, attr)))
    _, bad = check_free(MUTATION_CASE, expect_pass=False)
    assert bad, f'{name}: the comparison passed'


def test_report_worst_err_over_bound():
    """Runs last: prints the worst err/bound per (method, dtype) over the module."""
    for (meth, dt), r in sorted(WORST.items()):
        print(f'adaptive worst err/bound  {meth:20s} {dt:8s} {r:.3g}')
    assert all(r <= 1.0 for r in WORST.values())
