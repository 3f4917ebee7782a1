"""Gradients of `sdeint` and of `sdeint_adjoint`'s reversible pair against float64 central differences of the forward
solve (tests/gradient_ref.py), on counter noise: a `BrownianInterval` bound to the solver grid, whose increments the
autograd path materialises (NoiseFeed.tensors) and feeds back to the tableau kernels (NoiseFeed.from_tensors).  Every
forward solve builds a fresh interval with the same entropy, so the perturbed solves see the same increments; they run
with options={'overlap': False}, the unfused tableau kernels the autograd path launches.

(a) Small shapes, float64, the full Jacobian (B = 3, d in {2, 3}, m in {1, 2, 3}; outputs on the grid and between grid
    points, the latter through tsde_linear_interp's backward), w.r.t. y0 and every parameter:

        method              sde_type        diagonal  scalar  additive  general   protocols
        euler               ito             x         x       x         x         fused, g_prod, f_and_g_prod
        milstein            ito, strat      x         x       x                   fused (+ g_prod: additive)
        milstein grad-free  ito, strat      x         x                           fused
        srk                 ito             x         x       x                   fused (+ g_prod: additive)
        midpoint            strat           x         x       x         x         fused, g_prod, f_and_g_prod
        heun                strat           x         x       x         x         fused, g_prod, f_and_g_prod
        euler_heun          strat           x         x       x         x         fused, g_prod, f_and_g_prod
        reversible_heun     strat           x         x       x         x         fused
        log_ode             strat           x         x       x         x         fused (+ g_prod, f_and_g_prod: not
                                                                                  general)

    Every other (method, noise, protocol) must raise rather than return a None gradient
    (test_refused_combinations_raise); which ones the library refuses is pinned against the reference in
    test_oracle_live_reference.  Also: a tensor f closes over that is not a parameter (the probe_requires_grad
    route), reversible Heun's `extra_solver_state`, and the log-ratio of `logqp=True` for diagonal and general noise.

(b) Route shapes, float64, one directional check per trajectory (gradient_ref.rowwise_directional), y0 and the
    per-trajectory (B, d) parameters of GBMPerTrajectory moved together, shared parameters along random directions:

        diagonal   euler, milstein, srk, heun, reversible_heun    d in {1, 3, 5, 33}, B in {1, 97, 4099}
        general    euler, midpoint, heun, euler_heun,             m in {1, 3, 4, 16, 32, 64} at B = 97, d = 4 (m = 1:
                   reversible_heun, srk (additive)                row-wise kernels / gen_kernel at m = 1, 3; else
                                                                  gen_cta_kernel), m = 5124 / 2564
                                                                  (with U) at B = 3 (gen_wide_kernel), m = 64 at
                                                                  B = 2100, d = 64 (gen_tma_kernel, one-g tableaus);
                                                                  dense g, and additive g = S.expand(B, d, m)
    The autograd solve's route is confirmed with the tile-kernel launch counters.  Under autograd an expanded g is
    made dense for the launch and its gradient reaches the (d, m) block through expand's backward; the forward solves
    of the central differences read the shared block (TSDE_FLAG_G_BROADCAST).

(c) The float32 gradient of every (b) case, per row, against the float64 central difference of the same solve on the
    float32 solve's increments.
(d) sdeint_adjoint with the reversible pair: the exact gradient of the discrete solve (output times on the step grid),
    so the same checks as (a) and (b); eagerly and with adjoint_options={'cuda_graph': True}, and with a strict subset
    of adjoint_params.
(e) Second order: central differences of verified first-order gradients against create_graph double backward, for
    plain sdeint (midpoint, Milstein, general-noise Euler) and the reversible pair (_ReversibleVJP).
(f) A coefficient of the transpose table scaled by (1 + 1e-5) makes (a) and (b) fail.
"""
import copy

import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200._core import autograd_ops
from . import gradient_ref as gr
from . import problems

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DT = 2.0 ** -4
T1 = 0.25
TS_GRID = (0.0, 0.125, 0.25)
TS_INTERP = (0.0, 0.1, 0.25)          # 0.1 lies between grid points: tsde_linear_interp
LEVY = {'srk': 'space-time', 'log_ode': 'foster'}
NO_FUSE = {'overlap': False}
GEN_CTA, GEN_TMA, GEN_WIDE = 0, 1, 2  # tsde_kernel_launches families
U32 = 2.0 ** -24


def _launches():
    from torchsde_b200 import _cabi
    lib = _cabi.lib()
    return tuple(lib.tsde_kernel_launches(f) for f in (GEN_CTA, GEN_TMA, GEN_WIDE))


def _bm(B, m, dtype, method, entropy=11):
    return tsde.BrownianInterval(0.0, T1, size=(B, m), dtype=dtype, device=DEV, entropy=entropy,
                                 levy_area_approximation=LEVY.get(method, 'none'))


class Closed:
    """Not a Module: f closes over the tensor k, which is no parameter (sdeint finds it through the probe)."""

    def __init__(self, base, k):
        self.base, self.k = base, k
        self.noise_type, self.sde_type = base.noise_type, base.sde_type

    def f(self, t, y):
        return self.base.f(t, y) + self.k * torch.sin(y)

    def g(self, t, y):
        return self.base.g(t, y)


def _problem(kind, d, m, sde_type, dtype=torch.float64, seed=1):
    if kind == 'diagonal':
        sde = problems.LatentPrior(d, 1, 'diagonal', sde_type, seed=seed, dtype=dtype)
        sde.S.requires_grad_(False)  # (diagonal noise does not use it)
        return sde.to(DEV)
    return problems.make({'scalar': 'scalar', 'additive': 'additive', 'general': 'general'}[kind], d, m, sde_type,
                         dtype=dtype, seed=seed).to(DEV)


def _bm_m(kind, d, m):
    return {'diagonal': d, 'scalar': 1}.get(kind, m)


# ---- (a) the full matrix at small shapes ------------------------------------------------------------------------
ITO = [('euler', k) for k in ('diagonal', 'scalar', 'additive', 'general')] + \
      [('milstein', k) for k in ('diagonal', 'scalar', 'additive')] + \
      [('milstein_gf', k) for k in ('diagonal', 'scalar')] + [('srk', k) for k in ('diagonal', 'scalar', 'additive')]
STRAT = [(mth, k) for mth in ('midpoint', 'heun', 'euler_heun', 'reversible_heun', 'log_ode')
         for k in ('diagonal', 'scalar', 'additive', 'general')] + \
        [('milstein', k) for k in ('diagonal', 'scalar', 'additive')] + \
        [('milstein_gf', k) for k in ('diagonal', 'scalar')]
SHAPES = {'diagonal': [(2, 2, TS_GRID), (3, 3, TS_INTERP)], 'scalar': [(2, 1, TS_INTERP), (3, 1, TS_GRID)],
          'additive': [(2, 1, TS_GRID), (3, 2, TS_INTERP), (2, 3, TS_GRID)],
          'general': [(2, 1, TS_INTERP), (3, 2, TS_GRID), (2, 3, TS_INTERP)]}
MATRIX = [(mth, st, k, d, m, ts, 'fused') for st, combos in (('ito', ITO), ('stratonovich', STRAT))
          for mth, k in combos for d, m, ts in SHAPES[k]]
PROTOCOLS = {'g_prod': ('f', 'g_prod'), 'f_and_g_prod': ('f_and_g_prod',)}
ACCEPTED_PROTOCOLS = [(mth, st, k, 3, _bm_m(k, 3, 2) if k != 'diagonal' else 3, TS_INTERP, p)
                      for st, combos in (('ito', ITO), ('stratonovich', STRAT)) for mth, k in combos
                      for p in PROTOCOLS
                      if (mth in ('euler', 'midpoint', 'heun', 'euler_heun'))
                      or (mth in ('milstein', 'srk') and k == 'additive' and p == 'g_prod')
                      or (mth == 'log_ode' and k != 'general')]


def _case_id(c):
    mth, st, k, d, m, ts, p = c
    return f"{mth}-{st[:5]}-{k}-d{d}m{m}-{'grid' if ts == TS_GRID else 'interp'}" + ('' if p == 'fused' else '-' + p)


def _setup(case, seed=1):
    """(solve, inputs) of an (a) case: solve() returns the flattened output of a fresh solve."""
    mth, st, kind, d, m, ts, protocol = case
    B = 3
    base = _problem(kind, d, m, st, seed=seed)
    sde = base if protocol == 'fused' else problems.WithProds(base, PROTOCOLS[protocol])
    gen = torch.Generator(device=DEV).manual_seed(seed)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).requires_grad_(True)
    ts_t = torch.tensor(ts, dtype=torch.float64, device=DEV)
    method = 'milstein' if mth == 'milstein_gf' else mth
    options = dict(NO_FUSE, grad_free=True) if mth == 'milstein_gf' else NO_FUSE
    bm_m = _bm_m(kind, d, m)

    def solve():
        return tsde.sdeint(sde, y0, ts_t, bm=_bm(B, bm_m, torch.float64, method), method=method, dt=DT,
                           options=options).reshape(-1)
    return solve, [y0] + [p for p in base.parameters() if p.requires_grad]


def _autograd_jacobian(solve, inputs):
    """Autograd's full Jacobian of solve() w.r.t. each input: one backward per output (None where it gives none)."""
    out = solve()
    rows = [[] for _ in inputs]
    for o in range(out.numel()):
        gs = torch.autograd.grad(out[o], inputs, retain_graph=True, allow_unused=True)
        for i, g in enumerate(gs):
            rows[i].append(None if g is None else g.reshape(-1))
    return [None if any(r is None for r in rs) else torch.stack(rs) for rs in rows]


def full_check(solve, inputs, label):
    """(a)'s check: the autograd Jacobian against the central-difference one; a list of failures."""
    out, jacs = gr.central_jacobian(solve, inputs)
    return gr.check_jacobian(out, jacs, _autograd_jacobian(solve, inputs), label)


@pytest.mark.parametrize('case', MATRIX + ACCEPTED_PROTOCOLS, ids=_case_id)
def test_small_full_jacobian(case):
    solve, inputs = _setup(case)
    bad = full_check(solve, inputs, _case_id(case))
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('method', ['euler', 'milstein', 'srk', 'heun', 'reversible_heun', 'midpoint'])
def test_closed_over_tensor(method):
    """A tensor f closes over, not a parameter of any Module: sdeint finds that gradients must flow by probing f."""
    st = 'ito' if method in ('euler', 'milstein', 'srk') else 'stratonovich'
    base = _problem('diagonal', 3, 3, st)
    base.requires_grad_(False)
    k = torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64, device=DEV, requires_grad=True)
    sde = Closed(base, k)
    y0 = torch.tensor([[0.3, 0.5, 0.7]] * 3, dtype=torch.float64, device=DEV)
    ts = torch.tensor(TS_INTERP, dtype=torch.float64, device=DEV)

    def solve():
        return tsde.sdeint(sde, y0, ts, bm=_bm(3, 3, torch.float64, method), method=method, dt=DT,
                           options=NO_FUSE).reshape(-1)
    bad = full_check(solve, [k], f'{method} closed-over k')
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('kind', ['diagonal', 'general'])
def test_reversible_heun_extra_solver_state(kind):
    """Gradients w.r.t. the solver state (f0, g0, z0) handed to a reversible-Heun solve, and w.r.t. y0."""
    d, m, B = 3, 2, 3
    sde = _problem(kind, d, m, 'stratonovich')
    sde.requires_grad_(False)
    gen = torch.Generator(device=DEV).manual_seed(4)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).requires_grad_(True)
    t0 = torch.zeros((), dtype=torch.float64, device=DEV)
    with torch.no_grad():
        f0, g0 = sde.f(t0, y0), sde.g(t0, y0)
    state = [(f0 + 0.01).clone().requires_grad_(True), (g0 * 1.01).clone().requires_grad_(True),
             (y0 + 0.02).detach().clone().requires_grad_(True)]
    ts = torch.tensor(TS_GRID, dtype=torch.float64, device=DEV)
    bm_m = d if kind == 'diagonal' else m

    def solve():
        return tsde.sdeint(sde, y0, ts, bm=_bm(B, bm_m, torch.float64, 'reversible_heun'), method='reversible_heun',
                           dt=DT, options=NO_FUSE, extra_solver_state=tuple(state)).reshape(-1)
    bad = full_check(solve, [y0] + state, f'reversible_heun {kind} extra_solver_state')
    assert not bad, '\n'.join(bad)


LOGQP = [('euler', 'ito', 'diagonal'), ('milstein', 'ito', 'diagonal'), ('srk', 'ito', 'diagonal'),
         ('midpoint', 'stratonovich', 'diagonal'), ('reversible_heun', 'stratonovich', 'diagonal'),
         ('euler', 'ito', 'general'), ('midpoint', 'stratonovich', 'general'), ('heun', 'stratonovich', 'general')]


@pytest.mark.parametrize('method,st,noise', LOGQP, ids=['-'.join(c) for c in LOGQP])
def test_logqp_log_ratio(method, st, noise):
    """`logqp=True`: the gradients of the path and of the log-ratio increments w.r.t. y0 and the parameters."""
    d, m, B = 3, 2, 3
    sde = problems.LatentPrior(d, m, noise, st, seed=2).to(DEV)
    (sde.S if noise == 'diagonal' else sde.s).requires_grad_(False)  # (the parameter this noise type does not use)
    gen = torch.Generator(device=DEV).manual_seed(5)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).requires_grad_(True)
    ts = torch.tensor(TS_INTERP, dtype=torch.float64, device=DEV)
    bm_m = d + 1 if noise == 'diagonal' else m  # (a diagonal-noise logqp solve has one channel more)

    def solve():
        ys, lr = tsde.sdeint(sde, y0, ts, bm=_bm(B, bm_m, torch.float64, method), method=method, dt=DT,
                             options=NO_FUSE, logqp=True)
        return torch.cat([ys.reshape(-1), lr.reshape(-1)])
    bad = full_check(solve, [y0] + [p for p in sde.parameters() if p.requires_grad], f'logqp {method} {noise}')
    assert not bad, '\n'.join(bad)


REFUSED_CANDIDATES = [(mth, st, k, p) for st, combos in (('ito', ITO), ('stratonovich', STRAT)) for mth, k in combos
                      for p in PROTOCOLS
                      if (mth, st, k, 3, _bm_m(k, 3, 2) if k != 'diagonal' else 3, TS_INTERP, p)
                      not in ACCEPTED_PROTOCOLS]


@pytest.mark.parametrize('mth,st,kind,protocol', REFUSED_CANDIDATES, ids=['-'.join(c) for c in REFUSED_CANDIDATES])
def test_refused_combinations_raise(mth, st, kind, protocol):
    """The (method, noise, protocol) combinations outside (a)'s matrix: the solve under autograd raises, the same error
    as without autograd; it never hands back a None gradient."""
    solve, inputs = _setup((mth, st, kind, 3, _bm_m(kind, 3, 2), TS_INTERP, protocol))
    errors = []
    for grad_mode in (True, False):
        with torch.set_grad_enabled(grad_mode):
            try:
                out = solve()
            except (ValueError, AttributeError, NotImplementedError, RuntimeError) as e:
                errors.append(type(e))
                continue
        if grad_mode:
            gs = torch.autograd.grad(out.sum(), inputs, allow_unused=True)
            assert all(g is not None for g in gs), 'accepted under autograd but a gradient is None'
            pytest.fail('accepted under autograd with gradients: add it to the matrix of (a)')
    assert errors and errors[0] == errors[-1] and len(errors) == 2, errors


# ---- (b) route shapes, per-row directional checks ---------------------------------------------------------------
DIAG_ROUTES = [(mth, d, B) for mth in ('euler', 'milstein', 'srk', 'heun', 'reversible_heun')
               for d in (1, 3, 5, 33) for B in (1, 97, 4099)]
GEN_METHODS = ('euler', 'midpoint', 'heun', 'euler_heun', 'reversible_heun', 'srk')
# (method, kind, B, d, m, expected route: None row-wise, else the counter family that must advance alone)
GEN_ROUTES = [(mth, kind, 97, 4, m, None if m in (1, 3) else GEN_CTA)
              for mth in GEN_METHODS for kind in ('dense', 'expand') for m in (1, 3, 4, 16, 32, 64)] + \
             [(mth, 'dense', 3, 2, 2564 if mth == 'srk' else 5124, GEN_WIDE) for mth in GEN_METHODS] + \
             [(mth, 'dense', 2100, 64, 64, GEN_TMA) for mth in ('euler', 'midpoint')]


def _diag_id(c):
    return f'{c[0]}-d{c[1]}-B{c[2]}'


def _gen_id(c):
    return f'{c[0]}-{c[1]}-B{c[2]}-d{c[3]}-m{c[4]}'


def _route_problem(case, dtype):
    """(sde, y0, per-row parameter tensors, shared parameters, method, sde_type, m) of a (b) case in `dtype`; the
    float32 problem holds the float64 one's values rounded."""
    if len(case) == 3:
        mth, d, B = case
        st = 'ito' if mth in ('euler', 'milstein', 'srk') else 'stratonovich'
        sde = problems.GBMPerTrajectory(B, d, st, seed=d, dtype=torch.float64).to(DEV).to(dtype)
        rows, shared, m = [sde.mu, sde.sigma], [], d
    else:
        mth, kind, B, d, m, _ = case
        st = 'ito' if mth in ('euler', 'srk') else 'stratonovich'
        if mth == 'srk' or kind == 'expand':
            sde = problems.make('additive_expand' if kind == 'expand' else 'additive', d, m, st, seed=m,
                                dtype=torch.float64)
            with torch.no_grad():
                sde.a.mul_(m ** -0.5)
        else:
            sde = problems.make('general', d, m, st, seed=m, dtype=torch.float64)
            with torch.no_grad():
                sde.S.mul_(m ** -0.5)  # the noise term of a step stays O(1) at any width
        sde = sde.to(DEV).to(dtype)
        rows, shared = [], list(sde.parameters())
    gen = torch.Generator(device=DEV).manual_seed(B + d)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).to(dtype).requires_grad_(True)
    return sde, y0, rows, shared, mth, st, m


def _route_solver(sde, y0, mth, m, dtype, adjoint=False, adjoint_options=None, adjoint_params=None, bm_factory=_bm,
                  ts_dtype=None):
    # (the reversible pair's adjoint is the exact gradient of the discrete solve when the output times lie on its grid:
    # its backward sweep steps back from each output time)
    ts = torch.tensor(TS_GRID if adjoint else TS_INTERP, dtype=ts_dtype or dtype, device=DEV).to(dtype)
    B = y0.shape[0]

    def solve():
        bm = bm_factory(B, m, dtype, mth)
        if adjoint:
            return tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun',
                                       adjoint_method='adjoint_reversible_heun', dt=DT, options=NO_FUSE,
                                       adjoint_options=adjoint_options, adjoint_params=adjoint_params)
        return tsde.sdeint(sde, y0, ts, bm=bm, method=mth, dt=DT, options=NO_FUSE)
    return solve


def _weights(shape, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=gen, dtype=torch.float64, device=DEV)


def rowwise_check(case, adjoint=False, adjoint_options=None, subset=False, check_route=True):
    """(b)'s check of one case.  Returns (failures, the gradients of y0 / per-row / shared parameters)."""
    sde, y0, rows, shared, mth, st, m = _route_problem(case, torch.float64)
    params = rows + shared
    adjoint_params = None
    if subset:  # a strict subset: the first shared parameter only
        adjoint_params = shared[:1]
    solve = _route_solver(sde, y0, mth, m, torch.float64, adjoint, adjoint_options, adjoint_params)
    before = _launches()
    ys = solve()
    after = _launches()
    w = _weights(ys.shape, 7)
    wanted = [y0] + (params if adjoint_params is None else rows + adjoint_params)
    grads = torch.autograd.grad((w * ys).sum(), wanted, allow_unused=True)
    label = _gen_id(case) if len(case) > 3 else _diag_id(case)
    bad = []
    if any(g is None for g in grads):
        return [f'{label}: a gradient is None'], None
    if check_route and len(case) > 3:  # (a general case: its expected tile-kernel family)
        expect = case[5]
        delta = [a - b for a, b in zip(after, before)]
        ok = all(x == 0 for x in delta) if expect is None else \
            (delta[expect] > 0 and all(x == 0 for i, x in enumerate(delta) if i != expect))
        if not ok:
            bad.append(f'{label}: (cta, tma, wide) launches {delta}, expected only family {expect}')
    g_y0, g_rows = grads[0], grads[1:1 + len(rows)]
    g_shared = grads[1 + len(rows):]
    V = _weights(y0.shape, 8)
    Vr = [_weights(p.shape, 9 + i) for i, p in enumerate(rows)]
    D, L = gr.rowwise_directional(solve, y0, V, w, row_inputs=list(zip(rows, Vr)))
    got = (g_y0 * V).sum(1) + sum((g * v).sum(1) for g, v in zip(g_rows, Vr))
    ok = gr.within(got, D, L)
    if not bool(ok.all()):
        r = int((~ok).nonzero()[0])
        bad.append(f'{label}: {int((~ok).sum())} of {ok.numel()} rows off the central difference (row {r}: '
                   f'autograd {got[r].item():.17g}, central difference {D[r].item():.17g}, scale {L[r].item():.3g})')
    checked = shared if adjoint_params is None else adjoint_params
    for k in range(3 if checked else 0):
        dirs = [_weights(p.shape, 20 + 3 * k + i) for i, p in enumerate(checked)]
        Dp, Lp = gr.directional(solve, checked, dirs, w)
        gp = sum(float((g * v).sum()) for g, v in zip(g_shared[:len(checked)], dirs))
        if not bool(gr.within(gp, Dp, Lp)):
            bad.append(f'{label}: shared parameters along direction {k}: autograd {gp:.17g}, central difference '
                       f'{Dp:.17g}, scale {Lp:.3g}')
    return bad, (g_y0, g_rows, g_shared)


@pytest.mark.parametrize('case', DIAG_ROUTES, ids=_diag_id)
def test_route_rowwise_diagonal(case):
    bad, _ = rowwise_check(case)
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('case', GEN_ROUTES, ids=_gen_id)
def test_route_rowwise_general(case):
    bad, _ = rowwise_check(case)
    assert not bad, '\n'.join(bad)


# ---- (c) float32 gradients --------------------------------------------------------------------------------------
# A float32 BrownianInterval draws its normals from other Philox words than a float64 one (oracle/philox.py), so the
# float32 gradient is compared with the float64 central difference of the same solve on the increments the float32
# autograd solve materialised (widened exactly, served as memory noise), from its inputs and output times widened.
C32 = 4  # ulp of float32 per rounded operation along the solve and its backward


def _recording_increments(monkeypatch):
    """Record every increment NoiseFeed materialises from now on: {(t0, t1): (W, U)}."""
    from torchsde_b200._core import base_solver
    real, seen = base_solver.NoiseFeed._tensors, {}

    def spy(self, c, want_u):
        w, u = real(self, c, want_u)
        seen[(c.ft0, c.ft1)] = (w.clone(), None if u is None else u.clone())
        return w, u
    monkeypatch.setattr(base_solver.NoiseFeed, '_tensors', spy)
    return seen


def _widened_replay(seen, levy):
    keys = sorted(seen)
    want_u = all(seen[k][1] is not None for k in keys)
    return problems.ReplayBM([k[0] for k in keys], [k[1] for k in keys], [seen[k][0].double() for k in keys],
                             [seen[k][1].double() for k in keys] if want_u else None, levy=levy)


@pytest.mark.parametrize('case', DIAG_ROUTES + GEN_ROUTES, ids=lambda c: _diag_id(c) if len(c) == 3 else _gen_id(c))
def test_route_float32_gradient(case, monkeypatch):
    """Per row, |g32 . V - D| <= (C32 (N_OPS + m) u32 + RTOL) (L + |D|): the float32 solve and its backward round at
    most N_OPS times per element plus the m products of each g.dW, each rounding by at most C32 ulp of the row's scale;
    RTOL is the central difference's own bound.  A float32-only routing or dtype error is an O(1) difference."""
    sde32, y32, rows32, shared32, mth, st, m = _route_problem(case, torch.float32)
    solve32 = _route_solver(sde32, y32, mth, m, torch.float32)
    seen = _recording_increments(monkeypatch)
    ys = solve32()
    monkeypatch.undo()
    w = _weights(ys.shape, 7)
    g32 = [g.double() for g in torch.autograd.grad((w.float() * ys).sum(), [y32] + rows32 + shared32)]
    sde = copy.deepcopy(sde32).to(torch.float64)
    y0 = y32.detach().double()
    rows = [sde.mu, sde.sigma] if rows32 else []
    shared = [] if rows32 else list(sde.parameters())
    replay = _widened_replay(seen, LEVY.get(mth, 'none'))
    solve = _route_solver(sde, y0, mth, m, torch.float64, bm_factory=lambda *_: replay, ts_dtype=torch.float32)
    V = _weights(y0.shape, 8)
    Vr = [_weights(p.shape, 9 + i) for i, p in enumerate(rows)]
    D, L = gr.rowwise_directional(solve, y0, V, w, row_inputs=list(zip(rows, Vr)))
    got = (g32[0] * V).sum(1) + sum((g * v).sum(1) for g, v in zip(g32[1:1 + len(rows)], Vr))
    rel = C32 * (gr.N_OPS + m) * U32 + gr.RTOL
    bad = []
    err = (got - D).abs() / (L + D.abs())
    if float(err.max()) > rel:
        r = int(torch.argmax(err))
        bad.append(f'{int((err > rel).sum())} of {err.numel()} rows off (row {r}: float32 {got[r].item():.9g}, '
                   f'float64 central difference {D[r].item():.9g}, relative {err[r].item():.3g} > {rel:.3g})')
    if shared:
        dirs = [_weights(p.shape, 20 + i) for i, p in enumerate(shared)]
        Dp, Lp = gr.directional(solve, shared, dirs, w)
        gp = sum(float((g * v).sum()) for g, v in zip(g32[1 + len(rows):], dirs))
        if abs(gp - Dp) > rel * (Lp + abs(Dp)):
            bad.append(f'shared parameters: float32 {gp:.9g}, float64 central difference {Dp:.9g}')
    assert not bad, '\n'.join(bad)


# ---- (d) the reversible pair's adjoint --------------------------------------------------------------------------
ADJ_SMALL = [(k, opts) for k in ('diagonal', 'scalar', 'additive', 'general') for opts in ('eager', 'graph')]


@pytest.mark.parametrize('kind,mode', ADJ_SMALL, ids=[f'{k}-{o}' for k, o in ADJ_SMALL])
def test_adjoint_reversible_pair_small(kind, mode):
    d, m, B = 3, 2, 3
    sde = _problem(kind, d, m, 'stratonovich')
    gen = torch.Generator(device=DEV).manual_seed(6)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).requires_grad_(True)
    ts = torch.tensor(TS_GRID, dtype=torch.float64, device=DEV)  # (on the grid: see _route_solver)
    opts = {'cuda_graph': True} if mode == 'graph' else None
    bm_m = _bm_m(kind, d, m)

    def solve():
        return tsde.sdeint_adjoint(sde, y0, ts, bm=_bm(B, bm_m, torch.float64, 'reversible_heun'),
                                   method='reversible_heun', adjoint_method='adjoint_reversible_heun', dt=DT,
                                   options=NO_FUSE, adjoint_options=opts).reshape(-1)
    params = [p for p in sde.parameters() if p.requires_grad]
    bad = full_check(solve, [y0] + params, f'adjoint {kind} {mode}')
    assert not bad, '\n'.join(bad)


ADJ_ROUTES = [(c, opts, subset) for c in GEN_ROUTES if c[0] == 'reversible_heun' and c[4] in (1, 16, 64, 5124)
              for opts, subset in (('eager', False), ('graph', False), ('eager', True))]


@pytest.mark.parametrize('case,mode,subset', ADJ_ROUTES,
                         ids=[f'{_gen_id(c)}-{o}' + ('-subset' if s else '') for c, o, s in ADJ_ROUTES])
def test_adjoint_reversible_pair_routes(case, mode, subset):
    bad, _ = rowwise_check(case, adjoint=True, adjoint_options={'cuda_graph': True} if mode == 'graph' else None,
                           subset=subset, check_route=False)
    assert not bad, '\n'.join(bad)


# ---- (e) second order -------------------------------------------------------------------------------------------
SECOND = [('midpoint', 'stratonovich', 'diagonal', False), ('milstein', 'ito', 'diagonal', False),
          ('milstein', 'stratonovich', 'scalar', False), ('euler', 'ito', 'general', False),
          ('reversible_heun', 'stratonovich', 'diagonal', True), ('reversible_heun', 'stratonovich', 'general', True)]


@pytest.mark.parametrize('method,st,kind,adjoint', SECOND, ids=[f'{c[0]}-{c[2]}' + ('-adjoint' if c[3] else '')
                                                                 for c in SECOND])
def test_second_order(method, st, kind, adjoint):
    """H u (double backward with create_graph) against the central difference of the first-order gradient along u,
    element by element within RTOL (max |grad| + |D|)."""
    d, m, B = 3, 2, 3
    sde = _problem(kind, d, m, st)
    params = [p for p in sde.parameters() if p.requires_grad]
    gen = torch.Generator(device=DEV).manual_seed(8)
    y0 = (0.2 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64, device=DEV)).requires_grad_(True)
    ts = torch.tensor(TS_GRID, dtype=torch.float64, device=DEV)
    bm_m = _bm_m(kind, d, m)
    inputs = [y0] + params
    w = _weights((len(TS_GRID), B, d), 3)

    def first(create_graph=False):
        bm = _bm(B, bm_m, torch.float64, method)
        if adjoint:
            ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method=method, adjoint_method='adjoint_reversible_heun',
                                     dt=DT, options=NO_FUSE)
        else:
            ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=DT, options=NO_FUSE)
        return torch.autograd.grad((w * ys).sum(), inputs, create_graph=create_graph)

    # the first-order gradient is itself checked first
    def solve():
        return tsde.sdeint(sde, y0, ts, bm=_bm(B, bm_m, torch.float64, method), method=method, dt=DT,
                           options=NO_FUSE)
    out, jacs = gr.central_jacobian(lambda: solve().reshape(-1), inputs)
    bad = gr.check_vjp(out, jacs, w, [g.detach() for g in first()], 'first order')
    u = [_weights(x.shape, 30 + i) for i, x in enumerate(inputs)]
    g1 = first(create_graph=True)
    hu = torch.autograd.grad(sum((g * v).sum() for g, v in zip(g1, u)), inputs)
    mag = max(float(x.detach().abs().max()) for x in inputs)
    s = gr.H_REL * max(mag, 1.0)
    with gr.shifted(inputs, [s * v for v in u]):
        plus = [g.detach() for g in first()]
    with gr.shifted(inputs, [-s * v for v in u]):
        minus = [g.detach() for g in first()]
    wabs = w.abs().reshape(-1)
    for i, (a, p, q, g, J) in enumerate(zip(hu, plus, minus, g1, jacs)):
        D = (p - q) / (2 * s)
        # the first-order gradient is a sum of |w|^T |J| in magnitude: its rounding, over 2s, bounds D's error
        scale = (wabs @ J.abs()).reshape(D.shape) + g.detach().abs()
        ok = gr.within(a, D, scale)
        if not bool(ok.all()):
            k = int((~ok).reshape(-1).nonzero()[0])
            bad.append(f'second order input {i} element {k}: autograd {a.reshape(-1)[k].item():.17g}, central '
                       f'difference {D.reshape(-1)[k].item():.17g}')
    assert not bad, '\n'.join(bad)


# ---- (f) sensitivity --------------------------------------------------------------------------------------------
def _scaled_table(entry, out_index, in_index):
    real = autograd_ops._table

    def table(name, sc, w, u):
        t = real(name, sc, w, u)
        if name == entry:
            kind, c = t[out_index][in_index]
            t[out_index][in_index] = (kind, c * (1 + 1e-5))
        return t
    return table


@pytest.mark.parametrize('entry,in_index,small,route', [
    ('tsde_step_euler', 2, ('euler', 'ito', 'general', 2, 3, TS_GRID, 'fused'),
     ('euler', 'dense', 97, 4, 16, GEN_CTA)),
    ('tsde_step_reversible_heun', 3, ('reversible_heun', 'stratonovich', 'diagonal', 3, 3, TS_GRID, 'fused'),
     ('reversible_heun', 3, 97)),
], ids=['general-euler-g', 'diagonal-reversible-heun-g0'])
def test_sensitivity_to_one_coefficient(monkeypatch, entry, in_index, small, route):
    """The g coefficient of one entry scaled by (1 + 1e-5): (a)'s full-Jacobian check and (b)'s per-row check fail."""
    solve, inputs = _setup(small)
    assert not full_check(solve, inputs, 'unmodified')
    assert not rowwise_check(route)[0]
    monkeypatch.setattr(autograd_ops, '_table', _scaled_table(entry, 0, in_index))
    assert full_check(solve, inputs, 'scaled'), '(a) missed a 1e-5 relative error in one coefficient'
    assert rowwise_check(route)[0], '(b) missed a 1e-5 relative error in one coefficient'
