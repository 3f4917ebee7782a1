"""The float64 restatement of the generic adjoint (tests/adjoint_ref.py) against the reference, on the CPU.

* It reproduces every generic-adjoint golden (`genadj_*`) and the logqp Milstein-adjoint golden, ys and gradients.
* Where the reference is staged under oracle/_ref, `PAIRS` is exactly the set of generic (method, adjoint_method,
  noise type) combinations the live reference runs, and randomised cases of every pair (grad-free Milstein,
  logqp=True, adjoint_params subsets and adjoint_adaptive=True included) match the live reference on the increments
  it consumed.
* Each deliberate error of `adjoint_ref.MUTATIONS` moves most of the elements it changes beyond the tolerance the GPU
  comparison (tests/test_gpu_generic_adjoint.py) applies, so that comparison would reject it.
"""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from . import adjoint_ref, helpers, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.path.join(ROOT, 'oracle', '_ref', 'site')
GOLDEN_CASES = helpers.golden_files('genadj_') + helpers.golden_files('logqp_diag_ito_milstein_adjoint')


def _golden_run(case, mutate=()):
    """Restated forward and backward of a golden case: (ys, [grad_y0, grad_param...], names)."""
    bm = helpers.replay_numpy(case)
    dt, ts, method = float(case['dt']), case['ts'], str(case['method'])
    if 'logqp' in case:
        base = problems.LatentPrior(int(case['d']), int(case['m']), str(case['noise']), str(case['sde_type']),
                                    seed=int(case['seed']), dtype=torch.float64)
        module = adjoint_ref.Logqp(base)
        y0 = np.concatenate([case['y0'], np.zeros((case['y0'].shape[0], 1))], axis=1)
        adjoint_method = adjoint_ref.default_adjoint_method(base.sde_type, base.noise_type)
    else:
        base = module = helpers.build_problem(case, dtype=torch.float64)
        y0 = case['y0']
        adjoint_method = str(case['adjoint_method']) or adjoint_ref.default_adjoint_method(base.sde_type,
                                                                                          base.noise_type)
    ys = adjoint_ref.forward(module, y0, ts, method, dt, bm)
    if 'logqp' in case:
        grad_ys = adjoint_ref.logqp_grad_ys(ys, case['wy'], case['wl'])
    else:
        grad_ys = case['weights']
    names = [n for n, _ in base.named_parameters()]
    adj_y0, adj_params, _ = adjoint_ref.backward(module, list(base.parameters()), ys, ts, grad_ys, adjoint_method, dt,
                                                 bm, mutate=mutate)
    if 'logqp' in case:
        ys, adj_y0 = ys[..., :-1], adj_y0[:, :-1]
    return ys, [adj_y0] + adj_params, names


def _golden_grads(case, names):
    return [case['grad_y0']] + [case['grad.' + n] for n in names]


@pytest.mark.parametrize('path', GOLDEN_CASES, ids=helpers.case_id)
def test_restatement_reproduces_the_reference_goldens(path):
    """Same increments as the reference consumed: ys and every gradient to 1e-12 of the reference's value."""
    case = helpers.load(path)
    ys, grads, names = _golden_run(case)
    np.testing.assert_allclose(ys, case['ys'], rtol=1e-12, atol=1e-15)
    for name, got, ref in zip(['y0'] + names, grads, _golden_grads(case, names)):
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-14 * adjoint_ref.scale(ref), err_msg=name)


# ---- mutations ---------------------------------------------------------------------------------------------------------
# (mutation, golden case it changes): each case is one where the mutated term carries weight
MUTATION_CASES = [('neighbour_dw', 'genadj_gbm_ito_euler'), ('neighbour_dw', 'genadj_general_strat_midpoint'),
                  ('milstein_v', 'genadj_gbm_ito_srk'), ('milstein_v', 'logqp_diag_ito_milstein_adjoint'),
                  ('no_ito', 'genadj_gbm_ito_euler'), ('no_ito', 'genadj_general_ito_euler'),
                  ('no_ito', 'genadj_scalar_ito_milstein'),
                  ('diag_columns', 'genadj_general_ito_euler'),
                  ('late_grad', 'genadj_gbm_strat_heun'), ('late_grad', 'genadj_additive_ito_srk'),
                  ('drop_params', 'genadj_gbm_strat_heun'), ('drop_params', 'genadj_scalar_strat_midpoint_eh')]


def rejected_share(got, ref):
    """Of the elements a mutation changes (beyond 1e-13 of the scale), the share the float64 GPU comparison
    (|got - ref| <= RTOL64 * scale) rejects."""
    s = adjoint_ref.scale(ref)
    changed = adjoint_ref.excess(got, ref, 1e-13 * s) > 1
    rejected = adjoint_ref.excess(got, ref, adjoint_ref.RTOL64 * s) > 1
    return int(changed.sum()), int((rejected & changed).sum())


def test_every_mutation_has_a_case():
    assert {m for m, _ in MUTATION_CASES} == set(adjoint_ref.MUTATIONS)


@pytest.mark.parametrize('mutation,name', MUTATION_CASES, ids=[f'{m}-{n}' for m, n in MUTATION_CASES])
def test_mutation_is_rejected(mutation, name):
    """The mutated restatement against the reference's gradients: on most of the elements the mutation changes, the
    difference exceeds the float64 GPU comparison's tolerance."""
    case = helpers.load(os.path.join(helpers.GOLDEN, name + '.npz'))
    _, grads, names = _golden_run(case, mutate=(mutation,))
    changed = rejected = 0
    for got, ref in zip(grads, _golden_grads(case, names)):
        c, r = rejected_share(got, ref)
        changed, rejected = changed + c, rejected + r
    assert changed > 0, f'{mutation} changes nothing in {name}'
    assert rejected > changed / 2, f'{mutation} in {name}: {rejected} of {changed} changed elements rejected'


# ---- the live reference ------------------------------------------------------------------------------------------------
def _reference():
    if not os.path.isdir(os.path.join(REFERENCE, 'torchsde')):
        pytest.skip("reference not staged under oracle/_ref: the golden vectors stand in")
    for p in (REFERENCE, os.path.join(ROOT, 'oracle', 'refshim')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torchsde
    return torchsde


class _Recorder:
    def __init__(self, bm):
        self.bm, self.shape, self.levy_area_approximation = bm, bm.shape, bm.levy_area_approximation
        self.log = []

    def __call__(self, ta, tb=None, return_U=False, return_A=False):
        if self.levy_area_approximation == 'none':
            W, U = self.bm(ta, tb), None
        else:
            W, U = self.bm(ta, tb, return_U=True)
        self.log.append((float(ta), float(tb), W.numpy().copy(), None if U is None else U.numpy().copy()))
        return (W, U) if return_U else W

    def replay(self):
        log = self.log
        return problems.ReplayBM([r[0] for r in log], [r[1] for r in log], [r[2] for r in log],
                                 None if log[0][3] is None else [r[3] for r in log], levy=self.levy_area_approximation)


def test_pairs_are_what_the_live_reference_accepts():
    """Every (sde_type, method, adjoint_method, noise kind) the reference runs forward and backward, and no other, is in
    adjoint_ref.PAIRS (the reversible pair and the refusals aside)."""
    torchsde = _reference()
    methods = [('euler', None), ('milstein', None), ('milstein', {'grad_free': True}), ('srk', None),
               ('midpoint', None), ('heun', None), ('euler_heun', None), ('reversible_heun', None)]
    adjoints = ['euler', 'milstein', 'srk', 'midpoint', 'heun', 'euler_heun', 'log_ode']
    accepted = set()
    for st in ('ito', 'stratonovich'):
        for kind in ('gbm', 'scalar', 'additive', 'general'):
            d, m = 3, {'gbm': 3, 'scalar': 1}.get(kind, 2)
            sde = problems.make(kind, d, m, st, dtype=torch.float64)
            for method, opts in methods:
                for adj in adjoints:
                    y0 = torch.ones(2, d, dtype=torch.float64, requires_grad=True)
                    try:
                        with warnings.catch_warnings():
                            warnings.simplefilter('ignore')
                            torchsde.sdeint_adjoint(sde, y0, [0.0, 0.1], method=method, adjoint_method=adj, dt=0.05,
                                                    options=None if opts is None else dict(opts)).sum().backward()
                    except (ValueError, NotImplementedError, RuntimeError):
                        continue
                    accepted.add((st, method, bool(opts), adj, kind))
    assert accepted == {(st, mt, bool(o), adj, kind) for st, mt, o, adj, kind in adjoint_ref.PAIRS}


def _live_case(torchsde, pair, seed):
    """One randomised case of `pair`: (reference ys, reference grads, restated ys, restated grads, label)."""
    st, method, opts, adj, kind = pair
    rng = np.random.RandomState(3000 + seed)
    B, d = int(rng.randint(3, 6)), int(rng.randint(1, 6))
    logqp = kind in ('gbm', 'general') and rng.rand() < 0.3
    if logqp:
        m = d if kind == 'gbm' else int(rng.randint(1, 4))
        base = problems.LatentPrior(d, m, 'diagonal' if kind == 'gbm' else 'general', st, seed=seed)
        bm_m = d + 1 if kind == 'gbm' else m
    else:
        m = 1 if kind == 'scalar' else (d if kind == 'gbm' else int(rng.randint(1, 5)))
        base = problems.make(kind, d, m, st, seed=seed)
        bm_m = m
    params = [p for _, p in base.named_parameters()]
    subset = rng.rand() < 0.3 and len(params) > 1
    adj_params = params[:1] if subset else params
    adaptive = rng.rand() < 0.25
    n_out = int(rng.randint(2, 5))
    ts = np.concatenate([[0.0], np.cumsum(rng.uniform(0.05, 0.2, size=n_out - 1))])
    if rng.randint(2):
        ts = np.round(ts * 32) / 32
        ts = np.concatenate([[0.0], np.maximum.accumulate(ts[1:] + np.arange(1, n_out) / 1024)])
    dt = float(rng.choice([2.0 ** -4, 2.0 ** -5, 0.05, 0.03]))
    torch.manual_seed(seed)
    y0 = (0.1 + 0.5 * torch.rand(B, d, dtype=torch.float64)).requires_grad_()
    tst = torch.tensor(ts, dtype=torch.float64)
    levy = 'space-time' if method == 'srk' else 'none'
    bm = torchsde.BrownianInterval(0.0, float(ts[-1]), size=(B, bm_m), dtype=torch.float64, entropy=seed,
                                   levy_area_approximation=levy)
    rec = _Recorder(bm)
    kw = dict(adjoint_adaptive=True, adjoint_rtol=1e-3, adjoint_atol=1e-3, dt_min=1e-3) if adaptive else {}
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        out = torchsde.sdeint_adjoint(base, y0, tst, bm=rec, method=method, adjoint_method=adj, dt=dt, logqp=logqp,
                                      options=None if opts is None else dict(opts), adjoint_params=adj_params, **kw)
    wy_shape = (n_out, B, d)
    wy = np.linspace(0.5, 1.5, int(np.prod(wy_shape))).reshape(wy_shape)
    if logqp:
        ys_ref, lq = out
        wl = np.linspace(1.0, 2.0, lq.numel()).reshape(tuple(lq.shape))
        loss = (ys_ref * torch.from_numpy(wy)).sum() + (lq * torch.from_numpy(wl)).sum()
    else:
        ys_ref = out
        loss = (ys_ref * torch.from_numpy(wy)).sum()
    ref_grads = torch.autograd.grad(loss, [y0] + adj_params)
    replay = rec.replay()
    module = adjoint_ref.Logqp(base) if logqp else base
    y0n = y0.detach().numpy()
    if logqp:
        y0n = np.concatenate([y0n, np.zeros((B, 1))], axis=1)
    ys = adjoint_ref.forward(module, y0n, ts, method, dt, replay, opts)
    grad_ys = adjoint_ref.logqp_grad_ys(ys, wy, wl) if logqp else wy
    adaptive_kw = dict(rtol=1e-3, atol=1e-3, dt_min=1e-3) if adaptive else None
    adj_y0, adj_p, _ = adjoint_ref.backward(module, adj_params, ys, ts, grad_ys, adj, dt, replay, adaptive=adaptive_kw)
    if logqp:
        ys, adj_y0 = ys[..., :-1], adj_y0[:, :-1]
    label = f'{adjoint_ref.pair_id(pair)} seed={seed} B={B} d={d} m={m} logqp={logqp} subset={subset} ' \
            f'adaptive={adaptive} ts={ts} dt={dt}'
    return ys_ref.detach().numpy(), [g.numpy() for g in ref_grads], ys, [adj_y0] + adj_p, label


@pytest.mark.parametrize('pair', adjoint_ref.PAIRS, ids=adjoint_ref.pair_id)
def test_restatement_equals_live_reference(pair):
    torchsde = _reference()
    for seed in range(2):
        ref_ys, ref_grads, ys, grads, label = _live_case(torchsde, pair, adjoint_ref.PAIRS.index(pair) * 2 + seed)
        np.testing.assert_allclose(ys, ref_ys, rtol=1e-12, atol=1e-14, err_msg=label)
        for got, ref in zip(grads, ref_grads):
            np.testing.assert_allclose(got, ref, rtol=1e-11, atol=1e-13 * adjoint_ref.scale(ref), err_msg=label)
