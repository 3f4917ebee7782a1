"""Self-checks of tests/adaptive_ref.py, the restatement of the adaptive loop that tests/test_gpu_adaptive.py compares
`sdeint(adaptive=True)` with.  No GPU needed.

  * On every golden adaptive fixture (the reference's own increments, replayed), free mode makes the reference's
    queries in the reference's order, as many proposals as the reference made, and gives its ys.  The reference forms
    its error estimate with torch's mean, the restatement with numpy's sum: their step sizes differ in the last bits,
    and so may a proposal's next_t (free mode `snap`s it, adaptive_ref's docstring); every other bit of the queries,
    and every decision, must be the reference's.
  * Driven mode, fed free mode's own history, reproduces free mode bit for bit: states, errors, decisions.
  * Where build() has staged the reference under oracle/_ref, free mode's history equals the live reference's on
    random configurations: the same queries and the same error estimate per proposal (float64 solves, where the
    reference's state-dtype error estimate is the restatement's float64 one).
"""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from oracle import solvers
from . import adaptive_ref, helpers, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.path.join(ROOT, 'oracle', '_ref', 'site')
ADAPTIVE_CASES = helpers.golden_files('adaptive_')


def _golden(path):
    case = helpers.load(path)
    solver = solvers.make(str(case['method']), problems.NumpySDE(helpers.build_problem(case)),
                          helpers.replay_numpy(case), float(case['dt']))
    args = (case['y0'], case['ts'], float(case['rtol']), float(case['atol']), float(case['dt_min']))
    return case, solver, args


def test_golden_fixtures_present():
    assert len(ADAPTIVE_CASES) >= 6


@pytest.mark.parametrize('path', ADAPTIVE_CASES, ids=helpers.case_id)
def test_free_mode_is_the_reference_on_its_increments(path):
    case, solver, args = _golden(path)
    queries = [(float(a), float(b)) for a, b in zip(case['ta'], case['tb'])]
    res = adaptive_ref.integrate_adaptive(solver, *args, snap=adaptive_ref.times_of(queries))
    assert 3 * len(res.history) == int(case['n_queries'])
    assert adaptive_ref.queries_of(res.history) == queries
    np.testing.assert_allclose(res.ys, case['ys'], rtol=1e-12, atol=1e-14)
    assert res.history[-1].accepted


@pytest.mark.parametrize('path', ADAPTIVE_CASES, ids=helpers.case_id)
def test_driven_mode_reproduces_free_mode(path):
    _, solver, args = _golden(path)
    free = adaptive_ref.integrate_adaptive(solver, *args, keep_states=True)
    driven = adaptive_ref.integrate_adaptive(solver, *args, driven=free.history, keep_states=True)
    assert driven.history == free.history
    assert np.array_equal(driven.ys, free.ys)
    for (a, b), (c, d) in zip(driven.states, free.states):
        assert np.array_equal(a, c) and np.array_equal(b, d)
    for a, b in zip(driven.extra, free.extra):
        assert np.array_equal(a, b)


def test_driven_mode_refuses_a_history_that_does_not_fit():
    _, solver, args = _golden(ADAPTIVE_CASES[0])
    free = adaptive_ref.integrate_adaptive(solver, *args)
    h = list(free.history)
    k = next(i for i, p in enumerate(h) if p.accepted)
    h[k] = h[k]._replace(accepted=False)   # a rejection where the solve moved on: the next proposal starts elsewhere
    with pytest.raises(AssertionError):
        adaptive_ref.integrate_adaptive(solver, *args, driven=h)
    with pytest.raises(AssertionError):
        adaptive_ref.integrate_adaptive(solver, *args, driven=free.history[:-1])


def test_snapping_adopts_only_last_bit_differences():
    """Free mode snaps to a given history's next_t only within SNAP_REL: a history whose times are off by 1e-9 is not
    adopted, so its queries stay the restatement's own."""
    _, solver, args = _golden(ADAPTIVE_CASES[0])
    free = adaptive_ref.integrate_adaptive(solver, *args)
    near = [p._replace(next_t=float(np.nextafter(p.next_t, 0.0))) for p in free.history]
    snapped = adaptive_ref.integrate_adaptive(solver, *args, snap=near)
    assert snapped.snapped > 0
    off = [p._replace(next_t=p.next_t * (1 - 1e-9)) for p in free.history]
    res = adaptive_ref.integrate_adaptive(solver, *args, snap=off)
    assert res.snapped == 0 and res.history == free.history


def test_error_estimate_is_float64_and_clamped():
    y = np.array([[1.0, 2.0]], np.float32)
    z = y + np.float32(1e-3)
    x = (y.astype(np.float64) - z.astype(np.float64)) / (1e-3 * np.maximum(np.abs(y), np.abs(z)).astype(np.float64)
                                                       + 1e-3)
    assert adaptive_ref.error_estimate(y, z, 1e-3, 1e-3) == float(np.sqrt((x ** 2).mean()))
    assert adaptive_ref.error_estimate(y, y, 1e-3, 1e-3) == adaptive_ref.EPS


# ---- against the live reference, where build() staged it -------------------------------------------------------------
MENU = [
    ('euler', None, 'ito', ('gbm', 'scalar', 'additive', 'general')),
    ('milstein', None, 'ito', ('gbm', 'scalar', 'additive')),
    ('milstein', {'grad_free': True}, 'ito', ('gbm', 'scalar')),
    ('srk', None, 'ito', ('gbm', 'scalar', 'additive')),
    ('milstein', None, 'stratonovich', ('gbm', 'scalar')),
    ('heun', None, 'stratonovich', ('gbm', 'scalar', 'additive', 'general')),
    ('midpoint', None, 'stratonovich', ('gbm', 'scalar', 'additive', 'general')),
    ('euler_heun', None, 'stratonovich', ('gbm', 'scalar', 'additive', 'general')),
    ('reversible_heun', None, 'stratonovich', ('gbm', 'scalar', 'additive', 'general')),
]


def _reference():
    if not os.path.isdir(os.path.join(REFERENCE, 'torchsde')):
        pytest.skip("reference not staged under oracle/_ref: the golden fixtures stand in")
    for p in (REFERENCE, os.path.join(ROOT, 'oracle', 'refshim')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torchsde
    return torchsde


@pytest.mark.parametrize('seed', range(24))
def test_free_mode_history_equals_the_live_reference(seed, monkeypatch):
    torchsde = _reference()
    from torchsde._core import adaptive_stepping
    rng = np.random.RandomState(7000 + seed)
    method, opts, sde_type, kinds = MENU[seed % len(MENU)]
    kind = kinds[rng.randint(len(kinds))]
    B, d = int(rng.randint(1, 5)), int(rng.randint(1, 6))
    m = 1 if kind == 'scalar' else (d if kind == 'gbm' else int(rng.randint(1, 5)))
    ts = np.concatenate([[0.0], np.cumsum(rng.uniform(0.1, 0.5, size=int(rng.randint(1, 4))))])
    dt0 = float(rng.choice([0.3, 0.2, 0.125]))
    rtol, atol = float(rng.choice([1e-2, 1e-3, 3e-4])), float(rng.choice([1e-2, 1e-3, 3e-4]))
    dt_min = float(rng.choice([1e-4, 2e-2]))
    sde = problems.make(kind, d, m, sde_type, dtype=torch.float64, seed=seed)
    y0 = 0.1 + 0.5 * torch.rand(B, d, dtype=torch.float64, generator=torch.Generator().manual_seed(seed))
    tst = torch.tensor(ts, dtype=torch.float64)
    levy = 'space-time' if method == 'srk' else 'none'
    bm = torchsde.BrownianInterval(0.0, float(ts[-1]), size=(B, m), dtype=torch.float64, entropy=seed,
                                   levy_area_approximation=levy)
    log, errors = [], []
    real = adaptive_stepping.compute_error

    def compute_error(*a, **kw):
        e = real(*a, **kw)
        errors.append(float(e))
        return e
    monkeypatch.setattr(adaptive_stepping, 'compute_error', compute_error)

    class Recorder:
        shape, levy_area_approximation = bm.shape, bm.levy_area_approximation

        def __call__(self, ta, tb=None, return_U=False, return_A=False):
            W, U = (bm(ta, tb), None) if levy == 'none' else bm(ta, tb, return_U=True)
            log.append((float(ta), float(tb), W.numpy().copy(), None if U is None else U.numpy().copy()))
            return (W, U) if return_U else W

    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = torchsde.sdeint(sde, y0, tst, bm=Recorder(), method=method, dt=dt0, adaptive=True, rtol=rtol,
                              atol=atol, dt_min=dt_min, options=opts).numpy()
    replay = problems.ReplayBM(np.array([r[0] for r in log]), np.array([r[1] for r in log]),
                               np.stack([r[2] for r in log]),
                               None if log[0][3] is None else np.stack([r[3] for r in log]), levy=levy)
    solver = solvers.make(method, problems.NumpySDE(sde), replay, dt0, opts or {})
    queries = [(a, b) for a, b, _, _ in log]
    res = adaptive_ref.integrate_adaptive(solver, y0.numpy(), ts, rtol, atol, dt_min,
                                          snap=adaptive_ref.times_of(queries))
    what = f"{method} {opts} {sde_type} {kind} B={B} d={d} m={m} ts={ts} dt={dt0} rtol={rtol} atol={atol}"
    assert adaptive_ref.queries_of(res.history) == queries, what
    np.testing.assert_allclose([h.error for h in res.history], errors, rtol=1e-9, err_msg=what)
    np.testing.assert_allclose(res.ys, ref, rtol=1e-11, atol=1e-13, err_msg=what)
