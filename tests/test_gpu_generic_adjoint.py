"""sdeint_adjoint's generic adjoint on counter noise against the float64 restatement of the reference's algorithm.

Every adjoint method but the reversible pair integrates the adjoint SDE (torchsde_b200/_core/adjoint_sde.py) backwards
on the flat (1, N) augmented state, N = 2 B d + sum |params|.  On a grid-bound `BrownianInterval` the backward solve
binds the reversed grid (`GridBinding.reversed`) and materialises each step's (B, m) increment from the forward's
Philox cells, merging cells where a step spans several; the row-wise kernels then run at rows = 1, d = N, with the
products supplied (unit noise).  Here ys, y0.grad and every parameter gradient of such solves are compared with
tests/adjoint_ref.py, which restates the reference's adjoint in float64 on the CPU and is itself checked against the
reference (tests/test_host_adjoint_ref.py).  Its increments are the same Brownian motion's:
  * float64 on the grid: the oracle's Philox cells (helpers.oracle_grid_bm), which raise for any query off the grid;
  * float64 off the grid (output times off the step grid, adjoint_adaptive): the interval-tree oracle of
    test_gpu_brownian_paths.py, walking the interval's own tree, so only queries the solve made can be answered;
  * float32: the increments the float32 interval itself returns, widened (a float32 and a float64 interval with the
    same entropy draw different normals).

Bounds.
  * float64: |got - ref| <= RTOL64 scale, RTOL64 = 1e-9 and scale = max |ref| of the compared tensor.  The kernels
    follow the reference's operation order; what differs is the rounding of reductions (torch's autograd sums over
    rows, bmm) and of libm, a few ulp per step, so over these solves (<= 64 steps, a few tens of rounded operations per
    element and step) the difference stays below 1e-12 scale.  The bound leaves three orders of magnitude, as
    test_gpu_pointwise_fuzz.py does, and tests/test_host_adjoint_ref.py shows that each restated error of
    adjoint_ref.MUTATIONS exceeds it.
  * float32: |got - ref| <= e * n * K * u * scale, u = 2^-24.  n counts the forward and backward steps (each queries
    the Brownian motion once), K = 64 bounds the rounded float32 operations one step performs per element (the user's
    f and g and their vjps, the Ito correction's double vjp, the diffusion product, the tableau), and e bounds the
    growth of an error through the linearised steps of these problems (Lipschitz constants <= 2, horizons <= 0.5).
    The forward's rounding enters the backward through ys, and is counted in n.  A parameter gradient is in addition
    a float32 sum over the B rows at every step; its rounding errors, of either sign, add up like a random walk, so
    the sum's error stays within 4 sqrt(B) u of its scale (four standard deviations), and the bound of a parameter
    gradient is e n (K + 4 sqrt(B)) u scale.
The worst err/bound per (adjoint method, dtype) is printed at the end of the module (`-s`).

Routes: flat states with N % 4 != 0 (generic row-wise kernel) and N % 4 == 0 (fast kernel), B = 4099, and one Euler
adjoint whose flat state exceeds 2^26 elements, so a row's quad index passes 2^24.  A spy on `GridBinding.reversed` and
on `BrownianInterval.__call__` confirms that on-grid backward solves take the reversed binding and query nothing (so
run no bridge), and that off-grid and adaptive ones query exactly what the restatement queries.  A reversed binding
that serves each step its neighbour's cell must fail the comparison.
"""
import contextlib
import math
import warnings

import numpy as np
import pytest
import torch

from torchsde_b200._brownian import interval as iv

from . import adjoint_ref, helpers, problems
from .test_gpu_brownian_paths import _TreeOracle

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K_OPS = 64
U32 = 2.0 ** -24
WORST = {}


def f32_bound(n_steps, rows=1):
    """e n (K + 4 sqrt(rows)) u: the float32 bound of the module docstring; `rows` summands per parameter gradient."""
    return math.e * n_steps * (K_OPS + 4 * math.sqrt(rows)) * U32


def _tsde():
    import torchsde_b200
    return torchsde_b200


@contextlib.contextmanager
def _spy():
    """Counts reversed grid bindings and records the Brownian queries made inside the block."""
    seen = {'reversed': 0, 'queries': []}
    rev, call = iv.GridBinding.reversed, iv.BrownianInterval.__call__

    def reversed_(self):
        seen['reversed'] += 1
        return rev(self)

    def call_(self, ta, tb=None, return_U=False, return_A=False):
        seen['queries'].append((float(ta), float(tb)))
        return call(self, ta, tb, return_U=return_U, return_A=return_A)

    iv.GridBinding.reversed, iv.BrownianInterval.__call__ = reversed_, call_
    try:
        yield seen
    finally:
        iv.GridBinding.reversed, iv.BrownianInterval.__call__ = rev, call


def _increments(bm, dtype, B, m, source, snap=()):
    """The restatement's bm(ta, tb[, return_U]) in forward time, and the list of queries it answered.

    `snap`: queries the GPU solve made.  An adaptive solve's step sizes are continuous functions of its error estimates,
    which the GPU and the restatement round differently, so their query times may differ in the last bits: a query
    within 1e-9 of one the GPU made is answered, and recorded, as that one."""
    asked = []
    snap = list(snap)

    def snapped(ta, tb):
        ta, tb = float(ta), float(tb)
        near = min(snap, key=lambda q: abs(q[0] - ta) + abs(q[1] - tb), default=None)
        if near is not None and abs(near[0] - ta) + abs(near[1] - tb) <= 1e-9:
            return near
        return ta, tb

    if dtype == torch.float32:
        def raw(ta, tb, want_u):
            out = bm(float(ta), float(tb), return_U=want_u)
            return tuple(x.double().cpu().numpy() for x in out) if want_u else out.double().cpu().numpy()
    elif source == 'grid':
        grid = helpers.oracle_grid_bm(bm, np.arange(B), m, np.float64, bm._have_H)

        def raw(ta, tb, want_u):
            return grid(ta, tb, return_U=want_u)
    else:
        tree = _TreeOracle(bm, np.float64)

        def raw(ta, tb, want_u):
            W, U, _ = tree.query(float(ta), float(tb))
            return (W.v, U.v) if want_u else W.v

    def query(ta, tb, return_U=False):
        ta, tb = snapped(ta, tb)
        asked.append((ta, tb))
        return raw(ta, tb, return_U)
    return query, asked


def _check(what, got, ref, bound, key, bad):
    """Compares got with ref within bound * scale(ref); records the worst err/bound under `key` (None: nowhere)."""
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else got
    if got.shape != ref.shape:
        bad.append(f'{what}: shape {got.shape} != {ref.shape}')
        return
    r = float(np.max(adjoint_ref.excess(got, ref, bound * adjoint_ref.scale(ref))))
    if key is not None:
        WORST[key] = max(WORST.get(key, 0.0), r)
    if not r <= 1.0:
        bad.append(f'{what}: worst err/bound {r:.3g}')


def solve_and_compare(pair, dtype=torch.float64, B=3, d=None, m=None, ts=(0.0, 0.125, 0.25, 0.375), dt=2.0 ** -5,
                      bm_dt=None, logqp=False, subset=False, adaptive=False, graph=False, source='grid', seed=0,
                      expect_binding=True, expect_pass=True):
    """One sdeint_adjoint solve and backward on the GPU, checked against the restatement on the same Brownian motion."""
    tsde = _tsde()
    st, method, opts, adj, kind = pair
    d = d or {'gbm': 4, 'scalar': 3, 'additive': 3, 'general': 4}[kind]
    m = m or {'gbm': d, 'scalar': 1, 'additive': 2, 'general': 3}[kind]
    if logqp:
        noise = 'diagonal' if kind == 'gbm' else 'general'
        base = problems.LatentPrior(d, m, noise, st, seed=seed, dtype=dtype)
        bm_m = d + 1 if noise == 'diagonal' else m
    else:
        base = problems.make(kind, d, m, st, dtype=dtype, seed=seed)
        bm_m = m
    cpu = base.double()
    dev = (problems.LatentPrior(d, m, noise, st, seed=seed, dtype=dtype) if logqp
           else problems.make(kind, d, m, st, dtype=dtype, seed=seed)).to(DEV)
    names = [n for n, _ in dev.named_parameters()]
    pick = names[-1:] if subset else names
    gen = torch.Generator().manual_seed(100 + seed)
    y0 = (0.1 + 0.5 * torch.rand(B, d, generator=gen, dtype=torch.float64)).to(dtype)
    ts_np = np.asarray(ts, dtype={torch.float32: np.float32, torch.float64: np.float64}[dtype])
    tst = torch.from_numpy(ts_np).to(DEV)
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(float(ts_np[0]), float(ts_np[-1]), size=(B, bm_m), dtype=dtype, device=DEV,
                               entropy=7 + seed, levy_area_approximation=levy, dt=bm_dt)
    y0_dev = y0.to(DEV).requires_grad_()
    ad = dict(adjoint_adaptive=True, adjoint_rtol=1e-3, adjoint_atol=1e-3, dt_min=1e-3) if adaptive else {}
    options = dict(opts or {})
    if graph:
        options['cuda_graph'] = True
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        out = tsde.sdeint_adjoint(dev, y0_dev, tst, bm=bm, method=method, adjoint_method=adj, dt=dt, logqp=logqp,
                                  options=options, adjoint_params=[dict(dev.named_parameters())[n] for n in pick],
                                  **ad)
    T = len(ts)
    wy = np.linspace(0.5, 1.5, T * B * d).reshape(T, B, d)
    ys = out[0] if logqp else out
    loss = (ys * torch.from_numpy(wy).to(DEV, dtype)).sum()
    if logqp:
        wl = np.linspace(1.0, 2.0, (T - 1) * B).reshape(T - 1, B)
        loss = loss + (out[1] * torch.from_numpy(wl).to(DEV, dtype)).sum()
    with _spy() as seen:
        loss.backward()
    torch.cuda.synchronize()

    query, asked = _increments(bm, dtype, B, bm_m, source, seen['queries'])
    module = adjoint_ref.Logqp(cpu) if logqp else cpu
    y0_ref = y0.double().numpy()
    if logqp:
        y0_ref = np.concatenate([y0_ref, np.zeros((B, 1))], axis=1)
    ys_ref = adjoint_ref.forward(module, y0_ref, ts_np, method, dt, query, opts)
    n_fwd = len(asked)
    grad_ys = adjoint_ref.logqp_grad_ys(ys_ref, wy, wl) if logqp else wy
    params = [dict(cpu.named_parameters())[n] for n in pick]
    adaptive_kw = dict(rtol=1e-3, atol=1e-3, dt_min=1e-3) if adaptive else None
    adj_y0, adj_p, _ = adjoint_ref.backward(module, params, ys_ref, ts_np, grad_ys, adj, dt, query, adaptive=adaptive_kw)
    if logqp:
        ys_ref, adj_y0 = ys_ref[..., :-1], adj_y0[:, :-1]

    bad = []
    label = f'{adjoint_ref.pair_id(pair)} {dtype} B={B} d={d} m={m} logqp={logqp} subset={subset} ' \
            f'adaptive={adaptive} graph={graph} bm_dt={bm_dt} ts={list(ts)}'
    bound = adjoint_ref.RTOL64 if dtype == torch.float64 else f32_bound(len(asked))
    key = (adj, str(dtype).replace('torch.', '')) if expect_pass else None
    _check('ys', ys, ys_ref, bound, key, bad)
    _check('y0.grad', y0_dev.grad, adj_y0, bound, key, bad)
    p_bound = bound if dtype == torch.float64 else f32_bound(len(asked), B)
    for n, ref in zip(pick, adj_p):
        _check(f'{n}.grad', dict(dev.named_parameters())[n].grad, ref, p_bound, key, bad)
    for n, p in dev.named_parameters():
        if n not in pick and p.grad is not None:
            bad.append(f'{n}: a gradient outside adjoint_params')
    back_queries = asked[n_fwd:]
    if expect_binding:
        if seen['reversed'] < 1 or seen['queries']:
            bad.append(f"backward: {seen['reversed']} reversed bindings, {len(seen['queries'])} queries")
    elif dtype == torch.float64 and sorted(seen['queries']) != sorted(back_queries):
        bad.append(f"backward queries {len(seen['queries'])} differ from the restatement's {len(back_queries)}")
    if expect_pass:
        assert not bad, label + ': ' + '; '.join(bad)
    return bad


# ---- every accepted pair ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pair', adjoint_ref.PAIRS, ids=adjoint_ref.pair_id)
def test_every_pair_float64(pair):
    """B = 3 or 4 alternately, so both flat-state routes (N % 4 == 0 and != 0) occur across the pairs."""
    i = adjoint_ref.PAIRS.index(pair)
    solve_and_compare(pair, B=3 + i % 2, seed=i)


F32_PAIRS = [p for p in adjoint_ref.PAIRS if p[2] is None and (
    (p[0] == 'ito' and p[1] == 'euler') or (p[0] == 'stratonovich' and p[1] == 'midpoint') or
    (p[1] == 'milstein' and p[3] == 'milstein'))]


@pytest.mark.parametrize('pair', F32_PAIRS, ids=adjoint_ref.pair_id)
def test_float32_against_the_float64_restatement(pair):
    i = adjoint_ref.PAIRS.index(pair)
    solve_and_compare(pair, dtype=torch.float32, B=5, seed=i)


# ---- routes of the flat backward launches ----------------------------------------------------------------------------
@pytest.mark.parametrize('B', [3, 4], ids=['N%4==0', 'N%4!=0'])
@pytest.mark.parametrize('adj', ['euler', 'milstein'])
def test_flat_state_routes(B, adj):
    """gbm with d = 3: N = 6 B + 6 is 24 at B = 3 (the fast kernel) and 30 at B = 4 (the generic row-wise kernel)."""
    solve_and_compare(('ito', 'euler', None, adj, 'gbm'), B=B, d=3, seed=40 + B)


@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'milstein', 'gbm'), ('stratonovich', 'heun', None, 'midpoint',
                                                                               'general')], ids=adjoint_ref.pair_id)
def test_4099_trajectories(pair):
    solve_and_compare(pair, B=4099, ts=(0.0, 0.125, 0.25), seed=50)


def test_flat_state_past_2_26_elements():
    """Euler adjoint of a float32 GBM with B d = 2^25 + 256: the flat state has N = 2 B d + 8 > 2^26 elements, so a row's
    quad index passes 2^24.  Rows are independent in the adjoint of a diagonal SDE and the parameter adjoint is their
    sum, so the restatement runs in row blocks; y0.grad is compared on every row and the parameter gradients in full."""
    tsde = _tsde()
    B, d, dt = 2 ** 23 + 64, 4, 2.0 ** -5
    assert 2 * B * d + 2 * d > 2 ** 26
    ts_np = np.array([0.0, 2.0 ** -4], dtype=np.float32)
    dev = problems.make('gbm', d, d, 'ito', dtype=torch.float32, seed=3).to(DEV)
    cpu = problems.make('gbm', d, d, 'ito', dtype=torch.float32, seed=3).double()
    y0 = torch.full((B, d), 0.3, device=DEV) + 0.2 * torch.rand(B, d, device=DEV, generator=torch.Generator(
        device=DEV).manual_seed(1))
    y0.requires_grad_()
    bm = tsde.BrownianInterval(0.0, float(ts_np[-1]), size=(B, d), dtype=torch.float32, device=DEV, entropy=5)
    ys = tsde.sdeint_adjoint(dev, y0, torch.from_numpy(ts_np).to(DEV), bm=bm, method='euler', adjoint_method='euler',
                             dt=dt)
    with _spy() as seen:
        ys.sum().backward()
    torch.cuda.synchronize()
    assert seen['reversed'] >= 1 and not seen['queries'], seen['reversed']
    grads = [p.grad.double().cpu().numpy() for p in dev.parameters()]
    worst, bad = 0.0, []
    refs_p = [np.zeros(p.shape) for p in cpu.parameters()]
    block = 2 ** 21
    y0_all = y0.detach()
    ref_blocks = []
    n_steps = 0
    for r0 in range(0, B, block):
        r1 = min(B, r0 + block)
        asked = []

        def query(ta, tb, return_U=False, _r=(r0, r1), _asked=asked):
            _asked.append(ta)
            return bm(float(ta), float(tb))[_r[0]:_r[1]].double().cpu().numpy()
        yb = y0_all[r0:r1].double().cpu().numpy()
        ys_ref = adjoint_ref.forward(cpu, yb, ts_np, 'euler', dt, query)
        adj_y0, adj_p, _ = adjoint_ref.backward(cpu, list(cpu.parameters()), ys_ref, ts_np, np.ones_like(ys_ref),
                                                'euler', dt, query)
        n_steps = len(asked)
        for acc, a in zip(refs_p, adj_p):
            acc += a
        ref_blocks.append((r0, r1, ys_ref, adj_y0))
    bound = f32_bound(n_steps)
    for r0, r1, ys_ref, adj_y0 in ref_blocks:
        for what, got, ref in (('ys', ys[:, r0:r1], ys_ref), ('y0.grad', y0.grad[r0:r1], adj_y0)):
            got = got.detach().double().cpu().numpy()
            r = float(np.max(adjoint_ref.excess(got, ref, bound * adjoint_ref.scale(ref))))
            worst = max(worst, r)
            if r > 1:
                bad.append(f'{what} rows {r0}:{r1}: err/bound {r:.3g}')
    for (n, _), got, ref in zip(cpu.named_parameters(), grads, refs_p):
        r = float(np.max(adjoint_ref.excess(got, ref, f32_bound(n_steps, B) * adjoint_ref.scale(ref))))
        worst = max(worst, r)
        if r > 1:
            bad.append(f'{n}.grad: err/bound {r:.3g}')
    key = ('euler 2^26', 'float32')
    WORST[key] = max(WORST.get(key, 0.0), worst)
    assert not bad, '; '.join(bad)


# ---- increments --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'euler', 'general'), ('stratonovich', 'midpoint', None,
                                                                             'euler_heun', 'gbm'),
                                  ('ito', 'milstein', None, 'milstein', 'gbm')], ids=adjoint_ref.pair_id)
def test_steps_merge_finer_brownian_cells(pair):
    """Brownian dt a quarter of the solver's: each backward step materialises the merge of four cells."""
    solve_and_compare(pair, B=4, dt=2.0 ** -4, bm_dt=2.0 ** -6, seed=60)


@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'milstein', 'gbm'), ('stratonovich', 'heun', None, 'heun',
                                                                                'general'),
                                  ('ito', 'srk', None, 'euler', 'additive')], ids=adjoint_ref.pair_id)
def test_output_times_off_the_step_grid(pair):
    """ts off the step grid: the reversed steps are not the forward's, the binding fails and the backward queries the
    interval; every query must be one the tree oracle answers, and the restatement's."""
    solve_and_compare(pair, B=4, ts=(0.0, 0.1, 0.23, 0.3), dt=2.0 ** -5, source='tree', expect_binding=False, seed=70)


@pytest.mark.parametrize('pair', [('ito', 'srk', None, 'milstein', 'gbm'), ('ito', 'srk', None, 'euler', 'scalar')],
                         ids=adjoint_ref.pair_id)
def test_srk_forward_space_time_interval(pair):
    """SRK's interval carries H; the generic adjoint reads W only, through the reversed binding."""
    solve_and_compare(pair, B=5, seed=80)


# ---- options -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'euler', 'general'), ('ito', 'euler', None, 'milstein', 'gbm'),
                                  ('stratonovich', 'midpoint', None, 'midpoint', 'scalar'),
                                  ('stratonovich', 'heun', None, 'euler_heun', 'additive'),
                                  ('stratonovich', 'euler_heun', None, 'heun', 'gbm')], ids=adjoint_ref.pair_id)
def test_adjoint_adaptive(pair):
    """adjoint_adaptive=True: the restatement's accept / reject history asks the same queries the GPU solve asked."""
    solve_and_compare(pair, B=3, ts=(0.0, 0.25, 0.5), dt=0.125, adaptive=True, source='tree', expect_binding=False,
                      seed=90)


@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'milstein', 'gbm'), ('ito', 'euler', None, 'euler', 'general'),
                                  ('stratonovich', 'midpoint', None, 'midpoint', 'gbm'),
                                  ('stratonovich', 'heun', None, 'heun', 'general')], ids=adjoint_ref.pair_id)
def test_logqp(pair):
    solve_and_compare(pair, B=4, d=3, m=3 if pair[4] == 'gbm' else 2, logqp=True, seed=100)


@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'milstein', 'gbm'), ('ito', 'euler', None, 'euler', 'general'),
                                  ('stratonovich', 'midpoint', None, 'heun', 'additive')], ids=adjoint_ref.pair_id)
def test_adjoint_params_subset(pair):
    solve_and_compare(pair, B=4, subset=True, seed=110)


@pytest.mark.parametrize('pair', [('ito', 'euler', None, 'milstein', 'gbm'), ('stratonovich', 'midpoint', None,
                                                                                'midpoint', 'general')],
                         ids=adjoint_ref.pair_id)
def test_cuda_graph_forward(pair):
    solve_and_compare(pair, B=4, graph=True, seed=120)


# ---- sensitivity ---------------------------------------------------------------------------------------------------------
def test_neighbour_cell_in_the_reversed_binding_fails():
    """A reversed binding that serves each backward step its neighbour's cell must fail the comparison."""
    fill = iv.GridBinding.fill

    def neighbour_fill(self, nz, k, want_u, key_ptr, row_offset=0):
        if self.reverse:
            k = k + 1 if k + 1 < self.n_steps else k - 1
        return fill(self, nz, k, want_u, key_ptr, row_offset)

    iv.GridBinding.fill = neighbour_fill
    try:
        bad = solve_and_compare(('ito', 'euler', None, 'milstein', 'gbm'), B=4, seed=130, expect_pass=False)
    finally:
        iv.GridBinding.fill = fill
    assert any('grad' in b for b in bad), bad


def test_report_worst_err_over_bound():
    """Runs last: prints the worst err/bound per (adjoint method, dtype) over the module."""
    for (adj, dt), r in sorted(WORST.items()):
        print(f'generic adjoint worst err/bound  {adj:12s} {dt:8s} {r:.3g}')
    assert all(r <= 1.0 for r in WORST.values())
