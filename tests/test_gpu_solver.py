"""Parity of the CUDA solver path (through the C ABI) with the reference and the oracle.

* golden replay: torchsde_b200.sdeint on cuda, fed the increments the REFERENCE consumed when the
  golden file was generated (duck-typed bm, SURVEY fact 3) -> compared with the reference's ys.
  GBM problems use IEEE +,* only in f/g, there the result must be BIT-IDENTICAL to the reference.
* counter path: sdeint with this repo's BrownianInterval (increments regenerated in registers)
  vs the numpy oracle integrating the same Philox-defined path.
"""
import numpy as np
import pytest
import torch

from oracle import brownian as obm
from oracle import solvers
from . import helpers, problems

pytestmark = pytest.mark.gpu

SOLVER_CASES = helpers.golden_files('solver_')
MASK = (1 << 64) - 1


def _tsde():
    import torchsde_b200
    return torchsde_b200


@pytest.fixture(autouse=True)
def _inference_mode():
    """These tests exercise the fused fast path: like the reference's diagnostics / benchmarks they solve
    under torch.no_grad() (with autograd enabled and parameters requiring grad, `sdeint` takes the
    differentiable path, which tests/test_gpu_adjoint.py covers)."""
    with torch.no_grad():
        yield


@pytest.mark.parametrize('path', SOLVER_CASES, ids=helpers.case_id)
def test_golden_replay(path):
    tsde = _tsde()
    case = helpers.load(path)
    dev = torch.device('cuda')
    sde = helpers.build_problem(case, device=dev)
    bm = helpers.replay_torch(case, dev)
    opts = {'grad_free': True} if bool(case['grad_free']) else None
    y0 = torch.from_numpy(case['y0']).to(dev)
    ts = torch.from_numpy(case['ts']).to(dev)
    method = str(case['method'])
    out = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=float(case['dt']), options=opts,
                      extra=method == 'reversible_heun')
    ys, extra = out if method == 'reversible_heun' else (out, ())
    ys = ys.cpu().numpy()
    ref = case['ys']
    assert ys.shape == ref.shape and ys.dtype == ref.dtype
    kind = str(case['kind'])
    if kind == 'gbm':
        assert np.array_equal(ys, ref), f"max abs diff {np.abs(ys - ref).max()}"
    else:
        np.testing.assert_allclose(ys, ref, **helpers.tol_for(str(case['dtype']), kind == 'scalar'))
    for i, e in enumerate(extra):
        np.testing.assert_allclose(e.cpu().numpy(), case[f'extra{i}'], **helpers.tol_for(str(case['dtype']), False))


@pytest.mark.parametrize('path', helpers.golden_files('ito_diagonal_'), ids=helpers.case_id)
@pytest.mark.parametrize('dtype', ['f64', 'f32'])
def test_ito_diagonal_fixture(path, dtype):
    """north_star: outputs within 1e-5 rel of the reference on diagnostics/ito_diagonal (fp32);
    fp64 <= 1e-10 (SURVEY §8c)."""
    tsde = _tsde()
    case = helpers.load(path)
    dev = torch.device('cuda')
    tdt = torch.float64 if dtype == 'f64' else torch.float32
    mod = problems.MLPDiagonal(int(case['d'])).double()
    mod.load_state_dict({k[len('param.'):]: torch.from_numpy(v) for k, v in case.items() if k.startswith('param.')})
    mod = mod.to(tdt).to(dev)
    Ws = [torch.from_numpy(w).to(tdt).to(dev) for w in case['W']]
    Us = [torch.from_numpy(u).to(tdt).to(dev) for u in case['U']]
    bm = problems.ReplayBM(case['ta'], case['tb'], Ws, Us, levy='space-time')
    y0 = torch.from_numpy(case['y0']).to(tdt).to(dev)
    ts = torch.from_numpy(case['ts']).to(tdt).to(dev)  # linspace(0, 2, 10), dt = 0.1 (diagnostics/ito_diagonal.py:31-33)
    ys = tsde.sdeint(mod, y0, ts, bm=bm, method=str(case['method']), dt=float(case['dt']),
                     options={'grad_free': True} if bool(case['grad_free']) else None)
    ys = ys.double().cpu().numpy()
    ref = case['ys']
    if dtype == 'f64':
        np.testing.assert_allclose(ys, ref, rtol=1e-10, atol=1e-12)
    else:
        assert np.all(np.abs(ys - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref)))


def _oracle_bm_from(bm, rows, m, npdt, have_h):
    """numpy view of the Brownian path of a grid-bound torchsde_b200.BrownianInterval."""
    grid, key = bm._root, bm._key

    def query(ta, tb, return_U=False):
        i = grid.bounds.index(float(ta))
        j = grid.bounds.index(float(tb))
        lengths = [grid.bounds[k + 1] - grid.bounds[k] for k in range(i, j)]
        W, H = obm.cells(key, (grid.cell_base + i) & MASK, lengths, rows, m, npdt, have_h)
        if return_U:
            return W, obm.h_to_u(W, H, float(tb) - float(ta))
        return W
    return query


COUNTER_CASES = [
    ('gbm', 'ito', 'euler', None, 8, 8), ('gbm', 'ito', 'milstein', None, 6, 6),
    ('gbm', 'ito', 'milstein', {'grad_free': True}, 8, 8), ('gbm', 'ito', 'srk', None, 8, 8),
    ('gbm', 'stratonovich', 'heun', None, 8, 8), ('gbm', 'stratonovich', 'midpoint', None, 5, 5),
    ('gbm', 'stratonovich', 'euler_heun', None, 8, 8), ('gbm', 'stratonovich', 'reversible_heun', None, 8, 8),
    ('gbm', 'stratonovich', 'milstein', None, 8, 8),
    ('scalar', 'ito', 'milstein', None, 6, 1), ('scalar', 'ito', 'srk', None, 6, 1),
    ('scalar', 'stratonovich', 'heun', None, 6, 1),
    ('general', 'ito', 'euler', None, 4, 8), ('general', 'stratonovich', 'heun', None, 3, 2),
    ('general', 'stratonovich', 'midpoint', None, 4, 16), ('general', 'stratonovich', 'reversible_heun', None, 4, 8),
    ('general', 'stratonovich', 'euler_heun', None, 4, 8),
    ('additive', 'ito', 'srk', None, 4, 8), ('additive', 'ito', 'milstein', None, 3, 2),
    ('additive', 'ito', 'euler', None, 32, 16),
]


@pytest.mark.parametrize('kind,sde_type,method,opts,d,m', COUNTER_CASES)
@pytest.mark.parametrize('dtype', ['f32', 'f64'])
def test_counter_path_vs_oracle(kind, sde_type, method, opts, d, m, dtype):
    tsde = _tsde()
    dev = torch.device('cuda')
    tdt, npdt = (torch.float64, np.float64) if dtype == 'f64' else (torch.float32, np.float32)
    B = 37
    sde = problems.make(kind, d, m, sde_type, dtype=tdt, seed=2)
    bm_m = d if kind == 'gbm' else m
    y0 = (0.2 + 0.3 * torch.rand(B, d, generator=torch.Generator().manual_seed(5), dtype=torch.float64)).to(tdt)
    ts = np.array([0.0, 0.125, 0.25, 0.375], dtype=npdt)
    dt = 2.0 ** -4
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, 0.375, size=(B, bm_m), dtype=tdt, device=dev, entropy=4242,
                               levy_area_approximation=levy)
    sde_dev = problems.make(kind, d, m, sde_type, dtype=tdt, seed=2).to(dev)
    ys = tsde.sdeint(sde_dev, y0.to(dev), torch.from_numpy(ts).to(dev), bm=bm, method=method, dt=dt,
                     options=opts)
    assert bm._root.kind == 2, "solver did not bind its grid (fast path not taken)"
    sde_cpu = problems.make(kind, d, m, sde_type, dtype=tdt, seed=2)
    oracle_bm = _oracle_bm_from(bm, B, bm_m, npdt, levy != 'none')
    ref, _ = solvers.make(method, problems.NumpySDE(sde_cpu), oracle_bm, dt, opts).integrate(y0.numpy(), ts)
    tol = dict(rtol=1e-11, atol=1e-12) if dtype == 'f64' else dict(rtol=5e-5, atol=1e-5)
    np.testing.assert_allclose(ys.cpu().numpy(), ref, **tol)


@pytest.mark.parametrize('kind,sde_type,method,d,m', [('gbm', 'ito', 'milstein', 64, 64), ('gbm', 'ito', 'srk', 12, 12),
                                                      ('general', 'stratonovich', 'heun', 8, 16),
                                                      ('scalar', 'ito', 'euler', 7, 1)])
def test_registers_equal_materialised(kind, sde_type, method, d, m):
    """The increment regenerated in registers inside the tableau kernel is bit-identical to the one
    BrownianInterval.__call__ materialises for the same interval."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B = 129
    sde = problems.make(kind, d, m, sde_type, dtype=torch.float32, seed=1).to(dev)
    bm_m = d if kind == 'gbm' else m
    y0 = torch.full((B, d), 0.3, device=dev)
    ts = torch.tensor([0.0, 0.25, 0.5], device=dev)
    dt = 2.0 ** -3
    levy = 'space-time' if method == 'srk' else 'none'
    bm = tsde.BrownianInterval(0.0, 0.5, size=(B, bm_m), dtype=torch.float32, device=dev, entropy=9,
                               levy_area_approximation=levy)
    fast = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt)

    class Materialised:  # same path, but through __call__ (memory source)
        shape = bm.shape
        levy_area_approximation = levy
        dtype = bm.dtype
        device = bm.device

        def __call__(self, ta, tb=None, return_U=False, return_A=False):
            return bm(ta, tb, return_U=return_U)

    slow = tsde.sdeint(sde, y0, ts, bm=Materialised(), method=method, dt=dt)
    assert torch.equal(fast, slow)


def test_batch_sharding_is_invisible():
    """Rows are independent Philox streams keyed by the GLOBAL row: solving shards separately
    reproduces the unsharded solve bit for bit (SURVEY §8e)."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B, D = 96, 16
    sde = problems.GBMDiagonal(D, 'ito', seed=4, dtype=torch.float32).to(dev)
    y0 = torch.rand(B, D, device=dev) + 0.1
    ts = torch.tensor([0.0, 0.5, 1.0], device=dev)
    full = tsde.sdeint(sde, y0, ts, bm=tsde.BrownianInterval(0., 1., size=(B, D), dtype=torch.float32, device=dev,
                                                             entropy=31), method='milstein', dt=0.125)
    parts = []
    for r0, r1 in ((0, 40), (40, 96)):
        bm = tsde.BrownianInterval(0., 1., size=(r1 - r0, D), dtype=torch.float32, device=dev, entropy=31)
        bm.shard_rows(r0)
        parts.append(tsde.sdeint(sde, y0[r0:r1].contiguous(), ts, bm=bm, method='milstein', dt=0.125))
    assert torch.equal(full, torch.cat(parts, dim=1))


def test_specialised_functions_agree():
    """Reference tests/test_sdeint.py:79-98: six ways of supplying f/g/f_and_g/g_prod/f_and_g_prod.
    Here the fused contraction and the user's own bmm may differ by summation-order rounding, so
    the variants agree to rounding instead of bit for bit (documented in DESIGN.md)."""
    tsde = _tsde()
    dev = torch.device('cuda')
    d, m, B = 3, 2, 4
    vector = torch.randn(m, dtype=torch.float64, device=dev)

    def gmat(y):
        return y.unsqueeze(-1).sigmoid() * vector

    def gprod(y, v):
        return gmat(y).bmm(v.unsqueeze(-1)).squeeze(-1)

    class Base(torch.nn.Module):
        noise_type = 'general'

        def __init__(self, sde_type):
            super().__init__()
            self.sde_type = sde_type

    class FG(Base):
        def f(self, t, y): return -y
        def g(self, t, y): return gmat(y)

    class FAndG(Base):
        def f_and_g(self, t, y): return -y, gmat(y)

    class GProd(Base):
        def f(self, t, y): return -y
        def g_prod(self, t, y, v): return gprod(y, v)

    class FAndGProd(Base):
        def f_and_g_prod(self, t, y, v): return -y, gprod(y, v)

    class FAndGGProd1(Base):
        def f_and_g(self, t, y): return -y, gmat(y)
        def g_prod(self, t, y, v): return gprod(y, v)

    class FAndGGProd2(Base):
        def f(self, t, y): return -y
        def f_and_g(self, t, y): return -y, gmat(y)
        def g_prod(self, t, y, v): return gprod(y, v)

    y0 = torch.randn(B, d, dtype=torch.float64, device=dev)
    for sde_type, method in (('ito', 'euler'), ('stratonovich', 'midpoint')):
        outs = []
        for cls in (FG, FAndG, GProd, FAndGProd, FAndGGProd1, FAndGGProd2):
            bm = tsde.BrownianInterval(0.0, 0.3, (B, m), dtype=torch.float64, device=dev, entropy=45678)
            outs.append(tsde.sdeint(cls(sde_type), y0, [0.0, 0.3], dt=0.05, bm=bm, method=method)[1])
        for o in outs[1:]:
            assert o.shape == outs[0].shape
            torch.testing.assert_close(o, outs[0], rtol=1e-12, atol=1e-13)


def test_ragged_ts_interpolation_and_reuse():
    """Output times that are not multiples of dt (linear_interp, interp.py:15-18) and later solves on the same bm
    with a coarser, nested grid: each coarse step merges 8 bound cells in the kernel (n_cells > 1, cell lengths read
    from the device, and for SRK the H-merge rule).  Both against the oracle, which merges the same cells."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B, D = 16, 4
    sde = problems.GBMDiagonal(D, 'ito', seed=4, dtype=torch.float64).to(dev)
    sde_cpu = problems.GBMDiagonal(D, 'ito', seed=4, dtype=torch.float64)
    y0 = torch.full((B, D), 0.5, dtype=torch.float64, device=dev)
    bm = tsde.BrownianInterval(0., 1., size=(B, D), dtype=torch.float64, device=dev, entropy=3,
                               levy_area_approximation='space-time')
    ts = np.linspace(0, 1, 7)
    fine = tsde.sdeint(sde, y0, torch.from_numpy(ts).to(dev), bm=bm, method='euler', dt=2.0 ** -6)
    assert fine.shape == (7, B, D)
    oracle_bm = _oracle_bm_from(bm, B, D, np.float64, True)
    ref, _ = solvers.make('euler', problems.NumpySDE(sde_cpu), oracle_bm, 2.0 ** -6).integrate(y0.cpu().numpy(), ts)
    np.testing.assert_allclose(fine.cpu().numpy(), ref, rtol=1e-11, atol=1e-12)
    # coarser nested grid re-uses the same cells (merged): the Brownian path is the same object
    w_all = bm(0.0, 1.0)
    ts = np.array([0.0, 0.3, 0.55, 0.8, 1.0])
    for method in ('euler', 'srk'):
        with torch.no_grad():  # the fused step kernels
            coarse = tsde.sdeint(sde, y0, torch.from_numpy(ts).to(dev), bm=bm, method=method, dt=2.0 ** -3)
        ref, _ = solvers.make(method, problems.NumpySDE(sde_cpu), oracle_bm, 2.0 ** -3).integrate(
            y0.cpu().numpy(), ts)
        np.testing.assert_allclose(coarse.cpu().numpy(), ref, rtol=1e-11, atol=1e-12, err_msg=method)
    s = sum(bm(k / 8, (k + 1) / 8) for k in range(8))
    torch.testing.assert_close(s, w_all, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize('kind,sde_type,method,d,m', [('gbm', 'ito', 'milstein', 64, 64), ('gbm', 'ito', 'srk', 8, 8),
                                                      ('general', 'stratonovich', 'heun', 8, 16),
                                                      ('gbm', 'stratonovich', 'reversible_heun', 8, 8)])
def test_cuda_graph_equals_eager(kind, sde_type, method, d, m):
    """options={'cuda_graph': True}: replayed solves are bit-identical to the eager loop, including
    replays with a new Brownian key / new y0 (only static buffers are refreshed)."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B = 64
    sde = problems.make(kind, d, m, sde_type, dtype=torch.float32, seed=1).to(dev)
    bm_m = d if kind == 'gbm' else m
    ts = torch.tensor([0.0, 0.125, 0.25, 0.5], device=dev)
    levy = 'space-time' if method == 'srk' else 'none'
    for entropy, fill in ((11, 0.3), (12, 0.6), (11, 0.3)):
        y0 = torch.full((B, d), fill, device=dev)
        outs = []
        for graph in (False, True):
            bm = tsde.BrownianInterval(0.0, 0.5, size=(B, bm_m), dtype=torch.float32, device=dev, entropy=entropy,
                                       levy_area_approximation=levy)
            outs.append(tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=2.0 ** -4,
                                    options={'cuda_graph': graph}).clone())
        assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('path', helpers.golden_files('adaptive_'), ids=helpers.case_id)
def test_adaptive_golden_replay(path):
    """adaptive=True on the reference's increments: same accept/reject history, same ys."""
    import warnings
    tsde = _tsde()
    case = helpers.load(path)
    dev = torch.device('cuda')
    sde = helpers.build_problem(case, device=dev)
    bm = helpers.replay_torch(case, dev)
    calls = []
    inner = bm.__call__

    class Counting:
        shape, levy_area_approximation = bm.shape, bm.levy_area_approximation

        def __call__(self, ta, tb=None, return_U=False, return_A=False):
            calls.append((float(ta), float(tb)))
            return bm(ta, tb, return_U=return_U)

    y0 = torch.from_numpy(case['y0']).to(dev)
    ts = torch.from_numpy(case['ts']).to(dev)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ys = tsde.sdeint(sde, y0, ts, bm=Counting(), method=str(case['method']), dt=float(case['dt']), adaptive=True,
                         rtol=float(case['rtol']), atol=float(case['atol']), dt_min=float(case['dt_min']))
    assert len(calls) == int(case['n_queries'])
    np.testing.assert_allclose(ys.cpu().numpy(), case['ys'], rtol=1e-9, atol=1e-11)


@pytest.mark.parametrize('path', helpers.golden_files('logode_'), ids=helpers.case_id)
def test_log_ode_golden_replay(path):
    """methods/log_ode.py on the reference's increments and Levy areas."""
    tsde = _tsde()
    case = helpers.load(path)
    dev = torch.device('cuda')
    sde = helpers.build_problem(case, device=dev)
    Ws = [torch.from_numpy(w).to(dev) for w in case['W']]
    Us = [torch.from_numpy(u).to(dev) for u in case['U']]
    As = [torch.from_numpy(a).to(dev) for a in case['A']]
    bm = problems.ReplayBM(case['ta'], case['tb'], Ws, Us, levy=str(case['levy']), As=As)
    y0 = torch.from_numpy(case['y0']).to(dev)
    ts = torch.from_numpy(case['ts']).to(dev)
    ys = tsde.sdeint(sde, y0, ts, bm=bm, method='log_ode', dt=float(case['dt']))
    np.testing.assert_allclose(ys.cpu().numpy(), case['ys'], rtol=1e-11, atol=1e-13)


def test_log_ode_and_logqp_with_own_brownian():
    """log_ode with this repo's BrownianInterval (foster Levy area from the counter), and logqp=True
    (reference tests/test_sdeint.py:50-68,203-216: shapes (T,B,d) and (T-1,B))."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B, d, m, T = 8, 4, 3, 5
    sde = problems.TanhGeneral(d, m, 'stratonovich', dtype=torch.float64).to(dev)
    y0 = torch.full((B, d), 0.2, dtype=torch.float64, device=dev)
    ts = torch.linspace(0, 0.4, T, dtype=torch.float64, device=dev)
    ys = tsde.sdeint(sde, y0, ts, method='log_ode', dt=0.05)  # default bm -> foster (sdeint.py:262-270)
    assert ys.shape == (T, B, d) and torch.isfinite(ys).all()

    class WithPrior(problems.GBMDiagonal):
        def h(self, t, y):
            return torch.zeros_like(y)

    sde2 = WithPrior(d, 'ito', dtype=torch.float64).to(dev)
    ys2, logqp = tsde.sdeint(sde2, y0, ts, method='euler', dt=0.05, logqp=True)
    assert ys2.shape == (T, B, d) and logqp.shape == (T - 1, B) and (logqp >= 0).all()


def test_row_split_graph_is_bit_identical():
    tsde = _tsde()
    dev = torch.device('cuda')
    B, d = 100, 8
    sde = problems.GBMDiagonal(d, 'ito', seed=3, dtype=torch.float32).to(dev)
    ts = torch.tensor([0.0, 0.25, 0.5], device=dev)
    y0 = torch.rand(B, d, device=dev) + 0.1
    outs = []
    for opts in ({}, {'cuda_graph': True, 'row_split': 2}, {'cuda_graph': True, 'row_split': 3}):
        bm = tsde.BrownianInterval(0.0, 0.5, size=(B, d), dtype=torch.float32, device=dev, entropy=21)
        outs.append(tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=2.0 ** -4, options=opts).clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize('d,m', [(33, 4), (64, 16), (40, 8), (128, 32), (5, 128)])
def test_general_kernel_shapes_vs_oracle(d, m):
    """General-noise fused GEMV tile across row lengths that take the row-major sweep (d*m/4 >= 128,
    including lengths that are not a multiple of the warp size) and the flat sweep."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B = 19
    sde = problems.TanhGeneral(d, m, 'stratonovich', seed=5, dtype=torch.float64).to(dev)
    sde_cpu = problems.TanhGeneral(d, m, 'stratonovich', seed=5, dtype=torch.float64)
    y0 = torch.full((B, d), 0.25, dtype=torch.float64)
    ts = np.array([0.0, 0.125, 0.25])
    bm = tsde.BrownianInterval(0.0, 0.25, size=(B, m), dtype=torch.float64, device=dev, entropy=77)
    ys = tsde.sdeint(sde, y0.to(dev), torch.from_numpy(ts).to(dev), bm=bm, method='heun', dt=2.0 ** -4)
    ref, _ = solvers.make('heun', problems.NumpySDE(sde_cpu), _oracle_bm_from(bm, B, m, np.float64, False),
                          2.0 ** -4).integrate(y0.numpy(), ts)
    np.testing.assert_allclose(ys.cpu().numpy(), ref, rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize('d', [12, 20, 48, 100, 36])
def test_fast_kernel_non_power_of_two_rows(d):
    """d % 4 == 0 with d/4 not a power of two takes the specialised kernel through the magic-number
    division: registers == materialised increments (bit-equal) and shard invariance."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B = 257
    sde = problems.GBMDiagonal(d, 'ito', seed=d, dtype=torch.float32).to(dev)
    y0 = torch.full((B, d), 0.3, device=dev)
    ts = torch.tensor([0.0, 0.25], device=dev)
    bm = tsde.BrownianInterval(0.0, 0.25, size=(B, d), dtype=torch.float32, device=dev, entropy=d)
    fast = tsde.sdeint(sde, y0, ts, bm=bm, method='srk' if d == 36 else 'milstein', dt=2.0 ** -3) if d != 36 else None
    if d == 36:
        bm = tsde.BrownianInterval(0.0, 0.25, size=(B, d), dtype=torch.float32, device=dev, entropy=d,
                                   levy_area_approximation='space-time')
        fast = tsde.sdeint(sde, y0, ts, bm=bm, method='srk', dt=2.0 ** -3)

    class Mat:
        shape, levy_area_approximation = bm.shape, bm.levy_area_approximation

        def __call__(self, ta, tb=None, return_U=False, return_A=False):
            return bm(ta, tb, return_U=return_U)

    slow = tsde.sdeint(sde, y0, ts, bm=Mat(), method='srk' if d == 36 else 'milstein', dt=2.0 ** -3)
    assert torch.equal(fast, slow)


def test_strong_orders_on_one_brownian_path():
    """Convergence orders as in the reference's diagnostics (diagnostics/inspection.py:71-140), against the
    analytic GBM solution y0 exp((mu - sigma^2/2) t + sigma W_t) with W_t read from the SAME Brownian object:
    checks that solves on nested grids (merged primary cells) and `bm(0, t)` describe one consistent path, and
    that Euler / Milstein / SRK show strong orders 0.5 / 1.0 / 1.5."""
    tsde = _tsde()
    dev = torch.device('cuda')
    B, d = 16384, 4
    sde = problems.GBMDiagonal(d, 'ito', seed=7, dtype=torch.float64).to(dev)
    y0 = torch.full((B, d), 0.5, dtype=torch.float64, device=dev)
    ts = torch.tensor([0.0, 1.0], dtype=torch.float64, device=dev)
    bm = tsde.BrownianInterval(0.0, 1.0, size=(B, d), dtype=torch.float64, device=dev, entropy=2024,
                               levy_area_approximation='space-time')
    tsde.sdeint(sde, y0, ts, bm=bm, method='euler', dt=2.0 ** -9)       # binds the finest grid first
    W1 = bm(0.0, 1.0)
    mu, sigma = sde.mu.detach(), sde.sigma.detach()
    exact = y0 * torch.exp((mu - 0.5 * sigma ** 2) * 1.0 + sigma * W1)
    dts = [2.0 ** -k for k in range(2, 8)]
    slopes = {}
    for method in ('euler', 'milstein', 'srk'):
        errs = []
        for dt in dts:
            y1 = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt)[-1]
            errs.append(float(((y1 - exact) ** 2).sum(1).mean().sqrt()))
        slopes[method] = np.polyfit(np.log(dts), np.log(errs), 1)[0]
    assert 0.4 < slopes['euler'] < 0.65, slopes
    assert 0.85 < slopes['milstein'] < 1.15, slopes
    assert 1.3 < slopes['srk'] < 1.7, slopes
