"""BrownianInterval / Path / Tree on the GPU: the reference's own test properties
(tests/test_brownian_interval.py: shapes :69-107, determinism :110-161, KS tests of marginals
:164-195 and of the conditional bridge law :198-258, consistency identities :261-288,
entropy-determinism of the halfway tree :291-334) plus CUDA-vs-oracle checks of every Brownian
kernel of the C ABI."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import brownian as obm
from . import helpers

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MASK = (1 << 64) - 1


def _tsde():
    import torchsde_b200
    return torchsde_b200


@pytest.mark.parametrize('levy', ['none', 'space-time', 'davie', 'foster'])
@pytest.mark.parametrize('size', [(16, 3), (16,), ()])
def test_shapes(levy, size):
    tsde = _tsde()
    bm = tsde.BrownianInterval(0.0, 1.0, size=size, dtype=torch.float64, device=DEV, entropy=1,
                               levy_area_approximation=levy)
    for ta, tb in ((0.0, 1.0), (0.2, 0.6), (0.6, 0.9), (0.3, 0.3)):
        W = bm(ta, tb)
        assert W.shape == size
        if levy != 'none':
            W, U = bm(ta, tb, return_U=True)
            assert U.shape == size
        if levy in ('davie', 'foster'):
            W, U, A = bm(ta, tb, return_U=True, return_A=True)
            if ta != tb:  # (for ta == tb the reference returns zeros of shape (*size, size[-1]), :613-621)
                assert A.shape == ((*size, *size[-1:]) if len(size) >= 2 else size)
            W2, A2 = bm(ta, tb, return_A=True)
            assert A2.shape == A.shape


@pytest.mark.parametrize('levy', ['none', 'space-time', 'foster'])
def test_determinism_and_consistency(levy):
    tsde = _tsde()
    kw = dict(size=(64, 5), dtype=torch.float64, device=DEV, entropy=77, levy_area_approximation=levy)
    bm = tsde.BrownianInterval(0.0, 1.0, cache_size=3, **kw)
    pts = np.sort(np.random.RandomState(0).rand(12))
    first = [bm(a, b, return_U=levy != 'none') for a, b in zip(pts[:-1], pts[1:])]
    again = [bm(a, b, return_U=levy != 'none') for a, b in zip(pts[:-1], pts[1:])]
    for x, y in zip(first, again):
        x, y = (x, y) if levy == 'none' else (x[0], y[0])
        assert torch.equal(x, y)
    # additivity W(a,c) = W(a,b) + W(b,c); U identity of tests/test_brownian_interval.py:284-288
    a, b, c = 0.15, 0.4, 0.85
    if levy == 'none':
        torch.testing.assert_close(bm(a, c), bm(a, b) + bm(b, c), rtol=1e-10, atol=1e-12)
    else:
        W, U = bm(a, c, return_U=True)
        W1, U1 = bm(a, b, return_U=True)
        W2, U2 = bm(b, c, return_U=True)
        torch.testing.assert_close(W, W1 + W2, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(U, U1 + U2 + (c - b) * W1, rtol=1e-10, atol=1e-12)
    # same entropy, fresh object, different query order -> halfway tree gives the same path
    t1 = tsde.BrownianInterval(0.0, 1.0, halfway_tree=True, tol=1e-6, **kw)
    t2 = tsde.BrownianInterval(0.0, 1.0, halfway_tree=True, tol=1e-6, **kw)
    qs = [(0.1, 0.3), (0.5, 0.75), (0.3, 0.5), (0.0, 1.0), (0.62, 0.63)]
    r1 = [t1(a_, b_) for a_, b_ in qs]
    r2 = [t2(a_, b_) for a_, b_ in reversed(qs)][::-1]
    for x, y in zip(r1, r2):
        torch.testing.assert_close(x, y, rtol=1e-9, atol=1e-10)


def _ks(x, std):
    return stats.kstest(x.double().cpu().numpy().ravel(), lambda v: stats.norm.cdf(v, scale=std)).pvalue


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_marginal_laws(dtype):
    """W ~ N(0, h), H ~ N(0, h/12) (KS, alpha = 1e-5, 131072 samples)."""
    tsde = _tsde()
    n = 131072
    bm = tsde.BrownianInterval(0.0, 1.0, size=(n, 1), dtype=dtype, device=DEV, entropy=2021,
                               levy_area_approximation='space-time')
    for ta, tb in ((0.0, 1.0), (0.25, 0.5), (0.1, 0.37)):
        W, U = bm(ta, tb, return_U=True)
        h = tb - ta
        H = U / h - 0.5 * W
        assert _ks(W, math.sqrt(h)) > 1e-5
        assert _ks(H, math.sqrt(h / 12)) > 1e-5
    # grid cells (dt hint): the path the solver sees
    g = tsde.BrownianInterval(0.0, 1.0, size=(n, 1), dtype=dtype, device=DEV, entropy=5, dt=0.125,
                              levy_area_approximation='space-time')
    W, U = g(0.25, 0.375, return_U=True)
    assert _ks(W, math.sqrt(0.125)) > 1e-5
    W, U = g(0.0, 1.0, return_U=True)  # merge of 8 cells
    assert _ks(W, 1.0) > 1e-5
    assert _ks(U / 1.0 - 0.5 * W, math.sqrt(1 / 12)) > 1e-5
    W, U = g(0.3, 0.6, return_U=True)  # partial cells through the in-cell bridge
    assert _ks(W, math.sqrt(0.3)) > 1e-5
    assert _ks(U / 0.3 - 0.5 * W, math.sqrt(0.3 / 12)) > 1e-5


def test_conditional_bridge_law():
    """tests/test_brownian_interval.py:198-258: law of W(ta,t) given W(ta,tb) (and H)."""
    tsde = _tsde()
    n = 131072
    ta, t, tb = 0.2, 0.5, 0.9
    bm = tsde.BrownianInterval(0.0, 1.0, size=(n, 1), dtype=torch.float64, device=DEV, entropy=8)
    W = bm(ta, tb)
    W1 = bm(ta, t)
    mean = (t - ta) / (tb - ta) * W
    std = math.sqrt((t - ta) * (tb - t) / (tb - ta))
    assert _ks(W1 - mean, std) > 1e-5
    # independence of non-overlapping increments (correlation ~ 0)
    W2 = bm(t, tb)
    corr = torch.corrcoef(torch.stack([W1.ravel(), W2.ravel()]))[0, 1].abs().item()
    assert corr < 0.02


def test_user_W_and_tree_and_path():
    tsde = _tsde()
    w0 = torch.zeros(32, 4, dtype=torch.float64, device=DEV)
    w1 = torch.randn(32, 4, dtype=torch.float64, device=DEV)
    tree = tsde.BrownianTree(t0=0.0, w0=w0, t1=1.0, w1=w1, entropy=3, tol=1e-8)
    torch.testing.assert_close(tree(0.0, 1.0), w1 - w0)
    torch.testing.assert_close(tree(0.0, 0.4) + tree(0.4, 1.0), w1 - w0, rtol=1e-9, atol=1e-10)
    path = tsde.BrownianPath(t0=0.0, w0=w0)
    a = path(0.0, 0.5)
    assert torch.equal(a, path(0.0, 0.5))
    with pytest.warns(UserWarning):
        p = path(0.5)
    torch.testing.assert_close(p, a + w0)
    rev = tsde.ReverseBrownian(tree)
    torch.testing.assert_close(rev(-0.4, -0.1), tree(0.1, 0.4))
    like = tsde.brownian_interval_like(w1, entropy=4)
    assert like.shape == w1.shape and like.dtype == w1.dtype and like.device == w1.device


def test_errors_and_warnings():
    tsde = _tsde()
    with pytest.raises(ValueError):
        tsde.BrownianInterval(1.0, 0.0, size=(2, 2), device=DEV)
    with pytest.raises(ValueError):
        tsde.BrownianInterval(0.0, 1.0, size=(2, 2), device=DEV, levy_area_approximation='bogus')
    with pytest.raises(ValueError):
        tsde.BrownianInterval(0.0, 1.0, size=(2, 2), device=DEV, halfway_tree=True)
    with pytest.raises(ValueError):
        tsde.BrownianInterval(0.0, 1.0, device=DEV)
    bm = tsde.BrownianInterval(0.0, 1.0, size=(2, 2), device=DEV)
    with pytest.raises(RuntimeError):
        bm(0.7, 0.3)
    with pytest.warns(UserWarning):
        bm(-0.5, 0.5)
    with pytest.warns(UserWarning):
        bm(0.5, 1.5)


# ---- kernels vs oracle -----------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['f32', 'f64'])
@pytest.mark.parametrize('levy', ['none', 'space-time'])
@pytest.mark.parametrize('size', [(33, 8), (17, 5), (9, 1)])
def test_cells_and_bridge_vs_oracle(dtype, levy, size):
    tsde = _tsde()
    tdt, npdt = (torch.float64, np.float64) if dtype == 'f64' else (torch.float32, np.float32)
    tol = dict(rtol=1e-12, atol=1e-13) if dtype == 'f64' else dict(rtol=2e-5, atol=5e-6)
    have_h = levy != 'none'
    rows, m = size
    # (1) grid cells + merges
    bm = tsde.BrownianInterval(0.0, 1.0, size=size, dtype=tdt, device=DEV, entropy=99, dt=0.125,
                               levy_area_approximation=levy)
    out = bm(0.25, 0.75, return_U=have_h)
    grid = bm._root
    assert grid.kind == 2
    W, H = obm.cells(bm._key, (grid.cell_base + 2) & MASK, [0.125] * 4, rows, m, npdt, have_h)
    if have_h:
        np.testing.assert_allclose(out[0].cpu().numpy(), W, **tol)
        np.testing.assert_allclose(out[1].cpu().numpy(), obm.h_to_u(W, H, 0.5), **tol)
    else:
        np.testing.assert_allclose(out.cpu().numpy(), W, **tol)
    # (2) binary bridge below the root
    bm2 = tsde.BrownianInterval(0.0, 1.0, size=size, dtype=tdt, device=DEV, entropy=123,
                                levy_area_approximation=levy)
    from torchsde_b200._brownian.interval import child_id
    out = bm2(0.3, 0.45, return_U=have_h)
    root = bm2._root
    W0, H0 = obm.cell(bm2._key, root.id, 1.0, rows, m, npdt, have_h)
    # tree built by the query: root split at 0.3 -> right [0.3,1] split at 0.45 -> left [0.3,0.45]
    right_id = child_id(root.id, 1)
    W, H = obm.bridge_chain(bm2._key, W0, H0, [(root.id, False, 0.0, 0.3, 1.0), (right_id, True, 0.3, 0.45, 1.0)])
    if have_h:
        np.testing.assert_allclose(out[0].cpu().numpy(), W, **tol)
        np.testing.assert_allclose(out[1].cpu().numpy(), obm.h_to_u(W, H, 0.45 - 0.3), **tol)
    else:
        np.testing.assert_allclose(out.cpu().numpy(), W, **tol)


@pytest.mark.parametrize('dtype', ['f32', 'f64'])
@pytest.mark.parametrize('levy', ['davie', 'foster'])
@pytest.mark.parametrize('rows,m', [(21, 4), (300, 16), (70, 8), (9, 5), (6, 40), (11, 2)])
def test_levy_area_vs_oracle(dtype, levy, rows, m):
    tsde = _tsde()
    tdt, npdt = (torch.float64, np.float64) if dtype == 'f64' else (torch.float32, np.float32)
    tol = dict(rtol=1e-12, atol=1e-13) if dtype == 'f64' else dict(rtol=3e-5, atol=1e-5)
    bm = tsde.BrownianInterval(0.0, 2.0, size=(rows, m), dtype=tdt, device=DEV, entropy=5,
                               levy_area_approximation=levy)
    W_, U_, A_ = bm(0.0, 2.0, return_U=True, return_A=True)
    root = bm._root
    W, H = obm.cell(bm._key, root.id, 2.0, rows, m, npdt, True)
    A = obm.davie_foster(W, H, 2.0, levy == 'foster', obm.levy_noise(bm._key, root.id, rows, m, npdt))
    np.testing.assert_allclose(A_.cpu().numpy(), A, **tol)
    # antisymmetry and the merged query
    assert torch.allclose(A_, -A_.transpose(-1, -2))
    W2, U2, A2 = bm(0.5, 1.5, return_U=True, return_A=True)
    assert torch.allclose(A2, -A2.transpose(-1, -2), atol=1e-6)


@pytest.mark.parametrize('path', helpers.golden_files('bridge_'), ids=helpers.case_id)
def test_bridge_kernel_vs_reference_golden(path):
    """tsde_brownian_bridge against the REFERENCE's bridge outputs: same parent (W,H), same split
    geometry; since the kernel draws its own normals, the check is through the oracle identity
    out = lin(W,H) + noise-part with the reference's recorded normals replaced -> compare the
    deterministic (noise-free) part by differencing two entropies."""
    # The kernel's arithmetic is pinned to the oracle (test_cells_and_bridge_vs_oracle) and the
    # oracle's bridge() is pinned to the reference (tests/test_oracle_golden.py); here we add the
    # direct statistical check that the kernel reproduces the reference's *conditional mean*.
    tsde = _tsde()
    case = helpers.load(path)
    levy = str(case['levy'])
    if levy not in ('none', 'space-time'):
        pytest.skip('mean check done on W/H variants')
    f64 = path.endswith('f64.npz')
    tdt = torch.float64 if f64 else torch.float32
    W0 = torch.from_numpy(case['W0']).to(DEV)
    H0 = torch.from_numpy(case['H0']).to(DEV)
    reps = 4096
    Wb = W0.repeat(reps, 1).contiguous()
    Hb = H0.repeat(reps, 1).contiguous()
    bm = tsde.BrownianInterval(0.0, 1.0, size=tuple(Wb.shape), dtype=tdt, device=DEV, entropy=1,
                               levy_area_approximation=levy, W=Wb, H=Hb if levy != 'none' else None)
    W = bm(0.0, 0.3)
    # E[W(0,0.3) | W, H] = 0.3 W + 6*0.3*0.7 H (brownian_interval.py:214-216) ; W-only: 0.3 W
    mean = W.reshape(reps, *W0.shape).mean(0)
    expect = 0.3 * W0 + (6 * 0.3 * 0.7 * H0 if levy != 'none' else 0)
    assert (mean - expect).abs().max().item() < 0.05


@pytest.mark.parametrize('kind', ['path', 'tree'])
def test_path_and_tree_bridge_law(kind):
    """Reference tests/test_brownian_path.py:72-96 and test_brownian_tree.py:79-103: KS test of W(t) at a
    random time t given the end points (alpha = 1e-5)."""
    tsde = _tsde()
    n = 65536
    rng = np.random.RandomState(3)
    t0, t1 = 0.0, 1.0
    w0 = torch.zeros(n, 1, dtype=torch.float64, device=DEV)
    if kind == 'tree':
        w1 = torch.randn(n, 1, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
        bm = tsde.BrownianTree(t0=t0, w0=w0, t1=t1, w1=w1, entropy=9, tol=1e-10, pool_size=100)
        end = w1
    else:
        bm = tsde.BrownianPath(t0=t0, w0=w0)
        end = bm(t0, t1)
    for _ in range(3):
        t = float(rng.uniform(0.05, 0.95))
        wt = bm(t0, t)
        mean = (t - t0) / (t1 - t0) * end
        std = math.sqrt((t - t0) * (t1 - t) / (t1 - t0))
        assert _ks(wt - mean, std) > 1e-5
    # determinism + repr / properties
    assert torch.equal(bm(0.2, 0.6), bm(0.2, 0.6))
    assert 'Brownian' in repr(bm) and bm.shape == (n, 1) and bm.dtype == torch.float64
    assert bm.levy_area_approximation == 'none'


def test_interval_properties_and_cache_sizes():
    tsde = _tsde()
    for cache_size in (None, 0, 5):
        bm = tsde.BrownianInterval(0.0, 1.0, size=(8, 2), dtype=torch.float32, device=DEV, entropy=1,
                                   cache_size=cache_size, pool_size=16, tol=0.0)
        pts = np.linspace(0, 1, 30)
        a = [bm(x, y) for x, y in zip(pts[:-1], pts[1:])]
        b = [bm(x, y) for x, y in zip(pts[:-1], pts[1:])]
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        torch.testing.assert_close(sum(a), bm(0.0, 1.0), rtol=1e-4, atol=1e-5)
        assert bm.cache_size == cache_size and bm.pool_size == 16 and bm.entropy == 1 and bm.tol == 0.0
        assert bm.dt is None and bm.halfway_tree is False and bm.size() == (8, 2)
    e1 = tsde.BrownianInterval(0.0, 1.0, size=(8, 2), device=DEV, entropy=1)(0.1, 0.4)
    e2 = tsde.BrownianInterval(0.0, 1.0, size=(8, 2), device=DEV, entropy=2)(0.1, 0.4)
    assert not torch.equal(e1, e2)
    r = tsde.BrownianInterval(0.0, 1.0, size=(8, 2), device=DEV)  # entropy from numpy's global RNG (:489-490)
    assert isinstance(r.entropy, int)


@pytest.mark.parametrize('levy', ['davie', 'foster'])
@pytest.mark.parametrize('m', [2, 3, 16, 24])
def test_levy_area_noise_law(levy, m):
    """The Levy-area noise is drawn as ONE normal per pair i < j (csrc/brownian.cu): (A_ij - (H_i W_j - W_i H_j)) /
    std_ij must be N(0, 2) like the reference's antisymmetrised iid matrix N - N^T (brownian_interval.py:88-90),
    independent across pairs, and A exactly antisymmetric with a zero diagonal."""
    tsde = _tsde()
    n = 32768
    h = 0.5
    bm = tsde.BrownianInterval(0.0, h, size=(n, m), dtype=torch.float64, device=DEV, entropy=17,
                               levy_area_approximation=levy)
    W, U, A = bm(0.0, h, return_U=True, return_A=True)
    H = U / h - 0.5 * W
    assert torch.equal(A, -A.transpose(1, 2)) and float(A.diagonal(dim1=1, dim2=2).abs().max()) == 0.0
    base = H.unsqueeze(2) * W.unsqueeze(1) - W.unsqueeze(2) * H.unsqueeze(1)
    if levy == 'foster':
        H2 = H ** 2
        std = torch.sqrt(0.1 * h * (0.1 * h + H2.unsqueeze(2) + H2.unsqueeze(1)))
    else:
        std = torch.full_like(base, math.sqrt(h * h / 12))
    z = (A - base) / std
    iu = torch.triu_indices(m, m, offset=1)
    zu = z[:, iu[0], iu[1]]                                   # (n, npairs)
    assert _ks(zu[:, 0], math.sqrt(2.0)) > 1e-5 and _ks(zu[:, -1], math.sqrt(2.0)) > 1e-5
    assert _ks(zu.reshape(-1)[:262144], math.sqrt(2.0)) > 1e-5
    if zu.shape[1] >= 2:
        corr = torch.corrcoef(zu[:, :min(8, zu.shape[1])].T)
        off = corr - torch.diag(torch.diag(corr))
        assert float(off.abs().max()) < 0.03


@pytest.mark.parametrize('levy', ['davie', 'foster'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('size', [(257, 8), (1030, 16), (77, 4), (45, 32), (19, 12), (5, 64)])
def test_fused_cell_levy_query_equals_general_path(levy, dtype, size):
    """tsde_brownian_cell_levy (W, U, A of one whole grid cell in one launch) against the three-kernel general path
    (cells -> levy_area -> h_to_u) on the same Brownian motion: bit-identical.  The fused kernel draws the W | H
    normals of 64/m rows per warp pass: the row counts are not multiples of that group."""
    tsde = _tsde()
    kw = dict(size=size, dtype=dtype, device=DEV, entropy=99, dt=0.125, levy_area_approximation=levy)
    fused = tsde.BrownianInterval(0.0, 1.0, **kw)
    general = tsde.BrownianInterval(0.0, 1.0, **kw)
    for k in (0, 3, 7):
        ta, tb = k * 0.125, (k + 1) * 0.125
        Wf, Uf, Af = fused(ta, tb, return_U=True, return_A=True)
        general(ta, tb, return_U=True)                      # materialises (and caches) the cell: no fused launch next
        Wg, Ug, Ag = general(ta, tb, return_U=True, return_A=True)
        assert torch.equal(Wf, Wg) and torch.equal(Uf, Ug) and torch.equal(Af, Ag)
    # a two-cell query cannot use the fused launch: the run of cells is one piece with its own Levy noise (like a
    # parent node of the reference's tree, whose area is drawn from its merged (W, H), :78-99) — still antisymmetric,
    # and its W is the sum of the cells' increments
    W2, A2 = fused(0.0, 0.25, return_A=True)
    W0 = general(0.0, 0.125)
    W1 = general(0.125, 0.25)
    torch.testing.assert_close(W2, W0 + W1, rtol=1e-5, atol=1e-6)
    assert torch.equal(A2, -A2.transpose(1, 2))
