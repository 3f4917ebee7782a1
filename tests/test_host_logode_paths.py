"""CPU tests of the restatements and bounds tests/test_gpu_logode_paths.py and tests/test_gpu_index_paths.py hold the
log-ODE product, the diagonal KL rate and the noise-free row-wise ops to:

* the restatements agree with the package's torch formula (`_kl_rate`), with `oracle/solvers.py` (the SRK stage values
  H0 / H1 and the gradient-free Milstein predictor) and, one log-ODE step at a time, with the reference's general-noise
  log-ODE goldens;
* each bound rejects plausible wrong formulas on at least 75 % of the elements the mistake changes;
* the library refuses `tsde_bmm_ga` for non-general noise and the diagonal `tsde_logqp_augment` past d = 2^24."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import solvers
from torchsde_b200 import _cabi
from . import helpers, logode_ref as ref
from . import test_gpu_index_paths as ip

DTYPES = [np.float32, np.float64]


def _rejects(changed, rejected, what):
    assert changed.sum() > 0, f'{what} changes nothing'
    share = float((rejected & changed).sum()) / float(changed.sum())
    assert share >= 0.75, f'{what}: rejected on {share:.0%} of the {int(changed.sum())} elements it changes'


# ---- the KL rate ---------------------------------------------------------------------------------------------------
def _logqp_operands(npdt, B=64, d=45):
    from .test_gpu_logode_paths import _logqp_inputs
    return _logqp_inputs(np.random.default_rng(3), B, d, npdt)


@pytest.mark.parametrize('npdt', DTYPES)
def test_logqp_emulation_matches_kl_rate(npdt):
    """The emulation against `_kl_rate` (torch, CPU) on the GPU test's operands, the epsilon edge, +-0, subnormals, NaN
    and Inf included: the same non-finite rows, and within the float64 bound elsewhere (torch sums in another order).
    torch compares |g| > 1e-7 in the tensor's dtype, as the kernel does; at |g| = T(1e-7) both branches give g."""
    from torchsde_b200._core.base_sde import _kl_rate
    f, g, h = _logqp_operands(npdt)
    emu = ref.logqp_rate_emulated(f, g, h)
    tr = _kl_rate(*(torch.from_numpy(x) for x in (f, g, h)), True)[:, 0].numpy()
    assert tr.dtype == npdt
    assert np.array_equal(np.isnan(emu), np.isnan(tr)) and np.array_equal(np.isinf(emu), np.isinf(tr))
    fin = np.isfinite(emu)
    ex = ref.logqp_rate_exact(f, g, h)
    assert np.all(np.abs(tr[fin].astype(np.float64) - ex[fin]) <= ref.logqp_bound(ex[fin], f.shape[1], npdt))
    _, out = ref.logqp_violations(emu, f, g, h)
    assert not out.any()
    e = npdt(ref.LOGQP_EPS)
    edge = torch.from_numpy(np.array([e, np.nextafter(e, npdt(0)), np.nextafter(e, npdt(1))], dtype=npdt))
    assert (edge.abs() > 1e-7).tolist() == [False, False, True]


LOGQP_MISTAKES = ['>=', 'eps unrounded', 'sign(0) = 1', 'no 0.5', 'f + h']


@pytest.mark.parametrize('npdt', DTYPES)
@pytest.mark.parametrize('mistake', LOGQP_MISTAKES)
def test_logqp_checks_reject_mistakes(mistake, npdt):
    """Each mistake fails the GPU test's checks (bits, then the float64 bound) on >= 75 % of the rows it changes.
    `>=` for `>` changes nothing: at |g| = eps both branches give g.  Not rounding eps to T changes only the last
    bits of some fp32 rates (eps / T(eps) - 1 ~ 1e-8): only the bit comparison sees it, which is why it is there."""
    f, g, h = _logqp_operands(npdt, B=512, d=37)
    good = ref.logqp_rate_emulated(f, g, h)
    bad = ref.logqp_rate_emulated(f, g, h, mistake=mistake)
    uint = np.uint32 if npdt == np.float32 else np.uint64
    changed = good.view(uint) != bad.view(uint)
    changed &= ~(np.isnan(good) & np.isnan(bad))
    not_bits, out_of_bound = ref.logqp_violations(bad, f, g, h)
    if mistake == '>=':
        assert not changed.any()
        return
    if mistake == 'eps unrounded':
        if npdt == np.float64:
            assert not changed.any()   # T(1e-7) == 1e-7
            return
        _rejects(changed, not_bits, mistake)
        return
    _rejects(changed, out_of_bound, mistake)


# ---- the g.A product -----------------------------------------------------------------------------------------------
def _round(x, npdt):
    return np.ascontiguousarray(x).astype(npdt)


@pytest.mark.parametrize('npdt', DTYPES)
@pytest.mark.parametrize('m', [3, 8, 32])
def test_bmm_bound_rejects_mistakes(m, npdt):
    """The correctly rounded product passes; g.A^T, the output in (rows, d, m) order, a row given its neighbour's A
    and the last k term dropped each fail on >= 75 % of the elements they change (general and antisymmetric A)."""
    rng = np.random.default_rng(m)
    for anti in (False, True):
        B, d = 33, 7
        g = rng.standard_normal((B, d, m)).astype(npdt)
        a = rng.standard_normal((B, m, m))
        a = (a - a.transpose(0, 2, 1) if anti else a).astype(npdt)
        good = _round(ref.bmm_exact(g, a), npdt)
        assert not ref.bmm_violations(good, g, a).any()
        rows_d_m = _round(np.matmul(g.astype(np.float64), a.astype(np.float64)), npdt)
        mistakes = {
            'g A^T': _round(ref.bmm_exact(g, a.transpose(0, 2, 1)), npdt),
            '(rows, d, m) order': rows_d_m.reshape(m, B, d),
            "neighbour's A": _round(ref.bmm_exact(g, np.roll(a, 1, axis=0)), npdt),
            'last k dropped': _round(ref.bmm_exact(np.ascontiguousarray(g[..., :-1]),
                                                   np.ascontiguousarray(a[:, :-1, :])), npdt),
        }
        for what, got in mistakes.items():
            _rejects(got != good, ref.bmm_violations(got, g, a), f'{what} (anti={anti})')


# ---- the noise-free row-wise ops -----------------------------------------------------------------------------------
def _plain_inputs(npdt, n=4096):
    rng = np.random.default_rng(5)
    return [(rng.random((n // 16, 16)) + 0.5).astype(npdt) for _ in range(5)]


@pytest.mark.parametrize('npdt', DTYPES)
def test_plain_op_emulations_match_formulas(npdt):
    """The numpy emulation of each noise-free op (its written order in T) is within the GPU test's tolerance of the
    op's float64 formula."""
    x = _plain_inputs(npdt)
    for op in ip.PLAIN_OPS:
        emu = ip.plain_emulated(op, x)
        ref64 = op[5]([v.astype(np.float64) for v in x[:op[1]]], None, None)
        for e, r in zip(emu, ref64):
            np.testing.assert_allclose(e, r, **ip.tol_of(npdt), err_msg=ip._op_id(op))


@pytest.mark.parametrize('npdt', DTYPES)
def test_plain_op_checks_reject_mistakes(npdt):
    """ito branches swapped, stage-1 outputs swapped, stage-3 g0 / g1 coefficients swapped and the interpolation
    weights swapped each fail the formula check on >= 75 % of the elements they change."""
    x = _plain_inputs(npdt)
    ops = {ip._op_id(op): op for op in ip.PLAIN_OPS}
    T = npdt
    sq, dt = T(ip.SQ), T(ip.DT)

    def check(op, got, what):
        r = op[5]([v.astype(np.float64) for v in x[:op[1]]], None, None)
        for gi, ri, ei in zip(got, r, ip.plain_emulated(op, x)):
            _rejects(gi != ei, ~np.isclose(gi, ri, **ip.tol_of(npdt)), what)

    y0, f, g = x[0], x[1], x[2]
    check(ops['milstein_gf_predict'], [y0 + g * sq], 'ito ignored')
    check(ops['milstein_gf_predict_strat'], [(y0 + dt * f) + g * sq], 'ito applied to the Stratonovich branch')
    check(ops['srk_diag_stage1'], ip.plain_emulated(ops['srk_diag_stage1'], x)[::-1], 'stage-1 outputs swapped')
    y0, g0, g1, f2, g2 = x
    h1 = y0 + (T(2) * g1) * sq
    h1 = h1 + (T(-1) * g0) * sq
    check(ops['srk_diag_stage3'], [(h1 + (T(0.25) * f2) * dt) + (T(0.5) * g2) * sq], 'stage-3 g0 / g1 swapped')
    lerp = ops['linear_interp_0.3_0.7']
    check(lerp, [T(lerp[4][1]) * x[0] + T(lerp[4][0]) * x[1]], 'interpolation weights swapped')


class _Recording:
    """numpy SDE for the oracle that logs every (t, y) it is evaluated at."""
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self):
        self.f_at, self.g_at = [], []

    def f(self, t, y):
        self.f_at.append(y.copy())
        return (np.sin(y) + 0.3 * y).astype(y.dtype)

    def g(self, t, y):
        self.g_at.append(y.copy())
        return (0.5 + 0.2 * np.cos(y)).astype(y.dtype)


def test_plain_op_formulas_match_oracle():
    """The float64 formulas of tsde_srk_diag_stage1 / stage3 are the oracle SRK's stage values H0 / H1, and that of
    tsde_milstein_gf_predict (both branches) is the gradient-free Milstein predictor's y0'."""
    rng = np.random.default_rng(9)
    B, d = 6, 5
    y0 = rng.random((B, d)) + 0.5
    W, U = rng.standard_normal((B, d)) * ip.SQ, rng.standard_normal((B, d)) * ip.DT
    ops = {ip._op_id(op): op for op in ip.PLAIN_OPS}
    tol = dict(rtol=1e-14, atol=1e-15)

    sde = _Recording()
    solvers.make('srk', sde, lambda ta, tb, return_U=False: (W, U) if return_U else W, ip.DT).step(
        np.float64(0.0), np.float64(ip.DT), y0, ())
    # stage s evaluates f at H0_j and g at H1_j for j < s, then f at H0_s and g at H1_s: calls 0, 2, 5 and 9 are the
    # stage values H_0 = y0, H_1, H_2, H_3
    H0, H1 = [sde.f_at[i] for i in (0, 2, 5, 9)], [sde.g_at[i] for i in (0, 2, 5, 9)]
    f0, g0 = sde.f(0, y0), sde.g(0, y0)
    h0_1, h1_1 = ops['srk_diag_stage1'][5]([y0, f0, g0], None, None)
    np.testing.assert_allclose(h0_1, H0[1], **tol)
    np.testing.assert_allclose(h1_1, H1[1], **tol)
    g1, f2, g2 = sde.g(0, H1[1]), sde.f(0, H0[2]), sde.g(0, H1[2])
    h1_3, = ops['srk_diag_stage3'][5]([y0, g0, g1, f2, g2], None, None)
    np.testing.assert_allclose(h1_3, H1[3], **tol)

    for ito, name in ((True, 'milstein_gf_predict'), (False, 'milstein_gf_predict_strat')):
        sde = _Recording()
        sde.sde_type = 'ito' if ito else 'stratonovich'
        solvers.make('milstein', sde, lambda ta, tb, return_U=False: W, ip.DT, {'grad_free': True}).step(
            np.float64(0.0), np.float64(ip.DT), y0, ())
        yp, = ops[name][5]([y0, sde.f(0, y0), sde.g(0, y0)], None, None)
        np.testing.assert_allclose(yp, sde.g_at[1], **tol)


# ---- log-ODE -------------------------------------------------------------------------------------------------------
def _replay(case, area=lambda A: A):
    """ys of float64 log-ODE steps on a golden's increments and Levy areas (each area passed through `area`)."""
    sde = helpers.build_problem(case)
    y = torch.from_numpy(case['y0'])
    got = [y]
    for ta, tb, W, A in zip(case['ta'], case['tb'], case['W'], case['A']):
        y = ref.log_ode_step(sde, ta, tb - ta, y, torch.from_numpy(W), area(torch.from_numpy(A)))
        if np.any(np.isclose(tb, case['ts'][1:], rtol=0, atol=1e-12)):
            got.append(y)
    assert len(got) == len(case['ts'])
    return torch.stack(got).numpy()


WRONG_AREAS = {'A^T': lambda A: A.transpose(-1, -2), '-A': lambda A: -A}


@pytest.mark.parametrize('path', helpers.golden_files('logode_general'), ids=helpers.case_id)
def test_log_ode_restatement_replays_goldens(path):
    """One float64 log-ODE step at a time (g(y') A, the column-l tangent for column l of g) on the reference's
    increments and Levy areas reproduces the reference's ys.  On the m = 2 ... 32 goldens (TanhMixedGeneral) the
    area term is non-zero and odd in A, so this pins which way round the step takes A; on the older m = 3, 4 goldens
    (TanhGeneral, whose area term vanishes for antisymmetric A) it pins only the rest of the step."""
    case = helpers.load(path)
    np.testing.assert_allclose(_replay(case), case['ys'], rtol=1e-11, atol=1e-13)


@pytest.mark.parametrize('wrong', sorted(WRONG_AREAS))
@pytest.mark.parametrize('path', helpers.golden_files('logode_general_m'), ids=helpers.case_id)
def test_log_ode_goldens_reject_wrong_area_orientation(path, wrong):
    """A step that takes A the wrong way round (A^T, or -A: the same for an antisymmetric area) fails the golden
    replay's fp64 tolerance and the fp32 tolerance of the fp32 replay on >= 75 % of the solution's elements."""
    case = helpers.load(path)
    got = _replay(case, WRONG_AREAS[wrong])[1:]
    ys = case['ys'][1:]
    changed = np.ones(ys.shape, bool)
    _rejects(changed, ~np.isclose(got, ys, rtol=1e-11, atol=1e-13), f'{wrong} vs the fp64 golden')
    _rejects(changed, ~np.isclose(got, ys, **helpers.tol_for('f32', False)), f'{wrong} vs the fp32 tolerance')


@pytest.mark.parametrize('m', [2, 5, 8, 16, 32])
def test_log_ode_route_case_sees_wrong_area_orientation(m):
    """On the solve the GPU route test compares no-grad against grad-tracked, the same steps with -A (= A^T) differ
    from those with A beyond the fp32 tolerance on >= 75 % of the elements: a step that took the product the wrong way
    round on one path only would fail that comparison."""
    sde, y0, tas, Ws, As = ref.log_ode_route_case(m, torch.float64)
    ys = {}
    for sign in (1, -1):
        y = y0
        for ta, W, A in zip(tas, Ws, As):
            y = ref.log_ode_step(sde, ta, ref.LOG_ODE_DT, y, W, sign * A)
        ys[sign] = y.numpy()
    _rejects(np.ones(ys[1].shape, bool), ~np.isclose(ys[-1], ys[1], **helpers.tol_for('f32', False)), '-A')


# ---- library validation --------------------------------------------------------------------------------------------
def _lib_or_skip():
    try:
        return _cabi.lib()
    except _cabi.LibraryNotBuilt:
        pytest.skip('CUDA library not built')


@pytest.mark.parametrize('dtype', [_cabi.F32, _cabi.F64])
def test_launch_validation(dtype):
    lib = _lib_or_skip()
    p = ctypes.c_void_p(256)
    for noise in (_cabi.NOISE_DIAGONAL, 2, -1):   # diagonal, and values no noise type has
        L = _cabi.Launch(dtype, noise, 4, 8, 8, None)
        assert lib.tsde_bmm_ga(ctypes.byref(L), p, p, p) == _cabi.EINVAL
    L = _cabi.Launch(dtype, _cabi.NOISE_DIAGONAL, 4, (1 << 24) + 1, (1 << 24) + 1, None)
    assert lib.tsde_logqp_augment(ctypes.byref(L), p, p, p, 1e-7, p, p) == _cabi.EINVAL
