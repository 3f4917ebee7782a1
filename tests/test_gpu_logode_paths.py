"""The log-ODE product `tsde_bmm_ga` and the diagonal-noise KL rate `tsde_logqp_augment` against float64 (or wider)
restatements of their formulas (tests/logode_ref.py), and log-ODE solves on every route of the product:

* tsde_bmm_ga on every route bmm_ga_impl (csrc/logode.cu) takes: the tile kernel at each compiled m, over d on both
  sides of 32 and 256 (one row per CTA from there on), with one row and with a partial last CTA, rows per CTA set by
  256 / d or by the 32 KiB shared-memory cap; the generic kernel at other m, for unaligned operands at m % 4 == 0 and
  past d = 2^20; B = 0.  Every element is within gamma_m sum_k |g_k||A_kl| of the exact product, every launch runs
  the kernel the route rule predicts (torch.profiler), and the generic kernel gives the tile kernel's bits;
* tsde_logqp_augment (diagonal noise): the rate bit for bit against a numpy emulation of the kernel's operations,
  within (ceil(d/32) + 8) u sum u^2 of float64, at the epsilon guard's edge, on +-0, subnormal, NaN and Inf operands
  and through the grid-stride row loop; f and g copied bit for bit, a +0 written in g's extra column;
* log-ODE solves (general noise, m = 2, 5, 8, 16, 32) through tsde_bmm_ga agree with the grad-tracked solve, which
  forms the product with torch.bmm, and fp32 solves on the reference's goldens at those m agree with its fp64 solve.
  Their problem's Levy-area term changes sign with A, so both would see the product taken the wrong way round.

Outputs are prefilled with NaN and guarded by sentinels on both sides."""
import ctypes

import numpy as np
import pytest
import torch

from . import helpers, logode_ref as ref, problems

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SENT = 4                       # sentinel elements on each side of an output (keeps it 16-byte aligned)
LO, HI = -7.25, 7.25           # the sentinel values
DTYPES = [torch.float32, torch.float64]
NP = {torch.float32: np.float32, torch.float64: np.float64}
TORCH = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}
TAG = {torch.float32: 'float', torch.float64: 'double'}


def _cabi():
    from torchsde_b200 import _cabi
    return _cabi


def _guarded(n, dtype):
    buf = torch.full((n + 2 * SENT,), float('nan'), dtype=dtype, device=DEV)
    buf[:SENT], buf[-SENT:] = LO, HI
    return buf


def _body(buf):
    """(body as numpy, whether both sentinel runs are intact)."""
    h = buf.cpu().numpy()
    return h[SENT:len(h) - SENT], bool(np.all(h[:SENT] == LO) and np.all(h[len(h) - SENT:] == HI))


def _on_device(x, misalign):
    """x's values on the device, 16-byte aligned or one element past that; returns (buffer, address)."""
    dtype = TORCH[x.dtype]
    buf = torch.empty(x.size + 1, dtype=dtype, device=DEV)
    view = buf[1:] if misalign else buf[:x.size]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(-1)))
    return buf, view.data_ptr()


def _bmm_kernels(fn):
    """Names of the tsde_bmm_ga kernels `fn` launches, in launch order.  (A device op and a synchronisation come first,
    so the trace is running before the first launch.)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device=DEV).add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'bmm_ga' in e.name]
    return [e.name for e in sorted(evs, key=lambda e: e.time_range.start)]


WORST = {}


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print(f'worst err/bound {key}: {WORST[key]:.3g}')


# ---- tsde_bmm_ga ---------------------------------------------------------------------------------------------------
def _bmm_launch(g, a, misalign_g=False, misalign_a=False, rows=None):
    """One tsde_bmm_ga call; returns (code, guarded output buffer)."""
    c = _cabi()
    rows = g.shape[0] if rows is None else rows
    _, d, m = g.shape
    dtype = TORCH[g.dtype]
    gb, gp = _on_device(g, misalign_g)
    ab, ap = _on_device(a, misalign_a)
    out = _guarded(rows * d * m, dtype)
    L = c.make_launch(dtype, c.NOISE_GENERAL, rows, d, m)
    code = c.lib().tsde_bmm_ga(ctypes.byref(L), gp, ap, out.data_ptr() + SENT * g.itemsize)
    del gb, ab
    return code, out


# the shapes (B, d, m) of the torch.bmm comparison this file replaces
OLD_BMM_SHAPES = [(8192, 32, 16), (257, 5, 3), (64, 7, 8), (33, 4, 2), (100, 40, 32), (50, 6, 5), (3, 2, 20)]


BMM_GROUPS = [str(m) for m in ref.TILE_M] + ['generic', 'unaligned', 'old']
TRACE_ATTEMPTS = 5   # traces of the same launches taken before a short one counts as a missing kernel


def _bmm_cases(dtype, group):
    """(B, d, m, antisymmetric, scaled, misalign_g, misalign_a) of one group of routing cases: one tile m over d, the
    generic kernel's m, operands off alignment, or the shapes of the torch.bmm comparison this file replaces."""
    es = torch.finfo(dtype).bits // 8
    cases = []
    if group == 'generic':
        for m in (1, 5, 7, 12, 33, 64, 100):
            for d, B in ((1, 37), (3, 1), (33, 5), (257, 3)):
                cases.append((B, d, m, m % 2 == 0, True, False, False))
    elif group == 'unaligned':
        for m in (2, 3, 4, 8, 16, 32):
            for d, B in ((5, 57), (64, 9)):
                cases.append((B, d, m, True, True, True, False))
                cases.append((B, d, m, False, True, False, True))
    elif group == 'old':
        for B, d, m in OLD_BMM_SHAPES:
            for anti in (False, True):
                cases.append((B, d, m, anti, False, False, False))
    else:
        m = int(group)
        for d in (1, 3, 32, 33, 255, 256, 257, 1000):
            rpc = ref.bmm_route(m, d, es)[1]
            for B in (1, 2 * rpc + 1):
                for anti in (False, True):
                    cases.append((B, d, m, anti, True, False, False))
    return cases


@pytest.mark.parametrize('group', BMM_GROUPS)
@pytest.mark.parametrize('dtype', DTYPES)
def test_bmm_ga_routes_vs_exact(dtype, group):
    """Every case within gamma_m sum_k |g_k||A_kl| (+ m eta) of the exact product, on the kernel the route rule
    predicts; the unaligned cases also give the bits of the same operands aligned (the tile kernel: both kernels run
    the k-ascending fma chain from 0)."""
    npdt, es = NP[dtype], torch.finfo(dtype).bits // 8
    rng = np.random.default_rng(20261016)
    cases = _bmm_cases(dtype, group)
    if group == '32' or (group == '16' and dtype == torch.float64):
        # the 32 KiB cap, not 256 / d, sets rows per CTA at small d
        assert any(ref.bmm_route(m, d, es)[1] < -(-256 // d) for _, d, m, *_ in cases)
    operands = [ref.bmm_operands(rng, B, d, m, npdt, anti) if scaled else
                (rng.standard_normal((B, d, m)).astype(npdt), _plain_a(rng, B, m, npdt, anti))
                for B, d, m, anti, scaled, _, _ in cases]
    results = []

    def run():
        results.clear()
        for (B, d, m, anti, scaled, mg, ma), (g, a) in zip(cases, operands):
            results.append(_bmm_launch(g, a, mg, ma))
            if mg or ma:
                results.append(_bmm_launch(g, a))
    expect = []
    for B, d, m, anti, scaled, mg, ma in cases:
        expect.append(ref.bmm_route(m, d, es, not mg, not ma)[0])
        if mg or ma:
            expect.append(ref.bmm_route(m, d, es)[0])
    names = _bmm_kernels(run)
    codes = [code for code, _ in results]
    assert codes == [0] * len(expect), codes
    counts = [len(names)]
    while len(names) != len(expect) and len(counts) < TRACE_ATTEMPTS:
        # every launch returned 0, but the trace holds fewer kernel records than launches (the profiler now and then
        # loses a few records of a busy process, and can lose them in consecutive traces): capture the same launches
        # again (their outputs are checked below either way)
        names = _bmm_kernels(run)
        counts.append(len(names))
        assert [code for code, _ in results] == [0] * len(expect)
    assert len(names) == len(expect), f'{len(expect)} launches; kernel records per trace: {counts}'
    wrong = [(i, n, e) for i, (n, e) in enumerate(zip(names, expect)) if ref.bmm_kernel_name(e, TAG[dtype]) not in n]
    assert not wrong, wrong[:5]
    bad, it = [], iter(results)
    for (B, d, m, anti, scaled, mg, ma), (g, a) in zip(cases, operands):
        code, out = next(it)
        body, sent = _body(out)
        got = body.reshape(m, B, d)
        tag = (B, d, m, 'anti' if anti else 'gen', 'g+1' if mg else ('A+1' if ma else ''))
        if code != 0 or not sent or np.isnan(got).any():
            bad.append(f'{tag}: code {code}, sentinels {sent}, unwritten {int(np.isnan(got).sum())}')
            continue
        viol = ref.bmm_violations(got, g, a)
        if viol.any():
            bad.append(f'{tag}: {int(viol.sum())} of {viol.size} elements outside the bound')
        err = ref.bmm_error(got, g, a)
        _note(('bmm_ga', ref.bmm_route(m, d, es, not mg, not ma)[0], TAG[dtype]), np.max(err / ref.bmm_bound(g, a)))
        if mg or ma:
            _, aligned = next(it)
            if not torch.equal(out.view(torch.int64 if es == 8 else torch.int32),
                               aligned.view(torch.int64 if es == 8 else torch.int32)):
                bad.append(f'{tag}: unaligned (generic kernel) != aligned (tile kernel) bits')
    assert not bad, '\n'.join(bad[:20])


def _plain_a(rng, B, m, npdt, anti):
    a = rng.standard_normal((B, m, m))
    return (a - a.transpose(0, 2, 1) if anti else a).astype(npdt)


@pytest.mark.parametrize('dtype', DTYPES)
def test_bmm_ga_tile_limit_and_empty_batch(dtype):
    """d = 2^20 takes the tile kernel, d = 2^20 + 1 the generic one (m = 4); on the first 2^20 channels they give the
    same bits, and both are within the bound.  B = 0 returns 0 and writes nothing, on a tile shape (m = 4, d = 32) and
    on the generic one."""
    npdt, es = NP[dtype], torch.finfo(dtype).bits // 8
    rng = np.random.default_rng(7)
    big = ref.TILE_MAX_D
    g = rng.standard_normal((1, big + 1, 4)).astype(npdt)
    a = _plain_a(rng, 1, 4, npdt, True)
    res = []
    names = _bmm_kernels(lambda: res.extend([_bmm_launch(np.ascontiguousarray(g[:, :big]), a), _bmm_launch(g, a)]))
    assert [ref.bmm_route(4, big, es)[0], ref.bmm_route(4, big + 1, es)[0]] == ['tile', 'generic']
    assert len(names) == 2 and ref.bmm_kernel_name('tile', TAG[dtype]) in names[0] \
        and ref.bmm_kernel_name('generic', TAG[dtype]) in names[1], names
    (c0, o0), (c1, o1) = res
    b0, s0 = _body(o0)
    b1, s1 = _body(o1)
    assert c0 == 0 and c1 == 0 and s0 and s1
    t0, t1 = b0.reshape(4, 1, big), b1.reshape(4, 1, big + 1)
    assert np.array_equal(t0.view(np.uint8), np.ascontiguousarray(t1[:, :, :big]).view(np.uint8))
    assert not ref.bmm_violations(t1, g, a).any()
    # (the library returns before choosing a route when B = 0: a tile shape and a generic one)
    for gz, az in ((np.zeros((0, 32, 4), npdt), np.zeros((0, 4, 4), npdt)), (g[:0], a[:0])):
        code, out = _bmm_launch(gz, az, rows=0)
        body, sent = _body(out)
        assert code == 0 and sent and body.size == 0


# ---- tsde_logqp_augment, diagonal noise ------------------------------------------------------------------------------
def _special_triples(npdt):
    """(f, g, h) triples at the edges of the kernel's guard and arithmetic."""
    T = npdt
    eps = T(ref.LOGQP_EPS)
    below, above = np.nextafter(eps, T(0)), np.nextafter(eps, T(1))
    tiny = np.finfo(npdt).smallest_subnormal
    sub = T(1e-40) if npdt == np.float32 else T(1e-310)
    nan_payload = (np.array([0x7fc00123], np.uint32).view(np.float32)[0] if npdt == np.float32 else
                   np.array([0x7ff8000000000123], np.uint64).view(np.float64)[0])
    inf = T(np.inf)
    out = []
    for gv in (eps, below, above, -eps, -below, -above):
        out += [(T(1.5), gv, T(0.25)), (T(3e-7), gv, T(-1e-7))]
    for gv in (T(0.0), T(-0.0)):
        out += [(T(0.5), gv, T(0.5)), (T(0.5), gv, T(-0.25)), (T(-0.0), gv, T(0.0))]
    for gv in (tiny, -tiny, sub, -sub):
        out += [(T(2.0), gv, T(1.0)), (T(1e-30), gv, T(0.0))]
    out += [(T(1.0), tiny, T(1.0))]
    for x in (nan_payload, inf, -inf):
        out += [(x, T(0.3), T(0.1)), (T(0.2), x, T(0.1)), (T(0.2), T(0.3), x)]
    out += [(T(1e-20), T(0.7), T(0.0)), (T(3e18 if npdt == np.float32 else 3e150), T(1e-3), T(0.0))]
    return out


def _logqp_inputs(rng, B, d, npdt):
    f = rng.standard_normal((B, d)).astype(npdt)
    h = rng.standard_normal((B, d)).astype(npdt)
    g = (rng.standard_normal((B, d)) * np.exp2(rng.integers(-30, 4, size=(B, d)))).astype(npdt)
    for i, (fv, gv, hv) in enumerate(_special_triples(npdt)):
        k = (i * 37 + i // 3) % (B * d)
        f.flat[k], g.flat[k], h.flat[k] = fv, gv, hv
    return f, g, h


# the shapes (B, d) of the torch comparison this file replaces
OLD_LOGQP_SHAPES = [(1000, 7), (33, 1), (4096, 128), (5, 200)]


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('d', [1, 31, 32, 33, 64, 1000, 'old'])
def test_logqp_diagonal_vs_emulation(d, dtype):
    """f_aug[:, d] equals the emulation bit for bit (NaN where it is NaN) and is within the float64 bound; f_aug[:, :d]
    and g_aug[:, :d] are bit copies of f and g (NaN payloads included), g_aug[:, d] is +0.0.  B = 1 and
    B = 3 (sm_count 64) + 5: more rows than the capped grid (sm_count x 8 CTAs of 8 warps) has warps."""
    c = _cabi()
    npdt = NP[dtype]
    uint = np.uint32 if dtype == torch.float32 else np.uint64
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    shapes = OLD_LOGQP_SHAPES if d == 'old' else [(1, d), (3 * sms * 64 + 5, d)]
    rng = np.random.default_rng(99)
    bad = []
    for B, dd in shapes:
        f, g, h = _logqp_inputs(rng, B, dd, npdt)
        ft, gt, ht = (torch.from_numpy(x).to(DEV) for x in (f, g, h))
        fa, ga = _guarded(B * (dd + 1), dtype), _guarded(B * (dd + 1), dtype)
        es = g.itemsize
        L = c.make_launch(dtype, c.NOISE_DIAGONAL, B, dd, dd)
        code = c.lib().tsde_logqp_augment(ctypes.byref(L), ft.data_ptr(), gt.data_ptr(), ht.data_ptr(), ref.LOGQP_EPS,
                                          fa.data_ptr() + SENT * es, ga.data_ptr() + SENT * es)
        fb, fs = _body(fa)
        gb, gs = _body(ga)
        tag = (B, dd)
        if code != 0 or not fs or not gs:
            bad.append(f'{tag}: code {code}, sentinels {fs}, {gs}')
            continue
        fb, gb = fb.reshape(B, dd + 1), gb.reshape(B, dd + 1)
        if not np.array_equal(fb[:, :dd].view(uint), f.view(uint)):
            bad.append(f'{tag}: f_aug[:, :d] is not a bit copy of f')
        if not np.array_equal(gb[:, :dd].view(uint), g.view(uint)):
            bad.append(f'{tag}: g_aug[:, :d] is not a bit copy of g')
        if not np.all(gb[:, dd].view(uint) == 0):
            bad.append(f'{tag}: g_aug[:, d] is not +0.0')
        got = np.ascontiguousarray(fb[:, dd])
        not_bits, out_of_bound = ref.logqp_violations(got, f, g, h)
        if not_bits.any():
            r = int(np.flatnonzero(not_bits)[0])
            bad.append(f'{tag}: {int(not_bits.sum())} rates differ from the emulation (row {r}: {got[r]!r} vs '
                       f'{ref.logqp_rate_emulated(f[r:r + 1], g[r:r + 1], h[r:r + 1])[0]!r})')
        if out_of_bound.any():
            bad.append(f'{tag}: {int(out_of_bound.sum())} rates outside the float64 bound')
        ex = ref.logqp_rate_exact(f, g, h)
        fin = np.isfinite(got) & np.isfinite(ex) & (ex > 0)
        if fin.any():
            _note(('logqp_augment', TAG[dtype]),
                  np.max(np.abs(got[fin].astype(np.float64) - ex[fin]) / ref.logqp_bound(ex[fin], dd, npdt)))
    assert not bad, '\n'.join(bad)


# ---- log-ODE solves ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('m', [2, 5, 8, 16, 32])
def test_log_ode_solve_routes(m, dtype):
    """The no-grad log-ODE solve forms g.A with tsde_bmm_ga on the kernel the route rule predicts, once per step, and
    agrees with the same solve with y0.requires_grad_(), which forms it with torch.bmm inside autograd.  The problem's
    Levy-area term changes sign with A: the same solve on the negated areas (-A = A^T, the product taken the wrong way
    round) must differ beyond that tolerance, so the comparison sees such a slip."""
    import torchsde_b200 as tsde
    es = torch.finfo(dtype).bits // 8
    route, rpc = ref.bmm_route(m, ref.LOG_ODE_D, es)
    assert route == 'generic' or (ref.LOG_ODE_B > rpc and ref.LOG_ODE_B % rpc), (route, rpc)
    sde, y0, tas, Ws, As = ref.log_ode_route_case(m, dtype)
    sde, y0 = sde.to(DEV), y0.to(DEV)
    Ws, As = [w.to(DEV) for w in Ws], [a.to(DEV) for a in As]
    ts = torch.tensor(ref.LOG_ODE_TS, dtype=dtype, device=DEV)
    dt = ref.LOG_ODE_DT

    def solve(areas, **kw):
        bm = problems.ReplayBM(tas, tas + dt, Ws, None, levy='foster', As=areas)
        return tsde.sdeint(sde, y0, ts, bm=bm, method='log_ode', dt=dt, **kw)
    out = []

    def no_grad():
        with torch.no_grad():
            out.append(solve(As))
    names = _bmm_kernels(no_grad)
    assert len(names) == len(tas) and all(ref.bmm_kernel_name(route, TAG[dtype]) in n for n in names), names
    tol = helpers.tol_for('f64' if dtype == torch.float64 else 'f32', False)
    bm = problems.ReplayBM(tas, tas + dt, Ws, None, levy='foster', As=As)
    ys_grad = tsde.sdeint(sde, y0.clone().requires_grad_(), ts, bm=bm, method='log_ode', dt=dt)
    got = out[0].cpu().numpy()
    np.testing.assert_allclose(got, ys_grad.detach().cpu().numpy(), **tol)
    with torch.no_grad():
        flipped = solve([-a for a in As]).cpu().numpy()
    assert np.mean(~np.isclose(flipped[1:], got[1:], **tol)) >= 0.75


@pytest.mark.parametrize('path', helpers.golden_files('logode_general_m'), ids=helpers.case_id)
def test_log_ode_golden_fp32(path):
    """An fp32 log-ODE solve on the reference's increments and Levy areas agrees with the reference's fp64 solve (the
    problem's area term is odd in A: the CPU tests show a step taking A^T would miss this tolerance)."""
    import torchsde_b200 as tsde
    case = helpers.load(path)
    f32 = torch.float32
    sde = helpers.build_problem(case, dtype=f32, device=DEV)
    conv = [[torch.from_numpy(x).to(DEV, f32) for x in case[k]] for k in ('W', 'U', 'A')]
    bm = problems.ReplayBM(case['ta'], case['tb'], conv[0], conv[1], levy=str(case['levy']), As=conv[2])
    y0 = torch.from_numpy(case['y0']).to(DEV, f32)
    ts = torch.from_numpy(case['ts']).to(DEV, f32)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='log_ode', dt=float(case['dt']))
    np.testing.assert_allclose(ys.cpu().numpy(), case['ys'], **helpers.tol_for('f32', False))
