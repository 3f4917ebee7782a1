"""SDEs whose drift / diffusion return bfloat16 or float16 (torch.autocast), with a float32 state.

The contract: a solve whose SDE outputs are 16-bit is bit-identical to the same solve with every such output widened
by `.float()` (widening is exact, and the kernels run the float32 arithmetic on the widened values).  Checked at the C
ABI on every kernel route, then through `sdeint` / `sdeint_adjoint`, their gradients and the host-side fallbacks."""
import ctypes

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from . import helpers
from . import problems

pytestmark = pytest.mark.gpu

dev = torch.device('cuda')
HALF = (torch.bfloat16, torch.float16)
DT = 2.0 ** -6
SENTINEL = 16  # guard elements on each side of every output


# ---- entry points ----------------------------------------------------------------------------------------------------
# name -> (scalars, noise: None | 'w' | 'wu', outputs as input-name-like shape tags, row-wise only)
ENTRIES = {
    'tsde_step_euler': ((DT,), 'w', ('y',), False),
    'tsde_milstein_vjp_seed': ((DT, 1), 'w', ('g',), True),
    'tsde_step_milstein': ((DT,), 'w', ('y',), True),
    'tsde_milstein_gf_predict': ((DT, DT ** 0.5, 1), None, ('y',), True),
    'tsde_step_milstein_gf': ((DT, 2 * DT ** 0.5, 1), 'w', ('y',), True),
    'tsde_step_heun': ((DT,), 'w', ('y',), False),
    'tsde_midpoint_predict': ((DT / 2,), 'w', ('y',), False),
    'tsde_euler_heun_predict': ((), 'w', ('y',), False),
    'tsde_step_euler_heun': ((DT,), 'w', ('y',), False),
    'tsde_reversible_heun_z': ((DT,), 'w', ('y',), False),
    'tsde_step_reversible_heun': ((DT / 2,), 'w', ('y',), False),
    'tsde_srk_diag_stage1': ((DT, DT ** 0.5), None, ('y', 'y'), True),
    'tsde_srk_diag_stage2': ((DT, 1 / DT, DT ** 0.5), 'wu', ('y', 'y'), True),
    'tsde_srk_diag_stage3': ((DT, DT ** 0.5), None, ('y',), True),
    'tsde_step_srk_diag': ((DT, 1 / DT, DT ** 0.5, 3 * DT), 'wu', ('y',), True),
    'tsde_srk_additive_stage': ((DT, 1 / DT), 'wu', ('y',), False),
    'tsde_step_srk_additive': ((DT, 1 / DT), 'wu', ('y',), False),
    'tsde_adjoint_reversible_heun_a': ((DT, DT / 2), 'w', ('y', 'y', 'g'), False),
    'tsde_adjoint_reversible_heun_b': ((DT, DT / 2), 'w', ('y', 'y', 'y', 'y', 'g'), False),
}
GENERAL_ONLY = ('tsde_srk_additive_stage', 'tsde_step_srk_additive')
# (label, noise layout, rows, d, m): row-wise fast kernel at chunk edges, row-wise generic kernel, the per-thread-load
# tile kernel (m/4 a power of two), the generic tile kernel, scalar noise
ROWWISE_SHAPES = [('fast', 'diag', 513, 4, 4), ('fast', 'diag', 171, 12, 12), ('fast', 'diag', 16, 64, 64),
                  ('fast', 'diag', 1, 4, 4), ('generic', 'diag', 37, 6, 6), ('scalar', 'general', 77, 8, 1)]
GENERAL_SHAPES = [('cta', 'general', 67, 8, m) for m in (4, 8, 16, 32, 64, 128)] + \
                 [('generic', 'general', 53, 6, m) for m in (3, 5, 40)]


def _is_g(arg):
    return arg.startswith('g') and arg != 'gdg' or arg == 'adj_g0'


def _guarded(shape, dtype, misalign=0):
    """An uninitialised-looking tensor of `shape` with SENTINEL guard elements on both sides (optionally shifted by
    `misalign` elements, to move it off 16-byte alignment).  Returns (buffer, view)."""
    n = int(torch.Size(shape).numel())
    buf = torch.full((n + 2 * SENTINEL + misalign,), -7.25, dtype=dtype, device=dev)
    return buf, buf[SENTINEL + misalign:SENTINEL + misalign + n].view(shape)


def _guards_intact(buf, n, misalign=0):
    lo, hi = buf[:SENTINEL + misalign], buf[SENTINEL + misalign + n:]
    return bool((lo == -7.25).all()) and bool((hi == -7.25).all())


def _call(name, noise, rows, d, m, ins, outs, word, nz, bcast):
    L = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL if noise == 'diag' else _cabi.NOISE_GENERAL, rows, d, m)
    L.dtype = word
    args = [ctypes.byref(L)] + ([ctypes.byref(nz)] if ENTRIES[name][1] else [])
    return getattr(_cabi.lib(), name)(*args, *[t.data_ptr() for t in ins], *ENTRIES[name][0],
                                      *[o.data_ptr() for o in outs])


def _run_pair(name, half, src, shape, bcast=False, misalign=0):
    """Launch `name` with its SDE outputs in `half` and once with widened float32 copies; both results, guarded."""
    _, noise, rows, d, m = shape
    scalars, want, out_kinds, _ = ENTRIES[name]
    gshape = (d, m) if bcast else ((rows, d) if (noise == 'diag' or m == 1) else (rows, d, m))
    gen = torch.Generator(device=dev).manual_seed(rows * 131 + d * 7 + m)
    ins16, ins32, word = [], [], _cabi.F32
    for i, arg in enumerate(_cabi.INPUTS[name]):
        shp = gshape if _is_g(arg) else (rows, d)
        x = torch.randn(shp, generator=gen, device=dev)
        if arg in _cabi.SDE_OUTPUT_NAMES:
            _, x16 = _guarded(shp, half, misalign)
            x16.copy_(x.to(half))
            ins16.append(x16)
            # the float32 copy shifted by as many elements: a 2-byte-aligned 16-bit operand takes the generic kernel,
            # and so does its 4-byte-aligned copy (the generic tile kernel sums in another order than the tile kernel)
            _, x32 = _guarded(shp, torch.float32, misalign)
            x32.copy_(x16.float())
            ins32.append(x32)
            word |= (_cabi.FMT_BF16 if half == torch.bfloat16 else _cabi.FMT_F16) << (8 + 2 * i)
        else:
            ins16.append(x)
            ins32.append(x)
    key = torch.tensor([20261016], dtype=torch.int64, device=dev)
    w = torch.randn(rows, m, generator=gen, device=dev) * DT ** 0.5
    u = torch.randn(rows, m, generator=gen, device=dev) * DT
    nz = None
    if want:
        nz = helpers.general_noise(key=key, cell_id=5) if src == 'counter' else \
            helpers.general_noise(w=w.data_ptr(), u=u.data_ptr(), want_u=want == 'wu')
        nz.want_u = int(want == 'wu')
        nz.flags = _cabi.FLAG_G_BROADCAST if bcast else 0
    res = []
    for ins, wd in ((ins16, word), (ins32, _cabi.F32)):
        bufs, outs = [], []
        for kind in out_kinds:
            shp = (rows, d, m) if (kind == 'g' and noise == 'general' and m > 1) else (rows, d)
            odt = ins[0].dtype if name == 'tsde_milstein_vjp_seed' else torch.float32
            buf, o = _guarded(shp, odt)
            bufs.append((buf, o.numel()))
            outs.append(o)
        assert _call(name, noise, rows, d, m, ins, outs, wd, nz, bcast) == 0, name
        torch.cuda.synchronize()
        assert all(_guards_intact(b, n) for b, n in bufs), f"{name}: write outside an output"
        res.append(outs)
    return res


def _assert_pair(res, what):
    for a, b in zip(*res):
        if a.dtype != b.dtype:  # Milstein's go, written in g's format: the float32 result rounded to nearest even
            assert what[0] == 'tsde_milstein_vjp_seed' and a.dtype in HALF, what
            b = b.to(a.dtype)
        assert torch.equal(a, b), what


@pytest.mark.parametrize('src', ['counter', 'memory'])
@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name', list(ENTRIES))
def test_entry_point_equals_widened_launch(name, half, src):
    rowwise_only = ENTRIES[name][3]
    shapes = [] if name in GENERAL_ONLY else list(ROWWISE_SHAPES)
    if not rowwise_only:
        shapes += GENERAL_SHAPES
    for shape in shapes:
        if name in GENERAL_ONLY and shape[4] == 1:
            continue
        _assert_pair(_run_pair(name, half, src, shape), (name, shape))
    if name not in GENERAL_ONLY:
        # 16-bit operands 8-byte but not 16-byte aligned (the fast row-wise kernel), and 2-byte aligned (generic)
        for misalign in (4, 1):
            _assert_pair(_run_pair(name, half, src, ROWWISE_SHAPES[0], misalign=misalign), (name, misalign))
    if not rowwise_only:
        # a 16-bit g 8-byte aligned stays on the per-thread-load tile kernel, a 2-byte aligned one takes gen_kernel
        for misalign, cta in ((4, 2), (1, 0)):
            before = helpers.tile_launches()[0]
            _assert_pair(_run_pair(name, half, src, GENERAL_SHAPES[1], misalign=misalign), (name, 'tile', misalign))
            assert helpers.tile_launches()[0] - before == cta, (name, misalign)


def _kernels_of(fn):
    """Names of the CUDA kernels `fn` launches (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize('name', ['tsde_step_milstein', 'tsde_milstein_vjp_seed', 'tsde_step_reversible_heun'])
def test_rowwise_route_follows_16bit_alignment(name):
    """16-bit operands need 8-byte alignment for the fast row-wise kernel (float32 ones 16): 16- and 8-byte aligned
    take `ew_fast_kernel`, 2-byte aligned the generic `ew_kernel`."""
    for misalign, kernel in ((0, 'ew_fast_kernel'), (4, 'ew_fast_kernel'), (1, 'ew_kernel')):
        names = _kernels_of(lambda: _run_pair(name, torch.bfloat16, 'counter', ROWWISE_SHAPES[0], misalign=misalign))
        mixed = [n for n in names if 'Mixed' in n]
        assert len(mixed) == 1 and ('tsde::' + kernel + '<') in mixed[0], (misalign, names)


@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name', [op for op in helpers.GENERAL_BROADCAST_OPS])
def test_broadcast_g_equals_widened_launch(name, half):
    for m in (8, 16, 5):
        _assert_pair(_run_pair(name, half, 'counter', ('cta', 'general', 300, 8, m), bcast=True), (name, m))


def test_16bit_g_leaves_the_tma_route():
    """cfg3_euler_general_large's tile (m = 16, B = 65536) takes the TMA-staged kernel in float32 and the
    per-thread-load kernel with a 16-bit g; both give the widened result."""
    rows, d, m = 65536, 32, 16
    before = helpers.tile_launches()
    res = _run_pair('tsde_step_euler', torch.bfloat16, 'counter', ('large', 'general', rows, d, m))
    after = helpers.tile_launches()
    assert after[1] - before[1] == 1 and after[0] - before[0] == 1, (before, after)
    _assert_pair(res, 'cfg3 large')


# ---- solves ----------------------------------------------------------------------------------------------------------
class Cast(nn.Module):
    """`base` with its outputs stored in 16 bits (what autocast hands back), optionally widened again."""

    def __init__(self, base, f_dtype, g_dtype, widened=False, prods=False, fused_prod=False):
        super().__init__()
        self.base, self.fd, self.gd, self.widened = base, f_dtype, g_dtype, widened
        self.noise_type, self.sde_type = base.noise_type, base.sde_type
        if prods:
            self.g_prod = self._g_prod
        if fused_prod:
            self.f_and_g_prod = self._f_and_g_prod

    def _out(self, x, dtype):
        wide = x.dtype  # the base SDE computes in the state dtype
        x = x.to(dtype)
        return x.to(wide) if self.widened else x

    def f(self, t, y):
        return self._out(self.base.f(t, y), self.fd)

    def g(self, t, y):
        return self._out(self.base.g(t, y), self.gd)

    def _f_and_g_prod(self, t, y, v):
        return self.f(t, y), self._g_prod(t, y, v)

    def _g_prod(self, t, y, v):
        g = self.base.g(t, y)
        prod = g * v if self.noise_type == 'diagonal' else torch.bmm(g, v.unsqueeze(-1)).squeeze(-1)
        return self._out(prod, self.gd)


def _problem(noise, sde_type, dtype=torch.float32):
    d, m = 8, {'diagonal': 8, 'scalar': 1, 'additive': 4, 'general': 4}[noise]
    base = {'diagonal': lambda: problems.GBMDiagonal(d, sde_type, seed=3, dtype=dtype),
            'scalar': lambda: problems.CosScalar(d, sde_type, seed=3, dtype=dtype),
            'additive': lambda: problems.TimeAdditive(d, m, sde_type, seed=3, dtype=dtype),
            'general': lambda: problems.TanhGeneral(d, m, sde_type, seed=3, dtype=dtype)}[noise]()
    return base.to(dev), d, m


SOLVES = [(meth, noise, 'ito') for meth in ('euler', 'milstein', 'srk')
          for noise in ('diagonal', 'scalar', 'additive', 'general')
          if not (meth != 'euler' and noise == 'general')] + \
         [(meth, noise, 'stratonovich') for meth in ('heun', 'midpoint', 'euler_heun', 'reversible_heun', 'milstein')
          for noise in ('diagonal', 'scalar', 'additive', 'general') if not (meth == 'milstein' and noise == 'general')]


def _solve(sde, y0, d, m, method, options=None, dtype=torch.float32, levy='none', **kw):
    bm = tsde.BrownianInterval(0.0, 0.25, size=(y0.size(0), m), dtype=dtype, device=dev, entropy=77,
                               levy_area_approximation=levy)
    return tsde.sdeint(sde, y0, [0.0, 0.125, 0.25], bm=bm, method=method, dt=DT, options=options, **kw)


@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('method,noise,sde_type', SOLVES)
def test_solve_equals_widened_solve(method, noise, sde_type, half):
    base, d, m = _problem(noise, sde_type)
    levy = 'space-time' if method == 'srk' else 'none'
    y0 = torch.full((96, d), 0.3, device=dev)
    with torch.no_grad():
        ref = _solve(Cast(base, half, half, widened=True), y0, d, m, method, levy=levy)
        for options in (None, {'cuda_graph': True}, {'cuda_graph': True, 'row_split': 2}):
            got = _solve(Cast(base, half, half), y0, d, m, method, options, levy=levy)
            assert got.dtype == torch.float32 and torch.equal(got, ref), (options, (got - ref).abs().max())
        # cfg4's shape (16-bit drift, float32 diffusion), and mixed formats
        for fd, gd in ((half, torch.float32), (torch.bfloat16, torch.float16)):
            ref = _solve(Cast(base, fd, gd, widened=True), y0, d, m, method, levy=levy)
            got = _solve(Cast(base, fd, gd), y0, d, m, method, levy=levy)
            assert torch.equal(got, ref), (fd, gd)


@pytest.mark.parametrize('fused', [False, True], ids=['g_prod', 'f_and_g_prod'])
@pytest.mark.parametrize('method', ['euler', 'milstein', 'srk', 'euler_heun_strat', 'heun_strat'])
def test_g_prod_protocol_equals_widened(method, fused):
    sde_type = 'stratonovich' if method.endswith('_strat') else 'ito'
    method = method.replace('_strat', '')
    base, d, m = _problem('diagonal', sde_type)
    levy = 'space-time' if method == 'srk' else 'none'
    y0 = torch.full((64, d), 0.3, device=dev)
    with torch.no_grad():
        kw = dict(prods=not fused, fused_prod=fused)
        ref = _solve(Cast(base, torch.bfloat16, torch.bfloat16, widened=True, **kw), y0, d, m, method, levy=levy)
        got = _solve(Cast(base, torch.bfloat16, torch.bfloat16, **kw), y0, d, m, method, levy=levy)
    assert torch.equal(got, ref)


class MLPDrift(nn.Module):
    noise_type, sde_type = 'diagonal', 'stratonovich'

    def __init__(self, d, widened=False):
        super().__init__()
        torch.manual_seed(5)
        self.net = nn.Sequential(nn.Linear(d, 64), nn.Tanh(), nn.Linear(64, d))
        self.sigma = nn.Parameter(torch.full((d,), 0.3))
        self.widened = widened

    def f(self, t, y):
        out = self.net(y)
        return out.float() if self.widened else out

    def g(self, t, y):
        return self.sigma * torch.tanh(y)


@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
def test_mlp_under_autocast_equals_widened(half):
    d = 16
    y0 = torch.randn(128, d, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    sde, wide = MLPDrift(d).to(dev), MLPDrift(d, widened=True).to(dev)
    wide.load_state_dict(sde.state_dict())
    with torch.no_grad(), torch.autocast('cuda', dtype=half):
        ref = _solve(wide, y0, d, d, 'reversible_heun')
        for options in (None, {'cuda_graph': True}):
            got = _solve(sde, y0, d, d, 'reversible_heun', options)
            assert torch.equal(got, ref), options


# ---- gradients -------------------------------------------------------------------------------------------------------
def _grads(sde, y0, fn):
    y0 = y0.clone().requires_grad_()
    ys = fn(sde, y0)
    loss = (ys ** 2).sum()
    params = [p for p in sde.parameters() if p.requires_grad]
    return (ys.detach(),) + torch.autograd.grad(loss, [y0] + params)


def _assert_grads(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and torch.equal(x, y), (x - y).abs().max()


@pytest.mark.parametrize('method,noise,sde_type', [('euler', 'general', 'ito'), ('milstein', 'diagonal', 'ito'),
                                                   ('srk', 'scalar', 'ito'), ('reversible_heun', 'diagonal',
                                                                                'stratonovich'),
                                                   ('heun', 'additive', 'stratonovich')])
def test_backprop_through_sdeint_equals_widened(method, noise, sde_type):
    base, d, m = _problem(noise, sde_type)
    levy = 'space-time' if method == 'srk' else 'none'
    y0 = torch.full((32, d), 0.3, device=dev)
    run = lambda s, y: _solve(s, y, d, m, method, levy=levy)  # noqa: E731
    _assert_grads(_grads(Cast(base, torch.bfloat16, torch.bfloat16), y0, run),
                  _grads(Cast(base, torch.bfloat16, torch.bfloat16, widened=True), y0, run))


ADJOINTS = [('reversible_heun', 'adjoint_reversible_heun', 'diagonal', 'stratonovich', None),
            ('reversible_heun', 'adjoint_reversible_heun', 'general', 'stratonovich', None),
            ('reversible_heun', 'adjoint_reversible_heun', 'diagonal', 'stratonovich', {'cuda_graph': True}),
            ('milstein', 'milstein', 'diagonal', 'ito', None),
            ('midpoint', 'midpoint', 'general', 'stratonovich', None)]


@pytest.mark.parametrize('half', HALF, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('method,adjoint_method,noise,sde_type,adjoint_options', ADJOINTS)
def test_sdeint_adjoint_equals_widened(method, adjoint_method, noise, sde_type, adjoint_options, half):
    base, d, m = _problem(noise, sde_type)
    y0 = torch.full((32, d), 0.3, device=dev)

    def run(s, y):
        bm = tsde.BrownianInterval(0.0, 0.25, size=(y.size(0), m), device=dev, entropy=9)
        return tsde.sdeint_adjoint(s, y, [0.0, 0.125, 0.25], bm=bm, method=method, adjoint_method=adjoint_method,
                                   dt=DT, adjoint_options=adjoint_options)
    _assert_grads(_grads(Cast(base, half, half), y0, run), _grads(Cast(base, half, half, widened=True), y0, run))


def test_double_backward_equals_widened():
    base, d, m = _problem('diagonal', 'stratonovich')
    y0 = torch.full((16, d), 0.3, device=dev)

    def gradgrad(sde):
        y = y0.clone().requires_grad_()
        ys = _solve(sde, y, d, m, 'midpoint')
        g, = torch.autograd.grad((ys ** 2).sum(), y, create_graph=True)
        return torch.autograd.grad(g.sum(), [y] + list(sde.parameters()))
    _assert_grads(gradgrad(Cast(base, torch.bfloat16, torch.bfloat16)),
                  gradgrad(Cast(base, torch.bfloat16, torch.bfloat16, widened=True)))


# ---- fallbacks and plans ---------------------------------------------------------------------------------------------
def test_float64_state_widens_on_the_host():
    base, d, m = _problem('diagonal', 'ito', dtype=torch.float64)
    y0 = torch.full((32, d), 0.3, dtype=torch.float64, device=dev)
    with torch.no_grad():
        got = _solve(Cast(base, torch.bfloat16, torch.bfloat16), y0, d, m, 'milstein', dtype=torch.float64)
        ref = _solve(Cast(base, torch.bfloat16, torch.bfloat16, widened=True), y0, d, m, 'milstein',
                     dtype=torch.float64)
    assert got.dtype == torch.float64 and torch.equal(got, ref)


class LogqpCast(Cast):
    def h(self, t, y):
        return self._out(-self.base.f(t, y), self.fd)


@pytest.mark.parametrize('noise', ['diagonal', 'general'])
def test_logqp_equals_widened(noise):
    base, d, m = _problem(noise, 'ito')
    y0 = torch.full((32, d), 0.3, device=dev)
    with torch.no_grad():
        m = m + 1 if noise == 'diagonal' else m  # (the log-ratio channel of a diagonal SDE has its own noise)
        got = _solve(LogqpCast(base, torch.bfloat16, torch.bfloat16), y0, d, m, 'euler', logqp=True)
        ref = _solve(LogqpCast(base, torch.bfloat16, torch.bfloat16, widened=True), y0, d, m, 'euler', logqp=True)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


@pytest.mark.parametrize('noise', ['diagonal', 'general'])
def test_log_ode_equals_widened(noise):
    base, d, m = _problem(noise, 'stratonovich')
    y0 = torch.full((32, d), 0.3, device=dev)
    with torch.no_grad():
        got = _solve(Cast(base, torch.bfloat16, torch.bfloat16), y0, d, m, 'log_ode', levy='foster')
        ref = _solve(Cast(base, torch.bfloat16, torch.bfloat16, widened=True), y0, d, m, 'log_ode', levy='foster')
    assert torch.equal(got, ref)


def test_plan_captured_under_autocast_is_not_replayed_without_it():
    d = 16
    y0 = torch.randn(128, d, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    sde = MLPDrift(d).to(dev)
    with torch.no_grad():
        eager = _solve(sde, y0, d, d, 'reversible_heun')
        with torch.autocast('cuda', dtype=torch.bfloat16):
            _solve(sde, y0, d, d, 'reversible_heun', {'cuda_graph': True})
        plain = _solve(sde, y0, d, d, 'reversible_heun', {'cuda_graph': True})
    assert torch.equal(plain, eager)


def test_float64_drift_with_float32_state_raises():
    base, d, m = _problem('diagonal', 'ito')
    y0 = torch.full((8, d), 0.3, device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match='float64'):
        _solve(Cast(base, torch.float64, torch.float32), y0, d, m, 'euler')
