"""Every general-noise kernel path against a float64 restatement of its entry point on the oracle's increments.

The general / additive-noise entry points contract g (rows, d, m) with the Brownian increment W (rows, m) (and U for
SRK) on one of five routes, picked by shape (csrc/tableau_general.cu `launch_gen`, csrc/cabi.cu):

* `gen_tma_kernel`, the TMA-staged tile kernel: a batch that fills its pipeline at m = 64, or m = 16 with one g operand;
* `gen_cta_kernel`, the per-thread-load tile kernel: m / 4 a power of two up to 32, aligned operands;
* `gen_kernel`, the generic tile kernel: every other m, and g or a memory-noise W / U off 16-byte alignment;
* the row-wise generic kernel (`ew_kernel`, one increment broadcast over d): scalar noise, m = 1;
* `gen_kernel` at m = 1: the SRK-additive entry points with one-channel additive noise.

Each launch runs with counter noise on one cell, counter noise on three cells of unequal length (lengths on the
device) and memory noise, in fp32 and fp64.  Every row of every output must lie within
    |got - ref| <= 4 (m + 16) u S  (+ for fp32 counter noise the SFU Box-Muller's per-normal agreement x S_noise)
of the float64 formula `ref` of its entry point, S being the same expression with every product and addend replaced by
its absolute value (over several cells the increments are themselves sums over the cells, taken term by term: the
kernel forms that merge too, and W summed from cells can cancel to far below its terms).  Outputs are prefilled with NaN (every slot must be written) and guarded by sentinel elements on
both sides (nothing outside may be).  The launch counters confirm each route.

The formulas are pinned to oracle/solvers.py, and the bound is shown to reject subtly wrong formulas, by CPU tests.
"""
import collections
import math

import numpy as np
import pytest
import torch

from oracle import brownian as obm
from oracle import solvers
from . import helpers
from .helpers import GEN_DT as DT, GENERAL_OPS

DEV = 'cuda'
FLAG_G_BROADCAST = 1                             # TSDE_FLAG_G_BROADCAST
KEY = 20261016                                   # Philox key
CELL = 11                                        # counter id of the (first) cell
CELLS3 = (2.0 ** -8, 3 * 2.0 ** -8, 2.0 ** -7)   # three cells of unequal length
SOURCES = ('counter1', 'counter3', 'memory')
GUARD = 64                                       # sentinel elements before and after every output
SENTINEL = -1234.5
UNIT = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
# per-normal agreement of the device's fp32 SFU Box-Muller with the oracle's float64 one (test_gpu_brownian.py
# test_cells_and_bridge_vs_oracle): |dN| <= ATOL_N + RTOL_N |N|
ATOL_N, RTOL_N = 5e-6, 2e-5


# ---- the float64 formulas ------------------------------------------------------------------------------------------
# One per entry point, on numpy arrays or torch tensors: E the (rows, d) operands and G the (rows, d, m) ones in argument
# order, w / u the increments (rows, m), sc the scalar arguments, half the 0.5 of the adjoint's outer products.  Each
# returns (ref, S) per output.  They restate torchsde_b200/csrc/tableau_general.cu (which cites the reference's
# methods/*.py lines) and are checked against oracle/solvers.py below.
def _mv(g, v):
    return (g * v[..., None, :]).sum(-1)


def _outer(a, v):
    return a[..., :, None] * v[..., None, :]


def _euler(E, G, w, u, aw, au, sc, half):
    (y0, f), (g,), (dt,) = E, G, sc
    return [(y0 + f * dt + _mv(g, w), abs(y0) + abs(f) * dt + _mv(abs(g), aw))]


def _midpoint_predict(E, G, w, u, aw, au, sc, half):
    (y0, f), (g,), (half_dt,) = E, G, sc
    return [(y0 + half_dt * f + 0.5 * _mv(g, w), abs(y0) + half_dt * abs(f) + 0.5 * _mv(abs(g), aw))]


def _euler_heun_predict(E, G, w, u, aw, au, sc, half):
    (y0,), (g,) = E, G
    return [(y0 + _mv(g, w), abs(y0) + _mv(abs(g), aw))]


def _reversible_heun_z(E, G, w, u, aw, au, sc, half):
    (y0, z0, f0), (g0,), (dt,) = E, G, sc
    return [(2 * y0 - z0 + f0 * dt + _mv(g0, w), 2 * abs(y0) + abs(z0) + abs(f0) * dt + _mv(abs(g0), aw))]


def _srk_additive_stage(E, G, w, u, aw, au, sc, half):
    (y0, f0), (ga,), (dt, rdt) = E, G, sc
    return [(y0 + 0.75 * f0 * dt + _mv(ga, 1.5 * u * rdt),
             abs(y0) + 0.75 * abs(f0) * dt + _mv(abs(ga), 1.5 * au * rdt))]


def _heun(E, G, w, u, aw, au, sc, half):
    (y0, f, fp), (g, gp), (dt,) = E, G, sc
    return [(y0 + (dt * (f + fp) + _mv(g, w) + _mv(gp, w)) * 0.5,
             abs(y0) + (dt * (abs(f) + abs(fp)) + _mv(abs(g), aw) + _mv(abs(gp), aw)) * 0.5)]


def _euler_heun(E, G, w, u, aw, au, sc, half):
    (y0, f), (g, gp), (dt,) = E, G, sc
    return [(y0 + dt * f + (_mv(g, w) + _mv(gp, w)) * 0.5,
             abs(y0) + dt * abs(f) + (_mv(abs(g), aw) + _mv(abs(gp), aw)) * 0.5)]


def _reversible_heun(E, G, w, u, aw, au, sc, half):
    (y0, f0, f1), (g0, g1), (half_dt,) = E, G, sc
    return [(y0 + (f0 + f1) * half_dt + _mv(g0 + g1, 0.5 * w),
             abs(y0) + (abs(f0) + abs(f1)) * half_dt + _mv(abs(g0) + abs(g1), 0.5 * aw))]


def _srk_additive(E, G, w, u, aw, au, sc, half):
    (y0, f0, f1), (ga, gb), (dt, rdt) = E, G, sc
    return [(y0 + f0 * dt / 3 + _mv(ga, w - u * rdt) + 2 * f1 * dt / 3 + _mv(gb, u * rdt),
             abs(y0) + abs(f0) * dt / 3 + _mv(abs(ga), aw + au * rdt) + 2 * abs(f1) * dt / 3
             + _mv(abs(gb), au * rdt))]


def _adjoint_a(E, G, w, u, aw, au, sc, half):
    (y0, z0, f0, adj_y0, adj_f0), (g0, adj_g0), (dt, half_dt) = E, G, sc
    return [(2 * y0 - z0 - f0 * dt - _mv(g0, w), 2 * abs(y0) + abs(z0) + abs(f0) * dt + _mv(abs(g0), aw)),
            (adj_f0 + adj_y0 * half_dt, abs(adj_f0) + abs(adj_y0) * half_dt),
            (adj_g0 + _outer(adj_y0, half * w), abs(adj_g0) + _outer(abs(adj_y0), half * aw))]


def _adjoint_b(E, G, w, u, aw, au, sc, half):
    (y0, f0, f1, adj_y0, adj_z0, vjp_z), (g0, g1), (dt, half_dt) = E, G, sc
    a, sa = adj_z0 + vjp_z, abs(adj_z0) + abs(vjp_z)
    return [(y0 - (f0 + f1) * half_dt - _mv(g0 + g1, 0.5 * w),
             abs(y0) + (abs(f0) + abs(f1)) * half_dt + _mv(abs(g0) + abs(g1), 0.5 * aw)),
            (adj_y0 + 2 * a, abs(adj_y0) + 2 * sa),
            (-a, sa),
            (adj_y0 * half_dt + a * dt, abs(adj_y0) * half_dt + sa * dt),
            (_outer(adj_y0, half * w) + _outer(a, w), _outer(abs(adj_y0), half * aw) + _outer(sa, aw))]


FORMULAS = {
    'tsde_step_euler': _euler,
    'tsde_midpoint_predict': _midpoint_predict,
    'tsde_euler_heun_predict': _euler_heun_predict,
    'tsde_reversible_heun_z': _reversible_heun_z,
    'tsde_srk_additive_stage': _srk_additive_stage,
    'tsde_adjoint_reversible_heun_a': _adjoint_a,
    'tsde_step_heun': _heun,
    'tsde_step_euler_heun': _euler_heun,
    'tsde_step_reversible_heun': _reversible_heun,
    'tsde_step_srk_additive': _srk_additive,
    'tsde_adjoint_reversible_heun_b': _adjoint_b,
}
assert FORMULAS.keys() == GENERAL_OPS.keys()


def formula(op, E, G, w, u, scalars=None, half=0.5, aw=None, au=None):
    """[(ref, S)] of entry point `op` on its (rows, d) operands E and (rows, d, m) operands G.  aw / au: the
    magnitudes S takes for the increments (default |w|, |u|)."""
    aw = abs(w) if aw is None else aw
    au = abs(u) if au is None else au
    return FORMULAS[op](E, G, w, u, aw, au, GENERAL_OPS[op].scalars if scalars is None else scalars, half)


def bound(S, m, dtype, allow=0):
    return 4 * (m + 16) * UNIT[dtype] * S + allow


def magnitudes(op, E, G, inc, scalars=None, half=0.5):
    """Per output: S with the increments' own magnitudes (inc.aW, inc.aU), and the allowance for the fp32 SFU
    Box-Muller (every formula is linear in (w, u): S on (dW, dU) minus S without noise; 0 without an allowance)."""
    S = [s for _, s in formula(op, E, G, inc.W, inc.U, scalars, half, inc.aW, inc.aU)]
    if inc.dW is None:
        return S, [0] * len(S)
    hi = formula(op, E, G, inc.W, inc.U, scalars, half, inc.dW, inc.dU)
    lo = formula(op, E, G, inc.W, inc.U, scalars, half, 0 * inc.dW, 0 * inc.dU)
    return S, [a[1] - b[1] for a, b in zip(hi, lo)]


# ---- operands and increments (one generator for the CPU and the GPU cases) -----------------------------------------
def _placed(x, shift):
    """x, or the same values `shift` elements past a 16-byte boundary."""
    if not shift:
        return x
    buf = torch.empty(x.numel() + shift, device=x.device, dtype=x.dtype)
    buf[shift:].copy_(x.reshape(-1))
    return buf[shift:].view(x.shape)


def operands(B, d, m, dtype, device, seed, bcast=False, g_shift=0):
    """Six (B, d) operands in [-1, 1) and two g operands in [-0.5, 0.5): (B, d, m), or one (d, m) block each with
    `bcast`; enough for every entry point (`op_operands`)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    E = [2 * torch.rand(B, d, generator=gen, device=device, dtype=dtype) - 1 for _ in range(6)]
    G = [_placed(torch.rand(*((d, m) if bcast else (B, d, m)), generator=gen, device=device, dtype=dtype) - 0.5,
                 g_shift) for _ in range(2)]
    return E, G


def op_operands(op, E, G):
    """The operands of `op` in argument order, taken in turn from the pools E and G."""
    e, g = iter(E), iter(G)
    return [next(e) if k == 'e' else next(g) for k in GENERAL_OPS[op].args]


Increments = collections.namedtuple('Increments', 'source w u W U aW aU dW dU lengths')


def increments(source, B, m, dtype, device, row_offset=0, seed=0, shift=0):
    """One noise source over rows [0, B): the device tensors a memory-noise launch reads (w, u), the float64 (W, U)
    the formulas use (memory noise: the tensors themselves; counter noise: the oracle's cells at `row_offset`), the
    magnitudes S takes for them (aW, aU: over several cells W and U are sums over the cells, taken term by term in
    absolute value) and, for fp32 counter noise, the allowance (dW, dU) of the device's Box-Muller."""
    to = dict(device=device, dtype=torch.float64)
    if source == 'memory':
        gen = torch.Generator(device=device).manual_seed(seed + 1)
        w, u = (_placed(torch.randn(B, m, generator=gen, device=device, dtype=dtype) * DT ** 0.5, shift)
                for _ in range(2))
        W, U = w.double(), u.double()
        return Increments(source, w, u, W, U, W.abs(), U.abs(), None, None, None)
    npdt = np.float32 if dtype == torch.float32 else np.float64
    lengths = (DT,) if source == 'counter1' else CELLS3
    ht = sum(lengths)
    cells = [tuple(x.astype(np.float64) for x in obm.cell(KEY, CELL + c, h, B, m, npdt, True, row_offset))
             for c, h in enumerate(lengths)]
    if len(lengths) == 1:
        W, H = obm.cell(KEY, CELL, lengths[0], B, m, npdt, True, row_offset)
    else:
        W, H = obm.cells(KEY, CELL, list(lengths), B, m, npdt, True, row_offset)
    U = obm.h_to_u(W, H, ht)
    # the merge of oracle/brownian.py `cells` on magnitudes
    aW, aH = np.abs(cells[0][0]), np.abs(cells[0][1])
    elapsed = lengths[0]
    for h, (Wc, Hc) in zip(lengths[1:], cells[1:]):
        aH = (h * (np.abs(Hc) + 0.5 * aW) + elapsed * (aH + 0.5 * np.abs(Wc))) / (elapsed + h)
        aW = aW + np.abs(Wc)
        elapsed += h
    dW = dU = None
    if dtype == torch.float32:
        dW = sum(ATOL_N * math.sqrt(h) + RTOL_N * np.abs(Wc) for h, (Wc, _) in zip(lengths, cells))
        dH = sum(ATOL_N * math.sqrt(h / 12) + RTOL_N * np.abs(Hc) for h, (_, Hc) in zip(lengths, cells))
        dW, dU = torch.tensor(dW, **to), torch.tensor(ht * (dW + dH), **to)
    t = lambda x: torch.tensor(np.asarray(x, dtype=np.float64), **to)   # noqa: E731
    return Increments(source, None, None, t(W), t(U), t(aW), t(ht * (0.5 * aW + aH)), dW, dU, lengths)


# ---- CPU: the formulas against oracle/solvers.py -------------------------------------------------------------------
class _Scripted:
    """An SDE whose f(t, y) and g(t, y) return fixed arrays chosen by t, recording the states they are called at."""

    def __init__(self, f, g, noise_type='general'):
        self._f, self._g, self.noise_type, self.calls = f, g, noise_type, []

    def f(self, t, y):
        self.calls.append(('f', float(t), y))
        return self._f[float(t)]

    def g(self, t, y):
        self.calls.append(('g', float(t), y))
        return self._g[float(t)]

    def state(self, kind, t):
        (y,) = {id(y): y for k, tt, y in self.calls if k == kind and tt == float(t)}.values()
        return y


def _agree(name, got, ref_s, m):
    ref, S = ref_s
    err = np.abs(np.asarray(got, dtype=np.float64) - ref)
    lim = bound(S, m, torch.float64)
    assert np.all(err <= lim), f'{name}: max err/bound {np.max(err / lim):.3g}'


@pytest.mark.parametrize('m', [1, 3, 8])
def test_formulas_match_oracle_solvers(m):
    """Each formula restates what oracle/solvers.py computes with the same operands and increments, to float64
    rounding: the steps' predictor states (recorded where the SDE is evaluated) and results, the SRA1 stage and final
    update, and both halves of the reversible-Heun adjoint step."""
    rng = np.random.default_rng(m)
    B, d = 7, 5
    e = lambda: rng.uniform(-1, 1, (B, d))              # noqa: E731
    g = lambda: rng.uniform(-0.5, 0.5, (B, d, m))       # noqa: E731
    w, u = rng.standard_normal((B, m)) * DT ** 0.5, rng.standard_normal((B, m)) * DT ** 0.5
    bm = lambda ta, tb, return_U=False: (w, u) if return_U else w   # noqa: E731
    t0 = 0.25
    t1, half_dt = t0 + DT, 0.5 * DT
    y0, z0, F0, F1, G0, G1 = e(), e(), e(), e(), g(), g()
    sc = lambda *x: tuple(x)                            # noqa: E731

    def run(method, f, gg, noise_type='general', extra=()):
        sde = _Scripted(f, gg, noise_type)
        return sde, solvers.make(method, sde, bm, DT).step(t0, t1, y0, extra)

    sde, (y1, _) = run('euler', {t0: F0}, {t0: G0})
    _agree('euler', y1, formula('tsde_step_euler', [y0, F0], [G0], w, u)[0], m)
    sde, (y1, _) = run('heun', {t0: F0, t1: F1}, {t0: G0, t1: G1})
    _agree('heun predictor', sde.state('f', t1), formula('tsde_step_euler', [y0, F0], [G0], w, u)[0], m)
    _agree('heun', y1, formula('tsde_step_heun', [y0, F0, F1], [G0, G1], w, u)[0], m)
    tp = t0 + half_dt
    sde, (y1, _) = run('midpoint', {t0: F0, tp: F1}, {t0: G0, tp: G1})
    _agree('midpoint predictor', sde.state('f', tp), formula('tsde_midpoint_predict', [y0, F0], [G0], w, u)[0], m)
    _agree('midpoint', y1, formula('tsde_step_euler', [y0, F1], [G1], w, u)[0], m)
    sde, (y1, _) = run('euler_heun', {t0: F0}, {t0: G0, t1: G1})
    _agree('euler-heun predictor', sde.state('g', t1), formula('tsde_euler_heun_predict', [y0], [G0], w, u)[0], m)
    _agree('euler-heun', y1, formula('tsde_step_euler_heun', [y0, F0], [G0, G1], w, u)[0], m)
    sde, (y1, (_, _, z1)) = run('reversible_heun', {t1: F1}, {t1: G1}, extra=(F0, G0, z0))
    _agree('reversible-heun z', z1, formula('tsde_reversible_heun_z', [y0, z0, F0], [G0], w, u)[0], m)
    _agree('reversible-heun', y1, formula('tsde_step_reversible_heun', [y0, F0, F1], [G0, G1], w, u)[0], m)
    # SRA1: f at t0 and t0 + 3/4 dt, gA = g(t1, y0), gB = g(t0, y0)
    ts = t0 + 0.75 * DT
    sde, (y1, _) = run('srk', {t0: F0, ts: F1}, {t1: G0, t0: G1}, noise_type='additive')
    _agree('srk stage', sde.state('f', ts), formula('tsde_srk_additive_stage', [y0, F0], [G0], w, u)[0], m)
    _agree('srk final', y1, formula('tsde_step_srk_additive', [y0, F0, F1], [G0, G1], w, u)[0], m)
    # the adjoint step (reversed times t0 < t1: the forward SDE is evaluated at -t1)
    adj_y0, adj_f0, adj_z0, vjp_z, adj_g0 = e(), e(), e(), e(), g()
    seen = {}

    def vjp(t, z, adj_f, adj_g):
        seen.update(adj_f=adj_f, adj_g=adj_g)
        return vjp_z

    sde = _Scripted({-t1: F1}, {-t1: G1})
    (y1, z1, _, _), (adj_y1, adj_f1, adj_g1, adj_z1) = solvers.adjoint_reversible_heun_step(
        sde, t0, t1, y0, z0, F0, G0, adj_y0, adj_f0, adj_g0, adj_z0, w, vjp)
    a = formula('tsde_adjoint_reversible_heun_a', [y0, z0, F0, adj_y0, adj_f0], [G0, adj_g0], w, u,
                sc(DT, half_dt))
    for name, got, ref in zip(('z1', "adj_f0'", "adj_g0'"), (z1, seen['adj_f'], seen['adj_g']), a):
        _agree(f'adjoint a {name}', got, ref, m)
    b = formula('tsde_adjoint_reversible_heun_b', [y0, F0, F1, adj_y0, adj_z0, vjp_z], [G0, G1], w, u,
                sc(DT, half_dt))
    for name, got, ref in zip(('y1', 'adj_y1', 'adj_z1', 'adj_f1', 'adj_g1'), (y1, adj_y1, adj_z1, adj_f1, adj_g1), b):
        _agree(f'adjoint b {name}', got, ref, m)


# ---- CPU: the bound rejects subtly wrong formulas ------------------------------------------------------------------
def _group_rows(B, m):
    """Rows r whose group of 32 / (m / 4) rows (gen_cta_kernel's CTA) ends at r, with a row r + 1 after them."""
    rw = 128 // m
    return np.arange(rw - 1, B - 1, rw)


def _mutations(op, m, B):
    """(name, kwargs of the mutated formula call) for every mutation that applies to `op` at this shape."""
    spec = GENERAL_OPS[op]
    out = [('last channel dropped', dict(drop=True))]
    if m % 4 == 0 and 128 % m == 0 and 128 // m > 1 and len(_group_rows(B, m)):
        out.append(("group's last row given the next row's increments", dict(shift_rows=True)))
    if spec.want_u:
        out.append(('W and U swapped', dict(swap=True)))
    if op in ('tsde_midpoint_predict', 'tsde_step_reversible_heun'):
        out.append(('dt for half_dt', dict(scalars=(DT,))))
    if 'adjoint' in op:
        out.append(('dt for half_dt', dict(scalars=(DT, DT))))
        out.append(('dW for 0.5 dW in the outer products', dict(half=1.0)))
    return out


def _mutated(op, E, G, inc, B, m, drop=False, shift_rows=False, swap=False, scalars=None, half=0.5):
    w, u = inc.W.clone(), inc.U.clone()
    if drop:
        w[:, -1] = 0
        u[:, -1] = 0
    if shift_rows:
        r = torch.from_numpy(_group_rows(B, m))
        w[r], u[r] = inc.W[r + 1], inc.U[r + 1]
    if swap:
        w, u = u, w
    return formula(op, E, G, w, u, scalars, half)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_bound_rejects_wrong_formulas(dtype):
    """On the GPU cases' operand generator and the oracle's increments, at shapes of three routes and with every
    noise source (fp32 counter noise with its Box-Muller allowance, the loosest bound), the bound rejects each
    mutated formula on a clear majority (>= 75 %) of the output elements the mutation changes: the last Brownian channel
    dropped; the last row of each 32/(m/4)-row group given the next row's increments; W and U swapped in the SRK
    weights; dt where half_dt belongs; dW for 0.5 dW in the adjoint's outer products."""
    bad, seen = [], set()
    for B, d, m in ((41, 33, 16), (37, 7, 12), (19, 4, 64), (9, 3, 256), (21, 5, 1)):
        E, G = operands(B, d, m, dtype, 'cpu', seed=B * d + m)
        E, G = [x.double() for x in E], [x.double() for x in G]
        for source in SOURCES:
            inc = increments(source, B, m, dtype, 'cpu', seed=m)
            for op in GENERAL_OPS:
                xe, xg = [], []
                for k, x in zip(GENERAL_OPS[op].args, op_operands(op, E, G)):
                    (xe if k == 'e' else xg).append(x)
                true = formula(op, xe, xg, inc.W, inc.U)
                S, allow = magnitudes(op, xe, xg, inc)
                for name, kw in _mutations(op, m, B):
                    wrong = _mutated(op, xe, xg, inc, B, m, **kw)
                    for i, ((ref, _), (mut, _), Si, al) in enumerate(zip(true, wrong, S, allow)):
                        changed = mut != ref
                        if not changed.any():
                            continue
                        seen.add(name)
                        caught = ((mut - ref).abs() > bound(Si, m, dtype, al))[changed].double().mean().item()
                        if caught < 0.75:
                            bad.append(f'{name}: {op[5:]} out{i} m={m} {source}: caught on {caught:.1%}')
    assert len(seen) == 5, seen
    assert not bad, '\n'.join(bad)


# ---- GPU: the launch matrix ----------------------------------------------------------------------------------------
class _Report:
    """Worst err / bound per (route, dtype, noise source) and the (entry point, output) pairs each route ran."""

    def __init__(self):
        self.worst = collections.defaultdict(float)
        self.pairs = collections.defaultdict(set)

    def add(self, key, op, i, ratio):
        self.worst[key] = max(self.worst[key], ratio)
        self.pairs[key[0]].add((op, i))

    def print(self):
        for key in sorted(self.worst):
            print(f'{" / ".join(key):44s} worst err/bound {self.worst[key]:.3f}')
        for route in sorted(self.pairs):
            print(f'{route}: {len(self.pairs[route])} (entry point, output) pairs')


def _run_case(route, op, dtype, B, d, m, E, G, E64, G64, inc, key, cell_h, report, bad, bcast=False,
              row_offset=0, expect=None):
    """One launch of `op` on the pools' operands with noise `inc`, checked against its formula."""
    spec = GENERAL_OPS[op]
    n = {'e': B * d, 'g': B * d * m}
    bufs = [torch.full((n[k] + 2 * GUARD,), SENTINEL, device=DEV, dtype=dtype) for k in spec.outs]
    outs = [b[GUARD:GUARD + n[k]] for b, k in zip(bufs, spec.outs)]
    for o in outs:
        o.fill_(float('nan'))
    if inc.source == 'memory':
        nz = helpers.general_noise(w=inc.w.data_ptr(), u=inc.u.data_ptr(), want_u=spec.want_u)
    else:
        nz = helpers.general_noise(key=key, cell_id=CELL, h=inc.lengths[0], h_total=sum(inc.lengths),
                                   cell_h=cell_h if len(inc.lengths) > 1 else None, row_offset=row_offset,
                                   want_u=spec.want_u)
    nz.row_offset, nz.flags = row_offset, FLAG_G_BROADCAST if bcast else 0
    n0 = helpers.tile_launches()
    helpers.general_call(op, dtype, B, d, m, [x.data_ptr() for x in op_operands(op, E, G)], nz,
                         [o.data_ptr() for o in outs])
    n1 = helpers.tile_launches()
    routed = (n1[0] - n0[0], n1[1] - n0[1])
    where = f'{route} {op[5:]} {str(dtype)[6:]} {inc.source} B={B} d={d} m={m}'
    if expect is not None and routed != expect:
        bad.append(f'{where}: launched (per-thread-load, TMA-staged) = {routed}, expected {expect}')
        return
    xe, xg = [], []
    for k, x in zip(spec.args, op_operands(op, E64, G64)):
        (xe if k == 'e' else xg).append(x)
    refs = formula(op, xe, xg, inc.W, inc.U)
    Ss, allows = magnitudes(op, xe, xg, inc)
    for i, (buf, o, (ref, _), S, al, k) in enumerate(zip(bufs, outs, refs, Ss, allows, spec.outs)):
        if not (torch.equal(buf[:GUARD], torch.full_like(buf[:GUARD], SENTINEL))
                and torch.equal(buf[-GUARD:], torch.full_like(buf[-GUARD:], SENTINEL))):
            bad.append(f'{where} out{i}: wrote outside its output')
        if not torch.isfinite(o).all():
            rows = (~torch.isfinite(o)).nonzero()[:, 0] // (n[k] // B)
            bad.append(f'{where} out{i}: {rows.numel()} slots not written (first row {int(rows[0])})')
            continue
        got = o.view(ref.shape).double()
        lim = bound(S, m, dtype, al)
        err = (got - ref).abs()
        ratio = torch.where(lim > 0, err / lim, torch.where(err > 0, math.inf, 0.0))
        worst = ratio.max().item()
        report.add((route, str(dtype)[6:], inc.source), op, i, worst)
        if worst > 1:
            rows = (ratio > 1).reshape(B, -1).any(1).nonzero()[:, 0]
            bad.append(f'{where} out{i}: {rows.numel()} rows off the formula (first {rows[:4].tolist()}), '
                       f'worst err/bound {worst:.3g}')


def _run_shapes(route, dtype, shapes, report, bad, sources=SOURCES, bcast=False, near_limit=False):
    """shapes: (B, d, m, ops, expected launch counts, g shift, memory W / U shift)."""
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    cell_h = torch.tensor(CELLS3, dtype=torch.float64, device=DEV)
    for B, d, m, ops, expect, g_shift, w_shift in shapes:
        E, G = operands(B, d, m, dtype, DEV, seed=B * d + m, bcast=bcast, g_shift=g_shift)
        E64 = [x.double() for x in E]
        G64 = [x.double()[None] if bcast else x.double() for x in G]
        row_offset = (1 << 32) - 1 - B if near_limit else 0
        for source in sources:
            if w_shift and source != 'memory':
                continue
            inc = increments(source, B, m, dtype, DEV, row_offset=row_offset, seed=B + m, shift=w_shift)
            for op in ops:
                _run_case(route, op, dtype, B, d, m, E, G, E64, G64, inc, key, cell_h, report, bad, bcast=bcast,
                          row_offset=row_offset, expect=expect)
            del inc
        del E, G, E64, G64
    torch.cuda.empty_cache()


ALL = list(GENERAL_OPS)
CTA, TMA, NONE = (1, 0), (0, 1), (0, 0)


def _tma_ops(m, max_g=2):
    return [op for op, mm in helpers.GENERAL_TMA_REACHABLE if mm == m and GENERAL_OPS[op].tile_g <= max_g]


def _route_shapes(route, dtype):
    if route == 'tma':   # ragged last tile everywhere
        shapes = [(65539, 32, 16, _tma_ops(16), TMA, 0, 0), (16387, 32, 64, _tma_ops(64), TMA, 0, 0),
                  (65539, 4, 64, _tma_ops(64), TMA, 0, 0)]
        if dtype == torch.float32:   # one 32 KiB g row per stage (one g operand only)
            shapes.append((2100, 128, 64, _tma_ops(64, max_g=1), TMA, 0, 0))
        return shapes
    if route == 'cta':   # B = 1 and B = k * 32/(m/4) +- 1 (ragged last group)
        return [(B, d, m, ALL, CTA, 0, 0) for m in (4, 8, 16, 32, 64, 128)
                for B, d in ((1, 1), (3 * 128 // m + 1, 3), (2 * 128 // m - 1, 33), (128 // m + 1, 129))]
    if route == 'gen':   # m % 4 != 0, m / 4 not a power of two, m > 128, unaligned g / W / U
        return [(37, 7, 2, ALL, NONE, 0, 0), (5, 300, 3, ALL, NONE, 0, 0), (129, 7, 5, ALL, NONE, 0, 0),
                (3, 5000, 12, ALL, NONE, 0, 0), (16901, 7, 12, ALL, NONE, 0, 0), (17, 300, 24, ALL, NONE, 0, 0),
                (65, 7, 40, ALL, NONE, 0, 0), (3, 300, 132, ALL, NONE, 0, 0), (2, 5000, 256, ALL, NONE, 0, 0),
                (9, 7, 256, ALL, NONE, 0, 0), (37, 7, 16, ALL, NONE, 1, 0), (21, 300, 8, ALL, NONE, 0, 1)]
    if route == 'rowwise':
        return [(B, d, 1, helpers.GENERAL_ROWWISE_OPS, NONE, 0, 0) for B, d in ((37, 1), (1000, 5), (3, 64))]
    srk = ['tsde_srk_additive_stage', 'tsde_step_srk_additive']
    return [(37, 1, 1, srk, NONE, 0, 0), (300, 6, 1, srk, NONE, 0, 0)]


ROUTES = ['tma', 'cta', 'gen', 'rowwise', 'gen_m1']


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('route', ROUTES)
def test_route_vs_formula(route, dtype):
    """Every entry point the route serves, at shapes chosen to take it (confirmed by the launch counters), with every
    noise source: every row of every output within the bound of its float64 formula, every slot written, nothing
    written outside."""
    report, bad = _Report(), []
    _run_shapes(route, dtype, _route_shapes(route, dtype), report, bad)
    report.print()
    assert not bad, '\n'.join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_broadcast_g_vs_formula(dtype):
    """TSDE_FLAG_G_BROADCAST (one (d, m) block, row stride 0) on per-thread-load shapes (also a batch that would
    otherwise take the TMA-staged kernel) and generic shapes, for the seven entry points that accept it."""
    report, bad = _Report(), []
    ops = helpers.GENERAL_BROADCAST_OPS
    _run_shapes('cta+bcast', dtype, [(33, 3, 8, ops, CTA, 0, 0), (16387, 32, 64, ops, CTA, 0, 0)], report, bad,
                bcast=True)
    _run_shapes('gen+bcast', dtype, [(37, 7, 12, ops, NONE, 0, 0), (9, 300, 5, ops, NONE, 0, 0)], report, bad,
                bcast=True)
    report.print()
    assert not bad, '\n'.join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_row_offset_near_limit_vs_formula(dtype):
    """row_offset = 2^32 - 1 - B, the last valid global rows, on one shape per route: counter noise must be the
    oracle's rows at that offset (memory noise ignores the offset)."""
    report, bad = _Report(), []
    for route, shape in (('tma', (16387, 32, 64, _tma_ops(64), TMA, 0, 0)), ('cta', (17, 33, 16, ALL, CTA, 0, 0)),
                         ('gen', (37, 7, 5, ALL, NONE, 0, 0)),
                         ('rowwise', (37, 5, 1, helpers.GENERAL_ROWWISE_OPS, NONE, 0, 0)),
                         ('gen_m1', _route_shapes('gen_m1', dtype)[0])):
        _run_shapes(route + '@2^32', dtype, [shape], report, bad, near_limit=True)
    report.print()
    assert not bad, '\n'.join(bad)
