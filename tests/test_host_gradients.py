"""The transpose table of plain `sdeint`'s backward (torchsde_b200/_core/autograd_ops.py) against autograd of a float64
restatement of each kernel's forward formula, and the finite-difference harness of tests/gradient_ref.py on a
pure-torch solve.  CPU only: `TableauFn.backward` is pure torch and is called with a stand-in `ctx`.

Every entry of `autograd_ops._table` is restated from the kernels' formulas (csrc/tableau_diag_ops.cuh and the
general-noise ops of csrc/tableau_general.cu), written with one product P(g, v) whose meaning depends on the operand
layout the solvers produce:

    layout      g                        increments        P(g, v)
    diagonal    (rows, d)                (rows, d)         g * v
    scalar      (rows, d, 1)             (rows, 1)         g v, the increment broadcast over d
    general     (rows, d, m), m = 1, 3   (rows, m)         batched matrix-vector product
    expanded    (d, m).expand(rows, ...)  (rows, m)        the same, gradient taken w.r.t. the (d, m) block
    unit        (rows, d): g_prod        none (W == 1)      the user's product itself

The restatements of the diagonal layout are first checked against the formulas the GPU suite verifies the kernels
with (test_gpu_index_paths.NOISE_OPS / PLAIN_OPS), so the table is compared with the kernels' arithmetic, not with
itself.  The vector-Jacobian product of the table must equal `torch.autograd.grad` of the restatement for random
cotangents to a few ulp, and the table check must catch each of a list of single-token mutations of autograd_ops.py.
"""
import inspect
import math
import re
import types

import numpy as np
import pytest
import torch

from torchsde_b200._core import autograd_ops
from . import gradient_ref
from .test_gpu_index_paths import DT, NOISE_OPS, PLAIN_OPS, RDT, SQ

ROWS, D = 5, 3
ULP = 2.0 ** -52


class Layout:
    def __init__(self, kind, m=None):
        self.kind, self.m = kind, m

    def P(self, g, v):
        """The product g.v of a diffusion operand and a weight of the increment's shape."""
        if self.kind in ('diagonal', 'unit'):
            return g * v
        return (g * v.unsqueeze(-2)).sum(-1)

    def E(self, g):
        """A diffusion operand used element-wise (the diagonal / scalar SRK stages): its (rows, d) view."""
        return g.reshape(g.shape[0], g.shape[1])

    def G(self, g, v):
        """A g-shaped result: every column of g times its weight (Milstein's vjp seed)."""
        return g * v.unsqueeze(-2) if g.dim() == 3 else g * v


def _srk_weights(w, u, dt, rdt, sq, three_dt):
    """srid2's noise weights of srk.py (gw_s): the kernel's SrkDiagFinalOp."""
    ikk = (w * w - dt) * 0.5
    i3 = (w * w * w - three_dt * w) / 6
    b1, b2, b3, b4 = (-1, 4 / 3, 2 / 3, 0), (1, -4 / 3, 1 / 3, 0), (2, -4 / 3, -2 / 3, 0), (-2, 5 / 3, -2 / 3, 1)
    return [b1[s] * w + b2[s] * ikk / sq + b3[s] * u * rdt + b4[s] * i3 * rdt for s in range(4)]


def _srk_final(x, w, u, sc, L):
    dt, rdt, sq, three_dt = sc
    gw = _srk_weights(w, u, dt, rdt, sq, three_dt)
    y1 = x[0] + (x[1] / 6 + x[2] / 6 + x[3] * (2 / 3)) * dt
    for s in range(4):
        y1 = y1 + L.E(x[4 + s]) * gw[s]
    return [y1]


def _gf(x, w, u, sc, L):
    dt, two_sq, ito = sc
    v = (w * w - dt if ito else w * w) / two_sq
    return [x[0] + x[1] * dt + L.P(x[2], w) + L.P(x[3] - x[2], v)]


# entry -> (argument kinds: 'e' a (rows, d) operand, 'g' a diffusion operand; number of outputs; wants U;
#           forward restatement (inputs, W, U, scalars, layout) -> outputs)
RESTATED = {
    'tsde_step_euler': ('eeg', 1, False, lambda x, w, u, sc, L: [x[0] + x[1] * sc[0] + L.P(x[2], w)]),
    'tsde_milstein_vjp_seed': ('g', 1, False,
                               lambda x, w, u, sc, L: [L.G(x[0], 0.5 * (w * w - sc[0] if sc[1] else w * w))]),
    'tsde_step_milstein': ('eege', 1, False, lambda x, w, u, sc, L: [x[0] + x[1] * sc[0] + L.P(x[2], w) + x[3]]),
    'tsde_milstein_gf_predict': ('eeg', 1, False,
                                 lambda x, w, u, sc, L: [x[0] + (sc[0] * x[1] if sc[2] else 0) + L.E(x[2]) * sc[1]]),
    'tsde_step_milstein_gf': ('eegg', 1, False, _gf),
    'tsde_step_heun': ('eeegg', 1, False,
                       lambda x, w, u, sc, L: [x[0] + 0.5 * sc[0] * (x[1] + x[2])
                                               + 0.5 * (L.P(x[3], w) + L.P(x[4], w))]),
    'tsde_midpoint_predict': ('eeg', 1, False, lambda x, w, u, sc, L: [x[0] + sc[0] * x[1] + 0.5 * L.P(x[2], w)]),
    'tsde_euler_heun_predict': ('eg', 1, False, lambda x, w, u, sc, L: [x[0] + L.P(x[1], w)]),
    'tsde_step_euler_heun': ('eegg', 1, False,
                             lambda x, w, u, sc, L: [x[0] + sc[0] * x[1] + 0.5 * (L.P(x[2], w) + L.P(x[3], w))]),
    'tsde_reversible_heun_z': ('eeeg', 1, False,
                               lambda x, w, u, sc, L: [2 * x[0] - x[1] + sc[0] * x[2] + L.P(x[3], w)]),
    'tsde_step_reversible_heun': ('eeegg', 1, False,
                                  lambda x, w, u, sc, L: [x[0] + sc[0] * (x[1] + x[2])
                                                          + 0.5 * (L.P(x[3], w) + L.P(x[4], w))]),
    'tsde_srk_diag_stage1': ('eeg', 2, False,
                             lambda x, w, u, sc, L: [x[0] + sc[0] * x[1],
                                                     x[0] + 0.25 * sc[0] * x[1] - 0.5 * sc[1] * L.E(x[2])]),
    'tsde_srk_diag_stage2': ('eegeg', 2, True,
                             lambda x, w, u, sc, L: [x[0] + 0.25 * sc[0] * x[1] + L.E(x[2]) * u * sc[1]
                                                     + 0.25 * sc[0] * x[3] + 0.5 * L.E(x[4]) * u * sc[1],
                                                     x[0] + sc[0] * x[1] + sc[2] * L.E(x[2])]),
    'tsde_srk_diag_stage3': ('eggeg', 1, False,
                             lambda x, w, u, sc, L: [x[0] + (2 * L.E(x[1]) - L.E(x[2]) + 0.5 * L.E(x[4])) * sc[1]
                                                     + 0.25 * sc[0] * x[3]]),
    'tsde_step_srk_diag': ('eeeegggg', 1, True, _srk_final),
    'tsde_srk_additive_stage': ('eeg', 1, True,
                                lambda x, w, u, sc, L: [x[0] + 0.75 * sc[0] * x[1] + L.P(x[2], 1.5 * u * sc[1])]),
    'tsde_step_srk_additive': ('eeegg', 1, True,
                               lambda x, w, u, sc, L: [x[0] + sc[0] / 3 * x[1] + 2 * sc[0] / 3 * x[2]
                                                       + L.P(x[3], w - u * sc[1]) + L.P(x[4], u * sc[1])]),
    'tsde_linear_interp': ('ee', 1, False, lambda x, w, u, sc, L: [sc[0] * x[0] + sc[1] * x[1]]),
}
NOISE_FREE = ('tsde_milstein_gf_predict', 'tsde_srk_diag_stage1', 'tsde_srk_diag_stage3', 'tsde_linear_interp')
GENERAL_FAMILY = ('tsde_step_euler', 'tsde_midpoint_predict', 'tsde_euler_heun_predict', 'tsde_step_euler_heun',
                  'tsde_reversible_heun_z', 'tsde_step_reversible_heun', 'tsde_step_heun', 'tsde_srk_additive_stage',
                  'tsde_step_srk_additive')
# the entries a user-supplied g_prod / f_and_g_prod feeds (methods.py: _f_and_g_prod / _g_prod and the adjoint SDE's
# Milstein step), with the unit-noise launch
UNIT_FAMILY = ('tsde_step_euler', 'tsde_midpoint_predict', 'tsde_euler_heun_predict', 'tsde_step_euler_heun',
               'tsde_step_heun', 'tsde_step_milstein')


def _scalars(name, ito=1, dt=0.0625):
    """The scalar arguments methods.py passes to `name` for a step of length dt."""
    sq = math.sqrt(dt)
    return {'tsde_step_euler': (dt,), 'tsde_milstein_vjp_seed': (dt, ito), 'tsde_step_milstein': (dt,),
            'tsde_milstein_gf_predict': (dt, sq, ito), 'tsde_step_milstein_gf': (dt, 2 * sq, ito),
            'tsde_step_heun': (dt,), 'tsde_midpoint_predict': (dt / 2,), 'tsde_euler_heun_predict': (),
            'tsde_step_euler_heun': (dt,), 'tsde_reversible_heun_z': (dt,), 'tsde_step_reversible_heun': (dt / 2,),
            'tsde_srk_diag_stage1': (dt, sq), 'tsde_srk_diag_stage2': (dt, 1 / dt, sq),
            'tsde_srk_diag_stage3': (dt, sq), 'tsde_step_srk_diag': (dt, 1 / dt, sq, 3 * dt),
            'tsde_srk_additive_stage': (dt, 1 / dt), 'tsde_step_srk_additive': (dt, 1 / dt),
            'tsde_linear_interp': (0.3, 0.7)}[name]


def _cases():
    """(entry, layout, ito) for every operand layout the solvers hand the entry."""
    out = []
    for name in RESTATED:
        itos = (1, 0) if name in ('tsde_milstein_vjp_seed', 'tsde_milstein_gf_predict', 'tsde_step_milstein_gf') \
            else (1,)
        layouts = []
        if name not in ('tsde_srk_additive_stage', 'tsde_step_srk_additive'):
            layouts += [Layout('diagonal'), Layout('scalar', 1)]
        if name in GENERAL_FAMILY:
            layouts += [Layout('general', 1), Layout('general', 3), Layout('expanded', 3)]
        if name in UNIT_FAMILY:
            layouts.append(Layout('unit'))
        out += [(name, lay, ito) for lay in layouts for ito in itos]
    return out


CASES = _cases()


def _case_id(case):
    name, lay, ito = case
    return f'{name[5:]}-{lay.kind}{lay.m or ""}' + ('' if ito else '-strat')


def _operands(name, lay, gen):
    """Leaf inputs (what autograd differentiates w.r.t.), the operands the entry sees, W, U."""
    kinds, _, want_u, _ = RESTATED[name]
    m = {'diagonal': D, 'unit': D}.get(lay.kind, lay.m)
    leaves, ops = [], []
    for k in kinds:
        if k == 'e' or lay.kind in ('diagonal', 'unit'):
            x = torch.rand(ROWS, D, generator=gen, dtype=torch.float64) + 0.5
            leaves.append(x.requires_grad_(True))
            ops.append(x)
        elif lay.kind == 'expanded':
            s = (torch.rand(D, m, generator=gen, dtype=torch.float64) + 0.5).requires_grad_(True)
            leaves.append(s)
            ops.append(s.expand(ROWS, D, m))
        else:
            x = (torch.rand(ROWS, D, m, generator=gen, dtype=torch.float64) + 0.5).requires_grad_(True)
            leaves.append(x)
            ops.append(x)
    if lay.kind == 'unit':
        w = u = None
    else:
        w = torch.randn(ROWS, m, generator=gen, dtype=torch.float64) * 0.25
        u = torch.randn(ROWS, m, generator=gen, dtype=torch.float64) * 0.05 if want_u else None
    if name in NOISE_FREE:
        w = u = None
    return leaves, ops, w, u


def table_mismatches(module, cases=CASES, seed=0):
    """The cases whose table vector-Jacobian product (module.TableauFn.backward, stand-in ctx) differs from autograd of
    the restatement by more than a few ulp: a list of messages (a backward that raises counts as a mismatch)."""
    bad = []
    for i, (name, lay, ito) in enumerate(cases):
        gen = torch.Generator().manual_seed(seed * 1000 + i)
        sc = _scalars(name, ito)
        leaves, ops, w, u = _operands(name, lay, gen)
        fw = RESTATED[name][3]
        # the kernel with unit noise sees W == 1
        outs = fw(ops, 1.0 if lay.kind == 'unit' and name not in NOISE_FREE else w, u, sc, lay)
        cots = [torch.randn(o.shape, generator=gen, dtype=torch.float64) for o in outs]
        ref = torch.autograd.grad(outs, leaves, cots, allow_unused=True)
        ctx = types.SimpleNamespace(name=name, scalars=sc, noise=None if w is None else (w, u),
                                    unit=lay.kind == 'unit', use_general=lay.kind != 'unit',
                                    in_shapes=[tuple(o.shape) for o in ops])
        try:
            with torch.no_grad():
                got = module.TableauFn.backward(ctx, *cots)[7:]
        except Exception as e:  # a mutated backward may fail to broadcast
            bad.append(f'{_case_id((name, lay, ito))}: backward raised {type(e).__name__}: {e}')
            continue
        for j, (g, r, leaf) in enumerate(zip(got, ref, leaves)):
            r = torch.zeros_like(leaf) if r is None else r
            if g is None:
                bad.append(f'{_case_id((name, lay, ito))} input {j}: None')
                continue
            if lay.kind == 'expanded' and g.dim() == 3 and leaf.dim() == 2:
                g = g.sum(0)  # what autograd's expand backward does with the (rows, d, m) gradient
            scale = r.abs().max().item() + 1.0
            if g.shape != r.shape or not torch.allclose(g, r, rtol=16 * ULP, atol=16 * ULP * scale):
                err = (g - r).abs().max().item() if g.shape == r.shape else f'shape {tuple(g.shape)}'
                bad.append(f'{_case_id((name, lay, ito))} input {j}: max |table - autograd| {err}')
    return bad


# ---- the restatements are the formulas the kernels are verified against ----------------------------------------
# (the adjoint engine's halves and the Brownian queries are not autograd nodes)
@pytest.mark.parametrize('op', [op for op in NOISE_OPS + PLAIN_OPS if op[0] in RESTATED],
                         ids=lambda op: op[0][5:] + '_%d' % len(op[4]))
def test_restatement_matches_kernel_formula(op):
    name, nin, nout, want_u, scalars, formula = op
    rng = np.random.default_rng(nin)
    x = [rng.random((ROWS, D)) + 0.5 for _ in range(nin)]
    w, u = rng.standard_normal((ROWS, D)) * SQ, rng.standard_normal((ROWS, D)) * SQ
    ref = formula(x, w, u if want_u else None)
    sc = scalars
    if name == 'tsde_step_srk_diag':
        assert scalars == (DT, RDT, SQ, 3 * DT)
    got = RESTATED[name][3]([torch.from_numpy(a) for a in x], torch.from_numpy(w), torch.from_numpy(u), sc,
                            Layout('diagonal'))
    assert len(got) == nout
    for a, b in zip(got, ref):
        np.testing.assert_allclose(a.numpy(), b, rtol=1e-14, atol=1e-14)


def test_every_table_entry_is_restated():
    """Each name _table answers for has a restatement here (and a case), and nothing else."""
    names = {n for n in RESTATED}
    for n in names:
        autograd_ops._table(n, _scalars(n), torch.ones(1), torch.ones(1))
    with pytest.raises(NotImplementedError):
        autograd_ops._table('tsde_not_an_entry', (), None, None)
    src = inspect.getsource(autograd_ops._table)
    assert sorted(names) == sorted(set(re.findall(r"name == '(tsde_\w+)'", src)))
    assert {c[0] for c in CASES} == names


# ---- the table --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_table_vjp_matches_autograd_of_restatement(case):
    bad = table_mismatches(autograd_ops, [case])
    assert not bad, '\n'.join(bad)


# single-token mutations of autograd_ops.py the table test must catch: (label, source text, replacement)
MUTATIONS = [
    ('heun_g_coefficient_without_half',
     "(G, 0.5 * w), (G, 0.5 * w)]]\n    if name == 'tsde_midpoint_predict'",
     "(G, w), (G, 0.5 * w)]]\n    if name == 'tsde_midpoint_predict'"),
    ('milstein_gf_w_minus_v_as_w', "(G, w - v), (G, v)", "(G, w), (G, v)"),
    ('outer_product_transposed', "g_o.unsqueeze(-1) * c.unsqueeze(-2)", "c.unsqueeze(-1) * g_o.unsqueeze(-2)"),
    ('srk_ikk_sign_flipped', "b2[s] * ikk / sqrt_dt", "- b2[s] * ikk / sqrt_dt"),
]


def _mutant(source, new):
    text = inspect.getsource(autograd_ops)
    assert text.count(source) == 1, f'mutation site not found once in autograd_ops.py: {source!r}'
    module = types.ModuleType('autograd_ops_mutant')
    exec(compile(text.replace(source, new), 'autograd_ops_mutant', 'exec'), module.__dict__)
    return module


@pytest.mark.parametrize('label,source,new', MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_table_check_catches_mutation(label, source, new):
    assert not table_mismatches(_mutant(source, source))  # the unmutated copy passes
    assert table_mismatches(_mutant(source, new)), f'mutation {label} not detected'


# ---- the finite-difference harness on a pure-torch solve --------------------------------------------------------
def _euler_gbm(y0, mu, sigma, dW, dt):
    """Euler-Maruyama for dy = mu y dt + sigma y dW (element-wise), all outputs (T, B, d)."""
    ys = [y0]
    for k in range(dW.shape[0]):
        ys.append(ys[-1] + mu * ys[-1] * dt + sigma * ys[-1] * dW[k])
    return torch.stack(ys)


def test_harness_accepts_analytic_gradient_and_rejects_one_scaled_row():
    """The analytic gradient of a CPU Euler solve (d y_t / d y0 = prod_k (1 + mu dt + sigma dW_k)) passes both the
    per-row directional check and the full Jacobian check; the same gradient scaled by (1 + 1e-5) in one row fails
    both, in that row only."""
    B, d, n, dt = 7, 3, 6, 0.0625
    gen = torch.Generator().manual_seed(3)
    y0 = torch.rand(B, d, generator=gen, dtype=torch.float64) + 0.2
    mu = -torch.rand(d, generator=gen, dtype=torch.float64)
    sigma = torch.rand(d, generator=gen, dtype=torch.float64)
    dW = torch.randn(n, B, d, generator=gen, dtype=torch.float64) * math.sqrt(dt)
    w = torch.randn(n + 1, B, d, generator=gen, dtype=torch.float64)
    fn = lambda: _euler_gbm(y0, mu, sigma, dW, dt)  # noqa: E731

    factors = torch.cumprod(torch.cat([torch.ones(1, B, d, dtype=torch.float64), 1 + mu * dt + sigma * dW]), 0)
    grad = (w * factors).sum(0)
    wrong = grad.clone()
    wrong[4] *= 1 + 1e-5

    V = torch.randn(B, d, generator=gen, dtype=torch.float64)
    D, L = gradient_ref.rowwise_directional(fn, y0, V, w)
    assert bool(gradient_ref.within((grad * V).sum(1), D, L).all())
    ok = gradient_ref.within((wrong * V).sum(1), D, L)
    assert ok.tolist() == [r != 4 for r in range(B)]

    out, (J,) = gradient_ref.central_jacobian(fn, [y0])
    assert not gradient_ref.check_vjp(out, [J], w, [grad])
    bad = gradient_ref.check_vjp(out, [J], w, [wrong])
    assert len(bad) == 1 and any(f'element {4 * d + j}:' in bad[0] for j in range(d)), bad
    # parameters shared across rows: a plain directional check
    dmu = torch.randn(d, generator=gen, dtype=torch.float64)
    Dp, Lp = gradient_ref.directional(fn, [mu], [dmu], w)
    mu_l = mu.clone().requires_grad_(True)
    g_mu, = torch.autograd.grad((w * _euler_gbm(y0, mu_l, sigma, dW, dt)).sum(), mu_l)
    assert bool(gradient_ref.within((g_mu * dmu).sum(), Dp, Lp))
    assert not bool(gradient_ref.within((g_mu * dmu).sum() * (1 + 1e-5), Dp, Lp))
