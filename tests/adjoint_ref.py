"""Float64 restatement of the reference's generic stochastic adjoint (google-research/torchsde v0.2.6).

`sdeint_adjoint` with any adjoint method but the reversible pair integrates the continuous adjoint SDE backwards on
the flat augmented state (y, adj_y, adj_params...) with a dummy batch dimension.  Its result is that algorithm's, not
the exact gradient of the discrete forward solve, so central differences cannot check it; this module restates the
algorithm itself, in float64 on the CPU:

* `AdjointSDE`       the drift, the diffusion-vector products and the corrections on the flat state
                     (reference _core/adjoint_sde.py): none for Stratonovich and additive noise, the diagonal Ito
                     correction, the default Ito correction column by column, Milstein's `g_prod_and_gdg_prod` for
                     diagonal noise.  The vector-Jacobian products are taken with float64 torch autograd through a CPU
                     copy of the test's SDE, as `problems.NumpySDE` does for the forward oracle.
* `STEPS`            every adjoint method the reference accepts, calling `f`, `g_prod`, `f_and_g_prod` and
                     `g_prod_and_gdg_prod` as _core/methods/*.py do when the SDE only offers products; the time loop,
                     the interpolation and the adaptive controller are oracle/solvers.py's.
* `backward`         the loop of _core/adjoint.py:65-127: newest interval first, y reset to ys[i-1], grad_ys[i-1]
                     added, the parameter adjoints accumulated in the state, only `adjoint_params` differentiated.
* `Logqp`            the `logqp=True` augmentation (_core/base_sde.py SDELogqp) and `logqp_grad_ys`, the cotangent of
                     the augmented solve for a loss of (ys, log-ratio increments) (_core/sdeint.py parse_return).

Increments come from a callable `bm(ta, tb)` in forward time, as oracle/solvers.py takes them; the backward solve asks
`bm(-tb, -ta)` (ReverseBrownian, _brownian/derived.py:27-30).

`mutate` names deliberate errors, used only to show that the comparisons reject them (tests/test_host_adjoint_ref.py):
  'neighbour_dw'   every backward step gets the increment of the neighbouring step
  'milstein_v'     the Ito and Stratonovich forms of Milstein's v swapped in the Milstein adjoint
  'no_ito'         the Ito correction dropped
  'diag_columns'   the default correction's per-column products replaced by the diagonal form's single product
  'late_grad'      grad_ys[i-1] added one interval late
  'drop_params'    the parameter adjoint of the last interval [ts[-2], ts[-1]] dropped

Test infrastructure only; like oracle/ it does not import torchsde_b200.
"""
import numpy as np
import torch

from oracle import solvers

MUTATIONS = ('neighbour_dw', 'milstein_v', 'no_ito', 'diag_columns', 'late_grad', 'drop_params')


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64))


def _time(t):
    return torch.tensor(float(t), dtype=torch.float64)


def _vjp(outputs, inputs, grad_outputs=None, create_graph=False):
    """misc.vjp with allow_unused: zeros for inputs the outputs do not reach."""
    if not outputs.requires_grad:
        return [torch.zeros_like(x) for x in inputs]
    grads = torch.autograd.grad(outputs, inputs, grad_outputs, allow_unused=True, retain_graph=True,
                                create_graph=create_graph)
    return [torch.zeros_like(x) if g is None else g for g, x in zip(grads, inputs)]


def _jvp(output, inp, tangent):
    """misc.jvp: the Jacobian-vector product by the double-vjp trick, differentiable in `inp`."""
    if not output.requires_grad:
        return torch.zeros_like(output)
    dummy = torch.zeros_like(output, requires_grad=True)
    vjp, = torch.autograd.grad(output, inp, dummy, create_graph=True, allow_unused=True)
    if vjp is None or not vjp.requires_grad:
        return torch.zeros_like(output)
    out, = torch.autograd.grad(vjp, dummy, tangent, create_graph=True, retain_graph=True, allow_unused=True)
    return torch.zeros_like(output) if out is None else out


def _prod(noise_type, g, v):
    # base_sde.py:98-102
    if noise_type == 'diagonal':
        return g * v
    return torch.bmm(g, v.unsqueeze(-1)).squeeze(-1)


class Logqp(torch.nn.Module):
    """The reference's SDELogqp (base_sde.py:240-306): the state gains a last channel that integrates
    0.5 |u|^2, u = (f - h) / g (diagonal, with misc.stable_division) or pinv(g) (f - h); that channel has no noise."""

    def __init__(self, base):
        super().__init__()
        self.base = base
        self.noise_type, self.sde_type = base.noise_type, base.sde_type

    def _fgh(self, t, y):
        y = y[:, :-1]
        f, g, h = self.base.f(t, y), self.base.g(t, y), self.base.h(t, y)
        if self.noise_type == 'diagonal':
            den = torch.where(g.abs().detach() > 1e-7, g, torch.full_like(g, 1e-7) * g.sign())
            u = (f - h) / den
            g_lq = y.new_zeros(size=(y.size(0), 1))
        else:
            u = torch.bmm(g.pinverse(), (f - h).unsqueeze(-1)).squeeze(-1)
            g_lq = y.new_zeros(size=(g.size(0), 1, g.size(-1)))
        return torch.cat([f, .5 * (u ** 2).sum(dim=1, keepdim=True)], dim=1), torch.cat([g, g_lq], dim=1)

    def f(self, t, y):
        return self._fgh(t, y)[0]

    def g(self, t, y):
        return self._fgh(t, y)[1]


def logqp_grad_ys(ys_aug, wy, wl):
    """Cotangent of the augmented solve ys_aug (T, B, d + 1) for the loss sum(wy * ys) + sum(wl * log-ratio
    increments), through the reference's parse_return."""
    ys = _t(ys_aug).requires_grad_()
    y, lr = ys.split((ys.size(2) - 1, 1), dim=2)
    inc = torch.stack([b - a for b, a in zip(lr[1:], lr[:-1])], dim=0).squeeze(dim=2)
    ((y * _t(wy)).sum() + (inc * _t(wl)).sum()).backward()
    return ys.grad.numpy()


class AdjointSDE:
    """adjoint_sde.py:23-377 on numpy (1, N) states: `module` is the forward SDE on the CPU in float64, `params` the
    adjoint parameters (tensors of that module), `shapes` those of (y, adj_y, *params)."""

    def __init__(self, module, params, shapes, mutate=()):
        self.fwd = module
        self.params = list(params)
        self.shapes = [tuple(s) for s in shapes]
        self.numels = [int(np.prod(s)) for s in self.shapes]
        self.mutate = frozenset(mutate)
        self.fwd_noise = module.noise_type
        self.sde_type = module.sde_type
        self.noise_type = {'additive': 'general'}.get(module.noise_type, module.noise_type)   # :33-38
        ito = module.sde_type == 'ito'
        if not ito or self.fwd_noise == 'additive' or 'no_ito' in self.mutate:                  # :48-56
            self.correction = None
        elif self.fwd_noise == 'diagonal':
            self.correction = 'diagonal'
        else:
            self.correction = 'default'

    def _state(self, y_aug):
        flat = _t(y_aug).reshape(-1)
        n0, n1 = self.numels[:2]
        y = flat[:n0].reshape(self.shapes[0]).clone().requires_grad_()
        adj_y = flat[n0:n0 + n1].reshape(self.shapes[1]).clone()
        return y, adj_y

    @staticmethod
    def _flat(parts):
        return torch.cat([p.detach().reshape(-1) for p in parts]).unsqueeze(0).numpy().copy()

    # ---- drift (:111-216) --------------------------------------------------------------------------------------
    def _drift(self, f, g, y, adj_y):
        inputs = [y] + self.params
        if self.correction == 'diagonal':
            g_dg, = _vjp(g, [y], g, create_graph=True)
            f = f - g_dg
            vjps = _vjp(f, inputs, adj_y)
            a_dg, = _vjp(g, [y], adj_y)
            vjps = [a + b for a, b in zip(vjps, _vjp(g, inputs, a_dg))]
        elif self.correction == 'default':
            cols = [c.squeeze(dim=-1) for c in g.split(1, dim=-1)]
            f = f - sum(_jvp(c, y, c) for c in cols)
            vjps = _vjp(f, inputs, adj_y)
            if 'diag_columns' in self.mutate:
                a_dg, = _vjp(g, [y], adj_y.unsqueeze(-1).expand_as(g))
                vjps = [a + b for a, b in zip(vjps, _vjp(g, inputs, a_dg.unsqueeze(-1).expand_as(g)))]
            else:
                for c in cols:
                    a_dg, = _vjp(c, [y], adj_y)
                    vjps = [a + b for a, b in zip(vjps, _vjp(c, inputs, a_dg))]
        else:
            vjps = _vjp(f, inputs, adj_y)
        return self._flat([-f] + vjps)

    def _diffusion(self, g_prod, y, adj_y):
        return self._flat([-g_prod] + _vjp(g_prod, [y] + self.params, adj_y))   # :218-230

    def f(self, t, y_aug):
        y, adj_y = self._state(y_aug)
        t = _time(-t)
        with torch.enable_grad():
            if self.correction is None:
                return self._drift(self.fwd.f(t, y), None, y, adj_y)
            return self._drift(self.fwd.f(t, y), self.fwd.g(t, y), y, adj_y)

    def g_prod(self, t, y_aug, v):
        y, adj_y = self._state(y_aug)
        with torch.enable_grad():
            return self._diffusion(_prod(self.fwd_noise, self.fwd.g(_time(-t), y), _t(v)), y, adj_y)

    def f_and_g_prod(self, t, y_aug, v):
        y, adj_y = self._state(y_aug)
        t = _time(-t)
        with torch.enable_grad():
            f, g = self.fwd.f(t, y), self.fwd.g(t, y)
            g_prod = _prod(self.fwd_noise, g, _t(v))
            return self._drift(f, g, y, adj_y), self._diffusion(g_prod, y, adj_y)

    def g_prod_and_gdg_prod(self, t, y_aug, v1, v2):
        """:332-377 (diagonal noise; the reference raises NotImplementedError for the others)."""
        if self.fwd_noise != 'diagonal':
            raise NotImplementedError
        y, adj_y = self._state(y_aug)
        v2 = _t(v2)
        inputs = [y] + self.params
        with torch.enable_grad():
            g = self.fwd.g(_time(-t), y)
            g_prod = g * _t(v1)
            vg_dg, = _vjp(g, [y], v2 * g)
            dgdy, = _vjp(g.sum(), [y], None, create_graph=True)
            prod_partials = _vjp(g, inputs, adj_y * v2 * dgdy)
            avg_dg, = _vjp(g, [y], (adj_y * v2 * g).detach(), create_graph=True)
            mixed_partials = _vjp(avg_dg.sum(), inputs, None)
            vjps = [a - b for a, b in zip(prod_partials, mixed_partials)]
            return self._diffusion(g_prod, y, adj_y), self._flat([vg_dg] + vjps)


# ---- the solvers' steps through the product protocol (methods/*.py) ----------------------------------------------
def _sc(x):
    return np.float64(x)


class Euler(solvers.Solver):
    # methods/euler.py:29-37
    def step(self, t0, t1, y0, extra0):
        dt = t1 - t0
        I_k = self.bm(t0, t1)
        f, g_prod = self.sde.f_and_g_prod(t0, y0, I_k)
        return y0 + f * _sc(dt) + g_prod, ()


class Milstein(solvers.Solver):
    # methods/milstein.py:52-94, derivative-using (grad_free is refused for adjoint SDEs, :34-40)
    def step(self, t0, t1, y0, extra0):
        dt = t1 - t0
        I_k = self.bm(t0, t1)
        ito = (self.sde.sde_type == 'ito') != ('milstein_v' in self.sde.mutate)
        v = I_k ** 2 - _sc(dt) if ito else I_k ** 2
        f = self.sde.f(t0, y0)
        g_prod, gdg_prod = self.sde.g_prod_and_gdg_prod(t0, y0, I_k, _sc(0.5) * v)
        return y0 + f * _sc(dt) + g_prod + gdg_prod, ()


class Midpoint(solvers.Solver):
    # methods/midpoint.py:29-45
    def step(self, t0, t1, y0, extra0):
        dt = t1 - t0
        I_k = self.bm(t0, t1)
        f, g_prod = self.sde.f_and_g_prod(t0, y0, I_k)
        half_dt = np.asarray(dt).dtype.type(0.5 * dt)
        t_prime = t0 + half_dt
        y_prime = y0 + _sc(half_dt) * f + _sc(0.5) * g_prod
        f_prime, g_prod_prime = self.sde.f_and_g_prod(t_prime, y_prime, I_k)
        return y0 + _sc(dt) * f_prime + g_prod_prime, ()


class Heun(solvers.Solver):
    # methods/heun.py:35-48
    def step(self, t0, t1, y0, extra0):
        dt = _sc(t1 - t0)
        I_k = self.bm(t0, t1)
        f, g_prod = self.sde.f_and_g_prod(t0, y0, I_k)
        y0_prime = y0 + dt * f + g_prod
        f_prime, g_prod_prime = self.sde.f_and_g_prod(t1, y0_prime, I_k)
        return y0 + (dt * (f + f_prime) + g_prod + g_prod_prime) * _sc(0.5), ()


class EulerHeun(solvers.Solver):
    # methods/euler_heun.py:29-42
    def step(self, t0, t1, y0, extra0):
        dt = _sc(t1 - t0)
        I_k = self.bm(t0, t1)
        f, g_prod = self.sde.f_and_g_prod(t0, y0, I_k)
        y_prime = y0 + g_prod
        g_prod_prime = self.sde.g_prod(t1, y_prime, I_k)
        return y0 + dt * f + (g_prod + g_prod_prime) * _sc(0.5), ()


STEPS = {'euler': Euler, 'milstein': Milstein, 'midpoint': Midpoint, 'heun': Heun, 'euler_heun': EulerHeun}


def _neighbour(bm, lo, hi):
    """`bm` serving each query the increment of the step of the same length next to it (the one before at the end
    of [lo, hi])."""
    def query(ta, tb, return_U=False):
        h = tb - ta
        if tb + h <= hi:
            return bm(ta + h, tb + h)
        return bm(ta - h, tb - h)
    return query


def backward(module, params, ys, ts, grad_ys, adjoint_method, dt, bm, adaptive=None, mutate=()):
    """adjoint.py:65-127 for a generic adjoint_method: returns (adj_y0, [adj_param...], n_proposals).

    module    forward SDE (CPU, float64; `Logqp` for logqp=True), params: its adjoint parameters;
    ys        (T, B, d) float64 forward solution, ts: numpy output times in ts' dtype, grad_ys: (T, B, d) cotangent;
    bm        forward-time increments bm(ta, tb) -> (B, m) float64;
    adaptive  None, or dict(rtol=, atol=, dt_min=) for adjoint_adaptive=True (base_solver.py:117-142)."""
    mutate = frozenset(mutate)
    ys, grad_ys = np.asarray(ys, np.float64), np.asarray(grad_ys, np.float64)
    ts = np.asarray(ts)
    shapes = [ys.shape[1:], ys.shape[1:]] + [tuple(p.shape) for p in params]
    numels = [int(np.prod(s)) for s in shapes]
    sde = AdjointSDE(module, params, shapes, mutate)
    fwd_bm = _neighbour(bm, float(ts[0]), float(ts[-1])) if 'neighbour_dw' in mutate else bm

    def reverse_bm(ta, tb, return_U=False):
        return fwd_bm(-tb, -ta)

    solver = STEPS[adjoint_method](sde, reverse_bm, dt)
    parts = [ys[-1], grad_ys[-1]] + [np.zeros(s) for s in shapes[2:]]
    pending = None
    n_prop = 0
    for i in range(len(ts) - 1, 0, -1):
        aug = np.concatenate([p.reshape(-1) for p in parts])[None]
        span = np.array([-ts[i], -ts[i - 1]], dtype=ts.dtype)
        if adaptive is None:
            out, _ = solver.integrate(aug, span)
        else:
            out, _, n = solvers.integrate_adaptive(solver, aug, span, adaptive['rtol'], adaptive['atol'],
                                                   adaptive['dt_min'])
            n_prop += n
        flat = out[-1][0]
        parts = [flat[a:a + n].reshape(s) for a, n, s in zip(np.cumsum([0] + numels[:-1]), numels, shapes)]
        if 'drop_params' in mutate and i == len(ts) - 1:
            parts[2:] = [np.zeros_like(p) for p in parts[2:]]
        parts[0] = ys[i - 1]
        if 'late_grad' in mutate:
            if pending is not None:
                parts[1] = parts[1] + pending
            pending = grad_ys[i - 1]
        else:
            parts[1] = parts[1] + grad_ys[i - 1]
    if pending is not None:
        parts[1] = parts[1] + pending
    return parts[1], parts[2:], n_prop


def forward(module, y0, ts, method, dt, bm, options=None):
    """The forward solve the adjoint starts from: oracle/solvers.py on the same increments."""
    from . import problems
    ys, _ = solvers.make(method, problems.NumpySDE(module), bm, dt, options or {}).integrate(
        np.asarray(y0, np.float64), np.asarray(ts))
    return ys


# ---- what sdeint_adjoint accepts, and the comparison every test uses --------------------------------------------------
# (sde_type, forward method, forward options, adjoint method, noise kinds of tests/problems.py): every generic pair the
# reference runs forward and backward (tests/test_host_adjoint_ref.py checks this list against the live reference).
# srk refuses adjoint SDEs, log_ode needs a Levy area the default Brownian motion lacks, and Milstein's adjoint
# products exist for diagonal noise only.
_ALL = ('gbm', 'scalar', 'additive', 'general')
_FWD = {'ito': [('euler', None, _ALL), ('milstein', None, ('gbm', 'scalar', 'additive')),
                ('milstein', {'grad_free': True}, ('gbm', 'scalar', 'additive')),
                ('srk', None, ('gbm', 'scalar', 'additive'))],
        'stratonovich': [('midpoint', None, _ALL), ('heun', None, _ALL), ('euler_heun', None, _ALL),
                         ('milstein', None, ('gbm', 'scalar', 'additive')),
                         ('milstein', {'grad_free': True}, ('gbm', 'scalar', 'additive')),
                         ('reversible_heun', None, _ALL)]}
_ADJ = {'ito': [('euler', _ALL), ('milstein', ('gbm',))],
        'stratonovich': [('midpoint', _ALL), ('heun', _ALL), ('euler_heun', _ALL), ('milstein', ('gbm',))]}
PAIRS = [(st, method, opts, adj, kind)
         for st in ('ito', 'stratonovich') for method, opts, kinds in _FWD[st] for adj, adj_kinds in _ADJ[st]
         for kind in kinds if kind in adj_kinds]


def default_adjoint_method(sde_type, noise_type):
    """adjoint.py:281-296 for a non-reversible forward method."""
    if sde_type == 'ito':
        return 'milstein' if noise_type == 'diagonal' else 'euler'
    return 'midpoint'


def pair_id(pair):
    st, method, opts, adj, kind = pair
    return f"{st[:5]}-{method}{'_gf' if opts else ''}-{adj}-{kind}"


# float64: a float64 solve follows the reference's operation order, so it differs from this restatement only by the
# rounding of its reductions and of libm; over these short solves (<= 100 steps, tens of rounded operations per element
# and step) that is below 1e-12 of the output's scale.  RTOL64 = 1e-9 leaves three orders of magnitude for it, as the
# other oracle comparisons of the suite do, and still rejects every error the mutations above introduce.
RTOL64 = 1e-9


def scale(ref):
    return max(float(np.max(np.abs(ref))), 1e-300)


def excess(got, ref, bound):
    """Elementwise |got - ref| / bound (bound: a scalar or an array)."""
    return np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)) / bound
