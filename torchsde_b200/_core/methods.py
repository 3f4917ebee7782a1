"""The step tableaus, as host-side drivers of the fused CUDA kernels.

One class per method of the reference (torchsde/_core/methods/*.py), with the same class
attributes (strong/weak order, sde_type, noise_types, levy_area_approximations) and the same
constructor-time errors; ``select`` mirrors methods/__init__.py:26-48.  Each ``_step`` issues the
user's drift/diffusion calls in the reference's order and replaces the ATen arithmetic of the
reference's ``step`` by one or two launches through the C ABI (include/torchsde_b200.h), issued via
``self._k(name, L, nz, inputs, scalars, outputs)`` (base_solver.py) — a direct launch on the fast path,
an autograd node when gradients must flow through the solve.
"""

import numpy as np
import torch

from . import base_solver
from . import pointwise
from .base_sde import widen
from .base_solver import _contig, _gop
from .. import _cabi
from ..settings import SDE_TYPES, NOISE_TYPES, LEVY_AREA_APPROXIMATIONS, METHODS, METHOD_OPTIONS



def _ieee_sqrt(dt):
    """sqrt of a 0-d CPU tensor, correctly rounded in its dtype.  The reference writes `dt.sqrt()` on a tensor that lives
    on the solve's device — on a GPU that is the IEEE square root.  PyTorch's *CPU* sqrt kernel is not correctly rounded
    on AVX-512 builds (about 1 % of inputs come out one ulp off, e.g. sqrt(2^-5) in fp64), so evaluating the same
    expression on the host would make SRK / derivative-free Milstein depend on the host's vector ISA; numpy's sqrt is the
    hardware instruction."""
    return torch.tensor(np.sqrt(dt.detach().numpy()), dtype=dt.dtype)

class _WidenedSDE:
    """The callables an SRK step with a user g_prod computes on in torch, returning 16-bit outputs widened."""

    def __init__(self, sde, dtype):
        self._sde, self._dtype = sde, dtype

    def f(self, t, y):
        return widen(self._sde.f(t, y), self._dtype)

    def g(self, t, y):
        return widen(self._sde.g(t, y), self._dtype)

    def g_prod(self, t, y, v):
        return widen(self._sde.g_prod(t, y, v), self._dtype)


class _ProposalMixin:
    """An adaptive solve's proposals as one kernel each (pointwise.propose) once the first one has recorded the SDE's
    element-wise program; `_proposal` is the method's TSDE_PROPOSAL_*."""
    _proposal = None

    def _propose(self, curr_t, next_t, midpoint_t, curr_y, curr_extra):
        if pointwise.proposing(self):
            return pointwise.propose(self, self._proposal, curr_t, next_t, midpoint_t, curr_y) + (curr_extra,)
        return super()._propose(curr_t, next_t, midpoint_t, curr_y, curr_extra)


class _ProdMixin:
    """Shared handling of the reference's `f_and_g_prod` / `g_prod` call sites (base_sde.py:51-56)."""

    def _f_and_g_prod(self, c, t, y, rec=None):
        """Evaluate drift and diffusion at (t, y) the way ForwardSDE.f_and_g_prod would.  Returns
        (L, nz, f, g) where (L, nz, g) is either (noise-type launch, step noise, g) or
        (element-wise launch, unit noise, user-computed g_prod).  `rec` (pointwise.pc_recorder) records f and g."""
        sde = self.sde
        mode = sde.f_and_g_prod_mode
        if mode == 'fused':
            if rec is not None:
                f, g = self._fork(lambda: rec.evaluation('f', lambda: sde.f(t, y), t, y),
                                  lambda: rec.evaluation('g', lambda: sde.g(t, y), t, y))
            else:
                f, g = self._f_and_g(t, y)
            return self._L, self._feed.get(c, self.want_u), _contig(f), _gop(g)
        w, _ = self._feed.tensors(c)
        w = w.reshape(self.bm.shape)
        if mode == 'f_and_g_prod':
            f, gp = sde.f_and_g_prod(t, y, w)
        else:
            f, gp = sde.f(t, y), sde.g_prod(t, y, w)
        return self._LU, self._feed.unit(), _contig(f), _contig(gp)

    def _g_prod(self, c, t, y, rec=None):
        sde = self.sde
        if sde.g_prod_mode == 'fused':
            g = rec.evaluation('g', lambda: sde.g(t, y), t, y) if rec is not None else sde.g(t, y)
            return self._L, self._feed.get(c, self.want_u), _gop(g)
        w, _ = self._feed.tensors(c)
        return self._LU, self._feed.unit(), _contig(sde.g_prod(t, y, w.reshape(self.bm.shape)))


class Euler(_ProposalMixin, _ProdMixin, base_solver.BaseSDESolver):
    """methods/euler.py:19-37."""
    _proposal = _cabi.PROPOSAL_EULER
    weak_order = 1.0
    sde_type = SDE_TYPES.ito
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    _pw_method = 'euler'
    _pw_general = True  # general / additive noise fuses too (pointwise.general)
    _pw_layout = _cabi.PW_LAYOUT_GENERAL

    def __init__(self, sde, **kwargs):
        self.strong_order = 1.0 if sde.noise_type == NOISE_TYPES.additive else 0.5
        super(Euler, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected

    def _chunks_ready(self):
        return pointwise.ready(self)

    def _step_chunk(self, ctxs, y0, extra0, outs):
        # the recorded element-wise programs (pointwise.py), several steps per kernel with the state in registers
        return pointwise.solve_chunk(self, ctxs, y0, outs, 'euler'), ()

    def _step(self, c, y0, extra0, out):
        if pointwise.ready(self):
            # a single step is a chunk of one
            return self._step_chunk([c], y0, extra0, [out if out is not None else torch.empty_like(y0)])
        # the first step of an eligible solve runs as always, with the user's two evaluations recorded
        rec = pointwise.pc_recorder(self, y0, c.t0, 'fg')
        L, nz, f, g = self._f_and_g_prod(c, c.t0, y0, rec)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_euler', L, nz, (y0, f, g), (c.dt,), out), ()


class BaseMilstein(_ProposalMixin, _ProdMixin, base_solver.BaseSDESolver):
    """methods/milstein.py:22-74."""
    strong_order = 1.0
    weak_order = 1.0
    noise_types = (NOISE_TYPES.additive, NOISE_TYPES.diagonal, NOISE_TYPES.scalar)
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()
    ito = None
    _pw_method = 'milstein'

    def __init__(self, sde, options, **kwargs):
        # milstein.py:29-41
        if METHOD_OPTIONS.grad_free not in options:
            options[METHOD_OPTIONS.grad_free] = False
        if options[METHOD_OPTIONS.grad_free]:
            if sde.noise_type == NOISE_TYPES.additive:
                options[METHOD_OPTIONS.grad_free] = False
        if options[METHOD_OPTIONS.grad_free]:
            if getattr(sde, 'is_adjoint_sde', False):
                raise ValueError(f"Derivative-free Milstein cannot be used for adjoint SDEs, because it requires "
                                 f"direct access to the diffusion, whilst adjoint SDEs rely on a more efficient "
                                 f"diffusion-vector product. Use derivative-using Milstein instead: "
                                 f"`adjoint_options=dict({METHOD_OPTIONS.grad_free}=False)`")
        super(BaseMilstein, self).__init__(sde=sde, options=options, **kwargs)
        self._ones = None
        self._pw = None  # the element-wise program of the step (pointwise.py), False once rejected

    def scalars(self, dt):
        sqrt_dt = _ieee_sqrt(dt)
        return {'sqrt_dt': float(sqrt_dt), 'two_sqrt_dt': float(2 * sqrt_dt)}

    def _chunks_ready(self):
        return pointwise.ready(self)

    def _step_chunk(self, ctxs, y0, extra0, outs):
        # the recorded element-wise program (pointwise.py), several steps per kernel with the state in registers
        return pointwise.solve_chunk(self, ctxs, y0, outs, 'milstein', ito=1 if self.ito else 0), ()

    def _step(self, c, y0, extra0, out):
        sde = self.sde
        ito = 1 if self.ito else 0
        if self.options[METHOD_OPTIONS.grad_free]:
            # milstein.py:58-67
            f, g = self._f_and_g(c.t0, y0)
            f, g = _contig(f), _contig(g)
            yp = self._k('tsde_milstein_gf_predict', self._LU, None, (y0, f, g), (c.dt, c.scalars['sqrt_dt'], ito),
                         None)
            g_prime = _contig(sde.g(c.t0, yp))
            return self._k('tsde_step_milstein_gf', self._L, self._feed.get(c), (y0, f, g, g_prime),
                           (c.dt, c.scalars['two_sqrt_dt'], ito), out), ()
        if getattr(sde, 'is_adjoint_sde', False):
            # adjoint SDE: it forms g.v and Milstein's correction itself (adjoint_sde.py:332-377);
            # v2 = 0.5 v is produced by the seed kernel applied to a tensor of ones
            f = _contig(sde.f(c.t0, y0))
            w, _ = self._feed.tensors(c)
            if self._ones is None or self._ones.shape != w.shape:
                self._ones = torch.ones_like(w)
            v2 = self._k('tsde_milstein_vjp_seed', self._LB, self._feed.from_tensors(w), (self._ones,), (c.dt, ito),
                         None, raw=True)
            gp, gdg = sde.g_prod_and_gdg_prod(c.t0, y0, w.reshape(self.bm.shape), v2.reshape(self.bm.shape))
            return self._k('tsde_step_milstein', self._LU, self._feed.unit(), (y0, f, _contig(gp), _contig(gdg)),
                           (c.dt,), out), ()
        if sde.noise_type == NOISE_TYPES.additive:
            f = _contig(sde.f(c.t0, y0))
            # g_prod_and_gdg_prod_additive: (g_prod(t, y, v1), 0.)  base_sde.py:157-158
            L, nz, g = self._g_prod(c, c.t0, y0)
            return self._k('tsde_step_euler', L, nz, (y0, f, g), (c.dt,), out), ()
        # g_prod_and_gdg_prod_{diagonal,default}: vjp of g wrt y with grad_outputs g * (0.5 v)
        # base_sde.py:127-155 (always calls self.g, never g_prod)
        if pointwise.ready(self):
            # f, g and the vjp were recorded as an element-wise program (pointwise.py): the whole step is one kernel
            return pointwise.launch(self, 'tsde_step_milstein_pointwise', self._feed.get(c), y0,
                                    (c.t0.data_ptr(), c.dt, ito), out), ()
        track = self._autograd
        # the first step of an eligible solve runs as always, with the user's ops recorded
        rec = pointwise.Recorder(y0, c.t0, pointwise.transcendental(self)) if pointwise.recording(self) else None
        raw = {}

        def user(name, fn, **kw):
            raw[name] = rec.segment(fn, **kw) if rec is not None else fn()
            return raw[name]

        def diffusion_chain():
            with torch.enable_grad():
                y = y0 if (track and y0.requires_grad) else y0.detach().requires_grad_(True)
                g = user('g', lambda: sde.g(c.t0, y), y=y)
                gd = _contig(g if track else g.detach())
                go = self._k('tsde_milstein_vjp_seed', self._L, self._feed.get(c), (gd,), (c.dt, ito), None)
                if g.requires_grad:
                    gdg, = user('gdg', lambda: torch.autograd.grad(g, y, grad_outputs=go.view_as(g), allow_unused=True,
                                                                   retain_graph=track, create_graph=track), go=go)
                else:
                    gdg = None
            return gd, (torch.zeros_like(y0) if gdg is None else _contig(gdg))

        # f and the chain g -> seed -> vjp are independent given y0 (reference order: f first, milstein.py:68)
        f, (gd, gdg) = self._fork(lambda: _contig(user('f', lambda: sde.f(c.t0, y0))), diffusion_chain, main=1)
        if rec is not None:
            res = rec.finish(raw['f'], raw['g'], raw.get('gdg', (None,))[0])
            self._pw = pointwise.compile_milstein(rec, res, self.adaptive) or False
        return self._k('tsde_step_milstein', self._L, self._feed.get(c), (y0, f, gd, gdg), (c.dt,), out), ()


class MilsteinIto(BaseMilstein):
    sde_type = SDE_TYPES.ito
    ito = True
    _proposal = _cabi.PROPOSAL_MILSTEIN_ITO


class MilsteinStratonovich(BaseMilstein):
    sde_type = SDE_TYPES.stratonovich
    ito = False
    _proposal = _cabi.PROPOSAL_MILSTEIN_STRATONOVICH


class Heun(_ProposalMixin, _ProdMixin, base_solver.BaseSDESolver):
    """methods/heun.py:25-48."""
    _proposal = _cabi.PROPOSAL_HEUN
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    def __init__(self, sde, **kwargs):
        self.strong_order = 0.5 if sde.noise_type == NOISE_TYPES.general else 1.0
        super(Heun, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected

    def _step(self, c, y0, extra0, out):
        if pointwise.ready(self):
            # f and g were recorded as element-wise programs (pointwise.py): the whole step is one kernel
            return pointwise.launch(self, 'tsde_step_predictor_corrector_pointwise', self._feed.get(c), y0,
                                    (c.t0.data_ptr(), c.t1.data_ptr(), _cabi.PC_HEUN, c.dt, 0.0), out), ()
        # the first step of an eligible solve runs as always, with the user's four evaluations recorded
        rec = pointwise.pc_recorder(self, y0, c.t0, 'fgfg')
        L, nz, f, g = self._f_and_g_prod(c, c.t0, y0, rec)
        yp = self._k('tsde_step_euler', L, nz, (y0, f, g), (c.dt,), None)
        L, nz, fp, gp = self._f_and_g_prod(c, c.t1, yp, rec)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_heun', L, nz, (y0, f, fp, g, gp), (c.dt,), out), ()


class Midpoint(_ProposalMixin, _ProdMixin, base_solver.BaseSDESolver):
    """methods/midpoint.py:19-45."""
    _proposal = _cabi.PROPOSAL_MIDPOINT
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    _pw_general = True  # general / additive noise fuses too (pointwise.general)
    _pw_layout = _cabi.PW_LAYOUT_GENERAL

    def __init__(self, sde, **kwargs):
        self.strong_order = 0.5 if sde.noise_type == NOISE_TYPES.general else 1.0
        super(Midpoint, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected

    def aux_times(self, t0, t1, dt):
        return [t0 + 0.5 * dt]  # t_prime = t0 + half_dt, midpoint.py:35-37

    def scalars(self, dt):
        return {'half_dt': float(0.5 * dt)}

    def _step(self, c, y0, extra0, out):
        if pointwise.ready(self):
            # f and g were recorded as element-wise programs (pointwise.py): the whole step is one kernel (for
            # general / additive noise, on the solver's GENERAL launch)
            return pointwise.launch(self, 'tsde_step_predictor_corrector_pointwise', self._feed.get(c), y0,
                                    (c.t0.data_ptr(), c.aux_t[0].data_ptr(), _cabi.PC_MIDPOINT, c.dt,
                                     c.scalars['half_dt']), out), ()
        # the first step of an eligible solve runs as always, with the user's four evaluations recorded
        rec = pointwise.pc_recorder(self, y0, c.t0, 'fgfg')
        L, nz, f, g = self._f_and_g_prod(c, c.t0, y0, rec)
        yp = self._k('tsde_midpoint_predict', L, nz, (y0, f, g), (c.scalars['half_dt'],), None)
        L, nz, fp, gp = self._f_and_g_prod(c, c.aux_t[0], yp, rec)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_euler', L, nz, (y0, fp, gp), (c.dt,), out), ()


class EulerHeun(_ProposalMixin, _ProdMixin, base_solver.BaseSDESolver):
    """methods/euler_heun.py:19-42."""
    _proposal = _cabi.PROPOSAL_EULER_HEUN
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    _pw_general = True  # general / additive noise fuses too (pointwise.general)
    _pw_layout = _cabi.PW_LAYOUT_GENERAL_EULER_HEUN

    def __init__(self, sde, **kwargs):
        self.strong_order = 0.5 if sde.noise_type == NOISE_TYPES.general else 1.0
        super(EulerHeun, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected

    def _step(self, c, y0, extra0, out):
        sde = self.sde
        if pointwise.ready(self):
            # f and g were recorded as element-wise programs (pointwise.py): the whole step is one kernel (for
            # general / additive noise, on the solver's GENERAL launch)
            return pointwise.launch(self, 'tsde_step_predictor_corrector_pointwise', self._feed.get(c), y0,
                                    (c.t0.data_ptr(), c.t1.data_ptr(), _cabi.PC_EULER_HEUN, c.dt, 0.0), out), ()
        # the first step of an eligible solve runs as always, with the user's three evaluations recorded
        rec = pointwise.pc_recorder(self, y0, c.t0, 'fgg')
        L, nz, f, g = self._f_and_g_prod(c, c.t0, y0, rec)
        unit = L is self._LU
        yp = self._k('tsde_euler_heun_predict', L, nz, (y0, g), (), None)
        if unit:
            # first product came from the user's (f_and_)g_prod; the reference then calls sde.g_prod (:38)
            w, _ = self._feed.tensors(c)
            w = w.reshape(self.bm.shape)
            if sde.user_g_prod:
                gp = sde.g_prod(c.t1, yp, w)
            elif not hasattr(sde._base_sde, 'g'):
                # (deliberate superset of the reference, which raises "Method `g` has not been provided" here: an SDE
                # that only offers the fused callable still solves — same value)
                gp = sde.f_and_g_prod(c.t1, yp, w)[1]
            else:
                # f_and_g_prod and g, no g_prod: the reference's second product is g_prod_default =
                # prod(g(t1, y'), dW) (euler_heun.py:38, base_sde.py:108-109).  The first product is already a tensor,
                # so form the second one as a tensor too: 0 + g(t1, y').dW in the predictor kernel (adding to an
                # exact zero does not round).
                g1 = _contig(sde.g(c.t1, yp))
                gp = self._k('tsde_euler_heun_predict', self._L, self._feed.get(c), (torch.zeros_like(y0), g1), (),
                             None)
            L2, nz2, gp = self._LU, self._feed.unit(), _contig(gp)
        else:
            L2, nz2, gp = self._g_prod(c, c.t1, yp, rec)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_euler_heun', L2, nz2, (y0, f, g, gp), (c.dt,), out), ()


class ReversibleHeun(base_solver.BaseSDESolver):
    """methods/reversible_heun.py:48-73."""
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    _pw_method = 'reversible_heun'
    _pw_general = True  # general / additive noise fuses too (pointwise.general)
    _pw_layout = _cabi.PW_LAYOUT_GENERAL_REVERSIBLE_HEUN

    def __init__(self, sde, **kwargs):
        self.strong_order = 1.0 if sde.noise_type == NOISE_TYPES.additive else 0.5
        super(ReversibleHeun, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected
        self._halves = False  # per solve: pointwise.halves_exactly of its steps
        self._pw_state = None  # per solve: the two alternating (f, g, z) sets the chunks store their state to

    def scalars(self, dt):
        return {'half_dt': float(0.5 * dt)}

    def init_extra_solver_state(self, t0, y0):
        return self.sde.f_and_g(t0, y0) + (y0,)

    def _run(self, sched, ctxs, ys, extra):
        self._halves = pointwise.halves_exactly(self.dtype, ctxs)
        self._pw_state = None  # allocated at the solve's first chunk (under capture, from the graph's pool)
        return super()._run(sched, ctxs, ys, extra)

    def _chunks_ready(self):
        return self._halves and pointwise.ready(self)

    def _step_chunk(self, ctxs, y0, extra0, outs):
        state = tuple(_contig(x) for x in extra0)
        if not pointwise.state_fits(self, state):
            # a state the kernel cannot read (a captured solve starts from the caller's): the ordinary steps
            y1 = y0
            for c, out in zip(ctxs, outs):
                y1, extra0 = self._unfused_step(c, y1, extra0, out)
            return y1, extra0
        if self._pw_state is None:
            # (f, g, z); a general- or additive-noise g is (rows, d, m)
            g_shape = tuple(state[1].shape)
            self._pw_state = [(torch.empty_like(y0), y0.new_empty(g_shape), torch.empty_like(y0)) for _ in range(2)]
        # the recorded element-wise programs (pointwise.py), several steps per kernel with y, z, f and g in registers;
        # the chunk stores its state to the set it does not read
        a, b = self._pw_state
        f1, g1, z1 = b if state[0] is a[0] else a
        f0, g0, z0 = state
        y1 = pointwise.solve_chunk(self, ctxs, y0, outs, 'reversible_heun', state=((z0, f0, g0), (z1, f1, g1)))
        return y1, (f1, g1, z1)

    def _step(self, c, y0, extra0, out):
        if self._chunks_ready():
            # a single step is a chunk of one
            return self._step_chunk([c], y0, extra0, [out if out is not None else torch.empty_like(y0)])
        return self._unfused_step(c, y0, extra0, out)

    def _unfused_step(self, c, y0, extra0, out):
        sde = self.sde
        f0, g0, z0 = (_contig(x) for x in extra0)
        z1 = self._k('tsde_reversible_heun_z', self._L, self._feed.get(c), (y0, z0, f0, g0), (c.dt,), None)
        # the first step of an eligible solve runs as always, with the user's f and g at (t1, z1) recorded
        rec = None
        if self._halves and pointwise.state_fits(self, (f0, g0, z0)):
            rec = pointwise.pc_recorder(self, z1, c.t1, 'fg')
        if rec is not None:
            f1, g1 = self._fork(lambda: rec.evaluation('f', lambda: sde.f(c.t1, z1), c.t1, z1),
                                lambda: rec.evaluation('g', lambda: sde.g(c.t1, z1), c.t1, z1))
            self._pw = pointwise.finish(self, rec)
        else:
            f1, g1 = self._f_and_g(c.t1, z1)
        f1, g1 = _contig(f1), _contig(g1)
        y1 = self._k('tsde_step_reversible_heun', self._L, self._feed.get(c), (y0, f0, f1, g0, g1),
                     (c.scalars['half_dt'],), out)
        return y1, (f1, g1, z1)


class SRK(_ProposalMixin, base_solver.BaseSDESolver):
    """methods/srk.py:31-111 (srid2 for diagonal/scalar noise, sra1 for additive noise)."""
    _proposal = _cabi.PROPOSAL_SRK
    strong_order = 1.5
    weak_order = 1.5
    sde_type = SDE_TYPES.ito
    noise_types = (NOISE_TYPES.additive, NOISE_TYPES.diagonal, NOISE_TYPES.scalar)
    levy_area_approximations = (LEVY_AREA_APPROXIMATIONS.space_time,
                                LEVY_AREA_APPROXIMATIONS.davie,
                                LEVY_AREA_APPROXIMATIONS.foster)
    want_u = True
    _pw_general = True  # additive noise fuses too (pointwise.general)
    _pw_layout = _cabi.PW_LAYOUT_GENERAL_SRA

    def __init__(self, sde, **kwargs):
        if getattr(sde, 'is_adjoint_sde', False):
            raise ValueError("Stochastic Runge–Kutta methods cannot be used for adjoint SDEs, because it requires "
                             "direct access to the diffusion, whilst adjoint SDEs rely on a more efficient "
                             "diffusion-vector product. Use a different method instead.")
        self._additive = sde.noise_type == NOISE_TYPES.additive
        super(SRK, self).__init__(sde=sde, **kwargs)
        self._pw = None  # the element-wise programs of the step (pointwise.py), False once rejected

    def aux_times(self, t0, t1, dt):
        if self._additive:
            # sra1: C0 = (0, 3/4), C1 = (1, 0)                         tableaus/sra1.py:21-22
            return [t0 + 1 * dt, t0 + (3 / 4) * dt, t0 + 0 * dt]
        # srid2: C0 = (0, 1, 1/2, 0), C1 = (0, 1/4, 1, 1/4)            tableaus/srid2.py:21-22
        return [t0 + 0 * dt, t0 + 1 * dt, t0 + (1 / 4) * dt, t0 + (1 / 2) * dt]

    def scalars(self, dt):
        return {'rdt': float(1 / dt), 'sqrt_dt': float(_ieee_sqrt(dt)), 'three_dt': float(3 * dt)}

    def _step(self, c, y0, extra0, out):
        if self.sde.user_g_prod:
            y1 = self._additive_step_user_prod(c, y0) if self._additive else self._diagonal_step_user_prod(c, y0)
            if out is not None and not self._autograd:
                out.copy_(y1)
                return out, ()
            return y1, ()
        if self._additive:
            return self._additive_step(c, y0, out), ()
        return self._diagonal_or_scalar_step(c, y0, out), ()

    # -- user-supplied g_prod (srk.py:87,102,109 call sde.g_prod) -----------------------------------------------
    # The products are the user's own code, so the weights they are applied to have to exist as tensors: W and U are
    # materialised and the tableau arithmetic around the user's calls is a handful of element-wise torch ops in the
    # order of the fused kernels (csrc/tableau_diag_ops.cuh SrkDiagFinalOp, tableau_general.cu GSra*Op).  Not a fast
    # path — SDEs that want the fused one provide g — but the reference accepts it, so it has to work.
    def _weights(self, c):
        w, u = self._feed.tensors(c, True)
        shape = self.bm.shape
        return w.reshape(shape), u.reshape(shape)

    def _diagonal_step_user_prod(self, c, y0):
        sde, s = _WidenedSDE(self.sde, y0.dtype), c.scalars
        t_00, t_1, t_q, t_h = c.aux_t
        dt, rdt, sqrt_dt, three_dt = c.dt, s['rdt'], s['sqrt_dt'], s['three_dt']
        w, u = self._weights(c)
        ikk = (w * w - dt) * 0.5                                  # srk.py:63
        ikkk = ((w * w) * w - three_dt * w) * (1.0 / 6.0)         # srk.py:64
        b1, b2, b3, b4 = (-1, 4 / 3, 2 / 3, 0), (1, -4 / 3, 1 / 3, 0), (2, -4 / 3, -2 / 3, 0), (-2, 5 / 3, -2 / 3, 1)
        gw = [((b1[i] * w + (b2[i] * ikk) / sqrt_dt) + (b3[i] * u) * rdt) + (b4[i] * ikkk) * rdt for i in range(4)]
        LU = self._LU
        f0, g0 = _contig(sde.f(t_00, y0)), _contig(sde.g(t_00, y0))
        h0_1, h1_1 = self._k('tsde_srk_diag_stage1', LU, None, (y0, f0, g0), (dt, sqrt_dt), None, n_out=2)
        f1, g1 = _contig(sde.f(t_1, h0_1)), _contig(sde.g(t_q, h1_1))
        # stage 2 needs U inside the kernel: hand it the materialised increments
        nz = self._feed.from_tensors(*self._feed.tensors(c, True))
        h0_2, h1_2 = self._k('tsde_srk_diag_stage2', self._L, nz, (y0, f0, g0, f1, g1), (dt, rdt, sqrt_dt), None,
                             n_out=2)
        f2, g2 = _contig(sde.f(t_h, h0_2)), _contig(sde.g(t_1, h1_2))
        h1_3 = self._k('tsde_srk_diag_stage3', LU, None, (y0, g0, g1, f2, g2), (dt, sqrt_dt), None)
        y1 = y0
        for f, alpha, (t, h1), weight in zip((f0, f1, f2, None), (1 / 6, 1 / 6, 2 / 3, 0.0),
                                             ((t_00, y0), (t_q, h1_1), (t_1, h1_2), (t_q, h1_3)), gw):
            gp = sde.g_prod(t, h1, weight)
            y1 = (y1 + (alpha * f) * dt) + gp if f is not None else y1 + gp   # alpha[3] = 0: an exact zero
        return y1

    def _additive_step_user_prod(self, c, y0):
        sde, s = _WidenedSDE(self.sde, y0.dtype), c.scalars
        t_1, t_34, t_00 = c.aux_t
        dt, rdt = c.dt, s['rdt']
        w, u = self._weights(c)
        f0 = sde.f(t_00, y0)
        h0_1 = (y0 + (0.75 * f0) * dt) + sde.g_prod(t_1, y0, (1.5 * u) * rdt)          # srk.py:99-104
        f1 = sde.f(t_34, h0_1)
        y1 = (y0 + ((1 / 3) * f0) * dt) + sde.g_prod(t_1, y0, 1 * w + (-1 * u) * rdt)   # srk.py:107-110, i = 0
        y1 = (y1 + ((2 / 3) * f1) * dt) + sde.g_prod(t_00, y0, 0 * w + (1 * u) * rdt)   # i = 1
        return y1

    def _diagonal_or_scalar_step(self, c, y0, out):
        """srk.py:57-88.  Distinct evaluations only: f0,g0 at (t0,y0); f1 at (t0+dt, H0_1);
        g1 at (t0+dt/4, H1_1); f2 at (t0+dt/2, H0_2); g2 at (t0+dt, H1_2); g3 at (t0+dt/4, H1_3)."""
        sde, s = self.sde, c.scalars
        t_00, t_1, t_q, t_h = c.aux_t  # t0 + 0*dt, t0 + dt, t0 + dt/4, t0 + dt/2
        LU, L = self._LU, self._L
        if pointwise.ready(self):
            # f and g were recorded as element-wise programs (pointwise.py): the whole step is one kernel
            return pointwise.launch(self, 'tsde_step_srk_diag_pointwise', self._feed.get(c, True), y0,
                                    (t_00.data_ptr(), t_1.data_ptr(), t_q.data_ptr(), t_h.data_ptr(), c.dt, s['rdt'],
                                     s['sqrt_dt'], s['three_dt']), out)
        # the first step of an eligible solve runs as always, with the user's seven evaluations recorded
        rec = pointwise.SrkRecorder(y0, t_00, transcendental=pointwise.transcendental(self)) \
            if pointwise.recording(self) else None

        def f(t, y):
            return _contig(rec.evaluation('f', lambda: sde.f(t, y), t, y) if rec is not None else sde.f(t, y))

        def g(t, y):
            return _contig(rec.evaluation('g', lambda: sde.g(t, y), t, y) if rec is not None else sde.g(t, y))

        f0, g0 = self._fork(lambda: f(t_00, y0), lambda: g(t_00, y0))
        h0_1, h1_1 = self._k('tsde_srk_diag_stage1', LU, None, (y0, f0, g0), (c.dt, s['sqrt_dt']), None, n_out=2)
        f1, g1 = self._fork(lambda: f(t_1, h0_1), lambda: g(t_q, h1_1))
        h0_2, h1_2 = self._k('tsde_srk_diag_stage2', L, self._feed.get(c, True), (y0, f0, g0, f1, g1),
                             (c.dt, s['rdt'], s['sqrt_dt']), None, n_out=2)
        f2, g2 = self._fork(lambda: f(t_h, h0_2), lambda: g(t_1, h1_2))
        h1_3 = self._k('tsde_srk_diag_stage3', LU, None, (y0, g0, g1, f2, g2), (c.dt, s['sqrt_dt']), None)
        g3 = g(t_q, h1_3)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_srk_diag', L, self._feed.get(c, True), (y0, f0, f1, f2, g0, g1, g2, g3),
                       (c.dt, s['rdt'], s['sqrt_dt'], s['three_dt']), out)

    def _additive_step(self, c, y0, out):
        """srk.py:90-111: f0 = f(t0, y0); gA = g(t0+dt, y0); f1 = f(t0+3/4dt, H0_1); gB = g(t0, y0)."""
        sde, s = self.sde, c.scalars
        t_1, t_34, t_00 = c.aux_t
        if pointwise.ready(self):
            # f and g were recorded as element-wise programs (pointwise.py): the whole step is one kernel
            # (on the solver's GENERAL launch: the sra1 step, t_q = t_34, t_h and the last two scalars unused)
            return pointwise.launch(self, 'tsde_step_srk_diag_pointwise', self._feed.get(c, True), y0,
                                    (t_00.data_ptr(), t_1.data_ptr(), t_34.data_ptr(), None, c.dt, s['rdt'], 0.0,
                                     0.0), out)
        # the first step of an eligible solve runs as always, with the user's four evaluations recorded
        rec = pointwise.pc_recorder(self, y0, t_00, pointwise.SRA_PATTERN)

        def f(t, y):
            return _contig(rec.evaluation('f', lambda: sde.f(t, y), t, y) if rec is not None else sde.f(t, y))

        def g(t, y):
            return _gop(rec.evaluation('g', lambda: sde.g(t, y), t, y) if rec is not None else sde.g(t, y))

        # f0, g(t1, y0) and g(t0, y0) share their inputs: three parallel branches
        f0, ga, gb = self._fork(lambda: f(t_00, y0), lambda: g(t_1, y0), lambda: g(t_00, y0))
        h0_1 = self._k('tsde_srk_additive_stage', self._L, self._feed.get(c, True), (y0, f0, ga), (c.dt, s['rdt']),
                       None)
        f1 = f(t_34, h0_1)
        if rec is not None:
            self._pw = pointwise.finish(self, rec)
        return self._k('tsde_step_srk_additive', self._L, self._feed.get(c, True), (y0, f0, f1, ga, gb),
                       (c.dt, s['rdt']), out)


class LogODEMidpoint(_ProdMixin, base_solver.BaseSDESolver):
    """methods/log_ode.py:25-56: midpoint scheme plus the Levy-area term sum_{j,k,l} dg_il/dy_j g_jk A_kl
    (base_sde.py:165-206).  The Levy area A comes from the Brownian motion (davie / foster); the
    jvp's through the user's g are autograd glue, the tableau arithmetic runs in the fused kernels."""
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = (LEVY_AREA_APPROXIMATIONS.davie, LEVY_AREA_APPROXIMATIONS.foster)
    needs_levy_area = True  # increments are always materialised (W and A) through bm(ta, tb, return_A=True)

    def __init__(self, sde, **kwargs):
        if getattr(sde, 'is_adjoint_sde', False):
            raise ValueError("Log-ODE schemes cannot be used for adjoint SDEs, because they require "
                             "direct access to the diffusion, whilst adjoint SDEs rely on a more efficient "
                             "diffusion-vector product. Use a different method instead.")
        self.strong_order = 0.5 if sde.noise_type == NOISE_TYPES.general else 1.0
        super(LogODEMidpoint, self).__init__(sde=sde, **kwargs)

    def aux_times(self, t0, t1, dt):
        return [t0 + 0.5 * dt]

    def scalars(self, dt):
        return {'half_dt': float(0.5 * dt)}

    def _dg_ga_jvp_column_sum(self, t, y, a):
        """base_sde.py:165-185 (v1); zero for non-general noise (:71,205-206)."""
        from .adjoint_sde import _jvp
        track = self._autograd
        with torch.enable_grad():
            y = y if (track and y.requires_grad) else y.detach().requires_grad_(True)
            g = widen(self.sde.g(t, y), y.dtype)  # (bmm_ga and the jvp's below take the state dtype)
            if track:
                # gradients flow through the tangents as well (create_graph): keep the product in autograd
                ga_cols = torch.bmm(g, a).unbind(-1)
            else:
                # fused fp32 kernel, result transposed to (m, rows, d): one contiguous tangent per column
                ga_t = torch.empty((g.size(-1), g.size(0), g.size(1)), dtype=g.dtype, device=g.device)
                _cabi.check(self._lib.tsde_bmm_ga(self._L, _contig(g.detach()).data_ptr(), _contig(a).data_ptr(),
                                                  ga_t.data_ptr()), "tsde_bmm_ga")
                ga_cols = ga_t.unbind(0)
            total = None
            for col in range(g.size(-1)):
                term = _jvp(g[..., col], y, ga_cols[col], create_graph=track)
                total = term if total is None else total + term
        return total if track else total.detach()

    def _step(self, c, y0, extra0, out):
        W, A = self.bm(c.ft0, c.ft1, return_A=True)
        self._feed.prime(c, _contig(W))  # the products below reuse this increment
        L, nz, f, g = self._f_and_g_prod(c, c.t0, y0)
        yp = self._k('tsde_midpoint_predict', L, nz, (y0, f, g), (c.scalars['half_dt'],), None)
        L, nz, fp, gp = self._f_and_g_prod(c, c.aux_t[0], yp)
        general = self.sde.noise_type == NOISE_TYPES.general
        tmp = self._k('tsde_step_euler', L, nz, (y0, fp, gp), (c.dt,), None if general else out)
        if not general:
            return tmp, ()
        dg_ga = _contig(self._dg_ga_jvp_column_sum(c.aux_t[0], yp, A))
        # y1 = (y0 + dt*f' + g'.dW) + dg_ga                                             log_ode.py:54
        return self._k('tsde_linear_interp', self._LU, None, (tmp, dg_ga), (1.0, 1.0), out), ()


def select(method, sde_type):
    """methods/__init__.py:26-48."""
    if method == METHODS.euler:
        return Euler
    elif method == METHODS.milstein and sde_type == SDE_TYPES.ito:
        return MilsteinIto
    elif method == METHODS.srk:
        return SRK
    elif method == METHODS.midpoint:
        return Midpoint
    elif method == METHODS.reversible_heun:
        return ReversibleHeun
    elif method == METHODS.adjoint_reversible_heun:
        from .adjoint import AdjointReversibleHeun
        return AdjointReversibleHeun
    elif method == METHODS.heun:
        return Heun
    elif method == METHODS.milstein and sde_type == SDE_TYPES.stratonovich:
        return MilsteinStratonovich
    elif method == METHODS.log_ode_midpoint:
        return LogODEMidpoint
    elif method == METHODS.euler_heun:
        return EulerHeun
    else:
        raise ValueError(f"Method '{method}' does not match any known method.")
