"""`sdeint_adjoint`: custom autograd node around the forward solve, with three backward engines.

Reference: torchsde/_core/adjoint.py (`_SdeintAdjointMethod` :29-127, `sdeint_adjoint` :130-278,
`_select_default_adjoint_method` :281-296), methods/reversible_heun.py:76-144 (`AdjointReversibleHeun.step`) and
_core/adjoint_sde.py (the augmented backward SDE).

* Reversible pair (method='reversible_heun', adjoint_method='adjoint_reversible_heun'): the reference packs
  (y, adj_y, adj_f, adj_g, adj_z, adj_params...) into one flat vector with a dummy batch dimension and re-enters
  `autograd.Function.apply` once per output interval, copying the whole augmented state through `flatten` /
  `flat_to_shape` on every step (adjoint.py:75-79,114-119; reversible_heun.py:142; adjoint_sde.py:104).  Here the
  augmented state stays in separate buffers, and one backward step is exactly
      kernel A (reconstruct z1, first half of the adjoint bookkeeping)
      user f_and_g at z0 + one torch.autograd.grad (the vjp)          <- user code, stays in torch
      user f_and_g at z1
      kernel B (reconstruct y1, second half of the bookkeeping)
  with the Brownian increment of the step regenerated from the Philox counter in both kernels (the same cells the
  forward pass consumed, addressed in reverse: `ReverseBrownian` semantics, _brownian/derived.py:27-30).  The sweep
  can be captured as a CUDA graph (`adjoint_options={'cuda_graph': True}`); with `adjoint_adaptive=True` it runs the
  reference's adaptive controller on the augmented state (`_BackwardEngine.run_adaptive`).  With
  `adjoint_options={'fused_backward': True}` and an element-wise diagonal-noise SDE, the first step is recorded
  (pointwise.AdjointRecorder) and the whole sweep runs as chunks of up to TSDE_PW_MAX_STEPS steps per kernel
  (`_BackwardEngine._fused_sweep`).
* Every other pair: the generic `AdjointSDE` (adjoint_sde.py) integrated backwards by the ordinary solvers on the flat
  augmented state (`_generic_backward`).
* Double backward (create_graph=True): the generic path re-enters `_SdeintAdjointMethod.apply` per interval exactly
  like the reference (adjoint.py:97-113); the reversible pair — which the reference cannot double-backward — goes
  through `_ReversibleVJP`.
"""
import ctypes
import warnings

import torch
from torch import nn

from . import base_solver
from . import methods
from . import pointwise
from . import schedule as schedule_lib
from . import sdeint as sdeint_mod
from .base_sde import widen
from .base_solver import _contig
from .. import _cabi
from .._brownian import BrownianInterval, ReverseBrownian
from ..settings import METHODS, NOISE_TYPES, SDE_TYPES, LEVY_AREA_APPROXIMATIONS

_check = _cabi.check


def _p(t):
    return t.data_ptr()


class AdjointReversibleHeun(base_solver.BaseSDESolver):
    """Class-attribute / constructor contract of methods/reversible_heun.py:76-96.  It can only be
    used as `adjoint_method`; the backward integration is driven by `_ReversibleAdjoint` below."""
    weak_order = 1.0
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    def __init__(self, sde, **kwargs):
        if not getattr(sde, 'is_adjoint_sde', False):
            raise ValueError(f"{METHODS.adjoint_reversible_heun} can only be used for adjoint_method.")
        self.strong_order = 1.0 if sde.noise_type == NOISE_TYPES.additive else 0.5
        super(AdjointReversibleHeun, self).__init__(sde=sde, **kwargs)

    def init_extra_solver_state(self, t0, y0):
        raise RuntimeError("Please report a bug to torchsde_b200.")

    def _step(self, c, y0, extra0, out):
        raise RuntimeError("Please report a bug to torchsde_b200.")


class _BackwardEngine(base_solver.BaseSDESolver):
    """Runs AdjointReversibleHeun.step (reversible_heun.py:98-144) over the reversed time grid."""
    weak_order = 1.0
    strong_order = 0.5
    sde_type = SDE_TYPES.stratonovich
    noise_types = NOISE_TYPES.all()
    levy_area_approximations = LEVY_AREA_APPROXIMATIONS.all()

    _pw_method = 'adjoint_reversible_heun'  # (pointwise.chunk_length)

    def __init__(self, sde, bm, dt, params, adjoint_options=None):
        super(_BackwardEngine, self).__init__(sde=sde, bm=bm, dt=dt, adaptive=False, rtol=None, atol=None,
                                              dt_min=None, options={})
        self.params = list(params)
        self.adjoint_options = adjoint_options or {}
        self._pw = None  # the fused sweep's program (pointwise.AdjointRecorder.finish), False when it cannot fuse

    def aux_times(self, t0, t1, dt):
        return [-t0, -t1]  # forward-time arguments of f_and_g (reversible_heun.py:122,133)

    def scalars(self, dt):
        return {'half_dt': float(0.5 * dt)}

    def _step(self, c, y0, extra0, out):
        raise RuntimeError("internal")

    def _half(self, name, L, nz, ins, scalars, outs):
        """Kernel A or B of a backward step, with the formats of 16-bit SDE outputs (f0, g0, f1, g1) declared like
        those of every tableau launch (_cabi.operands)."""
        word, ins = _cabi.operands(name, self.dtype, ins)
        self._launch(name, L, nz, ins, scalars, outs, word)

    def plan(self, ys, ts):
        """Host-side plan of the backward sweep: one schedule per interval [-ts[i], -ts[i-1]], exactly
        as the reference re-enters integrate() (adjoint.py:97-113), merged into one step list."""
        T = ts.numel()
        y = _contig(ys[-1])
        self._prepare(y)
        neg_ts = -ts
        self.scheds = [schedule_lib.build_schedule(torch.stack([neg_ts[i], neg_ts[i - 1]]), self.dt)
                       for i in range(T - 1, 0, -1)]
        bounds = [self.scheds[0].bounds[0]]
        for s in self.scheds:
            bounds.extend(s.bounds[1:])
        merged = schedule_lib.Schedule(None, [st for s in self.scheds for st in s.steps], [])
        merged.bounds = bounds
        self.binding = self._bind(merged)
        self._feed = base_solver.NoiseFeed(self, self.bm, self.binding)
        self.ctxs = self._contexts(merged, ts)
        self.T = T

    def param_names(self):
        """Names of the adjoint parameters inside the SDE module tree (None if some are foreign tensors)."""
        by_id = {id(p): n for n, p in self.sde.named_parameters()}
        names = [by_id.get(id(p)) for p in self.params]
        return None if any(n is None for n in names) else names

    def sweep(self, ys, grad_ys, extras, grad_extras, alias_names=None):
        """Backward sweep over all output intervals (adjoint.py:97-119).  Capturable: no host syncs.
        Returns adj_y0, (adj_f, adj_g, adj_z), adj_params.

        alias_names (graph capture only): differentiate w.r.t. fresh detached aliases of the parameters,
        swapped into the module for the duration of the call.  A parameter's cached AccumulateGrad node
        remembers the stream it was created on (usually the legacy default stream); when a parameter
        receives gradient from two paths autograd synchronises *that* stream with the producer, which is
        illegal while another stream is capturing.  Aliases created under capture do not have this problem
        and give bit-identical gradients."""
        if alias_names is not None:
            from torch.nn.utils import stateless
            aliases = {n: p.detach().requires_grad_() for n, p in zip(alias_names, self.params)}
            with stateless._reparametrize_module(self.sde, aliases):
                return self._sweep(ys, grad_ys, extras, grad_extras, [aliases[n] for n in alias_names])
        return self._sweep(ys, grad_ys, extras, grad_extras, self.params)

    def _sweep(self, ys, grad_ys, extras, grad_extras, params):
        self._refresh_stream()
        if self.adjoint_options.get('fused_backward', False) and self._pw is not False:
            out = self._fused_sweep(ys, grad_ys, extras, grad_extras, params)
            if out is not None:
                return out
        L = self._L
        T = self.T
        y = _contig(ys[-1])
        f0, g0, z0 = (_contig(x.detach()) for x in extras)
        adj_y = _contig(grad_ys[-1]).clone()
        adj_f, adj_g, adj_z = (_contig(x).clone() for x in grad_extras)
        adj_params = [torch.zeros_like(p) for p in params]
        sde = self.sde
        k = 0
        # The reference evaluates f_and_g twice per backward step: with autograd at (t0, z0) for the vjp (:119-129) and
        # without at (t1, z1) for the reconstruction (:133) — and notes "it should be possible to make one fewer
        # forward call by re-using the forward computation in the previous step" (:117-118).  It is: step k's z1 IS
        # step k+1's z0 (same time, same tensor), so the evaluation at (t1, z1) is recorded by autograd and kept as
        # `pending` for the next step's vjp.  Same numbers (the kernels are deterministic), one user forward
        # evaluation per step instead of two.
        pending = None
        for n, sched in enumerate(self.scheds):
            i = T - 1 - n
            for _ in range(sched.n_steps):
                c = self.ctxs[k]
                k += 1
                t_fwd0, t_fwd1 = c.aux_t
                half_dt = c.scalars['half_dt']
                z1 = torch.empty_like(y)
                adj_f_mid = torch.empty_like(adj_f)
                adj_g_mid = torch.empty_like(adj_g)
                self._half('tsde_adjoint_reversible_heun_a', L, self._feed.get(c),
                           (y, z0, f0, g0, adj_y, adj_f, adj_g), (c.dt, half_dt), (z1, adj_f_mid, adj_g_mid))
                with torch.enable_grad():
                    if pending is None:
                        z0r = z0.detach().requires_grad_()
                        re_f0, re_g0 = sde.f_and_g(t_fwd0, z0r)
                    else:
                        z0r, re_f0, re_g0 = pending
                    outs, gouts = [], []
                    for o, go in ((re_f0, adj_f_mid), (re_g0, adj_g_mid)):
                        if o.requires_grad:
                            outs.append(widen(o, go.dtype))
                            gouts.append(go.view_as(o))
                    if outs:
                        vjps = torch.autograd.grad(outs, [z0r] + list(params), gouts, allow_unused=True)
                    else:
                        vjps = [None] * (1 + len(params))
                    del re_f0, re_g0, outs
                    z1r = z1.detach().requires_grad_()
                    f1_graph, g1_graph = sde.f_and_g(t_fwd1, z1r)
                    pending = (z1r, f1_graph, g1_graph)
                vjp_z = vjps[0] if vjps[0] is not None else torch.zeros_like(z0)
                for ap, v in zip(adj_params, vjps[1:]):
                    if v is not None:
                        ap.add_(v)
                f1, g1 = _contig(f1_graph.detach()), _contig(g1_graph.detach())
                y1 = torch.empty_like(y)
                adj_y1 = torch.empty_like(adj_y)
                adj_z1 = torch.empty_like(adj_z)
                adj_f1 = torch.empty_like(adj_f)
                adj_g1 = torch.empty_like(adj_g)
                self._half('tsde_adjoint_reversible_heun_b', L, self._feed.get(c),
                           (y, f0, f1, g0, g1, adj_y, adj_z, _contig(vjp_z)), (c.dt, half_dt),
                           (y1, adj_y1, adj_z1, adj_f1, adj_g1))
                y, adj_y, adj_z, adj_f, adj_g = y1, adj_y1, adj_z1, adj_f1, adj_g1
                f0, g0, z0 = f1, g1, z1
            # adjoint.py:114-116
            y = _contig(ys[i - 1])
            adj_y = adj_y + grad_ys[i - 1]
        return adj_y, (adj_f, adj_g, adj_z), adj_params

    # ---- the fused sweep (adjoint_options={'fused_backward': True}) -------------------------------------------
    def _record(self, ys, grad_ys, extras, grad_extras, params):
        """The first backward step, run the ordinary way (kernel A, f and g, the vjp, f and g again) under an
        AdjointRecorder; its results are discarded: the chunks start from the same state."""
        c = self.ctxs[0]
        y = _contig(ys[-1])
        f0, g0, z0 = (_contig(x.detach()) for x in extras)
        adj_f, adj_g, _ = (_contig(x) for x in grad_extras)
        z1, adj_f_mid, adj_g_mid = torch.empty_like(y), torch.empty_like(adj_f), torch.empty_like(adj_g)
        self._half('tsde_adjoint_reversible_heun_a', self._L, self._feed.get(c),
                   (y, z0, f0, g0, _contig(grad_ys[-1]), adj_f, adj_g), (c.dt, c.scalars['half_dt']),
                   (z1, adj_f_mid, adj_g_mid))
        t_fwd0, t_fwd1 = c.aux_t
        sde = self.sde
        with torch.enable_grad():
            z0r = z0.detach().requires_grad_()
            rec = pointwise.AdjointRecorder(z0r, t_fwd0, len(params),
                                            bool(self.adjoint_options.get('transcendental', False)))
            re_f0, re_g0 = rec.forward(lambda: sde.f_and_g(t_fwd0, z0r))
            pairs = [(o, go) for o, go in ((re_f0, adj_f_mid), (re_g0, adj_g_mid)) if o.requires_grad]
            if not pairs:
                rec.reject("f and g depend on neither the state nor a parameter")
                return rec
            rec.vjp(lambda: torch.autograd.grad([widen(o, go.dtype) for o, go in pairs], [z0r] + list(params),
                                                [go.view_as(o) for o, go in pairs], allow_unused=True),
                    adj_f_mid, adj_g_mid, params)
            z1r = z1.detach().requires_grad_()
            rec.again(lambda: sde.f_and_g(t_fwd1, z1r), t_fwd1, z1r)
        return rec

    def _fused_sweep(self, ys, grad_ys, extras, grad_extras, params):
        """The sweep as chunks of the adjoint program (tsde_solve_reversible_heun_pointwise), or None (after a warning
        with the reason) when it cannot fuse.  Records and compiles the program on first use: under graph capture that
        is the warm-up sweep (_backward_plan), and the captured sweep only launches chunks and the final reductions."""
        y = _contig(ys[-1])
        state = [y] + [_contig(x.detach()) for x in (extras[2], extras[0], extras[1])] + \
            [_contig(grad_ys[-1])] + [_contig(x) for x in grad_extras]   # y, z, f, g, adj_y, adj_f, adj_g, adj_z
        if self._pw is None:
            reason = pointwise.adjoint_refusal(self, self.adjoint_options)
            if reason is None and not pointwise.state_fits(self, state[2:4] + state[1:2]):
                reason = "the solver state (f0, g0, z0) is not made of (rows, d) tensors of the state dtype"
            if reason is None and any(s.n_steps == 0 for s in self.scheds):
                reason = "an output interval without steps"
            res = None
            if reason is None:
                rec = self._record(ys, grad_ys, extras, grad_extras, params)
                res = pointwise.compile_adjoint(rec, rec.finish())
                reason = rec.reason
            self._pw = res or False
            if not res:
                warn_unfused(reason)
                return None
        self._out = []  # per step: the output index whose row the step ends on, or -1
        for n, sched in enumerate(self.scheds):
            self._out += [-1] * (sched.n_steps - 1) + [self.T - 2 - n]
        n_steps = len(self._out)
        kinds = self._pw[2]
        partials = [torch.zeros_like(y) for kind in kinds if kind is not None]
        ys_c, gys_c = _contig(ys), _contig(grad_ys)
        multi = [k for k in range(n_steps) if self.binding.cell(self.ctxs[k].k)[2] > 1]
        chunks = pointwise.plan_chunks(0, n_steps, multi_cell=multi, max_steps=pointwise.chunk_length(self))
        # a chunk stores its state to the set it did not read: the caller's tensors are read once, so a sweep of one
        # chunk needs one set, any other two
        sets = [[torch.empty_like(y) for _ in state] for _ in range(min(len(chunks), 2))]
        for j, (k0, k1) in enumerate(chunks):
            t0 = self.ctxs[0].aux_t[0] if k0 == 0 else self.ctxs[k0 - 1].aux_t[1]
            pointwise.solve_adjoint_chunk(self, range(k0, k1), t0, state, sets[j % 2], ys_c, gys_c, partials)
            state = sets[j % 2]
        # each parameter's contributions, reduced once over the batch as autograd's sum_to reduces one step's
        adj_params = [torch.zeros_like(p) for p in params]
        live = iter(partials)
        for ap, kind in zip(adj_params, kinds):
            if kind is not None:
                part = next(live)
                ap.add_((part.sum(0) if kind == pointwise.REDUCE_ROWS else
                         part.sum() if kind == pointwise.REDUCE_ALL else part).view_as(ap))
        return state[4], (state[5], state[6], state[7]), adj_params

    def run(self, ys, ts, grad_ys, extras, grad_extras):
        self.plan(ys, ts)
        return self.sweep(ys, grad_ys, extras, grad_extras)

    # ---- adaptive backward sweep (adjoint_adaptive=True) ------------------------------------------------------
    # The reference warns that the reversible pair "does not save the time steps used" and then simply runs the
    # adjoint solver's `integrate` with adaptive=True on every output interval (adjoint.py:245-249, 97-113;
    # base_solver.py:117-142): one full step against two half steps of AdjointReversibleHeun.step, the error taken
    # over the whole augmented state (y, adj_y, adj_f, adj_g, adj_z, adj_params), the solver state (f, g, z) carried
    # along.  Same here: kernels A / B per trial step, increments queried at the data-dependent times through
    # ReverseBrownian (memory source), one device->host scalar per proposal.
    def _bstep(self, ta, tb, st, params):
        """One AdjointReversibleHeun.step from reversed time ta to tb (0-d CPU tensors).  `st` = (y, z0, f0, g0, adj_y,
        adj_f, adj_g, adj_z, adj_params); returns the new state without modifying `st`."""
        y, z0, f0, g0, adj_y, adj_f, adj_g, adj_z, adj_params = st
        h = tb - ta
        dt, half_dt = float(h), float(0.5 * h)
        w = _contig(self.bm(float(ta), float(tb)))
        nz = self._feed.from_tensors(w.reshape(self.bm_rows, self.m))
        t_fwd0 = (-ta).to(self.device)
        t_fwd1 = (-tb).to(self.device)
        z1, adj_f_mid, adj_g_mid = torch.empty_like(y), torch.empty_like(adj_f), torch.empty_like(adj_g)
        self._half('tsde_adjoint_reversible_heun_a', self._L, nz, (y, z0, f0, g0, adj_y, adj_f, adj_g),
                   (dt, half_dt), (z1, adj_f_mid, adj_g_mid))
        with torch.enable_grad():
            z0r = z0.detach().requires_grad_()
            re_f0, re_g0 = self.sde.f_and_g(t_fwd0, z0r)
            pairs = [(widen(o, go.dtype), go.view_as(o)) for o, go in ((re_f0, adj_f_mid), (re_g0, adj_g_mid))
                     if o.requires_grad]
            if pairs:
                vjps = torch.autograd.grad([o for o, _ in pairs], [z0r] + list(params), [g for _, g in pairs],
                                           allow_unused=True)
            else:
                vjps = [None] * (1 + len(params))
        vjp_z = _contig(vjps[0]) if vjps[0] is not None else torch.zeros_like(z0)
        new_params = [ap if v is None else ap + v for ap, v in zip(adj_params, vjps[1:])]
        f1, g1 = self.sde.f_and_g(t_fwd1, z1)
        f1, g1 = _contig(f1), _contig(g1)
        y1, adj_y1, adj_z1 = torch.empty_like(y), torch.empty_like(adj_y), torch.empty_like(adj_z)
        adj_f1, adj_g1 = torch.empty_like(adj_f), torch.empty_like(adj_g)
        self._half('tsde_adjoint_reversible_heun_b', self._L, nz, (y, f0, f1, g0, g1, adj_y, adj_z, vjp_z),
                   (dt, half_dt), (y1, adj_y1, adj_z1, adj_f1, adj_g1))
        return (y1, z1, f1, g1, adj_y1, adj_f1, adj_g1, adj_z1, new_params)

    def _aug_error(self, a, b, rtol, atol):
        """compute_error (adaptive_stepping.py:42-76) over the augmented state: RMS over ALL elements of the flat
        vector the reference integrates."""
        eps = 1e-7
        lib = _cabi.lib()
        parts = [(a[0], b[0])] + [(a[k], b[k]) for k in (4, 5, 6, 7)] + list(zip(a[8], b[8]))
        if self._err_buf is None or self._err_buf.numel() < 1024 + len(parts):
            self._err_buf = torch.zeros(1024 + len(parts), dtype=torch.float64, device=self.device)
        buf = self._err_buf
        stream = torch.cuda.current_stream(self.device).cuda_stream
        total = 0
        for k, (x, y) in enumerate(parts):
            x, y = _contig(x), _contig(y)
            n = x.numel()
            total += n
            L = _cabi.make_launch(self.dtype, _cabi.NOISE_DIAGONAL, 1, n, n, stream)
            _check(lib.tsde_adaptive_error_sumsq(ctypes.byref(L), _p(x), _p(y), float(rtol), float(atol),
                                                 eps, buf[len(parts):].data_ptr(), buf[k:].data_ptr()),
                   "tsde_adaptive_error_sumsq")
        err = (float(buf[:len(parts)].sum().item()) / total) ** 0.5
        assert err == err, ('Found nans in the error estimate. Try increasing the tolerance or regularizing '
                            'the dynamics.')
        return max(err, eps)

    def run_adaptive(self, ys, ts, grad_ys, extras, grad_extras, rtol, atol, dt_min):
        y_last = _contig(ys[-1])
        self._prepare(y_last)
        self._refresh_stream()
        self._feed = base_solver.NoiseFeed(self, self.bm, None)
        self._err_buf = None
        T = ts.numel()
        neg = (-ts).detach().to('cpu')
        dt0 = self.dt.detach().to('cpu') if torch.is_tensor(self.dt) else self.dt
        f0, g0, z0 = (_contig(x.detach()) for x in extras)
        adj_f, adj_g, adj_z = (_contig(x).clone() for x in grad_extras)
        st = (y_last, z0, f0, g0, _contig(grad_ys[-1]).clone(), adj_f, adj_g, adj_z,
              [torch.zeros_like(p) for p in self.params])
        params = self.params
        for i in range(T - 1, 0, -1):
            curr_t, end_t = neg[i], neg[i - 1]
            step_size, prev_error_ratio = dt0, None                 # (every interval is a fresh `integrate` call)
            while curr_t < end_t:
                next_t = min(curr_t + step_size, end_t)
                full = self._bstep(curr_t, next_t, st, params)
                mid_t = 0.5 * (curr_t + next_t)
                half = self._bstep(curr_t, mid_t, st, params)
                two = self._bstep(mid_t, next_t, half, params)
                error_estimate = self._aug_error(full, two, rtol, atol)
                step_size, prev_error_ratio = self._update_step_size(
                    error_estimate=error_estimate, prev_step_size=step_size, prev_error_ratio=prev_error_ratio)
                if step_size < dt_min:
                    warnings.warn("Hitting minimum allowed step size in adaptive time-stepping.")
                    step_size = dt_min
                    prev_error_ratio = None
                if error_estimate <= 1 or step_size <= dt_min:
                    curr_t, st = next_t, two
            # adjoint.py:114-116 (the interval ends exactly on -ts[i-1]: interpolation is the identity)
            st = (_contig(ys[i - 1]), st[1], st[2], st[3], st[4] + grad_ys[i - 1]) + st[5:]
        return st[4], (st[5], st[6], st[7]), st[8]


_BWD_PLANS = __import__('weakref').WeakKeyDictionary()
_WARNED = set()


def warn_unfused(reason):
    """adjoint_options={'fused_backward': True} was given, but the sweep keeps its unfused steps: say why, once per
    reason."""
    if reason not in _WARNED:
        _WARNED.add(reason)
        warnings.warn(f"sdeint_adjoint: the backward sweep keeps its unfused steps ({reason}).")


def drop_plans(sde):
    """Release every cached backward-sweep plan of `sde`."""
    from . import graph as graph_mod
    owner, _ = graph_mod.cache_owner(sde)
    try:
        _BWD_PLANS.pop(owner, None)
    except TypeError:
        pass


def _backward_plan(engine, ys, ts, extras):
    """Capture (once) the backward sweep as a CUDA graph.  Called from the *forward* pass, i.e. from
    the user's thread: stream capture cannot be started from inside the autograd engine's worker
    thread (its stream bookkeeping touches the legacy stream).  Same design as graph.py: static
    inputs refreshed by copies, Philox key read from a static 8-byte buffer."""
    from . import graph as graph_mod
    engine.plan(ys, ts)
    binding = engine.binding
    names = engine.param_names()
    if binding is None or names is None:
        return None
    sde_obj, _ = graph_mod.cache_owner(engine.sde)
    # (the adjoint options decide what the sweep launches: a plan captured with fused_backward must not serve a solve
    # without it, nor the other way round)
    key = ('bwd',) + graph_mod._plan_key(engine, ys[0], ts, tuple(extras), binding) + (
        tuple(tuple(p.shape) for p in engine.params),
        tuple(sorted((k, repr(v)) for k, v in engine.adjoint_options.items() if k != 'cuda_graph')))
    plans = graph_mod.plans_of(_BWD_PLANS, sde_obj)
    if plans is None:
        return None
    plan = plans.get(key)
    if plan is not None:
        return plan
    plan = graph_mod._Plan()
    plan.binding = binding  # (no reference to the engine / the SDE: plans must not keep their cache key alive)
    plan.ys = ys.detach().clone()
    plan.grad_ys = torch.zeros_like(plan.ys)
    plan.extras = tuple(_contig(e.detach()).clone() for e in extras)
    plan.grad_extras = tuple(torch.zeros_like(e, dtype=ys.dtype) for e in plan.extras)  # (see _backward)
    plan.key = binding.interval.key_tensor().clone()
    engine._feed._key_ptr = plan.key.data_ptr()
    dev = ys.device
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    # warm-up (cuBLAS handles, autograd, allocator): first interval only
    with torch.cuda.stream(side), graph_mod.uncached_autocast():
        saved = engine.scheds, engine.T
        engine.scheds, engine.T = [engine.scheds[0]], 2
        engine.sweep(plan.ys[-2:], plan.grad_ys[-2:], plan.extras, plan.grad_extras, alias_names=names)
        engine.scheds, engine.T = saved
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    g = torch.cuda.CUDAGraph()
    with graph_mod.no_gc(), torch.cuda.graph(g), graph_mod.uncached_autocast():
        plan.out = engine.sweep(plan.ys, plan.grad_ys, plan.extras, plan.grad_extras, alias_names=names)
    plan.time_table = getattr(engine, '_time_table', None)
    plan.graph = g
    graph_mod._remember(plans, key, plan)
    return plan


def _replay_backward(plan, bm, ys, grad_ys, extras, grad_extras):
    plan.ys.copy_(ys)
    plan.grad_ys.copy_(grad_ys)
    for d, s_ in zip(plan.extras, extras):
        d.copy_(s_)
    for d, s_ in zip(plan.grad_extras, grad_extras):
        d.copy_(s_)
    plan.key.copy_(bm.key_tensor())
    plan.graph.replay()
    adj_y, adj_extras, adj_params = plan.out
    # hand out copies: the static outputs are overwritten by the next replay
    return adj_y.clone(), tuple(a.clone() for a in adj_extras), [a.clone() for a in adj_params]


class _AdjointMarker:
    """Stands in for the reference's AdjointSDE where only its type/attributes are inspected."""
    is_adjoint_sde = True

    def __init__(self, forward_sde):
        self.forward_sde = forward_sde
        self.sde_type = forward_sde.sde_type
        # adjoint_sde.py:33-38
        self.noise_type = {
            NOISE_TYPES.general: NOISE_TYPES.general,
            NOISE_TYPES.additive: NOISE_TYPES.general,
            NOISE_TYPES.scalar: NOISE_TYPES.scalar,
            NOISE_TYPES.diagonal: NOISE_TYPES.diagonal,
        }[forward_sde.noise_type]


def _generic_backward(sde, bm, dt, ys, ts, grad_ys, params, cfg, differentiable=False):
    """Backward pass through the augmented adjoint SDE (adjoint.py:65-127) for non-reversible pairs:
    integrate (y, adj_y, adj_params) from -ts[i] to -ts[i-1] with `adjoint_method`, newest interval
    first, resetting y to the stored ys[i-1] and adding grad_ys[i-1] in between.  `differentiable`: the caller
    differentiates this backward pass (create_graph=True, i.e. double backward).  As in the reference
    (adjoint.py:97-113) every interval then RE-ENTERS `_SdeintAdjointMethod.apply` with the augmented adjoint SDE as
    the SDE: the second-order gradient is the continuous adjoint of the adjoint solve (same `adjoint_method`), with
    AdjointSDE building its vjp's with create_graph (adjoint_sde.py:97,118,138,183).  The reference's limits are
    inherited: an Ito SDE whose adjoint needs the Ito correction cannot be double-backwarded (its AdjointSDE has no
    `f_and_g`, adjoint_sde.py:267-271)."""
    from .adjoint_sde import AdjointSDE
    if hasattr(sde, 'widen_outputs'):
        sde.widen_outputs(ys.dtype)  # the backward SDE is torch code on the forward SDE's outputs
    aug = [ys[-1], grad_ys[-1]] + [torch.zeros_like(p) for p in params]
    shapes = [t.size() for t in aug]
    numels = [t.numel() for t in aug]
    adjoint_sde = AdjointSDE(sde, params, shapes)
    reverse_bm = ReverseBrownian(bm)
    solver_fn = methods.select(method=cfg['adjoint_method'], sde_type=adjoint_sde.sde_type)
    solver = solver_fn(sde=adjoint_sde, bm=reverse_bm, dt=dt, adaptive=cfg['adjoint_adaptive'],
                       rtol=cfg['adjoint_rtol'], atol=cfg['adjoint_atol'], dt_min=cfg['dt_min'],
                       options=cfg['adjoint_options'])
    flat = torch.cat([t.reshape(-1) for t in aug]).unsqueeze(0)
    inner_options = {'_cfg': cfg}
    for i in range(ys.size(0) - 1, 0, -1):
        if differentiable:
            out, = _SdeintAdjointMethod.apply(adjoint_sde, torch.stack([-ts[i], -ts[i - 1]]), dt, reverse_bm, solver, {},
                                              inner_options, 0, flat, *params)
        else:
            out, _ = solver.integrate(flat, torch.stack([-ts[i], -ts[i - 1]]), ())
        parts = [p.reshape(s) for p, s in zip(out[-1].squeeze(0).split(numels), shapes)]
        parts[0] = ys[i - 1]
        parts[1] = parts[1] + grad_ys[i - 1]
        flat = torch.cat([t.reshape(-1) for t in parts]).unsqueeze(0)
    return parts[1], parts[2:]


def _recomputed_solve(sde, bm, dt, ts, y0, extras0):
    """Reversible-Heun forward solve with every tableau launch recorded as an autograd node."""
    solver = methods.ReversibleHeun(sde=sde, bm=bm, dt=dt, adaptive=False, rtol=None, atol=None, dt_min=None, options={})
    solver._autograd = True
    sde.widen_outputs(y0.dtype)
    ys, extras = solver.integrate(y0, ts, tuple(widen(e, y0.dtype) for e in extras0))
    return [ys, *extras]


class _ReversibleVJP(torch.autograd.Function):
    """Differentiable backward pass of the reversible pair, for double backward (create_graph=True).

    The reference cannot do this at all (its re-entered Function finds no saved solver state and
    AdjointReversibleHeun.init_extra_solver_state raises, reversible_heun.py:93-96).  Reversible Heun's adjoint IS the
    exact gradient of the discrete forward solve, so the same vector-Jacobian product is obtained by re-running the
    forward solve from the outer Function's saved INPUTS (y0, initial solver state, parameters) with autograd nodes.
    It is wrapped in a Function of its own so that it returns PARTIAL derivatives w.r.t. each input (the initial solver
    state (f0, g0, z0) is itself a function of y0 and the parameters upstream; differentiating through that history
    here would count those paths twice) while staying differentiable: `backward` rebuilds the solve on detached leaves
    and differentiates the first-order gradients (second order; no third).  Memory O(T) like backprop through the
    solver; first-order backward passes never come here."""

    @staticmethod
    def forward(ctx, sde, bm, dt, ts, n_extras, *tensors):
        ctx.sde, ctx.bm, ctx.dt, ctx.n_extras = sde, bm, dt, n_extras
        ctx.save_for_backward(ts, *tensors)
        gouts = tensors[:1 + n_extras]
        with torch.enable_grad():
            leaves = [t.detach().requires_grad_() for t in tensors[1 + n_extras:2 + 2 * n_extras]]
            params = list(tensors[2 + 2 * n_extras:])
            outs = _recomputed_solve(sde, bm, dt, ts, leaves[0], leaves[1:])
            pairs = [(o, g) for o, g in zip(outs, gouts) if o.requires_grad]
            grads = torch.autograd.grad([o for o, _ in pairs], leaves + params, [g for _, g in pairs], allow_unused=True)
        return tuple(torch.zeros_like(x) if g is None else g.detach() for g, x in zip(grads, leaves + params))

    @staticmethod
    def backward(ctx, *gg):
        ts, *tensors = ctx.saved_tensors
        n = ctx.n_extras
        with torch.enable_grad():
            gouts = [t.detach().requires_grad_() for t in tensors[:1 + n]]
            leaves = [t.detach().requires_grad_() for t in tensors[1 + n:2 + 2 * n]]
            params = list(tensors[2 + 2 * n:])
            outs = _recomputed_solve(ctx.sde, ctx.bm, ctx.dt, ts, leaves[0], leaves[1:])
            pairs = [(o, g) for o, g in zip(outs, gouts) if o.requires_grad]
            first = torch.autograd.grad([o for o, _ in pairs], leaves + params, [g for _, g in pairs], create_graph=True,
                                        allow_unused=True)
            sel = [(f, g) for f, g in zip(first, gg) if f is not None and f.requires_grad and g is not None]
            inputs = gouts + leaves + params
            if sel:
                second = torch.autograd.grad([f for f, _ in sel], inputs, [g for _, g in sel], allow_unused=True)
            else:
                second = [None] * len(inputs)
        return (None, None, None, None, None, *second)


def _reversible_backward_differentiable(sde, bm, dt, ts, y0, extras0, params, grad_ys, grad_extras):
    """Gradients w.r.t. (y0, initial solver state, parameters) as differentiable tensors: see _ReversibleVJP."""
    n = len(extras0)
    grads = _ReversibleVJP.apply(sde, bm, dt, ts, n, grad_ys, *grad_extras, y0, *extras0, *params)
    return grads[0], tuple(grads[1:1 + n]), list(grads[1 + n:])


class _SdeintAdjointMethod(torch.autograd.Function):

    @staticmethod
    def forward(ctx, sde, ts, dt, bm, solver, options, adjoint_options, n_extras, y0, *extras_and_params):
        ctx.sde, ctx.dt, ctx.bm, ctx.n_extras = sde, dt, bm, n_extras
        ctx.adjoint_options = adjoint_options
        extras = tuple(x.detach() for x in extras_and_params[:n_extras])
        params = extras_and_params[n_extras:]
        # (with cuda_graph the engine hands out copies of the plan's static buffers: what autograd saves here must
        # not be overwritten by the next solve)
        ys, extras_out = sdeint_mod._integrate(solver, y0.detach(), ts, extras, options)
        ctx.bwd_plan = None
        if adjoint_options.get('cuda_graph', False) and isinstance(bm, BrownianInterval) \
                and adjoint_options_reversible(adjoint_options) and adjoint_options.get('_adaptive') is None:
            engine = _BackwardEngine(sde, ReverseBrownian(bm), dt, params, adjoint_options)
            ctx.bwd_plan = _backward_plan(engine, ys, ts, extras_out)
        # (y0 and the initial solver state are saved as well: the differentiable backward of the reversible pair
        # re-runs the solve from the Function's INPUTS, see _reversible_backward_differentiable)
        ctx.save_for_backward(ys, ts, *extras_out, *params, y0, *extras_and_params[:n_extras])
        return (ys, *extras_out)

    @staticmethod
    def backward(ctx, grad_ys, *grad_extras):
        with _cabi.device_guard(grad_ys.device), _cabi.nvtx_range('tsde: adjoint backward'):
            return _SdeintAdjointMethod._backward(ctx, grad_ys, *grad_extras)

    @staticmethod
    def _backward(ctx, grad_ys, *grad_extras):
        ys, ts, *rest = ctx.saved_tensors
        n_in = 1 + ctx.n_extras
        y0_in, extras_in = rest[-n_in], rest[len(rest) - n_in + 1:]
        rest = rest[:-n_in]
        extras = rest[:ctx.n_extras]
        params = rest[ctx.n_extras:]
        # Double backward (reference adjoint.py:97-113 re-enters the Function so that the backward pass is itself
        # differentiable): when this backward runs with grad mode on (autograd.grad(..., create_graph=True)), the
        # sweep is executed with differentiable operations instead of the fused no-grad kernels.
        differentiable = torch.is_grad_enabled()
        if not adjoint_options_reversible(ctx.adjoint_options):
            # generic adjoint: the solver's extra state is not part of the augmented system (adjoint.py:57-60)
            with (torch.enable_grad() if differentiable else torch.no_grad()):
                adj_y, adj_params = _generic_backward(ctx.sde, ctx.bm, ctx.dt, ys, ts, grad_ys, list(params),
                                                      ctx.adjoint_options['_cfg'], differentiable)
            return (None, None, None, None, None, None, None, None, adj_y, *([None] * ctx.n_extras), *adj_params)
        # (the adjoint state is kept in the state dtype also for 16-bit solver state (f0, g0))
        grad_extras = [widen(torch.zeros_like(e) if g is None else g, ys.dtype) for g, e in zip(grad_extras, extras)]
        if ctx.adjoint_options.get('fused_backward', False) and (differentiable or
                                                                 ctx.adjoint_options.get('_adaptive') is not None):
            warn_unfused("create_graph (double backward)" if differentiable else "adjoint_adaptive")
        if differentiable:
            adj_y, adj_extras, adj_params = _reversible_backward_differentiable(
                ctx.sde, ctx.bm, ctx.dt, ts, y0_in, extras_in, list(params), grad_ys, grad_extras)
            return (None, None, None, None, None, None, None, None, adj_y, *adj_extras, *adj_params)
        with torch.no_grad():
            if ctx.adjoint_options.get('_adaptive') is not None:
                engine = _BackwardEngine(ctx.sde, ReverseBrownian(ctx.bm), ctx.dt, params)
                adj_y, adj_extras, adj_params = engine.run_adaptive(ys, ts, grad_ys, extras, grad_extras,
                                                                    **ctx.adjoint_options['_adaptive'])
            elif ctx.bwd_plan is not None:
                adj_y, adj_extras, adj_params = _replay_backward(ctx.bwd_plan, ctx.bm, ys, grad_ys, extras,
                                                                 grad_extras)
            else:
                engine = _BackwardEngine(ctx.sde, ReverseBrownian(ctx.bm), ctx.dt, params, ctx.adjoint_options)
                adj_y, adj_extras, adj_params = engine.run(ys, ts, grad_ys, extras, grad_extras)
        return (None, None, None, None, None, None, None, None, adj_y, *adj_extras, *adj_params)


def sdeint_adjoint(sde, y0, ts, bm=None, method=None, adjoint_method=None, dt=1e-3, adaptive=False,
                   adjoint_adaptive=False, rtol=1e-5, adjoint_rtol=1e-5, atol=1e-4, adjoint_atol=1e-4,
                   dt_min=1e-5, options=None, adjoint_options=None, adjoint_params=None, names=None,
                   logqp=False, extra=False, extra_solver_state=None, **unused_kwargs):
    """Numerically integrate an SDE with stochastic adjoint support (reference docstring:
    adjoint.py:152-222)."""
    sdeint_mod.handle_unused_kwargs(unused_kwargs, msg="`sdeint_adjoint`")
    del unused_kwargs

    if adjoint_params is None and not isinstance(sde, nn.Module):
        raise ValueError('`sde` must be an instance of nn.Module to specify the adjoint parameters; alternatively they '
                         'can be specified explicitly via the `adjoint_params` argument. If there are no parameters '
                         'then it is allowable to set `adjoint_params=()`.')

    sde, y0, ts, bm, method, options = sdeint_mod.check_contract(sde, y0, ts, bm, method, adaptive, options, names,
                                                                 logqp)
    sdeint_mod.assert_no_grad(['ts', 'dt', 'rtol', 'adjoint_rtol', 'atol', 'adjoint_atol', 'dt_min'],
                              [ts, dt, rtol, adjoint_rtol, atol, adjoint_atol, dt_min])
    adjoint_params = tuple(sde.parameters()) if adjoint_params is None else tuple(adjoint_params)
    adjoint_params = [p for p in adjoint_params if p.requires_grad]
    adjoint_method = _select_default_adjoint_method(sde, method, adjoint_method)
    adjoint_options = {} if adjoint_options is None else adjoint_options.copy()

    if method == METHODS.reversible_heun:  # adjoint.py:243-257
        if adjoint_method != METHODS.adjoint_reversible_heun:
            warnings.warn(f"method={repr(method)}, but adjoint_method!={repr(METHODS.adjoint_reversible_heun)}.")
        if adaptive or adjoint_adaptive:
            warnings.warn(f"A limitation of the current method={repr(method)} implementation is "
                          f"that it does not save the time steps used. This means that it may not be perfectly "
                          f"accurate when used with `adaptive` or `adjoint_adaptive`.")
        else:
            num_steps = (ts - ts[0]) / dt
            if not torch.allclose(num_steps, num_steps.round()):
                warnings.warn(f"The spacing between time points `ts` is not an integer multiple of the time step `dt`. "
                              f"This means that the backward pass (which is forced to step to each of `ts` to get "
                              f"dL/dy(t) for t in ts) will not perfectly mimick the forward pass (which does not step "
                              f"to each `ts`, and instead interpolates to them). This means that "
                              f"method={repr(method)} may not be perfectly accurate.")

    solver_fn = methods.select(method=method, sde_type=sde.sde_type)
    solver = solver_fn(sde=sde, bm=bm, dt=dt, adaptive=adaptive, rtol=rtol, atol=atol, dt_min=dt_min,
                       options=options)
    # constructor-time contract of the adjoint solver (errors as in the reference)
    adjoint_solver_fn = methods.select(method=adjoint_method, sde_type=sde.sde_type)
    adjoint_solver_fn(sde=_AdjointMarker(sde), bm=ReverseBrownian(bm), dt=dt, adaptive=adjoint_adaptive,
                      rtol=adjoint_rtol, atol=adjoint_atol, dt_min=dt_min, options=adjoint_options)
    reversible = method == METHODS.reversible_heun and adjoint_method == METHODS.adjoint_reversible_heun
    if adjoint_method == METHODS.adjoint_reversible_heun and not reversible:
        raise ValueError(f"adjoint_method={repr(adjoint_method)} requires method={repr(METHODS.reversible_heun)}.")
    if reversible and adjoint_adaptive:
        # (the reference has already warned above that this "may not be perfectly accurate", adjoint.py:245-249, and
        # then runs the adjoint solver adaptively; so does the backward engine, see _BackwardEngine.run_adaptive)
        adjoint_options['_adaptive'] = dict(rtol=adjoint_rtol, atol=adjoint_atol, dt_min=dt_min)
    if not reversible:
        # generic AdjointSDE path: remember the adjoint solver's configuration for backward()
        adjoint_options['_cfg'] = dict(adjoint_method=adjoint_method, adjoint_adaptive=adjoint_adaptive,
                                       adjoint_rtol=adjoint_rtol, adjoint_atol=adjoint_atol, dt_min=dt_min,
                                       adjoint_options={k: v for k, v in adjoint_options.items() if k != '_cfg'})

    _cabi.require_cuda(y0)
    if extra_solver_state is None:
        # built with autograd enabled (adjoint.py:270-271): the adjoints of (f0, g0, z0) returned by
        # backward() flow on to y0 and the parameters through these ordinary torch ops
        extra_solver_state = solver.init_extra_solver_state(ts[0], y0)

    with _cabi.device_guard(y0.device):
        ys, *extra_solver_state = _SdeintAdjointMethod.apply(
            sde, ts, dt, bm, solver, options, adjoint_options, len(extra_solver_state), y0, *extra_solver_state,
            *adjoint_params)
    return sdeint_mod.parse_return(y0, ys, extra_solver_state, extra, logqp)


def adjoint_options_reversible(adjoint_options):
    return adjoint_options.get('_cfg') is None


def _select_default_adjoint_method(sde, method, adjoint_method):
    """adjoint.py:281-296."""
    if adjoint_method is not None:
        return adjoint_method
    elif method == METHODS.reversible_heun:
        return METHODS.adjoint_reversible_heun
    else:
        return {
            SDE_TYPES.ito: {
                NOISE_TYPES.diagonal: METHODS.milstein,
                NOISE_TYPES.additive: METHODS.euler,
                NOISE_TYPES.scalar: METHODS.euler,
                NOISE_TYPES.general: METHODS.euler,
            }[sde.noise_type],
            SDE_TYPES.stratonovich: METHODS.midpoint,
        }[sde.sde_type]
