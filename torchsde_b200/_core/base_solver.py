"""Fixed-step SDE solver engine: host-planned time grid + fused CUDA tableau kernels.

Per-step operator contract = the reference's (torchsde/_core/base_solver.py:29-90):
``BaseSDESolver(sde, bm, dt, adaptive, rtol, atol, dt_min, options)`` with class attributes
``strong_order, weak_order, sde_type, noise_types, levy_area_approximations``, the constructor
compatibility checks (:49-58 -> ValueError), ``init_extra_solver_state(t0, y0)`` (:72-73),
``step(t0, t1, y0, extra0) -> (y1, extra1)`` (:75-90) and ``integrate(y0, ts, extra0)``
(:92-149).

What changed underneath:
* ``integrate`` no longer loops over 0-d device tensors.  The grid is planned on the host
  (schedule.py), the Brownian motion is asked once to *bind* that grid (so each step's increment
  is a counter lookup regenerated in registers), every step is {user f/g (torch ops) -> one or
  two fused tableau launches through the C ABI}, ``ys`` is preallocated and each step writes its
  ``y1`` straight into its output row (no ``torch.stack``, no ``linear_interp`` for aligned
  rows; reference :147,149).
* The whole loop — user callables included — can be captured once into a CUDA graph and replayed
  (``options={'cuda_graph': True}``, see graph.py), removing all per-step host work.
"""
import abc
import ctypes
import warnings

import torch

from . import pointwise
from . import schedule as schedule_lib
from .. import _cabi
from .._brownian import BrownianInterval, ReverseBrownian
from ..settings import NOISE_TYPES


def _contig(t):
    return t if t.is_contiguous() else t.contiguous()


def _is_row_broadcast(t):
    """A (rows, d, m) diffusion that is one dense (d, m) block shared by all rows (`sigma.expand(B, d, m)`)."""
    return t.dim() == 3 and t.size(0) > 1 and t.stride(0) == 0 and t.stride(2) == 1 and t.stride(1) == t.size(2) \
        and t.size(2) > 1


def _gop(g):
    """Diffusion operand of a tableau launch: dense, or left as the batch-broadcast view it is (additive noise
    written as `sigma.expand(B, d, m)`): the tile kernels read the shared (d, m) block (TSDE_FLAG_G_BROADCAST)
    instead of a densified copy (at the cfg3 size a 16 MiB write + read per evaluation that the reference pays in
    `repeat` / `bmm`, tests/problems.py:113-116, misc.py:62-63)."""
    if g.is_contiguous() or _is_row_broadcast(g):
        return g
    return g.contiguous()


class StepContext:
    """Everything one step needs besides tensors; built once per solve for every step."""
    __slots__ = ('k', 't0', 't1', 'ft0', 'ft1', 'dt', 'scalars', 'aux_t', 'solver')

    def __init__(self, solver, k, t0, t1, ft0, ft1, dt, scalars, aux_t):
        self.solver = solver
        self.k = k
        self.t0 = t0          # 0-d device tensors handed to the user's f/g
        self.t1 = t1
        self.ft0 = ft0        # python floats (exact values of t0, t1)
        self.ft1 = ft1
        self.dt = dt          # float(t1 - t0), computed in ts' dtype
        self.scalars = scalars  # dict of derived scalars (python floats)
        self.aux_t = aux_t      # list of 0-d device tensors (stage times)


class NoiseFeed:
    """Hands the tableau kernels their Brownian increment for step k.

    counter mode : the bm bound the solver's grid (GridBinding) -> kernels regenerate dW from the
                   Philox counter, nothing is materialised (unless a user g_prod needs the tensor).
    memory mode  : any other BaseBrownian-like object -> bm(ta, tb) is called as the reference does
                   (base_solver.py:54-57 duck typing) and the kernels read its tensors.
    """

    def __init__(self, solver, bm, binding):
        self.solver = solver
        self.bm = bm
        self.binding = binding
        self._nz = _cabi.Noise()
        self._keep = None
        self._cached = None
        if binding is not None:
            self._key_ptr = binding.interval.key_tensor().data_ptr()
            self._row_offset = binding.interval._row_offset
        self._unit = _cabi.Noise()
        self._unit.source = _cabi.SRC_UNIT
        self._unit_ref = ctypes.byref(self._unit)
        self._nz_ref = ctypes.byref(self._nz)

    def unit(self):
        return self._unit_ref

    def prime(self, c, w, u=None):
        """Declare the already-materialised increment of step c (log-ODE queries W and A together)."""
        self._cached = (c, w, u)

    def tensors(self, c, want_u=False):
        """Materialised (W, U) for step c (needed by user-supplied g_prod / f_and_g_prod).
        Cached per step so that the Brownian motion is queried once per step, as in the reference."""
        if self._cached is not None and self._cached[0] is c and (self._cached[2] is not None or not want_u):
            return self._cached[1], self._cached[2]
        w, u = self._tensors(c, want_u)
        self._cached = (c, w, u)
        return w, u

    def _tensors(self, c, want_u):
        s = self.solver
        if self.binding is None:
            if want_u:
                w, u = self.bm(c.ft0, c.ft1, return_U=True)
            else:
                w, u = self.bm(c.ft0, c.ft1), None
            w = _contig(w)
            u = _contig(u) if u is not None else None
            _cabi.require_cuda(w, u)
            if w.dtype != s.dtype:
                raise ValueError(f"Brownian motion returned dtype {w.dtype}, expected {s.dtype}.")
            return w, u
        nz = self.binding.fill(self._nz, c.k, want_u, self._key_ptr, self._row_offset)
        w = torch.empty((s.bm_rows, s.m), dtype=s.dtype, device=s.device)
        u = torch.empty_like(w) if want_u else None
        _cabi.check(_cabi.lib().tsde_brownian_cells(ctypes.byref(s.launch_bm), ctypes.byref(nz), w.data_ptr(),
                                                    None if u is None else u.data_ptr(), None),
                    "tsde_brownian_cells")
        return w, u

    def get(self, c, want_u=False):
        """ctypes reference to a filled `tsde_noise` for step c."""
        if self.binding is not None:
            self.binding.fill(self._nz, c.k, want_u, self._key_ptr, self._row_offset)
            return self._nz_ref
        w, u = self.tensors(c, want_u)
        return self.from_tensors(w, u)

    def from_tensors(self, w, u=None):
        nz = self._nz
        nz.source = _cabi.SRC_MEMORY
        nz.want_u = 0 if u is None else 1
        nz.w = w.data_ptr()
        nz.u = None if u is None else u.data_ptr()
        nz.key = None
        nz.n_cells = 1
        nz.cell_h = None
        self._keep = (w, u)  # keep alive until the launch that consumes it has been enqueued
        return self._nz_ref


class BaseSDESolver(metaclass=abc.ABCMeta):
    """API of the solvers: fixed-step (`integrate` / `_run`) and adaptive (`_integrate_adaptive`)."""

    strong_order = None
    weak_order = None
    sde_type = None
    noise_types = None
    levy_area_approximations = None
    want_u = False  # whether step() needs the space-time Levy area U

    def __init__(self, sde, bm, dt, adaptive, rtol, atol, dt_min, options, **kwargs):
        super(BaseSDESolver, self).__init__(**kwargs)
        # base_solver.py:49-58
        if sde.sde_type != self.sde_type:
            raise ValueError(f"SDE is of type {sde.sde_type} but solver is for type {self.sde_type}")
        if sde.noise_type not in self.noise_types:
            raise ValueError(f"SDE has noise type {sde.noise_type} but solver only supports noise types "
                             f"{self.noise_types}")
        if bm.levy_area_approximation not in self.levy_area_approximations:
            raise ValueError(f"SDE solver requires one of {self.levy_area_approximations} set as the "
                             f"`levy_area_approximation` on the Brownian motion.")
        if sde.noise_type == NOISE_TYPES.scalar and torch.Size(bm.shape[1:]).numel() != 1:  # noqa
            raise ValueError("The Brownian motion for scalar SDEs must of dimension 1.")

        self.sde = sde
        self.bm = bm
        self.dt = dt
        self.adaptive = adaptive
        self.rtol = rtol
        self.atol = atol
        self.dt_min = dt_min
        self.options = options
        self._prepared = False
        self._side_streams = []
        self._err_buf = None
        self._autograd = False
        self._cur_c = None

    def __repr__(self):
        return f"{self.__class__.__name__} of strong order: {self.strong_order}, and weak order: {self.weak_order}"

    # ------------------------------------------------------------------------------------------
    def init_extra_solver_state(self, t0, y0):
        return ()

    def aux_times(self, t0, t1, dt):
        """Stage times other than t0, t1, as 0-d CPU tensors (same expressions as the reference)."""
        return []

    def scalars(self, dt):
        """Derived scalars of a step, from the 0-d CPU tensor dt (same expressions as the reference)."""
        return {}

    @abc.abstractmethod
    def _step(self, c, y0, extra0, out):
        """Advance one step.  Returns (y1, extra1); on the fast path y1 is written into `out` (a (rows, d)
        tensor, e.g. a row of ys) when `out` is given."""
        raise NotImplementedError

    # ------------------------------------------------------------------------------------------
    # launching
    # ------------------------------------------------------------------------------------------
    def _out_like(self, name, ins):
        if name == 'tsde_milstein_vjp_seed':
            return torch.empty_like(ins[0])  # grad_outputs has g's shape
        return torch.empty((self.rows, self.d), dtype=self.dtype, device=self.device)

    def _launch(self, name, L, nz, ins, scalars, outs, dtype_word):
        """`dtype_word`: the state dtype and the formats of 16-bit SDE outputs (_cabi.operands); the shared launch
        descriptor carries it for this call only."""
        flags = 0
        g3 = [t for t in ins if t.dim() == 3 and not t.is_contiguous()]
        if g3:
            every = [t for t in ins if t.dim() == 3]
            # the flag describes ALL (rows, d, m) operands of the launch, and only the general-noise tile kernels
            # fed by the step's own noise descriptor understand it
            if len(g3) == len(every) and L is self._L and self.m > 1 and nz is self._feed._nz_ref \
                    and all(_is_row_broadcast(t) for t in g3):
                flags = _cabi.FLAG_G_BROADCAST
            else:
                ins = [_contig(t) for t in ins]
        if nz is self._feed._nz_ref:
            self._feed._nz.flags = flags
        args = [L] if nz is None else [L, nz]
        args += [t.data_ptr() for t in ins]
        args += list(scalars)
        args += [o.data_ptr() for o in outs]
        launch = L._obj
        launch.dtype = dtype_word
        try:
            code = getattr(self._lib, name)(*args)
        finally:
            launch.dtype = dtype_word & 0xff
        _cabi.check(code, name)

    def _k(self, name, L, nz, ins, scalars, out, n_out=1, raw=False):
        """One C-ABI tableau launch `name(L, [nz], *ins, *scalars, *outs)`.  Fast path: direct launch into
        `out` (allocated if None).  When gradients flow through the solve (`sdeint` under autograd) the
        launch becomes an autograd node (autograd_ops.TableauFn)."""
        if self._autograd and not raw:
            from .autograd_ops import TableauFn
            unit = nz is not None and nz is self._feed._unit_ref
            noise = None
            if nz is not None and not unit:
                noise = self._feed.tensors(self._cur_c, self.want_u)
            return TableauFn.apply(self, name, L is self._L, unit, noise, tuple(scalars), n_out, *ins)
        word, ins = _cabi.operands(name, self.dtype, ins)
        if n_out == 1:
            o = out if out is not None else self._out_like(name, ins)
            self._launch(name, L, nz, ins, scalars, (o,), word)
            return o
        outs = tuple(self._out_like(name, ins) for _ in range(n_out))
        self._launch(name, L, nz, ins, scalars, outs, word)
        return outs

    def _launch_raw(self, name, use_general, unit, noise, ins, scalars, n_out):
        """Forward of an autograd node: same kernel, increments taken from the saved tensors."""
        L = self._L if use_general else self._LU
        if unit:
            nz = self._feed.unit()
        elif noise is not None:
            nz = self._feed.from_tensors(noise[0], noise[1])
        else:
            nz = None
        word, ins = _cabi.operands(name, self.dtype, [_contig(t) for t in ins])
        outs = tuple(self._out_like(name, ins) for _ in range(n_out))
        self._launch(name, L, nz, ins, scalars, outs, word)
        return outs

    # ------------------------------------------------------------------------------------------
    def _prepare(self, y0):
        _cabi.require_cuda(y0)
        _cabi.lib()  # fail loudly if the CUDA library is missing
        self.dtype = y0.dtype
        self.device = y0.device
        self.rows, self.d = y0.shape
        self.m = int(torch.Size(self.bm.shape[1:]).numel()) if len(self.bm.shape) > 1 else 1
        # rows of the Brownian tensors; differs from the state's rows only for the flat (1, N) augmented
        # state of the generic adjoint, whose products are formed by AdjointSDE itself
        self.bm_rows = int(self.bm.shape[0]) if len(self.bm.shape) > 1 else 1
        diag = self.sde.noise_type == NOISE_TYPES.diagonal
        nt = _cabi.NOISE_DIAGONAL if diag else _cabi.NOISE_GENERAL
        stream = torch.cuda.current_stream(self.device).cuda_stream
        self.launch = _cabi.make_launch(self.dtype, nt, self.rows, self.d, self.m, stream)
        # user-supplied products arrive as (rows, d): element-wise launch with unit noise
        self.launch_unit = _cabi.make_launch(self.dtype, _cabi.NOISE_DIAGONAL, self.rows, self.d, self.d, stream)
        # Brownian tensors are (rows, m)
        self.launch_bm = _cabi.make_launch(self.dtype, _cabi.NOISE_DIAGONAL, self.bm_rows, self.m, self.m, stream)
        self._L = ctypes.byref(self.launch)
        self._LU = ctypes.byref(self.launch_unit)
        self._LB = ctypes.byref(self.launch_bm)
        self._lib = _cabi.lib()
        self._prepared = True

    # -- independent user callables as parallel branches -------------------------------------------------------
    # Within a step f(t, y) and g(t, y) (and the stage evaluations of SRK that share their inputs) are independent
    # given y.  Issued on different streams they become parallel branches of the captured graph (fork / join), so
    # their kernels' launch latencies overlap instead of adding up.  That is what limits small-state workloads: at
    # the cfg3 size (1 MiB states) a step is a chain of 4-30 tiny PyTorch kernels of the user's f / g at ~2.5 us of
    # dependent-launch latency each, while the solver's own kernels take a few us.  On by default;
    # `options={'overlap': False}` turns it off.
    # Memory discipline: a branch's results are allocated on its side stream and consumed on the main stream after
    # the join; they are freed (returned to the side stream's pool) only after that consumer has been enqueued, and
    # the side stream reuses the block only after its next fork, i.e. after waiting for the main stream — so no
    # `record_stream` is needed (under graph capture it would defer every free to the end of the capture).
    # Evaluation order of f and g is not observable for pure callables; SDEs whose callables have side effects can
    # set options={'overlap': False}.
    def _overlap_now(self):
        if self._autograd:
            return False  # (AccumulateGrad nodes remember the stream they were created on: keep one stream)
        opt = self.options.get('overlap')
        return True if opt is None else bool(opt)

    def _fork(self, *thunks, main=0):
        """Results of independent thunks, called in the order given (the reference's call order).  thunks[main] runs
        on the current stream (it may contain this library's launches, which go to that stream), the others on side
        streams."""
        if len(thunks) == 1 or not self._overlap_now():
            return [t() for t in thunks]
        cur = torch.cuda.current_stream(self.device)
        while len(self._side_streams) < len(thunks) - 1:
            self._side_streams.append(torch.cuda.Stream(device=self.device))
        sides = iter(self._side_streams)
        used = []
        outs = []
        fork_point = cur.record_event()  # every branch depends on what precedes the fork, not on its siblings
        for i, thunk in enumerate(thunks):
            if i == main:
                outs.append(thunk())
                continue
            side = next(sides)
            side.wait_event(fork_point)
            with torch.cuda.stream(side):
                outs.append(thunk())
            used.append(side)
        for side in used:
            cur.wait_stream(side)
        return outs

    def _f_and_g(self, t, y):
        """sde.f_and_g(t, y); when the user did not fuse them, f and g are evaluated as parallel branches."""
        sde = self.sde
        if getattr(sde, 'user_f_and_g', True) or getattr(sde, 'is_adjoint_sde', False):
            return sde.f_and_g(t, y)
        return self._fork(lambda: sde.f(t, y), lambda: sde.g(t, y))

    def _refresh_stream(self):
        stream = torch.cuda.current_stream(self.device).cuda_stream
        self.launch.stream = stream
        self.launch_unit.stream = stream
        self.launch_bm.stream = stream

    def _bind(self, sched):
        """Ask the Brownian motion to adopt the solver grid (fast path) if it can."""
        bm = self.bm
        binding = None
        if getattr(self, 'needs_levy_area', False):
            return None
        if isinstance(bm, BrownianInterval):
            binding = bm.bind_grid(sched.bounds)
        elif isinstance(bm, ReverseBrownian) and isinstance(bm.base_brownian, BrownianInterval):
            fwd = bm.base_brownian.bind_grid([-b for b in reversed(sched.bounds)])
            binding = None if fwd is None else fwd.reversed()
        return binding

    def _contexts(self, sched, ts):
        """Per-step contexts; all scalar arithmetic in ts' dtype on the host, one H2D copy."""
        n = sched.n_steps
        if n == 0:
            return []
        cpu_t0 = [s[0] for s in sched.steps]
        cpu_t1 = [s[1] for s in sched.steps]
        cpu_dt = [b - a for a, b in sched.steps]
        aux = [self.aux_times(a, b, h) for a, b, h in zip(cpu_t0, cpu_t1, cpu_dt)]
        n_aux = len(aux[0])
        table = torch.stack([torch.stack([a, b] + list(x)) for a, b, x in zip(cpu_t0, cpu_t1, aux)])
        table = table.to(ts.dtype).to(self.device, non_blocking=False)  # (n, 2 + n_aux)
        self._time_table = table  # keep alive (static addresses for graph replay)
        ctxs = []
        for k in range(n):
            row = table[k]
            ctxs.append(StepContext(self, k, row[0], row[1], sched.bounds[k], sched.bounds[k + 1],
                                    float(cpu_dt[k]), self.scalars(cpu_dt[k]),
                                    [row[2 + j] for j in range(n_aux)]))
        return ctxs

    # ------------------------------------------------------------------------------------------
    def _context(self, t0, t1):
        """The context of a single step from t0 to t1 (`step`, and the sub-steps of a fused adaptive proposal)."""
        t0 = torch.as_tensor(t0)
        t1 = torch.as_tensor(t1)
        c0, c1 = t0.detach().cpu(), t1.detach().cpu()
        dt = c1 - c0
        aux = [a.to(self.device) for a in self.aux_times(c0, c1, dt)]
        return StepContext(self, 0, t0.to(self.device), t1.to(self.device), float(c0), float(c1), float(dt),
                           self.scalars(dt), aux)

    def step(self, t0, t1, y0, extra0):
        """Reference-compatible single step (base_solver.py:75-90): queries ``self.bm(t0, t1)``."""
        if not self._prepared:
            self._prepare(y0)
        self._refresh_stream()
        c = self._context(t0, t1)
        self._feed = NoiseFeed(self, self.bm, None)
        self._cur_c = c
        if self._autograd:
            return self._step(c, y0, extra0, None)
        with torch.no_grad():
            return self._step(c, _contig(y0.detach()), extra0, None)

    def integrate(self, y0, ts, extra0):
        """Integrate along trajectory.  Returns ys (T, batch, d) and the final extra state
        (base_solver.py:92-149, fixed-step branch)."""
        if self.adaptive:
            return self._integrate_adaptive(y0, ts, extra0)
        sched = schedule_lib.get_schedule(ts, self.dt)
        if self._autograd:
            y0 = _contig(y0)
            self._prepare(y0)
            self._feed = NoiseFeed(self, self.bm, self._bind(sched))
            return self._run_autograd(sched, self._contexts(sched, ts), y0, tuple(extra0))
        y0 = _contig(y0.detach())
        self._prepare(y0)
        binding = self._bind(sched)
        self._feed = NoiseFeed(self, self.bm, binding)
        ctxs = self._contexts(sched, ts)
        T = ts.numel()
        ys = torch.empty((T, self.rows, self.d), dtype=self.dtype, device=self.device)
        ys[0].copy_(y0)
        extra = tuple(extra0)
        with torch.no_grad():
            extra = self._run(sched, ctxs, ys, extra)
        return ys, extra

    # ------------------------------------------------------------------------------------------
    # adaptive time-stepping (base_solver.py:117-142, adaptive_stepping.py:21-76)
    # ------------------------------------------------------------------------------------------
    def _error_estimate(self, y_full, y_half):
        """compute_error of adaptive_stepping.py:42-69: RMS of (y11 - y12) / tol, reduced on the GPU."""
        eps = 1e-7
        # (an empty batch has no error to estimate: the reference's mean over zero elements is nan and trips the
        # same assertion, adaptive_stepping.py:67-68)
        assert y_full.numel() > 0, ('Found nans in the error estimate. Try increasing the tolerance or regularizing '
                                    'the dynamics.')
        if self._err_buf is None:
            self._err_buf = torch.zeros(1024, dtype=torch.float64, device=self.device)
        buf = self._err_buf
        _cabi.check(self._lib.tsde_adaptive_error_sumsq(self._LU, y_full.data_ptr(), y_half.data_ptr(),
                                                        float(self.rtol), float(self.atol), eps,
                                                        buf[1:].data_ptr(), buf.data_ptr()),
                    "tsde_adaptive_error_sumsq")
        total = float(buf[0].item())  # the one host sync per step, as in the reference (:69)
        err = (total / y_full.numel()) ** 0.5
        assert err == err, ('Found nans in the error estimate. Try increasing the tolerance or regularizing '
                            'the dynamics.')
        return max(err, eps)

    @staticmethod
    def _update_step_size(error_estimate, prev_step_size, safety=0.9, facmin=0.2, facmax=1.4,
                          prev_error_ratio=None):
        """PI step-size controller, adaptive_stepping.py:21-39."""
        if error_estimate > 1:
            pfactor, ifactor = 0, 1 / 1.5
        else:
            pfactor, ifactor = 0.13, 1 / 4.5
        error_ratio = safety / error_estimate
        if prev_error_ratio is None:
            prev_error_ratio = error_ratio
        factor = error_ratio ** ifactor * (error_ratio / prev_error_ratio) ** pfactor
        if error_estimate <= 1:
            prev_error_ratio = error_ratio
            facmin = 1.0
        factor = min(facmax, max(facmin, factor))
        return prev_step_size * factor, prev_error_ratio

    def _propose(self, curr_t, next_t, midpoint_t, curr_y, curr_extra):
        """One proposal of the adaptive loop: the full step to next_t and the two half steps through midpoint_t, as
        (y_full, y_next, extra_next).  Methods whose proposal can run as one kernel override it (methods.py)."""
        next_y_full, _ = self.step(curr_t, next_t, curr_y, curr_extra)
        midpoint_y, midpoint_extra = self.step(curr_t, midpoint_t, curr_y, curr_extra)
        next_y, next_extra = self.step(midpoint_t, next_t, midpoint_y, midpoint_extra)
        return next_y_full, next_y, next_extra

    def _integrate_adaptive(self, y0, ts, extra0):
        """One full step vs two half steps per proposal; accept / reject on the host.  Step sizes are
        data dependent, so this branch is an eager loop (one device->host scalar per proposal, exactly
        the reference's sync count) and the Brownian motion is queried at arbitrary times through
        ``bm(ta, tb)``; every step still runs the fused tableau kernels, and an element-wise SDE's proposal is one
        kernel (`_propose`, pointwise.propose).  When gradients flow through the solve
        (`self._autograd`) every launch is an autograd node, as in the fixed-step loop; the error estimate
        never carries gradient (the reference turns it into a Python float, base_solver.py:127-134)."""
        track = self._autograd
        y0 = _contig(y0 if track else y0.detach())
        self._prepare(y0)
        self._err_buf = None
        ts_cpu = ts.detach().to('cpu')
        step_size = self.dt.detach().to('cpu') if torch.is_tensor(self.dt) else self.dt
        prev_t = curr_t = ts_cpu[0]
        prev_y = curr_y = y0
        curr_extra = tuple(extra0)
        T = ts.numel()
        if track:
            rows = [y0]
        else:
            ys = torch.empty((T, self.rows, self.d), dtype=self.dtype, device=self.device)
            ys[0].copy_(y0)
        prev_error_ratio = None
        with (torch.enable_grad() if track else torch.no_grad()):
            for i in range(1, T):
                out_t = ts_cpu[i]
                while curr_t < out_t:
                    next_t = min(curr_t + step_size, ts_cpu[-1])
                    midpoint_t = 0.5 * (curr_t + next_t)
                    next_y_full, next_y, next_extra = self._propose(curr_t, next_t, midpoint_t, curr_y, curr_extra)
                    error_estimate = self._error_estimate(_contig(next_y_full.detach()), _contig(next_y.detach()))
                    step_size, prev_error_ratio = self._update_step_size(
                        error_estimate=error_estimate, prev_step_size=step_size, prev_error_ratio=prev_error_ratio)
                    if step_size < self.dt_min:
                        warnings.warn("Hitting minimum allowed step size in adaptive time-stepping.")
                        step_size = self.dt_min
                        prev_error_ratio = None
                    if error_estimate <= 1 or step_size <= self.dt_min:
                        prev_t, prev_y = curr_t, curr_y
                        curr_t, curr_y, curr_extra = next_t, next_y, next_extra
                # interp.py:15-18
                if bool(curr_t == out_t):
                    out = curr_y
                    w0 = w1 = None
                else:
                    w0 = float((curr_t - out_t) / (curr_t - prev_t))
                    w1 = float((out_t - prev_t) / (curr_t - prev_t))
                if track:
                    rows.append(curr_y if w0 is None else
                                self._k('tsde_linear_interp', self._LU, None, (prev_y, curr_y), (w0, w1), None))
                elif w0 is None:
                    ys[i].copy_(curr_y)
                else:
                    _cabi.check(self._lib.tsde_linear_interp(self._LU, prev_y.data_ptr(), curr_y.data_ptr(), w0, w1,
                                                             ys[i].data_ptr()), "tsde_linear_interp")
        if track:
            return torch.stack(rows, dim=0), curr_extra
        return ys, curr_extra

    def _chunks_ready(self):
        """Whether the steps from here on may run several per launch (`_step_chunk`)."""
        return False

    def _step_chunk(self, ctxs, y0, extra0, outs):
        """Advance the consecutive steps `ctxs` in one launch, storing step j's y1 to outs[j] (None: not stored; the
        last is given).  Returns (y1 of the last step, extra1)."""
        raise NotImplementedError

    def _run(self, sched, ctxs, ys, extra):
        """The time loop proper: capturable (no syncs, no host-dependent control flow).  Once `_chunks_ready`, steps
        run in the chunks of pointwise.plan_chunks."""
        self._refresh_stream()
        curr = ys[0]
        prev = curr
        scratch = [None, None]
        flip = 0

        def dest(k):  # where the state after step k must be: its output row, else a scratch buffer
            nonlocal flip
            row = sched.aligned_row(k)
            if row is not None:
                return ys[row]
            if scratch[flip] is None:
                scratch[flip] = torch.empty_like(ys[0])
            flip ^= 1
            return scratch[flip ^ 1]

        chunks = None
        k = 0
        while k < len(ctxs):
            if chunks is None and self._chunks_ready():
                interpolated = [j for j, os in sched.outputs_after.items() if any(not o.aligned for o in os)]
                multi = [j for j in range(k, len(ctxs)) if self._feed.binding.cell(ctxs[j].k)[2] > 1]
                chunks = iter(pointwise.plan_chunks(k, len(ctxs), interpolated, multi, pointwise.chunk_length(self)))
            k1 = next(chunks)[1] if chunks is not None else k + 1
            self._cur_c = ctxs[k1 - 1]
            if k1 == k + 1:
                y1, extra = self._step(ctxs[k], curr, extra, dest(k))
            else:
                rows = [sched.aligned_row(j) for j in range(k, k1 - 1)]
                outs = [None if r is None else ys[r] for r in rows] + [dest(k1 - 1)]
                y1, extra = self._step_chunk(ctxs[k:k1], curr, extra, outs)
            k = k1
            prev, curr = curr, y1
            for o in sched.outputs_after.get(k - 1, ()):
                if not o.aligned:
                    # interp.py:15-18
                    _cabi.check(self._lib.tsde_linear_interp(self._LU, prev.data_ptr(), curr.data_ptr(),
                                                             o.w0, o.w1, ys[o.index].data_ptr()),
                                "tsde_linear_interp")
        return extra

    def _run_autograd(self, sched, ctxs, y0, extra):
        """Differentiable time loop (plain `sdeint` under autograd): every launch is an autograd node,
        outputs are collected and stacked like the reference does (base_solver.py:112,147,149)."""
        self._refresh_stream()
        ys = [y0]
        prev = curr = y0
        for k, c in enumerate(ctxs):
            self._cur_c = c
            y1, extra = self._step(c, curr, extra, None)
            prev, curr = curr, y1
            for o in sched.outputs_after.get(k, ()):
                if o.aligned:
                    ys.append(curr)
                else:
                    ys.append(self._k('tsde_linear_interp', self._LU, None, (prev, curr), (o.w0, o.w1), None))
        return torch.stack(ys, dim=0), extra
