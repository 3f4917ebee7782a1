"""`sdeint`: public entry point of the forward solve.

Signature, defaults, validation errors and return conventions follow the reference
(torchsde/_core/sdeint.py: `sdeint` :27-112, `check_contract` :115-281, `parse_return`
:284-300); the integration itself is done by the CUDA engine (base_solver.py, methods.py).

Known differences, by design:
* tensors must live on a CUDA device (there is no CPU path);
* gradients flow through `sdeint` (each tableau launch is an autograd node, autograd_ops.py) when autograd
  is enabled and y0 / the SDE's parameters require grad; that path is an eager loop with materialised
  increments — wrap inference in `torch.no_grad()` (or use `sdeint_adjoint`) to get the fused fast path;
* `adaptive=True` runs the reference's controller as an eager loop (data-dependent step sizes cannot be
  graph-captured); every proposal still uses the fused kernels.
"""
import warnings

import torch

from . import base_sde
from . import methods
from . import schedule as schedule_lib
from .. import _cabi
from .._brownian import BrownianInterval
from ..settings import LEVY_AREA_APPROXIMATIONS, METHODS, NOISE_TYPES, SDE_TYPES


def handle_unused_kwargs(unused_kwargs, msg=None):
    # misc.py:26-31
    if len(unused_kwargs) > 0:
        if msg is not None:
            warnings.warn(f"{msg}: Unexpected arguments {unused_kwargs}")
        else:
            warnings.warn(f"Unexpected arguments {unused_kwargs}")


def assert_no_grad(names, maybe_tensors):
    # misc.py:20-23
    for name, maybe_tensor in zip(names, maybe_tensors):
        if torch.is_tensor(maybe_tensor) and maybe_tensor.requires_grad:
            raise ValueError(f"Argument {name} must not require gradient.")


def sdeint(sde, y0, ts, bm=None, method=None, dt=1e-3, adaptive=False, rtol=1e-5, atol=1e-4, dt_min=1e-5,
           options=None, names=None, logqp=False, extra=False, extra_solver_state=None, **unused_kwargs):
    """Numerically integrate an SDE (reference docstring: sdeint.py:43-92).

    Returns ys of size (T, batch_size, d); with `logqp` also the log-ratio increments (T-1, batch);
    with `extra` also the solver's final extra state.
    """
    handle_unused_kwargs(unused_kwargs, msg="`sdeint`")
    del unused_kwargs

    sde, y0, ts, bm, method, options = check_contract(sde, y0, ts, bm, method, adaptive, options, names, logqp)
    assert_no_grad(['ts', 'dt', 'rtol', 'atol', 'dt_min'], [ts, dt, rtol, atol, dt_min])

    solver_fn = methods.select(method=method, sde_type=sde.sde_type)
    solver = solver_fn(sde=sde, bm=bm, dt=dt, adaptive=adaptive, rtol=rtol, atol=atol, dt_min=dt_min,
                       options=options)
    _cabi.require_cuda(y0)
    with _cabi.device_guard(y0.device), _cabi.nvtx_range(f'tsde: sdeint {method}'):
        # (launches go to y0's device whatever the caller's current device is)
        return _solve(sde, solver, y0, ts, adaptive, options, logqp, extra, extra_solver_state)


def _solve(sde, solver, y0, ts, adaptive, options, logqp, extra, extra_solver_state):
    if _needs_autograd(sde, y0, extra_solver_state):
        # gradients must flow through the solve: every tableau launch becomes an autograd node
        # (autograd_ops.py); eager loop, increments materialised (memory O(T), like the reference).  Adaptive
        # solves take the same route: their accepted steps are ordinary (differentiable) steps.
        solver._autograd = True
        sde.widen_outputs(y0.dtype)  # each 16-bit output widened once: see ForwardSDE.widen_outputs
        if extra_solver_state is None:
            extra_solver_state = solver.init_extra_solver_state(ts[0], y0)
        ys, extra_solver_state = solver.integrate(y0, ts, extra_solver_state)
        return parse_return(y0, ys, extra_solver_state, extra, logqp)
    with torch.no_grad():
        if extra_solver_state is None:
            extra_solver_state = solver.init_extra_solver_state(ts[0], y0)
        ys, extra_solver_state = _integrate(solver, y0, ts, extra_solver_state, options)
    return parse_return(y0, ys, extra_solver_state, extra, logqp)


def _needs_autograd(sde, y0, extra_solver_state):
    """Do gradients have to flow through this solve?  Yes if autograd is on and y0, a parameter of the SDE, the given
    solver state, or — for SDEs that are not Modules, or that close over foreign tensors such as an encoder's context
    (`contextualize`) — anything f / g returned while the contract was probed requires grad."""
    if not torch.is_grad_enabled():
        return False
    if y0.requires_grad or any(p.requires_grad for p in sde.parameters()):
        return True
    if getattr(sde, 'probe_requires_grad', False):
        return True
    return any(torch.is_tensor(e) and e.requires_grad for e in (extra_solver_state or ()))


def _integrate(solver, y0, ts, extra_solver_state, options, static_ok=False):
    if options.get('cuda_graph', False) and not solver.adaptive:
        from . import graph
        return graph.integrate_captured(solver, y0, ts, extra_solver_state, static_ok)
    return solver.integrate(y0, ts, extra_solver_state)


class _Sizes:
    """Collects the batch / state / noise sizes seen while probing the SDE (sdeint.py:168-248)."""

    def __init__(self, noise_type):
        self.noise_type = noise_type
        self.batch, self.state, self.noise = [], [], []
        self.requires_grad = False  # did any probed output carry gradient (see _needs_autograd)?

    def seen(self, *tensors):
        self.requires_grad = self.requires_grad or any(torch.is_tensor(t) and t.requires_grad for t in tensors)
        return tensors[0] if len(tensors) == 1 else tensors

    def two_d(self, name, shape):
        if len(shape) != 2:
            raise ValueError(f"{name} must be of shape (batch, state_channels), but got {shape}.")
        self.batch.append(shape[0])
        self.state.append(shape[1])

    def diffusion(self, name, shape):
        if self.noise_type == NOISE_TYPES.diagonal:
            if len(shape) != 2:
                raise ValueError(f"{name} must be of shape (batch, state_channels), but got {shape}.")
            self.batch.append(shape[0])
            self.state.append(shape[1])
            self.noise.append(shape[1])
        else:
            if len(shape) != 3:
                raise ValueError(f"{name} must be of shape (batch, state_channels, noise_channels), but got {shape}.")
            self.batch.append(shape[0])
            self.state.append(shape[1])
            self.noise.append(shape[2])

    def need_noise_size(self):
        if len(self.noise) == 0:
            raise ValueError("Cannot infer noise size (i.e. number of Brownian motion channels). Either pass `bm` "
                             "explicitly, or specify one of the `g`, `f_and_g` functions.`")

    def consistent(self):
        if any(b != self.batch[0] for b in self.batch[1:]):
            raise ValueError("Batch sizes not consistent.")
        if any(s != self.state[0] for s in self.state[1:]):
            raise ValueError("State sizes not consistent.")
        if any(n != self.noise[0] for n in self.noise[1:]):
            raise ValueError("Noise sizes not consistent.")


_TS_FROM_LIST = {}


def _tensor_from_list(values, dtype, device):
    """`ts` given as a list/tuple of floats (sdeint.py:161-164): the tensor is built once per distinct
    (values, dtype, device) so that the host-side plan of the grid can be reused across calls."""
    key = (values, dtype, str(device))
    t = _TS_FROM_LIST.get(key)
    if t is None:
        if len(_TS_FROM_LIST) >= 16:
            _TS_FROM_LIST.pop(next(iter(_TS_FROM_LIST)))
        t = _TS_FROM_LIST[key] = torch.tensor(values, dtype=dtype, device=device)
    return t


def default_method(sde_type, noise_type):
    """Solver used when `method` is None (reference sdeint.py:147-153): midpoint for Stratonovich SDEs, else Euler for
    general noise and SRK for the noise types SRK supports."""
    if sde_type == SDE_TYPES.stratonovich:
        return METHODS.midpoint
    return METHODS.euler if noise_type == NOISE_TYPES.general else METHODS.srk


def default_levy_area(method):
    """Levy-area mode of the BrownianInterval created when `bm` is None (reference sdeint.py:262-268)."""
    return {METHODS.srk: LEVY_AREA_APPROXIMATIONS.space_time,
            METHODS.log_ode_midpoint: LEVY_AREA_APPROXIMATIONS.foster}.get(method, LEVY_AREA_APPROXIMATIONS.none)


def _checked_kinds(sde):
    for attr, allowed, label in (('noise_type', NOISE_TYPES, 'noise type'), ('sde_type', SDE_TYPES, 'sde type')):
        if not hasattr(sde, attr):
            raise ValueError(f"sde does not have the attribute {attr}.")
        if getattr(sde, attr) not in allowed:
            raise ValueError(f"Expected {label} in {allowed}, but found {getattr(sde, attr)}.")


def _time_tensor(ts, like):
    """`ts` as a 1-D tensor in y0's dtype / device, strictly increasing (reference sdeint.py:161-166)."""
    if not torch.is_tensor(ts):
        floats = isinstance(ts, (tuple, list)) and all(isinstance(t, (float, int)) for t in ts)
        if not floats:
            raise ValueError("Evaluation times `ts` must be a 1-D Tensor or list/tuple of floats.")
        ts = _tensor_from_list(tuple(ts), like.dtype, like.device)
    values = schedule_lib.ts_values(ts)
    if not all(earlier < later for earlier, later in zip(values, values[1:])):  # (a NaN time fails here too)
        raise ValueError("Evaluation times `ts` must be strictly increasing.")
    return ts


def _probe(sde, t0, y0, sizes):
    """Call every callable the SDE offers once and record the sizes it reports (reference sdeint.py:168-243).  Returns
    (drift available, diffusion available)."""
    have_f = have_g = False

    def test_vector():
        sizes.need_noise_size()
        return torch.randn(sizes.batch[0], sizes.noise[0], dtype=y0.dtype, device=y0.device)

    # (the reference probes under no_grad; here the probe also records whether the SDE's outputs carry gradient,
    # so it runs in the caller's grad mode — the outputs are dropped immediately either way)
    if hasattr(sde, 'f'):
        have_f = True
        sizes.two_d('Drift', tuple(sizes.seen(sde.f(t0, y0)).size()))
    if hasattr(sde, 'g'):
        have_g = True
        sizes.diffusion('Diffusion', tuple(sizes.seen(sde.g(t0, y0)).size()))
    if hasattr(sde, 'f_and_g'):
        have_f = have_g = True
        drift, diffusion = sizes.seen(*sde.f_and_g(t0, y0))
        sizes.two_d('Drift', tuple(drift.size()))
        sizes.diffusion('Diffusion', tuple(diffusion.size()))
    if hasattr(sde, 'g_prod'):
        have_g = True
        sizes.two_d('Diffusion-vector product', tuple(sizes.seen(sde.g_prod(t0, y0, test_vector())).size()))
    if hasattr(sde, 'f_and_g_prod'):
        have_f = have_g = True
        drift, product = sizes.seen(*sde.f_and_g_prod(t0, y0, test_vector()))
        sizes.two_d('Drift', tuple(drift.size()))
        sizes.two_d('Diffusion-vector product', tuple(product.size()))
    return have_f, have_g


def check_contract(sde, y0, ts, bm, method, adaptive, options, names, logqp):
    """Validate and normalise the arguments of a solve; every violation is a ValueError, as in the reference
    (sdeint.py:115-281).  Returns (ForwardSDE, y0, ts tensor, bm, method, options copy)."""
    if names:
        known = ("drift", "diffusion", "prior_drift", "drift_and_diffusion", "drift_and_diffusion_prod")
        rename = {role: names[role] for role in known if role in names}
        if rename:
            sde = base_sde.RenameMethodsSDE(sde, **rename)
    _checked_kinds(sde)

    if not torch.is_tensor(y0):
        raise ValueError("`y0` must be a torch.Tensor.")
    if y0.dim() != 2:
        raise ValueError("`y0` must be a 2-dimensional tensor of shape (batch, channels).")
    if logqp:  # one more state channel integrates the KL rate (v0.1.1 compatibility, sdeint.py:141-145)
        sde = base_sde.SDELogqp(sde)
        y0 = torch.cat((y0, y0.new_zeros(size=(y0.size(0), 1))), dim=1)

    if method is None:
        method = default_method(sde.sde_type, sde.noise_type)
    if method not in METHODS:
        raise ValueError(f"Expected method in {METHODS}, but found {method}.")
    ts = _time_tensor(ts, y0)

    sizes = _Sizes(sde.noise_type)
    sizes.batch.append(y0.size(0))
    sizes.state.append(y0.size(1))
    if bm is not None:
        if len(bm.shape) != 2:
            raise ValueError("`bm` must be of shape (batch, noise_channels).")
        sizes.batch.append(bm.shape[0])
        sizes.noise.append(bm.shape[1])
    have_f, have_g = _probe(sde, ts[0], y0, sizes)
    if not have_f:
        raise ValueError("sde must define at least one of `f`, `f_and_g`, or `f_and_g_prod`. (Or possibly more "
                         "depending on the method chosen.)")
    if not have_g:
        raise ValueError("sde must define at least one of `g`, `f_and_g`, `g_prod` or `f_and_g_prod`. (Or possibly "
                         "more depending on the method chosen.)")
    sizes.consistent()
    if sde.noise_type == NOISE_TYPES.scalar and sizes.noise[0] != 1:
        raise ValueError(f"Scalar noise must have only one channel; the diffusion has {sizes.noise[0]} noise channels.")

    sde = base_sde.ForwardSDE(sde)
    sde.probe_requires_grad = sizes.requires_grad
    if y0.dtype == torch.float64:
        sde.widen_outputs(torch.float64)  # (the kernels take 16-bit SDE outputs with a float32 state only)
    if bm is None:
        span = schedule_lib.ts_values(ts)
        bm = BrownianInterval(t0=span[0], t1=span[-1], size=(sizes.batch[0], sizes.noise[0]), dtype=y0.dtype,
                              device=y0.device, levy_area_approximation=default_levy_area(method))
    if adaptive and method == METHODS.euler and sde.noise_type != NOISE_TYPES.additive:
        warnings.warn("Numerical solution is not guaranteed to converge to the correct solution when using adaptive "
                      "time-stepping with the Euler--Maruyama method with non-additive noise.")
    return sde, y0, ts, bm, method, ({} if options is None else options.copy())


def parse_return(y0, ys, extra_solver_state, extra, logqp):
    """What `sdeint` hands back (reference sdeint.py:284-300): ys; with `logqp` the state's last channel is split off
    and returned as per-interval increments of the log-ratio; with `extra` the solver's final extra state is appended."""
    out = [ys]
    if logqp:
        ys, log_ratio = ys.split(split_size=(y0.size(1) - 1, 1), dim=2)
        out = [ys, (log_ratio[1:] - log_ratio[:-1]).squeeze(dim=2)]
    if extra:
        out.append(extra_solver_state)
    return out[0] if len(out) == 1 else tuple(out)
