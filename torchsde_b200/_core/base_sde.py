"""SDE base classes and the one-time function table the solver calls up into.

API mirror of the reference's ``torchsde/_core/base_sde.py``: ``BaseSDE`` (:25-39),
``ForwardSDE`` (:42-73), ``RenameMethodsSDE`` (:212-224), ``SDEIto`` / ``SDEStratonovich``
(:227-236), ``SDELogqp`` (:240-306).

Difference to the reference: ``ForwardSDE`` does not implement ``prod`` / ``g_prod_default`` /
``f_and_g_prod_default*`` with ATen ops.  Those products (``g*v``, ``bmm(g, v)``;
base_sde.py:98-120) are fused into the CUDA tableau kernels; the table only records *which* of
the user's callables exist so that the solver reproduces the reference's call pattern
(base_sde.py:51-61): a user-supplied ``f_and_g_prod`` / ``g_prod`` is honoured (the increment is
then materialised for it), otherwise ``f_and_g`` / ``f``,``g`` are evaluated and the product
happens inside the kernel.
"""
import abc

import torch
from torch import nn

from ..settings import NOISE_TYPES, SDE_TYPES


_HALF = (torch.bfloat16, torch.float16)


def widen(x, dtype):
    """A bfloat16 / float16 tensor (an SDE output computed under torch.autocast) converted to `dtype`, exactly; anything
    else as it is.  The package's own torch code computes only on widened outputs: ATen's promotion rules would round
    intermediates such as `f * dt` to 16 bits otherwise."""
    return x.to(dtype) if torch.is_tensor(x) and x.dtype in _HALF else x


def _widened(fn, dtype):
    def call(*args):
        out = fn(*args)
        return tuple(widen(o, dtype) for o in out) if isinstance(out, tuple) else widen(out, dtype)
    return call


class BaseSDE(abc.ABC, nn.Module):
    """Base class for all SDEs; validates `noise_type` and `sde_type` (base_sde.py:25-39)."""

    def __init__(self, noise_type, sde_type):
        super(BaseSDE, self).__init__()
        if noise_type not in NOISE_TYPES:
            raise ValueError(f"Expected noise type in {NOISE_TYPES}, but found {noise_type}")
        if sde_type not in SDE_TYPES:
            raise ValueError(f"Expected sde type in {SDE_TYPES}, but found {sde_type}")
        self.noise_type = noise_type
        self.sde_type = sde_type


class ForwardSDE(BaseSDE):

    def __init__(self, sde):
        super(ForwardSDE, self).__init__(sde_type=sde.sde_type, noise_type=sde.noise_type)
        self._base_sde = sde
        # Which specialised callables did the user provide? (base_sde.py:51-61)
        self.user_f_and_g_prod = hasattr(sde, 'f_and_g_prod')
        self.user_g_prod = hasattr(sde, 'g_prod')
        self.user_f_and_g = hasattr(sde, 'f_and_g')
        self.f = getattr(sde, 'f', self.f_default)
        self.g = getattr(sde, 'g', self.g_default)
        self.f_and_g = getattr(sde, 'f_and_g', self.f_and_g_default)
        if self.user_g_prod:
            self.g_prod = sde.g_prod
        if self.user_f_and_g_prod:
            self.f_and_g_prod = sde.f_and_g_prod
        self.widened_to = None

    def widen_outputs(self, dtype):
        """From now on hand out every bfloat16 / float16 output of the user's callables widened to `dtype` (exact).
        Used where the solve is not a chain of this library's launches: gradients through `sdeint` (each output is
        widened once, so autograd accumulates its gradient in `dtype` before rounding it to 16 bits), the backward
        SDE of the generic adjoints, and float64 states.  Idempotent."""
        if self.widened_to is not None:
            return
        self.widened_to = dtype
        for name in ('f', 'g', 'f_and_g', 'g_prod', 'f_and_g_prod'):
            if name in vars(self):
                setattr(self, name, _widened(getattr(self, name), dtype))

    def f_default(self, t, y):
        raise RuntimeError("Method `f` has not been provided, but is required for this method.")

    def g_default(self, t, y):
        raise RuntimeError("Method `g` has not been provided, but is required for this method.")

    def f_and_g_default(self, t, y):
        return self.f(t, y), self.g(t, y)

    # How the solver obtains (f, g.v) for a `f_and_g_prod`-style call site (base_sde.py:51-56):
    #   'f_and_g_prod' : user's f_and_g_prod(t, y, v)
    #   'g_prod'       : user's f(t, y) and g_prod(t, y, v)          (f_and_g_prod_default1 :115-116)
    #   'fused'        : f_and_g(t, y), product inside the kernel    (f_and_g_prod_default2 :118-120)
    @property
    def f_and_g_prod_mode(self):
        if self.user_f_and_g_prod:
            return 'f_and_g_prod'
        if hasattr(self._base_sde, 'f') and self.user_g_prod:
            return 'g_prod'
        return 'fused'

    # How the solver obtains g.v for a `g_prod` call site (base_sde.py:54, :108-109).
    @property
    def g_prod_mode(self):
        return 'g_prod' if self.user_g_prod else 'fused'


class RenameMethodsSDE(BaseSDE):
    """View of a user SDE whose callables live under other attribute names (`names=` of sdeint; reference
    base_sde.py:212-224).  Only the names that resolve are bound, a missing one surfaces later as the usual
    "method has not been provided" error."""
    _STANDARD = ('f', 'g', 'h', 'g_prod', 'f_and_g', 'f_and_g_prod')

    def __init__(self, sde, drift='f', diffusion='g', prior_drift='h', diffusion_prod='g_prod',
                 drift_and_diffusion='f_and_g', drift_and_diffusion_prod='f_and_g_prod'):
        BaseSDE.__init__(self, noise_type=sde.noise_type, sde_type=sde.sde_type)
        self._base_sde = sde
        theirs = (drift, diffusion, prior_drift, diffusion_prod, drift_and_diffusion, drift_and_diffusion_prod)
        self._plan_tag = ('rename',) + theirs  # part of the CUDA-graph plan key (graph.cache_owner)
        for ours, attr in zip(self._STANDARD, theirs):
            bound = getattr(sde, attr, None)
            if bound is not None:
                setattr(self, ours, bound)


class SDEIto(BaseSDE):
    """Convenience base class fixing sde_type='ito' (base_sde.py:227-230)."""

    def __init__(self, noise_type):
        BaseSDE.__init__(self, noise_type=noise_type, sde_type=SDE_TYPES.ito)


class SDEStratonovich(BaseSDE):
    """Convenience base class fixing sde_type='stratonovich' (base_sde.py:233-236)."""

    def __init__(self, noise_type):
        BaseSDE.__init__(self, noise_type=noise_type, sde_type=SDE_TYPES.stratonovich)


def _kl_rate(f, g, h, diagonal, epsilon=1e-7):
    """0.5 |u|^2 with g u = f - h: the integrand of the KL divergence between the posterior SDE (drift f) and the
    prior SDE (drift h) that share the diffusion g.  Diagonal noise divides element-wise, guarding |g| < epsilon the way
    the reference's `stable_division` does (misc.py:66-68); otherwise u is the least-squares solution through the
    pseudo-inverse of g (base_sde.py:266-306)."""
    gap = f - h
    if diagonal:
        safe = torch.where(g.abs().detach() > epsilon, g, torch.full_like(g, fill_value=epsilon) * g.sign())
        u = gap / safe
    else:
        u = torch.bmm(g.pinverse(), gap.unsqueeze(-1)).squeeze(-1)
    return .5 * (u ** 2).sum(dim=1, keepdim=True)


class SDELogqp(BaseSDE):
    """State augmented by one channel that integrates the KL rate (`logqp=True`; base_sde.py:240-306): drift
    (f, 0.5|u|^2), diffusion (g, 0).  User-level model code made of the user's own f / g / h (torch ops), solved by the
    same engine as any other SDE."""

    def __init__(self, sde):
        BaseSDE.__init__(self, noise_type=sde.noise_type, sde_type=sde.sde_type)
        self._base_sde = sde
        self._plan_tag = 'logqp'
        missing = [name for name in ('f', 'g', 'h') if not hasattr(sde, name)]
        if missing:
            raise AttributeError("If using logqp then drift, diffusion and prior drift must all be specified.")
        self._diagonal = sde.noise_type == NOISE_TYPES.diagonal

    def _pad_diffusion(self, g):
        # the extra channel carries no noise: a zero entry (diagonal) or a zero row of the (d, m) matrix
        zeros = g.new_zeros((g.size(0), 1) if self._diagonal else (g.size(0), 1, g.size(-1)))
        return torch.cat([g, zeros], dim=1)

    def f_and_g(self, t, y):
        state = y[:, :-1]
        base = self._base_sde
        f, g, h = (widen(x, y.dtype) for x in (base.f(t, state), base.g(t, state), base.h(t, state)))
        differentiated = torch.is_grad_enabled() and (f.requires_grad or g.requires_grad or h.requires_grad)
        if not differentiated and self._on_device(f):
            if self._diagonal:
                return self._fused_augment(f, g, h)
            from .. import _cabi
            if _cabi.logqp_general_fits(g.size(1), g.size(2)):
                return self._fused_augment_general(f, g, h)
        rate = _kl_rate(f, g, h, self._diagonal)
        return torch.cat([f, rate], dim=1), self._pad_diffusion(g)

    @staticmethod
    def _on_device(t):
        from .. import _cabi
        try:
            _cabi.require_cuda(t)
            return True
        except RuntimeError:
            return False

    @staticmethod
    def _fused_augment(f, g, h, epsilon=1e-7):
        """One kernel instead of ~10 ATen launches when nothing has to be differentiated (inference solves and the
        no-grad forward pass of `sdeint_adjoint`; the vjp's of the backward pass go through the torch ops above)."""
        import ctypes
        from .. import _cabi
        f, g, h = (x if x.is_contiguous() else x.contiguous() for x in (f, g, h))
        rows, d = f.shape
        f_aug = torch.empty((rows, d + 1), dtype=f.dtype, device=f.device)
        g_aug = torch.empty_like(f_aug)
        L = _cabi.make_launch(f.dtype, _cabi.NOISE_DIAGONAL, rows, d, d, device=f.device)
        _cabi.check(_cabi.lib().tsde_logqp_augment(ctypes.byref(L), f.data_ptr(), g.data_ptr(), h.data_ptr(), epsilon,
                                                   f_aug.data_ptr(), g_aug.data_ptr()), "tsde_logqp_augment")
        return f_aug, g_aug

    @staticmethod
    def _fused_augment_general(f, g, h, rcond=1e-15):
        """General, additive and scalar noise: |pinverse(g) (f - h)|^2 by a per-row Jacobi SVD in one kernel instead of
        a batched SVD that synchronises the host, so such solves can be captured into a CUDA graph.  An `expand`ed g
        (additive noise) is materialised first, as the torch path's `cat` does."""
        import ctypes
        from .. import _cabi
        f, g, h = (x if x.is_contiguous() else x.contiguous() for x in (f, g, h))
        rows, d, m = g.shape
        f_aug = torch.empty((rows, d + 1), dtype=f.dtype, device=f.device)
        g_aug = torch.empty((rows, d + 1, m), dtype=g.dtype, device=g.device)
        L = _cabi.make_launch(f.dtype, _cabi.NOISE_GENERAL, rows, d, m, device=f.device)
        _cabi.check(_cabi.lib().tsde_logqp_augment(ctypes.byref(L), f.data_ptr(), g.data_ptr(), h.data_ptr(), rcond,
                                                   f_aug.data_ptr(), g_aug.data_ptr()), "tsde_logqp_augment")
        return f_aug, g_aug

    def f(self, t, y):
        return self.f_and_g(t, y)[0]

    def g(self, t, y):
        return self._pad_diffusion(widen(self._base_sde.g(t, y[:, :-1]), y.dtype))
