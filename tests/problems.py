"""Synthetic SDEs used by the parity tests, the golden-vector generator and the benchmark.

Plain ``nn.Module``s carrying ``noise_type`` / ``sde_type`` (the user-SDE protocol of the reference,
torchsde/_core/sdeint.py:124-243), so the same object can be handed to the reference solver (when
generating golden vectors), wrapped for the numpy oracle, or solved by torchsde_b200 on the GPU.
Shapes and formulas follow the reference's test problems (tests/problems.py:39-132 Rackauckas-Nie
examples; :135-255 small MLPs) but the code is this repository's own.
"""
import numpy as np
import torch
from torch import nn


def _gen(seed):
    return torch.Generator().manual_seed(seed)


class GBMDiagonal(nn.Module):
    """Per-channel geometric Brownian motion, diagonal noise: f = mu*y (Ito), g = sigma*y.
    Only IEEE +,* are used, so CPU and CUDA evaluations of f/g are bit-identical."""
    noise_type = 'diagonal'

    def __init__(self, d, sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.sde_type = sde_type
        g = _gen(seed)
        sigma = torch.sigmoid(torch.randn(d, generator=g, dtype=torch.float64))
        mu = -sigma ** 2 - torch.sigmoid(torch.randn(d, generator=g, dtype=torch.float64))
        self.mu = nn.Parameter(mu.to(dtype))
        self.sigma = nn.Parameter(sigma.to(dtype))

    def f(self, t, y):
        if self.sde_type == 'ito':
            return self.mu * y
        return self.mu * y - .5 * (self.sigma ** 2) * y

    def g(self, t, y):
        return self.sigma * y


class GBMPerTrajectory(nn.Module):
    """GBM whose drift/volatility differ per trajectory (parameter sweeps, heterogeneous ensembles):
    mu, sigma are (B, d) tensors, so f and g are contiguous element-wise products — the case in which
    PyTorch uses its vectorised element-wise kernel instead of the (3x slower) broadcasting one."""
    noise_type = 'diagonal'

    def __init__(self, batch, d, sde_type='ito', seed=0, dtype=torch.float32):
        super().__init__()
        self.sde_type = sde_type
        g = _gen(seed)
        sigma = torch.sigmoid(torch.randn(batch, d, generator=g, dtype=torch.float64))
        mu = -sigma ** 2 - torch.sigmoid(torch.randn(batch, d, generator=g, dtype=torch.float64))
        self.mu = nn.Parameter(mu.to(dtype))
        self.sigma = nn.Parameter(sigma.to(dtype))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return self.sigma * y


class CosScalar(nn.Module):
    """Scalar noise (m = 1): g = (p cos^2 y)[..., None]."""
    noise_type = 'scalar'

    def __init__(self, d, sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.sde_type = sde_type
        self.p = nn.Parameter(torch.sigmoid(torch.randn(d, generator=_gen(seed), dtype=torch.float64)).to(dtype))

    def f(self, t, y):
        if self.sde_type == 'ito':
            return -self.p ** 2. * torch.sin(y) * torch.cos(y) ** 3.
        return torch.zeros_like(y)

    def g(self, t, y):
        return (self.p * torch.cos(y) ** 2).unsqueeze(dim=-1)


class TimeAdditive(nn.Module):
    """Additive noise: g(t) = a b / sqrt(1+t) broadcast to (B, d, m)."""
    noise_type = 'additive'

    def __init__(self, d, m, sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.sde_type = sde_type
        self.m = m
        g = _gen(seed)
        self.a = nn.Parameter(torch.sigmoid(torch.randn(d, m, generator=g, dtype=torch.float64)).to(dtype))
        self.b = nn.Parameter(torch.sigmoid(torch.randn(d, generator=g, dtype=torch.float64)).to(dtype))

    def f(self, t, y):
        return self.b / torch.sqrt(1. + t) - y / (2. + 2. * t)

    def g(self, t, y):
        val = self.a * (self.b / torch.sqrt(1. + t)).unsqueeze(-1)
        return val.unsqueeze(0).repeat(y.size(0), 1, 1)


class TimeAdditiveExpand(TimeAdditive):
    """Same SDE; g returns a stride-0 (batch-broadcast) view instead of a dense copy — what a user who knows that the
    diffusion does not depend on y writes.  The tile kernels read the shared (d, m) block without densifying it."""

    def g(self, t, y):
        val = self.a * (self.b / torch.sqrt(1. + t)).unsqueeze(-1)
        return val.unsqueeze(0).expand(y.size(0), -1, -1)


class TanhGeneral(nn.Module):
    """General noise: g = tanh(y)[:, :, None] * S, f = mu * y."""
    noise_type = 'general'

    def __init__(self, d, m, sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.sde_type = sde_type
        g = _gen(seed)
        self.S = nn.Parameter((0.5 * torch.rand(d, m, generator=g, dtype=torch.float64)).to(dtype))
        self.mu = nn.Parameter((-torch.rand(d, generator=g, dtype=torch.float64)).to(dtype))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return torch.tanh(y).unsqueeze(-1) * self.S


class TanhMixedGeneral(nn.Module):
    """General noise whose columns see the state at different rates: g_il = tanh(c_l y_i) S_il, f = mu * y.  Unlike
    TanhGeneral, sum_{k,l} dg_il/dy_i g_ik A_kl = sum_{k,l} c_l sech^2(c_l y_i) tanh(c_k y_i) S_il S_ik A_kl is not
    symmetric in (k, l), so the log-ODE's Levy-area term does not vanish for an antisymmetric A and changes sign with
    it: a step that takes A the wrong way round (g A^T = -g A) gives a different solution."""
    noise_type = 'general'

    def __init__(self, d, m, sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.sde_type = sde_type
        g = _gen(seed)
        self.S = nn.Parameter((0.5 * torch.rand(d, m, generator=g, dtype=torch.float64)).to(dtype))
        self.mu = nn.Parameter((-torch.rand(d, generator=g, dtype=torch.float64)).to(dtype))
        self.c = nn.Parameter((0.25 + 2.0 * torch.rand(m, generator=g, dtype=torch.float64)).to(dtype))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return torch.tanh(y.unsqueeze(-1) * self.c) * self.S


class MLPDiagonal(nn.Module):
    """Architecture of the reference's NeuralDiagonal (tests/problems.py:135-162): the fixture SDE
    of diagnostics/ito_diagonal.py.  Weights are loaded from the golden file."""
    noise_type = 'diagonal'

    def __init__(self, d, sde_type='ito'):
        super().__init__()
        self.sde_type = sde_type
        self.f_net = nn.Sequential(nn.Linear(d + 1, 8), nn.Softplus(), nn.Linear(8, d))
        self.g_net = nn.Sequential(nn.Linear(d + 1, 8), nn.Softplus(), nn.Linear(8, d), nn.Sigmoid())

    def f(self, t, y):
        ty = torch.cat([t.expand(y.size(0), 1), y], dim=1)
        return self.f_net(ty)

    def g(self, t, y):
        ty = torch.cat([t.expand(y.size(0), 1), y], dim=1)
        return 0.1 * self.g_net(ty)


class LatentLike(nn.Module):
    """Stratonovich diagonal latent-SDE-like model of BASELINE config 4 (SURVEY §8d.4):
    f = MLP(D+1 -> H -> D) softplus, g = 0.1 sigmoid(w*y + b) element-wise."""
    noise_type = 'diagonal'
    sde_type = 'stratonovich'

    def __init__(self, d, hidden=128, seed=0, dtype=torch.float32):
        super().__init__()
        torch.manual_seed(seed)
        self.f_net = nn.Sequential(nn.Linear(d + 1, hidden), nn.Softplus(), nn.Linear(hidden, d)).to(dtype)
        self.w = nn.Parameter(torch.randn(d, dtype=dtype) * 0.5)
        self.b = nn.Parameter(torch.zeros(d, dtype=dtype))

    def f_and_g(self, t, y):
        ty = torch.cat([t.expand(y.size(0), 1), y], dim=1)
        return self.f_net(ty), 0.1 * torch.sigmoid(self.w * y + self.b)


class WithProds(nn.Module):
    """View of a problem that offers a chosen subset of the user-SDE protocol (reference sdeint.py:168-243):
    `g_prod` / `f_and_g_prod` are built from the base problem's g with the reference's own product (g * v for
    diagonal noise, batched matrix-vector product otherwise; base_sde.py:98-102, misc.py:62-63)."""

    def __init__(self, base, offered):
        super().__init__()
        self.base = base
        self.noise_type, self.sde_type = base.noise_type, base.sde_type
        self.offered = tuple(offered)

    def __getattr__(self, name):
        if name in ('f', 'g', 'f_and_g', 'g_prod', 'f_and_g_prod'):
            if name in self.__dict__.get('offered', ()):
                return getattr(self, '_' + name)
            raise AttributeError(name)
        return super().__getattr__(name)

    def _f(self, t, y):
        return self.base.f(t, y)

    def _g(self, t, y):
        return self.base.g(t, y)

    def _f_and_g(self, t, y):
        return self.base.f(t, y), self.base.g(t, y)

    def _g_prod(self, t, y, v):
        g = self.base.g(t, y)
        if self.noise_type == 'diagonal':
            return g * v
        return torch.bmm(g, v.unsqueeze(-1)).squeeze(-1)

    def _f_and_g_prod(self, t, y, v):
        return self.base.f(t, y), self._g_prod(t, y, v)


class LatentPrior(nn.Module):
    """Posterior / prior pair for `logqp=True` (reference base_sde.py:240-306, examples/latent_sde.py): drift f,
    prior drift h, shared diffusion g; diagonal or general noise."""

    def __init__(self, d, m, noise_type='diagonal', sde_type='ito', seed=0, dtype=torch.float64):
        super().__init__()
        self.noise_type, self.sde_type = noise_type, sde_type
        g = _gen(seed)
        self.a = nn.Parameter((0.5 * torch.rand(d, generator=g, dtype=torch.float64)).to(dtype))
        self.c = nn.Parameter((0.3 * torch.rand(d, generator=g, dtype=torch.float64)).to(dtype))
        self.s = nn.Parameter((0.2 + 0.3 * torch.rand(d, generator=g, dtype=torch.float64)).to(dtype))
        self.S = nn.Parameter((0.2 + 0.5 * torch.rand(d, m, generator=g, dtype=torch.float64)).to(dtype))

    def f(self, t, y):
        return self.c - self.a * y + 0.1 * torch.sin(y)

    def h(self, t, y):
        return -0.5 * y

    def g(self, t, y):
        if self.noise_type == 'diagonal':
            return self.s * (1.0 + 0.2 * torch.cos(y))
        return (1.0 + 0.2 * torch.cos(y)).unsqueeze(-1) * self.S


PROBLEMS = {'gbm': GBMDiagonal, 'scalar': CosScalar, 'additive': TimeAdditive, 'general': TanhGeneral,
            'additive_expand': TimeAdditiveExpand, 'general_mixed': TanhMixedGeneral}


def make(kind, d, m, sde_type, dtype=torch.float64, seed=0):
    if kind in ('gbm', 'scalar'):
        return PROBLEMS[kind](d, sde_type=sde_type, seed=seed, dtype=dtype)
    return PROBLEMS[kind](d, m, sde_type=sde_type, seed=seed, dtype=dtype)


# ---- adapters --------------------------------------------------------------------------------
class NumpySDE:
    """Wraps a torch CPU module for the numpy oracle (oracle/solvers.py): numpy in, numpy out.
    `gdg` is the Milstein vjp  vjp_y(g; g * v2)  (base_sde.py:127-155) via torch autograd on CPU."""

    def __init__(self, module):
        self.module = module
        self.noise_type = module.noise_type
        self.sde_type = module.sde_type

    def _t(self, t, y):
        yt = torch.from_numpy(np.ascontiguousarray(y))
        return torch.tensor(float(t), dtype=torch.from_numpy(np.asarray(t)).dtype), yt

    def f(self, t, y):
        tt, yt = self._t(t, y)
        with torch.no_grad():
            if hasattr(self.module, 'f'):
                return self.module.f(tt, yt).numpy().copy()
            return self.module.f_and_g(tt, yt)[0].numpy().copy()

    def g(self, t, y):
        tt, yt = self._t(t, y)
        with torch.no_grad():
            if hasattr(self.module, 'g'):
                return self.module.g(tt, yt).numpy().copy()
            return self.module.f_and_g(tt, yt)[1].numpy().copy()

    def gdg(self, t, y, v2):
        tt, yt = self._t(t, y)
        with torch.enable_grad():
            yt = yt.requires_grad_(True)
            g = self.module.g(tt, yt)
            v = torch.from_numpy(np.ascontiguousarray(v2))
            go = g * (v.unsqueeze(-2) if g.dim() == 3 else v)
            out, = torch.autograd.grad(g, yt, go.detach(), allow_unused=True)
        return (torch.zeros_like(yt) if out is None else out).detach().numpy().copy()

    def vjp_fg(self, t, z, adj_f, adj_g):
        """vjp of (f, g) wrt z and the parameters (reversible_heun.py:119-129)."""
        tt, zt = self._t(t, z)
        with torch.enable_grad():
            return self._vjp_fg(tt, zt, adj_f, adj_g)

    def _vjp_fg(self, tt, zt, adj_f, adj_g):
        zt = zt.requires_grad_(True)
        if hasattr(self.module, 'f_and_g'):
            f, g = self.module.f_and_g(tt, zt)
        else:
            f, g = self.module.f(tt, zt), self.module.g(tt, zt)
        params = [p for p in self.module.parameters() if p.requires_grad]
        pairs = [(o, torch.from_numpy(np.ascontiguousarray(a))) for o, a in ((f, adj_f), (g, adj_g))
                 if o.requires_grad]
        if pairs:
            outs = torch.autograd.grad([o for o, _ in pairs], [zt] + params, [a for _, a in pairs],
                                       allow_unused=True)
        else:
            outs = [None] * (1 + len(params))
        outs = [torch.zeros_like(x) if o is None else o for o, x in zip(outs, [zt] + params)]
        return outs[0].numpy().copy(), [o.numpy().copy() for o in outs[1:]]


class ReplayBM:
    """Duck-typed Brownian motion serving recorded increments keyed by (ta, tb) — the
    'same-increment replay' parity device of SURVEY.md fact 3 (the reference solver accepts any
    object with .shape, .levy_area_approximation and __call__, base_solver.py:54-57)."""

    def __init__(self, tas, tbs, Ws, Us=None, levy='none', to_torch=None, As=None):
        self.table = {}
        self.areas = {}
        for i, (a, b) in enumerate(zip(tas, tbs)):
            self.table[(float(a), float(b))] = (Ws[i], None if Us is None else Us[i])
            if As is not None:
                self.areas[(float(a), float(b))] = As[i]
        self.shape = tuple(Ws[0].shape)
        self.levy_area_approximation = levy
        self.to_torch = to_torch
        self.dtype = None
        self.device = None

    def __call__(self, ta, tb=None, return_U=False, return_A=False):
        key = (float(ta), float(tb))
        if key not in self.table:  # e.g. an fp32 time grid replaying increments recorded on an fp64 grid
            near = min(self.table, key=lambda k: abs(k[0] - key[0]) + abs(k[1] - key[1]))
            if abs(near[0] - key[0]) + abs(near[1] - key[1]) > 1e-5:
                raise KeyError(key)
            key = near
        W, U = self.table[key]
        if self.to_torch is not None:
            W = self.to_torch(W)
            U = None if U is None else self.to_torch(U)
        if return_A:
            A = self.areas[key]
            if self.to_torch is not None:
                A = self.to_torch(A)
            return (W, U, A) if return_U else (W, A)
        return (W, U) if return_U else W
