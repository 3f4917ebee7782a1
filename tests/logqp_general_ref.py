"""Shared by the general-noise logqp tests and their golden fixtures: a float64 restatement of the KL rate that
`tsde_logqp_augment` computes for general / additive / scalar noise, the error bound its GPU test holds the kernel
to, and the latent-SDE problems the fixtures were recorded on.

The rate is the reference's (torchsde base_sde.py:285-306):  u = pinverse(g) (f - h),  rate = 0.5 |u|^2,  with
pinverse's rule that a singular value s is kept only if s > rcond * s_max (rcond = 1e-15).  A row whose g or f - h
is not finite gets NaN, as the kernel gives it.
"""
import numpy as np
import torch
from torch import nn

RCOND = 1e-15
UNIT = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53, torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
# err <= C_BOUND (n + k) u kappa_2(g) scale, per row (see `bound`); calibrated on the H100 test cases, where the
# worst err / bound is reported by tests/test_gpu_logqp_general.py
C_BOUND = 16.0


def finite_rows(f, g, h):
    r = np.asarray(f, np.float64) - np.asarray(h, np.float64)
    return np.isfinite(np.asarray(g, np.float64)).all(axis=(1, 2)) & np.isfinite(r).all(axis=1)


def kl_rate(f, g, h, rcond=RCOND, variant=None):
    """0.5 |pinv(g) (f - h)|^2 per row, float64.  `variant` names a deliberate mistake (for the tests showing that
    the bound rejects it): 'sigma' (s for s^2), 'no_cutoff', 'plus' (f + h), 'neighbour' (row i given row i-1's g),
    'swapped' (the wide formula on a tall matrix: r projected on V instead of U; square rows only)."""
    f, g, h = (np.asarray(x, np.float64) for x in (f, g, h))
    ok = finite_rows(f, g, h)
    r = f + h if variant == 'plus' else f - h
    g = np.where(ok[:, None, None], g, 0.0)
    r = np.where(ok[:, None], r, 0.0)
    if variant == 'neighbour':
        g = np.roll(g, 1, axis=0)
    U, S, Vt = np.linalg.svd(g, full_matrices=False)
    smax = S.max(axis=1, keepdims=True) if S.shape[1] else np.zeros((len(S), 1))
    keep = np.ones_like(S, bool) if variant == 'no_cutoff' else S > rcond * smax
    if variant == 'swapped':
        proj = np.einsum('bij,bj->bi', Vt, r)                          # V^T r (d == m)
    else:
        proj = np.einsum('bji,bj->bi', U, r)                           # U^T r
    with np.errstate(divide='ignore', invalid='ignore'):
        # |u|^2 = sum_i (U_i . r)^2 / s_i^2 over the kept s_i ('sigma': one power of s short)
        terms = proj ** 2 / (S if variant == 'sigma' else S ** 2)
        rate = 0.5 * np.where(keep, terms, 0.0).sum(axis=1)
    return np.where(ok, rate, np.nan)


def bound(f, g, h, dtype, c=C_BOUND):
    """Per-row error bound c (n + k) u kappa_2(g) scale, scale = 0.5 |f - h|^2 / s_min^2 (an upper bound of the rate),
    with kappa_2 and s_min over the singular values pinverse keeps; 0 for a row whose g is zero."""
    f, g, h = (np.asarray(x, np.float64) for x in (f, g, h))
    d, m = g.shape[1], g.shape[2]
    ok = finite_rows(f, g, h)
    g = np.where(ok[:, None, None], g, 0.0)
    r = np.where(ok[:, None], f - h, 0.0)
    S = np.linalg.svd(g, compute_uv=False)
    smax = S.max(axis=1)
    kept = S > RCOND * smax[:, None]
    smin = np.where(kept, S, np.inf).min(axis=1)
    with np.errstate(divide='ignore', invalid='ignore'):
        kappa = np.where(np.isfinite(smin), smax / smin, 0.0)
        scale = np.where(np.isfinite(smin), 0.5 * (r ** 2).sum(axis=1) / smin ** 2, 0.0)
    return c * (d + m) * UNIT[dtype] * kappa * scale


def conditioned(rng, B, d, m, kappa):
    """(B, d, m) float64 matrices with singular values log-spaced from 1 down to 1/kappa."""
    n = min(d, m)
    U = np.linalg.qr(rng.standard_normal((B, d, n)))[0]
    V = np.linalg.qr(rng.standard_normal((B, m, n)))[0]
    s = np.logspace(0.0, -np.log10(kappa), n)
    return np.einsum('bin,n,bjn->bij', U, s, V)


class LatentGeneral(nn.Module):
    """Posterior / prior pair for `logqp=True` with general, additive or scalar noise (reference base_sde.py:240-306):
    drift f, prior drift h, shared diffusion g.  `zero_col` / `zero_row` make that column / row of every row's g
    structurally zero (pinverse then drops a singular value, or the state channel carries no noise)."""

    def __init__(self, d, m, noise_type='general', sde_type='ito', seed=0, dtype=torch.float64, zero_col=None,
                 zero_row=None):
        super().__init__()
        self.noise_type, self.sde_type = noise_type, sde_type
        gen = torch.Generator().manual_seed(1000 + seed)
        self.a = nn.Parameter((0.5 * torch.rand(d, generator=gen, dtype=torch.float64)).to(dtype))
        self.c = nn.Parameter((0.3 * torch.rand(d, generator=gen, dtype=torch.float64)).to(dtype))
        self.S = nn.Parameter((0.2 + 0.5 * torch.rand(d, m, generator=gen, dtype=torch.float64)).to(dtype))
        mask = torch.ones(d, m, dtype=dtype)
        if zero_col is not None:
            mask[:, zero_col] = 0
        if zero_row is not None:
            mask[zero_row, :] = 0
        self.register_buffer('mask', mask)

    def f(self, t, y):
        return self.c - self.a * y + 0.1 * torch.sin(y)

    def h(self, t, y):
        return -0.5 * y

    def g(self, t, y):
        S = self.S * self.mask
        if self.noise_type == 'additive':
            return S.expand(y.size(0), *S.shape)
        return (1.0 + 0.2 * torch.cos(y)).unsqueeze(-1) * S


# name -> (d, m, noise_type, sde_type, method, adjoint, zero_col, zero_row); recorded by make_golden_logqp_general.py
GOLDEN_CASES = {
    'wide_ito_euler': (3, 5, 'general', 'ito', 'euler', False, None, None),
    'square_strat_heun': (4, 4, 'general', 'stratonovich', 'heun', False, None, None),
    'scalar_ito_euler': (4, 1, 'scalar', 'ito', 'euler', False, None, None),
    'additive_ito_srk': (4, 3, 'additive', 'ito', 'srk', False, None, None),
    'zerocol_strat_midpoint': (4, 3, 'general', 'stratonovich', 'midpoint', False, 1, None),
    'zerorow_ito_euler': (4, 3, 'general', 'ito', 'euler', False, None, 2),
    'wide_strat_reversible_heun_adjoint': (3, 5, 'general', 'stratonovich', 'reversible_heun', True, None, None),
    'scalar_strat_reversible_heun_adjoint': (4, 1, 'scalar', 'stratonovich', 'reversible_heun', True, None, None),
}
