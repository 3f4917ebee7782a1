"""Restatements of what `tsde_bmm_ga` (the log-ODE product g.A) and the diagonal-noise `tsde_logqp_augment` compute,
the route and error bound their GPU tests (tests/test_gpu_logode_paths.py) hold the kernels to, and one log-ODE
midpoint step in torch float64.  CPU tests (tests/test_host_logode_paths.py) pin them to the package's torch formulas
and show the bounds reject plausible slips."""
import math

import numpy as np
import torch

# ---- tsde_bmm_ga: out[l, r, dd] = sum_k g[r, dd, k] A[r, k, l] ---------------------------------------------------
TILE_M = (2, 3, 4, 8, 16, 32)
TILE_MAX_D = 1 << 20
TILE_THREADS = 256
TILE_SMEM = 32 * 1024


def bmm_route(m, d, itemsize, g_aligned=True, a_aligned=True):
    """('tile', rows per CTA) or ('generic', None), as bmm_ga_impl (csrc/logode.cu) chooses: the tile kernel
    bmm_ga_kernel<T, M> for d <= 2^20 and m in TILE_M when g and A are 16-byte aligned or m % 4 != 0 (its 128-bit
    loads are only issued for m % 4 == 0); min(ceil(256 / d), floor(32 KiB / (m^2 sizeof T))) rows per CTA."""
    if d <= TILE_MAX_D and m in TILE_M and ((g_aligned and a_aligned) or m % 4 != 0):
        return 'tile', max(1, min(-(-TILE_THREADS // d), TILE_SMEM // (m * m * itemsize)))
    return 'generic', None


def bmm_kernel_name(route, dtype_name):
    """The substring torch.profiler shows for the kernel of `route`."""
    return ('bmm_ga_kernel<' if route == 'tile' else 'bmm_ga_generic_kernel<') + dtype_name


def bmm_exact(g, a):
    """The product in extended precision (float64 for float32 operands, whose products are then exact; long double
    otherwise), transposed to the kernel's (m, rows, d)."""
    wide = np.float64 if g.dtype == np.float32 else np.longdouble
    out = np.matmul(g.astype(wide), a.astype(wide))
    return np.ascontiguousarray(out.transpose(2, 0, 1))


def bmm_bound(g, a):
    """gamma_m sum_k |g_k||A_kl| + m eta per element, (m, rows, d): an m-term fma chain from 0 rounds m times
    (gamma_m = m u / (1 - m u)), and each rounding may also be one of the underflow unit eta."""
    fi = np.finfo(g.dtype)
    m = g.shape[-1]
    u = float(fi.eps) / 2
    gamma = m * u / (1 - m * u)
    mag = np.matmul(np.abs(g).astype(np.float64), np.abs(a).astype(np.float64))
    return np.ascontiguousarray(mag.transpose(2, 0, 1)) * gamma + m * float(fi.smallest_subnormal)


def bmm_operands(rng, rows, d, m, npdt, antisymmetric):
    """g with entries scaled by 2^-20, 1 or 2^20 at random (large terms swamp small ones and random signs cancel),
    and A general or antisymmetric (the Levy area), its rows scaled the same way."""
    scale = np.exp2(rng.choice([-20.0, 0.0, 20.0], size=(rows, d, m)))
    g = (rng.standard_normal((rows, d, m)) * scale).astype(npdt)
    a = rng.standard_normal((rows, m, m))
    if antisymmetric:
        a = a - a.transpose(0, 2, 1)
    a = (a * np.exp2(rng.choice([-20.0, 0.0, 20.0], size=(rows, m, 1)))).astype(npdt)
    return g, a


def bmm_error(got, g, a):
    """|got - exact| per element, (m, rows, d), subtracted in the exact product's precision (the difference of a
    result and the exact value is then exact or nearly so, not rounded to a whole ulp of the result)."""
    exact = bmm_exact(g, a)
    return np.abs(got.astype(exact.dtype) - exact).astype(np.float64)


def bmm_violations(got, g, a):
    """Elements of `got` (m, rows, d) outside the bound (NaN counts as outside)."""
    return ~(bmm_error(got, g, a) <= bmm_bound(g, a))


# ---- tsde_logqp_augment, diagonal noise --------------------------------------------------------------------------
LOGQP_EPS = 1e-7   # SDELogqp._fused_augment's epsilon


def logqp_rate_emulated(f, g, h, eps=LOGQP_EPS, mistake=None):
    """logqp_augment_kernel's f_aug[:, d] bit for bit, in the operands' dtype T and the kernel's order: eps rounded to T,
    safe = g where |g| > eps else eps * sign(g) (sign(+-0) = sign(NaN) = 0), u = (f - h) / safe, lane c % 32
    accumulates acc + u * u over c ascending, then the xor butterfly 16, 8, 4, 2, 1 read at lane 0, times 0.5.
    (The library is built with -fmad=false and IEEE division, without flush-to-zero.)
    `mistake` computes one of the wrong formulas the CPU tests show the checks reject."""
    T = f.dtype.type
    e = T(eps)
    sgn = np.where(g > 0, T(1), np.where(g < 0, T(-1), T(0 if mistake != 'sign(0) = 1' else 1))).astype(f.dtype)
    guard = np.abs(g) >= e if mistake == '>=' else np.abs(g) > e
    safe = np.where(guard, g, e * sgn)
    with np.errstate(all='ignore'):
        if mistake == 'eps unrounded':
            u = ((f - h).astype(np.float64) / np.where(guard, g.astype(np.float64), eps * sgn.astype(np.float64)))
            u = u.astype(f.dtype)
        else:
            u = ((f + h) if mistake == 'f + h' else (f - h)) / safe
        sq = u * u
        rows, d = f.shape
        pad = np.zeros((rows, -(-d // 32) * 32), f.dtype)   # +0 terms: acc + 0 == acc (acc is never -0)
        pad[:, :d] = sq
        acc = np.zeros((rows, 32), f.dtype)
        for j in range(0, pad.shape[1], 32):
            acc = acc + pad[:, j:j + 32]
        for off in (16, 8, 4, 2, 1):
            acc = acc + acc[:, np.arange(32) ^ off]
        return acc[:, 0] if mistake == 'no 0.5' else T(0.5) * acc[:, 0]


def logqp_rate_exact(f, g, h, eps=LOGQP_EPS):
    """The same rate in float64 from the T-rounded eps guard (the guard itself is a comparison, exact in T)."""
    T = f.dtype.type
    e = float(T(eps))
    f64, g64, h64 = (x.astype(np.float64) for x in (f, g, h))
    safe = np.where(np.abs(g64) > e, g64, e * np.where(g64 > 0, 1.0, np.where(g64 < 0, -1.0, 0.0)))
    with np.errstate(all='ignore'):
        u = (f64 - h64) / safe
        return 0.5 * np.sum(u * u, axis=1)


def logqp_bound(rate64, d, npdt):
    """(ceil(d/32) + 5 + 3) u sum u^2 (+ d eta for squares that underflow): the lane chains, five butterfly levels,
    and the quotient's rounding (twice, once squared) and the square's."""
    fi = np.finfo(npdt)
    return (math.ceil(d / 32) + 5 + 3) * (float(fi.eps) / 2) * 2 * np.abs(rate64) + d * float(fi.smallest_subnormal)


def logqp_violations(got, f, g, h):
    """Rows whose rate is not the emulation's bits (NaN where it is NaN), or is outside the float64 bound."""
    emu = logqp_rate_emulated(f, g, h)
    nan = np.isnan(emu)
    bits_ok = np.where(nan, np.isnan(got), got.view(_uint(got)) == emu.view(_uint(emu)))
    ref = logqp_rate_exact(f, g, h)
    # (a sum of squares past T's range overflows to inf on the way, as it should)
    ref = np.where(2 * np.abs(ref) > float(np.finfo(f.dtype).max), np.inf, ref)
    with np.errstate(invalid='ignore'):
        in_bound = np.where(np.isfinite(ref), np.abs(got.astype(np.float64) - ref) <= logqp_bound(ref, f.shape[1],
                                                                                                  f.dtype),
                            (got.astype(np.float64) == ref) | (np.isnan(ref) & np.isnan(got)))
    return ~bits_ok, ~in_bound


def _uint(x):
    return np.uint32 if x.dtype == np.float32 else np.uint64


# ---- log-ODE solves ------------------------------------------------------------------------------------------------
LOG_ODE_B, LOG_ODE_D = 9, 40     # more rows than one tile CTA holds (7, or 4 at m = 32 in fp64), not a multiple
LOG_ODE_TS, LOG_ODE_DT = (0.0, 0.125, 0.25), 0.0625


def log_ode_route_case(m, dtype):
    """The general-noise log-ODE solve of the route tests on the CPU: (sde, y0, step starts, Ws, As), a
    TanhMixedGeneral problem (its Levy-area term changes sign with A) and seeded increments and antisymmetric areas."""
    from . import problems
    sde = problems.make('general_mixed', LOG_ODE_D, m, 'stratonovich', dtype=dtype, seed=m)
    rng = np.random.default_rng(m)
    y0 = torch.from_numpy(0.1 + 0.5 * rng.random((LOG_ODE_B, LOG_ODE_D))).to(dtype)
    tas = np.arange(LOG_ODE_TS[0], LOG_ODE_TS[-1], LOG_ODE_DT)
    Ws, As = [], []
    for _ in tas:
        Ws.append(torch.from_numpy(rng.standard_normal((LOG_ODE_B, m)) * math.sqrt(LOG_ODE_DT)).to(dtype))
        a = rng.standard_normal((LOG_ODE_B, m, m)) * (LOG_ODE_DT / math.sqrt(12))
        As.append(torch.from_numpy(a - a.transpose(0, 2, 1)).to(dtype))
    return sde, y0, tas, Ws, As


# ---- one log-ODE midpoint step (methods/log_ode.py:39-56, base_sde.py:165-185), torch float64 on the CPU ----------
def log_ode_step(sde, t0, dt, y0, W, A):
    """y' = y0 + dt/2 f + 1/2 g W;  y1 = y0 + dt f(y') + g(y') W + sum_l d g[:, :, l] / dy . (g(y') A)[:, :, l]."""
    t0 = torch.as_tensor(t0, dtype=y0.dtype)
    with torch.no_grad():
        yp = y0 + 0.5 * dt * sde.f(t0, y0) + 0.5 * torch.einsum('bdm,bm->bd', sde.g(t0, y0), W)
    tm = t0 + 0.5 * dt
    y = yp.detach().requires_grad_(True)
    with torch.enable_grad():
        g = sde.g(tm, y)
        ga = torch.matmul(g, A)
        corr = torch.zeros_like(yp)
        for col in range(g.shape[-1]):
            corr = corr + torch.func.jvp(lambda z, c=col: sde.g(tm, z)[..., c], (yp,), (ga[..., col].detach(),))[1]
    with torch.no_grad():
        return y0 + dt * sde.f(tm, yp) + torch.einsum('bdm,bm->bd', g.detach(), W) + corr
