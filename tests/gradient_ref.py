"""Finite-difference oracle for the gradients of a solve.

Once the Brownian path is fixed, a fixed-step solve is a smooth, deterministic function of y0, of the SDE's parameters
and of any tensor f / g close over: every forward solve here builds a fresh `BrownianInterval` with the same entropy,
so the perturbed solves see bit-identical increments and differ only through the perturbed input.  The forward solve
is verified against the oracle elsewhere in the suite, so a gradient that disagrees with the central difference of the
forward solve is wrong, whichever path (tableau transpose table, materialised counter noise, adjoint engine) produced
it.  Nothing here reads golden files or the reference.

Error bound of a central difference D = (l(x + h) - l(x - h)) / 2h in float64, h = H_REL * max(|x|, 1):
  * truncation  h^2 |l'''| / 6, about 1.5e-13 |l'''| at H_REL = 2^-20;
  * roundoff    n u L / h: each solve's result carries at most n u L of rounding (L = sum |w . ys| the loss's scale,
    n < 100 rounded operations per element along these short solves, u = 2^-53), so u / h = 2^-33 ~ 1.2e-10 and
    the term is below 1.2e-8 L.
Both together stay below RTOL * (L + |D|) with RTOL = 1e-7 (the derivatives of these smooth problems are O(L)), which
is what every comparison below asserts.  A wrong coefficient of relative size 1e-5 in a term that carries a few per cent
of the gradient moves it by ~1e-7 L and beyond: tests/test_gpu_gradients.py (f) shows that such an error fails.
"""
import contextlib

import torch

H_REL = 2.0 ** -20
U64 = 2.0 ** -53
N_OPS = 100                       # rounded operations per element along a solve (bound)
RTOL = 1e-7                       # >= N_OPS * U64 / H_REL (1.2e-8) + the truncation term, with margin


@contextlib.contextmanager
def shifted(tensors, deltas):
    """The tensors shifted in place by deltas (None: unchanged) for the duration of the block."""
    with torch.no_grad():
        saved = [t.detach().clone() for t in tensors]
        for t, dx in zip(tensors, deltas):
            if dx is not None:
                t.add_(dx)
    try:
        yield
    finally:
        with torch.no_grad():
            for t, s in zip(tensors, saved):
                t.copy_(s)


def _eval(fn):
    with torch.no_grad():
        return fn().detach().double()


def central_jacobian(fn, inputs, h=H_REL):
    """Full float64 Jacobian of fn() (a tensor) with respect to each tensor of `inputs`, by central differences: one
    element at a time, two forward solves each, step h * max(|x_e|, 1).  `fn` reads the inputs (y0, parameters, closed-
    over tensors), which are shifted in place and restored.  Returns (out, [J_i]) with J_i of shape
    (out.numel(), inputs[i].numel())."""
    out = _eval(fn)
    jacs = []
    for i, x in enumerate(inputs):
        steps = h * torch.clamp(x.detach().abs(), min=1.0)
        J = torch.empty(out.numel(), x.numel(), dtype=torch.float64, device=out.device)
        for e in range(x.numel()):
            dx = torch.zeros_like(x)
            dx.view(-1)[e] = steps.view(-1)[e]
            deltas = [None] * len(inputs)
            deltas[i] = dx
            with shifted(inputs, deltas):
                plus = _eval(fn)
            deltas[i] = -dx
            with shifted(inputs, deltas):
                minus = _eval(fn)
            J[:, e] = ((plus - minus) / (2 * steps.view(-1)[e].double())).reshape(-1)
        jacs.append(J)
    return out, jacs


def check_vjp(out, jacs, w, grads, label=''):
    """Every element of grads[i] (autograd's gradient of sum(w * out)) against w^T J_i, within
    RTOL * (|w|^T (|out| + |J_i|)): the module docstring's bound, summed over the outputs.  Returns a list of
    failures."""
    wf = w.detach().double().reshape(-1)
    scale_out = (wf.abs() * out.abs().reshape(-1)).sum()
    bad = []
    for i, (J, g) in enumerate(zip(jacs, grads)):
        ref = wf @ J
        if g is None:
            bad.append(f'{label} input {i}: no gradient (None)')
            continue
        got = g.detach().double().reshape(-1)
        tol = RTOL * (scale_out + wf.abs() @ J.abs())
        err = (got - ref).abs()
        if not bool((err <= tol).all()):
            k = int(torch.argmax(err / tol))
            bad.append(f'{label} input {i} element {k}: autograd {got[k].item():.17g}, central difference '
                       f'{ref[k].item():.17g}, |diff| {err[k].item():.3g} > bound {tol[k].item():.3g}')
    return bad


def check_jacobian(out, jacs, auto, label=''):
    """Autograd's full Jacobians `auto` (one (out.numel(), x.numel()) matrix per input, None: no gradient) against the
    central-difference ones, entry by entry within RTOL * (|out_o| + |J_oe|).  Returns a list of failures."""
    scale = out.abs().reshape(-1, 1)
    bad = []
    for i, (J, A) in enumerate(zip(jacs, auto)):
        if A is None:
            bad.append(f'{label} input {i}: no gradient (None)')
            continue
        tol = RTOL * (scale + J.abs())
        err = (A.double() - J).abs()
        if not bool((err <= tol).all()):
            k = int(torch.argmax(err / tol))
            o, e = divmod(k, J.shape[1])
            bad.append(f'{label} input {i} d out[{o}] / d x[{e}]: autograd {A.reshape(-1)[k].item():.17g}, central '
                       f'difference {J.reshape(-1)[k].item():.17g}, |diff| {err.reshape(-1)[k].item():.3g} > bound '
                       f'{tol.reshape(-1)[k].item():.3g}')
    return bad


def directional(fn, inputs, directions, w, h=H_REL):
    """Central difference of the loss sum(w * fn()) along `directions` (one tensor per input, None: not moved), the
    step h relative to the largest magnitude of the moved inputs.  Returns (D, L) with L = sum |w * fn()|."""
    out = _eval(fn)
    mag = max(float(x.detach().abs().max()) for x, v in zip(inputs, directions) if v is not None)
    s = h * max(mag, 1.0)
    with shifted(inputs, [None if v is None else s * v for v in directions]):
        plus = (w * _eval(fn)).sum()
    with shifted(inputs, [None if v is None else -s * v for v in directions]):
        minus = (w * _eval(fn)).sum()
    return float((plus - minus) / (2 * s)), float((w * out).abs().sum())


def rowwise_directional(fn, y0, V, w, h=H_REL, row_inputs=()):
    """One directional check per trajectory from a single pair of solves.  Trajectories are independent, so moving
    every row r of y0 (and of each per-row tensor in `row_inputs`, (B, ...) with its direction) by s * V[r] at once
    gives each row's own derivative: the central difference of l_r = sum_{t,j} w[t, r, j] ys[t, r, j].  fn() returns
    ys of shape (T, B, d).  Returns (D, L), both (B,): D[r] the central difference of l_r and L[r] = sum |w . ys| over
    row r, the scale of the bound.  The caller compares D[r] with (grad_y0[r] * V[r]).sum() (plus the per-row
    parameter terms), a wrong gradient in any one row failing on its own."""
    inputs = [y0] + [x for x, _ in row_inputs]
    dirs = [V] + [v for _, v in row_inputs]
    out = _eval(fn)
    mag = max(float(x.detach().abs().max()) for x in inputs)
    s = h * max(mag, 1.0)
    with shifted(inputs, [s * v for v in dirs]):
        plus = (w * _eval(fn)).sum(dim=(0, 2))
    with shifted(inputs, [-s * v for v in dirs]):
        minus = (w * _eval(fn)).sum(dim=(0, 2))
    return (plus - minus) / (2 * s), (w * out).abs().sum(dim=(0, 2))


def within(got, D, L):
    """|got - D| <= RTOL * (L + |D|), element-wise (the module docstring's bound).  Returns the boolean mask."""
    got = torch.as_tensor(got, dtype=torch.float64)
    D = torch.as_tensor(D, dtype=torch.float64, device=got.device)
    L = torch.as_tensor(L, dtype=torch.float64, device=got.device)
    return (got - D).abs() <= RTOL * (L + D.abs())
