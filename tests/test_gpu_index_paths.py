"""Every index path of the row-wise kernel framework (csrc/ew.cuh launch_ew) against a float64 restatement of each op
on the oracle's increments, and the paths against one another:

* the fast kernel with the shift (quads per row a power of two) and with the multiply-high division (any other
  quads per row), past local row 2^24 where a 2^40 reciprocal wraps 64 bits;
* the generic kernel (unaligned operands), which must give the fast kernel's bits on the same shape;
* multi-cell counter noise and the linear interpolation of output times (tests/test_gpu_solver.py
  test_ragged_ts_interpolation_and_reuse), and the adaptive-step error reduction.

The entry points are called through the C ABI.  Operand tensors are reused across slots to keep the large shapes
within an 80 GB device."""
import ctypes
import gc
import math

import numpy as np
import pytest
import torch

from oracle import brownian as obm
from oracle import solvers
from . import helpers, problems

pytestmark = pytest.mark.gpu
DEV = 'cuda'

BIG = 1 << 24      # first local row a 2^40 reciprocal gets wrong
TAIL = 4099        # rows past 2^24: TAIL * d/4 is not a multiple of 512 (256 threads x 2 quads) for d = 12, 20
KEY = 20261015     # Philox key (the key tensor holds it as int64)
CELL = 7           # counter id of the cell
H = 2.0 ** -4      # cell length = dt: every derived scalar (sqrt, 1/dt, dt/2) is exact in fp32
DT, SQ, RDT = H, math.sqrt(H), 1.0 / H

# ---- the entry points: (name, inputs, outputs, wants U, scalar arguments, float64 formula) ------------------------
# Inputs x, increment w, U u: float64 arrays.  The formulas restate torchsde_b200/csrc/tableau_diag_ops.cuh (which
# cites the reference's methods/*.py lines); brownian_cells returns the increment itself.


def _srk_final(x, w, u):
    y0, f, g = x[0], x[1:4], x[4:8]
    alpha, b1, b2 = (1 / 6, 1 / 6, 2 / 3), (-1, 4 / 3, 2 / 3), (1, -4 / 3, 1 / 3)
    b3, b4 = (2, -4 / 3, -2 / 3), (-2, 5 / 3, -2 / 3, 1)
    ikk = (w * w - DT) * 0.5
    i3 = (w * w * w - 3 * DT * w) / 6
    y1 = y0
    for s in range(3):
        y1 = y1 + alpha[s] * f[s] * DT + g[s] * (b1[s] * w + b2[s] * ikk / SQ + b3[s] * u * RDT + b4[s] * i3 * RDT)
    return [y1 + g[3] * (b4[3] * i3 * RDT)]


def _adj_b(x, w, u):
    y0, f0, f1, g0, g1, adj_y0, adj_z0, vjp_z = x
    a = adj_z0 + vjp_z
    return [y0 - (f0 + f1) * (DT / 2) - (g0 + g1) * (0.5 * w), adj_y0 + 2 * a, -a, adj_y0 * (DT / 2) + a * DT,
            adj_y0 * (0.5 * w) + a * w]


NOISE_OPS = [
    ('tsde_step_euler', 3, 1, False, (DT,), lambda x, w, u: [x[0] + x[1] * DT + x[2] * w]),
    ('tsde_milstein_vjp_seed', 1, 1, False, (DT, 1), lambda x, w, u: [x[0] * (0.5 * (w * w - DT))]),
    ('tsde_step_milstein', 4, 1, False, (DT,), lambda x, w, u: [x[0] + x[1] * DT + x[2] * w + x[3]]),
    ('tsde_step_milstein_gf', 4, 1, False, (DT, 2 * SQ, 1),
     lambda x, w, u: [x[0] + x[1] * DT + x[2] * w + (x[3] - x[2]) * (w * w - DT) / (2 * SQ)]),
    ('tsde_step_heun', 5, 1, False, (DT,),
     lambda x, w, u: [x[0] + (DT * (x[1] + x[2]) + x[3] * w + x[4] * w) * 0.5]),
    ('tsde_midpoint_predict', 3, 1, False, (DT / 2,), lambda x, w, u: [x[0] + DT / 2 * x[1] + 0.5 * (x[2] * w)]),
    ('tsde_euler_heun_predict', 2, 1, False, (), lambda x, w, u: [x[0] + x[1] * w]),
    ('tsde_step_euler_heun', 4, 1, False, (DT,), lambda x, w, u: [x[0] + DT * x[1] + (x[2] * w + x[3] * w) * 0.5]),
    ('tsde_reversible_heun_z', 4, 1, False, (DT,), lambda x, w, u: [2 * x[0] - x[1] + x[2] * DT + x[3] * w]),
    ('tsde_step_reversible_heun', 5, 1, False, (DT / 2,),
     lambda x, w, u: [x[0] + (x[1] + x[2]) * (DT / 2) + (x[3] + x[4]) * (0.5 * w)]),
    ('tsde_srk_diag_stage2', 5, 2, True, (DT, RDT, SQ),
     lambda x, w, u: [x[0] + 0.25 * x[1] * DT + x[2] * u * RDT + 0.25 * x[3] * DT + 0.5 * x[4] * u * RDT,
                      x[0] + x[1] * DT + x[2] * SQ]),
    ('tsde_step_srk_diag', 8, 1, True, (DT, RDT, SQ, 3 * DT), _srk_final),
    ('tsde_adjoint_reversible_heun_a', 7, 3, False, (DT, DT / 2),
     lambda x, w, u: [2 * x[0] - x[1] - x[2] * DT - x[3] * w, x[5] + x[4] * (DT / 2), x[6] + x[4] * (0.5 * w)]),
    ('tsde_adjoint_reversible_heun_b', 8, 5, False, (DT, DT / 2), _adj_b),
    ('tsde_brownian_cells', 0, 1, False, (), lambda x, w, u: [w]),
    ('tsde_brownian_cells', 0, 2, True, (), lambda x, w, u: [w, u]),
]
# element-wise entry points without noise: milstein.py:63 (ito, then Stratonovich), the SRK stage values H0_1 / H1_1
# and H1_3 (srk.py:70-76), and linear_interp as output times and log-ODE (weights 1, 1) use it
PLAIN_OPS = [
    ('tsde_milstein_gf_predict', 3, 1, False, (DT, SQ, 1), lambda x, w, u: [x[0] + DT * x[1] + x[2] * SQ]),
    ('tsde_milstein_gf_predict', 3, 1, False, (DT, SQ, 0), lambda x, w, u: [x[0] + x[2] * SQ]),
    ('tsde_srk_diag_stage1', 3, 2, False, (DT, SQ),
     lambda x, w, u: [x[0] + x[1] * DT, x[0] + 0.25 * x[1] * DT - 0.5 * x[2] * SQ]),
    ('tsde_srk_diag_stage3', 5, 1, False, (DT, SQ),
     lambda x, w, u: [x[0] + (2 * x[1] - x[2] + 0.5 * x[4]) * SQ + 0.25 * x[3] * DT]),
    ('tsde_linear_interp', 2, 1, False, (0.3, 0.7), lambda x, w, u: [0.3 * x[0] + 0.7 * x[1]]),
    ('tsde_linear_interp', 2, 1, False, (1.0, 1.0), lambda x, w, u: [x[0] + x[1]]),
]


def plain_emulated(op, x):
    """The outputs of noise-free op `op` on numpy inputs x in T, in the op's written order (tableau_diag_ops.cuh: one
    IEEE rounding per operation, no fma under -fmad=false); the double scalars are cast to T."""
    name, nin, _, _, scalars, _ = op
    T = x[0].dtype.type
    s = [T(v) for v in scalars]
    if name == 'tsde_milstein_gf_predict':
        y0, f, g = x[:3]
        fac = s[0] * f if scalars[2] else np.zeros_like(f)
        return [(y0 + fac) + g * s[1]]
    if name == 'tsde_srk_diag_stage1':
        y0, f0, g0 = x[:3]
        return [y0 + (T(1) * f0) * s[0], (y0 + (T(0.25) * f0) * s[0]) + (T(-0.5) * g0) * s[1]]
    if name == 'tsde_srk_diag_stage3':
        y0, g0, g1, f2, g2 = x[:5]
        h1 = y0 + (T(2) * g0) * s[1]
        h1 = h1 + (T(-1) * g1) * s[1]
        return [(h1 + (T(0.25) * f2) * s[0]) + (T(0.5) * g2) * s[1]]
    assert name == 'tsde_linear_interp'
    return [s[0] * x[0] + s[1] * x[1]]


def tol_of(npdt):
    """The formula checks' tolerance."""
    return dict(rtol=5e-5, atol=1e-5) if npdt == np.float32 else dict(rtol=1e-11, atol=1e-12)


def _op_id(op):
    if op[0] == 'tsde_milstein_gf_predict' and not op[4][2]:
        return 'milstein_gf_predict_strat'
    if op[0] == 'tsde_linear_interp':
        return 'linear_interp_%g_%g' % op[4]
    return op[0][5:] + ('_wu' if op[0] == 'tsde_brownian_cells' and op[2] == 2 else '')


def _cabi():
    from torchsde_b200 import _cabi
    return _cabi


def _noise(key, want_u, row_offset=0, mem=None):
    """Counter noise of cell CELL (or, with mem = (w_ptr, u_ptr), the same increments read from memory)."""
    c = _cabi()
    nz = c.Noise()
    nz.source, nz.want_u, nz.key, nz.cell_id, nz.n_cells = c.SRC_COUNTER, int(want_u), key.data_ptr(), CELL, 1
    nz.h, nz.h_total, nz.row_offset = H, H, row_offset
    if mem is not None:
        nz.source, nz.w, nz.u = c.SRC_MEMORY, mem[0], mem[1]
    return nz


def _launch(op, dtype, rows, d, ins, outs, nz):
    """One call of entry point `op` on `rows` rows; ins / outs are device addresses."""
    c = _cabi()
    name, nin, nout, want_u, scalars, _ = op
    L = c.make_launch(dtype, c.NOISE_DIAGONAL, rows, d, d)
    if name == 'tsde_brownian_cells':
        args = [outs[0], outs[1] if nout == 2 else None, None]
    else:
        args = list(ins[:nin]) + list(scalars) + list(outs[:nout])
    head = [ctypes.byref(L)] + ([ctypes.byref(nz)] if op in NOISE_OPS else [])
    c.check(getattr(c.lib(), name)(*head, *args), name)


def _ins(pool, nin, shift=0):
    """Device addresses of the op's inputs: slot i reads pool tensor i % len(pool), `shift` bytes in."""
    return [pool[i % len(pool)].data_ptr() + shift for i in range(nin)]


def _free_memory():
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


# ---- (a) local rows past 2^24 --------------------------------------------------------------------------------------
@pytest.mark.parametrize('d,dtype', [(12, torch.float32), (20, torch.float32), (12, torch.float64)])
def test_rows_past_2_24(d, dtype):
    """B = 2^24 + 4099 rows with d/4 not a power of two: the fast kernel's multiply-high row division.  For every
    counter-noise diagonal entry point and the Brownian W / (W, U) materialisation:
      * the launch split at row 2^24 (second launch at row_offset 2^24) gives the same bits on every row;
      * the same operands one element off 16-byte alignment (the generic kernel) give the same bits;
      * sampled rows (0, 2^24 - 1, 2^24, 2^24 + 1, B - 1 and 256 random rows past 2^24) match the op's float64
        formula on the oracle's increments for those rows."""
    B, es = BIG + TAIL, torch.finfo(dtype).bits // 8
    n = B * d
    need = 16 * (n + 1) * es  # 3 inputs, their unaligned copies, 5 + 5 outputs
    if _free_memory() < 1.1 * need + (1 << 30):
        pytest.skip(f'needs ~{need / 2 ** 30:.0f} GiB of free device memory')
    npdt = np.float32 if dtype == torch.float32 else np.float64
    tol = tol_of(npdt)
    gen = torch.Generator(device=DEV).manual_seed(d)
    pool = [torch.rand(B, d, generator=gen, device=DEV, dtype=dtype) + 0.5 for _ in range(3)]
    pool_u = []  # the same values one element past a 16-byte boundary
    for x in pool:
        buf = torch.empty(n + 1, device=DEV, dtype=dtype)
        buf[1:].copy_(x.view(-1))
        pool_u.append(buf)
    out_a = [torch.empty(B, d, device=DEV, dtype=dtype) for _ in range(5)]
    out_b = [torch.empty(n + 1, device=DEV, dtype=dtype) for _ in range(5)]
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    rng = np.random.default_rng(d)
    rows = np.unique(np.concatenate([[0, BIG - 1, BIG, BIG + 1, B - 1], rng.integers(BIG, B, 256)]))
    rows_dev = torch.from_numpy(rows).to(DEV)
    x_rows = [x[rows_dev].double().cpu().numpy() for x in pool]
    bad = []
    for op in NOISE_OPS + PLAIN_OPS:
        name, nin, nout, want_u, _, formula = op
        _launch(op, dtype, B, d, _ins(pool, nin), [o.data_ptr() for o in out_a], _noise(key, want_u))
        # the same work as two launches split at local row 2^24
        off = BIG * d * es
        _launch(op, dtype, BIG, d, _ins(pool, nin), [o.data_ptr() for o in out_b], _noise(key, want_u))
        _launch(op, dtype, TAIL, d, _ins(pool, nin, off), [o.data_ptr() + off for o in out_b],
                _noise(key, want_u, row_offset=BIG))
        for i in range(nout):
            if not torch.equal(out_a[i].view(-1), out_b[i][:n]):
                first = int((out_a[i].view(-1) != out_b[i][:n]).nonzero()[0]) // d
                bad.append(f'{_op_id(op)} out{i}: one launch != split at 2^24 (first differing row {first})')
        # float64 formula on the oracle's increments, sampled rows
        W = U = None
        if op in NOISE_OPS:
            W, Hh = obm.cell(KEY, CELL, H, len(rows), d, npdt, want_u, row_ids=rows)
            U = obm.h_to_u(W, Hh, H).astype(np.float64) if want_u else None
            W = W.astype(np.float64)
        ref = formula([x_rows[i % 3] for i in range(nin)], W, U)
        for i in range(nout):
            got = out_a[i][rows_dev].double().cpu().numpy()
            if not np.allclose(got, ref[i], **tol):
                wrong = rows[~np.all(np.isclose(got, ref[i], **tol), axis=1)]
                bad.append(f'{_op_id(op)} out{i}: {len(wrong)} of {len(rows)} sampled rows off the oracle '
                           f'(first {wrong[:3].tolist()})')
        # the generic kernel on unaligned operands
        _launch(op, dtype, B, d, _ins(pool_u, nin, es), [o.data_ptr() + es for o in out_b], _noise(key, want_u))
        for i in range(nout):
            if not torch.equal(out_a[i].view(-1), out_b[i][1:]):
                bad.append(f'{_op_id(op)} out{i}: fast kernel != generic kernel')
    del pool, pool_u, out_a, out_b
    torch.cuda.empty_cache()
    assert not bad, '\n'.join(bad)


# ---- (b) a solve and Brownian queries at that size -----------------------------------------------------------------
def test_solve_and_queries_past_2_24_rows():
    """sdeint (Ito Milstein, diagonal noise, d = 12) on 2^24 + 4099 trajectories:
      * sampled rows match the oracle solver on the oracle's increments;
      * the tail solved alone (shard_rows(2^24)) is bit-identical to the same rows of the whole solve;
      * a space-time BrownianInterval's whole-cell (W, U) query equals two half-cell queries of a fresh interval
        with the same entropy, W = W1 + W2 and U = U1 + U2 + h2 W1 (the half-cell queries draw the cell through a
        different kernel, with 64-bit row arithmetic), to fp32 rounding."""
    import torchsde_b200 as tsde
    B, d = BIG + TAIL, 12
    if _free_memory() < 24 * B * d * 4 + (2 << 30):
        pytest.skip(f'needs ~{24 * B * d * 4 / 2 ** 30 + 2:.0f} GiB of free device memory')
    sde = problems.GBMDiagonal(d, 'ito', seed=12, dtype=torch.float32).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    y0 = 0.2 + 0.3 * torch.rand(B, d, generator=gen, device=DEV)
    ts = torch.tensor([0.0, 0.125, 0.25], device=DEV)
    dt = 2.0 ** -4
    bm = tsde.BrownianInterval(0.0, 0.25, size=(B, d), dtype=torch.float32, device=DEV, entropy=2024)
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=dt)
    rows = helpers.sample_rows(B, 256, seed=1)
    rows = np.unique(np.concatenate([rows, [BIG - 1, BIG, BIG + 1], np.random.default_rng(2).integers(BIG, B, 256)]))
    rows_dev = torch.from_numpy(rows).to(DEV)
    sde_cpu = problems.GBMDiagonal(d, 'ito', seed=12, dtype=torch.float32)
    ref, _ = solvers.make('milstein', problems.NumpySDE(sde_cpu),
                          helpers.oracle_grid_bm(bm, rows, d, np.float32, False), dt).integrate(
        y0[rows_dev].cpu().numpy(), ts.cpu().numpy())
    np.testing.assert_allclose(ys[:, rows_dev].cpu().numpy(), ref, rtol=5e-5, atol=1e-5)

    tail_bm = tsde.BrownianInterval(0.0, 0.25, size=(TAIL, d), dtype=torch.float32, device=DEV, entropy=2024)
    tail_bm.shard_rows(BIG)
    with torch.no_grad():
        tail = tsde.sdeint(sde, y0[BIG:].contiguous(), ts, bm=tail_bm, method='milstein', dt=dt)
    assert torch.equal(ys[:, BIG:], tail)
    del ys, tail, y0, bm, tail_bm
    torch.cuda.empty_cache()

    kw = dict(size=(B, d), dtype=torch.float32, device=DEV, entropy=77, dt=0.25, levy_area_approximation='space-time')
    whole = tsde.BrownianInterval(0.0, 1.0, **kw)
    halves = tsde.BrownianInterval(0.0, 1.0, **kw)
    W, U = whole(0.25, 0.5, return_U=True)
    W1, U1 = halves(0.25, 0.375, return_U=True)
    W2, U2 = halves(0.375, 0.5, return_U=True)
    torch.testing.assert_close(W[BIG:], (W1 + W2)[BIG:], rtol=1e-5, atol=5e-6)
    torch.testing.assert_close(U[BIG:], (U1 + U2 + 0.125 * W1)[BIG:], rtol=1e-5, atol=5e-6)
    torch.testing.assert_close(W[:BIG], (W1 + W2)[:BIG], rtol=1e-5, atol=5e-6)


# ---- (c) generic kernel == fast kernel -----------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('d', [4, 12, 64])
def test_generic_kernel_equals_fast_kernel(d, dtype):
    """Operands one element off 16-byte alignment take the generic kernel (ew_kernel); aligned ones take the fast
    kernel (ew_fast_kernel).  Every diagonal entry point, with counter and with memory noise, must give the same bits
    either way.  Batch sizes cover one partial CTA, and full grids whose per-CTA slices end in a partial iteration of
    the two-quads-per-thread ops.  The noise-free ops must also give the bits of a numpy emulation of their written
    order in T."""
    es = torch.finfo(dtype).bits // 8
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(d)
    bad, host = [], None
    for B in (1, 37, 1000, 300007):
        n = B * d
        pool_u = [torch.rand(n + 1, generator=gen, device=DEV, dtype=dtype) + 0.5 for _ in range(5)]
        pool = [x[1:].clone() for x in pool_u]  # the same values, aligned
        mem_u = [torch.randn(n + 1, generator=gen, device=DEV, dtype=dtype) * SQ for _ in range(2)]  # W, U
        mem = [x[1:].clone() for x in mem_u]
        out_a = [torch.empty(n, device=DEV, dtype=dtype) for _ in range(5)]
        out_b = [torch.empty(n + 1, device=DEV, dtype=dtype) for _ in range(5)]
        for op in NOISE_OPS + PLAIN_OPS:
            sources = ('counter', 'memory') if op in NOISE_OPS and op[0] != 'tsde_brownian_cells' else ('counter',)
            for src in sources:
                nz_a = _noise(key, op[3], mem=(mem[0].data_ptr(), mem[1].data_ptr()) if src == 'memory' else None)
                nz_b = _noise(key, op[3], mem=(mem_u[0].data_ptr() + es, mem_u[1].data_ptr() + es)
                              if src == 'memory' else None)
                _launch(op, dtype, B, d, _ins(pool, op[1]), [o.data_ptr() for o in out_a], nz_a)
                _launch(op, dtype, B, d, _ins(pool_u, op[1], es), [o.data_ptr() + es for o in out_b], nz_b)
                for i in range(op[2]):
                    if not torch.equal(out_a[i], out_b[i][1:]):
                        bad.append(f'B={B} {_op_id(op)} {src} out{i}: fast kernel != generic kernel')
                if op in PLAIN_OPS:
                    host = host or [x.cpu().numpy() for x in pool]
                    for i, e in enumerate(plain_emulated(op, host[:op[1]])):
                        if not np.array_equal(out_a[i].cpu().numpy().view(np.uint8), e.view(np.uint8)):
                            bad.append(f'B={B} {_op_id(op)} out{i}: not the numpy emulation\'s bits')
        host = None
    assert not bad, ', '.join(bad)


# ---- (e) adaptive-step error reduction -----------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_adaptive_error_sumsq_vs_numpy(dtype):
    """tsde_adaptive_error_sumsq over 3 000 017 elements (a grid-stride loop over the 592 fixed partials, a partial
    last CTA): sum of ((y11 - y12) / tol)^2, tol = max(rtol * max(|y11|, |y12|) + atol, eps), each term rounded in the
    tensor dtype and summed in float64, against numpy; with elements whose tolerance clamps to eps and elements where
    y11 == y12.  Two launches give the same bits."""
    c = _cabi()
    npdt = np.float32 if dtype == torch.float32 else np.float64
    n = 3_000_017
    rng = np.random.default_rng(11)
    y11 = rng.standard_normal(n).astype(npdt)
    y12 = (y11 + rng.standard_normal(n).astype(npdt) * npdt(1e-3)).astype(npdt)
    y12[::7] = y11[::7]                       # equal: zero terms
    tiny = np.arange(3, n, 13)
    y11[tiny] *= npdt(1e-9)                   # tolerance below eps: clamped
    y12[tiny] = (y11[tiny] + npdt(2e-9)).astype(npdt)
    rtol, atol, eps = 1e-3, 1e-9, 1e-7
    t = np.maximum(npdt(rtol) * np.maximum(np.abs(y11), np.abs(y12)) + npdt(atol), npdt(eps))
    assert (t == npdt(eps)).sum() > 1000
    r = (y11 - y12) / t
    ref = float(np.sum((r * r).astype(np.float64)))
    a, b = torch.from_numpy(y11).to(DEV), torch.from_numpy(y12).to(DEV)
    scratch = torch.empty(592, dtype=torch.float64, device=DEV)
    outs = []
    for _ in range(2):
        out = torch.empty(1, dtype=torch.float64, device=DEV)
        L = c.make_launch(dtype, c.NOISE_DIAGONAL, n, 1, 1)
        c.check(c.lib().tsde_adaptive_error_sumsq(ctypes.byref(L), a.data_ptr(), b.data_ptr(), rtol, atol, eps,
                                                  scratch.data_ptr(), out.data_ptr()), 'tsde_adaptive_error_sumsq')
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    got = float(outs[0].item())
    assert abs(got - ref) <= 1e-12 * ref, (got, ref)
