"""Every index path of the fused element-wise kernels (torchsde_b200/csrc/pointwise.cu, pw_device.cuh and the NVRTC
units of pw_milstein_source / pw_general_source) at batch sizes where their index arithmetic can go wrong.

Each kernel maps its flat quad index to (row, quad of the row) in one of three ways (fill_quad_map): a shift when the
quads per row are a power of two, a 32-bit multiply-high division (rowdiv.cuh) while there are fewer than 2^31 quads,
and a 64-bit division beyond.  pw_begin serves the SRK and predictor-corrector kernels, pw_locate every other one, and
pw_general_noise draws a general-noise row's increments on its global row.

(1) sdeint on B = 2^24 + 4099 trajectories (the last CTA is partial), at d = 12 (three quads per row: the division,
    16-byte quads), d = 11 (the division, a three-lane last quad, the element path) and d = 16 (the shift, as a
    control), one case per fused kernel family, each confirmed by its launch counter:
      1. the fused solve gives the bits of the same solve with the tape rejected (the unfused step);
      2. sampled rows (0, 1, 2^24 - 2 .. 2^24 + 1, B - 2, B - 1 and 256 random ones) match the numpy oracle
         (oracle/solvers.py) on the oracle's own increments for their global rows: |got - ref| <= tol * max(|ref|,
         scale), tol = 1e-5 in float32 and 1e-11 in float64, scale a tenth of the largest |ref|.  This does not lean on
         the unfused path, so it also checks the unfused general-noise tile kernels past local row 2^24;
      3. rows 0, 1 and 2^24 - 2 .. 2^24 + 1 start from the same state, so they must end in different states in every
         channel: a row that draws its neighbour's increments, or row 0's, is named as such.
    Variants on one diagonal and one general family: steps that span several Brownian cells, a CUDA-graph solve with
    row blocks, and a shard whose global rows end at the top of the Philox row space (rows + offset = 2^32 - 1, the
    most a launch accepts).
(2) the 64-bit division, through the C ABI: more than 2^31 quads in one launch, with quads per row not a power of
    two.

Every case frees its tensors; a case skips, naming the free and the needed bytes, where the device has too little
memory.  test_report_worst_ratio prints the worst error / bound of check 2 per dtype."""
import ctypes
import gc
import json

import numpy as np
import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import graph
from oracle import brownian as obm
from oracle import solvers
from . import helpers, problems
from .test_gpu_pointwise import SDE as DiagonalSDE, same_bits
from .test_gpu_pointwise_adaptive import unfused
from .test_gpu_pointwise_general import SDE as GeneralSDE
from .test_gpu_pointwise_sra import SDE as AdditiveSDE

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = _cabi.PW_MAX_STEPS
BIG = 1 << 24                 # the first local row a 24-bit or 2^40-reciprocal row index gets wrong
B = BIG + 4099                # as tests/test_gpu_index_paths.py: the last CTA is partial at d = 11, 12, 16
TOP = (1 << 32) - 1 - B       # a shard whose last global row is 2^32 - 2, the last row a launch may draw
DT = 2.0 ** -6
T = K + 2                     # the chunk kernels run a chunk of K steps, then one of 2
SAME = [0, 1, BIG - 2, BIG - 1, BIG, BIG + 1]   # rows that start from one state (check 3)
NEIGHBOURS = [(BIG - 2, BIG - 1), (BIG - 1, BIG), (BIG, BIG + 1), (0, BIG), (1, BIG + 1), (0, 1)]
ROWS = np.unique(np.concatenate([SAME, [B - 2, B - 1], np.random.default_rng(24).integers(0, B, 256)]))
TOL = {torch.float32: 1e-5, torch.float64: 1e-11}
WORST = {}                    # dtype -> worst err / bound of check 2 over this file's cases

COUNTER = {'milstein': _cabi.KERNEL_PW_MILSTEIN, 'euler': _cabi.KERNEL_PW_CHUNK,
           'reversible_heun': _cabi.KERNEL_PW_CHUNK, 'srk': _cabi.KERNEL_PW_SRK, 'heun': _cabi.KERNEL_PW_PC,
           'midpoint': _cabi.KERNEL_PW_PC, 'euler_heun': _cabi.KERNEL_PW_PC}
SDE_TYPE = {'euler': 'ito', 'midpoint': 'stratonovich', 'euler_heun': 'stratonovich', 'reversible_heun': 'stratonovich'}


def launches(counter):
    return _cabi.lib().tsde_kernel_launches(counter)


@pytest.fixture(autouse=True)
def memory():
    """Each case starts and ends with the device memory of the cases before it returned."""
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def need(nbytes):
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes:
        pytest.skip(f'needs {nbytes} bytes of free device memory, {free} free')


def start(d, dtype):
    """y0 in [0.2, 0.5), the rows of SAME set to row 0's."""
    gen = torch.Generator(device=DEV).manual_seed(d)
    y0 = 0.2 + 0.3 * torch.rand(B, d, generator=gen, device=DEV, dtype=dtype)
    y0[SAME] = y0[0].clone()
    return y0


def solve(sde, y0, method, m, levy, options, bm_dt, row_offset, adaptive):
    t1 = 0.25 if adaptive else T * DT  # (adaptive: two or three proposals from dt = 0.125)
    bm = tsde.BrownianInterval(0.0, t1, size=(B, m), dtype=y0.dtype, device=DEV, entropy=2024, dt=bm_dt,
                               levy_area_approximation=levy)
    if row_offset:
        bm.shard_rows(row_offset)
    ts = torch.tensor([0.0, t1], dtype=y0.dtype, device=DEV)
    kw = dict(adaptive=True, rtol=0.1, atol=0.01, dt_min=1e-3) if adaptive else {}
    with torch.no_grad():
        ys = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=0.125 if adaptive else DT,
                         options=dict(options or {}), **kw)
    graph.drop_plans(sde)
    return ys, bm, ts


def check(make, method, d, m, dtype, counter, levy='none', options=None, bm_dt=None, row_offset=0, adaptive=False,
          oracle=True):
    """Checks 1-3 of the module docstring for the SDE make(device_or_None) solved by `method` with m Brownian
    channels; `counter` is the fused kernel's launch counter."""
    es = torch.finfo(dtype).bits // 8
    g_wide = m if make(False).noise_type != 'diagonal' else 0   # the unfused general step materialises g
    need(es * B * d * (10 + 4 * g_wide) + (1 << 30))
    y0 = start(d, dtype)
    sde = make(True)
    n0 = launches(counter)
    ys, bm, ts = solve(sde, y0, method, m, levy, options, bm_dt, row_offset, adaptive)
    assert launches(counter) > n0, "the steps were not fused"
    with unfused():
        n1 = launches(counter)
        ref, _, _ = solve(sde, y0, method, m, levy, options, bm_dt, row_offset, adaptive)
        assert launches(counter) == n1
    if not same_bits(ys, ref):
        it = torch.int32 if dtype == torch.float32 else torch.int64
        first = int((ys.view(it) != ref.view(it)).any(-1).any(0).nonzero()[0])
        pytest.fail(f"fused != unfused (first differing row {first})")
    del ref
    last = ys[-1]
    for a, b in NEIGHBOURS:
        assert bool((last[a] != last[b]).all()), f"rows {a} and {b} drew the same increments"
    if not oracle:
        return
    rows_dev = torch.from_numpy(ROWS).to(DEV)
    got = ys[:, rows_dev].double().cpu().numpy()
    npdt = np.float32 if dtype == torch.float32 else np.float64
    want, _ = solvers.make(method, problems.NumpySDE(make(False)),
                           helpers.oracle_grid_bm(bm, ROWS, m, npdt, levy != 'none'), DT).integrate(
        y0[rows_dev].cpu().numpy(), ts.cpu().numpy())
    want = want.astype(np.float64)
    bound = TOL[dtype] * np.maximum(np.abs(want), 0.1 * np.abs(want).max())
    ratio = np.abs(got - want) / bound
    name = str(dtype).replace('torch.', '')
    WORST[name] = max(WORST.get(name, 0.0), float(ratio.max()))
    print(f"{method} d={d} m={m} {name}: worst err / bound {ratio.max():.3g}")
    wrong = ROWS[(ratio > 1).any(axis=(0, 2))]
    assert not len(wrong), f"{len(wrong)} of {len(ROWS)} sampled rows off the oracle (first {wrong[:4].tolist()})"


# ---- (1) diagonal noise ---------------------------------------------------------------------------------------------
def diagonal(sde_type, d, dtype):
    def make(on_device):
        sde = DiagonalSDE('gbm', sde_type, B, d, dtype)
        return sde.to(DEV) if on_device else sde
    return make


VARIANTS = {'': {}, 'multi_cell': {'bm_dt': DT / 4}, 'graph': {'options': {'cuda_graph': True}},
            'graph_row_split': {'options': {'cuda_graph': True, 'row_split': 3}}, 'top_shard': {'row_offset': TOP}}
F32, F64 = torch.float32, torch.float64
DIAGONAL = [('milstein', 'ito', 12, F32, ''), ('milstein', 'stratonovich', 11, F32, ''),
            ('milstein', 'ito', 12, F64, ''), ('milstein', 'ito', 16, F32, ''),
            ('milstein', 'ito', 12, F32, 'multi_cell'), ('milstein', 'ito', 12, F32, 'graph_row_split'),
            ('milstein', 'ito', 12, F32, 'top_shard'),
            ('euler', 'ito', 12, F32, ''), ('reversible_heun', 'stratonovich', 11, F32, ''),
            ('srk', 'ito', 12, F32, ''),
            ('heun', 'stratonovich', 12, F32, ''), ('midpoint', 'stratonovich', 11, F32, ''),
            ('euler_heun', 'stratonovich', 12, F32, '')]


@pytest.mark.parametrize('method,sde_type,d,dtype,variant', DIAGONAL,
                         ids=[f"{c[0]}-{c[1][:5]}-d{c[2]}-{str(c[3])[-7:]}{'-' + c[4] if c[4] else ''}"
                              for c in DIAGONAL])
def test_diagonal_rows_past_2_24(method, sde_type, d, dtype, variant):
    """Milstein (Ito at d = 12, 16 and in float64; Stratonovich at d = 11), Euler, reversible Heun, SRK (which also
    draws U), Heun, midpoint and Euler-Heun on diagonal GBM; with Milstein, multi-cell steps, a graph with row blocks
    and the shard at the top of the row space."""
    check(diagonal(sde_type, d, dtype), method, d, d, dtype, COUNTER[method],
          levy='space-time' if method == 'srk' else 'none', **VARIANTS[variant])


# ---- (1) general and additive noise ---------------------------------------------------------------------------------
GENERAL = [(method, m, '') for method in ('euler', 'midpoint', 'euler_heun', 'reversible_heun') for m in (1, 3, 4)]
GENERAL += [('euler', 3, 'multi_cell'), ('euler', 4, 'graph_row_split'), ('midpoint', 3, 'top_shard'),
            ('reversible_heun', 3, 'graph')]


@pytest.mark.parametrize('method,m,variant', GENERAL,
                         ids=[f"{c[0]}-m{c[1]}{'-' + c[2] if c[2] else ''}" for c in GENERAL])
def test_general_rows_past_2_24(method, m, variant):
    """Euler, midpoint, Euler-Heun and reversible Heun on correlated GBM (g = y * S, S of shape (d, m)) at d = 12, in
    float32; m = 1, 3 and 4 take the row-wise, generic and tile contraction orders.  With Euler, multi-cell steps and a
    graph with row blocks; the shard at the top of the row space with midpoint; a graph solve of reversible Heun (whose
    solver state rules out row blocks)."""
    d, dtype = 12, torch.float32

    def make(on_device):
        sde = GeneralSDE('gbm', SDE_TYPE[method], d, m, dtype)
        return sde.to(DEV) if on_device else sde
    check(make, method, d, m, dtype, _cabi.KERNEL_PW_GENERAL, **VARIANTS[variant])


def test_additive_sra1_rows_past_2_24():
    """SRK on additive noise (sra1, which draws U) with m = 3, on OU with an `expand`ed (d, m) diffusion."""
    d, m, dtype = 12, 3, torch.float32

    def make(on_device):
        sde = AdditiveSDE('ou', d, m, dtype)
        return sde.to(DEV) if on_device else sde
    check(make, 'srk', d, m, dtype, _cabi.KERNEL_PW_GENERAL, levy='space-time')


@pytest.mark.filterwarnings('ignore:Numerical solution is not guaranteed')
@pytest.mark.parametrize('method', ['euler', 'milstein'])
def test_adaptive_proposals_rows_past_2_24(method):
    """The step-doubling proposal kernel of an adaptive Euler and Ito Milstein solve, two or three proposals.  Its
    increments are Brownian queries off the solver grid, which the oracle's grid-bound Brownian motion cannot restate:
    checks 1 and 3 only."""
    check(diagonal('ito', 12, F32), method, 12, 12, F32, _cabi.KERNEL_PW_ADAPTIVE,
          adaptive=True, oracle=False)


# ---- (2) more than 2^31 quads through the C ABI ---------------------------------------------------------------------
ROWS64, D64, M64 = (1 << 23) + (1 << 16), 1020, 4   # 255 quads per row (not a power of two), 2^31 + 8323072 quads
EDGE = (1 << 31) // 255                             # the row whose quad 128 is flat quad 2^31
KEY, CELL, H = 20261018, 41, 2.0 ** -4


def _program(reserved, g_kind, mu, g_operand):
    """f = mu * y | g = s * y: operand 0 is mu (CHANNEL), operand 1 s (CHANNEL sigma, or DM S of a general layout)."""
    prog = _cabi.Pointwise()
    prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands = 2, 1, 2, 2
    prog.f_src, prog.g_src, prog.gdg_src, prog.reserved = 0, 1, 0, reserved
    for j, (op, dst, a, b) in enumerate([(_cabi.PW_MUL, 0, _cabi.PW_OPERAND0, _cabi.PW_SRC_Y),
                                         (_cabi.PW_MUL, 1, _cabi.PW_OPERAND0 + 1, _cabi.PW_SRC_Y)]):
        prog.instr[j].op, prog.instr[j].dst, prog.instr[j].a, prog.instr[j].b = op, dst, a, b
    prog.operand[0].kind, prog.operand[0].ptr = _cabi.PW_CHANNEL, mu.data_ptr()
    prog.operand[1].kind, prog.operand[1].ptr = g_kind, g_operand.data_ptr()
    return prog


def test_more_than_2_31_quads():
    """rows x ceil(d / 4) = 8454144 x 255 quads, past 2^31, with 255 quads per row: the 64-bit division of pw_locate
    and pw_begin (d = 1024 would take the shift).  One float32 tensor y is updated in place by three launches, each a
    fused kernel that reads a thread's quad before it writes it (y0 == y1 is accepted by the host code: no entry point
    compares them):
      * tsde_solve_euler_pointwise, two Euler steps of diagonal GBM with (d,) CHANNEL operands (pw_locate);
      * tsde_step_predictor_corrector_pointwise, one midpoint step (pw_begin);
      * the general-noise Euler unit with m = 4, g = y * S with S a (d, m) DM operand (pw_locate, pw_general_noise).
    After each, rows 0, 1, the middle ones, the three around flat quad 2^31 and the last two match a float64
    restatement of the step on the oracle's increments for those rows (obm.cell(..., row_ids=...))."""
    es = 4
    nbytes = ROWS64 * D64 * es
    need(nbytes + (2 << 30))
    lib = _cabi.lib()
    gen = torch.Generator().manual_seed(64)
    mu = (torch.rand(D64, generator=gen) - 0.5).to(DEV)
    sigma = (0.1 + 0.5 * torch.rand(D64, generator=gen)).to(DEV)
    S = (0.05 + 0.25 * torch.rand(D64, M64, generator=gen)).to(DEV)
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    t0 = torch.zeros(1, device=DEV)
    t_half = torch.full((1,), H / 2, device=DEV)
    rows = np.array([0, 1, ROWS64 // 2 - 1, ROWS64 // 2, EDGE - 1, EDGE, EDGE + 1, ROWS64 - 2, ROWS64 - 1])
    rows_dev = torch.from_numpy(rows).to(DEV)
    y = torch.empty(ROWS64, D64, device=DEV)
    y.copy_(torch.linspace(0.2, 0.6, D64, device=DEV).expand(ROWS64, D64))
    want = y[rows_dev].double().cpu().numpy()
    mu64, sigma64, S64 = (x.double().cpu().numpy() for x in (mu, sigma, S))

    def noise(cell):
        nz = _cabi.Noise()
        nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, key.data_ptr(), cell, 1, H, H
        return nz

    def increments(cell, m):
        return obm.cell(KEY, cell, H, len(rows), m, np.float32, False, row_ids=rows)[0].astype(np.float64)

    def compare(what, counter, n0):
        torch.cuda.synchronize()
        assert launches(counter) > n0, f"{what}: no fused launch"
        got = y[rows_dev].double().cpu().numpy()
        bound = 1e-5 * np.maximum(np.abs(want), 0.1 * np.abs(want).max())
        ratio = np.abs(got - want) / bound
        WORST['float32'] = max(WORST.get('float32', 0.0), float(ratio.max()))
        print(f"{what}: worst err / bound {ratio.max():.3g}")
        wrong = rows[(ratio > 1).any(axis=1)]
        assert not len(wrong), f"{what}: rows {wrong.tolist()} off the float64 restatement"

    # two Euler steps, the first kept in registers
    L = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL, ROWS64, D64, D64)
    prog = _program(0, _cabi.PW_CHANNEL, mu, sigma)
    steps = (_cabi.PwStep * 2)()
    for j in range(2):
        steps[j].cell_id, steps[j].h, steps[j].dt, steps[j].t0 = CELL + j, H, H, t0.data_ptr()
    steps[1].y1 = y.data_ptr()
    n0 = launches(_cabi.KERNEL_PW_CHUNK)
    _cabi.check(lib.tsde_solve_euler_pointwise(ctypes.byref(L), ctypes.byref(noise(CELL)), ctypes.byref(prog),
                                               y.data_ptr(), steps, 2), 'tsde_solve_euler_pointwise')
    for j in range(2):
        want = want + mu64 * want * H + sigma64 * want * increments(CELL + j, D64)
    compare('Euler chunk', _cabi.KERNEL_PW_CHUNK, n0)

    # one midpoint step (Stratonovich): y' = y + H/2 f(y) + 0.5 g(y) W, y1 = y + H f(y') + g(y') W
    n0 = launches(_cabi.KERNEL_PW_PC)
    _cabi.check(lib.tsde_step_predictor_corrector_pointwise(
        ctypes.byref(L), ctypes.byref(noise(CELL + 2)), ctypes.byref(prog), y.data_ptr(), t0.data_ptr(),
        t_half.data_ptr(), _cabi.PC_MIDPOINT, H, H / 2, y.data_ptr()), 'tsde_step_predictor_corrector_pointwise')
    W = increments(CELL + 2, D64)
    mid = want + H / 2 * mu64 * want + 0.5 * sigma64 * want * W
    want = want + H * mu64 * mid + sigma64 * mid * W
    compare('midpoint step', _cabi.KERNEL_PW_PC, n0)

    # one general-noise Euler step, m = 4
    LG = _cabi.make_launch(torch.float32, _cabi.NOISE_GENERAL, ROWS64, D64, M64)
    gprog = _program(_cabi.PW_LAYOUT_GENERAL, _cabi.PW_DM, mu, S)
    step = (_cabi.PwStep * 1)()
    step[0].cell_id, step[0].h, step[0].dt, step[0].t0, step[0].y1 = CELL + 3, H, H, t0.data_ptr(), y.data_ptr()
    n0 = launches(_cabi.KERNEL_PW_GENERAL)
    _cabi.check(lib.tsde_solve_euler_pointwise(ctypes.byref(LG), ctypes.byref(noise(CELL + 3)), ctypes.byref(gprog),
                                               y.data_ptr(), step, 1), 'tsde_solve_euler_pointwise (general)')
    W = increments(CELL + 3, M64)
    want = want + mu64 * want * H + np.einsum('rd,dk,rk->rd', want, S64, W)
    compare('general Euler step', _cabi.KERNEL_PW_GENERAL, n0)
    del y


def test_report_worst_ratio():
    """(runs after the cases above) the worst err / bound of the oracle checks per dtype."""
    if not WORST:
        pytest.skip('no case ran')
    print('worst err/bound', json.dumps(WORST))
    assert all(v <= 1.0 for v in WORST.values())
