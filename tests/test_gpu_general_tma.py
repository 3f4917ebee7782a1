"""The TMA-staged general-noise tile kernel (`gen_tma_kernel`) against the per-thread-load tile kernel (`gen_cta_kernel`).

Both kernels use the same chunk -> lane mapping, the same fused multiply-add chain inside a 4-chunk and the same
xor-tree across chunks, so for identical increments their outputs must be BIT-IDENTICAL; both kernels are pinned
against the oracle / the reference's golden files in test_gpu_solver.py and, launch by launch, against a float64
formula on the oracle's increments in test_gpu_general_paths.py.

Which kernel runs is decided by shape alone (csrc/tableau_general.cu `tma_route` and the eligibility checks of
`launch_gen_tma`): a batch that fills the pipeline at m = 64, or at m = 16 for tableaus with one g operand, takes the
TMA-staged kernel; a small batch takes the per-thread-load kernel.  Rows are independent Philox streams, so each test
launches a batch that takes the TMA-staged kernel, then the same rows again as slices small enough for the
per-thread-load kernel (counter noise: `row_offset`; memory noise: offset pointers), confirms both routes with the
launch counters and compares the outputs bit for bit.
"""
import pytest
import torch

from . import helpers, problems
from .helpers import GENERAL_OPS, GENERAL_TMA_REACHABLE as REACHABLE, tile_launches as _launches

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SLICE = 512        # rows per per-thread-load slice: too few tiles to fill the TMA pipeline at every tested shape


def _call(op, dtype, rows, d, m, r0, args, w, u, key, outs):
    """One launch of `op` on rows [r0, r0 + rows) of the operands and outputs."""
    spec = GENERAL_OPS[op]
    s = torch.finfo(dtype).bits // 8
    if key is not None:
        nz = helpers.general_noise(key=key, cell_id=5, row_offset=r0, want_u=spec.want_u)
    else:
        nz = helpers.general_noise(w=w.data_ptr() + r0 * m * s, u=u.data_ptr() + r0 * m * s, want_u=spec.want_u)
    per_row = {'e': d * s, 'g': d * m * s}
    helpers.general_call(op, dtype, rows, d, m, [x.data_ptr() + r0 * per_row[k] for k, x in zip(spec.args, args)],
                         nz, [o.data_ptr() + r0 * per_row[k] for k, o in zip(spec.outs, outs)])


def _whole_and_sliced(op, dtype, B, d, m, memory, first_slice=SLICE):
    """The launch over all B rows and the same rows launched as slices (the first `first_slice` rows, then SLICE rows
    at a time); returns both lists of outputs and the (per-thread-load, TMA-staged) launch counts of each."""
    spec = GENERAL_OPS[op]
    gen = torch.Generator(device=DEV).manual_seed(B * d + m)
    shape = {'e': (B, d), 'g': (B, d, m)}
    args = [torch.rand(*shape[k], generator=gen, device=DEV, dtype=dtype) - (0.5 if k == 'g' else 0.0)
            for k in spec.args]
    w = u = key = None
    if memory:
        w, u = (torch.randn(B, m, generator=gen, device=DEV, dtype=dtype) * helpers.GEN_DT ** 0.5 for _ in range(2))
    else:
        key = torch.tensor([31], dtype=torch.int64, device=DEV)
    whole, sliced = ([torch.full(shape[k], float('nan'), device=DEV, dtype=dtype) for k in spec.outs]
                     for _ in range(2))
    n0 = _launches()
    _call(op, dtype, B, d, m, 0, args, w, u, key, whole)
    n1 = _launches()
    r0 = 0
    while r0 < B:
        rows = min(first_slice if r0 == 0 else SLICE, B - r0)
        _call(op, dtype, rows, d, m, r0, args, w, u, key, sliced)
        r0 += rows
    n2 = _launches()
    return whole, sliced, (n1[0] - n0[0], n1[1] - n0[1]), (n2[0] - n1[0], n2[1] - n1[1])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('memory', [False, True], ids=['counter', 'memory'])
@pytest.mark.parametrize('op,m', REACHABLE, ids=[f'{op[5:]}-m{m}' for op, m in REACHABLE])
def test_tma_path_bit_identical(op, m, memory, dtype):
    """Every (op, m) the TMA-staged kernel is built for, with a ragged last tile (odd B), against the per-thread-load
    kernel on the same rows.  The first slice is 3 rows: fewer tiles than stages, which the per-thread-load kernel
    takes."""
    B = 65539 if m == 16 else 16387
    whole, sliced, route, slice_route = _whole_and_sliced(op, dtype, B, 32, m, memory, first_slice=3)
    assert route == (0, 1), f"B={B} was not routed to the TMA-staged kernel: {route}"
    n_slices = 1 + -(-(B - 3) // SLICE)
    assert slice_route == (n_slices, 0), f"slices were not routed to the per-thread-load kernel: {slice_route}"
    for i, (a, b) in enumerate(zip(whole, sliced)):
        assert torch.isfinite(a).all(), f"output {i} not written everywhere"
        assert torch.equal(a, b), f"output {i}: max abs diff {(a - b).abs().max().item()}"


ROUTES = [
    # entry point, dtype, B, d, m, takes the TMA-staged kernel
    ('tsde_step_euler', torch.float32, 65536, 32, 64, True),
    ('tsde_step_euler', torch.float32, 256, 32, 64, False),       # too few tiles to fill the pipeline
    ('tsde_step_euler', torch.float32, 3, 4, 64, False),          # fewer tiles than stages
    ('tsde_step_euler', torch.float32, 65536, 32, 16, True),
    ('tsde_step_euler', torch.float32, 256, 32, 16, False),
    ('tsde_step_euler', torch.float32, 65536, 32, 8, False),      # m = 8 and 32: per-thread loads at every size
    ('tsde_midpoint_predict', torch.float32, 65536, 16, 32, False),
    ('tsde_step_heun', torch.float32, 65536, 32, 16, False),      # two g operands at m = 16
    ('tsde_step_euler_heun', torch.float64, 32768, 16, 16, False),
    ('tsde_step_euler', torch.float32, 2100, 128, 64, True),      # one 32 KiB g row per stage
    ('tsde_step_euler', torch.float64, 2100, 128, 64, False),     # a 64 KiB row exceeds a stage
]


def test_default_routing():
    """The route of each shape, and its output equal to the per-thread-load kernel's on slices of the same rows."""
    bad = []
    for op, dtype, B, d, m, tma in ROUTES:
        whole, sliced, route, slice_route = _whole_and_sliced(op, dtype, B, d, m, memory=False)
        if route != ((0, 1) if tma else (1, 0)) or slice_route[1] != 0 or slice_route[0] < 1:
            bad.append(f'{op} {dtype} B={B} d={d} m={m}: routes {route}, slices {slice_route}')
        elif not all(torch.equal(a, b) for a, b in zip(whole, sliced)):
            bad.append(f'{op} {dtype} B={B} d={d} m={m}: output differs from the per-thread-load slices')
    assert not bad, '; '.join(bad)


def test_tma_path_in_cuda_graph():
    """A graph-captured Heun solve at m = 64 (both tableaus on the TMA-staged kernel) equals the same solve split with
    `shard_rows` into slices that take the per-thread-load kernel, bit for bit."""
    import torchsde_b200 as tsde
    B, d, m = 8192, 32, 64
    sde = problems.make('general', d, m, 'stratonovich', dtype=torch.float32, seed=11).to(DEV)
    y0 = torch.full((B, d), 0.25, device=DEV)
    ts = torch.tensor([0.0, 0.125, 0.25], device=DEV)

    def solve(rows, r0, graph):
        bm = tsde.BrownianInterval(0.0, 0.25, size=(rows, m), dtype=torch.float32, device=DEV, entropy=99)
        bm.shard_rows(r0)
        with torch.no_grad():
            return tsde.sdeint(sde, y0[r0:r0 + rows].contiguous(), ts, bm=bm, method='heun', dt=2.0 ** -5,
                               options={'cuda_graph': True} if graph else None).clone()

    n0 = _launches()
    whole = solve(B, 0, graph=True)
    n1 = _launches()
    parts = [solve(min(SLICE, B - r0), r0, graph=False) for r0 in range(0, B, SLICE)]
    n2 = _launches()
    assert n1[1] > n0[1], "the captured solve did not take the TMA-staged kernel"
    assert n2[1] == n1[1] and n2[0] > n1[0], "the sliced solves did not take the per-thread-load kernel"
    assert torch.equal(whole, torch.cat(parts, dim=1))
