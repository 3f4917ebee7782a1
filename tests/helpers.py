"""Shared helpers of the parity tests."""
import collections
import ctypes
import glob
import os

import numpy as np
import torch

from . import problems

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


# ---- the general-noise entry points, called through the C ABI ------------------------------------------------------
GEN_DT = 2.0 ** -6
# args / outs: the operands / outputs in argument order, 'e' for a (rows, d) tensor and 'g' for a (rows, d, m) one;
# tile_g: g operands of the (rows, d, m) tile kernel the entry point launches (the adjoint halves also launch
# element-wise and outer-product kernels)
GeneralOp = collections.namedtuple('GeneralOp', 'args scalars want_u outs tile_g')
GENERAL_OPS = {
    'tsde_step_euler': GeneralOp('eeg', (GEN_DT,), False, 'e', 1),
    'tsde_midpoint_predict': GeneralOp('eeg', (GEN_DT / 2,), False, 'e', 1),
    'tsde_euler_heun_predict': GeneralOp('eg', (), False, 'e', 1),
    'tsde_reversible_heun_z': GeneralOp('eeeg', (GEN_DT,), False, 'e', 1),
    'tsde_srk_additive_stage': GeneralOp('eeg', (GEN_DT, 1 / GEN_DT), True, 'e', 1),
    'tsde_adjoint_reversible_heun_a': GeneralOp('eeegeeg', (GEN_DT, GEN_DT / 2), False, 'eeg', 1),
    'tsde_step_heun': GeneralOp('eeegg', (GEN_DT,), False, 'e', 2),
    'tsde_step_euler_heun': GeneralOp('eegg', (GEN_DT,), False, 'e', 2),
    'tsde_step_reversible_heun': GeneralOp('eeegg', (GEN_DT / 2,), False, 'e', 2),
    'tsde_step_srk_additive': GeneralOp('eeegg', (GEN_DT, 1 / GEN_DT), True, 'e', 2),
    'tsde_adjoint_reversible_heun_b': GeneralOp('eeeggeee', (GEN_DT, GEN_DT / 2), False, 'eeeeg', 2),
}
# every (op, m) the TMA-staged tile kernel is compiled for: one tile g operand at m = 16 and 64, two at m = 64
GENERAL_TMA_REACHABLE = [(op, m) for op, spec in GENERAL_OPS.items() for m in ((16, 64) if spec.tile_g == 1 else (64,))]
# the entry points that accept TSDE_FLAG_G_BROADCAST (the reversible-Heun family keeps its g operands dense)
GENERAL_BROADCAST_OPS = [op for op in GENERAL_OPS if 'reversible_heun' not in op]
# the entry points cabi.cu routes to the row-wise kernels at m = 1 (the SRK-additive pair keeps the tile kernels)
GENERAL_ROWWISE_OPS = [op for op in GENERAL_OPS if 'srk_additive' not in op]
GEN_CTA, GEN_TMA = 0, 1  # tsde_kernel_launches families


def tile_launches():
    """(per-thread-load, TMA-staged) general-noise tile kernel launches this process has issued so far."""
    from torchsde_b200 import _cabi
    lib = _cabi.lib()
    return lib.tsde_kernel_launches(GEN_CTA), lib.tsde_kernel_launches(GEN_TMA)


def general_noise(key=None, cell_id=0, h=GEN_DT, cell_h=None, h_total=None, row_offset=0, w=None, u=None,
                  want_u=False, flags=0):
    """tsde_noise of a general-noise launch: counter noise of `key` (device int64 tensor) over one cell of length h,
    or over the cells whose lengths the device float64 tensor `cell_h` holds; without a key, memory noise read
    from the device addresses w (and u)."""
    from torchsde_b200 import _cabi
    nz = _cabi.Noise()
    nz.want_u, nz.flags = int(want_u), flags
    if key is not None:
        nz.source, nz.key, nz.cell_id, nz.row_offset = _cabi.SRC_COUNTER, key.data_ptr(), cell_id, row_offset
        nz.n_cells, nz.h, nz.h_total = 1, h, h if h_total is None else h_total
        if cell_h is not None:
            nz.n_cells, nz.cell_h = cell_h.numel(), cell_h.data_ptr()
    else:
        nz.source, nz.n_cells, nz.w, nz.u = _cabi.SRC_MEMORY, 1, w, u if want_u else None
    return nz


def general_call(op, dtype, rows, d, m, args, nz, outs):
    """One launch of general-noise entry point `op`; args / outs are device addresses in argument order."""
    from torchsde_b200 import _cabi
    L = _cabi.make_launch(dtype, _cabi.NOISE_GENERAL, rows, d, m)
    _cabi.check(getattr(_cabi.lib(), op)(ctypes.byref(L), ctypes.byref(nz), *args, *GENERAL_OPS[op].scalars, *outs),
                op)


def golden_files(prefix):
    return sorted(glob.glob(os.path.join(GOLDEN, prefix + '*.npz')))


def load(path):
    z = np.load(path, allow_pickle=False)
    return {k: z[k] for k in z.files}


def case_id(path):
    return os.path.basename(path)[:-4]


def build_problem(case, dtype=None, device='cpu'):
    tdt = {'f64': torch.float64, 'f32': torch.float32}[str(case['dtype'])] if dtype is None else dtype
    sde = problems.make(str(case['kind']), int(case['d']), int(case['m']), str(case['sde_type']), dtype=tdt,
                        seed=int(case['seed']))
    return sde.to(device)


def replay_numpy(case):
    levy = 'space-time' if 'U' in case else 'none'
    return problems.ReplayBM(case['ta'], case['tb'], case['W'], case.get('U'), levy=levy)


def replay_torch(case, device):
    levy = 'space-time' if 'U' in case else 'none'
    Ws = [torch.from_numpy(w).to(device) for w in case['W']]
    Us = [torch.from_numpy(u).to(device) for u in case['U']] if 'U' in case else None
    bm = problems.ReplayBM(case['ta'], case['tb'], Ws, Us, levy=levy)
    bm.dtype = Ws[0].dtype
    bm.device = Ws[0].device
    return bm


def tol_for(dtype_str, diag):
    """Tolerances of the parity tests (stated per BASELINE north_star: <= 1e-5 rel in fp32).
    Diagonal/scalar noise follows the reference's op order exactly -> far tighter in practice."""
    if dtype_str == 'f64':
        return dict(rtol=1e-12, atol=1e-13)
    return dict(rtol=1e-5, atol=1e-6)


# ---- oracle view of a grid-bound torchsde_b200.BrownianInterval on a SAMPLE of rows ------------------
MASK64 = (1 << 64) - 1


def sample_rows(n_rows, n_sample, seed):
    """Sorted random sample of global row indices that always contains the first and the last row."""
    rng = np.random.default_rng(seed)
    n_sample = min(n_sample, n_rows)
    rows = set(rng.choice(n_rows, size=n_sample, replace=False).tolist()) | {0, n_rows - 1}
    return np.array(sorted(rows), dtype=np.int64)


def oracle_grid_bm(bm, row_ids, m, npdt, have_h):
    """numpy `bm(ta, tb, return_U=False)` reproducing — for the global rows `row_ids` only — the path of a
    BrownianInterval whose root is a GRID node (what a fixed-step solve binds): every query must be a run of
    whole primary cells.  Rows are independent Philox streams (oracle/philox.py), so a full-size solve can be
    checked on a sample of its trajectories."""
    from oracle import brownian as obm
    grid, key = bm._root, bm._key
    assert grid.kind == 2, "the Brownian motion is not grid-bound"
    index = {b: i for i, b in enumerate(grid.bounds)}
    row_ids = np.asarray(row_ids, dtype=np.int64) + int(bm._row_offset)

    def query(ta, tb, return_U=False):
        i, j = index[float(ta)], index[float(tb)]
        lengths = [grid.bounds[k + 1] - grid.bounds[k] for k in range(i, j)]
        W, H = obm.cells(key, (grid.cell_base + i) & MASK64, lengths, len(row_ids), m, npdt, have_h,
                         row_ids=row_ids)
        if return_U:
            return W, obm.h_to_u(W, H, float(tb) - float(ta))
        return W
    return query


def rel_err(got, ref, floor=1e-6):
    """max |got - ref| / max(|ref|, floor) over all elements."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), floor)))
