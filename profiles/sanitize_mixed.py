"""One launch of every 16-bit-operand (`Mixed<Op>`) kernel route, with exactly sized buffers, for compute-sanitizer:

    PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool memcheck python profiles/sanitize_mixed.py

Without the caching allocator every tensor is its own cudaMalloc, and every 16-bit operand here is sized to a multiple
of the allocator's 512-byte granule, so the allocation ends exactly where the operand does and memcheck sees a read
past it.  Routes: the fast row-wise kernel (d % 4 == 0, 16-byte and 8-byte aligned 16-bit operands, the 8-byte one
placed at the very end of its allocation), the generic row-wise kernel (d % 4 != 0), scalar noise, the per-thread-load
tile kernel (m = 16), the generic tile kernel (m = 5) and a batch-broadcast g; counter and memory noise; bfloat16 and
float16.  Every result is compared with the float32 launch on widened copies, so a clean but wrong kernel still fails.
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from torchsde_b200 import _cabi  # noqa: E402

dev = torch.device('cuda')
lib = _cabi.lib()
DT = 2.0 ** -6
key = torch.tensor([7], dtype=torch.int64, device=dev)
# name -> (scalars, noise, outputs ('y' state-shaped, 'g' g-shaped), row-wise only)
ENTRIES = {
    'tsde_step_euler': ((DT,), 'w', 'y', False),
    'tsde_milstein_vjp_seed': ((DT, 1), 'w', 'g', True),
    'tsde_step_milstein': ((DT,), 'w', 'y', True),
    'tsde_milstein_gf_predict': ((DT, DT ** 0.5, 1), None, 'y', True),
    'tsde_step_milstein_gf': ((DT, 2 * DT ** 0.5, 1), 'w', 'y', True),
    'tsde_step_heun': ((DT,), 'w', 'y', False),
    'tsde_midpoint_predict': ((DT / 2,), 'w', 'y', False),
    'tsde_euler_heun_predict': ((), 'w', 'y', False),
    'tsde_step_euler_heun': ((DT,), 'w', 'y', False),
    'tsde_reversible_heun_z': ((DT,), 'w', 'y', False),
    'tsde_step_reversible_heun': ((DT / 2,), 'w', 'y', False),
    'tsde_srk_diag_stage1': ((DT, DT ** 0.5), None, 'yy', True),
    'tsde_srk_diag_stage2': ((DT, 1 / DT, DT ** 0.5), 'wu', 'yy', True),
    'tsde_srk_diag_stage3': ((DT, DT ** 0.5), None, 'y', True),
    'tsde_step_srk_diag': ((DT, 1 / DT, DT ** 0.5, 3 * DT), 'wu', 'y', True),
    'tsde_srk_additive_stage': ((DT, 1 / DT), 'wu', 'y', False),
    'tsde_step_srk_additive': ((DT, 1 / DT), 'wu', 'y', False),
    'tsde_adjoint_reversible_heun_a': ((DT, DT / 2), 'w', 'yyg', False),
    'tsde_adjoint_reversible_heun_b': ((DT, DT / 2), 'w', 'yyyyg', False),
}
GENERAL_ONLY = ('tsde_srk_additive_stage', 'tsde_step_srk_additive')
# (route, noise layout, rows, d, m, 16-bit operand placed 8 bytes into its allocation); every 16-bit operand is a
# multiple of 512 bytes (the 8-byte-offset one: together with its 4 leading elements)
ROUTES = [('fast', 'diag', 256, 64, 64, False), ('fast, 8-byte aligned', 'diag', 63, 4, 4, True),
          ('generic', 'diag', 256, 6, 6, False), ('scalar', 'general', 256, 8, 1, False),
          ('cta', 'general', 64, 8, 16, False), ('generic tile', 'general', 256, 6, 5, False),
          ('broadcast g', 'general', 64, 16, 16, False)]


def exact16(shape, x, dtype, offset):
    """`x` in 16 bits in an allocation of exactly its size (plus `offset` leading elements)."""
    n = x.numel()
    buf = torch.empty(n + offset, dtype=dtype, device=dev)
    view = buf[offset:].view(shape)
    view.copy_(x.to(dtype))
    return view


def run(name, half, src, route):
    label, noise, rows, d, m, offset8 = route
    scalars, want, outs, _ = ENTRIES[name]
    bcast = label == 'broadcast g'
    gshape = (d, m) if bcast else ((rows, d) if noise == 'diag' or m == 1 else (rows, d, m))
    gen = torch.Generator(device=dev).manual_seed(rows + d + m)
    fmt = _cabi.FMT_BF16 if half == torch.bfloat16 else _cabi.FMT_F16
    ins16, ins32, word = [], [], _cabi.F32
    for i, arg in enumerate(_cabi.INPUTS[name]):
        is_g = (arg.startswith('g') and arg != 'gdg') or arg == 'adj_g0'
        shape = gshape if is_g else (rows, d)
        x = torch.randn(shape, generator=gen, device=dev)
        if arg in _cabi.SDE_OUTPUT_NAMES:
            x16 = exact16(shape, x, half, 4 if offset8 else 0)
            ins16.append(x16)
            ins32.append(x16.float())
            word |= fmt << (8 + 2 * i)
        else:
            ins16.append(x)
            ins32.append(x)
    w = torch.randn(rows, m, generator=gen, device=dev) * DT ** 0.5
    u = torch.randn(rows, m, generator=gen, device=dev) * DT
    nz = _cabi.Noise()
    if src == 'counter':
        nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, key.data_ptr(), 3, 1, DT, DT
    else:
        nz.source, nz.n_cells, nz.w = _cabi.SRC_MEMORY, 1, w.data_ptr()
        nz.u = u.data_ptr() if want == 'wu' else None
    nz.want_u = int(want == 'wu')
    nz.flags = _cabi.FLAG_G_BROADCAST if bcast else 0
    res = []
    for ins, wd in ((ins16, word), (ins32, _cabi.F32)):
        o = []
        for kind in outs:
            shape = (rows, d, m) if kind == 'g' and noise == 'general' and m > 1 else (rows, d)
            if name == 'tsde_milstein_vjp_seed' and wd != _cabi.F32:
                o.append(torch.empty(shape, dtype=half, device=dev))
            else:
                o.append(torch.empty(shape, device=dev))
        L = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL if noise == 'diag' else _cabi.NOISE_GENERAL,
                              rows, d, m)
        L.dtype = wd
        args = [ctypes.byref(L)] + ([ctypes.byref(nz)] if want else [])
        _cabi.check(getattr(lib, name)(*args, *[t.data_ptr() for t in ins], *scalars, *[t.data_ptr() for t in o]),
                    name)
        res.append(o)
    for a, b in zip(*res):
        assert torch.equal(a, b.to(a.dtype)), (name, half, src, label)


checked = 0
for name, (_, want, _, rowwise_only) in ENTRIES.items():
    for route in ROUTES:
        general_route = route[1] == 'general' and route[4] > 1
        if (rowwise_only and general_route) or (name in GENERAL_ONLY and not general_route):
            continue
        if route[0] == 'broadcast g' and 'reversible_heun' in name:
            continue  # (the reversible-Heun family keeps its g operands dense)
        for half in (torch.bfloat16, torch.float16):
            for src in (('counter', 'memory') if want else ('counter',)):
                run(name, half, src, route)
                checked += 1
torch.cuda.synchronize()
print('sanitize_mixed ok,', checked, 'checked launch pairs')
