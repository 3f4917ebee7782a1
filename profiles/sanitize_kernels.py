"""Small launches of the kernels with shared-memory / mbarrier synchronisation, for compute-sanitizer:

    compute-sanitizer --tool racecheck  python profiles/sanitize_kernels.py
    compute-sanitizer --tool synccheck  python profiles/sanitize_kernels.py
    compute-sanitizer --tool memcheck   python profiles/sanitize_kernels.py

Covers the warp-specialised TMA-staged tile kernel (producer warp + two-phase consumers on an mbarrier ring, taken by
the one batch per dtype that fills its pipeline at m = 64), the per-thread-load tile kernel (the small batches), the
Levy tile kernel (warp-private shared tiles), the fused cell-Levy query, bmm_ga (shared A tiles) and the row-wise
kernels; results are compared with torch so that a sanitizer-clean but wrong kernel would still fail, and the launch
counters confirm that both tile kernels ran.
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402

dev = torch.device('cuda')
lib = _cabi.lib()
key = torch.tensor([42], dtype=torch.int64, device=dev)
dt = 2.0 ** -6


def noise(w=None, u=None):
    nz = _cabi.Noise()
    if w is None:
        nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, key.data_ptr(), 3, 1, dt, dt
    else:
        nz.source, nz.w, nz.n_cells = _cabi.SRC_MEMORY, w.data_ptr(), 1
        if u is not None:
            nz.u, nz.want_u = u.data_ptr(), 1
    return nz


checked = 0
for dtype in (torch.float32, torch.float64):
    launches = [lib.tsde_kernel_launches(k) for k in (0, 1)]  # per-thread-load, TMA-staged tile kernel
    # small batches: per-thread-load tile kernel; 8195 x 32 x 64 fills the TMA pipeline (ragged last tile)
    for (B, D, M) in ((1024, 32, 16), (777, 16, 64), (512, 8, 8), (300, 4, 32), (8195, 32, 64)):
        y, f, f1 = (torch.randn(B, D, dtype=dtype, device=dev) for _ in range(3))
        g, g1 = (torch.randn(B, D, M, dtype=dtype, device=dev) for _ in range(2))
        w, u = torch.randn(B, M, dtype=dtype, device=dev), torch.randn(B, M, dtype=dtype, device=dev)
        o = torch.empty(B, D, dtype=dtype, device=dev)
        L = _cabi.make_launch(dtype, _cabi.NOISE_GENERAL, B, D, M)
        nz = noise(w)
        _cabi.check(lib.tsde_step_euler(ctypes.byref(L), ctypes.byref(nz), y.data_ptr(), f.data_ptr(), g.data_ptr(), dt,
                                        o.data_ptr()), 'euler')
        ref = y + f * dt + torch.bmm(g, w.unsqueeze(-1)).squeeze(-1)
        torch.testing.assert_close(o, ref, rtol=1e-4 if dtype == torch.float32 else 1e-11, atol=1e-4 if dtype == torch.float32 else 1e-11)
        _cabi.check(lib.tsde_step_heun(ctypes.byref(L), ctypes.byref(nz), y.data_ptr(), f.data_ptr(), f1.data_ptr(),
                                       g.data_ptr(), g1.data_ptr(), dt, o.data_ptr()), 'heun')
        ref = y + (dt * (f + f1) + torch.bmm(g, w.unsqueeze(-1)).squeeze(-1) + torch.bmm(g1, w.unsqueeze(-1)).squeeze(-1)) * 0.5
        torch.testing.assert_close(o, ref, rtol=1e-4 if dtype == torch.float32 else 1e-11, atol=1e-4 if dtype == torch.float32 else 1e-11)
        nzu = noise(w, u)
        _cabi.check(lib.tsde_step_srk_additive(ctypes.byref(L), ctypes.byref(nzu), y.data_ptr(), f.data_ptr(),
                                               f1.data_ptr(), g.data_ptr(), g1.data_ptr(), dt, 1 / dt, o.data_ptr()),
                    'srk_additive')
        nzc = noise()  # counter source: the producer warp also draws the tile's increments
        _cabi.check(lib.tsde_step_euler(ctypes.byref(L), ctypes.byref(nzc), y.data_ptr(), f.data_ptr(), g.data_ptr(),
                                        dt, o.data_ptr()), 'euler counter')
        checked += 4
        # bmm_ga
        if M <= 32:
            a = torch.randn(B, M, M, dtype=dtype, device=dev)
            out = torch.empty(M, B, D, dtype=dtype, device=dev)
            _cabi.check(lib.tsde_bmm_ga(ctypes.byref(L), g.data_ptr(), a.data_ptr(), out.data_ptr()), 'bmm_ga')
            torch.testing.assert_close(out, torch.bmm(g, a).permute(2, 0, 1), rtol=1e-4 if dtype == torch.float32 else 1e-11,
                                       atol=1e-4 if dtype == torch.float32 else 1e-11)
            checked += 1
    ran = [lib.tsde_kernel_launches(k) - n for k, n in zip((0, 1), launches)]
    assert ran[0] > 0 and ran[1] > 0, f"{dtype}: tile kernel launches (per-thread-load, TMA-staged) = {ran}"
    # Levy tiles (separate and fused) + bridge + row-wise kernels through the public API
    for levy in ('davie', 'foster'):
        bm = tsde.BrownianInterval(0.0, 1.0, size=(513, 8), dtype=dtype, device=dev, entropy=5, dt=0.25,
                                   levy_area_approximation=levy)
        W, U, A = bm(0.25, 0.5, return_U=True, return_A=True)          # fused cell query
        W2, U2, A2 = bm(0.1, 0.9, return_U=True, return_A=True)        # bridge + merges + separate Levy kernel
        assert torch.equal(A, -A.transpose(1, 2)) and bool(torch.isfinite(A2).all())
        checked += 2
torch.cuda.synchronize()
print('sanitize_kernels ok,', checked, 'checked launches')
