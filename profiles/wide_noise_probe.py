"""CUDA-event probe of the general-noise tile kernels at Brownian widths past gen_kernel's shared-memory staging.

    python profiles/wide_noise_probe.py [--out FILE]

Launches are captured into a CUDA graph and replayed on rotating buffer sets whose total is larger than the 50 MB L2
(cold buffers, as profiles/kernel_probe.py times the row-wise kernels).  Shapes (counter noise, one cell):
  * Euler, dense g, fp32, B = 1024, d = 16, m = 16384                     (gen_wide_kernel)
  * SRK-additive final step, batch-broadcast g, fp64, B = 8192, d = 64, m = 4096   (gen_wide_kernel)
  * Euler, fp32, B = 1024, d = 16, m = 10240 (gen_kernel, its widest row) and m = 10244 (gen_wide_kernel)
Prints per shape: the route (launch counters), microseconds per launch, the algorithmic bytes (every g operand read
once: d * m * s per row, or once in all for a broadcast g; the element-wise operands and outputs d * s per row) and
their share of the H100 SXM data-sheet HBM bandwidth, 3.35 TB/s.  The GPU's name, power limit and clocks go first.
"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torchsde_b200 import _cabi  # noqa: E402

PEAK = 3350.0  # GB/s, H100 SXM data sheet (HBM3)
COLD_BYTES = 256 << 20  # buffer sets per shape: at least this many bytes in all, so no launch finds its operands in L2
DT = 2.0 ** -6
dev = torch.device('cuda')
lib = _cabi.lib()
key = torch.tensor([987654321], dtype=torch.int64, device=dev)
ROUTES = ['gen_cta_kernel', 'gen_tma_kernel', 'gen_wide_kernel']


def noise(want_u, bcast):
    nz = _cabi.Noise()
    nz.source, nz.want_u, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = \
        _cabi.SRC_COUNTER, int(want_u), key.data_ptr(), 7, 1, DT, DT
    nz.flags = _cabi.FLAG_G_BROADCAST if bcast else 0
    return nz


# name: (entry point, dtype, B, d, m, element-wise inputs, g operands, scalars, broadcast g, U)
SHAPES = {
    'euler fp32 dense g m=16384': ('tsde_step_euler', torch.float32, 1024, 16, 16384, 2, 1, (DT,), False, False),
    'srk-additive final fp64 bcast g m=4096': ('tsde_step_srk_additive', torch.float64, 8192, 64, 4096, 3, 2,
                                               (DT, 1 / DT), True, True),
    'euler fp32 m=10240 (widest staged row)': ('tsde_step_euler', torch.float32, 1024, 16, 10240, 2, 1, (DT,), False,
                                               False),
    'euler fp32 m=10244': ('tsde_step_euler', torch.float32, 1024, 16, 10244, 2, 1, (DT,), False, False),
}


def probe(entry, dtype, B, d, m, ne, ng, scalars, bcast, want_u):
    s = torch.finfo(dtype).bits // 8
    gshape = (d, m) if bcast else (B, d, m)
    g_bytes = ng * d * m * s * (1 if bcast else B)
    set_bytes = g_bytes + (ne + 1) * B * d * s
    nset = max(2, -(-COLD_BYTES // set_bytes))
    sets = [([torch.rand(B, d, device=dev, dtype=dtype) for _ in range(ne)],
             [torch.rand(gshape, device=dev, dtype=dtype) - 0.5 for _ in range(ng)],
             torch.empty(B, d, device=dev, dtype=dtype)) for _ in range(nset)]
    nz = noise(want_u, bcast)
    L = _cabi.make_launch(dtype, _cabi.NOISE_GENERAL, B, d, m)
    fn = getattr(lib, entry)

    def launch(st):
        e, g, o = st
        _cabi.check(fn(ctypes.byref(L), ctypes.byref(nz), *(x.data_ptr() for x in e + g), *scalars, o.data_ptr()),
                    entry)

    before = [lib.tsde_kernel_launches(k) for k in range(3)]
    for st in sets:
        launch(st)
    torch.cuda.synchronize()
    route = [r for k, r in enumerate(ROUTES) if lib.tsde_kernel_launches(k) > before[k]] or ['gen_kernel']
    reps = max(nset, 12)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.stream = torch.cuda.current_stream(dev).cuda_stream
        for i in range(reps):
            launch(sets[i % nset])
    L.stream = torch.cuda.current_stream(dev).cuda_stream
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(9):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / reps)
    us = float(np.median(times))
    nbytes = g_bytes + (ne + 1) * B * d * s
    del graph, sets
    torch.cuda.empty_cache()
    return route[0], us, min(times), max(times), nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the report to this file')
    args = ap.parse_args()
    lines = []
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True)
    lines.append(f'gpu: {smi.stdout.strip() or "(nvidia-smi unavailable)"}')
    lines.append(f'lib = {_cabi.LIB_PATH}')
    for name, shape in SHAPES.items():
        route, us, lo, hi, nbytes = probe(*shape)
        gbs = nbytes / us / 1e3
        lines.append(f'{name:42s} {route:16s} {us:9.1f} us (min {lo:.1f}, max {hi:.1f})  {nbytes / 1e6:9.1f} MB  '
                     f'{gbs:7.1f} GB/s  {gbs / PEAK * 100:5.1f} % of {PEAK:.0f}')
        print(lines[-1], flush=True)
    lines.append('gpu after: ' + subprocess.run(
        ['nvidia-smi', '--query-gpu=clocks.sm,power.draw', '--format=csv,noheader'], capture_output=True,
        text=True).stdout.strip())
    print(lines[0])
    print(lines[-1])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
