"""CUDA-event probe of gen_kernel, the generic general-noise tile kernel (shapes no other tile kernel takes).

    python profiles/gen_kernel_probe.py [--out FILE]

Launches are captured into a CUDA graph and replayed on rotating buffer sets whose total is larger than the 50 MB L2
(cold buffers, as profiles/wide_noise_probe.py does).  Shapes:
  * Euler, fp32, counter noise, B = 1024, d = 16, m = 10240 (gen_kernel's widest staged row)
  * Euler, fp64, memory noise, B = 65536, d = 16, m = 12 (m / 4 not a power of two)
Prints per shape: microseconds per launch (median, min and max of 9 replays), and a CRC of the first buffer set's
output, so that two builds of the library can be compared bit for bit (TORCHSDE_B200_LIB selects the build).  The
launch counters confirm that no other tile kernel ran.  The GPU's name, power limit and clocks go first.
"""
import argparse
import ctypes
import os
import subprocess
import sys
import zlib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torchsde_b200 import _cabi  # noqa: E402

COLD_BYTES = 256 << 20  # buffer sets per shape: at least this many bytes in all
DT = 2.0 ** -6
dev = torch.device('cuda')
lib = _cabi.lib()
key = torch.tensor([987654321], dtype=torch.int64, device=dev)

# name: (dtype, B, d, m, memory noise)
SHAPES = {
    'euler fp32 counter B=1024 d=16 m=10240': (torch.float32, 1024, 16, 10240, False),
    'euler fp64 memory B=65536 d=16 m=12': (torch.float64, 65536, 16, 12, True),
}


def probe(dtype, B, d, m, memory):
    s = torch.finfo(dtype).bits // 8
    set_bytes = (B * d * m + 3 * B * d + (B * m if memory else 0)) * s
    nset = max(2, -(-COLD_BYTES // set_bytes))
    gen = torch.Generator(device=dev).manual_seed(20261016)

    def rand(*shape):
        return torch.rand(shape, device=dev, dtype=dtype, generator=gen) - 0.5
    sets = []
    for _ in range(nset):
        nz = _cabi.Noise()
        nz.want_u, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total, nz.flags = 0, key.data_ptr(), 7, 1, DT, DT, 0
        w = rand(B, m) * DT ** 0.5 if memory else None
        nz.source = _cabi.SRC_MEMORY if memory else _cabi.SRC_COUNTER
        nz.w = w.data_ptr() if memory else None
        sets.append((nz, w, rand(B, d), rand(B, d), rand(B, d, m), torch.empty(B, d, device=dev, dtype=dtype)))
    L = _cabi.make_launch(dtype, _cabi.NOISE_GENERAL, B, d, m)

    def launch(st):
        nz, _, y0, f, g, o = st
        _cabi.check(lib.tsde_step_euler(ctypes.byref(L), ctypes.byref(nz), y0.data_ptr(), f.data_ptr(), g.data_ptr(),
                                        DT, o.data_ptr()), 'tsde_step_euler')

    before = [lib.tsde_kernel_launches(k) for k in range(3)]  # CTA, TMA, wide tile kernels
    for st in sets:
        launch(st)
    torch.cuda.synchronize()
    assert [lib.tsde_kernel_launches(k) for k in range(3)] == before, 'a shape left gen_kernel'
    crc = zlib.crc32(sets[0][5].cpu().numpy().tobytes())
    reps = max(nset, 12)
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
    del graph, sets
    torch.cuda.empty_cache()
    return float(np.median(times)), min(times), max(times), crc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the report to this file')
    args = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True)
    lines = [f'gpu: {smi.stdout.strip() or "(nvidia-smi unavailable)"}', f'lib = {_cabi.LIB_PATH}']
    for name, shape in SHAPES.items():
        us, lo, hi, crc = probe(*shape)
        lines.append(f'{name:42s} gen_kernel {us:9.1f} us (min {lo:.1f}, max {hi:.1f})  out crc {crc:08x}')
        print(lines[-1], flush=True)
    print(lines[0])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
