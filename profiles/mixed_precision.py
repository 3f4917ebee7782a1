"""16-bit SDE outputs (torch.autocast) against float32 ones: kernel probe and cfg4 end to end, in one process.

    python profiles/mixed_precision.py > out/mixed_precision.txt

Kernel probe: the tableau kernels at the cfg2 (diagonal, 65536 x 64) and cfg3 (general, D = 32, M = 16) sizes, with
float32 operands and with 16-bit f / g, timed as the solver issues them (launches captured into a CUDA graph and
replayed) on rotating buffer sets larger than the 50 MB L2 ('cold': HBM traffic).  Bytes are computed from the shapes.
cfg3 runs at two batch sizes: 65536 rows, where float32 takes the TMA-staged tile kernel (16-bit g never does), and
4096 rows, where both take the per-thread-load tile kernel.

cfg4 end to end: the latent-SDE-like model (MLP drift, element-wise g), reversible Heun + its adjoint, B = 32768,
D = 128, T = 256 steps, forward + backward, in three variants alternated in this process: float32; autocast(bfloat16)
with the drift widened by `.float()` inside the SDE (what a user had to write before); autocast on the 16-bit path.
max |delta| of ys and of the parameter gradients of the last two must be 0.
"""
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402
from tests import problems  # noqa: E402

dev = torch.device('cuda')
lib = _cabi.lib()
PEAK = 3350.0  # GB/s, H100 SXM data sheet (HBM3)
dt = 2.0 ** -10
key = torch.tensor([987654321], dtype=torch.int64, device=dev)
BF = torch.bfloat16


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    return q or 'nvidia-smi unavailable'


def noise(flags=0):
    nz = _cabi.Noise()
    nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total, nz.flags = \
        _cabi.SRC_COUNTER, key.data_ptr(), 7, 1, dt, dt, flags
    return nz


def probe(name, launch, shapes, dtypes, out_shapes, rows):
    """Median microseconds per launch over rotating buffer sets, and the bytes one launch moves."""
    set_bytes = sum(int(np.prod(s)) * torch.tensor([], dtype=t).element_size() for s, t in zip(shapes, dtypes)) + \
        sum(int(np.prod(s)) * 4 for s in out_shapes)
    nset = max(2, int(np.ceil(160e6 / set_bytes)))  # > 3x the 50 MB L2
    reps = 2 * nset
    sets = [([torch.rand(s, device=dev).to(t) for s, t in zip(shapes, dtypes)],
             [torch.empty(s, device=dev) for s in out_shapes]) for _ in range(nset)]
    for s in sets:
        assert launch(*s) == 0, name
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(reps):
            launch(*sets[i % nset])
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
    return us, set_bytes


def kernel_probe():
    print('## kernel probe (cold: rotating buffer sets > L2)')
    P = lambda t: t.data_ptr()  # noqa: E731
    B, D = 65536, 64
    for half in (False, True):
        h = BF if half else torch.float32
        fmt = _cabi.FMT_BF16 if half else 0
        Ld = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL, B, D, D)
        nz = noise()

        def mil(ins, outs, Ld=Ld, fmt=fmt):
            Ld.dtype = _cabi.F32 | (fmt << 10) | (fmt << 12)  # f, g
            Ld.stream = torch.cuda.current_stream().cuda_stream
            return lib.tsde_step_milstein(ctypes.byref(Ld), ctypes.byref(nz), *map(P, ins), dt, P(outs[0]))

        def rh(ins, outs, Ld=Ld, fmt=fmt):
            Ld.dtype = _cabi.F32 | sum(fmt << (8 + 2 * i) for i in (1, 2, 3, 4))
            Ld.stream = torch.cuda.current_stream().cuda_stream
            return lib.tsde_step_reversible_heun(ctypes.byref(Ld), ctypes.byref(nz), *map(P, ins), dt / 2, P(outs[0]))

        def rh_cfg4(ins, outs, Ld=Ld, fmt=fmt):  # 16-bit f, float32 g
            Ld.dtype = _cabi.F32 | (fmt << 10) | (fmt << 12)
            Ld.stream = torch.cuda.current_stream().cuda_stream
            return lib.tsde_step_reversible_heun(ctypes.byref(Ld), ctypes.byref(nz), *map(P, ins), dt / 2, P(outs[0]))

        f32 = torch.float32
        for name, fn, dts in (('Milstein tableau (cfg2)', mil, (f32, h, h, f32)),
                              ('reversible-Heun step (cfg2)', rh, (f32, h, h, h, h)),
                              ('reversible-Heun step, 16-bit f only', rh_cfg4, (f32, h, h, f32, f32))):
            us, nb = probe(name, fn, [(B, D)] * len(dts), dts, [(B, D)], B)
            print(f"{name:40s} {'16-bit' if half else 'fp32  '}: {us:8.2f} us  {nb / B / D:4.0f} B/elt  "
                  f"{nb / us / 1e3:7.1f} GB/s = {nb / us / 1e3 / PEAK * 100:5.1f} % of {PEAK:.0f}")
    D, M = 32, 16
    for B in (65536, 4096):
        for half in (False, True):
            h = BF if half else torch.float32
            fmt = _cabi.FMT_BF16 if half else 0
            Lg = _cabi.make_launch(torch.float32, _cabi.NOISE_GENERAL, B, D, M)
            nz = noise()

            def eu(ins, outs, Lg=Lg, fmt=fmt):
                Lg.dtype = _cabi.F32 | (fmt << 10) | (fmt << 12)
                Lg.stream = torch.cuda.current_stream().cuda_stream
                return lib.tsde_step_euler(ctypes.byref(Lg), ctypes.byref(nz), *map(P, ins), dt, P(outs[0]))
            before = [lib.tsde_kernel_launches(k) for k in (0, 1)]
            us, nb = probe('euler general', eu, [(B, D), (B, D), (B, D, M)], (torch.float32, h, h), [(B, D)], B)
            route = ['per-thread-load', 'TMA-staged'][int(lib.tsde_kernel_launches(1) > before[1])]
            print(f"Euler general D=32 M=16 B={B:<6d} {route:16s} {'16-bit' if half else 'fp32  '}: {us:8.2f} us  "
                  f"{nb / B:5.0f} B/row  {nb / us / 1e3:7.1f} GB/s = {nb / us / 1e3 / PEAK * 100:5.1f} % of {PEAK:.0f}")


class Widened(torch.nn.Module):
    """cfg4's SDE with its outputs widened by `.float()`: what a user writes without 16-bit operand support."""
    noise_type, sde_type = 'diagonal', 'stratonovich'

    def __init__(self, base):
        super().__init__()
        self.base = base

    def f_and_g(self, t, y):
        f, g = self.base.f_and_g(t, y)
        return f.float(), g.float()


def cfg4():
    B, D, T = 32768, 128, 256
    sde = problems.LatentLike(D, hidden=128, seed=0).to(dev)
    ts = (torch.arange(T + 1, dtype=torch.float32) * dt).to(dev)
    y0 = torch.full((B, D), 0.1, device=dev)
    params = list(sde.parameters())

    def run(variant):
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, D), dtype=torch.float32, device=dev, entropy=3)
        model = Widened(sde) if variant == 'autocast, widened' else sde
        with torch.autocast('cuda', dtype=BF, enabled=variant != 'fp32'):
            ys = tsde.sdeint_adjoint(model, y0, ts, bm=bm, method='reversible_heun',
                                     adjoint_method='adjoint_reversible_heun', dt=dt, adjoint_params=params)
        grads = torch.autograd.grad(ys[-1].pow(2).sum(1).mean(), params)
        return ys.detach(), grads

    variants = ('fp32', 'autocast, widened', 'autocast, 16-bit operands')
    results = {v: run(v) for v in variants}  # warm-up (and the outputs compared below)
    times = {v: [] for v in variants}
    for _ in range(3):
        for v in variants:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1))
    print('## cfg4 end to end (forward + backward, B=32768 D=128 T=256)')
    for v in variants:
        print(f"{v:28s}: median {np.median(times[v]):8.1f} ms   runs {' '.join(f'{t:.1f}' for t in times[v])}")
    (ya, ga), (yb, gb) = results['autocast, widened'], results['autocast, 16-bit operands']
    dy = (ya - yb).abs().max().item()
    dg = max((a - b).abs().max().item() for a, b in zip(ga, gb))
    print(f"max |delta| vs 'autocast, widened': ys {dy}  parameter gradients {dg}")


if __name__ == '__main__':
    print('card:', card())
    kernel_probe()
    cfg4()
    print('card:', card())
