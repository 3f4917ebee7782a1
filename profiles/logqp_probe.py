"""CUDA-event probe of the general-noise `logqp=True` KL augmentation.

    python profiles/logqp_probe.py

1. Kernel time: `tsde_logqp_augment` (general noise: per-row Jacobi SVD) against the torch path it replaces
   (`_kl_rate`, i.e. a batched `pinverse`, plus the two `cat`s), fp32, B in {4096, 65536}, (d, m) in {(16,16),
   (32,8), (8,32), (64,64)}.  Operands rotate over enough buffer sets to exceed the 50 MB L2.  With the sweep count
   of a float32 restatement of the kernel's Jacobi loop it prints the flop count per row, 6 k n (n - 1) per sweep
   (three length-k dot products and one rotation of two length-k columns per pair, n (n - 1) / 2 pairs) plus 4 n k
   for the final norms and projections, where n = min(d, m) and k = max(d, m).
2. Solve time: a 100-step general-noise logqp `euler` solve (B = 4096, d = 32, m = 8, fp32): the eager loop on the
   torch path (what runs for shapes over the kernel's bound), the eager loop on the kernel, and the CUDA graph on the
   kernel, alternated in one process.
Prints one JSON line per measurement, with the device name and power limit.
"""
import ctypes
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402
from torchsde_b200._core import base_sde  # noqa: E402

dev = torch.device('cuda')
L2 = 50 * 2 ** 20


def card():
    name = torch.cuda.get_device_name(dev)
    try:
        watts = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        watts = 'unknown'
    return name, watts


def sweeps(g, tol_u=2.0 ** -24, cap=30):
    """Sweeps the kernel's Jacobi loop takes on these rows (float32 restatement: same pair order, same test)."""
    g = g.astype(np.float32)
    B, d, m = g.shape
    A = np.swapaxes(g, 1, 2).copy() if d >= m else g.copy()      # (B, n, k): the n columns being orthogonalised
    n, k = A.shape[1], A.shape[2]
    n2 = n + (n & 1)
    tol = np.float32(((k + 31) // 32 + 5) * tol_u)
    for s in range(cap):
        rotated = False
        for rnd in range(n2 - 1):
            for p in range(n2 // 2):
                a = 0 if p == 0 else (p - 1 + rnd) % (n2 - 1) + 1
                b = (n2 - 2 - p + rnd) % (n2 - 1) + 1
                if a >= n or b >= n:
                    continue
                x, y = A[:, a], A[:, b]
                app, aqq, apq = (x * x).sum(1), (y * y).sum(1), (x * y).sum(1)
                rot = np.abs(apq) > tol * np.sqrt(app) * np.sqrt(aqq)
                if not rot.any():
                    continue
                rotated = True
                with np.errstate(divide='ignore', invalid='ignore'):
                    zeta = (aqq - app) / (2 * apq)
                    t = np.sign(zeta + (zeta == 0)) / (np.abs(zeta) + np.sqrt(1 + zeta * zeta))
                c = 1 / np.sqrt(1 + t * t)
                sn = c * t
                c, sn = np.where(rot, c, 1)[:, None], np.where(rot, sn, 0)[:, None]
                A[:, a], A[:, b] = c * x - sn * y, sn * x + c * y
        if not rotated:
            return s + 1
    return cap


def time_events(fn, reps):
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(reps):
        fn(i)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps * 1e3     # microseconds per call


def kernel_vs_torch(name, watts):
    for B in (4096, 65536):
        for d, m in ((16, 16), (32, 8), (8, 32), (64, 64)):
            set_bytes = 4 * B * (2 * d + d * m) * 2
            nset = max(1, min(8, math.ceil(2 * L2 / set_bytes)))
            sets = [(torch.randn(B, d, device=dev), 0.3 * torch.randn(B, d, m, device=dev), torch.randn(B, d, device=dev))
                    for _ in range(nset)]
            outs = [(torch.empty(B, d + 1, device=dev), torch.empty(B, d + 1, m, device=dev)) for _ in range(nset)]
            Lc = _cabi.make_launch(torch.float32, _cabi.NOISE_GENERAL, B, d, m)
            lib = _cabi.lib()

            def kern(i=0):
                f, g, h = sets[i % nset]
                fa, ga = outs[i % nset]
                assert lib.tsde_logqp_augment(ctypes.byref(Lc), f.data_ptr(), g.data_ptr(), h.data_ptr(), 1e-15,
                                              fa.data_ptr(), ga.data_ptr()) == 0

            def torch_path(i=0):
                f, g, h = sets[i % nset]
                rate = base_sde._kl_rate(f, g, h, False)
                torch.cat([f, rate], dim=1)
                torch.cat([g, g.new_zeros(B, 1, m)], dim=1)

            with torch.no_grad():
                t_k = time_events(kern, 50)
                t_t = time_events(torch_path, 3 if B * d * m > 2 ** 24 else 10)
            n, k = min(d, m), max(d, m)
            sw = sweeps(sets[0][1][:64].cpu().numpy())
            flops = sw * 6 * k * n * (n - 1) + 4 * n * k
            print(json.dumps(dict(what='kernel time', card=name, power_limit_w=watts, B=B, d=d, m=m, dtype='fp32',
                                  kernel_us=round(t_k, 1), torch_us=round(t_t, 1), speedup=round(t_t / t_k, 1),
                                  sweeps=sw, flop_per_row=flops,
                                  kernel_tflops=round(flops * B / (t_k * 1e-6) / 1e12, 2))), flush=True)
            del sets, outs


class Latent(torch.nn.Module):
    noise_type, sde_type = 'general', 'ito'

    def __init__(self, d, m):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.a = torch.nn.Parameter(0.5 * torch.rand(d, generator=gen))
        self.S = torch.nn.Parameter(0.2 + 0.5 * torch.rand(d, m, generator=gen) / math.sqrt(m))

    def f(self, t, y):
        return -self.a * y + 0.1 * torch.sin(y)

    def h(self, t, y):
        return -0.5 * y

    def g(self, t, y):
        return (1.0 + 0.2 * torch.cos(y)).unsqueeze(-1) * self.S


def solve_times(name, watts, B=4096, d=32, m=8, steps=100, rounds=5):
    import warnings
    sde = Latent(d, m).to(dev)
    y0 = torch.full((B, d), 0.2, device=dev)
    dt = 2.0 ** -7
    t1 = steps * dt
    real_fits = _cabi.logqp_general_fits

    def run(mode):
        bm = tsde.BrownianInterval(0.0, t1, size=(B, m), device=dev, entropy=5)
        opts = {'cuda_graph': True} if mode == 'graph' else None
        _cabi.logqp_general_fits = (lambda d_, m_: False) if mode == 'eager_torch' else real_fits
        try:
            with torch.no_grad(), warnings.catch_warnings():
                warnings.simplefilter('ignore')
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                tsde.sdeint(sde, y0, [0.0, t1], bm=bm, method='euler', dt=dt, logqp=True, options=opts)
                e.record()
                torch.cuda.synchronize()
        finally:
            _cabi.logqp_general_fits = real_fits
        return s.elapsed_time(e)

    modes = ('eager_torch', 'eager_kernel', 'graph')
    for mode in modes:
        run(mode)                                  # warm-up (and the graph's capture)
    times = {mode: [] for mode in modes}
    for _ in range(rounds):
        for mode in modes:
            times[mode].append(run(mode))
    print(json.dumps(dict(what='solve time', card=name, power_limit_w=watts, B=B, d=d, m=m, steps=steps,
                          method='euler', dtype='fp32',
                          median_ms={k: round(float(np.median(v)), 2) for k, v in times.items()},
                          min_ms={k: round(float(np.min(v)), 2) for k, v in times.items()})), flush=True)


if __name__ == '__main__':
    name, watts = card()
    kernel_vs_torch(name, watts)
    solve_times(name, watts)
