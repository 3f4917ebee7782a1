"""Per-proposal time of adaptive solves, fused (tsde_adaptive_proposal_pointwise) against unfused, alternated in one
process.

    python profiles/adaptive_pointwise_probe.py [--reps 3] [--methods milstein,euler,srk] [--B 65536] [--D 64]

cfg2's SDE (GBM, Ito, diagonal noise, fp32, B = 65536, d = 64) solved with adaptive=True from t = 0 to 1 (dt = 0.01,
rtol = 1e-5, atol = 1e-6) on a BrownianInterval (space-time Levy area for SRK).  fused: every proposal after the first
is the three Brownian queries, one proposal kernel and the error reduction; unfused: the same solve with the recorded
tape rejected (the recorders' `finish` returns None), i.e. three unfused steps per proposal.  Each repetition runs
both variants on a fresh Brownian motion of the same entropy; a solve is timed with the host clock around it (it ends
in a synchronise) and divided by its number of proposals.  `queries_ms` is the three Brownian queries of a proposal
alone: the fused solve's query sequence replayed on a fresh Brownian motion.  The outputs of the two variants must be
byte-identical.  Prints one JSON line with the card's name, power limit and SM clock (read after the timed solves).
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402
from torchsde_b200._core import base_solver, pointwise  # noqa: E402

DEV = torch.device('cuda')


class GBM(nn.Module):
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, d):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen) * 0.5)

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return self.sigma * y


@contextlib.contextmanager
def unfused():
    saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


@contextlib.contextmanager
def counting():
    """The number of proposals of the solves inside."""
    n, real = [0], base_solver.BaseSDESolver._error_estimate

    def estimate(self, *a):
        n[0] += 1
        return real(self, *a)
    base_solver.BaseSDESolver._error_estimate = estimate
    try:
        yield n
    finally:
        base_solver.BaseSDESolver._error_estimate = real


class Logged:
    def __init__(self, bm, log):
        self._bm, self._log = bm, log

    def __getattr__(self, name):
        return getattr(self._bm, name)

    def __call__(self, ta, tb=None, return_U=False, return_A=False):
        self._log.append((ta, tb, return_U))
        return self._bm(ta, tb, return_U=return_U, return_A=return_A)


def gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[torch.cuda.current_device()] if q else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--B', type=int, default=65536)
    ap.add_argument('--D', type=int, default=64)
    ap.add_argument('--methods', default='milstein,euler,srk')
    a = ap.parse_args()
    sde = GBM(a.D).to(DEV)
    y0 = torch.full((a.B, a.D), 0.1, device=DEV)
    ts = torch.tensor([0.0, 1.0], device=DEV)

    def bm(method):
        return tsde.BrownianInterval(0.0, 1.0, size=(a.B, a.D), device=DEV, entropy=2024,
                                     levy_area_approximation='space-time' if method == 'srk' else 'none')

    def run(method, ctx, log=None):
        with ctx(), counting() as n, torch.no_grad():
            n0 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE)
            b = bm(method) if log is None else Logged(bm(method), log)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ys = tsde.sdeint(sde, y0, ts, bm=b, method=method, dt=0.01, adaptive=True, rtol=1e-5, atol=1e-6)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            fused = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE) > n0
        return ys, ms / n[0], n[0], fused

    out = {'B': a.B, 'D': a.D, 'dtype': 'float32', 'methods': {}}
    identical = True
    for method in a.methods.split(','):
        run(method, contextlib.nullcontext)    # warm-up: modules, the program's compilation, allocator
        run(method, unfused)
        res = {'fused_ms': [], 'unfused_ms': [], 'queries_ms': []}
        same = True
        for _ in range(a.reps):
            log = []
            yf, tf, nf, ff = run(method, contextlib.nullcontext, log)
            yu, tu, nu, fu = run(method, unfused)
            assert ff and not fu and nf == nu, (method, ff, fu, nf, nu)
            same = same and torch.equal(yf.view(torch.int32), yu.view(torch.int32))
            b = bm(method)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for ta, tb, u in log:
                b(ta, tb, return_U=u)
            torch.cuda.synchronize()
            res['queries_ms'].append(round((time.perf_counter() - t0) * 1e3 / nf, 4))
            res['fused_ms'].append(round(tf, 4))
            res['unfused_ms'].append(round(tu, 4))
            res['proposals'] = nf
        res['byte_identical'] = same
        res['speedup_median'] = round(float(np.median(res['unfused_ms']) / np.median(res['fused_ms'])), 2)
        identical = identical and same
        out['methods'][method] = res
    out['gpu'] = gpu()
    out['byte_identical'] = identical
    print(json.dumps(out), flush=True)
    if not identical:
        sys.exit(1)


if __name__ == '__main__':
    main()
