"""Fused against unfused Heun, midpoint and Euler-Heun solves of cfg2's SDE in Stratonovich form, alternated in one
process.

    python profiles/pc_pointwise_probe.py [--reps 3] [--solves 5] [--steps 1000] [--methods heun,midpoint,euler_heun]

cfg2's SDE (GBM, diagonal noise, fp32, B = 65536, d = 64, dt = 2^-10) with sde_type='stratonovich', whose drift is
f = mu*y - 0.5*sigma^2*y, solved with options={'cuda_graph': True, 'static_output': True}.  fused: every step after
the first is tsde_step_predictor_corrector_pointwise; unfused: the same solve with the recorded tape rejected
(pointwise.SrkRecorder.finish returns None), i.e. the user's f and g twice (g only, the second time, for Euler-Heun)
and two solver kernels per step.  Each repetition builds a fresh plan for each variant, runs it once to capture, then
times `--solves` replays with CUDA events.  The outputs of the two variants must be byte-identical.  Prints one JSON
line with the card's name, power limit and SM clock (read after the timed solves).
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402
from torchsde_b200._core import graph, pointwise  # noqa: E402

DEV = torch.device('cuda')


class GBM(nn.Module):
    noise_type, sde_type = 'diagonal', 'stratonovich'

    def __init__(self, d):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen) * 0.5)

    def f(self, t, y):
        return self.mu * y - .5 * (self.sigma ** 2) * y

    def g(self, t, y):
        return self.sigma * y


@contextlib.contextmanager
def unfused():
    finish = pointwise.SrkRecorder.finish
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.SrkRecorder.finish = finish


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
    ap.add_argument('--solves', type=int, default=5)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--B', type=int, default=65536)
    ap.add_argument('--D', type=int, default=64)
    ap.add_argument('--methods', default='heun,midpoint,euler_heun')
    a = ap.parse_args()
    dt = 2.0 ** -10
    sde = GBM(a.D).to(DEV)
    y0 = torch.full((a.B, a.D), 0.1, device=DEV)
    ts = torch.arange(a.steps + 1, device=DEV, dtype=torch.float32) * dt

    def run(method):
        bm = tsde.BrownianInterval(0.0, a.steps * dt, size=(a.B, a.D), device=DEV, entropy=2024)
        with torch.no_grad():
            return tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt,
                               options={'cuda_graph': True, 'static_output': True})

    def variant(method, ctx):
        with ctx():
            graph.drop_plans(sde)
            n0 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_PC)
            run(method)                      # capture (and the recorded first step)
            fused = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_PC) > n0
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.solves):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ys = run(method)
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            ys = ys.clone()                  # (the static output buffer dies with the plan)
            graph.drop_plans(sde)
            return ys, float(np.median(ms)), fused

    out = {'B': a.B, 'D': a.D, 'steps': a.steps, 'methods': {}}
    identical = True
    for method in a.methods.split(','):
        res = {'fused_ms': [], 'unfused_ms': []}
        same = True
        for _ in range(a.reps):
            yf, tf, ff = variant(method, contextlib.nullcontext)
            yu, tu, fu = variant(method, unfused)
            assert ff and not fu, (method, ff, fu)
            same = same and torch.equal(yf.view(torch.int32), yu.view(torch.int32))
            res['fused_ms'].append(round(tf, 3))
            res['unfused_ms'].append(round(tu, 3))
        res['byte_identical'] = same
        identical = identical and same
        out['methods'][method] = res
    out['gpu'] = gpu()
    out['byte_identical'] = identical
    print(json.dumps(out), flush=True)
    if not identical:
        sys.exit(1)


if __name__ == '__main__':
    main()
