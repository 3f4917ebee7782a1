"""Fused against unfused solves of a full-truncation CIR SDE, alternated in one process.

    python profiles/clamp_pointwise_probe.py [--reps 3] [--solves 5] [--steps 1000] [--methods euler,milstein]

The SDE: dv = kappa (theta - v+) dt + xi sqrt(v+) dW with v+ = v.clamp(min=0), diagonal noise, fp32, B = 65536,
d = 64, dt = 2^-10, v0 = 0.04, options={'cuda_graph': True, 'static_output': True}, with method='euler' and
method='milstein' (Ito; its vjp of g holds autograd's clamp backward: ge, where).  fused: every step after the
recorded first one runs in tsde_solve_euler_pointwise / tsde_solve_milstein_pointwise chunks of up to 64 steps;
unfused: the same solve with the recorded tape rejected (Recorder.finish and SrkRecorder.finish return None), i.e.
the user's f and g (and for Milstein the vjp) and the solver's kernels at every step.  Each repetition builds a fresh
plan per variant, runs it once to capture, then times `--solves` replays of the captured graph with CUDA events.  The
outputs of the two variants must be byte-identical.  Prints one JSON line with the card's name, power limit and SM
clock (read after the timed solves).
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


class CIR(nn.Module):
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, d):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.kappa = nn.Parameter(torch.rand(d, generator=gen) + 0.5)
        self.theta = nn.Parameter(torch.rand(d, generator=gen) * 0.05 + 0.02)
        self.xi = nn.Parameter(torch.rand(d, generator=gen) * 0.5 + 0.3)

    def f(self, t, v):
        return self.kappa * (self.theta - v.clamp(min=0))

    def g(self, t, v):
        return self.xi * torch.sqrt(v.clamp(min=0))


@contextlib.contextmanager
def unfused():
    saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


def gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[torch.cuda.current_device()] if q else None
    except Exception:
        return None


def launches():
    return sum(_cabi.lib().tsde_kernel_launches(k) for k in (_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_CHUNK))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--solves', type=int, default=5)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--B', type=int, default=65536)
    ap.add_argument('--D', type=int, default=64)
    ap.add_argument('--methods', default='euler,milstein')
    a = ap.parse_args()
    dt = 2.0 ** -10
    sde = CIR(a.D).to(DEV)
    y0 = torch.full((a.B, a.D), 0.04, device=DEV)
    ts = torch.arange(a.steps + 1, device=DEV, dtype=torch.float32) * dt
    opts = {'cuda_graph': True, 'static_output': True}

    def variant(method, ctx, ref=None):
        """(a copy of the output when `ref` is None, median ms per replay, whether it fused, whether the output equals
        `ref` byte for byte)."""
        with ctx():
            graph.drop_plans(sde)
            bm = tsde.BrownianInterval(0.0, a.steps * dt, size=(a.B, a.D), device=DEV, entropy=2024)
            n0 = launches()
            with torch.no_grad():
                out = tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=opts)  # capture and first run
            fused = launches() > n0
            plan = graph.LAST_PLAN
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.solves):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                plan.graph.replay()
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            kept = same = None
            if ref is None:
                kept = out.clone()
            else:
                same = torch.equal(out.view(torch.int32), ref.view(torch.int32))
            del out, plan
            graph.drop_plans(sde)
        torch.cuda.empty_cache()
        return kept, float(np.median(ms)), fused, same

    res = {'B': a.B, 'D': a.D, 'steps': a.steps, 'methods': {}}
    identical = True
    for method in a.methods.split(','):
        r = {'fused_ms': [], 'unfused_ms': []}
        same = True
        for _ in range(a.reps):
            xf, tf, ff, _ = variant(method, contextlib.nullcontext)
            _, tu, fu, s = variant(method, unfused, xf)
            del xf
            assert ff and not fu, (method, ff, fu)
            same = same and s
            r['fused_ms'].append(round(tf, 3))
            r['unfused_ms'].append(round(tu, 3))
        for v in ('fused', 'unfused'):
            r[f'{v}_us_per_step'] = round(1e3 * float(np.median(r[f'{v}_ms'])) / a.steps, 2)
        r['speedup'] = round(r['unfused_us_per_step'] / r['fused_us_per_step'], 2)
        r['byte_identical'] = same
        identical = identical and same
        res['methods'][method] = r
    res['gpu'] = gpu()
    res['byte_identical'] = identical
    print(json.dumps(res), flush=True)
    if not identical:
        sys.exit(1)


if __name__ == '__main__':
    main()
