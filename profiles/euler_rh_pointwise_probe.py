"""Fused against unfused Euler and reversible-Heun solves of cfg2's SDE, alternated in one process.

    python profiles/euler_rh_pointwise_probe.py [--reps 3] [--solves 5] [--steps 1000] [--adjoint-steps 200]
                                                [--workloads euler,reversible_heun,adjoint]

cfg2's SDE (GBM, diagonal noise, fp32, B = 65536, d = 64, dt = 2^-10), with options={'cuda_graph': True,
'static_output': True}:
  euler            the Ito SDE (f = mu*y, g = sigma*y), method='euler';
  reversible_heun  its Stratonovich form (f = mu*y - 0.5*sigma^2*y), method='reversible_heun';
  adjoint          `sdeint_adjoint` with the reversible pair on the Stratonovich form, forward and backward, with
                   adjoint_options={'cuda_graph': True}, at --adjoint-steps steps (the output series of a 1000-step
                   solve would not leave room for the backward sweep's buffers next to it).
fused: every step after the recorded first one runs in tsde_solve_euler_pointwise / tsde_solve_reversible_heun_pointwise
chunks of up to 64 steps; unfused: the same solve with the recorded tape rejected (pointwise.SrkRecorder.finish
returns None), i.e. the user's f and g and one (Euler) or two (reversible Heun) solver kernels per step.  The
backward sweep of `adjoint` is unfused in both.  Each repetition builds a fresh plan for each variant, runs it once to
capture, then times `--solves` solves with CUDA events, whole `sdeint` calls (which include its host-side set-up) and,
for the two forward workloads, replays of the captured graph alone.  The outputs of the two variants (and for `adjoint` the
gradients of y0 and of every parameter) must be byte-identical.  Prints one JSON line with the card's name, power limit
and SM clock (read after the timed solves).
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
    noise_type = 'diagonal'

    def __init__(self, d, sde_type):
        super().__init__()
        self.sde_type = sde_type
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen) * 0.5)

    def f(self, t, y):
        if self.sde_type == 'ito':
            return self.mu * y
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


def launches():
    return _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_CHUNK)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--solves', type=int, default=5)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--adjoint-steps', type=int, default=200)
    ap.add_argument('--B', type=int, default=65536)
    ap.add_argument('--D', type=int, default=64)
    ap.add_argument('--workloads', default='euler,reversible_heun,adjoint')
    a = ap.parse_args()
    dt = 2.0 ** -10
    sdes = {'euler': GBM(a.D, 'ito').to(DEV), 'reversible_heun': GBM(a.D, 'stratonovich').to(DEV)}
    sdes['adjoint'] = sdes['reversible_heun']
    y0 = torch.full((a.B, a.D), 0.1, device=DEV)
    opts = {'cuda_graph': True, 'static_output': True}

    def run(work):
        sde = sdes[work]
        steps = a.adjoint_steps if work == 'adjoint' else a.steps
        ts = torch.arange(steps + 1, device=DEV, dtype=torch.float32) * dt
        bm = tsde.BrownianInterval(0.0, steps * dt, size=(a.B, a.D), device=DEV, entropy=2024)
        if work != 'adjoint':
            with torch.no_grad():
                return [tsde.sdeint(sde, y0, ts, bm=bm, method=work, dt=dt, options=opts)]
        y = y0.clone().requires_grad_(True)
        for p in sde.parameters():
            p.grad = None
        ys = tsde.sdeint_adjoint(sde, y, ts, bm=bm, method='reversible_heun', dt=dt, options=opts,
                                 adjoint_options={'cuda_graph': True})
        ys.pow(2).sum().backward()
        return [ys.detach(), y.grad] + [p.grad for p in sde.parameters()]

    def variant(work, ctx, ref=None):
        """(a copy of the outputs when `ref` is None, median ms per solve, whether it fused, whether the outputs equal
        `ref` byte for byte).  Only one copy of a 1000-step output series is held at a time."""
        with ctx():
            graph.drop_plans(sdes[work])
            n0 = launches()
            run(work)                        # capture (and the recorded first step)
            fused = launches() > n0
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.solves):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = run(work)
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            # the captured solve alone, without sdeint's host-side work (not for `adjoint`, whose backward sweep is
            # another graph)
            replay_ms = None
            if work != 'adjoint':
                plan, rs = graph.LAST_PLAN, []
                for _ in range(a.solves):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    plan.graph.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    rs.append(e0.elapsed_time(e1))
                replay_ms = float(np.median(rs))
                del plan
            kept, same = None, None
            if ref is None:
                kept = [x.clone() for x in out]  # (the static output buffer dies with the plan)
            else:
                same = all(torch.equal(p.view(torch.int32), q.view(torch.int32)) for p, q in zip(out, ref))
            del out
            graph.drop_plans(sdes[work])
        torch.cuda.empty_cache()
        return kept, float(np.median(ms)), replay_ms, fused, same

    out = {'B': a.B, 'D': a.D, 'steps': a.steps, 'adjoint_steps': a.adjoint_steps, 'workloads': {}}
    identical = True
    for work in a.workloads.split(','):
        steps = a.adjoint_steps if work == 'adjoint' else a.steps
        res = {'fused_ms': [], 'unfused_ms': [], 'fused_replay_ms': [], 'unfused_replay_ms': []}
        same = True
        for _ in range(a.reps):
            xf, tf, rf, ff, _ = variant(work, contextlib.nullcontext)
            _, tu, ru, fu, s = variant(work, unfused, xf)
            del xf
            assert ff and not fu, (work, ff, fu)
            same = same and s
            res['fused_ms'].append(round(tf, 3))
            res['unfused_ms'].append(round(tu, 3))
            if rf is not None:
                res['fused_replay_ms'].append(round(rf, 3))
                res['unfused_replay_ms'].append(round(ru, 3))
        # per step: of the captured solve alone where there is one, else of the whole call
        for v in ('fused', 'unfused'):
            ms = res[f'{v}_replay_ms'] or res[f'{v}_ms']
            res[f'{v}_us_per_step'] = round(1e3 * float(np.median(ms)) / steps, 2)
        res['byte_identical'] = same
        identical = identical and same
        out['workloads'][work] = res
    out['gpu'] = gpu()
    out['byte_identical'] = identical
    print(json.dumps(out), flush=True)
    if not identical:
        sys.exit(1)


if __name__ == '__main__':
    main()
