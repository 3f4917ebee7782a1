"""Fused against unfused solves of SDEs with transcendental ops (options={'transcendental': True}): TanhGeneral
(tests/problems.py, g = tanh(y)[..., None] * S) with Euler at cfg3_euler_general's shape (B = 8192, d = 32, m = 16,
T = 500) and at cfg3_euler_general_large's (B = 65536, d = 64, m = 16, T = 100), and a diagonal Milstein SDE with exp
in g (f = mu * y, g = sigma * exp(-y * y)) at cfg2's shape (B = 65536, d = 64, T = 1000), as captured graphs.  The
unfused run is the same solve with the tape rejected.  Both are alternated three times in one process; prints ms per
solve and us per step, with the GPU's name, SM clock and power limit read in the same call.  Case names on the command
line select cases.

    python profiles/transcendental_pointwise_probe.py [tanh_general] [tanh_general_large] [milstein_exp]
"""
import contextlib
import json
import os
import subprocess
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200._core import pointwise  # noqa: E402
from tests import problems  # noqa: E402

DEV = 'cuda'
OPTIONS = {'cuda_graph': True, 'transcendental': True}


class ExpMilstein(nn.Module):
    noise_type, sde_type = 'diagonal', 'ito'

    def __init__(self, d):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen) * 0.3 + 0.1)

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return self.sigma * torch.exp(-y * y)


@contextlib.contextmanager
def unfused():
    finish, srk_finish = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
    pointwise.Recorder.finish = lambda self, *a: None
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.Recorder.finish, pointwise.SrkRecorder.finish = finish, srk_finish


def clocks():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,clocks.sm,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out.splitlines()[0] if out else 'n/a'
    except Exception:
        return 'n/a'


CASES = {  # name: (method, B, d, m, T, dt)
    'tanh_general': ('euler', 8192, 32, 16, 500, 2.0 ** -8),
    'tanh_general_large': ('euler', 65536, 64, 16, 100, 2.0 ** -8),
    'milstein_exp': ('milstein', 65536, 64, 64, 1000, 2.0 ** -10),
}


def timed(name, fused, reps=5):
    method, B, d, m, T, dt = CASES[name]
    sde = (ExpMilstein(d) if method == 'milstein' else problems.TanhGeneral(d, m, 'ito', dtype=torch.float32)).to(DEV)
    y0 = torch.full((B, d), 0.5, device=DEV)
    ts = torch.tensor([0.0, T * dt], device=DEV)
    ctx = contextlib.nullcontext() if fused else unfused()
    with ctx, torch.no_grad():
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), device=DEV, entropy=1)
        tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=OPTIONS)  # record, capture
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options=OPTIONS)
        end.record()
        torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    names = [n for n in CASES if not sys.argv[1:] or n in sys.argv[1:]]
    print(json.dumps({'gpu_clocks_sm_power_limit': clocks()}))
    for name in names:
        method, B, d, m, T, _ = CASES[name]
        res = {'fused': [], 'unfused': []}
        for _ in range(3):
            for fused in (True, False):
                res['fused' if fused else 'unfused'].append(timed(name, fused))
        for k, v in res.items():
            print(json.dumps({'case': name, 'method': method, 'B': B, 'd': d, 'm': m, 'T': T, 'path': k,
                              'ms_per_solve': [round(x, 3) for x in v],
                              'us_per_step': [round(1000 * x / T, 2) for x in v]}))
    print(json.dumps({'gpu_clocks_sm_power_limit_after': clocks()}))


if __name__ == '__main__':
    main()
