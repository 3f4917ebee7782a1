"""Fused against unfused general- and additive-noise solves (GENERAL launches of tsde_solve_euler_pointwise,
tsde_solve_reversible_heun_pointwise, tsde_step_predictor_corrector_pointwise and tsde_step_srk_diag_pointwise):
correlated multi-asset GBM, f = mu * y, g = y.unsqueeze(-1) * S, with Euler, midpoint, Euler-Heun and reversible Heun,
and cfg3's additive SDE (tests/problems.py TimeAdditiveExpand) with SRK, as captured graphs; and `adjoint`, a
200-step sdeint_adjoint of the Stratonovich GBM with the reversible pair, forward and backward (eager: the forward
solve fuses, the backward keeps its kernels).  The unfused run is the same solve with the tape rejected.  Both are
alternated three times in one process; prints ms per solve and us per step, with the card's name, SM clock and power
limit read in the same call.  Method names on the command line select cases.

    python profiles/general_pointwise_probe.py [euler] [midpoint] [srk] [euler_heun] [reversible_heun] [adjoint]
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


class CorrelatedGBM(nn.Module):
    noise_type = 'general'

    def __init__(self, d, m, sde_type):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.sde_type = sde_type
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.S = nn.Parameter(torch.rand(d, m, generator=gen) * (0.3 / m ** 0.5))

    def f(self, t, y):
        return self.mu * y

    def g(self, t, y):
        return y.unsqueeze(-1) * self.S


@contextlib.contextmanager
def unfused():
    finish = pointwise.SrkRecorder.finish
    pointwise.SrkRecorder.finish = lambda self: None
    try:
        yield
    finally:
        pointwise.SrkRecorder.finish = finish


def clocks():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,clocks.sm,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out.splitlines()[0] if out else 'n/a'
    except Exception:
        return 'n/a'


def timed(B, d, m, T, method, fused, reps=5):
    if method == 'srk':  # sra1 on cfg3's additive SDE, g = (a b / sqrt(1 + t)).expand(B, d, m)
        sde = problems.TimeAdditiveExpand(d, m, 'ito', dtype=torch.float32).to(DEV)
    else:
        sde = CorrelatedGBM(d, m, 'ito' if method == 'euler' else 'stratonovich').to(DEV)
    y0 = torch.full((B, d), 1.0, device=DEV)
    if method == 'adjoint':
        return timed_adjoint(sde, y0, m, T, fused, reps)
    dt = 2.0 ** -8
    ts = torch.tensor([0.0, T * dt], device=DEV)
    ctx = contextlib.nullcontext() if fused else unfused()
    with ctx, torch.no_grad():
        bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), device=DEV, entropy=1,
                                   levy_area_approximation='space-time' if method == 'srk' else 'none')
        tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options={'cuda_graph': True})  # record, capture
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            tsde.sdeint(sde, y0, ts, bm=bm, method=method, dt=dt, options={'cuda_graph': True})
        end.record()
        torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def timed_adjoint(sde, y0, m, T, fused, reps):
    """sdeint_adjoint with the reversible pair, forward and backward through the loss sum(y_T^2)."""
    B = y0.shape[0]
    dt = 2.0 ** -8
    ts = torch.tensor([0.0, T * dt], device=DEV)
    y0 = y0.clone().requires_grad_(True)
    bm = tsde.BrownianInterval(0.0, T * dt, size=(B, m), device=DEV, entropy=1)

    def once():
        ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=dt)
        torch.autograd.grad((ys[-1] ** 2).sum(), [y0] + list(sde.parameters()))
    with contextlib.nullcontext() if fused else unfused():
        once()  # record (and compile)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            once()
        end.record()
        torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    cases = [('euler', 8192, 32, 16, 500), ('euler', 65536, 64, 16, 100), ('midpoint', 8192, 32, 16, 500),
             ('srk', 8192, 32, 16, 500), ('reversible_heun', 8192, 32, 16, 500),
             ('reversible_heun', 65536, 64, 16, 100), ('euler_heun', 8192, 32, 16, 500),
             ('euler_heun', 65536, 64, 16, 100), ('adjoint', 8192, 32, 16, 200)]
    if sys.argv[1:]:
        cases = [c for c in cases if c[0] in sys.argv[1:]]
    print(json.dumps({'gpu': torch.cuda.get_device_name(), 'clocks_sm_power_limit': clocks()}))
    for method, B, d, m, T in cases:
        res = {'fused': [], 'unfused': []}
        for _ in range(3):
            for fused in (True, False):
                res['fused' if fused else 'unfused'].append(timed(B, d, m, T, method, fused))
        for k, v in res.items():
            print(json.dumps({'method': method, 'B': B, 'd': d, 'm': m, 'T': T, 'path': k,
                              'ms_per_solve': [round(x, 3) for x in v],
                              'us_per_step': [round(1000 * x / T, 2) for x in v]}))
    print(json.dumps({'clocks_sm_power_limit_after': clocks()}))


if __name__ == '__main__':
    main()
