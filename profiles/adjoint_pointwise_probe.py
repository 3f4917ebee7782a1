"""The reversible-Heun adjoint's backward sweep, fused (adjoint_options={'fused_backward': True}) against unfused,
alternated in one process.

    python profiles/adjoint_pointwise_probe.py [--reps 3] [--solves 5] [--steps 200] [--batch 65536] [--dim 64]

cfg2's SDE in Stratonovich form (GBM, diagonal noise, fp32, B = 65536, d = 64, dt = 2^-10), 200 steps of
`sdeint_adjoint` with the reversible pair, the loss sum(w * ys).  The drift is written with sigma broadcast before it is
squared, f = mu*y - sigma*(sigma*(0.5*y)), so that each parameter's gradient is a batch reduction of a (rows, d) value
(pointwise.AdjointRecorder rejects a parameter transformed before it is broadcast, as in .5*(sigma**2)*y).  Four
variants, each repetition running them in turn: eager and captured (adjoint_options={'cuda_graph': True}), each fused
and unfused.  Per variant, after one untimed solve (recording, compilation, capture), --solves timed forward + backward
passes: CUDA events around sdeint_adjoint (forward) and around backward() (the backward sweep, a graph replay when
captured).  ys, y0's gradient and the extra-state gradients of fused and unfused must be byte-identical, and the
parameter gradients close (their largest relative difference is printed).  Prints one JSON line with the card's name,
power limit and SM clock (read after the timed solves), the median times in ms and the compiled kernel's launches.
"""
import argparse
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
from torchsde_b200._core import adjoint  # noqa: E402

DEV = torch.device('cuda')


class GBM(nn.Module):
    sde_type, noise_type = 'stratonovich', 'diagonal'

    def __init__(self, d):
        super().__init__()
        gen = torch.Generator().manual_seed(0)
        self.mu = nn.Parameter(torch.rand(d, generator=gen) * 0.1)
        self.sigma = nn.Parameter(torch.rand(d, generator=gen) * 0.5)

    def f(self, t, y):
        return self.mu * y - self.sigma * (self.sigma * (0.5 * y))

    def g(self, t, y):
        return self.sigma * y


def run(args, fused, graphs, timed):
    B, d, T, dt = args.batch, args.dim, args.steps, 2.0 ** -10
    sde = GBM(d).to(DEV)
    ts = torch.arange(T + 1, device=DEV, dtype=torch.float32) * dt
    y0 = torch.full((B, d), 0.1, device=DEV, requires_grad=True)
    w = torch.linspace(-1, 1, (T + 1) * B * d, device=DEV).view(T + 1, B, d)
    opts = {}
    if fused:
        opts['fused_backward'] = True
    if graphs:
        opts['cuda_graph'] = True
    fwd, bwd = [], []
    out = None
    for i in range(1 + timed):
        y0.grad = None
        for p in sde.parameters():
            p.grad = None
        bm = tsde.BrownianInterval(0.0, float(ts[-1]), size=(B, d), device=DEV, entropy=1)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        ys = tsde.sdeint_adjoint(sde, y0, ts, bm=bm, method='reversible_heun', dt=dt, adjoint_options=dict(opts))
        loss = (w * ys).sum()
        e[1].record()
        loss.backward()
        e[2].record()
        torch.cuda.synchronize()
        if i:
            fwd.append(e[0].elapsed_time(e[1]))
            bwd.append(e[1].elapsed_time(e[2]))
        out = (ys.detach(), y0.grad.clone(), [p.grad.clone() for p in sde.parameters()])
    adjoint.drop_plans(sde)
    return fwd, bwd, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--solves', type=int, default=5)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--batch', type=int, default=65536)
    ap.add_argument('--dim', type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("adjoint_pointwise_probe: no CUDA device; nothing is measured")
    variants = [(f, g) for g in (False, True) for f in (False, True)]
    times = {v: ([], []) for v in variants}
    outs = {}
    n0 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADJOINT)
    for _ in range(args.reps):
        for v in variants:
            fwd, bwd, outs[v] = run(args, *v, args.solves)
            times[v][0].extend(fwd)
            times[v][1].extend(bwd)
    fused_launches = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADJOINT) - n0
    same, rel = True, 0.0
    for g in (False, True):
        a, b = outs[(True, g)], outs[(False, g)]
        same = same and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        for pa, pb in zip(a[2], b[2]):
            rel = max(rel, float(((pa - pb).abs() / pb.abs().clamp_min(1e-30)).max()))
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    name = {(False, False): 'unfused_eager', (True, False): 'fused_eager', (False, True): 'unfused_graph',
            (True, True): 'fused_graph'}
    res = {'gpu': smi, 'B': args.batch, 'd': args.dim, 'steps': args.steps, 'reps': args.reps,
           'solves': args.solves, 'ys_and_y0_grad_identical': same, 'param_grad_max_rel_diff': rel,
           'fused_kernel_launches': fused_launches}
    for v in variants:
        res[name[v] + '_fwd_ms'] = float(np.median(times[v][0]))
        res[name[v] + '_bwd_ms'] = float(np.median(times[v][1]))
        res[name[v] + '_bwd_ms_min_max'] = [float(min(times[v][1])), float(max(times[v][1]))]
    print(json.dumps(res))


if __name__ == '__main__':
    main()
