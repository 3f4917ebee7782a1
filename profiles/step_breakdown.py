"""In-situ time of each kernel of the cfg2 Milstein step, from torch.profiler over a graph-replayed solve.

    python profiles/step_breakdown.py [out.json]    [TORCHSDE_B200_LIB=<other build> for an A/B on the same box]

Full cfg2 batch and state (65536 x 64 fp32), NSTEPS (default 100) steps, solved once to capture the CUDA graph and
then replayed under the profiler.  A step is five kernels: the user's f = mu*y on a parallel branch, and g = sigma*y
-> tsde_milstein_vjp_seed -> autograd's go*sigma -> tsde_step_milstein.  f and g are reported together (the same
broadcast multiply; they run side by side).  A kernel launched with programmatic dependent launch
starts before its predecessor ends, so its in-situ duration includes the overlap.  Prints one JSON line with the
mean microseconds per step of each kernel and the replay's wall time per step.
"""
import json
import os
import sys
import tempfile
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import torchsde_b200 as tsde  # noqa: E402

w = dict(bench.WORKLOADS['cfg2'])
n = int(os.environ.get('NSTEPS', '100'))
dev = torch.device('cuda')
sde = bench.build_sde(w, dev)
ts = (torch.arange(n + 1, dtype=torch.float32) * w['dt']).to(dev)
y0 = torch.full((w['B'], w['D']), 0.1, device=dev)


def solve(entropy):
    bm = tsde.BrownianInterval(0.0, n * w['dt'], size=(w['B'], w['D']), dtype=torch.float32, device=dev,
                               entropy=entropy)
    with torch.no_grad():
        return tsde.sdeint(sde, y0, ts, bm=bm, method='milstein', dt=w['dt'],
                           options={'cuda_graph': True, 'static_output': True})


for i in range(3):
    solve(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
solve(10)
e1.record()
torch.cuda.synchronize()
wall_us = e0.elapsed_time(e1) * 1e3 / n

with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    solve(11)
    torch.cuda.synchronize()
with tempfile.TemporaryDirectory() as tmp:
    path = os.path.join(tmp, 'trace.json')
    prof.export_chrome_trace(path)
    trace = json.load(open(path))
kernels = sorted((e for e in trace['traceEvents'] if e.get('cat') == 'kernel'), key=lambda e: e['ts'])
# A replayed graph does not keep a branch on one stream, so the multiplies are told apart by order: within a step,
# f and g start before the seed, the vjp after it.
dur = defaultdict(list)
other = defaultdict(list)
after_seed = False
for e in kernels:
    name = e['name']
    if 'MilsteinSeedOp' in name:
        r, after_seed = 'seed', True
    elif 'MilsteinOp' in name:
        r, after_seed = 'tableau', False
    elif 'mul' in name.lower():
        r = 'vjp=go*sigma' if after_seed else 'f=mu*y, g=sigma*y'
    else:
        other[name[:100]].append(e['dur'])
        continue
    dur[r].append(e['dur'])
res = {'lib': os.environ.get('TORCHSDE_B200_LIB', 'in-tree'), 'steps': n, 'wall_us_per_step': round(wall_us, 2),
       'kernels_us': {k: {'mean': round(float(np.mean(v)), 2), 'count': len(v)} for k, v in sorted(dur.items())},
       'other_kernels': {k: {'mean': round(float(np.mean(v)), 2), 'count': len(v)} for k, v in other.items()}}
print(json.dumps(res), flush=True)
if len(sys.argv) > 1:
    json.dump(res, open(sys.argv[1], 'w'), indent=1)
