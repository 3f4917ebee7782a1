"""CUDA-event probe of the producer -> consumer handoffs of the cfg2 Milstein step (65536 x 64 fp32, 16 MiB tensors).

    python profiles/handoff_probe.py           [TORCHSDE_B200_LIB=<other build> for an A/B on the same box]

Each pair is launched the way the solver issues it: back-to-back launches captured into a CUDA graph and replayed.
Pair k works on buffer set k % 4 (at least 256 MiB in all, five times the 50 MB L2), so the only operand a consumer
can find in L2 is the one its producer has just written.  The consumer's in-situ time is the time of the pair minus
the time of the producer replayed alone on the same sets; the consumer alone on the same sets ('cold') is printed
beside it.  Pairs:
  g -> seed         torch broadcast multiply sigma*y writes g, tsde_milstein_vjp_seed reads it (the user's g, ascending)
  vjp -> tableau    torch multiply go*sigma writes gdg, tsde_step_milstein reads it with cold y0, f, g
  tableau -> f      tsde_step_milstein writes y1, torch multiply mu*y1 reads it (the next step's f)
Prints one JSON line.
"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torchsde_b200 import _cabi  # noqa: E402

dev = torch.device('cuda')
lib = _cabi.lib()
B, D = int(os.environ.get('PROBE_B', 65536)), int(os.environ.get('PROBE_D', 64))
dt = 2.0 ** -10
NSET, REPS = 4, 24
key = torch.tensor([987654321], dtype=torch.int64, device=dev)
L = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL, B, D, D)
nz = _cabi.Noise()
nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, key.data_ptr(), 7, 1, dt, dt
sigma = torch.rand(D, device=dev) * 0.5
mu = torch.rand(D, device=dev) * 0.5
P = lambda t: t.data_ptr()  # noqa


def seed(s):
    _cabi.check(lib.tsde_milstein_vjp_seed(ctypes.byref(L), ctypes.byref(nz), P(s['g']), dt, 1, P(s['go'])), 'seed')


def tableau(s):
    _cabi.check(lib.tsde_step_milstein(ctypes.byref(L), ctypes.byref(nz), P(s['y0']), P(s['f']), P(s['g']),
                                       P(s['gdg']), dt, P(s['y1'])), 'tableau')


PAIRS = {
    'g->seed': (lambda s: torch.mul(s['y0'], sigma, out=s['g']), seed),
    'vjp->tableau': (lambda s: torch.mul(s['go'], sigma, out=s['gdg']), tableau),
    'tableau->f': (tableau, lambda s: torch.mul(s['y1'], mu, out=s['f'])),
}
sets = [{k: torch.rand(B, D, device=dev) + 0.5 for k in ('y0', 'f', 'g', 'go', 'gdg', 'y1')} for _ in range(NSET)]


def timed(fns):
    """Microseconds per repetition of `fns` (each called on the repetition's buffer set), graph-captured."""
    for s in sets:
        for fn in fns:
            fn(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.stream = torch.cuda.current_stream(dev).cuda_stream  # launch on the capturing stream
        for i in range(REPS):
            for fn in fns:
                fn(sets[i % NSET])
    L.stream = torch.cuda.current_stream(dev).cuda_stream
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(9):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / REPS)
    del graph
    return float(np.median(times))


out = {'lib': os.environ.get('TORCHSDE_B200_LIB', 'in-tree'), 'B': B, 'D': D}
for name, (prod, cons) in PAIRS.items():
    pair, p_alone, c_cold = timed([prod, cons]), timed([prod]), timed([cons])
    out[name] = {'pair_us': round(pair, 2), 'producer_us': round(p_alone, 2), 'consumer_in_situ_us': round(pair - p_alone, 2),
                 'consumer_cold_us': round(c_cold, 2)}
print(json.dumps(out), flush=True)
