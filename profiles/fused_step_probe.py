"""CUDA-event probe of the fused Milstein step (tsde_step_milstein_pointwise) and of chunks of K steps per launch
(tsde_solve_milstein_pointwise) at the cfg2 size (65536 x 64 fp32).

    python profiles/fused_step_probe.py

The program is the one the solver records for cfg2's SDE (f = mu*y, g = sigma*y, vjp go*sigma).
  cold     back-to-back launches captured into a CUDA graph, launch k on buffer set k % NSET (y0, y1 pairs of 16 MiB,
           256 MiB in all, five times the 50 MB L2): y0 comes from HBM
  in situ  the launches chained as the solver chains them: y1 of launch k is y0 of launch k + 1
  seed     tsde_milstein_vjp_seed on the same sets, cold: the same Philox + Box-Muller work per quad with one tensor
           read and one written, i.e. the RNG-bound time of a kernel of this shape
  chunk_K  K consecutive steps in one launch, every step's y1 stored to its row of an output series (as cfg2 stores
           every step), in situ (the next launch starts from the last row) and cold (y0 from the rotating sets);
           microseconds per step and the achieved write bandwidth.  K = 128 does not fit the step table
           (TSDE_PW_MAX_STEPS = 64, bounded by the 4 KiB parameter space) and is reported as such.  The write bandwidth is also
           given as a share of the H100 SXM data sheet's 3.35 TB/s and of the measured fill floor, the floor of a step
           being its y1 store.  Each chunk runs on a uniform grid (consecutive cells: the kernel's loop of one back-edge,
           PwSteps::uniform) and, as chunk_K_table_*, on cells two apart, which the kernel runs through its step table
           (the general loop) with the same work per step.
  fill     torch's fill_ of the 64 rows of one output series (64 x 16 MiB at cfg2), in microseconds per row: the store
           floor of a step as this card reaches it.
  compile  the one-time cost of the program's kernels: tsde_pointwise_compile (NVRTC to an sm_90a cubin, then the
           library load) in a process that has not compiled the program yet, in ms.  The solver pays it on the recording
           step, outside bench.py's timed region; a later program of the same structure pays nothing.
Algorithmic bytes of the fused step: 2 * D * 4 per trajectory (y0 read, y1 written).  Prints one JSON line with the
card's name and power limit.
"""
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from torchsde_b200 import _cabi  # noqa: E402
from torchsde_b200._core import pointwise  # noqa: E402

dev = torch.device('cuda')
lib = _cabi.lib()
B, D = int(os.environ.get('PROBE_B', 65536)), int(os.environ.get('PROBE_D', 64))
dt = 2.0 ** -10
NSET, REPS = 8, 32
key = torch.tensor([987654321], dtype=torch.int64, device=dev)
L = _cabi.make_launch(torch.float32, _cabi.NOISE_DIAGONAL, B, D, D)
nz = _cabi.Noise()
nz.source, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, key.data_ptr(), 7, 1, dt, dt
sigma = torch.rand(D, device=dev) * 0.5
mu = torch.rand(D, device=dev) * 0.5
t0 = torch.zeros((), device=dev)
P = lambda t: t.data_ptr()  # noqa


def record_program():
    """The solver's recording of one cfg2 step (pointwise.Recorder), on tensors of the cfg2 shape."""
    y0 = torch.rand(B, D, device=dev)
    rec = pointwise.Recorder(y0, t0)
    f = rec.segment(lambda: mu * y0)
    with torch.enable_grad():
        s = sigma.detach().requires_grad_(True)
        y = y0.detach().requires_grad_(True)
        g = rec.segment(lambda: s * y, y=y)
        go = torch.rand_like(y0)
        gdg, = rec.segment(lambda: torch.autograd.grad(g, y, grad_outputs=go), go=go)
    res = rec.finish(f, g, gdg)
    assert res is not None, rec.reason
    return res[0]


prog = record_program()
_t = time.perf_counter()
_cabi.check(_cabi.compile_pointwise(prog, torch.float32), 'compile')
compile_ms = (time.perf_counter() - _t) * 1e3
sets = [{k: torch.rand(B, D, device=dev) + 0.5 for k in ('y0', 'y1')} for _ in range(NSET)]


def fused(s_in, s_out):
    _cabi.check(lib.tsde_step_milstein_pointwise(ctypes.byref(L), ctypes.byref(nz), ctypes.byref(prog), P(s_in), P(t0),
                                                 dt, 1, P(s_out)), 'fused')


series = [torch.empty(_cabi.PW_MAX_STEPS, B, D, device=dev) for _ in range(2)]


def chunk(k, y0, rows, cell_step=1):
    steps = (_cabi.PwStep * k)()
    for j, st in enumerate(steps):
        st.cell_id, st.h, st.dt, st.t0, st.y1 = 7 + cell_step * j, dt, dt, P(t0), P(rows[j])
    _cabi.check(lib.tsde_solve_milstein_pointwise(ctypes.byref(L), ctypes.byref(nz), ctypes.byref(prog), P(y0), steps,
                                                  k, 1), 'chunk')


def timed_chunk(k, chained, cell_step=1):
    """Microseconds per launch of a k-step chunk, graph-captured."""
    def issue():
        for i in range(REPS):
            src, dst = series[i % 2], series[(i + 1) % 2]
            chunk(k, src[k - 1] if chained else sets[i % NSET]['y0'], dst, cell_step)
    return timed_issue(issue)


def timed_fill():
    """Microseconds per 16 MiB row of torch's fill_ of one whole output series."""
    def issue():
        for i in range(REPS):
            series[i % 2].fill_(float(i))
    return timed_issue(issue) / _cabi.PW_MAX_STEPS


def seed(s_in, s_out):
    _cabi.check(lib.tsde_milstein_vjp_seed(ctypes.byref(L), ctypes.byref(nz), P(s_in), dt, 1, P(s_out)), 'seed')


def timed(launch, chained):
    """Microseconds per launch, graph-captured."""
    def issue():
        for i in range(REPS):
            if chained:
                a, b = sets[0]['y0'], sets[0]['y1']
                launch(a, b) if i % 2 == 0 else launch(b, a)
            else:
                s = sets[i % NSET]
                launch(s['y0'], s['y1'])
    return timed_issue(issue)


def timed_issue(issue):
    """Microseconds per launch of REPS launches `issue()`, graph-captured."""
    issue()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.stream = torch.cuda.current_stream(dev).cuda_stream  # launch on the capturing stream
        issue()
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


def gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        q = q.stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else None
    except Exception:
        return None


nbytes = 2 * D * 4 * B
out = {'gpu': gpu(), 'B': B, 'D': D, 'program': {'instructions': prog.n_instr, 'registers': prog.n_regs},
       'algorithmic_bytes_per_launch': nbytes, 'compile_ms': round(compile_ms, 1)}
DATASHEET_GBPS = 3350.0
for name, launch, chained in (('fused_cold', fused, False), ('fused_in_situ', fused, True), ('seed_cold', seed, False)):
    us = timed(launch, chained)
    out[name] = {'us': round(us, 2), 'GBps': round(nbytes / (us * 1e-6) / 1e9, 1)}
fill_us = timed_fill()
fill_gbps = B * D * 4 / (fill_us * 1e-6) / 1e9
out['fill'] = {'us_per_row': round(fill_us, 2), 'GBps': round(fill_gbps, 1)}
for k in (1, 8, 16, 32, 64, 128):
    if k > _cabi.PW_MAX_STEPS:
        out[f'chunk_{k}'] = 'exceeds TSDE_PW_MAX_STEPS'
        continue
    for grid, cell_step in (('', 1), ('table_', 2)):
        if grid and k == 1:  # (a one-step chunk is always uniform)
            continue
        for mode, chained in (('in_situ', True), ('cold', False)):
            us = timed_chunk(k, chained, cell_step)
            gbps = k * B * D * 4 / (us * 1e-6) / 1e9
            out[f'chunk_{k}_{grid}{mode}'] = {'us_per_step': round(us / k, 2), 'write_GBps': round(gbps, 1),
                                              'of_datasheet': round(gbps / DATASHEET_GBPS, 3),
                                              'of_fill': round(gbps / fill_gbps, 3)}
print(json.dumps(out), flush=True)
