"""CUDA-graph time loop.

The reference's `integrate` (torchsde/_core/base_solver.py:107-147) is a Python loop with two or
three host<->device syncs per step.  Here the *whole solve* — for every step {user f/g as ordinary
torch ops (and Milstein's autograd vjp) -> fused tableau kernels} — is captured once into a CUDA
graph and replayed per call, so a solve costs one graph launch: no Python, no launch gaps beyond
the graph's own dependencies, `ys[i]` written in place by the step that produces it.

What makes this possible (and what it requires):
* the time grid is planned on the host (schedule.py) and all per-step scalars are launch arguments;
* the Brownian increments come from the Philox counter: per call only the 8-byte key changes, and
  the kernels read it from a static device buffer that is refreshed before each replay;
* `y0` (and a solver's extra state) are copied into static buffers before each replay;
* `f`/`g` must be pure functions of (t, y) and of tensors that are updated *in place*
  (nn.Parameters, buffers): their addresses are baked into the graph.  Host-side control flow on
  tensor values (`.item()`, `float(t)`) inside f/g cannot be captured; such SDEs run with the
  default eager loop.

Enable with ``options={'cuda_graph': True}``.

Ownership of the result.  A captured graph writes into buffers whose addresses are baked in, so the plan owns
one output series `ys` (T x B x D).  By default `sdeint` returns a *copy* of it (a fresh tensor, the reference's
semantics: results of successive solves never alias).  ``options={'cuda_graph': True, 'static_output': True}``
returns the plan's buffer itself — no copy (for cfg2 the copy would move 2 x 16.8 GB) — and
the caller must consume it before the next solve that reuses the plan overwrites it (the usual contract of
CUDA-graph inference engines).  `bench.py` uses the static output and says so in its JSON line.

Plan cache.  Plans are cached per *user SDE object* (the innermost object behind ForwardSDE / SDELogqp /
RenameMethodsSDE wrappers, which are re-created on every call) and keyed by (wrapper kinds, method, parameter
addresses, shapes, dtype, grid, dt, Brownian structure).  The cache is a WeakKeyDictionary and a plan keeps NO
reference to the SDE (only tensors and the graph), so dropping the SDE frees its plans — each of which pins a
full output series, hence also the small bound MAX_PLANS_PER_SDE.
"""
import contextlib
import gc
import weakref

import torch

from . import base_solver
from . import schedule as schedule_lib
from .._cabi import nvtx_range as _nvtx

_PLANS = weakref.WeakKeyDictionary()
MAX_PLANS_PER_SDE = 4  # every plan owns its output series (T x B x D): keep the cache small


def plans_of(cache, sde_obj):
    """The per-object plan dict, or None for an SDE object that can be neither hashed nor weakly referenced
    (a class with `__slots__`, or `__eq__` without `__hash__`): such objects run without a cached plan."""
    try:
        return cache.setdefault(sde_obj, {})
    except TypeError:
        return None


def _remember(plans, key, plan):
    while len(plans) >= MAX_PLANS_PER_SDE:
        plans.pop(next(iter(plans)))  # oldest first (dicts keep insertion order)
    plans[key] = plan


class _Plan:
    pass


def drop_plans(sde):
    """Release every cached forward plan of `sde` (each pins a full output series in device memory)."""
    owner, _ = cache_owner(sde)
    try:
        _PLANS.pop(owner, None)
    except TypeError:
        pass


def _tensor_signature(obj):
    """Addresses (and shapes / dtypes) of the tensors an SDE object owns.  A captured graph has them baked in, so a
    plan must not be replayed after `sde.to(...)`, `sde.double()` or `sde.mu = nn.Parameter(...)` replaced them;
    in-place updates (optimiser steps, `load_state_dict`) keep the addresses and keep the plan valid."""
    if isinstance(obj, torch.nn.Module):
        tensors = list(obj.parameters()) + list(obj.buffers())
    else:
        tensors = [v for v in vars(obj).values() if torch.is_tensor(v)] if hasattr(obj, '__dict__') else []
    return tuple((t.data_ptr(), tuple(t.shape), t.dtype) for t in tensors)


def cache_owner(sde):
    """(innermost user object, tags of the wrappers around it).  `sdeint` wraps the user's SDE afresh on every call
    (ForwardSDE always; SDELogqp for logqp=True; RenameMethodsSDE for names=...), so the wrapper objects cannot
    key a cache: plans hang on the user's own object, and the wrapper chain is part of the plan key."""
    tags = []
    obj = sde
    while hasattr(obj, '_base_sde'):
        tags.append(getattr(obj, '_plan_tag', type(obj).__name__))
        obj = obj._base_sde
    return obj, tuple(tags)


def _plan_key(solver, y0, ts, extra0, binding):
    node = binding.node
    owner, tags = cache_owner(solver.sde)
    return (type(solver).__name__, tags, _tensor_signature(owner),
            tuple(y0.shape), y0.dtype, str(y0.device),
            schedule_lib.ts_values(ts), str(ts.dtype),
            float(solver.dt) if not torch.is_tensor(solver.dt) else float(solver.dt),
            tuple(sorted((k, repr(v)) for k, v in solver.options.items() if k != 'static_output')),
            solver.bm.levy_area_approximation, tuple(solver.bm.shape),
            node.cell_base, tuple(binding.first), tuple(binding.count), binding.reverse,
            binding.interval._row_offset,
            tuple((tuple(e.shape), e.dtype) for e in extra0),
            # f / g may return 16-bit tensors under autocast, and the captured launches have their formats baked in
            torch.is_autocast_enabled('cuda'), torch.get_autocast_dtype('cuda'))


def uncached_autocast():
    """The caller's CUDA autocast state, without its cast cache, for warm-up and capture: a cached 16-bit copy of a
    parameter lives only as long as the caller's autocast region, while the graph reads it on every later replay."""
    if not torch.is_autocast_enabled('cuda'):
        return contextlib.nullcontext()
    return torch.autocast('cuda', dtype=torch.get_autocast_dtype('cuda'), cache_enabled=False)


@contextlib.contextmanager
def no_gc():
    """No cyclic garbage collection while a graph is captured.  A collection can free an unreachable SDE object, and
    with it the CUDA graphs of its cached plans; destroying a graph while a stream captures invalidates the capture
    (and leaves torch's CUDA generator in capture mode).  Which allocation triggers a collection is arbitrary."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if enabled:
            gc.enable()


def _hand_out(plan, solver, static_ok):
    """The plan's output series, or a copy of it (see the module docstring)."""
    if static_ok or solver.options.get('static_output', False):
        return plan.ys, plan.extra_out
    return plan.ys.clone(), tuple(e.clone() for e in plan.extra_out)


LAST_PLAN = None  # the plan replayed most recently (bench.py reads its launch count)


def integrate_captured(solver, y0, ts, extra0, static_ok=False):
    global LAST_PLAN
    if int(solver.options.get('row_split', 1)) > 1 and not extra0:
        return _integrate_captured_split(solver, y0, ts, static_ok)
    sde_obj, _ = cache_owner(solver.sde)
    sched = schedule_lib.get_schedule(ts, solver.dt)
    y0 = base_solver._contig(y0.detach())
    solver._prepare(y0)
    binding = solver._bind(sched)
    if binding is None or solver.adaptive:
        # arbitrary Brownian objects keep host-side state per query: not replayable
        return solver.integrate(y0, ts, extra0)
    extra0 = tuple(base_solver._contig(e.detach()) for e in extra0)
    key = _plan_key(solver, y0, ts, extra0, binding)
    plans = plans_of(_PLANS, sde_obj)
    if plans is None:
        return solver.integrate(y0, ts, extra0)  # nothing to hang the plan on: ordinary eager loop
    plan = plans.get(key)
    if plan is None and key not in plans:
        try:
            with _nvtx('tsde: capture solve'):
                plan = _capture(solver, sched, binding, y0, ts, extra0)
        except RuntimeError as e:
            # f / g did something a stream capture cannot record (a host sync or a host<->device copy — e.g.
            # `.item()` in user code, or `pinverse` in the KL rate of a general-noise logqp=True solve whose (d, m)
            # is over tsde_logqp_augment's bound).  Such SDEs run with the ordinary eager loop; remember it so that
            # the capture is not attempted on every call.
            if 'captur' not in str(e).lower():
                raise
            import warnings
            warnings.warn("torchsde_b200: this SDE's f/g cannot be captured into a CUDA graph "
                          f"({str(e).splitlines()[0][:160]}); falling back to the eager time loop.")
            torch.cuda.synchronize(y0.device)
            plan = None
        _remember(plans, key, plan)
    if plan is None:
        return solver.integrate(y0, ts, extra0)
    plan.y0.copy_(y0)
    plan.key.copy_(binding.interval.key_tensor())
    for dst, src in zip(plan.extra_in, extra0):
        dst.copy_(src)
    with _nvtx('tsde: replay solve'):
        plan.graph.replay()
    LAST_PLAN = plan
    return _hand_out(plan, solver, static_ok)


def _capture(solver, sched, binding, y0, ts, extra0):
    from .. import _cabi
    plan = _Plan()
    dev = y0.device
    plan.binding = binding  # keeps the grid node (and its device-side cell lengths) alive
    plan.y0 = torch.empty_like(y0)
    plan.key = torch.empty(1, dtype=torch.int64, device=dev)
    plan.extra_in = tuple(torch.empty_like(e) for e in extra0)
    T = ts.numel()
    plan.ys = torch.empty((T, solver.rows, solver.d), dtype=solver.dtype, device=dev)
    plan.y0.copy_(y0)
    plan.key.copy_(binding.interval.key_tensor())
    for dst, src in zip(plan.extra_in, extra0):
        dst.copy_(src)

    feed = base_solver.NoiseFeed(solver, solver.bm, binding)
    feed._key_ptr = plan.key.data_ptr()  # kernels read the key from the static buffer
    solver._feed = feed
    ctxs = solver._contexts(sched, ts)
    # the 0-d time tensors handed to the user's f/g are views of this table: it must outlive the graph.  Nothing
    # else of the solver is kept (launch descriptors and scalars were copied into the kernel nodes at capture
    # time), in particular no reference to the SDE: see the module docstring.
    plan.time_table = getattr(solver, '_time_table', None)

    def body():
        plan.ys[0].copy_(plan.y0)
        return solver._run(sched, ctxs, plan.ys, plan.extra_in)

    # Warm-up on a side stream (lazy initialisations: cuBLAS handles, autograd, allocator)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side), torch.no_grad(), uncached_autocast():
        plan.ys[0].copy_(plan.y0)
        n_warm = min(3, sched.n_steps)
        if n_warm:
            class _Few:
                pass
            few = _Few()
            few.aligned_row = lambda k: None
            few.outputs_after = {}
            ys_tmp = plan.ys
            solver._run(few, ctxs[:n_warm], ys_tmp, plan.extra_in)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)

    graph = torch.cuda.CUDAGraph()
    launches0 = _cabi.LAUNCHES
    with no_gc(), torch.no_grad(), torch.cuda.graph(graph), uncached_autocast():
        extra_out = body()
    plan.abi_launches = _cabi.LAUNCHES - launches0  # kernels of THIS library captured in the graph (per replay)
    plan.graph = graph
    plan.extra_out = tuple(extra_out)
    return plan


# ---- row-split pipelining ------------------------------------------------------------------------
# options={'cuda_graph': True, 'row_split': k}: the batch is cut into k contiguous row blocks that are
# captured as k *independent chains* of one graph (fork/join on k streams).  Trajectories never interact
# (same property that lets the batch shard over GPUs, SURVEY §8e) and the Brownian rows are keyed by their
# global index, so the result is bit-identical; what changes is that while one chain's kernel drains or the
# next one ramps up, the other chain's kernel keeps the SMs busy (per-kernel fixed cost ~3 us on 16 MiB tensors).
# Requires f/g to act row-wise on (t, y) — true for any SDE whose trajectories are independent.
def _integrate_captured_split(solver, y0, ts, static_ok=False):
    global LAST_PLAN
    k = int(solver.options['row_split'])
    sde_obj, _ = cache_owner(solver.sde)
    sched = schedule_lib.get_schedule(ts, solver.dt)
    y0 = base_solver._contig(y0.detach())
    solver._prepare(y0)
    binding = solver._bind(sched)
    if binding is None or y0.shape[0] < k:
        opts = dict(solver.options)
        opts.pop('row_split')
        solver.options = opts
        return integrate_captured(solver, y0, ts, (), static_ok)
    key = ('split', k) + _plan_key(solver, y0, ts, (), binding)
    plans = plans_of(_PLANS, sde_obj)
    if plans is None:
        return solver.integrate(y0, ts, ())
    plan = plans.get(key)
    if plan is None and key not in plans:
        plan = _capture_split(solver, sched, binding, y0, ts, k)
        _remember(plans, key, plan)
    if plan is None:  # (f / g cannot be captured: the ordinary eager loop, as integrate_captured falls back)
        return solver.integrate(y0, ts, ())
    plan.y0.copy_(y0)
    plan.key.copy_(binding.interval.key_tensor())
    plan.graph.replay()
    LAST_PLAN = plan
    return _hand_out(plan, solver, static_ok)


def _capture_split(solver, sched, binding, y0, ts, k):
    """The plan of a row-split solve: k row blocks captured as k chains of one graph; None (with a warning) when f / g
    do something a stream capture cannot record, as `integrate_captured` does for an unsplit solve."""
    import copy
    from .. import _cabi
    plan = _Plan()
    dev = y0.device
    B = y0.shape[0]
    plan.binding = binding
    plan.y0 = y0.clone()
    plan.key = binding.interval.key_tensor().clone()
    T = ts.numel()
    # (k, T, rows_i, d) blocks so that every chain writes contiguous rows; returned as one (T, B, d) view
    plan.ys = torch.empty((T, B, solver.d), dtype=solver.dtype, device=dev)
    bounds = [(B * i) // k for i in range(k + 1)]
    subs = []
    for i in range(k):
        sub = copy.copy(solver)
        sub._side_streams = []
        sub._err_buf = None
        lo, hi = bounds[i], bounds[i + 1]
        sub._prepare(plan.y0[lo:hi])
        feed = base_solver.NoiseFeed(sub, solver.bm, binding)
        feed._key_ptr = plan.key.data_ptr()
        feed._row_offset = binding.interval._row_offset + lo
        sub._feed = feed
        sub_ctxs = sub._contexts(sched, ts)
        subs.append((sub, sub_ctxs, lo, hi))
    plan.time_table = [getattr(sub, '_time_table', None) for sub, _, _, _ in subs]  # (no reference to the sub-solvers / the SDE)
    streams = [torch.cuda.Stream(device=dev) for _ in range(k - 1)]

    def body(n_steps=None):
        main = torch.cuda.current_stream(dev)
        plan.ys[0].copy_(plan.y0)
        for j, (sub, sub_ctxs, lo, hi) in enumerate(subs):
            st = main if j == 0 else streams[j - 1]
            if st is not main:
                st.wait_stream(main)
            with torch.cuda.stream(st):
                view = plan.ys[:, lo:hi]
                if n_steps is None:
                    sub._run(sched, sub_ctxs, view, ())
                else:
                    class _Few:
                        aligned_row = staticmethod(lambda kk: None)
                        outputs_after = {}
                    sub._run(_Few, sub_ctxs[:n_steps], view, ())
        for st in streams:
            main.wait_stream(st)

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side), torch.no_grad(), uncached_autocast():
        body(min(3, sched.n_steps))
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    launches0 = _cabi.LAUNCHES
    try:
        with no_gc(), torch.no_grad(), torch.cuda.graph(graph), uncached_autocast():
            body()
    except RuntimeError as e:
        if 'captur' not in str(e).lower():
            raise
        import warnings
        warnings.warn("torchsde_b200: this SDE's f/g cannot be captured into a CUDA graph "
                      f"({str(e).splitlines()[0][:160]}); falling back to the eager time loop.")
        torch.cuda.synchronize(dev)
        return None
    plan.abi_launches = _cabi.LAUNCHES - launches0
    plan.graph = graph
    plan.extra_out = ()
    return plan
