"""Restatement of the reference's adaptive time loop with its proposal history, for checking `sdeint(adaptive=True)`.

`integrate_adaptive` is oracle/solvers.integrate_adaptive (the reference's base_solver.py:117-142 and
adaptive_stepping.py) with two differences that this library makes too:
  * the time arithmetic is done in the dtype of `ts` (numpy scalars of that dtype; under NumPy 2 a float32 scalar
    plus a Python float stays float32, as a 0-d float32 CPU tensor does in BaseSDESolver._integrate_adaptive);
  * the error estimate is formed in float64 whatever the state's dtype (`error_estimate`), where the reference forms
    it in the state dtype.
Each proposal is recorded as a `Proposal` (curr_t, next_t, midpoint_t, error, accepted, hit_dt_min).

Two modes:
  * free    the restatement makes its own accept / reject decisions and step sizes.  `snap` (a GPU history) lets it
            adopt the GPU's next_t of the same proposal when its own lies within SNAP_REL of it: the step size is a
            continuous function of the error estimate, which the GPU and the restatement round differently, so the
            times may differ in the last bits; snapping keeps one such difference from shifting every later query.
            The decisions stay the restatement's own, and the largest snapped deviation is reported (`snapped`).
  * driven  the restatement follows a given history: its times and decisions are taken from it, and only states and
            error estimates are computed.  Once the history is fixed rows are independent, so a driven solve can
            restate a sample of global rows, and it is a smooth function of y0 and the parameters.

Increments (`increments`), in forward time, with every query recorded in order:
  * float64: the interval-tree oracle of tests/test_gpu_brownian_paths.py (`_TreeOracle`), which walks the interval's
    own tree and evaluates each piece from the oracle's Philox normals (oracle/philox.py), so it answers only queries
    the GPU solve made;
  * float32, small batches: the increments the float32 interval itself returns, widened to float64 (a float32 and a
    float64 interval with the same entropy draw different normals), as tests/test_gpu_generic_adjoint.py does;
  * float32, sampled rows of a large batch (`rows=`): the tree oracle again, on the float32 specification of the
    normals of those global rows only (`philox.normals(row_ids=...)`).

Test infrastructure only; like oracle/ it does not import torchsde_b200 (the tree oracle is imported when asked for).
"""
import collections

import numpy as np

from oracle import solvers

Proposal = collections.namedtuple('Proposal', 'curr_t next_t midpoint_t error accepted hit_dt_min')
EPS = 1e-7
SNAP_REL = 1e-12


def error_estimate(y11, y12, rtol, atol, eps=EPS):
    """compute_error of adaptive_stepping.py:42-76, in float64."""
    y11 = np.asarray(y11, np.float64)
    y12 = np.asarray(y12, np.float64)
    tol = np.maximum(rtol * np.maximum(np.abs(y11), np.abs(y12)) + atol, eps)
    x = (y11 - y12) / tol
    return float(max(np.sqrt((x ** 2).sum() / x.size), eps))


def linear_interp(t0, y0, t1, y1, t):
    """interp.py:15-18, weights in the dtype of the times."""
    return solvers.linear_interp(t0, y0, t1, y1, t)


def propose(solver, curr_t, next_t, midpoint_t, y, extra):
    """The full step and the two half steps of one proposal (base_solver.py:122-125)."""
    y_full, _ = solver.step(curr_t, next_t, y, extra)
    mid_y, mid_extra = solver.step(curr_t, midpoint_t, y, extra)
    y_next, next_extra = solver.step(midpoint_t, next_t, mid_y, mid_extra)
    return y_full, y_next, next_extra


class Result:
    """ys, the final extra state, the history, the per-proposal states (y_full, y_next) when asked for, and the
    largest relative deviation of a snapped time (free mode)."""

    def __init__(self, ys, extra, history, states, snapped):
        self.ys, self.extra, self.history, self.states, self.snapped = ys, extra, history, states, snapped


def integrate_adaptive(solver, y0, ts, rtol, atol, dt_min, driven=None, snap=None, keep_states=False, extra0=None):
    """The adaptive loop on `solver` (an oracle/solvers.Solver whose bm is `increments`' query).  `driven`: a history
    (list of Proposal) to follow; `snap`: a history whose next_t free mode may adopt (module docstring)."""
    ts = np.asarray(ts)
    tt = ts.dtype.type
    step_size = solver.dt
    prev_t = curr_t = ts[0]
    prev_y = curr_y = y0
    curr_extra = solver.init_extra(ts[0], y0) if extra0 is None else extra0
    ys = [y0]
    prev_error_ratio = None
    history, states, snapped = [], [], 0.0
    for out_t in ts[1:]:
        while curr_t < out_t:
            k = len(history)
            if driven is not None:
                if k >= len(driven):
                    raise AssertionError(f'the driving history ends after {k} proposals before t = {float(out_t)}')
                h = driven[k]
                if float(h.curr_t) != float(curr_t):
                    raise AssertionError(f'proposal {k}: the history starts at {h.curr_t!r}, the solve is at '
                                         f'{float(curr_t)!r}')
                next_t, midpoint_t = tt(h.next_t), tt(h.midpoint_t)
            else:
                next_t = min(curr_t + step_size, ts[-1])
                if snap is not None and k < len(snap) and float(snap[k].curr_t) == float(curr_t):
                    dev = abs(float(next_t) - float(snap[k].next_t)) / max(abs(float(next_t)), 1e-300)
                    if dev <= SNAP_REL:
                        snapped = max(snapped, dev)
                        next_t = tt(snap[k].next_t)
                midpoint_t = tt(0.5 * (curr_t + next_t))
            y_full, y_next, next_extra = propose(solver, curr_t, next_t, midpoint_t, curr_y, curr_extra)
            err = error_estimate(y_full, y_next, rtol, atol)
            if keep_states:
                states.append((y_full, y_next))
            if driven is not None:
                accepted, hit = bool(driven[k].accepted), bool(driven[k].hit_dt_min)
            else:
                step_size, prev_error_ratio = solvers.update_step_size(err, step_size,
                                                                       prev_error_ratio=prev_error_ratio)
                hit = step_size < dt_min
                if hit:
                    step_size = dt_min
                    prev_error_ratio = None
                accepted = err <= 1 or step_size <= dt_min
            history.append(Proposal(float(curr_t), float(next_t), float(midpoint_t), err, accepted, hit))
            if accepted:
                prev_t, prev_y = curr_t, curr_y
                curr_t, curr_y, curr_extra = next_t, y_next, next_extra
        ys.append(linear_interp(prev_t, prev_y, curr_t, curr_y, out_t))
    if driven is not None and len(history) != len(driven):
        raise AssertionError(f'the solve ended after {len(history)} of the history\'s {len(driven)} proposals')
    return Result(np.stack(ys, axis=0), curr_extra, history, states, snapped)


def queries_of(history):
    """The Brownian queries a history makes: full step, first half step, second half step, per proposal."""
    out = []
    for h in history:
        out += [(h.curr_t, h.next_t), (h.curr_t, h.midpoint_t), (h.midpoint_t, h.next_t)]
    return out


def times_of(queries):
    """The proposal times (curr_t, next_t, midpoint_t) of a solve's Brownian queries, three per proposal, as a history
    whose errors and decisions are unknown (None): what `snap` reads."""
    assert len(queries) % 3 == 0, len(queries)
    return [Proposal(queries[k][0], queries[k][1], queries[k + 1][1], None, None, None)
            for k in range(0, len(queries), 3)]


def increments(bm, npdt, rows=None):
    """The restatement's bm(ta, tb[, return_U]) for the torchsde_b200 BrownianInterval `bm`, and the list of queries
    it answered (module docstring).  `rows`: global rows to restate (float32 large batches)."""
    asked = []
    if npdt == np.float32 and rows is None:
        def raw(ta, tb, want_u):
            out = bm(float(ta), float(tb), return_U=want_u)
            return tuple(x.double().cpu().numpy() for x in out) if want_u else out.double().cpu().numpy()
    else:
        from .test_gpu_brownian_paths import Src, _TreeOracle
        tree = _TreeOracle(bm, npdt)
        if rows is not None:
            tree.src = Src(len(rows), npdt, bm._row_offset, row_ids=np.asarray(rows, np.int64), key=bm._key)
        shape = (bm._rows if rows is None else len(rows), bm._m)

        def raw(ta, tb, want_u):
            if float(ta) == float(tb):
                # an empty interval, which the Brownian motion answers with zeros without splitting its tree: a
                # proposal one ulp long has a midpoint that rounds onto one of its ends
                return (np.zeros(shape), np.zeros(shape)) if want_u else np.zeros(shape)
            W, U, _ = tree.query(float(ta), float(tb))
            return (W.v, U.v) if want_u else W.v

    def query(ta, tb, return_U=False):
        asked.append((float(ta), float(tb)))
        return raw(ta, tb, return_U)
    return query, asked
