"""BrownianInterval: host-side interval tree + device-side counter-based evaluation.

Drop-in for ``torchsde.BrownianInterval`` (reference: torchsde/_brownian/brownian_interval.py).
Same constructor (:394-408), same ``__call__(ta, tb=None, return_U=False, return_A=False)``
contract (:589-687: clamping + warnings :598-609, RuntimeError on ta > tb :610-611, zero
increments for ta == tb :613-621, aggregation of several sub-intervals :643-672, U = h(W/2+H)
:674-676) and the same properties (:744-785).

What is different is *where the numbers come from*.  The reference stores, per tree node, seeds
for ``torch.Generator`` and caches (batch, m) tensors of every visited node.  Here the tree holds
no tensors at all: every node owns a 64-bit id, and any node's (W, H) is a pure function
    (key(entropy), ids along the path, row, channel)  ->  value
evaluated on the GPU by Philox4x32-10 (csrc/philox.cuh).  Three node kinds exist:

* LEAF    not split yet.
* BINARY  split at ``mid`` into two children whose (W,H) are the reference's Brownian-bridge
          functions of the parent's (W,H) and two normals X1,X2 (:188-241)  -> tsde_brownian_bridge.
* GRID    split into N consecutive *primary cells* whose (W,H) are independent direct draws
          W ~ N(0,h), H ~ N(0,h/12) (the law used for the top interval, :551-558); the node's own
          value is the exact left-to-right merge of its cells (:643-672).  A fixed-step solver
          binds its step grid as a GRID node, so step k needs exactly one Philox draw per
          channel — generated in registers inside the fused tableau kernel, never stored.
          This is the O(1)-per-step replacement of the reference's dependency tree
          (``_create_dependency_tree`` :689-712) + LRU cache (:114-126).

Any query is decomposed into nodes / runs of whole cells exactly as ``_loc`` does (:271-315);
a query strictly inside a cell bridges inside that cell, so the path stays consistent for
arbitrary, repeated and out-of-order queries (tests/test_brownian_interval.py:261-288).

``halfway_tree=True`` never creates GRID nodes: the tree is the dyadic tree and ids are
structural, so the sample path is a function of ``entropy`` alone (:536-540).
"""
import bisect
import ctypes
import math
import warnings

import numpy as np
import torch

from . import brownian_base
from .. import _cabi
from ..settings import LEVY_AREA_APPROXIMATIONS

_MASK64 = (1 << 64) - 1
_LEAF, _BINARY, _GRID = 0, 1, 2
# channels of one row: channel / 4 is a 24-bit field of the Philox counter (csrc/philox.cuh); the library refuses more
MAX_CHANNELS = 1 << 26


def mix64(x):
    """splitmix64 finaliser (public-domain constant set); bijective on 64 bits."""
    x &= _MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _MASK64
    return x ^ (x >> 31)


def child_id(parent_id, index):
    return mix64((parent_id + 0x9E3779B97F4A7C15 * (index + 1)) & _MASK64)


def key_from_entropy(entropy):
    """Fold an arbitrary Python int into the 64-bit Philox key."""
    e = int(entropy)
    sign = 1 if e < 0 else 0
    e = abs(e)
    k = mix64(0x5851F42D4C957F2D + sign)
    while True:
        k = mix64(k ^ (e & _MASK64))
        e >>= 64
        if e == 0:
            break
    return k


_ROOT_ID = mix64(0x746F7263687364)  # "torchsd"


def _is_scalar(x):
    return isinstance(x, int) or isinstance(x, float) or (isinstance(x, torch.Tensor) and x.numel() == 1)


def _assert_floating_tensor(name, tensor):
    if not torch.is_tensor(tensor):
        raise ValueError(f"{name}={tensor} should be a Tensor.")
    if not tensor.is_floating_point():
        raise ValueError(f"{name}={tensor} should be floating point.")


def _check_tensor_info(*tensors, size, dtype, device):
    """Same contract as brownian_interval.py:46-75."""
    tensors = list(filter(torch.is_tensor, tensors))
    if dtype is None and len(tensors) == 0:
        dtype = torch.get_default_dtype()
    if device is None and len(tensors) == 0:
        # the reference says "cpu" here (brownian_interval.py:50-51); torch's default device IS the cpu unless the
        # user changed it with torch.set_default_device, which factory code written today is expected to honour
        device = torch.get_default_device() if hasattr(torch, 'get_default_device') else torch.device("cpu")
    sizes = [] if size is None else [size]
    sizes += [t.shape for t in tensors]
    dtypes = [] if dtype is None else [dtype]
    dtypes += [t.dtype for t in tensors]
    devices = [] if device is None else [device]
    devices += [t.device for t in tensors]
    if len(sizes) == 0:
        raise ValueError("Must either specify `size` or pass in `W` or `H` to implicitly define the size.")
    if not all(tuple(i) == tuple(sizes[0]) for i in sizes):
        raise ValueError("Multiple sizes found. Make sure `size` and `W` or `H` are consistent.")
    if not all(i == dtypes[0] for i in dtypes):
        raise ValueError("Multiple dtypes found. Make sure `dtype` and `W` or `H` are consistent.")
    def _norm(dv):
        dv = torch.device(dv)
        if dv.type == 'cuda' and dv.index is None and torch.cuda.is_available():
            dv = torch.device('cuda', torch.cuda.current_device())
        return dv
    if not all(_norm(i) == _norm(devices[0]) for i in devices):
        raise ValueError("Multiple devices found. Make sure `device` and `W` or `H` are consistent.")
    return tuple(sizes[0]), dtypes[0], devices[0]


class _LRU(dict):
    """brownian_interval.py:114-126."""

    def __init__(self, max_size):
        super().__init__()
        self._max_size = max_size
        self._keys = []

    def __setitem__(self, key, value):
        if key in self:
            self._keys.remove(key)
        elif len(self) >= self._max_size:
            del self[self._keys.pop(0)]
        super().__setitem__(key, value)
        self._keys.append(key)


class _Node:
    __slots__ = ('start', 'end', 'parent', 'id', 'kind', 'mid', 'left', 'right', 'is_left',
                 'bounds', 'cells', 'cell_index', 'cell_base', 'cell_h_dev')

    def __init__(self, start, end, parent, node_id, is_left=None, cell_index=None):
        self.start = start
        self.end = end
        self.parent = parent
        self.id = node_id
        self.kind = _LEAF
        self.mid = None
        self.left = None
        self.right = None
        self.is_left = is_left
        self.bounds = None
        self.cells = None
        self.cell_index = cell_index  # not None: primary cell of a GRID parent
        self.cell_base = None
        self.cell_h_dev = None

    def cell(self, k):
        c = self.cells.get(k)
        if c is None:
            c = _Node(self.bounds[k], self.bounds[k + 1], self, (self.cell_base + k) & _MASK64, cell_index=k)
            self.cells[k] = c
        return c


class GridBinding:
    """What a fixed-step solver needs to regenerate step k's increment in registers."""

    __slots__ = ('interval', 'node', 'first', 'count', 'bounds', 'reverse')

    def __init__(self, interval, node, first, count, bounds, reverse=False):
        self.interval = interval   # BrownianInterval
        self.node = node           # GRID node
        self.first = first         # first[k]: index of the first primary cell of step k
        self.count = count         # count[k]: number of primary cells merged in step k
        self.bounds = bounds       # solver step boundaries (python floats)
        self.reverse = reverse

    def reversed(self):
        return GridBinding(self.interval, self.node, self.first, self.count, self.bounds, not self.reverse)

    @property
    def n_steps(self):
        return len(self.first)

    def cell(self, k):
        """(counter id, length) of the first primary cell of solver step k, and the number of cells the step merges:
        what `fill` puts in cell_id, h and n_cells."""
        if self.reverse:
            k = len(self.first) - 1 - k
        i = self.first[k]
        return (self.node.cell_base + i) & _MASK64, self.node.bounds[i + 1] - self.node.bounds[i], self.count[k]

    def fill(self, nz, k, want_u, key_ptr, row_offset=0):
        """Fill a `_cabi.Noise` for solver step k (k counts in solver order; for a reversed
        binding the solver's step k is the forward grid's step n-1-k)."""
        if self.reverse:
            k = len(self.first) - 1 - k
        node = self.node
        i, n = self.first[k], self.count[k]
        nz.source = _cabi.SRC_COUNTER
        nz.want_u = 1 if want_u else 0
        nz.w = None
        nz.u = None
        nz.key = key_ptr
        nz.cell_id = (node.cell_base + i) & _MASK64
        nz.row_offset = row_offset
        nz.n_cells = n
        nz.h = node.bounds[i + 1] - node.bounds[i]
        nz.h_total = self.bounds[k + 1] - self.bounds[k]
        if n > 1:
            nz.cell_h = self.interval._cell_h_dev(node).data_ptr() + 8 * i
        else:
            nz.cell_h = None
        return nz


class BrownianInterval(brownian_base.BaseBrownian):
    """Brownian interval with fixed entropy (see module docstring)."""

    def __init__(self, t0=0., t1=1., size=None, dtype=None, device=None, entropy=None, dt=None, tol=0.,
                 pool_size=8, cache_size=45, halfway_tree=False,
                 levy_area_approximation=LEVY_AREA_APPROXIMATIONS.none, W=None, H=None):
        # --- brownian_interval.py:460-494 -------------------------------------------------------
        if not _is_scalar(t0):
            raise ValueError('Initial time t0 should be a float or 0-d torch.Tensor.')
        if not _is_scalar(t1):
            raise ValueError('Terminal time t1 should be a float or 0-d torch.Tensor.')
        if dt is not None and not _is_scalar(dt):
            raise ValueError('Expected average time step dt should be a float or 0-d torch.Tensor.')
        if t0 > t1:
            raise ValueError(f'Initial time {t0} should be less than terminal time {t1}.')
        t0 = float(t0)
        t1 = float(t1)
        if dt is not None:
            dt = float(dt)
        if halfway_tree:
            if tol <= 0.:
                raise ValueError("`tol` should be positive.")
            if dt is not None:
                raise ValueError("`dt` is not used and should be set to `None` if `halfway_tree` is True.")
        else:
            if tol < 0.:
                raise ValueError("`tol` should be non-negative.")
        size, dtype, device = _check_tensor_info(W, H, size=size, dtype=dtype, device=device)
        if entropy is None:
            entropy = np.random.randint(0, 2 ** 31 - 1)
        if levy_area_approximation not in LEVY_AREA_APPROXIMATIONS:
            raise ValueError(f"`levy_area_approximation` must be one of {LEVY_AREA_APPROXIMATIONS}, but got "
                             f"'{levy_area_approximation}'.")
        device = torch.device(device)
        self._size = size
        self._dtype = dtype
        self._device = device
        self._entropy = entropy
        self._levy_area_approximation = levy_area_approximation
        self._dt = dt
        self._tol = tol
        self._pool_size = pool_size  # accepted for API compatibility; the Philox key is always 64 bit
        self._cache_size = cache_size
        self._halfway_tree = halfway_tree

        if cache_size is None:
            self._cache = {}
        elif cache_size == 0:
            self._cache = None
        else:
            self._cache = _LRU(max_size=cache_size)

        self._have_H = levy_area_approximation in (LEVY_AREA_APPROXIMATIONS.space_time,
                                                   LEVY_AREA_APPROXIMATIONS.davie,
                                                   LEVY_AREA_APPROXIMATIONS.foster)
        self._have_A = levy_area_approximation in (LEVY_AREA_APPROXIMATIONS.davie,
                                                   LEVY_AREA_APPROXIMATIONS.foster)
        if tol == 0.:
            self._round = lambda x: x
        else:
            ndigits = -int(math.log10(tol))
            self._round = lambda x: round(x, ndigits)

        # (rows, m) view of `size`: rank >= 2 -> batch dims x channels; rank 1 -> one row of n
        # channels; rank 0 -> one row, one channel.  (Levy area treats rank 0/1 as batch, :81-84.)
        if len(size) >= 2:
            self._rows = int(np.prod(size[:-1]))
            self._m = int(size[-1])
        elif len(size) == 1:
            self._rows, self._m = 1, int(size[0])
        else:
            self._rows, self._m = 1, 1
        if self._m > MAX_CHANNELS:
            raise ValueError(f"BrownianInterval supports at most 2**26 channels (the last dimension of `size`), got "
                             f"{self._m}: the samples are drawn from a counter whose channel field has 26 bits, so "
                             f"further channels would repeat the normals of other channels.")

        self._key = key_from_entropy(entropy)
        self._key_dev = None
        self._row_offset = 0

        self._root = _Node(self._round(t0), self._round(t1), None, _ROOT_ID)
        self._last = self._root
        if W is not None:
            _assert_floating_tensor('W', W)
        if H is not None:
            _assert_floating_tensor('H', H)
        if dtype not in (torch.float32, torch.float64):
            # Integer dtypes fail in the reference's constructor as well (it draws the top-level increment eagerly and
            # `torch.randn` has no integer kernel, brownian_interval.py:30-32); half precision is not implemented here.
            raise NotImplementedError(f"BrownianInterval is implemented for torch.float32 and torch.float64, not {dtype}.")
        self._user_W = W
        self._user_H = H
        self._root_value = None  # (W, H) once observed

    # ------------------------------------------------------------------------------------------
    # device plumbing
    # ------------------------------------------------------------------------------------------
    def _require_cuda(self):
        if self._device.type != 'cuda':
            raise RuntimeError(
                "torchsde_b200.BrownianInterval generates its samples with CUDA kernels: construct it with "
                "device='cuda'. There is no CPU path (use the reference torchsde on CPU).")

    def key_tensor(self):
        if self._key_dev is None:
            self._require_cuda()
            k = self._key if self._key < (1 << 63) else self._key - (1 << 64)
            # (a fill kernel, not a host-to-device copy: creating an interval does not synchronise the host with the
            # work already queued on the device)
            self._key_dev = torch.full((1,), k, dtype=torch.int64, device=self._device)
        return self._key_dev

    def _launch(self):
        return _cabi.make_launch(self._dtype, _cabi.NOISE_DIAGONAL, self._rows, self._m, self._m, device=self._device)

    def _new(self, *extra):
        return torch.empty((self._rows, self._m, *extra), dtype=self._dtype, device=self._device)

    def _new_out(self, *extra):
        """An output buffer already in the caller-visible shape (same contiguous (rows, m[, m]) memory): the
        single-launch query paths hand it out as is, without a reshape."""
        return torch.empty((*self._size, *extra), dtype=self._dtype, device=self._device)

    def _cell_h_dev(self, node):
        if node.cell_h_dev is None:
            b = node.bounds
            h = [b[i + 1] - b[i] for i in range(len(b) - 1)]
            node.cell_h_dev = torch.tensor(h, dtype=torch.float64, device=self._device)
        return node.cell_h_dev

    # ------------------------------------------------------------------------------------------
    # node values
    # ------------------------------------------------------------------------------------------
    def _draw_cells(self, grid, i, n, h_total):
        """(W, H) of the merge of primary cells i..i+n-1 of GRID node `grid`."""
        self._require_cuda()
        nz = _cabi.Noise()
        nz.source = _cabi.SRC_COUNTER
        nz.want_u = 1 if self._have_H else 0
        nz.key = self.key_tensor().data_ptr()
        nz.cell_id = (grid.cell_base + i) & _MASK64
        nz.row_offset = self._row_offset
        nz.n_cells = n
        nz.h = grid.bounds[i + 1] - grid.bounds[i]
        nz.h_total = h_total
        nz.cell_h = self._cell_h_dev(grid).data_ptr() + 8 * i if n > 1 else None
        W = self._new()
        H = self._new() if self._have_H else None
        L = self._launch()
        _cabi.check(_cabi.lib().tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), W.data_ptr(), None,
                                                    None if H is None else H.data_ptr()),
                    "tsde_brownian_cells")
        return W, H

    def _draw_single(self, node_id, h):
        self._require_cuda()
        nz = _cabi.Noise()
        nz.source = _cabi.SRC_COUNTER
        nz.want_u = 1 if self._have_H else 0
        nz.key = self.key_tensor().data_ptr()
        nz.cell_id = node_id
        nz.row_offset = self._row_offset
        nz.n_cells = 1
        nz.h = h
        nz.h_total = h
        nz.cell_h = None
        W = self._new()
        H = self._new() if self._have_H else None
        L = self._launch()
        _cabi.check(_cabi.lib().tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), W.data_ptr(), None,
                                                    None if H is None else H.data_ptr()),
                    "tsde_brownian_cells")
        return W, H

    def _root_wh(self):
        """Top-level increment and space-time Levy area (:551-561), drawn lazily so that a solver
        can still bind its grid to a fresh interval."""
        if self._root_value is None:
            root = self._root
            if root.kind == _GRID:
                W, H = self._draw_cells(root, 0, len(root.bounds) - 1, root.end - root.start)
            else:
                W, H = self._draw_single(root.id, root.end - root.start)
                # A user-supplied W and/or H replaces the draw (:553-560).
                if self._user_W is not None:
                    self._require_cuda()
                    W = self._user_W.detach().to(self._dtype).reshape(self._rows, self._m).contiguous()
                if self._user_H is not None and self._have_H:
                    H = self._user_H.detach().to(self._dtype).reshape(self._rows, self._m).contiguous()
            self._root_value = (W, H)
        return self._root_value

    def _cache_get(self, node):
        if self._cache is None:
            return None
        return self._cache.get(node)

    def _cache_put(self, node, value):
        if self._cache is not None:
            self._cache[node] = value

    def _bridge(self, base_value, chain):
        """Descend `chain` (list of nodes, each a binary child of the previous / of the base)."""
        W0, H0 = base_value
        depth = len(chain)
        ids = (ctypes.c_uint64 * depth)()
        lefts = (ctypes.c_int32 * depth)()
        times = (ctypes.c_double * (3 * depth))()
        for l, node in enumerate(chain):
            p = node.parent
            ids[l] = p.id
            lefts[l] = 1 if node.is_left else 0
            times[3 * l], times[3 * l + 1], times[3 * l + 2] = p.start, p.mid, p.end
        W = self._new()
        H = self._new() if self._have_H else None
        L = self._launch()
        _cabi.check(_cabi.lib().tsde_brownian_bridge(
            ctypes.byref(L), self.key_tensor().data_ptr(), self._row_offset, depth, ids, lefts, times,
            W0.data_ptr(), None if H0 is None else H0.data_ptr(), W.data_ptr(),
            None if H is None else H.data_ptr()), "tsde_brownian_bridge")
        return W, H

    def _value(self, node):
        """(W, H) of an arbitrary tree node."""
        chain = []
        cur = node
        while True:
            if cur.parent is None:
                base = self._root_wh()
                break
            v = self._cache_get(cur)
            if v is not None:
                base = v
                break
            if cur.cell_index is not None:
                base = self._draw_cells(cur.parent, cur.cell_index, 1, cur.end - cur.start)
                self._cache_put(cur, base)
                break
            chain.append(cur)
            cur = cur.parent
        if not chain:
            return base
        chain.reverse()
        if len(chain) > 1:
            # materialise (and cache) the target's parent: sequential queries keep descending from it,
            # exactly the node the reference finds in its LRU cache (:190-194).
            base = self._bridge(base, chain[:-1])
            self._cache_put(chain[-2], base)
        out = self._bridge(base, chain[-1:])
        self._cache_put(node, out)
        return out

    # ------------------------------------------------------------------------------------------
    # tree manipulation (:271-350)
    # ------------------------------------------------------------------------------------------
    def _split_exact(self, node, midway):
        node.mid = self._round(midway)
        node.kind = _BINARY
        node.left = _Node(node.start, self._round(midway), node, child_id(node.id, 0), is_left=True)
        node.right = _Node(self._round(midway), node.end, node, child_id(node.id, 1), is_left=False)

    def _split(self, node, midway):
        if self._halfway_tree:
            while True:
                self._split_exact(node, 0.5 * (node.end + node.start))
                if midway > node.mid:
                    node = node.right
                elif midway < node.mid:
                    node = node.left
                else:
                    return
                if node.kind != _LEAF:
                    return
        else:
            self._split_exact(node, midway)

    def _locate(self, ta, tb):
        """Decompose [ta, tb] into tree pieces, left to right (the reference's `_loc`, :271-315).
        A piece is a `_Node`, or a tuple (grid_node, i, j): the merge of whole primary cells i..j-1."""
        node = self._last
        while ta < node.start or tb > node.end:
            node = node.parent
        out = []
        stack = [(node, ta, tb)]  # LIFO; sub-queries are pushed right-to-left so output is left-to-right
        while stack:
            node, a, b = stack.pop()
            if a is None:  # deferred run of whole cells
                out.append(node)
                continue
            while True:
                if a == node.start and b == node.end:
                    out.append(node)
                    break
                if node.kind == _LEAF:
                    self._split(node, b if a == node.start else a)
                if node.kind == _BINARY:
                    if b <= node.mid:
                        node = node.left
                    elif a >= node.mid:
                        node = node.right
                    else:
                        stack.append((node.right, node.mid, b))
                        b = node.mid
                        node = node.left
                    continue
                # GRID node: head partial cell, run of whole cells, tail partial cell
                bounds = node.bounds
                work = []
                i = bisect.bisect_right(bounds, a) - 1
                done = False
                if bounds[i] != a:
                    hi = min(b, bounds[i + 1])
                    work.append((node.cell(i), a, hi))
                    done = hi == b
                    i += 1
                if not done:
                    j = bisect.bisect_right(bounds, b) - 1
                    if j > i:
                        work.append(((node, i, j), None, None))
                    if bounds[j] != b:
                        work.append((node.cell(j), bounds[j], b))
                stack.extend(reversed(work))
                break
        return out

    # ------------------------------------------------------------------------------------------
    # queries (:589-687)
    # ------------------------------------------------------------------------------------------
    def __call__(self, ta, tb=None, return_U=False, return_A=False):
        with _cabi.device_guard(self._device):
            return self._call(ta, tb, return_U, return_A)

    def _call(self, ta, tb, return_U, return_A):
        if tb is None:
            warnings.warn(f"{self.__class__.__name__} is optimised for interval-based queries, not point evaluation.")
            ta, tb = self._root.start, ta
            tb_name = 'ta'
        else:
            tb_name = 'tb'
        ta = float(ta)
        tb = float(tb)
        start, end = self._root.start, self._root.end
        if ta < start:
            warnings.warn(f"Should have ta>=t0 but got ta={ta} and t0={start}.")
            ta = start
        if tb < start:
            warnings.warn(f"Should have {tb_name}>=t0 but got {tb_name}={tb} and t0={start}.")
            tb = start
        if ta > end:
            warnings.warn(f"Should have ta<=t1 but got ta={ta} and t1={end}.")
            ta = end
        if tb > end:
            warnings.warn(f"Should have {tb_name}<=t1 but got {tb_name}={tb} and t1={end}.")
            tb = end
        if ta > tb:
            raise RuntimeError(f"Query times ta={ta:.3f} and tb={tb:.3f} must respect ta <= tb.")

        self._require_cuda()
        if ta == tb:
            W = torch.zeros(self._size, dtype=self._dtype, device=self._device)
            H = torch.zeros(self._size, dtype=self._dtype, device=self._device) if self._have_H else None
            A = None
            if self._have_A:
                A = torch.zeros((*self._size, *self._size[-1:]), dtype=self._dtype, device=self._device)
            U = H
        else:
            ta_r = self._round(ta)
            tb_r = self._round(tb)
            if self._dt is not None and self._root.kind == _LEAF and self._root_value is None \
                    and self._user_W is None and self._user_H is None and not self._halfway_tree:
                self._bind_uniform(self._dt)
            if self._have_A and return_A:
                fused = self._query_cell_levy(ta_r, tb_r)
                if fused is not None:
                    W, U, A = fused
                    return (W, U, A) if return_U else (W, A)
            fast = self._query_cells_wu(ta_r, tb_r, tb - ta) if not self._have_A else None
            if fast is not None:
                W, U = fast
                if return_U:
                    return (W, U, None) if return_A else (W, U)
                return (W, None) if return_A else W
            W, H, A = self._query(ta_r, tb_r)
            U = None
            if self._have_H:
                U = self._new()
                L = self._launch()
                _cabi.check(_cabi.lib().tsde_brownian_h_to_u(ctypes.byref(L), W.data_ptr(), H.data_ptr(),
                                                             tb - ta, U.data_ptr()), "tsde_brownian_h_to_u")
                U = U.reshape(self._size)
            W = W.reshape(self._size)
            if A is not None:
                # rank 0/1: zero Levy area with the shape of W (brownian_interval.py:81-84)
                A = A.reshape(self._size if len(self._size) < 2 else (*self._size, *self._size[-1:]))

        if return_U:
            if return_A:
                return W, U, A
            return W, U
        if return_A:
            return W, A
        return W

    def _query_cells_wu(self, ta, tb, h_total):
        """Single-launch answer (W, U) when [ta, tb] is exactly a run of whole primary cells of the root
        grid (the access pattern of a fixed-step solver / of sequential dt-spaced queries): U is formed in
        the same kernel as W, H is never materialised (U is None without a space-time Levy area; the launch is the
        one `_draw_cells` makes for the same cells, so the numbers are those of the general path)."""
        root = self._root
        if root.kind != _GRID:
            return None
        b = root.bounds
        i = bisect.bisect_left(b, ta)
        if i >= len(b) or b[i] != ta:
            return None
        j = bisect.bisect_left(b, tb, i)
        if j >= len(b) or b[j] != tb or j <= i:
            return None
        nz = _cabi.Noise()
        nz.source = _cabi.SRC_COUNTER
        nz.want_u = 1 if self._have_H else 0
        nz.key = self.key_tensor().data_ptr()
        nz.cell_id = (root.cell_base + i) & _MASK64
        nz.row_offset = self._row_offset
        nz.n_cells = j - i
        nz.h = b[i + 1] - b[i]
        nz.h_total = h_total
        nz.cell_h = self._cell_h_dev(root).data_ptr() + 8 * i if j - i > 1 else None
        W = self._new_out()
        U = self._new_out() if self._have_H else None
        L = self._launch()
        _cabi.check(_cabi.lib().tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), W.data_ptr(),
                                                    None if U is None else U.data_ptr(), None), "tsde_brownian_cells")
        self._last = root
        return W, U

    def _query_cell_levy(self, ta, tb):
        """Single-launch answer (W, U, A) when [ta, tb] is exactly ONE primary cell of the root grid — the access
        pattern of a Levy-area method (log-ODE) stepping on its grid, or of sequential dt-spaced queries: the cell's
        W and H are drawn inside the kernel that forms the area, H is never materialised.  Same numbers as the general
        path (cells -> levy_area -> h_to_u), which serves every other query."""
        root = self._root
        if root.kind != _GRID or len(self._size) < 2 or self._m % 4 != 0 or not (4 <= self._m <= 64):
            return None
        b = root.bounds
        i = bisect.bisect_left(b, ta)
        if i + 1 >= len(b) or b[i] != ta or b[i + 1] != tb:
            return None
        cell = root.cell(i)
        if self._cache_get(cell) is not None:
            return None  # (the cell's (W, H) was already materialised: answer from it, as the general path does)
        nz = _cabi.Noise()
        nz.source = _cabi.SRC_COUNTER
        nz.want_u = 1
        nz.key = self.key_tensor().data_ptr()
        nz.cell_id = cell.id
        nz.row_offset = self._row_offset
        nz.n_cells = 1
        nz.h = b[i + 1] - b[i]
        nz.h_total = nz.h
        nz.cell_h = None
        W, U, A = self._new_out(), self._new_out(), self._new_out(self._m)
        L = self._launch()
        foster = 1 if self._levy_area_approximation == LEVY_AREA_APPROXIMATIONS.foster else 0
        _cabi.check(_cabi.lib().tsde_brownian_cell_levy(ctypes.byref(L), ctypes.byref(nz), cell.id, foster,
                                                        W.data_ptr(), U.data_ptr(), A.data_ptr()),
                    "tsde_brownian_cell_levy")
        self._last = root
        return W, U, A

    def _piece_value(self, piece):
        if isinstance(piece, _Node):
            W, H = self._value(piece)
            return W, H, piece.end - piece.start, piece.start, piece.end, piece.id
        grid, i, j = piece
        if j - i == 1:
            W, H = self._value(grid.cell(i))
            a_id = grid.cell(i).id
        else:
            W, H = self._draw_cells(grid, i, j - i, grid.bounds[j] - grid.bounds[i])
            a_id = mix64(child_id(grid.id, i) ^ mix64(j))
        return W, H, grid.bounds[j] - grid.bounds[i], grid.bounds[i], grid.bounds[j], a_id

    def _levy_area(self, W, H, h, a_id):
        """Davie / Foster approximation for one piece (:78-99)."""
        if not self._have_A:
            return None
        if len(self._size) in (0, 1):
            return torch.zeros_like(W)
        A = self._new(self._m)
        L = self._launch()
        foster = 1 if self._levy_area_approximation == LEVY_AREA_APPROXIMATIONS.foster else 0
        _cabi.check(_cabi.lib().tsde_brownian_levy_area(
            ctypes.byref(L), self.key_tensor().data_ptr(), self._row_offset, a_id, W.data_ptr(), H.data_ptr(),
            h, foster, A.data_ptr()), "tsde_brownian_levy_area")
        return A

    def _query(self, ta, tb):
        pieces = self._locate(ta, tb)
        last = pieces[-1]
        self._last = last if isinstance(last, _Node) else last[0]
        W, H, h, _, _, a_id = self._piece_value(pieces[0])
        A = self._levy_area(W, H, h, a_id)
        if len(pieces) > 1:
            lib = _cabi.lib()
            L = self._launch()
            W = W.clone()  # never modify cached node values
            H = H.clone() if H is not None else None
            for piece in pieces[1:]:
                Wi, Hi, hi, si, ei, ai_id = self._piece_value(piece)
                Ai = self._levy_area(Wi, Hi, hi, ai_id)
                if A is not None and len(self._size) not in (0, 1):
                    # uses W *before* the update, :671
                    _cabi.check(lib.tsde_brownian_merge_area(ctypes.byref(L), A.data_ptr(), Ai.data_ptr(),
                                                             W.data_ptr(), Wi.data_ptr()),
                                "tsde_brownian_merge_area")
                _cabi.check(lib.tsde_brownian_merge(
                    ctypes.byref(L), W.data_ptr(), None if H is None else H.data_ptr(), Wi.data_ptr(),
                    None if Hi is None else Hi.data_ptr(), si - ta, ei - si, ei - ta), "tsde_brownian_merge")
        return W, H, A

    # ------------------------------------------------------------------------------------------
    # grids
    # ------------------------------------------------------------------------------------------
    def _make_grid(self, node, bounds):
        node.kind = _GRID
        node.bounds = list(bounds)
        node.cells = {}
        node.cell_base = child_id(node.id, 2)
        node.cell_h_dev = None

    def _bind_uniform(self, dt):
        """`dt` hint (:436-440, :572-575): pre-split [t0, t1] into primary cells of length dt."""
        root = self._root
        n = int(math.ceil((root.end - root.start) / dt - 1e-9))
        if n < 2 or n > (1 << 26):
            return
        bounds = [self._round(root.start + k * dt) for k in range(n)] + [root.end]
        if any(b1 <= b0 for b0, b1 in zip(bounds[:-1], bounds[1:])):
            return
        self._make_grid(root, bounds)

    def bind_grid(self, bounds):
        """Called by the fixed-step solver with its step boundaries (python floats, increasing).
        Returns a `GridBinding` if every step is a run of whole primary cells of a root-level GRID
        (creating that GRID when the interval is still untouched), else None — the solver then falls
        back to ordinary ``bm(ta, tb)`` queries, which are always valid."""
        if self._halfway_tree or self._device.type != 'cuda':
            return None
        root = self._root
        bounds = [self._round(float(b)) for b in bounds]
        if len(bounds) < 2:
            return None
        if root.kind == _LEAF:
            if bounds[0] != root.start or bounds[-1] != root.end:
                return None
            if self._root_value is not None or self._user_W is not None or self._user_H is not None:
                return None
            if self._dt is not None:
                # honour an explicit dt hint only if the solver grid is made of those cells
                self._bind_uniform(self._dt)
                if root.kind == _GRID:
                    return self.bind_grid(bounds)
                return None
            self._make_grid(root, bounds)
        if root.kind != _GRID:
            return None
        gb = root.bounds
        first, count = [], []
        pos = 0
        for a, b in zip(bounds[:-1], bounds[1:]):
            i = bisect.bisect_left(gb, a, pos)
            if i >= len(gb) or gb[i] != a:
                return None
            j = bisect.bisect_left(gb, b, i)
            if j >= len(gb) or gb[j] != b:
                return None
            first.append(i)
            count.append(j - i)
            pos = j
        return GridBinding(self, root, first, count, bounds)

    # ------------------------------------------------------------------------------------------
    # batch sharding (one process per GPU): rows are independent Philox streams
    # ------------------------------------------------------------------------------------------
    def shard_rows(self, row_offset):
        """Declare that local row 0 is global row `row_offset`: every rank of a batch-sharded solve
        then reproduces exactly the rows it would own in the unsharded Brownian motion."""
        self._row_offset = int(row_offset)
        return self

    # ------------------------------------------------------------------------------------------
    def __repr__(self):
        dt = None if self._dt is None else f"{self._dt:.3f}"
        return (f"{self.__class__.__name__}("
                f"t0={self._root.start:.3f}, "
                f"t1={self._root.end:.3f}, "
                f"size={self._size}, "
                f"dtype={self._dtype}, "
                f"device={repr(self._device)}, "
                f"entropy={self._entropy}, "
                f"dt={dt}, "
                f"tol={self._tol}, "
                f"pool_size={self._pool_size}, "
                f"cache_size={self._cache_size}, "
                f"levy_area_approximation={repr(self._levy_area_approximation)}"
                f")")

    def display_binary_tree(self):
        stack = [(self._root, 0)]
        out = []
        while stack:
            elem, depth = stack.pop()
            out.append(" " * depth + f"({elem.start}, {elem.end})")
            if elem.kind == _BINARY:
                stack.append((elem.right, depth + 1))
                stack.append((elem.left, depth + 1))
            elif elem.kind == _GRID:
                out.append(" " * (depth + 1) + f"[grid of {len(elem.bounds) - 1} cells]")
        print("\n".join(out))

    @property
    def shape(self):
        return self._size

    @property
    def dtype(self):
        return self._dtype

    @property
    def device(self):
        return self._device

    @property
    def entropy(self):
        return self._entropy

    @property
    def levy_area_approximation(self):
        return self._levy_area_approximation

    @property
    def dt(self):
        return self._dt

    @property
    def tol(self):
        return self._tol

    @property
    def pool_size(self):
        return self._pool_size

    @property
    def cache_size(self):
        return self._cache_size

    @property
    def halfway_tree(self):
        return self._halfway_tree

    def size(self):
        return self._size
