"""Every Brownian-source kernel and query path against a float64 restatement with a propagated error bound.

The Brownian kernels (csrc/brownian.cu) materialise whole cells (`CellsOp` through the row-wise fast and generic
kernels, `cells_wh_kernel` when H is wanted), descend Brownian bridges (`bridge_kernel`, one launch per 24 levels,
continuing in place), merge pieces (`MergeWHOp`, `AddOp`, `HToUOp`, `merge_area_kernel`) and form Davie / Foster Levy
areas (`levy_tile_kernel` for m <= 64, compile-time m = 8 and 16, one pass up to m = 16 and several above; the
generating mode of `tsde_brownian_cell_levy`; `levy_area_kernel` for m > 64).

Each output element must satisfy |got - ref| <= E.  `ref` is the kernel's formula evaluated in float64 on the float64
normals of the launch dtype's specification (oracle/philox.py before its final rounding).  E is a first-order bound
carried alongside `ref` through every operation the kernel performs (`Val`): a rounded operation adds
u (|x| + E_x + |y| + E_y) plus the underflow unit, a coefficient the host rounds to the launch dtype one more
u |c| (|x| + E_x), a normal |c| (ATOL_N + RTOL_N |N|) (the fp32 SFU Box-Muller's agreement with float64, a few ulp in
fp64), and the fp32 square root of Foster's std the relative error the PTX ISA states for `sqrt.approx.f32`.  So deep
bridges, cancelling differences (a right child at a split near its parent's end, W summed over many cells) and merges
get the bound their operands carry, not a fixed tolerance.  Outputs are prefilled with NaN (every slot must be
written) and guarded by sentinels on both sides.

CPU tests pin the formulas to oracle/brownian.py and show that the bound rejects subtly wrong formulas.
"""
import collections
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import brownian as obm
from oracle import philox
from torchsde_b200 import _cabi
from torchsde_b200._brownian import interval as iv

DEV = 'cuda'
KEY = 20261016                    # Philox key
CELL = 11                         # counter id of the (first) cell
GUARD = 64                        # sentinel elements before and after every output
SENTINEL = -1234.5
MASK = (1 << 64) - 1
NP = {torch.float32: np.float32, torch.float64: np.float64}
UNIT = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}
TINY = {np.float32: 2.0 ** -150, np.float64: 2.0 ** -1075}   # underflow: half the smallest subnormal
# per-normal agreement |dN| <= ATOL + RTOL |N| of the device's generator with the oracle's float64 evaluation: the fp32
# SFU Box-Muller (as in test_gpu_general_paths.py), and libm's log / sincospi against numpy's in fp64
NORMAL_AGREEMENT = {np.float32: (5e-6, 2e-5), np.float64: (2.0 ** -52, 2.0 ** -49)}
SQRT_APPROX = 2.0 ** -23          # max relative error of sqrt.approx.f32 (PTX ISA)
C2 = 2 * 0.70710678118654752440   # N_ij - N_ji = z * 2 / sqrt(2)


# ---- float64 values with a propagated bound ------------------------------------------------------------------------
class Val:
    """float64 values `v` and a bound `e` on |device - v|, elementwise, for a launch of unit roundoff `u`."""
    __array_ufunc__ = None   # (numpy scalars * Val -> Val.__rmul__)

    def __init__(self, v, e, npdt):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.broadcast_to(np.asarray(e, dtype=np.float64), self.v.shape).copy()
        self.dt = npdt

    @property
    def u(self):
        return UNIT[self.dt]

    @classmethod
    def exact(cls, x, npdt):
        return cls(np.asarray(x, dtype=np.float64), 0.0, npdt)

    @classmethod
    def coef(cls, c, npdt):
        """a constant the host rounds to the launch dtype"""
        return cls(c, UNIT[npdt] * abs(c), npdt)

    def mag(self):
        return np.abs(self.v) + self.e

    def map(self, f):
        return Val(f(self.v), f(self.e), self.dt)

    def _round(self, terms):
        return self.u * terms + TINY[self.dt]

    def _sum(self, o, s):
        return Val(self.v + s * o.v, self.e + o.e + self._round(self.mag() + o.mag()), self.dt)

    def __add__(self, o):
        return self._sum(o, 1.0)

    def __sub__(self, o):
        return self._sum(o, -1.0)

    def __neg__(self):
        return Val(-self.v, self.e, self.dt)

    def __mul__(self, o):
        if isinstance(o, Val):
            return Val(self.v * o.v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
                       + self._round(self.mag() * o.mag()), self.dt)
        c = float(o)   # a coefficient rounded to the launch dtype, then the product
        return Val(c * self.v, abs(c) * self.e + 2 * self._round(abs(c) * self.mag()), self.dt)

    __rmul__ = __mul__

    def __truediv__(self, c):
        c = float(c)
        return Val(self.v / c, self.e / abs(c) + 2 * self._round(self.mag() / abs(c)), self.dt)

    def sqrt(self):
        rel = SQRT_APPROX if self.dt == np.float32 else self.u
        v = np.sqrt(np.maximum(self.v, 0.0))
        with np.errstate(divide='ignore', invalid='ignore'):
            prop = np.minimum(np.where(v > 0, self.e / v, np.inf), np.sqrt(self.e))
        return Val(v, prop + rel * np.sqrt(self.mag()) + TINY[self.dt], self.dt)


class Src:
    """The counter source of a launch: key, rows (or the sampled global rows `row_ids`), dtype, row offset."""

    def __init__(self, rows, npdt, row_offset=0, row_ids=None, key=KEY, agree=True):
        self.rows, self.dt, self.row_offset, self.row_ids, self.key, self.agree = rows, npdt, row_offset, row_ids, key, agree

    def normal(self, node_id, stream, m):
        n = philox.normals(self.key, node_id & MASK, stream, self.rows, m, self.dt, self.row_offset, self.row_ids,
                           exact=True)
        atol, rtol = NORMAL_AGREEMENT[self.dt] if self.agree else (0.0, 0.0)
        return Val(n, atol + rtol * np.abs(n), self.dt)


# ---- the kernels' formulas (csrc/brownian.cu, csrc/ew.cuh counter_noise), in their order of operations -------------
def cells_f(src, cell_id, lengths, m, have_h=True):
    """(W, H) of the merge of primary cells cell_id, cell_id + 1, ... (counter_wh / counter_noise)."""
    def draw(c, h):
        cid = (cell_id + c) & MASK
        W = math.sqrt(h) * src.normal(cid, philox.STREAM_W, m)
        return W, (math.sqrt(h / 12.0) * src.normal(cid, philox.STREAM_H, m) if have_h else None)
    W, H = draw(0, lengths[0])
    elapsed = lengths[0]
    for c, ln in enumerate(lengths[1:], 1):
        Wi, Hi = draw(c, ln)
        if have_h:
            H = (ln * (Hi + 0.5 * W) + elapsed * (H - 0.5 * Wi)) / (elapsed + ln)
        W = W + Wi
        elapsed += ln
    return W, H


def bridge_f(W, H, start, mid, end, is_left, X1, X2=None):
    """One level of bridge_kernel with the coefficients bridge_impl forms in double."""
    h_rec = 1.0 / (end - start)
    ld, rd = mid - start, end - mid
    if H is not None:
        ld2, rd2 = ld * ld, rd * rd
        v = 0.5 * math.sqrt(ld * rd / (ld * ld2 + rd * rd2))
        a, b, c = v * ld2 * h_rec, v * rd2 * h_rec, v * 0.57735026918962584
        third = 2 * (a * ld + b * rd) * h_rec
        if is_left:
            first = ld * h_rec
            k = (first, 6 * first * rd * h_rec, third, first * first, -a, c * rd)
        else:
            first = rd * h_rec
            k = (first, -(6 * first * ld * h_rec), -third, first * first, -b, -(c * ld))
        return (k[0] * W + k[1] * H) + k[2] * X1, (k[3] * H + k[4] * X1) + k[5] * X2
    left_w = (ld * W) * h_rec + math.sqrt(ld * rd * h_rec) * X1
    return (left_w if is_left else W - left_w), None


def bridge_chain_f(src, W, H, levels, m):
    """levels: (parent id, is_left, start, mid, end) from the top down."""
    for pid, is_left, start, mid, end in levels:
        X1 = src.normal(pid, philox.STREAM_X1, m)
        X2 = src.normal(pid, philox.STREAM_X2, m) if H is not None else None
        W, H = bridge_f(W, H, start, mid, end, is_left, X1, X2)
    return W, H


def merge_f(W, H, Wi, Hi, len0, len1, tot):
    """MergeWHOp / AddOp: the running (W, H) over [ta, s] with the piece [s, e]; len0 = s - ta, len1 = e - s."""
    if H is not None:
        H = (len1 * (Hi + 0.5 * W) + len0 * (H - 0.5 * Wi)) / tot
    return W + Wi, H


def h_to_u_f(W, H, h):
    return h * (0.5 * W + H)


def levy_pairs(m):
    return np.triu_indices(m, k=1)   # pair p = (i, j), i < j, row-major: channel p of STREAM_A


def levy_f(W, H, h, foster, Z, m):
    """(rows, m, m) Davie / Foster area from (rows, m) W, H and the (rows, m(m-1)/2) pair normals Z."""
    iu, ju = levy_pairs(m)
    col = lambda x, idx: x.map(lambda a: a[:, idx])   # noqa: E731
    Wi, Wj, Hi, Hj = col(W, iu), col(W, ju), col(H, iu), col(H, ju)
    a = Hi * Wj - Wi * Hj
    noise = C2 * Z.map(lambda z: z[:, :len(iu)])
    if foster:
        th = Val.coef(0.1 * h, W.dt)
        std = (th * ((th + Hi * Hi) + Hj * Hj)).sqrt()
    else:
        std = Val.coef(math.sqrt((1.0 / 12.0) * h * h), W.dt)
    pv = a + std * noise
    rows = W.v.shape[0]
    A = Val(np.zeros((rows, m, m)), 0.0, W.dt)
    A.v[:, iu, ju], A.v[:, ju, iu] = pv.v, -pv.v
    A.e[:, iu, ju], A.e[:, ju, iu] = pv.e, pv.e
    return A


def merge_area_f(A, Ai, W, Wi):
    x = W.map(lambda a: a[..., :, None]) * Wi.map(lambda a: a[..., None, :]) \
        - Wi.map(lambda a: a[..., :, None]) * W.map(lambda a: a[..., None, :])
    return (A + Ai) + 0.5 * x


# ---- CPU: the formulas against oracle/brownian.py ------------------------------------------------------------------
def _agree(name, mine, ref):
    """float64 rounding: within the float64 bound on each side."""
    err = np.abs(np.asarray(ref, dtype=np.float64) - mine.v)
    assert np.all(err <= 2 * mine.e), f'{name}: max err/bound {np.max(err / (2 * mine.e)):.3g}'


@pytest.mark.parametrize('m', [1, 3, 6])
def test_formulas_match_oracle_brownian(m):
    f64 = np.float64
    src = Src(9, f64, row_offset=5, agree=False)
    rng = np.random.default_rng(m)
    W, H, Wi, Hi = (rng.standard_normal((9, m)) * s for s in (0.7, 0.2, 0.5, 0.1))
    V = lambda x: Val.exact(x, f64)   # noqa: E731
    X1, X2 = src.normal(77, philox.STREAM_X1, m), src.normal(77, philox.STREAM_X2, m)
    for is_left in (True, False):
        for start, mid, end in ((0.25, 0.4, 1.0), (0.0, 1e-6, 1.0), (0.5, 0.75 - 1e-7, 0.75)):
            w, h = bridge_f(V(W), V(H), start, mid, end, is_left, X1, X2)
            ow, oh = obm.bridge(W, H, start, mid, end, is_left, X1.v, X2.v)
            _agree('bridge W', w, ow)
            _agree('bridge H', h, oh)
            w, _ = bridge_f(V(W), None, start, mid, end, is_left, X1)
            _agree('bridge W (no H)', w, obm.bridge(W, None, start, mid, end, is_left, X1.v)[0])
    ta, s, e = 0.1, 0.35, 0.9
    w, h = merge_f(V(W), V(H), V(Wi), V(Hi), s - ta, e - s, e - ta)
    ow, oh = obm.merge(W, H, Wi, Hi, ta, s, e)
    _agree('merge W', w, ow)
    _agree('merge H', h, oh)
    _agree('h_to_u', h_to_u_f(V(W), V(H), 0.3), obm.h_to_u(W, H, 0.3))
    A0 = rng.standard_normal((9, m, m))
    A1 = rng.standard_normal((9, m, m))
    _agree('merge_area', merge_area_f(V(A0), V(A1), V(W), V(Wi)), obm.merge_area(A0, A1, W, Wi))
    npairs = max(m * (m - 1) // 2, 1)
    Z = src.normal(99, philox.STREAM_A, npairs)
    noise = obm.levy_noise(KEY, 99, 9, m, f64, row_offset=5)
    for foster in (False, True):
        _agree(f'davie_foster foster={foster}', levy_f(V(W), V(H), 0.3, foster, Z, m),
               obm.davie_foster(W, H, 0.3, foster, noise))
    lengths = [2.0 ** -8, 3 * 2.0 ** -8, 2.0 ** -7]
    w, h = cells_f(src, CELL, lengths, m)
    ow, oh = obm.cells(KEY, CELL, lengths, 9, m, f64, True, row_offset=5)
    _agree('cells W', w, ow)
    _agree('cells H', h, oh)


def test_exact_normals_are_the_specification_before_rounding():
    for dt in (np.float32, np.float64):
        a = philox.normals(KEY, 3, philox.STREAM_H, 5, 7, dt, 9, exact=True)
        assert a.dtype == np.float64
        assert np.array_equal(a.astype(dt), philox.normals(KEY, 3, philox.STREAM_H, 5, 7, dt, 9))


# ---- CPU: the bound rejects subtly wrong formulas ------------------------------------------------------------------
def _mutations():
    """(name, true Val, mutated values) on fp32 counter noise, the loosest bound."""
    f32, rows, m = np.float32, 64, 6
    src = Src(rows, f32, row_offset=3)
    out = []
    Wp, Hp = cells_f(src, CELL, [1.0], m)
    lv = (0x1234567, 0.25, 0.4, 1.0)
    pid, start, mid, end = lv
    X1, X2 = src.normal(pid, philox.STREAM_X1, m), src.normal(pid, philox.STREAM_X2, m)
    for is_left in (True, False):
        w, h = bridge_f(Wp, Hp, start, mid, end, is_left, X1, X2)
        mw, mh = bridge_f(Wp, Hp, start, mid, end, not is_left, X1, X2)
        out += [('left and right child swapped', w, mw.v), ('left and right child swapped', h, mh.v)]
        w0, _ = bridge_f(Wp, None, start, mid, end, is_left, X1)
        out.append(('left and right child swapped', w0, bridge_f(Wp, None, start, mid, end, not is_left, X1)[0].v))
        mw, mh = bridge_f(Wp, Hp, start, mid, end, is_left, X2, X1)
        out += [('X1 and X2 swapped', w, mw.v), ('X1 and X2 swapped', h, mh.v)]
        cid = iv.child_id(pid, 0 if is_left else 1)
        C1, C2_ = src.normal(cid, philox.STREAM_X1, m), src.normal(cid, philox.STREAM_X2, m)
        mw, mh = bridge_f(Wp, Hp, start, mid, end, is_left, C1, C2_)
        out += [("the child's id for the parent's", w, mw.v), ("the child's id for the parent's", h, mh.v)]
        out.append(("the child's id for the parent's", w0, bridge_f(Wp, None, start, mid, end, is_left, C1)[0].v))
    Wi, Hi = cells_f(src, CELL + 5, [0.3], m)
    _, h = merge_f(Wp, Hp, Wi, Hi, 0.1, 0.3, 0.4)
    out.append(('len0 and len1 swapped in the H-merge', h, merge_f(Wp, Hp, Wi, Hi, 0.3, 0.1, 0.4)[1].v))
    Z, Zi = src.normal(5, philox.STREAM_A, 15), src.normal(6, philox.STREAM_A, 15)
    A, Ai = levy_f(Wp, Hp, 1.0, True, Z, m), levy_f(Wi, Hi, 0.3, True, Zi, m)
    ma = merge_area_f(A, Ai, Wp, Wi)
    out.append(('pieces merged right to left in merge_area', ma, merge_area_f(A, Ai, Wi, Wp).v))
    out.append(("Davie's std for Foster's", A, levy_f(Wp, Hp, 1.0, False, Z, m).v))
    out.append(('the pair noise transposed', A, levy_f(Wp, Hp, 1.0, True, -Z, m).v))
    lengths = [0.1, 0.5, 0.25]
    W3, H3 = cells_f(src, CELL + 9, lengths, m)
    out.append(('U formed with h instead of h_total', h_to_u_f(W3, H3, sum(lengths)), h_to_u_f(W3, H3, lengths[0]).v))
    pw, ph = cells_f(src, CELL + 9, [0.25, 0.1, 0.5], m)
    out += [('the cell lengths of a 3-cell run permuted', W3, pw.v), ('the cell lengths of a 3-cell run permuted', H3, ph.v)]
    return out


def test_bound_rejects_wrong_formulas():
    """The bound rejects each mistake on >= 75 % of the elements it changes: left and right child swapped, X1 and X2
    swapped, a bridge level drawing with the child's id, len0 / len1 swapped in the H-merge, merge_area with the pieces
    in the wrong order, Davie's std used for Foster, the pair noise transposed, U formed with h instead of h_total, and
    the lengths of an unequal 3-cell run permuted."""
    bad, seen = [], set()
    for name, true, wrong in _mutations():
        changed = wrong != true.v
        if not changed.any():
            continue
        seen.add(name)
        caught = (np.abs(wrong - true.v) > true.e)[changed].mean()
        if caught < 0.75:
            bad.append(f'{name}: caught on {caught:.1%}')
    assert len(seen) == 9, seen
    assert not bad, '\n'.join(bad)


def test_merge_area_with_the_updated_w_is_the_same_area():
    """merge_area with W after the update is not a mistake: (W + Wi) x Wi - Wi x (W + Wi) = W x Wi - Wi x W, so the bound
    must (and does) accept it."""
    src = Src(64, np.float32)
    W, H = cells_f(src, CELL, [0.5], 6)
    Wi, Hi = cells_f(src, CELL + 1, [0.5], 6)
    A = levy_f(W, H, 0.5, True, src.normal(1, philox.STREAM_A, 15), 6)
    Ai = levy_f(Wi, Hi, 0.5, True, src.normal(2, philox.STREAM_A, 15), 6)
    true = merge_area_f(A, Ai, W, Wi)
    assert np.all(np.abs(merge_area_f(A, Ai, W + Wi, Wi).v - true.v) <= true.e)


# ---- CPU: refusal of counter noise past 2^26 channels ----------------------------------------------------------------
def test_interval_refuses_more_than_2_26_channels():
    with pytest.raises(ValueError, match='2\\*\\*26 channels'):
        iv.BrownianInterval(0.0, 1.0, size=(2 ** 26 + 4,), device='cpu')
    with pytest.raises(ValueError, match='2\\*\\*26 channels'):
        iv.BrownianInterval(0.0, 1.0, size=(2, 2 ** 26 + 1), device='cpu')
    assert iv.BrownianInterval(0.0, 1.0, size=(2, 2 ** 26), device='cpu')._m == 2 ** 26


LIMIT_BUFFERS = ('w', 'u', 'h', 'w2', 'h2', 'zero', 'one', 'y1')


def _channel_limit_calls(lib, dtype, m, p, key_ptr):
    """(entry point, return code) of every counter-noise launch of one row of m Brownian channels, on the buffers
    p[name] (LIMIT_BUFFERS): cells write w, u, h; the bridge descends from (w, h) into (w2, h2); the diagonal Euler
    step y1 = y0 + f dt + g dW runs on y0 = f = zero, g = one."""
    w, u, h, w2, h2 = (p[k] for k in LIMIT_BUFFERS[:5])
    L = _cabi.Launch(dtype, _cabi.NOISE_DIAGONAL, 1, m, m, None)
    nz = _cabi.Noise()
    nz.source, nz.want_u, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, 1, key_ptr, CELL, 1, 0.5, 0.5
    ids, lefts, times = (ctypes.c_uint64 * 1)(7), (ctypes.c_int32 * 1)(1), (ctypes.c_double * 3)(0.0, 0.25, 0.5)
    out = [('cells W', lib.tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), w, None, None)),
           ('cells W U', lib.tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), w, u, None)),
           ('cells W H', lib.tsde_brownian_cells(ctypes.byref(L), ctypes.byref(nz), w, None, h)),
           ('bridge W', lib.tsde_brownian_bridge(ctypes.byref(L), key_ptr, 0, 1, ids, lefts, times, w, None, w2, None)),
           ('bridge W H', lib.tsde_brownian_bridge(ctypes.byref(L), key_ptr, 0, 1, ids, lefts, times, w, h, w2, h2))]
    out.append(('step_euler', lib.tsde_step_euler(ctypes.byref(L), ctypes.byref(nz), p['zero'], p['zero'], p['one'],
                                                  0.25, p['y1'])))
    return out


@pytest.mark.skipif(torch.cuda.is_available(), reason='with a device, the GPU test below makes the same launches on '
                                                      'real buffers')
@pytest.mark.parametrize('dtype', [_cabi.F32, _cabi.F64], ids=['f32', 'f64'])
def test_counter_noise_past_2_26_channels_refused_without_device(dtype):
    """Refused before any CUDA call at 2^26 + 1 channels; at 2^26 the launch goes ahead (and, without a device, fails
    in the CUDA runtime instead)."""
    try:
        lib = _cabi.lib()
    except _cabi.LibraryNotBuilt:
        pytest.skip('CUDA library not built')
    key = ctypes.c_int64(KEY)
    fake = {k: 4096 * (i + 1) for i, k in enumerate(LIMIT_BUFFERS)}   # never dereferenced: no device
    for name, rc in _channel_limit_calls(lib, dtype, 2 ** 26 + 1, fake, ctypes.addressof(key)):
        assert rc == _cabi.EINVAL, (name, rc)
    for name, rc in _channel_limit_calls(lib, dtype, 2 ** 26, fake, ctypes.addressof(key)):
        assert rc not in (0, _cabi.EINVAL), (name, rc)


# ---- GPU helpers -------------------------------------------------------------------------------------------------
class _Report:
    """Worst err / bound per (kernel, dtype), and the failures."""

    def __init__(self):
        self.worst = collections.defaultdict(float)
        self.bad = []

    def out(self, n, dtype, shift=0, init=None):
        """(guarded buffer, output view of n elements `shift` elements past a 16-byte boundary)."""
        buf = torch.full((n + 2 * GUARD + shift,), SENTINEL, device=DEV, dtype=dtype)
        view = buf[GUARD + shift:GUARD + shift + n]
        if init is None:
            view.fill_(float('nan'))
        else:
            view.copy_(init.reshape(-1))
        return buf, view

    def check(self, kernel, dtype, where, buf, view, ref, row_ids=None):
        n = view.numel()
        lo = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
        if not (bool((buf[:lo] == SENTINEL).all()) and bool((buf[lo + n:] == SENTINEL).all())):
            self.bad.append(f'{kernel} {where}: wrote outside its output')
        got = view.double().cpu().numpy().reshape((-1,) + ref.v.shape[1:])
        if row_ids is not None:
            got = got[row_ids]
        if not np.isfinite(got).all():
            self.bad.append(f'{kernel} {where}: {int((~np.isfinite(got)).sum())} slots not written')
            return got
        err = np.abs(got - ref.v)
        with np.errstate(divide='ignore', invalid='ignore'):
            ratio = np.where(ref.e > 0, err / ref.e, np.where(err > 0, np.inf, 0.0))
        worst = float(ratio.max()) if ratio.size else 0.0
        key = (kernel, str(dtype)[6:])
        self.worst[key] = max(self.worst[key], worst)
        if worst > 1:
            self.bad.append(f'{kernel} {where}: {int((ratio > 1).sum())} elements off the formula, worst err/bound '
                            f'{worst:.3g}')
        return got

    def finish(self):
        for key in sorted(self.worst):
            print(f'{" / ".join(key):36s} worst err/bound {self.worst[key]:.3f}')
        assert not self.bad, '\n'.join(self.bad[:40])


def _lib():
    return _cabi.lib()


def _launch(dtype, rows, m):
    return _cabi.make_launch(dtype, _cabi.NOISE_DIAGONAL, rows, m, m)


def _key():
    return torch.tensor([KEY], dtype=torch.int64, device=DEV)


def _placed(x, shift):
    if not shift:
        return x.contiguous()
    buf = torch.empty(x.numel() + shift, device=x.device, dtype=x.dtype)
    buf[shift:].copy_(x.reshape(-1))
    return buf[shift:].view(x.shape)


def _wh(rows, m, h, dtype, seed):
    """device (W, H) of an interval of length h"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    W = torch.randn(rows, m, generator=gen, device=DEV, dtype=dtype) * math.sqrt(h)
    H = torch.randn(rows, m, generator=gen, device=DEV, dtype=dtype) * math.sqrt(h / 12)
    return W, H


def _exact(t, npdt, row_ids=None):
    x = t.double().cpu().numpy()
    return Val.exact(x if row_ids is None else x[row_ids], npdt)


# ---- GPU: cells ------------------------------------------------------------------------------------------------------
def _cells_case(rep, dtype, rows, m, lengths, mode, shift=0, row_offset=0):
    npdt = NP[dtype]
    key = _key()
    n = len(lengths)
    ch = torch.tensor(lengths, dtype=torch.float64, device=DEV)
    nz = _cabi.Noise()
    nz.source, nz.want_u, nz.key, nz.cell_id, nz.row_offset = _cabi.SRC_COUNTER, int('u' in mode), key.data_ptr(), CELL, row_offset
    nz.n_cells, nz.h, nz.h_total = n, lengths[0], sum(lengths)
    nz.cell_h = ch.data_ptr() if n > 1 else None
    outs = {c: rep.out(rows * m, dtype, shift) for c in mode}
    ptr = lambda c: outs[c][1].data_ptr() if c in outs else None   # noqa: E731
    _cabi.check(_lib().tsde_brownian_cells(ctypes.byref(_launch(dtype, rows, m)), ctypes.byref(nz), ptr('w'), ptr('u'),
                                           ptr('h')), 'tsde_brownian_cells')
    torch.cuda.synchronize()
    W, H = cells_f(Src(rows, npdt, row_offset), CELL, lengths, m)
    refs = {'w': W, 'h': H, 'u': h_to_u_f(W, H, sum(lengths))}
    kernel = 'cells_wh_kernel' if 'h' in mode else ('CellsOp W U' if 'u' in mode else 'CellsOp W')
    where = f'B={rows} m={m} cells={n} shift={shift} row_offset={row_offset} out={mode}'
    for c, (buf, view) in outs.items():
        rep.check(kernel, dtype, f'{where} {c}', buf, view, refs[c])


CELL_SHAPES = [(37, m, n) for m in (1, 3, 4, 5, 64) for n in (1, 3)] + [(5, 1000, 1), (5, 1000, 3), (9, 4, 257),
                                                                        (9, 5, 257)]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_cells_vs_formula(dtype):
    """tsde_brownian_cells: W (CellsOp), W and U (CellsOp, fast kernel at m % 4 == 0 on one cell, else generic) and W,
    U, H (cells_wh_kernel); one cell, three and 257 of unequal length (lengths on the device); one element off
    alignment; the last valid global rows."""
    rep = _Report()
    rng = np.random.default_rng(1)
    for rows, m, n in CELL_SHAPES:
        lengths = [2.0 ** -6] if n == 1 else ([2.0 ** -8, 3 * 2.0 ** -8, 2.0 ** -7] if n == 3
                                              else [float(x) for x in rng.uniform(1e-4, 1e-2, n)])
        for mode in ('w', 'wu', 'wuh'):
            _cells_case(rep, dtype, rows, m, lengths, mode)
        if (m, n) in ((4, 1), (64, 3), (5, 3)):
            for mode in ('wu', 'wuh'):
                _cells_case(rep, dtype, rows, m, lengths, mode, shift=1)
                _cells_case(rep, dtype, rows, m, lengths, mode, row_offset=(1 << 32) - 1 - rows)
    rep.finish()


# ---- GPU: bridge -----------------------------------------------------------------------------------------------------
def _levels(rng, depth):
    """A random descent from [0, 1]: splits at random fractions and at 1e-6 / 1 - 1e-6 of the parent, both children of
    the latter visited (the small one a few times only, so that every interval stays resolvable in double)."""
    start, end, pid = 0.0, 1.0, int(rng.integers(1 << 63)) * 2 + 1
    out = []
    for _ in range(depth):
        span = end - start
        r = rng.uniform()
        if r < 0.5 and span > 1e-9:
            frac, left = rng.uniform(0.2, 0.8), bool(rng.integers(2))
        else:
            frac = 1e-6 if rng.integers(2) else 1 - 1e-6
            small = rng.uniform() < 0.25 and span > 1e-4
            left = (frac < 0.5) == small
        mid = start + frac * span
        out.append((pid, left, start, mid, end))
        start, end = (start, mid) if left else (mid, end)
        pid = iv.child_id(pid, 0 if left else 1)
    return out


def _bridge_case(rep, dtype, rows, m, depth, have_h, rng, shift=0, row_offset=0):
    npdt = NP[dtype]
    levels = _levels(rng, depth)
    W, H = _wh(rows, m, 1.0, dtype, seed=depth * 7 + m)
    W, H = _placed(W, shift), (_placed(H, shift) if have_h else None)
    ow = rep.out(rows * m, dtype, shift)
    oh = rep.out(rows * m, dtype, shift) if have_h else None
    ids = (ctypes.c_uint64 * depth)(*[lv[0] for lv in levels])
    lefts = (ctypes.c_int32 * depth)(*[int(lv[1]) for lv in levels])
    times = (ctypes.c_double * (3 * depth))(*[t for lv in levels for t in lv[2:]])
    _cabi.check(_lib().tsde_brownian_bridge(
        ctypes.byref(_launch(dtype, rows, m)), _key().data_ptr(), row_offset, depth, ids, lefts, times, W.data_ptr(),
        H.data_ptr() if have_h else None, ow[1].data_ptr(), oh[1].data_ptr() if have_h else None), 'bridge')
    torch.cuda.synchronize()
    rW, rH = bridge_chain_f(Src(rows, npdt, row_offset), _exact(W, npdt), _exact(H, npdt) if have_h else None, levels, m)
    where = f'B={rows} m={m} depth={depth} H={have_h} shift={shift} row_offset={row_offset}'
    rep.check('bridge_kernel', dtype, where + ' W', *ow, rW)
    if have_h:
        rep.check('bridge_kernel', dtype, where + ' H', *oh, rH)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_bridge_vs_formula(dtype):
    """tsde_brownian_bridge at depth 1, 24 (one launch), 25, 48, 49, 60 (two and three, continuing in place), random
    children and splits at 1e-6 / 1 - 1e-6 of the parent, with and without H, m = 1, 3, 4, 17; unaligned input and
    output; the last valid global rows."""
    rep = _Report()
    rng = np.random.default_rng(2)
    for rows, m in ((33, 1), (33, 3), (33, 4), (9, 17)):
        for depth in (1, 24, 25, 48, 49, 60):
            for have_h in (True, False):
                _bridge_case(rep, dtype, rows, m, depth, have_h, rng)
    for have_h in (True, False):
        _bridge_case(rep, dtype, 33, 4, 25, have_h, rng, shift=1)
        _bridge_case(rep, dtype, 33, 3, 49, have_h, rng, row_offset=(1 << 32) - 1 - 33)
    rep.finish()


# ---- GPU: merges -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_merges_vs_formula(dtype):
    """tsde_brownian_merge (W only: AddOp; W and H: MergeWHOp) and tsde_brownian_h_to_u, m odd and a multiple of 4,
    aligned and one element off, len0 << len1 and the reverse; tsde_brownian_merge_area at m = 1, 3, 16, 65."""
    rep, npdt, lib = _Report(), NP[dtype], _lib()
    for m in (3, 5, 8, 12):
        for shift in (0, 1):
            for len0, len1 in ((1e-6, 0.5), (0.5, 1e-6), (0.25, 0.125)):
                rows = 37
                W, H = _wh(rows, m, len0, dtype, seed=m)
                Wi, Hi = _wh(rows, m, len1, dtype, seed=m + 100)
                Wi, Hi = _placed(Wi, shift), _placed(Hi, shift)
                where = f'B={rows} m={m} shift={shift} len0={len0} len1={len1}'
                for have_h in (False, True):
                    ow = rep.out(rows * m, dtype, shift, init=W)
                    oh = rep.out(rows * m, dtype, shift, init=H) if have_h else None
                    _cabi.check(lib.tsde_brownian_merge(
                        ctypes.byref(_launch(dtype, rows, m)), ow[1].data_ptr(), oh[1].data_ptr() if have_h else None,
                        Wi.data_ptr(), Hi.data_ptr() if have_h else None, len0, len1, len0 + len1), 'merge')
                    torch.cuda.synchronize()
                    rW, rH = merge_f(_exact(W, npdt), _exact(H, npdt) if have_h else None, _exact(Wi, npdt),
                                     _exact(Hi, npdt), len0, len1, len0 + len1)
                    rep.check('MergeWHOp' if have_h else 'AddOp', dtype, where + ' W', *ow, rW)
                    if have_h:
                        rep.check('MergeWHOp', dtype, where + ' H', *oh, rH)
                ou = rep.out(rows * m, dtype, shift)
                _cabi.check(lib.tsde_brownian_h_to_u(ctypes.byref(_launch(dtype, rows, m)), Wi.data_ptr(), Hi.data_ptr(),
                                                     len0 + len1, ou[1].data_ptr()), 'h_to_u')
                torch.cuda.synchronize()
                rep.check('HToUOp', dtype, where, *ou, h_to_u_f(_exact(Wi, npdt), _exact(Hi, npdt), len0 + len1))
    for m in (1, 3, 16, 65):
        rows = 17
        gen = torch.Generator(device=DEV).manual_seed(m)
        A0, A1 = (torch.randn(rows, m, m, generator=gen, device=DEV, dtype=dtype) * 0.01 for _ in range(2))
        W0, W1 = (torch.randn(rows, m, generator=gen, device=DEV, dtype=dtype) * 0.1 for _ in range(2))
        oa = rep.out(rows * m * m, dtype, init=A0)
        _cabi.check(lib.tsde_brownian_merge_area(ctypes.byref(_launch(dtype, rows, m)), oa[1].data_ptr(), A1.data_ptr(),
                                                 W0.data_ptr(), W1.data_ptr()), 'merge_area')
        torch.cuda.synchronize()
        rep.check('merge_area_kernel', dtype, f'B={rows} m={m}', *oa,
                  merge_area_f(_exact(A0, npdt), _exact(A1, npdt), _exact(W0, npdt), _exact(W1, npdt)))
    rep.finish()


# ---- GPU: Levy area --------------------------------------------------------------------------------------------------
def _levy_kernel_name(m):
    if m > 64:
        return 'levy_area_kernel'
    return f'levy_tile_kernel MT={m if m in (8, 16) else 0}' + (' multi-pass' if m > 16 else '')


def _check_area(rep, kernel, dtype, where, oa, ref, row_ids=None):
    got = rep.check(kernel, dtype, where, *oa, ref, row_ids)
    if np.isfinite(got).all():   # A = -A^T and a zero diagonal, exactly
        if not (np.array_equal(got, -np.swapaxes(got, 1, 2)) and not np.diagonal(got, axis1=1, axis2=2).any()):
            rep.bad.append(f'{kernel} {where}: not exactly antisymmetric')


def _levy_case(rep, dtype, rows, m, foster, h, shift=0, row_offset=0, sample=None):
    npdt = NP[dtype]
    a_id = 0x5EED0000 + m
    W, H = _wh(rows, m, h, dtype, seed=rows + m)
    oa = rep.out(rows * m * m, dtype, shift)
    _cabi.check(_lib().tsde_brownian_levy_area(ctypes.byref(_launch(dtype, rows, m)), _key().data_ptr(), row_offset, a_id,
                                               W.data_ptr(), H.data_ptr(), h, int(foster), oa[1].data_ptr()), 'levy')
    torch.cuda.synchronize()
    row_ids = None if sample is None else np.unique(np.r_[0, rows - 1, np.random.default_rng(m).integers(0, rows, sample)])
    src = Src(rows, npdt, row_offset, row_ids)
    Z = src.normal(a_id, philox.STREAM_A, max(m * (m - 1) // 2, 1))
    ref = levy_f(_exact(W, npdt, row_ids), _exact(H, npdt, row_ids), h, foster, Z, m)
    where = f'B={rows} m={m} foster={foster} h={h:.3g} shift={shift} row_offset={row_offset}'
    _check_area(rep, _levy_kernel_name(m) + (' foster' if foster else ' davie'), dtype, where, oa, ref, row_ids)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_levy_area_vs_formula(dtype):
    """tsde_brownian_levy_area, Davie and Foster: the tile kernel at m = 2 ... 64 (compile-time m = 8, 16; one pass up to
    m = 16, several above), out_a one element off alignment (copy-out without vector stores), 37 rows (not a multiple
    of the warps per CTA) and 5003 rows (more than one row per warp, sampled); `levy_area_kernel` at m = 65, 96, 130."""
    rep = _Report()
    for foster in (False, True):
        for m in (2, 3, 5, 8, 12, 16, 17, 24, 33, 64, 65, 96, 130):
            _levy_case(rep, dtype, 37, m, foster, 2.0 ** -5)
        for m in (8, 12, 16, 64):
            _levy_case(rep, dtype, 37, m, foster, 2.0 ** -5, shift=1)
        _levy_case(rep, dtype, 5003, 16, foster, 2.0 ** -5, sample=200)
        _levy_case(rep, dtype, 3001, 5, foster, 2.0 ** -5, sample=200, row_offset=(1 << 32) - 1 - 3001)
    rep.finish()


def _cell_levy_case(rep, dtype, rows, m, foster, h, shift=0, sample=None):
    npdt = NP[dtype]
    a_id, key = 0xA0A0 + m, _key()
    nz = _cabi.Noise()
    nz.source, nz.want_u, nz.key, nz.cell_id, nz.n_cells, nz.h, nz.h_total = _cabi.SRC_COUNTER, 1, key.data_ptr(), CELL, 1, h, h
    ow, ou = rep.out(rows * m, dtype), rep.out(rows * m, dtype)
    oa = rep.out(rows * m * m, dtype, shift)
    _cabi.check(_lib().tsde_brownian_cell_levy(ctypes.byref(_launch(dtype, rows, m)), ctypes.byref(nz), a_id, int(foster),
                                               ow[1].data_ptr(), ou[1].data_ptr(), oa[1].data_ptr()), 'cell_levy')
    torch.cuda.synchronize()
    row_ids = None if sample is None else np.unique(np.r_[0, rows - 1, np.random.default_rng(m).integers(0, rows, sample)])
    src = Src(rows, npdt, 0, row_ids)
    W, H = cells_f(src, CELL, [h], m)
    A = levy_f(W, H, h, foster, src.normal(a_id, philox.STREAM_A, m * (m - 1) // 2), m)
    kernel = f'levy_tile_kernel GEN MT={m if m in (8, 16) else 0}' + (' foster' if foster else ' davie')
    where = f'B={rows} m={m} foster={foster} h={h:.3g} shift={shift}'
    rep.check(kernel, dtype, where + ' W', *ow, W, row_ids)
    rep.check(kernel, dtype, where + ' U', *ou, h_to_u_f(W, H, h), row_ids)
    _check_area(rep, kernel, dtype, where + ' A', oa, A, row_ids)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_cell_levy_vs_formula(dtype):
    """tsde_brownian_cell_levy (W, U and A of one cell in one launch), Davie and Foster, m = 4 ... 64 at 1, R - 1 and
    R + 1 rows for the R = 64 / m rows a warp draws per pass, out_a one element off alignment, and 20011 rows sampled."""
    rep = _Report()
    for foster in (False, True):
        for m in (4, 8, 12, 16, 32, 64):
            R = 64 // m
            for rows in sorted({1, R - 1, R + 1} - {0}):
                _cell_levy_case(rep, dtype, rows, m, foster, 2.0 ** -6)
        _cell_levy_case(rep, dtype, 9, 12, foster, 2.0 ** -6, shift=1)
        _cell_levy_case(rep, dtype, 20011, 16, foster, 2.0 ** -6, sample=200)
    rep.finish()


@pytest.mark.gpu
def test_foster_fp32_on_very_short_intervals():
    """Foster's variance ~0.027 h^2 is subnormal in fp32 for h below ~2^-60, where the noise term is as large as the
    cross term: every fp32 Foster kernel (compile-time m = 8, 16, run-time m, several passes, generating mode, m > 64)
    must keep it, at h = 2^-62 and 2^-58."""
    rep = _Report()
    for h in (2.0 ** -62, 2.0 ** -58):
        for m in (4, 8, 16, 17, 65):
            _levy_case(rep, torch.float32, 37, m, True, h)
        for m in (8, 12, 16):
            _cell_levy_case(rep, torch.float32, 9, m, True, h)
    rep.finish()


# ---- GPU: 2^26 channels --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_counter_noise_channel_limit_on_device():
    """One row of 2^26 channels (the most a channel quad's 24 counter bits address) is drawn, and correctly at its last
    quad; 2^26 + 1 channels are refused before anything is launched."""
    lib, key = _lib(), _key()
    n = 2 ** 26 + 1
    bufs = {k: torch.full((n,), float('nan'), device=DEV) for k in LIMIT_BUFFERS}
    bufs['zero'].zero_()
    bufs['one'].fill_(1.0)
    ptrs = {k: b.data_ptr() for k, b in bufs.items()}
    for name, rc in _channel_limit_calls(lib, _cabi.F32, n, ptrs, key.data_ptr()):
        assert rc == _cabi.EINVAL, (name, rc)
    torch.cuda.synchronize()
    assert all(bool(bufs[k].isnan().all()) for k in ('w', 'u', 'h', 'w2', 'h2', 'y1')), 'a refused launch wrote'
    for name, rc in _channel_limit_calls(lib, _cabi.F32, n - 1, ptrs, key.data_ptr()):
        assert rc == 0, (name, rc)
    torch.cuda.synchronize()
    # the first two and the last two quads (the last has channel quad 2^24 - 1)
    cols = np.r_[0:8, n - 9:n - 1]
    full = lambda s: Src(1, np.float32).normal(CELL, s, n - 1).map(lambda a: a[:, cols])   # noqa: E731
    W = math.sqrt(0.5) * full(philox.STREAM_W)
    H = math.sqrt(0.5 / 12) * full(philox.STREAM_H)
    rep = _Report()
    for name, ref in (('w', W), ('h', H), ('y1', W)):
        got = bufs[name][torch.from_numpy(cols).to(DEV)].double().cpu().numpy()[None]
        err = np.abs(got - ref.v)
        if not (err <= ref.e).all():
            rep.bad.append(f'{name} at 2^26 channels: worst err/bound {np.max(err / ref.e):.3g}')
    for k in ('w', 'u', 'h', 'w2', 'h2', 'y1'):
        if not (bool(bufs[k][n - 1].isnan()) and not bool(bufs[k][:n - 1].isnan().any())):
            rep.bad.append(f'{k}: not exactly the 2^26 channels written')
    rep.finish()


# ---- GPU: queries through the public API -----------------------------------------------------------------------------
class _TreeOracle:
    """Evaluates the pieces of a query by walking the interval's own tree: node ids, kinds, bounds and cell_base give
    the walk; a binary child is a bridge on its parent's id, a grid cell is cell_base + k, a run of cells is their merge
    with Levy id mix64(child_id(grid.id, i) ^ mix64(j)); pieces merge left to right, merge_area before merge."""

    def __init__(self, bm, npdt):
        self.bm, self.dt, self.memo = bm, npdt, {}
        self.m = bm._m
        self.src = Src(bm._rows, npdt, bm._row_offset, key=bm._key)

    def value(self, node):
        got = self.memo.get(id(node))
        if got is not None:
            return got
        bm, have_h = self.bm, self.bm._have_H
        if node.parent is None:
            if node.kind == iv._GRID:
                b = node.bounds
                out = cells_f(self.src, node.cell_base, [b[i + 1] - b[i] for i in range(len(b) - 1)], self.m, have_h)
            else:
                out = cells_f(self.src, node.id, [node.end - node.start], self.m, have_h)
                if bm._user_W is not None:
                    out = (Val.exact(bm._user_W.double().cpu().numpy().reshape(bm._rows, self.m), self.dt), out[1])
                if bm._user_H is not None and have_h:
                    out = (out[0], Val.exact(bm._user_H.double().cpu().numpy().reshape(bm._rows, self.m), self.dt))
        elif node.cell_index is not None:
            out = cells_f(self.src, node.id, [node.end - node.start], self.m, have_h)
        else:
            p = node.parent
            W, H = self.value(p)
            out = bridge_chain_f(self.src, W, H, [(p.id, node.is_left, p.start, p.mid, p.end)], self.m)
        self.memo[id(node)] = out
        return out

    def pieces(self, node, a, b):
        if a == node.start and b == node.end:
            return [node]
        if node.kind == iv._BINARY:
            if b <= node.mid:
                return self.pieces(node.left, a, b)
            if a >= node.mid:
                return self.pieces(node.right, a, b)
            return self.pieces(node.left, a, node.mid) + self.pieces(node.right, node.mid, b)
        assert node.kind == iv._GRID, 'the query left a leaf unsplit'
        bounds, out = node.bounds, []
        i = int(np.searchsorted(bounds, a, side='right')) - 1
        if bounds[i] != a:
            hi = min(b, bounds[i + 1])
            out += self.pieces(node.cells[i], a, hi)
            if hi == b:
                return out
            i += 1
        j = int(np.searchsorted(bounds, b, side='right')) - 1
        if j > i:
            out.append((node, i, j))
        if bounds[j] != b:
            out += self.pieces(node.cells[j], bounds[j], b)
        return out

    def piece(self, p):
        if isinstance(p, tuple):
            grid, i, j = p   # (one cell: the cell's own value and id; its node may never have been created)
            b, cid = grid.bounds, (grid.cell_base + i) & MASK
            W, H = cells_f(self.src, cid, [b[k + 1] - b[k] for k in range(i, j)], self.m, self.bm._have_H)
            a_id = cid if j - i == 1 else iv.mix64(iv.child_id(grid.id, i) ^ iv.mix64(j))
            return W, H, b[j] - b[i], b[i], b[j], a_id
        W, H = self.value(p)
        return W, H, p.end - p.start, p.start, p.end, p.id

    def area(self, W, H, h, a_id):
        if not self.bm._have_A or len(self.bm._size) < 2:
            return None
        npairs = max(self.m * (self.m - 1) // 2, 1)
        foster = self.bm._levy_area_approximation == 'foster'
        return levy_f(W, H, h, foster, self.src.normal(a_id, philox.STREAM_A, npairs), self.m)

    def query(self, ta, tb):
        ta_r, tb_r = self.bm._round(ta), self.bm._round(tb)
        ps = self.pieces(self.bm._root, ta_r, tb_r)
        W, H, h, _, _, a_id = self.piece(ps[0])
        A = self.area(W, H, h, a_id)
        for p in ps[1:]:
            Wi, Hi, hi, si, ei, ai = self.piece(p)
            if A is not None:
                A = merge_area_f(A, self.area(Wi, Hi, hi, ai), W, Wi)
            W, H = merge_f(W, H, Wi, Hi, si - ta_r, ei - si, ei - ta_r)
        U = h_to_u_f(W, H, tb - ta) if H is not None else None
        return W, U, A


def _sequence(rng, sequential, tiny=True):
    if sequential:   # the tree grows one level per query: without a cache every query descends from the root
        pts = np.round(np.cumsum(rng.uniform(0.5, 1.5, 41)) / 45, 6)
        return [(float(a), float(b)) for a, b in zip(pts[:-1], pts[1:])]
    qs = [(0.3, 0.7), (0.125, 0.5), (0.25, 0.375), (0.3, 0.31), (0.0, 1.0), (0.4, 0.4), (0.3, 0.7), (0.05, 0.95),
          (0.5, 0.625)]
    if tiny:   # (a halfway tree rounds query times to its tolerance)
        qs += [(0.0, 2.0 ** -58), (0.0, 2.0 ** -62)]
    for _ in range(6):
        a, b = np.sort(np.round(rng.uniform(0, 1, 2), 6))
        qs.append((float(a), float(b)))
    return qs + qs[::-1]


def _run_queries(rep, bm, dtype, label, seq):
    oracle = _TreeOracle(bm, NP[dtype])
    size, m, rows = bm._size, bm._m, bm._rows
    outs = []
    for ta, tb in seq:
        got = bm(ta, tb, return_U=True, return_A=True)
        outs.append(got)
        W, U, A = got
        where = f'{label} [{ta!r}, {tb!r}]'
        if ta == tb:
            if any(x is not None and bool(x.ne(0).any()) for x in got):
                rep.bad.append(f'{where}: nonzero increment of an empty interval')
            continue
        rW, rU, rA = oracle.query(ta, tb)
        for name, t, ref in (('W', W, rW), ('U', U, rU), ('A', A, rA)):
            if ref is None:
                if t is not None and name == 'A' and bool(t.ne(0).any()):
                    rep.bad.append(f'{where}: nonzero Levy area of rank {len(size)}')
                continue
            if tuple(t.shape) != (tuple(size) + ((m,) if name == 'A' else ())):
                rep.bad.append(f'{where} {name}: shape {tuple(t.shape)}')
                continue
            flat = t.reshape(-1)
            rep.check(f'query {name}', dtype, f'{where} {name}', flat, flat, ref)
    return outs


QUERY_CONFIGS = {
    'none': ('none', (7, 5), {}),
    'space-time dt': ('space-time', (7, 5), dict(dt=0.125)),
    'davie dt m=8': ('davie', (3, 8), dict(dt=0.125)),
    'foster dt rank 3': ('foster', (2, 3, 4), dict(dt=0.125)),
    'foster': ('foster', (6, 5), {}),
    'davie rank 1': ('davie', (5,), {}),
    'space-time rank 0': ('space-time', (), {}),
    'foster halfway': ('foster', (4, 4), dict(halfway_tree=True, tol=1e-6)),
    'space-time cache 0': ('space-time', (4, 6), dict(cache_size=0)),
    'foster cache None': ('foster', (4, 6), dict(cache_size=None)),
    'foster shard 2^31': ('foster', (3, 4), dict(shard=1 << 31)),
    'space-time user W H': ('space-time', (5, 3), dict(user='WH')),
    'none user W': ('none', (5, 3), dict(user='W')),
}


def _make_bm(levy, size, kw, dtype, entropy):
    kw = dict(kw)
    shard, user = kw.pop('shard', None), kw.pop('user', '')
    if user:
        gen = torch.Generator(device=DEV).manual_seed(entropy)
        kw['W'] = torch.randn(*size, generator=gen, device=DEV, dtype=dtype)
        if 'H' in user:
            kw['H'] = torch.randn(*size, generator=gen, device=DEV, dtype=dtype) / math.sqrt(12)
    else:
        kw.update(size=size, dtype=dtype, device=DEV)
    bm = iv.BrownianInterval(0.0, 1.0, entropy=entropy, levy_area_approximation=levy, **kw)
    return bm.shard_rows(shard) if shard else bm


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('config', list(QUERY_CONFIGS))
def test_queries_vs_tree_oracle(config, dtype):
    """A seeded sequence of queries (off-grid points, partial cells, runs of cells, pieces of binary nodes, ta == tb,
    intervals down to 2^-62, repeats, reversed order): every W, U and A within the bound of the float64 oracle that
    walks the interval's own tree."""
    levy, size, kw = QUERY_CONFIGS[config]
    rep = _Report()
    bm = _make_bm(levy, size, kw, dtype, entropy=len(config))
    _run_queries(rep, bm, dtype, config, _sequence(np.random.default_rng(len(config)), False,
                                                  tiny=not kw.get('halfway_tree')))
    rep.finish()


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('levy', ['none', 'space-time', 'foster'])
def test_sequential_queries_without_cache(levy, dtype):
    """40 sequential queries grow the tree to depth 40: without a cache each descends from the root, past 24 levels in
    several in-place launches; with an unbounded cache from the last node.  Both must give the same bits, and the
    oracle's values."""
    rep = _Report()
    seq = _sequence(np.random.default_rng(7), True)
    runs = []
    for cache in (0, None):
        bm = _make_bm(levy, (4, 6), dict(cache_size=cache), dtype, entropy=11)
        runs.append(_run_queries(rep, bm, dtype, f'{levy} cache={cache}', seq))
    for k, (x, y) in enumerate(zip(*runs)):
        for a, b in zip(x, y):
            if (a is None) != (b is None) or (a is not None and not torch.equal(a, b)):
                rep.bad.append(f'{levy}: query {k} differs between cache_size=0 and cache_size=None')
    rep.finish()
