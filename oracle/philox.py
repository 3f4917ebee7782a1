"""Philox4x32-10 + Box-Muller normals: CPU restatement of torchsde_b200/csrc/philox.cuh.

Test infrastructure only (see oracle/__init__.py).  The reference draws its normals with
`torch.Generator(device).manual_seed(seed)` + `torch.randn` (torchsde/_brownian/
brownian_interval.py:30-32); that stream is unpinned, so the definition below is the spec.
"""
import numpy as np

M0 = np.uint64(0xD2511F53)
M1 = np.uint64(0xCD9E8D57)
W0 = 0x9E3779B9
W1 = 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)

STREAM_W, STREAM_H, STREAM_X1, STREAM_X2, STREAM_A = 0, 1, 2, 3, 4


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised over numpy uint32 arrays c0..c3; k0,k1 python ints.  Returns 4 uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) for x in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    for _ in range(10):
        p0 = M0 * c0
        p1 = M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c0, c1, c2, c3 = (hi1 ^ c1 ^ np.uint64(k0)), lo1, (hi0 ^ c3 ^ np.uint64(k1)), lo0
        k0 = (k0 + W0) & 0xFFFFFFFF
        k1 = (k1 + W1) & 0xFFFFFFFF
    return tuple(x.astype(np.uint32) for x in (c0, c1, c2, c3))


def _box_muller(a, b):
    r = np.sqrt(-2.0 * np.log(a))
    th = 2.0 * np.pi * b
    return r * np.cos(th), r * np.sin(th)


def _box_muller_f64(a, b):
    """BoxMuller(a, b) with cos / sin of 2 pi b evaluated as the device's sincospi(2 b) does: b is reduced exactly to
    the nearest quarter turn, so both keep their relative accuracy near their zeros.  (`cos(2.0 * pi * b)` rounds the
    angle by up to ~4e-16 absolute, ~20 ulp of a normal close to zero.)"""
    r = np.sqrt(-2.0 * np.log(a))
    t = 4.0 * b                          # exact
    k = np.rint(t)
    th = (t - k) * (0.5 * np.pi)         # t - k exact, |th| <= pi / 4
    c, s = np.cos(th), np.sin(th)
    k = k.astype(np.int64) & 3           # 2 pi b = k pi / 2 + th
    return r * np.choose(k, [c, -s, -c, s]), r * np.choose(k, [s, c, -s, -c])


def normals(key, node_id, stream, rows, m, dtype, row_offset=0, row_ids=None, exact=False):
    """(rows, m) normals of (key, node_id, stream).  Mirrors normal4() for every quad.

    `exact`: return the float64 values the specification of `dtype` is computed in, before the final rounding to
    `dtype` (for a float64 restatement of a kernel that bounds its own rounding errors).

    `row_ids` (optional 1-D integer array) selects arbitrary global rows instead of the contiguous block
    row_offset .. row_offset + rows - 1: rows are independent streams, which is what lets the full-size
    parity tests check a random sample of trajectories of a 65536-row solve.

    fp32: computed in float64 from the float32 uniforms, rounded to float32 at the end (the device
    uses float32 libm: agreement to a few ulp, tests use rtol 2e-6 / atol 2e-6).
    """
    key = int(key)
    node_id = int(node_id)
    k0, k1 = key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF
    qpr = (m + 3) // 4
    if row_ids is not None:
        row_ids = np.asarray(row_ids, dtype=np.uint64)
        rows = int(row_ids.shape[0])
        row = (row_ids + np.uint64(row_offset)).astype(np.uint32)[:, None]
    else:
        row = (np.arange(rows, dtype=np.uint64) + np.uint64(row_offset)).astype(np.uint32)[:, None]
    q = np.arange(qpr, dtype=np.uint32)[None, :]
    id_lo, id_hi = node_id & 0xFFFFFFFF, (node_id >> 32) & 0xFFFFFFFF
    out = np.empty((rows, qpr * 4), dtype=np.float64)
    if np.dtype(dtype) == np.float32:
        x = philox4x32_10(q | np.uint32(stream << 24), row, id_lo, id_hi, k0, k1)
        # radius uniform a = fmaf(uint2float_rn(x), 2^-32, 2^-33): x is rounded to float32 by the conversion, the
        # product with 2^-32 is exact, the sum rounds once more — the device's two instructions, bit for bit
        def radius_uniform(xi):
            a = np.float32(np.float32(xi) * np.float32(2.3283064365386963e-10) + np.float32(1.1641532182693481e-10))
            return a.astype(np.float64)

        # angle fraction b = (x >> 9) * 2^-23 in [0, 1) (the device builds it into a float's mantissa)
        def angle_fraction(xi):
            return (xi >> np.uint32(9)).astype(np.float64) * 2.0 ** -23

        n0, n1 = _box_muller(radius_uniform(x[0]), angle_fraction(x[1]))
        n2, n3 = _box_muller(radius_uniform(x[2]), angle_fraction(x[3]))
        out[:, 0::4], out[:, 1::4], out[:, 2::4], out[:, 3::4] = n0, n1, n2, n3
    else:
        for call in (0, 1):
            x = philox4x32_10(q | np.uint32(stream << 24) | np.uint32(call << 31), row, id_lo, id_hi, k0, k1)
            ua = ((((x[0].astype(np.uint64) << np.uint64(32)) | x[1].astype(np.uint64)) >> np.uint64(11))
                  .astype(np.float64) + 0.5) * 1.1102230246251565e-16
            ub = ((((x[2].astype(np.uint64) << np.uint64(32)) | x[3].astype(np.uint64)) >> np.uint64(11))
                  .astype(np.float64) + 0.5) * 1.1102230246251565e-16
            n0, n1 = _box_muller_f64(ua, ub)
            out[:, 2 * call::4], out[:, 2 * call + 1::4] = n0, n1
    return out[:, :m] if exact else out[:, :m].astype(dtype)
