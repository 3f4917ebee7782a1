"""The general-noise element-wise tapes on the host (no GPU): what GeneralRecorder accepts and rejects, the
contraction order the generated source spells out for every m (the route of the unfused launch: row-wise, tile or
generic kernel) and both alignments of g, and the calls the library refuses before launching anything."""
import ctypes

import pytest
import torch

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise

B, D = 6, 8


def record(f, g, m, pattern='fg', dtype=torch.float32, layout=None):
    y = torch.rand(B, D, dtype=dtype) + 0.1
    t = torch.tensor(0.25, dtype=dtype)
    rec = pointwise.GeneralRecorder(y, t, pattern, m, layout=layout)
    for kind in pattern:
        rec.evaluation(kind, (lambda: f(t, y)) if kind == 'f' else (lambda: g(t, y)), t, y)
    return rec, rec.finish()


def params(m, dtype=torch.float32):
    gen = torch.Generator().manual_seed(0)
    return (torch.rand(D, generator=gen).to(dtype), torch.rand(D, m, generator=gen).to(dtype),
            torch.rand(m, generator=gen).to(dtype))


def accepted(m=16, dtype=torch.float32):
    mu, S, v = params(m, dtype)
    return {
        'correlated_gbm': (lambda t, y: mu * y, lambda t, y: y.unsqueeze(-1) * S),
        'none_index': (lambda t, y: mu * y, lambda t, y: y[..., None] * S),
        'ou_expand': (lambda t, y: mu - y, lambda t, y: S.expand(B, D, m)),
        'time_additive': (lambda t, y: mu / torch.sqrt(1. + t) - y,
                          lambda t, y: (S / torch.sqrt(1. + t)).expand(B, D, m)),
        'channel_row': (lambda t, y: mu * y, lambda t, y: (y * mu).unsqueeze(-1) * v),
        'lifted_expand': (lambda t, y: mu * y, lambda t, y: (2.0 * y).unsqueeze(-1).expand(B, D, m)),
        'where_clamp': (lambda t, y: mu * y,
                        lambda t, y: torch.where(y[..., None] > 0.5, y[..., None] * S, torch.clamp(S, 0.1, 0.6))),
    }


@pytest.mark.parametrize('kind', sorted(accepted()))
@pytest.mark.parametrize('pattern', ['fg', 'fgfg'])  # Euler, midpoint
def test_the_recorder_accepts_the_general_shapes(kind, pattern):
    f, g = accepted()[kind]
    rec, res = record(f, g, 16, pattern)
    assert res is not None, rec.reason
    src = _cabi.general_pointwise_source(res[0], torch.float32, D, 16)
    assert 'tsde_pw_general_euler_single' in src and 'tsde_pw_general_midpoint_multi' in src


def test_operand_kinds():
    _, res = record(*accepted()['channel_row'], 16)
    kinds = {res[0].operand[k].kind for k in range(res[0].n_operands)}
    assert kinds == {_cabi.PW_CHANNEL, _cabi.PW_M}
    _, res = record(*accepted()['ou_expand'], 16)
    k = res[0].g_src - _cabi.PW_OPERAND0
    assert 0 <= k < res[0].n_operands and res[0].operand[k].kind == _cabi.PW_DM


@pytest.mark.parametrize('case', ['stack', 'cat', 'repeat', 'tanh', 'exp', 'sum', 'factory', 'foreign', 'y_unlifted',
                                  'f_per_channel'])
def test_the_recorder_rejects(case):
    m = 4
    mu, S, _ = params(m)
    foreign = torch.rand(B, D, m)
    gs = {
        'stack': lambda t, y: torch.stack([y] * m, -1),
        'cat': lambda t, y: torch.cat([y.unsqueeze(-1)] * m, -1),
        'repeat': lambda t, y: S.unsqueeze(0).repeat(B, 1, 1),
        'tanh': lambda t, y: torch.tanh(y).unsqueeze(-1) * S,
        'exp': lambda t, y: torch.exp(y).unsqueeze(-1) * S,
        'sum': lambda t, y: y.sum(-1)[:, None, None] * S,
        'factory': lambda t, y: y.unsqueeze(-1) * torch.ones(B, D, m),
        'foreign': lambda t, y: y.unsqueeze(-1) * foreign,
        'y_unlifted': lambda t, y: y.unsqueeze(0).expand(m, B, D).permute(1, 2, 0) * 1.0,
        'f_per_channel': lambda t, y: y.unsqueeze(-1) * S,
    }
    f = (lambda t, y: y.unsqueeze(-1) * S) if case == 'f_per_channel' else (lambda t, y: mu * y)
    rec, res = record(f, gs[case], m)
    assert res is None and rec.reason


ROWWISE, TILE, GENERIC = 'rowwise', 'tile', 'generic'


def _route(m, quads):
    """cabi.cu and launch_gen, restated: m == 1 the row-wise kernels; the tile kernels for m / 4 a power of two <= 32
    with g loadable as quads; otherwise gen_kernel (gen_wide_kernel only past 40 KiB of increments per row, far above
    TSDE_PW_GENERAL_MAX_M)."""
    if m == 1:
        return ROWWISE
    mq = m // 4
    if quads and m % 4 == 0 and 1 <= mq <= 32 and mq & (mq - 1) == 0:
        return TILE
    return GENERIC


def _expected_contraction(route, m, fs='f'):
    """The summation order of each route, as the statements the generated source must hold."""
    if route == ROWWISE:
        return ['const T acc = G(0) * w[0];']
    if route == GENERIC:
        return ['T acc = T(0);'] + [f'acc = acc + G({k}) * w[{k}];' for k in range(m)]
    out, level = [], []
    for q in range(m // 4):
        out.append(f'T s{q} = fma{fs}(G({4 * q}), w[{4 * q}], T(0));')
        out += [f's{q} = fma{fs}(G({4 * q + j}), w[{4 * q + j}], s{q});' for j in range(1, 4)]
        level.append(f's{q}')
    lvl = 0
    while len(level) > 1:  # the xor-butterfly: a pairwise tree in natural order
        up = []
        for p in range(0, len(level), 2):
            name = f'a{lvl}_{p // 2}'
            out.append(f'const T {name} = {level[p]} + {level[p + 1]};')
            up.append(name)
        level, lvl = up, lvl + 1
    return out + [f'const T acc = {level[0]};']


def _contraction(src):
    lines = [ln.strip() for ln in src.splitlines()]
    return lines[lines.index('};', lines.index('auto G = [&](int k) -> T {')) + 1:lines.index('out[j] = acc;')]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', list(range(1, _cabi.PW_GENERAL_MAX_M + 1)))
def test_the_generated_contraction_follows_the_route(m, dtype):
    fs = 'f' if dtype == torch.float32 else ''
    rec, res = record(*accepted(m, dtype)['correlated_gbm'], m, dtype=dtype)
    assert res is not None, rec.reason
    assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
        _route(m, True), m, fs)
    # additive noise returning the user's (d, m) block: the unfused launch reads it where it is, so a misaligned
    # block takes gen_kernel's order
    store = torch.zeros(D * m + 1, dtype=dtype)
    for S, quads in ((torch.rand(D, m, dtype=dtype), True), (store[1:].view(D, m), False)):
        rec, res = record(lambda t, y: -y, lambda t, y: S.expand(B, D, m), m, dtype=dtype)
        assert res is not None, rec.reason
        aligned = S.data_ptr() % 16 == 0
        assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
            _route(m, quads and aligned), m, fs)


def test_wider_noise_is_refused():
    rec, res = record(*accepted(4)['correlated_gbm'], 4)
    prog = res[0]
    assert _cabi.general_pointwise_source(prog, torch.float32, D, _cabi.PW_GENERAL_MAX_M + 1) is None


def test_bad_calls_are_refused_without_a_launch():
    lib = _cabi.lib()
    _, res = record(*accepted(4)['correlated_gbm'], 4)
    prog = res[0]
    n0 = lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL)
    nz = _cabi.Noise()
    nz.source = _cabi.SRC_COUNTER
    steps = (_cabi.PwStep * 1)()
    steps[0].t0, steps[0].y1 = 16, 32
    general = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, 4, None)
    diagonal = _cabi.Launch(_cabi.F32, _cabi.NOISE_DIAGONAL, 4, D, D, None)
    wide = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, _cabi.PW_GENERAL_MAX_M + 1, None)
    p = ctypes.byref(prog)
    for L, n_steps, y0 in ((diagonal, 1, 16), (wide, 1, 16), (general, 0, 16), (general, _cabi.PW_MAX_STEPS + 1, 16),
                           (general, 1, None)):
        assert lib.tsde_solve_euler_pointwise(ctypes.byref(L), ctypes.byref(nz), p, y0, steps,
                                              n_steps) == _cabi.EINVAL
    for method, t0 in ((_cabi.PC_MIDPOINT, None), (_cabi.PC_HEUN, 16), (_cabi.PC_EULER_HEUN, 16)):
        assert lib.tsde_step_predictor_corrector_pointwise(ctypes.byref(general), ctypes.byref(nz), p, 16, t0, 16,
                                                           method, 0.1, 0.05, 32) == _cabi.EINVAL
    memory = _cabi.Noise()
    memory.source = _cabi.SRC_MEMORY
    assert lib.tsde_solve_euler_pointwise(ctypes.byref(general), ctypes.byref(memory), p, 16, steps, 1) == _cabi.EINVAL
    # a DM operand read by f
    bad = _cabi.Pointwise.from_buffer_copy(prog)
    bad.operand[bad.n_operands].kind, bad.operand[bad.n_operands].ptr = _cabi.PW_DM, 64
    bad.instr[0].b = _cabi.PW_OPERAND0 + bad.n_operands
    bad.n_operands += 1
    assert lib.tsde_solve_euler_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(bad), 16, steps,
                                          1) == _cabi.EINVAL
    assert _cabi.general_pointwise_source(bad, torch.float32, D, 4) is None
    # a program not tagged as the general layout
    untagged = _cabi.Pointwise.from_buffer_copy(prog)
    untagged.reserved = 0
    assert lib.tsde_solve_euler_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(untagged), 16, steps,
                                          1) == _cabi.EINVAL
    assert _cabi.general_pointwise_source(untagged, torch.float32, D, 4) is None
    assert lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL) == n0
