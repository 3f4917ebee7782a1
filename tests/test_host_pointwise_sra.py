"""The additive-noise SRK (sra1) element-wise step on the host (no GPU): what GeneralRecorder accepts and rejects for
the step's four evaluations ('fggf'), the contraction order the generated sra1 source spells out for every m (the
route of the unfused sra1 launches, which call launch_gen directly: m = 1 takes gen_kernel's order there), the
unchanged Euler / midpoint unit, the calls the library refuses before launching anything, and a dry run of the
solver reaching the GENERAL launch of tsde_step_srk_diag_pointwise that runs the step."""
import ctypes

import pytest
import torch

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import problems
from .test_host_dry_run import dry  # noqa: F401  (the fixture)
from .test_host_pointwise_general import (B, D, GENERIC, _contraction, _expected_contraction, _route, accepted,
                                          record)

ADDITIVE = ['ou_expand', 'time_additive', 'where_clamp']


def record_sra(f, g, m, dtype=torch.float32, g_b=None, f_1=None):
    """GeneralRecorder over one sra1 step's evaluations f0, gA, gB, f1 (`g_b` / `f_1`: another gB / f1)."""
    y = torch.rand(B, D, dtype=dtype) + 0.1
    t = torch.tensor(0.25, dtype=dtype)
    rec = pointwise.GeneralRecorder(y, t, pointwise.SRA_PATTERN, m)
    for kind, fn in zip('fggf', (f, g, g_b or g, f_1 or f)):
        rec.evaluation(kind, lambda: fn(t, y), t, y)
    return rec, rec.finish()


def sra_route(m, quads):
    """The route of the unfused sra1 launches: launch_gen's, whose m = 1 is gen_kernel's left-to-right sum from 0."""
    route = _route(m, quads)
    return GENERIC if m == 1 else route


@pytest.mark.parametrize('kind', ADDITIVE)
def test_the_recorder_accepts_the_additive_shapes_and_tags_them(kind):
    rec, res = record_sra(*accepted()[kind], 16)
    assert res is not None, rec.reason
    assert res[0].reserved == _cabi.PW_LAYOUT_GENERAL_SRA
    src = _cabi.general_pointwise_source(res[0], torch.float32, D, 16)
    assert 'tsde_pw_general_sra1_single' in src and 'tsde_pw_general_sra1_multi' in src
    assert 'tsde_pw_general_euler_single' not in src


def test_evaluations_that_differ_are_rejected():
    mu, S = torch.rand(D), torch.rand(D, 4)
    f, g = (lambda t, y: mu - y), (lambda t, y: S.expand(B, D, 4))
    # a Python branch on t: g at t0 is another program than g at t0 + dt
    rec, res = record_sra(f, g, 4, g_b=lambda t, y: (S * 2.0).expand(B, D, 4))
    assert res is None and 'g evaluations differ' in rec.reason
    rec, res = record_sra(f, g, 4, f_1=lambda t, y: mu - 2.0 * y)
    assert res is None and 'f evaluations differ' in rec.reason
    # and the step's evaluations are four
    y, t = torch.rand(B, D), torch.tensor(0.25)
    rec = pointwise.GeneralRecorder(y, t, pointwise.SRA_PATTERN, 4)
    for kind in 'fgf':
        rec.evaluation(kind, lambda: f(t, y) if kind == 'f' else g(t, y), t, y)
    assert rec.finish() is None and rec.reason


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('m', list(range(1, _cabi.PW_GENERAL_MAX_M + 1)))
def test_the_generated_sra1_contraction_follows_the_route(m, dtype):
    fs = 'f' if dtype == torch.float32 else ''
    rec, res = record_sra(*accepted(m, dtype)['where_clamp'], m, dtype=dtype)
    assert res is not None, rec.reason
    assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
        sra_route(m, True), m, fs)
    # a DM operand as g: the unfused launches read the user's block where it is, so a misaligned one takes
    # gen_kernel's order
    store = torch.zeros(D * m + 1, dtype=dtype)
    for S, quads in ((torch.rand(D, m, dtype=dtype), True), (store[1:].view(D, m), False)):
        rec, res = record_sra(lambda t, y: -y, lambda t, y: S.expand(B, D, m), m, dtype=dtype)
        assert res is not None, rec.reason
        aligned = S.data_ptr() % 16 == 0
        assert _contraction(_cabi.general_pointwise_source(res[0], dtype, D, m)) == _expected_contraction(
            sra_route(m, quads and aligned), m, fs)


@pytest.mark.parametrize('m', [1, 3, 16])
def test_the_euler_midpoint_unit_is_unchanged(m):
    """A LAYOUT_GENERAL program's source is the Euler / midpoint unit (m = 1: the row-wise single product), and the
    same program re-tagged SRA gives the sra1 unit with the same `Prog`."""
    rec, res = record(*accepted(m)['correlated_gbm'], m)
    assert res is not None, rec.reason
    prog = res[0]
    assert prog.reserved == _cabi.PW_LAYOUT_GENERAL
    src = _cabi.general_pointwise_source(prog, torch.float32, D, m)
    assert 'tsde_pw_general_midpoint_multi' in src and 'sra1' not in src
    if m == 1:
        assert _contraction(src) == ['const T acc = G(0) * w[0];']
    sra = _cabi.Pointwise.from_buffer_copy(prog)
    sra.reserved = _cabi.PW_LAYOUT_GENERAL_SRA
    src_sra = _cabi.general_pointwise_source(sra, torch.float32, D, m)
    prog_part = src.split('\nextern "C"')[0]
    assert src_sra.split('\nextern "C"')[0] == (prog_part if m > 1 else prog_part.replace(
        'const T acc = G(0) * w[0];', 'T acc = T(0);\n      acc = acc + G(0) * w[0];'))


def test_bad_calls_are_refused_without_a_launch():
    lib = _cabi.lib()
    _, res = record_sra(*accepted(4)['ou_expand'], 4)
    prog = res[0]
    n0 = lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL)
    nz = _cabi.Noise()
    nz.source = _cabi.SRC_COUNTER
    general = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, 4, None)
    diagonal = _cabi.Launch(_cabi.F32, _cabi.NOISE_DIAGONAL, 4, D, D, None)
    wide = _cabi.Launch(_cabi.F32, _cabi.NOISE_GENERAL, 4, D, _cabi.PW_GENERAL_MAX_M + 1, None)
    half = _cabi.Launch(_cabi.F32 | _cabi.FMT_BF16 << 8, _cabi.NOISE_GENERAL, 4, D, 4, None)

    def step(L, p, noise=nz, times=(16, 16, 16)):
        return lib.tsde_step_srk_diag_pointwise(ctypes.byref(L), ctypes.byref(noise), ctypes.byref(p), 16, *times,
                                                None, 0.1, 10.0, 0.0, 0.0, 32)

    for L in (diagonal, wide, half):
        assert step(L, prog) == _cabi.EINVAL
    for times in ((None, 16, 16), (16, None, 16), (16, 16, None)):
        assert step(general, prog, times=times) == _cabi.EINVAL
    memory = _cabi.Noise()
    memory.source = _cabi.SRC_MEMORY
    assert step(general, prog, memory) == _cabi.EINVAL
    flagged = _cabi.Noise()
    flagged.source, flagged.flags = _cabi.SRC_COUNTER, _cabi.FLAG_G_BROADCAST
    assert step(general, prog, flagged) == _cabi.EINVAL
    # programs without the SRA tag: untagged, or the Euler / midpoint layout
    for tag in (0, _cabi.PW_LAYOUT_GENERAL):
        other = _cabi.Pointwise.from_buffer_copy(prog)
        other.reserved = tag
        assert step(general, other) == _cabi.EINVAL
    # ... and the Euler and midpoint entries refuse an SRA program
    steps = (_cabi.PwStep * 1)()
    steps[0].t0, steps[0].y1 = 16, 32
    assert lib.tsde_solve_euler_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(prog), 16, steps,
                                          1) == _cabi.EINVAL
    assert lib.tsde_step_predictor_corrector_pointwise(ctypes.byref(general), ctypes.byref(nz), ctypes.byref(prog),
                                                       16, 16, 16, _cabi.PC_MIDPOINT, 0.1, 0.05, 32) == _cabi.EINVAL
    assert _cabi.general_pointwise_source(prog, torch.float32, D, _cabi.PW_GENERAL_MAX_M + 1) is None
    assert lib.tsde_kernel_launches(_cabi.KERNEL_PW_GENERAL) == n0


@pytest.mark.parametrize('options', [{}, {'cuda_graph': True}])
def test_an_additive_expand_srk_solve_reaches_the_fused_step(dry, options):  # noqa: F811
    d, m = 3, 2
    sde = problems.make('additive_expand', d, m, 'ito', dtype=torch.float32)
    bm = tsde.BrownianInterval(0.0, 0.25, size=(4, m), dtype=torch.float32, device='cpu',
                               levy_area_approximation='space-time')
    with torch.no_grad():
        tsde.sdeint(sde, torch.ones(4, d), torch.tensor([0.0, 0.125, 0.25]), bm=bm, method='srk', dt=0.0625,
                    options=options)
    assert dry.calls.get('tsde_pointwise_compile', 0) == 1
    assert dry.calls.get('tsde_step_srk_diag_pointwise', 0) > 0
    # the recording step ran the unfused pair
    assert dry.calls.get('tsde_step_srk_additive', 0) >= 1
