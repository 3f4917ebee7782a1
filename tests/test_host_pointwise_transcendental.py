"""The transcendental ops of the element-wise tapes on the host (no GPU): exp, log, sin, cos, tanh, log1p, expm1, rsqrt,
sigmoid, a general power and the tanh / sigmoid backward ops, which the tapes take only with
options={'transcendental': True} and only in the layouts the library compiles (Milstein, its adaptive proposal, and
the general / additive-noise Euler, midpoint and sra1 kernels).  Here: which recorders accept them, the opcodes they
record (the vjp's backward ops, the pow ladder), the NVRTC version guard, the generated sources (calls of the helper
functions, and the digests that pin every generator's text, with and without them), the refusal of the interpreted
entry points, and the helper and program translation units compiled and linked as the library links them, with their
registers and stack."""
import ctypes
import hashlib
import re

import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import test_host_pointwise as milstein
from . import test_host_pointwise_compile as compile_
from . import test_host_pointwise_general as general
from . import test_host_pointwise_select as select
from . import test_host_pointwise_validation as validation

ROWS, D = milstein.ROWS, milstein.D

# op name -> (the element-wise function, its opcode)
OPS = {
    'exp': (torch.exp, _cabi.PW_EXP), 'log': (torch.log, _cabi.PW_LOG), 'sin': (torch.sin, _cabi.PW_SIN),
    'cos': (torch.cos, _cabi.PW_COS), 'tanh': (torch.tanh, _cabi.PW_TANH), 'log1p': (torch.log1p, _cabi.PW_LOG1P),
    'expm1': (torch.expm1, _cabi.PW_EXPM1), 'rsqrt': (torch.rsqrt, _cabi.PW_RSQRT),
    'sigmoid': (torch.sigmoid, _cabi.PW_SIGMOID), 'pow': (lambda x: x ** 1.7, _cabi.PW_POW),
}


def _milstein(op, where, transcendental=True, dtype=torch.float32):
    """A Milstein tape with op in f ('f') or in g ('g', so in the vjp too), recorded as BaseMilstein._step does."""
    fn = OPS[op][0]
    f = (lambda t, y, p: fn(y) * p['a']) if where == 'f' else (lambda t, y, p: p['a'] * y)
    g = (lambda t, y, p: fn(y) * p['b']) if where == 'g' else (lambda t, y, p: p['b'] * y)
    cls = lambda y, t: pointwise.Recorder(y, t, transcendental)  # noqa: E731
    rec, res, _, _ = milstein._record(f, g, dtype, cls)
    return rec, res


def _general(op, pattern='fg', transcendental=True, m=4, dtype=torch.float32, layout=None):
    """A general-noise tape whose g is op(y)[..., None] * S (TanhGeneral's shape)."""
    fn = OPS[op][0]
    mu, S, _ = general.params(m, dtype)
    y = torch.rand(general.B, general.D, dtype=dtype) + 0.1
    t = torch.tensor(0.25, dtype=dtype)
    rec = pointwise.GeneralRecorder(y, t, pattern, m, transcendental, layout)
    for kind in pattern:
        fg = (lambda: mu * y) if kind == 'f' else (lambda: fn(y)[..., None] * S)
        rec.evaluation(kind, fg, t, y)
    return rec, rec.finish()


def _ops(prog):
    return [prog.instr[i].op for i in range(prog.n_instr)]


@pytest.mark.parametrize('where', ['f', 'g'])
@pytest.mark.parametrize('op', sorted(OPS))
def test_milstein_takes_each_op_with_the_option_only(op, where):
    rec, res = _milstein(op, where)
    assert res is not None, rec.reason
    assert OPS[op][1] in _ops(res[0])
    rec, res = _milstein(op, where, transcendental=False)
    assert res is None and rec.reason


@pytest.mark.parametrize('pattern', ['fg', 'fgfg', 'fggf'])  # Euler, midpoint, sra1
@pytest.mark.parametrize('op', sorted(OPS))
def test_the_general_layouts_take_each_op_with_the_option_only(op, pattern):
    rec, res = _general(op, pattern)
    assert res is not None, rec.reason
    assert OPS[op][1] in _ops(res[0])
    rec, res = _general(op, pattern, transcendental=False)
    assert res is None and rec.reason


@pytest.mark.parametrize('pattern', ['fgfgfgg', 'fgfg', 'fgg', 'fg'])  # SRK, Heun / midpoint, Euler-Heun, Euler
@pytest.mark.parametrize('op', sorted(OPS))
def test_the_interpreted_layouts_reject_each_op_even_with_the_option(op, pattern):
    fn = OPS[op][0]
    y = torch.rand(ROWS, D) + 0.25
    t = torch.tensor(0.5)
    a = torch.rand(D) + 0.5
    rec = pointwise.SrkRecorder(y, t, pattern, _cabi.PW_MAX_REGS, transcendental=True)
    for kind in pattern:
        rec.evaluation(kind, (lambda: a * y) if kind == 'f' else (lambda: fn(y) * a), t, y)
    assert rec.finish() is None and 'compiled kernels only' in rec.reason


@pytest.mark.parametrize('op,backward', [('tanh', _cabi.PW_TANH_BACKWARD), ('sigmoid', _cabi.PW_SIGMOID_BACKWARD)])
def test_the_vjp_of_tanh_and_sigmoid_holds_the_backward_opcode(op, backward):
    rec, (prog, _) = _milstein(op, 'g')
    ops = _ops(prog)
    assert backward in ops[prog.n_fg:] and backward not in ops[:prog.n_fg]
    # (grad, result): the forward result is the register f / g computed it in
    assert prog.instr[ops.index(backward)].b < _cabi.PW_OPERAND0 and ops[:prog.n_fg].count(OPS[op][1]) == 1


# exponent -> the opcodes of pow(y, p) (2 and 3: multiplications; -1 and -2: divisions of 1; else the helpers)
LADDER = {0.5: [_cabi.PW_SQRT], -0.5: [_cabi.PW_RSQRT], -1: [_cabi.PW_DIV], 2: [_cabi.PW_MUL],
          3: [_cabi.PW_MUL, _cabi.PW_MUL], -2: [_cabi.PW_MUL, _cabi.PW_DIV], 2.5: [_cabi.PW_POW],
          -3: [_cabi.PW_POW], 1.7: [_cabi.PW_POW]}


def _pow_program(p, transcendental=True, dtype=torch.float32):
    cls = lambda y, t: pointwise.Recorder(y, t, transcendental)  # noqa: E731
    return milstein._record(lambda t, y, q: y ** p, lambda t, y, q: q['b'] * y, dtype, cls)[:2]


@pytest.mark.parametrize('p', sorted(LADDER))
def test_the_pow_ladder(p):
    rec, res = _pow_program(p)
    assert res is not None, rec.reason
    prog = res[0]
    assert _ops(prog)[:prog.n_fg - 1] == LADDER[p]  # (then g = b * y)
    last = prog.instr[prog.n_fg - 2]
    if LADDER[p][-1] == _cabi.PW_DIV:  # 1 / x
        assert prog.operand[last.a - _cabi.PW_OPERAND0].imm == 1.0
    if LADDER[p] == [_cabi.PW_POW]:  # the exponent as ATen rounds it, an immediate
        o = prog.operand[last.b - _cabi.PW_OPERAND0]
        assert o.kind == _cabi.PW_IMM and o.imm == float(np.float32(p))
    if p != 2:
        rec, res = _pow_program(p, transcendental=False)
        assert res is None and 'exponent' in rec.reason


@pytest.mark.parametrize('p', [0, 1, 0.0, 1.0])
def test_pow_zero_and_one_stay_rejected(p):
    rec, res = _pow_program(p)
    assert res is None and 'exponent' in rec.reason


def test_pow_exponent_rounds_to_the_state_dtype_before_the_ladder():
    """ATen casts the exponent to the dtype and then compares with 2, 3 and -2 (0.5, -0.5 and -1 before the cast)."""
    rec, (prog, _) = _pow_program(3 + 1e-9)
    assert _ops(prog)[:2] == [_cabi.PW_MUL, _cabi.PW_MUL]
    rec, (prog, _) = _pow_program(3 + 1e-9, dtype=torch.float64)
    assert _ops(prog)[0] == _cabi.PW_POW


@pytest.mark.parametrize('version', [(12, 6), (13, 0), None])
def test_the_nvrtc_version_guard(version, monkeypatch):
    monkeypatch.setattr(_cabi, 'nvrtc_version', lambda: version)
    rec, res = _milstein('tanh', 'g')
    assert res is None and 'NVRTC' in rec.reason
    rec, res = _general('exp')
    assert res is None and 'NVRTC' in rec.reason
    # a tape without the ops does not ask
    rec, res, _, _ = milstein._record(*milstein.ACCEPTED['gbm_ito'], torch.float32,
                                      lambda y, t: pointwise.Recorder(y, t, True))
    assert res is not None, rec.reason


def test_no_nvjitlink_rejects(monkeypatch):
    monkeypatch.setattr(_cabi, 'nvjitlink', lambda: None)
    rec, res = _milstein('exp', 'f')
    assert res is None and 'nvJitLink' in rec.reason


def test_the_guard_compares_with_the_cuda_pytorch_was_built_with(monkeypatch):
    want = torch.version.cuda
    if want is None:
        pytest.skip('a PyTorch without CUDA')
    monkeypatch.setattr(_cabi, 'nvrtc_version', lambda: tuple(int(x) for x in want.split('.')[:2]))
    assert pointwise.nvrtc_mismatch() is None


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('op', sorted(OPS))
def test_generated_sources_call_the_helpers(op, dtype):
    T = 'float' if dtype == torch.float32 else 'double'
    name = {'pow': 'pow'}.get(op, op)
    _, (prog, _) = _milstein(op, 'g', dtype=dtype)
    src = _cabi.pointwise_source(prog, dtype)
    assert f'__device__ {T} pw_{name}({T}' in src and re.search(rf'= pw_{name}\(y\[j\]', src)
    _, (prog, _) = _general(op, 'fg', dtype=dtype)
    src = _cabi.general_pointwise_source(prog, dtype, general.D, 4)
    # the per-element op runs once per lane, before the channel loop
    narrow = src[src.index('void gp('):src.index('auto G = [&]')]
    assert re.search(rf'n\d+\[j\] = pw_{name}\(y\[j\]', narrow)


# sha256 of the generated sources of the programs below, in the order below.  host, select and general-fg / -fggf:
# the existing tests' programs, written by the generators before the transcendental ops existed.  general-eulerheun /
# -revheun: those programs under the Euler-Heun and reversible-Heun tags.  widths: every tagged unit at Brownian
# widths around each route's edges, with g also the user's (d, m) block, 16-byte aligned or not (so the row-wise,
# tile and generic contractions all appear).  transcendental: a program per op, Milstein and every general unit.
SOURCES = {
    'host-float32': 'c47308dbab452dbf4772981850f754c9b50c0e3389e088f2b07ac335c19dbf6a',
    'host-float64': '60dca03978eff78bc00df009e8bd6b62b72ab41c552bded8e6925ae02713474d',
    'select-float32': 'b7ba3c78f33a8ca087664c74b88298577b11cff290962ea67e8bcec0815d44b6',
    'select-float64': 'b0c3490642560c11855407cb28f5eafe9b5a6f4a8962551b49b48a6b27414ce5',
    'general-fg-float32': 'af3c95586aab9d5ab789eb2b26f4c95735cfe35d2c7ca9d56b8e9d5de689cee0',
    'general-fg-float64': '9670665a269f1c6499ce1e367a503e3db2a37af3405c24370f84c5f3612fd627',
    'general-fggf-float32': '0f8938695716053e0b5267b10c235906d18e53f7de2f34fae0b60f39daf89698',
    'general-fggf-float64': 'cf34954570a1b377e0eaa00f46b381969773ceb6929fadf14372bd10729b819b',
    'general-eulerheun-float32': 'c0ea862bdce9217b9ad7f2126e2e03d9184f1c9107e4a965bc4c857df0cbf9ba',
    'general-eulerheun-float64': 'ce98b518dbcc370cc58850544d04e55904811d65af5b057dfe638b5a0cf5122d',
    'general-revheun-float32': '4cf36b5a13b3ee199589bb9a571076aa7bab818028105aae6359358cb4aef2fa',
    'general-revheun-float64': '92bb442f095a45fab2217ad58ceffedcc12e840a235f2261290b0aab3773e29b',
    'widths-float32': 'd9e0b58f710d5af3ec61647161ce1b42e77c2ff3b0c215fe171723105b7c7bf4',
    'widths-float64': '08e074cfd1cb32269ba0170d736e266470d1086a508b403e8b22376ecfc94ddf',
    'transcendental-float32': '80be0f6f672771e5e71b2d23809664bbe3707e97b096db25d11b4948b82e712c',
    'transcendental-float64': '6ed18d3ca8a7f4d7b030aedb0f77636d58597f2262a483271e76ec91193ce0fb',
}

# the general units: (evaluation pattern, layout tag)
UNITS = {'fg': ('fg', _cabi.PW_LAYOUT_GENERAL), 'fggf': ('fggf', _cabi.PW_LAYOUT_GENERAL_SRA),
         'eulerheun': ('fgg', _cabi.PW_LAYOUT_GENERAL_EULER_HEUN),
         'revheun': ('fg', _cabi.PW_LAYOUT_GENERAL_REVERSIBLE_HEUN)}
WIDTHS = (1, 2, 4, 5, 8, 17, 32)


def _sources(key):
    """The generated sources that `key`'s digest covers, in order."""
    parts = key.split('-')
    dtype = getattr(torch, parts[-1])
    if parts[0] in ('host', 'select'):
        table = milstein.ACCEPTED if parts[0] == 'host' else select.ACCEPTED
        for name in sorted(table):
            _, res, _, _ = milstein._record(*table[name], dtype)
            yield _cabi.pointwise_source(res[0], dtype)
    elif parts[0] == 'general':
        pattern, layout = UNITS[parts[1]]
        for m in (1, 3, 16):
            acc = general.accepted(m, dtype)
            for name in sorted(acc):
                _, res = general.record(*acc[name], m, pattern, dtype, layout)
                if res is not None:
                    yield _cabi.general_pointwise_source(res[0], dtype, general.D, m)
    elif parts[0] == 'widths':
        for m in WIDTHS:
            store = torch.zeros(general.D * m + 1, dtype=dtype)
            blocks = (torch.rand(general.D, m, dtype=dtype), store[1:].view(general.D, m))
            for unit in sorted(UNITS):
                pattern, layout = UNITS[unit]
                acc = general.accepted(m, dtype)
                fgs = [acc[name] for name in sorted(acc)]
                fgs += [(lambda t, y: -y, lambda t, y, S=S: S.expand(general.B, general.D, m)) for S in blocks]
                for f, g in fgs:
                    rec, res = general.record(f, g, m, pattern, dtype, layout)
                    assert res is not None, rec.reason
                    yield _cabi.general_pointwise_source(res[0], dtype, general.D, m)
    else:
        for op in sorted(OPS):
            for where in 'fg':
                yield _cabi.pointwise_source(_milstein(op, where, dtype=dtype)[1][0], dtype)
            for unit in sorted(UNITS):
                pattern, layout = UNITS[unit]
                for m in (1, 4, 5):
                    rec, res = _general(op, pattern, m=m, dtype=dtype, layout=layout)
                    assert res is not None, rec.reason
                    yield _cabi.general_pointwise_source(res[0], dtype, general.D, m)


@pytest.mark.parametrize('key', sorted(SOURCES))
def test_the_sources_of_programs_without_the_ops_are_unchanged(key):
    h = hashlib.sha256()
    for src in _sources(key):
        assert src is not None
        h.update(src.encode())
    assert h.hexdigest() == SOURCES[key]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('op', ['exp', 'tanh', 'pow', 'tanh_backward', 'sigmoid_backward'])
def test_the_interpreted_entry_points_refuse_the_opcodes_before_a_launch(op, dtype):
    step = validation._Step(dtype, validation.DEVICE)
    code = {'exp': _cabi.PW_EXP, 'tanh': _cabi.PW_TANH, 'pow': _cabi.PW_POW,
            'tanh_backward': _cabi.PW_TANH_BACKWARD, 'sigmoid_backward': _cabi.PW_SIGMOID_BACKWARD}[op]
    prog = validation._srk(step.mem)
    prog.instr[2].op = code  # g = op(r0, y)
    before = step.launches()
    assert step.srk(prog) == _cabi.EINVAL
    assert step.launches() == before


def test_pow_needs_an_immediate_exponent():
    _, (prog, _) = _pow_program(1.7)
    assert _cabi.pointwise_source(prog, torch.float32) is not None
    ins = prog.instr[0]
    ins.b = _cabi.PW_SRC_Y
    assert _cabi.pointwise_source(prog, torch.float32) is None
    assert _cabi.compile_pointwise(prog, torch.float32) == _cabi.EINVAL


# -- the translation units, compiled and linked as the library does (pw_nvrtc_linked) ----------------------------------
def _helpers_source():
    """kPwHelpers, the helper translation unit, as the library holds it."""
    text = open(compile_.os.path.join(compile_.CSRC, 'pointwise.cu')).read()
    body = re.search(r'static const char kPwHelpers\[\] =\n(.*?);\n', text, re.S).group(1)
    return ''.join(bytes(s, 'utf-8').decode('unicode_escape') for s in re.findall(r'"((?:[^"\\]|\\.)*)"', body))


def _cubin(src, options, name='tsde_pw_milstein.cu'):
    nv = compile_._nvrtc()
    names = list(compile_.HEADERS) + ['stdint.h']
    bodies = [open(p).read() for p in compile_.HEADERS.values()] + [compile_.STDINT]
    arr = lambda xs: (ctypes.c_char_p * len(xs))(*[x.encode() for x in xs])  # noqa: E731
    prog = ctypes.c_void_p()
    assert nv.nvrtcCreateProgram(ctypes.byref(prog), src.encode(), name.encode(), len(names), arr(bodies),
                                 arr(names)) == 0
    rc = nv.nvrtcCompileProgram(prog, len(options), arr(options))
    n = ctypes.c_size_t()
    nv.nvrtcGetProgramLogSize(prog, ctypes.byref(n))
    log = ctypes.create_string_buffer(n.value)
    nv.nvrtcGetProgramLog(prog, log)
    assert rc == 0, log.value.decode()
    nv.nvrtcGetCUBINSize(prog, ctypes.byref(n))
    out = ctypes.create_string_buffer(n.value)
    nv.nvrtcGetCUBIN(prog, out)
    nv.nvrtcDestroyProgram(ctypes.byref(prog))
    return out.raw, log.value.decode()


def _link(cubins, capfd):
    """nvJitLink's verbose report (on stderr) of linking `cubins` without LTO: {kernel: (registers, stack bytes)}."""
    nj = _cabi.nvjitlink()
    if nj is None:
        pytest.skip('nvJitLink (libnvJitLink.so.12) is not installed')
    opts = (ctypes.c_char_p * 2)(b'-arch=sm_90a', b'-verbose')
    h = ctypes.c_void_p()
    assert nj.__nvJitLinkCreate_12_0(ctypes.byref(h), 2, opts) == 0
    for i, c in enumerate(cubins):
        assert nj.__nvJitLinkAddData_12_0(h, 1, c, len(c), f'in{i}'.encode()) == 0  # NVJITLINK_INPUT_CUBIN
    rc = nj.__nvJitLinkComplete_12_0(h)
    n = ctypes.c_size_t()
    nj.__nvJitLinkGetErrorLogSize_12_0(h, ctypes.byref(n))
    err = ctypes.create_string_buffer(n.value + 1)
    nj.__nvJitLinkGetErrorLog_12_0(h, err)
    nj.__nvJitLinkDestroy_12_0(ctypes.byref(h))
    assert rc == 0, err.value.decode()
    return {m.group(1): (int(m.group(2)), int(m.group(3))) for m in re.finditer(
        r"Function properties for '(\w+)':\ninfo\s*: used (\d+) registers.*?, (\d+) stack", capfd.readouterr().err)}


LIBRARY = ['-arch=sm_90a', '-std=c++17', '-prec-div=true', '-prec-sqrt=true', '-ftz=false', '-default-device',
           '-rdc=true']


def linked_usage(src, capfd):
    helpers, _ = _cubin(_helpers_source(), LIBRARY + ['-fmad=true'], 'tsde_pw_helpers.cu')
    prog, _ = _cubin(src, LIBRARY + ['-fmad=false'])
    capfd.readouterr()
    return _link([prog, helpers], capfd)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('op', sorted(OPS))
def test_the_programs_link_with_the_helpers(op, dtype, capfd):
    _, (prog, _) = _milstein(op, 'g', dtype=dtype)
    usage = linked_usage(_cabi.pointwise_source(prog, dtype), capfd)
    assert set(usage) == {'tsde_pw_milstein_single', 'tsde_pw_milstein_multi'}
    # within the launch bounds the chunk length counts on: (256, 4) in float32, (256, 2) in float64
    assert all(regs <= (64 if dtype == torch.float32 else 128) for regs, _ in usage.values()), usage
    _, (prog, _) = _general(op, 'fggf', dtype=dtype)
    assert set(linked_usage(_cabi.general_pointwise_source(prog, dtype, general.D, 4), capfd)) == {
        'tsde_pw_general_sra1_single', 'tsde_pw_general_sra1_multi'}
