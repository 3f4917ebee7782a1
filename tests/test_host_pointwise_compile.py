"""The kernels the library compiles for Milstein programs (csrc/pointwise.cu, pw_milstein_source), on the CPU.

The library writes one CUDA translation unit per program structure and compiles it with NVRTC when the program is
first used.  Here the source comes from tsde_pointwise_source, which needs no device, and is compiled with NVRTC as the
library compiles it, from the device headers in csrc/: every Milstein tape the host tests accept (including the
comparison and selection ones) and a program at the TSDE_PW_MAX_INSTR / MAX_REGS / MAX_OPERANDS limits compile for
sm_90a in float32 and float64; cfg2's program compiles in float32 with no spill, no stack frame and at most 64
registers (4 resident CTAs of 256 threads); programs that differ only in operand values or addresses have one source,
which is the key of the library's kernel cache; and invalid programs are refused before any compilation."""
import ctypes
import os
import re

import pytest
import torch

from torchsde_b200 import _cabi
from . import test_host_pointwise as milstein
from . import test_host_pointwise_select as select

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'torchsde_b200', 'csrc')
# the headers as pw_device.cuh includes them, and the <stdint.h> NVRTC lacks
HEADERS = {'pw_device.cuh': os.path.join(CSRC, 'pw_device.cuh'), 'philox.cuh': os.path.join(CSRC, 'philox.cuh'),
           'rowdiv.cuh': os.path.join(CSRC, 'rowdiv.cuh'),
           '../../include/torchsde_b200.h': os.path.join(ROOT, 'include', 'torchsde_b200.h')}
STDINT = ('typedef signed char int8_t; typedef short int16_t; typedef int int32_t; typedef long long int64_t;\n'
          'typedef unsigned char uint8_t; typedef unsigned short uint16_t; typedef unsigned int uint32_t;\n'
          'typedef unsigned long long uint64_t; typedef unsigned long long uintptr_t;\n')
# the library's options (pw_nvrtc), and ptxas's report
OPTIONS = ['-arch=sm_90a', '-std=c++17', '-fmad=false', '-prec-div=true', '-prec-sqrt=true', '-ftz=false',
           '-default-device', '--ptxas-options=-v']


def _nvrtc():
    _cabi.lib()  # (preloads NVRTC from the nvidia-cuda-nvrtc package when it is installed)
    try:
        return ctypes.CDLL('libnvrtc.so.12')
    except OSError:
        pytest.skip('NVRTC (libnvrtc.so.12) is not installed')


def compile_source(src):
    """NVRTC's log of compiling `src` as the library does; fails the test on a compile error."""
    nv = _nvrtc()
    names = list(HEADERS) + ['stdint.h']
    bodies = [open(p).read() for p in HEADERS.values()] + [STDINT]
    prog = ctypes.c_void_p()
    arr = lambda xs: (ctypes.c_char_p * len(xs))(*[x.encode() for x in xs])  # noqa: E731
    assert nv.nvrtcCreateProgram(ctypes.byref(prog), src.encode(), b'tsde_pw_milstein.cu', len(names), arr(bodies),
                                 arr(names)) == 0
    rc = nv.nvrtcCompileProgram(prog, len(OPTIONS), arr(OPTIONS))
    n = ctypes.c_size_t()
    nv.nvrtcGetProgramLogSize(prog, ctypes.byref(n))
    log = ctypes.create_string_buffer(n.value)
    nv.nvrtcGetProgramLog(prog, log)
    nv.nvrtcGetCUBINSize(prog, ctypes.byref(n))
    nv.nvrtcDestroyProgram(ctypes.byref(prog))
    assert rc == 0 and n.value > 0, log.value.decode()
    return log.value.decode()


def usage(log):
    """{kernel: (registers, stack frame bytes, spill store bytes, spill load bytes)} from ptxas's report."""
    out = {}
    for m in re.finditer(r"Function properties for (\w+)\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log, re.S):
        out[m.group(1)] = (int(m.group(5)), int(m.group(2)), int(m.group(3)), int(m.group(4)))
    return out


def _tape(table, name, dtype):
    rec, res, _, _ = milstein._record(*table[name], dtype)
    assert res is not None, rec.reason
    return res[0]


def _limits():
    """A valid program at every limit: TSDE_PW_MAX_INSTR instructions, TSDE_PW_MAX_REGS registers and
    TSDE_PW_MAX_OPERANDS operands of every kind, with every opcode."""
    prog = _cabi.Pointwise()
    n, regs = _cabi.PW_MAX_INSTR, _cabi.PW_MAX_REGS
    prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands = n, n // 2, regs, _cabi.PW_MAX_OPERANDS
    kinds = [_cabi.PW_IMM, _cabi.PW_T0, _cabi.PW_SCALAR, _cabi.PW_CHANNEL, _cabi.PW_ROW]
    for k in range(_cabi.PW_MAX_OPERANDS):
        o = prog.operand[k]
        o.kind = kinds[k % len(kinds)]
        o.ptr = None if o.kind in (_cabi.PW_IMM, _cabi.PW_T0) else 0x10000 + 0x100 * k
        o.imm = 0.5 + k
    ops = list(range(6)) + list(range(8, 15))
    for i in range(n):
        ins = prog.instr[i]
        ins.dst = i % regs
        if i < regs:  # every register written first, from the operands and y
            ins.op, ins.a, ins.b = _cabi.PW_MUL, _cabi.PW_OPERAND0 + i % _cabi.PW_MAX_OPERANDS, _cabi.PW_SRC_Y
        else:
            ins.op = ops[i % len(ops)]
            ins.a = (i - 1) % regs
            ins.b = _cabi.PW_SRC_GO if i >= prog.n_fg and i % 3 == 0 else _cabi.PW_OPERAND0 + i % 24
    prog.f_src, prog.g_src, prog.gdg_src = 0, 1, (n - 1) % regs
    return prog


PROGRAMS = [('host', n) for n in sorted(milstein.ACCEPTED)] + [('select', n) for n in sorted(select.ACCEPTED)] + \
    [('limits', None)]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('table,name', PROGRAMS)
def test_every_accepted_milstein_program_compiles_for_sm_90a(table, name, dtype):
    prog = _limits() if table == 'limits' else _tape(milstein.ACCEPTED if table == 'host' else select.ACCEPTED, name,
                                                     dtype)
    src = _cabi.pointwise_source(prog, dtype)
    assert src is not None
    kernels = usage(compile_source(src))
    assert set(kernels) == {'tsde_pw_milstein_single', 'tsde_pw_milstein_multi'}


def test_cfg2_program_compiles_without_spills_at_four_ctas_per_sm():
    prog = _tape(milstein.ACCEPTED, 'gbm_ito', torch.float32)
    regs, stack, spill_st, spill_ld = usage(compile_source(_cabi.pointwise_source(prog, torch.float32)))[
        'tsde_pw_milstein_single']
    assert (stack, spill_st, spill_ld) == (0, 0, 0) and regs <= 64, (regs, stack, spill_st, spill_ld)


def test_operand_values_and_addresses_are_not_in_the_source():
    dtype = torch.float32
    a, b = _tape(milstein.ACCEPTED, 'ou', dtype), _tape(milstein.ACCEPTED, 'ou', dtype)
    for k in range(b.n_operands):
        o = b.operand[k]
        o.imm = o.imm * 3 + 1
        if o.ptr:
            o.ptr = o.ptr + 4096
    assert _cabi.pointwise_source(a, dtype) == _cabi.pointwise_source(b, dtype)
    assert _cabi.pointwise_source(a, torch.float64) != _cabi.pointwise_source(a, dtype)
    c = _tape(milstein.ACCEPTED, 'div', dtype)
    assert _cabi.pointwise_source(c, dtype) != _cabi.pointwise_source(a, dtype)


BROKEN = {
    'reserved opcode': lambda p: setattr(p.instr[0], 'op', 6),
    'register past n_regs': lambda p: setattr(p.instr[0], 'dst', p.n_regs),
    'unwritten register read': lambda p: setattr(p.instr[0], 'a', p.n_regs - 1),
    'go in the f / g part': lambda p: setattr(p.instr[0], 'a', _cabi.PW_SRC_GO),
    'operand past the table': lambda p: setattr(p.instr[0], 'a', _cabi.PW_OPERAND0 + p.n_operands),
    'too many instructions': lambda p: setattr(p, 'n_instr', _cabi.PW_MAX_INSTR + 1),
    'null device operand': lambda p: setattr(p.operand[0], 'ptr', None),
}


@pytest.mark.parametrize('name', sorted(BROKEN))
def test_invalid_programs_are_refused_before_any_compilation(name):
    prog = _tape(milstein.ACCEPTED, 'gbm_ito', torch.float32)
    BROKEN[name](prog)
    # (a valid program gets as far as loading its kernels, which needs a device; EINVAL is the validation's answer)
    assert _cabi.pointwise_source(prog, torch.float32) is None
    assert _cabi.compile_pointwise(prog, torch.float32) == _cabi.EINVAL
    assert _cabi.compile_pointwise(prog, torch.float64) == _cabi.EINVAL
