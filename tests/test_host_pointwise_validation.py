"""What tsde_step_milstein_pointwise and tsde_step_srk_diag_pointwise refuse: a program that would index the kernel's
shared-memory register file or the operand table out of range, read a register before it is written, or name a source
its layout does not have is TSDE_EINVAL before anything is launched (include/torchsde_b200.h describes the two
layouts).  Every malformed program is a well-formed one with one thing changed.  The library checks the program before
its first CUDA call, so the table runs against the real library without a device; that the well-formed programs
launch needs one."""
import ctypes

import pytest
import torch

from torchsde_b200 import _cabi

ROWS, D = 4, 8
Y, GO, K0 = _cabi.PW_SRC_Y, _cabi.PW_SRC_GO, _cabi.PW_OPERAND0
MUL, ADD = _cabi.PW_MUL, _cabi.PW_ADD


def _lib_or_skip():
    try:
        return _cabi.lib()
    except _cabi.LibraryNotBuilt:
        pytest.skip('CUDA library not built')


def _program(instrs, n_fg, n_regs, results, mem):
    """A tsde_pointwise with a (d,) operand and a one-element operand, both in `mem`."""
    prog = _cabi.Pointwise()
    prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands = len(instrs), n_fg, n_regs, 2
    prog.f_src, prog.g_src, prog.gdg_src = results
    for j, (op, dst, a, b) in enumerate(instrs):
        prog.instr[j].op, prog.instr[j].dst, prog.instr[j].a, prog.instr[j].b = op, dst, a, b
    prog.operand[0].kind, prog.operand[0].ptr = _cabi.PW_CHANNEL, mem.data_ptr()
    prog.operand[1].kind, prog.operand[1].ptr = _cabi.PW_SCALAR, mem.data_ptr()
    return prog


def _milstein(mem):  # f = k0 * y, g = k1 * y | vjp = go * k1
    return _program([(MUL, 0, K0, Y), (MUL, 1, K0 + 1, Y), (MUL, 2, GO, K0 + 1)], 2, 3, (0, 1, 2), mem)


def _srk(mem):  # f = k0 * y | g = k1 * y + y
    return _program([(MUL, 0, K0, Y), (MUL, 0, K0 + 1, Y), (ADD, 1, 0, Y)], 1, 2, (0, 1, 0), mem)


def _set(path, value):
    """A change of one field: 'n_regs', 'f_src', 'instr.2.a', 'operand.1.ptr'."""
    def change(prog):
        obj, names = prog, path.split('.')
        for name in names[:-1]:
            obj = obj[int(name)] if name.isdigit() else getattr(obj, name)
        setattr(obj, names[-1], value)
    return change


def _all(*changes):
    def change(prog):
        for c in changes:
            c(prog)
    return change


BOTH = {
    'register read before it is written': _set('instr.0.a', 1),
    'destination past n_regs': _all(_set('instr.0.dst', 3), _set('n_regs', 3)),
    'operand index past n_operands': _set('instr.0.a', K0 + 2),
    'n_fg past n_instr': _set('n_fg', 4),
    'negative n_instr': _set('n_instr', -1),
    'n_instr past the limit': _set('n_instr', _cabi.PW_MAX_INSTR + 1),
    'n_operands past the limit': _set('n_operands', _cabi.PW_MAX_OPERANDS + 1),
    'null pointer in a one-element operand': _set('operand.1.ptr', None),
    'unknown operand kind': _set('operand.0.kind', _cabi.PW_ROW + 1),
    'opcode 6': _set('instr.0.op', 6),
    'f result in a register never written': _set('f_src', 2),
    'register source past the register file': _set('instr.0.a', _cabi.PW_MAX_REGS),
}
MILSTEIN = dict(BOTH, **{
    'n_regs 25': _set('n_regs', _cabi.PW_MAX_REGS + 1),
    'go in the f / g part': _set('instr.1.b', GO),
    'go as the f result': _set('f_src', GO),
    'go as the g result': _set('g_src', GO),
    'g result written only by the vjp part': _set('g_src', 2),
    'vjp result in a register never written': _all(_set('n_regs', 4), _set('gdg_src', 3)),
})
SRK = dict(BOTH, **{
    'n_regs 19': _set('n_regs', _cabi.PW_SRK_MAX_REGS + 1),
    'g reads a register only f wrote': _set('instr.1.dst', 1),
    'g result in a register only f wrote': _all(_set('instr.1.dst', 1), _set('instr.2.a', 1), _set('g_src', 0)),
    'go in the f program': _set('instr.0.b', GO),
    'go in the g program': _set('instr.2.b', GO),
    'go as the f result': _set('f_src', GO),
    'go as the g result': _set('g_src', GO),
})


class _Step:
    """One call of either entry point on (ROWS, D) with counter noise."""

    def __init__(self, dtype, device):
        self.lib = _lib_or_skip()
        self.mem = torch.full((D,), 0.5, dtype=dtype, device=device)
        self.y0 = torch.full((ROWS, D), 0.25, dtype=dtype, device=device)
        self.y1 = torch.zeros_like(self.y0)
        self.t = torch.zeros(4, dtype=dtype, device=device)
        self.key = torch.zeros(2, dtype=torch.int32, device=device)
        self.L = _cabi.Launch(_cabi.dtype_code(dtype), _cabi.NOISE_DIAGONAL, ROWS, D, D, None)
        self.nz = _cabi.Noise(source=_cabi.SRC_COUNTER, key=self.key.data_ptr(), n_cells=1, h=0.125, h_total=0.125)

    def launches(self):
        return [self.lib.tsde_kernel_launches(k) for k in (_cabi.KERNEL_PW_MILSTEIN, _cabi.KERNEL_PW_SRK)]

    def milstein(self, prog):
        return self.lib.tsde_step_milstein_pointwise(ctypes.byref(self.L), ctypes.byref(self.nz), ctypes.byref(prog),
                                                     self.y0.data_ptr(), self.t.data_ptr(), 0.125, 1,
                                                     self.y1.data_ptr())

    def srk(self, prog):
        t = [self.t[i:].data_ptr() for i in range(4)]
        return self.lib.tsde_step_srk_diag_pointwise(ctypes.byref(self.L), ctypes.byref(self.nz), ctypes.byref(prog),
                                                     self.y0.data_ptr(), *t, 0.125, 8.0, 0.125 ** 0.5, 0.375,
                                                     self.y1.data_ptr())


DEVICE = 'cuda' if torch.cuda.is_available() else 'cpu'  # (a refused call never reads through a pointer)
CASES = [('milstein', name) for name in MILSTEIN] + [('srk', name) for name in SRK]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('method,name', CASES)
def test_malformed_programs_are_refused_without_a_launch(method, name, dtype):
    step = _Step(dtype, DEVICE)
    prog = (_milstein if method == 'milstein' else _srk)(step.mem)
    (MILSTEIN if method == 'milstein' else SRK)[name](prog)
    before = step.launches()
    assert getattr(step, method)(prog) == _cabi.EINVAL
    assert step.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_the_programs_the_table_starts_from_launch(dtype):
    step = _Step(dtype, 'cuda')
    before = step.launches()
    assert step.milstein(_milstein(step.mem)) == 0
    assert step.srk(_srk(step.mem)) == 0
    torch.cuda.synchronize()
    assert step.launches() == [n + 1 for n in before]
    assert torch.isfinite(step.y1).all()
