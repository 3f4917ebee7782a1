"""The element-wise tape of a Milstein step (torchsde_b200/_core/pointwise.py) on the CPU: which SDEs it accepts, and
that the program it compiles computes what the recorded ops computed.  The program is run here by a numpy restatement
of the kernel's interpreter (tsde_step_milstein_pointwise), one rounding per instruction in the state dtype; the GPU
suite compares the kernel itself with the unfused step (tests/test_gpu_pointwise.py)."""
import numpy as np
import pytest
import torch

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise

ROWS, D = 5, 8


def _params(dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {k: (torch.rand(D, generator=g, dtype=dtype) + 0.5) for k in ('a', 'b')} | \
        {'r': torch.rand(ROWS, D, generator=g, dtype=dtype) + 0.5, 's': torch.rand(1, generator=g, dtype=dtype) + 0.5}


# (f, g) as functions of (t, y, params); every pair the tape accepts
ACCEPTED = {
    'gbm_ito': (lambda t, y, p: p['a'] * y, lambda t, y, p: p['b'] * y),
    'gbm_strat': (lambda t, y, p: p['a'] * y - .5 * (p['b'] ** 2) * y, lambda t, y, p: p['b'] * y),
    'per_row': (lambda t, y, p: p['r'] * y, lambda t, y, p: p['r'] * y + p['s']),
    'ou': (lambda t, y, p: p['a'] * (p['b'] - y), lambda t, y, p: p['s'] * y),
    'time': (lambda t, y, p: t * y, lambda t, y, p: (t + 1) * y),
    'div': (lambda t, y, p: y / p['a'], lambda t, y, p: y / 3),
    'square': (lambda t, y, p: -y, lambda t, y, p: y * y),
    'sqrt_rsub': (lambda t, y, p: 2 - y, lambda t, y, p: torch.sqrt(y) + y.sub(p['a'], alpha=-1)),
    'views': (lambda t, y, p: p['a'].unsqueeze(0).expand(ROWS, D) * y.view(ROWS, D),
              lambda t, y, p: y.view(1, ROWS, D).view(ROWS, D) * p['b'].view(1, D)),
}


def _written_in_place(t, y, p):
    a = p['a'] * y
    a.add_(1)
    return a


def _written_through_detach_and_returned(t, y, p):
    b = (p['a'] * y).detach()
    b.mul_(2)
    return b


def _f_cached(t, y, p):
    p['cache'] = p['a'] * y
    return p['cache']


def _written_through(how):
    """f = a = mu*y, then a is written in place through an alias of its storage, and `a` itself is returned."""
    def f(t, y, p):
        a = p['a'] * y
        {'detach': lambda: a.detach().add_(1), 'data': lambda: a.data.mul_(2),
         'view': lambda: a.view(ROWS, D).sub_(p['b'])}[how]()
        return a
    return f


ACCEPTED.update({
    'in_place': (_written_in_place, lambda t, y, p: p['b'] * y),
    'in_place_returned_alias': (_written_through_detach_and_returned, lambda t, y, p: p['b'] * y),
    # f's value is read by g and again by three vjp instructions, long after the f / g boundary
    'f_value_in_vjp': (_f_cached, lambda t, y, p: p['cache'] * y * y),
})
REJECTED = {
    'written_through_detach': (_written_through('detach'), lambda t, y, p: p['b'] * y),
    'written_through_data': (_written_through('data'), lambda t, y, p: p['b'] * y),
    'written_through_view': (_written_through('view'), lambda t, y, p: p['b'] * y),
    'exp': (lambda t, y, p: torch.exp(y), lambda t, y, p: p['b'] * y),
    'sigmoid_g': (lambda t, y, p: y, lambda t, y, p: torch.sigmoid(y)),
    'matmul': (lambda t, y, p: y @ torch.eye(D, dtype=y.dtype), lambda t, y, p: p['b'] * y),
    'item': (lambda t, y, p: y * p['s'].item(), lambda t, y, p: p['b'] * y),
    'alpha': (lambda t, y, p: torch.add(y, p['a'], alpha=2), lambda t, y, p: p['b'] * y),
    'pow3': (lambda t, y, p: y ** 3, lambda t, y, p: p['b'] * y),
    'reduction': (lambda t, y, p: y - y.mean(dim=1, keepdim=True), lambda t, y, p: p['b'] * y),
    'in_place_param': (lambda t, y, p: p['a'].mul_(1) * y, lambda t, y, p: p['b'] * y),
    'transpose': (lambda t, y, p: p['a'].unsqueeze(1).expand(D, ROWS).t() * y, lambda t, y, p: p['b'] * y),
    'half': (lambda t, y, p: (p['a'] * y).to(torch.bfloat16).to(y.dtype), lambda t, y, p: p['b'] * y),
    'constant_g': (lambda t, y, p: y, lambda t, y, p: p['b'].expand(ROWS, D)),
    'column_operand': (lambda t, y, p: p['r'][:, :1] * y, lambda t, y, p: p['b'] * y),
    'factory': (lambda t, y, p: torch.ones_like(y) * y, lambda t, y, p: p['b'] * y),
}


def _record(f, g, dtype, rec_cls=pointwise.Recorder):
    """One step's f, g and vjp under the recorder, as BaseMilstein._step runs them."""
    p = _params(dtype)
    y0 = torch.rand(ROWS, D, generator=torch.Generator().manual_seed(1), dtype=dtype) + 0.25
    t0 = torch.tensor(0.375, dtype=dtype)
    rec = rec_cls(y0, t0)
    fv = rec.segment(lambda: f(t0, y0, p))
    with torch.enable_grad():
        y = y0.detach().requires_grad_(True)
        gv = rec.segment(lambda: g(t0, y, p), y=y)
        go = torch.rand(ROWS, D, generator=torch.Generator().manual_seed(2), dtype=dtype) - 0.5
        gdg = None
        if gv.requires_grad:
            gdg, = rec.segment(lambda: torch.autograd.grad(gv, y, grad_outputs=go.view_as(gv), allow_unused=True),
                               go=go)
    return rec, rec.finish(fv, gv, gdg), (y0, t0, go), (fv, gv, gdg)


def _interpret(prog, y0, t0, go, dtype):
    """numpy restatement of the kernel's interpreter: every register and operand as a (rows, d) array."""
    npt = np.float32 if dtype == torch.float32 else np.float64
    y0, t0, go = y0.numpy(), t0.numpy(), go.numpy()
    regs = [None] * prog.n_regs

    def fetch(s, vjp):
        if s == _cabi.PW_SRC_Y:
            return y0
        if s == _cabi.PW_SRC_GO:
            assert vjp
            return go
        if s < _cabi.PW_OPERAND0:
            assert regs[s] is not None
            return regs[s]
        o = prog.operand[s - _cabi.PW_OPERAND0]
        if o.kind == _cabi.PW_IMM:
            return np.full((ROWS, D), npt(o.imm))
        if o.kind == _cabi.PW_T0:
            return np.full((ROWS, D), t0)
        n = {_cabi.PW_SCALAR: 1, _cabi.PW_CHANNEL: D, _cabi.PW_ROW: ROWS * D}[o.kind]
        flat = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_byte * (n * np.dtype(npt).itemsize)).from_address(o.ptr))
        return np.broadcast_to(flat.view(npt).reshape(-1 if n == ROWS * D else 1, n if n != ROWS * D else D)
                               if o.kind != _cabi.PW_SCALAR else flat.view(npt)[0], (ROWS, D))

    out = {}
    with np.errstate(all='ignore'):
        for i in range(prog.n_instr + 1):
            if i == prog.n_fg:
                out['f'], out['g'] = fetch(prog.f_src, False).copy(), fetch(prog.g_src, False).copy()
            if i == prog.n_instr:
                break
            ins = prog.instr[i]
            a = fetch(ins.a, i >= prog.n_fg)
            b = fetch(ins.b, i >= prog.n_fg) if ins.op not in (_cabi.PW_NEG, _cabi.PW_SQRT) else None
            r = {_cabi.PW_MUL: lambda: a * b, _cabi.PW_ADD: lambda: a + b, _cabi.PW_SUB: lambda: a - b,
                 _cabi.PW_DIV: lambda: a / b, _cabi.PW_NEG: lambda: -a, _cabi.PW_SQRT: lambda: np.sqrt(a)}[ins.op]()
            regs[ins.dst] = np.asarray(r, dtype=npt)
        out['gdg'] = fetch(prog.gdg_src, True).copy()
    return out


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('name', sorted(ACCEPTED))
def test_accepted_tapes_restate_the_recorded_ops(name, dtype):
    rec, res, (y0, t0, go), (f, g, gdg) = _record(*ACCEPTED[name], dtype)
    assert res is not None, rec.reason
    prog, keep = res
    assert 0 < prog.n_instr <= _cabi.PW_MAX_INSTR and prog.n_regs <= _cabi.PW_MAX_REGS
    got = _interpret(prog, y0, t0, go, dtype)
    for k, want in (('f', f), ('g', g), ('gdg', gdg)):
        w = np.ascontiguousarray(want.detach().numpy())
        assert got[k].dtype == w.dtype, k
        if name == 'div' and k != 'f':
            # a Python-number divisor: ATen's CUDA kernel (restated by the tape) multiplies by the reciprocal, its CPU
            # kernel divides; the GPU suite checks the bits
            np.testing.assert_allclose(got[k], w, rtol=4 * np.finfo(w.dtype).eps)
        else:
            assert np.array_equal(got[k].view(np.uint8), w.view(np.uint8)), k


@pytest.mark.parametrize('name', sorted(REJECTED))
def test_rejected_tapes(name):
    rec, res, _, _ = _record(*REJECTED[name], torch.float32)
    assert res is None and rec.reason


def test_cfg2_tape_is_three_multiplications_in_two_registers():
    """The headline SDE (f = mu*y, g = sigma*y): f and g, then autograd's `grad * sigma`."""
    rec, (prog, _), _, _ = _record(*ACCEPTED['gbm_ito'], torch.float32)
    assert (prog.n_instr, prog.n_fg, prog.n_regs, prog.n_operands) == (3, 2, 2, 2)
    assert [prog.instr[i].op for i in range(3)] == [_cabi.PW_MUL] * 3
    assert prog.instr[2].a == _cabi.PW_SRC_GO


def test_scalar_divisor_is_a_reciprocal_rounded_in_the_state_dtype():
    rec, (prog, _), _, _ = _record(lambda t, y, p: y / 3, ACCEPTED['gbm_ito'][1], torch.float32)
    ins = prog.instr[0]
    assert ins.op == _cabi.PW_MUL and ins.b >= _cabi.PW_OPERAND0
    assert prog.operand[ins.b - _cabi.PW_OPERAND0].imm == float(np.float32(1) / np.float32(3))


def test_time_of_another_dtype_rejects():
    """The kernel reads t0 in the state dtype: a time tensor of another dtype is no operand."""
    y0 = torch.rand(ROWS, D)
    t0 = torch.tensor(0.5, dtype=torch.float64)
    rec = pointwise.Recorder(y0, t0)
    rec.segment(lambda: t0 * y0)
    assert not rec.ok
