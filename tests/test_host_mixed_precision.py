"""16-bit SDE outputs on the host side (no GPU): the format bits every launch carries, the host-side widening of the
fallback paths, and the library's validation of the format bits (tsde_launch.dtype)."""
import contextlib
import ctypes
import warnings

import pytest
import torch
from torch import nn

import torchsde_b200 as tsde
from torchsde_b200 import _cabi
from torchsde_b200._brownian import interval as interval_mod
from . import problems


class _RecordingLib:
    """Stand-in for the C library (as in test_host_dry_run.py) that also records every launch's dtype word."""

    def __init__(self):
        self.calls = {}
        self.words = []

    def __getattr__(self, name):
        if name not in _cabi.SIGNATURES:
            raise AttributeError(name)
        arity = len(_cabi.SIGNATURES[name])

        def entry(*args):
            assert len(args) == arity, f"{name}: {len(args)} arguments, the C ABI declares {arity}"
            self.calls[name] = self.calls.get(name, 0) + 1
            self.words.append((name, args[0]._obj.dtype))
            return 0
        return entry

    def tsde_abi_version(self):
        return 1

    def tsde_kernel_launches(self, family):
        return 0


@pytest.fixture
def dry(monkeypatch):
    lib = _RecordingLib()
    monkeypatch.setattr(_cabi, '_lib', lib)
    monkeypatch.setattr(_cabi, 'lib', lambda: lib)
    monkeypatch.setattr(_cabi, 'require_cuda', lambda *a, **k: None)
    monkeypatch.setattr(interval_mod.BrownianInterval, '_require_cuda', lambda self: None)
    real_bind = interval_mod.BrownianInterval.bind_grid

    def bind_grid(self, bounds):
        device, self._device = self._device, torch.device('cuda')
        try:
            return real_bind(self, bounds)
        finally:
            self._device = device

    monkeypatch.setattr(interval_mod.BrownianInterval, 'bind_grid', bind_grid)
    monkeypatch.setattr(torch.cuda, 'synchronize', lambda *a, **k: None)

    class _Stream:
        cuda_stream = 0

        def __init__(self, *a, **k):
            pass

        def wait_stream(self, other):
            pass

        def record_event(self):
            return object()

        def wait_event(self, event):
            pass

    class _Graph:
        def replay(self):
            pass

    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a, **k: _Stream())
    monkeypatch.setattr(torch.cuda, 'Stream', _Stream)
    monkeypatch.setattr(torch.cuda, 'stream', lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, 'CUDAGraph', _Graph)
    monkeypatch.setattr(torch.cuda, 'graph', lambda g, **k: contextlib.nullcontext())
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        yield lib


class Cast(nn.Module):
    def __init__(self, base, dtype):
        super().__init__()
        self.base, self.dt16 = base, dtype
        self.noise_type, self.sde_type = base.noise_type, base.sde_type

    def f(self, t, y):
        return self.base.f(t, y).to(self.dt16)

    def g(self, t, y):
        return self.base.g(t, y).to(self.dt16)

    def h(self, t, y):
        return -self.base.f(t, y).to(self.dt16)


CASES = [('gbm', 'ito', 'euler', 'none'), ('gbm', 'ito', 'milstein', 'none'), ('gbm', 'ito', 'srk', 'space-time'),
         ('gbm', 'stratonovich', 'milstein', 'none'), ('scalar', 'stratonovich', 'midpoint', 'none'),
         ('additive', 'ito', 'srk', 'space-time'), ('additive', 'ito', 'milstein', 'none'),
         ('general', 'ito', 'euler', 'none'), ('general', 'stratonovich', 'heun', 'none'),
         ('general', 'stratonovich', 'reversible_heun', 'none'), ('gbm', 'stratonovich', 'euler_heun', 'none'),
         ('gbm', 'stratonovich', 'reversible_heun', 'none'), ('scalar', 'ito', 'srk', 'davie')]
TS = [0.0, 0.09375, 0.25]
DT = 0.0625


def _setup(kind, sde_type, levy, dtype, half):
    d, m = 3, {'gbm': 3, 'scalar': 1}.get(kind, 2)
    sde = Cast(problems.make(kind, d, m, sde_type, dtype=dtype), half)
    bm = tsde.BrownianInterval(0.0, TS[-1], size=(4, m), dtype=dtype, device='cpu', levy_area_approximation=levy)
    return sde, torch.ones(4, d, dtype=dtype), bm


def _expected(name, state, fmt):
    word = _cabi.dtype_code(state)
    for i, arg in enumerate(_cabi.INPUTS[name]):
        if arg in _cabi.SDE_OUTPUT_NAMES and arg != 'gdg':
            word |= fmt << (8 + 2 * i)
    return word


@pytest.mark.parametrize('half,fmt', [(torch.bfloat16, _cabi.FMT_BF16), (torch.float16, _cabi.FMT_F16)])
@pytest.mark.parametrize('kind,sde_type,method,levy', CASES)
def test_every_launch_declares_its_16bit_operands(dry, kind, sde_type, method, levy, half, fmt):
    sde, y0, bm = _setup(kind, sde_type, levy, torch.float32, half)
    with torch.no_grad():
        tsde.sdeint(sde, y0, TS, bm=bm, method=method, dt=DT)
    tableau = [(n, w) for n, w in dry.words if n in _cabi.INPUTS and n != 'tsde_linear_interp']
    assert tableau
    for name, word in tableau:  # every SDE-output slot holds what f / g returned
        assert word == _expected(name, torch.float32, fmt), (name, hex(word))
    assert all(w == _cabi.F32 for n, w in dry.words if n not in _cabi.INPUTS or n == 'tsde_linear_interp')


@pytest.mark.parametrize('kind,sde_type,method,levy', CASES)
def test_float64_state_widens(dry, kind, sde_type, method, levy):
    sde, y0, bm = _setup(kind, sde_type, levy, torch.float64, torch.bfloat16)
    with torch.no_grad():
        tsde.sdeint(sde, y0, TS, bm=bm, method=method, dt=DT)
    assert dry.words and all(w == _cabi.F64 for _, w in dry.words)


@pytest.mark.parametrize('kind,sde_type,method,levy', [c for c in CASES if c[2] != 'srk'][:6])
def test_gradients_through_sdeint_widen(dry, kind, sde_type, method, levy):
    """Backprop through the solver widens each 16-bit output once (so autograd accumulates its gradient in float32)."""
    sde, y0, bm = _setup(kind, sde_type, levy, torch.float32, torch.bfloat16)
    ys = tsde.sdeint(sde, y0.requires_grad_(), TS, bm=bm, method=method, dt=DT)
    ys.sum().backward()
    assert dry.words and all(w == _cabi.F32 for _, w in dry.words)


def test_logqp_and_log_ode_widen(dry):
    sde, y0, bm = _setup('gbm', 'ito', 'none', torch.float32, torch.bfloat16)
    with torch.no_grad():
        tsde.sdeint(sde, y0, TS, method='euler', dt=DT, logqp=True)  # (the augmented state needs its own bm)
    assert dry.calls.get('tsde_logqp_augment') and all(w == _cabi.F32 for _, w in dry.words)
    dry.words.clear()
    sde, y0, bm = _setup('general', 'stratonovich', 'foster', torch.float32, torch.bfloat16)
    with torch.no_grad():
        tsde.sdeint(sde, y0, TS, bm=bm, method='log_ode', dt=DT)
    assert dry.calls.get('tsde_bmm_ga') and all(w == _cabi.F32 for n, w in dry.words if n == 'tsde_bmm_ga')


def test_operands_rule():
    f32, bf = torch.zeros(2, 3), torch.zeros(2, 3, dtype=torch.bfloat16)
    word, ins = _cabi.operands('tsde_step_euler', torch.float32, [f32, bf, bf.half()])
    assert word == _cabi.F32 | (_cabi.FMT_BF16 << 10) | (_cabi.FMT_F16 << 12) and ins[1] is bf
    word, ins = _cabi.operands('tsde_step_euler', torch.float64, [f32.double(), bf, bf])
    assert word == _cabi.F64 and all(t.dtype == torch.float64 for t in ins)
    with pytest.raises(ValueError, match='`f`'):
        _cabi.operands('tsde_step_euler', torch.float32, [f32, f32.double(), f32])
    with pytest.raises(ValueError, match='`y0`'):
        _cabi.operands('tsde_step_euler', torch.float32, [bf, f32, f32])
    with pytest.raises(ValueError, match='`gdg`'):
        _cabi.operands('tsde_step_milstein', torch.float32, [f32, f32, f32, bf])


# ---- the library's own validation (ctypes, no device: every case returns before any CUDA call) --------------------
def _lib_or_skip():
    try:
        return _cabi.lib()
    except _cabi.LibraryNotBuilt:
        pytest.skip('CUDA library not built')


def _euler(lib, dtype_word, rows):
    L = _cabi.Launch(dtype_word, _cabi.NOISE_DIAGONAL, rows, 4, 4, None)
    nz = _cabi.Noise()
    nz.source = _cabi.SRC_UNIT
    return lib.tsde_step_euler(ctypes.byref(L), ctypes.byref(nz), None, None, None, 0.1, None)


FMT = lambda i, f: f << (8 + 2 * i)  # noqa: E731  (TSDE_OPERAND_FMT)


@pytest.mark.parametrize('rows', [0, 4])
@pytest.mark.parametrize('word', [
    _cabi.F32 | FMT(0, _cabi.FMT_BF16),                        # y0 is not an SDE output
    _cabi.F64 | FMT(1, _cabi.FMT_BF16),                        # 16-bit operands need a float32 state
    _cabi.F32 | FMT(1, 3),                                     # no format 3
    _cabi.F32 | FMT(3, _cabi.FMT_F16),                         # past the entry point's inputs
    7,                                                         # unknown state dtype
])
def test_invalid_format_bits_rejected(word, rows):
    assert _euler(_lib_or_skip(), word, rows) == _cabi.EINVAL


def test_empty_launch_with_format_bits_is_a_no_op():
    lib = _lib_or_skip()
    assert _euler(lib, _cabi.F32 | FMT(1, _cabi.FMT_BF16) | FMT(2, _cabi.FMT_F16), 0) == 0
    L = _cabi.Launch(_cabi.F32 | FMT(0, _cabi.FMT_BF16), _cabi.NOISE_DIAGONAL, 0, 4, 4, None)
    assert lib.tsde_milstein_vjp_seed(ctypes.byref(L), None, None, 0.1, 1, None) == 0


def test_out_of_scope_entry_points_reject_format_bits():
    lib = _lib_or_skip()
    L = _cabi.Launch(_cabi.F32 | FMT(0, _cabi.FMT_BF16), _cabi.NOISE_DIAGONAL, 0, 4, 4, None)
    assert lib.tsde_linear_interp(ctypes.byref(L), None, None, 0.5, 0.5, None) == _cabi.EINVAL
    assert lib.tsde_logqp_augment(ctypes.byref(L), None, None, None, 1e-7, None, None) == _cabi.EINVAL
    L.noise_type = _cabi.NOISE_GENERAL
    assert lib.tsde_bmm_ga(ctypes.byref(L), None, None, None) == _cabi.EINVAL
