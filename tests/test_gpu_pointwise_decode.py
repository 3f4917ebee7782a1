"""The decoded element-wise program (torchsde_b200/csrc/pointwise.cu, PwProg): every source kind reaches the kernels
through its slot of the shared-memory register file, in every fused kernel.

Each fused solve must give the bits of the same solve with the tape rejected, as in the other pointwise tests.  The
SDEs here read every source kind (IMM, T0, SCALAR, CHANNEL, ROW, the state y and, in Milstein's vjp, go) both as the
first and as the second operand of an instruction, and use every op (mul, add, sub, div, neg, sqrt).  `Many` reads
more CHANNEL / ROW operands than fit the hoisted slots, so that the ones past them are read from global memory.
Covered in float32 and float64: the Milstein step and Milstein chunks, Euler and reversible-Heun chunks, SRK and the
midpoint step."""
import contextlib

import pytest
import torch
from torch import nn

from torchsde_b200 import _cabi
from torchsde_b200._core import pointwise
from . import test_gpu_pointwise as milstein
from . import test_gpu_pointwise_euler_rh as euler_rh
from . import test_gpu_pointwise_pc as pc
from . import test_gpu_pointwise_srk as srk

pytestmark = pytest.mark.gpu
DEV = 'cuda'
B, D = 96, 16
DTYPES = [torch.float32, torch.float64]
K = _cabi.PW_MAX_STEPS


class AllSources(nn.Module):
    """f and g read every source kind as a and as b, with every op; the vjp of g reads go."""
    noise_type = 'diagonal'

    def __init__(self, sde_type, dtype):
        super().__init__()
        self.sde_type = sde_type
        gen = torch.Generator().manual_seed(3)
        rand = lambda *shape: torch.rand(shape, generator=gen, dtype=torch.float64).to(dtype)  # noqa: E731
        self.c = nn.Parameter(rand(D) + 0.5)     # CHANNEL
        self.r = nn.Parameter(rand(B, D) + 0.5)  # ROW
        self.s = nn.Parameter(rand(1) + 0.5)     # SCALAR

    def f(self, t, y):
        # T0 as a / y as b; y as a / SCALAR as b; CHANNEL as a; ROW as a / IMM as b; IMM as a (rsub); T0 as b
        return ((t * y - y * self.s) + (self.c * y) / (self.r + 2.0)) - (1.0 - y) * t

    def g(self, t, y):
        # SCALAR as a; ROW as b; CHANNEL as b (div); neg; sqrt of a ROW operand
        return ((self.s * y) * 0.1 + (y * self.r) * 0.2) - (-(y / self.c)) * 0.05 + torch.sqrt(self.r) * 0.01


class Many(nn.Module):
    """f and g read N_OPERANDS distinct CHANNEL and ROW operands: more than the hoisted slots hold."""
    noise_type = 'diagonal'
    N_OPERANDS = 22

    def __init__(self, sde_type, dtype):
        super().__init__()
        self.sde_type = sde_type
        gen = torch.Generator().manual_seed(4)
        shapes = [(D,) if k % 2 else (B, D) for k in range(self.N_OPERANDS)]
        self.p = nn.ParameterList(
            nn.Parameter((torch.rand(s, generator=gen, dtype=torch.float64) * 0.2 + 0.05).to(dtype)) for s in shapes)

    def f(self, t, y):
        acc = self.p[0] * y
        for p in self.p[1:self.N_OPERANDS // 2]:
            acc = acc + p * y
        return acc

    def g(self, t, y):
        acc = y * self.p[self.N_OPERANDS // 2]
        for p in self.p[self.N_OPERANDS // 2 + 1:]:
            acc = acc - y * p
        return acc


SDES = {'all_sources': AllSources, 'many_operands': Many}


def y0_of(dtype):
    gen = torch.Generator().manual_seed(5)
    return (torch.rand(B, D, generator=gen, dtype=torch.float64) * 0.5 + 0.25).to(dtype).to(DEV)


@contextlib.contextmanager
def chunks_of(n):
    """Steps per launch of the chunked kernels: these batches are below one wave, which runs one step per launch."""
    length = pointwise.chunk_length
    pointwise.chunk_length = lambda solver: n
    try:
        yield
    finally:
        pointwise.chunk_length = length


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('sde', sorted(SDES))
@pytest.mark.parametrize('chunk', [1, K])
def test_milstein(sde, dtype, chunk):
    with chunks_of(chunk):
        milstein.check_fused(SDES[sde]('ito', dtype).to(DEV), y0_of(dtype), 2 * K + 5, 2.0 ** -7,
                             {'cuda_graph': True})


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('sde', sorted(SDES))
@pytest.mark.parametrize('method', euler_rh.METHODS)
def test_euler_and_reversible_heun_chunks(method, sde, dtype):
    ts = (torch.arange(2 * K + 5) * 2.0 ** -7).to(dtype)  # a time in the state dtype: T0 is an operand
    with chunks_of(K):
        euler_rh.check(SDES[sde](euler_rh.SDE_TYPE[method], dtype).to(DEV), y0_of(dtype), ts, 2.0 ** -7, method,
                       {'cuda_graph': True})


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('sde', sorted(SDES))
def test_srk(sde, dtype):
    srk.check_fused(SDES[sde]('ito', dtype).to(DEV), y0_of(dtype), 12, 2.0 ** -7, {'cuda_graph': True})


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('sde', sorted(SDES))
def test_midpoint(sde, dtype):
    pc.check_fused(SDES[sde]('stratonovich', dtype).to(DEV), y0_of(dtype), 12, 2.0 ** -7, 'midpoint',
                   {'cuda_graph': True})
