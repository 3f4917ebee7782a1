"""The fast row-wise kernel (csrc/ew.cuh ew_fast_kernel) gives each CTA one chunk of 256 quads (one per thread) or
512 quads (two per thread, the light fp32 ops).  At batch sizes on and around those chunk edges, and one row past a
full wave of resident CTAs, every diagonal entry point must give the generic kernel's bits (ew_kernel, taken by
operands one element off 16-byte alignment), with counter and with memory noise."""
import pytest
import torch

from .test_gpu_index_paths import DEV, KEY, NOISE_OPS, PLAIN_OPS, SQ, _ins, _launch, _noise, _op_id

pytestmark = pytest.mark.gpu


def _chunk_edge_rows(d):
    qpr = d // 4  # quads per row
    return (1,                                   # one row
            (256 - 1) // qpr, 256 // qpr + 1,    # one quad short of / past a 256-quad chunk
            (512 - 1) // qpr, 512 // qpr + 1,    # the same for a 512-quad chunk
            132 * 8 * 512 // qpr + 1)            # one row past a wave of 132 SMs x 8 CTAs of 512 quads


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('d', [4, 12, 64])
def test_fast_kernel_chunk_edges_equal_generic_kernel(d, dtype):
    es = torch.finfo(dtype).bits // 8
    key = torch.tensor([KEY], dtype=torch.int64, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(d)
    bad = []
    for B in _chunk_edge_rows(d):
        n = B * d
        pool_u = [torch.rand(n + 1, generator=gen, device=DEV, dtype=dtype) + 0.5 for _ in range(5)]
        pool = [x[1:].clone() for x in pool_u]  # the same values, aligned
        mem_u = [torch.randn(n + 1, generator=gen, device=DEV, dtype=dtype) * SQ for _ in range(2)]  # W, U
        mem = [x[1:].clone() for x in mem_u]
        out_a = [torch.empty(n, device=DEV, dtype=dtype) for _ in range(5)]
        out_b = [torch.empty(n + 1, device=DEV, dtype=dtype) for _ in range(5)]
        for op in NOISE_OPS + PLAIN_OPS:
            sources = ('counter', 'memory') if op in NOISE_OPS and op[0] != 'tsde_brownian_cells' else ('counter',)
            for src in sources:
                nz_a = _noise(key, op[3], mem=(mem[0].data_ptr(), mem[1].data_ptr()) if src == 'memory' else None)
                nz_b = _noise(key, op[3], mem=(mem_u[0].data_ptr() + es, mem_u[1].data_ptr() + es)
                              if src == 'memory' else None)
                _launch(op, dtype, B, d, _ins(pool, op[1]), [o.data_ptr() for o in out_a], nz_a)
                _launch(op, dtype, B, d, _ins(pool_u, op[1], es), [o.data_ptr() + es for o in out_b], nz_b)
                for i in range(op[2]):
                    if not torch.equal(out_a[i], out_b[i][1:]):
                        bad.append(f'B={B} {_op_id(op)} {src} out{i}')
    assert not bad, 'fast kernel != generic kernel: ' + ', '.join(bad)
