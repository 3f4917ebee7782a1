"""Small launches of the adaptive proposal kernels (tsde_adaptive_proposal_pointwise), for compute-sanitizer:

    compute-sanitizer --tool memcheck   python profiles/sanitize_adaptive.py
    compute-sanitizer --tool racecheck  python profiles/sanitize_adaptive.py

Every method (the interpreted Euler, SRK and predictor-corrector kernels and the compiled Milstein one), float32 and
float64, on the vector path (d % 4 == 0) and the element path (d = 5, 13: a partial last quad), with a batch whose
last CTA is partly empty.  Each fused solve is compared with the unfused one bit for bit, so that a sanitizer-clean
but wrong kernel would still fail, and the launch counter confirms that the proposal kernels ran.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch import nn  # noqa: E402

import torchsde_b200 as tsde  # noqa: E402
from torchsde_b200 import _cabi  # noqa: E402
from torchsde_b200._core import pointwise  # noqa: E402

DEV = torch.device('cuda')
METHODS = [('euler', 'ito'), ('milstein', 'ito'), ('milstein', 'stratonovich'), ('srk', 'ito'),
           ('heun', 'stratonovich'), ('midpoint', 'stratonovich'), ('euler_heun', 'stratonovich')]


class CIR(nn.Module):
    noise_type = 'diagonal'

    def __init__(self, sde_type, d, dtype):
        super().__init__()
        self.sde_type = sde_type
        gen = torch.Generator().manual_seed(1)
        self.kappa = nn.Parameter((torch.rand(d, generator=gen, dtype=torch.float64) + 0.5).to(dtype))
        self.xi = nn.Parameter((torch.rand(d, generator=gen, dtype=torch.float64) * 0.4 + 0.2).to(dtype))

    def f(self, t, y):
        return self.kappa * (0.05 - y.clamp(min=0))

    def g(self, t, y):
        return self.xi * torch.sqrt(y.clamp(min=0))


def solve(method, sde_type, B, d, dtype, reject):
    sde = CIR(sde_type, d, dtype).to(DEV)
    if reject:
        saved = pointwise.Recorder.finish, pointwise.SrkRecorder.finish
        pointwise.Recorder.finish = lambda self, *a: None
        pointwise.SrkRecorder.finish = lambda self: None
    try:
        bm = tsde.BrownianInterval(0.0, 0.2, size=(B, d), dtype=dtype, device=DEV, entropy=3,
                                   levy_area_approximation='space-time' if method == 'srk' else 'none')
        with torch.no_grad():
            return tsde.sdeint(sde, torch.full((B, d), 0.05, dtype=dtype, device=DEV),
                               torch.tensor([0.0, 0.07, 0.2], dtype=dtype, device=DEV), bm=bm, method=method,
                               dt=0.05, adaptive=True, rtol=1e-3, atol=1e-4)
    finally:
        if reject:
            pointwise.Recorder.finish, pointwise.SrkRecorder.finish = saved


checked = 0
for dtype in (torch.float32, torch.float64):
    for B, d in ((300, 8), (77, 5), (129, 13)):
        for method, sde_type in METHODS:
            n0 = _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE)
            ys = solve(method, sde_type, B, d, dtype, False)
            assert _cabi.lib().tsde_kernel_launches(_cabi.KERNEL_PW_ADAPTIVE) > n0, (method, B, d, dtype)
            ref = solve(method, sde_type, B, d, dtype, True)
            bits = torch.int32 if dtype == torch.float32 else torch.int64
            assert torch.equal(ys.view(bits), ref.view(bits)), (method, sde_type, B, d, dtype)
            checked += 1
torch.cuda.synchronize()
print('sanitize_adaptive ok,', checked, 'checked solves')
