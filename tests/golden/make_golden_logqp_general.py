"""Generate tests/golden/logqpgen_*.npz by running the REFERENCE (google-research/torchsde v0.2.6) on the CPU:
`logqp=True` solves with general-noise shapes beyond the d = 4, m = 3 of make_golden.py's logqp cases — d < m,
d = m, scalar (m = 1) and additive noise, and a diffusion with a structurally zero column or row — forward solves
under no_grad, and the gradients of a loss of ys and the log-ratio through sdeint_adjoint.

    python tests/golden/make_golden_logqp_general.py

The problems are tests/logqp_general_ref.py's LatentGeneral, named by logqp_general_ref.GOLDEN_CASES.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle', 'refshim'))
sys.path.insert(0, os.path.join(ROOT, 'oracle', '_ref', 'site'))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torchsde  # noqa: E402  (the reference)

from tests import logqp_general_ref as lg  # noqa: E402
from tests.golden.make_golden import Recorder, _rec_save  # noqa: E402

assert torchsde.__version__ == '0.2.6'


def main():
    for i, (name, (d, m, noise, sde_type, method, adjoint, zc, zr)) in enumerate(lg.GOLDEN_CASES.items()):
        torch.manual_seed(4700 + i)
        tdt = torch.float64
        sde = lg.LatentGeneral(d, m, noise, sde_type, seed=i, dtype=tdt, zero_col=zc, zero_row=zr)
        B = 5
        y0 = (0.1 + 0.5 * torch.rand(B, d, dtype=tdt)).requires_grad_(adjoint)
        ts = torch.tensor([0.0, 0.1, 0.2, 0.3], dtype=tdt)
        levy = 'space-time' if method == 'srk' else 'none'
        bm = torchsde.BrownianInterval(0.0, 0.3, size=(B, m), dtype=tdt, entropy=4700 + i, levy_area_approximation=levy)
        rec = Recorder(bm)
        save = dict(ts=ts.numpy(), dt=np.float64(0.05), name=name, seed=i)
        if adjoint:
            ys, logqp = torchsde.sdeint_adjoint(sde, y0, ts, bm=rec, method=method, dt=0.05, logqp=True)
            wy = torch.linspace(0.5, 1.5, ys.numel(), dtype=tdt).reshape(ys.shape)
            wl = torch.linspace(1.0, 2.0, logqp.numel(), dtype=tdt).reshape(logqp.shape)
            ((ys * wy).sum() + (logqp * wl).sum()).backward()
            save.update(wy=wy.numpy(), wl=wl.numpy(), grad_y0=y0.grad.numpy())
            for n, p in sde.named_parameters():
                save['grad.' + n] = (torch.zeros_like(p) if p.grad is None else p.grad).numpy()
        else:
            with torch.no_grad():
                ys, logqp = torchsde.sdeint(sde, y0, ts, bm=rec, method=method, dt=0.05, logqp=True)
        save.update(y0=y0.detach().numpy(), ys=ys.detach().numpy(), logqp=logqp.detach().numpy())
        np.savez_compressed(os.path.join(HERE, f'logqpgen_{name}.npz'), **_rec_save(rec, save))
        print('wrote logqpgen', name)


if __name__ == '__main__':
    main()
