"""Golden Hessians for the DimeNet++ Hessian-vector pass: the float64 oracle's double backward (oracle/dimenet.py) of the unscaled prediction
on fixture molecules 26, 3 and 99 (29, 30 and 54 atoms), at the config's sizes (6 blocks, L = 50, K = 32) with the shared test weights
(make_golden_dimenet.load_test_weights).  The oracle runs on the CPU only and 339 double-backward passes take minutes, so the GPU test reads
them from here.  Stored in float32: the tests hold the engine to 1e-4 of max |H|.

    python tests/golden/make_golden_dimenet_hessian.py      # writes tests/golden/dimenet_hessian.npz
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, HERE); sys.path.insert(0, os.path.dirname(HERE))
from make_golden_dimenet import SCALER, load_test_weights  # noqa: E402

MOLS = [26, 3, 99]


def oracle_hessian(ora, z, pos) -> np.ndarray:
    """[3n, 3n] float64: d^2 y / dR dR of one molecule's unscaled prediction, one backward per column."""
    pos = torch.as_tensor(pos).double().detach().requires_grad_(True)
    g = ora.net(z=torch.as_tensor(z).long(), pos=pos, batch=torch.zeros(len(z), dtype=torch.long))
    dy = torch.autograd.grad(ora.regr_or_cls_nn(g).sum(), pos, create_graph=True)[0].reshape(-1)
    n3 = dy.numel()
    eye = torch.eye(n3, dtype=torch.float64)
    return torch.stack([torch.autograd.grad(dy, pos, grad_outputs=eye[k], retain_graph=True)[0].reshape(-1)
                        for k in range(n3)], 1).numpy()


def main():
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    torch.manual_seed(0)
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(node_latent_dim=50, scaler=SCALER, dimenet_num_blocks=6, dimenet_max_num_neighbors=32,
                                                           do_postprocessing=True).double().eval())
    fx = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    out = {}
    for m in MOLS:
        a, b = fx["ptr"][m], fx["ptr"][m + 1]
        pos = fx["pos"][a:b].astype(np.float32)  # the positions the fp32 engine sees
        out[f"hessian_{m}"] = oracle_hessian(ora, fx["z"][a:b], pos).astype(np.float32)
        print(m, b - a, float(np.abs(out[f"hessian_{m}"]).max()))
    np.savez_compressed(os.path.join(HERE, "dimenet_hessian.npz"), mols=np.array(MOLS), **out)


if __name__ == "__main__":
    main()
