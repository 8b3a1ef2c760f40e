"""Golden force Jacobians for the GemNet-OC tangent pass: -(dF/dR) of the float64 oracle's direct forces (oracle/gemnet_oc.py) by reverse-mode
autograd, one backward per row, on fixture molecules 26 and 3 (29 and 30 atoms) at the config's sizes with the shared test weights
(tests/test_gemnet_emu._models(True): golden weights, random scale factors).  The oracle runs on the CPU only and 177 backward passes at these
sizes take minutes, so the GPU test reads them from here.  Stored in float32: the tests hold the engine to 1e-4 of max |J|.

    python tests/golden/make_golden_gemnet_oc_jacobian.py      # writes tests/golden/gemnet_oc_jacobian.npz
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, HERE); sys.path.insert(0, os.path.dirname(HERE))
from test_gemnet_emu import _models  # noqa: E402

MOLS = [26, 3]


def oracle_jacobian(ora, z, pos) -> np.ndarray:
    """[3n, 3n] float64: J[i, j] = -dF_i / dR_j of one molecule (rows and columns ordered (atom, xyz))."""
    pos = torch.as_tensor(pos).double().detach().requires_grad_(True)
    f = ora(torch.as_tensor(z).long(), pos, torch.zeros(len(z), dtype=torch.long))[1].reshape(-1)
    eye = torch.eye(f.numel(), dtype=torch.float64)
    return -torch.stack([torch.autograd.grad(f, pos, grad_outputs=eye[k], retain_graph=True)[0].reshape(-1) for k in range(f.numel())]).numpy()


def main():
    _, ora = _models(True)
    ora = ora.double().eval()
    fx = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    out = {}
    for m in MOLS:
        a, b = fx["ptr"][m], fx["ptr"][m + 1]
        pos = fx["pos"][a:b].astype(np.float32)  # the positions the fp32 engine sees
        out[f"jacobian_{m}"] = oracle_jacobian(ora, fx["z"][a:b], pos).astype(np.float32)
        print(m, b - a, float(np.abs(out[f"jacobian_{m}"]).max()), flush=True)
    np.savez_compressed(os.path.join(HERE, "gemnet_oc_jacobian.npz"), mols=np.array(MOLS), **out)


if __name__ == "__main__":
    main()
