#!/usr/bin/env python
"""Relax a batch of fixture molecules with the batched L-BFGS, then check each relaxed conformer with its exact normal modes: the lowest
non-rigid wavenumbers and the count of imaginary modes (what `PYGAseInterface.compute_normal_modes` does with ASE Vibrations, one
molecule at a time).  --model picks the spk representation, PaiNN or SchNet, or GemNet-OC (config/model/gemnet-oc.yaml).  GemNet-OC predicts
its forces directly: its "Hessian" is the symmetric part of the force Jacobian -(dF/dR), what ASE `Vibrations` computes from central
differences, and the ASE-style summary of every molecule is printed with the size of the discarded non-conservative part."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from helpers import load_fixture, load_golden_weights  # noqa: E402

from nabladft_b200 import spk  # noqa: E402
from nabladft_b200 import vibrations as vib  # noqa: E402
from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms, SpkBatchwiseCalculator  # noqa: E402


def gemnet_oc(weights):
    import yaml

    from nabladft_b200.gemnet_oc import GemNetOC

    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "gemnet-oc-b200.yaml")))["net"]
    cfg.pop("_target_")
    model = GemNetOC(**cfg)
    if weights:
        model.load_state_dict(torch.load(weights, map_location="cpu"), strict=True)
    else:
        from weights import golden_state_dict

        sd = model.state_dict()  # the seeded test weights; the scale factors stay unfitted (identity)
        for k, val in golden_state_dict(sd, bias_std=0.02, weight_scale=0.5).items():
            if not k.endswith("scale_factor"):
                sd[k] = torch.as_tensor(np.asarray(val)).float().reshape(sd[k].shape)
        model.load_state_dict(sd, strict=True)
    return model.eval()


class PyGBatch:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, nargs="+", default=[0, 3, 26, 99])
    ap.add_argument("--model", default="painn", choices=["painn", "schnet", "gemnet-oc"])
    ap.add_argument("--weights", help="state dict of the model (default: the seeded test weights)")
    ap.add_argument("--fmax", type=float, default=1e-4)
    ap.add_argument("--steps", type=int, default=1000)
    a = ap.parse_args()
    if a.model == "gemnet-oc":
        model = gemnet_oc(a.weights)
    else:
        rep = spk.PaiNN if a.model == "painn" else spk.SchNet
        model = spk.NeuralNetworkPotential(
            representation=rep(n_atom_basis=128, n_interactions=3, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                               cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
            input_modules=[spk.PairwiseDistances()], output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()])
        if a.weights:
            model.load_state_dict(torch.load(a.weights, map_location="cpu"), strict=True)
        else:
            load_golden_weights(model, torch.float32)
    z, pos, batch = load_fixture(a.mols)
    sizes = torch.bincount(batch).tolist()
    atoms, start = [], 0
    for n in sizes:
        atoms.append(SimpleAtoms(pos[start:start + n].numpy(), z[start:start + n].numpy()))
        start += n
    calculator = PyGBatchwiseCalculator if a.model == "gemnet-oc" else SpkBatchwiseCalculator
    calc = calculator(model, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None)
    converged = opt.run(atoms, fmax=a.fmax, steps=a.steps)
    relaxed = torch.cat([torch.from_numpy(x.get_positions()) for x in opt.atoms]).float().cuda()
    if a.model == "gemnet-oc":
        inputs = PyGBatch(z.cuda(), relaxed, batch.cuda())
    else:
        inputs = {"_atomic_numbers": z.cuda(), "_positions": relaxed, "_idx_m": batch.cuda(), "_n_atoms": torch.tensor(sizes).cuda()}
    with torch.no_grad():
        hs = vib.hessians(model, inputs)
    masses = vib.masses_of(z)
    ptr = [0] + torch.tensor(sizes).cumsum(0).tolist()
    modes = [vib.normal_modes_from_hessian(h, masses[p:q].to(h.device), relaxed[p:q], project=True) for h, p, q in zip(hs, ptr[:-1], ptr[1:])]
    print(f"relaxation converged: {converged}")
    if a.model == "gemnet-oc":
        print(f"non-conservative part of the direct forces: max |J_ij - J_ji| = {hs.max_asymmetry:.3e} Ha/A^2 (discarded by the symmetrisation)")
        for mol, nm in zip(a.mols, modes):
            print(f"molecule {mol}:")
            print(vib.summary(nm))
    for mol, n, nm in zip(a.mols, sizes, modes):
        n_rigid = 3 if n == 1 else 5 if n == 2 else 6
        nu = nm.wavenumbers.cpu()
        order = nu.abs().argsort()
        vib_nu = nu[order[n_rigid:]].sort().values  # rigid-body modes are the exact zeros left by the projection
        print(f"molecule {mol:3d}: {n:2d} atoms, lowest wavenumbers (cm^-1) {[round(x, 1) for x in vib_nu[:4].tolist()]}, "
              f"imaginary modes {int((vib_nu < 0).sum())}")


if __name__ == "__main__":
    main()
