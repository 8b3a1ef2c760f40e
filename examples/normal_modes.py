#!/usr/bin/env python
"""Relax a batch of fixture molecules with the batched L-BFGS, then check each relaxed conformer with its exact normal modes: the lowest
non-rigid wavenumbers and the count of imaginary modes (what `PYGAseInterface.compute_normal_modes` does with ASE Vibrations, one
molecule at a time).  --model picks the spk representation: PaiNN or SchNet."""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from helpers import load_fixture, load_golden_weights  # noqa: E402

from nabladft_b200 import spk  # noqa: E402
from nabladft_b200 import vibrations as vib  # noqa: E402
from nabladft_b200.optimization import ASEBatchwiseLBFGS, SimpleAtoms, SpkBatchwiseCalculator  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, nargs="+", default=[0, 3, 26, 99])
    ap.add_argument("--model", default="painn", choices=["painn", "schnet"])
    ap.add_argument("--weights", help="state dict of the spk model (default: the seeded test weights)")
    ap.add_argument("--fmax", type=float, default=1e-4)
    ap.add_argument("--steps", type=int, default=1000)
    a = ap.parse_args()
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
    calc = SpkBatchwiseCalculator(model, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None)
    converged = opt.run(atoms, fmax=a.fmax, steps=a.steps)
    relaxed = torch.cat([torch.from_numpy(x.get_positions()) for x in opt.atoms]).float().cuda()
    inputs = {"_atomic_numbers": z.cuda(), "_positions": relaxed, "_idx_m": batch.cuda(), "_n_atoms": torch.tensor(sizes).cuda()}
    with torch.no_grad():
        modes = vib.normal_modes(model, inputs, project=True)
    print(f"relaxation converged: {converged}")
    for mol, n, nm in zip(a.mols, sizes, modes):
        n_rigid = 3 if n == 1 else 5 if n == 2 else 6
        nu = nm.wavenumbers.cpu()
        order = nu.abs().argsort()
        vib_nu = nu[order[n_rigid:]].sort().values  # rigid-body modes are the exact zeros left by the projection
        print(f"molecule {mol:3d}: {n:2d} atoms, lowest wavenumbers (cm^-1) {[round(x, 1) for x in vib_nu[:4].tolist()]}, "
              f"imaginary modes {int((vib_nu < 0).sum())}")


if __name__ == "__main__":
    main()
