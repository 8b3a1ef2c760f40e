#!/usr/bin/env python
"""Relax a batch of fixture molecules with the batched L-BFGS, equilibrate them with Langevin dynamics at 300 K, then run NVE and print
each molecule's temperature and total-energy drift: the reference's `init_md` / `run_md` (PYGAseInterface, ASE dynamics of one molecule)
for a whole batch on the GPU.  `--model painn` (default: spk PaiNN) or `--model dimenetplusplus` (config/model/dimenetplusplus.yaml, run
without postprocessing so that the logged total energy is the one the forces conserve, DESIGN.md 3.15.3)."""
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
from make_golden_dimenet import load_test_weights  # noqa: E402

from nabladft_b200 import spk  # noqa: E402
from nabladft_b200.md import BatchwiseMD  # noqa: E402
from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms, SpkBatchwiseCalculator  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, nargs="+", default=[0, 3, 26, 99])
    ap.add_argument("--model", choices=["painn", "dimenetplusplus"], default="painn")
    ap.add_argument("--weights", help="state dict of the model (default: the seeded test weights)")
    ap.add_argument("--nvt-steps", type=int, default=2000)
    ap.add_argument("--nve-steps", type=int, default=2000)
    ap.add_argument("--workdir", help="write {name}_{i}.log (and .traj with ASE) here")
    a = ap.parse_args()
    if a.model == "dimenetplusplus":
        import yaml

        from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential

        cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "dimenetplusplus-b200.yaml")))["net"]
        cfg.pop("_target_")
        cfg["do_postprocessing"] = False
        model = DimeNetPlusPlusPotential(**cfg)
    else:
        model = spk.NeuralNetworkPotential(
            representation=spk.PaiNN(n_atom_basis=128, n_interactions=3, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                     cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
            input_modules=[spk.PairwiseDistances()], output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()])
    if a.weights:
        model.load_state_dict(torch.load(a.weights, map_location="cpu"), strict=True)
    elif a.model == "dimenetplusplus":
        load_test_weights(model, torch.float32)
    else:
        load_golden_weights(model, torch.float32)
    z, pos, batch = load_fixture(a.mols)
    sizes = torch.bincount(batch).tolist()
    off = np.concatenate([[0], np.cumsum(sizes)])
    atoms = [SimpleAtoms(pos[off[i]:off[i + 1]].numpy(), z[off[i]:off[i + 1]].numpy()) for i in range(len(sizes))]
    calculator = PyGBatchwiseCalculator if a.model == "dimenetplusplus" else SpkBatchwiseCalculator
    calc = calculator(model, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None)
    print(f"relaxation converged: {opt.run(atoms, fmax=1e-3, steps=1000)} after {opt.nsteps} steps")

    md = BatchwiseMD(calc, opt.atoms, working_dir=a.workdir, seed=0)
    md.init_md("nvt", time_step=0.5, temp_init=300, temp_bath=300, interval=10)
    md.run_md(a.nvt_steps)
    t_nvt = md.log[md.log.shape[0] // 2:, :, 4].mean(0)
    md.init_md("nve", time_step=0.5, interval=10)  # keeps the equilibrated velocities
    md.run_md(a.nve_steps)
    etot = md.log[:, :, 1]
    mass = md._mass.cpu().numpy()
    for i, mol in enumerate(a.mols):
        # ASE 3.22's fixcm leaves T_bath (n - 2 + sum(m) sum(1/m) / n^2) / n for free particles of unequal masses (DESIGN.md section 3.14)
        m, n = mass[off[i]:off[i + 1]], sizes[i]
        target = 300 * (n - 2 + m.sum() * (1 / m).sum() / n ** 2) / n
        print(f"molecule {mol:3d}: {n:2d} atoms, Langevin mean T {t_nvt[i]:6.1f} K (free-particle value {target:.1f} K), "
              f"NVE mean T {md.log[:, i, 4].mean():6.1f} K, Etot drift {etot[-1, i] - etot[0, i]:+.5f} eV, "
              f"max |Etot - Etot(0)| {np.abs(etot[:, i] - etot[0, i]).max():.5f} eV")


if __name__ == "__main__":
    main()
