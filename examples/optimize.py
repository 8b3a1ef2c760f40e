#!/usr/bin/env python
"""Batched L-BFGS relaxation of every molecule of a packed dataset (reference: job_type optimize, config/schnet_optim.yaml and
config/gemnet-oc_optim.yaml, config/dimenetplusplus_optim-b200.yaml): `--model painn` (default), `--model gemnet-oc` or
`--model dimenetplusplus` (without --weights: the seeded test weights of tests/golden/make_golden_dimenet.py).
`--optimizer quasinewton` relaxes with ASE's QuasiNewton per molecule instead (PYGAseInterface.optimize, BatchwiseQuasiNewton)."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from nabladft_b200.data import PackedEnergyDataset  # noqa: E402
from nabladft_b200.optimization import (ASEBatchwiseLBFGS, BatchwiseQuasiNewton, PackedOptimizeTask, PyGBatchwiseCalculator,  # noqa: E402
                                        SpkBatchwiseCalculator)
from train_painn import build_model  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("cache")
    ap.add_argument("--weights")
    ap.add_argument("--model", choices=["painn", "gemnet-oc", "dimenetplusplus"], default="painn")
    ap.add_argument("--batch", type=int, default=32)   # config/schnet_optim.yaml: batch_size 32, fmax 1e-5, steps 500
    ap.add_argument("--fmax", type=float, default=1e-5)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--optimizer", choices=["lbfgs", "quasinewton"], default="lbfgs")
    a = ap.parse_args()
    if a.model == "gemnet-oc":
        import yaml

        from nabladft_b200.gemnet_oc import GemNetOC

        cfg = yaml.safe_load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "config", "model", "gemnet-oc-b200.yaml")))["net"]
        cfg.pop("_target_")
        model = GemNetOC(**cfg)
    elif a.model == "dimenetplusplus":
        import yaml
        from make_golden_dimenet import load_test_weights

        from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential

        cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "dimenetplusplus-b200.yaml")))["net"]
        cfg.pop("_target_")
        model = DimeNetPlusPlusPotential(**cfg)
        if not a.weights:
            load_test_weights(model, torch.float32)  # PyG initialises the output layers to zero: zero forces, nothing would move
    else:
        model = build_model()
    if a.weights:
        model.load_state_dict(torch.load(a.weights, map_location="cpu"), strict=True)
    calculator = SpkBatchwiseCalculator if a.model == "painn" else PyGBatchwiseCalculator
    calc = calculator(model, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    if a.optimizer == "quasinewton":
        opt = BatchwiseQuasiNewton(calc, logfile="-", check_every=10)  # pyg_opt.py: optimize(fmax=1e-4, steps=100)
    else:
        opt = ASEBatchwiseLBFGS(calc, logfile="-", check_every=10)
    out = PackedOptimizeTask(PackedEnergyDataset.load(a.cache), opt, a.batch, a.fmax, a.steps).run()
    np.savez_compressed("relaxed.npz", **out)
    print("batches", len(out["nsteps"]), "steps per batch", out["nsteps"].tolist()[:8], "-> relaxed.npz")


if __name__ == "__main__":
    main()
