#!/usr/bin/env python
"""DimeNet++ energy + conservative forces (config/model/dimenetplusplus.yaml sizes): molecules/s of the CUDA path (CUDA events) on a batch of
synthetic molecules and on tiled fixture molecules, graph sizes, the engine's per-category split (GEMM separated from the triplet / basis
kernels), GEMM FLOP/s from shapes over GEMM kernel time, the CPU float64 oracle on a bounded sample, and the card it ran on.  One JSON line.

    python bench_dimenet.py --batch 256 [--steps 5 --warmup 2 --oracle-mols 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

CATS = ["neighbor_build", "bases", "embedding", "gemm", "elementwise", "triplet_fwd", "triplet_bwd", "readout", "force_assembly"]


def gemm_macs(n_atoms: int, n_edges: int, num_blocks: int = 6, latent: int = 50) -> int:
    """Multiply-accumulates of the dense layers of one energy + forces call (csrc/dimenet.cu): the forward, the reverse pass (one transposed
    GEMM per forward GEMM) and the recompute of num_blocks - 1 interaction blocks in the reverse pass."""
    E, N, H = n_edges, n_atoms, 256
    inter = E * H * H * 2 + E * H * 64 * 2 + E * H * H * 6 + E * H * H  # lin_ji, lin_kj, down, up, 3 residual layers, lin
    out = N * H * H * 4 + N * H * latent                                 # lin_up, 3 lins, lin
    emb = E * H * H
    fwd = emb + num_blocks * inter + (num_blocks + 1) * out
    return 2 * fwd + (num_blocks - 1) * inter


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-mols", type=int, default=2, help="molecules the CPU float64 oracle runs (its time is scaled to the batch)")
    args = ap.parse_args()
    import ctypes

    import numpy as np
    import torch
    import yaml
    from make_golden_dimenet import load_test_weights

    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from nabladft_b200.synth import synth_batch
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    if not torch.cuda.is_available():
        raise SystemExit("bench_dimenet.py measures the CUDA path: no GPU")
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "dimenetplusplus-b200.yaml")))["net"]
    cfg.pop("_target_")
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(**cfg).double().eval())
    net = DimeNetPlusPlusPotential(**cfg).eval()
    net.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    net = net.cuda()

    class D:
        def __init__(self, z, pos, batch):
            self.z, self.pos, self.batch = z, pos, batch

    def batch_of(z, pos, mol_ptr):
        batch = np.repeat(np.arange(len(mol_ptr) - 1), np.diff(mol_ptr))
        return D(torch.from_numpy(z).long().cuda(), torch.from_numpy(pos).float().cuda(), torch.from_numpy(batch).long().cuda())

    def timed(data):
        for _ in range(args.warmup):
            net(data)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            net(data)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    runner = net._get_runner()
    s = synth_batch(0, args.batch)
    synth = batch_of(s["z"], s["pos"], s["mol_ptr"])
    ms_synth = timed(synth)
    counts = dict(runner.last_counts)
    n_atoms = int(len(s["z"]))
    # per-category split of one call
    lib = runner.lib
    lib.nb200_engine_set_timing(runner._h, 1)
    net(synth)
    torch.cuda.synchronize()
    ms_cat = (ctypes.c_float * 16)()
    n_cat = (ctypes.c_int32 * 16)()
    lib.nb200_engine_read_timings(runner._h, ms_cat, n_cat, 16)
    lib.nb200_engine_set_timing(runner._h, 0)
    split = {CATS[i]: round(ms_cat[i], 3) for i in range(len(CATS))}
    macs = gemm_macs(n_atoms, counts["edges"], net.num_blocks, net.node_latent_dim)
    # tiled fixture molecules
    fx = np.load(os.path.join(ROOT, "tests", "golden", "fixture_molecules.npz"))
    ids = [m % (len(fx["ptr"]) - 1) for m in range(args.batch)]
    zf = np.concatenate([fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in ids]).astype(np.int32)
    pf = np.concatenate([fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in ids]).astype(np.float32)
    ptr_f = np.concatenate([[0], np.cumsum([fx["ptr"][m + 1] - fx["ptr"][m] for m in ids])])
    ms_fix = timed(batch_of(zf, pf, ptr_f))
    counts_fix = dict(runner.last_counts)
    # CPU oracle on a bounded sample
    k = max(1, min(args.oracle_mols, args.batch))
    t0 = time.perf_counter()
    for m in range(k):
        a, b = s["mol_ptr"][m], s["mol_ptr"][m + 1]
        ora(torch.from_numpy(s["z"][a:b]).long(), torch.from_numpy(s["pos"][a:b]).double(), torch.zeros(b - a, dtype=torch.long))
    oracle_s_per_mol = (time.perf_counter() - t0) / k
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as exc:  # noqa: BLE001
        card = f"{torch.cuda.get_device_name()} (power limit unknown: {exc})"
    out = {
        "metric": "dimenet_energy_forces_molecules_per_s", "value": round(args.batch / (ms_synth / 1e3), 2),
        "batch": args.batch, "ms_per_call_synth": round(ms_synth, 3),
        "atoms": n_atoms, "edges": counts["edges"], "triplets": counts["triplets"],
        "fixture_tiled": {"molecules_per_s": round(args.batch / (ms_fix / 1e3), 2), "ms_per_call": round(ms_fix, 3), "atoms": int(len(zf)),
                          "edges": counts_fix["edges"], "triplets": counts_fix["triplets"]},
        "ms_by_category": split,
        "gemm": {"flop": 2 * macs, "ms": split["gemm"], "tflops": round(2 * macs / (split["gemm"] * 1e-3) / 1e12, 2) if split["gemm"] > 0 else None},
        "oracle_cpu_float64": {"molecules": k, "s_per_molecule": round(oracle_s_per_mol, 3),
                               "speedup_vs_oracle": round(oracle_s_per_mol * args.batch / (ms_synth / 1e3), 1)},
        "card": card, "steps": args.steps, "warmup": args.warmup,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
