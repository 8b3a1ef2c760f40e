#!/usr/bin/env python
"""DimeNet++ energy + conservative forces (config/model/dimenetplusplus.yaml sizes): molecules/s of the CUDA path (CUDA events) on a batch of
synthetic molecules and on tiled fixture molecules, graph sizes, the engine's per-category split (GEMM separated from the triplet / basis
kernels), GEMM FLOP/s from shapes over GEMM kernel time, the CPU float64 oracle on a bounded sample, and the card it ran on.  One JSON line.

    python bench_dimenet.py --batch 256 [--steps 5 --warmup 2 --oracle-mols 2]
    python bench_dimenet.py --train [--batch 256 --steps 5 --warmup 2]

--train: one training step (forward, L1(E) + L1(F), backward through nb200_dimenet_train_grads, Adam lr 1e-4 as the yaml has it) on the same
synthetic batch: ms per step (CUDA events, warm-up excluded), molecules/s, the per-category split of the gradient call (weight-gradient
reductions are counted as force_assembly there: that call assembles no forces) and its workspace bytes.
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
    ap.add_argument("--train", action="store_true", help="time a training step instead of the energy + forces call")
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
    if args.train:
        return train_main(args, net, runner, synth, s)
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


def card_name() -> str:
    import torch

    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as exc:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unknown: {exc})"


def train_main(args, net, runner, synth, s):
    import ctypes

    import torch

    from nabladft_b200.dimenetplusplus import DimeNetEnergyFn

    gen = torch.Generator().manual_seed(0)
    e_t = (torch.randn(args.batch, generator=gen) - 40.0).cuda()
    f_t = (0.1 * torch.randn(len(s["z"]), 3, generator=gen)).cuda()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    net.train()

    def step():
        opt.zero_grad(set_to_none=True)
        e, f = net(synth)
        loss = (e - e_t).abs().mean() + (f - f_t).abs().mean()
        loss.backward()
        opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        step()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / args.steps
    counts = dict(runner.last_counts)
    # per-category split of the gradient call alone (nb200_dimenet_train_grads)
    lib = runner.lib
    z, pos, mol_ptr, n_mol = net.batch_args(synth.z, synth.pos, synth.batch)
    flat, offs = net._export_impl(detach=True)
    runner.bind(net, flat, offs)
    se, sf = torch.ones(n_mol, device="cuda"), torch.ones(len(s["z"]), 3, device="cuda")
    runner.train_grads(z, pos, mol_ptr, n_mol, se, sf)
    torch.cuda.synchronize()
    c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    lib.nb200_engine_set_timing(runner._h, 1)
    c0.record()
    runner.train_grads(z, pos, mol_ptr, n_mol, se, sf)
    c1.record()
    torch.cuda.synchronize()
    ms_cat = (ctypes.c_float * 16)()
    n_cat = (ctypes.c_int32 * 16)()
    lib.nb200_engine_read_timings(runner._h, ms_cat, n_cat, 16)
    lib.nb200_engine_set_timing(runner._h, 0)
    names = list(CATS)
    names[CATS.index("force_assembly")] = "weight_gradients"
    split = {names[i]: round(ms_cat[i], 3) for i in range(len(CATS))}
    cnt = (ctypes.c_int64 * 4)(counts["edges"], counts["triplets"], 0, 0)
    ws = lib.nb200_dimenet_train_workspace_bytes(ctypes.byref(runner._w), n_mol, len(s["z"]), cnt)
    out = {
        "metric": "dimenet_train_step_molecules_per_s", "value": round(args.batch / (ms / 1e3), 2), "batch": args.batch, "ms_per_step": round(ms, 3),
        "atoms": int(len(s["z"])), "edges": counts["edges"], "triplets": counts["triplets"],
        "train_grads_call_ms_timed": round(c0.elapsed_time(c1), 3), "train_grads_ms_by_category": split, "train_workspace_bytes": int(ws),
        "peak_memory_bytes": int(torch.cuda.max_memory_allocated()), "card": card_name(), "steps": args.steps, "warmup": args.warmup,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
