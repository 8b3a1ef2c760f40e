#!/usr/bin/env python
"""QHNet Hamiltonian prediction (BASELINE.json configs[3]: def2-SVP, 64-molecule batch, 1xH100): molecules/s of the
CUDA path, a per-stage breakdown with CUDA events, and the CPU oracle on one molecule.  Secondary benchmark
(the driver's headline is bench.py); prints one JSON line."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

ORBITALS = {1: [0, 0, 1], 6: [0, 0, 0, 1, 1, 2], 7: [0, 0, 0, 1, 1, 2], 8: [0, 0, 0, 1, 1, 2], 9: [0, 0, 0, 1, 1, 2],
            16: [0, 0, 0, 0, 1, 1, 1, 2], 17: [0, 0, 0, 0, 1, 1, 1, 2], 35: [0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu", action="store_true", help="also time the CPU oracle on one molecule")
    ap.add_argument("--profile", action="store_true", help="per-op CUDA-event breakdown of one forward (GEMM classes)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from helpers import load_golden_weights

    from nabladft_b200.qhnet import QHNet
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    net = QHNet(sh_lmax=4, hidden_size=128, bottle_hidden_size=32, num_gnn_layers=5, max_radius=12, num_nodes=83, radius_embed_dim=32, orbitals=ORBITALS)
    load_golden_weights(net, torch.float32, style="e3")
    net = net.eval().to(dev)
    b = synth_batch(1, args.batch)

    class D:
        pass

    d = D()
    d.z = torch.from_numpy(b["z"]).to(dev)
    d.pos = (torch.from_numpy(b["pos"]) * 1.8897261).to(dev)  # Hamiltonian DBs are in bohr
    d.batch = torch.from_numpy(b["batch"]).to(dev)
    d.ptr = torch.from_numpy(b["mol_ptr"]).long().to(dev)
    n_per = np.diff(b["mol_ptr"])
    for _ in range(args.warmup):
        H = net(d, keep_blocks=True)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        H = net(d, keep_blocks=True)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / args.steps
    out = {"metric": "molecules/sec (QHNet H blocks forward)", "value": args.batch / (ms / 1e3), "ms_per_step": ms, "batch": args.batch,
           "atoms": int(b["z"].shape[0]), "pairs": int((n_per * (n_per - 1)).sum()), "peak_mem_gb": torch.cuda.max_memory_allocated() / 2**30,
           "dtype": "f32", "data": "synthetic"}
    if args.profile:
        net.profile = {}
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record(); net(d, keep_blocks=True); t1.record(); torch.cuda.synchronize()
        out["profile_ms"] = {k: round(sum(a.elapsed_time(b) for a, b in v), 3) for k, v in net.profile.items()}
        out["profile_ms"]["total_with_events"] = round(t0.elapsed_time(t1), 3)
        out["profile_calls"] = {k: len(v) for k, v in net.profile.items()}
        net.profile = None
    if args.cpu:
        from oracle.qhnet import QHNetOracle
        ora = QHNetOracle(orbitals=ORBITALS)
        ora.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, strict=True)
        torch.set_num_threads(min(32, os.cpu_count() or 1))
        n0 = int(b["mol_ptr"][1])
        z, pos, bt = d.z[:n0].cpu().long(), d.pos[:n0].cpu(), d.batch[:n0].cpu()
        with torch.no_grad():
            t0 = time.perf_counter()
            ora.blocks(z, pos, bt)
            dt = time.perf_counter() - t0
        out["cpu_baseline"] = {"value": 1.0 / dt, "unit": "molecules/s", "cores": torch.get_num_threads(), "kind": "port",
                               "sample": f"1 molecule ({n0} atoms), oracle restatement fp32"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
