#!/usr/bin/env python
"""PhiSNet Hamiltonian + overlap prediction (nabladft_b200.phisnet.NeuralNetwork at the shipped hyperparameters of
phisnet/configs/args_nablaDFT_*.txt, def2-SVP output basis of the fixture DB): molecules/s of the CUDA forward with full H and S
(--core adds the core-Hamiltonian head), at batch 2 (the configs' train_batch_size) and batch 32 of synthetic molecules (converted to bohr),
peak memory, a per-stage CUDA-event split (--profile), and the FLOPs / bytes of the output heads with the sparse fused head against the
full-width head GEMMs it replaces, computed from the shapes of this batch.  Secondary benchmark; prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception:  # noqa: BLE001 -- informational only
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def head_costs(net, z, sizes, with_core):
    """FLOPs and HBM bytes of the output stage per forward: full-width head (per-order Linear to all irreps columns on every atom / pair row,
    [rows*25, F] x [F, width], result written) against the sparse fused head (only the irreps each block uses; reads one feature row per
    block direction, writes the matrices)."""
    a, F = net._asm, net.num_features
    el = {z_: i for i, z_ in enumerate(a["elems"])}
    n_heads = 3 if with_core else 2
    rng = a["ent_range"]
    ent_work = lambda kind, ea, eb: int(sum(2 * L + 1 for L in a["ent_L"][rng[kind, ea, eb, 0]:rng[kind, ea, eb, 1]]))
    N, P = len(z), int(sum(n * (n - 1) for n in sizes))
    w_ii, w_ij = net.output_full_ii.num_out, net.output_full_ij.num_out
    full_flops = 2 * 25 * F * (N * w_ii + P * w_ij)
    full_bytes = 4 * 25 * (N * (F + w_ii) + P * (F + w_ij)) + 4 * 25 * F * (w_ii + w_ij)
    sp_flops, off = 0, 0
    norb2 = 0
    for n in sizes:
        zz = z[off:off + n]
        for i in range(n):
            sp_flops += 2 * F * ent_work(0, el[zz[i]], el[zz[i]])
            for j in range(n):
                if i != j:
                    sp_flops += 2 * F * ent_work(1, el[zz[i]], el[zz[j]])
        norb2 += sum(int(a["n_rows"][el[x]]) for x in zz) ** 2
        off += n
    sp_bytes = 4 * 25 * F * (N + P) + 4 * norb2
    return {"heads": n_heads, "full_width": {"gflop": round(n_heads * full_flops / 1e9, 3), "mbytes": round(n_heads * full_bytes / 1e6, 2)},
            "sparse_fused": {"gflop": round(n_heads * sp_flops / 1e9, 3), "mbytes": round(n_heads * sp_bytes / 1e6, 2)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[2, 32])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--core", action="store_true", help="also run the core-Hamiltonian head")
    ap.add_argument("--profile", action="store_true", help="per-stage CUDA-event split of one forward at the largest batch")
    ap.add_argument("--cpu", action="store_true", help="also time the float64 CPU oracle (oracle/phisnet_model.py) on one molecule")
    args = ap.parse_args()
    import numpy as np
    import torch
    from make_golden_phisnet_model import HYPER, max_orbitals_from_db, model_state_dict

    from nabladft_b200.phisnet import NeuralNetwork
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    net = NeuralNetwork(max_orbitals=max_orbitals_from_db(), **HYPER)
    sd = net.state_dict()
    net.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in model_state_dict(sd).items()}, strict=True)
    net = net.eval().to(dev)
    net.calculate_core_hamiltonian = args.core
    orb = {o[0][0]: o for o in net.max_orbitals}
    name, power = gpu_info()
    out = {"metric": "molecules/sec (PhiSNet full H + S forward)" + (" + core H" if args.core else ""), "gpu": name, "power_limit": power,
           "dtype": "f32", "data": "synthetic", "runs": []}
    for bs in args.batch:
        b = synth_batch(1, bs)
        sizes = np.diff(b["mol_ptr"]).tolist()
        z = b["z"].astype(np.int64)
        batch = {"positions": (torch.from_numpy(b["pos"]).double() * 1.8897261).float().to(dev), "atomic_numbers": torch.from_numpy(z).to(dev),
                 "orbitals": tuple(orb[int(x)] for x in z), "molecule_size": torch.tensor(sizes)}
        torch.cuda.reset_peak_memory_stats()
        for _ in range(args.warmup):
            net(batch, packed=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            net(batch, packed=True)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        run = {"batch": bs, "value": bs / (ms / 1e3), "ms_per_step": round(ms, 3), "atoms": int(len(z)), "pairs": int(sum(n * (n - 1) for n in sizes)),
               "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 3), "output_heads": head_costs(net, z.tolist(), sizes, args.core)}
        out["runs"].append(run)
    out["value"] = out["runs"][-1]["value"]
    if args.profile:
        net.profile = {}
        net(batch, packed=True)
        torch.cuda.synchronize()
        marks = net.profile["_marks"]
        out["profile_ms"] = {n0: round(a.elapsed_time(b_), 3) for (n0, a), (_, b_) in zip(marks[:-1], marks[1:])}
        net.profile = None
    if args.cpu:
        import time

        sys.path.insert(0, ROOT)
        from oracle.phisnet_model import NeuralNetwork as Oracle

        ora = Oracle(max_orbitals_from_db(), **HYPER).double()
        ora.load_state_dict({k: v.detach().cpu().double() for k, v in net.state_dict().items()}, strict=True)
        torch.set_num_threads(min(32, os.cpu_count() or 1))
        b = synth_batch(1, 1)
        heads = ("full", "over") + (("core",) if args.core else ())
        t0 = time.perf_counter()
        ora(torch.from_numpy(b["pos"]).double() * 1.8897261, torch.from_numpy(b["z"]).long(), [len(b["z"])], heads=heads)
        dt = time.perf_counter() - t0
        out["cpu_baseline"] = {"value": 1.0 / dt, "unit": "molecules/s", "cores": torch.get_num_threads(), "kind": "oracle restatement, float64",
                               "sample": f"1 synthetic molecule ({len(b['z'])} atoms)"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
