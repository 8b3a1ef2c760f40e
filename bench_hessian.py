"""Throughput of exact Hessians (nb200_painn_hvp, nb200_schnet_hvp) on the config-2 batch: 256 synthetic conformations (synth.py), one JSON
line.

    python bench_hessian.py [--model painn|painn-oc|schnet] [--max-dir D] [--repeats R]

Reports Hessians / s and HVP directions / s for the whole batch (3 n_max shared directions, chunks of --max-dir), peak device memory, ms per
direction split into the tangent forward and the backward (CUDA events around the engine's launch categories), and the same Hessians by
batched central finite differences of the inference engine (nb200_painn_energy_forces, nb200_schnet_energy_forces; two force calls per
direction, step 1e-3 A) with their deviation from the analytic ones.  For SchNet the per-direction split is also given per launch category
(marginal ms per direction of each, from the engine's CUDA-event timing of an n_dir call minus a one-direction call).  Card name and power
limit come from the same run.  Writes nothing into the tree.
"""
import argparse
import ctypes
import json
import subprocess
import time

import numpy as np


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="painn", choices=["painn", "painn-oc", "schnet"])
    ap.add_argument("--max-dir", type=int, default=None)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fd-step", type=float, default=1e-3)
    args = ap.parse_args()

    import torch

    from bench import build_model
    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    model = build_model(args.model, dev)
    b = synth_batch(1, 256)
    z = torch.from_numpy(b["z"]).to(dev)
    pos = torch.from_numpy(b["pos"]).to(dev)
    bt = torch.from_numpy(b["batch"]).to(dev)
    if args.model in ("painn", "schnet"):
        batch = {"_atomic_numbers": z.long(), "_positions": pos, "_idx_m": bt, "_n_atoms": torch.bincount(bt)}
    else:
        class D:
            pass

        batch = D()
        batch.z, batch.pos, batch.batch = z.long(), pos, bt
    eng, zi, posf, mol_ptr, n_mol = vib._engine_inputs(model, batch)
    ptr = mol_ptr.cpu().tolist()
    n_max = max(b - a for a, b in zip(ptr[:-1], ptr[1:]))
    n_dir = 3 * n_max
    N = zi.numel()

    # analytic: warm-up, then timed repeats
    hs = vib.hessians(model, batch, args.max_dir)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    times = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        hs = vib.hessians(model, batch, args.max_dir)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    t_an = float(np.median(times))
    peak = torch.cuda.max_memory_allocated(dev)

    # per direction: (T(n_dir) - T(1)) / (n_dir - 1) removes the once-per-call graph, filters and primal forward; the tangent forward's share
    # is its CAT_MSG_FWD event scope (engine timing on; that category also holds the primal's L message kernels, once per call)
    lib = eng.lib
    v = vib.shared_directions(ptr, 0, n_dir, dev)

    def timed(vv):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.run_hvp(zi, posf, mol_ptr, n_mol, vv, with_forces=False)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    t1 = float(np.median([timed(v[:1]) for _ in range(args.repeats)]))
    tn = float(np.median([timed(v) for _ in range(args.repeats)]))
    per_dir = (tn - t1) / (n_dir - 1)
    def categories(vv):
        lib.nb200_engine_set_timing(eng._h, 1)
        eng.run_hvp(zi, posf, mol_ptr, n_mol, vv, with_forces=False)
        ms = (ctypes.c_float * 16)()
        cnt = (ctypes.c_int32 * 16)()
        lib.nb200_engine_read_timings(eng._h, ms, cnt, 16)
        lib.nb200_engine_set_timing(eng._h, 0)
        return list(ms)

    ms = categories(v)
    tan_fwd = ms[5] / n_dir  # ms
    split = None
    if args.model == "schnet":
        ms1 = categories(v[:1])
        names = ("graph", "filter", "embed", "gemm", "node", "msg_fwd", "msg_bwd", "readout", "edge_grad_and_assembly")
        split = {k: (ms[i] - ms1[i]) / (n_dir - 1) for i, k in enumerate(names)}
        edges = eng.last_edges
        tan_fwd = split["msg_fwd"]  # the once-per-call primal message kernels cancel in the difference
        eng.run(zi, posf, mol_ptr, n_mol, True)  # sizes the inference engine's edge capacity for the finite-difference launches

    # finite differences: two batched force calls per shared direction
    h = args.fd_step
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cols = []
    for d in range(n_dir):  # enqueued without host synchronisation (the capacity was validated by the calls above)
        dv = v[d] * h
        _, fp, _ = eng.launch(zi, (posf + dv).contiguous(), mol_ptr, n_mol, True, e_cap=eng.e_cap)
        _, fm, _ = eng.launch(zi, (posf - dv).contiguous(), mol_ptr, n_mol, True, e_cap=eng.e_cap)
        cols.append(-(fp - fm) / (2 * h))
    torch.cuda.synchronize()
    t_fd = time.perf_counter() - t0
    hv_fd = torch.stack(cols)
    fd = vib.hessians_from_hvp(lambda vv: hv_fd[:vv.shape[0]], ptr)  # one chunk, same layout
    dev_rel = max(float((a - b).abs().max() / a.abs().max()) for a, b in zip(hs, fd))

    name, limit = card()
    rec = {
        "metric": "schnet_hessians" if args.model == "schnet" else "painn_hessians", "model": args.model, "batch": n_mol, "atoms": N, "n_max": n_max, "directions": n_dir,
        "hessians_per_s": n_mol / t_an, "directions_per_s": n_dir / t_an, "ms_per_batch": 1e3 * t_an, "ms_per_direction": 1e3 * t_an / n_dir,
        "ms_once_per_call": 1e3 * (t1 - per_dir), "ms_per_direction_marginal": 1e3 * per_dir,
        "ms_per_direction_tangent_forward": tan_fwd, "ms_per_direction_backward": 1e3 * per_dir - tan_fwd,
        "peak_mem_gb": peak / 1e9,
        "fd_ms_per_batch": 1e3 * t_fd, "fd_hessians_per_s": n_mol / t_fd, "fd_step_A": h, "fd_max_rel_dev": dev_rel,
        "analytic_speedup_vs_fd": t_fd / t_an, "max_asymmetry": hs.max_asymmetry,
        "card": name, "power_limit": limit,
    }
    if split is not None:
        rec["ms_per_direction_by_category"] = split
        rec["edges"] = edges
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
