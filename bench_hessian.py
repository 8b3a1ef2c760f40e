"""Throughput of exact Hessians (nb200_painn_hvp, nb200_schnet_hvp, nb200_dimenet_hvp, nb200_gemnet_oc_jvp) on the config-2 batch: 256 synthetic conformations
(synth.py), one JSON line.

    python bench_hessian.py [--model painn|painn-oc|schnet|dimenetplusplus|gemnet-oc] [--max-dir D] [--repeats R] [--batch B]

Reports Hessians / s and HVP directions / s for the whole batch (3 n_max shared directions, chunks of --max-dir), peak device memory, ms per
direction split into the tangent forward and the backward (CUDA events around the engine's launch categories), and the same Hessians by
batched central finite differences of the inference engine (nb200_painn_energy_forces, nb200_schnet_energy_forces; two force calls per
direction, step 1e-3 A) with their deviation from the analytic ones.  For SchNet the per-direction split is also given per launch category
(marginal ms per direction of each, from the engine's CUDA-event timing of an n_dir call minus a one-direction call).  Card name and power
limit come from the same run.  Writes nothing into the tree.

--model dimenetplusplus (config/model/dimenetplusplus.yaml sizes, the tests' weights, synth_batch(0, B) as bench_dimenet.py): one analytic
pass over the 3 n_max shared directions (its cost per direction is about that of a training gradient call, so it is not repeated), the
per-direction and once-per-call costs from one- and --probe-direction calls, and the same Hessians by central differences with two
nb200_dimenet_energy_forces calls per direction.

--model gemnet-oc (config/model/gemnet-oc.yaml sizes, the tests' weights, synth_batch(0, B), B = 32 unless --batch is given): the same, with
force-Jacobian products (the direct forces' Jacobian, symmetrised as ASE does) against two two-phase nb200_gemnet_oc_energy_forces calls per
direction, plus the workspace of the call at B and the largest synth_batch(0, B') whose workspace fits the card's free memory (bisection on
the size query, graph phase only).
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
    ap.add_argument("--model", default="painn", choices=["painn", "painn-oc", "schnet", "dimenetplusplus", "gemnet-oc"])
    ap.add_argument("--max-dir", type=int, default=None)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fd-step", type=float, default=1e-3)
    ap.add_argument("--batch", type=int, default=None,
                    help="molecules (dimenetplusplus: 256, gemnet-oc: 32 by default; the other models use the config-2 batch)")
    ap.add_argument("--probe-directions", type=int, default=8,
                    help="directions of the call the per-direction cost is taken from (dimenetplusplus, gemnet-oc)")
    args = ap.parse_args()
    if args.model == "dimenetplusplus":
        args.batch = args.batch or 256
        return dimenet_main(args)
    if args.model == "gemnet-oc":
        args.batch = args.batch or 32
        return gemnet_main(args)

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
    eng, zi, posf, mol_ptr, n_mol = model.engine_inputs(batch)
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


def dimenet_main(args):
    import os
    import sys

    import torch
    import yaml

    root = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(root, "tests", "golden"))
    from make_golden_dimenet import load_test_weights

    from nabladft_b200 import vibrations as vib
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from nabladft_b200.synth import synth_batch
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    dev = torch.device("cuda:0")
    cfg = yaml.safe_load(open(os.path.join(root, "config", "model", "dimenetplusplus-b200.yaml")))["net"]
    cfg.pop("_target_")
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(**cfg).double().eval())
    model = DimeNetPlusPlusPotential(**cfg).eval()
    model.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    model = model.to(dev)

    class D:
        pass

    b = synth_batch(0, args.batch)
    batch = D()
    batch.z = torch.from_numpy(b["z"]).long().to(dev)
    batch.pos = torch.from_numpy(b["pos"]).to(dev)
    batch.batch = torch.from_numpy(b["batch"]).to(dev)
    runner, zi, posf, mol_ptr, n_mol = model.engine_inputs(batch)
    ptr = mol_ptr.cpu().tolist()
    n_max = max(q - p for p, q in zip(ptr[:-1], ptr[1:]))
    n_dir = 3 * n_max
    v = vib.shared_directions(ptr, 0, n_dir, dev)
    k = max(2, min(args.probe_directions, n_dir))

    def timed(vv):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        runner.run_hvp(zi, posf, mol_ptr, n_mol, vv, with_forces=False)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    timed(v[:1])  # workspace allocation
    torch.cuda.reset_peak_memory_stats(dev)
    t1 = timed(v[:1])
    tk = timed(v[:k])
    per_dir = (tk - t1) / (k - 1)
    # analytic Hessians of the whole batch, once
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hs = vib.hessians(model, batch, args.max_dir)
    torch.cuda.synchronize()
    t_an = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(dev)
    counts = dict(runner.last_counts)
    ws = runner.lib.nb200_dimenet_hvp_workspace_bytes(ctypes.byref(runner._w), n_mol, zi.numel(),
                                                      (ctypes.c_int64 * 4)(counts["edges"], counts["triplets"], 0, 0))

    # finite differences: two energy-and-forces calls per shared direction
    h = args.fd_step
    runner.run(zi, posf, mol_ptr, n_mol)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cols = []
    for d in range(n_dir):
        dv = v[d] * h
        fp = runner.run(zi, (posf + dv).contiguous(), mol_ptr, n_mol)[1]
        fm = runner.run(zi, (posf - dv).contiguous(), mol_ptr, n_mol)[1]
        cols.append(-(fp - fm) / (2 * h))
    torch.cuda.synchronize()
    t_fd = time.perf_counter() - t0
    hv_fd = torch.stack(cols)
    fd = vib.hessians_from_hvp(lambda vv: hv_fd[:vv.shape[0]], ptr)
    devs = [float((a - c).abs().max() / a.abs().max()) for a, c in zip(hs, fd)]
    # a molecule of more than max_neighbors + 1 atoms can have truncated candidate lists (radius_graph keeps the first K + 1 in index
    # order); a step that moves a pair across the cutoff then changes the edge set and the forces jump, so only the others are smooth
    kcap = model.max_num_neighbors + 1
    smooth = [d for d, p0, p1 in zip(devs, ptr[:-1], ptr[1:]) if p1 - p0 <= kcap]

    name, limit = card()
    print(json.dumps({
        "metric": "dimenet_hessians", "model": args.model, "batch": n_mol, "atoms": int(zi.numel()), "edges": counts["edges"],
        "triplets": counts["triplets"], "n_max": n_max, "directions": n_dir,
        "hessians_per_s": n_mol / t_an, "directions_per_s": n_dir / t_an, "ms_per_batch": 1e3 * t_an, "ms_per_direction": 1e3 * t_an / n_dir,
        "ms_once_per_call": 1e3 * (t1 - per_dir), "ms_per_direction_marginal": 1e3 * per_dir, "probe_directions": k,
        "peak_mem_gb": peak / 1e9, "hvp_workspace_gb": ws / 1e9,
        "fd_ms_per_batch": 1e3 * t_fd, "fd_ms_per_direction": 1e3 * t_fd / n_dir, "fd_hessians_per_s": n_mol / t_fd, "fd_step_A": h,
        "fd_max_rel_dev": max(devs), "fd_median_rel_dev": float(np.median(devs)),
        "fd_max_rel_dev_untruncated": max(smooth) if smooth else None, "untruncated_molecules": len(smooth), "analytic_speedup_vs_fd": t_fd / t_an, "max_asymmetry": hs.max_asymmetry,
        "card": name, "power_limit": limit,
    }))


def gemnet_main(args):
    import os
    import sys

    import torch

    root = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(root, "tests"))
    sys.path.insert(0, os.path.join(root, "tests", "golden"))
    from test_gemnet_emu import _models

    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    model = _models(True)[0].to(dev).eval()

    class D:
        pass

    def make_batch(n_mol):
        b = synth_batch(0, n_mol)
        d = D()
        d.z = torch.from_numpy(b["z"]).long().to(dev)
        d.pos = torch.from_numpy(b["pos"]).to(dev)
        d.batch = torch.from_numpy(b["batch"]).to(dev)
        return d

    batch = make_batch(args.batch)
    runner, zi, posf, mol_ptr, n_mol = model.engine_inputs(batch)
    ptr = mol_ptr.cpu().tolist()
    n_max = max(q - p for p, q in zip(ptr[:-1], ptr[1:]))
    n_dir = 3 * n_max
    v = vib.shared_directions(ptr, 0, n_dir, dev)
    k = max(2, min(args.probe_directions, n_dir))

    def timed(vv):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        runner.run_hvp(zi, posf, mol_ptr, n_mol, vv, with_forces=False)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    timed(v[:1])  # workspace allocation
    torch.cuda.reset_peak_memory_stats(dev)
    t1 = timed(v[:1])
    tk = timed(v[:k])
    per_dir = (tk - t1) / (k - 1)
    ws = runner.last_workspace_bytes
    counts = dict(runner.last_counts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hs = vib.hessians(model, batch, args.max_dir)
    torch.cuda.synchronize()
    t_an = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(dev)

    # central differences of the direct forces: two two-phase inference calls per shared direction
    h = args.fd_step
    max_atoms = n_max
    runner.run(zi, posf, mol_ptr, n_mol, max_atoms)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cols = []
    for d in range(n_dir):
        dv = v[d] * h
        fp = runner.run(zi, (posf + dv).contiguous(), mol_ptr, n_mol, max_atoms)[1]
        fm = runner.run(zi, (posf - dv).contiguous(), mol_ptr, n_mol, max_atoms)[1]
        cols.append(-(fp - fm) / (2 * h))
    torch.cuda.synchronize()
    t_fd = time.perf_counter() - t0
    hv_fd = torch.stack(cols)
    fd = vib.hessians_from_hvp(lambda vv: hv_fd[:vv.shape[0]], ptr)
    devs = [float((a - c).abs().max() / a.abs().max()) for a, c in zip(hs, fd)]

    # the largest synth_batch(0, B) whose jvp workspace fits what the card has free now (graph phase and size query only, no model pass)
    # drop the runner's buffers first: a small one carved from the cached jvp segment would pin that whole segment through empty_cache()
    runner.release_hvp_workspace()
    runner._ws = runner._graph_buf = None
    del hv_fd, cols
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info(dev)[0] - (1 << 30)  # 1 GiB for v, jv, the graph buffer and the allocator

    def ws_bytes(n_mol_):
        d = make_batch(n_mol_)
        _, z_, p_, mp_, nm_ = model.engine_inputs(d)
        pt = mp_.cpu()
        _, cnt = runner._graph(p_, mp_, nm_, int((pt[1:] - pt[:-1]).max()))
        return runner._bytes("nb200_gemnet_oc_jvp_workspace_bytes", ctypes.byref(runner._w), nm_, int(z_.numel()), cnt)

    lo, hi = args.batch, 2 * args.batch
    if ws_bytes(lo) > free:
        lo, hi = 0, lo
    else:
        while ws_bytes(hi) <= free:
            lo, hi = hi, 2 * hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ws_bytes(mid) <= free else (lo, mid)

    name, limit = card()
    print(json.dumps({
        "metric": "gemnet_oc_hessians", "model": args.model, "batch": n_mol, "atoms": int(zi.numel()), "counts": counts, "n_max": n_max,
        "directions": n_dir, "hessians_per_s": n_mol / t_an, "ms_per_batch": 1e3 * t_an, "ms_per_direction": 1e3 * t_an / n_dir,
        "ms_once_per_call": 1e3 * (t1 - per_dir), "ms_per_direction_marginal": 1e3 * per_dir, "probe_directions": k,
        "peak_mem_gb": peak / 1e9, "jvp_workspace_gb": ws / 1e9, "largest_batch_fitting": lo, "free_gb_for_workspace": free / 1e9,
        "fd_ms_per_batch": 1e3 * t_fd, "fd_ms_per_direction": 1e3 * t_fd / n_dir, "fd_step_A": h,
        "fd_max_rel_dev": max(devs), "fd_median_rel_dev": float(np.median(devs)), "analytic_speedup_vs_fd": t_fd / t_an,
        "max_asymmetry": hs.max_asymmetry, "card": name, "power_limit": limit,
    }))


if __name__ == "__main__":
    main()
