#!/usr/bin/env python
"""Batched geometry optimisation (SURVEY.md section 8f-1; reference job `job_type: optimize`, config/schnet_optim.yaml): relax one
batch of synthetic molecules with PaiNN (config/model/painn.yaml) for a fixed number of L-BFGS steps through the public API
(`nabladft_b200.optimization.ASEBatchwiseLBFGS.run`), host Atoms in -> host Atoms out.  Reports optimiser steps/s for the whole
batch and molecule-steps/s; `--cpu` times the oracle loop (oracle L-BFGS + oracle PaiNN) on a few molecules for comparison.
Secondary benchmark (the driver's headline is bench.py); prints one JSON line.

`--model gemnet-oc` relaxes with GemNet-OC (reference job config/gemnet-oc_optim.yaml) at batch 32 and 256 and alternates two arms in one
process: the device loop (asynchronous forward sized by per-batch upper bounds, one host look per `check_every` steps) and the same loop with
the synchronous two-phase forward (`GemNetOCRunner.run`, which waits for the edge counts) at every step.  It also reports the host
synchronisations of a run, real count / bound of the five edge counts, the workspace size, and the card's name and power limit.
`--model dimenetplusplus` does the same for DimeNet++ (config/model/dimenetplusplus.yaml, seeded test weights), and also times one
asynchronous against one two-phase forward at the start geometry with CUDA events.

`--optimizer quasinewton` relaxes with `BatchwiseQuasiNewton` instead (PaiNN at `--batch`, or `--model dimenetplusplus` at batch 32): optimiser
steps/s, engine launches per optimiser step, `nb200_qn_step` against engine time per launch from CUDA events, host synchronisations, and a
host-driven arm (the oracle's numpy state machine on the same engine, one synchronisation per evaluation)."""
import argparse
from ctypes import c_int64
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def gemnet_main(args):
    import subprocess

    import numpy as np
    import torch
    import yaml
    from weights import golden_state_dict

    from nabladft_b200.gemnet_oc import C_NAMES, GemNetOC, GemNetOCEngine
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "gemnet-oc-b200.yaml")))["net"]
    cfg.pop("_target_")
    net = GemNetOC(**cfg).eval()
    sd = net.state_dict()
    new = golden_state_dict(sd, bias_std=0.02, weight_scale=0.5)
    for k in sd:
        if k.endswith("scale_factor"):
            sd[k] = torch.ones_like(sd[k])
        elif k in new:
            sd[k] = torch.as_tensor(np.asarray(new[k])).float().reshape(sd[k].shape)
    net.load_state_dict(sd, strict=True)

    class SyncEngine(GemNetOCEngine):
        """Comparison arm: the two-phase forward, which copies the edge counts to the host, at every step."""

        def launch(self, z, pos, mol_ptr, n_mol, e_cap=None):
            energy, forces = self.runner.run(z, pos, mol_ptr, n_mol, self._batch[1])
            return energy, forces, torch.zeros(8, dtype=torch.int32, device=pos.device)

    class SyncCalculator(PyGBatchwiseCalculator):
        def engine(self):
            if getattr(self, "_sync_engine", None) is None:
                self._sync_engine = SyncEngine(self.model, self.model._get_runner())
            return self._sync_engine

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        card, power = (v.strip() for v in q.stdout.strip().split(","))
    except Exception as exc:  # noqa: BLE001
        card, power = torch.cuda.get_device_name(0), f"unavailable ({exc})"
    out = {"metric": "L-BFGS steps/sec (GemNet-OC E+F + batched L-BFGS, B molecules per step)", "card": card, "power_limit": power, "steps": args.steps,
           "check_every": args.check_every, "memory": args.memory, "dtype": "f32 model / f64 positions", "data": "synthetic",
           "timing": "host wall clock around ASEBatchwiseLBFGS.run ending in a device synchronise; arms alternated, best of the repeats", "batches": []}
    for batch in args.batches:
        b = synth_batch(1, batch)
        ptr = b["mol_ptr"]
        atoms = [SimpleAtoms(b["pos"][ptr[m]:ptr[m + 1]], b["z"][ptr[m]:ptr[m + 1]]) for m in range(batch)]
        arms = {"device_loop": PyGBatchwiseCalculator(net, device=dev, energy_unit="Hartree", position_unit="Ang"),
                "sync_forward_per_step": SyncCalculator(net, device=dev, energy_unit="Hartree", position_unit="Ang")}
        opts = {k: ASEBatchwiseLBFGS(c, logfile=None, memory=args.memory, check_every=args.check_every) for k, c in arms.items()}
        times = {k: [] for k in arms}
        for k, o in opts.items():
            o.run(atoms, fmax=1e-9, steps=3)  # warm-up: allocations, module loads
        torch.cuda.synchronize()
        for _ in range(args.repeats):
            for k, o in opts.items():
                o.initialize()
                t0 = time.perf_counter()
                o.run(atoms, fmax=1e-9, steps=args.steps)
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
                if k == "device_loop":
                    last = arms[k].engine().runner._status.cpu().tolist()  # status words of the last launch: the counts at the final geometry
        eng = arms["device_loop"].engine()
        z, pos, mol_ptr, _ = arms["device_loop"].pack(atoms)
        _, _, st = eng.run(z, pos.float().contiguous(), mol_ptr, batch)  # start geometry: real counts against the bounds
        real = dict(zip(C_NAMES, [int(st[4]), int(st[0]), int(st[5]), int(st[6]), int(st[7])]))
        same = all(np.array_equal(arms["device_loop"].results[k], arms["sync_forward_per_step"].results[k]) for k in ("energy", "forces"))
        row = {"batch": batch, "atoms": int(ptr[-1]), "workspace_bytes": eng.runner.last_workspace_bytes,
               "count_over_bound": {k: round(real[k] / max(1, eng.bounds[k]), 4) for k in C_NAMES}, "bounds": eng.bounds,
               "count_over_bound_at_the_final_geometry": {k: round(v / max(1, eng.bounds[k]), 4) for k, v in
                                                          zip(C_NAMES, [last[4], last[0], last[5], last[6], last[7]])},
               "final_results_bitwise_equal_between_arms": bool(same)}
        for k, o in opts.items():
            dt = min(times[k])
            row[k] = {"steps_per_s": o.nsteps / dt, "molecule_steps_per_s": o.nsteps * batch / dt, "ms_per_step": dt / o.nsteps * 1e3,
                      "all_runs_s": [round(t, 4) for t in times[k]], "host_syncs_of_the_loop": o.host_syncs,
                      "host_syncs_inside_each_forward": 0 if k == "device_loop" else 5}
        out["batches"].append(row)
    print(json.dumps(out))


def card_and_power():
    import subprocess

    import torch

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = (v.strip() for v in q.stdout.strip().split(","))
    except Exception as exc:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), f"unavailable ({exc})"
    return name, power


def dimenet_model(dev, postprocessing=True):
    """DimeNet++ of config/model/dimenetplusplus-b200.yaml with the seeded test weights (tests/golden/make_golden_dimenet.py)."""
    import torch
    import yaml
    from make_golden_dimenet import load_test_weights

    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential

    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "dimenetplusplus-b200.yaml")))["net"]
    cfg.pop("_target_")
    cfg["do_postprocessing"] = postprocessing
    net = DimeNetPlusPlusPotential(**cfg).eval()
    load_test_weights(net, torch.float32)
    return net.to(dev)


def dimenet_sync_calculator():
    """A `PyGBatchwiseCalculator` whose engine runs the two-phase forward (`DimeNetRunner.run`, which waits for the edge and triplet counts)
    at every step: the comparison arm of the device loops."""
    import torch

    from nabladft_b200.dimenetplusplus import DimeNetEngine
    from nabladft_b200.optimization import PyGBatchwiseCalculator

    class SyncEngine(DimeNetEngine):
        def launch(self, z, pos, mol_ptr, n_mol, e_cap=None):
            energy, forces, _ = self.runner.run(z, pos, mol_ptr, n_mol)
            return energy, forces, torch.zeros(8, dtype=torch.int32, device=pos.device)

    class SyncCalculator(PyGBatchwiseCalculator):
        def engine(self):
            if getattr(self, "_sync_engine", None) is None:
                self._sync_engine = SyncEngine(self.model, self.model._get_runner())
            return self._sync_engine

    return SyncCalculator


def dimenet_forward_compare(calc, atoms, n=10):
    """One asynchronous forward against one two-phase forward at the start geometry (CUDA events around n calls each, alternated in three
    rounds, the best round), the counts against the bounds and both workspaces."""
    from ctypes import byref

    import torch

    eng = calc.engine()
    z, pos, mol_ptr, sizes = calc.pack(atoms)
    pos = pos.float().contiguous()
    _, _, st = eng.run(z, pos, mol_ptr, len(sizes))
    r = eng.runner
    r.run(z, pos, mol_ptr, len(sizes))
    counts = (c_int64 * 4)(r.last_counts["edges"], r.last_counts["triplets"], 0, 0)
    ws_exact = r._bytes("nb200_dimenet_workspace_bytes", byref(r._w), len(sizes), int(z.shape[0]), counts)
    arms = {"async": lambda: eng.launch(z, pos, mol_ptr, len(sizes)), "two_phase": lambda: r.run(z, pos, mol_ptr, len(sizes))}
    best = {k: float("inf") for k in arms}
    for _ in range(3):
        for k, fn in arms.items():
            fn()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(n):
                fn()
            b.record()
            b.synchronize()
            best[k] = min(best[k], a.elapsed_time(b) / n)
    return {"ms_per_async_forward": round(best["async"], 3), "ms_per_two_phase_forward": round(best["two_phase"], 3),
            "edges": int(st[0]), "triplet_slots": int(st[4]), "bounds": eng.bounds,
            "count_over_bound": {"edges": round(int(st[0]) / max(1, eng.bounds["edges"]), 4),
                                 "triplets": round(int(st[4]) / max(1, eng.bounds["triplets"]), 4)},
            "workspace_bytes_async": r.last_workspace_bytes, "workspace_bytes_two_phase": ws_exact}


def dimenet_main(args):
    import numpy as np
    import torch

    from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    net = dimenet_model(dev)
    name, power = card_and_power()
    out = {"metric": "L-BFGS steps/sec (DimeNet++ E+F + batched L-BFGS, B molecules per step)", "card": name, "power_limit": power, "steps": args.steps,
           "check_every": args.check_every, "memory": args.memory, "dtype": "f32 model / f64 positions", "data": "synthetic, seeded test weights",
           "timing": "host wall clock around ASEBatchwiseLBFGS.run ending in a device synchronise; arms alternated, best of the repeats", "batches": []}
    for batch in args.batches:
        b = synth_batch(1, batch)
        ptr = b["mol_ptr"]
        atoms = [SimpleAtoms(b["pos"][ptr[m]:ptr[m + 1]], b["z"][ptr[m]:ptr[m + 1]]) for m in range(batch)]
        arms = {"device_loop": PyGBatchwiseCalculator(net, device=dev, energy_unit="Hartree", position_unit="Ang"),
                "sync_forward_per_step": dimenet_sync_calculator()(net, device=dev, energy_unit="Hartree", position_unit="Ang")}
        row = {"batch": batch, "atoms": int(ptr[-1]), "start_geometry": dimenet_forward_compare(arms["device_loop"], atoms)}
        opts = {k: ASEBatchwiseLBFGS(c, logfile=None, memory=args.memory, check_every=args.check_every) for k, c in arms.items()}
        times = {k: [] for k in arms}
        for k, o in opts.items():
            o.run(atoms, fmax=1e-9, steps=3)  # warm-up
        torch.cuda.synchronize()
        for _ in range(args.repeats):
            for k, o in opts.items():
                o.initialize()
                t0 = time.perf_counter()
                o.run(atoms, fmax=1e-9, steps=args.steps)
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
                if k == "device_loop":
                    last = arms[k].engine().runner._status.cpu().tolist()
        eng = arms["device_loop"].engine()
        row["count_over_bound_at_the_final_geometry"] = {"edges": round(last[0] / max(1, eng.bounds["edges"]), 4),
                                                          "triplets": round(last[4] / max(1, eng.bounds["triplets"]), 4)}
        row["final_results_bitwise_equal_between_arms"] = bool(all(np.array_equal(arms["device_loop"].results[k], arms["sync_forward_per_step"].results[k])
                                                                   for k in ("energy", "forces")))
        for k, o in opts.items():
            dt = min(times[k])
            row[k] = {"steps_per_s": o.nsteps / dt, "molecule_steps_per_s": o.nsteps * batch / dt, "ms_per_step": dt / o.nsteps * 1e3,
                      "all_runs_s": [round(t, 4) for t in times[k]], "host_syncs_of_the_loop": o.host_syncs,
                      "host_syncs_inside_each_forward": 0 if k == "device_loop" else 1}
        out["batches"].append(row)
    print(json.dumps(out))


def qn_main(args):
    """`--optimizer quasinewton`: BatchwiseQuasiNewton (ASE's QuasiNewton per molecule) with PaiNN at batch `--batch` or DimeNet++ at batch 32."""
    import numpy as np
    import torch

    from nabladft_b200.optimization import BatchwiseQuasiNewton, PyGBatchwiseCalculator, SimpleAtoms, SpkBatchwiseCalculator, convert_units
    from nabladft_b200.synth import synth_batch
    from oracle.quasinewton import BatchQuasiNewton

    dev = torch.device("cuda:0")
    if args.model == "dimenetplusplus":
        batch, calc = 32, PyGBatchwiseCalculator(dimenet_model(dev), device=dev, energy_unit="Hartree", position_unit="Ang")
    else:
        from bench import build_model

        batch, calc = args.batch, SpkBatchwiseCalculator(build_model("painn", dev), device=dev, energy_unit="Hartree", position_unit="Ang")
    name, power = card_and_power()
    b = synth_batch(1, batch)
    ptr = b["mol_ptr"]
    atoms = [SimpleAtoms(b["pos"][ptr[m]:ptr[m + 1]], b["z"][ptr[m]:ptr[m + 1]]) for m in range(batch)]
    opt = BatchwiseQuasiNewton(calc, check_every=args.check_every)
    opt.run(atoms, fmax=1e-9, steps=3)  # warm-up
    torch.cuda.synchronize()
    opt.initialize()
    t0 = time.perf_counter()
    opt.run(atoms, fmax=1e-9, steps=args.steps)  # fmax unreachable: every molecule takes `steps` BFGS steps
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    mol_steps = int(opt.nsteps.sum())
    out = {"metric": f"QuasiNewton steps/sec ({args.model} E+F + batched BFGSLineSearch, B molecules)", "card": name, "power_limit": power,
           "model": args.model, "batch": batch, "atoms": int(ptr[-1]), "steps": args.steps, "check_every": args.check_every,
           "value": float(opt.nsteps.mean()) / dt, "molecule_steps_per_s": mol_steps / dt, "ms_per_launch": dt / opt.launches * 1e3,
           "engine_launches": opt.launches, "engine_launches_used": opt.launches_used,
           "launches_per_optimiser_step": opt.launches_used / float(opt.nsteps.max()),
           "force_calls_per_step_mean": float(opt.force_calls.sum()) / mol_steps, "host_syncs": opt.host_syncs,
           "hessian_bytes": int(((3 * np.diff(ptr)) ** 2).sum() * 8),
           "timing": "host wall clock around BatchwiseQuasiNewton.run ending in a device synchronise (includes packing, H2D, final D2H)"}

    # per-launch device time of nb200_qn_step against the engine launch: CUDA events around each call, in a separate run
    eng = calc.engine()
    lib, times = opt.lib, {"qn": [], "engine": []}

    class Timed:
        def __init__(self, fn, key):
            self.fn, self.key = fn, key

        def __call__(self, *a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = self.fn(*a, **k)
            e1.record()
            times[self.key].append((e0, e1))
            return r

    class TimedLib:
        def __getattr__(self, n):
            return Timed(getattr(lib, n), "qn") if n == "nb200_qn_step" else getattr(lib, n)

    launch = eng.launch
    eng.launch = Timed(launch, "engine")
    opt.lib = TimedLib()
    try:
        opt.initialize()
        opt.run(atoms, fmax=1e-9, steps=min(args.steps, 10))
        torch.cuda.synchronize()
    finally:
        eng.launch, opt.lib = launch, lib
    ms = {k: float(np.mean([a.elapsed_time(c) for a, c in v])) for k, v in times.items()}
    out["qn_step_ms_per_launch"] = round(ms["qn"], 4)
    out["engine_ms_per_launch"] = round(ms["engine"], 4)
    out["qn_step_share_of_engine"] = round(ms["qn"] / ms["engine"], 4)

    # host-driven arm: the oracle's numpy state machine stepping the same engine, one synchronisation per evaluation (the reference's cost
    # model, batched)
    z, pos, mol_ptr, sizes = calc.pack(atoms)
    e_scale = calc.energy_conversion * convert_units("Hartree", "eV")
    f_scale = np.float32(e_scale / calc.position_conversion)

    def ff(p):
        e, f, _ = eng.launch(z, torch.from_numpy(np.asarray(p, dtype=np.float32)).to(dev), mol_ptr, batch, e_cap=eng.e_cap)
        return e.cpu().numpy().astype(np.float64) * e_scale, f.cpu().numpy() * f_scale

    host = BatchQuasiNewton(ff, sizes)
    t0 = time.perf_counter()
    host.run(pos.cpu().numpy(), fmax=1e-9, steps=args.host_steps)
    dth = time.perf_counter() - t0
    out["host_driven"] = {"steps": args.host_steps, "value": float(host.nsteps.mean()) / dth, "molecule_steps_per_s": float(host.nsteps.sum()) / dth,
                          "ms_per_launch": dth / host.n_calls * 1e3, "host_syncs": host.n_calls,
                          "kind": "oracle/quasinewton.py numpy state machine + the same engine, a device synchronisation per evaluation"}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["painn", "gemnet-oc", "dimenetplusplus"], default="painn")
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 256], help="gemnet-oc, dimenetplusplus: batch sizes to run")
    ap.add_argument("--repeats", type=int, default=2, help="gemnet-oc, dimenetplusplus: timed runs of each arm (alternated)")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--memory", type=int, default=100)
    ap.add_argument("--check-every", type=int, default=10)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--cpu-mols", type=int, default=8)
    ap.add_argument("--cpu-steps", type=int, default=3)
    ap.add_argument("--optimizer", choices=["lbfgs", "quasinewton"], default="lbfgs")
    ap.add_argument("--host-steps", type=int, default=5, help="quasinewton: BFGS steps of the host-driven arm")
    args = ap.parse_args()
    if args.optimizer == "quasinewton":
        if args.model == "gemnet-oc":
            raise SystemExit("--optimizer quasinewton: --model painn or dimenetplusplus")
        return qn_main(args)
    if args.model == "gemnet-oc":
        return gemnet_main(args)
    if args.model == "dimenetplusplus":
        return dimenet_main(args)
    import numpy as np
    import torch

    from bench import build_model
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, SimpleAtoms, SpkBatchwiseCalculator
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    model = build_model("painn", dev)
    b = synth_batch(1, args.batch)
    ptr = b["mol_ptr"]
    atoms = [SimpleAtoms(b["pos"][ptr[m]:ptr[m + 1]], b["z"][ptr[m]:ptr[m + 1]]) for m in range(args.batch)]
    calc = SpkBatchwiseCalculator(model, device=dev, energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None, memory=args.memory, check_every=args.check_every)
    opt.run(atoms, fmax=1e-9, steps=5)  # warm-up (allocations, cuBLAS handles)
    torch.cuda.synchronize()
    opt.initialize()
    t0 = time.perf_counter()
    opt.run(atoms, fmax=1e-9, steps=args.steps)  # fmax unreachable: exactly `steps` E+F + L-BFGS steps, like the reference would run
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    f = calc.results["forces"]
    out = {"metric": "L-BFGS steps/sec (PaiNN E+F + batched L-BFGS, B molecules per step)", "value": opt.nsteps / dt,
           "molecule_steps_per_s": opt.nsteps * args.batch / dt, "ms_per_step": dt / opt.nsteps * 1e3, "batch": args.batch, "steps": opt.nsteps,
           "memory": args.memory, "check_every": args.check_every, "atoms": int(ptr[-1]), "n_normalizations": opt.n_normalizations,
           "timing": "host wall clock around ASEBatchwiseLBFGS.run (includes packing Atoms, H2D, final D2H)",
           "dtype": "f32 model / f64 positions", "data": "synthetic"}
    if args.cpu:
        from bench import build_oracle, oracle_pass
        from oracle.lbfgs import BatchLBFGS

        ref = build_oracle("painn", model)
        nm = args.cpu_mols
        best = None
        for nt in (8, 16, 32):
            torch.set_num_threads(min(nt, os.cpu_count()))

            def ff(pos):
                bb = dict(b)
                bb["pos"] = np.concatenate([np.asarray(pos, dtype=np.float32), b["pos"][ptr[nm]:]])
                e, fo = oracle_pass("painn", ref, bb, nm)
                return e.detach().numpy(), fo.detach().numpy()

            o = BatchLBFGS(ff, np.diff(ptr[:nm + 1]), memory=args.memory)
            t0 = time.perf_counter()
            o.run(b["pos"][:ptr[nm]].astype(np.float64), fmax=1e-9, steps=args.cpu_steps, record=False)
            d = time.perf_counter() - t0
            rate = o.nsteps * nm / d
            if best is None or rate > best[0]:
                best = (rate, nt)
        out["cpu_baseline"] = {"value": best[0], "unit": "molecule-steps/s", "cores": best[1], "kind": "port",
                               "sample": f"{args.cpu_steps} steps on the first {nm} molecules: oracle L-BFGS (reference-pinned) + oracle PaiNN, neighbour list per step"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
