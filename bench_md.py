#!/usr/bin/env python
"""Batched molecular dynamics (the reference's `init_md` / `run_md`, nablaDFT/optimization/pyg_ase_interface.py): spk PaiNN
(config/model/painn.yaml, 6 layers) on the config-2 batch of 256 synthetic molecules, through the public API
(`nabladft_b200.md.BatchwiseMD`), NVE velocity Verlet and Langevin at 300 K.  Reports MD steps/s, molecule-steps/s and simulated ps/day
per thermostat, the integrator's and the engine's kernel time per step (torch.profiler, separate run), host synchronisations per chunk and, with
`--batch1`, the same at one molecule.  `--host-loop` times the shape of the reference's ASE loop on the same engine: per step a D2H copy of
the forces, a numpy velocity-Verlet step and an H2D copy of the positions.  Secondary benchmark (the headline is bench.py); prints one
JSON line with the card's name and power limit."""
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


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit_and_max_sm_clock"] = "unavailable"
    return out


def event_ms(fn, n):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def run_md(calc, atoms, bath, steps, warmup, check_every):
    import torch

    from nabladft_b200.md import BatchwiseMD, FS

    md = BatchwiseMD(calc, atoms, seed=0, check_every=check_every)
    md.init_md("bench", time_step=0.5, temp_init=300, temp_bath=bath, interval=10 ** 9)
    md.run_md(warmup)
    torch.cuda.synchronize()
    syncs0 = md.host_syncs
    t0 = time.perf_counter()
    md.run_md(steps)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    chunks = -(-steps // check_every)
    rate = steps / dt
    out = {"steps_per_s": rate, "molecule_steps_per_s": rate * len(atoms), "ms_per_step": 1e3 / rate,
           "simulated_ps_per_day": rate * 86400 * md.dt / (1000 * FS), "host_syncs_per_chunk": (md.host_syncs - syncs0) / chunks,
           "replays": md.replays}
    out.update(device_time_per_step(md, min(steps, 100)))
    out.update(host_time_per_step(md, min(steps, 100)))
    return out


def host_time_per_step(md, steps):
    """Host time per MD step spent inside the engine's launch call and the integrator's launch call (the Python and C enqueue work), over
    `steps` more steps; when it approaches the device time per step, the loop is bound by the host."""
    import torch

    eng, acc = md._eng, {"engine": 0.0, "integrator": 0.0}

    def timed(fn, key):
        def call(*a, **kw):
            t = time.perf_counter()
            r = fn(*a, **kw)
            acc[key] += time.perf_counter() - t
            return r
        return call

    eng.launch, md._launch = timed(eng.launch, "engine"), timed(md._launch, "integrator")
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        md.run_md(steps)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        del eng.launch, md._launch  # back to the class methods
    return {"host_engine_launch_ms_per_step": 1e3 * acc["engine"] / steps, "host_integrator_launch_ms_per_step": 1e3 * acc["integrator"] / steps,
            "host_timed_wall_ms_per_step": 1e3 * wall / steps}


def device_time_per_step(md, steps):
    """Kernel time per MD step from torch.profiler (CUDA activities) over `steps` more steps of run_md: the integrator kernel
    (k_md_step), everything the engine launches, copies / memsets, and the device-idle time left in the profiled wall time.  The profiled run
    is separate from the timed one, since tracing slows the host."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        md.run_md(steps)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    integ = engine = copies = 0.0
    n_integ = 0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        if "k_md_step" in ev.name:
            integ += us
            n_integ += 1
        elif "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            copies += us
        else:
            engine += us
    ms = 1e-3 / steps
    busy = (integ + engine + copies) * ms
    return {"profiled_wall_ms_per_step": 1e3 * wall / steps, "integrator_kernel_ms_per_step": integ * ms, "integrator_launches": n_integ,
            "engine_kernels_ms_per_step": engine * ms, "copies_memsets_ms_per_step": copies * ms, "device_busy_ms_per_step": busy,
            "integrator_share_of_engine": integ / max(engine, 1e-9)}


def host_loop(calc, atoms, steps, warmup):
    """The reference's loop shape on this engine: forces D2H, numpy velocity Verlet, positions H2D, every step."""
    import numpy as np
    import torch

    from nabladft_b200.md import FS
    from nabladft_b200.optimization import convert_units
    from nabladft_b200.vibrations import masses_of

    z, pos, mol_ptr, sizes = calc.pack(atoms)
    eng = calc.engine()
    m = masses_of(z).numpy()[:, None]
    es = calc.energy_conversion * convert_units("Hartree", "eV") / calc.position_conversion
    x = pos.cpu().numpy()
    p = np.zeros_like(x)
    dt = 0.5 * FS
    _, f, st = eng.run(z, pos.float().contiguous(), mol_ptr, len(sizes))
    eng.e_cap = max(eng.e_cap, int(1.5 * int(st[0])) + 1024)
    fh = f.cpu().numpy().astype(np.float64) * es

    def one():
        nonlocal fh, p, x
        p = p + 0.5 * dt * fh
        x = x + dt * p / m
        _, f, _ = eng.launch(z, torch.from_numpy(x.astype(np.float32)).to(z.device), mol_ptr, len(sizes), e_cap=eng.e_cap)
        fh = f.cpu().numpy().astype(np.float64) * es
        p = p + 0.5 * dt * fh

    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    dt_wall = time.perf_counter() - t0
    eng.raise_on_status(eng._status.cpu())
    rate = steps / dt_wall
    return {"steps_per_s": rate, "molecule_steps_per_s": rate * len(atoms), "ms_per_step": 1e3 / rate, "host_syncs_per_step": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--check-every", type=int, default=50)
    ap.add_argument("--host-loop", action="store_true")
    ap.add_argument("--batch1", action="store_true", help="also time one molecule (the first of the batch)")
    args = ap.parse_args()
    import numpy as np
    import torch

    from bench import build_model
    from nabladft_b200.optimization import SimpleAtoms, SpkBatchwiseCalculator
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda:0")
    model = build_model("painn", dev)
    b = synth_batch(1, args.batch)
    p = b["mol_ptr"]
    atoms = [SimpleAtoms(b["pos"][p[i]:p[i + 1]].astype(np.float64), b["z"][p[i]:p[i + 1]]) for i in range(args.batch)]
    calc = SpkBatchwiseCalculator(model, device=dev, energy_unit="Hartree", position_unit="Ang")
    out = {"metric": "MD steps/sec (spk PaiNN E+F + one integrator launch, B molecules per step)", "batch": args.batch, "atoms": int(p[-1]),
           "steps": args.steps, "check_every": args.check_every, "time_step_fs": 0.5, "card": card(),
           "timing": "host wall clock around BatchwiseMD.run_md; kernel times from torch.profiler in a separate profiled run", "data": "synthetic"}
    out["nve"] = run_md(calc, atoms, None, args.steps, args.warmup, args.check_every)
    out["langevin_300K"] = run_md(calc, atoms, 300.0, args.steps, args.warmup, args.check_every)
    out["value"] = out["nve"]["steps_per_s"]
    if args.batch1:
        out["batch1_nve"] = run_md(calc, atoms[:1], None, args.steps, args.warmup, args.check_every)
    if args.host_loop:
        out["host_loop_nve"] = host_loop(calc, atoms, max(20, args.steps // 4), 5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
