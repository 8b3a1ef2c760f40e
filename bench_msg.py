#!/usr/bin/env python
"""bench_msg.py -- time and HBM throughput of the PaiNN message kernels (painn_msg.cu) at the shape bench.py runs.

Builds the engine and the four seeded 256-molecule batches exactly as bench.py does, then
  * times every message launch of the E+F call with CUDA events (the engine's timing scopes, one per launch) over `--reps` calls
    after warm-up, and reports per kernel: ms per launch, the unique bytes a launch must move across HBM, and their rate;
  * probes whether the second read of a pair's filter record is served by L2: the backward alone on the graph of batch 0, timed
      pairs     -- one [W | dW/dd] record of 6F per undirected pair, edge e reads row min(e, rev[e]) (the E+F path);
      pairs_2x  -- the same pair rows in two arrays W, dW of 3F (two bulk copies per edge, the layout training uses);
      edges_2x  -- one row per directed edge in two arrays (`rev` = NULL, the public nb200_painn_msg_bwd): twice the record bytes, no sharing.
    pairs_2x vs edges_2x isolates the sharing; pairs vs pairs_2x the copy count;
  * measures the L2 -> SM gather ceiling at the kernels' access pattern: each kernel alone on batch 0 against a load-only kernel that
    reads the same rows per edge (nb200_msg_gather_probe).
Prints one JSON line.  `--lib` times another build of libnabla_b200.so (A/B comparisons in one run).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

F, L = 128, 6
HBM_PEAK_TBS = 3.35  # H100 SXM data sheet


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["sm_max_mhz"] = float(q[0]), float(q[1])
    except Exception as exc:  # the name still identifies the card
        out["power_limit_w"] = f"unavailable ({exc})"
    return out


def unique_bytes(n_atoms, n_edges):
    """Bytes one launch must move across HBM at least once: each pair's record once (6F fp32 for the backward, its first 3F for the forward),
    the per-atom rows read and written, the per-edge metadata (col, rev, geom) and, in the backward, the egrad reductions."""
    pairs = n_edges / 2
    meta = n_edges * (4 + 4 + 16)
    fwd = pairs * 3 * F * 4 + n_atoms * (3 * F + 3 * F + F + F + 3 * F) * 4 + meta  # xh, mu, q read; q_out, mu_out written
    bwd = pairs * 6 * F * 4 + n_atoms * (3 * F + 3 * F + F + 3 * F + 3 * F + 3 * F) * 4 + meta + n_edges * 16  # xh mu g_q g_mu; g_xh g_mu_in; egrad
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50, help="timed E+F calls (and timed launches of each probe)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", default=None, help="path of the libnabla_b200.so to time (default: the one in the tree)")
    ap.add_argument("--tag", default=None, help="label copied into the output line")
    args = ap.parse_args()
    reps = max(args.reps, 50)

    import torch

    from nabladft_b200 import _lib

    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    lib = _lib.load()
    from bench import B_PER_GPU, N_POOL, build_model
    from nabladft_b200.synth import synth_batch

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = build_model("painn", dev)
    eng = model.engine(True)
    pool_host = [synth_batch(1 + k, B_PER_GPU) for k in range(N_POOL)]
    pool = [dict(z=torch.from_numpy(b["z"]).to(dev), pos=torch.from_numpy(b["pos"]).to(dev), mol_ptr=torch.from_numpy(b["mol_ptr"]).to(dev))
            for b in pool_host]
    n_atoms = [int(b["z"].shape[0]) for b in pool_host]
    eng.e_cap = max(n_atoms) * 32

    def step(k):
        d = pool[k % N_POOL]
        return eng.launch(d["z"], d["pos"], d["mol_ptr"], B_PER_GPU, with_forces=True)

    for k in range(max(args.warmup, N_POOL)):
        _, _, st = step(k)
        sth = st.cpu()
        if int(sth[1]) == -4:
            eng.e_cap = int(int(sth[0]) * 1.1) + 1024
            _, _, st = step(k)
            sth = st.cpu()
        eng.raise_on_status(sth)
    stats = []
    for k in range(N_POOL):
        _, _, st = step(k)
        sth = st.cpu().tolist()
        stats.append(sth)
    torch.cuda.synchronize()

    # ---- every message launch of `reps` E+F calls, cycling the pool as bench.py does
    import ctypes

    _lib.check(lib.nb200_engine_set_timing(eng._h, 1), "set_timing")
    for k in range(reps):
        step(k)
    torch.cuda.synchronize()
    ms_cat, n_cat = (ctypes.c_float * 16)(), (ctypes.c_int32 * 16)()
    _lib.check(lib.nb200_engine_read_timings(eng._h, ms_cat, n_cat, 16), "read_timings")
    lib.nb200_engine_set_timing(eng._h, 0)
    from bench import CATS

    N_avg = sum(n_atoms[k % N_POOL] for k in range(reps)) / reps
    E_avg = sum(stats[k % N_POOL][0] for k in range(reps)) / reps
    b_fwd, b_bwd = unique_bytes(N_avg, E_avg)
    kernels = {}
    for name, cat, nbytes in (("k_painn_msg_fwd", "msg_fwd", b_fwd), ("k_painn_msg_bwd", "msg_bwd", b_bwd)):
        c = CATS.index(cat)
        ms = ms_cat[c] / n_cat[c]
        kernels[name] = {"ms_per_launch": ms, "launches": int(n_cat[c]), "unique_bytes_per_launch": nbytes,
                         "tb_per_s": nbytes / (ms * 1e-3) / 1e12, "frac_of_hbm_peak": nbytes / (ms * 1e-3) / 1e12 / HBM_PEAK_TBS}

    # ---- L2 probe: the backward alone on batch 0's graph, three filter row layouts
    d = pool[0]
    N, B = n_atoms[0], B_PER_GPU
    e_cap = eng.e_cap
    row_ptr = torch.zeros(N + 1, dtype=torch.int32, device=dev)
    col = torch.zeros(e_cap, dtype=torch.int32, device=dev)
    rev = torch.zeros(e_cap, dtype=torch.int32, device=dev)
    geom = torch.zeros(e_cap, 4, dtype=torch.float32, device=dev)
    deg = torch.zeros(N, dtype=torch.int32, device=dev)
    status = torch.zeros(4, dtype=torch.int32, device=dev)
    _lib.check(lib.nb200_neighbor_build(_lib.ptr(d["pos"]), _lib.ptr(d["mol_ptr"]), B, N, 5.0, 100, e_cap, _lib.ptr(row_ptr), _lib.ptr(col),
                                        _lib.ptr(rev), _lib.ptr(geom), _lib.ptr(deg), _lib.ptr(status), _lib.current_stream()), "neighbor_build")
    torch.cuda.synchronize()
    E = int(status[0])
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *shape: torch.randn(*shape, device=dev, generator=g) * 0.1  # noqa: E731
    xh, bias, mu, gq, gmu = rnd(N, 3 * F), rnd(3 * F), rnd(N, 3 * F), rnd(N, F), rnd(N, 3 * F)
    g_xh, g_mu_in, egrad = torch.empty(N, 3 * F, device=dev), torch.empty(N, 3 * F, device=dev), torch.zeros(e_cap, 4, device=dev)
    rec = rnd(E, 6 * F)                                   # pairs: [W | dW] per row, rows min(e, rev[e]) used
    W2, dW2 = rec[:, :3 * F].contiguous(), rec[:, 3 * F:].contiguous()  # pairs_2x / edges_2x: two arrays, every row used by edges_2x
    s = _lib.current_stream()
    probes = {"pairs": (rec, rec[:, 3 * F:], 6 * F, rev), "pairs_2x": (W2, dW2, 3 * F, rev), "edges_2x": (W2, dW2, 3 * F, None)}
    probe_ms, probe_run = {}, {}
    for name, (Wt, dWt, stride, rv) in probes.items():
        def run(Wt=Wt, dWt=dWt, stride=stride, rv=rv, name=name):
            _lib.check(lib.nb200_painn_msg_bwd_ex(_lib.ptr(xh), _lib.ptr(bias), _lib.ptr(mu), c_ptr(Wt), c_ptr(dWt), stride, _lib.ptr(rv), _lib.ptr(geom),
                                                  _lib.ptr(row_ptr), _lib.ptr(col), N, _lib.ptr(gq), _lib.ptr(gmu), _lib.ptr(g_xh), _lib.ptr(g_mu_in),
                                                  _lib.ptr(egrad), None, None, 0, s), name)
        probe_run[name] = run
        probe_ms[name] = timed(run, reps)
    record_bytes = {"pairs": E / 2 * 6 * F * 4, "pairs_2x": E / 2 * 6 * F * 4, "edges_2x": E * 6 * F * 4}

    # ---- L2 -> SM gather ceiling at this access pattern: each kernel alone on batch 0 (pair records, the E+F layout) against a load-only
    # kernel that reads the same bytes per edge (nb200_msg_gather_probe); bytes per edge L2 -> SM: forward 1.5 KB record + 3 KB of xh[j],
    # mu[j]; backward 3 KB record + 2 KB of g_q[i], g_mu[i]
    q, q_out, mu_out = rnd(N, F), torch.empty(N, F, device=dev), torch.empty(N, 3 * F, device=dev)
    sink = torch.empty(N * 32, device=dev)
    gather = {
        "fwd": (lambda: _lib.check(lib.nb200_painn_msg_fwd_ex(_lib.ptr(xh), _lib.ptr(bias), _lib.ptr(q), _lib.ptr(mu), c_ptr(rec), 6 * F, _lib.ptr(rev),
                                                              _lib.ptr(geom), _lib.ptr(row_ptr), _lib.ptr(col), N, _lib.ptr(q_out), _lib.ptr(mu_out), 0, s),
                                   "fwd"),
                lambda: _lib.check(lib.nb200_msg_gather_probe(_lib.ptr(xh), _lib.ptr(mu), c_ptr(rec), 6 * F, _lib.ptr(rev), _lib.ptr(row_ptr),
                                                              _lib.ptr(col), N, 0, _lib.ptr(sink), s), "probe fwd"),
                E * (3 * F + 3 * F + 3 * F) * 4),
        "bwd": (lambda: probe_run["pairs"](),
                lambda: _lib.check(lib.nb200_msg_gather_probe(_lib.ptr(gq), _lib.ptr(gmu), c_ptr(rec), 6 * F, _lib.ptr(rev), _lib.ptr(row_ptr),
                                                              _lib.ptr(col), N, 1, _lib.ptr(sink), s), "probe bwd"),
                E * (F + 3 * F + 6 * F) * 4),
    }
    ceiling = {}
    for name, (kern, probe, nbytes) in gather.items():
        ms_k, ms_p = timed(kern, reps), timed(probe, reps)
        ceiling[name] = {"kernel_ms": ms_k, "probe_ms": ms_p, "l2_to_sm_bytes": nbytes, "kernel_tb_per_s": nbytes / ms_k / 1e9,
                         "probe_tb_per_s": nbytes / ms_p / 1e9, "kernel_frac_of_probe": ms_p / ms_k}
    line = {"bench": "bench_msg", "tag": args.tag, "lib": _lib.LIB_PATH, "card": card(), "reps": reps,
            "atoms_per_batch": n_atoms, "edges_per_batch": [s_[0] for s_ in stats], "max_degree_per_batch": [s_[2] for s_ in stats],
            "kernels": kernels,
            "l2_probe": {"atoms": N, "edges": E, "ms_per_launch": probe_ms, "record_bytes": record_bytes,
                         "note": "backward alone on batch 0: pairs = E+F layout; pairs_2x = pair rows in two arrays; edges_2x = per-directed-edge rows"},
            "gather_ceiling": ceiling}
    print(json.dumps(line), flush=True)


def timed(fn, reps):
    """ms per call of `fn` (CUDA events around `reps` calls after 5 warm-up calls)."""
    import torch

    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def c_ptr(t):
    import ctypes

    return ctypes.c_void_p(t.data_ptr())


if __name__ == "__main__":
    main()
