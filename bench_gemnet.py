#!/usr/bin/env python
"""GemNet-OC energy + direct forces (BASELINE.json configs[4]: 512-molecule mixed-size batch, <= 60 atoms): molecules/s of the CUDA path with
CUDA events, the engine's per-category split, and the CPU oracle on a bounded sample.  Secondary benchmark (the driver's headline is
bench.py); prints one JSON line.  NOT YET RUN ON A DEVICE (DESIGN.md 3.9): written together with the first correct path so that the next
round starts from a measurement.

    python bench_gemnet.py --batch 512 --steps 3 --warmup 3 [--cpu]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 bench_gemnet.py --batch 512
(weak scaling: every rank runs its own 512-molecule batch, no data-path collective; time = max over ranks, value = all molecules / time)
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def dense_macs(n_atoms: int, counts: dict, nb: int = 4) -> int:
    """Multiply-accumulates of the dense layers of ONE forward (csrc/gemnet_oc.cu), from the graph sizes: the algorithmic work of the dominant
    (tensor-core) kernel class.  E main edges, P a2ee2a edges, Q qint edges, A a2a edges, N atoms."""
    E, P, Q, A, N = counts["MAIN"], counts["AE"], counts["Q"], counts["A2A"], n_atoms
    res = lambda M, C: 2 * M * C * C
    basis = E * 128 * 1920 + E * 128 * 512 + P * 128 * 128 + Q * 128 * 128 + A * 128 * 64
    embed = 2 * N * 256 * 512
    out_block = N * 512 * 256 + 6 * res(N, 256) + 3 * res(E, 512)
    inter = (E * 512 * 512 * 4                      # dense_ca, dense_ba (trip), dense_db, dense_ba (edge->atom)
             + E * 512 * 64 * 2 + E * 512 * 32      # down projections (trip, edge->atom, quad)
             + E * 1024 * 64 * 2 + E * 1024 * 32    # bilinear layers on main edges (trip, atom->edge, quad)
             + E * 64 * 512 * 4 + E * 32 * 512 * 2  # up projections ca / ac
             + N * 256 * 256 + P * 256 * 64         # atom->edge: dense_ba on atoms, down projection on a2ee2a edges
             + N * 1024 * 64 * 2 + N * 64 * 256 * 2 + N * 256 * 64  # edge->atom and atom->atom bilinear / up / down
             + 5 * res(E, 512)                      # before skip (2), after skip (2), residual_m (1)
             + N * 512 * 256 + 3 * res(N, 256)      # atom update
             + 2 * N * 256 * 512 + E * 512 * 512)   # concat layer
    final = N * 256 * (nb + 1) * 256 + 2 * res(N, 256) + E * 512 * (nb + 1) * 512 + 2 * res(E, 512)
    return basis + embed + (nb + 1) * out_block + nb * inter + final


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--heavy-max", type=int, default=30, help="heavy atoms per molecule (30 heavy + H stays below 60 atoms)")
    ap.add_argument("--cpu", action="store_true", help="also time the CPU oracle on the first two molecules")
    ap.add_argument("--train", action="store_true", help="time training steps (L1 energy + L2 force loss as GemNetOCLightning, AdamW) instead of inference; "
                                                         "keeps every activation: use a training-sized batch, e.g. --batch 16")
    args = ap.parse_args()
    import numpy as np
    import torch
    import yaml
    from weights import golden_state_dict

    from nabladft_b200.gemnet_oc import GemNetOC
    from nabladft_b200.synth import synth_batch

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
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
    torch.cuda.set_device(dev)
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)
    net = net.to(dev)
    b = synth_batch(5 + rank, args.batch, heavy_max=args.heavy_max)

    class D:
        pass

    d = D()
    d.z, d.pos, d.batch = torch.from_numpy(b["z"]).to(dev), torch.from_numpy(b["pos"]).to(dev), torch.from_numpy(b["batch"]).to(dev)
    if args.train:
        from nabladft_b200.losses import L2Loss
        from nabladft_b200.parallel import allreduce_gradients

        net.train()
        opt = torch.optim.AdamW(net.parameters(), lr=1e-5, amsgrad=True, betas=(0.9, 0.95), weight_decay=0)  # config/model/gemnet-oc.yaml
        e_t, f_t = torch.randn(args.batch, device=dev), 0.1 * torch.randn(b["pos"].shape[0], 3, device=dev)
        l2 = L2Loss()

        def step():
            opt.zero_grad(set_to_none=True)
            E_, F_ = net(d)
            (torch.nn.functional.l1_loss(E_, e_t) + 100.0 * l2(F_, f_t)).backward()
            allreduce_gradients(net.parameters())
            opt.step()
            return E_, F_
    else:
        def step():
            with torch.no_grad():
                return net(d)
    for _ in range(args.warmup):
        E, F = step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        E, F = step()
    ev1.record()
    torch.cuda.synchronize()
    E, F = E.detach(), F.detach()
    ms = ev0.elapsed_time(ev1) / args.steps
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)  # the only collective, outside the timed region
        ms = float(t.item())
        dist.barrier()
    out = {"metric": "molecules/sec (GemNet-OC training step, L1(E) + 100 L2(F), AdamW)" if args.train else "molecules/sec (GemNet-OC E + direct F forward)", "value": world * args.batch / (ms / 1e3), "unit": "molecules/s", "ms_per_step": ms,
           "n_gpus": world, "scaling": "weak", "batch": args.batch, "atoms": int(b["z"].shape[0]), "counts": net._runner.last_counts,
           "peak_mem_gb": torch.cuda.max_memory_allocated() / 2**30, "dtype": "f32", "data": "synthetic", "finite": bool(torch.isfinite(E).all() and torch.isfinite(F).all())}
    if not args.train:
        # tensor roofline of the dense layers: algorithmic fp32 FLOPs / time against the measured bf16 peak / 6 (TF32 runs at half the bf16
        # rate and an fp32-accurate 3xTF32 product issues three MMAs).  The whole forward is timed, so `frac` is a lower bound for the GEMMs.
        peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
        bf16 = None
        if os.path.exists(peaks_path):
            pk = json.load(open(peaks_path))
            bf16 = pk.get("bf16_tflops_sustained") or pk.get("bf16_tflops")  # the dense layers run inside a long step: sustained figure
        flops = 2.0 * dense_macs(int(b["z"].shape[0]), net._runner.last_counts, net.num_blocks)
        ach = flops / (ms / 1e3) / 1e12
        peak = (bf16 / 6.0) if bf16 else 2250.0 / 6.0
        out["roofline"] = {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s (fp32-accurate, 3xTF32)", "frac": ach / peak,
                           "traffic": None, "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained / 6" if bf16 else "nominal 2250 TF/s bf16 / 6 (no MEASURED_PEAKS.json)",
                           "algorithmic_flops_per_forward": flops, "note": "whole forward timed: lower bound for the dense kernels"}
    if args.cpu and rank == 0:
        from oracle.gemnet_oc import GemNetOCOracle

        ora = GemNetOCOracle().float().eval()
        ora.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, strict=True)
        torch.set_num_threads(min(32, os.cpu_count() or 1))
        n0 = int(b["mol_ptr"][2])
        z, pos, bt = d.z[:n0].cpu().long(), d.pos[:n0].cpu(), d.batch[:n0].cpu().long()
        with torch.no_grad():
            t0 = time.perf_counter()
            E0, F0 = ora(z, pos, bt)
            dt = time.perf_counter() - t0
        out["cpu_baseline"] = {"value": 2.0 / dt, "unit": "molecules/s", "cores": torch.get_num_threads(), "kind": "port",
                               "sample": f"2 molecules ({n0} atoms), oracle restatement fp32"}
        out["parity_vs_oracle"] = {"dE": float((E[:2].cpu() - E0).abs().max()), "dF": float((F[:n0].cpu() - F0).abs().max())}
    if rank == 0:
        print(json.dumps(out), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
