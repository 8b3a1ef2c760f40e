"""Role timing inside the fused node kernels (painn_fused.cu built with -DNF_PROF): where the MMA issuer and the worker warps wait.
    NB200_NVCC_EXTRA=-DNF_PROF python -m nabladft_b200.build --force && python tools/nf_prof.py
Prints average cycles per kernel launch and CTA."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import torch

import bench
from nabladft_b200 import _lib
from nabladft_b200.synth import synth_batch

dev = torch.device("cuda:0")
model = bench.build_model("painn", dev)
eng = model.engine(True)
lib = _lib.load()
b = synth_batch(1, 256)
d = dict(z=torch.from_numpy(b["z"]).to(dev), pos=torch.from_numpy(b["pos"]).to(dev), mol_ptr=torch.from_numpy(b["mol_ptr"]).to(dev))
eng.e_cap = int(b["z"].shape[0]) * 32
for _ in range(5):
    eng.launch(d["z"], d["pos"], d["mol_ptr"], 256)
torch.cuda.synchronize()
out = (ctypes.c_ulonglong * 16)()
fn = lib.nb200_debug_nf_prof
fn.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
fn(out, 1)
steps = 10
for _ in range(steps):
    eng.launch(d["z"], d["pos"], d["mol_ptr"], 256)
torch.cuda.synchronize()
fn(out, 0)
names = ["issuer total", "issuer waits X", "issuer waits staging", "issuer waits W ring", "worker total", "worker waits accumulator", "worker waits X release"]
for base, tag in ((0, "k_node_fwd"), (8, "k_node_bwd")):
    n = out[base + 7]
    print(f"{tag}: {n} CTA runs ({n / steps:.0f} per step)")
    for i, nm in enumerate(names):
        print(f"   {nm:28s} {out[base + i] / max(n, 1):10.0f} cycles per CTA run")

if hasattr(lib, "nb200_debug_nf_phase"):
    ph = (ctypes.c_ulonglong * 64)()
    fp = lib.nb200_debug_nf_phase
    fp.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    fp(ph, 0)
    n = out[7]
    labels = {0: "load_x(mu_x) x3", 1: "wait+drain U tiles x6", 21: "epilogue U tiles (store VW) x6", 2: "(after U loop)", 3: "nrm -> X (registers), store nrm/dot", 4: "load_x(q_mid)",
              5: "-", 6: "wait+drain g1 nrm half", 7: "-", 8: "wait+drain g1 q_mid half", 9: "epilogue g1 final (silu -> X)",
              10: "wait+drain y1", 11: "epilogue y1 (mu update)", 12: "wait+drain y0", 13: "epilogue y0", 14: "wait+drain y2", 15: "epilogue y2 (q_next -> X)",
              16: "wait+drain h1", 17: "epilogue h1 (silu -> X)", 18: "wait+drain xh x3 (+ epilogue of previous)", 19: "last xh epilogue", 20: "readout tile"}
    print("k_node_fwd phases (worker thread 0, cycles per CTA run; all fwd launch kinds averaged):")
    for i in sorted(labels):
        print(f"   {labels[i]:45s} {ph[i] / max(n, 1):9.0f}")
