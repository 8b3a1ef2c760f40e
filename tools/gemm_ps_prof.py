"""Role timing inside k_gemm_ps (gemm_ps.cu built with -DNF_PROF): where the MMA issuer and the worker warps spend their cycles.
    NB200_NVCC_EXTRA=-DNF_PROF python -m nabladft_b200.build --force && python tools/gemm_ps_prof.py [M N K]
Prints average cycles per CTA and per output tile."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from nabladft_b200 import _lib

M, N, K = (int(v) for v in sys.argv[1:4]) if len(sys.argv) >= 4 else (16384, 8320, 128)
lib = _lib.load()
dev = torch.device("cuda:0")
A = torch.randn(M, K, device=dev)
B = torch.randn(N, K, device=dev) * 0.1
C = torch.empty(M, N, device=dev)
call = lambda: _lib.check(lib.nb200_gemm_tf32x3(M, N, K, _lib.ptr(A), K, _lib.ptr(B), K, 0, _lib.ptr(C), N, 0, None, None, _lib.current_stream()), "gemm")
for _ in range(3):
    call()
torch.cuda.synchronize()
out = (ctypes.c_ulonglong * 16)()
fn = lib.nb200_debug_gemm_ps_prof
fn.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
fn(out, 1)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 5
e0.record()
for _ in range(reps):
    call()
e1.record()
torch.cuda.synchronize()
fn(out, 0)
n = max(out[7], 1)
tiles = ((N + 127) // 128) * ((K + 127) // 128)
m_tiles = (M + 127) // 128
print(f"[{M} x {N} x {K}]: {e0.elapsed_time(e1) / reps * 1e3:.1f} us per call (with profiling code), {n / reps:.0f} CTAs per call, ~{tiles * m_tiles / (n / reps):.1f} (N tile, K chunk) units per CTA")
names = ["issuer total", "issuer waits X", "issuer waits staging", "issuer waits W ring", "worker total", "worker waits accumulator + drain", "worker waits X release", "(CTAs)",
         "worker epilogue (global stores)"]
for i, nm in enumerate(names):
    if i == 7:
        continue
    print(f"   {nm:36s} {out[i] / n:12.0f} cycles per CTA   {out[i] / n / (tiles * m_tiles / (n / reps)):9.0f} per unit")
