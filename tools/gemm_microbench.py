"""Time the wgmma 3xTF32 GEMM against torch.matmul (cuBLAS SGEMM) on the shapes the engines use."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from nabladft_b200 import _lib
lib = _lib.load()
dev = "cuda:0"
shapes = [(9673, 128, 128, 0), (9673, 384, 128, 0), (29019, 256, 128, 0), (9673, 128, 384, 1), (29019, 128, 256, 1), (9673, 64, 128, 0),
          (372544, 128, 128, 0), (100096, 8320, 128, 0), (100096, 640, 640, 0), (50000, 5376, 32, 1), (100096, 128, 768, 0),
          (576636, 512, 512, 0), (576636, 64, 1024, 0), (576636, 32, 1024, 0), (76598, 1920, 128, 0)]
res = []
for M, N, K, tb in shapes:
    A = torch.randn(M, K, device=dev); B = torch.randn(K, N, device=dev) if tb else torch.randn(N, K, device=dev); C = torch.empty(M, N, device=dev)
    def tc():
        _lib.check(lib.nb200_gemm_tf32x3(M, N, K, _lib.ptr(A), K, _lib.ptr(B), N if tb else K, tb, _lib.ptr(C), N, 0, None, None, _lib.current_stream()), "g")
    def cb():
        torch.matmul(A, B if tb else B.t(), out=C)
    out = {}
    for name, fn in (("tc", tc), ("cublas", cb)):
        for _ in range(3): fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 20 if M * N * K < 1e12 else 5
        e0.record()
        for _ in range(reps): fn()
        e1.record(); torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps * 1e3
    gf = 2.0 * M * N * K / 1e9
    res.append(dict(M=M, N=N, K=K, trans_b=tb, tc_us=round(out["tc"], 1), cublas_us=round(out["cublas"], 1), tc_tflops=round(gf / out["tc"] * 1e-3 * 1e3, 1), cublas_tflops=round(gf / out["cublas"] * 1e-3 * 1e3, 1)))
    print(res[-1], flush=True)
json.dump(res, open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out", "gemm_microbench_" + os.environ.get("NB200_GEMM_VARIANT", "default") + ".json"), "w"))
