"""Debug harness of the wgmma weight-gradient kernel: structured inputs whose products identify operand-layout mistakes."""
import sys
import torch
sys.path.insert(0, ".")
from nabladft_b200 import _lib

lib = _lib.load()
dev = torch.device("cuda:0")
torch.set_printoptions(linewidth=200, precision=3, sci_mode=False)


def run(G, X, out, inn, bias=True):
    M = G.shape[0]
    dW = torch.zeros(out, inn, device=dev)
    db = torch.zeros(out, device=dev) if bias else None
    _lib.check(lib.nb200_linear_wgrad(M, out, inn, _lib.ptr(G), _lib.ptr(X), None, None, out, inn, _lib.ptr(dW), inn, 1.0, _lib.ptr(db), 1.0, None, 1,
                                      _lib.current_stream()), "wgrad")
    torch.cuda.synchronize()
    return dW, db


for M in (8, 32, 128, 200):
    out, inn = 128, 128
    o = torch.arange(out, device=dev, dtype=torch.float32)
    i = torch.arange(inn, device=dev, dtype=torch.float32)
    a = torch.arange(M, device=dev, dtype=torch.float32)
    cases = {
        "ones": (torch.ones(M, out, device=dev), torch.ones(M, inn, device=dev)),
        "G=o+1": ((o + 1)[None, :].repeat(M, 1).contiguous(), torch.ones(M, inn, device=dev)),
        "X=i+1": (torch.ones(M, out, device=dev), (i + 1)[None, :].repeat(M, 1).contiguous()),
        "G=delta(a0)": ((a == 0).float()[:, None].repeat(1, out).contiguous(), torch.ones(M, inn, device=dev)),
        "G=a+1": ((a + 1)[:, None].repeat(1, out).contiguous(), torch.ones(M, inn, device=dev)),
    }
    for name, (G, X) in cases.items():
        dW, db = run(G, X, out, inn)
        ref = G.double().T @ X.double()
        err = (dW.double() - ref).abs().max().item()
        print(f"M={M} {name}: max err {err:.3g}; dW[0:3,0:6]={dW[0:3, 0:6].flatten().tolist()} dW[64,5]={dW[64, 5].item()} ref[0:3,0:2]={ref[0:3, 0:2].flatten().tolist()} "
              f"bias[0:3]={db[0:3].tolist()} nonzero={int((dW != 0).sum())}")
g = torch.Generator().manual_seed(0)
G, X = torch.randn(4676, 384, generator=g).to(dev), torch.randn(4676, 128, generator=g).to(dev)
dW, db = run(G, X, 384, 128)
ref = G.double().T @ X.double()
print("random 4676x384x128: rel err", ((dW.double() - ref).abs().max() / ref.abs().max()).item(), " |dW| max", dW.abs().max().item(), " ref max", ref.abs().max().item())
