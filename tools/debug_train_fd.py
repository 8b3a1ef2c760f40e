"""Experiment behind the decision recorded in nabladft_b200/training.py: a central finite difference of the analytic energy gradient as the
force-loss gradient, against the oracle's exact double backward.  Result (3 fixture molecules, 3 layers, fp32):
    h 1e-3: whole-gradient rel L2 error 0.80 | 3e-3: 0.27 | 1e-2: 0.12 | 3e-2: 0.10 | 1e-1: 0.45   (worst tensor off by > 100 %)
=> rejected.  The script reimplements the difference on top of PainnEngine.run_train so that it keeps working."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import warnings
import torch
from helpers import load_fixture
from test_gpu_painn import _Data, _oc_model, dev
from oracle.painn_oc import PaiNNOC
warnings.simplefilter("ignore")
L = 3
kw = dict(hidden_channels=128, num_layers=L, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)
net = _oc_model(L)
ref = PaiNNOC(**kw).double()
ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
z, pos, batch = load_fixture([0, 4, 7])
g = torch.Generator().manual_seed(3)
f_t = 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
e_ref, f_ref = ref(z, pos.clone(), batch, create_graph=True)
((f_ref - f_t) ** 2).mean().backward()   # force term only
ref_g = {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for k, p in ref.named_parameters()}
net = net.to(dev()).train()
from nabladft_b200.engine import PainnEngine
eng = PainnEngine()
t, sc = net._export()
eng.set_weights(object(), t, sc)
zd, pd = z.int().to(dev()), pos.float().to(dev())
mol_ptr = torch.zeros(4, dtype=torch.int32, device=dev()); mol_ptr[1:] = torch.cumsum(torch.bincount(batch), 0).to(dev())
_, f0, _ = eng.run(zd, pd, mol_ptr, 3)
v = 2.0 * (f0 - f_t.float().to(dev())) / f0.numel()          # dLoss/dF
vmax = float(v.abs().max())
for h in (1e-3, 3e-3, 1e-2, 3e-2, 1e-1):
    _, _, gp = eng.run_train(zd, (pd + v * (h / vmax)).contiguous(), mol_ptr, 3, None)
    _, _, gm = eng.run_train(zd, (pd - v * (h / vmax)).contiguous(), mol_ptr, 3, None)
    canon = {k: (gp[k] - gm[k]) * (-vmax / (2 * h)) for k in gp}
    tt, _ = net._export_impl(detach=False)                  # carry the canonical gradients back to the named parameters
    net.zero_grad()
    torch.autograd.backward([tt[k] for k in canon], [canon[k] for k in canon])
    errs = {k: float((p.grad.double().cpu() - ref_g[k]).abs().max() / (ref_g[k].abs().max() + 1e-30)) for k, p in net.named_parameters() if float(ref_g[k].abs().max()) > 0}
    tot = sum(float(((p.grad.double().cpu() - ref_g[k]) ** 2).sum()) for k, p in net.named_parameters()) ** 0.5 / sum(float((v ** 2).sum()) for v in ref_g.values()) ** 0.5
    wk = max(errs, key=errs.get)
    print(f"h {h:7.0e}  worst per-tensor rel {errs[wk]:9.2e} ({wk})  whole-gradient rel L2 {tot:9.2e}")
