"""DimeNet++ on the device through the mirror's forward() (nabladft_b200/dimenetplusplus.py -> csrc/dimenet.cu) against the float64 oracle."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_dimenet import SCALER, grid_molecule, load_test_weights  # noqa: E402

pytestmark = pytest.mark.gpu
E_TOL, F_TOL = 1e-5, 1e-4  # Ha, Ha/A, at test weights whose energies are of order 1 Ha
E_REL = 4e-6  # above 2.5 Ha: fp32 keeps ~7 digits; the 48-atom grid's 19.5 Ha energy was reached to 3.5e-5 (1.8e-6 relative) on an H100


class _Data:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def _models(num_blocks=6):
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    kw = dict(node_latent_dim=50, scaler=SCALER, dimenet_hidden_channels=256, dimenet_num_blocks=num_blocks, do_postprocessing=True)
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(**kw).double().eval())
    net = DimeNetPlusPlusPotential(**kw).eval()
    net.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    return net.cuda(), ora


def _dev(z, pos, batch):
    return _Data(torch.as_tensor(z).long().cuda(), torch.as_tensor(pos).float().cuda(), torch.as_tensor(batch).long().cuda())


@pytest.fixture(scope="module")
def models():
    return _models()


def test_gpu_golden_and_oracle(models):
    net, ora = models
    g = np.load(os.path.join(HERE, "golden", "dimenet_f64.npz"))
    e, f = net(_dev(g["z"], g["pos"], g["batch"]))
    assert np.abs(e.double().cpu().numpy() - g["energy"]).max() < E_TOL
    assert np.abs(f.double().cpu().numpy() - g["forces"]).max() < F_TOL


def test_gpu_edge_cases(models):
    """The 48-atom grid (the K + 1 truncation, collinear triplets), an isolated atom, a one-atom molecule."""
    net, ora = models
    z, pos = grid_molecule()
    far = np.array([[30.0, 0, 0], [0, 40.0, 0]], dtype=np.float32)
    z = np.concatenate([z, np.array([1, 8], dtype=np.int32)])
    pos = np.concatenate([pos, far])
    batch = np.array([0] * 49 + [1])
    e, f = net(_dev(z, pos, batch))
    e_ref, f_ref, _ = ora(torch.from_numpy(z).long(), torch.from_numpy(pos).double(), torch.from_numpy(batch).long())
    assert ((e.double().cpu() - e_ref).abs() < torch.clamp(E_REL * e_ref.abs(), min=E_TOL)).all()
    assert (f.double().cpu() - f_ref).abs().max() < F_TOL
    assert (f[48:] == 0).all()


def test_gpu_benchmark_batch_against_oracle_and_bitwise_repeat(models):
    """256 synthetic molecules (the bench_dimenet.py shape); the oracle on every 16th molecule (molecules do not interact)."""
    from nabladft_b200.synth import synth_batch

    net, ora = models
    b = synth_batch(0, 256)
    data = _dev(b["z"], b["pos"], b["batch"])
    e1, f1 = net(data)
    e2, f2 = net(data)
    assert torch.equal(e1, e2) and torch.equal(f1, f2)
    ptr = b["mol_ptr"]
    worst_e = worst_f = 0.0
    for m in range(0, 256, 16):
        s, t = ptr[m], ptr[m + 1]
        e_ref, f_ref, _ = ora(torch.from_numpy(b["z"][s:t]).long(), torch.from_numpy(b["pos"][s:t]).double(), torch.zeros(t - s, dtype=torch.long))
        worst_e = max(worst_e, abs(e1[m].item() - e_ref.item()))
        worst_f = max(worst_f, (f1[s:t].double().cpu() - f_ref).abs().max().item())
    assert worst_e < E_TOL and worst_f < F_TOL, (worst_e, worst_f)


def test_gpu_reference_style_shapes():
    """tests/model/test_torch_models.py:20-27 of the reference: the shipped config on a random batch -> (energy [B], forces [N, 3])."""
    import yaml

    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential

    cfg = yaml.safe_load(open(os.path.join(HERE, "..", "config", "model", "dimenetplusplus-b200.yaml")))["net"]
    cfg.pop("_target_")
    net = DimeNetPlusPlusPotential(**cfg).cuda().eval()
    g = torch.Generator().manual_seed(0)
    n = 30
    pos = (torch.rand(n, 3, generator=g) * 6).cuda()
    z = torch.randint(1, 10, (n,), generator=g).cuda()
    batch = torch.tensor([0] * 10 + [1] * 20).cuda()
    e, f = net(_Data(z, pos, batch))
    assert e.shape == (2,) and f.shape == (n, 3) and torch.isfinite(e).all() and torch.isfinite(f).all()


def test_gpu_errors_raise(models):
    from nabladft_b200._lib import NablaB200Error

    net, _ = models
    g = np.load(os.path.join(HERE, "golden", "dimenet_f64.npz"))
    z = g["z"].copy()
    z[1] = 95
    with pytest.raises(NablaB200Error, match="EINVAL"):
        net(_dev(z, g["pos"], g["batch"]))
    pos = g["pos"].copy()
    pos[2, 0] = np.inf
    with pytest.raises(NablaB200Error, match="EINVAL"):
        net(_dev(g["z"], pos, g["batch"]))
    with pytest.raises(NablaB200Error):
        net(_Data(torch.as_tensor(g["z"]).long(), torch.as_tensor(g["pos"]), torch.as_tensor(g["batch"]).long()))  # CPU tensors
