"""DimeNet++ Hessians on the device (nb200_dimenet_hvp through nabladft_b200.vibrations) at the config's sizes with the shared test weights:
full Hessians of fixture molecules against the float64 oracle's double backward (tests/golden/dimenet_hessian.npz), collinear triplets
against central differences of the oracle's forces, the 256-molecule benchmark batch against the oracle on 4 molecules, bitwise
repeatability and chunking, and normal modes against the oracle Hessian's."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_dimenet import grid_molecule  # noqa: E402
from test_dimenet_emu import _fixture, _models  # noqa: E402
from test_dimenet_hvp_emu import REL, _close, _dirs, _oracle_fd_hvp, _oracle_hvp  # noqa: E402

pytestmark = pytest.mark.gpu


class D:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def _data(z, pos, batch):
    return D(torch.as_tensor(z).long().cuda(), torch.as_tensor(pos).float().cuda(), torch.as_tensor(batch).long().cuda())


@pytest.fixture(scope="module")
def models():
    net, ora = _models()  # 6 blocks, L = 50, K = 32, scaler on
    return net.cuda(), ora


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "dimenet_hessian.npz"))


@pytest.mark.parametrize("mol", [26, 3, 99])
def test_gpu_full_hessian_against_oracle(models, golden, mol):
    from nabladft_b200 import vibrations as vib

    net, _ = models
    hs = vib.hessians(net, _data(*_fixture([mol])))
    ref = torch.from_numpy(golden[f"hessian_{mol}"]).double()
    _close(hs[0].cpu(), ref, f"Hessian of molecule {mol}")
    scale = ref.abs().max().item()
    assert hs.max_asymmetry <= REL * scale, hs.max_asymmetry
    # translation sum rule: moving every atom along c does not change the forces
    n = ref.shape[0] // 3
    colsum = hs[0].cpu().double().reshape(n, 3, 3 * n).sum(0)
    assert colsum.abs().max().item() <= REL * scale, colsum.abs().max().item()
    e, f = net(_data(*_fixture([mol])))
    assert torch.equal(hs.energy, e)


def test_gpu_grid_molecule_against_central_differences(models):
    """48 atoms on a grid (K + 1 truncation, asymmetric edges, many exactly collinear triplets)."""
    net, ora = models
    z, pos = grid_molecule()
    batch = np.zeros(len(z), dtype=np.int64)
    vs = _dirs(2, len(z), 11)
    from nabladft_b200 import vibrations as vib

    _, _, hv = vib.hessian_vector_product(net, _data(z, pos, batch), vs.float().cuda())
    ref = _oracle_fd_hvp(ora, z, pos, batch, vs)
    for k in range(len(vs)):
        _close(hv[k].cpu(), ref[k], f"grid direction {k}")


def test_gpu_benchmark_batch_directions_on_four_molecules(models):
    """synth_batch(0, 256), directions supported on 4 molecules: hv equals the oracle's on those 4 molecules alone and is exactly 0 elsewhere,
    so batching does not leak between molecules."""
    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import synth_batch

    net, ora = models
    s = synth_batch(0, 256)
    ptr = s["mol_ptr"]
    batch = np.repeat(np.arange(256), np.diff(ptr))
    chosen = [0, 97, 180, 255]
    vs_all = torch.zeros(2, len(s["z"]), 3, dtype=torch.float64)
    zs, ps, bs, vs = [], [], [], []
    for k, m in enumerate(chosen):
        a, b = ptr[m], ptr[m + 1]
        vs_all[:, a:b] = _dirs(2, b - a, 20 + k)
        zs.append(s["z"][a:b]); ps.append(s["pos"][a:b]); bs.append(np.full(b - a, k)); vs.append(vs_all[:, a:b])
    _, _, hv = vib.hessian_vector_product(net, _data(s["z"], s["pos"], batch), vs_all.float().cuda())
    hv = hv.cpu()
    ref = _oracle_hvp(ora, np.concatenate(zs), np.concatenate(ps), np.concatenate(bs), torch.cat(vs, 1))
    rows = np.concatenate([np.arange(ptr[m], ptr[m + 1]) for m in chosen])
    for k in range(2):
        _close(hv[k, rows], ref[k], f"batch direction {k}")
    mask = torch.ones(len(s["z"]), dtype=torch.bool)
    mask[rows] = False
    assert (hv[:, mask] == 0).all()


def test_gpu_bitwise_repeatable_chunking_and_inference_outputs(models):
    from nabladft_b200 import vibrations as vib

    net, _ = models
    data = _data(*_fixture([26, 3]))
    vs = _dirs(3, data.z.numel(), 12).float().cuda()
    a = vib.hessian_vector_product(net, data, vs)
    b = vib.hessian_vector_product(net, data, vs)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    e, f = net(data)
    assert torch.equal(a[0], e) and torch.equal(a[1], f)
    h1 = vib.hessians(net, data, max_dir=1)
    h7 = vib.hessians(net, data, max_dir=7)
    assert all(torch.equal(x, y) for x, y in zip(h1, h7)) and h1.max_asymmetry == h7.max_asymmetry


def test_gpu_normal_modes_against_oracle_eigenvalues(models, golden):
    """Projected normal modes of molecule 26: by Weyl's inequality every |lambda_i - lambda_i,ref| is at most the spectral norm of the
    difference of the two mass-weighted, projected Hessians."""
    from nabladft_b200 import vibrations as vib

    net, _ = models
    z, pos, batch = _fixture([26])
    modes = vib.normal_modes(net, _data(z, pos, batch), project=True)[0]
    hs = vib.hessians(net, _data(z, pos, batch))
    m = vib.masses_of(z)
    ref_h = torch.from_numpy(golden["hessian_26"]).double()
    ref = vib.normal_modes_from_hessian(ref_h, m, pos.double(), project=True)

    def mass_weighted(h):
        inv = m.repeat_interleave(3).rsqrt()
        q = vib._rigid_basis(pos.double(), m)
        p = torch.eye(h.shape[0], dtype=torch.float64) - q @ q.t()
        d = p @ (h.double() * inv[:, None] * inv[None, :]) @ p
        return 0.5 * (d + d.t())

    bound = torch.linalg.matrix_norm(mass_weighted(hs[0].cpu()) - mass_weighted(ref_h), ord=2).item()
    dev = (modes.eigenvalues.cpu() - ref.eigenvalues).abs().max().item()
    print(f"max |lambda - lambda_ref| {dev:.3e}, Weyl bound {bound:.3e}")
    assert dev <= bound * (1 + 1e-9) + 1e-12


def test_gpu_refuses_cpu_tensors_and_training_mode(models):
    from nabladft_b200 import vibrations as vib
    from nabladft_b200._lib import NablaB200Error

    net, _ = models
    z, pos, batch = _fixture([26])
    with pytest.raises(NablaB200Error):
        vib.hessians(net, D(z, pos, batch))
    net.train()
    try:
        with pytest.raises(NotImplementedError):
            vib.hessians(net, _data(z, pos, batch))
    finally:
        net.eval()
