"""GemNet-OC force-Jacobian products on the device (nb200_gemnet_oc_jvp through nabladft_b200.vibrations) at the config's sizes with the
shared test weights: full Jacobians of fixture molecules against the float64 oracle's (tests/golden/gemnet_oc_jacobian.npz), the translation
sum rule and rotation covariance on a 64-molecule batch, bitwise repeatability and chunking, normal modes against the oracle Jacobian's, and
energies and forces against the inference and training forwards.  The same arithmetic on the host-emulation build is
tests/test_gemnet_hvp_emu.py."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))

from test_gemnet_emu import _models  # noqa: E402
from test_gemnet_hvp_emu import REL, _close, _dirs  # noqa: E402

pytestmark = pytest.mark.gpu
E_TOL, F_TOL = 1e-5, 1e-4  # Ha, Ha/A: the GemNet-OC forward's tolerances (tests/test_zz_gpu_first_runs.py)


class D:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def _fixture(mols):
    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    zs, ps, bs = [], [], []
    for k, m in enumerate(mols):
        a, b = fx["ptr"][m], fx["ptr"][m + 1]
        zs.append(fx["z"][a:b]); ps.append(fx["pos"][a:b]); bs.append(np.full(b - a, k))
    return np.concatenate(zs), np.concatenate(ps).astype(np.float32), np.concatenate(bs)


def _data(z, pos, batch):
    return D(torch.as_tensor(z).long().cuda(), torch.as_tensor(pos).float().cuda(), torch.as_tensor(batch).long().cuda())


@pytest.fixture(scope="module")
def net():
    return _models(True)[0].cuda().eval()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "gemnet_oc_jacobian.npz"))


def _raw_jacobians(net, data, max_dir=64):
    """Per-molecule J = -(dF/dR), [3n, 3n] float64 on the host, NOT symmetrised: column 3k + c from the shared direction 3k + c."""
    from nabladft_b200 import vibrations as vib

    runner, z, pos, mol_ptr, n_mol = net.engine_inputs(data)
    ptr = mol_ptr.cpu().tolist()
    sizes = [b - a for a, b in zip(ptr[:-1], ptr[1:])]
    n_dir = 3 * max(sizes)
    cols = torch.cat([runner.run_hvp(z, pos, mol_ptr, n_mol, vib.shared_directions(ptr, d0, min(d0 + max_dir, n_dir), pos.device),
                                     with_forces=False)[2].cpu() for d0 in range(0, n_dir, max_dir)]).double()
    return [cols[:3 * n, a:a + n].reshape(3 * n, 3 * n).t() for a, n in zip(ptr[:-1], sizes)], dict(runner.last_counts)


@pytest.mark.parametrize("mol", [26, 3])
def test_gpu_full_jacobian_against_oracle(net, golden, mol):
    J = _raw_jacobians(net, _data(*_fixture([mol])))[0][0]
    ref = torch.from_numpy(golden[f"jacobian_{mol}"]).double()
    _close(J, ref, f"Jacobian of molecule {mol}")
    n = ref.shape[0] // 3
    colsum = J.reshape(3 * n, n, 3).sum(1)  # translation sum rule: moving every atom along c does not change the forces
    assert colsum.abs().max().item() <= REL * ref.abs().max().item(), colsum.abs().max().item()
    print(f"molecule {mol}: max |J - J^T| = {(J - J.t()).abs().max().item():.3e} (oracle {(ref - ref.t()).abs().max().item():.3e}), "
          f"max |J| {ref.abs().max().item():.3e}")


def _rotation(seed):
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    return q if torch.det(q) > 0 else -q


def test_gpu_translation_sum_rule_and_rotation_covariance_on_64_molecules(net):
    """64 synthetic molecules of 6-10 heavy atoms (990 atoms, 57 shared directions; 17 GB of workspace -- 64 fixture molecules would need
    92 GB): every Jacobian obeys sum_j dF_i/dR_j = 0, and rotating the batch by Q gives J(QR) = (I x Q) J(R) (I x Q)^T within the fp32
    tolerance."""
    from nabladft_b200.synth import synth_batch

    s = synth_batch(1, 64, heavy_min=6, heavy_max=10)
    z, pos, batch = s["z"], s["pos"], s["batch"]
    Js, counts = _raw_jacobians(net, _data(z, pos, batch))
    Q = _rotation(3)
    pos_r = (torch.from_numpy(pos).double() @ Q.t()).float().numpy()
    Jr, counts_r = _raw_jacobians(net, _data(z, pos_r, batch))
    assert counts == counts_r  # the same graphs (membership depends on distances only)
    worst_sum, worst_rot = 0.0, 0.0
    for J, JQ in zip(Js, Jr):
        n = J.shape[0] // 3
        scale = J.abs().max().item()
        worst_sum = max(worst_sum, J.reshape(3 * n, n, 3).sum(1).abs().max().item() / scale)
        B = torch.block_diag(*[Q] * n)
        worst_rot = max(worst_rot, (JQ - B @ J @ B.t()).abs().max().item() / scale)
    print(f"64 molecules: worst translation sum {worst_sum:.2e}, worst rotation covariance deviation {worst_rot:.2e} (of max |J|)")
    assert worst_sum <= REL and worst_rot <= REL


def test_gpu_bitwise_repeatable_and_chunk_independent(net):
    from nabladft_b200 import vibrations as vib

    data = _data(*_fixture([26, 3]))
    vs = _dirs(6, data.z.numel(), 12).float().cuda()
    a = vib.hessian_vector_product(net, data, vs)
    b = vib.hessian_vector_product(net, data, vs)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    ones = torch.cat([vib.hessian_vector_product(net, data, vs[k:k + 1])[2] for k in range(6)])
    assert torch.equal(ones, a[2])  # 1 x 6 directions == 6 x 1
    h1 = vib.hessians(net, data, max_dir=1)
    h7 = vib.hessians(net, data, max_dir=7)
    assert all(torch.equal(x, y) for x, y in zip(h1, h7)) and h1.max_asymmetry == h7.max_asymmetry


def test_gpu_energy_and_forces_match_training_and_inference_forwards(net):
    from nabladft_b200 import vibrations as vib

    data = _data(*_fixture([26, 3, 99]))
    e, f, _ = vib.hessian_vector_product(net, data, _dirs(1, data.z.numel(), 5)[0].float().cuda())
    runner, z, pos, mol_ptr, n_mol = net.engine_inputs(data)
    e_tr, f_tr, _ = runner.run_train(z, pos, mol_ptr, n_mol, int((mol_ptr[1:] - mol_ptr[:-1]).max()))
    assert torch.equal(e, e_tr) and torch.equal(f, f_tr)
    with torch.no_grad():
        e_inf, f_inf = net(data)
    de, df = (e - e_inf).abs().max().item(), (f - f_inf).abs().max().item()
    print(f"against the inference forward: max |dE| {de:.2e} Ha, max |dF| {df:.2e} Ha/A")
    assert de < E_TOL and df < F_TOL


def test_gpu_normal_modes_against_oracle_eigenvalues(net, golden):
    """Projected normal modes of molecule 26 from the symmetrised Jacobian: by Weyl's inequality every |lambda_i - lambda_i,ref| is at most
    the spectral norm of the difference of the two mass-weighted, projected, symmetrised matrices."""
    from nabladft_b200 import vibrations as vib

    z, pos, batch = _fixture([26])
    modes = vib.normal_modes(net, _data(z, pos, batch), project=True)[0]
    hs = vib.hessians(net, _data(z, pos, batch))
    m = vib.masses_of(torch.as_tensor(z))
    ref_j = torch.from_numpy(golden["jacobian_26"]).double()
    pos64 = torch.from_numpy(pos).double()
    ref = vib.normal_modes_from_hessian(0.5 * (ref_j + ref_j.t()), m, pos64, project=True)

    def mass_weighted(h):
        inv = m.repeat_interleave(3).rsqrt()
        q = vib._rigid_basis(pos64, m)
        p = torch.eye(h.shape[0], dtype=torch.float64) - q @ q.t()
        d = p @ (h.double() * inv[:, None] * inv[None, :]) @ p
        return 0.5 * (d + d.t())

    bound = torch.linalg.matrix_norm(mass_weighted(hs[0].cpu()) - mass_weighted(ref_j), ord=2).item()
    dev = (modes.eigenvalues.cpu() - ref.eigenvalues).abs().max().item()
    print(f"max |lambda - lambda_ref| {dev:.3e}, Weyl bound {bound:.3e}")
    print(vib.summary(modes))
    assert dev <= bound * (1 + 1e-9) + 1e-12


def test_gpu_refuses_cpu_tensors_and_training_mode(net):
    from nabladft_b200 import vibrations as vib
    from nabladft_b200._lib import NablaB200Error

    z, pos, batch = _fixture([26])
    with pytest.raises(NablaB200Error):
        vib.hessians(net, D(torch.as_tensor(z).long(), torch.as_tensor(pos), torch.as_tensor(batch).long()))
    net.train()
    try:
        with pytest.raises(NotImplementedError):
            vib.hessians(net, _data(z, pos, batch))
    finally:
        net.eval()


def test_gpu_workspace_released_after_hessians_and_a_batch_too_large_is_refused_clearly(net):
    """`hessians` hands the jvp workspace (the training arena twice) back to the allocator when it is done; a batch whose workspace exceeds
    the card (64 fixture molecules need 92 GB) raises NablaB200Error asking for a split, not a bare allocator error."""
    from nabladft_b200 import vibrations as vib
    from nabladft_b200._lib import NablaB200Error

    hs = vib.hessians(net, _data(*_fixture([26])))
    assert len(hs) == 1 and getattr(net._get_runner(), "_jvp_ws", None) is None
    with pytest.raises(NablaB200Error, match="split the batch by molecules"):
        vib.hessians(net, _data(*_fixture(range(64))))
    assert getattr(net._get_runner(), "_jvp_ws", None) is None
    torch.cuda.empty_cache()
