"""SchNet Hessian-vector products (csrc/schnet_hvp.inc) checked on the CPU: the host-emulation build of csrc/schnet_train.cu (tests/emu) driven
through the product's own host code (`PainnEngine.run_hvp`, `vibrations.hessians_from_hvp`) against the float64 double backward of the oracle
(oracle/spk.py).  As tests/test_schnet_train_emu.py: this validates the arithmetic and the host plumbing, not the launch configuration; every
call poisons the reused workspace and checks the guard zones behind its sub-buffers."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from helpers import load_fixture, load_golden_weights  # noqa: E402

N_INTERACTIONS = 3


@pytest.fixture(scope="module")
def lib():
    from emu_driver import load

    return load("schnet_train", ["nb200_schnet_train", "nb200_schnet_hvp"])


@pytest.fixture(scope="module")
def models():
    from nabladft_b200 import spk
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkSchNet

    m = spk.NeuralNetworkPotential(
        representation=spk.SchNet(n_atom_basis=128, n_interactions=N_INTERACTIONS, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                  cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()], output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()],
        postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32, weight_scale=1.0)
    m.postprocessors[0].mean.fill_(0.02)
    ref = OracleNNP(SpkSchNet(n_interactions=N_INTERACTIONS)).double()
    sd = m.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    return m.eval(), ref


@pytest.fixture(scope="module")
def engine(lib, models):
    """The product's SchNet engine on the emulation library: host tensors, no streams."""
    from emu_driver import poisoned

    from nabladft_b200.engine import PainnEngine
    from nabladft_b200.schnet_train import SchnetTrainRunner

    m, _ = models
    eng = poisoned(PainnEngine, checked=["run_hvp"])("schnet", lib=lib)
    tensors, scalars = m._export_schnet(postprocess=True)
    eng._weights, eng._keep = SchnetTrainRunner._struct(tensors, scalars), tensors  # set_weights() takes CUDA tensors only
    return eng


def _inputs(mols):
    z, pos, batch = load_fixture(mols)
    mol_ptr = torch.zeros(len(mols) + 1, dtype=torch.int32)
    mol_ptr[1:] = torch.cumsum(torch.bincount(batch), 0)
    return z, pos, batch, mol_ptr


def _oracle(ref, z, pos, batch):
    """energy (with the AddOffsets shift), forces and the full [3N, 3N] Hessian by float64 double backward of the oracle's forces."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr

    p = pos.detach().clone().double().requires_grad_(True)
    idx_i, idx_j = ase_neighbor_list(p.detach(), batch_to_ptr(batch), 5.0)
    out = ref({"_atomic_numbers": z, "_positions": p, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=True, create_graph=True)
    f = out["forces"].reshape(-1)
    rows = [torch.autograd.grad(-f[i], p, retain_graph=True, allow_unused=True)[0] for i in range(f.numel())]
    h = torch.stack([torch.zeros_like(p).reshape(-1) if r is None else r.reshape(-1) for r in rows]).detach()
    return out["energy"].detach(), out["forces"].detach(), h


def _hessians(engine, z, pos, mol_ptr, max_dir=None):
    from nabladft_b200 import vibrations as vib

    z32, p32 = z.to(torch.int32), pos.float().contiguous()
    return vib.hessians_from_hvp(lambda v: engine.run_hvp(z32, p32, mol_ptr, mol_ptr.numel() - 1, v, with_forces=False)[2], mol_ptr.tolist(),
                                 max_dir)


def test_schnet_hessians_energy_and_forces_match_oracle_double_backward(engine, models):
    _, ref = models
    z, pos, batch, mol_ptr = _inputs([26, 3])  # 29 and 30 atoms
    e_ref, f_ref, h_ref = _oracle(ref, z, pos, batch)
    hs = _hessians(engine, z, pos, mol_ptr)
    ptr = mol_ptr.tolist()
    worst = []
    for k, h in enumerate(hs):
        a, b = 3 * ptr[k], 3 * ptr[k + 1]
        r = h_ref[a:b, a:b]
        r = 0.5 * (r + r.t())
        worst.append(float((h.double() - r).abs().max() / r.abs().max()))
    print("worst |H - H_ref| / max|H_ref| per molecule:", worst, "raw asymmetry", hs.max_asymmetry)
    assert max(worst) < 2e-5
    # the call's own energies and forces
    e, f, hv = engine.run_hvp(z.to(torch.int32), pos.float().contiguous(), mol_ptr, 2, torch.zeros(1, z.numel(), 3))
    print("energy error", float((e.double() - e_ref).abs().max()), "force error", float((f.double() - f_ref).abs().max()))
    assert float((e.double() - e_ref).abs().max()) < 1e-5
    assert float((f.double() - f_ref).abs().max()) < 1e-4
    assert torch.equal(hv, torch.zeros_like(hv))  # zero direction: exactly zero


def test_schnet_hvp_random_directions_match_oracle(engine, models):
    _, ref = models
    z, pos, batch, mol_ptr = _inputs([99])  # 54 atoms
    _, _, h_ref = _oracle(ref, z, pos, batch)
    g = torch.Generator().manual_seed(11)
    v = torch.randn(3, z.numel(), 3, generator=g)
    _, _, hv = engine.run_hvp(z.to(torch.int32), pos.float().contiguous(), mol_ptr, 1, v.contiguous())
    hv_ref = (h_ref @ v.double().reshape(3, -1).t()).t().reshape(3, -1, 3)
    err = float((hv.double() - hv_ref).abs().max() / hv_ref.abs().max())
    print("random directions: max |Hv - Hv_ref| / max|Hv_ref|", err)
    assert err < 2e-5


def test_schnet_hessians_do_not_depend_on_direction_chunking(engine):
    z, pos, _, mol_ptr = _inputs([0, 4])
    hs7 = _hessians(engine, z, pos, mol_ptr, max_dir=7)
    hs1 = _hessians(engine, z, pos, mol_ptr, max_dir=1)
    assert all(torch.equal(a, b) for a, b in zip(hs1, hs7))


def test_schnet_hvp_c_abi_argument_checks(lib, engine):
    """Null v / hv, n_dir < 1, a short workspace and a bad config are refused with NB200_EINVAL before any launch; the size function of
    libnabla_b200.so (pure host code) agrees with the emulation build up to the guard zones."""
    from ctypes import byref, c_int64

    from nabladft_b200 import _lib

    z, pos, _, mol_ptr = _inputs([3])
    z32, pos32, n = z.to(torch.int32), pos.float().contiguous(), z.numel()
    w = engine._weights
    row_ptr, scratch, n_edges = torch.empty(n + 1, dtype=torch.int32), torch.empty(2 * n, dtype=torch.int32), c_int64(0)
    assert lib.nb200_schnet_train_count(byref(w), pos32.data_ptr(), mol_ptr.data_ptr(), 1, n, row_ptr.data_ptr(), scratch.data_ptr(), byref(n_edges), None) == 0
    need = lib.nb200_schnet_hvp_workspace_bytes(byref(w), 1, n, n_edges.value)
    real = _lib.load()
    assert 0 < real.nb200_schnet_hvp_workspace_bytes(byref(w), 1, n, n_edges.value) <= need
    assert real.nb200_schnet_hvp_workspace_bytes(byref(w), 1, n, -1) == -1
    ws, energy, forces = torch.zeros(need, dtype=torch.uint8), torch.zeros(1), torch.zeros(n, 3)
    v, hv = torch.randn(2, n, 3), torch.zeros(2, n, 3)

    def call(n_dir=2, v_=v, hv_=hv, ws_bytes=need, w_=w):
        return lib.nb200_schnet_hvp(engine._h, byref(w_), z32.data_ptr(), pos32.data_ptr(), mol_ptr.data_ptr(), 1, n, row_ptr.data_ptr(),
                                    n_edges.value, ws.data_ptr(), ws_bytes, n_dir, None if v_ is None else v_.data_ptr(), energy.data_ptr(),
                                    forces.data_ptr(), None if hv_ is None else hv_.data_ptr(), None)

    energy.fill_(7.0)
    assert call(v_=None) == -1
    assert call(hv_=None) == -1
    assert call(n_dir=0) == -1
    assert call(ws_bytes=need - 1) == -1
    bad = type(w).from_buffer_copy(w)
    bad.n_feat = 64
    assert call(w_=bad) == -1
    assert float(energy[0]) == 7.0 and torch.equal(hv, torch.zeros_like(hv))  # nothing ran
    lib.nb200_emu_check_guards()
    assert call() == 0 and bool(torch.isfinite(hv).all()) and bool(torch.isfinite(forces).all())
    lib.nb200_emu_check_guards()
