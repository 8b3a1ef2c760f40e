"""SchNet energy-loss training (BASELINE configs[0]) checked on the CPU: csrc/schnet_train.cu through its host-emulation build (tests/emu), driven
by the product's own host code (`spk.NeuralNetworkPotential._train_schnet_with`, `schnet_train.SchnetEnergyFn`), against the autograd of the
oracle (oracle/spk.py) in float64 for EVERY schnetpack-named parameter.  Same caveat as tests/test_gemnet_emu.py: this validates the arithmetic
and the autograd plumbing, not the launch configuration; the emulation library is test infrastructure and is never loaded by the package."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from helpers import load_fixture, load_golden_weights  # noqa: E402


@pytest.fixture(scope="module")
def runner():
    from emu_driver import load, poisoned

    from nabladft_b200.schnet_train import SchnetTrainRunner

    lib = load("schnet_train", ["nb200_schnet_train", "nb200_schnet_energy_grads"])
    return poisoned(SchnetTrainRunner, checked=["energy_grads"])(lib)


def _models(with_forces: bool, n_interactions=6):
    from nabladft_b200 import spk
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkSchNet

    out = [spk.Atomwise(n_in=128, output_key="energy")] + ([spk.Forces()] if with_forces else [])
    m = spk.NeuralNetworkPotential(
        representation=spk.SchNet(n_atom_basis=128, n_interactions=n_interactions, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                  cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()], output_modules=out, postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32, weight_scale=1.0)
    m.postprocessors[0].mean.fill_(0.02)
    ref = OracleNNP(SpkSchNet(n_interactions=n_interactions)).double()
    sd = m.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    return m.train(), ref.train()


def _batch(mols):
    from oracle.graph import ase_neighbor_list, batch_to_ptr

    z, pos, batch = load_fixture(mols)
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    n_mol = int(batch.max()) + 1
    mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32)
    mol_ptr[1:] = torch.cumsum(torch.bincount(batch), 0)
    return z, pos, batch, idx_i, idx_j, mol_ptr, n_mol


def test_schnet_energy_and_every_parameter_gradient_match_oracle_autograd(runner):
    m, ref = _models(with_forces=False)
    z, pos, batch, idx_i, idx_j, mol_ptr, n_mol = _batch([10, 11, 12, 60])
    c = torch.tensor([0.7, -1.3, 0.4, 2.1], dtype=torch.float64)  # dLoss/dE_m of some energy loss
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False, create_graph=True)
    (out_ref["energy"] * c).sum().backward()
    out = m._train_schnet_with(runner, None, z.to(torch.int32), pos.float().contiguous(), mol_ptr, n_mol)
    assert set(out) == {"energy"} and runner.last_edges == idx_i.numel()
    e, e_ref = out["energy"], out_ref["energy"].detach()
    assert (e.double() - e_ref).abs().max() < 1e-5  # training semantics: no AddOffsets shift
    (e * c.float()).sum().backward()
    refp = dict(ref.named_parameters())
    worst = 0.0
    for name, p in m.named_parameters():
        g_ref = refp[name].grad
        assert p.grad is not None and g_ref is not None, name
        scale = g_ref.abs().max().item()
        err = (p.grad.double() - g_ref).abs().max().item()
        worst = max(worst, err / max(scale, 1e-12))
        assert err <= 2e-5 * scale + 1e-9, (name, err, scale)
    print(f"worst relative gradient error over {len(refp)} tensors: {worst:.2e}")


class _OracleForces:
    """Stands in for the (device-verified) inference engine that supplies the force VALUES in training mode; not available on the CPU."""

    def __init__(self, forces):
        self.forces = forces

    def run(self, z_, pos_, mol_ptr_, n_mol_, with_forces=True):
        return None, self.forces.float().contiguous(), None


def test_schnet_energy_plus_force_loss_gradients_match_oracle_double_backward(runner):
    """loss = sum_m c_m E_m + sum_i v_i . F_i  (any energy + force loss has this form to first order): every parameter gradient against the
    oracle's create_graph=True double backward in float64 -- the force term through the engine's tangent pass."""
    m, ref = _models(with_forces=True)
    z, pos, batch, idx_i, idx_j, mol_ptr, n_mol = _batch([10, 11, 12, 60])
    g = torch.Generator().manual_seed(3)
    c = torch.tensor([0.7, -1.3, 0.4, 2.1], dtype=torch.float64)
    v = torch.randn(z.shape[0], 3, generator=g, dtype=torch.float64)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False, create_graph=True)
    ((out_ref["energy"] * c).sum() + (out_ref["forces"] * v).sum()).backward()
    refp = dict(ref.named_parameters())
    for only_forces in (False, True):
        m.zero_grad()
        out = m._train_schnet_with(runner, _OracleForces(out_ref["forces"].detach()), z.to(torch.int32), pos.float().contiguous(), mol_ptr, n_mol)
        assert out["forces"].shape == (z.shape[0], 3)
        if only_forces:
            (out["forces"] * v.float()).sum().backward()
            continue  # exercised for the seed-less energy branch; compared below through the sum only
        ((out["energy"] * c.float()).sum() + (out["forces"] * v.float()).sum()).backward()
        worst = 0.0
        for name, p in m.named_parameters():
            g_ref = refp[name].grad
            scale = g_ref.abs().max().item()
            err = (p.grad.double() - g_ref).abs().max().item()
            worst = max(worst, err / max(scale, 1e-12))
            assert err <= 5e-5 * scale + 1e-9, (name, err, scale)
        print(f"E+F loss: worst relative gradient error over {len(refp)} tensors: {worst:.2e}")


def test_schnet_training_step_with_an_optimizer(runner):
    """One SGD step on an MSE energy + force loss moves the parameters the way the oracle's step does."""
    m, ref = _models(with_forces=True, n_interactions=3)
    z, pos, batch, idx_i, idx_j, mol_ptr, n_mol = _batch([3, 4])
    target = torch.tensor([-0.4, 0.9])
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    f_target = torch.zeros(z.shape[0], 3)
    opt, opt_ref = torch.optim.SGD(m.parameters(), lr=0.05), torch.optim.SGD(ref.parameters(), lr=0.05)  # (Adam's first step is lr * sign(g): ill-conditioned where g ~ 0)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False, create_graph=True)
    (torch.nn.functional.mse_loss(out_ref["energy"], target.double()) + torch.nn.functional.mse_loss(out_ref["forces"], f_target.double())).backward()
    opt_ref.step()
    out = m._train_schnet_with(runner, _OracleForces(out_ref["forces"].detach()), z.to(torch.int32), pos.float().contiguous(), mol_ptr, n_mol)
    (torch.nn.functional.mse_loss(out["energy"], target) + torch.nn.functional.mse_loss(out["forces"], f_target)).backward()
    opt.step()
    refp = dict(ref.named_parameters())
    for name, p in m.named_parameters():
        moved = (refp[name].detach() - sd0[name].double()).abs().max().item()
        assert (p.detach().double() - refp[name].detach()).abs().max() <= 5e-5 * moved + 1e-8, (name, moved)
    assert max((refp[n].detach() - sd0[n].double()).abs().max().item() for n in refp) > 1e-4  # the step did move the weights


def test_schnet_train_c_abi_argument_checks(runner):
    """Null pointers, a short workspace and a missing gradient struct are refused with NB200_EINVAL before any launch; the size function of
    libnabla_b200.so (pure host code) agrees with the emulation build up to the guard zones."""
    from ctypes import byref, c_int64

    from nabladft_b200 import _lib

    m, _ = _models(with_forces=False, n_interactions=2)
    tensors, scalars = m._export_schnet_impl(False, detach=True)
    w = runner._struct(tensors, scalars)
    z, pos, batch, idx_i, idx_j, mol_ptr, n_mol = _batch([3])
    z32, pos32, n = z.to(torch.int32), pos.float().contiguous(), z.shape[0]
    row_ptr, scratch, n_edges = torch.empty(n + 1, dtype=torch.int32), torch.empty(2 * n, dtype=torch.int32), c_int64(0)
    lib = runner.lib
    assert lib.nb200_schnet_train_count(byref(w), None, mol_ptr.data_ptr(), n_mol, n, row_ptr.data_ptr(), scratch.data_ptr(), byref(n_edges), None) == -1
    assert lib.nb200_schnet_train_count(byref(w), pos32.data_ptr(), mol_ptr.data_ptr(), n_mol, n, row_ptr.data_ptr(), scratch.data_ptr(), byref(n_edges), None) == 0
    assert n_edges.value == idx_i.numel() and int(row_ptr[-1]) == n_edges.value
    need = lib.nb200_schnet_train_workspace_bytes(byref(w), n_mol, n, n_edges.value, 0)
    need_t = lib.nb200_schnet_train_workspace_bytes(byref(w), n_mol, n, n_edges.value, 1)
    real = _lib.load()
    assert 0 < real.nb200_schnet_train_workspace_bytes(byref(w), n_mol, n, n_edges.value, 0) <= need < need_t
    assert real.nb200_schnet_train_workspace_bytes(byref(w), n_mol, n, -1, 0) == -1
    ws, energy, seed = torch.zeros(need, dtype=torch.uint8), torch.zeros(n_mol), torch.ones(n_mol)
    call = lambda ws_bytes, seed_ptr, grads_ptr: lib.nb200_schnet_energy_grads(
        runner._h, byref(w), z32.data_ptr(), pos32.data_ptr(), mol_ptr.data_ptr(), n_mol, n, row_ptr.data_ptr(), n_edges.value, ws.data_ptr(), ws_bytes,
        seed_ptr, None, grads_ptr, energy.data_ptr(), None)
    assert call(need - 1, None, None) == -1            # short workspace
    assert call(need, seed.data_ptr(), None) == -1     # a seed without gradient buffers
    assert call(need, None, None) == 0 and bool(torch.isfinite(energy).all())   # forward only
    lib.nb200_emu_check_guards()
