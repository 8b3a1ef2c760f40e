"""GemNet-OC engine source (nabladft_b200/csrc/gemnet_oc.cu) checked on the CPU through its host-emulation build (tests/emu): the SAME
functors the GPU launches, run as loops, driven through the SAME C ABI and the SAME Python host code (export of the reference-named weights,
two-phase graph/workspace protocol), compared with the pinned oracle (oracle/gemnet_oc.py) and the golden outputs of the reference's own
classes.  This validates index logic, bases, weight layout and scale folding without a GPU; it says nothing about launch configuration or the
tensor-core GEMM, which only `-m gpu` covers.  The emulation library is test infrastructure -- the package never loads it."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.gemnet_oc import GemNetOCRunner

    lib = load("gemnet_oc", ["nb200_gemnet_oc_"])
    EmuRunner = poisoned(GemNetOCRunner, checked=["run", "run_train"])
    return lambda: EmuRunner(lib)


def _yaml_kwargs():
    import yaml

    cfg = yaml.safe_load(open(os.path.join(HERE, "..", "config", "model", "gemnet-oc-b200.yaml")))["net"]
    cfg.pop("_target_")
    return cfg


def _models(scales: bool):
    """The product module and the oracle with the same name-keyed golden weights (scale factors 1, or random in [0.5, 1.5])."""
    from weights import golden_state_dict

    from nabladft_b200.gemnet_oc import GemNetOC
    from oracle.gemnet_oc import GemNetOCOracle

    net = GemNetOC(**_yaml_kwargs()).eval()
    ora = GemNetOCOracle().float().eval()
    sd = ora.state_dict()
    assert set(sd) == set(net.state_dict()) and len(sd) == 429
    new = golden_state_dict(sd, bias_std=0.02, weight_scale=0.5)
    rng = np.random.default_rng(5)
    shared = {}
    for k in sd:
        if k.endswith("scale_factor"):
            # the three parents of `radial_basis_spherical` hold ONE parameter in the reference
            grp = "sph" if k in ("sbf_basis_qint.radial_basis.scale_rbf.scale_factor", "cbf_basis_aeint.radial_basis.scale_rbf.scale_factor",
                                 "cbf_basis_tint.radial_basis.scale_rbf.scale_factor") else k
            if grp not in shared:
                shared[grp] = float(rng.uniform(0.5, 1.5)) if scales else 1.0
            sd[k] = torch.tensor(shared[grp])
        elif k in new:
            sd[k] = torch.as_tensor(np.asarray(new[k])).float().reshape(sd[k].shape)
    ora.load_state_dict(sd, strict=True)
    net.load_state_dict(sd, strict=True)
    return net, ora


def _run(emu, net, z, pos, batch):
    r = emu()
    r.set_weights(net, torch.device("cpu"))
    n_mol = int(batch.max()) + 1
    cnt = torch.bincount(batch, minlength=n_mol)
    mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32)
    mol_ptr[1:] = torch.cumsum(cnt, 0)
    out = r.run(z.to(torch.int32).contiguous(), pos.float().contiguous(), mol_ptr, n_mol, int(cnt.max()), return_h=True)
    return out, r.last_counts


def test_emu_graph_counts_match_reference_indices(emu):
    """Edge counts of the four graphs and the number of input-triplet slots against the index arrays of the reference's own classes."""
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    net, _ = _models(False)
    (_, _, _), counts = _run(emu, net, torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"]))
    assert counts["MAIN"] == int(g["main_edges"]) and counts["A2A"] == int(g["a2a_edges"])
    assert counts["AE"] == int(g["a2ee2a_edges"]) and counts["Q"] == int(g["qint_edges"])
    # one slot per (qint edge b->a, main edge into b); the reference drops the d == a pairs: at most one per qint edge
    n_tin = int(g["quad/triplet_in/in"].shape[0])
    assert n_tin <= counts["TIN"] <= n_tin + counts["Q"]


def test_emu_matches_reference_golden_outputs(emu):
    """Energies, forces and the final atom embedding against what the reference's own GemNet-OC classes produced (float32, scale factors 1)."""
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    net, _ = _models(False)
    (E, F, h), _ = _run(emu, net, torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"]))
    assert np.abs(h.numpy() - g["int3/h"]).max() < 2e-4 * np.abs(g["int3/h"]).max()
    assert np.abs(E.numpy() - g["energy"].reshape(-1)).max() < 2e-4 * np.abs(g["energy"]).max()
    assert np.abs(F.numpy() - g["forces"]).max() < 2e-4 * np.abs(g["forces"]).max()


def test_emu_matches_oracle_with_fitted_scale_factors(emu):
    """Second batch (three molecules), every scale factor different from 1: exercises the folding of the basis scales into the concatenated
    matrices and the per-block factors.  The oracle is pinned at scale 1; a scale factor is one multiplication (scale_factor.py:139-154)."""
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    z, pos, batch = torch.from_numpy(g["b2/z"]), torch.from_numpy(g["b2/pos"]), torch.from_numpy(g["b2/batch"])
    net, ora = _models(True)
    with torch.no_grad():
        E0, F0 = ora(z, pos, batch)
    (E, F, h), _ = _run(emu, net, z, pos, batch)
    assert np.abs(h.numpy() - ora.trace["int3/h"].numpy()).max() < 2e-4 * np.abs(ora.trace["int3/h"].numpy()).max()
    assert np.abs(E.numpy() - E0.numpy()).max() < 2e-4 * np.abs(E0.numpy()).max()
    assert np.abs(F.numpy() - F0.numpy()).max() < 2e-4 * np.abs(F0.numpy()).max()


def test_emu_module_forward_host_logic(emu):
    """GemNetOC._forward_with (everything forward() does after its CUDA check) driven with the emulation runner: weight re-export when a
    parameter changes, molecule pointers, unsorted-batch refusal."""
    from nabladft_b200._lib import NablaB200Error

    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    net, _ = _models(False)

    class D:
        z, pos, batch = torch.from_numpy(g["z"]).long(), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"]).long()

    r = emu()
    E, F = net._forward_with(r, D())
    assert np.abs(E.numpy() - g["energy"].reshape(-1)).max() < 2e-4 * np.abs(g["energy"]).max()
    with torch.no_grad():
        net.out_energy.linear.weight.mul_(2.0)   # in-place update, as an optimiser step or a checkpoint load does
    E2, F2 = net._forward_with(r, D())
    assert np.allclose(E2.numpy(), 2.0 * E.numpy(), rtol=1e-5) and np.allclose(F2.numpy(), F.numpy(), atol=1e-7)
    D.batch = torch.flip(D.batch, [0])
    with pytest.raises(NablaB200Error):
        net._forward_with(r, D())


def test_emu_ragged_batch_with_single_atom_and_diatomic_molecules(emu):
    """Seven molecules of 11 .. 53 atoms plus a lone atom (no edges at all) and a diatomic (one pair, no triplets): energies and forces
    against the oracle, scale factors != 1."""
    from nabladft_b200.synth import synth_batch

    b = synth_batch(11, 5, heavy_min=3, heavy_max=30)
    z = torch.from_numpy(np.concatenate([b["z"], [8], [1, 1]])).long()
    pos = torch.from_numpy(np.concatenate([b["pos"], [[0, 0, 0]], [[0, 0, 0], [0.74, 0, 0]]]).astype(np.float32))
    batch = torch.from_numpy(np.concatenate([b["batch"], [5], [6, 6]])).long()
    net, ora = _models(True)
    with torch.no_grad():
        E0, F0 = ora(z, pos, batch)
    (E, F, _), counts = _run(emu, net, z, pos, batch)
    d2 = ((pos[:, None, :] - pos[None, :, :]) ** 2).sum(-1)
    same = (batch[:, None] == batch[None, :]) & ~torch.eye(len(z), dtype=torch.bool)
    assert counts["A2A"] == int(((d2 < 144.0) & same).sum()) < int(same.sum())  # the largest molecule is wider than the 12 A cutoff
    assert np.abs(E.numpy() - E0.numpy()).max() < 2e-6 * max(1.0, np.abs(E0.numpy()).max())
    assert np.abs(F.numpy() - F0.numpy()).max() < 2e-5 * np.abs(F0.numpy()).max()
    assert np.abs(F.numpy()[-3]).max() == 0.0  # the lone atom feels no force


def test_emu_reference_style_pyg_model_gemnet_oc(emu):
    """The reference's own `test_pyg_model[GemNet-OC]` (tests/model/test_torch_models.py:9-27) restated: a one-molecule PyG-style batch from
    our data path, `energy.shape == batch.y.shape`, `forces.shape == batch.forces.shape` (host code + emulated engine; the device variant
    is tests/test_zz_gpu_first_runs.py)."""
    from nabladft_b200.data import DeviceBatcher, PackedEnergyDataset

    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    ds = PackedEnergyDataset(fx["z"].astype(np.int32), fx["pos"].astype(np.float32), fx["forces"].astype(np.float32), fx["energy"].astype(np.float32),
                             fx["ptr"].astype(np.int64))
    batch = next(iter(DeviceBatcher(ds, batch_size=1, device="cpu"))).as_pyg()
    net, _ = _models(False)
    energy, forces = net._forward_with(emu(), batch)
    assert energy.shape == batch.y.shape and forces.shape == batch.forces.shape
    assert bool(torch.isfinite(energy).all() and torch.isfinite(forces).all())


def test_c_abi_argument_checks_and_size_functions_agree_with_the_cuda_library(emu):
    """Error behaviour of the C ABI (same source in both builds): null pointers / short buffers -> NB200_EINVAL before any launch; the pure
    host size functions of libnabla_b200.so (callable without a GPU) return what the emulation build returns."""
    from ctypes import byref, c_int64

    from nabladft_b200 import _lib
    from nabladft_b200.gemnet_oc import N_COUNTS

    net, _ = _models(False)
    r = emu()
    r.set_weights(net, torch.device("cpu"))
    real = _lib.load()
    counts = (c_int64 * N_COUNTS)(3034, 2350, 1580, 632, 19215, 0, 0, 0)
    for n, mx in ((79, 40), (1, 1), (25000, 60)):
        # the emulation build adds a 1 KB guard zone behind each of the six arrays of the graph buffer
        assert 0 < real.nb200_gemnet_oc_graph_bytes(n, mx) == r.lib.nb200_gemnet_oc_graph_bytes(n, mx) - 6 * 1024
    assert real.nb200_gemnet_oc_graph_bytes(-1, 4) == -1 and real.nb200_gemnet_oc_graph_bytes(4, 0) == -1
    wb = r.lib.nb200_gemnet_oc_workspace_bytes(byref(r._w), 2, 79, counts)
    wb_real = real.nb200_gemnet_oc_workspace_bytes(byref(r._w), 2, 79, counts)
    assert wb > wb_real > 2350 * 512 * 4 * 8 and (wb - wb_real) % 1024 == 0 and wb - wb_real < 64 * 1024
    assert real.nb200_gemnet_oc_workspace_bytes(None, 2, 79, counts) == -1
    # phase 1 with a graph buffer that is too small, phase 2 with a workspace that is too small: refused, nothing touched
    z, pos = torch.ones(4, dtype=torch.int32), torch.rand(4, 3)
    mol_ptr = torch.tensor([0, 4], dtype=torch.int32)
    small = torch.zeros(64, dtype=torch.uint8)
    out = (c_int64 * N_COUNTS)()
    assert r.lib.nb200_gemnet_oc_graph_count(byref(r._w), pos.data_ptr(), mol_ptr.data_ptr(), 1, 4, 4, small.data_ptr(), small.numel(), out, None) == -1
    assert r.lib.nb200_gemnet_oc_graph_count(byref(r._w), None, mol_ptr.data_ptr(), 1, 4, 4, small.data_ptr(), small.numel(), out, None) == -1
    gb = torch.zeros(r.lib.nb200_gemnet_oc_graph_bytes(4, 4), dtype=torch.uint8)
    assert r.lib.nb200_gemnet_oc_graph_count(byref(r._w), pos.data_ptr(), mol_ptr.data_ptr(), 1, 4, 4, gb.data_ptr(), gb.numel(), out, None) == 0
    assert [out[k] for k in range(4)] == [12, 12, 12, 12]  # four atoms inside every cutoff: all ordered pairs in all four graphs
    e, f = torch.zeros(1), torch.zeros(4, 3)
    assert r.lib.nb200_gemnet_oc_energy_forces(r._h, byref(r._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), 1, 4, 4, gb.data_ptr(), gb.numel(), out,
                                               small.data_ptr(), small.numel(), e.data_ptr(), f.data_ptr(), None) == -1
