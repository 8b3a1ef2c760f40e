"""GPU tests of the whole PhiSNet model (nabladft_b200.phisnet.NeuralNetwork) against the reference's own NeuralNetwork run in float64 at the
shipped hyperparameters on a two-molecule batch of fixture molecule 0 (tests/golden/phisnet_model.npz): full, core and overlap matrices,
dense and packed; structure (block diagonal, exact symmetry, unit overlap diagonal); rotation / permutation invariance of the spectra;
determinism; batch independence; the head flags and the error paths."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden_phisnet_model import HYPER, max_orbitals_from_db, model_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "phisnet_model.npz"))
REL = 1e-5  # of each matrix's largest entry
DEV = "cuda:0"
KEYS = (("full", "full_hamiltonian"), ("core", "core_hamiltonian"), ("over", "overlap_matrix"))


@pytest.fixture(scope="module")
def net():
    from nabladft_b200 import phisnet as ph

    m = ph.NeuralNetwork(max_orbitals=max_orbitals_from_db(), **HYPER)
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in model_state_dict(sd).items()}, strict=True)
    return m.to(DEV).eval()


def orbitals_of(net, z):
    table = {o[0][0]: o for o in net.max_orbitals}
    return tuple(table[int(a)] for a in z)


def batch_of(net, pos, z, sizes):
    return {"positions": torch.as_tensor(pos, dtype=torch.float32).to(DEV), "atomic_numbers": torch.as_tensor(z).long().to(DEV),
            "orbitals": orbitals_of(net, z), "molecule_size": torch.as_tensor(sizes).long()}


def golden_batch(net):
    return batch_of(net, G["positions"], G["atomic_numbers"], G["molecule_size"])


def full_sym(tri, n):
    m = np.zeros((n, n))
    iu = np.triu_indices(n)
    m[iu] = tri
    m.T[iu] = tri
    return m


def rel_err(got, ref):
    return float(np.abs(got - ref).max() / np.abs(ref).max())


def test_golden_parity_packed_and_dense(net):
    out = net(golden_batch(net), packed=True)
    dense = net(golden_batch(net))
    off = 0
    for m in range(2):
        for tag, key in KEYS:
            got = out[key][m].double().cpu().numpy()
            ref = full_sym(G[f"{tag}/{m}"], got.shape[0])
            err = rel_err(got, ref)
            print(f"mol {m} {tag}: max err / max|ref| = {err:.2e}")
            assert err < REL, (m, tag, err)
            assert torch.equal(out[key][m], out[key][m].T)
            d = dense[key][0]
            n = got.shape[0]
            assert torch.equal(d[off:off + n, off:off + n], out[key][m])
        assert torch.all(torch.diagonal(out["overlap_matrix"][m]) == 1)
        off += out["full_hamiltonian"][m].shape[0]
    n0 = out["full_hamiltonian"][0].shape[0]
    for _, key in KEYS:
        d = dense[key][0]
        assert d.shape[0] == off and torch.count_nonzero(d[:n0, n0:]) == 0 and torch.count_nonzero(d[n0:, :n0]) == 0
    assert dense["energy"].shape == (1, 1) and torch.count_nonzero(dense["energy"]) == 0
    assert dense["forces"].shape == (G["positions"].shape[0], 3) and dense["orbital_coefficients"].shape == dense["full_hamiltonian"].shape
    assert dense["orbital_energies"].shape == (1, off)


def spectra(mats):
    return [torch.linalg.eigvalsh(m.double()).cpu().numpy() for m in mats]


def test_rotation_and_permutation_invariance(net):
    b = golden_batch(net)
    base = net(b, packed=True)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(3), dtype=torch.float64))
    rb = dict(b, positions=(b["positions"].double() @ q.to(DEV).T).float())
    rot = net(rb, packed=True)
    sizes = [int(s) for s in G["molecule_size"]]
    perm = torch.cat([torch.randperm(sizes[0], generator=torch.Generator().manual_seed(5)),
                      sizes[0] + torch.randperm(sizes[1], generator=torch.Generator().manual_seed(6))])
    z = G["atomic_numbers"][perm.numpy()]
    pb = batch_of(net, G["positions"][perm.numpy()], z, G["molecule_size"])
    per = net(pb, packed=True)
    for _, key in KEYS:
        for a, r, p in zip(spectra(base[key]), spectra(rot[key]), spectra(per[key])):
            scale = np.abs(a).max()
            assert np.abs(a - r).max() < 2e-5 * scale and np.abs(a - p).max() < 2e-5 * scale


def test_deterministic_and_batch_independent(net):
    b = golden_batch(net)
    o1, o2 = net(b, packed=True), net(b, packed=True)
    for _, key in KEYS:
        for a, c in zip(o1[key], o2[key]):
            assert torch.equal(a, c)
    # molecule 1 alone, and inside a batch together with a copy of molecule 0
    n0 = int(G["molecule_size"][0])
    solo = net(batch_of(net, G["positions"][n0:], G["atomic_numbers"][n0:], [G["molecule_size"][1]]), packed=True)
    pos = np.concatenate([G["positions"][n0:], G["positions"]])
    z = np.concatenate([G["atomic_numbers"][n0:], G["atomic_numbers"]])
    trio = net(batch_of(net, pos, z, [G["molecule_size"][1], *G["molecule_size"]]), packed=True)
    for _, key in KEYS:
        assert torch.equal(solo[key][0], o1[key][1])
        assert torch.equal(trio[key][0], solo[key][0]) and torch.equal(trio[key][2], o1[key][1])


def test_flags_return_identity(net):
    b = golden_batch(net)
    ref = net(b, packed=True)
    net.calculate_core_hamiltonian = False
    net.calculate_overlap_matrix = False
    try:
        out = net(b, packed=True)
        for m in range(2):
            n = out["full_hamiltonian"][m].shape[0]
            assert torch.equal(out["core_hamiltonian"][m], torch.eye(n, device=DEV))
            assert torch.equal(out["overlap_matrix"][m], torch.eye(n, device=DEV))
            assert torch.equal(out["full_hamiltonian"][m], ref["full_hamiltonian"][m])
    finally:
        net.calculate_core_hamiltonian = net.calculate_overlap_matrix = True


def test_errors(net):
    from nabladft_b200._lib import NablaB200Error

    b = golden_batch(net)
    with pytest.raises(NablaB200Error, match="CUDA only"):
        net(dict(b, positions=b["positions"].cpu()))
    for flag in ("predict_energy", "calculate_forces"):
        setattr(net, flag, True)
        try:
            with pytest.raises(NotImplementedError):
                net(b)
        finally:
            setattr(net, flag, False)
    z = b["atomic_numbers"].clone()
    z[0] = 5  # boron is not in the fixture DB's max_orbitals
    with pytest.raises(ValueError, match="max_orbitals"):
        net(dict(b, atomic_numbers=z))
    bad = list(b["orbitals"])
    bad[0] = bad[-1]  # a carbon given hydrogen's orbitals
    with pytest.raises(ValueError, match="orbitals"):
        net(dict(b, orbitals=tuple(bad)))
    net.train()
    try:
        with pytest.raises(NotImplementedError):
            net(b)
    finally:
        net.eval()


def test_oracle_parity_full_fixture_molecule_and_synthetic(net):
    """Sizes the golden does not cover: all 38 atoms of fixture molecule 0 plus two synthetic molecules, against the float64 oracle."""
    from nabladft_b200.data import read_hamiltonian_db
    from nabladft_b200.synth import synth_batch
    from oracle.phisnet_model import NeuralNetwork as Oracle

    db = read_hamiltonian_db(os.path.join(GOLDEN, "hamiltonian_mol0.db"))
    sb = synth_batch(7, 2, heavy_min=8, heavy_max=12)
    pos = np.concatenate([db["pos"].astype(np.float64), sb["pos"].astype(np.float64) * 1.8897261])
    z = np.concatenate([db["z"], sb["z"]]).astype(np.int64)
    sizes = [len(db["z"])] + np.diff(sb["mol_ptr"]).tolist()
    got = net(batch_of(net, pos, z, sizes), packed=True)
    ora = Oracle(max_orbitals_from_db(), **HYPER).double()
    ora.load_state_dict({k: v.detach().cpu().double() for k, v in net.state_dict().items()}, strict=True)
    ref = ora(torch.from_numpy(pos), torch.from_numpy(z), sizes)
    for tag, key in KEYS:
        for m in range(len(sizes)):
            err = rel_err(got[key][m].double().cpu().numpy(), ref[tag][m].numpy())
            print(f"oracle parity mol {m} ({sizes[m]} atoms) {tag}: {err:.2e}")
            assert err < REL, (tag, m, err)
