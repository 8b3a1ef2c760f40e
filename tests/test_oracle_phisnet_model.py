"""The float64 CPU oracle of the whole PhiSNet model (oracle/phisnet_model.py) against the reference's own NeuralNetwork
(tests/golden/phisnet_model.npz, make_golden_phisnet_model.py), and the O(P) neighbour sum of the pair features against the reference's
pindex gather, both evaluated by the oracle."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden_phisnet_model import HYPER, max_orbitals_from_db, model_state_dict  # noqa: E402

from oracle.phisnet_model import NeuralNetwork  # noqa: E402

G = np.load(os.path.join(GOLDEN, "phisnet_model.npz"))
TAGS = ("full", "core", "over")


def oracle():
    m = NeuralNetwork(max_orbitals_from_db(), **HYPER).double()
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in model_state_dict(sd).items()}, strict=True)
    return m.eval()


@pytest.fixture(scope="module")
def ora():
    return oracle()


def golden_inputs():
    return torch.from_numpy(G["positions"]), torch.from_numpy(G["atomic_numbers"]), [int(s) for s in G["molecule_size"]]


def test_oracle_state_dict_names_equal_reference(ora):
    assert sorted(ora.state_dict()) == list(G["state_keys"])


def test_oracle_matches_reference_golden(ora):
    out = ora(*golden_inputs())
    for m in range(2):
        for tag in TAGS:
            got = out[tag][m].numpy()
            ref = G[f"{tag}/{m}"]
            tri = got[np.triu_indices(got.shape[0])]
            err = np.abs(tri - ref).max() / np.abs(ref).max()
            assert err <= 1e-10, (m, tag, err)


def test_oracle_neighbour_sum_equals_pindex_formulation(ora):
    """The O(P) T_i - own term form and the reference's pindex gather give the same pair features (and the same matrices)."""
    pos, z, sizes = golden_inputs()
    idx_pi, idx_pj, off = [], [], 0
    for n in sizes:
        idx_pi.append(torch.from_numpy(G[f"pindex/{n}/i"]).long() + off)
        idx_pj.append(torch.from_numpy(G[f"pindex/{n}/j"]).long() + off)
        off += n * (n - 1)
    pindex = (torch.cat(idx_pi), torch.cat(idx_pj))
    idx_i, idx_j = ora.pairs(sizes)
    gen = torch.Generator().manual_seed(0)
    F, P = HYPER["num_features"], len(idx_i)
    fij = [torch.randn(P, 2 * L + 1, F, generator=gen, dtype=torch.float64) for L in range(5)]
    fpn = [torch.randn(len(z), 2 * L + 1, F, generator=gen, dtype=torch.float64) for L in range(5)]
    rbf = torch.rand(P, 1, HYPER["num_basis_functions"], generator=gen, dtype=torch.float64)
    a = ora.pair_neighbour_sum(fij, fpn, rbf, idx_i, idx_j)
    b = ora.pair_neighbour_sum(fij, fpn, rbf, idx_i, idx_j, pindex)
    for x, y in zip(a, b):
        assert torch.allclose(x, y, rtol=0, atol=1e-12)
    full_p = ora(pos, z, sizes, pindex=pindex, heads=("full",))["full"]
    full = ora(pos, z, sizes, heads=("full",))["full"]
    for x, y in zip(full, full_p):
        assert torch.allclose(x, y, rtol=0, atol=1e-11 * float(y.abs().max()))
