"""Host-side pieces of the PhiSNet model mirror (nabladft_b200.phisnet.NeuralNetwork), pinned to the reference's own NeuralNetwork
(tests/golden/phisnet_model.npz, written by tests/golden/make_golden_phisnet_model.py): computed electron-configuration table, module tree /
state-dict names and shapes, the irreps and assembly tables, and the O(P) rewrite of the reference's pindex sum."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden_phisnet_model import HYPER, max_orbitals_from_db, model_state_dict  # noqa: E402

from nabladft_b200 import phisnet as ph  # noqa: E402

G = np.load(os.path.join(GOLDEN, "phisnet_model.npz"))


@pytest.fixture(scope="module")
def net():
    return ph.NeuralNetwork(max_orbitals=max_orbitals_from_db(), **HYPER)


def test_electron_config_table_equals_reference():
    t = ph.electron_configurations()
    assert t.dtype == torch.float32 and tuple(t.shape) == (87, 16)
    assert np.array_equal(t.numpy().astype(np.float64), G["electron_config"])


def test_state_dict_names_and_shapes_equal_reference(net):
    sd = net.state_dict()
    assert sorted(sd) == list(G["state_keys"])
    for k, shape in zip(G["state_keys"], G["state_shapes"]):
        assert ",".join(str(s) for s in sd[k].shape) == shape, k
    vals = model_state_dict(sd)
    res = net.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in vals.items()}, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    # a reference state dict also carries the CG-table buffers: they are accepted and ignored
    extra = dict(net.state_dict())
    extra["module.0.interaction.mixing.clebsch_gordan.cg_0_0_0"] = torch.zeros(1)
    net.load_state_dict(extra, strict=True)


def test_irreps_tables_reproduce_compute_matrix_irreps(net):
    ii, w_ii, ij, w_ij = ph.irreps_tables(max_orbitals_from_db())
    assert (w_ii, w_ij) == (258, 1810)
    assert net.output_full_ii.num_out == 258 and net.output_full_ij.num_out == 1810
    # first-seen numbering per L, as compute_matrix_irreps does it (keys of each element pair in (n_i, n_j, L) order)
    assert ii[(1, 1, 0, 0, 0)] == 0 and ij[(1, 1, 0, 0, 0)] == 0
    for table, width in ((ii, w_ii), (ij, w_ij)):
        per_L = {}
        for (_, _, _, _, L), c in table.items():
            per_L.setdefault(L, []).append(c)
        for cs in per_L.values():
            assert sorted(cs) == list(range(len(cs)))
        assert max(len(c) for c in per_L.values()) == width


def test_assembly_tables_cover_every_block(net):
    a = net._asm
    assert not a["missing"]
    for kind, table in ((0, net.irreps_ii), (1, net.irreps_ij)):
        orbs = {o[0][0]: o for o in net.max_orbitals}
        for ea, za in enumerate(a["elems"]):
            for eb, zb in enumerate(a["elems"]):
                if kind == 0 and ea != eb:
                    continue
                k0, k1 = a["ent_range"][kind, ea, eb]
                want = [(table[(za, zb, si, sj, L)], L) for si, (_, li) in enumerate(orbs[za]) for sj, (_, lj) in enumerate(orbs[zb])
                        for L in range(abs(li - lj), li + lj + 1)]
                assert list(zip(a["ent_col"][k0:k1], a["ent_L"][k0:k1])) == want
                assert a["n_rows"][ea] == sum(2 * l + 1 for _, l in orbs[za])


@pytest.mark.parametrize("n", [10, 14])
def test_pair_sum_rewrite_equals_pindex_formulation(n):
    """sum_{k != i,j} radial(rbf_ik) fpn[k]  ==  T_i - radial(rbf_ij) fpn[j],  T_i = sum_{k != i} ..., against the reference's pindex lists."""
    pi, pj = G[f"pindex/{n}/i"], G[f"pindex/{n}/j"]
    gen = torch.Generator().manual_seed(n)
    idx_i = torch.tensor([i for i in range(n) for j in range(n) if i != j])
    idx_j = torch.tensor([j for i in range(n) for j in range(n) if i != j])
    fpn_j = torch.randn(len(idx_i), 7, generator=gen, dtype=torch.float64)  # radial(rbf_ij) * fpn[j] per ordered pair
    ref = torch.zeros_like(fpn_j).index_add(0, torch.from_numpy(pi).long(), fpn_j[torch.from_numpy(pj).long()])
    T = torch.zeros(n, 7, dtype=torch.float64).index_add(0, idx_i, fpn_j)
    assert torch.allclose(T[idx_i] - fpn_j, ref, rtol=0, atol=1e-12)
