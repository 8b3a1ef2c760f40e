"""CPU checks of the DimeNet++ oracle (oracle/dimenet.py), the golden file of the reference's wrapper, the b200 yaml and the mirror's
state-dict contract (nabladft_b200/dimenetplusplus.py)."""
import hashlib
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_dimenet import SCALER, grid_molecule, load_test_weights  # noqa: E402

from oracle import dimenet as od  # noqa: E402


def test_bessel_zeros_normalizers_and_bases_against_scipy():
    from scipy.special import spherical_jn, sph_harm_y

    from nabladft_b200.dimenetplusplus import sbf_radial_constants

    z = od.bessel_zeros(7, 6)
    for l in range(7):
        assert np.abs(spherical_jn(l, z[l])).max() < 1e-12
        assert np.all(np.diff(z[l]) > 0) and z[l, 0] > l  # the first zeros, in order
    assert np.allclose(z[0], np.pi * np.arange(1, 7))
    norms = od.bessel_normalizers(z)
    assert np.allclose(norms, 1.0 / np.sqrt(0.5 * np.stack([spherical_jn(l + 1, z[l]) ** 2 for l in range(7)])), rtol=1e-14)
    zm, nm = sbf_radial_constants()  # the mirror's copy, which the engine receives
    assert np.allclose(zm, z, rtol=1e-13) and np.allclose(nm, norms, rtol=1e-12)
    x = torch.linspace(0.3, 30.0, 500, dtype=torch.float64)
    for l in range(7):
        assert np.allclose(od.spherical_jn_torch(l, x).numpy(), spherical_jn(l, x.numpy()), atol=1e-9)
    th = torch.linspace(0.0, math.pi, 101, dtype=torch.float64)
    Y = od.legendre_y0(7, torch.cos(th))
    for l in range(7):
        ref = sph_harm_y(l, 0, th.numpy(), 0.0).real
        assert np.allclose(Y[l].numpy(), ref, atol=1e-12)


def test_radius_graph_keeps_k_plus_one_candidates():
    z, pos = grid_molecule()
    ei = od.radius_graph_kp1(torch.from_numpy(pos).double(), torch.zeros(len(z), dtype=torch.long), 5.0, 32)
    deg = torch.bincount(ei[1], minlength=len(z))
    assert (deg[:33] == 32).all() and (deg[33:] == 33).all()  # atom 33 is not among its own first 33 candidates
    # sources ascending per target, no self loops, CSR by target
    assert (ei[0] != ei[1]).all() and bool((ei[1][1:] >= ei[1][:-1]).all())
    for a in (0, 40):
        s = ei[0][ei[1] == a]
        assert bool((s[1:] > s[:-1]).all())
    assert s.tolist() == list(range(33))  # atom 40 keeps its first 33 candidates, 0..32


def test_triplets_against_brute_force():
    from helpers import load_fixture

    z, pos, batch = load_fixture([2, 9])
    ei = od.radius_graph_kp1(pos, batch, 5.0, 32)
    i, j, idx_i, idx_j, idx_k, idx_kj, idx_ji = od.triplets(ei, len(z))
    src, tgt = ei[0].tolist(), ei[1].tolist()
    brute = []
    for e in range(len(src)):
        for kj in sorted((f for f in range(len(src)) if tgt[f] == src[e] and src[f] != tgt[e]), key=lambda f: src[f]):
            brute.append((kj, e))
    assert list(zip(idx_kj.tolist(), idx_ji.tolist())) == brute
    assert (idx_j == j[idx_ji]).all() and (idx_i == i[idx_ji]).all() and (idx_k == j[idx_kj]).all()


def test_oracle_forces_are_minus_energy_gradient():
    from helpers import load_fixture

    ora = load_test_weights(od.DimeNetPlusPlusPotentialOracle(dimenet_num_blocks=2, scaler=SCALER, do_postprocessing=True).double().eval())
    z, pos, batch = load_fixture([4])
    _, f, _ = ora(z, pos, batch)
    h = 1e-5
    for a, t in ((0, 0), (3, 2), (7, 1)):
        pp, pm = pos.clone(), pos.clone()
        pp[a, t] += h
        pm[a, t] -= h
        ep, _, _ = ora(z, pp, batch)
        em, _, _ = ora(z, pm, batch)
        fd = -(ep - em).item() / (2 * h) / SCALER["scale_"]  # forces come from the UNSCALED prediction (dimenetplusplus.py:97-112)
        assert abs(fd - f[a, t].item()) < 1e-7 * max(1.0, abs(fd)), (a, t, fd, f[a, t].item())


def test_oracle_matches_golden_of_reference_wrapper():
    g = np.load(os.path.join(HERE, "golden", "dimenet_f64.npz"))
    ora = load_test_weights(od.DimeNetPlusPlusPotentialOracle(scaler=SCALER, do_postprocessing=True).double().eval())
    e, f, emb = ora(torch.from_numpy(g["z"]).long(), torch.from_numpy(g["pos"]).double(), torch.from_numpy(g["batch"]))
    assert np.abs(e.numpy() - g["energy"]).max() < 1e-10
    assert np.abs(f.numpy() - g["forces"]).max() < 1e-10
    assert np.abs(emb.numpy() - g["graph_emb"]).max() < 1e-10
    assert np.ptp(g["energy"]) > 0.3 and np.abs(g["forces"]).max() > 0.1  # the test weights make the model respond


def test_b200_yaml_matches_reference_and_instantiates():
    import importlib

    import yaml

    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "dimenetplusplus-b200.yaml")))
    ref = json.load(open(os.path.join(HERE, "golden", "reference_dimenet_yaml.json")))["dimenetplusplus.yaml"]

    def strip(node):
        if isinstance(node, dict):
            return {k: ("<cls>" if k == "_target_" and str(v).startswith(("nabladft_b200.", "nablaDFT.")) else strip(v)) for k, v in node.items()}
        return [strip(v) for v in node] if isinstance(node, list) else node

    assert list(cfg.keys()) == ref["top_level_keys"]
    assert hashlib.sha256(json.dumps(strip(cfg), sort_keys=True, default=str).encode()).hexdigest() == ref["sha256_without_model_targets"]
    assert cfg["_target_"] == "nablaDFT.dimenetplusplus.DimeNetPlusPlusLightning"
    net_cfg = dict(cfg["net"])
    mod, name = net_cfg.pop("_target_").rsplit(".", 1)
    assert mod == "nabladft_b200.dimenetplusplus"
    model = getattr(importlib.import_module(mod), name)(**net_cfg)
    assert model.num_blocks == 6 and model.node_latent_dim == 50 and model._scale_mean() == (SCALER["scale_"], SCALER["mean_"])


def test_mirror_state_dict_matches_oracle_and_loads_strict():
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential

    kw = dict(node_latent_dim=50, scaler=SCALER, dimenet_hidden_channels=256, dimenet_num_blocks=6, do_postprocessing=True)
    net = DimeNetPlusPlusPotential(**kw)
    ora = od.DimeNetPlusPlusPotentialOracle(**kw)
    a, b = net.state_dict(), ora.state_dict()
    assert list(a) == list(b) and all(a[k].shape == b[k].shape for k in a)
    assert "net.rbf.freq" in a and "regr_or_cls_nn.6.bias" in a and "net.interaction_blocks.5.layers_after_skip.1.lin2.weight" in a
    load_test_weights(ora)
    net.load_state_dict(ora.state_dict(), strict=True)
    assert all(torch.equal(net.state_dict()[k], ora.state_dict()[k].float()) for k in a)
    buf, offs = net.export(torch.device("cpu"))
    assert len(offs) == 16 + 14 * 6 + 5 * 7 and buf.dtype == torch.float32
    with pytest.raises(NablaB200Error):
        DimeNetPlusPlusPotential(node_latent_dim=50, dimenet_hidden_channels=128)  # the reference's default width is not built
    net.train()
    with pytest.raises(NotImplementedError):
        net(type("D", (), dict(z=torch.zeros(2, dtype=torch.long), pos=torch.zeros(2, 3), batch=torch.zeros(2, dtype=torch.long)))())
