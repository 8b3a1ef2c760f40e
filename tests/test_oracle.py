"""CPU tests: the oracle against the golden vectors produced by the reference's own code,
plus the value-level properties the reference's suite lacks (SURVEY.md §4)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_fixture, load_golden_weights, random_rotation
from oracle.graph import ase_neighbor_list, batch_to_ptr, radius_graph
from oracle.painn_oc import PaiNNOC
from oracle.spk import NeuralNetworkPotential, SpkPaiNN, SpkSchNet


def _oc(dtype):
    torch.set_default_dtype(dtype)
    try:
        net = load_golden_weights(PaiNNOC().to(dtype), dtype)
    finally:
        torch.set_default_dtype(torch.float32)
    return net.eval()


@pytest.mark.parametrize("tag,dtype,etol,ftol", [("f64", torch.float64, 1e-9, 1e-9), ("f32", torch.float32, 2e-5, 2e-5)])
def test_painn_oc_oracle_matches_reference_golden(tag, dtype, etol, ftol):
    g = np.load(os.path.join(GOLDEN, f"painn_oc_{tag}.npz"))
    net = _oc(dtype)
    e, f = net(torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"]))
    assert np.abs(e.detach().numpy() - g["energy"]).max() < etol * max(1.0, np.abs(g["energy"]).max())
    assert np.abs(f.detach().numpy() - g["forces"]).max() < ftol


def test_painn_oc_fp32_vs_fp64_within_north_star_tolerance():
    g = np.load(os.path.join(GOLDEN, "painn_oc_f64.npz"))
    net = _oc(torch.float32)
    e, f = net(torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]).float(), torch.from_numpy(g["batch"]))
    assert np.abs(e.detach().numpy() - g["energy"]).max() < 1e-4  # fp32 eager itself: ~1e-5 at |E|~10
    assert np.abs(f.detach().numpy() - g["forces"]).max() < 1e-4


def test_radius_graph_semantics():
    z, pos, batch = load_fixture([0, 1])
    ei = radius_graph(pos, 5.0, batch, 100)
    j, i = ei
    assert (batch[j] == batch[i]).all() and (j != i).all()
    d = (pos[j] - pos[i]).norm(dim=1)
    assert (d < 5.0).all()
    assert (i[1:] >= i[:-1]).all()  # grouped by target
    # symmetric when uncapped
    fwd = set(zip(j.tolist(), i.tolist()))
    assert all((b, a) in fwd for a, b in fwd)
    # cap keeps the first K sources in ascending order
    ei3 = radius_graph(pos, 5.0, batch, 3)
    for t in range(5):
        full = j[i == t]
        assert ei3[0][ei3[1] == t].tolist() == full[:3].tolist()
    n_pairs = sum(int(((pos[batch == m][:, None] - pos[batch == m][None]).norm(dim=-1) < 5.0).sum()) - int((batch == m).sum()) for m in range(2))
    assert ei.shape[1] == n_pairs


def test_painn_oc_symmetries_and_finite_difference_forces():
    net = _oc(torch.float64)
    z, pos, batch = load_fixture([3])
    e0, f0 = net(z, pos.clone(), batch)
    R = random_rotation(1)
    e1, f1 = net(z, (pos @ R.T + 0.37).clone(), batch)
    assert torch.allclose(e0, e1, atol=1e-9)
    assert torch.allclose(f0 @ R.T, f1, atol=1e-9)
    perm = torch.randperm(z.numel(), generator=torch.Generator().manual_seed(0))
    e2, f2 = net(z[perm], pos[perm].clone(), batch[perm])
    assert torch.allclose(e0, e2, atol=1e-9) and torch.allclose(f0[perm], f2, atol=1e-9)
    h = 1e-5
    for a, c in ((0, 0), (7, 2), (20, 1)):
        p, m = pos.clone(), pos.clone()
        p[a, c] += h
        m[a, c] -= h
        fd = -(net(z, p, batch)[0] - net(z, m, batch)[0]) / (2 * h)
        assert abs(fd.item() - f0[a, c].item()) < 1e-6


def _spk_inputs(mols, dtype):
    z, pos, batch = load_fixture(mols, dtype)
    ptr = batch_to_ptr(batch)
    idx_i, idx_j = ase_neighbor_list(pos, ptr, 5.0)
    return {"_atomic_numbers": z, "_positions": pos, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}


@pytest.mark.parametrize("rep", [SpkPaiNN, SpkSchNet])
def test_spk_models_symmetries_and_fd_forces(rep):
    torch.set_default_dtype(torch.float64)
    try:
        model = load_golden_weights(NeuralNetworkPotential(rep()).double(), torch.float64).eval()
    finally:
        torch.set_default_dtype(torch.float32)
    model.postprocessors[0].mean.zero_()
    inp = _spk_inputs([2], torch.float64)
    out = model(dict(inp))
    assert out["energy"].shape == (1,) and out["forces"].shape == inp["_positions"].shape
    R = random_rotation(2)
    inp2 = dict(inp)
    inp2["_positions"] = (inp["_positions"].detach() @ R.T).clone()
    out2 = model(inp2)
    assert torch.allclose(out["energy"], out2["energy"], atol=1e-9)
    assert torch.allclose(out["forces"] @ R.T, out2["forces"], atol=1e-9)
    h = 1e-5
    for a, c in ((1, 0), (11, 2)):
        ip, im = dict(inp), dict(inp)
        ip["_positions"] = inp["_positions"].detach().clone()
        im["_positions"] = inp["_positions"].detach().clone()
        ip["_positions"][a, c] += h
        im["_positions"][a, c] -= h
        fd = -(model(ip)["energy"] - model(im)["energy"]) / (2 * h)
        assert abs(fd.item() - out["forces"][a, c].item()) < 1e-6
    # AddOffsets: eval-time E += mean * n_atoms (ase_model/task.py:43,63 call self(batch))
    model.postprocessors[0].mean.fill_(-0.25)
    out3 = model(dict(inp))
    n_atoms = inp["_atomic_numbers"].numel()
    assert torch.allclose(out3["energy"], out["energy"] - 0.25 * n_atoms, atol=1e-9)


def test_spk_painn_matches_painn_oc_roles():
    """spk PaiNNInteraction/Mixing and the in-repo PaiNNMessage/Update are one layer up to a
    relabelling of weight chunks (SURVEY.md A.2 vs A.3): pins the [3P-memory] restatement to
    the reference's in-repo code at layer level."""
    from oracle.painn_oc import MessageOC, UpdateOC
    from oracle.spk import _PaiNNInteraction, _PaiNNMixing

    torch.manual_seed(0)
    n, N, E = 16, 9, 40
    dt = torch.float64
    q, mu = torch.randn(N, n, dtype=dt), torch.randn(N, 3, n, dtype=dt)
    idx_i, idx_j = torch.randint(0, N, (E,)), torch.randint(0, N, (E,))
    Wij, dirs = torch.randn(E, 3 * n, dtype=dt), torch.randn(E, 3, dtype=dt)
    inter, mix = _PaiNNInteraction(n).double(), _PaiNNMixing(n).double()
    msg, upd = MessageOC(n, 5).double(), UpdateOC(n).double()
    for lin in (inter.interatomic_context_net[0], inter.interatomic_context_net[1], mix.intraatomic_context_net[0], mix.intraatomic_context_net[1]):
        lin.bias.data.normal_()
    swap = torch.cat([torch.arange(0, n), torch.arange(2 * n, 3 * n), torch.arange(n, 2 * n)])
    # message: OC chunk order (scalar, vec-term, dir-term) = spk (scalar, dir-term, vec-term) swapped
    msg.x_proj[0].load_state_dict(inter.interatomic_context_net[0].state_dict())
    msg.x_proj[2].weight.data = inter.interatomic_context_net[1].weight.data[swap]
    msg.x_proj[2].bias.data = inter.interatomic_context_net[1].bias.data[swap]
    q1, mu1 = inter(q[:, None], mu, Wij[:, None], dirs, idx_i, idx_j, N)
    xh = msg.x_proj(q)
    s, xh2, xh3 = torch.split(xh[idx_j] * Wij[:, swap], n, dim=-1)
    v = mu[idx_j] * xh2.unsqueeze(1) + xh3.unsqueeze(1) * dirs.unsqueeze(2)
    q1_oc = q + torch.zeros_like(q).index_add_(0, idx_i, s)
    mu1_oc = mu + torch.zeros_like(mu).index_add_(0, idx_i, v)
    assert torch.allclose(q1.squeeze(1), q1_oc, atol=1e-12) and torch.allclose(mu1, mu1_oc, atol=1e-12)
    # update: OC (vec1, vec2) = spk (mu_W, mu_V); OC chunks (h1, h2, h3) = spk (dq, dqmu, dmu)
    half = torch.cat([torch.arange(n, 2 * n), torch.arange(0, n)])
    upd.vec_proj.weight.data = mix.mu_channel_mix.weight.data[half]
    upd.xvec_proj[0].load_state_dict(mix.intraatomic_context_net[0].state_dict())
    upd.xvec_proj[2].weight.data = mix.intraatomic_context_net[1].weight.data[swap]
    upd.xvec_proj[2].bias.data = mix.intraatomic_context_net[1].bias.data[swap]
    q2, mu2 = mix(q1, mu1)
    dx, dvec = upd(q1.squeeze(1), mu1)
    assert torch.allclose(q2.squeeze(1), q1.squeeze(1) + dx, atol=1e-12)
    assert torch.allclose(mu2, mu1 + dvec, atol=1e-12)


def test_gemnet_oc_golden_file_is_present_and_consistent():
    """SURVEY.md section 8 a19: outputs of the reference's own GemNet-OC classes on fixture molecules (tests/golden/make_golden_gemnet_oc.py),
    consumed by the oracle tests below and by the engine tests (test_gemnet_emu.py, test_zz_gpu_first_runs.py); this check keeps the file
    honest."""
    import os

    import numpy as np

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemnet_oc_f32.npz"))
    n = len(g["z"])
    assert g["pos"].shape == (n, 3) and g["forces"].shape == (n, 3) and g["energy"].reshape(-1).shape == (2,)
    assert int(g["n_params"]) == 37815873 and int(g["main_edges"]) == 2350 and int(g["qint_edges"]) == 632
    assert np.isfinite(g["energy"]).all() and 0.01 < np.abs(g["forces"]).max() < 1.0
    # graph indices and per-block intermediates
    assert g["main/edge_index"].shape == (2, 2350) and g["id_swap"].shape == (2350,) and g["trip_e2e/in"].shape == g["trip_e2e/out"].shape
    ei = g["main/edge_index"]
    assert np.array_equal(ei[:, g["id_swap"]][::-1], ei)   # id_swap maps every edge to its reverse
    assert all(g[f"int{i}/h"].shape == (n, 256) and g[f"int{i}/m_rownorm"].shape == (2350,) for i in range(4))


def test_gemnet_oc_graph_oracle_matches_reference_indices_exactly():
    """oracle/gemnet_graph.py against the index arrays produced by the reference's own GemNet-OC classes (integer work: bit-exact)."""
    import os

    import numpy as np
    import torch

    import hashlib

    from oracle.gemnet_graph import build_all_indices

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemnet_oc_f32.npz"))
    pos, batch = torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"])
    o = build_all_indices(pos, batch)
    for name in ("main", "a2a", "a2ee2a", "qint"):
        assert np.array_equal(o[name]["edge_index"].numpy(), g[f"{name}/edge_index"]), name
    assert np.abs(o["main"]["distance"].numpy() - g["main/distance"]).max() < 1e-6
    assert np.array_equal(o["id_swap"].numpy(), g["id_swap"])
    for name in ("trip_e2e", "trip_a2e", "trip_e2a"):
        for k in ("in", "out", "out_agg"):
            assert np.array_equal(o[name][k].numpy(), g[f"{name}/{k}"]), (name, k)
    for k in ("out", "trip_in_to_quad", "trip_out_to_quad", "out_agg"):  # stored as sha1 of the int32 array + its length
        a = np.ascontiguousarray(o["quad"][k].numpy().astype(np.int32))
        assert a.shape[0] == int(g[f"quad/{k}/len"]) and hashlib.sha1(a.tobytes()).hexdigest() == str(g[f"quad/{k}/sha1"]), k
    for tk in ("triplet_in", "triplet_out"):
        for k in ("in", "out"):
            assert np.array_equal(o["quad"][tk][k].numpy(), g[f"quad/{tk}/{k}"]), (tk, k)
    for name in ("a2a", "a2ee2a"):
        assert np.array_equal(o[name]["target_neighbor_idx"].numpy(), g[f"{name}/target_neighbor_idx"])


def test_gemnet_oc_oracle_matches_reference_outputs_and_intermediates():
    """The whole GemNet-OC oracle (oracle/gemnet_oc.py) vs energies, forces and per-block intermediates recorded from the reference's own
    classes with the same name-keyed weights (weight_scale 0.5, scale factors 1): float32 against float32, tolerances relative to the
    largest entry of each tensor."""
    import os

    import numpy as np
    import torch

    from oracle.gemnet_oc import GemNetOCOracle
    from weights import golden_state_dict

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemnet_oc_f32.npz"))
    net = GemNetOCOracle().float().eval()
    sd = net.state_dict()
    assert len(sd) == 429 and sum(p.numel() for p in net.parameters()) == int(g["n_params"])
    new = golden_state_dict(sd, bias_std=0.02, weight_scale=float(g["weight_scale"]))
    for k in sd:
        if k.endswith("scale_factor"):
            sd[k] = torch.ones_like(sd[k])
        elif k in new:
            sd[k] = torch.as_tensor(np.asarray(new[k])).float().reshape(sd[k].shape)
    net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        E, F = net(torch.from_numpy(g["z"]), torch.from_numpy(g["pos"]), torch.from_numpy(g["batch"]))
    t = {k: v.numpy() for k, v in net.trace.items()}

    def close(a, b, rel):
        return np.abs(a - b).max() <= rel * np.abs(b).max()

    assert np.abs(t["atom_emb/h"] - g["atom_emb/h"]).max() == 0.0
    assert close(np.linalg.norm(t["edge_emb/m"], axis=1), g["edge_emb/m_rownorm"], 2e-5)
    for i in range(4):
        assert close(t[f"int{i}/h"], g[f"int{i}/h"], 2e-4), i
        assert close(np.linalg.norm(t[f"int{i}/m"], axis=1), g[f"int{i}/m_rownorm"], 2e-4), i
    for i in range(5):
        assert close(t[f"out{i}/x_E"], g[f"out{i}/x_E"], 2e-4), i
        assert close(np.linalg.norm(t[f"out{i}/x_F"], axis=-1), g[f"out{i}/x_F_rownorm"], 2e-4), i
    assert np.abs(E.numpy() - g["energy"].reshape(-1)).max() < 2e-4 * np.abs(g["energy"]).max()
    assert np.abs(F.numpy() - g["forces"]).max() < 2e-4 * np.abs(g["forces"]).max()


def test_gemnet_oc_oracle_second_batch_indices_and_outputs():
    """Three other fixture molecules: every index array hashes to what the reference's own classes produced; E and F agree."""
    import hashlib
    import os

    import numpy as np
    import torch

    from oracle.gemnet_graph import build_all_indices
    from oracle.gemnet_oc import GemNetOCOracle
    from weights import golden_state_dict

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemnet_oc_f32.npz"))
    z, pos, batch = torch.from_numpy(g["b2/z"]), torch.from_numpy(g["b2/pos"]), torch.from_numpy(g["b2/batch"])
    o = build_all_indices(pos, batch)
    sha = lambda t: hashlib.sha1(np.ascontiguousarray(t.numpy().astype(np.int32)).tobytes()).hexdigest()
    got = {"b2/main": sha(o["main"]["edge_index"]), "b2/a2a": sha(o["a2a"]["edge_index"]), "b2/a2ee2a": sha(o["a2ee2a"]["edge_index"]),
           "b2/qint": sha(o["qint"]["edge_index"]), "b2/id_swap": sha(o["id_swap"]), "b2/trip_e2e_in": sha(o["trip_e2e"]["in"]),
           "b2/trip_a2e_in": sha(o["trip_a2e"]["in"]), "b2/trip_e2a_in": sha(o["trip_e2a"]["in"]), "b2/quad_out": sha(o["quad"]["out"]),
           "b2/quad_in": sha(o["quad"]["trip_in_to_quad"]), "b2/quad_outmap": sha(o["quad"]["trip_out_to_quad"])}
    for k, v in got.items():
        assert v == str(g[k]), k
    net = GemNetOCOracle().float().eval()
    sd = net.state_dict()
    new = golden_state_dict(sd, bias_std=0.02, weight_scale=float(g["weight_scale"]))
    for k in sd:
        sd[k] = torch.ones_like(sd[k]) if k.endswith("scale_factor") else (torch.as_tensor(np.asarray(new[k])).float().reshape(sd[k].shape) if k in new else sd[k])
    net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        E, F = net(z, pos, batch)
    assert np.abs(E.numpy() - g["b2/energy"].reshape(-1)).max() < 2e-4 * np.abs(g["b2/energy"]).max()
    assert np.abs(F.numpy() - g["b2/forces"]).max() < 2e-4 * np.abs(g["b2/forces"]).max()
