"""Exact Hessian-vector products of the PaiNN engine (nb200_painn_hvp, nabladft_b200.vibrations) against the float64 oracle's double backward,
their symmetry / invariance properties, edge cases, output guards and the normal modes built on them."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import load_fixture, random_rotation
from test_gpu_painn import _Data, _oc_model, _spk_model, dev

pytestmark = pytest.mark.gpu

PARITY_MOLS = [26, 3, 99]  # 29, 30 and 54 atoms


def _oc_ref(net):
    from oracle.painn_oc import PaiNNOC

    ref = PaiNNOC(hidden_channels=128, num_layers=net.num_layers, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100).double()
    ref.load_state_dict({k: v.double().cpu() for k, v in net.state_dict().items()}, strict=True)
    return ref


def _spk_ref(model):
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkPaiNN

    ref = OracleNNP(SpkPaiNN(n_interactions=len(model.representation.interactions))).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double().cpu() for k in ref.state_dict()}, strict=True)
    return ref


def _oracle_hessian(kind, ref, z, pos, batch):
    """Full [3N, 3N] float64 Hessian by autograd double backward (create_graph=True) of the oracle's forces."""
    p = pos.detach().clone().double().requires_grad_(True)
    if kind == "oc":
        _, f = ref(z, p, batch, create_graph=True)
    else:
        from oracle.graph import ase_neighbor_list, batch_to_ptr

        idx_i, idx_j = ase_neighbor_list(p.detach(), batch_to_ptr(batch), 5.0)
        f = ref({"_atomic_numbers": z, "_positions": p, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False,
                create_graph=True)["forces"]
    f = f.reshape(-1)
    rows = [torch.autograd.grad(-f[i], p, retain_graph=True, allow_unused=True)[0] for i in range(f.numel())]
    return torch.stack([torch.zeros_like(p).reshape(-1) if r is None else r.reshape(-1) for r in rows]).detach()


def _model(kind, layers=3):
    return (_oc_model(layers) if kind == "oc" else _spk_model(layers)).to(dev()).eval()


def _batch(kind, z, pos, batch):
    if kind == "oc":
        return _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev()))
    return {"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
            "_n_atoms": torch.bincount(batch).to(dev())}


def _forces(kind, model, b):
    with torch.no_grad():
        if kind == "oc":
            e, f = model(b)
        else:
            out = model(b)
            e, f = out["energy"], out["forces"]
    torch.cuda.synchronize()
    return e, f


def _blocks(h, sizes):
    out, a = [], 0
    for n in sizes:
        out.append(h[3 * a:3 * (a + n), 3 * a:3 * (a + n)])
        a += n
    return out


@pytest.mark.parametrize("kind", ["oc", "spk"])
def test_hessian_matches_oracle_double_backward(kind):
    from nabladft_b200 import vibrations as vib

    z, pos, batch = load_fixture(PARITY_MOLS)
    sizes = torch.bincount(batch).tolist()
    assert len(set(sizes)) == 3
    model = _model(kind)
    b = _batch(kind, z, pos, batch)
    hs = vib.hessians(model, b)
    ref_blocks = _blocks(_oracle_hessian(kind, _oc_ref(model) if kind == "oc" else _spk_ref(model), z, pos, batch), sizes)
    worst = []
    for h, r in zip(hs, ref_blocks):
        r = 0.5 * (r + r.t())
        worst.append(float((h.double().cpu() - r).abs().max() / r.abs().max()))
    print(kind, "worst |H - H_ref| / max|H_ref| per molecule:", worst, "raw asymmetry", hs.max_asymmetry)
    assert max(worst) < 2e-5  # first run on an H100: 6.6e-6 (PaiNN-OC), 9.1e-6 (spk)
    # energies and forces of the HVP call are those of the inference engine
    e_ref, f_ref = _forces(kind, model, b)
    e, f, _ = vib.hessian_vector_product(model, b, torch.zeros(1, z.numel(), 3, device=dev()))
    assert float((f - f_ref).abs().max()) <= 1e-6
    assert float((e - e_ref).abs().max()) <= 1e-6 * float(e_ref.abs().max())


def test_hessian_properties():
    from nabladft_b200 import vibrations as vib

    z, pos, batch = load_fixture([0, 4, 7])
    model = _model("oc")
    b = _batch("oc", z, pos, batch)
    N = z.numel()
    g = torch.Generator().manual_seed(5)
    vw = torch.randn(2, N, 3, generator=g).to(dev())
    _, _, hv = vib.hessian_vector_product(model, b, vw)
    a, c = float((vw[1] * hv[0]).sum()), float((vw[0] * hv[1]).sum())
    scale = float(vw[1].norm() * hv[0].norm())
    print("symmetry |w.Hv - v.Hw| / (|w||Hv|):", abs(a - c) / scale)
    assert abs(a - c) < 1e-5 * scale

    hs = vib.hessians(model, b)
    hs2 = vib.hessians(model, b)
    assert all(torch.equal(x, y) for x, y in zip(hs, hs2))  # bitwise repeatable
    for h in hs:  # translation sum rule: sum_j H_ij = 0
        n = h.shape[0] // 3
        s = h.reshape(n, 3, n, 3).sum(2).abs().max()
        assert float(s) < 1e-4 * float(h.abs().max())
    # direction chunking does not change anything
    for md in (1, 7):
        assert all(torch.equal(x, y) for x, y in zip(vib.hessians(model, b, max_dir=md), hs))

    # rotation covariance: r_i -> Q r_i gives H' = (I (x) Q) H (I (x) Q)^T
    q = random_rotation(3)
    hr = vib.hessians(model, _batch("oc", z, pos @ q.t(), batch))
    for h, h2 in zip(hs, hr):
        n = h.shape[0] // 3
        big = torch.block_diag(*([q] * n)).to(dev()).float()
        err = float((big @ h @ big.t() - h2).abs().max() / h.abs().max())
        assert err < 2e-5, err


def test_batch_independence_64():
    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import synth_batch

    s = synth_batch(7, 64)
    z, pos, bt = torch.from_numpy(s["z"]).long(), torch.from_numpy(s["pos"]), torch.from_numpy(s["batch"])
    model = _model("spk")
    hs = vib.hessians(model, _batch("spk", z, pos, bt))
    ptr = s["mol_ptr"]
    for m in (0, 31, 63):
        a, e = ptr[m], ptr[m + 1]
        alone = vib.hessians(model, _batch("spk", z[a:e], pos[a:e], torch.zeros(e - a, dtype=torch.int64)))[0]
        err = float((alone - hs[m]).abs().max() / alone.abs().max())
        assert err < 1e-6, (m, err)


def _edge_case_batch():
    """1-atom molecule, a 2-atom molecule with no edge inside the 5 A cutoff, a C-H pair 4.9995 A apart and fixture molecule 1."""
    z0, p0, _ = load_fixture([1])
    zs = [torch.tensor([1]), torch.tensor([6, 8]), torch.tensor([6, 1]), z0]
    ps = [torch.zeros(1, 3, dtype=torch.float64), torch.tensor([[0.0, 0.0, 0.0], [5.3, 1.0, 0.0]], dtype=torch.float64),
          torch.tensor([[0.1, 0.2, 0.3], [0.1 + 4.9995 * 0.6, 0.2, 0.3 + 4.9995 * 0.8]], dtype=torch.float64), p0]
    batch = torch.cat([torch.full((len(x),), i, dtype=torch.int64) for i, x in enumerate(zs)])
    return torch.cat(zs), torch.cat(ps), batch


@pytest.mark.parametrize("kind", ["oc", "spk"])
def test_edge_cases(kind):
    from nabladft_b200 import vibrations as vib

    z, pos, batch = _edge_case_batch()
    model = _model(kind)
    b = _batch(kind, z, pos, batch)
    hs = vib.hessians(model, b)
    assert torch.equal(hs[0], torch.zeros(3, 3, device=dev()))
    assert torch.equal(hs[1], torch.zeros(6, 6, device=dev()))
    # the pair just inside the cutoff, alone, against the oracle
    ref = _oc_ref(model) if kind == "oc" else _spk_ref(model)
    r = _oracle_hessian(kind, ref, z[3:5], pos[3:5], torch.zeros(2, dtype=torch.int64))
    # the envelope and its derivatives are ~(1e-4)^k small there and evaluated in fp32, so the error is bounded against the batch's Hessian
    # scale (fixture molecule 1), as in the parity test
    assert float(r.abs().max()) > 0
    err = float((hs[2].double().cpu() - r).abs().max())
    print(kind, "near-cutoff pair: max|H_ref|", float(r.abs().max()), "error", err, "batch max|H|", float(hs[3].abs().max()))
    assert err < 1e-5 * float(hs[3].abs().max())
    # n_dir = 1 and n_dir > 3 n_max: the extra (zero) directions give exactly zero
    n_max = int(torch.bincount(batch).max())
    v = vib.shared_directions(torch.cat([torch.zeros(1), torch.cumsum(torch.bincount(batch), 0)]).long().tolist(), 0, 3 * n_max, dev())
    v = torch.cat([v, torch.zeros(5, z.numel(), 3, device=dev())])
    _, _, hv = vib.hessian_vector_product(model, b, v)
    assert torch.equal(hv[3 * n_max:], torch.zeros_like(hv[3 * n_max:]))
    _, _, hv1 = vib.hessian_vector_product(model, b, v[4])
    assert torch.equal(hv1, hv[4])


def test_output_guards_and_argument_checks():
    from nabladft_b200 import _lib

    lib = _lib.load()
    model = _model("oc")
    eng = model.engine()
    z, pos, batch = load_fixture([0, 4])
    z, pos = z.to(torch.int32).to(dev()), pos.float().to(dev())
    from nabladft_b200.engine import mol_ptr_from_batch

    mol_ptr, B = mol_ptr_from_batch(batch.to(dev()))
    N, n_dir, T = z.numel(), 4, 64
    e_cap = N * 64
    ws_bytes = lib.nb200_painn_hvp_workspace_bytes(ctypes.byref(eng._weights), B, N, e_cap, n_dir)
    assert ws_bytes > 0 and lib.nb200_painn_hvp_workspace_bytes(ctypes.byref(eng._weights), B, N, e_cap, 0) == -1
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    status = torch.zeros(4, dtype=torch.int32, device=dev())
    v = torch.randn(n_dir, N, 3, device=dev())
    sentinel = 12345.5
    energy = torch.full((B + T,), float("nan"), device=dev()); energy[B:] = sentinel
    forces = torch.full((3 * N + T,), float("nan"), device=dev()); forces[3 * N:] = sentinel
    hv = torch.full((n_dir * 3 * N + T,), float("nan"), device=dev()); hv[n_dir * 3 * N:] = sentinel
    P = _lib.ptr
    stream = _lib.current_stream()

    def call(n_dir_=n_dir, v_=v, bytes_=ws_bytes, hv_=hv):
        return lib.nb200_painn_hvp(eng._h, ctypes.byref(eng._weights), P(z), P(pos), P(mol_ptr), B, N, e_cap, P(ws), bytes_, n_dir_, P(v_),
                                   P(energy), P(forces), P(hv_), P(status), stream)

    before = lib.nb200_engine_own_launches(eng._h)
    assert call(v_=None) == -1
    assert call(hv_=None) == -1
    assert call(n_dir_=0) == -1
    assert call(bytes_=ws_bytes - 1) == -1
    assert lib.nb200_engine_own_launches(eng._h) == before
    assert call() == 0
    torch.cuda.synchronize()
    assert int(status[1]) == 0
    for t, n in ((energy, B), (forces, 3 * N), (hv, n_dir * 3 * N)):
        assert not torch.isnan(t[:n]).any()
        assert bool((t[n:] == sentinel).all())
    # a capacity error turns energy, forces and hv into NaN
    assert lib.nb200_painn_hvp(eng._h, ctypes.byref(eng._weights), P(z), P(pos), P(mol_ptr), B, N, 100, P(ws), ws_bytes, n_dir, P(v), P(energy),
                               P(forces), P(hv), P(status), stream) == 0
    torch.cuda.synchronize()
    assert int(status[1]) == -4
    for t, n in ((energy, B), (forces, 3 * N), (hv, n_dir * 3 * N)):
        assert torch.isnan(t[:n]).all() and bool((t[n:] == sentinel).all())


def _relaxed(net, mol):
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms

    z, pos, _ = load_fixture([mol])
    calc = PyGBatchwiseCalculator(net, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None)
    opt.run([SimpleAtoms(pos.numpy(), z.numpy())], fmax=1e-4, steps=1000)
    return z, torch.from_numpy(opt.atoms[0].get_positions()).double()


def test_normal_modes_relaxed_and_unrelaxed_against_oracle():
    from nabladft_b200 import vibrations as vib

    net = _model("oc")
    ref = _oc_ref(net)
    z, pos = _relaxed(net, 26)
    batch = torch.zeros(z.numel(), dtype=torch.int64)
    nm = vib.normal_modes(net, _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())))[0]
    nu = nm.wavenumbers.cpu()
    mags = nu.abs().sort().values
    print("six smallest |nu| (cm^-1):", mags[:6].tolist(), "first vibrational:", float(mags[6]))
    assert float(mags[5]) < 0.5 * float(mags[6])
    m = vib.masses_of(z)
    nu_ref = vib.normal_modes_from_hessian(_oracle_hessian("oc", ref, z, pos, batch), m).wavenumbers
    hi = nu_ref > 100
    err = (nu[hi] - nu_ref[hi]).abs()
    print("worst frequency error above 100 cm^-1:", float(err.max()), "relative", float((err / nu_ref[hi]).max()))
    assert bool((err < torch.clamp(2e-5 * nu_ref[hi], min=0.1)).all())

    # the unrelaxed fixture geometry: same count of imaginary (non-rigid) modes as the oracle
    z, pos, batch = load_fixture([26])
    nm = vib.normal_modes(net, _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())), project=True)[0]
    ref_nm = vib.normal_modes_from_hessian(_oracle_hessian("oc", ref, z, pos, batch), vib.masses_of(z), pos, project=True)
    count = int((nm.wavenumbers < -5).sum())
    print("imaginary modes of the unrelaxed geometry:", count, "oracle", int((ref_nm.wavenumbers < -5).sum()))
    assert count == int((ref_nm.wavenumbers < -5).sum())
