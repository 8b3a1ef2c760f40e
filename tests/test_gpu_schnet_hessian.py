"""Exact Hessian-vector products of the SchNet engine (nb200_schnet_hvp, nabladft_b200.vibrations) against the float64 oracle's double
backward, their symmetry / invariance properties, edge cases, argument checks and the normal modes built on them (the SchNet counterpart of
test_gpu_hessian.py)."""
import ctypes

import pytest
import torch

from helpers import load_fixture, load_golden_weights, random_rotation
from test_gpu_hessian import _blocks, _edge_case_batch

pytestmark = pytest.mark.gpu

PARITY_MOLS = [26, 3, 99]  # 29, 30 and 54 atoms
E_TOL, F_TOL = 1e-5, 1e-4  # Ha, Ha/A (north_star, absolute)


def dev():
    return torch.device("cuda:0")


def _model(layers=3, weight_scale=1.0):
    """weight_scale=None: the golden weights' default scale, whose smoother energy surface L-BFGS relaxes to fmax 1e-4 (at 1.0 it does not
    converge in 4000 steps)."""
    from nabladft_b200 import spk

    m = spk.NeuralNetworkPotential(
        representation=spk.SchNet(n_atom_basis=128, n_interactions=layers, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                  cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()], output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()],
        postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32, **({} if weight_scale is None else {"weight_scale": weight_scale}))
    m.postprocessors[0].mean.fill_(0.02)
    return m.to(dev()).eval()


def _ref(model):
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkSchNet

    ref = OracleNNP(SpkSchNet(n_interactions=len(model.representation.interactions))).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double().cpu() for k in ref.state_dict()}, strict=True)
    return ref


def _oracle(ref, z, pos, batch):
    """energy (with the AddOffsets shift), forces and the full [3N, 3N] float64 Hessian by double backward of the oracle's forces."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr

    p = pos.detach().clone().double().requires_grad_(True)
    idx_i, idx_j = ase_neighbor_list(p.detach(), batch_to_ptr(batch), 5.0)
    out = ref({"_atomic_numbers": z, "_positions": p, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=True, create_graph=True)
    f = out["forces"].reshape(-1)
    rows = [torch.autograd.grad(-f[i], p, retain_graph=True, allow_unused=True)[0] for i in range(f.numel())]
    h = torch.stack([torch.zeros_like(p).reshape(-1) if r is None else r.reshape(-1) for r in rows]).detach()
    return out["energy"].detach(), out["forces"].detach(), h


def _batch(z, pos, batch):
    return {"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
            "_n_atoms": torch.bincount(batch).to(dev())}


def test_schnet_hessian_matches_oracle_double_backward():
    from nabladft_b200 import vibrations as vib

    z, pos, batch = load_fixture(PARITY_MOLS)
    sizes = torch.bincount(batch).tolist()
    model = _model()
    b = _batch(z, pos, batch)
    hs = vib.hessians(model, b)
    e_ref, f_ref, h_ref = _oracle(_ref(model), z, pos, batch)
    worst = []
    for h, r in zip(hs, _blocks(h_ref, sizes)):
        r = 0.5 * (r + r.t())
        worst.append(float((h.double().cpu() - r).abs().max() / r.abs().max()))
    print("worst |H - H_ref| / max|H_ref| per molecule:", worst, "raw asymmetry", hs.max_asymmetry)
    assert max(worst) < 2e-5
    # energies and forces of the HVP call: against the inference engine (reported) and the oracle (north_star)
    with torch.no_grad():
        out = model(b)
    torch.cuda.synchronize()
    e, f, hv = vib.hessian_vector_product(model, b, torch.zeros(1, z.numel(), 3, device=dev()))
    print("HVP call vs inference engine: |dE|", float((e - out["energy"]).abs().max()), "|dF|", float((f - out["forces"]).abs().max()))
    de, df = float((e.double().cpu() - e_ref).abs().max()), float((f.double().cpu() - f_ref).abs().max())
    print("HVP call vs oracle: |dE|", de, "|dF|", df)
    assert de < E_TOL and df < F_TOL
    assert torch.equal(hv, torch.zeros_like(hv))


def test_schnet_hessian_properties():
    from nabladft_b200 import vibrations as vib

    z, pos, batch = load_fixture([0, 4, 7])
    model = _model()
    b = _batch(z, pos, batch)
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
    for md in (1, 7):  # direction chunking does not change anything
        assert all(torch.equal(x, y) for x, y in zip(vib.hessians(model, b, max_dir=md), hs))

    q = random_rotation(3)  # rotation covariance: r_i -> Q r_i gives H' = (I (x) Q) H (I (x) Q)^T
    hr = vib.hessians(model, _batch(z, pos @ q.t(), batch))
    for h, h2 in zip(hs, hr):
        n = h.shape[0] // 3
        big = torch.block_diag(*([q] * n)).to(dev()).float()
        err = float((big @ h @ big.t() - h2).abs().max() / h.abs().max())
        assert err < 2e-5, err


def test_schnet_batch_independence_64():
    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import synth_batch

    s = synth_batch(7, 64)
    z, pos, bt = torch.from_numpy(s["z"]).long(), torch.from_numpy(s["pos"]), torch.from_numpy(s["batch"])
    model = _model()
    hs = vib.hessians(model, _batch(z, pos, bt))
    ptr = s["mol_ptr"]
    for m in (0, 31, 63):
        a, e = ptr[m], ptr[m + 1]
        alone = vib.hessians(model, _batch(z[a:e], pos[a:e], torch.zeros(e - a, dtype=torch.int64)))[0]
        err = float((alone - hs[m]).abs().max() / alone.abs().max())
        assert err < 1e-6, (m, err)


def test_schnet_edge_cases():
    from nabladft_b200 import vibrations as vib

    z, pos, batch = _edge_case_batch()
    model = _model()
    b = _batch(z, pos, batch)
    hs = vib.hessians(model, b)
    assert torch.equal(hs[0], torch.zeros(3, 3, device=dev()))
    assert torch.equal(hs[1], torch.zeros(6, 6, device=dev()))
    # the pair just inside the cutoff, alone, against the oracle (error bounded against the batch's Hessian scale, as for PaiNN)
    _, _, r = _oracle(_ref(model), z[3:5], pos[3:5], torch.zeros(2, dtype=torch.int64))
    assert float(r.abs().max()) > 0
    err = float((hs[2].double().cpu() - r).abs().max())
    print("near-cutoff pair: max|H_ref|", float(r.abs().max()), "error", err, "batch max|H|", float(hs[3].abs().max()))
    assert err < 1e-5 * float(hs[3].abs().max())
    # n_dir > 3 n_max: the extra (zero) directions give exactly zero; one direction alone equals the same direction in a batch of them
    n_max = int(torch.bincount(batch).max())
    v = vib.shared_directions(torch.cat([torch.zeros(1), torch.cumsum(torch.bincount(batch), 0)]).long().tolist(), 0, 3 * n_max, dev())
    v = torch.cat([v, torch.zeros(5, z.numel(), 3, device=dev())])
    _, _, hv = vib.hessian_vector_product(model, b, v)
    assert torch.equal(hv[3 * n_max:], torch.zeros_like(hv[3 * n_max:]))
    _, _, hv1 = vib.hessian_vector_product(model, b, v[4])
    assert torch.equal(hv1, hv[4])


def test_schnet_hvp_argument_checks_and_output_bounds():
    from nabladft_b200 import _lib

    lib = _lib.load()
    model = _model()
    z, pos, batch = load_fixture([0, 4])
    eng, z, pos, mol_ptr, B = model._prepare(_batch(z, pos, batch))
    mol_ptr = mol_ptr.contiguous()
    N, n_dir, T = z.numel(), 4, 64
    row_ptr, scratch, n_edges = torch.empty(N + 1, dtype=torch.int32, device=dev()), torch.empty(2 * N, dtype=torch.int32, device=dev()), ctypes.c_int64()
    P, stream = _lib.ptr, _lib.current_stream()
    assert lib.nb200_schnet_train_count(ctypes.byref(eng._weights), P(pos), P(mol_ptr), B, N, P(row_ptr), P(scratch), ctypes.byref(n_edges), stream) == 0
    ws_bytes = lib.nb200_schnet_hvp_workspace_bytes(ctypes.byref(eng._weights), B, N, n_edges.value)
    assert ws_bytes > 0 and lib.nb200_schnet_hvp_workspace_bytes(ctypes.byref(eng._weights), B, N, -1) == -1
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    v = torch.randn(n_dir, N, 3, device=dev())
    sentinel = 12345.5
    energy = torch.full((B + T,), float("nan"), device=dev()); energy[B:] = sentinel
    forces = torch.full((3 * N + T,), float("nan"), device=dev()); forces[3 * N:] = sentinel
    hv = torch.full((n_dir * 3 * N + T,), float("nan"), device=dev()); hv[n_dir * 3 * N:] = sentinel

    def call(n_dir_=n_dir, v_=v, bytes_=ws_bytes, hv_=hv):
        return lib.nb200_schnet_hvp(eng._h, ctypes.byref(eng._weights), P(z), P(pos), P(mol_ptr), B, N, P(row_ptr), n_edges.value, P(ws), bytes_,
                                    n_dir_, P(v_), P(energy), P(forces), P(hv_), stream)

    before = lib.nb200_engine_own_launches(eng._h)
    assert call(v_=None) == -1
    assert call(hv_=None) == -1
    assert call(n_dir_=0) == -1
    assert call(bytes_=ws_bytes - 1) == -1
    assert lib.nb200_engine_own_launches(eng._h) == before
    assert call() == 0
    torch.cuda.synchronize()
    for t, n in ((energy, B), (forces, 3 * N), (hv, n_dir * 3 * N)):
        assert not torch.isnan(t[:n]).any()
        assert bool((t[n:] == sentinel).all())


def _relaxed(model, mol):
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, SimpleAtoms, SpkBatchwiseCalculator

    z, pos, _ = load_fixture([mol])
    calc = SpkBatchwiseCalculator(model, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None)
    assert opt.run([SimpleAtoms(pos.numpy(), z.numpy())], fmax=1e-4, steps=1000)
    return z, torch.from_numpy(opt.atoms[0].get_positions()).double()


def test_schnet_normal_modes_relaxed_and_unrelaxed_against_oracle():
    from nabladft_b200 import vibrations as vib

    model = _model(weight_scale=None)
    ref = _ref(model)
    z, pos = _relaxed(model, 26)
    batch = torch.zeros(z.numel(), dtype=torch.int64)
    nm = vib.normal_modes(model, _batch(z, pos, batch))[0]
    nu = nm.wavenumbers.cpu()
    mags = nu.abs().sort().values
    print("six smallest |nu| (cm^-1):", mags[:6].tolist(), "first vibrational:", float(mags[6]))
    assert float(mags[5]) < 0.5 * float(mags[6])
    nu_ref = vib.normal_modes_from_hessian(_oracle(ref, z, pos, batch)[2], vib.masses_of(z)).wavenumbers
    hi = nu_ref > 100
    err = (nu[hi] - nu_ref[hi]).abs()
    print("worst frequency error above 100 cm^-1:", float(err.max()), "relative", float((err / nu_ref[hi]).max()))
    assert bool((err < torch.clamp(2e-5 * nu_ref[hi], min=0.1)).all())

    # the unrelaxed fixture geometry: same count of imaginary (non-rigid) modes as the oracle
    z, pos, batch = load_fixture([26])
    nm = vib.normal_modes(model, _batch(z, pos, batch), project=True)[0]
    ref_nm = vib.normal_modes_from_hessian(_oracle(ref, z, pos, batch)[2], vib.masses_of(z), pos, project=True)
    count = int((nm.wavenumbers < -5).sum())
    print("imaginary modes of the unrelaxed geometry:", count, "oracle", int((ref_nm.wavenumbers < -5).sum()))
    assert count == int((ref_nm.wavenumbers < -5).sum())
