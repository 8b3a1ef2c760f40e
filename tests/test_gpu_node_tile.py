"""The fused PaiNN node kernels run 80-atom tiles when that saves enough waves of CTAs (DESIGN.md §3), else 64-atom tiles.  Molecules do
not interact, so a molecule must come out the same whatever else is in its batch: molecules of a large batch (80-atom tiles) are compared
bit for bit with a 100-molecule batch of the same molecules (64-atom tiles)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

E_TOL = 1e-5  # Ha
F_TOL = 1e-4  # Ha/A
N_SMALL = 100


def dev():
    return torch.device("cuda:0")


def _spk_model():
    from helpers import load_golden_weights

    from nabladft_b200 import spk

    m = spk.NeuralNetworkPotential(
        representation=spk.PaiNN(n_atom_basis=128, n_interactions=6, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                 cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()],
        output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()],
        postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32)
    m.postprocessors[0].mean.fill_(-0.01)
    return m.eval()


def _batch(seed, n_mol, n_take):
    """The first n_take molecules of synth_batch(seed, n_mol), as CPU tensors."""
    from nabladft_b200.synth import synth_batch

    b = synth_batch(seed, n_mol)
    n = int(b["mol_ptr"][n_take])
    return torch.from_numpy(b["z"][:n]).long(), torch.from_numpy(b["pos"][:n]), torch.from_numpy(b["batch"][:n]).long()


def _run(model, z, pos, batch):
    out = model({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
                 "_n_atoms": torch.bincount(batch).to(dev())})
    return out["energy"].detach(), out["forces"].detach()


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wide(n_atoms):
    """The tile rule of painn_fused.cu: 80-atom tiles when they need fewer waves of CTAs than 64-atom tiles."""
    waves = lambda nt: -(-(-(-n_atoms // nt)) // _n_sm())
    return waves(80) < waves(64)


def _mol_slice(z, pos, batch, m0, m1):
    """Molecules [m0, m1) as a batch of their own, and their atom range in the original batch."""
    a, b = (int(torch.searchsorted(batch, torch.tensor(m))) for m in (m0, m1))
    return (z[a:b], pos[a:b], batch[a:b] - m0), a, b


# (seed, molecules generated, molecules run): 9,750 and 9,565 atoms (one wave of 80-atom tiles instead of two of 64), 19,505 atoms
# (two waves instead of three), 9,441 atoms (the last 80-atom tile holds 1 atom)
@pytest.mark.parametrize("seed,n_mol,n_take", [(1, 256, 256), (2, 256, 256), (1, 520, 520), (1, 400, 247)])
def test_wide_tiles_match_narrow_tiles_bitwise(seed, n_mol, n_take):
    """The first and the last N_SMALL molecules of a batch that runs 80-atom tiles, against batches of just those molecules (64-atom tiles)."""
    model = _spk_model().to(dev())
    z, pos, batch = _batch(seed, n_mol, n_take)
    N = z.numel()
    assert _wide(N)
    if n_take == 247:
        assert N % 80 == 1
    e_big, f_big = _run(model, z, pos, batch)
    for m0 in (0, n_take - N_SMALL):
        small, a, b = _mol_slice(z, pos, batch, m0, m0 + N_SMALL)
        assert not _wide(b - a)
        e_small, f_small = _run(model, *small)
        de = (e_big[m0:m0 + N_SMALL] - e_small).abs().max().item()
        df = (f_big[a:b] - f_small).abs().max().item()
        print(f"seed {seed}, {n_take} molecules / {N} atoms, molecules [{m0}, {m0 + N_SMALL}) / atoms [{a}, {b}) run alone: "
              f"max|dE| {de:.3e} Ha, max|dF| {df:.3e} Ha/A")
        assert torch.equal(e_big[m0:m0 + N_SMALL], e_small) and torch.equal(f_big[a:b], f_small)


def test_wide_tiles_match_fp64_oracle():
    """All 256 molecules of a batch that runs 80-atom tiles against the fp64 oracle, evaluated 32 molecules at a time on the CPU."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkPaiNN

    model = _spk_model()
    ref = OracleNNP(SpkPaiNN()).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    z, pos, batch = _batch(1, 256, 256)
    assert _wide(z.numel())
    e, f = _run(model.to(dev()), z, pos, batch)
    e, f = e.double().cpu(), f.double().cpu()
    ptr = batch_to_ptr(batch)
    de = df = 0.0
    for m0 in range(0, 256, 32):
        a, b = int(ptr[m0]), int(ptr[m0 + 32])
        p = pos[a:b].double().clone()
        idx_i, idx_j = ase_neighbor_list(p, ptr[m0:m0 + 33] - a, 5.0)
        out = ref({"_atomic_numbers": z[a:b], "_positions": p, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch[a:b] - m0})
        de = max(de, (e[m0:m0 + 32] - out["energy"].detach()).abs().max().item())
        df = max(df, (f[a:b] - out["forces"].detach()).abs().max().item())
    print(f"256 molecules / {z.numel()} atoms vs fp64 oracle: max|dE| {de:.2e} Ha, max|dF| {df:.2e} Ha/A")
    assert de < E_TOL and df < F_TOL
