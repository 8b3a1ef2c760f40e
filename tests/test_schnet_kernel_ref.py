"""The float64 restatement of the SchNet inference kernels (schnet_kernel_ref.py), checked without a GPU: composed into the whole model it
reproduces the oracle's SchNet energies and forces, its derivatives agree with central differences, every term the kernels compute moves
some output by far more than the GPU tolerance on the GPU tests' inputs, and the 16-centre band of a shifted Gaussian basis misses most
of the filter -- which is why the export refuses such a basis."""
import math

import numpy as np
import pytest
import torch

import schnet_kernel_ref as ref
from helpers import load_fixture, load_golden_weights

CUTOFF, K = 5.0, 100


def _csr_of(idx_i, idx_j, pos):
    """CSR (target i major, source j ascending) of an oracle edge list -> row_ptr, col, rev, d, unit vectors r_ij / d."""
    N = pos.shape[0]
    order = np.lexsort((idx_j.numpy(), idx_i.numpy()))
    ti, sj = idx_i[order], idx_j[order]
    r = pos[sj] - pos[ti]
    d = r.norm(dim=1)
    index = {(int(a), int(b)): e for e, (a, b) in enumerate(zip(ti, sj))}
    rev = torch.tensor([index[(int(b), int(a))] for a, b in zip(ti, sj)], dtype=torch.int32)
    row_ptr = torch.zeros(N + 1, dtype=torch.int32)
    row_ptr[1:] = torch.cumsum(torch.bincount(ti, minlength=N), 0)
    return row_ptr, sj.int(), rev, d, r / d[:, None], ti


def _compose(model, z, pos, batch, idx_i, idx_j):
    """SchNet energy and forces from the kernels' restatement: per layer in2f, filter1 over all K, the second filter layer, cfconv, f2out;
    the reverse sweep through cfconv_bwd, and forces from the per-edge dE/dd."""
    rep, (ro0, ro1) = model.representation, model.output_modules[0].outnet
    row_ptr, col, rev, d, unit, tgt = _csr_of(idx_i, idx_j, pos)
    coeff = float(-0.5 / rep.radial_basis.widths[0] ** 2)
    offsets = rep.radial_basis.offsets
    x = rep.embedding.weight[z]
    saved = []
    for it in rep.interactions:
        f0, f1 = it.filter_network
        y = x @ it.in2f.weight.T
        h, dh, _, _ = ref.filter1(d, f0.weight.T, f0.bias, offsets, coeff, CUTOFF)
        G1, G2 = h @ f1.weight.T, dh @ f1.weight.T
        agg, _ = ref.cfconv_fwd(y, G1, f1.bias, d, row_ptr, col, CUTOFF)
        t = agg @ it.f2out[0].weight.T + it.f2out[0].bias
        x = x + ref.ssp(t) @ it.f2out[1].weight.T + it.f2out[1].bias
        saved.append((it, y, G1, G2, t))
    pre = x @ ro0.weight.T + ro0.bias
    eps = torch.nn.functional.silu(pre) @ ro1.weight.T + ro1.bias
    n_mol = int(batch.max()) + 1
    energy = torch.zeros(n_mol, dtype=torch.float64).index_add_(0, batch, eps[:, 0])
    energy = energy + model.postprocessors[0].mean * torch.bincount(batch, minlength=n_mol)
    s = torch.sigmoid(pre)
    gx = (ro1.weight * s * (1 + pre * (1 - s))) @ ro0.weight
    egrad = torch.zeros(d.numel(), dtype=torch.float64)
    for it, y, G1, G2, t in reversed(saved):
        gt = (gx @ it.f2out[1].weight) * torch.sigmoid(t)
        gagg = gt @ it.f2out[0].weight
        gy, _, egrad, _ = ref.cfconv_bwd(y, G1, G2, it.filter_network[1].bias, d, row_ptr, col, rev, CUTOFF, gagg, egrad)
        gx = gx + gy @ it.in2f.weight
    dE = torch.zeros_like(pos)
    dE.index_add_(0, col.long(), egrad[:, None] * unit).index_add_(0, tgt, -egrad[:, None] * unit)
    return energy, -dE


def test_composed_reference_matches_oracle():
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential, SpkSchNet

    model = NeuralNetworkPotential(SpkSchNet()).double()
    load_golden_weights(model, torch.float64, weight_scale=1.0)
    model.postprocessors[0].mean.fill_(0.02)
    z, pos, batch = load_fixture([10, 11, 12, 60])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), CUTOFF)
    out = model({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch})
    with torch.no_grad():
        e, f = _compose(model, z, pos, batch, idx_i, idx_j)
    de = (e - out["energy"].detach()).abs().max().item()
    df = (f - out["forces"]).abs().max().item()
    print(f"composed restatement vs oracle SpkSchNet: max|dE| {de:.1e} (|E| <= {out['energy'].abs().max().item():.2f}), max|dF| {df:.1e}")
    assert de < 1e-10 and df < 1e-10


def test_derivatives_match_central_differences():
    g = torch.Generator().manual_seed(3)
    w1, b1 = ref.filter_weights(1, K, seed=3)
    w1, b1 = w1[0].double(), b1[0].double()
    offsets = torch.linspace(0, CUTOFF, K, dtype=torch.float64)
    coeff = -0.5 / ref.spacing(CUTOFF, K) ** 2
    d = torch.rand(64, generator=g, dtype=torch.float64) * 4.9 + 0.02
    h_of = lambda dd: ref.filter1(dd, w1, b1, offsets, coeff, CUTOFF)[0]
    _, dh, _, _ = ref.filter1(d, w1, b1, offsets, coeff, CUTOFF)
    step = 1e-6
    fd = (h_of(d + step) - h_of(d - step)) / (2 * step)
    err = (fd - dh).abs().max().item()
    assert err < 1e-6 * dh.abs().max().item(), err
    # egrad: derivative of L = sum_i agg_i . gagg_i with G1 = h W2^T and G2 = dh W2^T of the same distances, per undirected pair
    row_ptr, col, rev, d = ref.random_graph(12, 30, CUTOFF, seed=4)
    d = d.double()
    x = ref.cfconv_inputs(12, d.numel(), seed=4)
    W2 = torch.randn(ref.F, ref.F, generator=g, dtype=torch.float64) / math.sqrt(ref.F)
    y, b2, gagg = x["y"].double(), x["b2"].double(), x["gagg"].double()

    def loss(dd):
        h = ref.filter1(dd, w1, b1, offsets, coeff, CUTOFF)[0]
        return (ref.cfconv_fwd(y, h @ W2.T, b2, dd, row_ptr, col, CUTOFF)[0] * gagg).sum()

    h, dh, _, _ = ref.filter1(d, w1, b1, offsets, coeff, CUTOFF)
    _, _, eg, _ = ref.cfconv_bwd(y, h @ W2.T, dh @ W2.T, b2, d, row_ptr, col, rev, CUTOFF, gagg, torch.zeros(d.numel(), dtype=torch.float64))
    worst = 0.0
    for e in range(0, d.numel(), 5):
        dp = d.clone(); dp[[e, int(rev[e])]] += step
        dm = d.clone(); dm[[e, int(rev[e])]] -= step
        fd = (loss(dp) - loss(dm)).item() / (2 * step)
        worst = max(worst, abs(fd - (eg[e] + eg[int(rev[e])]).item()) / (abs(fd) + 1))
    print(f"central differences: dh {err:.1e}, egrad (per pair, relative) {worst:.1e}")
    assert worst < 1e-6


def test_edge_case_graph_reaches_the_kernel_edges():
    c = ref.kernel_case()
    deg = (c["row_ptr"][1:] - c["row_ptr"][:-1]).tolist()
    for want in (0, 1, 3, 4, 5, 9, 150):
        assert want in deg
    assert torch.equal(c["col"][c["rev"].long()], torch.repeat_interleave(torch.arange(len(deg)), torch.tensor(deg)).int())
    bins = np.clip(np.floor(c["d"].numpy() * (np.float32(1) / (np.float32(CUTOFF) / np.float32(K - 1)))).astype(int), 0, K - 1)
    counts = np.bincount(bins, minlength=K)
    assert (counts[:K - 1] > 0).all() and counts[K - 1] == 0
    assert counts.max() > ref.SPLIT * ref.CHUNK and counts.max() % ref.SPLIT != 0 and (counts[counts > 0] < ref.SPLIT).any()
    k0 = ref.band_start(c["d"].numpy(), CUTOFF, K)
    assert int(k0.min()) == 0 and int(k0.max()) == K - ref.BAND


@pytest.mark.parametrize("drop", ref.DROPS)
def test_each_term_is_visible(drop):
    """Leaving out one term moves some output by more than 10x its bound A on the GPU tests' inputs, so the GPU tests can see it."""
    c = ref.kernel_case()
    h, dh, A_h, A_dh = ref.filter1(c["d"], c["w1"][0], c["b1"][0], c["offsets"], c["coeff"], CUTOFF)
    h2, dh2, _, _ = ref.filter1(c["d"], c["w1"][0], c["b1"][0], c["offsets"], c["coeff"], CUTOFF, drop=drop)
    args = (c["y"], c["G1"], c["b2"], c["d"], c["row_ptr"], c["col"], CUTOFF)
    agg, A_agg = ref.cfconv_fwd(*args)
    agg2, _ = ref.cfconv_fwd(*args, drop=drop)
    bargs = (c["y"], c["G1"], c["G2"], c["b2"], c["d"], c["row_ptr"], c["col"], c["rev"], CUTOFF, c["gagg"], c["egrad0"][:, 3])
    gy, A_gy, eg, A_eg = ref.cfconv_bwd(*bargs)
    gy2, _, eg2, _ = ref.cfconv_bwd(*bargs, drop=drop)
    moved = max(ref.max_ratio((a - b).abs(), A) for a, b, A in ((h, h2, A_h), (dh, dh2, A_dh), (agg, agg2, A_agg), (gy, gy2, A_gy), (eg, eg2, A_eg)))
    print(f"without {drop}: max |change| / A = {moved:.1e}")
    assert moved > 10


def test_shifted_basis_is_mis_banded():
    """GaussianRBF(100, 5.0, start=0.5) passes the kernels' width check (coeff (7 dx)^2 = -30.2 < -23), yet the band chosen from
    floor(d / dx) with dx = cutoff / (K - 1) misses most of sum_k phi_k at some distances; the basis starting at 0 misses nothing."""
    d = torch.linspace(0.01, CUTOFF - 0.01, 4000, dtype=torch.float64)
    missed = {}
    for start in (0.0, 0.5):
        offsets = torch.linspace(start, CUTOFF, K, dtype=torch.float64)
        coeff = -0.5 / float(offsets[1] - offsets[0]) ** 2
        dx = ref.spacing(CUTOFF, K)
        assert coeff * (7 * dx) ** 2 < -23  # not refused by the kernels' own check
        phi, _, _ = ref.gaussians(d, offsets, coeff)
        band = ref.in_band(d.numpy(), CUTOFF, K).double()
        missed[start] = ((phi * (1 - band)).sum(1) / phi.sum(1)).max().item()
    print(f"largest fraction of sum phi outside the band: start 0 {missed[0.0]:.1e}, start 0.5 {missed[0.5]:.2f}")
    assert missed[0.0] < 1e-12 and missed[0.5] > 0.9


def _spk_model(rep_cls, start=0.0):
    from nabladft_b200 import spk

    return spk.NeuralNetworkPotential(
        representation=rep_cls(n_atom_basis=128, n_interactions=1, radial_basis=spk.GaussianRBF(n_rbf=K, cutoff=CUTOFF, start=start),
                               cutoff_fn=spk.CosineCutoff(cutoff=CUTOFF)),
        input_modules=[spk.PairwiseDistances()], output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()])


@pytest.mark.parametrize("rep", ["SchNet", "PaiNN"])
def test_export_refuses_a_basis_the_band_cannot_evaluate(rep):
    from nabladft_b200 import spk

    cls = getattr(spk, rep)
    _, scalars = _spk_model(cls)._export(False)
    assert scalars["rbf_coeff"] == pytest.approx(-0.5 / ref.spacing(CUTOFF, K) ** 2, rel=1e-6)
    with pytest.raises(NotImplementedError, match="offsets"):
        _spk_model(cls, start=0.5)._export(False)
    m = _spk_model(cls)
    m.representation.radial_basis.widths.mul_(1.5)  # a checkpoint's buffer
    with pytest.raises(NotImplementedError, match="widths"):
        m._export(False)
    m = _spk_model(cls)
    m.representation.radial_basis.offsets.add_(0.01)
    with pytest.raises(NotImplementedError, match="offsets"):
        m._export(False)
