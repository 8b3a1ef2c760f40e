"""PaiNN training gradients at the benchmark batch (synth_batch(1, 256): 9,750 atoms, 80-atom node tiles, ~312k edges) against the float64
oracle's double backward, for every parameter, fp32 and bf16 edge storage.

The loss is L = sum_m c_m E_m + sum_i v_i . F_i with fixed seeds c and v (not an MSE against targets, so the fp32 energy error does not leak
into the seeds).  Molecules do not interact, so
  * dL/dtheta of the whole batch is the sum of dL/dtheta over disjoint slices of molecules: the oracle runs 32 molecules at a time on the
    CPU while the device runs the full batch;
  * with c and v zero outside a molecule set S, the device's full-batch gradient equals the oracle's gradient on S alone.  The device still
    runs every node tile, weight-gradient chunk and side-stream leaf of the full batch, and a one-molecule S makes a defect in its tile or
    chunk a large share of the result.  S is the first molecule, the first molecule across an 80-atom tile boundary, a molecule with an atom
    whose three xyz rows of the 3N-row dU weight gradient straddle a 128-row chunk, or the last molecule (ragged last node tile and chunk).

Every layer block of a stacked parameter is compared on its own (max|g - g_ref| / max|g_ref|), and only the embedding rows of elements in the
batch; rows of absent elements must be exactly zero."""
import time

import pytest
import torch

from test_gpu_node_tile import _wide
from test_gpu_painn import _Data, _oc_model, _spk_model

L, F = 6, 128
# Gates, with the largest values measured on an H100 80GB HBM3 (700 W power limit) beside them.
E_TOL, F_TOL = 1e-5, 1e-4      # Ha, Ha/A, fp32 (measured 5.3e-6, 6.3e-7)
# fp32 gradients: each block within G_TOL of its largest entry (measured: full batch 1.3e-5, masked energy-only 2.4e-6).  Seeding the
# forces of ONE molecule with random v leaves gradients that are small sums of large terms: the oracle itself, run in float32 autograd on
# the CPU, misses the fp64 gradient of the oc update_layers.3.vec_proj block by 1.0e-4 on the tile-boundary molecule, so the masked E + F
# cases get G_TOL_EF (device measured 6.7e-5 on that block).
G_TOL, G_TOL_EF = 5e-5, 1.5e-4
# bf16 edge storage (8 mantissa bits in the per-edge filter rows W, dW/dd and the per-edge filter gradients), against float64.  Measured:
# max|dE| 2.1e-4 Ha, max|dF| 4.0e-4 Ha/A; gradients 2.4e-2 (full batch), 3.4e-3 (masked energy-only), 2.4e-1 max / 4.9e-2 norm-relative
# (masked E + F, ill-conditioned as above: bf16 rounding is amplified like fp32 rounding is).
BF16_E_TOL, BF16_F_TOL = 5e-4, 1e-3
BF16_G_TOL, BF16_G_TOL_E, BF16_G_TOL_EF, BF16_G_NORM_TOL_EF = 5e-2, 1e-2, 5e-1, 1e-1
N_SLICE = 32                   # molecules per oracle slice
OC_KW = dict(hidden_channels=128, num_layers=L, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)


def dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------ batches and seeds
def _batch(seed, n_mol, n_take):
    """The first n_take molecules of synth_batch(seed, n_mol) as CPU tensors: z [N], pos [N, 3] (float32 values), batch [N], mol_ptr [B + 1]."""
    from nabladft_b200.synth import synth_batch

    b = synth_batch(seed, n_mol)
    ptr = torch.from_numpy(b["mol_ptr"][:n_take + 1]).long()
    n = int(ptr[-1])
    return torch.from_numpy(b["z"][:n]).long(), torch.from_numpy(b["pos"][:n]), torch.from_numpy(b["batch"][:n]).long(), ptr


def _seeds(n_mol, n_atoms, gen_seed):
    """c ~ N(0, 1) per molecule and v ~ N(0, 1) per atom component, drawn in float32 so device and oracle see the same values."""
    g = torch.Generator().manual_seed(gen_seed)
    return torch.randn(n_mol, generator=g), torch.randn(n_atoms, 3, generator=g)


def _masked(c, v, ptr, mols):
    """The seeds c, v with every molecule outside `mols` zeroed."""
    cm, vm = torch.zeros_like(c), torch.zeros_like(v)
    for m in mols:
        a, b = int(ptr[m]), int(ptr[m + 1])
        cm[m], vm[a:b] = c[m], v[a:b]
    return cm, vm


PROBES = ("first", "tile_boundary", "chunk_boundary", "last")


def _probe_molecules(ptr, batch, tile=80, chunk=128):
    """The seeded molecule of each masked case: the first molecule; the first molecule across a `tile`-atom node tile boundary; a further
    molecule holding an atom a whose rows 3a..3a+2 of the 3N-row dU weight gradient straddle a `chunk`-row chunk; the last molecule."""
    n_mol = ptr.numel() - 1
    across_tile = next(m for m in range(n_mol) if int(ptr[m]) // tile != (int(ptr[m + 1]) - 1) // tile)
    straddling = (a for a in range(batch.numel()) if (3 * a) // chunk != (3 * a + 2) // chunk)
    across_chunk = next(m for m in (int(batch[a]) for a in straddling) if m not in (0, across_tile))
    return dict(zip(PROBES, (0, across_tile, across_chunk, n_mol - 1)))


def _sub_batch(z, pos, ptr, mols):
    """Molecules `mols` (ascending) as a batch of their own, and their atom indices in the original batch."""
    idx = torch.cat([torch.arange(int(ptr[m]), int(ptr[m + 1])) for m in mols])
    batch = torch.cat([torch.full((int(ptr[m + 1] - ptr[m]),), k, dtype=torch.long) for k, m in enumerate(mols)])
    return z[idx], pos[idx], batch, idx


# ------------------------------------------------------------------ float64 oracle
def _oracle(flavour, state_dict):
    if flavour == "spk":
        from oracle.spk import NeuralNetworkPotential as OracleNNP
        from oracle.spk import SpkPaiNN

        ref = OracleNNP(SpkPaiNN(n_interactions=L)).double()
        ref.load_state_dict({k: state_dict[k].double().cpu() for k in ref.state_dict()}, strict=True)
    else:
        from oracle.painn_oc import PaiNNOC

        ref = PaiNNOC(**OC_KW).double()
        ref.load_state_dict({k: v.double().cpu() for k, v in state_dict.items()}, strict=True)
    return ref


def _oracle_grads(flavour, ref, z, pos, batch, c, v=None):
    """E, F and d(sum_m c_m E_m [+ sum_i v_i . F_i])/dtheta of the float64 oracle on one batch (double backward through the forces)."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr

    ref.zero_grad(set_to_none=True)
    p = pos.double().clone()
    if flavour == "spk":
        idx_i, idx_j = ase_neighbor_list(p, batch_to_ptr(batch), 5.0)
        out = ref({"_atomic_numbers": z, "_positions": p, "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False,
                  create_graph=True)
        e, f = out["energy"], out["forces"]
    else:
        e, f = ref(z, p, batch, create_graph=True)
    loss = (c.double() * e).sum()
    if v is not None:
        loss = loss + (v.double() * f).sum()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in ref.named_parameters() if p.grad is not None}
    return grads, e.detach(), f.detach()


def _oracle_sum_of_slices(flavour, ref, z, pos, ptr, c, v, n_slice):
    """The oracle's gradient of the whole batch as the sum over slices of n_slice molecules, and its E, F."""
    n_mol = ptr.numel() - 1
    total, es, fs = None, [], []
    for m0 in range(0, n_mol, n_slice):
        m1 = min(m0 + n_slice, n_mol)
        a, b = int(ptr[m0]), int(ptr[m1])
        batch = torch.repeat_interleave(torch.arange(m1 - m0), ptr[m0 + 1:m1 + 1] - ptr[m0:m1])
        g, e, f = _oracle_grads(flavour, ref, z[a:b], pos[a:b], batch, c[m0:m1], None if v is None else v[a:b])
        total = g if total is None else {k: total[k] + g[k] for k in total}
        es.append(e)
        fs.append(f)
    return total, torch.cat(es), torch.cat(fs)


# ------------------------------------------------------------------ comparison
def _emb_name(flavour):
    return "representation.embedding.weight" if flavour == "spk" else "atom_emb.embeddings.weight"


def _blocks(flavour, name, g):
    """(label, tensor) per layer block: the stacked spk filter network splits into its L row blocks of 3F."""
    if flavour == "spk" and name.startswith("representation.filter_net."):
        return [(f"{name}[{l}]", g[l * 3 * F:(l + 1) * 3 * F]) for l in range(L)]
    return [(name, g)]


def _compare(flavour, ours, ref_g, z, tag):
    """{block: (max|g - g_ref| / max|g_ref|, ||g - g_ref|| / ||g_ref||)} over every parameter the oracle differentiates; prints the worst."""
    emb_rows = torch.unique(z) - (0 if flavour == "spk" else 1)
    stats = {}
    for name, gr in ref_g.items():
        g = ours.get(name)
        assert g is not None and g.shape == gr.shape, name
        g = g.double().cpu()
        if name == _emb_name(flavour):
            absent = torch.ones(g.shape[0], dtype=torch.bool)
            absent[emb_rows] = False
            assert torch.count_nonzero(g[absent]) == 0, f"{tag}: embedding rows of elements absent from the batch have a gradient"
            g, gr = g[emb_rows], gr[emb_rows]
        for (label, gb), (_, rb) in zip(_blocks(flavour, name, g), _blocks(flavour, name, gr)):
            den_max, den_norm = float(rb.abs().max()), float(rb.norm())
            assert den_max > 0, f"{tag}: the oracle's {label} block is zero"
            stats[label] = (float((gb - rb).abs().max()) / den_max, float((gb - rb).norm()) / den_norm)
    worst = max(stats, key=lambda k: stats[k][0])
    print(f"{tag}: worst block {worst}: max-rel {stats[worst][0]:.2e}, norm-rel {stats[worst][1]:.2e}")
    return stats


def _assert_within(stats, tol, tag):
    bad = {k: v for k, v in stats.items() if v[0] > tol}
    assert not bad, f"{tag}: blocks above {tol:.0e} of their largest entry: {bad}"


# ------------------------------------------------------------------ device
def _device_model(flavour):
    return (_spk_model(L) if flavour == "spk" else _oc_model(L)).to(dev()).train()


def _device_step(flavour, net, z, pos, batch, ptr, c, v, storage, recompute=False):
    """One training step through the public module: E, F and d(sum c E [+ sum v . F])/dtheta per named parameter.  With `recompute` a
    second training forward runs before backward(), so the backward takes the one-call path that recomputes the forward
    (nb200_painn_energy_forces_grads) instead of the kept activations."""
    if flavour == "spk":
        inputs = {"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
                  "_n_atoms": (ptr[1:] - ptr[:-1]).to(dev())}
        call = lambda: (lambda o: (o["energy"], o["forces"]))(net(inputs))
    else:
        inputs = _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev()))
        call = lambda: net(inputs)
    net.train_edge_storage = storage
    net.zero_grad(set_to_none=True)
    e, f = call()
    eng = net._train_engine
    assert eng.edge_storage == storage
    token = eng._kept_token
    if recompute:
        call()
        assert not eng.kept(token)
    else:
        assert eng.kept(token)
    loss = (c.to(dev()) * e).sum()
    if v is not None:
        loss = loss + (v.to(dev()) * f).sum()
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    return grads, e.detach().double().cpu(), f.detach().double().cpu()


# ------------------------------------------------------------------ full batch against the oracle's sum of slices
@pytest.fixture(scope="module")
def full_batch():
    """synth_batch(1, 256), its seeds and the oracle's E, F and gradients (sum over 8 slices of 32 molecules), computed once."""
    z, pos, batch, ptr = _batch(1, 256, 256)
    c, v = _seeds(256, z.numel(), 7)
    ref = _oracle("spk", _spk_model(L).state_dict())
    t0 = time.perf_counter()
    g, e, f = _oracle_sum_of_slices("spk", ref, z, pos, ptr, c, v, N_SLICE)
    print(f"\nfloat64 oracle, {z.numel()} atoms in {256 // N_SLICE} slices of {N_SLICE} molecules: {time.perf_counter() - t0:.1f} s "
          f"on {torch.get_num_threads()} threads")
    return dict(z=z, pos=pos, batch=batch, ptr=ptr, c=c, v=v, g=g, e=e, f=f)


def _check_full(fb, storage, recompute, e_tol, f_tol, g_tol, tag):
    assert _wide(fb["z"].numel())   # 9,750 atoms: one wave of 80-atom tiles
    net = _device_model("spk")
    g, e, f = _device_step("spk", net, fb["z"], fb["pos"], fb["batch"], fb["ptr"], fb["c"], fb["v"], storage, recompute)
    de, df = float((e - fb["e"]).abs().max()), float((f - fb["f"]).abs().max())
    print(f"{tag}: max|dE| {de:.2e} Ha, max|dF| {df:.2e} Ha/A")
    stats = _compare("spk", g, fb["g"], fb["z"], tag)
    assert de < e_tol and df < f_tol, (de, df)
    _assert_within(stats, g_tol, tag)
    return g, e


@pytest.mark.gpu
def test_full_batch_gradients_match_oracle_sum_of_slices(full_batch):
    _check_full(full_batch, "f32", False, E_TOL, F_TOL, G_TOL, "full batch, fp32, two-call")


@pytest.mark.gpu
def test_full_batch_one_call_path_matches_oracle(full_batch):
    _check_full(full_batch, "f32", True, E_TOL, F_TOL, G_TOL, "full batch, fp32, one-call")


@pytest.mark.gpu
def test_full_batch_bf16_edge_storage_matches_oracle(full_batch):
    fb = full_batch
    _, e16 = _check_full(fb, "bf16", False, BF16_E_TOL, BF16_F_TOL, BF16_G_TOL, "full batch, bf16, two-call")
    _, e32, _ = _device_step("spk", _device_model("spk"), fb["z"], fb["pos"], fb["batch"], fb["ptr"], fb["c"], None, "f32")
    assert not torch.equal(e16, e32)   # the bf16 step did run with bf16 edge rows


@pytest.mark.gpu
def test_full_batch_gradients_repeat_run_to_run():
    """Two identical steps: the weight-gradient atomics flush in a different order (measured 2e-6 of a tensor's largest entry); a side-stream
    leaf reading a buffer the chain already overwrote would show as a larger difference."""
    z, pos, batch, ptr = _batch(1, 256, 256)
    c, v = _seeds(256, z.numel(), 7)
    net = _device_model("spk")
    g1, _, _ = _device_step("spk", net, z, pos, batch, ptr, c, v, "f32")
    g2, _, _ = _device_step("spk", net, z, pos, batch, ptr, c, v, "f32")
    diff = {}
    for name in g1:
        for (label, a), (_, b) in zip(_blocks("spk", name, g1[name].double()), _blocks("spk", name, g2[name].double())):
            diff[label] = float((a - b).abs().max() / a.abs().max().clamp_min(1e-30))
    worst = max(diff, key=diff.get)
    print(f"run to run: worst block {worst}: {diff[worst]:.2e} of its largest entry")
    assert diff[worst] < 1e-5, {k: d for k, d in diff.items() if d >= 1e-5}


# ------------------------------------------------------------------ masked seeds: one tile, chunk or tail at a time
_MASKED_ORACLE = {}


@pytest.mark.gpu
@pytest.mark.parametrize("probe", PROBES)
@pytest.mark.parametrize("shape", [(1, 256, 256), (1, 400, 247)], ids=["b256", "b247"])
@pytest.mark.parametrize("loss", ["energy", "energy_forces"])
@pytest.mark.parametrize("storage", ["f32", "bf16"])
@pytest.mark.parametrize("flavour", ["spk", "oc"])
def test_masked_seed_gradients_match_oracle_on_the_seeded_molecule(flavour, storage, loss, shape, probe):
    """Seeds on one molecule of a full batch.  Energy-only seeds run the primal weight-gradient leaves (wg_primal, nb_filter_wgrad); E + F
    seeds run wgrad_tc3 and the tangent leaves.  synth_batch(1, 400) cut to 247 molecules has 9,441 atoms: its last 80-atom tile holds one
    atom."""
    z, pos, batch, ptr = _batch(*shape)
    N = z.numel()
    assert _wide(N)
    if shape[2] == 247:
        assert N % 80 == 1
    mols = [_probe_molecules(ptr, batch)[probe]]
    c, v = _masked(*_seeds(ptr.numel() - 1, N, 11), ptr, mols)
    if loss == "energy":
        v = None
    net = _device_model(flavour)
    key = (flavour, loss, shape, probe)
    if key not in _MASKED_ORACLE:   # shared by the f32 and bf16 cases
        zs, ps, bs, idx = _sub_batch(z, pos, ptr, mols)
        ref = _oracle(flavour, net.state_dict())
        _MASKED_ORACLE[key] = _oracle_grads(flavour, ref, zs, ps, bs, c[mols], None if v is None else v[idx]) + (idx,)
    g_ref, e_ref, f_ref, idx = _MASKED_ORACLE[key]
    g, e, f = _device_step(flavour, net, z, pos, batch, ptr, c, v, storage)
    tag = f"masked {flavour} {storage} {loss}, {shape[2]} molecules / {N} atoms, {probe} molecule {mols[0]} (atoms {int(idx[0])}..{int(idx[-1])})"
    de, df = float((e[mols] - e_ref).abs().max()), float((f[idx] - f_ref).abs().max())
    print(f"{tag}: max|dE| {de:.2e} Ha, max|dF| {df:.2e} Ha/A")
    stats = _compare(flavour, g, g_ref, z, tag)
    if storage == "f32":
        e_tol, f_tol, g_tol = E_TOL, F_TOL, (G_TOL if loss == "energy" else G_TOL_EF)
    else:
        e_tol, f_tol, g_tol = BF16_E_TOL, BF16_F_TOL, (BF16_G_TOL_E if loss == "energy" else BF16_G_TOL_EF)
    assert de < e_tol and df < f_tol, (de, df)
    _assert_within(stats, g_tol, tag)
    if storage == "bf16" and loss == "energy_forces":
        bad = {k: s for k, s in stats.items() if s[1] > BF16_G_NORM_TOL_EF}
        assert not bad, f"{tag}: blocks above {BF16_G_NORM_TOL_EF:.0e} norm-relative: {bad}"


# ------------------------------------------------------------------ the comparison itself, on the CPU
@pytest.mark.parametrize("flavour", ["spk", "oc"])
def test_oracle_gradient_is_a_sum_over_molecules(flavour):
    """The arithmetic the GPU cases rest on, in float64: the gradient of an 8-molecule batch equals the sum over two slices of 4, and with
    seeds zero outside S it equals the gradient of S run as a batch of its own, to 1e-12 of each tensor's largest entry."""
    z, pos, batch, ptr = _batch(3, 8, 8)
    c, v = _seeds(8, z.numel(), 5)
    sd = (_spk_model(L) if flavour == "spk" else _oc_model(L)).state_dict()
    ref = _oracle(flavour, sd)
    whole, e, f = _oracle_grads(flavour, ref, z, pos, batch, c, v)
    sliced, es, fs = _oracle_sum_of_slices(flavour, ref, z, pos, ptr, c, v, 4)

    def rel(a, b):
        return max(float((a[k] - b[k]).abs().max() / b[k].abs().max()) for k in b)

    assert set(whole) == set(sliced)
    assert rel(sliced, whole) < 1e-12
    assert float((es - e).abs().max()) < 1e-12 and float((fs - f).abs().max()) < 1e-12
    mols = [1, 6]
    cm, vm = _masked(c, v, ptr, mols)
    masked, _, _ = _oracle_grads(flavour, ref, z, pos, batch, cm, vm)
    zs, ps, bs, idx = _sub_batch(z, pos, ptr, mols)
    alone, e_s, f_s = _oracle_grads(flavour, ref, zs, ps, bs, c[mols], v[idx])
    assert rel(masked, alone) < 1e-12
    assert float((e_s - e[mols]).abs().max()) < 1e-12 and float((f_s - f[idx]).abs().max()) < 1e-12
    # every oracle block the GPU cases compare is non-zero, so "relative to its largest entry" is defined
    for k, g in alone.items():
        if k == _emb_name(flavour):
            g = g[torch.unique(zs) - (0 if flavour == "spk" else 1)]
        for label, gb in _blocks(flavour, k, g):
            assert float(gb.abs().max()) > 0, label
