"""Training through the CUDA engine (energy losses): parameter gradients against the oracle's autograd."""
import numpy as np
import pytest
import torch

from helpers import load_fixture, load_golden_weights
from test_gpu_painn import _Data, _oc_model, _spk_model, dev

pytestmark = pytest.mark.gpu


def _rel_err(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _check(ours_named, ref_named, tol):
    worst = {}
    for k, g_ref in ref_named.items():
        g = ours_named[k]
        assert g is not None and g.shape == g_ref.shape, k
        worst[k] = _rel_err(g.double().cpu(), g_ref)
    bad = {k: v for k, v in worst.items() if v > tol}
    assert not bad, bad
    return worst


def test_painn_oc_energy_loss_param_grads_match_oracle():
    from oracle.painn_oc import PaiNNOC

    kw = dict(hidden_channels=128, num_layers=3, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)
    net = _oc_model(3)
    ref = PaiNNOC(**kw).double()
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
    z, pos, batch = load_fixture([0, 4, 7])
    c = torch.tensor([0.7, -1.3, 0.4], dtype=torch.float64)
    e_ref, f_ref = ref(z, pos.clone(), batch, create_graph=True)
    (c * e_ref).sum().backward()
    ref_g = {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}

    net = net.to(dev()).train()
    e, f = net(_Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())))
    assert e.requires_grad
    (c.float().to(dev()) * e).sum().backward()
    ours = {k: p.grad for k, p in net.named_parameters()}
    assert np.abs(e.detach().cpu().numpy() - e_ref.detach().numpy()).max() < 1e-5
    assert np.abs(f.detach().cpu().numpy() - f_ref.detach().numpy()).max() < 1e-4
    # fp32 sums over ~130 atoms / ~2600 edges against fp64: 2e-4 of each tensor's largest entry
    _check(ours, ref_g, 2e-4)
    assert set(ref_g) <= set(k for k, g in ours.items() if g is not None)


def test_spk_painn_energy_loss_param_grads_match_oracle():
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkPaiNN

    model = _spk_model(3)
    ref = OracleNNP(SpkPaiNN(n_interactions=3)).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    ref.train()
    z, pos, batch = load_fixture([10, 11, 60])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False,
                  create_graph=True)
    target = torch.tensor([-3.0, 1.0, 0.5], dtype=torch.float64)
    ((out_ref["energy"] - target) ** 2).mean().backward()
    ref_g = {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}

    model = model.to(dev()).train()
    n_atoms = torch.bincount(batch)
    out = model({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": n_atoms.to(dev())})
    ((out["energy"] - target.float().to(dev())) ** 2).mean().backward()
    ours = {k: p.grad for k, p in model.named_parameters()}
    _check(ours, ref_g, 5e-4)  # the loss seed 2 (E - t) / B carries the fp32 energy error (1e-6 relative) into every gradient


@pytest.mark.parametrize("which", ["force_only", "energy_and_force"])
def test_force_loss_param_grads_match_oracle_double_backward(which):
    """loss = MSE(E) + MSE(F) as the reference trains (painn.py:642-653).  Oracle: autograd double backward (create_graph=True).
    Ours: forward-over-reverse tangent pass in the engine (painn_tangent.cu) -- exact, so the same 1e-6-level agreement as the
    energy term is expected; tolerance 5e-5 of each tensor's largest entry."""
    from oracle.painn_oc import PaiNNOC

    kw = dict(hidden_channels=128, num_layers=3, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)
    net = _oc_model(3)
    ref = PaiNNOC(**kw).double()
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
    z, pos, batch = load_fixture([0, 4, 7])
    g = torch.Generator().manual_seed(3)
    e_t = torch.tensor([-9.0, -12.0, -10.5], dtype=torch.float64)
    f_t = 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
    we = 0.0 if which == "force_only" else 1.0

    def loss(e, f, dt):
        return we * ((e - e_t.to(dt).to(e.device)) ** 2).mean() + ((f - f_t.to(dt).to(f.device)) ** 2).mean()

    e_ref, f_ref = ref(z, pos.clone(), batch, create_graph=True)
    loss(e_ref, f_ref, torch.float64).backward()
    ref_g = {k: p.grad for k, p in ref.named_parameters() if p.grad is not None and float(p.grad.abs().max()) > 0}
    net = net.to(dev()).train()
    e, f = net(_Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())))
    loss(e, f, torch.float32).backward()
    ours = {k: p.grad for k, p in net.named_parameters()}
    worst = _check(ours, ref_g, 5e-5)
    print(which, "worst relative error per tensor:", max(worst.values()))


def test_spk_painn_energy_and_force_loss_grads_match_oracle():
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkPaiNN

    model = _spk_model(3)
    ref = OracleNNP(SpkPaiNN(n_interactions=3)).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    ref.train()
    z, pos, batch = load_fixture([10, 11, 60])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch}, postprocess=False,
                  create_graph=True)
    g = torch.Generator().manual_seed(5)
    e_t = torch.tensor([-3.0, 1.0, 0.5], dtype=torch.float64)
    f_t = 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
    (((out_ref["energy"] - e_t) ** 2).mean() + 10.0 * ((out_ref["forces"] - f_t) ** 2).mean()).backward()
    ref_g = {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}
    model = model.to(dev()).train()
    n_atoms = torch.bincount(batch)
    out = model({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": n_atoms.to(dev())})
    (((out["energy"] - e_t.float().to(dev())) ** 2).mean() + 10.0 * ((out["forces"] - f_t.float().to(dev())) ** 2).mean()).backward()
    ours = {k: p.grad for k, p in model.named_parameters()}
    _check(ours, ref_g, 5e-4)


def test_full_size_energy_force_step_cfg3_shape():
    """BASELINE configs[2] batch shape (256 synthetic conformations per GPU): one E+F training step through the reference-facing
    spk module; size-independent property -- a gradient step sized to remove 10 % of the loss to first order removes 10 %."""
    from nabladft_b200.synth import synth_batch

    b = synth_batch(2, 256)
    model = _spk_model(6).to(dev()).train()
    n_atoms = torch.from_numpy(b["mol_ptr"][1:] - b["mol_ptr"][:-1]).to(dev())
    inputs = {"_atomic_numbers": torch.from_numpy(b["z"]).to(dev()), "_positions": torch.from_numpy(b["pos"]).to(dev()),
              "_idx_m": torch.from_numpy(b["batch"]).to(dev()), "_n_atoms": n_atoms}
    gen = torch.Generator(device="cpu").manual_seed(1)
    with torch.no_grad():
        model.eval(); out0 = model(inputs); model.train()
    e_t = out0["energy"] + 0.2 * torch.randn(256, generator=gen).to(dev())
    f_t = out0["forces"] + 0.05 * torch.randn(out0["forces"].shape, generator=gen).to(dev())

    def loss_of(out):
        return ((out["energy"] - e_t) ** 2).mean() + ((out["forces"] - f_t) ** 2).mean()

    loss = loss_of(model(inputs))
    loss.backward()
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert all(torch.isfinite(g).all() for g in grads)
    g2 = sum(float((g.double() ** 2).sum()) for g in grads)
    eta = 0.1 * float(loss.detach()) / g2
    with torch.no_grad():
        for p in model.parameters():
            if p.grad is not None:
                p -= eta * p.grad
    ratio = float(loss_of(model(inputs)).detach() / loss.detach())
    assert 0.85 < ratio < 0.95, ratio


def test_gradient_step_reduces_energy_mse_as_predicted():
    """One plain gradient step sized to remove 10 % of the loss to first order must remove 10 % +- second-order terms: checks the
    whole gradient (every tensor, the export permutations, the autograd bridge) as a directional derivative on the device."""
    net = _oc_model(2).to(dev()).train()
    z, pos, batch = load_fixture([3, 5, 8, 9])
    data = _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev()))
    with torch.no_grad():
        net.eval()
        e0, _ = net(data)
        net.train()
    target = e0 + torch.tensor([0.3, -0.2, 0.1, 0.25], device=dev())
    e, _ = net(data)
    loss = ((e - target) ** 2).mean()
    loss.backward()
    g2 = sum(float((p.grad.double() ** 2).sum()) for p in net.parameters() if p.grad is not None)
    eta = 0.1 * float(loss.detach()) / g2
    with torch.no_grad():
        for p in net.parameters():
            if p.grad is not None:
                p -= eta * p.grad
    e1, _ = net(data)
    ratio = float(((e1.detach() - target) ** 2).mean() / loss.detach())
    assert 0.85 < ratio < 0.95, ratio


def test_two_call_training_step_matches_the_recomputing_path():
    """The training forward keeps its activations in the engine workspace and the backward call builds the gradients from them
    (nb200_painn_train_forward / _backward); a second forward on the same engine before the backward invalidates the kept state and the
    backward falls back to the one-call form that recomputes.  Both must give the same gradients (both run the fused node forward; the
    weight-gradient kernels accumulate with atomics, so their sums are reordered: agreement within 5e-5 of each tensor's largest entry)."""
    z, pos, batch = load_fixture([0, 4, 7, 9])
    g = torch.Generator().manual_seed(11)
    e_t = torch.tensor([-9.0, -12.0, -10.5, -8.0])
    f_t = 0.05 * torch.randn(pos.shape, generator=g)
    data = _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev()))

    def grads_of(net, invalidate):
        net.zero_grad(set_to_none=True)
        e, f = net(data)
        eng = net._train_engine
        kept_before = eng._kept_token
        if invalidate:
            net(data)   # a second training forward on the same engine: the workspace now holds ITS activations (other weights key)
            assert not eng.kept(kept_before)
        else:
            assert eng.kept(kept_before) and kept_before != 0
        (((e - e_t.to(dev())) ** 2).mean() + ((f - f_t.to(dev())) ** 2).mean()).backward()
        return {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}, e.detach().clone(), f.detach().clone()

    net = _oc_model(3).to(dev()).train()
    kept, e1, f1 = grads_of(net, invalidate=False)
    redo, e2, f2 = grads_of(net, invalidate=True)
    assert float((e1 - e2).abs().max()) < 1e-5 and float((f1 - f2).abs().max()) < 1e-5
    assert set(kept) == set(redo)
    worst = {k: _rel_err(kept[k].double(), redo[k].double()) for k in kept}
    print("kept vs recomputed, worst relative difference per tensor:", max(worst.values()))
    assert max(worst.values()) < 5e-5, {k: v for k, v in worst.items() if v > 5e-5}


@pytest.mark.parametrize("flavour", ["oc", "spk"])
def test_bf16_edge_storage_training_step_tracks_the_fp32_step(flavour):
    """BASELINE configs[2] "bf16": the per-edge arrays of the training calls (filter rows W, dW/dd, per-edge filter gradients) stored as
    bf16, fp32 arithmetic and accumulation (nb200_engine_set_edge_storage).  Its own, looser gate -- bf16 keeps 8 mantissa bits, and the
    rounding errors of ~20 filter rows per atom average out: energies within 2e-3 Ha and forces within 2e-3 Ha/A of the fp32 engine,
    every parameter gradient of an MSE(E) + MSE(F) loss within 2 % of its largest entry (measured: see the printed numbers)."""
    z, pos, batch = load_fixture([0, 4, 7, 9])
    g = torch.Generator().manual_seed(5)
    e_t = torch.tensor([-9.0, -12.0, -10.5, -8.0])
    f_t = 0.05 * torch.randn(pos.shape, generator=g)
    if flavour == "oc":
        net = _oc_model(3).to(dev()).train()
        inputs = _Data(z.to(dev()), pos.float().to(dev()), batch.to(dev()))
        call = lambda: net(inputs)
    else:
        net = _spk_model(3).to(dev()).train()
        inputs = {"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": torch.bincount(batch).to(dev())}
        call = lambda: (lambda o: (o["energy"], o["forces"]))(net(inputs))

    def run(storage):
        net.train_edge_storage = storage
        net.zero_grad(set_to_none=True)
        e, f = call()
        assert net._train_engine.edge_storage == storage
        (((e - e_t.to(dev())) ** 2).mean() + ((f - f_t.to(dev())) ** 2).mean()).backward()
        return {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}, e.detach().clone(), f.detach().clone()

    g32, e32, f32 = run("f32")
    g16, e16, f16 = run("bf16")
    g32b, _, _ = run("f32")   # switching back restores the fp32 path exactly
    de, df = float((e16 - e32).abs().max()), float((f16 - f32).abs().max())
    worst = {k: _rel_err(g16[k].double(), g32[k].double()) for k in g32}
    print(f"bf16 edge storage ({flavour}): max|dE| {de:.2e} Ha, max|dF| {df:.2e} Ha/A, worst relative gradient difference {max(worst.values()):.2e} ({max(worst, key=worst.get)})")
    assert de > 0 and de < 2e-3 and df < 2e-3
    assert max(worst.values()) < 2e-2, {k: v for k, v in worst.items() if v > 2e-2}
    assert max(_rel_err(g32b[k].double(), g32[k].double()) for k in g32) < 1e-5


def test_two_call_training_c_abi_argument_checks():
    """nb200_painn_train_forward / _backward and nb200_engine_set_edge_storage refuse inconsistent arguments before touching the device."""
    from ctypes import byref

    from nabladft_b200 import _lib

    net = _oc_model(2).to(dev()).train()
    z, pos, batch = load_fixture([0, 4])
    e, f = net(_Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())))   # sizes the training engine's workspace
    eng = net._train_engine
    lib, h, w = eng.lib, eng._h, eng._weights
    n_mol, n_atoms, e_cap, wfs, _, _ = eng._kept_args
    zz, pp = z.to(dev()).int().contiguous(), pos.float().to(dev()).contiguous()
    mp = torch.tensor([0, int((batch == 0).sum()), n_atoms], dtype=torch.int32, device=dev())
    en, fo = torch.empty(n_mol, device=dev()), torch.empty(n_atoms, 3, device=dev())
    ws, st = eng._ws, eng._status
    EINVAL = -1
    assert _lib.ERRORS[EINVAL].startswith("NB200_EINVAL")
    # forward without a forces buffer
    assert lib.nb200_painn_train_forward(h, byref(w), _lib.ptr(zz), _lib.ptr(pp), _lib.ptr(mp), n_mol, n_atoms, e_cap, _lib.ptr(ws), ws.numel(), 1,
                                         _lib.ptr(en), None, _lib.ptr(st), _lib.current_stream()) == EINVAL
    # workspace too small for the training layout
    assert lib.nb200_painn_train_forward(h, byref(w), _lib.ptr(zz), _lib.ptr(pp), _lib.ptr(mp), n_mol, n_atoms, e_cap, _lib.ptr(ws), 1024, 1,
                                         _lib.ptr(en), _lib.ptr(fo), _lib.ptr(st), _lib.current_stream()) == EINVAL
    # backward with a force seed although the workspace was sized without the tangent pass
    grads, gw = eng._grad_struct()
    seed = torch.ones(n_mol, device=dev())
    assert lib.nb200_painn_train_backward(h, byref(w), _lib.ptr(zz), _lib.ptr(mp), n_mol, n_atoms, e_cap, _lib.ptr(ws), ws.numel(), 0, _lib.ptr(seed),
                                          _lib.ptr(fo), byref(gw), _lib.ptr(st), _lib.current_stream()) == EINVAL
    # backward without gradient buffers
    assert lib.nb200_painn_train_backward(h, byref(w), _lib.ptr(zz), _lib.ptr(mp), n_mol, n_atoms, e_cap, _lib.ptr(ws), ws.numel(), 1, _lib.ptr(seed),
                                          None, None, _lib.ptr(st), _lib.current_stream()) == EINVAL
    # a weight-gradient array that is not 16-byte aligned (the weight-gradient kernel writes 16-byte rows)
    gw.A1 = grads["A1"].data_ptr() + 4
    assert lib.nb200_painn_train_backward(h, byref(w), _lib.ptr(zz), _lib.ptr(mp), n_mol, n_atoms, e_cap, _lib.ptr(ws), ws.numel(), wfs, _lib.ptr(seed),
                                          None, byref(gw), _lib.ptr(st), _lib.current_stream()) == EINVAL
    assert lib.nb200_engine_set_edge_storage(h, 2) == EINVAL
    with pytest.raises(ValueError):
        eng.set_edge_storage("fp8")
    torch.cuda.synchronize()
