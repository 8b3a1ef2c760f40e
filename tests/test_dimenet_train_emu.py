"""DimeNet++ training gradients (nabladft_b200/csrc/dimenet_train.inc) checked on the CPU through the host-emulation build (tests/emu,
name="dimenet"): the parameter gradients of sum_m c_m E_m + sum_i v_i . F_i, from nb200_dimenet_train_grads through the differentiable weight
export, against float64 autograd of the oracle with create_graph=True (the reference's force loss).  Every buffer is poisoned with 0xFF
bytes before a call and the guard zones behind every workspace array are checked after it."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))

from make_golden_dimenet import SCALER, grid_molecule, load_test_weights  # noqa: E402
from test_dimenet_emu import _fixture, _models  # noqa: E402

REL = 1e-4  # of max |g_ref| of each tensor


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.dimenetplusplus import DimeNetRunner

    lib = load("dimenet", ["nb200_dimenet_"])
    EmuRunner = poisoned(DimeNetRunner, checked=["train_grads"])
    return lambda: EmuRunner(lib), lib


def _engine_grads(emu, net, z, pos, batch, c, v):
    """name -> gradient of the mirror's parameters, through train_grads and the differentiable export."""
    make, _ = emu
    r = make()
    net.zero_grad(set_to_none=True)
    flat, offs = net._export_impl(detach=False)
    r.bind(net, flat.detach(), offs)
    zz, pp, mol_ptr, n_mol = net.batch_args(torch.as_tensor(z), torch.as_tensor(pos).float(), torch.as_tensor(batch).long())
    g = r.train_grads(zz, pp, mol_ptr, n_mol, None if c is None else c.float(), None if v is None else v.float())
    assert torch.isfinite(g).all()
    flat.backward(g)
    return {k: (p.grad if p.grad is not None else torch.zeros_like(p)).double() for k, p in net.named_parameters()}


def _oracle_grads(ora, z, pos, batch, c, v):
    """float64 autograd of sum c_m E_m + sum v . F with F = -d(sum y)/dR kept in the graph (create_graph=True)."""
    ora.zero_grad(set_to_none=True)
    pos = torch.as_tensor(pos).double().detach().requires_grad_(True)
    g = ora.net(z=torch.as_tensor(z).long(), pos=pos, batch=torch.as_tensor(batch).long())
    y = ora.regr_or_cls_nn(g).flatten()
    loss = torch.zeros((), dtype=torch.float64)
    if c is not None:
        loss = loss + (c.double() * (SCALER["scale_"] * y + SCALER["mean_"])).sum()
    if v is not None:
        dy = torch.autograd.grad(y.sum(), pos, create_graph=True, allow_unused=True)[0]
        if dy is not None:
            loss = loss - (v.double() * dy).sum()
    if loss.requires_grad:
        loss.backward()
    return {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in ora.named_parameters()}


def _check(got, ref, n_params, nonzero=True, zero_ok=()):
    assert len(ref) == n_params and set(got) == set(ref)
    worst = (0.0, "")
    for k, gr in ref.items():
        scale = gr.abs().max().item()
        if nonzero and k not in zero_ok:
            assert scale > 0, f"{k}: reference gradient is zero"
        err = (got[k] - gr).abs().max().item()
        worst = max(worst, (err / (scale + 1e-30), k))
        assert err <= REL * scale + 1e-9, (k, err, scale)
    print(f"worst relative error {worst[0]:.2e} in {worst[1]}")


def _seeds(n_mol, n_atoms, seed=0):
    gen = torch.Generator().manual_seed(seed)
    c = torch.randn(n_mol, generator=gen, dtype=torch.float64)
    c[::2] *= -1.0
    return c, torch.randn(n_atoms, 3, generator=gen, dtype=torch.float64)


@pytest.mark.parametrize("layout", [(6, 50, [0, 1, 2]), (2, 16, [3, 11])])
def test_emu_energy_loss_gradients(emu, layout):
    """sum c_m E_m with mixed signs: every reference-named parameter (221 at 6 blocks, 89 at 2)."""
    nb, latent, mols = layout
    net, ora = _models(num_blocks=nb, latent=latent)
    z, pos, batch = _fixture(mols)
    c, _ = _seeds(len(mols), len(z))
    _check(_engine_grads(emu, net, z, pos, batch, c, None), _oracle_grads(ora, z, pos, batch, c, None), 221 if nb == 6 else 89)


@pytest.mark.parametrize("layout", [(6, 50, [0, 1, 2]), (2, 16, [3, 11])])
def test_emu_energy_and_force_loss_gradients(emu, layout):
    nb, latent, mols = layout
    net, ora = _models(num_blocks=nb, latent=latent)
    z, pos, batch = _fixture(mols)
    c, v = _seeds(len(mols), len(z), 1)
    _check(_engine_grads(emu, net, z, pos, batch, c, v), _oracle_grads(ora, z, pos, batch, c, v), 221 if nb == 6 else 89)


def test_emu_force_only_and_grid_molecule(emu):
    """Force-only seeds on fixture molecules, and E + F on the 48-atom grid (K + 1 truncation, asymmetric edges, collinear triplets)."""
    net, ora = _models(num_blocks=2, latent=16)
    z, pos, batch = _fixture([5, 7])
    _, v = _seeds(2, len(z), 2)
    # the forces do not depend on the last bias of the head
    _check(_engine_grads(emu, net, z, pos, batch, None, v), _oracle_grads(ora, z, pos, batch, None, v), 89, zero_ok={"regr_or_cls_nn.6.bias"})
    zg, pg = grid_molecule()
    bg = np.zeros(len(zg), dtype=np.int64)
    c, v = _seeds(1, len(zg), 3)
    _check(_engine_grads(emu, net, zg, pg, bg, c, v), _oracle_grads(ora, zg, pg, bg, c, v), 89)


def test_emu_degenerate_batches(emu):
    """An isolated atom and a one-atom molecule give finite gradients equal to the oracle's.  In an edge-free batch only the head and the
    per-atom layers of the output blocks (lins, lin: silu(bias) chains) are reached."""
    net, ora = _models(num_blocks=2, latent=16)
    chain = np.array([[0, 0, 0], [1.2, 0, 0], [2.4, 0.3, 0], [3.6, 0, 0.2], [20.0, 0, 0]], dtype=np.float32)
    pos = np.concatenate([chain, np.array([[0.0, 1.0, 2.0]], dtype=np.float32)])
    z = np.array([6, 6, 8, 1, 1, 8], dtype=np.int32)
    batch = np.array([0, 0, 0, 0, 0, 1])
    c, v = _seeds(2, 6, 4)
    _check(_engine_grads(emu, net, z, pos, batch, c, v), _oracle_grads(ora, z, pos, batch, c, v), 89, nonzero=False)
    far = np.array([[0, 0, 0], [9, 0, 0], [0, 9, 0]], dtype=np.float32)
    c, v = _seeds(2, 3, 5)
    got = _engine_grads(emu, net, np.array([1, 6, 8], dtype=np.int32), far, np.array([0, 0, 1]), c, v)
    ref = _oracle_grads(ora, np.array([1, 6, 8]), far, np.array([0, 0, 1]), c, v)
    _check(got, ref, 89, nonzero=False)
    assert all(got[k].abs().max() > 0 for k in got if k.startswith("regr_or_cls_nn"))
    edge_free = [k for k in got if k.startswith(("net.rbf", "net.emb", "net.interaction_blocks")) or ".lin_rbf." in k or ".lin_up." in k]
    assert len(edge_free) == 1 + 5 + 2 * 24 + 3 * 2 and all(got[k].abs().max() == 0 for k in edge_free)


def test_emu_sgd_step_matches_oracle(emu):
    """One SGD step on L1(E) + L1(F) moves every parameter as the oracle's step does."""
    net, ora = _models(num_blocks=2, latent=16)
    z, pos, batch = _fixture([2, 9])
    e_t = torch.tensor([-40.0, -75.0], dtype=torch.float64)
    f_t = 0.1 * _seeds(2, len(z), 6)[1]
    e_ref, f_ref, _ = ora(torch.as_tensor(z).long(), torch.as_tensor(pos).double(), torch.as_tensor(batch).long())
    # seeds of mean-L1 losses at the oracle's (E, F): the engine's forward agrees with it to 1e-5 Ha, far from the kinks
    c = torch.sign(e_ref - e_t) / len(e_t)
    v = torch.sign(f_ref - f_t) / f_t.numel()
    got = _engine_grads(emu, net, z, pos, batch, c, v)
    ref = _oracle_grads(ora, z, pos, batch, c, v)
    lr = 1e-2
    before = {k: p.detach().double().clone() for k, p in net.named_parameters()}
    opt = torch.optim.SGD(net.parameters(), lr=lr)
    opt.step()
    for k, p in net.named_parameters():
        step, step_ref = p.detach().double() - before[k], -lr * ref[k]
        assert (step - step_ref).abs().max() <= REL * step_ref.abs().max() + 1e-6, k
    assert any((p.detach().double() - before[k]).abs().max() > 0 for k, p in net.named_parameters())


def test_emu_train_c_abi_argument_checks(emu):
    from nabladft_b200 import _lib

    NB200_EINVAL, NB200_EUNSUPPORTED = -1, -2
    make, lib = emu
    net, _ = _models(num_blocks=1)
    r = make()
    r.set_weights(net, torch.device("cpu"))
    z, pos, batch = _fixture([0])
    zz, pp, mol_ptr, n_mol = net.batch_args(torch.as_tensor(z), torch.as_tensor(pos).float(), torch.as_tensor(batch).long())
    gbuf, counts = r._graph(zz, pp, mol_ptr, n_mol)
    n = int(zz.shape[0])
    wbytes = lib.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts)
    assert wbytes > lib.nb200_dimenet_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) > 0
    ws = torch.empty(wbytes, dtype=torch.uint8)
    grads = torch.zeros_like(r._keep[0])
    seed = torch.ones(n_mol)

    def call(**kw):
        a = dict(eng=r._h, w=ctypes.byref(r._w), z=zz.data_ptr(), pos=pp.data_ptr(), mp=mol_ptr.data_ptr(), n_mol=n_mol, n=n, g=gbuf.data_ptr(),
                 gb=gbuf.numel(), counts=counts, ws=ws.data_ptr(), wb=wbytes, se=seed.data_ptr(), sf=None, grads=grads.data_ptr())
        a.update(kw)
        return lib.nb200_dimenet_train_grads(*a.values(), None)

    assert call() == 0
    for bad in (dict(eng=None), dict(z=None), dict(pos=None), dict(mp=None), dict(g=None), dict(ws=None), dict(grads=None), dict(wb=wbytes - 1),
                dict(gb=16), dict(n_mol=0), dict(n=0)):
        assert call(**bad) == NB200_EINVAL, bad
    assert lib.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, None) == NB200_EINVAL
    r._w.num_radial = 5
    assert call() == NB200_EUNSUPPORTED
    assert lib.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) == NB200_EUNSUPPORTED
    r._w.num_radial = 6
    # the real library (pure host code here) agrees with the emulation build up to the guard zones
    real = _lib.load()
    assert 0 < real.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) <= wbytes
    assert real.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) > \
        real.nb200_dimenet_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts)
