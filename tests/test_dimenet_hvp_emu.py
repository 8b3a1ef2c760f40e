"""DimeNet++ Hessian-vector products (nabladft_b200/csrc/dimenet_hvp.inc) checked on the CPU through the host-emulation build (tests/emu,
name="dimenet"): the second distance derivatives of the radial bases against float64 closed forms, hv = (d^2 y / dR dR) v of the unscaled
prediction y against the float64 oracle's double backward (models built with the scaler on and do_postprocessing=True), collinear geometries
against central differences of the oracle's forces, degenerate batches, bitwise repeatability and the C ABI argument checks.  Every buffer is
poisoned with 0xFF bytes before a call and the guard zones behind every workspace array are checked after it."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))

from make_golden_dimenet import grid_molecule  # noqa: E402
from test_dimenet_emu import _fixture, _models  # noqa: E402

REL = 1e-4  # of max |H_ref| (of max |hv_ref| for single directions): the criterion of the training gradients


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.dimenetplusplus import DimeNetRunner

    lib = load("dimenet", ["nb200_dimenet_"])
    EmuRunner = poisoned(DimeNetRunner, checked=["run_hvp", "run"])
    return lambda: EmuRunner(lib), lib


def _runner(emu, net, z, pos, batch):
    """(runner, z, pos, mol_ptr, n_mol) for the mirror on the host arrays."""
    make, _ = emu
    r = make()
    r.set_weights(net, torch.device("cpu"))
    return (r,) + tuple(net.batch_args(torch.as_tensor(z), torch.as_tensor(pos).float(), torch.as_tensor(batch).long()))


def _oracle_hvp(ora, z, pos, batch, vs):
    """float64 double backward of the unscaled prediction: [(d^2 sum_m y_m / dR dR) v for v in vs]; one forward, one backward per v."""
    pos = torch.as_tensor(pos).double().detach().requires_grad_(True)
    g = ora.net(z=torch.as_tensor(z).long(), pos=pos, batch=torch.as_tensor(batch).long())
    y = ora.regr_or_cls_nn(g).sum()
    dy = torch.autograd.grad(y, pos, create_graph=True)[0]
    return torch.stack([torch.autograd.grad(dy, pos, grad_outputs=torch.as_tensor(v).double(), retain_graph=True)[0] for v in vs])


def _oracle_fd_hvp(ora, z, pos, batch, vs, h=1e-5):
    """float64 central differences of the oracle's forces, -(F(R + h v) - F(R - h v)) / 2h, with the edge set checked equal at both sides."""
    from oracle.dimenet import radius_graph_kp1

    zz, bb = torch.as_tensor(z).long(), torch.as_tensor(batch).long()
    p0 = torch.as_tensor(pos).double()
    out = []
    for v in vs:
        v = torch.as_tensor(v).double()
        ep = radius_graph_kp1(p0 + h * v, bb, ora.net.cutoff, ora.net.max_num_neighbors)
        em = radius_graph_kp1(p0 - h * v, bb, ora.net.cutoff, ora.net.max_num_neighbors)
        assert torch.equal(ep, em), "the edge set changes within the finite-difference step"
        fp = ora(zz, p0 + h * v, bb)[1]
        fm = ora(zz, p0 - h * v, bb)[1]
        out.append(-(fp - fm) / (2 * h))
    return torch.stack(out)


def _dirs(n_dir, n_atoms, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(n_dir, n_atoms, 3, generator=gen, dtype=torch.float64)


def _close(got, ref, what):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"{what}: max |err| {err:.3e}, relative to max |ref| {err / (scale + 1e-30):.2e}")
    assert scale > 0 and err <= REL * scale, (what, err, scale)


def test_emu_radial_second_derivatives_against_float64(emu):
    """d^2 rbs / dd^2 and d^2 rbf / dd^2 from 0.05 A to the cutoff against float64 closed forms (scipy spherical_jn, j_l'' from the spherical
    Bessel equation), relative to each function's largest |value| over the range checked.  From 0.5 A (shorter than any bond): 2e-5 (the
    first derivative is held to 5e-6 there).  Over the whole range: 5e-4.  Below 0.5 A the three terms env'' j + 2 env' z j' + env z^2 j''
    are O(1 / x^2) larger than their sum for l = 1 and for rbf (whose values stay finite as x -> 0) and cancel in any fp32 evaluation of
    them, as the two terms of the first derivative do."""
    from scipy.special import spherical_jn

    from nabladft_b200.dimenetplusplus import DimeNetRunner, sbf_radial_constants

    _, lib = emu
    net, _ = _models(num_blocks=1)
    r = DimeNetRunner.__new__(DimeNetRunner)
    r.set_weights(net, torch.device("cpu"))
    m = 500
    d = torch.linspace(0.05, 4.99, m, dtype=torch.float32)
    d2rbs = torch.full((m, 42), float("nan"))
    d2rbf = torch.full((m, 6), float("nan"))
    assert lib.nb200_dimenet_debug_sbf_radial_d2(ctypes.byref(r._w), d.data_ptr(), m, d2rbs.data_ptr(), d2rbf.data_ptr(), None) == 0
    zn, norms = sbf_radial_constants()
    c = 5.0
    x = d.double().numpy() / c
    p = 6
    a, b, cc = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    env = 1 / x + a * x ** (p - 1) + b * x ** p + cc * x ** (p + 1)
    denv = -1 / x ** 2 + a * (p - 1) * x ** (p - 2) + b * p * x ** (p - 1) + cc * (p + 1) * x ** p
    d2env = 2 / x ** 3 + a * (p - 1) * (p - 2) * x ** (p - 3) + b * p * (p - 1) * x ** (p - 2) + cc * (p + 1) * p * x ** (p - 1)
    far = d.numpy() >= 0.5

    def rel(got, ref):
        e = np.abs(got.double().numpy() - ref)
        return e.max() / np.abs(ref).max(), e[far].max() / np.abs(ref[far]).max()

    worst = [0.0, 0.0]
    for l in range(7):
        for n in range(6):
            zz = zn[l, n]
            y = zz * x
            j, dj = spherical_jn(l, y), spherical_jn(l, y, derivative=True)
            d2j = -2.0 / y * dj + (l * (l + 1) / y ** 2 - 1.0) * j
            ref = norms[l, n] * (d2env * j + 2 * denv * zz * dj + env * zz ** 2 * d2j) / c ** 2
            err = rel(d2rbs[:, l * 6 + n], ref)
            worst = [max(worst[0], err[0]), max(worst[1], err[1])]
            assert err[0] <= 5e-4 and err[1] <= 2e-5, (l, n, err)
    freq = net.net.rbf.freq.detach().double().numpy()
    for n in range(6):
        f = freq[n]
        ref = (d2env * np.sin(f * x) + 2 * denv * f * np.cos(f * x) - env * f ** 2 * np.sin(f * x)) / c ** 2
        err = rel(d2rbf[:, n], ref)
        worst = [max(worst[0], err[0]), max(worst[1], err[1])]
        assert err[0] <= 5e-4 and err[1] <= 2e-5, (n, err)
    print(f"worst relative error {worst[0]:.2e} from 0.05 A, {worst[1]:.2e} from 0.5 A")


def test_emu_full_hessian_of_molecule_26(emu):
    """Every column of the 87 x 87 Hessian of fixture molecule 26 (29 atoms) at 2 blocks / L = 16; energies and forces of the same call are
    bitwise those of the inference call."""
    from nabladft_b200 import vibrations as vib

    net, ora = _models(num_blocks=2, latent=16)
    z, pos, batch = _fixture([26])
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    calls = []

    def hvp(v):
        e, f, hv = r.run_hvp(zz, pp, mol_ptr, n_mol, v)
        calls.append((e, f))
        return hv

    hs = vib.hessians_from_hvp(hvp, mol_ptr.tolist(), max_dir=29)
    n3 = 3 * len(z)
    ref = _oracle_hvp(ora, z, pos, batch, torch.eye(n3, dtype=torch.float64).reshape(n3, len(z), 3)).reshape(n3, n3)
    _close(hs[0], ref, "Hessian")
    assert hs.max_asymmetry <= REL * ref.abs().max().item()
    e_ref, f_ref, _ = r.run(zz, pp, mol_ptr, n_mol)
    assert len(calls) == 3 and all(torch.equal(e, e_ref) and torch.equal(f, f_ref) for e, f in calls)


def test_emu_random_directions_at_config_sizes(emu):
    """6 blocks, L = 50, K = 32: three random directions on two fixture molecules at once."""
    net, ora = _models()
    z, pos, batch = _fixture([3, 39])
    vs = _dirs(3, len(z), 0)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    _, _, hv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous(), with_forces=False)
    ref = _oracle_hvp(ora, z, pos, batch, vs)
    for k in range(3):
        _close(hv[k], ref[k], f"direction {k}")


def _chain():
    chain = np.array([[0, 0, 0], [1.2, 0, 0], [2.4, 0, 0], [3.6, 0, 0], [20.0, 0, 0]], dtype=np.float32)
    return np.array([6, 6, 8, 1, 1], dtype=np.int32), chain


@pytest.mark.parametrize("geometry", ["chain", "grid"])
def test_emu_collinear_triplets_against_central_differences(emu, geometry):
    """Exactly collinear triplets, where the oracle's atan2 angle has NaN second derivatives: random directions against float64 central
    differences of the oracle's forces at h = 1e-5 A (converged there: h = 1e-4 and 1e-5 agree to ~1e-6 relative)."""
    net, ora = _models(num_blocks=2, latent=16)
    z, pos = _chain() if geometry == "chain" else grid_molecule()
    batch = np.zeros(len(z), dtype=np.int64)
    vs = _dirs(2, len(z), 1)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    e, f, hv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous())
    ref = _oracle_fd_hvp(ora, z, pos, batch, vs)
    for k in range(len(vs)):
        _close(hv[k], ref[k], f"{geometry} direction {k}")
    if geometry == "chain":
        assert (hv[:, 4] == 0).all()  # the atom out of everyone's cutoff


def test_emu_isolated_one_atom_and_edge_free(emu):
    """An isolated atom and a one-atom molecule get hv = 0 exactly; an edge-free batch gives hv = 0 everywhere.  Energies and forces are the
    inference call's."""
    net, ora = _models(num_blocks=2, latent=16)
    zc, chain = _chain()
    z = np.concatenate([zc, np.array([8], dtype=np.int32)])
    pos = np.concatenate([chain, np.array([[0.0, 1.0, 2.0]], dtype=np.float32)])
    batch = np.array([0, 0, 0, 0, 0, 1])
    for z_, pos_, batch_ in ((z, pos, batch), (np.array([1, 6, 8], dtype=np.int32), np.array([[0, 0, 0], [9, 0, 0], [0, 9, 0]], dtype=np.float32),
                                                np.array([0, 0, 1]))):
        vs = _dirs(2, len(z_), 2)
        r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z_, pos_, batch_)
        e, f, hv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous())
        e_ref, f_ref, _ = r.run(zz, pp, mol_ptr, n_mol)
        assert torch.equal(e, e_ref) and torch.equal(f, f_ref)
        assert torch.isfinite(hv).all()
        if len(z_) == 6:
            assert (hv[:, 4:] == 0).all() and hv[:, :4].abs().max() > 0
            _close(hv[:, :4], _oracle_fd_hvp(ora, z_, pos_, batch_, vs)[:, :4], "chain + single atom")
        else:
            assert r.last_counts["edges"] == 0 and (hv == 0).all()


def test_emu_bitwise_repeatable_and_chunk_independent(emu):
    from nabladft_b200 import vibrations as vib

    net, _ = _models(num_blocks=1, latent=16)
    z, pos, batch = _fixture([26])
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z[:12], pos[:12], batch[:12])
    vs = _dirs(2, 12, 3).float().contiguous()
    a = r.run_hvp(zz, pp, mol_ptr, n_mol, vs)
    b = r.run_hvp(zz, pp, mol_ptr, n_mol, vs)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    e_ref, f_ref, _ = r.run(zz, pp, mol_ptr, n_mol)
    assert torch.equal(a[0], e_ref) and torch.equal(a[1], f_ref)

    def hvp(v):
        return r.run_hvp(zz, pp, mol_ptr, n_mol, v, with_forces=False)[2]

    h1 = vib.hessians_from_hvp(hvp, mol_ptr.tolist(), max_dir=1)
    h7 = vib.hessians_from_hvp(hvp, mol_ptr.tolist(), max_dir=7)
    assert torch.equal(h1[0], h7[0]) and h1.max_asymmetry == h7.max_asymmetry


def test_emu_hvp_c_abi_argument_checks(emu):
    from nabladft_b200 import _lib

    NB200_EINVAL, NB200_EUNSUPPORTED = -1, -2
    make, lib = emu
    net, _ = _models(num_blocks=1)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, *_fixture([0]))
    gbuf, counts = r._graph(zz, pp, mol_ptr, n_mol)
    n = int(zz.shape[0])
    wbytes = lib.nb200_dimenet_hvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts)
    assert wbytes > lib.nb200_dimenet_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) > 0
    ws = torch.empty(wbytes, dtype=torch.uint8)
    v = torch.zeros(2, n, 3)
    v[0, 0, 0] = v[1, 3, 2] = 1.0
    energy, forces, hv = torch.empty(n_mol), torch.empty(n, 3), torch.empty(2, n, 3)

    def call(**kw):
        a = dict(eng=r._h, w=ctypes.byref(r._w), z=zz.data_ptr(), pos=pp.data_ptr(), mp=mol_ptr.data_ptr(), n_mol=n_mol, n=n, g=gbuf.data_ptr(),
                 gb=gbuf.numel(), counts=counts, ws=ws.data_ptr(), wb=wbytes, n_dir=2, v=v.data_ptr(), e=energy.data_ptr(), f=forces.data_ptr(),
                 hv=hv.data_ptr())
        a.update(kw)
        return lib.nb200_dimenet_hvp(*a.values(), None)

    assert call() == 0 and call(f=None) == 0
    hv.fill_(7.0)
    big = (ctypes.c_int64 * 4)(n * 33 + 1, counts[1], 0, 0)  # more edges than the graph buffer holds
    for bad in (dict(eng=None), dict(z=None), dict(pos=None), dict(mp=None), dict(g=None), dict(counts=None), dict(ws=None), dict(v=None),
                dict(e=None), dict(hv=None), dict(n_dir=0), dict(n_dir=-1), dict(wb=wbytes - 1), dict(gb=16), dict(n_mol=0), dict(n=0),
                dict(counts=big)):
        assert call(**bad) == NB200_EINVAL, bad
    assert (hv == 7.0).all()  # nothing launched
    assert lib.nb200_emu_check_guards() < 0  # the zones of the calls above, checked while their buffers are alive
    assert lib.nb200_dimenet_hvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, None) == NB200_EINVAL
    r._w.num_radial = 5
    assert call() == NB200_EUNSUPPORTED
    assert lib.nb200_dimenet_hvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) == NB200_EUNSUPPORTED
    r._w.num_radial = 6
    # the real library (pure host code here) agrees with the emulation build up to the guard zones
    real = _lib.load()
    assert 0 < real.nb200_dimenet_hvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) <= wbytes
    with pytest.raises(Exception, match="v must be"):
        r.run_hvp(zz, pp, mol_ptr, n_mol, torch.zeros(0, n, 3))
