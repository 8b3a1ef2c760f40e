"""GemNet-OC force-Jacobian products (nabladft_b200/csrc/gemnet_oc_jvp.inc) checked on the CPU through the host-emulation build (tests/emu):
jv = -(dF/dR) v of the direct forces against the float64 oracle's autograd (oracle/gemnet_oc.py, test weights with random scale factors),
degenerate geometries against float64 central differences of the oracle's forces, trivial molecules, bitwise repeatability and chunking, the
outputs of the training forward and the C ABI argument checks.  Every buffer is poisoned with 0xFF bytes before a call and the guard zones
behind every workspace array, tangent mirror included, are checked after it."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))

from test_gemnet_emu import _models  # noqa: E402

REL = 1e-4  # of max |J_ref| (of max |jv_ref| for single directions): DimeNet++'s bound for its Hessians


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.gemnet_oc import GemNetOCRunner

    lib = load("gemnet_oc", ["nb200_gemnet_oc_"])
    EmuRunner = poisoned(GemNetOCRunner, checked=["run_hvp", "run_train"])
    return lambda: EmuRunner(lib), lib


@pytest.fixture(scope="module")
def models():
    net, ora = _models(True)  # scale factors != 1: the tangents pass through the folded basis matrices
    return net, ora.double()


def _runner(emu, net, z, pos, batch):
    """(runner, z int32, pos fp32, mol_ptr int32, n_mol) on the host arrays."""
    make, _ = emu
    r = make()
    r.set_weights(net, torch.device("cpu"))
    batch = torch.as_tensor(batch).long()
    n_mol = int(batch.max()) + 1
    mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32)
    mol_ptr[1:] = torch.cumsum(torch.bincount(batch, minlength=n_mol), 0)
    return r, torch.as_tensor(z).to(torch.int32).contiguous(), torch.as_tensor(pos).float().contiguous(), mol_ptr, n_mol


def _fixture(mol, n_atoms=None):
    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    a, b = fx["ptr"][mol], fx["ptr"][mol + 1]
    b = b if n_atoms is None else a + n_atoms
    return fx["z"][a:b].astype(np.int64), fx["pos"][a:b].astype(np.float32), np.zeros(b - a, dtype=np.int64)


def _forces(ora, z, batch):
    zz, bb = torch.as_tensor(z).long(), torch.as_tensor(batch).long()
    return lambda p: ora(zz, p, bb)[1]


def _oracle_jvp(ora, z, pos, batch, vs):
    """float64 -(dF/dR) v by autograd (a forward and a double backward per direction)."""
    f, p0 = _forces(ora, z, batch), torch.as_tensor(pos).double()
    return torch.stack([-torch.autograd.functional.jvp(f, p0, torch.as_tensor(v).double())[1] for v in vs])


def _oracle_jacobian(ora, z, pos, batch):
    """float64 [3n, 3n]: J[i, j] = -dF_i / dR_j, one backward per row."""
    p = torch.as_tensor(pos).double().detach().requires_grad_(True)
    f = _forces(ora, z, batch)(p).reshape(-1)
    eye = torch.eye(f.numel(), dtype=torch.float64)
    return -torch.stack([torch.autograd.grad(f, p, grad_outputs=eye[k], retain_graph=True)[0].reshape(-1) for k in range(f.numel())])


def _graphs(pos, batch):
    from oracle.gemnet_graph import build_all_indices

    g = build_all_indices(pos, torch.as_tensor(batch).long())
    return [g[k]["edge_index"] for k in ("main", "a2a", "a2ee2a", "qint")]


def _oracle_fd_jvp(ora, z, pos, batch, vs, h=1e-5):
    """float64 central differences of the oracle's forces, -(F(R + h v) - F(R - h v)) / 2h, with the four graphs checked equal at both sides."""
    f, p0 = _forces(ora, z, batch), torch.as_tensor(pos).double()
    out = []
    for v in vs:
        v = torch.as_tensor(v).double()
        gp, gm = _graphs(p0 + h * v, batch), _graphs(p0 - h * v, batch)
        assert all(torch.equal(a, b) for a, b in zip(gp, gm)), "a graph changes within the finite-difference step"
        out.append(-(f(p0 + h * v) - f(p0 - h * v)) / (2 * h))
    return torch.stack(out)


def _dirs(n_dir, n_atoms, seed):
    return torch.randn(n_dir, n_atoms, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _close(got, ref, what):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"{what}: max |err| {err:.3e}, relative to max |ref| {err / (scale + 1e-30):.2e}")
    assert scale > 0 and err <= REL * scale, (what, err, scale)


def test_emu_full_jacobian_of_a_fixture_fragment(emu, models):
    """Every column of the 30 x 30 Jacobian of the first 10 atoms of fixture molecule 26 at config sizes, in one call; energies and forces
    are bitwise those of the training forward; the translation sum rule sum_j dF_i/dR_j = 0 holds to fp32 accuracy."""
    net, ora = models
    z, pos, batch = _fixture(26, 10)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    n3 = 3 * len(z)
    e, f, jv = r.run_hvp(zz, pp, mol_ptr, n_mol, torch.eye(n3).reshape(n3, len(z), 3).contiguous())
    J = jv.reshape(n3, n3).t()  # column j = jv of direction j
    ref = _oracle_jacobian(ora, z, pos, batch)
    _close(J, ref, "Jacobian")
    asym = (ref - ref.t()).abs().max().item()
    print(f"non-conservative part of the oracle's Jacobian: max |J - J^T| = {asym:.3e} (max |J| {ref.abs().max().item():.3e})")
    colsum = J.double().reshape(n3, len(z), 3).sum(1)
    assert colsum.abs().max().item() <= REL * ref.abs().max().item(), colsum.abs().max().item()
    e_ref, f_ref, _ = r.run_train(zz, pp, mol_ptr, n_mol, len(z))
    assert torch.equal(e, e_ref) and torch.equal(f, f_ref)


def test_emu_random_directions_on_the_golden_batch(emu, models):
    """Two random directions on the golden batch (two molecules, 79 atoms) at config sizes against the oracle's float64 JVPs."""
    net, ora = models
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    z, pos, batch = g["z"].astype(np.int64), g["pos"], g["batch"].astype(np.int64)
    vs = _dirs(2, len(z), 0)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    _, f, jv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous(), with_forces=False)
    assert f is None
    ref = _oracle_jvp(ora, z, pos, batch, vs)
    for k in range(2):
        _close(jv[k], ref[k], f"direction {k}")


def _pentagon():
    """A planar 5-ring (z = 0): every quadruplet's dihedral is 0 or pi, where the kernel's |n1 x n2| sits at its 1e-9 clamp."""
    ang = 2 * np.pi * np.arange(5) / 5
    rad = 1.4 / (2 * np.sin(np.pi / 5))
    pos = np.stack([rad * np.cos(ang), rad * np.sin(ang), np.zeros(5)], 1).astype(np.float32)
    return np.array([6, 6, 7, 6, 8]), pos


def _linear(far=False):
    """O=C=O along x (exactly collinear triplets, no quadruplets: a quadruplet needs four distinct atoms), optionally with an atom 30 A away
    (outside everyone's 12 A cutoff)."""
    pos = [[-1.16, 0, 0], [0, 0, 0], [1.16, 0, 0]] + ([[30.0, 0, 0]] if far else [])
    return np.array([8, 6, 8] + ([1] if far else [])), np.array(pos, dtype=np.float32)


@pytest.mark.parametrize("geometry", ["planar_ring", "collinear"])
def test_emu_degenerate_geometries_against_central_differences(emu, models, geometry):
    """Where autograd through the oracle's atan2 / norm / clamp is unreliable: random directions against float64 central differences of the
    oracle's forces at h = 1e-5 A.  For the planar ring the tangent of every cos(dihedral) is zero (an extremum at +-1), and the differences
    see no first-order change either."""
    net, ora = models
    z, pos = _pentagon()
    batch = np.zeros(len(z), dtype=np.int64)
    if geometry == "collinear":  # next to the ring, whose quadruplets the oracle's bases need (it cannot build an empty quadruplet basis)
        zl, pl = _linear()
        z, pos, batch = np.concatenate([zl, z]), np.concatenate([pl, pos]), np.concatenate([np.zeros(3, dtype=np.int64), batch + 1])
    vs = _dirs(2, len(z), 1)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    _, _, jv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous())
    if geometry == "planar_ring":
        assert r.last_counts["Q"] > 0 and r.last_counts["TIN"] > 0  # quadruplets are there
    ref = _oracle_fd_jvp(ora, z, pos, batch, vs)
    for k in range(len(vs)):
        _close(jv[k], ref[k], f"{geometry} direction {k}")


def test_emu_one_atom_molecule_isolated_atom_and_edge_free_batch(emu, models):
    """A one-atom molecule and an atom outside everyone's cutoff get jv = 0 exactly, and their neighbours in the batch the jv they get alone; a
    batch without edges is refused as the forward refuses it."""
    from nabladft_b200._lib import NablaB200Error

    net, _ = models
    zl, pl = _linear(far=True)
    zr, pr = _pentagon()
    z = np.concatenate([zl, [7], zr])
    pos = np.concatenate([pl, np.array([[0.0, 5.0, 0.0]], dtype=np.float32), pr])
    batch = np.array([0, 0, 0, 0, 1, 2, 2, 2, 2, 2])
    vs = _dirs(2, len(z), 2)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    _, _, jv = r.run_hvp(zz, pp, mol_ptr, n_mol, vs.float().contiguous())
    assert (jv[:, 3:5] == 0).all() and jv[:, :3].abs().max() > 0 and jv[:, 5:].abs().max() > 0
    keep = [0, 1, 2, 5, 6, 7, 8, 9]
    r2, zz2, pp2, mol_ptr2, n_mol2 = _runner(emu, net, z[keep], pos[keep], np.array([0, 0, 0, 1, 1, 1, 1, 1]))
    alone = r2.run_hvp(zz2, pp2, mol_ptr2, n_mol2, vs[:, keep].float().contiguous())[2]
    _close(jv[:, keep], alone.double(), "next to trivial molecules vs alone")
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, np.array([1, 6]), np.array([[0, 0, 0], [20, 0, 0]], dtype=np.float32), np.array([0, 1]))
    with pytest.raises(NablaB200Error, match="ENOEDGES"):
        r.run_hvp(zz, pp, mol_ptr, n_mol, torch.ones(1, 2, 3))


def test_emu_bitwise_repeatable_chunk_independent_and_training_outputs(emu, models):
    from nabladft_b200 import vibrations as vib

    net, _ = models
    z, pos, batch = _fixture(26, 8)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    vs = _dirs(6, len(z), 3).float().contiguous()
    a = r.run_hvp(zz, pp, mol_ptr, n_mol, vs)
    b = r.run_hvp(zz, pp, mol_ptr, n_mol, vs)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    ones = torch.cat([r.run_hvp(zz, pp, mol_ptr, n_mol, vs[k:k + 1].contiguous())[2] for k in range(6)])
    assert torch.equal(ones, a[2])  # 1 x 6 directions == 6 x 1
    e_ref, f_ref, _ = r.run_train(zz, pp, mol_ptr, n_mol, len(z))
    assert torch.equal(a[0], e_ref) and torch.equal(a[1], f_ref)

    def hvp(v):
        return r.run_hvp(zz, pp, mol_ptr, n_mol, v, with_forces=False)[2]

    h1 = vib.hessians_from_hvp(hvp, mol_ptr.tolist(), max_dir=1)
    h7 = vib.hessians_from_hvp(hvp, mol_ptr.tolist(), max_dir=7)
    assert torch.equal(h1[0], h7[0]) and h1.max_asymmetry == h7.max_asymmetry


def test_emu_jvp_c_abi_argument_checks(emu, models):
    from nabladft_b200 import _lib

    NB200_EINVAL = -1
    _, lib = emu
    net, _ = models
    z, pos, batch = _fixture(26, 6)
    r, zz, pp, mol_ptr, n_mol = _runner(emu, net, z, pos, batch)
    n, mx = int(zz.shape[0]), int(zz.shape[0])
    gbuf, counts = r._graph(pp, mol_ptr, n_mol, mx)
    wbytes = lib.nb200_gemnet_oc_jvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts)
    assert wbytes > lib.nb200_gemnet_oc_train_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) > 0
    ws = torch.empty(wbytes, dtype=torch.uint8)
    v = torch.zeros(2, n, 3)
    v[0, 0, 0] = v[1, 3, 2] = 1.0
    energy, forces, jv = torch.empty(n_mol), torch.empty(n, 3), torch.empty(2, n, 3)

    def call(**kw):
        a = dict(eng=r._h, w=ctypes.byref(r._w), z=zz.data_ptr(), pos=pp.data_ptr(), mp=mol_ptr.data_ptr(), n_mol=n_mol, n=n, mx=mx, g=gbuf.data_ptr(),
                 gb=gbuf.numel(), counts=counts, ws=ws.data_ptr(), wb=wbytes, n_dir=2, v=v.data_ptr(), e=energy.data_ptr(), f=forces.data_ptr(),
                 jv=jv.data_ptr())
        a.update(kw)
        return lib.nb200_gemnet_oc_jvp(*a.values(), None)

    assert call() == 0 and call(f=None) == 0 and call(e=None) == 0
    jv.fill_(7.0)
    energy.fill_(7.0)
    forces.fill_(7.0)
    over = [int(counts[k]) for k in range(8)]
    over[1] = n * (mx - 1) + 2  # more main-graph edges than rows of mx - 1 sources hold
    big = (ctypes.c_int64 * 8)(*over)
    neg = (ctypes.c_int64 * 8)(*[int(counts[k]) if k != 4 else -1 for k in range(8)])
    for bad in (dict(eng=None), dict(z=None), dict(pos=None), dict(mp=None), dict(g=None), dict(counts=None), dict(ws=None), dict(v=None),
                dict(jv=None), dict(n_dir=0), dict(n_dir=-1), dict(wb=wbytes - 1), dict(gb=16), dict(n_mol=0), dict(n=0), dict(mx=0),
                dict(counts=big), dict(counts=neg)):
        assert call(**bad) == NB200_EINVAL, bad
    assert (jv == 7.0).all() and (energy == 7.0).all() and (forces == 7.0).all()  # nothing launched
    assert lib.nb200_emu_check_guards() < 0  # the zones of the calls above, checked while their buffers are alive
    assert lib.nb200_gemnet_oc_jvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, None) == NB200_EINVAL
    assert lib.nb200_gemnet_oc_jvp_workspace_bytes(ctypes.byref(r._w), 0, n, counts) == NB200_EINVAL
    # the real library (pure host code here) agrees with the emulation build up to the guard zones
    real = _lib.load()
    assert 0 < real.nb200_gemnet_oc_jvp_workspace_bytes(ctypes.byref(r._w), n_mol, n, counts) <= wbytes
    with pytest.raises(Exception, match="v must be"):
        r.run_hvp(zz, pp, mol_ptr, n_mol, torch.zeros(0, n, 3))
