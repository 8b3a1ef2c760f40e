"""DimeNet++ engine source (nabladft_b200/csrc/dimenet.cu) checked on the CPU through its host-emulation build (tests/emu, name="dimenet"):
the SAME functors the GPU launches, run as loops, driven through the SAME C ABI and Python host code (weight export, two-phase graph /
workspace protocol), against the float64 oracle (oracle/dimenet.py).  Every buffer is poisoned with 0xFF bytes before a call and the guard
zones behind every workspace array are checked after it.  Says nothing about the tensor-core GEMM or launch configuration (-m gpu does)."""
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

E_TOL, F_TOL = 1e-5, 1e-4  # Ha, Ha/A


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.dimenetplusplus import DimeNetRunner

    lib = load("dimenet", ["nb200_dimenet_"])
    EmuRunner = poisoned(DimeNetRunner, checked=["run"])
    return lambda: EmuRunner(lib), lib


def _models(num_blocks=6, latent=50, scaler=SCALER, max_nb=32):
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    kw = dict(node_latent_dim=latent, scaler=scaler, dimenet_hidden_channels=256, dimenet_num_blocks=num_blocks, dimenet_max_num_neighbors=max_nb,
              do_postprocessing=True)
    net = DimeNetPlusPlusPotential(**kw).eval()
    ora = DimeNetPlusPlusPotentialOracle(**kw).double().eval()
    load_test_weights(ora)
    net.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    return net, ora


def _run(emu, net, z, pos, batch):
    make, _ = emu
    r = make()
    r.set_weights(net, torch.device("cpu"))
    args = net.batch_args(torch.as_tensor(z), torch.as_tensor(pos).float(), torch.as_tensor(batch).long())
    e, f, g = r.run(*args)
    return e.double(), f.double(), g.double(), r.last_counts


def _fixture(mols):
    from helpers import load_fixture

    z, pos, batch = load_fixture(mols, dtype=torch.float32)
    return z, pos, batch


def _compare(emu, net, ora, z, pos, batch):
    e, f, g, counts = _run(emu, net, z, pos, batch)
    e_ref, f_ref, g_ref = ora(torch.as_tensor(z).long(), torch.as_tensor(pos).double(), torch.as_tensor(batch).long())
    assert torch.isfinite(e).all() and torch.isfinite(f).all()
    de, df = (e - e_ref).abs().max().item(), (f - f_ref).abs().max().item() if f.numel() else 0.0
    assert de < E_TOL and df < F_TOL, (de, df, e, e_ref)
    return e, f, g, e_ref, f_ref, g_ref, counts


def test_emu_matches_golden_and_oracle(emu):
    """Fixture molecules of the golden file: energies, forces and graph embeddings against the reference wrapper's float64 output."""
    gd = np.load(os.path.join(HERE, "golden", "dimenet_f64.npz"))
    net, ora = _models()
    e, f, g, e_ref, f_ref, g_ref, counts = _compare(emu, net, ora, gd["z"], gd["pos"], gd["batch"])
    assert np.abs(e.numpy() - gd["energy"]).max() < E_TOL
    assert np.abs(f.numpy() - gd["forces"]).max() < F_TOL
    assert np.abs(g.numpy() - gd["graph_emb"]).max() < 1e-4 * max(1.0, np.abs(gd["graph_emb"]).max())
    assert counts["edges"] > 0 and counts["triplets"] > counts["edges"]


def test_emu_two_layouts_of_the_model(emu):
    """Fewer blocks and another latent width (the limits the engine states), fresh fixture molecules."""
    net, ora = _models(num_blocks=2, latent=16)
    z, pos, batch = _fixture([3, 11])
    _compare(emu, net, ora, z, pos, batch)


def test_emu_truncation_keeps_k_plus_one(emu):
    z, pos = grid_molecule()
    batch = np.zeros(len(z), dtype=np.int64)
    net, ora = _models(num_blocks=1)
    *_, counts = _compare(emu, net, ora, z, pos, batch)
    assert counts["edges"] == 33 * 32 + 15 * 33


def test_emu_collinear_isolated_and_edge_free(emu):
    """A linear chain (angles of exactly 0 and pi), an atom out of everyone's cutoff, a one-atom molecule and a batch without edges."""
    net, ora = _models(num_blocks=2)
    chain = np.array([[0, 0, 0], [1.2, 0, 0], [2.4, 0, 0], [3.6, 0, 0], [20.0, 0, 0]], dtype=np.float32)
    z = np.array([6, 6, 8, 1, 1], dtype=np.int32)
    single = np.array([[0.0, 1.0, 2.0]], dtype=np.float32)
    pos = np.concatenate([chain, single])
    zz = np.concatenate([z, np.array([8], dtype=np.int32)])
    batch = np.array([0, 0, 0, 0, 0, 1])
    e, f, *_ = _compare(emu, net, ora, zz, pos, batch)
    assert (f[4] == 0).all() and (f[5] == 0).all()
    far = np.array([[0, 0, 0], [9, 0, 0], [0, 9, 0]], dtype=np.float32)
    e, f, *_ = _compare(emu, net, ora, np.array([1, 6, 8], dtype=np.int32), far, np.array([0, 0, 1]))
    assert (f == 0).all()


def test_emu_rejects_bad_elements_and_coordinates(emu):
    from nabladft_b200._lib import NablaB200Error

    net, _ = _models(num_blocks=1)
    z, pos, batch = _fixture([0])
    bad_z = z.clone()
    bad_z[2] = 95
    with pytest.raises(NablaB200Error, match="EINVAL"):
        _run(emu, net, bad_z, pos, batch)
    bad_pos = pos.clone()
    bad_pos[4, 1] = float("nan")
    with pytest.raises(NablaB200Error, match="EINVAL"):
        _run(emu, net, z, bad_pos, batch)


def test_emu_repeat_calls_are_bitwise_equal(emu):
    net, _ = _models(num_blocks=2)
    z, pos, batch = _fixture([5])
    a = _run(emu, net, z, pos, batch)
    b = _run(emu, net, z, pos, batch)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_emu_sbf_radial_basis_against_scipy(emu):
    """env(x) N_ln j_l(z_ln x) in fp32 against scipy in float64 down to 0.05 A (the series branch), and its distance derivative from 0.5 A
    (shorter than any bond; below it the two terms of the derivative, -N j / (c x^2) and N z j' / (c x), cancel in any fp32 evaluation)."""
    from scipy.special import spherical_jn

    from nabladft_b200.dimenetplusplus import sbf_radial_constants

    _, lib = emu
    net, _ = _models(num_blocks=1)
    from nabladft_b200.dimenetplusplus import DimeNetRunner

    r = DimeNetRunner.__new__(DimeNetRunner)
    r.set_weights(net, torch.device("cpu"))
    d = torch.linspace(0.05, 4.99, 400, dtype=torch.float32)
    rbs = torch.empty(400, 42)
    drbs = torch.empty(400, 42)
    assert lib.nb200_dimenet_debug_sbf_radial(ctypes.byref(r._w), d.data_ptr(), 400, rbs.data_ptr(), drbs.data_ptr(), None) == 0
    zn, norms = sbf_radial_constants()
    x = d.double().numpy() / 5.0
    p = 6
    a, b, c = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    env = 1 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)
    denv = -1 / x ** 2 + a * (p - 1) * x ** (p - 2) + b * p * x ** (p - 1) + c * (p + 1) * x ** p
    for l in range(7):
        for n in range(6):
            zz = zn[l, n]
            ref = env * norms[l, n] * spherical_jn(l, zz * x)
            dref = (denv * norms[l, n] * spherical_jn(l, zz * x) + env * norms[l, n] * zz * spherical_jn(l, zz * x, derivative=True)) / 5.0
            got, dgot = rbs[:, l * 6 + n].double().numpy(), drbs[:, l * 6 + n].double().numpy()
            assert np.abs(got - ref).max() <= 2e-6 * np.abs(ref).max() + 1e-7, (l, n)
            far = d.numpy() >= 0.5
            assert np.abs(dgot - dref)[far].max() <= 5e-6 * np.abs(dref[far]).max() + 1e-7, (l, n)
