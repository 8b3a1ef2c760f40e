"""CPU tests of the Hessian / normal-mode host side (nabladft_b200.vibrations) and of the float64 oracle Hessian the GPU tests compare with."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import load_fixture, load_golden_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oc_oracle():
    from nabladft_b200.painn_oc import PaiNN
    from oracle.painn_oc import PaiNNOC

    kw = dict(hidden_channels=128, num_layers=3, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)
    net = load_golden_weights(PaiNN(direct_forces=False, use_pbc=False, **kw), torch.float64)
    ref = PaiNNOC(**kw).double()
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
    return ref


def test_oracle_double_backward_hessian_matches_finite_differences():
    ref = _oc_oracle()
    z, pos, batch = load_fixture([26])
    p = pos.clone().requires_grad_(True)
    _, f = ref(z, p, batch, create_graph=True)
    f = f.reshape(-1)
    cols = [0, 1, 2, 5, 13, 40, 86]  # H is symmetric: row i of -dF/dR is column i
    h = torch.stack([torch.autograd.grad(-f[i], p, retain_graph=True)[0].reshape(-1) for i in cols])
    step = 1e-5
    for k, i in enumerate(cols):
        dp = torch.zeros_like(pos).reshape(-1)
        dp[i] = step
        _, fp = ref(z, (pos.reshape(-1) + dp).reshape(pos.shape).clone(), batch)
        _, fm = ref(z, (pos.reshape(-1) - dp).reshape(pos.shape).clone(), batch)
        fd = -(fp - fm).reshape(-1).detach() / (2 * step)
        err = float((fd - h[k]).abs().max() / h[k].abs().max())
        assert err < 1e-5, (i, err)


def test_wavenumber_conversion_harmonic_diatomic():
    from nabladft_b200 import vibrations as vib

    k = 0.35  # Ha / A^2, spring along x between two atoms
    m1, m2 = 12.011, 15.999
    h = torch.zeros(6, 6, dtype=torch.float64)
    h[0, 0] = h[3, 3] = k
    h[0, 3] = h[3, 0] = -k
    nm = vib.normal_modes_from_hessian(h, torch.tensor([m1, m2], dtype=torch.float64))
    mu = m1 * m2 / (m1 + m2)
    omega = math.sqrt(k * 4.3597447222071e-18 / (1e-20 * mu * 1.66053906660e-27))  # rad / s
    expect = omega / (2 * math.pi * 2.99792458e10)
    assert abs(float(nm.wavenumbers[-1]) - expect) < 1e-9 * expect
    assert torch.allclose(nm.wavenumbers[:-1], torch.zeros(5, dtype=torch.float64), atol=1e-4)  # sqrt of rounding-level eigenvalues
    # h c nu~ in meV, and an imaginary mode comes out negative
    assert abs(float(nm.energies_meV[-1]) - expect * 0.1239841984) < 1e-6 * expect
    neg = vib.normal_modes_from_hessian(-h, torch.tensor([m1, m2], dtype=torch.float64))
    assert abs(float(neg.wavenumbers[0]) + expect) < 1e-9 * expect and int((neg.wavenumbers < -1).sum()) == 1
    # with projection the rigid modes vanish exactly, the stretch stays
    pr = vib.normal_modes_from_hessian(h, torch.tensor([m1, m2], dtype=torch.float64),
                                       torch.tensor([[0.0, 0, 0], [1.2, 0, 0]], dtype=torch.float64), project=True)
    assert abs(float(pr.wavenumbers[-1]) - expect) < 1e-9 * expect


def test_mass_table_covers_every_element():
    from nabladft_b200 import vibrations as vib
    from nabladft_b200.synth import ELEMENTS

    fx = np.load(os.path.join(ROOT, "tests", "golden", "fixture_molecules.npz"))
    need = set(ELEMENTS.tolist()) | {1} | set(fx["z"].tolist())
    assert need <= set(vib.ATOMIC_MASSES)
    assert vib.ATOMIC_MASSES == {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999, 9: 18.998403163, 16: 32.06, 17: 35.45, 35: 79.904}
    with pytest.raises(ValueError):
        vib.masses_of(torch.tensor([6, 14]))


@pytest.mark.parametrize("max_dir", [None, 1, 4, 7, 100])
def test_hessians_direction_layout_and_chunking(max_dir):
    from nabladft_b200 import vibrations as vib

    sizes = [1, 4, 2, 3]
    ptr = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    g = torch.Generator().manual_seed(0)
    blocks = []
    for n in sizes:
        a = torch.randn(3 * n, 3 * n, generator=g, dtype=torch.float64)
        blocks.append(a + a.t())
    big = torch.block_diag(*blocks)
    calls = []

    def hvp(v):
        calls.append(v.shape[0])
        assert v.shape[1:] == (ptr[-1], 3)
        v = v.double()
        return (big @ v.reshape(v.shape[0], -1).t()).t().reshape(v.shape)

    hs = vib.hessians_from_hvp(hvp, ptr, max_dir)
    assert sum(calls) == 3 * max(sizes)
    assert max(calls) <= (max_dir or 3 * max(sizes))
    for h, b in zip(hs, blocks):
        assert torch.allclose(h, b, atol=1e-12)
    assert hs.max_asymmetry < 1e-12
    # every direction displaces atom k of each molecule with more than k atoms
    v = vib.shared_directions(ptr, 0, 3 * max(sizes))
    assert float(v.sum()) == 3 * sum(sizes)
    assert v[3 * 3 + 1, ptr[1] + 3, 1] == 1 and v[3 * 3 + 1].sum() == 1


def test_hessians_symmetrise_and_report_asymmetry():
    from nabladft_b200 import vibrations as vib

    a = torch.arange(36, dtype=torch.float64).reshape(6, 6)
    hs = vib.hessians_from_hvp(lambda v: (a @ v.double().reshape(v.shape[0], -1).t()).t().reshape(v.shape), [0, 2])
    assert torch.equal(hs[0], 0.5 * (a + a.t()))
    assert hs.max_asymmetry == float((a - a.t()).abs().max())


def test_header_declares_hvp_entry_points():
    from nabladft_b200 import _lib

    with open(os.path.join(ROOT, "include", "nabla_b200.h")) as f:
        hdr = f.read()
    for name in ("nb200_painn_hvp_workspace_bytes", "nb200_painn_hvp"):
        assert f"{name}(" in hdr and name in _lib.SIGNATURES
