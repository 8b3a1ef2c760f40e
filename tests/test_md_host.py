"""Molecular dynamics without a GPU: the oracle's Philox stream, integrators and velocity initialisation, units and log format."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import md as omd  # noqa: E402


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123 known-answer vectors for philox4x32-10."""
    got = omd.philox4x32_10(np.array([ctr], dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert tuple(int(v) for v in got[0]) == want


def test_normals_are_standard():
    n = 200_000
    for stream, step in ((omd.STREAM_MAXWELL, 0), (omd.STREAM_LANGEVIN, 7)):
        if stream == omd.STREAM_MAXWELL:
            x = omd.maxwell_normals(12345, n, step).reshape(-1)
        else:
            xi, eta = omd.langevin_normals(12345, n, step)
            x = np.concatenate([xi.reshape(-1), eta.reshape(-1)])
        m = x.size
        # mean and variance of N(0, 1) samples: standard errors 1/sqrt(m) and sqrt(2/m); 5 sigma
        assert abs(x.mean()) < 5 / math.sqrt(m)
        assert abs(x.var() - 1.0) < 5 * math.sqrt(2.0 / m)
        assert np.isfinite(x).all()
    # distinct counters give distinct numbers: other step, other seed
    a = omd.langevin_normals(1, 64, 3)[0]
    assert not np.array_equal(a, omd.langevin_normals(1, 64, 4)[0])
    assert not np.array_equal(a, omd.langevin_normals(2, 64, 3)[0])


def test_velocity_verlet_matches_the_discrete_harmonic_recurrence():
    """One atom on a spring along x: velocity Verlet is the linear map M = [[a, dt/m], [c, a]], a = 1 - h^2/2, c = -k dt (1 - h^2/4),
    h = omega dt, det M = 1, so M^n = cos(n theta) I + sin(n theta) / sin(theta) (M - a I) with cos(theta) = a."""
    k, m, steps = 2.5, 12.011, 400

    def force(pos):
        return np.array([0.5 * k * pos[0, 0] ** 2]), -k * pos * np.array([[1.0, 0.0, 0.0]])

    md = omd.BatchMD(force, [1], [m], np.array([[0.3, 0.0, 0.0]]))
    md.init_md(time_step=1.0, temp_init=0)
    md.mom = np.array([[0.7, 0.0, 0.0]])
    md.run_md(steps)
    dt = 1.0 * omd.FS
    h2 = k / m * dt * dt
    a, b, c = 1 - h2 / 2, dt / m, -k * dt * (1 - h2 / 4)
    th = math.acos(a)
    n = np.arange(steps + 1)
    x = np.cos(n * th) * 0.3 + np.sin(n * th) / math.sin(th) * b * 0.7
    p = np.cos(n * th) * 0.7 + np.sin(n * th) / math.sin(th) * c * 0.3
    assert np.abs(np.stack(md.frames)[:, 0, 0] - x).max() < 1e-12
    assert abs(md.mom[0, 0] - p[-1]) < 1e-12
    log = np.stack(md.log)
    assert np.allclose(log[:, 0, 0], n * dt / (1000 * omd.FS), rtol=0, atol=1e-15)


def _springs(sizes, pos0, k=3.0):
    """Harmonic springs between every pair of each molecule at its starting distances: forces sum to zero per molecule."""
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    pairs = []
    for a, b in zip(ptr[:-1], ptr[1:]):
        for i in range(a, b):
            for j in range(i + 1, b):
                pairs.append((i, j, np.linalg.norm(pos0[i] - pos0[j])))

    def force(pos):
        f = np.zeros_like(pos)
        e = np.zeros(len(sizes))
        mol = np.repeat(np.arange(len(sizes)), sizes)
        for i, j, r0 in pairs:
            d = pos[i] - pos[j]
            r = np.linalg.norm(d)
            g = k * (r - r0) / r * d
            f[i] -= g
            f[j] += g
            e[mol[i]] += 0.5 * k * (r - r0) ** 2
        return e, f
    return force


def _batch(seed=3):
    rng = np.random.default_rng(seed)
    sizes = [5, 1, 2, 7]
    pos = np.concatenate([rng.normal(size=(n, 3)) * 1.2 for n in sizes])
    masses = rng.choice([1.008, 12.011, 14.007, 15.999], size=sum(sizes))
    return sizes, pos, masses


def test_langevin_keeps_total_momentum_zero():
    sizes, pos, masses = _batch()
    md = omd.BatchMD(_springs(sizes, pos), sizes, masses, pos, seed=11)
    md.init_md(time_step=0.5, temp_init=300, temp_bath=500)
    md.run_md(200)
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    for a, b in zip(ptr[:-1], ptr[1:]):
        assert np.abs(md.mom[a:b].sum(0)).max() < 1e-10
    assert np.abs(md.mom).max() > 1e-2  # the bath heats the molecules


def test_initialisation_has_no_drift_or_rotation_and_keeps_the_drawn_temperature():
    sizes, pos, masses = _batch(5)
    kT = 300 * omd.KB
    p = omd.init_momenta(masses, pos, sizes, kT, seed=9, noise_step=4)
    raw = omd.maxwell_normals(9, len(masses), 4) * np.sqrt(masses * kT)[:, None]
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    assert np.isfinite(p).all()
    for n, a, b in zip(sizes, ptr[:-1], ptr[1:]):
        m, q, r = masses[a:b], p[a:b], pos[a:b]
        if n == 1:
            assert np.array_equal(q, np.zeros((1, 3)))
            continue
        assert np.abs(q.sum(0)).max() < 1e-13
        x = r - (m[:, None] * r).sum(0) / m.sum()
        assert np.abs(np.cross(x, q).sum(0)).max() < 1e-12
        t_raw = omd.temperature(raw[a:b], m)
        assert abs(omd.temperature(q, m) - t_raw) < 1e-12 * t_raw


def test_units_and_mdlogger_format():
    from nabladft_b200 import md

    # ASE 3.22 defaults: CODATA 2014
    e, amu, kb_si = 1.6021766208e-19, 1.660539040e-27, 1.38064852e-23
    assert md.FS == omd.FS and md.KB == omd.KB
    assert abs(md.FS - 1e-15 * math.sqrt(e / amu) * 1e10) < 1e-15 * md.FS
    assert abs(md.KB - kb_si / e) < 1e-15 * md.KB
    assert md.LANGEVIN_FRICTION == 1.0 / (100.0 * md.FS)
    assert md.mdlogger_header() == "Time[ps]      Etot[eV]     Epot[eV]     Ekin[eV]    T[K]"
    assert md.mdlogger_line(0.0005, -1.5, 0.25, 300.04, 29) == "0.0005          -1.2500      -1.5000       0.2500   300.0"
    assert md.mdlogger_line(1.0, -1234.5, 2.0, 15.0, 150) == "1.0000        -1232.500    -1234.500        2.000    15.0"


def test_md_refuses_gemnet_oc_whose_forces_are_not_the_gradient_of_its_energy():
    """The refusal comes before the library is loaded, so a stand-in calculator on a CUDA device runs it without a GPU."""
    import torch
    import yaml

    from nabladft_b200.gemnet_oc import GemNetOC
    from nabladft_b200.md import BatchwiseMD

    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "model", "gemnet-oc-b200.yaml")))["net"]
    cfg.pop("_target_")

    class Calculator:
        device = torch.device("cuda")
        model = GemNetOC(**cfg)

    with pytest.raises(NotImplementedError, match="GemNet-OC"):
        BatchwiseMD(Calculator(), [])
