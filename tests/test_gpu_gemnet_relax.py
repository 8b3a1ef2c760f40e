"""GemNet-OC relaxation on the device: the asynchronous forward (nb200_gemnet_oc_energy_forces_async) against the two-phase forward, its
error path, and `ASEBatchwiseLBFGS(PyGBatchwiseCalculator(GemNetOC))` against a host-driven loop and the float64 oracle.  The same checks on
the host-emulation build (guard zones included) are tests/test_gemnet_relax_emu.py."""
import math
import os
import sys
from ctypes import c_int64

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
from test_gemnet_emu import _models  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_ORDER = ("A2A", "MAIN", "AE", "Q", "TIN")


def _fixture(mols, jitter=0.0, seed=0):
    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    rng = np.random.default_rng(seed)
    zs = [fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols]
    ps = [fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]].astype(np.float64) + jitter * rng.normal(size=(len(z), 3)) for m, z in zip(mols, zs)]
    return zs, ps


def _golden():
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    b = g["batch"]
    return [g["z"][b == m] for m in range(int(b.max()) + 1)], [g["pos"][b == m].astype(np.float64) for m in range(int(b.max()) + 1)]


def _tensors(zs, ps):
    sizes = [len(z) for z in zs]
    z = torch.from_numpy(np.concatenate(zs).astype(np.int32)).to(DEV)
    pos = torch.from_numpy(np.concatenate(ps).astype(np.float32)).to(DEV).contiguous()
    mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(DEV)
    return z, pos, mol_ptr, sizes


@pytest.fixture(scope="module")
def model():
    net, ora = _models(True)
    return net.to(DEV).eval(), ora.double()


@pytest.fixture()
def runner(model):
    from emu_driver import poisoned

    from nabladft_b200.gemnet_oc import GemNetOCRunner

    r = poisoned(GemNetOCRunner, emulated=False)()  # every (re)used buffer is filled with `fill` bytes before the call
    r.set_weights(model[0], torch.device(DEV))
    return r


@pytest.mark.parametrize("which", ["golden", "fixture32"])
def test_async_forward_equals_two_phase_forward_and_dead_rows_are_dead(runner, which):
    z, pos, mol_ptr, sizes = _tensors(*(_golden() if which == "golden" else _fixture(range(32))))
    E0, F0 = runner.run(z, pos, mol_ptr, len(sizes), max(sizes))
    counts = dict(runner.last_counts)
    bounds = runner.count_bounds(sizes)
    assert all(counts[k] <= int(bounds[i]) for i, k in enumerate(C_ORDER)) and any(counts[k] < int(bounds[i]) for i, k in enumerate(C_ORDER))
    # a GEMM takes its row count from the host: the bound here, the count in the two-phase call.  Rows are independent in every GEMM kernel,
    # but nb_gemm_ps_wanted (gemm_ps.cu) hands problems of >= 2048 rows to the pre-split-weight kernel, whose K loop is chunked differently
    # from gemm_tc.cu's: where count and bound fall on different sides of 2048 the two calls may differ in the last bits
    same_kernels = all((counts[k] >= 2048) == (int(bounds[i]) >= 2048) for i, k in enumerate(C_ORDER[:4]))
    outs = []
    for fill in (255, 0):
        runner.fill = fill
        E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), max(sizes), bounds)
        outs.append((E.clone(), F.clone(), st.cpu().tolist()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])  # nothing stored past a real count reaches an output
    E, F, st = outs[0]
    assert st[:2] == [counts["MAIN"], 0] and st[4:] == [counts["A2A"], counts["AE"], counts["Q"], counts["TIN"]]
    assert 0 < st[2] <= max(sizes) - 1 and st[3] == 0
    if same_kernels:
        assert torch.equal(E, E0) and torch.equal(F, F0)
    else:
        assert float((E - E0).abs().max()) <= 1e-6 * float(E0.abs().max()) and float((F - F0).abs().max()) <= 1e-6 * float(F0.abs().max())


def test_bound_too_small_and_non_finite_positions_give_error_code_and_nan_outputs(runner):
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.gemnet_oc import GemNetOCEngine

    z, pos, mol_ptr, sizes = _tensors(*_fixture([3, 26]))
    runner.run(z, pos, mol_ptr, len(sizes), max(sizes))
    real = [runner.last_counts[k] for k in C_ORDER]
    for k in range(5):
        short = (c_int64 * 8)(*[r - (1 if i == k else 0) for i, r in enumerate(real)], 0, 0, 0)
        E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), max(sizes), short)
        st = st.cpu().tolist()
        assert st[1] == -4 and st[0] == real[1] and st[4:] == [real[0], real[2], real[3], real[4]], (k, st)
        assert bool(torch.isnan(E).all() and torch.isnan(F).all())
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        GemNetOCEngine.raise_on_status(st)
    bounds = runner.count_bounds(sizes)
    bad = pos.clone()
    bad[5, 2] = float("nan")
    E, F, st = runner.launch(z, bad, mol_ptr, len(sizes), max(sizes), bounds)
    assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), max(sizes), bounds)
    E0, F0 = runner.run(z, pos, mol_ptr, len(sizes), max(sizes))
    assert int(st[1]) == 0 and float((F - F0).abs().max()) <= 1e-6 * float(F0.abs().max())


def _relax(model, zs, ps, steps, check_every, fixed=None, record=False, calc_cls=None):
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator, SimpleAtoms

    calc = (calc_cls or PyGBatchwiseCalculator)(model[0], device=DEV, energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None, check_every=check_every, fixed_atoms_mask=fixed)
    opt.record_positions = record
    opt.run([SimpleAtoms(p, z) for p, z in zip(ps, zs)], fmax=1e-5, steps=steps)
    return opt, calc


def test_lbfgs_relaxation_of_32_molecules(model):
    from nabladft_b200.gemnet_oc import GemNetOCEngine
    from nabladft_b200.optimization import PyGBatchwiseCalculator

    zs, ps = _fixture(range(32), jitter=0.05, seed=1)
    steps = 50
    o1, c1 = _relax(model, zs, ps, steps, 1)
    o10, c10 = _relax(model, zs, ps, steps, 10)
    assert o1.nsteps == o10.nsteps == steps
    p1, p10 = np.concatenate([a.get_positions() for a in o1.atoms]), np.concatenate([a.get_positions() for a in o10.atoms])
    assert np.array_equal(p1, p10) and np.array_equal(c1.results["energy"], c10.results["energy"]) and np.array_equal(c1.results["forces"], c10.results["forces"])
    assert np.abs(p1 - np.concatenate(ps)).max() > 0.1
    # one wait at the start, one per check_every steps, one at the end
    assert o1.host_syncs == 1 + steps + 1 and o10.host_syncs == 1 + math.ceil(steps / 10) + 1

    class HostDriven(GemNetOCEngine):  # the two-phase forward, which waits for the edge counts, at every step
        def launch(self, z, pos, mol_ptr, n_mol, e_cap=None):
            energy, forces = self.runner.run(z, pos, mol_ptr, n_mol, self._batch[1])
            return energy, forces, torch.zeros(8, dtype=torch.int32, device=pos.device)

    class HostCalc(PyGBatchwiseCalculator):
        def engine(self):
            if getattr(self, "_e", None) is None:
                self._e = HostDriven(self.model, self.model._get_runner())
            return self._e

    oh, ch = _relax(model, zs, ps, steps, 10, calc_cls=HostCalc)
    ph = np.concatenate([a.get_positions() for a in oh.atoms])
    # every count of this batch and its bound are far above the 2048 rows where the GEMM dispatch changes: same kernels, same bits
    assert np.array_equal(ph, p10) and np.array_equal(ch.results["energy"], c10.results["energy"]) and np.array_equal(ch.results["forces"], c10.results["forces"])
    # energies and forces of the final geometry against the float64 oracle (four of the molecules: the oracle materialises every quadruplet)
    ora = model[1]
    off = np.concatenate([[0], np.cumsum([len(z) for z in zs])])
    for m in (0, 9, 20, 31):
        pm = torch.from_numpy(p1[off[m]:off[m + 1]].astype(np.float32)).double()
        with torch.no_grad():
            E, F = ora(torch.from_numpy(zs[m]).long(), pm, torch.zeros(len(zs[m]), dtype=torch.long))
        assert abs(float(E) - float(c1.results["energy"][m])) < 1e-5 * max(1.0, abs(float(E)))
        assert np.abs(F.numpy() - c1.results["forces"][off[m]:off[m + 1]]).max() < 1e-4 * max(1.0, float(F.abs().max()))


def test_fixed_atoms_do_not_move(model):
    zs, ps = _fixture([4, 11, 17], jitter=0.05, seed=2)
    fixed = [0, 3, len(zs[0]) + 2, len(zs[0]) + len(zs[1]) + 5]
    opt, calc = _relax(model, zs, ps, 10, 4, fixed=fixed)
    p = np.concatenate([a.get_positions() for a in opt.atoms])
    p0 = np.concatenate(ps)
    free = np.setdiff1d(np.arange(len(p0)), fixed)
    assert np.array_equal(p[fixed], p0[fixed]) and np.abs(p[free] - p0[free]).max() > 1e-3
    assert np.all(calc.results["forces"][fixed] == 0.0) and opt.host_syncs == 1 + 3 + 1


def test_device_relaxation_follows_the_float64_oracle_loop(model):
    from oracle.lbfgs import BatchLBFGS

    rng = np.random.default_rng(5)
    zs = [rng.choice([1, 6, 7, 8], size=k) for k in (6, 4)]
    ps = [rng.normal(size=(k, 3)) * 1.3 for k in (6, 4)]
    opt, _ = _relax(model, zs, ps, 5, 1, record=True)
    ora, sizes = model[1], [6, 4]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))
    z = torch.from_numpy(np.concatenate(zs)).long()

    def f_oracle(p):
        with torch.no_grad():
            E, F = ora(z, torch.from_numpy(p), batch)
        return E.numpy(), F.numpy().astype(np.float32)

    _, _, traj = BatchLBFGS(f_oracle, sizes).run(np.concatenate(ps), fmax=1e-5, steps=5)
    got = opt.positions_history + [np.concatenate([a.get_positions() for a in opt.atoms])]
    assert len(traj) == 6 and len(got) >= 6
    for k in range(6):
        assert np.abs(got[k] - traj[k]).max() < 1e-4, k


def test_molecular_dynamics_still_refuses_gemnet_oc(model):
    from nabladft_b200.md import BatchwiseMD
    from nabladft_b200.optimization import PyGBatchwiseCalculator, SimpleAtoms

    zs, ps = _fixture([0])
    calc = PyGBatchwiseCalculator(model[0], device=DEV, energy_unit="Hartree", position_unit="Ang")
    with pytest.raises(NotImplementedError, match="GemNet-OC"):
        BatchwiseMD(calc, [SimpleAtoms(ps[0], zs[0])])
