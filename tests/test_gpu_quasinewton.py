"""Device QuasiNewton loop (csrc/quasinewton.cu through nabladft_b200.optimization.BatchwiseQuasiNewton) against oracle/quasinewton.py."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_quasinewton import branch_scenarios, qn_scenarios, qn_setup, toy_forces  # noqa: E402

from oracle.quasinewton import BatchQuasiNewton  # noqa: E402

pytestmark = pytest.mark.gpu


class _ToyEngine:
    """Stands in for a model engine: same run / launch / e_cap / raise_on_status surface, forces from the analytic potential."""

    def __init__(self, pot):
        self.pot, self.e_cap = pot, 0

    def run(self, z, pos32, mol_ptr, n_mol, with_forces=True):
        e, f, st = self.launch(z, pos32, mol_ptr, n_mol)
        return e, f, st.cpu()

    def launch(self, z, pos32, mol_ptr, n_mol, with_forces=True, e_cap=None):
        e, f = self.pot.torch(pos32)
        return e.float(), f.contiguous(), torch.zeros(4, dtype=torch.int32, device=pos32.device)

    @staticmethod
    def raise_on_status(st):
        assert int(st[1]) == 0


def _toy_run(name, check_every):
    from nabladft_b200.optimization import BatchwiseCalculator, BatchwiseQuasiNewton, SimpleAtoms

    sc, zs, ps, pot = qn_setup(name)
    eng = _ToyEngine(pot)

    class ToyCalc(BatchwiseCalculator):
        def engine(self_inner):
            return eng

    # energy_unit eV: the toy energies and forces enter the optimiser unscaled, as the oracle sees them
    calc = ToyCalc(torch.nn.Identity(), device="cuda:0", energy_unit="eV", position_unit="Ang")
    opt = BatchwiseQuasiNewton(calc, fixed_atoms_mask=sc["fixed"], check_every=check_every)
    conv = opt.run([SimpleAtoms(p, z) for p, z in zip(ps, zs)], fmax=sc["fmax"], steps=sc["steps"])
    return opt, conv, calc


def _teacher_force(sizes, pos0, force_fn, kw, fmax, steps, fixed_atoms=None):
    """Every evaluation of the oracle's run, one kernel call each, through the C ABI: the positions, float32 energies and forces the
    oracle saw are uploaded, so each comparison isolates one launch of arithmetic: the next trial point, the status and the counters."""
    from nabladft_b200 import _lib

    lib = _lib.load()
    sizes = np.asarray(sizes)
    opt_kw = dict(maxstep=0.2, c1=0.23, c2=0.46, alpha=10.0, stpmax=50.0)
    opt_kw.update(kw)
    orc = BatchQuasiNewton(force_fn, sizes, fixed_atoms_mask=fixed_atoms, **opt_kw)
    orc.run(pos0, fmax=fmax, steps=steps, record=True)
    n_mol, n_atoms = len(sizes), int(sizes.sum())
    dev = "cuda:0"
    mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(dev)
    h = np.concatenate([[0], np.cumsum((3 * sizes) ** 2)]).astype(np.int64)
    h_off = torch.from_numpy(h[:-1].copy()).to(dev)
    state = torch.zeros(int(lib.nb200_qn_state_bytes(n_mol, n_atoms, int(h[-1]))), dtype=torch.uint8, device=dev)
    info = torch.zeros(n_mol, 4, dtype=torch.int32, device=dev)
    running = torch.zeros(1, dtype=torch.int32, device=dev)
    fixed = None
    if fixed_atoms is not None:
        fixed = torch.zeros(n_atoms, dtype=torch.uint8, device=dev)
        fixed[torch.tensor(fixed_atoms, device=dev)] = 1
    pos32 = torch.empty(n_atoms, 3, dtype=torch.float32, device=dev)
    mol_of_atom = np.repeat(np.arange(n_mol), sizes)
    worst = 0.0
    for (p_in, e, f), (p_out, status, nsteps, fcalls, fncalls) in zip(orc.evals, orc.after):
        pos = torch.from_numpy(p_in.copy()).to(dev)
        energy = torch.from_numpy(e.astype(np.float32)).to(dev)
        forces = torch.from_numpy(f.copy()).to(dev)
        rc = lib.nb200_qn_step(_lib.ptr(state), state.numel(), _lib.ptr(mol_ptr), _lib.ptr(h_off), n_mol, n_atoms, int(sizes.max()), int(h[-1]),
                               float(fmax), int(steps), opt_kw["maxstep"], opt_kw["c1"], opt_kw["c2"], opt_kw["alpha"], opt_kw["stpmax"], 1.0, 1.0,
                               _lib.ptr(fixed), _lib.ptr(energy), _lib.ptr(forces), _lib.ptr(pos), _lib.ptr(pos32), _lib.ptr(info), _lib.ptr(running),
                               _lib.current_stream())
        _lib.check(rc, "nb200_qn_step")
        got, mi = pos.cpu().numpy(), info.cpu().numpy()
        worst = max(worst, np.abs(got - p_out).max())
        moved = mi[mol_of_atom, 0] == 0
        assert np.array_equal(pos32.cpu().numpy()[moved], got.astype(np.float32)[moved])
        assert np.array_equal(mi[:, 0], status) and np.array_equal(mi[:, 1], nsteps) and np.array_equal(mi[:, 2], fcalls)
        assert np.array_equal(mi[:, 3], fncalls)
        assert int(running.item()) == int((status == 0).sum())
        if fixed is not None:
            assert np.array_equal(got[fixed_atoms], p_in[fixed_atoms])
    assert worst < 1e-8, worst
    return orc


@pytest.mark.parametrize("name", list(qn_scenarios()))
def test_qn_step_kernel_teacher_forced(name):
    sc, zs, ps, pot = qn_setup(name)
    _teacher_force([len(z) for z in zs], np.concatenate(ps), toy_forces(pot), {}, sc["fmax"], sc["steps"], sc["fixed"])


@pytest.mark.parametrize("name", list(branch_scenarios()))
def test_qn_step_kernel_teacher_forced_through_every_line_search_branch(name):
    """The oracle runs replayed here reach, between them, every `update` case bracketed and not, CONVERGENCE, the ROUNDING, STP =
    maxstep and STP = minstep warnings, no_update, the |p| rescale and a failed START (tests/test_oracle_quasinewton.py checks that
    coverage on the same runs), so each of those branches of the kernel is compared with the oracle launch by launch."""
    b = branch_scenarios()[name]
    orc = _teacher_force(b["sizes"], b["pos0"], b["force_fn"], b["kw"], b["fmax"], b["steps"])
    assert len(orc.evals) > 0


# Free-running loop.  The algorithm itself amplifies a 1-ulp perturbation of the float32 forces (forces * (1 + 6e-8 randn), four seeds, in
# oracle/quasinewton.py) to at most 1.1e-4 A ("basic"), 2.9e-4 ("mixed_sizes"), 8.9e-4 ("fixed_atoms") and 5.5e-6 ("steps_cap") in the
# final positions without changing any molecule's nsteps, force_calls or status; the bounds below are three times those.
_FREE_TOL = {"basic": 4e-4, "mixed_sizes": 1e-3, "fixed_atoms": 3e-3, "steps_cap": 2e-5}


@pytest.mark.parametrize("name", list(qn_scenarios()))
def test_device_qn_loop_follows_oracle(name):
    sc, zs, ps, pot = qn_setup(name)
    orc = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs], fixed_atoms_mask=sc["fixed"])
    pos_o, st_o = orc.run(np.concatenate(ps), fmax=sc["fmax"], steps=sc["steps"])
    opt, conv, calc = _toy_run(name, check_every=1)
    assert np.array_equal(opt.nsteps, orc.nsteps) and np.array_equal(opt.force_calls, orc.force_calls)
    assert np.array_equal(opt.function_calls, orc.function_calls) and np.array_equal(opt.status, st_o)
    assert conv == bool((st_o == 1).all())
    pos_d = np.concatenate([a.get_positions() for a in opt.atoms])
    assert np.abs(pos_d - pos_o).max() < _FREE_TOL[name], np.abs(pos_d - pos_o).max()
    if sc["fixed"] is not None:
        assert np.array_equal(pos_d[sc["fixed"]], np.concatenate(ps)[sc["fixed"]])
        assert not calc.results["forces"][sc["fixed"]].any()
    assert opt.host_syncs == opt.launches + 1  # check_every = 1: one look per launch, plus the first evaluation's and the final read
    assert opt.launches_used == orc.n_calls and opt.launches == opt.launches_used + 1


@pytest.mark.parametrize("name", ["mixed_sizes", "fixed_atoms"])
def test_check_every_does_not_change_the_result(name):
    a, conv_a, _ = _toy_run(name, check_every=1)
    b, conv_b, _ = _toy_run(name, check_every=7)
    assert conv_a == conv_b
    for k in ("nsteps", "force_calls", "function_calls", "status"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    pa = np.concatenate([x.get_positions() for x in a.atoms]); pb = np.concatenate([x.get_positions() for x in b.atoms])
    assert np.array_equal(pa, pb)  # launches after a molecule stopped move nothing, bit for bit
    assert b.host_syncs < a.host_syncs


class _NumpyEngine(_ToyEngine):
    """A toy engine over a numpy force field (a host round trip per launch: fine for a test)."""

    def __init__(self, force_fn):
        self.force_fn, self.e_cap = force_fn, 0

    def launch(self, z, pos32, mol_ptr, n_mol, with_forces=True, e_cap=None):
        e, f = self.force_fn(pos32.cpu().numpy().astype(np.float64))
        dev = pos32.device
        return (torch.from_numpy(np.asarray(e, np.float32)).to(dev), torch.from_numpy(np.ascontiguousarray(f, np.float32)).to(dev),
                torch.zeros(4, dtype=torch.int32, device=dev))


def test_failed_line_search_raises_for_exactly_the_failed_molecules():
    from nabladft_b200.optimization import BatchwiseCalculator, BatchwiseQuasiNewton, SimpleAtoms

    b = branch_scenarios()["stpmax_below_one"]
    orc = BatchQuasiNewton(b["force_fn"], b["sizes"], **b["kw"])
    pos_o, st_o = orc.run(b["pos0"], fmax=b["fmax"], steps=b["steps"])
    assert orc.failed == [0, 2] and st_o[1] == 1
    eng = _NumpyEngine(b["force_fn"])

    class Calc(BatchwiseCalculator):
        def engine(self_inner):
            return eng

    calc = Calc(torch.nn.Identity(), device="cuda:0", energy_unit="eV", position_unit="Ang")
    opt = BatchwiseQuasiNewton(calc, check_every=4, **b["kw"])
    off = np.concatenate([[0], np.cumsum(b["sizes"])])
    atoms = [SimpleAtoms(b["pos0"][off[i]:off[i + 1]], np.full(b["sizes"][i], 6)) for i in range(len(b["sizes"]))]
    with pytest.raises(RuntimeError, match=r"LineSearch failed! \(molecules \[0, 2\]\)"):
        opt.run(atoms, fmax=b["fmax"], steps=b["steps"])
    assert np.array_equal(opt.status, st_o) and np.array_equal(opt.nsteps, orc.nsteps)
    assert np.array_equal(np.concatenate([a.get_positions() for a in opt.atoms]), pos_o)


def test_qn_abi_rejects_bad_arguments():
    from nabladft_b200 import _lib

    lib = _lib.load()
    dev = "cuda:0"
    sizes = np.array([3, 4])
    n_atoms, hess = 7, int(((3 * sizes) ** 2).sum())
    need = int(lib.nb200_qn_state_bytes(2, n_atoms, hess))
    assert need > hess * 8 and lib.nb200_qn_state_bytes(-1, n_atoms, hess) == -1 and lib.nb200_qn_state_bytes(2, n_atoms, -1) == -1
    t = lambda n, dt: torch.zeros(n, dtype=dt, device=dev)
    state, mol_ptr, h_off = t(need, torch.uint8), torch.tensor([0, 3, 7], dtype=torch.int32, device=dev), torch.tensor([0, 81], dtype=torch.int64, device=dev)
    e, f, pos, pos32, info, run = t(2, torch.float32), t(21, torch.float32), t(21, torch.float64), t(21, torch.float32), t(8, torch.int32), t(1, torch.int32)
    P = _lib.ptr

    def call(state_ptr=P(state), nbytes=need, energy=P(e), forces=P(f), mp=P(mol_ptr), ho=P(h_off), alpha=10.0):
        return lib.nb200_qn_step(state_ptr, nbytes, mp, ho, 2, n_atoms, 4, hess, 0.05, 10, 0.2, 0.23, 0.46, alpha, 50.0, 1.0, 1.0, None, energy,
                                 forces, P(pos), P(pos32), P(info), P(run), _lib.current_stream())

    assert call(state_ptr=None) == -1
    assert call(nbytes=need - 1) == -1
    assert call(energy=None) == -1 and call(forces=None) == -1 and call(mp=None) == -1 and call(ho=None) == -1
    assert call(alpha=0.0) == -1
    torch.cuda.synchronize()
    assert not info.any()  # nothing was launched


def _real_model_check(net, calc_cls, zs, ps, ref_forces, steps, tol):
    from nabladft_b200.optimization import BatchwiseQuasiNewton, SimpleAtoms, convert_units

    sizes = [len(z) for z in zs]
    calc = calc_cls(net, device="cuda:0", energy_unit="Hartree", position_unit="Ang")
    e_scale = calc.energy_conversion * convert_units("Hartree", "eV")
    f_scale = np.float32(e_scale / calc.position_conversion)

    def oracle_forces(pos):  # what the reference's PYGCalculator hands ASE: float32 model outputs times the unit factors
        e, f = ref_forces(pos)
        return np.asarray(e, np.float32).astype(np.float64) * e_scale, np.asarray(f, np.float32) * f_scale

    orc = BatchQuasiNewton(oracle_forces, sizes)
    pos_o, st_o = orc.run(np.concatenate(ps), fmax=1e-4, steps=steps)
    opt = BatchwiseQuasiNewton(calc, check_every=3)
    conv = opt.run([SimpleAtoms(p, z) for p, z in zip(ps, zs)], fmax=1e-4, steps=steps)
    pos_d = np.concatenate([a.get_positions() for a in opt.atoms])
    assert np.array_equal(opt.nsteps, orc.nsteps) and np.array_equal(opt.status, st_o) and conv == bool((st_o == 1).all())
    assert np.array_equal(opt.force_calls, orc.force_calls)
    assert np.abs(pos_d - pos_o).max() < tol, np.abs(pos_d - pos_o).max()


def test_painn_oc_relaxation_matches_oracle_loop():
    """PaiNN-OC (capacity-sized engine) through the public API against the oracle loop driven by the oracle model."""
    from helpers import load_fixture, load_golden_weights
    from nabladft_b200.optimization import PyGBatchwiseCalculator
    from nabladft_b200.painn_oc import PaiNN
    from oracle.painn_oc import PaiNNOC

    mols = [0, 5]
    zcat, pcat, batch = load_fixture(mols, dtype=torch.float64)
    off = np.concatenate([[0], np.cumsum(torch.bincount(batch).tolist())])
    zs = [zcat[off[i]:off[i + 1]].numpy() for i in range(len(mols))]
    ps = [pcat[off[i]:off[i + 1]].numpy() for i in range(len(mols))]
    kw = dict(hidden_channels=128, num_layers=3, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100)
    net = load_golden_weights(PaiNN(direct_forces=False, use_pbc=False, **kw), torch.float32)
    ref = PaiNNOC(**kw).float()
    ref.load_state_dict(net.state_dict(), strict=True)

    def ref_forces(pos):
        e, f = ref(zcat, torch.from_numpy(np.asarray(pos, dtype=np.float32)), batch)
        return e.detach().numpy(), f.detach().numpy()

    # forces agree to ~1e-6 Ha/A per call (test_gpu_painn); a few line-searched BFGS steps amplify that mildly
    _real_model_check(net.cuda().eval(), PyGBatchwiseCalculator, zs, ps, ref_forces, steps=4, tol=2e-4)


def test_dimenetplusplus_relaxation_matches_oracle_loop():
    """DimeNet++ (bounds-sized engine) through the public API against the oracle loop driven by the float64 oracle model."""
    from make_golden_dimenet import SCALER, load_test_weights
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from nabladft_b200.optimization import PyGBatchwiseCalculator
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    kw = dict(node_latent_dim=50, scaler=SCALER, dimenet_hidden_channels=256, dimenet_num_blocks=6, do_postprocessing=True)
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(**kw).double().eval())
    net = DimeNetPlusPlusPotential(**kw).eval()
    net.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    rng = np.random.default_rng(5)
    sizes = [6, 4]
    zs = [rng.choice([1, 6, 7, 8], size=k) for k in sizes]
    ps = [rng.normal(size=(k, 3)) * 1.3 for k in sizes]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))
    z = torch.from_numpy(np.concatenate(zs)).long()

    def ref_forces(pos):
        E, F, _ = ora(z, torch.from_numpy(np.asarray(pos, dtype=np.float32).astype(np.float64)), batch)
        return E.detach().numpy(), F.detach().numpy()

    _real_model_check(net.to("cuda:0"), PyGBatchwiseCalculator, zs, ps, ref_forces, steps=4, tol=1e-4)
