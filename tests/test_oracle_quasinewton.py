"""oracle/quasinewton.py: the scalar line search against calls recorded from the reference's own routines, and the BFGS driver's
properties (rank-2 update = ASE's product, strong Wolfe at CONVERGENCE, fixed atoms, steps cap, initial convergence, |p| rescale)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_quasinewton import TASKS, branch_scenarios, qn_scenarios, qn_setup, toy_forces  # noqa: E402

from oracle.quasinewton import CONVERGED, FAILED, MAX_STEPS, BatchQuasiNewton, LineSearch, _Mol, ase_update, rank2_update  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "quasinewton_ls_ref.npz"))
NAMES = [str(n) for n in GOLD["names"]]


@pytest.mark.parametrize("name", NAMES)
def test_line_search_matches_reference_bit_for_bit(name):
    g = {k: GOLD[f"{name}/{k}"] for k in ("pk", "params", "stp", "f", "g", "old_stp", "out", "task", "case", "no_update", "isave", "dsave")}
    maxstep, stpmax = g["params"]
    ls = LineSearch(maxstep=float(maxstep), stpmax=float(stpmax))
    for i in range(len(g["stp"])):
        ls.case = 0
        out = ls.step(float(g["stp"][i]), float(g["f"][i]), float(g["g"][i]), 0.23, 0.46, g["pk"], float(g["old_stp"][i]))
        assert TASKS.index(ls.task) == g["task"][i], (i, ls.task)
        assert float(out) == g["out"][i] or (np.isnan(out) and np.isnan(g["out"][i])), (i, out, g["out"][i])
        assert bool(ls.no_update) == bool(g["no_update"][i]) and ls.case == g["case"][i]
        assert np.array_equal(ls.isave, g["isave"][i])
        assert np.array_equal(ls.dsave, g["dsave"][i], equal_nan=True), i


def test_golden_covers_the_line_search():
    """The recorded calls reach every update case from a bracketed and an unbracketed interval, the maxstep cap, no_update, the
    XTOL / STP = maxstep / STP = minstep warnings and the START error."""
    seen_cases, tasks = set(), set()
    for name in NAMES:
        isave, case = GOLD[f"{name}/isave"], GOLD[f"{name}/case"]
        for i in range(1, len(case)):
            seen_cases.add((int(case[i]), int(isave[i - 1][0])))
        tasks |= set(int(t) for t in GOLD[f"{name}/task"])
    assert {(c, b) for c in (1, 2, 3, 4) for b in (0, 1)} <= seen_cases, sorted(seen_cases)
    assert {TASKS.index(t) for t in ("CONVERGENCE", "WARNING: XTOL TEST SATISFIED", "WARNING: STP = maxstep", "WARNING: STP = minstep",
                                     "ERROR: INITIAL G >= 0")} <= tasks
    assert any(GOLD[f"{n}/no_update"].any() for n in NAMES)
    assert GOLD["quadratic_capped/out"][0] < 1.0  # determine_step shortened the first step


def test_rank2_update_equals_ase_product_over_a_trajectory(monkeypatch):
    """Every update of a relaxation, applied by both forms to the same H: 1e-12 relative, and the rank-2 form keeps H symmetric."""
    import oracle.quasinewton as qn

    sc, zs, ps, pot = qn_setup("basic")
    seen = []

    def both(H, dr, dg, rhok):
        H2, Ha = rank2_update(H, dr, dg, rhok), ase_update(H, dr, dg, rhok)
        seen.append(np.abs(H2 - Ha).max() / np.abs(Ha).max())
        assert np.array_equal(H2, H2.T)
        return H2

    monkeypatch.setattr(qn, "rank2_update", both)
    o = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs])
    o.run(np.concatenate(ps), fmax=sc["fmax"], steps=sc["steps"])
    assert len(seen) > 20 and max(seen) < 1e-12, max(seen)
    for mol in o.mols:
        assert np.linalg.eigvalsh(mol.H).min() > 0


@pytest.mark.parametrize("name", list(qn_scenarios()))
def test_every_convergence_is_a_strong_wolfe_point(name):
    """Each line search that ends in CONVERGENCE accepted the last evaluated point, and that point satisfies the strong Wolfe
    conditions phi <= phi(0) + c1 stp phi'(0) and |phi'| <= c2 |phi'(0)|."""
    sc, zs, ps, pot = qn_setup(name)
    checked = []
    orig = _Mol.consume

    def spy(self, pos, e, f):
        ls, n, stp, p, r = self.ls, len(self.tasks), self.stp, self.p, getattr(self, "r", None)
        out = orig(self, pos, e, f)
        if ls is not None and self.tasks[n:n + 1] == ["CONVERGENCE"]:
            g = -np.asarray(f, np.float32).reshape(-1) / np.float32(self.alpha)
            phi, dphi = e / self.alpha, float(np.dot(g, p))
            ginit, finit = ls.dsave[0], ls.dsave[4]
            assert ginit < 0 and phi <= finit + stp * 0.23 * ginit and abs(dphi) <= 0.46 * -ginit
            assert np.array_equal(pos.reshape(-1), r + stp * p)
            checked.append(1)
        return out

    _Mol.consume = spy
    try:
        o = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs], fixed_atoms_mask=sc["fixed"])
        o.run(np.concatenate(ps), fmax=sc["fmax"], steps=sc["steps"])
    finally:
        _Mol.consume = orig
    assert len(checked) >= int(o.nsteps.sum()) // 2 and len(checked) > 0
    assert all(t in ("FG", "CONVERGENCE") for mol in o.mols for t in mol.tasks)


def test_fixed_atoms_never_move():
    sc, zs, ps, pot = qn_setup("fixed_atoms")
    o = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs], fixed_atoms_mask=sc["fixed"])
    pos0 = np.concatenate(ps)
    pos, st = o.run(pos0, fmax=sc["fmax"], steps=sc["steps"], record=True)
    assert (st == CONVERGED).all()
    for after in o.after:
        assert np.array_equal(after[0][sc["fixed"]], pos0[sc["fixed"]])
    assert not np.array_equal(pos, pos0)


def test_steps_cap_initial_convergence_and_rescale():
    sc, zs, ps, pot = qn_setup("steps_cap")
    o = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs])
    pos, st = o.run(np.concatenate(ps), fmax=sc["fmax"], steps=sc["steps"])
    assert (st == MAX_STEPS).all() and (o.nsteps == sc["steps"]).all()
    assert (o.function_calls == o.force_calls + o.nsteps).all()
    # converged at the start: no step, one call, nothing moves
    o = BatchQuasiNewton(toy_forces(pot), [len(z) for z in zs])
    pos0 = np.concatenate(ps)
    pos, st = o.run(pos0, fmax=100.0)
    assert (st == CONVERGED).all() and o.n_calls == 1 and (o.nsteps == 0).all() and np.array_equal(pos, pos0)
    # a shallow harmonic well: |p| <= sqrt(n 1e-10) is rescaled to that length, so the first trial moves every atom by more than |g|
    x0 = pos0[:5].copy()
    well = lambda x: (np.array([0.5 * 1e-6 * ((x - x0) ** 2).sum()]), (-1e-6 * (x - x0)).astype(np.float32))
    o = BatchQuasiNewton(well, [5])
    o.run(x0 + 1e-3, fmax=1e-12, steps=1)
    assert o.mols[0].rescaled >= 1
    p = o.mols[0].p
    assert abs(np.sqrt((p ** 2).sum()) - np.sqrt(5 * 1e-10)) < 1e-18


def test_branch_scenarios_reach_every_line_search_branch():
    """The runs that tests/test_gpu_quasinewton.py replays through the kernel launch by launch reach every `update` case from a
    bracketed and an unbracketed interval, CONVERGENCE, three of the four WARNING tasks, no_update, the |p| rescale and a failed START.
    (XTOL TEST SATISFIED needs an interval of 1e-14 relative width, finer than the float32 positions a model sees.)"""
    cases, tasks, no_update, rescaled, status = set(), set(), 0, 0, set()
    for b in branch_scenarios().values():
        o = BatchQuasiNewton(b["force_fn"], b["sizes"], **b["kw"])
        o.run(b["pos0"], fmax=b["fmax"], steps=b["steps"])
        for m in o.mols:
            cases |= set(m.cases)
            tasks |= set(m.tasks)
            no_update += m.no_update_accepts
            rescaled += m.rescaled
        status |= set(o.status.tolist())
    assert {(c, b) for c in (1, 2, 3, 4) for b in (0, 1)} <= cases, sorted(cases)
    assert {"CONVERGENCE", "WARNING: ROUNDING ERRORS PREVENT PROGRESS", "WARNING: STP = maxstep", "WARNING: STP = minstep",
            "ERROR: STP .GT. maxstep"} <= tasks, sorted(tasks)
    assert no_update > 0 and rescaled > 0 and {CONVERGED, MAX_STEPS, FAILED} <= status


def test_failed_line_search_stops_only_that_molecule():
    """stpmax < 1: the START of every line search (stp = 1) is an ERROR, as in ASE; the molecule converged at the start never starts one."""
    b = branch_scenarios()["stpmax_below_one"]
    o = BatchQuasiNewton(b["force_fn"], b["sizes"], **b["kw"])
    pos, st = o.run(b["pos0"], fmax=b["fmax"], steps=b["steps"])
    assert st.tolist() == [FAILED, CONVERGED, FAILED] and o.failed == [0, 2]
    assert o.n_calls == 1 and np.array_equal(pos, b["pos0"])
    assert [m.tasks for m in o.mols] == [["ERROR: STP .GT. maxstep"], [], ["ERROR: STP .GT. maxstep"]]
