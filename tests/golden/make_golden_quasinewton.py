"""Golden calls of the reference's scalar line search (`/root/reference/nablaDFT/optimization/line_search.py`, unmodified, imported
where it lies: it needs only numpy), one configuration at a time.

`LineSearch.step` / `update` / `determine_step` are driven the way ASE 3.22's `LineSearch._line_search` drives them for one
configuration: START at stp = 1 with (phi(0), phi'(0)), then while the task is FG evaluate phi and phi' at the returned step, pass
the evaluated step as `old_stp`, and stop after the evaluation that follows a call which set `no_update`.  (The reference's own
batched `_line_search` crashes: tools/probe_reference_line_search.py.)  Sequences come from
    * analytic 1-D functions phi(t) along a fixed direction pk, chosen to reach all four `update` cases bracketed and not, the
      `determine_step` maxstep cap, the stpmax / no_update condition, the XTOL, STP = maxstep and STP = minstep warnings and the
      START error for phi'(0) >= 0 (no sequence found here reaches ROUNDING ERRORS PREVENT PROGRESS without the XTOL test, which
      the routine checks after it and which then wins);
    * ToyPotential molecules (tests/golden/toy_potential.py) along steepest-descent directions, a few accepted steps each.
After every call: the inputs (stp, f, g, old_stp, scenario) and the outputs (task, returned stp, no_update, isave, dsave, case).

    python tests/golden/make_golden_quasinewton.py      # writes tests/golden/quasinewton_ls_ref.npz
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = "/root/reference/nablaDFT/optimization/line_search.py"
from toy_potential import ToyPotential  # noqa: E402

TASKS = ["START", "FG", "CONVERGENCE", "WARNING: ROUNDING ERRORS PREVENT PROGRESS", "WARNING: XTOL TEST SATISFIED", "WARNING: STP = maxstep",
         "WARNING: STP = minstep", "ERROR: INITIAL G >= 0"]
C1, C2, XTOL = 0.23, 0.46, 1e-14


def analytic_scenarios():
    """name -> (phi(t) -> (f, g), pk [n,3], maxstep, stpmax).  phi' is the derivative along pk (what g.p is in the optimiser)."""
    rng = np.random.default_rng(7)
    small = 0.01 * rng.standard_normal((4, 3))   # |pk| per atom ~0.02: the maxstep cap never binds below stp ~ 10
    big = 0.5 * rng.standard_normal((3, 3))      # the cap binds at stp = 1
    quad = lambda a, t0: (lambda t: (0.5 * a * (t - t0) ** 2, a * (t - t0)))
    return {
        "quadratic_short": (quad(1.0, 0.3), small, 0.2, 50.0),        # overshoot: case 1, bracketed
        "quadratic_long": (quad(1.0, 6.0), small, 0.2, 50.0),         # extrapolation: case 3 unbracketed, then case 2
        "quadratic_capped": (quad(1.0, 6.0), big, 0.2, 50.0),         # determine_step caps every step at maxstep
        "quartic": (lambda t: (t ** 4 - 3.0 * t ** 2 - 1.2 * t, 4 * t ** 3 - 6.0 * t - 1.2), small, 0.2, 50.0),
        "linear_to_stpmax": (lambda t: (-t, -1.0), small, 0.2, 50.0),  # case 4 unbracketed -> stpmax -> STP = maxstep
        "linear_low_stpmax": (lambda t: (-t, -1.0), small, 0.2, 3.0),
        "linear_inconsistent": (lambda t: (-0.1 * t, -1.0), small, 0.2, 50.0),  # f falls slower than g says: stpmax with no_update
        "concave_bump": (lambda t: (-np.sin(1.3 * t) + 0.05 * t ** 3, -1.3 * np.cos(1.3 * t) + 0.15 * t ** 2), small, 0.2, 50.0),
        "steep_well": (lambda t: (np.exp(4.0 * (t - 2.5)) - 4.0 * t, 4.0 * np.exp(4.0 * (t - 2.5)) - 4.0), small, 0.2, 50.0),
        "inconsistent_up": (lambda t: (1.0 + t, -1.0), small, 0.2, 50.0),  # f rises, g says it falls: bisects to stpmin
        "flat_noise": (lambda t: (1e-17 * np.sin(1e3 * t), -1e-9 + 1e-9 * np.cos(7.0 * t)), small, 0.2, 50.0),
        "kink": (lambda t: (abs(t - 0.7) - 0.7, -1.0 if t < 0.7 else 1.0), small, 0.2, 50.0),  # derivative jumps: cases 1, 2, 4 bracketed, XTOL warning
        "uphill_start": (quad(1.0, -1.0), small, 0.2, 50.0),          # phi'(0) > 0: ERROR at START
        "zero_slope_start": (quad(1.0, 0.0), small, 0.2, 50.0),       # phi'(0) = 0: ERROR at START
    }


def drive(LineSearch, phi, pk, maxstep, stpmax, max_calls=60):
    """One line search on phi along pk with the reference's routines; returns the list of recorded calls."""
    ls = LineSearch(xtol=XTOL)
    ls.tasks = ["START"]
    ls.isave = np.zeros((1, 2), np.intc)
    ls.dsave = np.zeros((1, 13), float)
    ls.stpmin, ls.stpmax, ls.xtrapl, ls.xtrapu, ls.maxstep = 1e-8, stpmax, 1.1, 4.0, maxstep
    ls.no_update = False
    pk = np.asarray(pk, dtype=np.float64).ravel()
    stp, old_stp = 1.0, 0.0
    f, g = phi(0.0)
    rows = []
    for _ in range(max_calls):
        ls.case = 0
        out = ls.step(stp, f, g, C1, C2, pk, old_stp, 0, XTOL, ls.isave, ls.dsave)
        rows.append(dict(stp=stp, f=f, g=g, old_stp=old_stp, task=TASKS.index(ls.tasks[0]), out=float(out), no_update=bool(ls.no_update),
                         isave=ls.isave[0].copy(), dsave=ls.dsave[0].copy(), case=ls.case))
        if ls.tasks[0][:2] != "FG":
            break
        stp = old_stp = float(out)
        f, g = phi(stp)
        f, g = float(f), float(g)
        if ls.no_update:
            break
    return rows


def toy_sequences(LineSearch, n_steps=4, alpha=10.0):
    """Line searches of a steepest-descent loop on ToyPotential molecules: phi(t) = E(x + t p) / alpha, phi'(t) = (-F / alpha) . p."""
    fix = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    rng = np.random.default_rng(11)
    out = {}
    for m in (0, 3, 9):
        a, b = int(fix["ptr"][m]), int(fix["ptr"][m + 1])
        pos = fix["pos"][a:b].astype(np.float64) + 0.1 * rng.standard_normal((b - a, 3))
        pot = ToyPotential([fix["z"][a:b]], [fix["pos"][a:b]])
        for k in range(n_steps):
            e, f = pot.numpy(pos)
            gvec = -f.reshape(-1) / np.float32(alpha)
            p = -gvec.astype(np.float64)
            x0 = pos.reshape(-1).copy()

            def phi(t, x0=x0, p=p):
                ee, ff = pot.numpy((x0 + t * p).reshape(-1, 3))
                return float(ee[0]) / alpha, float(np.dot(-ff.reshape(-1) / np.float32(alpha), p))

            rows = drive(LineSearch, phi, p, 0.2, 50.0)
            out[f"toy_mol{m}_step{k}"] = rows
            pos = (x0 + rows[-1]["stp"] * p).reshape(-1, 3) if rows[-1]["task"] in (1, 2, 3, 4, 5, 6) else pos
            out[f"toy_mol{m}_step{k}/pk"] = p
    return out


def main():
    spec = importlib.util.spec_from_file_location("reference_line_search", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    LineSearch = mod.LineSearch
    seqs, pks, params = {}, {}, {}
    for name, (phi, pk, maxstep, stpmax) in analytic_scenarios().items():
        seqs[name] = drive(LineSearch, phi, pk, maxstep, stpmax)
        pks[name], params[name] = np.asarray(pk, dtype=np.float64).ravel(), (maxstep, stpmax)
    toy = toy_sequences(LineSearch)
    for k, v in toy.items():
        if k.endswith("/pk"):
            pks[k[:-3]], params[k[:-3]] = v, (0.2, 50.0)
        else:
            seqs[k] = v
    out = {"names": np.array(list(seqs))}
    for name, rows in seqs.items():
        out[f"{name}/pk"] = pks[name]
        out[f"{name}/params"] = np.array(params[name])
        for key in ("stp", "f", "g", "old_stp", "out"):
            out[f"{name}/{key}"] = np.array([r[key] for r in rows], dtype=np.float64)
        for key in ("task", "case"):
            out[f"{name}/{key}"] = np.array([r[key] for r in rows], dtype=np.int32)
        out[f"{name}/no_update"] = np.array([r["no_update"] for r in rows])
        out[f"{name}/isave"] = np.stack([r["isave"] for r in rows]).astype(np.int32)
        out[f"{name}/dsave"] = np.stack([r["dsave"] for r in rows])
        print(f"{name:24s} calls {len(rows):3d} tasks {[TASKS[r['task']][:12] for r in rows][-3:]} cases {sorted({(r['case'], int(r['isave'][0])) for r in rows})}")
    np.savez_compressed(os.path.join(HERE, "quasinewton_ls_ref.npz"), **out)


def qn_scenarios():
    """ToyPotential relaxations for the optimiser tests: name -> dict(mols=[fixture indices], fmax, steps, fixed, jitter, seed).  Chosen
    off line-search ties: perturbing the float32 forces by 1 ulp (x (1 + 6e-8 randn), four seeds) changes no molecule's nsteps,
    force_calls or status in the oracle, and moves the final positions by at most the amounts in tests/test_gpu_quasinewton.py."""
    return {
        "basic": dict(mols=[0, 3, 7], fmax=2e-3, steps=80, fixed=None, jitter=0.1, seed=200),
        "mixed_sizes": dict(mols=[1, 12, 5, 13, 9], fmax=5e-3, steps=80, fixed=None, jitter=0.12, seed=201),
        "fixed_atoms": dict(mols=[12, 13], fmax=2e-3, steps=80, fixed=[0, 5, 40, 47], jitter=0.05, seed=202),
        "steps_cap": dict(mols=[4, 6], fmax=1e-6, steps=5, fixed=None, jitter=0.1, seed=203),
    }


def qn_setup(name):
    """(scenario, atomic numbers, start positions, ToyPotential) of one qn_scenarios() entry."""
    from make_golden_lbfgs import start_geometry

    sc = qn_scenarios()[name]
    fix = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    zs, ps = start_geometry(fix, sc["mols"], sc["jitter"], seed=sc["seed"])
    pot = ToyPotential(zs, [fix["pos"][int(fix["ptr"][m]):int(fix["ptr"][m + 1])] for m in sc["mols"]])
    return sc, zs, ps, pot


def toy_forces(pot):
    """force_fn for oracle.quasinewton: the energies rounded to float32, as an engine hands them over."""
    def ff(pos):
        e, f = pot.numpy(pos)
        return e.astype(np.float32).astype(np.float64), f
    return ff



def _line_fields():
    """One-atom molecules, each with a 1-D field along its own unit direction d through x0: E = psi_E(s), F = -psi_F'(s) d with
    s = (x - x0).d.  The first BFGS direction is along d (H = I), so each molecule's first line search is the 1-D problem
    (psi_E, psi_F') -- consistent or not -- seen along it."""
    rng = np.random.default_rng(3)
    specs = [
        (lambda s: abs(s - 0.07) - 0.07, lambda s: -1.0 if s < 0.07 else 1.0),    # kink: bracketed cases 1, 2, 4, rounding warning
        (lambda s: 1.0 + s, lambda s: -1.0),                                       # f rises while g says it falls: STP = minstep
        (lambda s: -s, lambda s: -1.0),                                            # constant push: case 4 unbracketed, STP = maxstep
        (lambda s: -0.1 * s, lambda s: -1.0),                                      # f falls slower than g says: no_update
        (lambda s: 0.5e-2 * (s - 5e-3) ** 2, lambda s: 1e-2 * (s - 5e-3)),         # shallow well: |p| rescaled
        (lambda s: s ** 4 - 0.3 * s ** 2 - 0.1 * s, lambda s: 4 * s ** 3 - 0.6 * s - 0.1),
    ]
    d = rng.normal(size=(len(specs), 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x0 = rng.normal(size=(len(specs), 3))

    def ff(pos):
        x = np.asarray(pos, np.float32).astype(np.float64)
        e, f = np.zeros(len(specs)), np.zeros_like(x)
        for m, (pe, pf) in enumerate(specs):
            s = float((x[m] - x0[m]) @ d[m])
            e[m], f[m] = pe(s), -pf(s) * d[m]
        return e.astype(np.float32).astype(np.float64), f.astype(np.float32)
    return [1] * len(specs), x0, ff


def _curl_field(n=6, k=1e-3, w=10.0, seed=0):
    """A weak harmonic well plus a strong rotation about z through the centroid: forces that are not -grad E."""
    x0 = np.random.default_rng(seed).normal(size=(n, 3)) * 1.5

    def ff(pos):
        x = np.asarray(pos, np.float32).astype(np.float64)
        d = x - x.mean(0)
        f = -k * d + w * np.stack([-d[:, 1], d[:, 0], np.zeros(n)], 1)
        return np.array([np.float32(0.5 * k * (d ** 2).sum())], np.float64), f.astype(np.float32)
    return [n], x0, ff


def _failing_batch():
    """Three ToyPotential molecules, the middle one with zero forces (converged at the start).  With stpmax < 1 every START of a line
    search (at stp = 1) is 'ERROR: STP .GT. maxstep', so exactly the molecules that take a step fail: 0 and 2."""
    sc, zs, ps, pot = qn_setup("basic")
    sizes = [len(z) for z in zs]
    ptr = np.concatenate([[0], np.cumsum(sizes)])

    def ff(pos):
        e, f = toy_forces(pot)(pos)
        f = f.copy()
        f[ptr[1]:ptr[2]] = 0.0
        return e, f
    return sizes, np.concatenate(ps), ff


def branch_scenarios():
    """Relaxations whose line searches reach the branches the smooth ToyPotential runs of qn_scenarios() do not: every `update` case
    from a bracketed and an unbracketed interval, the CONVERGENCE and WARNING tasks, no_update, the |p| rescale and a failed line
    search.  name -> dict(sizes, pos0, force_fn, kw = BatchwiseQuasiNewton arguments, fmax, steps)."""
    from make_golden_lbfgs import start_geometry

    fix = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    zs, ps = start_geometry(fix, [0, 3, 7], 0.3, seed=210)
    pot = ToyPotential(zs, [fix["pos"][int(fix["ptr"][m]):int(fix["ptr"][m + 1])] for m in [0, 3, 7]])
    out = {"toy_wide_jitter": dict(sizes=[len(z) for z in zs], pos0=np.concatenate(ps), force_fn=toy_forces(pot), kw={}, fmax=2e-3, steps=40)}
    sizes, x0, ff = _curl_field()
    out["curl"] = dict(sizes=sizes, pos0=x0, force_fn=ff, kw={}, fmax=1e-4, steps=10)
    sizes, x0, ff = _line_fields()
    out["line_fields"] = dict(sizes=sizes, pos0=x0, force_fn=ff, kw=dict(stpmax=3.0), fmax=1e-7, steps=2)
    sizes, x0, ff = _failing_batch()
    out["stpmax_below_one"] = dict(sizes=sizes, pos0=x0, force_fn=ff, kw=dict(stpmax=0.5), fmax=2e-3, steps=10)
    return out


if __name__ == "__main__":
    main()
