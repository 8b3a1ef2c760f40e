"""CPU restatement of the reference's QuasiNewton relaxation (`PYGAseInterface.optimize`, nablaDFT/optimization/pyg_ase_interface.py:296-315:
ASE's `QuasiNewton` = `BFGSLineSearch` + `LineSearch`) for a batch of independent molecules.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Every molecule runs exactly as ASE 3.22 runs it alone; the batch only shares the force calls.  `force_fn` evaluates every molecule at
its own current point once per call (a molecule that has stopped is evaluated where it stopped), so the number of calls equals the
number of engine launches of the device loop (csrc/quasinewton.cu, nabladft_b200.optimization.BatchwiseQuasiNewton).

Per molecule (`_Mol.consume` is one device launch):
    Optimizer.irun        forces at the start; while not converged and nsteps < steps: step(); nsteps += 1
    converged             (F**2).sum(1).max() < fmax**2, evaluated in float32 (numpy >= 2 casts the Python float to float32)
    BFGSLineSearch.step   g = -F / alpha; update(r, g, r0, g0, p0); e = E / alpha; p = -H g; |p| rescale; fresh LineSearch at stp = 1
    BFGSLineSearch.update first call H = I; skipped unless (alpha_k or 0) > 0 and |g.p0| - |g0.p0| < 0, and when the previous line
                          search set no_update; rhok = 1 / (dg.dr), 1000 when that is inf; then the rank-2 form (`rank2_update`)
    LineSearch._line_search   step -> FG: evaluate at r + stp p, phi = E / alpha, derphi = g.p, old_stp = stp, stop after that
                          evaluation when no_update is set; CONVERGENCE / WARNING*: accept; ERROR*: RuntimeError('LineSearch failed!')
    accepted point        always the last point evaluated: alpha_k = the last stp

dtypes (numpy):
    float32  F (forces, fixed atoms zeroed), g = -F / np.float32(alpha), dg = g - g0, the fmax test
    float64  positions r, r0, p, H, E, e0, phi, every dot product (float32 operands are widened), all line-search scalars

Judgements where the brief ("ASE 3.22's driver from memory") meets the reference's per-configuration routines
(nablaDFT/optimization/line_search.py), which win:
    * `LineSearch.step` / `update` / `determine_step` here are the reference's routines line for line (`LineSearch` below): the
      per-configuration arguments `pk` and `old_stp` are explicit, `isave` / `dsave` are per-configuration rows, and `no_update` is the
      attribute `step` sets (`self.no_update = True`, line_search.py:303).
    * `old_stp` passed to `step` is the last EVALUATED step (ASE: `self.old_stp = alpha1` after each evaluation), 0 at START.  The
      reference's batched `_line_search` passes the previous input step instead (line_search.py:105), but that driver crashes
      (tools/probe_reference_line_search.py) and is not used.
    * A WARNING task ends the line search without failing the molecule: ASE's `_line_search` tests `task[1:4] == 'WARN'`, which never
      matches.  The step is accepted at the last evaluated point.
    * The fmax test is float32 against float32(fmax**2), as numpy 2 evaluates `(forces ** 2).sum(axis=1).max() < self.fmax ** 2`.

The BFGS update is the O(n^2) rank-2 form of ASE's `A1 @ H @ A2 + rhok * dr dr^T` (`ase_update` is ASE's form, kept for the tests):
    u = H dg,  H' = H - rhok (dr u^T + u dr^T) + (rhok^2 dg.u + rhok) dr dr^T
which equals ASE's product for symmetric H up to rounding and keeps H exactly symmetric.

Pin status: the scalar line search (`LineSearch`) is PINNED to the reference's line_search.py: tests/test_oracle_quasinewton.py replays
every call recorded from the reference's own routines (tests/golden/make_golden_quasinewton.py -> tests/golden/quasinewton_ls_ref.npz)
and compares task, stp, no_update, isave and dsave bit for bit.  The BFGS driver (`_Mol`) is restated from ASE 3.22
(ase/optimize/bfgslinesearch.py, ase/optimize/optimize.py) and is UNPINNED: ASE cannot be installed here.
"""
import numpy as np

RUNNING, CONVERGED, MAX_STEPS, FAILED = 0, 1, 2, 3


class LineSearch:
    """The reference's LineSearch.step / update / determine_step (line_search.py:126-498) for ONE configuration."""

    def __init__(self, maxstep=0.2, stpmax=50.0, stpmin=1e-8, xtrapl=1.1, xtrapu=4.0, xtol=1e-14):
        self.maxstep, self.stpmax, self.stpmin, self.xtrapl, self.xtrapu, self.xtol = maxstep, stpmax, stpmin, xtrapl, xtrapu, xtol
        self.task = "START"
        self.isave = np.zeros(2, np.intc)
        self.dsave = np.zeros(13, float)
        self.bracket = False
        self.no_update = False
        self.case = 0

    def _save(self, stage, rest):
        self.isave[0] = 1 if self.bracket else 0
        self.isave[1] = stage
        self.dsave[:] = rest

    def step(self, stp, f, g, c1, c2, pk, old_stp):
        if self.task[:5] == "START":
            if stp < self.stpmin:
                self.task = "ERROR: STP .LT. minstep"
            if stp > self.stpmax:
                self.task = "ERROR: STP .GT. maxstep"
            if g >= 0:
                self.task = "ERROR: INITIAL G >= 0"
            if c1 < 0:
                self.task = "ERROR: c1 .LT. 0"
            if c2 < 0:
                self.task = "ERROR: c2 .LT. 0"
            if self.xtol < 0:
                self.task = "ERROR: XTOL .LT. 0"
            if self.stpmin < 0:
                self.task = "ERROR: minstep .LT. 0"
            if self.stpmax < self.stpmin:
                self.task = "ERROR: maxstep .LT. minstep"
            if self.task[:5] == "ERROR":
                return stp
            self.bracket = False
            stage = 1
            finit, ginit = f, g
            gtest = c1 * ginit
            width = self.stpmax - self.stpmin
            width1 = width / 0.5
            stx, fx, gx = 0, finit, ginit
            sty, fy, gy = 0, finit, ginit
            stmin = 0
            stmax = stp + self.xtrapu * stp
            self.task = "FG"
            self._save(stage, (ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1))
            return self.determine_step(stp, old_stp, pk)
        self.bracket = self.isave[0] == 1
        stage = self.isave[1]
        ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1 = self.dsave
        ftest = finit + stp * gtest
        if stage == 1 and f < ftest and g >= 0.0:
            stage = 2
        if self.bracket and (stp <= stmin or stp >= stmax):
            self.task = "WARNING: ROUNDING ERRORS PREVENT PROGRESS"
        if self.bracket and stmax - stmin <= self.xtol * stmax:
            self.task = "WARNING: XTOL TEST SATISFIED"
        if stp == self.stpmax and f <= ftest and g <= gtest:
            self.task = "WARNING: STP = maxstep"
        if stp == self.stpmin and (f > ftest or g >= gtest):
            self.task = "WARNING: STP = minstep"
        if f <= ftest and abs(g) <= c2 * (-ginit):
            self.task = "CONVERGENCE"
        if self.task[:4] == "WARN" or self.task[:4] == "CONV":
            self._save(stage, (ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1))
            return stp
        stx, sty, stp, gx, fx, gy, fy = self.update(stx, fx, gx, sty, fy, gy, stp, f, g, stmin, stmax, old_stp, pk)
        if self.bracket:
            if abs(sty - stx) >= 0.66 * width1:
                stp = stx + 0.5 * (sty - stx)
            width1 = width
            width = abs(sty - stx)
        if self.bracket:
            stmin = min(stx, sty)
            stmax = max(stx, sty)
        else:
            stmin = stp + self.xtrapl * (stp - stx)
            stmax = stp + self.xtrapu * (stp - stx)
        stp = max(stp, self.stpmin)
        stp = min(stp, self.stpmax)
        if stx == stp and stp == self.stpmax and stmin > self.stpmax:
            self.no_update = True
        if (self.bracket and stp < stmin or stp >= stmax) or (self.bracket and stmax - stmin < self.xtol * stmax):
            stp = stx
        self.task = "FG"
        self._save(stage, (ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1))
        return stp

    def update(self, stx, fx, gx, sty, fy, gy, stp, fp, gp, stpmin, stpmax, old_stp, pk):
        sign = gp * (gx / abs(gx))
        if fp > fx:
            self.case = 1
            theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp
            s = max(abs(theta), abs(gx), abs(gp))
            gamma = s * np.sqrt((theta / s) ** 2.0 - (gx / s) * (gp / s))
            if stp < stx:
                gamma = -gamma
            p = (gamma - gx) + theta
            q = ((gamma - gx) + gamma) + gp
            r = p / q
            stpc = stx + r * (stp - stx)
            stpq = stx + ((gx / ((fx - fp) / (stp - stx) + gx)) / 2.0) * (stp - stx)
            if abs(stpc - stx) < abs(stpq - stx):
                stpf = stpc
            else:
                stpf = stpc + (stpq - stpc) / 2.0
            self.bracket = True
        elif sign < 0:
            self.case = 2
            theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp
            s = max(abs(theta), abs(gx), abs(gp))
            gamma = s * np.sqrt((theta / s) ** 2 - (gx / s) * (gp / s))
            if stp > stx:
                gamma = -gamma
            p = (gamma - gp) + theta
            q = ((gamma - gp) + gamma) + gx
            r = p / q
            stpc = stp + r * (stx - stp)
            stpq = stp + (gp / (gp - gx)) * (stx - stp)
            if abs(stpc - stp) > abs(stpq - stp):
                stpf = stpc
            else:
                stpf = stpq
            self.bracket = True
        elif abs(gp) < abs(gx):
            self.case = 3
            theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp
            s = max(abs(theta), abs(gx), abs(gp))
            gamma = s * np.sqrt(max(0.0, (theta / s) ** 2 - (gx / s) * (gp / s)))
            if stp > stx:
                gamma = -gamma
            p = (gamma - gp) + theta
            q = (gamma + (gx - gp)) + gamma
            r = p / q
            if r < 0.0 and gamma != 0:
                stpc = stp + r * (stx - stp)
            elif stp > stx:
                stpc = stpmax
            else:
                stpc = stpmin
            stpq = stp + (gp / (gp - gx)) * (stx - stp)
            if self.bracket:
                if abs(stpc - stp) < abs(stpq - stp):
                    stpf = stpc
                else:
                    stpf = stpq
                if stp > stx:
                    stpf = min(stp + 0.66 * (sty - stp), stpf)
                else:
                    stpf = max(stp + 0.66 * (sty - stp), stpf)
            else:
                if abs(stpc - stp) > abs(stpq - stp):
                    stpf = stpc
                else:
                    stpf = stpq
                stpf = min(stpmax, stpf)
                stpf = max(stpmin, stpf)
        else:
            self.case = 4
            if self.bracket:
                theta = 3.0 * (fp - fy) / (sty - stp) + gy + gp
                s = max(abs(theta), abs(gy), abs(gp))
                gamma = s * np.sqrt((theta / s) ** 2 - (gy / s) * (gp / s))
                if stp > sty:
                    gamma = -gamma
                p = (gamma - gp) + theta
                q = ((gamma - gp) + gamma) + gy
                r = p / q
                stpc = stp + r * (sty - stp)
                stpf = stpc
            elif stp > stx:
                stpf = stpmax
            else:
                stpf = stpmin
        if fp > fx:
            sty, fy, gy = stp, fp, gp
        else:
            if sign < 0:
                sty, fy, gy = stx, fx, gx
            stx, fx, gx = stp, fp, gp
        stp = self.determine_step(stpf, old_stp, pk)
        return stx, sty, stp, gx, fx, gy, fy

    def determine_step(self, stp, old_stp, pk):
        dr = stp - old_stp
        x = np.reshape(pk, (-1, 3))
        steplengths = ((dr * x) ** 2).sum(1) ** 0.5
        maxsteplength = max(steplengths)
        if maxsteplength >= self.maxstep:
            dr *= self.maxstep / maxsteplength
        return old_stp + dr


def rank2_update(H, dr, dg, rhok):
    """H' = A1 H A2 + rhok dr dr^T for symmetric H, in O(n^2): the form csrc/quasinewton.cu evaluates, element for element."""
    dg = dg.astype(np.float64)
    u = H @ dg
    c = rhok * rhok * np.dot(dg, u) + rhok
    return H - rhok * (np.outer(dr, u) + np.outer(u, dr)) + c * np.outer(dr, dr)


def ase_update(H, dr, dg, rhok):
    """ASE 3.22's BFGSLineSearch.update product, O(n^3)."""
    eye = np.eye(len(dr), dtype=int)
    A1 = eye - dr[:, np.newaxis] * dg[np.newaxis, :] * rhok
    A2 = eye - dg[:, np.newaxis] * dr[np.newaxis, :] * rhok
    return np.dot(A1, np.dot(H, A2)) + rhok * dr[:, np.newaxis] * dr[np.newaxis, :]


class _Mol:
    """BFGSLineSearch + LineSearch for one molecule, driven one evaluation at a time."""

    def __init__(self, n_at, fixed, maxstep, c1, c2, alpha, stpmax, fmax, max_steps):
        self.n_at, self.fixed = n_at, fixed
        self.maxstep, self.c1, self.c2, self.alpha, self.stpmax = maxstep, c1, c2, alpha, stpmax
        self.fmax, self.max_steps = fmax, max_steps
        self.status, self.started = RUNNING, False
        self.nsteps = self.force_calls = self.function_calls = 0
        self.H = self.r0 = self.g0 = self.p = self.alpha_k = self.e0 = None
        self.ls = None  # the current line search; its no_update is BFGSLineSearch.no_update
        self.stp = None
        self.tasks = []   # every line-search task, in order (tests)
        self.cases = []   # (update case, bracketed before the call) of every LineSearch.update (tests)
        self.rescaled = 0  # steps whose |p| was rescaled (tests)
        self.no_update_accepts = 0  # line searches ended by no_update (tests)

    def _converged(self, f):
        return bool((f ** 2).sum(axis=1).max() < np.float32(self.fmax ** 2))

    def consume(self, pos, e, f):
        """E (float64, eV) and F (float32 [n,3], eV/A) at `pos` (float64 [n,3], the current trial point).  Returns the next point."""
        f = np.array(f, dtype=np.float32)
        if self.fixed is not None:
            f[self.fixed] = 0.0
        if not self.started:
            self.started = True
            if self._converged(f):
                self.status = CONVERGED
                return pos
            if self.nsteps >= self.max_steps:
                self.status = MAX_STEPS
                return pos
            return self._start_step(pos, e, f)
        self.force_calls += 1
        self.function_calls += 1
        if not self.ls.no_update:
            g = -f.reshape(-1) / np.float32(self.alpha)
            bracketed, self.ls.case = int(self.ls.isave[0]), 0
            stp = self.ls.step(self.stp, e / self.alpha, np.dot(g, self.p), self.c1, self.c2, self.p, self.stp)
            self.tasks.append(self.ls.task)
            if self.ls.case:
                self.cases.append((self.ls.case, bracketed))
            if self.ls.task[:2] == "FG":
                self.stp = stp
                return (self.r + stp * self.p).reshape(-1, 3)
            if self.ls.task[:5] == "ERROR":
                self.status = FAILED
                return pos
        else:
            self.no_update_accepts += 1
        self.alpha_k = self.stp
        self.r0, self.g0 = self.r, self.g
        self.nsteps += 1
        if self._converged(f):
            self.status = CONVERGED
            return pos
        if self.nsteps >= self.max_steps:
            self.status = MAX_STEPS
            return pos
        return self._start_step(pos, e, f)

    def _start_step(self, pos, e, f):
        r = pos.reshape(-1).astype(np.float64)
        g = -f.reshape(-1) / np.float32(self.alpha)
        self._update(r, g)
        self.function_calls += 1
        phi0 = e / self.alpha
        p = -np.dot(self.H, g.astype(np.float64))
        p_size = np.sqrt((p ** 2).sum())
        if p_size <= np.sqrt(self.n_at * 1e-10):
            p /= (p_size / np.sqrt(self.n_at * 1e-10))
            self.rescaled += 1
        if self.fixed is not None:
            assert not p.reshape(-1, 3)[self.fixed].any(), "a fixed atom would move"
        self.r, self.g, self.p, self.e0 = r, g, p, phi0
        self.ls = LineSearch(maxstep=self.maxstep, stpmax=self.stpmax)
        stp = self.ls.step(1.0, phi0, np.dot(g, p), self.c1, self.c2, p, 0)
        self.tasks.append(self.ls.task)
        if self.ls.task[:5] == "ERROR":
            self.status = FAILED
            return pos
        self.stp = stp
        return (r + stp * p).reshape(-1, 3)

    def _update(self, r, g):
        if self.H is None:
            self.H = np.eye(3 * self.n_at)
            return
        dr = r - self.r0
        dg = g - self.g0
        if not ((self.alpha_k or 0) > 0 and abs(np.dot(g, self.p)) - abs(np.dot(self.g0, self.p)) < 0):
            return
        if self.ls.no_update:
            return
        with np.errstate(divide="ignore"):
            rhok = 1.0 / np.dot(dg, dr)
        if np.isinf(rhok):
            rhok = 1000.0
        self.H = rank2_update(self.H, dr, dg, rhok)


class BatchQuasiNewton:
    """force_fn(pos [N,3] float64) -> (energy [B] float64 in eV, forces [N,3] float32 in eV/A).  `sizes` = atoms per molecule;
    `fixed_atoms_mask` = global atom indices held in place (FixAtoms)."""

    def __init__(self, force_fn, sizes, maxstep=0.2, c1=0.23, c2=0.46, alpha=10.0, stpmax=50.0, fixed_atoms_mask=None):
        self.force_fn, self.sizes = force_fn, np.asarray(sizes, dtype=np.int64)
        self.ptr = np.concatenate([[0], np.cumsum(self.sizes)])
        self.kw = dict(maxstep=maxstep, c1=c1, c2=c2, alpha=alpha, stpmax=stpmax)
        fixed = np.zeros(int(self.ptr[-1]), dtype=bool)
        if fixed_atoms_mask is not None:
            fixed[np.asarray(fixed_atoms_mask, dtype=np.int64)] = True
        self.fixed = [fixed[self.ptr[m]:self.ptr[m + 1]] if fixed[self.ptr[m]:self.ptr[m + 1]].any() else None for m in range(len(self.sizes))]

    def run(self, pos0, fmax=0.05, steps=None, record=False):
        """Relax every molecule; returns (positions [N,3] float64, status [B]).  With `record`, `self.evals` holds (pos, E, F) of every
        call and `self.after` the (next positions, status, nsteps, force_calls, function_calls) after consuming it."""
        max_steps = steps if steps else 100000000
        self.mols = [_Mol(int(n), self.fixed[m], fmax=fmax, max_steps=max_steps, **self.kw) for m, n in enumerate(self.sizes)]
        pos = np.asarray(pos0, dtype=np.float64).copy()
        self.n_calls, self.evals, self.after = 0, [], []
        while any(m.status == RUNNING for m in self.mols):
            e, f = self.force_fn(pos)
            e, f = np.asarray(e, dtype=np.float64), np.asarray(f, dtype=np.float32)
            self.n_calls += 1
            if record:
                self.evals.append((pos.copy(), e.copy(), f.copy()))
            for m, mol in enumerate(self.mols):
                if mol.status != RUNNING:
                    continue
                a, b = self.ptr[m], self.ptr[m + 1]
                pos[a:b] = mol.consume(pos[a:b].copy(), float(e[m]), f[a:b])
            if record:
                self.after.append((pos.copy(), self.status.copy(), self.nsteps.copy(), self.force_calls.copy(), self.function_calls.copy()))
        self.final_energy, self.final_forces = e, f
        return pos, self.status

    @property
    def status(self): return np.array([m.status for m in self.mols])
    @property
    def nsteps(self): return np.array([m.nsteps for m in self.mols])
    @property
    def force_calls(self): return np.array([m.force_calls for m in self.mols])
    @property
    def function_calls(self): return np.array([m.function_calls for m in self.mols])

    @property
    def failed(self):
        return [m for m, mol in enumerate(self.mols) if mol.status == FAILED]
