"""Batched molecular dynamics on the GPU: the reference's `init_md` / `run_md` for a whole batch of molecules.

The reference's `PYGAseInterface` (nablaDFT/optimization/pyg_ase_interface.py:207-294) runs ASE dynamics on one molecule: NVE velocity
Verlet, or Langevin NVT when `temp_bath` is given, with every step's forces coming through `PYGCalculator.calculate` -- a model call plus a
device -> host -> device round trip.  `BatchwiseMD` keeps positions (float64), momenta (float64) and the model's buffers on the device:
a step is the engine's energy + forces launch followed by ONE integrator launch (`nb200_md_step`, csrc/md.cu), and the host looks at the
device only once per chunk of `check_every` steps.  Semantics are ASE 3.22's (restated in oracle/md.py), including its units.

    md = BatchwiseMD(calculator, atoms, working_dir=None, masses=None, seed=0, check_every=50)
    md.init_md("equilibration", time_step=0.5, temp_init=300, temp_bath=300)
    md.run_md(2000)
    md.atoms, md.momenta, md.nsteps, md.log, md.frames

Random numbers come from a counter-based Philox stream keyed by `seed`, so a run is reproducible bit for bit, whatever `check_every`, and
however `run_md` splits the steps.  An edge-capacity overflow of the engine in a chunk is recovered by replaying the chunk from its
start with a larger capacity; the replay draws the same noise.
"""
import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import NablaB200Error, check, current_stream, ptr
from .optimization import _like, convert_units
from .vibrations import masses_of

# ASE 3.22 units (ase.units, CODATA 2014): eV, Angstrom, u; time in ASE units
FS = 0.09822694788464063       # 1 fs
KB = 8.617330337217213e-05     # Boltzmann constant, eV / K
LANGEVIN_FRICTION = 1.0 / (100.0 * FS)  # the reference's Langevin friction, 1 / (100 fs)

_FINISH, _START = 1, 2
_ECAPACITY = -4


def mdlogger_header() -> str:
    """Header line of ASE's MDLogger(peratom=False) with a time column."""
    return "%-9s " % "Time[ps]" + "%12s %12s %12s  %6s" % ("Etot[eV]", "Epot[eV]", "Ekin[eV]", "T[K]")


def mdlogger_line(time_ps: float, epot: float, ekin: float, temp: float, n_atoms: int) -> str:
    """One MDLogger row: energies with 4 decimals up to 100 atoms, fewer for larger systems, as ASE chooses."""
    digits = 4 if n_atoms <= 100 else 3 if n_atoms <= 1000 else 2 if n_atoms <= 10000 else 1
    e = "%%12.%df " % digits
    return ("%-10.4f " + 3 * e + " %6.1f") % (time_ps, epot + ekin, epot, ekin, temp)


class BatchwiseMD:
    """Molecular dynamics of a batch of molecules with `SpkBatchwiseCalculator` (spk PaiNN, SchNet) or `PyGBatchwiseCalculator` (PaiNN-OC).

    `masses` [n_atoms] in u overrides the standard atomic weights; `seed` keys the random stream; `check_every` is the number of steps
    between host looks at the device (status word, logs).  `fixed_atoms` is not supported."""

    def __init__(self, calculator, atoms: Sequence, working_dir: Optional[str] = None, masses=None, seed: int = 0, check_every: int = 50,
                 fixed_atoms=None):
        if fixed_atoms is not None or any(len(getattr(a, "constraints", ()) or ()) for a in atoms):
            raise NotImplementedError("fixed atoms are not supported by the device MD loop (ASE FixAtoms with Langevin fixcm is not restated)")
        dev = calculator.device
        if dev.type != "cuda":
            raise NablaB200Error("BatchwiseMD runs on CUDA only (no CPU fallback)")
        if int(check_every) < 1:
            raise ValueError("check_every must be >= 1")
        self.calculator, self.working_dir, self.seed, self.check_every = calculator, working_dir, int(seed), int(check_every)
        if not 0 <= self.seed < 2 ** 64:
            raise ValueError("seed must be in [0, 2^64)")
        self.lib = _lib.load()
        self._templates = list(atoms)
        self._z, pos, self._mol_ptr, self._sizes = calculator.pack(self._templates)
        self.n_mol, self.n_atoms = len(self._sizes), int(self._sizes.sum())
        if masses is None:
            m = masses_of(self._z)
        else:
            m = torch.as_tensor(masses, dtype=torch.float64).detach().cpu().reshape(-1)
            if m.numel() != self.n_atoms or not bool((m > 0).all()):
                raise ValueError(f"masses must be {self.n_atoms} positive values (u)")
        self._mass = m.to(dev).contiguous()
        self._pos = pos.contiguous()
        self._pos32 = pos.float().contiguous()
        self._mom = torch.zeros_like(self._pos)
        # model units -> eV, eV/A through the calculator's declared units
        self.e_scale = calculator.energy_conversion * convert_units("Hartree", "eV")
        self.f_scale = self.e_scale / calculator.position_conversion
        self._energy = self._forces = None
        self._eng = None
        self.noise_step = 0  # Philox counter: one per velocity draw and per MD step, never reused
        self.dynamics = None
        self.nsteps = 0
        self.log = np.zeros((0, self.n_mol, 5))
        self.frames = np.zeros((0, self.n_atoms, 3))
        self.host_syncs = 0
        self.replays = 0
        self._trajs = None

    # ------------------------------------------------------------------------------------------------------------------ reference API
    def init_md(self, name: str, time_step: float = 0.5, temp_init: float = 300, temp_bath: Optional[float] = None, reset: bool = False,
                interval: int = 1) -> None:
        """A new dynamics object: velocities are drawn only for the first one or with reset=True; nsteps and the logged time restart at 0."""
        if time_step <= 0 or temp_init < 0 or (temp_bath is not None and temp_bath < 0) or int(interval) < 1:
            raise ValueError("need time_step > 0, temperatures >= 0 and interval >= 1")
        if self.dynamics is None or reset:
            rc = self.lib.nb200_md_init_momenta(ptr(self._mol_ptr), self.n_mol, ptr(self._mass), ptr(self._pos), float(temp_init) * KB, self.seed,
                                                self.noise_step, ptr(self._mom), current_stream())
            check(rc, "nb200_md_init_momenta")
            self.noise_step += 1
        self.name, self.dt, self.interval = name, float(time_step) * FS, int(interval)
        self.thermostat = 0 if temp_bath is None else 1
        self.kT = 0.0 if temp_bath is None else float(temp_bath) * KB
        self.gamma = 0.0 if temp_bath is None else LANGEVIN_FRICTION
        self.dynamics = "VelocityVerlet" if temp_bath is None else "Langevin"
        self.nsteps = 0
        self.log = np.zeros((0, self.n_mol, 5))
        self.frames = np.zeros((0, self.n_atoms, 3))
        self._frame_mom = np.zeros((0, self.n_atoms, 3))
        self.close()
        if self.working_dir is not None:
            os.makedirs(self.working_dir, exist_ok=True)
            for i in range(self.n_mol):
                with open(os.path.join(self.working_dir, f"{name}_{i}.log"), "a") as f:
                    f.write(mdlogger_header() + "\n")
            try:
                from ase.io.trajectory import Trajectory
            except ImportError:  # like the optimiser's `trajectory`, .traj files need ASE
                Trajectory = None
            if Trajectory is not None:
                self._trajs = [Trajectory(os.path.join(self.working_dir, f"{name}_{i}.traj"), "w") for i in range(self.n_mol)]

    def close(self) -> None:
        """Close the .traj files of the current dynamics (the next init_md and garbage collection do this too)."""
        for traj in getattr(self, "_trajs", None) or ():
            traj.close()
        self._trajs = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run_md(self, steps: int) -> None:
        if not self.dynamics:
            raise AttributeError("Dynamics need to be initialized using the 'setup_md' function")
        steps = int(steps)
        if steps < 0:
            raise ValueError("steps must be >= 0")
        if self._forces is None:  # Dynamics.irun evaluates the forces before the first step; the calculator caches them afterwards
            self._eng = self.calculator.engine()
            energy, forces, st = self._eng.run(self._z, self._pos32, self._mol_ptr, self.n_mol)
            self._eng.e_cap = max(self._eng.e_cap, int(1.5 * int(st[0])) + 1024)  # head-room: the geometry moves without the host looking
            self._energy, self._forces = energy, forces
        if self.nsteps == 0:
            logs, fpos, fmom = self._buffers(1)
            self._launch(0, self.noise_step - 1, logs[0], fpos[0], fmom[0])
            self._append(logs, fpos, fmom, [0])
        done = 0
        while done < steps:
            k = min(self.check_every, steps - done)
            self._chunk(k)
            done += k

    @property
    def atoms(self) -> List:
        host = self._pos.cpu().numpy()
        mom = self._mom.cpu().numpy()
        off = np.concatenate([[0], np.cumsum(self._sizes)])
        out = []
        for i, a in enumerate(self._templates):
            at = _like(a, host[off[i]:off[i + 1]])
            if hasattr(at, "set_momenta"):
                at.set_momenta(mom[off[i]:off[i + 1]])
            out.append(at)
        return out

    @property
    def momenta(self) -> np.ndarray:
        """[n_atoms, 3] float64, u A / ASE time."""
        return self._mom.cpu().numpy()

    @property
    def positions(self) -> np.ndarray:
        return self._pos.cpu().numpy()

    # ------------------------------------------------------------------------------------------------------------------ device loop
    def _buffers(self, n_log: int):
        dev = self._pos.device
        return (torch.empty(n_log, self.n_mol, 2, dtype=torch.float64, device=dev),
                torch.empty(n_log, self.n_atoms, 3, dtype=torch.float64, device=dev),
                torch.empty(n_log, self.n_atoms, 3, dtype=torch.float64, device=dev))

    def _launch(self, phase, step, log=None, fpos=None, fmom=None, status=None, worst=None):
        rc = self.lib.nb200_md_step(ptr(self._mol_ptr), self.n_mol, ptr(self._mass), phase, self.thermostat, self.dt, self.kT, self.gamma, self.seed,
                                    step, self.f_scale, self.e_scale, ptr(self._pos), ptr(self._mom), ptr(self._pos32), ptr(self._forces),
                                    ptr(self._energy), ptr(log), ptr(fpos), ptr(fmom), ptr(status), ptr(worst), current_stream())
        check(rc, "nb200_md_step")

    def _chunk(self, k: int) -> None:
        """k steps: START, then per step one engine launch and one FINISH|START launch (FINISH alone at the end); one host look at the end.
        On NB200_ECAPACITY the chunk is replayed from copies taken at its start with a larger edge capacity."""
        eng = self._eng
        saved = [t.clone() for t in (self._pos, self._mom, self._pos32, self._forces, self._energy)]
        logged = [self.nsteps + j + 1 for j in range(k) if (self.nsteps + j + 1) % self.interval == 0]
        for _ in range(8):
            logs, fpos, fmom = self._buffers(len(logged))
            worst = torch.zeros(4, dtype=torch.int32, device=self._pos.device)
            self._launch(_START, self.noise_step - 1)
            slot = 0
            for j in range(k):
                energy, forces, status = eng.launch(self._z, self._pos32, self._mol_ptr, self.n_mol, e_cap=eng.e_cap)
                self._energy, self._forces = energy, forces
                log = (self.nsteps + j + 1) % self.interval == 0
                self._launch(_FINISH | (_START if j < k - 1 else 0), self.noise_step + j, logs[slot] if log else None, fpos[slot] if log else None,
                             fmom[slot] if log else None, status, worst)
                slot += int(log)
            host = worst.cpu()  # the one synchronisation of the chunk
            self.host_syncs += 1
            if int(host[3]):
                # overflow: restore the chunk's starting state and replay it; the counter-based noise makes the replay draw the same numbers
                eng.e_cap = int(1.25 * int(host[0])) + 1024
                self._pos.copy_(saved[0]); self._mom.copy_(saved[1]); self._pos32.copy_(saved[2])
                self._forces, self._energy = saved[3].clone(), saved[4].clone()
                self.replays += 1
                continue
            if int(host[1]):
                # any other engine error: leave the state as it was at the chunk start (nsteps and the noise step have not advanced), then raise
                self._pos.copy_(saved[0]); self._mom.copy_(saved[1]); self._pos32.copy_(saved[2])
                self._forces, self._energy = saved[3], saved[4]
                eng.raise_on_status(host)
            self.noise_step += k
            self.nsteps += k
            self._append(logs, fpos, fmom, logged)
            return
        raise NablaB200Error("edge capacity regrow failed")

    def _append(self, logs, fpos, fmom, steps: List[int]) -> None:
        if not steps:
            return
        lg = logs.cpu().numpy()
        epot, ekin = lg[..., 0], lg[..., 1]
        t = np.asarray(steps, dtype=np.float64)[:, None] * self.dt / (1000.0 * FS) * np.ones((1, self.n_mol))
        temp = 2.0 * ekin / (3 * self._sizes[None, :] * KB)
        rows = np.stack([t, epot + ekin, epot, ekin, temp], -1)
        self.log = np.concatenate([self.log, rows])
        fp, fm = fpos.cpu().numpy(), fmom.cpu().numpy()
        self.frames = np.concatenate([self.frames, fp])
        self._frame_mom = np.concatenate([self._frame_mom, fm])
        if self.working_dir is None:
            return
        for i in range(self.n_mol):
            with open(os.path.join(self.working_dir, f"{self.name}_{i}.log"), "a") as f:
                for r in rows[:, i]:
                    f.write(mdlogger_line(r[0], r[2], r[3], r[4], int(self._sizes[i])) + "\n")
        if self._trajs is not None:
            from ase import Atoms  # the inputs may be SimpleAtoms: the frames are written as ase.Atoms with momenta

            off = np.concatenate([[0], np.cumsum(self._sizes)])
            for i, (traj, a) in enumerate(zip(self._trajs, self._templates)):
                for s in range(len(steps)):
                    traj.write(Atoms(numbers=a.get_atomic_numbers(), positions=fp[s, off[i]:off[i + 1]], momenta=fm[s, off[i]:off[i + 1]]))
