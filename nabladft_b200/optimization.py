"""Batch-wise geometry optimisation: mirror of `nablaDFT/optimization/{calculator,optimizers,task}.py` (SURVEY.md section 8f-1).

Same class names, constructor arguments, `run(atoms, fmax, steps)` / `initialize()` / `.atoms` / `calculator.results` contract
as the reference, so `config/optimizer/batchwise_lbfgs.yaml` and `config/calculator/*_calculator.yaml` work with the
`_target_`s pointed here (nablaDFT/pipelines.py:54-81).  What changes is where the loop runs: the reference does, per step,
model -> D2H -> numpy two-loop recursion over Python lists -> new ase.Atoms list -> CPU neighbour list -> H2D
(optimizers.py:436-548, calculator.py:125-176).  Here positions, forces and the L-BFGS history stay in HBM; a step is the
engine's E+F launch followed by ONE kernel (`nb200_lbfgs_step`, csrc/lbfgs.cu) on the same stream, and the host only looks at a
device counter every `check_every` steps.  Converged molecules are frozen exactly as in the reference (optimizers.py:505-506),
so running past global convergence moves nothing and the final geometry equals the reference's stopping point.

Not built: `use_line_search=True` -- the reference documents it as "Not implemented yet" (optimizers.py:360-361), every shipped config sets
it False, and its own class crashes on it (TypeError at line_search.py:81 in two of the four golden scenarios, NaN positions for molecules that
converge early: tools/probe_reference_line_search.py), so there is no reference behaviour to reproduce; `restart` pickles.
"""
import sys
import time
from math import sqrt
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import NablaB200Error, check, current_stream, ptr

_HARTREE = {"hartree": 1.0, "ha": 1.0, "ev": 1.0 / 27.211386245988, "kcal/mol": 1.0 / 627.5094740631, "kj/mol": 1.0 / 2625.4996394799}
_ANGSTROM = {"ang": 1.0, "angstrom": 1.0, "a": 1.0, "bohr": 0.529177210903, "nm": 10.0}


def convert_units(src: str, dst: str) -> float:
    """schnetpack.units.convert_units for the units the reference's calculator configs use: value_dst = value_src * factor."""
    s, d = src.lower(), dst.lower()
    for table in (_HARTREE, _ANGSTROM):
        if s in table and d in table:
            return table[s] / table[d]
    raise ValueError(f"cannot convert {src!r} to {dst!r}")


class SimpleAtoms:
    """The slice of ase.Atoms the optimisation path touches (numbers, positions, pbc, cell, ==, copy).  Used when ASE is not
    installed; with ASE present, ase.Atoms objects go in and come out."""

    def __init__(self, positions=None, numbers=None, pbc=None, cell=None):
        self.positions = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.numbers = np.array(numbers, dtype=np.int64)
        self.pbc = np.zeros(3, dtype=bool) if pbc is None else np.array(pbc, dtype=bool)
        self.cell = np.zeros((3, 3)) if cell is None else np.array(cell, dtype=np.float64)

    def get_positions(self): return self.positions.copy()
    def get_atomic_numbers(self): return self.numbers.copy()
    def copy(self): return SimpleAtoms(self.positions, self.numbers, self.pbc, self.cell)
    def __len__(self): return len(self.numbers)

    def __eq__(self, other):
        return (np.array_equal(self.numbers, other.numbers) and np.array_equal(self.positions, other.positions)
                and np.array_equal(self.pbc, other.pbc) and np.array_equal(self.cell, other.cell))

    def __ne__(self, other): return not self.__eq__(other)


def _like(template, positions):
    """New Atoms object of the template's type with updated positions (optimizers.py:518-528)."""
    at = type(template)(positions=positions, numbers=template.get_atomic_numbers())
    at.pbc = template.pbc
    at.cell = template.cell
    return at


class BatchwiseCalculator:
    """calculator.py:15-96.  `model` is one of this package's CUDA models; `device` must be a CUDA device."""

    def __init__(self, model, device="cuda", energy_key: str = "energy", force_key: str = "forces", energy_unit: str = "eV",
                 position_unit: str = "Ang", dtype: torch.dtype = torch.float32):
        self.results: Optional[Dict[str, np.ndarray]] = None
        self.atoms = None
        self.device = torch.device(device) if isinstance(device, str) else device
        if self.device.type != "cuda":
            raise NablaB200Error("nabladft_b200 calculators run on CUDA only (no CPU fallback)")
        if dtype != torch.float32:
            raise NotImplementedError("the CUDA engines compute in float32 (the reference default, calculator.py:35)")
        self.dtype = dtype
        self.energy_key, self.force_key = energy_key, force_key
        self.energy_conversion = convert_units(energy_unit, "Hartree")
        self.position_conversion = convert_units(position_unit, "Angstrom")
        self.property_units = {energy_key: self.energy_conversion, force_key: self.energy_conversion / self.position_conversion}
        self.model = model
        self.model.to(device=self.device, dtype=self.dtype)
        self.model.eval()

    # ---- device side (used by the optimiser loop) -------------------------------------------------------------------
    def engine(self):
        raise NotImplementedError

    def pack(self, atoms: Sequence) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, np.ndarray]:
        sizes = np.array([len(a) for a in atoms], dtype=np.int64)
        z = torch.from_numpy(np.concatenate([np.asarray(a.get_atomic_numbers()) for a in atoms]).astype(np.int32)).to(self.device)
        pos = torch.from_numpy(np.concatenate([np.asarray(a.get_positions(), dtype=np.float64) for a in atoms])).to(self.device)
        mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(self.device)
        return z, pos, mol_ptr, sizes

    # ---- host side (reference API) -----------------------------------------------------------------------------------
    def _requires_calculation(self, property_keys: List[str], atoms: Sequence) -> bool:
        if self.results is None or any(k not in self.results for k in property_keys):
            return True
        if len(self.atoms) != len(atoms):
            return True
        return any(a != b for a, b in zip(atoms, self.atoms))

    def get_forces(self, atoms: Sequence, fixed_atoms_mask: Optional[List[int]] = None) -> np.ndarray:
        if self._requires_calculation([self.energy_key, self.force_key], atoms):
            self.calculate(atoms)
        f = self.results[self.force_key]
        if fixed_atoms_mask is not None:
            f[fixed_atoms_mask] = 0.0
        return f

    def get_potential_energy(self, atoms: Sequence) -> np.ndarray:
        if self._requires_calculation([self.energy_key], atoms):
            self.calculate(atoms)
        return self.results[self.energy_key]

    def calculate(self, atoms: Sequence) -> None:
        z, pos, mol_ptr, sizes = self.pack(atoms)
        energy, forces, _ = self.engine().run(z, pos.float().contiguous(), mol_ptr, len(sizes))
        self.set_results(energy, forces, atoms)

    def set_results(self, energy: torch.Tensor, forces: torch.Tensor, atoms: Sequence) -> None:
        self.results = {self.energy_key: energy.cpu().numpy() * self.property_units[self.energy_key],
                        self.force_key: forces.cpu().numpy() * self.property_units[self.force_key]}
        self.atoms = [a.copy() for a in atoms]


class PyGBatchwiseCalculator(BatchwiseCalculator):
    """calculator.py:98-129 for `nabladft_b200.painn_oc.PaiNN`, `nabladft_b200.gemnet_oc.GemNetOC` and
    `nabladft_b200.dimenetplusplus.DimeNetPlusPlusPotential` (net(data) -> (energy, forces))."""

    def engine(self):
        return self.model.engine()


class SpkBatchwiseCalculator(BatchwiseCalculator):
    """calculator.py:132-182 for `nabladft_b200.spk.NeuralNetworkPotential`.  `atoms_converter` (schnetpack AtomsConverter +
    ASENeighborList, config/calculator/spk_calculator.yaml:3-8) is accepted and ignored: the neighbour list is built on the device."""

    def __init__(self, model, atoms_converter=None, device="cuda", energy_key: str = "energy", force_key: str = "forces",
                 energy_unit: str = "eV", position_unit: str = "Ang", dtype: torch.dtype = torch.float32):
        super().__init__(model, device, energy_key, force_key, energy_unit, position_unit, dtype)
        self.atoms_converter = atoms_converter

    def engine(self):
        return self.model.engine(self.model.do_postprocessing and not self.model.training)


def _fold_status(worst: torch.Tensor, status: torch.Tensor) -> None:
    """Fold an engine launch's status words into `worst` on the device: the engine rewrites them at every launch, so a loop that looks
    at them once per chunk keeps the worst error code and the largest edge count / degree of the chunk, and an overflow in the middle
    of a chunk cannot hide behind a later clean launch."""
    torch.minimum(worst[1:2], status[1:2], out=worst[1:2])   # error codes are negative
    torch.maximum(worst[0:1], status[0:1], out=worst[0:1])   # edges
    torch.maximum(worst[2:3], status[2:3], out=worst[2:3])   # max degree


class BatchwiseOptimizer:
    """optimizers.py:126-289 (the parts that do not depend on ASE's Dynamics base class)."""

    defaults = {"maxstep": 0.2}

    def __init__(self, calculator: BatchwiseCalculator, restart=None, logfile: Optional[str] = None, trajectory: Optional[str] = None,
                 master=None, append_trajectory: bool = False, log_every_step: bool = False, fixed_atoms_mask: Optional[List[int]] = None):
        if restart is not None:
            raise NotImplementedError("restart pickles (optimizers.py:278-289) are not supported by the device loop")
        self.calculator, self.trajectory, self.log_every_step, self.fixed_atoms_mask = calculator, trajectory, log_every_step, fixed_atoms_mask
        self.logfile = sys.stdout if logfile == "-" else (open(logfile, "a") if isinstance(logfile, str) else None)
        self.restart, self.fmax, self.atoms = None, None, None
        self.nsteps, self.max_steps = 0, 100000000
        self.initialize()

    def todict(self) -> Dict:
        return {"type": "optimization", "optimizer": self.__class__.__name__}

    def initialize(self):
        pass

    def converged(self, forces: Optional[np.ndarray] = None) -> bool:
        if forces is None:
            forces = self.calculator.get_forces(self.atoms, fixed_atoms_mask=self.fixed_atoms_mask)
        return bool((forces ** 2).sum(axis=1).max() < self.fmax ** 2)

    def log(self, forces: Optional[np.ndarray] = None) -> None:  # optimizers.py:249-272
        if forces is None:
            forces = self.calculator.get_forces(self.atoms, fixed_atoms_mask=self.fixed_atoms_mask)
        fmax = sqrt((forces ** 2).sum(axis=1).max())
        t = time.localtime()
        if self.logfile is not None:
            name = self.__class__.__name__
            if self.nsteps == 0:
                self.logfile.write("%s  %4s %8s %12s\n" % (" " * len(name), "Step", "Time", "fmax"))
            self.logfile.write("%s:  %3d %02d:%02d:%02d %12.4f\n" % (name, self.nsteps, t[3], t[4], t[5], fmax))
            self.logfile.flush()
        if self.trajectory is not None:
            from ase.io import write  # needs ASE, like the reference

            for idx, at in enumerate(self.atoms):
                write(self.trajectory + f"_{idx}.xyz", at, format="extxyz", append=self.nsteps != 0)

    def _sync_atoms(self, pos: torch.Tensor) -> None:
        """`.atoms` = new Atoms objects at the device positions (float64 [n_atoms, 3]), split by `n_ats_per_config`."""
        host = pos.cpu().numpy()
        off = np.concatenate([[0], np.cumsum(self.n_ats_per_config)])
        self.atoms = [_like(a, host[off[i]:off[i + 1]]) for i, a in enumerate(self.atoms)]

    def get_relaxation_results(self):
        self.calculator.get_forces(self.atoms)
        return self.atoms, self.calculator.results


class ASEBatchwiseLBFGS(BatchwiseOptimizer):
    """optimizers.py:292-659 with the loop on the device.  Extra argument: `check_every` = steps between host looks at the
    device convergence counter (1 reproduces the reference's per-step check; the result is the same for any value)."""

    def __init__(self, calculator: BatchwiseCalculator, restart=None, logfile: Optional[str] = "-", trajectory: Optional[str] = None,
                 maxstep: Optional[float] = None, memory: int = 100, damping: float = 1.0, alpha: float = 1.0, use_line_search: bool = False,
                 master=None, log_every_step: bool = False, fixed_atoms_mask: Optional[List[int]] = None, verbose: bool = False,
                 check_every: int = 10):
        super().__init__(calculator, restart, logfile, trajectory, master, False, log_every_step, fixed_atoms_mask)
        self.maxstep = maxstep if maxstep is not None else self.defaults["maxstep"]
        if self.maxstep > 1.0:
            raise ValueError("You are using a much too large value for the maximum step size: %.1f Angstrom" % maxstep)
        if use_line_search:
            raise NotImplementedError("use_line_search=True: 'Not implemented yet' in the reference (optimizers.py:360-361; its class raises TypeError "
                                      "at line_search.py:81, see tools/probe_reference_line_search.py); config/optimizer/batchwise_lbfgs.yaml uses False")
        self.memory, self.H0, self.damping, self.verbose = int(memory), 1.0 / alpha, damping, verbose
        self.use_line_search = False
        self.check_every = 1 if (log_every_step or trajectory is not None) else max(1, int(check_every))
        self.record_positions = False  # tests: with check_every = 1 keep the float64 positions after every step
        self.lib = _lib.load()

    def initialize(self) -> None:  # optimizers.py:405-421
        self.nsteps = self.iteration = 0
        self.function_calls = self.force_calls = self.n_normalizations = 0
        self.host_syncs = 0  # times run() waited for the device: 1 at the start, 1 per `check_every` steps, 1 at the end (+ 1 per logged step)
        self._state = None

    # ------------------------------------------------------------------------------------------------------------------
    def run(self, atoms: Sequence, fmax: float = 0.05, steps: Optional[int] = None) -> bool:
        calc, dev = self.calculator, self.calculator.device
        self.atoms, self.fmax = list(atoms), fmax
        self.n_configs = len(self.atoms)
        if steps:
            self.max_steps = steps
        z, pos, mol_ptr, sizes = calc.pack(self.atoms)
        self.n_ats, self.n_ats_per_config = int(sizes.sum()), sizes
        n_mol, n_atoms, max_at = len(sizes), int(sizes.sum()), int(sizes.max()) if len(sizes) else 0
        f_unit = calc.property_units[calc.force_key]
        need = self.lib.nb200_lbfgs_state_bytes(n_mol, n_atoms, self.memory)
        if need < 0:
            check(int(need), "nb200_lbfgs_state_bytes")
        state = torch.empty(int(need), dtype=torch.uint8, device=dev)
        pos32 = pos.float().contiguous()
        fixed = None
        if self.fixed_atoms_mask is not None:
            fixed = torch.zeros(n_atoms, dtype=torch.uint8, device=dev)
            fixed[torch.as_tensor(list(self.fixed_atoms_mask), dtype=torch.long, device=dev)] = 1
        chunk = self.check_every
        unconv = torch.full((chunk,), -1, dtype=torch.int32, device=dev)
        n_norm = torch.zeros(1, dtype=torch.int32, device=dev)

        eng = calc.engine()
        energy, forces, st = eng.run(z, pos32, mol_ptr, n_mol)  # first evaluation: synchronous, sizes the edge capacity
        eng.e_cap = max(eng.e_cap, int(1.5 * int(st[0])) + 1024)  # head-room: the geometry moves without the host looking
        self.host_syncs += 1
        if f_unit != 1.0:
            forces = forces * f_unit
        if self.nsteps == 0:
            self._log_device(forces, fixed)
        self.positions_history = [pos.cpu().numpy().copy()]
        worst = torch.zeros(4, dtype=torch.int32, device=dev)
        done_at, it = None, 0
        while it < self.max_steps and done_at is None:
            n_chunk = min(chunk, self.max_steps - it)
            for k in range(n_chunk):
                rc = self.lib.nb200_lbfgs_step(ptr(state), state.numel(), ptr(mol_ptr), n_mol, n_atoms, max_at, self.memory, self.iteration,
                                               float(fmax), float(self.maxstep), float(self.damping), float(self.H0), ptr(fixed), ptr(pos),
                                               ptr(forces), ptr(pos32), unconv[k:].data_ptr(), ptr(n_norm), current_stream())
                check(rc, "nb200_lbfgs_step")
                self.iteration += 1
                energy, forces, status = eng.launch(z, pos32, mol_ptr, n_mol, e_cap=eng.e_cap)
                _fold_status(worst, status)
                if f_unit != 1.0:
                    forces = forces * f_unit
            host = unconv[:n_chunk].cpu()  # the only host<->device synchronisation of the loop
            self.host_syncs += 1
            eng.raise_on_status(worst.cpu())
            zero = (host == 0).nonzero()
            if len(zero):
                done_at = it + int(zero[0])  # the reference's converged() was true before this step: it ran `done_at` steps
            it += n_chunk
            if self.record_positions and chunk == 1 and done_at is None:
                self.positions_history.append(pos.cpu().numpy().copy())
            if self.log_every_step and done_at is None:
                self.nsteps = it
                self._sync_atoms(pos)
                self._log_device(forces, fixed)
                self.host_syncs += 1
        self.nsteps = done_at if done_at is not None else it
        self.force_calls += self.nsteps
        self.function_calls += self.nsteps
        # normalisations counted after the stopping point belong to frozen molecules: there are none (p = 0 there)
        self.n_normalizations += int(n_norm.item())
        self.host_syncs += 1  # this and the reads of the final geometry, energies and forces below
        if fixed is not None:
            forces = forces.masked_fill(fixed.bool()[:, None], 0.0)  # the reference's final log() zeroes them in results (calculator.py:86-88)
        self._sync_atoms(pos)
        calc.results = {calc.energy_key: energy.cpu().numpy() * calc.property_units[calc.energy_key], calc.force_key: forces.cpu().numpy()}
        calc.atoms = [a.copy() for a in self.atoms]
        self.log(calc.results[calc.force_key])
        return self.converged(calc.results[calc.force_key])

    def _log_device(self, forces: torch.Tensor, fixed) -> None:
        if self.logfile is None and self.trajectory is None:
            return
        f = forces if fixed is None else forces.masked_fill(fixed.bool()[:, None], 0.0)
        self.log(f.cpu().numpy())


class BatchwiseQuasiNewton(BatchwiseOptimizer):
    """`PYGAseInterface.optimize()` (pyg_ase_interface.py:296-315: ASE's QuasiNewton = BFGSLineSearch) for a whole batch on the device.
    Every molecule follows its own BFGS + More-Thuente line-search trajectory exactly as ASE runs it alone (oracle/quasinewton.py); the
    batch shares the force calls.  The loop is the engine's E+F launch followed by ONE kernel (`nb200_qn_step`, csrc/quasinewton.cu) on
    the same stream; the host looks at a device counter of running molecules every `check_every` launches.  Energies and forces enter
    the optimiser in eV and eV/A, converted from the calculator's declared units as `PYGCalculator` does.

    After `run`: `.atoms`, `calculator.results` (the calculator's units, fixed atoms' forces zeroed), and per molecule `nsteps`,
    `force_calls`, `function_calls` and `status` (0 running, 1 converged, 2 reached `steps`, 3 line search failed) as numpy arrays;
    `launches` = engine launches of the run, `launches_used` = those whose evaluation some molecule consumed (the rest are the no-op
    tail of the last `check_every` chunk), `host_syncs` = times the loop waited for the device.  Every `run` starts these afresh."""

    def __init__(self, calculator: BatchwiseCalculator, logfile: Optional[str] = None, maxstep: Optional[float] = None, c1: float = 0.23,
                 c2: float = 0.46, alpha: float = 10.0, stpmax: float = 50.0, fixed_atoms_mask: Optional[List[int]] = None, check_every: int = 10):
        super().__init__(calculator, None, logfile, None, None, False, False, fixed_atoms_mask)
        self.maxstep = maxstep if maxstep is not None else self.defaults["maxstep"]
        self.c1, self.c2, self.alpha, self.stpmax = float(c1), float(c2), float(alpha), float(stpmax)
        self.check_every = max(1, int(check_every))
        self.lib = _lib.load()

    def initialize(self) -> None:
        self.nsteps = self.force_calls = self.function_calls = self.status = None
        self.launches = self.launches_used = self.host_syncs = 0

    def run(self, atoms: Sequence, fmax: float = 0.05, steps: Optional[int] = None) -> bool:
        if any(len(getattr(a, "constraints", ()) or ()) for a in atoms):
            raise NotImplementedError("ase.Atoms constraints are not read by the device loop: pass the fixed atoms as fixed_atoms_mask "
                                      "(global indices into the batch) instead of a FixAtoms constraint")
        self.initialize()
        calc, dev = self.calculator, self.calculator.device
        self.atoms, self.fmax = list(atoms), fmax
        max_steps = steps if steps else 100000000
        z, pos, mol_ptr, sizes = calc.pack(self.atoms)
        self.n_ats_per_config = sizes
        n_mol, n_atoms, max_at = len(sizes), int(sizes.sum()), int(sizes.max()) if len(sizes) else 0
        e_scale = calc.energy_conversion * convert_units("Hartree", "eV")
        f_scale = e_scale / calc.position_conversion
        h_off = np.concatenate([[0], np.cumsum((3 * sizes) ** 2)]).astype(np.int64)
        hess_elems = int(h_off[-1])
        h_off = torch.from_numpy(h_off[:-1].copy()).to(dev)
        need = self.lib.nb200_qn_state_bytes(n_mol, n_atoms, hess_elems)
        if need < 0:
            check(int(need), "nb200_qn_state_bytes")
        state = torch.zeros(int(need), dtype=torch.uint8, device=dev)
        info = torch.zeros(n_mol, 4, dtype=torch.int32, device=dev)
        pos32 = pos.float().contiguous()
        fixed = None
        if self.fixed_atoms_mask is not None:
            fixed = torch.zeros(n_atoms, dtype=torch.uint8, device=dev)
            fixed[torch.as_tensor(list(self.fixed_atoms_mask), dtype=torch.long, device=dev)] = 1
        chunk = self.check_every
        running = torch.full((chunk,), -1, dtype=torch.int32, device=dev)

        eng = calc.engine()
        energy, forces, st = eng.run(z, pos32, mol_ptr, n_mol)  # first evaluation: synchronous, sizes the edge capacity
        eng.e_cap = max(eng.e_cap, int(1.5 * int(st[0])) + 1024)  # head-room: the geometry moves without the host looking
        self.host_syncs += 1
        self.launches = self.launches_used = 1
        worst = torch.zeros(4, dtype=torch.int32, device=dev)
        while True:
            for k in range(chunk):
                rc = self.lib.nb200_qn_step(ptr(state), state.numel(), ptr(mol_ptr), ptr(h_off), n_mol, n_atoms, max_at, hess_elems, float(fmax),
                                            int(max_steps), float(self.maxstep), self.c1, self.c2, self.alpha, self.stpmax, float(e_scale),
                                            float(f_scale), ptr(fixed), ptr(energy), ptr(forces), ptr(pos), ptr(pos32), ptr(info),
                                            running[k:].data_ptr(), current_stream())
                check(rc, "nb200_qn_step")
                energy, forces, status = eng.launch(z, pos32, mol_ptr, n_mol, e_cap=eng.e_cap)
                _fold_status(worst, status)
                self.launches += 1
            host, mol = running.cpu(), info.cpu().numpy()  # the only host<->device synchronisation of the loop
            self.host_syncs += 1
            self.launches_used += int((host > 0).sum())  # the launch after a step that left molecules running is consumed by the next step
            eng.raise_on_status(worst.cpu())
            self.status, self.nsteps, self.force_calls, self.function_calls = (mol[:, i].copy() for i in range(4))
            if (self.status == 4).any():
                raise NablaB200Error("nb200_qn_step: a molecule larger than max_atoms_per_mol or inverse-Hessian offsets outside the state buffer")
            failed = np.flatnonzero(self.status == 3)
            if len(failed):
                self._sync_atoms(pos)
                raise RuntimeError(f"LineSearch failed! (molecules {failed.tolist()})")
            if int(host[-1]) == 0:
                break
        if fixed is not None:
            forces = forces.masked_fill(fixed.bool()[:, None], 0.0)
        self._sync_atoms(pos)
        calc.results = {calc.energy_key: energy.cpu().numpy() * calc.property_units[calc.energy_key],
                        calc.force_key: forces.cpu().numpy() * calc.property_units[calc.force_key]}
        calc.atoms = [a.copy() for a in self.atoms]
        self.host_syncs += 1
        if self.logfile is not None:
            f = calc.results[calc.force_key]
            self.logfile.write("%s: %d molecules, %d converged, steps %d..%d, force calls %d..%d, %d engine launches, fmax %.4f\n"
                               % (self.__class__.__name__, n_mol, int((self.status == 1).sum()), int(self.nsteps.min(initial=0)),
                                  int(self.nsteps.max(initial=0)), int(self.force_calls.min(initial=0)), int(self.force_calls.max(initial=0)),
                                  self.launches, sqrt(float((f ** 2).sum(axis=1).max(initial=0.0)))))
            self.logfile.flush()
        return bool((self.status == 1).all())


class BatchwiseOptimizeTask:
    """task.py:9-73: walks an ASE database in batches, relaxes each batch, writes geometries + model energy/forces to the output
    database.  Needs ASE for the database I/O, exactly like the reference."""

    def __init__(self, input_datapath: str, output_datapath: str, optimizer: BatchwiseOptimizer, batch_size: int, fmax: float, steps: int):
        from ase.db import connect

        self.optimizer, self.bs, self.fmax, self.steps = optimizer, batch_size, fmax, steps
        self.data_db_conn, self.out_db_conn = connect(input_datapath), connect(output_datapath)

    def optimize_batch(self, atoms_list: List):
        self.optimizer.initialize()
        self.optimizer.run(atoms_list, fmax=self.fmax, steps=self.steps)
        return self.optimizer.atoms

    def run(self):
        db_len = len(self.data_db_conn)
        for start in range(0, db_len, self.bs):
            ids = range(start, min(db_len, start + self.bs))
            atoms_list = self.optimize_batch([self.data_db_conn.get(i + 1).toatoms() for i in ids])
            res, force_idx = self.optimizer.calculator.results, 0
            for rel, i in enumerate(ids):
                row = self.data_db_conn.get(i + 1)
                data = row.data
                data["model_energy"] = [float(res["energy"][rel])]
                data["model_forces"] = res["forces"][force_idx:force_idx + row.natoms]
                force_idx += row.natoms  # the reference never advances force_idx (task.py:55-64): every row gets molecule 0's slice
                self.out_db_conn.write(atoms_list[rel], data=data, moses_id=row.moses_id, conformation_id=row.conformation_id, smiles=row.smiles)


class PackedOptimizeTask:
    """`BatchwiseOptimizeTask` without ASE: walks a `nabladft_b200.data.PackedEnergyDataset` in batches (task.py:45-69 semantics: batch i =
    molecules [i * bs, (i + 1) * bs), `optimizer.initialize()` before each batch) and returns, per molecule, the relaxed positions and the
    model energy / forces at the relaxed geometry -- what the reference writes to the output database as `model_energy` / `model_forces`."""

    def __init__(self, dataset, optimizer: BatchwiseOptimizer, batch_size: int, fmax: float, steps: int):
        self.dataset, self.optimizer, self.bs, self.fmax, self.steps = dataset, optimizer, int(batch_size), fmax, steps

    def run(self) -> Dict[str, np.ndarray]:
        d = self.dataset
        pos_out = np.zeros((len(d.z), 3), dtype=np.float64)
        forces_out = np.zeros((len(d.z), 3), dtype=np.float32)
        energy_out = np.zeros(len(d), dtype=np.float32)
        nsteps = []
        for start in range(0, len(d), self.bs):
            ids = range(start, min(len(d), start + self.bs))
            atoms = [SimpleAtoms(np.asarray(d.pos[int(d.ptr[i]):int(d.ptr[i + 1])], dtype=np.float64), np.asarray(d.z[int(d.ptr[i]):int(d.ptr[i + 1])]))
                     for i in ids]
            self.optimizer.initialize()
            self.optimizer.run(atoms, fmax=self.fmax, steps=self.steps)
            res = self.optimizer.calculator.results
            a, b = int(d.ptr[ids[0]]), int(d.ptr[ids[-1] + 1])
            pos_out[a:b] = np.concatenate([at.get_positions() for at in self.optimizer.atoms])
            forces_out[a:b] = res[self.optimizer.calculator.force_key]
            energy_out[ids[0]:ids[-1] + 1] = res[self.optimizer.calculator.energy_key]
            nsteps.append(int(np.max(self.optimizer.nsteps)))  # BatchwiseQuasiNewton counts per molecule: the batch's longest
        return {"positions": pos_out, "model_forces": forces_out, "model_energy": energy_out, "nsteps": np.asarray(nsteps)}
