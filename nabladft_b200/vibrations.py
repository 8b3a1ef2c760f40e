"""Analytic Hessians and normal modes of the PaiNN, SchNet, DimeNet++ and GemNet-OC models on the GPU.

The reference's `PYGAseInterface.compute_normal_modes` (nablaDFT/optimization/pyg_ase_interface.py) runs ASE `Vibrations`: central finite
differences of the forces, one molecule at a time, 6N + 1 force calls per molecule with a 0.01 A step.  Here the engine computes exact
Hessian-vector products H v = -(dF/dR) v (`PainnEngine.run_hvp`, `DimeNetRunner.run_hvp`, `GemNetOCRunner.run_hvp`; DESIGN.md section
3.13 for PaiNN, 3.13.1 for SchNet, 3.15.2 for DimeNet++, 3.9.1 for GemNet-OC), and since
molecules do not interact, ONE direction displaces atom k of every molecule of the batch at once: the Hessians of a whole batch take
3 * n_max directions, n_max = the atom count of the largest molecule.

    hessian_vector_product(model, batch, v) -> (energy, forces, hv)
    hessians(model, batch, max_dir=None)    -> per-molecule [3n, 3n] Hessians, Ha/A^2
    normal_modes(model, batch, masses=None) -> per-molecule eigenvalues, modes, wavenumbers (cm^-1) and ASE-style energies (meV)

`model` is `spk.NeuralNetworkPotential` (PaiNN or SchNet representation; `batch` = its inputs dict), `painn_oc.PaiNN` (`batch` has
.z, .pos, .batch and optionally .ptr), `dimenetplusplus.DimeNetPlusPlusPotential` or `gemnet_oc.GemNetOC` (`batch` has .z, .pos and a sorted
.batch).  H is the Hessian of the energy the forces are the gradient of: for DimeNet++ that is the unscaled prediction (the scaler touches
the energy only).  GemNet-OC predicts its forces directly, so there H is the force Jacobian -(dF/dR), which is not symmetric; `hessians`
reports its symmetric part, which is what ASE `Vibrations` computes from central differences of the same forces.  Everything runs in fp32 on the device except the diagonalisation (float64, `torch.linalg.eigh`).
"""
import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import torch


# Standard atomic weights in u: IUPAC conventional values as used by ASE 3.22 (`ase.data.atomic_masses`), for the elements of nablaDFT.
ATOMIC_MASSES: Dict[int, float] = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999, 9: 18.998403163, 16: 32.06, 17: 35.45, 35: 79.904}

# CODATA 2018 (exact where the SI defines them)
HARTREE_J = 4.3597447222071e-18   # E_h
AMU_KG = 1.66053906660e-27        # u
ANGSTROM_M = 1e-10
C_CM_PER_S = 2.99792458e10        # c
PLANCK_JS = 6.62607015e-34        # h
EV_J = 1.602176634e-19            # e

# sqrt(lambda [Ha / (A^2 u)]) -> angular frequency in 1/s; / (2 pi c) -> cm^-1
_OMEGA_PER_SQRT_LAMBDA = math.sqrt(HARTREE_J / (ANGSTROM_M ** 2 * AMU_KG))
CM1_PER_SQRT_LAMBDA = _OMEGA_PER_SQRT_LAMBDA / (2.0 * math.pi * C_CM_PER_S)
MEV_PER_CM1 = 1e3 * PLANCK_JS * C_CM_PER_S / EV_J  # h c in meV cm


# ---------------------------------------------------------------------------------------------------------------- model plumbing
def _engine_inputs(model, batch):
    """(engine, z int32, pos fp32, mol_ptr int32, n_mol) of `model.engine_inputs(batch)`, with the errors the model raises."""
    if not hasattr(model, "engine_inputs"):
        raise NotImplementedError("Hessians need nabladft_b200.spk.NeuralNetworkPotential, nabladft_b200.painn_oc.PaiNN, "
                                  "nabladft_b200.dimenetplusplus.DimeNetPlusPlusPotential or nabladft_b200.gemnet_oc.GemNetOC, "
                                  f"not {type(model).__name__}")
    return model.engine_inputs(batch)


def hessian_vector_product(model, batch, v: torch.Tensor):
    """(energy [B], forces [N, 3], hv) with hv = H v in Ha/A for v [N, 3] or [n_dir, N, 3] in A (hv has v's shape).  For GemNet-OC, whose
    forces are a direct output, hv = -(dF/dR) v is the product with the force Jacobian, which is not symmetric."""
    eng, z, pos, mol_ptr, n_mol = _engine_inputs(model, batch)
    vv = v.detach().to(device=pos.device, dtype=torch.float32)
    one = vv.dim() == 2
    vv = (vv.unsqueeze(0) if one else vv).contiguous()
    energy, forces, hv = eng.run_hvp(z, pos, mol_ptr, n_mol, vv)
    return energy, forces, (hv[0] if one else hv)


# ---------------------------------------------------------------------------------------------------------------- Hessians
class Hessians(list):
    """Per-molecule symmetrised Hessians (H + H^T) / 2, [3n_m, 3n_m] in Ha/A^2, rows and columns ordered (atom, xyz).
    `max_asymmetry`: the largest |H_ij - H_ji| of the raw products (Ha/A^2), a check of the fp32 arithmetic; `energy`: [B] in Ha.
    For GemNet-OC the raw products are those of the direct forces' Jacobian, which no energy has as its Hessian: there `max_asymmetry`
    measures the model's non-conservative part, not fp32 error.  That part is what ASE `Vibrations` discards when it symmetrises."""

    max_asymmetry: float = 0.0
    energy: Optional[torch.Tensor] = None


def shared_directions(mol_ptr: Sequence[int], d0: int, d1: int, device=None) -> torch.Tensor:
    """Directions d0 <= d < d1 of the shared layout, [d1 - d0, N, 3]: direction d = 3 k + c is a unit displacement along axis c of atom k
    of every molecule with more than k atoms."""
    mol_ptr = [int(p) for p in mol_ptr]
    starts = torch.tensor(mol_ptr[:-1], dtype=torch.int64)
    sizes = torch.tensor([b - a for a, b in zip(mol_ptr[:-1], mol_ptr[1:])], dtype=torch.int64)
    v = torch.zeros(d1 - d0, mol_ptr[-1], 3, dtype=torch.float32)
    for j, d in enumerate(range(d0, d1)):
        k, c = divmod(d, 3)
        v[j, starts[sizes > k] + k, c] = 1.0
    return v.to(device) if device is not None else v


def hessians_from_hvp(hvp: Callable[[torch.Tensor], torch.Tensor], mol_ptr: Sequence[int], max_dir: Optional[int] = None,
                      device=None) -> Hessians:
    """Per-molecule Hessians from a Hessian-vector-product callable hv = hvp(v), v and hv [n_dir, N, 3].  The 3 n_max shared directions
    (`shared_directions`) go through `hvp` in chunks of at most `max_dir`; column 3k + c of molecule m's Hessian is hv of direction 3k + c
    restricted to m's atoms."""
    mol_ptr = [int(p) for p in mol_ptr]
    sizes = [b - a for a, b in zip(mol_ptr[:-1], mol_ptr[1:])]
    n_dir = 3 * max(sizes)
    step = n_dir if max_dir is None else int(max_dir)
    if step < 1:
        raise ValueError("max_dir must be >= 1")
    raw = [None] * len(sizes)
    for d0 in range(0, n_dir, step):
        d1 = min(d0 + step, n_dir)
        hv = hvp(shared_directions(mol_ptr, d0, d1, device))
        for m, (a, n) in enumerate(zip(mol_ptr[:-1], sizes)):
            hi = min(d1, 3 * n)
            if hi <= d0:
                continue
            if raw[m] is None:
                raw[m] = torch.zeros(3 * n, 3 * n, dtype=hv.dtype, device=hv.device)
            raw[m][:, d0:hi] = hv[:hi - d0, a:a + n].reshape(hi - d0, 3 * n).t()
    out = Hessians()
    worst = 0.0
    for h in raw:
        if h.numel():
            worst = max(worst, float((h - h.t()).abs().max()))
        out.append(0.5 * (h + h.t()))
    out.max_asymmetry = worst
    return out


def hessians(model, batch, max_dir: Optional[int] = None) -> Hessians:
    """Exact per-molecule Hessians of the energy whose gradient the forces are (for DimeNet++ the unscaled prediction), [3n_m, 3n_m] in
    Ha/A^2 (symmetrised; see `Hessians`).  `max_dir` bounds the directions per
    engine call, hence the v and hv buffers (n_dir x N x 3 floats each); the engine workspace does not depend on it, and every call re-runs
    the primal forward once."""
    eng, z, pos, mol_ptr, n_mol = _engine_inputs(model, batch)
    ptr_host = mol_ptr.cpu().tolist()
    energy = []

    def hvp(v):
        e, _, hv = eng.run_hvp(z, pos, mol_ptr, n_mol, v, with_forces=False)
        energy.append(e)
        return hv

    try:
        out = hessians_from_hvp(hvp, ptr_host, max_dir, pos.device)
    finally:
        release = getattr(eng, "release_hvp_workspace", None)  # GemNet-OC: the workspace holds the training arena twice
        if release is not None:
            release()
    out.energy = energy[0]
    return out


# ---------------------------------------------------------------------------------------------------------------- normal modes
@dataclass
class NormalModes:
    """One molecule.  eigenvalues [3n] of the mass-weighted Hessian, Ha / (A^2 u), ascending; modes [3n, 3n]: its orthonormal eigenvectors
    (columns); wavenumbers [3n] in cm^-1 and energies [3n] in meV (h c nu~, ASE `Vibrations.summary`), imaginary modes as negative values."""

    eigenvalues: torch.Tensor
    modes: torch.Tensor
    wavenumbers: torch.Tensor
    energies_meV: torch.Tensor

    @property
    def n_imaginary(self) -> int:
        return int((self.wavenumbers < 0).sum())


def wavenumbers_from_eigenvalues(lam: torch.Tensor) -> torch.Tensor:
    """nu~ = sqrt(lambda E_h / (A^2 u)) / (2 pi c) in cm^-1 for eigenvalues in Ha / (A^2 u); negative lambda -> -nu~ of |lambda|."""
    return torch.sign(lam) * torch.sqrt(lam.abs()) * CM1_PER_SQRT_LAMBDA


def masses_of(z: torch.Tensor) -> torch.Tensor:
    """Standard atomic weights (u, float64) from `ATOMIC_MASSES`; ValueError for an element outside the table."""
    zs = [int(a) for a in z.cpu().tolist()]
    missing = sorted(set(zs) - set(ATOMIC_MASSES))
    if missing:
        raise ValueError(f"no standard atomic weight for Z = {missing}; pass masses=")
    return torch.tensor([ATOMIC_MASSES[a] for a in zs], dtype=torch.float64)


def _rigid_basis(pos: torch.Tensor, m: torch.Tensor) -> torch.Tensor:
    """Orthonormal basis [3n, r] of the mass-weighted translations and rotations (r = 6, 5 for a linear molecule, 3 for one atom)."""
    sm = m.sqrt()
    x = pos - (m[:, None] * pos).sum(0) / m.sum()
    n = pos.shape[0]
    vecs = []
    for c in range(3):
        t = torch.zeros(n, 3, dtype=torch.float64, device=pos.device)
        t[:, c] = sm
        vecs.append(t.reshape(-1))
    for c in range(3):
        e = torch.zeros(3, dtype=torch.float64, device=pos.device)
        e[c] = 1.0
        vecs.append((sm[:, None] * torch.linalg.cross(e.expand(n, 3), x)).reshape(-1))
    u, s, _ = torch.linalg.svd(torch.stack(vecs, 1), full_matrices=False)
    return u[:, s > 1e-6 * s.max()]


def normal_modes_from_hessian(h: torch.Tensor, masses: torch.Tensor, positions: Optional[torch.Tensor] = None,
                              project: bool = False) -> NormalModes:
    """Diagonalise the mass-weighted Hessian in float64.  h [3n, 3n] in Ha/A^2, masses [n] in u.  project=True (needs `positions` [n, 3], A)
    removes the rigid-body translations and rotations first; they then come out as exact zeros."""
    h = h.to(torch.float64)
    inv = masses.to(device=h.device, dtype=torch.float64).repeat_interleave(3).rsqrt()
    d = h * inv[:, None] * inv[None, :]
    if project:
        if positions is None:
            raise ValueError("project=True needs the positions")
        q = _rigid_basis(positions.to(device=h.device, dtype=torch.float64), masses.to(device=h.device, dtype=torch.float64))
        p = torch.eye(d.shape[0], dtype=torch.float64, device=h.device) - q @ q.t()
        d = p @ d @ p
    d = 0.5 * (d + d.t())
    lam, modes = torch.linalg.eigh(d)
    nu = wavenumbers_from_eigenvalues(lam)
    return NormalModes(lam, modes, nu, nu * MEV_PER_CM1)


def normal_modes(model, batch, masses: Optional[torch.Tensor] = None, project: bool = False,
                 max_dir: Optional[int] = None) -> List[NormalModes]:
    """Normal modes of every molecule of the batch from its exact Hessian.  `masses` [N] in u (default: `ATOMIC_MASSES` by element).
    As ASE `Vibrations`, no rigid-body projection by default: the six (five) translations and rotations show up as small, possibly
    imaginary, modes.  project=True removes them."""
    _, z, pos, mol_ptr, _ = _engine_inputs(model, batch)
    hs = hessians(model, batch, max_dir)
    m_all = masses_of(z) if masses is None else masses.detach().to(torch.float64).cpu()
    ptr = mol_ptr.cpu().tolist()
    out = []
    for i, h in enumerate(hs):
        a, b = ptr[i], ptr[i + 1]
        out.append(normal_modes_from_hessian(h, m_all[a:b].to(h.device), pos[a:b], project))
    return out


def summary(modes: NormalModes) -> str:
    """The table ASE `Vibrations.summary` prints (meV and cm^-1, imaginary values with an i)."""
    lines = ["---------------------", "  #    meV     cm^-1", "---------------------"]
    for i, (e, nu) in enumerate(zip(modes.energies_meV.tolist(), modes.wavenumbers.tolist())):
        tag = "i" if nu < 0 else " "
        lines.append(f"{i:3d} {abs(e):6.1f}{tag} {abs(nu):7.1f}{tag}")
    lines.append("---------------------")
    return "\n".join(lines)
