"""SchNet training on energy and force losses through the CUDA engine (config/model/schnet.yaml; BASELINE configs[0]; SURVEY.md section 8 a8 /
a10 / a11).

The reference trains schnetpack's SchNet by `loss.backward()` through the eager graph (nablaDFT/ase_model/task.py, config/model/schnet.yaml).
Here `spk.NeuralNetworkPotential(SchNet)` in training mode returns `energy` (and `forces`) attached to ONE autograd node (`SchnetEnergyFn`): its
backward hands dLoss/dE_m and dLoss/dF_i to `nb200_schnet_energy_grads` (csrc/schnet_train.cu), which re-runs the forward with saved
activations and returns the gradient w.r.t. the canonical weight tensors; autograd carries it through the differentiable export
(`spk._export_schnet_impl(detach=False)`) back to the schnetpack-named parameters, so torch.optim / Lightning / DDP work unchanged.

Both terms are exact: the energy term is a reverse sweep seeded with dLoss/dE; the force term (the reference's create_graph double backward)
is the tangent pass of DESIGN.md 3.7: sum_i v_i . dF_i/dtheta = -(v . d/dR)[dE_tot/dtheta] with v = dLoss/dF.  The force VALUES come from the
inference engine (csrc/schnet.cu).
STATUS (round 1): first correct path, verified against the oracle's autograd under host emulation (tests/test_schnet_train_emu.py); not yet run
on a device.  No CPU fallback: the product entry (`spk.NeuralNetworkPotential.forward`) accepts CUDA tensors only.
"""
from ctypes import byref, c_int64
from typing import Dict, List, Optional

import torch

from ._lib import EngineDriver, NablaB200Error, SchnetWeights, check

GRAD_KEYS = ("emb", "w_f1", "b_f1", "W_f2", "b_f2", "I1", "P1", "p1", "P2", "p2", "R1", "e1", "R2", "e2")
SCALAR_KEYS = ("n_layers", "n_feat", "n_rbf", "n_elem", "z_offset", "cutoff", "rbf_coeff", "energy_shift_per_atom")


def count_edges(driver: EngineDriver, w: SchnetWeights, pos, mol_ptr, n_mol: int, ws_fn: str, *ws_args):
    """The exact-count step of the SchNet training and Hessian calls: `nb200_schnet_train_count` (one host sync) builds the CSR row pointer
    of the batch's graph in the driver's count buffer and returns its edge count, which sizes the workspace `ws_fn(w, n_mol, n_atoms, n_edges,
    *ws_args)`.  -> (row_ptr, n_edges, workspace)."""
    n, dev = int(pos.shape[0]), pos.device
    off = (4 * (n + 1) + 255) // 256 * 256  # row_ptr [N + 1] int32, then scratch [2 N] int32 on its own 256-byte boundary
    buf = driver._buffer("_count_buf", off + 8 * n, dev)
    row_ptr, scratch = buf[:4 * (n + 1)].view(torch.int32), buf[off:off + 8 * n].view(torch.int32)
    n_edges = c_int64(0)
    check(driver.lib.nb200_schnet_train_count(byref(w), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, row_ptr.data_ptr(), scratch.data_ptr(),
                                              byref(n_edges), driver._stream()), "nb200_schnet_train_count")
    driver.last_edges = int(n_edges.value)
    ws = driver._buffer("_ws", driver._bytes(ws_fn, byref(w), n_mol, n, n_edges.value, *ws_args), dev)
    return row_ptr, n_edges.value, ws


class SchnetTrainRunner(EngineDriver):
    """Host driver of `nb200_schnet_train_count` / `_workspace_bytes` / `nb200_schnet_energy_grads`."""

    @staticmethod
    def _struct(tensors: Dict[str, torch.Tensor], scalars: Dict) -> SchnetWeights:
        w = SchnetWeights()
        for k in SCALAR_KEYS:
            setattr(w, k, scalars[k])
        for k in GRAD_KEYS + ("rbf_offsets",):
            t = tensors[k]
            if not (t.dtype == torch.float32 and t.is_contiguous()):
                raise NablaB200Error(f"weight {k}: need a contiguous fp32 tensor")
            setattr(w, k, t.data_ptr())
        return w

    def energy_grads(self, tensors: Dict[str, torch.Tensor], scalars: Dict, z, pos, mol_ptr, n_mol: int, seed: Optional[torch.Tensor] = None,
                     force_seed: Optional[torch.Tensor] = None):
        """-> (energy [B], grads or None).  grads: dict of fresh tensors shaped like the canonical weights,
        d(sum_m seed_m E_m + sum_i force_seed_i . F_i)/d(weight)."""
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        self._check_seeds(seed, force_seed, n_mol, n, dev)
        w = self._struct(tensors, scalars)
        row_ptr, n_edges, ws = count_edges(self, w, pos, mol_ptr, n_mol, "nb200_schnet_train_workspace_bytes", int(force_seed is not None))
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        grads = gw = None
        if seed is not None or force_seed is not None:
            grads = {k: torch.empty_like(tensors[k]) for k in GRAD_KEYS}
            gw = self._struct({**grads, "rbf_offsets": tensors["rbf_offsets"]}, scalars)
        check(lib.nb200_schnet_energy_grads(self._h, byref(w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, row_ptr.data_ptr(), n_edges,
                                            ws.data_ptr(), ws.numel(), seed.data_ptr() if seed is not None else None,
                                            force_seed.data_ptr() if force_seed is not None else None, byref(gw) if gw is not None else None,
                                            energy.data_ptr(), self._stream()), "nb200_schnet_energy_grads")
        return energy, grads


class SchnetEnergyFn(torch.autograd.Function):
    """(energy, forces) = f(canonical weights).  `forces_value` (or None) are the force values from the inference engine; they leave the node as
    a differentiable output so that dLoss/dF reaches backward()."""

    @staticmethod
    def forward(ctx, runner: SchnetTrainRunner, scalars: Dict, z, pos, mol_ptr, n_mol: int, names: List[str], forces_value, *canon):
        tensors = {n: t.detach().contiguous() for n, t in zip(names, canon)}
        energy, _ = runner.energy_grads(tensors, scalars, z, pos, mol_ptr, n_mol, None, None)
        ctx.runner, ctx.names, ctx.n_mol, ctx.tensors, ctx.scalars = runner, names, n_mol, tensors, scalars
        ctx.save_for_backward(z, pos, mol_ptr)
        ctx.set_materialize_grads(False)
        if forces_value is None:
            ctx.mark_non_differentiable(empty := pos.new_zeros(0))
            return energy, empty
        return energy, forces_value.clone()

    @staticmethod
    def backward(ctx, g_energy, g_forces):
        z, pos, mol_ptr = ctx.saved_tensors
        n_fixed = 8
        if g_energy is None and g_forces is None:
            return (None,) * (n_fixed + len(ctx.names))
        seed = g_energy.to(torch.float32).contiguous() if g_energy is not None else None
        fseed = g_forces.to(torch.float32).contiguous() if g_forces is not None else None
        _, grads = ctx.runner.energy_grads(ctx.tensors, ctx.scalars, z, pos, mol_ptr, ctx.n_mol, seed, fseed)
        return (None,) * n_fixed + tuple(grads.get(n) for n in ctx.names)


def schnet_energy_training(runner: SchnetTrainRunner, tensors: Dict[str, torch.Tensor], scalars: Dict, z, pos, mol_ptr, n_mol: int, forces_value=None):
    """-> (energy, forces or None), both attached to the autograd graph of the canonical tensors."""
    names = list(tensors)
    energy, forces = SchnetEnergyFn.apply(runner, scalars, z, pos, mol_ptr, n_mol, names, forces_value, *[tensors[n] for n in names])
    return energy, (forces if forces_value is not None else None)
