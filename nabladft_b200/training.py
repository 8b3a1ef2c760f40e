"""Training through the CUDA engine: autograd bridge for energy losses (SURVEY.md section 8 a10/a11, BASELINE configs[2]).

The reference trains by `loss.backward()` through the eager graph (painn_pyg/painn.py:642-653; schnetpack AtomisticTask via
ase_model/task.py).  Here the model's `forward` in training mode returns `energy` attached to ONE autograd node
(`PainnEnergyFn`): its backward hands dLoss/dE_m to `nb200_painn_energy_forces_grads`, which returns the gradient w.r.t. the
canonical weight tensors; autograd then carries it through the (differentiable) export permutations back to the module's
reference-named parameters, so `torch.optim.*`, Lightning's optimiser loop and DDP's gradient all-reduce work unchanged.

Built, both exact (analytic; 1e-6 .. 2e-5 of each tensor's largest entry against the fp64 oracle's autograd / double backward):
  * energy term: d/dtheta sum_m c_m E_m with c = dLoss/dE -- the engine's backward holds dE/d(activation); weight gradients are the
    seed-scaled sums over atoms / edges (painn_train.cu);
  * force term (the reference's create_graph=True double backward): with v = dLoss/dF,
        d/dtheta sum_i v_i . F_i = - (v . d/dR) [ dE_tot/dtheta ]          (mixed partials commute)
    i.e. the directional derivative, along v in POSITION space, of the first-order gradient.  The weights carry no tangent, so the
    engine propagates tangents of every activation and of every backward quantity (forward-over-reverse): each Linear layer is the
    same GEMM applied to the tangent array, the pointwise / gather steps use the product rule (painn_tangent.cu), and every weight
    gradient gets  -(g^T x + g x^T)  added.  One engine call produces both terms.
A central finite difference of the energy gradient was tried first and rejected (10-80 % error in fp32, tools/debug_train_fd.py).
"""
from typing import Dict, List

import torch

from .engine import PainnEngine


class PainnEnergyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine: PainnEngine, scalars: Dict, z, pos, mol_ptr, n_mol: int, names: List[str], *canon):
        tensors = {n: t.detach().contiguous() for n, t in zip(names, canon)}
        engine._wkey = None  # weights change every optimiser step: always re-bind
        wkey = object()
        engine.set_weights(wkey, tensors, scalars)
        # training-mode forward: its activations stay in the engine's workspace for the backward call (no forward recompute); no host sync
        # after the first (capacity-sizing) batch, status check deferred.
        energy, forces, ctx.token = engine.run_train_forward(z, pos, mol_ptr, n_mol)
        ctx.wkey = wkey
        ctx.engine, ctx.names, ctx.n_mol = engine, names, n_mol
        ctx.tensors, ctx.scalars = tensors, scalars
        ctx.save_for_backward(z, pos, mol_ptr)
        ctx.set_materialize_grads(False)
        return energy, forces

    @staticmethod
    def backward(ctx, g_energy, g_forces):
        z, pos, mol_ptr = ctx.saved_tensors
        n_fixed = 7
        if g_energy is None and g_forces is None:
            return (None,) * (n_fixed + len(ctx.names))
        eng = ctx.engine
        seed = g_energy.to(torch.float32).contiguous() if g_energy is not None else torch.zeros(ctx.n_mol, dtype=torch.float32, device=z.device)
        fseed = g_forces.to(torch.float32).contiguous() if g_forces is not None else None
        if eng.kept(ctx.token) and eng._wkey is ctx.wkey:  # the workspace still holds this forward: gradients from the kept activations
            grads = eng.run_train_backward(ctx.token, z, mol_ptr, seed, fseed)
        else:  # another forward ran on this engine since: one call that recomputes the forward
            eng._wkey = None
            eng.set_weights(object(), ctx.tensors, ctx.scalars)
            _, _, grads = eng.run_train(z, pos, mol_ptr, ctx.n_mol, seed, fseed)
        return (None,) * n_fixed + tuple(grads.get(n) for n in ctx.names)


def energy_forces_training(engine: PainnEngine, tensors: Dict[str, torch.Tensor], scalars: Dict, z, pos, mol_ptr, n_mol: int):
    names = list(tensors)
    return PainnEnergyFn.apply(engine, scalars, z, pos, mol_ptr, n_mol, names, *[tensors[n] for n in names])
