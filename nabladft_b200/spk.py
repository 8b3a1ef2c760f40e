"""H100-native drop-ins for the schnetpack classes named by config/model/{painn,schnet}.yaml.

The reference instantiates (Hydra `_target_`, config/model/painn.yaml:5-28)

    schnetpack.model.NeuralNetworkPotential(
        representation=schnetpack.representation.PaiNN(n_atom_basis=128, n_interactions=6,
            radial_basis=schnetpack.nn.radial.GaussianRBF(n_rbf=100, cutoff=5.0),
            cutoff_fn=schnetpack.nn.cutoff.CosineCutoff(cutoff=5.0)),
        input_modules=[schnetpack.atomistic.PairwiseDistances()],
        output_modules=[schnetpack.atomistic.Atomwise(n_in=128, output_key="energy"),
                        schnetpack.atomistic.Forces()],
        postprocessors=[schnetpack.transform.AddOffsets(property="energy", add_mean=True)],
        do_postprocessing=True)

Swapping the `schnetpack.` prefixes for `nabladft_b200.spk.` (config/model/painn-b200.yaml)
gives a module with the same constructor arguments, the same `forward(inputs) -> {"energy",
"forces"}` contract on spk batch dicts (keys `_atomic_numbers, _positions, _idx_m, _n_atoms`;
SURVEY.md section 8b) and the same state_dict names, whose arithmetic runs in
libnabla_b200.so.  The neighbour list is rebuilt on the device (same semantics as
ASENeighborList(5 A) for molecules), so `_idx_i/_idx_j/_offsets` in the batch are not read.
"""
from typing import Dict, List, Optional

import os
import torch
from torch import nn

from ._lib import RADIAL_SPK, NablaB200Error
from .engine import PainnEngine, mol_ptr_from_batch, refuse_training

INT32_MAX = 2**31 - 1


# ------------------------------------------------------------------ configuration holders
class GaussianRBF(nn.Module):
    """schnetpack.nn.radial.GaussianRBF(n_rbf, cutoff, start=0.0): buffers `offsets`, `widths`."""

    def __init__(self, n_rbf: int, cutoff: float, start: float = 0.0, trainable: bool = False):
        super().__init__()
        if trainable:
            raise NotImplementedError("trainable RBF")
        self.n_rbf, self.cutoff = n_rbf, cutoff
        offsets = torch.linspace(start, cutoff, n_rbf)
        self.register_buffer("offsets", offsets)
        self.register_buffer("widths", torch.abs(offsets[1] - offsets[0]) * torch.ones_like(offsets))


class CosineCutoff(nn.Module):
    def __init__(self, cutoff: float):
        super().__init__()
        self.register_buffer("cutoff", torch.tensor([cutoff], dtype=torch.float32))


class PairwiseDistances(nn.Module):
    """Marker: Rij = R[idx_j] - R[idx_i] is computed inside the neighbour kernel."""


class Forces(nn.Module):
    def __init__(self, calc_forces: bool = True, calc_stress: bool = False, energy_key: str = "energy", force_key: str = "forces"):
        super().__init__()
        if calc_stress:
            raise NotImplementedError("stress")
        self.calc_forces, self.energy_key, self.force_key = calc_forces, energy_key, force_key


class AddOffsets(nn.Module):
    """schnetpack.transform.AddOffsets(property, add_mean=True): eval-time E += mean * n_atoms."""

    def __init__(self, property: str = "energy", add_mean: bool = False, add_atomrefs: bool = False, is_extensive: bool = True):
        super().__init__()
        if add_atomrefs:
            raise NotImplementedError("atomrefs")
        self.property, self.add_mean = property, add_mean
        self.register_buffer("mean", torch.zeros(1))
        # schnetpack registers a persistent `atomref` buffer (zeros[zmax]) even when add_atomrefs=False, so reference checkpoints carry
        # `postprocessors.N.atomref`; a strict load needs the key (any length: `_load_from_state_dict` below adopts the stored shape)
        self.register_buffer("atomref", torch.zeros(100))

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        ref = state_dict.get(prefix + "atomref")
        if ref is not None:
            if bool((ref != 0).any()):
                raise NotImplementedError("AddOffsets: a checkpoint with non-zero atomrefs needs add_atomrefs, which this engine does not apply")
            if ref.shape != self.atomref.shape:
                self.atomref = torch.zeros_like(ref, device=self.atomref.device)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


def _banded_rbf_coeff(rep) -> float:
    """`rbf_coeff` of the representation's Gaussian basis.  The filter kernels evaluate only the 16 centres around bin floor(d / dx),
    dx = cutoff / (K - 1), so they need offsets[k] = k dx and widths equal to dx; a shifted basis (GaussianRBF(start != 0)) or another
    width, e.g. from a checkpoint's buffers, would silently lose most of the filter."""
    rbf, cutoff = rep.radial_basis, float(rep.cutoff_fn.cutoff.item())
    K = rbf.n_rbf
    dx = cutoff / (K - 1)
    offsets, widths = rbf.offsets.detach().double().cpu(), rbf.widths.detach().double().cpu()
    if (offsets - dx * torch.arange(K, dtype=torch.float64)).abs().max().item() > 1e-6 * cutoff:
        raise NotImplementedError("Gaussian RBF offsets other than k * cutoff / (n_rbf - 1) (a basis that starts at 0 and ends at the cutoff)")
    if (widths - dx).abs().max().item() > 1e-6 * dx:
        raise NotImplementedError("Gaussian RBF widths other than the centre spacing cutoff / (n_rbf - 1)")
    return float(-0.5 / widths[0].item() ** 2)


def _dense(n_in, n_out, bias=True):
    lin = nn.Linear(n_in, n_out, bias=bias)
    nn.init.xavier_uniform_(lin.weight)
    if bias:
        nn.init.zeros_(lin.bias)
    return lin


class Atomwise(nn.Module):
    """schnetpack.atomistic.Atomwise(n_in, output_key): outnet = Dense(n_in, n_in/2, silu), Dense(n_in/2, 1)."""

    def __init__(self, n_in: int, n_out: int = 1, output_key: str = "y", aggregation_mode: str = "sum"):
        super().__init__()
        if n_out != 1 or aggregation_mode != "sum":
            raise NotImplementedError("Atomwise: n_out=1, sum aggregation only")
        self.output_key = output_key
        self.outnet = nn.ModuleList([_dense(n_in, n_in // 2), _dense(n_in // 2, 1)])


class _Interaction(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.interatomic_context_net = nn.ModuleList([_dense(n, n), _dense(n, 3 * n)])


class _Mixing(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.intraatomic_context_net = nn.ModuleList([_dense(2 * n, n), _dense(n, 3 * n)])
        self.mu_channel_mix = _dense(n, 2 * n, bias=False)


class PaiNN(nn.Module):
    """schnetpack.representation.PaiNN parameter container (names of 2.0.4)."""

    def __init__(self, n_atom_basis: int, n_interactions: int, radial_basis: nn.Module, cutoff_fn: Optional[nn.Module] = None,
                 activation=None, max_z: int = 100, shared_interactions: bool = False, shared_filters: bool = False, epsilon: float = 1e-8):
        super().__init__()
        if n_atom_basis != 128:
            raise NotImplementedError("nabladft_b200 kernels are compiled for n_atom_basis=128 (config/model/painn.yaml)")
        if shared_interactions or shared_filters:
            raise NotImplementedError("shared interactions / filters")
        if not isinstance(cutoff_fn, CosineCutoff):
            raise NotImplementedError("cutoff_fn must be nabladft_b200.spk.CosineCutoff")
        self.n_atom_basis, self.n_interactions, self.epsilon = n_atom_basis, n_interactions, epsilon
        self.radial_basis, self.cutoff_fn = radial_basis, cutoff_fn
        self.cutoff = float(cutoff_fn.cutoff.item())
        self.embedding = nn.Embedding(max_z, n_atom_basis, padding_idx=0)
        self.filter_net = _dense(radial_basis.n_rbf, n_interactions * 3 * n_atom_basis)
        self.interactions = nn.ModuleList(_Interaction(n_atom_basis) for _ in range(n_interactions))
        self.mixing = nn.ModuleList(_Mixing(n_atom_basis) for _ in range(n_interactions))


class _SchNetInteraction(nn.Module):
    def __init__(self, n, n_rbf, n_filters):
        super().__init__()
        self.in2f = _dense(n, n_filters, bias=False)
        self.f2out = nn.ModuleList([_dense(n_filters, n), _dense(n, n)])
        self.filter_network = nn.ModuleList([_dense(n_rbf, n_filters), _dense(n_filters, n_filters)])


class SchNet(nn.Module):
    """schnetpack.representation.SchNet parameter container (names of 2.0.4)."""

    def __init__(self, n_atom_basis: int, n_interactions: int, radial_basis: nn.Module, cutoff_fn: nn.Module, n_filters: int = None,
                 shared_interactions: bool = False, max_z: int = 100, activation=None):
        super().__init__()
        n_filters = n_filters or n_atom_basis
        if n_atom_basis != 128 or n_filters != 128:
            raise NotImplementedError("nabladft_b200 kernels are compiled for n_atom_basis = n_filters = 128 (config/model/schnet.yaml)")
        if shared_interactions:
            raise NotImplementedError("shared interactions")
        if not isinstance(cutoff_fn, CosineCutoff):
            raise NotImplementedError("cutoff_fn must be nabladft_b200.spk.CosineCutoff")
        self.n_atom_basis, self.n_interactions = n_atom_basis, n_interactions
        self.radial_basis, self.cutoff_fn = radial_basis, cutoff_fn
        self.cutoff = float(cutoff_fn.cutoff.item())
        self.embedding = nn.Embedding(max_z, n_atom_basis, padding_idx=0)
        self.interactions = nn.ModuleList(_SchNetInteraction(n_atom_basis, radial_basis.n_rbf, n_filters) for _ in range(n_interactions))


class NeuralNetworkPotential(nn.Module):
    def __init__(self, representation: nn.Module, input_modules: Optional[List[nn.Module]] = None,
                 output_modules: Optional[List[nn.Module]] = None, postprocessors: Optional[List[nn.Module]] = None,
                 input_dtype_str: str = "float32", do_postprocessing: bool = True):
        super().__init__()
        if not isinstance(representation, (PaiNN, SchNet)):
            raise NotImplementedError("representation must be nabladft_b200.spk.PaiNN or nabladft_b200.spk.SchNet")
        self._kind = "painn" if isinstance(representation, PaiNN) else "schnet"
        self.representation = representation
        self.input_modules = nn.ModuleList(input_modules or [])
        self.output_modules = nn.ModuleList(output_modules or [])
        self.postprocessors = nn.ModuleList(postprocessors or [])
        self.do_postprocessing = do_postprocessing
        atomwise = [m for m in self.output_modules if isinstance(m, Atomwise)]
        if len(atomwise) != 1:
            raise NotImplementedError("exactly one Atomwise output module (config/model/painn.yaml:19-23)")
        self._atomwise = atomwise[0]
        self._forces = any(isinstance(m, Forces) and m.calc_forces for m in self.output_modules)
        self._engine = None
        self._train_engine = None
        # storage of the per-edge arrays in TRAINING mode: "f32" (reference precision) or "bf16" (BASELINE configs[2]; NB200_TRAIN_STORAGE sets the default)
        self.train_edge_storage = os.environ.get("NB200_TRAIN_STORAGE", "f32")
        self._schnet_runner = None

    def _weights_key(self, postprocess):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers())) + (postprocess,)

    @torch.no_grad()
    def _export(self, postprocess: bool):
        if self._kind == "schnet":
            return self._export_schnet(postprocess)
        return self._export_impl(postprocess, detach=True)

    def _export_impl(self, postprocess: bool, detach: bool):
        """detach=False keeps the autograd graph from the schnetpack-named parameters to the canonical tensors (training.py)."""
        rep, f32 = self.representation, torch.float32
        n, L, K = rep.n_atom_basis, rep.n_interactions, rep.radial_basis.n_rbf
        c = lambda t: (t.detach() if detach else t).to(f32).contiguous()
        stack = lambda ts: c(torch.stack(list(ts)))
        shift = 0.0
        if postprocess:
            for p in self.postprocessors:
                if isinstance(p, AddOffsets) and p.add_mean:
                    shift += float(p.mean.item())
        rbf_coeff = _banded_rbf_coeff(rep)
        tensors = {
            "emb": c(rep.embedding.weight),
            "w_rbf": c(rep.filter_net.weight.view(L, 3 * n, K).transpose(1, 2)),  # [L*3n, K] -> [L, K, 3n]
            "b_rbf": c(rep.filter_net.bias.view(L, 3 * n)),
            "A1": stack(i.interatomic_context_net[0].weight for i in rep.interactions),
            "c1": stack(i.interatomic_context_net[0].bias for i in rep.interactions),
            "A2": stack(i.interatomic_context_net[1].weight for i in rep.interactions),
            "c2": stack(i.interatomic_context_net[1].bias for i in rep.interactions),
            "U": stack(m.mu_channel_mix.weight for m in rep.mixing),
            "B1": stack(m.intraatomic_context_net[0].weight for m in rep.mixing),
            "d1": stack(m.intraatomic_context_net[0].bias for m in rep.mixing),
            "B2": stack(m.intraatomic_context_net[1].weight for m in rep.mixing),
            "d2": stack(m.intraatomic_context_net[1].bias for m in rep.mixing),
            "R1": c(self._atomwise.outnet[0].weight), "e1": c(self._atomwise.outnet[0].bias),
            "R2": c(self._atomwise.outnet[1].weight), "e2": c(self._atomwise.outnet[1].bias),
            "rbf_offsets": c(rep.radial_basis.offsets),
        }
        scalars = dict(
            n_layers=L, n_feat=n, n_rbf=K, n_elem=rep.embedding.num_embeddings, radial_mode=RADIAL_SPK, z_offset=0,
            cutoff=float(rep.cutoff_fn.cutoff.item()), epsilon=float(rep.epsilon), rbf_coeff=rbf_coeff, rbf_xscale=1.0,
            energy_shift_per_atom=shift, max_neighbors=INT32_MAX,
        )
        return tensors, scalars

    def _shift(self, postprocess: bool) -> float:
        shift = 0.0
        if postprocess:
            for p in self.postprocessors:
                if isinstance(p, AddOffsets) and p.add_mean:
                    shift += float(p.mean.item())
        return shift

    @torch.no_grad()
    def _export_schnet(self, postprocess: bool):
        return self._export_schnet_impl(postprocess, detach=True)

    def _export_schnet_impl(self, postprocess: bool, detach: bool):
        """detach=False keeps the autograd graph from the schnetpack-named parameters to the canonical tensors (schnet_train.py)."""
        rep, f32 = self.representation, torch.float32
        c = lambda t: (t.detach() if detach else t).to(f32).contiguous()
        stack = lambda ts: c(torch.stack(list(ts)))
        I = rep.interactions
        rbf_coeff = _banded_rbf_coeff(rep)
        tensors = {
            "emb": c(rep.embedding.weight),
            "w_f1": stack(i.filter_network[0].weight.t() for i in I),  # [F, K] -> K-major [K, F]
            "b_f1": stack(i.filter_network[0].bias for i in I),
            "W_f2": stack(i.filter_network[1].weight for i in I), "b_f2": stack(i.filter_network[1].bias for i in I),
            "I1": stack(i.in2f.weight for i in I),
            "P1": stack(i.f2out[0].weight for i in I), "p1": stack(i.f2out[0].bias for i in I),
            "P2": stack(i.f2out[1].weight for i in I), "p2": stack(i.f2out[1].bias for i in I),
            "R1": c(self._atomwise.outnet[0].weight), "e1": c(self._atomwise.outnet[0].bias),
            "R2": c(self._atomwise.outnet[1].weight), "e2": c(self._atomwise.outnet[1].bias),
            "rbf_offsets": c(rep.radial_basis.offsets),
        }
        scalars = dict(
            n_layers=rep.n_interactions, n_feat=rep.n_atom_basis, n_rbf=rep.radial_basis.n_rbf, n_elem=rep.embedding.num_embeddings,
            z_offset=0, cutoff=float(rep.cutoff_fn.cutoff.item()), rbf_coeff=rbf_coeff,
            energy_shift_per_atom=self._shift(postprocess),
        )
        return tensors, scalars

    def engine(self, postprocess: bool) -> PainnEngine:
        """Engine bound to the CURRENT CUDA stream (one cuBLAS handle + workspace per stream, shared weights),
        so that independent batches submitted from different streams overlap on the GPU."""
        if self._engine is None:
            self._engine = PainnEngine(self._kind)
            self._stream_engines = {}
        key = self._weights_key(postprocess)
        if key != self._engine._wkey:
            self._engine.set_weights(key, *self._export(postprocess))
            self._stream_engines = {}
        sid = torch.cuda.current_stream().cuda_stream
        if sid == torch.cuda.default_stream().cuda_stream:
            return self._engine
        if sid not in self._stream_engines:
            self._stream_engines[sid] = self._engine.clone_for_stream()
        return self._stream_engines[sid]

    def _prepare(self, inputs):
        z, pos, idx_m = inputs["_atomic_numbers"], inputs["_positions"], inputs["_idx_m"]
        if not pos.is_cuda:
            raise NablaB200Error("nabladft_b200.spk.NeuralNetworkPotential runs on CUDA only (no CPU fallback)")
        if "_pbc" in inputs and bool(inputs["_pbc"].any()):
            raise NotImplementedError("periodic systems")
        n_atoms = inputs.get("_n_atoms")
        if n_atoms is not None:
            n_mol = n_atoms.numel()
            mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32, device=pos.device)
            mol_ptr[1:] = torch.cumsum(n_atoms, 0)
        else:
            mol_ptr, n_mol = mol_ptr_from_batch(idx_m)
        # nablaDFT's test/predict steps call self(batch) => post-processing on (ase_model/task.py:43,63)
        post = self.do_postprocessing and not self.training
        return self.engine(post), z.to(torch.int32).contiguous(), pos.detach().to(torch.float32).contiguous(), mol_ptr, n_mol

    def engine_inputs(self, inputs: Dict[str, torch.Tensor]):
        """(engine, z int32, pos fp32, mol_ptr int32, n_mol) of `inputs` for the inference engine: the inputs of `PainnEngine.run_hvp`
        (`vibrations`)."""
        eng, z, pos, mol_ptr, n_mol = self._prepare(inputs)  # raises on CPU inputs and periodic systems
        refuse_training(self)
        return eng, z, pos, mol_ptr, n_mol

    def _pack(self, energy, forces):
        out = {self._atomwise.output_key: energy}
        if self._forces:
            out["forces"] = forces
        return out

    def _training_mode(self) -> bool:
        return self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())

    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        eng, z, pos, mol_ptr, n_mol = self._prepare(inputs)
        if self._training_mode():
            # energy and force losses train through the engines (training.py for PaiNN, schnet_train.py for SchNet)
            from .training import energy_forces_training

            if self._kind == "schnet":
                if self._schnet_runner is None:
                    from .schnet_train import SchnetTrainRunner

                    self._schnet_runner = SchnetTrainRunner()
                return self._train_schnet_with(self._schnet_runner, eng, z, pos, mol_ptr, n_mol)
            if not self._forces:
                raise NotImplementedError("training PaiNN through the CUDA path needs the Forces output module (config/model/painn.yaml)")
            if self._train_engine is None:
                self._train_engine = PainnEngine("painn")
            if self._train_engine.edge_storage != self.train_edge_storage:
                self._train_engine.set_edge_storage(self.train_edge_storage)
            tensors, scalars = self._export_impl(False, detach=False)
            energy, forces = energy_forces_training(self._train_engine, tensors, scalars, z, pos, mol_ptr, n_mol)
            return self._pack(energy, forces)
        # inference: enqueue and return (no host synchronisation; the status check is deferred to the next call / `check()`)
        energy, forces = eng.run_async(z, pos, mol_ptr, n_mol, with_forces=self._forces)
        return self._pack(energy, forces)

    def check(self) -> None:
        """Raise errors of earlier asynchronous forward() calls now (synchronises with their completion)."""
        for e in [self._engine] + list(getattr(self, "_stream_engines", {}).values()):
            if e is not None:
                e.check_pending(wait=True)

    def _train_schnet_with(self, runner, eng, z, pos, mol_ptr, n_mol):
        """SchNet in training mode: energy and forces attached to ONE autograd node over the parameters (schnet_train.py); the force VALUES
        come from the inference engine."""
        from .schnet_train import schnet_energy_training

        tensors, scalars = self._export_schnet_impl(False, detach=False)
        f = None
        if self._forces:
            with torch.no_grad():
                _, f, _ = eng.run(z, pos, mol_ptr, n_mol, with_forces=True)
        energy, forces = schnet_energy_training(runner, tensors, scalars, z, pos, mol_ptr, n_mol, f)
        return self._pack(energy, forces)

    def forward_async(self, inputs: Dict[str, torch.Tensor]):
        """Enqueue on the current CUDA stream without any host synchronisation.  Returns (outputs, status):
        `status` is the device int32[4] of nb200_neighbor_build; pass its host copy to
        `PainnEngine.raise_on_status` once the stream has been synchronised (a too-small edge capacity shows up
        there as NB200_ECAPACITY; `forward` handles that case by re-running)."""
        if self._training_mode():
            raise NotImplementedError("forward_async is an inference entry point; call forward() in training mode")
        eng, z, pos, mol_ptr, n_mol = self._prepare(inputs)
        energy, forces, status = eng.launch(z, pos, mol_ptr, n_mol, with_forces=self._forces)
        return self._pack(energy, forces), status
