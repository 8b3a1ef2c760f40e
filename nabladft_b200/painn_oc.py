"""H100-native drop-in for `nablaDFT.painn_pyg.PaiNN` (config/model/painn-oc.yaml).

Same constructor signature, same `forward(data) -> (energy, forces)` contract and the same
state_dict names/shapes as the reference class (`nablaDFT/painn_pyg/painn.py:22-148`,
SURVEY.md section 8b), so `config/model/painn-oc.yaml` works with
`_target_: nabladft_b200.painn_oc.PaiNN` and reference checkpoints load with strict=True.
The arithmetic runs in `libnabla_b200.so` (hand-written sm_90a kernels + cuBLAS SGEMM).

Inference: energy + autograd-free analytic forces.  Training mode returns (energy, forces) on one autograd node
(`training.PainnEnergyFn`): analytic parameter gradients, the `create_graph=True` force term (painn.py:142) as an exact tangent pass.
"""
import os
import math
from typing import Dict, Union

import torch
from torch import nn

from ._lib import RADIAL_OC, NablaB200Error
from .engine import PainnEngine, mol_ptr_from_batch


class _GaussianSmearing(nn.Module):
    def __init__(self, start=0.0, stop=1.0, num_gaussians=100):
        super().__init__()
        offset = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
        self.register_buffer("offset", offset)


class _RadialBasis(nn.Module):
    def __init__(self, num_radial, cutoff):
        super().__init__()
        self.inv_cutoff = 1 / cutoff
        self.rbf = _GaussianSmearing(0.0, 1.0, num_radial)


class _AtomEmbedding(nn.Module):
    def __init__(self, emb_size, num_elements):
        super().__init__()
        self.embeddings = nn.Embedding(num_elements, emb_size)
        nn.init.uniform_(self.embeddings.weight, a=-math.sqrt(3), b=math.sqrt(3))  # layers.py:213


def _xavier(lin):
    nn.init.xavier_uniform_(lin.weight)
    if lin.bias is not None:
        lin.bias.data.fill_(0)
    return lin


class _Message(nn.Module):  # parameter holder with the names of painn.py:459-464
    def __init__(self, h, num_rbf):
        super().__init__()
        self.x_proj = nn.Sequential(_xavier(nn.Linear(h, h)), nn.SiLU(), _xavier(nn.Linear(h, 3 * h)))
        self.rbf_proj = _xavier(nn.Linear(num_rbf, 3 * h))


class _Update(nn.Module):  # painn.py:520-525
    def __init__(self, h):
        super().__init__()
        self.vec_proj = _xavier(nn.Linear(h, 2 * h, bias=False))
        self.xvec_proj = nn.Sequential(_xavier(nn.Linear(2 * h, h)), nn.SiLU(), _xavier(nn.Linear(h, 3 * h)))


def _swap12(t: torch.Tensor, h: int) -> torch.Tensor:
    """swap chunks 1 and 2 of the leading 3h dimension."""
    return torch.cat([t[:h], t[2 * h:3 * h], t[h:2 * h]], dim=0)


class PaiNN(nn.Module):
    def __init__(
        self,
        hidden_channels: int = 512,
        num_layers: int = 6,
        num_rbf: int = 128,
        cutoff: float = 12.0,
        max_neighbors: int = 50,
        rbf: Dict[str, str] = {"name": "gaussian"},
        envelope: Dict[str, Union[str, int]] = {"name": "polynomial", "exponent": 5},
        regress_forces: bool = True,
        direct_forces: bool = True,
        use_pbc: bool = True,
        otf_graph: bool = True,
        num_elements: int = 83,
    ) -> None:
        super().__init__()
        if hidden_channels != 128:
            raise NotImplementedError("nabladft_b200 kernels are compiled for hidden_channels=128 (config/model/painn-oc.yaml)")
        if rbf.get("name", "").lower() != "gaussian" or envelope.get("name", "").lower() != "polynomial" or int(envelope.get("exponent", 5)) != 5:
            raise NotImplementedError("only rbf=gaussian, envelope=polynomial(5) (config/model/painn-oc.yaml)")
        if direct_forces and regress_forces:
            raise NotImplementedError("direct_forces head (PaiNNOutput) is unused by the shipped config and not built")
        if use_pbc or not otf_graph:
            raise NotImplementedError("molecules only: use_pbc=False, otf_graph=True (config/model/painn-oc.yaml)")
        self.hidden_channels, self.num_layers, self.num_rbf = hidden_channels, num_layers, num_rbf
        self.cutoff, self.max_neighbors = cutoff, max_neighbors
        self.regress_forces, self.direct_forces, self.otf_graph, self.use_pbc = regress_forces, direct_forces, otf_graph, use_pbc
        self.atom_emb = _AtomEmbedding(hidden_channels, num_elements)
        self.radial_basis = _RadialBasis(num_rbf, cutoff)
        self.message_layers = nn.ModuleList(_Message(hidden_channels, num_rbf) for _ in range(num_layers))
        self.update_layers = nn.ModuleList(_Update(hidden_channels) for _ in range(num_layers))
        self.out_energy = nn.Sequential(
            _xavier(nn.Linear(hidden_channels, hidden_channels // 2)), nn.SiLU(), _xavier(nn.Linear(hidden_channels // 2, 1)))
        self._engine = None
        self._train_engine = None
        # storage of the per-edge arrays in TRAINING mode: "f32" (reference precision) or "bf16" (BASELINE configs[2]; NB200_TRAIN_STORAGE sets the default)
        self.train_edge_storage = os.environ.get("NB200_TRAIN_STORAGE", "f32")

    # -------------------------------------------------------------- canonical export
    def _weights_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters()) + (str(next(self.parameters()).device),)

    @torch.no_grad()
    def _export(self):
        return self._export_impl(detach=True)

    def _export_impl(self, detach: bool):
        """detach=False keeps the autograd graph from the reference-named parameters to the canonical tensors (training.py)."""
        h, f32 = self.hidden_channels, torch.float32
        half = lambda t: torch.cat([t[h:2 * h], t[:h]], dim=0)  # canonical: normed half first, gated half second
        c = lambda t: (t.detach() if detach else t).to(f32).contiguous()
        stack = lambda ts: c(torch.stack(list(ts)))
        M, U = self.message_layers, self.update_layers
        tensors = {
            "emb": c(self.atom_emb.embeddings.weight),
            # Linear weight [3h, K] -> chunk roles (S, V, D) -> canonical (S, D, V) -> K-major [K, 3h]
            "w_rbf": stack(_swap12(m.rbf_proj.weight, h).t() for m in M),
            "b_rbf": stack(_swap12(m.rbf_proj.bias, h) for m in M),
            "A1": stack(m.x_proj[0].weight for m in M), "c1": stack(m.x_proj[0].bias for m in M),
            "A2": stack(_swap12(m.x_proj[2].weight, h) for m in M), "c2": stack(_swap12(m.x_proj[2].bias, h) for m in M),
            "U": stack(half(u.vec_proj.weight) for u in U),
            "B1": stack(u.xvec_proj[0].weight for u in U), "d1": stack(u.xvec_proj[0].bias for u in U),
            "B2": stack(_swap12(u.xvec_proj[2].weight, h) for u in U), "d2": stack(_swap12(u.xvec_proj[2].bias, h) for u in U),
            "R1": c(self.out_energy[0].weight), "e1": c(self.out_energy[0].bias),
            "R2": c(self.out_energy[2].weight), "e2": c(self.out_energy[2].bias),
            "rbf_offsets": c(self.radial_basis.rbf.offset),
        }
        scalars = dict(
            n_layers=self.num_layers, n_feat=h, n_rbf=self.num_rbf, n_elem=self.atom_emb.embeddings.num_embeddings,
            radial_mode=RADIAL_OC, z_offset=1, cutoff=float(self.cutoff), epsilon=1e-8,
            rbf_coeff=float(self.radial_basis.rbf.coeff), rbf_xscale=float(self.radial_basis.inv_cutoff),
            energy_shift_per_atom=0.0, max_neighbors=int(self.max_neighbors),
        )
        return tensors, scalars

    def engine(self) -> PainnEngine:
        if self._engine is None:
            self._engine = PainnEngine()
        key = self._weights_key()
        if key != self._engine._wkey:
            self._engine.set_weights(key, *self._export())
        return self._engine

    # -------------------------------------------------------------- forward
    def forward(self, data):
        """`data` exposes .z [N], .pos [N,3], .batch [N] (sorted) and optionally .ptr / .num_graphs,
        as a PyG Batch does (painn.py:90-104). Returns (energy [B], forces [N,3]) or energy."""
        pos, z = data.pos, data.z
        if not pos.is_cuda:
            raise NablaB200Error("nabladft_b200.PaiNN runs on CUDA only (no CPU fallback)")
        ptr_attr = getattr(data, "ptr", None)
        if ptr_attr is not None:
            mol_ptr, n_mol = ptr_attr.to(torch.int32), ptr_attr.numel() - 1
        else:
            mol_ptr, n_mol = mol_ptr_from_batch(data.batch, getattr(data, "num_graphs", None))
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # energy and force losses train through the engine (training.py: analytic gradients, tangent pass for the force term)
            from .training import energy_forces_training

            if not self.regress_forces:
                raise NotImplementedError("training needs regress_forces=True (the engine's backward produces the forces anyway)")
            if self._train_engine is None:
                self._train_engine = PainnEngine()
            if self._train_engine.edge_storage != self.train_edge_storage:
                self._train_engine.set_edge_storage(self.train_edge_storage)
            tensors, scalars = self._export_impl(detach=False)
            return energy_forces_training(self._train_engine, tensors, scalars, z.to(torch.int32).contiguous(),
                                          pos.detach().to(torch.float32).contiguous(), mol_ptr.contiguous(), n_mol)
        # inference: enqueue and return (no host synchronisation; the status check is deferred to the next call / `check()`)
        energy, forces = self.engine().run_async(
            z.to(torch.int32).contiguous(), pos.detach().to(torch.float32).contiguous(), mol_ptr.contiguous(), n_mol,
            with_forces=self.regress_forces)
        return (energy, forces) if self.regress_forces else energy

    def check(self) -> None:
        """Raise errors of earlier asynchronous forward() calls now (synchronises with their completion)."""
        if self._engine is not None:
            self._engine.check_pending(wait=True)

    @property
    def num_params(self) -> int:
        return sum(p.numel() for p in self.parameters())
