"""H100-native drop-in for `nablaDFT.dimenetplusplus.DimeNetPlusPlusPotential` (config/model/dimenetplusplus.yaml).

Same constructor signature (nablaDFT/dimenetplusplus/dimenetplusplus.py:22-91), same `forward(data) -> (energy [B], forces [N, 3])` contract
(dimenetplusplus.py:93-113: forces are -d(unscaled prediction)/d pos, the scaler is applied to the energy only, after the gradient) and the
same state-dict names and shapes (`net.*` as torch_geometric's DimeNetPlusPlus, `regr_or_cls_nn.{0,2,4,6}`), so the yaml works with
`_target_: nabladft_b200.dimenetplusplus.DimeNetPlusPlusPotential` and reference checkpoints load with strict=True.  The arithmetic -- the
radius graph, the triplets, the bases, the embedding / interaction / output blocks, the regression head and the reverse pass for the forces --
runs in `libnabla_b200.so` (`csrc/dimenet.cu`, C ABI `nb200_dimenet_*` in include/nabla_b200.h).  This file owns the parameters and their
export into the flat buffer the C ABI takes (lin_rbf2 . lin_rbf1 and lin_sbf2 . lin_sbf1 folded, the embedding's atom thirds turned into
per-element tables).

Training: in training mode with autograd the forward goes through `DimeNetEnergyFn`, whose backward is `nb200_dimenet_train_grads` (the
parameter gradients of energy and force losses, the force term by forward-over-reverse, DESIGN.md 3.15.1); the export is then differentiable,
so autograd carries the flat-buffer gradient back to every reference-named parameter.  Hessians: `DimeNetRunner.run_hvp` (nb200_dimenet_hvp,
DESIGN.md 3.15.2) gives exact Hessian-vector products of the unscaled prediction; `vibrations.hessians` / `normal_modes` take this model.
Relaxation and molecular dynamics: `engine()` is the interface of `optimization.ASEBatchwiseLBFGS` and `md.BatchwiseMD`; its forward is the
asynchronous call, sized by per-batch upper bounds of the edge and triplet counts (DESIGN.md 3.15.3).  Supported: the shipped sizes, with
1 <= dimenet_num_blocks <= 16, 2 <= node_latent_dim <= 64 and dimenet_max_num_neighbors <= 64; anything else raises at construction.  No CPU
fallback: CPU tensors raise NablaB200Error in eval mode and NotImplementedError in training mode.
"""
import ctypes
from ctypes import POINTER, byref, c_int64
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import DimeNetWeights, EngineDriver, NablaB200Error, check
from .engine import BoundedEngine, refuse_training

# ---- canonical layout: keep in step with the enums of include/nabla_b200.h -----------------------------------------------------------------
G_NAMES = ["FREQ", "ZEROS", "NORMS", "EMB_TI", "EMB_TJ", "EMB_RBF_W", "EMB_RBF_B", "EMB_W3", "HEAD_W0", "HEAD_B0", "HEAD_W1", "HEAD_B1",
           "HEAD_W2", "HEAD_B2", "HEAD_W3", "HEAD_B3"]
I_NAMES = ["RBF", "SBF", "SBF1", "SBF2", "JI_W", "JI_B", "KJ_W", "KJ_B", "DOWN", "UP", "RES_W", "RES_B", "LIN_W", "LIN_B"]
O_NAMES = ["RBF", "UP", "LINS_W", "LINS_B", "LIN"]
N_COUNTS = 4
_FIXED = dict(dimenet_hidden_channels=256, dimenet_int_emb_size=64, dimenet_basis_emb_size=8, dimenet_out_emb_channels=256,
              dimenet_num_spherical=7, dimenet_num_radial=6, dimenet_envelope_exponent=5, dimenet_num_before_skip=1, dimenet_num_after_skip=2,
              dimenet_num_output_layers=3)


def bind(lib):
    """The DimeNet++ prototypes on `lib`, e.g. an emulation build of csrc/dimenet.cu, which exports no other engine."""
    return _lib.bind(lib, ["nb200_dimenet_"])


def sbf_radial_constants(num_spherical: int = 7, num_radial: int = 6) -> Tuple[np.ndarray, np.ndarray]:
    """(z_ln, N_ln) [num_spherical, num_radial]: the first zeros of the spherical Bessel functions j_l (those of j_l interlace those of
    j_{l-1}) and the normalisers 1 / sqrt(0.5 j_{l+1}(z_ln)^2) of PyG's SphericalBasisLayer."""
    from scipy.optimize import brentq
    from scipy.special import spherical_jn

    k = num_radial + num_spherical
    z = np.zeros((num_spherical, k))
    z[0] = np.pi * np.arange(1, k + 1)
    for l in range(1, num_spherical):
        for m in range(k - l):
            z[l, m] = brentq(lambda x, l=l: spherical_jn(l, x), z[l - 1, m], z[l - 1, m + 1], xtol=1e-15)
    z = z[:, :num_radial]
    norms = np.stack([np.sqrt(2.0) / np.abs(spherical_jn(l + 1, z[l])) for l in range(num_spherical)])
    return z, norms


# ---- parameter holders with torch_geometric's attribute names -----------------------------------------------------------------------------
class _Swish(nn.Module):
    def forward(self, x):
        return x * x.sigmoid()


class _Bessel(nn.Module):
    def __init__(self, num_radial):
        super().__init__()
        self.freq = nn.Parameter(torch.arange(1, num_radial + 1, dtype=torch.float32) * np.pi)


class _Embedding(nn.Module):
    def __init__(self, num_radial, hidden):
        super().__init__()
        self.emb = nn.Embedding(95, hidden)
        nn.init.uniform_(self.emb.weight, -3 ** 0.5, 3 ** 0.5)
        self.lin_rbf = nn.Linear(num_radial, hidden)
        self.lin = nn.Linear(3 * hidden, hidden)


class _Residual(nn.Module):
    def __init__(self, hidden):
        super().__init__()
        self.lin1 = nn.Linear(hidden, hidden)
        self.lin2 = nn.Linear(hidden, hidden)


class _Interaction(nn.Module):
    def __init__(self, hidden, int_emb, basis_emb, num_spherical, num_radial, num_before_skip, num_after_skip):
        super().__init__()
        self.lin_rbf1 = nn.Linear(num_radial, basis_emb, bias=False)
        self.lin_rbf2 = nn.Linear(basis_emb, hidden, bias=False)
        self.lin_sbf1 = nn.Linear(num_spherical * num_radial, basis_emb, bias=False)
        self.lin_sbf2 = nn.Linear(basis_emb, int_emb, bias=False)
        self.lin_kj = nn.Linear(hidden, hidden)
        self.lin_ji = nn.Linear(hidden, hidden)
        self.lin_down = nn.Linear(hidden, int_emb, bias=False)
        self.lin_up = nn.Linear(int_emb, hidden, bias=False)
        self.layers_before_skip = nn.ModuleList([_Residual(hidden) for _ in range(num_before_skip)])
        self.lin = nn.Linear(hidden, hidden)
        self.layers_after_skip = nn.ModuleList([_Residual(hidden) for _ in range(num_after_skip)])


class _Output(nn.Module):
    def __init__(self, num_radial, hidden, out_emb, out_channels, num_layers):
        super().__init__()
        self.lin_rbf = nn.Linear(num_radial, hidden, bias=False)
        self.lin_up = nn.Linear(hidden, out_emb, bias=False)
        self.lins = nn.ModuleList([nn.Linear(out_emb, out_emb) for _ in range(num_layers)])
        self.lin = nn.Linear(out_emb, out_channels, bias=False)
        nn.init.zeros_(self.lin.weight)  # PyG's output_initializer='zeros'


class _Core(nn.Module):
    def __init__(self, hidden, out_channels, num_blocks, int_emb, basis_emb, out_emb, num_spherical, num_radial, num_before_skip, num_after_skip,
                 num_output_layers):
        super().__init__()
        self.rbf = _Bessel(num_radial)
        self.emb = _Embedding(num_radial, hidden)
        self.output_blocks = nn.ModuleList([_Output(num_radial, hidden, out_emb, out_channels, num_output_layers) for _ in range(num_blocks + 1)])
        self.interaction_blocks = nn.ModuleList([_Interaction(hidden, int_emb, basis_emb, num_spherical, num_radial, num_before_skip, num_after_skip)
                                                 for _ in range(num_blocks)])


class DimeNetPlusPlusPotential(nn.Module):
    def __init__(self, node_latent_dim: int, scaler=None, dimenet_hidden_channels=128, dimenet_num_blocks=4, dimenet_int_emb_size=64,
                 dimenet_basis_emb_size=8, dimenet_out_emb_channels=256, dimenet_num_spherical=7, dimenet_num_radial=6, dimenet_max_num_neighbors=32,
                 dimenet_envelope_exponent=5, dimenet_num_before_skip=1, dimenet_num_after_skip=2, dimenet_num_output_layers=3, cutoff=5.0,
                 do_postprocessing=False):
        super().__init__()
        given = dict(locals())
        bad = [f"{k}={given[k]!r} (built: {v!r})" for k, v in _FIXED.items() if given[k] != v]
        if not 1 <= dimenet_num_blocks <= 16:
            bad.append(f"dimenet_num_blocks={dimenet_num_blocks} (built: 1..16)")
        if not 2 <= node_latent_dim <= 64:
            bad.append(f"node_latent_dim={node_latent_dim} (built: 2..64)")
        if not 1 <= dimenet_max_num_neighbors <= 64:
            bad.append(f"dimenet_max_num_neighbors={dimenet_max_num_neighbors} (built: 1..64)")
        if not cutoff > 0:
            bad.append(f"cutoff={cutoff}")
        if bad:
            raise NablaB200Error("DimeNetPlusPlusPotential: configuration outside the compiled path (config/model/dimenetplusplus.yaml): " + "; ".join(bad))
        self.scaler, self.do_postprocessing = scaler, do_postprocessing
        self.node_latent_dim, self.num_blocks = node_latent_dim, dimenet_num_blocks
        self.max_num_neighbors, self.cutoff = dimenet_max_num_neighbors, float(cutoff)
        self.net = _Core(dimenet_hidden_channels, node_latent_dim, dimenet_num_blocks, dimenet_int_emb_size, dimenet_basis_emb_size,
                         dimenet_out_emb_channels, dimenet_num_spherical, dimenet_num_radial, dimenet_num_before_skip, dimenet_num_after_skip,
                         dimenet_num_output_layers)
        L = node_latent_dim
        self.regr_or_cls_nn = nn.Sequential(nn.Linear(L, L), _Swish(), nn.Linear(L, L // 2), _Swish(), nn.Linear(L // 2, L // 2), _Swish(),
                                            nn.Linear(L // 2, 1))
        self._runner: Optional[DimeNetRunner] = None
        self._engine: Optional[DimeNetEngine] = None
        self._export_key = None

    # ---- export: reference-named tensors -> flat buffer (include/nabla_b200.h NB200_DPP_*) ---------------------------------------------------
    def export(self, device) -> Tuple[torch.Tensor, List[int]]:
        buf, offs = self._export_impl(detach=True)
        return buf.to(device), offs

    def _export_impl(self, detach: bool) -> Tuple[torch.Tensor, List[int]]:
        """The flat float32 buffer on the parameters' device, folds in float64.  detach=False keeps the graph, so a gradient w.r.t. the
        buffer (nb200_dimenet_train_grads) reaches every reference-named parameter, the folded lin_rbf1/2, lin_sbf1/2 and emb included."""
        f = (lambda t: t.detach().to(torch.float64)) if detach else (lambda t: t.to(torch.float64))
        net, H = self.net, 256
        dev = net.rbf.freq.device
        z, norms = sbf_radial_constants()
        W = f(net.emb.lin.weight)
        emb = f(net.emb.emb.weight)
        head = [f(t) for m in (0, 2, 4, 6) for t in (self.regr_or_cls_nn[m].weight, self.regr_or_cls_nn[m].bias)]
        entries: List = [f(net.rbf.freq), torch.from_numpy(z).reshape(-1).to(dev), torch.from_numpy(norms).reshape(-1).to(dev),
                         emb @ W[:, :H].t() + f(net.emb.lin.bias), emb @ W[:, H:2 * H].t(), f(net.emb.lin_rbf.weight), f(net.emb.lin_rbf.bias),
                         W[:, 2 * H:]] + head
        for b in net.interaction_blocks:
            res = list(b.layers_before_skip) + list(b.layers_after_skip)
            entries += [f(b.lin_rbf2.weight) @ f(b.lin_rbf1.weight), f(b.lin_sbf2.weight) @ f(b.lin_sbf1.weight), f(b.lin_sbf1.weight),
                        f(b.lin_sbf2.weight), f(b.lin_ji.weight), f(b.lin_ji.bias), f(b.lin_kj.weight), f(b.lin_kj.bias), f(b.lin_down.weight),
                        f(b.lin_up.weight), [f(getattr(r, n).weight) for r in res for n in ("lin1", "lin2")],
                        [f(getattr(r, n).bias) for r in res for n in ("lin1", "lin2")], f(b.lin.weight), f(b.lin.bias)]
        for o in net.output_blocks:
            entries += [f(o.lin_rbf.weight), f(o.lin_up.weight), [f(l.weight) for l in o.lins], [f(l.bias) for l in o.lins], f(o.lin.weight)]
        assert len(entries) == len(G_NAMES) + len(I_NAMES) * self.num_blocks + len(O_NAMES) * (self.num_blocks + 1)
        pieces, offs, pos = [], [], 0
        for ent in entries:
            start = (pos + 63) // 64 * 64  # 256-byte alignment of every matrix
            if start > pos:
                pieces.append(torch.zeros(start - pos, dtype=torch.float32, device=dev))
            offs.append(start)
            pos = start
            for t_ in (ent if isinstance(ent, list) else [ent]):
                pieces.append(t_.reshape(-1).to(torch.float32))
                pos += t_.numel()
        pieces.append(torch.zeros(64, dtype=torch.float32, device=dev))
        return torch.cat(pieces), offs

    def _scale_mean(self) -> Tuple[float, float]:
        if self.scaler and self.do_postprocessing:
            return float(self.scaler["scale_"]), float(self.scaler["mean_"])
        return 1.0, 0.0

    # ---- forward ------------------------------------------------------------------------------------------------------------------------------
    def forward(self, data):
        """data.z [N], data.pos [N,3], data.batch [N] (sorted) -> (energy [B], forces [N,3])   (dimenetplusplus.py:93-113).  In training mode
        with autograd the outputs are differentiable w.r.t. every parameter (DimeNetEnergyFn), forces included: what the reference gets from
        create_graph=True.  They are bitwise equal to the eval-mode outputs."""
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            if not data.pos.is_cuda:
                raise NotImplementedError("nabladft_b200 DimeNetPlusPlusPotential trains on CUDA tensors only (sm_90a engine; there is no CPU path)")
            runner = self._get_runner()
            flat, offs = self._export_impl(detach=False)
            self._export_key = None  # the runner now holds this step's buffer; the next eval call exports again
            z, pos, mol_ptr, n_mol = self.batch_args(data.z, data.pos, data.batch)
            return DimeNetEnergyFn.apply(flat, self, runner, offs, z, pos, mol_ptr, n_mol)
        energy, forces, _ = self.run(data.z, data.pos, data.batch)
        return energy, forces

    def run(self, z, pos, batch):
        """-> (energy [B], forces [N,3], graph embeddings [B, node_latent_dim])."""
        runner = self._cuda_runner(pos)
        self._sync_weights(runner, pos.device)
        return runner.run(*self.batch_args(z, pos, batch))

    def engine(self) -> "DimeNetEngine":
        """The engine interface of the batch-wise optimiser and MD loops (`optimization.ASEBatchwiseLBFGS`, `md.BatchwiseMD`)."""
        if self._engine is None:
            self._engine = DimeNetEngine(self, self._get_runner())
        return self._engine

    def engine_inputs(self, data):
        """(runner, z int32, pos fp32, mol_ptr int32, n_mol) of `data` for the inference engine, with the weights synced: the inputs of
        `DimeNetRunner.run_hvp` (`vibrations`)."""
        runner = self._cuda_runner(data.pos)
        refuse_training(self)
        self._sync_weights(runner, data.pos.device)
        return (runner, *self.batch_args(data.z, data.pos, data.batch))

    def _cuda_runner(self, pos) -> "DimeNetRunner":
        if not pos.is_cuda:
            raise NablaB200Error("DimeNetPlusPlusPotential runs on CUDA tensors only (sm_90a engine; there is no CPU path)")
        return self._get_runner()

    def _get_runner(self) -> "DimeNetRunner":
        if self._runner is None:
            self._runner = DimeNetRunner()
        return self._runner

    def _sync_weights(self, runner: "DimeNetRunner", device) -> None:
        key = (id(runner), str(device), self._scale_mean()) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if key != self._export_key:
            runner.set_weights(self, device)
            self._export_key = key

    @staticmethod
    def batch_args(z, pos, batch):
        if batch.numel() and bool((batch[1:] < batch[:-1]).any()):
            raise NablaB200Error("DimeNetPlusPlusPotential: `batch` must be sorted (atoms of a molecule contiguous), as PyG collation produces it")
        n_mol = int(batch[-1].item()) + 1 if batch.numel() else 0
        counts = torch.bincount(batch, minlength=n_mol)
        mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32, device=pos.device)
        mol_ptr[1:] = torch.cumsum(counts, 0)
        return z.to(torch.int32).contiguous(), pos.detach().to(torch.float32).contiguous(), mol_ptr, n_mol


class DimeNetRunner(EngineDriver):
    """Host driver of `nb200_dimenet_*`: owns the engine handle, the exported weights, the graph buffer and the workspace."""

    def __init__(self, lib=None):
        super().__init__(lib)
        self._w = None
        self._keep = None
        self._status = None
        self.last_counts: Dict[str, int] = {}
        self.last_workspace_bytes = 0

    def set_weights(self, model: DimeNetPlusPlusPotential, device):
        self.bind(model, *model.export(device))

    def bind(self, model: DimeNetPlusPlusPotential, buf: torch.Tensor, offs: List[int]):
        """Use `buf` (a flat float32 buffer in the layout of `model.export`, kept alive here) as the weights."""
        off_arr = (c_int64 * len(offs))(*offs)
        scale, mean = model._scale_mean()
        w = DimeNetWeights(model.num_blocks, model.node_latent_dim, 256, 64, 8, 256, 7, 6, 1, 2, 3, 5, model.max_num_neighbors, model.cutoff,
                           scale, mean, buf.data_ptr(), ctypes.cast(off_arr, POINTER(c_int64)))
        self._w, self._keep = w, (buf, off_arr)

    def run(self, z, pos, mol_ptr, n_mol: int):
        """Two-phase call: graph (one synchronisation for the counts), workspace, energies / forces / graph embeddings."""
        if self._w is None:
            raise NablaB200Error("DimeNetRunner.run before set_weights")
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        s = self._stream()
        gbuf, counts = self._graph(z, pos, mol_ptr, n_mol)
        ws = self._buffer("_ws", self._bytes("nb200_dimenet_workspace_bytes", byref(self._w), n_mol, n, counts), dev)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n, 3, dtype=torch.float32, device=dev)
        emb = torch.empty(n_mol, self._w.node_latent_dim, dtype=torch.float32, device=dev)
        check(lib.nb200_dimenet_energy_forces(self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, gbuf.data_ptr(),
                                              gbuf.numel(), counts, ws.data_ptr(), ws.numel(), energy.data_ptr(), forces.data_ptr(), emb.data_ptr(), s),
              "nb200_dimenet_energy_forces")
        return energy, forces, emb

    def _graph(self, z, pos, mol_ptr, n_mol: int):
        lib, n = self.lib, int(z.shape[0])
        if n == 0 or n_mol == 0:
            raise NablaB200Error("DimeNetPlusPlusPotential: empty batch")
        gbuf = self._buffer("_graph_buf", self._graph_bytes(n), pos.device)
        counts = (c_int64 * N_COUNTS)()
        check(lib.nb200_dimenet_graph_count(byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, gbuf.data_ptr(), gbuf.numel(),
                                            counts, self._stream()), "nb200_dimenet_graph_count")
        self.last_counts = {"edges": int(counts[0]), "triplets": int(counts[1])}
        return gbuf, counts

    def _graph_bytes(self, n: int) -> int:
        return self._bytes("nb200_dimenet_graph_bytes", byref(self._w), n)

    def count_bounds(self, sizes):
        """Upper bounds of {edges, triplet slots} for molecules of `sizes` atoms (host, nb200_dimenet_count_bounds): they hold for every
        geometry, see DESIGN.md 3.15.3."""
        return self._count_bounds("nb200_dimenet", sizes, N_COUNTS)

    def launch(self, z, pos, mol_ptr, n_mol: int, bounds):
        """Asynchronous forward (nb200_dimenet_energy_forces_async) sized by n_atoms and `bounds` (count_bounds): see
        `EngineDriver._launch_bounded`."""
        return self._launch_bounded("nb200_dimenet", z, pos, mol_ptr, n_mol, bounds)

    def train_grads(self, z, pos, mol_ptr, n_mol: int, seed_energy: Optional[torch.Tensor], seed_forces: Optional[torch.Tensor]) -> torch.Tensor:
        """d(sum_m seed_energy[m] E_m + sum_i seed_forces[i] . F_i)/d(flat weight buffer), in the buffer's layout (nb200_dimenet_train_grads).
        Either seed may be None.  Builds the graph again (one synchronisation for the counts), so it does not depend on an earlier call."""
        if self._w is None:
            raise NablaB200Error("DimeNetRunner.train_grads before set_weights / bind")
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        seeds = [None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous() for t in (seed_energy, seed_forces)]
        self._check_seeds(*seeds, n_mol, n, dev)
        gbuf, counts = self._graph(z, pos, mol_ptr, n_mol)
        ws = self._buffer("_ws", self._bytes("nb200_dimenet_train_workspace_bytes", byref(self._w), n_mol, n, counts), dev)
        grads = torch.zeros_like(self._keep[0])  # the call writes up to the end of the last entry
        ptr = [0 if t is None else t.data_ptr() for t in seeds]
        check(lib.nb200_dimenet_train_grads(self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, gbuf.data_ptr(),
                                            gbuf.numel(), counts, ws.data_ptr(), ws.numel(), ptr[0] or None, ptr[1] or None, grads.data_ptr(),
                                            self._stream()), "nb200_dimenet_train_grads")
        return grads

    def run_hvp(self, z, pos, mol_ptr, n_mol: int, v, with_forces: bool = True):
        """Exact Hessian-vector products (nb200_dimenet_hvp): v [n_dir, N, 3] (or [N, 3]) fp32 in Angstrom.  Returns (energy [B], forces [N, 3]
        or None, hv [n_dir, N, 3]) with hv = -(dF/dR) v in Ha/A -- the Hessian of the unscaled prediction, whose gradient the forces are --
        and energy / forces bitwise those of `run`.  Builds the graph (one synchronisation for the counts), then one call."""
        if self._w is None:
            raise NablaB200Error("DimeNetRunner.run_hvp before set_weights / bind")
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        v = self._directions(v, n, dev)
        n_dir = int(v.shape[0])
        gbuf, counts = self._graph(z, pos, mol_ptr, n_mol)
        ws = self._buffer("_ws", self._bytes("nb200_dimenet_hvp_workspace_bytes", byref(self._w), n_mol, n, counts), dev)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n, 3, dtype=torch.float32, device=dev) if with_forces else None
        hv = torch.empty(n_dir, n, 3, dtype=torch.float32, device=dev)
        check(lib.nb200_dimenet_hvp(self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, gbuf.data_ptr(), gbuf.numel(),
                                    counts, ws.data_ptr(), ws.numel(), n_dir, v.data_ptr(), energy.data_ptr(),
                                    None if forces is None else forces.data_ptr(), hv.data_ptr(), self._stream()), "nb200_dimenet_hvp")
        return energy, forces, hv


class DimeNetEngine(BoundedEngine):
    """`BoundedEngine` of DimeNet++: edge and triplet-slot bounds."""

    label = "DimeNet++"
    einval_text = "atomic number outside [0, 94] or non-finite atom coordinates"
    count_names = ("edges", "triplets")


class DimeNetEnergyFn(torch.autograd.Function):
    """(flat weights) -> (energy [B], forces [N,3]) through nb200_dimenet_energy_forces; backward = nb200_dimenet_train_grads with the
    incoming gradients as seeds (the force term by forward-over-reverse, DESIGN.md 3.15.1).  Once differentiable; pos gets no gradient."""

    @staticmethod
    def forward(ctx, flat, model, runner, offs, z, pos, mol_ptr, n_mol):
        runner.bind(model, flat.detach(), offs)
        energy, forces, _ = runner.run(z, pos, mol_ptr, n_mol)
        ctx.runner, ctx.w, ctx.keep, ctx.n_mol = runner, runner._w, runner._keep, n_mol
        ctx.save_for_backward(z, pos, mol_ptr)
        return energy, forces

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_energy, g_forces):
        z, pos, mol_ptr = ctx.saved_tensors
        runner = ctx.runner
        runner._w, runner._keep = ctx.w, ctx.keep
        grads = runner.train_grads(z, pos, mol_ptr, ctx.n_mol, g_energy, g_forces)
        return grads, None, None, None, None, None, None, None
