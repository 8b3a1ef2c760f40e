"""Host-side driver of the PaiNN energy+forces engine (`nb200_painn_energy_forces`), and `BoundedEngine`, the same interface for the
forwards sized by per-batch upper bounds (DimeNet++, GemNet-OC).

Owns: the C engine object, the device workspace, the canonical weight export.
The model classes (`painn_oc.PaiNN`, `spk.NeuralNetworkPotential`) only describe how their
reference-named parameters map onto the canonical layout.
"""
from ctypes import byref
from typing import Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import EngineDriver, NablaB200Error, PainnWeights, SchnetWeights, check, ptr
from .schnet_train import count_edges

_KINDS = {
    "painn": (PainnWeights, "nb200_painn_workspace_bytes", "nb200_painn_energy_forces",
              ("emb", "w_rbf", "b_rbf", "A1", "c1", "A2", "c2", "U", "B1", "d1", "B2", "d2", "R1", "e1", "R2", "e2", "rbf_offsets")),
    "schnet": (SchnetWeights, "nb200_schnet_workspace_bytes", "nb200_schnet_energy_forces",
               ("emb", "w_f1", "b_f1", "W_f2", "b_f2", "I1", "P1", "p1", "P2", "p2", "R1", "e1", "R2", "e2", "rbf_offsets")),
}


class PainnEngine(EngineDriver):
    """One engine per (module, device). Not thread-safe; one CUDA stream per call."""

    SLACK = 1.05  # the capacity-sized workspace is the largest buffer of the project (the filter rows alone: ~3.5 GB per bench.py step)

    def __init__(self, kind: str = "painn", lib=None):
        super().__init__(lib)
        self.kind = kind
        self._wtype, self._ws_fn, self._run_fn, self._wkeys = _KINDS[kind]
        self._ws: Optional[torch.Tensor] = None
        self._status: Optional[torch.Tensor] = None
        self._weights = None
        self._keep: Dict[str, torch.Tensor] = {}
        self._wkey = None
        self.e_cap = 0
        self.edges_per_atom_guess = 32
        # deferred status checks of `run_async` (pinned host copies + events), oldest first
        self._pending = []
        self._validated_ratio = 0.0   # largest edges / atom seen by a CHECKED launch: async launches size their capacity from it
        self.e_cap_slack = 1024       # + 25 % + this many edges on top of validated_ratio * n_atoms
        # two-call training step: token of the forward whose activations the workspace still holds (0: none), its sizes
        self._kept_token = 0
        self._kept_serial = 0
        self._kept_args = None
        self.edge_storage = "f32"

    def set_edge_storage(self, kind: str) -> None:
        """'f32' (default) or 'bf16': storage of the per-edge arrays of the TRAINING calls (`nb200_engine_set_edge_storage`)."""
        if kind not in ("f32", "bf16"):
            raise ValueError("edge storage: 'f32' or 'bf16'")
        check(self.lib.nb200_engine_set_edge_storage(self._h, int(kind == "bf16")), "nb200_engine_set_edge_storage")
        self.edge_storage = kind
        self._kept_token = 0

    # ------------------------------------------------------------------ weights
    def set_weights(self, key, tensors: Dict[str, torch.Tensor], scalars: Dict[str, float]):
        """tensors: canonical fp32 contiguous CUDA tensors (see include/nabla_b200.h)."""
        if key == self._wkey:
            return
        w = self._wtype()
        for k in self._wkeys:
            t = tensors[k]
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise NablaB200Error(f"weight {k}: need contiguous fp32 CUDA tensor")
            setattr(w, k, t.data_ptr())
        for k, v in scalars.items():
            setattr(w, k, v)
        self._keep = dict(tensors)  # keep the exported copies alive
        self._weights = w
        self._wkey = key

    # ------------------------------------------------------------------ run
    def _workspace(self, fn_name: str, *args, device) -> torch.Tensor:
        """The workspace sized by `fn_name(weights, *args)`, and the device status word of the calls."""
        if self._status is None or self._status.device != device:
            self._status = torch.zeros(4, dtype=torch.int32, device=device)
        return self._buffer("_ws", self._bytes(fn_name, byref(self._weights), *args), device)

    def _cap(self, n_atoms: int, validated: bool = False) -> int:
        """Edge capacity of the next launch (never below the current one): the first-batch guess, or, once a checked launch has measured
        the edges per atom, 25 % + `e_cap_slack` above that."""
        want = int(1.25 * self._validated_ratio * n_atoms) + self.e_cap_slack if validated else n_atoms * self.edges_per_atom_guess
        return max(self.e_cap, want)

    def _regrow(self, call):
        """Synchronous: `call()` launches with `_cap` and fills the status word; on NB200_ECAPACITY the capacity grows to the reported
        edge count and the call runs once more.  -> (what `call` returned, status on the host)."""
        for _ in range(2):
            out = call()
            st = self._status.cpu()
            if int(st[1]) == -4:
                self.e_cap = int(int(st[0]) * 1.1) + 1024
                continue
            self.raise_on_status(st)
            return out, st
        raise NablaB200Error("edge capacity regrow failed")

    def _defer_status(self, n_atoms: int) -> None:
        """Queue the status word of the launch just enqueued for `check_pending`: a pinned host copy behind the results, and an event."""
        host = torch.empty(5, dtype=torch.int32, pin_memory=True)
        host[4] = n_atoms
        host[:4].copy_(self._status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pending.append((host, ev))

    def _first_run(self, z, pos, mol_ptr, n_mol, with_forces):
        """The synchronous `run` of an engine's first batch, which sizes the capacity of the asynchronous launches after it."""
        energy, forces, st = self.run(z, pos, mol_ptr, n_mol, with_forces)
        self._validated_ratio = float(int(st[0])) / max(1, z.shape[0])
        self.e_cap = max(self.e_cap, int(1.25 * int(st[0])) + 1024)
        return energy, forces

    def launch(self, z: torch.Tensor, pos: torch.Tensor, mol_ptr: torch.Tensor, n_mol: int, with_forces: bool = True,
               e_cap: Optional[int] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor], torch.Tensor]:
        """Asynchronous: enqueue one batch on the current stream. Returns (energy, forces, status);
        `status` is a device int32[4] = {n_edges, error_code, max_degree, n_isolated}; the caller
        must eventually validate it with `raise_on_status`."""
        if self._weights is None:
            raise NablaB200Error("set_weights() first")
        n_atoms = z.shape[0]
        if not (self._on_device(z) and z.dtype == torch.int32 and pos.dtype == torch.float32 and mol_ptr.dtype == torch.int32):
            raise NablaB200Error("launch(): need CUDA int32 z / mol_ptr and fp32 pos")
        self.e_cap = e_cap = self._cap(n_atoms) if e_cap is None else e_cap
        self._kept_token = 0  # this launch overwrites the workspace a kept training forward lives in
        ws = self._workspace(self._ws_fn, n_mol, n_atoms, e_cap, int(with_forces), device=z.device)
        energy = torch.empty(n_mol, dtype=torch.float32, device=z.device)
        forces = torch.empty(n_atoms, 3, dtype=torch.float32, device=z.device) if with_forces else None
        status = self._status
        rc = getattr(self.lib, self._run_fn)(
            self._h, byref(self._weights), ptr(z), ptr(pos), ptr(mol_ptr), n_mol, n_atoms, e_cap,
            ptr(ws), ws.numel(), ptr(energy), ptr(forces), ptr(status), self._stream())
        check(rc, self._run_fn)
        return energy, forces, status

    @staticmethod
    def raise_on_status(status_host) -> None:
        n_edges, err, max_deg, n_iso = (int(v) for v in status_host)
        if err == -4:
            raise NablaB200Error(f"NB200_ECAPACITY: batch has {n_edges} edges")
        if err != 0:
            raise NablaB200Error(f"neighbour build failed: {_lib.ERRORS.get(err, err)} (max degree {max_deg})")

    # ------------------------------------------------------------------ training
    GRAD_KEYS = ("emb", "w_rbf", "b_rbf", "A1", "c1", "A2", "c2", "U", "B1", "d1", "B2", "d2", "R1", "e1", "R2", "e2")

    def _grad_struct(self):
        """Fresh gradient tensors shaped like the exported weights, and the weight struct of the gradient calls that points at them
        (rbf_offsets: the weights' own)."""
        grads = {k: torch.empty_like(self._keep[k]) for k in self.GRAD_KEYS}
        gw = self._wtype()
        for k in self._wkeys:
            setattr(gw, k, (grads[k] if k in grads else self._keep[k]).data_ptr())
        return grads, gw

    def run_train(self, z, pos, mol_ptr, n_mol, seed: Optional[torch.Tensor], force_seed: Optional[torch.Tensor] = None):
        """One training step of the PaiNN engine in one call (`nb200_painn_energy_forces_grads`: the fused forward of
        `run_train_forward`, then the backward of `run_train_backward`): energy, true forces and
        d(sum_m seed_m E_m + sum_i force_seed_i . F_i)/d(canonical weights) as a dict of fresh tensors shaped like the exported weights.
        The first call of an engine is synchronous (checks the device status; regrows the edge capacity once like `run`); later calls
        enqueue and defer the status check like `run_async`."""
        if self.kind != "painn":
            raise NotImplementedError("training is built for the PaiNN engine only")
        if self._weights is None:
            raise NablaB200Error("set_weights() first")
        n_atoms = z.shape[0]
        dev = z.device
        self._kept_token = 0
        grads, gw = self._grad_struct()
        self._check_seeds(seed, force_seed, n_mol, n_atoms, dev)
        validated = self._validated_ratio > 0.0  # a checked launch has sized the edge capacity: no host sync in this call then

        def call():
            self.e_cap = e_cap = self._cap(n_atoms, validated)
            ws = self._workspace("nb200_painn_train_workspace_bytes", n_mol, n_atoms, e_cap, int(force_seed is not None), device=dev)
            energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
            forces = torch.empty(n_atoms, 3, dtype=torch.float32, device=dev)
            rc = self.lib.nb200_painn_energy_forces_grads(
                self._h, byref(self._weights), ptr(z), ptr(pos), ptr(mol_ptr), n_mol, n_atoms, e_cap, ptr(ws), ws.numel(),
                ptr(seed), ptr(force_seed), byref(gw), ptr(energy), ptr(forces), ptr(self._status), self._stream())
            check(rc, "nb200_painn_energy_forces_grads")
            return energy, forces

        if validated:
            # deferred status check (as run_async): a failed launch has NaN energies / forces, and its gradients came from an empty graph;
            # the next call (or check_pending(wait=True)) raises
            energy, forces = call()
            self._defer_status(n_atoms)
        else:
            (energy, forces), st = self._regrow(call)
            self._validated_ratio = max(self._validated_ratio, float(int(st[0])) / max(1, n_atoms))
        return energy, forces, grads

    # ------------------------------------------------------------------ training step in two calls (forward kept for the backward)
    def run_train_forward(self, z, pos, mol_ptr, n_mol, with_force_seed: bool = True):
        """Training-mode forward (`nb200_painn_train_forward`): energy, forces and a token.  The activations stay in the workspace until
        another launch of this engine overwrites them; `run_train_backward(token, ...)` then produces the parameter gradients without
        recomputing the forward.  Asynchronous with a deferred status check like `run_async` (the first batch of an engine is sized by one
        synchronous inference launch)."""
        if self.kind != "painn":
            raise NotImplementedError("training is built for the PaiNN engine only")
        self.check_pending()
        n_atoms, dev = z.shape[0], z.device
        if self._validated_ratio == 0.0:
            self._first_run(z, pos, mol_ptr, n_mol, True)
        self.e_cap = e_cap = self._cap(n_atoms, validated=True)
        ws = self._workspace("nb200_painn_train_workspace_bytes", n_mol, n_atoms, e_cap, int(with_force_seed), device=dev)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n_atoms, 3, dtype=torch.float32, device=dev)
        rc = self.lib.nb200_painn_train_forward(self._h, byref(self._weights), ptr(z), ptr(pos), ptr(mol_ptr), n_mol, n_atoms, e_cap, ptr(ws),
                                                ws.numel(), int(with_force_seed), ptr(energy), ptr(forces), ptr(self._status), self._stream())
        check(rc, "nb200_painn_train_forward")
        self._defer_status(n_atoms)
        self._kept_serial += 1
        self._kept_token = self._kept_serial
        self._kept_args = (n_mol, n_atoms, e_cap, int(with_force_seed), ws.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        return energy, forces, self._kept_token

    def kept(self, token: int) -> bool:
        return token != 0 and token == self._kept_token

    def run_train_backward(self, token: int, z, mol_ptr, seed: Optional[torch.Tensor], force_seed: Optional[torch.Tensor] = None):
        """Parameter gradients from the forward `token` refers to (`nb200_painn_train_backward`); same result as `run_train`."""
        if not self.kept(token):
            raise NablaB200Error("run_train_backward(): the forward's activations are gone (another launch used this engine since)")
        n_mol, n_atoms, e_cap, wfs, ws_ptr, stream = self._kept_args
        if self._ws.data_ptr() != ws_ptr or torch.cuda.current_stream(z.device).cuda_stream != stream:
            raise NablaB200Error("run_train_backward(): workspace or stream changed since the forward")
        if force_seed is not None and not wfs:
            raise NablaB200Error("run_train_backward(): the forward was run without room for the force-seed tangent pass")
        self._check_seeds(seed, force_seed, n_mol, n_atoms, z.device)
        grads, gw = self._grad_struct()
        rc = self.lib.nb200_painn_train_backward(self._h, byref(self._weights), ptr(z), ptr(mol_ptr), n_mol, n_atoms, e_cap, ptr(self._ws), self._ws.numel(),
                                                 wfs, ptr(seed), ptr(force_seed), byref(gw), ptr(self._status), self._stream())
        check(rc, "nb200_painn_train_backward")
        self._kept_token = 0  # the backward reuses transient buffers; a second backward of the same forward recomputes
        return grads

    # ------------------------------------------------------------------ Hessian-vector products
    def run_hvp(self, z, pos, mol_ptr, n_mol, v, with_forces: bool = True):
        """Exact Hessian-vector products of the energy (`nb200_painn_hvp`, `nb200_schnet_hvp`): v [n_dir, n_atoms, 3] (or [n_atoms, 3]) fp32
        CUDA, in Angstrom.  Returns (energy [B], forces [N, 3] or None, hv [n_dir, N, 3] = H v in Ha/A).  Synchronous like `run`: the PaiNN
        engine checks the device status and regrows the edge capacity once; the SchNet engine counts the edges first (one host sync)."""
        if self.kind not in ("painn", "schnet"):
            raise NotImplementedError(f"Hessian-vector products are not built for the {self.kind} engine")
        if self._weights is None:
            raise NablaB200Error("set_weights() first")
        n_atoms, dev = z.shape[0], z.device
        if not (self._on_device(z) and z.dtype == torch.int32 and pos.dtype == torch.float32 and mol_ptr.dtype == torch.int32):
            raise NablaB200Error("run_hvp(): need CUDA int32 z / mol_ptr and fp32 pos")
        v = self._directions(v, n_atoms, dev)
        n_dir = v.shape[0]
        self._kept_token = 0  # this call overwrites the workspace a kept training forward lives in
        if self.kind == "schnet":
            return self._run_schnet_hvp(z, pos, mol_ptr, n_mol, v, with_forces)

        def call():
            self.e_cap = e_cap = self._cap(n_atoms)
            ws = self._workspace("nb200_painn_hvp_workspace_bytes", n_mol, n_atoms, e_cap, n_dir, device=dev)
            energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
            forces = torch.empty(n_atoms, 3, dtype=torch.float32, device=dev) if with_forces else None
            hv = torch.empty(n_dir, n_atoms, 3, dtype=torch.float32, device=dev)
            rc = self.lib.nb200_painn_hvp(self._h, byref(self._weights), ptr(z), ptr(pos), ptr(mol_ptr), n_mol, n_atoms, e_cap, ptr(ws),
                                          ws.numel(), n_dir, ptr(v), ptr(energy), ptr(forces), ptr(hv), ptr(self._status), self._stream())
            check(rc, "nb200_painn_hvp")
            return energy, forces, hv

        return self._regrow(call)[0]

    def _run_schnet_hvp(self, z, pos, mol_ptr, n_mol, v, with_forces):
        """`nb200_schnet_train_count` (exact edge count, one host sync), then `nb200_schnet_hvp` on the engine's weights."""
        n_atoms, dev, n_dir = z.shape[0], z.device, v.shape[0]
        row_ptr, n_edges, ws = count_edges(self, self._weights, pos, mol_ptr, n_mol, "nb200_schnet_hvp_workspace_bytes")
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n_atoms, 3, dtype=torch.float32, device=dev) if with_forces else None
        hv = torch.empty(n_dir, n_atoms, 3, dtype=torch.float32, device=dev)
        check(self.lib.nb200_schnet_hvp(self._h, byref(self._weights), ptr(z), ptr(pos), ptr(mol_ptr), n_mol, n_atoms, ptr(row_ptr), n_edges,
                                        ptr(ws), ws.numel(), n_dir, ptr(v), ptr(energy), ptr(forces), ptr(hv), self._stream()), "nb200_schnet_hvp")
        return energy, forces, hv

    # ------------------------------------------------------------------ asynchronous inference (the reference-facing forward())
    _MAX_PENDING = 8

    def check_pending(self, wait: bool = False) -> None:
        """Validate the device status words of earlier `run_async` launches whose results have arrived (all of them if `wait`).
        A failed launch already turned its own outputs into NaN on the device (k_poison_on_error); here the error becomes an exception:
        a too-small edge capacity grows the capacity for the following launches first."""
        while self._pending:
            host, ev = self._pending[0]
            if not wait and len(self._pending) < self._MAX_PENDING and not ev.query():
                return
            ev.synchronize()
            self._pending.pop(0)
            n_edges, err = int(host[0]), int(host[1])
            if err == -4:
                self.e_cap = int(n_edges * 1.1) + 1024
                raise NablaB200Error(f"NB200_ECAPACITY in an earlier asynchronous forward: that batch had {n_edges} edges, its outputs were set "
                                     "to NaN; the edge capacity has been grown -- re-submit the batch")
            self.raise_on_status(host[:4])
            self._validated_ratio = max(self._validated_ratio, float(n_edges) / max(1, int(host[4])))

    def run_async(self, z, pos, mol_ptr, n_mol, with_forces=True):
        """Enqueue one batch on the current stream and return (energy, forces) WITHOUT synchronising: the status word travels to pinned
        host memory behind the results and is checked by the next call / `check_pending(wait=True)`.  The first batch of an engine (and
        any batch larger than what has been validated) takes the synchronous path once, which sizes the edge capacity from the
        measured edges per atom (+25 %).  Errors of an asynchronous launch surface late but never silently: the launch's outputs
        are NaN and the next call raises."""
        self.check_pending()
        n_atoms = z.shape[0]
        if self._validated_ratio == 0.0:
            return self._first_run(z, pos, mol_ptr, n_mol, with_forces)
        energy, forces, _ = self.launch(z, pos, mol_ptr, n_mol, with_forces, e_cap=self._cap(n_atoms, validated=True))
        self._defer_status(n_atoms)
        return energy, forces

    def clone_for_stream(self) -> "PainnEngine":
        """A second engine (own cuBLAS handle, workspace and status word) sharing this one's exported
        weights: lets independent batches run concurrently on different CUDA streams."""
        other = PainnEngine(self.kind)
        other._weights, other._keep, other._wkey = self._weights, self._keep, self._wkey
        other.e_cap, other.edges_per_atom_guess = self.e_cap, self.edges_per_atom_guess
        other._validated_ratio, other.e_cap_slack = self._validated_ratio, self.e_cap_slack
        return other

    def run(self, z, pos, mol_ptr, n_mol, with_forces=True):
        """Synchronous convenience: launch, check the device status, regrow the edge capacity once
        if the guess was too small (the only host<->device sync of the whole path)."""
        (energy, forces, _), st = self._regrow(lambda: self.launch(z, pos, mol_ptr, n_mol, with_forces))
        return energy, forces, st


class BoundedEngine:
    """What `optimization.ASEBatchwiseLBFGS` and `md.BatchwiseMD` need from a model whose forward is sized by per-batch upper bounds, with
    `PainnEngine`'s method names.  `run` derives the bounds from the molecule sizes and `launch` sizes everything by them (`e_cap` is ignored):
    there is no capacity to grow, and a count above its bound is a bug.  A model's subclass (`DimeNetEngine`, `GemNetOCEngine`) declares
    `label` and `einval_text` for messages, the `count_names` behind `bounds`, and may refine `check_sizes` and `size_args`."""

    grows_capacity = False

    def __init__(self, model, runner):
        self.model, self.runner, self.e_cap = model, runner, 0
        self._batch = None
        self.last_status = None

    @staticmethod
    def check_sizes(model, max_atoms: int) -> None:
        """Host check of the largest molecule of a batch (the bounds refuse counts past int32)."""

    @staticmethod
    def size_args(max_atoms: int) -> tuple:
        """What the runner's `launch` takes between n_mol and the bounds."""
        return ()

    def run(self, z, pos, mol_ptr, n_mol: int):
        """First evaluation of a batch: checks the batch on the host (once, not per step), fixes its bounds, launches and validates.
        -> (energy, forces, status words on the host)."""
        ptr_host = mol_ptr.cpu()
        sizes = ptr_host[1:] - ptr_host[:-1]
        if len(sizes) != n_mol or n_mol < 1 or int(ptr_host[0]) != 0 or int(sizes.min()) < 1 or int(ptr_host[-1]) != z.shape[0]:
            raise NablaB200Error(f"{self.label}: `mol_ptr` must hold n_mol + 1 increasing atom offsets starting at 0 (atoms of a molecule "
                                 "contiguous)")
        max_atoms = int(sizes.max())
        self.check_sizes(self.model, max_atoms)
        self.model._sync_weights(self.runner, pos.device)
        self._batch = ((mol_ptr.data_ptr(), n_mol, int(z.shape[0])), *self.size_args(max_atoms), self.runner.count_bounds(sizes))
        energy, forces, status = self.launch(z, pos, mol_ptr, n_mol)
        host = status.cpu()
        self.raise_on_status(host)
        self.last_status = host
        return energy, forces, host

    def launch(self, z, pos, mol_ptr, n_mol: int, e_cap=None):
        if self._batch is None or self._batch[0] != (mol_ptr.data_ptr(), n_mol, int(z.shape[0])):
            raise NablaB200Error(f"{type(self).__name__}.launch: call run() on this batch first (it derives the bounds the launch is sized by)")
        return self.runner.launch(z, pos, mol_ptr, n_mol, *self._batch[1:])

    @property
    def bounds(self) -> Dict[str, int]:
        return {k: int(self._batch[-1][i]) for i, k in enumerate(self.count_names)} if self._batch else {}

    @classmethod
    def raise_on_status(cls, status_host) -> None:
        """`status_host`: the status words of a launch on the host; the first four read like `PainnEngine`'s.  Atoms without neighbours are
        not an error."""
        n_edges, err, max_deg, n_iso = (int(v) for v in status_host[:4])
        if err == -4:
            raise NablaB200Error(f"NB200_ECAPACITY: a count exceeds its bound ({n_edges} edges); `mol_ptr` changed under the engine?")
        if err == -1:
            raise NablaB200Error(f"{cls.label}: {cls.einval_text}")
        if err != 0:
            raise NablaB200Error(f"{cls.label} graph construction failed: {_lib.ERRORS.get(err, err)} (max degree {max_deg}, {n_iso} atoms "
                                 "without neighbours)")


def refuse_training(model) -> None:
    """Hessian-vector products run through the inference engine: refuse a model in training mode with autograd on."""
    if model.training and torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters()):
        raise NotImplementedError("Hessians run through the inference engine; call .eval() or torch.no_grad()")


def mol_ptr_from_batch(batch: torch.Tensor, n_mol: Optional[int] = None) -> Tuple[torch.Tensor, int]:
    """PyG `batch` vector (sorted graph ids) -> int32 CSR pointer. Syncs once if n_mol is unknown."""
    if n_mol is None:
        n_mol = int(batch[-1].item()) + 1 if batch.numel() else 0
    counts = torch.bincount(batch, minlength=n_mol)
    mp = torch.zeros(n_mol + 1, dtype=torch.int32, device=batch.device)
    mp[1:] = torch.cumsum(counts, 0)
    return mp, n_mol
