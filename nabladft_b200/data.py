"""Data path for the energy / force models (SURVEY.md section 8f-2): ASE-sqlite reader -> packed flat arrays -> device batches.

The reference feeds the models through Python datasets: `PyGNablaDFT.process` walks `ase.db` rows into a list of PyG `Data`
objects and collates them (nablaDFT/dataset/pyg_datasets.py:101-119); the schnetpack path (`ASENablaDFT`, nablaDFT_dataset.py:120-159)
additionally runs `ASENeighborList` per sample in 8 dataloader workers.  At 10^4-10^5 molecules/s per GPU that is the bottleneck.
Here:
  * `read_ase_energy_db`  -- the same row semantics (numbers -> z, positions -> float32 pos, data["energy"] -> y, data["forces"] ->
    float32 forces) with only sqlite3 + numpy (ASE's "bytes" container of the `data` column is decoded directly), no per-row objects;
  * `PackedEnergyDataset` -- Z, R, E, F as flat arrays + a CSR offset per molecule, saved as .npy files and memory-mapped;
  * `DeviceBatcher`       -- epoch iterator that slices contiguous or shuffled molecule sets into batches, stages them in pinned
    buffers and copies them on a side stream one batch ahead; what arrives on the device is exactly what the engines take
    (z int32, pos float32, mol_ptr int32) -- the neighbour list is built there.  Ranks own atom-balanced shards of every epoch.
"""
import json
import os
import sqlite3
import struct
from typing import Dict, Iterator

import numpy as np
import torch

from .parallel import balanced_ranges


def _decode_ase_bytes(blob: bytes) -> Dict[str, np.ndarray]:
    """ASE's binary `data` container: int64 offset of a trailing JSON index, raw arrays in front (ase/io/bytes.py semantics)."""
    off = struct.unpack("<q", blob[:8])[0]
    meta = json.loads(blob[off:].decode())
    out = {}
    for key, val in meta.items():
        if isinstance(val, dict) and "__ndarray__" in val:
            shape, dtype, start = val["__ndarray__"]
            out[key] = np.frombuffer(blob, dtype=dtype, count=int(np.prod(shape)), offset=start).reshape(shape)
        else:
            out[key] = np.asarray(val)
    return out


def _decode_data(data) -> Dict[str, np.ndarray]:
    if data is None:
        return {}
    if isinstance(data, (bytes, memoryview)):
        return _decode_ase_bytes(bytes(data))
    return {k: np.asarray(v) for k, v in json.loads(data).items()}  # older ASE versions store JSON text


def read_ase_energy_db(path: str) -> Dict[str, np.ndarray]:
    """All rows of an nablaDFT energy database, in id order: flat z / pos / forces, per-molecule energy and offsets."""
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        rows = con.execute("select numbers, positions, natoms, data from systems order by id").fetchall()
    finally:
        con.close()
    z, pos, forces, energy, ptr = [], [], [], [], [0]
    for numbers, positions, natoms, data in rows:
        zz = np.frombuffer(numbers, dtype=np.int32)
        pp = np.frombuffer(positions, dtype=np.float64).reshape(-1, 3)
        d = _decode_data(data)
        ff = np.asarray(d["forces"], dtype=np.float64).reshape(-1, 3)
        if not (len(zz) == natoms == len(pp) == len(ff)):
            raise ValueError(f"{path}: inconsistent row (natoms {natoms}, numbers {len(zz)}, positions {len(pp)}, forces {len(ff)})")
        z.append(zz); pos.append(pp); forces.append(ff)
        energy.append(float(np.asarray(d["energy"]).reshape(-1)[0]))
        ptr.append(ptr[-1] + int(natoms))
    cat = lambda xs, shape, dt: (np.concatenate(xs) if xs else np.zeros(shape)).astype(dt)
    return {"z": cat(z, (0,), np.int32), "pos": cat(pos, (0, 3), np.float32), "forces": cat(forces, (0, 3), np.float32),
            "energy": np.asarray(energy, dtype=np.float32), "ptr": np.asarray(ptr, dtype=np.int64)}


class PackedEnergyDataset:
    """Z, R, E, F as flat arrays + CSR offsets.  `save` / `load` use one .npy per array (memory-mapped on load)."""

    FIELDS = ("z", "pos", "forces", "energy", "ptr")

    def __init__(self, z, pos, forces, energy, ptr):
        self.z, self.pos, self.forces, self.energy, self.ptr = z, pos, forces, energy, ptr
        if not (len(ptr) == len(energy) + 1 and int(ptr[-1]) == len(z) == len(pos) == len(forces)):
            raise ValueError("inconsistent packed arrays")

    @classmethod
    def from_ase_db(cls, path: str) -> "PackedEnergyDataset":
        return cls(**read_ase_energy_db(path))

    def save(self, directory: str) -> None:
        os.makedirs(directory, exist_ok=True)
        for f in self.FIELDS:
            np.save(os.path.join(directory, f + ".npy"), np.ascontiguousarray(getattr(self, f)))

    @classmethod
    def load(cls, directory: str, mmap: bool = True) -> "PackedEnergyDataset":
        return cls(**{f: np.load(os.path.join(directory, f + ".npy"), mmap_mode="r" if mmap else None) for f in cls.FIELDS})

    def __len__(self) -> int:
        return len(self.energy)

    @property
    def n_atoms(self) -> np.ndarray:
        return np.diff(np.asarray(self.ptr))

    def molecule(self, i: int) -> Dict[str, np.ndarray]:
        a, b = int(self.ptr[i]), int(self.ptr[i + 1])
        return {"z": self.z[a:b], "pos": self.pos[a:b], "forces": self.forces[a:b], "energy": self.energy[i]}


class DeviceBatch:
    """One batch on the device.  `as_pyg()` / `as_spk()` give the two input contracts of the reference (SURVEY.md section 8b)."""

    def __init__(self, z, pos, mol_ptr, energy, forces, index):
        self.z, self.pos, self.mol_ptr, self.energy, self.forces, self.index = z, pos, mol_ptr, energy, forces, index
        self.n_mol = energy.shape[0]

    def _batch_vector(self):
        counts = (self.mol_ptr[1:] - self.mol_ptr[:-1]).long()
        return torch.repeat_interleave(torch.arange(self.n_mol, device=self.z.device), counts), counts

    def as_pyg(self):
        b, _ = self._batch_vector()

        class _Data:
            pass

        d = _Data()
        d.z, d.pos, d.batch, d.ptr, d.y, d.forces, d.num_graphs = self.z.long(), self.pos, b, self.mol_ptr.long(), self.energy, self.forces, self.n_mol
        return d

    def as_spk(self) -> Dict[str, torch.Tensor]:
        b, counts = self._batch_vector()
        return {"_atomic_numbers": self.z.long(), "_positions": self.pos, "_idx_m": b, "_n_atoms": counts, "energy": self.energy, "forces": self.forces,
                "_idx": self.index}


class DeviceBatcher:
    """Epoch iterator over a PackedEnergyDataset.

    batch_size molecules per batch (last one smaller unless drop_last); `shuffle` permutes molecules per epoch with `seed + epoch`
    (the same permutation on every rank); rank r of `world` owns an atom-balanced contiguous slice of the epoch's molecule sequence and
    cuts it into the same NUMBER of batches as every other rank (`_n_batches`), ~batch_size molecules each.
    On CUDA devices batches are gathered into pinned host buffers and copied on a side stream one batch ahead of the consumer."""

    def __init__(self, data: PackedEnergyDataset, batch_size: int, device="cuda", shuffle: bool = False, seed: int = 0, drop_last: bool = False,
                 rank: int = 0, world: int = 1):
        self.data, self.batch_size, self.shuffle, self.seed, self.drop_last = data, int(batch_size), shuffle, seed, drop_last
        self.device = torch.device(device)
        self.rank, self.world, self.epoch = rank, world, 0
        self._cuda = self.device.type == "cuda"
        self._stream = torch.cuda.Stream(self.device) if self._cuda else None
        # two sets of pinned staging buffers, reused across batches (cudaHostAlloc per batch costs more than the copy itself)
        self._pool = [dict(), dict()]
        self._pool_event = [None, None]
        self._turn = 0

    def _pinned(self, which: int, name: str, shape, dtype) -> torch.Tensor:
        n = int(np.prod(shape))
        buf = self._pool[which].get(name)
        if buf is None or buf.numel() < n or buf.dtype != dtype:
            buf = torch.empty(max(n, 1) * 5 // 4 + 16, dtype=dtype, pin_memory=True)
            self._pool[which][name] = buf
        return buf[:n].view(*shape)

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def _order(self) -> np.ndarray:
        n = len(self.data)
        order = np.random.default_rng(self.seed + self.epoch).permutation(n) if self.shuffle else np.arange(n)
        if self.world > 1:
            lo, hi = balanced_ranges(torch.from_numpy(self.data.n_atoms[order].astype(np.int64)), self.world)[self.rank]
            order = order[lo:hi]
        return order

    def _n_batches(self) -> int:
        """Steps per epoch -- the SAME number on every rank (each rank calls one gradient all-reduce per step, so a rank with more
        batches would block in NCCL forever).  world == 1: the usual len // batch_size (drop_last) or ceil.  world > 1: the atom-balanced
        shards hold different numbers of molecules, so the count is derived from the GLOBAL molecule count and every rank cuts its own
        shard into that many nearly equal batches (~batch_size molecules, similar atom counts per rank and step)."""
        n = len(self.data)
        per_step = self.batch_size * self.world
        nb = n // per_step if self.drop_last else (n + per_step - 1) // per_step
        return nb if self.world == 1 else max(nb, 1 if n >= self.world else 0)

    def _batches(self, order: np.ndarray):
        nb = self._n_batches()
        if self.world == 1:
            return [order[k * self.batch_size:(k + 1) * self.batch_size] for k in range(nb)]
        return [b for b in np.array_split(order, nb)] if nb else []

    def __len__(self) -> int:
        return self._n_batches()

    def _gather(self, idx: np.ndarray):
        d = self.data
        ptr = np.asarray(d.ptr)
        counts = (ptr[idx + 1] - ptr[idx]).astype(np.int64)
        mol_ptr = np.zeros(len(idx) + 1, dtype=np.int32)
        np.cumsum(counts, out=mol_ptr[1:])
        n_at = int(mol_ptr[-1])
        pin = self._cuda
        if pin:
            which = self._turn
            self._turn ^= 1
            if self._pool_event[which] is not None:
                self._pool_event[which].synchronize()  # the copy that last read this buffer set (two batches ago) has finished
            z = self._pinned(which, "z", (n_at,), torch.int32)
            pos = self._pinned(which, "pos", (n_at, 3), torch.float32)
            forces = self._pinned(which, "forces", (n_at, 3), torch.float32)
        else:
            z = torch.empty(n_at, dtype=torch.int32)
            pos = torch.empty(n_at, 3, dtype=torch.float32)
            forces = torch.empty(n_at, 3, dtype=torch.float32)
        zn, pn, fn = z.numpy(), pos.numpy(), forces.numpy()
        contiguous = len(idx) > 0 and bool(np.all(np.diff(idx) == 1))
        if contiguous:  # unshuffled epochs: one slice per array
            a, b = int(ptr[idx[0]]), int(ptr[idx[-1] + 1])
            zn[:] = d.z[a:b]; pn[:] = d.pos[a:b]; fn[:] = d.forces[a:b]
        else:  # shuffled epochs: one vectorised gather per array (atom index = molecule start + position inside the molecule)
            atom_idx = np.repeat(ptr[idx] - mol_ptr[:-1].astype(np.int64), counts) + np.arange(n_at, dtype=np.int64)
            np.take(d.z, atom_idx, axis=0, out=zn); np.take(d.pos, atom_idx, axis=0, out=pn); np.take(d.forces, atom_idx, axis=0, out=fn)
        energy = torch.from_numpy(np.asarray(d.energy)[idx].astype(np.float32))
        mol_ptr_t, idx_t = torch.from_numpy(mol_ptr), torch.from_numpy(idx.astype(np.int64))
        if pin:
            e_pin = self._pinned(which, "energy", (len(idx),), torch.float32); e_pin.copy_(energy)
            p_pin = self._pinned(which, "mol_ptr", (len(idx) + 1,), torch.int32); p_pin.copy_(mol_ptr_t)
            i_pin = self._pinned(which, "index", (len(idx),), torch.int64); i_pin.copy_(idx_t)
            energy, mol_ptr_t, idx_t = e_pin, p_pin, i_pin
        host = (z, pos, mol_ptr_t, energy, forces, idx_t)
        if not self._cuda:
            return DeviceBatch(*host), None
        with torch.cuda.stream(self._stream):
            dev = [t.to(self.device, non_blocking=True) for t in host]
            done = torch.cuda.Event()
            done.record(self._stream)
        self._pool_event[which] = done
        return DeviceBatch(*dev), (done, host)

    def __iter__(self) -> Iterator[DeviceBatch]:
        batches = self._batches(self._order())
        nxt = self._gather(batches[0]) if batches else None
        for k in range(len(batches)):
            cur = nxt
            nxt = self._gather(batches[k + 1]) if k + 1 < len(batches) else None
            batch, pending = cur
            if pending is not None:
                consumer = torch.cuda.current_stream(self.device)
                consumer.wait_event(pending[0])
                # the tensors were allocated on the copy stream: tell the caching allocator that the consumer stream uses them, or a
                # block freed by the consumer could be handed to the next H2D copy while kernels still read it (async inference paths)
                for t in (batch.z, batch.pos, batch.mol_ptr, batch.energy, batch.forces, batch.index):
                    if isinstance(t, torch.Tensor) and t.is_cuda:
                        t.record_stream(consumer)
            yield batch


# ------------------------------------------------------------------------------------------------------------------ Hamiltonian databases
def read_hamiltonian_db(path: str, include_overlap: bool = False) -> Dict[str, np.ndarray]:
    """All rows of an nablaDFT Hamiltonian database (`HamiltonianDatabase`, nablaDFT/dataset/hamiltonian_dataset.py:71-106): table `data`
    holds float32 / int32 blobs (Z, R, E, F, H, S, C); N atoms = len(R) / 12, Norb = sqrt(len(H) / 4).  Positions stay in the DB's unit
    (bohr, SURVEY.md section 8 units caveat) exactly as `PyGHamiltonianNablaDFT.get` passes them on (pyg_datasets.py:195-215).
    H (and S) are returned PACKED: one flat float32 array of all Norb x Norb matrices + `h_off` (offsets of each matrix), the layout the
    QHNet mirror produces (`QHNet.last_blocks`) and `losses.HamiltonianLoss.packed` consumes -- no block_diag over the batch
    (qhnet/qhnet.py:368-373 builds a dense [sum Norb]^2 target on the CPU every step)."""
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        n = con.execute("select N from metadata where id=0").fetchone()[0]
        rows = con.execute("select Z, R, E, F, H, S from data order by id").fetchall()
        ids = con.execute("select MOSES_ID, CONFORMER_ID from dataset_ids order by id").fetchall()
        basis = {int(zz): np.frombuffer(b, dtype=np.int32).copy() for zz, b in con.execute("select Z, orbitals from basisset").fetchall()}
    finally:
        con.close()
    if len(rows) != n:
        raise ValueError(f"{path}: metadata says {n} rows, data has {len(rows)}")
    z, pos, forces, energy, ptr, h, s, h_off, norb = [], [], [], [], [0], [], [], [0], []
    for Zb, Rb, E, Fb, Hb, Sb in rows:
        na = len(Rb) // 12
        zz = np.frombuffer(Zb, dtype=np.int32)
        if len(zz) != na:
            raise ValueError(f"{path}: Z / R length mismatch")
        no = int(round((len(Hb) // 4) ** 0.5))
        if no * no * 4 != len(Hb):
            raise ValueError(f"{path}: H blob is not a square float32 matrix")
        z.append(zz); pos.append(np.frombuffer(Rb, dtype=np.float32).reshape(na, 3))
        forces.append(np.frombuffer(Fb, dtype=np.float32).reshape(na, 3) if Fb is not None else np.zeros((na, 3), np.float32))
        energy.append(0.0 if E is None else E)
        h.append(np.frombuffer(Hb, dtype=np.float32))
        if include_overlap:
            s.append(np.frombuffer(Sb, dtype=np.float32))
        ptr.append(ptr[-1] + na); h_off.append(h_off[-1] + no * no); norb.append(no)
    out = {"z": np.concatenate(z).astype(np.int32), "pos": np.concatenate(pos), "forces": np.concatenate(forces),
           "energy": np.asarray(energy, dtype=np.float32), "ptr": np.asarray(ptr, dtype=np.int64), "H": np.concatenate(h),
           "h_off": np.asarray(h_off, dtype=np.int64), "norb": np.asarray(norb, dtype=np.int32),
           "moses_id": np.asarray([i[0] for i in ids], dtype=np.int64), "conformer_id": np.asarray([i[1] for i in ids], dtype=np.int64)}
    if include_overlap:
        out["S"] = np.concatenate(s)
    out["basis"] = basis  # {Z: orbital angular momenta}, the table config/model/qhnet.yaml:14-22 restates for def2-SVP
    return out


def read_hamiltonian_max_orbitals(path: str):
    """`max_orbitals` of a Hamiltonian database as `HamiltonianDataset.__init__` builds it (hamiltonian_dataset.py:331-335): one tuple of
    (Z, l) per entry of the `nuclear_charges` row, the l values from the `basisset` table.  PhiSNet's output layout is defined by it."""
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        if not con.execute("select name from sqlite_master where type='table' and name='nuclear_charges'").fetchone():
            return None  # older databases without the table: no PhiSNet layout
        zs = np.frombuffer(con.execute("select Z from nuclear_charges where id=0").fetchone()[0], dtype=np.int32)
        basis = {int(zz): np.frombuffer(b, dtype=np.int32) for zz, b in con.execute("select Z, orbitals from basisset").fetchall()}
    finally:
        con.close()
    return tuple(tuple((int(zz), int(l)) for l in basis[int(zz)]) for zz in zs)


class PackedHamiltonianDataset:
    """Z, R (bohr), H packed + offsets; `batch(indices, device)` returns what `QHNet.forward(data, keep_blocks=True)` and
    `HamiltonianLoss.packed` take: a data object (z, pos, batch, ptr) and the list of per-molecule target matrices on the device."""

    def __init__(self, arrays: Dict[str, np.ndarray]):
        self.a = arrays

    @classmethod
    def from_db(cls, path: str, include_overlap: bool = False) -> "PackedHamiltonianDataset":
        ds = cls(read_hamiltonian_db(path, include_overlap=include_overlap))
        ds.max_orbitals = read_hamiltonian_max_orbitals(path)
        return ds

    def __len__(self) -> int:
        return len(self.a["energy"])

    def hamiltonian(self, i: int) -> np.ndarray:
        no = int(self.a["norb"][i])
        return self.a["H"][int(self.a["h_off"][i]):int(self.a["h_off"][i + 1])].reshape(no, no)

    def phisnet_batch(self, indices, device="cuda"):
        """What `nabladft_b200.phisnet.NeuralNetwork.forward` takes, with the semantics of `HamiltonianDataset.collate_fn`
        (hamiltonian_dataset.py:354-405): `atoms_batch` = {positions [N,3] (bohr), atomic_numbers [N] int64, orbitals (one (Z, l) tuple per
        atom, from the basisset table), molecule_size [B] int64 (host)} on `device`, plus the packed targets: lists of the per-molecule H
        and S matrices on `device` instead of the reference's dense block diagonals.  Needs `from_db(path, include_overlap=True)`."""
        a, idx = self.a, np.asarray(indices, dtype=np.int64)
        if "S" not in a:
            raise ValueError("overlap matrices were not read: build the dataset with PackedHamiltonianDataset.from_db(path, include_overlap=True)")
        ptr, hoff = a["ptr"], a["h_off"]
        z = np.concatenate([a["z"][ptr[m]:ptr[m + 1]] for m in idx]).astype(np.int64)
        pos = np.concatenate([a["pos"][ptr[m]:ptr[m + 1]] for m in idx])
        dev = torch.device(device)
        orb = {zz: tuple((int(zz), int(l)) for l in ls) for zz, ls in a["basis"].items()}
        atoms_batch = {"positions": torch.from_numpy(pos).to(dev), "atomic_numbers": torch.from_numpy(z).to(dev),
                       "orbitals": tuple(orb[int(zz)] for zz in z), "molecule_size": torch.from_numpy(ptr[idx + 1] - ptr[idx])}
        mats = {}
        for key in ("H", "S"):
            mats[key] = [torch.from_numpy(a[key][hoff[m]:hoff[m + 1]].reshape(int(a["norb"][m]), int(a["norb"][m]))).to(dev) for m in idx]
        return atoms_batch, mats["H"], mats["S"]

    def batch(self, indices, device="cuda"):
        a, idx = self.a, np.asarray(indices, dtype=np.int64)
        ptr, hoff = a["ptr"], a["h_off"]
        counts = ptr[idx + 1] - ptr[idx]
        z = torch.from_numpy(np.concatenate([a["z"][ptr[m]:ptr[m + 1]] for m in idx]))
        pos = torch.from_numpy(np.concatenate([a["pos"][ptr[m]:ptr[m + 1]] for m in idx]))
        h_flat = torch.from_numpy(np.concatenate([a["H"][hoff[m]:hoff[m + 1]] for m in idx]))
        dev = torch.device(device)
        if dev.type == "cuda":
            z, pos, h_flat = z.pin_memory(), pos.pin_memory(), h_flat.pin_memory()
        z, pos, h_flat = z.to(dev, non_blocking=True), pos.to(dev, non_blocking=True), h_flat.to(dev, non_blocking=True)

        class _Data:
            pass

        d = _Data()
        d.z, d.pos = z.long(), pos
        d.ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)).to(dev)
        d.batch = torch.repeat_interleave(torch.arange(len(idx), device=dev), torch.from_numpy(counts).to(dev))
        d.num_graphs = len(idx)
        targets, o = [], 0
        for m in idx:
            no = int(a["norb"][m])
            targets.append(h_flat[o:o + no * no].view(no, no))
            o += no * no
        return d, targets
