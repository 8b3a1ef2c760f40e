"""Golden outputs of the whole PhiSNet model: the REFERENCE'S OWN `NeuralNetwork` (`nablaDFT/phisnet/nn/neural_network.py`, unmodified;
torch, numpy and scipy only) run in float64 at the shipped hyperparameters (`phisnet/configs/args_nablaDFT_*.txt`) on a two-molecule batch cut
from fixture molecule 0 of tests/golden/hamiltonian_mol0.db.  The `nn` package is loaded by file path under a synthetic package name, as
make_golden_phisnet.py does for the layer modules, so `nablaDFT/__init__.py` never runs.

`max_orbitals` is built from the DB the way `HamiltonianDataset.__init__` does (hamiltonian_dataset.py:331-335): one orbital tuple per entry of
the `nuclear_charges` row, orbitals from the `basisset` table.

Weights are name-keyed and seeded (`model_state_dict` below, imported by the tests): no path is degenerate -- the zero-initialised output
layers and second residual linears get non-zero values, swish alpha / beta stay near 1 and 1.702, buffers keep their constructor values.

Writes tests/golden/phisnet_model.npz:
  positions, atomic_numbers, molecule_size        the batch (bohr; fragments A = atoms 0-9 + 22-25, B = atoms 14-21 + 26-27 of molecule 0)
  {full,core,over}/{0,1}                          upper triangle (np.triu_indices) of each molecule's diagonal block, float64
  electron_config                                 the reference's [87, 16] table (Embedding buffer)
  state_keys, state_shapes                        the reference's state-dict keys (sorted) and their shapes, CG buffers excluded
  pindex/{n}/{i,j}                                the reference's pindex_dict entries for the two molecule sizes

    python tests/golden/make_golden_phisnet_model.py
"""
import importlib
import os
import sqlite3
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
NN_DIR = "/root/reference/nablaDFT/phisnet/nn"
DB = os.path.join(HERE, "hamiltonian_mol0.db")

# args_nablaDFT_*.txt
HYPER = dict(order=4, num_features=128, num_basis_functions=128, num_modules=5, num_residual_pre_x=1, num_residual_post_x=1,
             num_residual_pre_vi=1, num_residual_pre_vj=1, num_residual_post_v=1, num_residual_output=1, num_residual_pc=1,
             num_residual_pn=1, num_residual_ii=1, num_residual_ij=1, num_residual_full_ii=2, num_residual_full_ij=2,
             num_residual_core_ii=2, num_residual_core_ij=2, num_residual_over_ij=2, basis_functions="exp-bernstein", cutoff=15.0,
             activation="swish")
FRAGMENTS = (list(range(0, 10)) + list(range(22, 26)), list(range(14, 22)) + [26, 27])


def max_orbitals_from_db(path=DB):
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        zs = np.frombuffer(con.execute("select Z from nuclear_charges where id=0").fetchone()[0], dtype=np.int32)
        basis = {int(z): np.frombuffer(b, dtype=np.int32) for z, b in con.execute("select Z, orbitals from basisset").fetchall()}
    finally:
        con.close()
    return tuple(tuple((int(z), int(l)) for l in basis[int(z)]) for z in zs)


def fixture_batch(path=DB):
    """(positions [N,3] bohr float64, atomic_numbers [N] int64, molecule_size [2]) of the two fragments of molecule 0."""
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        zb, rb = con.execute("select Z, R from data order by id limit 1").fetchone()
    finally:
        con.close()
    z = np.frombuffer(zb, dtype=np.int32).astype(np.int64)
    r = np.frombuffer(rb, dtype=np.float32).reshape(-1, 3).astype(np.float64)
    idx = np.concatenate([np.asarray(f) for f in FRAGMENTS])
    return r[idx], z[idx], np.asarray([len(f) for f in FRAGMENTS], dtype=np.int64)


def model_state_dict(template):
    """name -> float64 array for every parameter / buffer name in `template` (name -> tensor); values depend on the name only."""
    out = {}
    for name, ref in template.items():
        shape, leaf = tuple(ref.shape), name.rsplit(".", 1)[-1]
        if "clebsch_gordan" in name or leaf in ("electron_config", "cutoff", "logc", "n", "v", "_alpha"):
            out[name] = ref.detach().double().numpy().copy()  # buffers and the RBF width keep their constructor values
            continue
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        if leaf == "alpha":
            w = 1.0 + 0.1 * rng.standard_normal(shape)
        elif leaf == "beta":
            w = 1.702 + 0.1 * rng.standard_normal(shape)
        elif leaf.startswith(("keepcoeff", "mixcoeff")):
            w = rng.uniform(-0.6, 0.6, size=shape)
        elif leaf == "element_embedding":
            w = rng.uniform(-np.sqrt(3.0), np.sqrt(3.0), size=shape)
        elif len(shape) == 2:
            bound = np.sqrt(6.0 / (shape[0] + shape[1]))
            w = rng.uniform(-bound, bound, size=shape)
        else:
            w = 0.05 * rng.standard_normal(shape)
        out[name] = np.asarray(w, dtype=np.float64).reshape(shape)
    return out


def ref_nn():
    pkg = types.ModuleType("refphisnn")
    pkg.__path__ = [NN_DIR]
    sys.modules["refphisnn"] = pkg
    return importlib.import_module("refphisnn.neural_network")


def main():
    nnmod = ref_nn()
    max_orb = max_orbitals_from_db()
    torch.manual_seed(0)
    net = nnmod.NeuralNetwork(max_orbitals=max_orb, **HYPER).double()
    sd = net.state_dict()
    vals = model_state_dict(sd)
    net.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in vals.items()}, strict=True)
    net.eval()
    pos, z, ms = fixture_batch()
    orbitals = tuple(dict((o[0][0], o) for o in max_orb)[int(zz)] for zz in z)
    batch = {"positions": torch.from_numpy(pos), "atomic_numbers": torch.from_numpy(z), "orbitals": orbitals,
             "molecule_size": torch.from_numpy(ms)}
    res = net(batch)
    out = {"positions": pos, "atomic_numbers": z, "molecule_size": ms}
    norb = [sum(2 * l + 1 for _, l in orbitals[i]) for i in range(len(z))]
    a0, o0 = 0, 0
    for m, n in enumerate(ms):
        no = sum(norb[a0:a0 + n])
        iu = np.triu_indices(no)
        for tag, key in (("full", "full_hamiltonian"), ("core", "core_hamiltonian"), ("over", "overlap_matrix")):
            blk = res[key][0, o0:o0 + no, o0:o0 + no].detach().numpy()
            out[f"{tag}/{m}"] = blk[iu]
            print(f"mol {m}: {tag:4s} norb {no}  max|.| {np.abs(blk).max():.4g}  rms {np.sqrt((blk ** 2).mean()):.4g}")
        a0, o0 = a0 + n, o0 + no
    out["electron_config"] = net.embedding.embedding.electron_config.numpy().astype(np.float64)
    keys = sorted(k for k in sd if "clebsch_gordan.cg_" not in k)
    out["state_keys"] = np.asarray(keys)
    out["state_shapes"] = np.asarray([",".join(str(s) for s in sd[k].shape) for k in keys])
    for n in sorted(set(int(s) for s in ms)):
        pi, pj = net.idx_pdict[n]
        out[f"pindex/{n}/i"], out[f"pindex/{n}/j"] = np.asarray(pi, dtype=np.int32), np.asarray(pj, dtype=np.int32)
    np.savez_compressed(os.path.join(HERE, "phisnet_model.npz"), **out)
    print("wrote phisnet_model.npz:", len(out), "arrays,", os.path.getsize(os.path.join(HERE, "phisnet_model.npz")), "bytes")


if __name__ == "__main__":
    main()
