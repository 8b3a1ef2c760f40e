"""PackedHamiltonianDataset.phisnet_batch against HamiltonianDataset.collate_fn semantics (hamiltonian_dataset.py:354-405), restated here from
the fixture database tests/golden/hamiltonian_mol0.db with plain sqlite: per-atom orbital tuples from the basisset table, max_orbitals from
the nuclear_charges row, concatenated positions / numbers, molecule sizes and the H / S matrices of each molecule."""
import os
import shutil
import sqlite3

import numpy as np
import torch

from helpers import GOLDEN

from nabladft_b200.data import PackedHamiltonianDataset

DB = os.path.join(GOLDEN, "hamiltonian_mol0.db")


def with_overlap(tmp_path):
    """The fixture stores no S: a copy gets a symmetric float32 S per row so that the overlap targets are exercised."""
    path = str(tmp_path / "ham_s.db")
    shutil.copy(DB, path)
    con = sqlite3.connect(path)
    rng = np.random.default_rng(0)
    for rid, hb in con.execute("select id, H from data").fetchall():
        n = int(round((len(hb) // 4) ** 0.5))
        a = rng.standard_normal((n, n)).astype(np.float32)
        con.execute("update data set S = ? where id = ?", ((a + a.T).tobytes(), rid))
    con.commit()
    con.close()
    return path


def raw(path):
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    try:
        rows = con.execute("select Z, R, H, S from data order by id").fetchall()
        basis = {int(z): np.frombuffer(b, dtype=np.int32) for z, b in con.execute("select Z, orbitals from basisset").fetchall()}
        zs = np.frombuffer(con.execute("select Z from nuclear_charges where id=0").fetchone()[0], dtype=np.int32)
    finally:
        con.close()
    return rows, basis, zs


def test_phisnet_batch_follows_collate_fn(tmp_path):
    path = with_overlap(tmp_path)
    rows, basis, zs = raw(path)
    ds = PackedHamiltonianDataset.from_db(path, include_overlap=True)
    assert ds.max_orbitals == tuple(tuple((int(z), int(l)) for l in basis[int(z)]) for z in zs)
    idx = [0, 0]  # the fixture holds one molecule; a batch of two copies exercises the concatenation
    ab, H, S = ds.phisnet_batch(idx, device="cpu")
    Zs = [np.frombuffer(rows[m][0], dtype=np.int32) for m in idx]
    Rs = [np.frombuffer(rows[m][1], dtype=np.float32).reshape(-1, 3) for m in idx]
    assert torch.equal(ab["atomic_numbers"], torch.from_numpy(np.concatenate(Zs)).long())
    assert torch.equal(ab["positions"], torch.from_numpy(np.concatenate(Rs)))
    assert ab["molecule_size"].tolist() == [len(z) for z in Zs]
    assert ab["orbitals"] == tuple(tuple((int(z), int(l)) for l in basis[int(z)]) for zz in Zs for z in zz)
    for k, m in enumerate(idx):
        n = int(round((len(rows[m][2]) // 4) ** 0.5))
        assert n == sum(2 * l + 1 for o in ab["orbitals"][:len(Zs[0])] for _, l in o)
        assert torch.equal(H[k], torch.from_numpy(np.frombuffer(rows[m][2], dtype=np.float32).reshape(n, n)))
        assert torch.equal(S[k], torch.from_numpy(np.frombuffer(rows[m][3], dtype=np.float32).reshape(n, n)))
