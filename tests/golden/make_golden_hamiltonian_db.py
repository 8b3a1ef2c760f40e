"""Shrunk copy of the reference's Hamiltonian fixture database (`tests/data/raw/test_hamiltonian_database.db` of the reference
checkout, 25 molecules, 30 MB) for tests/test_data.py: the same schema and blob layout, molecule 0 only (38 atoms, 396 orbitals), its
overlap blob S set NULL, the metadata row count set to 1; the basisset, nuclear_charges and information tables copied whole.

    python tests/golden/make_golden_hamiltonian_db.py [path/to/test_hamiltonian_database.db]   # writes tests/golden/hamiltonian_mol0.db
"""
import os
import sqlite3
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "hamiltonian_mol0.db")


def main(src):
    if os.path.exists(OUT):
        os.remove(OUT)
    s = sqlite3.connect(f"file:{src}?mode=ro", uri=True)
    d = sqlite3.connect(OUT)
    for (sql,) in s.execute("select sql from sqlite_master where sql is not null and name not like 'sqlite_%' order by rowid"):
        d.execute(sql)
    row = s.execute("select id, Z, R, E, F, H, C from data where id = 0").fetchone()
    d.execute("insert into data (id, Z, R, E, F, H, S, C) values (?, ?, ?, ?, ?, ?, NULL, ?)", row)
    d.execute("insert into dataset_ids (id, MOSES_ID, CONFORMER_ID) values (?, ?, ?)", s.execute("select id, MOSES_ID, CONFORMER_ID from dataset_ids where id = 0").fetchone())
    d.execute("insert into metadata (id, N) values (0, 1)")
    for table in ("basisset", "nuclear_charges", "information"):
        rows = s.execute(f"select * from {table}").fetchall()
        if rows:
            d.executemany(f"insert into {table} values ({', '.join('?' * len(rows[0]))})", rows)
    d.commit()
    d.execute("vacuum")
    d.close()
    s.close()
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests/data/raw/test_hamiltonian_database.db")
