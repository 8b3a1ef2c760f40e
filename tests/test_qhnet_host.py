"""Host-side QHNet checks that need no GPU: the generated tensor-product source is what tools/gen_qhnet_tp.py makes from oracle/e3.py
today, and batches or settings the kernels cannot handle are refused before any CUDA call."""
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_qhnet import ORBITALS, _Data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tp_source_matches_generator(tmp_path):
    """qhnet_tp_gen.inc unrolls every Clebsch-Gordan coefficient and path normalisation as a literal: regenerating it from the oracle must
    give the committed file byte for byte, so the kernels cannot drift from oracle/e3.py."""
    out = tmp_path / "qhnet_tp_gen.inc"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_qhnet_tp.py"), str(out)], check=True, cwd=tmp_path, capture_output=True)
    with open(os.path.join(ROOT, "nabladft_b200", "csrc", "qhnet_tp_gen.inc"), "rb") as f:
        committed = f.read()
    assert out.read_bytes() == committed, "qhnet_tp_gen.inc is stale: rerun tools/gen_qhnet_tp.py"


@pytest.fixture(scope="module")
def net():
    from nabladft_b200.qhnet import QHNet

    return QHNet(num_nodes=83, orbitals=ORBITALS).eval()


@pytest.mark.parametrize("bad", [15, 50, 83, 200, -1], ids=["not-in-table", "past-table", "num_nodes", "past-num_nodes", "negative"])
def test_forward_refuses_unsupported_elements(net, bad):
    """Z = 15 has an embedding row but no orbitals (it would vanish from H); 50 lies past the orbital table; 83 and 200 have no embedding
    row; -1 is no element.  Each is refused with a ValueError that names it, before the CUDA-only check."""
    z = torch.tensor([6, 1, bad, 1])
    data = _Data(z, torch.randn(4, 3), torch.zeros(4, dtype=torch.long))
    with pytest.raises(ValueError, match=f"\\[{bad}\\]"):
        net(data)


def test_forward_accepts_table_elements_up_to_cuda_check(net):
    from nabladft_b200._lib import NablaB200Error

    z = torch.tensor(sorted(ORBITALS))
    data = _Data(z, torch.randn(len(z), 3), torch.zeros(len(z), dtype=torch.long))
    with pytest.raises(NablaB200Error, match="CUDA only"):
        net(data)


@pytest.mark.parametrize("value", ["0", "-3"])
def test_pair_chunk_must_be_positive(monkeypatch, net, value):
    """NB200_QH_PAIR_CHUNK = 0 used to fail in range(); a negative value skipped the pair loops and left H uninitialised."""
    from nabladft_b200.qhnet import QHNet

    monkeypatch.setenv("NB200_QH_PAIR_CHUNK", value)
    with pytest.raises(ValueError, match="NB200_QH_PAIR_CHUNK"):
        QHNet(num_nodes=83, orbitals=ORBITALS)
    monkeypatch.setattr(net, "pair_chunk", int(value))
    z = torch.tensor([6, 1])
    with pytest.raises(ValueError, match="pair_chunk"):
        net(_Data(z, torch.randn(2, 3), torch.zeros(2, dtype=torch.long)))
