"""GPU parity tests for the QHNet kernels (C ABI) against the CPU oracle (oracle/qhnet.py, oracle/e3.py),
op by op and end to end (Hamiltonian blocks within 1e-6 Ha, the north-star tolerance)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_golden_weights

pytestmark = pytest.mark.gpu

ORBITALS = {1: [0, 0, 1], 6: [0, 0, 0, 1, 1, 2], 7: [0, 0, 0, 1, 1, 2], 8: [0, 0, 0, 1, 1, 2], 9: [0, 0, 0, 1, 1, 2],
            16: [0, 0, 0, 0, 1, 1, 1, 2], 17: [0, 0, 0, 0, 1, 1, 1, 2], 35: [0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2]}
H_TOL = 1e-6  # Ha, Hamiltonian blocks (BASELINE.json north_star)
DEV = "cuda:0"


def to_cm(flat, c=128):
    """e3nn flat [R, 25c] (per l: [mul, 2l+1]) -> component-major [R, 25, c]."""
    R, out, off = flat.shape[0], [], 0
    for l in range(5):
        n = c * (2 * l + 1)
        out.append(flat[:, off:off + n].reshape(R, c, 2 * l + 1).permute(0, 2, 1))
        off += n
    return torch.cat(out, dim=1).contiguous()


def from_cm(cm):
    R, _, c = cm.shape
    out, lm = [], 0
    for l in range(5):
        out.append(cm[:, lm:lm + 2 * l + 1, :].permute(0, 2, 1).reshape(R, -1))
        lm += 2 * l + 1
    return torch.cat(out, dim=1)


@pytest.fixture(scope="module")
def models():
    from nabladft_b200.qhnet import QHNet
    from oracle.qhnet import QHNetOracle

    torch.set_default_dtype(torch.float64)
    try:
        ora = load_golden_weights(QHNetOracle(orbitals=ORBITALS), torch.float64, style="e3").eval()
    finally:
        torch.set_default_dtype(torch.float32)
    net = QHNet(sh_lmax=4, hidden_size=128, bottle_hidden_size=32, num_gnn_layers=5, max_radius=12, num_nodes=83, radius_embed_dim=32,
                orbitals=ORBITALS)
    sd_o = ora.state_dict()
    sd_n = net.state_dict()
    assert set(sd_o.keys()) == set(sd_n.keys()), set(sd_o.keys()) ^ set(sd_n.keys())
    net.load_state_dict({k: v.float() for k, v in sd_o.items()}, strict=True)
    return ora, net.eval().to(DEV)


class _Data:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch
        counts = torch.bincount(batch)
        self.ptr = torch.zeros(counts.numel() + 1, dtype=torch.long, device=z.device)
        self.ptr[1:] = torch.cumsum(counts, 0)
        self.num_nodes = z.shape[0]


def _small(n=14):
    g = np.load(os.path.join(GOLDEN, "qhnet_f64.npz"))
    return torch.from_numpy(g["a.z"])[:n], torch.from_numpy(g["a.pos"])[:n], torch.from_numpy(g["a.batch"])[:n]


def test_qh_linear_tall_rows_pre_split_path(models):
    """o3.Linear over >= 2048 rows takes the pre-split-weight kernel batched over the 25 (l,m) slices (gemm_ps.cu::nb_gemm_ps_lm):
    per-pair features of config 4 (1e5 rows).  Checked against the float64 product with the exported per-order weights, 128 -> 128
    (with the residual accumulate) and 128 -> 32 (a quarter of an output tile, bias on the l = 0 slice)."""
    _, net = models
    w = net._export(torch.device(DEV))
    o = net._ops(torch.device(DEV))
    g = torch.Generator().manual_seed(5)
    R = 2300
    l_of = [0] + [1] * 3 + [2] * 5 + [3] * 7 + [4] * 9
    for name, wl, acc in (("pair.out", w["pair"][0]["out"], True), ("out_ij", w["out_ij"], False)):
        Wl, b = wl
        c_in, c_out = Wl.shape[1], Wl.shape[2]
        x = torch.randn(R, 25, c_in, generator=g).to(DEV)
        y0 = torch.randn(R, 25, c_out, generator=g).to(DEV)
        y = o.linear(x, wl, accumulate_into=y0.clone() if acc else None)
        torch.cuda.synchronize()
        ref = torch.stack([x[:, lm].double() @ Wl[l_of[lm]].double() for lm in range(25)], dim=1)
        if b is not None:
            ref[:, 0] += b.double()
        if acc:
            ref += y0.double()
        err = (y.double() - ref).abs().max().item() / ref.abs().max().item()
        print(f"qh_linear tall {name} [{R} x 25 x {c_in}] -> {c_out}: rel err {err:.2e}")
        assert err < 2e-6


def test_qhnet_blocks_and_matrix_match_oracle(models):
    ora, net = models
    z, pos, batch = _small(14)
    with torch.no_grad():
        d_ref, o_ref, fdst, fsrc = ora.blocks(z, pos, batch)
        H_ref = ora.assemble(z, batch, d_ref, o_ref, fdst, fsrc)
    data = _Data(z.to(DEV), pos.float().to(DEV), batch.to(DEV))
    H = net(data)
    blocks = net(data, keep_blocks=True)
    d_sym = d_ref + d_ref.transpose(-1, -2)
    print("max |H| ref", float(H_ref.abs().max()), "dH", float((H.cpu().double() - H_ref).abs().max()),
          "d diag blocks", float((blocks["hamiltonian_diagonal_blocks"].cpu().double() - d_sym).abs().max()))
    assert H.shape == H_ref.shape
    assert (blocks["hamiltonian_diagonal_blocks"].cpu().double() - d_sym).abs().max() < H_TOL
    assert (H.cpu().double() - H_ref).abs().max() < H_TOL
    assert float((H - H.T).abs().max()) == 0.0


def test_qhnet_matches_reference_golden_and_batches(models):
    """Full molecule vs the golden H produced by the reference's own classes; 2-molecule batch is block diagonal."""
    ora, net = models
    g = np.load(os.path.join(GOLDEN, "qhnet_f64.npz"))
    data = _Data(torch.from_numpy(g["a.z"]).to(DEV), torch.from_numpy(g["a.pos"]).float().to(DEV), torch.from_numpy(g["a.batch"]).to(DEV))
    H = net(data)
    err = np.abs(H.cpu().numpy() - g["a.H"]).max()
    print("golden: max|H|", np.abs(g["a.H"]).max(), "max err", err)
    assert err < H_TOL
    datab = _Data(torch.from_numpy(g["b.z"]).to(DEV), torch.from_numpy(g["b.pos"]).float().to(DEV), torch.from_numpy(g["b.batch"]).to(DEV))
    Hb = net(datab)
    n = H.shape[0]
    assert float(Hb[:n, n:].abs().max()) == 0.0 and (Hb[:n, :n] - H).abs().max() < 1e-7
    assert np.abs(Hb.sum(1).cpu().numpy() - g["b.H_rowsum"]).max() < 2e-5


def test_qhnet_full_size_properties_cfg4(models):
    """BASELINE configs[3] size (64 synthetic molecules in bohr, ~2.5 k atoms, ~10^5 ordered pairs): size-independent properties.
    (1) every molecule's H is symmetric; (2) bitwise determinism; (3) a molecule's H does not depend on its batch mates or on its
    position in the batch; (4) SO(3) equivariance: rotating a molecule transforms H by a block-diagonal orthogonal matrix (real
    Wigner-D per shell), so the eigenvalue spectrum of each molecule's H is invariant."""
    from helpers import random_rotation
    from nabladft_b200.synth import synth_batch

    _, net = models
    b = synth_batch(3, 64)
    z = torch.from_numpy(b["z"]).to(DEV)
    pos = (torch.from_numpy(b["pos"]) * 1.8897261).to(DEV)
    batch = torch.from_numpy(b["batch"]).to(DEV)
    H0 = [h.clone() for h in net(_Data(z, pos, batch), packed=True)]
    assert len(H0) == 64 and all(float((h - h.T).abs().max()) == 0.0 for h in H0)          # M + M^T assembled exactly
    assert all(torch.equal(a, c) for a, c in zip(H0, net(_Data(z, pos, batch), packed=True)))   # deterministic
    # molecules 5..9 alone, reversed order
    ptr = b["mol_ptr"]
    sel = [9, 8, 7, 6, 5]
    idx = torch.cat([torch.arange(int(ptr[m]), int(ptr[m + 1])) for m in sel]).to(DEV)
    sub_batch = torch.repeat_interleave(torch.arange(len(sel)), torch.tensor([int(ptr[m + 1] - ptr[m]) for m in sel])).to(DEV)
    sub = net(_Data(z[idx], pos[idx], sub_batch), packed=True)
    for k, m in enumerate(sel):
        assert float((sub[k] - H0[m]).abs().max()) < 2e-6                                   # fp32 reduction order inside kernels only
    # rotation + translation of the whole batch
    R = random_rotation(11, torch.float32).to(DEV)
    Hr = net(_Data(z, pos @ R.T + 0.7, batch), packed=True)
    for m in (0, 17, 63):
        ev0 = torch.linalg.eigvalsh(H0[m].double())
        ev1 = torch.linalg.eigvalsh(Hr[m].double())
        assert float((ev0 - ev1).abs().max()) < 5e-5 * max(1.0, float(ev0.abs().max()))
        assert float((Hr[m] - H0[m]).abs().max()) > 1e-4                                    # ... while H itself does change


def test_qhnet_cfg4_slice_values_match_oracle(models):
    """VALUE parity at config size (VERDICT r1 item 2): the 64-molecule synthetic batch of BASELINE configs[3] runs on the device, and the
    Hamiltonians of its first molecules are compared entry by entry with a float64 oracle pass on those molecules alone (molecules do not
    interact; the oracle takes ~10 s per molecule, hence 3 of them).  Tolerance: north_star's 1e-6 Ha on Hamiltonian blocks."""
    from nabladft_b200.synth import synth_batch

    ora, net = models
    b = synth_batch(3, 64)
    z = torch.from_numpy(b["z"])
    pos = torch.from_numpy(b["pos"]).double() * 1.8897261
    batch = torch.from_numpy(b["batch"])
    H = net(_Data(z.to(DEV), pos.float().to(DEV), batch.to(DEV)), packed=True)
    ptr = b["mol_ptr"]
    worst, hmax = 0.0, 0.0
    for m in range(3):
        a0, a1 = int(ptr[m]), int(ptr[m + 1])
        zm, pm, bm = z[a0:a1], pos[a0:a1], torch.zeros(a1 - a0, dtype=torch.long)
        with torch.no_grad():
            d_ref, o_ref, fdst, fsrc = ora.blocks(zm, pm, bm)
            H_ref = ora.assemble(zm, bm, d_ref, o_ref, fdst, fsrc)
        assert H[m].shape == H_ref.shape
        worst = max(worst, float((H[m].double().cpu() - H_ref).abs().max()))
        hmax = max(hmax, float(H_ref.abs().max()))
    print(f"cfg 4 slice: 3 of 64 molecules, max|dH| {worst:.2e} Ha (max|H| {hmax:.2f})")
    assert worst < H_TOL
