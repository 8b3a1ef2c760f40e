"""GPU parity tests (run on an H100 with `-m gpu`): every call goes through the C ABI
(libnabla_b200.so) and is compared with the CPU oracle / the golden vectors generated from
the reference's own code.  Tolerances are the north-star ones: |dE| <= 1e-5 Ha, |dF| <= 1e-4
Ha/A (fp32 path vs fp64 oracle), written next to each assert."""
import ctypes
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_fixture, load_golden_weights, random_rotation

pytestmark = pytest.mark.gpu

E_TOL = 1e-5  # Ha
F_TOL = 1e-4  # Ha/A


def dev():
    return torch.device("cuda:0")


def _graph(pos, mol_ptr, cutoff=5.0, max_nb=100, e_cap=None):
    from nabladft_b200 import _lib

    lib = _lib.load()
    N, B = pos.shape[0], mol_ptr.numel() - 1
    e_cap = e_cap or N * 64
    d = pos.device
    row_ptr = torch.zeros(N + 1, dtype=torch.int32, device=d)
    col = torch.zeros(e_cap, dtype=torch.int32, device=d)
    rev = torch.zeros(e_cap, dtype=torch.int32, device=d)
    geom = torch.zeros(e_cap, 4, dtype=torch.float32, device=d)
    deg = torch.zeros(N, dtype=torch.int32, device=d)
    status = torch.zeros(4, dtype=torch.int32, device=d)
    rc = lib.nb200_neighbor_build(_lib.ptr(pos), _lib.ptr(mol_ptr), B, N, cutoff, max_nb, e_cap, _lib.ptr(row_ptr), _lib.ptr(col),
                                  _lib.ptr(rev), _lib.ptr(geom), _lib.ptr(deg), _lib.ptr(status), _lib.current_stream())
    _lib.check(rc, "nb200_neighbor_build")
    torch.cuda.synchronize()
    return row_ptr, col, rev, geom, status


def _fixture_cuda(mols):
    z, pos, batch = load_fixture(mols, torch.float32)
    from nabladft_b200.engine import mol_ptr_from_batch

    mol_ptr, n_mol = mol_ptr_from_batch(batch)
    return z, pos, batch, mol_ptr, n_mol


def test_neighbor_build_matches_oracle_bit_exact_indices():
    from oracle.graph import radius_graph

    z, pos, batch, mol_ptr, n_mol = _fixture_cuda([0, 1, 2, 50])
    row_ptr, col, rev, geom, status = _graph(pos.to(dev()), mol_ptr.to(dev()))
    ei = radius_graph(pos.double(), 5.0, batch, 10**9)
    E = ei.shape[1]
    st = status.cpu().tolist()
    assert st[0] == E and st[1] == 0 and st[3] == 0
    row_ptr, col, rev, geom = row_ptr.cpu().long(), col.cpu().long()[:E], rev.cpu().long()[:E], geom.cpu()[:E]
    tgt = torch.repeat_interleave(torch.arange(pos.shape[0]), row_ptr[1:] - row_ptr[:-1])
    assert torch.equal(col, ei[0]) and torch.equal(tgt, ei[1])  # same edges, same (target-major, source-ascending) order
    assert torch.equal(col[rev], tgt) and torch.equal(tgt[rev], col) and torch.equal(rev[rev], torch.arange(E))
    r = pos.double()[col] - pos.double()[tgt]
    d = r.norm(dim=1)
    assert (geom[:, 3].double() - d).abs().max() < 1e-6
    assert (geom[:, :3].double() - r / d[:, None]).abs().max() < 1e-6
    assert st[2] == int((row_ptr[1:] - row_ptr[:-1]).max())


def test_neighbor_build_error_flags():
    z, pos, batch, mol_ptr, n_mol = _fixture_cuda([0, 1])
    _, _, _, _, status = _graph(pos.to(dev()), mol_ptr.to(dev()), e_cap=100)
    assert status.cpu().tolist()[1] == -4  # NB200_ECAPACITY, nothing written out of bounds
    row_ptr, _, _, _, status = _graph(pos.to(dev()), mol_ptr.to(dev()), max_nb=5)
    assert status.cpu().tolist()[1] == -5 and int(row_ptr.abs().sum()) == 0  # NB200_ENEIGHBORS, rows emptied


def _filter(geom, status, e_cap, t, s, with_dw=True):
    from nabladft_b200 import _lib

    lib = _lib.load()
    L, K, F = s["n_layers"], s["n_rbf"], s["n_feat"]
    d = geom.device
    W = torch.zeros(L, e_cap, 3 * F, dtype=torch.float32, device=d)
    dW = torch.zeros_like(W) if with_dw else None
    scr = torch.zeros(e_cap + 1024, dtype=torch.int32, device=d)
    rc = lib.nb200_painn_filter(_lib.ptr(geom), _lib.ptr(status), e_cap, _lib.ptr(t["w_rbf"]), _lib.ptr(t["b_rbf"]), L, K, F,
                                s["radial_mode"], s["cutoff"], _lib.ptr(t["rbf_offsets"]), s["rbf_coeff"], s["rbf_xscale"],
                                _lib.ptr(W), _lib.ptr(dW), _lib.ptr(scr), _lib.current_stream())
    _lib.check(rc, "nb200_painn_filter")
    torch.cuda.synchronize()
    return W, dW


def _oc_model(num_layers=6):
    from nabladft_b200.painn_oc import PaiNN

    net = PaiNN(hidden_channels=128, num_layers=num_layers, num_rbf=100, cutoff=5.0, max_neighbors=100, direct_forces=False,
                use_pbc=False, num_elements=100)
    return load_golden_weights(net, torch.float32).eval()


def _spk_model(n_interactions=6):
    from nabladft_b200 import spk

    m = spk.NeuralNetworkPotential(
        representation=spk.PaiNN(n_atom_basis=128, n_interactions=n_interactions, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                 cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()],
        output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()],
        postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32)
    m.postprocessors[0].mean.fill_(-0.01)
    return m.eval()


@pytest.mark.parametrize("kind", ["oc", "spk"])
def test_filter_kernel_matches_dense_fp64(kind):
    """Banded register-blocked filter == dense fp64 phi @ W (+ analytic dW/dd == autograd)."""
    import math

    z, pos, batch, mol_ptr, n_mol = _fixture_cuda([3, 4])
    row_ptr, col, rev, geom, status = _graph(pos.to(dev()), mol_ptr.to(dev()))
    E = int(status[0])
    model = _oc_model(2).to(dev()) if kind == "oc" else _spk_model(2).to(dev())
    t, s = model._export() if kind == "oc" else model._export(True)
    W, dW = _filter(geom, status, geom.shape[0], t, s)
    d = geom[:E, 3].double().cpu().requires_grad_(True)
    x = d * s["rbf_xscale"]
    phi = torch.exp(s["rbf_coeff"] * (x[:, None] - t["rbf_offsets"].double().cpu()[None]) ** 2)
    if kind == "spk":
        s1 = 0.5 * (torch.cos(d * math.pi / s["cutoff"]) + 1)
        s2 = s1
    else:
        xs = d / s["cutoff"]
        s1 = 1 - 21 * xs**5 + 35 * xs**6 - 15 * xs**7
        s2 = torch.ones_like(s1)
    for l in range(2):
        ref = s1[:, None] * (phi @ t["w_rbf"][l].double().cpu()) + s2[:, None] * t["b_rbf"][l].double().cpu()
        assert (W[l, :E].double().cpu() - ref.detach()).abs().max() < 2e-6
        # derivative: check 8 random channels by autograd
        for ch in (0, 5, 127, 128, 200, 255, 300, 383):
            g = torch.autograd.grad(ref[:, ch].sum(), d, retain_graph=True)[0]
            assert (dW[l, :E, ch].double().cpu() - g).abs().max() < 5e-5


def test_msg_fwd_bwd_match_autograd():
    """K_msg forward vs the oracle formula, and its analytic backward vs fp64 autograd
    (gradients w.r.t. xh, mu, and -- through u and d -- positions)."""
    from nabladft_b200 import _lib

    lib = _lib.load()
    torch.manual_seed(0)
    z, pos, batch, mol_ptr, n_mol = _fixture_cuda([7, 8])
    N, F = pos.shape[0], 128
    row_ptr, col, rev, geom, status = _graph(pos.to(dev()), mol_ptr.to(dev()))
    E = int(status[0])
    model = _oc_model(1).to(dev())
    t, s = model._export()
    W, dW = _filter(geom, status, geom.shape[0], t, s)
    xh = torch.randn(N, 3 * F, device=dev()) * 0.5
    bias = torch.randn(3 * F, device=dev()) * 0.1
    q = torch.randn(N, F, device=dev())
    mu = torch.randn(N, 3, F, device=dev()) * 0.5
    q_out, mu_out = torch.empty_like(q), torch.empty_like(mu)
    _lib.check(lib.nb200_painn_msg_fwd(_lib.ptr(xh), _lib.ptr(bias), _lib.ptr(q), _lib.ptr(mu), _lib.ptr(W[0]), _lib.ptr(geom),
                                       _lib.ptr(row_ptr), _lib.ptr(col), N, _lib.ptr(q_out), _lib.ptr(mu_out), _lib.current_stream()), "msg_fwd")
    gq = torch.randn(N, F, device=dev())
    gmu = torch.randn(N, 3, F, device=dev())
    g_xh, g_mu_in = torch.empty_like(xh), torch.empty_like(mu)
    egrad = torch.zeros(geom.shape[0], 4, device=dev())
    forces = torch.empty(N, 3, device=dev())
    _lib.check(lib.nb200_painn_msg_bwd(_lib.ptr(xh), _lib.ptr(bias), _lib.ptr(mu), _lib.ptr(W[0]), _lib.ptr(dW[0]), _lib.ptr(geom),
                                       _lib.ptr(row_ptr), _lib.ptr(col), N, _lib.ptr(gq), _lib.ptr(gmu), _lib.ptr(g_xh), _lib.ptr(g_mu_in),
                                       _lib.ptr(egrad), _lib.current_stream()), "msg_bwd")
    _lib.check(lib.nb200_edge_forces(_lib.ptr(egrad), _lib.ptr(geom), _lib.ptr(row_ptr), _lib.ptr(rev), N, _lib.ptr(forces),
                                     _lib.current_stream()), "edge_forces")
    torch.cuda.synchronize()
    # fp64 autograd reference of the same op, filters regenerated from positions so that d/dpos flows
    import math
    P = pos.double().requires_grad_(True)
    j = col[:E].cpu().long()
    i = torch.repeat_interleave(torch.arange(N), (row_ptr[1:] - row_ptr[:-1]).cpu().long())
    r = P[j] - P[i]
    d = r.norm(dim=1)
    u = r / d[:, None]
    x = d * s["rbf_xscale"]
    phi = torch.exp(s["rbf_coeff"] * (x[:, None] - t["rbf_offsets"].double().cpu()[None]) ** 2)
    xs = d / s["cutoff"]
    env = 1 - 21 * xs**5 + 35 * xs**6 - 15 * xs**7
    Wr = env[:, None] * (phi @ t["w_rbf"][0].double().cpu()) + t["b_rbf"][0].double().cpu()
    XH = xh.double().cpu().requires_grad_(True)
    MU = mu.double().cpu().requires_grad_(True)
    p = (XH + bias.double().cpu())[j] * Wr
    a, b, c = p[:, :F], p[:, F:2 * F], p[:, 2 * F:]
    qo = q.double().cpu() + torch.zeros(N, F, dtype=torch.float64).index_add_(0, i, a)
    muo = MU + torch.zeros(N, 3, F, dtype=torch.float64).index_add_(0, i, b[:, None, :] * u[:, :, None] + c[:, None, :] * MU[j])
    assert (q_out.double().cpu() - qo.detach()).abs().max() < 2e-4 * max(1.0, qo.abs().max().item())
    assert (mu_out.double().cpu() - muo.detach()).abs().max() < 2e-4 * max(1.0, muo.abs().max().item())
    loss = (qo * gq.double().cpu()).sum() + (muo * gmu.double().cpu()).sum()
    gXH, gMU, gP = torch.autograd.grad(loss, [XH, MU, P])
    scale = lambda v: max(1.0, v.abs().max().item())
    assert (g_xh.double().cpu() - gXH).abs().max() < 2e-5 * scale(gXH)
    assert (g_mu_in.double().cpu() - gMU).abs().max() < 2e-5 * scale(gMU)
    assert (forces.double().cpu() + gP).abs().max() < 2e-5 * scale(gP)  # forces = -dLoss/dpos


class _Data:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def test_painn_oc_engine_matches_reference_golden():
    """End to end through the reference-facing module vs outputs of the reference's own classes."""
    g = np.load(os.path.join(GOLDEN, "painn_oc_f64.npz"))
    net = _oc_model(6).to(dev())
    data = _Data(torch.from_numpy(g["z"]).to(dev()), torch.from_numpy(g["pos"]).float().to(dev()), torch.from_numpy(g["batch"]).to(dev()))
    e, f = net(data)
    assert np.abs(e.cpu().numpy() - g["energy"]).max() < E_TOL  # north_star: 1e-5 Ha absolute
    assert np.abs(f.cpu().numpy() - g["forces"]).max() < F_TOL


def test_spk_painn_engine_matches_oracle():
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkPaiNN

    model = _spk_model(6)
    ref = OracleNNP(SpkPaiNN()).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    z, pos, batch = load_fixture([10, 11, 12, 60])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch})
    model = model.to(dev())
    n_atoms = torch.bincount(batch)
    out = model({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": n_atoms.to(dev())})
    e_ref, f_ref = out_ref["energy"].detach().numpy(), out_ref["forces"].numpy()
    assert np.abs(out["energy"].cpu().numpy() - e_ref).max() < E_TOL
    assert np.abs(out["forces"].cpu().numpy() - f_ref).max() < F_TOL


def test_full_size_properties_cfg2():
    """BASELINE config 2 size (256 synthetic conformations): size-independent properties --
    rotation/translation invariance, zero net force per molecule, permutation of molecules,
    bitwise determinism, energy-only == energy of the E+F pass."""
    from nabladft_b200.synth import synth_batch

    b = synth_batch(0, 256)
    net = _oc_model(6).to(dev())
    z = torch.from_numpy(b["z"]).to(dev())
    pos = torch.from_numpy(b["pos"]).to(dev())
    batch = torch.from_numpy(b["batch"]).to(dev())
    e0, f0 = net(_Data(z, pos, batch))
    e0b, f0b = net(_Data(z, pos, batch))
    assert torch.equal(e0, e0b) and torch.equal(f0, f0b)  # deterministic segmented sums: bitwise reproducible
    escale = 1.0  # absolute tolerances (north_star)
    R = random_rotation(5, torch.float32).to(dev())
    e1, f1 = net(_Data(z, pos @ R.T + 3.0, batch))
    assert (e0 - e1).abs().max() < 3 * E_TOL * escale
    assert (f0 @ R.T - f1).abs().max() < F_TOL
    net_f = torch.zeros(256, 3, device=dev()).index_add_(0, batch, f0)
    assert net_f.abs().max() < F_TOL  # translation invariance
    # reverse the molecule order: energies permute
    order = torch.arange(255, -1, -1)
    ptr = torch.from_numpy(b["mol_ptr"]).long()
    idx = torch.cat([torch.arange(ptr[m], ptr[m + 1]) for m in order.tolist()]).to(dev())
    batch2 = torch.repeat_interleave(torch.arange(256), (ptr[1:] - ptr[:-1])[order]).to(dev())
    e2, f2 = net(_Data(z[idx], pos[idx], batch2))
    assert (e2 - e0[order.to(dev())]).abs().max() < E_TOL * escale and (f2 - f0[idx]).abs().max() < F_TOL
    net.regress_forces = False
    e3 = net(_Data(z, pos, batch))
    assert torch.equal(e3, e0)


def test_engine_edge_cases():
    net = _oc_model(2).to(dev())
    # smallest molecule: two atoms 1.1 A apart; and a ragged batch (2 atoms + fixture molecule)
    z1 = torch.tensor([1, 1], device=dev())
    p1 = torch.tensor([[0.0, 0, 0], [1.1, 0, 0]], device=dev())
    e, f = net(_Data(z1, p1, torch.zeros(2, dtype=torch.long, device=dev())))
    assert e.shape == (1,) and torch.isfinite(e).all() and (f[0] + f[1]).abs().max() < 1e-6
    z, pos, batch = load_fixture([20], torch.float32)
    zz = torch.cat([z1.cpu(), z]).to(dev())
    pp = torch.cat([p1.cpu(), pos]).to(dev())
    bb = torch.cat([torch.zeros(2, dtype=torch.long), batch + 1]).to(dev())
    e2, f2 = net(_Data(zz, pp, bb))
    assert (e2[0] - e[0]).abs() < 1e-6 and (f2[:2] - f).abs().max() < 1e-6
    # capacity regrow on the synchronous (first batch of an engine) path: a tiny guess, the driver must retry and succeed
    from nabladft_b200._lib import NablaB200Error
    eng = net.engine()
    eng.check_pending(wait=True)
    eng.e_cap, eng.edges_per_atom_guess, eng._validated_ratio = 0, 1, 0.0
    e3, f3 = net(_Data(zz, pp, bb))
    assert torch.equal(e3, e2) and torch.equal(f3, f2)
    # forward() is asynchronous afterwards (deferred status check): an overflowing capacity can not go unnoticed -- the batch's outputs are
    # NaN, the next check raises and grows the capacity, the re-submitted batch is right
    eng.check_pending(wait=True)
    eng.e_cap, eng._validated_ratio, eng.e_cap_slack = 0, 1e-3, 8
    e4, f4 = net(_Data(zz, pp, bb))
    assert torch.isnan(e4).all() and torch.isnan(f4).all()
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        net.check()
    eng.e_cap_slack = 1024
    e5, f5 = net(_Data(zz, pp, bb))
    net.check()
    assert torch.equal(e5, e2) and torch.equal(f5, f2)
    # atomic number outside the embedding table -> NaN outputs and a loud (deferred) error, not garbage
    bad = zz.clone(); bad[0] = 0
    eb, fb = net(_Data(bad, pp, bb))
    assert torch.isnan(eb).all()
    with pytest.raises(NablaB200Error):
        net.check()
    # more neighbours than max_neighbors -> loud error (the reference would silently truncate)
    net.max_neighbors = 3
    net._engine._wkey = None
    en, fn = net(_Data(zz, pp, bb))
    assert torch.isnan(en).all()
    with pytest.raises(NablaB200Error):
        net.check()


@pytest.mark.parametrize("M,N,K,trans_b,accumulate,with_bias,with_act", [
    (1000, 128, 128, 0, 0, True, True),
    (257, 384, 128, 0, 0, False, False),
    (130, 64, 128, 0, 0, False, False),
    (515, 128, 384, 1, 0, False, False),
    (300, 128, 64, 1, 1, False, False),
    (3 * 211, 256, 128, 0, 0, False, False),
    (640, 128, 256, 1, 1, False, False),
    (129, 128, 128, 0, 1, True, True),
    (2050, 8320, 128, 0, 0, True, False),   # A-stationary variant (QHNet weight generation)
    (1500, 5376, 32, 1, 0, False, False),
    (1100, 640, 128, 0, 0, True, True),
    (40000, 1024, 64, 1, 0, False, False),
    # tall problems -> pre-split-weight kernel (gemm_ps.cu): accumulate + bias + activation, N tail / K padding, K > 128 in chunks (both layouts)
    (4100, 384, 128, 0, 1, True, True),
    (2500, 200, 96, 0, 0, True, False),
    (3000, 128, 384, 1, 0, False, False),
    (2300, 512, 512, 0, 1, False, True),
    # K < 128 on the pre-split-weight kernel: only the 32-k stages that carry data are streamed and multiplied (QHNet radial layers, K = 32)
    (2500, 5376, 32, 1, 0, False, False),
    (4000, 128, 32, 1, 0, True, True),
    (2100, 200, 64, 0, 1, True, False),
    (2200, 136, 96, 1, 0, False, False),
])
def test_gemm_tf32x3_matches_fp64(M, N, K, trans_b, accumulate, with_bias, with_act):
    """wgmma 3xTF32 GEMM (node-level dense layers) == fp64 matmul to fp32-level accuracy."""
    from nabladft_b200 import _lib

    lib = _lib.load()
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(dev())
    B = (torch.randn(K, N, generator=g) if trans_b else torch.randn(N, K, generator=g)).to(dev()) * 0.2
    C = torch.randn(M, N, generator=g).to(dev())
    C0 = C.clone()
    bias = torch.randn(N, generator=g).to(dev()) if with_bias else None
    act = torch.zeros(M, N, device=dev()) if with_act else None
    _lib.check(lib.nb200_gemm_tf32x3(M, N, K, _lib.ptr(A), K, _lib.ptr(B), N if trans_b else K, trans_b, _lib.ptr(C), N, accumulate,
                                     _lib.ptr(bias), _lib.ptr(act), _lib.current_stream()), "gemm")
    torch.cuda.synchronize()
    ref = A.double() @ (B.double() if trans_b else B.double().T)
    if accumulate:
        ref = ref + C0.double()
    if with_bias:
        ref = ref + bias.double()
    scale = ref.abs().max().item()
    err = (C.double() - ref).abs().max().item()
    sgemm_err = ((A @ (B if trans_b else B.T) + (C0 if accumulate else 0) + (bias if with_bias else 0)).double() - ref).abs().max().item()
    print(f"gemm {M}x{N}x{K} trans_b={trans_b}: rel err wgmma-3xTF32 {err / scale:.2e}  torch fp32 {sgemm_err / scale:.2e}")
    if not (with_act and N >= 512 and K <= 128 and M >= 1024):
        assert err < 2e-6 * scale, f"rel err {err / scale:.2e}"  # fp32 SGEMM itself: ~1e-6 at K=384
    if with_act:
        assert (act.double() - torch.nn.functional.silu(ref)).abs().max().item() < 3e-6 * scale
        if N >= 512:
            return  # the A-stationary epilogue writes only the activation


@pytest.mark.parametrize("M,out,inn,terms,bias,scale_div,lddw_extra", [
    (4676, 384, 128, 1, True, 1, 0),      # A2 / B2 of a config-2 batch: ragged last 128-atom chunk (4676 = 36 * 128 + 68)
    (3 * 4676, 256, 128, 1, False, 3, 0), # U over the (atom, xyz) rows, per-atom seed
    (4676, 128, 128, 2, True, 0, 128),    # B1 half: two tangent terms, dW is a column block of a [128, 256] matrix
    (4676, 64, 128, 2, True, 0, 0),       # readout R1: 64 outputs (half an output tile)
    (37, 128, 64, 1, True, 1, 0),         # one partial stage, narrow input
    (128, 8, 16, 1, True, 0, 0),          # smallest shapes the kernel takes
])
def test_linear_wgrad_matches_fp64(M, out, inn, terms, bias, scale_div, lddw_extra):
    """wgmma split-K weight-gradient kernel (wgrad_tc.cu) == fp64 grad_out^T @ input / grad_out.sum(0) to fp32 accuracy, accumulated."""
    from nabladft_b200 import _lib

    lib = _lib.load()
    g = torch.Generator().manual_seed(M * 7 + out + inn)
    G = [torch.randn(M, out, generator=g).to(dev()) for _ in range(terms)]
    X = [torch.randn(M, inn, generator=g).to(dev()) for _ in range(terms)]
    lddw = inn + lddw_extra
    dWfull = torch.randn(out, lddw, generator=g).to(dev())
    dW0 = dWfull.clone()
    db = torch.randn(out, generator=g).to(dev()) if bias else None
    db0 = db.clone() if bias else None
    c = torch.rand((M + scale_div - 1) // scale_div, generator=g).to(dev()) + 0.5 if scale_div else None
    alpha, balpha = (-1.0, -1.0) if terms == 2 else (1.0, 1.0)
    _lib.check(lib.nb200_linear_wgrad(M, out, inn, _lib.ptr(G[0]), _lib.ptr(X[0]), _lib.ptr(G[1]) if terms == 2 else None,
                                      _lib.ptr(X[1]) if terms == 2 else None, out, inn, _lib.ptr(dWfull), lddw, alpha, _lib.ptr(db), balpha,
                                      _lib.ptr(c), max(scale_div, 1), _lib.current_stream()), "wgrad")
    torch.cuda.synchronize()
    G0 = G[0].double()
    if scale_div:
        G0 = G0 * c.double().repeat_interleave(scale_div)[:M, None]
    ref = G0.T @ X[0].double()
    if terms == 2:
        ref = ref + G[1].double().T @ X[1].double()
    ref_full = dW0.double().clone()
    ref_full[:, :inn] += alpha * ref
    scale = ref.abs().max().item()
    err = (dWfull.double() - ref_full).abs().max().item()
    print(f"wgrad M={M} out={out} in={inn} terms={terms}: rel err {err / scale:.2e}")
    assert err < 2e-6 * scale, f"rel err {err / scale:.2e}"
    assert torch.equal(dWfull[:, inn:], dW0[:, inn:])  # the neighbouring column block is untouched
    if bias:
        refb = db0.double() + balpha * G0.sum(0)
        errb = (db.double() - refb).abs().max().item()
        assert errb < 2e-6 * G0.abs().sum(0).max().item(), f"bias err {errb:.2e}"


def test_backend_setters_accept_only_the_remaining_paths():
    """The node GEMMs are the wgmma kernels and the PaiNN node forward is the fused one: nb200_engine_set_gemm_backend and
    nb200_engine_set_node_backend accept 1, refuse 0 (the cuBLAS SGEMM and one-launch-per-op paths, which no longer exist) with
    NB200_EUNSUPPORTED and any other value with NB200_EINVAL, and a PaiNN call after them returns bitwise what it returned before."""
    net = _oc_model(6).to(dev())
    z, pos, batch = load_fixture([30, 31, 32], torch.float32)
    d = _Data(z.to(dev()), pos.to(dev()), batch.to(dev()))
    e1, f1 = net(d)
    eng = net.engine()
    for setter in (eng.lib.nb200_engine_set_gemm_backend, eng.lib.nb200_engine_set_node_backend):
        assert setter(eng._h, 0) == -2
        assert setter(eng._h, 2) == -1
        assert setter(eng._h, 1) == 0
    e0, f0 = net(d)
    assert torch.equal(e1, e0) and torch.equal(f1, f0)


def test_fused_node_forward_at_cfg2_size():
    """The fused per-layer node kernels (painn_fused.cu), whole model, at BASELINE config 2 size (256 synthetic conformations, ragged last
    128-atom tile) and on a 2-molecule batch (single partial tile): finite and bitwise deterministic, and the 2-molecule batch matches the
    fp64 oracle (at 256 molecules test_cfg2_slice_values_match_oracle[oc] checks the values of the same model and batch)."""
    from nabladft_b200.synth import synth_batch
    from oracle.painn_oc import PaiNNOC

    net = _oc_model(6)
    ref = PaiNNOC(hidden_channels=128, num_layers=6, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100).double()
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
    net = net.to(dev())
    for n_mol in (256, 2):
        b = synth_batch(0, n_mol)
        d = _Data(torch.from_numpy(b["z"]).to(dev()), torch.from_numpy(b["pos"]).to(dev()), torch.from_numpy(b["batch"]).to(dev()))
        e1, f1 = net(d)
        e1b, f1b = net(d)
        assert torch.isfinite(e1).all() and torch.isfinite(f1).all()
        assert torch.equal(e1, e1b) and torch.equal(f1, f1b)  # deterministic
        if n_mol == 2:
            e_ref, f_ref = ref(torch.from_numpy(b["z"]).long(), torch.from_numpy(b["pos"]).double(), torch.from_numpy(b["batch"]).long())
            de = (e1.double().cpu() - e_ref.detach()).abs().max().item()
            df = (f1.double().cpu() - f_ref.detach()).abs().max().item()
            print(f"fused vs fp64 oracle, {n_mol} molecules: dE {de:.2e} Ha (|E| <= {e_ref.abs().max().item():.1f}), dF {df:.2e} Ha/A")
            assert de < E_TOL and df < F_TOL


@pytest.mark.parametrize("flavour", ["oc", "spk"])
def test_cfg2_slice_values_match_oracle(flavour):
    """VALUE parity at config size: the first 32 molecules of the BASELINE config 2 synthetic batch, run INSIDE the full 256-molecule
    batch on the device, against the fp64 oracle on those 32 molecules (molecules do not interact, so the slice is exact)."""
    from nabladft_b200.synth import synth_batch
    from oracle.graph import ase_neighbor_list, batch_to_ptr

    b = synth_batch(0, 256)
    n32 = int(b["mol_ptr"][32])
    z, pos, batch = torch.from_numpy(b["z"]).long(), torch.from_numpy(b["pos"]).double(), torch.from_numpy(b["batch"]).long()
    if flavour == "oc":
        from oracle.painn_oc import PaiNNOC

        net = _oc_model(6)
        ref = PaiNNOC(hidden_channels=128, num_layers=6, num_rbf=100, cutoff=5.0, max_neighbors=100, num_elements=100).double()
        ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()}, strict=True)
        e_ref, f_ref = ref(z[:n32], pos[:n32].clone(), batch[:n32])
        e, f = net.to(dev())(_Data(z.to(dev()), pos.float().to(dev()), batch.to(dev())))
    else:
        from oracle.spk import NeuralNetworkPotential as OracleNNP
        from oracle.spk import SpkPaiNN

        model = _spk_model(6)
        ref = OracleNNP(SpkPaiNN()).double()
        sd = model.state_dict()
        ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
        idx_i, idx_j = ase_neighbor_list(pos[:n32], batch_to_ptr(batch[:n32]), 5.0)
        out_ref = ref({"_atomic_numbers": z[:n32], "_positions": pos[:n32].clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch[:n32]})
        e_ref, f_ref = out_ref["energy"], out_ref["forces"]
        out = model.to(dev())({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
                               "_n_atoms": torch.bincount(batch).to(dev())})
        e, f = out["energy"], out["forces"]
    de = (e[:32].double().cpu() - e_ref.detach()).abs().max().item()
    df = (f[:n32].double().cpu() - f_ref.detach()).abs().max().item()
    print(f"cfg 2 slice ({flavour}): 32 molecules / {n32} atoms, max|dE| {de:.2e} Ha (|E| <= {e_ref.abs().max().item():.1f}), max|dF| {df:.2e} Ha/A")
    assert de < E_TOL and df < F_TOL


def _spk_schnet_model(n_interactions=6):
    from nabladft_b200 import spk

    m = spk.NeuralNetworkPotential(
        representation=spk.SchNet(n_atom_basis=128, n_interactions=n_interactions, radial_basis=spk.GaussianRBF(n_rbf=100, cutoff=5.0),
                                  cutoff_fn=spk.CosineCutoff(cutoff=5.0)),
        input_modules=[spk.PairwiseDistances()],
        output_modules=[spk.Atomwise(n_in=128, output_key="energy"), spk.Forces()],
        postprocessors=[spk.AddOffsets(property="energy", add_mean=True)])
    load_golden_weights(m, torch.float32, weight_scale=1.0)
    m.postprocessors[0].mean.fill_(0.02)
    return m.eval()


def test_spk_schnet_engine_matches_oracle():
    """SchNet (config/model/schnet.yaml) E+F through the CUDA path vs the fp64 oracle; also energy-only
    (BASELINE config 1 is SchNet energy-only)."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkSchNet

    model = _spk_schnet_model(6)
    ref = OracleNNP(SpkSchNet()).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    z, pos, batch = load_fixture([10, 11, 12, 60])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch})
    model = model.to(dev())
    inp = {"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": torch.bincount(batch).to(dev())}
    out = model(inp)
    e_ref, f_ref = out_ref["energy"].detach().numpy(), out_ref["forces"].numpy()
    de = np.abs(out["energy"].cpu().numpy() - e_ref).max()
    df = np.abs(out["forces"].cpu().numpy() - f_ref).max()
    print(f"schnet: |E| {np.abs(e_ref).max():.3f} dE {de:.2e} |F| {np.abs(f_ref).max():.3f} dF {df:.2e}")
    assert de < E_TOL and df < F_TOL
    model._forces = False
    out_e = model(inp)
    assert "forces" not in out_e and torch.equal(out_e["energy"], out["energy"])


def test_schnet_engine_edge_cases():
    """SchNet keeps run_async's promise as PaiNN does (test_engine_edge_cases): an overflowing edge capacity or an atomic number outside the
    embedding table makes every energy and force of the launch NaN, and the next check raises; energy-only calls included."""
    from nabladft_b200._lib import NablaB200Error

    model = _spk_schnet_model(2).to(dev())
    z, pos, batch = load_fixture([20, 21], torch.float32)
    inp = {"_atomic_numbers": z.to(dev()), "_positions": pos.to(dev()), "_idx_m": batch.to(dev()), "_n_atoms": torch.bincount(batch).to(dev())}
    good = model(inp)
    eng = model._engine
    for forces in (True, False):
        model._forces = forces
        eng.check_pending(wait=True)
        eng.e_cap, eng._validated_ratio, eng.e_cap_slack = 0, 1e-3, 8
        out = model(inp)
        assert torch.isnan(out["energy"]).all() and (not forces or torch.isnan(out["forces"]).all())
        with pytest.raises(NablaB200Error, match="ECAPACITY"):
            model.check()
        eng.e_cap_slack = 1024
        again = model(inp)
        model.check()
        assert torch.equal(again["energy"], good["energy"]) and (not forces or torch.equal(again["forces"], good["forces"]))
        bad = dict(inp, _atomic_numbers=inp["_atomic_numbers"].clone())
        bad["_atomic_numbers"][0] = 100  # the table has rows 0 .. 99
        out = model(bad)
        assert torch.isnan(out["energy"]).all() and (not forces or torch.isnan(out["forces"]).all())
        with pytest.raises(NablaB200Error):
            model.check()


def test_schnet_c_entry_nans_outputs_on_overflow_and_refuses_other_widths():
    """nb200_schnet_energy_forces itself: with a too-small e_cap, energy-only and E+F calls return all-NaN energies and forces (and
    NB200_ECAPACITY in status); a Gaussian width other than the centre spacing is NB200_EUNSUPPORTED."""
    from nabladft_b200 import _lib
    from nabladft_b200.engine import mol_ptr_from_batch

    model = _spk_schnet_model(2).to(dev())
    eng = model.engine(True)
    z, pos, batch = load_fixture([20, 21], torch.float32)
    mol_ptr, n_mol = mol_ptr_from_batch(batch.to(dev()))
    z, pos = z.to(dev()).int(), pos.to(dev())
    for with_forces in (False, True):
        energy, forces, status = eng.launch(z, pos, mol_ptr, n_mol, with_forces, e_cap=16)
        torch.cuda.synchronize()
        assert int(status[1]) == -4 and torch.isnan(energy).all() and (not with_forces or torch.isnan(forces).all())
    w = _lib.SchnetWeights.from_buffer_copy(eng._weights)
    w.rbf_coeff = -0.5 / (1.5 * 5.0 / 99) ** 2
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=dev())
    e = torch.zeros(n_mol, device=dev())
    rc = eng.lib.nb200_schnet_energy_forces(eng._h, ctypes.byref(w), _lib.ptr(z), _lib.ptr(pos), _lib.ptr(mol_ptr), n_mol, z.shape[0], 4096,
                                            _lib.ptr(ws), ws.numel(), _lib.ptr(e), None, _lib.ptr(torch.zeros(4, dtype=torch.int32, device=dev())),
                                            _lib.current_stream())
    assert rc == -2


def test_spk_schnet_isolated_pair_and_dense_cluster_match_oracle():
    """SchNet E+F against the float64 oracle on one batch of an isolated atom, a two-atom molecule and a dense 300-atom cluster whose rows
    hold well over 100 edges (the fixture molecules reach a few tens)."""
    from oracle.graph import ase_neighbor_list, batch_to_ptr
    from oracle.spk import NeuralNetworkPotential as OracleNNP
    from oracle.spk import SpkSchNet

    model = _spk_schnet_model(6)
    ref = OracleNNP(SpkSchNet()).double()
    sd = model.state_dict()
    ref.load_state_dict({k: sd[k].double() for k in ref.state_dict()}, strict=True)
    g = torch.Generator().manual_seed(11)
    grid = torch.stack(torch.meshgrid(*[torch.arange(7, dtype=torch.float64)] * 3, indexing="ij"), -1).reshape(-1, 3)[:300]
    cluster = grid * 0.95 + (torch.rand(300, 3, generator=g, dtype=torch.float64) - 0.5) * 0.3  # ~1 A apart, a 6 A cube
    pos = torch.cat([torch.zeros(1, 3, dtype=torch.float64), torch.tensor([[0.0, 0, 0], [0.0, 0.0, 1.2]], dtype=torch.float64), cluster])
    z = torch.cat([torch.tensor([8, 1, 1]), torch.randint(1, 10, (300,), generator=g)])
    batch = torch.cat([torch.tensor([0, 1, 1]), torch.full((300,), 2)])
    idx_i, idx_j = ase_neighbor_list(pos, batch_to_ptr(batch), 5.0)
    max_deg = int(torch.bincount(idx_i).max())
    assert max_deg > 100
    out_ref = ref({"_atomic_numbers": z, "_positions": pos.clone(), "_idx_i": idx_i, "_idx_j": idx_j, "_idx_m": batch})
    model = model.to(dev())
    out = model({"_atomic_numbers": z.to(dev()), "_positions": pos.float().to(dev()), "_idx_m": batch.to(dev()),
                 "_n_atoms": torch.bincount(batch).to(dev())})
    e_ref, f_ref = out_ref["energy"].detach(), out_ref["forces"]
    de = (out["energy"].double().cpu() - e_ref).abs()
    df = (out["forces"].double().cpu() - f_ref).abs().max().item()
    print(f"schnet, isolated atom / pair / 300-atom cluster (max degree {max_deg}): |E| {e_ref.abs().tolist()}  dE {de.tolist()}  "
          f"|F| <= {f_ref.abs().max().item():.2f}  dF {df:.2e}")
    # fp32 sums over 300 atoms of ~250 edges each: the cluster's tolerances grow with its energy and largest force
    assert (de < E_TOL + 1e-5 * e_ref.abs()).all() and df < F_TOL + 1e-5 * f_ref.abs().max().item()
