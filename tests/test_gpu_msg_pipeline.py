"""PaiNN message kernels (painn_msg.cu) on graphs the benchmark batches do not contain: a row longer than the metadata staging cap (the
chunked path), rows of degree 0 and 1, every filter row layout, bf16 storage and the training variant that writes per-edge filter gradients.
Each launch is compared with the kernels' formulas in float64, and repeated launches must be bitwise equal."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F = 128
STAGE_CAP = 64  # MSG_STAGE_CAP in painn_msg.cu


def dev():
    return torch.device("cuda:0")


def _batch():
    """One 300-atom cluster (interior degrees above the staging cap), a lone atom (degree 0), a 2-atom molecule (degree 1) and two
    small random molecules."""
    rng = np.random.default_rng(7)
    mols = [rng.uniform(0.0, 12.0, size=(300, 3)), np.zeros((1, 3)), np.array([[0.0, 0.0, 0.0], [1.1, 0.2, -0.3]]),
            rng.uniform(0.0, 4.0, size=(9, 3)), rng.uniform(0.0, 3.0, size=(5, 3))]
    pos = torch.from_numpy(np.concatenate(mols)).float()
    mol_ptr = torch.tensor(np.concatenate([[0], np.cumsum([len(m) for m in mols])]), dtype=torch.int32)
    return pos, mol_ptr


def _graph(pos, mol_ptr):
    from nabladft_b200 import _lib

    lib = _lib.load()
    N, B = pos.shape[0], mol_ptr.numel() - 1
    e_cap = N * 160
    d = dev()
    row_ptr = torch.zeros(N + 1, dtype=torch.int32, device=d)
    col = torch.zeros(e_cap, dtype=torch.int32, device=d)
    rev = torch.zeros(e_cap, dtype=torch.int32, device=d)
    geom = torch.zeros(e_cap, 4, dtype=torch.float32, device=d)
    deg = torch.zeros(N, dtype=torch.int32, device=d)
    status = torch.zeros(4, dtype=torch.int32, device=d)
    _lib.check(lib.nb200_neighbor_build(_lib.ptr(pos.to(d)), _lib.ptr(mol_ptr.to(d)), B, N, 5.0, 1000, e_cap, _lib.ptr(row_ptr), _lib.ptr(col),
                                        _lib.ptr(rev), _lib.ptr(geom), _lib.ptr(deg), _lib.ptr(status), _lib.current_stream()), "neighbor_build")
    torch.cuda.synchronize()
    E = int(status[0])
    return row_ptr, col[:E].contiguous(), rev[:E].contiguous(), geom[:E].contiguous(), status.cpu().tolist()


@pytest.fixture(scope="module")
def case():
    torch.manual_seed(3)
    pos, mol_ptr = _batch()
    row_ptr, col, rev, geom, st = _graph(pos, mol_ptr)
    N, E = pos.shape[0], col.shape[0]
    degree = (row_ptr[1:] - row_ptr[:-1]).cpu()
    assert st[2] > STAGE_CAP and int(degree.max()) == st[2]  # the chunked staging path runs
    assert int((degree == 0).sum()) >= 1 and int((degree == 1).sum()) >= 2
    d = dev()
    t = dict(row_ptr=row_ptr, col=col, rev=rev, geom=geom, N=N, E=E,
             xh=torch.randn(N, 3 * F, device=d) * 0.5, bias=torch.randn(3 * F, device=d) * 0.1, q=torch.randn(N, F, device=d),
             mu=torch.randn(N, 3 * F, device=d) * 0.5, gq=torch.randn(N, F, device=d), gmu=torch.randn(N, 3 * F, device=d),
             seed=torch.rand(N, device=d) + 0.5,
             W=torch.randn(E, 3 * F, device=d) * 0.2, dW=torch.randn(E, 3 * F, device=d) * 0.2)
    return t


def _rows(t, use_rev, dtype):
    """Filter rows each edge reads (float64) and the stored arrays in the kernel's layout: with `rev` only row min(e, rev[e]) is read."""
    e = torch.arange(t["E"], device=dev())
    r = torch.minimum(e, t["rev"].long()) if use_rev else e
    W, dW = t["W"].to(dtype), t["dW"].to(dtype)
    return W.double()[r].cpu(), dW.double()[r].cpu(), W, dW


def _ref(t, We, dWe):
    """float64 restatement of the forward and backward formulas in painn_msg.cu."""
    N, E = t["N"], t["E"]
    c = lambda x: x.double().cpu()  # noqa: E731
    row_ptr = c(t["row_ptr"]).long()
    tgt = torch.repeat_interleave(torch.arange(N), row_ptr[1:] - row_ptr[:-1])
    src = c(t["col"]).long()
    u = c(t["geom"])[:, :3]
    xb = c(t["xh"]) + c(t["bias"])
    mu = c(t["mu"]).view(N, 3, F)
    a, b, cc = xb[:, :F], xb[:, F:2 * F], xb[:, 2 * F:]
    Wa, Wb, Wc = We[:, :F], We[:, F:2 * F], We[:, 2 * F:]
    q_out = c(t["q"]).index_add(0, tgt, Wa * a[src])
    msg = (Wb * b[src])[:, None, :] * u[:, :, None] + (Wc * cc[src])[:, None, :] * mu[src]
    mu_out = mu.index_add(0, tgt, msg).view(N, 3 * F)
    # backward by source atom j = tgt[e], far atom i = src[e]
    j, i = tgt, src
    gq, gmu = c(t["gq"]), c(t["gmu"]).view(N, 3, F)
    tb = -(gmu[i] * u[:, :, None]).sum(1)
    tc = (gmu[i] * mu[j]).sum(1)
    g_xh = torch.zeros(N, 3 * F, dtype=torch.float64)
    g_xh[:, :F].index_add_(0, j, Wa * gq[i])
    g_xh[:, F:2 * F].index_add_(0, j, Wb * tb)
    g_xh[:, 2 * F:].index_add_(0, j, Wc * tc)
    g_mu_in = gmu.index_add(0, j, (Wc * cc[j])[:, None, :] * gmu[i]).view(N, 3 * F)
    ta, tbb, tcc = a[j] * gq[i], b[j] * tb, cc[j] * tc
    gd = (dWe[:, :F] * ta + dWe[:, F:2 * F] * tbb + dWe[:, 2 * F:] * tcc).sum(1)
    gu = ((Wb * b[j])[:, None, :] * gmu[i]).sum(2)
    egrad = torch.cat([gu, gd[:, None]], 1)
    gW = torch.cat([ta, tbb, tcc], 1) * c(t["seed"])[j][:, None]
    return q_out, mu_out, g_xh, g_mu_in, egrad, gW


def _fwd(t, W, stride, rev, bf16):
    from nabladft_b200 import _lib

    lib = _lib.load()
    q_out, mu_out = torch.empty_like(t["q"]), torch.empty_like(t["mu"])
    _lib.check(lib.nb200_painn_msg_fwd_ex(_lib.ptr(t["xh"]), _lib.ptr(t["bias"]), _lib.ptr(t["q"]), _lib.ptr(t["mu"]), _lib.ptr(W), stride, _lib.ptr(rev),
                                          _lib.ptr(t["geom"]), _lib.ptr(t["row_ptr"]), _lib.ptr(t["col"]), t["N"], _lib.ptr(q_out), _lib.ptr(mu_out),
                                          bf16, _lib.current_stream()), "msg_fwd_ex")
    torch.cuda.synchronize()
    return q_out, mu_out


def _bwd(t, W, dW, stride, rev, bf16, train):
    from nabladft_b200 import _lib

    lib = _lib.load()
    g_xh, g_mu_in = torch.empty_like(t["xh"]), torch.empty_like(t["mu"])
    egrad = torch.zeros(t["E"], 4, device=dev())
    gW = torch.zeros(t["E"], 3 * F, device=dev(), dtype=W.dtype) if train else None
    _lib.check(lib.nb200_painn_msg_bwd_ex(_lib.ptr(t["xh"]), _lib.ptr(t["bias"]), _lib.ptr(t["mu"]), _lib.ptr(W), _lib.ptr(dW), stride, _lib.ptr(rev),
                                          _lib.ptr(t["geom"]), _lib.ptr(t["row_ptr"]), _lib.ptr(t["col"]), t["N"], _lib.ptr(t["gq"]), _lib.ptr(t["gmu"]),
                                          _lib.ptr(g_xh), _lib.ptr(g_mu_in), _lib.ptr(egrad), _lib.ptr(gW), _lib.ptr(t["seed"] if train else None), bf16,
                                          _lib.current_stream()), "msg_bwd_ex")
    torch.cuda.synchronize()
    return g_xh, g_mu_in, egrad, gW


def _close(got, ref, tol):
    got = got.double().cpu()
    err = float((got - ref).abs().max())
    assert err <= tol * max(1.0, float(ref.abs().max())), err


# (w_stride, rev): one [W | dW] record per pair (E+F path), pair rows in two arrays (training), per-directed-edge rows (public ABI)
LAYOUTS = [("record", True), ("rows", True), ("rows", False)]


# the training variant reads W and dW as two arrays only (test_train_variant_rejects_record_layout)
CASES = [(layout, use_rev, train) for layout, use_rev in LAYOUTS for train in (False, True) if not (train and layout == "record")]


@pytest.mark.parametrize("storage", ["f32", "bf16"])
@pytest.mark.parametrize("layout,use_rev,train", CASES)
def test_msg_kernels_match_fp64(case, storage, layout, use_rev, train):
    t = case
    dtype = torch.bfloat16 if storage == "bf16" else torch.float32
    bf16 = 1 if storage == "bf16" else 0
    We, dWe, W, dW = _rows(t, use_rev, dtype)
    rev = t["rev"] if use_rev else None
    if layout == "record":
        rec = torch.cat([W, dW], 1).contiguous()
        args_f, args_b = (rec, 6 * F), (rec, rec, 6 * F)
    else:
        args_f, args_b = (W.contiguous(), 3 * F), (W.contiguous(), dW.contiguous(), 3 * F)
    q_ref, mu_ref, gxh_ref, gmu_ref, eg_ref, gW_ref = _ref(t, We, dWe)
    tol = 2e-5  # fp32 arithmetic on exactly representable inputs, sums of up to ~100 edges
    q_out, mu_out = _fwd(t, args_f[0], args_f[1], rev, bf16)
    _close(q_out, q_ref, tol)
    _close(mu_out, mu_ref, tol)
    g_xh, g_mu_in, egrad, gW = _bwd(t, *args_b, rev, bf16, train)
    _close(g_xh, gxh_ref, tol)
    _close(g_mu_in, gmu_ref, tol)
    _close(egrad, eg_ref, tol)
    if train:
        _close(gW, gW_ref, 2e-5 if storage == "f32" else 4e-3)  # bf16 store: round to nearest, 8 significant bits
    # repeat launches: bitwise equal (no atomics race: one RED per egrad address per launch)
    q2, mu2 = _fwd(t, args_f[0], args_f[1], rev, bf16)
    assert torch.equal(q2, q_out) and torch.equal(mu2, mu_out)
    g2 = _bwd(t, *args_b, rev, bf16, train)
    assert torch.equal(g2[0], g_xh) and torch.equal(g2[1], g_mu_in) and torch.equal(g2[2], egrad)
    if train:
        assert torch.equal(g2[3], gW)


def test_train_variant_rejects_record_layout(case):
    from nabladft_b200 import _lib

    t = case
    lib = _lib.load()
    rec = torch.zeros(t["E"], 6 * F, device=dev())
    out = torch.empty_like(t["xh"])
    rc = lib.nb200_painn_msg_bwd_ex(_lib.ptr(t["xh"]), _lib.ptr(t["bias"]), _lib.ptr(t["mu"]), _lib.ptr(rec), _lib.ptr(rec), 6 * F, _lib.ptr(t["rev"]),
                                    _lib.ptr(t["geom"]), _lib.ptr(t["row_ptr"]), _lib.ptr(t["col"]), t["N"], _lib.ptr(t["gq"]), _lib.ptr(t["gmu"]),
                                    _lib.ptr(out), _lib.ptr(torch.empty_like(t["mu"])), _lib.ptr(torch.zeros(t["E"], 4, device=dev())),
                                    _lib.ptr(torch.zeros(t["E"], 3 * F, device=dev())), _lib.ptr(t["seed"]), 0, _lib.current_stream())
    assert rc == -1  # NB200_EINVAL
