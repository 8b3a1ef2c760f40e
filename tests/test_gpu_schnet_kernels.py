"""The SchNet inference kernels (csrc/schnet.cu) one launch at a time, through nb200_schnet_test_op, against the float64 restatement of
schnet_kernel_ref.py within its per-element bound A: the banded first filter layer over the bin sort, cfconv forward and backward, and the
shifted-softplus output of the GEMM at row counts on both sides of its tall-GEMM switch.  The synthetic graph reaches the kernels' edges
(see schnet_kernel_ref.edge_case_graph); outputs are NaN-filled first, so a row not written, or written past the edge count, shows."""
import ctypes

import pytest
import torch

import schnet_kernel_ref as ref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F, CUTOFF, K = ref.F, 5.0, 100
EINVAL, EUNSUPPORTED = -1, -2


def _L():
    from nabladft_b200 import _lib

    return _lib


def call(op, **kw):
    L = _L()
    a = L.SchnetTestArgs()
    a.op = op if isinstance(op, int) else L.SC_OPS.index(op)
    for k, v in kw.items():
        setattr(a, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    rc = L.load().nb200_schnet_test_op(ctypes.byref(a), L.current_stream())
    torch.cuda.synchronize()
    return rc


def nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def bits(t):
    return t.view(torch.int32).clone()


def check(name, out, want, A):
    """|out - want| <= A everywhere (float64); returns the worst ratio."""
    err = (out.double().cpu() - want).abs()
    r = ref.max_ratio(err, A)
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    assert r <= 1.0, f"{name}: max |err| / A = {r:.2f}"
    return r


def _graph(c):
    return {k: c[k].to(DEV) for k in ("row_ptr", "col")} | {"geom": ref.geom_of(c["d"]).to(DEV)}


@pytest.mark.parametrize("L", [1, 6])
def test_filter1(L):
    c = ref.kernel_case(L, seed=L)
    E = c["d"].numel()
    e_stride = E + 37
    g = _graph(c)
    status = torch.tensor([E, 0, 0, 0], dtype=torch.int32, device=DEV)
    kw = dict(n_layers=L, n_rbf=K, n_edges=E, e_stride=e_stride, cutoff=CUTOFF, rbf_coeff=c["coeff"], status=status, geom=g["geom"],
              rbf_offsets=c["offsets"].to(DEV), w_f1=c["w1"].to(DEV), b_f1=c["b1"].to(DEV),
              sort_scratch=torch.zeros(768 + E, dtype=torch.int32, device=DEV))
    HH = nan(L, 2, e_stride, F)
    assert call("FILTER1", HH=HH, **kw) == 0
    worst = [0.0, 0.0]
    for l in range(L):
        h, dh, A_h, A_dh = ref.filter1(c["d"], c["w1"][l], c["b1"][l], c["offsets"], c["coeff"], CUTOFF)
        worst[0] = max(worst[0], check(f"h layer {l}", HH[l, 0, :E], h, A_h))
        worst[1] = max(worst[1], check(f"dh layer {l}", HH[l, 1, :E], dh, A_dh))
    assert torch.isnan(HH[:, :, E:]).all(), "rows at or past the edge count were written"
    again = nan(L, 2, e_stride, F)
    assert call("FILTER1", HH=again, **kw) == 0
    assert torch.equal(bits(again), bits(HH)), "repeated launches differ"
    status[1] = -4
    untouched = nan(L, 2, e_stride, F)
    assert call("FILTER1", HH=untouched, **kw) == 0
    assert torch.isnan(untouched).all(), "status[1] != 0 still wrote"
    print(f"k_schnet_filter1 L={L}, {E} edges: max |err| / A  h {worst[0]:.1e}  dh {worst[1]:.1e}")


def test_cfconv_fwd_bwd():
    c = ref.kernel_case()
    N, E = c["row_ptr"].numel() - 1, c["d"].numel()
    g = _graph(c)
    dv = {k: c[k].to(DEV) for k in ("y", "G1", "G2", "b2", "gagg")}
    fwd = dict(n_atoms=N, cutoff=CUTOFF, y=dv["y"], G1=dv["G1"], b2=dv["b2"], geom=g["geom"], row_ptr=g["row_ptr"], col=g["col"])
    agg = nan(N, F)
    assert call("CFCONV_FWD", agg=agg, **fwd) == 0
    want, A = ref.cfconv_fwd(c["y"], c["G1"], c["b2"], c["d"], c["row_ptr"], c["col"], CUTOFF)
    r_fwd = check("agg", agg, want, A)
    again = nan(N, F)
    assert call("CFCONV_FWD", agg=again, **fwd) == 0
    assert torch.equal(bits(again), bits(agg))

    egrad0 = c["egrad0"].to(DEV)
    bwd = dict(fwd, G2=dv["G2"], gagg=dv["gagg"])
    gy, egrad = nan(N, F), egrad0.clone()
    assert call("CFCONV_BWD", gy=gy, egrad=egrad, **bwd) == 0
    want_gy, A_gy, want_eg, A_eg = ref.cfconv_bwd(c["y"], c["G1"], c["G2"], c["b2"], c["d"], c["row_ptr"], c["col"], c["rev"], CUTOFF,
                                                  c["gagg"], c["egrad0"][:, 3])
    r_gy = check("gy", gy, want_gy, A_gy)
    r_eg = check("egrad", egrad[:, 3], want_eg, A_eg)
    assert torch.equal(bits(egrad[:, :3]), bits(egrad0[:, :3])), "egrad slots 0-2 were written"
    gy2, egrad2 = nan(N, F), egrad0.clone()
    assert call("CFCONV_BWD", gy=gy2, egrad=egrad2, **bwd) == 0
    assert torch.equal(bits(gy2), bits(gy)) and torch.equal(bits(egrad2), bits(egrad))
    print(f"k_cfconv_fwd / k_cfconv_bwd, {N} atoms, {E} edges (rows of 0 to 150): max |err| / A  agg {r_fwd:.1e}  gy {r_gy:.1e}  egrad {r_eg:.1e}")


@pytest.mark.parametrize("M", [1, 127, 129, 2047, 2048, 20000])
def test_linear_ssp(M):
    """f2out.0 with its shifted-softplus output on gemm_tc (M < 2048) and gemm_ps (M >= 2048), pre-activations over [-100, 100]: both
    sides of softplus's threshold at 20."""
    gen = torch.Generator().manual_seed(M)
    X = torch.randn(M, F, generator=gen)
    W = torch.randn(F, F, generator=gen) * F ** -0.5 * 4
    b = torch.rand(F, generator=gen) * 200 - 100
    Y, act = nan(M, F), nan(M, F)
    assert call("LINEAR_ACT", m=M, X=X.to(DEV), W=W.to(DEV), bias=b.to(DEV), Y=Y, act=act) == 0
    want, A_Y, want_act, A_act = ref.linear_ssp(X, W, b)
    assert (want > 20).any() and (want < -20).any()
    r_y, r_a = check("Y", Y, want, A_Y), check("ssp(Y)", act, want_act, A_act)
    print(f"linear + ssp M={M}: max |err| / A  Y {r_y:.1e}  act {r_a:.1e}")


def test_act_bwd_ssp():
    """nb_act_bwd with NB_ACT_SSP (g *= sigmoid(pre), the backward of f2out.0's activation) over [-100, 100], through the PaiNN node test
    entry that calls the same wrapper."""
    L = _L()
    gen = torch.Generator().manual_seed(7)
    n = 1000 * F
    g0, pre = torch.randn(n, generator=gen), torch.rand(n, generator=gen) * 200 - 100
    g = g0.to(DEV)
    a = L.PainnNodeArgs()
    a.op, a.n, a.kind, a.g, a.pre = L.PN_OPS.index("ACT_BWD"), n, 1, g.data_ptr(), pre.to(DEV).data_ptr()
    assert L.load().nb200_painn_test_node(ctypes.byref(a), L.current_stream()) == 0
    torch.cuda.synchronize()
    s = torch.sigmoid(pre.double())
    A = 8 * ref.U * g0.double().abs() * s * (1 + pre.double().abs()) + g0.double().abs() * 2.0 ** -126  # fp32 underflow of sigmoid
    print(f"nb_act_bwd ssp: max |err| / A {check('g', g, g0.double() * s, A):.1e}")


def test_entry_refuses_bad_arguments():
    c = ref.kernel_case()
    N, E = c["row_ptr"].numel() - 1, c["d"].numel()
    g = _graph(c)
    status = torch.tensor([E, 0, 0, 0], dtype=torch.int32, device=DEV)
    HH = nan(2, E + 4, F)
    base = dict(n_layers=1, n_rbf=K, n_edges=E, e_stride=E, cutoff=CUTOFF, rbf_coeff=c["coeff"], status=status, geom=g["geom"],
                rbf_offsets=c["offsets"].to(DEV), w_f1=c["w1"].to(DEV), b_f1=c["b1"].to(DEV),
                sort_scratch=torch.zeros(768 + E, dtype=torch.int32, device=DEV), HH=HH)
    dx = CUTOFF / (K - 1)
    bad = [(EINVAL, dict(e_stride=E - 1)), (EINVAL, dict(n_layers=-1)), (EINVAL, dict(n_edges=-1)), (EINVAL, dict(w_f1=0)),
           (EINVAL, dict(HH=HH.data_ptr() + 4)), (EINVAL, dict(b_f1=base["b_f1"].data_ptr() + 8)), (EUNSUPPORTED, dict(n_rbf=15)),
           (EUNSUPPORTED, dict(n_rbf=257)), (EUNSUPPORTED, dict(rbf_coeff=-0.5 / (1.5 * dx) ** 2)), (EUNSUPPORTED, dict(rbf_coeff=0.0))]
    for want, change in bad:
        assert call("FILTER1", **(base | change)) == want, change
    for op in (-1, len(_L().SC_OPS)):
        assert call(op, **base) == EINVAL
    agg = nan(N, F)
    fwd = dict(n_atoms=N, cutoff=CUTOFF, y=c["y"].to(DEV), G1=c["G1"].to(DEV), b2=c["b2"].to(DEV), geom=g["geom"], row_ptr=g["row_ptr"],
               col=g["col"], agg=agg)
    for change in (dict(n_atoms=-1), dict(col=0), dict(y=fwd["y"].data_ptr() + 4), dict(agg=agg.data_ptr() + 4)):
        assert call("CFCONV_FWD", **(fwd | change)) == EINVAL, change
    for change in (dict(gagg=0), dict(G2=fwd["G1"].data_ptr() + 4), dict(egrad=0)):
        assert call("CFCONV_BWD", **(fwd | dict(G2=fwd["G1"], gagg=fwd["y"], gy=nan(N, F), egrad=nan(E, 4)) | change)) == EINVAL, change
    X = torch.zeros(8, F, device=DEV)
    for change in (dict(m=-1), dict(act=0), dict(X=X.data_ptr() + 4)):
        assert call("LINEAR_ACT", **(dict(m=8, X=X, W=torch.zeros(F, F, device=DEV), bias=torch.zeros(F, device=DEV), Y=nan(8, F),
                                          act=nan(8, F)) | change)) == EINVAL, change
    assert torch.isnan(HH).all() and torch.isnan(agg).all(), "a refused call launched"
