"""The PaiNN tangent and Hessian-vector-product kernels one at a time on the H100, each against its float64 reference
(tests/painn_tangent_ref.py), through nb200_painn_test_tangent (the host wrappers the engine calls):

* painn_tangent.cu: k_geom_tan, k_mul_dact, k_act_bwd_tan, k_readout_bwd_tan, k_msg_fwd_tan (fp32 and bf16 rows), k_upd_norm_tan,
  k_upd_combine_tan, k_upd_combine_bwd_tan, k_upd_norm_bwd_tan, k_msg_bwd_tan (training: fp32 and bf16; Hessian: d2W, t_egrad),
  k_edge_forces_hvp; the message kernels with one filter row per undirected pair (`rev`) and with one row per directed edge (no `rev`);
* filter.cu: k_filter<true, float, true> (W, dW/dd, d2W/dd2) and k_filter_wgrad_bal (primal and tangent, fp32 and bf16 gradient rows)
  after the bin sort over every directed edge, in both radial modes.

On a graph with rows of degree 0 to 5, 31 to 33, 63 to 65 and 310, 626 atoms (a partial last CTA), filter rows that the kernels must not
read set to NaN, in-place outputs pre-filled with random values, norms at their floor, and synthetic distances at both band clamps, just
below the cutoff, in empty bins, in bins whose group ranges straddle every ring depth and in a bin split into parts.  Checked: |kernel -
reference| <= C A elementwise (C_POINT / C_SUM of painn_tangent_ref.py; plus half a bf16 ulp of |reference| for bf16 stored outputs);
rows at or past n_atoms (or E) keep a sentinel bitwise; two launches are bitwise equal for every kernel without atomics; and the entry
point's refusals.  Each check prints its largest error as a fraction of A."""
import ctypes

import pytest
import torch

import painn_tangent_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F = ref.F
EINVAL, EUNSUPPORTED = -1, -2
PAD = 8  # sentinel rows after every output


def _L():
    from nabladft_b200 import _lib

    return _lib


def call(op, bf16=0, tan=0, n_atoms=0, n=0, width=0, e_cap=0, radial=None, **ptrs):
    L = _L()
    a = L.PainnTanArgs()
    a.op = op if isinstance(op, int) else L.PT_OPS.index(op)
    a.bf16, a.tan, a.n_atoms, a.n, a.width, a.e_cap = bf16, tan, n_atoms, n, width, e_cap
    for k, t in ptrs.items():
        setattr(a, k, None if t is None else (t if isinstance(t, int) else t.data_ptr()))
    for k, v in (radial or {}).items():
        setattr(a, k, v)
    rc = L.load().nb200_painn_test_tangent(ctypes.byref(a), L.current_stream())
    torch.cuda.synchronize()
    return rc


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def sentinel(rows, cols, dtype=torch.float32):
    bits = ref.SENTINEL_BITS if dtype == torch.float32 else ref.SENTINEL_BITS >> 16
    it = torch.int32 if dtype == torch.float32 else torch.int16
    return torch.full((rows + PAD, cols), bits, dtype=it, device=DEV).view(dtype)


def prefilled(pre):
    out = sentinel(pre.shape[0], pre.shape[1])
    out[:pre.shape[0]] = pre.to(DEV)
    return out


def run(op, outs, **kw):
    """Two launches, each on fresh copies of the initial `outs`; asserts status 0 and returns the first launch's outputs and the second's."""
    res = []
    for _ in range(2):
        o = {k: v.clone() for k, v in outs.items()}
        rc = call(op, **kw, **o)
        assert rc == 0, f"{op}: status {rc}"
        res.append(o)
    return res


def check(what, got, want, A, C, rows, bf16_out=False):
    """|got[:rows] - want| <= C A (+ half a bf16 ulp of |want|), and got[rows:] is the sentinel."""
    assert bool((_bits(got[rows:]) == _bits(sentinel(0, got.shape[1], got.dtype)[:1])).all()), f"{what}: a row at or past the end was written"
    g = got[:rows].double().cpu()
    err = (g - want).abs()
    tol = C * A + (ref.BF16_HALF_ULP * want.abs() if bf16_out else 0)
    nz = A > 0
    worst = float((err[nz] / A[nz]).max()) if bool(nz.any()) else 0.0
    print(f"{what}: max |err| / A = {worst:.2e} (bound {C:.0e}{' + half bf16 ulp' if bf16_out else ''})")
    bad = ~(err <= tol)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {err.numel()} elements beyond the bound, first at {bad.nonzero()[0].tolist()}"


def same(what, a, b):
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), f"{what}: {k} differs between two launches"


@pytest.fixture(scope="module")
def case():
    g = ref.tangent_graph()
    d = ref.node_inputs(g)
    dev = {k: v.to(DEV).contiguous() for k, v in d.items()}
    dev.update({k: v.to(DEV) for k, v in g.tensors().items()})
    return g, d, dev, {}


def _memo(memo, key, fn):
    if key not in memo:
        memo[key] = fn()
    return memo[key]


# ------------------------------------------------------------------------------------------------------------------- per-atom ops
def test_geom_tan(case):
    g, d, t, memo = case
    a, b = run("GEOM_TAN", dict(t_geom=sentinel(g.E, 4)), n_atoms=g.n, geom=t["geom"], row_ptr=t["row_ptr"], col=t["col"], v=t["v"])
    want, A = ref.geom_tan(g, d)
    check("k_geom_tan", a["t_geom"], want, A, ref.C_POINT, g.E)
    same("k_geom_tan", a, b)


def test_activation_tangents(case):
    g, d, t, memo = case
    N = g.n
    a, b = run("MUL_DACT", dict(out=sentinel(N, F)), n=N * F, pre=t["pre"], x=t["x"])
    check("k_mul_dact", a["out"], *ref.mul_dact(d), ref.C_POINT, N)
    same("k_mul_dact", a, b)
    a, b = run("ACT_BWD_TAN", dict(t_g=prefilled(d["t_g"])), n=N * F, g_pre=t["g_pre"], pre=t["pre"], t_pre=t["t_pre"])
    check("k_act_bwd_tan", a["t_g"], *ref.act_bwd_tan(d), ref.C_POINT, N)
    same("k_act_bwd_tan", a, b)
    a, b = run("READOUT_BWD_TAN", dict(t_g_pre=sentinel(N, F // 2), t_act=sentinel(N, F // 2)), n_atoms=N, width=F // 2, pre=t["pre_ro"],
               t_pre=t["t_pre_ro"], R2=t["R2"])
    (tg, Ag), (ta, Aa) = ref.readout_bwd_tan(d)
    check("k_readout_bwd_tan t_g_pre", a["t_g_pre"], tg, Ag, ref.C_POINT, N)
    check("k_readout_bwd_tan t_act", a["t_act"], ta, Aa, ref.C_POINT, N)
    same("k_readout_bwd_tan", a, b)


def test_update_tangents(case):
    g, d, t, memo = case
    N = g.n
    upd = dict(VW=t["VW"], t_VW=t["t_VW"])
    a, b = run("UPD_NORM_TAN", dict(t_nrm=sentinel(N, F)), n_atoms=N, nrm=t["nrm"], **upd)
    check("k_upd_norm_tan", a["t_nrm"], *ref.upd_norm_tan(d), ref.C_POINT, N)
    same("k_upd_norm_tan", a, b)
    a, b = run("UPD_COMBINE_TAN", dict(t_q=prefilled(d["prefill_q"]), t_mu=prefilled(d["prefill_mu"])), n_atoms=N, y=t["y"], t_y=t["t_y"], **upd)
    (tq, tm), (Aq, Am) = ref.upd_combine_tan(d)
    check("k_upd_combine_tan t_q (accumulated)", a["t_q"], tq, Aq, ref.C_POINT, N)
    check("k_upd_combine_tan t_mu (accumulated)", a["t_mu"], tm, Am, ref.C_POINT, N)
    same("k_upd_combine_tan", a, b)
    a, b = run("UPD_COMBINE_BWD_TAN", dict(t_gy=sentinel(N, 3 * F), t_gVW=sentinel(N, 6 * F)), n_atoms=N, g_q=t["g_q"], t_g_q=t["t_g_q"],
               g_mu=t["g_mu"], t_g_mu=t["t_g_mu"], y=t["y"], t_y=t["t_y"], **upd)
    (ty, tv), (Ay, Av) = ref.upd_combine_bwd_tan(d)
    check("k_upd_combine_bwd_tan t_gy", a["t_gy"], ty, Ay, ref.C_POINT, N)
    check("k_upd_combine_bwd_tan t_gVW", a["t_gVW"], tv, Av, ref.C_POINT, N)
    same("k_upd_combine_bwd_tan", a, b)
    a, b = run("UPD_NORM_BWD_TAN", dict(t_gVW=prefilled(d["prefill_gVW"])), n_atoms=N, gn=t["gn"], t_gn=t["t_gn"], nrm=t["nrm"], t_nrm=t["t_nrm"],
               **upd)
    check("k_upd_norm_bwd_tan t_gVW (accumulated; norms at the floor included)", a["t_gVW"], *ref.upd_norm_bwd_tan(d), ref.C_POINT, N)
    same("k_upd_norm_bwd_tan", a, b)


# ------------------------------------------------------------------------------------------------------------------- message
def _msg_in(t, rows, rev):
    W, dW = rows[0], rows[1]
    return dict(xh=t["xh"], t_xh=t["t_xh"], xh_bias=t["xh_bias"], mu=t["mu"], t_mu=t["t_mu"], W=W.to(DEV), dW=dW.to(DEV), geom=t["geom"],
                t_geom=t["t_geom"], row_ptr=t["row_ptr"], col=t["col"], rev=t["rev"] if rev else None)


LAYOUTS = [("f32", True), ("bf16", True), ("f32", False), ("bf16", False)]


@pytest.mark.parametrize("storage,use_rev", LAYOUTS, ids=[f"{s}-{'pair' if r else 'edge'}-rows" for s, r in LAYOUTS])
def test_msg_fwd_tan(case, storage, use_rev):
    g, d, t, memo = case
    dtype = torch.bfloat16 if storage == "bf16" else torch.float32
    stored, read = ref.filter_rows(g, d, use_rev, dtype)
    a, b = run("MSG_FWD_TAN", dict(t_q=prefilled(d["prefill_q"]), t_mu_out=sentinel(g.n, 3 * F)), bf16=int(storage == "bf16"), n_atoms=g.n,
               **_msg_in(t, stored, use_rev))
    (tq, Aq), (tm, Am) = _memo(memo, ("fwd", storage, use_rev), lambda: ref.Msg(g, d, read).fwd_tan(d))
    what = f"k_msg_fwd_tan<{storage}> {'pair' if use_rev else 'edge'} rows"
    check(f"{what} t_q (accumulated)", a["t_q"], tq, Aq, ref.C_SUM, g.n)
    check(f"{what} t_mu_out", a["t_mu_out"], tm, Am, ref.C_SUM, g.n)
    same(what, a, b)


@pytest.mark.parametrize("storage,use_rev", LAYOUTS, ids=[f"{s}-{'pair' if r else 'edge'}-rows" for s, r in LAYOUTS])
def test_msg_bwd_tan(case, storage, use_rev):
    g, d, t, memo = case
    dtype = torch.bfloat16 if storage == "bf16" else torch.float32
    stored, read = ref.filter_rows(g, d, use_rev, dtype)
    outs = dict(t_g_xh=sentinel(g.n, 3 * F), t_g_mu_in=sentinel(g.n, 3 * F), t_gW=sentinel(g.E, 3 * F, dtype), gWd=sentinel(g.E, 3 * F, dtype))
    a, b = run("MSG_BWD_TAN", outs, bf16=int(storage == "bf16"), n_atoms=g.n, g_q=t["g_q"], t_g_q=t["t_g_q"], g_mu=t["g_mu"], t_g_mu=t["t_g_mu"],
               **_msg_in(t, stored, use_rev))
    r = _memo(memo, ("bwd", storage, use_rev), lambda: ref.Msg(g, d, read).bwd_tan(d))
    what = f"k_msg_bwd_tan<{storage}> {'pair' if use_rev else 'edge'} rows"
    check(f"{what} t_g_xh", a["t_g_xh"], *r["t_g_xh"], ref.C_SUM, g.n)
    check(f"{what} t_g_mu_in", a["t_g_mu_in"], *r["t_g_mu_in"], ref.C_SUM, g.n)
    check(f"{what} t_gW", a["t_gW"], *r["t_gW"], ref.C_SUM, g.E, bf16_out=storage == "bf16")
    check(f"{what} gWd", a["gWd"], *r["gWd"], ref.C_SUM, g.E, bf16_out=storage == "bf16")
    same(what, a, b)


def test_msg_bwd_hvp(case):
    g, d, t, memo = case
    stored, read = ref.filter_rows(g, d, True)
    outs = dict(t_g_xh=sentinel(g.n, 3 * F), t_g_mu_in=sentinel(g.n, 3 * F), t_egrad=prefilled(d["prefill_egrad"]))
    a, b = run("MSG_BWD_HVP", outs, n_atoms=g.n, g_q=t["g_q"], t_g_q=t["t_g_q"], g_mu=t["g_mu"], t_g_mu=t["t_g_mu"], d2W=stored[2].to(DEV),
               **_msg_in(t, stored, True))
    r = ref.Msg(g, d, read).bwd_tan(d, hvp=True)
    check("k_msg_bwd_tan<float, HVP> t_g_xh", a["t_g_xh"], *r["t_g_xh"], ref.C_SUM, g.n)
    check("k_msg_bwd_tan<float, HVP> t_g_mu_in", a["t_g_mu_in"], *r["t_g_mu_in"], ref.C_SUM, g.n)
    check("k_msg_bwd_tan<float, HVP> t_egrad (accumulated)", a["t_egrad"], *r["t_egrad"], ref.C_SUM, g.E)
    same("k_msg_bwd_tan<float, HVP>", a, b)


def test_edge_forces_hvp(case):
    g, d, t, memo = case
    t_geom = ref.geom_tan(g, d)[0].float().to(DEV)  # the tangent geometry of v, as k_geom_tan hands it on
    a, b = run("EDGE_FORCES_HVP", dict(hv=sentinel(g.n, 3)), n_atoms=g.n, egrad=t["egrad"], t_egrad=t["t_egrad"], geom=t["geom"], t_geom=t_geom,
               row_ptr=t["row_ptr"], rev=t["rev"])
    check("k_edge_forces_hvp", a["hv"], *ref.edge_forces_hvp(g, d), ref.C_SUM, g.n)
    same("k_edge_forces_hvp", a, b)


# ------------------------------------------------------------------------------------------------------------------- radial filter
def _radial_args(rad):
    return dict(radial_mode=rad.mode, n_rbf=rad.K, n_layers=2, cutoff=rad.cutoff, rbf_coeff=rad.coeff, rbf_xscale=rad.xscale, sign=1.0)


def _edges(dist):
    E = dist.numel()
    geom = torch.zeros(E, 4)
    geom[:, 0], geom[:, 3] = 1.0, dist
    return geom.to(DEV), torch.tensor([E, 0, 0, 0], dtype=torch.int32, device=DEV), torch.zeros(768 + E, dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("mode", [0, 1], ids=["spk", "oc"])
def test_filter_d2(mode):
    """W, dW/dd, d2W/dd2 of both layers into rows of stride e_cap > E: canonical rows against the dense float64 filter, every other row
    (the opposite edges and the rows past E) untouched."""
    rad = ref.Radial(mode)
    dist = torch.from_numpy(ref.filter_d2_distances(rad))
    P = dist.numel()
    E, e_cap = 2 * P, 2 * P + PAD
    geom, status, scr = _edges(torch.cat([dist, dist]))
    geom[P:, 0] = -1.0
    rev = torch.cat([torch.arange(P, 2 * P), torch.arange(P)]).int().to(DEV)
    init = torch.full((2, e_cap, 3 * F), ref.SENTINEL_BITS, dtype=torch.int32, device=DEV).view(torch.float32)
    outs = dict(W=init.clone(), dW=init.clone(), d2W=init.clone())
    a, b = run("FILTER_D2", outs, e_cap=e_cap, radial=_radial_args(rad), geom=geom, status=status, rev=rev, sort_scratch=scr,
               rbf_offsets=rad.offsets.to(DEV), w_rbf=rad.w.to(DEV), b_rbf=rad.b.to(DEV))
    d64 = dist.double()
    for layer in range(2):
        want, A = rad.derivs(d64, layer), rad.d2_bounds(d64, layer)
        for k, name in enumerate(("W", "dW", "d2W")):
            got = a[name][layer]
            check(f"k_filter<true, float, true> {['spk', 'oc'][mode]} layer {layer} {name}", torch.cat([got[:P], got[E:]]), want[k], A[k],
                  ref.C_SUM, P)
            assert bool((_bits(got[P:E]) == ref.SENTINEL_BITS).all()), f"{name}: a non-canonical row was written"
    same("k_filter<true, float, true>", a, b)


WG = [(mode, tan, storage) for mode in (0, 1) for tan in (False, True) for storage in ("f32", "bf16")]


@pytest.mark.parametrize("mode,tan,storage", WG, ids=[f"{['spk', 'oc'][m]}-{'tan' if t else 'primal'}-{s}" for m, t, s in WG])
def test_filter_wgrad(mode, tan, storage):
    """g_w [K, 3F], g_b [3F] of one layer, pre-filled: prefill + (sign *) the contraction over every directed edge.  e_cap = 4 E: spare CTAs
    exit.  Atomics: not bitwise repeatable, so one launch."""
    rad = ref.Radial(mode)
    dist = torch.from_numpy(ref.wgrad_distances(rad))
    E = dist.numel()
    geom, status, scr = _edges(dist)
    gen = torch.Generator().manual_seed(11 + mode)
    dtype = torch.bfloat16 if storage == "bf16" else torch.float32
    rows = [(torch.randn(E, 3 * F, generator=gen) * 0.5).to(dtype) for _ in range(2)]
    dd = torch.rand(E, generator=gen).double() + 0.25
    pw, pb = torch.randn(rad.K, 3 * F, generator=gen), torch.randn(1, 3 * F, generator=gen)
    g_w, g_b = prefilled(pw), prefilled(pb)
    radial = dict(_radial_args(rad), sign=-1.0 if tan else 1.0)
    ins = dict(t_gW=rows[0].to(DEV), gWd=rows[1].to(DEV)) if tan else dict(gW=rows[0].to(DEV))
    rc = call("FILTER_WGRAD", bf16=int(storage == "bf16"), tan=int(tan), e_cap=4 * E, radial=radial, geom=geom, status=status, sort_scratch=scr,
              rbf_offsets=rad.offsets.to(DEV), g_w=g_w, g_b=g_b, **ins)
    assert rc == 0
    if tan:
        want, A = ref.wgrad_ref(rad, dist, None, t_gW=rows[0], gWd=rows[1], dd=dd, sign=-1.0)
    else:
        want, A = ref.wgrad_ref(rad, dist, rows[0])
    pre = torch.cat([pw, pb]).double()
    what = f"k_filter_wgrad_bal<{'true' if tan else 'false'}, {storage}> {['spk', 'oc'][mode]}"
    check(f"{what} g_w (accumulated)", g_w, pre[:rad.K] + want[:rad.K], pre[:rad.K].abs() + A[:rad.K], ref.C_SUM, rad.K)
    check(f"{what} g_b (accumulated)", g_b, pre[rad.K:] + want[rad.K:], pre[rad.K:].abs() + A[rad.K:], ref.C_SUM, 1)


# ------------------------------------------------------------------------------------------------------------------- refusals
REQUIRED = {
    "GEOM_TAN": "geom row_ptr col v t_geom",
    "MUL_DACT": "pre x out",
    "ACT_BWD_TAN": "t_g g_pre pre t_pre",
    "READOUT_BWD_TAN": "pre t_pre R2 t_g_pre t_act",
    "MSG_FWD_TAN": "xh t_xh xh_bias mu t_mu W dW geom t_geom row_ptr col t_q t_mu_out",
    "UPD_NORM_TAN": "VW t_VW nrm t_nrm",
    "UPD_COMBINE_TAN": "t_q t_mu VW t_VW y t_y",
    "UPD_COMBINE_BWD_TAN": "g_q t_g_q g_mu t_g_mu y t_y VW t_VW t_gy t_gVW",
    "UPD_NORM_BWD_TAN": "gn t_gn VW t_VW nrm t_nrm t_gVW",
    "MSG_BWD_TAN": "xh t_xh xh_bias mu t_mu W dW geom t_geom row_ptr col g_q t_g_q g_mu t_g_mu t_g_xh t_g_mu_in t_gW gWd",
    "MSG_BWD_HVP": "xh t_xh xh_bias mu t_mu W dW d2W geom t_geom row_ptr col rev g_q t_g_q g_mu t_g_mu t_g_xh t_g_mu_in t_egrad",
    "EDGE_FORCES_HVP": "egrad t_egrad geom t_geom row_ptr rev hv",
    "FILTER_D2": "geom status rev sort_scratch rbf_offsets w_rbf b_rbf W dW d2W",
    "FILTER_WGRAD": "geom status sort_scratch rbf_offsets g_w g_b gW",
    "FILTER_WGRAD_TAN": "geom status sort_scratch rbf_offsets g_w g_b t_gW gWd",
}
BF16_OPS = ("MSG_FWD_TAN", "MSG_BWD_TAN", "FILTER_WGRAD")


def test_refusals():
    """Every refusal returns NB200_EINVAL (radial parameters outside the kernels: NB200_EUNSUPPORTED) before anything is launched: the
    buffer every pointer points to keeps its sentinel."""
    L = _L()
    buf = sentinel(4096 - PAD, 1024)
    fields = [f for f, _ in L.PainnTanArgs._fields_ if _ is ctypes.c_void_p]
    rad = ref.Radial(1)
    base = dict(n_atoms=8, n=1024, width=64, e_cap=0, radial=_radial_args(rad), **{f: buf for f in fields})

    def rc(op, **kw):
        args = dict(base)
        args.update(kw)
        tan = 1 if op == "FILTER_WGRAD_TAN" else args.pop("tan", 0)
        return call("FILTER_WGRAD" if op == "FILTER_WGRAD_TAN" else op, tan=tan, **args)

    for op, req in REQUIRED.items():
        for f in req.split():
            assert rc(op, **{f: None}) == EINVAL, f"{op}: NULL {f} not refused"
        assert rc(op, n_atoms=-1) == EINVAL and rc(op, n=-4) == EINVAL and rc(op, e_cap=-1) == EINVAL, op
        if op not in BF16_OPS and op != "FILTER_WGRAD_TAN":
            assert rc(op, bf16=1) == EINVAL, f"{op}: bf16 not refused"
        if op not in ("FILTER_WGRAD", "FILTER_WGRAD_TAN"):
            assert rc(op, tan=1) == EINVAL, f"{op}: tan not refused"
    for op in ("MUL_DACT", "ACT_BWD_TAN"):
        assert rc(op, n=1022) == EINVAL, f"{op}: n % 4 != 0 not refused"
    assert rc("READOUT_BWD_TAN", width=0) == EINVAL
    assert rc(-1) == EINVAL and rc(len(L.PT_OPS)) == EINVAL
    for op in ("FILTER_D2", "FILTER_WGRAD", "FILTER_WGRAD_TAN"):
        assert rc(op, radial=dict(_radial_args(rad), rbf_coeff=1.0)) == EUNSUPPORTED, op
        assert rc(op, radial=dict(_radial_args(rad), n_rbf=8)) == EUNSUPPORTED, op
    assert bool((_bits(buf) == ref.SENTINEL_BITS).all()), "a refused call wrote memory"
