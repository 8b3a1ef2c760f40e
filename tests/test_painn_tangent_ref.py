"""The float64 references of tests/painn_tangent_ref.py on the CPU: each tangent against central differences of its primal, and each
tangent input (or the d2W term) shown to matter by more than 10x the GPU tolerance, so that a kernel dropping one product-rule term fails
tests/test_gpu_painn_tangent.py."""
import pytest
import torch
from torch.func import vjp

import painn_tangent_ref as ref

H = 1e-4  # central-difference step (float64, extrapolated: truncation ~H^4, rounding ~1e-16 / H)
H_FLOOR = 1e-6  # for the norm, whose curvature is 1 / nrm = 1e4 at its floor
H_FILTER = 1e-7  # for the filter, so that no step crosses the cutoff from d = rc (1 - 1e-6)


@pytest.fixture(scope="module")
def case():
    g = ref.tangent_graph()
    return g, ref.node_inputs(g)


def _cd(f, prim, tang, h=H):
    """Central differences along `tang`, Richardson-extrapolated: (4 D(h / 2) - D(h)) / 3, truncation O(h^4)."""
    def D(s):
        plus = f(*(p + s * t for p, t in zip(prim, tang)))
        minus = f(*(p - s * t for p, t in zip(prim, tang)))
        return tuple((a - b) / (2 * s) for a, b in zip(plus, minus)) if isinstance(plus, tuple) else ((plus - minus) / (2 * s),)

    out = tuple((4 * a - b) / 3 for a, b in zip(D(h / 2), D(h)))
    return out if len(out) > 1 else out[0]


def _close(got, want, A, what):
    """|jvp - central difference| <= 1e-6 A + 1e-9 max|want|."""
    got, want = (got if isinstance(got, tuple) else (got,)), (want if isinstance(want, tuple) else (want,))
    A = A if isinstance(A, tuple) else (A,)
    for k, (a, b, bound) in enumerate(zip(got, want, A)):
        err = (a - b).abs()
        tol = 1e-6 * bound + 1e-9 * float(b.abs().max())
        assert bool((err <= tol).all()), f"{what}[{k}]: jvp and central difference differ by {float(err.max()):.3e}"


def _D(d, *names):
    return tuple(ref.d64(d[k]) for k in names)


def test_geometry_and_forces(case):
    g, d = case
    pos = torch.from_numpy(g.pos).double()
    t, A = ref.geom_tan(g, d)
    _close(t, _cd(lambda p: ref.geom_of(g, p), (pos,), _D(d, "v")), A, "geom")
    hv, A = ref.edge_forces_hvp(g, d)
    _close(hv, -_cd(lambda p, e: ref.forces_of(g, p, e), (pos, ref.d64(d["egrad"])), _D(d, "v", "t_egrad")), A, "forces")


def test_activations(case):
    g, d = case
    t, A = ref.mul_dact(d)
    _close(t, _cd(ref.silu, _D(d, "pre"), _D(d, "x")), A, "mul_dact")
    t, A = ref.act_bwd_tan(d)
    _close(t, _cd(ref.act_bwd, _D(d, "g_pre", "pre"), _D(d, "t_g", "t_pre")), A, "act_bwd")
    (t1, A1), (t2, A2) = ref.readout_bwd_tan(d)
    pre, t_pre, R2 = _D(d, "pre_ro", "t_pre_ro", "R2")
    grad = lambda p: vjp(lambda q: (ref.silu(q) * R2).sum(), p)[1](torch.ones((), dtype=torch.float64))[0]  # noqa: E731
    _close(t1, _cd(grad, (pre,), (t_pre,)), A1, "readout g_pre")
    _close(t2, _cd(ref.silu, (pre,), (t_pre,)), A2, "readout act")


def test_update_steps(case):
    g, d = case
    VW, t_VW = _D(d, "VW", "t_VW")
    t, A = ref.upd_norm_tan(d)
    _close(t, _cd(ref.norm, (VW,), (t_VW,), H_FLOOR), A, "norm")
    t, A = ref.upd_norm_bwd_tan(d)
    pre = ref.d64(d["prefill_gVW"])
    _close(t - pre, _cd(ref.norm_bwd, _D(d, "gn", "VW", "nrm"), _D(d, "t_gn", "t_VW", "t_nrm"), H_FLOOR), A, "norm bwd")
    z = torch.zeros(g.n, ref.F, dtype=torch.float64)
    (tq, tm), A = ref.upd_combine_tan(d)
    _close((tq, tm), _cd(ref.combine, (z, z.repeat(1, 3), VW, ref.d64(d["y"])), _D(d, "prefill_q", "prefill_mu", "t_VW", "t_y")), A, "combine")
    t, A = ref.upd_combine_bwd_tan(d)
    _close(t, _cd(ref.combine_bwd, _D(d, "VW", "y", "g_q", "g_mu"), _D(d, "t_VW", "t_y", "t_g_q", "t_g_mu")), A, "combine bwd")


def test_norm_bwd_is_the_vjp_of_the_norm(case):
    """norm_bwd (the primal k_upd_norm_bwd, nrm as an input) is the vjp of the norm when nrm is the norm of V."""
    g, d = case
    VW, gn = _D(d, "VW", "gn")
    want = vjp(ref.norm, VW)[1](gn)[0]
    assert torch.allclose(ref.norm_bwd(gn, VW, ref.norm(VW)), want, rtol=1e-12, atol=0)


@pytest.mark.parametrize("hvp", [False, True], ids=["train", "hvp"])
def test_message(case, hvp):
    g, d = case
    m = ref.Msg(g, d, ref.filter_rows(g, d, True)[1])
    prim, tang = m.point(d)
    Z = torch.zeros(g.E, 3 * ref.F, dtype=torch.float64)
    (tq, A_q), (tmu, A_mu) = m.fwd_tan(d)
    cd_q, cd_mu = _cd(m.fwd, prim + (Z,), tang + (Z,))
    _close((tq - ref.d64(d["prefill_q"]), tmu), (cd_q, cd_mu), (A_q, A_mu), "msg fwd")
    out = m.bwd_tan(d, hvp=hvp)
    if not hvp:
        m.W2 = torch.zeros_like(m.W2)
    cd = _cd(m.bwd, prim + _D(d, "g_q", "g_mu"), tang + _D(d, "t_g_q", "t_g_mu"))
    r = m.rev
    _close(out["t_g_xh"][0], cd[0], out["t_g_xh"][1], "msg bwd g_xh")
    _close(out["t_g_mu_in"][0], cd[1], out["t_g_mu_in"][1], "msg bwd g_mu")
    if hvp:
        eg = torch.cat([cd[2][r], cd[3][r][:, None]], 1)
        _close(out["t_egrad"][0] - ref.d64(d["prefill_egrad"]), eg, out["t_egrad"][1], "msg bwd egrad")
    else:
        _close(out["t_gW"][0], cd[4][r], out["t_gW"][1], "msg bwd gW")


@pytest.mark.parametrize("mode", [0, 1], ids=["spk", "oc"])
def test_filter_derivatives(mode):
    rad = ref.Radial(mode)
    d = torch.from_numpy(ref.filter_d2_distances(rad)).double()
    one = torch.ones_like(d)
    W, dW, d2W = rad.derivs(d, 1)
    A = rad.d2_bounds(d, 1)
    _close(dW, _cd(lambda x: rad.W(x, 1), (d,), (one,), H_FILTER), A[1], "dW")
    _close(d2W, _cd(lambda x: rad.derivs(x, 1)[1], (d,), (one,), H_FILTER), A[2], "d2W")
    assert bool(((W - rad.W(d, 1)).abs() == 0).all())


@pytest.mark.parametrize("mode", [0, 1], ids=["spk", "oc"])
def test_filter_wgrad(mode):
    rad = ref.Radial(mode)
    d = torch.from_numpy(ref.wgrad_distances(rad)).double()
    gen = torch.Generator().manual_seed(4)
    E = d.numel()
    t_gW, gWd = torch.randn(E, 3 * ref.F, generator=gen), torch.randn(E, 3 * ref.F, generator=gen)
    dd = torch.rand(E, generator=gen).double() + 0.5
    t, A = ref.wgrad_ref(rad, d, None, t_gW=t_gW, gWd=gWd, dd=dd, sign=-1.0)
    cd = _cd(rad.wgrad, (d, gWd.double() / dd[:, None]), (dd, t_gW.double()), H_FILTER)
    _close(t, -cd, A, "wgrad tan")


# ---------------------------------------------------------------------------------------------------------------- sensitivity
def _moves(a, b, A, C):
    """Largest |a - b| / (C A): how far a change moves the reference in units of the GPU tolerance."""
    return float(((a - b).abs() / (C * A).clamp_min(1e-300)).max())


SENS = [("msg_fwd", z) for z in ("t_mu", "t_xh", "t_geom.w", "t_geom.xyz")] + \
       [("msg_bwd", z) for z in ("t_mu", "t_xh", "t_geom.w", "t_geom.xyz", "t_g_q", "t_g_mu")] + [("msg_hvp", "d2W")] + \
       [("norm_bwd", z) for z in ("t_nrm", "t_VW", "t_gn")] + [("combine", z) for z in ("t_VW", "t_y")] + \
       [("combine_bwd", z) for z in ("t_g_q", "t_g_mu", "t_VW", "t_y")] + [("act_bwd", "t_pre")]


def _outputs(g, d, op, zero):
    if op.startswith("msg"):
        m = ref.Msg(g, d, ref.filter_rows(g, d, True)[1])
        if op == "msg_fwd":
            return list(m.fwd_tan(d, zero))
        return list(m.bwd_tan(d, zero, hvp=op == "msg_hvp").values())
    if op == "norm_bwd":
        return [ref.upd_norm_bwd_tan(d, zero)]
    if op == "combine":
        (tq, tm), (Aq, Am) = ref.upd_combine_tan(d, zero)
        return [(tq, Aq), (tm, Am)]
    if op == "combine_bwd":
        (ty, tv), (Ay, Av) = ref.upd_combine_bwd_tan(d, zero)
        return [(ty, Ay), (tv, Av)]
    return [ref.act_bwd_tan(d, zero)]


@pytest.mark.parametrize("op,zero", SENS, ids=[f"{o}-{z}" for o, z in SENS])
def test_dropping_a_term_exceeds_tolerance(case, op, zero):
    """Zeroing one tangent input (or the d2W term) moves the reference by more than 10x the GPU tolerance somewhere."""
    g, d = case
    C = ref.C_POINT if op in ("norm_bwd", "combine", "combine_bwd", "act_bwd") else ref.C_SUM
    full = _outputs(g, d, op, ())
    cut = _outputs(g, d, op, (zero,))
    worst = max(_moves(a[0], b[0], a[1], C) for a, b in zip(full, cut))
    print(f"{op} without {zero}: moves by {worst:.3g} x the tolerance")
    assert worst > 10, f"dropping {zero} from {op} moves the reference by only {worst:.3g} x the tolerance"
