"""The GemNet-OC edge aggregations one at a time on the CPU: nb200_gemnet_oc_test_aggregate of the host-emulation build (tests/emu; it runs
the functors TripEdgeK, QuadK, TripEdgeTK and QuadTK for both forms) on synthetic graphs against the float64 references of
tests/gemnet_kernel_ref.py, at the row shapes, excluded positions and degenerate geometries of tests/test_gpu_gemnet_kernels.py.  This proves
the references, the graph builder and the tolerances without a GPU; the sensitivity checks prove that the tolerance at a long row sees a single
missing input at a chunk boundary."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

import gemnet_kernel_ref as ref  # noqa: E402

C_AGG = 1e-5  # |O - O64| <= C_AGG * A elementwise
EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    from emu_driver import load

    return load("gemnet_oc", ["nb200_gemnet_oc_"])


def _trip(case, overshoot):
    pairing, repeats, ldr, col = case
    return ref.Problem(False, "cpu", seed=repeats + ldr + col, pairing=pairing, repeats=repeats, ldr=ldr, col=col, overshoot=overshoot)


@pytest.mark.parametrize("case", ref.TRIP_CASES, ids=lambda c: f"{c[0]}-x{c[1]}-ldr{c[2]}-col{c[3]}")
@pytest.mark.parametrize("tangent", [False, True], ids=["primal", "tangent"])
def test_triplet_functor_matches_fp64(lib, case, tangent):
    p = _trip(case, overshoot=not tangent)
    rc, out = p.run(lib, None, form=1, tangent=tangent)
    assert rc == 0
    O64, A = p.reference(tangent)
    ref.compare(out, O64, A, C_AGG, f"emu {p.label()} {'tangent' if tangent else 'primal'}")


@pytest.mark.parametrize("collinear,tangent", [(True, False), (False, False), (False, True)], ids=["collinear-primal", "primal", "tangent"])
def test_quadruplet_functor_matches_fp64(lib, collinear, tangent):
    p = ref.Problem(True, "cpu", seed=3, ldr=ref.QUAD_LDR, col=ref.QUAD_COL, collinear=collinear)
    rc, out = p.run(lib, None, form=1, tangent=tangent)
    assert rc == 0
    O64, A = p.reference(tangent)
    ref.compare(out, O64, A, C_AGG, f"emu {p.label()} {'tangent' if tangent else 'primal'}")


@pytest.mark.parametrize("quad", [False, True], ids=["trip", "quad"])
def test_device_count_keeps_rows_past_it(lib, quad):
    p = ref.Problem(quad, "cpu", seed=5, ldr=ref.QUAD_LDR if quad else 1920, col=ref.QUAD_COL if quad else 80)
    O64, A = p.reference(False)
    for count in (0, p.E // 2, p.E, p.E + 5):
        dev = torch.tensor([count], dtype=torch.int32)
        rc, out = p.run(lib, None, form=1, tangent=False, E_dev=dev)
        assert rc == 0
        rows = min(count, p.E)
        assert bool((out[rows:].view(torch.int32) == ref.SENTINEL_BITS).all()), f"count {count}: a row at or past the count was written"
        if rows:
            ref.compare(out[:rows], O64[:rows], A[:rows], C_AGG, f"emu {p.label()} E_dev={count}")


def test_sensitivity_of_the_tolerance():
    """Dropping one input at a chunk boundary of a long row moves the float64 reference by more than 10x the tolerance at that element."""
    p = ref.Problem(False, "cpu", seed=9, pairing="mn_ae", ldr=1920, col=192)
    probes = ref.long_row_probes(p.go, p.gi)
    assert len(probes) >= 8
    O64, A = p.reference(False)
    te, tk = p.terms
    for e, k in probes:
        keep = ~((te == e) & (tk == k))
        assert int((~keep).sum()) == 1
        Od, _ = p.reference(False, (te[keep], tk[keep]))
        ratio = float(((Od[e] - O64[e]).abs() / (C_AGG * A[e])).max())
        assert ratio > 10, f"edge {e}, input {k}: dropping it moves the reference by only {ratio:.1f}x the tolerance"
    q = ref.Problem(True, "cpu", seed=9, ldr=ref.QUAD_LDR, col=ref.QUAD_COL)
    O64, A = q.reference(False)
    qe_e, qe_q, qe_k, qe_t = q.terms
    n = 0
    for qe in range(q.gi.ne):
        b = int(q.gi.src[qe])
        r = list(q.go.row(b))
        if len(r) < 33:
            continue
        for pos in (31, 32):
            hit = (qe_q == qe) & (qe_k == r[pos])
            if not bool(hit.any()):
                continue
            j = int(torch.nonzero(hit)[0])
            keep = torch.ones_like(hit)
            keep[j] = False
            Od, _ = q.reference(False, tuple(t[keep] for t in q.terms))
            e = int(qe_e[j])
            ratio = float(((Od[e] - O64[e]).abs() / (C_AGG * A[e])).max())
            assert ratio > 10, f"quadruplet {j}: dropping it moves the reference by only {ratio:.1f}x the tolerance"
            n += 1
    assert n >= 8


def test_argument_checks(lib):
    """NB200_EINVAL before anything is written: a NULL required pointer, E_bound < 0, a short ldr, a device count with a tangent form."""
    p = ref.Problem(False, "cpu", seed=11, pairing="mn_ae")
    out = torch.full((p.E, 1024), ref.SENTINEL_BITS, dtype=torch.int32).view(torch.float32)
    saved = dict(p.t), dict(p.i)
    p.t["x"] = None
    assert p.run(lib, None, 1, False, out=out)[0] == EINVAL
    p.t.update(saved[0]); p.i["ptr"] = None
    assert p.run(lib, None, 1, False, out=out)[0] == EINVAL
    p.i.update(saved[1])
    assert p.run(lib, None, 1, False, E_bound=-1, out=out)[0] == EINVAL
    assert p.run(lib, None, 1, True, E_dev=torch.tensor([p.E], dtype=torch.int32), out=out)[0] == EINVAL
    p.ldr = 111
    assert p.run(lib, None, 1, False, out=out)[0] == EINVAL
    q = ref.Problem(True, "cpu", seed=11, ldr=ref.LDR_QUAD + 1)
    q.ldr = ref.LDR_QUAD - 1
    assert q.run(lib, None, 1, False, out=out)[0] == EINVAL
    q.q_tin = None
    q.ldr = ref.LDR_QUAD
    assert q.run(lib, None, 1, False, out=out)[0] == EINVAL
    assert bool((out.view(torch.int32) == ref.SENTINEL_BITS).all())
