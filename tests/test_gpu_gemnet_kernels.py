"""The GemNet-OC device kernels one at a time on the H100, each against a float64 reference of the same operation (tests/gemnet_kernel_ref.py):

* the warp-per-edge aggregations k_trip_edges / k_quad_edges and their tangents k_trip_edges_t / k_quad_edges_t, reached through the host
  dispatch the model calls (nb200_gemnet_oc_test_aggregate, form 0), and the functors TripEdgeK / QuadK / TripEdgeTK / QuadTK the training
  forward runs on the device (form 1), on synthetic graphs with every row length around the 4-wide unrolled loop and the 32-input chunks,
  excluded inputs on either side of a chunk boundary, cos exactly +-1 and past it, parallel and planar quadruplets, R read at the column
  offsets of B_main, 20 150 output edges (more than two passes of the capped grid) and a device row count below, at and above its bound;
* the fused ScaledSiLU and residual tails of the tall-layer GEMM (nb200_gemm_tf32x3_epi) at GemNet-OC's layer shapes.

Each check prints the largest error as a fraction of its bound, and for the aggregations how many elements of the device kernel and the
functor are not bitwise equal."""
import pytest
import torch

import gemnet_kernel_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_AGG = 1e-5     # aggregations: |O - O64| <= C_AGG * A elementwise (emulation, worst 1.4e-6)
C_SAME = 1e-6    # device kernel against functor: |O_kernel - O_functor| <= C_SAME * A
GEMM_REL = 2e-6  # 3xTF32 GEMM, of max |o| at K <= 384 (tests/test_gpu_painn.py::test_gemm_tf32x3_matches_fp64); x sqrt(K / 384) beyond,
                 # as fp32 accumulation error grows (K = 2560 measured 5.6e-6 of max |o| after the activation)
SLOPE = 1.9      # max |ScaledSiLU'| = 1.0998 / 0.6
NB_EPI_ACT, NB_EPI_RESIDUAL, NB_ACT_SSILU = 1, 2, 3
EINVAL, EUNSUPPORTED = -1, -2


def _lib():
    from nabladft_b200 import _lib

    return _lib.load()


def _stream():
    from nabladft_b200 import _lib

    return _lib.current_stream()


def _both_forms(p, tangent, **kw):
    lib = _lib()
    outs = []
    for form in (0, 1):
        rc, out = p.run(lib, _stream(), form, tangent, **kw)
        assert rc == 0, f"form {form}: status {rc}"
        outs.append(out)
    torch.cuda.synchronize()
    return outs


def _kernel_vs_functor(kern, func, A, what):
    kern, func = kern.cpu(), func.cpu()
    diff = int((kern.view(torch.int32) != func.view(torch.int32)).sum())
    err = (kern.double() - func.double()).abs()
    print(f"{what}: device kernel vs functor: {diff} of {kern.numel()} elements not bitwise equal, max |diff| / A = "
          f"{float((err[A > 0] / A[A > 0]).max()) if bool((A > 0).any()) else 0.0:.2e}")
    assert bool((err <= C_SAME * A).all()), f"{what}: device kernel and functor disagree beyond {C_SAME:.0e} A"


@pytest.mark.parametrize("case", ref.TRIP_CASES, ids=lambda c: f"{c[0]}-x{c[1]}-ldr{c[2]}-col{c[3]}")
@pytest.mark.parametrize("tangent", [False, True], ids=["primal", "tangent"])
def test_triplet_kernels_match_fp64(case, tangent):
    pairing, repeats, ldr, col = case
    p = ref.Problem(False, DEV, seed=repeats + ldr + col, pairing=pairing, repeats=repeats, ldr=ldr, col=col, overshoot=not tangent)
    kern, func = _both_forms(p, tangent)
    O64, A = p.reference(tangent)
    what = f"{p.label()} {'tangent' if tangent else 'primal'}"
    ref.compare(kern, O64, A, C_AGG, f"{what} device kernel")
    ref.compare(func, O64, A, C_AGG, f"{what} functor")
    _kernel_vs_functor(kern, func, A, what)


@pytest.mark.parametrize("collinear,tangent", [(True, False), (False, False), (False, True)], ids=["collinear-primal", "primal", "tangent"])
def test_quadruplet_kernels_match_fp64(collinear, tangent):
    p = ref.Problem(True, DEV, seed=3, ldr=ref.QUAD_LDR, col=ref.QUAD_COL, collinear=collinear)
    kern, func = _both_forms(p, tangent)
    O64, A = p.reference(tangent)
    what = f"{p.label()} {'tangent' if tangent else 'primal'}{' collinear' if collinear else ''}"
    ref.compare(kern, O64, A, C_AGG, f"{what} device kernel")
    ref.compare(func, O64, A, C_AGG, f"{what} functor")
    _kernel_vs_functor(kern, func, A, what)


@pytest.mark.parametrize("quad", [False, True], ids=["trip", "quad"])
def test_device_count_keeps_rows_past_it(quad):
    """E_dev = 0, below the bound, equal to it and above it (clamped): rows at or past the count keep the sentinel bitwise."""
    p = ref.Problem(quad, DEV, seed=5, ldr=ref.QUAD_LDR if quad else 1920, col=ref.QUAD_COL if quad else 80, repeats=1 if quad else 50)
    O64, A = p.reference(False)
    for count in (0, p.E // 2 + 3, p.E, p.E + 5):
        dev = torch.tensor([count], dtype=torch.int32, device=DEV)
        kern, func = _both_forms(p, False, E_dev=dev)
        rows = min(count, p.E)
        for out, form in ((kern, "device kernel"), (func, "functor")):
            out = out.cpu()
            assert bool((out[rows:].view(torch.int32) == ref.SENTINEL_BITS).all()), f"{form}, count {count}: a row at or past it was written"
            if rows:
                ref.compare(out[:rows], O64[:rows], A[:rows], C_AGG, f"{p.label()} E_dev={count} {form}")


# ---------------------------------------------------------------------------------------------------------------- fused GEMM tails
def _ssilu(x):
    return x * torch.sigmoid(x) / 0.6


def _gemm_case(M, N, K, epi, ldc=None, seed=0):
    g = torch.Generator().manual_seed(seed + M + N + K)
    ldc = N if ldc is None else ldc
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) * (2.0 / K) ** 0.5  # pre-activations of order 1, where the activation bends
    C = torch.randn(M, ldc, generator=g)
    o64 = A.double() @ W.double().T
    x64 = C[:, :N].double()
    want = _ssilu(o64) if epi == NB_EPI_ACT else (x64 + _ssilu(o64)) * ref.ISQ2
    return A.to(DEV), W.to(DEV), C.to(DEV), C.clone(), o64, x64, want, ldc


@pytest.mark.parametrize("M,N,K,epi,ldc", [
    (2350, 512, 512, NB_EPI_ACT, None),
    (2350, 64, 512, NB_EPI_ACT, None),
    (2350, 32, 512, NB_EPI_ACT, None),
    (2350, 256, 1280, NB_EPI_ACT, None),
    (2350, 512, 2560, NB_EPI_ACT, None),
    (4100, 256, 256, NB_EPI_ACT, 288),
    (2048, 512, 512, NB_EPI_RESIDUAL, None),
    (2049, 512, 512, NB_EPI_RESIDUAL, None),
    (2350, 512, 512, NB_EPI_RESIDUAL, 544),
    (9000, 512, 512, NB_EPI_RESIDUAL, None),
    (2048, 256, 256, NB_EPI_RESIDUAL, None),
    (2049, 256, 256, NB_EPI_RESIDUAL, None),
    (2350, 256, 256, NB_EPI_RESIDUAL, None),
    (9000, 256, 256, NB_EPI_RESIDUAL, 320),
])
def test_fused_tail_matches_fp64(M, N, K, epi, ldc):
    """C = ssilu(A W^T) (Dense + ScaledSiLU) or C = (C + ssilu(A W^T)) / sqrt 2 (ResidualLayer tail): within the GEMM's bound times the
    activation's slope; columns at and past N untouched."""
    A, W, C, C0, o64, x64, want, ldc = _gemm_case(M, N, K, epi, ldc)
    alpha = ref.ISQ2 if epi == NB_EPI_RESIDUAL else 1.0
    rc = _lib().nb200_gemm_tf32x3_epi(M, N, K, A.data_ptr(), K, W.data_ptr(), K, 0, C.data_ptr(), ldc, None, epi, NB_ACT_SSILU, alpha, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    C = C.cpu()
    got = C[:, :N].double()
    scale = float(o64.abs().max())
    tol = alpha * SLOPE * GEMM_REL * max(1.0, (K / 384) ** 0.5) * scale + 1e-6 * want.abs() + (2e-7 * x64.abs() if epi == NB_EPI_RESIDUAL else 0)
    err = (got - want).abs()
    print(f"fused tail epi={epi} {M}x{N}x{K} ldc={ldc}: max |err| / bound = {float((err / tol).max()):.2e}, max |err| / max|o| = {float(err.max()) / scale:.2e}")
    assert bool((err <= tol).all()), f"{int((err > tol).sum())} elements beyond the bound"
    if ldc > N:
        assert torch.equal(C[:, N:], C0[:, N:]), "columns at and past N were written"


def test_fused_tail_refusals():
    """A == C, epi = 0 (no tail) or 3: NB200_EINVAL; K % 4 != 0: NB200_EUNSUPPORTED; nothing is written."""
    M, N, K = 2350, 256, 256
    A, W, C, C0, *_ = _gemm_case(M, N, K, NB_EPI_ACT)
    f, s = _lib().nb200_gemm_tf32x3_epi, _stream()
    assert f(M, N, K, A.data_ptr(), K, W.data_ptr(), K, 0, A.data_ptr(), N, None, NB_EPI_ACT, NB_ACT_SSILU, 1.0, s) == EINVAL
    for epi in (0, 3):
        assert f(M, N, K, A.data_ptr(), K, W.data_ptr(), K, 0, C.data_ptr(), N, None, epi, NB_ACT_SSILU, 1.0, s) == EINVAL
    assert f(M, N, K - 2, A.data_ptr(), K, W.data_ptr(), K, 0, C.data_ptr(), N, None, NB_EPI_ACT, NB_ACT_SSILU, 1.0, s) == EUNSUPPORTED
    torch.cuda.synchronize()
    assert torch.equal(C.cpu(), C0), "a refused call wrote C"
    assert torch.equal(A.cpu(), _gemm_case(M, N, K, NB_EPI_ACT)[0].cpu()), "a refused call wrote A"
