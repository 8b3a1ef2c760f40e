"""GPU tests of the PhiSNet model kernels one C-ABI entry point at a time (csrc/phisnet_model.cu, and the exp-Bernstein / spherical-harmonics
edge basis of csrc/qhnet.cu), each against a float64 reference of the same operation built from the CPU oracle (oracle/phisnet.py,
oracle/phisnet_model.py) and evaluated on the same float32 inputs; then the whole model at the feature widths, elements and molecule sizes
the shipped-size tests of tests/test_gpu_phisnet_model.py do not reach.

Every kernel runs at num_features 32, 64, 96 and 128.  The pair kernels walk the CSR graph of nb200_neighbor_build (cutoff 1e4, as
nabladft_b200.phisnet does) of one batch holding a 1-atom molecule (an empty row), a 2-atom molecule, fixture molecule 0 and a 199-atom
synthetic molecule (long rows).  Outputs are pre-filled with NaN, so every row must be written, and carry a guard tail of GUARD rows holding
SENTINEL, which must survive.  Each check prints its measured error next to the assert."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
from make_golden_phisnet_model import HYPER, max_orbitals_from_db, model_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REL = 2e-6         # kernel outputs: of max|ref| per order L, or of the row's sum of |terms| where the kernel sums over pairs (worst 5.9e-7 measured)
REL_RBF = 1e-6     # exp-Bernstein basis: of each row's largest value (2.6e-7 measured; the all-fp32 kernel was 1.0e-5 at K = 128)
ABS_SH = 2e-6      # spherical harmonics, absolute (1.3e-6 measured)
REL_MODEL = 1e-5   # whole model: of each matrix's largest entry, as tests/test_gpu_phisnet_model.py (worst 3.9e-7 measured)
REL_BLOCK = 5e-6   # whole model: of each atom-pair block's own largest entry, for blocks of at least 1e-3 of the matrix max (worst 9.1e-7 measured)
GUARD = 64
SENTINEL = -1.25e30
FEATS = (32, 64, 96, 128)
KEYS = (("full", "full_hamiltonian"), ("core", "core_hamiltonian"), ("over", "overlap_matrix"))
EINVAL, EUNSUPPORTED = -1, -2


# ---------------------------------------------------------------------------------------------------------------- plumbing
def lib():
    from nabladft_b200 import _lib

    return _lib.load()


def P(t):
    from nabladft_b200._lib import ptr

    return ptr(t)


def call(fn, *args):
    from nabladft_b200 import _lib

    _lib.check(fn(*args, _lib.current_stream()), fn.__name__)


def guarded(rows, *shape):
    """(buffer [rows + GUARD, *shape], view of its first `rows` rows): NaN in the view, SENTINEL in the tail."""
    buf = torch.full((rows + GUARD, *shape), SENTINEL, dtype=torch.float32, device=DEV)
    buf[:rows] = float("nan")
    return buf, buf[:rows]


def assert_written(buf, rows, what):
    torch.cuda.synchronize()
    assert not bool(torch.isnan(buf[:rows]).any()), f"{what}: rows left unwritten (NaN from the pre-fill)"
    assert bool((buf[rows:] == SENTINEL).all()), f"{what}: written past the last row"


def split(x):
    """[R, 25, F] -> list over L of [R, 2L+1, F] (float64, CPU)."""
    x = x.double().cpu() if x.is_cuda else x.double()
    return [x[:, L * L:(L + 1) ** 2] for L in range(5)]


def order_of(lm):
    return 0 if lm < 1 else 1 if lm < 4 else 2 if lm < 9 else 3 if lm < 16 else 4


class Cols(torch.nn.Module):
    """Stands in for a coefficient Linear of the oracle: the kernels take the coefficients rbf . W^T ready-made, so the oracle reads the same
    float32 values as columns [a, b) of its `rbf` argument."""

    def __init__(self, a, b):
        super().__init__()
        self.a, self.b = a, b

    def forward(self, x):
        return x[..., self.a:self.b]


def cg():
    from oracle.phisnet import ClebschGordan

    return ClebschGordan()


def pair_mixing(F):
    """oracle PairMixing(4, 4, 4) whose path (l1, l2, L) number p reads coefficient columns [p F, (p + 1) F), as coeff[e][p][F] is laid out."""
    from oracle import phisnet as op

    pm = op.PairMixing(4, 4, 4, 1, F, cg())
    for p, (l1, l2, L) in enumerate(op.paths(4, 4, 4)):
        setattr(pm, f"coeff_{l1}_{l2}_{L}", Cols(p * F, (p + 1) * F))
    return pm


def angular(w, b):
    """oracle SphericalLinear(4, 1, 4, F, mix_orders=False) with weights w [5][F] and bias b [F] (angular_fn of the model)."""
    from oracle.phisnet import SphericalLinear

    F = w.shape[1]
    m = SphericalLinear(4, 1, 4, F, cg(), mix_orders=False).double()
    with torch.no_grad():
        for L in range(5):
            m.linear[L].weight.copy_(w[L].double().cpu()[:, None])
        m.linear[0].bias.copy_(b.double().cpu())
    return m


def report(what, err, scale, bound):
    r = float((err / scale).max())
    print(f"{what}: err / scale = {r:.2e} (bound {bound:.0e})")
    assert r <= bound, (what, r)
    return r


def per_L(got, ref, what, bound=REL):
    """|got - ref| <= bound * max|ref| per order L."""
    for L in range(5):
        err = (got[L] - ref[L]).abs().max()
        report(f"{what} L={L}", err, ref[L].abs().max().clamp_min(1e-30), bound)


def per_row_L(got, ref, absum, what, bound=REL):
    """|got - ref| <= bound * max(max|ref_L|, the row's float64 sum of |terms|) per row and order L."""
    worst = 0.0
    for L in range(5):
        err = (got[L] - ref[L]).abs().amax(dim=(1, 2))
        scale = torch.maximum(absum[L].amax(dim=(1, 2)), ref[L].abs().max().expand_as(err)).clamp_min(1e-30)
        worst = max(worst, report(f"{what} L={L}", err, scale, bound))
    return worst


# ---------------------------------------------------------------------------------------------------------------- pair graphs
def build_graph(pos, sizes):
    """The full pair graph of nabladft_b200.phisnet.NeuralNetwork._forward: device CSR (row_ptr, col, rev, tgt, geom [P, 4] = (u, d))."""
    L = lib()
    N, n_pairs = int(sum(sizes)), int(sum(n * (n - 1) for n in sizes))
    cap = max(n_pairs, 1)
    posd = torch.as_tensor(np.asarray(pos), dtype=torch.float32).to(DEV).contiguous()
    mol_ptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=DEV)
    I = lambda n: torch.empty(n, dtype=torch.int32, device=DEV)
    g = dict(row_ptr=I(N + 1), col=I(cap), rev=I(cap), tgt=I(cap), geom=torch.empty(cap, 4, device=DEV),
             status=torch.zeros(4, dtype=torch.int32, device=DEV))
    scratch = I(N)
    call(L.nb200_neighbor_build, P(posd), P(mol_ptr), len(sizes), N, 10000.0, 2 ** 31 - 1, cap, P(g["row_ptr"]), P(g["col"]), P(g["rev"]),
         P(g["geom"]), P(scratch), P(g["status"]))
    st = g["status"].cpu()
    assert int(st[0]) == n_pairs and int(st[1]) == 0, st
    call(L.nb200_qh_expand_rows, P(g["row_ptr"]), N, P(g["tgt"]))
    torch.cuda.synchronize()
    g.update(N=N, P=n_pairs, sizes=list(sizes), idx_i=g["tgt"][:n_pairs].long().cpu(), idx_j=g["col"][:n_pairs].long().cpu(),
             row_ptr_h=g["row_ptr"].long().cpu())
    return g


@pytest.fixture(scope="module")
def graph():
    """1-atom, 2-atom, fixture molecule 0 (38 atoms) and a 199-atom synthetic molecule; `sel` = atoms whose rows the references cover (all
    of the small molecules, 8 rows spread over the large one) and `sel_e` = their pairs."""
    from nabladft_b200.data import read_hamiltonian_db
    from nabladft_b200.synth import synth_batch
    from oracle.phisnet_model import NeuralNetwork as Oracle

    db = read_hamiltonian_db(os.path.join(GOLDEN, "hamiltonian_mol0.db"))
    big = synth_batch(11, 1, heavy_min=105, heavy_max=105)
    pos = np.concatenate([np.array([[0.5, -1.0, 2.0]]), np.array([[3.0, 0.0, 0.0], [3.4, 1.9, -0.7]]), db["pos"].astype(np.float64),
                          big["pos"].astype(np.float64) * 1.8897261])
    sizes = [1, 2, len(db["z"]), len(big["z"])]
    g = build_graph(pos, sizes)
    ii, jj = Oracle.pairs(sizes)
    assert torch.equal(g["idx_i"], ii) and torch.equal(g["idx_j"], jj), "CSR pair order differs from the reference's fill_idx order"
    sh = torch.empty(g["P"], 25, device=DEV)
    call(lib().nb200_qh_edge_basis, P(g["geom"]), P(g["status"]), g["P"], 0.5, 15.0, 1.0, None, 1, None, P(sh))
    g["sh"] = sh
    a0 = sum(sizes[:3])
    sel = list(range(a0)) + [int(a) for a in np.linspace(a0, a0 + sizes[3] - 1, 8).round()]
    g["sel"] = torch.tensor(sel)
    g["sel_e"] = torch.cat([torch.arange(int(g["row_ptr_h"][a]), int(g["row_ptr_h"][a + 1])) for a in sel])
    loc = torch.full((g["N"],), -1, dtype=torch.long)
    loc[g["sel"]] = torch.arange(len(sel))
    g["loc"] = loc
    g["empty_atom"], g["two_atoms"], g["big_rows"] = 0, torch.tensor([1, 2]), torch.tensor(sel[a0:])
    print(f"graph: {g['N']} atoms, {g['P']} pairs; references on {len(sel)} rows, {len(g['sel_e'])} pairs")
    return g


def rand(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen, device=DEV) * scale).contiguous()


def cuda_gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------- edge basis
@pytest.fixture(scope="module")
def probe_graph():
    """Pair distances from 0.05 bohr past 25 bohr, with pairs at exactly 12 and 15 bohr (QHNet's max_radius, PhiSNet's cutoff); plus fixture
    molecule 0 and a 2-atom molecule."""
    from nabladft_b200.data import read_hamiltonian_db

    rng = np.random.default_rng(2)
    dirs = rng.standard_normal((60, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    probe = np.concatenate([np.zeros((1, 3)), dirs * np.geomspace(0.05, 25.0, 60)[:, None], [[12.0, 0, 0], [0, 15.0, 0], [0, 0, -15.0]]])
    db = read_hamiltonian_db(os.path.join(GOLDEN, "hamiltonian_mol0.db"))
    pos = np.concatenate([probe, db["pos"].astype(np.float64), [[0.0, 0.0, 0.0], [0.0, 0.0, 14.99]]])
    return build_graph(pos, [len(probe), len(db["z"]), 2])


@pytest.mark.parametrize("caller,sign,cutoff,K", [("phisnet", 1.0, 15.0, 128), ("phisnet", 1.0, 15.0, 32), ("phisnet", 1.0, 15.0, 96),
                                                  ("phisnet", 1.0, 15.0, 160), ("qhnet", -1.0, 12.0, 32)])
def test_edge_basis_matches_fp64(probe_graph, caller, sign, cutoff, K):
    """nb200_qh_edge_basis against ExponentialBernsteinRadialBasisFunctions and spherical_harmonics of the oracle, evaluated in float64 at the
    float32 distance and direction stored in geom, so that position rounding is not counted."""
    from oracle.phisnet_model import ExponentialBernsteinRadialBasisFunctions, spherical_harmonics

    g = probe_graph
    n = g["P"]
    rb = ExponentialBernsteinRadialBasisFunctions(K, cutoff).double()
    alpha = float(torch.nn.functional.softplus(rb._alpha.detach()))
    logc = rb.logc.to(DEV).contiguous()
    rbuf, rbf = guarded(n, K)
    sbuf, sh = guarded(n, 25)
    call(lib().nb200_qh_edge_basis, P(g["geom"]), P(g["status"]), n, alpha, cutoff, sign, P(logc), K, P(rbf), P(sh))
    assert_written(rbuf, n, "rbf")
    assert_written(sbuf, n, "sh")
    geom = g["geom"][:n].double().cpu()
    d = geom[:, 3:]
    print(f"{caller} K={K}: {n} pairs, d from {float(d.min()):.3f} to {float(d.max()):.2f} bohr")
    with torch.no_grad():
        ref = rb(d)
    got = rbf.double().cpu()
    out = (d[:, 0] >= cutoff)
    assert int(out.sum()) >= 3 and bool((d[:, 0] == cutoff).any()), "the probe must reach and pass the cutoff"
    assert bool((got[out] == 0).all()), "the basis must be exactly 0 at and beyond the cutoff"
    # a row whose float64 values all lie below float32's smallest normal (d within ~0.3 bohr of the cutoff, where the cutoff function is
    # below 1e-38) cannot carry a relative error: it must be below that normal in absolute value
    tiny = torch.finfo(torch.float32).tiny
    inside = ~out & (ref.abs().amax(dim=1) >= tiny)
    under = ~out & ~inside
    assert bool((got[under].abs() <= tiny).all())
    print(f"  {int(inside.sum())} rows inside the cutoff, {int(under.sum())} below float32's range, {int(out.sum())} at or past the cutoff")
    err = (got[inside] - ref[inside]).abs().amax(dim=1)
    scale = ref[inside].abs().amax(dim=1)
    r = err / scale
    for lo, hi in ((0.0, 1.0), (1.0, 5.0), (5.0, 10.0), (10.0, 13.5), (13.5, cutoff)):
        m = (d[inside, 0] >= lo) & (d[inside, 0] < hi)
        if bool(m.any()):
            print(f"  d in [{lo}, {hi}): max err / row max = {float(r[m].max()):.2e}")
    report(f"{caller} K={K} rbf", err, scale, REL_RBF)
    u = geom[:, :3] * sign
    ref_sh = torch.cat(spherical_harmonics(u), dim=-1)
    err_sh = (sh.double().cpu() - ref_sh).abs().max()
    print(f"{caller} sh: max abs err = {float(err_sh):.2e} (bound {ABS_SH:.0e})")
    assert float(err_sh) <= ABS_SH


# ---------------------------------------------------------------------------------------------------------------- atom-row kernels
@pytest.mark.parametrize("rows", [37, 2051])
@pytest.mark.parametrize("F", FEATS)
@pytest.mark.parametrize("act", [True, False], ids=["swish", "noswish"])
def test_swish_self_mixing_matches_fp64(F, rows, act):
    from oracle.phisnet import SelfMixing, paths
    from oracle.phisnet_model import Swish

    gen = cuda_gen(F * 7 + rows + act)
    x = rand(gen, rows, 25, F)
    alpha = (1.0 + rand(gen, F, scale=0.1)) if act else None
    beta = (1.702 + rand(gen, F, scale=0.1)) if act else None
    pth = paths(4, 4, 4, strict_upper=True)
    mix, keep = rand(gen, len(pth), F, scale=0.5), rand(gen, 5, F, scale=0.5)
    buf, y = guarded(rows, 25, F)
    call(lib().nb200_phis_swish_self_mixing, P(x), P(alpha), P(beta), P(mix), P(keep), rows, F, P(y))
    assert_written(buf, rows, "swish_self_mixing")
    sm = SelfMixing(4, 4, F, cg()).double()
    with torch.no_grad():
        for p, (l1, l2, L) in enumerate(pth):
            getattr(sm, f"mixcoeff_{l1}_{l2}_{L}").copy_(mix[p].double().cpu())
        for L in range(5):
            getattr(sm, f"keepcoeff_{L}").copy_(keep[L].double().cpu())
        xs = split(x)
        if act:
            sw = Swish(F).double()
            sw.alpha.copy_(alpha.double().cpu())
            sw.beta.copy_(beta.double().cpu())
            xs[0] = sw(xs[0])
        ref = sm(xs)
    per_L(split(y), ref, f"swish_self_mixing F={F} rows={rows} act={act}")


@pytest.mark.parametrize("rows", [37, 2051])
@pytest.mark.parametrize("F", FEATS)
@pytest.mark.parametrize("accumulate", [0, 1])
def test_linear_ex_matches_fp64(F, rows, accumulate):
    """Per-order Linear y[:, lm] (+)= x[:, lm] W_l[order(lm)] (+ bias on L = 0): the plain GEMM below 2048 rows, the tall per-order GEMM
    at 2051 (a partial row tile; a partial 96-column tile at F = 96)."""
    gen = cuda_gen(F * 5 + rows + accumulate)
    x, W, b = rand(gen, rows, 25, F), rand(gen, 5, F, F, scale=F ** -0.5), rand(gen, F)
    y0 = rand(gen, rows, 25, F)
    buf, y = guarded(rows, 25, F)
    if accumulate:
        y.copy_(y0)
    call(lib().nb200_phis_linear_ex, P(x), P(W), P(b), rows, F, F, 4, accumulate, P(y))
    assert_written(buf, rows, "linear_ex")
    xd, Wd = x.double().cpu(), W.double().cpu()
    ref = torch.stack([xd[:, lm] @ Wd[order_of(lm)] for lm in range(25)], dim=1)
    ref[:, 0] += b.double().cpu()
    if accumulate:
        ref += y0.double().cpu()
    per_L(split(y), split(ref), f"linear_ex F={F} rows={rows} acc={accumulate}")


@pytest.mark.parametrize("K", [32, 96, 128, 160])
@pytest.mark.parametrize("F", FEATS)
def test_coefficient_gemm_matches_fp64(F, K):
    """nb200_dense(rbf, W) as the model forms its pair coefficients: N = 65F (mix_s), 70F (interaction), 75F (pair features), plain and
    tall row counts."""
    gen = cuda_gen(F * 3 + K)
    for rows in (1000, 2051):
        A = torch.rand(rows, K, generator=gen, device=DEV)
        for n in (65 * F, 70 * F, 75 * F):
            Wt = rand(gen, n, K, scale=K ** -0.5)
            buf, y = guarded(rows, n)
            call(lib().nb200_dense, rows, n, K, P(A), K, P(Wt), K, 0, P(y), n, 0, None, None, 0)
            assert_written(buf, rows, "dense")
            ref = A.double().cpu() @ Wt.double().cpu().T
            err = (y.double().cpu() - ref).abs().max()
            report(f"dense rows={rows} N={n} K={K}", err, ref.abs().max(), REL)


# ---------------------------------------------------------------------------------------------------------------- pair kernels
@pytest.mark.parametrize("F", FEATS)
def test_interaction_matches_fp64(graph, F):
    """yi.index_add(idx_i, PairMixing(yj[idx_j], angular_fn1(sph), rbf) + radial_fn_L(rbf) angular_fn2(sph)_L yj[idx_j]_0)
    (InteractionBlock.forward of the oracle without its residual stacks)."""
    g = graph
    N, n = g["N"], g["P"]
    gen = cuda_gen(100 + F)
    yi, yj = rand(gen, N, 25, F), rand(gen, N, 25, F)
    coeff = rand(gen, n, 70 * F, scale=0.5)
    wa1, ba1, wa2, ba2 = rand(gen, 5, F), rand(gen, F), rand(gen, 5, F), rand(gen, F)
    buf, y = guarded(N, 25, F)
    call(lib().nb200_phis_interaction, P(yi), P(yj), P(g["sh"]), P(coeff), P(wa1), P(ba1), P(wa2), P(ba2), P(g["row_ptr"]), P(g["col"]),
         N, F, P(y))
    assert_written(buf, N, "interaction")
    a = g["empty_atom"]
    assert torch.equal(y[a], yi[a]), "an atom without pairs must come out as yi"
    e, sel, loc = g["sel_e"], g["sel"], g["loc"]
    ii, jj = g["idx_i"][e], g["idx_j"][e]
    c = coeff[e.to(DEV)].double().cpu()[:, None, :]
    sph = split(g["sh"][e.to(DEV)][:, :, None])  # [pairs, 2L+1, 1]
    with torch.no_grad():
        yjs = [t[jj] for t in split(yj)]
        vs = pair_mixing(F).double()(yjs, angular(wa1, ba1)(sph), c)
        a2 = angular(wa2, ba2)(sph)
        terms = [vs[L] + c[..., (65 + L) * F:(66 + L) * F] * a2[L] * yjs[0] for L in range(5)]
    yis = [t[sel] for t in split(yi)]
    ref = [yis[L].index_add(0, loc[ii], terms[L]) for L in range(5)]
    absum = [yis[L].abs().index_add(0, loc[ii], terms[L].abs()) for L in range(5)]
    per_row_L([t[sel] for t in split(y)], ref, absum, f"interaction F={F}")


@pytest.mark.parametrize("F", FEATS)
def test_pair_features_match_fp64(graph, F):
    """fii = fpc.index_add(idx_i, radial_ii(rbf) fpn[idx_j]) and fij = mix_ij(fpc[idx_i], fpc[idx_j], rbf) + the neighbour sum
    sum_{k != i, j} radial_ij(rbf_ik) fpn[k] (oracle NeuralNetwork.forward and pair_neighbour_sum); coeff = [65 mix_ij | radial_ii | radial_ij]."""
    from oracle.phisnet_model import NeuralNetwork as Oracle

    g = graph
    N, n = g["N"], g["P"]
    gen = cuda_gen(200 + F)
    fpc, fpn = rand(gen, N, 25, F), rand(gen, N, 25, F)
    coeff = rand(gen, n, 75 * F, scale=0.5)
    e, sel, loc = g["sel_e"], g["sel"], g["loc"]
    ii, jj = g["idx_i"][e], g["idx_j"][e]
    c = coeff[e.to(DEV)].double().cpu()[:, None, :]
    fpcs, fpns = split(fpc), split(fpn)
    radial_ij = types.SimpleNamespace(order=4, radial_ij=[Cols((70 + L) * F, (71 + L) * F) for L in range(5)])
    for neighbour_only in (False, True):
        cf = coeff
        if neighbour_only:  # mixing paths and radial_ii off: fij is the neighbour sum alone
            cf = coeff.clone()
            cf[:, :70 * F] = 0
        ibuf, fii = guarded(N, 25, F)
        jbuf, fij = guarded(n, 25, F)
        call(lib().nb200_phis_pair_features, P(fpc), P(fpn), P(cf), P(g["row_ptr"]), P(g["col"]), N, F, P(fii), P(fij))
        assert_written(ibuf, N, "fii")
        assert_written(jbuf, n, "fij")
        c_ = cf[e.to(DEV)].double().cpu()[:, None, :]
        with torch.no_grad():
            rii = [c_[..., (65 + L) * F:(66 + L) * F] * fpns[L][jj] for L in range(5)]
            ref_ii = [fpcs[L][sel].index_add(0, loc[ii], rii[L]) for L in range(5)]
            abs_ii = [fpcs[L][sel].abs().index_add(0, loc[ii], rii[L].abs()) for L in range(5)]
            mixed = pair_mixing(F).double()([t[ii] for t in fpcs], [t[jj] for t in fpcs], c_)
            ref_ij = Oracle.pair_neighbour_sum(radial_ij, mixed, fpns, c_, ii, jj)
            rij = [c_[..., (70 + L) * F:(71 + L) * F] * fpns[L][jj] for L in range(5)]
            T_abs = [torch.zeros_like(fpns[L]).index_add(0, ii, rij[L].abs()) for L in range(5)]
            abs_ij = [T_abs[L][ii] + mixed[L].abs() for L in range(5)]
        tag = f"F={F}" + (" neighbour sum only" if neighbour_only else "")
        if not neighbour_only:
            a = g["empty_atom"]
            assert torch.equal(fii[a], fpc[a]), "an atom without pairs must come out as fpc"
        per_row_L([t[sel] for t in split(fii)], ref_ii, abs_ii, f"fii {tag}")
        got_ij = [t[e] for t in split(fij)]
        per_row_L(got_ij, ref_ij, abs_ij, f"fij {tag}")
        if neighbour_only:
            # the 2-atom molecule: T_i - own term cancels to 0; the 199-atom rows: the largest cancellation, against the sum of |terms|
            two = torch.isin(ii, g["two_atoms"])
            big = torch.isin(ii, g["big_rows"])
            for what, m in (("2-atom", two), ("199-atom", big)):
                err = max(float((got_ij[L][m] - ref_ij[L][m]).abs().max() / abs_ij[L][m].abs().max()) for L in range(5))
                print(f"neighbour sum F={F} {what} rows: err / sum|terms| = {err:.2e}")
                assert err <= REL, (what, err)
            assert max(float(ref_ij[L][two].abs().max()) for L in range(5)) == 0.0


@pytest.mark.parametrize("F", FEATS)
def test_overlap_pairs_match_fp64(graph, F):
    """s_ij = mix_s(x[idx_i], [x[idx_j]_0] + angular_fn(sph)[1:], rbf) (oracle NeuralNetwork.forward, overlap branch)."""
    g = graph
    N, n = g["N"], g["P"]
    gen = cuda_gen(300 + F)
    x = rand(gen, N, 25, F)
    coeff = rand(gen, n, 65 * F, scale=0.5)
    wa, ba = rand(gen, 5, F), rand(gen, F)
    buf, s = guarded(n, 25, F)
    call(lib().nb200_phis_overlap_pairs, P(x), P(g["sh"]), P(coeff), P(wa), P(g["row_ptr"]), P(g["col"]), N, F, P(s))
    assert_written(buf, n, "overlap_pairs")
    e = g["sel_e"]
    ii, jj = g["idx_i"][e], g["idx_j"][e]
    c = coeff[e.to(DEV)].double().cpu()[:, None, :]
    sph = split(g["sh"][e.to(DEV)][:, :, None])
    xs = split(x)
    with torch.no_grad():
        a = angular(wa, ba)(sph)
        ref = pair_mixing(F).double()([t[ii] for t in xs], [xs[0][jj]] + a[1:], c)
    per_L([t[e] for t in split(s)], ref, f"overlap_pairs F={F}")


# ---------------------------------------------------------------------------------------------------------------- assembly
def element_batch():
    """(pos bohr float64, Z, sizes): a 1-atom Br molecule, a 2-atom S-H molecule and a 23-atom synthetic molecule whose heavy atoms are
    overwritten with C N O F S Cl Br Br ... -- every element of the fixture DB's max_orbitals, two Br atoms (the 32 x 32 Br-Br block) in one
    molecule."""
    from nabladft_b200.synth import synth_batch

    sb = synth_batch(5, 1, heavy_min=12, heavy_max=12)
    z = sb["z"].astype(np.int64).copy()
    heavy = np.flatnonzero(z != 1)
    assert len(heavy) >= 8
    z[heavy[:8]] = [6, 7, 8, 9, 16, 17, 35, 35]
    pos = np.concatenate([[[1.0, 2.0, -0.5]], [[0.0, 0.0, 0.0], [0.7, 2.3, 0.4]], sb["pos"].astype(np.float64) * 1.8897261])
    pos = pos.astype(np.float32).astype(np.float64)  # both sides see the same positions
    return pos, np.concatenate([[35, 16, 1], z]), [1, 2, len(z)]


@pytest.mark.parametrize("F", FEATS)
def test_assemble_matches_fp64(F):
    """nb200_phis_assemble against the output SphericalLinear's per-order Linear followed by NeuralNetwork._assemble of the oracle, with the
    head widths of irreps_tables(max_orbitals_from_db()), unit_diagonal 0 and 1."""
    from nabladft_b200.phisnet import assembly_tables, irreps_tables
    from oracle.phisnet_model import NeuralNetwork as Oracle
    from oracle.phisnet_model import _irreps

    max_orb = tuple(tuple((int(z), int(l)) for z, l in o) for o in max_orbitals_from_db())
    pos, Z, sizes = element_batch()
    g = build_graph(pos, sizes)
    N, n = g["N"], g["P"]
    ii_tab, w_ii, ij_tab, w_ij = irreps_tables(max_orb)
    a = assembly_tables(max_orb, ii_tab, ij_tab)
    assert not a["missing"]
    elems = a["elems"]
    assert set(elems) <= set(Z.tolist()) and int((Z[3:] == 35).sum()) == 2
    gen = cuda_gen(400 + F)
    Xd, Xo = rand(gen, N, 25, F), rand(gen, n, 25, F)
    Wd, bd = rand(gen, 5, w_ii, F, scale=F ** -0.5), rand(gen, w_ii)
    Wo, bo = rand(gen, 5, w_ij, F, scale=F ** -0.5), rand(gen, w_ij)
    el_of_z = {z: i for i, z in enumerate(elems)}
    el = torch.tensor([el_of_z[int(z)] for z in Z], dtype=torch.int32, device=DEV)
    T = {k: torch.from_numpy(np.ascontiguousarray(a[k]).reshape(-1)).to(DEV) for k in ("row_orb", "row_m", "orb_l", "n_rows", "ent_range",
                                                                                       "op_base", "ent_col", "ent_L")}
    norb = np.array([int(a["n_rows"][el_of_z[int(z)]]) for z in Z])
    atom_mol = np.repeat(np.arange(len(sizes)), sizes)
    starts = np.concatenate([[0], np.cumsum(sizes)])
    atom_off = np.concatenate([np.concatenate([[0], np.cumsum(norb[s:e])[:-1]]) for s, e in zip(starts[:-1], starts[1:])])
    mol_norb = np.array([norb[s:e].sum() for s, e in zip(starts[:-1], starts[1:])])
    mol_off = np.concatenate([[0], np.cumsum(mol_norb ** 2)])
    i32 = lambda v: torch.tensor(np.asarray(v), dtype=torch.int32, device=DEV)
    atom_mol_d, atom_off_d, mol_norb_d = i32(atom_mol), i32(atom_off), i32(mol_norb)  # held: a pointer does not keep its tensor alive
    mol_off_d = torch.tensor(mol_off, dtype=torch.int64, device=DEV)
    total = int(mol_off[-1])
    ns = types.SimpleNamespace(elem_orbs={o[0][0]: o for o in max_orb}, cg=cg())
    ns.irreps_ii, _, ns.irreps_ij, _, _ = _irreps(max_orb)
    out_lin = lambda X, W, b: [torch.einsum("rmf,cf->rmc", x, W[L].double().cpu()) + (b.double().cpu() if L == 0 else 0)
                               for L, x in enumerate(split(X))]
    with torch.no_grad():
        fd, fo = out_lin(Xd, Wd, bd), out_lin(Xo, Wo, bo)
    for unit in (0, 1):
        buf, M = guarded(total)
        call(lib().nb200_phis_assemble, P(Xd), P(Xo), P(Wd), P(bd), w_ii, P(Wo), P(bo), w_ij, F, P(el), P(T["row_orb"]), P(T["row_m"]),
             P(T["orb_l"]), P(T["n_rows"]), P(T["ent_range"]), P(T["op_base"]), P(T["ent_col"]), P(T["ent_L"]), len(elems), a["max_ent"],
             P(g["tgt"]), P(g["col"]), P(g["rev"]), N, n, P(atom_mol_d), P(atom_off_d), P(mol_off_d), P(mol_norb_d), unit, P(M))
        assert_written(buf, total, "assemble")
        with torch.no_grad():
            ref = Oracle._assemble(ns, fd, fo, torch.from_numpy(Z), sizes, g["idx_i"], g["idx_j"], unit)
        for m in range(len(sizes)):
            got = M[int(mol_off[m]):int(mol_off[m + 1])].view(int(mol_norb[m]), int(mol_norb[m]))
            assert torch.equal(got, got.T), "matrices must be exactly symmetric"
            if unit:
                assert bool((torch.diagonal(got) == 1).all())
            err = (got.double().cpu() - ref[m]).abs().max()
            report(f"assemble F={F} unit={unit} mol {m} ({sizes[m]} atoms, {int(mol_norb[m])} orbitals)", err, ref[m].abs().max(), REL)


# ---------------------------------------------------------------------------------------------------------------- argument checks
def _arg_cases():
    """Per entry point: (name, argument list with a count of 0, indices of required pointers, indices of the feature-width arguments,
    indices of outputs).  Every pointer is a small valid device buffer, and every case keeps the count at 0, so no kernel is launched."""
    b = lambda *s: torch.full(s, SENTINEL, device=DEV)
    i = lambda n: torch.zeros(n, dtype=torch.int32, device=DEV)
    F = 32
    x, w, out, out2 = b(4, 25, F), b(64, F), b(4, 25, F), b(4, 25, F)
    rp = i(2)
    asm = [b(4, 25, F), b(4, 25, F), b(5, 8, F), b(8), 8, b(5, 8, F), b(8), 8, F] + [i(64) for _ in range(9)] + [1, 1] + [i(4)] * 3 + [0, 0] \
        + [i(4), i(4), torch.zeros(2, dtype=torch.int64, device=DEV), i(4), 0, out]
    return [
        ("nb200_phis_swish_self_mixing", [x, w, w, w, w, 0, F, out], (0, 3, 4, 7), (6,), (7,)),
        ("nb200_phis_linear_ex", [x, b(5, F, F), w, 0, F, F, 4, 0, out], (0, 1, 8), (4, 5), (8,)),
        ("nb200_phis_interaction", [x, x, w, w, w, w, w, w, rp, rp, 0, F, out], tuple(range(10)) + (12,), (11,), (12,)),
        ("nb200_phis_pair_features", [x, x, w, rp, rp, 0, F, out, out2], (0, 1, 2, 3, 4, 7, 8), (6,), (7, 8)),
        ("nb200_phis_overlap_pairs", [x, w, w, w, rp, rp, 0, F, out], (0, 1, 2, 3, 4, 5, 8), (7,), (8,)),
        ("nb200_phis_assemble", asm, (0, 2, 3) + tuple(range(9, 18)) + (25, 26, 27, 28, 30), (8,), (30,)),
    ]


def _raw(name, args):
    from nabladft_b200._lib import current_stream

    conv = [P(a) if isinstance(a, torch.Tensor) else a for a in args]
    return getattr(lib(), name)(*conv, current_stream())


@pytest.mark.parametrize("case", ["nb200_phis_swish_self_mixing", "nb200_phis_linear_ex", "nb200_phis_interaction",
                                  "nb200_phis_pair_features", "nb200_phis_overlap_pairs", "nb200_phis_assemble"])
def test_argument_checks(case):
    """n_feat 48 -> NB200_EUNSUPPORTED, a null required pointer -> NB200_EINVAL, a count of 0 -> NB200_OK with nothing written."""
    name, args, required, feat, outs = next(c for c in _arg_cases() if c[0] == case)
    assert _raw(name, args) == 0
    torch.cuda.synchronize()
    for k in outs:
        assert bool((args[k] == SENTINEL).all()), f"{name}: a count of 0 wrote output {k}"
    for k in required:
        bad = list(args)
        bad[k] = None
        assert _raw(name, bad) == EINVAL, (name, "null argument", k)
    bad = list(args)
    for k in feat:
        bad[k] = 48
    assert _raw(name, bad) == EUNSUPPORTED, (name, "n_feat 48")
    if name == "nb200_phis_swish_self_mixing":  # alpha without beta
        bad = list(args)
        bad[2] = None
        assert _raw(name, bad) == EINVAL
    if name == "nb200_phis_assemble":  # pair inputs may be null only without pairs
        for k in (1, 5, 6, 20, 21, 22):
            bad = list(args)
            bad[k], bad[24] = None, 1
            assert _raw(name, bad) == EINVAL, (name, "null pair argument", k)
        bad = list(args)
        for k in (1, 5, 6, 20, 21, 22):
            bad[k] = None
        assert _raw(name, bad) == 0
    torch.cuda.synchronize()
    for k in outs:
        assert bool((args[k] == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------- whole model
def load_pair(hyper):
    from nabladft_b200 import phisnet as ph
    from oracle.phisnet_model import NeuralNetwork as Oracle

    m = ph.NeuralNetwork(max_orbitals=max_orbitals_from_db(), **hyper)
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v).to(sd[k].dtype) for k, v in model_state_dict(sd).items()}, strict=True)
    m = m.to(DEV).eval()
    ora = Oracle(max_orbitals_from_db(), **hyper).double()
    ora.load_state_dict({k: v.detach().cpu().double() for k, v in m.state_dict().items()}, strict=True)
    return m, ora


def run_both(m, ora, pos, Z, sizes):
    table = {o[0][0]: o for o in m.max_orbitals}
    batch = {"positions": torch.as_tensor(pos, dtype=torch.float32).to(DEV), "atomic_numbers": torch.as_tensor(Z).long().to(DEV),
             "orbitals": tuple(table[int(z)] for z in Z), "molecule_size": torch.as_tensor(sizes).long()}
    got = m(batch, packed=True)
    ref = ora(torch.from_numpy(np.asarray(pos, dtype=np.float32).astype(np.float64)), torch.as_tensor(Z).long(), sizes)
    return got, ref


@pytest.fixture(scope="module", params=[(32, 32), (64, 96), (96, 160)], ids=lambda p: f"F{p[0]}-K{p[1]}")
def width_model(request):
    F, K = request.param
    return (F, K) + load_pair(dict(HYPER, num_features=F, num_basis_functions=K, num_modules=2))


def test_model_widths_and_edges_match_oracle(width_model):
    """All three heads at F/K = 32/32, 64/96, 96/160 on a 1-atom Br molecule, a 2-atom molecule and a molecule with every element of
    max_orbitals and two Br atoms, against the float64 oracle: of each matrix's max, and per atom-pair block of the block's own max."""
    F, K, m, ora = width_model
    pos, Z, sizes = element_batch()
    got, ref = run_both(m, ora, pos, Z, sizes)
    table = {o[0][0]: o for o in m.max_orbitals}
    norb = [sum(2 * l + 1 for _, l in table[int(z)]) for z in Z]
    a0 = 0
    for mol, n_at in enumerate(sizes):
        offs = np.concatenate([[0], np.cumsum(norb[a0:a0 + n_at])])
        for tag, key in KEYS:
            g = got[key][mol].double().cpu()
            r = ref[tag][mol]
            assert not bool(torch.isnan(g).any()) and torch.equal(got[key][mol], got[key][mol].T)
            mx = float(r.abs().max())
            err = float((g - r).abs().max()) / mx
            worst, where = 0.0, None
            for p in range(n_at):
                for q in range(n_at):
                    rb = r[offs[p]:offs[p + 1], offs[q]:offs[q + 1]]
                    bmax = float(rb.abs().max())
                    if bmax < 1e-3 * mx:
                        continue
                    be = float((g[offs[p]:offs[p + 1], offs[q]:offs[q + 1]] - rb).abs().max()) / bmax
                    if be > worst:
                        worst, where = be, (int(Z[a0 + p]), int(Z[a0 + q]))
            print(f"F={F} K={K} mol {mol} ({n_at} atoms) {tag}: err / matrix max = {err:.2e}; worst block err / block max = {worst:.2e} "
                  f"(Z pair {where})")
            assert err < REL_MODEL, (F, K, mol, tag, err)
            assert worst < REL_BLOCK, (F, K, mol, tag, worst, where)
        a0 += n_at


def test_model_config_size_slice_matches_oracle():
    """The bench's batch (synth_batch(1, 32), bohr) at the shipped hyperparameters: the first two molecules of the batch-32 forward against
    the float64 oracle run on those two molecules alone."""
    from nabladft_b200.synth import synth_batch

    m, ora = load_pair(HYPER)
    b = synth_batch(1, 32)
    sizes = np.diff(b["mol_ptr"]).tolist()
    pos = (b["pos"].astype(np.float64) * 1.8897261).astype(np.float32)
    Z = b["z"].astype(np.int64)
    table = {o[0][0]: o for o in m.max_orbitals}
    batch = {"positions": torch.from_numpy(pos).to(DEV), "atomic_numbers": torch.from_numpy(Z).to(DEV),
             "orbitals": tuple(table[int(z)] for z in Z), "molecule_size": torch.tensor(sizes)}
    got = m(batch, packed=True)
    n2 = sizes[0] + sizes[1]
    ref = ora(torch.from_numpy(pos[:n2].astype(np.float64)), torch.from_numpy(Z[:n2]), sizes[:2])
    for tag, key in KEYS:
        for mol in range(2):
            r = ref[tag][mol]
            err = float((got[key][mol].double().cpu() - r).abs().max() / r.abs().max())
            print(f"batch-32 slice mol {mol} ({sizes[mol]} atoms) {tag}: err / matrix max = {err:.2e}")
            assert err < REL_MODEL, (tag, mol, err)
