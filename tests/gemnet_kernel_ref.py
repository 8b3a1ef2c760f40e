"""Float64 references of the GemNet-OC edge aggregations (csrc/gemnet_oc_kernels.cuh TripEdgeK / QuadK, their tangents TripEdgeTK / QuadTK,
and the device kernels that stand in for them) and a builder of synthetic CSR graphs to run them on.  Helper module of
tests/test_gemnet_kernels_emu.py and tests/test_gpu_gemnet_kernels.py, not a test file.

The operations are restated from their definitions (oracle/gemnet_oc.py, efficient.py of the reference model), not ported from the kernels:
  Y_l(z) = sqrt((2l + 1) / 4 pi) P_l(z), l = 0..6, P_l from numpy's Legendre series;
  triplet     O[e, 64 i + ch] = sum_s R[e, 7 i + s] sum_{k in in-row(tgt e), in.src[k] != src e} Y_s(clamp(V_e . V_k)) x[k, ch]
  quadruplet  O[e, 32 i + ch] = sum_{l1, l2} R[e, 49 i + 7 l1 + l2] sum_{qe in q-row(a), b != c} sum_{k in mn-row(b), d not in {a, c}}
                                Y_l1(clamp(V_ca . V_ba)) Y_l2(cos phi) x_t[q_tin[qe] + k - mn.ptr[b], ch]
              n1 = V_ca x V_ba, n2 = V_db x V_ba, xx = n1 . n2, yy = max(|n1 x n2|, 1e-9), cos phi = xx / sqrt(xx^2 + yy^2).
Tangents are torch.func.jvp of the same float64 functions.  Each output element also gets a magnitude bound A: the same sums over the absolute
value of every factor (primal and tangent); tolerances are multiples of A, so an empty or fully excluded row must come out exactly 0.

Graphs are synthetic, not molecules, so that row lengths, excluded positions and vectors can be chosen freely.  They keep what the kernels
rely on: rows by target with a monotone ptr, src / tgt consistent with the rows, sources distinct within a row and never the target,
unit vectors V (float32), and q_tin[qe] the running slot base over the mn-rows of the qint sources, as FillK lays it out."""
import numpy as np
import torch

NS, TI, QI = 7, 64, 32
LDR_TRIP, LDR_QUAD = 16 * NS, 32 * NS * NS
YY_MIN = float(np.float32(1e-9))  # the kernels' clamp of |n1 x n2|, a float32 constant
ISQ2 = float(np.float32(2 ** -0.5))  # the ResidualLayer's 1 / sqrt 2 as the kernels hold it
CHUNK = 1 << 15                   # terms per float64 chunk: [CHUNK, 49, 32] doubles = 400 MB at most, the tangent's dual included


def _legendre_power_coeffs(deriv: int) -> torch.Tensor:
    """[NS, NS] power-series coefficients (column p = z^p) of the deriv-th derivative of Y_l."""
    C = np.zeros((NS, NS))
    for l in range(NS):
        c = np.polynomial.legendre.leg2poly([0.0] * l + [1.0]) * np.sqrt((2 * l + 1) / (4 * np.pi))
        c = np.polynomial.polynomial.polyder(c, deriv) if deriv else c
        C[l, :len(c)] = c
    return torch.tensor(C, dtype=torch.float64)


_Y, _DY = _legendre_power_coeffs(0), _legendre_power_coeffs(1)


def sph(z: torch.Tensor) -> torch.Tensor:
    """[..., 7]: Y_l(z)."""
    return torch.stack([z ** p for p in range(NS)], -1) @ _Y.T


def dsph(z: torch.Tensor) -> torch.Tensor:
    """[..., 7]: dY_l / dz."""
    return torch.stack([z ** p for p in range(NS)], -1) @ _DY.T


def clamp1(c: torch.Tensor) -> torch.Tensor:
    """clamp to [-1, 1] whose derivative is 1 on the closed interval and 0 outside (torch.clamp's, the oracle's _clamped_dot's)."""
    one = torch.ones_like(c)
    return torch.where(c > 1, one, torch.where(c < -1, -one, c))


def absdot(a, b):
    return (a.abs() * b.abs()).sum(-1)


# ------------------------------------------------------------------------------------------------------------------- graphs
class Graph:
    """CSR rows by target: ptr [n + 1], src / tgt [ne] int32, V [ne, 3] float32 (unit vectors source -> target)."""

    def __init__(self, n, rows, V):
        """rows[a]: list of the sources of target a (distinct, != a); V[a]: [len(rows[a]), 3] vectors."""
        self.n = n
        deg = np.array([len(rows.get(a, ())) for a in range(n)], dtype=np.int64)
        self.ptr = np.zeros(n + 1, dtype=np.int32)
        self.ptr[1:] = np.cumsum(deg)
        self.src = np.concatenate([np.asarray(rows.get(a, []), dtype=np.int32) for a in range(n)] + [np.zeros(0, np.int32)])
        self.tgt = np.repeat(np.arange(n, dtype=np.int32), deg)
        self.V = np.concatenate([np.asarray(V[a], dtype=np.float32).reshape(-1, 3) for a in range(n) if deg[a]] + [np.zeros((0, 3), np.float32)])
        for a in range(n):
            s = self.src[self.ptr[a]:self.ptr[a + 1]]
            assert len(set(s.tolist())) == len(s) and a not in s, "sources distinct within a row and never the target"
        assert np.all(np.abs(np.linalg.norm(self.V.astype(np.float64), axis=1) - 1) < 1e-6)

    @property
    def ne(self):
        return int(self.ptr[-1])

    def row(self, a):
        return range(int(self.ptr[a]), int(self.ptr[a + 1]))


def unit(rng, k, planar=False):
    """k random float32 unit vectors; planar: z = 0 exactly."""
    v = rng.standard_normal((k, 3))
    if planar:
        v[:, 2] = 0
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def overshoot_vector():
    """A float32 unit vector v whose exact v . v exceeds 1 by more than 2 ulp(1): its float32 dot product with itself rounds past 1 however
    it is summed, so clamp1 is active in the kernels and in the reference alike."""
    u = unit(np.random.default_rng(7), 1)[0].astype(np.float64)
    for step in range(1, 16):
        v = (u * (1 + step * 2.0 ** -24)).astype(np.float32)
        if (v.astype(np.float64) ** 2).sum() > 1 + 2.5 * 2.0 ** -23:
            return v
    raise AssertionError("no float32 vector found")


def q_slot_bases(mn: Graph, q: Graph) -> np.ndarray:
    """q_tin [Q + 1]: the running sum of deg_mn(q.src[qe]) over the qint edges in order (FillK), q_tin[Q] = number of slots."""
    deg = np.diff(mn.ptr.astype(np.int64))
    out = np.zeros(q.ne + 1, dtype=np.int32)
    out[1:] = np.cumsum(deg[q.src])
    return out


def triplets(o: Graph, inp: Graph):
    """(e, k) int64 index arrays of every (output edge, input edge) term, k ascending within e."""
    es, ks = [], []
    for e in range(o.ne):
        r = np.arange(inp.ptr[o.tgt[e]], inp.ptr[o.tgt[e] + 1])
        r = r[inp.src[r] != o.src[e]]
        es.append(np.full(len(r), e)); ks.append(r)
    return torch.from_numpy(np.concatenate(es).astype(np.int64)), torch.from_numpy(np.concatenate(ks).astype(np.int64))


def quadruplets(mn: Graph, q: Graph, q_tin):
    """(e, qe, k, t) int64 index arrays of every quadruplet term d -> b -> a <- c, t the x_t slot."""
    out = [[], [], [], []]
    for e in range(mn.ne):
        a, c = mn.tgt[e], mn.src[e]
        for qe in q.row(a):
            b = q.src[qe]
            if b == c:
                continue
            k = np.arange(mn.ptr[b], mn.ptr[b + 1])
            k = k[(mn.src[k] != a) & (mn.src[k] != c)]
            for lst, v in zip(out, (np.full(len(k), e), np.full(len(k), qe), k, q_tin[qe] + k - mn.ptr[b])):
                lst.append(v)
    return tuple(torch.from_numpy(np.concatenate(v).astype(np.int64)) if v else torch.zeros(0, dtype=torch.int64) for v in out)


# ------------------------------------------------------------------------------------------------------------------- references
def _accumulate(E, n_terms, width, chunk_terms):
    """S [E, width, ch] = sum over terms of chunk_terms(lo, hi) -> (e [m], contributions [m, width, ch]); out-of-place, so jvp can trace it."""
    S = None
    for lo in range(0, max(n_terms, 1), CHUNK):
        e, c = chunk_terms(lo, min(lo + CHUNK, n_terms))
        S = c.new_zeros(E, *c.shape[1:]).index_add(0, e, c) if S is None else S.index_add(0, e, c)
    return S


def trip_ref(Vo, Vi, x, R, tri, E):
    """Triplet aggregation O [E, 1024] in float64; R [E, 112]."""
    te, tk = tri

    def chunk(lo, hi):
        e, k = te[lo:hi], tk[lo:hi]
        Y = sph(clamp1((Vo[e] * Vi[k]).sum(-1)))
        return e, Y[:, :, None] * x[k][:, None, :]

    S = _accumulate(E, len(te), NS, chunk)  # [E, 7, 64]
    return torch.einsum("eis,esc->eic", R.reshape(E, 16, NS), S).reshape(E, 16 * TI)


def trip_bound(Vo, Vi, x, R, tri, E, Vot=None, Vit=None, xt=None, Rt=None):
    """A [E, 1024]: trip_ref over absolute values; with the tangents, the bound of the tangent's terms."""
    te, tk = tri

    def terms(lo, hi, prim):
        e, k = te[lo:hi], tk[lo:hi]
        c = (Vo[e] * Vi[k]).sum(-1)
        Y = sph(clamp1(c)).abs()
        if prim:
            return e, Y[:, :, None] * x[k].abs()[:, None, :]
        ct = (absdot(Vot[e], Vi[k]) + absdot(Vo[e], Vit[k])) * ((c >= -1) & (c <= 1))
        dY = dsph(clamp1(c)).abs() * ct[:, None]
        return e, dY[:, :, None] * x[k].abs()[:, None, :] + Y[:, :, None] * xt[k].abs()[:, None, :]

    S = _accumulate(E, len(te), NS, lambda lo, hi: terms(lo, hi, True))
    Ra = R.abs().reshape(E, 16, NS)
    if Vot is None:
        return torch.einsum("eis,esc->eic", Ra, S).reshape(E, -1)
    St = _accumulate(E, len(te), NS, lambda lo, hi: terms(lo, hi, False))
    return (torch.einsum("eis,esc->eic", Rt.abs().reshape(E, 16, NS), S) + torch.einsum("eis,esc->eic", Ra, St)).reshape(E, -1)


def _quad_geometry(vca, vba, vdb):
    """(cos(c, a, b) clamped, cos phi) per quadruplet, float64, differentiable; on the yy clamp yy is a constant (its tangent an explicit 0),
    and the norm is never differentiated at 0."""
    n1 = torch.linalg.cross(vca, vba, dim=-1)
    n2 = torch.linalg.cross(vdb, vba, dim=-1)
    xx = (n1 * n2).sum(-1)
    n3 = torch.linalg.cross(n1, n2, dim=-1)
    sq = (n3 * n3).sum(-1)
    on = sq > YY_MIN * YY_MIN
    yy = torch.where(on, torch.sqrt(torch.where(on, sq, torch.ones_like(sq))), torch.full_like(sq, YY_MIN))
    return clamp1((vca * vba).sum(-1)), xx / torch.sqrt(xx * xx + yy * yy)


def quad_ref(Vm, Vq, xt, R, quads, E):
    """Quadruplet aggregation O [E, 1024] in float64; R [E, 1568]."""
    qe_e, qe_q, qe_k, qe_t = quads

    def chunk(lo, hi):
        e, qq, k, t = qe_e[lo:hi], qe_q[lo:hi], qe_k[lo:hi], qe_t[lo:hi]
        c1, cp = _quad_geometry(Vm[e], Vq[qq], Vm[k])
        Y = (sph(c1)[:, :, None] * sph(cp)[:, None, :]).reshape(-1, NS * NS)
        return e, Y[:, :, None] * xt[t][:, None, :]

    S = _accumulate(E, len(qe_e), NS * NS, chunk)  # [E, 49, 32]
    return torch.einsum("eis,esc->eic", R.reshape(E, 32, NS * NS), S).reshape(E, 32 * QI)


def quad_bound(Vm, Vq, xt, R, quads, E, Vmt=None, Vqt=None, xtt=None, Rt=None):
    """A [E, 1024] of quad_ref; with the tangents, the bound of the tangent's terms.  The factor cos phi' enters as the absolute terms of
    (xx' - cos phi r r' / r) / r, the form the kernels evaluate, so that its rounding is covered where cos phi' itself vanishes (planar)."""
    qe_e, qe_q, qe_k, qe_t = quads

    def terms(lo, hi, prim):
        e, qq, k, t = qe_e[lo:hi], qe_q[lo:hi], qe_k[lo:hi], qe_t[lo:hi]
        vca, vba, vdb = Vm[e], Vq[qq], Vm[k]
        c1, cp = _quad_geometry(vca, vba, vdb)
        Yp, Yt = sph(c1).abs(), sph(cp).abs()
        x = xt[t].abs()
        if prim:
            return e, ((Yp[:, :, None] * Yt[:, None, :]).reshape(-1, NS * NS))[:, :, None] * x[:, None, :]
        c1raw = (vca * vba).sum(-1)
        c1t = (absdot(Vmt[e], vba) + absdot(vca, Vqt[qq])) * ((c1raw >= -1) & (c1raw <= 1))
        n1, n2 = torch.linalg.cross(vca, vba, dim=-1), torch.linalg.cross(vdb, vba, dim=-1)
        n1t = torch.linalg.cross(Vmt[e], vba, dim=-1).abs() + torch.linalg.cross(vca, Vqt[qq], dim=-1).abs()  # >= |n1'| elementwise
        n2t = torch.linalg.cross(Vmt[k], vba, dim=-1).abs() + torch.linalg.cross(vdb, Vqt[qq], dim=-1).abs()
        xx = (n1 * n2).sum(-1)
        n3 = torch.linalg.cross(n1, n2, dim=-1)
        nrm = torch.sqrt((n3 * n3).sum(-1))
        r = torch.sqrt(xx * xx + torch.clamp(nrm, min=YY_MIN) ** 2)
        xxt = absdot(n1t, n2) + absdot(n1, n2t)
        rrt = torch.where(nrm > YY_MIN, absdot(n1, n1t) * (n2 * n2).sum(-1) + (n1 * n1).sum(-1) * absdot(n2, n2t), xx.abs() * xxt)
        cpt = (xxt + cp.abs() * rrt / r) / r
        dYp, dYt = dsph(c1).abs() * c1t[:, None], dsph(cp).abs() * cpt[:, None]
        Yd = (dYp[:, :, None] * Yt[:, None, :] + Yp[:, :, None] * dYt[:, None, :]).reshape(-1, NS * NS)
        Y = (Yp[:, :, None] * Yt[:, None, :]).reshape(-1, NS * NS)
        return e, Yd[:, :, None] * x[:, None, :] + Y[:, :, None] * xtt[t].abs()[:, None, :]

    S = _accumulate(E, len(qe_e), NS * NS, lambda lo, hi: terms(lo, hi, True))
    Ra = R.abs().reshape(E, 32, NS * NS)
    if Vmt is None:
        return torch.einsum("eis,esc->eic", Ra, S).reshape(E, -1)
    St = _accumulate(E, len(qe_e), NS * NS, lambda lo, hi: terms(lo, hi, False))
    return (torch.einsum("eis,esc->eic", Rt.abs().reshape(E, 32, NS * NS), S) + torch.einsum("eis,esc->eic", Ra, St)).reshape(E, -1)


def jvp(fn, primals, tangents):
    """The tangent of fn at primals (float64 tensors) in the direction tangents."""
    return torch.func.jvp(fn, tuple(primals), tuple(tangents))[1]


# ------------------------------------------------------------------------------------------------------------------- cases
LENS = (0, 1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 100)  # the empty row, every tail of a 4-wide loop, both sides of each 32-chunk boundary
AXES = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32)


def _row_sources(rng, n, a, L, pinned=()):
    """L distinct sources != a, with pinned = ((position, source), ...) in place."""
    pinned = [(p if p >= 0 else L + p, s) for p, s in pinned]
    taken = {s for _, s in pinned} | {a}
    pool = rng.permutation([j for j in range(n) if j not in taken])
    src = list(pool[:L])
    for p, s in pinned:
        src[p] = s
    assert len(set(src)) == L and a not in src
    return src


def trip_case(pairing: str, overshoot: bool, repeats: int = 1, seed: int = 0):
    """(o, in) graphs for the triplet kernel.

    pairing "mn_mn": one graph, every edge an output; targets with in-rows of every length of LENS (`repeats` times), so each edge excludes
    itself at every position, first, 31, 32 and last included; the row of length 1 is wholly excluded.  In some rows the first inputs carry
    the axis vectors +-x, +-y (cos exactly +-1 in float32 and float64) and, with `overshoot`, two carry a vector whose float32 dot with
    itself rounds past 1.
    pairing "mn_ae": input rows (a2ee2a) of every length of LENS; the output edges into a target have the sources of its input row at
    positions 0, 31, 32 and last (those inputs are excluded), plus one source outside the row; targets whose input row is empty or a single
    excluded edge give rows of exact zeros."""
    rng = np.random.default_rng(seed)
    lens = [L for _ in range(repeats) for L in LENS]
    n = len(lens) + 110
    ov = overshoot_vector()
    rows, V = {}, {}
    for a, L in enumerate(lens):
        rows[a] = _row_sources(rng, n, a, L)
        V[a] = unit(rng, L)
        if L >= 6 and a % 3 == 0:
            V[a][:4] = [AXES[0], -AXES[0], AXES[1], AXES[0]]  # cos = +-1 exactly between inputs 0, 1, 3 and 0 / 2 orthogonal
            if overshoot:
                V[a][4] = V[a][5] = ov
    inp = Graph(n, rows, V)
    if pairing == "mn_mn":
        return inp, inp
    orows, oV = {}, {}
    for a, L in enumerate(lens):
        srcs = [rows[a][p] for p in sorted({0, 31, 32, L - 1}) if 0 <= p < L]
        srcs.append(int(rng.choice([j for j in range(n) if j != a and j not in rows[a]])))
        orows[a] = srcs
        oV[a] = unit(rng, len(srcs))
        if L >= 6 and a % 3 == 0:
            oV[a][0] = AXES[0]  # against inputs 0..3: cos = 1, -1, 0, 1
            if overshoot:
                oV[a][-1] = ov
    return Graph(n, orows, oV), inp


QLENS = (0, 1, 31, 32, 33, 64, 65, 5)  # mn-row lengths of the eight qint sources of a full hub


def quad_case(collinear: bool, seed: int = 1):
    """(mn, q, q_tin) for the quadruplet kernel; every mn edge is an output edge.

    Hubs (targets with qint rows): a row of 0 qint edges; one of 1; two of 8 whose sources b have mn-rows of the lengths QLENS, one b also an
    output source c (b == c, skipped), the hub itself (d == a) and output sources (d == c) at positions 0, 31, 32 and last of the long rows;
    a hub whose qint vectors are axes and some of whose d -> b vectors are +-V_ba exactly (n2 = 0, cos phi = 0); a hub where every vector
    has z = 0 exactly (planar: n1 x n2 = 0 in float32 too, the yy clamp with cos phi = +-1); with `collinear`, a hub where V_ca = +-V_ba
    (n1 = 0).  Every other atom has an empty qint row."""
    rng = np.random.default_rng(seed)
    n = 300
    rows, V = {}, {}
    qrows, qV = {}, {}
    nxt = iter(range(10, n))  # b atoms, never reused

    def full_hub(a, planar):
        bs = [next(nxt) for _ in QLENS]
        cs = [next(nxt) for _ in range(3)]
        # per long row: (position of a, positions of c0, c1, c2); position -1 = last
        pins = {31: ((0, -1),), 32: ((-1, 0),), 33: ((32, 0, 31),), 64: ((31, 0, 32, -1),), 65: ((0, 31, 32, -1),)}
        for b, L in zip(bs, QLENS):
            pin = []
            if L in pins:
                pa, *pc = pins[L][0]
                pin = [(pa, a)] + [(p, c) for p, c in zip(pc, cs)]
            rows[b] = _row_sources(rng, n, b, L, pin)
            V[b] = unit(rng, L, planar)
        rows[a] = cs + [bs[3], next(nxt)]  # bs[3] (mn-row of 32) is also an output source: b == c
        V[a] = unit(rng, len(rows[a]), planar)
        qrows[a] = bs
        qV[a] = unit(rng, len(bs), planar)

    rows[0] = [next(nxt)]; V[0] = unit(rng, 1)  # qint row of 0 edges
    b = next(nxt)
    rows[b] = _row_sources(rng, n, b, 33); V[b] = unit(rng, 33)
    rows[1] = [next(nxt), next(nxt)]; V[1] = unit(rng, 2)
    qrows[1] = [b]; qV[1] = unit(rng, 1)  # qint row of 1 edge
    full_hub(2, False)
    full_hub(3, False)
    full_hub(4, True)
    # parallel d -> b and b -> a
    bs = [next(nxt), next(nxt)]
    qrows[5], qV[5] = bs, AXES[[0, 1]].copy()
    for j, bb in enumerate(bs):
        rows[bb] = _row_sources(rng, n, bb, 6)
        V[bb] = unit(rng, 6)
        V[bb][1], V[bb][4] = AXES[j], -AXES[j]
    rows[5] = [next(nxt), next(nxt), next(nxt)]; V[5] = unit(rng, 3)
    if collinear:  # c - a - b on one line
        bs = [next(nxt), next(nxt)]
        qrows[6], qV[6] = bs, np.stack([AXES[2], -AXES[2]])
        for bb in bs:
            rows[bb] = _row_sources(rng, n, bb, 7); V[bb] = unit(rng, 7)
        rows[6] = [next(nxt), next(nxt)]; V[6] = np.stack([AXES[2], unit(rng, 1)[0]])
    mn, q = Graph(n, rows, V), Graph(n, qrows, qV)
    return mn, q, q_slot_bases(mn, q)


def long_row_probes(o: Graph, inp: Graph, min_len=33):
    """(e, k) pairs: for every input row of at least `min_len` inputs, one output edge into its target and the inputs at positions 31 and 32
    (either side of the first chunk boundary) and 63 / 64 where they exist, none of them excluded."""
    out, seen = [], set()
    for e in range(o.ne):
        a = int(o.tgt[e])
        r = list(inp.row(a))
        if len(r) < min_len or a in seen:
            continue
        seen.add(a)
        out += [(e, r[p]) for p in (31, 32, 63, 64) if p < len(r) and inp.src[r[p]] != o.src[e]]
    return out


# ------------------------------------------------------------------------------------------------------------------- running a case
SENTINEL_BITS = 0x7FBADBAD  # a NaN payload no kernel produces: rows at or past a device count must keep it bitwise
TRIP_CASES = (  # (pairing, repeats of LENS, ldr, first column of R): R read as B_main is (columns 80 / 192 of 1920) and packed (112)
    ("mn_mn", 50, 1920, 80),  # 20 150 output edges: the capped grid (8 CTAs x 8 warps per SM) strides over the edges more than twice
    ("mn_ae", 1, 1920, 192),
    ("mn_mn", 1, 112, 0),
    ("mn_ae", 1, 112, 0),
)
QUAD_LDR, QUAD_COL = 1920, 304


def _dev(g: Graph, device):
    return {k: torch.from_numpy(getattr(g, k)).to(device) for k in ("ptr", "src", "tgt", "V")}


class Problem:
    """One aggregation problem: graphs and float32 inputs on `device`, their float64 copies, the term lists of the reference."""

    def __init__(self, quad: bool, device, seed: int, pairing="mn_mn", repeats=1, ldr=LDR_TRIP, col=0, overshoot=False, collinear=False):
        self.quad, self.device, self.ldr, self.col = quad, device, ldr, col
        if quad:
            self.go, self.gi, q_tin = quad_case(collinear)
            self.q_tin = torch.from_numpy(q_tin).to(device)
            self.terms = quadruplets(self.go, self.gi, q_tin)
            rows, width, self.nr = int(q_tin[-1]), QI, LDR_QUAD
        else:
            self.go, self.gi = trip_case(pairing, overshoot, repeats)
            self.q_tin = None
            self.terms = triplets(self.go, self.gi)
            rows, width, self.nr = self.gi.ne, TI, LDR_TRIP
        assert col + self.nr <= ldr
        self.E = self.go.ne
        g = torch.Generator().manual_seed(seed)
        f32 = dict(x=torch.randn(rows, width, generator=g), R=torch.randn(self.E, ldr, generator=g),
                   Vot=torch.randn(self.go.ne, 3, generator=g), Vit=torch.randn(self.gi.ne, 3, generator=g),
                   xt=torch.randn(rows, width, generator=g), Rt=torch.randn(self.E, ldr, generator=g))
        self.t = {k: v.to(device) for k, v in f32.items()}
        self.o, self.i = _dev(self.go, device), _dev(self.gi, device)
        d = {k: v.double() for k, v in f32.items()}
        self.primals = (torch.from_numpy(self.go.V).double(), torch.from_numpy(self.gi.V).double(), d["x"], d["R"][:, col:col + self.nr])
        self.tangents = (d["Vot"], d["Vit"], d["xt"], d["Rt"][:, col:col + self.nr])

    def run(self, lib, stream, form: int, tangent: bool, E_bound=None, E_dev=None, out=None):
        """The library's aggregation into `out` (default: a fresh [E, 1024] buffer of SENTINEL_BITS); returns (status, out)."""
        import ctypes

        from nabladft_b200._lib import GemNetOCAggArgs

        E_bound = self.E if E_bound is None else E_bound
        if out is None:
            out = torch.full((max(E_bound, 1), 1024), SENTINEL_BITS, dtype=torch.int32, device=self.device).view(torch.float32)
        p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        col = lambda t: t.data_ptr() + 4 * self.col  # noqa: E731
        a = GemNetOCAggArgs(quad=int(self.quad), form=form, tangent=int(tangent), ldr=self.ldr, E_bound=E_bound, E_dev=p(E_dev),
                            o_ptr=p(self.o["ptr"]), o_src=p(self.o["src"]), o_tgt=p(self.o["tgt"]), o_V=p(self.o["V"]),
                            in_ptr=p(self.i["ptr"]), in_src=p(self.i["src"]), in_V=p(self.i["V"]), q_tin=p(self.q_tin),
                            x=p(self.t["x"]), R=col(self.t["R"]))
        if tangent:
            a.Vot, a.Vit, a.xt, a.Rt, a.Ot = p(self.t["Vot"]), p(self.t["Vit"]), p(self.t["xt"]), col(self.t["Rt"]), p(out)
        else:
            a.O = p(out)
        return lib.nb200_gemnet_oc_test_aggregate(ctypes.byref(a), stream), out

    def reference(self, tangent: bool, terms=None):
        """(O64, A) [E, 1024]: the float64 output (or its tangent) and the magnitude bound of its terms."""
        terms = self.terms if terms is None else terms
        ref, bound = (quad_ref, quad_bound) if self.quad else (trip_ref, trip_bound)
        fn = lambda *a: ref(*a, terms, self.E)  # noqa: E731
        if not tangent:
            return fn(*self.primals), bound(*self.primals, terms, self.E)
        return jvp(fn, self.primals, self.tangents), bound(*self.primals, terms, self.E, *self.tangents)

    def label(self):
        return f"{'quad' if self.quad else 'trip'} E={self.E} ldr={self.ldr} col={self.col}"


def compare(got, O64, A, c, what):
    """|got - O64| <= c A elementwise (A = 0: exactly 0); returns the largest error as a fraction of A and prints it."""
    got = got.double().cpu()
    err = (got - O64).abs()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    zero = A == 0
    assert bool((got[zero] == 0).all()), f"{what}: {int((got[zero] != 0).sum())} elements of empty / fully excluded sums are not exactly 0"
    worst = float((err[~zero] / A[~zero]).max()) if bool((~zero).any()) else 0.0
    n_zero_rows = int(zero.all(1).sum())
    print(f"{what}: max |err| / A = {worst:.2e} (bound {c:.0e}); {n_zero_rows} rows exactly 0")
    bad = err > c * A
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements beyond {c:.0e} A (worst {worst:.2e})"
    return worst
