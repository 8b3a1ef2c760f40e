"""Float64 references of the PaiNN tangent and Hessian-vector-product kernels (csrc/painn_tangent.cu, the d2W and weight-gradient kernels of
csrc/filter.cu) and the synthetic inputs they run on.  Helper module of tests/test_painn_tangent_ref.py and tests/test_gpu_painn_tangent.py,
not a test file.

Each reference is the float64 PRIMAL operation, taken from its definition in painn_msg.cu, painn_node.cu, painn_fused.cu and filter.cu:
  geometry        pos -> (u, d) of every edge, r = pos[src] - pos[tgt]
  message         dq_i = sum_e Wa(e) a_j ;  mu'_i[x] = mu_i[x] + sum_e Wb(e) b_j u_e[x] + Wc(e) c_j mu_j[x]   ((a, b, c) = xh_j + bias)
                  with the filter row W(e) = W0 + W1 delta_e + W2 delta_e^2 / 2 + Z_e a function of delta_e = d_e - d_e0 (W0, W1, W2 = W,
                  dW/dd, d2W/dd2 of the row the kernel reads) and Z_e = 0 an additive per-edge input whose gradient is dE/dW_e
  message bwd     the vjp of the message with cotangents (gq, gmu)
  update          nrm = sqrt(sum_x V_x^2 + eps);  q'' = q + y0 + y2 <V, Wv>,  mu''[x] = mu[x] + y1 Wv[x]; its vjp; the norm's vjp gn V / nrm
  activations     silu, its vjp g silu'(p); the readout energy sum_k silu(p_k) R2_k
  forces          F_j = -sum_{e in row j} (G(e) - G(rev e)),  G(e) = (gu - (gu.u') u') / d + gd u',  u' = -u_e, (gu, gd) = egrad[e]
  filter          W(d) = s1(d) sum_k phi_k(d) w[k] + s2(d) b over all K centres, phi_k = exp(coeff (d xscale - o_k)^2)
  filter wgrad    g_w[k] = sum_e s1 phi_k(d_e) gW[e],  g_b = sum_e s2 gW[e]
Tangents are torch.func.jvp of those functions, and tangents of backward steps the jvp of their torch.func.vjp: no product rule is typed
here, so a term the kernel drops cannot be dropped here as well.

Every output element also gets a magnitude bound A: the same expression with every factor replaced by its absolute value.  For the
multilinear steps this is the jvp of the same function at |inputs| along |tangents| with every subtraction made an addition (`ab = True`);
for a transcendental factor f(t) of a rounded argument t it is |f| + |t f'(t)|, its sensitivity to a relative change of t.

The graphs are synthetic: rows by target with ascending sources, `rev` found by binary search as graph.cu does, geom from float32
positions in float64 and rounded once, so geom[rev e] = (-u_e, d_e) bitwise."""
import math

import numpy as np
import torch
from torch.func import jvp, vjp

F = 128
EPS = 1e-8  # PaiNN's norm epsilon (painn_fused.cu: nrm = sqrt(sum_x V_x^2 + eps); epsilon of painn_oc.py and spk.PaiNN)
SENTINEL_BITS = 0x7FBADBAD  # a NaN payload no kernel writes: rows at or past n_atoms (or E) must keep it bitwise
STAR_DEGREES = (1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 310)
D64 = torch.float64
# GPU tolerances, |kernel - reference| <= C * A elementwise.  fp32 has u = 2^-24 = 6e-8; a sum of n terms in fp32 is off by at most about
# n u sum|terms| and, with rounding errors of random sign, typically sqrt(n) u sum|terms|.
C_POINT = 2e-6  # per-element ops (activations, update steps, geometry): at most ~10 roundings and one expf / division each: 10 u < 1e-6
C_SUM = 1e-5    # sums over a CSR row (message kernels, forces: rows up to 310 edges, sqrt(310) u = 1e-6, x10 for products of a few roundings
                # per term), over the 16-centre band (d2W: 48 fused terms, plus expf / cosf / sinf at 1-2 ulp) and over a distance bin
                # (weight gradient: up to 1700 edges as 3 parts of 4 groups, about 140 sequential terms per thread, then atomics)
BF16_HALF_ULP = 2.0 ** -8  # bf16 keeps 8 significant bits: a stored output rounds by at most 2^-8 of its magnitude


def d64(t):
    return t.detach().to("cpu", D64)


# ------------------------------------------------------------------------------------------------------------------- graph
class Graph:
    """CSR by target over n atoms from undirected pairs; float32 positions, geom [E, 4] float32."""

    def __init__(self, pos, pairs):
        n = pos.shape[0]
        rows = [[] for _ in range(n)]
        for a, b in pairs:
            rows[a].append(b)
            rows[b].append(a)
        for r in rows:
            r.sort()
            assert len(set(r)) == len(r)
        self.n = n
        self.deg = np.array([len(r) for r in rows], dtype=np.int64)
        self.ptr = np.zeros(n + 1, dtype=np.int32)
        self.ptr[1:] = np.cumsum(self.deg)
        self.src = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows] + [np.zeros(0, np.int32)])
        self.tgt = np.repeat(np.arange(n, dtype=np.int32), self.deg)
        E = self.E
        self.rev = np.empty(E, dtype=np.int32)
        for e in range(E):  # the opposite edge (tgt = src[e], src = tgt[e]) by binary search in row src[e], as graph.cu does
            j = self.src[e]
            lo = self.ptr[j]
            self.rev[e] = lo + np.searchsorted(self.src[lo:self.ptr[j + 1]], self.tgt[e])
        assert np.all(self.rev[self.rev] == np.arange(E)) and np.all(self.src[self.rev] == self.tgt)
        self.pos = np.asarray(pos, dtype=np.float32)
        r = self.pos.astype(np.float64)[self.src] - self.pos.astype(np.float64)[self.tgt]
        d = np.linalg.norm(r, axis=1)
        self.geom = np.concatenate([r / d[:, None], d[:, None]], 1).astype(np.float32)
        assert np.array_equal(self.geom[self.rev, :3], -self.geom[:, :3]) and np.array_equal(self.geom[self.rev, 3], self.geom[:, 3])

    @property
    def E(self):
        return int(self.ptr[-1])

    def canon(self):
        """Row each edge reads with `rev`: min(e, rev[e])."""
        return np.minimum(np.arange(self.E), self.rev)

    def tensors(self):
        return dict(row_ptr=torch.from_numpy(self.ptr), col=torch.from_numpy(self.src), rev=torch.from_numpy(self.rev), geom=torch.from_numpy(self.geom))


def tangent_graph(seed=0):
    """Stars whose hubs have degrees 1..5, 31..33, 63..65 and 310 (leaves joined in a chain: degrees 1..3) plus one isolated atom (degree 0):
    626 atoms, not a multiple of the 8 atoms per 256-thread CTA nor of 256."""
    rng = np.random.default_rng(seed)
    pos, pairs = [np.zeros((1, 3))], []
    n = 1
    for s, D in enumerate(STAR_DEGREES):
        hub = n
        v = rng.standard_normal((D, 3))
        leaves = 10.0 * s + v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(0.8, 4.5, (D, 1))
        pos += [np.full((1, 3), 10.0 * s), leaves]
        pairs += [(hub, hub + 1 + k) for k in range(D)] + [(hub + 1 + k, hub + 2 + k) for k in range(D - 1) if D >= 3]
        n += D + 1
    g = Graph(np.concatenate(pos), pairs)
    deg = set(g.deg.tolist())
    assert {0, 1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65}.issubset(deg) and max(deg) > 300 and g.n % 8 != 0
    return g


# ------------------------------------------------------------------------------------------------------------------- inputs
def _mirror_tgeom(g, t):
    """t_geom [E, 4] with the opposite edge's tangent: t_u[rev e] = -t_u[e], dd[rev e] = dd[e] (canonical edge's values)."""
    c = g.canon()
    out = t[c].clone()
    flip = torch.from_numpy(np.arange(g.E) != c)
    out[flip, :3] = -out[flip, :3]
    return out


def node_inputs(g, seed=1):
    """float32 CPU tensors of every per-atom and per-edge input of the tangent kernels.  A tenth of the atoms have V of order sqrt(eps) (an
    atom whose mu is still near zero: the norm at its floor) with O(1) tangents."""
    gen = torch.Generator().manual_seed(seed)
    N, E = g.n, g.E

    def r(*shape, s=1.0):
        return torch.randn(*shape, generator=gen) * s

    VW = r(N, 3, 2, F, s=0.7)
    floor = torch.rand(N, generator=gen) < 0.1
    VW[floor, :, 0] *= 1e-4
    VW = VW.reshape(N, 6 * F).contiguous()
    V = VW.view(N, 3, 2, F)[:, :, 0].double()
    t_VW = r(N, 6 * F, s=0.5)
    nrm = torch.sqrt((V * V).sum(1) + EPS).float()
    d = dict(
        xh=r(N, 3 * F, s=0.5), t_xh=r(N, 3 * F, s=0.5), xh_bias=r(3 * F, s=0.1), mu=r(N, 3 * F, s=0.5), t_mu=r(N, 3 * F, s=0.5),
        g_q=r(N, F), t_g_q=r(N, F, s=0.5), g_mu=r(N, 3 * F), t_g_mu=r(N, 3 * F, s=0.5),
        W=r(E, 3 * F, s=0.2), dW=r(E, 3 * F, s=0.2), d2W=r(E, 3 * F, s=0.2),
        t_geom=_mirror_tgeom(g, torch.cat([r(E, 3, s=0.3), r(E, 1, s=0.5)], 1)),
        VW=VW, t_VW=t_VW, nrm=nrm, y=r(N, 3 * F), t_y=r(N, 3 * F, s=0.5), gn=r(N, F), t_gn=r(N, F, s=0.5),
        pre=r(N, F, s=2.0), t_pre=r(N, F), x=r(N, F), g_pre=r(N, F), t_g=r(N, F), R2=r(F // 2), pre_ro=r(N, F // 2, s=2.0), t_pre_ro=r(N, F // 2),
        egrad=r(E, 4), t_egrad=r(E, 4, s=0.5), v=r(N, 3, s=0.3),
        prefill_q=r(N, F), prefill_mu=r(N, 3 * F), prefill_gVW=r(N, 6 * F), prefill_egrad=r(E, 4),
    )
    d["t_nrm"] = upd_norm_tan(d)[0].float()  # the kernel's t_nrm input: the tangent of nrm along t_VW
    return d


def filter_rows(g, d, use_rev, dtype=torch.float32):
    """Stored filter rows (W, dW, d2W) in the kernel's layout and storage type, and the float64 rows each edge reads.  With `rev` only row
    min(e, rev[e]) is read, so every other row is NaN; without it every edge reads its own row, equal for both edges of a pair."""
    c = torch.from_numpy(g.canon()).long()
    stored, read = [], []
    for name in ("W", "dW", "d2W"):
        rows = d[name][c].to(dtype)
        if use_rev:
            rows = rows.clone()
            rows[torch.arange(g.E) != c] = float("nan")
        stored.append(rows.contiguous())
        read.append(rows.double()[c])
    return stored, read


# ------------------------------------------------------------------------------------------------------------------- helpers
def _abs_args(args):
    return tuple(a.abs() if torch.is_tensor(a) else a for a in args)


def ref_and_bound(f, primals, tangents):
    """(jvp of f(ab = False), jvp of f(ab = True) at |primals| along |tangents|): reference tangents and their magnitude bounds."""
    _, t = jvp(lambda *p: f(*p, ab=False), primals, tangents)
    _, A = jvp(lambda *p: f(*p, ab=True), _abs_args(primals), _abs_args(tangents))
    return t, A


def _sub(ab):
    return 1.0 if ab else -1.0


def silu(x):
    return x * torch.sigmoid(x)


def dsilu_bound(x):
    """|silu'| = |s (1 + x (1 - s))| term by term, 1 - s counted as 1 + s: in fp32 1 - s is off by u, not by u (1 - s)."""
    s = torch.sigmoid(x)
    return s * (1 + x.abs() * (1 + s))


def d2silu_bound(x):
    """|silu''| = |s (1 - s) (2 + x (1 - 2 s))| term by term (every difference a sum): at large x the kernels' 1 - s cancels, and the
    value is accurate to u s (1 + s) (2 + |x| (1 + 2 s)), not to u |silu''|."""
    s = torch.sigmoid(x)
    return s * (1 + s) * (2 + x.abs() * (1 + 2 * s))


# ------------------------------------------------------------------------------------------------------------------- geometry
def geom_of(g, pos):
    src, tgt = torch.from_numpy(g.src).long(), torch.from_numpy(g.tgt).long()
    r = pos[src] - pos[tgt]
    dd = torch.sqrt((r * r).sum(1))
    return torch.cat([r / dd[:, None], dd[:, None]], 1)


def geom_tan(g, d):
    """t_geom = jvp of pos -> (u, d) along v; A = (|dr| + |u| A_dd) / d and A_dd = sum |u| |dr|."""
    pos, v = torch.from_numpy(g.pos).double(), d64(d["v"])
    _, t = jvp(lambda p: geom_of(g, p), (pos,), (v,))
    src, tgt = torch.from_numpy(g.src).long(), torch.from_numpy(g.tgt).long()
    dr = v[src].abs() + v[tgt].abs()
    u = torch.from_numpy(g.geom).double()
    Add = (u[:, :3].abs() * dr).sum(1)
    A = torch.cat([(dr + u[:, :3].abs() * Add[:, None]) / u[:, 3:], Add[:, None]], 1)
    return t, A


# ------------------------------------------------------------------------------------------------------------------- activations
def mul_dact(d):
    pre, x = d64(d["pre"]), d64(d["x"])
    _, t = jvp(silu, (pre,), (x,))
    return t, dsilu_bound(pre) * x.abs()


def act_bwd(g_, p):
    """k_silu_bwd: the vjp of silu at p with cotangent g."""
    return vjp(silu, p)[1](g_)[0]


def act_bwd_tan(d, zero=()):
    t_g, g_pre, pre, t_pre = (d64(d[k]) for k in ("t_g", "g_pre", "pre", "t_pre"))
    _, t = jvp(act_bwd, (g_pre, pre), (t_g, torch.zeros_like(t_pre) if "t_pre" in zero else t_pre))
    return t, t_g.abs() * dsilu_bound(pre) + g_pre.abs() * d2silu_bound(pre) * t_pre.abs()


def readout_bwd_tan(d):
    """(t_g_pre, t_act): the jvp of the readout's pre-activation gradient R2 silu'(pre) and of silu."""
    pre, t_pre, R2 = d64(d["pre_ro"]), d64(d["t_pre_ro"]), d64(d["R2"])
    grad = lambda p: vjp(lambda q: (silu(q) * R2).sum(), p)[1](torch.ones((), dtype=D64))[0]  # noqa: E731
    _, t_g_pre = jvp(grad, (pre,), (t_pre,))
    _, t_act = jvp(silu, (pre,), (t_pre,))
    return (t_g_pre, R2.abs() * d2silu_bound(pre) * t_pre.abs()), (t_act, dsilu_bound(pre) * t_pre.abs())


# ------------------------------------------------------------------------------------------------------------------- update
def _V(VW):
    return VW.view(-1, 3, 2, F)[:, :, 0]


def _Wv(VW):
    return VW.view(-1, 3, 2, F)[:, :, 1]


def norm(VW):
    V = _V(VW)
    return torch.sqrt((V * V).sum(1) + EPS)


def upd_norm_tan(d):
    VW, t_VW = d64(d["VW"]), d64(d["t_VW"])
    _, t = jvp(norm, (VW,), (t_VW,))
    return t, (_V(VW).abs() * _V(t_VW).abs()).sum(1) / norm(VW)


def norm_bwd(gn, VW, nrm):
    """k_upd_norm_bwd: gV[x] = gn V[x] / nrm, the vjp of `norm` (nrm as the kernel receives it; test_norm_bwd_is_the_vjp_of_the_norm)."""
    out = torch.zeros_like(VW).view(-1, 3, 2, F)
    out[:, :, 0] = gn[:, None] * _V(VW) / nrm[:, None]
    return out.view(-1, 6 * F)


def upd_norm_bwd_tan(d, zero=()):
    """t_gVW = prefill + jvp of norm_bwd along (t_gn, t_VW, t_nrm); the Wv halves keep the prefill."""
    gn, VW, nrm, t_gn, t_VW, t_nrm, pre = (d64(d[k]) for k in ("gn", "VW", "nrm", "t_gn", "t_VW", "t_nrm", "prefill_gVW"))
    tang = [t_gn, t_VW, t_nrm]
    for k, name in enumerate(("t_gn", "t_VW", "t_nrm")):
        if name in zero:
            tang[k] = torch.zeros_like(tang[k])
    _, t = jvp(norm_bwd, (gn, VW, nrm), tuple(tang))
    A = torch.zeros_like(VW).view(-1, 3, 2, F)
    A[:, :, 0] = ((t_gn.abs() / nrm + gn.abs() * t_nrm.abs() / nrm ** 2)[:, None] * _V(VW).abs() + (gn.abs() / nrm)[:, None] * _V(t_VW).abs())
    return pre + t, pre.abs() + A.view(-1, 6 * F)


def combine(q, mu, VW, y, ab=False):
    """q'' = q + y0 + y2 <V, Wv>,  mu''[x] = mu[x] + y1 Wv[x]  (painn_node.cu, painn_fused.cu)."""
    y0, y1, y2 = y[:, :F], y[:, F:2 * F], y[:, 2 * F:]
    S = (_V(VW) * _Wv(VW)).sum(1)
    return q + y0 + y2 * S, (mu.view(-1, 3, F) + y1[:, None] * _Wv(VW)).reshape(-1, 3 * F)


def upd_combine_tan(d, zero=()):
    """(t_q, t_mu) = prefill + jvp of combine along (t_VW, t_y) (prefills = the tangents of q and mu)."""
    q, mu, VW, y = d64(d["prefill_q"]) * 0, d64(d["prefill_mu"]) * 0, d64(d["VW"]), d64(d["y"])
    tang = (d64(d["prefill_q"]), d64(d["prefill_mu"]), d64(d["t_VW"]) * (0 if "t_VW" in zero else 1), d64(d["t_y"]) * (0 if "t_y" in zero else 1))
    return ref_and_bound(combine, (q, mu, VW, y), tang)


def combine_bwd(VW, y, gq, gmu, ab=False):
    """k_upd_combine_bwd: the vjp of combine w.r.t. (VW, y) with cotangents (gq, gmu) -> (gy, gVW)."""
    z = torch.zeros_like(gq)
    gVW, gy = vjp(lambda VW_, y_: combine(z, torch.zeros_like(gmu), VW_, y_), VW, y)[1]((gq, gmu))
    return gy, gVW


def upd_combine_bwd_tan(d, zero=()):
    prim = tuple(d64(d[k]) for k in ("VW", "y", "g_q", "g_mu"))
    tang = tuple(d64(d[k]) * (0 if k in zero else 1) for k in ("t_VW", "t_y", "t_g_q", "t_g_mu"))
    return ref_and_bound(combine_bwd, prim, tang)


# ------------------------------------------------------------------------------------------------------------------- message
class Msg:
    """The message step on graph g with the float64 filter rows each edge reads (W0, W1, W2 = W, dW/dd, d2W/dd2)."""

    def __init__(self, g, d, rows):
        self.g, self.N, self.E = g, g.n, g.E
        self.src, self.tgt = torch.from_numpy(g.src).long(), torch.from_numpy(g.tgt).long()
        self.rev = torch.from_numpy(g.rev).long()
        self.W0, self.W1, self.W2 = rows
        self.bias = d64(d["xh_bias"])

    def fwd(self, xh, mu, u, delta, Z, ab=False):
        """(dq, mu'): dq_i = sum_e Wa a_j, mu'_i[x] = mu_i[x] + sum_e Wb b_j u_e[x] + Wc c_j mu_j[x] (painn_msg.cu k_painn_msg_fwd)."""
        W0, W1, W2, bias = (t.abs() for t in (self.W0, self.W1, self.W2, self.bias)) if ab else (self.W0, self.W1, self.W2, self.bias)
        We = W0 + W1 * delta[:, None] + 0.5 * W2 * (delta * delta)[:, None] + Z
        xb = xh + bias
        a, b, c = xb[:, :F], xb[:, F:2 * F], xb[:, 2 * F:]
        s, t = self.src, self.tgt
        dq = torch.zeros(self.N, F, dtype=D64).index_add(0, t, We[:, :F] * a[s])
        mu3 = mu.view(self.N, 3, F)
        msg = (We[:, F:2 * F] * b[s])[:, None, :] * u[:, :, None] + (We[:, 2 * F:] * c[s])[:, None, :] * mu3[s]
        return dq, mu3.index_add(0, t, msg).reshape(self.N, 3 * F)

    def bwd(self, xh, mu, u, delta, gq, gmu, ab=False):
        """The vjp of fwd with cotangents (gq, gmu): (g_xh, g_mu_in, g_u, g_delta, g_Z) per atom / per edge (k_painn_msg_bwd)."""
        Z = torch.zeros(self.E, 3 * F, dtype=D64)
        return vjp(lambda *p: self.fwd(*p, ab=ab), xh, mu, u, delta, Z)[1]((gq, gmu))

    def point(self, d, zero=()):
        """Primals and tangents (xh, mu, u, delta) of the kernels' inputs; `zero` names tangents to drop."""
        geom = torch.from_numpy(self.g.geom).double()
        tg = d64(d["t_geom"])
        prim = (d64(d["xh"]), d64(d["mu"]), geom[:, :3], torch.zeros(self.E, dtype=D64))
        tang = (d64(d["t_xh"]), d64(d["t_mu"]), tg[:, :3], tg[:, 3])
        names = ("t_xh", "t_mu", "t_geom.xyz", "t_geom.w")
        return prim, tuple(torch.zeros_like(t) if n in zero else t for t, n in zip(tang, names))

    def fwd_tan(self, d, zero=()):
        """(t_q, t_mu_out) of k_msg_fwd_tan: prefill + jvp of dq; jvp of mu' (which carries t_mu of the target itself)."""
        prim, tang = self.point(d, zero)
        Z = torch.zeros(self.E, 3 * F, dtype=D64)
        (t_dq, t_mu), (A_dq, A_mu) = ref_and_bound(self.fwd, prim + (Z,), tang + (Z,))
        pre = d64(d["prefill_q"])
        return (pre + t_dq, pre.abs() + A_dq), (t_mu, A_mu)

    def bwd_tan(self, d, zero=(), hvp=False):
        """Tangents of the message backward in the kernel's slots.  Slot e (row j = tgt e) carries the opposite edge e' = rev e:
        t_gW[e] = (dE/dW_e')^, gWd[e] = dE/dW_e' dd_e;  HVP: t_egrad[e] += (dE/du_e', dE/dd_e')^."""
        prim, tang = self.point(d, zero)
        gq, gmu = d64(d["g_q"]), d64(d["g_mu"])
        t_gq = d64(d["t_g_q"]) * (0 if "t_g_q" in zero else 1)
        t_gmu = d64(d["t_g_mu"]) * (0 if "t_g_mu" in zero else 1)
        W2 = self.W2
        if not hvp or "d2W" in zero:
            self.W2 = torch.zeros_like(W2)
        try:
            outs, A = ref_and_bound(self.bwd, prim + (gq, gmu), tang + (t_gq, t_gmu))
            prim_out = self.bwd(*prim, gq, gmu)
        finally:
            self.W2 = W2
        (t_gxh, t_gmu_in, t_gu, t_gd, t_gZ), (A_gxh, A_gmu_in, A_gu, A_gd, A_gZ) = outs, A
        r = self.rev
        res = dict(t_g_xh=(t_gxh, A_gxh), t_g_mu_in=(t_gmu_in, A_gmu_in))
        if hvp:
            pre = d64(d["prefill_egrad"])
            res["t_egrad"] = (pre + torch.cat([t_gu[r], t_gd[r][:, None]], 1), pre.abs() + torch.cat([A_gu[r], A_gd[r][:, None]], 1))
        else:
            dd = d64(d["t_geom"])[:, 3:]
            gZ = prim_out[4]
            _, Ab = self.bwd_abs_primal(prim, gq, gmu)
            res["t_gW"] = (t_gZ[r], A_gZ[r])
            res["gWd"] = (gZ[r] * dd, Ab[r] * dd.abs())
        return res

    def bwd_abs_primal(self, prim, gq, gmu):
        out = self.bwd(*_abs_args(prim), gq.abs(), gmu.abs(), ab=True)
        return None, out[4]


# ------------------------------------------------------------------------------------------------------------------- forces
def forces_of(g, pos, egrad):
    """k_edge_forces: F_j = -sum_{e in row j} (G(e) - G(rev e)) with the geometry of `pos`."""
    geom = geom_of(g, pos)
    up, d = -geom[:, :3], geom[:, 3:]
    gu, gd = egrad[:, :3], egrad[:, 3:]
    G = (gu - (gu * up).sum(1, keepdim=True) * up) / d + gd * up
    rev, tgt = torch.from_numpy(g.rev).long(), torch.from_numpy(g.tgt).long()
    return -torch.zeros(g.n, 3, dtype=D64).index_add(0, tgt, G - G[rev])


def _forces_poly(g, up, w, egrad, ab=False):
    """The same assembly as a polynomial in (u', w = 1/d, egrad), for the bound (ab = True: every subtraction an addition)."""
    sg = _sub(ab)
    gu, gd = egrad[:, :3], egrad[:, 3:]
    G = (gu + sg * (gu * up).sum(1, keepdim=True) * up) * w + gd * up
    rev, tgt = torch.from_numpy(g.rev).long(), torch.from_numpy(g.tgt).long()
    return torch.zeros(g.n, 3, dtype=D64).index_add(0, tgt, G + sg * G[rev])


def edge_forces_hvp(g, d):
    """hv = -F^ along (positions <- v, egrad <- t_egrad)."""
    pos, v, eg, t_eg = torch.from_numpy(g.pos).double(), d64(d["v"]), d64(d["egrad"]), d64(d["t_egrad"])
    _, tF = jvp(lambda p, e: forces_of(g, p, e), (pos, eg), (v, t_eg))
    geom = torch.from_numpy(g.geom).double()
    tg = geom_tan(g, d)[0]
    w = 1.0 / geom[:, 3:]
    _, A = jvp(lambda up, w_, e: _forces_poly(g, up, w_, e, ab=True), (geom[:, :3].abs(), w, eg.abs()),
               (tg[:, :3].abs(), tg[:, 3:].abs() * w * w, t_eg.abs()))
    return -tF, A


# ------------------------------------------------------------------------------------------------------------------- radial filter
class Radial:
    """The radial filter of one layer in float64: W(d) = s1(d) phi(d) @ w + s2(d) b over all K centres (filter.cu; painn_oc.py / spk)."""

    def __init__(self, mode, K=100, seed=0):
        self.mode = mode  # 0 = spk cosine cutoff on the whole filter, 1 = OC polynomial envelope (p = 5), bias unmasked
        # cutoffs whose xscale and distance bins are exact in float32 (spk: xscale 1; OC: d / 4 = d * 0.25), so that the Gaussian
        # argument the kernel forms carries the rounding of d only
        self.cutoff = 5.0 if mode == 0 else 4.0
        self.xscale = 1.0 if mode == 0 else 0.25
        self.K = K
        span = self.cutoff * self.xscale
        self.offsets = torch.linspace(0, span, K).float()
        self.coeff = float(np.float32(-0.5 / (span / (K - 1)) ** 2))
        gen = torch.Generator().manual_seed(seed + mode)
        self.w = (torch.randn(2, K, 3 * F, generator=gen) * 0.3).float()
        self.b = (torch.randn(2, 3 * F, generator=gen) * 0.3).float()

    def s(self, d):
        """(s1, s2) as functions of d (torch: differentiable)."""
        rc = self.cutoff
        if self.mode == 0:
            s1 = torch.where(d < rc, 0.5 * (torch.cos(d * (math.pi / rc)) + 1), torch.zeros_like(d))
            return s1, s1
        x = d / rc
        s1 = torch.where(x < 1, 1 - 21 * x ** 5 + 35 * x ** 6 - 15 * x ** 7, torch.zeros_like(d))
        return s1, torch.ones_like(d)

    def phi(self, d):
        t = d[:, None] * self.xscale - self.offsets.double()[None]
        return torch.exp(self.coeff * t * t)

    def W(self, d, layer):
        s1, s2 = self.s(d)
        return s1[:, None] * (self.phi(d) @ self.w[layer].double()) + s2[:, None] * self.b[layer].double()

    def derivs(self, d, layer):
        """W, dW/dd, d2W/dd2 by nested forward-mode derivatives of W(d) (each edge depends on its own d only)."""
        one = torch.ones_like(d)
        dW = lambda x: jvp(lambda y: self.W(y, layer), (x,), (one,))[1]  # noqa: E731
        W, d1 = jvp(lambda y: self.W(y, layer), (d,), (one,))
        _, d2 = jvp(dW, (d,), (one,))
        return W, d1, d2

    def scalar_bounds(self, d):
        """Bounds of (s1, s1', s1'', s2, s2', s2'') per edge: sums of absolute terms; cos / sin of theta = pi d / rc also get
        |theta f'(theta)| for the rounding of their argument."""
        rc = self.cutoff
        inside = (d < rc).double()
        if self.mode == 0:
            a = math.pi / rc
            th = d * a
            c, s = torch.cos(th).abs(), torch.sin(th).abs()
            b0 = 0.5 * (c + 1 + th * s)
            b1 = 0.5 * a * (s + th * c)
            b2 = 0.5 * a * a * (c + th * s)
            return tuple(t * inside for t in (b0, b1, b2, b0, b1, b2))
        x = d / rc
        b0 = 1 + 21 * x ** 5 + 35 * x ** 6 + 15 * x ** 7
        b1 = (105 * x ** 4 + 210 * x ** 5 + 105 * x ** 6) / rc
        b2 = (420 * x ** 3 + 1050 * x ** 4 + 630 * x ** 5) / rc ** 2
        z = torch.zeros_like(d)
        return b0 * inside, b1 * inside, b2 * inside, torch.ones_like(d), z, z

    def phi_bounds(self, d):
        """Bounds of (phi, phi', phi'') [E, K]: |f| + |t f'(t)| for exp of its argument c t^2, then the factors 2 c xscale t and
        2 c xscale^2 (1 + 2 c t^2) as sums of absolute terms."""
        t = d[:, None] * self.xscale - self.offsets.double()[None]
        c = abs(self.coeff)
        p = torch.exp(self.coeff * t * t) * (1 + c * t * t)
        return p, p * 2 * c * self.xscale * t.abs(), p * 2 * c * self.xscale ** 2 * (1 + 2 * c * t * t)

    def d2_bounds(self, d, layer):
        b0, b1, b2, c0, c1, c2 = self.scalar_bounds(d)
        p0, p1, p2 = self.phi_bounds(d)
        w, b = self.w[layer].double().abs(), self.b[layer].double().abs()
        P0, P1, P2 = p0 @ w, p1 @ w, p2 @ w
        return (b0[:, None] * P0 + c0[:, None] * b, b1[:, None] * P0 + b0[:, None] * P1 + c1[:, None] * b,
                b2[:, None] * P0 + 2 * b1[:, None] * P1 + b0[:, None] * P2 + c2[:, None] * b)

    def basis(self, d):
        """[E, K + 1]: s1 phi_k and s2, the factors of the weight gradient."""
        s1, s2 = self.s(d)
        return torch.cat([s1[:, None] * self.phi(d), s2[:, None]], 1)

    def wgrad(self, d, gW):
        """[K + 1, 3F]: g_w[k] = sum_e s1 phi_k gW[e] (rows 0..K-1) and g_b = sum_e s2 gW[e] (row K)."""
        return self.basis(d).T @ gW

    def wgrad_bound_basis(self, d):
        b0, b1, _, c0, c1, _ = self.scalar_bounds(d)
        p0, p1, _ = self.phi_bounds(d)
        return torch.cat([b0[:, None] * p0, c0[:, None]], 1), torch.cat([b1[:, None] * p0 + b0[:, None] * p1, c1[:, None]], 1)


def wgrad_distances(radial, seed=0):
    """Synthetic edge lengths for the weight gradient: bins with no edge, the band clamped at k0 = 0 and k0 = K - 16, d just below the
    cutoff, per-bin counts whose group range ceil(count / 4) is D - 1, D and D + 1 for the ring depths D = 8, 16, 32, some ragged, and one
    bin above 768 edges (split into parts)."""
    rng = np.random.default_rng(seed)
    rc, K = radial.cutoff, radial.K
    dx = rc / (K - 1)  # bin width in distance
    counts = {2: 28, 3: 32, 5: 36, 9: 60, 20: 64, 31: 68, 40: 124, 52: 128, 61: 132, 70: 125, 77: 61, 85: 1700, 92: 29, 97: 33, 98: 5}
    d = []
    for b, n in counts.items():
        d.append((b + rng.uniform(0.02, 0.98, n)) * dx)
    d.append(np.array([rc * (1 - 1e-4), rc * (1 - 1e-6), 0.01 * dx, 0.5 * dx]))
    d = np.concatenate(d).astype(np.float32)
    rng.shuffle(d)
    assert d.max() < rc
    return d


def filter_d2_distances(radial, seed=0):
    """Pair lengths for d2W: the band clamp at both ends, d just below the cutoff and spread over the range."""
    rng = np.random.default_rng(seed + 1)
    rc, K = radial.cutoff, radial.K
    dx = rc / (K - 1)
    d = np.concatenate([rng.uniform(0.02, 0.98, 40) * 8 * dx, rc - rng.uniform(0.0, 8 * dx, 40), rng.uniform(0.05, rc, 300),
                        [rc * (1 - 1e-4), rc * (1 - 1e-6), 1e-3]]).astype(np.float32)
    assert d.max() < rc
    return d


def wgrad_ref(radial, d, gW, t_gW=None, gWd=None, dd=None, sign=1.0):
    """(reference, bound) [K + 1, 3F] of the contribution: primal wgrad(d, gW), or TAN sign * jvp of wgrad along (gW <- t_gW, d <- dd) at
    gW = gWd / dd, the gradient the kernel receives folded with dd."""
    d = torch.as_tensor(d).double()
    B0, B1 = radial.wgrad_bound_basis(d)
    if t_gW is None:
        return radial.wgrad(d, d64(gW)), B0.T @ d64(gW).abs()
    gWd64, dd64 = d64(gWd), torch.as_tensor(dd).double()
    _, t = jvp(radial.wgrad, (d, gWd64 / dd64[:, None]), (dd64, d64(t_gW)))
    return sign * t, abs(sign) * (B0.T @ d64(t_gW).abs() + B1.T @ gWd64.abs())
