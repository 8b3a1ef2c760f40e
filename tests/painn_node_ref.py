"""Float64 references of the fused PaiNN node kernels (csrc/painn_fused.cu: k_prep_painn, k_node_fwd, k_node_bwd) and of the primal
per-atom kernels of csrc/painn_node.cu, and the synthetic weights and inputs they run on.  Helper module of tests/test_painn_node_ref.py
and tests/test_gpu_painn_node.py, not a test file.

The primal programs come from the model's definition (oracle/spk.py), in the canonical weight roles of include/nabla_b200.h:
  update       _PaiNNMixing:  [V | Wv]_x = mu_x U^T,  nrm = sqrt(sum_x V_x^2 + eps),  dot = sum_x V_x Wv_x,
               g1pre = [q | nrm] B1^T + d1,  y = (y0, y1, y2) = silu(g1pre) B2^T + d2,
               q' = q + y0 + y2 dot,  mu'_x = mu_x + y1 Wv_x
  message MLP  _PaiNNInteraction.interatomic_context_net without the c2 bias (the message kernel adds it):
               h1pre = q A1^T + c1,  xh = silu(h1pre) A2^T
  readout      Atomwise outnet[0] without e1 (k_readout adds it):  ro_pre = q R1^T
A forward program of the kernel is the update of layer l followed by the message MLP of layer l + 1 or by the readout, or the message MLP
alone; its saved intermediates are the primal's named intermediates above.  A backward program is torch.func.vjp of the composed forward
program with the kernel's inputs as cotangents (gq_a, cur, g_xh, and g_ro = R2 silu'(ro_pre + e1) for the readout); its hand-off arrays
are the cotangents of zero additive inputs at q' (gq_b), at dot (gdot) and at nrm (gn, stored as gn / nrm).  No product rule is typed here.

Each output element also gets a magnitude bound A, first-order error propagation through the same chain: GEMM |W| A_in + |b|, product
A_a |b| + |a| A_b, silu 1.1 A_x + |silu(x)|, sqrt and division their derivatives times A, and A >= |value| everywhere.  The GPU tests
check |kernel - reference| <= C A elementwise."""
import math

import numpy as np
import torch
from torch.func import vjp

F = 128
L = 6                       # layers of the synthetic weights; drawn independently, so a kernel that reads another layer's tile fails
N_MAX = 997                 # atoms of the synthetic inputs (every test N is a prefix)
EPS = float(np.float32(1e-8))  # PaiNN's norm epsilon as the kernels see it (nb200_painn_weights.epsilon)
SENTINEL_BITS = 0x7FBADBAD  # a NaN payload no kernel writes: rows at or past n_atoms must keep it bitwise
D64 = torch.float64
# GPU tolerance of the fused programs, |kernel - reference| <= C A: 3xTF32 GEMMs with K <= 384 and fp32 epilogues.  The largest err / A
# measured on an H100 is 1.7e-7 (VW); a 3xTF32 product that loses one of its correction terms is off by about 2^-12 |w x| per term
C_NODE = 2e-6
# the per-atom kernels: at most ~10 roundings and one expf / division per element (C_POINT); sums over 64 or up to thousands of terms (C_SUM)
C_POINT = 2e-6
C_SUM = 1e-5
NT = (64, 80)  # the tile widths of the fused kernels


def silu(x):
    return x * torch.sigmoid(x)


def dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def dsilu_bound(x):
    """|silu'| term by term, 1 - s counted as 1 + s (in fp32 1 - s is off by u, not by u (1 - s))."""
    s = torch.sigmoid(x)
    return s * (1 + x.abs() * (1 + s))


def dsilu_sens(x):
    """Bound of silu' of a rounded argument: dsilu_bound plus |x silu''| term by term (expf's error grows with |x|)."""
    s = torch.sigmoid(x)
    return dsilu_bound(x) + x.abs() * s * (1 + s) * (2 + x.abs() * (1 + 2 * s))


def _m(A, v):
    return torch.maximum(A, v.abs())


# ------------------------------------------------------------------------------------------------------------------- weights, inputs
def weights(seed=0, n_elem=10):
    """Canonical weight arrays (float32, CPU) of L layers, Xavier-uniform matrices and non-zero biases."""
    gen = torch.Generator().manual_seed(seed)

    def xav(*shape):
        fan = shape[-1] + shape[-2]
        return (torch.rand(*shape, generator=gen) * 2 - 1) * math.sqrt(6.0 / fan)

    def r(*shape, s):
        return torch.randn(*shape, generator=gen) * s

    return dict(A1=xav(L, F, F), c1=r(L, F, s=0.3), A2=xav(L, 3 * F, F), c2=r(L, 3 * F, s=0.1), U=xav(L, 2 * F, F), B1=xav(L, F, 2 * F),
                d1=r(L, F, s=0.3), B2=xav(L, 3 * F, F), d2=r(L, 3 * F, s=0.3), R1=xav(F // 2, F), e1=r(F // 2, s=0.3), R2=r(F // 2, s=0.2),
                e2=r(1, s=0.1), emb=r(n_elem, F, s=1.0))


def inputs(n=N_MAX, seed=1):
    """Inputs of the forward programs (float32, CPU).  Row magnitudes span 1e-3 to 10; every 11th atom has |q| ~ 40 (silu saturates in
    g1pre, h1pre and ro_pre); atom 0 and every 7th atom have mu_mid exactly zero (an isolated atom: nrm at its sqrt(eps) floor)."""
    gen = torch.Generator().manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, 1, generator=gen) * 4 - 3)
    scale[::11] = 40.0
    q_mid = torch.randn(n, F, generator=gen) * scale
    mu_mid = torch.randn(n, 3, F, generator=gen) * (10.0 ** (torch.rand(n, 1, 1, generator=gen) * 3 - 2))
    mu_mid[::7] = 0.0
    q_mlp_in = torch.randn(n, F, generator=gen) * scale.flip(0)
    return dict(q_mid=q_mid, mu_mid=mu_mid.reshape(n, 3 * F), q_mlp_in=q_mlp_in)


def cotangents(n=N_MAX, seed=2):
    """The backward programs' gradient inputs (float32, CPU): gq_a (dE/dq' from the message backward), cur (dE/dmu'), g_xh."""
    gen = torch.Generator().manual_seed(seed)
    s = 10.0 ** (torch.rand(n, 1, generator=gen) * 3 - 2)
    return dict(gq_a=torch.randn(n, F, generator=gen) * s, cur=torch.randn(n, 3 * F, generator=gen) * s.flip(0),
                g_xh=torch.randn(n, 3 * F, generator=gen) * 0.5)


def d64(w):
    return {k: v.to(D64) for k, v in w.items()}


# ------------------------------------------------------------------------------------------------------------------- primal programs
def update(w, l, q, mu, z_nrm=0.0, z_dot=0.0, z_qn=0.0, drop=()):
    """_PaiNNMixing of layer l on q [N, F], mu [N, 3F]; z_*: zero additive inputs at nrm, dot and q' whose cotangents are the hand-off
    arrays.  `drop` removes one term ("eps", "y2dot", "residual", "d2_y1") or takes U, B1, B2 from layer l + 1 ("neighbour")."""
    lm = l + 1 if "neighbour" in drop else l
    N = q.shape[0]
    VW = torch.einsum("nxk,ok->nxo", mu.reshape(N, 3, F), w["U"][lm])
    V, Wv = VW[..., :F], VW[..., F:]
    nrm = torch.sqrt((V * V).sum(1) + (0.0 if "eps" in drop else EPS)) + z_nrm
    dot = (V * Wv).sum(1) + z_dot
    g1pre = torch.cat([q, nrm], 1) @ w["B1"][lm].T + w["d1"][l]
    d2 = w["d2"][l].clone()
    if "d2_y1" in drop:
        d2[F:2 * F] = 0
    y = silu(g1pre) @ w["B2"][lm].T + d2
    y0, y1, y2 = y[:, :F], y[:, F:2 * F], y[:, 2 * F:]
    q_next = (0.0 if "residual" in drop else q) + y0 + (0.0 if "y2dot" in drop else y2 * dot) + z_qn
    mu_next = mu.reshape(N, 3, F) + y1[:, None] * Wv
    return dict(VW=VW.reshape(N, 6 * F), nrm=nrm, dot=dot, g1pre=g1pre, y=y, q_next=q_next, mu_next=mu_next.reshape(N, 3 * F))


def mlp(w, l, q):
    h1pre = q @ w["A1"][l].T + w["c1"][l]
    return dict(h1pre=h1pre, xh=silu(h1pre) @ w["A2"][l].T)


def readout(w, q):
    return dict(ro_pre=q @ w["R1"].T)


def update_bound(w, l, q, mu, v):
    """A of every output of `update` (values v)."""
    N = q.shape[0]
    Aq, Amu = q.abs(), mu.abs().reshape(N, 3, F)
    VW = v["VW"].reshape(N, 3, 2 * F)
    V, Wv = VW[..., :F], VW[..., F:]
    AVW = _m(torch.einsum("nxk,ok->nxo", Amu, w["U"][l].abs()), VW)
    AV, AW = AVW[..., :F], AVW[..., F:]
    nrm, dot = v["nrm"], v["dot"]
    Anrm = _m(((2 * V.abs() * AV).sum(1) + EPS) / (2 * nrm), nrm)
    Adot = _m((AV * Wv.abs() + V.abs() * AW).sum(1), dot)
    Ag1 = _m(torch.cat([Aq, Anrm], 1) @ w["B1"][l].abs().T + w["d1"][l].abs(), v["g1pre"])
    Aact = 1.1 * Ag1 + silu(v["g1pre"]).abs()
    y = v["y"]
    Ay = _m(Aact @ w["B2"][l].abs().T + w["d2"][l].abs(), y)
    Aqn = _m(Aq + Ay[:, :F] + Ay[:, 2 * F:] * dot.abs() + y[:, 2 * F:].abs() * Adot, v["q_next"])
    Amun = _m(Amu + Ay[:, None, F:2 * F] * Wv.abs() + y[:, None, F:2 * F].abs() * AW, v["mu_next"].reshape(N, 3, F))
    return dict(VW=AVW.reshape(N, 6 * F), nrm=Anrm, dot=Adot, g1pre=Ag1, y=Ay, q_next=Aqn, mu_next=Amun.reshape(N, 3 * F))


def mlp_bound(w, l, Aq, v):
    Ah = _m(Aq @ w["A1"][l].abs().T + w["c1"][l].abs(), v["h1pre"])
    return dict(h1pre=Ah, xh=_m((1.1 * Ah + silu(v["h1pre"]).abs()) @ w["A2"][l].abs().T, v["xh"]))


def readout_bound(w, Aq, v):
    return dict(ro_pre=_m(Aq @ w["R1"].abs().T, v["ro_pre"]))


# ------------------------------------------------------------------------------------------------------------------- kernel programs
FWD_KINDS = ("mlp", "upd_mlp", "upd_ro")   # (-1, l, 0), (l, l + 1, 0), (l, -1, 1)
BWD_KINDS = ("ro_upd", "mlp_upd")          # readout + update(l), message MLP(l + 1) + update(l)
FWD_OUT = dict(mlp=("h1pre", "xh"), upd_mlp=("VW", "nrm", "dot", "g1pre", "y", "q_next", "mu_next", "h1pre", "xh"),
               upd_ro=("VW", "nrm", "dot", "g1pre", "y", "q_next", "mu_next", "ro_pre"))
BWD_OUT = ("gq_b", "gdot", "gn", "gq_a", "cur")


def program(kind, l):
    """(layer_upd, layer_mlp, readout) of a forward kind, or (readout, layer_mlp, layer_upd) of a backward kind, at layer l."""
    return dict(mlp=(-1, l, 0), upd_mlp=(l, l + 1, 0), upd_ro=(l, -1, 1), ro_upd=(1, -1, l), mlp_upd=(0, l + 1, l))[kind]


def fwd_program(w, kind, l, x, drop=()):
    """Values and bounds (float64 [N, cols]) of every output of a forward program; w float64, x the float32 inputs."""
    if kind == "mlp":
        q = x["q_mlp_in"].to(D64)
        v = mlp(w, l, q)
        return v, mlp_bound(w, l, q.abs(), v)
    q, mu = x["q_mid"].to(D64), x["mu_mid"].to(D64)
    v = update(w, l, q, mu, drop=drop)
    A = update_bound(w, l, q, mu, v)
    if kind == "upd_mlp":
        m = mlp(w, l + 1, v["q_next"])
        A.update(mlp_bound(w, l + 1, A["q_next"], m))
    else:
        m = readout(w, v["q_next"])
        A.update(readout_bound(w, A["q_next"], m))
    v.update(m)
    return v, A


def bwd_inputs(w32, kind, l, x, g):
    """float32 inputs of a backward program: the saved forward arrays (rounded from the float64 forward; ro_pre with e1 added in fp32, as
    k_readout leaves it) and the gradient inputs."""
    w = d64(w32)
    v, _ = fwd_program(w, "upd_ro" if kind == "ro_upd" else "upd_mlp", l, x)
    s = {k: v[k].float() for k in ("VW", "nrm", "dot", "g1pre", "y")}
    s["cur"] = g["cur"]
    if kind == "ro_upd":
        s["ro_pre"] = v["ro_pre"].float() + w32["e1"]
    else:
        s["h1pre"], s["g_xh"], s["gq_a"] = v["h1pre"].float(), g["g_xh"], g["gq_a"]
    return s


def bwd_program(w, kind, l, x, b, drop=()):
    """Values and bounds (float64) of every output of a backward program: vjp of the composed forward of (q_mid, mu_mid) with the
    cotangents the kernel reads (b: bwd_inputs), and the hand-off arrays as cotangents of zero inputs at q', dot and nrm."""
    N = x["q_mid"].shape[0]
    q, mu = x["q_mid"].to(D64), x["mu_mid"].to(D64)
    z = torch.zeros(N, F, dtype=D64)
    cur = b["cur"].to(D64)

    if kind == "ro_upd":
        g_ro = w["R2"] * dsilu(b["ro_pre"].to(D64))

        def f(q, mu, zn, zd, zq):
            u = update(w, l, q, mu, zn, zd, zq, drop=drop)
            return readout(w, u["q_next"])["ro_pre"], u["mu_next"]

        cot = (g_ro, cur)
    else:
        def f(q, mu, zn, zd, zq):
            u = update(w, l, q, mu, zn, zd, zq, drop=drop)
            return mlp(w, l + 1, u["q_next"])["xh"], u["q_next"], u["mu_next"]

        cot = (b["g_xh"].to(D64), b["gq_a"].to(D64), cur)
    _, pull = vjp(f, q, mu, z, z, z)
    gq_a, g_mu, g_nrm, g_dot, g_qn = pull(cot)
    nrm = b["nrm"].to(D64)
    v = dict(gq_b=g_qn, gdot=g_dot, gn=g_nrm / nrm, gq_a=gq_a, cur=g_mu)

    # bounds, first-order through the kernel's chain
    VW = b["VW"].to(D64).reshape(N, 3, 2 * F)
    V, Wv = VW[..., :F].abs(), VW[..., F:].abs()
    y = b["y"].to(D64).abs()
    if kind == "ro_upd":
        Agro = w["R2"].abs() * dsilu_bound(b["ro_pre"].to(D64))
        Agqb = Agro @ w["R1"].abs()
    else:
        Agt = (b["g_xh"].to(D64).abs() @ w["A2"][l + 1].abs()) * dsilu_bound(b["h1pre"].to(D64))
        Agqb = b["gq_a"].to(D64).abs() + Agt @ w["A1"][l + 1].abs()
    Agqb = _m(Agqb, v["gq_b"])
    Agdot = _m(Agqb * y[:, 2 * F:], v["gdot"])
    acur = cur.abs().reshape(N, 3, F)
    Agy = torch.cat([Agqb, (acur * Wv).sum(1), Agqb * b["dot"].to(D64).abs()], 1)
    Agt2 = (Agy @ w["B2"][l].abs()) * dsilu_bound(b["g1pre"].to(D64))
    Agq_a = _m(Agqb + Agt2 @ w["B1"][l][:, :F].abs(), v["gq_a"])
    As = _m((Agt2 @ w["B1"][l][:, F:].abs()) / nrm, v["gn"])
    AgV = Agdot[:, None] * Wv + As[:, None] * V
    AgW = acur * y[:, None, F:2 * F] + Agdot[:, None] * V
    Acur = acur + AgV @ w["U"][l][:F].abs() + AgW @ w["U"][l][F:].abs()
    A = dict(gq_b=Agqb, gdot=Agdot, gn=As, gq_a=Agq_a, cur=_m(Acur.reshape(N, 3 * F), v["cur"]))
    return v, A


# ------------------------------------------------------------------------------------------------------------------- weight images
TILES_PER_LAYER = 22


def tile_source(w, idx):
    """The 128 x 128 block (float32 numpy, zero padded) that tile idx of the prepared buffer holds: row r = output feature (forward
    tiles) or input feature (transposed tiles), column k = the reduction index.  Restated from the tile list above k_prep_painn."""
    out = np.zeros((128, 128), np.float32)
    nL = w["U"].shape[0]
    if idx >= nL * TILES_PER_LAYER:
        R1 = w["R1"].numpy()
        if idx == nL * TILES_PER_LAYER:
            out[:F // 2] = R1          # rows 64..127 are padding
        else:
            out[:, :F // 2] = R1.T     # k 64..127 are padding
        return out
    l, t = divmod(idx, TILES_PER_LAYER)
    A1, A2, U, B1, B2 = (w[k][l].numpy() for k in ("A1", "A2", "U", "B1", "B2"))
    fwd = [U[:F], U[F:], B1[:, :F], B1[:, F:], B2[:F], B2[F:2 * F], B2[2 * F:], A1, A2[:F], A2[F:2 * F], A2[2 * F:]]
    if t < len(fwd):
        return fwd[t].copy()
    # transposed: element (r = input feature, k = output feature)
    trans = [B2[:F].T, B2[F:2 * F].T, B2[2 * F:].T, B1[:, :F].T, B1[:, F:].T, U[:F].T, U[F:].T, A2[:F].T, A2[F:2 * F].T, A2[2 * F:].T, A1.T]
    return np.ascontiguousarray(trans[t - len(fwd)])


def decode_tile(raw):
    """(hi, lo) [128 rows, 128 k] of one 128 KB tile image: per stage of 32 k, hi then lo, each 8 chunks of 4 k x 128 rows x 16 bytes."""
    t = np.asarray(raw, np.float32).reshape(4, 2, 8, 128, 4)  # stage, hi / lo, chunk, row, k % 4
    t = t.transpose(1, 3, 0, 2, 4).reshape(2, 128, 128)
    return t[0], t[1]


def rna_tf32(x):
    """cvt.rna.tf32.f32 (split_tf32 in wgmma.cuh): round to nearest, ties away from zero, to 10 explicit mantissa bits."""
    u = np.asarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def split_tf32(x):
    x = np.asarray(x, np.float32)
    hi = rna_tf32(x)
    return hi, rna_tf32((x - hi).astype(np.float32))
