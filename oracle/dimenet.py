"""CPU restatement of DimeNet++ as nablaDFT wraps it (config/model/dimenetplusplus.yaml).  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The wrapper `DimeNetPlusPlusPotential` (nablaDFT/dimenetplusplus/dimenetplusplus.py:22-113) is the reference's own code and is PINNED through
tests/golden/dimenet_f64.npz (tests/golden/make_golden_dimenet.py runs the reference file with this module's core in place of PyG's class).
The core `torch_geometric.nn.models.DimeNetPlusPlus` (torch-geometric 2.4.0, torch-cluster 1.6.3, setup.py:39,41) is not installed, so
everything marked [3P-memory] below restates the published semantics of those packages from memory.  When the real packages are available,
re-check in this order:
  1. [3P-memory] the angle of DimeNetPlusPlus: atan2(|pos_ij x pos_jk|, pos_ij . pos_jk) with pos_ij = pos[i] - pos[j], pos_jk = pos[j] - pos[k]
     (the plain DimeNet branch uses pos_ji = pos[j] - pos[i], pos_ki = pos[k] - pos[i] instead);
  2. [3P-memory] radius_graph(pos, r, batch, loop=False, max_num_neighbors=K) asks `radius` for K + 1 sources per target, candidates in
     ascending source index within the molecule, d^2 < r^2 strictly, the target itself included; the self loop is dropped afterwards, so a
     target keeps K sources when it is among its own first K + 1 candidates and K + 1 otherwise (oracle/graph.py keeps the first K);
  3. [3P-memory] DimeNet.triplets: for every edge j -> i the triplets k -> j -> i are the edges into j with k != i, ordered by the ji edge,
     then by ascending k;
  4. [3P-memory] bases: Envelope(p = exponent + 1), BesselBasisLayer env(d/c) sin(freq_n d/c) with learnable freq (init n pi),
     SphericalBasisLayer env(d_kj/c) N_ln j_l(z_ln d_kj/c) Y_l^0(angle), flattened l-major;
  5. [3P-memory] blocks: EmbeddingBlock (Embedding(95, H), row = z), InteractionPPBlock, OutputPPBlock (lin zero-initialised by PyG), swish.
"""
import math

import numpy as np
import torch
from torch import nn


# ---- graph ---------------------------------------------------------------------------------------------------------------------------------
def radius_graph_kp1(pos: torch.Tensor, batch: torch.Tensor, r: float, max_num_neighbors: int) -> torch.Tensor:
    """[3P-memory] torch_cluster.radius_graph(loop=False): -> edge_index [2, E] = (source j, target i), CSR by target, sources ascending."""
    src, tgt = [], []
    p = pos.detach()
    b = batch.tolist()
    n = p.shape[0]
    start = 0
    while start < n:
        end = start
        while end < n and b[end] == b[start]:
            end += 1
        d2 = ((p[start:end, None, :] - p[None, start:end, :]) ** 2).sum(-1)
        for a in range(end - start):
            cand = [j for j in range(end - start) if d2[a, j] < r * r][: max_num_neighbors + 1]
            for j in cand:
                if j != a:
                    src.append(start + j)
                    tgt.append(start + a)
        start = end
    return torch.tensor([src, tgt], dtype=torch.long).reshape(2, -1)


def triplets(edge_index: torch.Tensor, num_nodes: int):
    """[3P-memory] DimeNet.triplets -> (i, j, idx_i, idx_j, idx_k, idx_kj, idx_ji); edge e is j -> i."""
    j, i = edge_index
    into = [[] for _ in range(num_nodes)]  # edges into each atom, ascending source
    for e in range(j.numel()):
        into[int(i[e])].append(e)
    for lst in into:
        lst.sort(key=lambda e: int(j[e]))
    idx_kj, idx_ji = [], []
    for e in range(j.numel()):
        for kj in into[int(j[e])]:
            if int(j[kj]) != int(i[e]):
                idx_kj.append(kj)
                idx_ji.append(e)
    idx_kj = torch.tensor(idx_kj, dtype=torch.long)
    idx_ji = torch.tensor(idx_ji, dtype=torch.long)
    return i, j, i[idx_ji], j[idx_ji], j[idx_kj], idx_kj, idx_ji


# ---- bases ---------------------------------------------------------------------------------------------------------------------------------
def bessel_zeros(n: int, k: int) -> np.ndarray:
    """z[l, m]: the first k positive zeros of the spherical Bessel function j_l, l < n (zeros of j_l interlace those of j_{l-1})."""
    from scipy.optimize import brentq
    from scipy.special import spherical_jn

    z = np.zeros((n, k + n))
    z[0] = np.arange(1, k + n + 1) * np.pi
    for l in range(1, n):
        for m in range(k + n - l):
            z[l, m] = brentq(lambda x: spherical_jn(l, x), z[l - 1, m], z[l - 1, m + 1])
    return z[:, :k]


def bessel_normalizers(z: np.ndarray) -> np.ndarray:
    from scipy.special import spherical_jn

    return np.stack([1.0 / np.sqrt(0.5 * spherical_jn(l + 1, z[l]) ** 2) for l in range(z.shape[0])])


def spherical_jn_torch(l: int, x: torch.Tensor) -> torch.Tensor:
    """j_l by its closed sin / cos form (what the sympy-generated functions evaluate); float64 here."""
    s, c = torch.sin(x), torch.cos(x)
    j0 = s / x
    if l == 0:
        return j0
    j1 = s / x ** 2 - c / x
    a, b = j0, j1
    for m in range(1, l):
        a, b = b, (2 * m + 1) / x * b - a
    return b


def legendre_y0(l_max: int, ct: torch.Tensor):
    """Y_l^0 = sqrt((2l+1)/(4 pi)) P_l(cos theta), l < l_max."""
    out = [torch.ones_like(ct), ct]
    for l in range(1, l_max - 1):
        out.append(((2 * l + 1) * ct * out[l] - l * out[l - 1]) / (l + 1))
    return [math.sqrt((2 * l + 1) / (4 * math.pi)) * out[l] for l in range(l_max)]


class Envelope(nn.Module):
    def __init__(self, exponent):
        super().__init__()
        self.p = exponent + 1
        self.a = -(self.p + 1) * (self.p + 2) / 2
        self.b = self.p * (self.p + 2)
        self.c = -self.p * (self.p + 1) / 2

    def forward(self, x):
        p, a, b, c = self.p, self.a, self.b, self.c
        x0 = x.pow(p - 1)
        return (1.0 / x + a * x0 + b * x0 * x + c * x0 * x * x) * (x < 1.0).to(x.dtype)


class BesselBasisLayer(nn.Module):
    def __init__(self, num_radial, cutoff, envelope_exponent):
        super().__init__()
        self.cutoff = cutoff
        self.envelope = Envelope(envelope_exponent)
        self.freq = nn.Parameter(torch.arange(1, num_radial + 1, dtype=torch.float32) * math.pi)

    def forward(self, dist):
        dist = dist.unsqueeze(-1) / self.cutoff
        return self.envelope(dist) * (self.freq * dist).sin()


class SphericalBasisLayer(nn.Module):
    def __init__(self, num_spherical, num_radial, cutoff, envelope_exponent):
        super().__init__()
        self.ns, self.nr, self.cutoff = num_spherical, num_radial, cutoff
        self.envelope = Envelope(envelope_exponent)
        z = bessel_zeros(num_spherical, num_radial)
        self.zeros, self.norms = z, bessel_normalizers(z)

    def forward(self, dist, angle, idx_kj):
        x = dist / self.cutoff
        zt = torch.as_tensor(self.zeros, dtype=x.dtype)
        nt = torch.as_tensor(self.norms, dtype=x.dtype)
        rbf = torch.stack([nt[l, m] * spherical_jn_torch(l, zt[l, m] * x) for l in range(self.ns) for m in range(self.nr)], dim=1)
        rbf = self.envelope(x).unsqueeze(-1) * rbf
        cbf = torch.stack(legendre_y0(self.ns, torch.cos(angle)), dim=1)
        return (rbf[idx_kj].view(-1, self.ns, self.nr) * cbf.view(-1, self.ns, 1)).view(-1, self.ns * self.nr)


# ---- blocks --------------------------------------------------------------------------------------------------------------------------------
def swish(x):
    return x * x.sigmoid()


class EmbeddingBlock(nn.Module):
    def __init__(self, num_radial, hidden):
        super().__init__()
        self.emb = nn.Embedding(95, hidden)
        self.lin_rbf = nn.Linear(num_radial, hidden)
        self.lin = nn.Linear(3 * hidden, hidden)

    def forward(self, z, rbf, i, j):
        x = self.emb(z)
        rbf = swish(self.lin_rbf(rbf))
        return swish(self.lin(torch.cat([x[i], x[j], rbf], dim=-1)))


class ResidualLayer(nn.Module):
    def __init__(self, hidden):
        super().__init__()
        self.lin1 = nn.Linear(hidden, hidden)
        self.lin2 = nn.Linear(hidden, hidden)

    def forward(self, x):
        return x + swish(self.lin2(swish(self.lin1(x))))


class InteractionPPBlock(nn.Module):
    def __init__(self, hidden, int_emb, basis_emb, num_spherical, num_radial, num_before_skip, num_after_skip):
        super().__init__()
        self.lin_rbf1 = nn.Linear(num_radial, basis_emb, bias=False)
        self.lin_rbf2 = nn.Linear(basis_emb, hidden, bias=False)
        self.lin_sbf1 = nn.Linear(num_spherical * num_radial, basis_emb, bias=False)
        self.lin_sbf2 = nn.Linear(basis_emb, int_emb, bias=False)
        self.lin_kj = nn.Linear(hidden, hidden)
        self.lin_ji = nn.Linear(hidden, hidden)
        self.lin_down = nn.Linear(hidden, int_emb, bias=False)
        self.lin_up = nn.Linear(int_emb, hidden, bias=False)
        self.layers_before_skip = nn.ModuleList([ResidualLayer(hidden) for _ in range(num_before_skip)])
        self.lin = nn.Linear(hidden, hidden)
        self.layers_after_skip = nn.ModuleList([ResidualLayer(hidden) for _ in range(num_after_skip)])

    def forward(self, x, rbf, sbf, idx_kj, idx_ji):
        x_ji = swish(self.lin_ji(x))
        x_kj = swish(self.lin_kj(x))
        x_kj = x_kj * self.lin_rbf2(self.lin_rbf1(rbf))
        x_kj = swish(self.lin_down(x_kj))
        x_kj = x_kj[idx_kj] * self.lin_sbf2(self.lin_sbf1(sbf))
        x_kj = torch.zeros(x.shape[0], x_kj.shape[1], dtype=x.dtype).index_add_(0, idx_ji, x_kj)
        x_kj = swish(self.lin_up(x_kj))
        h = x_ji + x_kj
        for layer in self.layers_before_skip:
            h = layer(h)
        h = swish(self.lin(h)) + x
        for layer in self.layers_after_skip:
            h = layer(h)
        return h


class OutputPPBlock(nn.Module):
    def __init__(self, num_radial, hidden, out_emb, out_channels, num_layers):
        super().__init__()
        self.lin_rbf = nn.Linear(num_radial, hidden, bias=False)
        self.lin_up = nn.Linear(hidden, out_emb, bias=False)
        self.lins = nn.ModuleList([nn.Linear(out_emb, out_emb) for _ in range(num_layers)])
        self.lin = nn.Linear(out_emb, out_channels, bias=False)
        nn.init.zeros_(self.lin.weight)  # [3P-memory] output_initializer='zeros'

    def forward(self, x, rbf, i, num_nodes):
        x = self.lin_rbf(rbf) * x
        x = torch.zeros(num_nodes, x.shape[1], dtype=x.dtype).index_add_(0, i, x)
        x = self.lin_up(x)
        for lin in self.lins:
            x = swish(lin(x))
        return self.lin(x)


class DimeNetPlusPlus(nn.Module):
    """[3P-memory] torch_geometric.nn.models.DimeNetPlusPlus (2.4.0): forward(z, pos, batch) -> [B, out_channels]."""

    def __init__(self, hidden_channels, out_channels, num_blocks, int_emb_size, basis_emb_size, out_emb_channels, num_spherical=7,
                 num_radial=6, cutoff=5.0, max_num_neighbors=32, envelope_exponent=5, num_before_skip=1, num_after_skip=2,
                 num_output_layers=3, act="swish"):
        super().__init__()
        assert act == "swish"
        self.cutoff, self.max_num_neighbors, self.num_blocks = cutoff, max_num_neighbors, num_blocks
        self.rbf = BesselBasisLayer(num_radial, cutoff, envelope_exponent)
        self.sbf = SphericalBasisLayer(num_spherical, num_radial, cutoff, envelope_exponent)
        self.emb = EmbeddingBlock(num_radial, hidden_channels)
        self.output_blocks = nn.ModuleList([OutputPPBlock(num_radial, hidden_channels, out_emb_channels, out_channels, num_output_layers)
                                            for _ in range(num_blocks + 1)])
        self.interaction_blocks = nn.ModuleList([InteractionPPBlock(hidden_channels, int_emb_size, basis_emb_size, num_spherical, num_radial,
                                                                    num_before_skip, num_after_skip) for _ in range(num_blocks)])

    def forward(self, z, pos, batch=None):
        if batch is None:
            batch = torch.zeros(z.shape[0], dtype=torch.long)
        edge_index = radius_graph_kp1(pos, batch, self.cutoff, self.max_num_neighbors)
        i, j, idx_i, idx_j, idx_k, idx_kj, idx_ji = triplets(edge_index, z.shape[0])
        dist = (pos[i] - pos[j]).pow(2).sum(dim=-1).sqrt()
        pos_jk, pos_ij = pos[idx_j] - pos[idx_k], pos[idx_i] - pos[idx_j]  # [3P-memory] the DimeNetPlusPlus branch
        a = (pos_ij * pos_jk).sum(dim=-1)
        b = torch.cross(pos_ij, pos_jk, dim=-1).norm(dim=-1)
        angle = torch.atan2(b, a)
        rbf = self.rbf(dist)
        sbf = self.sbf(dist, angle, idx_kj)
        x = self.emb(z, rbf, i, j)
        P = self.output_blocks[0](x, rbf, i, num_nodes=pos.shape[0])
        for blk, out in zip(self.interaction_blocks, self.output_blocks[1:]):
            x = blk(x, rbf, sbf, idx_kj, idx_ji)
            P = P + out(x, rbf, i, num_nodes=pos.shape[0])
        n_mol = int(batch.max()) + 1 if batch.numel() else 0
        return torch.zeros(n_mol, P.shape[1], dtype=P.dtype).index_add_(0, batch, P)


class DimeNetPlusPlusPotentialOracle(nn.Module):
    """The wrapper, restated from nablaDFT/dimenetplusplus/dimenetplusplus.py:22-113 (same parameter names: `net.*`, `regr_or_cls_nn.*`)."""

    def __init__(self, node_latent_dim=50, scaler=None, dimenet_hidden_channels=256, dimenet_num_blocks=6, dimenet_int_emb_size=64,
                 dimenet_basis_emb_size=8, dimenet_out_emb_channels=256, dimenet_num_spherical=7, dimenet_num_radial=6,
                 dimenet_max_num_neighbors=32, dimenet_envelope_exponent=5, dimenet_num_before_skip=1, dimenet_num_after_skip=2,
                 dimenet_num_output_layers=3, cutoff=5.0, do_postprocessing=False):
        super().__init__()
        self.scaler, self.do_postprocessing = scaler, do_postprocessing
        self.net = DimeNetPlusPlus(dimenet_hidden_channels, node_latent_dim, dimenet_num_blocks, dimenet_int_emb_size, dimenet_basis_emb_size,
                                   dimenet_out_emb_channels, dimenet_num_spherical, dimenet_num_radial, cutoff, dimenet_max_num_neighbors,
                                   dimenet_envelope_exponent, dimenet_num_before_skip, dimenet_num_after_skip, dimenet_num_output_layers)
        L = node_latent_dim
        self.regr_or_cls_nn = nn.Sequential(nn.Linear(L, L), nn.SiLU(), nn.Linear(L, L // 2), nn.SiLU(), nn.Linear(L // 2, L // 2), nn.SiLU(),
                                            nn.Linear(L // 2, 1))

    def forward(self, z, pos, batch):
        """-> (energy [B], forces [N, 3], graph embeddings [B, L]); forces = -d(unscaled prediction)/d pos (dimenetplusplus.py:93-113)."""
        with torch.enable_grad():
            pos = pos.detach().requires_grad_(True)
            g = self.net(z=z, pos=pos, batch=batch)
            pred = torch.flatten(self.regr_or_cls_nn(g).contiguous())
            grad = torch.autograd.grad(pred, pos, grad_outputs=torch.ones_like(pred), allow_unused=True)[0]
            forces = -grad if grad is not None else torch.zeros_like(pos)  # no edges at all: pos never entered the graph
        if self.scaler and self.do_postprocessing:
            pred = self.scaler["scale_"] * pred + self.scaler["mean_"]
        return pred.detach(), forces.detach(), g.detach()
