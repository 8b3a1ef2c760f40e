"""CPU oracle (TEST INFRASTRUCTURE, never imported by the package) for the whole PhiSNet model -- a float64 restatement of
`nablaDFT/phisnet/nn/neural_network.py` (NeuralNetwork.forward :717-995) on top of the layer oracles of oracle/phisnet.py.

Same module tree and parameter names as the reference (and as nabladft_b200.phisnet.NeuralNetwork), so one state dict serves all three.
Features are lists over L of [rows, 2L+1, F]; pairs are all ordered i != j inside each molecule, i-major and j ascending (fill_idx).
The neighbour sum of the pair features is sum_{k != i,j} radial_ij(rbf_ik) fpn[k] = T_i - radial_ij(rbf_ij) fpn[j] (O(P)); passing the
reference's pindex lists to `forward(..., pindex=...)` evaluates the reference's own gather formulation instead.
The block assembly is vectorised over all blocks of one element pair (matrix_block / generate_matrix_from_irreps, :636-706).
PINNED: tests/test_oracle_phisnet_model.py compares it with outputs of the reference's own NeuralNetwork (tests/golden/phisnet_model.npz).
"""
import math
import os
from typing import Dict, List

import numpy as np
import torch
from torch import nn

from .phisnet import ClebschGordan, PairMixing, SphericalLinear

_GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "phisnet_model.npz")


def spherical_harmonics(u: torch.Tensor) -> List[torch.Tensor]:
    """Real spherical harmonics l = 0..4 of unit vectors u [P,3] in PhiSNet's convention: m = -l..l, Condon-Shortley phase, no 1/sqrt(4 pi)."""
    x, y, z = u[:, 0], u[:, 1], u[:, 2]
    x2, y2, z2 = x * x, y * y, z * z
    s = math.sqrt
    Y0 = [torch.ones_like(x)]
    Y1 = [s(3) * y, s(3) * z, s(3) * x]
    Y2 = [s(15) * x * y, s(15) * y * z, s(5) / 2 * (3 * z2 - 1), s(15) * x * z, s(15) / 2 * (x2 - y2)]
    Y3 = [s(70) / 4 * y * (3 * x2 - y2), s(105) * x * y * z, s(42) / 4 * y * (5 * z2 - 1), s(7) / 2 * z * (5 * z2 - 3),
          s(42) / 4 * x * (5 * z2 - 1), s(105) / 2 * z * (x2 - y2), s(70) / 4 * x * (x2 - 3 * y2)]
    Y4 = [3 * s(35) / 2 * x * y * (x2 - y2), 3 * s(70) / 4 * y * z * (3 * x2 - y2), s(45) / 2 * x * y * (7 * z2 - 1),
          3 * s(10) / 4 * y * z * (7 * z2 - 3), 3 / 8 * (35 * z2 * z2 - 30 * z2 + 3), 3 * s(10) / 4 * x * z * (7 * z2 - 3),
          s(45) / 4 * (x2 - y2) * (7 * z2 - 1), 3 * s(70) / 4 * x * z * (x2 - 3 * y2), 3 * s(35) / 8 * (x2 * x2 - 6 * x2 * y2 + y2 * y2)]
    return [torch.stack(Y, dim=-1) for Y in (Y0, Y1, Y2, Y3, Y4)]


class Swish(nn.Module):
    def __init__(self, num_features):
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(num_features))
        self.beta = nn.Parameter(torch.full((num_features,), 1.702))

    def forward(self, x):
        return self.alpha * x * torch.sigmoid(self.beta * x)


class Embedding(nn.Module):
    def __init__(self, num_features, Zmax=87):
        super().__init__()
        self.register_buffer("electron_config", torch.from_numpy(np.load(_GOLDEN)["electron_config"]).float())
        self.element_embedding = nn.Parameter(torch.zeros(Zmax, num_features))
        self.config_linear = nn.Linear(16, num_features, bias=False)

    def forward(self, Z):
        return (self.element_embedding + self.config_linear(self.electron_config.to(self.element_embedding.dtype)))[Z]


class SphericalEmbedding(nn.Module):
    def __init__(self, order, num_features, Zmax=87):
        super().__init__()
        self.order = order
        self.embedding = Embedding(num_features, Zmax)

    def forward(self, Z):
        e = self.embedding(Z)
        return [e[:, None, :]] + [e.new_zeros(e.shape[0], 2 * L + 1, e.shape[1]) for L in range(1, self.order + 1)]


class ExponentialBernsteinRadialBasisFunctions(nn.Module):
    def __init__(self, num_basis_functions, cutoff):
        super().__init__()
        k = num_basis_functions
        logfact = np.zeros(k)
        for i in range(2, k):
            logfact[i] = logfact[i - 1] + np.log(i)
        v = np.arange(k)
        n = (k - 1) - v
        self.register_buffer("cutoff", torch.tensor(cutoff, dtype=torch.float64))
        self.register_buffer("logc", torch.tensor(logfact[-1] - logfact[v] - logfact[n], dtype=torch.float64))
        self.register_buffer("n", torch.tensor(n, dtype=torch.float64))
        self.register_buffer("v", torch.tensor(v, dtype=torch.float64))
        # softplus_inverse(ini_alpha) evaluated in float32 and stored in a float64 parameter, as the reference initialises it
        a = torch.tensor(0.5)
        self._alpha = nn.Parameter((a + torch.log(-torch.expm1(-a))).to(torch.float64))

    def forward(self, r):  # r [P, 1]; exp-Bernstein polynomials times PhiSNet's cutoff function (functional.py)
        x = -torch.nn.functional.softplus(self._alpha) * r
        x = self.logc + self.n * x + self.v * torch.log(-torch.expm1(x))
        c = self.cutoff
        inside = r < c
        r_ = torch.where(inside, r, torch.zeros_like(r))
        fc = torch.where(inside, torch.exp(-(r_ ** 2) / ((c - r_) * (c + r_))), torch.zeros_like(r))
        return fc * torch.exp(x)


class ResidualBlock(nn.Module):
    def __init__(self, order, num_features, cg):
        super().__init__()
        self.activation_pre, self.activation_post = Swish(num_features), Swish(num_features)
        self.linear1 = SphericalLinear(order, num_features, order, num_features, cg)
        self.linear2 = SphericalLinear(order, num_features, order, num_features, cg)

    def forward(self, xs):
        ys = list(xs)
        ys[0] = self.activation_pre(ys[0])
        ys = self.linear1(ys)
        ys[0] = self.activation_post(ys[0])
        ys = self.linear2(ys)
        return [x + y for x, y in zip(xs, ys)]


class ResidualStack(nn.Module):
    def __init__(self, num_blocks, order, num_features, cg):
        super().__init__()
        self.stack = nn.ModuleList([ResidualBlock(order, num_features, cg) for _ in range(num_blocks)])

    def forward(self, xs):
        for b in self.stack:
            xs = b(xs)
        return list(xs)


class InteractionBlock(nn.Module):
    def __init__(self, order, F, K, n_vi, n_vj, n_v, cg):
        super().__init__()
        self.order = order
        self.activation_i, self.activation_j, self.activation_v = Swish(F), Swish(F), Swish(F)
        self.angular_fn1 = SphericalLinear(order, 1, order, F, cg, mix_orders=False)
        self.angular_fn2 = SphericalLinear(order, 1, order, F, cg, mix_orders=False)
        self.radial_fn = nn.ModuleList([nn.Linear(K, F, bias=False) for _ in range(order + 1)])
        self.mixing = PairMixing(order, order, order, K, F, cg)
        self.linear_i = SphericalLinear(order, F, order, F, cg)
        self.linear_j = SphericalLinear(order, F, order, F, cg)
        self.linear_v = SphericalLinear(order, F, order, F, cg)
        self.residual_pre_vi = ResidualStack(n_vi, order, F, cg)
        self.residual_pre_vj = ResidualStack(n_vj, order, F, cg)
        self.residual_post_v = ResidualStack(n_v, order, F, cg)

    def forward(self, xs, rbf, sph, idx_i, idx_j):  # interaction_block.py:129-150
        yi = self.residual_pre_vi(xs)
        yi[0] = self.activation_i(yi[0])
        yi = self.linear_i(yi)
        yj = self.residual_pre_vj(xs)
        yj[0] = self.activation_j(yj[0])
        yj = [y[idx_j] for y in self.linear_j(yj)]
        vs = self.mixing(yj, self.angular_fn1(sph), rbf)
        a = self.angular_fn2(sph)
        vs = [yi[L].index_add(0, idx_i, vs[L] + self.radial_fn[L](rbf) * a[L] * yj[0]) for L in range(self.order + 1)]
        vs = self.residual_post_v(vs)
        vs[0] = self.activation_v(vs[0])
        vs = self.linear_v(vs)
        return [x + v for x, v in zip(xs, vs)]


class ModularBlock(nn.Module):
    def __init__(self, order, F, K, n_pre_x, n_post_x, n_vi, n_vj, n_v, n_out, cg):
        super().__init__()
        self.interaction = InteractionBlock(order, F, K, n_vi, n_vj, n_v, cg)
        self.residual_pre_x = ResidualStack(n_pre_x, order, F, cg)
        self.residual_post_x = ResidualStack(n_post_x, order, F, cg)
        self.residual_out = ResidualStack(n_out, order, F, cg)

    def forward(self, xs, rbf, sph, idx_i, idx_j):
        xs = self.residual_pre_x(xs)
        xs = self.interaction(xs, rbf, sph, idx_i, idx_j)
        xs = self.residual_post_x(xs)
        return xs, self.residual_out(xs)


class EnergyLayer(nn.Module):
    def __init__(self, num_in, num_out, activation):
        super().__init__()
        self.linear_diagonal = nn.Linear(num_in, num_out)
        self.linear_offdiagonal = nn.Linear(num_in, num_out)
        self.linear_out = nn.Linear(2 * num_out, 1)
        self.activation = activation


def _irreps(max_orbitals):
    def add(oi, oj, irreps, nl):
        for n_i, (z_i, l_i) in enumerate(oi):
            for n_j, (z_j, l_j) in enumerate(oj):
                for L in range(abs(l_i - l_j), l_i + l_j + 1):
                    if (z_i, z_j, n_i, n_j, L) not in irreps:
                        irreps[(z_i, z_j, n_i, n_j, L)] = nl[L]
                        nl[L] += 1
    lmax = max(l for o in max_orbitals for _, l in o)
    ii, nl_ii, ij, nl_ij = {}, [0] * (2 * lmax + 1), {}, [0] * (2 * lmax + 1)
    for o in max_orbitals:
        add(o, o, ii, nl_ii)
    for a, oa in enumerate(max_orbitals):
        for b, ob in enumerate(max_orbitals):
            if a != b:
                add(oa, ob, ij, nl_ij)
    return ii, max(nl_ii), ij, max(nl_ij), lmax


class NeuralNetwork(nn.Module):
    def __init__(self, max_orbitals, order, num_features, num_basis_functions, num_modules, num_residual_pre_x, num_residual_post_x,
                 num_residual_pre_vi, num_residual_pre_vj, num_residual_post_v, num_residual_output, num_residual_pc, num_residual_pn,
                 num_residual_ii, num_residual_ij, num_residual_full_ii, num_residual_full_ij, num_residual_core_ii, num_residual_core_ij,
                 num_residual_over_ij, basis_functions="exp-bernstein", cutoff=15.0, activation="swish", Zmax=87, num_energy_features=64):
        super().__init__()
        assert basis_functions == "exp-bernstein" and activation == "swish"
        self.max_orbitals = tuple(tuple((int(z), int(l)) for z, l in o) for o in max_orbitals)
        self.order = order
        F, K = num_features, num_basis_functions
        cg = self.cg = ClebschGordan()
        self.embedding = SphericalEmbedding(order, F, Zmax)
        self.radial_basis_functions = ExponentialBernsteinRadialBasisFunctions(K, cutoff)
        self.module = nn.ModuleList([ModularBlock(order, F, K, num_residual_pre_x, num_residual_post_x, num_residual_pre_vi, num_residual_pre_vj,
                                                  num_residual_post_v, num_residual_output, cg) for _ in range(num_modules)])
        self.angular_fn = SphericalLinear(order, 1, order, F, cg, mix_orders=False)
        self.mix_s = PairMixing(order, order, order, K, F, cg)
        self.mix_ij = PairMixing(order, order, order, K, F, cg)
        self.radial_ii = nn.ModuleList([nn.Linear(K, F, bias=False) for _ in range(order + 1)])
        self.radial_ij = nn.ModuleList([nn.Linear(K, F, bias=False) for _ in range(order + 1)])
        n_res = dict(pc=num_residual_pc, pn=num_residual_pn, ii=num_residual_ii, ij=num_residual_ij, full_ii=num_residual_full_ii,
                     full_ij=num_residual_full_ij, core_ii=num_residual_core_ii, core_ij=num_residual_core_ij, over_ij=num_residual_over_ij)
        for name, n in n_res.items():
            self.add_module(f"residual_{name}", ResidualStack(n, order, F, cg))
        for name in ("full_ii", "full_ij", "core_ii", "core_ij", "over_ij"):
            self.add_module(f"activation_{name}", Swish(F))
        self.activation_energy = Swish(num_energy_features)
        self.irreps_ii, w_ii, self.irreps_ij, w_ij, lmax = _irreps(self.max_orbitals)
        for name, w in (("full_ii", w_ii), ("core_ii", w_ii), ("over_ii", w_ii), ("full_ij", w_ij), ("core_ij", w_ij), ("over_ij", w_ij)):
            self.add_module(f"output_{name}", SphericalLinear(order, F, 2 * lmax, w, cg))
        self.energy_predictor = EnergyLayer(F, num_energy_features, self.activation_energy)
        self.elem_orbs = {o[0][0]: o for o in self.max_orbitals}

    @staticmethod
    def pairs(sizes):
        """fill_idx order: all ordered i != j inside each molecule, i-major, j ascending (global atom indices)."""
        ii, jj, a0 = [], [], 0
        for n in sizes:
            for i in range(n):
                for j in range(n):
                    if i != j:
                        ii.append(a0 + i)
                        jj.append(a0 + j)
            a0 += n
        return torch.tensor(ii, dtype=torch.long), torch.tensor(jj, dtype=torch.long)

    def pair_neighbour_sum(self, fij, fpn, rbf, idx_i, idx_j, pindex=None):
        """fij[L] += sum_{k != i,j} radial_ij(rbf_ik) fpn[k]: O(P) as T_i - own term, or the reference's pindex gather (neural_network.py:830-838)
        when pindex = (idx_pi, idx_pj) is given (per-molecule lists already offset to global pair indices)."""
        out = []
        for L in range(self.order + 1):
            fpn_j = self.radial_ij[L](rbf) * fpn[L][idx_j]
            if pindex is None:
                T = torch.zeros_like(fpn[L]).index_add(0, idx_i, fpn_j)
                out.append(fij[L] + T[idx_i] - fpn_j)
            else:
                out.append(fij[L].index_add(0, pindex[0], fpn_j[pindex[1]]))
        return out

    def _assemble(self, ii_feats, ij_feats, Z, sizes, idx_i, idx_j, unit_diagonal):
        """Per-molecule matrices B + B^T from the output irreps (matrix_block; diagonal = 1 for the overlap)."""
        norb = [sum(2 * l + 1 for _, l in self.elem_orbs[int(z)]) for z in Z]
        starts, mol_of, a0 = [], [], 0
        mats = []
        for m, n in enumerate(sizes):
            o = 0
            for a in range(a0, a0 + n):
                starts.append(o)
                mol_of.append(m)
                o += norb[a]
            mats.append(ii_feats[0].new_zeros(o, o))
            a0 += n
        blocks = {}  # (kind, za, zb) -> list of (feature row, atom i, atom j)
        for a in range(len(Z)):
            blocks.setdefault((0, int(Z[a]), int(Z[a])), []).append((a, a, a))
        for p, (i, j) in enumerate(zip(idx_i.tolist(), idx_j.tolist())):
            blocks.setdefault((1, int(Z[i]), int(Z[j])), []).append((p, i, j))
        for (kind, za, zb), lst in blocks.items():
            feats, table = (ii_feats, self.irreps_ii) if kind == 0 else (ij_feats, self.irreps_ij)
            rows = torch.tensor([r for r, _, _ in lst])
            oa, ob = self.elem_orbs[za], self.elem_orbs[zb]
            B = feats[0].new_zeros(len(lst), sum(2 * l + 1 for _, l in oa), sum(2 * l + 1 for _, l in ob))
            ra = 0
            for si, (_, li) in enumerate(oa):
                rb = 0
                for sj, (_, lj) in enumerate(ob):
                    for L in range(abs(li - lj), li + lj + 1):
                        irr = feats[L][rows, :, table[(za, zb, si, sj, L)]]  # [blocks, 2L+1]
                        cg = math.sqrt(2 * L + 1) * self.cg(li, lj, L).to(irr.dtype)
                        B[:, ra:ra + 2 * li + 1, rb:rb + 2 * lj + 1] += torch.einsum("abc,pc->pab", cg, irr)
                    rb += 2 * lj + 1
                ra += 2 * li + 1
            for k, (_, i, j) in enumerate(lst):
                M = mats[mol_of[i]]
                M[starts[i]:starts[i] + norb[i], starts[j]:starts[j] + norb[j]] = B[k]
        out = []
        for M in mats:
            M = M + M.T
            if unit_diagonal:
                M.fill_diagonal_(1.0)
            out.append(M)
        return out

    @torch.no_grad()
    def forward(self, pos, Z, sizes, pindex=None, heads=("full", "core", "over")) -> Dict[str, List[torch.Tensor]]:
        """pos [N,3] bohr, Z [N], sizes list of molecule sizes -> {"full"|"core"|"over": [per-molecule Norb x Norb]}."""
        dt = self.radial_ii[0].weight.dtype
        pos, Z = pos.to(dt), Z.long()
        sizes = [int(s) for s in sizes]
        idx_i, idx_j = self.pairs(sizes)
        r = pos[idx_j] - pos[idx_i]
        d = r.norm(dim=-1, keepdim=True)
        rbf = self.radial_basis_functions(d).to(dt)[:, None, :]
        sph = [y[..., None] for y in spherical_harmonics(r / d)]
        xs = self.embedding(Z)
        out = {}
        if "over" in heads:
            fii_over = self.output_over_ii(xs)
            a = self.angular_fn(sph)
            sij = self.mix_s([x[idx_i] for x in xs], [xs[0][idx_j]] + a[1:], rbf)
            f = self.residual_over_ij(sij)
            f[0] = self.activation_over_ij(f[0])
            out["over"] = self._assemble(fii_over, self.output_over_ij(f), Z, sizes, idx_i, idx_j, True)
        fs = [torch.zeros_like(x) for x in xs]
        for mod in self.module:
            xs, ys = mod(xs, rbf, sph, idx_i, idx_j)
            fs = [f + y for f, y in zip(fs, ys)]
        fpc, fpn = self.residual_pc(fs), self.residual_pn(fs)
        fii = [fpc[L].index_add(0, idx_i, self.radial_ii[L](rbf) * fpn[L][idx_j]) for L in range(self.order + 1)]
        fii = self.residual_ii(fii)
        fij = self.mix_ij([f[idx_i] for f in fpc], [f[idx_j] for f in fpc], rbf)
        fij = self.residual_ij(self.pair_neighbour_sum(fij, fpn, rbf, idx_i, idx_j, pindex))
        for head in ("full", "core"):
            if head in heads:
                a = getattr(self, f"residual_{head}_ii")(fii)
                a[0] = getattr(self, f"activation_{head}_ii")(a[0])
                b = getattr(self, f"residual_{head}_ij")(fij)
                b[0] = getattr(self, f"activation_{head}_ij")(b[0])
                out[head] = self._assemble(getattr(self, f"output_{head}_ii")(a), getattr(self, f"output_{head}_ij")(b), Z, sizes, idx_i, idx_j, False)
        return out
