"""PhiSNet Clebsch-Gordan mixing layers on the H100 engine (SURVEY.md section 8 f4) -- mirrors of
`nablaDFT/phisnet/nn/modules/{clebsch_gordan,pair_mixing,self_mixing,spherical_linear}.py`: same constructor signatures, parameter names
(`coeff_{l1}_{l2}_{L}.weight`, `mixcoeff_{l1}_{l2}_{L}`, `keepcoeff_{L}`, `mixing.*`, `linear.{L}.*`) and call contracts (features = lists
over the order L of tensors [..., 2L+1, F]), so a reference state dict loads with strict=True and a PhiSNet built from the reference's
`neural_network.py` can swap these modules in.  The arithmetic is in csrc/phisnet.cu (CG contractions, real CG table of the reference
compiled in) and the wgmma 3xTF32 GEMM (distance-dependent coefficients, per-order Linear).  Inference only; CUDA only (no CPU fallback).
"""
from typing import List

import torch
from torch import nn

from . import _lib
from ._lib import NablaB200Error, check, current_stream, ptr


def _paths(o1, o2, oo, strict_upper=False):
    return [(l1, l2, L) for l1 in range(o1 + 1) for l2 in range((l1 + 1) if strict_upper else 0, o2 + 1)
            for L in range(abs(l1 - l2), min(l1 + l2, oo) + 1)]


def _pack(xs: List[torch.Tensor]):
    """list over L of [..., 2L+1, F] -> ([rows, (order+1)^2, F] contiguous fp32, leading shape)."""
    lead = xs[0].shape[:-2]
    if not xs[0].is_cuda:
        raise NablaB200Error("nabladft_b200.phisnet runs on CUDA only (no CPU fallback)")
    return torch.cat([x.reshape(-1, x.shape[-2], x.shape[-1]) for x in xs], dim=1).to(torch.float32).contiguous(), lead


def _unpack(y: torch.Tensor, order: int, lead) -> List[torch.Tensor]:
    return [y[:, L * L:(L + 1) * (L + 1), :].reshape(*lead, 2 * L + 1, y.shape[-1]) for L in range(order + 1)]


def _no_training(mod):
    if torch.is_grad_enabled() and any(p.requires_grad for p in mod.parameters()) and mod.training:
        raise NotImplementedError("nabladft_b200.phisnet layers are inference-only: call .eval() / torch.no_grad()")


class ClebschGordan(nn.Module):
    """Constructor-compatible placeholder: the real CG tensors (l <= 4) are compiled into the kernels (csrc/phisnet_cg_gen.inc)."""

    def forward(self, l1, l2, l3):
        raise NablaB200Error("the CG tensors live inside the CUDA kernels; use the mixing layers")


class PairMixing(nn.Module):
    def __init__(self, order_in1, order_in2, order_out, num_basis_functions, num_features, clebsch_gordan=None):
        super().__init__()
        self.order_in1, self.order_in2, self.order_out = order_in1, order_in2, order_out
        self.num_basis_functions, self.num_features = num_basis_functions, num_features
        self._paths = _paths(order_in1, order_in2, order_out)
        for l1, l2, L in self._paths:
            lin = nn.Linear(num_basis_functions, num_features, bias=False)
            nn.init.orthogonal_(lin.weight)
            self.add_module(f"coeff_{l1}_{l2}_{L}", lin)

    def coeff(self, l1, l2, L):
        return getattr(self, f"coeff_{l1}_{l2}_{L}")

    @torch.no_grad()
    def forward(self, x1s, x2s, rbf):
        _no_training(self)
        lib = _lib.load()
        x1, lead = _pack(x1s[: self.order_in1 + 1])
        x2, _ = _pack(x2s[: self.order_in2 + 1])
        R, F, K, npath = x1.shape[0], self.num_features, self.num_basis_functions, len(self._paths)
        r = rbf.reshape(-1, K).to(torch.float32).contiguous()
        if r.shape[0] != R:
            r = r.expand(R, K).contiguous()
        wcat = torch.cat([self.coeff(*p).weight for p in self._paths], dim=0).to(torch.float32).contiguous()  # [n_paths * F, K]
        coeff = torch.empty(R, npath * F, dtype=torch.float32, device=x1.device)
        check(lib.nb200_dense(R, npath * F, K, ptr(r), K, ptr(wcat), K, 0, ptr(coeff), npath * F, 0, None, None, 0, current_stream()), "nb200_dense")
        y = torch.empty(R, (self.order_out + 1) ** 2, F, dtype=torch.float32, device=x1.device)
        check(lib.nb200_phis_pair_mixing(ptr(x1), ptr(x2), ptr(coeff), R, F, self.order_in1, self.order_in2, self.order_out, ptr(y), current_stream()),
              "nb200_phis_pair_mixing")
        return _unpack(y, self.order_out, lead)


class SelfMixing(nn.Module):
    def __init__(self, order_in, order_out, num_features, clebsch_gordan=None):
        super().__init__()
        self.order_in, self.order_out, self.num_features = order_in, order_out, num_features
        self._paths = _paths(order_in, order_in, order_out, strict_upper=True)
        count = [0] * (order_out + 1)
        for L in range(min(order_in, order_out) + 1):
            count[L] += 1
        for _, _, L in self._paths:
            count[L] += 1
        for l1, l2, L in self._paths:
            self.register_parameter(f"mixcoeff_{l1}_{l2}_{L}", nn.Parameter(torch.empty(num_features).uniform_(-(3 / count[L]) ** 0.5, (3 / count[L]) ** 0.5)))
        for L in range(min(order_in, order_out) + 1):
            self.register_parameter(f"keepcoeff_{L}", nn.Parameter(torch.empty(num_features).uniform_(-(3 / count[L]) ** 0.5, (3 / count[L]) ** 0.5)))

    def keepcoeff(self, L):
        return getattr(self, f"keepcoeff_{L}")

    def mixcoeff(self, l1, l2, L):
        return getattr(self, f"mixcoeff_{l1}_{l2}_{L}")

    def _run(self, x, lib):
        F = self.num_features
        dev = x.device
        mix = (torch.stack([self.mixcoeff(*p) for p in self._paths]) if self._paths else torch.zeros(1, F, device=dev)).to(torch.float32).contiguous()
        keep = torch.stack([self.keepcoeff(L) for L in range(min(self.order_in, self.order_out) + 1)]).to(torch.float32).contiguous()
        y = torch.empty(x.shape[0], (self.order_out + 1) ** 2, F, dtype=torch.float32, device=dev)
        check(lib.nb200_phis_self_mixing(ptr(x), ptr(mix), ptr(keep), x.shape[0], F, self.order_in, self.order_out, ptr(y), current_stream()),
              "nb200_phis_self_mixing")
        return y

    @torch.no_grad()
    def forward(self, xs):
        _no_training(self)
        x, lead = _pack(xs[: self.order_in + 1])
        return _unpack(self._run(x, _lib.load()), self.order_out, lead)


class SphericalLinear(nn.Module):
    def __init__(self, order_in, num_in, order_out, num_out, clebsch_gordan=None, mix_orders=True, bias=True, zero_init=False):
        super().__init__()
        self.order_in, self.num_in, self.order_out, self.num_out = order_in, num_in, order_out, num_out
        self.bias, self.mix_orders = bias, mix_orders
        if mix_orders:
            self.mixing = SelfMixing(order_in, order_out, num_in, clebsch_gordan)
        elif order_in != order_out:
            raise ValueError("the order can only change if mixing is enabled")
        self.linear = nn.ModuleList([nn.Linear(num_in, num_out, bias=(bias and L == 0)) for L in range(order_out + 1)])
        for lin in self.linear:
            nn.init.zeros_(lin.weight) if zero_init else nn.init.orthogonal_(lin.weight)
        if bias:
            nn.init.zeros_(self.linear[0].bias)

    @torch.no_grad()
    def forward(self, xs):
        _no_training(self)
        lib = _lib.load()
        x, lead = _pack(xs[: self.order_in + 1])
        if self.mix_orders:
            x = self.mixing._run(x, lib)
        w_l = torch.stack([lin.weight.t() for lin in self.linear]).to(torch.float32).contiguous()  # [order_out+1][c_in][c_out]
        b = self.linear[0].bias.to(torch.float32).contiguous() if self.bias else None
        y = torch.empty(x.shape[0], (self.order_out + 1) ** 2, self.num_out, dtype=torch.float32, device=x.device)
        check(lib.nb200_phis_linear(ptr(x), ptr(w_l), ptr(b) if b is not None else None, x.shape[0], self.num_in, self.num_out, self.order_out, ptr(y),
                                    current_stream()), "nb200_phis_linear")
        return _unpack(y, self.order_out, lead)


# ====================================================================================================== the whole model (neural_network.py)
# Parameter holders with the reference's module tree and names (modules/{swish,embedding,spherical_embedding,residual_block,residual_stack,
# interaction_block,modular_block,energy_layer,exponential_bernstein_radial_basis_functions}.py).  The arithmetic is in csrc/phisnet_model.cu.
_SHELLS = [(1, 0), (2, 0), (2, 1), (3, 0), (3, 1), (3, 2), (4, 0), (4, 1), (4, 2), (4, 3), (5, 0), (5, 1), (5, 2), (6, 0), (6, 1)]
# ground states that differ from Madelung filling: Z -> {shell: electrons moved}
_CONFIG_EXCEPTIONS = {24: {(3, 2): 1, (4, 0): -1}, 29: {(3, 2): 1, (4, 0): -1}, 41: {(4, 2): 1, (5, 0): -1}, 42: {(4, 2): 1, (5, 0): -1},
                      44: {(4, 2): 1, (5, 0): -1}, 45: {(4, 2): 1, (5, 0): -1}, 46: {(4, 2): 2, (5, 0): -2}, 47: {(4, 2): 1, (5, 0): -1},
                      57: {(4, 3): -1, (5, 2): 1}, 58: {(4, 3): -1, (5, 2): 1}, 64: {(4, 3): -1, (5, 2): 1}, 78: {(5, 2): 1, (6, 0): -1},
                      79: {(5, 2): 1, (6, 0): -1}}


def electron_configurations(zmax: int = 87) -> torch.Tensor:
    """[zmax, 16] float32: Z / 86, then the fill fraction of the shells 1s 2s 2p 3s 3p 3d 4s 4p 4d 4f 5s 5p 5d 6s 6p (n-major order),
    filled in Madelung (n + l, n) order with the ground-state exceptions of the transition metals and lanthanides."""
    madelung = sorted(_SHELLS, key=lambda s: (s[0] + s[1], s[0]))
    rows = []
    for z in range(zmax):
        occ, left = {}, z
        for s in madelung:
            occ[s] = min(2 * (2 * s[1] + 1), left)
            left -= occ[s]
        for s, d in _CONFIG_EXCEPTIONS.get(z, {}).items():
            occ[s] += d
        rows.append([z / 86.0] + [occ[s] / (2 * (2 * s[1] + 1)) for s in _SHELLS])
    return torch.tensor(rows, dtype=torch.float64).to(torch.float32)


class Swish(nn.Module):
    def __init__(self, num_features, initial_alpha=1.0, initial_beta=1.702):
        super().__init__()
        self.num_features = num_features
        self.alpha = nn.Parameter(torch.full((num_features,), float(initial_alpha)))
        self.beta = nn.Parameter(torch.full((num_features,), float(initial_beta)))


class Embedding(nn.Module):
    def __init__(self, num_features, Zmax=87):
        super().__init__()
        self.num_features, self.Zmax = num_features, Zmax
        self.register_buffer("electron_config", electron_configurations(Zmax))
        self.element_embedding = nn.Parameter(torch.empty(Zmax, num_features).uniform_(-3 ** 0.5, 3 ** 0.5))
        self.config_linear = nn.Linear(16, num_features, bias=False)
        nn.init.orthogonal_(self.config_linear.weight)


class SphericalEmbedding(nn.Module):
    def __init__(self, order, num_features, Zmax=87):
        super().__init__()
        self.order, self.num_features, self.Zmax = order, num_features, Zmax
        self.embedding = Embedding(num_features, Zmax)


class ExponentialBernsteinRadialBasisFunctions(nn.Module):
    def __init__(self, num_basis_functions, cutoff, ini_alpha=0.5):
        super().__init__()
        import numpy as np
        k = num_basis_functions
        logfact = np.zeros(k)
        for i in range(2, k):
            logfact[i] = logfact[i - 1] + np.log(i)
        v = np.arange(k)
        n = (k - 1) - v
        self.num_basis_functions = k
        self.register_buffer("cutoff", torch.tensor(cutoff, dtype=torch.float64))
        self.register_buffer("logc", torch.tensor(logfact[-1] - logfact[v] - logfact[n], dtype=torch.float64))
        self.register_buffer("n", torch.tensor(n, dtype=torch.float64))
        self.register_buffer("v", torch.tensor(v, dtype=torch.float64))
        # softplus_inverse(ini_alpha) evaluated in float32 and stored in a float64 parameter, as the reference initialises it
        a = torch.tensor(float(ini_alpha))
        self._alpha = nn.Parameter((a + torch.log(-torch.expm1(-a))).to(torch.float64))


class ResidualBlock(nn.Module):
    def __init__(self, order, num_features, clebsch_gordan=None, mix_orders=True, activation="swish"):
        super().__init__()
        self.order, self.num_features, self.mix_orders = order, num_features, mix_orders
        self.activation_pre, self.activation_post = Swish(num_features), Swish(num_features)
        self.linear1 = SphericalLinear(order, num_features, order, num_features, None, mix_orders)
        self.linear2 = SphericalLinear(order, num_features, order, num_features, None, mix_orders, zero_init=True)


class ResidualStack(nn.Module):
    def __init__(self, num_blocks, order, num_features, clebsch_gordan=None, mix_orders=True, activation="swish"):
        super().__init__()
        self.num_blocks, self.order, self.num_features = num_blocks, order, num_features
        self.stack = nn.ModuleList([ResidualBlock(order, num_features, None, mix_orders, activation) for _ in range(num_blocks)])


class InteractionBlock(nn.Module):
    def __init__(self, order, num_features, num_basis_functions, num_residual_pre_vi, num_residual_pre_vj, num_residual_post_v,
                 clebsch_gordan=None, mix_orders=True, activation="swish"):
        super().__init__()
        self.order, self.num_features, self.num_basis_functions = order, num_features, num_basis_functions
        self.activation_i, self.activation_j, self.activation_v = Swish(num_features), Swish(num_features), Swish(num_features)
        self.angular_fn1 = SphericalLinear(order, 1, order, num_features, None, mix_orders=False)
        self.angular_fn2 = SphericalLinear(order, 1, order, num_features, None, mix_orders=False)
        self.radial_fn = nn.ModuleList([nn.Linear(num_basis_functions, num_features, bias=False) for _ in range(order + 1)])
        for lin in self.radial_fn:
            nn.init.orthogonal_(lin.weight)
        self.mixing = PairMixing(order, order, order, num_basis_functions, num_features)
        self.linear_i = SphericalLinear(order, num_features, order, num_features, None, mix_orders)
        self.linear_j = SphericalLinear(order, num_features, order, num_features, None, mix_orders)
        self.linear_v = SphericalLinear(order, num_features, order, num_features, None, mix_orders)
        self.residual_pre_vi = ResidualStack(num_residual_pre_vi, order, num_features, None, mix_orders, activation)
        self.residual_pre_vj = ResidualStack(num_residual_pre_vj, order, num_features, None, mix_orders, activation)
        self.residual_post_v = ResidualStack(num_residual_post_v, order, num_features, None, mix_orders, activation)


class ModularBlock(nn.Module):
    def __init__(self, order, num_features, num_basis_functions, num_residual_pre_x, num_residual_post_x, num_residual_pre_vi,
                 num_residual_pre_vj, num_residual_post_v, num_residual_output, clebsch_gordan=None, mix_orders=True, activation="swish"):
        super().__init__()
        self.order, self.num_features, self.num_basis_functions = order, num_features, num_basis_functions
        self.interaction = InteractionBlock(order, num_features, num_basis_functions, num_residual_pre_vi, num_residual_pre_vj, num_residual_post_v,
                                            None, mix_orders, activation)
        self.residual_pre_x = ResidualStack(num_residual_pre_x, order, num_features, None, mix_orders, activation)
        self.residual_post_x = ResidualStack(num_residual_post_x, order, num_features, None, mix_orders, activation)
        self.residual_out = ResidualStack(num_residual_output, order, num_features, None, mix_orders, activation)


class EnergyLayer(nn.Module):
    """Parameter holder only: energy prediction is not built (the nablaDFT configs train with energy_weight = forces_weight = 0)."""

    def __init__(self, num_in, num_out, activation, zero_init=False):
        super().__init__()
        self.num_in, self.num_out, self.zero_init = num_in, num_out, zero_init
        self.linear_diagonal = nn.Linear(num_in, num_out)
        self.linear_offdiagonal = nn.Linear(num_in, num_out)
        self.linear_out = nn.Linear(2 * num_out, 1)
        self.activation = activation


def compute_matrix_irreps(orbitals_i, orbitals_j, irreps, number_L):
    """neural_network.py:610-621: one output column per new key (z_i, z_j, n_i, n_j, L), numbered per L in first-seen order."""
    for n_i, (z_i, l_i) in enumerate(orbitals_i):
        for n_j, (z_j, l_j) in enumerate(orbitals_j):
            for L in range(abs(l_i - l_j), l_i + l_j + 1):
                key = (z_i, z_j, n_i, n_j, L)
                if key not in irreps:
                    irreps[key] = number_L[L]
                    number_L[L] += 1
    return irreps, number_L


def irreps_tables(max_orbitals):
    """(irreps_ii, width_ii, irreps_ij, width_ij) exactly as NeuralNetwork.__init__ builds them (neural_network.py:368-442)."""
    order_max = max(l for orbs in max_orbitals for _, l in orbs)
    ii, nl = {}, [0] * (2 * order_max + 1)
    for o in max_orbitals:
        ii, nl = compute_matrix_irreps(o, o, ii, nl)
    w_ii = max(nl)
    ij, nl = {}, [0] * (2 * order_max + 1)
    for a, oa in enumerate(max_orbitals):
        for b, ob in enumerate(max_orbitals):
            if a != b:
                ij, nl = compute_matrix_irreps(oa, ob, ij, nl)
    return ii, w_ii, ij, max(nl)


def assembly_tables(max_orbitals, irreps_ii, irreps_ij):
    """Host tables of nb200_phis_assemble: per element its orbital rows and shells, per (block kind, element pair) the list of irreps the
    block uses -- (output column, L) in the reference's (n_i, n_j, L) order -- and the first entry of every shell pair."""
    import numpy as np
    elem_orbs = {}
    for orbs in max_orbitals:
        elem_orbs.setdefault(orbs[0][0], tuple(orbs))
    elems = sorted(elem_orbs)
    ne = len(elems)
    row_orb, row_m = np.zeros((ne, 32), np.int32), np.zeros((ne, 32), np.int32)
    orb_l, n_rows = np.zeros((ne, 16), np.int32), np.zeros(ne, np.int32)
    for e, z in enumerate(elems):
        r = 0
        for s, (_, l) in enumerate(elem_orbs[z]):
            orb_l[e, s] = l
            for m in range(2 * l + 1):
                row_orb[e, r], row_m[e, r] = s, m
                r += 1
        n_rows[e] = r
    ent_range = np.full((2, ne, ne, 2), 0, np.int32)
    op_base = np.zeros((2, ne, ne, 16, 16), np.int32)
    cols, Ls, missing = [], [], []
    for kind, table in ((0, irreps_ii), (1, irreps_ij)):
        for a, za in enumerate(elems):
            for b, zb in enumerate(elems):
                if kind == 0 and a != b:
                    continue
                k0 = len(cols)
                for si, (_, li) in enumerate(elem_orbs[za]):
                    for sj, (_, lj) in enumerate(elem_orbs[zb]):
                        op_base[kind, a, b, si, sj] = len(cols)
                        for L in range(abs(li - lj), li + lj + 1):
                            key = (za, zb, si, sj, L)
                            if key not in table:
                                missing.append((kind, za, zb))
                            cols.append(table.get(key, 0))
                            Ls.append(L)
                ent_range[kind, a, b] = (k0, len(cols))
    max_ent = int((ent_range[..., 1] - ent_range[..., 0]).max())
    return dict(elems=elems, row_orb=row_orb, row_m=row_m, orb_l=orb_l, n_rows=n_rows, ent_range=ent_range, op_base=op_base,
                ent_col=np.asarray(cols, np.int32), ent_L=np.asarray(Ls, np.int32), max_ent=max_ent, missing=set(missing))


class NeuralNetwork(nn.Module):
    """Mirror of `nablaDFT.phisnet.nn.NeuralNetwork` (neural_network.py:31-995): same constructor, module tree, parameter names, flags and
    `forward(atoms_batch)` contract (dict of full_hamiltonian, core_hamiltonian, overlap_matrix [1, sum Norb, sum Norb] and zero energy /
    forces / orbital_energies / orbital_coefficients, fp32).  `forward(atoms_batch, packed=True)` returns per-molecule matrices instead of
    the block diagonal.  The forward runs in csrc/phisnet_model.cu + phisnet.cu + the wgmma GEMM; inference only, CUDA only.

    Supported: order 4, exp-Bernstein radial basis, swish, orbitals up to d (2 * l_max <= order), num_features in {32, 64, 96, 128},
    num_basis_functions % 32 == 0.  The reference's CG-table buffers (`*clebsch_gordan.cg_*`) are compiled into the kernels instead.
    """

    def __init__(self, max_orbitals=None, order=None, num_features=None, num_basis_functions=None, num_modules=None, num_residual_pre_x=None,
                 num_residual_post_x=None, num_residual_pre_vi=None, num_residual_pre_vj=None, num_residual_post_v=None, num_residual_output=None,
                 num_residual_pc=None, num_residual_pn=None, num_residual_ii=None, num_residual_ij=None, num_residual_full_ii=None,
                 num_residual_full_ij=None, num_residual_core_ii=None, num_residual_core_ij=None, num_residual_over_ij=None, basis_functions=None,
                 cutoff=None, activation=None, load_from=None, Zmax=87, num_energy_features=64, fallback_args=None):
        super().__init__()
        self.calculate_full_hamiltonian = True
        self.calculate_core_hamiltonian = True
        self.calculate_overlap_matrix = True
        self.calculate_energy = False
        self.predict_energy = False
        self.calculate_forces = False
        self.create_graph = True
        saved_state = None
        if load_from is not None:  # neural_network.py:98-142: hyperparameters come from the file
            from argparse import Namespace
            saved_state = torch.load(load_from, map_location="cpu", weights_only=False)
            args = saved_state["args"] if "args" in saved_state else Namespace(**saved_state)
            max_orbitals = args.max_orbitals if max_orbitals is None else max_orbitals
            (order, num_features, num_basis_functions, num_modules, num_residual_pre_x, num_residual_post_x, num_residual_pre_vi,
             num_residual_pre_vj, num_residual_post_v, num_residual_output, num_residual_pc, num_residual_pn, num_residual_ii, num_residual_ij,
             num_residual_full_ii, num_residual_full_ij, num_residual_core_ii, num_residual_core_ij, num_residual_over_ij, basis_functions,
             cutoff, activation) = (getattr(args, k) for k in (
                "order", "num_features", "num_basis_functions", "num_modules", "num_residual_pre_x", "num_residual_post_x", "num_residual_pre_vi",
                "num_residual_pre_vj", "num_residual_post_v", "num_residual_output", "num_residual_pc", "num_residual_pn", "num_residual_ii",
                "num_residual_ij", "num_residual_full_ii", "num_residual_full_ij", "num_residual_core_ii", "num_residual_core_ij",
                "num_residual_over_ij", "basis_functions", "cutoff", "activation"))
        self.max_orbitals = tuple(tuple((int(z), int(l)) for z, l in orbs) for orbs in max_orbitals)
        self.order, self.num_features, self.num_basis_functions, self.num_modules = order, num_features, num_basis_functions, num_modules
        self.num_residual_pre_x, self.num_residual_post_x = num_residual_pre_x, num_residual_post_x
        self.num_residual_pre_vi, self.num_residual_pre_vj, self.num_residual_post_v = num_residual_pre_vi, num_residual_pre_vj, num_residual_post_v
        self.num_residual_output, self.num_residual_pc, self.num_residual_pn = num_residual_output, num_residual_pc, num_residual_pn
        self.num_residual_ii, self.num_residual_ij = num_residual_ii, num_residual_ij
        self.num_residual_full_ii, self.num_residual_full_ij = num_residual_full_ii, num_residual_full_ij
        self.num_residual_core_ii, self.num_residual_core_ij, self.num_residual_over_ij = num_residual_core_ii, num_residual_core_ij, num_residual_over_ij
        self.basis_functions, self.cutoff, self.activation, self.Zmax = basis_functions, cutoff, activation, Zmax
        self.num_energy_features = num_energy_features
        order_max = max(l for orbs in self.max_orbitals for _, l in orbs)
        if order != 4 or basis_functions != "exp-bernstein" or activation != "swish" or order_max != 2:
            raise NotImplementedError("nabladft_b200.phisnet.NeuralNetwork is built for order 4, exp-bernstein, swish and orbitals up to d (l_max = 2)")
        if num_features not in (32, 64, 96, 128) or num_basis_functions % 32:
            raise NotImplementedError("num_features must be 32, 64, 96 or 128 and num_basis_functions a multiple of 32")
        F, K = num_features, num_basis_functions
        stack = lambda n: ResidualStack(n, order, F)
        self.embedding = SphericalEmbedding(order, F, Zmax)
        self.radial_basis_functions = ExponentialBernsteinRadialBasisFunctions(K, cutoff)
        self.module = nn.ModuleList([ModularBlock(order, F, K, num_residual_pre_x, num_residual_post_x, num_residual_pre_vi, num_residual_pre_vj,
                                                  num_residual_post_v, num_residual_output) for _ in range(num_modules)])
        self.angular_fn = SphericalLinear(order, 1, order, F, None, mix_orders=False)
        self.mix_s = PairMixing(order, order, order, K, F)
        self.mix_ij = PairMixing(order, order, order, K, F)
        self.radial_ii = nn.ModuleList([nn.Linear(K, F, bias=False) for _ in range(order + 1)])
        self.radial_ij = nn.ModuleList([nn.Linear(K, F, bias=False) for _ in range(order + 1)])
        for lin in list(self.radial_ii) + list(self.radial_ij):
            nn.init.orthogonal_(lin.weight)
        for name in ("pc", "pn", "ii", "ij", "full_ii", "full_ij", "core_ii", "core_ij", "over_ij"):
            self.add_module(f"residual_{name}", stack(getattr(self, f"num_residual_{name}")))
        for name in ("full_ii", "full_ij", "core_ii", "core_ij", "over_ij"):
            self.add_module(f"activation_{name}", Swish(F))
        self.activation_energy = Swish(num_energy_features)
        self.irreps_ii, w_ii, self.irreps_ij, w_ij = irreps_tables(self.max_orbitals)
        for name, width in (("full_ii", w_ii), ("core_ii", w_ii), ("over_ii", w_ii), ("full_ij", w_ij), ("core_ij", w_ij), ("over_ij", w_ij)):
            self.add_module(f"output_{name}", SphericalLinear(order, F, 2 * order_max, width, None, zero_init=True))
        for lin in self.output_over_ii.linear:
            lin.weight.requires_grad = False
        self._asm = assembly_tables(self.max_orbitals, self.irreps_ii, self.irreps_ij)
        if saved_state is not None:
            sd = saved_state.get("model_state_dict", saved_state.get("state_dict"))
            self.load_state_dict(sd, strict=False)
        self.energy_predictor = EnergyLayer(F, num_energy_features, zero_init=False, activation=self.activation_energy)
        self.profile = None  # dict -> per-stage CUDA-event times are appended (bench_phisnet.py --profile)
        self._cache_key, self._w, self._dev_tables = None, None, None

    def load_state_dict(self, state_dict, strict=True, assign=False):
        """The reference's CG-table buffers have no counterpart here (the table is compiled into the kernels): they are skipped."""
        sd = {k: v for k, v in state_dict.items() if "clebsch_gordan.cg_" not in k}
        return super().load_state_dict(sd, strict=strict, assign=assign)

    # ------------------------------------------------------------------ weight export (cached per parameter version and device)
    @torch.no_grad()
    def _export(self, dev):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters()) + (str(dev),)
        if key == self._cache_key:
            return self._w
        c = lambda t: t.detach().to(dev, torch.float32).contiguous()

        def sl(m):  # SphericalLinear -> (mixcoeff, keepcoeff, W_l [5][in][out], bias)
            mix = keep = None
            if m.mix_orders:
                mix = c(torch.stack([m.mixing.mixcoeff(*p) for p in m.mixing._paths]))
                keep = c(torch.stack([m.mixing.keepcoeff(L) for L in range(min(m.order_in, m.order_out) + 1)]))
            return dict(mix=mix, keep=keep, W=c(torch.stack([lin.weight.t() for lin in m.linear])), b=c(m.linear[0].bias) if m.bias else None)

        sw = lambda a: (c(a.alpha), c(a.beta))
        rs = lambda s: [dict(pre=sw(b.activation_pre), post=sw(b.activation_post), l1=sl(b.linear1), l2=sl(b.linear2)) for b in s.stack]
        ang = lambda m: (c(torch.stack([lin.weight[:, 0] for lin in m.linear])), c(m.linear[0].bias))
        mixw = lambda pm: torch.cat([pm.coeff(*p).weight for p in pm._paths], dim=0)
        w = {}
        e = self.embedding.embedding
        w["emb"] = c(e.element_embedding.double() + e.electron_config.double() @ e.config_linear.weight.double().t())
        w["alpha"] = float(torch.nn.functional.softplus(self.radial_basis_functions._alpha.double()))
        w["logc"] = self.radial_basis_functions.logc.detach().to(dev, torch.float64).contiguous()  # the edge basis sums its exponent in double
        w["mods"] = []
        for mb in self.module:
            it = mb.interaction
            w["mods"].append(dict(pre_x=rs(mb.residual_pre_x), post_x=rs(mb.residual_post_x), out=rs(mb.residual_out), pre_vi=rs(it.residual_pre_vi),
                                  pre_vj=rs(it.residual_pre_vj), post_v=rs(it.residual_post_v), act_i=sw(it.activation_i), act_j=sw(it.activation_j),
                                  act_v=sw(it.activation_v), lin_i=sl(it.linear_i), lin_j=sl(it.linear_j), lin_v=sl(it.linear_v),
                                  ang1=ang(it.angular_fn1), ang2=ang(it.angular_fn2),
                                  coeff=c(torch.cat([mixw(it.mixing)] + [lin.weight for lin in it.radial_fn], dim=0))))
        w["coeff_s"] = c(mixw(self.mix_s))
        w["coeff_p"] = c(torch.cat([mixw(self.mix_ij)] + [lin.weight for lin in self.radial_ii] + [lin.weight for lin in self.radial_ij], dim=0))
        w["ang"] = ang(self.angular_fn)
        for name in ("pc", "pn", "ii", "ij", "full_ii", "full_ij", "core_ii", "core_ij", "over_ij"):
            w["res_" + name] = rs(getattr(self, "residual_" + name))
        for name in ("full_ii", "full_ij", "core_ii", "core_ij", "over_ij"):
            w["act_" + name] = sw(getattr(self, "activation_" + name))
        for name in ("full_ii", "full_ij", "core_ii", "core_ij", "over_ii", "over_ij"):
            m = getattr(self, "output_" + name)
            w["out_" + name] = dict(mix=c(torch.stack([m.mixing.mixcoeff(*p) for p in m.mixing._paths])),
                                    keep=c(torch.stack([m.mixing.keepcoeff(L) for L in range(5)])),
                                    W=c(torch.stack([lin.weight for lin in m.linear])), b=c(m.linear[0].bias), n=m.num_out)
        self._w, self._cache_key = w, key
        return w

    def _tables(self, dev):
        if self._dev_tables is None or self._dev_tables[0] != str(dev):
            a = self._asm
            el_of_z = torch.full((max(max(a["elems"]) + 1, self.Zmax),), -1, dtype=torch.int32)
            for i, z in enumerate(a["elems"]):
                el_of_z[z] = i
            t = {k: torch.from_numpy(a[k].reshape(-1)).to(dev) for k in ("row_orb", "row_m", "orb_l", "n_rows", "ent_range", "op_base", "ent_col", "ent_L")}
            t["el_of_z"] = el_of_z.to(dev)
            t["norb_of_el"] = torch.from_numpy(a["n_rows"].astype("int64")).to(dev)
            self._dev_tables = (str(dev), t)
        return self._dev_tables[1]

    # ------------------------------------------------------------------ forward
    def forward(self, atoms_batch, packed: bool = False):
        if self.predict_energy or self.calculate_forces:
            raise NotImplementedError("nabladft_b200.phisnet.NeuralNetwork predicts matrices only: energy / forces prediction is not built")
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("PhiSNet training through the CUDA path is not built (inference only); call .eval() or torch.no_grad()")
        with torch.no_grad():
            return self._forward(atoms_batch, packed)

    def _forward(self, batch, packed):
        R = batch["positions"]
        if not R.is_cuda:
            raise NablaB200Error("nabladft_b200.phisnet.NeuralNetwork runs on CUDA only (no CPU fallback)")
        dev, F, K = R.device, self.num_features, self.num_basis_functions
        lib = _lib.load()
        s = current_stream
        w, tb = self._export(dev), self._tables(dev)
        E = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        prof = self.profile

        def stage(name):
            if prof is not None:
                ev = torch.cuda.Event(enable_timing=True)
                ev.record()
                prof.setdefault("_marks", []).append((name, ev))

        stage("graph")
        Z = batch["atomic_numbers"].reshape(-1).to(device=dev, dtype=torch.int64)
        sizes = torch.as_tensor(batch["molecule_size"]).reshape(-1).to(torch.int64).cpu()
        N, n_mol = Z.numel(), sizes.numel()
        if int(sizes.sum()) != N or R.shape[0] != N:
            raise ValueError("molecule_size, positions and atomic_numbers disagree")
        if int(Z.max()) >= tb["el_of_z"].numel() or bool((tb["el_of_z"][Z] < 0).any()):
            raise ValueError("an atom's element is not in max_orbitals: its orbitals and output irreps are undefined")
        orbitals = batch.get("orbitals")
        if orbitals is not None:  # the layout follows each atom's element in max_orbitals; a batch that says otherwise is refused
            table = {o[0][0]: o for o in self.max_orbitals}
            if len(orbitals) != N or any(tuple(tuple(int(v) for v in t) for t in o) != table[z] for o, z in zip(orbitals, Z.cpu().tolist())):
                raise ValueError("atoms_batch['orbitals'] disagrees with max_orbitals: every atom's orbitals must be those of its element")
        if self._asm["missing"]:
            pairs = {(a, b) for _, a, b in self._asm["missing"]}
            zs = set(Z.unique().tolist())
            if any(a in zs and b in zs for a, b in pairs):
                raise ValueError("max_orbitals lacks an element pair present in this batch (the reference would fail the irreps lookup)")
        P = int((sizes * (sizes - 1)).sum())
        pos = R.detach().to(torch.float32).contiguous()
        mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32)
        mol_ptr[1:] = torch.cumsum(sizes, 0)
        mol_ptr = mol_ptr.to(dev)
        I = lambda n: torch.empty(n, dtype=torch.int32, device=dev)
        row_ptr, col, rev, tgt, geom = I(N + 1), I(max(P, 1)), I(max(P, 1)), I(max(P, 1)), E(max(P, 1), 4)
        status = torch.zeros(4, dtype=torch.int32, device=dev)
        check(lib.nb200_neighbor_build(ptr(pos), ptr(mol_ptr), n_mol, N, 10000.0, 2 ** 31 - 1, max(P, 1), ptr(row_ptr), ptr(col), ptr(rev), ptr(geom),
                                       ptr(I(N)), ptr(status), s()), "nb200_neighbor_build")
        st = status.cpu()  # the host-side pair count P sizes the buffers and the assembly grid: the device build must agree with it
        if int(st[1]) != 0 or int(st[0]) != P:
            raise NablaB200Error(f"pair build failed (status {st.tolist()}, expected {P} pairs): a molecule over 1024 atoms, non-finite positions "
                                 "or atoms more than 1e4 bohr apart")
        check(lib.nb200_qh_expand_rows(ptr(row_ptr), N, ptr(tgt), s()), "nb200_qh_expand_rows")
        # distances, unit vectors, exp-Bernstein RBF with PhiSNet's cutoff function and the l <= 4 spherical harmonics: the closed forms of
        # the QHNet edge basis coincide term by term with PhiSNet's (m = -l..l, no 1/sqrt(4 pi)), so that kernel serves both (sign +1: r_j - r_i)
        rbf, sh = E(max(P, 1), K), E(max(P, 1), 25)
        check(lib.nb200_qh_edge_basis(ptr(geom), ptr(status), max(P, 1), w["alpha"], float(self.cutoff), 1.0, ptr(w["logc"]), K, ptr(rbf), ptr(sh), s()),
              "nb200_qh_edge_basis")

        def dense(x, W):  # x [rows, K] . W^T, W [n, K]
            y = E(x.shape[0], W.shape[0])
            check(lib.nb200_dense(x.shape[0], W.shape[0], K, ptr(x), K, ptr(W), K, 0, ptr(y), W.shape[0], 0, None, None, 0, s()), "nb200_dense")
            return y

        def mix(x, p, act=None, n_feat=F):  # SelfMixing(4, 4) of swish(x) on component 0
            y = E(x.shape[0], 25, n_feat)
            check(lib.nb200_phis_swish_self_mixing(ptr(x), ptr(act[0]) if act else None, ptr(act[1]) if act else None, ptr(p["mix"]), ptr(p["keep"]),
                                                   x.shape[0], n_feat, ptr(y), s()), "nb200_phis_swish_self_mixing")
            return y

        def linear(x, p, act=None, into=None):  # SphericalLinear(4 -> 4) of swish(x); into: y += result (the residual add)
            h = mix(x, p, act)
            y = E(x.shape[0], 25, F) if into is None else into
            check(lib.nb200_phis_linear_ex(ptr(h), ptr(p["W"]), ptr(p["b"]), x.shape[0], F, F, 4, 0 if into is None else 1, ptr(y), s()),
                  "nb200_phis_linear_ex")
            return y

        def residual(x, blocks, inplace=False):  # ResidualStack: x + linear2(swish(linear1(swish(x))))
            if not inplace and blocks:
                x = x.clone()
            for b in blocks:
                linear(linear(x, b["l1"], b["pre"]), b["l2"], b["post"], into=x)
            return x

        stage("embedding")
        xs = torch.zeros(N, 25, F, dtype=torch.float32, device=dev)
        xs[:, 0, :] = w["emb"].index_select(0, Z)
        X_over_ii = X_over_ij = None
        if self.calculate_overlap_matrix:
            stage("overlap_branch")
            X_over_ii = mix(xs, w["out_over_ii"])
            sij = E(max(P, 1), 25, F)
            check(lib.nb200_phis_overlap_pairs(ptr(xs), ptr(sh), ptr(dense(rbf, w["coeff_s"])), ptr(w["ang"][0]), ptr(row_ptr), ptr(col), N, F, ptr(sij),
                                               s()), "nb200_phis_overlap_pairs")
            X_over_ij = mix(residual(sij, w["res_over_ij"], inplace=True), w["out_over_ij"], w["act_over_ij"])
            del sij
        fs = None
        for li, m in enumerate(w["mods"]):
            stage(f"module{li}")
            xs = residual(xs, m["pre_x"], inplace=True)
            yi = linear(residual(xs, m["pre_vi"]), m["lin_i"], m["act_i"])
            yj = linear(residual(xs, m["pre_vj"]), m["lin_j"], m["act_j"])
            coeff = dense(rbf, m["coeff"])
            v = E(N, 25, F)
            check(lib.nb200_phis_interaction(ptr(yi), ptr(yj), ptr(sh), ptr(coeff), ptr(m["ang1"][0]), ptr(m["ang1"][1]), ptr(m["ang2"][0]),
                                             ptr(m["ang2"][1]), ptr(row_ptr), ptr(col), N, F, ptr(v), s()), "nb200_phis_interaction")
            del coeff, yi, yj
            v = residual(v, m["post_v"], inplace=True)
            linear(v, m["lin_v"], m["act_v"], into=xs)
            xs = residual(xs, m["post_x"], inplace=True)
            ys = residual(xs, m["out"])
            if fs is None:
                fs = ys if m["out"] else ys.clone()
            else:
                check(lib.nb200_axpy(ptr(fs), ptr(ys), fs.numel(), s()), "nb200_axpy")
        stage("pair_features")
        fpc = residual(fs, w["res_pc"])
        fpn = residual(fs, w["res_pn"], inplace=True)
        fii, fij = E(N, 25, F), E(max(P, 1), 25, F)
        check(lib.nb200_phis_pair_features(ptr(fpc), ptr(fpn), ptr(dense(rbf, w["coeff_p"])), ptr(row_ptr), ptr(col), N, F, ptr(fii), ptr(fij), s()),
              "nb200_phis_pair_features")
        del fpc, fpn
        stage("heads")
        fii = residual(fii, w["res_ii"], inplace=True)
        fij = residual(fij, w["res_ij"], inplace=True)
        X = {}
        for head, flag in (("full", self.calculate_full_hamiltonian), ("core", self.calculate_core_hamiltonian)):
            if flag:
                X[head] = (mix(residual(fii, w[f"res_{head}_ii"]), w[f"out_{head}_ii"], w[f"act_{head}_ii"]),
                           mix(residual(fij, w[f"res_{head}_ij"]), w[f"out_{head}_ij"], w[f"act_{head}_ij"]))
        if self.calculate_overlap_matrix:
            X["over"] = (X_over_ii, X_over_ij)
        del fii, fij

        stage("assembly")
        el = tb["el_of_z"][Z]
        norb_atom = tb["norb_of_el"][el.long()]
        atom_mol = torch.repeat_interleave(torch.arange(n_mol, device=dev), sizes.to(dev))
        csum = torch.cumsum(norb_atom, 0)
        first = mol_ptr[:-1].long()
        atom_off = (csum - norb_atom - (csum - norb_atom)[first][atom_mol]).to(torch.int32)
        mol_norb = torch.zeros(n_mol, dtype=torch.int64, device=dev).index_add_(0, atom_mol, norb_atom)
        mol_off = torch.zeros(n_mol + 1, dtype=torch.int64, device=dev)
        mol_off[1:] = torch.cumsum(mol_norb * mol_norb, 0)
        norbs = mol_norb.cpu().tolist()
        offs = mol_off.cpu().tolist()
        atom_mol32, mol_norb32 = atom_mol.to(torch.int32), mol_norb.to(torch.int32)
        mats = {}
        for head in ("full", "core", "over"):
            if head not in X:
                mats[head] = [torch.eye(n, dtype=torch.float32, device=dev) for n in norbs]
                continue
            Xd, Xo = X[head]
            od, oo = w[f"out_{head}_ii"], w[f"out_{head}_ij"]
            M = E(max(offs[-1], 1))
            check(lib.nb200_phis_assemble(ptr(Xd), ptr(Xo), ptr(od["W"]), ptr(od["b"]), od["n"], ptr(oo["W"]), ptr(oo["b"]), oo["n"], F, ptr(el),
                                          ptr(tb["row_orb"]), ptr(tb["row_m"]), ptr(tb["orb_l"]), ptr(tb["n_rows"]), ptr(tb["ent_range"]),
                                          ptr(tb["op_base"]), ptr(tb["ent_col"]), ptr(tb["ent_L"]), len(self._asm["elems"]), self._asm["max_ent"],
                                          ptr(tgt), ptr(col), ptr(rev), N, P, ptr(atom_mol32), ptr(atom_off), ptr(mol_off), ptr(mol_norb32),
                                          1 if head == "over" else 0, ptr(M), s()), "nb200_phis_assemble")
            mats[head] = [M[offs[i]:offs[i + 1]].view(norbs[i], norbs[i]) for i in range(n_mol)]
        stage("end")
        if packed:
            return {"full_hamiltonian": mats["full"], "core_hamiltonian": mats["core"], "overlap_matrix": mats["over"]}
        dense_of = lambda ms: torch.block_diag(*ms).unsqueeze(0)
        full, core, over = dense_of(mats["full"]), dense_of(mats["core"]), dense_of(mats["over"])
        return {"full_hamiltonian": full, "core_hamiltonian": core, "overlap_matrix": over,
                "energy": torch.zeros(1, 1, dtype=torch.float32, device=dev), "forces": torch.zeros(N, 3, dtype=torch.float32, device=dev),
                "orbital_energies": torch.zeros(1, full.shape[-1], dtype=torch.float32, device=dev), "orbital_coefficients": torch.zeros_like(full)}
