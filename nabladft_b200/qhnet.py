"""H100-native drop-in for `nablaDFT.qhnet.QHNet` (config/model/qhnet.yaml): Hamiltonian prediction.

Same constructor signature, `forward(data, keep_blocks=False)` contract and state_dict names/shapes
as the reference class (`nablaDFT/qhnet/qhnet.py:24-342`, `layers.py`), so
`config/model/qhnet-b200.yaml` only swaps the `_target_`.  The arithmetic runs in libnabla_b200.so:
neighbour build, exp-Bernstein/spherical-harmonic edge basis, NormGate pieces, invariant edge
features, the three Clebsch-Gordan tensor products (coefficients unrolled as literals), e3nn
Linear / MLP layers on the wgmma 3xTF32 GEMM, Expansion and the block assembly (which replaces the
reference's O(n^2 P) Python loop with one kernel).  PyTorch here only allocates buffers and
sequences the calls.  Inference only (no autograd through the kernels).

Shipped configuration only: sh_lmax=4, hidden_size=128, bottle_hidden_size=32, radius_embed_dim=32.
"""
import ctypes
import os
import math
from typing import Dict

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import NablaB200Error, check, current_stream, ptr

LM = 25
ACT_SILU, ACT_SSP, ACT_SSP_N = 0, 1, 2


# ------------------------------------------------------------------ parameter holders (reference names)
class _E3Linear(nn.Module):
    """e3nn o3.Linear between 5-block irreps (l = 0..4): flat `weight` of 5 [c_in, c_out] blocks, `bias` on 0e."""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.c_in, self.c_out = c_in, c_out
        self.weight = nn.Parameter(torch.randn(5 * c_in * c_out))
        self.bias = nn.Parameter(torch.zeros(c_out))


class _FCN(nn.Module):
    """e3nn FullyConnectedNet([a, b, c], ssp): layer0.weight [a,b], layer1.weight [b,c]."""

    class _L(nn.Module):
        def __init__(self, a, b):
            super().__init__()
            self.weight = nn.Parameter(torch.randn(a, b))

    def __init__(self, a, b, c):
        super().__init__()
        self.layer0, self.layer1 = _FCN._L(a, b), _FCN._L(b, c)


class _NormGate(nn.Module):
    def __init__(self, n=640):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(n, n), nn.SiLU(), nn.Linear(n, n))


class _Conv(nn.Module):
    def __init__(self, first: bool, hs=128, red=32):
        super().__init__()
        nw = 5 * hs if first else 42 * hs
        self.fc_node = _FCN(red, 32, nw)
        self.layer_l0 = _FCN(2 * hs if first else 6 * hs, 32, nw)
        self.linear_out = _E3Linear(hs, hs)
        if not first:
            self.norm_gate = _NormGate(5 * hs)
            self.linear_node = _E3Linear(hs, hs)
            self.linear_node_pre = _E3Linear(hs, hs)


class _ConvNet(nn.Module):
    def __init__(self, first):
        super().__init__()
        self.conv = _Conv(first)


class _SelfNet(nn.Module):
    def __init__(self, hs=128):
        super().__init__()
        self.linear_node_1, self.linear_node_2, self.linear_node_3 = _E3Linear(hs, hs), _E3Linear(hs, hs), _E3Linear(hs, hs)

        class _TP(nn.Module):
            def __init__(self):
                super().__init__()
                self.weight = nn.Parameter(torch.randn(65 * hs))

        self.tp = _TP()
        self.norm_gate, self.norm_gate_1, self.norm_gate_2 = _NormGate(5 * hs), _NormGate(5 * hs), _NormGate(5 * hs)


class _PairNet(nn.Module):
    def __init__(self, hs=128, red=32):
        super().__init__()
        self.linear_node_pair_n, self.linear_node_pair_inner = _E3Linear(hs, hs), _E3Linear(hs, hs)
        self.fc_node_pair = _FCN(red, hs, 65 * hs)
        self.linear_node_pair = _E3Linear(hs, hs)
        self.norm_gate, self.norm_gate_pre = _NormGate(5 * hs), _NormGate(5 * hs)
        self.fc = nn.Sequential(nn.Linear(6 * hs, hs), nn.SiLU(), nn.Linear(hs, 65 * hs))


class _Expansion(nn.Module):
    def __init__(self, n_path, n_bias):
        super().__init__()
        self.num_path_weight, self.num_bias = n_path, n_bias
        self.weights = nn.Parameter(torch.rand(n_path + n_bias))  # present in the reference, unused by forward


class _ExpBernstein(nn.Module):
    def __init__(self, k, cutoff, ini_alpha=0.5):
        super().__init__()
        logfact = np.zeros(k)
        for i in range(2, k):
            logfact[i] = logfact[i - 1] + np.log(i)
        v = np.arange(k)
        n = (k - 1) - v
        self.register_buffer("cutoff", torch.tensor(cutoff, dtype=torch.float32))
        self.register_buffer("logc", torch.tensor(logfact[-1] - logfact[v] - logfact[n], dtype=torch.float32))
        self.register_buffer("n", torch.tensor(n, dtype=torch.float32))
        self.register_buffer("v", torch.tensor(v, dtype=torch.float32))
        a = torch.tensor(float(ini_alpha))
        self._alpha = nn.Parameter(a + torch.log(-torch.expm1(-a)))


def _expansion_tables(n_shell=(5, 4, 3), lin_max=4):
    """Instruction list of Expansion.get_expansion_path (layers.py:664-671) and w3j(l1,l2,l_in)/32, padded to [19][5][5][9]."""
    # real Wigner-3j via the same Racah/real-basis recipe as e3nn (no dependency on the test oracle at run time)
    ins, cg = [], []
    woff = boff = 0
    for lin in range(lin_max + 1):
        for l1 in range(3):
            for l2 in range(3):
                if abs(l1 - l2) <= lin <= l1 + l2:
                    n1, n2 = n_shell[l1], n_shell[l2]
                    ins.append((lin, l1, l2, woff, boff if lin == 0 else 0))
                    woff += 32 * n1 * n2
                    if lin == 0:
                        boff += n1 * n2
                    C = _w3j(l1, l2, lin) / 32.0
                    pad = np.zeros((5, 5, 9), dtype=np.float32)
                    pad[: 2 * l1 + 1, : 2 * l2 + 1, : 2 * lin + 1] = C
                    cg.append(pad)
    return np.asarray(ins, dtype=np.int32), np.stack(cg).astype(np.float32), woff, boff


def _su2_cg(j1, m1, j2, m2, j3, m3):
    if m3 != m1 + m2:
        return 0.0
    f = math.factorial
    vmin = int(max(-j1 + j2 + m3, -j1 + m1, 0))
    vmax = int(min(j2 + j3 + m1, j3 - j1 + j2, j3 + m3))
    C = math.sqrt((2.0 * j3 + 1.0) * f(j3 + j1 - j2) * f(j3 - j1 + j2) * f(j1 + j2 - j3) * f(j3 + m3) * f(j3 - m3)
                  / (f(j1 + j2 + j3 + 1) * f(j1 - m1) * f(j1 + m1) * f(j2 - m2) * f(j2 + m2)))
    S = 0.0
    for v in range(vmin, vmax + 1):
        S += (-1.0) ** (v + j2 + m2) / f(v) * f(j2 + j3 + m1 - v) * f(j1 - m1 + v) / f(j3 - j1 + j2 - v) / f(j3 + m3 - v) / f(v + j1 - j2 - m3)
    return C * S


def _w3j(l1, l2, l3):
    """Real Wigner-3j in e3nn's basis (SU(2) CG conjugated by (-i)^l q_l), Frobenius norm 1."""
    def q(l):
        m_ = np.zeros((2 * l + 1, 2 * l + 1), dtype=np.complex128)
        for m in range(-l, 0):
            m_[l + m, l + abs(m)] = 1 / math.sqrt(2)
            m_[l + m, l - abs(m)] = -1j / math.sqrt(2)
        m_[l, l] = 1
        for m in range(1, l + 1):
            m_[l + m, l + abs(m)] = (-1) ** m / math.sqrt(2)
            m_[l + m, l - abs(m)] = 1j * (-1) ** m / math.sqrt(2)
        return (-1j) ** l * m_

    C = np.zeros((2 * l1 + 1, 2 * l2 + 1, 2 * l3 + 1), dtype=np.complex128)
    for m1 in range(-l1, l1 + 1):
        for m2 in range(-l2, l2 + 1):
            if abs(m1 + m2) <= l3:
                C[l1 + m1, l2 + m2, l3 + m1 + m2] = _su2_cg(l1, m1, l2, m2, l3, m1 + m2)
    R = np.einsum("ij,kl,mn,ikn->jlm", q(l1), q(l2), np.conj(q(l3).T), C).real
    return R / np.linalg.norm(R)


class QHNet(nn.Module):
    def __init__(self, in_node_features=1, sh_lmax=4, hidden_size=128, bottle_hidden_size=32, num_gnn_layers=5, max_radius=12,
                 num_nodes=10, radius_embed_dim=32, orbitals: Dict = None):
        super().__init__()
        if sh_lmax != 4 or hidden_size != 128 or bottle_hidden_size != 32 or radius_embed_dim != 32:
            raise NotImplementedError("nabladft_b200.qhnet kernels are compiled for the shipped config/model/qhnet.yaml sizes")
        if orbitals is None:
            raise ValueError("orbitals table required (config/model/qhnet.yaml:14-22)")
        orbitals = {int(k): [int(v) for v in vs] for k, vs in dict(orbitals).items()}  # Hydra may pass a DictConfig with int keys
        self.hs, self.hbs, self.max_radius, self.num_gnn_layers, self.radius_embed_dim = 128, 32, max_radius, num_gnn_layers, 32
        self.order, self.start_layer = sh_lmax, 2
        self.pair_chunk = int(os.environ.get("NB200_QH_PAIR_CHUNK", 16384))  # atom pairs whose path weights [chunk, 8320] exist at a time
        if self.pair_chunk < 1:
            raise ValueError(f"NB200_QH_PAIR_CHUNK must be a positive number of atom pairs, got {self.pair_chunk}")
        self.node_embedding = nn.Embedding(num_nodes, self.hs)
        self.distance_expansion = _ExpBernstein(radius_embed_dim, max_radius)
        self.orbital_mask, counts = self._get_mask(orbitals)
        if counts != (5, 4, 3):
            raise NotImplementedError("output basis other than 5s4p3d (largest element of the def2-SVP table)")
        self.e3_gnn_layer = nn.ModuleList(_ConvNet(i == 0) for i in range(num_gnn_layers))
        n_extra = max(0, num_gnn_layers - 1 - self.start_layer)
        self.e3_gnn_node_layer = nn.ModuleList(_SelfNet() for _ in range(n_extra))
        self.e3_gnn_node_pair_layer = nn.ModuleList(_PairNet() for _ in range(n_extra))
        ins, cg, n_path, n_bias = _expansion_tables()
        self._exp_ins, self._exp_cg = ins, cg
        hs = self.hs
        mk = lambda n_in, n_out: nn.Sequential(nn.Linear(n_in, hs), nn.SiLU(), nn.Linear(hs, n_out))
        self.expand_ii = nn.ModuleDict({"hamiltonian": _Expansion(n_path, n_bias)})
        self.expand_ij = nn.ModuleDict({"hamiltonian": _Expansion(n_path, n_bias)})
        self.fc_ii = nn.ModuleDict({"hamiltonian": mk(hs, n_path)})
        self.fc_ii_bias = nn.ModuleDict({"hamiltonian": mk(hs, n_bias)})
        self.fc_ij = nn.ModuleDict({"hamiltonian": mk(2 * hs, n_path)})
        self.fc_ij_bias = nn.ModuleDict({"hamiltonian": mk(2 * hs, n_bias)})
        self.output_ii, self.output_ij = _E3Linear(hs, self.hbs), _E3Linear(hs, self.hbs)
        self._cache_key, self._w, self._tables_dev, self._z_ok = None, None, None, {}

    # qhnet.py:323-342
    @staticmethod
    def _get_mask(orbitals):
        max_z = max(orbitals.keys())
        _, counts = np.unique(orbitals[max_z], return_counts=True)
        s_max, p_max, d_max = (int(c) for c in counts)
        ranges = [list(range(s_max)), [s_max + i for i in range(3 * p_max)], [s_max + 3 * p_max + i for i in range(5 * d_max)]]
        masks = {}
        for z, ls in orbitals.items():
            _, cnt = np.unique(ls, return_counts=True)
            m = []
            for t, c in enumerate(cnt):
                m += ranges[t][: int(c) * (1, 3, 5)[t]]
            masks[z] = torch.tensor(m)
        return masks, (s_max, p_max, d_max)

    def set(self):  # reference API (qhnet.py:170-173): masks are uploaded with the weights here
        return self

    # ------------------------------------------------------------------ weight export
    @torch.no_grad()
    def _export(self, dev):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters()) + (str(dev),)
        if key == self._cache_key:
            return self._w
        f32 = torch.float32
        c = lambda t: t.detach().to(dev, f32).contiguous()

        def lin(m):  # e3nn path normalisation 1/sqrt(fan_in) folded into the weights
            return c(m.weight.view(5, m.c_in, m.c_out) / math.sqrt(m.c_in)), c(m.bias)

        def fcn(m):  # x W / sqrt(fan_in); weights stored [in, out]
            return c(m.layer0.weight / math.sqrt(m.layer0.weight.shape[0])), c(m.layer1.weight / math.sqrt(m.layer1.weight.shape[0]))

        def mlp(seq, pad_out=None):
            w2, b2 = seq[2].weight, seq[2].bias
            if pad_out is not None and w2.shape[0] != pad_out:  # GEMM wants N % 4 == 0: zero rows
                w2 = torch.cat([w2, w2.new_zeros(pad_out - w2.shape[0], w2.shape[1])])
                b2 = torch.cat([b2, b2.new_zeros(pad_out - b2.shape[0])])
            return c(seq[0].weight), c(seq[0].bias), c(w2), c(b2)

        # the model's float32 logc, widened: the edge basis takes it in double
        w = {"emb": c(self.node_embedding.weight), "logc": self.distance_expansion.logc.detach().to(dev, torch.float64).contiguous()}
        w["alpha"] = float(torch.nn.functional.softplus(self.distance_expansion._alpha))
        w["conv"] = []
        for i, layer in enumerate(self.e3_gnn_layer):
            cv = layer.conv
            d = {"fc_node": fcn(cv.fc_node), "layer_l0": fcn(cv.layer_l0), "linear_out": lin(cv.linear_out)}
            if i > 0:
                d.update(norm_gate=mlp(cv.norm_gate.fc), linear_node=lin(cv.linear_node), linear_node_pre=lin(cv.linear_node_pre))
            w["conv"].append(d)
        w["self"] = [dict(l1=lin(s.linear_node_1), l2=lin(s.linear_node_2), l3=lin(s.linear_node_3), tp=c(s.tp.weight),
                          ng=mlp(s.norm_gate.fc), ng1=mlp(s.norm_gate_1.fc), ng2=mlp(s.norm_gate_2.fc)) for s in self.e3_gnn_node_layer]
        w["pair"] = [dict(n=lin(p.linear_node_pair_n), inner=lin(p.linear_node_pair_inner), out=lin(p.linear_node_pair),
                          fc_node_pair=fcn(p.fc_node_pair), ng=mlp(p.norm_gate.fc), ng_pre=mlp(p.norm_gate_pre.fc), fc=mlp(p.fc))
                     for p in self.e3_gnn_node_pair_layer]
        w["out_ii"], w["out_ij"] = lin(self.output_ii), lin(self.output_ij)
        w["fc_ii"], w["fc_ii_bias"] = mlp(self.fc_ii["hamiltonian"]), mlp(self.fc_ii_bias["hamiltonian"], pad_out=52)
        ij, ijb = self.fc_ij["hamiltonian"], self.fc_ij_bias["hamiltonian"]
        hs = self.hs
        w["fc_ij"] = (c(ij[0].weight[:, :hs]), c(ij[0].weight[:, hs:]), c(ij[0].bias), c(ij[2].weight), c(ij[2].bias))
        w2, b2 = ijb[2].weight, ijb[2].bias
        w["fc_ij_bias"] = (c(ijb[0].weight[:, :hs]), c(ijb[0].weight[:, hs:]), c(ijb[0].bias),
                           c(torch.cat([w2, w2.new_zeros(2, w2.shape[1])])), c(torch.cat([b2, b2.new_zeros(2)])))
        # orbital masks: table [z][32] of block indices + count (qhnet.py:323-342)
        zmax = max(self.orbital_mask.keys()) + 1
        mask_tab = torch.zeros(zmax, 32, dtype=torch.int32)
        norb_tab = torch.zeros(zmax, dtype=torch.int32)
        for z, m in self.orbital_mask.items():
            mask_tab[z, : len(m)] = m.to(torch.int32)
            norb_tab[z] = len(m)
        w["mask_tab"], w["norb_tab"] = mask_tab.to(dev), norb_tab.to(dev)
        self._w, self._cache_key = w, key
        return w

    # ------------------------------------------------------------------ op helpers
    def _ops(self, dev):
        lib = _lib.load()
        s = current_stream
        E = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)

        class O:
            pass

        o = O()

        def dense(x, W, b, n_out, trans_b, act_kind=None, accumulate=None):
            M, K = x.shape
            y = E(M, n_out) if accumulate is None else accumulate
            a = E(M, n_out) if act_kind is not None else None
            check(lib.nb200_dense(M, n_out, K, ptr(x), K, ptr(W), W.shape[1], trans_b, ptr(y), n_out, 0 if accumulate is None else 1,
                                  ptr(b), ptr(a), act_kind or 0, s()), "nb200_dense")
            return a if act_kind is not None else y

        def fcn(x, ws):  # e3nn FullyConnectedNet: normalize2mom(ssp) hidden layer, linear output; weights [in, out]
            h = dense(x, ws[0], None, ws[0].shape[1], 1, act_kind=ACT_SSP_N)
            return dense(h, ws[1], None, ws[1].shape[1], 1)

        def mlp(x, ws):  # nn.Linear -> SiLU -> nn.Linear; weights [out, in]
            h = dense(x, ws[0], ws[1], ws[0].shape[0], 0, act_kind=ACT_SILU)
            return dense(h, ws[2], ws[3], ws[2].shape[0], 0)

        def linear(x, wl, accumulate_into=None):
            Wl, b = wl
            rows, c_in, c_out = x.shape[0], Wl.shape[1], Wl.shape[2]
            y = E(rows, LM, c_out) if accumulate_into is None else accumulate_into
            check(lib.nb200_qh_linear(ptr(x), ptr(Wl), ptr(b), rows, c_in, c_out, 0 if accumulate_into is None else 1, ptr(y), s()), "nb200_qh_linear")
            return y

        def norm_gate(x, ws):
            rows = x.shape[0]
            f0 = E(rows, 640)
            check(lib.nb200_qh_norm_feats(ptr(x), rows, ptr(f0), s()), "nb200_qh_norm_feats")
            g = mlp(f0, ws)
            y = E(rows, LM, 128)
            check(lib.nb200_qh_gate(ptr(x), ptr(g), rows, ptr(y), s()), "nb200_qh_gate")
            return y

        def axpy(y, x):
            check(lib.nb200_axpy(ptr(y), ptr(x), y.numel(), s()), "nb200_axpy")
            return y

        prof = getattr(self, "profile", None)
        if prof is not None:  # optional per-op CUDA-event timing (bench_qhnet.py --profile); never on by default
            def timed(name, fn):
                def wrapped(*a, **k):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    r = fn(*a, **k)
                    e1.record()
                    prof.setdefault(name, []).append((e0, e1))
                    return r
                return wrapped
            dense_t = timed("dense", dense)

            def fcn(x, ws):  # noqa: F811 (re-bind so the nested calls are attributed to "dense")
                h = dense_t(x, ws[0], None, ws[0].shape[1], 1, act_kind=ACT_SSP_N)
                return dense_t(h, ws[1], None, ws[1].shape[1], 1)

            def mlp(x, ws):  # noqa: F811
                h = dense_t(x, ws[0], ws[1], ws[0].shape[0], 0, act_kind=ACT_SILU)
                return dense_t(h, ws[2], ws[3], ws[2].shape[0], 0)

            def norm_gate(x, ws):  # noqa: F811
                rows = x.shape[0]
                f0 = E(rows, 640)
                check(lib.nb200_qh_norm_feats(ptr(x), rows, ptr(f0), s()), "nb200_qh_norm_feats")
                g = mlp(f0, ws)
                y = E(rows, LM, 128)
                check(lib.nb200_qh_gate(ptr(x), ptr(g), rows, ptr(y), s()), "nb200_qh_gate")
                return y
            dense, linear = dense_t, timed("e3_linear", linear)
        o.dense, o.fcn, o.mlp, o.linear, o.norm_gate, o.axpy, o.E, o.lib, o.s = dense, fcn, mlp, linear, norm_gate, axpy, E, lib, s
        return o

    def _graph(self, o, pos, mol_ptr, n_mol, cutoff, e_cap):
        dev, N = pos.device, pos.shape[0]
        I = lambda n: torch.empty(n, dtype=torch.int32, device=dev)
        g = dict(row_ptr=I(N + 1), col=I(e_cap), rev=I(e_cap), tgt=I(e_cap), geom=o.E(e_cap, 4), status=torch.zeros(4, dtype=torch.int32, device=dev))
        deg = I(N)
        check(o.lib.nb200_neighbor_build(ptr(pos), ptr(mol_ptr), n_mol, N, float(cutoff), 2**31 - 1, e_cap, ptr(g["row_ptr"]), ptr(g["col"]),
                                         ptr(g["rev"]), ptr(g["geom"]), ptr(deg), ptr(g["status"]), o.s()), "nb200_neighbor_build")
        check(o.lib.nb200_qh_expand_rows(ptr(g["row_ptr"]), N, ptr(g["tgt"]), o.s()), "nb200_qh_expand_rows")
        return g

    # ------------------------------------------------------------------ forward (qhnet.py:186-252)
    def forward(self, data, keep_blocks=False, packed: bool = False):
        # inference only: a training-mode call with autograd on would silently return graph-less outputs -- fail loudly instead
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("QHNet training through the CUDA path is not built (inference only); call .eval() or torch.no_grad()")
        with torch.no_grad():
            return self._forward(data, keep_blocks, packed)

    def _unsupported(self, z):
        """Mask of the atoms whose Z has no embedding row or no orbital-table entry, computed where z lives without a host read.  The
        kernels index both tables by Z unchecked, and an element without orbitals would silently vanish from H."""
        ok = self._z_ok.get(str(z.device))
        if ok is None:  # built once per device: True for every Z with both an embedding row and orbitals
            ok = torch.zeros(self.node_embedding.num_embeddings, dtype=torch.bool)
            ok[[k for k in self.orbital_mask if k < ok.numel()]] = True
            ok = self._z_ok.setdefault(str(z.device), ok.to(z.device))
        zl = z.reshape(-1).long()
        return ~(ok[zl.clamp(0, ok.numel() - 1)] & (zl >= 0) & (zl < ok.numel()))

    def _refuse(self, z, bad):
        raise ValueError(f"atomic numbers {torch.unique(z.reshape(-1)[bad]).tolist()} are not supported: the orbital table has "
                         f"{sorted(self.orbital_mask)} and the embedding has num_nodes = {self.node_embedding.num_embeddings}")

    def _forward(self, data, keep_blocks, packed):
        if self.pair_chunk < 1:
            raise ValueError(f"pair_chunk must be a positive number of atom pairs, got {self.pair_chunk}")
        pos = data.pos
        if not pos.is_cuda:
            z = getattr(data, "z", None)
            bad = None if z is None else self._unsupported(z)
            if bad is not None and bool(bad.any()):  # the same refusal as on the device, before the CUDA-only error
                self._refuse(z, bad)
            raise NablaB200Error("nabladft_b200.qhnet.QHNet runs on CUDA only (no CPU fallback)")
        bad = self._unsupported(data.z)
        dev = pos.device
        w = self._export(dev)
        o = self._ops(dev)
        lib = o.lib
        if self._tables_dev != str(dev):
            check(lib.nb200_qh_expand_setup(self._exp_ins.ctypes.data_as(ctypes.c_void_p), self._exp_cg.ctypes.data_as(ctypes.c_void_p)), "expand_setup")
            self._tables_dev = str(dev)
        z = data.z.reshape(-1).to(torch.int32).contiguous()
        pos = pos.detach().to(torch.float32).contiguous()
        mol_ptr = data.ptr.to(torch.int32).contiguous()
        n_mol, N = mol_ptr.numel() - 1, z.shape[0]
        n_per = (mol_ptr[1:] - mol_ptr[:-1]).to(torch.int64)
        # ordered pairs, known from the batch structure, and the unsupported-element count: one host read, before any kernel launch
        P, n_bad = torch.stack([(n_per * (n_per - 1)).sum(), bad.sum()]).tolist()
        if n_bad:
            self._refuse(z, bad)
        gf = self._graph(o, pos, mol_ptr, n_mol, 10000.0, max(P, 1))
        gc = self._graph(o, pos, mol_ptr, n_mol, self.max_radius, max(P, 1))  # E <= P
        st = gc["status"].cpu()
        if int(st[1]) != 0 or int(gf["status"].cpu()[0]) != P:
            raise NablaB200Error(f"neighbour build failed: status {st.tolist()}")
        E_ = int(st[0])
        rbf_c, sh_c = o.E(max(E_, 1), 32), o.E(max(E_, 1), LM)
        check(lib.nb200_qh_edge_basis(ptr(gc["geom"]), ptr(gc["status"]), E_, w["alpha"], float(self.max_radius), -1.0, ptr(w["logc"]), 32,
                                      ptr(rbf_c), ptr(sh_c), o.s()), "nb200_qh_edge_basis")
        rbf_f = o.E(max(P, 1), 32)
        check(lib.nb200_qh_edge_basis(ptr(gf["geom"]), ptr(gf["status"]), P, w["alpha"], float(self.max_radius), -1.0, ptr(w["logc"]), 32,
                                      ptr(rbf_f), None, o.s()), "nb200_qh_edge_basis")
        emb = w["emb"].index_select(0, z.long())  # nn.Embedding lookup (qhnet.py:188)

        def invariants(f, g, n_e, mode, width):
            out = o.E(max(n_e, 1), width)
            check(lib.nb200_qh_invariants(ptr(f), ptr(g["tgt"]), ptr(g["col"]), ptr(g["status"]), n_e, mode, ptr(out), o.s()), "nb200_qh_invariants")
            return out

        x, fii, fij = None, None, None
        for li in range(self.num_gnn_layers):
            cw = w["conv"][li]
            w1 = o.fcn(rbf_c, cw["fc_node"])
            out = o.E(N, LM, 128)
            if li == 0:
                w2 = o.fcn(invariants(emb, gc, E_, 1, 256), cw["layer_l0"])
                check(lib.nb200_qh_tp_conv(ptr(emb), ptr(sh_c), ptr(w1), ptr(w2), ptr(gc["row_ptr"]), ptr(gc["col"]), N, 1, 0, ptr(out), o.s()), "tp_conv")
                x = o.linear(out, cw["linear_out"])
            else:
                pre = o.linear(x, cw["linear_node_pre"])
                w2 = o.fcn(invariants(pre, gc, E_, 0, 768), cw["layer_l0"])
                xl = o.linear(o.norm_gate(x, cw["norm_gate"]), cw["linear_node"])
                check(lib.nb200_qh_tp_conv(ptr(xl), ptr(sh_c), ptr(w1), ptr(w2), ptr(gc["row_ptr"]), ptr(gc["col"]), N, 0, 1, ptr(out), o.s()), "tp_conv")
                x = o.axpy(o.linear(out, cw["linear_out"]), x)  # ConvNetLayer residual (layers.py:338-343)
            if li > self.start_layer:
                k = li - self.start_layer - 1
                sw, pw = w["self"][k], w["pair"][k]
                # SelfNetLayer (layers.py:565-578)
                xl = o.linear(o.norm_gate(x, sw["ng1"]), sw["l1"])
                xr = o.linear(o.norm_gate(x, sw["ng2"]), sw["l2"])
                t = o.E(N, LM, 128)
                check(lib.nb200_qh_tp_self(ptr(xl), ptr(xr), ptr(sw["tp"]), ptr(x), N, ptr(t), o.s()), "tp_self")
                f_new = o.linear(o.norm_gate(t, sw["ng"]), sw["l3"])
                fii = f_new if fii is None else o.axpy(f_new, fii)
                # PairNetLayer (layers.py:465-492).  The per-pair path weights [P, 8320] (two of them, 3.3 GB each at config 4) are generated
                # and consumed chunk by chunk of the pair list: they never exist for all pairs at once (13.2 -> 4 GB peak), and a chunk's
                # rows are still in L2 when the tensor-product kernel reads them.
                a0 = o.linear(x, pw["inner"])
                xn = o.linear(o.norm_gate(x, pw["ng_pre"]), pw["n"])
                pair = o.E(max(P, 1), LM, 128)
                for p0 in range(0, P, self.pair_chunk):
                    pc = min(self.pair_chunk, P - p0)
                    inv = o.E(pc, 768)
                    check(lib.nb200_qh_invariants(ptr(a0), ptr(gf["tgt"][p0:]), ptr(gf["col"][p0:]), ptr(gf["status"]), pc, 2, ptr(inv), o.s()),
                          "nb200_qh_invariants")
                    wp2 = o.mlp(inv, pw["fc"])
                    wp1 = o.fcn(rbf_f[p0:p0 + pc], pw["fc_node_pair"])
                    check(lib.nb200_qh_tp_pair(ptr(xn), ptr(wp1), ptr(wp2), ptr(gf["tgt"][p0:]), ptr(gf["col"][p0:]), ptr(gf["status"]), pc,
                                               ptr(pair[p0:]), o.s()), "tp_pair")
                    del wp1, wp2, inv
                p_new = o.linear(o.norm_gate(pair, pw["ng"]), pw["out"])
                fij = p_new if fij is None else o.axpy(p_new, fij)
        fii_b, fij_b = o.linear(fii, w["out_ii"]), o.linear(fij, w["out_ij"])
        diag, offd = o.E(N, 32, 32), o.E(max(P, 1), 32, 32)
        Wii, Bii = o.mlp(emb, w["fc_ii"]), o.mlp(emb, w["fc_ii_bias"])
        check(lib.nb200_qh_expand(ptr(fii_b), ptr(Wii), ptr(Bii), 52, N, ptr(diag), o.s()), "expand_ii")

        A_w, B_w = [o.dense(emb, w["fc_ij"][i], None, 128, 0) for i in (0, 1)]
        A_b, B_b = [o.dense(emb, w["fc_ij_bias"][i], None, 128, 0) for i in (0, 1)]
        for p0 in range(0, P, self.pair_chunk):  # expansion weights [P, 8320] chunk by chunk, as above
            pc = min(self.pair_chunk, P - p0)

            def pair_mlp(ws, A, Bn):
                h = o.E(pc, 128)
                check(lib.nb200_qh_pair_hidden(ptr(A), ptr(Bn), ptr(ws[2]), ptr(gf["tgt"][p0:]), ptr(gf["col"][p0:]), ptr(gf["status"]), pc, ptr(h), o.s()),
                      "pair_hidden")
                return o.dense(h, ws[3], ws[4], ws[3].shape[0], 0)

            Wij, Bij = pair_mlp(w["fc_ij"], A_w, B_w), pair_mlp(w["fc_ij_bias"], A_b, B_b)
            check(lib.nb200_qh_expand(ptr(fij_b[p0:]), ptr(Wij), ptr(Bij), 52, pc, ptr(offd[p0:]), o.s()), "expand_ij")
            del Wij, Bij
        if keep_blocks:
            # symmetrised blocks (qhnet.py:240-251); transpose_edge_index == rev of the full CSR
            return {"hamiltonian_diagonal_blocks": diag + diag.transpose(-1, -2),
                    "hamiltonian_non_diagonal_blocks": offd + offd[gf["rev"][:P].long()].transpose(-1, -2)}
        # ---- block assembly + H + H^T, per molecule (qhnet.py:293-321, 234-238)
        norb_atom = w["norb_tab"][z.long()].to(torch.int64)
        atom_mol = torch.repeat_interleave(torch.arange(n_mol, device=dev), n_per).to(torch.int32)
        csum = torch.cumsum(norb_atom, 0)
        mol_first = mol_ptr[:-1].long()
        mol_base = (csum - norb_atom)[mol_first]  # orbital offset of each molecule's first atom
        atom_orb_off = (csum - norb_atom - mol_base[atom_mol.long()]).to(torch.int32)
        mol_norb = torch.zeros(n_mol, dtype=torch.int64, device=dev).index_add_(0, atom_mol.long(), norb_atom)
        mol_h_off = torch.zeros(n_mol + 1, dtype=torch.int64, device=dev)
        mol_h_off[1:] = torch.cumsum(mol_norb * mol_norb, 0)
        H = torch.zeros(int(mol_h_off[-1].item()), dtype=torch.float32, device=dev)
        check(lib.nb200_qh_assemble(ptr(diag), ptr(offd), ptr(z), ptr(gf["tgt"]), ptr(gf["col"]), ptr(gf["rev"]), N, P, ptr(w["mask_tab"].reshape(-1)),
                                    ptr(w["norb_tab"]), ptr(atom_mol), ptr(atom_orb_off), ptr(mol_h_off), ptr(mol_norb.to(torch.int32)), ptr(H), o.s()),
              "nb200_qh_assemble")
        mats = [H[int(mol_h_off[m]):int(mol_h_off[m + 1])].view(int(mol_norb[m]), int(mol_norb[m])) for m in range(n_mol)]
        self.last_blocks = mats  # per-molecule dense Hamiltonians (what HamiltonianLoss.packed consumes)
        if packed:  # extension: the list itself -- the reference's dense block diagonal is 2.5 GB at config 4 (>98 % structural zeros)
            return mats
        return mats[0] if n_mol == 1 else torch.block_diag(*mats)
