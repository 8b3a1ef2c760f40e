"""H100-native drop-in for `nablaDFT.gemnet_oc.GemNetOC` (config/model/gemnet-oc.yaml): SURVEY.md section 8 a19 / f3.

Same constructor signature (`nablaDFT/gemnet_oc/gemnet_oc.py:171-228`), same `forward(data) -> (energy [B], forces [N, 3])` contract
(gemnet_oc.py:1121-1251) and the same state-dict names / shapes (429 entries for the shipped config), so the yaml works with
`_target_: nabladft_b200.gemnet_oc.GemNetOC` and reference checkpoints load with strict=True.  The arithmetic -- the four graphs, the
triplet / quadruplet enumeration, bases, interaction and output blocks, coupled direct forces -- runs in `libnabla_b200.so`
(`csrc/gemnet_oc.cu`, C ABI `nb200_gemnet_oc_*` in include/nabla_b200.h).  This file owns the parameters and the export of the
reference-named tensors into the flat canonical buffer the C ABI takes (basis scale factors folded into the concatenated basis matrices).

Supported: the shipped configuration (non-periodic, direct coupled forces, all four extra interactions, the yaml's sizes).  Everything
else raises at construction.  Training mode returns (energy, forces) on one autograd node (`GemNetOCFn`): the engine back-propagates dLoss/dE
and dLoss/dF through every kernel (csrc/gemnet_oc_train.inc) and autograd un-folds the flat export.  No CPU fallback.

Relaxation: `GemNetOC.engine()` hands `optimization.ASEBatchwiseLBFGS` a forward that never waits for the host
(`nb200_gemnet_oc_energy_forces_async`, sized by per-batch upper bounds of the edge counts: DESIGN.md 3.9).

Normal modes: `GemNetOCRunner.run_hvp` gives exact products with the direct forces' Jacobian, jv = -(dF/dR) v
(`nb200_gemnet_oc_jvp`, one tangent pass through the training forward: DESIGN.md 3.9.1); `vibrations.hessians` / `normal_modes` use it.

STATUS (round 1): every kernel has been checked against the oracle through the host-emulation build of the same source
(tests/emu, tests/test_gemnet_emu.py); the GPU run of `tests/test_zz_gpu_first_runs.py` is the first execution on a device.
"""
import ctypes
import math
import re
from ctypes import POINTER, byref, c_float, c_int64
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from ._lib import EngineDriver, GemNetOCWeights, NablaB200Error, check
from .engine import BoundedEngine, refuse_training

# ---- canonical layout: keep in step with the enums of include/nabla_b200.h (tests/test_host.py compares the names) -------------------
G_NAMES = ["RBF_OFFSET", "EMB", "CAT_MAIN", "CAT_AE", "CAT_Q", "CAT_A2A", "EDGE_EMB", "OUT_E0", "OUT_E_RES", "OUT_ENERGY", "OUT_F0", "OUT_F_RES",
           "OUT_FORCES"]
I_NAMES = ["DENSE_CA", "T_BA", "T_RBF", "T_BIL", "T_DOWN", "T_UPCA", "T_UPAC", "Q_DB", "Q_RBF", "Q_CBF", "Q_BIL", "Q_DOWN", "Q_UPCA", "Q_UPAC",
           "AE_BA", "AE_RBF", "AE_BIL", "AE_DOWN", "AE_UPCA", "AE_UPAC", "EA_BA", "EA_RBF", "EA_BIL", "EA_DOWN", "EA_UP", "AA_BIL", "AA_DOWN",
           "AA_UP", "BEFORE_SKIP", "AFTER_SKIP", "AU_RBF", "AU_L0", "AU_RES", "CONCAT", "RES_M"]
O_NAMES = ["RBF", "L0", "RES", "E2", "F", "RBF_F"]
S_NAMES = ["T_RBF", "Q_RBF", "Q_CBF", "AE_RBF", "EA_RBF", "AU_SUM"]
SO_NAMES = ["SUM", "RBF_F"]
C_NAMES = ["A2A", "MAIN", "AE", "Q", "TIN"]
N_COUNTS = 8
LD_MAIN = 1920
SIGNATURES = {k: v for k, v in _lib.SIGNATURES.items() if k.startswith("nb200_gemnet_oc_")}


def bind(lib):
    """The GemNet-OC prototypes on `lib`, e.g. an emulation build of csrc/gemnet_oc.cu, which exports no other engine."""
    return _lib.bind(lib, ["nb200_gemnet_oc_"])


# ---- parameter holders with the reference's attribute names ----------------------------------------------------------------------------
def _he_orthogonal_(w: torch.Tensor) -> torch.Tensor:
    """Orthogonal directions rescaled to variance 1 / fan_in (the intent of initializers.py he_orthogonal_init; checkpoints overwrite it)."""
    with torch.no_grad():
        nn.init.orthogonal_(w)
        fan_in = w.shape[1] if w.dim() == 2 else w.shape[:-1].numel()
        w.mul_(math.sqrt(1.0 / fan_in) / float(w.std().clamp_min(1e-12)))
    return w


class _Dense(nn.Module):  # base_layers.py:15-63 (bias=False everywhere in this model)
    def __init__(self, n_in, n_out):
        super().__init__()
        self.linear = nn.Linear(n_in, n_out, bias=False)
        _he_orthogonal_(self.linear.weight)


class _Scale(nn.Module):  # scale_factor.py: 0 = not fitted = identity
    def __init__(self):
        super().__init__()
        self.scale_factor = nn.Parameter(torch.tensor(0.0), requires_grad=False)


class _Gaussian(nn.Module):
    def __init__(self, num):
        super().__init__()
        self.register_buffer("offset", torch.linspace(0.0, 1.0, num))


class _RadialBasis(nn.Module):  # radial_basis.py:176-220
    def __init__(self, num_radial, scale_basis):
        super().__init__()
        self.rbf = _Gaussian(num_radial)
        if scale_basis:
            self.scale_rbf = _Scale()


class _AngleBasis(nn.Module):  # spherical_basis.py: CircularBasisLayer / SphericalBasisLayer
    def __init__(self, radial_basis, scale_name, scale_basis):
        super().__init__()
        self.radial_basis = radial_basis
        if scale_basis:
            setattr(self, scale_name, _Scale())


class _BasisEmbedding(nn.Module):  # efficient.py:15-140
    def __init__(self, num_radial, emb_size_interm, num_spherical=None):
        super().__init__()
        shape = (emb_size_interm, num_radial) if num_spherical is None else (num_radial, num_spherical, emb_size_interm)
        self.weight = nn.Parameter(_he_orthogonal_(torch.empty(shape)), requires_grad=True)


class _Residual(nn.Module):  # base_layers.py:78-97
    def __init__(self, units):
        super().__init__()
        self.dense_mlp = nn.Sequential(_Dense(units, units), _Dense(units, units))


def _mlp(units_in, units, n_hidden):  # atom_update_block.py get_mlp
    return nn.ModuleList(([_Dense(units_in, units)] if units_in != units else []) + [_Residual(units) for _ in range(n_hidden)])


class _EffBilinear(nn.Module):  # efficient.py:143-253
    def __init__(self, emb_in, emb_interm, emb_out):
        super().__init__()
        self.bilinear = _Dense(emb_in * emb_interm, emb_out)


class _Triplet(nn.Module):  # interaction_block.py TripletInteraction
    def __init__(self, emb_in, emb_out, trip_in, trip_out, rbf, cbf, symmetric_mp):
        super().__init__()
        self.dense_ba = _Dense(emb_in, emb_in)
        self.mlp_rbf, self.scale_rbf = _Dense(rbf, emb_in), _Scale()
        self.mlp_cbf, self.scale_cbf_sum = _EffBilinear(trip_in, cbf, trip_out), _Scale()
        self.down_projection = _Dense(emb_in, trip_in)
        self.up_projection_ca = _Dense(trip_out, emb_out)
        if symmetric_mp:
            self.up_projection_ac = _Dense(trip_out, emb_out)


class _Quadruplet(nn.Module):
    def __init__(self, ee, quad_in, quad_out, rbf, cbf, sbf):
        super().__init__()
        self.dense_db = _Dense(ee, ee)
        self.mlp_rbf, self.scale_rbf = _Dense(rbf, ee), _Scale()
        self.mlp_cbf, self.scale_cbf = _Dense(cbf, quad_in), _Scale()
        self.mlp_sbf, self.scale_sbf_sum = _EffBilinear(quad_in, sbf, quad_out), _Scale()
        self.down_projection = _Dense(ee, quad_in)
        self.up_projection_ca = _Dense(quad_out, ee)
        self.up_projection_ac = _Dense(quad_out, ee)


class _Pair(nn.Module):
    def __init__(self, ea, pair_in, pair_out, rbf):
        super().__init__()
        self.bilinear, self.scale_rbf_sum = _Dense(rbf * pair_in, pair_out), _Scale()
        self.down_projection = _Dense(ea, pair_in)
        self.up_projection = _Dense(pair_out, ea)


class _AtomUpdate(nn.Module):  # atom_update_block.py:15-91
    def __init__(self, ea, ee, rbf, n_hidden):
        super().__init__()
        self.dense_rbf, self.scale_sum = _Dense(rbf, ee), _Scale()
        self.layers = _mlp(ee, ea, n_hidden)


class _Output(nn.Module):  # atom_update_block.py:93-172 (direct forces)
    def __init__(self, ea, ee, rbf, n_hidden, n_hidden_afteratom):
        super().__init__()
        self.dense_rbf, self.scale_sum = _Dense(rbf, ee), _Scale()
        self.layers = _mlp(ee, ea, n_hidden)
        self.seq_energy_pre = self.layers  # the reference registers the same list under both names
        self.seq_energy2 = _mlp(ea, ea, n_hidden_afteratom)
        self.scale_rbf_F = _Scale()
        self.seq_forces = _mlp(ee, ee, n_hidden)
        self.dense_rbf_F = _Dense(rbf, ee)


class _EdgeEmbedding(nn.Module):
    def __init__(self, atom_features, edge_features, out_features):
        super().__init__()
        self.dense = _Dense(2 * atom_features + edge_features, out_features)


class _AtomEmbedding(nn.Module):
    def __init__(self, emb_size, num_elements):
        super().__init__()
        self.embeddings = nn.Embedding(num_elements, emb_size)
        nn.init.uniform_(self.embeddings.weight, a=-math.sqrt(3), b=math.sqrt(3))


class _Interaction(nn.Module):  # interaction_block.py:19-290
    def __init__(self, ea, ee, trip_in, trip_out, quad_in, quad_out, a2a_in, a2a_out, rbf, cbf, sbf, n_before, n_after, n_concat, n_atom):
        super().__init__()
        self.dense_ca = _Dense(ee, ee)
        self.trip_interaction = _Triplet(ee, ee, trip_in, trip_out, rbf, cbf, True)
        self.quad_interaction = _Quadruplet(ee, quad_in, quad_out, rbf, cbf, sbf)
        self.atom_edge_interaction = _Triplet(ea, ee, trip_in, trip_out, rbf, cbf, True)
        self.edge_atom_interaction = _Triplet(ee, ea, trip_in, trip_out, rbf, cbf, False)
        self.atom_interaction = _Pair(ea, a2a_in, a2a_out, rbf)
        self.layers_before_skip = nn.ModuleList([_Residual(ee) for _ in range(n_before)])
        self.layers_after_skip = nn.ModuleList([_Residual(ee) for _ in range(n_after)])
        self.atom_emb_layers = nn.ModuleList([])
        self.atom_update = _AtomUpdate(ea, ee, rbf, n_atom)
        self.concat_layer = _EdgeEmbedding(ea, ee, ee)
        self.residual_m = nn.ModuleList([_Residual(ee) for _ in range(n_concat)])


_FIXED = dict(num_targets=1, num_spherical=7, num_radial=128, emb_size_atom=256, emb_size_edge=512, emb_size_trip_in=64, emb_size_trip_out=64,
              emb_size_quad_in=32, emb_size_quad_out=32, emb_size_aint_in=64, emb_size_aint_out=64, emb_size_rbf=16, emb_size_cbf=16, emb_size_sbf=32,
              num_before_skip=2, num_after_skip=2, num_concat=1, num_atom=3, num_output_afteratom=3, num_atom_emb_layers=0, num_global_out_layers=2,
              regress_forces=True, direct_forces=True, use_pbc=False, extensive=True, forces_coupled=True, activation="silu", quad_interaction=True,
              atom_edge_interaction=True, edge_atom_interaction=True, atom_interaction=True, enforce_max_neighbors_strictly=True)


class GemNetOC(nn.Module):
    def __init__(self, num_targets: int, num_spherical: int, num_radial: int, num_blocks: int, emb_size_atom: int, emb_size_edge: int,
                 emb_size_trip_in: int, emb_size_trip_out: int, emb_size_quad_in: int, emb_size_quad_out: int, emb_size_aint_in: int,
                 emb_size_aint_out: int, emb_size_rbf: int, emb_size_cbf: int, emb_size_sbf: int, num_before_skip: int, num_after_skip: int,
                 num_concat: int, num_atom: int, num_output_afteratom: int, num_atom_emb_layers: int = 0, num_global_out_layers: int = 2,
                 regress_forces: bool = True, direct_forces: bool = False, use_pbc: bool = True, scale_backprop_forces: bool = False,
                 cutoff: float = 6.0, cutoff_qint: Optional[float] = None, cutoff_aeaint: Optional[float] = None, cutoff_aint: Optional[float] = None,
                 max_neighbors: int = 50, max_neighbors_qint: Optional[int] = None, max_neighbors_aeaint: Optional[int] = None,
                 max_neighbors_aint: Optional[int] = None, enforce_max_neighbors_strictly: bool = True, rbf: Dict[str, str] = {"name": "gaussian"},
                 rbf_spherical: Optional[dict] = None, envelope: Dict = {"name": "polynomial", "exponent": 5},
                 cbf: Dict[str, str] = {"name": "spherical_harmonics"}, sbf: Dict[str, str] = {"name": "spherical_harmonics"},
                 extensive: bool = True, forces_coupled: bool = False, output_init: str = "HeOrthogonal", activation: str = "silu",
                 quad_interaction: bool = False, atom_edge_interaction: bool = False, edge_atom_interaction: bool = False,
                 atom_interaction: bool = False, scale_basis: bool = False, num_elements: int = 83, otf_graph: bool = False,
                 scale_file: Optional[str] = None) -> None:
        super().__init__()
        given = dict(locals())
        bad = [f"{k}={given[k]!r} (built: {v!r})" for k, v in _FIXED.items() if given[k] != v]
        cut = [cutoff, cutoff_qint or cutoff, cutoff_aeaint or cutoff, cutoff_aint or cutoff]
        if max(cut) != min(cut):
            bad.append(f"cutoffs {cut} (built: all equal)")
        if rbf.get("name") != "gaussian" or (rbf_spherical and rbf_spherical.get("name") != "gaussian"):
            bad.append("rbf (built: gaussian)")
        if envelope.get("name") != "polynomial" or envelope.get("exponent") != 5:
            bad.append("envelope (built: polynomial, exponent 5)")
        if cbf.get("name") != "spherical_harmonics" or sbf.get("name") != "legendre_outer":
            bad.append("cbf / sbf (built: spherical_harmonics / legendre_outer)")
        if scale_file is not None:
            bad.append("scale_file (load the fitted factors through the state dict instead)")
        if bad:
            raise NablaB200Error("GemNetOC: configuration outside the compiled path (config/model/gemnet-oc.yaml): " + "; ".join(bad))
        self.num_blocks, self.cutoff, self.num_elements = num_blocks, float(cutoff), num_elements
        # the forces are a direct output of the model, not the gradient of its energy (`md.BatchwiseMD` refuses such a model)
        self.regress_forces, self.direct_forces = regress_forces, direct_forces
        self.max_neighbors = max_neighbors
        self.max_neighbors_qint = max_neighbors_qint or max_neighbors
        self.max_neighbors_aeaint = max_neighbors_aeaint or max_neighbors
        self.max_neighbors_aint = max_neighbors_aint or max_neighbors
        ea, ee, nr, ns = emb_size_atom, emb_size_edge, num_radial, num_spherical
        rbf_, cbf_, sbf_ = emb_size_rbf, emb_size_cbf, emb_size_sbf
        rb = lambda: _RadialBasis(nr, scale_basis)
        # gemnet_oc.py:356-470 (init_basis_functions / init_shared_basis_layers): `radial_basis_spherical` is ONE module under three parents
        self.radial_basis = rb()
        shared_sph = rb()
        self.cbf_basis_qint = _AngleBasis(rb(), "scale_cbf", scale_basis)
        self.sbf_basis_qint = _AngleBasis(shared_sph, "scale_sbf", scale_basis)
        self.radial_basis_aeaint = rb()
        self.cbf_basis_aeint = _AngleBasis(shared_sph, "scale_cbf", scale_basis)
        self.cbf_basis_eaint = _AngleBasis(rb(), "scale_cbf", scale_basis)
        self.radial_basis_aint = rb()
        self.cbf_basis_tint = _AngleBasis(shared_sph, "scale_cbf", scale_basis)
        self.mlp_rbf_qint = _Dense(nr, rbf_)
        self.mlp_cbf_qint = _BasisEmbedding(nr, cbf_, ns)
        self.mlp_sbf_qint = _BasisEmbedding(nr, sbf_, ns ** 2)
        self.mlp_rbf_aeint = _Dense(nr, rbf_)
        self.mlp_cbf_aeint = _BasisEmbedding(nr, cbf_, ns)
        self.mlp_rbf_eaint = _Dense(nr, rbf_)
        self.mlp_cbf_eaint = _BasisEmbedding(nr, cbf_, ns)
        self.mlp_rbf_aint = _BasisEmbedding(nr, rbf_)
        self.mlp_rbf_tint = _Dense(nr, rbf_)
        self.mlp_cbf_tint = _BasisEmbedding(nr, cbf_, ns)
        self.mlp_rbf_h = _Dense(nr, rbf_)
        self.mlp_rbf_out = _Dense(nr, rbf_)
        self.atom_emb = _AtomEmbedding(ea, num_elements)
        self.edge_emb = _EdgeEmbedding(ea, nr, ee)
        self.int_blocks = nn.ModuleList([
            _Interaction(ea, ee, emb_size_trip_in, emb_size_trip_out, emb_size_quad_in, emb_size_quad_out, emb_size_aint_in, emb_size_aint_out,
                         rbf_, cbf_, sbf_, num_before_skip, num_after_skip, num_concat, num_atom) for _ in range(num_blocks)])
        self.out_blocks = nn.ModuleList([_Output(ea, ee, rbf_, num_atom, num_output_afteratom) for _ in range(num_blocks + 1)])
        self.out_mlp_E = nn.Sequential(_Dense(ea * (num_blocks + 1), ea), *[_Residual(ea) for _ in range(num_global_out_layers)])
        self.out_energy = _Dense(ea, 1)
        self.out_mlp_F = nn.Sequential(_Dense(ee * (num_blocks + 1), ee), *[_Residual(ee) for _ in range(num_global_out_layers)])
        self.out_forces = _Dense(ee, 1)
        self._runner: Optional[GemNetOCRunner] = None
        self._export_key = None
        self._engine: Optional[GemNetOCEngine] = None

    @property
    def num_params(self) -> int:
        return sum(p.numel() for p in self.parameters())

    # ---- export: reference-named tensors -> canonical flat buffer (include/nabla_b200.h NB200_GOC_*) -----------------------------------
    @staticmethod
    def _s(scale_module: Optional[nn.Module]) -> float:
        if scale_module is None:
            return 1.0
        v = float(scale_module.scale_factor.detach())
        return v if v != 0.0 else 1.0  # scale_factor.py:77,148: an unfitted factor (0) is the identity

    def _rs(self, radial: _RadialBasis) -> float:
        return self._s(getattr(radial, "scale_rbf", None))

    def export(self, device, detach: bool = True) -> Tuple[torch.Tensor, List[int], List[float]]:
        """-> (flat fp32 weights on `device`, offsets in floats, per-block scale factors), in the order of the NB200_GOC_* enums.
        detach=False keeps the autograd graph from the reference-named parameters to the flat buffer (training: the engine returns the
        gradient w.r.t. the flat buffer and autograd un-folds concatenations, transposes and scale factors)."""
        f = lambda t: (t.detach() if detach else t).to(torch.float32)
        lin = lambda d: f(d.linear.weight)
        res = lambda r: [lin(r.dense_mlp[0]), lin(r.dense_mlp[1])]
        bemb = lambda b: f(b.weight).reshape(b.weight.shape[0], -1).t()  # [num_radial, S * interm] -> rows = output columns
        offsets = {self.radial_basis.rbf.offset, self.cbf_basis_qint.radial_basis.rbf.offset, self.sbf_basis_qint.radial_basis.rbf.offset,
                   self.radial_basis_aeaint.rbf.offset, self.cbf_basis_eaint.radial_basis.rbf.offset, self.radial_basis_aint.rbf.offset}
        off0 = self.radial_basis.rbf.offset.detach().to(torch.float32)
        if any(not torch.equal(o.detach().to(torch.float32), off0) for o in offsets):
            raise NablaB200Error("GemNetOC: the radial bases carry different Gaussian offsets; the compiled path shares one table")
        s_main, s_sph = self._rs(self.radial_basis), self._rs(self.cbf_basis_tint.radial_basis)
        a_scale = lambda m, n: self._s(getattr(m, n, None))
        pdev = self.atom_emb.embeddings.weight.device  # build on the parameters' device: no host round trip per training step
        cat_main = torch.zeros(LD_MAIN, 128, device=pdev)
        for k, d in enumerate((self.mlp_rbf_qint, self.mlp_rbf_eaint, self.mlp_rbf_tint, self.mlp_rbf_h, self.mlp_rbf_out)):
            cat_main[16 * k:16 * (k + 1)] = lin(d) * s_main
        cat_main[80:192] = bemb(self.mlp_cbf_tint) * (s_sph * a_scale(self.cbf_basis_tint, "scale_cbf"))
        cat_main[192:304] = bemb(self.mlp_cbf_aeint) * (self._rs(self.cbf_basis_aeint.radial_basis) * a_scale(self.cbf_basis_aeint, "scale_cbf"))
        cat_main[304:1872] = bemb(self.mlp_sbf_qint) * (self._rs(self.sbf_basis_qint.radial_basis) * a_scale(self.sbf_basis_qint, "scale_sbf"))
        cat_ae = torch.zeros(128, 128, device=pdev)
        cat_ae[0:16] = lin(self.mlp_rbf_aeint) * self._rs(self.radial_basis_aeaint)
        cat_ae[16:128] = bemb(self.mlp_cbf_eaint) * (self._rs(self.cbf_basis_eaint.radial_basis) * a_scale(self.cbf_basis_eaint, "scale_cbf"))
        cat_q = torch.zeros(128, 128, device=pdev)
        cat_q[0:112] = bemb(self.mlp_cbf_qint) * (self._rs(self.cbf_basis_qint.radial_basis) * a_scale(self.cbf_basis_qint, "scale_cbf"))
        cat_a2a = torch.zeros(64, 128, device=pdev)
        cat_a2a[0:16] = f(self.mlp_rbf_aint.weight) * self._rs(self.radial_basis_aint)
        edge_emb = lin(self.edge_emb.dense).clone()
        edge_emb[:, 512:] *= s_main
        glob = [off0, f(self.atom_emb.embeddings.weight), cat_main, cat_ae, cat_q, cat_a2a, edge_emb, lin(self.out_mlp_E[0]),
                res(self.out_mlp_E[1]) + res(self.out_mlp_E[2]), lin(self.out_energy).reshape(-1), lin(self.out_mlp_F[0]),
                res(self.out_mlp_F[1]) + res(self.out_mlp_F[2]), lin(self.out_forces).reshape(-1)]
        entries: List = list(glob)
        scales: List[float] = []
        for b in self.int_blocks:
            t, q, ae, ea, aa, au = b.trip_interaction, b.quad_interaction, b.atom_edge_interaction, b.edge_atom_interaction, b.atom_interaction, b.atom_update
            entries += [lin(b.dense_ca),
                        lin(t.dense_ba), lin(t.mlp_rbf), lin(t.mlp_cbf.bilinear) * self._s(t.scale_cbf_sum), lin(t.down_projection), lin(t.up_projection_ca), lin(t.up_projection_ac),
                        lin(q.dense_db), lin(q.mlp_rbf), lin(q.mlp_cbf), lin(q.mlp_sbf.bilinear) * self._s(q.scale_sbf_sum), lin(q.down_projection), lin(q.up_projection_ca),
                        lin(q.up_projection_ac),
                        lin(ae.dense_ba), lin(ae.mlp_rbf), lin(ae.mlp_cbf.bilinear) * self._s(ae.scale_cbf_sum), lin(ae.down_projection), lin(ae.up_projection_ca),
                        lin(ae.up_projection_ac),
                        lin(ea.dense_ba), lin(ea.mlp_rbf), lin(ea.mlp_cbf.bilinear) * self._s(ea.scale_cbf_sum), lin(ea.down_projection), lin(ea.up_projection_ca),
                        lin(aa.bilinear) * self._s(aa.scale_rbf_sum), lin(aa.down_projection), lin(aa.up_projection),
                        [w for r in b.layers_before_skip for w in res(r)], [w for r in b.layers_after_skip for w in res(r)],
                        lin(au.dense_rbf), lin(au.layers[0]), [w for r in list(au.layers)[1:] for w in res(r)],
                        lin(b.concat_layer.dense), [w for r in b.residual_m for w in res(r)]]
            # the factors behind a bilinear Dense (scale_cbf_sum, scale_sbf_sum, scale_rbf_sum) are folded into its weights above
            scales += [self._s(t.scale_rbf), self._s(q.scale_rbf), self._s(q.scale_cbf), self._s(ae.scale_rbf), self._s(ea.scale_rbf), self._s(au.scale_sum)]
        for o in self.out_blocks:
            entries += [lin(o.dense_rbf), lin(o.layers[0]), [w for r in list(o.layers)[1:] for w in res(r)], [w for r in o.seq_energy2 for w in res(r)],
                        [w for r in o.seq_forces for w in res(r)], lin(o.dense_rbf_F)]
            scales += [self._s(o.scale_sum), self._s(o.scale_rbf_F)]
        n_expected = len(G_NAMES) + len(I_NAMES) * self.num_blocks + len(O_NAMES) * (self.num_blocks + 1)
        assert len(entries) == n_expected, (len(entries), n_expected)
        flat, offs, pos = [], [], 0
        for ent in entries:
            pos = (pos + 63) // 64 * 64  # 256-byte alignment of every matrix
            offs.append(pos)
            for t_ in (ent if isinstance(ent, list) else [ent]):
                flat.append((pos, t_.reshape(-1)))
                pos += t_.numel()
        buf = torch.zeros(pos + 64, dtype=torch.float32, device=device)
        for p0, t_ in flat:
            buf[p0:p0 + t_.numel()] = t_.to(device)
        return buf, offs, scales

    # ---- forward ------------------------------------------------------------------------------------------------------------------------
    def forward(self, data):
        """data.z [N], data.pos [N,3], data.batch [N] (sorted) -> (E_t [B], F_t [N,3])   (gemnet_oc.py:1121-1251)."""
        runner = self._cuda_runner(data.pos)
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return self._train_with(runner, data)
        return self._forward_with(runner, data)

    def engine_inputs(self, data):
        """(runner, z int32, pos fp32, mol_ptr int32, n_mol) of `data` for the inference engine, with the weights synced: the inputs of
        `GemNetOCRunner.run_hvp` (`vibrations`)."""
        runner = self._cuda_runner(data.pos)
        refuse_training(self)
        self._sync_weights(runner, data.pos.device)
        z, pos, mol_ptr, n_mol, _ = self._batch_args(data)
        return runner, z, pos, mol_ptr, n_mol

    def _cuda_runner(self, pos) -> "GemNetOCRunner":
        if not pos.is_cuda:
            raise NablaB200Error("GemNetOC runs on CUDA tensors only (sm_90a engine; there is no CPU path)")
        return self._get_runner()

    def _get_runner(self) -> "GemNetOCRunner":
        if self._runner is None:
            self._runner = GemNetOCRunner()
        return self._runner

    def _sync_weights(self, runner: "GemNetOCRunner", device) -> None:
        """(Re-)export the weights into `runner` when a parameter changed since the last export."""
        key = (id(runner),) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if key != self._export_key:
            runner.set_weights(self, device)
            self._export_key = key

    def engine(self) -> "GemNetOCEngine":
        """The engine interface of the batch-wise optimiser loop (`optimization.ASEBatchwiseLBFGS`), as `PaiNN.engine()`."""
        if self._engine is None:
            self._engine = GemNetOCEngine(self, self._get_runner())
        return self._engine

    def _batch_args(self, data):
        pos, batch, z = data.pos, data.batch, data.z
        n_mol = int(batch[-1].item()) + 1
        counts = torch.bincount(batch, minlength=n_mol)
        if bool((batch[1:] < batch[:-1]).any()):
            raise NablaB200Error("GemNetOC: `batch` must be sorted (atoms of a molecule contiguous), as PyG collation produces it")
        max_atoms = int(counts.max().item())
        GemNetOCEngine.check_sizes(self, max_atoms)
        mol_ptr = torch.zeros(n_mol + 1, dtype=torch.int32, device=pos.device)
        mol_ptr[1:] = torch.cumsum(counts, 0)
        return z.to(torch.int32).contiguous(), pos.detach().to(torch.float32).contiguous(), mol_ptr, n_mol, max_atoms

    def _train_with(self, runner: "GemNetOCRunner", data):
        """Training mode: (energy, forces) attached to ONE autograd node over the flat export of the parameters (direct forces: first-order
        back-propagation from dLoss/dE and dLoss/dF, as the reference's loss.backward())."""
        z, pos, mol_ptr, n_mol, max_atoms = self._batch_args(data)
        buf, offs, scales = self.export(pos.device, detach=False)
        return GemNetOCFn.apply(runner, self, offs, scales, z, pos, mol_ptr, n_mol, max_atoms, buf)

    def _forward_with(self, runner: "GemNetOCRunner", data):
        """Host side of forward(): (re-)export the weights when a parameter changed, molecule pointers, the two-phase engine call."""
        self._sync_weights(runner, data.pos.device)
        z, pos, mol_ptr, n_mol, max_atoms = self._batch_args(data)
        return runner.run(z, pos, mol_ptr, n_mol, max_atoms)


class GemNetOCRunner(EngineDriver):
    """Host driver of `nb200_gemnet_oc_*`: owns the engine handle, the exported weights, the graph buffers and the workspaces."""

    def __init__(self, lib=None):
        super().__init__(lib)
        self._w = None
        self._keep = None
        self._status = None
        self.last_counts: Dict[str, int] = {}

    def set_weights(self, model: GemNetOC, device):
        self.set_weights_from(model, *model.export(device))

    def set_weights_from(self, model: GemNetOC, buf: torch.Tensor, offs: List[int], scales: List[float]):
        off_arr = (c_int64 * len(offs))(*offs)
        sc_arr = (c_float * len(scales))(*scales)
        w = GemNetOCWeights(model.num_blocks, model.num_elements, model.cutoff, model.max_neighbors, model.max_neighbors_qint, model.max_neighbors_aeaint,
                            buf.data_ptr(), ctypes.cast(off_arr, POINTER(c_int64)), ctypes.cast(sc_arr, POINTER(c_float)))
        self._w, self._keep = w, (buf, off_arr, sc_arr)

    def _graph(self, pos, mol_ptr, n_mol: int, max_atoms_per_mol: int, attr: str = "_graph_buf"):
        """Phase one of a two-phase call: the four graphs in the buffer `self.<attr>` and their counts (one synchronisation)."""
        n = int(pos.shape[0])
        gbuf = self._buffer(attr, self._graph_bytes(n, max_atoms_per_mol), pos.device)
        counts = (c_int64 * N_COUNTS)()
        check(self.lib.nb200_gemnet_oc_graph_count(byref(self._w), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, max_atoms_per_mol, gbuf.data_ptr(),
                                                   gbuf.numel(), counts, self._stream()), "nb200_gemnet_oc_graph_count")
        self.last_counts = {k: int(counts[i]) for i, k in enumerate(C_NAMES)}
        return gbuf, counts

    def _graph_bytes(self, n: int, max_atoms_per_mol: int) -> int:
        return self._bytes("nb200_gemnet_oc_graph_bytes", n, max_atoms_per_mol)

    def run_train(self, z, pos, mol_ptr, n_mol: int, max_atoms_per_mol: int, seed_energy=None, seed_forces=None, keep: bool = False):
        """nb200_gemnet_oc_energy_forces_grads with the weights bound by set_weights_from.
        seeds given: -> (energy, forces, flat gradient).  No seeds: forward only -> (energy, forces, None), or with keep=True
        -> (energy, forces, (token, gradient buffer)): the engine keeps the tape and `backward(token, ...)` fills the buffer without
        recomputing the forward.  Training has its own graph buffer and workspace so that an inference call in between cannot disturb a kept
        forward."""
        if self._w is None:
            raise NablaB200Error("GemNetOCRunner.run_train before set_weights")
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        self._check_seeds(seed_energy, seed_forces, n_mol, n, dev)
        buf = self._keep[0]
        gbuf, counts = self._graph(pos, mol_ptr, n_mol, max_atoms_per_mol, "_train_graph_buf")
        ws = self._buffer("_train_ws", self._bytes("nb200_gemnet_oc_train_workspace_bytes", byref(self._w), n_mol, n, counts), dev)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n, 3, dtype=torch.float32, device=dev)
        seeded = seed_energy is not None or seed_forces is not None
        grads = torch.empty_like(buf) if (seeded or keep) else None
        token = c_int64(0)
        check(lib.nb200_gemnet_oc_energy_forces_grads(
            self._h, byref(self._w), buf.numel(), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, max_atoms_per_mol, gbuf.data_ptr(), gbuf.numel(),
            counts, ws.data_ptr(), ws.numel(), seed_energy.data_ptr() if seed_energy is not None else None,
            seed_forces.data_ptr() if seed_forces is not None else None, grads.data_ptr() if grads is not None else None, energy.data_ptr(), forces.data_ptr(),
            byref(token) if (keep and not seeded) else None, self._stream()), "nb200_gemnet_oc_energy_forces_grads")
        if keep and not seeded:
            return energy, forces, (int(token.value), grads)
        return energy, forces, grads

    def run_hvp(self, z, pos, mol_ptr, n_mol: int, v, with_forces: bool = True):
        """Exact force-Jacobian products (nb200_gemnet_oc_jvp): v [n_dir, N, 3] (or [N, 3]) fp32 in Angstrom.  Returns (energy [B], forces
        [N, 3] or None, jv [n_dir, N, 3]) with jv = -(dF/dR) v in Ha/A, F the direct forces, and energy / forces bitwise those of `run_train`
        without seeds.  The direct forces are not a gradient, so this Jacobian is not symmetric (`vibrations.hessians` reports its symmetric
        part, as ASE `Vibrations` does with finite differences); the name is the one `vibrations` calls for every model.  Builds the graph
        (one synchronisation for the counts), then one call.  The workspace holds every activation of the training forward twice (44 GB for
        32 molecules of 10-30 heavy atoms).  It is a buffer of its own, kept for the next call until `release_hvp_workspace()`
        (`vibrations.hessians` releases it when it is done); a batch whose workspace does not fit raises NablaB200Error: split it by
        molecules."""
        if self._w is None:
            raise NablaB200Error("GemNetOCRunner.run_hvp before set_weights")
        lib, n, dev = self.lib, int(z.shape[0]), pos.device
        v = self._directions(v, n, dev)
        n_dir = int(v.shape[0])
        ptr_host = mol_ptr.cpu()
        max_atoms = int((ptr_host[1:] - ptr_host[:-1]).max())
        gbuf, counts = self._graph(pos, mol_ptr, n_mol, max_atoms)
        self.last_workspace_bytes = self._bytes("nb200_gemnet_oc_jvp_workspace_bytes", byref(self._w), n_mol, n, counts)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n, 3, dtype=torch.float32, device=dev) if with_forces else None
        jv = torch.empty(n_dir, n, 3, dtype=torch.float32, device=dev)
        try:
            ws = self._buffer("_jvp_ws", self.last_workspace_bytes, dev)
        except torch.cuda.OutOfMemoryError as exc:
            raise NablaB200Error(f"GemNetOC run_hvp: the workspace for these {n_mol} molecules ({n} atoms) needs {self.last_workspace_bytes / 1e9:.1f} GB, "
                                 "more than the device has free; split the batch by molecules") from exc
        check(lib.nb200_gemnet_oc_jvp(self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, max_atoms, gbuf.data_ptr(),
                                      gbuf.numel(), counts, ws.data_ptr(), ws.numel(), n_dir, v.data_ptr(), energy.data_ptr(),
                                      None if forces is None else forces.data_ptr(), jv.data_ptr(), self._stream()), "nb200_gemnet_oc_jvp")
        return energy, forces, jv

    def release_hvp_workspace(self):
        """Hand the workspace of `run_hvp` (tens of GB for a few dozen molecules) back to the allocator."""
        self._jvp_ws = None

    def backward(self, token: int, seed_energy, seed_forces) -> bool:
        """Replay the tape of the forward kept under `token` into the gradient buffer handed out by that forward.  False: the engine no
        longer holds it (another training forward ran on this runner) -- the caller recomputes."""
        rc = self.lib.nb200_gemnet_oc_backward(self._h, token, seed_energy.data_ptr() if seed_energy is not None else None,
                                               seed_forces.data_ptr() if seed_forces is not None else None, self._stream())
        if rc == -1:
            return False
        check(rc, "nb200_gemnet_oc_backward")
        return True

    def run(self, z, pos, mol_ptr, n_mol: int, max_atoms_per_mol: int, return_h: bool = False):
        if self._w is None:
            raise NablaB200Error("GemNetOCRunner.run before set_weights")
        lib, n = self.lib, int(z.shape[0])
        s = self._stream()
        gbuf, counts = self._graph(pos, mol_ptr, n_mol, max_atoms_per_mol)
        ws = self._buffer("_ws", self._bytes("nb200_gemnet_oc_workspace_bytes", byref(self._w), n_mol, n, counts), pos.device)
        energy = torch.empty(n_mol, dtype=torch.float32, device=pos.device)
        forces = torch.empty(n, 3, dtype=torch.float32, device=pos.device)
        check(lib.nb200_gemnet_oc_energy_forces(self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, max_atoms_per_mol,
                                                gbuf.data_ptr(), gbuf.numel(), counts, ws.data_ptr(), ws.numel(), energy.data_ptr(), forces.data_ptr(), s),
              "nb200_gemnet_oc_energy_forces")
        if return_h:
            h = torch.empty(n, 256, dtype=torch.float32, device=pos.device)
            check(lib.nb200_gemnet_oc_debug_h(ws.data_ptr(), byref(self._w), n_mol, n, counts, h.data_ptr(), s), "nb200_gemnet_oc_debug_h")
            return energy, forces, h
        return energy, forces

    def count_bounds(self, sizes):
        """Upper bounds of the five counts for molecules of `sizes` atoms (host): they hold for every geometry, see DESIGN.md 3.9."""
        return self._count_bounds("nb200_gemnet_oc", sizes, N_COUNTS)

    def launch(self, z, pos, mol_ptr, n_mol: int, max_atoms_per_mol: int, bounds):
        """Asynchronous forward (nb200_gemnet_oc_energy_forces_async) sized by n_atoms, the largest molecule and `bounds` (count_bounds):
        see `EngineDriver._launch_bounded`."""
        return self._launch_bounded("nb200_gemnet_oc", z, pos, mol_ptr, n_mol, bounds, max_atoms_per_mol)


class GemNetOCEngine(BoundedEngine):
    """`BoundedEngine` of GemNet-OC: bounds of the five counts; the launch also takes the largest molecule."""

    label = "GemNetOC"
    einval_text = "non-finite atom coordinates"
    count_names = C_NAMES

    @staticmethod
    def check_sizes(model: GemNetOC, max_atoms: int) -> None:
        """Refuse a molecule of more than `max_neighbors_aint` + 1 atoms."""
        if max_atoms - 1 > model.max_neighbors_aint:
            raise NablaB200Error(f"GemNetOC: a molecule has {max_atoms} atoms, more than max_neighbors_aint + 1 = {model.max_neighbors_aint + 1}; "
                                 "the atom-atom graph of the compiled path keeps every in-cutoff pair")

    @staticmethod
    def size_args(max_atoms: int) -> tuple:
        return (max_atoms,)


class GemNetOCFn(torch.autograd.Function):
    """(energy, forces) = f(flat weights).  forward runs the training engine and asks it to keep its tape; backward replays the tape with
    dLoss/dE, dLoss/dF (no forward recompute).  If another training forward ran on the same runner in between, backward falls back to the
    one-call form (forward + backward)."""

    @staticmethod
    def forward(ctx, runner, model, offs, scales, z, pos, mol_ptr, n_mol, max_atoms, buf):
        flat = buf.detach().contiguous()
        runner.set_weights_from(model, flat, offs, scales)
        energy, forces, (token, gbuf) = runner.run_train(z, pos, mol_ptr, n_mol, max_atoms, keep=True)
        ctx.args = (runner, model, offs, scales, n_mol, max_atoms, flat, token, gbuf)
        ctx.save_for_backward(z, pos, mol_ptr)
        ctx.set_materialize_grads(False)
        return energy, forces

    @staticmethod
    def backward(ctx, g_energy, g_forces):
        if g_energy is None and g_forces is None:
            return (None,) * 10
        runner, model, offs, scales, n_mol, max_atoms, flat, token, gbuf = ctx.args
        z, pos, mol_ptr = ctx.saved_tensors
        se = g_energy.to(torch.float32).contiguous() if g_energy is not None else None
        sf = g_forces.to(torch.float32).contiguous() if g_forces is not None else None
        if runner.backward(token, se, sf):
            return (None,) * 9 + (gbuf,)
        runner.set_weights_from(model, flat, offs, scales)  # the runner was re-bound since: recompute
        _, _, grads = runner.run_train(z, pos, mol_ptr, n_mol, max_atoms, se, sf)
        return (None,) * 9 + (grads,)


def header_enum_names(header_text: str, prefix: str) -> List[str]:
    """Names of the `NB200_GOC_<prefix>_*` enumerators in declaration order (used by tests/test_host.py to keep this file in step)."""
    names = re.findall(r"\bNB200_GOC_" + prefix + r"_([A-Z0-9_]+)\b\s*(?:=\s*\d+)?\s*,", re.sub(r"/\*.*?\*/", "", header_text, flags=re.S))
    out = []
    for nme in names:
        if nme != "COUNT" and nme not in out:
            out.append(nme)
    return out
