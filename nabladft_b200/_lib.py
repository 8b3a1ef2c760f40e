"""ctypes binding of the C ABI declared in `include/nabla_b200.h`.

This is the reference-side stub a nablaDFT maintainer would add (see INTEGRATION.md): plain
pointers and sizes, `torch.Tensor.data_ptr()` for device memory, the current CUDA stream.
There is NO fallback: if the shared library is missing or a call fails, we raise.
"""
import ctypes
import os
from ctypes import c_double, POINTER, byref, c_float, c_int32, c_int64, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnabla_b200.so")

NB200_OK = 0
ERRORS = {
    -1: "NB200_EINVAL (bad argument)",
    -2: "NB200_EUNSUPPORTED (configuration outside the compiled fast path)",
    -3: "NB200_ECUDA (CUDA runtime / cuBLAS error)",
    -4: "NB200_ECAPACITY (edge capacity exceeded)",
    -5: "NB200_ENEIGHBORS (an atom has more than max_neighbors neighbours)",
    -6: "NB200_ENOEDGES (an atom has no neighbours)",
}
RADIAL_SPK, RADIAL_OC = 0, 1

_fp = POINTER(c_float)


class PainnWeights(ctypes.Structure):
    """Mirror of `struct nb200_painn_weights` (include/nabla_b200.h)."""

    _fields_ = [
        ("n_layers", c_int32), ("n_feat", c_int32), ("n_rbf", c_int32), ("n_elem", c_int32),
        ("radial_mode", c_int32), ("z_offset", c_int32),
        ("cutoff", c_float), ("epsilon", c_float),
        ("rbf_coeff", c_float), ("rbf_xscale", c_float),
        ("rbf_offsets", c_void_p),
        ("energy_shift_per_atom", c_float),
        ("max_neighbors", c_int32),
        ("emb", c_void_p), ("w_rbf", c_void_p), ("b_rbf", c_void_p),
        ("A1", c_void_p), ("c1", c_void_p), ("A2", c_void_p), ("c2", c_void_p),
        ("U", c_void_p),
        ("B1", c_void_p), ("d1", c_void_p), ("B2", c_void_p), ("d2", c_void_p),
        ("R1", c_void_p), ("e1", c_void_p), ("R2", c_void_p), ("e2", c_void_p),
    ]


class SchnetWeights(ctypes.Structure):
    """Mirror of `struct nb200_schnet_weights` (include/nabla_b200.h)."""

    _fields_ = [
        ("n_layers", c_int32), ("n_feat", c_int32), ("n_rbf", c_int32), ("n_elem", c_int32),
        ("z_offset", c_int32),
        ("cutoff", c_float), ("rbf_coeff", c_float),
        ("energy_shift_per_atom", c_float),
        ("rbf_offsets", c_void_p),
        ("emb", c_void_p),
        ("w_f1", c_void_p), ("b_f1", c_void_p), ("W_f2", c_void_p), ("b_f2", c_void_p),
        ("I1", c_void_p),
        ("P1", c_void_p), ("p1", c_void_p), ("P2", c_void_p), ("p2", c_void_p),
        ("R1", c_void_p), ("e1", c_void_p), ("R2", c_void_p), ("e2", c_void_p),
    ]


# name -> (restype, argtypes); every symbol declared in include/nabla_b200.h
class GemNetOCWeights(ctypes.Structure):
    """Mirror of `struct nb200_gemnet_oc_weights` (include/nabla_b200.h)."""

    _fields_ = [("num_blocks", c_int32), ("n_elem", c_int32), ("cutoff", c_float), ("max_neighbors", c_int32), ("max_neighbors_qint", c_int32),
                ("max_neighbors_aeaint", c_int32), ("w", c_void_p), ("off_host", POINTER(c_int64)), ("scale_host", POINTER(c_float))]


class GemNetOCAggArgs(ctypes.Structure):
    """Mirror of `struct nb200_gemnet_oc_agg_args` (include/nabla_b200.h)."""

    _fields_ = [("quad", c_int32), ("form", c_int32), ("tangent", c_int32), ("ldr", c_int32), ("E_bound", c_int64), ("E_dev", c_void_p),
                ("o_ptr", c_void_p), ("o_src", c_void_p), ("o_tgt", c_void_p), ("o_V", c_void_p), ("in_ptr", c_void_p), ("in_src", c_void_p),
                ("in_V", c_void_p), ("q_tin", c_void_p), ("x", c_void_p), ("R", c_void_p), ("O", c_void_p), ("Vot", c_void_p), ("Vit", c_void_p),
                ("xt", c_void_p), ("Rt", c_void_p), ("Ot", c_void_p)]


class PainnTanArgs(ctypes.Structure):
    """Mirror of `struct nb200_painn_tan_args` (include/nabla_b200.h)."""

    _fields_ = [("op", c_int32), ("bf16", c_int32), ("tan", c_int32), ("n_atoms", c_int32), ("n", c_int64), ("width", c_int32), ("e_cap", c_int32)] + [
        (name, c_void_p) for name in (
            "row_ptr", "col", "rev", "status", "sort_scratch", "geom", "v", "t_geom", "xh", "t_xh", "xh_bias", "mu", "t_mu", "t_q", "t_mu_out",
            "W", "dW", "d2W", "g_q", "t_g_q", "g_mu", "t_g_mu", "t_g_xh", "t_g_mu_in", "gW", "t_gW", "gWd", "VW", "t_VW", "nrm", "y", "t_y",
            "gn", "t_gn", "t_nrm", "t_gy", "t_gVW", "pre", "t_pre", "x", "g_pre", "R2", "out", "t_g", "t_g_pre", "t_act", "egrad", "t_egrad", "hv")
    ] + [("radial_mode", c_int32), ("n_rbf", c_int32), ("n_layers", c_int32), ("cutoff", c_float), ("rbf_coeff", c_float), ("rbf_xscale", c_float),
         ("sign", c_float), ("rbf_offsets", c_void_p), ("w_rbf", c_void_p), ("b_rbf", c_void_p), ("g_w", c_void_p), ("g_b", c_void_p)]


# nb200_painn_test_tangent ops (enum NB200_PT_*)
PT_OPS = ("GEOM_TAN", "MUL_DACT", "ACT_BWD_TAN", "READOUT_BWD_TAN", "MSG_FWD_TAN", "UPD_NORM_TAN", "UPD_COMBINE_TAN", "UPD_COMBINE_BWD_TAN",
          "UPD_NORM_BWD_TAN", "MSG_BWD_TAN", "MSG_BWD_HVP", "EDGE_FORCES_HVP", "FILTER_D2", "FILTER_WGRAD")


class PainnNodeArgs(ctypes.Structure):
    """Mirror of `struct nb200_painn_node_args` (include/nabla_b200.h)."""

    _fields_ = [(name, c_int32) for name in ("op", "n_atoms", "tile", "layer_upd", "layer_mlp", "readout")] + [
        ("w", POINTER(PainnWeights))] + [(name, c_void_p) for name in (
            "wtiles", "q_mid", "mu_mid", "q_mlp_in", "g_xh", "VW", "nrm", "dot", "g1pre", "y", "q_next", "mu_next", "h1pre", "xh", "ro_pre",
            "gq_a", "gq_b", "cur", "gn", "gdot", "z", "mol_ptr", "status")] + [("n_mol", c_int32), ("kind", c_int32), ("n", c_int64)] + [
        (name, c_void_p) for name in ("gq", "gmu", "q", "mu", "g", "pre", "gy", "gVW", "eps_atom", "energy", "forces", "g_pre")]


# nb200_painn_test_node ops (enum NB200_PN_*)
PN_OPS = ("PREP", "NODE_FWD", "NODE_BWD", "EMBED", "ACT_BWD", "UPD_COMBINE_BWD", "UPD_NORM_BWD", "READOUT", "MOL_SUM", "READOUT_BWD", "POISON")


class SchnetTestArgs(ctypes.Structure):
    """Mirror of `struct nb200_schnet_test_args` (include/nabla_b200.h)."""

    _fields_ = [(name, c_int32) for name in ("op", "n_layers", "n_rbf", "n_atoms", "n_edges", "e_stride", "m")] + [
        ("cutoff", c_float), ("rbf_coeff", c_float)] + [(name, c_void_p) for name in (
            "status", "row_ptr", "col", "sort_scratch", "geom", "rbf_offsets", "w_f1", "b_f1", "y", "G1", "G2", "b2", "gagg", "X", "W", "bias",
            "HH", "agg", "gy", "egrad", "Y", "act")]


# nb200_schnet_test_op ops (enum NB200_SC_*)
SC_OPS = ("FILTER1", "CFCONV_FWD", "CFCONV_BWD", "LINEAR_ACT")


class DimeNetWeights(ctypes.Structure):
    """Mirror of `struct nb200_dimenet_weights` (include/nabla_b200.h)."""

    _fields_ = [("num_blocks", c_int32), ("node_latent_dim", c_int32), ("hidden", c_int32), ("int_emb", c_int32), ("basis_emb", c_int32),
                ("out_emb", c_int32), ("num_spherical", c_int32), ("num_radial", c_int32), ("num_before_skip", c_int32), ("num_after_skip", c_int32),
                ("num_output_layers", c_int32), ("envelope_exponent", c_int32), ("max_neighbors", c_int32), ("cutoff", c_float), ("scale", c_float),
                ("mean", c_float), ("w", c_void_p), ("off_host", POINTER(c_int64))]


SIGNATURES = {
    "nb200_version": (c_int32, []),
    "nb200_last_cuda_error": (c_int32, []),
    "nb200_neighbor_build": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_float, c_int32, c_int32,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_filter": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                     c_float, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_msg_fwd": (c_int32, [c_void_p] * 8 + [c_int32, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_msg_bwd": (c_int32, [c_void_p] * 8 + [c_int32] + [c_void_p] * 6),
    "nb200_edge_forces": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p]),
    "nb200_painn_msg_fwd_ex": (c_int32, [c_void_p] * 5 + [c_int32] + [c_void_p] * 4 + [c_int32] + [c_void_p] * 2 + [c_int32, c_void_p]),
    "nb200_painn_msg_bwd_ex": (c_int32, [c_void_p] * 5 + [c_int32] + [c_void_p] * 4 + [c_int32] + [c_void_p] * 7 + [c_int32, c_void_p]),
    "nb200_msg_gather_probe": (c_int32, [c_void_p] * 3 + [c_int32] + [c_void_p] * 3 + [c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_engine_create": (c_int32, [POINTER(c_void_p)]),
    "nb200_engine_destroy": (c_int32, [c_void_p]),
    "nb200_engine_set_timing": (c_int32, [c_void_p, c_int32]),
    "nb200_engine_read_timings": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32]),
    "nb200_engine_own_launches": (c_int64, [c_void_p]),
    "nb200_engine_set_gemm_backend": (c_int32, [c_void_p, c_int32]),
    "nb200_engine_set_node_backend": (c_int32, [c_void_p, c_int32]),
    "nb200_phis_n_paths": (c_int32, [c_int32, c_int32, c_int32, c_int32]),
    "nb200_phis_pair_mixing": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_self_mixing": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_linear": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_swish_self_mixing": (c_int32, [c_void_p] * 5 + [c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_linear_ex": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_interaction": (c_int32, [c_void_p] * 10 + [c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_pair_features": (c_int32, [c_void_p] * 5 + [c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "nb200_phis_overlap_pairs": (c_int32, [c_void_p] * 6 + [c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_phis_assemble": (c_int32, [c_void_p] * 4 + [c_int32] + [c_void_p] * 2 + [c_int32, c_int32] + [c_void_p] * 9 + [c_int32, c_int32]
                            + [c_void_p] * 3 + [c_int32, c_int32] + [c_void_p] * 4 + [c_int32, c_void_p, c_void_p]),
    "nb200_gemm_tf32x3": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_int32,
                                    c_int32, c_void_p, c_void_p, c_void_p]),
    "nb200_gemm_tf32x3_rows": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_int32,
                                         c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_gemm_tf32x3_epi": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_int32,
                                        c_void_p, c_int32, c_int32, c_float, c_void_p]),
    "nb200_linear_wgrad": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int32, c_float,
                                     c_void_p, c_float, c_void_p, c_int32, c_void_p]),
    "nb200_qh_expand_rows": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p]),
    "nb200_qh_edge_basis": (c_int32, [c_void_p, c_void_p, c_int32, c_double, c_float, c_float, c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "nb200_qh_norm_feats": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p]),
    "nb200_qh_gate": (c_int32, [c_void_p, c_void_p, c_int32, c_void_p, c_void_p]),
    "nb200_qh_invariants": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_qh_tp_conv": (c_int32, [c_void_p] * 6 + [c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_qh_tp_pair": (c_int32, [c_void_p] * 6 + [c_int32, c_void_p, c_void_p]),
    "nb200_qh_tp_self": (c_int32, [c_void_p] * 4 + [c_int32, c_void_p, c_void_p]),
    "nb200_qh_linear": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_dense": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_int32, c_int32,
                              c_void_p, c_void_p, c_int32, c_void_p]),
    "nb200_qh_expand_setup": (c_int32, [c_void_p, c_void_p]),
    "nb200_qh_expand": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]),
    "nb200_qh_pair_hidden": (c_int32, [c_void_p] * 6 + [c_int32, c_void_p, c_void_p]),
    "nb200_qh_assemble": (c_int32, [c_void_p] * 6 + [c_int32, c_int32] + [c_void_p] * 8),
    "nb200_axpy": (c_int32, [c_void_p, c_void_p, c_int64, c_void_p]),
    "nb200_lbfgs_state_bytes": (c_int64, [c_int32, c_int32, c_int32]),
    "nb200_lbfgs_step": (c_int32, [c_void_p, c_int64, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_double, c_double, c_double,
                                   c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_qn_state_bytes": (c_int64, [c_int32, c_int32, c_int64]),
    "nb200_qn_step": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int64, c_double, c_int32] + [c_double] * 7
                      + [c_void_p] * 8),
    "nb200_md_init_momenta": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_double, c_uint64, c_int64, c_void_p, c_void_p]),
    "nb200_md_step": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_double, c_double, c_double, c_uint64, c_int64, c_double, c_double]
                      + [c_void_p] * 11),
    "nb200_painn_workspace_bytes": (c_int64, [POINTER(PainnWeights), c_int32, c_int32, c_int32, c_int32]),
    "nb200_schnet_workspace_bytes": (c_int64, [POINTER(SchnetWeights), c_int32, c_int32, c_int32, c_int32]),
    "nb200_schnet_energy_forces": (c_int32, [c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                             c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_train_workspace_bytes": (c_int64, [POINTER(PainnWeights), c_int32, c_int32, c_int32, c_int32]),
    "nb200_painn_energy_forces_grads": (c_int32, [c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                  c_void_p, c_int64, c_void_p, c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_void_p,
                                                  c_void_p]),
    "nb200_engine_set_edge_storage": (c_int32, [c_void_p, c_int32]),
    "nb200_painn_train_forward": (c_int32, [c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                            c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_train_backward": (c_int32, [c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                             c_void_p, c_int64, c_int32, c_void_p, c_void_p, POINTER(PainnWeights), c_void_p, c_void_p]),
    "nb200_painn_energy_forces": (c_int32, [c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                            c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_hvp_workspace_bytes": (c_int64, [POINTER(PainnWeights), c_int32, c_int32, c_int32, c_int32]),
    "nb200_painn_hvp": (c_int32, [c_void_p, POINTER(PainnWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64,
                                  c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_painn_test_tangent": (c_int32, [POINTER(PainnTanArgs), c_void_p]),
    "nb200_painn_test_node": (c_int32, [POINTER(PainnNodeArgs), c_void_p]),
    "nb200_schnet_test_op": (c_int32, [POINTER(SchnetTestArgs), c_void_p]),

    "nb200_gemnet_oc_graph_bytes": (c_int64, [c_int32, c_int32]),
    "nb200_gemnet_oc_graph_count": (c_int32, [POINTER(GemNetOCWeights), c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64,
                                              POINTER(c_int64), c_void_p]),
    "nb200_gemnet_oc_workspace_bytes": (c_int64, [POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_energy_forces": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                c_void_p, c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "nb200_gemnet_oc_count_bounds": (c_int32, [POINTER(GemNetOCWeights), POINTER(c_int32), c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_energy_forces_async": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                      c_void_p, c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_gemnet_oc_debug_h": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64), c_void_p, c_void_p]),
    "nb200_gemnet_oc_test_aggregate": (c_int32, [POINTER(GemNetOCAggArgs), c_void_p]),
    "nb200_schnet_train_count": (c_int32, [POINTER(SchnetWeights), c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, POINTER(c_int64), c_void_p]),
    "nb200_schnet_train_workspace_bytes": (c_int64, [POINTER(SchnetWeights), c_int32, c_int32, c_int64, c_int32]),
    "nb200_schnet_energy_grads": (c_int32, [c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_void_p,
                                            c_int64, c_void_p, c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p]),
    "nb200_schnet_hvp_workspace_bytes": (c_int64, [POINTER(SchnetWeights), c_int32, c_int32, c_int64]),
    "nb200_schnet_hvp": (c_int32, [c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_void_p,
                                   c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_gemnet_oc_train_workspace_bytes": (c_int64, [POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_energy_forces_grads": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                      c_void_p, c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                      POINTER(c_int64), c_void_p]),
    "nb200_gemnet_oc_backward": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "nb200_gemnet_oc_jvp_workspace_bytes": (c_int64, [POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_jvp": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64,
                                      POINTER(c_int64), c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_graph_bytes": (c_int64, [POINTER(DimeNetWeights), c_int32]),
    "nb200_dimenet_graph_count": (c_int32, [POINTER(DimeNetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64,
                                            POINTER(c_int64), c_void_p]),
    "nb200_dimenet_workspace_bytes": (c_int64, [POINTER(DimeNetWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_dimenet_energy_forces": (c_int32, [c_void_p, POINTER(DimeNetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64,
                                              POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_count_bounds": (c_int32, [POINTER(DimeNetWeights), POINTER(c_int32), c_int32, POINTER(c_int64)]),
    "nb200_dimenet_energy_forces_async": (c_int32, [c_void_p, POINTER(DimeNetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p,
                                                    c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_train_workspace_bytes": (c_int64, [POINTER(DimeNetWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_dimenet_train_grads": (c_int32, [c_void_p, POINTER(DimeNetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64,
                                            POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_debug_sbf_radial": (c_int32, [POINTER(DimeNetWeights), c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_hvp_workspace_bytes": (c_int64, [POINTER(DimeNetWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_dimenet_hvp": (c_int32, [c_void_p, POINTER(DimeNetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64,
                                    POINTER(c_int64), c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_dimenet_debug_sbf_radial_d2": (c_int32, [POINTER(DimeNetWeights), c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
}

_lib = None


class NablaB200Error(RuntimeError):
    pass


def bind(lib, prefixes=None):
    """Attach the prototypes of SIGNATURES to `lib`: all of them, or those of the symbols whose names start with one of `prefixes` plus the
    engine handle's create / destroy (an emulation build of one engine exports only its own).  A declared symbol that `lib` does not export
    raises AttributeError."""
    for name, (res, args) in SIGNATURES.items():
        if prefixes is None or name.startswith(tuple(prefixes)) or name in ("nb200_engine_create", "nb200_engine_destroy"):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def load():
    """Load libnabla_b200.so (once). Raises if it has not been built -- never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NablaB200Error(
            f"{LIB_PATH} is missing: build it with `python -m nabladft_b200.build` "
            "(nvcc, sm_90a). There is no CPU / eager fallback for this path."
        )
    _lib = bind(ctypes.CDLL(LIB_PATH))
    return _lib


def check(rc: int, what: str):
    if rc != NB200_OK:
        detail = ERRORS.get(rc, f"error {rc}")
        cuda = load().nb200_last_cuda_error() if rc == -3 else 0
        raise NablaB200Error(f"{what} failed: {detail}" + (f" [cudaError {cuda}]" if cuda else ""))


def ptr(t):
    """Device pointer of a contiguous torch tensor (or None)."""
    if t is None:
        return None
    assert t.is_contiguous(), "C ABI takes contiguous buffers"
    return c_void_p(t.data_ptr())


def current_stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


class EngineDriver:
    """Host side of one `nb200_engine` handle, shared by the model drivers: the handle's lifecycle, the stream and device checks of their
    calls (`_stream`, `_on_device`: what the emulation tests replace), size queries and the growth of the buffers they size."""

    _ws = None  # the workspace every driver has (`_buffer("_ws", ...)` sizes it)
    SLACK = 1.25  # a grown buffer holds this many times the bytes asked for (+ 256): headroom for the next, slightly larger batch

    def __init__(self, lib=None):
        """`lib`: a bound library exporting the C ABI (default: libnabla_b200.so)."""
        self.lib = load() if lib is None else lib
        h = c_void_p()
        check(self.lib.nb200_engine_create(byref(h)), "nb200_engine_create")
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.nb200_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _stream(self):
        return current_stream()

    def _on_device(self, t) -> bool:
        return t.is_cuda

    def _bytes(self, fn_name: str, *args) -> int:
        """A size query of the C ABI; a negative return is its error code."""
        n = getattr(self.lib, fn_name)(*args)
        if n < 0:
            check(int(n), fn_name)
        return int(n)

    def _buffer(self, attr: str, nbytes: int, device):
        """The byte buffer `self.<attr>`, replaced by a larger one (the old one freed first) when it holds fewer than `nbytes` or sits on
        another device."""
        cur = getattr(self, attr, None)
        if cur is None or cur.numel() < nbytes or cur.device != device:
            setattr(self, attr, None)
            cur = torch.empty(int(nbytes * self.SLACK) + 256, dtype=torch.uint8, device=device)
            setattr(self, attr, cur)
        return cur

    def _check_seeds(self, seed, force_seed, n_mol: int, n_atoms: int, device) -> None:
        """The loss seeds of a gradient call, dLoss/dE [n_mol] and dLoss/dF [n_atoms, 3]; either may be None."""
        for t, n in ((seed, n_mol), (force_seed, 3 * n_atoms)):
            if t is not None and not (t.device == device and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n):
                raise NablaB200Error("seeds must be contiguous fp32 tensors [n_mol] / [n_atoms, 3] on the batch's device")

    def _directions(self, v, n_atoms: int, device):
        """The directions of a Hessian-vector-product call, v [n_atoms, 3] or [n_dir, n_atoms, 3], as [n_dir, n_atoms, 3]."""
        if v.dim() == 2:
            v = v.unsqueeze(0)
        if not (self._on_device(v) and v.device == device and v.dtype == torch.float32 and v.is_contiguous() and v.dim() == 3
                and v.shape[1:] == (n_atoms, 3) and v.shape[0] >= 1):
            raise NablaB200Error(f"run_hvp(): v must be a contiguous fp32 CUDA tensor [n_dir, {n_atoms}, 3] with n_dir >= 1 on {device}")
        return v

    # ---- forwards sized by per-batch upper bounds (DimeNet++, GemNet-OC): the C calls `<prefix>_count_bounds`, `<prefix>_graph_bytes`,
    # `<prefix>_workspace_bytes` and `<prefix>_energy_forces_async` on the weights the driver binds as `_w`
    def _count_bounds(self, prefix: str, sizes, n_counts: int):
        """Upper bounds of the `n_counts` counts for molecules of `sizes` atoms (host, `<prefix>_count_bounds`): they hold for every geometry."""
        if self._w is None:
            raise NablaB200Error(f"{type(self).__name__}.count_bounds before set_weights")
        mol_ptr = (c_int32 * (len(sizes) + 1))(0, *[int(v) for v in torch.as_tensor(sizes).cumsum(0)])
        bounds = (c_int64 * n_counts)()
        check(getattr(self.lib, prefix + "_count_bounds")(byref(self._w), mol_ptr, len(sizes), bounds), prefix + "_count_bounds")
        return bounds

    def _launch_bounded(self, prefix: str, z, pos, mol_ptr, n_mol: int, bounds, *size_args):
        """Asynchronous forward (`<prefix>_energy_forces_async`): one enqueue on the current stream, no host read.  -> (energy, forces,
        status); `status` is a device int32[8] that the next launch rewrites (include/nabla_b200.h).  `size_args`: the per-batch sizes the
        call takes after n_atoms (GemNet-OC: the largest molecule); the graph buffer holds `self._graph_bytes(n_atoms, *size_args)` bytes.
        Graph buffer and workspace are sized by n_atoms and `bounds`, hence once per batch: later launches of the same batch reuse them."""
        if self._w is None:
            raise NablaB200Error(f"{type(self).__name__}.launch before set_weights")
        n, dev = int(z.shape[0]), pos.device
        gbytes = self._graph_bytes(n, *size_args)
        self.last_workspace_bytes = self._bytes(prefix + "_workspace_bytes", byref(self._w), n_mol, n, bounds)
        gbuf, ws = self._buffer("_graph_buf", gbytes, dev), self._buffer("_ws", self.last_workspace_bytes, dev)
        if self._status is None or self._status.device != dev:
            self._status = torch.zeros(8, dtype=torch.int32, device=dev)
        energy = torch.empty(n_mol, dtype=torch.float32, device=dev)
        forces = torch.empty(n, 3, dtype=torch.float32, device=dev)
        check(getattr(self.lib, prefix + "_energy_forces_async")(
            self._h, byref(self._w), z.data_ptr(), pos.data_ptr(), mol_ptr.data_ptr(), n_mol, n, *size_args, gbuf.data_ptr(), gbuf.numel(),
            bounds, ws.data_ptr(), ws.numel(), energy.data_ptr(), forces.data_ptr(), self._status.data_ptr(), self._stream()),
            prefix + "_energy_forces_async")
        return energy, forces, self._status
