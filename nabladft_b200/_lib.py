"""ctypes binding of the C ABI declared in `include/nabla_b200.h`.

This is the reference-side stub a nablaDFT maintainer would add (see INTEGRATION.md): plain
pointers and sizes, `torch.Tensor.data_ptr()` for device memory, the current CUDA stream.
There is NO fallback: if the shared library is missing or a call fails, we raise.
"""
import ctypes
import os
from ctypes import c_double, POINTER, c_float, c_int32, c_int64, c_uint64, c_void_p

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

    "nb200_gemnet_oc_graph_bytes": (c_int64, [c_int32, c_int32]),
    "nb200_gemnet_oc_graph_count": (c_int32, [POINTER(GemNetOCWeights), c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64,
                                              POINTER(c_int64), c_void_p]),
    "nb200_gemnet_oc_workspace_bytes": (c_int64, [POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_energy_forces": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                c_void_p, c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "nb200_gemnet_oc_debug_h": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64), c_void_p, c_void_p]),
    "nb200_schnet_train_count": (c_int32, [POINTER(SchnetWeights), c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, POINTER(c_int64), c_void_p]),
    "nb200_schnet_train_workspace_bytes": (c_int64, [POINTER(SchnetWeights), c_int32, c_int32, c_int64, c_int32]),
    "nb200_schnet_energy_grads": (c_int32, [c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_void_p,
                                            c_int64, c_void_p, c_void_p, POINTER(SchnetWeights), c_void_p, c_void_p]),
    "nb200_gemnet_oc_train_workspace_bytes": (c_int64, [POINTER(GemNetOCWeights), c_int32, c_int32, POINTER(c_int64)]),
    "nb200_gemnet_oc_energy_forces_grads": (c_int32, [c_void_p, POINTER(GemNetOCWeights), c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                                      c_void_p, c_int64, POINTER(c_int64), c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                      POINTER(c_int64), c_void_p]),
    "nb200_gemnet_oc_backward": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
}

_lib = None


class NablaB200Error(RuntimeError):
    pass


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
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


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
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
