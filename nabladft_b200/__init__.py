"""nabladft_b200 -- H100-native (sm_90a) engine for nablaDFT's model-forward hot path.

Only what the path needs: `csrc/` (CUDA kernels + C ABI, built into libnabla_b200.so),
the ctypes binding (`_lib`), the engine driver and the host-side mirrors of the reference's
model interfaces (`painn_oc.PaiNN`, `spk.NeuralNetworkPotential`, `qhnet.QHNet`, `gemnet_oc.GemNetOC`), the training bridges
(`training`, `schnet_train`), the batched L-BFGS driver (`optimization`) and the data path (`data`).  No CPU fallback.
"""
from . import _lib  # noqa: F401
from .painn_oc import PaiNN  # noqa: F401

__all__ = ["PaiNN", "spk", "synth", "qhnet", "gemnet_oc", "training", "schnet_train", "optimization", "data", "losses", "parallel"]
