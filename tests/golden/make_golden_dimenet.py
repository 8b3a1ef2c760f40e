"""Golden vectors for DimeNet++ (config/model/dimenetplusplus.yaml) from the REFERENCE'S OWN wrapper
`nablaDFT/dimenetplusplus/dimenetplusplus.py` (unmodified, imported where it lies) on fixture molecules, in float64.

Shims: `pytorch_lightning` and `torch_geometric.data.Data` become attribute bags, and `torch_geometric.nn.models.DimeNetPlusPlus` is the
oracle's restatement (oracle/dimenet.py), since torch-geometric is not installed.  So this file pins the WRAPPER (regression head, scaler
after the gradient, force sign and scaling, parameter names) to the reference's code and pins the oracle against later drift; it cannot
pin the PyG core.

Test weights: `dimenet_test_state_dict`, shared with the tests.  PyG's initialiser zeroes each output block's `lin`, which would make every
energy a constant and every force 0, so the weights come from weights.py::golden_state_dict with two of its name heuristics overridden here
(existing goldens depend on weights.py as it is): `net.emb.lin*` would get the uniform(+-sqrt 3) embedding draw, and `net.rbf.freq` the small
bias noise.

    python tests/golden/make_golden_dimenet.py      # writes tests/golden/dimenet_f64.npz
"""
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
from weights import golden_state_dict  # noqa: E402

REF = "/root/reference/nablaDFT/dimenetplusplus/dimenetplusplus.py"
MOLS = [0, 7, 23]
SCALER = {"scale_": 0.870582896669776, "mean_": -7.349405628928332}  # config/model/dimenetplusplus.yaml


def dimenet_test_state_dict(template: dict, weight_scale: float = 0.85) -> dict:
    """name -> float64 ndarray for every entry of `template` (a DimeNetPlusPlusPotential state dict).  weight_scale 0.85 gives unscaled
    predictions that vary by about 1 Ha between fixture molecules and forces up to about 0.5 Ha/A (0.5: 1e-4 Ha/A, 1.0: 200 Ha/A)."""
    out = golden_state_dict(template, bias_std=0.02, weight_scale=weight_scale)
    for name in ("net.emb.lin.weight", "net.emb.lin_rbf.weight"):
        shape = tuple(template[name].shape)
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        bound = np.sqrt(6.0 / (shape[0] + shape[1])) * weight_scale
        out[name] = rng.uniform(-bound, bound, size=shape)
    rng = np.random.default_rng(zlib.crc32(b"net.rbf.freq"))
    n = int(template["net.rbf.freq"].shape[0])
    out["net.rbf.freq"] = np.pi * np.arange(1, n + 1) * (1.0 + 0.02 * rng.standard_normal(n))
    return out


def load_test_weights(module: torch.nn.Module, dtype=torch.float64):
    sd = module.state_dict()
    for k, v in dimenet_test_state_dict(sd).items():
        sd[k] = torch.from_numpy(np.asarray(v)).to(dtype).reshape(sd[k].shape)
    module.load_state_dict(sd, strict=True)
    return module


def grid_molecule():
    """48 atoms on a 4 x 4 x 3 grid of 1 A: every pair is inside 5 A, so with K = 32 atoms 0..32 are among their own first K + 1
    candidates and keep 32 sources, atoms 33..47 are not and keep 33.  Many triplets are exactly collinear."""
    g = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(3), indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    z = np.array([6, 1, 8, 1, 7, 1][:3] * 16, dtype=np.int32)
    return z, g


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _Data:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def main():
    import importlib.util

    from oracle.dimenet import DimeNetPlusPlus

    _mod("pytorch_lightning", LightningModule=torch.nn.Module)
    _mod("torch_geometric")
    _mod("torch_geometric.data", Data=_Data)
    _mod("torch_geometric.nn")
    _mod("torch_geometric.nn.models", DimeNetPlusPlus=DimeNetPlusPlus)
    spec = importlib.util.spec_from_file_location("ref_dimenetplusplus", REF)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    import yaml

    cfg = yaml.safe_load(open("/root/reference/config/model/dimenetplusplus.yaml"))["net"]
    cfg.pop("_target_")
    torch.manual_seed(0)
    net = ref.DimeNetPlusPlusPotential(**cfg).double().eval()
    load_test_weights(net)
    fx = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    z, pos, batch = [], [], []
    for k, m in enumerate(MOLS):
        a, e = fx["ptr"][m], fx["ptr"][m + 1]
        z.append(fx["z"][a:e]); pos.append(fx["pos"][a:e]); batch.append(np.full(e - a, k))
    z, pos, batch = np.concatenate(z), np.concatenate(pos).astype(np.float32), np.concatenate(batch)
    data = _Data(z=torch.from_numpy(z).long(), pos=torch.from_numpy(pos.astype(np.float64)), batch=torch.from_numpy(batch).long())
    energy, forces = net(data)
    g = net.net(pos=data.pos, z=data.z, batch=data.batch)
    assert cfg["scaler"] == SCALER and cfg["do_postprocessing"]
    np.savez_compressed(os.path.join(HERE, "dimenet_f64.npz"), z=z.astype(np.int32), pos=pos, batch=batch.astype(np.int64),
                        energy=energy.detach().numpy(), forces=forces.detach().numpy(), graph_emb=g.detach().numpy())
    print("energy", energy.detach().numpy(), "max|F|", float(forces.abs().max()))


if __name__ == "__main__":
    main()
