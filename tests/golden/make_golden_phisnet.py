"""Golden vectors for the PhiSNet pair-mixing / self-mixing / spherical-linear layers (SURVEY.md section 8 f4): the REFERENCE'S OWN
MODULES (`/root/reference/nablaDFT/phisnet/nn/modules/{pair_mixing,self_mixing,spherical_linear,clebsch_gordan}.py`, unmodified; they need
torch and numpy only) executed in the build container.  The modules are loaded by file path under a synthetic package so that
`nablaDFT/__init__.py` (which imports every model family and its missing third-party wheels) never runs.

Writes
  tests/golden/phisnet_cg_L4.npz   real Clebsch-Gordan tensors of the reference's vendored table
                                   (`clebsch_gordan_coefficients_L10.npz`) for every (l1, l2, l3) with l <= 4 that satisfies the triangle
                                   rule, in the module's own index order (all permutations expanded as `ClebschGordan.__init__` does)
  tests/golden/phisnet_mixing.npz  seeded inputs and the modules' outputs, float64; the weights are the name-keyed seeded ones of weights.py
                                   (`golden_state_dict({tag + '.' + name: ...}, bias_std=0.05, weight_scale=1.0)`), rebuilt by the tests

    python tests/golden/make_golden_phisnet.py
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from weights import golden_state_dict  # noqa: E402

MOD_DIR = "/root/reference/nablaDFT/phisnet/nn/modules"


def ref_modules():
    pkg = types.ModuleType("refphis")
    pkg.__path__ = [MOD_DIR]
    sys.modules["refphis"] = pkg
    return {n: importlib.import_module("refphis." + n) for n in ("clebsch_gordan", "pair_mixing", "self_mixing", "spherical_linear")}


def load_weights(mod, seed_prefix):
    sd = mod.state_dict()
    new = golden_state_dict({seed_prefix + k: v for k, v in sd.items() if not k.startswith("clebsch_gordan") and ".clebsch_gordan" not in k},
                            bias_std=0.05, weight_scale=1.0)
    for k in sd:
        if seed_prefix + k in new:
            sd[k] = torch.from_numpy(new[seed_prefix + k]).double().reshape(sd[k].shape)
    mod.load_state_dict(sd, strict=True)
    return sorted(k for k in sd if "clebsch_gordan" not in k)  # weights are NOT stored: tests rebuild them from the same names (weights.py)


def feats(gen, n, order, F):
    return [torch.randn(1, n, 2 * L + 1, F, generator=gen, dtype=torch.float64) for L in range(order + 1)]


def main():
    m = ref_modules()
    cg = m["clebsch_gordan"].ClebschGordan().double()
    table = {}
    for l1 in range(5):
        for l2 in range(5):
            for l3 in range(abs(l1 - l2), min(l1 + l2, 4) + 1):
                table[f"{l1}_{l2}_{l3}"] = cg(l1, l2, l3).numpy().astype(np.float64)
    np.savez_compressed(os.path.join(HERE, "phisnet_cg_L4.npz"), **table)

    out = {}
    gen = torch.Generator().manual_seed(7)
    F, K, P, N = 128, 128, 4, 3
    # PairMixing as the interaction block uses it (order 4 x order 4 -> order 4, distance-dependent coefficients), and a ragged variant
    for tag, (o1, o2, oo) in {"pair444": (4, 4, 4), "pair214": (2, 1, 4)}.items():
        pm = m["pair_mixing"].PairMixing(o1, o2, oo, K, F, cg).double()
        w = load_weights(pm, tag + ".")
        x1, x2 = feats(gen, P, o1, F), feats(gen, P, o2, F)
        rbf = torch.rand(1, P, 1, K, generator=gen, dtype=torch.float64)
        ys = pm(x1, x2, rbf)
        for L, t in enumerate(x1):
            out[f"{tag}/x1/{L}"] = t.numpy()
        for L, t in enumerate(x2):
            out[f"{tag}/x2/{L}"] = t.numpy()
        out[f"{tag}/rbf"] = rbf.numpy()
        for L, t in enumerate(ys):
            out[f"{tag}/y/{L}"] = t.detach().numpy()
    for tag, (oi, oo) in {"self44": (4, 4), "self42": (4, 2), "self24": (2, 4)}.items():
        sm = m["self_mixing"].SelfMixing(oi, oo, F, cg).double()
        w = load_weights(sm, tag + ".")
        xs = feats(gen, N, oi, F)
        ys = sm(xs)
        for L, t in enumerate(xs):
            out[f"{tag}/x/{L}"] = t.numpy()
        for L, t in enumerate(ys):
            out[f"{tag}/y/{L}"] = t.detach().numpy()
    for tag, (oi, fi, oo, fo, mix) in {"lin44": (4, F, 4, F, True), "lin40": (4, F, 0, 64, True), "lin22n": (2, F, 2, 64, False)}.items():
        sl = m["spherical_linear"].SphericalLinear(oi, fi, oo, fo, cg, mix_orders=mix, bias=True).double()
        w = load_weights(sl, tag + ".")
        xs = feats(gen, N, oi, fi)
        ys = sl(xs)
        for L, t in enumerate(xs):
            out[f"{tag}/x/{L}"] = t.numpy()
        for L, t in enumerate(ys):
            out[f"{tag}/y/{L}"] = t.detach().numpy()
    # every layer acts row by row (pair / atom), so the stored pair rows are cut to the first 3 of the 4 generated: the file stays under 1 MB
    out = {k: np.ascontiguousarray(v[:, :3]) if k.startswith("pair") else v for k, v in out.items()}
    np.savez_compressed(os.path.join(HERE, "phisnet_mixing.npz"), **out)
    print("wrote phisnet_cg_L4.npz (%d tensors) and phisnet_mixing.npz (%d arrays)" % (len(table), len(out)))


if __name__ == "__main__":
    main()
