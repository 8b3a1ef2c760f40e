"""Golden vectors for GemNet-OC (SURVEY.md section 8 a19, BASELINE configs[4]) produced by the REFERENCE'S OWN CLASSES
(`/root/reference/nablaDFT/gemnet_oc/**`, unmodified, imported where they lie) on fixture molecules, in the build container.
Groundwork for the next round: no kernel of this model exists yet; these files pin what the oracle and the CUDA path will have to match.

Third-party primitives the reference imports are provided as semantic shims (published behaviour of the pinned wheels):
    torch_scatter.scatter(reduce='add'|'sum'|'mean'), segment_coo, segment_csr            (2.1.2)
    torch_sparse.SparseTensor: (row, col, value, sparse_sizes) constructor sorted by (row, col) with a STABLE sort, row selection
        `adj[idx]` (repeats allowed, rows come out in the order of idx), .storage.{row,col,value}(), .coo(), .sparse_sizes(),
        .set_value_(v, layout='coo')                                                             (0.6.18)
    torch_geometric.nn.radius_graph == torch_cluster.radius_graph (oracle.graph), torch_geometric.data.Data (attribute bag)
    pytorch_lightning.LightningModule (only subclassed)

    python tests/golden/make_golden_gemnet_oc.py      # writes tests/golden/gemnet_oc_f32.npz
"""
import hashlib
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
REF = "/root/reference/nablaDFT/gemnet_oc"
from weights import golden_state_dict  # noqa: E402
from make_golden_painn_oc import _scatter, _segment_coo, _segment_csr  # noqa: E402  (same shims as for PaiNN-OC)


def _scatter_any(src, index, dim=0, out=None, dim_size=None, reduce="sum"):
    if reduce == "mean":
        s = _scatter(src, index, dim=dim, dim_size=dim_size, reduce="sum")
        cnt = _scatter(torch.ones_like(src), index, dim=dim, dim_size=dim_size, reduce="sum").clamp(min=1)
        return s / cnt
    return _scatter(src, index, dim=dim, dim_size=dim_size, reduce="sum" if reduce == "add" else reduce)


class _Storage:
    def __init__(self, row, col, value):
        self._row, self._col, self._value = row, col, value

    def row(self): return self._row
    def col(self): return self._col
    def value(self): return self._value


class SparseTensor:
    def __init__(self, row=None, col=None, value=None, sparse_sizes=None, is_sorted=False):
        if not is_sorted:
            order = torch.argsort(row * int(sparse_sizes[1]) + col, stable=True)
            row, col = row[order], col[order]
            value = value[order] if value is not None else None
        self.storage = _Storage(row, col, value)
        self._sizes = tuple(int(x) for x in sparse_sizes)

    def sparse_sizes(self): return self._sizes
    def coo(self): return self.storage.row(), self.storage.col(), self.storage.value()

    def set_value_(self, value, layout=None):
        self.storage._value = value
        return self

    def __getitem__(self, idx):
        row, col, val = self.coo()
        counts = torch.bincount(row, minlength=self._sizes[0])
        ptr = torch.zeros(self._sizes[0] + 1, dtype=torch.long)
        ptr[1:] = torch.cumsum(counts, 0)
        idx = idx.long()
        n_per = counts[idx]
        new_row = torch.repeat_interleave(torch.arange(idx.numel()), n_per)
        start = torch.repeat_interleave(ptr[idx], n_per)
        inner = torch.arange(int(n_per.sum())) - torch.repeat_interleave(torch.cumsum(n_per, 0) - n_per, n_per)
        src = start + inner
        return SparseTensor(new_row, col[src], None if val is None else val[src], (idx.numel(), self._sizes[1]), is_sorted=True)


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _Data:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def install_shims():
    from oracle.graph import radius_graph

    _mod("torch_scatter", scatter=_scatter_any, segment_coo=_segment_coo, segment_csr=_segment_csr)
    _mod("torch_sparse", SparseTensor=SparseTensor)
    _mod("torch_geometric"); _mod("torch_geometric.nn", radius_graph=lambda x, r, batch=None, max_num_neighbors=32, **k: radius_graph(x, r, batch, max_num_neighbors))
    _mod("torch_geometric.data", Data=_Data)
    _mod("pytorch_lightning", LightningModule=torch.nn.Module)
    pkg = _mod("nablaDFT"); pkg.__path__ = []
    sub = _mod("nablaDFT.gemnet_oc"); sub.__path__ = [REF]
    lay = _mod("nablaDFT.gemnet_oc.layers"); lay.__path__ = [os.path.join(REF, "layers")]

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    for n in ("initializers", "utils", "loss"):
        load(f"nablaDFT.gemnet_oc.{n}", os.path.join(REF, f"{n}.py"))
    return load


def main():
    load = install_shims()
    # submodules import each other relatively; let the import system resolve them from the package paths registered above
    import importlib

    gem = importlib.import_module("nablaDFT.gemnet_oc.gemnet_oc")
    import yaml

    cfg = yaml.safe_load(open("/root/reference/config/model/gemnet-oc.yaml"))["net"]
    cfg.pop("_target_")
    torch.manual_seed(0)
    net = gem.GemNetOC(**cfg).float().eval()  # the reference graph code allocates float32 buffers: it only runs in its default dtype
    sd = net.state_dict()
    WS = float(os.environ.get("GEM_WS", "0.5"))
    new = golden_state_dict(sd, bias_std=0.02, weight_scale=WS)
    merged = {}
    for k, v in sd.items():
        if k.endswith("scale_factor"):
            merged[k] = torch.ones_like(v)  # "fitted" and neutral: scale_file is null in config/model/gemnet-oc.yaml
        elif k in new:
            merged[k] = torch.as_tensor(np.asarray(new[k])).float().reshape(v.shape)
        else:
            merged[k] = v
    net.load_state_dict(merged, strict=True)
    fx = np.load(os.path.join(HERE, "fixture_molecules.npz"))
    mols = [0, 7]
    z = torch.from_numpy(np.concatenate([fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols])).long()
    pos = torch.from_numpy(np.concatenate([fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols])).float()
    batch = torch.repeat_interleave(torch.arange(len(mols)), torch.tensor([int(fx["ptr"][m + 1] - fx["ptr"][m]) for m in mols]))
    data = _Data(z=z, pos=pos, batch=batch, natoms=torch.bincount(batch), num_nodes=z.numel())
    # intermediates for the next round's kernels: atom embeddings h after the embedding and after every interaction block (full), edge
    # embeddings m as per-edge L2 norms (the full [E, 512] tensors would be 5 MB each), per-block (E, F) contributions of the output blocks
    inter = {}

    def keep(name):
        def hook(mod, inp, out):
            if name.startswith("int"):
                inter[name + "/h"] = out[0].detach().numpy().copy()
                inter[name + "/m_rownorm"] = out[1].detach().norm(dim=1).numpy().copy()
            elif name.startswith("out"):
                inter[name + "/x_E"] = out[0].detach().numpy().copy()
                inter[name + "/x_F_rownorm"] = out[1].detach().norm(dim=-1).numpy().copy() if out[1].dim() > 1 else out[1].detach().numpy().copy()
            else:
                inter[name] = out.detach().numpy().copy() if out.shape[-1] <= 256 else out.detach().norm(dim=1).numpy().copy()
        return hook

    handles = [net.atom_emb.register_forward_hook(keep("atom_emb/h")), net.edge_emb.register_forward_hook(keep("edge_emb/m_rownorm"))]
    for i, blk in enumerate(net.int_blocks):
        handles.append(blk.register_forward_hook(keep(f"int{i}")))
    for i, blk in enumerate(net.out_blocks):
        handles.append(blk.register_forward_hook(keep(f"out{i}")))
    out = net(data)
    e, f = out[0].detach().numpy(), out[1].detach().numpy()
    for hd in handles:  # the second batch below must not overwrite the recorded intermediates
        hd.remove()
    g = net.get_graphs_and_indices(data)  # (main_graph, a2a, a2ee2a, qint graphs, id_swap, trip_idx_e2e, ..., quad_idx)
    sizes = {"main_edges": int(g[0]["edge_index"].shape[1]), "a2a_edges": int(g[1]["edge_index"].shape[1]), "a2ee2a_edges": int(g[2]["edge_index"].shape[1]),
             "qint_edges": int(g[3]["edge_index"].shape[1])}
    print(sizes)
    graphs = {"main/edge_index": g[0]["edge_index"].numpy().astype(np.int32), "main/distance": g[0]["distance"].numpy(),
              "a2a/edge_index": g[1]["edge_index"].numpy().astype(np.int32), "a2ee2a/edge_index": g[2]["edge_index"].numpy().astype(np.int32),
              "qint/edge_index": g[3]["edge_index"].numpy().astype(np.int32), "id_swap": g[4].numpy().astype(np.int32)}
    trip = g[5]
    for k in ("in", "out", "out_agg"):
        if k in trip:
            graphs[f"trip_e2e/{k}"] = trip[k].numpy().astype(np.int32)
    for name, t in (("trip_a2e", g[6]), ("trip_e2a", g[7])):
        for k in ("in", "out", "out_agg"):
            graphs[f"{name}/{k}"] = t[k].numpy().astype(np.int32)
    q = g[8]
    for k in ("out", "trip_in_to_quad", "trip_out_to_quad", "out_agg"):
        a = np.ascontiguousarray(q[k].numpy().astype(np.int32))  # 526 k entries each: stored as sha1 + length (the file stays under 1 MB)
        graphs[f"quad/{k}/sha1"], graphs[f"quad/{k}/len"] = np.asarray(hashlib.sha1(a.tobytes()).hexdigest()), np.asarray(a.shape[0])
    for tk in ("triplet_in", "triplet_out"):
        for k in ("in", "out"):
            graphs[f"quad/{tk}/{k}"] = q[tk][k].numpy().astype(np.int32)
    graphs["a2a/target_neighbor_idx"] = g[1]["target_neighbor_idx"].numpy().astype(np.int32)
    graphs["a2ee2a/target_neighbor_idx"] = g[2]["target_neighbor_idx"].numpy().astype(np.int32)
    print({k: v.shape for k, v in graphs.items()}, {k: v.shape for k, v in inter.items()})
    print("E", e.ravel(), "max|F|", np.abs(f).max(), "params", sum(p.numel() for p in net.parameters()))
    # a second batch (three other molecules): outputs + SHA-1 of every index array, to harden the pin without growing the file

    mols2 = [3, 12, 41]
    z2 = torch.from_numpy(np.concatenate([fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols2])).long()
    pos2 = torch.from_numpy(np.concatenate([fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols2])).float()
    batch2 = torch.repeat_interleave(torch.arange(len(mols2)), torch.tensor([int(fx["ptr"][m + 1] - fx["ptr"][m]) for m in mols2]))
    data2 = _Data(z=z2, pos=pos2, batch=batch2, natoms=torch.bincount(batch2), num_nodes=z2.numel())
    out2 = net(data2)
    g2 = net.get_graphs_and_indices(data2)
    sha = lambda t: hashlib.sha1(np.ascontiguousarray(t.numpy().astype(np.int32)).tobytes()).hexdigest()
    hashes = {"b2/main": sha(g2[0]["edge_index"]), "b2/a2a": sha(g2[1]["edge_index"]), "b2/a2ee2a": sha(g2[2]["edge_index"]), "b2/qint": sha(g2[3]["edge_index"]),
              "b2/id_swap": sha(g2[4]), "b2/trip_e2e_in": sha(g2[5]["in"]), "b2/trip_a2e_in": sha(g2[6]["in"]), "b2/trip_e2a_in": sha(g2[7]["in"]),
              "b2/quad_out": sha(g2[8]["out"]), "b2/quad_in": sha(g2[8]["trip_in_to_quad"]), "b2/quad_outmap": sha(g2[8]["trip_out_to_quad"])}
    print("batch 2: E", out2[0].detach().numpy().ravel(), "quads", int(g2[8]["out"].numel()))
    np.savez_compressed(os.path.join(HERE, "gemnet_oc_f32.npz"), **{k: np.asarray(v) for k, v in hashes.items()}, **{
        "b2/mols": np.asarray(mols2), "b2/z": z2.numpy(), "b2/pos": pos2.numpy(), "b2/batch": batch2.numpy(), "b2/energy": out2[0].detach().numpy(),
        "b2/forces": out2[1].detach().numpy()}, mols=np.asarray(mols), z=z.numpy(), pos=pos.numpy(), batch=batch.numpy(), energy=e, forces=f, weight_scale=np.asarray(WS), **graphs, **inter, **{k: np.asarray(v) for k, v in sizes.items()},
                        n_params=np.asarray(sum(p.numel() for p in net.parameters())))


if __name__ == "__main__":
    main()
