"""GPU tests of the QHNet kernels one C-ABI entry point at a time (csrc/qhnet.cu and the GEMMs behind nb200_dense / nb200_qh_linear), each
against a float64 reference of the same operation built from the CPU oracle (oracle/qhnet.py, oracle/e3.py) and evaluated on the same float32
inputs; then the whole model where tests/test_gpu_qhnet.py does not look: pair chunks past the first, chunk sizes, and graph edge cases.

The graph kernels walk the CSR graphs of nb200_neighbor_build + nb200_qh_expand_rows, at cutoff 12 (the convolution graph) and 1e4 (the full
pair graph), of one batch holding a 1-atom Br molecule (an empty row in both graphs), a 2-atom molecule whose atoms are 20 bohr apart (no
convolution edge, 2 pairs), golden molecule `a` with one H atom moved 15 bohr from everything (an empty convolution row inside a molecule) and
a 199-atom synthetic molecule (long rows).  Outputs are pre-filled with NaN, so every row must be written, and carry a guard tail of GUARD
rows holding SENTINEL, which must survive.  Each check prints its measured error next to its bound."""
import copy
import math
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN
from oracle.e3 import NORM2MOM
from test_gpu_phisnet_ops import SENTINEL, P, assert_written, call, cuda_gen, guarded, lib, per_L, per_row_L, rand, report, split
from test_gpu_qhnet import H_TOL, ORBITALS, _Data, from_cm, models, to_cm  # noqa: F401 (models is a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Bounds set from the first H100 run with a margin of about 4x or more; worst measured value in brackets.
REL = 2e-6         # kernel outputs: of max|ref| per order L, of the row's float64 sum of |terms| where the kernel sums over edges, and of each
                   # entry's sum of |terms| for the GEMMs (tp_conv 5.1e-7, tp_pair 2.6e-7, tp_self 1.9e-7, qh_linear 3.5e-7, expand 2.4e-7)
REL_PATH = 2e-6    # one tensor-product path alone, same scale (2.5e-7; a 1e-4 relative change of one (4,4,4) literal reads 1.9e-5)
CHUNK_TOL = 1e-7   # Ha: whole model, any pair_chunk against the default; only the GEMM path of the chunked layers changes (3.7e-9)
EINVAL, EUNSUPPORTED = -1, -2
HIDDEN = "128x0e+128x1o+128x2e+128x3o+128x4e"
BASE = "128x0e+128x1e+128x2e+128x3e+128x4e"


# ---------------------------------------------------------------------------------------------------------------- batch and graphs
def golden_isolated():
    """Golden molecule `a` (39 atoms) with its last H atom moved 15 bohr along x past every other atom."""
    g = np.load(os.path.join(GOLDEN, "qhnet_f64.npz"))
    z, pos = g["a.z"].astype(np.int64), g["a.pos"].astype(np.float64).copy()
    assert z[-1] == 1
    pos[-1] = [pos[:-1, 0].max() + 15.0, pos[:-1, 1].mean(), pos[:-1, 2].mean()]
    return z, pos


def edge_molecules():
    """[(z, pos bohr)]: 1-atom Br, H and C 20 bohr apart, golden `a` with an isolated H."""
    return [(np.array([35]), np.array([[0.5, -1.0, 2.0]])), (np.array([1, 6]), np.array([[0.0, 0.0, 0.0], [20.0, 0.0, 0.0]])),
            golden_isolated()]


def qh_graph(pos_d, mol_ptr_d, n_mol, cutoff, cap):
    """QHNet._graph: device CSR (row_ptr, col, rev, tgt, geom, status) at `cutoff`."""
    N = pos_d.shape[0]
    I = lambda n: torch.empty(n, dtype=torch.int32, device=DEV)
    g = dict(row_ptr=I(N + 1), col=I(cap), rev=I(cap), tgt=I(cap), geom=torch.empty(cap, 4, device=DEV),
             status=torch.zeros(4, dtype=torch.int32, device=DEV))
    scratch = I(N)
    call(lib().nb200_neighbor_build, P(pos_d), P(mol_ptr_d), n_mol, N, float(cutoff), 2 ** 31 - 1, cap, P(g["row_ptr"]), P(g["col"]),
         P(g["rev"]), P(g["geom"]), P(scratch), P(g["status"]))
    call(lib().nb200_qh_expand_rows, P(g["row_ptr"]), N, P(g["tgt"]))
    st = g["status"].cpu()
    assert int(st[1]) == 0, st
    n = int(st[0])
    g.update(N=N, E=n, tgt_h=g["tgt"][:n].long().cpu(), col_h=g["col"][:n].long().cpu(), row_ptr_h=g["row_ptr"].long().cpu())
    return g


def rows_edges(g, rows):
    return torch.cat([torch.arange(int(g["row_ptr_h"][a]), int(g["row_ptr_h"][a + 1])) for a in rows])


@pytest.fixture(scope="module")
def batch():
    from nabladft_b200.synth import synth_batch

    big = synth_batch(11, 1, heavy_min=105, heavy_max=105)
    mols = edge_molecules() + [(big["z"].astype(np.int64), big["pos"].astype(np.float64) * 1.8897261)]
    sizes = [len(z) for z, _ in mols]
    pos = torch.tensor(np.concatenate([p for _, p in mols]), dtype=torch.float32, device=DEV)
    mol_ptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=DEV)
    n_pairs = int(sum(n * (n - 1) for n in sizes))
    b = dict(sizes=sizes, z=np.concatenate([z for z, _ in mols]), N=int(sum(sizes)), P=n_pairs, pos=pos, mol_ptr=mol_ptr)
    b["full"] = qh_graph(pos, mol_ptr, len(sizes), 10000.0, n_pairs)
    b["conv"] = qh_graph(pos, mol_ptr, len(sizes), 12.0, n_pairs)
    assert b["full"]["E"] == n_pairs
    gc = b["conv"]
    sh = torch.empty(max(gc["E"], 1), 25, device=DEV)
    call(lib().nb200_qh_edge_basis, P(gc["geom"]), P(gc["status"]), gc["E"], 0.5, 12.0, -1.0, None, 32, None, P(sh))
    gc["sh"] = sh
    a0 = sum(sizes[:3])
    sel = list(range(a0)) + [int(a) for a in np.linspace(a0, a0 + sizes[3] - 1, 8).round()]
    b["sel"] = torch.tensor(sel)
    loc = torch.full((b["N"],), -1, dtype=torch.long)
    loc[b["sel"]] = torch.arange(len(sel))
    b["loc"] = loc
    deg = gc["row_ptr_h"][1:] - gc["row_ptr_h"][:-1]
    b["empty_conv"] = [0, 1, 2, a0 - 1]  # Br, the 2-atom molecule, the isolated H
    assert all(int(deg[a]) == 0 for a in b["empty_conv"]) and int(deg[3:a0 - 1].min()) > 0
    print(f"batch: {b['N']} atoms, {gc['E']} conv edges, {n_pairs} pairs; references on {len(sel)} rows")
    return b


@pytest.fixture(scope="module")
def tps():
    """The oracle's four tensor products: ConvLayer.tp_node of layer 0 and of the later layers, PairNetLayer.tp_node_pair, SelfNetLayer.tp."""
    from oracle.e3 import Irreps
    from oracle.qhnet import ConvLayer, PairNetLayer, SelfNetLayer

    hidden, base, sh = Irreps(HIDDEN), Irreps(BASE), Irreps.spherical_harmonics(4)
    t = dict(conv0=ConvLayer(Irreps("128x0e"), hidden, hidden, sh, 32, use_norm_gate=False).tp_node, conv=ConvLayer(hidden, hidden, hidden, sh, 32).tp_node,
             pair=PairNetLayer(base, base, base, 32, 128).tp_node_pair, self=SelfNetLayer(base, base, base).tp)
    assert [len(t[k].paths) for k in ("conv0", "conv", "pair", "self")] == [5, 42, 65, 65]
    return t


def only_path(tp, p):
    """The oracle tensor product restricted to its path p (the others contribute nothing)."""
    t = copy.copy(tp)
    t.paths = [tp.paths[p]]
    return t


def path_l(tp, p):
    return tp.irreps_out[tp.paths[p]["io"]].ir.l


def f64(t):
    return t.double().cpu()


def flat(x):
    """device [R, 25, C] -> e3nn flat float64 [R, 25 C]."""
    return from_cm(f64(x))


# ---------------------------------------------------------------------------------------------------------------- tensor products
def conv_inputs(b, layer0, seed, n_atoms=None):
    gc = b["conv"]
    gen = cuda_gen(seed)
    N = b["N"]
    nw = 640 if layer0 else 5376
    E = gc["E"] if n_atoms is None else int(gc["row_ptr_h"][n_atoms])
    x = rand(gen, N, 128) if layer0 else rand(gen, N, 25, 128)
    return x, rand(gen, E, nw), rand(gen, E, nw)


def conv_reference(tp, b, x, w1, w2, rows, add_self):
    """ConvLayer.forward's message + aggregation: index_add over dst of tp_node(x[src], sh, w1 w2), plus x[dst] with add_self."""
    gc = b["conv"]
    e = rows_edges(gc, rows)
    ed = e.to(DEV)
    src, dst = gc["col_h"][e], gc["tgt_h"][e]
    xf = f64(x) if x.dim() == 2 else flat(x)
    lrow = torch.full((b["N"],), -1, dtype=torch.long)
    lrow[torch.as_tensor(rows)] = torch.arange(len(rows))
    with torch.no_grad():
        msg = tp(xf[src], f64(gc["sh"][ed]), f64(w1[ed]) * f64(w2[ed]))
    ref = torch.zeros(len(rows), 3200, dtype=torch.float64).index_add_(0, lrow[dst], msg)
    absum = torch.zeros(len(rows), 3200, dtype=torch.float64).index_add_(0, lrow[dst], msg.abs())
    if add_self:
        ref += xf[rows]
        absum += xf[rows].abs()
    return split(to_cm(ref)), split(to_cm(absum))


@pytest.mark.parametrize("layer0,add_self", [(1, 0), (0, 0), (0, 1)], ids=["layer0", "general", "general+self"])
def test_tp_conv(batch, tps, layer0, add_self):
    """nb200_qh_tp_conv over the convolution graph against ConvLayer.tp_node + index_add (layers.py:263-271), per row and order."""
    b = batch
    N = b["N"]
    x, w1, w2 = conv_inputs(b, layer0, 10 + 2 * layer0 + add_self)
    buf, out = guarded(N, 25, 128)
    call(lib().nb200_qh_tp_conv, P(x), P(b["conv"]["sh"]), P(w1), P(w2), P(b["conv"]["row_ptr"]), P(b["conv"]["col"]), N, layer0, add_self, P(out))
    assert_written(buf, N, "tp_conv")
    for a in b["empty_conv"]:
        want = x[a] if add_self else torch.zeros_like(out[a])
        assert torch.equal(out[a], want), f"row {a} has no edges: must be exactly {'x[t]' if add_self else '0'}"
    sel = b["sel"].tolist()
    ref, absum = conv_reference(tps["conv0" if layer0 else "conv"], b, x, w1, w2, sel, add_self)
    per_row_L(split(out[b["sel"].to(DEV)]), ref, absum, f"tp_conv layer0={layer0} add_self={add_self}")


def path_errors(name, tp, run, rows_ref):
    """Per-path isolation: for each path p, run(p) -> (got, ref, absum) with every weight but path p's zero.  The path's own order must be
    within REL_PATH of max(max|ref_L|, the row's sum of |terms|); every other order must be exactly 0."""
    errs = []
    for p in range(len(tp.paths)):
        got, ref, absum = run(p)
        L = path_l(tp, p)
        assert all(bool((got[l] == 0).all()) for l in range(5) if l != L), f"{name} path {p} wrote outside its order {L}"
        err = (got[L] - ref[L]).abs().amax(dim=(1, 2))
        scale = torch.maximum(absum[L].amax(dim=(1, 2)), ref[L].abs().max().expand_as(err)).clamp_min(1e-30)
        errs.append(float((err / scale).max()))
    worst = int(np.argmax(errs))
    pa = tp.paths[worst]
    lls = (tp.irreps_in1[pa["i1"]].ir.l, tp.irreps_in2[pa["i2"]].ir.l, path_l(tp, worst))
    print(f"{name}: {len(errs)} paths one at a time on {rows_ref} rows, worst err / scale = {errs[worst]:.2e} at path {worst} {lls} "
          f"(bound {REL_PATH:.0e}); per path " + " ".join(f"{e:.1e}" for e in errs))
    bad = [(p, e) for p, e in enumerate(errs) if e > REL_PATH]
    assert not bad, (name, bad)


@pytest.mark.parametrize("layer0,add_self", [(1, 0), (0, 0), (0, 1)], ids=["layer0", "general", "general+self"])
def test_tp_conv(batch, tps, layer0, add_self):
    """nb200_qh_tp_conv over the convolution graph against ConvLayer.tp_node + index_add (layers.py:263-271), per row and order."""
    b = batch
    N = b["N"]
    x, w1, w2 = conv_inputs(b, layer0, 10 + 2 * layer0 + add_self)
    buf, out = guarded(N, 25, 128)
    call(lib().nb200_qh_tp_conv, P(x), P(b["conv"]["sh"]), P(w1), P(w2), P(b["conv"]["row_ptr"]), P(b["conv"]["col"]), N, layer0, add_self,
         P(out))
    assert_written(buf, N, "tp_conv")
    for a in b["empty_conv"]:
        want = x[a] if add_self else torch.zeros_like(out[a])
        assert torch.equal(out[a], want), f"row {a} has no edges: must be exactly {'x[t]' if add_self else '0'}"
    sel = b["sel"].tolist()
    ref, absum = conv_reference(tps["conv0" if layer0 else "conv"], b, x, w1, w2, sel, add_self)
    per_row_L(split(out[b["sel"].to(DEV)]), ref, absum, f"tp_conv layer0={layer0} add_self={add_self}")


@pytest.mark.parametrize("layer0", [1, 0], ids=["tp_conv0", "tp_conv"])
def test_tp_conv_per_path(batch, tps, layer0):
    """qh_tp_conv0 (5 paths) and qh_tp_conv (42 paths) of qhnet_tp_gen.inc one path at a time, over the first three molecules' rows."""
    b = batch
    n_at = sum(b["sizes"][:3])
    rows = [3, 12, 24, n_at - 2]
    x, w1, w2 = conv_inputs(b, layer0, 20 + layer0, n_atoms=n_at)
    tp = tps["conv0" if layer0 else "conv"]
    gc = b["conv"]

    def run(p):
        w1p = torch.zeros_like(w1)
        w1p[:, p * 128:(p + 1) * 128] = w1[:, p * 128:(p + 1) * 128]
        buf, out = guarded(n_at, 25, 128)
        call(lib().nb200_qh_tp_conv, P(x), P(gc["sh"]), P(w1p), P(w2), P(gc["row_ptr"]), P(gc["col"]), n_at, layer0, 0, P(out))
        assert_written(buf, n_at, "tp_conv")
        ref, absum = conv_reference(only_path(tp, p), b, x, w1p, w2, rows, 0)
        return split(out[rows]), ref, absum

    path_errors("tp_conv0" if layer0 else "tp_conv", tp, run, len(rows))


def pair_reference(tp, x, w1, w2, tgt, col, pairs):
    """PairNetLayer.forward's tp_node_pair(x[src], x[dst], w1 w2): src = row owner, dst = col."""
    pd = pairs.to(DEV)
    xf = flat(x)
    with torch.no_grad():
        return tp(xf[tgt[pairs]], xf[col[pairs]], f64(w1[pd]) * f64(w2[pd]))


def test_tp_pair(batch, tps):
    """nb200_qh_tp_pair over the full pair graph against PairNetLayer.tp_node_pair (layers.py:481-485), on every pair of the referenced rows."""
    b = batch
    g, N, n = b["full"], b["N"], b["P"]
    gen = cuda_gen(30)
    x, w1, w2 = rand(gen, N, 25, 128), rand(gen, n, 8320), rand(gen, n, 8320)
    buf, out = guarded(n, 25, 128)
    call(lib().nb200_qh_tp_pair, P(x), P(w1), P(w2), P(g["tgt"]), P(g["col"]), P(g["status"]), n, P(out))
    assert_written(buf, n, "tp_pair")
    e = rows_edges(g, b["sel"].tolist())
    ref = split(to_cm(pair_reference(tps["pair"], x, w1, w2, g["tgt_h"], g["col_h"], e)))
    per_L(split(out[e.to(DEV)]), ref, f"tp_pair ({len(e)} pairs)")


def test_tp_pair_per_path(batch, tps):
    """qh_tp_uuu2 of qhnet_tp_gen.inc (65 paths, two per-pair weights) one path at a time, on pairs of the 2-atom and the golden molecule."""
    b = batch
    g, N = b["full"], b["N"]
    n = sum(k * (k - 1) for k in b["sizes"][:3])
    gen = cuda_gen(31)
    x, w1, w2 = rand(gen, N, 25, 128), rand(gen, n, 8320), rand(gen, n, 8320)
    pairs = torch.cat([torch.tensor([0, 1]), torch.arange(2, n, 23)])
    tp = tps["pair"]

    def run(p):
        w1p = torch.zeros_like(w1)
        w1p[:, p * 128:(p + 1) * 128] = w1[:, p * 128:(p + 1) * 128]
        buf, out = guarded(n, 25, 128)
        call(lib().nb200_qh_tp_pair, P(x), P(w1p), P(w2), P(g["tgt"]), P(g["col"]), P(g["status"]), n, P(out))
        assert_written(buf, n, "tp_pair")
        ref = split(to_cm(pair_reference(only_path(tp, p), x, w1p, w2, g["tgt_h"], g["col_h"], pairs)))
        return split(out[pairs.to(DEV)]), ref, [r.abs() for r in ref]

    path_errors("tp_uuu2", tp, run, len(pairs))


def self_tp(tp, w):
    t = copy.copy(tp)
    t._parameters = {"weight": torch.nn.Parameter(f64(w), requires_grad=False)}
    return t


@pytest.mark.parametrize("rows", [1, 37, 2051])
def test_tp_self(tps, rows):
    """nb200_qh_tp_self against SelfNetLayer.tp (internal weights) with and without the residual (layers.py:571-573)."""
    gen = cuda_gen(40 + rows)
    xl, xr, res, w = rand(gen, rows, 25, 128), rand(gen, rows, 25, 128), rand(gen, rows, 25, 128), rand(gen, 8320)
    with torch.no_grad():
        tp_ref = self_tp(tps["self"], w)(flat(xl), flat(xr))
    for r in (None, res):
        buf, out = guarded(rows, 25, 128)
        call(lib().nb200_qh_tp_self, P(xl), P(xr), P(w), P(r), rows, P(out))
        assert_written(buf, rows, "tp_self")
        ref = to_cm(tp_ref + (flat(r) if r is not None else 0))
        per_L(split(out), split(ref), f"tp_self rows={rows} res={r is not None}")


def test_tp_self_per_path(tps):
    """qh_tp_uuu1 of qhnet_tp_gen.inc (65 paths, one shared weight vector) one path at a time."""
    gen = cuda_gen(45)
    rows = 16
    xl, xr, w = rand(gen, rows, 25, 128), rand(gen, rows, 25, 128), rand(gen, 8320)
    tp = tps["self"]

    def run(p):
        wp = torch.zeros_like(w)
        wp[p * 128:(p + 1) * 128] = w[p * 128:(p + 1) * 128]
        buf, out = guarded(rows, 25, 128)
        call(lib().nb200_qh_tp_self, P(xl), P(xr), P(wp), None, rows, P(out))
        assert_written(buf, rows, "tp_self")
        with torch.no_grad():
            ref = split(to_cm(only_path(self_tp(tp, wp), p)(flat(xl), flat(xr))))
        return split(out), ref, [r.abs() for r in ref]

    path_errors("tp_uuu1", tp, run, rows)


# ---------------------------------------------------------------------------------------------------------------- invariants, norm gate, pair MLP
def chunk_starts(n):
    return [p0 for p0 in (1000, 16384, n - 7) if 0 < p0 < n]


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["conv", "conv-layer0", "pair"])
def test_invariants(batch, mode):
    """nb200_qh_invariants against inner_product and the concatenations of ConvLayer.forward (mode 0: [pre[dst]_0, pre[dst]_0, ip], mode 1:
    [x[dst], x[dst]]) and PairNetLayer.forward (mode 2: [a0[dst]_0, a0[src]_0, ip]); in mode 2 also through the chunk-offset pointers
    QHNet._forward passes."""
    from oracle.e3 import Irreps
    from oracle.qhnet import inner_product

    b = batch
    g = b["full"] if mode == 2 else b["conv"]
    N, E = b["N"], g["E"]
    gen = cuda_gen(50 + mode)
    f = rand(gen, N, 128) if mode == 1 else rand(gen, N, 25, 128)
    width = 256 if mode == 1 else 768
    buf, out = guarded(E, width)
    call(lib().nb200_qh_invariants, P(f), P(g["tgt"]), P(g["col"]), P(g["status"]), E, mode, P(out))
    assert_written(buf, E, f"invariants mode {mode}")
    tgt_d, col_d = g["tgt"][:E].long(), g["col"][:E].long()
    if mode == 1:
        assert torch.equal(out, torch.cat([f[tgt_d], f[tgt_d]], dim=1))
        print(f"invariants mode 1: {E} edges, exact copies")
        return
    dst_d, src_d = (tgt_d, col_d) if mode == 0 else (col_d, tgt_d)
    assert torch.equal(out[:, :128], f[dst_d, 0]) and torch.equal(out[:, 128:256], f[dst_d if mode == 0 else src_d, 0]), \
        "the scalar blocks must be exact copies"
    e = rows_edges(g, b["sel"].tolist())
    dst, src = (g["tgt_h"][e], g["col_h"][e]) if mode == 0 else (g["col_h"][e], g["tgt_h"][e])
    ff = flat(f)
    ip = inner_product(Irreps(HIDDEN), ff[dst], ff[src])
    got = f64(out[e.to(DEV)])
    for l in range(1, 5):
        r = ip[:, l * 128:(l + 1) * 128]
        report(f"invariants mode {mode} <f, f>_{l}", (got[:, (l + 1) * 128:(l + 2) * 128] - r).abs().max(), r.abs().max(), REL)
    if mode == 2:
        for p0 in chunk_starts(E):
            pc = min(2048, E - p0)
            cbuf, cout = guarded(pc, width)
            call(lib().nb200_qh_invariants, P(f), P(g["tgt"][p0:]), P(g["col"][p0:]), P(g["status"]), pc, mode, P(cout))
            assert_written(cbuf, pc, "invariants chunk")
            assert torch.equal(cout, out[p0:p0 + pc]), f"chunk at pair {p0} differs from the whole-graph call"


@pytest.mark.parametrize("rows", [1, 37, 2051])
def test_norm_feats_and_gate(rows):
    """nb200_qh_norm_feats against [x_0, Norm(x)_{l>=1}] and nb200_qh_gate against NormGate's [gates_0, x_l gates_l] (layers.py:123-147);
    rows 2, 5, 8, ... have their l >= 1 parts exactly zero."""
    from oracle.e3 import ElementwiseTensorProduct, Irreps, Norm

    gen = cuda_gen(60 + rows)
    x = rand(gen, rows, 25, 128)
    x[2::3, 1:] = 0
    gates = rand(gen, rows, 640)
    fbuf, f0 = guarded(rows, 640)
    call(lib().nb200_qh_norm_feats, P(x), rows, P(f0))
    assert_written(fbuf, rows, "norm_feats")
    assert torch.equal(f0[:, :128], x[:, 0])
    xf = flat(x)
    norms = Norm(Irreps(HIDDEN))(xf)[:, 128:]
    got = f64(f0[:, 128:])
    assert bool((got[2::3] == 0).all())
    rel = float(((got - norms).abs() / norms.clamp_min(1e-30))[norms > 0].max())
    print(f"norm_feats rows={rows}: max relative err of each norm = {rel:.2e} (bound {REL:.0e})")
    assert rel <= REL
    ybuf, y = guarded(rows, 25, 128)
    call(lib().nb200_qh_gate, P(x), P(gates), rows, P(y))
    assert_written(ybuf, rows, "gate")
    g64 = f64(gates)
    prod = ElementwiseTensorProduct(Irreps(HIDDEN)[1:], Irreps("512x0e"))(xf[:, 128:], g64[:, 128:])
    ref = to_cm(torch.cat([g64[:, :128], prod], dim=1))
    assert bool((y[2::3, 1:] == 0).all())
    err = float(((f64(y) - ref).abs() - 2.0 ** -24 * ref.abs()).max())
    print(f"gate rows={rows}: every entry within one fp32 rounding of x gate: {err <= 0}")
    assert err <= 0


def dense_call(M, N, K, A, B, trans_b, bias=None, act_kind=None, C=None, act=None):
    C = torch.empty(M, N, device=DEV) if C is None else C
    call(lib().nb200_dense, M, N, K, P(A), A.shape[1], P(B), B.shape[1], trans_b, P(C), N, 0, P(bias), P(act), act_kind or 0)
    return C


def test_pair_hidden(batch):
    """nb200_qh_pair_hidden after the two per-atom GEMMs QHNet._forward runs, against silu(W[:, :128] e_dst + W[:, 128:] e_src + b)
    (qhnet.py:227-232) in float64; also through the chunk-offset pointers."""
    b = batch
    g, N, n = b["full"], b["N"], b["P"]
    gen = cuda_gen(70)
    emb, W, bias = rand(gen, N, 128), rand(gen, 128, 256, scale=256 ** -0.5), rand(gen, 128, scale=0.3)
    A = dense_call(N, 128, 128, emb, W[:, :128].contiguous(), 0)
    Bn = dense_call(N, 128, 128, emb, W[:, 128:].contiguous(), 0)
    buf, h = guarded(n, 128)
    call(lib().nb200_qh_pair_hidden, P(A), P(Bn), P(bias), P(g["tgt"]), P(g["col"]), P(g["status"]), n, P(h))
    assert_written(buf, n, "pair_hidden")
    e = rows_edges(g, b["sel"].tolist())
    e64, W64 = f64(emb), f64(W)
    pre = e64[g["col_h"][e]] @ W64[:, :128].T + e64[g["tgt_h"][e]] @ W64[:, 128:].T + f64(bias)
    ref = torch.nn.functional.silu(pre)
    report(f"pair_hidden ({len(e)} pairs)", (f64(h[e.to(DEV)]) - ref).abs().max(), ref.abs().max(), REL)
    for p0 in chunk_starts(n):
        pc = min(2048, n - p0)
        cbuf, ch = guarded(pc, 128)
        call(lib().nb200_qh_pair_hidden, P(A), P(Bn), P(bias), P(g["tgt"][p0:]), P(g["col"][p0:]), P(g["status"]), pc, P(ch))
        assert_written(cbuf, pc, "pair_hidden chunk")
        assert torch.equal(ch, h[p0:p0 + pc]), f"chunk at pair {p0} differs from the whole-graph call"


# ---------------------------------------------------------------------------------------------------------------- GEMMs
DENSE_SHAPES = [  # (K, N, trans_b, act_kind or None, bias): every dense layer of QHNet._forward, and plain ssp once
    (32, 32, 1, 2, False),      # FullyConnectedNet hidden layer on the radial basis (fc_node)
    (32, 128, 1, 2, False),     # fc_node_pair hidden layer
    (32, 5376, 1, None, False),  # fc_node / layer_l0 output, convolution layers 1-4
    (32, 640, 1, None, False),  # fc_node / layer_l0 output, convolution layer 0
    (768, 32, 1, 2, False),     # layer_l0 hidden layer on the invariants
    (768, 128, 0, 0, True),     # PairNetLayer.fc hidden layer (silu)
    (256, 32, 1, 2, False),     # layer_l0 hidden layer, convolution layer 0
    (640, 640, 0, 0, True),     # NormGate.fc hidden layer
    (640, 640, 0, None, True),  # NormGate.fc output
    (128, 8320, 0, None, True),  # PairNetLayer.fc output, fc_ii / fc_ij output
    (128, 8320, 1, None, False),  # fc_node_pair output
    (128, 52, 0, None, True),   # fc_ii_bias / fc_ij_bias output (50 padded to 52)
    (128, 128, 0, 0, True),     # fc_ii / fc_ii_bias hidden layer
    (128, 128, 0, None, False),  # fc_ij hidden layer halves
    (128, 128, 0, 1, True),     # ssp
]


def act_ref(x, kind):
    from oracle.qhnet import ssp

    return torch.nn.functional.silu(x) if kind == 0 else ssp(x) if kind == 1 else NORM2MOM["ssp"] * ssp(x)


@pytest.mark.parametrize("K,N,trans_b,act,bias", DENSE_SHAPES, ids=[f"{k}x{n}-t{t}-a{a}" for k, n, t, a, _ in DENSE_SHAPES])
def test_dense(K, N, trans_b, act, bias):
    """nb200_dense at the shapes QHNet._forward uses, at row counts on both sides of the pre-split switch (2048) and at 20000 rows: C and the
    activation copy against float64, per entry of its sum of |terms| (values checked on all rows up to 2049, on 288 spread rows and the last
    64 beyond)."""
    for M in (37, 2047, 2049, 20000):
        gen = cuda_gen(K + N + M + 7 * trans_b)
        A = rand(gen, M, K)
        B = rand(gen, K, N, scale=K ** -0.5) if trans_b else rand(gen, N, K, scale=K ** -0.5)
        bb = rand(gen, N, scale=0.3) if bias else None
        cbuf, C = guarded(M, N)
        abuf, Aout = guarded(M, N) if act is not None else (None, None)
        dense_call(M, N, K, A, B, trans_b, bb, act, C, Aout)
        assert_written(cbuf, M, "dense C")
        if act is not None:
            assert_written(abuf, M, "dense act")
        rows = torch.arange(M) if M <= 2049 else torch.unique(torch.cat([torch.linspace(0, M - 1, 288).round().long(), torch.arange(M - 64, M)]))
        rd = rows.to(DEV)
        Bt = f64(B) if trans_b else f64(B).T
        ref = f64(A[rd]) @ Bt + (f64(bb) if bias else 0)
        scale = f64(A[rd]).abs() @ Bt.abs() + (f64(bb).abs() if bias else 0)  # float64 sum of |terms| of each entry
        report(f"dense M={M} K={K} N={N} trans_b={trans_b} C", (f64(C[rd]) - ref).abs(), scale, REL)
        if act is not None:
            ra = act_ref(ref, act)
            slope = NORM2MOM["ssp"] if act == 2 else 1.1  # largest |act'|: ssp' = sigmoid <= 1, silu' < 1.1
            report(f"dense M={M} K={K} N={N} act_kind={act}", (f64(Aout[rd]) - ra).abs(), slope * scale + ra.abs(), REL)


@pytest.mark.parametrize("rows", [1, 37, 2047, 2049, 2300])
@pytest.mark.parametrize("c_out,acc", [(128, 1), (32, 0)], ids=["128-acc", "32"])
def test_linear(rows, c_out, acc):
    """nb200_qh_linear (e3nn o3.Linear, weights pre-scaled by 1/sqrt(c_in), bias on 0e) against the oracle's Linear, 128 -> 128 accumulating
    into the output and 128 -> 32, on both sides of the per-order tall GEMM switch."""
    from oracle.e3 import Irreps, Linear

    gen = cuda_gen(80 + rows + c_out)
    x, W, bias = rand(gen, rows, 25, 128), rand(gen, 5, 128, c_out, scale=128 ** -0.5), rand(gen, c_out)
    y0 = rand(gen, rows, 25, c_out)
    buf, y = guarded(rows, 25, c_out)
    if acc:
        y.copy_(y0)
    call(lib().nb200_qh_linear, P(x), P(W), P(bias), rows, 128, c_out, acc, P(y))
    assert_written(buf, rows, "qh_linear")
    lin = Linear(Irreps(HIDDEN), Irreps("+".join(f"{c_out}x{l}{'eo'[l % 2]}" for l in range(5)))).double()
    with torch.no_grad():
        lin.weight.copy_((f64(W) * math.sqrt(128)).reshape(-1))
        lin.bias.copy_(f64(bias))
        ref = to_cm(lin(flat(x)), c_out) + (f64(y0) if acc else 0)
    per_L(split(y), split(ref), f"qh_linear rows={rows} 128->{c_out} acc={acc}")


# ---------------------------------------------------------------------------------------------------------------- expansion, assembly
@pytest.fixture(scope="module")
def expansion():
    import ctypes

    from nabladft_b200._lib import check
    from nabladft_b200.qhnet import _expansion_tables
    from oracle.e3 import Irreps
    from oracle.qhnet import Expansion

    ins, cg, n_path, n_bias = _expansion_tables()
    assert (n_path, n_bias, len(ins)) == (8320, 50, 19)
    check(lib().nb200_qh_expand_setup(ins.ctypes.data_as(ctypes.c_void_p), cg.ctypes.data_as(ctypes.c_void_p)), "expand_setup")
    out_irr = Irreps("5x0e+4x1e+3x2e")
    ex = Expansion(Irreps("32x0e+32x1e+32x2e+32x3e+32x4e"), out_irr, out_irr)
    assert (ex.num_path_weight, ex.num_bias) == (n_path, n_bias)
    return ins, ex


@pytest.mark.parametrize("rows", [1, 37, 4097])
def test_expand(expansion, rows):
    """nb200_qh_expand against Expansion.forward (layers.py:598-662); 4097 rows leave a partial last CTA.  At 37 rows also each of the 19
    instructions alone (weights and biases of the others zero)."""
    ins, ex = expansion
    gen = cuda_gen(90 + rows)
    x, W, Bw = rand(gen, rows, 25, 32), rand(gen, rows, 8320), rand(gen, rows, 52)

    def run(W_, B_):
        buf, blk = guarded(rows, 32, 32)
        call(lib().nb200_qh_expand, P(x), P(W_), P(B_), 52, rows, P(blk))
        assert_written(buf, rows, "expand")
        with torch.no_grad():
            ref = ex(flat(x), f64(W_), f64(B_[:, :50]))
        return (f64(blk) - ref).abs().max(), ref.abs().max()

    report(f"expand rows={rows}", *run(W, Bw), REL)
    if rows != 37:
        return
    errs = []
    for lin, l1, l2, woff, boff in ins.tolist():
        n12 = (5, 4, 3)[l1] * (5, 4, 3)[l2]
        Wi, Bi = torch.zeros_like(W), torch.zeros_like(Bw)
        Wi[:, woff:woff + 32 * n12] = W[:, woff:woff + 32 * n12]
        if lin == 0:
            Bi[:, boff:boff + n12] = Bw[:, boff:boff + n12]
        err, scale = run(Wi, Bi)
        errs.append(float(err / scale))
    print("expand per instruction (l_in, l1, l2): " + " ".join(f"{tuple(i[:3])}={e:.1e}" for i, e in zip(ins.tolist(), errs)))
    assert max(errs) <= REL, errs


def assembly_batch():
    """(z, pos bohr, sizes): 1-atom Br, H and C 20 bohr apart, and a molecule with every element of ORBITALS and two Br atoms."""
    rng = np.random.default_rng(3)
    zc = np.array([1, 6, 7, 8, 9, 16, 17, 35, 35, 1, 6, 1])
    pos = np.concatenate([[[0.5, -1.0, 2.0]], [[0.0, 0.0, 0.0], [20.0, 0.0, 0.0]], rng.uniform(-6, 6, (len(zc), 3))])
    return np.concatenate([[35, 1, 6], zc]), pos, [1, 2, len(zc)]


def test_assemble():
    """nb200_qh_assemble against QHNetOracle.assemble (build_final_matrix + H + H^T, qhnet.py:293-321): each entry within one fp32 rounding of
    the exact sum of its two block entries, every entry of H written, the guard intact."""
    from types import SimpleNamespace

    from nabladft_b200.qhnet import QHNet
    from oracle.qhnet import QHNetOracle, orbital_masks

    z, pos, sizes = assembly_batch()
    N = len(z)
    n = int(sum(k * (k - 1) for k in sizes))
    pos_d = torch.tensor(pos, dtype=torch.float32, device=DEV)
    mol_ptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=DEV)
    g = qh_graph(pos_d, mol_ptr, len(sizes), 10000.0, n)
    masks, _ = QHNet._get_mask(ORBITALS)
    zmax = max(masks) + 1
    mask_tab, norb_tab = torch.zeros(zmax, 32, dtype=torch.int32), torch.zeros(zmax, dtype=torch.int32)
    for k, m in masks.items():
        mask_tab[k, :len(m)] = m.to(torch.int32)
        norb_tab[k] = len(m)
    norb = norb_tab[torch.from_numpy(z)].long().numpy()
    atom_mol = np.repeat(np.arange(len(sizes)), sizes)
    starts = np.concatenate([[0], np.cumsum(sizes)])
    atom_off = np.concatenate([np.concatenate([[0], np.cumsum(norb[s:e])[:-1]]) for s, e in zip(starts[:-1], starts[1:])])
    mol_norb = np.array([norb[s:e].sum() for s, e in zip(starts[:-1], starts[1:])])
    mol_off = np.concatenate([[0], np.cumsum(mol_norb ** 2)])
    i32 = lambda v: torch.tensor(np.asarray(v), dtype=torch.int32, device=DEV)
    z_d, mask_d, norb_d, atom_mol_d, atom_off_d, mol_norb_d = i32(z), mask_tab.to(DEV), norb_tab.to(DEV), i32(atom_mol), i32(atom_off), i32(mol_norb)
    mol_off_d = torch.tensor(mol_off, dtype=torch.int64, device=DEV)
    gen = cuda_gen(95)
    diag, offd = rand(gen, N, 32, 32), rand(gen, n, 32, 32)
    total = int(mol_off[-1])
    buf, H = guarded(total)
    call(lib().nb200_qh_assemble, P(diag), P(offd), P(z_d), P(g["tgt"]), P(g["col"]), P(g["rev"]), N, n, P(mask_d.reshape(-1)), P(norb_d),
         P(atom_mol_d), P(atom_off_d), P(mol_off_d), P(mol_norb_d), P(H))
    assert_written(buf, total, "assemble")
    ns = SimpleNamespace(orbital_mask=orbital_masks(ORBITALS)[0])
    d64, o64 = f64(diag), f64(offd)
    p0 = 0
    for m, k in enumerate(sizes):
        a0, a1, np_m = int(starts[m]), int(starts[m + 1]), k * (k - 1)
        zm = torch.from_numpy(z[a0:a1])
        ref = QHNetOracle.assemble(ns, zm, torch.zeros(k, dtype=torch.long), d64[a0:a1], o64[p0:p0 + np_m],
                                   g["col_h"][p0:p0 + np_m] - a0, g["tgt_h"][p0:p0 + np_m] - a0)
        got = H[int(mol_off[m]):int(mol_off[m + 1])].view(int(mol_norb[m]), int(mol_norb[m]))
        assert torch.equal(got, got.T)
        excess = float(((f64(got) - ref).abs() - 2.0 ** -24 * ref.abs()).max())
        print(f"assemble mol {m} ({k} atoms, {int(mol_norb[m])} orbitals): within one fp32 rounding of the float64 sum: {excess <= 0}")
        assert excess <= 0, (m, excess)
        p0 += np_m


# ---------------------------------------------------------------------------------------------------------------- argument checks
def _raw(name, args):
    from nabladft_b200._lib import current_stream

    conv = [P(a) if isinstance(a, torch.Tensor) else a for a in args]
    return getattr(lib(), name)(*conv, current_stream())


def _arg_cases():
    """(name, arguments with a count of 0, indices of required pointers, index of the count, indices of outputs, [(index, bad value, code)]).
    Every buffer is big enough for a count of 4, so a wrongly launched kernel would stay in bounds; the outputs must keep SENTINEL."""
    b = lambda *s: torch.full(s, SENTINEL, device=DEV)
    i = lambda k: torch.zeros(k, dtype=torch.int32, device=DEV)
    st = i(4)
    x, f0 = b(4, 25, 128), b(4, 640)
    return [
        ("nb200_qh_norm_feats", [x, 0, b(4, 640)], (0, 2), 1, (2,), []),
        ("nb200_qh_gate", [x, f0, 0, b(4, 25, 128)], (0, 1, 3), 2, (3,), []),
        ("nb200_qh_invariants", [x, i(4), i(4), st, 0, 0, b(4, 768)], (0, 1, 2, 3, 6), 4, (6,), [(5, 3, EINVAL), (5, -1, EINVAL)]),
        ("nb200_qh_tp_conv", [x, b(4, 25), b(4, 5376), b(4, 5376), i(5), i(4), 0, 0, 1, b(4, 25, 128)], (0, 1, 2, 3, 4, 5, 9), 6, (9,), []),
        ("nb200_qh_tp_pair", [x, b(4, 8320), b(4, 8320), i(4), i(4), st, 0, b(4, 25, 128)], (0, 1, 2, 3, 4, 5, 7), 6, (7,), []),
        ("nb200_qh_tp_self", [x, x, b(8320), x, 0, b(4, 25, 128)], (0, 1, 2, 5), 4, (5,), []),
        ("nb200_qh_linear", [b(4, 25, 48), b(5, 48, 128), b(128), 0, 128, 128, 0, b(4, 25, 128)], (0, 1, 7), 3, (7,), [(4, 48, EUNSUPPORTED)]),
        ("nb200_dense", [0, 128, 128, b(4, 128), 128, b(128, 128), 128, 0, b(4, 128), 128, 0, b(128), b(4, 128), 2], (3, 5, 8), 0, (8, 12),
         [(2, 48, EUNSUPPORTED), (1, 50, EUNSUPPORTED)]),
        ("nb200_qh_expand", [b(4, 25, 32), b(4, 8320), b(4, 52), 52, 0, b(4, 32, 32)], (0, 1, 2, 5), 4, (5,), [(3, 49, EINVAL)]),
        ("nb200_qh_pair_hidden", [b(4, 128), b(4, 128), b(128), i(4), i(4), st, 0, b(4, 128)], (0, 1, 2, 3, 4, 5, 7), 6, (7,), []),
        ("nb200_qh_assemble", [b(4, 32, 32), b(4, 32, 32), i(4), i(4), i(4), i(4), 0, 0, i(64), i(2), i(4), i(4),
                               torch.zeros(2, dtype=torch.int64, device=DEV), i(1), b(64)], (0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12, 13, 14), 6, (14,), []),
        ("nb200_axpy", [b(8), b(8), 0], (0, 1), 2, (0,), [(2, 6, EINVAL), (2, -4, EINVAL)]),
    ]


ARG_CASES = ["nb200_qh_norm_feats", "nb200_qh_gate", "nb200_qh_invariants", "nb200_qh_tp_conv", "nb200_qh_tp_pair", "nb200_qh_tp_self",
             "nb200_qh_linear", "nb200_dense", "nb200_qh_expand", "nb200_qh_pair_hidden", "nb200_qh_assemble", "nb200_axpy"]


@pytest.mark.parametrize("case", ARG_CASES)
def test_argument_checks(case):
    """A count of 0 -> NB200_OK with nothing written; a null required pointer -> NB200_EINVAL; and the refusals with work to do (count 4):
    invariants mode 3, c_in 48 in nb200_qh_linear, K 48 or N 50 in nb200_dense, bw_stride 49 in nb200_qh_expand, n % 4 != 0 in nb200_axpy.
    None of these launches a kernel: every output keeps SENTINEL."""
    name, args, required, count, outs, bad_values = next(c for c in _arg_cases() if c[0] == case)
    assert _raw(name, args) == 0
    for k in required:
        bad = list(args)
        bad[k] = None
        assert _raw(name, bad) == EINVAL, (name, "null argument", k)
    for k, v, code in bad_values:
        bad = list(args)
        bad[k] = v
        if k != count:
            bad[count] = 4
        assert _raw(name, bad) == code, (name, k, v)
    torch.cuda.synchronize()
    for k in outs:
        assert bool((args[k] == SENTINEL).all()), f"{name}: output {k} was written"


# ---------------------------------------------------------------------------------------------------------------- whole model
def oracle_h(ora, z, pos):
    """float64 oracle H of one molecule (positions given in bohr, rounded to float32 as the device sees them)."""
    zt = torch.as_tensor(z).long()
    pt = torch.from_numpy(np.asarray(pos, dtype=np.float32).astype(np.float64))
    bt = torch.zeros(len(zt), dtype=torch.long)
    with torch.no_grad():
        d, o, fd, fs = ora.blocks(zt, pt, bt)
        return ora.assemble(zt, bt, d, o, fd, fs)


def device_data(mols):
    z = torch.tensor(np.concatenate([m[0] for m in mols])).long().to(DEV)
    pos = torch.tensor(np.concatenate([m[1] for m in mols]), dtype=torch.float32).to(DEV)
    batch = torch.repeat_interleave(torch.arange(len(mols)), torch.tensor([len(m[0]) for m in mols])).to(DEV)
    return _Data(z, pos, batch)


@pytest.fixture(scope="module")
def cfg4(models):
    """BASELINE config 4's batch (synth_batch(3, 64), bohr) and its Hamiltonians at the default pair chunk."""
    from nabladft_b200.synth import synth_batch

    _, net = models
    b = synth_batch(3, 64)
    z, pos = b["z"].astype(np.int64), b["pos"].astype(np.float64) * 1.8897261
    ptr = b["mol_ptr"].astype(np.int64)
    mols = [(z[ptr[m]:ptr[m + 1]], pos[ptr[m]:ptr[m + 1]]) for m in range(64)]
    data = device_data(mols)
    n = np.diff(ptr)
    pair_off = np.concatenate([[0], np.cumsum(n * (n - 1))])
    return dict(mols=mols, data=data, pair_off=pair_off, H0=[h.clone() for h in net(data, packed=True)], chunk=net.pair_chunk)


def test_pair_chunk_invariance_cfg4(models, cfg4):
    """The config-4 batch (102,528 pairs) with pair_chunk = P (one chunk), 16384, 2049, 2048, 2047 and 1000 against the default: the chunk only
    decides which GEMM path (tall pre-split or plain) forms each chunk's path weights."""
    _, net = models
    n_pairs = int(cfg4["pair_off"][-1])
    try:
        for chunk in (n_pairs, 16384, 2049, 2048, 2047, 1000):
            net.pair_chunk = chunk
            H = net(cfg4["data"], packed=True)
            d = max(float((a - c).abs().max()) for a, c in zip(H, cfg4["H0"]))
            print(f"cfg 4: pair_chunk {chunk} ({-(-n_pairs // chunk)} chunks) vs {cfg4['chunk']}: max|dH| = {d:.2e} Ha (bound {CHUNK_TOL:.0e})")
            assert d <= CHUNK_TOL, (chunk, d)
    finally:
        net.pair_chunk = cfg4["chunk"]


def test_later_pair_chunks_match_oracle_cfg4(models, cfg4):
    """Molecules 10 and 47 of the config-4 forward straddle boundaries of the default 16384-pair chunks (47 holds Br), and 63 lies in the last
    chunk: each against the float64 oracle on that molecule alone, at the north-star 1e-6 Ha."""
    ora, _ = models
    off, chunk = cfg4["pair_off"], cfg4["chunk"]
    assert chunk == 16384
    for m in (10, 47):
        assert off[m] // chunk != (off[m + 1] - 1) // chunk, f"molecule {m} no longer straddles a chunk boundary"
    assert 35 in cfg4["mols"][47][0] and off[63] // chunk == (off[64] - 1) // chunk and off[63] >= chunk * ((off[64] - 1) // chunk)
    for m in (10, 47, 63):
        ref = oracle_h(ora, *cfg4["mols"][m])
        err = float((cfg4["H0"][m].double().cpu() - ref).abs().max())
        print(f"cfg 4 molecule {m} (pairs {off[m]}..{off[m + 1] - 1}): max|dH| = {err:.2e} Ha (max|H| {float(ref.abs().max()):.2f})")
        assert err < H_TOL, (m, err)


@pytest.fixture(scope="module")
def edge_refs(models):
    ora, _ = models
    mols = edge_molecules() + [(np.array([6]), np.array([[1.0, 2.0, 3.0]]))]
    return mols, [oracle_h(ora, z, pos) for z, pos in mols]


@pytest.mark.parametrize("which", [[0], [0, 3], [1], [2], [0, 1, 2]], ids=["1-atom", "two-1-atom", "2-atoms-20-bohr", "isolated-H", "three"])
def test_graph_edge_cases_match_oracle(models, edge_refs, which):
    """Batches without pairs (P = 0), without convolution edges (E = 0, P = 2), and with an atom that has no convolution edge inside a
    molecule, against the float64 oracle."""
    _, net = models
    mols, refs = edge_refs
    H = net(device_data([mols[k] for k in which]), packed=True)
    for k, h in zip(which, H):
        assert h.shape == refs[k].shape
        err = float((h.double().cpu() - refs[k]).abs().max())
        print(f"edge case {which}: molecule {k} ({len(mols[k][0])} atoms): max|dH| = {err:.2e} Ha")
        assert err < H_TOL, (k, err)


def test_small_pair_chunks_match_oracle(models, edge_refs):
    """pair_chunk = 1 and 7 on the three-molecule edge batch (1484 pairs) against the float64 oracle."""
    _, net = models
    mols, refs = edge_refs
    chunk = net.pair_chunk
    try:
        for c in (1, 7):
            net.pair_chunk = c
            H = net(device_data(mols[:3]), packed=True)
            err = max(float((h.double().cpu() - r).abs().max()) for h, r in zip(H, refs))
            print(f"pair_chunk {c}: max|dH| = {err:.2e} Ha")
            assert err < H_TOL, (c, err)
    finally:
        net.pair_chunk = chunk


@pytest.mark.parametrize("bad", [15, 50, 83, -1])
def test_unsupported_elements_refused_then_forward_matches(models, edge_refs, bad):
    """Z without orbitals (15, 50), without an embedding row (83) or negative is refused on the host before any launch; the next forward is
    unaffected."""
    _, net = models
    mols, refs = edge_refs
    with pytest.raises(ValueError, match=f"\\[{bad}\\]"):
        net(device_data([(np.array([1, bad]), np.array([[0.0, 0.0, 0.0], [1.4, 0.0, 0.0]]))]))
    H = net(device_data([mols[1]]))
    assert float((H.double().cpu() - refs[1]).abs().max()) < H_TOL
