"""Float64 restatement of the SchNet inference kernels (csrc/schnet.cu), built from the model's definition (schnetpack SchNet), not from the
kernels: the first filter layer over ALL K Gaussians, the continuous-filter convolution and its reverse, and the shifted softplus.  Every op
also returns a first-order error bound A per element for the fp32 kernel: a small multiple of u = 2^-24 times the float64 sum of |terms| of
that element (the rounding of every product and of the sum), plus the Gaussians the 16-centre band leaves out where the kernel drops them.

Shared by tests/test_schnet_kernel_ref.py (CPU: the restatement against the oracle, central differences, and the sensitivity of each term)
and tests/test_gpu_schnet_kernels.py (each kernel against it), which also share the synthetic graphs built here."""
import math

import numpy as np
import torch

F = 128
BAND = 16  # NB_BAND: centres k0 .. k0 + 15 around the distance bin
U = 2.0 ** -24
LN2 = math.log(2.0)
SPLIT, CHUNK = 8, 32  # SF1_SPLIT, SF1_CHUNK: edges of one bin are split 8 ways, 32 at a time
DROPS = ("b2", "dfc", "fcG2", "b1", "rev")  # terms whose omission the GPU tests must be able to see


def ssp(x):
    """schnetpack shifted softplus, with torch's threshold-20 linearisation."""
    return torch.nn.functional.softplus(x) - LN2


def spacing(cutoff, K):
    return cutoff / (K - 1)


def band_start(d, cutoff, K):
    """k0 the kernels pick: bin = floor(d * (1 / dx)) in fp32 (nb_bin_sort), clamped to [0, K - 1], then k0 = clamp(bin - 7, 0, K - 16)."""
    dx = np.float32(cutoff) / np.float32(K - 1)
    inv = np.float32(1.0) / dx
    b = np.floor(np.asarray(d, dtype=np.float32) * np.float32(1.0) * inv).astype(np.int64)
    b = np.clip(b, 0, K - 1)
    return torch.from_numpy(np.clip(b - (BAND // 2 - 1), 0, K - BAND))


def in_band(d, cutoff, K):
    k0 = band_start(d, cutoff, K)
    k = torch.arange(K)
    return (k[None, :] >= k0[:, None]) & (k[None, :] < k0[:, None] + BAND)


def gaussians(d, offsets, coeff):
    t = d[:, None] - offsets[None, :]
    phi = torch.exp(coeff * t * t)
    return phi, 2.0 * coeff * t * phi, t


def fcut(d, cutoff):
    a = math.pi / cutoff
    inside = (d < cutoff).to(d.dtype)
    return 0.5 * (torch.cos(d * a) + 1.0) * inside, -0.5 * a * torch.sin(d * a) * inside


def filter1(d, w1, b1, offsets, coeff, cutoff, drop=None):
    """One layer of filter_network.0: h = ssp(sum_k phi_k W1[k] + b1), dh = dh/dd = sigmoid(pre) sum_k phi'_k W1[k], over all K centres.
    d [E], w1 [K, F], b1 [F], offsets [K]  ->  h, dh, A_h, A_dh  [E, F]."""
    d, w1, b1, offsets = (x.double() for x in (d, w1, b1, offsets))
    K = offsets.numel()
    phi, dphi, t = gaussians(d, offsets, coeff)
    pre = phi @ w1 + (0.0 if drop == "b1" else b1)
    dpre = dphi @ w1
    sig = torch.sigmoid(pre)
    h, dh = ssp(pre), sig * dpre
    # |terms|; each Gaussian is off by ~|coeff t^2| u from the rounding of its exponent's argument
    rel = 1.0 + (coeff * t * t).abs()
    band = in_band(d.numpy(), cutoff, K).double()
    s_pre = (phi * rel) @ w1.abs() + b1.abs()
    s_dpre = (dphi.abs() * rel) @ w1.abs()
    trunc = (phi * (1 - band)) @ w1.abs()  # the kernel's 16-centre band drops these
    dtrunc = (dphi.abs() * (1 - band)) @ w1.abs()
    a_pre = 32 * U * s_pre + trunc
    a_dpre = 32 * U * s_dpre + dtrunc
    A_h = sig * a_pre + 8 * U * (h.abs() + 1.0)
    A_dh = sig * a_dpre + 0.25 * dpre.abs() * a_pre + 8 * U * dh.abs()
    return h, dh, A_h, A_dh


def cfconv_fwd(y, G1, b2, d, row_ptr, col, cutoff, drop=None):
    """agg_i = sum_{e in row i} y[col e] fcut(d_e) (G1_e + b2)  ->  agg, A  [N, F]."""
    y, G1, b2, d = (x.double() for x in (y, G1, b2, d))
    N = row_ptr.numel() - 1
    tgt = torch.repeat_interleave(torch.arange(N), (row_ptr[1:] - row_ptr[:-1]).long())
    fc, _ = fcut(d, cutoff)
    w = G1 + (0.0 if drop == "b2" else b2)
    yj = y[col.long()]
    agg = torch.zeros(N, F, dtype=torch.float64).index_add_(0, tgt, yj * w * fc[:, None])
    mag = yj.abs() * (G1.abs() + b2.abs())
    deg = (row_ptr[1:] - row_ptr[:-1]).double()[:, None]
    # sequential fp32 sum of deg terms; fcut has an absolute error of a few u
    A = U * ((deg + 8) * torch.zeros(N, F, dtype=torch.float64).index_add_(0, tgt, mag * fc[:, None])
             + 8 * torch.zeros(N, F, dtype=torch.float64).index_add_(0, tgt, mag))
    return agg, A


def cfconv_bwd(y, G1, G2, b2, d, row_ptr, col, rev, cutoff, gagg, egrad0, drop=None):
    """By source atom j over its row (edge symmetry):  gy_j = sum_{e in row j} fcut (G1_e + b2) gagg[col e];
    egrad[4e + 3] = egrad0[e] + sum_c (fcut' (G1_e + b2) + fcut G2_e)_c y_j,c gagg[col e]_c.  drop="rev" reads the filter rows of rev[e].
    -> gy, A_gy [N, F], egrad, A_egrad [E]."""
    y, G1, G2, b2, d, gagg, egrad0 = (x.double() for x in (y, G1, G2, b2, d, gagg, egrad0))
    N = row_ptr.numel() - 1
    if drop == "rev":
        G1, G2 = G1[rev.long()], G2[rev.long()]
    src = torch.repeat_interleave(torch.arange(N), (row_ptr[1:] - row_ptr[:-1]).long())  # the row's atom j
    fc, dfc = fcut(d, cutoff)
    g1 = G1 + (0.0 if drop == "b2" else b2)
    ga = gagg[col.long()]
    yj = y[src]
    gy = torch.zeros(N, F, dtype=torch.float64).index_add_(0, src, g1 * fc[:, None] * ga)
    dw = (0.0 if drop == "dfc" else g1 * dfc[:, None]) + (0.0 if drop == "fcG2" else G2 * fc[:, None])
    eg = egrad0 + (dw * yj * ga).sum(1)
    mag = (G1.abs() + b2.abs()) * ga.abs()
    deg = (row_ptr[1:] - row_ptr[:-1]).double()[:, None]
    A_gy = U * ((deg + 8) * torch.zeros(N, F, dtype=torch.float64).index_add_(0, src, mag * fc[:, None])
                + 8 * torch.zeros(N, F, dtype=torch.float64).index_add_(0, src, mag))
    a = math.pi / cutoff
    yg = (yj * ga).abs()
    A_eg = U * (16 * (yg * ((G1.abs() + b2.abs()) * dfc.abs()[:, None] + G2.abs() * fc[:, None])).sum(1)
                + 8 * (yg * ((G1.abs() + b2.abs()) * a + G2.abs())).sum(1) + 2 * eg.abs())
    return gy, A_gy, eg, A_eg


def linear_ssp(X, W, b):
    """f2out.0: Y = X W^T + b and ssp(Y)  ->  Y, A_Y, act, A_act."""
    X, W, b = X.double(), W.double(), b.double()
    Y = X @ W.T + b
    A_Y = 48 * U * (X.abs() @ W.abs().T + b.abs())  # 3xTF32 products and fp32 accumulation
    act = ssp(Y)
    return Y, A_Y, act, torch.sigmoid(Y) * A_Y + 8 * U * (act.abs() + 1.0)


# ---------------------------------------------------------------------------------------------------------- synthetic graphs
def _csr(n_atoms, pairs, dist):
    """Symmetric CSR (target-major, source-ascending as nb200_neighbor_build) of undirected pairs with distances -> row_ptr, col, rev, d."""
    pairs = np.asarray(pairs, dtype=np.int64)
    tgt = np.concatenate([pairs[:, 0], pairs[:, 1]])
    src = np.concatenate([pairs[:, 1], pairs[:, 0]])
    dd = np.concatenate([dist, dist]).astype(np.float32)
    P = len(pairs)
    partner = np.concatenate([np.arange(P) + P, np.arange(P)])
    order = np.lexsort((src, tgt))
    inv = np.empty_like(order)
    inv[order] = np.arange(len(order))
    rev = inv[partner[order]]
    row_ptr = np.zeros(n_atoms + 1, dtype=np.int64)
    np.add.at(row_ptr, tgt + 1, 1)
    row_ptr = np.cumsum(row_ptr)
    return (torch.from_numpy(row_ptr).int(), torch.from_numpy(src[order]).int(), torch.from_numpy(rev).int(), torch.from_numpy(dd[order]))


def edge_case_distances(cutoff, K, seed=0):
    """Distances at the kernels' edges: the band clamped at 0 (1e-4, 0.3 dx), k dx and k dx -+ 1 ulp for every k (every bin 0 .. K - 2 gets
    a few edges, fewer than the 8 splits), next to the cutoff (k0 clamped at K - 16, fcut -> 0), and one crowded bin of 151 pairs: 302
    directed edges, more than 8 x 32 and not a multiple of 8, so every split runs two chunks.  Bin K - 1 stays empty."""
    rng = np.random.default_rng(seed)
    dx = np.float32(cutoff) / np.float32(K - 1)
    d = [np.float32(1e-4), np.float32(0.3) * dx, np.float32(cutoff) * np.float32(1 - 1e-6)]
    for k in range(1, K - 1):
        c = np.float32(k) * dx
        d += [np.nextafter(c, np.float32(0)), c, np.nextafter(c, np.float32(cutoff))]
    d += list(((K // 3) + rng.uniform(0.05, 0.95, 151)).astype(np.float32) * dx)
    return np.array(d, dtype=np.float32)


def edge_case_graph(cutoff=5.0, K=100, seed=0):
    """Atom 0 has no edge; stars give rows of degree 1, 3, 4, 5 and 9 (around CF_STAGES = 4), a hub a row of 150, and a random pool takes
    the remaining distances.  Distances are shuffled over the pairs.  -> row_ptr, col, rev, d (fp32)."""
    rng = np.random.default_rng(seed)
    dist = edge_case_distances(cutoff, K, seed)
    rng.shuffle(dist)
    pairs, n = [], 1
    for deg in (1, 3, 4, 5, 9, 150):
        pairs += [(n, n + 1 + k) for k in range(deg)]
        n += deg + 1
    pool, rest = 48, len(dist) - len(pairs)
    seen = set()
    while len(seen) < rest:
        a, b = sorted(rng.choice(pool, 2, replace=False))
        seen.add((n + a, n + b))
    pairs += sorted(seen)
    return _csr(n + pool, pairs, dist)


def random_graph(n_atoms, n_pairs, cutoff, seed):
    rng = np.random.default_rng(seed)
    seen = set()
    while len(seen) < n_pairs:
        a, b = sorted(rng.choice(n_atoms, 2, replace=False))
        seen.add((a, b))
    return _csr(n_atoms, sorted(seen), rng.uniform(0.02, 0.999, n_pairs).astype(np.float32) * cutoff)


def geom_of(d, seed=0):
    """geom [E, 4]: a unit vector (unused by these kernels) and d in slot 3."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(d.numel(), 3, generator=g)
    return torch.cat([v / v.norm(dim=1, keepdim=True), d.float()[:, None]], 1)


def filter_weights(L, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(L, K, F, generator=g) * 0.7, torch.randn(L, F, generator=g)


def cfconv_inputs(N, E, seed=0):
    """y, G1, G2 [E, F] (independent per directed edge, so that reading rev[e]'s rows shows), b2, gagg and a non-zero egrad prefill."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    return dict(y=r(N, F), G1=r(E, F), G2=r(E, F), b2=r(F), gagg=r(N, F), egrad0=r(E, 4))


def kernel_case(L=1, seed=0, cutoff=5.0, K=100):
    """The inputs of the kernel tests: the edge-case graph, L layers of filter weights, the module's basis, and the cfconv operands."""
    row_ptr, col, rev, d = edge_case_graph(cutoff, K, seed)
    w1, b1 = filter_weights(L, K, seed)
    offsets = torch.linspace(0, cutoff, K)
    return dict(row_ptr=row_ptr, col=col, rev=rev, d=d, w1=w1, b1=b1, offsets=offsets, coeff=-0.5 / float(offsets[1] - offsets[0]) ** 2,
                **cfconv_inputs(row_ptr.numel() - 1, d.numel(), seed))


def max_ratio(err, A):
    """max |err| / A; an exact zero (an empty row, where A = 0 too) counts as 0."""
    r = torch.where(err == 0, torch.zeros_like(err), err / A)
    return float(r.max()) if r.numel() else 0.0
