"""Oracle: the e3nn==0.5.1 primitives QHNet uses -- TEST INFRASTRUCTURE ONLY (oracle/__init__.py).

e3nn is an un-vendored dependency of the reference (`/root/reference/setup.py:51`) and is not
installable here; this file restates its published algorithms (SURVEY.md Appendix A.4/A.4.1):

  o3.Irrep / o3.Irreps              -> Irrep, Irreps (parsing, slices, sort, products)
  o3.wigner_3j                      -> wigner_3j      (SU(2) Clebsch-Gordan via Racah's formula,
                                       conjugated into e3nn's real basis, Frobenius norm 1)
  o3.spherical_harmonics            -> spherical_harmonics (real SH l <= 4, y is the polar axis,
                                       'component' normalisation, m = -l..l)
  o3.TensorProduct                  -> TensorProduct  ('uvu', 'uuu', 'uvw'; component / element
                                       normalisation; external or internal weights)
  o3.Linear, o3.Norm, o3.ElementwiseTensorProduct, nn.FullyConnectedNet (normalize2mom)

Conventions pinned offline (tests/test_oracle_e3.py): w3j(1,1,1) = +eps_ijk/sqrt 6,
w3j(0,l,l) = +delta/sqrt(2l+1), sum_ij w3j(l,1,l+1) Y_l Y_1 = +c Y_{l+1} (how e3nn builds its SH),
invariance of every w3j under the Wigner-D matrices induced by the SH.  In the build container
the golden generator additionally checks SH and w3j against the e3nn-convention Wigner-D of the
reference's vendored `equiformer_v2/Jd.pt` (tests/golden/make_golden_qhnet.py).
PARITY WITH THE e3nn WHEEL ITSELF IS UNPINNED (cannot be imported); a sign/normalisation slip
here would still give a self-consistent equivariant model but would not load pretrained weights.
"""
import math
import re
from functools import lru_cache
from typing import List, Tuple

import numpy as np
import torch
from torch import nn

# e3nn.nn.FullyConnectedNet wraps activations with normalize2mom: act / sqrt(E_{z~N(0,1)} act(z)^2),
# the constant estimated from 1e6 seed-0 float64 samples (SURVEY.md A.4): ssp and silu
NORM2MOM = {"ssp": 1.8782046685, "silu": 1.6791767924}


# ------------------------------------------------------------------------------------- irreps
class Irrep:
    def __init__(self, l: int, p: int):
        self.l, self.p = int(l), int(p)

    @property
    def dim(self):
        return 2 * self.l + 1

    def __mul__(self, other):
        return [Irrep(l, self.p * other.p) for l in range(abs(self.l - other.l), self.l + other.l + 1)]

    def __eq__(self, o):
        return isinstance(o, Irrep) and (self.l, self.p) == (o.l, o.p)

    def __hash__(self):
        return hash((self.l, self.p))

    def __lt__(self, o):  # e3nn order: by l, then natural parity (-1)^l first
        return (self.l, -self.p * (-1) ** self.l) < (o.l, -o.p * (-1) ** o.l)

    def __repr__(self):
        return f"{self.l}{'e' if self.p == 1 else 'o'}"


class MulIr(tuple):
    mul = property(lambda s: s[0])
    ir = property(lambda s: s[1])
    dim = property(lambda s: s[0] * s[1].dim)


class Irreps(tuple):
    def __new__(cls, spec=()):
        if isinstance(spec, Irreps):
            return tuple.__new__(cls, spec)
        items = []
        if isinstance(spec, str):
            for tok in [t.strip() for t in spec.split("+") if t.strip()]:
                m = re.fullmatch(r"(?:(\d+)x)?(\d+)([eo])", tok)
                items.append(MulIr((int(m.group(1) or 1), Irrep(int(m.group(2)), 1 if m.group(3) == "e" else -1))))
        else:
            for it in spec:
                if isinstance(it, Irrep):
                    items.append(MulIr((1, it)))
                else:
                    mul, ir = it
                    if isinstance(ir, str):
                        ir = Irreps(ir)[0].ir
                    items.append(MulIr((int(mul), ir)))
        return tuple.__new__(cls, items)

    @staticmethod
    def spherical_harmonics(lmax):
        return Irreps([(1, Irrep(l, (-1) ** l)) for l in range(lmax + 1)])

    @property
    def dim(self):
        return sum(m.dim for m in self)

    def slices(self):
        out, i = [], 0
        for m in self:
            out.append(slice(i, i + m.dim))
            i += m.dim
        return out

    def count(self, ir):
        return sum(m.mul for m in self if m.ir == ir)

    def __contains__(self, ir):
        return any(m.ir == ir for m in self)

    def __getitem__(self, i):
        r = tuple.__getitem__(self, i)
        return Irreps(r) if isinstance(i, slice) else r

    def sort(self):
        out = sorted([(m.ir, i, m.mul) for i, m in enumerate(self)], key=lambda t: (t[0], t[1]))
        inv = [i for _, i, _ in out]
        p = [0] * len(inv)
        for new, old in enumerate(inv):
            p[old] = new
        return Irreps([(mul, ir) for ir, _, mul in out]), p, inv

    def simplify(self):
        out = []
        for m in self:
            if out and out[-1][1] == m.ir:
                out[-1] = (out[-1][0] + m.mul, m.ir)
            elif m.mul > 0:
                out.append((m.mul, m.ir))
        return Irreps(out)

    def __repr__(self):
        return "+".join(f"{m.mul}x{m.ir}" for m in self)


# ------------------------------------------------------------------------------------- wigner 3j
def _su2_cg_coeff(j1, m1, j2, m2, j3, m3):
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


def _real_to_complex(l):
    q = np.zeros((2 * l + 1, 2 * l + 1), dtype=np.complex128)
    for m in range(-l, 0):
        q[l + m, l + abs(m)] = 1 / math.sqrt(2)
        q[l + m, l - abs(m)] = -1j / math.sqrt(2)
    q[l, l] = 1
    for m in range(1, l + 1):
        q[l + m, l + abs(m)] = (-1) ** m / math.sqrt(2)
        q[l + m, l - abs(m)] = 1j * (-1) ** m / math.sqrt(2)
    return (-1j) ** l * q


@lru_cache(maxsize=None)
def _w3j_np(l1, l2, l3):
    C = np.zeros((2 * l1 + 1, 2 * l2 + 1, 2 * l3 + 1))
    for m1 in range(-l1, l1 + 1):
        for m2 in range(-l2, l2 + 1):
            m3 = m1 + m2
            if abs(m3) <= l3:
                C[l1 + m1, l2 + m2, l3 + m3] = _su2_cg_coeff(l1, m1, l2, m2, l3, m3)
    Q1, Q2, Q3 = _real_to_complex(l1), _real_to_complex(l2), _real_to_complex(l3)
    R = np.einsum("ij,kl,mn,ikn->jlm", Q1, Q2, np.conj(Q3.T), C.astype(np.complex128))
    assert np.abs(R.imag).max() < 1e-10
    R = R.real
    return R / np.linalg.norm(R)


def wigner_3j(l1, l2, l3, dtype=torch.float64):
    if not (abs(l1 - l2) <= l3 <= l1 + l2):
        raise ValueError("triangle")
    return torch.from_numpy(_w3j_np(int(l1), int(l2), int(l3))).to(dtype)


# ------------------------------------------------------------------------------------- spherical harmonics
def _sh_std(l, x, y, z):
    """Orthonormal real SH (z polar, positive leading coefficients), m = -l..l; unit vectors."""
    pi = math.pi
    if l == 0:
        return [torch.full_like(x, 0.5 * math.sqrt(1 / pi))]
    if l == 1:
        c = math.sqrt(3 / (4 * pi))
        return [c * y, c * z, c * x]
    if l == 2:
        return [0.5 * math.sqrt(15 / pi) * x * y, 0.5 * math.sqrt(15 / pi) * y * z, 0.25 * math.sqrt(5 / pi) * (3 * z * z - 1),
                0.5 * math.sqrt(15 / pi) * x * z, 0.25 * math.sqrt(15 / pi) * (x * x - y * y)]
    if l == 3:
        return [0.25 * math.sqrt(35 / (2 * pi)) * y * (3 * x * x - y * y), 0.5 * math.sqrt(105 / pi) * x * y * z,
                0.25 * math.sqrt(21 / (2 * pi)) * y * (5 * z * z - 1), 0.25 * math.sqrt(7 / pi) * (5 * z**3 - 3 * z),
                0.25 * math.sqrt(21 / (2 * pi)) * x * (5 * z * z - 1), 0.25 * math.sqrt(105 / pi) * (x * x - y * y) * z,
                0.25 * math.sqrt(35 / (2 * pi)) * x * (x * x - 3 * y * y)]
    if l == 4:
        return [0.75 * math.sqrt(35 / pi) * x * y * (x * x - y * y), 0.75 * math.sqrt(35 / (2 * pi)) * y * (3 * x * x - y * y) * z,
                0.75 * math.sqrt(5 / pi) * x * y * (7 * z * z - 1), 0.75 * math.sqrt(5 / (2 * pi)) * y * (7 * z**3 - 3 * z),
                (3.0 / 16.0) * math.sqrt(1 / pi) * (35 * z**4 - 30 * z * z + 3), 0.75 * math.sqrt(5 / (2 * pi)) * x * (7 * z**3 - 3 * z),
                (3.0 / 8.0) * math.sqrt(5 / pi) * (x * x - y * y) * (7 * z * z - 1), 0.75 * math.sqrt(35 / (2 * pi)) * x * (x * x - 3 * y * y) * z,
                (3.0 / 16.0) * math.sqrt(35 / pi) * (x**4 - 6 * x * x * y * y + y**4)]
    raise NotImplementedError("l <= 4")


def spherical_harmonics(lmax_or_irreps, vec, normalize=True, normalization="component"):
    """e3nn `o3.spherical_harmonics`: y is the polar axis, i.e. the standard (z-polar) real SH at
    (x_s, y_s, z_s) = (z, x, y); 'component': |Y_l|^2 = 2l+1."""
    assert normalize and normalization == "component"
    ls = [m.ir.l for m in lmax_or_irreps] if isinstance(lmax_or_irreps, Irreps) else list(range(lmax_or_irreps + 1))
    v = vec / vec.norm(dim=-1, keepdim=True)
    xe, ye, ze = v[..., 0], v[..., 1], v[..., 2]
    out = []
    for l in ls:
        out += [c * math.sqrt(4 * math.pi) for c in _sh_std(l, ze, xe, ye)]
    return torch.stack(out, dim=-1)


# ------------------------------------------------------------------------------------- tensor product & friends
class TensorProduct(nn.Module):
    """instructions: (i_in1, i_in2, i_out, mode, has_weight[, path_weight]); modes 'uvu', 'uuu', 'uvw'.
    Coefficient of a path = sqrt(alpha), alpha = dim(ir_out)/sum_{paths -> same out} num_elements * path_weight
    (irrep_normalization='component', path_normalization='element')."""

    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions, shared_weights=None, internal_weights=None,
                 irrep_normalization="component"):
        super().__init__()
        self.irreps_in1, self.irreps_in2, self.irreps_out = Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out)
        ins = [tuple(i) + ((1.0,) if len(i) == 5 else ()) for i in instructions]

        def nelem(i):
            return {"uvw": self.irreps_in1[i[0]].mul * self.irreps_in2[i[1]].mul, "uvu": self.irreps_in2[i[1]].mul,
                    "uvv": self.irreps_in1[i[0]].mul, "uuw": self.irreps_in1[i[0]].mul, "uuu": 1}[i[3]]

        self.paths = []
        off = 0
        for i in ins:
            m1, m2, mo = self.irreps_in1[i[0]], self.irreps_in2[i[1]], self.irreps_out[i[2]]
            assert abs(m1.ir.l - m2.ir.l) <= mo.ir.l <= m1.ir.l + m2.ir.l
            alpha = {"component": mo.ir.dim, "norm": m1.ir.dim * m2.ir.dim, "none": 1}[irrep_normalization]
            x = sum(nelem(k) for k in ins if k[2] == i[2])
            if x > 0:
                alpha /= x
            alpha *= i[5]
            shape = {"uvw": (m1.mul, m2.mul, mo.mul), "uvu": (m1.mul, m2.mul), "uuu": (m1.mul,)}[i[3]] if i[4] else None
            n = int(np.prod(shape)) if shape else 0
            self.paths.append(dict(i1=i[0], i2=i[1], io=i[2], mode=i[3], coeff=math.sqrt(alpha), wshape=shape, woff=off, wn=n))
            off += n
        self.weight_numel = off
        if internal_weights is None:
            internal_weights = shared_weights is not False and off > 0 and shared_weights is not None
        self.internal_weights = bool(internal_weights)
        if self.internal_weights:
            self.weight = nn.Parameter(torch.randn(off))

    def forward(self, x1, x2, weight=None):
        B = x1.shape[0]
        s1, s2 = self.irreps_in1.slices(), self.irreps_in2.slices()
        if self.internal_weights:
            weight = self.weight
        outs = [None] * len(self.irreps_out)
        for p in self.paths:
            m1, m2, mo = self.irreps_in1[p["i1"]], self.irreps_in2[p["i2"]], self.irreps_out[p["io"]]
            a = x1[:, s1[p["i1"]]].reshape(B, m1.mul, m1.ir.dim)
            b = x2[:, s2[p["i2"]]].reshape(B, m2.mul, m2.ir.dim)
            C = wigner_3j(m1.ir.l, m2.ir.l, mo.ir.l, dtype=x1.dtype)
            w = None
            if p["wshape"] is not None:
                w = weight[..., p["woff"]:p["woff"] + p["wn"]]
                w = w.reshape((B,) + p["wshape"]) if w.dim() == 2 else w.reshape((1,) + p["wshape"])
            if p["mode"] == "uvu":
                r = torch.einsum("zuv,ijk,zui,zvj->zuk", w.expand(B, *p["wshape"]), C, a, b)
            elif p["mode"] == "uuu":
                r = torch.einsum("ijk,zui,zuj->zuk", C, a, b)
                if w is not None:
                    r = r * w.expand(B, *p["wshape"])[..., None]
            elif p["mode"] == "uvw":
                r = torch.einsum("zuvw,ijk,zui,zvj->zwk", w.expand(B, *p["wshape"]), C, a, b)
            else:
                raise NotImplementedError(p["mode"])
            r = (p["coeff"] * r).reshape(B, mo.dim)
            outs[p["io"]] = r if outs[p["io"]] is None else outs[p["io"]] + r
        return torch.cat([o if o is not None else x1.new_zeros(B, self.irreps_out[k].dim) for k, o in enumerate(outs)], dim=-1)


class Linear(nn.Module):
    """o3.Linear(irreps_in, irreps_out, biases=True): y[w,m] = sum_u W[u,w] x[u,m] / sqrt(fan_in); bias on 0e."""

    def __init__(self, irreps_in, irreps_out, internal_weights=True, shared_weights=True, biases=True):
        super().__init__()
        self.irreps_in, self.irreps_out = Irreps(irreps_in), Irreps(irreps_out)
        self.paths = [(i, o) for i, mi in enumerate(self.irreps_in) for o, mo in enumerate(self.irreps_out) if mi.ir == mo.ir]
        self.weight = nn.Parameter(torch.randn(sum(self.irreps_in[i].mul * self.irreps_out[o].mul for i, o in self.paths)))
        self.bias_slots = [o for o, mo in enumerate(self.irreps_out) if biases and mo.ir.l == 0 and mo.ir.p == 1]
        nb = sum(self.irreps_out[o].mul for o in self.bias_slots)
        if nb:
            self.bias = nn.Parameter(torch.zeros(nb))

    def forward(self, x):
        B = x.shape[0]
        si = self.irreps_in.slices()
        outs = [x.new_zeros(B, mo.mul, mo.ir.dim) for mo in self.irreps_out]
        off = 0
        for i, o in self.paths:
            mi, mo = self.irreps_in[i], self.irreps_out[o]
            fan_in = sum(self.irreps_in[i2].mul for i2, o2 in self.paths if o2 == o)
            W = self.weight[off:off + mi.mul * mo.mul].reshape(mi.mul, mo.mul)
            off += mi.mul * mo.mul
            outs[o] = outs[o] + torch.einsum("zum,uw->zwm", x[:, si[i]].reshape(B, mi.mul, mi.ir.dim), W) / math.sqrt(fan_in)
        boff = 0
        for o in self.bias_slots:
            n = self.irreps_out[o].mul
            outs[o] = outs[o] + self.bias[boff:boff + n][None, :, None]
            boff += n
        return torch.cat([t.reshape(B, mo.dim) for t, mo in zip(outs, self.irreps_out)], dim=-1)  # B may be 0 (no pairs)


class Norm(nn.Module):
    """o3.Norm: per channel L2 norm over m -> mul scalars per block."""

    def __init__(self, irreps):
        super().__init__()
        self.irreps = Irreps(irreps)

    def forward(self, x):
        B = x.shape[0]
        return torch.cat([x[:, s].reshape(B, m.mul, m.ir.dim).pow(2).sum(-1).relu().sqrt() for s, m in zip(self.irreps.slices(), self.irreps)], dim=-1)


class ElementwiseTensorProduct(nn.Module):
    """o3.ElementwiseTensorProduct(irreps, 'Nx0e'): channel-wise product with scalars."""

    def __init__(self, irreps_in1, irreps_in2):
        super().__init__()
        self.irreps = Irreps(irreps_in1)

    def forward(self, x, scalars):
        B = x.shape[0]
        out, off = [], 0
        for s, m in zip(self.irreps.slices(), self.irreps):
            out.append((x[:, s].reshape(B, m.mul, m.ir.dim) * scalars[:, off:off + m.mul, None]).reshape(B, m.dim))
            off += m.mul
        return torch.cat(out, dim=-1)


class FullyConnectedNet(nn.Sequential):
    """e3nn.nn.FullyConnectedNet(hs, act): h = c_act act(x W / sqrt(fan_in)); last layer linear; W ~ N(0,1)."""

    class _Layer(nn.Module):
        def __init__(self, h_in, h_out, act, cst):
            super().__init__()
            self.weight = nn.Parameter(torch.randn(h_in, h_out))
            self.h_in, self.act, self.cst = h_in, act, cst

        def forward(self, x):
            y = x @ (self.weight / math.sqrt(self.h_in))
            return self.cst * self.act(y) if self.act is not None else y

    def __init__(self, hs, act, act_name="ssp"):
        super().__init__()
        self.hs = list(hs)
        for i, (a, b) in enumerate(zip(hs[:-1], hs[1:])):
            last = i == len(hs) - 2
            setattr(self, f"layer{i}", FullyConnectedNet._Layer(a, b, None if last else act, NORM2MOM[act_name]))
