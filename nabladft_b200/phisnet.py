"""PhiSNet Clebsch-Gordan mixing layers on the H100 engine (SURVEY.md section 8 f4) -- mirrors of
`nablaDFT/phisnet/nn/modules/{clebsch_gordan,pair_mixing,self_mixing,spherical_linear}.py`: same constructor signatures, parameter names
(`coeff_{l1}_{l2}_{L}.weight`, `mixcoeff_{l1}_{l2}_{L}`, `keepcoeff_{L}`, `mixing.*`, `linear.{L}.*`) and call contracts (features = lists
over the order L of tensors [..., 2L+1, F]), so a reference state dict loads with strict=True and a PhiSNet built from the reference's
`neural_network.py` can swap these modules in.  The arithmetic is in csrc/phisnet.cu (CG contractions, real CG table of the reference
compiled in) and the wgmma 3xTF32 GEMM (distance-dependent coefficients, per-order Linear).  Inference only; CUDA only (no CPU fallback).
"""
from typing import List

import torch
from torch import nn

from . import _lib
from ._lib import NablaB200Error, check, current_stream, ptr


def _paths(o1, o2, oo, strict_upper=False):
    return [(l1, l2, L) for l1 in range(o1 + 1) for l2 in range((l1 + 1) if strict_upper else 0, o2 + 1)
            for L in range(abs(l1 - l2), min(l1 + l2, oo) + 1)]


def _pack(xs: List[torch.Tensor]):
    """list over L of [..., 2L+1, F] -> ([rows, (order+1)^2, F] contiguous fp32, leading shape)."""
    lead = xs[0].shape[:-2]
    if not xs[0].is_cuda:
        raise NablaB200Error("nabladft_b200.phisnet runs on CUDA only (no CPU fallback)")
    return torch.cat([x.reshape(-1, x.shape[-2], x.shape[-1]) for x in xs], dim=1).to(torch.float32).contiguous(), lead


def _unpack(y: torch.Tensor, order: int, lead) -> List[torch.Tensor]:
    return [y[:, L * L:(L + 1) * (L + 1), :].reshape(*lead, 2 * L + 1, y.shape[-1]) for L in range(order + 1)]


def _no_training(mod):
    if torch.is_grad_enabled() and any(p.requires_grad for p in mod.parameters()) and mod.training:
        raise NotImplementedError("nabladft_b200.phisnet layers are inference-only: call .eval() / torch.no_grad()")


class ClebschGordan(nn.Module):
    """Constructor-compatible placeholder: the real CG tensors (l <= 4) are compiled into the kernels (csrc/phisnet_cg_gen.inc)."""

    def forward(self, l1, l2, l3):
        raise NablaB200Error("the CG tensors live inside the CUDA kernels; use the mixing layers")


class PairMixing(nn.Module):
    def __init__(self, order_in1, order_in2, order_out, num_basis_functions, num_features, clebsch_gordan=None):
        super().__init__()
        self.order_in1, self.order_in2, self.order_out = order_in1, order_in2, order_out
        self.num_basis_functions, self.num_features = num_basis_functions, num_features
        self._paths = _paths(order_in1, order_in2, order_out)
        for l1, l2, L in self._paths:
            lin = nn.Linear(num_basis_functions, num_features, bias=False)
            nn.init.orthogonal_(lin.weight)
            self.add_module(f"coeff_{l1}_{l2}_{L}", lin)

    def coeff(self, l1, l2, L):
        return getattr(self, f"coeff_{l1}_{l2}_{L}")

    @torch.no_grad()
    def forward(self, x1s, x2s, rbf):
        _no_training(self)
        lib = _lib.load()
        x1, lead = _pack(x1s[: self.order_in1 + 1])
        x2, _ = _pack(x2s[: self.order_in2 + 1])
        R, F, K, npath = x1.shape[0], self.num_features, self.num_basis_functions, len(self._paths)
        r = rbf.reshape(-1, K).to(torch.float32).contiguous()
        if r.shape[0] != R:
            r = r.expand(R, K).contiguous()
        wcat = torch.cat([self.coeff(*p).weight for p in self._paths], dim=0).to(torch.float32).contiguous()  # [n_paths * F, K]
        coeff = torch.empty(R, npath * F, dtype=torch.float32, device=x1.device)
        check(lib.nb200_dense(R, npath * F, K, ptr(r), K, ptr(wcat), K, 0, ptr(coeff), npath * F, 0, None, None, 0, current_stream()), "nb200_dense")
        y = torch.empty(R, (self.order_out + 1) ** 2, F, dtype=torch.float32, device=x1.device)
        check(lib.nb200_phis_pair_mixing(ptr(x1), ptr(x2), ptr(coeff), R, F, self.order_in1, self.order_in2, self.order_out, ptr(y), current_stream()),
              "nb200_phis_pair_mixing")
        return _unpack(y, self.order_out, lead)


class SelfMixing(nn.Module):
    def __init__(self, order_in, order_out, num_features, clebsch_gordan=None):
        super().__init__()
        self.order_in, self.order_out, self.num_features = order_in, order_out, num_features
        self._paths = _paths(order_in, order_in, order_out, strict_upper=True)
        count = [0] * (order_out + 1)
        for L in range(min(order_in, order_out) + 1):
            count[L] += 1
        for _, _, L in self._paths:
            count[L] += 1
        for l1, l2, L in self._paths:
            self.register_parameter(f"mixcoeff_{l1}_{l2}_{L}", nn.Parameter(torch.empty(num_features).uniform_(-(3 / count[L]) ** 0.5, (3 / count[L]) ** 0.5)))
        for L in range(min(order_in, order_out) + 1):
            self.register_parameter(f"keepcoeff_{L}", nn.Parameter(torch.empty(num_features).uniform_(-(3 / count[L]) ** 0.5, (3 / count[L]) ** 0.5)))

    def keepcoeff(self, L):
        return getattr(self, f"keepcoeff_{L}")

    def mixcoeff(self, l1, l2, L):
        return getattr(self, f"mixcoeff_{l1}_{l2}_{L}")

    def _run(self, x, lib):
        F = self.num_features
        dev = x.device
        mix = (torch.stack([self.mixcoeff(*p) for p in self._paths]) if self._paths else torch.zeros(1, F, device=dev)).to(torch.float32).contiguous()
        keep = torch.stack([self.keepcoeff(L) for L in range(min(self.order_in, self.order_out) + 1)]).to(torch.float32).contiguous()
        y = torch.empty(x.shape[0], (self.order_out + 1) ** 2, F, dtype=torch.float32, device=dev)
        check(lib.nb200_phis_self_mixing(ptr(x), ptr(mix), ptr(keep), x.shape[0], F, self.order_in, self.order_out, ptr(y), current_stream()),
              "nb200_phis_self_mixing")
        return y

    @torch.no_grad()
    def forward(self, xs):
        _no_training(self)
        x, lead = _pack(xs[: self.order_in + 1])
        return _unpack(self._run(x, _lib.load()), self.order_out, lead)


class SphericalLinear(nn.Module):
    def __init__(self, order_in, num_in, order_out, num_out, clebsch_gordan=None, mix_orders=True, bias=True, zero_init=False):
        super().__init__()
        self.order_in, self.num_in, self.order_out, self.num_out = order_in, num_in, order_out, num_out
        self.bias, self.mix_orders = bias, mix_orders
        if mix_orders:
            self.mixing = SelfMixing(order_in, order_out, num_in, clebsch_gordan)
        elif order_in != order_out:
            raise ValueError("the order can only change if mixing is enabled")
        self.linear = nn.ModuleList([nn.Linear(num_in, num_out, bias=(bias and L == 0)) for L in range(order_out + 1)])
        for lin in self.linear:
            nn.init.zeros_(lin.weight) if zero_init else nn.init.orthogonal_(lin.weight)
        if bias:
            nn.init.zeros_(self.linear[0].bias)

    @torch.no_grad()
    def forward(self, xs):
        _no_training(self)
        lib = _lib.load()
        x, lead = _pack(xs[: self.order_in + 1])
        if self.mix_orders:
            x = self.mixing._run(x, lib)
        w_l = torch.stack([lin.weight.t() for lin in self.linear]).to(torch.float32).contiguous()  # [order_out+1][c_in][c_out]
        b = self.linear[0].bias.to(torch.float32).contiguous() if self.bias else None
        y = torch.empty(x.shape[0], (self.order_out + 1) ** 2, self.num_out, dtype=torch.float32, device=x.device)
        check(lib.nb200_phis_linear(ptr(x), ptr(w_l), ptr(b) if b is not None else None, x.shape[0], self.num_in, self.num_out, self.order_out, ptr(y),
                                    current_stream()), "nb200_phis_linear")
        return _unpack(y, self.order_out, lead)
