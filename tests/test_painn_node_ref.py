"""The float64 references of the fused PaiNN node kernels (tests/painn_node_ref.py), checked on the CPU: the forward programs against the
oracle's modules, every backward program against extrapolated central differences, and the sensitivity of the GPU checks: dropping any one
term of the programs moves some output by more than 10x the GPU tolerance C_NODE (in units of its bound A)."""
import numpy as np
import pytest
import torch

import painn_node_ref as ref
from oracle.spk import _Atomwise, _PaiNNInteraction, _PaiNNMixing

F = ref.F
N = 40  # a prefix of the synthetic inputs: isolated atoms (0, 7, ...), saturated rows (0, 11, ...) and rows of every magnitude


@pytest.fixture(scope="module")
def case():
    w32 = ref.weights()
    x = {k: v[:N] for k, v in ref.inputs().items()}
    g = {k: v[:N] for k, v in ref.cotangents().items()}
    return w32, ref.d64(w32), x, g


def _oracle(w, l):
    mix, inter, ro = _PaiNNMixing(F, epsilon=ref.EPS).double(), _PaiNNInteraction(F).double(), _Atomwise(F).double()
    with torch.no_grad():
        mix.mu_channel_mix.weight.copy_(w["U"][l])
        mix.intraatomic_context_net[0].weight.copy_(w["B1"][l]); mix.intraatomic_context_net[0].bias.copy_(w["d1"][l])
        mix.intraatomic_context_net[1].weight.copy_(w["B2"][l]); mix.intraatomic_context_net[1].bias.copy_(w["d2"][l])
        nxt = inter.interatomic_context_net
        nxt[0].weight.copy_(w["A1"][l + 1]); nxt[0].bias.copy_(w["c1"][l + 1])
        nxt[1].weight.copy_(w["A2"][l + 1]); nxt[1].bias.copy_(w["c2"][l + 1])
        ro.outnet[0].weight.copy_(w["R1"]); ro.outnet[0].bias.copy_(w["e1"])
    return mix, inter, ro


@pytest.mark.parametrize("l", [0, 3])
def test_forward_matches_the_oracle_modules(case, l):
    """update(l) = _PaiNNMixing, message MLP(l + 1) = interatomic_context_net minus c2, readout = outnet[0] minus e1."""
    w32, w, x, g = case
    mix, inter, ro = _oracle(w, l)
    q, mu = x["q_mid"].double(), x["mu_mid"].double()
    with torch.no_grad():
        qn, mun = mix(q[:, None], mu.reshape(N, 3, F))
        qn = qn[:, 0]
        xh = inter.interatomic_context_net[1](torch.nn.functional.silu(inter.interatomic_context_net[0](qn)))
        ro_pre = ro.outnet[0](qn)
    v, _ = ref.fwd_program(w, "upd_mlp", l, x)
    torch.testing.assert_close(v["q_next"], qn, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(v["mu_next"], mun.reshape(N, 3 * F), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(v["xh"] + w["c2"][l + 1], xh, rtol=1e-12, atol=1e-12)
    v, _ = ref.fwd_program(w, "upd_ro", l, x)
    torch.testing.assert_close(v["ro_pre"] + w["e1"], ro_pre, rtol=1e-12, atol=1e-12)
    assert bool((v["nrm"][0] == ref.EPS ** 0.5).all()), "atom 0 is isolated: its norm sits at the sqrt(eps) floor"


@pytest.mark.parametrize("kind", ref.BWD_KINDS)
def test_backward_matches_central_differences(case, kind):
    """<cotangents, d outputs> along a random direction of (q_mid, mu_mid), Richardson-extrapolated central differences, equals
    <(gq_a, cur), direction> of the backward program."""
    w32, w, x, g = case
    l = 3
    b = ref.bwd_inputs(w32, kind, l, x, g)
    v, _ = ref.bwd_program(w, kind, l, x, b)
    gen = torch.Generator().manual_seed(5)
    dq, dmu = torch.randn(N, F, generator=gen, dtype=ref.D64), torch.randn(N, 3 * F, generator=gen, dtype=ref.D64)
    q, mu = x["q_mid"].double(), x["mu_mid"].double()
    # relative steps; an isolated atom's mu moves by 1e-10 at most, far below the sqrt(eps) floor of its norm
    scale, smu = q.abs().amax(1, keepdim=True).clamp_min(1e-3), mu.abs().amax(1, keepdim=True).clamp_min(1e-6)

    def J(h):
        def outs(s):
            u = ref.update(w, l, q + s * h * scale * dq, mu + s * h * smu * dmu)
            if kind == "ro_upd":
                cot = (w["R2"] * ref.dsilu(b["ro_pre"].double()), b["cur"].double())
                return (ref.readout(w, u["q_next"])["ro_pre"], u["mu_next"]), cot
            return (ref.mlp(w, l + 1, u["q_next"])["xh"], u["q_next"], u["mu_next"]), (b["g_xh"].double(), b["gq_a"].double(), b["cur"].double())
        (p, cot), (m, _) = outs(1.0), outs(-1.0)
        return sum(float((c * (a - bb)).sum()) for c, a, bb in zip(cot, p, m)) / (2 * h)

    h = 1e-4
    fd = (4 * J(h / 2) - J(h)) / 3
    an = float((v["gq_a"] * scale * dq).sum() + (v["cur"] * smu * dmu).sum())
    assert abs(fd - an) <= 1e-7 * max(1.0, abs(an)), (fd, an)


def _worst(v0, v1, A, keys):
    """Largest |change| / A over the outputs `keys` (an element with A = 0 counts only if it changes)."""
    return max(float(torch.nan_to_num((v1[k] - v0[k]).abs() / A[k], nan=0.0, posinf=float("inf")).max()) for k in keys)


@pytest.mark.parametrize("drop", ["eps", "y2dot", "d2_y1", "neighbour"])
def test_forward_terms_are_visible(case, drop):
    w32, w, x, g = case
    v0, A = ref.fwd_program(w, "upd_mlp", 3, x)
    v1, _ = ref.fwd_program(w, "upd_mlp", 3, x, drop=(drop,))
    worst = _worst(v0, v1, A, ref.FWD_OUT["upd_mlp"])
    print(f"forward without {drop}: max |change| / A = {worst:.2e}")
    assert worst > 10 * ref.C_NODE


@pytest.mark.parametrize("kind", ref.BWD_KINDS)
@pytest.mark.parametrize("drop", ["eps", "y2dot", "residual", "d2_y1", "neighbour"])
def test_backward_terms_are_visible(case, kind, drop):
    w32, w, x, g = case
    b = ref.bwd_inputs(w32, kind, 3, x, g)
    v0, A = ref.bwd_program(w, kind, 3, x, b)
    v1, _ = ref.bwd_program(w, kind, 3, x, b, drop=(drop,))
    worst = _worst(v0, v1, A, ref.BWD_OUT)
    print(f"{kind} backward without {drop}: max |change| / A = {worst:.2e}")
    assert worst > 10 * ref.C_NODE


def test_mlp_uses_its_own_layer(case):
    w32, w, x, g = case
    v0, A = ref.fwd_program(w, "mlp", 3, x)
    v1, _ = ref.fwd_program(w, "mlp", 4, x)
    assert _worst(v0, v1, A, ref.FWD_OUT["mlp"]) > 10 * ref.C_NODE


def test_weight_image_layout_and_split():
    """The numpy restatement of the tile images is self-consistent: decode inverts the documented layout, the split is exact to 2^-24,
    and the readout tiles' padding is zero."""
    w = ref.weights()
    raw = np.arange(128 * 128 * 2, dtype=np.float32).reshape(2, 128, 128)
    img = np.zeros((4, 2, 8, 128, 4), np.float32)
    for hl in range(2):
        for r in range(128):
            for k in range(128):
                img[k // 32, hl, (k % 32) // 4, r, k % 4] = raw[hl, r, k]
    hi, lo = ref.decode_tile(img.reshape(-1))
    assert np.array_equal(hi, raw[0]) and np.array_equal(lo, raw[1])
    src = np.concatenate([ref.tile_source(w, i) for i in range(ref.L * ref.TILES_PER_LAYER + 2)])
    hi, lo = ref.split_tf32(src)
    assert np.all((hi.view(np.uint32) & 0x1FFF) == 0) and np.all((lo.view(np.uint32) & 0x1FFF) == 0)
    # lo keeps 11 significant bits of the up to 13 that w - hi carries: the pair is w to half an ulp of bit 22 of w's mantissa
    assert np.all(np.abs(hi.astype(np.float64) + lo - src) <= 2.0 ** -23 * np.abs(src))
    n = ref.L * ref.TILES_PER_LAYER
    assert not ref.tile_source(w, n)[64:].any() and not ref.tile_source(w, n + 1)[:, 64:].any()
    assert np.array_equal(ref.rna_tf32(np.float32([1 + 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 2.0 ** -12])), np.float32([1 + 2.0 ** -10, -(1 + 2.0 ** -10), 1]))

