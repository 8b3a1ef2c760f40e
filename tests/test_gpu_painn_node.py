"""The fused PaiNN node kernels and their weight preparation (csrc/painn_fused.cu), and the primal per-atom kernels of csrc/painn_node.cu,
one at a time on the H100 against float64 (tests/painn_node_ref.py), through nb200_painn_test_node (the host wrappers the engine calls):

* k_prep_painn: every tile image decoded and compared bitwise with the TF32 hi / lo split of its weight block, padding included;
* k_node_fwd / k_node_bwd: every program the engine launches, at layers 0, 3 and 5 of six independently drawn layers, with 64- and
  80-atom tiles forced, at N = 1, 2, NT - 1, NT, NT + 1, 3 NT - 1 and 997: every output, saved intermediate and hand-off array within
  C_NODE A elementwise; outputs pre-filled with NaN, in-place arrays with their inputs, rows at and past N (inputs included) a NaN
  sentinel that the outputs must keep bitwise; two launches bitwise equal; the engine's width rule bitwise equal to the width it picks,
  and at N = 64 S and 64 S + 1 (S SMs) the width DESIGN.md gives;
* k_embed (and its status flag), k_silu_bwd, k_upd_combine_bwd, k_upd_norm_bwd, k_readout, k_mol_sum, k_readout_bwd, k_poison_on_error;
* every refusal of the entry point, none of which writes memory.
Each check prints its largest error as a fraction of A."""
import ctypes

import numpy as np
import pytest
import torch
from torch.func import vjp

import painn_node_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F = ref.F
EINVAL = -1
PAD = 8          # sentinel rows after every array
Z_OFFSET = 1
N_ELEM = 10
SHIFT = 0.25     # energy_shift_per_atom
ATOM_COUNTS = (1, 2, 63, 64, 65, 79, 80, 81, 191, 239, 997)  # the fused kernels' N at both widths, for the per-atom kernels
COLS = dict(q_mid=F, mu_mid=3 * F, q_mlp_in=F, VW=6 * F, nrm=F, dot=F, g1pre=F, y=3 * F, q_next=F, mu_next=3 * F, h1pre=F, xh=3 * F,
            ro_pre=F // 2, gq_a=F, gq_b=F, cur=3 * F, gn=F, gdot=F, g_xh=3 * F)


def _L():
    from nabladft_b200 import _lib

    return _lib


def call(env, op, w=True, **kw):
    """One call of nb200_painn_test_node -> (status, the tile width written back)."""
    L = _L()
    a = L.PainnNodeArgs()
    a.op = op if isinstance(op, int) else L.PN_OPS.index(op)
    if w is not None:
        a.w = ctypes.pointer(env["pw"] if w is True else w)
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(a, k, v)
    rc = L.load().nb200_painn_test_node(ctypes.byref(a), L.current_stream())
    torch.cuda.synchronize()
    return rc, a.tile


def _bits(t):
    return t.view(torch.int32)


def rows(N, cols, values=None, total=None):
    """[total (N + PAD), cols] fp32 on the GPU: rows < N = values[:N] (NaN if None), the other rows the sentinel."""
    out = torch.full((total or N + PAD, cols), ref.SENTINEL_BITS, dtype=torch.int32, device=DEV).view(torch.float32)
    out[:N] = float("nan") if values is None else values[:N].to(DEV)
    return out


def check(what, got, want, A, C, N, worst=None):
    """|got[:N] - want[:N]| <= C A (NaN fails), got[N:] the sentinel bitwise; returns the largest err / A."""
    assert bool((_bits(got[N:]) == ref.SENTINEL_BITS).all()), f"{what}: a row at or past N = {N} was written"
    g, want, A = got[:N].double(), want[:N].to(DEV), A[:N].to(DEV)
    err = (g - want).abs()
    bad = ~(err <= C * A)
    assert not bool(bad.any()), f"{what} N={N}: {int(bad.sum())} of {err.numel()} elements beyond {C:.0e} A, first at {bad.nonzero()[0].tolist()}"
    r = float(torch.nan_to_num(err / A, nan=0.0).max())
    return r if worst is None else max(worst, r)


@pytest.fixture(scope="module")
def env():
    L = _L()
    w32 = ref.weights(n_elem=N_ELEM)
    dw = {k: v.to(DEV).contiguous() for k, v in w32.items()}
    pw = L.PainnWeights(n_layers=ref.L, n_feat=F, n_elem=N_ELEM, z_offset=Z_OFFSET, epsilon=ref.EPS, energy_shift_per_atom=SHIFT)
    for k in ("emb", "A1", "c1", "A2", "c2", "U", "B1", "d1", "B2", "d2", "R1", "e1", "R2", "e2"):
        setattr(pw, k, dw[k].data_ptr())
    wt = torch.empty((ref.L * ref.TILES_PER_LAYER + 2) * 128 * 1024, dtype=torch.uint8, device=DEV)
    return dict(w32=w32, w=ref.d64(w32), dw=dw, pw=pw, wt=wt, x=ref.inputs(), g=ref.cotangents(), memo={})


# ------------------------------------------------------------------------------------------------------------------- weight images
def test_prep_weight_images(env):
    """Every tile: hi and lo bitwise equal to rna_tf32(w) and rna_tf32(w - hi) of its weight block and transposition, |hi + lo - w| <=
    2^-23 |w|, and the readout tiles' padding (rows 64-127, k 64-127 of the transposed tile) exactly zero."""
    env["wt"].fill_(0xFF)
    rc, _ = call(env, "PREP", wtiles=env["wt"])
    assert rc == 0
    img = env["wt"].cpu().numpy().view(np.float32).reshape(-1, 128 * 128 * 2)
    n = ref.L * ref.TILES_PER_LAYER
    for idx in range(n + 2):
        src = ref.tile_source(env["w32"], idx)
        hi, lo = ref.decode_tile(img[idx])
        want_hi, want_lo = ref.split_tf32(src)
        where = f"tile {idx} (layer {idx // ref.TILES_PER_LAYER}, t {idx % ref.TILES_PER_LAYER})" if idx < n else f"readout tile {idx - n}"
        assert np.array_equal(hi.view(np.uint32), want_hi.view(np.uint32)), f"{where}: hi differs from rna_tf32 of its weight block"
        assert np.array_equal(lo.view(np.uint32), want_lo.view(np.uint32)), f"{where}: lo differs from rna_tf32(w - hi)"
        assert np.all(np.abs(hi.astype(np.float64) + lo - src) <= 2.0 ** -23 * np.abs(src)), where
    hi, lo = ref.decode_tile(img[n])
    assert not hi[64:].view(np.uint32).any() and not lo[64:].view(np.uint32).any(), "readout tile: padding rows 64-127 not zero"
    hi, lo = ref.decode_tile(img[n + 1])
    assert not hi[:, 64:].view(np.uint32).any() and not lo[:, 64:].view(np.uint32).any(), "transposed readout tile: k 64-127 not zero"
    print(f"k_prep_painn: {n + 2} tiles bitwise equal to the split of their weight blocks")


# ------------------------------------------------------------------------------------------------------------------- fused programs
FWD_CASES = [(k, l) for k in ref.FWD_KINDS for l in (0, 3, 5) if not (k == "upd_mlp" and l == 5)]
BWD_CASES = [(k, l) for k in ref.BWD_KINDS for l in (0, 3, 5) if not (k == "mlp_upd" and l == 5)]


def _reference(env, kind, l):
    key = (kind, l)
    if key not in env["memo"]:
        if kind in ref.FWD_KINDS:
            v, A = ref.fwd_program(env["w"], kind, l, env["x"])
            ins = {k: env["x"][k] for k in (("q_mlp_in",) if kind == "mlp" else ("q_mid", "mu_mid"))}
            inplace = {}
        else:
            b = ref.bwd_inputs(env["w32"], kind, l, env["x"], env["g"])
            v, A = ref.bwd_program(env["w"], kind, l, env["x"], b)
            inplace = {k: b[k] for k in b if k in ("cur", "gq_a")}
            ins = {k: b[k] for k in b if k not in inplace}
        env["memo"][key] = ({k: t.to(DEV) for k, t in v.items()}, {k: t.to(DEV) for k, t in A.items()}, ins, inplace)
    return env["memo"][key]


def _launch(env, kind, l, N, tile, ins, inplace, outs):
    bufs = {k: rows(N, COLS[k], ins[k]) for k in ins}
    res = {k: rows(N, COLS[k], inplace.get(k)) for k in outs}
    if kind in ref.FWD_KINDS:
        upd, mlp, ro = ref.program(kind, l)
        op = "NODE_FWD"
    else:
        ro, mlp, upd = ref.program(kind, l)
        op = "NODE_BWD"
    rc, width = call(env, op, n_atoms=N, tile=tile, layer_upd=upd, layer_mlp=mlp, readout=ro, wtiles=env["wt"], **bufs, **res)
    assert rc == 0, f"{kind} layer {l} N={N} tile={tile}: status {rc}"
    return res, width


def _run_program(env, kind, l):
    v, A, ins, inplace = _reference(env, kind, l)
    outs = ref.FWD_OUT[kind] if kind in ref.FWD_KINDS else ref.BWD_OUT
    for nt in ref.NT:
        worst = {k: 0.0 for k in outs}
        for N in (1, 2, nt - 1, nt, nt + 1, 3 * nt - 1, ref.N_MAX):
            a, width = _launch(env, kind, l, N, nt, ins, inplace, outs)
            assert width == nt
            for k in outs:
                worst[k] = check(f"{kind} layer {l} NT={nt} {k}", a[k], v[k], A[k], ref.C_NODE, N, worst[k])
            b, _ = _launch(env, kind, l, N, nt, ins, inplace, outs)
            for k in outs:
                assert torch.equal(_bits(a[k]), _bits(b[k])), f"{kind} layer {l} NT={nt} N={N}: {k} differs between two launches"
            if nt == 64:  # the engine's rule picks 64-atom tiles below 64 S + 1 atoms
                c, width = _launch(env, kind, l, N, 0, ins, inplace, outs)
                assert width == 64, f"N={N}: the width rule chose {width}"
                for k in outs:
                    assert torch.equal(_bits(a[k]), _bits(c[k])), f"{kind} layer {l} N={N}: {k} of tile = 0 differs from forced 64"
        print(f"{kind} (layer {l}) NT={nt}: max |err| / A " + ", ".join(f"{k} {r:.1e}" for k, r in worst.items()) + f" (bound {ref.C_NODE:.0e})")


@pytest.mark.parametrize("kind,l", FWD_CASES, ids=[f"{k}-{l}" for k, l in FWD_CASES])
def test_node_fwd(env, kind, l):
    _run_program(env, kind, l)


@pytest.mark.parametrize("kind,l", BWD_CASES, ids=[f"{k}-{l}" for k, l in BWD_CASES])
def test_node_bwd(env, kind, l):
    _run_program(env, kind, l)


def test_width_rule(env):
    """At N = 64 S and 64 S + 1 (S SMs), tile = 0 picks the width of DESIGN.md §3 (80-atom tiles exactly when they need fewer waves), runs it
    bitwise as the forced width, and every row matches the reference."""
    S = torch.cuda.get_device_properties(0).multi_processor_count
    v, A, ins, _ = _reference(env, "mlp", 0)
    reps = (64 * S + 1 + ref.N_MAX - 1) // ref.N_MAX
    big = {k: t.repeat(reps, 1) for k, t in ins.items()}
    vb, Ab = {k: t.repeat(reps, 1) for k, t in v.items()}, {k: t.repeat(reps, 1) for k, t in A.items()}
    for N, want in ((64 * S, 64), (64 * S + 1, 80)):
        waves = {nt: ((N + nt - 1) // nt + S - 1) // S for nt in ref.NT}
        assert want == (80 if waves[80] < waves[64] else 64)
        a, width = _launch(env, "mlp", 0, N, 0, big, {}, ref.FWD_OUT["mlp"])
        assert width == want, f"N = {N} on {S} SMs: the rule picked {width}-atom tiles, DESIGN.md gives {want}"
        b, _ = _launch(env, "mlp", 0, N, want, big, {}, ref.FWD_OUT["mlp"])
        worst = 0.0
        for k in ref.FWD_OUT["mlp"]:
            assert torch.equal(_bits(a[k]), _bits(b[k])), f"N = {N}: {k} of tile = 0 differs from forced {want}"
            worst = check(f"width rule N={N} {k}", a[k], vb[k], Ab[k], ref.C_NODE, N, worst)
        print(f"N = {N} on {S} SMs: {width}-atom tiles, max |err| / A {worst:.1e}")


# ------------------------------------------------------------------------------------------------------------------- per-atom kernels
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def test_embed(env):
    gen = _gen(20)
    z = torch.randint(Z_OFFSET, Z_OFFSET + N_ELEM, (ref.N_MAX,), generator=gen, dtype=torch.int32)
    z[500], z[900] = 0, Z_OFFSET + N_ELEM  # elements outside the table
    emb = env["w32"]["emb"]
    for N in ATOM_COUNTS:
        status = torch.zeros(8, dtype=torch.int32, device=DEV)
        q, mu = rows(N, F), rows(N, 3 * F)
        zz = torch.full((N + PAD,), 10 ** 6, dtype=torch.int32, device=DEV)
        zz[:N] = z[:N].to(DEV)
        rc, _ = call(env, "EMBED", n_atoms=N, z=zz, q=q, mu=mu, status=status)
        assert rc == 0
        zi = (z[:N] - Z_OFFSET).long()
        badz = (zi < 0) | (zi >= N_ELEM)
        want_q = emb[torch.where(badz, 0, zi)]
        check("k_embed q", q, want_q.double(), want_q.double().abs(), 0.0, N)
        check("k_embed mu", mu, torch.zeros(N, 3 * F, dtype=torch.float64), torch.zeros(N, 3 * F, dtype=torch.float64), 0.0, N)
        want_status = EINVAL if bool(badz.any()) else 0
        assert int(status[1]) == want_status and int(status[0]) == 0 and not bool(status[2:].any()), (N, status.tolist())
    print("k_embed: q bitwise the table row (row 0 for an element outside it), mu zero, status[1] = NB200_EINVAL exactly when one is outside")


def test_act_bwd(env):
    gen = _gen(21)
    g0 = torch.randn(ref.N_MAX, F, generator=gen) * 10.0 ** (torch.rand(ref.N_MAX, 1, generator=gen) * 4 - 2)
    pre = torch.randn(ref.N_MAX, F, generator=gen) * 8
    p, gd = pre.double(), g0.double()
    s = torch.sigmoid(p)
    want = {0: gd * ref.dsilu(p), 1: gd * s}
    bound = {0: gd.abs() * ref.dsilu_sens(p), 1: gd.abs() * s * (1 + p.abs())}
    for kind, name in ((0, "silu"), (1, "ssp")):
        worst = 0.0
        for N in ATOM_COUNTS:
            g = rows(N, F, g0)
            rc, _ = call(env, "ACT_BWD", w=None, n=N * F, kind=kind, g=g, pre=rows(N, F, pre))
            assert rc == 0
            worst = check(f"k_silu_bwd {name}", g, want[kind], bound[kind], ref.C_POINT, N, worst)
        print(f"k_silu_bwd ({name}'): max |err| / A = {worst:.1e} (bound {ref.C_POINT:.0e})")


def _combine(VW, y):
    """The update's combine step of VW [N, 6F] and y [N, 3F]: (q' - q, mu' - mu); its vjp is k_upd_combine_bwd."""
    N = VW.shape[0]
    V, Wv = VW.view(N, 3, 2, F)[:, :, 0], VW.view(N, 3, 2, F)[:, :, 1]
    return y[:, :F] + y[:, 2 * F:] * (V * Wv).sum(1), (y[:, None, F:2 * F] * Wv).reshape(N, 3 * F)


def test_upd_combine_bwd(env):
    gen = _gen(22)
    n = ref.N_MAX
    VW, y = torch.randn(n, 6 * F, generator=gen), torch.randn(n, 3 * F, generator=gen)
    VW[::7] = 0.0
    gq, gmu = torch.randn(n, F, generator=gen), torch.randn(n, 3 * F, generator=gen)
    _, pull = vjp(_combine, VW.double(), y.double())
    gVW, gy = pull((gq.double(), gmu.double()))
    _, pull = vjp(_combine, VW.double().abs(), y.double().abs())
    AVW, Ay = pull((gq.double().abs(), gmu.double().abs()))
    Ay[:, :F] = gq.double().abs()
    wy, wv = 0.0, 0.0
    for N in ATOM_COUNTS:
        o_gy, o_gVW = rows(N, 3 * F), rows(N, 6 * F)
        rc, _ = call(env, "UPD_COMBINE_BWD", w=None, n_atoms=N, gq=rows(N, F, gq), gmu=rows(N, 3 * F, gmu), y=rows(N, 3 * F, y),
                     VW=rows(N, 6 * F, VW), gy=o_gy, gVW=o_gVW)
        assert rc == 0
        wy = check("k_upd_combine_bwd gy", o_gy, gy, Ay, ref.C_POINT, N, wy)
        wv = check("k_upd_combine_bwd gVW", o_gVW, gVW, AVW, ref.C_POINT, N, wv)
    print(f"k_upd_combine_bwd: max |err| / A gy {wy:.1e}, gVW {wv:.1e} (bound {ref.C_POINT:.0e})")


def test_upd_norm_bwd(env):
    gen = _gen(23)
    n = ref.N_MAX
    VW = torch.randn(n, 6 * F, generator=gen)
    VW[::7] = 0.0
    V = VW.double().view(n, 3, 2, F)[:, :, 0]
    nrm = torch.sqrt((V * V).sum(1) + ref.EPS).float()
    gn, pre = torch.randn(n, F, generator=gen), torch.randn(n, 6 * F, generator=gen)
    s = gn.double() / nrm.double()
    want = pre.double().clone().view(n, 3, 2, F)
    want[:, :, 0] += s[:, None] * V
    A = pre.double().abs().view(n, 3, 2, F).clone()
    A[:, :, 0] += s.abs()[:, None] * V.abs()
    worst = 0.0
    for N in ATOM_COUNTS:
        gVW = rows(N, 6 * F, pre)
        rc, _ = call(env, "UPD_NORM_BWD", w=None, n_atoms=N, gn=rows(N, F, gn), VW=rows(N, 6 * F, VW), nrm=rows(N, F, nrm), gVW=gVW)
        assert rc == 0
        worst = check("k_upd_norm_bwd gVW (accumulated)", gVW, want.reshape(n, 6 * F), A.reshape(n, 6 * F), ref.C_POINT, N, worst)
    print(f"k_upd_norm_bwd: max |err| / A = {worst:.1e} (bound {ref.C_POINT:.0e})")


def test_readout_and_readout_bwd(env):
    gen = _gen(24)
    n, w = ref.N_MAX, env["w32"]
    pre0 = torch.randn(n, F // 2, generator=gen) * 10.0 ** (torch.rand(n, 1, generator=gen) * 2 - 1)  # |pre| < 60: sigmoid stays normal
    p = pre0 + w["e1"]  # fp32, as k_readout adds it
    pd, R2 = p.double(), w["R2"].double()
    eps_atom = (ref.silu(pd) * R2).sum(1, keepdim=True) + w["e2"].double()
    A_eps = ref.silu(pd).abs() @ R2.abs()[:, None] + w["e2"].double().abs()
    g_pre, A_g = R2 * ref.dsilu(pd), R2.abs() * ref.dsilu_sens(pd)
    we, wg = 0.0, 0.0
    for N in ATOM_COUNTS:
        pre, out = rows(N, F // 2, pre0), rows(N, 1)
        rc, _ = call(env, "READOUT", n_atoms=N, pre=pre, eps_atom=out)
        assert rc == 0
        check("k_readout pre += e1", pre, pd, pd.abs(), 0.0, N)
        we = check("k_readout eps_atom", out, eps_atom, A_eps, ref.C_SUM, N, we)
        g = rows(N, F // 2)
        rc, _ = call(env, "READOUT_BWD", n_atoms=N, pre=pre, g_pre=g)
        assert rc == 0
        wg = check("k_readout_bwd g_pre", g, g_pre, A_g, ref.C_POINT, N, wg)
    print(f"k_readout: pre + e1 bitwise, eps_atom max |err| / A = {we:.1e} (bound {ref.C_SUM:.0e}); k_readout_bwd {wg:.1e} (bound {ref.C_POINT:.0e})")


def test_mol_sum(env):
    """Molecules of 0, 1, 31-33, 65 and 4,321 atoms next to each other, and one molecule per atom count of the other tests."""
    gen = _gen(25)
    layouts = [[0, 1, 31, 32, 33, 65, 0, 4321, 1, 0], [0], [4321]] + [[N] for N in ATOM_COUNTS]
    worst = 0.0
    for sizes in layouts:
        n = sum(sizes)
        eps = torch.randn(max(n, 1), generator=gen).double() * 10.0 ** (torch.rand(max(n, 1), generator=gen) * 4 - 2)
        eps = eps.float()
        ptr = torch.tensor([0] + list(np.cumsum(sizes)), dtype=torch.int32)
        want = torch.stack([eps[a:b].double().sum() + SHIFT * (b - a) for a, b in zip(ptr[:-1].tolist(), ptr[1:].tolist())])[:, None]
        A = torch.stack([eps[a:b].double().abs().sum() + SHIFT * (b - a) for a, b in zip(ptr[:-1].tolist(), ptr[1:].tolist())])[:, None]
        energy = rows(len(sizes), 1)
        rc, _ = call(env, "MOL_SUM", n_mol=len(sizes), eps_atom=rows(n, 1, eps[:n, None]), mol_ptr=ptr.to(DEV), energy=energy)
        assert rc == 0
        worst = check(f"k_mol_sum {sizes}", energy, want, A, ref.C_SUM, len(sizes), worst)
    print(f"k_mol_sum: max |err| / A = {worst:.1e} (bound {ref.C_SUM:.0e})")


def test_poison_on_error(env):
    for flag in (0, -4, 1):
        for with_forces in (True, False):
            n_mol, nf = 5, 3 * 997
            status = torch.tensor([7, flag, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV)
            e0, f0 = torch.randn(n_mol, 1), torch.randn(nf, 1)
            energy, forces = rows(n_mol, 1, e0), rows(nf, 1, f0)
            rc, _ = call(env, "POISON", w=None, status=status, energy=energy, n_mol=n_mol, forces=forces if with_forces else None, n=nf)
            assert rc == 0
            assert bool((_bits(energy[n_mol:]) == ref.SENTINEL_BITS).all()) and bool((_bits(forces[nf:]) == ref.SENTINEL_BITS).all())
            if flag == 0:
                assert torch.equal(energy[:n_mol].cpu(), e0) and torch.equal(forces[:nf].cpu(), f0), "poisoned without an error flag"
            else:
                assert bool(energy[:n_mol].isnan().all()), "an energy survived the error flag"
                if with_forces:
                    assert bool(forces[:nf].isnan().all()), "a force survived the error flag"
                else:
                    assert torch.equal(forces[:nf].cpu(), f0), "forces = NULL, yet the forces buffer was written"


# ------------------------------------------------------------------------------------------------------------------- refusals
ALIGNED_FWD = "q_mid mu_mid VW nrm dot g1pre y q_next mu_next"
OPS = {  # op -> (program, the fields it uses, those the float4 paths need aligned, the weight fields it uses)
    "PREP": (None, "wtiles", "wtiles", "A1 A2 U B1 B2 R1"),
    "FWD_MLP": ((-1, 0, 0), "wtiles q_mlp_in h1pre xh", "wtiles q_mlp_in h1pre xh", "A1 A2 U B1 B2 R1 c1"),
    "FWD_UPD_MLP": ((0, 1, 0), f"wtiles {ALIGNED_FWD} h1pre xh", f"wtiles {ALIGNED_FWD} h1pre xh", "A1 A2 U B1 B2 R1 d1 d2 c1"),
    "FWD_UPD_RO": ((5, -1, 1), f"wtiles {ALIGNED_FWD} ro_pre", f"wtiles {ALIGNED_FWD} ro_pre", "A1 A2 U B1 B2 R1 d1 d2"),
    "BWD_RO_UPD": ((1, -1, 5), "wtiles gq_a gq_b cur gn gdot y VW nrm dot g1pre ro_pre", "wtiles gq_a gq_b cur gn gdot y VW nrm dot g1pre ro_pre",
                   "A1 A2 U B1 B2 R1 R2"),
    "BWD_MLP_UPD": ((0, 1, 0), "wtiles gq_a gq_b cur gn gdot y VW nrm dot g1pre g_xh h1pre",
                    "wtiles gq_a gq_b cur gn gdot y VW nrm dot g1pre g_xh h1pre", "A1 A2 U B1 B2 R1"),
    "EMBED": (None, "z q mu status", "q mu", "emb"),
    "ACT_BWD": (None, "g pre", "g pre", ""),
    "UPD_COMBINE_BWD": (None, "gq gmu y VW gy gVW", "gq gmu y VW gy gVW", ""),
    "UPD_NORM_BWD": (None, "gn VW nrm gVW", "gn VW nrm gVW", ""),
    "READOUT": (None, "pre eps_atom", "", "e1 R2 e2"),
    "MOL_SUM": (None, "eps_atom mol_ptr energy", "", ""),
    "READOUT_BWD": (None, "pre g_pre", "", "R2"),
    "POISON": (None, "status energy", "", ""),
}
NULL_W = object()  # a NULL weights pointer
BAD_FWD = [(0, 2, 0), (0, 1, 1), (-1, 0, 1), (-1, -1, 0), (-1, -1, 1), (0, -1, 0), (5, 6, 0), (-1, 6, 0), (6, -1, 1), (-2, 0, 0), (0, -2, 1)]
BAD_BWD = [(1, 0, 0), (0, -1, 0), (0, 2, 0), (1, -1, -1), (0, 6, 5), (1, -1, 6), (0, 0, -1), (2, -1, 0), (0, -1, -1)]


def test_refusals(env):
    """Every refusal returns NB200_EINVAL before anything is launched: every pointer addresses one sentinel buffer (weights included),
    which must keep its sentinel."""
    L = _L()
    buf = torch.full((8 << 20,), ref.SENTINEL_BITS, dtype=torch.int32, device=DEV)
    mol_ptr = torch.zeros(64, dtype=torch.int32, device=DEV)
    ptr_fields = [f for f, t in L.PainnNodeArgs._fields_ if t is ctypes.c_void_p]
    wfields = [f for f, t in L.PainnWeights._fields_ if t is ctypes.c_void_p]

    def weights(**kw):
        pw = L.PainnWeights(n_layers=ref.L, n_feat=F, n_elem=N_ELEM, z_offset=Z_OFFSET, epsilon=ref.EPS)
        for f in wfields:
            setattr(pw, f, buf.data_ptr())
        for f, v in kw.items():
            setattr(pw, f, v)
        return pw

    def rc(name, prog=None, w=None, **kw):  # w: a PainnWeights, None (the default weights) or NULL_W
        p, used, al, wf = OPS[name]
        op = "NODE_FWD" if name.startswith("FWD") else "NODE_BWD" if name.startswith("BWD") else name
        args = {f: buf.data_ptr() for f in ptr_fields}
        args.update(mol_ptr=mol_ptr.data_ptr(), n_atoms=8, n=1024, n_mol=4, kind=0)
        prog = prog or p
        if prog is not None:
            if op == "NODE_FWD":
                args.update(layer_upd=prog[0], layer_mlp=prog[1], readout=prog[2])
            else:
                args.update(readout=prog[0], layer_mlp=prog[1], layer_upd=prog[2])
        args.update(kw)
        return call(env, op, w=None if w is NULL_W else w or weights(), **args)[0]

    n_cases = 0
    for name, (prog, used, al, wf) in OPS.items():
        cases = [dict(**{f: None}) for f in used.split()] + [dict(**{f: buf.data_ptr() + 4}) for f in al.split()]
        cases += [dict(w=weights(**{f: None})) for f in wf.split()]
        cases += [dict(n_atoms=-1), dict(n=-4), dict(n_mol=-1), dict(tile=32), dict(tile=-1), dict(tile=128)]
        if name not in ("ACT_BWD", "UPD_COMBINE_BWD", "UPD_NORM_BWD", "POISON"):
            cases.append(dict(w=NULL_W))
        if name == "ACT_BWD":
            cases += [dict(n=1022), dict(kind=2), dict(kind=-1)]
        if name.startswith("FWD"):
            cases += [dict(prog=p) for p in BAD_FWD]
        if name.startswith("BWD"):
            cases += [dict(prog=p) for p in BAD_BWD]
        for c in cases:
            got = rc(name, **c)
            assert got == EINVAL, f"{name}: {c} not refused (status {got})"
            n_cases += 1
    assert rc("FWD_MLP", tile=0, n_atoms=-1) == EINVAL and call(env, -1)[0] == EINVAL and call(env, len(L.PN_OPS))[0] == EINVAL
    assert bool((buf == ref.SENTINEL_BITS).all()), "a refused call wrote memory"
    assert not bool(mol_ptr.any())
    print(f"{n_cases} refusals, none of which wrote memory")
