"""The asynchronous DimeNet++ forward (nb200_dimenet_count_bounds + nb200_dimenet_energy_forces_async) on the host-emulation build of the
engine source (tests/emu): bounds against real counts, bitwise agreement with the two-phase call, the error paths, the device-count GEMM of
the emulation, the relaxation loop against the float64 oracle, and the host logic of `DimeNetEngine` and of `BatchwiseMD` for an engine that
cannot grow.  Buffers are poisoned before every call and the guard zones behind every workspace array are checked after it.  The device run
of the same code is tests/test_gpu_dimenet_relax.py."""
import os
import sys
from ctypes import byref, c_int32, c_int64

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))
from make_golden_dimenet import grid_molecule  # noqa: E402
from test_dimenet_emu import _models  # noqa: E402

K = 32  # dimenet_max_num_neighbors of the config


@pytest.fixture(scope="module")
def emu():
    from emu_driver import load, poisoned

    from nabladft_b200.dimenetplusplus import DimeNetRunner

    lib = load("dimenet", ["nb200_dimenet_"])
    net, ora = _models(num_blocks=2)
    r = poisoned(DimeNetRunner)(lib)
    r.set_weights(net, torch.device("cpu"))
    return r, net, ora


def _batch(zs, ps):
    sizes = [len(z) for z in zs]
    z = torch.from_numpy(np.concatenate(zs).astype(np.int32))
    pos = torch.from_numpy(np.concatenate(ps).astype(np.float32)).contiguous()
    mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32))
    return z, pos, mol_ptr, sizes


def _golden():
    g = np.load(os.path.join(HERE, "golden", "dimenet_f64.npz"))
    b = g["batch"]
    n = int(b.max()) + 1
    return _batch([g["z"][b == m] for m in range(n)], [g["pos"][b == m] for m in range(n)])


def _ragged():
    """Fixture molecules, a one-atom molecule, a molecule with an atom out of everyone's cutoff, a collinear chain."""
    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    zs = [fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in (3, 11)]
    ps = [fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in (3, 11)]
    zs += [np.array([8]), np.array([6, 1, 1]), np.array([6, 6, 8, 1])]
    ps += [np.zeros((1, 3)), np.array([[0, 0, 0], [1.1, 0, 0], [30.0, 0, 0]]), np.stack([np.arange(4) * 1.2, np.zeros(4), np.zeros(4)], 1)]
    return _batch(zs, ps)


def _small(seed=3, n=(7, 5)):
    rng = np.random.default_rng(seed)
    return _batch([rng.choice([1, 6, 7, 8], size=k) for k in n], [rng.normal(size=(k, 3)) * 1.3 for k in n])


def _counts(r, z, pos, mol_ptr, sizes):
    r.guarded(r.run, z, pos, mol_ptr, len(sizes))  # (every call is guarded: the check forgets the zones of buffers that may be freed next)
    return [r.last_counts["edges"], r.last_counts["triplets"]]


def _assert_bounded(r, ps):
    z, pos, mol_ptr, sizes = _batch([np.full(len(p), 6) for p in ps], ps)
    real, bound = list(_counts(r, z, pos, mol_ptr, sizes)), [int(v) for v in r.count_bounds(sizes)]
    assert bound[2:] == [0, 0] and real[0] <= bound[0] and real[1] <= bound[1], (sizes, real, bound)
    return real, bound[:2]


def test_bounds_hold_and_are_attained_by_a_compact_cluster(emu):
    r = emu[0]
    rng = np.random.default_rng(0)
    for m in (1, 2, 3, 10, K + 1):  # every pair within 1 A: all m - 1 sources kept, every triplet slot used
        real, bound = _assert_bounded(r, [rng.uniform(0, 1.0 / np.sqrt(3), size=(m, 3))])
        assert real == bound == [m * (m - 1), m * (m - 1) * max(m - 2, 0)], m
    for m in (K + 2, K + 10):  # truncated: the first K + 1 atoms keep K sources, the others K + 1; the edge bound is still attained
        real, bound = _assert_bounded(r, [rng.uniform(0, 1.0 / np.sqrt(3), size=(m, 3))])
        e = (K + 1) * K + (m - K - 1) * (K + 1)
        assert real[0] == bound[0] == e and real[1] <= bound[1] == e * min(m - 2, K + 1), m


def test_bounds_hold_on_the_grid_molecule_and_random_batches(emu):
    r = emu[0]
    _, g = grid_molecule()
    real, bound = _assert_bounded(r, [g.astype(np.float64)])
    assert real[0] == bound[0] == 33 * 32 + 15 * 33
    rng = np.random.default_rng(1)
    for _ in range(8):
        sizes = rng.integers(1, 48, size=rng.integers(1, 5))
        spread = rng.uniform(0.3, 4.0)
        _assert_bounded(r, [np.round(rng.normal(size=(k, 3)) * spread, 1) for k in sizes])  # rounding: ties and coincident atoms


def test_bounds_refuse_bad_molecule_pointers_and_int32_overflow(emu):
    r = emu[0]
    lib, w, out = r.lib, byref(r._w), (c_int64 * 4)()
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(0, 4, 9), 2, out) == 0
    assert list(out) == [12 + 20, 24 + 60, 0, 0]
    assert lib.nb200_dimenet_count_bounds(None, (c_int32 * 3)(0, 4, 9), 2, out) == -1
    assert lib.nb200_dimenet_count_bounds(w, None, 2, out) == -1 and lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(0, 4, 9), 2, None) == -1
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(0, 4, 9), 0, out) == -1
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(1, 4, 9), 2, out) == -1   # does not start at 0
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(0, 4, 4), 2, out) == -1   # empty molecule
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 3)(0, 4, 2), 2, out) == -1   # decreasing
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 2)(0, 2_000_000), 1, out) == -1  # 2.2e9 triplet slots
    assert lib.nb200_dimenet_count_bounds(w, (c_int32 * 2)(0, 70_000_000), 1, out) == -1  # 2.3e9 edges


@pytest.mark.parametrize("which", ["golden", "ragged"])
def test_async_call_equals_two_phase_call_bitwise(emu, which):
    r = emu[0]
    z, pos, mol_ptr, sizes = _golden() if which == "golden" else _ragged()
    E0, F0, _ = r.guarded(r.run, z, pos, mol_ptr, len(sizes))
    counts = dict(r.last_counts)
    bounds = r.count_bounds(sizes)
    assert counts["edges"] < bounds[0] and counts["triplets"] < bounds[1]  # there are dead rows
    outs = []
    for fill in (255, 0):  # rows at or past the real counts hold what the workspace held: NaN / -1 words, then zeros
        r.fill = fill
        E, F, st = r.guarded(r.launch, z, pos, mol_ptr, len(sizes), bounds)
        outs.append((E.clone(), F.clone(), st.clone()))
    r.fill = 255
    mol = np.repeat(np.arange(len(sizes)), sizes)
    d = np.linalg.norm(pos.numpy()[:, None, :] - pos.numpy()[None, :, :], axis=-1)
    iso = int((((d < 5.0) & (mol[:, None] == mol[None, :]) & ~np.eye(len(z), dtype=bool)).sum(1) == 0).sum())
    for E, F, st in outs:
        assert torch.equal(E, E0) and torch.equal(F, F0)
        assert st.tolist()[:2] == [counts["edges"], 0] and st.tolist()[3:] == [iso, counts["triplets"], 0, 0, 0]
        assert 0 < int(st[2]) <= K + 1
    assert (iso > 0) == (which == "ragged")


def test_edge_free_batch_and_isolated_atoms_match_the_two_phase_call(emu):
    r = emu[0]
    z, pos, mol_ptr, sizes = _batch([np.array([1, 6, 8]), np.array([7])], [np.array([[0, 0, 0], [9.0, 0, 0], [0, 9.0, 0]]), np.zeros((1, 3))])
    E0, F0, _ = r.guarded(r.run, z, pos, mol_ptr, len(sizes))
    E, F, st = r.guarded(r.launch, z, pos, mol_ptr, len(sizes), r.count_bounds(sizes))
    assert torch.equal(E, E0) and torch.equal(F, F0) and bool((F == 0).all())
    assert st.tolist() == [0, 0, 0, 4, 0, 0, 0, 0]


def test_bounds_below_the_counts_and_bad_inputs_give_an_error_code_nan_outputs_and_intact_guards(emu):
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.dimenetplusplus import DimeNetEngine

    r = emu[0]
    z, pos, mol_ptr, sizes = _small()
    real = list(_counts(r, z, pos, mol_ptr, sizes))
    E0, F0, st0 = r.guarded(r.launch, z, pos, mol_ptr, len(sizes), (c_int64 * 4)(*real, 0, 0))  # exact counts as bounds: fine
    assert int(st0[1]) == 0 and bool(torch.isfinite(E0).all() and torch.isfinite(F0).all())
    for k in range(2):
        short = (c_int64 * 4)(*[v - (1 if i == k else 0) for i, v in enumerate(real)], 0, 0)
        E, F, st = r.guarded(r.launch, z, pos, mol_ptr, len(sizes), short)
        assert int(st[1]) == -4 and [int(st[0]), int(st[4])] == real, (k, st.tolist())  # the real counts are still reported
        assert bool(torch.isnan(E).all() and torch.isnan(F).all())
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        DimeNetEngine.raise_on_status(st)
    bounds = r.count_bounds(sizes)
    for bad in (float("nan"), float("inf")):
        p = pos.clone()
        p[3, 1] = bad
        E, F, st = r.guarded(r.launch, z, p, mol_ptr, len(sizes), bounds)
        assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    zz = z.clone()
    zz[2] = 95
    E, F, st = r.guarded(r.launch, zz, pos, mol_ptr, len(sizes), bounds)
    assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    with pytest.raises(NablaB200Error, match="outside"):
        DimeNetEngine.raise_on_status(st)
    E, F, st = r.guarded(r.launch, z, pos, mol_ptr, len(sizes), bounds)  # and the engine is usable afterwards
    assert int(st[1]) == 0 and torch.equal(E, E0) and torch.equal(F, F0)


def test_emulated_device_count_gemm_stops_at_the_count(emu):
    from nabladft_b200 import _lib

    lib = _lib.bind(emu[0].lib, ["nb200_gemm_tf32x3_rows"])
    g = torch.Generator().manual_seed(0)
    M, N, Kd = 40, 64, 32
    A, B, bias = torch.randn(M, Kd, generator=g), torch.randn(N, Kd, generator=g), torch.randn(N, generator=g)
    for count in (17, 0, M, M + 5):
        rows = min(count, M)
        ref = torch.full((M, N), 7.0)
        assert lib.nb200_gemm_tf32x3_rows(rows, N, Kd, A.data_ptr(), Kd, B.data_ptr(), Kd, 0, ref.data_ptr(), N, 0, bias.data_ptr(), None, None, None) == 0
        C = torch.full((M, N), 7.0)
        dev = torch.tensor([count], dtype=torch.int32)
        assert lib.nb200_gemm_tf32x3_rows(M, N, Kd, A.data_ptr(), Kd, B.data_ptr(), Kd, 0, C.data_ptr(), N, 0, bias.data_ptr(), None, dev.data_ptr(), None) == 0
        assert torch.equal(C[:rows], ref[:rows]) and bool((C[rows:] == 7.0).all()), count
        if rows:
            assert torch.allclose(C[:rows], A[:rows] @ B.t() + bias, atol=1e-4)


def test_relaxation_loop_on_the_async_forward_follows_the_float64_oracle_loop(emu):
    """oracle/lbfgs.py steps (the device step kernel is CUDA only) driven by the emulated asynchronous forward, against the same loop driven
    by oracle/dimenet.py in float64."""
    from oracle.lbfgs import BatchLBFGS

    r, _, ora = emu
    z, pos, mol_ptr, sizes = _small(seed=5, n=(6, 4))
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    bounds = r.count_bounds(sizes)

    def f_engine(p):
        E, F, st = r.guarded(r.launch, z, torch.from_numpy(p.astype(np.float32)).contiguous(), mol_ptr, len(sizes), bounds)
        assert int(st[1]) == 0
        return E.numpy().copy(), F.numpy().copy()

    def f_oracle(p):
        E, F, _ = ora(z.long(), torch.from_numpy(p), batch)
        return E.detach().numpy(), F.detach().numpy().astype(np.float32)

    p0 = pos.numpy().astype(np.float64)
    _, _, traj_e = BatchLBFGS(f_engine, sizes).run(p0, fmax=1e-5, steps=5)
    _, _, traj_o = BatchLBFGS(f_oracle, sizes).run(p0, fmax=1e-5, steps=5)
    assert len(traj_e) == len(traj_o) == 6 and np.abs(traj_e[1] - p0).max() > 1e-3
    for k in range(6):
        assert np.abs(traj_e[k] - traj_o[k]).max() < 1e-5, k


def test_engine_adapter_host_logic(emu):
    """DimeNetEngine with the emulation runner: `run` validates the batch once and fixes the bounds, `launch` refuses another batch,
    weights are re-exported when a parameter changed, status errors raise and isolated atoms do not."""
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.dimenetplusplus import DimeNetEngine

    r, net, _ = emu
    eng = DimeNetEngine(net, type(r)(r.lib))
    assert eng.grows_capacity is False
    z, pos, mol_ptr, sizes = _small()
    E, F, host = eng.run(z, pos, mol_ptr, len(sizes))
    assert eng.bounds == {"edges": 7 * 6 + 5 * 4, "triplets": 7 * 6 * 5 + 5 * 4 * 3} and int(host[1]) == 0 and len(host) == 8
    E2, F2, _ = eng.launch(z, pos, mol_ptr, len(sizes), e_cap=123)
    assert torch.equal(E, E2) and torch.equal(F, F2)
    with pytest.raises(NablaB200Error, match="run\\(\\)"):
        eng.launch(z, pos, mol_ptr.clone(), len(sizes))
    with pytest.raises(NablaB200Error, match="mol_ptr"):
        eng.run(z, pos, torch.tensor([0, 7, 7, 12], dtype=torch.int32), 3)
    with torch.no_grad():
        net.regr_or_cls_nn[6].bias.add_(1.0)
    try:
        E3, _, _ = eng.run(z, pos, mol_ptr, len(sizes))
        assert np.allclose(E3.numpy() - E.numpy(), net._scale_mean()[0], rtol=1e-5)
    finally:
        with torch.no_grad():
            net.regr_or_cls_nn[6].bias.sub_(1.0)
    eng.raise_on_status(torch.tensor([10, 0, 3, 2]))  # atoms without neighbours are legal
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        eng.raise_on_status(torch.tensor([10, -4, 3, 0, 0, 0, 0, 0]))


class _OverflowingEngine:
    """An engine whose launches report NB200_ECAPACITY the first `bad` times (status on the host's CPU device)."""

    def __init__(self, grows, bad):
        if grows is not None:
            self.grows_capacity = grows
        self.e_cap, self.bad, self.calls = 0, bad, 0

    def launch(self, z, pos32, mol_ptr, n_mol, e_cap=None):
        self.calls += 1
        err = -4 if self.calls <= self.bad else 0
        return torch.zeros(n_mol), torch.zeros_like(pos32), torch.tensor([5, err, 2, 0], dtype=torch.int32)

    @staticmethod
    def raise_on_status(status_host):
        from nabladft_b200.dimenetplusplus import DimeNetEngine

        DimeNetEngine.raise_on_status(status_host)


def _md_on_host(eng):
    """A `BatchwiseMD` whose integrator launch only folds the status words as nb200_md_step does (csrc/md.cu), so its chunk logic runs
    on the CPU."""
    from nabladft_b200.md import BatchwiseMD

    md = BatchwiseMD.__new__(BatchwiseMD)
    md._pos, md._mom, md._pos32 = torch.zeros(3, 3, dtype=torch.float64), torch.zeros(3, 3, dtype=torch.float64), torch.zeros(3, 3)
    md._forces, md._energy = torch.zeros(3, 3), torch.zeros(1)
    md._z, md._mol_ptr, md.n_mol, md.n_atoms = torch.ones(3, dtype=torch.int32), torch.tensor([0, 3], dtype=torch.int32), 1, 3
    md.nsteps, md.interval, md.noise_step, md.host_syncs, md.replays, md._eng = 0, 1000, 1, 0, 0, eng

    def fold(phase, step, log=None, fpos=None, fmom=None, status=None, worst=None):
        if status is not None:
            worst[0] = max(int(worst[0]), int(status[0]))
            worst[1] = min(int(worst[1]), int(status[1]))
            worst[2] = max(int(worst[2]), int(status[2]))
            if int(status[1]) == -4:
                worst[3] = 1

    md._launch = fold
    md._append = lambda *a: None
    return md


def test_md_raises_at_once_on_ecapacity_from_an_engine_that_cannot_grow():
    from nabladft_b200._lib import NablaB200Error

    eng = _OverflowingEngine(False, bad=1)
    md = _md_on_host(eng)
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        md._chunk(5)
    assert md.replays == 0 and md.host_syncs == 1 and eng.calls == 5 and md.nsteps == 0 and md.noise_step == 1
    for grows in (None, True):  # PaiNN / SchNet engines (no attribute, or True): the chunk is replayed
        eng = _OverflowingEngine(grows, bad=1)
        md = _md_on_host(eng)
        md._chunk(5)
        assert md.replays == 1 and md.host_syncs == 2 and eng.calls == 10 and md.nsteps == 5


def test_c_abi_argument_checks_of_the_async_entry_and_exported_symbols(emu):
    from nabladft_b200 import _lib

    r = emu[0]
    for name in ("nb200_dimenet_count_bounds", "nb200_dimenet_energy_forces_async", "nb200_gemm_tf32x3_rows"):
        assert name in _lib.SIGNATURES and hasattr(r.lib, name) and hasattr(_lib.load(), name)
    hdr = open(os.path.join(HERE, "..", "include", "nabla_b200.h")).read()
    for name in ("nb200_dimenet_count_bounds", "nb200_dimenet_energy_forces_async", "nb200_gemm_tf32x3_rows"):
        assert f"int {name}(" in hdr
    real = _lib.load()  # the pure host function of the CUDA library agrees with the emulation build
    a, b, ptr = (c_int64 * 4)(), (c_int64 * 4)(), (c_int32 * 4)(0, 1, 3, 40)
    assert real.nb200_dimenet_count_bounds(byref(r._w), ptr, 3, a) == 0 == r.lib.nb200_dimenet_count_bounds(byref(r._w), ptr, 3, b)
    e37 = 33 * 32 + 4 * 33
    assert list(a) == list(b) == [0 + 2 + e37, 0 + 0 + e37 * 33, 0, 0]

    z, pos, mol_ptr, sizes = _small()
    lib, w, n = r.lib, r._w, len(z)
    bounds = r.count_bounds(sizes)
    gb = torch.zeros(lib.nb200_dimenet_graph_bytes(byref(w), n), dtype=torch.uint8)
    ws = torch.zeros(lib.nb200_dimenet_workspace_bytes(byref(w), len(sizes), n, bounds), dtype=torch.uint8)
    e, f, st = torch.zeros(2), torch.zeros(n, 3), torch.full((8,), 77, dtype=torch.int32)

    def call(**kw):
        a = dict(eng=r._h, w=byref(w), z=z.data_ptr(), pos=pos.data_ptr(), mol_ptr=mol_ptr.data_ptr(), n_mol=2, n=n, gb=gb.data_ptr(),
                 gbytes=gb.numel(), bounds=bounds, ws=ws.data_ptr(), wbytes=ws.numel(), e=e.data_ptr(), f=f.data_ptr(), st=st.data_ptr())
        a.update(kw)
        return lib.nb200_dimenet_energy_forces_async(*a.values(), None)

    for bad in (dict(eng=None), dict(w=None), dict(z=None), dict(pos=None), dict(mol_ptr=None), dict(n_mol=0), dict(n=0), dict(gb=None),
                dict(gbytes=gb.numel() - 1), dict(bounds=None), dict(ws=None), dict(wbytes=ws.numel() - 1), dict(e=None), dict(f=None),
                dict(st=None), dict(bounds=(c_int64 * 4)(-1, 1)), dict(bounds=(c_int64 * 4)(1, -1)), dict(bounds=(c_int64 * 4)(n * 33 + 1, 1)),
                dict(bounds=(c_int64 * 4)(1, 2 ** 31))):
        assert call(**bad) == -1, bad
    assert st.tolist() == [77] * 8 and float(f.abs().sum()) == 0.0  # refused before anything was touched
    assert call() == 0 and int(st[1]) == 0
