"""The asynchronous GemNet-OC forward (nb200_gemnet_oc_count_bounds + nb200_gemnet_oc_energy_forces_async) on the host-emulation build of
the engine source (tests/emu): bounds against real counts on adversarial geometries, bitwise agreement with the two-phase call, dead rows,
the error path of a bound that is too small, and the relaxation loop against the float64 oracle.  Workspaces are poisoned before every call
and the guard zones behind every workspace array are checked after it.  The device run of the same code is tests/test_gpu_gemnet_relax.py."""
import os
import sys
from ctypes import byref, c_int32, c_int64

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
from test_gemnet_emu import _models  # noqa: E402


@pytest.fixture(scope="module")
def runner():
    from emu_driver import load, poisoned

    from nabladft_b200.gemnet_oc import GemNetOCRunner

    net, _ = _models(True)
    r = poisoned(GemNetOCRunner)(load("gemnet_oc", ["nb200_gemnet_oc_"]))
    r.set_weights(net, torch.device("cpu"))
    return r


def _batch(zs, ps):
    sizes = [len(z) for z in zs]
    z = torch.from_numpy(np.concatenate(zs).astype(np.int32))
    pos = torch.from_numpy(np.concatenate(ps).astype(np.float32)).contiguous()
    mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32))
    return z, pos, mol_ptr, sizes


def _golden():
    g = np.load(os.path.join(HERE, "golden", "gemnet_oc_f32.npz"))
    b = g["batch"]
    return _batch([g["z"][b == m] for m in range(int(b.max()) + 1)], [g["pos"][b == m] for m in range(int(b.max()) + 1)])


def _ragged():
    from nabladft_b200.synth import synth_batch

    b = synth_batch(11, 5, heavy_min=3, heavy_max=30)
    zs = [b["z"][b["batch"] == m] for m in range(5)] + [np.array([8]), np.array([1, 1])]
    ps = [b["pos"][b["batch"] == m] for m in range(5)] + [np.zeros((1, 3)), np.array([[0, 0, 0], [0.74, 0, 0]])]
    return _batch(zs, ps)


def _small(seed=3, n=(7, 5)):
    rng = np.random.default_rng(seed)
    zs = [rng.choice([1, 6, 7, 8], size=k) for k in n]
    ps = [rng.normal(size=(k, 3)) * 1.3 for k in n]
    return _batch(zs, ps)


def _real_counts(runner, pos, mol_ptr, sizes):
    lib, n = runner.lib, int(mol_ptr[-1])
    gb = torch.empty(lib.nb200_gemnet_oc_graph_bytes(n, max(sizes)), dtype=torch.uint8).fill_(255)
    out = (c_int64 * 8)()
    assert lib.nb200_gemnet_oc_graph_count(byref(runner._w), pos.data_ptr(), mol_ptr.data_ptr(), len(sizes), n, max(sizes), gb.data_ptr(), gb.numel(), out, None) == 0
    return [int(out[k]) for k in range(5)]


def _assert_bounded(runner, ps):
    z, pos, mol_ptr, sizes = _batch([np.ones(len(p), dtype=np.int32) for p in ps], ps)
    real, bound = _real_counts(runner, pos, mol_ptr, sizes), [int(v) for v in runner.count_bounds(sizes)][:5]
    assert all(r <= b for r, b in zip(real, bound)), (sizes, real, bound)
    return real, bound


def test_bounds_hold_on_adversarial_geometries(runner):
    rng = np.random.default_rng(0)
    hub = np.concatenate([np.zeros((1, 3)), 11.0 * (v := rng.normal(size=(59, 3))) / np.linalg.norm(v, axis=1, keepdims=True)])  # a hub inside everybody's cutoff whose 59 mates tie at one distance
    hub_last = hub[::-1].copy()  # ... and with the highest index, where the symmetrised graph keeps what the OTHER atom selects
    chain = np.stack([np.arange(45) * 1.1, np.zeros(45), np.zeros(45)], 1)
    blob = rng.uniform(0, 1.0 / np.sqrt(3), size=(64, 3))  # all within 1 A: every cap binds, every pair is inside the cutoff
    for p in (hub, hub_last, chain, blob):
        _assert_bounded(runner, [p])
    real, bound = _assert_bounded(runner, [blob])
    assert real[0] == bound[0] == 64 * 63 and real[2] == bound[2] == 64 * 20 and real[3] == bound[3] == 64 * 8  # these bounds are attained
    real, bound = _assert_bounded(runner, [np.zeros((1, 3)), np.array([[0, 0, 0], [0.9, 0, 0]]), chain[:31], blob[:9], np.zeros((1, 3)) + 50.0])
    assert bound[:4] == [0 + 2 + 31 * 30 + 72, 0 + 2 + 31 * 30 + 72, 2 + 31 * 20 + 72, 2 + 31 * 8 + 72] and real[1] > 0
    big = rng.uniform(0, 40.0, size=(1001, 3))  # max_neighbors_aint + 1 atoms, most pairs outside the cutoff
    _assert_bounded(runner, [big])


def test_bounds_hold_on_random_batches(runner):
    from hypothesis import given, settings
    from hypothesis import strategies as st

    @settings(max_examples=30, deadline=None, derandomize=True)
    @given(st.lists(st.integers(1, 48), min_size=1, max_size=5), st.floats(0.3, 6.0), st.integers(0, 2 ** 31))
    def check(sizes, spread, seed):
        rng = np.random.default_rng(seed)
        ps = [np.round(rng.normal(size=(k, 3)) * spread, 1) for k in sizes]  # rounding makes distance ties (and coincident atoms) common
        _assert_bounded(runner, ps)

    check()


def test_bounds_refuse_bad_molecule_pointers_and_int32_overflow(runner):
    lib, out = runner.lib, (c_int64 * 8)()
    ok = (c_int32 * 3)(0, 4, 9)
    assert lib.nb200_gemnet_oc_count_bounds(byref(runner._w), ok, 2, out) == 0
    assert [out[k] for k in range(8)] == [12 + 20, 12 + 20, 12 + 20, 12 + 20, 12 * 3 + 20 * 4, 0, 0, 0]
    assert lib.nb200_gemnet_oc_count_bounds(None, ok, 2, out) == -1 and lib.nb200_gemnet_oc_count_bounds(byref(runner._w), None, 2, out) == -1
    assert lib.nb200_gemnet_oc_count_bounds(byref(runner._w), ok, 0, out) == -1 and lib.nb200_gemnet_oc_count_bounds(byref(runner._w), ok, 2, None) == -1
    assert lib.nb200_gemnet_oc_count_bounds(byref(runner._w), (c_int32 * 3)(1, 4, 9), 2, out) == -1   # does not start at 0
    assert lib.nb200_gemnet_oc_count_bounds(byref(runner._w), (c_int32 * 3)(0, 4, 4), 2, out) == -1   # empty molecule
    assert lib.nb200_gemnet_oc_count_bounds(byref(runner._w), (c_int32 * 2)(0, 50000), 1, out) == -1  # 2.5e9 atom-atom pairs


@pytest.mark.parametrize("which", ["golden", "ragged"])
def test_async_call_equals_two_phase_call_bitwise_and_dead_rows_are_dead(runner, which):
    z, pos, mol_ptr, sizes = _golden() if which == "golden" else _ragged()
    E0, F0 = runner.guarded(runner.run, z, pos, mol_ptr, len(sizes), max(sizes))
    counts = runner.last_counts
    bounds = runner.count_bounds(sizes)
    assert any(counts[k] < int(bounds[i]) for i, k in enumerate(("A2A", "MAIN", "AE", "Q", "TIN")))  # there ARE dead rows in this batch
    outs = []
    for fill in (255, 0):  # rows at or past the real counts hold whatever the workspace held: NaN / -1 words, then zeros
        runner.fill = fill
        E, F, st = runner.guarded(runner.launch, z, pos, mol_ptr, len(sizes), max(sizes), bounds)
        outs.append((E.clone(), F.clone(), st.clone()))
    runner.fill = 255
    mol = np.repeat(np.arange(len(sizes)), sizes)
    d = np.linalg.norm(pos.numpy()[:, None, :] - pos.numpy()[None, :, :], axis=-1)
    near = (d < 12.0) & (mol[:, None] == mol[None, :]) & ~np.eye(len(z), dtype=bool)
    for E, F, st in outs:
        assert torch.equal(E, E0) and torch.equal(F, F0)
        assert st.tolist()[:2] == [counts["MAIN"], 0] and st.tolist()[4:] == [counts["A2A"], counts["AE"], counts["Q"], counts["TIN"]]
        # an atom without any in-cutoff mate has no main-graph edge (and only such an atom: its nearest mate selects it or is selected by it)
        assert 0 < int(st[2]) <= max(sizes) - 1 and int(st[3]) == int((near.sum(1) == 0).sum())


def test_bound_that_is_too_small_ends_in_ecapacity_nan_outputs_and_intact_guards(runner):
    z, pos, mol_ptr, sizes = _small()
    real = _real_counts(runner, pos, mol_ptr, sizes)
    assert all(r > 0 for r in real)
    E0, F0, st0 = runner.guarded(runner.launch, z, pos, mol_ptr, len(sizes), max(sizes), (c_int64 * 8)(*real, 0, 0, 0))  # exact counts as bounds: fine
    assert int(st0[1]) == 0 and bool(torch.isfinite(E0).all() and torch.isfinite(F0).all())
    for k in range(5):
        short = (c_int64 * 8)(*[r - (1 if i == k else 0) for i, r in enumerate(real)], 0, 0, 0)
        E, F, st = runner.guarded(runner.launch, z, pos, mol_ptr, len(sizes), max(sizes), short)
        assert int(st[1]) == -4, (k, st.tolist())
        assert st.tolist()[0] == real[1] and st.tolist()[4:] == [real[0], real[2], real[3], real[4]]  # the real counts are still reported
        assert bool(torch.isnan(E).all() and torch.isnan(F).all())
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.gemnet_oc import GemNetOCEngine

    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        GemNetOCEngine.raise_on_status(st)


def test_no_edges_and_non_finite_positions_end_in_an_error_code_and_nan_outputs(runner):
    z, pos, mol_ptr, sizes = _small()
    bounds = runner.count_bounds(sizes)
    far = pos.clone()
    far[:, 0] += torch.arange(len(z)) * 100.0  # nobody inside anybody's cutoff
    E, F, st = runner.guarded(runner.launch, z, far.contiguous(), mol_ptr, len(sizes), max(sizes), bounds)
    assert st.tolist()[:4] == [0, -6, 0, len(z)] and bool(torch.isnan(E).all() and torch.isnan(F).all())
    for bad in (float("nan"), float("inf"), -float("inf")):
        p = pos.clone()
        p[3, 1] = bad
        E, F, st = runner.guarded(runner.launch, z, p, mol_ptr, len(sizes), max(sizes), bounds)
        assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    E, F, st = runner.guarded(runner.launch, z, pos, mol_ptr, len(sizes), max(sizes), bounds)  # and the engine is usable afterwards
    assert int(st[1]) == 0 and bool(torch.isfinite(F).all())


def test_relaxation_loop_on_the_async_forward_follows_the_float64_oracle_loop(runner):
    """oracle/lbfgs.py steps (the device step kernel is CUDA only) driven by the emulated asynchronous forward, against the same loop driven
    by oracle/gemnet_oc.py in float64."""
    from oracle.lbfgs import BatchLBFGS

    z, pos, mol_ptr, sizes = _small(seed=5, n=(6, 4))
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    _, ora = _models(True)
    ora = ora.double()
    bounds = runner.count_bounds(sizes)

    def f_engine(p):
        E, F, st = runner.guarded(runner.launch, z, torch.from_numpy(p.astype(np.float32)).contiguous(), mol_ptr, len(sizes), max(sizes), bounds)
        assert int(st[1]) == 0
        return E.numpy().copy(), F.numpy().copy()

    def f_oracle(p):
        with torch.no_grad():
            E, F = ora(z.long(), torch.from_numpy(p), batch)
        return E.numpy(), F.numpy().astype(np.float32)

    p0 = pos.numpy().astype(np.float64)
    _, _, traj_e = BatchLBFGS(f_engine, sizes).run(p0, fmax=1e-5, steps=5)
    _, _, traj_o = BatchLBFGS(f_oracle, sizes).run(p0, fmax=1e-5, steps=5)
    assert len(traj_e) == len(traj_o) == 6 and np.abs(traj_e[1] - p0).max() > 1e-3
    for k in range(6):
        assert np.abs(traj_e[k] - traj_o[k]).max() < 1e-5, k


def test_engine_adapter_host_logic(runner):
    """GemNetOCEngine with the emulation runner: `run` validates the batch once and fixes the bounds, `launch` refuses another batch,
    weights are re-exported when a parameter changed."""
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.gemnet_oc import GemNetOCEngine

    net, _ = _models(True)
    eng = GemNetOCEngine(net, type(runner)(runner.lib))
    z, pos, mol_ptr, sizes = _small()
    E, F, host = eng.run(z, pos, mol_ptr, len(sizes))
    assert eng.bounds["A2A"] == 7 * 6 + 5 * 4 and int(host[1]) == 0 and len(host) == 8
    E2, F2, _ = eng.launch(z, pos, mol_ptr, len(sizes), e_cap=123)
    assert torch.equal(E, E2) and torch.equal(F, F2)
    with torch.no_grad():
        net.out_energy.linear.weight.mul_(2.0)
    E3, _, _ = eng.run(z, pos, mol_ptr, len(sizes))
    assert np.allclose(E3.numpy(), 2.0 * E.numpy(), rtol=1e-5)
    other = mol_ptr.clone()
    with pytest.raises(NablaB200Error, match="run\\(\\)"):
        eng.launch(z, pos, other, len(sizes))
    with pytest.raises(NablaB200Error, match="mol_ptr"):
        eng.run(z, pos, torch.tensor([0, 7, 7, 12], dtype=torch.int32), 3)
    eng.raise_on_status(torch.tensor([10, 0, 3, 0]))
    with pytest.raises(NablaB200Error, match="non-finite"):
        eng.raise_on_status(torch.tensor([10, -1, 3, 0, 0, 0, 0, 0]))


def test_c_abi_argument_checks_of_the_async_entry_and_exported_symbols(runner):
    from nabladft_b200 import _lib

    for name in ("nb200_gemnet_oc_count_bounds", "nb200_gemnet_oc_energy_forces_async"):
        assert name in _lib.SIGNATURES and hasattr(runner.lib, name) and hasattr(_lib.load(), name)
    hdr = open(os.path.join(HERE, "..", "include", "nabla_b200.h")).read()
    assert "int nb200_gemnet_oc_count_bounds(" in hdr and "int nb200_gemnet_oc_energy_forces_async(" in hdr
    real = _lib.load()  # the pure host function of the CUDA library agrees with the emulation build
    a, b, ptr = (c_int64 * 8)(), (c_int64 * 8)(), (c_int32 * 4)(0, 1, 3, 40)
    assert real.nb200_gemnet_oc_count_bounds(byref(runner._w), ptr, 3, a) == 0 == runner.lib.nb200_gemnet_oc_count_bounds(byref(runner._w), ptr, 3, b)
    assert list(a) == list(b)

    z, pos, mol_ptr, sizes = _small()
    lib, w, n = runner.lib, runner._w, len(z)
    bounds = runner.count_bounds(sizes)
    gb = torch.zeros(lib.nb200_gemnet_oc_graph_bytes(n, max(sizes)), dtype=torch.uint8)
    ws = torch.zeros(lib.nb200_gemnet_oc_workspace_bytes(byref(w), len(sizes), n, bounds), dtype=torch.uint8)
    e, f, st = torch.zeros(2), torch.zeros(n, 3), torch.full((8,), 77, dtype=torch.int32)

    def call(**kw):
        a = dict(eng=runner._h, w=byref(w), z=z.data_ptr(), pos=pos.data_ptr(), mol_ptr=mol_ptr.data_ptr(), n_mol=2, n=n, mx=max(sizes), gb=gb.data_ptr(),
                 gbytes=gb.numel(), bounds=bounds, ws=ws.data_ptr(), wbytes=ws.numel(), e=e.data_ptr(), f=f.data_ptr(), st=st.data_ptr())
        a.update(kw)
        return lib.nb200_gemnet_oc_energy_forces_async(*a.values(), None)

    for bad in (dict(eng=None), dict(w=None), dict(z=None), dict(pos=None), dict(mol_ptr=None), dict(n_mol=0), dict(n=0), dict(mx=0), dict(gb=None),
                dict(gbytes=gb.numel() - 1), dict(bounds=None), dict(ws=None), dict(wbytes=ws.numel() - 1), dict(e=None), dict(f=None), dict(st=None),
                dict(bounds=(c_int64 * 8)(-1, 1, 1, 1, 1)), dict(bounds=(c_int64 * 8)(1, 2 ** 31, 1, 1, 1))):
        assert call(**bad) == -1, bad
    assert st.tolist() == [77] * 8 and float(f.abs().sum()) == 0.0  # refused before anything was touched
    assert call() == 0 and int(st[1]) == 0
