"""DimeNet++ relaxation and molecular dynamics on the device: the device-count GEMM (nb200_gemm_tf32x3_rows) on both GEMM kernels, the
asynchronous forward (nb200_dimenet_energy_forces_async) against the two-phase forward and its error paths, `ASEBatchwiseLBFGS` and
`BatchwiseMD` with `PyGBatchwiseCalculator(DimeNetPlusPlusPotential)` against host-driven loops and the float64 oracle.  The same checks on
the host-emulation build (guard zones included) are tests/test_dimenet_relax_emu.py."""
import math
import os
import sys
from ctypes import c_int64

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "emu"))
from make_golden_dimenet import SCALER, load_test_weights  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ES = 27.211386024367243  # Hartree -> eV (optimization.convert_units)


def _models(postprocessing=True, num_blocks=6):
    from nabladft_b200.dimenetplusplus import DimeNetPlusPlusPotential
    from oracle.dimenet import DimeNetPlusPlusPotentialOracle

    kw = dict(node_latent_dim=50, scaler=SCALER, dimenet_hidden_channels=256, dimenet_num_blocks=num_blocks, do_postprocessing=postprocessing)
    ora = load_test_weights(DimeNetPlusPlusPotentialOracle(**kw).double().eval())
    net = DimeNetPlusPlusPotential(**kw).eval()
    net.load_state_dict({k: v.float() for k, v in ora.state_dict().items()}, strict=True)
    return net.to(DEV), ora


def _fixture(mols, jitter=0.0, seed=0):
    fx = np.load(os.path.join(HERE, "golden", "fixture_molecules.npz"))
    rng = np.random.default_rng(seed)
    zs = [fx["z"][fx["ptr"][m]:fx["ptr"][m + 1]] for m in mols]
    ps = [fx["pos"][fx["ptr"][m]:fx["ptr"][m + 1]].astype(np.float64) + jitter * rng.normal(size=(len(z), 3)) for m, z in zip(mols, zs)]
    return zs, ps


def _synth(n_mol):
    from nabladft_b200.synth import synth_batch

    b = synth_batch(0, n_mol)
    p = b["mol_ptr"]
    return [b["z"][p[i]:p[i + 1]] for i in range(n_mol)], [b["pos"][p[i]:p[i + 1]].astype(np.float64) for i in range(n_mol)]


def _tensors(zs, ps):
    sizes = [len(z) for z in zs]
    z = torch.from_numpy(np.concatenate(zs).astype(np.int32)).to(DEV)
    pos = torch.from_numpy(np.concatenate(ps).astype(np.float32)).to(DEV).contiguous()
    mol_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(DEV)
    return z, pos, mol_ptr, sizes


def _atoms(zs, ps):
    from nabladft_b200.optimization import SimpleAtoms

    return [SimpleAtoms(p, z) for p, z in zip(ps, zs)]


@pytest.fixture(scope="module")
def model():
    return _models()


@pytest.fixture()
def runner(model):
    from emu_driver import poisoned

    from nabladft_b200.dimenetplusplus import DimeNetRunner

    r = poisoned(DimeNetRunner, emulated=False)()  # every (re)used buffer is filled with `fill` bytes before the call
    r.set_weights(model[0], torch.device(DEV))
    return r


# ------------------------------------------------------------------------------------------------------------ device-count GEMM
@pytest.mark.parametrize("M", [1000, 5000])  # below and above the 2048 rows where nb_gemm_tf32x3_ex switches to gemm_ps.cu
def test_gemm_with_a_device_row_count(M):
    from nabladft_b200 import _lib

    lib, s = _lib.load(), _lib.current_stream()
    g = torch.Generator(device=DEV).manual_seed(M)
    N, K = 256, 256
    A = torch.randn(M, K, device=DEV, generator=g)
    for trans in (0, 1):
        B = torch.randn(N, K, device=DEV, generator=g) if trans == 0 else torch.randn(K, N, device=DEV, generator=g)
        bias, C0 = torch.randn(N, device=DEV, generator=g), torch.randn(M, N, device=DEV, generator=g)
        for count in (M // 2 + 37, 0, M, 3 * M):
            rows = min(count, M)
            ref, ref_act = C0.clone(), torch.full((M, N), 5.0, device=DEV)
            _lib.check(lib.nb200_gemm_tf32x3(M, N, K, _lib.ptr(A), K, _lib.ptr(B), N if trans else K, trans, _lib.ptr(ref), N, 1, _lib.ptr(bias),
                                             _lib.ptr(ref_act), s), "nb200_gemm_tf32x3")
            C, act = C0.clone(), torch.full((M, N), 5.0, device=DEV)
            dev = torch.tensor([count], dtype=torch.int32, device=DEV)
            _lib.check(lib.nb200_gemm_tf32x3_rows(M, N, K, _lib.ptr(A), K, _lib.ptr(B), N if trans else K, trans, _lib.ptr(C), N, 1, _lib.ptr(bias),
                                                  _lib.ptr(act), _lib.ptr(dev), s), "nb200_gemm_tf32x3_rows")
            assert torch.equal(C[:rows], ref[:rows]) and torch.equal(act[:rows], ref_act[:rows]), (M, trans, count)
            assert torch.equal(C[rows:], C0[rows:]) and bool((act[rows:] == 5.0).all()), (M, trans, count)
            if rows and (rows >= 2048) == (M >= 2048):  # the plain call with M = count takes the same kernel
                small = C0[:rows].clone()
                _lib.check(lib.nb200_gemm_tf32x3(rows, N, K, _lib.ptr(A), K, _lib.ptr(B), N if trans else K, trans, _lib.ptr(small), N, 1,
                                                 _lib.ptr(bias), None, s), "nb200_gemm_tf32x3")
                assert torch.equal(C[:rows], small)
            none = C0.clone()
            _lib.check(lib.nb200_gemm_tf32x3_rows(M, N, K, _lib.ptr(A), K, _lib.ptr(B), N if trans else K, trans, _lib.ptr(none), N, 1, _lib.ptr(bias),
                                                  None, None, s), "nb200_gemm_tf32x3_rows")
            assert torch.equal(none, ref)  # m_dev == NULL: the plain call


# ------------------------------------------------------------------------------------------------------------ async forward
@pytest.mark.parametrize("which", ["fixture32", "synth256"])
def test_async_forward_equals_two_phase_forward(runner, which):
    z, pos, mol_ptr, sizes = _tensors(*(_fixture(range(32)) if which == "fixture32" else _synth(256)))
    E0, F0, _ = runner.run(z, pos, mol_ptr, len(sizes))
    counts = dict(runner.last_counts)
    bounds = runner.count_bounds(sizes)
    assert counts["edges"] < bounds[0] and counts["triplets"] <= bounds[1]
    outs = []
    for fill in (255, 0):
        runner.fill = fill
        E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), bounds)
        outs.append((E.clone(), F.clone(), st.cpu().tolist()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])  # nothing past a real count reaches an output
    E, F, st = outs[0]
    assert st[:2] == [counts["edges"], 0] and st[4:] == [counts["triplets"], 0, 0, 0] and 0 < st[2] <= 33
    print(f"{which}: {counts['edges']} edges (bound {bounds[0]}), {counts['triplets']} triplet slots (bound {bounds[1]}), "
          f"workspace {runner.last_workspace_bytes / 1e9:.2f} GB")
    # rows are independent in both GEMM kernels, but nb_gemm_ps_wanted hands >= 2048 rows to gemm_ps.cu, whose K loop is chunked
    # differently from gemm_tc.cu's: where count and bound fall on different sides of 2048 the calls may differ in the last bits
    if (counts["edges"] >= 2048) == (int(bounds[0]) >= 2048):
        assert torch.equal(E, E0) and torch.equal(F, F0)
    else:
        assert float((E - E0).abs().max()) <= 1e-6 * float(E0.abs().max()) and float((F - F0).abs().max()) <= 1e-5 * float(F0.abs().max())


def test_bounds_below_the_counts_and_bad_inputs_give_an_error_code_and_nan_outputs(runner):
    from nabladft_b200._lib import NablaB200Error
    from nabladft_b200.dimenetplusplus import DimeNetEngine

    z, pos, mol_ptr, sizes = _tensors(*_fixture([3, 26]))
    E0, F0, _ = runner.run(z, pos, mol_ptr, len(sizes))
    real = [runner.last_counts["edges"], runner.last_counts["triplets"]]
    for k in range(2):
        short = (c_int64 * 4)(*[v - (1 if i == k else 0) for i, v in enumerate(real)], 0, 0)
        E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), short)
        st = st.cpu().tolist()
        assert st[1] == -4 and [st[0], st[4]] == real, (k, st)
        assert bool(torch.isnan(E).all() and torch.isnan(F).all())
    with pytest.raises(NablaB200Error, match="ECAPACITY"):
        DimeNetEngine.raise_on_status(st)
    bounds = runner.count_bounds(sizes)
    bad = pos.clone()
    bad[5, 2] = float("nan")
    E, F, st = runner.launch(z, bad, mol_ptr, len(sizes), bounds)
    assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    zz = z.clone()
    zz[4] = 95
    E, F, st = runner.launch(zz, pos, mol_ptr, len(sizes), bounds)
    assert int(st[1]) == -1 and bool(torch.isnan(E).all() and torch.isnan(F).all())
    E, F, st = runner.launch(z, pos, mol_ptr, len(sizes), bounds)
    assert int(st[1]) == 0 and torch.equal(E, E0) and torch.equal(F, F0)  # a few hundred edges: both calls below 2048 rows


# ------------------------------------------------------------------------------------------------------------ L-BFGS
def _relax(model, zs, ps, steps, check_every, fixed=None, record=False, calc_cls=None, fmax=1e-5):
    from nabladft_b200.optimization import ASEBatchwiseLBFGS, PyGBatchwiseCalculator

    calc = (calc_cls or PyGBatchwiseCalculator)(model[0], device=DEV, energy_unit="Hartree", position_unit="Ang")
    opt = ASEBatchwiseLBFGS(calc, logfile=None, check_every=check_every, fixed_atoms_mask=fixed)
    opt.record_positions = record
    converged = opt.run(_atoms(zs, ps), fmax=fmax, steps=steps)
    return opt, calc, converged


def test_lbfgs_relaxation_of_32_molecules_reports_what_the_two_phase_forward_sees(model):
    """300 steps on 32 fixture molecules.  The test weights are not a physical potential (their NVE runs heat some fixture molecules to
    thousands of K), and 1000 steps do not bring all 32 below 5e-3 Ha/A, so this checks the loop's own verdict: the forces it returns are
    bitwise those of the two-phase forward at its final geometry, and it reports convergence exactly when those forces meet fmax."""
    zs, ps = _fixture(range(32), jitter=0.05, seed=1)
    fmax = 5e-3  # Ha / A
    opt, calc, converged = _relax(model, zs, ps, 300, 10, fmax=fmax)
    sizes = [len(x) for x in zs]
    off = np.concatenate([[0], np.cumsum(sizes)])
    p = np.concatenate([a.get_positions() for a in opt.atoms])
    z, pos, mol_ptr, _ = _tensors(zs, [p[a:b] for a, b in zip(off[:-1], off[1:])])
    _, F, _ = model[0]._get_runner().run(z, pos, mol_ptr, len(sizes))  # the two-phase forward at the final geometry
    F = F.cpu().numpy()
    fn = np.linalg.norm(F.astype(np.float64), axis=1)
    worst = np.array([fn[a:b].max() for a, b in zip(off[:-1], off[1:])])
    fn0 = np.linalg.norm(np.asarray(calc.results["forces"], dtype=np.float64), axis=1)
    print(f"L-BFGS, 32 fixture molecules: converged {converged} after {opt.nsteps} steps, {opt.host_syncs} host syncs; "
          f"{int((worst < fmax).sum())} molecules below fmax, largest force {worst.max():.3e} Ha/A")
    assert opt.host_syncs == 1 + math.ceil(opt.nsteps / 10) + 1 and np.isfinite(F).all()
    assert np.array_equal(F, calc.results["forces"]) and np.array_equal(fn, fn0)
    assert converged == bool((worst < fmax).all())


def test_lbfgs_device_loop_matches_a_host_driven_two_phase_loop(model):
    from nabladft_b200.dimenetplusplus import DimeNetEngine
    from nabladft_b200.optimization import PyGBatchwiseCalculator

    zs, ps = _fixture(range(32), jitter=0.05, seed=2)
    steps = 30
    o1, c1, _ = _relax(model, zs, ps, steps, 1)
    o10, c10, _ = _relax(model, zs, ps, steps, 10)
    assert o1.nsteps == o10.nsteps == steps and o1.host_syncs == 1 + steps + 1 and o10.host_syncs == 1 + 3 + 1
    p1, p10 = np.concatenate([a.get_positions() for a in o1.atoms]), np.concatenate([a.get_positions() for a in o10.atoms])
    assert np.array_equal(p1, p10) and np.array_equal(c1.results["forces"], c10.results["forces"])

    class HostDriven(DimeNetEngine):  # the two-phase forward, which waits for the counts, at every step
        def launch(self, z, pos, mol_ptr, n_mol, e_cap=None):
            energy, forces, _ = self.runner.run(z, pos, mol_ptr, n_mol)
            return energy, forces, torch.zeros(8, dtype=torch.int32, device=pos.device)

    class HostCalc(PyGBatchwiseCalculator):
        def engine(self):
            if getattr(self, "_e", None) is None:
                self._e = HostDriven(self.model, self.model._get_runner())
            return self._e

    oh, ch, _ = _relax(model, zs, ps, steps, 10, calc_cls=HostCalc)
    ph = np.concatenate([a.get_positions() for a in oh.atoms])
    # this batch has tens of thousands of edges: count and bound are both far above 2048 rows, same kernels, same bits
    assert np.array_equal(ph, p10) and np.array_equal(ch.results["energy"], c10.results["energy"])
    assert np.array_equal(ch.results["forces"], c10.results["forces"]) and np.abs(p1 - np.concatenate(ps)).max() > 1e-3


def test_fixed_atoms_do_not_move(model):
    zs, ps = _fixture([4, 11, 17], jitter=0.05, seed=2)
    fixed = [0, 3, len(zs[0]) + 2, len(zs[0]) + len(zs[1]) + 5]
    opt, calc, _ = _relax(model, zs, ps, 10, 4, fixed=fixed)
    p = np.concatenate([a.get_positions() for a in opt.atoms])
    p0 = np.concatenate(ps)
    free = np.setdiff1d(np.arange(len(p0)), fixed)
    assert np.array_equal(p[fixed], p0[fixed]) and np.abs(p[free] - p0[free]).max() > 1e-3
    assert np.all(calc.results["forces"][fixed] == 0.0) and opt.host_syncs == 1 + 3 + 1


def test_device_relaxation_follows_the_float64_oracle_loop(model):
    from oracle.lbfgs import BatchLBFGS

    rng = np.random.default_rng(5)
    sizes = [6, 4]
    zs = [rng.choice([1, 6, 7, 8], size=k) for k in sizes]
    ps = [rng.normal(size=(k, 3)) * 1.3 for k in sizes]
    opt, _, _ = _relax(model, zs, ps, 5, 1, record=True)
    ora = model[1]
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))
    z = torch.from_numpy(np.concatenate(zs)).long()

    def f_oracle(p):
        E, F, _ = ora(z, torch.from_numpy(p), batch)
        return E.detach().numpy(), F.detach().numpy().astype(np.float32)

    _, _, traj = BatchLBFGS(f_oracle, sizes).run(np.concatenate(ps), fmax=1e-5, steps=5)
    got = opt.positions_history + [np.concatenate([a.get_positions() for a in opt.atoms])]
    assert len(traj) == 6 and len(got) >= 6 and np.abs(traj[1] - traj[0]).max() > 1e-3
    for k in range(6):
        assert np.abs(got[k] - traj[k]).max() < 1e-4, k


# ------------------------------------------------------------------------------------------------------------ molecular dynamics
def _md(net, zs, ps, steps, check_every=50, seed=7, bath=None, dt=0.5, interval=1):
    from nabladft_b200.md import BatchwiseMD
    from nabladft_b200.optimization import PyGBatchwiseCalculator

    calc = PyGBatchwiseCalculator(net, device=DEV, energy_unit="Hartree", position_unit="Ang")
    md = BatchwiseMD(calc, _atoms(zs, ps), seed=seed, check_every=check_every)
    md.init_md("dpp", time_step=dt, temp_init=300, temp_bath=bath, interval=interval)
    md.run_md(steps)
    return md


def test_md_follows_the_float64_oracle(model):
    from nabladft_b200.vibrations import masses_of
    from oracle import md as omd

    net, ora = model
    zs, ps = _fixture([0, 5])
    z = torch.from_numpy(np.concatenate(zs)).long()
    batch = torch.repeat_interleave(torch.arange(2), torch.tensor([len(x) for x in zs]))

    def oracle_forces(pos):
        E, F, _ = ora(z, torch.from_numpy(np.asarray(pos, dtype=np.float32)).double(), batch)
        return E.detach().numpy(), F.detach().numpy()

    m = masses_of(torch.from_numpy(np.concatenate(zs))).numpy()
    for bath in (None, 300.0):
        md = _md(net, zs, ps, 20, check_every=8, bath=bath)
        o = omd.BatchMD(oracle_forces, [len(x) for x in zs], m, np.concatenate(ps), seed=7, e_scale=ES, f_scale=ES)
        o.init_md(time_step=0.5, temp_init=300, temp_bath=bath)
        o.run_md(20)
        dp, dm = np.abs(md.frames - np.stack(o.frames)).max(), np.abs(md.momenta - o.mom).max()
        print(f"DimeNet++ {o.dynamics}: 20 steps, max |dpos| {dp:.2e} A, max |dp| {dm:.2e}")
        assert dp < 1e-3 and dm < 2e-3


# Measured on an H100 (seed 1, fixture molecules 0 and 1, 2000 x 0.25 fs): the largest |Etot(t) - Etot(0)| is 0.018 and 0.007 eV at mean
# temperatures of about 6,100 and 6,400 K -- the test weights turn potential energy into heat.  Molecules 2-5 of the fixture heat further
# (to 9,500 K) and break up, which no fixed bound would describe; they are left out (DESIGN.md 3.15.3).
_NVE_DRIFT = 0.05  # eV


def test_nve_conserves_energy_without_postprocessing():
    net, _ = _models(postprocessing=False)
    zs, ps = _fixture([0, 1])
    md = _md(net, zs, ps, 2000, seed=1, dt=0.25, interval=10)
    etot = md.log[:, :, 1]
    drift = np.abs(etot - etot[0]).max(axis=0)
    print(f"NVE 2000 x 0.25 fs, DimeNet++ test weights, no postprocessing: max |Etot - Etot(0)| per molecule "
          f"{np.array2string(drift, precision=5)} eV; T(0) {np.array2string(md.log[0, :, 4], precision=1)} K; "
          f"mean T {np.array2string(md.log[:, :, 4].mean(0), precision=1)} K")
    assert np.isfinite(md.log).all() and drift.max() < _NVE_DRIFT


def test_md_is_deterministic_and_syncs_once_per_chunk(model):
    zs, ps = _fixture([0, 5])
    runs = {ce: _md(model[0], zs, ps, 100, check_every=ce, bath=300.0, seed=3) for ce in (1, 7, 50)}
    a = runs[50]
    for ce, md in runs.items():
        assert np.array_equal(md.positions, a.positions) and np.array_equal(md.momenta, a.momenta), ce
        assert np.array_equal(md.log, a.log) and np.array_equal(md.frames, a.frames), ce
        assert md.host_syncs == math.ceil(100 / ce) and md.replays == 0, (ce, md.host_syncs)
