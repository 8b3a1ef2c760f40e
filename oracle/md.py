"""CPU restatement of the reference's molecular dynamics jobs.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The reference's `PYGAseInterface.init_md` / `run_md` / `_init_velocities` (nablaDFT/optimization/pyg_ase_interface.py:207-294) drive ASE:
`VelocityVerlet(atoms, dt)` or `Langevin(atoms, dt, temp_bath * kB, 1 / (100 fs))` (fixcm=True), `MaxwellBoltzmannDistribution`,
`Stationary`, `ZeroRotation`, an `MDLogger` and a `Trajectory` attached with `interval`.

**[3P-memory]** ASE is not installed here: every algorithm below is restated from memory of ASE 3.22 (the version the reference pins)
and must be treated as "verify when a wheel is available":
    VelocityVerlet.step                 p += dt/2 F;  r += dt p / m;  F(r);  p += dt/2 F
    Langevin.updatevars / step          c1..c5 with sigma = sqrt(2 kT gamma / m); rnd_pos = c5 eta, rnd_vel = c3 xi - c4 eta, fixcm
                                        corrections, two half-kicks with the same xi, eta, v recomputed from the drift
    MaxwellBoltzmannDistribution        p = N(0, 1) sqrt(m kT)
    Stationary / ZeroRotation           preserve_temperature=True: force_temperature back to the temperature found on entry
    Dynamics.irun / MDLogger            forces once before the first step, log at nsteps % interval == 0 (step 0 only when nsteps == 0)
Units: ASE 3.22 defaults (CODATA 2014).  Two deliberate deviations, shared with the device code: a principal moment of inertia below
1e-10 of the largest counts as zero (ASE divides by rounding noise for linear molecules), and a molecule without kinetic energy is not
rescaled (ASE computes 0/0 for one atom).

The random numbers are not numpy's: the device draws them from a counter-based Philox4x32-10 stream (layout in
nabladft_b200/csrc/md.cu), restated here bit for bit so that the device can be compared with this oracle step by step.

Pin status: UNPINNED against ASE itself (not installable); tests/test_md_host.py checks the restatement against closed-form
recurrences and physical invariants, tests/test_gpu_md.py checks the device against it.
"""
import numpy as np

# ASE 3.22 units (ase.units, CODATA 2014)
FS = 0.09822694788464063       # 1 fs in ASE time
KB = 8.617330337217213e-05     # eV / K

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
STREAM_MAXWELL, STREAM_LANGEVIN = 0, 1


def philox4x32_10(counter, key):
    """Philox4x32-10 (Random123): counter uint32 [..., 4], key uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    counter = np.asarray(counter, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c = [counter[..., i] for i in range(4)]
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c, -1).astype(np.uint32)


def _u53(a, b):
    """53-bit uniform in (0, 1] from two words."""
    return ((a >> np.uint32(5)).astype(np.float64) * 67108864.0 + (b >> np.uint32(6)).astype(np.float64) + 1.0) * (1.0 / 9007199254740992.0)


def normal_pairs(seed, atoms, step, stream, call):
    """Two standard normals per atom from one Philox call: counter (atom, step, stream, call), key = the 64-bit seed."""
    atoms = np.asarray(atoms, dtype=np.uint64)
    ctr = np.stack([atoms, np.full_like(atoms, step), np.full_like(atoms, stream), np.full_like(atoms, call)], -1)
    seed = int(seed)
    w = philox4x32_10(ctr, np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64))
    r = np.sqrt(-2.0 * np.log(_u53(w[..., 0], w[..., 1])))
    th = 2.0 * np.pi * _u53(w[..., 2], w[..., 3])
    return r * np.cos(th), r * np.sin(th)


def maxwell_normals(seed, n_atoms, step):
    """[n, 3] normals of the Maxwell-Boltzmann draw: calls 0, 1 of stream 0 -> (x, y), (z, unused)."""
    a = np.arange(n_atoms)
    x, y = normal_pairs(seed, a, step, STREAM_MAXWELL, 0)
    z, _ = normal_pairs(seed, a, step, STREAM_MAXWELL, 1)
    return np.stack([x, y, z], -1)


def langevin_normals(seed, n_atoms, step):
    """(xi, eta), each [n, 3], of one Langevin step: calls 0, 1, 2 of stream 1 -> (xi_x, xi_y), (xi_z, eta_x), (eta_y, eta_z)."""
    a = np.arange(n_atoms)
    n = [normal_pairs(seed, a, step, STREAM_LANGEVIN, c) for c in range(3)]
    xi = np.stack([n[0][0], n[0][1], n[1][0]], -1)
    eta = np.stack([n[1][1], n[2][0], n[2][1]], -1)
    return xi, eta


# ---------------------------------------------------------------------------------------------------------------- ase.Atoms pieces
def kinetic_energy(p, m):
    return 0.5 * np.vdot(p, p / m[:, None])


def temperature(p, m):
    return 2.0 * kinetic_energy(p, m) / (3 * len(m) * KB)


def _force_temperature(p, m, temp0):
    eps = 2.0 * kinetic_energy(p, m) / (3 * len(m))
    if eps == 0.0:  # deviation: no 0/0
        return p
    return p * np.sqrt(temp0 * KB / eps)


def stationary(p, m):
    t0 = temperature(p, m)
    if len(m) == 1:
        p = np.zeros_like(p)  # p - (p / m) m can leave a rounding residue for one atom
    else:
        p = p - (p.sum(0) / m.sum()) * m[:, None]
    return _force_temperature(p, m, t0)


def zero_rotation(p, m, r):
    t0 = temperature(p, m)
    com = (m[:, None] * r).sum(0) / m.sum()
    x = r - com
    L = np.cross(x, p).sum(0)
    I = np.zeros((3, 3))
    I[0, 0] = (m * (x[:, 1] ** 2 + x[:, 2] ** 2)).sum()
    I[1, 1] = (m * (x[:, 0] ** 2 + x[:, 2] ** 2)).sum()
    I[2, 2] = (m * (x[:, 0] ** 2 + x[:, 1] ** 2)).sum()
    I[0, 1] = I[1, 0] = -(m * x[:, 0] * x[:, 1]).sum()
    I[0, 2] = I[2, 0] = -(m * x[:, 0] * x[:, 2]).sum()
    I[1, 2] = I[2, 1] = -(m * x[:, 1] * x[:, 2]).sum()
    ip, vecs = np.linalg.eigh(I)
    basis = vecs.T
    lp = basis @ L
    keep = ip > 1e-10 * ip.max()  # deviation: ASE keeps every I_p > 0
    omega = np.linalg.inv(basis) @ np.where(keep, lp / np.where(keep, ip, 1.0), 0.0)
    v = p / m[:, None] - np.cross(omega, x)
    return _force_temperature(v * m[:, None], m, t0)


def init_momenta(masses, positions, sizes, kT, seed, noise_step):
    """PYGAseInterface._init_velocities for every molecule of the batch: Maxwell-Boltzmann, Stationary, ZeroRotation."""
    m_all = np.asarray(masses, dtype=np.float64)
    p = maxwell_normals(seed, len(m_all), noise_step) * np.sqrt(m_all * kT)[:, None]
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    out = np.zeros_like(p)
    for a, b in zip(ptr[:-1], ptr[1:]):
        if b == a:
            continue
        q = stationary(p[a:b], m_all[a:b])
        out[a:b] = zero_rotation(q, m_all[a:b], np.asarray(positions[a:b], dtype=np.float64))
    return out


# ---------------------------------------------------------------------------------------------------------------- dynamics
class BatchMD:
    """The reference's init_md / run_md for a batch of independent molecules.  force_fn(pos [N,3] float64) -> (energy [B], forces [N,3]) in
    the model's units; e_scale / f_scale convert them to eV and eV/A (forces are widened to float64 first).  Noise step counter: one per
    velocity draw and one per MD step, never reset."""

    def __init__(self, force_fn, sizes, masses, positions, seed=0, e_scale=1.0, f_scale=1.0):
        self.force_fn, self.sizes = force_fn, np.asarray(sizes, dtype=np.int64)
        self.ptr = np.concatenate([[0], np.cumsum(self.sizes)])
        self.m = np.asarray(masses, dtype=np.float64)
        self.pos = np.asarray(positions, dtype=np.float64).copy()
        self.mom = np.zeros_like(self.pos)
        self.seed, self.e_scale, self.f_scale = int(seed), float(e_scale), float(f_scale)
        self.noise = 0
        self.dynamics = None
        self.forces = self.energy = None

    def init_md(self, time_step=0.5, temp_init=300, temp_bath=None, reset=False, interval=1):
        if self.dynamics is None or reset:
            self.mom = init_momenta(self.m, self.pos, self.sizes, temp_init * KB, self.seed, self.noise)
            self.noise += 1
        self.dt = time_step * FS
        self.langevin = temp_bath is not None
        self.kT = temp_bath * KB if self.langevin else 0.0
        self.gamma = 1.0 / (100.0 * FS)
        self.interval = int(interval)
        self.dynamics = "Langevin" if self.langevin else "VelocityVerlet"
        self.nsteps = 0
        self.log, self.frames = [], []

    def _evaluate(self):
        e, f = self.force_fn(self.pos)
        self.energy = np.asarray(e, dtype=np.float64) * self.e_scale
        self.forces = np.asarray(f).astype(np.float64) * self.f_scale

    def _record(self):
        ek = np.array([kinetic_energy(self.mom[a:b], self.m[a:b]) for a, b in zip(self.ptr[:-1], self.ptr[1:])])
        t = self.nsteps * self.dt / (1000.0 * FS)
        temp = 2.0 * ek / (3 * self.sizes * KB)
        self.log.append(np.stack([np.full_like(ek, t), self.energy + ek, self.energy, ek, temp], -1))
        self.frames.append(self.pos.copy())

    def run_md(self, steps):
        if self.dynamics is None:
            raise AttributeError("Dynamics need to be initialized using the 'setup_md' function")
        if self.forces is None:
            self._evaluate()
        if self.nsteps == 0:
            self._record()
        for _ in range(int(steps)):
            self.start(self.noise)
            self._evaluate()
            self.finish(self.noise)
            self.noise += 1
            self.nsteps += 1
            if self.nsteps % self.interval == 0:
                self._record()

    # -- one step = start (first half-kick + drift), force evaluation, finish (second half-kick)
    def _langevin_noise(self, step):
        xi, eta = langevin_normals(self.seed, len(self.m), step)
        m = self.m[:, None]
        dt, g = self.dt, self.gamma
        sigma = np.sqrt(2.0 * self.kT * g / m)
        c3 = np.sqrt(dt) * sigma / 2.0 - dt ** 1.5 * g * sigma / 8.0
        c5 = dt ** 1.5 * sigma / (2.0 * np.sqrt(3.0))
        c4 = g / 2.0 * c5
        rnd_pos, rnd_vel = c5 * eta, c3 * xi - c4 * eta
        for a, b in zip(self.ptr[:-1], self.ptr[1:]):  # fixcm, per molecule
            n = b - a
            rnd_pos[a:b] -= rnd_pos[a:b].sum(0) / n
            rnd_vel[a:b] -= (m[a:b] * rnd_vel[a:b]).sum(0) / (m[a:b] * n)
        return rnd_pos, rnd_vel

    def _coef(self):
        dt, g = self.dt, self.gamma
        return dt / 2.0 - dt * dt * g / 8.0, dt * g / 2.0 - dt * dt * g * g / 8.0

    def start(self, step):
        m = self.m[:, None]
        if not self.langevin:
            self.mom = self.mom + 0.5 * self.dt * self.forces
            self.pos = self.pos + self.dt * self.mom / m
            return
        c1, c2 = self._coef()
        rnd_pos, rnd_vel = self._langevin_noise(step)
        v = self.mom / m
        v = v + (c1 * self.forces / m - c2 * v + rnd_vel)
        x = self.pos
        self.pos = x + self.dt * v + rnd_pos
        self._v = (self.pos - x - rnd_pos) / self.dt
        self.mom = self._v * m

    def finish(self, step):
        m = self.m[:, None]
        if not self.langevin:
            self.mom = self.mom + 0.5 * self.dt * self.forces
            return
        c1, c2 = self._coef()
        _, rnd_vel = self._langevin_noise(step)
        v = self._v
        v = v + (c1 * self.forces / m - c2 * v + rnd_vel)
        self.mom = v * m
