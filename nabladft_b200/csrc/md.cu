// md.cu -- batched molecular dynamics on the device: velocity Verlet (NVE) and the reference's Langevin (NVT) integrator.
//
// Replaces the ASE loop behind PYGAseInterface.init_md / run_md (nablaDFT/optimization/pyg_ase_interface.py): there every step of ONE
// molecule is a model call plus a device -> host -> device round trip.  Here positions and momenta of a whole batch live in HBM next to
// the engine's buffers, one CTA per molecule (every reduction of the algorithms -- centre of mass, fixcm sums, kinetic energy -- is per
// molecule), and a step is one engine launch plus ONE launch of k_md_step on the same stream.  Semantics: ASE 3.22
// (ase.md.verlet.VelocityVerlet, ase.md.langevin.Langevin with fixcm=True, ase.md.velocitydistribution), restated in oracle/md.py.
//
// Precision: positions, momenta, masses and every reduction in float64; forces and energies arrive from the engine in fp32 and are
// widened and scaled to eV, eV/A (f_scale, e_scale) on use.  pos32 = (float)pos is the copy the engine reads.
//
// Random numbers (Langevin noise, Maxwell-Boltzmann draw): counter-based Philox4x32-10 (Salmon et al., SC'11; Random123), so that any
// step's noise can be regenerated from its counter -- both half-kicks of a Langevin step redraw the same xi, eta instead of storing them,
// and a replayed chunk draws exactly what the first attempt drew.
//   key     = (seed & 0xffffffff, seed >> 32)
//   counter = (global atom index, noise step, stream, call)      stream 0: Maxwell-Boltzmann, 1: Langevin
//   one call -> words w0..w3 -> u1 from (w0, w1), u2 from (w2, w3), u = ((w_a >> 5) * 2^26 + (w_b >> 6) + 1) * 2^-53 in (0, 1]
//            -> Box-Muller: r = sqrt(-2 ln u1), n0 = r cos(2 pi u2), n1 = r sin(2 pi u2)
//   Langevin, per atom and step: calls 0, 1, 2 -> (xi_x, xi_y), (xi_z, eta_x), (eta_y, eta_z)
//   Maxwell-Boltzmann, per atom:  calls 0, 1    -> (p_x, p_y), (p_z, unused)
// The caller never reuses a noise step for a given seed.
//
// k_md_step phases (one kernel, a mask): FINISH = second half-kick of step `step` with the new forces; then, if a log slot is given,
// per-molecule Epot / Ekin (and optionally the positions / momenta frame) of the completed step; then START = first half-kick and
// drift of step `step + 1`.  A run is START, (engine, FINISH|START) per step, engine, FINISH.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int MD_THREADS = 128;
constexpr int MD_WARPS = MD_THREADS / 32;
constexpr int MD_FINISH = 1, MD_START = 2;

// ------------------------------------------------------------------------------------------------------------ Philox4x32-10
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6) + 1.0) * (1.0 / 9007199254740992.0);
}
// two standard normals from one Philox call
__device__ __forceinline__ double2 normal2(uint64_t seed, uint32_t atom, uint32_t step, uint32_t stream, uint32_t call) {
    const uint4 w = philox4x32_10(make_uint4(atom, step, stream, call), (uint32_t)seed, (uint32_t)(seed >> 32));
    const double r = sqrt(-2.0 * log(u53(w.x, w.y)));
    double s, c;
    sincospi(2.0 * u53(w.z, w.w), &s, &c);  // = sin, cos(2 pi u2) without the large-argument reduction path of sin / cos
    return make_double2(r * c, r * s);
}

// ------------------------------------------------------------------------------------------------------------ block reductions
// K float64 sums over the CTA in a fixed order (warp butterfly, then the warps in order): bitwise reproducible run to run
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* red) {
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();  // protects `red` against the previous reduction's readers
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) red[warp * K + k] = v[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < MD_WARPS; ++w) t += red[w * K + k];
        v[k] = t;
    }
}

__device__ __forceinline__ double kinetic(const double* __restrict__ mom, const double* __restrict__ mass, int a0, int n_at, double* red) {
    double e[1] = {0.0};
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double* p = mom + 3 * (size_t)(a0 + i);
        e[0] += (p[0] * p[0] + p[1] * p[1] + p[2] * p[2]) / mass[a0 + i];
    }
    block_sum<1>(e, red);
    return 0.5 * e[0];
}

// momenta *= sqrt(e_target / e_now) (ASE force_temperature); a molecule without kinetic energy is left alone (one atom after Stationary)
__device__ __forceinline__ void rescale(double* __restrict__ mom, int a0, int n_at, double e_target, double e_now) {
    if (!(e_now > 0.0)) return;
    const double s = sqrt(e_target / e_now);
    for (int k = threadIdx.x; k < 3 * n_at; k += MD_THREADS) mom[3 * (size_t)a0 + k] *= s;
    __syncthreads();
}

// eigen-decomposition of a symmetric 3x3 matrix by cyclic Jacobi rotations (one thread): a is destroyed, w = eigenvalues,
// columns of v = eigenvectors
__device__ void jacobi3(double a[3][3], double w[3], double v[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
        const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
        if (off == 0.0 || off <= 1e-18 * diag) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (a[p][q] == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {  // A <- A J
                    const double akp = a[k][p], akq = a[k][q];
                    a[k][p] = c * akp - s * akq;
                    a[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {  // A <- J^T A
                    const double apk = a[p][k], aqk = a[q][k];
                    a[p][k] = c * apk - s * aqk;
                    a[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {  // V <- V J
                    const double vkp = v[k][p], vkq = v[k][q];
                    v[k][p] = c * vkp - s * vkq;
                    v[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < 3; ++i) w[i] = a[i][i];
}

// MaxwellBoltzmannDistribution, then Stationary and ZeroRotation, each with preserve_temperature=True (ase.md.velocitydistribution)
__global__ void __launch_bounds__(MD_THREADS) k_md_init_momenta(const int32_t* __restrict__ mol_ptr, const double* __restrict__ mass,
                                                               const double* __restrict__ pos, double kT, uint64_t seed, uint32_t noise_step,
                                                               double* __restrict__ mom) {
    __shared__ double red[MD_WARPS * 10];
    __shared__ double omega_sh[3];
    const int a0 = mol_ptr[blockIdx.x], n_at = mol_ptr[blockIdx.x + 1] - a0;
    if (n_at <= 0) return;

    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const int at = a0 + i;
        const double sd = sqrt(mass[at] * kT);
        const double2 n01 = normal2(seed, (uint32_t)at, noise_step, 0u, 0u), n23 = normal2(seed, (uint32_t)at, noise_step, 0u, 1u);
        double* p = mom + 3 * (size_t)at;
        p[0] = n01.x * sd; p[1] = n01.y * sd; p[2] = n23.x * sd;
    }
    __syncthreads();

    // ---- Stationary: p -= m P / M.  One atom: p = 0 exactly (p - (p / m) m can leave a rounding residue)
    double e0 = kinetic(mom, mass, a0, n_at, red);
    double s4[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double* p = mom + 3 * (size_t)(a0 + i);
        s4[0] += p[0]; s4[1] += p[1]; s4[2] += p[2]; s4[3] += mass[a0 + i];
    }
    block_sum<4>(s4, red);
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        double* p = mom + 3 * (size_t)(a0 + i);
        const double m = mass[a0 + i];
        for (int c = 0; c < 3; ++c) p[c] = n_at == 1 ? 0.0 : p[c] - s4[c] / s4[3] * m;
    }
    __syncthreads();
    rescale(mom, a0, n_at, e0, kinetic(mom, mass, a0, n_at, red));

    // ---- ZeroRotation: omega = sum over principal axes with I_k > 1e-10 max(I) of (L . e_k / I_k) e_k; v -= omega x (r - com)
    e0 = kinetic(mom, mass, a0, n_at, red);
    const double mtot = s4[3];
    double c3[3] = {0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double* r = pos + 3 * (size_t)(a0 + i);
        const double m = mass[a0 + i];
        c3[0] += m * r[0]; c3[1] += m * r[1]; c3[2] += m * r[2];
    }
    block_sum<3>(c3, red);
    const double cx = c3[0] / mtot, cy = c3[1] / mtot, cz = c3[2] / mtot;
    double li[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // L (3), then I_xx I_yy I_zz I_xy I_xz I_yz
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double* r = pos + 3 * (size_t)(a0 + i);
        const double* p = mom + 3 * (size_t)(a0 + i);
        const double m = mass[a0 + i];
        const double x = r[0] - cx, y = r[1] - cy, z = r[2] - cz;
        li[0] += y * p[2] - z * p[1]; li[1] += z * p[0] - x * p[2]; li[2] += x * p[1] - y * p[0];
        li[3] += m * (y * y + z * z); li[4] += m * (x * x + z * z); li[5] += m * (x * x + y * y);
        li[6] -= m * x * y; li[7] -= m * x * z; li[8] -= m * y * z;
    }
    block_sum<9>(li, red);
    if (threadIdx.x == 0) {
        double a[3][3] = {{li[3], li[6], li[7]}, {li[6], li[4], li[8]}, {li[7], li[8], li[5]}}, w[3], v[3][3];
        jacobi3(a, w, v);
        const double imax = fmax(fmax(w[0], w[1]), w[2]);
        double om[3] = {0.0, 0.0, 0.0};
        for (int k = 0; k < 3; ++k) {
            if (!(w[k] > 1e-10 * imax)) continue;  // zero moment (linear molecule, one atom): no rotation about this axis
            const double lp = (v[0][k] * li[0] + v[1][k] * li[1] + v[2][k] * li[2]) / w[k];
            for (int c = 0; c < 3; ++c) om[c] += lp * v[c][k];
        }
        omega_sh[0] = om[0]; omega_sh[1] = om[1]; omega_sh[2] = om[2];
    }
    __syncthreads();
    const double ox = omega_sh[0], oy = omega_sh[1], oz = omega_sh[2];
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double* r = pos + 3 * (size_t)(a0 + i);
        double* p = mom + 3 * (size_t)(a0 + i);
        const double m = mass[a0 + i];
        const double x = r[0] - cx, y = r[1] - cy, z = r[2] - cz;
        p[0] = (p[0] / m - (oy * z - oz * y)) * m;
        p[1] = (p[1] / m - (oz * x - ox * z)) * m;
        p[2] = (p[2] / m - (ox * y - oy * x)) * m;
    }
    __syncthreads();
    rescale(mom, a0, n_at, e0, kinetic(mom, mass, a0, n_at, red));
}

struct LangevinCoef {
    double c1, c2;  // dt/2 - dt^2 g/8, dt g/2 - dt^2 g^2/8
    double a3, a5;  // c3 = sigma a3, c5 = sigma a5 with sigma = sqrt(2 kT g / m)
    double two_kt_g, half_g;
};

// the fixcm-corrected random displacement and velocity kick of one atom (ASE 3.22 Langevin.step), given the molecule's sums
__device__ __forceinline__ void langevin_noise(const LangevinCoef& L, uint64_t seed, uint32_t step, int at, double m, double rp[3], double rv[3]) {
    const double2 n0 = normal2(seed, (uint32_t)at, step, 1u, 0u), n1 = normal2(seed, (uint32_t)at, step, 1u, 1u),
                  n2 = normal2(seed, (uint32_t)at, step, 1u, 2u);
    const double xi[3] = {n0.x, n0.y, n1.x}, eta[3] = {n1.y, n2.x, n2.y};
    const double sigma = sqrt(L.two_kt_g / m);
    const double c3 = sigma * L.a3, c5 = sigma * L.a5, c4 = L.half_g * c5;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        rp[c] = c5 * eta[c];
        rv[c] = c3 * xi[c] - c4 * eta[c];
    }
}

// per-molecule fixcm sums: (sum rnd_pos, sum m rnd_vel)
__device__ __forceinline__ void langevin_sums(const LangevinCoef& L, uint64_t seed, uint32_t step, const double* __restrict__ mass, int a0, int n_at,
                              double* red, double out[6]) {
    double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
        const double m = mass[a0 + i];
        double rp[3], rv[3];
        langevin_noise(L, seed, step, a0 + i, m, rp, rv);
        for (int c = 0; c < 3; ++c) { s[c] += rp[c]; s[3 + c] += m * rv[c]; }
    }
    block_sum<6>(s, red);
    for (int c = 0; c < 6; ++c) out[c] = s[c];
}

// __maxnreg__ instead of __launch_bounds__(MD_THREADS): with the latter ptxas settles on 80 registers and spills 32 bytes around
// the float64 division subroutine calls; 128 leaves it at 94 registers without spills (always launched with MD_THREADS)
__global__ void __maxnreg__(128) k_md_step(const int32_t* __restrict__ mol_ptr, const double* __restrict__ mass, int phase, int langevin,
                                                       double dt, LangevinCoef L, uint64_t seed, int64_t step, double f_scale, double e_scale,
                                                       double* __restrict__ pos, double* __restrict__ mom, float* __restrict__ pos32,
                                                       const float* __restrict__ forces, const float* __restrict__ energy,
                                                       double* __restrict__ log_slot, double* __restrict__ frame_pos, double* __restrict__ frame_mom,
                                                       const int32_t* __restrict__ status, int32_t* __restrict__ worst) {
    __shared__ double red[MD_WARPS * 6];
    const int mol = blockIdx.x;
    const int a0 = mol_ptr[mol], n_at = mol_ptr[mol + 1] - a0;
    // A failed engine launch (now or earlier in the chunk) has NaN outputs: leave the state untouched, so that the remaining launches of
    // the chunk still see finite positions.  The host then replays the chunk (capacity) or raises.  Every thread reaches the same verdict:
    // worst[1] can only change below when status[1] != 0.
    const bool failed = status && (status[1] != 0 || worst[1] != 0);
    if (status && mol == 0 && threadIdx.x == 0) {
        // fold the status word of the engine launch this FINISH consumes into the running worst: largest edge count, most severe error,
        // largest degree, and whether any launch ran out of edge capacity (later launches of a poisoned chunk may report other errors)
        worst[0] = max(worst[0], status[0]);
        worst[1] = min(worst[1], status[1]);
        worst[2] = max(worst[2], status[2]);
        if (status[1] == NB200_ECAPACITY) worst[3] = 1;
    }
    if (failed) return;
    const double hdt = 0.5 * dt;

    if (phase & MD_FINISH) {
        const uint32_t s = (uint32_t)step;
        if (langevin) {
            double sums[6];
            langevin_sums(L, seed, s, mass, a0, n_at, red, sums);
            for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
                const int at = a0 + i;
                const double m = mass[at];
                double rp[3], rv[3];
                langevin_noise(L, seed, s, at, m, rp, rv);
                double* p = mom + 3 * (size_t)at;
                const float* f = forces + 3 * (size_t)at;
                for (int c = 0; c < 3; ++c) {
                    const double rvc = rv[c] - sums[3 + c] / (m * n_at);
                    double v = p[c] / m;
                    v += L.c1 * ((double)f[c] * f_scale) / m - L.c2 * v + rvc;
                    p[c] = v * m;
                }
            }
        } else {
            for (int k = threadIdx.x; k < 3 * n_at; k += MD_THREADS) {
                const size_t j = 3 * (size_t)a0 + k;
                mom[j] += hdt * ((double)forces[j] * f_scale);
            }
        }
        __syncthreads();
    }

    if (log_slot) {
        const double ek = kinetic(mom, mass, a0, n_at, red);
        if (threadIdx.x == 0) {
            log_slot[2 * mol] = (double)energy[mol] * e_scale;
            log_slot[2 * mol + 1] = ek;
        }
        for (int k = threadIdx.x; k < 3 * n_at; k += MD_THREADS) {
            const size_t j = 3 * (size_t)a0 + k;
            if (frame_pos) frame_pos[j] = pos[j];
            if (frame_mom) frame_mom[j] = mom[j];
        }
        // the frame is copied coordinate by coordinate, START below writes atom by atom: another thread's START must not overwrite a
        // coordinate before it has been copied
        __syncthreads();
    }

    if (phase & MD_START) {
        const uint32_t s = (uint32_t)(step + 1);
        if (langevin) {
            double sums[6];
            langevin_sums(L, seed, s, mass, a0, n_at, red, sums);
            for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
                const int at = a0 + i;
                const double m = mass[at];
                double rp[3], rv[3];
                langevin_noise(L, seed, s, at, m, rp, rv);
                double* p = mom + 3 * (size_t)at;
                double* x = pos + 3 * (size_t)at;
                const float* f = forces + 3 * (size_t)at;
                for (int c = 0; c < 3; ++c) {
                    const double rpc = rp[c] - sums[c] / n_at;
                    const double rvc = rv[c] - sums[3 + c] / (m * n_at);
                    double v = p[c] / m;
                    v += L.c1 * ((double)f[c] * f_scale) / m - L.c2 * v + rvc;
                    const double x0 = x[c];
                    const double xn = x0 + dt * v + rpc;
                    v = (xn - x0 - rpc) / dt;
                    x[c] = xn;
                    p[c] = v * m;
                    pos32[3 * (size_t)at + c] = (float)xn;
                }
            }
        } else {
            for (int i = threadIdx.x; i < n_at; i += MD_THREADS) {
                const int at = a0 + i;
                const double m = mass[at];
                for (int c = 0; c < 3; ++c) {
                    const size_t j = 3 * (size_t)at + c;
                    const double p = mom[j] + hdt * ((double)forces[j] * f_scale);
                    mom[j] = p;
                    const double xn = pos[j] + dt * p / m;
                    pos[j] = xn;
                    pos32[j] = (float)xn;
                }
            }
        }
    }
}

}  // namespace

extern "C" int nb200_md_init_momenta(const int32_t* mol_ptr, int32_t n_mol, const double* mass, const double* pos, double kT, uint64_t seed,
                                     int64_t noise_step, double* mom, void* stream) {
    if (!mol_ptr || !mass || !pos || !mom || n_mol < 0 || !(kT >= 0.0) || noise_step < 0 || noise_step > 0xffffffffLL) return NB200_EINVAL;
    if (n_mol == 0) return NB200_OK;
    k_md_init_momenta<<<n_mol, MD_THREADS, 0, (cudaStream_t)stream>>>(mol_ptr, mass, pos, kT, seed, (uint32_t)noise_step, mom);
    return nb_check_launch();
}

extern "C" int nb200_md_step(const int32_t* mol_ptr, int32_t n_mol, const double* mass, int32_t phase, int32_t thermostat, double dt, double kT,
                             double gamma, uint64_t seed, int64_t step, double f_scale, double e_scale, double* pos, double* mom, float* pos32,
                             const float* forces, const float* energy, double* log_slot, double* frame_pos, double* frame_mom,
                             const int32_t* status, int32_t* worst, void* stream) {
    if (!mol_ptr || !mass || !pos || !mom || !pos32 || !forces || n_mol < 0 || phase < 0 || phase > (MD_FINISH | MD_START) || thermostat < 0 ||
        thermostat > 1 || !(dt > 0.0) || !(kT >= 0.0) || !(gamma >= 0.0) || (log_slot && !energy) || (status && !worst) || step < -1 ||
        step > 0xfffffffeLL)
        return NB200_EINVAL;
    if (n_mol == 0) return NB200_OK;
    LangevinCoef L{};
    if (thermostat == 1) {  // ASE 3.22 Langevin.updatevars
        L.c1 = dt / 2.0 - dt * dt * gamma / 8.0;
        L.c2 = dt * gamma / 2.0 - dt * dt * gamma * gamma / 8.0;
        L.a3 = sqrt(dt) / 2.0 - pow(dt, 1.5) * gamma / 8.0;
        L.a5 = pow(dt, 1.5) / (2.0 * sqrt(3.0));
        L.two_kt_g = 2.0 * kT * gamma;
        L.half_g = gamma / 2.0;
    }
    k_md_step<<<n_mol, MD_THREADS, 0, (cudaStream_t)stream>>>(mol_ptr, mass, phase, thermostat, dt, L, seed, step, f_scale, e_scale, pos, mom, pos32,
                                                              forces, energy, log_slot, frame_pos, frame_mom, status, worst);
    return nb_check_launch();
}
