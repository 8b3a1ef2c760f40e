// quasinewton.cu -- ASE's QuasiNewton (BFGSLineSearch + LineSearch, the optimiser of PYGAseInterface.optimize) for a batch of
// independent molecules, one launch per energy + forces evaluation.
//
// Each molecule is a small state machine that always waits for exactly one evaluation at its current trial point.  A launch
// consumes E and F there, runs every transition that needs no new evaluation (line-search step, acceptance, fmax test, BFGS update,
// new direction, START of the next line search) and stops either at a new trial point, written to `pos` (float64) and `pos32`, or
// because the molecule has stopped (converged, `max_steps` reached, line search failed).  A stopped molecule is a no-op in every
// later launch, so launches after the whole batch has stopped move nothing.  One CTA per molecule; the scalar line search runs
// redundantly in every thread (identical registers, uniform control flow), the vector work is spread over the CTA.
//
// State (caller-owned, zero-filled before the first launch): per molecule a QnMol record (line-search scalars, phase, counters that
// need no host look), the dense inverse Hessian H [3n x 3n] float64 at the caller's int64 offsets, and r (start of the current step),
// p (direction) float64 and g (= -F / alpha at r) float32, each [3N].  `mol_info` [n_mol][4] = status, nsteps, force_calls,
// function_calls is the part the host reads.
//
// Arithmetic follows numpy as oracle/quasinewton.py lists it: F, g, dg in float32; positions, H, p, energies, dot products and the
// line-search scalars in float64.  This file is compiled with -fmad=false so that every float64 expression of the line search and of
// the H update rounds after each operation, as Python does.  Reductions (dot products, |p|) are tree-ordered in float64 (numpy:
// pairwise / BLAS order), which moves them by ~1e-16 relative; maxima are exact.
//
// BFGS update: the O(n^2) rank-2 form  H' = H - rho (dr u^T + u dr^T) + (rho^2 dg.u + rho) dr dr^T,  u = H dg,  instead of ASE's
// O(n^3) A1 H A2 product (equal for symmetric H up to rounding; H stays exactly symmetric).  Traffic per launch that starts a step:
// H is read once for u (only when the update is taken) and once more while it is rewritten and p = -H' g is accumulated row by row,
// 2 reads + 1 write of 8 (3n)^2 bytes per molecule; a launch inside a line search touches O(n) bytes.
#include <cmath>

#include "common.cuh"

namespace {

constexpr int QN_THREADS = 256;
constexpr int QN_WARPS = QN_THREADS / 32;

enum : int32_t { QN_RUNNING = 0, QN_CONVERGED = 1, QN_MAX_STEPS = 2, QN_FAILED = 3, QN_BAD_LAYOUT = 4 };
enum : int32_t { T_START = 0, T_FG = 1, T_CONV = 2, T_WARN_ROUND = 3, T_WARN_XTOL = 4, T_WARN_STPMAX = 5, T_WARN_STPMIN = 6, T_ERROR = 7 };

struct QnMol {
    double stx, fx, gx, sty, fy, gy, stmin, stmax, width, width1, finit, ginit, gtest;  // LineSearch dsave
    double stp;      // step being evaluated; also old_stp of the next LineSearch.step call
    double alpha_k;  // step accepted by the previous line search (0 before the first)
    double e0;       // E / alpha at the start of the current step
    int32_t phase;   // 0: the first evaluation is pending; 1: a line search is running
    int32_t stage, bracket, task, no_update, has_h;
    int32_t pad[2];
};
static_assert(sizeof(QnMol) % 16 == 0, "QnMol keeps 16-byte alignment");

struct LsConst {
    double c1, c2, stpmin, stpmax, xtrapl, xtrapu, xtol, maxstep;
};

struct QnArgs {
    const int32_t* mol_ptr;
    const int64_t* hess_off;
    int64_t hess_elems;
    int max_nc, max_steps;
    float fmax2, alpha32;
    double alpha, e_scale, f_scale;
    LsConst ls;
    const uint8_t* fixed;
    const float* energy;
    const float* forces;
    double* pos;
    float* pos32;
    QnMol* mols;
    double* hess;
    double* r;
    double* p;
    float* g;
    int32_t* info;
    int32_t* running;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double block_sum(double v, double* red) {
    v = warp_sum(v);
    __syncthreads();  // protects `red` against the previous reduction's readers
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < QN_WARPS; ++w) t += red[w];
    return t;
}
__device__ __forceinline__ double block_max(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = red[0];
#pragma unroll
    for (int w = 1; w < QN_WARPS; ++w) t = fmax(t, red[w]);
    return t;
}
// Python's min / max of two numbers: the first argument unless the second is strictly smaller / larger
__device__ __forceinline__ double pmin(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double pmax(double a, double b) { return b > a ? b : a; }
__device__ __forceinline__ double pmax3(double a, double b, double c) { return pmax(pmax(a, b), c); }

// LineSearch.determine_step (line_search.py:490-498): cap the largest per-atom displacement of (stp - old_stp) p at maxstep.  Collective.
__device__ double determine_step(double stp, double old_stp, const double* p, int n_at, double maxstep, double* red) {
    double dr = stp - old_stp;
    double longest = 0.0;
    for (int at = threadIdx.x; at < n_at; at += QN_THREADS) {
        const double x = dr * p[3 * at], y = dr * p[3 * at + 1], z = dr * p[3 * at + 2];
        longest = fmax(longest, sqrt((x * x + y * y) + z * z));
    }
    longest = block_max(longest, red);
    if (longest >= maxstep) dr *= maxstep / longest;
    return old_stp + dr;
}

// LineSearch.step, task START (line_search.py:127-187).  Collective.
__device__ double ls_start(QnMol& s, double stp, double f, double g, const LsConst& c, const double* p, int n_at, double* red) {
    if (stp < c.stpmin || stp > c.stpmax || g >= 0 || c.c1 < 0 || c.c2 < 0 || c.xtol < 0 || c.stpmin < 0 || c.stpmax < c.stpmin) {
        s.task = T_ERROR;
        return stp;
    }
    s.bracket = 0;
    s.stage = 1;
    s.finit = f; s.ginit = g;
    s.gtest = c.c1 * g;
    s.width = c.stpmax - c.stpmin;
    s.width1 = s.width / 0.5;
    s.stx = 0.0; s.fx = f; s.gx = g;
    s.sty = 0.0; s.fy = f; s.gy = g;
    s.stmin = 0.0;
    s.stmax = stp + c.xtrapu * stp;
    s.task = T_FG;
    return determine_step(stp, 0.0, p, n_at, c.maxstep, red);
}

// LineSearch.step after START (line_search.py:188-341) with LineSearch.update (dcstep, :343-488) inlined.  `stp` is the evaluated step
// (also old_stp).  Collective.
__device__ double ls_continue(QnMol& s, double stp, double f, double g, const LsConst& c, const double* p, int n_at, double* red) {
    const double ftest = s.finit + stp * s.gtest;
    if (s.stage == 1 && f < ftest && g >= 0.0) s.stage = 2;
    int task = T_FG;
    if (s.bracket && (stp <= s.stmin || stp >= s.stmax)) task = T_WARN_ROUND;
    if (s.bracket && s.stmax - s.stmin <= c.xtol * s.stmax) task = T_WARN_XTOL;
    if (stp == c.stpmax && f <= ftest && g <= s.gtest) task = T_WARN_STPMAX;
    if (stp == c.stpmin && (f > ftest || g >= s.gtest)) task = T_WARN_STPMIN;
    if (f <= ftest && fabs(g) <= c.c2 * (-s.ginit)) task = T_CONV;
    s.task = task;
    if (task != T_FG) return stp;

    // ---- update (dcstep); lo / hi are its stpmin / stpmax arguments, the current interval
    double stx = s.stx, fx = s.fx, gx = s.gx, sty = s.sty, fy = s.fy, gy = s.gy;
    const double fp = f, gp = g, lo = s.stmin, hi = s.stmax;
    const double sign = gp * (gx / fabs(gx));
    double stpf;
    if (fp > fx) {  // case 1: higher function value, the minimum is bracketed
        const double theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp;
        const double sc = pmax3(fabs(theta), fabs(gx), fabs(gp));
        const double ts = theta / sc;
        double gamma = sc * sqrt(ts * ts - (gx / sc) * (gp / sc));
        if (stp < stx) gamma = -gamma;
        const double pp = (gamma - gx) + theta;
        const double q = ((gamma - gx) + gamma) + gp;
        const double r = pp / q;
        const double stpc = stx + r * (stp - stx);
        const double stpq = stx + ((gx / ((fx - fp) / (stp - stx) + gx)) / 2.0) * (stp - stx);
        stpf = fabs(stpc - stx) < fabs(stpq - stx) ? stpc : stpc + (stpq - stpc) / 2.0;
        s.bracket = 1;
    } else if (sign < 0) {  // case 2: lower value, derivatives of opposite sign
        const double theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp;
        const double sc = pmax3(fabs(theta), fabs(gx), fabs(gp));
        const double ts = theta / sc;
        double gamma = sc * sqrt(ts * ts - (gx / sc) * (gp / sc));
        if (stp > stx) gamma = -gamma;
        const double pp = (gamma - gp) + theta;
        const double q = ((gamma - gp) + gamma) + gx;
        const double r = pp / q;
        const double stpc = stp + r * (stx - stp);
        const double stpq = stp + (gp / (gp - gx)) * (stx - stp);
        stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
        s.bracket = 1;
    } else if (fabs(gp) < fabs(gx)) {  // case 3: lower value, same sign, |derivative| decreases
        const double theta = 3.0 * (fx - fp) / (stp - stx) + gx + gp;
        const double sc = pmax3(fabs(theta), fabs(gx), fabs(gp));
        const double ts = theta / sc;
        double gamma = sc * sqrt(pmax(0.0, ts * ts - (gx / sc) * (gp / sc)));
        if (stp > stx) gamma = -gamma;
        const double pp = (gamma - gp) + theta;
        const double q = (gamma + (gx - gp)) + gamma;
        const double r = pp / q;
        double stpc;
        if (r < 0.0 && gamma != 0) stpc = stp + r * (stx - stp);
        else if (stp > stx) stpc = hi;
        else stpc = lo;
        const double stpq = stp + (gp / (gp - gx)) * (stx - stp);
        if (s.bracket) {
            stpf = fabs(stpc - stp) < fabs(stpq - stp) ? stpc : stpq;
            stpf = stp > stx ? pmin(stp + 0.66 * (sty - stp), stpf) : pmax(stp + 0.66 * (sty - stp), stpf);
        } else {
            stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
            stpf = pmin(hi, stpf);
            stpf = pmax(lo, stpf);
        }
    } else {  // case 4: lower value, same sign, |derivative| does not decrease
        if (s.bracket) {
            const double theta = 3.0 * (fp - fy) / (sty - stp) + gy + gp;
            const double sc = pmax3(fabs(theta), fabs(gy), fabs(gp));
            const double ts = theta / sc;
            double gamma = sc * sqrt(ts * ts - (gy / sc) * (gp / sc));
            if (stp > sty) gamma = -gamma;
            const double pp = (gamma - gp) + theta;
            const double q = ((gamma - gp) + gamma) + gy;
            const double r = pp / q;
            stpf = stp + r * (sty - stp);
        } else {
            stpf = stp > stx ? hi : lo;
        }
    }
    if (fp > fx) {
        sty = stp; fy = fp; gy = gp;
    } else {
        if (sign < 0) { sty = stx; fy = fx; gy = gx; }
        stx = stp; fx = fp; gx = gp;
    }
    double nstp = determine_step(stpf, stp, p, n_at, c.maxstep, red);

    // ---- back in step: bisection, interval, bounds
    if (s.bracket) {
        if (fabs(sty - stx) >= 0.66 * s.width1) nstp = stx + 0.5 * (sty - stx);
        s.width1 = s.width;
        s.width = fabs(sty - stx);
    }
    if (s.bracket) {
        s.stmin = pmin(stx, sty);
        s.stmax = pmax(stx, sty);
    } else {
        s.stmin = nstp + c.xtrapl * (nstp - stx);
        s.stmax = nstp + c.xtrapu * (nstp - stx);
    }
    nstp = pmax(nstp, c.stpmin);
    nstp = pmin(nstp, c.stpmax);
    if (stx == nstp && nstp == c.stpmax && s.stmin > c.stpmax) s.no_update = 1;
    if ((s.bracket && nstp < s.stmin || nstp >= s.stmax) || (s.bracket && s.stmax - s.stmin < c.xtol * s.stmax)) nstp = stx;
    s.stx = stx; s.fx = fx; s.gx = gx; s.sty = sty; s.fy = fy; s.gy = gy;
    return nstp;
}

// |f|^2 of one atom as numpy evaluates (f**2).sum(-1) in float32
__device__ __forceinline__ float sq3(float x, float y, float z) { return (x * x + y * y) + z * z; }

__global__ void __launch_bounds__(QN_THREADS) k_qn_step(QnArgs a) {
    extern __shared__ __align__(16) unsigned char qn_smem[];
    const int m = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int32_t* info = a.info + 4 * (size_t)m;
    if (info[0] != QN_RUNNING) return;  // stopped molecules are a no-op
    const int a0 = a.mol_ptr[m], n_at = a.mol_ptr[m + 1] - a0, nc = 3 * n_at;
    const size_t base = 3 * (size_t)a0;
    if (n_at < 0 || nc > a.max_nc) {  // shared memory is sized by max_atoms_per_mol: refuse a larger molecule instead of overrunning it
        if (tid == 0) info[0] = QN_BAD_LAYOUT;
        return;
    }
    double* red = reinterpret_cast<double*>(qn_smem);  // [QN_WARPS]
    double* p_sm = red + QN_WARPS;                     // [max_nc] direction
    double* s_sm = p_sm + a.max_nc;                    // [max_nc] dr = r - r0
    double* y_sm = s_sm + a.max_nc;                    // [max_nc] dg = g - g0 (float32 values)
    double* u_sm = y_sm + a.max_nc;                    // [max_nc] u = H dg
    float* g_sm = reinterpret_cast<float*>(u_sm + a.max_nc);  // [max_nc] g = -F / alpha at the evaluated point

    QnMol s = a.mols[m];
    int32_t status = QN_RUNNING, nsteps = info[1], force_calls = info[2], function_calls = info[3];
    double* r_st = a.r + base;
    double* p_st = a.p + base;
    float* g_st = a.g + base;

    // ---- consume F: FixAtoms zeroes fixed atoms, g = -F / alpha (float32), fmax test, derphi = g.p inside a line search
    const bool in_ls = s.phase == 1;
    float fm = 0.f;
    double dphi = 0.0;
    for (int at = tid; at < n_at; at += QN_THREADS) {
        const bool fixed = a.fixed && a.fixed[a0 + at];
        float fv[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int k = 3 * at + c;
            float f = fixed ? 0.f : a.forces[base + k];
            if (a.f_scale != 1.0) f = f * (float)a.f_scale;
            fv[c] = f;
            const float g = -f / a.alpha32;
            g_sm[k] = g;
            if (in_ls) {
                const double pk = p_st[k];
                p_sm[k] = pk;
                dphi += (double)g * pk;
            }
        }
        fm = fmaxf(fm, sq3(fv[0], fv[1], fv[2]));
    }
    const bool conv = (float)block_max((double)fm, red) < a.fmax2;
    if (in_ls) dphi = block_sum(dphi, red);
    const double phi = (double)a.energy[m] * a.e_scale / a.alpha;

    bool start = false, trial = false;
    if (!in_ls) {  // Optimizer.irun: forces at the start, then the loop test
        if (conv) status = QN_CONVERGED;
        else if (nsteps >= a.max_steps) status = QN_MAX_STEPS;
        else start = true;
    } else {
        ++force_calls;
        ++function_calls;
        bool accept = true;
        if (!s.no_update) {  // _line_search stops right after the evaluation that follows no_update
            const double stp = ls_continue(s, s.stp, phi, dphi, a.ls, p_sm, n_at, red);
            if (s.task == T_FG) {
                s.stp = stp;
                accept = false;
                trial = true;
            }  // CONVERGENCE and WARNING* accept the last evaluated point (ASE never matches task[1:4] == 'WARN')
        }
        if (accept) {
            s.alpha_k = s.stp;
            ++nsteps;
            if (conv) status = QN_CONVERGED;
            else if (nsteps >= a.max_steps) status = QN_MAX_STEPS;
            else start = true;
        }
    }

    if (start) {  // BFGSLineSearch.step at the current point
        const int64_t h0 = a.hess_off[m];
        if (h0 < 0 || h0 + (int64_t)nc * nc > a.hess_elems) {
            status = QN_BAD_LAYOUT;
            start = false;
        }
    }
    if (start) {
        ++function_calls;  // e = self.func(r)
        double* H = a.hess + a.hess_off[m];
        const bool first = !s.has_h;
        double gp0 = 0.0, g0p0 = 0.0, sy = 0.0;
        for (int k = tid; k < nc; k += QN_THREADS) {
            const double r = a.pos[base + k];
            const float g = g_sm[k];
            if (!first) {
                const float g0 = g_st[k];
                const double p0 = p_st[k];
                const double dr = r - r_st[k];
                const float dg = g - g0;
                s_sm[k] = dr;
                y_sm[k] = (double)dg;
                gp0 += (double)g * p0;
                g0p0 += (double)g0 * p0;
                sy += (double)dg * dr;
            }
            r_st[k] = r;
            g_st[k] = g;
        }
        bool upd = false;
        double rho = 0.0, cc = 0.0;
        if (!first) {
            gp0 = block_sum(gp0, red);
            g0p0 = block_sum(g0p0, red);
            sy = block_sum(sy, red);
            upd = s.alpha_k > 0 && fabs(gp0) - fabs(g0p0) < 0 && !s.no_update;
            if (upd) {
                rho = 1.0 / sy;
                if (isinf(rho)) rho = 1000.0;
                for (int i = warp; i < nc; i += QN_WARPS) {  // u = H dg
                    const double* row = H + (size_t)i * nc;
                    double acc = 0.0;
                    for (int j = lane; j < nc; j += 32) acc += row[j] * y_sm[j];
                    acc = warp_sum(acc);
                    if (lane == 0) u_sm[i] = acc;
                }
                __syncthreads();
                double yu = 0.0;
                for (int k = tid; k < nc; k += QN_THREADS) yu += y_sm[k] * u_sm[k];
                yu = block_sum(yu, red);
                cc = rho * rho * yu + rho;
            }
        }
        // H = I (first step) or H' (rank-2 update), rewritten once, and p = -H g accumulated from the rows just written
        for (int i = warp; i < nc; i += QN_WARPS) {
            double* row = H + (size_t)i * nc;
            const double si = upd ? s_sm[i] : 0.0, ui = upd ? u_sm[i] : 0.0;
            double acc = 0.0;
            for (int j = lane; j < nc; j += 32) {
                double h;
                if (first) {
                    h = i == j ? 1.0 : 0.0;
                    row[j] = h;
                } else {
                    h = row[j];
                    if (upd) {
                        h = h - rho * (si * u_sm[j] + ui * s_sm[j]) + cc * (si * s_sm[j]);
                        row[j] = h;
                    }
                }
                acc += h * (double)g_sm[j];
            }
            acc = warp_sum(acc);
            if (lane == 0) p_sm[i] = -acc;
        }
        __syncthreads();
        double psq = 0.0;
        for (int k = tid; k < nc; k += QN_THREADS) psq += p_sm[k] * p_sm[k];
        psq = block_sum(psq, red);
        const double p_size = sqrt(psq), p_min = sqrt((double)n_at * 1e-10);
        double gp = 0.0;
        for (int k = tid; k < nc; k += QN_THREADS) {
            double pk = p_sm[k];
            if (p_size <= p_min) pk /= p_size / p_min;
            p_sm[k] = pk;
            p_st[k] = pk;
            gp += (double)g_sm[k] * pk;
        }
        gp = block_sum(gp, red);  // also publishes p_sm to determine_step
        s.has_h = 1;
        s.e0 = phi;
        s.no_update = 0;  // a fresh LineSearch
        const double stp = ls_start(s, 1.0, phi, gp, a.ls, p_sm, n_at, red);
        if (s.task == T_ERROR) {
            status = QN_FAILED;  // BFGSLineSearch raises RuntimeError('LineSearch failed!')
        } else {
            s.stp = stp;
            s.phase = 1;
            trial = true;
        }
    }
    if (trial) {  // the next evaluation: r + stp p
        for (int k = tid; k < nc; k += QN_THREADS) {
            const double x = r_st[k] + s.stp * p_sm[k];
            a.pos[base + k] = x;
            a.pos32[base + k] = (float)x;
        }
    }
    if (tid == 0) {
        a.mols[m] = s;
        info[0] = status;
        info[1] = nsteps;
        info[2] = force_calls;
        info[3] = function_calls;
        if (status == QN_RUNNING) atomicAdd(a.running, 1);
    }
}

size_t qn_align(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

extern "C" int64_t nb200_qn_state_bytes(int32_t n_mol, int32_t n_atoms, int64_t hess_elems) {
    if (n_mol < 0 || n_atoms < 0 || hess_elems < 0) return NB200_EINVAL;
    const size_t nc = 3 * (size_t)n_atoms;
    return (int64_t)(qn_align((size_t)n_mol * sizeof(QnMol)) + qn_align((size_t)hess_elems * 8) + 2 * qn_align(nc * 8) + qn_align(nc * 4));
}

extern "C" int nb200_qn_step(void* state, int64_t state_bytes, const int32_t* mol_ptr, const int64_t* hess_off, int32_t n_mol, int32_t n_atoms,
                             int32_t max_atoms_per_mol, int64_t hess_elems, double fmax, int32_t max_steps, double maxstep, double c1, double c2,
                             double alpha, double stpmax, double e_scale, double f_scale, const uint8_t* fixed_mask, const float* energy,
                             const float* forces, double* pos, float* pos32, int32_t* mol_info, int32_t* running_out, void* stream) {
    if (!state || !mol_ptr || !hess_off || !energy || !forces || !pos || !pos32 || !mol_info || !running_out || n_mol < 0 || n_atoms < 0 ||
        max_atoms_per_mol < 0 || hess_elems < 0 || max_steps < 0 || !(alpha > 0) || !(maxstep > 0))
        return NB200_EINVAL;
    const int64_t need = nb200_qn_state_bytes(n_mol, n_atoms, hess_elems);
    if (need < 0 || state_bytes < need) return NB200_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(running_out, 0, sizeof(int32_t), st) != cudaSuccess) return nb_check_launch();
    if (n_mol == 0) return NB200_OK;
    const size_t nc = 3 * (size_t)n_atoms;
    unsigned char* p = static_cast<unsigned char*>(state);
    QnArgs a;
    a.mols = reinterpret_cast<QnMol*>(p);  p += qn_align((size_t)n_mol * sizeof(QnMol));
    a.hess = reinterpret_cast<double*>(p); p += qn_align((size_t)hess_elems * 8);
    a.r = reinterpret_cast<double*>(p);    p += qn_align(nc * 8);
    a.p = reinterpret_cast<double*>(p);    p += qn_align(nc * 8);
    a.g = reinterpret_cast<float*>(p);
    a.mol_ptr = mol_ptr;
    a.hess_off = hess_off;
    a.hess_elems = hess_elems;
    a.max_nc = 3 * max_atoms_per_mol;
    a.max_steps = max_steps;
    a.fmax2 = (float)(fmax * fmax);
    a.alpha = alpha;
    a.alpha32 = (float)alpha;
    a.e_scale = e_scale;
    a.f_scale = f_scale;
    a.ls = LsConst{c1, c2, 1e-8, stpmax, 1.1, 4.0, 1e-14, maxstep};
    a.fixed = fixed_mask;
    a.energy = energy;
    a.forces = forces;
    a.pos = pos;
    a.pos32 = pos32;
    a.info = mol_info;
    a.running = running_out;
    const size_t smem = (QN_WARPS + 4 * (size_t)a.max_nc) * sizeof(double) + (size_t)a.max_nc * sizeof(float);
    if (smem > 200 * 1024) return NB200_EUNSUPPORTED;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k_qn_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return nb_check_launch();
    k_qn_step<<<n_mol, QN_THREADS, smem, st>>>(a);
    return nb_check_launch();
}
