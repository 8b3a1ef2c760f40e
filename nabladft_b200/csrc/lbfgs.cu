// lbfgs.cu -- one step of the reference's batch-wise L-BFGS geometry optimiser, entirely on the device.
//
// Replaces ASEBatchwiseLBFGS.step / update / determine_step (nablaDFT/optimization/optimizers.py:436-598): there every step
// copies forces to the host, runs the two-loop recursion in numpy over Python lists of per-step arrays, rebuilds a list of
// ase.Atoms and a neighbour list on the CPU and uploads the batch again.  Here the optimiser state (positions, the s / y / rho
// history ring, r0, f0) lives in HBM next to the model's buffers and a step is ONE kernel, one CTA per molecule (molecules are
// independent: every reduction of the algorithm is per molecule), launched back to back with the energy+forces engine on the
// same stream -- no host synchronisation inside the relaxation loop.
//
// Arithmetic mirrors the reference's mixed precision (see oracle/lbfgs.py): positions, s, a, b, rho in float64; forces, y, q, z,
// p, dr in float32, with float64 intermediates rounded exactly where numpy rounds them.  Reductions are tree-ordered in float64
// (numpy: sequential), which moves results by ~1e-16 relative.
//
// Traffic per step: the history is read twice (two loops): 2 * min(memory, it) * 3N * (8 + 4) bytes (72 MB at N = 10^4,
// memory = 100); the kernel is latency-bound on its 2 * min(memory, it) + 3 block reductions instead.
#include "common.cuh"

namespace {

constexpr int LB_THREADS = 128;

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();  // protects `red` against the previous reduction's readers
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < LB_THREADS / 32; ++w) t += red[w];
    return t;
}
__device__ __forceinline__ float block_max(float v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = (double)v;
    __syncthreads();
    float t = (float)red[0];
#pragma unroll
    for (int w = 1; w < LB_THREADS / 32; ++w) t = fmaxf(t, (float)red[w]);
    return t;
}
// |v|^2 the way numpy evaluates (f**2).sum(-1) in float32: three rounded squares, two rounded adds, no FMA contraction
__device__ __forceinline__ float sq3(float x, float y, float z) { return __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)); }

__global__ void __launch_bounds__(LB_THREADS) k_lbfgs_step(const int32_t* __restrict__ mol_ptr, int memory, int iteration, float fmax2_lo, double fmax2,
                                                          double maxstep, float damping, float h0, const uint8_t* __restrict__ fixed,
                                                          double* __restrict__ pos, float* __restrict__ forces, float* __restrict__ pos32,
                                                          double* __restrict__ s_hist, float* __restrict__ y_hist, double* __restrict__ rho_hist,
                                                          double* __restrict__ r0, float* __restrict__ f0, size_t n_coord, int n_mol,
                                                          int32_t* __restrict__ unconverged, int32_t* __restrict__ n_norm) {
    extern __shared__ __align__(16) unsigned char lb_smem[];
    const int m = blockIdx.x, tid = threadIdx.x;
    const int a0 = mol_ptr[m], a1 = mol_ptr[m + 1];
    const int n_at = a1 - a0, nc = 3 * n_at;
    const size_t base = 3 * (size_t)a0;
    double* red = reinterpret_cast<double*>(lb_smem);            // [4]
    double* a_sm = red + LB_THREADS / 32;                        // [memory]
    float* q = reinterpret_cast<float*>(a_sm + memory);          // [nc]  q, then z, then p
    (void)fmax2_lo;

    // ---- forces (fixed atoms -> 0, written back like calculator.py:86-88), q = -f, frozen flag (optimizers.py:446-456)
    float fm = 0.f;
    for (int at = tid; at < n_at; at += LB_THREADS) {
        float* fp = forces + base + 3 * at;
        float fx = fp[0], fy = fp[1], fz = fp[2];
        if (fixed && fixed[a0 + at]) { fx = fy = fz = 0.f; fp[0] = fp[1] = fp[2] = 0.f; }
        q[3 * at] = -fx; q[3 * at + 1] = -fy; q[3 * at + 2] = -fz;
        fm = fmaxf(fm, sq3(fx, fy, fz));
    }
    fm = block_max(fm, red);
    const bool frozen = (double)fm < fmax2;
    if (tid == 0 && !frozen) atomicAdd(unconverged, 1);

    // ---- update (optimizers.py:573-598): pair `iteration` goes to ring slot (iteration - 1) % memory
    if (iteration > 0) {
        const int slot = (iteration - 1) % memory;
        double* s_new = s_hist + (size_t)slot * n_coord + base;
        float* y_new = y_hist + (size_t)slot * n_coord + base;
        double ys = 0.0;
        for (int k = tid; k < nc; k += LB_THREADS) {
            const double s0 = pos[base + k] - r0[base + k];
            const float y0 = __fsub_rn(f0[base + k], -q[k]);  // f0 - f in float32
            s_new[k] = s0; y_new[k] = y0;
            ys += (double)y0 * s0;
        }
        ys = block_sum(ys, red);
        if (tid == 0) rho_hist[(size_t)slot * n_mol + m] = ys > 1e-8 ? 1.0 / ys : 1.0;
        __syncthreads();
    }
    const int loopmax = min(memory, iteration);

    // ---- two-loop recursion (optimizers.py:478-503)
    for (int i = loopmax - 1; i >= 0; --i) {
        const int slot = (iteration - loopmax + i) % memory;
        const double* s_i = s_hist + (size_t)slot * n_coord + base;
        const float* y_i = y_hist + (size_t)slot * n_coord + base;
        double acc = 0.0;
        for (int k = tid; k < nc; k += LB_THREADS) acc += s_i[k] * (double)q[k];
        const double ai = rho_hist[(size_t)slot * n_mol + m] * block_sum(acc, red);
        if (tid == 0) a_sm[i] = ai;
        for (int k = tid; k < nc; k += LB_THREADS) q[k] = (float)((double)q[k] - ai * (double)y_i[k]);
    }
    __syncthreads();
    for (int k = tid; k < nc; k += LB_THREADS) q[k] = __fmul_rn(h0, q[k]);  // z = H0 * q
    for (int i = 0; i < loopmax; ++i) {
        const int slot = (iteration - loopmax + i) % memory;
        const double* s_i = s_hist + (size_t)slot * n_coord + base;
        const float* y_i = y_hist + (size_t)slot * n_coord + base;
        double acc = 0.0;
        for (int k = tid; k < nc; k += LB_THREADS) acc += (double)__fmul_rn(y_i[k], q[k]);  // float32 products (numpy), float64 sum
        const double b = rho_hist[(size_t)slot * n_mol + m] * (double)(float)block_sum(acc, red);
        const double coef = a_sm[i] - b;
        for (int k = tid; k < nc; k += LB_THREADS) q[k] = (float)((double)q[k] + s_i[k] * coef);
    }
    __syncthreads();

    // ---- p = -z (0 for converged molecules), determine_step (optimizers.py:550-571), move, remember r0 / f0
    float longest = 0.f;
    for (int at = tid; at < n_at; at += LB_THREADS) {
        const float px = frozen ? 0.f : -q[3 * at], py = frozen ? 0.f : -q[3 * at + 1], pz = frozen ? 0.f : -q[3 * at + 2];
        q[3 * at] = px; q[3 * at + 1] = py; q[3 * at + 2] = pz;
        longest = fmaxf(longest, __fsqrt_rn(sq3(px, py, pz)));
    }
    longest = block_max(longest, red);
    float scale = 1.f;
    if ((double)longest >= maxstep) {
        scale = __fdiv_rn((float)maxstep, longest);
        if (tid == 0) atomicAdd(n_norm, 1);
    }
    for (int k = tid; k < nc; k += LB_THREADS) {
        float dr = q[k];
        if (scale != 1.f) dr = __fmul_rn(dr, scale);
        dr = __fmul_rn(dr, damping);
        const double r = pos[base + k];
        const double rn = r + (double)dr;
        r0[base + k] = r;
        f0[base + k] = forces[base + k];
        pos[base + k] = rn;
        pos32[base + k] = (float)rn;
    }
}

}  // namespace

static size_t lb_align(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" int64_t nb200_lbfgs_state_bytes(int32_t n_mol, int32_t n_atoms, int32_t memory) {
    if (n_mol < 0 || n_atoms < 0 || memory <= 0) return NB200_EINVAL;
    const size_t nc = 3 * (size_t)n_atoms;
    return (int64_t)(lb_align((size_t)memory * nc * 8) + lb_align((size_t)memory * nc * 4) + lb_align((size_t)memory * n_mol * 8) + lb_align(nc * 8) +
                     lb_align(nc * 4));
}

extern "C" int nb200_lbfgs_step(void* state, int64_t state_bytes, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol,
                                int32_t memory, int32_t iteration, double fmax, double maxstep, double damping, double h0,
                                const uint8_t* fixed_mask, double* pos, float* forces, float* pos32_out, int32_t* unconverged_out,
                                int32_t* n_normalizations, void* stream) {
    if (!state || !mol_ptr || !pos || !forces || !pos32_out || !unconverged_out || !n_normalizations || n_mol < 0 || n_atoms < 0 || memory <= 0 ||
        iteration < 0 || max_atoms_per_mol < 0)
        return NB200_EINVAL;
    if (state_bytes < nb200_lbfgs_state_bytes(n_mol, n_atoms, memory)) return NB200_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(unconverged_out, 0, sizeof(int32_t), s) != cudaSuccess) return nb_check_launch();
    if (n_mol == 0) return NB200_OK;
    const size_t nc = 3 * (size_t)n_atoms;
    unsigned char* p = static_cast<unsigned char*>(state);
    double* s_hist = reinterpret_cast<double*>(p); p += lb_align((size_t)memory * nc * 8);
    float* y_hist = reinterpret_cast<float*>(p);   p += lb_align((size_t)memory * nc * 4);
    double* rho = reinterpret_cast<double*>(p);    p += lb_align((size_t)memory * n_mol * 8);
    double* r0 = reinterpret_cast<double*>(p);     p += lb_align(nc * 8);
    float* f0 = reinterpret_cast<float*>(p);
    const size_t smem = (LB_THREADS / 32 + (size_t)memory) * sizeof(double) + 3 * (size_t)max_atoms_per_mol * sizeof(float);
    if (smem > 200 * 1024) return NB200_EUNSUPPORTED;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k_lbfgs_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return nb_check_launch();
    k_lbfgs_step<<<n_mol, LB_THREADS, smem, s>>>(mol_ptr, memory, iteration, 0.f, fmax * fmax, maxstep, (float)damping, (float)h0, fixed_mask, pos, forces,
                                                pos32_out, s_hist, y_hist, rho, r0, f0, nc, n_mol, unconverged_out, n_normalizations);
    return nb_check_launch();
}
