// painn_train.cu -- parameter-gradient kernels for training PaiNN through the CUDA engine (SURVEY.md section 8 a10/a11, cfg 3).
//
// The reference obtains dLoss/dtheta from torch.autograd over ~40 eager ops per layer (painn_pyg/painn.py:642-653,
// schnetpack AtomisticTask).  The engine's analytic backward (engine.cu) already holds dE/d(activation) for every layer with
// dE/dE_m = 1; because molecules do not interact, the gradient of sum_m c_m E_m w.r.t. a weight is the same sum over atoms /
// edges with each term scaled by c of its molecule.  The kernels here form those scaled sums:
//   k_scale_rows      gs[r,:] = c[atom(r)] * g[r,:]            (operand of the weight-gradient GEMM  dW = gs^T . X, cuBLAS)
//   k_colsum          bias gradients
//   k_act_only        act = silu(pre) (the forward keeps pre-activations only)
//   k_filter_wgrad    d/d w_rbf[l][k][c] = sum_e s1(d_e) phi_k(d_e) gW[e][c],  d/d b_rbf[l][c] = sum_e s2(d_e) gW[e][c]
//                     over the same distance-bin-sorted edge order as the forward filter kernel (filter.cu): the 16-centre band of a
//                     bin is accumulated in registers, one atomic add per (band row, channel) per CTA at the end
//   k_emb_grad        scatter of c_i * dE/dq0_i into the embedding rows
#include "common.cuh"
#include "painn_node.cuh"

namespace {

constexpr int TR_THREADS = 256;

__global__ void __launch_bounds__(TR_THREADS) k_scale_rows(const float* __restrict__ g, const float* __restrict__ seed_atom, int rows_per_atom,
                                                          int64_t n4, int width4, float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * TR_THREADS + threadIdx.x;
    if (t >= n4) return;
    const int64_t row = t / width4;
    const float c = __ldg(seed_atom + row / rows_per_atom);
    st4(out + 4 * t, ldg4(g + 4 * t) * c);
}

__global__ void __launch_bounds__(TR_THREADS) k_act_only(const float* __restrict__ pre, const float* __restrict__ seed_atom, int64_t n4, int width4,
                                                        int kind, float* __restrict__ act) {
    const int64_t t = (int64_t)blockIdx.x * TR_THREADS + threadIdx.x;
    if (t >= n4) return;
    const float c = seed_atom ? __ldg(seed_atom + t / width4) : 1.0f;
    const float4 p = ldg4(pre + 4 * t);
    st4(act + 4 * t, make_float4(c * actf_(p.x, kind), c * actf_(p.y, kind), c * actf_(p.z, kind), c * actf_(p.w, kind)));
}

// out[col] += alpha * sum_rows x[row, col]: grid = (column chunks of 32) x (row chunks of 256), 8 row lanes per CTA, one atomic add per
// (CTA, column), instead of one CTA walking all rows per 32 columns.
constexpr int CS_ROWS = 256;
__global__ void __launch_bounds__(TR_THREADS) k_colsum(const float* __restrict__ x, int64_t n_rows, int width, float alpha, float* __restrict__ out) {
    __shared__ float part[8][33];
    const int col = blockIdx.x * 32 + (threadIdx.x & 31), lane_row = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.y * CS_ROWS, r1 = min(r0 + CS_ROWS, n_rows);
    float acc = 0.f;
    if (col < width)
        for (int64_t r = r0 + lane_row; r < r1; r += 8) acc += x[r * width + col];
    part[lane_row][threadIdx.x & 31] = acc;
    __syncthreads();
    if (lane_row == 0 && col < width) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += part[k][threadIdx.x & 31];
        atomicAdd(out + col, alpha * s);
    }
}

__global__ void __launch_bounds__(TR_THREADS) k_seed_atom(const float* __restrict__ seed_mol, const int32_t* __restrict__ mol_ptr, int n_mol,
                                                         float* __restrict__ seed_atom) {
    const int m = blockIdx.x;
    if (m >= n_mol) return;
    const float c = seed_mol ? seed_mol[m] : 1.0f;
    for (int i = mol_ptr[m] + threadIdx.x; i < mol_ptr[m + 1]; i += TR_THREADS) seed_atom[i] = c;
}

__global__ void __launch_bounds__(TR_THREADS) k_emb_grad(const float* __restrict__ gq, const float* __restrict__ seed_atom, const int32_t* __restrict__ z,
                                                        int z_offset, int n_elem, int n_atoms, float sign, float* __restrict__ g_emb) {
    const int t = blockIdx.x * TR_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    int zi = z[i] - z_offset;
    if (zi < 0 || zi >= n_elem) return;  // flagged by the forward
    const float4 v = ldg4(gq + (size_t)i * NB_F + c) * (sign * (seed_atom ? __ldg(seed_atom + i) : 1.0f));
    float* dst = g_emb + (size_t)zi * NB_F + c;
    atomicAdd(dst, v.x); atomicAdd(dst + 1, v.y); atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
}

}  // namespace

static inline int tr_grid(int64_t n) { return (int)((n + TR_THREADS - 1) / TR_THREADS); }

int nb_seed_atom(const float* seed_mol, const int32_t* mol_ptr, int n_mol, float* seed_atom, cudaStream_t s) {
    k_seed_atom<<<n_mol, TR_THREADS, 0, s>>>(seed_mol, mol_ptr, n_mol, seed_atom);
    return nb_check_launch();
}
int nb_scale_rows(const float* g, const float* seed_atom, int rows_per_atom, int64_t n_rows, int width, float* out, cudaStream_t s) {
    const int64_t n4 = n_rows * width / 4;
    k_scale_rows<<<tr_grid(n4), TR_THREADS, 0, s>>>(g, seed_atom, rows_per_atom, n4, width / 4, out);
    return nb_check_launch();
}
int nb_act_only(const float* pre, const float* seed_atom, int64_t n_rows, int width, int kind, float* act, cudaStream_t s) {
    const int64_t n4 = n_rows * width / 4;
    k_act_only<<<tr_grid(n4), TR_THREADS, 0, s>>>(pre, seed_atom, n4, width / 4, kind, act);
    return nb_check_launch();
}
int nb_colsum(const float* x, int64_t n_rows, int width, float* out, cudaStream_t s, float alpha, int accumulate) {
    if (!accumulate && cudaMemsetAsync(out, 0, (size_t)width * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    if (n_rows <= 0) return NB200_OK;
    dim3 grid((width + 31) / 32, (unsigned)((n_rows + CS_ROWS - 1) / CS_ROWS));
    k_colsum<<<grid, TR_THREADS, 0, s>>>(x, n_rows, width, alpha, out);
    return nb_check_launch();
}
int nb_emb_grad(const float* gq, const float* seed_atom, const int32_t* z, int z_offset, int n_elem, int n_atoms, float* g_emb, cudaStream_t s,
                float sign) {
    k_emb_grad<<<tr_grid((int64_t)n_atoms * 32), TR_THREADS, 0, s>>>(gq, seed_atom, z, z_offset, n_elem, n_atoms, sign, g_emb);
    return nb_check_launch();
}
