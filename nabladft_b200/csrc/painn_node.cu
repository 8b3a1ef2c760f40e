// painn_node.cu -- per-atom elementwise kernels around the node GEMMs (K_upd and friends).
//
// Replaces the ~8 eager elementwise launches per layer of PaiNNMixing.forward (schnetpack;
// SURVEY.md A.2) / PaiNNUpdate.forward (nablaDFT/painn_pyg/painn.py:535-548), the embedding
// (layers.py:198-222), the readout MLP tail + per-molecule scatter (painn.py:79-83,127-128)
// and their autograd backward.  All arrays are N x (multiple of 128) fp32 and L2-resident at
// the reference's batch sizes; one warp per atom, lane = 4 channels (float4).
//
// Canonical roles (host permutes PaiNN-OC weights into them): VW = mu . U^T, V = first half
// (normed), Wv = second half (gated into mu);  y = (y0 scalar, y1 gate, y2 dot-scale).
//   q'' = q' + y0 + y2 * <V,Wv> ;  mu'' = mu' + y1 * Wv
#include "painn_node.cuh"

#define NODE_THREADS 256

__global__ void __launch_bounds__(NODE_THREADS) k_embed(const int32_t* __restrict__ z, const float* __restrict__ emb, int z_offset,
                                                       int n_elem, int n_atoms, float* __restrict__ q, float* __restrict__ mu,
                                                       int32_t* __restrict__ status) {
    const int t = blockIdx.x * NODE_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    int zi = z[i] - z_offset;
    if (zi < 0 || zi >= n_elem) {
        if (c == 0) atomicMin(&status[1], NB200_EINVAL);
        zi = 0;
    }
    st4(q + (size_t)i * NB_F + c, ldg4(emb + (size_t)zi * NB_F + c));
    float* m = mu + (size_t)i * 3 * NB_F + c;
    st4(m, f4(0.f)); st4(m + NB_F, f4(0.f)); st4(m + 2 * NB_F, f4(0.f));
}

__global__ void __launch_bounds__(NODE_THREADS) k_silu_bwd(float* __restrict__ g, const float* __restrict__ pre, int64_t n4, int kind) {
    const int64_t t = (int64_t)blockIdx.x * NODE_THREADS + threadIdx.x;
    if (t >= n4) return;
    const float4 p = ldg4(pre + 4 * t);
    float4 v = *reinterpret_cast<const float4*>(g + 4 * t);
    st4(g + 4 * t, make_float4(v.x * dactf_(p.x, kind), v.y * dactf_(p.y, kind), v.z * dactf_(p.z, kind), v.w * dactf_(p.w, kind)));
}

// gy =(gq, sum_x gmu[x]*Wv[x], gq*dot) ; gVW[x] = (gdot*Wv[x], gmu[x]*y1 + gdot*V[x]), gdot = gq*y2
__global__ void __launch_bounds__(NODE_THREADS) k_upd_combine_bwd(const float* __restrict__ gq, const float* __restrict__ gmu,
                                                                 const float* __restrict__ y, const float* __restrict__ VW, int n_atoms,
                                                                 float* __restrict__ gy, float* __restrict__ gVW) {
    const int t = blockIdx.x * NODE_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float4 g = ldg4(gq + (size_t)i * NB_F + c);
    const float* yi = y + (size_t)i * 3 * NB_F + c;
    const float4 y1 = ldg4(yi + NB_F), y2 = ldg4(yi + 2 * NB_F);
    const float4 gdot = g * y2;
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    const float* gm = gmu + (size_t)i * 3 * NB_F + c;
    float* gv = gVW + (size_t)i * 6 * NB_F + c;
    float4 dot = f4(0.f), gy1 = f4(0.f);
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        const float4 V = ldg4(v + x * 2 * NB_F), Wv = ldg4(v + x * 2 * NB_F + NB_F), h = ldg4(gm + x * NB_F);
        fma4(dot, V, Wv);
        fma4(gy1, h, Wv);
        st4(gv + x * 2 * NB_F, gdot * Wv);
        float4 gw = h * y1; fma4(gw, gdot, V);
        st4(gv + x * 2 * NB_F + NB_F, gw);
    }
    float* go = gy + (size_t)i * 3 * NB_F + c;
    st4(go, g); st4(go + NB_F, gy1); st4(go + 2 * NB_F, g * dot);
}

// gV[x] += gn * V[x] / nrm
__global__ void __launch_bounds__(NODE_THREADS) k_upd_norm_bwd(const float* __restrict__ gn, const float* __restrict__ VW,
                                                              const float* __restrict__ nrm, int n_atoms, float* __restrict__ gVW) {
    const int t = blockIdx.x * NODE_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float4 n = ldg4(nrm + (size_t)i * NB_F + c), g = ldg4(gn + (size_t)i * NB_F + c);
    const float4 s = make_float4(g.x / n.x, g.y / n.y, g.z / n.z, g.w / n.w);
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    float* gv = gVW + (size_t)i * 6 * NB_F + c;
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        float4 o = *reinterpret_cast<const float4*>(gv + x * 2 * NB_F);
        fma4(o, s, ldg4(v + x * 2 * NB_F));
        st4(gv + x * 2 * NB_F, o);
    }
}

// readout tail: pre += e1 (kept), eps_i = sum_k silu(pre[k]) R2[k] + e2.  width = F/2 = 64: 2 per lane.
__global__ void __launch_bounds__(NODE_THREADS) k_readout(float* __restrict__ pre, const float* __restrict__ e1, const float* __restrict__ R2,
                                                         const float* __restrict__ e2, int n_atoms, int width, float* __restrict__ eps_atom) {
    const int t = blockIdx.x * NODE_THREADS + threadIdx.x;
    const int i = t >> 5, lane = t & 31;
    if (i >= n_atoms) return;
    float acc = 0.f;
    for (int k = lane; k < width; k += 32) {
        const float p = pre[(size_t)i * width + k] + __ldg(e1 + k);
        pre[(size_t)i * width + k] = p;
        acc = fmaf(siluf_(p), __ldg(R2 + k), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) eps_atom[i] = acc + __ldg(e2);
}

// E_m = sum_{i in m} eps_i (+ shift * n_atoms): one warp per molecule, fixed order => deterministic
__global__ void __launch_bounds__(NODE_THREADS) k_mol_sum(const float* __restrict__ eps_atom, const int32_t* __restrict__ mol_ptr, int n_mol,
                                                         float shift_per_atom, float* __restrict__ energy) {
    const int t = blockIdx.x * NODE_THREADS + threadIdx.x;
    const int m = t >> 5, lane = t & 31;
    if (m >= n_mol) return;
    const int a = mol_ptr[m], b = mol_ptr[m + 1];
    float acc = 0.f;
    for (int i = a + lane; i < b; i += 32) acc += eps_atom[i];
    acc = warp_sum(acc);
    if (lane == 0) energy[m] = acc + shift_per_atom * (float)(b - a);
}

__global__ void __launch_bounds__(NODE_THREADS) k_readout_bwd(const float* __restrict__ pre, const float* __restrict__ R2, int64_t n, int width,
                                                             float* __restrict__ g_pre) {
    const int64_t t = (int64_t)blockIdx.x * NODE_THREADS + threadIdx.x;
    if (t >= n) return;
    g_pre[t] = __ldg(R2 + (int)(t % width)) * dsiluf_(pre[t]);
}

// error flag set by the neighbour build (capacity, neighbour cap, bad element): the outputs of this call become NaN, so that a caller who
// defers the status check (asynchronous forward) can never consume numbers computed on an empty / truncated graph
__global__ void __launch_bounds__(NODE_THREADS) k_poison_on_error(const int32_t* __restrict__ status, float* __restrict__ energy, int n_mol,
                                                                 float* __restrict__ forces, int64_t n_f) {
    if (status[1] == 0) return;
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t t = (int64_t)blockIdx.x * NODE_THREADS + threadIdx.x; t < n_mol + n_f; t += (int64_t)gridDim.x * NODE_THREADS) {
        if (t < n_mol) energy[t] = nan;
        else if (forces) forces[t - n_mol] = nan;
    }
}

static inline int grid_for(int64_t n) { return (int)((n + NODE_THREADS - 1) / NODE_THREADS); }
int nb_poison_on_error(const int32_t* status, float* energy, int n_mol, float* forces, int64_t n_f, cudaStream_t s) {
    k_poison_on_error<<<32, NODE_THREADS, 0, s>>>(status, energy, n_mol, forces, forces ? n_f : 0);
    return nb_check_launch();
}

int nb_embed(const int32_t* z, const float* emb, int z_offset, int n_elem, int n_atoms, float* q, float* mu, int32_t* status,
             cudaStream_t s) {
    k_embed<<<grid_for((int64_t)n_atoms * 32), NODE_THREADS, 0, s>>>(z, emb, z_offset, n_elem, n_atoms, q, mu, status);
    return nb_check_launch();
}
int nb_act_bwd(float* g, const float* pre, int64_t n, int kind, cudaStream_t s) {
    k_silu_bwd<<<grid_for(n / 4), NODE_THREADS, 0, s>>>(g, pre, n / 4, kind);
    return nb_check_launch();
}
int nb_upd_combine_bwd(const float* gq, const float* gmu, const float* y, const float* VW, int n_atoms, float* gy, float* gVW,
                       cudaStream_t s) {
    k_upd_combine_bwd<<<grid_for((int64_t)n_atoms * 32), NODE_THREADS, 0, s>>>(gq, gmu, y, VW, n_atoms, gy, gVW);
    return nb_check_launch();
}
int nb_upd_norm_bwd(const float* gn, const float* VW, const float* nrm, int n_atoms, float* gVW, cudaStream_t s) {
    k_upd_norm_bwd<<<grid_for((int64_t)n_atoms * 32), NODE_THREADS, 0, s>>>(gn, VW, nrm, n_atoms, gVW);
    return nb_check_launch();
}
int nb_readout(float* pre, const float* e1, const float* R2, const float* e2, int n_atoms, int width, float* eps_atom, cudaStream_t s) {
    k_readout<<<grid_for((int64_t)n_atoms * 32), NODE_THREADS, 0, s>>>(pre, e1, R2, e2, n_atoms, width, eps_atom);
    return nb_check_launch();
}
int nb_mol_sum(const float* eps_atom, const int32_t* mol_ptr, int n_mol, float shift_per_atom, float* energy, cudaStream_t s) {
    k_mol_sum<<<grid_for((int64_t)n_mol * 32), NODE_THREADS, 0, s>>>(eps_atom, mol_ptr, n_mol, shift_per_atom, energy);
    return nb_check_launch();
}
int nb_readout_bwd(const float* pre, const float* R2, int n_atoms, int width, float* g_pre, cudaStream_t s) {
    const int64_t n = (int64_t)n_atoms * width;
    k_readout_bwd<<<grid_for(n), NODE_THREADS, 0, s>>>(pre, R2, n, width, g_pre);
    return nb_check_launch();
}
