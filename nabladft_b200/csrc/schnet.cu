// schnet.cu -- SchNet (config/model/schnet.yaml) energy + analytic forces: continuous-filter convolution.
//
// Replaces schnetpack.representation.SchNet / SchNetInteraction (un-vendored schnetpack 2.0.4; SURVEY.md
// A.1, section 8 row a8) inside NeuralNetworkPotential(PairwiseDistances -> SchNet -> Atomwise -> Forces):
//   x = emb(Z);  6x:  y = in2f(x);  W_e = fcut(d_e) * (ssp(phi(d_e) W1 + b1) W2^T + b2)
//                     agg_i = sum_{e->i} y_j * W_e ;  x += f2out(agg) ,  f2out = Dense(ssp) -> Dense
// The filter network is an MLP, so only its first layer is banded (16 of the 100 Gaussians, edges
// grouped by distance bin as in filter.cu); the second layer is ONE tall GEMM per layer on the
// tensor cores (M = 2 E: h and dh/dd stacked, N = K = 128).  The cutoff, the second-layer bias and
// dW/dd = fcut' (h W2^T + b2) + fcut (dh W2^T) are applied on the fly inside the cfconv kernels, so
// the per-edge HBM streams are G1 (forward) and G1, G2 (backward): 512 B / 1 KB per edge per layer.
//
// cfconv kernels: same structure as K_msg (painn_msg.cu) with one channel chunk: warp per atom,
// lane = 4 channels, per-warp cp.async ring for the edge rows and the gathered neighbour rows,
// register accumulation in CSR order (deterministic, no atomics); backward by SOURCE atom using
// edge symmetry (W depends on d only).
#include <new>

#include "engine_common.cuh"

#define SF1_THREADS 128
#define SF1_CHUNK 32
#define SF1_SPLIT 8
#define CF_WARPS 1  // one warp per CTA, like K_msg: a CTA leaves the SM as soon as its atom is done (was 8)
#define CF_THREADS (CF_WARPS * 32)
#define CF_STAGES 4

namespace {

__device__ __forceinline__ void cp_async16_(float* smem_dst, const float* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_commit_() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait_() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// schnetpack CosineCutoff and its derivative
__device__ __forceinline__ void cos_cut(float d, float rc, float& fc, float& dfc) {
    const float a = 3.14159265358979323846f / rc;
    const bool in = d < rc;
    fc = in ? 0.5f * (cosf(d * a) + 1.0f) : 0.f;
    dfc = in ? -0.5f * a * sinf(d * a) : 0.f;
}

// first filter layer, banded:  h = ssp(phi W1 + b1),  dh = sigmoid(.) * (phi' W1)      HH[l][0|1][e][F]
__global__ void __launch_bounds__(SF1_THREADS) k_schnet_filter1(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                               const int32_t* __restrict__ scr, const float* __restrict__ w1,
                                                               const float* __restrict__ b1, const float* __restrict__ offsets, int n_rbf,
                                                               float coeff, size_t e_stride, float* __restrict__ HH) {
    __shared__ __align__(16) float sphi[SF1_CHUNK][2 * NB_BAND];
    __shared__ int32_t sedge[SF1_CHUNK];
    if (status[1] != 0) return;
    const int bin = blockIdx.x, split = blockIdx.y, layer = blockIdx.z;
    const int b0 = scr[SCR_START + bin], b1e = scr[SCR_START + bin + 1];
    const int cnt = b1e - b0;
    if (cnt == 0) return;
    const int per = (cnt + SF1_SPLIT - 1) / SF1_SPLIT;
    const int lo = b0 + split * per, hi = min(lo + per, b1e);
    if (lo >= hi) return;
    const int k0 = min(max(bin - (NB_BAND / 2 - 1), 0), n_rbf - NB_BAND);
    const int c4 = (threadIdx.x & 31) * 4, el = threadIdx.x >> 5;
    float4 wreg[NB_BAND];
    const float* wl = w1 + ((size_t)layer * n_rbf + k0) * NB_F + c4;
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) wreg[kk] = ldg4(wl + (size_t)kk * NB_F);
    const float4 bias = ldg4(b1 + (size_t)layer * NB_F + c4);
    float* H = HH + (size_t)layer * 2 * e_stride * NB_F;
    float* dH = H + e_stride * NB_F;
    for (int base = lo; base < hi; base += SF1_CHUNK) {
        const int nchunk = min(SF1_CHUNK, hi - base);
        if (threadIdx.x < nchunk) {
            const int e = scr[SCR_PERM + base + threadIdx.x];
            const float d = geom[4 * (size_t)e + 3];
            float* row = sphi[threadIdx.x];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                const float t = d - __ldg(offsets + k0 + kk);
                const float p = expf(coeff * (t * t));
                row[kk] = p;
                row[NB_BAND + kk] = p * (2.0f * coeff) * t;
            }
            sedge[threadIdx.x] = e;
        }
        __syncthreads();
        for (int t = el; t < nchunk; t += SF1_THREADS / 32) {
            const float4* row4 = reinterpret_cast<const float4*>(sphi[t]);
            float4 pre = bias, dpre = f4(0.f);
#pragma unroll
            for (int q4 = 0; q4 < NB_BAND / 4; ++q4) {
                const float4 p = row4[q4], dp = row4[NB_BAND / 4 + q4];
                fma4s(pre, wreg[4 * q4 + 0], p.x); fma4s(pre, wreg[4 * q4 + 1], p.y);
                fma4s(pre, wreg[4 * q4 + 2], p.z); fma4s(pre, wreg[4 * q4 + 3], p.w);
                fma4s(dpre, wreg[4 * q4 + 0], dp.x); fma4s(dpre, wreg[4 * q4 + 1], dp.y);
                fma4s(dpre, wreg[4 * q4 + 2], dp.z); fma4s(dpre, wreg[4 * q4 + 3], dp.w);
            }
            const size_t off = (size_t)sedge[t] * NB_F + c4;
            st4(H + off, make_float4(sspf_(pre.x), sspf_(pre.y), sspf_(pre.z), sspf_(pre.w)));
            st4(dH + off, make_float4(sigmoidf_(pre.x) * dpre.x, sigmoidf_(pre.y) * dpre.y, sigmoidf_(pre.z) * dpre.z, sigmoidf_(pre.w) * dpre.w));
        }
        __syncthreads();
    }
}

// agg_i = sum_{e in row i} y[col e] * fcut(d_e) * (G1_e + b2)
__global__ void __launch_bounds__(CF_THREADS) k_cfconv_fwd(const float* __restrict__ y, const float* __restrict__ G1, const float* __restrict__ b2,
                                                          const float* __restrict__ geom, const int32_t* __restrict__ row_ptr,
                                                          const int32_t* __restrict__ col, float cutoff, int n_atoms, float* __restrict__ agg) {
    __shared__ __align__(16) float ring_all[CF_WARPS * CF_STAGES * 2 * NB_F];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = blockIdx.x * CF_WARPS + warp;
    if (i >= n_atoms) return;
    const int c = lane * 4;
    float* ring = ring_all + warp * (CF_STAGES * 2 * NB_F) + c;
    const float4 bias = ldg4(b2 + c);
    float4 acc = f4(0.f);
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
#pragma unroll
    for (int s = 0; s < CF_STAGES; ++s) {
        if (e0 + s < e1) {
            const int j = __ldg(col + e0 + s);
            cp_async16_(ring + s * 2 * NB_F, G1 + (size_t)(e0 + s) * NB_F + c);
            cp_async16_(ring + s * 2 * NB_F + NB_F, y + (size_t)j * NB_F + c);
        }
        cp_commit_();
    }
    int j_pf = (e0 + CF_STAGES < e1) ? __ldg(col + e0 + CF_STAGES) : 0;
    float dn = (e0 < e1) ? __ldg(geom + 4 * (size_t)e0 + 3) : 0.f;
    int slot = 0;
    for (int e = e0; e < e1; ++e) {
        const float d = dn;
        if (e + 1 < e1) dn = __ldg(geom + 4 * (size_t)(e + 1) + 3);
        const int j_issue = j_pf;
        if (e + CF_STAGES + 1 < e1) j_pf = __ldg(col + e + CF_STAGES + 1);
        float fc, dfc;
        cos_cut(d, cutoff, fc, dfc);
        cp_wait_<CF_STAGES - 1>();
        float* row = ring + slot * 2 * NB_F;
        const float4 g1 = *reinterpret_cast<const float4*>(row), yj = *reinterpret_cast<const float4*>(row + NB_F);
        fma4(acc, yj, (g1 + bias) * fc);
        if (e + CF_STAGES < e1) {
            cp_async16_(row, G1 + (size_t)(e + CF_STAGES) * NB_F + c);
            cp_async16_(row + NB_F, y + (size_t)j_issue * NB_F + c);
        }
        cp_commit_();
        slot = (slot + 1 == CF_STAGES) ? 0 : slot + 1;
    }
    cp_wait_<0>();
    st4(agg + (size_t)i * NB_F + c, acc);
}

// backward by source atom j (edge symmetry):  gy_j = sum_e W_e * gagg_i ;  dE/dd(e') = sum_c dW_e y_j gagg_i
__global__ void __launch_bounds__(CF_THREADS) k_cfconv_bwd(const float* __restrict__ y, const float* __restrict__ G1, const float* __restrict__ G2,
                                                          const float* __restrict__ b2, const float* __restrict__ geom,
                                                          const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col, float cutoff,
                                                          int n_atoms, const float* __restrict__ gagg, float* __restrict__ gy,
                                                          float* __restrict__ egrad) {
    __shared__ __align__(16) float ring_all[CF_WARPS * CF_STAGES * 3 * NB_F];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * CF_WARPS + warp;
    if (j >= n_atoms) return;
    const int c = lane * 4;
    float* ring = ring_all + warp * (CF_STAGES * 3 * NB_F) + c;
    const float4 bias = ldg4(b2 + c);
    const float4 yj = ldg4(y + (size_t)j * NB_F + c);
    float4 acc = f4(0.f);
    const int e0 = row_ptr[j], e1 = row_ptr[j + 1];
#pragma unroll
    for (int s = 0; s < CF_STAGES; ++s) {
        if (e0 + s < e1) {
            const int i = __ldg(col + e0 + s);
            float* dst = ring + s * 3 * NB_F;
            cp_async16_(dst, G1 + (size_t)(e0 + s) * NB_F + c);
            cp_async16_(dst + NB_F, G2 + (size_t)(e0 + s) * NB_F + c);
            cp_async16_(dst + 2 * NB_F, gagg + (size_t)i * NB_F + c);
        }
        cp_commit_();
    }
    int i_pf = (e0 + CF_STAGES < e1) ? __ldg(col + e0 + CF_STAGES) : 0;
    float dn = (e0 < e1) ? __ldg(geom + 4 * (size_t)e0 + 3) : 0.f;
    int slot = 0;
    for (int e = e0; e < e1; ++e) {
        const float d = dn;
        if (e + 1 < e1) dn = __ldg(geom + 4 * (size_t)(e + 1) + 3);
        const int i_issue = i_pf;
        if (e + CF_STAGES + 1 < e1) i_pf = __ldg(col + e + CF_STAGES + 1);
        float fc, dfc;
        cos_cut(d, cutoff, fc, dfc);
        cp_wait_<CF_STAGES - 1>();
        float* row = ring + slot * 3 * NB_F;
        const float4 g1 = *reinterpret_cast<const float4*>(row) + bias, g2 = *reinterpret_cast<const float4*>(row + NB_F),
                     ga = *reinterpret_cast<const float4*>(row + 2 * NB_F);
        fma4(acc, g1 * fc, ga);
        float4 dw = g1 * dfc; fma4s(dw, g2, fc);
        float gd = warp_sum(hsum4(dw * (yj * ga)));
        if (lane == 0) atomicAdd(egrad + 4 * (size_t)e + 3, gd);  // fire-and-forget: no L2 round trip on the critical path (single writer)
        if (e + CF_STAGES < e1) {
            cp_async16_(row, G1 + (size_t)(e + CF_STAGES) * NB_F + c);
            cp_async16_(row + NB_F, G2 + (size_t)(e + CF_STAGES) * NB_F + c);
            cp_async16_(row + 2 * NB_F, gagg + (size_t)i_issue * NB_F + c);
        }
        cp_commit_();
        slot = (slot + 1 == CF_STAGES) ? 0 : slot + 1;
    }
    cp_wait_<0>();
    st4(gy + (size_t)j * NB_F + c, acc);
}

struct SWorkspace {
    int32_t *row_ptr, *col, *rev, *deg, *sort_scr;
    float *geom, *HH, *G;
    float *y[16], *t[16];
    float *x, *agg, *act, *ro_pre, *eps, *mu_dummy;
    float *gx, *gt, *gagg, *gy, *g_ro, *egrad;
    int64_t bytes;
};

SWorkspace s_carve(void* p, int L, int64_t N, int64_t E, bool forces) {
    SWorkspace w{};
    Carver c(p);
    const int F = NB_F;
    w.row_ptr = c.take<int32_t>(N + 1);
    w.col = c.take<int32_t>(E);
    w.rev = c.take<int32_t>(E);
    w.deg = c.take<int32_t>(N);
    w.sort_scr = c.take<int32_t>(E + 1024);
    w.geom = c.take<float>(4 * E);
    w.HH = c.take<float>((int64_t)L * 2 * E * F);
    w.G = c.take<float>((int64_t)L * 2 * E * F);
    for (int l = 0; l < L; ++l) {
        w.y[l] = c.take<float>(N * F);
        w.t[l] = c.take<float>(N * F);
    }
    w.x = c.take<float>(N * F);
    w.agg = c.take<float>(N * F);
    w.act = c.take<float>(N * F);
    w.mu_dummy = c.take<float>(N * 3 * F);  // nb_embed also zeroes a vector field; SchNet has none
    w.ro_pre = c.take<float>(N * (F / 2));
    w.eps = c.take<float>(N);
    if (forces) {
        w.gx = c.take<float>(N * F);
        w.gt = c.take<float>(N * F);
        w.gagg = c.take<float>(N * F);
        w.gy = c.take<float>(N * F);
        w.g_ro = c.take<float>(N * (F / 2));
        w.egrad = c.take<float>(4 * E);
    }
    w.bytes = (c.off + kAlign - 1) / kAlign * kAlign;
    return w;
}

bool s_weights_ok(const nb200_schnet_weights* w) {
    return w && w->emb && w->w_f1 && w->b_f1 && w->W_f2 && w->b_f2 && w->I1 && w->P1 && w->p1 && w->P2 && w->p2 && w->R1 && w->e1 && w->R2 &&
           w->e2 && w->rbf_offsets;
}

}  // namespace

int nb_schnet_filter1(const float* geom, const int32_t* status, const float* w1, const float* b1, const float* offsets, int n_layers, int n_rbf,
                      float cutoff, float coeff, size_t e_stride, int32_t* sort_scr, float* HH, cudaStream_t s) {
    const float dx = cutoff / (float)(n_rbf - 1);
    NB_TRY(nb_bin_sort(geom, status, 1.0f, 1.0f / dx, n_rbf, sort_scr, s));
    k_schnet_filter1<<<dim3(n_rbf, SF1_SPLIT, n_layers), SF1_THREADS, 0, s>>>(geom, status, sort_scr, w1, b1, offsets, n_rbf, coeff, e_stride, HH);
    return nb_check_launch();
}

int nb_schnet_cfconv_fwd(const float* y, const float* G1, const float* b2, const float* geom, const int32_t* row_ptr, const int32_t* col, float cutoff,
                         int n_atoms, float* agg, cudaStream_t s) {
    k_cfconv_fwd<<<(n_atoms + CF_WARPS - 1) / CF_WARPS, CF_THREADS, 0, s>>>(y, G1, b2, geom, row_ptr, col, cutoff, n_atoms, agg);
    return nb_check_launch();
}

int nb_schnet_cfconv_bwd(const float* y, const float* G1, const float* G2, const float* b2, const float* geom, const int32_t* row_ptr, const int32_t* col,
                         float cutoff, int n_atoms, const float* gagg, float* gy, float* egrad, cudaStream_t s) {
    k_cfconv_bwd<<<(n_atoms + CF_WARPS - 1) / CF_WARPS, CF_THREADS, 0, s>>>(y, G1, G2, b2, geom, row_ptr, col, cutoff, n_atoms, gagg, gy, egrad);
    return nb_check_launch();
}

extern "C" int64_t nb200_schnet_workspace_bytes(const nb200_schnet_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap,
                                                int32_t with_forces) {
    (void)b_cap;
    if (!w || w->n_layers <= 0 || w->n_layers > 16 || w->n_feat != NB_F || n_cap < 0 || e_cap < 0) return NB200_EINVAL;
    return s_carve(nullptr, w->n_layers, n_cap, e_cap, with_forces != 0).bytes;
}

extern "C" int nb200_schnet_energy_forces(nb200_engine* eng, const nb200_schnet_weights* w, const int32_t* z, const float* pos,
                                          const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace,
                                          int64_t workspace_bytes, float* energy, float* forces, int32_t* status, void* stream) {
    if (!eng || !s_weights_ok(w) || !z || !pos || !mol_ptr || !workspace || !energy || !status) return NB200_EINVAL;
    if (w->n_feat != NB_F || w->n_layers <= 0 || w->n_layers > 16 || w->n_rbf < NB_BAND || w->n_rbf > NB_NBINS_MAX) return NB200_EUNSUPPORTED;
    if (n_mol <= 0 || n_atoms <= 0 || e_cap <= 0) return NB200_EINVAL;
    const int L = w->n_layers, F = NB_F, K = w->n_rbf, N = n_atoms;
    const float dx = w->cutoff / (float)(K - 1);
    if (!(w->rbf_coeff < 0.f) || w->rbf_coeff * (7.0f * dx) * (7.0f * dx) > -23.0f) return NB200_EUNSUPPORTED;  // band truncation validity
    const bool want_f = forces != nullptr;
    SWorkspace ws = s_carve(workspace, L, N, e_cap, want_f);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;

    { Scope sc(eng, s, CAT_NBR, 3);
    NB_TRY(nb200_neighbor_build(pos, mol_ptr, n_mol, N, w->cutoff, 0x7fffffff, e_cap, ws.row_ptr, ws.col, ws.rev, ws.geom, ws.deg, status, s)); }
    const size_t es = (size_t)e_cap;
    { Scope sc(eng, s, CAT_FILTER, 4);
    NB_TRY(nb_schnet_filter1(ws.geom, status, w->w_f1, w->b_f1, w->rbf_offsets, L, K, w->cutoff, w->rbf_coeff, es, ws.sort_scr, ws.HH, s)); }
    // second filter layer: one tall GEMM per layer over the stacked (h, dh/dd) rows
    for (int l = 0; l < L; ++l)
        NB_TRY(linear_fwd(eng, s, 2 * e_cap, F, F, ws.HH + (size_t)l * 2 * es * F, F, w->W_f2 + (size_t)l * F * F, F, ws.G + (size_t)l * 2 * es * F, F,
                          false, nullptr, nullptr));
    { Scope sc(eng, s, CAT_EMBED, 1); NB_TRY(nb_embed(z, w->emb, w->z_offset, w->n_elem, N, ws.x, ws.mu_dummy, status, s)); }
    for (int l = 0; l < L; ++l) {
        const float* G1 = ws.G + (size_t)l * 2 * es * F;
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.x, F, w->I1 + (size_t)l * F * F, F, ws.y[l], F, false, nullptr, nullptr));
        { Scope sc(eng, s, CAT_MSG_FWD, 1);
        NB_TRY(nb_schnet_cfconv_fwd(ws.y[l], G1, w->b_f2 + (size_t)l * F, ws.geom, ws.row_ptr, ws.col, w->cutoff, N, ws.agg, s)); }
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.agg, F, w->P1 + (size_t)l * F * F, F, ws.t[l], F, false, w->p1 + (size_t)l * F, ws.act, NB_ACT_SSP));
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.act, F, w->P2 + (size_t)l * F * F, F, ws.x, F, true, w->p2 + (size_t)l * F, nullptr));  // x += f2out(agg)
    }
    NB_TRY(linear_fwd(eng, s, N, F / 2, F, ws.x, F, w->R1, F, ws.ro_pre, F / 2, false, nullptr, nullptr));
    { Scope sc(eng, s, CAT_READOUT, 2);
    NB_TRY(nb_readout(ws.ro_pre, w->e1, w->R2, w->e2, N, F / 2, ws.eps, s));
    NB_TRY(nb_mol_sum(ws.eps, mol_ptr, n_mol, w->energy_shift_per_atom, energy, s)); }
    // a failed graph build or embedding leaves finite numbers of an emptied graph behind: NaN them (as PaiNN) so that no error passes silently
    if (!want_f) { Scope sc(eng, s, CAT_READOUT, 1); return nb_poison_on_error(status, energy, n_mol, nullptr, 0, s); }

    if (cudaMemsetAsync(ws.egrad, 0, es * 4 * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_readout_bwd(ws.ro_pre, w->R2, N, F / 2, ws.g_ro, s)); }
    NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.g_ro, F / 2, w->R1, F, ws.gx, F, false));
    for (int l = L - 1; l >= 0; --l) {
        const float* G1 = ws.G + (size_t)l * 2 * es * F;
        const float* G2 = G1 + es * F;
        NB_TRY(linear_bwd(eng, s, N, F, F, ws.gx, F, w->P2 + (size_t)l * F * F, F, ws.gt, F, false));
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_act_bwd(ws.gt, ws.t[l], (int64_t)N * F, NB_ACT_SSP, s)); }
        NB_TRY(linear_bwd(eng, s, N, F, F, ws.gt, F, w->P1 + (size_t)l * F * F, F, ws.gagg, F, false));
        { Scope sc(eng, s, CAT_MSG_BWD, 1);
        NB_TRY(nb_schnet_cfconv_bwd(ws.y[l], G1, G2, w->b_f2 + (size_t)l * F, ws.geom, ws.row_ptr, ws.col, w->cutoff, N, ws.gagg, ws.gy, ws.egrad,
                                    s)); }
        if (l > 0) NB_TRY(linear_bwd(eng, s, N, F, F, ws.gy, F, w->I1 + (size_t)l * F * F, F, ws.gx, F, true));
    }
    { Scope sc(eng, s, CAT_FORCE, 2); NB_TRY(nb200_edge_forces(ws.egrad, ws.geom, ws.row_ptr, ws.rev, N, forces, s));
      NB_TRY(nb_poison_on_error(status, energy, n_mol, forces, (int64_t)3 * N, s)); }
    return NB200_OK;
}

// Test entry point (include/nabla_b200.h), not a supported API: one launch of nb200_schnet_energy_forces on caller-built inputs, through the
// wrapper the engine calls, so that tests/test_gpu_schnet_kernels.py can compare each with a float64 reference.
extern "C" int nb200_schnet_test_op(const nb200_schnet_test_args* a, void* stream) {
    auto all = [](auto... p) { return ((p != nullptr) && ...); };
    auto aligned = [](auto... p) { return ((reinterpret_cast<uintptr_t>(p) % 16 == 0) && ...); };
    if (!a || a->n_layers < 0 || a->n_atoms < 0 || a->n_edges < 0 || a->e_stride < 0 || a->m < 0) return NB200_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    const int F = NB_F;
    switch (a->op) {
    case NB200_SC_FILTER1: {
        if (!all(a->geom, a->status, a->w_f1, a->b_f1, a->rbf_offsets, a->sort_scratch, a->HH) || !aligned(a->w_f1, a->b_f1, a->HH)) return NB200_EINVAL;
        if (a->e_stride < a->n_edges) return NB200_EINVAL;
        const int K = a->n_rbf;
        if (K < NB_BAND || K > NB_NBINS_MAX) return NB200_EUNSUPPORTED;
        const float dx = a->cutoff / (float)(K - 1);  // as nb200_schnet_energy_forces
        if (!(a->rbf_coeff < 0.f) || a->rbf_coeff * (7.0f * dx) * (7.0f * dx) > -23.0f) return NB200_EUNSUPPORTED;
        if (a->n_layers == 0) return NB200_OK;
        return nb_schnet_filter1(a->geom, a->status, a->w_f1, a->b_f1, a->rbf_offsets, a->n_layers, K, a->cutoff, a->rbf_coeff, (size_t)a->e_stride,
                                 a->sort_scratch, a->HH, s);
    }
    case NB200_SC_CFCONV_FWD:
        if (!all(a->y, a->G1, a->b2, a->geom, a->row_ptr, a->col, a->agg) || !aligned(a->y, a->G1, a->b2, a->agg)) return NB200_EINVAL;
        if (a->n_atoms == 0) return NB200_OK;
        return nb_schnet_cfconv_fwd(a->y, a->G1, a->b2, a->geom, a->row_ptr, a->col, a->cutoff, a->n_atoms, a->agg, s);
    case NB200_SC_CFCONV_BWD:
        if (!all(a->y, a->G1, a->G2, a->b2, a->geom, a->row_ptr, a->col, a->gagg, a->gy, a->egrad) || !aligned(a->y, a->G1, a->G2, a->b2, a->gagg, a->gy))
            return NB200_EINVAL;
        if (a->n_atoms == 0) return NB200_OK;
        return nb_schnet_cfconv_bwd(a->y, a->G1, a->G2, a->b2, a->geom, a->row_ptr, a->col, a->cutoff, a->n_atoms, a->gagg, a->gy, a->egrad, s);
    case NB200_SC_LINEAR_ACT:  // linear_fwd(..., act, NB_ACT_SSP) of f2out.0
        if (!all(a->X, a->W, a->bias, a->Y, a->act) || !aligned(a->X, a->W, a->bias, a->Y, a->act)) return NB200_EINVAL;
        if (a->m == 0) return NB200_OK;
        return nb_gemm_tf32x3_ex(a->m, F, F, a->X, F, a->W, F, 0, a->Y, F, 0, a->bias, a->act, NB_ACT_SSP, s);
    }
    return NB200_EINVAL;
}
