// engine.cu -- whole-model PaiNN energy + analytic forces for one batch of conformations.
//
// Replaces `NeuralNetworkPotential.forward` as configured by config/model/painn.yaml
// (PairwiseDistances -> PaiNN -> Atomwise -> Forces -> AddOffsets; SURVEY.md section 3.1) and
// `PaiNN.forward` of nablaDFT/painn_pyg/painn.py:89-148 (config/model/painn-oc.yaml).
// The reference obtains forces with torch.autograd.grad through ~40 eager ops per layer;
// here the backward is hand-derived and runs as the mirrored kernel sequence on one stream,
// with no host synchronisation anywhere (edge count and error flags stay on the device).
//
// The node forward is the fused per-layer kernels of painn_fused.cu; the remaining node-level dense layers (tangent pass, training and
// Hessian backward) run on the wgmma 3xTF32 GEMM of gemm_tc.cu (fp32-accurate: the reference never uses reduced precision, SURVEY.md
// section 0.9).  The weight gradients of the training step run on the wgmma split-K kernel of wgrad_tc.cu.
// Every entry point is a short sequence of the same steps: graph + filters, the fused forward (`run_painn_fused`), the tangent forward
// (`tangent_fwd`, painn_tangent.cu), and the training backward (`train_bwd`, painn_train.cu) or the Hessian backward (`run_painn_hvp`).
#include <new>
#include <utility>

#include "engine_common.cuh"

thread_local int g_nb200_last_cuda_error = 0;

extern "C" int nb200_version(void) { return 100; }
extern "C" int nb200_last_cuda_error(void) { return g_nb200_last_cuda_error; }

extern "C" int nb200_engine_create(nb200_engine** out) {
    if (!out) return NB200_EINVAL;
    nb200_engine* e = new (std::nothrow) nb200_engine();
    if (!e) return NB200_EINVAL;
    if (cublasCreate(&e->blas) != CUBLAS_STATUS_SUCCESS) {
        delete e;
        return NB200_ECUDA;
    }
    cublasSetPointerMode(e->blas, CUBLAS_POINTER_MODE_HOST);
    cublasSetMathMode(e->blas, CUBLAS_DEFAULT_MATH);  // fp32 SGEMM, no TF32
    *out = e;
    return NB200_OK;
}

extern "C" int nb200_engine_set_timing(nb200_engine* eng, int32_t enable) {
    if (!eng) return NB200_EINVAL;
    eng->timing = enable != 0;
    eng->n_used = 0;
    return NB200_OK;
}

// The node GEMMs are the wgmma kernels and the PaiNN node forward is the fused one: both setters accept 1 and refuse 0 (the cuBLAS SGEMM /
// one-launch-per-op paths, which no longer exist) with NB200_EUNSUPPORTED.
extern "C" int nb200_engine_set_gemm_backend(nb200_engine* eng, int32_t backend) {
    if (!eng || (backend != 0 && backend != 1)) return NB200_EINVAL;
    return backend == 1 ? NB200_OK : NB200_EUNSUPPORTED;
}

extern "C" int nb200_engine_set_node_backend(nb200_engine* eng, int32_t backend) {
    if (!eng || (backend != 0 && backend != 1)) return NB200_EINVAL;
    return backend == 1 ? NB200_OK : NB200_EUNSUPPORTED;
}

// Storage of the per-edge arrays of the PaiNN TRAINING calls (nb200_painn_energy_forces_grads, nb200_painn_train_forward / _backward):
// 0 = fp32 (default), 1 = bf16 storage with fp32 arithmetic and accumulation (BASELINE configs[2] "bf16").  Inference is always fp32.
extern "C" int nb200_engine_set_edge_storage(nb200_engine* eng, int32_t bf16) {
    if (!eng || (bf16 != 0 && bf16 != 1)) return NB200_EINVAL;
    eng->edge_bf16 = bf16;
    return NB200_OK;
}

extern "C" int64_t nb200_engine_own_launches(nb200_engine* eng) { return eng ? eng->own_launches : NB200_EINVAL; }

extern "C" int nb200_engine_read_timings(nb200_engine* eng, float* ms_per_cat, int32_t* scopes_per_cat, int32_t n_cat) {
    if (!eng || !ms_per_cat || !scopes_per_cat || n_cat < NCAT) return NB200_EINVAL;
    for (int c = 0; c < n_cat; ++c) { ms_per_cat[c] = 0.f; scopes_per_cat[c] = 0; }
    for (size_t k = 0; k < eng->n_used; ++k) {
        float ms = 0.f;
        if (cudaEventSynchronize(eng->ev[2 * k + 1]) != cudaSuccess || cudaEventElapsedTime(&ms, eng->ev[2 * k], eng->ev[2 * k + 1]) != cudaSuccess) {
            g_nb200_last_cuda_error = (int)cudaGetLastError();
            return NB200_ECUDA;
        }
        ms_per_cat[eng->cat[k]] += ms;
        scopes_per_cat[eng->cat[k]] += 1;
    }
    eng->n_used = 0;
    return NB200_OK;
}

extern "C" int nb200_engine_destroy(nb200_engine* eng) {
    if (!eng) return NB200_EINVAL;
    for (cudaEvent_t e : eng->ev) cudaEventDestroy(e);
    for (cudaEvent_t e : eng->side_ev) cudaEventDestroy(e);
    if (eng->side) cudaStreamDestroy(eng->side);
    if (eng->session && eng->session_free) eng->session_free(eng->session);
    cublasDestroy(eng->blas);
    delete eng;
    return NB200_OK;
}

// ---------------------------------------------------------------------------------------------
// workspace carving (shared by the size query and the run)
namespace {

constexpr int kMaxLayers = 16;

struct Workspace {
    // graph
    int32_t *row_ptr, *col, *rev, *deg, *sort_scr, *sort_scr2;  // sort_scr2 (training): bin sort over ALL directed edges for the filter weight gradients
    float* geom;
    // filters
    float *W, *dW;
    // saved activations per layer
    float *h1pre[kMaxLayers], *xh[kMaxLayers], *VW[kMaxLayers], *nrm[kMaxLayers], *g1pre[kMaxLayers], *y[kMaxLayers];
    float* mu[kMaxLayers + 1];
    // transient
    float *ro_pre, *eps;
    // backward
    float *gq, *gmu_a, *gmu_b, *gy, *gVW, *gt, *gn, *g_ro, *egrad;
    // training only: activation scratch, per-edge filter gradients, per-atom energy seed
    float *act_t, *gW, *seed_atom;
    // force-loss tangent pass (painn_tangent.cu): t_X = directional derivative of X along the position-space direction v
    float *t_geom, *t_h1[kMaxLayers], *t_xh[kMaxLayers], *t_VW[kMaxLayers], *t_nrm[kMaxLayers], *t_g1[kMaxLayers], *t_y[kMaxLayers];
    float *t_q_in[kMaxLayers], *t_q_mid[kMaxLayers], *t_mu_mid[kMaxLayers], *t_mu[kMaxLayers + 1];
    float *t_q, *t_act, *t_ro, *t_gq, *t_gmu_a, *t_gmu_b, *t_gy, *t_gVW, *t_gt, *t_gn, *t_g_ro, *t_gW, *gWd;
    // Hessian-vector product (run_painn_hvp): d2W/dd2 rows [L][E][3F] next to W, dW; tangent of the per-edge geometric gradient
    float *d2W, *t_egrad;
    // fused node forward (painn_fused.cu): layer inputs fq_in[l] and post-message states fq_mid[l], fmu_mid[l] (mu[l + 1] is the layer's
    // output); the training backward reads them as the Linear inputs.  Prepared weight tiles.
    float *fq_in[kMaxLayers + 1], *fq_mid[kMaxLayers], *fmu_mid[kMaxLayers], *fdot[kMaxLayers], *gq_b, *fgn, *fgdot;
    void* wtiles;
    int64_t bytes;
};

// `hvp` (with forces and tangent, without train): the Hessian-vector product's workspace -- the tangent arrays minus those only the weight
// gradients read (t_q_in, t_q_mid, t_mu_mid, t_gW, gWd), plus d2W and t_egrad
Workspace carve(void* p, int L, int F, int64_t B, int64_t N, int64_t E, bool forces, bool train = false, bool tangent = false, bool hvp = false) {
    (void)B;
    Workspace w{};
    Carver c(p);
    w.row_ptr = c.take<int32_t>(N + 1);
    w.col = c.take<int32_t>(E);
    w.rev = c.take<int32_t>(E);
    w.deg = c.take<int32_t>(N);
    w.sort_scr = c.take<int32_t>(E + 1024);
    w.geom = c.take<float>(4 * E);
    // filters: [L][E][3F] W and the same for dW/dd (adjacent), or -- inference with forces -- ONE array [L][E][6F] of [W | dW/dd] records over
    // the same memory
    w.W = c.take<float>((int64_t)L * E * 3 * F * (forces ? 2 : 1));
    w.dW = forces ? w.W + (int64_t)L * E * 3 * F : nullptr;
    for (int l = 0; l < L; ++l) {
        w.h1pre[l] = c.take<float>(N * F);
        w.xh[l] = c.take<float>(N * 3 * F);
        w.VW[l] = c.take<float>(N * 6 * F);
        w.nrm[l] = c.take<float>(N * F);
        w.g1pre[l] = c.take<float>(N * F);
        w.y[l] = c.take<float>(N * 3 * F);
    }
    for (int l = 0; l <= L; ++l) w.mu[l] = c.take<float>(N * 3 * F);
    w.ro_pre = c.take<float>(N * (F / 2));
    w.eps = c.take<float>(N);
    if (forces) {
        w.gq = c.take<float>(N * F);
        w.gmu_a = c.take<float>(N * 3 * F);
        w.gmu_b = c.take<float>(N * 3 * F);
        w.gy = c.take<float>(N * 3 * F);
        w.gVW = c.take<float>(N * 6 * F);
        w.gt = c.take<float>(N * F);
        w.gn = c.take<float>(N * F);
        w.g_ro = c.take<float>(N * (F / 2));
        w.egrad = c.take<float>(4 * E);
    }
    if (train) {
        w.act_t = c.take<float>(N * F);
        w.gW = c.take<float>(E * 3 * F);
        w.seed_atom = c.take<float>(N);
        w.sort_scr2 = c.take<int32_t>(E + 1024);
    }
    if (tangent) {
        w.t_geom = c.take<float>(4 * E);
        for (int l = 0; l < L; ++l) {
            w.t_h1[l] = c.take<float>(N * F); w.t_xh[l] = c.take<float>(N * 3 * F); w.t_VW[l] = c.take<float>(N * 6 * F);
            w.t_nrm[l] = c.take<float>(N * F); w.t_g1[l] = c.take<float>(N * F); w.t_y[l] = c.take<float>(N * 3 * F);
            if (!hvp) { w.t_q_in[l] = c.take<float>(N * F); w.t_q_mid[l] = c.take<float>(N * F); w.t_mu_mid[l] = c.take<float>(N * 3 * F); }
        }
        for (int l = 0; l <= L; ++l) w.t_mu[l] = c.take<float>(N * 3 * F);
        w.t_q = c.take<float>(N * F); w.t_act = c.take<float>(N * F); w.t_ro = c.take<float>(N * (F / 2));
        // backward quantities as ADJACENT (primal, tangent) pairs: every Linear backward of the step is applied to [g ; g^] as ONE GEMM
        // over 2 M rows (same weights; a 9.7 k-atom batch alone covers only 76 of the 148 SMs with 128-row tiles).  The primal pointers
        // carved above stay valid for the inference path; with a tangent pass the backward works on these.
        static_assert((NB_F * sizeof(float)) % kAlign == 0, "pairs must be exactly adjacent");
        w.gq = c.take<float>(N * F); w.t_gq = c.take<float>(N * F);
        w.gmu_a = c.take<float>(N * 3 * F); w.t_gmu_a = c.take<float>(N * 3 * F);
        w.gmu_b = c.take<float>(N * 3 * F); w.t_gmu_b = c.take<float>(N * 3 * F);
        w.gy = c.take<float>(N * 3 * F); w.t_gy = c.take<float>(N * 3 * F);
        w.gVW = c.take<float>(N * 6 * F); w.t_gVW = c.take<float>(N * 6 * F);
        w.gt = c.take<float>(N * F); w.t_gt = c.take<float>(N * F);
        w.gn = c.take<float>(N * F); w.t_gn = c.take<float>(N * F);
        w.t_g_ro = c.take<float>(N * (F / 2));
        if (!hvp) { w.t_gW = c.take<float>(E * 3 * F); w.gWd = c.take<float>(E * 3 * F); }
    }
    if (hvp) {
        w.d2W = c.take<float>((int64_t)L * E * 3 * F);
        w.t_egrad = c.take<float>(4 * E);
    }
    for (int l = 0; l <= L; ++l) w.fq_in[l] = c.take<float>(N * F);
    for (int l = 0; l < L; ++l) { w.fq_mid[l] = c.take<float>(N * F); w.fmu_mid[l] = c.take<float>(N * 3 * F); w.fdot[l] = c.take<float>(N * F); }
    w.gq_b = forces ? c.take<float>(N * F) : nullptr;
    w.fgn = forces ? c.take<float>(N * F) : nullptr;
    w.fgdot = forces ? c.take<float>(N * F) : nullptr;
    w.wtiles = c.take<char>(nb_fused_wtile_bytes(L));
    w.bytes = (c.off + kAlign - 1) / kAlign * kAlign;
    return w;
}

bool weights_ok(const nb200_painn_weights* w) {
    return w && w->emb && w->w_rbf && w->b_rbf && w->rbf_offsets && w->A1 && w->c1 && w->A2 && w->c2 && w->U && w->B1 && w->d1 && w->B2 &&
           w->d2 && w->R1 && w->e1 && w->R2 && w->e2;
}

}  // namespace

extern "C" int64_t nb200_painn_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap,
                                               int32_t with_forces) {
    if (!w || w->n_layers <= 0 || w->n_layers > kMaxLayers || w->n_feat != NB_F || b_cap < 0 || n_cap < 0 || e_cap < 0) return NB200_EINVAL;
    return carve(nullptr, w->n_layers, w->n_feat, b_cap, n_cap, e_cap, with_forces != 0).bytes;
}

namespace {

// The Linear weight gradients are written in 16-byte rows by the wgmma split-K kernel (wgrad_tc.cu): their arrays must be 16-byte aligned.
bool grads_ok(const nb200_painn_weights* g) {
    auto al = [](const float* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    return g && g->emb && g->w_rbf && g->b_rbf && g->A1 && g->c1 && g->A2 && g->c2 && g->U && g->B1 && g->d1 && g->B2 && g->d2 && g->R1 && g->e1 &&
           g->R2 && g->e2 && al(g->A1) && al(g->A2) && al(g->U) && al(g->B1) && al(g->B2) && al(g->R1);
}

// Argument checks every PaiNN entry point makes after its own, before anything is launched.
int args_ok(const nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
            int32_t e_cap, const void* workspace, const int32_t* status) {
    if (!eng || !weights_ok(w) || !z || !mol_ptr || !workspace || !status) return NB200_EINVAL;
    if (w->n_feat != NB_F || w->n_layers <= 0 || w->n_layers > kMaxLayers) return NB200_EUNSUPPORTED;
    if (n_mol <= 0 || n_atoms <= 0 || e_cap <= 0) return NB200_EINVAL;
    return NB200_OK;
}

// Neighbour graph and radial filters (painn.py:104-108 / spk PairwiseDistances + filter_net).  W depends on the distance only (rows of e and
// rev[e] are bitwise equal), so ONE filter row is stored per undirected pair and edge e reads row min(e, rev[e]): half the filter kernel's
// work and writes; the second reader of a row mostly finds it in L2.  `records` (inference with forces): one interleaved [W | dW/dd] record
// per row, one bulk copy per edge in the backward; otherwise W and dW/dd in two arrays, the layout the gradient kernels read.  `train` adds
// the bin sort over every directed edge that the filter weight gradients walk (slot e holds the gradient of the opposite edge's row).
int graph_and_filters(nb200_engine* eng, const nb200_painn_weights* w, const Workspace& ws, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                      int N, int32_t e_cap, int32_t* status, cudaStream_t s, bool records, bool train) {
    const int K = w->n_rbf;
    const int bf16 = train ? eng->edge_bf16 : 0;  // bf16 rows use the first half of their fp32-sized blocks: all offsets stay in floats
    { Scope sc(eng, s, CAT_NBR, 3);
    NB_TRY(nb200_neighbor_build(pos, mol_ptr, n_mol, N, w->cutoff, w->max_neighbors, e_cap, ws.row_ptr, ws.col, ws.rev, ws.geom, ws.deg,
                                status, s)); }
    { Scope sc(eng, s, CAT_FILTER, 4);
    NB_TRY(nb_painn_filter_ex(ws.geom, status, e_cap, w->w_rbf, w->b_rbf, w->n_layers, K, NB_F, w->radial_mode, w->cutoff, w->rbf_offsets,
                              w->rbf_coeff, w->rbf_xscale, ws.W, ws.dW, ws.sort_scr, ws.rev, records ? 1 : 0, s, bf16)); }
    if (!train) return NB200_OK;
    const float dx = (w->cutoff * w->rbf_xscale) / (float)(K - 1);
    Scope sc(eng, s, CAT_FILTER, 3);
    return nb_bin_sort(ws.geom, status, w->rbf_xscale, 1.0f / dx, K, ws.sort_scr2, s, nullptr);
}

// The node forward (E, and with `forces` the analytic F) with the fused node kernels of painn_fused.cu: per layer ONE message kernel and
// ONE node kernel per direction.  The graph and the radial filters are already in the workspace.  q / mu are not updated in place: layer l
// reads fq_in[l], mu[l], the message kernel writes fq_mid[l], fmu_mid[l], the node kernel writes fq_in[l+1], mu[l+1]; every activation is
// written whether or not forces are asked for, so the tangent pass and the training / Hessian backward read them afterwards.
// `records` = false (training, Hessian): full filter rows in two separate arrays W / dW, the layout the gradient kernels read.
int run_painn_fused(nb200_engine* eng, const nb200_painn_weights* w, const Workspace& ws, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol,
                    int N, int32_t e_cap, float* energy, float* forces, int32_t* status, cudaStream_t s, bool records, int bf16) {
    const int L = w->n_layers, F = NB_F;
    const int w_stride = (forces && records) ? 6 * F : 3 * F;    // [W | dW/dd] records when the backward runs
    const size_t wl_stride = (size_t)e_cap * w_stride;
    const float* dW0 = records ? ws.W + 3 * F : ws.dW;
    { Scope sc(eng, s, CAT_EMBED, 1); NB_TRY(nb_embed(z, w->emb, w->z_offset, w->n_elem, N, ws.fq_in[0], ws.mu[0], status, s)); }
    { Scope sc(eng, s, CAT_GEMM, 1); NB_TRY(nb_fused_prep(w, ws.wtiles, s)); }
    NbFusedFwd f{};
    f.n_atoms = N; f.n_layers = L; f.wtiles = ws.wtiles; f.eps = w->epsilon; f.ro_pre = ws.ro_pre;
    {   // message MLP of layer 0 on the embedding
        f.layer_upd = -1; f.layer_mlp = 0; f.readout = 0;
        f.q_mlp_in = ws.fq_in[0]; f.c1 = w->c1; f.h1pre = ws.h1pre[0]; f.xh = ws.xh[0];
        Scope sc(eng, s, CAT_GEMM, 1);
        NB_TRY(nb_fused_node_fwd(f, s));
    }
    for (int l = 0; l < L; ++l) {
        { Scope sc(eng, s, CAT_MSG_FWD, 1);
        NB_TRY(nb_painn_msg_fwd_ex(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.fq_in[l], ws.mu[l], ws.W + l * wl_stride, w_stride, ws.rev, ws.geom,
                                   ws.row_ptr, ws.col, N, ws.fq_mid[l], ws.fmu_mid[l], s, bf16)); }
        const bool last = l + 1 == L;
        f.layer_upd = l; f.layer_mlp = last ? -1 : l + 1; f.readout = last ? 1 : 0;
        f.q_mid = ws.fq_mid[l]; f.mu_mid = ws.fmu_mid[l]; f.d1 = w->d1 + (size_t)l * F; f.d2 = w->d2 + (size_t)l * 3 * F;
        f.VW = ws.VW[l]; f.nrm = ws.nrm[l]; f.dot = ws.fdot[l]; f.g1pre = ws.g1pre[l]; f.y = ws.y[l]; f.q_next = ws.fq_in[l + 1]; f.mu_next = ws.mu[l + 1];
        f.q_mlp_in = nullptr;
        if (!last) { f.c1 = w->c1 + (size_t)(l + 1) * F; f.h1pre = ws.h1pre[l + 1]; f.xh = ws.xh[l + 1]; }
        Scope sc(eng, s, CAT_GEMM, 1);
        NB_TRY(nb_fused_node_fwd(f, s));
    }
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_readout(ws.ro_pre, w->e1, w->R2, w->e2, N, F / 2, ws.eps, s)); }
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_mol_sum(ws.eps, mol_ptr, n_mol, w->energy_shift_per_atom, energy, s)); }
    if (!forces) { Scope sc(eng, s, CAT_READOUT, 1); return nb_poison_on_error(status, energy, n_mol, nullptr, 0, s); }

    if (cudaMemsetAsync(ws.egrad, 0, (size_t)e_cap * 4 * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    if (cudaMemsetAsync(ws.gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    float *cur = ws.gmu_a, *other = ws.gmu_b;
    NbFusedBwd b{};
    b.n_atoms = N; b.n_layers = L; b.wtiles = ws.wtiles; b.gq_a = ws.gq; b.gq_b = ws.gq_b; b.gn = ws.fgn; b.gdot = ws.fgdot; b.ro_pre = ws.ro_pre; b.R2 = w->R2;
    b.g_xh = ws.gy;
    for (int l = L - 1; l >= 0; --l) {
        // readout backward (first pass) or message-MLP backward of layer l + 1, then the update backward of layer l
        b.readout = l == L - 1 ? 1 : 0; b.layer_mlp = l == L - 1 ? -1 : l + 1; b.layer_upd = l;
        b.cur = cur; b.h1pre = l == L - 1 ? nullptr : ws.h1pre[l + 1];
        b.y = ws.y[l]; b.VW = ws.VW[l]; b.nrm = ws.nrm[l]; b.dot = ws.fdot[l]; b.g1pre = ws.g1pre[l];
        { Scope sc(eng, s, CAT_GEMM, 1); NB_TRY(nb_fused_node_bwd(b, s)); }
        { Scope sc(eng, s, CAT_MSG_BWD, 1);
        NB_TRY(nb_painn_msg_bwd_ex(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.W + l * wl_stride, dW0 + l * wl_stride, w_stride,
                                   ws.rev, ws.geom, ws.row_ptr, ws.col, N, ws.gq, cur, ws.gy, other, ws.egrad, s, bf16)); }
        float* t = cur; cur = other; other = t;
        // layer 0: the embedding does not depend on positions, nothing below the message kernel is needed for forces
    }
    { Scope sc(eng, s, CAT_FORCE, 2); NB_TRY(nb200_edge_forces(ws.egrad, ws.geom, ws.row_ptr, ws.rev, N, forces, s));
      NB_TRY(nb_poison_on_error(status, energy, n_mol, forces, (int64_t)3 * N, s)); }
    return NB200_OK;
}

// Tangent forward along the position-space direction v (painn_tangent.cu): the directional derivative of every saved activation of the fused
// forward (weights carry no tangent).  The message and the update add to t_q and t_mu[l + 1] in place; `keep_inputs` keeps the values the
// Linear layers saw (t_q_in, t_q_mid, t_mu_mid) for the weight gradients of the training step -- the Hessian does not read them.
// The caller opens the timing scope (1 + 6 L own launches besides the GEMMs).
int tangent_fwd(nb200_engine* eng, const nb200_painn_weights* w, const Workspace& ws, const float* v, int N, int32_t e_cap, int bf16, bool keep_inputs,
                cudaStream_t s) {
    const int L = w->n_layers, F = NB_F;
    const size_t wl = (size_t)e_cap * 3 * F;
    NB_TRY(nb_geom_tan(ws.geom, ws.row_ptr, ws.col, v, N, ws.t_geom, s));
    if (cudaMemsetAsync(ws.t_q, 0, (size_t)N * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();        // embedding: no tangent
    if (cudaMemsetAsync(ws.t_mu[0], 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    for (int l = 0; l < L; ++l) {
        const float* A1 = w->A1 + (size_t)l * F * F;
        const float* A2 = w->A2 + (size_t)l * 3 * F * F;
        const float* U = w->U + (size_t)l * 2 * F * F;
        const float* B1 = w->B1 + (size_t)l * F * 2 * F;
        const float* B2 = w->B2 + (size_t)l * 3 * F * F;
        if (keep_inputs && cudaMemcpyAsync(ws.t_q_in[l], ws.t_q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
            return nb_check_launch();
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_q, F, A1, F, ws.t_h1[l], F, false, nullptr, nullptr));
        NB_TRY(nb_mul_dact(ws.h1pre[l], ws.t_h1[l], (int64_t)N * F, ws.t_act, s));
        NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.t_act, F, A2, F, ws.t_xh[l], 3 * F, false, nullptr, nullptr));
        NB_TRY(nb_msg_fwd_tan(ws.xh[l], ws.t_xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.t_mu[l], ws.W + l * wl, ws.dW + l * wl, ws.geom,
                              ws.t_geom, ws.row_ptr, ws.col, N, ws.t_q, ws.t_mu[l + 1], s, bf16, ws.rev));
        if (keep_inputs && (cudaMemcpyAsync(ws.t_q_mid[l], ws.t_q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
                            cudaMemcpyAsync(ws.t_mu_mid[l], ws.t_mu[l + 1], (size_t)N * 3 * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess))
            return nb_check_launch();
        NB_TRY(linear_fwd(eng, s, 3 * N, 2 * F, F, ws.t_mu[l + 1], F, U, F, ws.t_VW[l], 2 * F, false, nullptr, nullptr));
        NB_TRY(nb_upd_norm_tan(ws.VW[l], ws.t_VW[l], ws.nrm[l], N, ws.t_nrm[l], s));
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_q, F, B1, 2 * F, ws.t_g1[l], F, false, nullptr, nullptr));
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_nrm[l], F, B1 + F, 2 * F, ws.t_g1[l], F, true, nullptr, nullptr));
        NB_TRY(nb_mul_dact(ws.g1pre[l], ws.t_g1[l], (int64_t)N * F, ws.t_act, s));
        NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.t_act, F, B2, F, ws.t_y[l], 3 * F, false, nullptr, nullptr));
        NB_TRY(nb_upd_combine_tan(ws.t_q, ws.t_mu[l + 1], ws.VW[l], ws.t_VW[l], ws.y[l], ws.t_y[l], N, s));
    }
    return linear_fwd(eng, s, N, F / 2, F, ws.t_q, F, w->R1, F, ws.t_ro, F / 2, false, nullptr, nullptr);
}

// Training backward (painn_train.cu) from the activations the fused forward kept: d(sum_m seed_m E_m)/d(weights) -- and with a tangent pass
// (`tan`) the force-seed term -- into the arrays `grads` points to (same layout as the weights; overwritten).  With `forces` it also returns
// the true, unweighted -dE/dR of the same backward and poisons energy / forces on a device error.
int train_bwd(nb200_engine* eng, const nb200_painn_weights* w, const Workspace& ws, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol, int N,
              int32_t e_cap, const float* seed_mol, const nb200_painn_weights* grads, bool tan, float* energy, float* forces, int32_t* status,
              cudaStream_t s) {
    const int L = w->n_layers, F = NB_F, K = w->n_rbf;
    const size_t wl_stride = (size_t)e_cap * 3 * F;
    const int bf16 = eng->edge_bf16;
    const float* q_out = ws.fq_in[L];  // input of the readout
    // ---- analytic backward: forces = -dE/dR with dE/dE_m = 1 (painn.py:135-146)
    if (cudaMemsetAsync(ws.egrad, 0, (size_t)e_cap * 4 * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    if (cudaMemsetAsync(ws.gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_readout_bwd(ws.ro_pre, w->R2, N, F / 2, ws.g_ro, s)); }
    NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.g_ro, F / 2, w->R1, F, ws.gq, F, false));
    // energy-seed weight gradients: dW += (c o g)^T x and dbias += colsum(c o g), c = the per-atom seed (`rs_div` rows of g per atom: 3 for the
    // (atom, xyz) rows of U).  One wgmma split-K launch (wgrad_tc.cu: the row scale is applied while loading g).
    // Weight-gradient launches are LEAVES of the step: they read buffers of the backward chain and only add into `grads`.  They run on a
    // second stream of the engine, next to the chain (whose 76-CTA GEMMs and latency-bound steps leave SMs idle): fork = the side stream
    // waits for the chain's current point, and the chain waits for a leaf only right before it overwrites that leaf's inputs (`need`).  The
    // side stream is in order, so one event per input group is enough.
    bool use_side = true;
    if (!eng->side && cudaStreamCreateWithFlags(&eng->side, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); use_side = false; }
    const cudaStream_t ls = use_side ? eng->side : s;
    size_t ev_next = 0;
    auto ev_get = [&]() -> cudaEvent_t {
        if (ev_next == eng->side_ev.size()) {
            cudaEvent_t e = nullptr;
            if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
            eng->side_ev.push_back(e);
        }
        return eng->side_ev[ev_next++];
    };
    auto fork = [&]() {  // the leaves launched next see everything the chain has enqueued so far
        if (!use_side) return;
        if (cudaEvent_t e = ev_get()) { cudaEventRecord(e, s); cudaStreamWaitEvent(eng->side, e, 0); }
    };
    cudaEvent_t d_R = nullptr, d_B2 = nullptr, d_B1 = nullptr, d_U = nullptr, d_F = nullptr, d_A2 = nullptr, d_A1 = nullptr;
    cudaEvent_t* tag = &d_R;  // which input group the leaves launched next belong to
    auto leaf_done = [&]() {
        if (!use_side) return;
        if (cudaEvent_t e = ev_get()) { cudaEventRecord(e, eng->side); *tag = e; }
    };
    auto need = [&](cudaEvent_t& e) {  // the chain is about to overwrite what those leaves read
        if (e) { cudaStreamWaitEvent(s, e, 0); e = nullptr; }
    };
    struct Join {  // every exit path: the caller's stream waits for the side stream
        nb200_engine* eng; cudaStream_t s; bool on;
        ~Join() {
            if (!on) return;
            cudaEvent_t e = nullptr;
            if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) == cudaSuccess) { cudaEventRecord(e, eng->side); cudaStreamWaitEvent(s, e, 0); cudaEventDestroy(e); }
        }
    } join{eng, s, use_side};
    // Every PaiNN shape fits the kernel (n_feat == NB_F; workspace and gradient arrays 16-byte aligned, see grads_ok).
    // With a force seed the energy-seed term rides in the tangent call of the same Linear (one 3-term launch, wgrad_tc.cu::nb_wgrad_tc3).
    auto wg_primal = [&](int M, int out, int in, const float* g, int ldg, const float* x, int ldx, float* dW, int lddw, float* dbias, int rs_div) -> int {
        if (tan) return NB200_OK;
        if (!nb_wgrad_tc_ok(M, out, in, g, ldg, x, ldx, dW, lddw)) return NB200_EUNSUPPORTED;
        fork();
        const int rc = nb_wgrad_tc(M, out, in, g, x, nullptr, nullptr, ldg, ldx, dW, lddw, 1.0f, dbias, 1.0f, 0, ws.seed_atom, rs_div, ls);
        leaf_done();
        return rc;
    };
    {
        Scope sc(eng, s, CAT_NODE, 8);
        NB_TRY(nb_seed_atom(seed_mol, mol_ptr, n_mol, ws.seed_atom, s));
        // every gradient array starts at zero: the energy-seed terms and the force-seed (tangent) terms both ACCUMULATE into it
        const struct { const float* p; size_t n; } zero[] = {
            {grads->w_rbf, (size_t)L * K * 3 * F}, {grads->b_rbf, (size_t)L * 3 * F}, {grads->emb, (size_t)w->n_elem * F},
            {grads->A1, (size_t)L * F * F}, {grads->c1, (size_t)L * F}, {grads->A2, (size_t)L * 3 * F * F}, {grads->c2, (size_t)L * 3 * F},
            {grads->U, (size_t)L * 2 * F * F}, {grads->B1, (size_t)L * F * 2 * F}, {grads->d1, (size_t)L * F}, {grads->B2, (size_t)L * 3 * F * F},
            {grads->d2, (size_t)L * 3 * F}, {grads->R1, (size_t)(F / 2) * F}, {grads->e1, (size_t)F / 2}, {grads->R2, (size_t)F / 2}, {grads->e2, 1}};
        for (const auto& zr : zero)
            if (cudaMemsetAsync(const_cast<float*>(zr.p), 0, zr.n * sizeof(float), s) != cudaSuccess) return nb_check_launch();
        NB_TRY(nb_act_only(ws.ro_pre, ws.seed_atom, N, F / 2, NB_ACT_SILU, ws.act_t, s));                    // c_i silu(pre_i)
        NB_TRY(nb_colsum(ws.act_t, N, F / 2, const_cast<float*>(grads->R2), s, 1.0f, 1));
        NB_TRY(nb_colsum(ws.seed_atom, N, 1, const_cast<float*>(grads->e2), s, 1.0f, 1));
        NB_TRY(wg_primal(N, F / 2, F, ws.g_ro, F / 2, q_out, F, const_cast<float*>(grads->R1), F, const_cast<float*>(grads->e1), 1));
    }
    // tangent weight gradients enter with sign -1:  d/dtheta sum_i v_i.F_i = -(v.d/dR) dE_tot/dtheta   (seed 1, not the energy seed)
    // One launch: (c o g)^T x - tg^T x - g^T tx and the bias sums.
    auto wgrad_tan = [&](int M, int out, int in, const float* g, const float* tg, int ldg, const float* x, const float* tx, int ldx, float* dW,
                         int lddw, float* dbias = nullptr, int rs_div = 1) -> int {
        if (!nb_wgrad_tc_ok(M, out, in, g, ldg, x, ldx, dW, lddw)) return NB200_EUNSUPPORTED;
        fork();
        const int rc = nb_wgrad_tc3(M, out, in, g, tg, ldg, x, tx, ldx, dW, lddw, dbias, ws.seed_atom, rs_div, ls);
        leaf_done();
        return rc;
    };
    if (tan) {
        Scope sc(eng, s, CAT_NODE, 4);
        if (cudaMemsetAsync(ws.t_gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
        NB_TRY(nb_readout_bwd_tan(ws.ro_pre, ws.t_ro, w->R2, N, F / 2, ws.t_g_ro, ws.t_act, s));  // t_act [N, F/2] = silu'(pre) pre^
        NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.t_g_ro, F / 2, w->R1, F, ws.t_gq, F, false));
        NB_TRY(nb_colsum(ws.t_act, N, F / 2, const_cast<float*>(grads->R2), s, -1.0f, 1));
        NB_TRY(wgrad_tan(N, F / 2, F, ws.g_ro, ws.t_g_ro, F / 2, q_out, ws.t_q, F, const_cast<float*>(grads->R1), F, const_cast<float*>(grads->e1)));
    }
    float *t_cur = ws.t_gmu_a, *t_other = ws.t_gmu_b;
    float *cur = ws.gmu_a, *other = ws.gmu_b;
    const int PT = tan ? 2 : 1;  // with a tangent pass every Linear backward runs once on the stacked rows [primal ; tangent] (carve: adjacent pairs)
    for (int l = L - 1; l >= 0; --l) {
        const float* A1 = w->A1 + (size_t)l * F * F;
        const float* A2 = w->A2 + (size_t)l * 3 * F * F;
        const float* U = w->U + (size_t)l * 2 * F * F;
        const float* B1 = w->B1 + (size_t)l * F * 2 * F;
        const float* B2 = w->B2 + (size_t)l * 3 * F * F;
        // update backward
        need(d_A2); need(d_U);  // the leaves of the layer above read gy / act_t (dA2) and gVW (dU)
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_upd_combine_bwd(ws.gq, cur, ws.y[l], ws.VW[l], N, ws.gy, ws.gVW, s)); }
        tag = &d_B2;
        {   // dB2, dd2
            Scope sc(eng, s, CAT_NODE, 3);
            NB_TRY(nb_act_only(ws.g1pre[l], nullptr, N, F, NB_ACT_SILU, ws.act_t, s));
            NB_TRY(wg_primal(N, 3 * F, F, ws.gy, 3 * F, ws.act_t, F, const_cast<float*>(grads->B2) + (size_t)l * 3 * F * F, F,
                             const_cast<float*>(grads->d2) + (size_t)l * 3 * F, 1));
        }
        if (tan) {  // update backward, tangent: combine, dB2^, dd2^
            Scope sc(eng, s, CAT_NODE, 3);
            NB_TRY(nb_upd_combine_bwd_tan(ws.gq, ws.t_gq, cur, t_cur, ws.y[l], ws.t_y[l], ws.VW[l], ws.t_VW[l], N, ws.t_gy, ws.t_gVW, s));
            NB_TRY(nb_mul_dact(ws.g1pre[l], ws.t_g1[l], (int64_t)N * F, ws.t_act, s));  // act2^ ; act_t still holds act2 = silu(g1pre)
            NB_TRY(wgrad_tan(N, 3 * F, F, ws.gy, ws.t_gy, 3 * F, ws.act_t, ws.t_act, F, const_cast<float*>(grads->B2) + (size_t)l * 3 * F * F, F,
                             const_cast<float*>(grads->d2) + (size_t)l * 3 * F));
        }
        need(d_A1);  // dA1 of the layer above read gt
        NB_TRY(linear_bwd(eng, s, PT * N, 3 * F, F, ws.gy, 3 * F, B2, F, ws.gt, F, false));   // [gy ; gy^] -> [gt ; gt^]
        tag = &d_B1;
        if (tan) {
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(nb_act_bwd_tan(ws.t_gt, ws.gt, ws.g1pre[l], ws.t_g1[l], (int64_t)N * F, s));  // needs gt BEFORE the primal act_bwd
        }
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_act_bwd(ws.gt, ws.g1pre[l], (int64_t)N * F, NB_ACT_SILU, s)); }
        if (tan) {  // dB1^, dd1^
            Scope sc(eng, s, CAT_NODE, 1);
            float* gB1 = const_cast<float*>(grads->B1) + (size_t)l * F * 2 * F;
            NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.fq_mid[l], ws.t_q_mid[l], F, gB1, 2 * F, const_cast<float*>(grads->d1) + (size_t)l * F));
            NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.nrm[l], ws.t_nrm[l], F, gB1 + F, 2 * F));
        }
        {   // dB1 = [gt^T q_mid | gt^T nrm], dd1
            Scope sc(eng, s, CAT_NODE, 2);
            float* gB1 = const_cast<float*>(grads->B1) + (size_t)l * F * 2 * F;
            NB_TRY(wg_primal(N, F, F, ws.gt, F, ws.fq_mid[l], F, gB1, 2 * F, const_cast<float*>(grads->d1) + (size_t)l * F, 1));
            NB_TRY(wg_primal(N, F, F, ws.gt, F, ws.nrm[l], F, gB1 + F, 2 * F, nullptr, 1));
        }
        NB_TRY(linear_bwd(eng, s, PT * N, F, F, ws.gt, F, B1, 2 * F, ws.gq, F, true));
        NB_TRY(linear_bwd(eng, s, PT * N, F, F, ws.gt, F, B1 + F, 2 * F, ws.gn, F, false));
        if (tan) {
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(nb_upd_norm_bwd_tan(ws.gn, ws.t_gn, ws.VW[l], ws.t_VW[l], ws.nrm[l], ws.t_nrm[l], N, ws.t_gVW, s));
        }
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_upd_norm_bwd(ws.gn, ws.VW[l], ws.nrm[l], N, ws.gVW, s)); }
        tag = &d_U;
        if (tan) {  // dU^ ; then the tangent of the gradient w.r.t. the post-message mu
            NB_TRY(wgrad_tan(3 * N, 2 * F, F, ws.gVW, ws.t_gVW, 2 * F, ws.fmu_mid[l], ws.t_mu_mid[l], F, const_cast<float*>(grads->U) + (size_t)l * 2 * F * F, F,
                             nullptr, 3));
        }
        {   // dU over the 3N (atom, xyz) rows
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(wg_primal(3 * N, 2 * F, F, ws.gVW, 2 * F, ws.fmu_mid[l], F, const_cast<float*>(grads->U) + (size_t)l * 2 * F * F, F, nullptr, 3));
        }
        NB_TRY(linear_bwd(eng, s, PT * 3 * N, 2 * F, F, ws.gVW, 2 * F, U, F, cur, F, true));  // (cur, t_cur) = (gmu_a, t_gmu_a) or (gmu_b, t_gmu_b): adjacent
        // message backward (by source atom; uses edge symmetry)
        need(d_B2); need(d_F);  // it overwrites gy (read by dB2) and the per-edge filter gradients (read by the filter leaves of the layer above)
        { Scope sc(eng, s, CAT_MSG_BWD, 1);
        NB_TRY(nb_painn_msg_bwd_train(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride, ws.geom,
                                      ws.row_ptr, ws.col, N, ws.gq, cur, ws.gy, other, ws.egrad, ws.gW, ws.seed_atom, s, bf16, ws.rev)); }
        if (tan) {  // message backward tangent reads the same gq / cur the primal call just read; its outputs go to the t_ twins
            Scope sc(eng, s, CAT_NODE, 2);
            NB_TRY(nb_msg_bwd_tan(ws.xh[l], ws.t_xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.t_mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride,
                                  ws.geom, ws.t_geom, ws.row_ptr, ws.col, N, ws.gq, ws.t_gq, cur, t_cur, ws.t_gy, t_other, ws.t_gW, ws.gWd, s, bf16, ws.rev));
            tag = &d_F; fork();
            NB_TRY(nb_filter_wgrad_tan(ws.geom, ws.t_geom, status, ws.sort_scr2, w->rbf_offsets, K, w->radial_mode, w->cutoff, w->rbf_coeff, w->rbf_xscale,
                                       ws.t_gW, ws.gWd, -1.0f, const_cast<float*>(grads->w_rbf) + (size_t)l * K * 3 * F,
                                       const_cast<float*>(grads->b_rbf) + (size_t)l * 3 * F, ls, e_cap, bf16));
            leaf_done();
            float* tt = t_cur; t_cur = t_other; t_other = tt;
        }
        float* t = cur; cur = other; other = t;
        {   // filter weights of this layer, then dA2, dc2
            Scope sc(eng, s, CAT_NODE, 4);
            tag = &d_F; fork();
            NB_TRY(nb_filter_wgrad(ws.geom, status, ws.sort_scr2, w->rbf_offsets, K, w->radial_mode, w->cutoff, w->rbf_coeff, w->rbf_xscale, ws.gW,
                                   const_cast<float*>(grads->w_rbf) + (size_t)l * K * 3 * F, const_cast<float*>(grads->b_rbf) + (size_t)l * 3 * F, ls, e_cap, bf16));
            leaf_done();
            tag = &d_A2;
            NB_TRY(nb_act_only(ws.h1pre[l], nullptr, N, F, NB_ACT_SILU, ws.act_t, s));
            NB_TRY(wg_primal(N, 3 * F, F, ws.gy, 3 * F, ws.act_t, F, const_cast<float*>(grads->A2) + (size_t)l * 3 * F * F, F,
                             const_cast<float*>(grads->c2) + (size_t)l * 3 * F, 1));
        }
        if (tan) {  // dA2^, dc2^  (act_t holds act1 = silu(h1pre) from the block above)
            Scope sc(eng, s, CAT_NODE, 2);
            NB_TRY(nb_mul_dact(ws.h1pre[l], ws.t_h1[l], (int64_t)N * F, ws.t_act, s));
            NB_TRY(wgrad_tan(N, 3 * F, F, ws.gy, ws.t_gy, 3 * F, ws.act_t, ws.t_act, F, const_cast<float*>(grads->A2) + (size_t)l * 3 * F * F, F,
                             const_cast<float*>(grads->c2) + (size_t)l * 3 * F));
        }
        // message MLP backward, through layer 0: the embedding gradient needs dE/dq of the embedding
        need(d_B1);  // dB1 read gt
        NB_TRY(linear_bwd(eng, s, PT * N, 3 * F, F, ws.gy, 3 * F, A2, F, ws.gt, F, false));
        tag = &d_A1;
        if (tan) {
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(nb_act_bwd_tan(ws.t_gt, ws.gt, ws.h1pre[l], ws.t_h1[l], (int64_t)N * F, s));
        }
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_act_bwd(ws.gt, ws.h1pre[l], (int64_t)N * F, NB_ACT_SILU, s)); }
        if (tan) {  // dA1^, dc1^
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.fq_in[l], ws.t_q_in[l], F, const_cast<float*>(grads->A1) + (size_t)l * F * F, F,
                             const_cast<float*>(grads->c1) + (size_t)l * F));
        }
        {   // dA1, dc1
            Scope sc(eng, s, CAT_NODE, 2);
            NB_TRY(wg_primal(N, F, F, ws.gt, F, ws.fq_in[l], F, const_cast<float*>(grads->A1) + (size_t)l * F * F, F,
                             const_cast<float*>(grads->c1) + (size_t)l * F, 1));
        }
        NB_TRY(linear_bwd(eng, s, PT * N, F, F, ws.gt, F, A1, F, ws.gq, F, true));
    }
    { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_emb_grad(ws.gq, ws.seed_atom, z, w->z_offset, w->n_elem, N, const_cast<float*>(grads->emb), s)); }
    if (tan) { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_emb_grad(ws.t_gq, nullptr, z, w->z_offset, w->n_elem, N, const_cast<float*>(grads->emb), s, -1.0f)); }
    if (!forces) return NB200_OK;
    { Scope sc(eng, s, CAT_FORCE, 2); NB_TRY(nb200_edge_forces(ws.egrad, ws.geom, ws.row_ptr, ws.rev, N, forces, s));
      NB_TRY(nb_poison_on_error(status, energy, n_mol, forces, (int64_t)3 * N, s)); }
    return NB200_OK;
}

}  // namespace

// Inference: graph + filters with half-row [W | dW/dd] records, then the fused forward (and force backward).
extern "C" int nb200_painn_energy_forces(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos,
                                         const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace,
                                         int64_t workspace_bytes, float* energy, float* forces, int32_t* status, void* stream) {
    if (!pos || !energy) return NB200_EINVAL;
    NB_TRY(args_ok(eng, w, z, mol_ptr, n_mol, n_atoms, e_cap, workspace, status));
    const Workspace ws = carve(workspace, w->n_layers, NB_F, n_mol, n_atoms, e_cap, forces != nullptr);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    const cudaStream_t s = (cudaStream_t)stream;
    NB_TRY(graph_and_filters(eng, w, ws, pos, mol_ptr, n_mol, n_atoms, e_cap, status, s, forces != nullptr, false));
    return run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, n_atoms, e_cap, energy, forces, status, s, true, 0);
}

extern "C" int64_t nb200_painn_train_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap,
                                                     int32_t with_force_seed) {
    if (!w || w->n_layers <= 0 || w->n_layers > kMaxLayers || w->n_feat != NB_F || b_cap < 0 || n_cap < 0 || e_cap < 0) return NB200_EINVAL;
    return carve(nullptr, w->n_layers, w->n_feat, b_cap, n_cap, e_cap, true, true, with_force_seed != 0).bytes;
}

// Training step in two calls on one training workspace (sized by nb200_painn_train_workspace_bytes with the SAME with_force_seed flag for
// both): the forward + forces first, the parameter gradients once the loss has produced the seeds.  Nothing else may use the workspace in
// between; weights, z, mol_ptr, n_* and e_cap must be those of the forward call.
// Forward: graph + training filters + the directed-edge bin sort, then the fused forward with forces; every activation the backward reads
// stays in the workspace.
extern "C" int nb200_painn_train_forward(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                         int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes,
                                         int32_t with_force_seed, float* energy, float* forces, int32_t* status, void* stream) {
    if (!pos || !energy || !forces) return NB200_EINVAL;
    NB_TRY(args_ok(eng, w, z, mol_ptr, n_mol, n_atoms, e_cap, workspace, status));
    const Workspace ws = carve(workspace, w->n_layers, NB_F, n_mol, n_atoms, e_cap, true, true, with_force_seed != 0);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    const cudaStream_t s = (cudaStream_t)stream;
    NB_TRY(graph_and_filters(eng, w, ws, pos, mol_ptr, n_mol, n_atoms, e_cap, status, s, false, true));
    return run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, n_atoms, e_cap, energy, forces, status, s, false, eng->edge_bf16);
}

// Backward: the tangent forward if there is a force seed, then the training backward (energies / forces were returned, and poisoned on
// error, by the forward call).
extern "C" int nb200_painn_train_backward(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol,
                                          int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes, int32_t with_force_seed,
                                          const float* energy_seed, const float* force_seed, const nb200_painn_weights* grads, int32_t* status,
                                          void* stream) {
    if (!grads_ok(grads) || (force_seed && !with_force_seed)) return NB200_EINVAL;
    NB_TRY(args_ok(eng, w, z, mol_ptr, n_mol, n_atoms, e_cap, workspace, status));
    const Workspace ws = carve(workspace, w->n_layers, NB_F, n_mol, n_atoms, e_cap, true, true, with_force_seed != 0);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    const cudaStream_t s = (cudaStream_t)stream;
    if (force_seed) {
        Scope sc(eng, s, CAT_NODE, 1 + 6 * w->n_layers);
        NB_TRY(tangent_fwd(eng, w, ws, force_seed, n_atoms, e_cap, eng->edge_bf16, true, s));
    }
    return train_bwd(eng, w, ws, z, mol_ptr, n_mol, n_atoms, e_cap, energy_seed, grads, force_seed != nullptr, nullptr, nullptr, status, s);
}

// The training step in one call: the forward of nb200_painn_train_forward without its force backward (the training backward produces the
// forces), then the tangent forward and the training backward.
extern "C" int nb200_painn_energy_forces_grads(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos,
                                               const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace,
                                               int64_t workspace_bytes, const float* energy_seed, const float* force_seed,
                                               const nb200_painn_weights* grads, float* energy, float* forces, int32_t* status, void* stream) {
    if (!pos || !energy || !forces || !grads_ok(grads)) return NB200_EINVAL;
    NB_TRY(args_ok(eng, w, z, mol_ptr, n_mol, n_atoms, e_cap, workspace, status));
    const bool tan = force_seed != nullptr;
    const Workspace ws = carve(workspace, w->n_layers, NB_F, n_mol, n_atoms, e_cap, true, true, tan);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    const cudaStream_t s = (cudaStream_t)stream;
    NB_TRY(graph_and_filters(eng, w, ws, pos, mol_ptr, n_mol, n_atoms, e_cap, status, s, false, true));
    NB_TRY(run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, n_atoms, e_cap, energy, nullptr, status, s, false, eng->edge_bf16));
    if (tan) {
        Scope sc(eng, s, CAT_NODE, 1 + 6 * w->n_layers);
        NB_TRY(tangent_fwd(eng, w, ws, force_seed, n_atoms, e_cap, eng->edge_bf16, true, s));
    }
    return train_bwd(eng, w, ws, z, mol_ptr, n_mol, n_atoms, e_cap, energy_seed, grads, tan, energy, forces, status, s);
}

// ---------------------------------------------------------------------------------------------
// Hessian-vector products H v = -dF/dR . v (DESIGN.md section 3.13): the primal forward (fused node kernels, activations kept, as the first
// call of the two-call training step) runs once; then, per direction, the tangent forward and the stacked [primal ; tangent] backward of
// the training step without any weight gradient, the message backward tangent also producing the tangent of the per-edge geometric
// gradient (t_egrad), and the tangent of the force assembly.  The workspace holds ONE direction's tangent arrays whatever n_dir is.
namespace {

int run_painn_hvp(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                  int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes, int32_t n_dir, const float* v, float* energy, float* forces,
                  float* hv, int32_t* status, void* stream) {
    if (!pos || !v || !energy || !hv || n_dir < 1) return NB200_EINVAL;
    NB_TRY(args_ok(eng, w, z, mol_ptr, n_mol, n_atoms, e_cap, workspace, status));
    const int L = w->n_layers, F = NB_F, K = w->n_rbf, N = n_atoms;
    Workspace ws = carve(workspace, L, F, n_mol, N, e_cap, true, false, true, true);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t wl = (size_t)e_cap * 3 * F;
    { Scope sc(eng, s, CAT_NBR, 3);
    NB_TRY(nb200_neighbor_build(pos, mol_ptr, n_mol, N, w->cutoff, w->max_neighbors, e_cap, ws.row_ptr, ws.col, ws.rev, ws.geom, ws.deg, status, s)); }
    // W, dW/dd and d2W/dd2: one row per undirected pair, three arrays
    { Scope sc(eng, s, CAT_FILTER, 4);
    NB_TRY(nb_painn_filter_d2(ws.geom, status, e_cap, w->w_rbf, w->b_rbf, L, K, w->radial_mode, w->cutoff, w->rbf_offsets, w->rbf_coeff, w->rbf_xscale, ws.W,
                              ws.dW, ws.d2W, ws.sort_scr, ws.rev, s)); }
    // energies (and forces) with every activation the tangent pass reads kept: layer inputs / post-message states in fq_in, fmu_mid
    NB_TRY(run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, N, e_cap, energy, forces, status, s, false, 0));

    for (int32_t dir = 0; dir < n_dir; ++dir) {
        // ---- tangent forward along v_dir.  With timing on, its CAT_MSG_FWD scope brackets the whole tangent forward, GEMMs included
        // (bench_hessian.py splits forward / backward with it).
        { Scope sc(eng, s, CAT_MSG_FWD, 1 + 6 * L); NB_TRY(tangent_fwd(eng, w, ws, v + (size_t)dir * 3 * N, N, e_cap, 0, false, s)); }
        // ---- backward, primal and tangent: every Linear backward on the stacked rows [g ; g^] (carve: adjacent pairs)
        if (cudaMemsetAsync(ws.egrad, 0, (size_t)e_cap * 4 * sizeof(float), s) != cudaSuccess ||
            cudaMemsetAsync(ws.t_egrad, 0, (size_t)e_cap * 4 * sizeof(float), s) != cudaSuccess ||
            cudaMemsetAsync(ws.gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess ||
            cudaMemsetAsync(ws.t_gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess)
            return nb_check_launch();
        { Scope sc(eng, s, CAT_READOUT, 2);
          NB_TRY(nb_readout_bwd(ws.ro_pre, w->R2, N, F / 2, ws.g_ro, s));
          NB_TRY(nb_readout_bwd_tan(ws.ro_pre, ws.t_ro, w->R2, N, F / 2, ws.t_g_ro, ws.t_act, s)); }
        NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.g_ro, F / 2, w->R1, F, ws.gq, F, false));
        NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.t_g_ro, F / 2, w->R1, F, ws.t_gq, F, false));
        float *cur = ws.gmu_a, *other = ws.gmu_b, *t_cur = ws.t_gmu_a, *t_other = ws.t_gmu_b;
        for (int l = L - 1; l >= 0; --l) {
            const float* A1 = w->A1 + (size_t)l * F * F;
            const float* A2 = w->A2 + (size_t)l * 3 * F * F;
            const float* U = w->U + (size_t)l * 2 * F * F;
            const float* B1 = w->B1 + (size_t)l * F * 2 * F;
            const float* B2 = w->B2 + (size_t)l * 3 * F * F;
            { Scope sc(eng, s, CAT_NODE, 2);
              NB_TRY(nb_upd_combine_bwd(ws.gq, cur, ws.y[l], ws.VW[l], N, ws.gy, ws.gVW, s));
              NB_TRY(nb_upd_combine_bwd_tan(ws.gq, ws.t_gq, cur, t_cur, ws.y[l], ws.t_y[l], ws.VW[l], ws.t_VW[l], N, ws.t_gy, ws.t_gVW, s)); }
            NB_TRY(linear_bwd(eng, s, 2 * N, 3 * F, F, ws.gy, 3 * F, B2, F, ws.gt, F, false));
            { Scope sc(eng, s, CAT_NODE, 2);
              NB_TRY(nb_act_bwd_tan(ws.t_gt, ws.gt, ws.g1pre[l], ws.t_g1[l], (int64_t)N * F, s));  // needs gt BEFORE the primal act_bwd
              NB_TRY(nb_act_bwd(ws.gt, ws.g1pre[l], (int64_t)N * F, NB_ACT_SILU, s)); }
            NB_TRY(linear_bwd(eng, s, 2 * N, F, F, ws.gt, F, B1, 2 * F, ws.gq, F, true));
            NB_TRY(linear_bwd(eng, s, 2 * N, F, F, ws.gt, F, B1 + F, 2 * F, ws.gn, F, false));
            { Scope sc(eng, s, CAT_NODE, 2);
              NB_TRY(nb_upd_norm_bwd_tan(ws.gn, ws.t_gn, ws.VW[l], ws.t_VW[l], ws.nrm[l], ws.t_nrm[l], N, ws.t_gVW, s));
              NB_TRY(nb_upd_norm_bwd(ws.gn, ws.VW[l], ws.nrm[l], N, ws.gVW, s)); }
            NB_TRY(linear_bwd(eng, s, 2 * 3 * N, 2 * F, F, ws.gVW, 2 * F, U, F, cur, F, true));  // (cur, t_cur) adjacent
            // message backward of EVERY layer (egrad and its tangent collect contributions from all of them)
            { Scope sc(eng, s, CAT_MSG_BWD, 2);
              NB_TRY(nb_painn_msg_bwd_ex(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.W + l * wl, ws.dW + l * wl, 3 * F, ws.rev, ws.geom, ws.row_ptr, ws.col,
                                         N, ws.gq, cur, ws.gy, other, ws.egrad, s, 0));
              NB_TRY(nb_msg_bwd_hvp(ws.xh[l], ws.t_xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.t_mu[l], ws.W + l * wl, ws.dW + l * wl, ws.d2W + l * wl,
                                    ws.geom, ws.t_geom, ws.row_ptr, ws.col, ws.rev, N, ws.gq, ws.t_gq, cur, t_cur, ws.t_gy, t_other, ws.t_egrad, s)); }
            std::swap(cur, other); std::swap(t_cur, t_other);
            if (l == 0) break;  // the embedding does not depend on positions
            NB_TRY(linear_bwd(eng, s, 2 * N, 3 * F, F, ws.gy, 3 * F, A2, F, ws.gt, F, false));
            { Scope sc(eng, s, CAT_NODE, 2);
              NB_TRY(nb_act_bwd_tan(ws.t_gt, ws.gt, ws.h1pre[l], ws.t_h1[l], (int64_t)N * F, s));
              NB_TRY(nb_act_bwd(ws.gt, ws.h1pre[l], (int64_t)N * F, NB_ACT_SILU, s)); }
            NB_TRY(linear_bwd(eng, s, 2 * N, F, F, ws.gt, F, A1, F, ws.gq, F, true));
        }
        { Scope sc(eng, s, CAT_FORCE, 1);
          NB_TRY(nb_edge_forces_hvp(ws.egrad, ws.t_egrad, ws.geom, ws.t_geom, ws.row_ptr, ws.rev, N, hv + (size_t)dir * 3 * N, s)); }
    }
    { Scope sc(eng, s, CAT_FORCE, 1); NB_TRY(nb_poison_on_error(status, energy, 0, hv, (int64_t)n_dir * 3 * N, s)); }
    return NB200_OK;
}

}  // namespace

extern "C" int64_t nb200_painn_hvp_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap, int32_t n_dir) {
    if (!w || w->n_layers <= 0 || w->n_layers > kMaxLayers || w->n_feat != NB_F || b_cap < 0 || n_cap < 0 || e_cap < 0 || n_dir < 1) return NB200_EINVAL;
    return carve(nullptr, w->n_layers, w->n_feat, b_cap, n_cap, e_cap, true, false, true, true).bytes;
}

extern "C" int nb200_painn_hvp(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                               int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes, int32_t n_dir, const float* v,
                               float* energy, float* forces, float* hv, int32_t* status, void* stream) {
    return run_painn_hvp(eng, w, z, pos, mol_ptr, n_mol, n_atoms, e_cap, workspace, workspace_bytes, n_dir, v, energy, forces, hv, status, stream);
}
