// engine.cu -- whole-model PaiNN energy + analytic forces for one batch of conformations.
//
// Replaces `NeuralNetworkPotential.forward` as configured by config/model/painn.yaml
// (PairwiseDistances -> PaiNN -> Atomwise -> Forces -> AddOffsets; SURVEY.md section 3.1) and
// `PaiNN.forward` of nablaDFT/painn_pyg/painn.py:89-148 (config/model/painn-oc.yaml).
// The reference obtains forces with torch.autograd.grad through ~40 eager ops per layer;
// here the backward is hand-derived and runs as the mirrored kernel sequence on one stream,
// with no host synchronisation anywhere (edge count and error flags stay on the device).
//
// Node-level dense layers ([N,128]x[128,384] etc.) run on the wgmma 3xTF32 GEMM of gemm_tc.cu (fp32-accurate: the reference never
// uses reduced precision, SURVEY.md section 0.9); cuBLAS SGEMM stays selectable for A/B runs (nb200_engine_set_gemm_backend) and carries
// the weight-gradient GEMMs of the training step (reduction over the atom rows: a plain library GEMM).
// `run_painn` is the one orchestration for inference, the energy-seeded parameter gradients (painn_train.cu) and the force-loss tangent
// pass (painn_tangent.cu).
#include <new>

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

extern "C" int nb200_engine_set_gemm_backend(nb200_engine* eng, int32_t backend) {
    if (!eng || (backend != 0 && backend != 1)) return NB200_EINVAL;
    eng->gemm_backend = backend;
    return NB200_OK;
}

extern "C" int nb200_engine_set_node_backend(nb200_engine* eng, int32_t backend) {
    if (!eng || (backend != 0 && backend != 1)) return NB200_EINVAL;
    eng->node_backend = backend;
    return NB200_OK;
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
    float *q, *act, *ro_pre, *eps;
    // backward
    float *gq, *gmu_a, *gmu_b, *gy, *gVW, *gt, *gn, *g_ro, *egrad;
    // training only: layer inputs that the in-place forward overwrites, scaled-gradient / activation scratch, per-edge filter gradients
    float *q_in[kMaxLayers], *q_mid[kMaxLayers], *mu_mid[kMaxLayers], *gs, *act_t, *gW, *seed_atom;
    // force-loss tangent pass (painn_tangent.cu): t_X = directional derivative of X along the position-space direction v
    float *t_geom, *t_h1[kMaxLayers], *t_xh[kMaxLayers], *t_VW[kMaxLayers], *t_nrm[kMaxLayers], *t_g1[kMaxLayers], *t_y[kMaxLayers];
    float *t_q_in[kMaxLayers], *t_q_mid[kMaxLayers], *t_mu_mid[kMaxLayers], *t_mu[kMaxLayers + 1];
    float *t_q, *t_act, *t_ro, *t_gq, *t_gmu_a, *t_gmu_b, *t_gy, *t_gVW, *t_gt, *t_gn, *t_g_ro, *t_gW, *gWd;
    // fused node path (painn_fused.cu): per-layer inputs / post-message states instead of in-place q, mu; prepared weight tiles
    float *fq_in[kMaxLayers + 1], *fq_mid[kMaxLayers], *fmu_mid[kMaxLayers], *fdot[kMaxLayers], *gq_b, *fgn, *fgdot;
    void* wtiles;
    void* blas_ws;
    int64_t bytes;
};

Workspace carve(void* p, int L, int F, int64_t B, int64_t N, int64_t E, bool forces, bool train = false, bool tangent = false) {
    (void)B;
    Workspace w{};
    Carver c(p);
    w.row_ptr = c.take<int32_t>(N + 1);
    w.col = c.take<int32_t>(E);
    w.rev = c.take<int32_t>(E);
    w.deg = c.take<int32_t>(N);
    w.sort_scr = c.take<int32_t>(E + 1024);
    w.geom = c.take<float>(4 * E);
    // filters: [L][E][3F] W and the same for dW/dd (adjacent), or -- fused inference path -- ONE array [L][E][6F] of [W | dW/dd] records over
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
    w.q = c.take<float>(N * F);
    w.act = c.take<float>(N * F);
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
        for (int l = 0; l < L; ++l) { w.q_in[l] = c.take<float>(N * F); w.q_mid[l] = c.take<float>(N * F); w.mu_mid[l] = c.take<float>(N * 3 * F); }
        w.gs = c.take<float>(N * 6 * F);
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
            w.t_q_in[l] = c.take<float>(N * F); w.t_q_mid[l] = c.take<float>(N * F); w.t_mu_mid[l] = c.take<float>(N * 3 * F);
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
        w.t_gW = c.take<float>(E * 3 * F); w.gWd = c.take<float>(E * 3 * F);
    }
    for (int l = 0; l <= L; ++l) w.fq_in[l] = c.take<float>(N * F);
    for (int l = 0; l < L; ++l) { w.fq_mid[l] = c.take<float>(N * F); w.fmu_mid[l] = c.take<float>(N * 3 * F); w.fdot[l] = c.take<float>(N * F); }
    w.gq_b = forces ? c.take<float>(N * F) : nullptr;
    w.fgn = forces ? c.take<float>(N * F) : nullptr;
    w.fgdot = forces ? c.take<float>(N * F) : nullptr;
    w.wtiles = c.take<char>(nb_fused_wtile_bytes(L));
    w.blas_ws = c.take<char>(kBlasWs);
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

// dW[out,in] (lddw) (+)= gY[M,out]^T (ldgy) . X[M,in] (ldx): weight gradient of a Linear layer, reduction over the M rows (cuBLAS SGEMM)
int linear_wgrad(nb200_engine* e, cudaStream_t s, int M, int out, int in, const float* gY, int ldgy, const float* X, int ldx, float* dW, int lddw,
                 float alpha = 1.0f, float beta = 0.0f) {
    Scope sc(e, s, CAT_GEMM, 0);
    return cublasSgemm(e->blas, CUBLAS_OP_N, CUBLAS_OP_T, in, out, M, &alpha, X, ldx, gY, ldgy, &beta, dW, lddw) == CUBLAS_STATUS_SUCCESS ? NB200_OK
                                                                                                                                      : NB200_ECUDA;
}

// weight-gradient backend: wgmma split-K (wgrad_tc.cu) unless NB200_WGRAD=cublas
bool wgrad_tc_on() {
    static const bool on = [] { const char* e = getenv("NB200_WGRAD"); return !(e && e[0] == 'c'); }();
    return on;
}

bool grads_ok(const nb200_painn_weights* g) {
    return g && g->emb && g->w_rbf && g->b_rbf && g->A1 && g->c1 && g->A2 && g->c2 && g->U && g->B1 && g->d1 && g->B2 && g->d2 && g->R1 && g->e1 &&
           g->R2 && g->e2;
}

// Inference (E + analytic F) with the fused node kernels of painn_fused.cu: per layer ONE message kernel and ONE node kernel per direction.
// The graph and the radial filters are already in the workspace.  Same arithmetic as the unfused sequence below (which stays selectable with
// nb200_engine_set_node_backend(eng, 0) and carries the training step), except that q / mu are not updated in place: layer l reads
// fq_in[l], mu[l], the message kernel writes fq_mid[l], fmu_mid[l], the node kernel writes fq_in[l+1], mu[l+1].
// `records` = false (kept training forward): full filter rows in two separate arrays W / dW, the layout the gradient kernels read.
int run_painn_fused(nb200_engine* eng, const nb200_painn_weights* w, const Workspace& ws, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol,
                    int N, int32_t e_cap, float* energy, float* forces, int32_t* status, cudaStream_t s, bool records = true, int bf16 = 0,
                    bool half_rows_sep = false) {
    const int L = w->n_layers, F = NB_F;
    const int w_stride = (forces && records) ? 6 * F : 3 * F;    // [W | dW/dd] records when the backward runs
    const size_t wl_stride = (size_t)e_cap * w_stride;
    const int32_t* w_rev = (records || half_rows_sep) ? ws.rev : nullptr;  // one stored row per undirected pair / one row per edge
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
        NB_TRY(nb_painn_msg_fwd_ex(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.fq_in[l], ws.mu[l], ws.W + l * wl_stride, w_stride, w_rev, ws.geom,
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
                                   w_rev, ws.geom, ws.row_ptr, ws.col, N, ws.gq, cur, ws.gy, other, ws.egrad, s, bf16)); }
        float* t = cur; cur = other; other = t;
        // layer 0: the embedding does not depend on positions, nothing below the message kernel is needed for forces
    }
    { Scope sc(eng, s, CAT_FORCE, 2); NB_TRY(nb200_edge_forces(ws.egrad, ws.geom, ws.row_ptr, ws.rev, N, forces, s));
      NB_TRY(nb_poison_on_error(status, energy, n_mol, forces, (int64_t)3 * N, s)); }
    return NB200_OK;
}

// `grads` != nullptr: training step -- also writes d(sum_m seed_m E_m)/d(weights) into the arrays `grads` points to (same layout as the
// weights; overwritten) -- see painn_train.cu.  Forces stay the true, unweighted -dE/dR.
int run_painn(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
              int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes, float* energy, float* forces, int32_t* status,
              void* stream, const float* seed_mol, const nb200_painn_weights* grads, const float* v_dir = nullptr, int phase = 0,
              bool carve_tangent = false) {
    // phase 0: one call (inference, or the whole training step).  Training split over two calls on the SAME workspace (the forward is not
    // recomputed): phase 1 = graph + filters + fused forward + fused force backward, every activation the gradient pass reads stays in the
    // training workspace; phase 2 = tangent pass + backward with the weight gradients from those kept arrays.
    if (!eng || !weights_ok(w) || !z || !mol_ptr || !workspace || !status) return NB200_EINVAL;
    if (phase != 2 && (!pos || !energy)) return NB200_EINVAL;
    const bool train = grads != nullptr || phase == 1;
    if (phase != 1 && train && !grads_ok(grads)) return NB200_EINVAL;
    if (phase != 2 && train && !forces) return NB200_EINVAL;
    if (w->n_feat != NB_F || w->n_layers <= 0 || w->n_layers > kMaxLayers) return NB200_EUNSUPPORTED;
    if (n_mol <= 0 || n_atoms <= 0 || e_cap <= 0) return NB200_EINVAL;
    const int L = w->n_layers, F = NB_F, K = w->n_rbf, N = n_atoms;
    const bool want_f = forces != nullptr || phase == 2;
    const bool tan = train && v_dir != nullptr;
    Workspace ws = carve(workspace, L, F, n_mol, N, e_cap, want_f, train, phase ? carve_tangent : tan);
    if (ws.bytes > workspace_bytes) return NB200_EINVAL;
    if (phase == 2) {  // the fused forward of phase 1 left layer inputs / post-message states in its own arrays: same values, other names
        for (int l = 0; l < L; ++l) { ws.q_in[l] = ws.fq_in[l]; ws.q_mid[l] = ws.fq_mid[l]; ws.mu_mid[l] = ws.fmu_mid[l]; }
        ws.q = ws.fq_in[L];
    }
    cudaStream_t s = (cudaStream_t)stream;
    cublasHandle_t h = eng->blas;
    NB_BLAS(cublasSetStream(h, s) == CUBLAS_STATUS_SUCCESS);
    NB_BLAS(cublasSetWorkspace(h, ws.blas_ws, kBlasWs) == CUBLAS_STATUS_SUCCESS);

    const size_t wl_stride = (size_t)e_cap * 3 * F;
    const int bf16 = train ? eng->edge_bf16 : 0;  // bf16 rows use the first half of their fp32-sized blocks: all offsets below stay in floats
    // training, like inference, stores ONE filter row (W and dW/dd, two arrays here) per undirected pair: edge e reads row min(e, rev[e]).  Half the filter
    // kernel's work and writes; the second reader of a row mostly finds it in L2.  NB200_TRAIN_HALF_ROWS=0: one row per directed edge (round-2a layout).
    static const bool half_env = [] { const char* e = getenv("NB200_TRAIN_HALF_ROWS"); return !(e && e[0] == '0'); }();
    const bool half_train = train && half_env;
    const int32_t* t_rev = half_train ? ws.rev : nullptr;
    const int32_t* wg_scr = half_train ? ws.sort_scr2 : ws.sort_scr;
    if (phase != 2) {
    // ---- graph + radial filters (painn.py:104-108 / spk PairwiseDistances + filter_net)
    { Scope sc(eng, s, CAT_NBR, 3);
    NB_TRY(nb200_neighbor_build(pos, mol_ptr, n_mol, N, w->cutoff, w->max_neighbors, e_cap, ws.row_ptr, ws.col, ws.rev, ws.geom, ws.deg,
                                status, s)); }
    // fused inference path: ONE filter row per undirected pair (W depends on the distance only: rows of e and rev[e] are bitwise equal), and
    // with forces one interleaved [W | dW/dd] record per row -- half the filter work and HBM writes, one bulk copy per edge in the backward
    const bool half_rows = eng->node_backend == 1 && !train;
    { Scope sc(eng, s, CAT_FILTER, 4);
    NB_TRY(nb_painn_filter_ex(ws.geom, status, e_cap, w->w_rbf, w->b_rbf, L, K, F, w->radial_mode, w->cutoff, w->rbf_offsets, w->rbf_coeff,
                              w->rbf_xscale, ws.W, ws.dW, ws.sort_scr, (half_rows || half_train) ? ws.rev : nullptr, half_rows && want_f ? 1 : 0, s, bf16)); }
    if (half_train) {  // the filter weight gradients still walk every directed edge (slot e holds the gradient of the opposite edge's row): their own sort
        const float dx = (w->cutoff * w->rbf_xscale) / (float)(K - 1);
        Scope sc(eng, s, CAT_FILTER, 3);
        NB_TRY(nb_bin_sort(ws.geom, status, w->rbf_xscale, 1.0f / dx, K, ws.sort_scr2, s, nullptr));
    }
    if (eng->node_backend == 1 && !train) return run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, N, e_cap, energy, forces, status, s);
    if (phase == 1) return run_painn_fused(eng, w, ws, z, mol_ptr, n_mol, N, e_cap, energy, forces, status, s, false, bf16, half_train);
    // ---- embedding (painn.py:110-111)
    { Scope sc(eng, s, CAT_EMBED, 1); NB_TRY(nb_embed(z, w->emb, w->z_offset, w->n_elem, N, ws.q, ws.mu[0], status, s)); }

    for (int l = 0; l < L; ++l) {
        const float* A1 = w->A1 + (size_t)l * F * F;
        const float* A2 = w->A2 + (size_t)l * 3 * F * F;
        const float* U = w->U + (size_t)l * 2 * F * F;
        const float* B1 = w->B1 + (size_t)l * F * 2 * F;
        const float* B2 = w->B2 + (size_t)l * 3 * F * F;
        // message (painn.py:475-509): xh = MLP(q); q,mu += segmented sums
        if (train && cudaMemcpyAsync(ws.q_in[l], ws.q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess) return nb_check_launch();
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.q, F, A1, F, ws.h1pre[l], F, false, w->c1 + (size_t)l * F, ws.act));
        NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.act, F, A2, F, ws.xh[l], 3 * F, false, nullptr, nullptr));
        { Scope sc(eng, s, CAT_MSG_FWD, 1);
        NB_TRY(nb_painn_msg_fwd_ex(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.q, ws.mu[l], ws.W + l * wl_stride, 3 * F, t_rev, ws.geom, ws.row_ptr, ws.col,
                                   N, ws.q, ws.mu[l + 1], s, bf16)); }
        // the update below adds to q and mu[l+1] in place: training keeps the values the update's Linear layers saw
        if (train && (cudaMemcpyAsync(ws.q_mid[l], ws.q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
                      cudaMemcpyAsync(ws.mu_mid[l], ws.mu[l + 1], (size_t)N * 3 * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess))
            return nb_check_launch();
        // update / mixing (painn.py:535-548)
        NB_TRY(linear_fwd(eng, s, 3 * N, 2 * F, F, ws.mu[l + 1], F, U, F, ws.VW[l], 2 * F, false, nullptr, nullptr));
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_upd_norm(ws.VW[l], w->epsilon, N, ws.nrm[l], s)); }
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.q, F, B1, 2 * F, ws.g1pre[l], F, false, nullptr, nullptr));
        NB_TRY(linear_fwd(eng, s, N, F, F, ws.nrm[l], F, B1 + F, 2 * F, ws.g1pre[l], F, true, w->d1 + (size_t)l * F, ws.act));
        NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.act, F, B2, F, ws.y[l], 3 * F, false, nullptr, nullptr));
        { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_upd_combine(ws.q, ws.mu[l + 1], ws.VW[l], ws.y[l], w->d2 + (size_t)l * 3 * F, N, s)); }
    }
    // ---- readout (painn.py:127-128; spk Atomwise + AddOffsets)
    NB_TRY(linear_fwd(eng, s, N, F / 2, F, ws.q, F, w->R1, F, ws.ro_pre, F / 2, false, nullptr, nullptr));
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_readout(ws.ro_pre, w->e1, w->R2, w->e2, N, F / 2, ws.eps, s)); }
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_mol_sum(ws.eps, mol_ptr, n_mol, w->energy_shift_per_atom, energy, s)); }
    if (!want_f) { Scope sc(eng, s, CAT_READOUT, 1); return nb_poison_on_error(status, energy, n_mol, nullptr, 0, s); }
    }  // phase != 2

    // ---- force-loss tangent pass, forward half: directional derivative of every saved activation along v (weights carry no tangent)
    if (tan) {
        Scope sc(eng, s, CAT_NODE, 1 + 6 * L);
        NB_TRY(nb_geom_tan(ws.geom, ws.row_ptr, ws.col, v_dir, N, ws.t_geom, s));
        if (cudaMemsetAsync(ws.t_q, 0, (size_t)N * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();        // embedding: no tangent
        if (cudaMemsetAsync(ws.t_mu[0], 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
        for (int l = 0; l < L; ++l) {
            const float* A1 = w->A1 + (size_t)l * F * F;
            const float* A2 = w->A2 + (size_t)l * 3 * F * F;
            const float* U = w->U + (size_t)l * 2 * F * F;
            const float* B1 = w->B1 + (size_t)l * F * 2 * F;
            const float* B2 = w->B2 + (size_t)l * 3 * F * F;
            if (cudaMemcpyAsync(ws.t_q_in[l], ws.t_q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess) return nb_check_launch();
            NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_q, F, A1, F, ws.t_h1[l], F, false, nullptr, nullptr));
            NB_TRY(nb_mul_dact(ws.h1pre[l], ws.t_h1[l], (int64_t)N * F, ws.t_act, s));
            NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.t_act, F, A2, F, ws.t_xh[l], 3 * F, false, nullptr, nullptr));
            NB_TRY(nb_msg_fwd_tan(ws.xh[l], ws.t_xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.t_mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride,
                                  ws.geom, ws.t_geom, ws.row_ptr, ws.col, N, ws.t_q, ws.t_mu[l + 1], s, bf16, t_rev));
            if (cudaMemcpyAsync(ws.t_q_mid[l], ws.t_q, (size_t)N * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
                cudaMemcpyAsync(ws.t_mu_mid[l], ws.t_mu[l + 1], (size_t)N * 3 * F * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                return nb_check_launch();
            NB_TRY(linear_fwd(eng, s, 3 * N, 2 * F, F, ws.t_mu[l + 1], F, U, F, ws.t_VW[l], 2 * F, false, nullptr, nullptr));
            NB_TRY(nb_upd_norm_tan(ws.VW[l], ws.t_VW[l], ws.nrm[l], N, ws.t_nrm[l], s));
            NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_q, F, B1, 2 * F, ws.t_g1[l], F, false, nullptr, nullptr));
            NB_TRY(linear_fwd(eng, s, N, F, F, ws.t_nrm[l], F, B1 + F, 2 * F, ws.t_g1[l], F, true, nullptr, nullptr));
            NB_TRY(nb_mul_dact(ws.g1pre[l], ws.t_g1[l], (int64_t)N * F, ws.t_act, s));
            NB_TRY(linear_fwd(eng, s, N, 3 * F, F, ws.t_act, F, B2, F, ws.t_y[l], 3 * F, false, nullptr, nullptr));
            NB_TRY(nb_upd_combine_tan(ws.t_q, ws.t_mu[l + 1], ws.VW[l], ws.t_VW[l], ws.y[l], ws.t_y[l], N, s));
        }
        NB_TRY(linear_fwd(eng, s, N, F / 2, F, ws.t_q, F, w->R1, F, ws.t_ro, F / 2, false, nullptr, nullptr));
    }

    // ---- analytic backward: forces = -dE/dR with dE/dE_m = 1 (painn.py:135-146)
    if (cudaMemsetAsync(ws.egrad, 0, (size_t)e_cap * 4 * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    if (cudaMemsetAsync(ws.gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
    { Scope sc(eng, s, CAT_READOUT, 1); NB_TRY(nb_readout_bwd(ws.ro_pre, w->R2, N, F / 2, ws.g_ro, s)); }
    NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.g_ro, F / 2, w->R1, F, ws.gq, F, false));
    // energy-seed weight gradients: dW += (c o g)^T x and dbias += colsum(c o g), c = the per-atom seed (`rs_div` rows of g per atom: 3 for the
    // (atom, xyz) rows of U).  One wgmma split-K launch (wgrad_tc.cu: the row scale is applied while loading g); NB200_WGRAD=cublas keeps the
    // round-1 sequence (scale kernel + cuBLAS SGEMM + column-sum kernel).
    // Weight-gradient launches are LEAVES of the step: they read buffers of the backward chain and only add into `grads`.  They run on a
    // second stream of the engine, next to the chain (whose 76-CTA GEMMs and latency-bound phases leave SMs idle): fork = the side stream
    // waits for the chain's current point, and the chain waits for a leaf only right before it overwrites that leaf's inputs (`need`).  The
    // side stream is in order, so one event per input group is enough.  NB200_TRAIN_SIDE=0 keeps everything on the caller's stream.
    static const bool side_env = [] { const char* e = getenv("NB200_TRAIN_SIDE"); return !(e && e[0] == '0'); }();
    bool use_side = train && phase != 1 && side_env && wgrad_tc_on();
    if (use_side && !eng->side && cudaStreamCreateWithFlags(&eng->side, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); use_side = false; }
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
    // with a force seed the energy-seed term rides in the tangent call of the same Linear (one 3-term launch, wgrad_tc.cu::nb_wgrad_tc3)
    const bool tan_for_merge = train && v_dir != nullptr;
    auto merged = [&](int M, int out, int in, const float* g, int ldg, const float* x, int ldx, const float* dW, int lddw) {
        return tan_for_merge && wgrad_tc_on() && nb_wgrad_tc_ok(M, out, in, g, ldg, x, ldx, dW, lddw);
    };
    auto wg_primal = [&](int M, int out, int in, const float* g, int ldg, const float* x, int ldx, float* dW, int lddw, float* dbias, int rs_div) -> int {
        if (merged(M, out, in, g, ldg, x, ldx, dW, lddw)) return NB200_OK;
        if (wgrad_tc_on() && nb_wgrad_tc_ok(M, out, in, g, ldg, x, ldx, dW, lddw)) {
            fork();
            const int rc = nb_wgrad_tc(M, out, in, g, x, nullptr, nullptr, ldg, ldx, dW, lddw, 1.0f, dbias, 1.0f, 0, ws.seed_atom, rs_div, ls);
            leaf_done();
            return rc;
        }
        NB_TRY(nb_scale_rows(g, ws.seed_atom, rs_div, M, out, ws.gs, s));
        NB_TRY(linear_wgrad(eng, s, M, out, in, ws.gs, ldg, x, ldx, dW, lddw, 1.0f, 1.0f));
        return dbias ? nb_colsum(ws.gs, M, out, dbias, s, 1.0f, 1) : NB200_OK;
    };
    if (train) {
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
        NB_TRY(wg_primal(N, F / 2, F, ws.g_ro, F / 2, ws.q, F, const_cast<float*>(grads->R1), F, const_cast<float*>(grads->e1), 1));
    }
    // tangent weight gradients enter with sign -1:  d/dtheta sum_i v_i.F_i = -(v.d/dR) dE_tot/dtheta   (seed 1, not the energy seed)
    auto wgrad_tan = [&](int M, int out, int in, const float* g, const float* tg, int ldg, const float* x, const float* tx, int ldx, float* dW,
                         int lddw, float* dbias = nullptr, int rs_div = 1) -> int {
        if (merged(M, out, in, g, ldg, x, ldx, dW, lddw)) {  // (c o g)^T x - tg^T x - g^T tx and the bias sums, one launch
            fork();
            const int rc = nb_wgrad_tc3(M, out, in, g, tg, ldg, x, tx, ldx, dW, lddw, dbias, ws.seed_atom, rs_div, ls);
            leaf_done();
            return rc;
        }
        if (wgrad_tc_on() && nb_wgrad_tc_ok(M, out, in, tg, ldg, x, ldx, dW, lddw) && nb_wgrad_tc_ok(M, out, in, g, ldg, tx, ldx, dW, lddw)) {
            fork();
            const int rc = nb_wgrad_tc(M, out, in, tg, x, g, tx, ldg, ldx, dW, lddw, -1.0f, dbias, -1.0f, 0, nullptr, 1, ls);  // one launch: tg^T x + g^T tx, colsum(tg)
            leaf_done();
            return rc;
        }
        NB_TRY(linear_wgrad(eng, s, M, out, in, tg, ldg, x, ldx, dW, lddw, -1.0f, 1.0f));
        NB_TRY(linear_wgrad(eng, s, M, out, in, g, ldg, tx, ldx, dW, lddw, -1.0f, 1.0f));
        return dbias ? nb_colsum(tg, M, out, dbias, s, -1.0f, 1) : NB200_OK;
    };
    if (tan) {
        Scope sc(eng, s, CAT_NODE, 4);
        if (cudaMemsetAsync(ws.t_gmu_a, 0, (size_t)N * 3 * F * sizeof(float), s) != cudaSuccess) return nb_check_launch();
        NB_TRY(nb_readout_bwd_tan(ws.ro_pre, ws.t_ro, w->R2, N, F / 2, ws.t_g_ro, ws.t_act, s));  // t_act [N, F/2] = silu'(pre) pre^
        NB_TRY(linear_bwd(eng, s, N, F / 2, F, ws.t_g_ro, F / 2, w->R1, F, ws.t_gq, F, false));
        NB_TRY(nb_colsum(ws.t_act, N, F / 2, const_cast<float*>(grads->R2), s, -1.0f, 1));
        NB_TRY(wgrad_tan(N, F / 2, F, ws.g_ro, ws.t_g_ro, F / 2, ws.q, ws.t_q, F, const_cast<float*>(grads->R1), F, const_cast<float*>(grads->e1)));
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
        if (train) {  // dB2, dd2
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
            NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.q_mid[l], ws.t_q_mid[l], F, gB1, 2 * F, const_cast<float*>(grads->d1) + (size_t)l * F));
            NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.nrm[l], ws.t_nrm[l], F, gB1 + F, 2 * F));
        }
        if (train) {  // dB1 = [gt^T q_mid | gt^T nrm], dd1
            Scope sc(eng, s, CAT_NODE, 2);
            float* gB1 = const_cast<float*>(grads->B1) + (size_t)l * F * 2 * F;
            NB_TRY(wg_primal(N, F, F, ws.gt, F, ws.q_mid[l], F, gB1, 2 * F, const_cast<float*>(grads->d1) + (size_t)l * F, 1));
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
            NB_TRY(wgrad_tan(3 * N, 2 * F, F, ws.gVW, ws.t_gVW, 2 * F, ws.mu_mid[l], ws.t_mu_mid[l], F, const_cast<float*>(grads->U) + (size_t)l * 2 * F * F, F,
                             nullptr, 3));
        }
        if (train) {  // dU over the 3N (atom, xyz) rows
            Scope sc(eng, s, CAT_NODE, 1);
            NB_TRY(wg_primal(3 * N, 2 * F, F, ws.gVW, 2 * F, ws.mu_mid[l], F, const_cast<float*>(grads->U) + (size_t)l * 2 * F * F, F, nullptr, 3));
        }
        NB_TRY(linear_bwd(eng, s, PT * 3 * N, 2 * F, F, ws.gVW, 2 * F, U, F, cur, F, true));  // (cur, t_cur) = (gmu_a, t_gmu_a) or (gmu_b, t_gmu_b): adjacent
        // message backward (by source atom; uses edge symmetry)
        need(d_B2); need(d_F);  // it overwrites gy (read by dB2) and the per-edge filter gradients (read by the filter leaves of the layer above)
        { Scope sc(eng, s, CAT_MSG_BWD, 1);
        if (!train)
            NB_TRY(nb200_painn_msg_bwd(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride, ws.geom,
                                       ws.row_ptr, ws.col, N, ws.gq, cur, ws.gy, other, ws.egrad, s));
        else
            NB_TRY(nb_painn_msg_bwd_train(ws.xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride, ws.geom,
                                          ws.row_ptr, ws.col, N, ws.gq, cur, ws.gy, other, ws.egrad, ws.gW, ws.seed_atom, s, bf16, t_rev)); }
        if (tan) {  // message backward tangent reads the same gq / cur the primal call just read; its outputs go to the t_ twins
            Scope sc(eng, s, CAT_NODE, 2);
            NB_TRY(nb_msg_bwd_tan(ws.xh[l], ws.t_xh[l], w->c2 + (size_t)l * 3 * F, ws.mu[l], ws.t_mu[l], ws.W + l * wl_stride, ws.dW + l * wl_stride,
                                  ws.geom, ws.t_geom, ws.row_ptr, ws.col, N, ws.gq, ws.t_gq, cur, t_cur, ws.t_gy, t_other, ws.t_gW, ws.gWd, s, bf16, t_rev));
            tag = &d_F; fork();
            NB_TRY(nb_filter_wgrad_tan(ws.geom, ws.t_geom, status, wg_scr, w->rbf_offsets, K, w->radial_mode, w->cutoff, w->rbf_coeff, w->rbf_xscale,
                                       ws.t_gW, ws.gWd, -1.0f, const_cast<float*>(grads->w_rbf) + (size_t)l * K * 3 * F,
                                       const_cast<float*>(grads->b_rbf) + (size_t)l * 3 * F, ls, e_cap, bf16));
            leaf_done();
            float* tt = t_cur; t_cur = t_other; t_other = tt;
        }
        float* t = cur; cur = other; other = t;
        if (train) {  // filter weights of this layer, then dA2, dc2
            Scope sc(eng, s, CAT_NODE, 4);
            tag = &d_F; fork();
            NB_TRY(nb_filter_wgrad(ws.geom, status, wg_scr, w->rbf_offsets, K, w->radial_mode, w->cutoff, w->rbf_coeff, w->rbf_xscale, ws.gW,
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
        if (l > 0 || train) {  // inference: the embedding does not depend on positions, layer 0 stops here
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
                NB_TRY(wgrad_tan(N, F, F, ws.gt, ws.t_gt, F, ws.q_in[l], ws.t_q_in[l], F, const_cast<float*>(grads->A1) + (size_t)l * F * F, F,
                                 const_cast<float*>(grads->c1) + (size_t)l * F));
            }
            if (train) {  // dA1, dc1
                Scope sc(eng, s, CAT_NODE, 2);
                NB_TRY(wg_primal(N, F, F, ws.gt, F, ws.q_in[l], F, const_cast<float*>(grads->A1) + (size_t)l * F * F, F,
                                 const_cast<float*>(grads->c1) + (size_t)l * F, 1));
            }
            NB_TRY(linear_bwd(eng, s, PT * N, F, F, ws.gt, F, A1, F, ws.gq, F, true));
        }
    }
    if (train) { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_emb_grad(ws.gq, ws.seed_atom, z, w->z_offset, w->n_elem, N, const_cast<float*>(grads->emb), s)); }
    if (tan) { Scope sc(eng, s, CAT_NODE, 1); NB_TRY(nb_emb_grad(ws.t_gq, nullptr, z, w->z_offset, w->n_elem, N, const_cast<float*>(grads->emb), s, -1.0f)); }
    if (phase == 2) return NB200_OK;  // energies / forces were returned (and poisoned on error) by phase 1
    { Scope sc(eng, s, CAT_FORCE, 2); NB_TRY(nb200_edge_forces(ws.egrad, ws.geom, ws.row_ptr, ws.rev, N, forces, s));
      NB_TRY(nb_poison_on_error(status, energy, n_mol, forces, (int64_t)3 * N, s)); }
    return NB200_OK;
}

}  // namespace

extern "C" int nb200_painn_energy_forces(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos,
                                         const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace,
                                         int64_t workspace_bytes, float* energy, float* forces, int32_t* status, void* stream) {
    return run_painn(eng, w, z, pos, mol_ptr, n_mol, n_atoms, e_cap, workspace, workspace_bytes, energy, forces, status, stream, nullptr, nullptr);
}

extern "C" int64_t nb200_painn_train_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap,
                                                     int32_t with_force_seed) {
    if (!w || w->n_layers <= 0 || w->n_layers > kMaxLayers || w->n_feat != NB_F || b_cap < 0 || n_cap < 0 || e_cap < 0) return NB200_EINVAL;
    return carve(nullptr, w->n_layers, w->n_feat, b_cap, n_cap, e_cap, true, true, with_force_seed != 0).bytes;
}

// Training step in two calls on one training workspace (sized by nb200_painn_train_workspace_bytes with the SAME with_force_seed flag for
// both): the forward + forces first, the parameter gradients once the loss has produced the seeds.  Nothing else may use the workspace in
// between; weights, z, mol_ptr, n_* and e_cap must be those of the forward call.
extern "C" int nb200_painn_train_forward(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                         int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes,
                                         int32_t with_force_seed, float* energy, float* forces, int32_t* status, void* stream) {
    if (!forces) return NB200_EINVAL;
    return run_painn(eng, w, z, pos, mol_ptr, n_mol, n_atoms, e_cap, workspace, workspace_bytes, energy, forces, status, stream, nullptr, nullptr, nullptr,
                     1, with_force_seed != 0);
}

extern "C" int nb200_painn_train_backward(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const int32_t* mol_ptr, int32_t n_mol,
                                          int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes, int32_t with_force_seed,
                                          const float* energy_seed, const float* force_seed, const nb200_painn_weights* grads, int32_t* status,
                                          void* stream) {
    if (!grads || (force_seed && !with_force_seed)) return NB200_EINVAL;
    return run_painn(eng, w, z, nullptr, mol_ptr, n_mol, n_atoms, e_cap, workspace, workspace_bytes, nullptr, nullptr, status, stream, energy_seed, grads,
                     force_seed, 2, with_force_seed != 0);
}

extern "C" int nb200_painn_energy_forces_grads(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos,
                                               const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace,
                                               int64_t workspace_bytes, const float* energy_seed, const float* force_seed,
                                               const nb200_painn_weights* grads, float* energy, float* forces, int32_t* status, void* stream) {
    if (!grads) return NB200_EINVAL;
    return run_painn(eng, w, z, pos, mol_ptr, n_mol, n_atoms, e_cap, workspace, workspace_bytes, energy, forces, status, stream, energy_seed, grads,
                     force_seed);
}
