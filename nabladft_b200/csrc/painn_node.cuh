// painn_node.cuh -- launchers of the node-level (per-atom) kernels used by the engine.
#pragma once
#include "common.cuh"

int nb_embed(const int32_t* z, const float* emb, int z_offset, int n_elem, int n_atoms, float* q, float* mu, int32_t* status,
             cudaStream_t s);
int nb_bias_act(float* pre, const float* bias, float* act, int n_rows, int width, int kind, cudaStream_t s);
int nb_act_bwd(float* g, const float* pre, int64_t n, int kind, cudaStream_t s);
int nb_upd_norm(const float* VW, float eps, int n_atoms, float* nrm, cudaStream_t s);
int nb_upd_combine(float* q, float* mu, const float* VW, float* y, const float* y_bias, int n_atoms, cudaStream_t s);
int nb_upd_combine_bwd(const float* gq, const float* gmu, const float* y, const float* VW, int n_atoms, float* gy, float* gVW,
                       cudaStream_t s);
int nb_upd_norm_bwd(const float* gn, const float* VW, const float* nrm, int n_atoms, float* gVW, cudaStream_t s);
int nb_readout(float* pre, const float* e1, const float* R2, const float* e2, int n_atoms, int width, float* eps_atom, cudaStream_t s);
int nb_mol_sum(const float* eps_atom, const int32_t* mol_ptr, int n_mol, float shift_per_atom, float* energy, cudaStream_t s);
int nb_readout_bwd(const float* pre, const float* R2, int n_atoms, int width, float* g_pre, cudaStream_t s);
int nb_poison_on_error(const int32_t* status, float* energy, int n_mol, float* forces, int64_t n_f, cudaStream_t s);

// training helpers (painn_train.cu, filter.cu, painn_msg.cu)
int nb_seed_atom(const float* seed_mol, const int32_t* mol_ptr, int n_mol, float* seed_atom, cudaStream_t s);
int nb_scale_rows(const float* g, const float* seed_atom, int rows_per_atom, int64_t n_rows, int width, float* out, cudaStream_t s);
int nb_act_only(const float* pre, const float* seed_atom, int64_t n_rows, int width, int kind, float* act, cudaStream_t s);
int nb_colsum(const float* x, int64_t n_rows, int width, float* out, cudaStream_t s, float alpha = 1.0f, int accumulate = 0);
int nb_emb_grad(const float* gq, const float* seed_atom, const int32_t* z, int z_offset, int n_elem, int n_atoms, float* g_emb, cudaStream_t s,
                float sign = 1.0f);
int nb_filter_wgrad(const float* geom, const int32_t* status, const int32_t* sort_scratch, const float* rbf_offsets, int n_rbf, int radial_mode,
                    float cutoff, float rbf_coeff, float rbf_xscale, const float* gW, float* g_w, float* g_b, cudaStream_t s, int e_cap = 0, int bf16 = 0);
int nb_painn_msg_bwd_train(const float* xh, const float* xh_bias, const float* mu, const float* W, const float* dW, const float* geom,
                           const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q, const float* g_mu, float* g_xh,
                           float* g_mu_in, float* egrad, float* gW, const float* seed_atom, cudaStream_t stream, int bf16 = 0, const int32_t* rev = nullptr);

// force-loss tangent pass (painn_tangent.cu)
int nb_geom_tan(const float* geom, const int32_t* row_ptr, const int32_t* col, const float* v, int n_atoms, float* t_geom, cudaStream_t s);
int nb_mul_dact(const float* pre, const float* x, int64_t n, float* out, cudaStream_t s);
int nb_act_bwd_tan(float* t_g, const float* g_pre, const float* pre, const float* t_pre, int64_t n, cudaStream_t s);
int nb_msg_fwd_tan(const float* xh, const float* t_xh, const float* xh_bias, const float* mu, const float* t_mu, const float* W, const float* dW,
                   const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* col, int n_atoms, float* t_q, float* t_mu_out,
                   cudaStream_t s, int bf16 = 0, const int32_t* rev = nullptr);
int nb_upd_norm_tan(const float* VW, const float* t_VW, const float* nrm, int n_atoms, float* t_nrm, cudaStream_t s);
int nb_upd_combine_tan(float* t_q, float* t_mu, const float* VW, const float* t_VW, const float* y, const float* t_y, int n_atoms, cudaStream_t s);
int nb_readout_bwd_tan(const float* pre, const float* t_pre, const float* R2, int n_atoms, int width, float* t_g_pre, float* t_act, cudaStream_t s);
int nb_upd_combine_bwd_tan(const float* gq, const float* t_gq, const float* gmu, const float* t_gmu, const float* y, const float* t_y, const float* VW,
                           const float* t_VW, int n_atoms, float* t_gy, float* t_gVW, cudaStream_t s);
int nb_upd_norm_bwd_tan(const float* gn, const float* t_gn, const float* VW, const float* t_VW, const float* nrm, const float* t_nrm, int n_atoms,
                        float* t_gVW, cudaStream_t s);
int nb_msg_bwd_tan(const float* xh, const float* t_xh, const float* xh_bias, const float* mu, const float* t_mu, const float* W, const float* dW,
                   const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* col, int n_atoms, const float* g_q,
                   const float* t_g_q, const float* g_mu, const float* t_g_mu, float* t_g_xh, float* t_g_mu_in, float* t_gW, float* gWd,
                   cudaStream_t s, int bf16 = 0, const int32_t* rev = nullptr);
int nb_filter_wgrad_tan(const float* geom, const float* t_geom, const int32_t* status, const int32_t* sort_scratch, const float* rbf_offsets, int n_rbf,
                        int radial_mode, float cutoff, float rbf_coeff, float rbf_xscale, const float* t_gW, const float* gWd, float sign, float* g_w,
                        float* g_b, cudaStream_t s, int e_cap = 0, int bf16 = 0);

// fused per-layer node kernels (painn_fused.cu): wgmma chain of the update / message-MLP / readout Linear layers with their elementwise glue
struct NbFusedFwd {
    int n_atoms, n_layers;
    int layer_upd;   // layer whose update runs (-1: none)
    int layer_mlp;   // layer whose message MLP runs afterwards (-1: none)
    int readout;     // 1: the readout's first Linear runs afterwards
    const void* wtiles;
    const float *q_mid, *mu_mid, *d1, *d2;
    float *VW, *nrm, *dot, *g1pre, *y, *q_next, *mu_next;
    float eps;
    const float *q_mlp_in, *c1;
    float *h1pre, *xh, *ro_pre;
};
struct NbFusedBwd {
    int n_atoms, n_layers;
    int layer_mlp;   // layer whose message MLP is differentiated first (-1: none)
    int readout;     // 1: start from the readout instead
    int layer_upd;   // layer whose update is differentiated (-1: none)
    const void* wtiles;
    float *gq_a, *gq_b, *cur, *gn, *gdot;
    const float *g_xh, *h1pre, *ro_pre, *R2, *y, *VW, *nrm, *dot, *g1pre;
};
int64_t nb_fused_wtile_bytes(int n_layers);
int nb_fused_prep(const nb200_painn_weights* w, void* wtiles, cudaStream_t s);
int nb_fused_node_fwd(const NbFusedFwd& a, cudaStream_t s);
int nb_fused_node_bwd(const NbFusedBwd& a, cudaStream_t s);
