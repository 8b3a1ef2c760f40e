// painn_tangent_test.cu -- nb200_painn_test_tangent (include/nabla_b200.h): one kernel of the PaiNN tangent / Hessian-vector-product path
// on caller-built inputs, so that tests/test_gpu_painn_tangent.py can compare each with a float64 reference on row shapes, distances and
// atom counts the fixture molecules never produce.  Every op calls the host wrapper the engine calls, with the launch configuration the
// engine uses; nothing here is on a product path.
#include "painn_node.cuh"

namespace {

// the radial parameters the filter kernels support (the checks of nb_painn_filter_d2, which FILTER_WGRAD shares)
int radial_ok(const nb200_painn_tan_args* a) {
    if (a->n_rbf < NB_BAND || a->n_rbf > NB_NBINS_MAX) return NB200_EUNSUPPORTED;
    if (a->radial_mode != NB200_RADIAL_SPK && a->radial_mode != NB200_RADIAL_OC) return NB200_EUNSUPPORTED;
    const float dx = (a->cutoff * a->rbf_xscale) / (float)(a->n_rbf - 1);
    if (!(a->rbf_coeff < 0.f) || a->rbf_coeff * (7.0f * dx) * (7.0f * dx) > -23.0f) return NB200_EUNSUPPORTED;
    return NB200_OK;
}

template <class... P>
bool all(P... p) {
    return ((p != nullptr) && ...);
}

}  // namespace

extern "C" int nb200_painn_test_tangent(const nb200_painn_tan_args* a, void* stream) {
    if (!a || a->op < 0 || a->op >= NB200_PT_N_OPS || a->n_atoms < 0 || a->n < 0 || a->e_cap < 0) return NB200_EINVAL;
    const int op = a->op, N = a->n_atoms;
    const bool bf16_ok = op == NB200_PT_MSG_FWD_TAN || op == NB200_PT_MSG_BWD_TAN || op == NB200_PT_FILTER_WGRAD;
    if ((a->bf16 != 0 && (a->bf16 != 1 || !bf16_ok)) || (a->tan != 0 && (a->tan != 1 || op != NB200_PT_FILTER_WGRAD))) return NB200_EINVAL;
    if ((op == NB200_PT_MUL_DACT || op == NB200_PT_ACT_BWD_TAN) && a->n % 4 != 0) return NB200_EINVAL;  // the kernels run n / 4 float4s
    cudaStream_t s = (cudaStream_t)stream;
    const float* W = static_cast<const float*>(a->W);
    const float* dW = static_cast<const float*>(a->dW);
    switch (op) {
    case NB200_PT_GEOM_TAN:
        if (!all(a->geom, a->row_ptr, a->col, a->v, a->t_geom)) return NB200_EINVAL;
        return nb_geom_tan(a->geom, a->row_ptr, a->col, a->v, N, a->t_geom, s);
    case NB200_PT_MUL_DACT:
        if (!all(a->pre, a->x, a->out)) return NB200_EINVAL;
        return nb_mul_dact(a->pre, a->x, a->n, a->out, s);
    case NB200_PT_ACT_BWD_TAN:
        if (!all(a->t_g, a->g_pre, a->pre, a->t_pre)) return NB200_EINVAL;
        return nb_act_bwd_tan(a->t_g, a->g_pre, a->pre, a->t_pre, a->n, s);
    case NB200_PT_READOUT_BWD_TAN:
        if (!all(a->pre, a->t_pre, a->R2, a->t_g_pre, a->t_act) || a->width < 1) return NB200_EINVAL;
        return nb_readout_bwd_tan(a->pre, a->t_pre, a->R2, N, a->width, a->t_g_pre, a->t_act, s);
    case NB200_PT_MSG_FWD_TAN:
        if (!all(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->geom, a->t_geom, a->row_ptr, a->col, a->t_q, a->t_mu_out)) return NB200_EINVAL;
        return nb_msg_fwd_tan(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->geom, a->t_geom, a->row_ptr, a->col, N, a->t_q, a->t_mu_out, s,
                              a->bf16, a->rev);
    case NB200_PT_UPD_NORM_TAN:
        if (!all(a->VW, a->t_VW, a->nrm, a->t_nrm)) return NB200_EINVAL;
        return nb_upd_norm_tan(a->VW, a->t_VW, a->nrm, N, a->t_nrm, s);
    case NB200_PT_UPD_COMBINE_TAN:
        if (!all(a->t_q, a->t_mu, a->VW, a->t_VW, a->y, a->t_y)) return NB200_EINVAL;
        return nb_upd_combine_tan(a->t_q, a->t_mu, a->VW, a->t_VW, a->y, a->t_y, N, s);
    case NB200_PT_UPD_COMBINE_BWD_TAN:
        if (!all(a->g_q, a->t_g_q, a->g_mu, a->t_g_mu, a->y, a->t_y, a->VW, a->t_VW, a->t_gy, a->t_gVW)) return NB200_EINVAL;
        return nb_upd_combine_bwd_tan(a->g_q, a->t_g_q, a->g_mu, a->t_g_mu, a->y, a->t_y, a->VW, a->t_VW, N, a->t_gy, a->t_gVW, s);
    case NB200_PT_UPD_NORM_BWD_TAN:
        if (!all(a->gn, a->t_gn, a->VW, a->t_VW, a->nrm, a->t_nrm, a->t_gVW)) return NB200_EINVAL;
        return nb_upd_norm_bwd_tan(a->gn, a->t_gn, a->VW, a->t_VW, a->nrm, a->t_nrm, N, a->t_gVW, s);
    case NB200_PT_MSG_BWD_TAN:
        if (!all(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->geom, a->t_geom, a->row_ptr, a->col, a->g_q, a->t_g_q, a->g_mu, a->t_g_mu,
                 a->t_g_xh, a->t_g_mu_in, a->t_gW, a->gWd))
            return NB200_EINVAL;
        return nb_msg_bwd_tan(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->geom, a->t_geom, a->row_ptr, a->col, N, a->g_q, a->t_g_q, a->g_mu,
                              a->t_g_mu, a->t_g_xh, a->t_g_mu_in, static_cast<float*>(a->t_gW), static_cast<float*>(a->gWd), s, a->bf16, a->rev);
    case NB200_PT_MSG_BWD_HVP:
        if (!all(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->d2W, a->geom, a->t_geom, a->row_ptr, a->col, a->rev, a->g_q, a->t_g_q, a->g_mu,
                 a->t_g_mu, a->t_g_xh, a->t_g_mu_in, a->t_egrad))
            return NB200_EINVAL;
        return nb_msg_bwd_hvp(a->xh, a->t_xh, a->xh_bias, a->mu, a->t_mu, W, dW, a->d2W, a->geom, a->t_geom, a->row_ptr, a->col, a->rev, N, a->g_q,
                              a->t_g_q, a->g_mu, a->t_g_mu, a->t_g_xh, a->t_g_mu_in, a->t_egrad, s);
    case NB200_PT_EDGE_FORCES_HVP:
        if (!all(a->egrad, a->t_egrad, a->geom, a->t_geom, a->row_ptr, a->rev, a->hv)) return NB200_EINVAL;
        return nb_edge_forces_hvp(a->egrad, a->t_egrad, a->geom, a->t_geom, a->row_ptr, a->rev, N, a->hv, s);
    case NB200_PT_FILTER_D2:  // as run_painn_hvp: one row per undirected pair, rows of stride e_cap per layer
        if (!all(a->geom, a->status, a->rev, a->sort_scratch, a->rbf_offsets, a->w_rbf, a->b_rbf, W, dW, a->d2W)) return NB200_EINVAL;
        return nb_painn_filter_d2(a->geom, a->status, a->e_cap, a->w_rbf, a->b_rbf, a->n_layers, a->n_rbf, a->radial_mode, a->cutoff, a->rbf_offsets,
                                  a->rbf_coeff, a->rbf_xscale, static_cast<float*>(a->W), static_cast<float*>(a->dW), a->d2W, a->sort_scratch, a->rev, s);
    case NB200_PT_FILTER_WGRAD: {  // as the training step: the bin sort over every directed edge (engine.cu graph_and_filters), then one layer
        if (!all(a->geom, a->status, a->sort_scratch, a->rbf_offsets, a->g_w, a->g_b) || !(a->tan ? all(a->t_gW, a->gWd) : all(a->gW)))
            return NB200_EINVAL;
        if (int rc = radial_ok(a)) return rc;
        const float dx = (a->cutoff * a->rbf_xscale) / (float)(a->n_rbf - 1);
        if (int rc = nb_bin_sort(a->geom, a->status, a->rbf_xscale, 1.0f / dx, a->n_rbf, a->sort_scratch, s, nullptr)) return rc;
        if (a->tan)
            return nb_filter_wgrad_tan(a->geom, nullptr, a->status, a->sort_scratch, a->rbf_offsets, a->n_rbf, a->radial_mode, a->cutoff, a->rbf_coeff,
                                       a->rbf_xscale, static_cast<const float*>(a->t_gW), static_cast<const float*>(a->gWd), a->sign, a->g_w, a->g_b, s,
                                       a->e_cap, a->bf16);
        return nb_filter_wgrad(a->geom, a->status, a->sort_scratch, a->rbf_offsets, a->n_rbf, a->radial_mode, a->cutoff, a->rbf_coeff, a->rbf_xscale,
                               static_cast<const float*>(a->gW), a->g_w, a->g_b, s, a->e_cap, a->bf16);
    }
    }
    return NB200_EINVAL;
}
