// painn_node_test.cu -- nb200_painn_test_node (include/nabla_b200.h): the weight preparation and one program of the fused PaiNN node
// kernels (painn_fused.cu), or one primal per-atom kernel of painn_node.cu, on caller-built inputs, so that tests/test_gpu_painn_node.py can
// compare each with a float64 reference at tile widths and atom counts the engine's batches do not choose.  Every op calls the host wrapper
// the engine calls, with the launch configuration the engine uses; nothing here is on a product path.
#include "painn_node.cuh"

namespace {

template <class... P>
bool all(P... p) {
    return ((p != nullptr) && ...);
}
template <class... P>
bool aligned(P... p) {
    return ((reinterpret_cast<uintptr_t>(p) % 16 == 0) && ...);
}

// everything k_prep_painn reads
bool weights_ok(const nb200_painn_weights* w) {
    return w && w->n_feat == NB_F && w->n_layers > 0 && all(w->A1, w->A2, w->U, w->B1, w->B2, w->R1);
}

// The programs the engine launches (engine.cu run_painn_fused): any other combination would wait for an operand no code path writes.
bool fwd_program_ok(int upd, int mlp, int ro, int L) {
    auto in = [L](int l) { return l >= 0 && l < L; };
    return (upd == -1 && in(mlp) && ro == 0) || (in(upd) && mlp == upd + 1 && in(mlp) && ro == 0) || (in(upd) && mlp == -1 && ro == 1);
}
bool bwd_program_ok(int upd, int mlp, int ro, int L) {
    auto in = [L](int l) { return l >= 0 && l < L; };
    return in(upd) && ((ro == 1 && mlp == -1) || (ro == 0 && mlp == upd + 1 && in(mlp)));
}

int node_fwd(nb200_painn_node_args* a, cudaStream_t s) {
    const nb200_painn_weights* w = a->w;
    const int L = w->n_layers, F = NB_F, upd = a->layer_upd, mlp = a->layer_mlp;
    if (!fwd_program_ok(upd, mlp, a->readout, L)) return NB200_EINVAL;
    const bool u = upd >= 0, m = mlp >= 0;
    if (u && !(all(a->q_mid, a->mu_mid, a->VW, a->nrm, a->dot, a->g1pre, a->y, a->q_next, a->mu_next, w->d1, w->d2) &&
               aligned(a->q_mid, a->mu_mid, a->VW, a->nrm, a->dot, a->g1pre, a->y, a->q_next, a->mu_next)))
        return NB200_EINVAL;
    if (m && !(all(a->h1pre, a->xh, w->c1) && aligned(a->h1pre, a->xh))) return NB200_EINVAL;
    if (!u && !(a->q_mlp_in && aligned(a->q_mlp_in))) return NB200_EINVAL;
    if (a->readout && !(a->ro_pre && aligned(a->ro_pre))) return NB200_EINVAL;
    NbFusedFwd f{};  // as run_painn_fused
    f.n_atoms = a->n_atoms; f.n_layers = L; f.wtiles = a->wtiles; f.eps = w->epsilon; f.ro_pre = a->ro_pre;
    f.layer_upd = upd; f.layer_mlp = mlp; f.readout = a->readout;
    if (u) {
        f.q_mid = a->q_mid; f.mu_mid = a->mu_mid; f.d1 = w->d1 + (size_t)upd * F; f.d2 = w->d2 + (size_t)upd * 3 * F;
        f.VW = a->VW; f.nrm = a->nrm; f.dot = a->dot; f.g1pre = a->g1pre; f.y = a->y; f.q_next = a->q_next; f.mu_next = a->mu_next;
    } else {
        f.q_mlp_in = a->q_mlp_in;
    }
    if (m) { f.c1 = w->c1 + (size_t)mlp * F; f.h1pre = a->h1pre; f.xh = a->xh; }
    if (int rc = nb_fused_prep(w, a->wtiles, s)) return rc;
    return nb_fused_node_fwd(f, s, &a->tile);
}

int node_bwd(nb200_painn_node_args* a, cudaStream_t s) {
    const nb200_painn_weights* w = a->w;
    const int L = w->n_layers, upd = a->layer_upd, mlp = a->layer_mlp;
    if (!bwd_program_ok(upd, mlp, a->readout, L)) return NB200_EINVAL;
    if (!(all(a->gq_a, a->gq_b, a->cur, a->gn, a->gdot, a->y, a->VW, a->nrm, a->dot, a->g1pre) &&
          aligned(a->gq_a, a->gq_b, a->cur, a->gn, a->gdot, a->y, a->VW, a->nrm, a->dot, a->g1pre)))
        return NB200_EINVAL;
    if (mlp >= 0 && !(all(a->g_xh, a->h1pre) && aligned(a->g_xh, a->h1pre))) return NB200_EINVAL;
    if (a->readout && !(all(a->ro_pre, w->R2) && aligned(a->ro_pre, w->R2))) return NB200_EINVAL;
    NbFusedBwd b{};  // as run_painn_fused
    b.n_atoms = a->n_atoms; b.n_layers = L; b.wtiles = a->wtiles; b.gq_a = a->gq_a; b.gq_b = a->gq_b; b.gn = a->gn; b.gdot = a->gdot;
    b.ro_pre = a->ro_pre; b.R2 = w->R2; b.g_xh = a->g_xh;
    b.readout = a->readout; b.layer_mlp = mlp; b.layer_upd = upd;
    b.cur = a->cur; b.h1pre = mlp >= 0 ? a->h1pre : nullptr;
    b.y = a->y; b.VW = a->VW; b.nrm = a->nrm; b.dot = a->dot; b.g1pre = a->g1pre;
    if (int rc = nb_fused_prep(w, a->wtiles, s)) return rc;
    return nb_fused_node_bwd(b, s, &a->tile);
}

}  // namespace

extern "C" int nb200_painn_test_node(nb200_painn_node_args* a, void* stream) {
    if (!a || a->op < 0 || a->op >= NB200_PN_N_OPS || a->n_atoms < 0 || a->n < 0 || a->n_mol < 0) return NB200_EINVAL;
    if (a->tile != 0 && a->tile != 64 && a->tile != 80) return NB200_EINVAL;
    const int op = a->op, N = a->n_atoms, F = NB_F;
    const nb200_painn_weights* w = a->w;
    cudaStream_t s = (cudaStream_t)stream;
    switch (op) {
    case NB200_PN_PREP:
        if (!weights_ok(w) || !a->wtiles || !aligned(a->wtiles)) return NB200_EINVAL;
        return nb_fused_prep(w, a->wtiles, s);
    case NB200_PN_NODE_FWD:
    case NB200_PN_NODE_BWD:
        if (!weights_ok(w) || !a->wtiles || !aligned(a->wtiles)) return NB200_EINVAL;
        return op == NB200_PN_NODE_FWD ? node_fwd(a, s) : node_bwd(a, s);
    case NB200_PN_EMBED:
        if (!w || !all(a->z, w->emb, a->q, a->mu, a->status) || !aligned(w->emb, a->q, a->mu)) return NB200_EINVAL;
        return nb_embed(a->z, w->emb, w->z_offset, w->n_elem, N, a->q, a->mu, a->status, s);
    case NB200_PN_ACT_BWD:
        if (!all(a->g, a->pre) || !aligned(a->g, a->pre) || a->n % 4 != 0 || (a->kind != NB_ACT_SILU && a->kind != NB_ACT_SSP)) return NB200_EINVAL;
        return nb_act_bwd(a->g, a->pre, a->n, a->kind, s);
    case NB200_PN_UPD_COMBINE_BWD:
        if (!all(a->gq, a->gmu, a->y, a->VW, a->gy, a->gVW) || !aligned(a->gq, a->gmu, a->y, a->VW, a->gy, a->gVW)) return NB200_EINVAL;
        return nb_upd_combine_bwd(a->gq, a->gmu, a->y, a->VW, N, a->gy, a->gVW, s);
    case NB200_PN_UPD_NORM_BWD:
        if (!all(a->gn, a->VW, a->nrm, a->gVW) || !aligned(a->gn, a->VW, a->nrm, a->gVW)) return NB200_EINVAL;
        return nb_upd_norm_bwd(a->gn, a->VW, a->nrm, N, a->gVW, s);
    case NB200_PN_READOUT:
        if (!w || !all(a->pre, w->e1, w->R2, w->e2, a->eps_atom)) return NB200_EINVAL;
        return nb_readout(a->pre, w->e1, w->R2, w->e2, N, F / 2, a->eps_atom, s);
    case NB200_PN_MOL_SUM:
        if (!w || !all(a->eps_atom, a->mol_ptr, a->energy)) return NB200_EINVAL;
        return nb_mol_sum(a->eps_atom, a->mol_ptr, a->n_mol, w->energy_shift_per_atom, a->energy, s);
    case NB200_PN_READOUT_BWD:
        if (!w || !all(a->pre, w->R2, a->g_pre)) return NB200_EINVAL;
        return nb_readout_bwd(a->pre, w->R2, N, F / 2, a->g_pre, s);
    case NB200_PN_POISON:
        if (!all(a->status, a->energy)) return NB200_EINVAL;
        return nb_poison_on_error(a->status, a->energy, a->n_mol, a->forces, a->n, s);
    }
    return NB200_EINVAL;
}
