// painn_tangent.cu -- forward-mode tangent kernels for the force-loss term of PaiNN training (SURVEY.md section 8 a10, cfg 3).
//
// The reference gets d/dtheta of a force loss by autograd's double backward (create_graph=True, painn_pyg/painn.py:142).  With
// v = dLoss/dF:   d/dtheta sum_i v_i . F_i = - (v . d/dR) [ dE_tot/dtheta ]   (mixed partials commute): the directional derivative,
// along v in POSITION space, of the first-order parameter gradient the engine already produces.  The weights carry no tangent, so
// every Linear layer of the forward and of the backward is the same GEMM applied to the tangent array; only the pointwise and the
// gather/scatter steps need the product rule.  These kernels are those steps ("t_" / hat = tangent of the quantity of the same name
// in painn_node.cu / painn_msg.cu).  Plain LDG versions (one warp per atom, lane = 4 channels): correctness first -- training is
// GEMM- and launch-bound, see DESIGN.md section 3.7.
#include "common.cuh"
#include "painn_node.cuh"

namespace {

constexpr int TN_THREADS = 256;

__device__ __forceinline__ float d2siluf_(float x) {
    const float s = sigmoidf_(x);
    return s * (1.0f - s) * (2.0f + x * (1.0f - 2.0f * s));
}
__device__ __forceinline__ float4 map4(float4 p, float (*f)(float)) { return make_float4(f(p.x), f(p.y), f(p.z), f(p.w)); }
__device__ __forceinline__ float4 operator-(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float4 div4(float4 a, float4 b) { return make_float4(a.x / b.x, a.y / b.y, a.z / b.z, a.w / b.w); }

// t_geom[e] = (du[3], dd): r = pos_j - pos_i, d = |r|, u = r/d;  dr = v_j - v_i;  dd = u.dr;  du = (dr - u dd)/d
__global__ void __launch_bounds__(TN_THREADS) k_geom_tan(const float* __restrict__ geom, const int32_t* __restrict__ row_ptr,
                                                        const int32_t* __restrict__ col, const float* __restrict__ v, int n_atoms,
                                                        float* __restrict__ t_geom) {
    const int i = blockIdx.x * TN_THREADS + threadIdx.x;
    if (i >= n_atoms) return;
    const float vx = v[3 * i], vy = v[3 * i + 1], vz = v[3 * i + 2];
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
        const int j = col[e];
        const float4 g = ldg4(geom + 4 * (size_t)e);
        const float dx = v[3 * j] - vx, dy = v[3 * j + 1] - vy, dz = v[3 * j + 2] - vz;
        const float dd = g.x * dx + g.y * dy + g.z * dz;
        const float inv = 1.0f / g.w;
        st4(t_geom + 4 * (size_t)e, make_float4((dx - g.x * dd) * inv, (dy - g.y * dd) * inv, (dz - g.z * dd) * inv, dd));
    }
}

// out = f'(pre) * x   (tangent of an activation: act_hat = silu'(pre) * pre_hat)
__global__ void __launch_bounds__(TN_THREADS) k_mul_dact(const float* __restrict__ pre, const float* __restrict__ x, int64_t n4, float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * TN_THREADS + threadIdx.x;
    if (t >= n4) return;
    st4(out + 4 * t, map4(ldg4(pre + 4 * t), dsiluf_) * ldg4(x + 4 * t));
}

// tangent of act_bwd (g_post = g_pre * silu'(p)):  t_g <- t_g * silu'(p) + g_pre * silu''(p) * t_p   (call BEFORE the primal act_bwd)
__global__ void __launch_bounds__(TN_THREADS) k_act_bwd_tan(float* __restrict__ t_g, const float* __restrict__ g_pre, const float* __restrict__ pre,
                                                           const float* __restrict__ t_pre, int64_t n4) {
    const int64_t t = (int64_t)blockIdx.x * TN_THREADS + threadIdx.x;
    if (t >= n4) return;
    const float4 p = ldg4(pre + 4 * t);
    float4 o = *reinterpret_cast<const float4*>(t_g + 4 * t) * map4(p, dsiluf_);
    fma4(o, ldg4(g_pre + 4 * t) * map4(p, d2siluf_), ldg4(t_pre + 4 * t));
    st4(t_g + 4 * t, o);
}

// message forward tangent (painn_msg.cu k_painn_msg_fwd): W_hat = dW * dd of the edge.  WT = storage type of the per-edge rows (common.cuh)
template <class WT>
__global__ void __launch_bounds__(TN_THREADS) k_msg_fwd_tan(const float* __restrict__ xh, const float* __restrict__ t_xh, const float* __restrict__ xh_bias,
                                                           const float* __restrict__ mu, const float* __restrict__ t_mu,
                                                           const WT* __restrict__ W, const WT* __restrict__ dW,
                                                           const float* __restrict__ geom, const float* __restrict__ t_geom,
                                                           const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col, int n_atoms,
                                                           float* t_q, float* __restrict__ t_mu_out, const int32_t* __restrict__ rev) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float4 ba = ldg4(xh_bias + c), bb = ldg4(xh_bias + NB_F + c), bc = ldg4(xh_bias + 2 * NB_F + c);
    float4 dq = f4(0.f), dm0 = f4(0.f), dm1 = f4(0.f), dm2 = f4(0.f);
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
        const int j = col[e];
        const float4 g = ldg4(geom + 4 * (size_t)e), tg = ldg4(t_geom + 4 * (size_t)e);
        const size_t wr = rev ? (size_t)min(e, __ldg(rev + e)) : (size_t)e;  // `rev` given: ONE stored filter row per undirected pair (painn_msg.cu)
        const WT* w = W + wr * 3 * NB_F + c;
        const WT* dw = dW + wr * 3 * NB_F + c;
        const float4 wa = ldw4(w), wb = ldw4(w + NB_F), wc = ldw4(w + 2 * NB_F);
        const float4 ta = ldw4(dw) * tg.w, tb = ldw4(dw + NB_F) * tg.w, tc = ldw4(dw + 2 * NB_F) * tg.w;
        const float* xj = xh + (size_t)j * 3 * NB_F + c;
        const float* txj = t_xh + (size_t)j * 3 * NB_F + c;
        const float4 a = ldg4(xj) + ba, b = ldg4(xj + NB_F) + bb, cc = ldg4(xj + 2 * NB_F) + bc;
        const float4 a_h = ldg4(txj), b_h = ldg4(txj + NB_F), c_h = ldg4(txj + 2 * NB_F);
        const float* mj = mu + (size_t)j * 3 * NB_F + c;
        const float* tmj = t_mu + (size_t)j * 3 * NB_F + c;
        fma4(dq, ta, a); fma4(dq, wa, a_h);
        float4 pb_h = tb * b; fma4(pb_h, wb, b_h);       // (Wb b)^
        float4 pc_h = tc * cc; fma4(pc_h, wc, c_h);      // (Wc c)^
        const float4 pb = wb * b, pc = wc * cc;
        fma4s(dm0, pb_h, g.x); fma4s(dm0, pb, tg.x); fma4(dm0, pc_h, ldg4(mj)); fma4(dm0, pc, ldg4(tmj));
        fma4s(dm1, pb_h, g.y); fma4s(dm1, pb, tg.y); fma4(dm1, pc_h, ldg4(mj + NB_F)); fma4(dm1, pc, ldg4(tmj + NB_F));
        fma4s(dm2, pb_h, g.z); fma4s(dm2, pb, tg.z); fma4(dm2, pc_h, ldg4(mj + 2 * NB_F)); fma4(dm2, pc, ldg4(tmj + 2 * NB_F));
    }
    const size_t qi = (size_t)i * NB_F + c, mi = (size_t)i * 3 * NB_F + c;
    st4(t_q + qi, *reinterpret_cast<const float4*>(t_q + qi) + dq);
    st4(t_mu_out + mi, ldg4(t_mu + mi) + dm0); st4(t_mu_out + mi + NB_F, ldg4(t_mu + mi + NB_F) + dm1);
    st4(t_mu_out + mi + 2 * NB_F, ldg4(t_mu + mi + 2 * NB_F) + dm2);
}

// t_nrm = sum_x V V^ / nrm
__global__ void __launch_bounds__(TN_THREADS) k_upd_norm_tan(const float* __restrict__ VW, const float* __restrict__ t_VW, const float* __restrict__ nrm,
                                                            int n_atoms, float* __restrict__ t_nrm) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    const float* tv = t_VW + (size_t)i * 6 * NB_F + c;
    float4 s = ldg4(v) * ldg4(tv); fma4(s, ldg4(v + 2 * NB_F), ldg4(tv + 2 * NB_F)); fma4(s, ldg4(v + 4 * NB_F), ldg4(tv + 4 * NB_F));
    st4(t_nrm + (size_t)i * NB_F + c, div4(s, ldg4(nrm + (size_t)i * NB_F + c)));
}

// tangent of the update combine q += y0 + y2 S, mu[x] += y1 Wv[x], S = <V, Wv> (y is the stored, biased y; t_y has no bias):
// q^ += y0^ + y2^ S + y2 S^ ; mu^[x] += y1^ Wv[x] + y1 Wv^[x]
__global__ void __launch_bounds__(TN_THREADS) k_upd_combine_tan(float* __restrict__ t_q, float* __restrict__ t_mu, const float* __restrict__ VW,
                                                               const float* __restrict__ t_VW, const float* __restrict__ y,
                                                               const float* __restrict__ t_y, int n_atoms) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float* yi = y + (size_t)i * 3 * NB_F + c;
    const float* tyi = t_y + (size_t)i * 3 * NB_F + c;
    const float4 y1 = ldg4(yi + NB_F), y2 = ldg4(yi + 2 * NB_F), y0_h = ldg4(tyi), y1_h = ldg4(tyi + NB_F), y2_h = ldg4(tyi + 2 * NB_F);
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    const float* tv = t_VW + (size_t)i * 6 * NB_F + c;
    float4 S = f4(0.f), S_h = f4(0.f);
    float* m = t_mu + (size_t)i * 3 * NB_F + c;
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        const float4 V = ldg4(v + x * 2 * NB_F), Wv = ldg4(v + x * 2 * NB_F + NB_F);
        const float4 V_h = ldg4(tv + x * 2 * NB_F), Wv_h = ldg4(tv + x * 2 * NB_F + NB_F);
        fma4(S, V, Wv); fma4(S_h, V_h, Wv); fma4(S_h, V, Wv_h);
        float4 mx = *reinterpret_cast<const float4*>(m + x * NB_F);
        fma4(mx, y1_h, Wv); fma4(mx, y1, Wv_h);
        st4(m + x * NB_F, mx);
    }
    float4 qi = *reinterpret_cast<const float4*>(t_q + (size_t)i * NB_F + c) + y0_h;
    fma4(qi, y2_h, S); fma4(qi, y2, S_h);
    st4(t_q + (size_t)i * NB_F + c, qi);
}

// readout: t_g_pre = R2 silu''(pre) t_pre ;  t_act = silu'(pre) t_pre (operand of d R2)
__global__ void __launch_bounds__(TN_THREADS) k_readout_bwd_tan(const float* __restrict__ pre, const float* __restrict__ t_pre, const float* __restrict__ R2,
                                                               int64_t n, int width, float* __restrict__ t_g_pre, float* __restrict__ t_act) {
    const int64_t t = (int64_t)blockIdx.x * TN_THREADS + threadIdx.x;
    if (t >= n) return;
    const float p = pre[t], tp = t_pre[t];
    t_g_pre[t] = __ldg(R2 + (int)(t % width)) * d2siluf_(p) * tp;
    t_act[t] = dsiluf_(p) * tp;
}

// tangent of k_upd_combine_bwd
__global__ void __launch_bounds__(TN_THREADS) k_upd_combine_bwd_tan(const float* __restrict__ gq, const float* __restrict__ t_gq, const float* __restrict__ gmu,
                                                                   const float* __restrict__ t_gmu, const float* __restrict__ y,
                                                                   const float* __restrict__ t_y, const float* __restrict__ VW,
                                                                   const float* __restrict__ t_VW, int n_atoms, float* __restrict__ t_gy,
                                                                   float* __restrict__ t_gVW) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float4 g = ldg4(gq + (size_t)i * NB_F + c), g_h = ldg4(t_gq + (size_t)i * NB_F + c);
    const float* yi = y + (size_t)i * 3 * NB_F + c;
    const float* tyi = t_y + (size_t)i * 3 * NB_F + c;
    const float4 y1 = ldg4(yi + NB_F), y2 = ldg4(yi + 2 * NB_F), y1_h = ldg4(tyi + NB_F), y2_h = ldg4(tyi + 2 * NB_F);
    const float4 gS = g * y2;
    float4 gS_h = g_h * y2; fma4(gS_h, g, y2_h);
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    const float* tv = t_VW + (size_t)i * 6 * NB_F + c;
    const float* gm = gmu + (size_t)i * 3 * NB_F + c;
    const float* tgm = t_gmu + (size_t)i * 3 * NB_F + c;
    float* gv = t_gVW + (size_t)i * 6 * NB_F + c;
    float4 S = f4(0.f), S_h = f4(0.f), gy1_h = f4(0.f);
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        const float4 V = ldg4(v + x * 2 * NB_F), Wv = ldg4(v + x * 2 * NB_F + NB_F);
        const float4 V_h = ldg4(tv + x * 2 * NB_F), Wv_h = ldg4(tv + x * 2 * NB_F + NB_F);
        const float4 h = ldg4(gm + x * NB_F), h_h = ldg4(tgm + x * NB_F);
        fma4(S, V, Wv); fma4(S_h, V_h, Wv); fma4(S_h, V, Wv_h);
        fma4(gy1_h, h_h, Wv); fma4(gy1_h, h, Wv_h);
        float4 gV_h = gS_h * Wv; fma4(gV_h, gS, Wv_h);
        st4(gv + x * 2 * NB_F, gV_h);
        float4 gW_h = h_h * y1; fma4(gW_h, h, y1_h); fma4(gW_h, gS_h, V); fma4(gW_h, gS, V_h);
        st4(gv + x * 2 * NB_F + NB_F, gW_h);
    }
    float* go = t_gy + (size_t)i * 3 * NB_F + c;
    float4 gy2_h = g_h * S; fma4(gy2_h, g, S_h);
    st4(go, g_h); st4(go + NB_F, gy1_h); st4(go + 2 * NB_F, gy2_h);
}

// tangent of k_upd_norm_bwd: gV^[x] += gn^ V/n + gn V^/n - gn V n^/n^2
__global__ void __launch_bounds__(TN_THREADS) k_upd_norm_bwd_tan(const float* __restrict__ gn, const float* __restrict__ t_gn, const float* __restrict__ VW,
                                                                const float* __restrict__ t_VW, const float* __restrict__ nrm,
                                                                const float* __restrict__ t_nrm, int n_atoms, float* __restrict__ t_gVW) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int i = t >> 5, c = (t & 31) * 4;
    if (i >= n_atoms) return;
    const float4 n = ldg4(nrm + (size_t)i * NB_F + c), n_h = ldg4(t_nrm + (size_t)i * NB_F + c);
    const float4 g = ldg4(gn + (size_t)i * NB_F + c), g_h = ldg4(t_gn + (size_t)i * NB_F + c);
    const float4 s = div4(g, n);                         // gn / n
    const float4 s_h = div4(g_h - s * n_h, n);           // (gn/n)^ = (gn^ - (gn/n) n^) / n
    const float* v = VW + (size_t)i * 6 * NB_F + c;
    const float* tv = t_VW + (size_t)i * 6 * NB_F + c;
    float* gv = t_gVW + (size_t)i * 6 * NB_F + c;
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        float4 o = *reinterpret_cast<const float4*>(gv + x * 2 * NB_F);
        fma4(o, s_h, ldg4(v + x * 2 * NB_F)); fma4(o, s, ldg4(tv + x * 2 * NB_F));
        st4(gv + x * 2 * NB_F, o);
    }
}

// message backward tangent (by source atom j, slot e carries the opposite edge; painn_msg.cu k_painn_msg_bwd).  Also writes, per slot,
//   t_gW[e]  = tangent of the per-edge filter gradient,   gWd[e] = (unseeded filter gradient) * dd_e
// the two operands of the filter-weight gradient tangent (k_filter_wgrad_tan).
// HVP = true (Hessian-vector product, fp32 rows): no filter-gradient operands; instead the tangent of the per-edge geometric gradient
// egrad[e] = (dE/du'[3], dE/dd) the primal kernel accumulates is ADDED to t_egrad[e] (one lane per slot, layers run in order: deterministic):
//   dE/dd^    = sum_ch d2W dd fW + dW fW^          (fW = the per-edge filter gradient above, d2W = d2W/dd2 of the row)
//   dE/du'^[x] = sum_ch (Wb b)^ gmu_i[x] + (Wb b) gmu_i^[x]
template <class WT, bool HVP = false>
__global__ void __launch_bounds__(TN_THREADS) k_msg_bwd_tan(const float* __restrict__ xh, const float* __restrict__ t_xh, const float* __restrict__ xh_bias,
                                                           const float* __restrict__ mu, const float* __restrict__ t_mu,
                                                           const WT* __restrict__ W, const WT* __restrict__ dW,
                                                           const float* __restrict__ geom, const float* __restrict__ t_geom,
                                                           const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col, int n_atoms,
                                                           const float* __restrict__ g_q, const float* __restrict__ t_g_q,
                                                           const float* __restrict__ g_mu, const float* __restrict__ t_g_mu,
                                                           float* __restrict__ t_g_xh, float* __restrict__ t_g_mu_in, WT* __restrict__ t_gW,
                                                           WT* __restrict__ gWd, const int32_t* __restrict__ rev, const float* __restrict__ d2W = nullptr,
                                                           float* __restrict__ t_egrad = nullptr) {
    const int t = blockIdx.x * TN_THREADS + threadIdx.x;
    const int j = t >> 5, c = (t & 31) * 4;
    if (j >= n_atoms) return;
    const float* xj = xh + (size_t)j * 3 * NB_F + c;
    const float* txj = t_xh + (size_t)j * 3 * NB_F + c;
    const float4 a = ldg4(xj) + ldg4(xh_bias + c), b = ldg4(xj + NB_F) + ldg4(xh_bias + NB_F + c), cc = ldg4(xj + 2 * NB_F) + ldg4(xh_bias + 2 * NB_F + c);
    const float4 a_h = ldg4(txj), b_h = ldg4(txj + NB_F), c_h = ldg4(txj + 2 * NB_F);
    const float* mj = mu + (size_t)j * 3 * NB_F + c;
    const float* tmj = t_mu + (size_t)j * 3 * NB_F + c;
    const float4 m0 = ldg4(mj), m1 = ldg4(mj + NB_F), m2 = ldg4(mj + 2 * NB_F);
    const float4 m0_h = ldg4(tmj), m1_h = ldg4(tmj + NB_F), m2_h = ldg4(tmj + 2 * NB_F);
    float4 ga = f4(0.f), gb = f4(0.f), gc = f4(0.f), gm0 = f4(0.f), gm1 = f4(0.f), gm2 = f4(0.f);
    for (int e = row_ptr[j]; e < row_ptr[j + 1]; ++e) {
        const int i = col[e];
        const float4 g = ldg4(geom + 4 * (size_t)e), tg = ldg4(t_geom + 4 * (size_t)e);  // u' = -u, u'^ = -u^, dd' = dd
        const size_t wr = rev ? (size_t)min(e, __ldg(rev + e)) : (size_t)e;
        const WT* w = W + wr * 3 * NB_F + c;
        const WT* dw = dW + wr * 3 * NB_F + c;
        const float4 wa = ldw4(w), wb = ldw4(w + NB_F), wc = ldw4(w + 2 * NB_F);
        const float4 wa_h = ldw4(dw) * tg.w, wb_h = ldw4(dw + NB_F) * tg.w, wc_h = ldw4(dw + 2 * NB_F) * tg.w;
        const float4 gq = ldg4(g_q + (size_t)i * NB_F + c), gq_h = ldg4(t_g_q + (size_t)i * NB_F + c);
        const float* gmi = g_mu + (size_t)i * 3 * NB_F + c;
        const float* tgmi = t_g_mu + (size_t)i * 3 * NB_F + c;
        const float4 h0 = ldg4(gmi), h1 = ldg4(gmi + NB_F), h2 = ldg4(gmi + 2 * NB_F);
        const float4 h0_h = ldg4(tgmi), h1_h = ldg4(tgmi + NB_F), h2_h = ldg4(tgmi + 2 * NB_F);
        float4 tb = h0 * (-g.x); fma4s(tb, h1, -g.y); fma4s(tb, h2, -g.z);
        float4 tb_h = h0_h * (-g.x); fma4s(tb_h, h1_h, -g.y); fma4s(tb_h, h2_h, -g.z);
        fma4s(tb_h, h0, -tg.x); fma4s(tb_h, h1, -tg.y); fma4s(tb_h, h2, -tg.z);
        float4 tc = h0 * m0; fma4(tc, h1, m1); fma4(tc, h2, m2);
        float4 tc_h = h0_h * m0; fma4(tc_h, h1_h, m1); fma4(tc_h, h2_h, m2);
        fma4(tc_h, h0, m0_h); fma4(tc_h, h1, m1_h); fma4(tc_h, h2, m2_h);
        fma4(ga, wa_h, gq); fma4(ga, wa, gq_h);
        fma4(gb, wb_h, tb); fma4(gb, wb, tb_h);
        fma4(gc, wc_h, tc); fma4(gc, wc, tc_h);
        const float4 pc = wc * cc;
        float4 pc_h = wc_h * cc; fma4(pc_h, wc, c_h);
        fma4(gm0, pc_h, h0); fma4(gm0, pc, h0_h);
        fma4(gm1, pc_h, h1); fma4(gm1, pc, h1_h);
        fma4(gm2, pc_h, h2); fma4(gm2, pc, h2_h);
        // per-edge filter gradient (slot e <- opposite edge) and its tangent
        const float4 fa = a * gq, fb = b * tb, fc = cc * tc;
        float4 fa_h = a_h * gq; fma4(fa_h, a, gq_h);
        float4 fb_h = b_h * tb; fma4(fb_h, b, tb_h);
        float4 fc_h = c_h * tc; fma4(fc_h, cc, tc_h);
        if (!HVP) {
            WT* o = t_gW + (size_t)e * 3 * NB_F + c;
            stw4(o, fa_h); stw4(o + NB_F, fb_h); stw4(o + 2 * NB_F, fc_h);
            WT* o2 = gWd + (size_t)e * 3 * NB_F + c;
            stw4(o2, fa * tg.w); stw4(o2 + NB_F, fb * tg.w); stw4(o2 + 2 * NB_F, fc * tg.w);
        } else {
            const float* d2 = d2W + wr * 3 * NB_F + c;
            float4 sd = ldg4(d2) * fa; fma4(sd, ldg4(d2 + NB_F), fb); fma4(sd, ldg4(d2 + 2 * NB_F), fc);
            sd = sd * tg.w;
            fma4(sd, ldw4(dw), fa_h); fma4(sd, ldw4(dw + NB_F), fb_h); fma4(sd, ldw4(dw + 2 * NB_F), fc_h);
            const float4 pb = wb * b;
            float4 pb_h = wb_h * b; fma4(pb_h, wb, b_h);
            float4 u0 = pb_h * h0; fma4(u0, pb, h0_h);
            float4 u1 = pb_h * h1; fma4(u1, pb, h1_h);
            float4 u2 = pb_h * h2; fma4(u2, pb, h2_h);
            float r0 = hsum4(u0), r1 = hsum4(u1), r2 = hsum4(u2), r3 = hsum4(sd);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                r0 += __shfl_xor_sync(0xffffffffu, r0, o); r1 += __shfl_xor_sync(0xffffffffu, r1, o);
                r2 += __shfl_xor_sync(0xffffffffu, r2, o); r3 += __shfl_xor_sync(0xffffffffu, r3, o);
            }
            if ((t & 31) == 0) {
                float* te = t_egrad + 4 * (size_t)e;
                st4(te, *reinterpret_cast<const float4*>(te) + make_float4(r0, r1, r2, r3));
            }
        }
    }
    float* gx = t_g_xh + (size_t)j * 3 * NB_F + c;
    st4(gx, ga); st4(gx + NB_F, gb); st4(gx + 2 * NB_F, gc);
    const float* tgmj = t_g_mu + (size_t)j * 3 * NB_F + c;
    float* go = t_g_mu_in + (size_t)j * 3 * NB_F + c;
    st4(go, ldg4(tgmj) + gm0); st4(go + NB_F, ldg4(tgmj + NB_F) + gm1); st4(go + 2 * NB_F, ldg4(tgmj + 2 * NB_F) + gm2);
}

// Tangent of the force assembly (painn_msg.cu k_edge_forces): hv = H v = -F^.  Slot e holds eg = (gu[3], gd) of the opposite edge e',
// u' = -u_e, with  G = P/d + gd u',  P = gu - (gu.u') u':
//   G^ = P^/d - P d^/d^2 + gd^ u' + gd u'^,   P^ = gu^ - (gu^.u' + gu.u'^) u' - (gu.u') u'^
// One thread per atom over its own CSR row, like the primal: no atomics, bitwise repeatable.
__device__ __forceinline__ float3 edge_G_tan(const float4 eg, const float4 t_eg, const float4 g, const float4 t_g) {
    const float ux = -g.x, uy = -g.y, uz = -g.z, tux = -t_g.x, tuy = -t_g.y, tuz = -t_g.z;
    const float inv = 1.0f / g.w, t_d = t_g.w;
    const float dot = eg.x * ux + eg.y * uy + eg.z * uz;
    const float t_dot = t_eg.x * ux + t_eg.y * uy + t_eg.z * uz + eg.x * tux + eg.y * tuy + eg.z * tuz;
    const float px = eg.x - dot * ux, py = eg.y - dot * uy, pz = eg.z - dot * uz;
    const float tpx = t_eg.x - t_dot * ux - dot * tux, tpy = t_eg.y - t_dot * uy - dot * tuy, tpz = t_eg.z - t_dot * uz - dot * tuz;
    const float s = t_d * inv * inv;
    return make_float3(tpx * inv - px * s + t_eg.w * ux + eg.w * tux, tpy * inv - py * s + t_eg.w * uy + eg.w * tuy,
                       tpz * inv - pz * s + t_eg.w * uz + eg.w * tuz);
}

__global__ void __launch_bounds__(TN_THREADS) k_edge_forces_hvp(const float* __restrict__ egrad, const float* __restrict__ t_egrad,
                                                               const float* __restrict__ geom, const float* __restrict__ t_geom,
                                                               const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ rev, int n_atoms,
                                                               float* __restrict__ hv) {
    const int j = blockIdx.x * TN_THREADS + threadIdx.x;
    if (j >= n_atoms) return;
    float hx = 0.f, hy = 0.f, hz = 0.f;
    for (int e = row_ptr[j]; e < row_ptr[j + 1]; ++e) {
        const int r = rev[e];
        const float3 g1 = edge_G_tan(ldg4(egrad + 4 * (size_t)e), ldg4(t_egrad + 4 * (size_t)e), ldg4(geom + 4 * (size_t)e), ldg4(t_geom + 4 * (size_t)e));
        const float3 g2 = edge_G_tan(ldg4(egrad + 4 * (size_t)r), ldg4(t_egrad + 4 * (size_t)r), ldg4(geom + 4 * (size_t)r), ldg4(t_geom + 4 * (size_t)r));
        hx += g1.x - g2.x; hy += g1.y - g2.y; hz += g1.z - g2.z;
    }
    hv[3 * (size_t)j] = hx; hv[3 * (size_t)j + 1] = hy; hv[3 * (size_t)j + 2] = hz;
}

}  // namespace

static inline int tn_grid(int64_t n) { return (int)((n + TN_THREADS - 1) / TN_THREADS); }

int nb_geom_tan(const float* geom, const int32_t* row_ptr, const int32_t* col, const float* v, int n_atoms, float* t_geom, cudaStream_t s) {
    k_geom_tan<<<tn_grid(n_atoms), TN_THREADS, 0, s>>>(geom, row_ptr, col, v, n_atoms, t_geom);
    return nb_check_launch();
}
int nb_mul_dact(const float* pre, const float* x, int64_t n, float* out, cudaStream_t s) {
    k_mul_dact<<<tn_grid(n / 4), TN_THREADS, 0, s>>>(pre, x, n / 4, out);
    return nb_check_launch();
}
int nb_act_bwd_tan(float* t_g, const float* g_pre, const float* pre, const float* t_pre, int64_t n, cudaStream_t s) {
    k_act_bwd_tan<<<tn_grid(n / 4), TN_THREADS, 0, s>>>(t_g, g_pre, pre, t_pre, n / 4);
    return nb_check_launch();
}
int nb_msg_fwd_tan(const float* xh, const float* t_xh, const float* xh_bias, const float* mu, const float* t_mu, const float* W, const float* dW,
                   const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* col, int n_atoms, float* t_q, float* t_mu_out,
                   cudaStream_t s, int bf16, const int32_t* rev) {
    if (bf16)
        k_msg_fwd_tan<nb_bf16><<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(xh, t_xh, xh_bias, mu, t_mu, reinterpret_cast<const nb_bf16*>(W),
                                                                                    reinterpret_cast<const nb_bf16*>(dW), geom, t_geom, row_ptr, col, n_atoms, t_q,
                                                                                    t_mu_out, rev);
    else
        k_msg_fwd_tan<float><<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(xh, t_xh, xh_bias, mu, t_mu, W, dW, geom, t_geom, row_ptr, col, n_atoms, t_q,
                                                                                  t_mu_out, rev);
    return nb_check_launch();
}
int nb_upd_norm_tan(const float* VW, const float* t_VW, const float* nrm, int n_atoms, float* t_nrm, cudaStream_t s) {
    k_upd_norm_tan<<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(VW, t_VW, nrm, n_atoms, t_nrm);
    return nb_check_launch();
}
int nb_upd_combine_tan(float* t_q, float* t_mu, const float* VW, const float* t_VW, const float* y, const float* t_y, int n_atoms, cudaStream_t s) {
    k_upd_combine_tan<<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(t_q, t_mu, VW, t_VW, y, t_y, n_atoms);
    return nb_check_launch();
}
int nb_readout_bwd_tan(const float* pre, const float* t_pre, const float* R2, int n_atoms, int width, float* t_g_pre, float* t_act, cudaStream_t s) {
    const int64_t n = (int64_t)n_atoms * width;
    k_readout_bwd_tan<<<tn_grid(n), TN_THREADS, 0, s>>>(pre, t_pre, R2, n, width, t_g_pre, t_act);
    return nb_check_launch();
}
int nb_upd_combine_bwd_tan(const float* gq, const float* t_gq, const float* gmu, const float* t_gmu, const float* y, const float* t_y, const float* VW,
                           const float* t_VW, int n_atoms, float* t_gy, float* t_gVW, cudaStream_t s) {
    k_upd_combine_bwd_tan<<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(gq, t_gq, gmu, t_gmu, y, t_y, VW, t_VW, n_atoms, t_gy, t_gVW);
    return nb_check_launch();
}
int nb_upd_norm_bwd_tan(const float* gn, const float* t_gn, const float* VW, const float* t_VW, const float* nrm, const float* t_nrm, int n_atoms,
                        float* t_gVW, cudaStream_t s) {
    k_upd_norm_bwd_tan<<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(gn, t_gn, VW, t_VW, nrm, t_nrm, n_atoms, t_gVW);
    return nb_check_launch();
}
int nb_msg_bwd_tan(const float* xh, const float* t_xh, const float* xh_bias, const float* mu, const float* t_mu, const float* W, const float* dW,
                   const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* col, int n_atoms, const float* g_q,
                   const float* t_g_q, const float* g_mu, const float* t_g_mu, float* t_g_xh, float* t_g_mu_in, float* t_gW, float* gWd,
                   cudaStream_t s, int bf16, const int32_t* rev) {
    if (bf16)
        k_msg_bwd_tan<nb_bf16><<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(
            xh, t_xh, xh_bias, mu, t_mu, reinterpret_cast<const nb_bf16*>(W), reinterpret_cast<const nb_bf16*>(dW), geom, t_geom, row_ptr, col, n_atoms, g_q, t_g_q,
            g_mu, t_g_mu, t_g_xh, t_g_mu_in, reinterpret_cast<nb_bf16*>(t_gW), reinterpret_cast<nb_bf16*>(gWd), rev);
    else
        k_msg_bwd_tan<float><<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(xh, t_xh, xh_bias, mu, t_mu, W, dW, geom, t_geom, row_ptr, col, n_atoms, g_q,
                                                                                  t_g_q, g_mu, t_g_mu, t_g_xh, t_g_mu_in, t_gW, gWd, rev);
    return nb_check_launch();
}
int nb_msg_bwd_hvp(const float* xh, const float* t_xh, const float* xh_bias, const float* mu, const float* t_mu, const float* W, const float* dW,
                   const float* d2W, const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* col, const int32_t* rev, int n_atoms,
                   const float* g_q, const float* t_g_q, const float* g_mu, const float* t_g_mu, float* t_g_xh, float* t_g_mu_in, float* t_egrad,
                   cudaStream_t s) {
    k_msg_bwd_tan<float, true><<<tn_grid((int64_t)n_atoms * 32), TN_THREADS, 0, s>>>(xh, t_xh, xh_bias, mu, t_mu, W, dW, geom, t_geom, row_ptr, col, n_atoms,
                                                                                    g_q, t_g_q, g_mu, t_g_mu, t_g_xh, t_g_mu_in, nullptr, nullptr, rev, d2W,
                                                                                    t_egrad);
    return nb_check_launch();
}
int nb_edge_forces_hvp(const float* egrad, const float* t_egrad, const float* geom, const float* t_geom, const int32_t* row_ptr, const int32_t* rev,
                       int n_atoms, float* hv, cudaStream_t s) {
    k_edge_forces_hvp<<<tn_grid(n_atoms), TN_THREADS, 0, s>>>(egrad, t_egrad, geom, t_geom, row_ptr, rev, n_atoms, hv);
    return nb_check_launch();
}
