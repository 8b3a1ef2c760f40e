// painn_msg.cu -- PaiNN message + segmented scatter (K_msg), forward and analytic backward.
//
// Replaces  schnetpack PaiNNInteraction.forward (SURVEY.md A.2; config/model/painn.yaml) and
//           PaiNNMessage.forward/message/aggregate (nablaDFT/painn_pyg/painn.py:475-509):
//   gather xh[j], mu[j] -> multiply by the per-edge filter -> two scatter-adds (atomics) ->
//   residual add, with [E,384] / [E,3,128] temporaries in HBM.
// Here: one warp per atom, lane = 4 channels (float4), CSR rows streamed once, the sums are
// carried in registers and written once -- deterministic, no atomics, no temporaries.
//
// Canonical chunk roles (host permutes PaiNN-OC weights into them):
//   (a, b, c) = split(xh_j + bias),  (Wa, Wb, Wc) = split(W_e)
//   dq_i  = sum_e Wa*a ;  dmu_i[x] = sum_e (Wb*b) u_e[x] + (Wc*c) * mu_j[x]
//
// Algorithmic HBM bytes (SURVEY.md section 8d, definition A), F = 128, fp32:
//   forward : N*10F*4 + E*(3F*4 + 20)           = 5120 N + 1556 E
//   backward: N*16F*4 + E*(6F*4 + 32)           = 8192 N + 3104 E
#include "common.cuh"

// One warp per CTA (16 CTAs per SM): a CTA's shared memory and registers return to the SM as soon as ITS atom is done.  With 8 warps per
// CTA the slot was held until the slowest of 8 atoms (degrees 15..40) finished.
#define MSG_WARPS 1
#define MSG_THREADS (MSG_WARPS * 32)

// The v0 kernels (plain LDG for the filter rows) were latency-bound: low DRAM
// throughput with most stalls on long_scoreboard and ~3 loads in flight per warp.  v1 streams the filter rows -- the only HBM
// stream -- through a per-warp cp.async ring in shared memory: every lane prefetches its own
// 16-byte column of the next STAGES-1 edges, so ~100 KB of HBM requests stay in flight per SM
// without holding registers, and the gathers of the current edge overlap that stream.
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// Forward (v4): two rings per warp with independent depths.
//   * filter rows (the HBM stream, microsecond-scale loaded latency): FWD_WS = 5 stages, filled by the TMA engine --
//     one elected lane issues a 1536-byte `cp.async.bulk` per edge, completion on a per-stage mbarrier;
//   * gathered neighbour rows xh[j], mu[j] (L2): FWD_GS = 2 stages of per-lane cp.async (LDGSTS).
// cp.async groups retire in order, so one shared queue cannot give the two streams different depths (v2 had 3 / 3
// and reached 64 % of the HBM roofline; bytes of the HBM stream in flight were the limiter, not issue slots -- v3).
#define FWD_WS 5
#define FWD_GS 2
#define FWD_WROW (3 * NB_F)
#define FWD_GROW (6 * NB_F)
#define FWD_WARP_FLOATS (FWD_WS * FWD_WROW + FWD_GS * FWD_GROW)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(float* dst, const float* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ void fwd_gather_issue(float* dst, const float* xrow, const float* mrow) {
    cp_async16(dst, xrow); cp_async16(dst + NB_F, xrow + NB_F); cp_async16(dst + 2 * NB_F, xrow + 2 * NB_F);
    cp_async16(dst + 3 * NB_F, mrow); cp_async16(dst + 4 * NB_F, mrow + NB_F); cp_async16(dst + 5 * NB_F, mrow + 2 * NB_F);
}

// WT: storage type of the filter rows (float / nb_bf16); a ring stage keeps its fp32 size, a bf16 row fills the first half of it
template <class WT>
__global__ void __launch_bounds__(MSG_THREADS, 16) k_painn_msg_fwd(const float* __restrict__ xh, const float* __restrict__ xh_bias,
                                                                 const float* q, const float* __restrict__ mu,
                                                                 const WT* __restrict__ W, const float* __restrict__ geom,
                                                                 const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                                                 int n_atoms, float* q_out, float* __restrict__ mu_out, int wstride,
                                                                 const int32_t* __restrict__ rev) {
    // filter row of edge e: row e of `W` (rows of `wstride` floats), or -- `rev` given -- row min(e, rev[e]): ONE stored row per undirected
    // pair (the filter depends on the distance only; filter.cu then evaluates only the canonical edges)
    extern __shared__ __align__(128) float ring_dyn[];  // [warps][WS x W row | GS x gather row], then the mbarriers
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = blockIdx.x * MSG_WARPS + warp;
    if (i >= n_atoms) return;  // no block-level barrier below: a whole warp may leave
    const int c = lane * 4;
    float* wring = ring_dyn + warp * FWD_WARP_FLOATS;
    float* gring = wring + FWD_WS * FWD_WROW + c;  // my 16-byte column of every gathered row
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring_dyn + MSG_WARPS * FWD_WARP_FLOATS) + warp * FWD_WS;
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < FWD_WS; ++s) mbar_init(bars + s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#pragma unroll
        for (int s = 0; s < FWD_WS; ++s)
            if (e0 + s < e1) {
                mbar_expect_tx(bars + s, FWD_WROW * sizeof(WT));
                const int wr = rev ? min(e0 + s, __ldg(rev + e0 + s)) : e0 + s;
                bulk_g2s(wring + s * FWD_WROW, reinterpret_cast<const float*>(W + (size_t)wr * wstride), FWD_WROW * sizeof(WT), bars + s);
            }
    }
    int wr_pf = (e0 + FWD_WS < e1) ? (rev ? min(e0 + FWD_WS, __ldg(rev + e0 + FWD_WS)) : e0 + FWD_WS) : 0;  // row of the filter copy issued next
    const float* xcol = xh + c;
    const float* mcol = mu + c;
#pragma unroll
    for (int s = 0; s < FWD_GS; ++s) {
        if (e0 + s < e1) {
            const int j = __ldg(col + e0 + s);
            fwd_gather_issue(gring + s * FWD_GROW, xcol + (size_t)j * (3 * NB_F), mcol + (size_t)j * (3 * NB_F));
        }
        cp_async_commit();
    }
    __syncwarp();
    const float4 ba = ldg4(xh_bias + c), bb = ldg4(xh_bias + NB_F + c), bc = ldg4(xh_bias + 2 * NB_F + c);
    float4 dq = f4(0.f), dm0 = f4(0.f), dm1 = f4(0.f), dm2 = f4(0.f);
    int j_pf = (e0 + FWD_GS < e1) ? __ldg(col + e0 + FWD_GS) : 0;  // source of the edge whose gather is issued next
    float4 gn = (e0 < e1) ? ldg4(geom + 4 * (size_t)e0) : f4(0.f);
    int wslot = 0, gslot = 0;
    uint32_t wpar = 0;
    for (int e = e0; e < e1; ++e) {
        const float4 g = gn;
        if (e + 1 < e1) gn = ldg4(geom + 4 * (size_t)(e + 1));
        const int j_issue = j_pf;
        if (e + FWD_GS + 1 < e1) j_pf = __ldg(col + e + FWD_GS + 1);
        const int wr_issue = wr_pf;
        if (e + FWD_WS + 1 < e1) wr_pf = rev ? min(e + FWD_WS + 1, __ldg(rev + e + FWD_WS + 1)) : e + FWD_WS + 1;
        cp_async_wait<FWD_GS - 1>();     // my columns of xh[j], mu[j] of edge e have landed
        mbar_wait(bars + wslot, wpar);   // the filter row of edge e has landed
        const WT* wrow = reinterpret_cast<const WT*>(wring + wslot * FWD_WROW) + c;
        float* grow = gring + gslot * FWD_GROW;
        const float4 wa = ldw4_plain(wrow), wb = ldw4_plain(wrow + NB_F), wc = ldw4_plain(wrow + 2 * NB_F);
        const float4 a = lds4(grow) + ba, b = lds4(grow + NB_F) + bb, cc = lds4(grow + 2 * NB_F) + bc;
        const float4 m0 = lds4(grow + 3 * NB_F), m1 = lds4(grow + 4 * NB_F), m2 = lds4(grow + 5 * NB_F);
        fma4(dq, wa, a);
        const float4 pb = wb * b, pc = wc * cc;
        fma4s(dm0, pb, g.x); fma4(dm0, pc, m0);
        fma4s(dm1, pb, g.y); fma4(dm1, pc, m1);
        fma4s(dm2, pb, g.z); fma4(dm2, pc, m2);
        __syncwarp();  // every lane has read the filter stage before the TMA engine may overwrite it
        if (lane == 0 && e + FWD_WS < e1) {
            mbar_expect_tx(bars + wslot, FWD_WROW * sizeof(WT));
            bulk_g2s(wring + wslot * FWD_WROW, reinterpret_cast<const float*>(W + (size_t)wr_issue * wstride), FWD_WROW * sizeof(WT), bars + wslot);
        }
        if (e + FWD_GS < e1) fwd_gather_issue(grow, xcol + (size_t)j_issue * (3 * NB_F), mcol + (size_t)j_issue * (3 * NB_F));
        cp_async_commit();
        if (++wslot == FWD_WS) { wslot = 0; wpar ^= 1u; }
        gslot = (gslot + 1 == FWD_GS) ? 0 : gslot + 1;
    }
    cp_async_wait<0>();
    const size_t qi = (size_t)i * NB_F + c, mi = (size_t)i * (3 * NB_F) + c;
    st4(q_out + qi, *reinterpret_cast<const float4*>(q + qi) + dq);  // q_out may alias q (own row only)
    st4(mu_out + mi, ldg4(mu + mi) + dm0);
    st4(mu_out + mi + NB_F, ldg4(mu + mi + NB_F) + dm1);
    st4(mu_out + mi + 2 * NB_F, ldg4(mu + mi + 2 * NB_F) + dm2);
}

// Backward, organised by SOURCE atom j.  For e in CSR row j (target j, source i = col[e]) the
// opposite edge e' = (j -> i) has the same filter row (W depends on d only) and unit vector -u_e,
// so every quantity of e' is available while streaming row j contiguously:
//   g_a_j += Wa * gq_i ;  g_b_j += Wb * (gmu_i . u') ;  g_c_j += Wc * sum_x gmu_i[x]*mu_j[x]
//   g_mu_j[x] += (Wc*c_j) * gmu_i[x]
//   dE/dd(e')   = sum_ch dWa*(a_j*gq_i) + dWb*(b_j*(gmu_i.u')) + dWc*(c_j*sum_x gmu_i[x] mu_j[x])
//   dE/du'(e')[x] = sum_ch (Wb*b_j) * gmu_i[x]
// The four edge scalars are warp-reduced and accumulated into egrad[e] (slot of e, values of e').
// Backward v3: two rings per warp like the forward (v4).  v2 streamed (W, dW) through a 3-stage cp.async ring but gathered the far atom's
// gradient rows g_q[i], g_mu[i] (2 KB per edge) with plain loads at the top of every iteration: the profile showed low DRAM and issue utilisation,
// 7 warp-cycles of long_scoreboard per issue -- one L2 round trip per edge on the critical path, and at 122 registers no room to pipeline
// them in registers.  Now: (W, dW) rows by TMA bulk copies (one elected lane, BWD_WS = 3 stages x 3 KB, mbarrier per stage) and the
// gathered gradient rows by per-lane cp.async into a second ring (BWD_GS = 2 stages x 2 KB).  13 KB per warp, 104 KB per CTA, 2 CTAs/SM.
#define BWD_WS 3
#define BWD_GS 2
#define BWD_WROW (6 * NB_F)
#define BWD_GROW (4 * NB_F)
#define BWD_WARP_FLOATS (BWD_WS * BWD_WROW + BWD_GS * BWD_GROW)

__device__ __forceinline__ void bwd_gather_issue(float* dst, const float* gq_row, const float* gmu_row) {
    cp_async16(dst, gq_row); cp_async16(dst + NB_F, gmu_row); cp_async16(dst + 2 * NB_F, gmu_row + NB_F); cp_async16(dst + 3 * NB_F, gmu_row + 2 * NB_F);
}

template <bool WRITE_GW, class WT>
__global__ void __launch_bounds__(MSG_THREADS, 16) k_painn_msg_bwd(const float* __restrict__ xh, const float* __restrict__ xh_bias,
                                                                 const float* __restrict__ mu, const WT* __restrict__ W,
                                                                 const WT* __restrict__ dW, const float* __restrict__ geom,
                                                                 const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                                                 int n_atoms, const float* __restrict__ g_q, const float* __restrict__ g_mu,
                                                                 float* __restrict__ g_xh, float* __restrict__ g_mu_in,
                                                                 float* __restrict__ egrad, WT* __restrict__ gW,
                                                                 const float* __restrict__ seed_atom, int wstride, const int32_t* __restrict__ rev) {
    // wstride == 6F: ONE [W | dW/dd] record of 3 KB per edge in `W` (one bulk copy per edge instead of two: the TMA engine is paced by the
    // number of copies); `rev` given: row min(e, rev[e]) -- see the forward kernel
    extern __shared__ __align__(128) float ring_dyn[];  // [warps][WS x (W | dW) row | GS x (g_q | g_mu) row], then the mbarriers
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * MSG_WARPS + warp;
    if (j >= n_atoms) return;
    const int c = lane * 4;
    float* wring = ring_dyn + warp * BWD_WARP_FLOATS;
    float* gring = wring + BWD_WS * BWD_WROW + c;  // my 16-byte column of every gathered row
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring_dyn + MSG_WARPS * BWD_WARP_FLOATS) + warp * BWD_WS;
    const int e0 = row_ptr[j], e1 = row_ptr[j + 1];
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < BWD_WS; ++s) mbar_init(bars + s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#pragma unroll
        for (int s = 0; s < BWD_WS; ++s)
            if (e0 + s < e1) {
                mbar_expect_tx(bars + s, BWD_WROW * sizeof(WT));
                const int wr = rev ? min(e0 + s, __ldg(rev + e0 + s)) : e0 + s;
                WT* stage = reinterpret_cast<WT*>(wring + s * BWD_WROW);
                if (wstride == BWD_WROW) {
                    bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr * BWD_WROW), BWD_WROW * sizeof(WT), bars + s);
                } else {
                    bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr * (3 * NB_F)), 3 * NB_F * sizeof(WT), bars + s);
                    bulk_g2s(reinterpret_cast<float*>(stage + 3 * NB_F), reinterpret_cast<const float*>(dW + (size_t)wr * (3 * NB_F)), 3 * NB_F * sizeof(WT),
                             bars + s);
                }
            }
    }
    int wr_pf = (e0 + BWD_WS < e1) ? (rev ? min(e0 + BWD_WS, __ldg(rev + e0 + BWD_WS)) : e0 + BWD_WS) : 0;
    const float* gqcol = g_q + c;
    const float* gmcol = g_mu + c;
#pragma unroll
    for (int s = 0; s < BWD_GS; ++s) {
        if (e0 + s < e1) {
            const int i = __ldg(col + e0 + s);
            bwd_gather_issue(gring + s * BWD_GROW, gqcol + (size_t)i * NB_F, gmcol + (size_t)i * (3 * NB_F));
        }
        cp_async_commit();
    }
    __syncwarp();
    const float* xj = xh + (size_t)j * (3 * NB_F) + c;
    const float4 a = ldg4(xj) + ldg4(xh_bias + c), b = ldg4(xj + NB_F) + ldg4(xh_bias + NB_F + c),
                 cc = ldg4(xj + 2 * NB_F) + ldg4(xh_bias + 2 * NB_F + c);
    const float* mj = mu + (size_t)j * (3 * NB_F) + c;
    const float4 m0 = ldg4(mj), m1 = ldg4(mj + NB_F), m2 = ldg4(mj + 2 * NB_F);
    float4 ga = f4(0.f), gb = f4(0.f), gc = f4(0.f), gm0 = f4(0.f), gm1 = f4(0.f), gm2 = f4(0.f);
    const float seed = WRITE_GW ? __ldg(seed_atom + j) : 1.0f;
    int i_pf = (e0 + BWD_GS < e1) ? __ldg(col + e0 + BWD_GS) : 0;  // far atom of the edge whose gather is issued next
    float4 gn = (e0 < e1) ? ldg4(geom + 4 * (size_t)e0) : f4(0.f);
    int wslot = 0, gslot = 0;
    uint32_t wpar = 0;
    for (int e = e0; e < e1; ++e) {
        const float4 g = gn;  // u_e = (pos_i - pos_j)/d ; u' = -u_e
        if (e + 1 < e1) gn = ldg4(geom + 4 * (size_t)(e + 1));
        const int i_issue = i_pf;
        if (e + BWD_GS + 1 < e1) i_pf = __ldg(col + e + BWD_GS + 1);
        const int wr_issue = wr_pf;
        if (e + BWD_WS + 1 < e1) wr_pf = rev ? min(e + BWD_WS + 1, __ldg(rev + e + BWD_WS + 1)) : e + BWD_WS + 1;
        cp_async_wait<BWD_GS - 1>();     // my columns of g_q[i], g_mu[i] of edge e have landed
        mbar_wait(bars + wslot, wpar);   // the (W, dW) rows of edge e have landed
        const WT* row = reinterpret_cast<const WT*>(wring + wslot * BWD_WROW) + c;
        float* grow = gring + gslot * BWD_GROW;
        const float4 wa = ldw4_plain(row), wb = ldw4_plain(row + NB_F), wc = ldw4_plain(row + 2 * NB_F);
        const float4 da = ldw4_plain(row + 3 * NB_F), db = ldw4_plain(row + 4 * NB_F), dc = ldw4_plain(row + 5 * NB_F);
        const float4 gq = lds4(grow), h0 = lds4(grow + NB_F), h1 = lds4(grow + 2 * NB_F), h2 = lds4(grow + 3 * NB_F);
        // t_b = gmu_i . u'   (per channel), t_c = sum_x gmu_i[x] * mu_j[x]
        float4 tb = h0 * (-g.x); fma4s(tb, h1, -g.y); fma4s(tb, h2, -g.z);
        float4 tc = h0 * m0; fma4(tc, h1, m1); fma4(tc, h2, m2);
        fma4(ga, wa, gq); fma4(gb, wb, tb); fma4(gc, wc, tc);
        const float4 pc = wc * cc;
        fma4(gm0, pc, h0); fma4(gm1, pc, h1); fma4(gm2, pc, h2);
        // edge scalars
        const float4 ta = a * gq, tbb = b * tb, tcc = cc * tc;  // dE/dW of the opposite edge (same filter row: W depends on d only)
        if (WRITE_GW) {
            WT* gw = gW + (size_t)e * (3 * NB_F) + c;
            stw4(gw, ta * seed); stw4(gw + NB_F, tbb * seed); stw4(gw + 2 * NB_F, tcc * seed);
        }
        float4 sd = da * ta; fma4(sd, db, tbb); fma4(sd, dc, tcc);
        const float4 pb = wb * b;
        float gd = hsum4(sd), gu0 = hsum4(pb * h0), gu1 = hsum4(pb * h1), gu2 = hsum4(pb * h2);
        __syncwarp();  // every lane has read the (W, dW) stage before the TMA engine may overwrite it
        if (lane == 0 && e + BWD_WS < e1) {
            mbar_expect_tx(bars + wslot, BWD_WROW * sizeof(WT));
            WT* stage = reinterpret_cast<WT*>(wring + wslot * BWD_WROW);
            if (wstride == BWD_WROW) {
                bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr_issue * BWD_WROW), BWD_WROW * sizeof(WT), bars + wslot);
            } else {
                bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr_issue * (3 * NB_F)), 3 * NB_F * sizeof(WT), bars + wslot);
                bulk_g2s(reinterpret_cast<float*>(stage + 3 * NB_F), reinterpret_cast<const float*>(dW + (size_t)wr_issue * (3 * NB_F)), 3 * NB_F * sizeof(WT),
                         bars + wslot);
            }
        }
        if (e + BWD_GS < e1) bwd_gather_issue(grow, gqcol + (size_t)i_issue * NB_F, gmcol + (size_t)i_issue * (3 * NB_F));
        cp_async_commit();
        if (++wslot == BWD_WS) { wslot = 0; wpar ^= 1u; }
        gslot = (gslot + 1 == BWD_GS) ? 0 : gslot + 1;
        // 4-value warp reduction in 6 shuffles: fold pairs, then butterfly; lane 0 ends with all four
        {
            // step 1: lanes exchange halves so each lane carries two values
            const bool hi = lane & 16;
            const float s0 = hi ? gd : gu1, s1 = hi ? gu0 : gu2;          // what I give away
            float k0 = hi ? gu1 : gd, k1 = hi ? gu2 : gu0;                // what I keep
            k0 += __shfl_xor_sync(0xffffffffu, s0, 16);
            k1 += __shfl_xor_sync(0xffffffffu, s1, 16);
            // now lanes<16 hold partial (gd, gu0), lanes>=16 hold partial (gu1, gu2)
            const bool hi8 = lane & 8;
            const float s = hi8 ? k0 : k1;
            float k = hi8 ? k1 : k0;
            k += __shfl_xor_sync(0xffffffffu, s, 8);
            // lanes [0,8): gd, [8,16): gu0, [16,24): gu1, [24,32): gu2
            k += __shfl_xor_sync(0xffffffffu, k, 4);
            k += __shfl_xor_sync(0xffffffffu, k, 2);
            k += __shfl_xor_sync(0xffffffffu, k, 1);
            if ((lane & 7) == 0) {
                // lane 0 -> .w (gd), lane 8 -> .x (gu0), lane 16 -> .y (gu1), lane 24 -> .z (gu2)
                const int comp = (lane == 0) ? 3 : (lane >> 3) - 1;
                // fire-and-forget reduction (RED.ADD): `*p += k` would put one L2 round trip per edge on the warp's critical path (the load
                // feeds the add).  Exactly one thread of one warp touches this address per launch: still deterministic.
                atomicAdd(egrad + 4 * (size_t)e + comp, k);
            }
        }
    }
    cp_async_wait<0>();
    float* gx = g_xh + (size_t)j * (3 * NB_F) + c;
    st4(gx, ga); st4(gx + NB_F, gb); st4(gx + 2 * NB_F, gc);
    const float* gmj = g_mu + (size_t)j * (3 * NB_F) + c;
    float* go = g_mu_in + (size_t)j * (3 * NB_F) + c;
    st4(go, ldg4(gmj) + gm0); st4(go + NB_F, ldg4(gmj + NB_F) + gm1); st4(go + 2 * NB_F, ldg4(gmj + 2 * NB_F) + gm2);
}

// Forces from the accumulated edge gradients.  Slot e of row j holds, for the edge e' = (j -> i)
// with r' = pos_j - pos_i = -d u_e:  (dE/du'[3], dE/dd).  Chain rule through u' = r'/d, d = |r'|:
//   G(e) := dE/dr' = (gu - (gu.u') u')/d + gd u'
// pos_j receives +G(e) from its own row and -G(rev e) from the rows where it is the far end:
//   F_j = -dE/dpos_j = -sum_{e in row j} (G(e) - G(rev e))          (painn.py:135-146 autograd)
__device__ __forceinline__ float3 edge_G(const float4 eg, const float4 g) {
    const float ux = -g.x, uy = -g.y, uz = -g.z;  // u' of the opposite edge
    const float dot = eg.x * ux + eg.y * uy + eg.z * uz;
    const float inv = 1.0f / g.w;
    return make_float3((eg.x - dot * ux) * inv + eg.w * ux, (eg.y - dot * uy) * inv + eg.w * uy, (eg.z - dot * uz) * inv + eg.w * uz);
}

__global__ void __launch_bounds__(256) k_edge_forces(const float* __restrict__ egrad, const float* __restrict__ geom,
                                                    const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ rev, int n_atoms,
                                                    float* __restrict__ forces) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_atoms) return;
    float fx = 0.f, fy = 0.f, fz = 0.f;
    for (int e = row_ptr[j]; e < row_ptr[j + 1]; ++e) {
        const int r = rev[e];
        const float3 g1 = edge_G(ldg4(egrad + 4 * (size_t)e), ldg4(geom + 4 * (size_t)e));
        const float3 g2 = edge_G(ldg4(egrad + 4 * (size_t)r), ldg4(geom + 4 * (size_t)r));
        fx -= g1.x - g2.x; fy -= g1.y - g2.y; fz -= g1.z - g2.z;
    }
    forces[3 * (size_t)j] = fx; forces[3 * (size_t)j + 1] = fy; forces[3 * (size_t)j + 2] = fz;
}

int nb_painn_msg_fwd_ex(const float* xh, const float* xh_bias, const float* q, const float* mu, const float* W, int w_stride, const int32_t* rev,
                        const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, float* q_out, float* mu_out, cudaStream_t stream, int bf16) {
    if (!xh || !xh_bias || !q || !mu || !W || !geom || !row_ptr || !col || !q_out || !mu_out || n_atoms < 0) return NB200_EINVAL;
    if (w_stride != 3 * NB_F && w_stride != 6 * NB_F) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    const int smem = MSG_WARPS * (FWD_WARP_FLOATS * (int)sizeof(float) + FWD_WS * 8);
    static bool attr_set = false;  // idempotent; racing threads set the same value
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_fwd<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_fwd<nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)
        k_painn_msg_fwd<nb_bf16><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, q, mu, reinterpret_cast<const nb_bf16*>(W), geom, row_ptr, col, n_atoms,
                                                                     q_out, mu_out, w_stride, rev);
    else
        k_painn_msg_fwd<float><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, q, mu, W, geom, row_ptr, col, n_atoms, q_out, mu_out, w_stride, rev);
    return nb_check_launch();
}

extern "C" int nb200_painn_msg_fwd(const float* xh, const float* xh_bias, const float* q, const float* mu, const float* W,
                                   const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, float* q_out,
                                   float* mu_out, void* stream) {
    return nb_painn_msg_fwd_ex(xh, xh_bias, q, mu, W, 3 * NB_F, nullptr, geom, row_ptr, col, n_atoms, q_out, mu_out, (cudaStream_t)stream, 0);
}

int nb_painn_msg_bwd_ex(const float* xh, const float* xh_bias, const float* mu, const float* W, const float* dW, int w_stride, const int32_t* rev,
                        const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q, const float* g_mu,
                        float* g_xh, float* g_mu_in, float* egrad, cudaStream_t stream, int bf16) {
    if (!xh || !xh_bias || !mu || !W || !dW || !geom || !row_ptr || !col || !g_q || !g_mu || !g_xh || !g_mu_in || !egrad || n_atoms < 0)
        return NB200_EINVAL;
    if (g_mu == g_mu_in || (w_stride != 3 * NB_F && w_stride != 6 * NB_F)) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    const int smem = MSG_WARPS * (BWD_WARP_FLOATS * (int)sizeof(float) + BWD_WS * 8);
    static bool attr_set = false;  // idempotent; racing threads set the same value
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_bwd<false, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_bwd<false, nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)
        k_painn_msg_bwd<false, nb_bf16><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, mu, reinterpret_cast<const nb_bf16*>(W),
                                                                            reinterpret_cast<const nb_bf16*>(dW), geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh,
                                                                            g_mu_in, egrad, nullptr, nullptr, w_stride, rev);
    else
        k_painn_msg_bwd<false, float><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, mu, W, dW, geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad,
                                                                          nullptr, nullptr, w_stride, rev);
    return nb_check_launch();
}

extern "C" int nb200_painn_msg_bwd(const float* xh, const float* xh_bias, const float* mu, const float* W, const float* dW,
                                   const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q,
                                   const float* g_mu, float* g_xh, float* g_mu_in, float* egrad, void* stream) {
    return nb_painn_msg_bwd_ex(xh, xh_bias, mu, W, dW, 3 * NB_F, nullptr, geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad,
                               (cudaStream_t)stream, 0);
}

// training variant: additionally writes gW[e][3F] = seed[source atom] * dE/dW of the opposite edge into slot e (see painn_train.cu)
int nb_painn_msg_bwd_train(const float* xh, const float* xh_bias, const float* mu, const float* W, const float* dW, const float* geom,
                           const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q, const float* g_mu, float* g_xh,
                           float* g_mu_in, float* egrad, float* gW, const float* seed_atom, cudaStream_t stream, int bf16, const int32_t* rev) {
    const int smem = MSG_WARPS * (BWD_WARP_FLOATS * (int)sizeof(float) + BWD_WS * 8);
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_bwd<true, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_bwd<true, nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)  // bf16 storage: W, dW/dd AND the per-edge filter gradients written here
        k_painn_msg_bwd<true, nb_bf16><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, mu, reinterpret_cast<const nb_bf16*>(W),
                                                                           reinterpret_cast<const nb_bf16*>(dW), geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh,
                                                                           g_mu_in, egrad, reinterpret_cast<nb_bf16*>(gW), seed_atom, 3 * NB_F, rev);
    else
        k_painn_msg_bwd<true, float><<<grid, MSG_THREADS, smem, stream>>>(xh, xh_bias, mu, W, dW, geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad, gW,
                                                                         seed_atom, 3 * NB_F, rev);
    return nb_check_launch();
}

extern "C" int nb200_edge_forces(const float* egrad, const float* geom, const int32_t* row_ptr, const int32_t* rev, int32_t n_atoms,
                                 float* forces, void* stream) {
    if (!egrad || !geom || !row_ptr || !rev || !forces || n_atoms < 0) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    k_edge_forces<<<(n_atoms + 255) / 256, 256, 0, (cudaStream_t)stream>>>(egrad, geom, row_ptr, rev, n_atoms, forces);
    return nb_check_launch();
}
