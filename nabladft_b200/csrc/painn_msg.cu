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
#include "wgmma.cuh"

// One warp per CTA (11-16 CTAs per SM, see msg_blocks_per_sm): a CTA's shared memory and registers return to the SM as soon as ITS atom is done.  With 8 warps per
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

__device__ __forceinline__ void cp_async4(int32_t* smem_dst, const int32_t* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem_src) : "memory");
}

// v5: the edge metadata of a row -- col[e], rev[e] and geom[e] -- is staged into the warp's shared memory with one burst of cp.async before
// the first edge.  Up to v4 these were __ldg'ed one edge ahead inside the loop and the source index fed the address of the gather: one
// L2 round trip per edge on the warp's critical path, whatever the ring depths.  Now no load in the loop feeds an address.  Rows longer
// than MSG_STAGE_CAP edges (the benchmark batches reach degree 49) are streamed in chunks of MSG_STAGE_CAP: both rings drain at a chunk
// boundary, the sums carry on in registers in the same CSR order.
// Ring depths (filter WS / gather GS) tried with the staged metadata, ms per launch at the bench.py shape (9.6k atoms, 186k edges, fp32
// pair records), H100 SXM 80 GB at a 400 W power limit, CUDA events over 50 E+F calls (bench_msg.py); the two kernels are tuned apart, and
// each row is the mean of the runs that used that depth.  Differences below ~1 % are within run-to-run spread.
//   forward   WS/GS   ms          backward  WS/GS   ms
//   before: no staging  5/2   0.138-0.140   no staging  3/2   0.206-0.212
//             5/2   0.134                   3/2   0.199
//             4/3   0.131                   2/3   0.199
//             3/4   0.130                   2/4   0.194
//             5/3   0.129-0.132             3/3   0.186-0.190
//             5/4   0.131                   3/4   0.183
//             4/4   0.128-0.130 (kept)      4/3   0.183-0.184
//                                           4/4   0.181 (kept)
// Staging rows of at most 32 edges (chunked above) instead of 64 saves 0.75 KB per warp and changed neither kernel measurably.
// The deeper rings cost residency (fp32: 11 warps per SM in the forward, 10 in the backward; 15 and 16 before) and still win, because
// neither kernel is short of bytes in flight any more: each runs within 2-7 % of a load-only kernel that reads the same bytes per edge
// (nb200_msg_gather_probe, below).  That ceiling is the L2 -> SM stream of the gathers: per directed edge the forward reads its 1.5 KB
// filter row plus 3 KB of xh[j], mu[j] out of L2, the backward 3 KB + 2 KB, and the probe measures 6.6-7.3 TB/s on the forward's pattern
// and 5.5 TB/s on the backward's.  Going faster means fewer gathered bytes per edge (e.g. both edges of a pair in one visit), which
// reorders the sums.
#define MSG_STAGE_CAP 64
#define MSG_META_FLOATS (6 * MSG_STAGE_CAP)  // geom [CAP] float4 | col [CAP] | rev [CAP]

__device__ __forceinline__ void stage_meta(float* meta, const float* geom, const int32_t* col, const int32_t* rev, int s0, int n, int lane) {
    int32_t* cs = reinterpret_cast<int32_t*>(meta + 4 * MSG_STAGE_CAP);
    for (int k = lane; k < n; k += 32) {
        cp_async16(meta + 4 * k, geom + 4 * (size_t)(s0 + k));
        cp_async4(cs + k, col + s0 + k);
        if (rev) cp_async4(cs + MSG_STAGE_CAP + k, rev + s0 + k);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();  // every lane's copies are visible to the whole warp
}

// CTAs (= warps) per SM for __launch_bounds__: as many as the per-warp shared memory (+ the 1 KB the SM reserves per CTA) fits in 228 KB,
// at most `cap` -- the register budget: the forward fits 24 warps (85 registers), the backward 16 (128; at 20 warps the bf16 variant spills)
constexpr int msg_blocks_per_sm(int smem_bytes, int cap) { return 233472 / (smem_bytes + 1024) < cap ? 233472 / (smem_bytes + 1024) : cap; }

// Forward (v4): two rings per warp with independent depths.
//   * filter rows (the HBM stream, microsecond-scale loaded latency): FWD_WS stages, filled by the TMA engine --
//     one elected lane issues a 1536-byte `cp.async.bulk` per edge, completion on a per-stage mbarrier;
//   * gathered neighbour rows xh[j], mu[j] (L2): FWD_GS stages of per-lane cp.async (LDGSTS).
// cp.async groups retire in order, so one shared queue cannot give the two streams different depths (v2 had 3 / 3
// and reached 64 % of the HBM roofline; bytes of the HBM stream in flight were the limiter, not issue slots -- v3).
#define FWD_WS 4
#define FWD_GS 4
#define FWD_WROW (3 * NB_F)
#define FWD_GROW (6 * NB_F)

// WT: storage type of the filter rows (float / nb_bf16); a ring stage holds one stored row, so a bf16 stage is half the size of an fp32 one
template <class WT>
struct FwdRing {
    static constexpr int kRowFloats = FWD_WROW * (int)sizeof(WT) / 4;
    static constexpr int kWarpFloats = FWD_WS * kRowFloats + FWD_GS * FWD_GROW + MSG_META_FLOATS;
    static constexpr int kSmem = MSG_WARPS * (kWarpFloats * 4 + FWD_WS * 8);
    static constexpr int kBlocks = msg_blocks_per_sm(kSmem, 24);
};

__device__ __forceinline__ void fwd_gather_issue(float* dst, const float* xrow, const float* mrow) {
    cp_async16(dst, xrow); cp_async16(dst + NB_F, xrow + NB_F); cp_async16(dst + 2 * NB_F, xrow + 2 * NB_F);
    cp_async16(dst + 3 * NB_F, mrow); cp_async16(dst + 4 * NB_F, mrow + NB_F); cp_async16(dst + 5 * NB_F, mrow + 2 * NB_F);
}

template <class WT>
__global__ void __launch_bounds__(MSG_THREADS, FwdRing<WT>::kBlocks) k_painn_msg_fwd(const float* __restrict__ xh, const float* __restrict__ xh_bias,
                                                                                    const float* q, const float* __restrict__ mu,
                                                                                    const WT* __restrict__ W, const float* __restrict__ geom,
                                                                                    const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                                                                    int n_atoms, float* q_out, float* __restrict__ mu_out, int wstride,
                                                                                    const int32_t* __restrict__ rev) {
    // filter row of edge e: row e of `W` (rows of `wstride` elements), or -- `rev` given -- row min(e, rev[e]): ONE stored row per undirected
    // pair (the filter depends on the distance only; filter.cu then evaluates only the canonical edges)
    using R = FwdRing<WT>;
    extern __shared__ __align__(128) float ring_dyn[];  // [warps][WS x W row | GS x gather row | row metadata], then the mbarriers
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = blockIdx.x * MSG_WARPS + warp;
    if (i >= n_atoms) return;  // no block-level barrier below: a whole warp may leave
    const int c = lane * 4;
    float* wring = ring_dyn + warp * R::kWarpFloats;
    float* gring = wring + FWD_WS * R::kRowFloats + c;  // my 16-byte column of every gathered row
    float* meta = wring + FWD_WS * R::kRowFloats + FWD_GS * FWD_GROW;
    const float4* geom_s = reinterpret_cast<const float4*>(meta);
    const int32_t* col_s = reinterpret_cast<const int32_t*>(meta + 4 * MSG_STAGE_CAP);
    const int32_t* rev_s = col_s + MSG_STAGE_CAP;
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring_dyn + MSG_WARPS * R::kWarpFloats) + warp * FWD_WS;
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < FWD_WS; ++s) mbar_init(bars + s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const float* xcol = xh + c;
    const float* mcol = mu + c;
    const float4 ba = ldg4(xh_bias + c), bb = ldg4(xh_bias + NB_F + c), bc = ldg4(xh_bias + 2 * NB_F + c);
    float4 dq = f4(0.f), dm0 = f4(0.f), dm1 = f4(0.f), dm2 = f4(0.f);
    int wslot = 0, gslot = 0;  // ring slots of the next edge; they run on across chunks
    uint32_t wpar = 0;
    for (int s0 = e0; s0 < e1; s0 += MSG_STAGE_CAP) {
        const int n = min(e1 - s0, MSG_STAGE_CAP);
        stage_meta(meta, geom, col, rev, s0, n, lane);
        auto issue_w = [&](int slot, int k) {  // filter row of local edge k into ring slot `slot` (lane 0)
            const int wr = rev ? min(s0 + k, rev_s[k]) : s0 + k;
            mbar_expect_tx(bars + slot, FWD_WROW * sizeof(WT));
            bulk_g2s(wring + slot * R::kRowFloats, reinterpret_cast<const float*>(W + (size_t)wr * wstride), FWD_WROW * sizeof(WT), bars + slot);
        };
        auto issue_g = [&](float* dst, int k) {
            const int j = col_s[k];
            fwd_gather_issue(dst, xcol + (size_t)j * (3 * NB_F), mcol + (size_t)j * (3 * NB_F));
        };
        if (lane == 0) {
            int sl = wslot;
#pragma unroll
            for (int k = 0; k < FWD_WS; ++k) {
                if (k < n) issue_w(sl, k);
                sl = (sl + 1 == FWD_WS) ? 0 : sl + 1;
            }
        }
        {
            int sl = gslot;
#pragma unroll
            for (int k = 0; k < FWD_GS; ++k) {
                if (k < n) issue_g(gring + sl * FWD_GROW, k);
                cp_async_commit();
                sl = (sl + 1 == FWD_GS) ? 0 : sl + 1;
            }
        }
        for (int k = 0; k < n; ++k) {
            const float4 g = geom_s[k];
            cp_async_wait<FWD_GS - 1>();     // my columns of xh[j], mu[j] of edge k have landed
            mbar_wait(bars + wslot, wpar);   // the filter row of edge k has landed
            const WT* wrow = reinterpret_cast<const WT*>(wring + wslot * R::kRowFloats) + c;
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
            if (lane == 0 && k + FWD_WS < n) issue_w(wslot, k + FWD_WS);
            if (k + FWD_GS < n) issue_g(grow, k + FWD_GS);
            cp_async_commit();
            if (++wslot == FWD_WS) { wslot = 0; wpar ^= 1u; }
            gslot = (gslot + 1 == FWD_GS) ? 0 : gslot + 1;
        }
        cp_async_wait<0>();
        __syncwarp();  // the whole warp is done with this chunk's metadata before the next chunk is staged over it
    }
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
// them in registers.  Now: (W, dW) rows by TMA bulk copies (one elected lane, BWD_WS stages x 3 KB, mbarrier per stage) and the
// gathered gradient rows by per-lane cp.async into a second ring (BWD_GS stages x 2 KB).  v5 stages the row metadata as the forward does.
#define BWD_WS 4
#define BWD_GS 4
#define BWD_WROW (6 * NB_F)
#define BWD_GROW (4 * NB_F)

template <class WT>
struct BwdRing {
    static constexpr int kRowFloats = BWD_WROW * (int)sizeof(WT) / 4;
    static constexpr int kWarpFloats = BWD_WS * kRowFloats + BWD_GS * BWD_GROW + MSG_META_FLOATS;
    static constexpr int kSmem = MSG_WARPS * (kWarpFloats * 4 + BWD_WS * 8);
    static constexpr int kBlocks = msg_blocks_per_sm(kSmem, 16);
};

__device__ __forceinline__ void bwd_gather_issue(float* dst, const float* gq_row, const float* gmu_row) {
    cp_async16(dst, gq_row); cp_async16(dst + NB_F, gmu_row); cp_async16(dst + 2 * NB_F, gmu_row + NB_F); cp_async16(dst + 3 * NB_F, gmu_row + 2 * NB_F);
}

template <bool WRITE_GW, class WT>
__global__ void __launch_bounds__(MSG_THREADS, BwdRing<WT>::kBlocks) k_painn_msg_bwd(const float* __restrict__ xh, const float* __restrict__ xh_bias,
                                                                                    const float* __restrict__ mu, const WT* __restrict__ W,
                                                                                    const WT* __restrict__ dW, const float* __restrict__ geom,
                                                                                    const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                                                                    int n_atoms, const float* __restrict__ g_q, const float* __restrict__ g_mu,
                                                                                    float* __restrict__ g_xh, float* __restrict__ g_mu_in,
                                                                                    float* __restrict__ egrad, WT* __restrict__ gW,
                                                                                    const float* __restrict__ seed_atom, int wstride, const int32_t* __restrict__ rev) {
    // wstride == 6F: ONE [W | dW/dd] record of 3 KB per edge in `W` (one bulk copy per edge instead of two: the TMA engine is paced by the
    // number of copies); `rev` given: row min(e, rev[e]) -- see the forward kernel
    using R = BwdRing<WT>;
    extern __shared__ __align__(128) float ring_dyn[];  // [warps][WS x (W | dW) row | GS x (g_q | g_mu) row | row metadata], then the mbarriers
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * MSG_WARPS + warp;
    if (j >= n_atoms) return;
    const int c = lane * 4;
    float* wring = ring_dyn + warp * R::kWarpFloats;
    float* gring = wring + BWD_WS * R::kRowFloats + c;  // my 16-byte column of every gathered row
    float* meta = wring + BWD_WS * R::kRowFloats + BWD_GS * BWD_GROW;
    const float4* geom_s = reinterpret_cast<const float4*>(meta);
    const int32_t* col_s = reinterpret_cast<const int32_t*>(meta + 4 * MSG_STAGE_CAP);
    const int32_t* rev_s = col_s + MSG_STAGE_CAP;
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring_dyn + MSG_WARPS * R::kWarpFloats) + warp * BWD_WS;
    const int e0 = row_ptr[j], e1 = row_ptr[j + 1];
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < BWD_WS; ++s) mbar_init(bars + s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const float* gqcol = g_q + c;
    const float* gmcol = g_mu + c;
    const float* xj = xh + (size_t)j * (3 * NB_F) + c;
    const float4 a = ldg4(xj) + ldg4(xh_bias + c), b = ldg4(xj + NB_F) + ldg4(xh_bias + NB_F + c),
                 cc = ldg4(xj + 2 * NB_F) + ldg4(xh_bias + 2 * NB_F + c);
    const float* mj = mu + (size_t)j * (3 * NB_F) + c;
    const float4 m0 = ldg4(mj), m1 = ldg4(mj + NB_F), m2 = ldg4(mj + 2 * NB_F);
    float4 ga = f4(0.f), gb = f4(0.f), gc = f4(0.f), gm0 = f4(0.f), gm1 = f4(0.f), gm2 = f4(0.f);
    const float seed = WRITE_GW ? __ldg(seed_atom + j) : 1.0f;
    int wslot = 0, gslot = 0;  // ring slots of the next edge; they run on across chunks
    uint32_t wpar = 0;
    for (int s0 = e0; s0 < e1; s0 += MSG_STAGE_CAP) {
        const int n = min(e1 - s0, MSG_STAGE_CAP);
        stage_meta(meta, geom, col, rev, s0, n, lane);
        auto issue_w = [&](int slot, int k) {  // (W, dW) rows of local edge k into ring slot `slot` (lane 0)
            const int wr = rev ? min(s0 + k, rev_s[k]) : s0 + k;
            mbar_expect_tx(bars + slot, BWD_WROW * sizeof(WT));
            WT* stage = reinterpret_cast<WT*>(wring + slot * R::kRowFloats);
            if (wstride == BWD_WROW) {
                bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr * BWD_WROW), BWD_WROW * sizeof(WT), bars + slot);
            } else {
                bulk_g2s(reinterpret_cast<float*>(stage), reinterpret_cast<const float*>(W + (size_t)wr * (3 * NB_F)), 3 * NB_F * sizeof(WT), bars + slot);
                bulk_g2s(reinterpret_cast<float*>(stage + 3 * NB_F), reinterpret_cast<const float*>(dW + (size_t)wr * (3 * NB_F)), 3 * NB_F * sizeof(WT),
                         bars + slot);
            }
        };
        auto issue_g = [&](float* dst, int k) {
            const int i = col_s[k];
            bwd_gather_issue(dst, gqcol + (size_t)i * NB_F, gmcol + (size_t)i * (3 * NB_F));
        };
        if (lane == 0) {
            int sl = wslot;
#pragma unroll
            for (int k = 0; k < BWD_WS; ++k) {
                if (k < n) issue_w(sl, k);
                sl = (sl + 1 == BWD_WS) ? 0 : sl + 1;
            }
        }
        {
            int sl = gslot;
#pragma unroll
            for (int k = 0; k < BWD_GS; ++k) {
                if (k < n) issue_g(gring + sl * BWD_GROW, k);
                cp_async_commit();
                sl = (sl + 1 == BWD_GS) ? 0 : sl + 1;
            }
        }
        for (int k = 0; k < n; ++k) {
            const int e = s0 + k;
            const float4 g = geom_s[k];  // u_e = (pos_i - pos_j)/d ; u' = -u_e
            cp_async_wait<BWD_GS - 1>();     // my columns of g_q[i], g_mu[i] of edge e have landed
            mbar_wait(bars + wslot, wpar);   // the (W, dW) rows of edge e have landed
            const WT* row = reinterpret_cast<const WT*>(wring + wslot * R::kRowFloats) + c;
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
            if (lane == 0 && k + BWD_WS < n) issue_w(wslot, k + BWD_WS);
            if (k + BWD_GS < n) issue_g(grow, k + BWD_GS);
            cp_async_commit();
            if (++wslot == BWD_WS) { wslot = 0; wpar ^= 1u; }
            gslot = (gslot + 1 == BWD_GS) ? 0 : gslot + 1;
            // 4-value warp reduction in 6 shuffles: fold pairs, then butterfly; lane 0 ends with all four
            {
                // step 1: lanes exchange halves so each lane carries two values
                const bool hi = lane & 16;
                const float s0_ = hi ? gd : gu1, s1_ = hi ? gu0 : gu2;        // what I give away
                float k0 = hi ? gu1 : gd, k1 = hi ? gu2 : gu0;                // what I keep
                k0 += __shfl_xor_sync(0xffffffffu, s0_, 16);
                k1 += __shfl_xor_sync(0xffffffffu, s1_, 16);
                // now lanes<16 hold partial (gd, gu0), lanes>=16 hold partial (gu1, gu2)
                const bool hi8 = lane & 8;
                const float s = hi8 ? k0 : k1;
                float kk = hi8 ? k1 : k0;
                kk += __shfl_xor_sync(0xffffffffu, s, 8);
                // lanes [0,8): gd, [8,16): gu0, [16,24): gu1, [24,32): gu2
                kk += __shfl_xor_sync(0xffffffffu, kk, 4);
                kk += __shfl_xor_sync(0xffffffffu, kk, 2);
                kk += __shfl_xor_sync(0xffffffffu, kk, 1);
                if ((lane & 7) == 0) {
                    // lane 0 -> .w (gd), lane 8 -> .x (gu0), lane 16 -> .y (gu1), lane 24 -> .z (gu2)
                    const int comp = (lane == 0) ? 3 : (lane >> 3) - 1;
                    // fire-and-forget reduction (RED.ADD): `*p += k` would put one L2 round trip per edge on the warp's critical path (the load
                    // feeds the add).  Exactly one thread of one warp touches this address per launch: still deterministic.
                    atomicAdd(egrad + 4 * (size_t)e + comp, kk);
                }
            }
        }
        cp_async_wait<0>();
        __syncwarp();  // the whole warp is done with this chunk's metadata before the next chunk is staged over it
    }
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
    static bool attr_set = false;  // idempotent; racing threads set the same value
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_fwd<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, FwdRing<float>::kSmem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_fwd<nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, FwdRing<nb_bf16>::kSmem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)
        k_painn_msg_fwd<nb_bf16><<<grid, MSG_THREADS, FwdRing<nb_bf16>::kSmem, stream>>>(xh, xh_bias, q, mu, reinterpret_cast<const nb_bf16*>(W), geom, row_ptr, col, n_atoms,
                                                                     q_out, mu_out, w_stride, rev);
    else
        k_painn_msg_fwd<float><<<grid, MSG_THREADS, FwdRing<float>::kSmem, stream>>>(xh, xh_bias, q, mu, W, geom, row_ptr, col, n_atoms, q_out, mu_out, w_stride, rev);
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
    static bool attr_set = false;  // idempotent; racing threads set the same value
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_bwd<false, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdRing<float>::kSmem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_bwd<false, nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdRing<nb_bf16>::kSmem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)
        k_painn_msg_bwd<false, nb_bf16><<<grid, MSG_THREADS, BwdRing<nb_bf16>::kSmem, stream>>>(xh, xh_bias, mu, reinterpret_cast<const nb_bf16*>(W),
                                                                            reinterpret_cast<const nb_bf16*>(dW), geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh,
                                                                            g_mu_in, egrad, nullptr, nullptr, w_stride, rev);
    else
        k_painn_msg_bwd<false, float><<<grid, MSG_THREADS, BwdRing<float>::kSmem, stream>>>(xh, xh_bias, mu, W, dW, geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad,
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
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_painn_msg_bwd<true, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdRing<float>::kSmem) != cudaSuccess ||
            cudaFuncSetAttribute(k_painn_msg_bwd<true, nb_bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdRing<nb_bf16>::kSmem) != cudaSuccess)
            return nb_check_launch();
        attr_set = true;
    }
    const int grid = (n_atoms + MSG_WARPS - 1) / MSG_WARPS;
    if (bf16)  // bf16 storage: W, dW/dd AND the per-edge filter gradients written here
        k_painn_msg_bwd<true, nb_bf16><<<grid, MSG_THREADS, BwdRing<nb_bf16>::kSmem, stream>>>(xh, xh_bias, mu, reinterpret_cast<const nb_bf16*>(W),
                                                                           reinterpret_cast<const nb_bf16*>(dW), geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh,
                                                                           g_mu_in, egrad, reinterpret_cast<nb_bf16*>(gW), seed_atom, 3 * NB_F, rev);
    else
        k_painn_msg_bwd<true, float><<<grid, MSG_THREADS, BwdRing<float>::kSmem, stream>>>(xh, xh_bias, mu, W, dW, geom, row_ptr, col, n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad, gW,
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

// Gather-bandwidth probe (bench_msg.py): the L2 -> SM stream of a message kernel without its arithmetic, rings or reductions.  Per edge e
// of a row: the record row min(e, rev[e]) (its first RW floats) and the gathered rows A[col[e]] (AW floats) and B[col[e]] (3F floats), read
// with plain L2 loads (ld.global.cg) into a running sum.  8 warps per CTA, one atom per warp, two edges of loads in flight per warp:
// AW = 3F, RW = 3F is the forward's stream, AW = F, RW = 6F the backward's.
template <int AW, int RW>
__global__ void __launch_bounds__(256, 2) k_msg_gather_probe(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ rec,
                                                             int rec_stride, const int32_t* __restrict__ rev, const int32_t* __restrict__ row_ptr,
                                                             const int32_t* __restrict__ col, int n_atoms, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (i >= n_atoms) return;
    const int c = lane * 4;
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    float4 acc = f4(0.f);
    for (int s0 = e0; s0 < e1; s0 += 32) {
        const int n = min(32, e1 - s0);
        const int my_col = lane < n ? col[s0 + lane] : 0;
        const int my_wr = lane < n ? (rev ? min(s0 + lane, rev[s0 + lane]) : s0 + lane) : 0;
#pragma unroll 2
        for (int k = 0; k < n; ++k) {
            const int j = __shfl_sync(0xffffffffu, my_col, k), wr = __shfl_sync(0xffffffffu, my_wr, k);
            const float* a = A + (size_t)j * AW + c;
            const float* b = B + (size_t)j * (3 * NB_F) + c;
            const float* r = rec + (size_t)wr * rec_stride + c;
#pragma unroll
            for (int t = 0; t < AW / NB_F; ++t) acc = acc + __ldcg(reinterpret_cast<const float4*>(a + t * NB_F));
#pragma unroll
            for (int t = 0; t < 3; ++t) acc = acc + __ldcg(reinterpret_cast<const float4*>(b + t * NB_F));
#pragma unroll
            for (int t = 0; t < RW / NB_F; ++t) acc = acc + __ldcg(reinterpret_cast<const float4*>(r + t * NB_F));
        }
    }
    out[(size_t)i * 32 + lane] = hsum4(acc);
}

// `bwd_pattern` 0: the forward's stream (A = xh [N,3F], B = mu, first 3F of each record); 1: the backward's (A = g_q [N,F], B = g_mu, whole
// 6F record).  `rec_stride` >= the record floats read; out[N * 32].
extern "C" int nb200_msg_gather_probe(const float* A, const float* B, const float* rec, int32_t rec_stride, const int32_t* rev, const int32_t* row_ptr,
                                      const int32_t* col, int32_t n_atoms, int32_t bwd_pattern, float* out, void* stream) {
    if (!A || !B || !rec || !row_ptr || !col || !out || n_atoms < 0 || rec_stride < (bwd_pattern ? 6 * NB_F : 3 * NB_F)) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    const int grid = (n_atoms + 7) / 8;
    if (bwd_pattern)
        k_msg_gather_probe<NB_F, 6 * NB_F><<<grid, 256, 0, (cudaStream_t)stream>>>(A, B, rec, rec_stride, rev, row_ptr, col, n_atoms, out);
    else
        k_msg_gather_probe<3 * NB_F, 3 * NB_F><<<grid, 256, 0, (cudaStream_t)stream>>>(A, B, rec, rec_stride, rev, row_ptr, col, n_atoms, out);
    return nb_check_launch();
}

// Every instantiation of the two message kernels behind one C entry point each, for benchmarks and tests.  `w_stride` (3F or 6F) and `rev`
// select the filter row layout as in nb_painn_msg_fwd_ex / _bwd_ex, `bf16` the storage type of W / dW (and gW).  The backward with `gW` given
// is the training variant (W, dW in two arrays of rows of 3F): it also writes gW[e] = seed_atom[j] * dE/dW of the opposite edge.
extern "C" int nb200_painn_msg_fwd_ex(const float* xh, const float* xh_bias, const float* q, const float* mu, const void* W, int32_t w_stride,
                                      const int32_t* rev, const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, float* q_out,
                                      float* mu_out, int32_t bf16, void* stream) {
    return nb_painn_msg_fwd_ex(xh, xh_bias, q, mu, static_cast<const float*>(W), w_stride, rev, geom, row_ptr, col, n_atoms, q_out, mu_out,
                               (cudaStream_t)stream, bf16 ? 1 : 0);
}

extern "C" int nb200_painn_msg_bwd_ex(const float* xh, const float* xh_bias, const float* mu, const void* W, const void* dW, int32_t w_stride,
                                      const int32_t* rev, const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms,
                                      const float* g_q, const float* g_mu, float* g_xh, float* g_mu_in, float* egrad, void* gW,
                                      const float* seed_atom, int32_t bf16, void* stream) {
    if (!gW)
        return nb_painn_msg_bwd_ex(xh, xh_bias, mu, static_cast<const float*>(W), static_cast<const float*>(dW), w_stride, rev, geom, row_ptr, col,
                                   n_atoms, g_q, g_mu, g_xh, g_mu_in, egrad, (cudaStream_t)stream, bf16 ? 1 : 0);
    if (!xh || !xh_bias || !mu || !W || !dW || !geom || !row_ptr || !col || !g_q || !g_mu || !g_xh || !g_mu_in || !egrad || !seed_atom || n_atoms < 0)
        return NB200_EINVAL;
    if (g_mu == g_mu_in || w_stride != 3 * NB_F) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    return nb_painn_msg_bwd_train(xh, xh_bias, mu, static_cast<const float*>(W), static_cast<const float*>(dW), geom, row_ptr, col, n_atoms, g_q, g_mu,
                                  g_xh, g_mu_in, egrad, static_cast<float*>(gW), seed_atom, (cudaStream_t)stream, bf16 ? 1 : 0, rev);
}
