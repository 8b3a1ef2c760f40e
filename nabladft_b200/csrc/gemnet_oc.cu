// gemnet_oc.cu -- GemNet-OC energy + direct coupled forces, first correct path (SURVEY.md section 8 a19 / f3; DESIGN.md 3.9).
//
// Reference: nablaDFT/gemnet_oc/gemnet_oc.py (forward 1121-1251, graphs 694-1000, bases 1001-1120), interaction_indices.py,
// layers/{interaction_block,atom_update_block,embedding_block,efficient,radial_basis,spherical_basis,base_layers}.py.
//
// Design (GPU-first, not the reference's): the reference materialises index lists for triplets and quadruplets (526 k quadruplets for
// 79 atoms) and scatters every basis into zero-padded [edges, K_max, .] tensors so that aggregation becomes a batched matmul.  Here
// nothing of that is stored.  The four graphs are CSR rows by TARGET atom with sources ascending (the order in which the reference's
// SparseTensor rows enumerate input edges); an aggregation kernel owns one output (edge, channel) element, walks the CSR rows of the
// atoms involved, evaluates the Legendre bases of the angles on the fly and keeps the [spherical x channel] partial sums in registers;
// the radial factor is applied once per output.  The order of OUTPUT edges differs from the reference's ([directed | flipped] per
// molecule) -- a row permutation of every per-edge tensor that cancels in the per-atom sums (energy, forces, h).
// Dense layers run on the wgmma 3xTF32 GEMM (gemm_tc.cu) when the shape tiles, else on the functor fallback below.
// Every kernel is a functor launched through pfor() (gemnet_pf.cuh) so that the same source compiles for host emulation in tests/emu.
// Training (parameter gradients) is gemnet_oc_train.inc; force-Jacobian products, a tangent pass through that training forward for normal
// modes, are gemnet_oc_jvp.inc (DESIGN.md 3.9.1).
#include "gemnet_oc_kernels.cuh"

namespace {

// ------------------------------------------------------------------ host side
struct GraphBuf {
    int32_t *mol_id, *rank, *deg, *tcnt, *ptr, *tbase;  // deg[4][N], ptr[4][N+1]
    int64_t bytes;
};
GraphBuf carve_graph(void* p, int64_t n, int64_t mx) {
    Carve c(p);
    GraphBuf g;
    g.mol_id = c.take<int32_t>(n);
    g.rank = c.take<int32_t>(n * mx);
    g.deg = c.take<int32_t>(4 * n);
    g.tcnt = c.take<int32_t>(n);
    g.ptr = c.take<int32_t>(4 * (n + 1));
    g.tbase = c.take<int32_t>(n + 1);
    g.bytes = c.off + 256;
    return g;
}
struct Work {
    Graph a2a, mn, ae, q;
    int32_t *rev, *q_tin;
    float *rb, *B_main, *B_ae, *B_q, *B_a2a, *cbf16;
    float *h, *m, *hst, *XE, *XF;
    float *tE[3], *OE, *xdE, *tE64, *yP, *xdP, *xt;
    float *tN[3], *ON, *xdN, *tN64, *xa, *e_atom, *fst;
    int64_t bytes;
};
Work carve_work(void* p, const GraphBuf& gb, int64_t nb, int64_t n, const int64_t* cnt) {
    const int64_t A = cnt[NB200_GOC_C_A2A], E = cnt[NB200_GOC_C_MAIN], P = cnt[NB200_GOC_C_AE], Q = cnt[NB200_GOC_C_Q], T = cnt[NB200_GOC_C_TIN];
    Carve c(p);
    Work w;
    auto graph = [&](int idx, int64_t ne, bool tgt, bool vec) {
        Graph g;
        g.ptr = gb.ptr ? gb.ptr + idx * (n + 1) : nullptr;
        g.src = c.take<int32_t>(ne);
        g.tgt = tgt ? c.take<int32_t>(ne) : nullptr;
        g.d = c.take<float>(ne);
        g.V = vec ? c.take<float>(3 * ne) : nullptr;
        return g;
    };
    w.a2a = graph(0, A, false, false);
    w.mn = graph(1, E, true, true);
    w.ae = graph(2, P, true, true);
    w.q = graph(3, Q, true, true);
    w.rev = c.take<int32_t>(E);
    w.q_tin = c.take<int32_t>(Q + 1);
    int64_t mx = A > E ? A : E;
    mx = mx > P ? mx : P;
    mx = mx > Q ? mx : Q;
    w.rb = c.take<float>(mx * NR);
    w.B_main = c.take<float>(E * LD_MAIN);
    w.B_ae = c.take<float>(P * LD_AE);
    w.B_q = c.take<float>(Q * LD_Q);
    w.B_a2a = c.take<float>(A * LD_A2A);
    w.cbf16 = c.take<float>(T * RB);
    w.h = c.take<float>(n * EA);
    w.m = c.take<float>(E * EE);
    w.hst = c.take<float>(n * 2 * EE);
    w.XE = c.take<float>(n * EA * (nb + 1));
    w.XF = c.take<float>(E * EE * (nb + 1));
    for (int k = 0; k < 3; k++) w.tE[k] = c.take<float>(E * EE);
    w.OE = c.take<float>(E * 1024);
    w.xdE = c.take<float>(E * TI);
    w.tE64 = c.take<float>(E * TI);
    w.yP = c.take<float>(P * EA);
    w.xdP = c.take<float>(P * TI);
    w.xt = c.take<float>(T * QI);
    for (int k = 0; k < 3; k++) w.tN[k] = c.take<float>(n * EE);
    w.ON = c.take<float>(n * 1024);
    w.xdN = c.take<float>(n * TI);
    w.tN64 = c.take<float>(n * TI);
    w.xa = c.take<float>(n * EA);
    w.e_atom = c.take<float>(n);
    w.fst = c.take<float>(E);
    w.bytes = c.off + 256;
    return w;
}

bool config_ok(const nb200_gemnet_oc_weights* w) {
    return w && w->w && w->off_host && w->scale_host && w->num_blocks >= 1 && w->num_blocks <= 16 && w->n_elem >= 1 && w->cutoff > 0.0f &&
           w->max_neighbors >= 1 && w->max_neighbors_qint >= 1 && w->max_neighbors_aeaint >= 1;
}

struct Ctx {
    nb200_engine* e; cudaStream_t s; const nb200_gemnet_oc_weights* w;
    const float* G(int idx, int64_t extra = 0) const { return w->w + w->off_host[idx] + extra; }
    const float* I(int blk, int idx, int64_t extra = 0) const { return w->w + w->off_host[NB200_GOC_G_COUNT + blk * NB200_GOC_I_COUNT + idx] + extra; }
    const float* O(int blk, int idx, int64_t extra = 0) const {
        return w->w + w->off_host[NB200_GOC_G_COUNT + w->num_blocks * NB200_GOC_I_COUNT + blk * NB200_GOC_O_COUNT + idx] + extra;
    }
    float SI(int blk, int idx) const { return w->scale_host[blk * NB200_GOC_S_COUNT + idx]; }
    float SO(int blk, int idx) const { return w->scale_host[w->num_blocks * NB200_GOC_S_COUNT + blk * NB200_GOC_SO_COUNT + idx]; }

    // M.n rows are computed whether or not M.dev says fewer: rows are independent, and no kernel reads a row at or past the device count
    int gemm(Ext Mx, int N, int K, const float* A, int lda, const float* W, int ldw, float* C, int ldc) const {
        const int64_t M = Mx.n;
        if (M <= 0) return NB200_OK;
        if (M > 0x7fffffff) return NB200_EUNSUPPORTED;
        if (goc_tc_ok(N, K, lda, ldw, ldc)) return goc_tc_gemm(e, s, (int)M, N, K, A, lda, W, ldw, C, ldc);
        return pfor(e, s, CAT_GEMM, M * N, LinK{A, lda, W, ldw, C, ldc, N, K});
    }
    int act(float* x, Ext M, int C) const { return pfor(e, s, CAT_NODE, M, C, SsiluK{x}); }
    // tall layers on the device: the activation / residual tail runs in the GEMM's epilogue (gemm_ps.cu NB_EPI_*) -- one pass over the
    // [M, N] output instead of GEMM store + elementwise load / store (SsiluK + ResOutK: ~400 launches per forward)
    bool fused_tail(int64_t M, int N, int K, const void* A, const void* C) const {
#ifdef NB_EMU
        (void)M; (void)N; (void)K; (void)A; (void)C;
        return false;
#else
        return A != C && M <= 0x7fffffff && goc_tc_ok(N, K, K, K, N) && nb_gemm_ps_wanted((int)M, N, K);
#endif
    }
    int dense_act(Ext Mx, int N, int K, const float* A, int lda, const float* W, float* C) const {
#ifndef NB_EMU
        const int64_t M = Mx.n;
        if (lda == K && fused_tail(M, N, K, A, C)) {
            Scope sc(e, s, CAT_GEMM, 2);
            return nb_gemm_ps_epi((int)M, N, K, A, lda, W, K, 0, C, N, nullptr, NB_EPI_ACT, NB_ACT_SSILU, 1.0f, s);
        }
#endif
        NB_TRY(gemm(Mx, N, K, A, lda, W, K, C, N));
        return act(C, Mx, N);
    }
    // ResidualLayer with two Dense layers stored back to back ([C,C] each): x = (x + act(W2 act(W1 x))) / sqrt 2
    int residual(Ext Mx, int C, float* x, const float* W, float* t1, float* t2) const {
        NB_TRY(dense_act(Mx, C, C, x, C, W, t1));
#ifndef NB_EMU
        const int64_t M = Mx.n;
        if (fused_tail(M, C, C, t1, x)) {
            Scope sc(e, s, CAT_GEMM, 2);
            return nb_gemm_ps_epi((int)M, C, C, t1, C, W + (int64_t)C * C, C, 0, x, C, nullptr, NB_EPI_RESIDUAL, NB_ACT_SSILU, ISQ2, s);
        }
#endif
        NB_TRY(gemm(Mx, C, C, t1, C, W + (int64_t)C * C, C, t2, C));
        return pfor(e, s, CAT_NODE, Mx, C, ResOutK{x, t2});
    }
};

int output_block(const Ctx& c, const Work& w, int blk, int64_t n, Ext E) {
    const int nb1 = c.w->num_blocks + 1;
    // energy branch (atom_update_block.py:141-160)
    NB_TRY(pfor(c.e, c.s, CAT_READOUT, n * EE, AggAtomRbfK{w.mn.ptr, w.m, w.B_main + C_RBF_OUT, LD_MAIN, c.O(blk, NB200_GOC_O_RBF), c.SO(blk, NB200_GOC_SO_SUM), w.tN[0]}));
    NB_TRY(c.dense_act(n, EA, EE, w.tN[0], EE, c.O(blk, NB200_GOC_O_L0), w.tN[1]));
    for (int k = 0; k < 3; k++) NB_TRY(c.residual(n, EA, w.tN[1], c.O(blk, NB200_GOC_O_RES, (int64_t)k * 2 * EA * EA), w.tN[2], w.tN[0]));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, n * EA, AddScaleK{w.tN[1], w.h, ISQ2}));
    for (int k = 0; k < 3; k++) NB_TRY(c.residual(n, EA, w.tN[1], c.O(blk, NB200_GOC_O_E2, (int64_t)k * 2 * EA * EA), w.tN[2], w.tN[0]));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, n * EA, CopyColsK{w.tN[1], EA, w.XE + (int64_t)blk * EA, EA * nb1}));
    // force branch (atom_update_block.py:162-170)
    NB_TRY(goc_d2d(w.tE[0], w.m, (size_t)E.n * EE * sizeof(float), c.s));
    for (int k = 0; k < 3; k++) NB_TRY(c.residual(E, EE, w.tE[0], c.O(blk, NB200_GOC_O_F, (int64_t)k * 2 * EE * EE), w.tE[1], w.tE[2]));
    return pfor(c.e, c.s, CAT_READOUT, MulRbfRowsK::count(E.n, EE),
                MulRbfRowsK{w.tE[0], EE, nullptr, w.B_main + C_RBF_OUT, LD_MAIN, c.O(blk, NB200_GOC_O_RBF_F), c.SO(blk, NB200_GOC_SO_RBF_F),
                            w.XF + (int64_t)blk * EE, EE * nb1, EE, 0, E.n, E.dev});
}


#ifndef NB_EMU
// Device form of QuadK (gemnet_oc_kernels.cuh; same sums in the same order, bitwise equal to the functor on the H100 --
// tests/test_gpu_gemnet_kernels.py checks both against each other and against float64).  The functor launches one logical thread per
// (edge, channel): the 32 channel-threads of an edge all recompute the
// geometry of every quadruplet -- two cross products, a square root, a division and the Legendre recurrence, more instructions than the
// 49 FMAs they feed.  Here a WARP owns the edge (lane =
// channel): 32 quadruplets at a time, lane j evaluates the dihedral basis of quadruplet j ONCE and stages it in shared memory; the warp
// then walks the staged rows (two broadcast 16-byte loads per quadruplet); the chunk's x_t rows travel by cp.async while the bases are computed
// (first version: plain loads four quadruplets ahead -- one L2 round trip per four quadruplets and warp).
constexpr int QW_WARPS = 8;
__device__ __forceinline__ void qw_cp16(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__global__ void __launch_bounds__(32 * QW_WARPS) k_quad_edges(Graph mn, Graph q, const int32_t* __restrict__ q_tin, const float* __restrict__ xt,
                                                             const float* __restrict__ R, int32_t ldr, float* __restrict__ O, int64_t E_bound,
                                                             const int32_t* __restrict__ E_dev) {
    const int64_t E = ext_rows(E_bound, E_dev);
    __shared__ __align__(16) float sY[QW_WARPS][32][8];   // [.][quadruplet][Y_0..6 of the dihedral, valid flag]
    __shared__ __align__(16) float sX[QW_WARPS][32][QI];  // [.][quadruplet][channel]: the x_t rows of the chunk (cp.async, in flight during the geometry)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t e = (int64_t)blockIdx.x * QW_WARPS + warp; e < E; e += (int64_t)gridDim.x * QW_WARPS) {
        const int32_t a = mn.tgt[e], c = mn.src[e];
        const float vca[3] = {mn.V[3 * e], mn.V[3 * e + 1], mn.V[3 * e + 2]};
        float S[NS2];  // S[l1 NS + l2]: the 7 x 7 update of a quadruplet
#pragma unroll
        for (int l = 0; l < NS2; l++) S[l] = 0.0f;
        for (int32_t qe = q.ptr[a]; qe < q.ptr[a + 1]; qe++) {
            const int32_t b = q.src[qe];
            if (b == c) continue;
            const float vba[3] = {q.V[3 * (int64_t)qe], q.V[3 * (int64_t)qe + 1], q.V[3 * (int64_t)qe + 2]};
            float Yp[NS], n1[3];
            cir7(clamp1(dot3(vca, vba)), Yp);
            cross3(vca, vba, n1);
            const int64_t t0 = q_tin[qe];
            const int32_t k0 = mn.ptr[b], nk = mn.ptr[b + 1] - k0;
            for (int32_t base = 0; base < nk; base += 32) {
                const int cnt = min(32, nk - base);
                __syncwarp();  // the previous chunk's rows have been read
                // x_t rows of this chunk: cnt rows of 128 bytes, 8 lanes x 16 bytes per row, 4 rows per instruction
                {
                    const float* src = xt + (t0 + base) * QI;
#pragma unroll
                    for (int r4 = 0; r4 < 32; r4 += 4) {
                        const int row = r4 + (lane >> 3);
                        if (row < cnt) qw_cp16(&sX[warp][row][(lane & 7) * 4], src + (int64_t)row * QI + (lane & 7) * 4);
                    }
                    asm volatile("cp.async.commit_group;" ::: "memory");
                }
                float Yt[NS];
                float ok = 0.0f;
#pragma unroll
                for (int l = 0; l < NS; l++) Yt[l] = 0.0f;
                if (base + lane < nk) {
                    const int32_t k = k0 + base + lane, d = mn.src[k];
                    if (d != a && d != c) {
                        float n2[3], n3[3];
                        cross3(mn.V + 3 * (int64_t)k, vba, n2);
                        const float xx = dot3(n1, n2);
                        cross3(n1, n2, n3);
                        const float yy = fmaxf(sqrtf(dot3(n3, n3)), 1e-9f);
                        cir7(xx / sqrtf(xx * xx + yy * yy), Yt);  // cos(atan2(y, x))
                        ok = 1.0f;
                    }
                }
                *reinterpret_cast<float4*>(&sY[warp][lane][0]) = make_float4(Yt[0], Yt[1], Yt[2], Yt[3]);
                *reinterpret_cast<float4*>(&sY[warp][lane][4]) = make_float4(Yt[4], Yt[5], Yt[6], ok);
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                __syncwarp();
#pragma unroll 4
                for (int j = 0; j < cnt; j++) {
                    const float4 yb = *reinterpret_cast<const float4*>(&sY[warp][j][4]);
                    if (yb.w == 0.0f) continue;
                    const float4 ya = *reinterpret_cast<const float4*>(&sY[warp][j][0]);
                    const float xv = sX[warp][j][lane];
                    const float yt[NS] = {ya.x, ya.y, ya.z, ya.w, yb.x, yb.y, yb.z};
#pragma unroll
                    for (int l1 = 0; l1 < NS; l1++) {
                        const float f = Yp[l1] * xv;
#pragma unroll
                        for (int l2 = 0; l2 < NS; l2++) S[l1 * NS + l2] = fmaf(f, yt[l2], S[l1 * NS + l2]);
                    }
                }
            }
        }
        const float* Re = R + e * ldr;
        for (int i32 = 0; i32 < 32; i32++) {
            float acc = 0.0f;
#pragma unroll
            for (int s = 0; s < NS2; s++) acc += __ldg(Re + i32 * NS2 + s) * S[s];
            O[e * 1024 + i32 * QI + lane] = acc;
        }
    }
}
#endif
#ifndef NB_EMU
// Device form of TripEdgeK (same sums in the same order, bitwise equal to the functor on the H100; tests/test_gpu_gemnet_kernels.py): a warp
// owns an output edge, lane = channels (lane, lane + 32); 32 input edges at a time,
// lane j evaluates the Legendre basis of the angle to input edge j ONCE (the functor's 64 channel-threads each did) and stages it in shared memory.
constexpr int TW_WARPS = 8;
__global__ void __launch_bounds__(32 * TW_WARPS) k_trip_edges(Graph o, Graph in, const float* __restrict__ x, const float* __restrict__ R, int32_t ldr,
                                                             float* __restrict__ O, int64_t E_bound, const int32_t* __restrict__ E_dev) {
    const int64_t E = ext_rows(E_bound, E_dev);
    __shared__ __align__(16) float sY[TW_WARPS][32][8];  // [.][input edge][Y_0..6, valid flag]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t e = (int64_t)blockIdx.x * TW_WARPS + warp; e < E; e += (int64_t)gridDim.x * TW_WARPS) {
        const int32_t a = o.tgt[e], cs = o.src[e];
        const float v[3] = {o.V[3 * e], o.V[3 * e + 1], o.V[3 * e + 2]};
        float S0[NS], S1[NS];
#pragma unroll
        for (int s = 0; s < NS; s++) { S0[s] = 0.0f; S1[s] = 0.0f; }
        const int32_t k0 = in.ptr[a], nk = in.ptr[a + 1] - k0;
        for (int32_t base = 0; base < nk; base += 32) {
            float Y[NS];
            float ok = 0.0f;
#pragma unroll
            for (int l = 0; l < NS; l++) Y[l] = 0.0f;
            if (base + lane < nk) {
                const int32_t k = k0 + base + lane;
                if (in.src[k] != cs) { cir7(clamp1(dot3(v, in.V + 3 * (int64_t)k)), Y); ok = 1.0f; }
            }
            __syncwarp();
            *reinterpret_cast<float4*>(&sY[warp][lane][0]) = make_float4(Y[0], Y[1], Y[2], Y[3]);
            *reinterpret_cast<float4*>(&sY[warp][lane][4]) = make_float4(Y[4], Y[5], Y[6], ok);
            __syncwarp();
            const int cnt = min(32, nk - base);
            const float* xr = x + (int64_t)(k0 + base) * TI + lane;
            for (int j0 = 0; j0 < cnt; j0 += 4) {
                float xa[4], xb[4];
#pragma unroll
                for (int u = 0; u < 4; u++) { const int64_t off = (int64_t)min(j0 + u, cnt - 1) * TI; xa[u] = xr[off]; xb[u] = xr[off + 32]; }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (j0 + u >= cnt) break;
                    const float4 ya = *reinterpret_cast<const float4*>(&sY[warp][j0 + u][0]);
                    const float4 yb = *reinterpret_cast<const float4*>(&sY[warp][j0 + u][4]);
                    if (yb.w == 0.0f) continue;
                    const float y7[NS] = {ya.x, ya.y, ya.z, ya.w, yb.x, yb.y, yb.z};
#pragma unroll
                    for (int s = 0; s < NS; s++) { S0[s] += y7[s] * xa[u]; S1[s] += y7[s] * xb[u]; }
                }
            }
        }
        const float* Re = R + e * ldr;
        for (int i16 = 0; i16 < 16; i16++) {
            float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
            for (int s = 0; s < NS; s++) { const float r = __ldg(Re + i16 * NS + s); a0 += r * S0[s]; a1 += r * S1[s]; }
            O[e * 1024 + i16 * TI + lane] = a0;
            O[e * 1024 + i16 * TI + 32 + lane] = a1;
        }
    }
}
#endif
int trip_edge_aggregate(nb200_engine* eng, cudaStream_t s, const Graph& o, const Graph& in, const float* x, const float* R, int32_t ldr, float* O, Ext E) {
#ifdef NB_EMU
    return pfor(eng, s, CAT_MSG_FWD, E, TI, TripEdgeK{o, in, x, R, ldr, O});
#else
    if (E.n <= 0) return NB200_OK;
    Scope sc(eng, s, CAT_MSG_FWD, 1);
    const int64_t want = (E.n + TW_WARPS - 1) / TW_WARPS;
    k_trip_edges<<<(int)(want < nb_sm_count() * 8 ? want : nb_sm_count() * 8), 32 * TW_WARPS, 0, s>>>(o, in, x, R, ldr, O, E.n, E.dev);
    return nb_check_launch();
#endif
}
int quad_aggregate(nb200_engine* eng, cudaStream_t s, const Graph& mn, const Graph& q, const int32_t* q_tin, const float* xt, const float* R, int32_t ldr,
                   float* O, Ext E) {
#ifdef NB_EMU
    return pfor(eng, s, CAT_MSG_FWD, E, QI, QuadK{mn, q, q_tin, xt, R, ldr, O});
#else
    if (E.n <= 0) return NB200_OK;
    Scope sc(eng, s, CAT_MSG_FWD, 1);
    const int64_t want = (E.n + QW_WARPS - 1) / QW_WARPS;
    k_quad_edges<<<(int)(want < nb_sm_count() * 8 ? want : nb_sm_count() * 8), 32 * QW_WARPS, 0, s>>>(mn, q, q_tin, xt, R, ldr, O, E.n, E.dev);
    return nb_check_launch();
#endif
}

// act(x_pre) * mlp_rbf(basis), scale, down projection with activation (the common head of every interaction); `xsrc` holds the
// pre-activation of dense_ba / dense_db unless act_in = 0
int down_path(const Ctx& c, Ext M, int C, float* x, const int32_t* row_idx, const float* xsrc, int act_in, const float* rbf, int ldr, const float* Wrbf,
              float scale, const float* Wdown, int n_down, float* xd) {
    NB_TRY(pfor(c.e, c.s, CAT_NODE, MulRbfRowsK::count(M.n, C), MulRbfRowsK{xsrc, C, row_idx, rbf, ldr, Wrbf, scale, x, C, C, act_in, M.n, M.dev}));
    return c.dense_act(M, n_down, C, x, C, Wdown, xd);
}

int interaction_block(const Ctx& c, const Work& w, int blk, int64_t n, Ext E, Ext P, Ext Q) {
    float *x = w.tE[0], *t1 = w.tE[1], *t2 = w.tE[2];
    NB_TRY(c.gemm(E, EE, EE, w.m, EE, c.I(blk, NB200_GOC_I_DENSE_CA), EE, x, EE));  // pre-activation; activated by the first SymAddK
    // --- triplet interaction, edges -> edges (interaction_block.py TripletInteraction)
    NB_TRY(c.gemm(E, EE, EE, w.m, EE, c.I(blk, NB200_GOC_I_T_BA), EE, t1, EE));
    NB_TRY(down_path(c, E, EE, t1, nullptr, t1, 1, w.B_main + C_RBF_TINT, LD_MAIN, c.I(blk, NB200_GOC_I_T_RBF), c.SI(blk, NB200_GOC_S_T_RBF), c.I(blk, NB200_GOC_I_T_DOWN), TI, w.xdE));
    NB_TRY(trip_edge_aggregate(c.e, c.s, w.mn, w.mn, w.xdE, w.B_main + C_R_TINT, LD_MAIN, w.OE, E));
    NB_TRY(c.gemm(E, TI, 1024, w.OE, 1024, c.I(blk, NB200_GOC_I_T_BIL), 1024, w.tE64, TI));  // scale_cbf_sum folded into the weights
    NB_TRY(c.gemm(E, EE, TI, w.tE64, TI, c.I(blk, NB200_GOC_I_T_UPCA), TI, t1, EE));
    NB_TRY(c.gemm(E, EE, TI, w.tE64, TI, c.I(blk, NB200_GOC_I_T_UPAC), TI, t2, EE));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, EE, SymAddK{x, t1, t2, w.rev, 1, 1.0f}));
    // --- quadruplet interaction
    NB_TRY(c.gemm(E, EE, EE, w.m, EE, c.I(blk, NB200_GOC_I_Q_DB), EE, t1, EE));
    NB_TRY(down_path(c, E, EE, t1, nullptr, t1, 1, w.B_main + C_RBF_QINT, LD_MAIN, c.I(blk, NB200_GOC_I_Q_RBF), c.SI(blk, NB200_GOC_S_Q_RBF), c.I(blk, NB200_GOC_I_Q_DOWN), QI, w.xdE));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, Q, QI, QuadXtK{w.q, w.mn, w.q_tin, w.xdE, w.cbf16, c.I(blk, NB200_GOC_I_Q_CBF), c.SI(blk, NB200_GOC_S_Q_CBF), w.xt}));
    NB_TRY(quad_aggregate(c.e, c.s, w.mn, w.q, w.q_tin, w.xt, w.B_main + C_R_SBF, LD_MAIN, w.OE, E));
    NB_TRY(c.gemm(E, QI, 1024, w.OE, 1024, c.I(blk, NB200_GOC_I_Q_BIL), 1024, w.tE64, QI));
    NB_TRY(c.gemm(E, EE, QI, w.tE64, QI, c.I(blk, NB200_GOC_I_Q_UPCA), QI, t1, EE));
    NB_TRY(c.gemm(E, EE, QI, w.tE64, QI, c.I(blk, NB200_GOC_I_Q_UPAC), QI, t2, EE));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, EE, SymAddK{x, t1, t2, w.rev, 0, 1.0f}));
    // --- atoms -> edges
    NB_TRY(c.dense_act(n, EA, EA, w.h, EA, c.I(blk, NB200_GOC_I_AE_BA), w.xa));  // activated once per atom, gathered per a2ee2a edge below
    NB_TRY(down_path(c, P, EA, w.yP, w.ae.src, w.xa, 0, w.B_ae + C_AE_RBF, LD_AE, c.I(blk, NB200_GOC_I_AE_RBF), c.SI(blk, NB200_GOC_S_AE_RBF), c.I(blk, NB200_GOC_I_AE_DOWN), TI, w.xdP));
    NB_TRY(trip_edge_aggregate(c.e, c.s, w.mn, w.ae, w.xdP, w.B_main + C_R_AEINT, LD_MAIN, w.OE, E));
    NB_TRY(c.gemm(E, TI, 1024, w.OE, 1024, c.I(blk, NB200_GOC_I_AE_BIL), 1024, w.tE64, TI));
    NB_TRY(c.gemm(E, EE, TI, w.tE64, TI, c.I(blk, NB200_GOC_I_AE_UPCA), TI, t1, EE));
    NB_TRY(c.gemm(E, EE, TI, w.tE64, TI, c.I(blk, NB200_GOC_I_AE_UPAC), TI, t2, EE));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, EE, SymAddK{x, t1, t2, w.rev, 0, 0.5f}));  // 1 / sqrt(4 merged branches)
    // --- edges -> atoms
    NB_TRY(c.gemm(E, EE, EE, w.m, EE, c.I(blk, NB200_GOC_I_EA_BA), EE, t1, EE));
    NB_TRY(down_path(c, E, EE, t1, nullptr, t1, 1, w.B_main + C_RBF_EAINT, LD_MAIN, c.I(blk, NB200_GOC_I_EA_RBF), c.SI(blk, NB200_GOC_S_EA_RBF), c.I(blk, NB200_GOC_I_EA_DOWN), TI, w.xdE));
    NB_TRY(pfor(c.e, c.s, CAT_MSG_FWD, n * TI, TripAtomK{w.ae, w.mn, w.xdE, w.B_ae + C_AE_R, LD_AE, w.ON}));
    NB_TRY(c.gemm(n, TI, 1024, w.ON, 1024, c.I(blk, NB200_GOC_I_EA_BIL), 1024, w.tN64, TI));
    NB_TRY(c.gemm(n, EA, TI, w.tN64, TI, c.I(blk, NB200_GOC_I_EA_UP), TI, w.tN[0], EA));
    // --- atoms -> atoms
    NB_TRY(c.dense_act(n, TI, EA, w.h, EA, c.I(blk, NB200_GOC_I_AA_DOWN), w.xdN));
    NB_TRY(pfor(c.e, c.s, CAT_MSG_FWD, n * TI, PairK{w.a2a.ptr, w.a2a.src, w.B_a2a, LD_A2A, w.xdN, w.ON}));
    NB_TRY(c.gemm(n, TI, 1024, w.ON, 1024, c.I(blk, NB200_GOC_I_AA_BIL), 1024, w.tN64, TI));
    NB_TRY(c.gemm(n, EA, TI, w.tN64, TI, c.I(blk, NB200_GOC_I_AA_UP), TI, w.tN[1], EA));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, n * EA, CombineHK{w.h, w.tN[0], w.tN[1]}));
    // --- edge update
    for (int k = 0; k < 2; k++) NB_TRY(c.residual(E, EE, x, c.I(blk, NB200_GOC_I_BEFORE_SKIP, (int64_t)k * 2 * EE * EE), t1, t2));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, EE, AddScaleK{w.m, x, ISQ2}));
    for (int k = 0; k < 2; k++) NB_TRY(c.residual(E, EE, w.m, c.I(blk, NB200_GOC_I_AFTER_SKIP, (int64_t)k * 2 * EE * EE), t1, t2));
    // --- atom update (atom_update_block.py:15-91)
    NB_TRY(pfor(c.e, c.s, CAT_NODE, n * EE, AggAtomRbfK{w.mn.ptr, w.m, w.B_main + C_RBF_H, LD_MAIN, c.I(blk, NB200_GOC_I_AU_RBF), c.SI(blk, NB200_GOC_S_AU_SUM), w.tN[0]}));
    NB_TRY(c.dense_act(n, EA, EE, w.tN[0], EE, c.I(blk, NB200_GOC_I_AU_L0), w.tN[1]));
    for (int k = 0; k < 3; k++) NB_TRY(c.residual(n, EA, w.tN[1], c.I(blk, NB200_GOC_I_AU_RES, (int64_t)k * 2 * EA * EA), w.tN[2], w.tN[0]));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, n * EA, AddScaleK{w.h, w.tN[1], ISQ2}));
    // --- edge embedding from the new atom embeddings, residual, skip
    const float* Wc = c.I(blk, NB200_GOC_I_CONCAT);
    NB_TRY(c.gemm(n, EE, EA, w.h, EA, Wc, 2 * EE, w.hst, 2 * EE));
    NB_TRY(c.gemm(n, EE, EA, w.h, EA, Wc + EA, 2 * EE, w.hst + EE, 2 * EE));
    NB_TRY(c.gemm(E, EE, EE, w.m, EE, Wc + 2 * EA, 2 * EE, t1, EE));
    NB_TRY(pfor(c.e, c.s, CAT_EMBED, E, EE, EdgeEmbK{w.hst, t1, w.mn.src, w.mn.tgt, x}));
    NB_TRY(c.residual(E, EE, x, c.I(blk, NB200_GOC_I_RES_M), t1, t2));
    return pfor(c.e, c.s, CAT_NODE, E, EE, AddScaleK{w.m, x, ISQ2});
}

// graph phase: nearest-neighbour ranks, degrees, row pointers of the four graphs and the input-triplet slot bases; the five counts end up
// in g.ptr[k][n] and g.tbase[n] on the device
int graph_phase(nb200_engine* e, cudaStream_t s, const nb200_gemnet_oc_weights* w, const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n, int32_t Mx,
                const GraphBuf& g) {
    NB_TRY(pfor(e, s, CAT_NBR, n, MolIdK{mol_ptr, n_mol, g.mol_id}));
    NB_TRY(pfor(e, s, CAT_NBR, (int64_t)n * Mx, RankK{pos, mol_ptr, g.mol_id, Mx, w->cutoff * w->cutoff, g.rank}));
    const PairSel sel{g.rank, Mx, w->max_neighbors, w->max_neighbors_aeaint, w->max_neighbors_qint};
    NB_TRY(pfor(e, s, CAT_NBR, n, DegK{sel, mol_ptr, g.mol_id, n, g.deg}));
    NB_TRY(pfor(e, s, CAT_NBR, n, TcountK{sel, mol_ptr, g.mol_id, g.deg + n, g.tcnt}));
    for (int k = 0; k < 4; k++) NB_TRY(scan_excl(e, s, g.deg + (int64_t)k * n, n, g.ptr + (int64_t)k * (n + 1)));
    return scan_excl(e, s, g.tcnt, n, g.tbase);
}

// model phase, shared by the two-phase and the asynchronous entry: A, E, P, Q are the extents of the four edge lists (exact counts, or
// upper bounds with the counts on the device), `err` the status word FillK honours (nullptr in the two-phase form)
int model_phase(const Ctx& c, const GraphBuf& g, const Work& wk, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                int32_t max_atoms_per_mol, Ext A, Ext E, Ext P, Ext Q, bool any_triplets, const int32_t* err, float* energy, float* forces) {
    nb200_engine* eng = c.e;
    cudaStream_t s = c.s;
    const nb200_gemnet_oc_weights* w = c.w;
    const int64_t n = n_atoms;
    const int nb = w->num_blocks;
    // edge lists, geometry, id_swap
    const PairSel sel{g.rank, max_atoms_per_mol, w->max_neighbors, w->max_neighbors_aeaint, w->max_neighbors_qint};
    NB_TRY(pfor(eng, s, CAT_NBR, n, FillK{sel, pos, mol_ptr, g.mol_id, g.deg + n, g.tbase, n_atoms, wk.a2a, wk.mn, wk.ae, wk.q, wk.q_tin, err}));
    NB_TRY(pfor(eng, s, CAT_NBR, E, 1, RevK{wk.mn.ptr, wk.mn.src, wk.mn.tgt, wk.rev}));
    // radial bases and their embeddings: one GEMM per graph against the concatenated (scale-folded) basis matrices
    const float inv_cut = 1.0f / w->cutoff, coeff = -0.5f * (float)(NR - 1) * (float)(NR - 1);
    const float* off = c.G(NB200_GOC_G_RBF_OFFSET);
    NB_TRY(pfor(eng, s, CAT_FILTER, E, NR, RbfK{wk.mn.d, off, inv_cut, coeff, wk.rb}));
    NB_TRY(c.gemm(E, LD_MAIN, NR, wk.rb, NR, c.G(NB200_GOC_G_CAT_MAIN), NR, wk.B_main, LD_MAIN));
    NB_TRY(c.gemm(E, EE, NR, wk.rb, NR, c.G(NB200_GOC_G_EDGE_EMB, 2 * EA), 2 * EA + NR, wk.tE[1], EE));  // radial columns of the edge embedding
    NB_TRY(pfor(eng, s, CAT_FILTER, P, NR, RbfK{wk.ae.d, off, inv_cut, coeff, wk.rb}));
    NB_TRY(c.gemm(P, LD_AE, NR, wk.rb, NR, c.G(NB200_GOC_G_CAT_AE), NR, wk.B_ae, LD_AE));
    NB_TRY(pfor(eng, s, CAT_FILTER, Q, NR, RbfK{wk.q.d, off, inv_cut, coeff, wk.rb}));
    NB_TRY(c.gemm(Q, LD_Q, NR, wk.rb, NR, c.G(NB200_GOC_G_CAT_Q), NR, wk.B_q, LD_Q));
    NB_TRY(pfor(eng, s, CAT_FILTER, A, NR, RbfK{wk.a2a.d, off, inv_cut, coeff, wk.rb}));
    NB_TRY(c.gemm(A, LD_A2A, NR, wk.rb, NR, c.G(NB200_GOC_G_CAT_A2A), NR, wk.B_a2a, LD_A2A));
    if (any_triplets) NB_TRY(pfor(eng, s, CAT_FILTER, Q, RB, QuadCbfK{wk.q, wk.mn, wk.q_tin, wk.B_q, wk.cbf16}));
    // embeddings
    NB_TRY(pfor(eng, s, CAT_EMBED, n * EA, EmbedK{z, c.G(NB200_GOC_G_EMB), w->n_elem, wk.h}));
    const float* We = c.G(NB200_GOC_G_EDGE_EMB);
    NB_TRY(c.gemm(n, EE, EA, wk.h, EA, We, 2 * EA + NR, wk.hst, 2 * EE));
    NB_TRY(c.gemm(n, EE, EA, wk.h, EA, We + EA, 2 * EA + NR, wk.hst + EE, 2 * EE));
    NB_TRY(pfor(eng, s, CAT_EMBED, E, EE, EdgeEmbK{wk.hst, wk.tE[1], wk.mn.src, wk.mn.tgt, wk.m}));
    NB_TRY(output_block(c, wk, 0, n, E));
    for (int b = 0; b < nb; b++) {
        NB_TRY(interaction_block(c, wk, b, n, E, P, Q));
        NB_TRY(output_block(c, wk, b + 1, n, E));
    }
    // global output MLPs (gemnet_oc.py:1160-1215)
    NB_TRY(c.dense_act(n, EA, EA * (nb + 1), wk.XE, EA * (nb + 1), c.G(NB200_GOC_G_OUT_E0), wk.tN[1]));
    for (int k = 0; k < 2; k++) NB_TRY(c.residual(n, EA, wk.tN[1], c.G(NB200_GOC_G_OUT_E_RES, (int64_t)k * 2 * EA * EA), wk.tN[2], wk.tN[0]));
    NB_TRY(pfor(eng, s, CAT_READOUT, n, DotRowK{wk.tN[1], EA, c.G(NB200_GOC_G_OUT_ENERGY), wk.e_atom}));
    NB_TRY(pfor(eng, s, CAT_READOUT, n_mol, MolEnergyK{mol_ptr, wk.e_atom, energy}));
    NB_TRY(c.dense_act(E, EE, EE * (nb + 1), wk.XF, EE * (nb + 1), c.G(NB200_GOC_G_OUT_F0), wk.tE[0]));
    for (int k = 0; k < 2; k++) NB_TRY(c.residual(E, EE, wk.tE[0], c.G(NB200_GOC_G_OUT_F_RES, (int64_t)k * 2 * EE * EE), wk.tE[1], wk.tE[2]));
    NB_TRY(pfor(eng, s, CAT_READOUT, E, 1, DotRowK{wk.tE[0], EE, c.G(NB200_GOC_G_OUT_FORCES), wk.fst}));
    return pfor(eng, s, CAT_FORCE, n, ForceK{wk.mn.ptr, wk.rev, wk.fst, wk.mn.V, forces});
}

}  // namespace

extern "C" int64_t nb200_gemnet_oc_graph_bytes(int32_t n_atoms, int32_t max_atoms_per_mol) {
    if (n_atoms < 0 || max_atoms_per_mol < 1) return NB200_EINVAL;
    return carve_graph(nullptr, n_atoms, max_atoms_per_mol).bytes;
}

extern "C" int nb200_gemnet_oc_graph_count(const nb200_gemnet_oc_weights* w, const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                                           int32_t max_atoms_per_mol, void* graph_buf, int64_t graph_bytes, int64_t* counts_host, void* stream) {
    if (!config_ok(w) || !pos || !mol_ptr || !graph_buf || !counts_host || n_mol < 1 || n_atoms < 1 || max_atoms_per_mol < 1) return NB200_EINVAL;
    if (graph_bytes < carve_graph(nullptr, n_atoms, max_atoms_per_mol).bytes) return NB200_EINVAL;  // before any pointer is formed
    const GraphBuf g = carve_graph(graph_buf, n_atoms, max_atoms_per_mol);
    cudaStream_t s = (cudaStream_t)stream;
    nb200_engine* e = nullptr;
    const int32_t n = n_atoms;
#ifndef NB_EMU
    nb200_engine tmp_engine{};  // launch counting only; no cuBLAS handle is touched by the graph kernels
    e = &tmp_engine;
#endif
    NB_TRY(graph_phase(e, s, w, pos, mol_ptr, n_mol, n, max_atoms_per_mol, g));
    int32_t tot[5];
    for (int k = 0; k < 4; k++) NB_TRY(goc_d2h_sync(&tot[k], g.ptr + (int64_t)k * (n + 1) + n, sizeof(int32_t), s));
    NB_TRY(goc_d2h_sync(&tot[4], g.tbase + n, sizeof(int32_t), s));
    for (int k = 0; k < NB200_GOC_C_COUNT; k++) counts_host[k] = 0;
    for (int k = 0; k < 5; k++) {
        if (tot[k] < 0) return NB200_ECAPACITY;  // int32 overflow of an edge count
        counts_host[k] = tot[k];
    }
    return NB200_OK;
}

// Upper bounds of the five counts from the molecule sizes alone.  Every graph lives inside one molecule, so for a molecule of m atoms
// (PairSel::get decides membership from rank[a, j], the position of source j among the in-cutoff neighbours of target a, nearest first):
extern "C" int nb200_gemnet_oc_count_bounds(const nb200_gemnet_oc_weights* w, const int32_t* mol_ptr_host, int32_t n_mol, int64_t* counts_bound_host) {
    if (!config_ok(w) || !mol_ptr_host || !counts_bound_host || n_mol < 1 || mol_ptr_host[0] != 0) return NB200_EINVAL;
    int64_t b[NB200_GOC_C_COUNT] = {};
    for (int32_t i = 0; i < n_mol; i++) {
        const int64_t m = (int64_t)mol_ptr_host[i + 1] - mol_ptr_host[i];
        if (m < 1) return NB200_EINVAL;
        const auto capped = [m](int64_t cap) { return m * (cap < m - 1 ? cap : m - 1); };
        // a2a: rank != RANK_NONE, i.e. every other atom of the molecule inside the cutoff: at most m - 1 sources per target
        b[NB200_GOC_C_A2A] += m * (m - 1);
        // a2ee2a, qint: rank < cap and ranks of one target are distinct: at most min(cap, m - 1) sources per target
        b[NB200_GOC_C_AE] += capped(w->max_neighbors_aeaint);
        const int64_t q = capped(w->max_neighbors_qint);
        b[NB200_GOC_C_Q] += q;
        // main: the unordered pair {j < a} is kept iff rank[a, j] < max_neighbors, i.e. iff the LOWER-index atom is among the nearest
        // max_neighbors of the HIGHER-index one.  The atom with k lower-index mates (k = 0 .. m - 1) keeps at most min(max_neighbors, k)
        // such pairs, each pair is two directed edges; no atom exceeds m - 1 edges (DegK counts sources j != a of its molecule)
        int64_t pairs = 0;
        for (int64_t k = 0; k < m; k++) pairs += k < w->max_neighbors ? k : w->max_neighbors;
        b[NB200_GOC_C_MAIN] += 2 * pairs;
        // input-triplet slots: TcountK adds deg_main(source) <= m - 1 for every qint edge
        b[NB200_GOC_C_TIN] += q * (m - 1);
    }
    for (int k = 0; k < NB200_GOC_C_COUNT; k++) {
        if (b[k] > 0x7fffffff) return NB200_EINVAL;  // the engine indexes edges with int32
        counts_bound_host[k] = b[k];
    }
    return NB200_OK;
}

extern "C" int64_t nb200_gemnet_oc_workspace_bytes(const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host) {
    if (!config_ok(w) || !counts_host || n_mol < 1 || n_atoms < 1) return NB200_EINVAL;
    GraphBuf none{};
    return carve_work(nullptr, none, w->num_blocks, n_atoms, counts_host).bytes;
}

extern "C" int nb200_gemnet_oc_energy_forces(nb200_engine* eng, const nb200_gemnet_oc_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                             int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol, void* graph_buf, int64_t graph_bytes,
                                             const int64_t* counts_host, void* workspace, int64_t workspace_bytes, float* energy, float* forces, void* stream) {
    if (!eng || !config_ok(w) || !z || !pos || !mol_ptr || !graph_buf || !counts_host || !workspace || !energy || !forces || n_mol < 1 || n_atoms < 1)
        return NB200_EINVAL;
    {
        GraphBuf none{};
        if (max_atoms_per_mol < 1 || graph_bytes < carve_graph(nullptr, n_atoms, max_atoms_per_mol).bytes ||
            workspace_bytes < carve_work(nullptr, none, w->num_blocks, n_atoms, counts_host).bytes)
            return NB200_EINVAL;  // before any pointer is formed
    }
    const GraphBuf g = carve_graph(graph_buf, n_atoms, max_atoms_per_mol);
    const Work wk = carve_work(workspace, g, w->num_blocks, n_atoms, counts_host);
    if (counts_host[NB200_GOC_C_MAIN] < 1) return NB200_ENOEDGES;
    const Ctx c{eng, (cudaStream_t)stream, w};
    return model_phase(c, g, wk, z, pos, mol_ptr, n_mol, n_atoms, max_atoms_per_mol, counts_host[NB200_GOC_C_A2A], counts_host[NB200_GOC_C_MAIN],
                       counts_host[NB200_GOC_C_AE], counts_host[NB200_GOC_C_Q], counts_host[NB200_GOC_C_TIN] > 0, nullptr, energy, forces);
}

// Graph phase and model phase in one enqueue: the counts never leave the device, every extent is sized by its bound (DESIGN.md 3.9)
extern "C" int nb200_gemnet_oc_energy_forces_async(nb200_engine* eng, const nb200_gemnet_oc_weights* w, const int32_t* z, const float* pos,
                                                   const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol, void* graph_buf,
                                                   int64_t graph_bytes, const int64_t* counts_bound_host, void* workspace, int64_t workspace_bytes,
                                                   float* energy, float* forces, int32_t* status, void* stream) {
    if (!eng || !config_ok(w) || !z || !pos || !mol_ptr || !graph_buf || !counts_bound_host || !workspace || !energy || !forces || !status || n_mol < 1 ||
        n_atoms < 1 || max_atoms_per_mol < 1)
        return NB200_EINVAL;
    for (int k = 0; k < 5; k++)
        if (counts_bound_host[k] < 0 || counts_bound_host[k] > 0x7fffffff) return NB200_EINVAL;
    {
        GraphBuf none{};
        if (graph_bytes < carve_graph(nullptr, n_atoms, max_atoms_per_mol).bytes ||
            workspace_bytes < carve_work(nullptr, none, w->num_blocks, n_atoms, counts_bound_host).bytes)
            return NB200_EINVAL;  // before any pointer is formed
    }
    const GraphBuf g = carve_graph(graph_buf, n_atoms, max_atoms_per_mol);
    const Work wk = carve_work(workspace, g, w->num_blocks, n_atoms, counts_bound_host);
    cudaStream_t s = (cudaStream_t)stream;
    const int32_t n = n_atoms;
    NB_TRY(graph_phase(eng, s, w, pos, mol_ptr, n_mol, n, max_atoms_per_mol, g));
    // the counts against their bounds BEFORE any edge is written; on an error every row pointer is cleared, FillK writes nothing
    NB_TRY(goc_memset(status, 0, 8 * sizeof(int32_t), s));
    NB_TRY(pfor(eng, s, CAT_NBR, n, StatusAtomK{pos, g.deg + n, status}));
    StatusCountsK sc{g.ptr, g.tbase, n, {}, status};
    for (int k = 0; k < 5; k++) sc.bound[k] = (int32_t)counts_bound_host[k];
    NB_TRY(pfor(eng, s, CAT_NBR, 1, sc));
    NB_TRY(pfor(eng, s, CAT_NBR, 5 * ((int64_t)n + 1), ClearOnErrorK{status, g.ptr, 4 * ((int64_t)n + 1), g.tbase}));
    const auto ext = [&](int k) { return Ext(counts_bound_host[k], g.ptr + (int64_t)(k) * (n + 1) + n); };
    static_assert(NB200_GOC_C_A2A == 0 && NB200_GOC_C_MAIN == 1 && NB200_GOC_C_AE == 2 && NB200_GOC_C_Q == 3, "g.ptr holds the graphs in the order of the counts");
    const Ctx c{eng, s, w};
    NB_TRY(model_phase(c, g, wk, z, pos, mol_ptr, n_mol, n_atoms, max_atoms_per_mol, ext(NB200_GOC_C_A2A), ext(NB200_GOC_C_MAIN), ext(NB200_GOC_C_AE),
                       ext(NB200_GOC_C_Q), counts_bound_host[NB200_GOC_C_TIN] > 0, status + 1, energy, forces));
    return pfor(eng, s, CAT_READOUT, (int64_t)n_mol + 3 * (int64_t)n, NanOnErrorK{status, energy, n_mol, forces});
}

extern "C" int nb200_gemnet_oc_debug_h(const void* workspace, const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host,
                                       float* h_out, void* stream) {
    if (!workspace || !config_ok(w) || !counts_host || !h_out || n_mol < 1 || n_atoms < 1) return NB200_EINVAL;
    GraphBuf none{};
    const Work wk = carve_work(const_cast<void*>(workspace), none, w->num_blocks, n_atoms, counts_host);
    return goc_d2d(h_out, wk.h, (size_t)n_atoms * EA * sizeof(float), (cudaStream_t)stream);
}

#include "gemnet_oc_train.inc"
#include "gemnet_oc_jvp.inc"

// One aggregation on caller-built graphs (include/nabla_b200.h), so that the warp-per-edge device kernels can be compared with the functors
// and with a float64 reference on row shapes the fixture molecules never produce
extern "C" int nb200_gemnet_oc_test_aggregate(const nb200_gemnet_oc_agg_args* a, void* stream) {
    if (!a || a->E_bound < 0 || a->E_bound > 0x7fffffff || (a->form != 0 && a->form != 1) || (a->quad != 0 && a->quad != 1) ||
        (a->tangent != 0 && a->tangent != 1))
        return NB200_EINVAL;
    const bool quad = a->quad, tangent = a->tangent;
    if (a->ldr < (quad ? 32 * NS2 : 16 * NS)) return NB200_EINVAL;
    if (!a->o_src || !a->o_tgt || !a->o_V || !a->in_ptr || !a->in_src || !a->in_V || !a->x || !a->R || (quad && (!a->o_ptr || !a->q_tin)))
        return NB200_EINVAL;
    if (tangent ? (a->E_dev || !a->Vot || !a->Vit || !a->xt || !a->Rt || !a->Ot) : !a->O) return NB200_EINVAL;
    const Graph o{a->o_ptr, const_cast<int32_t*>(a->o_src), const_cast<int32_t*>(a->o_tgt), nullptr, const_cast<float*>(a->o_V)};
    const Graph in{a->in_ptr, const_cast<int32_t*>(a->in_src), nullptr, nullptr, const_cast<float*>(a->in_V)};
    cudaStream_t s = (cudaStream_t)stream;
    nb200_engine* e = nullptr;
#ifndef NB_EMU
    nb200_engine tmp_engine{};  // launch counting only
    e = &tmp_engine;
#endif
    const Ext E(a->E_bound, a->E_dev);
    if (!tangent) {
        if (a->form == 0)
            return quad ? quad_aggregate(e, s, o, in, a->q_tin, a->x, a->R, a->ldr, a->O, E) : trip_edge_aggregate(e, s, o, in, a->x, a->R, a->ldr, a->O, E);
        return quad ? pfor(e, s, CAT_MSG_FWD, E, QI, QuadK{o, in, a->q_tin, a->x, a->R, a->ldr, a->O})
                    : pfor(e, s, CAT_MSG_FWD, E, TI, TripEdgeK{o, in, a->x, a->R, a->ldr, a->O});
    }
    if (quad) {
        const QuadTK f{o, in, a->Vot, a->Vit, a->q_tin, a->x, a->xt, a->R, a->Rt, a->ldr, a->Ot};
        return a->form == 0 ? quad_aggregate_t(e, s, f, a->E_bound) : pfor(e, s, CAT_MSG_FWD, a->E_bound * QI, f);
    }
    const TripEdgeTK f{o, in, a->Vot, a->Vit, a->x, a->xt, a->R, a->Rt, a->ldr, a->Ot};
    return a->form == 0 ? trip_edge_aggregate_t(e, s, f, a->E_bound) : pfor(e, s, CAT_MSG_FWD, a->E_bound * TI, f);
}
