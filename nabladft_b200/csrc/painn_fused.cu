// painn_fused.cu -- the whole per-atom ("node") part of a PaiNN layer as ONE persistent wgmma kernel per direction.
//
// Replaces, per layer, the five nn.Linear GEMMs and the elementwise glue of
//   PaiNNUpdate.forward            nablaDFT/painn_pyg/painn.py:535-548   (schnetpack PaiNNMixing)
//   the message MLP x_proj         nablaDFT/painn_pyg/painn.py:459-464   (schnetpack interatomic_context_net)
//   the readout's first Linear     nablaDFT/painn_pyg/painn.py:79-83     (schnetpack Atomwise.outnet[0])
// and their autograd backward (painn.py:135-146), which would otherwise be 12 separate 3xTF32 GEMM launches + 6 elementwise launches per
// layer and direction, each re-staging and re-splitting its activation slab.
//
// Design (the pipeline itself is tc_pipe.cuh):
//   * CTA = 64 atoms.  Every GEMM of the chain is computed TRANSPOSED: D[feature, atom] = W[feature, k] . X[atom, k]^T, i.e. the weight
//     tile is the MMA's A operand (M = 128 output features, two warpgroups of 64) and the activations are the B operand (N = 64 atoms).
//     The staged result has features on rows and atoms on columns: an epilogue thread owns one feature and 32 atoms, so every global
//     store / load of an [atom][feature] array is a 128-byte coalesced warp access, the bias is a per-thread scalar, and writing the next
//     activation operand into shared memory ([atoms] x K, K-major) is a conflict-free 4-byte store pattern.
//   * weights are split into TF32 hi / lo ONCE per call by k_prep_painn into ready-made shared-memory images (one 128 x 128 tile =
//     4 stages x [hi | lo] x 16 KB, canonical no-swizzle K-major), streamed with one cp.async.bulk per stage through a 3-stage mbarrier ring.
//   * the activation operand X [64 atoms x 128 k] (hi + lo) is written by the 8 worker warps: either by a LOADER functor (coalesced global
//     loads, elementwise math fused in: sqrt-norm, the combine backward, silu' ...) or directly from the previous GEMM's epilogue registers
//     (silu(h) -> next operand) -- chained activations never go through global memory to be re-read as operands.
//   * 3xTF32: lo.hi + hi.lo into a correction accumulator, hi.hi alternating over two main accumulators so that no accumulator chain is
//     longer than 8 per 128 k (the tensor core truncates on accumulate, see gemm_tc.cu); the MMA warpgroups sum them into a shared-memory
//     staging tile, which the epilogues walk in 16-atom chunks inside ROLLED loops (compact code).  K > 128 (backward) accumulates over
//     several X operands in place.
//   * roles meet only through mbarriers: W ring full/empty, X ready/free, staging full / free.
// Forward  kernel = update(l) [+ message MLP(l+1) | readout Linear]
// Backward kernel = [message-MLP backward(l+1) | readout backward] + update backward(l)
#include "painn_node.cuh"

#include "tc_pipe.cuh"

namespace {

constexpr int TILES_PER_LAYER = 22;

// weight tiles of a layer (index into the prepared buffer, see k_prep_painn)
enum { T_UV = 0, T_UW, T_B1A, T_B1B, T_B2_0, T_B2_1, T_B2_2, T_A1, T_A2_0, T_A2_1, T_A2_2,
       T_B2T_0, T_B2T_1, T_B2T_2, T_B1AT, T_B1BT, T_UT_0, T_UT_1, T_A2T_0, T_A2T_1, T_A2T_2, T_A1T };

// ------------------------------------------------------------------------------------------------------------------
// Weight preparation: every 128 x 128 block a fused kernel uses, as TF32 hi / lo shared-memory images.
// tile t of layer l lives at (l * 22 + t) * WTILE_BYTES; the two readout tiles follow the last layer.
// element (row r, k) of a tile: stage k / KSTAGE, hi first then lo (KSTAGE / 4 chunks of 2 KB each), chunk (k % KSTAGE) / 4, then r * 16 + (k % 4) * 4 bytes.
struct TileSrc { const float* p; int ld, row0, k0, trans, rows, kvalid; };

__device__ __forceinline__ TileSrc tile_src(const nb200_painn_weights& w, int idx) {
    const int L = w.n_layers;
    TileSrc s{nullptr, F, 0, 0, 0, 128, 128};
    if (idx >= L * TILES_PER_LAYER) {  // readout Linear R1 [F/2][F]: forward tile (rows = outputs, 64 valid) and transposed tile (k = outputs)
        s.p = w.R1; s.ld = F;
        if (idx - L * TILES_PER_LAYER == 0) { s.rows = F / 2; } else { s.trans = 1; s.kvalid = F / 2; }
        return s;
    }
    const int l = idx / TILES_PER_LAYER, t = idx % TILES_PER_LAYER;
    const float* A1 = w.A1 + (size_t)l * F * F;
    const float* A2 = w.A2 + (size_t)l * 3 * F * F;
    const float* U = w.U + (size_t)l * 2 * F * F;
    const float* B1 = w.B1 + (size_t)l * F * 2 * F;
    const float* B2 = w.B2 + (size_t)l * 3 * F * F;
    switch (t) {
        case T_UV: s.p = U; break;
        case T_UW: s.p = U; s.row0 = F; break;
        case T_B1A: s.p = B1; s.ld = 2 * F; break;
        case T_B1B: s.p = B1; s.ld = 2 * F; s.k0 = F; break;
        case T_B2_0: case T_B2_1: case T_B2_2: s.p = B2; s.row0 = (t - T_B2_0) * F; break;
        case T_A1: s.p = A1; break;
        case T_A2_0: case T_A2_1: case T_A2_2: s.p = A2; s.row0 = (t - T_A2_0) * F; break;
        // transposed tiles (Linear backward w.r.t. the input): element (r = input feature, k = output feature) = W[k0 + k][row0 + r]
        case T_B2T_0: case T_B2T_1: case T_B2T_2: s.p = B2; s.trans = 1; s.k0 = (t - T_B2T_0) * F; break;
        case T_B1AT: s.p = B1; s.ld = 2 * F; s.trans = 1; break;
        case T_B1BT: s.p = B1; s.ld = 2 * F; s.trans = 1; s.row0 = F; break;
        case T_UT_0: case T_UT_1: s.p = U; s.trans = 1; s.k0 = (t - T_UT_0) * F; break;
        case T_A2T_0: case T_A2T_1: case T_A2T_2: s.p = A2; s.trans = 1; s.k0 = (t - T_A2T_0) * F; break;
        default: s.p = A1; s.trans = 1; break;  // T_A1T
    }
    return s;
}

__global__ void __launch_bounds__(256) k_prep_painn(nb200_painn_weights w, unsigned char* __restrict__ dst) {
    const int idx = blockIdx.x >> 2, st = blockIdx.x & 3;
    const TileSrc s = tile_src(w, idx);
    unsigned char* tile = dst + (size_t)idx * WTILE_BYTES;  // this block: k in [32 st, 32 st + 32)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int item = threadIdx.x + 256 * i;  // 1024 (chunk, row) pairs of the stage
        int kc, r;
        if (!s.trans) { kc = item & 7; r = item >> 3; } else { r = item & 127; kc = item >> 7; }  // coalesced along the source's contiguous axis
        const int k = st * 32 + kc * 4;
        float e[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool ok = r < s.rows && k + j < s.kvalid;
            e[j] = !ok ? 0.f : !s.trans ? __ldg(s.p + (size_t)(s.row0 + r) * s.ld + s.k0 + k + j) : __ldg(s.p + (size_t)(s.k0 + k + j) * s.ld + s.row0 + r);
        }
        float4 hi, lo;
        split4(make_float4(e[0], e[1], e[2], e[3]), hi, lo);
        const int kk = 32 * st + 4 * kc;  // first k of this chunk
        float* out_hi = reinterpret_cast<float*>(tile + (size_t)(kk / KSTAGE) * WST_BYTES + (size_t)((kk % KSTAGE) / 4) * WLBO) + r * 4;
        st4(out_hi, hi);
        st4(out_hi + (KSTAGE / 4) * WLBO / 4, lo);
    }
}

// ================================================================================================== forward
struct FwdParams {
    int xsplit;  // tc_pipe.cuh: activation operands handed over in two K halves
    int n_atoms, do_upd, do_mlp, do_ro;
    const unsigned char* wt;  // prepared weight tiles
    int tile_upd, tile_mlp, tile_ro;  // first tile of the layer updated / of the layer whose message MLP runs / readout forward tile
    // update (layer l): inputs after the message kernel, saved activations, outputs
    const float *q_mid, *mu_mid, *d1, *d2;
    float *VW, *nrm, *dot, *g1pre, *y, *q_next, *mu_next;  // dot = <V, Wv> per (atom, channel): saved for the backward
    float eps;
    // message MLP (layer l + 1; layer 0 when !do_upd): input when it is not produced in-kernel, saved pre-activation, output
    const float *q_mlp_in, *c1;
    float *h1pre, *xh;
    float* ro_pre;  // readout: [N, F/2] WITHOUT the bias e1 (k_readout adds it)
};

__global__ void __launch_bounds__(NTHREADS, CTAS_PER_SM) k_node_fwd(const FwdParams P) {
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ Prog prog;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        prog.n = 0;
        if (P.do_upd) {
            for (int x = 0; x < 3; ++x) {
                prog_add(prog, P.tile_upd + T_UV, U_NEWX | U_FIRST | U_LAST);
                prog_add(prog, P.tile_upd + T_UW, U_FIRST | U_LAST | U_XLAST);
            }
            prog_add(prog, P.tile_upd + T_B1A, U_NEWX | U_FIRST | U_LAST | U_XLAST);
            prog_add(prog, P.tile_upd + T_B1B, U_NEWX | U_FIRST | U_LAST | U_XLAST);
            prog_add(prog, P.tile_upd + T_B2_1, U_NEWX | U_FIRST | U_LAST);
            prog_add(prog, P.tile_upd + T_B2_0, U_FIRST | U_LAST);
            prog_add(prog, P.tile_upd + T_B2_2, U_FIRST | U_LAST | U_XLAST);
        }
        if (P.do_mlp) {
            prog_add(prog, P.tile_mlp + T_A1, U_NEWX | U_FIRST | U_LAST | U_XLAST);
            prog_add(prog, P.tile_mlp + T_A2_0, U_NEWX | U_FIRST | U_LAST);
            prog_add(prog, P.tile_mlp + T_A2_1, U_FIRST | U_LAST);
            prog_add(prog, P.tile_mlp + T_A2_2, U_FIRST | U_LAST | U_XLAST);
        }
        if (P.do_ro) prog_add(prog, P.tile_ro, U_NEWX | U_FIRST | U_LAST | U_XLAST);
    }
    Ctx c = setup(smem, tid, P.xsplit);
    NF_PROF_DO(const long long tk0_ = clock64(); c.t_last = tk0_;)
#define NF_BASE 0

    if (warp >= WARP_ISSUE) {
        run_issuer(c, prog, P.wt);
        NF_PROF_DO(if (warp == WARP_ISSUE && lane == 0) { atomicAdd(&g_nf_prof[0], (unsigned long long)(clock64() - tk0_)); atomicAdd(&g_nf_prof[1], (unsigned long long)c.w_x);
                   atomicAdd(&g_nf_prof[2], (unsigned long long)c.w_buf); atomicAdd(&g_nf_prof[3], (unsigned long long)c.w_full); })
    } else {
        const int N = P.n_atoms, A0 = blockIdx.x * NT;
        const int fl = 32 * (warp & 3) + lane;   // my feature inside a 128-row weight tile
        const int n0 = CPT * (warp >> 2);        // my first atom column
        const bool isE = role_epi(warp), isL = role_load(warp);  // both true for every worker warp in single-group builds
        const int ltid = load_tid(tid);
#define NF_LOAD(...) do { if (isL) load_x(c, ltid, __VA_ARGS__); else ++c.xg; } while (0)
        if (P.do_upd) {
            // ---- VW[(atom, x)] = mu_mid[(atom, x)] . U^T : V half, W half per cartesian component
#pragma unroll 1
            for (int x = 0; x < 3; ++x) {
                NF_LOAD([&](int r, int kc) { return A0 + r < N ? ldg4(P.mu_mid + (size_t)(A0 + r) * (3 * F) + x * F + 4 * kc) : f4(0.f); });
                NF_MARK(0);
#pragma unroll 1
                for (int half = 0; half < 2 && isE; ++half) {
                    drain(c, warp);
                    NF_MARK(1);
                    epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                        float* dst = P.VW + (size_t)(A0 + n0 + 16 * cb) * (6 * F) + x * 2 * F + half * F + fl;
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (A0 + n0 + 16 * cb + j < N) dst[(size_t)j * (6 * F)] = v[j];
                    });
                    NF_MARK(21);
                }
            }
            NF_MARK(2);
            if (isE) dep_signal(c, 0);  // VW of this tile is visible to the loader-mapped threads below
            // ---- g1pre = [q_mid | nrm] . B1^T + d1 as two K = 128 halves summed in the staging columns
            NF_LOAD([&](int r, int kc) { return A0 + r < N ? ldg4(P.q_mid + (size_t)(A0 + r) * F + 4 * kc) : f4(0.f); });
            NF_MARK(3);
            if (isL) {   // while the tensor core works on q_mid: nrm = sqrt(sum_x V_x^2 + eps) and dot = sum_x V_x Wv_x, 2 atoms per round
                // (|V|^2 and <V,Wv> are not kept in registers across the U tiles: 64 persistent registers would spill, and with ~195 KB of
                //  shared memory per CTA little L1 is left for local memory)
                dep_wait(c, 0);
                const int kc = ltid & 31, w = ltid >> 5;
#pragma unroll 1
                for (int it0 = 0; it0 < RPT; it0 += 2) {
                    float4 V[2][3], Wv[2][3];
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const int a = A0 + w + NLOAD * (it0 + b);
                        const float* vv = P.VW + (size_t)min(a, N - 1) * (6 * F) + 4 * kc;
#pragma unroll
                        for (int x = 0; x < 3; ++x) { V[b][x] = ld4(vv + x * 2 * F); Wv[b][x] = ld4(vv + x * 2 * F + F); }
                    }
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const int a = A0 + w + NLOAD * (it0 + b);
                        if (a < N) {
                            float4 sq = V[b][0] * V[b][0]; fma4(sq, V[b][1], V[b][1]); fma4(sq, V[b][2], V[b][2]);
                            float4 dt = f4(0.f); fma4(dt, V[b][0], Wv[b][0]); fma4(dt, V[b][1], Wv[b][1]); fma4(dt, V[b][2], Wv[b][2]);
                            st4(P.nrm + (size_t)a * F + 4 * kc, make_float4(sqrtf(sq.x + P.eps), sqrtf(sq.y + P.eps), sqrtf(sq.z + P.eps), sqrtf(sq.w + P.eps)));
                            st4(P.dot + (size_t)a * F + 4 * kc, dt);
                        }
                    }
                }
            }
            NF_MARK(4);
            if (isL) dep_signal(c, 1);  // nrm (read back by the same threads) and dot (read by the y2 epilogue threads) are visible
            NF_LOAD([&](int r, int kc) { return A0 + r < N ? ld4(P.nrm + (size_t)(A0 + r) * F + 4 * kc) : f4(0.f); });
            NF_MARK(5);
            if (isE) drain(c, warp);      // q_mid half: stays in the staging columns
            NF_MARK(6);
            NF_MARK(7);
            if (!isE) ++c.xg;             // the activation operand written by the epilogue group below
            else {
                drain(c, warp, 1);   // + nrm half
                NF_MARK(8);
                const float b = __ldg(P.d1 + fl);
                const XPut xp(c, fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {   // operand first: the tensor core restarts before anything is stored
#pragma unroll
                    for (int j = 0; j < 16; ++j) xp.put(n0 + 16 * cb + j, A0 + n0 + 16 * cb + j < N ? siluf_(v[j] + b) : 0.f);
                });
                xp.done(c);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float* g = P.g1pre + (size_t)(A0 + n0 + 16 * cb) * F + fl;
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) g[(size_t)j * F] = v[j] + b;
                });
            }
            NF_MARK(9);
            // ---- y = silu(g1pre) . B2^T + d2, tiles in the order (gate y1, scalar y0, dot-scale y2)
            if (isE) {   // y1: mu_next = mu_mid + y1 * Wv   (runs while the tensor core works on the y0 / y2 tiles)
                drain(c, warp);
                NF_MARK(10);
                const float b = __ldg(P.d2 + F + fl);
#pragma unroll 1
                for (int cb = 0; cb < CPT / 8; ++cb) {  // 8 atoms per round: 48 loads in flight per thread
                    float v16[16];
                    stage_ld16(c, warp, cb >> 1, v16);
                    float tw[8][3], tm[8][3];
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int a = min(A0 + n0 + 8 * cb + jj, N - 1);
                        const float* vw = P.VW + (size_t)a * (6 * F) + F + fl;
                        const float* mm = P.mu_mid + (size_t)a * (3 * F) + fl;
#pragma unroll
                        for (int x = 0; x < 3; ++x) { tw[jj][x] = vw[x * 2 * F]; tm[jj][x] = __ldg(mm + x * F); }
                    }
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int a = A0 + n0 + 8 * cb + jj;
                        if (a < N) {
                            const float y1 = ((cb & 1) ? v16[8 + jj] : v16[jj]) + b;
                            P.y[(size_t)a * (3 * F) + F + fl] = y1;
                            float* mo = P.mu_next + (size_t)a * (3 * F) + fl;
#pragma unroll
                            for (int x = 0; x < 3; ++x) mo[x * F] = fmaf(y1, tw[jj][x], tm[jj][x]);
                        }
                    }
                }
            }
            NF_MARK(11);
            if (isE) {   // y0: stored, and q_next <- q_mid + y0 (completed by the y2 tile)
                drain(c, warp);
                NF_MARK(12);
                const float b = __ldg(P.d2 + fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = __ldg(P.q_mid + (size_t)min(A0 + n0 + 16 * cb + j, N - 1) * F + fl);
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int a = A0 + n0 + 16 * cb + j;
                        if (a < N) {
                            const float y0 = v[j] + b;
                            P.y[(size_t)a * (3 * F) + fl] = y0;
                            P.q_next[(size_t)a * F + fl] = t[j] + y0;
                        }
                    }
                });
            }
            NF_MARK(13);
            if (!isE) ++c.xg;
            else {   // y2: q_next = (q_mid + y0) + y2 * <V, Wv>; it is the next operand (message MLP of the next layer / readout)
                dep_wait(c, 1);
                drain(c, warp);
                NF_MARK(14);
                const float b = __ldg(P.d2 + 2 * F + fl);
                const XPut xp(c, fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float tq[16], td[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const size_t a = (size_t)min(A0 + n0 + 16 * cb + j, N - 1);
                        tq[j] = P.q_next[a * F + fl];
                        td[j] = P.dot[a * F + fl];
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int a = A0 + n0 + 16 * cb + j;
                        float qn = 0.f;
                        if (a < N) {
                            qn = fmaf(v[j] + b, td[j], tq[j]);
                            P.q_next[(size_t)a * F + fl] = qn;
                        }
                        xp.put(n0 + 16 * cb + j, qn);
                    }
                });
                xp.done(c);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) P.y[(size_t)(A0 + n0 + 16 * cb + j) * (3 * F) + 2 * F + fl] = v[j] + b;
                });
            }
        } else {
            NF_LOAD([&](int r, int kc) { return A0 + r < N ? ldg4(P.q_mlp_in + (size_t)(A0 + r) * F + 4 * kc) : f4(0.f); });
        }
        NF_MARK(15);
        if (P.do_mlp && !isE) ++c.xg;
        if (P.do_mlp && isE) {
            {   // h1pre = q . A1^T + c1 ; silu -> operand (first), then the saved pre-activation
                drain(c, warp);
                NF_MARK(16);
                const float b = __ldg(P.c1 + fl);
                const XPut xp(c, fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) xp.put(n0 + 16 * cb + j, siluf_(v[j] + b));
                });
                xp.done(c);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) P.h1pre[(size_t)(A0 + n0 + 16 * cb + j) * F + fl] = v[j] + b;
                });
            }
            NF_MARK(17);
#pragma unroll 1
            for (int ct = 0; ct < 3; ++ct) {  // xh = act . A2^T  (bias c2 is added inside the message kernel)
                drain(c, warp);
                NF_MARK(18);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float* dst = P.xh + (size_t)(A0 + n0 + 16 * cb) * (3 * F) + ct * F + fl;
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) dst[(size_t)j * (3 * F)] = v[j];
                });
            }
        }
        NF_MARK(19);
        if (P.do_ro && isE) {
            drain(c, warp);
            epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                if (fl < F / 2) {
                    float* dst = P.ro_pre + (size_t)(A0 + n0 + 16 * cb) * (F / 2) + fl;
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) dst[(size_t)j * (F / 2)] = v[j];
                }
            });
        }
#undef NF_LOAD
    }
    NF_MARK(20);
#undef NF_BASE
    NF_PROF_DO(if (tid == 0) { atomicAdd(&g_nf_prof[4], (unsigned long long)(clock64() - tk0_)); atomicAdd(&g_nf_prof[5], (unsigned long long)c.w_acc);
                            atomicAdd(&g_nf_prof[6], (unsigned long long)c.w_xfree); atomicAdd(&g_nf_prof[7], 1ull); })
}

// ================================================================================================== backward
struct BwdParams {
    int xsplit;
    int n_atoms, do_mlp, do_ro, do_upd;
    const unsigned char* wt;
    int tile_mlp, tile_ro, tile_upd;  // layer whose message MLP is differentiated / readout transposed tile / layer whose update is differentiated
    // gradients: gq_a = dE/dq in (from the previous backward step) and out (dE/dq_mid of the updated layer); gq_b = scratch (dE/dq_in of
    // the layer above); cur = dE/dmu, in / out; g_xh = dE/dxh written by the message backward of the layer above
    float *gq_a, *gq_b, *cur, *gn, *gdot;  // gn holds s = gn / nrm, gdot = gq_b * y2 (scratch of this kernel)
    const float *g_xh, *h1pre, *dot;
    const float *ro_pre, *R2;      // readout backward: g_ro = R2 * silu'(ro_pre)   (ro_pre holds the biased pre-activation)
    const float *y, *VW, *nrm, *g1pre;
};

__global__ void __launch_bounds__(NTHREADS, CTAS_PER_SM) k_node_bwd(const BwdParams P) {
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ Prog prog;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        prog.n = 0;
        if (P.do_mlp) {
            prog_add(prog, P.tile_mlp + T_A2T_0, U_NEWX | U_FIRST | U_XLAST);
            prog_add(prog, P.tile_mlp + T_A2T_1, U_NEWX | U_XLAST);
            prog_add(prog, P.tile_mlp + T_A2T_2, U_NEWX | U_XLAST | U_LAST);
            prog_add(prog, P.tile_mlp + T_A1T, U_NEWX | U_FIRST | U_LAST | U_XLAST);
        } else if (P.do_ro) {
            prog_add(prog, P.tile_ro, U_NEWX | U_FIRST | U_LAST | U_XLAST);
        }
        if (P.do_upd) {
            prog_add(prog, P.tile_upd + T_B2T_0, U_NEWX | U_FIRST | U_XLAST);
            prog_add(prog, P.tile_upd + T_B2T_1, U_NEWX | U_XLAST);
            prog_add(prog, P.tile_upd + T_B2T_2, U_NEWX | U_XLAST | U_LAST);
            prog_add(prog, P.tile_upd + T_B1AT, U_NEWX | U_FIRST | U_LAST);
            prog_add(prog, P.tile_upd + T_B1BT, U_FIRST | U_LAST | U_XLAST);
            for (int x = 0; x < 3; ++x) {
                prog_add(prog, P.tile_upd + T_UT_0, U_NEWX | U_FIRST | U_XLAST);
                prog_add(prog, P.tile_upd + T_UT_1, U_NEWX | U_XLAST | U_LAST);
            }
        }
    }
    Ctx c = setup(smem, tid, P.xsplit);
    NF_PROF_DO(const long long tk0_ = clock64();)

    if (warp >= WARP_ISSUE) {
        run_issuer(c, prog, P.wt);
        NF_PROF_DO(if (warp == WARP_ISSUE && lane == 0) { atomicAdd(&g_nf_prof[8], (unsigned long long)(clock64() - tk0_)); atomicAdd(&g_nf_prof[9], (unsigned long long)c.w_x);
                   atomicAdd(&g_nf_prof[10], (unsigned long long)c.w_buf); atomicAdd(&g_nf_prof[11], (unsigned long long)c.w_full); })
    } else {
        const int N = P.n_atoms, A0 = blockIdx.x * NT;
        const int fl = 32 * (warp & 3) + lane;
        const int n0 = CPT * (warp >> 2);
        const bool isE = role_epi(warp), isL = role_load(warp);
        const int ltid = load_tid(tid);
#define NF_LOAD(...) do { if (isL) load_x(c, ltid, __VA_ARGS__); else ++c.xg; } while (0)
        if (P.do_mlp) {
            // ---- gt = g_xh . A2 (K = 384) ; gt *= silu'(h1pre) ; gq_b = gq_a + gt . A1
#pragma unroll 1
            for (int ck = 0; ck < 3; ++ck)
                NF_LOAD([&](int r, int kc) { return A0 + r < N ? ldg4(P.g_xh + (size_t)(A0 + r) * (3 * F) + ck * F + 4 * kc) : f4(0.f); });
            if (!isE) ++c.xg;
            else {
                drain(c, warp);
                const XPut xp(c, fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = __ldg(P.h1pre + (size_t)min(A0 + n0 + 16 * cb + j, N - 1) * F + fl);
#pragma unroll
                    for (int j = 0; j < 16; ++j) xp.put(n0 + 16 * cb + j, A0 + n0 + 16 * cb + j < N ? v[j] * dsiluf_(t[j]) : 0.f);
                });
                xp.done(c);
            }
        } else if (P.do_ro) {
            // ---- gq_b = g_ro . R1 with g_ro[k] = R2[k] silu'(ro_pre[k]), k < F/2 (zero-padded to K = 128)
            NF_LOAD([&](int r, int kc) {
                if (A0 + r >= N || kc >= F / 8) return f4(0.f);
                const float4 p = ldg4(P.ro_pre + (size_t)(A0 + r) * (F / 2) + 4 * kc), w2 = ldg4(P.R2 + 4 * kc);
                return make_float4(w2.x * dsiluf_(p.x), w2.y * dsiluf_(p.y), w2.z * dsiluf_(p.z), w2.w * dsiluf_(p.w));
            });
        }
        if ((P.do_mlp || P.do_ro) && isE) {  // gq_b = dE/dq_in of the layer above; gdot = gq_b * y2 is what the combine backward needs three times
            drain(c, warp);
            epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                float t[16], ty[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const size_t a = (size_t)min(A0 + n0 + 16 * cb + j, N - 1);
                    t[j] = P.do_mlp ? P.gq_a[a * F + fl] : 0.f;
                    ty[j] = P.do_upd ? __ldg(P.y + a * (3 * F) + 2 * F + fl) : 0.f;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int a = A0 + n0 + 16 * cb + j;
                    if (a < N) {
                        const float g = t[j] + v[j];
                        P.gq_b[(size_t)a * F + fl] = g;
                        if (P.do_upd) P.gdot[(size_t)a * F + fl] = g * ty[j];
                    }
                }
            });
        }
        if (P.do_upd) {
            if (isE) dep_signal(c, 0);  // gq_b, gdot visible to the loader-mapped threads
            if (isL) dep_wait(c, 0);
            // ---- gt = gy . B2 (K = 384) with gy = (gq, sum_x cur_x Wv_x, gq <V, Wv>) formed on the fly (combine backward)
            NF_LOAD([&](int r, int kc) { return A0 + r < N ? ld4(P.gq_b + (size_t)(A0 + r) * F + 4 * kc) : f4(0.f); });
            NF_LOAD([&](int r, int kc) {
                if (A0 + r >= N) return f4(0.f);
                const float* vw = P.VW + (size_t)(A0 + r) * (6 * F) + F + 4 * kc;
                const float* gm = P.cur + (size_t)(A0 + r) * (3 * F) + 4 * kc;
                float4 sacc = f4(0.f);
#pragma unroll
                for (int x = 0; x < 3; ++x) fma4(sacc, ld4(gm + x * F), ldg4(vw + x * 2 * F));
                return sacc;
            });
            NF_LOAD([&](int r, int kc) {
                return A0 + r < N ? ld4(P.gq_b + (size_t)(A0 + r) * F + 4 * kc) * ldg4(P.dot + (size_t)(A0 + r) * F + 4 * kc) : f4(0.f);
            });
            if (!isE) ++c.xg;
            else {
                drain(c, warp);
                const XPut xp(c, fl);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = __ldg(P.g1pre + (size_t)min(A0 + n0 + 16 * cb + j, N - 1) * F + fl);
#pragma unroll
                    for (int j = 0; j < 16; ++j) xp.put(n0 + 16 * cb + j, A0 + n0 + 16 * cb + j < N ? v[j] * dsiluf_(t[j]) : 0.f);
                });
                xp.done(c);
            }
            if (isE) {   // gq_a = gq_b + gt . B1[:, :F]   (dE/dq_mid of this layer: what the message backward reads)
                drain(c, warp);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = P.gq_b[(size_t)min(A0 + n0 + 16 * cb + j, N - 1) * F + fl];
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) P.gq_a[(size_t)(A0 + n0 + 16 * cb + j) * F + fl] = t[j] + v[j];
                });
            }
            if (isE) {   // gn = gt . B1[:, F:], stored as s = gn / nrm (norm backward: gV_x += s V_x)
                drain(c, warp);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = __ldg(P.nrm + (size_t)min(A0 + n0 + 16 * cb + j, N - 1) * F + fl);
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) P.gn[(size_t)(A0 + n0 + 16 * cb + j) * F + fl] = v[j] / t[j];
                });
            }
            if (isE) dep_signal(c, 1);  // s visible
            if (isL) dep_wait(c, 1);
            // ---- cur_x += gVW_x . U (K = 256: V chunk then Wv chunk), gVW formed on the fly (combine + norm backward)
#pragma unroll 1
            for (int x = 0; x < 3; ++x) {
                NF_LOAD([&](int r, int kc) {  // gV = gdot * Wv + s * V
                    if (A0 + r >= N) return f4(0.f);
                    const size_t a = (size_t)(A0 + r);
                    float4 o = ld4(P.gdot + a * F + 4 * kc) * ldg4(P.VW + a * (6 * F) + x * 2 * F + F + 4 * kc);
                    fma4(o, ld4(P.gn + a * F + 4 * kc), ldg4(P.VW + a * (6 * F) + x * 2 * F + 4 * kc));
                    return o;
                });
                NF_LOAD([&](int r, int kc) {  // gWv = cur_x * y1 + gdot * V
                    if (A0 + r >= N) return f4(0.f);
                    const size_t a = (size_t)(A0 + r);
                    float4 o = ld4(P.cur + a * (3 * F) + x * F + 4 * kc) * ldg4(P.y + a * (3 * F) + F + 4 * kc);
                    fma4(o, ld4(P.gdot + a * F + 4 * kc), ldg4(P.VW + a * (6 * F) + x * 2 * F + 4 * kc));
                    return o;
                });
                if (isE) {
                drain(c, warp);
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float t[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) t[j] = P.cur[(size_t)min(A0 + n0 + 16 * cb + j, N - 1) * (3 * F) + x * F + fl];
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (A0 + n0 + 16 * cb + j < N) P.cur[(size_t)(A0 + n0 + 16 * cb + j) * (3 * F) + x * F + fl] = t[j] + v[j];
                });
                }
            }
        }
#undef NF_LOAD
    }
    NF_PROF_DO(if (tid == 0) { atomicAdd(&g_nf_prof[12], (unsigned long long)(clock64() - tk0_)); atomicAdd(&g_nf_prof[13], (unsigned long long)c.w_acc);
                            atomicAdd(&g_nf_prof[14], (unsigned long long)c.w_xfree); atomicAdd(&g_nf_prof[15], 1ull); })
}

template <class K>
int set_smem(K kernel) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL) == cudaSuccess ? NB200_OK : nb_check_launch();
}

}  // namespace

#ifdef NF_PROF
extern "C" int nb200_debug_nf_prof(unsigned long long* out16, int reset) {
    if (cudaMemcpyFromSymbol(out16, g_nf_prof, sizeof(unsigned long long) * 16) != cudaSuccess) return -1;
    if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_nf_prof, z, sizeof(z)); }
    return 0;
}
extern "C" int nb200_debug_nf_phase(unsigned long long* out64, int reset) {
    if (cudaMemcpyFromSymbol(out64, g_nf_phase, sizeof(unsigned long long) * 64) != cudaSuccess) return -1;
    if (reset) { unsigned long long z[64] = {0}; cudaMemcpyToSymbol(g_nf_phase, z, sizeof(z)); }
    return 0;
}
#endif

int64_t nb_fused_wtile_bytes(int n_layers) { return (int64_t)(n_layers * TILES_PER_LAYER + 2) * WTILE_BYTES; }

int nb_fused_prep(const nb200_painn_weights* w, void* wtiles, cudaStream_t s) {
    const int n_tiles = w->n_layers * TILES_PER_LAYER + 2;
    k_prep_painn<<<n_tiles * 4, 256, 0, s>>>(*w, static_cast<unsigned char*>(wtiles));
    return nb_check_launch();
}

// NB200_NF_XSPLIT=1: hand the activation operands over in two K halves (tc_pipe.cuh).  Measured neutral for these kernels (122.4 k vs 122.8 k
// molecules/s, A/B run: most of their operands are written by the previous GEMM's epilogue, which the hand-over cannot
// start earlier), so the whole-operand protocol stays the default here; the pre-split-weight GEMM uses it for K > 128.
static int nf_xsplit() {
    static const int on = [] { const char* e = getenv("NB200_NF_XSPLIT"); return (e && e[0] == '1') ? 1 : 0; }();
    return on;
}

int nb_fused_node_fwd(const NbFusedFwd& a, cudaStream_t s) {
    static bool attr = false;
    if (!attr) { if (set_smem(k_node_fwd) != NB200_OK) return NB200_ECUDA; attr = true; }
    FwdParams P{};
    P.xsplit = nf_xsplit();
    P.n_atoms = a.n_atoms; P.do_upd = a.layer_upd >= 0; P.do_mlp = a.layer_mlp >= 0; P.do_ro = a.readout;
    P.wt = static_cast<const unsigned char*>(a.wtiles);
    P.tile_upd = a.layer_upd * TILES_PER_LAYER; P.tile_mlp = a.layer_mlp * TILES_PER_LAYER; P.tile_ro = a.n_layers * TILES_PER_LAYER;
    P.q_mid = a.q_mid; P.mu_mid = a.mu_mid; P.d1 = a.d1; P.d2 = a.d2; P.VW = a.VW; P.nrm = a.nrm; P.dot = a.dot; P.g1pre = a.g1pre; P.y = a.y;
    P.q_next = a.q_next; P.mu_next = a.mu_next; P.eps = a.eps; P.q_mlp_in = a.q_mlp_in; P.c1 = a.c1; P.h1pre = a.h1pre; P.xh = a.xh;
    P.ro_pre = a.ro_pre;
    if (a.n_atoms <= 0) return NB200_OK;
    k_node_fwd<<<(a.n_atoms + NT - 1) / NT, NTHREADS, SMEM_TOTAL, s>>>(P);
    return nb_check_launch();
}

int nb_fused_node_bwd(const NbFusedBwd& a, cudaStream_t s) {
    static bool attr = false;
    if (!attr) { if (set_smem(k_node_bwd) != NB200_OK) return NB200_ECUDA; attr = true; }
    BwdParams P{};
    P.xsplit = nf_xsplit();
    P.n_atoms = a.n_atoms; P.do_mlp = a.layer_mlp >= 0; P.do_ro = a.readout; P.do_upd = a.layer_upd >= 0;
    P.wt = static_cast<const unsigned char*>(a.wtiles);
    P.tile_mlp = a.layer_mlp * TILES_PER_LAYER; P.tile_ro = a.n_layers * TILES_PER_LAYER + 1; P.tile_upd = a.layer_upd * TILES_PER_LAYER;
    P.gq_a = a.gq_a; P.gq_b = a.gq_b; P.cur = a.cur; P.gn = a.gn; P.gdot = a.gdot; P.dot = a.dot; P.g_xh = a.g_xh; P.h1pre = a.h1pre; P.ro_pre = a.ro_pre; P.R2 = a.R2;
    P.y = a.y; P.VW = a.VW; P.nrm = a.nrm; P.g1pre = a.g1pre;
    if (a.n_atoms <= 0) return NB200_OK;
    k_node_bwd<<<(a.n_atoms + NT - 1) / NT, NTHREADS, SMEM_TOTAL, s>>>(P);
    return nb_check_launch();
}
