// wgrad_tc.cu -- weight gradients of the training step on the tensor cores (wgmma, sm_90a):
//
//     dW[o, i]  += alpha      * sum_t sum_a  G_t[a, o] * X_t[a, i]          (t = 1 or 2 terms: the tangent pass has tg^T x + g^T tx)
//     dbias[o]  += bias_alpha *       sum_a  G_b[a, o]                      (optional; b = the term that carries the bias gradient)
//
// i.e. what the reference gets from autograd for every nn.Linear of the model (torch: grad_weight = grad_out^T @ input,
// grad_bias = grad_out.sum(0)) -- instead of one cuBLAS SGEMM + splitKreduce + a column-sum kernel per Linear.  The contraction runs over ATOMS (K = 10^4), the output is at most 384 x 128: a split-K problem.
//
// One CTA per SM = 128 outputs x a strided set of (term, 128-atom chunk) sub-units, their products summed in the wgmma register accumulators
// and flushed with ONE set of vector atomics per CTA.  Both operands are read ONCE from global memory in their natural row-major layout
// ([atom, feature], 16-byte loads), split into TF32 hi / lo in registers and TRANSPOSED on the way into shared memory: K-major operands
// (K = atoms) written with 4-byte stores whose strides (160 B between 8-feature groups, = 16 B mod 128 between 4-atom chunks) make the
// 32 lanes of a store hit 32 banks (wgmma TF32 reads K-major operands only).  3xTF32 as in gemm_tc.cu: lo.hi + hi.lo into a correction
// accumulator, hi.hi into a main one; both are reset per (term, 128-atom) sub-unit and folded into fp32 register sums at its end (the
// tensor core truncates when it accumulates: chains of 16 main products, whatever M and the number of CTAs).  The bias gradient rides
// along as 16 extra B columns holding the constant 1 in the stages of the
// terms that carry it (column `in` of D = column sums of G).  Four warpgroups: outputs [64 (g & 1), +64) x B columns [72 (g >> 1), +72).
// Epilogue: registers -> shared-memory staging -> row-contiguous red.global.add.v4.f32 into the gradient bucket.  The sum over atom chunks
// is therefore atomic (fp32 addition order varies from run to run at the 1e-7 relative level; cuBLAS split-K was deterministic).
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int WG_THREADS = 512;
constexpr int WG_KS = 32;                       // atoms per stage (4 MMA k-steps of 8)
constexpr int WG_NB = 144;                      // B columns: 128 inputs + 16 (ones column for the bias gradient + padding to N % 16 == 0)
constexpr int WG_SBO = 160;                     // bytes between 8-row (feature) groups: a 128-byte core matrix + 32 (bank spread of the transposing stores)
constexpr int WG_A_LBO = 16 * WG_SBO + 16;      // bytes between 4-atom k-chunks of A (128 rows), = 16 mod 128
constexpr int WG_B_LBO = 23 * 128 + 16;         // same for B (144 rows = 18 groups = 2880 B, rounded up to 16 mod 128)
constexpr int WG_A_BYTES = (WG_KS / 4) * WG_A_LBO;  // one of hi / lo
constexpr int WG_B_BYTES = (WG_KS / 4) * WG_B_LBO;
constexpr int WG_STAGE = 2 * WG_A_BYTES + 2 * WG_B_BYTES;  // [A hi | A lo | B hi | B lo] = 88576 B
static_assert(WG_B_LBO >= (WG_NB / 8) * WG_SBO && WG_A_LBO % 128 == 16 && WG_B_LBO % 128 == 16, "operand strides");
constexpr int WG_SMEM_BARS = 2 * WG_STAGE;
constexpr int WG_SMEM = WG_SMEM_BARS + 64;
constexpr int WG_SROW = 132;                    // staging row stride (floats): 128 + 4, 16-byte stores of a quarter warp hit 8 bank groups
struct WgParams {
    const float* G[3];
    const float* X[3];
    float sign[3];           // per-term factor applied to G while loading (the merged primal + tangent call: +1, -1, -1)
    int scale_mask;          // bit t: term t's G rows are scaled by row_scale
    int bias_mask;           // bit t: term t contributes its column sums of G to dbias
    int n_terms, M, out, in, ldg, ldx, lddw;
    float* dW;
    float* dbias;
    const float* row_scale;  // optional per-row factor of G: row a is scaled by row_scale[a / rs_div] (the per-atom energy seed)
    int rs_div;
    float alpha, bias_alpha;
};

__device__ __forceinline__ void red4(float* p, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __launch_bounds__(WG_THREADS, 1) k_wgrad_tc(const WgParams P) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int o0 = blockIdx.y * 128;
    // sub-units of this CTA: u = blockIdx.x, + gridDim.x, ... over (term, 128-atom chunk); their products are summed in the accumulators
    const int n_chunks = (P.M + 127) >> 7, n_sub = n_chunks * P.n_terms;

    // loader mapping: a warp instruction covers 8 atoms x 16 features (lane = 8 * feature-quad + atom): 64-byte global segments.  Shared-memory
    // word of (feature f, atom a) = (f / 8) SBO + (f % 8) 16 + (a / 4) LBO + (a % 4) 4: for one of the 4 features of a lane's float4 the 32
    // lanes differ in a % 4 (words 0..3), a / 4 (+4 words), quad % 2 (+16 words), quad / 2 (+40 = 8 mod 32 words): 32 distinct banks.
    // Per stage 32 + 32 such instructions, 4 per warp.
    const int la = lane & 7, lq = lane >> 3;
    float4 v[4];
    auto load_stage = [&](int u, int st) {
        const int term = u / n_chunks, a0 = (u - term * n_chunks) << 7;
        const float* __restrict__ G = term == 0 ? P.G[0] : term == 1 ? P.G[1] : P.G[2];  // (no dynamic indexing: that would copy the parameters to local memory)
        const float* __restrict__ X = term == 0 ? P.X[0] : term == 1 ? P.X[1] : P.X[2];
        const float sgn = term == 0 ? P.sign[0] : term == 1 ? P.sign[1] : P.sign[2];
        const bool scaled = P.row_scale != nullptr && ((P.scale_mask >> term) & 1);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int inst = warp + 16 * j, kg = inst >> 3, fb = inst & 7;
            const int atom = a0 + st * WG_KS + kg * 8 + la, col = fb * 16 + lq * 4;
            const bool ok = atom < P.M;
            v[j] = (ok && o0 + col < P.out) ? ldg4(G + (size_t)atom * P.ldg + o0 + col) : f4(0.f);
            if (scaled && ok) v[j] = v[j] * __ldg(P.row_scale + atom / P.rs_div);
            if (sgn != 1.0f) v[j] = v[j] * sgn;
            v[2 + j] = (ok && col < P.in) ? ldg4(X + (size_t)atom * P.ldx + col) : f4(0.f);
        }
    };
    auto stages_of = [&](int u) {
        const int term = u / n_chunks, a0 = (u - term * n_chunks) << 7;
        return (min(128, P.M - a0) + WG_KS - 1) / WG_KS;
    };
    const int wg = warp >> 2, mh = wg & 1, nh = wg >> 1;
    float corr[36], acc[36], total[36];
#pragma unroll
    for (int i = 0; i < 36; ++i) { corr[i] = 0.f; acc[i] = 0.f; total[i] = 0.f; }
    int gs = 0;  // stages done so far (shared-memory buffer)
    if (blockIdx.x < n_sub) load_stage(blockIdx.x, 0);
#pragma unroll 1
    for (int u = blockIdx.x; u < n_sub; u += gridDim.x) {
        const int n_st = stages_of(u);
        const bool bias_on = P.dbias != nullptr && ((P.bias_mask >> (u / n_chunks)) & 1);
#pragma unroll 1
        for (int st = 0; st < n_st; ++st, ++gs) {
            unsigned char* sb = smem + (gs & 1) * WG_STAGE;
            __syncthreads();  // every warpgroup has waited for its MMAs of stage gs - 2, which read this buffer
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int inst = warp + 16 * j, kg = inst >> 3, fb = inst & 7;
                float4 hi, lo;
                // features fb * 16 + lq * 4 + c (c = 0..3): row group fb * 2 + lq / 2, row (lq % 2) * 4 + c; atom kg * 8 + la: chunk kg * 2 + la / 4, word la % 4
                const int row_off = (fb * 2 + (lq >> 1)) * WG_SBO + (lq & 1) * 64 + (la & 3) * 4;
                const int offa = (kg * 2 + (la >> 2)) * WG_A_LBO + row_off, offb = (kg * 2 + (la >> 2)) * WG_B_LBO + row_off;
                split4(v[j], hi, lo);
                float* ah = reinterpret_cast<float*>(sb + offa);
                float* al = reinterpret_cast<float*>(sb + WG_A_BYTES + offa);
                ah[0] = hi.x; ah[4] = hi.y; ah[8] = hi.z; ah[12] = hi.w;
                al[0] = lo.x; al[4] = lo.y; al[8] = lo.z; al[12] = lo.w;
                split4(v[2 + j], hi, lo);
                float* bh = reinterpret_cast<float*>(sb + 2 * WG_A_BYTES + offb);
                float* bl = reinterpret_cast<float*>(sb + 2 * WG_A_BYTES + WG_B_BYTES + offb);
                bh[0] = hi.x; bh[4] = hi.y; bh[8] = hi.z; bh[12] = hi.w;
                bl[0] = lo.x; bl[4] = lo.y; bl[8] = lo.z; bl[12] = lo.w;
            }
            if (tid < 2 * (WG_KS / 4) * 16) {  // the constant rows of B (inputs 128..143): hi = 1 in row 128 for a bias-carrying term, else 0
                const int r = tid & 15, kc = (tid >> 4) & 7, hl = tid >> 7;
                const float one = (hl == 0 && r == 0 && bias_on) ? 1.0f : 0.0f;
                *reinterpret_cast<float4*>(sb + 2 * WG_A_BYTES + hl * WG_B_BYTES + kc * WG_B_LBO + (16 + (r >> 3)) * WG_SBO + (r & 7) * 16) =
                    make_float4(one, one, one, one);
            }
            fence_proxy_async();
            __syncthreads();
            const uint32_t sa = s_u32(sb) + mh * 8 * WG_SBO, sbb = s_u32(sb) + 2 * WG_A_BYTES + nh * 9 * WG_SBO;
            wgmma_fence();
#pragma unroll
            for (int kg = 0; kg < WG_KS / 8; ++kg) {
                const uint64_t a_hi = gmma_desc(sa + 2 * kg * WG_A_LBO, WG_A_LBO, WG_SBO), a_lo = gmma_desc(sa + WG_A_BYTES + 2 * kg * WG_A_LBO, WG_A_LBO, WG_SBO);
                const uint64_t b_hi = gmma_desc(sbb + 2 * kg * WG_B_LBO, WG_B_LBO, WG_SBO), b_lo = gmma_desc(sbb + WG_B_BYTES + 2 * kg * WG_B_LBO, WG_B_LBO, WG_SBO);
                wgmma_tf32_n72(corr, a_lo, b_hi);
                wgmma_tf32_n72(corr, a_hi, b_lo);
                wgmma_tf32_n72(acc, a_hi, b_hi);
            }
            wgmma_commit();
            // next stage's global loads in flight while the tensor core works on this one (across the sub-unit boundary too)
            if (st + 1 < n_st) load_stage(u, st + 1);
            else if (u + (int)gridDim.x < n_sub) load_stage(u + gridDim.x, 0);
            wgmma_wait<1>();
        }
        wgmma_wait<0>();  // this sub-unit's products -> fp32 sums (RN adds), accumulators restart
#pragma unroll
        for (int i = 0; i < 36; ++i) { total[i] += corr[i] + acc[i]; corr[i] = 0.f; acc[i] = 0.f; }
    }

    // ---- epilogue: fragments -> staging rows [output][input] (the operand buffers: every MMA has completed) -> coalesced vector
    //      reductions into dW, one per CTA and output element.  Fragment: rows 64 mh + 16 (warp & 3) + lane / 4 (+ 8), B columns
    //      72 nh + 8 j + 2 (lane & 3) (+ 1); column 128 (nh = 1, j = 7, lane & 3 = 0) is the bias gradient.
    __syncthreads();
    float* stage = reinterpret_cast<float*>(smem);
    const int orow = 64 * mh + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 9; ++j) {
        const int col = 72 * nh + 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int e = 4 * j + 2 * hr, r = orow + 8 * hr;
            if (col < 128) {
                *reinterpret_cast<float2*>(stage + r * WG_SROW + col) = make_float2(total[e] * P.alpha, total[e + 1] * P.alpha);
            } else if (col == 128 && P.dbias != nullptr && o0 + r < P.out) {
                const float bsum = total[e];
                if (bsum != 0.f) atomicAdd(P.dbias + o0 + r, P.bias_alpha * bsum);
            }
        }
    }
    __syncthreads();
    if (4 * lane < P.in) {
#pragma unroll 4
        for (int r = warp; r < 128; r += 16) {
            if (o0 + r >= P.out) break;
            red4(P.dW + (size_t)(o0 + r) * P.lddw + 4 * lane, *reinterpret_cast<const float4*>(stage + r * WG_SROW + 4 * lane));
        }
    }
}

}  // namespace

// Shapes the kernel takes: in <= 128 and a multiple of 16 (16-feature loader blocks), out a multiple of 4, 16-byte aligned rows everywhere.
bool nb_wgrad_tc_ok(int M, int out, int in, const float* G0, int ldg, const float* X0, int ldx, const float* dW, int lddw) {
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    return M >= 1 && out >= 4 && out % 4 == 0 && in >= 16 && in <= 128 && in % 16 == 0 && ldg % 4 == 0 && ldx % 4 == 0 && lddw % 4 == 0 && al(G0) && al(X0) &&
           al(dW);
}

static int wgrad_launch(WgParams& P, cudaStream_t s) {
    static bool attr_set = false;  // per process; cudaFuncSetAttribute is idempotent, a race only repeats it
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM) != cudaSuccess) return nb_check_launch();
        attr_set = true;
    }
    const int n_sm = nb_sm_count();
    const int out_tiles = (P.out + 127) / 128, n_sub = ((P.M + 127) / 128) * P.n_terms;
    int groups = n_sm / out_tiles;  // one CTA per SM; each sums its (term, chunk) sub-units in registers before ONE atomic flush
    groups = groups < 1 ? 1 : groups > n_sub ? n_sub : groups;
    dim3 grid(groups, out_tiles, 1);
    k_wgrad_tc<<<grid, WG_THREADS, WG_SMEM, s>>>(P);
    return nb_check_launch();
}

int nb_wgrad_tc(int M, int out, int in, const float* G0, const float* X0, const float* G1, const float* X1, int ldg, int ldx, float* dW, int lddw,
                float alpha, float* dbias, float bias_alpha, int bias_term, const float* row_scale, int rs_div, cudaStream_t s) {
    WgParams P{};
    P.G[0] = G0; P.X[0] = X0; P.G[1] = G1 ? G1 : G0; P.X[1] = X1 ? X1 : X0; P.G[2] = G0; P.X[2] = X0;
    P.sign[0] = P.sign[1] = P.sign[2] = 1.0f;
    P.n_terms = G1 ? 2 : 1;
    P.M = M; P.out = out; P.in = in; P.ldg = ldg; P.ldx = ldx; P.lddw = lddw; P.bias_mask = 1 << bias_term; P.scale_mask = 1;
    P.row_scale = row_scale; P.rs_div = rs_div > 0 ? rs_div : 1;
    P.dW = dW; P.dbias = dbias; P.alpha = alpha; P.bias_alpha = bias_alpha;
    return wgrad_launch(P, s);
}

// Energy-seed term and force-seed (tangent) terms of ONE Linear layer's weight gradient in a single launch:
//   dW += (c o g)^T x - (tg^T x + g^T tx),   dbias += colsum(c o g) - colsum(tg)        (c = per-atom energy seed, rows / rs_div)
int nb_wgrad_tc3(int M, int out, int in, const float* g, const float* tg, int ldg, const float* x, const float* tx, int ldx, float* dW, int lddw,
                 float* dbias, const float* row_scale, int rs_div, cudaStream_t s) {
    WgParams P{};
    P.G[0] = g; P.X[0] = x; P.G[1] = tg; P.X[1] = x; P.G[2] = g; P.X[2] = tx;
    P.sign[0] = 1.0f; P.sign[1] = -1.0f; P.sign[2] = -1.0f;
    P.n_terms = 3; P.scale_mask = 1; P.bias_mask = 3;
    P.M = M; P.out = out; P.in = in; P.ldg = ldg; P.ldx = ldx; P.lddw = lddw;
    P.row_scale = row_scale; P.rs_div = rs_div > 0 ? rs_div : 1;
    P.dW = dW; P.dbias = dbias; P.alpha = 1.0f; P.bias_alpha = 1.0f;
    return wgrad_launch(P, s);
}

extern "C" int nb200_linear_wgrad(int32_t M, int32_t out, int32_t in, const float* G0, const float* X0, const float* G1, const float* X1, int32_t ldg,
                                  int32_t ldx, float* dW, int32_t lddw, float alpha, float* dbias, float bias_alpha, const float* row_scale,
                                  int32_t rs_div, void* stream) {
    if (!G0 || !X0 || !dW || (G1 == nullptr) != (X1 == nullptr) || !nb_wgrad_tc_ok(M, out, in, G0, ldg, X0, ldx, dW, lddw) ||
        (G1 && !nb_wgrad_tc_ok(M, out, in, G1, ldg, X1, ldx, dW, lddw)))
        return NB200_EINVAL;
    return nb_wgrad_tc(M, out, in, G0, X0, G1, X1, ldg, ldx, dW, lddw, alpha, dbias, bias_alpha, 0, row_scale, rs_div, (cudaStream_t)stream);
}
