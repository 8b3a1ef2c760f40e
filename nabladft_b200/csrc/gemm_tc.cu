// gemm_tc.cu -- node-level dense layers on the Hopper tensor cores (wgmma), fp32-accurate.
//
// Replaces the cuBLAS SGEMM calls of engine.cu (torch.nn.Linear forward / input-gradient of
// nablaDFT/painn_pyg/painn.py:459-464,520-525 and the schnetpack Dense layers) for the skinny
// problems of this model (M ~ 10^4 atoms, N,K in {64..384}).
//
// The reference never uses reduced precision (SURVEY.md section 0.9), so single-pass TF32 is
// out.  We use the 3xTF32 split: x = hi + lo with hi = tf32_rn(x), lo = tf32_rn(x - hi);
//   A.B ~= A_hi.B_hi + A_hi.B_lo + A_lo.B_hi       (dropped term ~2^-24 relative)
// three `wgmma.mma_async ... .tf32` per k-step accumulating in fp32 registers.  The operands are
// split on the fly while they are staged from global into shared memory by the CTA's threads
// (canonical no-swizzle K-major layout: 16-byte k-chunks, rows contiguous), so activations
// never need a pre-pass and weights need no transposed copies (`trans_b` loads B^T directly).
//
//   C[M,N] (ldc) = A[M,K] (lda) . op(B)  (+ C if accumulate)  (+ bias[N])
//   op(B) = B[N,K]^T (ldb, trans_b = 0: Linear forward)  |  B[K,N] (ldb, trans_b = 1: Linear backward)
//   optional second output  act[M,N] = silu(C)   (C then holds the pre-activation)
// k_gemm_tf32x3: tile 128 x 64 x 32, 512 threads = four warpgroups (each a 64 x 32 quarter of the tile), double-buffered stages with
// register prefetch.  Tall problems go to the pre-split-weight kernel of gemm_ps.cu.
#include <cstdlib>

#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int G_BM = 128;
constexpr int G_BN = 64;
constexpr int G_BK = 32;
constexpr int G_THREADS = 512;  // 16 warps: the hi/lo split is SIMT work and wants many threads

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// round-to-nearest split (cvt.rna.tf32.f32): |x - hi| <= 2^-12 |x| and the rounding of lo costs
// 2^-24 |x| -- fp32-level and unbiased.  (Masking the low 13 bits instead truncates toward zero.)
__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = tf32_rn(x);
    lo = tf32_rn(x - hi);
}
__device__ __forceinline__ void split4(const float4 v, float4& hi, float4& lo) {
    split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y); split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
}

// element (row r, k) of a [ROWS x 32] stage tile lives at float index ((k/4)*ROWS + r)*4 + k%4
struct Stage {
    float a_hi[G_BM * G_BK], a_lo[G_BM * G_BK], b_hi[G_BN * G_BK], b_lo[G_BN * G_BK];
};

__global__ void __launch_bounds__(G_THREADS, 1) k_gemm_tf32x3(int M, int N, int K, const float* __restrict__ A, int lda,
                                                             const float* __restrict__ B, int ldb, int trans_b, float* C, int ldc,
                                                             int accumulate, const float* __restrict__ bias, float* __restrict__ act, int act_kind,
                                                             int batch_kind, long long a_boff, long long b_boff, long long c_boff) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Stage* stages = reinterpret_cast<Stage*>(smem_raw);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * G_BM, n0 = blockIdx.y * G_BN;
    if (batch_kind != 0) {
        // batch over blockIdx.z: A and C advance by a fixed offset; B is selected per batch entry.
        // kind 1 = "lm blocks" of an equivariant feature [rows][(l,m)][channels]: z = (l,m) index,
        // the weight block is W_l (o3.Linear mixes channels per l), bias only on (l,m) = (0,0).
        const int z = blockIdx.z;
        const int bsel = (batch_kind == 1) ? (z >= 16 ? 4 : z >= 9 ? 3 : z >= 4 ? 2 : z >= 1 ? 1 : 0) : z;
        A += (size_t)z * a_boff;
        B += (size_t)bsel * b_boff;
        C += (size_t)z * c_boff;
        if (act) act += (size_t)z * c_boff;
        if (batch_kind == 1 && z > 0) bias = nullptr;
    }

    constexpr int BPT = G_BN * (G_BK / 4) / G_THREADS;  // B float4 per thread per chunk
    const int n_chunks = K / G_BK;
    constexpr int APT = G_BM * (G_BK / 4) / G_THREADS;  // A float4 per thread per chunk
    const int atile_row = tid % G_BM;                 // this thread stages k-chunks [akc0, akc0 + APT) of row `atile_row` of the A tile
    const int akc0 = (tid / G_BM) * APT;
    const int arow = m0 + atile_row;
    const bool arow_ok = arow < M;
    const int btile_row = tid % G_BN;                 // and k-chunks [bkc0, bkc0 + BPT) of row `btile_row` of the B tile
    const int bkc0 = (tid / G_BN) * BPT;
    const int brow = n0 + btile_row;
    const bool brow_ok = brow < N;
    // warpgroup g computes rows [64 (g & 1), +64) x columns [32 (g >> 1), +32) of the tile
    const int wg = warp >> 2, mh = wg & 1, nh = wg >> 1;
    // The tensor core truncates when it adds into the fp32 accumulator, so the error grows with the chain length: the O(2^-11)
    // correction terms get their own accumulator and the main term alternates over two; the three are summed with RN adds at the end.
    float corr[16], acc0[16], acc1[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) { corr[i] = 0.f; acc0[i] = 0.f; acc1[i] = 0.f; }

    // global -> registers (issued one chunk ahead of the shared-memory stores: the L2 latency of
    // chunk c+1 overlaps the split/store/MMA of chunk c)
    auto gload = [&](int ch, float4 (&ra)[APT], float4 (&rb)[BPT]) {
        const int k0 = ch * G_BK;
        const float* src = A + (size_t)arow * lda + k0;
#pragma unroll
        for (int i = 0; i < APT; ++i) ra[i] = arow_ok ? ldg4(src + 4 * (akc0 + i)) : f4(0.f);
#pragma unroll
        for (int i = 0; i < BPT; ++i) {
            const int kc = bkc0 + i;
            float4 v = f4(0.f);
            if (brow_ok) {
                if (!trans_b) {
                    v = ldg4(B + (size_t)brow * ldb + k0 + 4 * kc);
                } else {  // B[k][n]: four k-rows, coalesced across the threads of a warp (consecutive n)
                    const float* p = B + (size_t)(k0 + 4 * kc) * ldb + brow;
                    v = make_float4(__ldg(p), __ldg(p + ldb), __ldg(p + 2 * (size_t)ldb), __ldg(p + 3 * (size_t)ldb));
                }
            }
            rb[i] = v;
        }
    };
    // registers -> hi/lo split -> shared ([k-chunk][row] 16-byte units: conflict-free), then the MMAs of this warpgroup
    auto process = [&](int ch, const float4 (&ra)[APT], const float4 (&rb)[BPT]) {
        const int s = ch & 1;
        __syncthreads();  // every warpgroup has waited for its MMAs of chunk ch - 2, which read this buffer
        Stage& st = stages[s];
#pragma unroll
        for (int i = 0; i < APT; ++i) {
            float4 hi, lo;
            split4(ra[i], hi, lo);
            st4(st.a_hi + ((akc0 + i) * G_BM + atile_row) * 4, hi);
            st4(st.a_lo + ((akc0 + i) * G_BM + atile_row) * 4, lo);
        }
#pragma unroll
        for (int i = 0; i < BPT; ++i) {
            float4 hi, lo;
            split4(rb[i], hi, lo);
            st4(st.b_hi + ((bkc0 + i) * G_BN + btile_row) * 4, hi);
            st4(st.b_lo + ((bkc0 + i) * G_BN + btile_row) * 4, lo);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy smem writes -> visible to the MMA (async proxy)
        __syncthreads();
        const uint32_t ah = s_u32(st.a_hi) + mh * 64 * 16, al = s_u32(st.a_lo) + mh * 64 * 16;
        const uint32_t bh = s_u32(st.b_hi) + nh * 32 * 16, bl = s_u32(st.b_lo) + nh * 32 * 16;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < G_BK / 8; ++ks) {  // one MMA = 8 k-values = two 16-byte chunks
            const uint32_t ao = ks * 2 * G_BM * 16, bo = ks * 2 * G_BN * 16;
            const uint64_t dah = gmma_desc(ah + ao, G_BM * 16, 128), dal = gmma_desc(al + ao, G_BM * 16, 128);
            const uint64_t dbh = gmma_desc(bh + bo, G_BN * 16, 128), dbl = gmma_desc(bl + bo, G_BN * 16, 128);
            wgmma_tf32_n32(corr, dal, dbh);
            wgmma_tf32_n32(corr, dah, dbl);
            if (ks & 1) wgmma_tf32_n32(acc1, dah, dbh);
            else wgmma_tf32_n32(acc0, dah, dbh);
        }
        wgmma_commit();
        wgmma_wait<1>();  // chunk ch - 1 has completed (its buffer is rewritten after the next barrier)
    };

    {
        float4 ra0[APT], rb0[BPT], ra1[APT], rb1[BPT];
        gload(0, ra0, rb0);
        for (int ch = 0; ch < n_chunks; ch += 2) {
            if (ch + 1 < n_chunks) gload(ch + 1, ra1, rb1);
            process(ch, ra0, rb0);
            if (ch + 1 < n_chunks) {
                if (ch + 2 < n_chunks) gload(ch + 2, ra0, rb0);
                process(ch + 1, ra1, rb1);
            }
        }
    }
    wgmma_wait<0>();
    // ---- epilogue from the fragments: rows 64 mh + 16 (warp & 3) + lane / 4 (+ 8), columns 32 nh + 8 j + 2 (lane & 3) (+ 1)
    const int r0 = m0 + 64 * mh + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int n = n0 + 32 * nh + 8 * j + 2 * (lane & 3);
        if (n >= N) continue;  // N % 4 == 0: n < N implies n + 1 < N
        const float2 b = bias ? __ldg(reinterpret_cast<const float2*>(bias + n)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = r0 + 8 * hr;
            if (row >= M) continue;
            const int e = 4 * j + 2 * hr;
            float2 v = make_float2((corr[e] + acc0[e]) + acc1[e] + b.x, (corr[e + 1] + acc0[e + 1]) + acc1[e + 1] + b.y);
            float2* cp = reinterpret_cast<float2*>(C + (size_t)row * ldc + n);
            if (accumulate) { const float2 o = *cp; v.x += o.x; v.y += o.y; }
            *cp = v;
            if (act) *reinterpret_cast<float2*>(act + (size_t)row * ldc + n) = make_float2(actf_(v.x, act_kind), actf_(v.y, act_kind));
        }
    }
}

int launch(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
           const float* bias, float* act, int act_kind, int batch_kind, int n_batch, long long a_boff, long long b_boff, long long c_boff,
           cudaStream_t s) {
    const int smem = 2 * (int)sizeof(Stage);
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(k_gemm_tf32x3, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return nb_check_launch();
        attr_set = true;
    }
    dim3 grid((M + G_BM - 1) / G_BM, (N + G_BN - 1) / G_BN, batch_kind ? n_batch : 1);
    k_gemm_tf32x3<<<grid, G_THREADS, smem, s>>>(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, act_kind, batch_kind, a_boff,
                                                b_boff, c_boff);
    return nb_check_launch();
}

}  // namespace

// Constraints: K % 32 == 0, N % 4 == 0, lda/ldb/ldc % 4 == 0, 16-byte aligned pointers; `act` (optional) shares ldc with C.
int nb_gemm_tf32x3_ex(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
                      const float* bias, float* act, int act_kind, cudaStream_t s) {
    if (!A || !B || !C || M < 0 || N <= 0 || K <= 0) return NB200_EINVAL;
    if (K % G_BK || N % 4 || lda % 4 || ldb % 4 || ldc % 4) return NB200_EUNSUPPORTED;
    if (M == 0) return NB200_OK;
    // tall problems: weights pre-split once into shared-memory tile images and streamed (gemm_ps.cu); NB200_GEMM_VARIANT=tile keeps every
    // shape on the tile kernel below, =ps forces the pre-split kernel
    static const int variant = [] { const char* e = getenv("NB200_GEMM_VARIANT"); return !e ? 0 : (e[0] == 't') ? 1 : (e[0] == 'p') ? 3 : 0; }();
    if (variant == 3 || (variant == 0 && nb_gemm_ps_wanted(M, N, K)))
        return nb_gemm_ps(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, act_kind, nullptr, 0, s);
    return launch(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, act_kind, 0, 1, 0, 0, 0, s);
}

// batched over the 25 (l,m) rows of an equivariant feature: see batch_kind 1 in the kernel
int nb_gemm_tf32x3_lm(int M, int N, int K, const float* A, int lda, const float* W_l, long long w_l_stride, float* C, int ldc, int accumulate,
                      const float* bias, int n_lm, cudaStream_t s) {
    if (!A || !W_l || !C || M < 0 || N <= 0 || K <= 0) return NB200_EINVAL;
    if (K % G_BK || N % 4 || lda % 4 || ldc % 4) return NB200_EUNSUPPORTED;
    if (M == 0) return NB200_OK;
    // tall inputs (per-pair features of QHNet / PhiSNet: 1e5 rows x 25 slices): pre-split weights, one launch over (row slab, slice)
    static const bool ps_off = [] { const char* e = getenv("NB200_GEMM_VARIANT"); return e && e[0] == 't'; }();
    if (!ps_off && nb_gemm_ps_lm_wanted(M, N, K)) return nb_gemm_ps_lm(M, N, K, A, lda, W_l, w_l_stride, C, ldc, accumulate, bias, n_lm, s);
    return launch(M, N, K, A, lda, W_l, N, 1, C, ldc, accumulate, bias, nullptr, NB_ACT_SILU, 1, n_lm, K, w_l_stride, N, s);
}

extern "C" int nb200_gemm_tf32x3(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb,
                                 int32_t trans_b, float* C, int32_t ldc, int32_t accumulate, const float* bias, float* act,
                                 void* stream) {
    return nb_gemm_tf32x3_ex(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, NB_ACT_SILU, (cudaStream_t)stream);
}
