// gemnet_pf.cuh -- launch abstraction and dense layers of the functor engines (gemnet_oc.cu, schnet_train.cu, dimenet.cu).
//
// Every kernel of these engines is a functor with `operator()(int64_t i)`: one logical thread per output element, no shared memory, no warp
// intrinsics; forward aggregations are gathers over CSR rows (deterministic), only some backward scatters use atomicAdd.  `pfor` launches a
// functor as a grid-stride kernel sized to the SM count.  The same translation units also compile as plain C++ with -DNB_EMU (tests/emu/):
// there `pfor` is an OpenMP loop, the library GEMMs (wgmma, cuBLAS) are replaced by the functor GEMMs, and every workspace array gets a
// guard zone -- which lets the CPU test-suite check every functor against the oracle when no GPU is at hand.  The emulation build is TEST
// INFRASTRUCTURE: the package never loads it (nabladft_b200/_lib.py loads libnabla_b200.so only).
#pragma once
#ifdef NB_EMU
#include "emu_shim.h"
#else
#include "common.cuh"
#include "engine_common.cuh"
#include <cstdlib>
#include <cstring>
#endif

#define GD __device__ __forceinline__

// Extent of a launch or of a GEMM in rows.  `dev` == nullptr: exactly `n` rows.  `dev` set: `n` is an upper bound the host knows (it sizes the
// grid, the GEMM and the arrays) and the row count is read from device memory inside the kernel, so the host never waits for it.
struct Ext {
    int64_t n; const int32_t* dev;
    Ext(int64_t n_, const int32_t* dev_ = nullptr) : n(n_), dev(dev_) {}
};
GD int64_t ext_rows(int64_t bound, const int32_t* dev) {
    if (!dev) return bound;
    const int64_t r = *dev;
    return r < bound ? r : bound;  // a count above the bound is reported through the status words (StatusCountsK), never indexed
}
#ifdef NB_EMU
// host emulation of what the engines use beyond the stand-ins of emu_shim.h: int32 atomics of the status kernels (StatusAtomK) ...
inline int32_t atomicAdd(int32_t* p, int32_t v) {
    int32_t old;
#pragma omp atomic capture
    { old = *p; *p += v; }
    return old;
}
inline int32_t atomicMax(int32_t* p, int32_t v) {
    int32_t old;
#pragma omp critical(nb_emu_minmax)
    { old = *p; if (v > old) *p = v; }
    return old;
}
inline int32_t atomicMin(int32_t* p, int32_t v) {
    int32_t old;
#pragma omp critical(nb_emu_minmax)
    { old = *p; if (v < old) *p = v; }
    return old;
}
// ... and the launch over an extent whose row count lives on the "device"
template <class F>
inline int pfor(nb200_engine* e, cudaStream_t s, int category, Ext x, int64_t per_row, const F& f) {
    return pfor(e, s, category, ext_rows(x.n, x.dev) * per_row, f);  // host emulation: the "device" count is readable here
}
#endif

// Workspace carver shared by the functor engines: 256-byte aligned sub-buffers of ONE caller-owned allocation (base == nullptr: size query).
// Under host emulation every sub-buffer is followed by a guard zone filled with a sentinel; tests call nb200_emu_check_guards() after a run
// to prove that no kernel wrote past the end of its array (writes inside one allocation are invisible to ASan-style tools).
struct Carve {
    char* base; int64_t off = 0;
    explicit Carve(void* p) : base(static_cast<char*>(p)) {}
    template <class T>
    T* take(int64_t count) {
        off = (off + 255) / 256 * 256;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * (int64_t)sizeof(T);
#ifdef NB_EMU
        if (base) emu_guard_add(base + off);
        off += NB_EMU_GUARD_BYTES;
#endif
        return p;
    }
};

#ifndef NB_EMU
template <class F>
__global__ void __launch_bounds__(256) k_pfor(int64_t n, F f) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) f(i);
}
// grid: enough 256-thread CTAs to cover n, capped at 8 resident CTAs on each SM (grid-stride beyond that)
template <class F>
inline int pfor(nb200_engine* e, cudaStream_t s, int category, int64_t n, const F& f) {
    if (n <= 0) return NB200_OK;
    static_assert(sizeof(F) <= 4000, "functor must fit the kernel parameter space");
    Scope sc(e, s, category, 1);
    const int64_t want = (n + 255) / 256;
    const int blocks = (int)(want < nb_sm_count() * 8 ? want : nb_sm_count() * 8);
    k_pfor<F><<<blocks, 256, 0, s>>>(n, f);
    return nb_check_launch();
}

// the same for an extent whose row count lives on the device: grid from the bound, loop limit read inside the kernel
template <class F>
__global__ void __launch_bounds__(256) k_pfor_rows(int64_t bound, const int32_t* rows, int64_t per_row, F f) {
    const int64_t n = ext_rows(bound, rows) * per_row;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) f(i);
}
template <class F>
inline int pfor(nb200_engine* e, cudaStream_t s, int category, Ext x, int64_t per_row, const F& f) {
    if (!x.dev) return pfor(e, s, category, x.n * per_row, f);
    if (x.n <= 0) return NB200_OK;
    static_assert(sizeof(F) <= 4000, "functor must fit the kernel parameter space");
    Scope sc(e, s, category, 1);
    const int64_t want = (x.n * per_row + 255) / 256;
    const int blocks = (int)(want < nb_sm_count() * 8 ? want : nb_sm_count() * 8);
    k_pfor_rows<F><<<blocks, 256, 0, s>>>(x.n, x.dev, per_row, f);
    return nb_check_launch();
}

// single-CTA exclusive scan of int32 counts: out[0..n] (n+1 entries), out[n] = total
static __global__ void __launch_bounds__(1024) k_goc_scan(const int32_t* __restrict__ in, int32_t n, int32_t* __restrict__ out) {
    __shared__ int64_t part[1024];
    const int t = threadIdx.x;
    const int64_t chunk = ((int64_t)n + 1023) / 1024;
    const int64_t lo = t * chunk, hi = (lo + chunk < n) ? lo + chunk : n;
    int64_t sum = 0;
    for (int64_t i = lo; i < hi; i++) sum += in[i];
    part[t] = sum;
    __syncthreads();
    if (t == 0) {
        int64_t run = 0;
        for (int k = 0; k < 1024; k++) {
            const int64_t v = part[k];
            part[k] = run;
            run += v;
        }
        out[n] = (int32_t)run;
    }
    __syncthreads();
    int64_t run = part[t];
    for (int64_t i = lo; i < hi; i++) {
        out[i] = (int32_t)run;
        run += in[i];
    }
}
inline int scan_excl(nb200_engine* e, cudaStream_t s, const int32_t* in, int32_t n, int32_t* out) {
    Scope sc(e, s, CAT_NBR, 1);
    k_goc_scan<<<1, 1024, 0, s>>>(in, n, out);
    return nb_check_launch();
}
inline int goc_memset(void* p, int v, size_t bytes, cudaStream_t s) { return cudaMemsetAsync(p, v, bytes, s) == cudaSuccess ? NB200_OK : NB200_ECUDA; }
inline int goc_d2h_sync(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    if (cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess) return NB200_ECUDA;
    return cudaStreamSynchronize(s) == cudaSuccess ? NB200_OK : NB200_ECUDA;
}
inline int goc_d2d(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s) == cudaSuccess ? NB200_OK : NB200_ECUDA;
}
// the shape fits the tiling of the wgmma GEMM (nb_gemm_tf32x3_ex)
inline bool goc_tc_ok(int N, int K, int lda, int ldw, int ldc) {
    // N % 32: the 128 x 64 tile kernel masks the columns beyond N, so the quadruplet bilinear layer (1024 -> 32 per edge, ~6 % of the model's
    // FLOPs) runs on the tensor cores with a half-empty tile instead of the functor fallback
    return N % 32 == 0 && K % 32 == 0 && lda % 4 == 0 && ldw % 4 == 0 && ldc % 4 == 0;
}
// dW[out, in] (lddw) += alpha * gY[M, out]^T (ldgy) . X[M, in] (ldx): weight gradient of a Linear layer as ONE cuBLAS SGEMM (fp32, no TF32).
// false = not available (no handle, M beyond int32): the caller falls back to the row-chunked functor reduction.
inline bool goc_wgrad(nb200_engine* e, cudaStream_t s, int64_t M, int out, int in, const float* gY, int ldgy, const float* X, int ldx, float* dW, int lddw,
                      float alpha, int* rc) {
    if (!e || !e->blas || M > 0x7fffffff || M <= 0 || out <= 0 || in <= 0) return false;
    Scope sc(e, s, CAT_GEMM, 0);
    const float beta = 1.0f;
    *rc = (cublasSetStream(e->blas, s) == CUBLAS_STATUS_SUCCESS &&
           cublasSgemm(e->blas, CUBLAS_OP_N, CUBLAS_OP_T, in, out, (int)M, &alpha, X, ldx, gY, ldgy, &beta, dW, lddw) == CUBLAS_STATUS_SUCCESS)
              ? NB200_OK
              : NB200_ECUDA;
    return true;
}
#endif

// ---------------------------------------------------------------- dense layers of the functor engines
// Each layer runs on the wgmma 3xTF32 GEMM when its shape tiles and M fits int32, else on a functor GEMM; weight gradients run as one cuBLAS
// SGEMM, else as a row-chunked functor reduction.  Host emulation takes the functors, or with NB200_EMU_LIBGEMM=1 the library stand-ins of
// emu_shim.h.
namespace {
constexpr int WGRAD_ROWS = 512;  // rows one thread of DenseWgradK sums before its atomicAdd

GD float silu(float x) { return x / (1.0f + expf(-x)); }
struct ActK {  // y = silu(x)
    const float* x; float* y;
    GD void operator()(int64_t i) const { y[i] = silu(x[i]); }
};
struct DenseK {  // C[r, n] (+)= A[r, :] . W[n, :] (+ bias[n])
    const float* A; int32_t lda; const float* W; int32_t ldw; float* C; int32_t ldc; int32_t N, K; const float* bias; int32_t acc;
    GD void operator()(int64_t i) const {
        const int64_t r = i / N; const int n = (int)(i % N);
        const float* a = A + r * lda; const float* w = W + (int64_t)n * ldw;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
        int k = 0;
        for (; k + 4 <= K; k += 4) { s0 += a[k] * w[k]; s1 += a[k + 1] * w[k + 1]; s2 += a[k + 2] * w[k + 2]; s3 += a[k + 3] * w[k + 3]; }
        for (; k < K; k++) s0 += a[k] * w[k];
        float v = (s0 + s1) + (s2 + s3);
        if (bias) v += bias[n];
        float& c = C[r * ldc + n];
        c = acc ? c + v : v;
    }
};
struct DenseDgradK {  // gA[r, k] (+)= sum_n gC[r, n] W[n, k]
    const float* gC; int32_t ldc; const float* W; int32_t ldw; float* gA; int32_t lda; int32_t N, K; int32_t acc;
    GD void operator()(int64_t i) const {
        const int64_t r = i / K; const int k = (int)(i % K);
        const float* g = gC + r * ldc;
        float s0 = 0.0f, s1 = 0.0f;
        int n = 0;
        for (; n + 2 <= N; n += 2) { s0 += g[n] * W[(int64_t)n * ldw + k]; s1 += g[n + 1] * W[(int64_t)(n + 1) * ldw + k]; }
        if (n < N) s0 += g[n] * W[(int64_t)n * ldw + k];
        float& c = gA[r * lda + k];
        c = acc ? c + (s0 + s1) : (s0 + s1);
    }
};
struct DenseWgradK {  // gW[n, k] += alpha * sum over a chunk of rows of gC[r, n] A[r, k];  i = (chunk, n, k)
    const float* gC; int32_t ldc; const float* A; int32_t lda; float* gW; int32_t ldw; int32_t N, K; int64_t M; float alpha;
    GD void operator()(int64_t i) const {
        const int64_t nk = (int64_t)N * K, chunk = i / nk;
        const int n = (int)((i % nk) / K), k = (int)(i % K);
        const int64_t r0 = chunk * WGRAD_ROWS, r1 = r0 + WGRAD_ROWS < M ? r0 + WGRAD_ROWS : M;
        float s = 0.0f;
        for (int64_t r = r0; r < r1; r++) s += gC[r * ldc + n] * A[r * lda + k];
        atomicAdd(gW + (int64_t)n * ldw + k, alpha * s);
    }
};

// The wgmma GEMM nb_gemm_tf32x3_ex: C[M, N] (ldc) (+)= A[M, K] (lda) . op(W) (+ bias[N]), op(W) = W[N, K]^T (trans 0) | W[K, N] (trans 1);
// act != nullptr (ldc == N): act = silu(C).  Host emulation runs the stand-in goc_tc_gemm_ex of emu_shim.h over the rows below the "device"
// count (readable there) and applies the activation separately.
inline int tc_gemm(nb200_engine* e, cudaStream_t s, Ext M, int N, int K, const float* A, int lda, const float* W, int ldw, int trans, float* C, int ldc,
                   bool acc, const float* bias, float* act) {
#ifdef NB_EMU
    const int64_t rows = ext_rows(M.n, M.dev);
    if (rows > 0) NB_TRY(goc_tc_gemm_ex(e, s, (int)rows, N, K, A, lda, W, ldw, trans, C, ldc, acc, bias));
    return act ? pfor(e, s, CAT_NODE, M, N, ActK{C, act}) : NB200_OK;
#else
    Scope sc(e, s, CAT_GEMM, 1);
    return nb_gemm_tf32x3_ex((int)M.n, N, K, A, lda, W, ldw, trans, C, ldc, acc, bias, act, NB_ACT_SILU, s, M.dev);
#endif
}

// C[M, N] (ldc) (+)= A[M, K] (lda) . W[N, K]^T (ldw) (+ bias[N]);  act != nullptr (ldc == N): act = silu(C), C keeps the pre-activation.
// M.dev set: M.n is the bound, and rows at or past the device count are neither computed nor written.
inline int dense_fwd(nb200_engine* e, cudaStream_t s, Ext M, int N, int K, const float* A, int lda, const float* W, int ldw, float* C, int ldc,
                     bool acc = false, const float* bias = nullptr, float* act = nullptr) {
    if (M.n <= 0) return NB200_OK;
    if (M.n <= 0x7fffffff && goc_tc_ok(N, K, lda, ldw, ldc)) return tc_gemm(e, s, M, N, K, A, lda, W, ldw, 0, C, ldc, acc, bias, act);
    NB_TRY(pfor(e, s, CAT_GEMM, M, N, DenseK{A, lda, W, ldw, C, ldc, N, K, bias, acc}));
    return act ? pfor(e, s, CAT_NODE, M, N, ActK{C, act}) : NB200_OK;
}
// gA[M, K] (lda) (+)= gC[M, N] (ldc) . W[N, K] (ldw): the input gradient of dense_fwd.  M as in dense_fwd.
inline int dense_dgrad(nb200_engine* e, cudaStream_t s, Ext M, int N, int K, const float* gC, int ldc, const float* W, int ldw, float* gA, int lda,
                       bool acc) {
    if (M.n <= 0) return NB200_OK;
    if (M.n <= 0x7fffffff && goc_tc_ok(K, N, ldc, ldw, lda)) return tc_gemm(e, s, M, K, N, gC, ldc, W, ldw, 1, gA, lda, acc, nullptr, nullptr);
    return pfor(e, s, CAT_GEMM, M, K, DenseDgradK{gC, ldc, W, ldw, gA, lda, N, K, acc});
}
// gW[N, K] (ldw) += alpha * gC[M, N]^T (ldc) . A[M, K] (lda): the weight gradient of dense_fwd
inline int dense_wgrad(nb200_engine* e, cudaStream_t s, int64_t M, int N, int K, const float* gC, int ldc, const float* A, int lda, float* gW, int ldw,
                       float alpha = 1.0f) {
    if (M <= 0) return NB200_OK;
    int rc = NB200_OK;
    if (goc_wgrad(e, s, M, N, K, gC, ldc, A, lda, gW, ldw, alpha, &rc)) return rc;
    return pfor(e, s, CAT_GEMM, (M + WGRAD_ROWS - 1) / WGRAD_ROWS * N * K, DenseWgradK{gC, ldc, A, lda, gW, ldw, N, K, M, alpha});
}
}  // namespace
