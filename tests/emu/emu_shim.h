// emu_shim.h -- host stand-ins so that nabladft_b200/csrc/gemnet_oc.cu compiles as plain C++ (g++ -x c++ -DNB_EMU).
// TEST INFRASTRUCTURE ONLY: lets the CPU suite run every GemNet-OC functor serially against the oracle when no GPU is available.
// Nothing in nabladft_b200/ loads the resulting library; the product path is libnabla_b200.so on a GPU and fails loudly without it.
#pragma once
#include <stdint.h>

#include <cmath>
#include <cstdlib>
#include <cstring>

#include "../../include/nabla_b200.h"

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(x)
typedef void* cudaStream_t;
struct alignas(16) float4 { float x, y, z, w; };  // functors read 16-byte groups of 256-byte aligned rows (MulRbfRowsK)
struct nb200_engine {
    int64_t own_launches = 0;
    void* session = nullptr;
    void (*session_free)(void*) = nullptr;
};
enum { CAT_NBR = 0, CAT_FILTER, CAT_EMBED, CAT_GEMM, CAT_NODE, CAT_MSG_FWD, CAT_MSG_BWD, CAT_READOUT, CAT_FORCE, NCAT };
template <class T>
inline T __ldg(const T* p) { return *p; }
inline float atomicAdd(float* p, float v) {
    float old;
#pragma omp atomic capture
    { old = *p; *p += v; }
    return old;
}
// every functor owns its output element and only reads shared inputs, so the loop may run in parallel (which also checks exactly that)
template <class F>
inline int pfor(nb200_engine* e, cudaStream_t, int, int64_t n, const F& f) {
    if (e) e->own_launches++;
#pragma omp parallel for schedule(dynamic, 512)
    for (int64_t i = 0; i < n; i++) f(i);
    return NB200_OK;
}
static nb200_engine g_emu_engine;
extern "C" __attribute__((used, weak)) int nb200_engine_create(nb200_engine** out) { *out = &g_emu_engine; return NB200_OK; }
extern "C" __attribute__((used, weak)) int nb200_engine_destroy(nb200_engine*) { return NB200_OK; }
inline int scan_excl(nb200_engine*, cudaStream_t, const int32_t* in, int32_t n, int32_t* out) {
    int64_t run = 0;
    for (int32_t i = 0; i < n; i++) { out[i] = (int32_t)run; run += in[i]; }
    out[n] = (int32_t)run;
    return NB200_OK;
}
inline int goc_memset(void* p, int v, size_t bytes, cudaStream_t) { memset(p, v, bytes); return NB200_OK; }
inline int goc_d2h_sync(void* dst, const void* src, size_t bytes, cudaStream_t) { memcpy(dst, src, bytes); return NB200_OK; }
inline int goc_d2d(void* dst, const void* src, size_t bytes, cudaStream_t) { memcpy(dst, src, bytes); return NB200_OK; }
// NB200_EMU_LIBGEMM=1: take the SAME dispatch decisions as the device build and run reference loops with the exact interface semantics of the
// library GEMMs (nb_gemm_tf32x3_ex: strides, trans_b, accumulate, bias; cuBLAS SGEMM as called by goc_wgrad).  This checks the ARGUMENTS the
// engines pass to those libraries -- the part of the device path that the functor fallback never exercises.
inline bool emu_libgemm() {
    static const bool on = [] { const char* e = getenv("NB200_EMU_LIBGEMM"); return e && e[0] == '1'; }();
    return on;
}
inline bool goc_tc_ok(int N, int K, int lda, int ldw, int ldc) {
    return emu_libgemm() && N % 64 == 0 && K % 32 == 0 && lda % 4 == 0 && ldw % 4 == 0 && ldc % 4 == 0;
}
// C[M,N] (ldc) = A[M,K] (lda) . op(B) (+ C if accumulate) (+ bias[N]);  op(B) = B[N,K]^T (ldb, trans_b = 0) | B[K,N] (ldb, trans_b = 1)
inline int emu_ref_gemm(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate, const float* bias) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)M * N; i++) {
        const int64_t r = i / N; const int n = (int)(i % N);
        double s = 0.0;
        for (int k = 0; k < K; k++) s += (double)A[r * lda + k] * (trans_b ? B[(int64_t)k * ldb + n] : B[(int64_t)n * ldb + k]);
        C[r * ldc + n] = (float)(s + (accumulate ? C[r * ldc + n] : 0.0f) + (bias ? bias[n] : 0.0f));
    }
    return NB200_OK;
}
inline int goc_tc_gemm_ex(nb200_engine*, cudaStream_t, int M, int N, int K, const float* A, int lda, const float* W, int ldw, int trans_w, float* C, int ldc,
                          int accumulate, const float* bias) {
    return emu_ref_gemm(M, N, K, A, lda, W, ldw, trans_w, C, ldc, accumulate, bias);
}
// guard zones behind every carved sub-buffer (see Carve in gemnet_pf.cuh)
#include <vector>
#define NB_EMU_GUARD_BYTES 1024
static std::vector<unsigned char*> g_emu_guards;
inline void emu_guard_add(char* p) {
    memset(p, 0xA5, NB_EMU_GUARD_BYTES);
    g_emu_guards.push_back(reinterpret_cast<unsigned char*>(p));
}
// number of guard zones that were overwritten since the last call (0 = clean); forgets the zones
extern "C" __attribute__((used, weak)) int nb200_emu_check_guards() {
    int bad = 0;
    for (unsigned char* g : g_emu_guards)
        for (int k = 0; k < NB_EMU_GUARD_BYTES; k++)
            if (g[k] != 0xA5) { bad++; break; }
    const int n = (int)g_emu_guards.size();
    g_emu_guards.clear();
    return bad ? bad : -n;  // > 0: corrupted zones; <= 0: minus the number of intact zones checked
}
// cublasSgemm(OP_N, OP_T, in, out, M, alpha, X, ldx, gY, ldgy, beta = 1, dW, lddw) in row-major words: dW[out, in] += alpha gY^T X
inline bool goc_wgrad(nb200_engine*, cudaStream_t, int64_t M, int out, int in, const float* gY, int ldgy, const float* X, int ldx, float* dW, int lddw, float alpha,
                      int* rc) {
    if (!emu_libgemm() || M <= 0 || out <= 0 || in <= 0) return false;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)out * in; i++) {
        const int o = (int)(i / in), k = (int)(i % in);
        double s = 0.0;
        for (int64_t r = 0; r < M; r++) s += (double)gY[r * ldgy + o] * X[r * ldx + k];
        dW[(int64_t)o * lddw + k] += (float)(alpha * s);
    }
    *rc = NB200_OK;
    return true;
}
#define NB_TRY(expr)                     \
    do {                                 \
        int _rc = (expr);                \
        if (_rc != NB200_OK) return _rc; \
    } while (0)
