// common.cuh -- shared device helpers for the nabla_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nabla_b200.h"

#define NB_F 128          // hidden size of every SchNet/PaiNN config in the reference
#define NB_BAND 16        // Gaussian band width evaluated per edge (centres bin-7 .. bin+8)
#define NB_NBINS_MAX 256  // distance bins used to group edges for the filter kernel

// edge-sort scratch layout (int32): [0,256) cursor  [256,513) bin_start  [768, 768+E) perm
#define SCR_CURSOR 0
#define SCR_START 256
#define SCR_PERM 768

extern thread_local int g_nb200_last_cuda_error;

// streaming multiprocessors of the current device (queried once per process): grid sizing of the persistent / grid-stride launches
static inline int nb_sm_count() {
    static const int n = [] { int dev = 0, v = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev); return v > 0 ? v : 132; }();
    return n;
}

static inline int nb_check_launch() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        g_nb200_last_cuda_error = (int)e;
        return NB200_ECUDA;
    }
    return NB200_OK;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
// streaming load: read once, do not pollute L1
__device__ __forceinline__ float4 ldg4_stream(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4_stream(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

// ---- storage types of the per-edge arrays (filter rows W, dW/dd and the per-edge filter gradients): fp32, or bf16 storage with fp32
// arithmetic (BASELINE configs[2] "bf16": nb200_engine_set_edge_storage).  `nb_bf16` = 2 bytes, round-to-nearest-even on store.
typedef unsigned short nb_bf16;
__device__ __forceinline__ float4 bf16x4_to_f4(uint2 v) {
    return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xffff0000u));
}
__device__ __forceinline__ uint2 f4_to_bf16x4(float4 v) {
    uint2 r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r.x) : "f"(v.y), "f"(v.x));  // low half = second operand
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r.y) : "f"(v.w), "f"(v.z));
    return r;
}
// 4 consecutive elements: global read-only / plain (shared or global) / streaming load, plain / streaming store
__device__ __forceinline__ float4 ldw4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ldw4(const nb_bf16* p) { return bf16x4_to_f4(__ldg(reinterpret_cast<const uint2*>(p))); }
__device__ __forceinline__ float4 ldw4_plain(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ldw4_plain(const nb_bf16* p) { return bf16x4_to_f4(*reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ float4 ldw4_stream(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 ldw4_stream(const nb_bf16* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return bf16x4_to_f4(r);
}
__device__ __forceinline__ void stw4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void stw4(nb_bf16* p, float4 v) { *reinterpret_cast<uint2*>(p) = f4_to_bf16x4(v); }
__device__ __forceinline__ void stw4_stream(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void stw4_stream(nb_bf16* p, float4 v) {
    const uint2 r = f4_to_bf16x4(v);
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(r.x), "r"(r.y) : "memory");
}

__device__ __forceinline__ float4 f4(float a) { return make_float4(a, a, a, a); }
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 operator*(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 operator*(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ void fma4(float4& acc, float4 a, float4 b) {
    acc.x = fmaf(a.x, b.x, acc.x); acc.y = fmaf(a.y, b.y, acc.y); acc.z = fmaf(a.z, b.z, acc.z); acc.w = fmaf(a.w, b.w, acc.w);
}
__device__ __forceinline__ void fma4s(float4& acc, float4 a, float s) {
    acc.x = fmaf(a.x, s, acc.x); acc.y = fmaf(a.y, s, acc.y); acc.z = fmaf(a.z, s, acc.z); acc.w = fmaf(a.w, s, acc.w);
}
__device__ __forceinline__ float hsum4(float4 a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// accurate (non-fast-math) SiLU and derivative; expf is the full-precision CUDA routine
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x * sigmoidf_(x); }
__device__ __forceinline__ float dsiluf_(float x) {
    float s = sigmoidf_(x);
    return s * (1.0f + x * (1.0f - s));
}

// activation kinds fused into GEMM epilogues / bias kernels
#define NB_ACT_SILU 0  // PaiNN (painn_pyg/painn.py:461,522; schnetpack F.silu)
#define NB_ACT_SSP 1   // SchNet shifted softplus: softplus(x) - ln 2 (schnetpack.nn.activations.shifted_softplus)
#define NB_ACT_SSP_N 2 // e3nn FullyConnectedNet normalize2mom(ssp): 1.8782046685 * ssp(x)  (qhnet/layers.py:191-203)
#define NB_ACT_SSILU 3 // GemNet-OC ScaledSiLU: silu(x) / 0.6  (gemnet_oc/layers/base_layers.py:66-75); same expression as gemnet_oc_kernels.cuh::ssilu
__device__ __forceinline__ float sspf_(float x) {
    // softplus with torch's threshold-20 linearisation, accurate log1p/exp
    const float sp = x > 20.0f ? x : log1pf(expf(x));
    return sp - 0.69314718055994530942f;
}
__device__ __forceinline__ float actf_(float x, int kind) {
    return kind == NB_ACT_SSP ? sspf_(x) : kind == NB_ACT_SSP_N ? 1.8782046685f * sspf_(x) : kind == NB_ACT_SSILU ? x / (1.0f + expf(-x)) * (1.0f / 0.6f) : siluf_(x);
}
// derivative w.r.t. the pre-activation: silu' or ssp' (= sigmoid)
__device__ __forceinline__ float dactf_(float x, int kind) { return kind == NB_ACT_SSP ? sigmoidf_(x) : dsiluf_(x); }

int nb_gemm_tf32x3_ex(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
                      const float* bias, float* act, int act_kind, cudaStream_t s);
int nb_bin_sort(const float* geom, const int32_t* status, float xscale, float inv_dx, int n_bins, int32_t* scratch, cudaStream_t s,
                const int32_t* rev = nullptr);
int nb_painn_filter_ex(const float* geom, const int32_t* status, int32_t e_stride, const float* w_rbf, const float* b_rbf, int32_t n_layers,
                       int32_t n_rbf, int32_t n_feat, int32_t radial_mode, float cutoff, const float* rbf_offsets, float rbf_coeff, float rbf_xscale,
                       float* W, float* dW, int32_t* sort_scratch, const int32_t* rev, int interleave, cudaStream_t s, int bf16 = 0);
int nb_painn_msg_fwd_ex(const float* xh, const float* xh_bias, const float* q, const float* mu, const float* W, int w_stride, const int32_t* rev,
                        const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, float* q_out, float* mu_out, cudaStream_t s, int bf16 = 0);
int nb_painn_msg_bwd_ex(const float* xh, const float* xh_bias, const float* mu, const float* W, const float* dW, int w_stride, const int32_t* rev,
                        const float* geom, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q, const float* g_mu,
                        float* g_xh, float* g_mu_in, float* egrad, cudaStream_t s, int bf16 = 0);
bool nb_gemm_ps_wanted(int M, int N, int K);
size_t nb_gemm_ps_ws_bytes(int N, int K);
int nb_gemm_ps(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
               const float* bias, float* act, int act_kind, void* ws, size_t ws_bytes, cudaStream_t s);
// epilogue forms of the pre-split-weight GEMM: 0 C = o (+ optional activation copy), 1 C = act(o) (Dense + activation, no pre-activation kept),
// 2 C = (C + act(o)) * alpha (tail of a residual layer: C holds the layer input x)
enum { NB_EPI_PLAIN = 0, NB_EPI_ACT = 1, NB_EPI_RESIDUAL = 2 };
int nb_gemm_ps_epi(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, const float* bias, int epi,
                   int act_kind, float alpha, cudaStream_t s);
bool nb_gemm_ps_lm_wanted(int M, int N, int K);
int nb_gemm_ps_lm(int M, int N, int K, const float* A, int lda, const float* W_l, long long w_l_stride, float* C, int ldc, int accumulate,
                  const float* bias, int n_lm, cudaStream_t s);
int nb_gemm_tf32x3_lm(int M, int N, int K, const float* A, int lda, const float* W_l, long long w_l_stride, float* C, int ldc, int accumulate,
                      const float* bias, int n_lm, cudaStream_t s);
bool nb_wgrad_tc_ok(int M, int out, int in, const float* G0, int ldg, const float* X0, int ldx, const float* dW, int lddw);
int nb_wgrad_tc(int M, int out, int in, const float* G0, const float* X0, const float* G1, const float* X1, int ldg, int ldx, float* dW, int lddw,
                float alpha, float* dbias, float bias_alpha, int bias_term, const float* row_scale, int rs_div, cudaStream_t s);
int nb_wgrad_tc3(int M, int out, int in, const float* g, const float* tg, int ldg, const float* x, const float* tx, int ldx, float* dW, int lddw,
                 float* dbias, const float* row_scale, int rs_div, cudaStream_t s);
