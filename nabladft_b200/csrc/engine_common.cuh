// engine_common.cuh -- pieces shared by the model engines (engine.cu: PaiNN, schnet.cu: SchNet).
#pragma once
#include <cublas_v2.h>

#include <vector>

#include "painn_node.cuh"

// launch categories for the optional per-category CUDA-event timing (bench.py roofline leg)
enum { CAT_NBR = 0, CAT_FILTER, CAT_EMBED, CAT_GEMM, CAT_NODE, CAT_MSG_FWD, CAT_MSG_BWD, CAT_READOUT, CAT_FORCE, NCAT };

struct nb200_engine {
    cublasHandle_t blas;
    bool timing = false;
    int gemm_backend = 1;         // 1 = wgmma 3xTF32 (gemm_tc.cu), 0 = cuBLAS SGEMM
    int node_backend = 1;         // PaiNN inference: 1 = fused per-layer node kernels (painn_fused.cu), 0 = one launch per Linear / elementwise op
    cudaStream_t side = nullptr;  // PaiNN training: weight-gradient ("leaf") launches run here, next to the backward chain on the caller's stream
    std::vector<cudaEvent_t> side_ev;
    int edge_bf16 = 0;            // PaiNN training: per-edge arrays (filter rows W, dW/dd, per-edge filter gradients) stored as bf16, fp32 arithmetic
    std::vector<cudaEvent_t> ev;  // pairs (start, stop)
    std::vector<int> cat;
    size_t n_used = 0;            // pairs in flight since the last read
    int64_t own_launches = 0;     // hand-written kernels launched since creation (cuBLAS not counted)
    void* session = nullptr;      // state kept between a training forward and its backward (gemnet_oc_train.inc); freed by session_free
    void (*session_free)(void*) = nullptr;
};

// RAII scope: counts own-kernel launches and, when timing is on, brackets them with events
// recorded on the launch stream.
struct Scope {
    nb200_engine* e;
    cudaStream_t s;
    size_t idx = (size_t)-1;
    Scope(nb200_engine* e_, cudaStream_t s_, int category, int own_kernels) : e(e_), s(s_) {
        e->own_launches += own_kernels;
        if (!e->timing) return;
        if (e->n_used * 2 + 2 > e->ev.size()) {
            cudaEvent_t a, b;
            if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return;
            e->ev.push_back(a); e->ev.push_back(b); e->cat.push_back(category);
        }
        idx = e->n_used++;
        e->cat[idx] = category;
        cudaEventRecord(e->ev[2 * idx], s);
    }
    ~Scope() {
        if (idx != (size_t)-1) cudaEventRecord(e->ev[2 * idx + 1], s);
    }
};


constexpr int64_t kAlign = 256;
constexpr int64_t kBlasWs = 32ll << 20;

struct Carver {
    char* base;
    int64_t off = 0;
    explicit Carver(void* p) : base(static_cast<char*>(p)) {}
    template <typename T>
    T* take(int64_t count) {
        off = (off + kAlign - 1) / kAlign * kAlign;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * (int64_t)sizeof(T);
        return p;
    }
};


// Y[M,out] (ldy) = X[M,in] (ldx) . W[out,in]^T (ldw) (+ Y) (+ bias) ; optional act = silu(Y)   -- torch.nn.Linear forward
inline int linear_fwd(nb200_engine* e, cudaStream_t s, int M, int out, int in, const float* X, int ldx, const float* W, int ldw, float* Y,
                      int ldy, bool accumulate, const float* bias, float* act, int act_kind = NB_ACT_SILU) {
    if (e->gemm_backend == 1) {
        Scope sc(e, s, CAT_GEMM, 1);
        return nb_gemm_tf32x3_ex(M, out, in, X, ldx, W, ldw, 0, Y, ldy, accumulate ? 1 : 0, bias, act, act_kind, s);
    }
    {
        Scope sc(e, s, CAT_GEMM, 0);
        const float alpha = 1.0f, beta = accumulate ? 1.0f : 0.0f;
        if (cublasSgemm(e->blas, CUBLAS_OP_T, CUBLAS_OP_N, out, M, in, &alpha, W, ldw, X, ldx, &beta, Y, ldy) != CUBLAS_STATUS_SUCCESS)
            return NB200_ECUDA;
    }
    if (bias || act) {
        if (!bias || ldy != out) return NB200_EINVAL;  // cuBLAS path: bias (+ optional activation) on dense rows
        Scope sc(e, s, CAT_NODE, 1);
        return nb_bias_act(Y, bias, act, M, out, act_kind, s);
    }
    return NB200_OK;
}
// gX[M,in] (ldgx) = gY[M,out] (ldgy) . W[out,in] (ldw)  (+ gX)                                   -- Linear backward w.r.t. input
inline int linear_bwd(nb200_engine* e, cudaStream_t s, int M, int out, int in, const float* gY, int ldgy, const float* W, int ldw, float* gX,
                      int ldgx, bool accumulate) {
    Scope sc(e, s, CAT_GEMM, e->gemm_backend == 1 ? 1 : 0);
    if (e->gemm_backend == 1) return nb200_gemm_tf32x3(M, in, out, gY, ldgy, W, ldw, 1, gX, ldgx, accumulate ? 1 : 0, nullptr, nullptr, s);
    const float alpha = 1.0f, beta = accumulate ? 1.0f : 0.0f;
    return cublasSgemm(e->blas, CUBLAS_OP_N, CUBLAS_OP_N, in, M, out, &alpha, W, ldw, gY, ldgy, &beta, gX, ldgx) == CUBLAS_STATUS_SUCCESS
               ? NB200_OK
               : NB200_ECUDA;
}

#define NB_TRY(expr)                  \
    do {                              \
        int _rc = (expr);             \
        if (_rc != NB200_OK) return _rc; \
    } while (0)
#define NB_BLAS(expr)                 \
    do {                              \
        if (!(expr)) return NB200_ECUDA; \
    } while (0)

