// engine_common.cuh -- pieces shared by the model engines (engine.cu: PaiNN, schnet.cu: SchNet).
#pragma once
#include <cublas_v2.h>

#include <vector>

#include "painn_node.cuh"

// launch categories for the optional per-category CUDA-event timing (bench.py roofline leg)
enum { CAT_NBR = 0, CAT_FILTER, CAT_EMBED, CAT_GEMM, CAT_NODE, CAT_MSG_FWD, CAT_MSG_BWD, CAT_READOUT, CAT_FORCE, NCAT };

struct nb200_engine {
    cublasHandle_t blas;          // weight gradients of the GemNet-OC and SchNet training steps (goc_wgrad, gemnet_pf.cuh)
    bool timing = false;
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


// Linear layers on the wgmma 3xTF32 GEMM of gemm_tc.cu.
// Y[M,out] (ldy) = X[M,in] (ldx) . W[out,in]^T (ldw) (+ Y) (+ bias) ; optional act = silu(Y)   -- torch.nn.Linear forward
inline int linear_fwd(nb200_engine* e, cudaStream_t s, int M, int out, int in, const float* X, int ldx, const float* W, int ldw, float* Y,
                      int ldy, bool accumulate, const float* bias, float* act, int act_kind = NB_ACT_SILU) {
    Scope sc(e, s, CAT_GEMM, 1);
    return nb_gemm_tf32x3_ex(M, out, in, X, ldx, W, ldw, 0, Y, ldy, accumulate ? 1 : 0, bias, act, act_kind, s);
}
// gX[M,in] (ldgx) = gY[M,out] (ldgy) . W[out,in] (ldw)  (+ gX)                                   -- Linear backward w.r.t. input
inline int linear_bwd(nb200_engine* e, cudaStream_t s, int M, int out, int in, const float* gY, int ldgy, const float* W, int ldw, float* gX,
                      int ldgx, bool accumulate) {
    Scope sc(e, s, CAT_GEMM, 1);
    return nb200_gemm_tf32x3(M, in, out, gY, ldgy, W, ldw, 1, gX, ldgx, accumulate ? 1 : 0, nullptr, nullptr, s);
}

#define NB_TRY(expr)                  \
    do {                              \
        int _rc = (expr);             \
        if (_rc != NB200_OK) return _rc; \
    } while (0)

