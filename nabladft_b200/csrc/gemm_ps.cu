// gemm_ps.cu -- fp32-accurate dense layer C = A . op(W) for TALL problems (M >= ~2000 rows) on the pipeline of tc_pipe.cuh.
//
// Replaces the round-1 3xTF32 kernels of gemm_tc.cu where they were slowest: torch.nn.Linear / e3nn FullyConnectedNet layers applied to every
// atom pair or edge (QHNet weight generation [1e5 x 8320 x 128], qhnet/layers.py:191-203,376-459; GemNet-OC Dense layers [6e5 x 512 x 512],
// gemnet_oc/layers/base_layers.py; the per-Linear PaiNN / SchNet paths).  There the MMA issuer idled 70 % of the time waiting for producer
// warps that split the WEIGHT operand into TF32 hi / lo again for every 128-row slab.  Here
//   * the weight matrix is split ONCE per call into ready-made shared-memory tile images (k_prep_gemm, 128 KB per 128 x 128 tile) in a scratch
//     buffer, and streamed by single cp.async.bulk copies -- nobody splits weights inside the GEMM;
//   * the activation slab [64 rows x 128 k] is split once per CTA (K <= 128) or once per (N tile, K chunk);
//   * D[out feature, row] orientation: an epilogue thread owns one output feature and 32 rows (64 with two worker groups), so C stores are 128-byte coalesced per warp;
//   * the shared-memory staging tile decouples the epilogue of tile t from the MMAs of tile t + 1.
#include <map>
#include <mutex>

#include "tc_pipe.cuh"

namespace {

// W -> tiles [n_nt][KC] of 128 rows (output features) x 128 k, zero-padded; trans = 0: W[N][K] (ldw), trans = 1: W[K][N] (ldw)
__global__ void __launch_bounds__(256) k_prep_gemm(const float* __restrict__ W, int ldw, int trans, int N, int K, int KC, unsigned char* __restrict__ dst) {
    const int tile_i = blockIdx.x >> 2, st = blockIdx.x & 3;
    const int nt = tile_i / KC, kc_i = tile_i % KC;
    unsigned char* tile = dst + (size_t)tile_i * WTILE_BYTES;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int item = threadIdx.x + 256 * i;
        int kc, r;
        if (!trans) { kc = item & 7; r = item >> 3; } else { r = item & 127; kc = item >> 7; }
        const int kk = 32 * st + 4 * kc;            // k inside the tile
        const int n = nt * 128 + r, kg = kc_i * 128 + kk;
        float e[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool ok = n < N && kg + j < K;
            e[j] = !ok ? 0.f : !trans ? __ldg(W + (size_t)n * ldw + kg + j) : __ldg(W + (size_t)(kg + j) * ldw + n);
        }
        float4 hi, lo;
        split4(make_float4(e[0], e[1], e[2], e[3]), hi, lo);
        float* out_hi = reinterpret_cast<float*>(tile + (size_t)(kk / KSTAGE) * WST_BYTES + (size_t)((kk % KSTAGE) / 4) * WLBO) + r * 4;
        st4(out_hi, hi);
        st4(out_hi + (KSTAGE / 4) * WLBO / 4, lo);
    }
}

struct GemmParams {
    int M, N, K, KC, n_nt, tiles_per_cta;
    int spt;                      // 32-k stages per weight tile that carry data (K <= 96: fewer than 4)
    int epi; float epi_alpha;     // NB_EPI_* (common.cuh)
    int lm_batch;                 // 1: blockIdx.z = (l,m) row of an equivariant feature; weights per l, bias on lm = 0 only
    long long a_boff, c_boff, w_boff;
    const float* A; int lda;
    const unsigned char* wt;
    float* C; int ldc, accumulate;
    const float* bias;
    float* act; int act_kind;
    const int32_t* m_dev;         // optional row count in device memory (M is then the bound the grid is sized by)
};

// L (tc_pipe.cuh): OneGroup for K <= 128 and the lm path, TwoGroups for K > 128 (see gemm_ps_impl)
template <class L>
__global__ void __launch_bounds__(NTHREADS, CTAS_PER_SM) k_gemm_ps(const GemmParams P0) {
    extern __shared__ __align__(1024) unsigned char smem[];
    GemmParams P = P0;
    if (P.lm_batch) {  // o3.Linear: one (l,m) slice per blockIdx.z, W_l shared by the 2l + 1 slices of an order
        const int z = blockIdx.z, l = z >= 16 ? 4 : z >= 9 ? 3 : z >= 4 ? 2 : z >= 1 ? 1 : 0;
        P.A += (size_t)z * P.a_boff; P.C += (size_t)z * P.c_boff; P.wt += (size_t)l * P.w_boff;
        if (z > 0) P.bias = nullptr;
    }
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t_begin = blockIdx.y * P.tiles_per_cta, t_end = min(t_begin + P.tiles_per_cta, P.n_nt);
    if (t_begin >= t_end) return;
    if (P.m_dev) {  // a slab wholly beyond the device row count: the whole CTA leaves before any mbarrier exists or bulk copy is issued
        const int rows = min(P.M, *P.m_dev);
        if ((int)blockIdx.x * L::NT >= rows) return;
        P.M = rows;
    }
    const int n_it = t_end - t_begin, KC = P.KC, n_units = n_it * KC;
    Ctx<L> c = setup<L>(smem, tid);
    // unit u = (N tile t_begin + u / KC, K chunk u % KC).  K <= 128: the activation slab is written once and stays; else once per unit.
    auto flags_of = [&](int u) {
        const int kc = u % KC;
        return ((KC > 1 || u == 0) ? U_NEWX : 0) | (kc == 0 ? U_FIRST : 0) | (kc == KC - 1 ? U_LAST : 0) | ((KC > 1 || u == n_units - 1) ? U_XLAST : 0);
    };
    if (warp >= WARP_ISSUE) {
        run_issuer_t(c, n_units, flags_of, [&](int u) { return (t_begin + u / KC) * KC + u % KC; }, P.wt, P.spt);
    } else {
        const int M = P.M, m0 = blockIdx.x * L::NT;
        const int fl = 32 * (warp & 3) + lane, n0 = L::CPT * (warp >> 2);
        // epilogue warps [0, NEPI), loader warps [NWORK - NLOAD, NWORK): with one group every worker warp is both
        const bool isE = warp < L::NEPI, isL = warp >= NWORK - L::NLOAD;
        const int ltid = tid - 32 * (NWORK - L::NLOAD);
#pragma unroll 1
        for (int u = 0; u < n_units; ++u) {
            const int fg = flags_of(u), kc_i = u % KC;
            if (fg & U_NEWX) {
                if (isL)
                    load_x(c, ltid, [&](int r, int kc) {
                        const int k = kc_i * 128 + 4 * kc;
                        return (m0 + r < M && k < P.K) ? ldg4(P.A + (size_t)(m0 + r) * P.lda + k) : f4(0.f);
                    });
                else
                    ++c.xg;
            }
            if ((fg & U_LAST) && isE) {
                const int n = (t_begin + u / KC) * 128 + fl;
                drain(c, warp);
                const bool n_ok = n < P.N;
                const float b = (P.bias && n_ok) ? __ldg(P.bias + n) : 0.f;
                epi_chunks(c, warp, [&](int cb, float (&v)[16]) {
                    float* cp = P.C + (size_t)(m0 + n0 + 16 * cb) * P.ldc + n;
                    float t[16];
                    if (P.accumulate || P.epi == NB_EPI_RESIDUAL) {
#pragma unroll
                        for (int j = 0; j < 16; ++j) t[j] = (n_ok && m0 + n0 + 16 * cb + j < M) ? cp[(size_t)j * P.ldc] : 0.f;
                    }
                    if (P.epi != NB_EPI_PLAIN) {  // fused tails: activation in place, or (x + act(o)) * alpha over the layer input held in C
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (n_ok && m0 + n0 + 16 * cb + j < M) {
                                const float a = actf_(v[j] + b, P.act_kind);
                                cp[(size_t)j * P.ldc] = P.epi == NB_EPI_ACT ? a : (t[j] + a) * P.epi_alpha;
                            }
                        return;
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (n_ok && m0 + n0 + 16 * cb + j < M) {
                            const float o = v[j] + b + (P.accumulate ? t[j] : 0.f);
                            cp[(size_t)j * P.ldc] = o;
                            if (P.act) P.act[(size_t)(m0 + n0 + 16 * cb + j) * P.ldc + n] = actf_(o, P.act_kind);
                        }
                    }
                });
            }
        }
    }
}

// grow-only scratch for the prepared weights, one per (thread, stream): calls on one stream are ordered, so the buffer is reused safely
struct Scratch { void* p = nullptr; size_t bytes = 0; };
thread_local std::map<cudaStream_t, Scratch> g_scratch;

// Set-up shared by the entry points: `ws` (the prepared-weight buffer) becomes the stream's scratch, grown to `need` bytes, unless the caller
// passed one; the dynamic shared-memory limit of k_gemm_ps<L> is raised once per process and layout.
template <class L>
int gemm_ps_ready(void*& ws, size_t need, cudaStream_t s) {
    if (!ws) {
        Scratch& sc = g_scratch[s];
        if (sc.bytes < need) {
            if (sc.p) cudaFree(sc.p);
            if (cudaMalloc(&sc.p, need) != cudaSuccess) { sc = Scratch{}; return nb_check_launch(); }
            sc.bytes = need;
        }
        ws = sc.p;
    }
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(k_gemm_ps<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::SMEM_TOTAL) != cudaSuccess) return nb_check_launch();
        attr = true;
    }
    return NB200_OK;
}

}  // namespace

size_t nb_gemm_ps_ws_bytes(int N, int K) { return (size_t)((N + 127) / 128) * ((K + 127) / 128) * WTILE_BYTES; }

// worth it when the weight preparation is amortised over many row slabs
// (K = 32: the radial-basis layers of QHNet's convolution, [E, 32] x [32, 5376] -- one stage per tile, bound by the output write)
bool nb_gemm_ps_wanted(int M, int N, int K) { return M >= 2048 && N >= 64 && K >= 32 && K % 4 == 0; }

// `ws` (>= nb_gemm_ps_ws_bytes(N, K)) may be NULL: a per-stream grow-only scratch owned by this translation unit is used then.
static int gemm_ps_impl(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
                        const float* bias, float* act, int act_kind, void* ws, size_t ws_bytes, cudaStream_t s, int epi, float epi_alpha,
                        const int32_t* m_dev = nullptr) {
    if (!A || !B || !C || M < 0 || N <= 0 || K <= 0) return NB200_EINVAL;
    if (K % 4 || lda % 4 || ldc < N) return NB200_EUNSUPPORTED;
    if (M == 0) return NB200_OK;
    const int n_nt = (N + 127) / 128, KC = (K + 127) / 128;
    const size_t need = nb_gemm_ps_ws_bytes(N, K);
    if (ws && ws_bytes < need) return NB200_EINVAL;
    // K > 128: every (N tile, K chunk) needs a fresh activation operand.  With two worker groups, handing it over in K halves, the loaders
    // write the next operand while the epilogue group drains the finished tile and stores it, instead of after that.
    const bool two_groups = KC > 1;
    const int rc = two_groups ? gemm_ps_ready<TwoGroups>(ws, need, s) : gemm_ps_ready<OneGroup>(ws, need, s);
    if (rc != NB200_OK) return rc;
    k_prep_gemm<<<n_nt * KC * 4, 256, 0, s>>>(B, ldb, trans_b ? 1 : 0, N, K, KC, static_cast<unsigned char*>(ws));
    GemmParams P{};
    P.M = M; P.N = N; P.K = K; P.KC = KC; P.n_nt = n_nt; P.A = A; P.lda = lda; P.wt = static_cast<const unsigned char*>(ws);
    P.C = C; P.ldc = ldc; P.accumulate = accumulate; P.bias = bias; P.act = act; P.act_kind = act_kind;
    P.spt = KC == 1 ? (K + KSTAGE - 1) / KSTAGE : STAGES_PER_TILE;
    P.epi = epi; P.epi_alpha = epi_alpha;
    P.m_dev = m_dev;
    static_assert(OneGroup::NT == TwoGroups::NT, "one row tiling for both layouts");
    const int m_tiles = (M + OneGroup::NT - 1) / OneGroup::NT;
    int ny = 1;
    while (m_tiles * ny < nb_sm_count() && ny < n_nt) ++ny;  // few row slabs: split the N walk (the activation slab is re-staged per CTA)
    P.tiles_per_cta = (n_nt + ny - 1) / ny;
    dim3 grid(m_tiles, (n_nt + P.tiles_per_cta - 1) / P.tiles_per_cta);
    if (two_groups) k_gemm_ps<TwoGroups><<<grid, NTHREADS, TwoGroups::SMEM_TOTAL, s>>>(P);
    else k_gemm_ps<OneGroup><<<grid, NTHREADS, OneGroup::SMEM_TOTAL, s>>>(P);
    return nb_check_launch();
}

int nb_gemm_ps(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, int accumulate,
               const float* bias, float* act, int act_kind, void* ws, size_t ws_bytes, cudaStream_t s, const int32_t* m_dev) {
    return gemm_ps_impl(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, act_kind, ws, ws_bytes, s, NB_EPI_PLAIN, 1.0f, m_dev);
}

// Dense layer with a fused tail (GemNet-OC: Dense + ScaledSiLU in place; the (x + act(.)) / sqrt 2 tail of a ResidualLayer into x)
int nb_gemm_ps_epi(int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans_b, float* C, int ldc, const float* bias, int epi,
                   int act_kind, float alpha, cudaStream_t s) {
    if (epi != NB_EPI_ACT && epi != NB_EPI_RESIDUAL) return NB200_EINVAL;
    if (A == C) return NB200_EINVAL;  // rows of C are rewritten while other CTAs may still read A
    return gemm_ps_impl(M, N, K, A, lda, B, ldb, trans_b, C, ldc, 0, bias, nullptr, act_kind, nullptr, 0, s, epi, alpha);
}

extern "C" int nb200_gemm_tf32x3_epi(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb, int32_t trans_b,
                                     float* C, int32_t ldc, const float* bias, int32_t epi, int32_t act_kind, float alpha, void* stream) {
    return nb_gemm_ps_epi(M, N, K, A, lda, B, ldb, trans_b, C, ldc, bias, epi, act_kind, alpha, (cudaStream_t)stream);
}

// o3.Linear batched over the n_lm = 25 (l,m) rows of an equivariant feature (the call of nb_gemm_tf32x3_lm for tall inputs): slice z reads
// A + z K (row stride lda), writes C + z N (row stride ldc), uses W_l[l(z)] ([K][N], stride w_l_stride), bias on z = 0 only.
bool nb_gemm_ps_lm_wanted(int M, int N, int K) { return M >= 2048 && N >= 32 && K >= 32 && K % 4 == 0; }

int nb_gemm_ps_lm(int M, int N, int K, const float* A, int lda, const float* W_l, long long w_l_stride, float* C, int ldc, int accumulate,
                  const float* bias, int n_lm, cudaStream_t s) {
    if (!A || !W_l || !C || M < 0 || N <= 0 || K <= 0 || n_lm <= 0 || n_lm > 25) return NB200_EINVAL;
    if (K % 4 || lda % 4) return NB200_EUNSUPPORTED;
    if (M == 0) return NB200_OK;
    const int n_l = n_lm > 16 ? 5 : n_lm > 9 ? 4 : n_lm > 4 ? 3 : n_lm > 1 ? 2 : 1;
    const int n_nt = (N + 127) / 128, KC = (K + 127) / 128;
    const size_t per_w = nb_gemm_ps_ws_bytes(N, K), need = per_w * n_l;
    void* ws = nullptr;
    const int rc = gemm_ps_ready<OneGroup>(ws, need, s);
    if (rc != NB200_OK) return rc;
    for (int l = 0; l < n_l; ++l)
        k_prep_gemm<<<n_nt * KC * 4, 256, 0, s>>>(W_l + (size_t)l * w_l_stride, N, 1, N, K, KC, static_cast<unsigned char*>(ws) + (size_t)l * per_w);
    GemmParams P{};
    P.M = M; P.N = N; P.K = K; P.KC = KC; P.n_nt = n_nt; P.A = A; P.lda = lda; P.wt = static_cast<const unsigned char*>(ws);
    P.C = C; P.ldc = ldc; P.accumulate = accumulate; P.bias = bias; P.act = nullptr; P.act_kind = 0;
    P.spt = KC == 1 ? (K + KSTAGE - 1) / KSTAGE : STAGES_PER_TILE;
    P.lm_batch = 1; P.a_boff = K; P.c_boff = N; P.w_boff = (long long)per_w;
    P.tiles_per_cta = n_nt;
    dim3 grid((M + OneGroup::NT - 1) / OneGroup::NT, 1, n_lm);
    k_gemm_ps<OneGroup><<<grid, NTHREADS, OneGroup::SMEM_TOTAL, s>>>(P);
    return nb_check_launch();
}
