// filter.cu -- radial filter generation W[l][e][3F] (+ dW/dd) for every PaiNN layer.
//
// Replaces   spk: GaussianRBF(100, 5 A) -> filter_net Dense(100 -> 6*384) * CosineCutoff
//                 (config/model/painn.yaml:10-16; SURVEY.md A.2)
//            OC : RadialBasis = PolynomialEnvelope(5) * GaussianSmearing(d/rc)
//                 (nablaDFT/painn_pyg/layers.py:14-33,129-185) -> rbf_proj Linear(100 -> 384)
//                 per layer (painn_pyg/painn.py:464,479)
//   W_e  = s1(d) * sum_k phi_k(d) Wrbf[k,:] + s2(d) * b       spk: s1 = s2 = fcut ; OC: s1 = env, s2 = 1
//   dW_e = d/dd of the above (feeds the analytic force path; the reference gets it by autograd)
//
// The dense [E,100]x[100,384] GEMM is 16.4 GFLOP per layer at cfg 2 -- the largest FLOP
// term of the model -- but the Gaussians have width == spacing, so at a given distance only
// 16 consecutive centres contribute above 2.3e-11.  Edges are grouped by distance bin
// (counting sort, 3 tiny kernels); a CTA then owns (bin, split, layer), keeps the 16 band
// rows of Wrbf for its 4 channels in REGISTERS and streams its edges: 128 FMA per edge per
// thread instead of 800, no shared/L1 traffic for weights, output rows written once.  r2: with one record per undirected pair the kernel became
// FMA-bound (256 FFMA per edge-thread = 192 SM-cycles per edge and layer).
//
// Algorithmic HBM bytes: E*16 (geom) read + L*E*3F*4*(1 or 2) written  (cfg 2: 1.97 GB / 3.9 GB).
#include <cstdlib>

#include "common.cuh"

#define FLT_THREADS 96   // 3F/4 float4 channel groups for F = 128
#define FLT_CHUNK 32     // edges staged per phase
#define FLT_SPLIT 32     // CTAs per (bin, layer)
#define FLT_WSPLIT 48    // CTAs per bin in the weight-gradient kernels (one layer per launch; partial sums end in atomics)
#define SORT_THREADS 256
#define SORT_ITEMS 4


__device__ __forceinline__ int bin_of(float d, float xscale, float inv_dx, int n_bins) {
    int b = (int)floorf(d * xscale * inv_dx);
    return min(max(b, 0), n_bins - 1);
}

// `rev` != nullptr: only the CANONICAL edge of each undirected pair (e < rev[e]) is sorted, hence filtered -- a filter row depends on the
// distance only, so the opposite edge re-uses the row (painn_msg.cu reads row min(e, rev[e])).
__global__ void __launch_bounds__(SORT_THREADS) k_bin_hist(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                          float xscale, float inv_dx, int n_bins, int32_t* __restrict__ scr,
                                                          const int32_t* __restrict__ rev) {
    __shared__ int32_t sh[NB_NBINS_MAX];
    if (status[1] != 0) return;
    const int E = status[0];
    for (int t = threadIdx.x; t < n_bins; t += SORT_THREADS) sh[t] = 0;
    __syncthreads();
    for (int e = blockIdx.x * SORT_THREADS + threadIdx.x; e < E; e += gridDim.x * SORT_THREADS)
        if (!rev || rev[e] > e) atomicAdd(&sh[bin_of(geom[4 * (size_t)e + 3], xscale, inv_dx, n_bins)], 1);
    __syncthreads();
    for (int t = threadIdx.x; t < n_bins; t += SORT_THREADS)
        if (sh[t]) atomicAdd(&scr[SCR_START + 1 + t], sh[t]);  // counts land one slot up; scan turns them into starts
}

__global__ void k_bin_scan(int n_bins, int32_t* __restrict__ scr) {
    // one warp, n_bins <= 256: serial per-lane chunks + warp scan
    const int lane = threadIdx.x;
    const int chunk = (n_bins + 31) / 32;
    const int lo = min(lane * chunk, n_bins), hi = min(lo + chunk, n_bins);
    int s = 0;
    for (int i = lo; i < hi; ++i) s += scr[SCR_START + 1 + i];
    int v = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    int base = v - s;
    if (lane == 0) scr[SCR_START] = 0;
    for (int i = lo; i < hi; ++i) {
        const int c = scr[SCR_START + 1 + i];
        scr[SCR_CURSOR + i] = base;
        base += c;
        scr[SCR_START + 1 + i] = base;
    }
}

__global__ void __launch_bounds__(SORT_THREADS) k_bin_scatter(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                             float xscale, float inv_dx, int n_bins, int32_t* __restrict__ scr,
                                                             const int32_t* __restrict__ rev) {
    __shared__ int32_t scount[NB_NBINS_MAX];
    __shared__ int32_t sbase[NB_NBINS_MAX];
    if (status[1] != 0) return;
    const int E = status[0];
    const int tile = SORT_THREADS * SORT_ITEMS;
    for (int base = blockIdx.x * tile; base < E; base += gridDim.x * tile) {
        for (int t = threadIdx.x; t < n_bins; t += SORT_THREADS) scount[t] = 0;
        __syncthreads();
        int b[SORT_ITEMS], r[SORT_ITEMS];
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; ++k) {
            const int e = base + k * SORT_THREADS + threadIdx.x;
            b[k] = -1;
            if (e < E && (!rev || rev[e] > e)) {
                b[k] = bin_of(geom[4 * (size_t)e + 3], xscale, inv_dx, n_bins);
                r[k] = atomicAdd(&scount[b[k]], 1);
            }
        }
        __syncthreads();
        for (int t = threadIdx.x; t < n_bins; t += SORT_THREADS)
            if (scount[t]) sbase[t] = atomicAdd(&scr[SCR_CURSOR + t], scount[t]);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; ++k)
            if (b[k] >= 0) scr[SCR_PERM + sbase[b[k]] + r[k]] = base + k * SORT_THREADS + threadIdx.x;
        __syncthreads();
    }
}

// per-edge radial scalars
struct EdgeRad { float s1, ds1, s2, ds2; };

__device__ __forceinline__ EdgeRad radial_scalars(float d, int mode, float cutoff) {
    EdgeRad r;
    if (mode == NB200_RADIAL_SPK) {
        // schnetpack CosineCutoff: 0.5 (cos(pi d / rc) + 1) (d < rc)
        const float a = 3.14159265358979323846f / cutoff;
        const bool in = d < cutoff;
        r.s1 = in ? 0.5f * (cosf(d * a) + 1.0f) : 0.f;
        r.ds1 = in ? -0.5f * a * sinf(d * a) : 0.f;
        r.s2 = r.s1; r.ds2 = r.ds1;
    } else {
        // layers.py:23-33 PolynomialEnvelope(p=5): 1 - 21 x^5 + 35 x^6 - 15 x^7 for x < 1
        const float x = d * (1.0f / cutoff);
        const float x2 = x * x, x4 = x2 * x2, x5 = x4 * x;
        const bool in = x < 1.0f;
        r.s1 = in ? 1.0f + x5 * (-21.0f + x * (35.0f - 15.0f * x)) : 0.f;
        r.ds1 = in ? x4 * (-105.0f + x * (210.0f - 105.0f * x)) * (1.0f / cutoff) : 0.f;
        r.s2 = 1.0f; r.ds2 = 0.f;  // rbf_proj bias is added after the envelope (painn.py:479)
    }
    return r;
}

// WT = storage type of the rows (float, or nb_bf16: bf16 storage of the training path).  Layer l's rows start at the FLOAT offset
// l * layer_stride of `W` / `dW` whatever WT is (the engine carves fp32-sized arrays; bf16 rows use the first half of a layer's block).
template <bool WITH_DW, class WT>
__global__ void __launch_bounds__(FLT_THREADS) k_filter(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                       const int32_t* __restrict__ scr, const float* __restrict__ w_rbf,
                                                       const float* __restrict__ b_rbf, const float* __restrict__ offsets,
                                                       int n_rbf, int radial_mode, float cutoff, float coeff, float xscale,
                                                       size_t layer_stride, int row_stride, float* __restrict__ W, float* __restrict__ dW) {
    // rows of `row_stride` floats: 3F (W and dW/dd in two arrays) or 6F (ONE 3 KB record [W | dW/dd] per edge, dW = W + 3F)
    __shared__ __align__(16) float sphi[FLT_CHUNK][2 * NB_BAND + 4];
    __shared__ int32_t sedge[FLT_CHUNK];
    if (status[1] != 0) return;
    const int bin = blockIdx.x, split = blockIdx.y, layer = blockIdx.z;
    const int b0 = scr[SCR_START + bin], b1 = scr[SCR_START + bin + 1];
    const int cnt = b1 - b0;
    if (cnt == 0) return;
    const int per = (cnt + (int)gridDim.y - 1) / (int)gridDim.y;
    const int lo = b0 + split * per, hi = min(lo + per, b1);
    if (lo >= hi) return;
    const int k0 = min(max(bin - (NB_BAND / 2 - 1), 0), n_rbf - NB_BAND);
    const int c4 = threadIdx.x * 4;
    const int nf3 = 3 * NB_F;

    // band rows of this layer's weight for my 4 channels: registers for the whole CTA lifetime
    float4 wreg[NB_BAND];
    const float* wl = w_rbf + ((size_t)layer * n_rbf + k0) * nf3 + c4;
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) wreg[kk] = ldg4(wl + (size_t)kk * nf3);
    const float4 bias = ldg4(b_rbf + (size_t)layer * nf3 + c4);
    WT* Wl = reinterpret_cast<WT*>(W + (size_t)layer * layer_stride);
    WT* dWl = WITH_DW ? reinterpret_cast<WT*>(dW + (size_t)layer * layer_stride) : nullptr;

    for (int base = lo; base < hi; base += FLT_CHUNK) {
        const int nchunk = min(FLT_CHUNK, hi - base);
        if (threadIdx.x < nchunk) {
            const int e = scr[SCR_PERM + base + threadIdx.x];
            const float d = geom[4 * (size_t)e + 3];
            const EdgeRad r = radial_scalars(d, radial_mode, cutoff);
            const float x = d * xscale;
            float* row = sphi[threadIdx.x];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                const float t = x - __ldg(offsets + k0 + kk);
                const float p = expf(coeff * (t * t));  // torch.exp(coeff * pow(x - offset, 2))
                row[kk] = p;
                row[NB_BAND + kk] = p * (2.0f * coeff * xscale) * t;  // d phi / d d
            }
            row[2 * NB_BAND + 0] = r.s1; row[2 * NB_BAND + 1] = r.ds1;
            row[2 * NB_BAND + 2] = r.s2; row[2 * NB_BAND + 3] = r.ds2;
            sedge[threadIdx.x] = e;
        }
        __syncthreads();
        for (int t = 0; t < nchunk; ++t) {
            const float4* row4 = reinterpret_cast<const float4*>(sphi[t]);
            float4 acc0 = f4(0.f), acc1 = f4(0.f);
#pragma unroll
            for (int q4 = 0; q4 < NB_BAND / 4; ++q4) {
                const float4 p = row4[q4];
                fma4s(acc0, wreg[4 * q4 + 0], p.x); fma4s(acc0, wreg[4 * q4 + 1], p.y);
                fma4s(acc0, wreg[4 * q4 + 2], p.z); fma4s(acc0, wreg[4 * q4 + 3], p.w);
            }
            const float4 sc = row4[2 * NB_BAND / 4];
            const size_t off = (size_t)sedge[t] * row_stride + c4;
            float4 w = bias * sc.z;
            fma4s(w, acc0, sc.x);
            stw4(Wl + off, w);
            if (WITH_DW) {
#pragma unroll
                for (int q4 = 0; q4 < NB_BAND / 4; ++q4) {
                    const float4 p = row4[NB_BAND / 4 + q4];
                    fma4s(acc1, wreg[4 * q4 + 0], p.x); fma4s(acc1, wreg[4 * q4 + 1], p.y);
                    fma4s(acc1, wreg[4 * q4 + 2], p.z); fma4s(acc1, wreg[4 * q4 + 3], p.w);
                }
                float4 dw = bias * sc.w;
                fma4s(dw, acc0, sc.y);
                fma4s(dw, acc1, sc.x);
                stw4(dWl + off, dw);
            }
        }
        __syncthreads();
    }
}

// Training: gradient of the filter weights of ONE layer from the per-edge filter gradients gW[e][3F] (written by the message backward),
// over the same bin-sorted edge order: d w[k][c] += s1(d_e) phi_k(d_e) gW[e][c] for the 16 centres of the bin's band, d b[c] += s2(d_e) gW[e][c].
__global__ void __launch_bounds__(FLT_THREADS) k_filter_wgrad(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                             const int32_t* __restrict__ scr, const float* __restrict__ offsets, int n_rbf,
                                                             int radial_mode, float cutoff, float coeff, float xscale,
                                                             const float* __restrict__ gW, float* __restrict__ g_w, float* __restrict__ g_b) {
    __shared__ __align__(16) float sphi[FLT_CHUNK][NB_BAND + 4];
    __shared__ int32_t sedge[FLT_CHUNK];
    if (status[1] != 0) return;
    const int bin = blockIdx.x, split = blockIdx.y;
    const int b0 = scr[SCR_START + bin], b1 = scr[SCR_START + bin + 1];
    const int cnt = b1 - b0;
    if (cnt == 0) return;
    const int per = (cnt + FLT_WSPLIT - 1) / FLT_WSPLIT;
    const int lo = b0 + split * per, hi = min(lo + per, b1);
    if (lo >= hi) return;
    const int k0 = min(max(bin - (NB_BAND / 2 - 1), 0), n_rbf - NB_BAND);
    const int c4 = threadIdx.x * 4;
    const int nf3 = 3 * NB_F;
    float4 acc[NB_BAND];
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) acc[kk] = f4(0.f);
    float4 accb = f4(0.f);
    for (int base = lo; base < hi; base += FLT_CHUNK) {
        const int nchunk = min(FLT_CHUNK, hi - base);
        if (threadIdx.x < nchunk) {
            const int e = scr[SCR_PERM + base + threadIdx.x];
            const float d = geom[4 * (size_t)e + 3];
            const EdgeRad r = radial_scalars(d, radial_mode, cutoff);
            const float x = d * xscale;
            float* row = sphi[threadIdx.x];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                const float t = x - __ldg(offsets + k0 + kk);
                row[kk] = r.s1 * expf(coeff * (t * t));
            }
            row[NB_BAND] = r.s2;
            sedge[threadIdx.x] = e;
        }
        __syncthreads();
        // 8 gradient rows in flight per thread (r1 loaded one row per iteration: one L2 / HBM round trip per edge, 19 % of the HBM rate)
        for (int t0 = 0; t0 < nchunk; t0 += 8) {
            float4 g[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) g[u] = (t0 + u < nchunk) ? ldg4_stream(gW + (size_t)sedge[t0 + u] * nf3 + c4) : f4(0.f);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (t0 + u < nchunk) {
                    const float* row = sphi[t0 + u];
#pragma unroll
                    for (int kk = 0; kk < NB_BAND; ++kk) fma4s(acc[kk], g[u], row[kk]);
                    fma4s(accb, g[u], row[NB_BAND]);
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) {
        float* dst = g_w + (size_t)(k0 + kk) * nf3 + c4;
        atomicAdd(dst, acc[kk].x); atomicAdd(dst + 1, acc[kk].y); atomicAdd(dst + 2, acc[kk].z); atomicAdd(dst + 3, acc[kk].w);
    }
    atomicAdd(g_b + c4, accb.x); atomicAdd(g_b + c4 + 1, accb.y); atomicAdd(g_b + c4 + 2, accb.z); atomicAdd(g_b + c4 + 3, accb.w);
}

// Tangent of k_filter_wgrad along a position-space direction (painn_tangent.cu): with dd_e the tangent of the edge length,
//   d w^[k][c] = sum_e  gW^[e][c] s1 phi_k  +  (gW[e][c] dd_e) (s1' phi_k + s1 phi_k'),      d b^[c] = sum_e gW^ s2 + (gW dd) s2'
// t_gW = gW^ and gWd = gW dd are written by k_msg_bwd_tan.  `sign` (-1 for the force-loss term) scales what is added to g_w / g_b.
__global__ void __launch_bounds__(FLT_THREADS) k_filter_wgrad_tan(const float* __restrict__ geom, const int32_t* __restrict__ status,
                                                                 const int32_t* __restrict__ scr, const float* __restrict__ offsets, int n_rbf,
                                                                 int radial_mode, float cutoff, float coeff, float xscale,
                                                                 const float* __restrict__ t_gW, const float* __restrict__ gWd, float sign,
                                                                 float* __restrict__ g_w, float* __restrict__ g_b) {
    __shared__ __align__(16) float sphi[FLT_CHUNK][2 * NB_BAND + 4];
    __shared__ int32_t sedge[FLT_CHUNK];
    if (status[1] != 0) return;
    const int bin = blockIdx.x, split = blockIdx.y;
    const int b0 = scr[SCR_START + bin], b1 = scr[SCR_START + bin + 1];
    const int cnt = b1 - b0;
    if (cnt == 0) return;
    const int per = (cnt + FLT_WSPLIT - 1) / FLT_WSPLIT;
    const int lo = b0 + split * per, hi = min(lo + per, b1);
    if (lo >= hi) return;
    const int k0 = min(max(bin - (NB_BAND / 2 - 1), 0), n_rbf - NB_BAND);
    const int c4 = threadIdx.x * 4;
    const int nf3 = 3 * NB_F;
    float4 acc[NB_BAND];
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) acc[kk] = f4(0.f);
    float4 accb = f4(0.f);
    for (int base = lo; base < hi; base += FLT_CHUNK) {
        const int nchunk = min(FLT_CHUNK, hi - base);
        if (threadIdx.x < nchunk) {
            const int e = scr[SCR_PERM + base + threadIdx.x];
            const float d = geom[4 * (size_t)e + 3];
            const EdgeRad r = radial_scalars(d, radial_mode, cutoff);
            const float x = d * xscale;
            float* row = sphi[threadIdx.x];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                const float t = x - __ldg(offsets + k0 + kk);
                const float p = expf(coeff * (t * t));
                row[kk] = r.s1 * p;                                                    // s1 phi_k
                row[NB_BAND + kk] = r.ds1 * p + r.s1 * p * (2.0f * coeff * xscale) * t;  // d/dd (s1 phi_k)
            }
            row[2 * NB_BAND] = r.s2; row[2 * NB_BAND + 1] = r.ds2;
            sedge[threadIdx.x] = e;
        }
        __syncthreads();
        for (int t0 = 0; t0 < nchunk; t0 += 4) {  // 2 x 4 gradient rows in flight per thread
            float4 gh[4], gd[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const size_t off = (size_t)sedge[min(t0 + u, nchunk - 1)] * nf3 + c4;
                gh[u] = ldg4_stream(t_gW + off); gd[u] = ldg4_stream(gWd + off);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (t0 + u < nchunk) {
                    const float* row = sphi[t0 + u];
#pragma unroll
                    for (int kk = 0; kk < NB_BAND; ++kk) { fma4s(acc[kk], gh[u], row[kk]); fma4s(acc[kk], gd[u], row[NB_BAND + kk]); }
                    fma4s(accb, gh[u], row[2 * NB_BAND]); fma4s(accb, gd[u], row[2 * NB_BAND + 1]);
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int kk = 0; kk < NB_BAND; ++kk) {
        float* dst = g_w + (size_t)(k0 + kk) * nf3 + c4;
        atomicAdd(dst, sign * acc[kk].x); atomicAdd(dst + 1, sign * acc[kk].y); atomicAdd(dst + 2, sign * acc[kk].z); atomicAdd(dst + 3, sign * acc[kk].w);
    }
    atomicAdd(g_b + c4, sign * accb.x); atomicAdd(g_b + c4 + 1, sign * accb.y); atomicAdd(g_b + c4 + 2, sign * accb.z); atomicAdd(g_b + c4 + 3, sign * accb.w);
}


// r2: edge-balanced version of the two weight-gradient kernels above.  The (bin, 48 splits) grid ended every one of its 4800 three-warp CTAs
// in 68 x 96 float atomics -- 31 M atomics per launch, which (not the gradient rows) set the time per layer.  Here a CTA owns
// ~FW_TARGET consecutive edges of ONE bin in the sorted order (bins get CTAs in proportion to their edge count: no idle CTAs for the
// empty short-distance bins, no long tail for the crowded ones), its FW_GROUPS warp groups stream disjoint quarters of them with FW_ROWS
// gradient rows in flight per thread, the groups' band sums are combined through shared memory and flushed ONCE: ~12 x fewer atomics.
#define FW_GROUPS 4
#define FW_TARGET 768
#define FW_RING_BYTES 98304
// Gradient rows travel through a PER-THREAD cp.async ring in shared memory (thread = 4 channels of every row of its group): D rows (or row
// pairs) ahead of the arithmetic, no registers held, no synchronisation (a thread only ever touches its own 16 / 8 bytes of a slot).  First
// balanced version: 12 rows per thread in registers, consumed round by round, 12 warps
// per SM stalled on long_scoreboard + the group barrier.
template <int BYTES>
__device__ __forceinline__ void fw_cp_async(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    if (BYTES == 16) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
    else asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gmem_src) : "memory");
}
template <bool TAN, class GT>
__global__ void __launch_bounds__(FLT_THREADS* FW_GROUPS, 1)
    k_filter_wgrad_bal(const float* __restrict__ geom, const int32_t* __restrict__ status, const int32_t* __restrict__ scr,
                       const float* __restrict__ offsets, int n_rbf, int radial_mode, float cutoff, float coeff, float xscale,
                       const GT* __restrict__ gA, const GT* __restrict__ gB, float sign, float* __restrict__ g_w, float* __restrict__ g_b) {
    constexpr int NROW = (TAN ? 2 * NB_BAND : NB_BAND) + 4;
    constexpr int EL = 4 * (int)sizeof(GT);                                   // bytes of this thread's 4 channels of a row
    constexpr int NARR = TAN ? 2 : 1;
    constexpr int DEPTH_RAW = FW_RING_BYTES / (FLT_THREADS * FW_GROUPS * EL * NARR);
    constexpr int D = DEPTH_RAW >= 32 ? 32 : DEPTH_RAW >= 16 ? 16 : 8;       // rows in flight per thread (power of two)
    extern __shared__ __align__(16) unsigned char fw_ring[];                 // [array][slot][group][thread][EL]
    __shared__ __align__(16) float sphi[FW_GROUPS][FLT_CHUNK][NROW];
    __shared__ __align__(16) float4 sred[FW_GROUPS - 1][FLT_THREADS];
    __shared__ int32_t sparts[NB_NBINS_MAX];
    __shared__ int32_t s_item[3];  // bin, lo, hi
    if (status[1] != 0) return;
    const int tx = threadIdx.x, grp = threadIdx.y, flat = grp * FLT_THREADS + tx;
    // work item blockIdx.x -> (bin, part): bin b has ceil(count_b / FW_TARGET) parts
    for (int b = flat; b < n_rbf; b += FLT_THREADS * FW_GROUPS) sparts[b] = (scr[SCR_START + b + 1] - scr[SCR_START + b] + FW_TARGET - 1) / FW_TARGET;
    __syncthreads();
    if (flat == 0) {
        int item = blockIdx.x, bin = 0;
        while (bin < n_rbf && item >= sparts[bin]) { item -= sparts[bin]; ++bin; }
        s_item[0] = -1;
        if (bin < n_rbf) {
            const int b0 = scr[SCR_START + bin], b1 = scr[SCR_START + bin + 1];
            const int per = (b1 - b0 + sparts[bin] - 1) / sparts[bin];
            s_item[0] = bin; s_item[1] = b0 + item * per; s_item[2] = min(b0 + (item + 1) * per, b1);
        }
    }
    __syncthreads();
    const int bin = s_item[0];
    if (bin < 0) return;
    const int c_lo = s_item[1], c_hi = s_item[2];
    const int gper = (c_hi - c_lo + FW_GROUPS - 1) / FW_GROUPS;
    const int lo = c_lo + grp * gper, hi = min(lo + gper, c_hi);
    const int k0 = min(max(bin - (NB_BAND / 2 - 1), 0), n_rbf - NB_BAND);
    const int c4 = tx * 4;
    const int nf3 = 3 * NB_F;
    unsigned char* my = fw_ring + (size_t)(grp * FLT_THREADS + tx) * EL;
    constexpr size_t SLOT = (size_t)FW_GROUPS * FLT_THREADS * EL;
    auto issue = [&](int t) {  // row lo + t of this group's range -> slot t % D (own bytes only); always one commit
        if (lo + t < hi) {
            const size_t off = (size_t)__ldg(scr + SCR_PERM + lo + t) * nf3 + c4;
            fw_cp_async<EL>(my + (size_t)(t & (D - 1)) * SLOT, gA + off);
            if (TAN) fw_cp_async<EL>(my + (size_t)(D + (t & (D - 1))) * SLOT, gB + off);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll 1
    for (int d = 0; d < D; ++d) issue(d);
    float4 acc[NB_BAND + 1];  // [NB_BAND] = bias
#pragma unroll
    for (int kk = 0; kk <= NB_BAND; ++kk) acc[kk] = f4(0.f);
    for (int base = lo; base < hi; base += FLT_CHUNK) {
        const int nchunk = min(FLT_CHUNK, hi - base);
        if (tx < nchunk) {
            const int e = scr[SCR_PERM + base + tx];
            const float d = geom[4 * (size_t)e + 3];
            const EdgeRad r = radial_scalars(d, radial_mode, cutoff);
            const float x = d * xscale;
            float* row = sphi[grp][tx];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                const float t = x - __ldg(offsets + k0 + kk);
                const float p = expf(coeff * (t * t));
                row[kk] = r.s1 * p;                                                                  // s1 phi_k
                if (TAN) row[NB_BAND + kk] = r.ds1 * p + r.s1 * p * (2.0f * coeff * xscale) * t;     // d/dd (s1 phi_k)
            }
            if (TAN) { row[2 * NB_BAND] = r.s2; row[2 * NB_BAND + 1] = r.ds2; } else { row[NB_BAND] = r.s2; }
        }
        asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(FLT_THREADS) : "memory");
#pragma unroll 2
        for (int tt = 0; tt < nchunk; ++tt) {
            const int t = base - lo + tt;
            asm volatile("cp.async.wait_group %0;" ::"n"(D - 1) : "memory");  // row t (committed D - 1 groups before the newest) has landed
            const float4 gh = ldw4_plain(reinterpret_cast<const GT*>(my + (size_t)(t & (D - 1)) * SLOT));
            float4 gd = f4(0.f);
            if (TAN) gd = ldw4_plain(reinterpret_cast<const GT*>(my + (size_t)(D + (t & (D - 1))) * SLOT));
            issue(t + D);  // refill my bytes of the slot just read
            const float* row = sphi[grp][tt];
#pragma unroll
            for (int kk = 0; kk < NB_BAND; ++kk) {
                fma4s(acc[kk], gh, row[kk]);
                if (TAN) fma4s(acc[kk], gd, row[NB_BAND + kk]);
            }
            fma4s(acc[NB_BAND], gh, row[TAN ? 2 * NB_BAND : NB_BAND]);
            if (TAN) fma4s(acc[NB_BAND], gd, row[2 * NB_BAND + 1]);
        }
        asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(FLT_THREADS) : "memory");
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // combine the groups (fixed order: group 0 + 1 + 2 + 3), one flush per CTA
#pragma unroll
    for (int kk = 0; kk <= NB_BAND; ++kk) {
        if (grp > 0) sred[grp - 1][tx] = acc[kk];
        __syncthreads();
        if (grp == 0) {
            float4 v = acc[kk];
#pragma unroll
            for (int g = 0; g < FW_GROUPS - 1; ++g) { const float4 o = sred[g][tx]; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
            float* dst = kk < NB_BAND ? g_w + (size_t)(k0 + kk) * nf3 + c4 : g_b + c4;
            atomicAdd(dst, sign * v.x); atomicAdd(dst + 1, sign * v.y); atomicAdd(dst + 2, sign * v.z); atomicAdd(dst + 3, sign * v.w);
        }
        __syncthreads();
    }
}

template <bool TAN, class GT>
static int fw_launch(const float* geom, const int32_t* status, const int32_t* scr, const float* offsets, int n_rbf, int radial_mode, float cutoff,
                     float coeff, float xscale, const GT* gA, const GT* gB, float sign, float* g_w, float* g_b, int e_cap, cudaStream_t s) {
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(k_filter_wgrad_bal<TAN, GT>, cudaFuncAttributeMaxDynamicSharedMemorySize, FW_RING_BYTES) != cudaSuccess) return nb_check_launch();
        attr = true;
    }
    k_filter_wgrad_bal<TAN, GT><<<e_cap / FW_TARGET + n_rbf, dim3(FLT_THREADS, FW_GROUPS), FW_RING_BYTES, s>>>(geom, status, scr, offsets, n_rbf, radial_mode,
                                                                                                             cutoff, coeff, xscale, gA, gB, sign, g_w, g_b);
    return nb_check_launch();
}

static bool fw_balanced() {
    static const bool on = [] { const char* e = getenv("NB200_FWGRAD"); return !(e && e[0] == 'o'); }();  // NB200_FWGRAD=old: the (bin, 48 splits) kernels
    return on;
}

int nb_filter_wgrad_tan(const float* geom, const float* t_geom, const int32_t* status, const int32_t* sort_scratch, const float* rbf_offsets, int n_rbf,
                        int radial_mode, float cutoff, float rbf_coeff, float rbf_xscale, const float* t_gW, const float* gWd, float sign, float* g_w,
                        float* g_b, cudaStream_t s, int e_cap, int bf16) {
    (void)t_geom;  // dd_e is already folded into gWd by the message-backward tangent kernel
    if ((fw_balanced() || bf16) && e_cap > 0) {
        if (bf16)
            return fw_launch<true, nb_bf16>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale,
                                            reinterpret_cast<const nb_bf16*>(t_gW), reinterpret_cast<const nb_bf16*>(gWd), sign, g_w, g_b, e_cap, s);
        return fw_launch<true, float>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale, t_gW, gWd, sign, g_w, g_b, e_cap, s);
    }
    if (bf16) return NB200_EUNSUPPORTED;
    dim3 grid(n_rbf, FLT_WSPLIT, 1);
    k_filter_wgrad_tan<<<grid, FLT_THREADS, 0, s>>>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale, t_gW, gWd,
                                                   sign, g_w, g_b);
    return nb_check_launch();
}

// g_w [K][3F] and g_b [3F] of this layer must be zeroed by the caller; `sort_scratch` is the one the forward filter call left behind
int nb_filter_wgrad(const float* geom, const int32_t* status, const int32_t* sort_scratch, const float* rbf_offsets, int n_rbf, int radial_mode,
                    float cutoff, float rbf_coeff, float rbf_xscale, const float* gW, float* g_w, float* g_b, cudaStream_t s, int e_cap, int bf16) {
    if ((fw_balanced() || bf16) && e_cap > 0) {
        if (bf16)
            return fw_launch<false, nb_bf16>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale,
                                             reinterpret_cast<const nb_bf16*>(gW), nullptr, 1.0f, g_w, g_b, e_cap, s);
        return fw_launch<false, float>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale, gW,
                                       static_cast<const float*>(nullptr), 1.0f, g_w, g_b, e_cap, s);
    }
    if (bf16) return NB200_EUNSUPPORTED;
    dim3 grid(n_rbf, FLT_WSPLIT, 1);
    k_filter_wgrad<<<grid, FLT_THREADS, 0, s>>>(geom, status, sort_scratch, rbf_offsets, n_rbf, radial_mode, cutoff, rbf_coeff, rbf_xscale, gW, g_w, g_b);
    return nb_check_launch();
}

// counting sort of the edges by distance bin: scratch = [cursor | bin_start | perm] (common.cuh SCR_*)
int nb_bin_sort(const float* geom, const int32_t* status, float xscale, float inv_dx, int n_bins, int32_t* scratch, cudaStream_t s,
                const int32_t* rev) {
    if (cudaMemsetAsync(scratch, 0, SCR_PERM * sizeof(int32_t), s) != cudaSuccess) return nb_check_launch();
    k_bin_hist<<<296, SORT_THREADS, 0, s>>>(geom, status, xscale, inv_dx, n_bins, scratch, rev);
    k_bin_scan<<<1, 32, 0, s>>>(n_bins, scratch);
    k_bin_scatter<<<296, SORT_THREADS, 0, s>>>(geom, status, xscale, inv_dx, n_bins, scratch, rev);
    return nb_check_launch();
}

// `rev` (optional): filter only the canonical edge of every undirected pair; `interleave`: one [W | dW/dd] record of 6F floats per edge in
// `W` (dW ignored, must be non-null to request the derivative)
int nb_painn_filter_ex(const float* geom, const int32_t* status, int32_t e_stride, const float* w_rbf, const float* b_rbf, int32_t n_layers,
                       int32_t n_rbf, int32_t n_feat, int32_t radial_mode, float cutoff, const float* rbf_offsets, float rbf_coeff, float rbf_xscale,
                       float* W, float* dW, int32_t* sort_scratch, const int32_t* rev, int interleave, cudaStream_t s, int bf16) {
    if (!geom || !status || !w_rbf || !b_rbf || !rbf_offsets || !W || !sort_scratch) return NB200_EINVAL;
    if (bf16 && (!dW || interleave)) return NB200_EUNSUPPORTED;  // bf16 rows: the training layout only (W and dW/dd in two arrays)
    if (n_feat != NB_F || n_rbf < NB_BAND || n_rbf > NB_NBINS_MAX) return NB200_EUNSUPPORTED;
    if (radial_mode != NB200_RADIAL_SPK && radial_mode != NB200_RADIAL_OC) return NB200_EUNSUPPORTED;
    if (n_layers <= 0 || e_stride < 0 || (interleave && !dW)) return NB200_EINVAL;
    // band truncation is valid only when the Gaussian width equals the centre spacing:
    // dropped terms are <= exp(coeff * (7 dx)^2); require that below 1e-10.
    const float dx = (cutoff * rbf_xscale) / (float)(n_rbf - 1);
    if (!(rbf_coeff < 0.f) || rbf_coeff * (7.0f * dx) * (7.0f * dx) > -23.0f) return NB200_EUNSUPPORTED;
    if (int rc = nb_bin_sort(geom, status, rbf_xscale, 1.0f / dx, n_rbf, sort_scratch, s, rev)) return rc;
    static const int split = [] { const char* e = getenv("NB200_FLT_SPLIT"); return e ? atoi(e) : FLT_SPLIT; }();  // CTAs per (bin, layer)
    dim3 grid(n_rbf, split, n_layers);
    const int row_stride = interleave ? 6 * NB_F : 3 * NB_F;
    const size_t layer_stride = (size_t)e_stride * row_stride;
    if (bf16)
        k_filter<true, nb_bf16><<<grid, FLT_THREADS, 0, s>>>(geom, status, sort_scratch, w_rbf, b_rbf, rbf_offsets, n_rbf, radial_mode, cutoff,
                                                           rbf_coeff, rbf_xscale, layer_stride, row_stride, W, dW);
    else if (dW)
        k_filter<true, float><<<grid, FLT_THREADS, 0, s>>>(geom, status, sort_scratch, w_rbf, b_rbf, rbf_offsets, n_rbf, radial_mode, cutoff,
                                                         rbf_coeff, rbf_xscale, layer_stride, row_stride, W, interleave ? W + 3 * NB_F : dW);
    else
        k_filter<false, float><<<grid, FLT_THREADS, 0, s>>>(geom, status, sort_scratch, w_rbf, b_rbf, rbf_offsets, n_rbf, radial_mode, cutoff,
                                                          rbf_coeff, rbf_xscale, layer_stride, row_stride, W, dW);
    return nb_check_launch();
}

extern "C" int nb200_painn_filter(const float* geom, const int32_t* status, int32_t e_stride, const float* w_rbf,
                                  const float* b_rbf, int32_t n_layers, int32_t n_rbf, int32_t n_feat, int32_t radial_mode,
                                  float cutoff, const float* rbf_offsets, float rbf_coeff, float rbf_xscale, float* W, float* dW,
                                  int32_t* sort_scratch, void* stream) {
    return nb_painn_filter_ex(geom, status, e_stride, w_rbf, b_rbf, n_layers, n_rbf, n_feat, radial_mode, cutoff, rbf_offsets, rbf_coeff, rbf_xscale, W,
                              dW, sort_scratch, nullptr, 0, (cudaStream_t)stream, 0);
}
