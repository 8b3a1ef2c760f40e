// tc_pipe.cuh -- the warp-specialised wgmma pipeline shared by the fused PaiNN node kernels (painn_fused.cu) and the pre-split-weight GEMM
// (gemm_ps.cu): weight tiles as ready-made TF32 hi / lo shared-memory images streamed by cp.async.bulk through an mbarrier ring, the
// activation operand X written by worker warps (loader functors or epilogue registers), one MMA warpgroup (3xTF32: a correction and a main
// accumulator in registers), a shared-memory staging tile of the summed accumulators, epilogues in rolled 16-column chunks.
// D[feature, row] = W[feature, k] . X[row, k]^T: features on the staging rows, rows (atoms / edges / pairs) on its columns.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace {


constexpr int F = NB_F;
// CTA = NT atoms, 8 worker warps, two MMA warpgroups (features [0, 64) and [64, 128) of a weight tile) whose first thread also issues the
// weight copies (a separate producer warp made 17 warps, and ptxas then capped the registers at 96); 3 ring stages of 32 k.  An MMA
// warpgroup holds its 64 features x NT atoms three times (correction + two alternating main accumulators: 96 fp32 registers per thread
// at NT = 64; one warpgroup for all 128 features spilled), and the staging tile the epilogues read lives in shared memory next to the hi / lo activation operand and
// the weight ring: 65 + 96 + 34 KB at NT = 64 (NT = 128 would not fit the 227 KB of an SM).
constexpr int NT = 64, KSTAGE = 32, W_STAGES = 3, NWORK = 8, CTAS_PER_SM = 1;
constexpr int XLBO = NT * 16 + 16;         // bytes between 16-byte k-chunks of X (padded: the 8 chunk writers of a row hit 8 bank groups)
constexpr int XLBOF = XLBO / 4;
constexpr int X_BYTES = 32 * XLBO;         // one of hi / lo, K = 128
constexpr int WLBO = 128 * 16;             // weight stages are written by the bulk-copy engine: no padding needed
constexpr int WST_BYTES = 2 * (KSTAGE / 4) * WLBO;  // one ring stage: [hi | lo] x KSTAGE/4 chunks x 128 rows x 16 B
constexpr int STAGES_PER_TILE = 128 / KSTAGE;
constexpr int WTILE_BYTES = STAGES_PER_TILE * WST_BYTES;  // 128 rows x 128 k, hi + lo = 128 KB
constexpr int SROW = NT + 4;               // staging row stride (floats): the 16-byte reads of 8 consecutive feature rows hit 8 bank groups
constexpr int STAGE_BYTES = 128 * SROW * 4;
constexpr int SMEM_BARS = 2 * X_BYTES + W_STAGES * WST_BYTES + STAGE_BYTES;
constexpr int SMEM_TOTAL = SMEM_BARS + 256;
static_assert(SMEM_TOTAL <= 227 * 1024, "shared memory of one CTA");
// Worker warps.  Default: all NWORK warps load operands AND run epilogues, in program order.  NF_TWO_GROUPS: warps [0, NEPI) only drain /
// run epilogues / write chained operands, warps [NEPI, NEPI + NLOAD) only run the loader functors and therefore run AHEAD of the epilogues
// (their global loads overlap epilogue work and MMAs); the groups meet at mbarriers (operand ready / free, and `dep` for data handed over
// through global memory).
#ifdef NF_TWO_GROUPS
constexpr int NEPI = NWORK / 2, NLOAD = NWORK / 2;
#else
constexpr int NEPI = NWORK, NLOAD = NWORK;
#endif
constexpr int CPT = NT / (NEPI / 4);       // staged columns (atoms) per epilogue thread (4 feature groups of 32 x NEPI/4 column parts)
constexpr int RPT = NT / NLOAD;            // operand rows per loader thread
constexpr int WARP_ISSUE = NWORK;          // first warp of the two MMA warpgroups (warpgroups start at a multiple of 4 warps)
constexpr int NTHREADS = 32 * (NWORK + 8);
static_assert(NWORK % 4 == 0, "the MMA warpgroups must start on a warpgroup boundary");
enum { U_NEWX = 1, U_FIRST = 2, U_LAST = 4, U_XLAST = 8 };
#ifdef NF_PROF
// role timing (clock64, summed over CTAs): 0 issuer total, 1 issuer waits X, 2 issuer waits staging, 3 issuer waits W ring,
// 4 worker(thread 0) total, 5 worker waits accumulator, 6 worker waits X release, 7 CTAs       [fwd: 0..7, bwd: 8..15]
__device__ unsigned long long g_nf_prof[16];
__device__ unsigned long long g_nf_phase[64];  // worker thread 0: cycles between consecutive NF_MARK points [fwd 0..31 | bwd 32..63]
#define NF_PROF_DO(...) __VA_ARGS__
#define NF_MARK(i) do { if (tid == 0) { const long long now_ = clock64(); atomicAdd(&g_nf_phase[NF_BASE + (i)], (unsigned long long)(now_ - c.t_last)); c.t_last = now_; } } while (0)
#else
#define NF_PROF_DO(...)
#define NF_MARK(i)
#endif

struct Prog {
    int n;
    uint16_t tile[24];
    uint8_t flag[24];
};

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred P1;\nLAB_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n@P1 bra DONE;\nbra LAB_WAIT;\nDONE:\n}\n" ::"r"(
            s_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_u32(dst)), "l"(src), "r"(bytes),
                 "r"(s_u32(bar))
                 : "memory");
}
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
__device__ __forceinline__ void work_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(32 * NWORK) : "memory"); }  // all worker warps (single-group builds)
// plain (coherent) 16-byte load: for arrays written earlier in the SAME kernel (ld.global.nc / __ldg would be wrong there)
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// ------------------------------------------------------------------------------------------------------------------
struct Ctx {
    float *x_hi, *x_lo;
    unsigned char* ring;
    float* stage;  // [128 features][SROW]: the summed accumulators of the last finished output tile
    uint64_t *full, *empty, *x_ready, *x_free, *acc_full, *stage_free, *dep;
    // xsplit: the activation operand is handed over in two K halves (k < 64: x_ready / x_free, k >= 64: x_ready2 / x_free2), so that the next
    // operand's first half is written while the MMAs still read the second half of the current one (and the MMAs start on the first half while
    // the second is written): double buffering at half-operand granularity, no extra shared memory.
    uint64_t *x_ready2, *x_free2;
    int xsplit = 0;
    int xg = 0;  // X generations written so far (worker warps) / consumed (issuer)
    int o = 0;   // output tiles drained so far (worker warps) / staged (issuer)
    NF_PROF_DO(long long w_acc = 0, w_xfree = 0, w_x = 0, w_buf = 0, w_full = 0, t_last = 0;)
};

// MMA warpgroups (all 256 threads walk the program; warpgroup h owns features [64 h, +64) of the weight tile).  Per k-step of 8: lo.hi + hi.lo
// into the correction accumulator, hi.hi alternating over two main accumulators (the tensor core truncates when it accumulates: chains of 8
// per 128 k, one main accumulator measured 1.3e-5 Ha of PaiNN energy drift); both stay in registers across the units of an output tile (K > 128 accumulates over several
// X operands).  A ring stage is released when the wgmma group that read it has completed (one arrival per warp), the operand X after the last
// unit that reads it, and a finished tile is summed (RN) into the staging tile once the epilogues have called drain() for the previous one.
// The weight tiles of the units (tile_of(u) = index into the prepared buffer, STAGES_PER_TILE stages each; `spt` < STAGES_PER_TILE: K <= 32 spt,
// the remaining stages of a tile image are zeros and are neither copied nor multiplied) are streamed by the first thread of the warpgroups:
// one cp.async.bulk per stage, W_STAGES ahead; a slot is refilled once both warpgroups have released it.
template <class FlagFn, class TileFn>
__device__ __forceinline__ void run_issuer_t(Ctx& c, int n_units, FlagFn flags_of, TileFn tile_of, const unsigned char* wt, int spt = STAGES_PER_TILE) {
    const int wl = ((threadIdx.x >> 5) - WARP_ISSUE) & 3, h = ((threadIdx.x >> 5) - WARP_ISSUE) >> 2, lane = threadIdx.x & 31;
    float corr[NT / 2], main0[NT / 2], main1[NT / 2];
    const uint32_t x_hi0 = s_u32(c.x_hi), x_lo0 = s_u32(c.x_lo);
    const int n_q = n_units * spt;
    const bool leader = threadIdx.x == 32 * WARP_ISSUE;
    int q = 0, pending = -1;  // pending: the stage whose wgmma group may still be reading its ring slot
    auto release = [&](uint64_t* bar) { if (lane == 0) mbar_arrive(bar); };
    auto copy = [&](int qq) {
        if (!leader || qq >= n_q) return;
        const int slot = qq % W_STAGES;
        mbar_expect_tx(c.full + slot, WST_BYTES);
        bulk_g2s(c.ring + slot * WST_BYTES, wt + (size_t)tile_of(qq / spt) * WTILE_BYTES + (size_t)(qq % spt) * WST_BYTES, WST_BYTES, c.full + slot);
    };
    auto free_stage = [&](int pq) {
        const int slot = pq % W_STAGES;
        release(c.empty + slot);
        if (leader) { mbar_wait(c.empty + slot, (uint32_t)((pq / W_STAGES) & 1)); copy(pq + W_STAGES); }
    };
    for (int qq = 0; qq < W_STAGES; ++qq) copy(qq);
#pragma unroll 1
    for (int u = 0; u < n_units; ++u) {
        const int fl = flags_of(u);
        const bool newx = (fl & U_NEWX) != 0;
        if (newx) { NF_PROF_DO(const long long t0_ = clock64();) mbar_wait(c.x_ready, (uint32_t)(c.xg & 1)); ++c.xg; NF_PROF_DO(c.w_x += clock64() - t0_;) }
        if (fl & U_FIRST) {
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) { corr[i] = 0.f; main0[i] = 0.f; main1[i] = 0.f; }
        }
#pragma unroll 1
        for (int st = 0; st < spt; ++st, ++q) {
            const int slot = q % W_STAGES;
            if (c.xsplit && newx && st == STAGES_PER_TILE / 2) {  // the second K half of a new operand
                NF_PROF_DO(const long long t0_ = clock64();)
                mbar_wait(c.x_ready2, (uint32_t)((c.xg - 1) & 1));
                NF_PROF_DO(c.w_x += clock64() - t0_;)
            }
            NF_PROF_DO(const long long t1_ = clock64();)
            mbar_wait(c.full + slot, (uint32_t)((q / W_STAGES) & 1));
            NF_PROF_DO(c.w_full += clock64() - t1_;)
            const uint32_t wh = s_u32(c.ring + slot * WST_BYTES), wlo = wh + (KSTAGE / 4) * WLBO;
            const uint32_t xoff = (uint32_t)(st * (KSTAGE / 4) * XLBO);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KSTAGE / 8; ++ks) {
                const uint64_t dxh = gmma_desc(x_hi0 + xoff + 2 * ks * XLBO, XLBO, 128), dxl = gmma_desc(x_lo0 + xoff + 2 * ks * XLBO, XLBO, 128);
                const uint64_t dwh = gmma_desc(wh + 2 * ks * WLBO + h * 1024, WLBO, 128), dwl = gmma_desc(wlo + 2 * ks * WLBO + h * 1024, WLBO, 128);
                wgmma_tf32_n64(corr, dwl, dxh);
                wgmma_tf32_n64(corr, dwh, dxl);
                if (ks & 1) wgmma_tf32_n64(main1, dwh, dxh);
                else wgmma_tf32_n64(main0, dwh, dxh);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous stage's group has completed: free its ring slot
            if (pending >= 0) free_stage(pending);
            pending = q;
            if (c.xsplit && (fl & U_XLAST) && st == STAGES_PER_TILE / 2 - 1) {  // first K half: no later MMA reads it
                wgmma_wait<0>();
                free_stage(pending); pending = -1;
                release(c.x_free);
            }
        }
        wgmma_wait<0>();
        if (pending >= 0) { free_stage(pending); pending = -1; }
        if (fl & U_XLAST) {
            if (!c.xsplit) release(c.x_free);
            else { if (spt < STAGES_PER_TILE / 2) release(c.x_free); release(c.x_free2); }
        }
        if (fl & U_LAST) {
            if (c.o > 0) { NF_PROF_DO(const long long t2_ = clock64();) mbar_wait(c.stage_free, (uint32_t)((c.o - 1) & 1)); NF_PROF_DO(c.w_buf += clock64() - t2_;) }
            const int f = 64 * h + 16 * wl + (lane >> 2);
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(c.stage + f * SROW + n) = make_float2(corr[4 * j] + (main0[4 * j] + main1[4 * j]), corr[4 * j + 1] + (main0[4 * j + 1] + main1[4 * j + 1]));
                *reinterpret_cast<float2*>(c.stage + (f + 8) * SROW + n) = make_float2(corr[4 * j + 2] + (main0[4 * j + 2] + main1[4 * j + 2]), corr[4 * j + 3] + (main0[4 * j + 3] + main1[4 * j + 3]));
            }
            mbar_arrive(c.acc_full);
            ++c.o;
        }
    }
}
__device__ __forceinline__ void run_issuer(Ctx& c, const Prog& prog, const unsigned char* wt) {
    run_issuer_t(c, prog.n, [&](int u) { return (int)prog.flag[u]; }, [&](int u) { return (int)prog.tile[u]; }, wt);
}

// worker warps: fill the activation operand with f(row 0..127 of the tile, chunk 0..31) -> 4 consecutive k values.
// Two halves of 8 rows per thread (rolled).  Per half: ALL global loads are issued (and f's arithmetic done) BEFORE the thread waits for
// the previous operand to be released, so their latency overlaps the MMAs still reading that operand; only split + 16 shared-memory
// stores follow the wait.  (8 worker warps per SM: a load -> use -> store sequence per element would expose one L2 round trip each.)
template <class Fn>
__device__ __forceinline__ void load_x(Ctx& c, int wtid, Fn f) {
    if (c.xsplit) {
        // half-operand hand-over: the two K halves must be written by DIFFERENT WARPS -- a warp whose lanes wait on two barriers reconverges
        // after the wait loop, i.e. both halves would wait for the later barrier (first version, by lane: no gain at all).  Warps [0, NLOAD/2)
        // write k < 64, the others k >= 64; a warp instruction covers 2 rows x 16 chunks (two 256-byte global segments, conflict-free
        // 16-byte shared-memory stores per quarter warp).
        const int lane = wtid & 31, wrp = wtid >> 5, half = wrp >= NLOAD / 2 ? 1 : 0, w8 = wrp - half * (NLOAD / 2);
        const int kc = (lane & 15) + 16 * half, rsub = lane >> 4;
        constexpr int ITEMS = (NT * 16) / (32 * (NLOAD / 2));  // (row, chunk) pairs per thread: 8 for NT = 128, NLOAD = 16
        static_assert(ITEMS * 32 * (NLOAD / 2) == NT * 16 && ITEMS <= 16, "load_x xsplit mapping");
        float4 t[ITEMS];
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) t[it] = f(2 * (w8 + (NLOAD / 2) * it) + rsub, kc);
        NF_PROF_DO(const long long t0_ = clock64();)
        if (c.xg > 0) mbar_wait(half ? c.x_free2 : c.x_free, (uint32_t)((c.xg - 1) & 1));  // the MMAs that read my half of the previous operand have retired
        NF_PROF_DO(c.w_xfree += clock64() - t0_;)
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
            const int r = 2 * (w8 + (NLOAD / 2) * it) + rsub;
            float4 hi, lo;
            split4(t[it], hi, lo);
            st4(c.x_hi + kc * XLBOF + r * 4, hi);
            st4(c.x_lo + kc * XLBOF + r * 4, lo);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(half ? c.x_ready2 : c.x_ready);
        ++c.xg;
        return;
    }
    const int kc = wtid & 31, w = wtid >> 5;
#pragma unroll 1
    for (int h = 0; h < RPT / 8; ++h) {
        float4 t[8];
#pragma unroll
        for (int it = 0; it < 8; ++it) t[it] = f(w + NLOAD * (8 * h + it), kc);
        NF_PROF_DO(const long long t0_ = clock64();)
        if (c.xg > 0) mbar_wait(c.x_free, (uint32_t)((c.xg - 1) & 1));  // every MMA that read the previous operand has retired
        NF_PROF_DO(c.w_xfree += clock64() - t0_;)
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int r = w + NLOAD * (8 * h + it);
            float4 hi, lo;
            split4(t[it], hi, lo);
            st4(c.x_hi + kc * XLBOF + r * 4, hi);
            st4(c.x_lo + kc * XLBOF + r * 4, lo);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_arrive(c.x_ready);
    ++c.xg;
}

// worker warps, epilogue side: this thread's values (feature k, atom n) become the next operand
struct XPut {
    float *hi, *lo;
    bool second;  // my feature row k lies in the second K half
    __device__ __forceinline__ XPut(const Ctx& c, int k) {
        second = c.xsplit && k >= 64;
        if (c.xg > 0) mbar_wait(second ? c.x_free2 : c.x_free, (uint32_t)((c.xg - 1) & 1));
        hi = c.x_hi + (k >> 2) * XLBOF + (k & 3);
        lo = c.x_lo + (k >> 2) * XLBOF + (k & 3);
    }
    __device__ __forceinline__ void put(int n, float v) const {
        float h, l;
        split_tf32(v, h, l);
        hi[n * 4] = h;
        lo[n * 4] = l;
    }
    __device__ __forceinline__ void done(Ctx& c) const {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(second ? c.x_ready2 : c.x_ready);
        ++c.xg;
    }
};

// worker warps: wait for output tile `o` in the staging tile (after telling the issuer that this thread is done with the previous one).
// add_stage: K > 128 split over two output tiles (forward g1pre): this thread's part of the previous tile is kept and added to the new one.
__device__ __forceinline__ void drain(Ctx& c, int warp, int add_stage = 0) {
    NF_PROF_DO(const long long t0_ = clock64();)
    float* mine = c.stage + (32 * (warp & 3) + (threadIdx.x & 31)) * SROW + (warp >> 2) * CPT;
    if (add_stage) {
        float4 keep[CPT / 4];
#pragma unroll
        for (int i = 0; i < CPT / 4; ++i) keep[i] = reinterpret_cast<const float4*>(mine)[i];
        if (c.o > 0) mbar_arrive(c.stage_free);
        mbar_wait(c.acc_full, (uint32_t)(c.o & 1));
#pragma unroll
        for (int i = 0; i < CPT / 4; ++i) reinterpret_cast<float4*>(mine)[i] = reinterpret_cast<const float4*>(mine)[i] + keep[i];
    } else {
        if (c.o > 0) mbar_arrive(c.stage_free);
        mbar_wait(c.acc_full, (uint32_t)(c.o & 1));
    }
    NF_PROF_DO(c.w_acc += clock64() - t0_;)
    ++c.o;
}

// 16 staged values of this thread: atoms CPT (warp >> 2) + 16 cb .. + 15 of its feature
__device__ __forceinline__ void stage_ld16(const Ctx& c, int warp, int cb, float (&v)[16]) {
    const float4* src = reinterpret_cast<const float4*>(c.stage + (32 * (warp & 3) + (threadIdx.x & 31)) * SROW + (warp >> 2) * CPT + cb * 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float4 t = src[i];
        v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
}

__device__ __forceinline__ void prog_add(Prog& p, int tile, int flags) {
    p.tile[p.n] = (uint16_t)tile;
    p.flag[p.n] = (uint8_t)flags;
    ++p.n;
}

// common prologue: carve shared memory, init barriers
__device__ __forceinline__ Ctx setup(unsigned char* smem, int tid, int xsplit = 0) {
    Ctx c;
    c.xsplit = xsplit;
    c.x_hi = reinterpret_cast<float*>(smem);
    c.x_lo = reinterpret_cast<float*>(smem + X_BYTES);
    c.ring = smem + 2 * X_BYTES;
    c.stage = reinterpret_cast<float*>(smem + 2 * X_BYTES + W_STAGES * WST_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_BARS);
    c.full = bars; c.empty = bars + W_STAGES; c.x_ready = bars + 2 * W_STAGES; c.x_free = c.x_ready + 1; c.acc_full = c.x_ready + 2;
    c.stage_free = c.x_ready + 3;
    c.dep = c.x_ready + 6;  // 4 hand-over barriers between the worker groups
    c.x_ready2 = c.x_ready + 11; c.x_free2 = c.x_ready + 12;
    if (tid == 0) {
        for (int s = 0; s < W_STAGES; ++s) { mbar_init(c.full + s, 1); mbar_init(c.empty + s, 8); }  // empty / x_free: one arrival per MMA warp
        mbar_init(c.x_ready, xsplit ? 16 * NLOAD : 32 * NLOAD);  // == 32 * NEPI: one group writes a whole operand generation (half of it with xsplit)
        mbar_init(c.x_free, 8);
        mbar_init(c.x_ready2, 16 * NLOAD);
        mbar_init(c.x_free2, 8);
        mbar_init(c.acc_full, 256);
        mbar_init(c.stage_free, 32 * NEPI);
        for (int b = 0; b < 4; ++b) mbar_init(c.dep + b, 32 * NLOAD);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    return c;
}

// ---- worker roles
__device__ __forceinline__ bool role_epi(int warp) { return warp < NEPI; }
#ifdef NF_TWO_GROUPS
__device__ __forceinline__ bool role_load(int warp) { return warp >= NEPI && warp < NEPI + NLOAD; }
__device__ __forceinline__ int load_tid(int tid) { return tid - 32 * NEPI; }
#else
__device__ __forceinline__ bool role_load(int warp) { return warp < NLOAD; }
__device__ __forceinline__ int load_tid(int tid) { return tid; }
#endif
// data handed from one group to the other through GLOBAL memory (k = which hand-over of the kernel, each used once): the producers arrive
// after their stores, the consumers wait; single-group builds: one CTA-wide barrier of the worker warps at the producer's point
__device__ __forceinline__ void dep_signal(const Ctx& c, int k) {
#ifdef NF_TWO_GROUPS
    mbar_arrive(c.dep + k);
#else
    (void)c; (void)k;
    work_barrier();
#endif
}
__device__ __forceinline__ void dep_wait(const Ctx& c, int k) {
#ifdef NF_TWO_GROUPS
    mbar_wait(c.dep + k, 0u);
#else
    (void)c; (void)k;
#endif
}

// epilogue loop over this thread's part of the staged tile: chunks of 16 atoms, rolled (one copy of the body in the instruction cache)
template <class Body>
__device__ __forceinline__ void epi_chunks(const Ctx& c, int warp, Body body) {
#pragma unroll 1
    for (int cb = 0; cb < CPT / 16; ++cb) {
        float v[16];
        stage_ld16(c, warp, cb, v);
        body(cb, v);
    }
}


}  // namespace
