// tc_pipe.cuh -- the warp-specialised wgmma pipeline shared by the fused PaiNN node kernels (painn_fused.cu) and the pre-split-weight GEMM
// (gemm_ps.cu): weight tiles as ready-made TF32 hi / lo shared-memory images streamed by cp.async.bulk through an mbarrier ring, the
// activation operand X written by worker warps (loader functors or epilogue registers), one MMA warpgroup (3xTF32: a correction and a main
// accumulator in registers), a shared-memory staging tile of the summed accumulators, epilogues in rolled chunks of L::CW columns (16; 8 at NT = 80).
// D[feature, row] = W[feature, k] . X[row, k]^T: features on the staging rows, rows (atoms / edges / pairs) on its columns.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace {


constexpr int F = NB_F;
// CTA = NT atoms (the template parameter of Layout below), 8 worker warps, two MMA warpgroups (features [0, 64) and [64, 128) of a
// weight tile) whose first thread also issues the weight copies (a separate producer warp made 17 warps, and ptxas then capped the
// registers at 96); 3 ring stages of 32 k.  An MMA warpgroup holds its 64 features x NT atoms three times (correction + two alternating
// main accumulators: 3 NT / 2 fp32 registers per thread; one warpgroup for all 128 features spilled), and the staging tile the epilogues
// read lives in shared memory next to the hi / lo activation operand and the weight ring: 65 + 96 + 34 KB at NT = 64, 81 + 96 + 42 KB at
// NT = 80 (NT = 128 would not fit the 227 KB of an SM).
constexpr int KSTAGE = 32, W_STAGES = 3, NWORK = 8, CTAS_PER_SM = 1;
constexpr int WLBO = 128 * 16;             // weight stages are written by the bulk-copy engine: no padding needed
constexpr int WST_BYTES = 2 * (KSTAGE / 4) * WLBO;  // one ring stage: [hi | lo] x KSTAGE/4 chunks x 128 rows x 16 B
constexpr int STAGES_PER_TILE = 128 / KSTAGE;
constexpr int WTILE_BYTES = STAGES_PER_TILE * WST_BYTES;  // 128 rows x 128 k, hi + lo = 128 KB
// Worker layouts (the template parameter L of the pipeline below; the choice is fixed per kernel instantiation):
//   OneGroup:  all NWORK worker warps load operands AND run epilogues, in program order; the operand is handed over whole.
//   TwoGroups: warps [0, NEPI) only drain, run epilogues and write chained operands, warps [NEPI, NWORK) only run the loader functors and
//     therefore run AHEAD of the epilogues (their global loads overlap epilogue work and MMAs).  The operand is handed over in two K halves
//     (k < 64: x_ready / x_free, k >= 64: x_ready2 / x_free2), so that the next operand's first half is written while the MMAs still read
//     the second half of the current one (and the MMAs start on the first half while the second is written): double buffering at
//     half-operand granularity, no extra shared memory.
// NT_: atoms (rows) per CTA, the N of every wgmma: 64, or 80 for the fused PaiNN node kernels when 64-atom tiles need more than one wave.
template <bool TWO_GROUPS, int NT_ = 64>
struct Layout {
    static constexpr bool two_groups = TWO_GROUPS;
    static constexpr int NT = NT_;
    static constexpr int NEPI = TWO_GROUPS ? NWORK / 2 : NWORK, NLOAD = TWO_GROUPS ? NWORK / 2 : NWORK;
    static constexpr int CPT = NT / (NEPI / 4);  // staged columns (atoms) per epilogue thread (4 feature groups of 32 x NEPI/4 column parts)
    // epilogue chunk: staged columns per round of epi_chunks (CPT = 40 at NT = 80: chunks of 20 spilled in 88 worker registers)
    static constexpr int CW = CPT % 16 == 0 ? 16 : 8;
    static constexpr int RPT = NT / NLOAD;       // operand rows per loader thread
    static constexpr int XLBO = NT * 16 + 16;    // bytes between 16-byte k-chunks of X (padded: the 8 chunk writers of a row hit 8 bank groups)
    static constexpr int XLBOF = XLBO / 4;
    static constexpr int X_BYTES = 32 * XLBO;    // one of hi / lo, K = 128
    static constexpr int SROW = NT + 4;          // staging row stride (floats): the 16-byte reads of 8 consecutive feature rows hit 8 bank groups
    static constexpr int STAGE_BYTES = 128 * SROW * 4;
    static constexpr int SMEM_BARS = 2 * X_BYTES + W_STAGES * WST_BYTES + STAGE_BYTES;
    static constexpr int SMEM_TOTAL = SMEM_BARS + 256;
    // registers per thread of the worker / MMA warpgroups (setmaxnreg, see role_regs); 0: the even split of the launch (128 each).
    // At NT = 80 an MMA thread holds 120 accumulators; 2 x 128 x (88 + 168) = the 64 K registers of the SM.
    static constexpr int WORK_REGS = NT == 64 ? 0 : 88, MMA_REGS = NT == 64 ? 0 : 168;
    static_assert(NT == 64 || NT == 80, "the wgmma N of the pipeline (wgmma_tf32_nt)");
    static_assert(SMEM_TOTAL <= 227 * 1024, "shared memory of one CTA");
    static_assert((XLBO / 16) % 2 == 1 && XLBO % 128 == 16, "X padding: 8 chunk writers of a row / 32 feature writers of a column hit distinct banks");
    static_assert((SROW / 4) % 2 == 1, "staging padding: the 16-byte reads of 8 consecutive feature rows hit 8 bank groups");
    static_assert(CPT % CW == 0 && CW % 4 == 0, "epilogue chunks");
    static_assert(WORK_REGS + MMA_REGS == 0 || WORK_REGS + MMA_REGS == 2 * 128, "the register split must hand over exactly what it takes");
};
using OneGroup = Layout<false>;
using TwoGroups = Layout<true>;
constexpr int WARP_ISSUE = NWORK;          // first warp of the two MMA warpgroups (warpgroups start at a multiple of 4 warps)
constexpr int NTHREADS = 32 * (NWORK + 8);
static_assert(NWORK % 4 == 0, "the MMA warpgroups must start on a warpgroup boundary");
static_assert(NWORK * 32 == NTHREADS / 2, "role_regs: the worker and MMA warpgroups hold the same number of threads");

// Moves registers from the worker warpgroups to the MMA warpgroups (L::MMA_REGS > 0).  Called once by every thread at the role split; the
// launch must give 128 registers per thread (__launch_bounds__(NTHREADS, 1)), so that the MMA side's increase is exactly what the workers
// release (setmaxnreg.inc waits for free registers of the CTA).
template <class L>
__device__ __forceinline__ void role_regs(bool mma) {
    if constexpr (L::MMA_REGS > 0) {
        if (mma) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(L::MMA_REGS));
        else asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(L::WORK_REGS));
    }
}

template <int NT>
__device__ __forceinline__ void wgmma_tf32_nt(float (&d)[NT / 2], uint64_t da, uint64_t db) {
    if constexpr (NT == 64) wgmma_tf32_n64(d, da, db);
    else wgmma_tf32_n80(d, da, db);
}
enum { U_NEWX = 1, U_FIRST = 2, U_LAST = 4, U_XLAST = 8 };

struct Prog {
    int n;
    uint16_t tile[24];
    uint8_t flag[24];
};

__device__ __forceinline__ void work_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(32 * NWORK) : "memory"); }  // all worker warps (one group)
// plain (coherent) 16-byte load: for arrays written earlier in the SAME kernel (ld.global.nc / __ldg would be wrong there)
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// ------------------------------------------------------------------------------------------------------------------
template <class L>
struct Ctx {
    float *x_hi, *x_lo;
    unsigned char* ring;
    float* stage;  // [128 features][SROW]: the summed accumulators of the last finished output tile
    uint64_t *full, *empty, *x_ready, *x_free, *acc_full, *stage_free;
    uint64_t *x_ready2, *x_free2;  // TwoGroups: hand-over of the second K half
    int xg = 0;  // X generations written so far (worker warps) / consumed (issuer)
    int o = 0;   // output tiles drained so far (worker warps) / staged (issuer)
};

// MMA warpgroups (all 256 threads walk the program; warpgroup h owns features [64 h, +64) of the weight tile).  Per k-step of 8: lo.hi + hi.lo
// into the correction accumulator, hi.hi alternating over two main accumulators (the tensor core truncates when it accumulates: chains of 8
// per 128 k, one main accumulator measured 1.3e-5 Ha of PaiNN energy drift); both stay in registers across the units of an output tile (K > 128 accumulates over several
// X operands).  A ring stage is released when the wgmma group that read it has completed (one arrival per warp), the operand X after the last
// unit that reads it, and a finished tile is summed (RN) into the staging tile once the epilogues have called drain() for the previous one.
// The weight tiles of the units (tile_of(u) = index into the prepared buffer, STAGES_PER_TILE stages each; `spt` < STAGES_PER_TILE: K <= 32 spt,
// the remaining stages of a tile image are zeros and are neither copied nor multiplied) are streamed by the first thread of the warpgroups:
// one cp.async.bulk per stage, W_STAGES ahead; a slot is refilled once both warpgroups have released it.
template <class L, class FlagFn, class TileFn>
__device__ __forceinline__ void run_issuer_t(Ctx<L>& c, int n_units, FlagFn flags_of, TileFn tile_of, const unsigned char* wt, int spt = STAGES_PER_TILE) {
    constexpr int NT = L::NT, XLBO = L::XLBO;
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
        if (newx) { mbar_wait(c.x_ready, (uint32_t)(c.xg & 1)); ++c.xg; }
        if (fl & U_FIRST) {
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) { corr[i] = 0.f; main0[i] = 0.f; main1[i] = 0.f; }
        }
#pragma unroll 1
        for (int st = 0; st < spt; ++st, ++q) {
            const int slot = q % W_STAGES;
            if (L::two_groups && newx && st == STAGES_PER_TILE / 2)  // the second K half of a new operand
                mbar_wait(c.x_ready2, (uint32_t)((c.xg - 1) & 1));
            mbar_wait(c.full + slot, (uint32_t)((q / W_STAGES) & 1));
            const uint32_t wh = s_u32(c.ring + slot * WST_BYTES), wlo = wh + (KSTAGE / 4) * WLBO;
            const uint32_t xoff = (uint32_t)(st * (KSTAGE / 4) * XLBO);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KSTAGE / 8; ++ks) {
                const uint64_t dxh = gmma_desc(x_hi0 + xoff + 2 * ks * XLBO, XLBO, 128), dxl = gmma_desc(x_lo0 + xoff + 2 * ks * XLBO, XLBO, 128);
                const uint64_t dwh = gmma_desc(wh + 2 * ks * WLBO + h * 1024, WLBO, 128), dwl = gmma_desc(wlo + 2 * ks * WLBO + h * 1024, WLBO, 128);
                wgmma_tf32_nt<NT>(corr, dwl, dxh);
                wgmma_tf32_nt<NT>(corr, dwh, dxl);
                if (ks & 1) wgmma_tf32_nt<NT>(main1, dwh, dxh);
                else wgmma_tf32_nt<NT>(main0, dwh, dxh);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous stage's group has completed: free its ring slot
            if (pending >= 0) free_stage(pending);
            pending = q;
            if (L::two_groups && (fl & U_XLAST) && st == STAGES_PER_TILE / 2 - 1) {  // first K half: no later MMA reads it
                wgmma_wait<0>();
                free_stage(pending); pending = -1;
                release(c.x_free);
            }
        }
        wgmma_wait<0>();
        if (pending >= 0) { free_stage(pending); pending = -1; }
        if (fl & U_XLAST) {
            if (!L::two_groups) release(c.x_free);
            else { if (spt < STAGES_PER_TILE / 2) release(c.x_free); release(c.x_free2); }
        }
        if (fl & U_LAST) {
            if (c.o > 0) mbar_wait(c.stage_free, (uint32_t)((c.o - 1) & 1));
            const int f = 64 * h + 16 * wl + (lane >> 2);
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(c.stage + f * L::SROW + n) = make_float2(corr[4 * j] + (main0[4 * j] + main1[4 * j]), corr[4 * j + 1] + (main0[4 * j + 1] + main1[4 * j + 1]));
                *reinterpret_cast<float2*>(c.stage + (f + 8) * L::SROW + n) = make_float2(corr[4 * j + 2] + (main0[4 * j + 2] + main1[4 * j + 2]), corr[4 * j + 3] + (main0[4 * j + 3] + main1[4 * j + 3]));
            }
            mbar_arrive(c.acc_full);
            ++c.o;
        }
    }
}
template <class L>
__device__ __forceinline__ void run_issuer(Ctx<L>& c, const Prog& prog, const unsigned char* wt) {
    run_issuer_t(c, prog.n, [&](int u) { return (int)prog.flag[u]; }, [&](int u) { return (int)prog.tile[u]; }, wt);
}

// worker warps: fill the activation operand with f(row 0..NT-1 of the tile, chunk 0..31) -> 4 consecutive k values.
// One group: rounds of RB rows per thread (rolled; one round of 8 at NT = 64, two rounds of 5 at NT = 80).  Per round: ALL global loads are
// issued (and f's arithmetic done) BEFORE the thread waits for the previous operand to be released, so their latency overlaps the MMAs still
// reading that operand; only split + 2 RB shared-memory stores follow the wait.  (8 worker warps per SM: a load -> use -> store sequence per element would expose one L2 round trip each.)
// wtid: the thread's index among the loader warps.
template <class L, class Fn>
__device__ __forceinline__ void load_x(Ctx<L>& c, int wtid, Fn f) {
    constexpr int NLOAD = L::NLOAD, NT = L::NT, XLBOF = L::XLBOF;
    if constexpr (L::two_groups) {
        // half-operand hand-over: the two K halves must be written by DIFFERENT WARPS -- a warp whose lanes wait on two barriers reconverges
        // after the wait loop, i.e. both halves would wait for the later barrier (first version, by lane: no gain at all).  Warps [0, NLOAD/2)
        // write k < 64, the others k >= 64; a warp instruction covers 2 rows x 16 chunks (two 256-byte global segments, conflict-free
        // 16-byte shared-memory stores per quarter warp).
        const int lane = wtid & 31, wrp = wtid >> 5, half = wrp >= NLOAD / 2 ? 1 : 0, w8 = wrp - half * (NLOAD / 2);
        const int kc = (lane & 15) + 16 * half, rsub = lane >> 4;
        constexpr int ITEMS = (NT * 16) / (32 * (NLOAD / 2));  // (row, chunk) pairs per thread: 16 for NT = 64, NLOAD = 4
        static_assert(ITEMS * 32 * (NLOAD / 2) == NT * 16 && ITEMS <= 16, "load_x two-group mapping");
        float4 t[ITEMS];
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) t[it] = f(2 * (w8 + (NLOAD / 2) * it) + rsub, kc);
        if (c.xg > 0) mbar_wait(half ? c.x_free2 : c.x_free, (uint32_t)((c.xg - 1) & 1));  // the MMAs that read my half of the previous operand have retired
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
            const int r = 2 * (w8 + (NLOAD / 2) * it) + rsub;
            float4 hi, lo;
            split4(t[it], hi, lo);
            st4(c.x_hi + kc * XLBOF + r * 4, hi);
            st4(c.x_lo + kc * XLBOF + r * 4, lo);
        }
        fence_proxy_async();
        mbar_arrive(half ? c.x_ready2 : c.x_ready);
        ++c.xg;
        return;
    }
    // rows per round: 8, or 5 (two rounds) for the RPT = 10 rows of a thread at NT = 80 -- one round of 10 spilled in 88 worker registers
    constexpr int RB = L::RPT % 8 == 0 ? 8 : L::RPT / 2;
    static_assert(L::RPT % RB == 0, "load_x one-group mapping");
    const int kc = wtid & 31, w = wtid >> 5;
#pragma unroll 1
    for (int h = 0; h < L::RPT / RB; ++h) {
        float4 t[RB];
#pragma unroll
        for (int it = 0; it < RB; ++it) t[it] = f(w + NLOAD * (RB * h + it), kc);
        if (c.xg > 0) mbar_wait(c.x_free, (uint32_t)((c.xg - 1) & 1));  // every MMA that read the previous operand has retired
#pragma unroll
        for (int it = 0; it < RB; ++it) {
            const int r = w + NLOAD * (RB * h + it);
            float4 hi, lo;
            split4(t[it], hi, lo);
            st4(c.x_hi + kc * XLBOF + r * 4, hi);
            st4(c.x_lo + kc * XLBOF + r * 4, lo);
        }
    }
    fence_proxy_async();
    mbar_arrive(c.x_ready);
    ++c.xg;
}

// worker warps, epilogue side: this thread's values (feature k, atom n) become the next operand
template <class L>
struct XPut {
    float *hi, *lo;
    bool second;  // my feature row k lies in the second K half
    __device__ __forceinline__ XPut(const Ctx<L>& c, int k) {
        second = L::two_groups && k >= 64;
        if (c.xg > 0) mbar_wait(second ? c.x_free2 : c.x_free, (uint32_t)((c.xg - 1) & 1));
        hi = c.x_hi + (k >> 2) * L::XLBOF + (k & 3);
        lo = c.x_lo + (k >> 2) * L::XLBOF + (k & 3);
    }
    __device__ __forceinline__ void put(int n, float v) const {
        float h, l;
        split_tf32(v, h, l);
        hi[n * 4] = h;
        lo[n * 4] = l;
    }
    __device__ __forceinline__ void done(Ctx<L>& c) const {
        fence_proxy_async();
        mbar_arrive(second ? c.x_ready2 : c.x_ready);
        ++c.xg;
    }
};

// worker warps: wait for output tile `o` in the staging tile (after telling the issuer that this thread is done with the previous one).
// add_stage: K > 128 split over two output tiles (forward g1pre): this thread's part of the previous tile is kept and added to the new one.
template <class L>
__device__ __forceinline__ void drain(Ctx<L>& c, int warp, int add_stage = 0) {
    float* mine = c.stage + (32 * (warp & 3) + (threadIdx.x & 31)) * L::SROW + (warp >> 2) * L::CPT;
    if (add_stage) {
        float4 keep[L::CPT / 4];
#pragma unroll
        for (int i = 0; i < L::CPT / 4; ++i) keep[i] = reinterpret_cast<const float4*>(mine)[i];
        if (c.o > 0) mbar_arrive(c.stage_free);
        mbar_wait(c.acc_full, (uint32_t)(c.o & 1));
#pragma unroll
        for (int i = 0; i < L::CPT / 4; ++i) reinterpret_cast<float4*>(mine)[i] = reinterpret_cast<const float4*>(mine)[i] + keep[i];
    } else {
        if (c.o > 0) mbar_arrive(c.stage_free);
        mbar_wait(c.acc_full, (uint32_t)(c.o & 1));
    }
    ++c.o;
}

// W staged values of this thread: atoms CPT (warp >> 2) + col .. + W - 1 of its feature (col, W multiples of 4)
template <class L, int W>
__device__ __forceinline__ void stage_ld(const Ctx<L>& c, int warp, int col, float (&v)[W]) {
    const float4* src = reinterpret_cast<const float4*>(c.stage + (32 * (warp & 3) + (threadIdx.x & 31)) * L::SROW + (warp >> 2) * L::CPT + col);
#pragma unroll
    for (int i = 0; i < W / 4; ++i) {
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
template <class L>
__device__ __forceinline__ Ctx<L> setup(unsigned char* smem, int tid) {
    Ctx<L> c;
    c.x_hi = reinterpret_cast<float*>(smem);
    c.x_lo = reinterpret_cast<float*>(smem + L::X_BYTES);
    c.ring = smem + 2 * L::X_BYTES;
    c.stage = reinterpret_cast<float*>(smem + 2 * L::X_BYTES + W_STAGES * WST_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::SMEM_BARS);
    c.full = bars; c.empty = bars + W_STAGES; c.x_ready = bars + 2 * W_STAGES; c.x_free = c.x_ready + 1; c.acc_full = c.x_ready + 2;
    c.stage_free = c.x_ready + 3; c.x_ready2 = c.x_ready + 4; c.x_free2 = c.x_ready + 5;
    if (tid == 0) {
        for (int s = 0; s < W_STAGES; ++s) { mbar_init(c.full + s, 1); mbar_init(c.empty + s, 8); }  // empty / x_free: one arrival per MMA warp
        // x_ready: the threads that write one operand generation (== 32 * NEPI), one K half of it with two groups
        mbar_init(c.x_ready, L::two_groups ? 16 * L::NLOAD : 32 * L::NLOAD);
        mbar_init(c.x_free, 8);
        if (L::two_groups) {
            mbar_init(c.x_ready2, 16 * L::NLOAD);
            mbar_init(c.x_free2, 8);
        }
        mbar_init(c.acc_full, 256);
        mbar_init(c.stage_free, 32 * L::NEPI);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    return c;
}

// epilogue loop over this thread's part of the staged tile: chunks of L::CW atoms, rolled (one copy of the body in the instruction cache)
template <class L, class Body>
__device__ __forceinline__ void epi_chunks(const Ctx<L>& c, int warp, Body body) {
#pragma unroll 1
    for (int cb = 0; cb < L::CPT / L::CW; ++cb) {
        float v[L::CW];
        stage_ld(c, warp, L::CW * cb, v);
        body(cb, v);
    }
}


}  // namespace
