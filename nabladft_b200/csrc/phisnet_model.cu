// phisnet_model.cu -- the PhiSNet model forward (nablaDFT/phisnet/nn/neural_network.py:717-995) beyond the single mixing layers of phisnet.cu.
//
// Features are component-major [rows][25][F] (order 4, component l*l + m), one thread owns one feature channel, as in phisnet.cu.
//   nb200_phis_swish_self_mixing  SelfMixing with the learnable swish of the preceding activation applied to component 0 on load
//   nb200_phis_linear_ex          per-order Linear with accumulate: the residual add x + linear2(..) happens in the GEMM epilogue
//   nb200_phis_interaction        InteractionBlock's pair part (interaction_block.py:137-146): one CTA per target atom i walks its CSR row,
//                                 gathers yj[j], forms angular_fn1/2 from the 25 SH values on the fly, runs the 65 CG paths and the radial
//                                 term and keeps the sum in registers; writes yi + sum.  No [P,25,F] pair tensor, no index_add, no atomics.
//   nb200_phis_pair_features      fii and fij (neural_network.py:787-838); sum_{k != i,j} = T_i - own term with T_i = sum_{k != i}
//   nb200_phis_overlap_pairs      mix_s of the overlap branch (neural_network.py:753-774)
//   nb200_phis_assemble           output heads fused with the matrix assembly (neural_network.py:853-967): only the irreps a block uses
#include "common.cuh"
#include "phisnet_cg_gen.inc"
#include "phisnet_asm_cg.inc"

namespace {

constexpr int PLM = 25;
constexpr int ASM_MAX_ROWS = 32;  // orbitals per atom (def2-SVP: Br 5s4p3d = 32)
constexpr int ASM_MAX_ORB = 16;   // shells per atom

__device__ __forceinline__ int lm_order(int k) { return k < 1 ? 0 : k < 4 ? 1 : k < 9 ? 2 : k < 16 ? 3 : 4; }
__device__ __forceinline__ float swishf(float x, float a, float b) { return a * x / (1.f + expf(-b * x)); }

__global__ void __launch_bounds__(128) k_swish_self_mix(const float* __restrict__ x, const float* __restrict__ alpha, const float* __restrict__ beta,
                                                       const float* __restrict__ mix, const float* __restrict__ keep, float* __restrict__ y) {
    const int r = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    float a[PLM], o[PLM];
#pragma unroll
    for (int k = 0; k < PLM; ++k) a[k] = __ldg(x + ((size_t)r * PLM + k) * F + f);
    if (alpha) a[0] = swishf(a[0], __ldg(alpha + f), __ldg(beta + f));
#pragma unroll
    for (int k = 0; k < PLM; ++k) o[k] = __ldg(keep + (size_t)lm_order(k) * F + f) * a[k];
    phis_self_couple(a, a, mix + f, F, 4, 4, 4, o);
#pragma unroll
    for (int k = 0; k < PLM; ++k) y[((size_t)r * PLM + k) * F + f] = o[k];
}

// coeff[e][70][F]: 65 mixing paths, then radial_fn L = 0..4.  wa*: angular_fn Linear(1, F) weights [5][F], bias [F] (L = 0).
__global__ void __launch_bounds__(128) k_interaction(const float* __restrict__ yi, const float* __restrict__ yj, const float* __restrict__ sh,
                                                    const float* __restrict__ coeff, const float* __restrict__ wa1, const float* __restrict__ ba1,
                                                    const float* __restrict__ wa2, const float* __restrict__ ba2, const int32_t* __restrict__ row_ptr,
                                                    const int32_t* __restrict__ col, float* __restrict__ y) {
    const int i = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    float o[PLM], w1[5];
#pragma unroll
    for (int k = 0; k < PLM; ++k) o[k] = __ldg(yi + ((size_t)i * PLM + k) * F + f);
#pragma unroll
    for (int L = 0; L < 5; ++L) w1[L] = __ldg(wa1 + L * F + f);
    const float b1 = __ldg(ba1 + f);
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
        const int j = col[e];
        const float* s = sh + (size_t)e * PLM;
        float a[PLM], b[PLM];
#pragma unroll
        for (int k = 0; k < PLM; ++k) {
            a[k] = __ldg(yj + ((size_t)j * PLM + k) * F + f);
            b[k] = __ldg(s + k) * w1[lm_order(k)];
        }
        b[0] += b1;
        const float* c = coeff + (size_t)e * 70 * F + f;
        phis_pair_couple(a, b, c, F, 4, 4, 4, o);
        // + radial_fn_L(rbf) * angular_fn2(sph)_L * yj[0]
#pragma unroll
        for (int k = 0; k < PLM; ++k) {
            const int L = lm_order(k);
            const float ang = fmaf(__ldg(s + k), __ldg(wa2 + L * F + f), k == 0 ? __ldg(ba2 + f) : 0.f);
            o[k] = fmaf(__ldg(c + (65 + L) * F) * ang, a[0], o[k]);
        }
    }
#pragma unroll
    for (int k = 0; k < PLM; ++k) y[((size_t)i * PLM + k) * F + f] = o[k];
}

// coeff[e][75][F]: 65 mix_ij paths, radial_ii L = 0..4, radial_ij L = 0..4.
__global__ void __launch_bounds__(128) k_pair_features(const float* __restrict__ fpc, const float* __restrict__ fpn, const float* __restrict__ coeff,
                                                      const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col, float* __restrict__ fii,
                                                      float* __restrict__ fij) {
    extern __shared__ float t_sh[];  // T_i [25][F]: thread f owns column f
    const int i = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    {
        float p[PLM], t[PLM];
#pragma unroll
        for (int k = 0; k < PLM; ++k) { p[k] = __ldg(fpc + ((size_t)i * PLM + k) * F + f); t[k] = 0.f; }
        for (int e = e0; e < e1; ++e) {
            const int j = col[e];
            const float* c = coeff + (size_t)e * 75 * F + f;
            float rii[5], rij[5];
#pragma unroll
            for (int L = 0; L < 5; ++L) { rii[L] = __ldg(c + (65 + L) * F); rij[L] = __ldg(c + (70 + L) * F); }
#pragma unroll
            for (int k = 0; k < PLM; ++k) {
                const float v = __ldg(fpn + ((size_t)j * PLM + k) * F + f);
                p[k] = fmaf(rii[lm_order(k)], v, p[k]);
                t[k] = fmaf(rij[lm_order(k)], v, t[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < PLM; ++k) { fii[((size_t)i * PLM + k) * F + f] = p[k]; t_sh[k * F + f] = t[k]; }
    }
    for (int e = e0; e < e1; ++e) {
        const int j = col[e];
        const float* c = coeff + (size_t)e * 75 * F + f;
        float a[PLM], b[PLM], o[PLM];  // fpc[i] re-read per pair (L1 hit), as in k_overlap_pairs
#pragma unroll
        for (int k = 0; k < PLM; ++k) {
            a[k] = __ldg(fpc + ((size_t)i * PLM + k) * F + f);
            const float v = __ldg(fpn + ((size_t)j * PLM + k) * F + f);
            o[k] = fmaf(-__ldg(c + (70 + lm_order(k)) * F), v, t_sh[k * F + f]);
            b[k] = __ldg(fpc + ((size_t)j * PLM + k) * F + f);
        }
        phis_pair_couple(a, b, c, F, 4, 4, 4, o);
#pragma unroll
        for (int k = 0; k < PLM; ++k) fij[((size_t)e * PLM + k) * F + f] = o[k];
    }
}

// s_ij = mix_s(x[i], (x[j]_0, angular_fn(sph)_{L>0}), rbf); coeff[e][65][F]; wa: angular_fn weights [5][F] (its L = 0 output is unused)
__global__ void __launch_bounds__(128) k_overlap_pairs(const float* __restrict__ x, const float* __restrict__ sh, const float* __restrict__ coeff,
                                                      const float* __restrict__ wa, const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col,
                                                      float* __restrict__ s_out) {
    const int i = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    float w[5];
#pragma unroll
    for (int L = 0; L < 5; ++L) w[L] = __ldg(wa + L * F + f);
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
        const int j = col[e];
        float a[PLM], b[PLM], o[PLM];
        // x[i] is re-read per pair (L1 hit): a loop-invariant copy lets the compiler hoist CG products of it and spill
#pragma unroll
        for (int k = 0; k < PLM; ++k) a[k] = __ldg(x + ((size_t)i * PLM + k) * F + f);
        b[0] = __ldg(x + (size_t)j * PLM * F + f);
#pragma unroll
        for (int k = 1; k < PLM; ++k) b[k] = __ldg(sh + (size_t)e * PLM + k) * w[lm_order(k)];
#pragma unroll
        for (int k = 0; k < PLM; ++k) o[k] = 0.f;
        phis_pair_couple(a, b, coeff + (size_t)e * 65 * F + f, F, 4, 4, 4, o);
#pragma unroll
        for (int k = 0; k < PLM; ++k) s_out[((size_t)e * PLM + k) * F + f] = o[k];
    }
}

struct AsmTables {
    const int32_t* atom_el;    // [N] element index of each atom
    const int32_t* row_orb;    // [n_el][32] shell of each orbital row
    const int32_t* row_m;      // [n_el][32] m index (0 .. 2l) of each orbital row
    const int32_t* orb_l;      // [n_el][16] l of each shell
    const int32_t* n_rows;     // [n_el]
    const int32_t* ent_range;  // [2][n_el][n_el][2] entry range of a block kind (0 diagonal, 1 off-diagonal) and element pair
    const int32_t* op_base;    // [2][n_el][n_el][16][16] first entry of a shell pair (entries run over L = |li-lj| .. li+lj)
    const int32_t* ent_col;    // [n_ent] output column of an entry
    const int32_t* ent_L;      // [n_ent]
    int n_el;
};

// irreps of entries [k0, k1) from one feature row X[25][F] after the output layer's self-mixing: sum_f X[L][m][f] W_L[c][f] (+ bias on L = 0)
__device__ __forceinline__ void asm_irreps(const float* __restrict__ X, const float* __restrict__ W, const float* __restrict__ bias, int n_col, int F, const AsmTables& t,
                           int k0, int k1, float* __restrict__ irr) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warp = blockDim.x >> 5;
    for (int k = k0 + warp; k < k1; k += n_warp) {
        const int c = t.ent_col[k], L = t.ent_L[k];
        const float* w = W + ((size_t)L * n_col + c) * F;
        for (int m = 0; m < 2 * L + 1; ++m) {
            const float* x = X + (size_t)(L * L + m) * F;
            float s = 0.f;
            for (int f = lane; f < F; f += 32) s = fmaf(__ldg(x + f), __ldg(w + f), s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) irr[(k - k0) * 9 + m] = s + (L == 0 ? __ldg(bias + c) : 0.f);
        }
    }
}

// B[p][q] = sum_{L, m} sqrt(2L+1) CG(li, lj, L)[mi][mj][m] irrep(shell(p), shell(q), L)[m]   (matrix_block, neural_network.py:636-660)
__device__ __forceinline__ void asm_block(const AsmTables& t, int kind, int ea, int eb, const float* __restrict__ irr, int k0, float* __restrict__ B) {
    const int na = t.n_rows[ea], nb = t.n_rows[eb];
    const int* base = t.op_base + (((size_t)kind * t.n_el + ea) * t.n_el + eb) * ASM_MAX_ORB * ASM_MAX_ORB;
    for (int pq = threadIdx.x; pq < na * nb; pq += blockDim.x) {
        const int p = pq / nb, q = pq % nb;
        const int si = t.row_orb[ea * ASM_MAX_ROWS + p], mi = t.row_m[ea * ASM_MAX_ROWS + p];
        const int sj = t.row_orb[eb * ASM_MAX_ROWS + q], mj = t.row_m[eb * ASM_MAX_ROWS + q];
        const int li = t.orb_l[ea * ASM_MAX_ORB + si], lj = t.orb_l[eb * ASM_MAX_ORB + sj];
        const int lo = li > lj ? li - lj : lj - li;
        const int k = base[si * ASM_MAX_ORB + sj] - k0;
        float v = 0.f;
        for (int L = lo; L <= li + lj; ++L) {
            const float* cg = c_phis_asm_cg + ((((li * 3 + lj) * 5 + L) * 5 + mi) * 5 + mj) * 9;
            const float* ir = irr + (k + L - lo) * 9;
            for (int m = 0; m < 2 * L + 1; ++m) v = fmaf(cg[m], ir[m], v);
        }
        B[p * (ASM_MAX_ROWS + 1) + q] = v;
    }
}

// CTA b < N: diagonal block of atom b.  CTA N + e: off-diagonal pair e = (i, j) with i < j (the CTA of (j, i) exits); it writes
// M_ij = B_ij + B_ji^T and its transpose M_ji, so each matrix is exactly symmetric and every element has one writer.
__global__ void __launch_bounds__(128, 1) k_assemble(const float* __restrict__ Xd, const float* __restrict__ Xo, const float* __restrict__ Wd,
                                                 const float* __restrict__ bd, int n_col_d, const float* __restrict__ Wo, const float* __restrict__ bo,
                                                 int n_col_o, int F, AsmTables t, const int32_t* __restrict__ tgt, const int32_t* __restrict__ col,
                                                 const int32_t* __restrict__ rev, int n_atoms, const int32_t* __restrict__ atom_mol,
                                                 const int32_t* __restrict__ atom_off, const int64_t* __restrict__ mol_off,
                                                 const int32_t* __restrict__ mol_norb, int unit_diagonal, int max_ent, float* __restrict__ M) {
    extern __shared__ float smem[];
    float* irr_a = smem;
    float* irr_b = irr_a + max_ent * 9;
    float* Ba = irr_b + max_ent * 9;
    float* Bb = Ba + ASM_MAX_ROWS * (ASM_MAX_ROWS + 1);
    const int b = blockIdx.x;
    int i, j, e = -1;
    if (b < n_atoms) {
        i = j = b;
    } else {
        e = b - n_atoms;
        i = tgt[e];
        j = col[e];
        if (i > j) return;
    }
    const int ea = t.atom_el[i], eb = t.atom_el[j], kind = e < 0 ? 0 : 1;
    const int* ra = t.ent_range + (((size_t)kind * t.n_el + ea) * t.n_el + eb) * 2;
    if (e < 0) {
        asm_irreps(Xd + (size_t)i * PLM * F, Wd, bd, n_col_d, F, t, ra[0], ra[1], irr_a);
    } else {
        const int* rb = t.ent_range + (((size_t)kind * t.n_el + eb) * t.n_el + ea) * 2;
        asm_irreps(Xo + (size_t)e * PLM * F, Wo, bo, n_col_o, F, t, ra[0], ra[1], irr_a);
        asm_irreps(Xo + (size_t)rev[e] * PLM * F, Wo, bo, n_col_o, F, t, rb[0], rb[1], irr_b);
    }
    __syncthreads();
    asm_block(t, kind, ea, eb, irr_a, ra[0], Ba);
    if (e >= 0) asm_block(t, kind, eb, ea, irr_b, t.ent_range[(((size_t)kind * t.n_el + eb) * t.n_el + ea) * 2], Bb);
    __syncthreads();
    const int na = t.n_rows[ea], nb = t.n_rows[eb], mol = atom_mol[i], n = mol_norb[mol];
    float* Mm = M + mol_off[mol];
    const int oi = atom_off[i], oj = atom_off[j];
    const int ld = ASM_MAX_ROWS + 1;
    for (int pq = threadIdx.x; pq < na * nb; pq += blockDim.x) {
        const int p = pq / nb, q = pq % nb;
        if (e < 0) {
            const float v = Ba[p * ld + q] + Ba[q * ld + p];
            Mm[(size_t)(oi + p) * n + oi + q] = (unit_diagonal && p == q) ? 1.f : v;
        } else {
            const float v = Ba[p * ld + q] + Bb[q * ld + p];
            Mm[(size_t)(oi + p) * n + oj + q] = v;
            Mm[(size_t)(oj + q) * n + oi + p] = v;
        }
    }
}

bool feat_ok(int F) { return F == 32 || F == 64 || F == 96 || F == 128; }

}  // namespace

extern "C" int nb200_phis_swish_self_mixing(const float* x, const float* alpha, const float* beta, const float* mixcoeff, const float* keepcoeff,
                                            int32_t n_rows, int32_t n_feat, float* y, void* stream) {
    if (!x || !mixcoeff || !keepcoeff || !y || n_rows < 0 || (!alpha != !beta)) return NB200_EINVAL;
    if (!feat_ok(n_feat)) return NB200_EUNSUPPORTED;
    if (n_rows == 0) return NB200_OK;
    k_swish_self_mix<<<n_rows, n_feat, 0, (cudaStream_t)stream>>>(x, alpha, beta, mixcoeff, keepcoeff, y);
    return nb_check_launch();
}

extern "C" int nb200_phis_linear_ex(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in, int32_t c_out, int32_t order,
                                    int32_t accumulate, float* y, void* stream) {
    if (!x || !W_l || !y || order < 0 || order > 4) return NB200_EINVAL;
    const int nc = (order + 1) * (order + 1);
    return nb_gemm_tf32x3_lm(n_rows, c_out, c_in, x, nc * c_in, W_l, (long long)c_in * c_out, y, nc * c_out, accumulate ? 1 : 0, bias, nc,
                             (cudaStream_t)stream);
}

extern "C" int nb200_phis_interaction(const float* yi, const float* yj, const float* sh, const float* coeff, const float* wa1, const float* ba1,
                                      const float* wa2, const float* ba2, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, int32_t n_feat,
                                      float* y, void* stream) {
    if (!yi || !yj || !sh || !coeff || !wa1 || !ba1 || !wa2 || !ba2 || !row_ptr || !col || !y || n_atoms < 0) return NB200_EINVAL;
    if (!feat_ok(n_feat)) return NB200_EUNSUPPORTED;
    if (n_atoms == 0) return NB200_OK;
    k_interaction<<<n_atoms, n_feat, 0, (cudaStream_t)stream>>>(yi, yj, sh, coeff, wa1, ba1, wa2, ba2, row_ptr, col, y);
    return nb_check_launch();
}

extern "C" int nb200_phis_pair_features(const float* fpc, const float* fpn, const float* coeff, const int32_t* row_ptr, const int32_t* col,
                                        int32_t n_atoms, int32_t n_feat, float* fii, float* fij, void* stream) {
    if (!fpc || !fpn || !coeff || !row_ptr || !col || !fii || !fij || n_atoms < 0) return NB200_EINVAL;
    if (!feat_ok(n_feat)) return NB200_EUNSUPPORTED;
    if (n_atoms == 0) return NB200_OK;
    k_pair_features<<<n_atoms, n_feat, PLM * n_feat * sizeof(float), (cudaStream_t)stream>>>(fpc, fpn, coeff, row_ptr, col, fii, fij);
    return nb_check_launch();
}

extern "C" int nb200_phis_overlap_pairs(const float* x, const float* sh, const float* coeff, const float* wa, const int32_t* row_ptr,
                                        const int32_t* col, int32_t n_atoms, int32_t n_feat, float* s, void* stream) {
    if (!x || !sh || !coeff || !wa || !row_ptr || !col || !s || n_atoms < 0) return NB200_EINVAL;
    if (!feat_ok(n_feat)) return NB200_EUNSUPPORTED;
    if (n_atoms == 0) return NB200_OK;
    k_overlap_pairs<<<n_atoms, n_feat, 0, (cudaStream_t)stream>>>(x, sh, coeff, wa, row_ptr, col, s);
    return nb_check_launch();
}

extern "C" int nb200_phis_assemble(const float* Xd, const float* Xo, const float* Wd, const float* bd, int32_t n_col_d, const float* Wo, const float* bo,
                                   int32_t n_col_o, int32_t n_feat, const int32_t* atom_el, const int32_t* row_orb, const int32_t* row_m,
                                   const int32_t* orb_l, const int32_t* n_rows, const int32_t* ent_range, const int32_t* op_base, const int32_t* ent_col,
                                   const int32_t* ent_L, int32_t n_el, int32_t max_ent, const int32_t* tgt, const int32_t* col, const int32_t* rev,
                                   int32_t n_atoms, int32_t n_pairs, const int32_t* atom_mol, const int32_t* atom_off, const int64_t* mol_off,
                                   const int32_t* mol_norb, int32_t unit_diagonal, float* M, void* stream) {
    if (!Xd || !Wd || !bd || !atom_el || !row_orb || !row_m || !orb_l || !n_rows || !ent_range || !op_base || !ent_col || !ent_L || !atom_mol ||
        !atom_off || !mol_off || !mol_norb || !M || n_atoms < 0 || n_pairs < 0 || n_el <= 0 || max_ent < 0)
        return NB200_EINVAL;
    if (n_pairs > 0 && (!Xo || !Wo || !bo || !tgt || !col || !rev)) return NB200_EINVAL;
    if (n_feat % 32 || n_feat <= 0) return NB200_EUNSUPPORTED;
    if (n_atoms == 0) return NB200_OK;
    const size_t smem = (2 * (size_t)max_ent * 9 + 2 * ASM_MAX_ROWS * (ASM_MAX_ROWS + 1)) * sizeof(float);
    if (smem > 227 * 1024) return NB200_EUNSUPPORTED;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k_assemble, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return nb_check_launch();
    AsmTables t{atom_el, row_orb, row_m, orb_l, n_rows, ent_range, op_base, ent_col, ent_L, n_el};
    k_assemble<<<n_atoms + n_pairs, 128, smem, (cudaStream_t)stream>>>(Xd, Xo, Wd, bd, n_col_d, Wo, bo, n_col_o, n_feat, t, tgt, col, rev, n_atoms,
                                                                      atom_mol, atom_off, mol_off, mol_norb, unit_diagonal, max_ent, M);
    return nb_check_launch();
}
