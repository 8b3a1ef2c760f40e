// qhnet.cu -- QHNet (config/model/qhnet.yaml) Hamiltonian-prediction kernels.
//
// Reference: nablaDFT/qhnet/qhnet.py + layers.py on top of e3nn 0.5.1 (SURVEY.md section 8 rows
// a12-a17, Appendix A.4).  Equivariant features live in HBM as [rows][25 (l,m)][C channels]
// ("component-major": channels contiguous), C = 128 (hidden) or 32 (bottle); one thread owns one
// channel, so every load is coalesced and the Clebsch-Gordan contractions run out of registers
// with the coefficients unrolled as literals (qhnet_tp_gen.inc, generated from oracle/e3.py).
//
// Graph convention (qhnet.py:254-264): `dst, src = radius_graph(...)`, edge_vec = pos[dst] - pos[src],
// messages flow src -> dst.  With our CSR (row = target t, col = source c, u = (pos[c]-pos[t])/d)
// the message INTO t from c is the reference edge (dst = t, src = c) whose vector is -d*u: every
// kernel below walks row t and uses sign = -1 for the spherical harmonics (Y_l(-v) = (-1)^l Y_l(v)).
// The full graph (radius 10000) is the same CSR with all n(n-1) pairs, in the reference's order
// (sorted by `src` = row owner, then `dst` = col), so pair index == CSR edge index.
#include "common.cuh"
#include "qhnet_tp_gen.inc"

#define QH_C 128
#define QH_LM 25
#define QH_B 32  // bottle channels

namespace {

__device__ __forceinline__ int l_of_lm(int lm) { return lm >= 16 ? 4 : lm >= 9 ? 3 : lm >= 4 ? 2 : lm >= 1 ? 1 : 0; }

__global__ void k_expand_rows(const int32_t* __restrict__ row_ptr, int n_atoms, int32_t* __restrict__ tgt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_atoms) return;
    for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) tgt[e] = i;
}

// ---- a12: exponential-Bernstein radial basis (layers.py:86-120) + real spherical harmonics l <= 4
// (qhnet.py:266-271: o3.spherical_harmonics(sh, edge_vec[:, [1,2,0]], normalize=True, 'component') ==
//  the standard z-polar real SH of edge_vec/|edge_vec| times sqrt(4 pi); oracle/e3.py::spherical_harmonics)
// The exponent logc_k + (K-1-k) x + k log(1 - e^x) sums terms of up to ~85 (logc at K = 128) that cancel to <= 0, so x, the log, logc and
// the sum are double; only the rounded exponent goes through expf.  In fp32 the basis was off by up to ~1e-5 of each row's largest value.
// The cutoff function's argument -d^2 / (c^2 - d^2) reaches -100 and beyond near the cutoff, where its fp32 rounding alone puts ~1e-5 on
// the whole row, so it is evaluated in double once per edge as well.
__global__ void __launch_bounds__(128) k_qh_edge_basis(const float* __restrict__ geom, const int32_t* __restrict__ status, double alpha,
                                                      float cutoff, float sign, const double* __restrict__ logc, int n_rbf,
                                                      float* __restrict__ rbf, float* __restrict__ sh) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (status[1] != 0 || e >= status[0]) return;
    const float4 g = ldg4(geom + 4 * (size_t)e);
    const float d = g.w;
    if (rbf) {
        const double x = -alpha * (double)d;
        const double lt = log(-expm1(x));
        float fc = 0.f;
        if (d < cutoff) {
            const double dd = d, c = cutoff;
            fc = (float)exp(-(dd * dd) / ((c - dd) * (c + dd)));
        }
        for (int k = 0; k < n_rbf; ++k)
            rbf[(size_t)e * n_rbf + k] = fc * expf((float)(__ldg(logc + k) + (double)(n_rbf - 1 - k) * x + (double)k * lt));
    }
    if (sh) {
        const float x = sign * g.x, y = sign * g.y, z = sign * g.z;
        const float x2 = x * x, y2 = y * y, z2 = z * z;
        float* o = sh + (size_t)e * QH_LM;
        o[0] = 1.0f;
        o[1] = 1.7320508075688772f * y; o[2] = 1.7320508075688772f * z; o[3] = 1.7320508075688772f * x;
        o[4] = 3.872983346207417f * x * y; o[5] = 3.872983346207417f * y * z; o[6] = 1.118033988749895f * (3.0f * z2 - 1.0f);
        o[7] = 3.872983346207417f * x * z; o[8] = 1.9364916731037085f * (x2 - y2);
        o[9] = 2.091650066335189f * y * (3.0f * x2 - y2); o[10] = 10.246950765959598f * x * y * z;
        o[11] = 1.620185174601965f * y * (5.0f * z2 - 1.0f); o[12] = 1.3228756555322954f * z * (5.0f * z2 - 3.0f);
        o[13] = 1.620185174601965f * x * (5.0f * z2 - 1.0f); o[14] = 5.123475382979799f * (x2 - y2) * z;
        o[15] = 2.091650066335189f * x * (x2 - 3.0f * y2);
        o[16] = 8.874119674649425f * x * y * (x2 - y2); o[17] = 6.274950199005566f * y * (3.0f * x2 - y2) * z;
        o[18] = 3.3541019662496847f * x * y * (7.0f * z2 - 1.0f); o[19] = 2.3717082451262845f * y * z * (7.0f * z2 - 3.0f);
        o[20] = 0.375f * (35.0f * z2 * z2 - 30.0f * z2 + 3.0f); o[21] = 2.3717082451262845f * x * z * (7.0f * z2 - 3.0f);
        o[22] = 1.6770509831248424f * (x2 - y2) * (7.0f * z2 - 1.0f); o[23] = 6.274950199005566f * x * (x2 - 3.0f * y2) * z;
        o[24] = 2.218529918662356f * (x2 * x2 - 6.0f * x2 * y2 + y2 * y2);
    }
}

// ---- NormGate (layers.py:123-147): f0 = [scalars, per-channel norms of l >= 1]; y = [gates0, x_l * gates_l]
__global__ void __launch_bounds__(QH_C) k_qh_norm_feats(const float* __restrict__ x, int n_rows, float* __restrict__ f0) {
    const int r = blockIdx.x, u = threadIdx.x;
    const float* xr = x + (size_t)r * QH_LM * QH_C + u;
    float* fr = f0 + (size_t)r * 5 * QH_C + u;
    fr[0] = xr[0];
    int lm = 1;
#pragma unroll
    for (int l = 1; l <= 4; ++l) {
        float s = 0.f;
        for (int m = 0; m < 2 * l + 1; ++m, ++lm) { const float v = xr[lm * QH_C]; s = fmaf(v, v, s); }
        fr[l * QH_C] = sqrtf(fmaxf(s, 0.f));
    }
}

__global__ void __launch_bounds__(QH_C) k_qh_gate(const float* __restrict__ x, const float* __restrict__ gates, int n_rows, float* __restrict__ y) {
    const int r = blockIdx.x, u = threadIdx.x;
    const float* xr = x + (size_t)r * QH_LM * QH_C + u;
    const float* gr = gates + (size_t)r * 5 * QH_C + u;
    float* yr = y + (size_t)r * QH_LM * QH_C + u;
    yr[0] = gr[0];
    for (int lm = 1; lm < QH_LM; ++lm) yr[lm * QH_C] = xr[lm * QH_C] * gr[l_of_lm(lm) * QH_C];
}

// ---- invariant edge features fed to the weight MLPs (layers.py:237-259, 469-476)
// mode 0: conv layers >= 1 : [f[t][0], f[t][0], <f[t], f[c]>_l / (2l+1), l = 1..4]      -> 768  (dst scalars twice)
// mode 1: conv layer 0     : [f[t], f[t]]  (f = [N,128] scalars only)                    -> 256
// mode 2: pair layer       : [f[c][0], f[t][0], <f[c], f[t]>_l / (2l+1)]                 -> 768  (dst = col, src = row owner)
__global__ void __launch_bounds__(QH_C) k_qh_invariants(const float* __restrict__ f, const int32_t* __restrict__ tgt,
                                                       const int32_t* __restrict__ col, const int32_t* __restrict__ status, int mode,
                                                       float* __restrict__ out) {
    const int e = blockIdx.x, u = threadIdx.x;
    if (status[1] != 0 || e >= status[0]) return;
    const int t = tgt[e], c = col[e];
    if (mode == 1) {
        const float v = f[(size_t)t * QH_C + u];
        out[(size_t)e * 2 * QH_C + u] = v;
        out[(size_t)e * 2 * QH_C + QH_C + u] = v;
        return;
    }
    const float* ft = f + (size_t)t * QH_LM * QH_C + u;
    const float* fcn = f + (size_t)c * QH_LM * QH_C + u;
    float* o = out + (size_t)e * 6 * QH_C + u;
    o[0] = mode == 0 ? ft[0] : fcn[0];
    o[QH_C] = ft[0];
    int lm = 1;
#pragma unroll
    for (int l = 1; l <= 4; ++l) {
        float s = 0.f;
        for (int m = 0; m < 2 * l + 1; ++m, ++lm) s = fmaf(ft[lm * QH_C], fcn[lm * QH_C], s);
        o[(l + 1) * QH_C] = s / (float)(2 * l + 1);
    }
}

// ---- a13: ConvLayer message + aggregation (layers.py:263-271): one CTA per target atom, thread = channel
//   out[t] = sum_{e in row t} TP_uvu(x[col e], Y_e, w1_e * w2_e)  (+ x[t] when in == out irreps)
template <bool LAYER0>
__global__ void __launch_bounds__(QH_C) k_qh_tp_conv(const float* __restrict__ x, const float* __restrict__ sh, const float* __restrict__ w1,
                                                    const float* __restrict__ w2, const int32_t* __restrict__ row_ptr,
                                                    const int32_t* __restrict__ col, int add_self, float* __restrict__ out) {
    const int t = blockIdx.x, u = threadIdx.x;
    float o[QH_LM];
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) o[k] = 0.f;
    constexpr int NW = LAYER0 ? QH_CONV0_WEIGHTS : QH_CONV_WEIGHTS;
    for (int e = row_ptr[t]; e < row_ptr[t + 1]; ++e) {
        const int c = col[e];
        float a[QH_LM], b[QH_LM];
#pragma unroll
        for (int k = 0; k < QH_LM; ++k) b[k] = __ldg(sh + (size_t)e * QH_LM + k);
        if (LAYER0) {
            a[0] = __ldg(x + (size_t)c * QH_C + u);
#pragma unroll
            for (int k = 1; k < QH_LM; ++k) a[k] = 0.f;
            qh_tp_conv0(a, b, w1 + (size_t)e * NW + u, w2 + (size_t)e * NW + u, QH_C, o);
        } else {
#pragma unroll
            for (int k = 0; k < QH_LM; ++k) a[k] = __ldg(x + ((size_t)c * QH_LM + k) * QH_C + u);
            qh_tp_conv(a, b, w1 + (size_t)e * NW + u, w2 + (size_t)e * NW + u, QH_C, o);
        }
    }
    float* ot = out + (size_t)t * QH_LM * QH_C + u;
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) ot[k * QH_C] = o[k] + ((add_self && !LAYER0) ? __ldg(x + ((size_t)t * QH_LM + k) * QH_C + u) : 0.f);
}

// ---- a14: PairNetLayer tensor product (layers.py:481-485): pair p = (src = row owner t, dst = col c)
//   out[p] = TP_uuu(x[src], x[dst], w1_p * w2_p)
__global__ void __launch_bounds__(QH_C) k_qh_tp_pair(const float* __restrict__ x, const float* __restrict__ w1, const float* __restrict__ w2,
                                                    const int32_t* __restrict__ tgt, const int32_t* __restrict__ col,
                                                    const int32_t* __restrict__ status, float* __restrict__ out) {
    const int p = blockIdx.x, u = threadIdx.x;
    if (status[1] != 0 || p >= status[0]) return;
    const int t = tgt[p], c = col[p];
    float a[QH_LM], b[QH_LM], o[QH_LM];
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) {
        a[k] = __ldg(x + ((size_t)t * QH_LM + k) * QH_C + u);
        b[k] = __ldg(x + ((size_t)c * QH_LM + k) * QH_C + u);
        o[k] = 0.f;
    }
    qh_tp_uuu2(a, b, w1 + (size_t)p * QH_UUU_WEIGHTS + u, w2 + (size_t)p * QH_UUU_WEIGHTS + u, QH_C, o);
    float* op = out + (size_t)p * QH_LM * QH_C + u;
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) op[k * QH_C] = o[k];
}

// ---- a15: SelfNetLayer tensor product with internal (shared) weights (layers.py:546-553,571-573)
//   out[n] = TP_uuu(xl[n], xr[n], w) + res[n]
__global__ void __launch_bounds__(QH_C) k_qh_tp_self(const float* __restrict__ xl, const float* __restrict__ xr, const float* __restrict__ w,
                                                    const float* __restrict__ res, float* __restrict__ out) {
    const int n = blockIdx.x, u = threadIdx.x;
    float a[QH_LM], b[QH_LM], o[QH_LM];
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) {
        a[k] = __ldg(xl + ((size_t)n * QH_LM + k) * QH_C + u);
        b[k] = __ldg(xr + ((size_t)n * QH_LM + k) * QH_C + u);
        o[k] = 0.f;
    }
    qh_tp_uuu1(a, b, w + u, QH_C, o);
    float* on = out + (size_t)n * QH_LM * QH_C + u;
#pragma unroll
    for (int k = 0; k < QH_LM; ++k) on[k * QH_C] = o[k] + (res ? __ldg(res + ((size_t)n * QH_LM + k) * QH_C + u) : 0.f);
}

// ---- a16: Expansion (layers.py:598-662): bottle features [R][25][32] + per-row path weights [R][8320] and
// biases [R][50] -> 32 x 32 block (5 s, 4 p, 3 d shells).  One warp per row, lane = input channel w.
// instruction table (l_in, l1, l2, weight offset, bias offset) in the reference's loop order; w3j(l1,l2,l_in).
struct ExpIns { int lin, l1, l2, woff, boff; };
__constant__ ExpIns c_exp_ins[19];
__constant__ float c_exp_cg[19 * 5 * 5 * 9];  // [ins][i][j][k], zero padded, already divided by mul_in = 32

template <int WARPS>
__global__ void __launch_bounds__(32 * WARPS) k_qh_expand(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ Bw,
                                                  int bw_stride, int n_rows, float* __restrict__ blocks) {
    // v1 had lane = input channel w and warp-reduced every (u,v,k): 5 k shuffles per row and 4-byte loads strided by
    // n1*n2.  v2: lane = (u,v)
    // entry of the instruction's weight slab, serial loop over w: the slab rows W[w][.][.] are contiguous (coalesced,
    // read once), x[w][k] is a shared-memory broadcast, no shuffles, and each lane owns its (u,v) sub-block of the tile.
    __shared__ float sblk[WARPS][32 * 32];
    __shared__ float sx[WARPS][QH_LM * QH_B];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * WARPS + warp;
    if (r >= n_rows) return;
    float* blk = sblk[warp];
    float* xs = sx[warp];
    const float* Wr = W + (size_t)r * 8320;
    for (int t = lane; t < 1024; t += 32) blk[t] = 0.f;
    for (int t = lane; t < QH_LM * QH_B; t += 32) xs[t] = __ldg(x + (size_t)r * QH_LM * QH_B + t);  // [lm][w]
    const float* Br = Bw + (size_t)r * bw_stride;
    __syncwarp();
    for (int ins = 0; ins < 19; ++ins) {
        const ExpIns I = c_exp_ins[ins];
        const int n1 = (I.l1 == 0) ? 5 : (I.l1 == 1) ? 4 : 3, n2 = (I.l2 == 0) ? 5 : (I.l2 == 1) ? 4 : 3;
        const int o1 = (I.l1 == 0) ? 0 : (I.l1 == 1) ? 5 : 17, o2 = (I.l2 == 0) ? 0 : (I.l2 == 1) ? 5 : 17;
        const int d1 = 2 * I.l1 + 1, d2 = 2 * I.l2 + 1, dk = 2 * I.lin + 1, nuv = n1 * n2;
        if (lane < nuv) {
            float rk[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) rk[k] = 0.f;
            const float* wp = Wr + I.woff + lane;
            const float* xk = xs + I.lin * I.lin * QH_B;
#pragma unroll 4
            for (int w = 0; w < QH_B; ++w) {
                const float wv = __ldg(wp + w * nuv);
#pragma unroll
                for (int k = 0; k < 9; ++k)
                    if (k < dk) rk[k] = fmaf(wv, xk[k * QH_B + w], rk[k]);
            }
            if (I.lin == 0) rk[0] += __ldg(Br + I.boff + lane);
            const int u = lane / n2, v = lane - u * n2;
            const float* cg = c_exp_cg + ins * 225;
            float* tile = blk + (o1 + u * d1) * 32 + o2 + v * d2;
            for (int i = 0; i < d1; ++i)
                for (int j = 0; j < d2; ++j) {
                    float acc = 0.f;
#pragma unroll
                    for (int k = 0; k < 9; ++k)
                        if (k < dk) acc = fmaf(cg[(i * 5 + j) * 9 + k], rk[k], acc);
                    tile[i * 32 + j] += acc;
                }
        }
        __syncwarp();
    }
    float* ob = blocks + (size_t)r * 1024;
    for (int t = lane; t < 1024; t += 32) ob[t] = blk[t];
}

// ---- a17: build_final_matrix + H + H^T (qhnet.py:293-321, 234-238).  One CTA per atom pair / atom:
// H_mol[orb(a) + i, orb(b) + j] = blk(dst=a,src=b)[mask_a[i], mask_b[j]] + blk(dst=b,src=a)[mask_b[j], mask_a[i]]
__global__ void __launch_bounds__(256) k_qh_assemble(const float* __restrict__ diag, const float* __restrict__ offd, const int32_t* __restrict__ z,
                                                    const int32_t* __restrict__ tgt, const int32_t* __restrict__ col, const int32_t* __restrict__ rev,
                                                    int n_atoms, int n_pairs, const int32_t* __restrict__ mask_tab, const int32_t* __restrict__ norb_tab,
                                                    const int32_t* __restrict__ atom_mol, const int32_t* __restrict__ atom_orb_off,
                                                    const int64_t* __restrict__ mol_h_off, const int32_t* __restrict__ mol_norb,
                                                    float* __restrict__ H) {
    const int b = blockIdx.x;
    int a_atom, b_atom;
    const float *blk_ab, *blk_ba;
    if (b < n_atoms) {
        a_atom = b_atom = b;
        blk_ab = blk_ba = diag + (size_t)b * 1024;
    } else {
        const int p = b - n_atoms;
        if (p >= n_pairs) return;
        a_atom = col[p];  // dst = row block
        b_atom = tgt[p];  // src = column block
        blk_ab = offd + (size_t)p * 1024;
        blk_ba = offd + (size_t)rev[p] * 1024;
    }
    const int za = z[a_atom], zb = z[b_atom];
    const int na = norb_tab[za], nb = norb_tab[zb];
    const int m = atom_mol[a_atom];
    const int ld = mol_norb[m];
    float* Hm = H + mol_h_off[m];
    const int ra = atom_orb_off[a_atom], cb = atom_orb_off[b_atom];
    for (int t = threadIdx.x; t < na * nb; t += blockDim.x) {
        const int i = t / nb, j = t % nb;
        const int mi = mask_tab[za * 32 + i], mj = mask_tab[zb * 32 + j];
        Hm[(size_t)(ra + i) * ld + cb + j] = blk_ab[mi * 32 + mj] + blk_ba[mj * 32 + mi];
    }
}

// hidden layer of fc_ij / fc_ij_bias (qhnet.py:227-232): silu(W [e_dst ; e_src] + b) without materialising the
// [P,256] concatenation: A = emb W[:, :128]^T and Bn = emb W[:, 128:]^T are per-atom, gathered per pair.
__global__ void __launch_bounds__(QH_C) k_qh_pair_hidden(const float* __restrict__ A, const float* __restrict__ Bn, const float* __restrict__ bias,
                                                        const int32_t* __restrict__ tgt, const int32_t* __restrict__ col,
                                                        const int32_t* __restrict__ status, float* __restrict__ h) {
    const int p = blockIdx.x, u = threadIdx.x;
    if (status[1] != 0 || p >= status[0]) return;
    const float v = A[(size_t)col[p] * QH_C + u] + Bn[(size_t)tgt[p] * QH_C + u] + bias[u];  // dst = col, src = row owner
    h[(size_t)p * QH_C + u] = siluf_(v);
}

__global__ void k_axpy(float* __restrict__ y, const float* __restrict__ x, int64_t n4) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n4) return;
    st4(y + 4 * t, *reinterpret_cast<const float4*>(y + 4 * t) + ldg4(x + 4 * t));
}

}  // namespace

// -------------------------------------------------------------------------------------------- C ABI
extern "C" int nb200_qh_expand_rows(const int32_t* row_ptr, int32_t n_atoms, int32_t* tgt, void* stream) {
    if (!row_ptr || !tgt || n_atoms < 0) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    k_expand_rows<<<(n_atoms + 127) / 128, 128, 0, (cudaStream_t)stream>>>(row_ptr, n_atoms, tgt);
    return nb_check_launch();
}

extern "C" int nb200_qh_edge_basis(const float* geom, const int32_t* status, int32_t e_cap, double alpha, float cutoff, float sign,
                                   const double* logc, int32_t n_rbf, float* rbf, float* sh, void* stream) {
    if (!geom || !status || e_cap < 0 || (rbf && !logc)) return NB200_EINVAL;
    if (e_cap == 0) return NB200_OK;
    k_qh_edge_basis<<<(e_cap + 127) / 128, 128, 0, (cudaStream_t)stream>>>(geom, status, alpha, cutoff, sign, logc, n_rbf, rbf, sh);
    return nb_check_launch();
}

extern "C" int nb200_qh_norm_feats(const float* x, int32_t n_rows, float* f0, void* stream) {
    if (!x || !f0 || n_rows < 0) return NB200_EINVAL;
    if (n_rows == 0) return NB200_OK;
    k_qh_norm_feats<<<n_rows, QH_C, 0, (cudaStream_t)stream>>>(x, n_rows, f0);
    return nb_check_launch();
}

extern "C" int nb200_qh_gate(const float* x, const float* gates, int32_t n_rows, float* y, void* stream) {
    if (!x || !gates || !y || n_rows < 0) return NB200_EINVAL;
    if (n_rows == 0) return NB200_OK;
    k_qh_gate<<<n_rows, QH_C, 0, (cudaStream_t)stream>>>(x, gates, n_rows, y);
    return nb_check_launch();
}

extern "C" int nb200_qh_invariants(const float* f, const int32_t* tgt, const int32_t* col, const int32_t* status, int32_t e_cap, int32_t mode,
                                   float* out, void* stream) {
    if (!f || !tgt || !col || !status || !out || e_cap < 0 || mode < 0 || mode > 2) return NB200_EINVAL;
    if (e_cap == 0) return NB200_OK;
    k_qh_invariants<<<e_cap, QH_C, 0, (cudaStream_t)stream>>>(f, tgt, col, status, mode, out);
    return nb_check_launch();
}

extern "C" int nb200_qh_tp_conv(const float* x, const float* sh, const float* w1, const float* w2, const int32_t* row_ptr, const int32_t* col,
                                int32_t n_atoms, int32_t layer0, int32_t add_self, float* out, void* stream) {
    if (!x || !sh || !w1 || !w2 || !row_ptr || !col || !out || n_atoms < 0) return NB200_EINVAL;
    if (n_atoms == 0) return NB200_OK;
    if (layer0) k_qh_tp_conv<true><<<n_atoms, QH_C, 0, (cudaStream_t)stream>>>(x, sh, w1, w2, row_ptr, col, add_self, out);
    else k_qh_tp_conv<false><<<n_atoms, QH_C, 0, (cudaStream_t)stream>>>(x, sh, w1, w2, row_ptr, col, add_self, out);
    return nb_check_launch();
}

extern "C" int nb200_qh_tp_pair(const float* x, const float* w1, const float* w2, const int32_t* tgt, const int32_t* col, const int32_t* status,
                                int32_t p_cap, float* out, void* stream) {
    if (!x || !w1 || !w2 || !tgt || !col || !status || !out || p_cap < 0) return NB200_EINVAL;
    if (p_cap == 0) return NB200_OK;
    k_qh_tp_pair<<<p_cap, QH_C, 0, (cudaStream_t)stream>>>(x, w1, w2, tgt, col, status, out);
    return nb_check_launch();
}

extern "C" int nb200_qh_tp_self(const float* xl, const float* xr, const float* w, const float* res, int32_t n_rows, float* out, void* stream) {
    if (!xl || !xr || !w || !out || n_rows < 0) return NB200_EINVAL;
    if (n_rows == 0) return NB200_OK;
    k_qh_tp_self<<<n_rows, QH_C, 0, (cudaStream_t)stream>>>(xl, xr, w, res, out);
    return nb_check_launch();
}

// o3.Linear over the 25 (l,m) rows: y[r][lm][:] = x[r][lm][:] . W_l (+ bias on lm = 0).  W_l: [5][c_in][c_out],
// already scaled by 1/sqrt(c_in) on export.  c_in must be a multiple of 32 (wgmma GEMM k-chunk).
extern "C" int nb200_qh_linear(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in, int32_t c_out, int32_t accumulate,
                               float* y, void* stream) {
    if (!x || !W_l || !y) return NB200_EINVAL;
    return nb_gemm_tf32x3_lm(n_rows, c_out, c_in, x, QH_LM * c_in, W_l, (long long)c_in * c_out, y, QH_LM * c_out, accumulate, bias, QH_LM,
                             (cudaStream_t)stream);
}

// generic fp32-accurate dense layer with an activation kind (0 silu, 1 ssp, 2 normalize2mom(ssp))
extern "C" int nb200_dense(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb, int32_t trans_b, float* C,
                           int32_t ldc, int32_t accumulate, const float* bias, float* act, int32_t act_kind, void* stream) {
    return nb_gemm_tf32x3_ex(M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, act, act_kind, (cudaStream_t)stream);
}

extern "C" int nb200_qh_expand_setup(const int32_t* ins_host, const float* cg_host) {
    if (!ins_host || !cg_host) return NB200_EINVAL;
    if (cudaMemcpyToSymbol(c_exp_ins, ins_host, sizeof(ExpIns) * 19) != cudaSuccess) return nb_check_launch();
    if (cudaMemcpyToSymbol(c_exp_cg, cg_host, sizeof(float) * 19 * 225) != cudaSuccess) return nb_check_launch();
    return NB200_OK;
}

extern "C" int nb200_qh_expand(const float* x, const float* W, const float* Bw, int32_t bw_stride, int32_t n_rows, float* blocks, void* stream) {
    if (!x || !W || !Bw || !blocks || n_rows < 0 || bw_stride < 50) return NB200_EINVAL;
    if (n_rows == 0) return NB200_OK;
    k_qh_expand<4><<<(n_rows + 3) / 4, 128, 0, (cudaStream_t)stream>>>(x, W, Bw, bw_stride, n_rows, blocks);
    return nb_check_launch();
}

extern "C" int nb200_qh_assemble(const float* diag, const float* offd, const int32_t* z, const int32_t* tgt, const int32_t* col, const int32_t* rev,
                                 int32_t n_atoms, int32_t n_pairs, const int32_t* mask_tab, const int32_t* norb_tab, const int32_t* atom_mol,
                                 const int32_t* atom_orb_off, const int64_t* mol_h_off, const int32_t* mol_norb, float* H, void* stream) {
    if (!diag || !offd || !z || !tgt || !col || !rev || !mask_tab || !norb_tab || !atom_mol || !atom_orb_off || !mol_h_off || !mol_norb || !H)
        return NB200_EINVAL;
    if (n_atoms + n_pairs == 0) return NB200_OK;
    k_qh_assemble<<<n_atoms + n_pairs, 256, 0, (cudaStream_t)stream>>>(diag, offd, z, tgt, col, rev, n_atoms, n_pairs, mask_tab, norb_tab, atom_mol,
                                                                      atom_orb_off, mol_h_off, mol_norb, H);
    return nb_check_launch();
}

extern "C" int nb200_qh_pair_hidden(const float* A, const float* Bn, const float* bias, const int32_t* tgt, const int32_t* col,
                                    const int32_t* status, int32_t p_cap, float* h, void* stream) {
    if (!A || !Bn || !bias || !tgt || !col || !status || !h || p_cap < 0) return NB200_EINVAL;
    if (p_cap == 0) return NB200_OK;
    k_qh_pair_hidden<<<p_cap, QH_C, 0, (cudaStream_t)stream>>>(A, Bn, bias, tgt, col, status, h);
    return nb_check_launch();
}

extern "C" int nb200_axpy(float* y, const float* x, int64_t n, void* stream) {
    if (!y || !x || n < 0 || n % 4) return NB200_EINVAL;
    if (n == 0) return NB200_OK;
    k_axpy<<<(int)((n / 4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(y, x, n / 4);
    return nb_check_launch();
}
