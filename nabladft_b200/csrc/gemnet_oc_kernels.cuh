// gemnet_oc_kernels.cuh -- constants and kernel functors of the GemNet-OC engines (gemnet_oc.cu: inference, gemnet_oc_train.cu: training).
// See gemnet_oc.cu for the design notes; every functor is launched through pfor() (gemnet_pf.cuh) and also compiles for host emulation.
#pragma once
#include "gemnet_pf.cuh"

namespace {


constexpr int EA = 256, EE = 512, TI = 64, QI = 32, RB = 16, NR = 128, NS = 7, NS2 = 49;
constexpr int LD_MAIN = 1920, LD_AE = 128, LD_Q = 128, LD_A2A = 64;
constexpr int C_RBF_QINT = 0, C_RBF_EAINT = 16, C_RBF_TINT = 32, C_RBF_H = 48, C_RBF_OUT = 64, C_R_TINT = 80, C_R_AEINT = 192, C_R_SBF = 304;
constexpr int C_AE_RBF = 0, C_AE_R = 16;
constexpr int32_t RANK_NONE = 0x3fffffff;
constexpr float ISQ2 = 0.70710678118654752440f, ISQ3 = 0.57735026918962576451f;

GD float ssilu(float x) { return x / (1.0f + expf(-x)) * (1.0f / 0.6f); }  // base_layers.py:66-75
GD float clamp1(float x) { return fminf(1.0f, fmaxf(-1.0f, x)); }
GD float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
GD void cross3(const float* a, const float* b, float* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
// Y_l0(z) = sqrt((2l+1)/(4 pi)) P_l(z), l = 0..6 (basis.py:84-106,273-295 with zero_m_only)
GD void cir7(float z, float* Y) {
    float p0 = 1.0f, p1 = z;
    Y[0] = 0.28209479177387814f;
    Y[1] = 0.4886025119029199f * z;
    const float c[5] = {0.6307831305050401f, 0.7463526651802308f, 0.8462843753216345f, 0.9356025796273888f, 1.0171072362820548f};
#pragma unroll
    for (int l = 1; l < 6; l++) {
        const float p2 = ((2 * l + 1) * z * p1 - l * p0) / (float)(l + 1);
        Y[l + 1] = c[l - 1] * p2;
        p0 = p1;
        p1 = p2;
    }
}

// ------------------------------------------------------------------ graph construction
struct MolIdK {
    const int32_t* mol_ptr; int32_t n_mol; int32_t* mol_id;
    GD void operator()(int64_t a) const {
        int lo = 0, hi = n_mol;  // largest m with mol_ptr[m] <= a
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (mol_ptr[mid] <= (int32_t)a) lo = mid; else hi = mid;
        }
        mol_id[a] = lo;
    }
};
// rank[a, jl]: position of source j = mol_start + jl among the in-cutoff neighbours of target a, nearest first (ties: lower index first;
// utils.get_max_neighbors_mask, utils.py:408-500).  RANK_NONE for j == a, padding slots and pairs outside the cutoff.
struct RankK {
    const float* pos; const int32_t* mol_ptr; const int32_t* mol_id; int32_t Mx; float cut2; int32_t* rank;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / Mx), jl = (int32_t)(i % Mx);
        const int32_t m0 = mol_ptr[mol_id[a]], nm = mol_ptr[mol_id[a] + 1] - m0, j = m0 + jl;
        if (jl >= nm || j == a) { rank[i] = RANK_NONE; return; }
        const float ax = pos[3 * a], ay = pos[3 * a + 1], az = pos[3 * a + 2];
        float dx = pos[3 * j] - ax, dy = pos[3 * j + 1] - ay, dz = pos[3 * j + 2] - az;
        const float d2 = dx * dx + dy * dy + dz * dz;
        if (!(d2 < cut2)) { rank[i] = RANK_NONE; return; }
        const float d = sqrtf(d2);
        int32_t r = 0;
        for (int32_t k = m0; k < m0 + nm; k++) {
            if (k == a) continue;
            dx = pos[3 * k] - ax; dy = pos[3 * k + 1] - ay; dz = pos[3 * k + 2] - az;
            const float e2 = dx * dx + dy * dy + dz * dz;
            if (!(e2 < cut2)) continue;
            const float dk = sqrtf(e2);
            r += (dk < d || (dk == d && k < j)) ? 1 : 0;
        }
        rank[i] = r;
    }
};
// membership of the pair (target a, source j) in the four graphs
struct PairSel {
    const int32_t* rank; int32_t Mx, Kmain, Kae, Kq;
    GD void get(int32_t a, int32_t j, int32_t m0, bool& a2a, bool& mn, bool& ae, bool& q) const {
        const int32_t r = rank[(int64_t)a * Mx + (j - m0)];
        a2a = r != RANK_NONE;
        ae = r < Kae;
        q = r < Kq;
        // symmetrised main graph (gemnet_oc.py:694-775): the pair survives iff its source<target copy is among the target's nearest Kmain
        mn = j < a ? r < Kmain : rank[(int64_t)j * Mx + (a - m0)] < Kmain;
    }
};
struct DegK {
    PairSel sel; const int32_t* mol_ptr; const int32_t* mol_id; int32_t n; int32_t* deg;  // deg[4][n]: a2a, main, ae, q
    GD void operator()(int64_t a) const {
        const int32_t m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        int32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
        for (int32_t j = m0; j < m1; j++) {
            if (j == (int32_t)a) continue;
            bool x0, x1, x2, x3;
            sel.get((int32_t)a, j, m0, x0, x1, x2, x3);
            c0 += x0; c1 += x1; c2 += x2; c3 += x3;
        }
        deg[a] = c0; deg[n + a] = c1; deg[2 * (int64_t)n + a] = c2; deg[3 * (int64_t)n + a] = c3;
    }
};
// slots for the input triplets (d->b, b->a) of the quadruplet interaction: one per (qint edge b->a, main edge into b)
struct TcountK {
    PairSel sel; const int32_t* mol_ptr; const int32_t* mol_id; const int32_t* deg_main; int32_t* tcnt;
    GD void operator()(int64_t a) const {
        const int32_t m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        int32_t t = 0;
        for (int32_t j = m0; j < m1; j++) {
            if (j == (int32_t)a) continue;
            bool x0, x1, x2, x3;
            sel.get((int32_t)a, j, m0, x0, x1, x2, x3);
            if (x3) t += deg_main[j];
        }
        tcnt[a] = t;
    }
};
struct Graph {  // CSR by target, sources ascending; V = unit vector source -> target (gemnet_oc.py:820-868: -(pos[src]-pos[tgt])/d)
    const int32_t* ptr; int32_t* src; int32_t* tgt; float* d; float* V;
};
struct FillK {
    PairSel sel; const float* pos; const int32_t* mol_ptr; const int32_t* mol_id; const int32_t* deg_main; const int32_t* tbase;
    int32_t n; Graph a2a, mn, ae, q; int32_t* q_tin;
    const int32_t* err;  // asynchronous forward: status word 1; non-zero (a count above its bound, ...) = write nothing.  nullptr otherwise
    GD void put(const Graph& g, int32_t e, int32_t a, int32_t j, float d, const float* v) const {
        g.src[e] = j;
        if (g.tgt) g.tgt[e] = a;
        g.d[e] = d;
        if (g.V) { g.V[3 * (int64_t)e] = v[0]; g.V[3 * (int64_t)e + 1] = v[1]; g.V[3 * (int64_t)e + 2] = v[2]; }
    }
    GD void operator()(int64_t ai) const {
        if (err && *err) return;
        const int32_t a = (int32_t)ai, m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        int32_t e0 = a2a.ptr[a], e1 = mn.ptr[a], e2 = ae.ptr[a], e3 = q.ptr[a], tt = tbase[a];
        for (int32_t j = m0; j < m1; j++) {
            if (j == a) continue;
            bool x0, x1, x2, x3;
            sel.get(a, j, m0, x0, x1, x2, x3);
            if (!(x0 || x1)) continue;
            float v[3] = {pos[3 * a] - pos[3 * j], pos[3 * a + 1] - pos[3 * j + 1], pos[3 * a + 2] - pos[3 * j + 2]};
            const float d = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            v[0] /= d; v[1] /= d; v[2] /= d;
            if (x0) put(a2a, e0++, a, j, d, v);
            if (x1) put(mn, e1++, a, j, d, v);
            if (x2) put(ae, e2++, a, j, d, v);
            if (x3) { q_tin[e3] = tt; tt += deg_main[j]; put(q, e3++, a, j, d, v); }
        }
        if (a == n - 1) q_tin[q.ptr[n]] = tbase[n];
    }
};
// ------------------------------------------------------------------ status of the asynchronous forward (nb200_gemnet_oc_energy_forces_async)
// status[8] (zeroed before): {main-graph edges, error code, max main-graph degree, atoms without a main-graph neighbour, a2a edges, a2ee2a
// edges, qint edges, input-triplet slots}.  Words 0-3 read like the PaiNN engine's status.
GD bool finite_f(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    return (u & 0x7f800000u) != 0x7f800000u;
}
GD float quiet_nan() {
    const uint32_t u = 0x7fc00000u;
    float x;
    memcpy(&x, &u, 4);
    return x;
}
struct StatusAtomK {
    const float* pos; const int32_t* deg_main; int32_t* status;
    GD void operator()(int64_t a) const {
        // a non-finite coordinate fails every `d2 < cutoff^2` test of RankK, so the atom silently loses all its edges: report it instead
        if (!(finite_f(pos[3 * a]) && finite_f(pos[3 * a + 1]) && finite_f(pos[3 * a + 2]))) atomicMin(status + 1, (int32_t)NB200_EINVAL);
        const int32_t d = deg_main[a];
        atomicMax(status + 2, d);
        if (d == 0) atomicAdd(status + 3, 1);
    }
};
struct StatusCountsK {  // one thread, after StatusAtomK: the five counts against their bounds
    const int32_t* ptr; const int32_t* tbase; int32_t n; int32_t bound[5]; int32_t* status;
    GD void operator()(int64_t) const {
        const int32_t c[5] = {ptr[n], ptr[(int64_t)(n + 1) + n], ptr[2 * (int64_t)(n + 1) + n], ptr[3 * (int64_t)(n + 1) + n], tbase[n]};
        bool over = false;
        for (int k = 0; k < 5; k++) over = over || c[k] < 0 || c[k] > bound[k];  // < 0: int32 overflow of the scan
        status[0] = c[NB200_GOC_C_MAIN];
        status[4] = c[NB200_GOC_C_A2A]; status[5] = c[NB200_GOC_C_AE]; status[6] = c[NB200_GOC_C_Q]; status[7] = c[NB200_GOC_C_TIN];
        if (status[1] == 0) status[1] = over ? NB200_ECAPACITY : (c[NB200_GOC_C_MAIN] == 0 ? NB200_ENOEDGES : NB200_OK);
    }
};
// after an error every CSR row and every count becomes empty: no later kernel indexes an edge array (FillK wrote none)
struct ClearOnErrorK {
    const int32_t* status; int32_t* ptr; int64_t n_ptr; int32_t* tbase;
    GD void operator()(int64_t i) const {
        if (status[1] == 0) return;
        if (i < n_ptr) ptr[i] = 0; else tbase[i - n_ptr] = 0;
    }
};
struct NanOnErrorK {
    const int32_t* status; float* energy; int64_t n_mol; float* forces;
    GD void operator()(int64_t i) const {
        if (status[1] == 0) return;
        if (i < n_mol) energy[i] = quiet_nan(); else forces[i - n_mol] = quiet_nan();
    }
};
struct RevK {  // id_swap: position of the edge (t -> s) for every edge (s -> t)
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; int32_t* rev;
    GD void operator()(int64_t e) const {
        const int32_t s = src[e], t = tgt[e];
        int32_t r = -1;
        for (int32_t k = ptr[s]; k < ptr[s + 1]; k++)
            if (src[k] == t) r = k;
        rev[e] = r;
    }
};

// ------------------------------------------------------------------ bases
// unscaled radial basis: polynomial envelope (p = 5) x Gaussian smearing of d / cutoff (radial_basis.py:19-39,57-77,176-220)
struct RbfK {
    const float* d; const float* offset; float inv_cut, coeff; float* out;
    GD void operator()(int64_t i) const {
        const int64_t e = i / NR; const int r = (int)(i % NR);
        const float x = d[e] * inv_cut;
        const float x2 = x * x, x5 = x2 * x2 * x;
        const float env = x < 1.0f ? 1.0f + x5 * (-21.0f + x * (35.0f - 15.0f * x)) : 0.0f;
        const float t = x - offset[r];
        out[i] = env * expf(coeff * t * t);
    }
};
// per (qint edge b->a, main edge d->b): cbf16[t, i] = sum_s Rq[q, i, s] Y_s(cos(a,b,d))   (gemnet_oc.py:596-656; efficient.py:103-140)
struct QuadCbfK {
    Graph q, mn; const int32_t* q_tin; const float* Rq; float* cbf;
    GD void operator()(int64_t i) const {
        const int32_t qe = (int32_t)(i / RB), i16 = (int32_t)(i % RB);
        const int32_t b = q.src[qe], a = q.tgt[qe];
        const float* vq = q.V + 3 * (int64_t)qe;
        const float* R = Rq + (int64_t)qe * LD_Q + i16 * NS;
        int64_t t = q_tin[qe];
        for (int32_t k = mn.ptr[b]; k < mn.ptr[b + 1]; k++, t++) {
            float acc = 0.0f;
            if (mn.src[k] != a) {
                float Y[NS];
                cir7(clamp1(dot3(vq, mn.V + 3 * (int64_t)k)), Y);
#pragma unroll
                for (int s = 0; s < NS; s++) acc += R[s] * Y[s];
            }
            cbf[t * RB + i16] = acc;
        }
    }
};

// ------------------------------------------------------------------ elementwise / gather kernels
struct EmbedK {
    const int32_t* z; const float* emb; int32_t n_elem; float* h;
    GD void operator()(int64_t i) const {
        int32_t zz = z[i / EA] - 1;
        zz = zz < 0 ? 0 : (zz >= n_elem ? n_elem - 1 : zz);
        h[i] = emb[(int64_t)zz * EA + (i % EA)];
    }
};
// EdgeEmbedding (embedding_block.py:48-92): act(W [h_s | h_t | m]) with the three column blocks of W applied before the gather
struct EdgeEmbK {
    const float* hst; const float* mr; const int32_t* src; const int32_t* tgt; float* out;
    GD void operator()(int64_t i) const {
        const int64_t e = i / EE; const int c = (int)(i % EE);
        out[i] = ssilu(hst[(int64_t)src[e] * (2 * EE) + c] + hst[(int64_t)tgt[e] * (2 * EE) + EE + c] + mr[i]);
    }
};
struct SsiluK {
    float* x;
    GD void operator()(int64_t i) const { x[i] = ssilu(x[i]); }
};
struct ResOutK {  // ResidualLayer tail (base_layers.py:78-97): x = (x + act(t)) / sqrt 2
    float* x; const float* t;
    GD void operator()(int64_t i) const { x[i] = (x[i] + ssilu(t[i])) * ISQ2; }
};
struct AddScaleK {  // y = (y + b) * alpha
    float* y; const float* b; float alpha;
    GD void operator()(int64_t i) const { y[i] = (y[i] + b[i]) * alpha; }
};
// acc = (f(acc) + (act(u_ca) + act(u_ac)[id_swap]) / sqrt 2) * out_scale   (interaction_block.py symmetric message passing);
// f = act for the first merged branch (acc then holds the pre-activation of dense_ca), out_scale = 1/sqrt(#branches) on the last one
struct SymAddK {
    float* acc; const float* uca; const float* uac; const int32_t* rev; int32_t act_acc; float out_scale;
    GD void operator()(int64_t i) const {
        const int64_t e = i / EE; const int c = (int)(i % EE);
        const float a = acc[i];
        acc[i] = ((act_acc ? ssilu(a) : a) + (ssilu(uca[i]) + ssilu(uac[(int64_t)rev[e] * EE + c])) * ISQ2) * out_scale;
    }
};
struct CombineHK {  // h = (h + act(a) + act(b)) / sqrt 3
    float* h; const float* a; const float* b;
    GD void operator()(int64_t i) const { h[i] = (h[i] + ssilu(a[i]) + ssilu(b[i])) * ISQ3; }
};
struct CopyColsK {
    const float* x; int32_t C; float* out; int32_t ldo;
    GD void operator()(int64_t i) const { out[(i / C) * ldo + (i % C)] = x[i]; }
};
// out[r, c] = f(x[row(r), c]) * (rbf16[r] . W[c]) * scale, f = act if act_in else identity
// (x * mlp_rbf(basis) with the K = 16 Dense evaluated in place; act_in fuses the activation of the Dense that produced x)
struct MulRbfK {
    const float* x; int32_t ldx; const int32_t* row_idx; const float* rbf; int32_t ldr; const float* W; float scale; float* out; int32_t ldo; int32_t C;
    int32_t act_in;
    GD void operator()(int64_t i) const {
        const int64_t r = i / C; const int c = (int)(i % C);
        const float* b = rbf + r * ldr; const float* w = W + (int64_t)c * RB;
        float dot = 0.0f;
#pragma unroll
        for (int k = 0; k < RB; k++) dot += b[k] * w[k];
        const int64_t xr = row_idx ? row_idx[r] : r;
        const float xv = x[xr * ldx + c];
        out[r * ldo + c] = (act_in ? ssilu(xv) : xv) * dot * scale;
    }
};
// The same arithmetic (bitwise), MRB_ROWS rows per logical thread: the 16 weights of channel c stay in registers, consecutive threads are
// consecutive channels.  MulRbfK read W[c][0..15] again for every output -- 64 bytes per thread at a 64-byte stride, 16 L1 wavefronts per
// warp load -- and was 10 % of the first measured forward; here a warp's per-row traffic is the
// broadcast basis row + one coalesced load + one coalesced store.  i = (row block, channel); n = ceil(M / MRB_ROWS) * C.
constexpr int MRB_ROWS = 16;
struct MulRbfRowsK {
    const float* x; int32_t ldx; const int32_t* row_idx; const float* rbf; int32_t ldr; const float* W; float scale; float* out; int32_t ldo; int32_t C;
    int32_t act_in; int64_t M;
    const int32_t* M_dev;  // row count on the device when M is an upper bound (Ext), else nullptr
    static int64_t count(int64_t M, int C) { return (M + MRB_ROWS - 1) / MRB_ROWS * C; }
    GD void operator()(int64_t i) const {
        const int64_t rb = i / C; const int c = (int)(i % C);
        // 16-byte loads (the basis columns start at multiples of 16 floats of 256-byte aligned rows; ldr % 4 == 0): the scalar form issued
        // 16 + 1 loads and a store per output row and warp and was bound by the load/store unit's instruction rate
        float w[RB];
        const float4* w4 = reinterpret_cast<const float4*>(W + (int64_t)c * RB);
#pragma unroll
        for (int k = 0; k < RB / 4; k++) { const float4 t = w4[k]; w[4 * k] = t.x; w[4 * k + 1] = t.y; w[4 * k + 2] = t.z; w[4 * k + 3] = t.w; }
        const int64_t Mr = ext_rows(M, M_dev), r1 = (rb + 1) * MRB_ROWS < Mr ? (rb + 1) * MRB_ROWS : Mr;
        for (int64_t r = rb * MRB_ROWS; r < r1; r++) {
            const float4* b4 = reinterpret_cast<const float4*>(rbf + r * ldr);
            float b[RB];
#pragma unroll
            for (int k = 0; k < RB / 4; k++) { const float4 t = b4[k]; b[4 * k] = t.x; b[4 * k + 1] = t.y; b[4 * k + 2] = t.z; b[4 * k + 3] = t.w; }
            float dot = 0.0f;
#pragma unroll
            for (int k = 0; k < RB; k++) dot += b[k] * w[k];
            const int64_t xr = row_idx ? row_idx[r] : r;
            const float xv = x[xr * ldx + c];
            out[r * ldo + c] = (act_in ? ssilu(xv) : xv) * dot * scale;
        }
    }
};
// atom_update_block.py:60-91: out[a, c] = scale * sum over edges into a of m[e, c] * (rbf16[e] . W[c])
struct AggAtomRbfK {
    const int32_t* ptr; const float* m; const float* rbf; int32_t ldr; const float* W; float scale; float* out;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / EE); const int c = (int)(i % EE);
        float w[RB];  // 16-byte loads as in MulRbfRowsK (rows of the basis and of W are 64-byte aligned)
        const float4* w4 = reinterpret_cast<const float4*>(W + (int64_t)c * RB);
#pragma unroll
        for (int k = 0; k < RB / 4; k++) { const float4 t = w4[k]; w[4 * k] = t.x; w[4 * k + 1] = t.y; w[4 * k + 2] = t.z; w[4 * k + 3] = t.w; }
        float acc = 0.0f;
        for (int32_t e = ptr[a]; e < ptr[a + 1]; e++) {
            const float4* b4 = reinterpret_cast<const float4*>(rbf + (int64_t)e * ldr);
            float b[RB];
#pragma unroll
            for (int k = 0; k < RB / 4; k++) { const float4 t = b4[k]; b[4 * k] = t.x; b[4 * k + 1] = t.y; b[4 * k + 2] = t.z; b[4 * k + 3] = t.w; }
            float dot = 0.0f;
#pragma unroll
            for (int k = 0; k < RB; k++) dot += b[k] * w[k];
            acc += m[(int64_t)e * EE + c] * dot;
        }
        out[i] = acc * scale;
    }
};
struct DotRowK {
    const float* x; int32_t C; const float* w; float* out;
    GD void operator()(int64_t r) const {
        const float* a = x + r * C;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
        for (int k = 0; k < C; k += 4) { s0 += a[k] * w[k]; s1 += a[k + 1] * w[k + 1]; s2 += a[k + 2] * w[k + 2]; s3 += a[k + 3] * w[k + 3]; }
        out[r] = (s0 + s1) + (s2 + s3);
    }
};
struct MolEnergyK {  // extensive: sum over the molecule's atoms (gemnet_oc.py:1196-1206)
    const int32_t* mol_ptr; const float* e_atom; float* energy;
    GD void operator()(int64_t m) const {
        float s = 0.0f;
        for (int32_t a = mol_ptr[m]; a < mol_ptr[m + 1]; a++) s += e_atom[a];
        energy[m] = s;
    }
};
struct ForceK {  // coupled direct forces (gemnet_oc.py:1217-1242): F_a = sum over edges into a of mean(F_st[e], F_st[swap e]) V[e]
    const int32_t* ptr; const int32_t* rev; const float* fst; const float* V; float* F;
    GD void operator()(int64_t a) const {
        float fx = 0.0f, fy = 0.0f, fz = 0.0f;
        for (int32_t e = ptr[a]; e < ptr[a + 1]; e++) {
            const float f = 0.5f * (fst[e] + fst[rev[e]]);
            fx += f * V[3 * (int64_t)e]; fy += f * V[3 * (int64_t)e + 1]; fz += f * V[3 * (int64_t)e + 2];
        }
        F[3 * a] = fx; F[3 * a + 1] = fy; F[3 * a + 2] = fz;
    }
};

// ------------------------------------------------------------------ aggregation kernels (efficient.py:143-253 without the padding)
// output edge e = (c -> a) of the main graph, inputs = edges into a of `in` whose source differs from c:
//   O[e, i, ch] = sum_s R[e, i, s] * sum_in Y_s(cos(V_e, V_in)) x[in, ch]
struct TripEdgeK {
    Graph o, in; const float* x; const float* R; int32_t ldr; float* O;
    GD void operator()(int64_t i) const {
        const int32_t e = (int32_t)(i / TI); const int ch = (int)(i % TI);
        const int32_t a = o.tgt[e], cs = o.src[e];
        const float* v = o.V + 3 * (int64_t)e;
        float S[NS];
#pragma unroll
        for (int s = 0; s < NS; s++) S[s] = 0.0f;
        for (int32_t k = in.ptr[a]; k < in.ptr[a + 1]; k++) {
            if (in.src[k] == cs) continue;
            float Y[NS];
            cir7(clamp1(dot3(v, in.V + 3 * (int64_t)k)), Y);
            const float xv = x[(int64_t)k * TI + ch];
#pragma unroll
            for (int s = 0; s < NS; s++) S[s] += Y[s] * xv;
        }
        const float* Re = R + (int64_t)e * ldr;
        for (int i16 = 0; i16 < 16; i16++) {
            float acc = 0.0f;
#pragma unroll
            for (int s = 0; s < NS; s++) acc += Re[i16 * NS + s] * S[s];
            O[(int64_t)e * 1024 + i16 * TI + ch] = acc;
        }
    }
};
// edge -> atom: for atom a, sum over a2ee2a edges p into a of R[p] . S[p], S[p] over main edges into a whose source differs from p's
struct TripAtomK {
    Graph ae, mn; const float* x; const float* R; int32_t ldr; float* O;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / TI); const int ch = (int)(i % TI);
        float acc[16];
#pragma unroll
        for (int k = 0; k < 16; k++) acc[k] = 0.0f;
        for (int32_t p = ae.ptr[a]; p < ae.ptr[a + 1]; p++) {
            const int32_t ps = ae.src[p];
            const float* v = ae.V + 3 * (int64_t)p;
            float S[NS];
#pragma unroll
            for (int s = 0; s < NS; s++) S[s] = 0.0f;
            for (int32_t k = mn.ptr[a]; k < mn.ptr[a + 1]; k++) {
                if (mn.src[k] == ps) continue;
                float Y[NS];
                cir7(clamp1(dot3(v, mn.V + 3 * (int64_t)k)), Y);
                const float xv = x[(int64_t)k * TI + ch];
#pragma unroll
                for (int s = 0; s < NS; s++) S[s] += Y[s] * xv;
            }
            const float* Rp = R + (int64_t)p * ldr;
#pragma unroll
            for (int i16 = 0; i16 < 16; i16++) {
                float t = 0.0f;
#pragma unroll
                for (int s = 0; s < NS; s++) t += Rp[i16 * NS + s] * S[s];
                acc[i16] += t;
            }
        }
#pragma unroll
        for (int i16 = 0; i16 < 16; i16++) O[(int64_t)a * 1024 + i16 * TI + ch] = acc[i16];
    }
};
// atom -> atom (interaction_block.py PairInteraction): O[a, i, ch] = sum over a2a edges into a of rbf16[edge, i] x[src, ch]
struct PairK {
    const int32_t* ptr; const int32_t* src; const float* rbf; int32_t ldr; const float* x; float* O;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / TI); const int ch = (int)(i % TI);
        float acc[16];
#pragma unroll
        for (int k = 0; k < 16; k++) acc[k] = 0.0f;
        for (int32_t e = ptr[a]; e < ptr[a + 1]; e++) {
            const float xv = x[(int64_t)src[e] * TI + ch];
            const float* b = rbf + (int64_t)e * ldr;
#pragma unroll
            for (int k = 0; k < 16; k++) acc[k] += b[k] * xv;
        }
#pragma unroll
        for (int k = 0; k < 16; k++) O[(int64_t)a * 1024 + k * TI + ch] = acc[k];
    }
};
// x_t[t, ch] = x_down[d->b, ch] * (W_cbf[ch] . cbf16[t]) * scale_cbf      (interaction_block.py QuadrupletInteraction)
struct QuadXtK {
    Graph q, mn; const int32_t* q_tin; const float* xd; const float* cbf; const float* W; float scale; float* xt;
    GD void operator()(int64_t i) const {
        const int32_t qe = (int32_t)(i / QI); const int ch = (int)(i % QI);
        const int32_t b = q.src[qe];
        float w[RB];
        const float4* w4 = reinterpret_cast<const float4*>(W + ch * RB);
#pragma unroll
        for (int j = 0; j < RB / 4; j++) { const float4 v = w4[j]; w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w; }
        int64_t t = q_tin[qe];
        for (int32_t k = mn.ptr[b]; k < mn.ptr[b + 1]; k++, t++) {
            const float4* cb4 = reinterpret_cast<const float4*>(cbf + t * RB);
            float cb[RB];
#pragma unroll
            for (int j = 0; j < RB / 4; j++) { const float4 v = cb4[j]; cb[4 * j] = v.x; cb[4 * j + 1] = v.y; cb[4 * j + 2] = v.z; cb[4 * j + 3] = v.w; }
            float dot = 0.0f;
#pragma unroll
            for (int j = 0; j < RB; j++) dot += cb[j] * w[j];
            xt[t * QI + ch] = xd[(int64_t)k * QI + ch] * dot * scale;
        }
    }
};
// quadruplets d -> b -> a <- c for the output edge e = (c -> a): b over the qint edges into a (b != c), d over the main edges into b
// (d != a, d != c).  S[(l_phi, l_theta), ch] += Y_l_phi(cos(c,a,b)) Y_l_theta(cos of the dihedral) x_t[(b->a, d->b), ch];
// O[e, i, ch] = sum_s R_sbf[e, i, s] S[s]      (gemnet_oc.py:596-656, spherical_basis.py legendre_outer, efficient.py)
struct QuadK {
    Graph mn, q; const int32_t* q_tin; const float* xt; const float* R; int32_t ldr; float* O;
    GD void operator()(int64_t i) const {
        const int32_t e = (int32_t)(i / QI); const int ch = (int)(i % QI);
        const int32_t a = mn.tgt[e], c = mn.src[e];
        const float* vca = mn.V + 3 * (int64_t)e;
        float S[NS2];
#pragma unroll
        for (int s = 0; s < NS2; s++) S[s] = 0.0f;
        for (int32_t qe = q.ptr[a]; qe < q.ptr[a + 1]; qe++) {
            const int32_t b = q.src[qe];
            if (b == c) continue;
            const float* vba = q.V + 3 * (int64_t)qe;
            float Yp[NS], n1[3];
            cir7(clamp1(dot3(vca, vba)), Yp);
            cross3(vca, vba, n1);
            int64_t t = q_tin[qe];
            for (int32_t k = mn.ptr[b]; k < mn.ptr[b + 1]; k++, t++) {
                const int32_t d = mn.src[k];
                if (d == a || d == c) continue;
                float n2[3], n3[3], Yt[NS];
                cross3(mn.V + 3 * (int64_t)k, vba, n2);
                const float xx = dot3(n1, n2);
                cross3(n1, n2, n3);
                const float yy = fmaxf(sqrtf(dot3(n3, n3)), 1e-9f);
                cir7(xx / sqrtf(xx * xx + yy * yy), Yt);  // cos(atan2(y, x))
                const float xv = xt[t * QI + ch];
#pragma unroll
                for (int l1 = 0; l1 < NS; l1++) {
                    const float f = Yp[l1] * xv;
#pragma unroll
                    for (int l2 = 0; l2 < NS; l2++) S[l1 * NS + l2] += f * Yt[l2];
                }
            }
        }
        const float* Re = R + (int64_t)e * ldr;
        for (int i32 = 0; i32 < 32; i32++) {
            float acc = 0.0f;
#pragma unroll
            for (int s = 0; s < NS2; s++) acc += Re[i32 * NS2 + s] * S[s];
            O[(int64_t)e * 1024 + i32 * QI + ch] = acc;
        }
    }
};


}  // namespace
