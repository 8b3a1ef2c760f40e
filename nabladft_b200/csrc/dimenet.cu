// dimenet.cu -- DimeNet++ energy + conservative forces (DESIGN.md 3.15), config/model/dimenetplusplus.yaml.
//
// Reference: nablaDFT/dimenetplusplus/dimenetplusplus.py:22-113 (DimeNetPlusPlusPotential: core, regr_or_cls_nn, forces = -d(prediction)/d pos,
// scaler after the gradient) around torch_geometric.nn.models.DimeNetPlusPlus 2.4.0 (restated in oracle/dimenet.py).
//
// Graph: CSR by target atom, sources ascending, with radius_graph's truncation (the first max_neighbors + 1 in-cutoff candidates in index
// order, the target itself included, then the self loop dropped), plus the by-source permutation (oeid) -- after truncation the edge set is not
// symmetric, so the out-edges of an atom are not the reverses of its in-edges.  Triplets k -> j -> i (edge kj into j, k != i) are never
// stored: kernels enumerate them from CSR rows.  The only per-triplet array is the reverse pass's dE/dcos(angle), in the order of the
// reference's triplet list (by ji edge, then ascending k): slot(ji, kj) = tptr[ji] + (kj - ptr[j]) - [edge i -> j exists and k > i].
//
// Forward keeps the block outputs X[0..nb]; the reverse pass recomputes one interaction block at a time into a shared scratch.  Every sum is a
// gather in a fixed order (no atomics), so two calls are bitwise equal.  Dense layers run on the wgmma 3xTF32 GEMM when the shape tiles
// (every [E,256] and [E,64] layer), else on the functor GEMM.  Every kernel is a functor launched through pfor() (gemnet_pf.cuh), so the same
// source builds for host emulation (tests/emu, name="dimenet").
//
// Two entries share the energy-and-forces pass (DESIGN.md 3.15.3): the two-phase call sizes every edge extent by the exact count it read back
// from the graph phase; the asynchronous call sizes them by upper bounds that follow from the molecule sizes (nb200_dimenet_count_bounds),
// leaves the counts on the device, and every edge-row launch and GEMM stops at the device count (Ext, gemnet_pf.cuh).
#include "gemnet_pf.cuh"

namespace {
#ifdef NB_EMU
using std::isfinite;
#endif

constexpr int H = 256, IE = 64, BE = 8, NSPH = 7, NRAD = 6, NSR = 42, OE = 256, NRES = 3, NLIN = 3, MAXL = 64, NZ = 95;

GD float silu(float x) { return x / (1.0f + expf(-x)); }
GD float dsilu(float x) {
    const float s = 1.0f / (1.0f + expf(-x));
    return s * (1.0f + x * (1.0f - s));
}
// Envelope(p = exponent + 1 = 6) (PyG Envelope): 1/x + a x^5 + b x^6 + c x^7 for x < 1, and its derivative
GD float env6(float x) {
    const float x5 = x * x * x * x * x;
    return x < 1.0f ? 1.0f / x + x5 * (-28.0f + x * (48.0f - 21.0f * x)) : 0.0f;
}
GD float denv6(float x) {
    const float x4 = x * x * x * x;
    return x < 1.0f ? -1.0f / (x * x) + x4 * (-140.0f + x * (288.0f - 147.0f * x)) : 0.0f;
}
// spherical Bessel j_l(x) and j_{l+1}(x), l <= 6.  Below x = l + 2 the closed sin / cos forms (and the upward recurrence built on them) cancel
// badly in fp32, so there the power series x^l / (2l+1)!! sum_k (-x^2/2)^k / (k! (2l+3)(2l+5)...(2l+2k+1)) is summed (16 terms: < 1e-8
// relative for x < 9); above it, the upward recurrence from sin x / x.
GD float jn_series(int l, float x) {
    float lead = 1.0f;
    for (int m = 1; m <= l; m++) lead *= x / (float)(2 * m + 1);
    const float h = -0.5f * x * x;
    float term = 1.0f, sum = 1.0f;
    for (int k = 1; k <= 16; k++) {
        term *= h / (float)(k * (2 * l + 2 * k + 1));
        sum += term;
    }
    return lead * sum;
}
GD void sph_jn2(int l, float x, float& jl, float& jl1) {
    if (x < (float)(l + 2)) {
        jl = jn_series(l, x);
        jl1 = jn_series(l + 1, x);
        return;
    }
    const float s = sinf(x), c = cosf(x), ix = 1.0f / x;
    float a = s * ix, b = (a - c) * ix;  // j_0, j_1
    for (int m = 1; m <= l; m++) {
        const float t = (float)(2 * m + 1) * ix * b - a;
        a = b;
        b = t;
    }
    jl = a;
    jl1 = b;
}
// Y_l^0(ct) = sqrt((2l+1)/(4 pi)) P_l(ct) and d/dct, l < 7
GD void ylm7(float ct, float* Y, float* dY) {
    const float cn[NSPH] = {0.28209479177387814f, 0.4886025119029199f, 0.6307831305050401f, 0.7463526651802308f,
                            0.8462843753216345f, 0.9356025796273888f, 1.0171072362820548f};
    float p0 = 1.0f, p1 = ct, d0 = 0.0f, d1 = 1.0f;
    Y[0] = cn[0];
    dY[0] = 0.0f;
    Y[1] = cn[1] * ct;
    dY[1] = cn[1];
    for (int l = 1; l < NSPH - 1; l++) {
        const float p2 = ((float)(2 * l + 1) * ct * p1 - (float)l * p0) / (float)(l + 1);
        const float d2 = d0 + (float)(2 * l + 1) * p1;  // P'_{l+1} = P'_{l-1} + (2l+1) P_l
        Y[l + 1] = cn[l + 1] * p2;
        dY[l + 1] = cn[l + 1] * d2;
        p0 = p1; p1 = p2; d0 = d1; d1 = d2;
    }
}
GD float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// ------------------------------------------------------------------ graph phase
struct MolIdK {
    const int32_t* mol_ptr; int32_t n_mol; int32_t* mol_id;
    GD void operator()(int64_t a) const {
        int lo = 0, hi = n_mol;
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (mol_ptr[mid] <= (int32_t)a) lo = mid; else hi = mid;
        }
        mol_id[a] = lo;
    }
};
GD bool finite3(const float* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }
// sources of target a: the first kcap (= max_neighbors + 1) atoms j of the molecule, ascending, with d^2 < cut2 (j == a included), minus a
struct NbrK {
    const float* pos; const int32_t* z; const int32_t* mol_ptr; const int32_t* mol_id; float cut2; int32_t kcap;
    const int32_t* ptr;  // nullptr: count pass (deg, bad); else fill pass (src, tgt)
    int32_t* deg; int32_t* bad; int32_t* src; int32_t* tgt;
    GD void operator()(int64_t ai) const {
        const int32_t a = (int32_t)ai, m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        const float* pa = pos + 3 * (int64_t)a;
        if (!ptr) bad[a] = (z[a] < 0 || z[a] >= NZ || !finite3(pa)) ? 1 : 0;
        int32_t cand = 0, kept = 0, e = ptr ? ptr[a] : 0;
        for (int32_t j = m0; j < m1 && cand < kcap; j++) {
            const float* pj = pos + 3 * (int64_t)j;
            const float dx = pj[0] - pa[0], dy = pj[1] - pa[1], dz = pj[2] - pa[2];
            if (!(dx * dx + dy * dy + dz * dz < cut2)) continue;
            cand++;
            if (j == a) continue;
            if (ptr) { src[e] = j; tgt[e] = a; e++; }
            kept++;
        }
        if (!ptr) deg[a] = kept;
    }
};
// edge id of (source s -> target t) or -1: binary search in the ascending sources of row t
GD int32_t find_edge(const int32_t* ptr, const int32_t* src, int32_t s, int32_t t) {
    int32_t lo = ptr[t], hi = ptr[t + 1];
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (src[mid] < s) lo = mid + 1; else hi = mid;
    }
    return (lo < ptr[t + 1] && src[lo] == s) ? lo : -1;
}
struct RevK {  // rev[e] = the edge tgt(e) -> src(e), or -1
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; int32_t* rev;
    GD void operator()(int64_t e) const { rev[e] = find_edge(ptr, src, tgt[e], src[e]); }
};
// out-edges of atom j in ascending edge id (= ascending target): count pass (optr == nullptr) and fill pass
struct OutK {
    const int32_t* ptr; const int32_t* src; const int32_t* mol_ptr; const int32_t* mol_id; const int32_t* optr; int32_t* odeg; int32_t* oeid;
    GD void operator()(int64_t ji) const {
        const int32_t j = (int32_t)ji, m0 = mol_ptr[mol_id[j]], m1 = mol_ptr[mol_id[j] + 1];
        int32_t c = 0;
        for (int32_t t = m0; t < m1; t++) {
            const int32_t e = find_edge(ptr, src, j, t);
            if (e < 0) continue;
            if (optr) oeid[optr[j] + c] = e;
            c++;
        }
        if (!optr) odeg[j] = c;
    }
};
struct TcntK {  // triplets of edge j -> i: edges into j except i -> j
    const int32_t* ptr; const int32_t* src; const int32_t* rev; const int32_t* n_edges; int32_t* tcnt;
    GD void operator()(int64_t e) const {
        if (e >= *n_edges) { tcnt[e] = 0; return; }
        const int32_t j = src[e];
        tcnt[e] = ptr[j + 1] - ptr[j] - (rev[e] >= 0 ? 1 : 0);
    }
};
struct TotK {
    const int32_t* a; const int32_t* b; const int32_t* c; int32_t* tot;
    GD void operator()(int64_t) const { tot[0] = *a; tot[1] = *b; tot[2] = *c; }
};
// status words of the asynchronous call (include/nabla_b200.h): 1 error, 2 largest in-degree, 3 atoms without a source
struct StatusAtomK {
    const int32_t* bad; const int32_t* deg; int32_t* status;
    GD void operator()(int64_t a) const {
        if (bad[a]) atomicMin(status + 1, (int32_t)NB200_EINVAL);  // z outside [0, 94] or a non-finite coordinate (NbrK)
        atomicMax(status + 2, deg[a]);
        if (deg[a] == 0) atomicAdd(status + 3, 1);
    }
};
struct StatusCountsK {  // one thread, after StatusAtomK: 0 edges, 4 triplet slots, both against their bounds
    const int32_t* n_edges; const int32_t* n_slots; int32_t e_bound, t_bound; int32_t* status;
    GD void operator()(int64_t) const {
        const int32_t E = *n_edges, T = *n_slots;
        status[0] = E;
        status[4] = T;
        if (status[1] == 0 && (E < 0 || E > e_bound || T < 0 || T > t_bound)) status[1] = NB200_ECAPACITY;  // < 0: int32 overflow of the scan
    }
};
// after an error every CSR row (by target and by source) is empty and the device edge count is 0: no later kernel reaches an edge row
struct ClearOnErrorK {
    const int32_t* status; int32_t* ptr; int32_t* optr; int64_t n1;
    GD void operator()(int64_t i) const {
        if (status[1] == 0) return;
        if (i < n1) ptr[i] = 0; else optr[i - n1] = 0;
    }
};
GD float quiet_nan() {
    const uint32_t u = 0x7fc00000u;
    float x;
    memcpy(&x, &u, 4);
    return x;
}
struct NanOnErrorK {
    const int32_t* status; float* energy; int64_t n_mol; float* forces;
    GD void operator()(int64_t i) const {
        if (status[1] == 0) return;
        if (i < n_mol) energy[i] = quiet_nan(); else forces[i - n_mol] = quiet_nan();
    }
};

// ------------------------------------------------------------------ bases
struct GeomK {  // V = pos[target] - pos[source], d = |V|
    const float* pos; const int32_t* src; const int32_t* tgt; float* V; float* d;
    GD void operator()(int64_t e) const {
        const float* pi = pos + 3 * (int64_t)tgt[e];
        const float* pj = pos + 3 * (int64_t)src[e];
        const float v[3] = {pi[0] - pj[0], pi[1] - pj[1], pi[2] - pj[2]};
        V[3 * e] = v[0]; V[3 * e + 1] = v[1]; V[3 * e + 2] = v[2];
        d[e] = sqrtf(dot3(v, v));
    }
};
struct RbfK {  // BesselBasisLayer: env(x) sin(freq_n x), x = d / cutoff
    const float* d; const float* freq; float inv_cut; float* rbf;
    GD void operator()(int64_t i) const {
        const int64_t e = i / NRAD;
        const int n = (int)(i % NRAD);
        const float x = d[e] * inv_cut;
        rbf[i] = env6(x) * sinf(freq[n] * x);
    }
};
struct RbsK {  // SphericalBasisLayer radial part: env(x) N_ln j_l(z_ln x); optional d/d(dist)
    const float* d; const float* zeros; const float* norms; float inv_cut; float* rbs; float* drbs;
    GD void operator()(int64_t i) const {
        const int64_t e = i / NSR;
        const int ln = (int)(i % NSR), l = ln / NRAD;
        const float x = d[e] * inv_cut, zz = zeros[ln];
        float jl, jl1;
        sph_jn2(l, zz * x, jl, jl1);
        const float en = env6(x);
        rbs[i] = en * norms[ln] * jl;
        if (drbs) {
            const float y = zz * x;
            const float djl = (float)l / y * jl - jl1;  // j_l' = (l/y) j_l - j_{l+1}
            drbs[i] = norms[ln] * (denv6(x) * jl + en * zz * djl) * inv_cut;
        }
    }
};

// ------------------------------------------------------------------ dense helpers
struct GemmK {  // C[r, n] = (acc ? C : 0) + bias[n] + sum_k A[r, k] op(B)[k, n];  op(B) = B[n, k] (trans 0) | B[k, n] (trans 1)
    const float* A; int32_t lda; const float* B; int32_t ldb; int32_t trans; float* C; int32_t ldc; int32_t N, K; int32_t acc; const float* bias;
    GD void operator()(int64_t i) const {
        const int64_t r = i / N;
        const int n = (int)(i % N);
        float s = 0.0f;
        for (int k = 0; k < K; k++) s += A[r * lda + k] * (trans ? B[(int64_t)k * ldb + n] : B[(int64_t)n * ldb + k]);
        if (bias) s += bias[n];
        C[r * ldc + n] = acc ? C[r * ldc + n] + s : s;
    }
};
struct ActK {  // y = silu(x)
    const float* x; float* y;
    GD void operator()(int64_t i) const { y[i] = silu(x[i]); }
};
struct DActMulK {  // y = g * silu'(pre)
    const float* g; const float* pre; float* y;
    GD void operator()(int64_t i) const { y[i] = g[i] * dsilu(pre[i]); }
};
struct AddActK {  // y = base + silu(x)
    const float* base; const float* x; float* y;
    GD void operator()(int64_t i) const { y[i] = base[i] + silu(x[i]); }
};
// r[e, c] = sum_k W[c, k] rbf[e, k]  (a 6 -> C linear map without bias, evaluated in place of a GEMM with K = 6)
GD float rbf_lin(const float* W, const float* rbf, int64_t e, int c) {
    float s = 0.0f;
    for (int k = 0; k < NRAD; k++) s += W[c * NRAD + k] * rbf[e * NRAD + k];
    return s;
}
struct EmbRbfK {  // hr = lin_rbf(rbf) (pre-activation), hra = silu(hr)
    const float* rbf; const float* W; const float* b; float* hr; float* hra;
    GD void operator()(int64_t i) const {
        const int64_t e = i / H;
        const int c = (int)(i % H);
        const float v = rbf_lin(W, rbf, e, c) + b[c];
        hr[i] = v;
        hra[i] = silu(v);
    }
};
struct EmbAddK {  // epre += Ti[z_i] + Tj[z_j]; x = silu(epre)
    const int32_t* z; const int32_t* src; const int32_t* tgt; const float* Ti; const float* Tj; float* epre; float* x;
    GD void operator()(int64_t i) const {
        const int64_t e = i / H;
        const int c = (int)(i % H);
        const float v = epre[i] + Ti[(int64_t)z[tgt[e]] * H + c] + Tj[(int64_t)z[src[e]] * H + c];
        epre[i] = v;
        x[i] = silu(v);
    }
};
struct MulRbfK {  // t = xk * (W rbf)
    const float* xk; const float* rbf; const float* W; float* t;
    GD void operator()(int64_t i) const { t[i] = xk[i] * rbf_lin(W, rbf, i / H, (int)(i % H)); }
};
struct LinOutK {  // h2 = silu(lpre) + x
    const float* lpre; const float* x; float* h2;
    GD void operator()(int64_t i) const { h2[i] = silu(lpre[i]) + x[i]; }
};

// ------------------------------------------------------------------ triplets
// forward aggregation, one (ji edge, channel): agg[ji, c] = sum_{kj into j, k != i} xd[kj, c] * sum_ln Wsbf[c, ln] Y_l(cos a) rbs[kj, ln]
struct TripFwdK {
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; const float* V; const float* d; const float* rbs; const float* Wsbf;
    const float* xd; float* agg;
    GD void operator()(int64_t idx) const {
        const int64_t e = idx / IE;
        const int c = (int)(idx % IE);
        const int32_t j = src[e], i = tgt[e];
        const float u[3] = {V[3 * e], V[3 * e + 1], V[3 * e + 2]};
        const float du = d[e];
        float W[NSR];
        for (int q = 0; q < NSR; q++) W[q] = Wsbf[c * NSR + q];
        float acc = 0.0f;
        for (int32_t kj = ptr[j]; kj < ptr[j + 1]; kj++) {
            if (src[kj] == i) continue;
            const float ct = dot3(u, V + 3 * (int64_t)kj) / (du * d[kj]);
            float Y[NSPH], dY[NSPH];
            ylm7(ct, Y, dY);
            const float* rb = rbs + (int64_t)kj * NSR;
            float s = 0.0f;
            for (int l = 0; l < NSPH; l++) {
                float r = 0.0f;
                for (int n = 0; n < NRAD; n++) r += W[l * NRAD + n] * rb[l * NRAD + n];
                s += Y[l] * r;
            }
            acc += xd[(int64_t)kj * IE + c] * s;
        }
        agg[idx] = acc;
    }
};
// reverse, one (kj edge, channel): gxd[kj, c] = sum_{ji out of j, i != k} gagg[ji, c] * s_(ji,kj)[c]
struct TripBwdXK {
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; const int32_t* optr; const int32_t* oeid; const float* V; const float* d;
    const float* rbs; const float* Wsbf; const float* gagg; float* gxd;
    GD void operator()(int64_t idx) const {
        const int64_t kj = idx / IE;
        const int c = (int)(idx % IE);
        const int32_t k = src[kj], j = tgt[kj];
        const float v[3] = {V[3 * kj], V[3 * kj + 1], V[3 * kj + 2]};
        const float dv = d[kj];
        float R[NSPH];
        for (int l = 0; l < NSPH; l++) {
            float r = 0.0f;
            for (int n = 0; n < NRAD; n++) r += Wsbf[c * NSR + l * NRAD + n] * rbs[kj * NSR + l * NRAD + n];
            R[l] = r;
        }
        float acc = 0.0f;
        for (int32_t o = optr[j]; o < optr[j + 1]; o++) {
            const int32_t ji = oeid[o];
            if (tgt[ji] == k) continue;
            const float ct = dot3(V + 3 * (int64_t)ji, v) / (d[ji] * dv);
            float Y[NSPH], dY[NSPH];
            ylm7(ct, Y, dY);
            float s = 0.0f;
            for (int l = 0; l < NSPH; l++) s += Y[l] * R[l];
            acc += gagg[(int64_t)ji * IE + c] * s;
        }
        gxd[idx] = acc;
    }
};
// reverse, one kj edge: for every triplet (ji, kj) the gradient w.r.t. sbf, q[ln] = sum_m W1[m, ln] sum_c W2[c, m] gagg[ji, c] xd[kj, c];
// grbs[kj, ln] += Y_l q[ln]; gct[slot] += sum_l Y_l'(cos a) sum_n rbs[kj, ln] q[ln]
struct TripBwdGK {
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; const int32_t* rev; const int32_t* optr; const int32_t* oeid; const int32_t* tptr;
    const float* V; const float* d; const float* rbs; const float* W1; const float* W2; const float* gagg; const float* xd; float* grbs; float* gct;
    GD void operator()(int64_t kj) const {
        const int32_t k = src[kj], j = tgt[kj];
        const float v[3] = {V[3 * kj], V[3 * kj + 1], V[3 * kj + 2]};
        const float dv = d[kj];
        const float* rb = rbs + kj * NSR;
        const float* x = xd + kj * IE;
        float grb[NSR];
        for (int q = 0; q < NSR; q++) grb[q] = 0.0f;
        for (int32_t o = optr[j]; o < optr[j + 1]; o++) {
            const int32_t ji = oeid[o], i = tgt[ji];
            if (i == k) continue;
            const float ct = dot3(V + 3 * (int64_t)ji, v) / (d[ji] * dv);
            float Y[NSPH], dY[NSPH];
            ylm7(ct, Y, dY);
            const float* ga = gagg + (int64_t)ji * IE;
            float p[BE];
            for (int m = 0; m < BE; m++) p[m] = 0.0f;
            for (int c = 0; c < IE; c++) {
                const float u = ga[c] * x[c];
                for (int m = 0; m < BE; m++) p[m] += W2[c * BE + m] * u;
            }
            float g = 0.0f;
            for (int l = 0; l < NSPH; l++) {
                float gy = 0.0f;
                for (int n = 0; n < NRAD; n++) {
                    const int ln = l * NRAD + n;
                    float q = 0.0f;
                    for (int m = 0; m < BE; m++) q += W1[m * NSR + ln] * p[m];
                    grb[ln] += Y[l] * q;
                    gy += rb[ln] * q;
                }
                g += gy * dY[l];
            }
            const int32_t slot = tptr[ji] + (int32_t)(kj - ptr[j]) - ((rev[ji] >= 0 && k > i) ? 1 : 0);
            gct[slot] += g;
        }
        for (int q = 0; q < NSR; q++) grbs[kj * NSR + q] += grb[q];
    }
};

// ------------------------------------------------------------------ output blocks
struct AggOutK {  // A[a, c] = sum_{e into a} (W rbf)[e, c] * x[e, c]
    const int32_t* ptr; const float* rbf; const float* W; const float* x; float* A;
    GD void operator()(int64_t i) const {
        const int64_t a = i / H;
        const int c = (int)(i % H);
        float s = 0.0f;
        for (int32_t e = ptr[a]; e < ptr[a + 1]; e++) s += rbf_lin(W, rbf, e, c) * x[(int64_t)e * H + c];
        A[i] = s;
    }
};
struct OutBwdXK {  // gx[e, c] (+)= gA[tgt e, c] * (W rbf)[e, c]
    const int32_t* tgt; const float* rbf; const float* W; const float* gA; float* gx; int32_t acc;
    GD void operator()(int64_t i) const {
        const int64_t e = i / H;
        const int c = (int)(i % H);
        const float v = gA[(int64_t)tgt[e] * H + c] * rbf_lin(W, rbf, e, c);
        gx[i] = acc ? gx[i] + v : v;
    }
};
// grbf[e, k] += sum_c g[e or tgt(e), c] * x[e, c] * W[c, k]   (x == nullptr: factor 1; tgt == nullptr: g is per edge)
struct RbfBwdK {
    const int32_t* tgt; const float* g; const float* x; const float* W; float* grbf;
    GD void operator()(int64_t i) const {
        const int64_t e = i / NRAD;
        const int k = (int)(i % NRAD);
        const float* gr = g + (tgt ? (int64_t)tgt[e] : e) * H;
        float s = 0.0f;
        for (int c = 0; c < H; c++) s += gr[c] * (x ? x[e * H + c] : 1.0f) * W[c * NRAD + k];
        grbf[i] += s;
    }
};
struct KjBwdK {  // gbk = gt * (W rbf) * silu'(bk)
    const float* gt; const float* rbf; const float* W; const float* bk; float* gbk;
    GD void operator()(int64_t i) const { gbk[i] = gt[i] * rbf_lin(W, rbf, i / H, (int)(i % H)) * dsilu(bk[i]); }
};
struct BcastK {  // gP[a, :] = gG[mol(a), :]
    const int32_t* mol_id; const float* gG; int32_t L; float* gP;
    GD void operator()(int64_t i) const { gP[i] = gG[(int64_t)mol_id[i / L] * L + i % L]; }
};

// ------------------------------------------------------------------ regression head (one molecule per thread)
struct HeadK {
    const int32_t* mol_ptr; const float* P; int32_t L; const float *W0, *b0, *W1, *b1, *W2, *b2, *W3, *b3; float scale, mean;
    float* G; float* gG; float* energy;
    GD void operator()(int64_t m) const {
        const int L2 = L / 2;
        float g[MAXL], h1[MAXL], p1[MAXL], h2[MAXL / 2], p2[MAXL / 2], h3[MAXL / 2], p3[MAXL / 2];
        for (int c = 0; c < L; c++) g[c] = 0.0f;
        for (int32_t a = mol_ptr[m]; a < mol_ptr[m + 1]; a++)
            for (int c = 0; c < L; c++) g[c] += P[(int64_t)a * L + c];
        for (int o = 0; o < L; o++) { float s = b0[o]; for (int c = 0; c < L; c++) s += W0[o * L + c] * g[c]; p1[o] = s; h1[o] = silu(s); }
        for (int o = 0; o < L2; o++) { float s = b1[o]; for (int c = 0; c < L; c++) s += W1[o * L + c] * h1[c]; p2[o] = s; h2[o] = silu(s); }
        for (int o = 0; o < L2; o++) { float s = b2[o]; for (int c = 0; c < L2; c++) s += W2[o * L2 + c] * h2[c]; p3[o] = s; h3[o] = silu(s); }
        float y = b3[0];
        for (int c = 0; c < L2; c++) y += W3[c] * h3[c];
        energy[m] = scale * y + mean;
        // reverse: dy/dG
        for (int c = 0; c < L2; c++) h3[c] = W3[c] * dsilu(p3[c]);
        for (int c = 0; c < L2; c++) { float s = 0.0f; for (int o = 0; o < L2; o++) s += W2[o * L2 + c] * h3[o]; h2[c] = s * dsilu(p2[c]); }
        for (int c = 0; c < L; c++) { float s = 0.0f; for (int o = 0; o < L2; o++) s += W1[o * L + c] * h2[o]; h1[c] = s * dsilu(p1[c]); }
        for (int c = 0; c < L; c++) {
            float s = 0.0f;
            for (int o = 0; o < L; o++) s += W0[o * L + c] * h1[o];
            gG[m * L + c] = s;
            if (G) G[m * L + c] = g[c];
        }
    }
};

// ------------------------------------------------------------------ geometry reverse and forces
// gV[e] = dE/dV[e]: the distance term (rbf and rbs of this edge) plus the angle terms of the triplets in which e is the ji edge (u) and those in
// which it is the kj edge (v); cos a = u.v / (|u||v|), d cos / du = (v - cos |v|/|u| u) / (|u||v|)
struct GeomBwdK {
    const int32_t* ptr; const int32_t* src; const int32_t* tgt; const int32_t* rev; const int32_t* optr; const int32_t* oeid; const int32_t* tptr;
    const float* V; const float* d; const float* rbf; const float* freq; float inv_cut; const float* grbf; const float* rbs_d; const float* grbs;
    const float* gct; float* gV;
    GD void operator()(int64_t e) const {
        const int32_t j = src[e], i = tgt[e];
        const float u[3] = {V[3 * e], V[3 * e + 1], V[3 * e + 2]};
        const float du = d[e], x = du * inv_cut;
        // distance: rbf = env(x) sin(f x)
        const float en = env6(x), den = denv6(x);
        float gd = 0.0f;
        for (int n = 0; n < NRAD; n++) gd += grbf[e * NRAD + n] * (den * sinf(freq[n] * x) + en * freq[n] * cosf(freq[n] * x)) * inv_cut;
        for (int q = 0; q < NSR; q++) gd += grbs[e * NSR + q] * rbs_d[e * NSR + q];
        float g[3] = {gd * u[0] / du, gd * u[1] / du, gd * u[2] / du};
        // e as the ji edge: triplets over the edges kj into j
        const int32_t skip = rev[e];
        for (int32_t kj = ptr[j]; kj < ptr[j + 1]; kj++) {
            const int32_t k = src[kj];
            if (k == i) continue;
            const float gc = gct[tptr[e] + (kj - ptr[j]) - ((skip >= 0 && k > i) ? 1 : 0)];
            const float* v = V + 3 * (int64_t)kj;
            const float dv = d[kj], ct = dot3(u, v) / (du * dv), f = gc / (du * dv), r = ct * dv / du;
            for (int t = 0; t < 3; t++) g[t] += f * (v[t] - r * u[t]);
        }
        // e as the kj edge (k = src e, j' = tgt e): triplets over the edges ji out of j'
        for (int32_t o = optr[i]; o < optr[i + 1]; o++) {
            const int32_t ji = oeid[o], ti = tgt[ji];
            if (ti == j) continue;
            const float gc = gct[tptr[ji] + (int32_t)(e - ptr[i]) - ((rev[ji] >= 0 && j > ti) ? 1 : 0)];
            const float* w = V + 3 * (int64_t)ji;
            const float dw = d[ji], ct = dot3(w, u) / (dw * du), f = gc / (dw * du), r = ct * dw / du;
            for (int t = 0; t < 3; t++) g[t] += f * (w[t] - r * u[t]);
        }
        gV[3 * e] = g[0]; gV[3 * e + 1] = g[1]; gV[3 * e + 2] = g[2];
    }
};
struct ForceK {  // F[a] = -(sum_{e into a} gV[e] - sum_{e out of a} gV[e])
    const int32_t* ptr; const int32_t* optr; const int32_t* oeid; const float* gV; float* F;
    GD void operator()(int64_t i) const {
        const int64_t a = i / 3;
        const int t = (int)(i % 3);
        float s = 0.0f;
        for (int32_t e = ptr[a]; e < ptr[a + 1]; e++) s += gV[3 * (int64_t)e + t];
        for (int32_t o = optr[a]; o < optr[a + 1]; o++) s -= gV[3 * (int64_t)oeid[o] + t];
        F[i] = -s;
    }
};

// ------------------------------------------------------------------ host side
struct GraphBuf {
    int32_t *mol_id, *deg, *ptr, *bad, *badscan, *odeg, *optr, *src, *tgt, *rev, *oeid, *tcnt, *tptr, *tot;
    int64_t emax, bytes;
};
GraphBuf carve_graph(void* p, int64_t n, int64_t kcap) {
    Carve c(p);
    GraphBuf g;
    g.emax = n * kcap;
    g.mol_id = c.take<int32_t>(n);
    g.deg = c.take<int32_t>(n);
    g.ptr = c.take<int32_t>(n + 1);
    g.bad = c.take<int32_t>(n);
    g.badscan = c.take<int32_t>(n + 1);
    g.odeg = c.take<int32_t>(n);
    g.optr = c.take<int32_t>(n + 1);
    g.src = c.take<int32_t>(g.emax);
    g.tgt = c.take<int32_t>(g.emax);
    g.rev = c.take<int32_t>(g.emax);
    g.oeid = c.take<int32_t>(g.emax);
    g.tcnt = c.take<int32_t>(g.emax);
    g.tptr = c.take<int32_t>(g.emax + 1);
    g.tot = c.take<int32_t>(4);
    g.bytes = c.off + 256;
    return g;
}
struct Work {
    float *V, *d, *rbf, *rbs, *drbs, *X, *hr, *hra, *epre;
    float *a, *h0, *bk, *xk, *t, *dpre, *xd, *agg, *upre, *q1[NRES], *q2[NRES], *h1, *lpre, *h2, *h3, *out;  // one interaction block
    float *oA, *oU, *oT1, *oT2, *oP, *P, *gP, *G, *gG;
    float *gX, *gI, *g1, *g2, *g3, *g64a, *g64b, *grbf, *grbs, *gct, *gV;
    int64_t bytes;
};
Work carve_work(void* p, int64_t nb, int64_t n_mol, int64_t n, int64_t E, int64_t T, int64_t L) {
    Carve c(p);
    Work w;
    const int64_t EH = E * H, NH = n * H;
    w.V = c.take<float>(3 * E);
    w.d = c.take<float>(E);
    w.rbf = c.take<float>(E * NRAD);
    w.rbs = c.take<float>(E * NSR);
    w.drbs = c.take<float>(E * NSR);
    w.X = c.take<float>((nb + 1) * EH);
    w.hr = c.take<float>(EH);
    w.hra = c.take<float>(EH);
    w.epre = c.take<float>(EH);
    for (float** f : {&w.a, &w.h0, &w.bk, &w.xk, &w.t, &w.upre, &w.h1, &w.lpre, &w.h2, &w.h3, &w.out}) *f = c.take<float>(EH);
    for (int k = 0; k < NRES; k++) { w.q1[k] = c.take<float>(EH); w.q2[k] = c.take<float>(EH); }
    w.dpre = c.take<float>(E * IE);
    w.xd = c.take<float>(E * IE);
    w.agg = c.take<float>(E * IE);
    w.oA = c.take<float>(NH);
    w.oU = c.take<float>(NH);
    w.oT1 = c.take<float>(NH);
    w.oT2 = c.take<float>(NH);
    w.oP = c.take<float>((nb + 1) * NLIN * NH);
    w.P = c.take<float>(n * L);
    w.gP = c.take<float>(n * L);
    w.G = c.take<float>(n_mol * L);
    w.gG = c.take<float>(n_mol * L);
    for (float** f : {&w.gX, &w.gI, &w.g1, &w.g2, &w.g3}) *f = c.take<float>(EH);
    w.g64a = c.take<float>(E * IE);
    w.g64b = c.take<float>(E * IE);
    w.grbf = c.take<float>(E * NRAD);
    w.grbs = c.take<float>(E * NSR);
    w.gct = c.take<float>(T);
    w.gV = c.take<float>(3 * E);
    w.bytes = c.off + 256;
    return w;
}

int config_rc(const nb200_dimenet_weights* w) {
    if (!w || !w->w || !w->off_host || !(w->cutoff > 0.0f)) return NB200_EINVAL;
    if (w->hidden != H || w->int_emb != IE || w->basis_emb != BE || w->out_emb != OE || w->num_spherical != NSPH || w->num_radial != NRAD ||
        w->num_before_skip != 1 || w->num_after_skip != 2 || w->num_output_layers != NLIN || w->envelope_exponent != 5 || w->num_blocks < 1 ||
        w->num_blocks > 16 || w->node_latent_dim < 2 || w->node_latent_dim > MAXL || w->max_neighbors < 1 || w->max_neighbors > 64)
        return NB200_EUNSUPPORTED;
    return NB200_OK;
}

#ifdef NB_EMU
// host emulation of nb_gemm_tf32x3_ex with a device row count: the "device" count is readable here, so the emulated library GEMM
// (goc_tc_gemm_ex) runs over min(M, *m_dev) rows and the rows beyond are not written
inline int emu_gemm_rows(nb200_engine* e, cudaStream_t s, int M, int N, int K, const float* A, int lda, const float* B, int ldb, int trans, float* C,
                         int ldc, int acc, const float* bias, const int32_t* m_dev) {
    const int64_t rows = ext_rows(M, m_dev);
    return rows > 0 ? goc_tc_gemm_ex(e, s, (int)rows, N, K, A, lda, B, ldb, trans, C, ldc, acc, bias) : NB200_OK;
}
#endif

struct Ctx {
    nb200_engine* e; cudaStream_t s; const nb200_dimenet_weights* w;
    const float* G(int idx) const { return w->w + w->off_host[idx]; }
    const float* I(int blk, int idx) const { return w->w + w->off_host[NB200_DPP_G_COUNT + blk * NB200_DPP_I_COUNT + idx]; }
    const float* O(int blk, int idx) const {
        return w->w + w->off_host[NB200_DPP_G_COUNT + w->num_blocks * NB200_DPP_I_COUNT + blk * NB200_DPP_O_COUNT + idx];
    }
    // C[M, N] (ldc = N) = (acc ? C : 0) + A[M, K] op(B) (+ bias); act != nullptr: act = silu(C) (C keeps the pre-activation).
    // Mx.dev set: Mx.n is the bound (grid, kernel choice), rows at or beyond the device count are neither computed nor written.
    int gemm(Ext Mx, int N, int K, const float* A, const float* B, int trans, float* C, int acc, const float* bias, float* act) const {
        const int64_t M = Mx.n;
        if (M <= 0) return NB200_OK;
        if (M > 0x7fffffff) return NB200_EUNSUPPORTED;
        const int ldb = trans ? N : K;
#ifndef NB_EMU
        if (goc_tc_ok(N, K, K, ldb, N)) {
            Scope sc(e, s, CAT_GEMM, 1);
            return nb_gemm_tf32x3_ex((int)M, N, K, A, K, B, ldb, trans, C, N, acc, bias, act, NB_ACT_SILU, s, Mx.dev);
        }
#else
        if (goc_tc_ok(N, K, K, ldb, N)) {
            NB_TRY(emu_gemm_rows(e, s, (int)M, N, K, A, K, B, ldb, trans, C, N, acc, bias, Mx.dev));
            return act ? pfor(e, s, CAT_NODE, Mx, N, ActK{C, act}) : NB200_OK;
        }
#endif
        NB_TRY(pfor(e, s, CAT_GEMM, Mx, N, GemmK{A, K, B, ldb, trans, C, N, N, K, acc, bias}));
        return act ? pfor(e, s, CAT_NODE, Mx, N, ActK{C, act}) : NB200_OK;
    }
    // ResidualLayer: out = in + silu(W2 silu(W1 in + b1) + b2); keeps q1, q2 (pre-activations); tmp holds silu(q1)
    int res_fwd(Ext E, const float* in, int r, int blk, float* q1, float* q2, float* tmp, float* out) const {
        const float* W = I(blk, NB200_DPP_I_RES_W) + (int64_t)2 * r * H * H;
        const float* b = I(blk, NB200_DPP_I_RES_B) + (int64_t)2 * r * H;
        NB_TRY(gemm(E, H, H, in, W, 0, q1, 0, b, tmp));
        NB_TRY(gemm(E, H, H, tmp, W + (int64_t)H * H, 0, q2, 0, b + H, nullptr));
        return pfor(e, s, CAT_NODE, E, H, AddActK{in, q2, out});
    }
    // its reverse: gin = gout + ((gout * silu'(q2)) W2 * silu'(q1)) W1
    int res_bwd(Ext E, const float* gout, int r, int blk, const float* q1, const float* q2, float* t1, float* t2, float* gin) const {
        const float* W = I(blk, NB200_DPP_I_RES_W) + (int64_t)2 * r * H * H;
        NB_TRY(pfor(e, s, CAT_NODE, E, H, DActMulK{gout, q2, t1}));
        NB_TRY(gemm(E, H, H, t1, W + (int64_t)H * H, 1, t2, 0, nullptr, nullptr));
        NB_TRY(pfor(e, s, CAT_NODE, E, H, DActMulK{t2, q1, t2}));
        NB_TRY(goc_d2d(gin, gout, (size_t)E.n * H * sizeof(float), s));  // whole extent: rows past the count are copied, never read
        return gemm(E, H, H, t2, W, 1, gin, 1, nullptr, nullptr);
    }
};

// E: the edge extent -- the exact count (Edev == nullptr), or the bound with the count in device memory at Edev (the asynchronous call)
struct Geo {
    const GraphBuf* g; int64_t n, E; const int32_t* Edev = nullptr;
    Ext e() const { return Ext(E, Edev); }
};

int interaction_fwd(const Ctx& c, const Work& w, const Geo& q, int blk, const float* x, float* out) {
    const Ext E = q.e();
    const GraphBuf& g = *q.g;
    NB_TRY(c.gemm(E, H, H, x, c.I(blk, NB200_DPP_I_JI_W), 0, w.a, 0, c.I(blk, NB200_DPP_I_JI_B), w.h0));
    NB_TRY(c.gemm(E, H, H, x, c.I(blk, NB200_DPP_I_KJ_W), 0, w.bk, 0, c.I(blk, NB200_DPP_I_KJ_B), w.xk));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, MulRbfK{w.xk, w.rbf, c.I(blk, NB200_DPP_I_RBF), w.t}));
    NB_TRY(c.gemm(E, IE, H, w.t, c.I(blk, NB200_DPP_I_DOWN), 0, w.dpre, 0, nullptr, w.xd));
    NB_TRY(pfor(c.e, c.s, CAT_MSG_FWD, E, IE, TripFwdK{g.ptr, g.src, g.tgt, w.V, w.d, w.rbs, c.I(blk, NB200_DPP_I_SBF), w.xd, w.agg}));
    NB_TRY(c.gemm(E, H, IE, w.agg, c.I(blk, NB200_DPP_I_UP), 0, w.upre, 0, nullptr, nullptr));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, AddActK{w.h0, w.upre, w.h0}));
    NB_TRY(c.res_fwd(E, w.h0, 0, blk, w.q1[0], w.q2[0], w.t, w.h1));
    NB_TRY(c.gemm(E, H, H, w.h1, c.I(blk, NB200_DPP_I_LIN_W), 0, w.lpre, 0, c.I(blk, NB200_DPP_I_LIN_B), nullptr));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, LinOutK{w.lpre, x, w.h2}));
    NB_TRY(c.res_fwd(E, w.h2, 1, blk, w.q1[1], w.q2[1], w.t, w.h3));
    return c.res_fwd(E, w.h3, 2, blk, w.q1[2], w.q2[2], w.t, out);
}

// reverse of interaction block `blk` whose forward state is in the scratch: gO = dE/d(output) -> gI = dE/d(input), grbf / grbs / gct accumulate
int interaction_bwd(const Ctx& c, const Work& w, const Geo& q, int blk, const float* gO, float* gI) {
    const Ext E = q.e();
    const GraphBuf& g = *q.g;
    NB_TRY(c.res_bwd(E, gO, 2, blk, w.q1[2], w.q2[2], w.g2, w.g3, w.g1));   // g1 = d/dh3
    NB_TRY(c.res_bwd(E, w.g1, 1, blk, w.q1[1], w.q2[1], w.g2, w.g3, gI));   // gI = d/dh2 (the skip: d/dx starts here)
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, DActMulK{gI, w.lpre, w.g2}));
    NB_TRY(c.gemm(E, H, H, w.g2, c.I(blk, NB200_DPP_I_LIN_W), 1, w.g3, 0, nullptr, nullptr));  // d/dh1
    float* gh0 = w.t;  // the forward's t is not read by the reverse pass
    NB_TRY(c.res_bwd(E, w.g3, 0, blk, w.q1[0], w.q2[0], w.g1, w.g2, gh0));  // d/dh0 = d/dx_ji = d/dx_kj(up)
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, DActMulK{gh0, w.a, w.g1}));
    NB_TRY(c.gemm(E, H, H, w.g1, c.I(blk, NB200_DPP_I_JI_W), 1, gI, 1, nullptr, nullptr));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, DActMulK{gh0, w.upre, w.g2}));
    NB_TRY(c.gemm(E, IE, H, w.g2, c.I(blk, NB200_DPP_I_UP), 1, w.g64a, 0, nullptr, nullptr));  // d/dagg
    NB_TRY(pfor(c.e, c.s, CAT_MSG_BWD, E, IE, TripBwdXK{g.ptr, g.src, g.tgt, g.optr, g.oeid, w.V, w.d, w.rbs, c.I(blk, NB200_DPP_I_SBF), w.g64a, w.g64b}));
    NB_TRY(pfor(c.e, c.s, CAT_MSG_BWD, E, 1, TripBwdGK{g.ptr, g.src, g.tgt, g.rev, g.optr, g.oeid, g.tptr, w.V, w.d, w.rbs, c.I(blk, NB200_DPP_I_SBF1),
                                                   c.I(blk, NB200_DPP_I_SBF2), w.g64a, w.xd, w.grbs, w.gct}));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, IE, DActMulK{w.g64b, w.dpre, w.g64b}));
    NB_TRY(c.gemm(E, H, IE, w.g64b, c.I(blk, NB200_DPP_I_DOWN), 1, w.g3, 0, nullptr, nullptr));  // d/dt
    NB_TRY(pfor(c.e, c.s, CAT_FILTER, E, NRAD, RbfBwdK{nullptr, w.g3, w.xk, c.I(blk, NB200_DPP_I_RBF), w.grbf}));
    NB_TRY(pfor(c.e, c.s, CAT_NODE, E, H, KjBwdK{w.g3, w.rbf, c.I(blk, NB200_DPP_I_RBF), w.bk, w.g1}));
    return c.gemm(E, H, H, w.g1, c.I(blk, NB200_DPP_I_KJ_W), 1, gI, 1, nullptr, nullptr);
}

// output block `blk` on x: P (+)= lin(silu(lins(... lin_up(sum_e (W_rbf rbf) * x)))), pre-activations kept in oP[blk]
int output_fwd(const Ctx& c, const Work& w, const Geo& q, int blk, const float* x) {
    const int64_t n = q.n, NH = n * H;
    const int L = c.w->node_latent_dim;
    NB_TRY(pfor(c.e, c.s, CAT_READOUT, NH, AggOutK{q.g->ptr, w.rbf, c.O(blk, NB200_DPP_O_RBF), x, w.oA}));
    NB_TRY(c.gemm(n, OE, H, w.oA, c.O(blk, NB200_DPP_O_UP), 0, w.oU, 0, nullptr, nullptr));
    const float* in = w.oU;
    float* tmp[2] = {w.oT1, w.oT2};
    for (int k = 0; k < NLIN; k++) {
        NB_TRY(c.gemm(n, OE, OE, in, c.O(blk, NB200_DPP_O_LINS_W) + (int64_t)k * OE * OE, 0, w.oP + ((int64_t)blk * NLIN + k) * NH, 0,
                      c.O(blk, NB200_DPP_O_LINS_B) + (int64_t)k * OE, tmp[k & 1]));
        in = tmp[k & 1];
    }
    return c.gemm(n, L, OE, in, c.O(blk, NB200_DPP_O_LIN), 0, w.P, blk > 0, nullptr, nullptr);
}
// its reverse from gP: gx (+)= d/dx, grbf += d/drbf
int output_bwd(const Ctx& c, const Work& w, const Geo& q, int blk, const float* x, float* gx, int acc) {
    const int64_t n = q.n, NH = n * H;
    const int L = c.w->node_latent_dim;
    NB_TRY(c.gemm(n, OE, L, w.gP, c.O(blk, NB200_DPP_O_LIN), 1, w.oT1, 0, nullptr, nullptr));
    float* cur = w.oT1;
    float* nxt = w.oT2;
    for (int k = NLIN - 1; k >= 0; k--) {
        NB_TRY(pfor(c.e, c.s, CAT_NODE, NH, DActMulK{cur, w.oP + ((int64_t)blk * NLIN + k) * NH, cur}));
        NB_TRY(c.gemm(n, OE, OE, cur, c.O(blk, NB200_DPP_O_LINS_W) + (int64_t)k * OE * OE, 1, nxt, 0, nullptr, nullptr));
        float* t = cur; cur = nxt; nxt = t;
    }
    NB_TRY(c.gemm(n, H, OE, cur, c.O(blk, NB200_DPP_O_UP), 1, w.oA, 0, nullptr, nullptr));  // d/dA
    NB_TRY(pfor(c.e, c.s, CAT_READOUT, q.e(), H, OutBwdXK{q.g->tgt, w.rbf, c.O(blk, NB200_DPP_O_RBF), w.oA, gx, acc}));
    return pfor(c.e, c.s, CAT_FILTER, q.e(), NRAD, RbfBwdK{q.g->tgt, w.oA, x, c.O(blk, NB200_DPP_O_RBF), w.grbf});
}

int graph_phase(nb200_engine* e, cudaStream_t s, const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                int32_t n_mol, int32_t n, const GraphBuf& g) {
    const float cut2 = w->cutoff * w->cutoff;
    const int32_t kcap = w->max_neighbors + 1;
    NB_TRY(pfor(e, s, CAT_NBR, n, MolIdK{mol_ptr, n_mol, g.mol_id}));
    NB_TRY(pfor(e, s, CAT_NBR, n, NbrK{pos, z, mol_ptr, g.mol_id, cut2, kcap, nullptr, g.deg, g.bad, nullptr, nullptr}));
    NB_TRY(scan_excl(e, s, g.deg, n, g.ptr));
    NB_TRY(scan_excl(e, s, g.bad, n, g.badscan));
    NB_TRY(pfor(e, s, CAT_NBR, n, NbrK{pos, z, mol_ptr, g.mol_id, cut2, kcap, g.ptr, g.deg, g.bad, g.src, g.tgt}));
    NB_TRY(pfor(e, s, CAT_NBR, Ext(g.emax, g.ptr + n), 1, RevK{g.ptr, g.src, g.tgt, g.rev}));
    NB_TRY(pfor(e, s, CAT_NBR, n, OutK{g.ptr, g.src, mol_ptr, g.mol_id, nullptr, g.odeg, g.oeid}));
    NB_TRY(scan_excl(e, s, g.odeg, n, g.optr));
    NB_TRY(pfor(e, s, CAT_NBR, n, OutK{g.ptr, g.src, mol_ptr, g.mol_id, g.optr, g.odeg, g.oeid}));
    NB_TRY(pfor(e, s, CAT_NBR, g.emax, TcntK{g.ptr, g.src, g.rev, g.ptr + n, g.tcnt}));
    NB_TRY(scan_excl(e, s, g.tcnt, (int32_t)g.emax, g.tptr));
    return pfor(e, s, CAT_NBR, 1, TotK{g.ptr + n, g.tptr + g.emax, g.badscan + n, g.tot});
}

bool sizes_ok(int32_t n_mol, int32_t n_atoms, int32_t max_neighbors) {
    return n_mol >= 1 && n_atoms >= 1 && (int64_t)n_atoms * (max_neighbors + 1) < 0x7fffffff;
}

// the energy-and-forces pass on a carved graph and workspace (arguments checked by the caller).  forces == nullptr: GeomBwdK and ForceK do not
// run; grbf, grbs and gct are left holding dy/drbf, dy/drbs and dy/dcos either way
int energy_forces_pass(const Ctx& c, const Work& wk, const Geo& q, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                       int64_t T, float* energy, float* forces, float* graph_emb) {
    nb200_engine* eng = c.e;
    cudaStream_t s = c.s;
    const nb200_dimenet_weights* w = c.w;
    const GraphBuf& g = *q.g;
    const int64_t E = q.E, n_atoms = q.n;
    const Ext Ex = q.e();  // every edge-row launch and GEMM stops at the device count when there is one
    const int nb = w->num_blocks, L = w->node_latent_dim;
    const int64_t EH = E * H;
    const float inv_cut = 1.0f / w->cutoff;
    // geometry and bases
    NB_TRY(pfor(eng, s, CAT_FILTER, Ex, 1, GeomK{pos, g.src, g.tgt, wk.V, wk.d}));
    NB_TRY(pfor(eng, s, CAT_FILTER, Ex, NRAD, RbfK{wk.d, c.G(NB200_DPP_G_FREQ), inv_cut, wk.rbf}));
    NB_TRY(pfor(eng, s, CAT_FILTER, Ex, NSR, RbsK{wk.d, c.G(NB200_DPP_G_ZEROS), c.G(NB200_DPP_G_NORMS), inv_cut, wk.rbs, wk.drbs}));
    // embedding block
    NB_TRY(pfor(eng, s, CAT_EMBED, Ex, H, EmbRbfK{wk.rbf, c.G(NB200_DPP_G_EMB_RBF_W), c.G(NB200_DPP_G_EMB_RBF_B), wk.hr, wk.hra}));
    NB_TRY(c.gemm(Ex, H, H, wk.hra, c.G(NB200_DPP_G_EMB_W3), 0, wk.epre, 0, nullptr, nullptr));
    NB_TRY(pfor(eng, s, CAT_EMBED, Ex, H, EmbAddK{z, g.src, g.tgt, c.G(NB200_DPP_G_EMB_TI), c.G(NB200_DPP_G_EMB_TJ), wk.epre, wk.X}));
    // blocks
    NB_TRY(output_fwd(c, wk, q, 0, wk.X));
    for (int b = 0; b < nb; b++) {
        NB_TRY(interaction_fwd(c, wk, q, b, wk.X + b * EH, wk.X + (b + 1) * EH));
        NB_TRY(output_fwd(c, wk, q, b + 1, wk.X + (b + 1) * EH));
    }
    // regression head: energy and dy/d(graph embedding)
    NB_TRY(pfor(eng, s, CAT_READOUT, n_mol, HeadK{mol_ptr, wk.P, L, c.G(NB200_DPP_G_HEAD_W0), c.G(NB200_DPP_G_HEAD_B0), c.G(NB200_DPP_G_HEAD_W1),
                                                  c.G(NB200_DPP_G_HEAD_B1), c.G(NB200_DPP_G_HEAD_W2), c.G(NB200_DPP_G_HEAD_B2), c.G(NB200_DPP_G_HEAD_W3),
                                                  c.G(NB200_DPP_G_HEAD_B3), w->scale, w->mean, graph_emb, wk.gG, energy}));
    // reverse pass
    NB_TRY(pfor(eng, s, CAT_READOUT, n_atoms * L, BcastK{g.mol_id, wk.gG, L, wk.gP}));
    if (E > 0) {
        NB_TRY(goc_memset(wk.grbf, 0, (size_t)E * NRAD * sizeof(float), s));
        NB_TRY(goc_memset(wk.grbs, 0, (size_t)E * NSR * sizeof(float), s));
        if (T > 0) NB_TRY(goc_memset(wk.gct, 0, (size_t)T * sizeof(float), s));
    }
    float* gx = wk.gX;
    float* gprev = wk.gI;
    NB_TRY(output_bwd(c, wk, q, nb, wk.X + nb * EH, gx, 0));
    for (int b = nb - 1; b >= 0; b--) {
        if (b != nb - 1) NB_TRY(interaction_fwd(c, wk, q, b, wk.X + b * EH, wk.out));  // the scratch holds block nb - 1 after the forward
        NB_TRY(interaction_bwd(c, wk, q, b, gx, gprev));
        NB_TRY(output_bwd(c, wk, q, b, wk.X + b * EH, gprev, 1));
        float* t = gx; gx = gprev; gprev = t;
    }
    // embedding block reverse: gx = d/dx0
    NB_TRY(pfor(eng, s, CAT_EMBED, Ex, H, DActMulK{gx, wk.epre, wk.g1}));
    NB_TRY(c.gemm(Ex, H, H, wk.g1, c.G(NB200_DPP_G_EMB_W3), 1, wk.g2, 0, nullptr, nullptr));
    NB_TRY(pfor(eng, s, CAT_EMBED, Ex, H, DActMulK{wk.g2, wk.hr, wk.g2}));
    NB_TRY(pfor(eng, s, CAT_FILTER, Ex, NRAD, RbfBwdK{nullptr, wk.g2, nullptr, c.G(NB200_DPP_G_EMB_RBF_W), wk.grbf}));
    if (!forces) return NB200_OK;
    // geometry reverse and forces
    NB_TRY(pfor(eng, s, CAT_FORCE, Ex, 1, GeomBwdK{g.ptr, g.src, g.tgt, g.rev, g.optr, g.oeid, g.tptr, wk.V, wk.d, wk.rbf, c.G(NB200_DPP_G_FREQ), inv_cut,
                                               wk.grbf, wk.drbs, wk.grbs, wk.gct, wk.gV}));
    return pfor(eng, s, CAT_FORCE, 3 * n_atoms, ForceK{g.ptr, g.optr, g.oeid, wk.gV, forces});
}

}  // namespace

extern "C" int64_t nb200_dimenet_graph_bytes(const nb200_dimenet_weights* w, int32_t n_atoms) {
    NB_TRY(config_rc(w));
    if (n_atoms < 1 || !sizes_ok(1, n_atoms, w->max_neighbors)) return NB200_EINVAL;
    return carve_graph(nullptr, n_atoms, w->max_neighbors + 1).bytes;
}

extern "C" int nb200_dimenet_graph_count(const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                                         int32_t n_atoms, void* graph_buf, int64_t graph_bytes, int64_t* counts_host, void* stream) {
    NB_TRY(config_rc(w));
    if (!z || !pos || !mol_ptr || !graph_buf || !counts_host || !sizes_ok(n_mol, n_atoms, w->max_neighbors)) return NB200_EINVAL;
    if (graph_bytes < carve_graph(nullptr, n_atoms, w->max_neighbors + 1).bytes) return NB200_EINVAL;
    const GraphBuf g = carve_graph(graph_buf, n_atoms, w->max_neighbors + 1);
    cudaStream_t s = (cudaStream_t)stream;
    nb200_engine* e = nullptr;
#ifndef NB_EMU
    nb200_engine tmp_engine{};  // launch counting only
    e = &tmp_engine;
#endif
    NB_TRY(graph_phase(e, s, w, z, pos, mol_ptr, n_mol, n_atoms, g));
    int32_t tot[4];
    NB_TRY(goc_d2h_sync(tot, g.tot, 3 * sizeof(int32_t), s));
    for (int k = 0; k < NB200_DPP_C_COUNT; k++) counts_host[k] = 0;
    if (tot[2] != 0) return NB200_EINVAL;  // z outside [0, 94] or a non-finite coordinate
    if (tot[0] < 0 || tot[1] < 0) return NB200_ECAPACITY;
    counts_host[NB200_DPP_C_EDGES] = tot[0];
    counts_host[NB200_DPP_C_TRIPLETS] = tot[1];
    return NB200_OK;
}

extern "C" int64_t nb200_dimenet_workspace_bytes(const nb200_dimenet_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host) {
    NB_TRY(config_rc(w));
    if (!counts_host || n_mol < 1 || n_atoms < 1 || counts_host[NB200_DPP_C_EDGES] < 0 || counts_host[NB200_DPP_C_TRIPLETS] < 0) return NB200_EINVAL;
    return carve_work(nullptr, w->num_blocks, n_mol, n_atoms, counts_host[NB200_DPP_C_EDGES], counts_host[NB200_DPP_C_TRIPLETS], w->node_latent_dim).bytes;
}

extern "C" int nb200_dimenet_energy_forces(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                           int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes, const int64_t* counts_host,
                                           void* workspace, int64_t workspace_bytes, float* energy, float* forces, float* graph_emb, void* stream) {
    NB_TRY(config_rc(w));
    if (!eng || !z || !pos || !mol_ptr || !graph_buf || !counts_host || !workspace || !energy || !forces || !sizes_ok(n_mol, n_atoms, w->max_neighbors))
        return NB200_EINVAL;
    const int64_t E = counts_host[NB200_DPP_C_EDGES], T = counts_host[NB200_DPP_C_TRIPLETS];
    const int64_t kcap = w->max_neighbors + 1;
    if (E < 0 || T < 0 || E > (int64_t)n_atoms * kcap || graph_bytes < carve_graph(nullptr, n_atoms, kcap).bytes ||
        workspace_bytes < carve_work(nullptr, w->num_blocks, n_mol, n_atoms, E, T, w->node_latent_dim).bytes)
        return NB200_EINVAL;  // before any pointer is formed
    const GraphBuf g = carve_graph(graph_buf, n_atoms, kcap);
    const Work wk = carve_work(workspace, w->num_blocks, n_mol, n_atoms, E, T, w->node_latent_dim);
    const Ctx c{eng, (cudaStream_t)stream, w};
    const Geo q{&g, n_atoms, E};
    return energy_forces_pass(c, wk, q, z, pos, mol_ptr, n_mol, T, energy, forces, graph_emb);
}

// Upper bounds of the counts from the molecule sizes alone (DESIGN.md 3.15.3).  Every edge lives inside one molecule.  For a molecule of m
// atoms and kcap = max_neighbors + 1, NbrK keeps the first kcap in-cutoff candidates of a target in index order, the target itself included
// (d = 0), then drops it.  A target at position t < kcap of its molecule has at most t atoms before it, so it is always among its own first
// kcap candidates and keeps at most min(m - 1, kcap - 1) sources; a later one keeps at most kcap.  Edge j -> i has indeg(j) - [i -> j
// exists] triplet slots (TcntK); indeg(j) <= min(m - 1, kcap), and indeg(j) = m - 1 means every other atom, i included, is a source of j, so
// an edge has at most min(m - 2, kcap) slots.  A compact molecule (every pair inside the cutoff) attains the edge bound, and for
// m <= kcap the slot bound too.
extern "C" int nb200_dimenet_count_bounds(const nb200_dimenet_weights* w, const int32_t* mol_ptr_host, int32_t n_mol, int64_t* bounds) {
    NB_TRY(config_rc(w));
    if (!mol_ptr_host || !bounds || n_mol < 1 || mol_ptr_host[0] != 0) return NB200_EINVAL;
    const int64_t kcap = w->max_neighbors + 1;
    int64_t E = 0, T = 0;
    for (int32_t i = 0; i < n_mol; i++) {
        const int64_t m = (int64_t)mol_ptr_host[i + 1] - mol_ptr_host[i];
        if (m < 1) return NB200_EINVAL;
        const int64_t lo = m < kcap ? m : kcap;  // targets among their own first kcap candidates
        const int64_t e = lo * (m - 1 < kcap - 1 ? m - 1 : kcap - 1) + (m - lo) * kcap;
        E += e;
        T += m < 2 ? 0 : e * (m - 2 < kcap ? m - 2 : kcap);
        if (E > 0x7fffffff || T > 0x7fffffff) return NB200_EINVAL;  // the row pointers (ptr, tptr) are int32 scans
    }
    if (!sizes_ok(n_mol, mol_ptr_host[n_mol], w->max_neighbors)) return NB200_EINVAL;
    for (int k = 0; k < NB200_DPP_C_COUNT; k++) bounds[k] = 0;
    bounds[NB200_DPP_C_EDGES] = E;
    bounds[NB200_DPP_C_TRIPLETS] = T;
    return NB200_OK;
}

// Graph phase and energy-and-forces pass in one enqueue: no host read, no synchronisation.  Edge extents are the bounds; the counts stay on
// the device and are checked against the bounds before the pass writes any edge or triplet row.
extern "C" int nb200_dimenet_energy_forces_async(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos,
                                                 const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes,
                                                 const int64_t* bounds, void* workspace, int64_t workspace_bytes, float* energy, float* forces,
                                                 int32_t* status, void* stream) {
    NB_TRY(config_rc(w));
    if (!eng || !z || !pos || !mol_ptr || !graph_buf || !bounds || !workspace || !energy || !forces || !status ||
        !sizes_ok(n_mol, n_atoms, w->max_neighbors))
        return NB200_EINVAL;
    const int64_t kcap = w->max_neighbors + 1, Eb = bounds[NB200_DPP_C_EDGES], Tb = bounds[NB200_DPP_C_TRIPLETS];
    if (Eb < 0 || Tb < 0 || Eb > (int64_t)n_atoms * kcap || Tb > 0x7fffffff || graph_bytes < carve_graph(nullptr, n_atoms, kcap).bytes ||
        workspace_bytes < carve_work(nullptr, w->num_blocks, n_mol, n_atoms, Eb, Tb, w->node_latent_dim).bytes)
        return NB200_EINVAL;  // before any pointer is formed
    const GraphBuf g = carve_graph(graph_buf, n_atoms, kcap);
    const Work wk = carve_work(workspace, w->num_blocks, n_mol, n_atoms, Eb, Tb, w->node_latent_dim);
    cudaStream_t s = (cudaStream_t)stream;
    NB_TRY(graph_phase(eng, s, w, z, pos, mol_ptr, n_mol, n_atoms, g));
    NB_TRY(goc_memset(status, 0, 8 * sizeof(int32_t), s));
    NB_TRY(pfor(eng, s, CAT_NBR, n_atoms, StatusAtomK{g.bad, g.deg, status}));
    NB_TRY(pfor(eng, s, CAT_NBR, 1, StatusCountsK{g.ptr + n_atoms, g.tptr + g.emax, (int32_t)Eb, (int32_t)Tb, status}));
    NB_TRY(pfor(eng, s, CAT_NBR, 2 * ((int64_t)n_atoms + 1), ClearOnErrorK{status, g.ptr, g.optr, (int64_t)n_atoms + 1}));
    const Ctx c{eng, s, w};
    const Geo q{&g, n_atoms, Eb, g.ptr + n_atoms};
    NB_TRY(energy_forces_pass(c, wk, q, z, pos, mol_ptr, n_mol, Tb, energy, forces, nullptr));
    return pfor(eng, s, CAT_READOUT, (int64_t)n_mol + 3 * (int64_t)n_atoms, NanOnErrorK{status, energy, n_mol, forces});
}

extern "C" int nb200_dimenet_debug_sbf_radial(const nb200_dimenet_weights* w, const float* dist, int32_t n, float* rbs, float* drbs, void* stream) {
    NB_TRY(config_rc(w));
    if (!dist || !rbs || !drbs || n < 0) return NB200_EINVAL;
    nb200_engine* e = nullptr;
#ifndef NB_EMU
    nb200_engine tmp_engine{};
    e = &tmp_engine;
#endif
    const Ctx c{e, (cudaStream_t)stream, w};
    return pfor(e, c.s, CAT_FILTER, (int64_t)n * NSR, RbsK{dist, c.G(NB200_DPP_G_ZEROS), c.G(NB200_DPP_G_NORMS), 1.0f / w->cutoff, rbs, drbs});
}

#ifdef NB_EMU
// the test entry of gemm_tc.cu in the emulation build, on the emulated GEMM (no act output: the engine applies the activation separately)
extern "C" int nb200_gemm_tf32x3_rows(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb, int32_t trans_b,
                                      float* C, int32_t ldc, int32_t accumulate, const float* bias, float* act, const int32_t* m_dev, void* stream) {
    if (!A || !B || !C || act || M < 0 || N <= 0 || K <= 0) return NB200_EINVAL;
    return emu_gemm_rows(nullptr, (cudaStream_t)stream, M, N, K, A, lda, B, ldb, trans_b, C, ldc, accumulate, bias, m_dev);
}
#endif

#include "dimenet_train.inc"
#include "dimenet_hvp.inc"
