// schnet_train.cu -- SchNet parameter gradients of an energy loss (SURVEY.md section 8 a8 + a10/a11; BASELINE configs[0]: SchNet energy-only
// training).  First correct path, NOT YET RUN ON A DEVICE: verified on the CPU through the host-emulation build (tests/emu,
// tests/test_schnet_train_emu.py) against the autograd of the oracle (oracle/spk.py).
//
// Reference: schnetpack 2.0.4 SchNet / Atomwise as wired by config/model/schnet.yaml (SURVEY.md A.1) trained by `loss.backward()` through the
// eager graph (nablaDFT/ase_model/task.py).  Here ONE call does the forward with saved activations and the reverse sweep:
//     grads = d( sum_m seed_m E_m ) / d(canonical weights),   seed = dLoss/dE from the autograd bridge (nabladft_b200/training.py).
// The neighbour relation is symmetric and the filter of an edge depends on its length only, so both the cfconv forward and its backward
// w.r.t. the source features are GATHERS over the CSR row of the receiving atom -- the same kernel (CfconvK) serves both; no atomics there.
// Weight gradients G^T X are row-chunked functor reductions with atomicAdd into zeroed buffers (cuBLAS would do on the device; the functor
// keeps the emulated and the device code identical).  A force loss (the reference's create_graph double backward) is handled as in the PaiNN
// engine (DESIGN.md 3.7): sum_i v_i . dF_i/dtheta = -(v . d/dR)[dE_tot/dtheta], i.e. a second reverse sweep with unit seeds that carries the
// tangent of every forward and backward quantity along v in position space.
#include "gemnet_pf.cuh"

namespace {

constexpr int F = 128;  // n_atom_basis = n_filters (config/model/schnet.yaml)
constexpr int H = 64;   // Atomwise hidden width F / 2
constexpr int WG_ROWS = 1024;
constexpr float LN2 = 0.69314718055994530942f;

GD float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }
GD float sspf(float x) { return (x > 20.0f ? x : log1pf(expf(x))) - LN2; }  // shifted softplus, torch's threshold-20 linearisation
GD float siluf(float x) { return x * sigm(x); }
GD float dsiluf(float x) { const float s = sigm(x); return s * (1.0f + x * (1.0f - s)); }

struct SMolIdK {
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
// ase.neighborlist.neighbor_list('ijS', cutoff) for a molecule: both directions, d < cutoff (strict), no self pairs
struct SDegK {
    const float* pos; const int32_t* mol_ptr; const int32_t* mol_id; float cut2; int32_t* deg;
    GD void operator()(int64_t a) const {
        const int32_t m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        const float ax = pos[3 * a], ay = pos[3 * a + 1], az = pos[3 * a + 2];
        int32_t c = 0;
        for (int32_t j = m0; j < m1; j++) {
            if (j == (int32_t)a) continue;
            const float dx = pos[3 * j] - ax, dy = pos[3 * j + 1] - ay, dz = pos[3 * j + 2] - az;
            c += (dx * dx + dy * dy + dz * dz < cut2) ? 1 : 0;
        }
        deg[a] = c;
    }
};
struct SFillK {
    const float* pos; const int32_t* mol_ptr; const int32_t* mol_id; const int32_t* row_ptr; float cut2, cutoff; int32_t* col; int32_t* tgt; float* d; float* rcut;
    GD void operator()(int64_t ai) const {
        const int32_t a = (int32_t)ai, m0 = mol_ptr[mol_id[a]], m1 = mol_ptr[mol_id[a] + 1];
        const float ax = pos[3 * a], ay = pos[3 * a + 1], az = pos[3 * a + 2];
        int32_t e = row_ptr[a];
        for (int32_t j = m0; j < m1; j++) {
            if (j == a) continue;
            const float dx = pos[3 * j] - ax, dy = pos[3 * j + 1] - ay, dz = pos[3 * j + 2] - az;
            const float d2 = dx * dx + dy * dy + dz * dz;
            if (!(d2 < cut2)) continue;
            const float dd = sqrtf(d2);
            col[e] = j; tgt[e] = a; d[e] = dd;
            rcut[e] = 0.5f * (cosf(dd * (3.14159265358979323846f / cutoff)) + 1.0f);  // CosineCutoff; d < cutoff holds here
            e++;
        }
    }
};
struct SPhiK {  // GaussianRBF: exp(coeff (d - mu_k)^2)
    const float* d; const float* offsets; float coeff; int32_t K; float* phi;
    GD void operator()(int64_t i) const {
        const float t = d[i / K] - offsets[i % K];
        phi[i] = expf(coeff * t * t);
    }
};
struct SEmbedK {
    const int32_t* z; const float* emb; int32_t n_elem, z_offset; float* x;
    GD void operator()(int64_t i) const {
        int32_t r = z[i / F] - z_offset;
        r = r < 0 ? 0 : (r >= n_elem ? n_elem - 1 : r);
        x[i] = emb[(int64_t)r * F + (i % F)];
    }
};
// out[r, n] = bias[n] + sum_k A[r, k] Wt[k, n]     (Wt K-major: the canonical layout of filter_network.0)
struct SLinKmajorK {
    const float* A; int32_t K; const float* Wt; const float* bias; float* out; int32_t N;
    GD void operator()(int64_t i) const {
        const int64_t r = i / N; const int n = (int)(i % N);
        const float* a = A + r * K;
        float s0 = 0.0f, s1 = 0.0f;
        int k = 0;
        for (; k + 2 <= K; k += 2) { s0 += a[k] * Wt[(int64_t)k * N + n]; s1 += a[k + 1] * Wt[(int64_t)(k + 1) * N + n]; }
        if (k < K) s0 += a[k] * Wt[(int64_t)k * N + n];
        out[i] = s0 + s1 + (bias ? bias[n] : 0.0f);
    }
};
// C[r, n] (+)= bias[n] + sum_k A[r, k] W[n, k]   (torch.nn.Linear forward)
struct SLinK {
    const float* A; int32_t K; const float* W; const float* bias; float* C; int32_t N; int32_t accumulate;
    GD void operator()(int64_t i) const {
        const int64_t r = i / N; const int n = (int)(i % N);
        const float* a = A + r * K; const float* w = W + (int64_t)n * K;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
        int k = 0;
        for (; k + 4 <= K; k += 4) { s0 += a[k] * w[k]; s1 += a[k + 1] * w[k + 1]; s2 += a[k + 2] * w[k + 2]; s3 += a[k + 3] * w[k + 3]; }
        for (; k < K; k++) s0 += a[k] * w[k];
        const float v = (s0 + s1) + (s2 + s3) + (bias ? bias[n] : 0.0f);
        C[i] = accumulate ? C[i] + v : v;
    }
};
// C[r, k] (+)= sum_n G[r, n] W[n, k]   (Linear backward w.r.t. its input)
struct SLinBwdK {
    const float* G; int32_t N; const float* W; float* C; int32_t K; int32_t accumulate;
    GD void operator()(int64_t i) const {
        const int64_t r = i / K; const int k = (int)(i % K);
        const float* g = G + r * N;
        float s0 = 0.0f, s1 = 0.0f;
        int n = 0;
        for (; n + 2 <= N; n += 2) { s0 += g[n] * W[(int64_t)n * K + k]; s1 += g[n + 1] * W[(int64_t)(n + 1) * K + k]; }
        if (n < N) s0 += g[n] * W[(int64_t)n * K + k];
        C[i] = accumulate ? C[i] + (s0 + s1) : (s0 + s1);
    }
};
// dW[n, k] += sum over a chunk of rows of G[r, n] X[r, k];  i = (chunk, n, k)
struct SWgradK {
    const float* G; int32_t N; const float* X; int32_t K; int64_t M; float* dW; float alpha;
    GD void operator()(int64_t i) const {
        const int64_t nk = (int64_t)N * K, chunk = i / nk;
        const int n = (int)((i % nk) / K), k = (int)(i % K);
        const int64_t r0 = chunk * WG_ROWS, r1 = r0 + WG_ROWS < M ? r0 + WG_ROWS : M;
        float s = 0.0f;
        for (int64_t r = r0; r < r1; r++) s += G[r * N + n] * X[r * K + k];
        atomicAdd(dW + (int64_t)n * K + k, alpha * s);
    }
};
struct SColsumK {  // db[n] += alpha * sum over a chunk of rows of G[r, n];  i = (chunk, n)
    const float* G; int32_t N; int64_t M; float* db; float alpha;
    GD void operator()(int64_t i) const {
        const int64_t chunk = i / N; const int n = (int)(i % N);
        const int64_t r0 = chunk * WG_ROWS, r1 = r0 + WG_ROWS < M ? r0 + WG_ROWS : M;
        float s = 0.0f;
        for (int64_t r = r0; r < r1; r++) s += G[r * N + n];
        atomicAdd(db + n, alpha * s);
    }
};
struct SSspK {  // out = ssp(x)
    const float* x; float* out;
    GD void operator()(int64_t i) const { out[i] = sspf(x[i]); }
};
struct SRowScaleK {  // x[e, :] *= s[e]
    float* x; const float* s;
    GD void operator()(int64_t i) const { x[i] *= s[i / F]; }
};
struct SMulSigK {  // g *= sigmoid(pre)   (ssp' = sigmoid)
    float* g; const float* pre;
    GD void operator()(int64_t i) const { g[i] *= sigm(pre[i]); }
};
// continuous-filter convolution as a gather: out[i, f] = sum over e in row i of src[col[e], f] * Wf[e, f]
struct SCfconvK {
    const int32_t* row_ptr; const int32_t* col; const float* src; const float* Wf; float* out;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / F); const int f = (int)(i % F);
        float s = 0.0f;
        for (int32_t e = row_ptr[a]; e < row_ptr[a + 1]; e++) s += src[(int64_t)col[e] * F + f] * Wf[(int64_t)e * F + f];
        out[i] = s;
    }
};
struct SEdgeProdK {  // g_filter_pre[e, f] = g_agg[tgt[e], f] * y[col[e], f] * rcut[e]
    const int32_t* tgt; const int32_t* col; const float* g_agg; const float* y; const float* rcut; float* out;
    GD void operator()(int64_t i) const {
        const int64_t e = i / F; const int f = (int)(i % F);
        out[i] = g_agg[(int64_t)tgt[e] * F + f] * y[(int64_t)col[e] * F + f] * rcut[e];
    }
};
struct SAddK {
    float* x; const float* v;
    GD void operator()(int64_t i) const { x[i] += v[i]; }
};
struct SReadoutK {  // e_atom = silu(rpre) . R2 + e2 + shift
    const float* rpre; const float* R2; const float* e2; float shift; float* e_atom;
    GD void operator()(int64_t a) const {
        const float* p = rpre + a * H;
        float s = 0.0f;
        for (int k = 0; k < H; k++) s += siluf(p[k]) * R2[k];
        e_atom[a] = s + e2[0] + shift;
    }
};
struct SMolSumK {
    const int32_t* mol_ptr; const float* e_atom; float* energy;
    GD void operator()(int64_t m) const {
        float s = 0.0f;
        for (int32_t a = mol_ptr[m]; a < mol_ptr[m + 1]; a++) s += e_atom[a];
        energy[m] = s;
    }
};
struct SSeedK {  // r = silu(rpre) (for dR2), g_rpre = seed[mol] * R2 * silu'(rpre), g_e = seed[mol]
    const int32_t* mol_id; const float* seed; const float* rpre; const float* R2; float* r; float* g_rpre; float* g_e;
    GD void operator()(int64_t i) const {
        const int64_t a = i / H; const int k = (int)(i % H);
        const float c = seed[mol_id[a]], p = rpre[i];
        r[i] = siluf(p);
        g_rpre[i] = c * R2[k] * dsiluf(p);
        if (k == 0) g_e[a] = c;
    }
};
struct SEmbGradK {  // dEmb[row, f] += alpha * sum over atoms of that element of g_x0[a, f];  i = (row, f)
    const int32_t* z; int32_t z_offset, n_elem; const float* g; int32_t n_atoms; float* demb; float alpha;
    GD void operator()(int64_t i) const {
        const int32_t row = (int32_t)(i / F); const int f = (int)(i % F);
        float s = 0.0f;
        for (int32_t a = 0; a < n_atoms; a++) {
            int32_t r = z[a] - z_offset;
            r = r < 0 ? 0 : (r >= n_elem ? n_elem - 1 : r);
            if (r == row) s += g[(int64_t)a * F + f];
        }
        demb[i] += alpha * s;
    }
};


// ------------------------------------------------------------------ tangent (directional derivative along v in position space) functors.
// The force term of a loss needs  sum_i v_i . dF_i/dtheta = -(v . d/dR)[ dE_tot/dtheta ]  (mixed partials commute, DESIGN.md 3.7): every
// forward activation x gets a tangent xd = (v . d/dR) x, every backward quantity g (seed 1) a tangent gd, and each weight gradient G^T X
// contributes -(Gd^T X + G^T Xd).
struct STanGeomK {  // dd = u . (v_j - v_i);  rcd = d rcut/dd * dd
    const float* pos; const float* v; const int32_t* col; const int32_t* tgt; const float* d; float cutoff; float* dd; float* rcd;
    GD void operator()(int64_t e) const {
        const int32_t i = tgt[e], j = col[e];
        const float rx = pos[3 * j] - pos[3 * i], ry = pos[3 * j + 1] - pos[3 * i + 1], rz = pos[3 * j + 2] - pos[3 * i + 2];
        const float t = (rx * (v[3 * j] - v[3 * i]) + ry * (v[3 * j + 1] - v[3 * i + 1]) + rz * (v[3 * j + 2] - v[3 * i + 2])) / d[e];
        const float a = 3.14159265358979323846f / cutoff;
        dd[e] = t;
        rcd[e] = -0.5f * a * sinf(d[e] * a) * t;
    }
};
struct SPhiTanK {  // phid = phi * 2 coeff (d - mu_k) dd
    const float* d; const float* dd; const float* offsets; float coeff; int32_t K; const float* phi; float* phid;
    GD void operator()(int64_t i) const {
        const int64_t e = i / K;
        phid[i] = phi[i] * 2.0f * coeff * (d[e] - offsets[i % K]) * dd[e];
    }
};
struct SMulSigOutK {  // out = in * sigmoid(pre)
    const float* in; const float* pre; float* out;
    GD void operator()(int64_t i) const { out[i] = in[i] * sigm(pre[i]); }
};
// filter = fpre * rcut and its tangent fpred * rcut + fpre * rcd, in place over (fpre, fpred)
struct SFilterTanK {
    float* f; float* fd; const float* rcut; const float* rcd;
    GD void operator()(int64_t i) const {
        const int64_t e = i / F;
        const float a = f[i];
        f[i] = a * rcut[e];
        fd[i] = fd[i] * rcut[e] + a * rcd[e];
    }
};
struct SCfconv2K {  // out[i] = sum_e (s1[col] W1[e] + s2[col] W2[e])
    const int32_t* row_ptr; const int32_t* col; const float* s1; const float* W1; const float* s2; const float* W2; float* out;
    GD void operator()(int64_t i) const {
        const int32_t a = (int32_t)(i / F); const int f = (int)(i % F);
        float s = 0.0f;
        for (int32_t e = row_ptr[a]; e < row_ptr[a + 1]; e++) {
            const int64_t c = (int64_t)col[e] * F + f, w = (int64_t)e * F + f;
            s += s1[c] * W1[w] + s2[c] * W2[w];
        }
        out[i] = s;
    }
};
// seed 1: r, rd, g_rpre = R2 silu'(p), gd_rpre = R2 silu''(p) pd
struct SSeedTanK {
    const float* rpre; const float* rpred; const float* R2; float* r; float* rd; float* g_rpre; float* gd_rpre; float* g_e;
    GD void operator()(int64_t i) const {
        const int k = (int)(i % H);
        const float p = rpre[i], pd = rpred[i], sg = sigm(p);
        const float d1 = sg * (1.0f + p * (1.0f - sg)), d2 = sg * (1.0f - sg) * (2.0f + p * (1.0f - 2.0f * sg));
        r[i] = p * sg;
        rd[i] = d1 * pd;
        g_rpre[i] = R2[k] * d1;
        gd_rpre[i] = R2[k] * d2 * pd;
        if (k == 0) g_e[i / H] = 1.0f;
    }
};
// through ssp backward: g <- g sigma(pre);  gd <- gd sigma(pre) + g_in sigma'(pre) pred
struct SMulSigTanK {
    float* g; float* gd; const float* pre; const float* pred;
    GD void operator()(int64_t i) const {
        const float sg = sigm(pre[i]), gi = g[i];
        g[i] = gi * sg;
        gd[i] = gd[i] * sg + gi * sg * (1.0f - sg) * pred[i];
    }
};
struct SEdgeProdTanK {  // out = ga[t] y[c] rcut;  outd = (gad[t] y[c] + ga[t] yd[c]) rcut + ga[t] y[c] rcd
    const int32_t* tgt; const int32_t* col; const float* ga; const float* gad; const float* y; const float* yd; const float* rcut; const float* rcd;
    float* out; float* outd;
    GD void operator()(int64_t i) const {
        const int64_t e = i / F; const int f = (int)(i % F);
        const int64_t t = (int64_t)tgt[e] * F + f, c = (int64_t)col[e] * F + f;
        const float a = ga[t], yy = y[c];
        out[i] = a * yy * rcut[e];
        outd[i] = (gad[t] * yy + a * yd[c]) * rcut[e] + a * yy * rcd[e];
    }
};

struct Work {
    int32_t *mol_id, *col, *tgt;
    float *d, *rcut, *phi;
    float *x;                     // [L+1][N, F]   atom features entering each layer (x[L] = final)
    float *h1pre, *Wf;            // [L][E, F]
    float *y, *agg, *tpre;        // [L][N, F]
    float *rpre, *r, *e_atom;     // [N, H], [N, H], [N]
    float *tE, *gE;               // [E, F] temporaries
    float *tN, *gx, *gy, *gN;     // [N, F] temporaries
    float *g_rpre, *g_e;          // [N, H], [N]
    // tangent pass (force losses only)
    float *dd, *rcd, *phid;       // [E], [E], [E, K]
    float *xd, *h1pred, *Wfd;     // [L+1][N, F], [L][E, F], [L][E, F]
    float *yd, *aggd, *tpred;     // [L][N, F]
    float *rpred, *rd, *gd_rpre;  // [N, H]
    float *tEd, *gEd, *uE;        // [E, F]
    float *tNd, *gxd, *gyd, *gNd, *uN;  // [N, F]
    int64_t bytes;
};
Work carve(void* p, int64_t L, int64_t K, int64_t n, int64_t E, bool tangent) {
    Carve c(p);
    Work w;
    w.mol_id = c.take<int32_t>(n);
    w.col = c.take<int32_t>(E);
    w.tgt = c.take<int32_t>(E);
    w.d = c.take<float>(E);
    w.rcut = c.take<float>(E);
    w.phi = c.take<float>(E * K);
    w.x = c.take<float>((L + 1) * n * F);
    w.h1pre = c.take<float>(L * E * F);
    w.Wf = c.take<float>(L * E * F);
    w.y = c.take<float>(L * n * F);
    w.agg = c.take<float>(L * n * F);
    w.tpre = c.take<float>(L * n * F);
    w.rpre = c.take<float>(n * H);
    w.r = c.take<float>(n * H);
    w.e_atom = c.take<float>(n);
    w.tE = c.take<float>(E * F);
    w.gE = c.take<float>(E * F);
    w.tN = c.take<float>(n * F);
    w.gx = c.take<float>(n * F);
    w.gy = c.take<float>(n * F);
    w.gN = c.take<float>(n * F);
    w.g_rpre = c.take<float>(n * H);
    w.g_e = c.take<float>(n);
    if (tangent) {
        w.dd = c.take<float>(E); w.rcd = c.take<float>(E); w.phid = c.take<float>(E * K);
        w.xd = c.take<float>((L + 1) * n * F); w.h1pred = c.take<float>(L * E * F); w.Wfd = c.take<float>(L * E * F);
        w.yd = c.take<float>(L * n * F); w.aggd = c.take<float>(L * n * F); w.tpred = c.take<float>(L * n * F);
        w.rpred = c.take<float>(n * H); w.rd = c.take<float>(n * H); w.gd_rpre = c.take<float>(n * H);
        w.tEd = c.take<float>(E * F); w.gEd = c.take<float>(E * F); w.uE = c.take<float>(E * F);
        w.tNd = c.take<float>(n * F); w.gxd = c.take<float>(n * F); w.gyd = c.take<float>(n * F); w.gNd = c.take<float>(n * F); w.uN = c.take<float>(n * F);
    }
    w.bytes = c.off + 256;
    return w;
}
bool config_ok(const nb200_schnet_weights* w) {
    return w && w->n_feat == F && w->n_layers >= 1 && w->n_layers <= 32 && w->n_rbf >= 1 && w->n_rbf <= 512 && w->n_elem >= 1 && w->cutoff > 0.0f &&
           w->rbf_offsets && w->emb && w->w_f1 && w->b_f1 && w->W_f2 && w->b_f2 && w->I1 && w->P1 && w->p1 && w->P2 && w->p2 && w->R1 && w->e1 && w->R2 && w->e2;
}
inline int64_t chunks(int64_t M) { return (M + WG_ROWS - 1) / WG_ROWS; }

struct Run {
    nb200_engine* e; cudaStream_t s;
    // dense layers: the wgmma 3xTF32 GEMM of gemm_tc.cu on the device (shapes of the classes its unit tests cover: N, K in {64, 128},
    // bias epilogue, trans_b, accumulate), the functor fallback under host emulation or NB200_GOC_GEMM=simt
    int lin(int64_t M, int N, int K, const float* A, const float* W, const float* bias, float* C, bool acc = false) const {
        if (M <= 0) return NB200_OK;
        if (M <= 0x7fffffff && goc_tc_ok(N, K, K, K, N)) return goc_tc_gemm_ex(e, s, (int)M, N, K, A, K, W, K, 0, C, N, acc ? 1 : 0, bias);
        return pfor(e, s, CAT_GEMM, M * N, SLinK{A, K, W, bias, C, N, acc ? 1 : 0});
    }
    // C[M, K] (+)= G[M, N] W[N, K]
    int lin_bwd(int64_t M, int N, int K, const float* G, const float* W, float* C, bool acc = false) const {
        if (M <= 0) return NB200_OK;
        if (M <= 0x7fffffff && goc_tc_ok(K, N, N, K, K)) return goc_tc_gemm_ex(e, s, (int)M, K, N, G, N, W, K, 1, C, K, acc ? 1 : 0, nullptr);
        return pfor(e, s, CAT_GEMM, M * K, SLinBwdK{G, N, W, C, K, acc ? 1 : 0});
    }
    // dW[N, K] += G[M, N]^T X[M, K];  db[N] += colsum(G)
    int wgrad(int64_t M, int N, int K, const float* G, const float* X, float* dW, float* db, float alpha = 1.0f) const {
        if (M <= 0) return NB200_OK;
        if (dW) {
            int rc = NB200_OK;
            if (goc_wgrad(e, s, M, N, K, G, N, X, K, dW, K, alpha, &rc)) NB_TRY(rc);  // cuBLAS on the device
            else NB_TRY(pfor(e, s, CAT_GEMM, chunks(M) * N * K, SWgradK{G, N, X, K, M, dW, alpha}));
        }
        if (db) NB_TRY(pfor(e, s, CAT_NODE, chunks(M) * N, SColsumK{G, N, M, db, alpha}));
        return NB200_OK;
    }
};

}  // namespace

/* Phase 1: degrees and CSR row pointers of the neighbour list; synchronises once to return the edge count. */
extern "C" int nb200_schnet_train_count(const nb200_schnet_weights* w, const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                                        int32_t* row_ptr, int32_t* scratch, int64_t* n_edges_host, void* stream) {
    if (!w || !(w->cutoff > 0.0f) || !pos || !mol_ptr || !row_ptr || !scratch || !n_edges_host || n_mol < 1 || n_atoms < 1) return NB200_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    nb200_engine* e = nullptr;
#ifndef NB_EMU
    nb200_engine tmp_engine{};
    e = &tmp_engine;
#endif
    int32_t* mol_id = scratch;            // scratch: [2 N] int32
    int32_t* deg = scratch + n_atoms;
    NB_TRY(pfor(e, s, CAT_NBR, n_atoms, SMolIdK{mol_ptr, n_mol, mol_id}));
    NB_TRY(pfor(e, s, CAT_NBR, n_atoms, SDegK{pos, mol_ptr, mol_id, w->cutoff * w->cutoff, deg}));
    NB_TRY(scan_excl(e, s, deg, n_atoms, row_ptr));
    int32_t tot = 0;
    NB_TRY(goc_d2h_sync(&tot, row_ptr + n_atoms, sizeof(int32_t), s));
    if (tot < 0) return NB200_ECAPACITY;
    *n_edges_host = tot;
    return NB200_OK;
}

extern "C" int64_t nb200_schnet_train_workspace_bytes(const nb200_schnet_weights* w, int32_t n_mol, int32_t n_atoms, int64_t n_edges, int32_t with_force_seed) {
    if (!w || w->n_feat != F || w->n_layers < 1 || w->n_rbf < 1 || n_mol < 1 || n_atoms < 1 || n_edges < 0) return NB200_EINVAL;
    return carve(nullptr, w->n_layers, w->n_rbf, n_atoms, n_edges, with_force_seed != 0).bytes;
}

/* Phase 2: energy[B] (training semantics: the caller decides about the AddOffsets shift through w->energy_shift_per_atom) and, when a seed is
 * given, grads = d( sum_m energy_seed[m] E_m + sum_i force_seed[i] . F_i ) / d(weights), F = -dE_tot/dR, written into the buffers `grads`
 * points to (same struct, same shapes; every buffer is zeroed first; rbf_offsets is ignored).  Either seed may be NULL. */
extern "C" int nb200_schnet_energy_grads(nb200_engine* eng, const nb200_schnet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                         int32_t n_mol, int32_t n_atoms, const int32_t* row_ptr, int64_t n_edges, void* workspace, int64_t workspace_bytes,
                                         const float* energy_seed, const float* force_seed, const nb200_schnet_weights* grads, float* energy, void* stream) {
    if (!eng || !config_ok(w) || !z || !pos || !mol_ptr || !row_ptr || !workspace || !energy || n_mol < 1 || n_atoms < 1 || n_edges < 0) return NB200_EINVAL;
    if ((energy_seed || force_seed) && !config_ok(grads)) return NB200_EINVAL;
    const bool tan = force_seed != nullptr;
    const int L = w->n_layers, K = w->n_rbf;
    const int64_t n = n_atoms, E = n_edges;
    if (workspace_bytes < carve(nullptr, L, K, n, E, tan).bytes) return NB200_EINVAL;  // before any pointer is formed
    const Work wk = carve(workspace, L, K, n, E, tan);
    cudaStream_t s = (cudaStream_t)stream;
    const Run R{eng, s};
    const int64_t NF = n * F, EF = E * F, FF = (int64_t)F * F;
    // ---- forward with saved activations (and, for a force seed, the tangents of every activation along v = force_seed)
    NB_TRY(pfor(eng, s, CAT_NBR, n, SMolIdK{mol_ptr, n_mol, wk.mol_id}));
    NB_TRY(pfor(eng, s, CAT_NBR, n, SFillK{pos, mol_ptr, wk.mol_id, row_ptr, w->cutoff * w->cutoff, w->cutoff, wk.col, wk.tgt, wk.d, wk.rcut}));
    NB_TRY(pfor(eng, s, CAT_FILTER, E * K, SPhiK{wk.d, w->rbf_offsets, w->rbf_coeff, K, wk.phi}));
    NB_TRY(pfor(eng, s, CAT_EMBED, NF, SEmbedK{z, w->emb, w->n_elem, w->z_offset, wk.x}));
    if (tan) {
        NB_TRY(pfor(eng, s, CAT_NBR, E, STanGeomK{pos, force_seed, wk.col, wk.tgt, wk.d, w->cutoff, wk.dd, wk.rcd}));
        NB_TRY(pfor(eng, s, CAT_FILTER, E * K, SPhiTanK{wk.d, wk.dd, w->rbf_offsets, w->rbf_coeff, K, wk.phi, wk.phid}));
        NB_TRY(goc_memset(wk.xd, 0, (size_t)NF * sizeof(float), s));  // the embedding does not depend on the positions
    }
    for (int l = 0; l < L; l++) {
        float *x = wk.x + l * NF, *xn = wk.x + (l + 1) * NF, *h1pre = wk.h1pre + l * EF, *Wf = wk.Wf + l * EF, *y = wk.y + l * NF, *agg = wk.agg + l * NF,
              *tpre = wk.tpre + l * NF;
        const float *W1 = w->w_f1 + (int64_t)l * K * F, *b1 = w->b_f1 + l * F;
        NB_TRY(pfor(eng, s, CAT_FILTER, EF, SLinKmajorK{wk.phi, K, W1, b1, h1pre, F}));
        NB_TRY(pfor(eng, s, CAT_FILTER, EF, SSspK{h1pre, wk.tE}));
        NB_TRY(R.lin(E, F, F, wk.tE, w->W_f2 + l * FF, w->b_f2 + l * F, Wf));                         // filter before the cutoff
        if (tan) {
            float *h1pred = wk.h1pred + l * EF, *Wfd = wk.Wfd + l * EF;
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SLinKmajorK{wk.phid, K, W1, nullptr, h1pred, F}));
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SMulSigOutK{h1pred, h1pre, wk.tEd}));                  // h1d
            NB_TRY(R.lin(E, F, F, wk.tEd, w->W_f2 + l * FF, nullptr, Wfd));
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SFilterTanK{Wf, Wfd, wk.rcut, wk.rcd}));
        } else {
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SRowScaleK{Wf, wk.rcut}));
        }
        NB_TRY(R.lin(n, F, F, x, w->I1 + l * FF, nullptr, y));
        NB_TRY(pfor(eng, s, CAT_MSG_FWD, NF, SCfconvK{row_ptr, wk.col, y, Wf, agg}));
        NB_TRY(R.lin(n, F, F, agg, w->P1 + l * FF, w->p1 + l * F, tpre));
        NB_TRY(pfor(eng, s, CAT_NODE, NF, SSspK{tpre, wk.tN}));
        NB_TRY(R.lin(n, F, F, wk.tN, w->P2 + l * FF, w->p2 + l * F, xn));
        NB_TRY(pfor(eng, s, CAT_NODE, NF, SAddK{xn, x}));
        if (tan) {
            float *xd = wk.xd + l * NF, *xdn = wk.xd + (l + 1) * NF, *yd = wk.yd + l * NF, *aggd = wk.aggd + l * NF, *tpred = wk.tpred + l * NF;
            NB_TRY(R.lin(n, F, F, xd, w->I1 + l * FF, nullptr, yd));
            NB_TRY(pfor(eng, s, CAT_MSG_FWD, NF, SCfconv2K{row_ptr, wk.col, yd, Wf, y, wk.Wfd + l * EF, aggd}));
            NB_TRY(R.lin(n, F, F, aggd, w->P1 + l * FF, nullptr, tpred));
            NB_TRY(pfor(eng, s, CAT_NODE, NF, SMulSigOutK{tpred, tpre, wk.tNd}));                      // td
            NB_TRY(R.lin(n, F, F, wk.tNd, w->P2 + l * FF, nullptr, xdn));
            NB_TRY(pfor(eng, s, CAT_NODE, NF, SAddK{xdn, xd}));
        }
    }
    const float* xL = wk.x + (int64_t)L * NF;
    NB_TRY(R.lin(n, H, F, xL, w->R1, w->e1, wk.rpre));
    NB_TRY(pfor(eng, s, CAT_READOUT, n, SReadoutK{wk.rpre, w->R2, w->e2, w->energy_shift_per_atom, wk.e_atom}));
    NB_TRY(pfor(eng, s, CAT_READOUT, n_mol, SMolSumK{mol_ptr, wk.e_atom, energy}));
    if (!energy_seed && !force_seed) return NB200_OK;
    const nb200_schnet_weights* g = grads;
    float* const gbuf[] = {(float*)g->emb, (float*)g->w_f1, (float*)g->b_f1, (float*)g->W_f2, (float*)g->b_f2, (float*)g->I1, (float*)g->P1, (float*)g->p1,
                           (float*)g->P2, (float*)g->p2, (float*)g->R1, (float*)g->e1, (float*)g->R2, (float*)g->e2};
    const int64_t gsize[] = {(int64_t)w->n_elem * F, (int64_t)L * K * F, (int64_t)L * F, L * FF, (int64_t)L * F, L * FF, L * FF, (int64_t)L * F,
                             L * FF, (int64_t)L * F, (int64_t)H * F, H, H, 1};
    for (int k = 0; k < 14; k++) NB_TRY(goc_memset(gbuf[k], 0, (size_t)gsize[k] * sizeof(float), s));
    // ---- reverse sweep for the energy term: seed c_m
    if (energy_seed) {
        NB_TRY(pfor(eng, s, CAT_READOUT, n * H, SSeedK{wk.mol_id, energy_seed, wk.rpre, w->R2, wk.r, wk.g_rpre, wk.g_e}));
        NB_TRY(R.wgrad(n, 1, H, wk.g_e, wk.r, (float*)g->R2, (float*)g->e2));           // dR2[1, H] = g_e^T r ; de2 = sum g_e
        NB_TRY(R.wgrad(n, H, F, wk.g_rpre, xL, (float*)g->R1, (float*)g->e1));
        NB_TRY(R.lin_bwd(n, H, F, wk.g_rpre, w->R1, wk.gx));                             // g_x = g_rpre R1
        for (int l = L - 1; l >= 0; l--) {
            const float *x = wk.x + l * NF, *h1pre = wk.h1pre + l * EF, *Wf = wk.Wf + l * EF, *y = wk.y + l * NF, *agg = wk.agg + l * NF, *tpre = wk.tpre + l * NF;
            // x_{l+1} = x_l + P2 ssp(P1 agg + p1) + p2 : g_v = g_x
            NB_TRY(pfor(eng, s, CAT_NODE, NF, SSspK{tpre, wk.tN}));
            NB_TRY(R.wgrad(n, F, F, wk.gx, wk.tN, (float*)g->P2 + l * FF, (float*)g->p2 + l * F));
            NB_TRY(R.lin_bwd(n, F, F, wk.gx, w->P2 + l * FF, wk.gN));                    // g_t
            NB_TRY(pfor(eng, s, CAT_NODE, NF, SMulSigK{wk.gN, tpre}));                   // g_tpre
            NB_TRY(R.wgrad(n, F, F, wk.gN, agg, (float*)g->P1 + l * FF, (float*)g->p1 + l * F));
            NB_TRY(R.lin_bwd(n, F, F, wk.gN, w->P1 + l * FF, wk.tN));                    // g_agg (tN reused)
            // cfconv: agg_i = sum_j y_j * Wf_ij
            NB_TRY(pfor(eng, s, CAT_MSG_BWD, NF, SCfconvK{row_ptr, wk.col, wk.tN, Wf, wk.gy}));              // g_y (symmetric list, Wf_ij = Wf_ji)
            NB_TRY(pfor(eng, s, CAT_MSG_BWD, EF, SEdgeProdK{wk.tgt, wk.col, wk.tN, y, wk.rcut, wk.gE}));     // grad of (W_f2 h1 + b_f2)
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SSspK{h1pre, wk.tE}));                                       // h1
            NB_TRY(R.wgrad(E, F, F, wk.gE, wk.tE, (float*)g->W_f2 + l * FF, (float*)g->b_f2 + l * F));
            NB_TRY(R.lin_bwd(E, F, F, wk.gE, w->W_f2 + l * FF, wk.tE));                  // g_h1 (tE reused)
            NB_TRY(pfor(eng, s, CAT_FILTER, EF, SMulSigK{wk.tE, h1pre}));                // g_h1pre
            // K-major layout: dw_f1[k, f] = sum_e phi[e, k] g_h1pre[e, f]  ->  "G" = phi [E, K], "X" = g_h1pre [E, F]
            NB_TRY(R.wgrad(E, K, F, wk.phi, wk.tE, (float*)g->w_f1 + (int64_t)l * K * F, nullptr));
            NB_TRY(R.wgrad(E, F, 0, wk.tE, nullptr, nullptr, (float*)g->b_f1 + l * F));  // bias only
            // y = I1 x
            NB_TRY(R.wgrad(n, F, F, wk.gy, x, (float*)g->I1 + l * FF, nullptr));
            NB_TRY(R.lin_bwd(n, F, F, wk.gy, w->I1 + l * FF, wk.gx, true));              // g_x += g_y I1   (residual: g_x already holds g_{x_{l+1}})
        }
        NB_TRY(pfor(eng, s, CAT_EMBED, (int64_t)w->n_elem * F, SEmbGradK{z, w->z_offset, w->n_elem, wk.gx, n_atoms, (float*)g->emb, 1.0f}));
    }
    if (!tan) return NB200_OK;
    // ---- reverse sweep with unit seeds carrying tangents: every weight gradient G^T X gets  -(Gd^T X + G^T Xd)  added
    const float A = -1.0f;
    NB_TRY(R.lin(n, H, F, wk.xd + (int64_t)L * NF, w->R1, nullptr, wk.rpred));
    NB_TRY(pfor(eng, s, CAT_READOUT, n * H, SSeedTanK{wk.rpre, wk.rpred, w->R2, wk.r, wk.rd, wk.g_rpre, wk.gd_rpre, wk.g_e}));
    NB_TRY(R.wgrad(n, 1, H, wk.g_e, wk.rd, (float*)g->R2, nullptr, A));                                   // g_e = 1 has no tangent; e2: none
    NB_TRY(R.wgrad(n, H, F, wk.gd_rpre, xL, (float*)g->R1, (float*)g->e1, A));
    NB_TRY(R.wgrad(n, H, F, wk.g_rpre, wk.xd + (int64_t)L * NF, (float*)g->R1, nullptr, A));
    NB_TRY(R.lin_bwd(n, H, F, wk.g_rpre, w->R1, wk.gx));
    NB_TRY(R.lin_bwd(n, H, F, wk.gd_rpre, w->R1, wk.gxd));
    for (int l = L - 1; l >= 0; l--) {
        const float *x = wk.x + l * NF, *xd = wk.xd + l * NF, *h1pre = wk.h1pre + l * EF, *h1pred = wk.h1pred + l * EF, *Wf = wk.Wf + l * EF,
                    *Wfd = wk.Wfd + l * EF, *y = wk.y + l * NF, *yd = wk.yd + l * NF, *agg = wk.agg + l * NF, *aggd = wk.aggd + l * NF,
                    *tpre = wk.tpre + l * NF, *tpred = wk.tpred + l * NF;
        float *dP2 = (float*)g->P2 + l * FF, *dP1 = (float*)g->P1 + l * FF, *dW2 = (float*)g->W_f2 + l * FF, *dI1 = (float*)g->I1 + l * FF,
              *dW1 = (float*)g->w_f1 + (int64_t)l * K * F;
        // f2out.1: v = P2 t + p2
        NB_TRY(pfor(eng, s, CAT_NODE, NF, SSspK{tpre, wk.tN}));                                            // t
        NB_TRY(pfor(eng, s, CAT_NODE, NF, SMulSigOutK{tpred, tpre, wk.tNd}));                              // td
        NB_TRY(R.wgrad(n, F, F, wk.gxd, wk.tN, dP2, (float*)g->p2 + l * F, A));
        NB_TRY(R.wgrad(n, F, F, wk.gx, wk.tNd, dP2, nullptr, A));
        NB_TRY(R.lin_bwd(n, F, F, wk.gx, w->P2 + l * FF, wk.gN));                                          // g_t
        NB_TRY(R.lin_bwd(n, F, F, wk.gxd, w->P2 + l * FF, wk.gNd));                                        // gd_t
        NB_TRY(pfor(eng, s, CAT_NODE, NF, SMulSigTanK{wk.gN, wk.gNd, tpre, tpred}));                       // g_tpre, gd_tpre
        // f2out.0: tpre = P1 agg + p1
        NB_TRY(R.wgrad(n, F, F, wk.gNd, agg, dP1, (float*)g->p1 + l * F, A));
        NB_TRY(R.wgrad(n, F, F, wk.gN, aggd, dP1, nullptr, A));
        NB_TRY(R.lin_bwd(n, F, F, wk.gN, w->P1 + l * FF, wk.tN));                                          // g_agg
        NB_TRY(R.lin_bwd(n, F, F, wk.gNd, w->P1 + l * FF, wk.tNd));                                        // gd_agg
        // cfconv
        NB_TRY(pfor(eng, s, CAT_MSG_BWD, NF, SCfconvK{row_ptr, wk.col, wk.tN, Wf, wk.gy}));                                  // g_y
        NB_TRY(pfor(eng, s, CAT_MSG_BWD, NF, SCfconv2K{row_ptr, wk.col, wk.tNd, Wf, wk.tN, Wfd, wk.gyd}));                  // gd_y
        NB_TRY(pfor(eng, s, CAT_MSG_BWD, EF, SEdgeProdTanK{wk.tgt, wk.col, wk.tN, wk.tNd, y, yd, wk.rcut, wk.rcd, wk.gE, wk.gEd}));
        // filter_network.1: fpre = W_f2 h1 + b_f2
        NB_TRY(pfor(eng, s, CAT_FILTER, EF, SSspK{h1pre, wk.tE}));                                         // h1
        NB_TRY(pfor(eng, s, CAT_FILTER, EF, SMulSigOutK{h1pred, h1pre, wk.tEd}));                          // h1d
        NB_TRY(R.wgrad(E, F, F, wk.gEd, wk.tE, dW2, (float*)g->b_f2 + l * F, A));
        NB_TRY(R.wgrad(E, F, F, wk.gE, wk.tEd, dW2, nullptr, A));
        NB_TRY(R.lin_bwd(E, F, F, wk.gE, w->W_f2 + l * FF, wk.tE));                                        // g_h1
        NB_TRY(R.lin_bwd(E, F, F, wk.gEd, w->W_f2 + l * FF, wk.tEd));                                      // gd_h1
        NB_TRY(pfor(eng, s, CAT_FILTER, EF, SMulSigTanK{wk.tE, wk.tEd, h1pre, h1pred}));                   // g_h1pre, gd_h1pre
        // filter_network.0 (K-major): dw_f1[k, f] = sum_e phi[e, k] g_h1pre[e, f]
        NB_TRY(R.wgrad(E, K, F, wk.phid, wk.tE, dW1, nullptr, A));
        NB_TRY(R.wgrad(E, K, F, wk.phi, wk.tEd, dW1, nullptr, A));
        NB_TRY(R.wgrad(E, F, 0, wk.tEd, nullptr, nullptr, (float*)g->b_f1 + l * F, A));
        // in2f: y = I1 x
        NB_TRY(R.wgrad(n, F, F, wk.gyd, x, dI1, nullptr, A));
        NB_TRY(R.wgrad(n, F, F, wk.gy, xd, dI1, nullptr, A));
        NB_TRY(R.lin_bwd(n, F, F, wk.gy, w->I1 + l * FF, wk.gx, true));
        NB_TRY(R.lin_bwd(n, F, F, wk.gyd, w->I1 + l * FF, wk.gxd, true));
    }
    return pfor(eng, s, CAT_EMBED, (int64_t)w->n_elem * F, SEmbGradK{z, w->z_offset, w->n_elem, wk.gxd, n_atoms, (float*)g->emb, A});
}

#include "schnet_hvp.inc"
