/*
 * nabla_b200.h -- C ABI of the H100-native nablaDFT model-forward hot path.
 *
 * The reference (AIRI-Institute/nablaDFT) is pure Python; its "plugin seam" for this path
 * is `torch.nn.Module.forward(batch)` reached through Hydra `_target_` strings
 * (SURVEY.md section 8b).  This header is the FFI a maintainer binds behind those modules
 * (ctypes stub in INTEGRATION.md).  Every entry point cites the reference code it replaces.
 *
 * Conventions
 *   - plain pointers + sizes; no torch types.  All pointers are DEVICE pointers unless the
 *     parameter name ends in `_host`.  fp32 data, int32 indices, row-major, 16-byte aligned.
 *   - caller owns every buffer (callee never allocates or frees device memory, except the
 *     cuBLAS handle owned by an engine object).
 *   - `stream` is a `cudaStream_t` passed as `void*`; every call is asynchronous on it.
 *   - return value: 0 on success, negative `NB200_E*` on error; no exceptions cross the ABI.
 *   - re-entrant; no global state; one engine object per host thread / stream.
 *   - hidden size F is 128 (every SchNet/PaiNN config of the reference:
 *     config/model/{schnet,painn,painn-oc}.yaml); other sizes return NB200_EUNSUPPORTED.
 *
 * Molecule batch ("conformations") layout in HBM
 *   z[N] int32, pos[N,3] f32, mol_ptr[B+1] int32 (atoms of molecule m are rows
 *   mol_ptr[m]..mol_ptr[m+1]).  Neighbour list = CSR by TARGET atom:
 *   row_ptr[N+1], col[E] (source atom, ascending inside a row), rev[E] (index of the
 *   opposite edge), geom[E,4] = (ux,uy,uz,d) with u = (pos[col]-pos[target])/d.
 */
#ifndef NABLA_B200_H
#define NABLA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB200_OK 0
#define NB200_EINVAL -1        /* bad argument (null pointer, negative size, ...)          */
#define NB200_EUNSUPPORTED -2  /* configuration outside the compiled fast path             */
#define NB200_ECUDA -3         /* CUDA launch / runtime error (see nb200_last_cuda_error)   */
#define NB200_ECAPACITY -4     /* edge capacity exceeded (reported by *_status)            */
#define NB200_ENEIGHBORS -5    /* an atom has more than max_neighbors neighbours            */
#define NB200_ENOEDGES -6      /* a molecule has an atom without neighbours                 */

#define NB200_RADIAL_SPK 0 /* schnetpack GaussianRBF + CosineCutoff on the whole filter    */
#define NB200_RADIAL_OC 1  /* GaussianSmearing(d/rc) * PolynomialEnvelope(p=5); bias unmasked */

int nb200_version(void);
int nb200_last_cuda_error(void); /* cudaError_t of the most recent failing call in this thread */

/* ----------------------------------------------------------------------------------------
 * Neighbour build on device.
 * Replaces torch_cluster.radius_graph + distance/unit-vector code
 *   (nablaDFT/painn_pyg/painn.py:411-423, 306-321; qhnet/qhnet.py:258-262) and, for the
 *   schnetpack models, ASENeighborList + PairwiseDistances
 *   (config/datamodule/nablaDFT_ase.yaml:13-14, config/model/painn.yaml:17-18).
 * Semantics: same-molecule pairs with |r|^2 < cutoff^2 (strict), no self loops.
 * `status[4]` (device int32) receives {n_edges, error_code, max_degree, n_isolated_atoms};
 * error_code is NB200_ECAPACITY if n_edges > e_cap (nothing is written past e_cap) or
 * NB200_ENEIGHBORS if a degree exceeds max_neighbors (the reference would truncate to the
 * first K sources, which breaks edge symmetry; no shipped config reaches it).
 * `deg_scratch[N]` is scratch.
 * -------------------------------------------------------------------------------------- */
int nb200_neighbor_build(const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                         float cutoff, int32_t max_neighbors, int32_t e_cap,
                         int32_t* row_ptr, int32_t* col, int32_t* rev, float* geom,
                         int32_t* deg_scratch, int32_t* status, void* stream);

/* ----------------------------------------------------------------------------------------
 * Radial filter generation  W[l][e][3F] (and dW/dd) for all L layers from edge distances.
 * Replaces  spk: GaussianRBF -> filter_net Dense(100 -> L*3F) * CosineCutoff
 *                (config/model/painn.yaml:10-16; SURVEY.md A.2)
 *           OC : RadialBasis (layers.py:129-185) -> rbf_proj Linear(100 -> 3F) per layer
 *                (painn_pyg/painn.py:464,479)
 * Gaussians have width == spacing (both libraries), so only a 16-wide band of the K centres
 * contributes above 2.3e-11; the kernel evaluates that band (edges are grouped by distance
 * bin so the band weights stay in registers).
 *   w_rbf  [L][K][3F]  (K-major transpose of the Linear weight), b_rbf [L][3F]
 *   W, dW  [L][E][3F]  (dW may be NULL: energy-only)
 *   rbf_offsets[K], rbf_coeff, rbf_xscale: phi_k = exp(rbf_coeff * (d*rbf_xscale - offsets[k])^2)
 *                 (spk: xscale 1, offsets = linspace(0,rc,K); OC: xscale 1/rc, linspace(0,1,K))
 *   sort_scratch: int32[ e_stride + 1024 ] scratch for the distance-bin grouping
 * n_edges is read from status[0] on the device (no host sync); e_stride = row stride count
 * of W per layer (>= n_edges, normally e_cap).
 * -------------------------------------------------------------------------------------- */
int nb200_painn_filter(const float* geom, const int32_t* status, int32_t e_stride,
                       const float* w_rbf, const float* b_rbf, int32_t n_layers, int32_t n_rbf,
                       int32_t n_feat, int32_t radial_mode, float cutoff,
                       const float* rbf_offsets, float rbf_coeff, float rbf_xscale,
                       float* W, float* dW, int32_t* sort_scratch, void* stream);

/* ----------------------------------------------------------------------------------------
 * PaiNN message + segmented scatter (forward):  q_out = q + dq, mu_out = mu + dmu
 *   dq_i  = sum_e Wa_e * a_j ;  dmu_i = sum_e (Wb_e*b_j) u_e + (Wc_e*c_j) * mu_j
 *   with (a,b,c) = split(xh[j] + xh_bias) and (Wa,Wb,Wc) = split(W_e)  [canonical spk roles]
 * Replaces PaiNNInteraction.forward (schnetpack 2.0.4; SURVEY.md A.2) and
 *   PaiNNMessage.message/aggregate (nablaDFT/painn_pyg/painn.py:493-509; chunks 2,3 swapped
 *   by the host when exporting weights).
 * Warp per target atom, register accumulation in CSR order: deterministic, no atomics.
 * -------------------------------------------------------------------------------------- */
int nb200_painn_msg_fwd(const float* xh, const float* xh_bias, const float* q, const float* mu,
                        const float* W, const float* geom, const int32_t* row_ptr,
                        const int32_t* col, int32_t n_atoms, float* q_out, float* mu_out,
                        void* stream);

/* Backward of the above w.r.t. xh, mu and the edge geometry (for forces = -dE/dR,
 * nablaDFT/painn_pyg/painn.py:135-146).  Uses edge symmetry (W_e == W_rev(e)).
 *   g_q, g_mu   : dE/d(q_out), dE/d(mu_out)                      [N,F], [N,3,F]
 *   g_xh        : out, dE/d(xh)                                   [N,3F]
 *   g_mu_in     : out, dE/d(mu) = g_mu + sum(...)  (must not alias g_mu)
 *   egrad[E,4]  : +=  (dE/du_x, dE/du_y, dE/du_z, dE/dd) of edge rev(e), accumulated over layers
 */
int nb200_painn_msg_bwd(const float* xh, const float* xh_bias, const float* mu,
                        const float* W, const float* dW, const float* geom,
                        const int32_t* row_ptr, const int32_t* col, int32_t n_atoms,
                        const float* g_q, const float* g_mu,
                        float* g_xh, float* g_mu_in, float* egrad, void* stream);

/* Test and benchmark entry points, not a supported API: they may change with the kernels they expose.
 * Every instantiation of the two kernels above.  `w_stride` 3F: rows of W (and dW) of 3F;
 * 6F: one [W | dW/dd] record per row (dW unused).  `rev` non-NULL: edge e reads row min(e, rev[e]), one row per
 * undirected pair; NULL: row e.  `bf16` != 0: W, dW (and gW) hold bf16.  Backward with `gW` non-NULL (w_stride 3F
 * only): also gW[e][3F] = seed_atom[j] * dE/dW of the opposite edge, for the filter's weight gradients. */
int nb200_painn_msg_fwd_ex(const float* xh, const float* xh_bias, const float* q, const float* mu,
                           const void* W, int32_t w_stride, const int32_t* rev, const float* geom,
                           const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, float* q_out,
                           float* mu_out, int32_t bf16, void* stream);
int nb200_painn_msg_bwd_ex(const float* xh, const float* xh_bias, const float* mu, const void* W,
                           const void* dW, int32_t w_stride, const int32_t* rev, const float* geom,
                           const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, const float* g_q,
                           const float* g_mu, float* g_xh, float* g_mu_in, float* egrad, void* gW,
                           const float* seed_atom, int32_t bf16, void* stream);
/* Gather-bandwidth probe (test and benchmark entry point): the per-edge L2 reads of the message kernels without
 * their arithmetic.  bwd_pattern 0: A = xh [N,3F], B = mu [N,3F], first 3F of record row min(e, rev[e]);
 * 1: A = g_q [N,F], B = g_mu [N,3F], whole 6F record.  out[N*32] receives sums that keep the loads alive. */
int nb200_msg_gather_probe(const float* A, const float* B, const float* rec, int32_t rec_stride,
                           const int32_t* rev, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms,
                           int32_t bwd_pattern, float* out, void* stream);

/* Forces from accumulated edge gradients:  F_j = -sum_{e in row j} (G(e) - G(rev e)). */
int nb200_edge_forces(const float* egrad, const float* geom, const int32_t* row_ptr,
                      const int32_t* rev, int32_t n_atoms, float* forces, void* stream);

/* ----------------------------------------------------------------------------------------
 * Whole-model engine: PaiNN energy + forces for one batch of conformations.
 * Replaces `NeuralNetworkPotential.forward` for config/model/painn.yaml (spk roles) and
 * `PaiNN.forward` (nablaDFT/painn_pyg/painn.py:89-148) for config/model/painn-oc.yaml.
 * The node forward runs as fused per-layer wgmma kernels; the other node-level dense layers run on the wgmma 3xTF32 GEMM
 * (fp32-accurate).
 * -------------------------------------------------------------------------------------- */
typedef struct nb200_painn_weights {
    int32_t n_layers, n_feat, n_rbf, n_elem; /* L, F(=128), K(=100), rows of emb            */
    int32_t radial_mode, z_offset;           /* NB200_RADIAL_*, 0 (spk) or 1 (OC: emb[z-1]) */
    float cutoff, epsilon;                   /* 5.0, 1e-8                                   */
    float rbf_coeff, rbf_xscale;             /* phi_k = exp(coeff (d*xscale - offsets[k])^2) */
    const float* rbf_offsets;                /* [K] Gaussian centres (module buffer); must be k dx, dx = cutoff xscale / (K - 1):
                                              * the filter evaluates only the 16 centres around bin floor(d xscale / dx) */
    float energy_shift_per_atom;             /* spk AddOffsets mean (eval); 0 otherwise     */
    int32_t max_neighbors;                   /* OC: 100; spk: INT32_MAX                     */
    const float* emb;                        /* [n_elem][F]                                 */
    const float* w_rbf;                      /* [L][K][3F]                                  */
    const float* b_rbf;                      /* [L][3F]                                     */
    const float* A1; const float* c1;        /* [L][F][F],  [L][F]     message MLP in       */
    const float* A2; const float* c2;        /* [L][3F][F], [L][3F]    message MLP out      */
    const float* U;                          /* [L][2F][F]             vector channel mix   */
    const float* B1; const float* d1;        /* [L][F][2F], [L][F]     update MLP in        */
    const float* B2; const float* d2;        /* [L][3F][F], [L][3F]    update MLP out       */
    const float* R1; const float* e1;        /* [F/2][F], [F/2]        readout              */
    const float* R2; const float* e2;        /* [1][F/2], [1]                                */
} nb200_painn_weights;

typedef struct nb200_engine nb200_engine;

int nb200_engine_create(nb200_engine** out);
int nb200_engine_destroy(nb200_engine* eng);
/* Optional per-category CUDA-event timing of the engine's launches (bench.py roofline leg).
 * Categories: 0 neighbour build, 1 radial filters, 2 embedding, 3 node GEMMs, 4 node
 * elementwise, 5 message fwd, 6 message bwd, 7 readout, 8 force assembly.
 * read_timings synchronises on the recorded events, sums elapsed ms per category and resets. */
int nb200_engine_set_timing(nb200_engine* eng, int32_t enable);
int nb200_engine_read_timings(nb200_engine* eng, float* ms_per_cat, int32_t* scopes_per_cat, int32_t n_cat);
/* Node-level dense layers: the hand-written wgmma 3xTF32 GEMM (fp32-accurate) is the only backend.
 * 1 -> NB200_OK; 0 (the former cuBLAS SGEMM backend) -> NB200_EUNSUPPORTED; anything else -> NB200_EINVAL. */
int nb200_engine_set_gemm_backend(nb200_engine* eng, int32_t backend);
/* PaiNN per-atom part of a layer (PaiNNUpdate.forward painn.py:535-548, x_proj painn.py:459-464, out_energy[0]
 * painn.py:79-83 and their backward): ONE fused wgmma kernel per layer and direction (painn_fused.cu: weights pre-split into
 * TF32 hi/lo shared-memory images, chained MMAs, elementwise glue in loaders / epilogues) is the only node forward.
 * 1 -> NB200_OK; 0 (the former one-launch-per-op sequence) -> NB200_EUNSUPPORTED; anything else -> NB200_EINVAL. */
int nb200_engine_set_node_backend(nb200_engine* eng, int32_t backend);
/* C[M,N] = A[M,K] . op(B) (+C) (+bias), optional act = silu(C); fp32 in/out, 3xTF32 on wgmma.
 * op(B) = B[N,K]^T (trans_b=0, torch.nn.Linear forward: nablaDFT/painn_pyg/painn.py:459-464)
 *       | B[K,N]   (trans_b=1, its input gradient).  K % 32 == 0, N % 4 == 0, ld* % 4 == 0. */
int nb200_gemm_tf32x3(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B,
                      int32_t ldb, int32_t trans_b, float* C, int32_t ldc, int32_t accumulate,
                      const float* bias, float* act, void* stream);
/* Test entry point: nb200_gemm_tf32x3 with the row count in device memory.  M is an upper bound: it sizes the grid and picks the kernel
 * (the same choice as nb200_gemm_tf32x3 with that M); rows at or beyond min(M, *m_dev) are neither computed nor written.  m_dev == NULL:
 * exactly nb200_gemm_tf32x3. */
int nb200_gemm_tf32x3_rows(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb, int32_t trans_b,
                           float* C, int32_t ldc, int32_t accumulate, const float* bias, float* act, const int32_t* m_dev, void* stream);
/* Test entry point: the tall-layer GEMM with a fused tail, as GemNet-OC's Dense layers run it (gemm_ps.cu).  With o = A . op(B) (+ bias):
 *   epi = 1 (activation): C = act(o);   epi = 2 (residual): C = (C + act(o)) * alpha, C holding the layer input.
 * act_kind: 3 = ScaledSiLU, silu(x) / 0.6.  Columns at and past N of each C row are not touched.  NB200_EINVAL (nothing launched) for
 * another epi or A == C; NB200_EUNSUPPORTED for K % 4 != 0, lda % 4 != 0 or ldc < N.  Device library only. */
int nb200_gemm_tf32x3_epi(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb, int32_t trans_b,
                          float* C, int32_t ldc, const float* bias, int32_t epi, int32_t act_kind, float alpha, void* stream);
/* Weight / bias gradient of a Linear layer (torch autograd: grad_weight = grad_out^T @ input, grad_bias = grad_out.sum(0); every
 * nn.Linear of nablaDFT/painn_pyg/painn.py), ACCUMULATED into dW / dbias:
 *   dW[out,in] += alpha * ( (c o G0)^T X0 + G1^T X1 ),   dbias[out] += bias_alpha * colsum(c o G0)
 * G*[M,out] (ldg), X*[M,in] (ldx); G1/X1 NULL = one term; dbias NULL = none; row_scale c NULL = none, else row a is scaled by
 * row_scale[a / rs_div].  wgmma 3xTF32 split-K over the M rows with atomic fp32 accumulation (wgrad_tc.cu).
 * in <= 128, in % 16 == 0, out % 4 == 0, ld* % 4 == 0, 16-byte aligned pointers; NB200_EINVAL otherwise. */
int nb200_linear_wgrad(int32_t M, int32_t out, int32_t in, const float* G0, const float* X0, const float* G1,
                       const float* X1, int32_t ldg, int32_t ldx, float* dW, int32_t lddw, float alpha,
                       float* dbias, float bias_alpha, const float* row_scale, int32_t rs_div, void* stream);
/* Storage of the per-edge arrays (radial filter rows W, dW/dd and the per-edge filter gradients) in the PaiNN TRAINING calls below:
 * 0 = fp32 (default), 1 = bf16 storage with fp32 arithmetic and accumulation -- BASELINE configs[2] ("PaiNN energy+forces training ... bf16";
 * the reference itself trains in fp32, SURVEY.md section 0.9).  Node-level activations, weights and gradients stay fp32; inference is always fp32. */
int nb200_engine_set_edge_storage(nb200_engine* eng, int32_t bf16);
/* Hand-written kernels launched by this engine since creation (cuBLAS GEMMs not counted). */
int64_t nb200_engine_own_launches(nb200_engine* eng);
/* Bytes of workspace the engine needs for a batch of at most (b_cap, n_cap, e_cap). */
int64_t nb200_painn_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap,
                                    int32_t e_cap, int32_t with_forces);
/* energy[B], forces[N,3] (NULL => energy only), status[4] as nb200_neighbor_build. */
int nb200_painn_energy_forces(nb200_engine* eng, const nb200_painn_weights* w,
                              const int32_t* z, const float* pos, const int32_t* mol_ptr,
                              int32_t n_mol, int32_t n_atoms, int32_t e_cap,
                              void* workspace, int64_t workspace_bytes,
                              float* energy, float* forces, int32_t* status, void* stream);
/* Training step (SURVEY.md section 8 a10/a11, BASELINE configs[2]; replaces loss.backward() through the eager graph of
 * nablaDFT/painn_pyg/painn.py:642-653 / schnetpack AtomisticTask): same forward + analytic backward, plus
 *     d/dtheta [ sum_m energy_seed[m] E_m + sum_i force_seed[i] . F_i ]
 * written into the arrays `grads` points to (a nb200_painn_weights whose pointers address gradient buffers of the same
 * shapes; scalars ignored; all overwritten).  energy_seed = dLoss/dE_m (NULL => ones); force_seed = dLoss/dF_i [n_atoms,3]
 * (NULL => no force term).  The force term is the reference's double backward (create_graph=True, painn.py:142), computed
 * as the directional derivative of the energy gradient along force_seed by a forward-mode tangent pass (painn_tangent.cu).
 * forces are the true -dE/dR (not seed-weighted). */
int64_t nb200_painn_train_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap,
                                          int32_t e_cap, int32_t with_force_seed);
int nb200_painn_energy_forces_grads(nb200_engine* eng, const nb200_painn_weights* w,
                                    const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                    int32_t n_mol, int32_t n_atoms, int32_t e_cap,
                                    void* workspace, int64_t workspace_bytes,
                                    const float* energy_seed, const float* force_seed,
                                    const nb200_painn_weights* grads,
                                    float* energy, float* forces, int32_t* status, void* stream);
/* The same training step as TWO calls, so that the forward is not recomputed once the loss has produced the seeds (the reference keeps its
 * autograd graph between model(batch) and loss.backward(), painn.py:642-653):
 *   nb200_painn_train_forward   graph, filters, fused forward and force backward; energy[B], forces[N,3]; every activation the gradient
 *                               pass reads stays in `workspace`
 *   nb200_painn_train_backward  tangent pass + backward with the weight gradients from the kept arrays; `grads` as above
 * `workspace` >= nb200_painn_train_workspace_bytes(w, b, n, e_cap, with_force_seed) with the SAME with_force_seed in both calls; nothing else
 * may touch it in between; w, z, mol_ptr, n_mol, n_atoms, e_cap must be those of the forward call.  force_seed != NULL needs with_force_seed. */
int nb200_painn_train_forward(nb200_engine* eng, const nb200_painn_weights* w,
                              const int32_t* z, const float* pos, const int32_t* mol_ptr,
                              int32_t n_mol, int32_t n_atoms, int32_t e_cap,
                              void* workspace, int64_t workspace_bytes, int32_t with_force_seed,
                              float* energy, float* forces, int32_t* status, void* stream);
int nb200_painn_train_backward(nb200_engine* eng, const nb200_painn_weights* w,
                               const int32_t* z, const int32_t* mol_ptr,
                               int32_t n_mol, int32_t n_atoms, int32_t e_cap,
                               void* workspace, int64_t workspace_bytes, int32_t with_force_seed,
                               const float* energy_seed, const float* force_seed,
                               const nb200_painn_weights* grads, int32_t* status, void* stream);
/* Hessian-vector products of the PaiNN energy (both radial flavours): for each of n_dir position-space directions v[d] ([N,3], Angstrom)
 *     hv[d] = H v[d] = -(dF/dR) v[d]       (H = d2 E / dR dR in Ha/A^2, so hv is in Ha/A)
 * exact (forward-over-reverse tangent pass, no finite step), fp32 arithmetic and storage.  The primal forward runs once per call, the
 * directions one after another; energy[B] and forces[N,3] (NULL => not written) are those of nb200_painn_energy_forces.  Molecules do not
 * interact: one direction may displace an atom of every molecule at once.  `workspace` >= nb200_painn_hvp_workspace_bytes(w, b, n, e_cap,
 * n_dir) (independent of n_dir >= 1).  Status and capacity conventions as nb200_painn_energy_forces; on a device error flag energy, forces
 * and hv are NaN.  NB200_EINVAL (nothing launched) for a null required pointer, n_dir < 1 or a short workspace. */
int64_t nb200_painn_hvp_workspace_bytes(const nb200_painn_weights* w, int32_t b_cap, int32_t n_cap, int32_t e_cap, int32_t n_dir);
int nb200_painn_hvp(nb200_engine* eng, const nb200_painn_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                    int32_t n_mol, int32_t n_atoms, int32_t e_cap, void* workspace, int64_t workspace_bytes,
                    int32_t n_dir, const float* v, float* energy, float* forces, float* hv, int32_t* status, void* stream);
/* Test entry point, not a supported API: ONE kernel of the PaiNN tangent / Hessian-vector-product path on caller-built inputs, through the
 * same host wrapper (hence launch configuration) the engine uses.  F = 128; per-atom arrays [n_atoms, k F] as in the engine; graph as in
 * the batch layout above.  `op` (NB200_PT_*) selects the kernel and the fields it reads and writes:
 *   GEOM_TAN          geom row_ptr col v -> t_geom
 *   MUL_DACT          pre x n -> out                                  (n % 4 == 0)
 *   ACT_BWD_TAN       t_g (in / out) g_pre pre t_pre n                 (n % 4 == 0)
 *   READOUT_BWD_TAN   pre t_pre R2 width -> t_g_pre t_act              ([n_atoms, width])
 *   MSG_FWD_TAN       xh t_xh xh_bias mu t_mu W dW geom t_geom row_ptr col [rev] -> t_q (accumulated) t_mu_out
 *   UPD_NORM_TAN      VW t_VW nrm -> t_nrm
 *   UPD_COMBINE_TAN   VW t_VW y t_y -> t_q t_mu (both accumulated)
 *   UPD_COMBINE_BWD_TAN  g_q t_g_q g_mu t_g_mu y t_y VW t_VW -> t_gy t_gVW
 *   UPD_NORM_BWD_TAN  gn t_gn VW t_VW nrm t_nrm -> t_gVW (accumulated)
 *   MSG_BWD_TAN       as MSG_FWD_TAN without t_q, plus g_q t_g_q g_mu t_g_mu -> t_g_xh t_g_mu_in t_gW gWd
 *   MSG_BWD_HVP       as MSG_BWD_TAN plus d2W, rev required -> t_g_xh t_g_mu_in t_egrad (accumulated)
 *   EDGE_FORCES_HVP   egrad t_egrad geom t_geom row_ptr rev -> hv
 *   FILTER_D2         geom status rev sort_scratch + radial fields, e_cap = row stride -> W dW d2W (one row per undirected pair)
 *   FILTER_WGRAD      geom status sort_scratch + radial fields, e_cap >= status[0]; gW (tan = 0) or t_gW gWd (tan = 1) -> g_w g_b
 *                     (accumulated; the entry sorts every directed edge by distance bin into sort_scratch first)
 * `rev` NULL for MSG_FWD_TAN / MSG_BWD_TAN: every edge reads its own filter row; otherwise row min(e, rev[e]).  bf16 = 1 (MSG_FWD_TAN,
 * MSG_BWD_TAN, FILTER_WGRAD only): W, dW, t_gW, gWd, gW hold bf16.  status = {n_edges, 0} in device memory; sort_scratch int32
 * [768 + n_edges].  NB200_EINVAL (nothing launched) for an unknown op, a NULL field the op reads or writes, n_atoms < 0, n < 0, n % 4 != 0
 * for the element-wise ops, width < 1, e_cap < 0, bf16 or tan where the op has no such instance; NB200_EUNSUPPORTED for radial
 * parameters the filter kernels do not support. */
enum {
    NB200_PT_GEOM_TAN = 0, NB200_PT_MUL_DACT, NB200_PT_ACT_BWD_TAN, NB200_PT_READOUT_BWD_TAN, NB200_PT_MSG_FWD_TAN, NB200_PT_UPD_NORM_TAN,
    NB200_PT_UPD_COMBINE_TAN, NB200_PT_UPD_COMBINE_BWD_TAN, NB200_PT_UPD_NORM_BWD_TAN, NB200_PT_MSG_BWD_TAN, NB200_PT_MSG_BWD_HVP,
    NB200_PT_EDGE_FORCES_HVP, NB200_PT_FILTER_D2, NB200_PT_FILTER_WGRAD, NB200_PT_N_OPS
};
typedef struct nb200_painn_tan_args {
    int32_t op, bf16, tan, n_atoms;
    int64_t n;
    int32_t width, e_cap;
    const int32_t *row_ptr, *col, *rev, *status;
    int32_t* sort_scratch;
    const float *geom, *v;
    float* t_geom;
    const float *xh, *t_xh, *xh_bias, *mu;
    float *t_mu, *t_q, *t_mu_out;
    void *W, *dW;
    float* d2W;
    const float *g_q, *t_g_q, *g_mu, *t_g_mu;
    float *t_g_xh, *t_g_mu_in;
    void *gW, *t_gW, *gWd;
    const float *VW, *t_VW, *nrm, *y, *t_y, *gn, *t_gn;
    float *t_nrm, *t_gy, *t_gVW;
    const float *pre, *t_pre, *x, *g_pre, *R2;
    float *out, *t_g, *t_g_pre, *t_act;
    const float* egrad;
    float *t_egrad, *hv;
    int32_t radial_mode, n_rbf, n_layers;
    float cutoff, rbf_coeff, rbf_xscale, sign;
    const float *rbf_offsets, *w_rbf, *b_rbf;
    float *g_w, *g_b;
} nb200_painn_tan_args;
int nb200_painn_test_tangent(const nb200_painn_tan_args* args, void* stream);
/* Test entry point, not a supported API: ONE program of the fused PaiNN node kernels (painn_fused.cu), their weight preparation, or one
 * primal per-atom kernel of painn_node.cu, on caller-built inputs, through the host wrapper the engine calls (hence its launch
 * configuration).  F = 128; per-atom arrays [n_atoms, k F] as in the engine; weights, eps and biases from `w` (n_feat = F).  `op`:
 *   PREP              w -> wtiles [nb_fused_wtile_bytes(n_layers) bytes: (22 n_layers + 2) tiles of 128 KB]
 *   NODE_FWD          prep into wtiles, then the forward program (layer_upd, layer_mlp, readout):
 *                       (-1, l, 0)   q_mlp_in -> h1pre xh                        (message MLP of layer l on the embedding)
 *                       (l, l+1, 0)  q_mid mu_mid -> VW nrm dot g1pre y q_next mu_next h1pre xh
 *                       (l, -1, 1)   q_mid mu_mid -> VW nrm dot g1pre y q_next mu_next ro_pre (without e1)
 *   NODE_BWD          prep into wtiles, then the backward program:
 *                       readout = 1, layer_mlp = -1, layer_upd = l:  ro_pre (with e1) y VW nrm dot g1pre, cur (in / out) -> gq_b gdot gn gq_a
 *                       readout = 0, layer_mlp = l+1, layer_upd = l: g_xh h1pre y VW nrm dot g1pre, gq_a cur (in / out) -> gq_b gdot gn
 *                     tile: 0 (the engine's rule), 64 or 80 atoms per CTA in; the width that ran out.
 *   EMBED             z -> q mu, status[1] = NB200_EINVAL for an element outside [z_offset, z_offset + n_elem)
 *   ACT_BWD           g (in / out) pre n kind (NB_ACT_SILU 0 or NB_ACT_SSP 1)      (n % 4 == 0)
 *   UPD_COMBINE_BWD   gq gmu y VW -> gy gVW
 *   UPD_NORM_BWD      gn VW nrm -> gVW (accumulated)
 *   READOUT           pre [n_atoms, F/2] (in / out: += e1) -> eps_atom
 *   MOL_SUM           eps_atom mol_ptr n_mol -> energy
 *   READOUT_BWD       pre -> g_pre [n_atoms, F/2]
 *   POISON            status energy n_mol, forces (may be NULL) n -> NaN where status[1] != 0
 * NB200_EINVAL (nothing launched) for an unknown op or program, a layer index outside [0, n_layers), tile not in {0, 64, 80}, n_atoms < 0,
 * n < 0, n_mol < 0, a NULL field the op uses, or a pointer the float4 paths read or write that is not 16-byte aligned. */
enum {
    NB200_PN_PREP = 0, NB200_PN_NODE_FWD, NB200_PN_NODE_BWD, NB200_PN_EMBED, NB200_PN_ACT_BWD, NB200_PN_UPD_COMBINE_BWD, NB200_PN_UPD_NORM_BWD,
    NB200_PN_READOUT, NB200_PN_MOL_SUM, NB200_PN_READOUT_BWD, NB200_PN_POISON, NB200_PN_N_OPS
};
typedef struct nb200_painn_node_args {
    int32_t op, n_atoms, tile, layer_upd, layer_mlp, readout;
    const nb200_painn_weights* w;
    void* wtiles;
    const float *q_mid, *mu_mid, *q_mlp_in, *g_xh;
    float *VW, *nrm, *dot, *g1pre, *y, *q_next, *mu_next, *h1pre, *xh, *ro_pre;
    float *gq_a, *gq_b, *cur, *gn, *gdot;
    const int32_t *z, *mol_ptr;
    int32_t* status;
    int32_t n_mol, kind;
    int64_t n;
    const float *gq, *gmu;
    float *q, *mu, *g, *pre, *gy, *gVW, *eps_atom, *energy, *forces, *g_pre;
} nb200_painn_node_args;
int nb200_painn_test_node(nb200_painn_node_args* args, void* stream);

/* ----------------------------------------------------------------------------------------
 * SchNet energy + forces (config/model/schnet.yaml: schnetpack.representation.SchNet inside
 * NeuralNetworkPotential; SURVEY.md A.1, section 8 row a8).  Same engine object, batch layout,
 * status and workspace conventions as the PaiNN entry point.
 * -------------------------------------------------------------------------------------- */
typedef struct nb200_schnet_weights {
    int32_t n_layers, n_feat, n_rbf, n_elem; /* 6, F(=128, n_filters == n_atom_basis), 100, rows of emb */
    int32_t z_offset;                        /* 0                                            */
    float cutoff, rbf_coeff;                 /* 5.0 ; phi_k = exp(coeff (d - offsets[k])^2)  */
    float energy_shift_per_atom;             /* AddOffsets mean (eval)                       */
    const float* rbf_offsets;                /* [K]; must be k dx, dx = cutoff / (K - 1): nb200_schnet_energy_forces evaluates only the
                                              * 16 centres around bin floor(d / dx) (the training and Hessian entries evaluate all K) */
    const float* emb;                        /* [n_elem][F]                                  */
    const float* w_f1; const float* b_f1;    /* [L][K][F] (K-major), [L][F]  filter_network.0 (ssp) */
    const float* W_f2; const float* b_f2;    /* [L][F][F], [L][F]            filter_network.1 */
    const float* I1;                         /* [L][F][F]                    in2f (no bias)   */
    const float* P1; const float* p1;        /* [L][F][F], [L][F]            f2out.0 (ssp)    */
    const float* P2; const float* p2;        /* [L][F][F], [L][F]            f2out.1          */
    const float* R1; const float* e1;        /* [F/2][F], [F/2]              Atomwise outnet  */
    const float* R2; const float* e2;        /* [1][F/2], [1]                                 */
} nb200_schnet_weights;

int64_t nb200_schnet_workspace_bytes(const nb200_schnet_weights* w, int32_t b_cap, int32_t n_cap,
                                     int32_t e_cap, int32_t with_forces);
int nb200_schnet_energy_forces(nb200_engine* eng, const nb200_schnet_weights* w,
                               const int32_t* z, const float* pos, const int32_t* mol_ptr,
                               int32_t n_mol, int32_t n_atoms, int32_t e_cap,
                               void* workspace, int64_t workspace_bytes,
                               float* energy, float* forces, int32_t* status, void* stream);
/* Test entry point, not a supported API: ONE launch of nb200_schnet_energy_forces (csrc/schnet.cu) on caller-built inputs, through the
 * wrapper the engine calls (hence its launch configuration).  F = 128; per-edge rows [E][F] in CSR order, geom [E][4] with d in slot 3.  `op`:
 *   FILTER1      geom status(= {n_edges, 0}) w_f1 b_f1 rbf_offsets n_layers n_rbf cutoff rbf_coeff e_stride, sort_scratch int32
 *                [768 + n_edges] -> HH [n_layers][2][e_stride][F] (h, dh/dd; rows at and past n_edges untouched)
 *   CFCONV_FWD   y G1 b2 geom row_ptr col cutoff n_atoms -> agg [n_atoms][F]
 *   CFCONV_BWD   y G1 G2 b2 geom row_ptr col cutoff n_atoms gagg -> gy [n_atoms][F], egrad[4 e + 3] (accumulated)
 *   LINEAR_ACT   X [m][F] W [F][F] bias [F] -> Y = X W^T + bias, act = ssp(Y)      (the GEMM the engine runs for f2out.0)
 * NB200_EINVAL (nothing launched) for an unknown op, a NULL field the op uses, a pointer the float4 paths read or write that is not 16-byte
 * aligned, a negative count or e_stride < n_edges; NB200_EUNSUPPORTED for n_rbf or rbf_coeff that nb200_schnet_energy_forces refuses. */
enum { NB200_SC_FILTER1 = 0, NB200_SC_CFCONV_FWD, NB200_SC_CFCONV_BWD, NB200_SC_LINEAR_ACT, NB200_SC_N_OPS };
typedef struct nb200_schnet_test_args {
    int32_t op, n_layers, n_rbf, n_atoms, n_edges, e_stride, m;
    float cutoff, rbf_coeff;
    const int32_t *status, *row_ptr, *col;
    int32_t* sort_scratch;
    const float *geom, *rbf_offsets, *w_f1, *b_f1, *y, *G1, *G2, *b2, *gagg, *X, *W, *bias;
    float *HH, *agg, *gy, *egrad, *Y, *act;
} nb200_schnet_test_args;
int nb200_schnet_test_op(const nb200_schnet_test_args* args, void* stream);

/* SchNet parameter gradients of energy and force losses (config/model/schnet.yaml; BASELINE configs[0]; SURVEY.md section 8 a8 / a10 / a11).
 * Replaces `loss.backward()` through schnetpack's eager SchNet + Atomwise graph (config/model/schnet.yaml, nablaDFT/ase_model/task.py) for
 * losses that depend on the energies only.  Two phases like the GemNet-OC entry points:
 *   nb200_schnet_train_count           CSR row pointers of the ASE-style neighbour list (d < cutoff, both directions); returns the edge
 *                                      count (ONE host synchronisation).  row_ptr: device int32 [N+1]; scratch: device int32 [2 N].
 *   nb200_schnet_train_workspace_bytes bytes for the saved activations of a batch with that many edges.
 *   nb200_schnet_energy_grads          forward with saved activations -> energy[B]; with a seed also the reverse sweep(s):
 *                                      grads->X = d(sum_m energy_seed[m] E_m + sum_i force_seed[i] . F_i)/dX, F = -dE_tot/dR, for every weight
 *                                      tensor X of the struct (same shapes, device buffers owned by the caller, zeroed by the call; rbf_offsets
 *                                      ignored).  energy_seed [B] and force_seed [N,3] are dLoss/dE and dLoss/dF; either may be NULL.  The force
 *                                      term replaces the reference's create_graph double backward by an exact tangent pass (DESIGN.md 3.7).
 * FIRST CORRECT PATH, verified under host emulation only (csrc/schnet_train.cu). */
int nb200_schnet_train_count(const nb200_schnet_weights* w, const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                             int32_t* row_ptr, int32_t* scratch, int64_t* n_edges_host, void* stream);
int64_t nb200_schnet_train_workspace_bytes(const nb200_schnet_weights* w, int32_t n_mol, int32_t n_atoms, int64_t n_edges,
                                           int32_t with_force_seed);
int nb200_schnet_energy_grads(nb200_engine* eng, const nb200_schnet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                              int32_t n_mol, int32_t n_atoms, const int32_t* row_ptr, int64_t n_edges, void* workspace,
                              int64_t workspace_bytes, const float* energy_seed, const float* force_seed,
                              const nb200_schnet_weights* grads, float* energy, void* stream);
/* Hessian-vector products of the SchNet energy (csrc/schnet_hvp.inc, DESIGN.md 3.13.1): for each of n_dir position-space directions v[d]
 * ([N,3], Angstrom)  hv[d] = H v[d] = -(dF/dR) v[d] in Ha/A, exact (forward-over-reverse, no finite step), fp32 arithmetic and storage.  The
 * primal forward, the filter's radial derivatives and the reverse sweep run once per call, the directions one after another, so the workspace
 * does not depend on n_dir.  energy[B] follows w->energy_shift_per_atom; forces[N,3] (NULL => not written) are those of the same pass.
 * row_ptr / n_edges come from nb200_schnet_train_count.  No atomics: bitwise repeatable, independent of how directions are chunked.
 * NB200_EINVAL (nothing launched) for a null required pointer, n_dir < 1, a short workspace or an invalid configuration. */
int64_t nb200_schnet_hvp_workspace_bytes(const nb200_schnet_weights* w, int32_t n_mol, int32_t n_atoms, int64_t n_edges);
int nb200_schnet_hvp(nb200_engine* eng, const nb200_schnet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                     int32_t n_mol, int32_t n_atoms, const int32_t* row_ptr, int64_t n_edges, void* workspace, int64_t workspace_bytes,
                     int32_t n_dir, const float* v, float* energy, float* forces, float* hv, void* stream);

/* ----------------------------------------------------------------------------------------
 * QHNet (config/model/qhnet.yaml; nablaDFT/qhnet/qhnet.py + layers.py over e3nn 0.5.1) operators.
 * Equivariant features: [rows][25 (l,m), l <= 4][channels] fp32, channels contiguous.
 * Graph: the CSR of nb200_neighbor_build (row = reference `src`... see csrc/qhnet.cu header);
 * `tgt[E]` = row owner of every CSR entry (nb200_qh_expand_rows).  n_edges is read from status[0].
 * -------------------------------------------------------------------------------------- */
int nb200_qh_expand_rows(const int32_t* row_ptr, int32_t n_atoms, int32_t* tgt, void* stream);
/* a12: ExponentialBernsteinRadialBasisFunctions (layers.py:86-120) + o3.spherical_harmonics l<=4 of
 * sign * edge direction (qhnet.py:264-271).  rbf [E][n_rbf] and/or sh [E][25] may be NULL.  alpha and
 * logc [n_rbf] (log binomial coefficients) are double: the basis exponent is summed in double. */
int nb200_qh_edge_basis(const float* geom, const int32_t* status, int32_t e_cap, double alpha, float cutoff,
                        float sign, const double* logc, int32_t n_rbf, float* rbf, float* sh, void* stream);
/* NormGate pieces (layers.py:123-147): f0 [R][640] = [scalars, norms l=1..4]; y = [gates0, x_l * gates_l] */
int nb200_qh_norm_feats(const float* x, int32_t n_rows, float* f0, void* stream);
int nb200_qh_gate(const float* x, const float* gates, int32_t n_rows, float* y, void* stream);
/* InnerProduct + concatenation feeding the weight MLPs (layers.py:237-259,469-476); mode 0 conv,
 * 1 conv layer 0 (scalars only), 2 pair. */
int nb200_qh_invariants(const float* f, const int32_t* tgt, const int32_t* col, const int32_t* status,
                        int32_t e_cap, int32_t mode, float* out, void* stream);
/* a13 ConvLayer tensor product 'uvu' + aggregation (layers.py:263-271) */
int nb200_qh_tp_conv(const float* x, const float* sh, const float* w1, const float* w2, const int32_t* row_ptr,
                     const int32_t* col, int32_t n_atoms, int32_t layer0, int32_t add_self, float* out, void* stream);
/* a14 PairNetLayer tensor product 'uuu' with per-pair weights (layers.py:481-485) */
int nb200_qh_tp_pair(const float* x, const float* w1, const float* w2, const int32_t* tgt, const int32_t* col,
                     const int32_t* status, int32_t p_cap, float* out, void* stream);
/* a15 SelfNetLayer tensor product 'uuu' with internal weights + residual (layers.py:571-573) */
int nb200_qh_tp_self(const float* xl, const float* xr, const float* w, const float* res, int32_t n_rows,
                     float* out, void* stream);
/* e3nn o3.Linear over the 25 (l,m) rows: W_l [5][c_in][c_out] pre-scaled by 1/sqrt(c_in); bias on (0,0) */
int nb200_qh_linear(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in,
                    int32_t c_out, int32_t accumulate, float* y, void* stream);
/* fp32-accurate dense layer (wgmma 3xTF32) with activation kind 0 silu, 1 ssp, 2 1.8782*ssp */
int nb200_dense(int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb,
                int32_t trans_b, float* C, int32_t ldc, int32_t accumulate, const float* bias, float* act,
                int32_t act_kind, void* stream);
/* a16 Expansion (layers.py:598-662): tables uploaded once (19 instructions, w3j/32) */
int nb200_qh_expand_setup(const int32_t* ins_host, const float* cg_host);
int nb200_qh_expand(const float* x, const float* W, const float* Bw, int32_t bw_stride, int32_t n_rows,
                    float* blocks, void* stream);
int nb200_qh_pair_hidden(const float* A, const float* Bn, const float* bias, const int32_t* tgt,
                         const int32_t* col, const int32_t* status, int32_t p_cap, float* h, void* stream);
/* a17 build_final_matrix + H + H^T (qhnet.py:293-321,234-238): per-molecule dense H, packed */
int nb200_qh_assemble(const float* diag, const float* offd, const int32_t* z, const int32_t* tgt,
                      const int32_t* col, const int32_t* rev, int32_t n_atoms, int32_t n_pairs,
                      const int32_t* mask_tab, const int32_t* norb_tab, const int32_t* atom_mol,
                      const int32_t* atom_orb_off, const int64_t* mol_h_off, const int32_t* mol_norb,
                      float* H, void* stream);
int nb200_axpy(float* y, const float* x, int64_t n, void* stream);

/* ----------------------------------------------------------------------------------------
 * Batch-wise L-BFGS geometry optimisation (SURVEY.md section 8f-1).
 * One call = ASEBatchwiseLBFGS.step + update + determine_step of
 * nablaDFT/optimization/optimizers.py:436-598 for a whole batch, on the device: one CTA per
 * molecule, mixed float64 / float32 arithmetic as in the reference (oracle/lbfgs.py).
 *   state            caller-owned device buffer of nb200_lbfgs_state_bytes() bytes holding the s / y / rho
 *                    history ring and (r0, f0); needs no initialisation (nothing is read at iteration 0)
 *   iteration        number of steps already taken with this state (self.iteration, optimizers.py:409,527)
 *   fmax             molecules whose largest |f| is below fmax are frozen (optimizers.py:446-456, 505-506)
 *   h0               1 / alpha (optimizers.py:396)
 *   fixed_mask       optional uint8 [n_atoms]: 1 = force zeroed (calculator.py:86-88; written back to `forces`)
 *   pos              double [n_atoms,3], in/out;  forces float [n_atoms,3], in;  pos32_out = (float)pos for the model
 *   unconverged_out  int32: number of molecules NOT frozen at this step (0 => BatchwiseOptimizer.converged,
 *                    optimizers.py:242-247, was true before the step and the step moved nothing)
 *   n_normalizations int32 counter, incremented per rescaled molecule (optimizers.py:567)
 * Asynchronous on `stream`; no host synchronisation. */
int64_t nb200_lbfgs_state_bytes(int32_t n_mol, int32_t n_atoms, int32_t memory);
int nb200_lbfgs_step(void* state, int64_t state_bytes, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms,
                     int32_t max_atoms_per_mol, int32_t memory, int32_t iteration, double fmax, double maxstep,
                     double damping, double h0, const uint8_t* fixed_mask, double* pos, float* forces,
                     float* pos32_out, int32_t* unconverged_out, int32_t* n_normalizations, void* stream);

/* ----------------------------------------------------------------------------------------
 * Batch-wise QuasiNewton geometry optimisation: ASE's BFGSLineSearch + LineSearch (the optimiser of
 * PYGAseInterface.optimize, nablaDFT/optimization/pyg_ase_interface.py:296-315) for every molecule of a batch
 * independently (csrc/quasinewton.cu, oracle/quasinewton.py).  Call once after each energy + forces evaluation:
 * every molecule consumes E and F at its current trial point and either writes its next trial point to pos /
 * pos32 or stops; a stopped molecule is never touched again.  One CTA per molecule.
 *   state        device buffer of nb200_qn_state_bytes() bytes, zero-filled before the first call: line-search
 *                scalars, the dense inverse Hessians (3n_i x 3n_i float64 at hess_off[i], hess_elems doubles in
 *                all), the start point, direction and scaled gradient of the current step
 *   hess_off     int64 [n_mol], element offset of molecule i's inverse Hessian
 *   fmax         stop a molecule when max |F| < fmax (tested in float32); max_steps caps its BFGS steps
 *   maxstep, c1, c2, alpha, stpmax   BFGSLineSearch arguments (ASE units: eV, A)
 *   e_scale, f_scale   energy [n_mol] / forces [n_atoms,3] float32 of the model times these = eV, eV/A
 *   fixed_mask   optional uint8 [n_atoms]: 1 = FixAtoms (force zeroed, position never changes)
 *   pos          double [n_atoms,3], in/out;  pos32 = (float)pos, out (unchanged for stopped molecules)
 *   max_atoms_per_mol   at least the largest mol_ptr[i+1] - mol_ptr[i]: it sizes the kernel's shared memory; a larger
 *                molecule is refused (status 4) without being touched
 *   mol_info     int32 [n_mol][4], zero-filled before the first call: status (0 running, 1 converged, 2 max_steps,
 *                3 line search failed, 4 molecule larger than max_atoms_per_mol or hess_off outside hess_elems), nsteps,
 *                force_calls, function_calls
 *   running_out  int32: molecules still running after this call
 * NB200_EINVAL (nothing launched) for a null required pointer, a negative size, alpha or maxstep <= 0, or a short
 * state.  Asynchronous on `stream`; no host synchronisation. */
int64_t nb200_qn_state_bytes(int32_t n_mol, int32_t n_atoms, int64_t hess_elems);
int nb200_qn_step(void* state, int64_t state_bytes, const int32_t* mol_ptr, const int64_t* hess_off, int32_t n_mol,
                  int32_t n_atoms, int32_t max_atoms_per_mol, int64_t hess_elems, double fmax, int32_t max_steps,
                  double maxstep, double c1, double c2, double alpha, double stpmax, double e_scale, double f_scale,
                  const uint8_t* fixed_mask, const float* energy, const float* forces, double* pos, float* pos32,
                  int32_t* mol_info, int32_t* running_out, void* stream);

/* ----------------------------------------------------------------------------------------
 * Batched molecular dynamics (PYGAseInterface.init_md / run_md of nablaDFT/optimization/pyg_ase_interface.py): ASE 3.22
 * VelocityVerlet and Langevin(fixcm=True) for a whole batch, one CTA per molecule, float64 positions and momenta (csrc/md.cu,
 * oracle/md.py).  ASE units: eV, A, u, ASE time.  Noise: counter-based Philox4x32-10, key = seed, counter = (global atom index,
 * noise step, stream, call); the layout is specified in csrc/md.cu.  The caller owns every buffer:
 *   mass   double [n_atoms] (u);  pos, mom  double [n_atoms,3], in/out;  pos32 float [n_atoms,3] = (float)pos for the engine
 *   forces float [n_atoms,3] and energy float [n_mol] in the engine's units; f_scale / e_scale convert them to eV/A and eV
 * nb200_md_init_momenta: MaxwellBoltzmannDistribution(kT), then Stationary and ZeroRotation, each rescaling back to the kinetic
 *   energy it found (preserve_temperature); noise step `noise_step`, stream 0.  A principal moment below 1e-10 of the largest counts as
 *   zero; a molecule without kinetic energy is not rescaled.
 * nb200_md_step: `phase` = 1 FINISH (second half-kick of the step with noise step `step`, with `forces` evaluated at `pos`) | 2 START
 *   (first half-kick and drift of step `step + 1`; writes pos, mom, pos32).  thermostat 0: velocity Verlet; 1: Langevin at kT with
 *   friction `gamma` (1 / ASE time).  log_slot (optional) double [n_mol][2]: Epot, Ekin after FINISH and before START; frame_pos /
 *   frame_mom (optional) double [n_atoms,3] copies of pos / mom at the same point.  status (optional, then worst required): the
 *   engine's int32[4] status word; worst[0] = max edges, [1] = min error code, [2] = max degree, [3] = 1 once a status reported
 *   NB200_ECAPACITY.  While status or worst shows an error, the call leaves pos, mom and pos32 untouched (the engine's outputs are NaN).
 * NB200_EINVAL (nothing launched) for a null required pointer, n_mol < 0, dt <= 0, kT < 0, gamma < 0, a bad phase or thermostat,
 * or a noise step outside [0, 2^32); NB200_OK with nothing written for n_mol == 0.  Asynchronous on `stream`. */
int nb200_md_init_momenta(const int32_t* mol_ptr, int32_t n_mol, const double* mass, const double* pos, double kT, uint64_t seed,
                          int64_t noise_step, double* mom, void* stream);
int nb200_md_step(const int32_t* mol_ptr, int32_t n_mol, const double* mass, int32_t phase, int32_t thermostat, double dt, double kT,
                  double gamma, uint64_t seed, int64_t step, double f_scale, double e_scale, double* pos, double* mom, float* pos32,
                  const float* forces, const float* energy, double* log_slot, double* frame_pos, double* frame_mom,
                  const int32_t* status, int32_t* worst, void* stream);

/* ----------------------------------------------------------------------------------------
 * GemNet-OC energy + direct coupled forces (SURVEY.md section 8 a19 / f3), config/model/gemnet-oc.yaml:
 * non-periodic, quadruplet + atom-edge + edge-atom + atom-atom interactions, `forces_coupled`, `extensive`.
 * Replaces GemNetOC.forward (nablaDFT/gemnet_oc/gemnet_oc.py:1121-1251) and everything below it: the four graphs and their
 * triplet / quadruplet index structures (gemnet_oc.py:694-1000, interaction_indices.py:14-305), the bases (gemnet_oc.py:1001-1120,
 * layers/radial_basis.py, spherical_basis.py, efficient.py) and the interaction / output blocks (layers/interaction_block.py,
 * atom_update_block.py, embedding_block.py).
 * FIRST CORRECT PATH: index structures are never materialised -- triplets and quadruplets are enumerated from CSR rows (by target
 * atom, sources ascending) inside the aggregation kernels and the Legendre bases are evaluated on the fly (DESIGN.md 3.9).
 * Sizes are fixed to the shipped config: emb_size_atom 256, emb_size_edge 512, trip 64/64, quad 32/32, aint 64/64, rbf 16, cbf 16,
 * sbf 32, num_radial 128, num_spherical 7, num_before_skip 2, num_after_skip 2, num_concat 1, num_atom 3, num_output_afteratom 3,
 * num_global_out_layers 2, no biases, activation silu; all four cutoffs equal.  Anything else: NB200_EUNSUPPORTED.
 *
 * Weights: ONE flat device buffer `w` plus a HOST table of offsets (in floats) `off_host`, laid out as
 *   [NB200_GOC_G_* globals][NB200_GOC_I_* per interaction block x num_blocks][NB200_GOC_O_* per output block x (num_blocks+1)]
 * every matrix row-major [out, in] exactly as torch.nn.Linear stores it.  The basis scale factors (scale_file) that multiply a basis
 * ahead of a linear map are folded into the concatenated basis matrices by the host (nabladft_b200/gemnet_oc.py); the per-block
 * scale factors travel in `scale_host` ([NB200_GOC_S_* x num_blocks] then [NB200_GOC_SO_* x (num_blocks+1)]). */
enum { /* globals */
    NB200_GOC_G_RBF_OFFSET = 0, /* [128]        GaussianBasis.offset (radial_basis.py:57-77)                                   */
    NB200_GOC_G_EMB,            /* [83, 256]    atom_emb.embeddings.weight (row z-1)                                            */
    NB200_GOC_G_CAT_MAIN,       /* [1920, 128]  rows 0:16 mlp_rbf_qint | 16:32 mlp_rbf_eaint | 32:48 mlp_rbf_tint | 48:64 mlp_rbf_h |
                                                64:80 mlp_rbf_out | 80:192 mlp_cbf_tint^T | 192:304 mlp_cbf_aeint^T | 304:1872 mlp_sbf_qint^T |
                                                zero padding                                                                   */
    NB200_GOC_G_CAT_AE,         /* [128, 128]   rows 0:16 mlp_rbf_aeint | 16:128 mlp_cbf_eaint^T                                */
    NB200_GOC_G_CAT_Q,          /* [128, 128]   rows 0:112 mlp_cbf_qint^T | zero padding                                        */
    NB200_GOC_G_CAT_A2A,        /* [64, 128]    rows 0:16 mlp_rbf_aint | zero padding                                           */
    NB200_GOC_G_EDGE_EMB,       /* [512, 640]   edge_emb.dense (columns 512:640 pre-multiplied by radial_basis.scale_rbf)       */
    NB200_GOC_G_OUT_E0,         /* [256, 1280]  out_mlp_E.0                                                                     */
    NB200_GOC_G_OUT_E_RES,      /* 4 x [256,256] out_mlp_E.{1,2}.dense_mlp.{0,1}                                                */
    NB200_GOC_G_OUT_ENERGY,     /* [256]        out_energy                                                                      */
    NB200_GOC_G_OUT_F0,         /* [512, 2560]  out_mlp_F.0                                                                     */
    NB200_GOC_G_OUT_F_RES,      /* 4 x [512,512] out_mlp_F.{1,2}.dense_mlp.{0,1}                                                */
    NB200_GOC_G_OUT_FORCES,     /* [512]        out_forces                                                                      */
    NB200_GOC_G_COUNT
};
enum { /* per interaction block (layers/interaction_block.py:19-739) */
    NB200_GOC_I_DENSE_CA = 0,   /* [512,512] */
    NB200_GOC_I_T_BA, NB200_GOC_I_T_RBF /* [512,16] */, NB200_GOC_I_T_BIL /* [64,1024] x scale_cbf_sum */, NB200_GOC_I_T_DOWN /* [64,512] */,
    NB200_GOC_I_T_UPCA /* [512,64] */, NB200_GOC_I_T_UPAC,
    NB200_GOC_I_Q_DB, NB200_GOC_I_Q_RBF, NB200_GOC_I_Q_CBF /* [32,16] */, NB200_GOC_I_Q_BIL /* [32,1024] */, NB200_GOC_I_Q_DOWN /* [32,512] */,
    NB200_GOC_I_Q_UPCA /* [512,32] */, NB200_GOC_I_Q_UPAC,
    NB200_GOC_I_AE_BA /* [256,256] */, NB200_GOC_I_AE_RBF /* [256,16] */, NB200_GOC_I_AE_BIL, NB200_GOC_I_AE_DOWN /* [64,256] */,
    NB200_GOC_I_AE_UPCA /* [512,64] */, NB200_GOC_I_AE_UPAC,
    NB200_GOC_I_EA_BA /* [512,512] */, NB200_GOC_I_EA_RBF, NB200_GOC_I_EA_BIL, NB200_GOC_I_EA_DOWN /* [64,512] */, NB200_GOC_I_EA_UP /* [256,64] */,
    NB200_GOC_I_AA_BIL /* [64,1024] */, NB200_GOC_I_AA_DOWN /* [64,256] */, NB200_GOC_I_AA_UP /* [256,64] */,
    NB200_GOC_I_BEFORE_SKIP,    /* 4 x [512,512]: layers_before_skip.{0,1}.dense_mlp.{0,1} */
    NB200_GOC_I_AFTER_SKIP,     /* 4 x [512,512] */
    NB200_GOC_I_AU_RBF /* [512,16] */, NB200_GOC_I_AU_L0 /* [256,512] */, NB200_GOC_I_AU_RES /* 6 x [256,256] */,
    NB200_GOC_I_CONCAT /* [512,1024] */, NB200_GOC_I_RES_M /* 2 x [512,512] */,
    NB200_GOC_I_COUNT
};
enum { /* per output block (layers/atom_update_block.py:93-172) */
    NB200_GOC_O_RBF = 0 /* [512,16] */, NB200_GOC_O_L0 /* [256,512] */, NB200_GOC_O_RES /* 6 x [256,256] */,
    NB200_GOC_O_E2 /* 6 x [256,256] */, NB200_GOC_O_F /* 6 x [512,512] */, NB200_GOC_O_RBF_F /* [512,16] */,
    NB200_GOC_O_COUNT
};
enum { /* per-interaction-block scale factors applied inside kernels (the factors that follow a bilinear Dense -- scale_cbf_sum,
          scale_sbf_sum, scale_rbf_sum -- are folded into that Dense's weights by the host) */
    NB200_GOC_S_T_RBF = 0, NB200_GOC_S_Q_RBF, NB200_GOC_S_Q_CBF, NB200_GOC_S_AE_RBF, NB200_GOC_S_EA_RBF, NB200_GOC_S_AU_SUM, NB200_GOC_S_COUNT
};
enum { NB200_GOC_SO_SUM = 0, NB200_GOC_SO_RBF_F, NB200_GOC_SO_COUNT }; /* per-output-block scale factors */
enum { /* counts_host[] written by nb200_gemnet_oc_graph_count */
    NB200_GOC_C_A2A = 0, /* atom-atom edges (all same-molecule pairs with d < cutoff_aint)                        */
    NB200_GOC_C_MAIN,    /* main-graph edges after the max_neighbors cut and symmetrisation                       */
    NB200_GOC_C_AE,      /* a2ee2a edges                                                                          */
    NB200_GOC_C_Q,       /* quadruplet-interaction edges                                                          */
    NB200_GOC_C_TIN,     /* slots for the (d->b, b->a) input triplets: sum over qint edges of deg_main(source)    */
    NB200_GOC_C_COUNT = 8
};
typedef struct nb200_gemnet_oc_weights {
    int32_t num_blocks;
    int32_t n_elem; /* rows of the embedding table */
    float cutoff;   /* cutoff = cutoff_qint = cutoff_aeaint = cutoff_aint */
    int32_t max_neighbors, max_neighbors_qint, max_neighbors_aeaint;
    const float* w;           /* device */
    const int64_t* off_host;  /* host [G_COUNT + I_COUNT*num_blocks + O_COUNT*(num_blocks+1)] */
    const float* scale_host;  /* host [S_COUNT*num_blocks + SO_COUNT*(num_blocks+1)] */
} nb200_gemnet_oc_weights;
/* Bytes of the graph buffer (pair ranks, degrees, CSR row pointers) for a batch. */
int64_t nb200_gemnet_oc_graph_bytes(int32_t n_atoms, int32_t max_atoms_per_mol);
/* Phase 1: nearest-neighbour ranks, degrees and row pointers of the four graphs; SYNCHRONISES once to return the edge counts
 * (the reference synchronises on every `.max()` / mask of its index construction). */
int nb200_gemnet_oc_graph_count(const nb200_gemnet_oc_weights* w, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                                int32_t n_atoms, int32_t max_atoms_per_mol, void* graph_buf, int64_t graph_bytes,
                                int64_t* counts_host, void* stream);
int64_t nb200_gemnet_oc_workspace_bytes(const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
/* Phase 2: edge lists + geometry, bases, embedding, interaction / output blocks, energy[B] and forces[N,3]. */
int nb200_gemnet_oc_energy_forces(nb200_engine* eng, const nb200_gemnet_oc_weights* w, const int32_t* z, const float* pos,
                                  const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol,
                                  void* graph_buf, int64_t graph_bytes, const int64_t* counts_host, void* workspace,
                                  int64_t workspace_bytes, float* energy, float* forces, void* stream);
/* Asynchronous form for loops that must not wait for the host (geometry optimisation): graph phase and model phase in ONE enqueue, no
 * stream synchronisation, no device-to-host copy.  Arrays, grids and GEMMs are sized by UPPER BOUNDS of the five counts that follow from
 * the molecule sizes alone, so they hold for every geometry of the batch (DESIGN.md 3.9):
 *   nb200_gemnet_oc_count_bounds: pure host function; mol_ptr_host[n_mol + 1] -> counts_bound_host[NB200_GOC_C_COUNT].  NB200_EINVAL for an empty
 *   molecule, a mol_ptr that does not start at 0, or a bound beyond int32.
 *   nb200_gemnet_oc_energy_forces_async: workspace_bytes >= nb200_gemnet_oc_workspace_bytes(.., counts_bound_host).  The real counts stay on the
 *   device; `status` is a device int32[8] rewritten by every call:
 *     {main-graph edges, error code, max main-graph degree, atoms without a main-graph neighbour,   (words 0-3 as nb200_painn_energy_forces)
 *      a2a edges, a2ee2a edges, qint edges, input-triplet slots}.
 *   Error codes in status[1]: NB200_ECAPACITY a count exceeds its bound (nothing is written past a bound), NB200_ENOEDGES no main-graph edge,
 *   NB200_EINVAL a non-finite coordinate.  With an error every energy and force of the call is NaN.  Same energies and forces as the two-phase
 *   form. */
int nb200_gemnet_oc_count_bounds(const nb200_gemnet_oc_weights* w, const int32_t* mol_ptr_host, int32_t n_mol, int64_t* counts_bound_host);
int nb200_gemnet_oc_energy_forces_async(nb200_engine* eng, const nb200_gemnet_oc_weights* w, const int32_t* z, const float* pos,
                                        const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol,
                                        void* graph_buf, int64_t graph_bytes, const int64_t* counts_bound_host, void* workspace,
                                        int64_t workspace_bytes, float* energy, float* forces, int32_t* status, void* stream);
/* Training (config/model/gemnet-oc.yaml trains with DIRECT forces: first-order back-propagation from dLoss/dE and dLoss/dF, the reference's
 * `loss.backward()` through GemNetOC.forward, gemnet_oc.py:1121-1251 + GemNetOCLightning.step 1361-1371).  Same two-phase protocol:
 * nb200_gemnet_oc_graph_count, then nb200_gemnet_oc_train_workspace_bytes (every activation is kept, mirrored by a gradient arena), then
 * nb200_gemnet_oc_energy_forces_grads: energy[B], forces[N,3] and
 *     grads[n_weights] = d( sum_m energy_seed[m] E_m + sum_i force_seed[i] . F_i ) / d(w->w)      (flat, same layout as the weights)
 * zeroed by the call.  Both seeds NULL = forward only.  FIRST CORRECT PATH, verified under host emulation only (csrc/gemnet_oc_train.inc). */
int64_t nb200_gemnet_oc_train_workspace_bytes(const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
int nb200_gemnet_oc_energy_forces_grads(nb200_engine* eng, const nb200_gemnet_oc_weights* w, int64_t n_weights, const int32_t* z,
                                        const float* pos, const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol,
                                        void* graph_buf, int64_t graph_bytes, const int64_t* counts_host, void* workspace,
                                        int64_t workspace_bytes, const float* energy_seed, const float* force_seed, float* grads,
                                        float* energy, float* forces, int64_t* keep_token_host, void* stream);
/* Two-call form for autograd (forward now, seeds later, no forward recompute): call the function above with both seeds NULL, `grads` given
 * and keep_token_host != NULL -- the engine keeps the tape and returns a token; then nb200_gemnet_oc_backward(eng, token, seeds) fills that
 * `grads` buffer.  NB200_EINVAL if the engine no longer holds that forward (another training forward ran on it): re-run the one-call form. */
int nb200_gemnet_oc_backward(nb200_engine* eng, int64_t token, const float* energy_seed, const float* force_seed, void* stream);
/* Force-Jacobian products (csrc/gemnet_oc_jvp.inc, DESIGN.md 3.9.1): for each of n_dir position-space directions v[d] ([n_atoms,3], Angstrom)
 *   jv[d] = -(dF/dR) v[d]   in Ha/A, F the direct forces,
 * exact (one forward-mode pass through the training forward, no finite step), fp32.  The forces are not a gradient, so this Jacobian is not
 * symmetric; ASE's `Vibrations` reports the symmetric part of the same matrix.  Same two-phase protocol: nb200_gemnet_oc_graph_count, then
 * nb200_gemnet_oc_jvp_workspace_bytes for the exact counts.  energy[n_mol] and forces[n_atoms,3] (NULL => not written) are bitwise those of
 * nb200_gemnet_oc_energy_forces_grads with both seeds NULL.  The primal pass runs once per call, the directions one after another, so the
 * workspace does not depend on n_dir.  No atomics: bitwise repeatable and independent of how the directions are split into calls.  The graph
 * is that of `pos`: membership is piecewise constant and not differentiated.  NB200_EINVAL (nothing launched) for a NULL required pointer,
 * n_dir < 1, counts above the graph capacity, or a short graph buffer or workspace; NB200_ENOEDGES for a batch without main-graph edges. */
int64_t nb200_gemnet_oc_jvp_workspace_bytes(const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
int nb200_gemnet_oc_jvp(nb200_engine* eng, const nb200_gemnet_oc_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                        int32_t n_mol, int32_t n_atoms, int32_t max_atoms_per_mol, void* graph_buf, int64_t graph_bytes,
                        const int64_t* counts_host, void* workspace, int64_t workspace_bytes, int32_t n_dir, const float* v,
                        float* energy, float* forces, float* jv, void* stream);
/* Debug / parity hooks: copies of the per-atom embedding h [N,256] after the last interaction block (NULL = skip). */
int nb200_gemnet_oc_debug_h(const void* workspace, const nb200_gemnet_oc_weights* w, int32_t n_mol, int32_t n_atoms,
                            const int64_t* counts_host, float* h_out, void* stream);
/* Test entry point, not a supported API: one edge aggregation of the GemNet-OC interaction block on caller-built graphs (CSR rows by target,
 * sources ascending, unit vectors V source -> target).
 *   quad = 0, triplet:    O[e, 64 i + ch] = sum_s R[e, 7 i + s] sum over k in in-row(tgt e), in.src[k] != src e of Y_s(V_e . V_k) x[k, ch]
 *                         (o, in) = (main, main) or (main, a2ee2a); o needs src, tgt, V; in needs ptr, src, V; ldr >= 112.
 *   quad = 1, quadruplet: o = the main graph (ptr, src, tgt, V), in = the qint graph (ptr, src, V), q_tin[qint edges] the input-triplet slot
 *                         bases, x = x_t [slots, 32]; O[e, 32 i + ch] as the QuadrupletInteraction sums it; ldr >= 1568.
 * O is [E_bound, 1024].  form = 0: the host dispatch the model calls (the warp-per-edge device kernels); form = 1: the one-thread-per-output
 * functor the training forward runs.  tangent = 1: the forward-mode tangent Ot of O for the tangents Vot, Vit of the two graphs' V, xt of x
 * and Rt of R (O is not written).  E_dev (primal only, may be NULL): the row count in device memory, E_bound then an upper bound; rows at or
 * past min(*E_dev, E_bound) are not written.  NB200_EINVAL (nothing launched) for a NULL required pointer, E_bound < 0, a short ldr, or
 * E_dev with tangent = 1.  The emulation build runs the functor for both forms. */
typedef struct nb200_gemnet_oc_agg_args {
    int32_t quad, form, tangent, ldr;
    int64_t E_bound;
    const int32_t* E_dev;
    const int32_t *o_ptr, *o_src, *o_tgt;
    const float* o_V;
    const int32_t *in_ptr, *in_src;
    const float* in_V;
    const int32_t* q_tin;
    const float *x, *R;
    float* O;
    const float *Vot, *Vit, *xt, *Rt;
    float* Ot;
} nb200_gemnet_oc_agg_args;
int nb200_gemnet_oc_test_aggregate(const nb200_gemnet_oc_agg_args* args, void* stream);

/* ----------------------------------------------------------------------------------------
 * DimeNet++ energy + conservative forces, config/model/dimenetplusplus.yaml: DimeNetPlusPlusPotential
 * (nablaDFT/dimenetplusplus/dimenetplusplus.py:22-113) around torch_geometric.nn.models.DimeNetPlusPlus (2.4.0).
 * energy[m] = scale * y_m + mean, forces = -dy/dpos of the UNSCALED prediction y (dimenetplusplus.py:97-112); scale = 1, mean = 0
 * without postprocessing.  nb200_dimenet_energy_forces runs a reverse pass through output blocks, interaction blocks, the triplet
 * aggregation and the bases; its sums are gathers (no atomics), so two calls on the same input are bitwise equal (DESIGN.md 3.15).
 * nb200_dimenet_train_grads gives the parameter gradients of an energy and force loss, nb200_dimenet_hvp Hessian-vector products.
 * Supported: hidden 256, int_emb 64, basis_emb 8, out_emb 256, num_spherical 7, num_radial 6, before / after skip 1 / 2, 3 output
 * layers, envelope exponent 5, 1 <= num_blocks <= 16, 2 <= node_latent_dim (= out_channels) <= 64, 1 <= max_neighbors <= 64;
 * anything else is NB200_EUNSUPPORTED.
 * Weights: one flat device buffer `w`, host offsets (floats) in the order
 *   [NB200_DPP_G_*][NB200_DPP_I_* x num_blocks][NB200_DPP_O_* x (num_blocks + 1)]. */
enum {
    NB200_DPP_G_FREQ = 0,  /* [6]       rbf.freq                                                             */
    NB200_DPP_G_ZEROS,     /* [42]      z_ln, first 6 zeros of j_l, l-major (SphericalBasisLayer)             */
    NB200_DPP_G_NORMS,     /* [42]      N_ln = 1 / sqrt(0.5 j_{l+1}(z_ln)^2)                                 */
    NB200_DPP_G_EMB_TI,    /* [95,256]  emb.lin.weight[:, 0:256] . emb.emb.weight[z] + emb.lin.bias (target)  */
    NB200_DPP_G_EMB_TJ,    /* [95,256]  emb.lin.weight[:, 256:512] . emb.emb.weight[z] (source)              */
    NB200_DPP_G_EMB_RBF_W, /* [256,6]   emb.lin_rbf.weight                                                   */
    NB200_DPP_G_EMB_RBF_B, /* [256]     emb.lin_rbf.bias                                                     */
    NB200_DPP_G_EMB_W3,    /* [256,256] emb.lin.weight[:, 512:768]                                           */
    NB200_DPP_G_HEAD_W0, NB200_DPP_G_HEAD_B0, /* regr_or_cls_nn.0  [L,L], [L]          */
    NB200_DPP_G_HEAD_W1, NB200_DPP_G_HEAD_B1, /* regr_or_cls_nn.2  [L/2,L], [L/2]      */
    NB200_DPP_G_HEAD_W2, NB200_DPP_G_HEAD_B2, /* regr_or_cls_nn.4  [L/2,L/2], [L/2]    */
    NB200_DPP_G_HEAD_W3, NB200_DPP_G_HEAD_B3, /* regr_or_cls_nn.6  [1,L/2], [1]        */
    NB200_DPP_G_COUNT
};
enum { /* per interaction block */
    NB200_DPP_I_RBF = 0, /* [256,6]  lin_rbf2.weight . lin_rbf1.weight */
    NB200_DPP_I_SBF,     /* [64,42]  lin_sbf2.weight . lin_sbf1.weight */
    NB200_DPP_I_SBF1,    /* [8,42]   lin_sbf1.weight                   */
    NB200_DPP_I_SBF2,    /* [64,8]   lin_sbf2.weight                   */
    NB200_DPP_I_JI_W, NB200_DPP_I_JI_B, NB200_DPP_I_KJ_W, NB200_DPP_I_KJ_B, /* [256,256], [256] */
    NB200_DPP_I_DOWN,    /* [64,256] */
    NB200_DPP_I_UP,      /* [256,64] */
    NB200_DPP_I_RES_W,   /* 6 x [256,256]: layers_before_skip.0.lin{1,2}, layers_after_skip.{0,1}.lin{1,2} */
    NB200_DPP_I_RES_B,   /* 6 x [256] */
    NB200_DPP_I_LIN_W, NB200_DPP_I_LIN_B,
    NB200_DPP_I_COUNT
};
enum { /* per output block */
    NB200_DPP_O_RBF = 0, /* [256,6]   lin_rbf      */
    NB200_DPP_O_UP,      /* [256,256] lin_up       */
    NB200_DPP_O_LINS_W,  /* 3 x [256,256] lins.*   */
    NB200_DPP_O_LINS_B,  /* 3 x [256]              */
    NB200_DPP_O_LIN,     /* [L,256]   lin          */
    NB200_DPP_O_COUNT
};
enum { NB200_DPP_C_EDGES = 0, NB200_DPP_C_TRIPLETS, NB200_DPP_C_COUNT = 4 }; /* counts_host[] of nb200_dimenet_graph_count */
typedef struct nb200_dimenet_weights {
    int32_t num_blocks, node_latent_dim, hidden, int_emb, basis_emb, out_emb, num_spherical, num_radial;
    int32_t num_before_skip, num_after_skip, num_output_layers, envelope_exponent, max_neighbors;
    float cutoff, scale, mean;
    const float* w;          /* device */
    const int64_t* off_host; /* host [G_COUNT + I_COUNT*num_blocks + O_COUNT*(num_blocks+1)] */
} nb200_dimenet_weights;
/* Bytes of the graph buffer for n_atoms (CSR by target with the radius_graph truncation: candidates in ascending index with d^2 < cutoff^2,
 * the target included, the first max_neighbors + 1 kept, the self loop dropped; the by-source permutation; triplet offsets). */
int64_t nb200_dimenet_graph_bytes(const nb200_dimenet_weights* w, int32_t n_atoms);
/* Phase 1: builds the graph from pos and SYNCHRONISES once; counts_host[NB200_DPP_C_COUNT] = {edges, triplets, 0, 0}.
 * NB200_EINVAL for z outside [0, 94] or a non-finite coordinate.  An atom without neighbours is not an error. */
int nb200_dimenet_graph_count(const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr, int32_t n_mol,
                              int32_t n_atoms, void* graph_buf, int64_t graph_bytes, int64_t* counts_host, void* stream);
int64_t nb200_dimenet_workspace_bytes(const nb200_dimenet_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
/* Phase 2 (same z, pos, mol_ptr and graph buffer as phase 1): energy[n_mol], forces[n_atoms,3] and, when graph_emb != NULL, the
 * per-molecule sums of the output blocks graph_emb[n_mol, node_latent_dim] (the input of regr_or_cls_nn). */
int nb200_dimenet_energy_forces(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                                int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes, const int64_t* counts_host,
                                void* workspace, int64_t workspace_bytes, float* energy, float* forces, float* graph_emb, void* stream);
/* Asynchronous form for loops that must not wait for the host (relaxation, molecular dynamics): graph phase and energy-and-forces pass in
 * ONE enqueue, no stream synchronisation, no device-to-host copy (DESIGN.md 3.15.3).
 *   nb200_dimenet_count_bounds: pure host function; mol_ptr_host[n_mol + 1] -> bounds[NB200_DPP_C_COUNT] = {edges, triplet slots, 0, 0},
 *   upper bounds that hold for every geometry of molecules of these sizes.  NB200_EINVAL for a mol_ptr that does not start at 0 or does not
 *   increase, or a bound beyond int32.
 *   nb200_dimenet_energy_forces_async: graph_bytes >= nb200_dimenet_graph_bytes(w, n_atoms), workspace_bytes >=
 *   nb200_dimenet_workspace_bytes(w, n_mol, n_atoms, bounds).  Edge rows and GEMMs are sized by the bounds and stop at the counts, which stay
 *   on the device; `status` is a device int32[8] rewritten by every call:
 *     {edges, error code, max in-degree, atoms without a neighbour, triplet slots, 0, 0, 0}   (words 0-3 as nb200_painn_energy_forces)
 *   Error codes in status[1]: NB200_ECAPACITY a count exceeds its bound, NB200_EINVAL z outside [0, 94] or a non-finite coordinate; both
 *   are found before any edge or triplet row is written, nothing is written past a bound, and every energy and force of the call is NaN.
 *   An atom without neighbours and a batch without edges are not errors.  Energies and forces are those of the two-phase form. */
int nb200_dimenet_count_bounds(const nb200_dimenet_weights* w, const int32_t* mol_ptr_host, int32_t n_mol, int64_t* bounds);
int nb200_dimenet_energy_forces_async(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos,
                                      const int32_t* mol_ptr, int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes,
                                      const int64_t* bounds, void* workspace, int64_t workspace_bytes, float* energy, float* forces,
                                      int32_t* status, void* stream);
/* Training (DESIGN.md 3.15.1): bytes of the workspace of nb200_dimenet_train_grads (the inference workspace plus the tangent arrays). */
int64_t nb200_dimenet_train_workspace_bytes(const nb200_dimenet_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
/* Parameter gradients of a loss L(E, F) (same z, pos, mol_ptr, graph buffer and counts as phase 1): given the seeds
 * seed_energy[n_mol] = dL/dE and seed_forces[n_atoms,3] = dL/dF (either may be NULL), writes
 *   grads = sum_m seed_energy[m] scale dy_m/dw + sum_i seed_forces[i] . dF_i/dw
 * into `grads`, a buffer with the layout and offsets of the weight buffer (zeroed first, up to the end of the last entry).  Entries y does not
 * read (ZEROS, NORMS, SBF1, SBF2) stay zero; the folded entries (I_RBF, I_SBF, EMB_TI, EMB_TJ) get the gradient w.r.t. the folded matrix.
 * One call recomputes the forward, runs the unit-seed reverse pass and, with seed_forces, its tangent along seed_forces (forward-over-
 * reverse).  Weight-gradient sums use atomics: two calls agree to rounding, not bitwise.  NB200_EINVAL for a NULL pointer (seeds excepted),
 * a short workspace or graph buffer; NB200_EUNSUPPORTED for a configuration outside the list above. */
int nb200_dimenet_train_grads(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                              int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes, const int64_t* counts_host,
                              void* workspace, int64_t workspace_bytes, const float* seed_energy, const float* seed_forces, float* grads,
                              void* stream);
/* Test entry point, not a supported API: the spherical radial basis env(x) N_ln j_l(z_ln x), x = dist / cutoff, and its derivative
 * with respect to dist, [n, 42] each, as the engine evaluates them in fp32. */
int nb200_dimenet_debug_sbf_radial(const nb200_dimenet_weights* w, const float* dist, int32_t n, float* rbs, float* drbs, void* stream);
/* Hessian-vector products (csrc/dimenet_hvp.inc, DESIGN.md 3.15.2): for each of n_dir position-space directions v[d] ([n_atoms,3], Angstrom)
 *   hv[d] = -(dF/dR) v[d] = (d^2 y / dR dR) v[d]   in Ha/A, y the UNSCALED prediction (the forces' y; the scaler touches the energy only),
 * exact (forward-over-reverse, no finite step), fp32.  Same z, pos, mol_ptr, graph buffer and counts as phase 1.  energy[n_mol] (scaled)
 * and forces[n_atoms,3] (NULL => not written) are bitwise those of nb200_dimenet_energy_forces.  The primal pass runs once per call, the
 * directions one after another, so the workspace does not depend on n_dir.  No atomics: bitwise repeatable and independent of how the
 * directions are split into calls.  NB200_EINVAL (nothing launched) for a NULL required pointer, n_dir < 1, counts above the graph capacity,
 * or a short graph buffer or workspace; NB200_EUNSUPPORTED for a configuration outside the list above. */
int64_t nb200_dimenet_hvp_workspace_bytes(const nb200_dimenet_weights* w, int32_t n_mol, int32_t n_atoms, const int64_t* counts_host);
int nb200_dimenet_hvp(nb200_engine* eng, const nb200_dimenet_weights* w, const int32_t* z, const float* pos, const int32_t* mol_ptr,
                      int32_t n_mol, int32_t n_atoms, void* graph_buf, int64_t graph_bytes, const int64_t* counts_host,
                      void* workspace, int64_t workspace_bytes, int32_t n_dir, const float* v, float* energy, float* forces,
                      float* hv, void* stream);
/* Test entry point, not a supported API: the second distance derivatives of the radial bases, d2rbs [n, 42] of env(x) N_ln j_l(z_ln x) and
 * d2rbf [n, 6] of env(x) sin(freq_n x), x = dist / cutoff, as the Hessian-vector pass evaluates them in fp32. */
int nb200_dimenet_debug_sbf_radial_d2(const nb200_dimenet_weights* w, const float* dist, int32_t n, float* d2rbs, float* d2rbf, void* stream);

/* ----------------------------------------------------------------------------------------
 * PhiSNet Clebsch-Gordan mixing layers (SURVEY.md section 8 f4).  Features are component-major:
 * x[rows][(order+1)^2][F], component index l*l + m (m = 0..2l), F in {32, 64, 96, 128}, orders <= 4.
 * Real CG tensors = the reference's vendored table (phisnet/nn/modules/clebsch_gordan_coefficients_L10.npz).
 *   nb200_phis_n_paths      number of (l1, l2, L) paths in the reference's loop order
 *                           (pair_mixing.py:28-36; strict_upper = 1: l1 < l2, self_mixing.py:18-25)
 *   nb200_phis_pair_mixing  PairMixing.forward (pair_mixing.py:47-69); coeff[rows][n_paths][F] = rbf . W_path^T
 *                           (one dense layer for all paths: nb200_dense)
 *   nb200_phis_self_mixing  SelfMixing.forward (self_mixing.py:55-83); mixcoeff[n_paths][F], keepcoeff[min(oi,oo)+1][F]
 *   nb200_phis_linear       the per-order Linear of SphericalLinear.forward (spherical_linear.py:50-59);
 *                           W_l[order+1][c_in][c_out] (transposed nn.Linear weights), bias[c_out] on component 0 or NULL
 * -------------------------------------------------------------------------------------- */
int nb200_phis_n_paths(int32_t order_in1, int32_t order_in2, int32_t order_out, int32_t strict_upper);
int nb200_phis_pair_mixing(const float* x1, const float* x2, const float* coeff, int32_t n_rows, int32_t n_feat,
                           int32_t order_in1, int32_t order_in2, int32_t order_out, float* y, void* stream);
int nb200_phis_self_mixing(const float* x, const float* mixcoeff, const float* keepcoeff, int32_t n_rows, int32_t n_feat,
                           int32_t order_in, int32_t order_out, float* y, void* stream);
int nb200_phis_linear(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in, int32_t c_out,
                      int32_t order, float* y, void* stream);

/* PhiSNet model forward (csrc/phisnet_model.cu, neural_network.py:717-995); order 4, features [rows][25][F].  Pair rows follow the full
 * CSR graph of nb200_neighbor_build (target-major, sources ascending = the reference's fill_idx order).
 *   nb200_phis_swish_self_mixing  SelfMixing(4, 4) of swish(x) (swish on component 0 only; alpha = beta = NULL: no swish)
 *   nb200_phis_linear_ex          nb200_phis_linear with accumulate (y += x . W_l): the residual add of ResidualBlock
 *   nb200_phis_interaction        y[i] = yi[i] + sum_j PairMixing(yj[j], angular_fn1(sh)) + radial_fn(rbf) angular_fn2(sh) yj[j]_0;
 *                                 coeff[P][70][F] = rbf . [65 mixing paths, 5 radial_fn]^T; wa*[5][F], ba*[F] = angular_fn Linear(1, F)
 *   nb200_phis_pair_features      fii[i] = fpc[i] + sum_j radial_ii(rbf) fpn[j];  fij[e] = mix_ij(fpc[i], fpc[j]) + sum_{k != i,j}
 *                                 radial_ij(rbf_ik) fpn[k]; coeff[P][75][F] = rbf . [65 mix_ij paths, 5 radial_ii, 5 radial_ij]^T
 *   nb200_phis_overlap_pairs      s[e] = mix_s(x[i], (x[j]_0, angular_fn(sh)_{L>0})); coeff[P][65][F]; wa[5][F]
 *   nb200_phis_assemble           output heads + matrix assembly: per block, only the irreps it uses, sum_f X[L][m][f] W_L[c][f] (+bias),
 *                                 contracted with sqrt(2L+1) CG(l_i, l_j, L); writes B + B^T into per-molecule matrices M (offsets mol_off);
 *                                 W[5][n_col][F] (nn.Linear weights), element / shell / entry tables built on the host (nabladft_b200/phisnet.py)
 */
int nb200_phis_swish_self_mixing(const float* x, const float* alpha, const float* beta, const float* mixcoeff, const float* keepcoeff,
                                 int32_t n_rows, int32_t n_feat, float* y, void* stream);
int nb200_phis_linear_ex(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in, int32_t c_out, int32_t order,
                         int32_t accumulate, float* y, void* stream);
int nb200_phis_interaction(const float* yi, const float* yj, const float* sh, const float* coeff, const float* wa1, const float* ba1,
                           const float* wa2, const float* ba2, const int32_t* row_ptr, const int32_t* col, int32_t n_atoms, int32_t n_feat,
                           float* y, void* stream);
int nb200_phis_pair_features(const float* fpc, const float* fpn, const float* coeff, const int32_t* row_ptr, const int32_t* col,
                             int32_t n_atoms, int32_t n_feat, float* fii, float* fij, void* stream);
int nb200_phis_overlap_pairs(const float* x, const float* sh, const float* coeff, const float* wa, const int32_t* row_ptr,
                             const int32_t* col, int32_t n_atoms, int32_t n_feat, float* s, void* stream);
int nb200_phis_assemble(const float* Xd, const float* Xo, const float* Wd, const float* bd, int32_t n_col_d, const float* Wo, const float* bo,
                        int32_t n_col_o, int32_t n_feat, const int32_t* atom_el, const int32_t* row_orb, const int32_t* row_m,
                        const int32_t* orb_l, const int32_t* n_rows, const int32_t* ent_range, const int32_t* op_base, const int32_t* ent_col,
                        const int32_t* ent_L, int32_t n_el, int32_t max_ent, const int32_t* tgt, const int32_t* col, const int32_t* rev,
                        int32_t n_atoms, int32_t n_pairs, const int32_t* atom_mol, const int32_t* atom_off, const int64_t* mol_off,
                        const int32_t* mol_norb, int32_t unit_diagonal, float* M, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NABLA_B200_H */
